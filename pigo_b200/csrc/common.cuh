// common.cuh -- shared device/host structures of libpigo_b200 (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pigo_b200.h"

namespace pigo {

// One entry of the scale ladder of RunCascade (core/pigo.go:226-231,:255), computed on the host
// in float64 exactly like the reference; the kernels only consume the resulting integers.
struct ScaleEntry {
  int32_t s;        // window size "scale"
  int32_t step;     // int(max(ShiftFactor*scale, 1))
  int32_t off;      // scale/2 + 1
  int32_t nrows;    // grid rows  : floor((Rows-2*off)/step)+1 (0 if empty)
  int32_t ncols;    // grid cols
  uint32_t wbase;   // index of this scale's first window in the frame's emission order
  uint32_t nwin;    // nrows*ncols
  uint32_t pad;     // gather role: index of this scale's first 16x16-window block among the gather scales
};

// Face cascade tables on the device.  `codes` keeps the reference's in-memory layout
// (core/pigo.go:79-86): 4 zero bytes, then 4*2^d-4 int8 codes per tree, so node idx (1-based heap)
// sits at byte 4*idx of its tree.  Everything is read-only after pigo_cascade_create.
struct FaceTables {
  const int8_t* codes;   // [ntrees][4*leaves]
  const float* preds;    // [ntrees][leaves]
  const float* thresh;   // [ntrees]
  const uint8_t* blocks; // depth 6: the block-interleaved copy read by the unrotated deep walk (kBlockBytes, below); else null
  int32_t depth, ntrees, leaves;
};

// Block-interleaved copy of a depth-6 cascade, for lane groups that walk 8 consecutive trees of one window.  Block b holds
// trees 8b..8b+7, tree 8b+k in slot k (pad slots of the last block repeat the last tree):
//   bytes 0..31          thresh of slot k at 4k
//   bytes 32..63         root code word (node 1) of slot k at 32 + 4k
//   bytes 64p..64p+63    p = 1..63: for slot k at 64p + 8k, the int2 of node p's two children -- code words 2p, 2p+1 for
//                        p < 32, leaves preds[2p-64], preds[2p-63] for p >= 32
// A 128-byte line holds the records of two nodes, so the 8 lanes of a group step read one line for the thresholds, the roots
// and the first level, then at most 1, 2, 4, 8, 8 lines for the five other levels, where each load of the reference layout
// (codes[t][256 B], preds[t][256 B]) touches 8 lines.  Thresholds and walks stay the reference's numbers, bit for bit.
constexpr int kBlockTrees = 8;
constexpr int kBlockBytes = 4096;

// Unsorted detection as produced by the scan kernels: the in-frame window index doubles as the
// sort key that restores the reference's emission order (scale, row, col).
struct RawDet {
  uint32_t wid;
  float q;
};

// A window whose evaluation continues in the deep kernel from tree `tree` with partial score `acc`.
struct DeepItem {
  uint32_t wid;
  uint32_t frame_si;   // frame (low 16 bits: < 65536 frames per call) | ladder entry (high 16 bits), so that the consumer needs no search
  int32_t tree;
  float acc;
};
__host__ __device__ __forceinline__ uint32_t pack_frame_si(int frame, int si) { return (uint32_t)frame | ((uint32_t)si << 16); }

// Rotated scan (core/pigo.go:150-191).  65536*r + qcos*c0 - qsin*c1 is clamped at 0 and THEN shifted (:167), and
//   max(0, 65536*r + x) >> 16  ==  max(0, r + (x >> 16))     for every integer r, x  (65536*r is a multiple of 65536),
// so a node's four sample coordinates are r + dr1, c + dc1, r + dr2, c + dc2 clamped to [0, nrows-1] (BOTH with nrows-1:
// the reference's column clamp quirk, :168,:171), where the four deltas depend only on (scale, table slot, node).
struct RotNode {
  int16_t dr1, dc1, dr2, dc2;
};

// One image of a mixed-size call (pigo_run_cascade_images).  Every image's ladder is a prefix of the call's longest ladder
// (off = s/2+1 never decreases, so the entries that fit an image come first), so ladder index si means the same
// (s, step, off) in every image and one rotated node table per table slot serves them all; only nrows/ncols/wbase/pad differ.
struct ImageDesc {
  const uint8_t* base;   // the image's pixels on the device, `dim` bytes per row
  int32_t rows, cols, dim;
  int32_t nscales;       // length of this image's ladder (a prefix of the longest ladder of the call)
  uint32_t plan_off;     // index of the image's first ScaleEntry in the call's concatenated plan
  uint32_t block_base;   // index of the image's first gather block in its group (ScaleEntry.pad counts within the image)
  uint32_t rot_off;      // rotated scan: the image's node table in ScanArgs.rot_tab, in units of 64 RotNode records
  int32_t rot_slot;      // the image's table slot int(32*a) (-1 = unrotated): RunDetector with PupWork.rot_slot == kRotSlotPerImage
  int32_t out_index;     // scan: the image's index in the caller's arrays (finalize writes its results there)
};

// PupWork.rot_slot / puploc_kernel's rot_slot of a call whose images each carry their own angle (ImageDesc.rot_slot).
constexpr int kRotSlotPerImage = -2;
constexpr int kRotSlotPerFace = -3;    // angle sweep: RunDetector with PupWork.face_rot[slot / stride]

struct ScanArgs {
  FaceTables tab;
  const uint8_t* frames;
  size_t frame_stride;
  int32_t nframes, rows, cols, dim;
  const ScaleEntry* plan;
  int32_t nscales;
  uint32_t wins_per_frame;
  // rotated path (angle > 0): table slot int(32*a), core/pigo.go:159-160
  int32_t rot_slot;  // -1 = unrotated
  // rotated path, table-driven kernels: per (ladder entry, tree, node) the four sample offsets of classifyRotatedRegion
  // (core/pigo.go:167-171) precomputed for this call's slot; nullptr = not built (universal gather kernel computes them)
  const RotNode* rot_tab;
  // outputs
  RawDet* raw;          // [nframes][cap]
  int32_t* raw_count;   // [nframes]
  int32_t cap;
  // work distribution
  unsigned long long* chunk_counter;
  uint32_t chunk;             // windows per chunk
  uint32_t chunks_per_frame;
  // gather-kernel window filter: only scales with index in [scale_lo, scale_hi) (tiled kernel takes the rest)
  int32_t scale_lo, scale_hi;
  int32_t batch_frames;       // frames of the whole API call (group-independent choices: gather block edge, deep group width)
  // Q2 "long" queue: windows that survived the shared-memory-resident trees, and the stragglers a tile warp still had alive
  // when it drained its tile (any tree index).  Consumed one item per lane group (GROUP trees evaluated in parallel) by the
  // deep kernel, which bounds the serial chain of a full survivor.
  DeepItem* longq;
  unsigned int* long_count;
  uint32_t long_cap;
  uint32_t frame_base;        // index of this group's first frame in the API call (for `ready`)
  // Host frames streamed in while the scan runs: *ready = number of leading frames of the call whose H2D copy has completed
  // (written by the copy stream after every chunk); a warp waits for its frame before it touches it.  nullptr = resident.
  const unsigned int* ready;
  // Mixed-size call: the group's images (frame index = image index in the group); `plan` is the concatenated per-image
  // plan and rows/cols/dim/frames/frame_stride are unused by the kernels' image-table variants.  nullptr = uniform batch.
  const ImageDesc* images;
  int32_t nimages;
};

// Waits until frame `need - 1` of the call has arrived (lane 0 polls with acquire semantics, the warp follows).
__device__ __forceinline__ void wait_frames(const unsigned int* ready, unsigned need) {
  if (ready == nullptr) return;
  if ((threadIdx.x & 31) == 0) {
    unsigned have;
    for (;;) {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(have) : "l"(ready) : "memory");
      if (have >= need) break;
      __nanosleep(256);
    }
  }
  __syncwarp();
}

// ---- tiled kernel -------------------------------------------------------------------------------------------
constexpr int kTiledMaxThreads = 1024;
// Tree record of the shared-memory table: 256 B node codes (node idx at byte 4*idx) | 64 f32 leaves | f32 threshold |
// 4 B pad = 520 B.  8-byte multiple so that the two children of a node (bytes 8*idx..8*idx+7, codes or -- for the last
// level -- leaves) can be fetched with one aligned 64-bit load; 130 words skew consecutive trees by two banks.
constexpr int kTreeRec = 520;
constexpr int kMaxBands = 4;
// dense-head kernel: entries of the per-warp survivor ring (12 bytes each), ladder entries with a head table, head trees
constexpr int kRing = 48;
constexpr int kRingEntry = 12;
constexpr int kHeadMaxScales = 16;
constexpr int kHeadTreesMax = 4;

// A band = consecutive ladder entries [scale_lo, scale_lo+nscales) served by one family of pixel tiles.
struct TileBand {
  int32_t scale_lo, nscales;   // <= 32 scales per band (one lane describes one scale)
  int32_t halo_lo;             // pixels needed above/left of a window centre:  ceil(s_max/2)
  int32_t core;                // core edge: a tile owns the windows whose centre lies in its core square
  int32_t org_x;               // x of the first core column; org_x - halo_lo is a multiple of 16
  int32_t tiles_x, ntiles;     // tiles per row / per frame
  int32_t pitch;               // shared-memory row pitch in bytes (multiple of 16)
  int32_t rows_t;              // tile rows: halo_lo + core + halo_hi
  // region role (a CTA-wide region of core x core_y window centres per band): core_y, and the rows of one TMA box of the
  // region's fill (a region is rows_t <= 2 * box_rows rows, filled by ceil(rows_t / box_rows) boxes of pitch x box_rows)
  int32_t core_y, box_rows;
};

// Region role of the fused kernel: every region buffer has this row pitch (= the widest TMA box).  A multiple of 128, it also
// keeps both buffers and every box of a region at the 128-byte alignment TMA tensor copies need.
constexpr int kRegionPitch = 256;
constexpr int kRegionMaxScales = 32;
// One ladder entry's window sub-grid inside a region: windows [start, next start) of the region's scale-major list.
struct RegionSub {
  int32_t start, s, step, nj;
  uint32_t magic;              // ceil(2^32 / nj): k / nj by __umulhi
  uint32_t base;               // shared-memory offset of the sub-grid's first window centre
  uint32_t wid0;               // its in-frame window index
  int32_t ncols;
};
// Control block of one region buffer, written by the warp that fills the buffer before the fill's mbarrier arrive.
struct RegionCtl {
  int32_t n;                   // windows of the region
  int32_t frame;               // -1: no region left for this CTA
  int32_t pad[2];
  RegionSub sub[kRegionMaxScales + 1];   // sub[nscales].start == n
};
// Region control in shared memory: RegionCtl[2], then full[2] and empty[2] mbarriers, the two buffers' dealing cursors and
// the sequence number each buffer is claimed for next (TiledArgs.region_ctl, 8-byte aligned).
constexpr uint32_t kRegionCtlBytes = 2 * sizeof(RegionCtl) + 48;

struct TiledArgs {
  ScanArgs scan;
  const uint8_t* tab_tiled;    // [ntrees] records of kTreeRec bytes
  int32_t ks;                  // trees resident in shared memory
  uint32_t tile_bytes;         // per-warp tile buffer
  int32_t nbands;
  int32_t aligned;             // frames, stride and Dim are 16-byte aligned: tiles are filled with cp.async 16 B
  int32_t tail_min;            // after a tile is drained, slot groups with fewer live items are handed to the deep queue
  TileBand band[kMaxBands];
  uint32_t tiles_per_frame;
  unsigned long long total_tiles;
  // warp specialisation inside the fused kernel
  int32_t tile_warps;                     // warps [0, tile_warps) own pixel tiles; the rest gather
  int32_t gather_scale_lo;                // first ladder entry scanned by the gather warps
  uint32_t gather_blocks_per_frame;       // 16x16-window blocks of those scales (ScaleEntry.pad = block prefix)
  unsigned long long* gather_counter;
  int32_t gb_shift;                       // log2 of the gather block edge in windows (4 -> 16x16, 3 -> 8x8)
  int32_t tile_prefetch;                  // tile role: fetch both children of a node with one 64-bit load
  int32_t gather_ni;                     // windows per lane in the gather role (ILP)
  // dense-head variant of the tile role (scan_head_kernel): the first `head_trees` trees of every tiled ladder entry have a
  // per-scale node table (two precomputed 16-bit sample offsets per node) at shared-memory offset head_off; survivors of the
  // head travel through a per-warp ring (ring_off, kRing entries of 12 bytes) to the generic lane-refill loop
  int32_t head_trees;                     // 0 = classic kernel
  int32_t head_nscales;                   // ladder entries [0, head_nscales) are tiled
  uint32_t head_off, ring_off, tiles_off;
  int32_t use_tmap;                       // tile fill: 1 = one 3-D TMA tensor copy per tile (TileMaps), 0 = one bulk copy per tile row
  int32_t gather_limit;                   // gather role: trees a window walks here before it is handed to the deep kernel (<= ks)
  unsigned long long* stats;              // developer counter (option walk_stats): [0] += live lanes, [1] += 1 per tile-role walk iteration
  // per-scale offset tables (scan_ptab_kernel): ptab = [tiled ladder entries][ptab_stride bytes] records of kTreeRec bytes for the
  // first kt trees; rounds = groups of tile_warps consecutive tiles of ONE band, strided statically over the CTAs
  const uint8_t* ptab;
  int32_t kt;                             // trees per table (0 = classic kernel)
  uint32_t ptab_stride;                   // bytes per ladder entry in ptab (kt * kTreeRec rounded up to 16)
  uint32_t ptab_off;                      // shared-memory offset of the two table buffers (ptab_stride + 16 bytes apart)
  uint32_t rounds_per_frame;
  uint32_t band_rounds[kMaxBands];
  int32_t head_back;                      // generic phase: with an empty ring and fewer live lanes than this, park them in the ring and go back to the head
  // region role (scan_tiled_kernel<1, 1024, true>): band[] / tiles_per_frame / total_tiles describe regions; two buffers of
  // region_bytes at region_off and region_off + region_bytes, their RegionCtl blocks and barriers at region_ctl
  int32_t region;
  uint32_t region_ctl, region_off, region_bytes;
};

// TMA descriptors of the frame batch, one per tile band (the box = the band's tile: pitch x rows_t x 1 frame), passed to the
// fused kernels as a __grid_constant__ parameter.
struct TileMaps {
  CUtensorMap m[kMaxBands];
};

__device__ __constant__ int c_qcos[33] = {256, 251, 236, 212, 181, 142, 97, 49, 0, -49, -97, -142, -181, -212, -236, -251, -256,
                                          -251, -236, -212, -181, -142, -97, -49, 0, 49, 97, 142, 181, 212, 236, 251, 256};
__device__ __constant__ int c_qsin[33] = {0, 49, 97, 142, 181, 212, 236, 251, 256, 251, 236, 212, 181, 142, 97, 49, 0,
                                          -49, -97, -142, -181, -212, -236, -251, -256, -251, -236, -212, -181, -142, -97, -49, 0};

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// Finds the ladder entry that contains in-frame window index `wid` (binary search over wbase).
__device__ __forceinline__ int find_scale(const ScaleEntry* __restrict__ plan, int nscales, uint32_t wid) {
  int lo = 0, hi = nscales - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (__ldg(&plan[mid].wbase) <= wid) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- mbarrier + TMA helpers (bulk copy of cascade records, tensor copy of pixel tiles) ---------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
// One tile = one 3-D tensor copy (x = byte column, y = row, z = frame); out-of-frame parts of the box are zero-filled and
// count towards the transaction bytes, so the barrier always expects the whole box.
__device__ __forceinline__ void tma_tile_g2s(uint32_t dst, const CUtensorMap* map, int x, int y, int z, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(z), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
// non-blocking test of a barrier phase
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(bar),
      "r"(parity)
      : "memory");
}

}  // namespace pigo
