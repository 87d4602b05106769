// scan_tiled.cu -- the hot kernels of RunCascade's (scale,row,col) grid (core/pigo.go:226-249) with classifyRegion
// (core/pigo.go:113-147): the warp-specialised FUSED kernel (tile warps + gather warps) and the gather-v2 kernel.
//
//  * Fused kernel: persistent CTA (one per SM).  The first KS trees of the cascade (codes, leaves, threshold: one
//    520-byte record per tree, see kTreeRec) are staged ONCE per CTA into
//    shared memory by the TMA bulk engine (cp.async.bulk + mbarrier).
//  * TILE WARPS, one warp per image tile: each warp owns a private pixel-tile buffer in shared memory.  A tile is an
//    image region (core + halo) that serves EVERY scale of a band (20..39 px) at once, so the frame is read from
//    L2/HBM once per band rather than once per scale; it is filled by one TMA bulk copy per (16-byte aligned) tile row
//    completing on the warp's own mbarrier.  Windows whose centre lies in the tile's core are evaluated one-per-lane
//    with LANE REFILL: every iteration each live lane walks ONE tree (6 levels: 1 LDS.32 for the node's 4 codes,
//    2 LDS.U8 pixel gathers); lanes whose window was rejected are re-armed with the next window of the tile via
//    ballot+popc (straight-line fast path), so warps stay full although ~60% of the windows die at tree 0.
//  * Long-lived windows must not pin a tile: whatever is still alive when fewer than `tail_min` windows remain after
//    the tile's list ran out, and any window that survives the KS resident trees, goes to the deep queue Q2 (finished
//    one lane group per window, several trees per step, by deep.cu, which can start a window at any tree).  If the queue
//    is full the lane simply keeps walking (rows beyond KS from global memory): the queue is an optimisation only.
//  * GATHER WARPS (same CTA, same shared cascade prefix): the scales too large for a per-warp tile, in 16x16-window
//    blocks, pixels by ld.global.nc.
//
// Scores are float32 sums in tree order and the result is bit-identical to the reference.
#include <algorithm>

#include "common.cuh"
#include "host.h"

namespace pigo {

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

constexpr uint32_t kCascOff = 384;  // mbarriers live in the first 272 bytes of shared memory, then the scale lookup table
// Window size -> ladder entry, for the queue items of the tile warps (their lanes carry the size, not the index): one byte per
// size < kLutSizes in the control region; 0xff / larger sizes = unknown, the consumer searches the ladder (find_scale).
constexpr uint32_t kLutOff = 272;
constexpr int kLutSizes = 112;
__device__ __forceinline__ int scale_index_of(const uint8_t* smem, int s) {
  const unsigned v = (unsigned)s < (unsigned)kLutSizes ? smem[kLutOff + s] : 0xffu;
  return v == 0xffu ? 0xffff : (int)v;
}
__device__ __forceinline__ int ceil_div_pos(int num, int den) { return num <= 0 ? 0 : (num + den - 1) / den; }



// sign-extended byte k of a packed code word: one PRMT (selector nibble with bit 3 set replicates the sign)
// (prmt.b32 default mode; __byte_perm() documents only 3 selector bits, so the PTX instruction is spelled out)
__device__ __forceinline__ int sx0(int w) { int r; asm("prmt.b32 %0, %1, 0, 0x8880;" : "=r"(r) : "r"(w)); return r; }
__device__ __forceinline__ int sx1(int w) { int r; asm("prmt.b32 %0, %1, 0, 0x9991;" : "=r"(r) : "r"(w)); return r; }
__device__ __forceinline__ int sx2(int w) { int r; asm("prmt.b32 %0, %1, 0, 0xAAA2;" : "=r"(r) : "r"(w)); return r; }
__device__ __forceinline__ int sx3(int w) { return w >> 24; }

// ---- gather role ---------------------------------------------------------------------------------------------
// Warps >= tile_warps of the fused kernel: the scales too large for a shared-memory tile.  Same lane-refill loop
// as scan_gather_kernel, but (a) node codes / leaves / thresholds of the first KS trees come from the shared-memory
// cascade prefix, and (b) work is handed out as 2-D blocks of 16x16 windows of one scale, so that the pixels a
// CTA touches stay L1-resident instead of streaming whole window rows through L2.
// One tree of classifyRotatedRegion (core/pigo.go:164-180) with the node's four sample deltas read from the per-call table
// (RotNode, common.cuh): `tn` = this (scale, tree)'s 64 node records.  Both children of a node are adjacent 8-byte records,
// fetched with one 16-byte load while the node's two pixels are in flight.  Returns the final heap index (64..127).
__device__ __forceinline__ int walk_rot_nodes(const RotNode* __restrict__ tn, const uint8_t* __restrict__ fb, int r, int c, int dim, int lim) {
  uint2 cur = __ldg(reinterpret_cast<const uint2*>(tn + 1));
  int idx = 1;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    uint4 kids = make_uint4(0, 0, 0, 0);
    if (j < 5) kids = __ldg(reinterpret_cast<const uint4*>(tn + 2 * idx));
    // min(nrows-1, max(0, .)) for rows AND columns: the reference's column clamp quirk (core/pigo.go:168,:171)
    const int r1 = __vimin_s32_relu(r + (int)(short)(cur.x & 0xffff), lim), c1 = __vimin_s32_relu(c + ((int)cur.x >> 16), lim);
    const int r2 = __vimin_s32_relu(r + (int)(short)(cur.y & 0xffff), lim), c2 = __vimin_s32_relu(c + ((int)cur.y >> 16), lim);
    const unsigned p1 = __ldg(fb + (size_t)r1 * dim + c1), p2 = __ldg(fb + (size_t)r2 * dim + c2);
    const bool right = p1 <= p2;                       // core/pigo.go:179
    cur = right ? make_uint2(kids.z, kids.w) : make_uint2(kids.x, kids.y);
    idx = 2 * idx + (right ? 1 : 0);
  }
  return idx;
}

// IMG = 1: a mixed-size call (S.images).  The block cursor then maps a global block index to (image, ladder entry, block)
// of the group, and pixels, row pitch and the rotated clamp come from that image; gather_blocks_per_frame holds the
// group's total block count.
template <int NG, int ROT, int IMG = 0>
__device__ __forceinline__ void gather_role(const TiledArgs& A, const uint8_t* smem, uint32_t casc, uint32_t casc_end) {
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const ScanArgs& S = A.scan;
  const FaceTables T = S.tab;
  const unsigned long long total_blocks = IMG ? (unsigned long long)A.gather_blocks_per_frame
                                              : (unsigned long long)A.gather_blocks_per_frame * S.nframes;
  bool blocks_more = total_blocks > 0;
  if (!blocks_more) return;
  const uint32_t tbo_last = casc + (uint32_t)T.ntrees * kTreeRec;   // record offset "one past the last tree"
  const int lim = S.rows - 1;

  // NG independent windows per lane: their dependent LDS -> L2 gather chains overlap (ILP), which is what hides the
  // ~600-cycle L2 latency when only a few gather warps fit beside the tile warps.
  // Per window: unrotated -- pc = centre pixel, sv = scale;  rotated -- pc = frame base, (wr, wc) = centre, sv = index of
  // the (scale, tree) node table in S.rot_tab (units of 64 RotNode records; advances by one per tree).
  bool alive[NG];
  const uint8_t* pc[NG];
  int sv[NG], fr[NG], wr[NG], wc[NG], wsi[NG];   // wsi = ladder entry of the window (travels with queue items)
  uint32_t tbo[NG], wid[NG];
  float acc[NG];
  int dm[NG], lm[NG];   // IMG: row pitch and rotated clamp (rows-1) of the window's image
#pragma unroll
  for (int u = 0; u < NG; ++u) {
    alive[u] = false; pc[u] = S.frames; sv[u] = 0; fr[u] = 0; wr[u] = 0; wc[u] = 0; wsi[u] = 0; tbo[u] = casc; wid[u] = 0; acc[u] = 0.f;
    dm[u] = 0; lm[u] = 0;
  }
  // per-warp block cursor (uniform)
  uint32_t cur = 0, end = 0;
  int b_s = 0, b_step = 0, b_r0 = 0, b_c0 = 0, b_w = 1, b_ncols = 0, cframe = 0, b_si = 0;
  int b_dim = 0, b_lim = 0, b_rot = 0;   // IMG: pitch, rotated clamp and node-table offset of the block's image
  const uint8_t* b_base = S.frames;
  uint32_t b_wid0 = 0;
  bool more = true;

  for (;;) {
    unsigned live_any = 0;
#pragma unroll
    for (int u = 0; u < NG; ++u) {
      unsigned need = __ballot_sync(FULL, !alive[u]);
      while (need && more) {
        if (cur == end) {
          unsigned long long g = 0;
          if (blocks_more) {
            if (lane == 0) g = atomicAdd(A.gather_counter, 1ull);
            g = __shfl_sync(FULL, g, 0);
            if (g >= total_blocks) blocks_more = false;
          }
          if (!blocks_more) {
            more = false;
            break;
          }
          uint32_t bidx;
          const ScaleEntry* plan = S.plan;
          int lo = A.gather_scale_lo, hi = S.nscales - 1;
          if (IMG) {
            // the last image whose first block is <= g (images without windows share their successor's block_base)
            int ilo = 0, ihi = S.nimages - 1;
            while (ilo < ihi) {
              const int mid = (ilo + ihi + 1) >> 1;
              if ((unsigned long long)__ldg(&S.images[mid].block_base) <= g) ilo = mid; else ihi = mid - 1;
            }
            const ImageDesc im = S.images[ilo];
            cframe = ilo;
            bidx = (uint32_t)(g - im.block_base);
            plan = S.plan + im.plan_off;
            lo = 0; hi = im.nscales - 1;
            b_base = im.base; b_dim = im.dim; b_lim = im.rows - 1;
            if (ROT) b_rot = (int)im.rot_off;
          } else {
            cframe = (int)(g / A.gather_blocks_per_frame);
            wait_frames(S.ready, S.frame_base + (unsigned)cframe + 1u);
            bidx = (uint32_t)(g % A.gather_blocks_per_frame);
          }
          while (lo < hi) {                                  // ladder entry whose block range contains bidx
            const int mid = (lo + hi + 1) >> 1;
            if (__ldg(&plan[mid].pad) <= bidx) lo = mid; else hi = mid - 1;
          }
          const ScaleEntry e = plan[lo];
          const uint32_t local = bidx - e.pad;
          const int gsh = A.gb_shift, GB = 1 << gsh;          // block edge in windows: 16 (default) or 8 (small batches)
          const uint32_t nbx = (uint32_t)(e.ncols + GB - 1) >> gsh;
          const uint32_t by = local / nbx, bx = local - by * nbx;
          b_w = min(GB, e.ncols - (int)(bx << gsh));
          const int b_h = min(GB, e.nrows - (int)(by << gsh));
          b_s = e.s; b_step = e.step; b_ncols = e.ncols; b_si = lo;
          b_r0 = e.off + (int)(by << gsh) * e.step;
          b_c0 = e.off + (int)(bx << gsh) * e.step;
          b_wid0 = e.wbase + (by << gsh) * (uint32_t)e.ncols + (bx << gsh);
          cur = 0; end = (uint32_t)(b_w * b_h);
          continue;
        }
        const uint32_t avail = end - cur;
        const uint32_t rank = __popc(need & lanemask_lt());
        if (!alive[u] && rank < avail) {
          const uint32_t k = cur + rank;
          const uint32_t ly = b_w == (1 << A.gb_shift) ? (k >> A.gb_shift) : k / (uint32_t)b_w;
          const uint32_t lx = k - ly * (uint32_t)b_w;
          const int r = b_r0 + (int)ly * b_step, c = b_c0 + (int)lx * b_step;
          wid[u] = b_wid0 + ly * (uint32_t)b_ncols + lx;
          fr[u] = cframe; wsi[u] = b_si;
          const uint8_t* fb = IMG ? b_base : S.frames + (size_t)cframe * S.frame_stride;
          if (ROT) { pc[u] = fb; wr[u] = r; wc[u] = c; sv[u] = (IMG ? b_rot : 0) + b_si * T.ntrees; }
          else { pc[u] = fb + (size_t)r * (IMG ? b_dim : S.dim) + c; sv[u] = b_s; }
          if (IMG) { dm[u] = b_dim; lm[u] = b_lim; }
          tbo[u] = casc; acc[u] = 0.f;
          alive[u] = true;
        }
        cur += min((uint32_t)__popc(need), avail);
        need = __ballot_sync(FULL, !alive[u]);
      }
      live_any |= ~need;
    }
    if (!live_any) break;

    // ---- one tree per live window; dead slots redo tree 0 (unrotated: at their last pixel with s = 0; rotated: the
    //      first node table at their last centre) -- harmless, results ignored
    bool beyond = false;
#pragma unroll
    for (int u = 0; u < NG; ++u) {
      if (!alive[u]) { tbo[u] = casc; sv[u] = 0; }
      beyond |= tbo[u] >= casc_end;
    }
    int idx[NG];
    float pred[NG], thr[NG];
    if (!__any_sync(FULL, beyond)) {
      if (ROT) {
#pragma unroll
        for (int u = 0; u < NG; ++u)
          idx[u] = walk_rot_nodes(S.rot_tab + (size_t)sv[u] * 64, pc[u], wr[u], wc[u], IMG ? dm[u] : S.dim, IMG ? lm[u] : lim);
      } else {
        // plain walk: one 32-bit node load per level from the shared cascade prefix (the node load is ~30 cycles next to a
        // ~600-cycle pixel gather, so prefetching it would only add shared-memory wavefronts to an L1TEX-bound kernel)
#pragma unroll
        for (int u = 0; u < NG; ++u) idx[u] = 1;
#pragma unroll
        for (int j = 0; j < 6; ++j) {
          int cw[NG];
#pragma unroll
          for (int u = 0; u < NG; ++u) cw[u] = *reinterpret_cast<const int*>(smem + tbo[u] + 4 * idx[u]);
          unsigned p1[NG], p2[NG];
#pragma unroll
          for (int u = 0; u < NG; ++u) {
            const int s = sv[u], dim = IMG ? dm[u] : S.dim;
            const int o1 = ((sx0(cw[u]) * s) >> 8) * dim + ((sx1(cw[u]) * s) >> 8);
            const int o2 = ((sx2(cw[u]) * s) >> 8) * dim + ((sx3(cw[u]) * s) >> 8);
            p1[u] = __ldg(pc[u] + o1);
            p2[u] = __ldg(pc[u] + o2);
          }
#pragma unroll
          for (int u = 0; u < NG; ++u) idx[u] = 2 * idx[u] + (p1[u] <= p2[u] ? 1 : 0);
        }
      }
#pragma unroll
      for (int u = 0; u < NG; ++u) {
        pred[u] = *reinterpret_cast<const float*>(smem + tbo[u] + 4 * idx[u]);
        thr[u] = *reinterpret_cast<const float*>(smem + tbo[u] + 512);
      }
    } else {
      // some window is past the resident prefix and could not be handed over (Q2 full): per-slot walk with a table-source
      // switch
#pragma unroll
      for (int u = 0; u < NG; ++u) {
        const bool res = tbo[u] < casc_end;
        const int tv = (int)((tbo[u] - casc) / kTreeRec);
        int ix = 1;
        if (ROT) {
          ix = walk_rot_nodes(S.rot_tab + (size_t)sv[u] * 64, pc[u], wr[u], wc[u], IMG ? dm[u] : S.dim, IMG ? lm[u] : lim);
        } else {
          const int* tc = reinterpret_cast<const int*>(T.codes + (size_t)tv * 256);
          const int s = sv[u], dim = IMG ? dm[u] : S.dim;
          for (int j = 0; j < 6; ++j) {
            const int cw = res ? *reinterpret_cast<const int*>(smem + tbo[u] + 4 * ix) : __ldg(tc + ix);
            const int o1 = ((sx0(cw) * s) >> 8) * dim + ((sx1(cw) * s) >> 8);
            const int o2 = ((sx2(cw) * s) >> 8) * dim + ((sx3(cw) * s) >> 8);
            const unsigned q1 = __ldg(pc[u] + o1), q2 = __ldg(pc[u] + o2);
            ix = 2 * ix + (q1 <= q2 ? 1 : 0);
          }
        }
        idx[u] = ix;
        pred[u] = res ? *reinterpret_cast<const float*>(smem + tbo[u] + 4 * ix) : __ldg(T.preds + (size_t)tv * 64 + ix - 64);
        thr[u] = res ? *reinterpret_cast<const float*>(smem + tbo[u] + 512) : __ldg(T.thresh + tv);
      }
    }
#pragma unroll
    for (int u = 0; u < NG; ++u) {
      if (alive[u]) {
        acc[u] += pred[u];                               // core/pigo.go:137
        tbo[u] += kTreeRec;
        if (ROT) sv[u] += 1;                             // next tree's node table
        if (acc[u] <= thr[u]) {                          // :139-141
          alive[u] = false;
        } else if (tbo[u] == tbo_last) {
          const float q = acc[u] - thr[u];               // :144
          if (q > 0.0f) {                                // :246
            const int pos = atomicAdd(S.raw_count + fr[u], 1);
            if (pos < S.cap) S.raw[(size_t)fr[u] * S.cap + pos] = RawDet{wid[u], q};
          }
          alive[u] = false;
        } else if (tbo[u] >= casc_end && S.longq != nullptr) {
          // survived the resident trees: hand over to the deep (GROUP-trees-per-step) kernel; if its queue is full
          // the window simply continues here on the global tables
          const unsigned pos = atomicAdd(S.long_count, 1u);
          if (pos < S.long_cap) {
            S.longq[pos] = DeepItem{wid[u], pack_frame_si(fr[u], wsi[u]), (int)((tbo[u] - casc) / kTreeRec), acc[u]};
            alive[u] = false;
          }
        }
      }
    }
  }
}

// Stages the first KS tree records into shared memory with the TMA bulk engine; returns after all threads see them.
__device__ __forceinline__ void stage_cascade(const TiledArgs& A, uint32_t smem_base, uint32_t casc, uint32_t casc_bytes) {
  const uint32_t bar = smem_base;
  if (threadIdx.x == 0) mbar_init(bar, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, casc_bytes);
    for (uint32_t off = 0; off < casc_bytes; off += 32768) {
      const uint32_t n = min(32768u, casc_bytes - off);
      tma_bulk_g2s(smem_base + casc + off, A.tab_tiled + off, n, bar);
    }
  }
  __syncthreads();
  mbar_wait(bar, 0);
}

// gather-v2: every warp plays the gather role (untiled scales in 16x16-window blocks), with the cascade prefix in shared
// memory.  256 threads, several CTAs per SM.
template <int NG, int MINB, int ROT, int IMG = 0>
__global__ void __launch_bounds__(256, MINB) scan_gather2_kernel(const TiledArgs A) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t smem_base = (uint32_t)__cvta_generic_to_shared(smem);
  const uint32_t casc = kCascOff;
  const uint32_t casc_bytes = (uint32_t)A.ks * kTreeRec;
  stage_cascade(A, smem_base, casc, (casc_bytes + 15u) & ~15u);
  gather_role<NG, ROT, IMG>(A, smem, casc, casc + casc_bytes);
}

template <int NI, int MAXT>
__global__ void __launch_bounds__(MAXT, 1) scan_tiled_kernel(const TiledArgs A, const __grid_constant__ TileMaps TM) {
  extern __shared__ __align__(128) uint8_t smem[];
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t smem_base = (uint32_t)__cvta_generic_to_shared(smem);
  const uint32_t wbar = smem_base + 16 + 8 * warp; // per-warp mbarrier: tile arrival
  const uint32_t casc = kCascOff;                 // byte offset of the cascade prefix records inside smem[]
  const uint32_t casc_bytes = (uint32_t)A.ks * kTreeRec;
  const uint32_t casc_end = casc + casc_bytes;    // record offset of tree KS (first tree NOT resident)
  const uint32_t tiles0 = (kCascOff + ((casc_bytes + 15u) & ~15u) + 127) & ~127u;
  const uint32_t my_tile = tiles0 + (uint32_t)warp * A.tile_bytes;

  // ---- stage the cascade prefix with the TMA bulk engine (one elected thread issues, all threads wait)
  if (lane == 0 && warp < A.tile_warps) mbar_init(wbar, 1);
  if (threadIdx.x < kLutSizes) smem[kLutOff + threadIdx.x] = 0xff;
  stage_cascade(A, smem_base, casc, (casc_bytes + 15u) & ~15u);
  if ((int)threadIdx.x < A.scan.nscales && threadIdx.x < 255) {
    const int sz = A.scan.plan[threadIdx.x].s;
    if (sz >= 0 && sz < kLutSizes) smem[kLutOff + sz] = (uint8_t)threadIdx.x;     // sizes are distinct along the ladder
  }
  __syncthreads();

  const ScanArgs& S = A.scan;
  if (warp >= A.tile_warps) {   // warp-specialised: the remaining warps scan the large scales by global-memory gathers
    // (a gather-role walk is a chain of L2 round trips, ~4000 cycles per tree: the host sets a low gather_limit so that
    // long-lived windows move early to the deep kernel, which walks several trees per step)
    const uint32_t g_end = casc + (uint32_t)min(A.ks, max(1, A.gather_limit)) * kTreeRec;
    if (A.gather_ni >= 2) gather_role<2, 0>(A, smem, casc, g_end);
    else gather_role<1, 0>(A, smem, casc, g_end);
    return;
  }
  uint32_t tile_phase = 0;
  const bool all_resident = A.ks >= S.tab.ntrees;  // then reaching casc_end means "survived the whole cascade"
  bool overflow_mode = false;                      // warp-uniform: a hand-over to the deep queue failed (queue full)

  for (;;) {
    // ---- next tile for this warp
    unsigned long long tg = 0;
    if (lane == 0) tg = atomicAdd(S.chunk_counter, 1ull);
    tg = __shfl_sync(FULL, tg, 0);
    if (tg >= A.total_tiles) break;
    const int frame = (int)(tg / A.tiles_per_frame);
    wait_frames(S.ready, S.frame_base + (unsigned)frame + 1u);
    int tf = (int)(tg % A.tiles_per_frame);
    int b = 0;
    while (b + 1 < A.nbands && tf >= A.band[b].ntiles) { tf -= A.band[b].ntiles; ++b; }
    const TileBand B = A.band[b];
    const int ty = tf / B.tiles_x, tx = tf - ty * B.tiles_x;
    const int cx0 = B.org_x + tx * B.core, cy0 = ty * B.core;          // core origin (window centres)
    const int gx0 = cx0 - B.halo_lo, gy0 = cy0 - B.halo_lo;            // tile origin in the frame (gx0 % 16 == 0)
    const int pitch = B.pitch;
    const uint8_t* fb = S.frames + (size_t)frame * S.frame_stride;

    // ---- per-scale window sub-grids of this tile: lane l describes band scale l
    int sc_i0 = 0, sc_j0 = 0, sc_nj = 0, sc_n = 0;
    ScaleEntry e{};
    if (lane < B.nscales) {
      e = S.plan[B.scale_lo + lane];
      const int i0 = ceil_div_pos(cy0 - e.off, e.step), i1 = min(e.nrows, ceil_div_pos(cy0 + B.core - e.off, e.step));
      const int j0 = ceil_div_pos(cx0 - e.off, e.step), j1 = min(e.ncols, ceil_div_pos(cx0 + B.core - e.off, e.step));
      sc_i0 = i0; sc_j0 = j0;
      sc_nj = max(0, j1 - j0);
      sc_n = max(0, i1 - i0) * sc_nj;
    }
    if (!__any_sync(FULL, sc_n > 0)) continue;  // no window centre falls into this core (frame border)

    // ---- fill the tile: rows [gy0, gy0+rows_t) x bytes [gx0, gx0+pitch) clipped to the frame
    __syncwarp();
    if (A.use_tmap) {
      // ONE TMA tensor copy per tile (3-D box pitch x rows_t x 1 frame, zero fill outside the frame), issued by lane 0
      if (lane == 0) {
        mbar_expect_tx(wbar, (uint32_t)(B.rows_t * pitch));
        tma_tile_g2s(smem_base + my_tile, &TM.m[b], gx0, gy0, frame, wbar);
      }
      mbar_wait(wbar, tile_phase);
      tile_phase ^= 1u;
    } else if (A.aligned) {
      // one TMA bulk copy per tile row (16-byte aligned, clipped to the frame), completion on the warp's mbarrier
      const int y_lo = max(gy0, 0), y_hi = min(gy0 + B.rows_t, S.rows);
      const int x_lo = max(gx0, 0), x_hi = min(gx0 + pitch, S.dim);
      const uint32_t row_bytes = (uint32_t)(x_hi - x_lo);
      if (lane == 0) mbar_expect_tx(wbar, row_bytes * (uint32_t)(y_hi - y_lo));
      __syncwarp();
      for (int y = y_lo + lane; y < y_hi; y += 32)
        tma_bulk_g2s(smem_base + my_tile + (uint32_t)((y - gy0) * pitch + (x_lo - gx0)), fb + (size_t)y * S.dim + x_lo, row_bytes, wbar);
      mbar_wait(wbar, tile_phase);
      tile_phase ^= 1u;
    } else {
      const int nbytes = B.rows_t * pitch;
      for (int q = lane; q < nbytes; q += 32) {
        const int row = q / pitch, xx = q - row * pitch;
        const int y = gy0 + row, x = gx0 + xx;
        if (y >= 0 && y < S.rows && x >= 0 && x < S.dim) smem[my_tile + q] = __ldg(fb + (size_t)y * S.dim + x);
      }
    }
    __syncwarp();

    // uniform cursor over the tile's window list (scale-major)
    int cur_si = -1, cur_k = 0, cur_n = 0;
    int u_s = 0, u_step = 0, u_nj = 1, u_ncols = 0, u_br = 0, u_bc = 0;
    uint32_t u_wid0 = 0, u_magic = 0;
    bool exhausted = false;

    bool alive[NI];
    uint32_t pb[NI], tbo[NI], wid[NI];
    int sv[NI];
    float acc[NI];
#pragma unroll
    for (int u = 0; u < NI; ++u) { alive[u] = false; pb[u] = my_tile; tbo[u] = casc; wid[u] = 0; sv[u] = 0; acc[u] = 0.f; }

    for (;;) {
      // ================= refill dead slots from the tile's window list ==========================================
      // Fast path (straight-line, one uniform branch): all dead slots of all NI groups take consecutive windows
      // of the current scale.  The serial path below handles scale changes, the end of the tile and its tail.
      unsigned need[NI];
      int total = 0;
#pragma unroll
      for (int u = 0; u < NI; ++u) { need[u] = __ballot_sync(FULL, !alive[u]); total += __popc(need[u]); }
      if (total != 0) {
        if (!exhausted && cur_k + total <= cur_n) {
          int base = cur_k;
#pragma unroll
          for (int u = 0; u < NI; ++u) {
            if (!alive[u]) {
              const uint32_t k = (uint32_t)(base + __popc(need[u] & lanemask_lt()));
              const uint32_t i = u_nj > 1 ? __umulhi(k, u_magic) : k;   // k / nj, exact for k*nj < 2^32
              const uint32_t j = k - i * (uint32_t)u_nj;
              pb[u] = my_tile + (uint32_t)((u_br + (int)i * u_step) * pitch + u_bc + (int)j * u_step);
              wid[u] = u_wid0 + i * (uint32_t)u_ncols + j;
              sv[u] = u_s; tbo[u] = casc; acc[u] = 0.f;
              alive[u] = true;
            }
            base += __popc(need[u]);
          }
          cur_k += total;
        } else {
          unsigned live_any = 0;
#pragma unroll
          for (int u = 0; u < NI; ++u) {
            unsigned nd = need[u];
            while (nd && !exhausted) {
              if (cur_k == cur_n) {
                // advance to the next scale of the band that has windows in this tile
                int nsi = cur_si + 1;
                int n = 0;
                while (nsi < B.nscales && (n = __shfl_sync(FULL, sc_n, nsi)) == 0) ++nsi;
                if (nsi >= B.nscales) { exhausted = true; break; }
                cur_si = nsi; cur_k = 0; cur_n = n;
                u_s = __shfl_sync(FULL, e.s, nsi); u_step = __shfl_sync(FULL, e.step, nsi);
                const int off = __shfl_sync(FULL, e.off, nsi), i0 = __shfl_sync(FULL, sc_i0, nsi), j0 = __shfl_sync(FULL, sc_j0, nsi);
                u_nj = __shfl_sync(FULL, sc_nj, nsi); u_ncols = __shfl_sync(FULL, e.ncols, nsi);
                u_br = off + i0 * u_step - gy0;   // tile row of the sub-grid's first window centre
                u_bc = off + j0 * u_step - gx0;
                u_wid0 = __shfl_sync(FULL, e.wbase, nsi) + (uint32_t)i0 * (uint32_t)u_ncols + (uint32_t)j0;
                u_magic = u_nj > 1 ? (uint32_t)((0x100000000ull + (unsigned)u_nj - 1) / (unsigned)u_nj) : 0u;  // ceil(2^32/nj)
                continue;
              }
              const int avail = cur_n - cur_k;
              const int rank = __popc(nd & lanemask_lt());
              if (!alive[u] && rank < avail) {
                const uint32_t k = (uint32_t)(cur_k + rank);
                const uint32_t i = u_nj > 1 ? __umulhi(k, u_magic) : k;
                const uint32_t j = k - i * (uint32_t)u_nj;
                pb[u] = my_tile + (uint32_t)((u_br + (int)i * u_step) * pitch + u_bc + (int)j * u_step);
                wid[u] = u_wid0 + i * (uint32_t)u_ncols + j;
                sv[u] = u_s; tbo[u] = casc; acc[u] = 0.f;
                alive[u] = true;
              }
              cur_k += min(__popc(nd), avail);
              nd = __ballot_sync(FULL, !alive[u]);
            }
            // ---- tail policy: once the tile is drained, a thin slot group is handed to the deep queue
            unsigned live = ~nd;
            if (exhausted && live != 0u && __popc(live) < A.tail_min && !overflow_mode) {
              unsigned qbase = 0;
              if (lane == 0) qbase = atomicAdd(S.long_count, (unsigned)__popc(live));
              qbase = __shfl_sync(FULL, qbase, 0);
              const unsigned pos = qbase + __popc(live & lanemask_lt());
              const int qsi = scale_index_of(smem, sv[u]);
              if (alive[u] && pos < S.long_cap) {
                S.longq[pos] = DeepItem{wid[u], pack_frame_si(frame, qsi), (int)((tbo[u] - casc) / kTreeRec), acc[u]};
                alive[u] = false;
              }
              live = __ballot_sync(FULL, alive[u]);
              if (live) overflow_mode = true;   // queue full: finish these items here
            }
            live_any |= live;
          }
          if (!live_any) break;
          // dead slots walk a harmless dummy (tree 0 at a valid pixel with s = 0)
#pragma unroll
          for (int u = 0; u < NI; ++u)
            if (!alive[u]) { tbo[u] = casc; sv[u] = 0; }
        }
      }

      if (A.stats != nullptr) {   // developer counter: useful (live) lanes per walk iteration of the tile role
        unsigned nlive = 0;
#pragma unroll
        for (int u = 0; u < NI; ++u) nlive += __popc(__ballot_sync(FULL, alive[u]));
        if (lane == 0) { atomicAdd(A.stats, (unsigned long long)nlive); atomicAdd(A.stats + 1, (unsigned long long)NI); }
      }
      // ================= one tree per live item =================================================================
      if (!overflow_mode) {
        int idx[NI], cw[NI];
        if (A.tile_prefetch) {
          // Child-pair prefetch: the two children of node idx sit at bytes 8*idx .. 8*idx+7 of the record (codes, or the
          // two leaves after the last level), so they are fetched with ONE 64-bit load issued together with the pixel
          // gathers of the current level; a select picks the child afterwards.  Shorter dependent chain, but a 64-bit
          // warp load costs at least two shared-memory wavefronts.
#pragma unroll
          for (int u = 0; u < NI; ++u) { idx[u] = 1; cw[u] = *reinterpret_cast<const int*>(smem + tbo[u] + 4); }
#pragma unroll
          for (int j = 0; j < 6; ++j) {
            int2 kids[NI];
#pragma unroll
            for (int u = 0; u < NI; ++u) kids[u] = *reinterpret_cast<const int2*>(smem + tbo[u] + 8 * idx[u]);
            uint32_t p1[NI], p2[NI];
#pragma unroll
            for (int u = 0; u < NI; ++u) {
              const int s = sv[u];
              const int o1 = ((sx0(cw[u]) * s) >> 8) * pitch + ((sx1(cw[u]) * s) >> 8);
              const int o2 = ((sx2(cw[u]) * s) >> 8) * pitch + ((sx3(cw[u]) * s) >> 8);
              p1[u] = smem[pb[u] + o1];
              p2[u] = smem[pb[u] + o2];
            }
#pragma unroll
            for (int u = 0; u < NI; ++u) {
              const bool right = p1[u] <= p2[u];                                  // core/pigo.go:129-135
              cw[u] = right ? kids[u].y : kids[u].x;
              idx[u] = 2 * idx[u] + (right ? 1 : 0);
            }
          }
        } else {
          // Plain walk: one 32-bit node load per level (fewest shared-memory wavefronts; the kernel is L1TEX-bound).
          // (Explicit 32-bit shared-window addresses via inline ld.shared save about three instructions per level on paper,
          // but the volatile asm loads pin the schedule.)
#pragma unroll
          for (int u = 0; u < NI; ++u) idx[u] = 1;
#pragma unroll
          for (int j = 0; j < 6; ++j) {
#pragma unroll
            for (int u = 0; u < NI; ++u) cw[u] = *reinterpret_cast<const int*>(smem + tbo[u] + 4 * idx[u]);
            uint32_t p1[NI], p2[NI];
#pragma unroll
            for (int u = 0; u < NI; ++u) {
              // ((r*256 + code*s) >> 8) == r + ((code*s) >> 8)  (core/pigo.go:126-127)
              const int s = sv[u];
              const int o1 = ((sx0(cw[u]) * s) >> 8) * pitch + ((sx1(cw[u]) * s) >> 8);
              const int o2 = ((sx2(cw[u]) * s) >> 8) * pitch + ((sx3(cw[u]) * s) >> 8);
              p1[u] = smem[pb[u] + o1];
              p2[u] = smem[pb[u] + o2];
            }
#pragma unroll
            for (int u = 0; u < NI; ++u) idx[u] = 2 * idx[u] + (p1[u] <= p2[u] ? 1 : 0);   // core/pigo.go:129-135
          }
#pragma unroll
          for (int u = 0; u < NI; ++u) cw[u] = *reinterpret_cast<const int*>(smem + tbo[u] + 4 * idx[u]);   // leaf (words 64..127)
        }
        bool hit = false;
        float thr_last[NI];
#pragma unroll
        for (int u = 0; u < NI; ++u) {
          const float pred = __int_as_float(cw[u]);         // after the last level the selected "child" is the leaf value
          const float thr = *reinterpret_cast<const float*>(smem + tbo[u] + 512);
          thr_last[u] = thr;
          acc[u] += pred;                                   // core/pigo.go:137 (float32, tree order)
          alive[u] = alive[u] && !(acc[u] <= thr);          // :139-141
          tbo[u] += kTreeRec;
          hit |= alive[u] && tbo[u] == casc_end;
          if (!alive[u]) { tbo[u] = casc; sv[u] = 0; }      // a dead slot walks a harmless dummy until it is refilled
        }
        if (__any_sync(FULL, hit)) {                        // some windows passed the last resident tree (rare)
#pragma unroll
          for (int u = 0; u < NI; ++u) {
            const bool at_end = alive[u] && tbo[u] == casc_end;
            const unsigned mb = __ballot_sync(FULL, at_end);
            if (!mb) continue;
            if (all_resident) {
              if (at_end) {
                const float q = acc[u] - thr_last[u];       // :144
                if (q > 0.0f) {                             // :246
                  const int pos = atomicAdd(S.raw_count + frame, 1);
                  if (pos < S.cap) S.raw[(size_t)frame * S.cap + pos] = RawDet{wid[u], q};
                }
                alive[u] = false;
              }
            } else {
              unsigned qbase = 0;
              if (lane == 0) qbase = atomicAdd(S.long_count, (unsigned)__popc(mb));
              qbase = __shfl_sync(FULL, qbase, 0);
              const unsigned pos = qbase + __popc(mb & lanemask_lt());
              bool failed = false;
              const int qsi = scale_index_of(smem, sv[u]);
              if (at_end) {
                if (pos < S.long_cap) {
                  S.longq[pos] = DeepItem{wid[u], pack_frame_si(frame, qsi), A.ks, acc[u]};
                  alive[u] = false;
                } else {
                  failed = true;
                }
              }
              if (__any_sync(FULL, failed)) overflow_mode = true;
            }
            if (!alive[u]) { tbo[u] = casc; sv[u] = 0; }
          }
        }
      } else {
        // ---- overflow mode (deep queue full, pathological): correct but slow; cascade rows beyond KS from global
#pragma unroll
        for (int u = 0; u < NI; ++u) {
          const int tv = (int)((tbo[u] - casc) / kTreeRec);
          const bool res = tbo[u] < casc_end;
          int idx = 1;
          for (int j = 0; j < 6; ++j) {
            const int cw = res ? *reinterpret_cast<const int*>(smem + tbo[u] + 4 * idx)
                               : __ldg(reinterpret_cast<const int*>(S.tab.codes + (size_t)tv * 256) + idx);
            const int s = sv[u];
            const int o1 = ((sx0(cw) * s) >> 8) * pitch + ((sx1(cw) * s) >> 8);
            const int o2 = ((sx2(cw) * s) >> 8) * pitch + ((sx3(cw) * s) >> 8);
            const uint32_t p1 = smem[pb[u] + o1], p2 = smem[pb[u] + o2];
            idx = 2 * idx + (p1 <= p2 ? 1 : 0);
          }
          const float pred = res ? *reinterpret_cast<const float*>(smem + tbo[u] + 4 * idx) : __ldg(S.tab.preds + (size_t)tv * 64 + idx - 64);
          const float thr = res ? *reinterpret_cast<const float*>(smem + tbo[u] + 512) : __ldg(S.tab.thresh + tv);
          if (alive[u]) {
            acc[u] += pred;
            tbo[u] += kTreeRec;
            if (acc[u] <= thr) {
              alive[u] = false;
            } else if (tv + 1 == S.tab.ntrees) {
              const float q = acc[u] - thr;
              if (q > 0.0f) {
                const int pos = atomicAdd(S.raw_count + frame, 1);
                if (pos < S.cap) S.raw[(size_t)frame * S.cap + pos] = RawDet{wid[u], q};
              }
              alive[u] = false;
            }
          }
        }
      }
    }
  }
}

// =============================================================================================================
// Per-scale offset tables (round 2, option tile_ptab).  Same warp specialisation, tiles, queues and results as the classic
// kernel; what changes is WHERE the tile role's node data comes from.  The classic walk derives a node's two sample positions
// from four int8 codes, the window size and the tile pitch at every level (3 PRMT, 4 IMAD, 3 SHF, 2 LEA, 2 IMAD: 24 instructions
// per level).  Here every tiled ladder entry has its own table of the first kt trees in global memory
// (ptab_kernel): a node is ONE word holding the two tile offsets ((code*s)>>8)*pitch + ((code*s)>>8), biased by
// halo*(pitch+1) so that both are unsigned 16-bit, and a level is LDS, LOP, 2 x IADD-class, 2 x LDS.U8, ISETP, index update.
// A table depends on the scale, so the tile warps of a CTA walk the scales in step: the CTA works in ROUNDS (tile_warps
// consecutive tiles of one band, assigned statically: round g -> CTA g % gridDim), every warp visits the band's scales in
// order, and two table buffers in shared memory hold the current and the next scale of the sequence.  A warp may have lanes in
// both (lane refill continues across a scale change); it LEAVES a scale when its last lane of that scale is done or evicted
// (mbarrier arrive), the warp that completes the barrier issues the TMA bulk copy of the table two steps ahead into the freed
// buffer, and a warp ENTERS the next scale when that copy has landed (mbarrier phase).  Windows alive after kt trees go to the
// deep queue.  Off by default (the classic kernel is the default; see DESIGN.md); kept as a tested option.
constexpr uint32_t kPtCtl = 384;    // full[0..1], empty[0..1] mbarriers (8 bytes each), then the two "filled for sequence" words
constexpr uint32_t kPtCasc = 448;   // raw cascade prefix of the gather role
constexpr uint32_t kPtGap = 16;     // bytes between the two table buffers ("one past the last tree" of buffer 0 is not buffer 1)

__device__ __forceinline__ int pt_band_of(const TiledArgs& A, uint32_t rem, uint32_t* rib) {
  int b = 0;
  while (b + 1 < A.nbands && rem >= A.band_rounds[b]) { rem -= A.band_rounds[b]; ++b; }
  *rib = rem;
  return b;
}
// Table of the sequence element `steps` after (round g, band scale k) in this CTA's order; nullptr past the CTA's last round.
__device__ __forceinline__ const uint8_t* pt_table_after(const TiledArgs& A, unsigned long long g, int k, int steps, unsigned long long total_rounds) {
  uint32_t rib;
  int b = pt_band_of(A, (uint32_t)(g % A.rounds_per_frame), &rib);
  for (int i = 0; i < steps; ++i) {
    if (++k >= A.band[b].nscales) {
      k = 0;
      g += gridDim.x;
      if (g >= total_rounds) return nullptr;
      b = pt_band_of(A, (uint32_t)(g % A.rounds_per_frame), &rib);
    }
  }
  return A.ptab + (size_t)(A.band[b].scale_lo + k) * A.ptab_stride;
}

// Finishes one window on the global tables from tree tv on (a queue was full: pathological, slow, correct).
// pix = tile address of the window centre.
// (arguments by value: a reference to the kernel's parameter struct would force a local copy of all of it)
__device__ __noinline__ void pt_finish_slow(const int8_t* codes, const float* preds, const float* thresh, int ntrees, int* raw_count, RawDet* raw, int cap,
                                            const uint8_t* smem, uint32_t pix, int pitch, int s, int tv, float acc, int frame, uint32_t wid) {
  float thr = 0.f;
  for (; tv < ntrees; ++tv) {
    const int* tc = reinterpret_cast<const int*>(codes + (size_t)tv * 256);
    int idx = 1;
    for (int j = 0; j < 6; ++j) {
      const int cw = __ldg(tc + idx);
      const int o1 = ((sx0(cw) * s) >> 8) * pitch + ((sx1(cw) * s) >> 8);
      const int o2 = ((sx2(cw) * s) >> 8) * pitch + ((sx3(cw) * s) >> 8);
      idx = 2 * idx + (smem[pix + o1] <= smem[pix + o2] ? 1 : 0);      // core/pigo.go:129-135
    }
    acc += __ldg(preds + (size_t)tv * 64 + idx - 64);                    // :137
    thr = __ldg(thresh + tv);
    if (acc <= thr) return;                                              // :139-141
  }
  const float q = acc - thr;                                             // :144
  if (q > 0.0f) {                                                        // :246
    const int pos = atomicAdd(raw_count + frame, 1);
    if (pos < cap) raw[(size_t)frame * cap + pos] = RawDet{wid, q};
  }
}

template <int MAXT>
__global__ void __launch_bounds__(MAXT, 1) scan_ptab_kernel(const TiledArgs A, const __grid_constant__ TileMaps TM) {
  extern __shared__ __align__(128) uint8_t smem[];
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t smem_base = (uint32_t)__cvta_generic_to_shared(smem);
  const uint32_t wbar = smem_base + 16 + 8 * warp;   // per-warp mbarrier: tile arrival
  const uint32_t fullbar = smem_base + kPtCtl;       // + 8 * buffer: table arrival
  const uint32_t emptybar = smem_base + kPtCtl + 16; // + 8 * buffer: every tile warp has left the table (count = tile warps)
  unsigned int* issued = reinterpret_cast<unsigned int*>(smem + kPtCtl + 32);   // sequence number each buffer was last filled for
  const uint32_t casc = kPtCasc;
  const uint32_t casc_bytes = (uint32_t)A.ks * kTreeRec;
  const uint32_t tab0 = A.ptab_off, tab_bytes = (uint32_t)A.kt * kTreeRec, bstride = A.ptab_stride + kPtGap;
  const uint32_t my_tile = A.tiles_off + (uint32_t)warp * A.tile_bytes;
  const int W = A.tile_warps;
  const ScanArgs& S = A.scan;
  const unsigned long long total_rounds = (unsigned long long)A.rounds_per_frame * (unsigned long long)S.nframes;

  if (lane == 0 && warp < W) mbar_init(wbar, 1);
  if (threadIdx.x == 0) {
    mbar_init(fullbar, 1); mbar_init(fullbar + 8, 1);
    mbar_init(emptybar, 32u * (uint32_t)W); mbar_init(emptybar + 8, 32u * (uint32_t)W);
    issued[0] = 0; issued[1] = 1;
  }
  if (threadIdx.x < kLutSizes) smem[kLutOff + threadIdx.x] = 0xff;
  stage_cascade(A, smem_base, casc, (casc_bytes + 15u) & ~15u);   // (its fence + barrier also publish the barriers above)
  if ((int)threadIdx.x < S.nscales && threadIdx.x < 255) {
    const int sz = S.plan[threadIdx.x].s;
    if (sz >= 0 && sz < kLutSizes) smem[kLutOff + sz] = (uint8_t)threadIdx.x;
  }
  if (threadIdx.x == 0 && blockIdx.x < total_rounds) {            // the first two tables of this CTA's sequence
    for (int i = 0; i < 2; ++i) {
      const uint8_t* src = pt_table_after(A, blockIdx.x, 0, i, total_rounds);
      if (src) {
        mbar_expect_tx(fullbar + 8 * i, A.ptab_stride);
        tma_bulk_g2s(smem_base + tab0 + (uint32_t)i * bstride, src, A.ptab_stride, fullbar + 8 * i);
      }
    }
  }
  __syncthreads();

  if (warp >= W) {
    const uint32_t g_end = casc + (uint32_t)min(A.ks, max(1, A.gather_limit)) * kTreeRec;
    if (A.gather_ni >= 2) gather_role<2, 0>(A, smem, casc, g_end);
    else gather_role<1, 0>(A, smem, casc, g_end);
    return;
  }

  uint32_t tile_phase = 0;
  const bool all_resident = A.kt >= S.tab.ntrees;   // then surviving a table means surviving the cascade
  uint32_t q_round = 0;                             // sequence number of band scale 0 of the current round

  for (unsigned long long g = blockIdx.x; g < total_rounds; g += gridDim.x) {
    const int frame = (int)(g / A.rounds_per_frame);
    uint32_t rib;
    const int b = pt_band_of(A, (uint32_t)(g % A.rounds_per_frame), &rib);
    const TileBand B = A.band[b];
    const int tf = (int)rib * W + warp;
    const bool has_tile = tf < B.ntiles;
    const int ty = tf / B.tiles_x, tx = tf - ty * B.tiles_x;
    const int cx0 = B.org_x + tx * B.core, cy0 = ty * B.core;
    const int gx0 = cx0 - B.halo_lo, gy0 = cy0 - B.halo_lo;
    const int pitch = B.pitch;
    const uint32_t bias = (uint32_t)(B.halo_lo * (pitch + 1));

    // leaving band scale kk of this round (sequence q = q_round + kk): arrive on the buffer's "empty" barrier; whoever sees the
    // phase complete (at least the warp that arrived last) and wins the claim on the sequence number refills the buffer with
    // the table two steps ahead.  The refill is ordered after every warp's reads by the barrier (arrive = release, test = acquire).
    auto leave = [&](int kk) {
      const uint32_t q = q_round + (uint32_t)kk, buf = q & 1u;
      mbar_arrive(emptybar + 8 * buf);   // every lane arrives for itself (it was a reader of the table): count = 32 * tile warps
      __syncwarp();
      if (lane == 0) {
        if (mbar_test(emptybar + 8 * buf, (q >> 1) & 1u) && atomicCAS(&issued[buf], q, q + 2u) == q) {
          const uint8_t* src = pt_table_after(A, g, kk, 2, total_rounds);
          if (src) {
            mbar_expect_tx(fullbar + 8 * buf, A.ptab_stride);
            tma_bulk_g2s(smem_base + tab0 + buf * bstride, src, A.ptab_stride, fullbar + 8 * buf);
          }
        }
      }
    };

    // ---- per-scale window sub-grids of this tile: lane l describes band scale l
    int sc_i0 = 0, sc_j0 = 0, sc_nj = 0, sc_n = 0;
    ScaleEntry e{};
    if (lane < B.nscales) {
      e = S.plan[B.scale_lo + lane];
      if (has_tile) {
        const int i0 = ceil_div_pos(cy0 - e.off, e.step), i1 = min(e.nrows, ceil_div_pos(cy0 + B.core - e.off, e.step));
        const int j0 = ceil_div_pos(cx0 - e.off, e.step), j1 = min(e.ncols, ceil_div_pos(cx0 + B.core - e.off, e.step));
        sc_i0 = i0; sc_j0 = j0;
        sc_nj = max(0, j1 - j0);
        sc_n = max(0, i1 - i0) * sc_nj;
      }
    }
    int k = -1;   // band scale open for refill (entered); -1 = none yet
    if (__any_sync(FULL, sc_n > 0)) {
      // ---- fill the tile (as the classic kernel)
      wait_frames(S.ready, S.frame_base + (unsigned)frame + 1u);
      const uint8_t* fb = S.frames + (size_t)frame * S.frame_stride;
      __syncwarp();
      if (A.use_tmap) {
        if (lane == 0) {
          mbar_expect_tx(wbar, (uint32_t)(B.rows_t * pitch));
          tma_tile_g2s(smem_base + my_tile, &TM.m[b], gx0, gy0, frame, wbar);
        }
        mbar_wait(wbar, tile_phase);
        tile_phase ^= 1u;
      } else if (A.aligned) {
        const int y_lo = max(gy0, 0), y_hi = min(gy0 + B.rows_t, S.rows);
        const int x_lo = max(gx0, 0), x_hi = min(gx0 + pitch, S.dim);
        const uint32_t row_bytes = (uint32_t)(x_hi - x_lo);
        if (lane == 0) mbar_expect_tx(wbar, row_bytes * (uint32_t)(y_hi - y_lo));
        __syncwarp();
        for (int y = y_lo + lane; y < y_hi; y += 32)
          tma_bulk_g2s(smem_base + my_tile + (uint32_t)((y - gy0) * pitch + (x_lo - gx0)), fb + (size_t)y * S.dim + x_lo, row_bytes, wbar);
        mbar_wait(wbar, tile_phase);
        tile_phase ^= 1u;
      } else {
        const int nbytes = B.rows_t * pitch;
        for (int q = lane; q < nbytes; q += 32) {
          const int row = q / pitch, xx = q - row * pitch;
          const int y = gy0 + row, x = gx0 + xx;
          if (y >= 0 && y < S.rows && x >= 0 && x < S.dim) smem[my_tile + q] = __ldg(fb + (size_t)y * S.dim + x);
        }
      }
      __syncwarp();

      bool old_open = false;   // band scale k-1 still has live lanes of this warp (its table buffer is still in use)
      uint32_t cur_tab = tab0 + (q_round & 1u) * bstride;
      int cur_k = 0, cur_n = 0;
      int u_step = 0, u_nj = 1, u_ncols = 0, u_br = 0, u_bc = 0, u_s = 0, u_s_old = 0;
      uint32_t u_wid0 = 0, u_magic = 0;
      bool exhausted = false;
      bool alive = false;
      uint32_t pb = my_tile, tbo = cur_tab, wid = 0;
      int tleft = 0;
      float acc = 0.f;

      for (;;) {
        // ---- leave the older scale once its last lane is gone
        if (old_open) {
          const uint32_t old_lo = tab0 + ((q_round + (uint32_t)k - 1u) & 1u) * bstride;
          if (!__any_sync(FULL, alive && (tbo - old_lo) < bstride)) { leave(k - 1); old_open = false; }
        }
        // ---- refill dead lanes from the tile's window list (scale-major)
        const unsigned need = __ballot_sync(FULL, !alive);
        if (need) {
          const int total = __popc(need);
          if (!exhausted && cur_k + total <= cur_n) {
            if (!alive) {
              const uint32_t kk = (uint32_t)(cur_k + __popc(need & lanemask_lt()));
              const uint32_t i = u_nj > 1 ? __umulhi(kk, u_magic) : kk;
              const uint32_t j = kk - i * (uint32_t)u_nj;
              pb = my_tile + (uint32_t)((u_br + (int)i * u_step) * pitch + u_bc + (int)j * u_step) - bias;
              wid = u_wid0 + i * (uint32_t)u_ncols + j;
              tbo = cur_tab; acc = 0.f; tleft = A.kt;
              alive = true;
            }
            cur_k += total;
          } else {
            unsigned nd = need;
            while (nd && !exhausted) {
              if (cur_k == cur_n) {
                // ---- enter the next band scale: needs the older one left and the table landed.  Lanes still in the older
                //      scale would hold its buffer (and with it every warp of the CTA) for up to kt trees: they are evicted
                //      to the deep queue Q2 instead (a few per cent of the windows; the deep kernel finishes them).
                if (old_open) {
                  const uint32_t old_lo = tab0 + ((q_round + (uint32_t)k - 1u) & 1u) * bstride;
                  const bool mine = alive && (tbo - old_lo) < bstride;
                  const unsigned mm = __ballot_sync(FULL, mine);
                  if (mm) {
                    unsigned qbase = 0;
                    if (lane == 0) qbase = atomicAdd(S.long_count, (unsigned)__popc(mm));
                    qbase = __shfl_sync(FULL, qbase, 0);
                    const unsigned pos = qbase + __popc(mm & lanemask_lt());
                    if (mine) {
                      const int tv = A.kt - tleft;
                      if (pos < S.long_cap) S.longq[pos] = DeepItem{wid, pack_frame_si(frame, B.scale_lo + k - 1), tv, acc};
                      else pt_finish_slow(S.tab.codes, S.tab.preds, S.tab.thresh, S.tab.ntrees, S.raw_count, S.raw, S.cap, smem, pb + bias, pitch, u_s_old, tv, acc, frame, wid);
                      alive = false;
                    }
                  }
                  leave(k - 1);
                  old_open = false;
                  nd = __ballot_sync(FULL, !alive);
                }
                if (k + 1 >= B.nscales) { exhausted = true; break; }
                const uint32_t qn = q_round + (uint32_t)(k + 1);
                const uint32_t fbq = fullbar + 8 * (qn & 1u), par = (qn >> 1) & 1u;
                if (!mbar_test(fbq, par)) {
                  if (nd != FULL) break;          // live lanes: keep walking, look again after the next tree
                  mbar_wait(fbq, par);
                }
                if (k >= 0) {
                  if (nd != FULL) old_open = true; else leave(k);
                }
                ++k;
                cur_tab = tab0 + (qn & 1u) * bstride;
                cur_k = 0; cur_n = __shfl_sync(FULL, sc_n, k);
                u_s_old = u_s;
                u_s = __shfl_sync(FULL, e.s, k); u_step = __shfl_sync(FULL, e.step, k);
                const int off = __shfl_sync(FULL, e.off, k), i0 = __shfl_sync(FULL, sc_i0, k), j0 = __shfl_sync(FULL, sc_j0, k);
                u_nj = __shfl_sync(FULL, sc_nj, k); u_ncols = __shfl_sync(FULL, e.ncols, k);
                u_br = off + i0 * u_step - gy0;
                u_bc = off + j0 * u_step - gx0;
                u_wid0 = __shfl_sync(FULL, e.wbase, k) + (uint32_t)i0 * (uint32_t)u_ncols + (uint32_t)j0;
                u_magic = u_nj > 1 ? (uint32_t)((0x100000000ull + (unsigned)u_nj - 1) / (unsigned)u_nj) : 0u;
                continue;
              }
              const int avail = cur_n - cur_k;
              const int rank = __popc(nd & lanemask_lt());
              if (!alive && rank < avail) {
                const uint32_t kk = (uint32_t)(cur_k + rank);
                const uint32_t i = u_nj > 1 ? __umulhi(kk, u_magic) : kk;
                const uint32_t j = kk - i * (uint32_t)u_nj;
                pb = my_tile + (uint32_t)((u_br + (int)i * u_step) * pitch + u_bc + (int)j * u_step) - bias;
                wid = u_wid0 + i * (uint32_t)u_ncols + j;
                tbo = cur_tab; acc = 0.f; tleft = A.kt;
                alive = true;
              }
              cur_k += min(__popc(nd), avail);
              nd = __ballot_sync(FULL, !alive);
            }
            // ---- tail policy: once the tile is drained, a thin slot group is handed to the deep queue Q2
            unsigned live = __ballot_sync(FULL, alive);
            if (exhausted && live != 0u && __popc(live) < A.tail_min) {
              unsigned qbase = 0;
              if (lane == 0) qbase = atomicAdd(S.long_count, (unsigned)__popc(live));
              qbase = __shfl_sync(FULL, qbase, 0);
              const unsigned pos = qbase + __popc(live & lanemask_lt());
              if (alive) {
                const uint32_t old_lo = tab0 + ((q_round + (uint32_t)k - 1u) & 1u) * bstride;
                const bool in_old = old_open && (tbo - old_lo) < bstride;
                const int tv = A.kt - tleft;
                if (pos < S.long_cap) S.longq[pos] = DeepItem{wid, pack_frame_si(frame, B.scale_lo + (in_old ? k - 1 : k)), tv, acc};
                else pt_finish_slow(S.tab.codes, S.tab.preds, S.tab.thresh, S.tab.ntrees, S.raw_count, S.raw, S.cap, smem, pb + bias, pitch, in_old ? u_s_old : u_s, tv, acc, frame, wid);
                alive = false;
              }
              live = 0u;
            }
            if (live == 0u) {
              if (exhausted) break;      // round done for this warp
              continue;                  // nothing to walk: leave the older scale / wait for the table at the top
            }
          }
        }
        if (!alive) { tbo = cur_tab; pb = my_tile; }   // dead lanes walk a harmless dummy (tree 0 of a landed table at the tile origin)

        if (A.stats != nullptr) {
          const unsigned nlive = __popc(__ballot_sync(FULL, alive));
          if (lane == 0) { atomicAdd(A.stats, (unsigned long long)nlive); atomicAdd(A.stats + 1, 1ull); }
        }
        // ================= one tree per live lane ==================================================================
        int idx = 1;
#pragma unroll
        for (int j = 0; j < 6; ++j) {
          const uint32_t nw = *reinterpret_cast<const uint32_t*>(smem + tbo + 4 * idx);   // the node's two tile offsets
          const uint32_t p1 = smem[pb + (nw & 0xffffu)], p2 = smem[pb + (nw >> 16)];
          idx = 2 * idx + (p1 <= p2 ? 1 : 0);                                             // core/pigo.go:129-135
        }
        const float pred = *reinterpret_cast<const float*>(smem + tbo + 4 * idx);         // leaf (words 64..127)
        const float thr = *reinterpret_cast<const float*>(smem + tbo + 512);
        acc += pred;                                          // core/pigo.go:137 (float32, tree order)
        alive = alive && !(acc <= thr);                       // :139-141
        tbo += kTreeRec;
        --tleft;
        const bool at_end = alive && tleft == 0;
        const unsigned mb = __ballot_sync(FULL, at_end);
        if (mb) {                                             // some windows passed the last table tree (rare)
          if (all_resident) {
            if (at_end) {
              const float q = acc - thr;                      // :144
              if (q > 0.0f) {                                 // :246
                const int pos = atomicAdd(S.raw_count + frame, 1);
                if (pos < S.cap) S.raw[(size_t)frame * S.cap + pos] = RawDet{wid, q};
              }
              alive = false;
            }
          } else {
            unsigned qbase = 0;
            if (lane == 0) qbase = atomicAdd(S.long_count, (unsigned)__popc(mb));
            qbase = __shfl_sync(FULL, qbase, 0);
            const unsigned pos = qbase + __popc(mb & lanemask_lt());
            if (at_end) {
              const uint32_t old_lo = tab0 + ((q_round + (uint32_t)k - 1u) & 1u) * bstride;
              const bool in_old = old_open && (tbo - old_lo) < bstride;
              if (pos < S.long_cap) S.longq[pos] = DeepItem{wid, pack_frame_si(frame, B.scale_lo + (in_old ? k - 1 : k)), A.kt, acc};
              else pt_finish_slow(S.tab.codes, S.tab.preds, S.tab.thresh, S.tab.ntrees, S.raw_count, S.raw, S.cap, smem, pb + bias, pitch, in_old ? u_s_old : u_s, A.kt, acc, frame, wid);
              alive = false;
            }
          }
        }
      }
      if (old_open) leave(k - 1);   // (cannot happen: no live lanes -> left at the top of the loop; kept for safety)
      if (k >= 0) leave(k);
    }
    // ---- scales this warp never entered (no tile in this round, or no windows): pass through, in order
    for (int kk = k + 1; kk < B.nscales; ++kk) {
      const uint32_t qn = q_round + (uint32_t)kk;
      mbar_wait(fullbar + 8 * (qn & 1u), (qn >> 1) & 1u);
      leave(kk);
    }
    q_round += (uint32_t)B.nscales;
  }
}

// One thread per (tiled ladder entry, tree < kt, record word): the node words of the per-scale tables.
struct PtabGeom {
  int32_t nscales;                 // tiled ladder entries
  int32_t pitch[32], halo[32];     // of the band each entry belongs to
};
__global__ void __launch_bounds__(256) ptab_kernel(FaceTables T, const ScaleEntry* __restrict__ plan, PtabGeom G, int kt, uint32_t stride,
                                                   uint8_t* __restrict__ out) {
  const int words = kTreeRec / 4;
  const size_t total = (size_t)G.nscales * kt * words;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int wd = (int)(i % words);
    const size_t st = i / words;
    const int t = (int)(st % (size_t)kt), si = (int)(st / (size_t)kt);
    uint32_t v = 0;
    if (wd >= 1 && wd < 64) {
      const int s = plan[si].s, pitch = G.pitch[si], halo = G.halo[si];
      const int8_t* cd = T.codes + (size_t)t * 256 + 4 * wd;
      const int o1 = (((int)cd[0] * s) >> 8) * pitch + (((int)cd[1] * s) >> 8) + halo * (pitch + 1);   // core/pigo.go:126-127
      const int o2 = (((int)cd[2] * s) >> 8) * pitch + (((int)cd[3] * s) >> 8) + halo * (pitch + 1);
      v = (uint32_t)(o1 & 0xffff) | ((uint32_t)(o2 & 0xffff) << 16);
    } else if (wd >= 64 && wd < 128) {
      v = __float_as_uint(T.preds[(size_t)t * 64 + (wd - 64)]);
    } else if (wd == 128) {
      v = __float_as_uint(T.thresh[t]);
    }
    *reinterpret_cast<uint32_t*>(out + (size_t)si * stride + (size_t)t * kTreeRec + 4 * (size_t)wd) = v;
  }
}

// =============================================================================================================
// Dense-head variant of the fused kernel (round 2).  Same warp specialisation, same tiles, same queues; the tile role is
// split in two phases so that the first trees -- tree 0 and 1 are 63 % of all tree walks, and every window walks tree 0 --
// run on a cheaper instruction stream:
//   HEAD  : the warp takes 32 consecutive fresh windows of ONE scale and walks trees 0..head_trees-1 in lock-step.  All lanes
//           are on the same tree and scale, so a node is one word of a per-scale table holding the two precomputed sample
//           offsets (dr*pitch + dc as int16): a level is LDS, 2 x (extract, add), 2 x LDS.U8, compare, index = 11
//           instructions instead of 21, there is no per-lane tree / scale state and no refill bookkeeping per walk.
//           Lanes whose window was rejected idle until the batch ends (tree 1 runs at ~45 % of the lanes).
//   RING  : survivors (~16 % after two trees) are compacted (ballot + popc) into a per-warp ring in shared memory.
//   TAIL  : one iteration of the classic lane-refill walk (one tree per live lane, from tree head_trees on), its dead lanes
//           re-armed from the ring.  Head batches run whenever the ring cannot re-arm all dead lanes, so the generic walk
//           always runs with a (nearly) full warp; the live lanes keep their state in registers across head batches.
// Results are identical to the classic kernel by construction (same leaves, same order of float32 adds, same threshold tests).
// ring entry (kRingEntry = 12 bytes): pb (18 bits) | tree (6) | scale (8);  wid;  acc

template <int MAXT>
__global__ void __launch_bounds__(MAXT, 1) scan_head_kernel(const TiledArgs A, const __grid_constant__ TileMaps TM) {
  extern __shared__ __align__(128) uint8_t smem[];
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t smem_base = (uint32_t)__cvta_generic_to_shared(smem);
  const uint32_t wbar = smem_base + 16 + 8 * warp; // per-warp mbarrier: tile arrival
  const uint32_t casc = kCascOff;
  const uint32_t casc_bytes = (uint32_t)A.ks * kTreeRec;
  const uint32_t casc_end = casc + casc_bytes;
  const uint32_t my_tile = A.tiles_off + (uint32_t)warp * A.tile_bytes;
  const uint32_t my_ring = A.ring_off + (uint32_t)warp * (kRing * kRingEntry);
  const int HT = A.head_trees;

  if (lane == 0 && warp < A.tile_warps) mbar_init(wbar, 1);
  if (threadIdx.x < kLutSizes) smem[kLutOff + threadIdx.x] = 0xff;
  stage_cascade(A, smem_base, casc, (casc_bytes + 15u) & ~15u);
  if ((int)threadIdx.x < A.scan.nscales && threadIdx.x < 255) {
    const int sz = A.scan.plan[threadIdx.x].s;
    if (sz >= 0 && sz < kLutSizes) smem[kLutOff + sz] = (uint8_t)threadIdx.x;
  }
  // per-scale head tables: node (scale si, tree t, heap index idx) -> (o2 << 16) | (o1 & 0xffff), o = dr * pitch + dc with
  // dr = (code_r * s) >> 8, dc = (code_c * s) >> 8 exactly as the generic walk computes them (core/pigo.go:126-127)
  for (int q = threadIdx.x; q < A.head_nscales * HT * 64; q += blockDim.x) {
    const int idx = q & 63, t = (q >> 6) % HT, si = q / (64 * HT);
    int b = 0;
    while (b + 1 < A.nbands && si >= A.band[b].scale_lo + A.band[b].nscales) ++b;
    const int pitch = A.band[b].pitch, s = A.scan.plan[si].s;
    const int cw = *reinterpret_cast<const int*>(smem + casc + t * kTreeRec + 4 * idx);
    const int o1 = ((sx0(cw) * s) >> 8) * pitch + ((sx1(cw) * s) >> 8);
    const int o2 = ((sx2(cw) * s) >> 8) * pitch + ((sx3(cw) * s) >> 8);
    *reinterpret_cast<uint32_t*>(smem + A.head_off + 4 * q) = ((uint32_t)o2 << 16) | ((uint32_t)o1 & 0xffffu);
  }
  __syncthreads();

  const ScanArgs& S = A.scan;
  if (warp >= A.tile_warps) {
    if (A.gather_ni >= 2) gather_role<2, 0>(A, smem, casc, casc_end);
    else gather_role<1, 0>(A, smem, casc, casc_end);
    return;
  }
  uint32_t tile_phase = 0;
  const bool all_resident = A.ks >= S.tab.ntrees;
  bool overflow_mode = false;
  // generic-phase lane state
  bool alive = false;
  uint32_t pb = my_tile, tbo = casc, wid = 0;
  int sv = 0;
  float acc = 0.f;
  // ring (warp-uniform)
  int ring_head = 0, ring_cnt = 0;

  for (;;) {
    unsigned long long tg = 0;
    if (lane == 0) tg = atomicAdd(S.chunk_counter, 1ull);
    tg = __shfl_sync(FULL, tg, 0);
    if (tg >= A.total_tiles) break;
    const int frame = (int)(tg / A.tiles_per_frame);
    wait_frames(S.ready, S.frame_base + (unsigned)frame + 1u);
    int tf = (int)(tg % A.tiles_per_frame);
    int b = 0;
    while (b + 1 < A.nbands && tf >= A.band[b].ntiles) { tf -= A.band[b].ntiles; ++b; }
    const TileBand B = A.band[b];
    const int ty = tf / B.tiles_x, tx = tf - ty * B.tiles_x;
    const int cx0 = B.org_x + tx * B.core, cy0 = ty * B.core;
    const int gx0 = cx0 - B.halo_lo, gy0 = cy0 - B.halo_lo;
    const int pitch = B.pitch;
    const uint8_t* fb = S.frames + (size_t)frame * S.frame_stride;

    int sc_i0 = 0, sc_j0 = 0, sc_nj = 0, sc_n = 0;
    ScaleEntry e{};
    if (lane < B.nscales) {
      e = S.plan[B.scale_lo + lane];
      const int i0 = ceil_div_pos(cy0 - e.off, e.step), i1 = min(e.nrows, ceil_div_pos(cy0 + B.core - e.off, e.step));
      const int j0 = ceil_div_pos(cx0 - e.off, e.step), j1 = min(e.ncols, ceil_div_pos(cx0 + B.core - e.off, e.step));
      sc_i0 = i0; sc_j0 = j0;
      sc_nj = max(0, j1 - j0);
      sc_n = max(0, i1 - i0) * sc_nj;
    }
    if (!__any_sync(FULL, sc_n > 0)) continue;

    __syncwarp();
    if (A.use_tmap) {
      if (lane == 0) {
        mbar_expect_tx(wbar, (uint32_t)(B.rows_t * pitch));
        tma_tile_g2s(smem_base + my_tile, &TM.m[b], gx0, gy0, frame, wbar);
      }
      mbar_wait(wbar, tile_phase);
      tile_phase ^= 1u;
    } else if (A.aligned) {
      const int y_lo = max(gy0, 0), y_hi = min(gy0 + B.rows_t, S.rows);
      const int x_lo = max(gx0, 0), x_hi = min(gx0 + pitch, S.dim);
      const uint32_t row_bytes = (uint32_t)(x_hi - x_lo);
      if (lane == 0) mbar_expect_tx(wbar, row_bytes * (uint32_t)(y_hi - y_lo));
      __syncwarp();
      for (int y = y_lo + lane; y < y_hi; y += 32)
        tma_bulk_g2s(smem_base + my_tile + (uint32_t)((y - gy0) * pitch + (x_lo - gx0)), fb + (size_t)y * S.dim + x_lo, row_bytes, wbar);
      mbar_wait(wbar, tile_phase);
      tile_phase ^= 1u;
    } else {
      const int nbytes = B.rows_t * pitch;
      for (int q = lane; q < nbytes; q += 32) {
        const int row = q / pitch, xx = q - row * pitch;
        const int y = gy0 + row, x = gx0 + xx;
        if (y >= 0 && y < S.rows && x >= 0 && x < S.dim) smem[my_tile + q] = __ldg(fb + (size_t)y * S.dim + x);
      }
    }
    __syncwarp();

    // uniform cursor over the tile's window list (scale-major)
    int cur_si = -1, cur_k = 0, cur_n = 0;
    int u_s = 0, u_step = 0, u_nj = 1, u_ncols = 0, u_br = 0, u_bc = 0;
    uint32_t u_wid0 = 0, u_magic = 0, u_hb = A.head_off;
    bool exhausted = false;

    for (;;) {
      // ================= HEAD: batches of 32 fresh windows of one scale, trees 0..HT-1 in lock-step ==================
      // Run while the ring cannot re-arm the dead lanes of the generic phase (whose live lanes keep their state meanwhile).
      unsigned need = __ballot_sync(FULL, !alive);
      while (!exhausted && ring_cnt < __popc(need) && ring_cnt <= kRing - 32) {
        if (cur_k == cur_n) {
          int nsi = cur_si + 1;
          int n = 0;
          while (nsi < B.nscales && (n = __shfl_sync(FULL, sc_n, nsi)) == 0) ++nsi;
          if (nsi >= B.nscales) { exhausted = true; break; }
          cur_si = nsi; cur_k = 0; cur_n = n;
          u_s = __shfl_sync(FULL, e.s, nsi); u_step = __shfl_sync(FULL, e.step, nsi);
          const int off = __shfl_sync(FULL, e.off, nsi), i0 = __shfl_sync(FULL, sc_i0, nsi), j0 = __shfl_sync(FULL, sc_j0, nsi);
          u_nj = __shfl_sync(FULL, sc_nj, nsi); u_ncols = __shfl_sync(FULL, e.ncols, nsi);
          u_br = off + i0 * u_step - gy0;
          u_bc = off + j0 * u_step - gx0;
          u_wid0 = __shfl_sync(FULL, e.wbase, nsi) + (uint32_t)i0 * (uint32_t)u_ncols + (uint32_t)j0;
          u_magic = u_nj > 1 ? (uint32_t)((0x100000000ull + (unsigned)u_nj - 1) / (unsigned)u_nj) : 0u;
          u_hb = A.head_off + (uint32_t)(B.scale_lo + nsi) * (uint32_t)(HT * 256);
        }
        const int n_take = min(32, cur_n - cur_k);
        const uint32_t k = (uint32_t)(cur_k + min(lane, n_take - 1));      // surplus lanes repeat the last window (result ignored)
        cur_k += n_take;
        const uint32_t i = u_nj > 1 ? __umulhi(k, u_magic) : k;             // k / nj, exact for k*nj < 2^32
        const uint32_t j = k - i * (uint32_t)u_nj;
        const uint32_t hpb = my_tile + (uint32_t)((u_br + (int)i * u_step) * pitch + u_bc + (int)j * u_step);
        float hacc = 0.f;
        bool halive = lane < n_take;
        for (int t = 0; t < HT; ++t) {
          const uint32_t hb = u_hb + (uint32_t)t * 256u, rec = casc + (uint32_t)t * kTreeRec;
          int idx = 1;
#pragma unroll
          for (int lv = 0; lv < 6; ++lv) {
            const uint32_t nd = *reinterpret_cast<const uint32_t*>(smem + hb + 4 * idx);
            const uint32_t p1 = smem[hpb + (int)(short)(nd & 0xffffu)], p2 = smem[hpb + ((int)nd >> 16)];
            idx = 2 * idx + (p1 <= p2 ? 1 : 0);                             // core/pigo.go:129-135
          }
          hacc += *reinterpret_cast<const float*>(smem + rec + 4 * idx);   // :137 (float32, tree order)
          halive = halive && !(hacc <= *reinterpret_cast<const float*>(smem + rec + 512));   // :139-141
          if (!__any_sync(FULL, halive)) break;
        }
        const unsigned m = __ballot_sync(FULL, halive);
        if (m) {
          int slot = ring_head + ring_cnt + __popc(m & lanemask_lt());
          if (slot >= kRing) slot -= kRing;
          if (slot >= kRing) slot -= kRing;
          if (halive) {
            uint32_t* en = reinterpret_cast<uint32_t*>(smem + my_ring + slot * kRingEntry);
            en[0] = hpb | ((uint32_t)HT << 18) | ((uint32_t)u_s << 24);
            en[1] = u_wid0 + i * (uint32_t)u_ncols + j;
            en[2] = __float_as_uint(hacc);
          }
          ring_cnt += __popc(m);
          __syncwarp();
        }
      }

      // ================= TAIL: generic lane-refill walk, re-armed from the ring =======================================
      {
        const int take = min(__popc(need), ring_cnt);
        if (take > 0) {
          const int rank = __popc(need & lanemask_lt());
          if (!alive && rank < take) {
            int slot = ring_head + rank;
            if (slot >= kRing) slot -= kRing;
            const uint32_t* en = reinterpret_cast<const uint32_t*>(smem + my_ring + slot * kRingEntry);
            const uint32_t w0 = en[0];
            pb = w0 & 0x3ffffu; tbo = casc + ((w0 >> 18) & 0x3fu) * kTreeRec; sv = (int)(w0 >> 24);
            wid = en[1]; acc = __uint_as_float(en[2]);
            alive = true;
          }
          ring_head += take;
          if (ring_head >= kRing) ring_head -= kRing;
          ring_cnt -= take;
          __syncwarp();
        }
      }
      unsigned live = __ballot_sync(FULL, alive);
      if (!live) {
        if (exhausted && ring_cnt == 0) break;       // tile done
        continue;
      }
      if (exhausted && ring_cnt == 0 && !overflow_mode && __popc(live) < A.tail_min) {
        // tile drained: a thin group of stragglers goes to Q2 (finished by the deep kernel, one lane group per window)
        unsigned qbase = 0;
        if (lane == 0) qbase = atomicAdd(S.long_count, (unsigned)__popc(live));
        qbase = __shfl_sync(FULL, qbase, 0);
        const unsigned pos = qbase + __popc(live & lanemask_lt());
        const int qsi = scale_index_of(smem, sv);
        if (alive && pos < S.long_cap) {
          S.longq[pos] = DeepItem{wid, pack_frame_si(frame, qsi), (int)((tbo - casc) / kTreeRec), acc};
          alive = false;
        }
        live = __ballot_sync(FULL, alive);
        if (!live) break;
        overflow_mode = true;   // queue full: finish these items here
      }
      if (!alive) { tbo = casc; sv = 0; }   // dead lanes walk a harmless dummy (tree 0 at a valid pixel with s = 0)
      if (!overflow_mode) {
        int idx = 1, cw;
#pragma unroll
        for (int j = 0; j < 6; ++j) {
          cw = *reinterpret_cast<const int*>(smem + tbo + 4 * idx);
          const int o1 = ((sx0(cw) * sv) >> 8) * pitch + ((sx1(cw) * sv) >> 8);
          const int o2 = ((sx2(cw) * sv) >> 8) * pitch + ((sx3(cw) * sv) >> 8);
          const uint32_t p1 = smem[pb + o1], p2 = smem[pb + o2];
          idx = 2 * idx + (p1 <= p2 ? 1 : 0);                           // core/pigo.go:129-135
        }
        const float pred = *reinterpret_cast<const float*>(smem + tbo + 4 * idx);
        const float thr = *reinterpret_cast<const float*>(smem + tbo + 512);
        acc += pred;                                                   // core/pigo.go:137
        alive = alive && !(acc <= thr);                                // :139-141
        tbo += kTreeRec;
        const bool at_end = alive && tbo == casc_end;
        const unsigned mb = __ballot_sync(FULL, at_end);
        if (mb) {
          if (all_resident) {
            if (at_end) {
              const float q = acc - thr;                               // :144
              if (q > 0.0f) {                                          // :246
                const int pos = atomicAdd(S.raw_count + frame, 1);
                if (pos < S.cap) S.raw[(size_t)frame * S.cap + pos] = RawDet{wid, q};
              }
              alive = false;
            }
          } else {
            unsigned qbase = 0;
            if (lane == 0) qbase = atomicAdd(S.long_count, (unsigned)__popc(mb));
            qbase = __shfl_sync(FULL, qbase, 0);
            const unsigned pos = qbase + __popc(mb & lanemask_lt());
            const int qsi = scale_index_of(smem, sv);
            bool failed = false;
            if (at_end) {
              if (pos < S.long_cap) {
                S.longq[pos] = DeepItem{wid, pack_frame_si(frame, qsi), A.ks, acc};
                alive = false;
              } else {
                failed = true;
              }
            }
            if (__any_sync(FULL, failed)) overflow_mode = true;
          }
        }
      } else {
        // overflow mode (a queue was full, pathological): correct but slow; cascade rows beyond KS from global memory
        const int tv = (int)((tbo - casc) / kTreeRec);
        const bool res = tbo < casc_end;
        int idx = 1;
        for (int j = 0; j < 6; ++j) {
          const int cw = res ? *reinterpret_cast<const int*>(smem + tbo + 4 * idx)
                             : __ldg(reinterpret_cast<const int*>(S.tab.codes + (size_t)tv * 256) + idx);
          const int o1 = ((sx0(cw) * sv) >> 8) * pitch + ((sx1(cw) * sv) >> 8);
          const int o2 = ((sx2(cw) * sv) >> 8) * pitch + ((sx3(cw) * sv) >> 8);
          const uint32_t p1 = smem[pb + o1], p2 = smem[pb + o2];
          idx = 2 * idx + (p1 <= p2 ? 1 : 0);
        }
        const float pred = res ? *reinterpret_cast<const float*>(smem + tbo + 4 * idx) : __ldg(S.tab.preds + (size_t)tv * 64 + idx - 64);
        const float thr = res ? *reinterpret_cast<const float*>(smem + tbo + 512) : __ldg(S.tab.thresh + tv);
        if (alive) {
          acc += pred;
          tbo += kTreeRec;
          if (acc <= thr) {
            alive = false;
          } else if (tv + 1 == S.tab.ntrees) {
            const float q = acc - thr;
            if (q > 0.0f) {
              const int pos = atomicAdd(S.raw_count + frame, 1);
              if (pos < S.cap) S.raw[(size_t)frame * S.cap + pos] = RawDet{wid, q};
            }
            alive = false;
          }
        }
      }
    }
  }
}

template <int NI, int MAXT>
static void launch_tiled_ni(const TiledArgs& A, const TileMaps& TM, int grid, int threads, size_t smem, cudaStream_t st) {
  raise_dyn_smem((const void*)scan_tiled_kernel<NI, MAXT>, (int)smem);
  scan_tiled_kernel<NI, MAXT><<<grid, threads, smem, st>>>(A, TM);
}

static const void* gather2_fn(int ng, bool rot, bool img = false) {
  if (img) {   // mixed-size calls: the image-table variants of the same instantiations
    // (rotated, one window per lane: the per-image pitch and clamp do not fit the 40 registers of 6 CTAs per SM; the scan
    // runs 4 CTAs per SM by default, so 5 costs nothing)
    if (rot) return ng >= 2 ? (const void*)scan_gather2_kernel<2, 4, 1, 1> : (const void*)scan_gather2_kernel<1, 5, 1, 1>;
    if (ng >= 3) return (const void*)scan_gather2_kernel<3, 4, 0, 1>;
    if (ng == 2) return (const void*)scan_gather2_kernel<2, 4, 0, 1>;
    return (const void*)scan_gather2_kernel<1, 6, 0, 1>;
  }
  if (rot) return ng >= 2 ? (const void*)scan_gather2_kernel<2, 4, 1> : (const void*)scan_gather2_kernel<1, 6, 1>;
  if (ng >= 3) return (const void*)scan_gather2_kernel<3, 4, 0>;
  if (ng == 2) return (const void*)scan_gather2_kernel<2, 4, 0>;
  return (const void*)scan_gather2_kernel<1, 6, 0>;
}
void launch_scan_gather2(const TiledArgs& A, int grid, size_t smem, cudaStream_t st) {
  const void* fn = gather2_fn(A.gather_ni, A.scan.rot_slot >= 0, A.scan.images != nullptr);
  raise_dyn_smem(fn, (int)smem);
  void* args[] = {(void*)&A};
  cudaLaunchKernel(fn, dim3(grid), dim3(256), args, smem, st);
}
int gather2_ctas_per_sm(size_t smem, int ng, bool rot, bool img) {
  int n = 0;
  const void* fn = gather2_fn(ng, rot, img);
  raise_dyn_smem(fn, (int)smem);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, 256, smem) != cudaSuccess || n < 1) { cudaGetLastError(); n = 1; }
  return n;
}

int tiled_max_threads(int ni) { return ni == 1 ? 1024 : (ni == 2 ? 768 : 512); }

void launch_ptab_build(const FaceTables& T, const ScaleEntry* plan, const TiledArgs& A, int first_untiled, uint8_t* out, int grid, cudaStream_t st) {
  PtabGeom G{};
  G.nscales = std::min(first_untiled, 32);
  for (int b = 0; b < A.nbands; ++b)
    for (int i = 0; i < A.band[b].nscales; ++i) {
      const int si = A.band[b].scale_lo + i;
      if (si < 32) { G.pitch[si] = A.band[b].pitch; G.halo[si] = A.band[b].halo_lo; }
    }
  ptab_kernel<<<grid, 256, 0, st>>>(T, plan, G, A.kt, A.ptab_stride, out);
}

void launch_scan_tiled(const TiledArgs& A, const TileMaps& TM, int grid, int threads, size_t smem, int ni, cudaStream_t st) {
  if (A.kt > 0) {
    raise_dyn_smem((const void*)scan_ptab_kernel<1024>, (int)smem);
    scan_ptab_kernel<1024><<<grid, threads, smem, st>>>(A, TM);
    return;
  }
  if (A.head_trees > 0) {
    raise_dyn_smem((const void*)scan_head_kernel<1024>, (int)smem);
    scan_head_kernel<1024><<<grid, threads, smem, st>>>(A, TM);
    return;
  }
  switch (ni) {
    case 1: launch_tiled_ni<1, 1024>(A, TM, grid, threads, smem, st); break;
    case 2: launch_tiled_ni<2, 768>(A, TM, grid, threads, smem, st); break;
    case 3: launch_tiled_ni<3, 512>(A, TM, grid, threads, smem, st); break;
    default: launch_tiled_ni<4, 512>(A, TM, grid, threads, smem, st); break;
  }
}

}  // namespace pigo
