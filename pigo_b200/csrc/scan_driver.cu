// scan_driver.cu -- host-side planning and sequencing of the scan kernels for one RunCascade batch:
//   fused kernel     : tile warps (scales whose pixel tiles fit a per-warp shared-memory buffer) + gather warps (the rest)
//   gather-v2 kernel : the 16x16-window blocks the fused kernel did not take (gather_warps=0, no tile plan, rotated scan)
//   deep kernel      : queue Q2 (the tile warps' stragglers and every window that outlived the shared-memory trees),
//                      one lane group per window (8 lanes, 32 for small calls), one tree per lane and step; large calls
//                      sort Q2 into image order first
//   gather kernel    : universal fallback -- rotated scan, cascades of depth != 6, scan_mode=1
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>

#include "common.cuh"
#include "host.h"

namespace pigo {

static constexpr size_t kSmemPerCta = 232448;  // 227 KB opt-in maximum on sm_90

// Builds the shared-memory-layout cascade table: one 516-byte record per tree (depth 6 only).
int build_tiled_tables(const FaceTables& tab, const std::vector<int8_t>& codes, const std::vector<float>& preds,
                       const std::vector<float>& thr, DevBuf& out) {
  if (tab.depth != 6) return PIGO_OK;  // other depths use the gather kernel only
  const size_t n = (size_t)tab.ntrees;
  std::vector<uint8_t> rec(n * kTreeRec + 64, 0);   // 64 spare bytes: the prefix copy is rounded up to 16 bytes
  for (size_t t = 0; t < n; ++t) {
    memcpy(rec.data() + t * kTreeRec, codes.data() + t * 256, 256);
    memcpy(rec.data() + t * kTreeRec + 256, preds.data() + t * 64, 256);
    memcpy(rec.data() + t * kTreeRec + 512, thr.data() + t, 4);
  }
  int rc = out.reserve(rec.size());
  if (rc) return rc;
  if (cudaMemcpy(out.p, rec.data(), rec.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaGetLastError();
    return set_err(PIGO_E_CUDA, "tiled table upload failed");
  }
  return PIGO_OK;
}

// Builds the block-interleaved table the unrotated deep walk reads (depth 6 only; layout: kBlockBytes in common.cuh).
int build_block_tables(const FaceTables& tab, const std::vector<int8_t>& codes, const std::vector<float>& preds,
                       const std::vector<float>& thr, DevBuf& out) {
  if (tab.depth != 6 || tab.ntrees <= 0) return PIGO_OK;
  const int n = tab.ntrees, nblk = (n + kBlockTrees - 1) / kBlockTrees;
  std::vector<uint8_t> blk((size_t)nblk * kBlockBytes, 0);
  for (int i = 0; i < nblk * kBlockTrees; ++i) {
    const int t = std::min(i, n - 1);   // pad slots: a copy of the last tree
    uint8_t* b = blk.data() + (size_t)(i / kBlockTrees) * kBlockBytes;
    const int k = i % kBlockTrees;
    memcpy(b + 4 * k, thr.data() + t, 4);
    memcpy(b + 32 + 4 * k, codes.data() + (size_t)t * 256 + 4, 4);                         // node 1
    for (int p = 1; p < 64; ++p) {
      const void* kids = p < 32 ? (const void*)(codes.data() + (size_t)t * 256 + 8 * p)       // code words 2p, 2p+1
                                : (const void*)(preds.data() + (size_t)t * 64 + 2 * p - 64);  // leaves 2p-64, 2p-63
      memcpy(b + 64 * p + 8 * k, kids, 8);
    }
  }
  int rc = out.reserve(blk.size());
  if (rc) return rc;
  if (cudaMemcpy(out.p, blk.data(), blk.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaGetLastError();
    return set_err(PIGO_E_CUDA, "block table upload failed");
  }
  return PIGO_OK;
}

struct TilePlan {
  int nbands = 0;
  TileBand band[kMaxBands];
  int first_untiled = 0;  // ladder index of the first scale left to the gather kernel
  uint32_t tiles_per_frame = 0;
};

static TilePlan plan_bands(const std::vector<ScaleEntry>& plan, uint32_t tile_bytes, int max_scale, int ratio_pct, int min_core,
                           int min_core_steps, int core_cap = 512) {
  TilePlan tp;
  const int n = (int)plan.size();
  int a = 0;
  while (a < n && tp.nbands < kMaxBands) {
    const int s0 = plan[a].s;
    if (s0 > max_scale) break;
    // longest band [a, b) within the ratio whose tile still has a useful core
    int best_b = -1, best_core = 0;
    for (int b = a + 1; b <= n && b - a <= 32; ++b) {
      const int smax = plan[b - 1].s;
      if (smax > max_scale || (long long)smax * 100 > (long long)s0 * ratio_pct) break;
      const int halo_lo = (smax + 1) / 2, halo_hi = (127 * smax) >> 8;
      int core = 0;
      for (int c = 16; c <= 512 && c <= std::max(16, core_cap); c += 16) {
        const int rows_t = halo_lo + c + halo_hi;
        const int pitch = (rows_t + 15) & ~15;
        if ((size_t)rows_t * pitch <= tile_bytes) core = c; else break;
      }
      const int step_max = plan[b - 1].step;
      if (core >= min_core && core >= min_core_steps * step_max) { best_b = b; best_core = core; }
    }
    if (best_b < 0) break;
    TileBand B{};
    const int smax = plan[best_b - 1].s;
    B.scale_lo = a; B.nscales = best_b - a;
    B.halo_lo = (smax + 1) / 2;
    const int halo_hi = (127 * smax) >> 8;
    B.core = best_core;
    B.rows_t = B.halo_lo + B.core + halo_hi;
    B.pitch = (B.rows_t + 15) & ~15;
    int org = B.halo_lo % 16;
    const int off_min = plan[a].off;
    if (org > off_min) org -= 16;
    B.org_x = org;
    int max_c = 0, max_r = 0;
    for (int i = a; i < best_b; ++i) {
      max_c = std::max(max_c, plan[i].off + (plan[i].ncols - 1) * plan[i].step);
      max_r = std::max(max_r, plan[i].off + (plan[i].nrows - 1) * plan[i].step);
    }
    B.tiles_x = (max_c - B.org_x) / B.core + 1;
    const int tiles_y = max_r / B.core + 1;
    B.ntiles = B.tiles_x * tiles_y;
    tp.band[tp.nbands++] = B;
    tp.tiles_per_frame += (uint32_t)B.ntiles;
    a = best_b;
  }
  tp.first_untiled = a;
  return tp;
}

// Shared-memory layout of the fused kernel: mbarriers (384 B) | cascade prefix | per-warp tiles (128-byte aligned).
struct FusedLayout {
  bool ok = false;
  size_t tiles_off = 0, head_off = 0, ring_off = 0, ptab_off = 0;
  uint32_t tile_bytes = 0;
};
static FusedLayout fused_layout(int W, int ks, size_t smem_cap_req, int head_trees = 0, int kt = 0) {
  FusedLayout L;
  const size_t casc_bytes = ((size_t)ks * kTreeRec + 15) & ~(size_t)15;   // TMA bulk copies move multiples of 16 bytes
  L.head_off = 384 + casc_bytes;
  L.ring_off = L.head_off + (size_t)(head_trees > 0 ? kHeadMaxScales * head_trees * 256 : 0);
  L.tiles_off = (L.ring_off + (size_t)(head_trees > 0 ? W * kRing * kRingEntry : 0) + 127) & ~(size_t)127;
  if (kt > 0) {   // scan_ptab_kernel: control words up to 448, raw prefix, two table buffers 16 bytes apart
    const size_t stride = ((size_t)kt * kTreeRec + 15) & ~(size_t)15;
    L.ptab_off = 448 + casc_bytes;
    L.tiles_off = (L.ptab_off + 2 * stride + 16 + 127) & ~(size_t)127;
  }
  if (W <= 0 || L.tiles_off + 4096 * (size_t)W >= kSmemPerCta) return L;
  // fused_smem_kb < 227 leaves the rest of the SM's 256 KB to L1 (which the gather warps' pixel loads live in)
  size_t smem_cap = kSmemPerCta;
  if (smem_cap_req > 0) smem_cap = std::min<size_t>(kSmemPerCta, std::max<size_t>(smem_cap_req, L.tiles_off + 4096 * (size_t)W));
  L.tile_bytes = (uint32_t)(((smem_cap - L.tiles_off) / W) & ~(size_t)127);
  L.ok = true;
  return L;
}

// The fused kernel's schedule for one ladder under the current options: shared-memory layout + bands.  Used by run_scan and
// by describe_plan, so the CPU-side geometry tests see exactly what the GPU will run.
struct FusedPlan {
  FusedLayout L;
  TilePlan tp;
  int W = 0, ks = 0, ni = 1;
  int head = 0;   // trees of the dense head (0 = classic tile role)
  int kt = 0;     // trees of the per-scale offset tables (0 = classic tile role)
  int band_ratio = 0;   // a band spans scales up to band_ratio/100 x its first scale
};
static FusedPlan plan_fused(const std::vector<ScaleEntry>& plan, int ntrees, int batch_frames = 1 << 20) {
  FusedPlan P;
  P.ni = (int)std::min<long long>(std::max<long long>(1, g_opt.tile_ni.load()), 4);
  const int max_warps = tiled_max_threads(P.ni) / 32;
  P.W = (int)std::min<long long>(std::max<long long>(0, g_opt.tile_warps.load()), max_warps);
  const long long fit = (long long)((kSmemPerCta - 512) / kTreeRec);   // what one CTA's shared memory can hold at most
  P.ks = (int)std::min<long long>(std::min<long long>(std::max<long long>(1, g_opt.tile_ks.load()), ntrees), fit);
  int max_scale = (int)g_opt.tile_max_scale.load();
  if (max_scale <= 0) max_scale = 1 << 30;
  // dense head: needs its tables and rings in shared memory (a fixed reservation for kHeadMaxScales ladder entries), NI = 1,
  // a resident prefix longer than the head and short enough for the 6-bit tree field of a ring entry
  P.head = (int)std::min<long long>(std::max<long long>(0, g_opt.tile_head.load()), kHeadTreesMax);
  if (P.ni != 1 || P.ks <= P.head || P.ks > 63 || g_opt.tile_prefetch.load()) P.head = 0;
  // Optional cap on the tile core (developer knob; more, shorter tiles).
  long long core_cap = g_opt.tile_core_cap.load();
  if (core_cap <= 0) core_cap = 512;   // (16/32-pixel cores mean many more tile fills per frame)
  // per-scale offset tables: NI = 1, no head, its own (shorter) raw prefix for the gather warps
  if (g_opt.tile_ptab.load() != 0 && P.ni == 1 && P.W > 0) {
    P.kt = (int)std::min<long long>(std::min<long long>(std::max<long long>(1, g_opt.ptab_kt.load()), ntrees), 60);
    P.ks = (int)std::min<long long>(std::min<long long>(std::max<long long>(1, g_opt.ptab_ks.load()), ntrees), fit);
    P.head = 0;
  }
  // band width: 2x the band's first scale for throughput; a call of <= 2 M windows (one or two 1080p frames) takes narrower bands
  // (1.4x) -- more, shorter tiles, so that the slowest tile warp of the one partial wave finishes earlier
  unsigned long long call_windows = 0;
  for (const ScaleEntry& e : plan) call_windows += (unsigned long long)e.nrows * (unsigned long long)e.ncols;
  call_windows *= (unsigned long long)std::max(1, batch_frames);
  long long ratio_opt = g_opt.tile_band_ratio.load();
  if (ratio_opt <= 0) ratio_opt = call_windows <= 2000000ull ? 140 : 200;
  const int band_ratio = (int)std::max<long long>(100, ratio_opt);
  P.band_ratio = band_ratio;
  auto plan_with = [&](int head) {
    P.L = fused_layout(P.W, P.ks, (size_t)std::max<long long>(0, g_opt.fused_smem_kb.load()) * 1024, head, P.kt);
    P.tp = TilePlan();
    if (P.L.ok)
      P.tp = plan_bands(plan, P.L.tile_bytes, max_scale, band_ratio,
                        (int)std::min<long long>(std::max<long long>(16, g_opt.tile_min_core.load()), core_cap),
                        (int)std::max<long long>(1, core_cap < 512 ? 1 : g_opt.tile_min_core_steps.load()), (int)core_cap);
  };
  plan_with(P.head);
  if (P.head > 0) {
    // every tiled ladder entry needs a head table; its window size must fit the ring entry's 8-bit field and its offsets int16
    bool ok = P.L.ok && P.tp.nbands > 0 && P.tp.first_untiled <= kHeadMaxScales;
    for (int b = 0; ok && b < P.tp.nbands; ++b) {
      const TileBand& B = P.tp.band[b];
      if ((long long)(B.halo_lo + 1) * (B.pitch + 1) >= 32768) ok = false;
      if (plan[B.scale_lo + B.nscales - 1].s > 255) ok = false;
    }
    if (!ok) { P.head = 0; plan_with(0); }
  }
  if (P.kt > 0) {
    // every tiled ladder entry needs a table slot (32 at most) and unsigned 16-bit offsets
    bool ok = P.L.ok && P.tp.nbands > 0 && P.tp.first_untiled <= 32;
    for (int b = 0; ok && b < P.tp.nbands; ++b) {
      const TileBand& B = P.tp.band[b];
      if ((long long)B.rows_t * (B.pitch + 1) >= 65536) ok = false;
    }
    if (!ok) {   // fall back to the classic kernel with the classic prefix
      P.kt = 0;
      P.ks = (int)std::min<long long>(std::min<long long>(std::max<long long>(1, g_opt.tile_ks.load()), ntrees), fit);
      plan_with(0);
    }
  }
  return P;
}

// Stores the prefix of 16x16-window blocks of the ladder entries [lo, hi) in ScaleEntry.pad and refreshes the device copy.
static int upload_block_prefix(Workspace* w, int lo, int hi, int gb_shift, cudaStream_t st, uint32_t* blocks_per_frame) {
  uint32_t nb = 0;
  const int GB = 1 << gb_shift;
  for (int i = lo; i < hi; ++i) {
    ScaleEntry& e = w->plan_host[i];
    e.pad = nb;
    nb += (uint32_t)((e.ncols + GB - 1) / GB) * (uint32_t)((e.nrows + GB - 1) / GB);
  }
  *blocks_per_frame = nb;
  const int key = lo * 8 + gb_shift;
  if (w->pad_first_untiled != key) {
    if (cudaMemcpyAsync(w->plan.p, w->plan_host.data(), w->plan_host.size() * sizeof(ScaleEntry), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess)
      return set_err(PIGO_E_CUDA, "plan upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    w->pad_first_untiled = key;
  }
  return PIGO_OK;
}

// Host-only introspection of the scan plan (no device needed): which ladder entries go to per-warp tiles (and with what
// tile geometry), which go to the gather role, and which tile role the fused kernel runs (head > 0: dense head, ptab_kt > 0:
// per-scale offset tables, both 0: classic), for a call of `batch_frames` frames of this geometry (the frame count decides
// the band ratio, as in run_scan).  JSON text; used by tests/test_plan_cpu.py to check on the CPU that the tiles partition
// the windows of their scales exactly and that every sample stays inside its tile.
int describe_plan(const std::vector<ScaleEntry>& plan, uint64_t wins, int ntrees, int batch_frames, char* buf, size_t cap) {
  const FusedPlan P = plan_fused(plan, ntrees, batch_frames);
  const TilePlan& tp = P.tp;
  const uint32_t tile_bytes = P.L.ok ? P.L.tile_bytes : 0;
  std::string s = "{";
  char tmp[512];
  snprintf(tmp, sizeof(tmp), "\"nscales\": %d, \"windows\": %llu, \"tile_warps\": %d, \"tiles_off\": %zu, ", (int)plan.size(),
           (unsigned long long)wins, P.W, P.L.tiles_off);
  s += tmp;
  snprintf(tmp, sizeof(tmp), "\"tile_bytes\": %u, \"first_untiled\": %d, \"ptab_kt\": %d, \"head\": %d, \"ks\": %d, \"band_ratio\": %d, \"bands\": [",
           tile_bytes, tp.first_untiled, P.kt, P.head, P.ks, P.band_ratio);
  s += tmp;
  for (int b = 0; b < tp.nbands; ++b) {
    const TileBand& B = tp.band[b];
    snprintf(tmp, sizeof(tmp), "%s{\"scale_lo\": %d, \"nscales\": %d, \"halo_lo\": %d, \"core\": %d, \"org_x\": %d, \"tiles_x\": %d, \"ntiles\": %d, "
             "\"pitch\": %d, \"rows_t\": %d}", b ? ", " : "", B.scale_lo, B.nscales, B.halo_lo, B.core, B.org_x, B.tiles_x, B.ntiles, B.pitch, B.rows_t);
    s += tmp;
  }
  s += "], \"scales\": [";
  for (size_t i = 0; i < plan.size(); ++i) {
    const ScaleEntry& e = plan[i];
    snprintf(tmp, sizeof(tmp), "%s[%d, %d, %d, %d, %d, %u]", i ? ", " : "", e.s, e.step, e.off, e.nrows, e.ncols, e.wbase);
    s += tmp;
  }
  s += "]}";
  if (s.size() + 1 > cap) return set_err(PIGO_E_CAP, "plan description needs %zu bytes", s.size() + 1);
  memcpy(buf, s.c_str(), s.size() + 1);
  return PIGO_OK;
}

// ---- developer counter: live lanes per walk iteration of the tile role (option walk_stats) ----------------------------------
static unsigned long long* g_walk_stats[kMaxDevices] = {};
unsigned long long* walk_stats_buffer(int dev) {
  if (!g_opt.walk_stats.load() || dev < 0 || dev >= kMaxDevices) return nullptr;
  if (!g_walk_stats[dev]) {
    if (cudaMalloc((void**)&g_walk_stats[dev], 16) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    cudaMemset(g_walk_stats[dev], 0, 16);
  }
  return g_walk_stats[dev];
}
void walk_stats_reset() {
  int cur = 0;
  cudaGetDevice(&cur);
  for (int d = 0; d < kMaxDevices; ++d)
    if (g_walk_stats[d]) { cudaSetDevice(d); cudaMemset(g_walk_stats[d], 0, 16); }
  cudaSetDevice(cur);
}
long long walk_stats_query(int which) {
  long long total = 0;
  int cur = 0;
  cudaGetDevice(&cur);
  for (int d = 0; d < kMaxDevices; ++d)
    if (g_walk_stats[d]) {
      unsigned long long v[2] = {0, 0};
      cudaSetDevice(d);
      cudaDeviceSynchronize();
      cudaMemcpy(v, g_walk_stats[d], 16, cudaMemcpyDeviceToHost);
      total += (long long)v[which & 1];
    }
  cudaSetDevice(cur);
  return total;
}

// ---- TMA descriptors of the frame batch (one per tile band) ------------------------------------------------------------
// cuTensorMapEncodeTiled comes from the driver library; it is looked up through the runtime (no link dependency on libcuda).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = []() -> EncodeTiledFn {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
      cudaGetLastError();
      return nullptr;
    }
    return (EncodeTiledFn)p;
  }();
  return fn;
}
// frames [nframes][rows][dim] u8 (frames `frame_stride` bytes apart) as a 3-D tensor; box = one tile of band B
static bool encode_tile_map(CUtensorMap* m, const ScanArgs& A, const TileBand& B) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn || B.pitch > 256 || B.rows_t > 256 || (A.dim % 16) || (A.frame_stride % 16) || ((uintptr_t)A.frames % 16)) return false;
  const cuuint64_t gdim[3] = {(cuuint64_t)A.dim, (cuuint64_t)A.rows, (cuuint64_t)A.nframes};
  const cuuint64_t gstride[2] = {(cuuint64_t)A.dim, (cuuint64_t)A.frame_stride};
  const cuuint32_t box[3] = {(cuuint32_t)B.pitch, (cuuint32_t)B.rows_t, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  return fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void*)A.frames, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_err(PIGO_E_CUDA, "%s launch failed: %s", what, cudaGetErrorString(e));
  return PIGO_OK;
}

// The deep kernel takes Q2 in image order (sorted by frame and 64-pixel cell of the window centre, consumed in per-CTA runs of
// neighbouring windows that share an SM's L1) above this many windows per call.  Smaller calls (up to four 1080p frames or one
// 4K frame) keep one atomic per item: their queue is short, latency matters, and the ordered path was no faster on one frame.
static bool deep_ordered(uint64_t call_windows) { return call_windows > 4000000ull; }

// Sorts D.longq into the lane's second queue buffer and points D at it.  rows / cols: the largest frame of the group.
static int sort_deep_queue(Workspace* w, int lane, ScanArgs& D, int rows, int cols, uint64_t q2_cap, int num_sms, cudaStream_t st) {
  int rc;
  if ((rc = w->longq_sorted[lane].reserve(q2_cap * sizeof(DeepItem)))) return rc;
  if ((rc = w->longq_aux[lane].reserve(deep_sort_aux_bytes(rows, cols, D.nframes, q2_cap)))) return rc;
  if ((rc = launch_deep_sort(D, rows, cols, (DeepItem*)w->longq_sorted[lane].p, w->longq_aux[lane].p, num_sms, st))) return rc;
  if ((rc = check_launch("deep queue sort"))) return rc;
  D.longq = (DeepItem*)w->longq_sorted[lane].p;
  return PIGO_OK;
}

// The block/deep kernels need a depth-6 cascade with its tiled table and scan_mode != 1.  A rotated scan on them also needs
// rot_mode 0, windows of at most 32000 pixels and a node table (one RotNode per ladder entry, tree and node) of at most 512 MB.
bool block_path(const FaceReplica* c, bool rot, int max_scale, size_t rot_bytes) {
  if (c->tab.depth != 6 || c->tiled_tab.p == nullptr || g_opt.scan_mode.load() == 1) return false;
  return !rot || (g_opt.rot_mode.load() == 0 && max_scale <= 32000 && rot_bytes <= ((size_t)1 << 29));
}

// The choices a scan makes from the window count of its whole API call.  "Small call" = at most 4 M windows (a 1080p frame
// has 0.9 M, a 4K frame 3.7 M): latency matters, not throughput.  Small calls cannot fill the GPU with 256-window gather
// blocks (they use 64-window blocks) and give a window 32 deep lanes (the latency of a full survivor matters).  A gather
// window hands over to the deep kernel after 8 trees in a small rotated call or an unrotated one of up to 40 M windows,
// else after 24 trees (rotated) or `large_limit` (unrotated: run_scan and the mixed-size scan each give theirs).
ImagesSchedule images_schedule(uint64_t call_windows, bool rot, int large_limit) {
  ImagesSchedule P;
  const bool small = call_windows <= 4000000ull;
  long long glimit = g_opt.gather_limit.load();
  if (glimit <= 0) glimit = rot ? (small ? 8 : 24) : (call_windows <= 40000000ull ? 8 : large_limit);
  P.gather_limit = (int)std::min<long long>(glimit, 1 << 20);
  P.gb_shift = (g_opt.gather_block.load() == 8 || (g_opt.gather_block.load() == 0 && small)) ? 3 : 4;
  P.deep_group = (int)g_opt.deep_group.load();
  if (P.deep_group != 8 && P.deep_group != 16 && P.deep_group != 32) P.deep_group = small ? 32 : 8;
  P.deep_ordered = deep_ordered(call_windows);
  return P;
}

int run_scan(FaceReplica* c, Workspace* w, int lane, ScanArgs& A, unsigned long long* d_work, cudaStream_t st, int num_sms) {
  int rc;
  const bool rot = A.rot_slot >= 0;
  const long long mode = g_opt.scan_mode.load();
  // d_work (zeroed per call): [0] gather block cursor  [1] tile cursor  [2] Q2 consumer cursor  [3] Q2 count (u32)
  //                           [4] chunk cursor of the standalone gather kernel
  A.longq = nullptr; A.long_count = (unsigned int*)(d_work + 3); A.long_cap = 0;
  A.chunk = (uint32_t)std::max<long long>(32, g_opt.chunk.load());
  A.chunk_counter = d_work + 4;

  // Rotated scan on the block/deep structure: needs the per-call node table.
  const size_t rot_bytes = (size_t)A.nscales * (size_t)A.tab.ntrees * 64 * sizeof(RotNode);
  const int max_scale = w->plan_host.empty() ? 0 : w->plan_host.back().s;
  if (!block_path(c, rot, max_scale, rot_bytes)) {
    // ---- universal path: standalone gather kernel over every scale (any tree depth, scan_mode=1, rot_mode=1)
    ScanArgs G = A;
    G.scale_lo = 0; G.scale_hi = A.nscales;
    G.chunks_per_frame = (A.wins_per_frame + G.chunk - 1) / G.chunk;
    const int per_sm = gather_max_ctas_per_sm(A.tab.depth, rot);
    const unsigned long long total_chunks = (unsigned long long)G.chunks_per_frame * A.nframes;
    const long long grid = std::max(1ll, std::min<long long>((long long)num_sms * per_sm, (long long)((total_chunks + 7) / 8)));
    timing_begin(T_GATHER, st);
    launch_scan_gather(G, (int)grid, max_scale, st);
    timing_end(T_GATHER, st);
    g_launches++;
    return check_launch("gather scan");
  }
  if (rot) {
    if (w->rot_slot != A.rot_slot || w->rot_tab.p == nullptr) {
      if ((rc = w->rot_tab.reserve(rot_bytes))) return rc;
      timing_begin(T_ROTTAB, st);
      launch_rot_table(A.tab, A.plan, A.nscales, A.rot_slot, (RotNode*)w->rot_tab.p, num_sms * 8, st);
      timing_end(T_ROTTAB, st);
      g_launches++;
      if ((rc = check_launch("rotated node table"))) return rc;
      w->rot_slot = A.rot_slot;
    }
    A.rot_tab = (const RotNode*)w->rot_tab.p;
  }

  // ---- the deep queue: the tile warps' stragglers (up to 1/16 of the windows) + the windows that outlive the resident trees
  //      (1/32, 1/16 with the per-scale offset tables)
  const uint64_t total_windows = (uint64_t)A.wins_per_frame * A.nframes;
  const uint64_t q2_cap = std::min<uint64_t>(total_windows / 16 + total_windows / (g_opt.tile_ptab.load() != 0 ? 16 : 32) + 65536, 1ull << 26);
  // developer knob: a tiny queue forces the "queue full" paths of every producer (tests)
  const long long qlim = g_opt.queue_cap.load();
  const uint64_t q2_use = qlim > 0 ? std::min<uint64_t>(q2_cap, (uint64_t)qlim) : q2_cap;
  if ((rc = w->longq[lane].reserve(q2_cap * sizeof(DeepItem)))) return rc;
  A.longq = (DeepItem*)w->longq[lane].p; A.long_cap = (uint32_t)q2_use;

  TiledArgs T{};
  T.scan = A;
  T.scan.chunk_counter = d_work + 1;
  T.tab_tiled = (const uint8_t*)c->tiled_tab.p;
  T.gather_counter = d_work;
  T.gather_scale_lo = 0;
  T.gather_blocks_per_frame = 0;
  T.tile_prefetch = g_opt.tile_prefetch.load() ? 1 : 0;
  T.gather_ni = (int)std::min<long long>(std::max<long long>(1, g_opt.gather_ni.load()), 3);
  // how long a gather-role window stays in the fused kernel before it leaves for the deep kernel (which walks a window with a
  // lane group and is the cheaper place for long walks): calls of up to 40 M windows hand over after 8 trees, larger ones after
  // 16.  (H100, 256 x 1080p: 8 and 16 trees took 0.7 and 0.6 ms off the 24 used before; but 8 made the 64-frame ShiftFactor 0.1
  // batch 2 % slower than the previous build, and 16 did not.)  The rotated scan has no fused kernel: its block kernel keeps
  // 24 trees unless the call is small.  All of it is decided from the frames of the whole API call, not of this pipeline
  // group: the block prefix lives in the shared plan.
  const unsigned long long call_windows = (unsigned long long)A.wins_per_frame * (unsigned long long)std::max(1, A.batch_frames);
  const ImagesSchedule S = images_schedule(call_windows, rot, 16);
  T.gather_limit = S.gather_limit;
  T.gb_shift = S.gb_shift;

  // ---- fused kernel: tile warps over the small scales (+ optional gather warps over the rest)
  auto round_ks = [&](long long v) {
    const long long fit = (long long)((kSmemPerCta - 512) / kTreeRec);   // what one CTA's shared memory can hold at most
    return (int)std::min<long long>(std::min<long long>(std::max<long long>(1, v), A.tab.ntrees), fit);
  };
  int first_untiled = 0;
  bool blocks_done = false;
  if (mode != 3 && !rot) {
    FusedPlan P = plan_fused(w->plan_host, A.tab.ntrees, A.batch_frames);
    const TilePlan& tp = P.tp;
    const int W = P.W;
    int Wg = (int)std::min<long long>(std::max<long long>(0, g_opt.gather_warps.load()), tiled_max_threads(P.ni) / 32 - W);
    if (P.L.ok && tp.nbands > 0) {
      TiledArgs F = T;
      F.ks = P.ks; F.tile_bytes = P.L.tile_bytes; F.nbands = tp.nbands;
      F.tail_min = (int)g_opt.tile_tail_min.load();
      for (int b = 0; b < tp.nbands; ++b) F.band[b] = tp.band[b];
      F.tiles_per_frame = tp.tiles_per_frame;
      F.total_tiles = (unsigned long long)tp.tiles_per_frame * A.nframes;
      F.tile_warps = W;
      F.stats = walk_stats_buffer(c->device);
      F.head_trees = P.head; F.head_nscales = tp.first_untiled;
      F.head_off = (uint32_t)P.L.head_off; F.ring_off = (uint32_t)P.L.ring_off; F.tiles_off = (uint32_t)P.L.tiles_off;
      F.head_back = (int)std::min<long long>(std::max<long long>(1, g_opt.head_back.load()), kRing - 32);
      first_untiled = tp.first_untiled;
      if (Wg > 0 && first_untiled < A.nscales) {
        if ((rc = upload_block_prefix(w, first_untiled, A.nscales, T.gb_shift, st, &F.gather_blocks_per_frame))) return rc;
        F.gather_scale_lo = first_untiled;
        blocks_done = true;
      } else {
        Wg = 0;
      }
      F.aligned = ((A.dim % 16 == 0) && (A.frame_stride % 16 == 0) && (((uintptr_t)A.frames) % 16 == 0)) ? 1 : 0;
      long long grid = num_sms;
      if (Wg == 0) grid = std::max<long long>(1, std::min<long long>(num_sms, (long long)((F.total_tiles + W - 1) / W)));
      if (P.kt > 0) {
        // per-scale offset tables: rounds of W tiles of one band; tables cached per workspace for this geometry
        F.kt = P.kt;
        F.ptab_stride = (uint32_t)(((size_t)P.kt * kTreeRec + 15) & ~(size_t)15);
        F.ptab_off = (uint32_t)P.L.ptab_off;
        F.rounds_per_frame = 0;
        std::vector<int> sig = {P.kt, tp.first_untiled, W};
        for (int b = 0; b < tp.nbands; ++b) {
          F.band_rounds[b] = (uint32_t)((tp.band[b].ntiles + W - 1) / W);
          F.rounds_per_frame += F.band_rounds[b];
          sig.push_back(tp.band[b].scale_lo); sig.push_back(tp.band[b].nscales); sig.push_back(tp.band[b].pitch); sig.push_back(tp.band[b].halo_lo);
        }
        if (w->ptab_sig != sig || w->ptab.p == nullptr) {
          if ((rc = w->ptab.reserve((size_t)tp.first_untiled * F.ptab_stride + 64))) return rc;
          launch_ptab_build(A.tab, A.plan, F, tp.first_untiled, (uint8_t*)w->ptab.p, num_sms * 4, st);
          g_launches++;
          if ((rc = check_launch("offset tables"))) return rc;
          w->ptab_sig = sig;
        }
        F.ptab = (const uint8_t*)w->ptab.p;
        if (Wg == 0) grid = std::max<long long>(1, std::min<long long>(num_sms, (long long)F.rounds_per_frame * A.nframes));
      }
      const size_t smem = P.L.tiles_off + (size_t)P.L.tile_bytes * W;
      TileMaps TM{};
      F.use_tmap = (F.aligned && g_opt.tile_tmap.load() != 0) ? 1 : 0;
      for (int b = 0; b < tp.nbands && F.use_tmap; ++b)
        if (!encode_tile_map(&TM.m[b], A, tp.band[b])) F.use_tmap = 0;
      timing_begin(T_TILED, st);
      launch_scan_tiled(F, TM, (int)grid, (W + Wg) * 32, smem, P.ni, st);
      timing_end(T_TILED, st);
      g_launches++;
      if ((rc = check_launch("fused scan"))) return rc;
    }
  }

  // Streamed host frames: only the fused kernel waits in-kernel for its frames.  Everything queued behind it is ordered after
  // the group's last copy chunk (which the fused kernel has already seen, so this wait is free), and if the fused kernel
  // did not run for this geometry the same wait is what orders the scan behind the copy.
  if (A.ready != nullptr && w->group_copied != nullptr) {
    if (cudaStreamWaitEvent(st, w->group_copied, 0) != cudaSuccess) return set_err(PIGO_E_CUDA, "cudaStreamWaitEvent failed");
  }
  // ---- gather-v2: the 16x16-window blocks of the untiled scales, when the fused kernel's gather warps did not take them
  //      (gather_warps=0, no tile plan fits, or the rotated scan).  On the default path it does not run: the fused kernel is
  //      followed by the deep kernel alone.
  if (!blocks_done && first_untiled < A.nscales) {
    TiledArgs G = T;
    G.scan.ready = nullptr;
    G.ks = round_ks(std::min<long long>(g_opt.gather_ks.load(), T.gather_limit));
    G.tile_warps = 0;
    if ((rc = upload_block_prefix(w, first_untiled, A.nscales, T.gb_shift, st, &G.gather_blocks_per_frame))) return rc;
    G.gather_scale_lo = first_untiled;
    if (G.gather_blocks_per_frame > 0) {
      const size_t smem = ((384 + (size_t)G.ks * kTreeRec + 127) & ~(size_t)127);
      // unrotated, on H100 two CTAs per SM measured faster than four (256 x 1080p, when the kernel also drained the tile
      // warps' stragglers: 11 % less step time together with tile_tail_min 6); rotated, it is the whole scan and keeps four
      int per_sm = (int)g_opt.gather_ctas_per_sm.load();
      if (per_sm <= 0) per_sm = rot ? 4 : 2;
      if (rot) G.gather_ni = std::min(G.gather_ni, 2);
      const int occ = gather2_ctas_per_sm(smem, G.gather_ni, rot);
      if (per_sm > occ) per_sm = occ;
      timing_begin(T_GATHER, st);
      launch_scan_gather2(G, num_sms * per_sm, smem, st);
      timing_end(T_GATHER, st);
      g_launches++;
      if ((rc = check_launch("gather-v2 scan"))) return rc;
    }
  }

  // ---- deep kernel: Q2, one lane group per window
  {
    timing_begin(T_DEEP, st);
    int group = (int)g_opt.deep_group.load();
    const long long ds = g_opt.deep_smem.load();
    const bool smem_deep = !rot && A.tab.depth == 6 && c->tiled_tab.p != nullptr && (ds == 1 || (ds == 0 && false));
    if (smem_deep) {
      if (group != 4 && group != 8 && group != 16 && group != 32) group = 8;
      int threads = (int)g_opt.deep_smem_threads.load();
      threads = std::min(1024, std::max(128, threads)) & ~31;
      launch_deep_smem(A, d_work + 2, (const uint8_t*)c->tiled_tab.p, num_sms, threads, group, (int)std::min<long long>(std::max<long long>(0, g_opt.deep_smem_lo.load()), 1 << 20),
                       (int)std::min<long long>(std::max<long long>(2, g_opt.deep_smem_k.load()), 1 << 20), st);
    } else {
      ScanArgs D = A;
      if (S.deep_ordered && (rc = sort_deep_queue(w, lane, D, A.rows, A.cols, q2_cap, num_sms, st))) return rc;
      launch_deep(D, d_work + 2, num_sms, S.deep_group, S.deep_ordered, st);
    }
    timing_end(T_DEEP, st);
    g_launches++;
    if ((rc = check_launch("deep scan"))) return rc;
  }
  return PIGO_OK;
}

// ---- mixed-size calls (pigo_run_cascade_images) ------------------------------------------------------------------------
// One group of images: the gather-v2 kernel over every ladder entry of every image (in blocks of 16x16 or 8x8 windows,
// located through the image table), then the deep kernel over its survivors -- the kernel pair scan_mode=3 runs for a
// uniform batch.  The caller has set A.images / A.plan (block prefixes built for P.gb_shift) and, rotated, A.rot_tab.
int run_scan_images(FaceReplica* c, Workspace* w, ScanArgs& A, const ImagesSchedule& P, uint32_t group_blocks, uint64_t group_windows,
                    int max_rows, int max_cols, unsigned long long* d_work, cudaStream_t st, int num_sms) {
  int rc;
  const bool rot = A.rot_slot >= 0;
  // d_work (zeroed per call): [0] block cursor  [2] Q2 consumer cursor  [3] Q2 count (as run_scan)
  A.long_count = (unsigned int*)(d_work + 3);
  const uint64_t q2_cap = std::min<uint64_t>(group_windows / 32 + 65536, 1ull << 26);
  const long long qlim = g_opt.queue_cap.load();
  if ((rc = w->longq[0].reserve(q2_cap * sizeof(DeepItem)))) return rc;
  A.longq = (DeepItem*)w->longq[0].p;
  A.long_cap = (uint32_t)(qlim > 0 ? std::min<uint64_t>(q2_cap, (uint64_t)qlim) : q2_cap);

  TiledArgs G{};
  G.scan = A;
  G.tab_tiled = (const uint8_t*)c->tiled_tab.p;
  G.gather_counter = d_work;
  G.gather_scale_lo = 0;
  G.gather_blocks_per_frame = group_blocks;
  G.gather_limit = P.gather_limit;
  G.gb_shift = P.gb_shift;
  G.gather_ni = (int)std::min<long long>(std::max<long long>(1, g_opt.gather_ni.load()), 3);
  if (rot) G.gather_ni = std::min(G.gather_ni, 2);
  const long long fit = (long long)((kSmemPerCta - 512) / kTreeRec);
  G.ks = (int)std::min<long long>(std::min<long long>(std::max<long long>(1, std::min<long long>(g_opt.gather_ks.load(), P.gather_limit)),
                                                      A.tab.ntrees), fit);
  const size_t smem = ((384 + (size_t)G.ks * kTreeRec + 127) & ~(size_t)127);
  int per_sm = (int)g_opt.gather_ctas_per_sm.load();
  if (per_sm <= 0) per_sm = rot ? 4 : 2;   // as run_scan's gather-v2 launch
  per_sm = std::min(per_sm, gather2_ctas_per_sm(smem, G.gather_ni, rot, true));
  timing_begin(T_GATHER, st);
  launch_scan_gather2(G, num_sms * per_sm, smem, st);
  timing_end(T_GATHER, st);
  g_launches++;
  if ((rc = check_launch("gather-v2 scan (images)"))) return rc;

  timing_begin(T_DEEP, st);
  ScanArgs D = A;
  if (P.deep_ordered && (rc = sort_deep_queue(w, 0, D, max_rows, max_cols, q2_cap, num_sms, st))) return rc;
  launch_deep(D, d_work + 2, num_sms, P.deep_group, P.deep_ordered, st);
  timing_end(T_DEEP, st);
  g_launches++;
  return check_launch("deep scan (images)");
}

}  // namespace pigo
