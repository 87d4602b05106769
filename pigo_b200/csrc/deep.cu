// deep.cu -- finishes the windows that survived the shared-memory-resident trees (queue Q2): ONE LANE GROUP PER WINDOW,
// ONE TREE PER LANE.  The GROUP lanes walk GROUP consecutive trees of the same window in parallel (tree walks are
// independent of each other -- only the early-exit test couples them), then the group replays the reference's float32
// accumulation and threshold tests in tree order (core/pigo.go:137-141) with shuffles.  A full survivor of the 468-tree
// cascade costs 468/GROUP steps instead of a ~420-tree serial chain of dependent L2 round trips; trees evaluated past the
// rejecting one are wasted work, acceptable because windows that reach this kernel usually live long.
// Bit-exactness: each lane produces the same leaf the serial walk would, and the sum is formed in the same order.
//
// Round 2: (1) queue items carry their ladder entry, so the consumer needs no binary search; (2) ROT variant:
// classifyRotatedRegion (core/pigo.go:150-191) with the node's sample offsets read from the per-call table (RotNode,
// common.cuh) instead of being recomputed per node; (3) a flat-loop variant (deep_flat=1), measured and left off.
// The unrotated walk reads the cascade from its block-interleaved copy (FaceTables::blocks): the lane group's trees are
// consecutive, so their records of one node share cache lines instead of sitting 256 bytes apart.
#include <algorithm>

#include "common.cuh"
#include "host.h"

namespace pigo {

// One tree (index t) of the window: the leaf value.  Unrotated: pc = the window's centre pixel; rotated: pc = the frame,
// (r, c) the centre, rt = this scale's node table.  dim = row pitch of the window's frame.
template <int ROT>
__device__ __forceinline__ float deep_walk(const ScanArgs& A, const FaceTables& T, const uint8_t* __restrict__ pc, const RotNode* __restrict__ rt,
                                           int t, int r, int c, int s, int lim, int dim) {
  int idx = 1;
  if (ROT) {
    const int2* tp2 = reinterpret_cast<const int2*>(T.preds + (size_t)t * 64);
    // children of node idx are nodes 2idx, 2idx+1: adjacent 8-byte records, fetched with one 16-byte load while
    // this node's two pixels are in flight
    const RotNode* tn = rt + (size_t)t * 64;
    uint2 cur = __ldg(reinterpret_cast<const uint2*>(tn + 1));
    int leafbits = 0;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      uint4 kids = make_uint4(0, 0, 0, 0);
      int2 lv = make_int2(0, 0);
      if (j < 5) kids = __ldg(reinterpret_cast<const uint4*>(tn + 2 * idx));
      else lv = __ldg(tp2 + (idx - 32));
      const int r1 = __vimin_s32_relu(r + (int)(short)(cur.x & 0xffff), lim), c1 = __vimin_s32_relu(c + ((int)cur.x >> 16), lim);
      const int r2 = __vimin_s32_relu(r + (int)(short)(cur.y & 0xffff), lim), c2 = __vimin_s32_relu(c + ((int)cur.y >> 16), lim);
      const unsigned p1 = __ldg(pc + (size_t)r1 * dim + c1), p2 = __ldg(pc + (size_t)r2 * dim + c2);
      const bool right = p1 <= p2;                  // core/pigo.go:179
      cur = right ? make_uint2(kids.z, kids.w) : make_uint2(kids.x, kids.y);
      leafbits = right ? lv.y : lv.x;
      idx = 2 * idx + (right ? 1 : 0);
    }
    return __int_as_float(leafbits);
  } else {
    // child-pair prefetch: both children of node idx (code words, or the two leaves after the last level) are fetched
    // with one 64-bit load that is in flight together with the two pixel gathers.  The block-interleaved table puts the
    // GROUP lanes' records of one node side by side (common.cuh), so the group's loads share cache lines.
    const uint32_t blk = (uint32_t)(t >> 3) * kBlockBytes, rec = blk + 8 * (t & 7);   // 32-bit offsets: one register
    int cw = __ldg(reinterpret_cast<const int*>(T.blocks + blk + 32) + (t & 7));
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const int2 kids = __ldg(reinterpret_cast<const int2*>(T.blocks + rec + 64 * idx));
      const int o1 = (((int)(int8_t)(cw) * s) >> 8) * dim + (((int)(int8_t)(cw >> 8) * s) >> 8);
      const int o2 = (((int)(int8_t)(cw >> 16) * s) >> 8) * dim + (((cw >> 24) * s) >> 8);
      const unsigned p1 = __ldg(pc + o1), p2 = __ldg(pc + o2);
      const bool right = p1 <= p2;                  // core/pigo.go:129-135
      cw = right ? kids.y : kids.x;
      idx = 2 * idx + (right ? 1 : 0);
    }
    return __int_as_float(cw);
  }
}

// Tree t's threshold: unrotated from the block table that deep_walk<0> reads (the group's 8 thresholds are one 32-byte run).
template <int ROT>
__device__ __forceinline__ float deep_thresh(const FaceTables& T, int t) {
  if (ROT) return __ldg(T.thresh + t);
  return __ldg(reinterpret_cast<const float*>(T.blocks + (size_t)(t >> 3) * kBlockBytes) + (t & 7));
}

// Where a queue item's window lies: frame (IMG = 1: the image of the group), ladder entry, size and centre (r, c), from the
// ladder entry the producer packed (0xffff = not known: search).  The deep kernel and the queue sort decode items with it.
struct DeepPos {
  int frame, si, s, r, c;
};
template <int IMG>
__device__ __forceinline__ DeepPos deep_pos(const ScanArgs& A, const DeepItem& it) {
  DeepPos p;
  p.frame = (int)(it.frame_si & 0xffffu);
  const ScaleEntry* plan = A.plan;
  int nscales = A.nscales;
  if (IMG) { plan += A.images[p.frame].plan_off; nscales = A.images[p.frame].nscales; }
  p.si = (int)(it.frame_si >> 16);
  if (p.si == 0xffff) p.si = find_scale(plan, nscales, it.wid);
  const ScaleEntry e = plan[p.si];
  const uint32_t local = it.wid - e.wbase;
  const uint32_t ri = local / (uint32_t)e.ncols, ci = local - ri * (uint32_t)e.ncols;
  p.s = e.s;
  p.r = e.off + (int)ri * e.step; p.c = e.off + (int)ci * e.step;
  return p;
}

// Decodes a queue item for the walk.  IMG = 1 (mixed-size call): plan, pixels, pitch and clamp are the image's.
struct DeepWin {
  uint32_t wid;
  int frame, t0, s, r, c;
  int dim, lim;
  float acc;
  const uint8_t* pc;
  const RotNode* rt;
};
template <int ROT, int IMG = 0>
__device__ __forceinline__ DeepWin deep_fetch(const ScanArgs& A, const FaceTables& T, unsigned long long g) {
  const DeepItem it = A.longq[g];
  const DeepPos p = deep_pos<IMG>(A, it);
  DeepWin w;
  size_t rot_off = 0;   // IMG: the image's node table (units of 64 RotNode records)
  if (IMG) {
    const ImageDesc im = A.images[p.frame];
    w.pc = im.base; w.dim = im.dim; w.lim = im.rows - 1;
    if (ROT) rot_off = im.rot_off;
  } else {
    w.pc = A.frames + (size_t)p.frame * A.frame_stride; w.dim = A.dim; w.lim = A.rows - 1;
  }
  w.s = p.s; w.wid = it.wid; w.frame = p.frame; w.t0 = it.tree; w.acc = it.acc;
  w.r = p.r; w.c = p.c;
  w.rt = A.rot_tab;
  if (ROT) w.rt = A.rot_tab + (rot_off + (size_t)p.si * T.ntrees) * 64;
  else w.pc += (size_t)w.r * w.dim + w.c;
  return w;
}

// Ordered consumption (CHUNK > 0): a CTA claims CHUNK consecutive items of the sorted queue with one global atomic and its
// lane groups take them one by one from a shared-memory cursor, so that the windows resident on an SM at the same time are
// neighbours and their pixel footprints share its L1.  `claim` packs (first item of the run << 32) | items handed out of it.
// The group that draws ticket CHUNK claims the next run and takes its first item; groups that draw a later ticket wait for it.
// H100, 256 x 1080p: runs of 32 / 128 items, 256-thread CTAs and 32-pixel cells measured slower, 128-pixel cells the same.
constexpr int kDeepChunk = 64;
constexpr int kDeepOrdThreads = 1024;
template <int CHUNK>
__device__ __forceinline__ unsigned long long deep_claim(unsigned long long* claim, unsigned long long* counter) {
  for (;;) {
    const unsigned long long v = atomicAdd(claim, 1ull);
    const unsigned j = (unsigned)v;
    if (j < CHUNK) return (v >> 32) + j;
    if (j == CHUNK) {
      const unsigned long long base = atomicAdd(counter, (unsigned long long)CHUNK);
      atomicExch(claim, (base << 32) | 1ull);
      return base;
    }
    __nanosleep(64);
  }
}

// Round-1 loop structure: the lane groups of a warp fetch together, then the warp stays in the step loop until its slowest
// window is done (measured faster than the flat loop below: one fetch latency per 32/GROUP windows instead of one per window).
template <int GROUP, int ROT, int IMG = 0, int CHUNK = 0>
__global__ void __launch_bounds__(CHUNK ? kDeepOrdThreads : 256, CHUNK ? 2048 / kDeepOrdThreads : 1) deep_kernel(const ScanArgs A, unsigned long long* counter) {
  const int lane = threadIdx.x & 31;
  const int sub = lane & (GROUP - 1);
  const unsigned gmask = GROUP == 32 ? 0xffffffffu : (GROUP == 16 ? (0xffffu << (lane & 16)) : (0xffu << (lane & 24)));
  const int leader = lane & ~(GROUP - 1);
  const FaceTables T = A.tab;
  const uint32_t qn = min(*A.long_count, A.long_cap);
  const int lim = A.rows - 1;
  __shared__ unsigned long long claim;
  if (CHUNK) {
    if (threadIdx.x == 0) claim = atomicAdd(counter, (unsigned long long)CHUNK) << 32;
    __syncthreads();
  }
  for (;;) {
    unsigned long long g = 0;
    if constexpr (CHUNK > 0) {
      if (sub == 0) g = deep_claim<CHUNK>(&claim, counter);
    } else {
      if (sub == 0) g = atomicAdd(counter, 1ull);
    }
    g = __shfl_sync(gmask, g, leader);
    if (g >= qn) break;
    const DeepWin w = deep_fetch<ROT, IMG>(A, T, g);
    int t0 = w.t0;
    float acc = w.acc;
    bool rejected = false;
    float thr_prev = 0.f;
    while (t0 < T.ntrees && !rejected) {
      const int t = min(t0 + sub, T.ntrees - 1);      // lanes past the last tree redo it harmlessly
      const float thr = deep_thresh<ROT>(T, t);
      const float pred = deep_walk<ROT>(A, T, w.pc, w.rt, t, w.r, w.c, w.s, IMG ? w.lim : lim, IMG ? w.dim : A.dim);
      const int nvalid = min(GROUP, T.ntrees - t0);
      for (int j = 0; j < nvalid; ++j) {              // the reference's sequential accumulation, :137-141
        acc += __shfl_sync(gmask, pred, leader + j);
        thr_prev = __shfl_sync(gmask, thr, leader + j);
        if (acc <= thr_prev) { rejected = true; break; }
      }
      t0 += GROUP;
    }
    if (!rejected && sub == 0) {
      const float q = acc - thr_prev;                 // :144 (thr_prev == threshold of the last tree)
      if (q > 0.0f) {                                 // :246
        const int pos = atomicAdd(A.raw_count + w.frame, 1);
        if (pos < A.cap) A.raw[(size_t)w.frame * A.cap + pos] = RawDet{w.wid, q};
      }
    }
  }
}

// Shared-memory variant (unrotated, large calls): ONE CTA PER SM keeps the tree records [t_lo, t_lo + ktrees) of the tiled table
// (kTreeRec bytes each: codes, leaves, threshold -- the layout the fused kernel stages) in its 227 KB of shared memory, filled by
// the TMA bulk engine.  A walk then costs two pixel gathers per level through L1TEX instead of two gathers plus a divergent
// 64-bit node load: the kernel is bound by L1TEX sectors, and a third of them are node loads.  Consecutive
// trees sit 130 words apart, so the GROUP lanes of a window (consecutive trees, same node index at the root) read distinct banks.
// Trees below t_lo (thin-tail handoffs of the tile warps, latency-mode items) take the global path of deep_walk.
__device__ __forceinline__ float deep_walk_smem(const uint8_t* __restrict__ rec, const uint8_t* __restrict__ pc, int s, int dim) {
  int idx = 1;
  int cw = *reinterpret_cast<const int*>(rec + 4);
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const int2 kids = *reinterpret_cast<const int2*>(rec + 8 * idx);   // children codes, or the two leaves after the last level
    const int o1 = (((int)(int8_t)(cw) * s) >> 8) * dim + (((int)(int8_t)(cw >> 8) * s) >> 8);
    const int o2 = (((int)(int8_t)(cw >> 16) * s) >> 8) * dim + (((cw >> 24) * s) >> 8);
    const unsigned p1 = __ldg(pc + o1), p2 = __ldg(pc + o2);
    const bool right = p1 <= p2;                  // core/pigo.go:129-135
    cw = right ? kids.y : kids.x;
    idx = 2 * idx + (right ? 1 : 0);
  }
  return __int_as_float(cw);
}

constexpr uint32_t kDeepRecOff = 16;   // the mbarrier lives in the first 16 bytes

template <int GROUP>
__global__ void __launch_bounds__(1024) deep_smem_kernel(const ScanArgs A, unsigned long long* counter, const uint8_t* __restrict__ tab,
                                                            int t_lo, int ktrees) {
  extern __shared__ __align__(128) uint8_t dsm[];
  const uint32_t base = (uint32_t)__cvta_generic_to_shared(dsm);
  const uint32_t bytes = (uint32_t)ktrees * (uint32_t)kTreeRec;    // ktrees and t_lo are even: 16-byte multiples / alignment
  const FaceTables T = A.tab;
  const uint32_t qn = min(*A.long_count, A.long_cap);
  if (qn == 0) return;
  if (threadIdx.x == 0) mbar_init(base, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(base, bytes);
    for (uint32_t off = 0; off < bytes; off += 32768u)
      tma_bulk_g2s(base + kDeepRecOff + off, tab + (size_t)t_lo * kTreeRec + off, min(32768u, bytes - off), base);
  }
  __syncthreads();
  mbar_wait(base, 0);

  const int lane = threadIdx.x & 31;
  const int sub = lane & (GROUP - 1);
  const unsigned gmask = GROUP == 32 ? 0xffffffffu : (GROUP == 16 ? (0xffffu << (lane & 16)) : (GROUP == 8 ? (0xffu << (lane & 24)) : (0xfu << (lane & 28))));
  const int leader = lane & ~(GROUP - 1);
  const int t_hi = t_lo + ktrees;
  for (;;) {
    unsigned long long g = 0;
    if (sub == 0) g = atomicAdd(counter, 1ull);
    g = __shfl_sync(gmask, g, leader);
    if (g >= qn) break;
    const DeepWin w = deep_fetch<0>(A, T, g);
    int t0 = w.t0;
    float acc = w.acc;
    bool rejected = false;
    float thr_prev = 0.f;
    while (t0 < T.ntrees && !rejected) {
      const int t = min(t0 + sub, T.ntrees - 1);      // lanes past the last tree redo it harmlessly
      float thr, pred;
      if (t >= t_lo && t < t_hi) {
        const uint8_t* rec = dsm + kDeepRecOff + (uint32_t)(t - t_lo) * (uint32_t)kTreeRec;
        thr = *reinterpret_cast<const float*>(rec + 512);
        pred = deep_walk_smem(rec, w.pc, w.s, A.dim);
      } else {
        thr = __ldg(T.thresh + t);
        pred = deep_walk<0>(A, T, w.pc, w.rt, t, w.r, w.c, w.s, 0, A.dim);
      }
      const int nvalid = min(GROUP, T.ntrees - t0);
      for (int j = 0; j < nvalid; ++j) {              // the reference's sequential accumulation, :137-141
        acc += __shfl_sync(gmask, pred, leader + j);
        thr_prev = __shfl_sync(gmask, thr, leader + j);
        if (acc <= thr_prev) { rejected = true; break; }
      }
      t0 += GROUP;
    }
    if (!rejected && sub == 0) {
      const float q = acc - thr_prev;                 // :144
      if (q > 0.0f) {                                 // :246
        const int pos = atomicAdd(A.raw_count + w.frame, 1);
        if (pos < A.cap) A.raw[(size_t)w.frame * A.cap + pos] = RawDet{w.wid, q};
      }
    }
  }
}

// Resident range [t_lo, t_lo + k): t_lo and k even (16-byte alignment / size of the bulk copy), clipped to the cascade and to what
// one CTA's shared memory holds.  The launch puts as many CTAs on an SM as the range allows: a smaller range leaves more of the
// 256 KB L1/shared array to the L1 cache, which the pixel gathers live on.
static constexpr size_t kDeepSmemMax = 232448;
void launch_deep_smem(const ScanArgs& A, unsigned long long* counter, const uint8_t* tab_tiled, int num_sms, int threads, int group,
                      int t_lo, int k, cudaStream_t st) {
  const int ntrees = A.tab.ntrees;
  t_lo = std::max(0, std::min(t_lo, ntrees - 2)) & ~1;
  k = std::min(k, (int)((kDeepSmemMax - kDeepRecOff) / kTreeRec));
  k = std::max(2, std::min(k, ntrees - t_lo)) & ~1;
  const size_t smem = kDeepRecOff + (size_t)k * kTreeRec;
#define PIGO_DEEP_SMEM(G)                                                                                              \
  do {                                                                                                                 \
    raise_dyn_smem((const void*)deep_smem_kernel<G>, (int)smem);                                                     \
    int per_sm = 1;                                                                                                    \
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, deep_smem_kernel<G>, threads, smem) != cudaSuccess || per_sm < 1) { \
      cudaGetLastError();                                                                                              \
      per_sm = 1;                                                                                                      \
    }                                                                                                                  \
    deep_smem_kernel<G><<<num_sms * per_sm, threads, smem, st>>>(A, counter, tab_tiled, t_lo, k);                      \
  } while (0)
  if (group == 4) PIGO_DEEP_SMEM(4);
  else if (group == 16) PIGO_DEEP_SMEM(16);
  else if (group == 32) PIGO_DEEP_SMEM(32);
  else PIGO_DEEP_SMEM(8);
#undef PIGO_DEEP_SMEM
}

// Flat loop (option deep_flat=1): every iteration each lane group either fetches its next window or walks one step.  No group
// waits for another at a reconvergence point, but every fetch now delays the step of the three other groups; off by default,
// kept as a variant.
template <int GROUP, int ROT>
__global__ void __launch_bounds__(256) deep_flat_kernel(const ScanArgs A, unsigned long long* counter) {
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (GROUP - 1);
  const unsigned gmask = GROUP == 32 ? 0xffffffffu : (GROUP == 16 ? (0xffffu << (lane & 16)) : (0xffu << (lane & 24)));
  const int leader = lane & ~(GROUP - 1);
  const FaceTables T = A.tab;
  const uint32_t qn = min(*A.long_count, A.long_cap);
  const int lim = A.rows - 1;
  bool have = false, more = true;
  DeepWin w{};
  w.pc = A.frames; w.rt = A.rot_tab;
  for (;;) {
    if (!have && more) {
      unsigned long long g = 0;
      if (sub == 0) g = atomicAdd(counter, 1ull);
      g = __shfl_sync(gmask, g, leader);
      if (g >= qn) more = false;
      else { w = deep_fetch<ROT>(A, T, g); have = true; }
    }
    if (!__any_sync(FULL, have)) break;
    if (have) {
      const int t = min(w.t0 + sub, T.ntrees - 1);
      const float thr = __ldg(T.thresh + t);
      const float pred = deep_walk<ROT>(A, T, w.pc, w.rt, t, w.r, w.c, w.s, lim, A.dim);
      const int nvalid = min(GROUP, T.ntrees - w.t0);
      bool rejected = false;
      float thr_last = 0.f;
      for (int j = 0; j < nvalid; ++j) {
        w.acc += __shfl_sync(gmask, pred, leader + j);
        thr_last = __shfl_sync(gmask, thr, leader + j);
        if (w.acc <= thr_last) { rejected = true; break; }
      }
      w.t0 += GROUP;
      if (rejected) {
        have = false;
      } else if (w.t0 >= T.ntrees) {
        if (sub == 0) {
          const float q = w.acc - thr_last;
          if (q > 0.0f) {
            const int pos = atomicAdd(A.raw_count + w.frame, 1);
            if (pos < A.cap) A.raw[(size_t)w.frame * A.cap + pos] = RawDet{w.wid, q};
          }
        }
        have = false;
      }
    }
  }
}

template <int ROT, int FLAT>
static void launch_deep_g(const ScanArgs& A, unsigned long long* counter, int grid, int group, cudaStream_t st) {
  if (FLAT) {
    if (group == 8) deep_flat_kernel<8, ROT><<<grid, 256, 0, st>>>(A, counter);
    else if (group == 16) deep_flat_kernel<16, ROT><<<grid, 256, 0, st>>>(A, counter);
    else deep_flat_kernel<32, ROT><<<grid, 256, 0, st>>>(A, counter);
  } else {
    if (group == 8) deep_kernel<8, ROT><<<grid, 256, 0, st>>>(A, counter);
    else if (group == 16) deep_kernel<16, ROT><<<grid, 256, 0, st>>>(A, counter);
    else deep_kernel<32, ROT><<<grid, 256, 0, st>>>(A, counter);
  }
}

// Mixed-size calls: the round-1 loop only (deep_flat is a uniform-batch variant).
template <int ROT>
static void launch_deep_images(const ScanArgs& A, unsigned long long* counter, int grid, int group, cudaStream_t st) {
  if (group == 8) deep_kernel<8, ROT, 1><<<grid, 256, 0, st>>>(A, counter);
  else if (group == 16) deep_kernel<16, ROT, 1><<<grid, 256, 0, st>>>(A, counter);
  else deep_kernel<32, ROT, 1><<<grid, 256, 0, st>>>(A, counter);
}

// Ordered consumption: two 1024-thread CTAs per SM (every lane group of an SM draws from one of two runs), the L1/shared
// split set to the largest L1 (the kernel's only shared memory is its 8-byte cursor).
template <int GROUP, int ROT, int IMG>
static void launch_deep_chunked_g(const ScanArgs& A, unsigned long long* counter, int num_sms, cudaStream_t st) {
  cudaFuncSetAttribute(deep_kernel<GROUP, ROT, IMG, kDeepChunk>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxL1);
  deep_kernel<GROUP, ROT, IMG, kDeepChunk><<<num_sms * (2048 / kDeepOrdThreads), kDeepOrdThreads, 0, st>>>(A, counter);
}
template <int ROT, int IMG>
static void launch_deep_chunked(const ScanArgs& A, unsigned long long* counter, int num_sms, int group, cudaStream_t st) {
  if (group == 8) launch_deep_chunked_g<8, ROT, IMG>(A, counter, num_sms, st);
  else if (group == 16) launch_deep_chunked_g<16, ROT, IMG>(A, counter, num_sms, st);
  else launch_deep_chunked_g<32, ROT, IMG>(A, counter, num_sms, st);
}

void launch_deep(const ScanArgs& A, unsigned long long* counter, int num_sms, int group, bool ordered, cudaStream_t st) {
  const bool rot = A.rot_slot >= 0 && A.rot_tab != nullptr;
  const int grid = num_sms * 8;
  if (ordered) {
    if (A.images != nullptr) {
      if (rot) launch_deep_chunked<1, 1>(A, counter, num_sms, group, st); else launch_deep_chunked<0, 1>(A, counter, num_sms, group, st);
    } else {
      if (rot) launch_deep_chunked<1, 0>(A, counter, num_sms, group, st); else launch_deep_chunked<0, 0>(A, counter, num_sms, group, st);
    }
    return;
  }
  if (A.images != nullptr) {
    if (rot) launch_deep_images<1>(A, counter, grid, group, st); else launch_deep_images<0>(A, counter, grid, group, st);
    return;
  }
  const bool flat = g_opt.deep_flat.load() != 0;
  if (rot) { if (flat) launch_deep_g<1, 1>(A, counter, grid, group, st); else launch_deep_g<1, 0>(A, counter, grid, group, st); }
  else { if (flat) launch_deep_g<0, 1>(A, counter, grid, group, st); else launch_deep_g<0, 0>(A, counter, grid, group, st); }
}

// ---- Q2 in image order -------------------------------------------------------------------------------------
// A counting sort of the queue on (frame, cell of the window centre), cells of 2^shift x 2^shift pixels in row-major order:
// key + rank within the key's bin, an exclusive scan of the bins, a scatter.  Every kernel reads the item count on the
// device, so the sequence needs no host synchronisation.  The order within a bin is the order of the rank atomics, which
// changes nothing: the deep kernel appends detections with atomics and finalize_kernel sorts them.
struct DeepGrid {
  int shift, cells_x, cells;   // cell edge 2^shift, cells per row, cells per frame
};
static constexpr uint64_t kDeepMaxBins = 1u << 18;   // bins of one sort: the scan is one CTA
static DeepGrid deep_grid(int rows, int cols, int nframes) {
  DeepGrid g{6, 0, 0};   // 64-pixel cells, coarser when a group has too many frames for the bin budget
  for (;;) {
    g.cells_x = ((std::max(cols, 1) - 1) >> g.shift) + 1;
    g.cells = (((std::max(rows, 1) - 1) >> g.shift) + 1) * g.cells_x;
    if ((uint64_t)g.cells * (uint64_t)std::max(nframes, 1) <= kDeepMaxBins || g.shift >= 24) return g;
    ++g.shift;
  }
}

size_t deep_sort_aux_bytes(int rows, int cols, int nframes, size_t qcap) {
  const DeepGrid g = deep_grid(rows, cols, nframes);
  return (((size_t)g.cells * std::max(nframes, 1) + 1) & ~(size_t)1) * sizeof(uint32_t) + qcap * sizeof(uint2);
}

template <int IMG>
__global__ void __launch_bounds__(256) deep_key_kernel(const ScanArgs A, DeepGrid G, uint32_t* __restrict__ bins, uint2* __restrict__ keyrank) {
  const uint32_t qn = min(*A.long_count, A.long_cap);
  for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < qn; g += gridDim.x * blockDim.x) {
    const DeepPos p = deep_pos<IMG>(A, A.longq[g]);
    const uint32_t key = (uint32_t)p.frame * (uint32_t)G.cells + (uint32_t)((p.r >> G.shift) * G.cells_x + (p.c >> G.shift));
    keyrank[g] = make_uint2(key, atomicAdd(bins + key, 1u));
  }
}

// In-place exclusive scan of bins[0, n) by one CTA: each thread a contiguous segment.
__global__ void __launch_bounds__(1024) deep_scan_kernel(uint32_t* __restrict__ bins, int n) {
  __shared__ uint32_t warp_sum[32];
  const int per = (n + 1023) / 1024;
  const int lo = min(n, (int)threadIdx.x * per), hi = min(n, lo + per);
  uint32_t sum = 0;
  for (int i = lo; i < hi; ++i) sum += bins[i];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t incl = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) warp_sum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = warp_sum[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += v;
    }
    warp_sum[lane] = w;
  }
  __syncthreads();
  uint32_t run = incl - sum + (warp > 0 ? warp_sum[warp - 1] : 0u);
  for (int i = lo; i < hi; ++i) {
    const uint32_t v = bins[i];
    bins[i] = run;
    run += v;
  }
}

__global__ void __launch_bounds__(256) deep_scatter_kernel(const ScanArgs A, const uint32_t* __restrict__ bins, const uint2* __restrict__ keyrank,
                                                           DeepItem* __restrict__ sorted) {
  const uint32_t qn = min(*A.long_count, A.long_cap);
  for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < qn; g += gridDim.x * blockDim.x) {
    const uint2 kr = keyrank[g];
    sorted[bins[kr.x] + kr.y] = A.longq[g];
  }
}

// Sorts A.longq into `sorted`.  rows / cols: the frame size (mixed-size call: the largest of the group); aux: a buffer of
// deep_sort_aux_bytes(rows, cols, A.nframes, A.long_cap) bytes.
int launch_deep_sort(const ScanArgs& A, int rows, int cols, DeepItem* sorted, void* aux, int num_sms, cudaStream_t st) {
  const DeepGrid G = deep_grid(rows, cols, A.nframes);
  const int nbins = G.cells * std::max(A.nframes, 1);
  uint32_t* bins = (uint32_t*)aux;
  uint2* keyrank = (uint2*)(bins + ((nbins + 1) & ~1));
  if (cudaMemsetAsync(bins, 0, (size_t)nbins * sizeof(uint32_t), st) != cudaSuccess) return set_err(PIGO_E_CUDA, "cudaMemsetAsync failed");
  if (A.images != nullptr) deep_key_kernel<1><<<num_sms * 8, 256, 0, st>>>(A, G, bins, keyrank);
  else deep_key_kernel<0><<<num_sms * 8, 256, 0, st>>>(A, G, bins, keyrank);
  deep_scan_kernel<<<1, 1024, 0, st>>>(bins, nbins);
  deep_scatter_kernel<<<num_sms * 8, 256, 0, st>>>(A, bins, keyrank, sorted);
  g_launches += 3;
  return PIGO_OK;
}

// ---- rotated node table -------------------------------------------------------------------------------------
// One thread per (ladder entry, tree, node): the four deltas of core/pigo.go:167-171 in Go's 64-bit int arithmetic.
__global__ void __launch_bounds__(256) rot_table_kernel(FaceTables T, const ScaleEntry* __restrict__ plan, int nscales, int slot,
                                                        RotNode* __restrict__ out) {
  const size_t total = (size_t)nscales * T.ntrees * 64;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int idx = (int)(i & 63);
    const size_t st = i >> 6;
    const int t = (int)(st % (size_t)T.ntrees), si = (int)(st / (size_t)T.ntrees);
    const long long s = plan[si].s;
    const long long qsin = s * c_qsin[slot], qcos = s * c_qcos[slot];     // :159-160
    const int8_t* cd = T.codes + (size_t)t * 256 + 4 * idx;
    const long long k0 = cd[0], k1 = cd[1], k2 = cd[2], k3 = cd[3];
    RotNode n;
    n.dr1 = (int16_t)((qcos * k0 - qsin * k1) >> 16);
    n.dc1 = (int16_t)((qsin * k0 + qcos * k1) >> 16);
    n.dr2 = (int16_t)((qcos * k2 - qsin * k3) >> 16);
    n.dc2 = (int16_t)((qsin * k2 + qcos * k3) >> 16);
    out[i] = n;
  }
}

void launch_rot_table(const FaceTables& T, const ScaleEntry* plan, int nscales, int slot, RotNode* out, int grid, cudaStream_t st) {
  rot_table_kernel<<<grid, 256, 0, st>>>(T, plan, nscales, slot, out);
}

}  // namespace pigo
