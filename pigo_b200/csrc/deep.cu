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
#include <algorithm>

#include "common.cuh"
#include "host.h"

namespace pigo {

// One tree (index t) of the window: the leaf value.  Unrotated: pc = the window's centre pixel; rotated: pc = the frame,
// (r, c) the centre, rt = this scale's node table.
template <int ROT>
__device__ __forceinline__ float deep_walk(const ScanArgs& A, const FaceTables& T, const uint8_t* __restrict__ pc, const RotNode* __restrict__ rt,
                                           int t, int r, int c, int s, int lim) {
  const int2* tp2 = reinterpret_cast<const int2*>(T.preds + (size_t)t * 64);
  int idx = 1;
  if (ROT) {
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
      const unsigned p1 = __ldg(pc + (size_t)r1 * A.dim + c1), p2 = __ldg(pc + (size_t)r2 * A.dim + c2);
      const bool right = p1 <= p2;                  // core/pigo.go:179
      cur = right ? make_uint2(kids.z, kids.w) : make_uint2(kids.x, kids.y);
      leafbits = right ? lv.y : lv.x;
      idx = 2 * idx + (right ? 1 : 0);
    }
    return __int_as_float(leafbits);
  } else {
    // child-pair prefetch: both children of node idx (codes: bytes 8*idx.., leaves: floats 2*idx-64..) are fetched
    // with one 64-bit load that is in flight together with the two pixel gathers
    const int2* tc2 = reinterpret_cast<const int2*>(T.codes + (size_t)t * 256);
    int cw = __ldg(reinterpret_cast<const int*>(tc2) + 1);
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const int2 kids = j < 5 ? __ldg(tc2 + idx) : __ldg(tp2 + (idx - 32));
      const int o1 = (((int)(int8_t)(cw) * s) >> 8) * A.dim + (((int)(int8_t)(cw >> 8) * s) >> 8);
      const int o2 = (((int)(int8_t)(cw >> 16) * s) >> 8) * A.dim + (((cw >> 24) * s) >> 8);
      const unsigned p1 = __ldg(pc + o1), p2 = __ldg(pc + o2);
      const bool right = p1 <= p2;                  // core/pigo.go:129-135
      cw = right ? kids.y : kids.x;
      idx = 2 * idx + (right ? 1 : 0);
    }
    return __int_as_float(cw);
  }
}

// Decodes a queue item: window geometry from the ladder entry the producer packed (0xffff = not known: search).
struct DeepWin {
  uint32_t wid;
  int frame, t0, s, r, c;
  float acc;
  const uint8_t* pc;
  const RotNode* rt;
};
template <int ROT>
__device__ __forceinline__ DeepWin deep_fetch(const ScanArgs& A, const FaceTables& T, unsigned long long g) {
  const DeepItem it = A.longq[g];
  int si = (int)(it.frame_si >> 16);
  if (si == 0xffff) si = find_scale(A.plan, A.nscales, it.wid);
  const ScaleEntry e = A.plan[si];
  const uint32_t local = it.wid - e.wbase;
  const uint32_t ri = local / (uint32_t)e.ncols, ci = local - ri * (uint32_t)e.ncols;
  DeepWin w;
  w.s = e.s; w.wid = it.wid; w.frame = (int)(it.frame_si & 0xffffu); w.t0 = it.tree; w.acc = it.acc;
  w.r = e.off + (int)ri * e.step; w.c = e.off + (int)ci * e.step;
  w.pc = A.frames + (size_t)w.frame * A.frame_stride;
  w.rt = A.rot_tab;
  if (ROT) w.rt = A.rot_tab + (size_t)si * T.ntrees * 64;
  else w.pc += (size_t)w.r * A.dim + w.c;
  return w;
}

// Round-1 loop structure: the lane groups of a warp fetch together, then the warp stays in the step loop until its slowest
// window is done (measured faster than the flat loop below: one fetch latency per 32/GROUP windows instead of one per window).
template <int GROUP, int ROT>
__global__ void __launch_bounds__(256) deep_kernel(const ScanArgs A, unsigned long long* counter) {
  const int lane = threadIdx.x & 31;
  const int sub = lane & (GROUP - 1);
  const unsigned gmask = GROUP == 32 ? 0xffffffffu : (GROUP == 16 ? (0xffffu << (lane & 16)) : (0xffu << (lane & 24)));
  const int leader = lane & ~(GROUP - 1);
  const FaceTables T = A.tab;
  const uint32_t qn = min(*A.long_count, A.long_cap);
  const int lim = A.rows - 1;
  for (;;) {
    unsigned long long g = 0;
    if (sub == 0) g = atomicAdd(counter, 1ull);
    g = __shfl_sync(gmask, g, leader);
    if (g >= qn) break;
    const DeepWin w = deep_fetch<ROT>(A, T, g);
    int t0 = w.t0;
    float acc = w.acc;
    bool rejected = false;
    float thr_prev = 0.f;
    while (t0 < T.ntrees && !rejected) {
      const int t = min(t0 + sub, T.ntrees - 1);      // lanes past the last tree redo it harmlessly
      const float thr = __ldg(T.thresh + t);
      const float pred = deep_walk<ROT>(A, T, w.pc, w.rt, t, w.r, w.c, w.s, lim);
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
        pred = deep_walk<0>(A, T, w.pc, w.rt, t, w.r, w.c, w.s, 0);
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
    cudaFuncSetAttribute(deep_smem_kernel<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);                 \
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
      const float pred = deep_walk<ROT>(A, T, w.pc, w.rt, t, w.r, w.c, w.s, lim);
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

void launch_deep(const ScanArgs& A, unsigned long long* counter, int grid, int group, cudaStream_t st) {
  const bool rot = A.rot_slot >= 0 && A.rot_tab != nullptr;
  const bool flat = g_opt.deep_flat.load() != 0;
  if (rot) { if (flat) launch_deep_g<1, 1>(A, counter, grid, group, st); else launch_deep_g<1, 0>(A, counter, grid, group, st); }
  else { if (flat) launch_deep_g<0, 1>(A, counter, grid, group, st); else launch_deep_g<0, 0>(A, counter, grid, group, st); }
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
