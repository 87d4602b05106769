// cluster.cu -- ClusterDetections (core/pigo.go:262-308) on the device, one CTA per frame.
//
//  1. in-place sort of the frame's detections by Q ascending (:264-266).  Go's sort.Slice is unstable and
//     leaves tie order unspecified; we sort stably (rank = #{q_j < q_i} + #{q_j == q_i, j < i}).
//  2. greedy seed selection (:282-301): detection i is a seed iff no earlier seed overlapped it with
//     IoU > threshold.  Sequential over seeds, parallel over j; one barrier per SEED, not per detection.
//  3. per-seed accumulation, one thread per seed, j ascending so that the float32 q-sum (:298) has the
//     reference's addition order; integer sums and the truncating division (:303) as in Go.
// IoU is float64 with the reference's operation order (:268-278); the library is built with -fmad=false.
//
// The angle sweep (pigo_*_images_sweep) merges the lists of one image at several angles into one list D_i and clusters
// it with the same kernel: sweep_compact_kernel concatenates the lists with an angle tag per detection, a segmented radix
// sort orders each image's list by (Q, position in D_i) -- the stable sort of step 1 without its O(n^2) ranks -- and
// cluster_kernel<true> takes that order instead of step 1 and also reports, per cluster, the tag of its largest-Q member.
#include <cub/device/device_segmented_radix_sort.cuh>

#include "common.cuh"
#include "host.h"

namespace pigo {

__device__ __forceinline__ double calc_iou(const pigo_det& a, const pigo_det& b) {
  const double r1 = a.row, c1 = a.col, s1 = a.scale;
  const double r2 = b.row, c2 = b.col, s2 = b.scale;
  const double over_row = fmax(0.0, fmin(r1 + s1 / 2, r2 + s2 / 2) - fmax(r1 - s1 / 2, r2 - s2 / 2));
  const double over_col = fmax(0.0, fmin(c1 + s1 / 2, c2 + s2 / 2) - fmax(c1 - s1 / 2, c2 - s2 / 2));
  return __ddiv_rn(__dmul_rn(over_row, over_col),
                   __dsub_rn(__dadd_rn(__dmul_rn(s1, s1), __dmul_rn(s2, s2)), __dmul_rn(over_row, over_col)));
}

// scratch per frame: tmp[cap] (pigo_det), flags[cap] (u8: assigned), seeds[cap] (i32)
// TAGGED (sweep merge): step 1 takes the order of the segmented sort (SweepTags.keys: position in the low 32 bits) instead
// of ranking, and every cluster also gets the tag of its member with the largest Q (the first such member in sorted order,
// i.e. the earliest in D_i among equal Q) and that tag's rotation slot.
template <bool TAGGED>
__global__ void __launch_bounds__(256) cluster_kernel(pigo_det* __restrict__ dets, const int32_t* __restrict__ n_in, int cap,
                                                      double thr, pigo_det* __restrict__ tmp, uint8_t* flags,
                                                      int32_t* __restrict__ seeds, pigo_det* __restrict__ out, int out_cap,
                                                      int32_t* __restrict__ n_out, const SweepTags tg) {
  const int frame = blockIdx.x;
  const int n = max(0, min(n_in[frame], cap));
  pigo_det* d = dets + (size_t)frame * cap;
  pigo_det* tp = tmp + (size_t)frame * cap;
  uint8_t* asg = flags + (size_t)frame * cap;
  int32_t* sd = seeds + (size_t)frame * cap;
  const int tid = threadIdx.x, nt = blockDim.x;
  __shared__ int s_nseeds;

  // ---- 1. stable rank sort by q ascending
  const uint64_t* order = TAGGED ? tg.keys + (size_t)frame * cap : nullptr;
  for (int i = tid; i < n; i += nt) {
    if (TAGGED) {
      tp[i] = d[(uint32_t)order[i]];
    } else {
      const float qi = d[i].q;
      int rank = 0;
      for (int j = 0; j < n; ++j) {
        const float qj = d[j].q;
        rank += (qj < qi || (qj == qi && j < i)) ? 1 : 0;
      }
      tp[rank] = d[i];
    }
    asg[i] = 0;
  }
  __syncthreads();
  for (int i = tid; i < n; i += nt) d[i] = tp[i];
  if (tid == 0) { s_nseeds = 0; }
  __syncthreads();

  // ---- 2. seeds
  for (int i = 0; i < n; ++i) {
    // Uniform branch: asg[i] is written only inside the marking loops of EARLIER seed iterations, each of which ends in a
    // barrier.  The seed's own flag is deliberately not set below (j != i): the reference sets assignments[i] there
    // (IoU(i,i) = 1 > thr, core/pigo.go:290-296) but never reads it again, and setting it here would let a lagging warp
    // of this same iteration read 1 and skip the barrier the others are waiting at.
    if (*(volatile uint8_t*)(asg + i)) continue;
    const pigo_det di = d[i];
    for (int j = tid; j < n; j += nt)
      if (j != i && calc_iou(di, d[j]) > thr) asg[j] = 1;
    if (tid == 0) sd[s_nseeds++] = i;
    __syncthreads();
  }
  __syncthreads();
  const int nseeds = s_nseeds;

  // ---- 3. accumulate each seed's cluster (j ascending); tp[] is reused for the per-seed results
  for (int k = tid; k < nseeds; k += nt) {
    const pigo_det di = d[sd[k]];
    long long r = 0, c = 0, s = 0, cnt = 0;
    float q = 0.f;
    int best = -1;   // TAGGED: sorted position of the first member with the largest Q
    for (int j = 0; j < n; ++j) {
      const pigo_det dj = d[j];
      if (calc_iou(di, dj) > thr) {
        r += dj.row; c += dj.col; s += dj.scale;
        q = __fadd_rn(q, dj.q);
        if (TAGGED && (cnt == 0 || dj.q > d[best].q)) best = j;
        ++cnt;
      }
    }
    pigo_det o;
    if (cnt > 0) { o.row = (int)(r / cnt); o.col = (int)(c / cnt); o.scale = (int)(s / cnt); o.q = q; }
    else { o.row = o.col = 0; o.scale = -1; o.q = 0.f; }  // scale -1 marks "n == 0" (:302), dropped below
    tp[k] = o;
    if (TAGGED) sd[k] = best >= 0 ? tg.tag[(size_t)frame * cap + (uint32_t)order[best]] : -1;   // this thread's seed is read above
  }
  __syncthreads();
  if (tid == 0) {
    int m = 0;
    pigo_det* of = out + (size_t)frame * out_cap;
    for (int k = 0; k < nseeds; ++k) {
      if (tp[k].scale == -1 && tp[k].row == 0 && tp[k].col == 0) {
        // distinguish the marker from a genuine cluster: genuine clusters have cnt > 0 and scale >= 0 whenever
        // input scales are >= 0 (always true for RunCascade output)
        continue;
      }
      if (m < out_cap) {
        of[m] = tp[k];
        if (TAGGED && tg.out_tag) tg.out_tag[(size_t)frame * out_cap + m] = sd[k];
        if (TAGGED && tg.out_rot) tg.out_rot[(size_t)frame * out_cap + m] = tg.slot_of[sd[k]];
      }
      ++m;
    }
    n_out[frame] = m;
    for (int k = m; TAGGED && k < out_cap; ++k) {   // unused face slots: defined values
      if (tg.out_tag) tg.out_tag[(size_t)frame * out_cap + k] = -1;
      if (tg.out_rot) tg.out_rot[(size_t)frame * out_cap + k] = -1;
    }
  }
}

void launch_cluster(pigo_det* dets, const int32_t* n_in, int cap, double thr, pigo_det* tmp, uint8_t* flags, int32_t* seeds,
                    pigo_det* out, int out_cap, int32_t* n_out, int nframes, cudaStream_t st) {
  cluster_kernel<false><<<nframes, 256, 0, st>>>(dets, n_in, cap, thr, tmp, flags, seeds, out, out_cap, n_out, SweepTags{});
}

// ---- angle sweep merge -----------------------------------------------------------------------------------------------
// Q as an unsigned key that orders like the float (-0 and +0 equal, as the reference's < compares them).
__device__ __forceinline__ uint32_t q_key(float q) {
  const uint32_t b = q == 0.f ? 0u : __float_as_uint(q);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// One CTA per image: D_i = the lists of entries i*nangles .. i*nangles+nangles-1 (angle a's list raw[e][0..min(cnt, det_cap)))
// concatenated in angle order into merged[i][0..n_i), with tag[i][p] = a and key[i][p] = (q_key, p).
__global__ void __launch_bounds__(256) sweep_compact_kernel(const pigo_det* __restrict__ raw, const int32_t* __restrict__ raw_count,
                                                            int nangles, int det_cap, int seg_cap, pigo_det* __restrict__ merged,
                                                            int32_t* __restrict__ tag, uint64_t* __restrict__ keys,
                                                            int32_t* __restrict__ seg_begin, int32_t* __restrict__ seg_end,
                                                            int32_t* __restrict__ n_merged) {
  const int img = blockIdx.x, tid = threadIdx.x;
  const size_t base = (size_t)img * seg_cap;
  int pos = 0;   // prefix over this image's counts (every thread walks the same prefix)
  for (int a = 0; a < nangles; ++a) {
    const size_t e = (size_t)img * nangles + a;
    const int n = max(0, min(raw_count[e], det_cap));
    for (int j = tid; j < n; j += blockDim.x) {
      const pigo_det d = raw[e * det_cap + j];
      const int p = pos + j;
      merged[base + p] = d;
      tag[base + p] = a;
      keys[base + p] = ((uint64_t)q_key(d.q) << 32) | (uint32_t)p;
    }
    pos += n;
  }
  if (tid == 0) {
    seg_begin[img] = (int32_t)base;
    seg_end[img] = (int32_t)base + pos;
    n_merged[img] = pos;
  }
}

size_t sweep_sort_bytes(int nimages, int seg_cap) {
  size_t bytes = 0;
  cub::DeviceSegmentedRadixSort::SortKeys(nullptr, bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, nimages * seg_cap, nimages,
                                          (const int32_t*)nullptr, (const int32_t*)nullptr);
  return bytes;
}

int launch_sweep_merge(const pigo_det* raw, const int32_t* raw_count, int nimages, int nangles, int det_cap, double thr, const SweepScratch& S,
                       const int32_t* slot_of, pigo_det* out, int out_cap, int32_t* n_out, int32_t* out_tag, int32_t* out_rot, cudaStream_t st) {
  const int seg_cap = nangles * det_cap;
  sweep_compact_kernel<<<nimages, 256, 0, st>>>(raw, raw_count, nangles, det_cap, seg_cap, S.merged, S.tag, S.keys_in, S.seg_begin, S.seg_end,
                                                S.n_merged);
  size_t bytes = S.sort_bytes;
  if (cub::DeviceSegmentedRadixSort::SortKeys(S.sort_temp, bytes, S.keys_in, S.keys_out, nimages * seg_cap, nimages, S.seg_begin, S.seg_end,
                                              0, 64, st) != cudaSuccess)
    return -1;
  const SweepTags tg{S.keys_out, S.tag, slot_of, out_tag, out_rot};
  cluster_kernel<true><<<nimages, 256, 0, st>>>(S.merged, S.n_merged, seg_cap, thr, S.tmp, S.flags, S.seeds, out, out_cap, n_out, tg);
  return 0;
}

}  // namespace pigo
