// finalize.cu -- restores the reference's emission order of RunCascade (core/pigo.go:226-249: scale-major,
// then row, then col) from the unordered RawDet records the scan kernels append, and writes pigo_det.
// Detections are rare (tens..hundreds per frame), so a rank sort on the unique in-frame window index is
// enough: rank(i) = #{j : wid_j < wid_i}.  One thread per detection, keys streamed through shared memory.
#include "common.cuh"
#include "host.h"

namespace pigo {

// IMG = 1 (mixed-size call): frame = image, decoded against that image's plan (images[frame]); the results go to the
// caller's slot images[frame].out_index of out / n_out.
template <int IMG>
__global__ void __launch_bounds__(256) finalize_kernel(const RawDet* __restrict__ raw, const int32_t* __restrict__ raw_count,
                                                       int cap, const ScaleEntry* __restrict__ plan, int nscales,
                                                       pigo_det* __restrict__ out, int32_t* __restrict__ n_out,
                                                       const ImageDesc* __restrict__ images) {
  const int frame = blockIdx.y;
  const int total = raw_count[frame];
  const int n = min(total, cap);
  const int dst = IMG ? images[frame].out_index : frame;
  if (blockIdx.x == 0 && threadIdx.x == 0) n_out[dst] = total;  // required count (may exceed cap)
  if ((int)(blockIdx.x * blockDim.x) >= n) return;
  const RawDet* rf = raw + (size_t)frame * cap;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  RawDet me = (i < n) ? rf[i] : RawDet{0xffffffffu, 0.f};
  __shared__ uint32_t keys[256];
  int rank = 0;
  for (int base = 0; base < n; base += 256) {
    const int j = base + threadIdx.x;
    keys[threadIdx.x] = (j < n) ? rf[j].wid : 0xffffffffu;
    __syncthreads();
    const int m = min(256, n - base);
    for (int k = 0; k < m; ++k) rank += (keys[k] < me.wid) ? 1 : 0;
    __syncthreads();
  }
  if (i < n) {
    if (IMG) { plan += images[frame].plan_off; nscales = images[frame].nscales; }
    const int si = find_scale(plan, nscales, me.wid);
    const ScaleEntry e = plan[si];
    const uint32_t local = me.wid - e.wbase;
    const uint32_t ri = local / (uint32_t)e.ncols;
    const uint32_t ci = local - ri * (uint32_t)e.ncols;
    pigo_det d;
    d.row = e.off + (int)ri * e.step;
    d.col = e.off + (int)ci * e.step;
    d.scale = e.s;
    d.q = me.q;
    out[(size_t)dst * cap + rank] = d;
  }
}

void launch_finalize(const RawDet* raw, const int32_t* raw_count, int cap, const ScaleEntry* plan, int nscales, pigo_det* out,
                     int32_t* n_out, int nframes, cudaStream_t st) {
  dim3 grid((cap + 255) / 256, nframes);
  finalize_kernel<0><<<grid, 256, 0, st>>>(raw, raw_count, cap, plan, nscales, out, n_out, nullptr);
}

void launch_finalize_images(const RawDet* raw, const int32_t* raw_count, int cap, const ScaleEntry* plan, const ImageDesc* images,
                            pigo_det* out, int32_t* n_out, int nimages, cudaStream_t st) {
  dim3 grid((cap + 255) / 256, nimages);
  finalize_kernel<1><<<grid, 256, 0, st>>>(raw, raw_count, cap, plan, 0, out, n_out, images);
}

}  // namespace pigo
