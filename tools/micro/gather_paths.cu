// Micro-benchmark: lane-divergent 1-byte gathers (the access pattern of the straggler / deep / rotated / pupil kernels)
// through (a) ld.global.nc, (b) tex1Dfetch on a linear texture, (c) tex2D on a pitch-linear texture.
// Each thread emulates tree walks: 6 dependent levels, 2 byte samples per level inside an s x s patch around its window.
//   mkdir -p build && nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/gather_paths tools/micro/gather_paths.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <vector>

__device__ __forceinline__ uint32_t hash32(uint32_t x) { x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x; }

template <int MODE>
__global__ void __launch_bounds__(256) walk(const uint8_t* __restrict__ img, cudaTextureObject_t t1, cudaTextureObject_t t2, int rows, int cols,
                                            int nframes, int s, int walks, int coherent, unsigned* sink) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t h = hash32(tid * 2654435761u + 12345u);
  unsigned acc = 0;
  for (int w = 0; w < walks; ++w) {
    // window centre: coherent = neighbouring lanes are neighbouring windows (step s/5), else random
    int f, r, c;
    if (coherent) {
      const uint32_t g = (tid + w * gridDim.x * blockDim.x);
      const int step = s / 5 > 0 ? s / 5 : 1;
      const int ncol = (cols - 2 * s) / step, nrow = (rows - 2 * s) / step;
      c = s + (int)(g % ncol) * step; r = s + (int)((g / ncol) % nrow) * step; f = (int)((g / (ncol * nrow)) % nframes);
    } else {
      h = hash32(h + w);
      f = h % nframes; r = s + (hash32(h ^ 0x1234u) % (rows - 2 * s)); c = s + (hash32(h ^ 0x9876u) % (cols - 2 * s));
    }
    uint32_t idx = 1;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const uint32_t k = hash32(idx * 0x9E3779B9u + w);   // "node codes"
      const int dr1 = (int)(k & 0xff) * s / 256 - s / 2, dc1 = (int)((k >> 8) & 0xff) * s / 256 - s / 2;
      const int dr2 = (int)((k >> 16) & 0xff) * s / 256 - s / 2, dc2 = (int)(k >> 24) * s / 256 - s / 2;
      unsigned p1, p2;
      if (MODE == 0) {
        const uint8_t* b = img + (size_t)f * rows * cols;
        p1 = __ldg(b + (r + dr1) * cols + c + dc1); p2 = __ldg(b + (r + dr2) * cols + c + dc2);
      } else if (MODE == 1) {
        const int base = f * rows * cols;
        p1 = tex1Dfetch<unsigned char>(t1, base + (r + dr1) * cols + c + dc1); p2 = tex1Dfetch<unsigned char>(t1, base + (r + dr2) * cols + c + dc2);
      } else {
        p1 = tex2D<unsigned char>(t2, (float)(c + dc1), (float)(f * rows + r + dr1)); p2 = tex2D<unsigned char>(t2, (float)(c + dc2), (float)(f * rows + r + dr2));
      }
      idx = 2 * idx + (p1 <= p2 ? 1 : 0);
    }
    acc += idx;
  }
  if (acc == 0xdeadbeef) *sink = acc;
}

int main() {
  const int rows = 1080, cols = 1920;
  for (int nframes : {8, 60}) {
    const size_t n = (size_t)nframes * rows * cols;
    uint8_t* d; cudaMalloc(&d, n);
    std::vector<uint8_t> h(n); for (size_t i = 0; i < n; ++i) h[i] = (uint8_t)(i * 2654435761u >> 13);
    cudaMemcpy(d, h.data(), n, cudaMemcpyHostToDevice);
    cudaResourceDesc rd{}; rd.resType = cudaResourceTypeLinear; rd.res.linear.devPtr = d; rd.res.linear.desc = cudaCreateChannelDesc<unsigned char>(); rd.res.linear.sizeInBytes = n;
    cudaTextureDesc td{}; td.readMode = cudaReadModeElementType; td.filterMode = cudaFilterModePoint; td.addressMode[0] = td.addressMode[1] = cudaAddressModeClamp;
    cudaTextureObject_t t1 = 0, t2 = 0;
    cudaError_t e1 = cudaCreateTextureObject(&t1, &rd, &td, nullptr);
    cudaResourceDesc r2{}; r2.resType = cudaResourceTypePitch2D; r2.res.pitch2D.devPtr = d; r2.res.pitch2D.desc = cudaCreateChannelDesc<unsigned char>();
    r2.res.pitch2D.width = cols; r2.res.pitch2D.height = (size_t)nframes * rows; r2.res.pitch2D.pitchInBytes = cols;
    cudaError_t e2 = cudaCreateTextureObject(&t2, &r2, &td, nullptr);
    printf("frames=%d (%.0f MB) tex1D:%s tex2D:%s\n", nframes, n / 1e6, cudaGetErrorString(e1), cudaGetErrorString(e2));
    unsigned* sink; cudaMalloc(&sink, 4);
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    for (int s : {24, 100}) for (int coherent : {0, 1}) for (int mode = 0; mode < 3; ++mode) {
      if ((mode == 1 && e1) || (mode == 2 && e2)) continue;
      const int grid = 132 * 8, walks = 64;
      float best = 1e9;
      for (int rep = 0; rep < 4; ++rep) {
        cudaEventRecord(a);
        if (mode == 0) walk<0><<<grid, 256>>>(d, t1, t2, rows, cols, nframes, s, walks, coherent, sink);
        if (mode == 1) walk<1><<<grid, 256>>>(d, t1, t2, rows, cols, nframes, s, walks, coherent, sink);
        if (mode == 2) walk<2><<<grid, 256>>>(d, t1, t2, rows, cols, nframes, s, walks, coherent, sink);
        cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b); if (rep && ms < best) best = ms;
      }
      const double nw = (double)grid * 256 * walks;
      printf("  s=%3d %s mode=%s: %.3f ms  %.1f Gwalk/s  %.1f Gsample/s (%s)\n", s, coherent ? "coherent" : "random  ",
             mode == 0 ? "ldg  " : mode == 1 ? "tex1D" : "tex2D", best, nw / best / 1e6, nw * 12 / best / 1e6, cudaGetErrorString(cudaGetLastError()));
    }
    cudaDestroyTextureObject(t1); cudaDestroyTextureObject(t2); cudaFree(d); cudaFree(sink);
  }
  return 0;
}
