// blur.cu -- box blur of the detected faces of decoded images, in place (pigo_blur_faces, pigo_blur_decoded): what a photo or
// camera service does with the faces after detection (the reference's examples/facedet/faceblur.py blurs a disc around every
// face with Q >= 5).  Everything is planned on the device from the faces, so that device faces need no host round trip:
//   blur_plan_kernel   per face: eligibility, disc radius d, box radius R, the disc's rows inside the image (work items)
//   blur_scan_kernel   per entry: the first work item of each entry (an entry with none is left alone by every later kernel)
//   blur_row_kernel    per plane row: running sums along the row                      } the plane's summed-area table,
//   blur_col_kernel    per 32-column strip: running sums down the columns             } uint32 mod 2^32
//   blur_paint_kernel  per disc row: Rmax + 1 into the entry's luma map (atomicMax), so the result does not depend on face order
//   blur_apply_kernel  per sample: covered (its anchor's map entry) -> the box mean from the table
// Cost per blurred sample is four table reads per rectangle whatever R is.  A box sum is below 255 * 2047^2 < 2^32, so the
// table's inclusion-exclusion is exact in wrapping uint32 arithmetic however large the plane's total is.  The table is a
// copy of the input: the apply kernel writes the planes while other samples' boxes still read the values they had before.
#include <algorithm>

#include "common.cuh"
#include "host.h"

namespace pigo {

// Index of the last k in [0, n) with first[k] <= q (first[0] <= q, first non-decreasing).
__device__ __forceinline__ int last_le(const uint64_t* __restrict__ first, int n, uint64_t q) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(first + mid) <= q) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ bool entry_active(const BlurArgs& A, int e) { return A.entry_first[e + 1] > A.entry_first[e]; }

// Exact floor(sqrt(v)) for 0 <= v < 2^62.
__device__ __forceinline__ long long isqrt64(long long v) {
  long long s = (long long)sqrt((double)v);
  while (s > 0 && s * s > v) --s;
  while ((s + 1) * (s + 1) <= v) ++s;
  return s;
}

// One warp per entry: face k of entry e becomes recs[e*cap + k] with its disc's rows inside the image as work items, numbered
// from the entry's first (a warp-wide running sum); entry_count[e] = the entry's items.
__global__ void __launch_bounds__(32) blur_plan_kernel(BlurArgs A) {
  const int lane = threadIdx.x;
  for (int e = blockIdx.x; e < A.n; e += gridDim.x) {
    const BlurEntry E = A.entries[e];
    const int nf = min(max(A.n_faces[e], 0), A.cap);
    uint64_t carry = 0;
    for (int base = 0; base < nf; base += 32) {
      const int k = base + lane;
      BlurFace r{0, 0, 0, 0, 0, 0};
      uint64_t cnt = 0;
      if (k < nf) {
        const pigo_det f = A.faces[(size_t)e * A.cap + k];
        const long long lim = 1ll << 24;
        if ((double)f.q >= A.min_q && f.scale >= 0 && f.scale <= lim && f.row >= -lim && f.row <= lim && f.col >= -lim && f.col <= lim) {
          const long long d = (long long)((double)f.scale * A.disc_ratio);
          const long long R = min(1023ll, max((long long)A.radius, (long long)((double)f.scale * A.radius_ratio)));
          const long long r0 = max(0ll, f.row - d), r1 = min((long long)E.height - 1, f.row + d);
          const long long c0 = max(0ll, f.col - d), c1 = min((long long)E.width - 1, f.col + d);
          r.row = f.row; r.col = f.col; r.d2 = d * d; r.r0 = (int32_t)r0; r.R = (int32_t)R;
          if (r0 <= r1 && c0 <= c1) cnt = (uint64_t)(r1 - r0 + 1);
        }
      }
      uint64_t incl = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint64_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      r.first = carry + incl - cnt;
      if (k < nf) A.recs[(size_t)e * A.cap + k] = r;
      carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) A.entry_first[e + 1] = carry;   // the entry's count, turned into firsts by blur_scan_kernel
  }
}

// One warp: entry_first[0..n] = exclusive running sum of the counts blur_plan_kernel left in entry_first[1..n].
__global__ void __launch_bounds__(32) blur_scan_kernel(BlurArgs A) {
  const int lane = threadIdx.x;
  uint64_t carry = 0;
  for (int base = 0; base < A.n; base += 32) {
    const int e = base + lane;
    const uint64_t cnt = e < A.n ? A.entry_first[e + 1] : 0;
    uint64_t incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    __syncwarp();
    if (e < A.n) A.entry_first[e + 1] = carry + incl;
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) A.entry_first[0] = 0;
}

// One warp per (plane, row): the row's running sums per channel into the table.
template <int C>
__device__ __forceinline__ void row_sums(const BlurUnit& U, int row, int lane) {
  const uint8_t* src = U.plane + (size_t)row * U.stride;
  uint32_t* dst = U.sat + (size_t)row * U.w * C;
  uint32_t carry[C];
#pragma unroll
  for (int c = 0; c < C; ++c) carry[c] = 0;
  for (int x0 = 0; x0 < U.w; x0 += 32) {
    const int x = x0 + lane;
    uint32_t s[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
      s[c] = x < U.w ? (uint32_t)src[(size_t)x * C + c] : 0u;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, s[c], o);
        if (lane >= o) s[c] += v;
      }
      s[c] += carry[c];
      carry[c] = __shfl_sync(0xffffffffu, s[c], 31);
    }
    if (x < U.w) {
      if (C == 4) reinterpret_cast<uint4*>(dst)[x] = make_uint4(s[0], s[C > 1 ? 1 : 0], s[C > 2 ? 2 : 0], s[C > 3 ? 3 : 0]);
      else dst[x] = s[0];
    }
  }
}

__global__ void __launch_bounds__(256) blur_row_kernel(BlurArgs A, uint64_t total) {
  const int lane = threadIdx.x & 31;
  const uint64_t nwarps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  for (uint64_t q = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < total; q += nwarps) {
    const int u = last_le(A.row_first, A.nunits, q);
    const BlurUnit U = A.units[u];
    if (!entry_active(A, U.entry)) continue;
    const int row = (int)(q - A.row_first[u]);
    if (U.chans == 4) row_sums<4>(U, row, lane);
    else row_sums<1>(U, row, lane);
  }
}

// One 32x32 block per (plane, strip of 32 table columns): each of the 32 thread rows sums a band of rows, the bands' sums are
// added up in shared memory, and each thread then writes its band's running sums from its offset (in place).
__global__ void __launch_bounds__(1024) blur_col_kernel(BlurArgs A, uint64_t total) {
  __shared__ uint32_t band[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (uint64_t s = blockIdx.x; s < total; s += gridDim.x) {
    const int u = last_le(A.strip_first, A.nunits, s);
    const BlurUnit U = A.units[u];
    if (!entry_active(A, U.entry)) continue;   // the same for the whole block
    const long long cols = (long long)U.w * U.chans;
    const long long col = (long long)(s - A.strip_first[u]) * 32 + tx;
    const int per = (U.h + 31) >> 5, y0 = min(U.h, ty * per), y1 = min(U.h, y0 + per);
    uint32_t* p = U.sat + col;
    uint32_t sum = 0;
    if (col < cols)
      for (int y = y0; y < y1; ++y) sum += p[(size_t)y * cols];
    band[ty][tx] = sum;
    __syncthreads();
    uint32_t run = 0;
    for (int t = 0; t < ty; ++t) run += band[t][tx];
    if (col < cols)
      for (int y = y0; y < y1; ++y) {
        run += p[(size_t)y * cols];
        p[(size_t)y * cols] = run;
      }
    __syncthreads();
  }
}

// One warp per disc row inside the image: Rmax + 1 over the row's covered pixels.
__global__ void __launch_bounds__(256) blur_paint_kernel(BlurArgs A) {
  const int lane = threadIdx.x & 31;
  const uint64_t total = A.entry_first[A.n];
  const uint64_t nwarps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  for (uint64_t q = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < total; q += nwarps) {
    const int e = last_le(A.entry_first, A.n, q);
    const uint64_t local = q - A.entry_first[e];
    const BlurFace* recs = A.recs + (size_t)e * A.cap;
    int lo = 0, hi = min(max(A.n_faces[e], 0), A.cap) - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (recs[mid].first <= local) lo = mid; else hi = mid - 1;
    }
    const BlurFace r = recs[lo];
    const BlurEntry E = A.entries[e];
    const long long y = r.r0 + (long long)(local - r.first), dy = y - r.row;
    const long long dx = isqrt64(r.d2 - dy * dy);
    const long long x0 = max(0ll, r.col - dx), x1 = min((long long)E.width - 1, r.col + dx);
    uint32_t* m = E.map + (size_t)y * E.width;
    for (long long x = x0 + lane; x <= x1; x += 32) atomicMax(m + x, (uint32_t)r.R + 1u);
  }
}

// Table value(s) at (y, x) of channel block C, 0 above or left of the plane.
template <int C>
__device__ __forceinline__ void sat_at(const BlurUnit& U, int y, int x, uint32_t v[C]) {
  if (y < 0 || x < 0) {
#pragma unroll
    for (int c = 0; c < C; ++c) v[c] = 0;
    return;
  }
  const uint32_t* p = U.sat + ((size_t)y * U.w + x) * C;
  if (C == 4) {
    const uint4 q = __ldg(reinterpret_cast<const uint4*>(p));
    v[0] = q.x; v[C > 1 ? 1 : 0] = q.y; v[C > 2 ? 2 : 0] = q.z; v[C > 3 ? 3 : 0] = q.w;
  } else {
    v[0] = __ldg(p);
  }
}

// acc += wgt * (sum over rows y0..y1, columns x0..x1), mod 2^32.
template <int C>
__device__ __forceinline__ void add_rect(const BlurUnit& U, uint32_t wgt, int y0, int y1, int x0, int x1, uint32_t acc[C]) {
  uint32_t a[C], b[C], c_[C], d[C];
  sat_at<C>(U, y1, x1, a); sat_at<C>(U, y0 - 1, x1, b); sat_at<C>(U, y1, x0 - 1, c_); sat_at<C>(U, y0 - 1, x0 - 1, d);
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] += wgt * (a[c] - b[c] - c_[c] + d[c]);
}

// The box mean of sample (j, i) with radii (ry, rx), indices clamped to the plane: the clamped box is the in-plane box, plus
// the first / last row and column counted once more for every row / column the box reaches past them, plus the corners.
template <int C>
__device__ __forceinline__ void box_mean(const BlurUnit& U, int j, int i, int ry, int rx) {
  const int y0 = max(0, j - ry), y1 = min(U.h - 1, j + ry), x0 = max(0, i - rx), x1 = min(U.w - 1, i + rx);
  const uint32_t ey0 = (uint32_t)max(0, ry - j), ey1 = (uint32_t)max(0, j + ry - (U.h - 1));
  const uint32_t ex0 = (uint32_t)max(0, rx - i), ex1 = (uint32_t)max(0, i + rx - (U.w - 1));
  uint32_t acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 0;
  add_rect<C>(U, 1u, y0, y1, x0, x1, acc);
  if (ey0) add_rect<C>(U, ey0, 0, 0, x0, x1, acc);
  if (ey1) add_rect<C>(U, ey1, U.h - 1, U.h - 1, x0, x1, acc);
  if (ex0) add_rect<C>(U, ex0, y0, y1, 0, 0, acc);
  if (ex1) add_rect<C>(U, ex1, y0, y1, U.w - 1, U.w - 1, acc);
  if (ey0 && ex0) add_rect<C>(U, ey0 * ex0, 0, 0, 0, 0, acc);
  if (ey0 && ex1) add_rect<C>(U, ey0 * ex1, 0, 0, U.w - 1, U.w - 1, acc);
  if (ey1 && ex0) add_rect<C>(U, ey1 * ex0, U.h - 1, U.h - 1, 0, 0, acc);
  if (ey1 && ex1) add_rect<C>(U, ey1 * ex1, U.h - 1, U.h - 1, U.w - 1, U.w - 1, acc);
  const uint32_t n = (uint32_t)(2 * ry + 1) * (uint32_t)(2 * rx + 1);
  uint8_t* dst = U.plane + (size_t)j * U.stride + (size_t)i * C;
#pragma unroll
  for (int c = 0; c < C; ++c) dst[c] = (uint8_t)((acc[c] + n / 2) / n);
}

// One thread per sample of every plane: its anchor luma pixel's map entry says whether and with which R it is blurred.
__global__ void __launch_bounds__(256) blur_apply_kernel(BlurArgs A, uint64_t total) {
  for (uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (uint64_t)gridDim.x * blockDim.x) {
    const int u = last_le(A.px_first, A.nunits, q);
    const BlurUnit U = A.units[u];
    if (!entry_active(A, U.entry)) continue;
    const uint32_t local = (uint32_t)(q - A.px_first[u]);   // < w * h < 2^31
    const int j = (int)(local / (uint32_t)U.w), i = (int)(local - (uint32_t)j * (uint32_t)U.w);
    const BlurEntry E = A.entries[U.entry];
    const int ay = min(max(((U.min_y >> U.ys) + j) << U.ys, U.min_y), U.min_y + E.height - 1) - U.min_y;
    const int ax = min(max(((U.min_x >> U.xs) + i) << U.xs, U.min_x), U.min_x + E.width - 1) - U.min_x;
    const uint32_t m = E.map[(size_t)ay * E.width + ax];
    if (m == 0) continue;
    const int R = (int)m - 1;
    if (U.chans == 4) box_mean<4>(U, j, i, R >> U.ys, R >> U.xs);
    else box_mean<1>(U, j, i, R >> U.ys, R >> U.xs);
  }
}

void launch_blur(const BlurArgs& A, uint64_t rows, uint64_t strips, uint64_t samples, int num_sms, cudaStream_t st) {
  auto grid = [&](uint64_t want, uint64_t cap) { return (int)std::max<uint64_t>(1, std::min<uint64_t>(want, cap)); };
  const uint64_t cap = (uint64_t)num_sms * 16;
  timing_begin(T_BLUR, st);
  blur_plan_kernel<<<grid(A.n, cap * 8), 32, 0, st>>>(A);
  timing_end(T_BLUR, st);
  timing_begin(T_BLUR, st);
  blur_scan_kernel<<<1, 32, 0, st>>>(A);
  timing_end(T_BLUR, st);
  timing_begin(T_BLUR, st);
  blur_row_kernel<<<grid((rows + 7) / 8, cap), 256, 0, st>>>(A, rows);
  timing_end(T_BLUR, st);
  timing_begin(T_BLUR, st);
  blur_col_kernel<<<grid(strips, (uint64_t)num_sms * 2), dim3(32, 32), 0, st>>>(A, strips);
  timing_end(T_BLUR, st);
  timing_begin(T_BLUR, st);
  blur_paint_kernel<<<num_sms * 8, 256, 0, st>>>(A);
  timing_end(T_BLUR, st);
  timing_begin(T_BLUR, st);
  blur_apply_kernel<<<grid((samples + 255) / 256, cap), 256, 0, st>>>(A, samples);
  timing_end(T_BLUR, st);
  g_launches += 6;
}

}  // namespace pigo
