// grayscale.cu -- RgbToGrayscale (core/grayscale.go:8-23) for NRGBA pixels: the stage right before the hot path
// (SURVEY.md section 8f, row N2).  Pure streaming: 4 bytes in, 1 byte out per pixel => HBM-bound (5 B/pixel);
// 16 pixels per thread (4 x 16-byte loads, one 16-byte store), float64 arithmetic in the reference's operation order
// (the library is built with -fmad=false).
#include <algorithm>

#include "common.cuh"
#include "host.h"

namespace pigo {

// color.NRGBA.RGBA(): c = v | v<<8; c = c*A/0xff  (image/color)
__device__ __forceinline__ uint32_t luma(uint32_t px) {
  const uint32_t a = px >> 24;
  const uint32_t r = ((px & 0xffu) * 0x101u) * a / 0xffu;
  const uint32_t g = (((px >> 8) & 0xffu) * 0x101u) * a / 0xffu;
  const uint32_t b = (((px >> 16) & 0xffu) * 0x101u) * a / 0xffu;
  const double y = __dadd_rn(__dadd_rn(__dmul_rn(0.299, (double)r), __dmul_rn(0.587, (double)g)), __dmul_rn(0.114, (double)b));
  return (uint32_t)(int)(y / 256.0) & 0xffu;   // uint8(float64) truncation; y/256 < 256
}

__global__ void __launch_bounds__(256) gray_kernel(const uint32_t* __restrict__ rgba, size_t npix, uint8_t* __restrict__ gray, int vec_ok) {
  const size_t nvec = vec_ok ? npix / 16 : 0;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (size_t)gridDim.x * blockDim.x) {
    const uint4* src = reinterpret_cast<const uint4*>(rgba) + v * 4;
    uint4 q[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) q[k] = __ldg(src + k);
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = luma(q[k].x) | (luma(q[k].y) << 8) | (luma(q[k].z) << 16) | (luma(q[k].w) << 24);
    reinterpret_cast<uint4*>(gray)[v] = make_uint4(w[0], w[1], w[2], w[3]);
  }
  for (size_t i = nvec * 16 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x)
    gray[i] = (uint8_t)luma(__ldg(rgba + i));
}

void launch_gray(const uint8_t* rgba, size_t npix, uint8_t* gray, int grid, cudaStream_t st) {
  const int vec_ok = (((uintptr_t)rgba) % 16 == 0) && (((uintptr_t)gray) % 16 == 0);
  gray_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const uint32_t*>(rgba), npix, gray, vec_ok);
}

// ---- ImgToNRGBA for *image.YCbCr (core/image.go:60-76): section 8f row N3 ---------------------------------------------------
// The reference calls color.YCbCrToRGB (Go standard library, image/color/ycbcr.go, go1.22 per go.mod:3 -- not under the
// reference tree), restated here: JFIF conversion in 16.16 fixed point,
//   yy1 = y * 0x10101;  r = yy1 + 91881*cr1;  g = yy1 - 22554*cb1 - 46802*cr1;  b = yy1 + 116130*cb1   (cb1 = cb-128, cr1 = cr-128)
// each then clamped: a value whose bits 24..31 are all zero is shifted right by 16, anything else saturates to 0 (negative)
// or 255.  The constants are the ones the reference's own test restates (core/image_test.go:118-138, which rounds instead
// and therefore allows +-1); alpha is 0xff.  Chroma sample of pixel (x, y): image.YCbCr.COffset for the six subsample ratios,
// relative to the rectangle origin (min_x, min_y) like image.go:66-67.
// `gray` (optional) fuses RgbToGrayscale (core/grayscale.go:8-23) of the converted pixel, so the NRGBA image never has to
// make the round trip through HBM when only the detector's input is wanted.
__device__ __forceinline__ uint32_t sat16(int v) { return (uint32_t)v & 0xff000000u ? (uint32_t)(~(v >> 31)) & 0xffu : (uint32_t)(v >> 16); }

// color.YCbCrToRGB of one sample, as an NRGBA pixel with alpha 0xff.
__device__ __forceinline__ uint32_t ycbcr_px(int y, int cb, int cr) {
  const int yy1 = y * 0x10101, cb1 = cb - 128, cr1 = cr - 128;
  const uint32_t r = sat16(yy1 + 91881 * cr1), gg = sat16(yy1 - 22554 * cb1 - 46802 * cr1), b = sat16(yy1 + 116130 * cb1);
  return r | (b << 16) | (gg << 8) | 0xff000000u;   // (this operand order keeps ycbcr_kernel's SASS as it was before the factoring)
}

// image.YCbCr.COffset relative to the rectangle origin (min_x, min_y >= 0), split into its row and column parts.
__device__ __forceinline__ size_t coffset_row(int sy, int min_y, int ys, int c_stride) { return (size_t)((sy >> ys) - (min_y >> ys)) * c_stride; }
__device__ __forceinline__ size_t coffset_col(int sx, int min_x, int xs) { return (size_t)((sx >> xs) - (min_x >> xs)); }

// One thread converts 4 consecutive pixels of a row (32-bit index arithmetic, one 16-byte store for the NRGBA output).
__global__ void __launch_bounds__(256) ycbcr_kernel(const uint8_t* __restrict__ yp, const uint8_t* __restrict__ cbp, const uint8_t* __restrict__ crp,
                                                    int y_stride, int c_stride, int sub, int min_x, int min_y, int width, int height,
                                                    uint32_t* __restrict__ nrgba, uint8_t* __restrict__ gray, int vec_ok) {
  const int xs = chroma_xshift(sub), ys = chroma_yshift(sub);
  const unsigned chunks = (unsigned)(width + 3) >> 2;
  const unsigned total = chunks * (unsigned)height;                                // < 2^31: width * height < 2^31 is checked by the host
  for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < total; q += gridDim.x * blockDim.x) {
    const int dy = (int)(q / chunks), dx0 = (int)(q - (unsigned)dy * chunks) * 4;
    const int sy = min_y + dy;                                                     // image.go:66-67
    const uint8_t* yrow = yp + (size_t)dy * y_stride;                             // YOffset: (y-Rect.Min.Y)*YStride + (x-Rect.Min.X)
    const size_t crow = coffset_row(sy, min_y, ys, c_stride);
    uint32_t px[4], lum = 0;
    const int n = min(4, width - dx0);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      px[k] = 0;
      if (k < n) {
        const int dx = dx0 + k;
        const size_t sic = crow + coffset_col(min_x + dx, min_x, xs);
        px[k] = ycbcr_px(__ldg(yrow + dx), __ldg(cbp + sic), __ldg(crp + sic));
        if (gray) lum |= luma(px[k]) << (8 * k);
      }
    }
    const size_t o = (size_t)dy * width + dx0;
    if (nrgba) {
      if (vec_ok && n == 4) *reinterpret_cast<uint4*>(nrgba + o) = make_uint4(px[0], px[1], px[2], px[3]);
      else for (int k = 0; k < n; ++k) nrgba[o + k] = px[k];
    }
    if (gray) {
      if (vec_ok && n == 4) *reinterpret_cast<uint32_t*>(gray + o) = lum;
      else for (int k = 0; k < n; ++k) gray[o + k] = (uint8_t)(lum >> (8 * k));
    }
  }
}

void launch_ycbcr(const uint8_t* y, const uint8_t* cb, const uint8_t* cr, int y_stride, int c_stride, int subsample, int min_x, int min_y,
                  int width, int height, uint8_t* nrgba, uint8_t* gray, int grid, cudaStream_t st) {
  const size_t want = ((size_t)((width + 3) / 4) * height + 255) / 256;
  // vector stores need width % 4 == 0 (every row chunk starts at a multiple of 4 pixels) and aligned outputs
  const int vec_ok = (width % 4 == 0) && (((uintptr_t)nrgba) % 16 == 0) && (((uintptr_t)gray) % 4 == 0);
  ycbcr_kernel<<<(int)std::max<size_t>(1, std::min<size_t>(want, (size_t)grid)), 256, 0, st>>>(y, cb, cr, y_stride, c_stride, subsample, min_x, min_y, width,
                                                                                             height, reinterpret_cast<uint32_t*>(nrgba), gray, vec_ok);
}


// ---- RgbToGrayscale(ImgToNRGBA(img)) for a batch of decoded images (pigo_gray_images) ---------------------------------------
// ImgToNRGBA (core/image.go:35-90) then RgbToGrayscale (core/grayscale.go:8-23) per pixel, without the NRGBA image:
//   *image.YCbCr  luma(YCbCrToRGB(Y, Cb, Cr)), the `gray` output of ycbcr_kernel;
//   *image.NRGBA  luma of the pixel (the reference copies the rows);
//   *image.RGBA   luma(color.NRGBAModel(pixel)) -- rgba_to_nrgba below;
//   *image.Gray   luma(Y, Y, Y, 0xff) == Y for every Y (pinned by a CPU test), so the rows are copied;
//   *image.Gray16, RGBA64, NRGBA64, CMYK, Paletted   luma(color.NRGBAModel(pixel)) -- wide_chunk below.
// color.nrgbaModel (image/color/color.go) of a color.RGBA pixel: its RGBA() channels c*0x101 (alpha-premultiplied) back to
// straight 8-bit channels.  uint32 arithmetic as Go's: a == 0xffff -> c >> 8; a == 0 -> all zero; else (c*0xffff)/a >> 8,
// truncated to uint8 (a channel above alpha -- invalid premultiplied input -- wraps like the reference's conversion).
__device__ __forceinline__ uint32_t rgba_to_nrgba(uint32_t px) {
  const uint32_t a = (px >> 24) * 0x101u;
  if (a == 0xffffu) return px;
  if (a == 0) return 0;
  uint32_t out = px & 0xff000000u;                        // uint8(a >> 8)
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const uint32_t v = ((px >> (8 * c)) & 0xffu) * 0x101u;
    out |= (((v * 0xffffu) / a >> 8) & 0xffu) << (8 * c);   // v * 0xffff <= 0xfffe0001: no overflow
  }
  return out;
}

// color.nrgbaModel of the 16-bit alpha-premultiplied channels a Color.RGBA() returns, as an NRGBA pixel (uint32 like Go;
// c * 0xffff <= 0xfffe0001 cannot overflow, and a channel above alpha wraps through the uint8 conversion).
__device__ __forceinline__ uint32_t nrgba_model(uint32_t r, uint32_t g, uint32_t b, uint32_t a) {
  if (a == 0xffffu) return (r >> 8) | ((g >> 8) << 8) | ((b >> 8) << 16) | 0xff000000u;
  if (a == 0) return 0;
  return (((r * 0xffffu) / a >> 8) & 0xffu) | ((((g * 0xffffu) / a >> 8) & 0xffu) << 8) | ((((b * 0xffffu) / a >> 8) & 0xffu) << 16) |
         ((a >> 8) << 24);
}

// One *image.RGBA64 / *image.NRGBA64 pixel, R G B A as big-endian uint16: `rg` and `ba` are its two 4-byte halves as
// loaded (little-endian words).  NRGBA64.RGBA() premultiplies first (c*a/0xffff); the precision that loses is kept.
__device__ __forceinline__ uint32_t px64_to_nrgba(uint32_t rg, uint32_t ba, bool premul) {
  uint32_t r = __byte_perm(rg, 0, 0x4401), g = __byte_perm(rg, 0, 0x4423), b = __byte_perm(ba, 0, 0x4401);
  const uint32_t a = __byte_perm(ba, 0, 0x4423);
  if (!premul) { r = r * a / 0xffffu; g = g * a / 0xffffu; b = b * a / 0xffffu; }
  return nrgba_model(r, g, b, a);
}

// color.CMYK.RGBA() of one pixel (bytes C, M, Y, K), opaque, then nrgbaModel's a == 0xffff case.
__device__ __forceinline__ uint32_t cmyk_to_nrgba(uint32_t px) {
  const uint32_t w = 0xffffu - (px >> 24) * 0x101u;
  const uint32_t r = (0xffffu - (px & 0xffu) * 0x101u) * w / 0xffffu;
  const uint32_t g = (0xffffu - ((px >> 8) & 0xffu) * 0x101u) * w / 0xffffu;
  const uint32_t b = (0xffffu - ((px >> 16) & 0xffu) * 0x101u) * w / 0xffffu;
  return (r >> 8) | ((g >> 8) << 8) | ((b >> 8) << 16) | 0xff000000u;
}

// Pixel k of a 16-pixel chunk of 4-byte pixels: one of four 16-byte loads when the chunk is aligned and full, else bytes.
__device__ __forceinline__ uint32_t px32(const uint4* q, const uint8_t* p, bool vec, int k) {
  if (vec) { const uint4 v = q[k >> 2]; return (k & 3) == 0 ? v.x : (k & 3) == 1 ? v.y : (k & 3) == 2 ? v.z : v.w; }
  return (uint32_t)__ldg(p + 4 * k) | ((uint32_t)__ldg(p + 4 * k + 1) << 8) | ((uint32_t)__ldg(p + 4 * k + 2) << 16) | ((uint32_t)__ldg(p + 4 * k + 3) << 24);
}

// Palette entry i (an NRGBA pixel) of a Paletted source; a device palette need not be 4-byte aligned.
__device__ __forceinline__ uint32_t palette_px(const uint8_t* pal, uint32_t i) {
  return ((uintptr_t)pal & 3) == 0 ? __ldg(reinterpret_cast<const uint32_t*>(pal) + i) : px32(nullptr, pal + 4 * i, false, 0);
}

// The 16 gray bytes w[] of one chunk of a Gray16, RGBA64, NRGBA64, CMYK or Paletted source: p = the chunk's first pixel,
// n <= 16 pixels, vec = full and 16-byte aligned (2, 8, 4 and 1 16-byte loads; the 64-bit formats in two halves of four).
__device__ __forceinline__ void wide_chunk(const GraySrc& s, const uint8_t* p, int n, bool vec, uint32_t w[4]) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  if (s.format == PIGO_DECODED_GRAY16) {   // luma(Y>>8, Y>>8, Y>>8, 0xff) == Y>>8: the high (first) byte of each sample
    if (vec) {
      const uint4 a = __ldg(q), b = __ldg(q + 1);
      w[0] = __byte_perm(a.x, a.y, 0x6420); w[1] = __byte_perm(a.z, a.w, 0x6420);
      w[2] = __byte_perm(b.x, b.y, 0x6420); w[3] = __byte_perm(b.z, b.w, 0x6420);
    } else {
#pragma unroll
      for (int k = 0; k < 16; ++k)
        if (k < n) w[k >> 2] |= (uint32_t)__ldg(p + 2 * k) << (8 * (k & 3));
    }
  } else if (s.format == PIGO_DECODED_PALETTED) {
    const uint32_t len = (uint32_t)s.stride1;
    uint4 iv = make_uint4(0, 0, 0, 0);
    if (vec) iv = __ldg(q);
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      if (k < n) {
        const uint32_t iw = (k >> 2) == 0 ? iv.x : (k >> 2) == 1 ? iv.y : (k >> 2) == 2 ? iv.z : iv.w;
        const uint32_t i = vec ? (iw >> (8 * (k & 3))) & 0xffu : (uint32_t)__ldg(p + k);
        if (i < len) w[k >> 2] |= luma(palette_px(s.plane[1], i)) << (8 * (k & 3));   // past the palette: gray 0
      }
    }
  } else if (s.format == PIGO_DECODED_CMYK) {
    uint4 v[4];
    if (vec) {
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = __ldg(q + k);
    }
#pragma unroll
    for (int k = 0; k < 16; ++k)
      if (k < n) w[k >> 2] |= luma(cmyk_to_nrgba(px32(v, p, vec, k))) << (8 * (k & 3));
  } else {
    const bool premul = s.format == PIGO_DECODED_RGBA64;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint4 v[4];
      if (vec) {
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = __ldg(q + 4 * h + k);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = 8 * h + j;
        if (k < n) {
          // pixel j of the half is words 2j and 2j+1 of its four loads
          const uint32_t rg = px32(v, p + 64 * h, vec, 2 * j), ba = px32(v, p + 64 * h, vec, 2 * j + 1);
          w[k >> 2] |= luma(px64_to_nrgba(rg, ba, premul)) << (8 * (k & 3));
        }
      }
    }
  }
}

// One thread per (source, row, 16-pixel chunk) work item over every distinct source of the call; the source is found by a
// binary search over the sources' first work items.  16-byte stores where the slot row is aligned, bytes otherwise.
// Wide = the Gray16, RGBA64, NRGBA64, CMYK and Paletted sources: their conversions need about 90 registers where the
// YCbCr, NRGBA, RGBA and Gray ones need 57, so they run in an instantiation of their own over their own work range.
template <bool Wide>
__global__ void __launch_bounds__(256) gray_images_kernel(const GraySrc* __restrict__ src, const uint64_t* __restrict__ first, int nsrc, uint64_t total) {
  for (uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (uint64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = nsrc - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(first + mid) <= q) lo = mid; else hi = mid - 1;
    }
    const GraySrc& s = src[lo];
    const int width = s.width, format = s.format;
    const unsigned chunks = (unsigned)(width + 15) >> 4;
    const unsigned local = (unsigned)(q - __ldg(first + lo));   // < width * height < 2^31
    const int row = (int)(local / chunks), x0 = (int)(local - (unsigned)row * chunks) * 16;
    const int n = min(16, width - x0);
    const uint8_t* p = s.plane[0] + (size_t)row * s.stride0 + (size_t)x0 * (Wide ? decoded_bpp(format) : format == PIGO_DECODED_NRGBA || format == PIGO_DECODED_RGBA ? 4 : 1);
    const bool vec = n == 16 && ((uintptr_t)p & 15) == 0;
    uint32_t w[4] = {0, 0, 0, 0};
    if (Wide) {
      wide_chunk(s, p, n, vec, w);
    } else if (format == PIGO_DECODED_GRAY) {
      if (vec) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
        w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
      } else {
#pragma unroll
        for (int k = 0; k < 16; ++k)
          if (k < n) w[k >> 2] |= (uint32_t)__ldg(p + k) << (8 * (k & 3));
      }
    } else if (format == PIGO_DECODED_YCBCR) {
      const int xs = chroma_xshift(s.sub), ys = chroma_yshift(s.sub);
      const size_t crow = coffset_row(s.min_y + row, s.min_y, ys, s.stride1);
      uint4 yv = make_uint4(0, 0, 0, 0);
      if (vec) yv = __ldg(reinterpret_cast<const uint4*>(p));
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        if (k < n) {
          const uint32_t yw = (k >> 2) == 0 ? yv.x : (k >> 2) == 1 ? yv.y : (k >> 2) == 2 ? yv.z : yv.w;
          const uint32_t y = vec ? (yw >> (8 * (k & 3))) & 0xffu : (uint32_t)__ldg(p + k);
          const size_t sic = crow + coffset_col(s.min_x + x0 + k, s.min_x, xs);
          w[k >> 2] |= luma(ycbcr_px(y, __ldg(s.plane[1] + sic), __ldg(s.plane[2] + sic))) << (8 * (k & 3));
        }
      }
    } else {
      const bool premul = format == PIGO_DECODED_RGBA;
      uint4 v[4];
      if (vec) {
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = __ldg(reinterpret_cast<const uint4*>(p) + k);
      }
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        if (k < n) {
          const uint32_t px = px32(v, p, vec, k);
          w[k >> 2] |= luma(premul ? rgba_to_nrgba(px) : px) << (8 * (k & 3));
        }
      }
    }
    uint8_t* d = s.dst + (size_t)row * width + x0;
    if (n == 16 && ((uintptr_t)d & 15) == 0) *reinterpret_cast<uint4*>(d) = make_uint4(w[0], w[1], w[2], w[3]);
    else {
#pragma unroll
      for (int k = 0; k < 16; ++k)
        if (k < n) d[k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
    }
  }
}

void launch_gray_images(const GraySrc* src, const uint64_t* first, int nsrc, uint64_t total, bool wide, int grid, cudaStream_t st) {
  const uint64_t want = (total + 255) / 256;
  const int blocks = (int)std::max<uint64_t>(1, std::min<uint64_t>(want, (uint64_t)grid));
  if (wide) gray_images_kernel<true><<<blocks, 256, 0, st>>>(src, first, nsrc, total);
  else gray_images_kernel<false><<<blocks, 256, 0, st>>>(src, first, nsrc, total);
}

}  // namespace pigo
