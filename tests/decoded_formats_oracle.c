/* decoded_formats_oracle.c -- CPU restatements of the conversions of the decoded
 * image types pigo_gray_images takes beyond YCbCr, NRGBA, RGBA and Gray; test
 * infrastructure only, built by tests/decoded_formats_oracle.py into a temporary
 * directory.
 *
 * The other types the reference's image/jpeg and image/png decoders return go
 * through core/image.go:77-88 ImgToNRGBA's default case:
 * color.NRGBAModel.Convert(img.At(x, y)) with At's color type's RGBA()
 * (image/color/color.go, go1.22, Go standard library, not under the reference
 * tree), restated, in uint32:
 *   Gray16   y, y, y, 0xffff
 *   RGBA64   r, g, b, a as stored (alpha-premultiplied)
 *   NRGBA64  c*a/0xffff for each colour channel c, a
 *   CMYK     w = 0xffff - k*0x101; (0xffff - c*0x101)*w/0xffff for (c, m, y); 0xffff
 * then nrgbaModel on the 16-bit channels:
 *   a == 0xffff -> uint8(c >> 8); a == 0 -> NRGBA{0, 0, 0, 0};
 *   otherwise uint8(((c * 0xffff) / a) >> 8), alpha uint8(a >> 8)
 * (a channel above alpha overflows the 8 bits and is truncated, as in Go).
 * 16-bit samples are big-endian in Pix.  Paletted needs no model here: its pixel
 * is the palette entry. */
#include <stdint.h>

static void nrgba_model16(uint32_t r, uint32_t g, uint32_t b, uint32_t a, uint8_t *d) {
  const uint32_t c[3] = {r, g, b};
  for (int k = 0; k < 3; k++) {
    if (a == 0xffffu) d[k] = (uint8_t)(c[k] >> 8);
    else if (a == 0) d[k] = 0;
    else d[k] = (uint8_t)(((c[k] * 0xffffu) / a) >> 8);
  }
  d[3] = (uint8_t)(a >> 8);
}

static uint32_t be16(const uint8_t *p) { return ((uint32_t)p[0] << 8) | p[1]; }

void oracle_gray16_to_nrgba(const uint8_t *pix, int64_t npix, uint8_t *nrgba) {
  for (int64_t i = 0; i < npix; i++) {
    const uint32_t y = be16(pix + 2 * i);
    nrgba_model16(y, y, y, 0xffffu, nrgba + 4 * i);
  }
}

/* premultiplied != 0: *image.RGBA64, else *image.NRGBA64 */
void oracle_rgba64_to_nrgba(const uint8_t *pix, int64_t npix, int premultiplied, uint8_t *nrgba) {
  for (int64_t i = 0; i < npix; i++) {
    const uint8_t *s = pix + 8 * i;
    uint32_t r = be16(s), g = be16(s + 2), b = be16(s + 4);
    const uint32_t a = be16(s + 6);
    if (!premultiplied) {
      r = r * a / 0xffffu;
      g = g * a / 0xffffu;
      b = b * a / 0xffffu;
    }
    nrgba_model16(r, g, b, a, nrgba + 4 * i);
  }
}

void oracle_cmyk_to_nrgba(const uint8_t *pix, int64_t npix, uint8_t *nrgba) {
  for (int64_t i = 0; i < npix; i++) {
    const uint8_t *s = pix + 4 * i;
    const uint32_t w = 0xffffu - (uint32_t)s[3] * 0x101u;
    const uint32_t r = (0xffffu - (uint32_t)s[0] * 0x101u) * w / 0xffffu;
    const uint32_t g = (0xffffu - (uint32_t)s[1] * 0x101u) * w / 0xffffu;
    const uint32_t b = (0xffffu - (uint32_t)s[2] * 0x101u) * w / 0xffffu;
    nrgba_model16(r, g, b, 0xffffu, nrgba + 4 * i);
  }
}
