/* decoded_oracle.c -- CPU restatement of the one conversion of decoded images the
 * existing oracle (oracle/pigo_oracle.c) does not cover; test infrastructure only,
 * built by tests/decoded_oracle.py into a temporary directory.
 *
 * core/image.go:77-88 ImgToNRGBA, *image.RGBA via the default case:
 * color.NRGBAModel.Convert (image/color/color.go nrgbaModel, Go standard library,
 * not under the reference tree), restated: the RGBA() channels of a color.RGBA
 * pixel are c*0x101 (alpha-premultiplied, 16 bit); then
 *   a == 0xffff -> uint8(c >> 8); a == 0 -> NRGBA{0, 0, 0, 0};
 *   otherwise c = (c * 0xffff) / a, uint8(c >> 8), all in uint32, alpha uint8(a >> 8).
 * A channel above alpha (invalid premultiplied input) overflows the 8 bits and is
 * truncated by the uint8 conversion, as in Go. */
#include <stdint.h>

void oracle_rgba_to_nrgba(const uint8_t *rgba, int64_t npix, uint8_t *nrgba) {
  for (int64_t i = 0; i < npix; i++) {
    const uint8_t *s = rgba + 4 * i;
    uint8_t *d = nrgba + 4 * i;
    uint32_t a = (uint32_t)s[3] * 0x101u;
    for (int c = 0; c < 3; c++) {
      uint32_t v = (uint32_t)s[c] * 0x101u;
      if (a == 0xffffu) d[c] = (uint8_t)(v >> 8);
      else if (a == 0) d[c] = 0;
      else d[c] = (uint8_t)(((v * 0xffffu) / a) >> 8);
    }
    d[3] = a == 0 ? 0 : (uint8_t)(a >> 8);
  }
}
