/* blur_oracle.c -- CPU restatement of pigo_blur_faces (include/pigo_b200.h) for one decoded image; test infrastructure only,
 * built by decoded_oracle.compile_c into a temporary directory.  Plain loops: Rmax per luma pixel, face by face over the
 * disc's bounding box; then, per plane and channel, a 64-bit summed-area table of the plane padded by edge replication as
 * far as the largest box reaches, and each covered sample's box sum from it.  Channels are separate bytes and the table of a
 * channel is complete before any sample of it is written, so every mean is over the input as it was before the call. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

typedef struct {
  int32_t row, col, scale;
  float q;
} oracle_det;

static long long clampll(long long v, long long lo, long long hi) { return v < lo ? lo : v > hi ? hi : v; }

/* map[y*w + x] = Rmax of luma pixel (y, x), -1 where no blurred face covers it. */
static void rmax_map(int w, int h, const oracle_det *f, int nf, double min_q, double disc_ratio, double radius_ratio, int radius, int32_t *map) {
  for (long long k = 0; k < (long long)w * h; k++) map[k] = -1;
  const long long lim = 1ll << 24;
  for (int k = 0; k < nf; k++) {
    const oracle_det d = f[k];
    if (!((double)d.q >= min_q)) continue;
    if (d.scale < 0 || d.scale > lim || llabs(d.row) > lim || llabs(d.col) > lim) continue;
    const long long r = (long long)((double)d.scale * disc_ratio);
    long long R = (long long)((double)d.scale * radius_ratio);
    if (R < radius) R = radius;
    if (R > 1023) R = 1023;
    const long long y0 = clampll(d.row - r, 0, h), y1 = clampll(d.row + r, -1, h - 1);
    const long long x0 = clampll(d.col - r, 0, w), x1 = clampll(d.col + r, -1, w - 1);
    for (long long y = y0; y <= y1; y++)
      for (long long x = x0; x <= x1; x++) {
        const long long dy = y - d.row, dx = x - d.col;
        if (dy * dy + dx * dx <= r * r && map[y * w + x] < R) map[y * w + x] = (int32_t)R;
      }
  }
}

/* Blurs one plane in place: rows x cols samples of chans bytes, `stride` bytes apart; the anchor of sample (j, i) is luma
 * ((my>>ys)+j << ys, (mx>>xs)+i << xs) clamped into the rectangle [mx, mx+w) x [my, my+h), made relative. */
static void blur_plane(uint8_t *p, int stride, int cols, int rows, int chans, const int32_t *map, int w, int h, int xs, int ys, int mx, int my) {
  int pad_y = -1, pad_x = -1;
  int32_t *rm = malloc(sizeof(int32_t) * (size_t)rows * cols);
  for (int j = 0; j < rows; j++)
    for (int i = 0; i < cols; i++) {
      const long long ay = clampll((long long)((my >> ys) + j) << ys, my, (long long)my + h - 1) - my;
      const long long ax = clampll((long long)((mx >> xs) + i) << xs, mx, (long long)mx + w - 1) - mx;
      const int32_t R = map[ay * w + ax];
      rm[(size_t)j * cols + i] = R;
      if (R >= 0) {
        if ((R >> ys) > pad_y) pad_y = R >> ys;
        if ((R >> xs) > pad_x) pad_x = R >> xs;
      }
    }
  if (pad_y < 0) { free(rm); return; }
  const long long PH = rows + 2ll * pad_y, PW = cols + 2ll * pad_x;
  int64_t *S = calloc((size_t)(PH + 1) * (PW + 1), sizeof(int64_t));
  for (int c = 0; c < chans; c++) {
    for (long long y = 0; y < PH; y++)
      for (long long x = 0; x < PW; x++) {
        const long long sy = clampll(y - pad_y, 0, rows - 1), sx = clampll(x - pad_x, 0, cols - 1);
        S[(y + 1) * (PW + 1) + x + 1] = p[sy * stride + sx * chans + c] + S[y * (PW + 1) + x + 1] + S[(y + 1) * (PW + 1) + x] - S[y * (PW + 1) + x];
      }
    for (int j = 0; j < rows; j++)
      for (int i = 0; i < cols; i++) {
        const int32_t R = rm[(size_t)j * cols + i];
        if (R < 0) continue;
        const long long ry = R >> ys, rx = R >> xs;
        const long long y0 = j - ry + pad_y, y1 = j + ry + pad_y + 1, x0 = i - rx + pad_x, x1 = i + rx + pad_x + 1;
        const int64_t sum = S[y1 * (PW + 1) + x1] - S[y0 * (PW + 1) + x1] - S[y1 * (PW + 1) + x0] + S[y0 * (PW + 1) + x0];
        const int64_t n = (2 * ry + 1) * (2 * rx + 1);
        p[(size_t)j * stride + (size_t)i * chans + c] = (uint8_t)((sum + n / 2) / n);
      }
  }
  free(S);
  free(rm);
}

/* pigo_blur_faces of one source (format 0 YCbCr, 1 NRGBA, 2 RGBA, 3 Gray, 8 CMYK) around faces[0..nf). */
void oracle_blur(int format, int sub, int min_x, int min_y, int width, int height, uint8_t *p0, uint8_t *p1, uint8_t *p2, int s0, int s1,
                 const oracle_det *faces, int nf, double min_q, double disc_ratio, double radius_ratio, int radius) {
  int32_t *map = malloc(sizeof(int32_t) * (size_t)width * height);
  rmax_map(width, height, faces, nf, min_q, disc_ratio, radius_ratio, radius, map);
  if (format == 0) {
    const int xd[6] = {0, 1, 1, 0, 2, 2}, yd[6] = {0, 0, 1, 1, 0, 1};
    const int xs = xd[sub], ys = yd[sub];
    const int ch = ((min_y + height - 1) >> ys) - (min_y >> ys) + 1, cw = ((min_x + width - 1) >> xs) - (min_x >> xs) + 1;
    blur_plane(p0, s0, width, height, 1, map, width, height, 0, 0, min_x, min_y);
    blur_plane(p1, s1, cw, ch, 1, map, width, height, xs, ys, min_x, min_y);
    blur_plane(p2, s1, cw, ch, 1, map, width, height, xs, ys, min_x, min_y);
  } else {
    blur_plane(p0, s0, width, height, format == 3 ? 1 : 4, map, width, height, 0, 0, 0, 0);
  }
  free(map);
}
