/*
 * pigo_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C restatement of the arithmetic of esimov/pigo's detection path:
 *   core/pigo.go   :51-110  Unpack               -> oracle_face_create
 *   core/pigo.go   :113-147 classifyRegion       -> face_classify
 *   core/pigo.go   :150-191 classifyRotatedRegion-> face_classify_rotated
 *   core/pigo.go   :212-258 RunCascade           -> oracle_run_cascade
 *   core/pigo.go   :262-308 ClusterDetections    -> oracle_cluster
 *   core/puploc.go :38-103  UnpackCascade        -> oracle_puploc_create
 *   core/puploc.go :106-154 classifyRegion       -> puploc_classify
 *   core/puploc.go :157-217 classifyRotatedRegion-> puploc_classify_rotated
 *   core/puploc.go :239-277 RunDetector          -> oracle_puploc_run_detector
 *   core/flploc.go :36-57   GetLandmarkPoint     -> oracle_get_landmark_seed
 *   core/utils.go  :8-52    abs/min/max/round/pow
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may load this library, and only as the checker / CPU baseline.
 * The product (libpigo_b200.so) never links, loads or calls it.
 *
 * PARITY PINNING STATUS: "parity unpinned" for numeric values.  The reference
 * is Go; no Go toolchain exists in the build container or on the GPU box, and
 * the reference's own tests (core/pigo_test.go, puploc_test.go, flploc_test.go) hold no numeric golden vectors --
 * only existential assertions (>=1 clustered face on testdata/sample.jpg,
 * exactly one face with Scale>50, 15 landmark points with Row>0 && Col>0).
 * tests/test_oracle_pins.py checks this oracle against exactly those
 * assertions, and against an independently written numpy restatement
 * (oracle/np_oracle.py).  Two behaviours are unpinnable even in principle:
 *  - tie order of sort.Slice in ClusterDetections (Go std pdqsort, unstable):
 *    this oracle uses a STABLE sort by Q ascending (original index breaks ties);
 *  - where sort.Slice puts a NaN Q (its < is not an order then): this oracle
 *    sorts every NaN, of either sign, after +inf, equal to each other (so they
 *    keep their input order), and -0 equal to +0 -- np.argsort(kind="stable");
 *  - RunDetector's random stream (global auto-seeded math/rand) and stale
 *    sync.Pool contents: this oracle takes the randoms as an argument and
 *    starts from a fresh (zeroed) 63-slot pool.
 *
 * Go `int` is 64-bit on amd64: int64_t is used wherever the reference uses int.
 * Build with -ffp-contract=off: Go/amd64 does not fuse multiply-add.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <pthread.h>

typedef struct {
  int32_t row, col, scale;
  float q;
} oracle_det;

typedef struct {
  uint32_t depth;   /* treeDepth (levels) */
  uint32_t ntrees;  /* treeNum */
  int64_t leaves;   /* pow(2, depth) */
  int8_t *codes;    /* ntrees * 4*leaves bytes, 4 zero bytes prepended per tree */
  float *preds;     /* ntrees * leaves */
  float *thresh;    /* ntrees */
} oracle_face;

typedef struct {
  uint32_t stages, trees, depth;
  float scales;
  int64_t leaves;
  int8_t *codes;  /* stages*trees*(4*leaves-4) */
  float *preds;   /* stages*trees*leaves*2 */
} oracle_puploc;

/* ---- core/utils.go:8-52 ------------------------------------------------ */
static inline int64_t go_abs(int64_t x) { return x < 0 ? -x : x; }
static inline int64_t go_min(int64_t a, int64_t b) { return a < b ? a : b; }
static inline int64_t go_max(int64_t a, int64_t b) { return a > b ? a : b; }
/* utils.go:42-52: square-and-multiply in float64 */
static double go_pow(double base, int exp) {
  double result = 1.0;
  while (exp > 0) {
    if (exp % 2 == 1) result *= base;
    exp >>= 1;
    base *= base;
  }
  return result;
}
/* math.Round: half away from zero */
static inline double go_math_round(double x) { return round(x); }

static uint32_t rd_u32(const uint8_t *p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
static float rd_f32(const uint8_t *p) {
  uint32_t u = rd_u32(p);
  float f;
  memcpy(&f, &u, 4);
  return f;
}

/* ---- core/pigo.go:51-110 Unpack ---------------------------------------- */
/* Unlike the reference (which panics on short input) this returns -1. */
int oracle_face_create(const uint8_t *packet, size_t len, oracle_face **out) {
  if (len < 16) return -1;
  size_t pos = 8;                               /* pigo.go:61 skip 8 bytes */
  uint32_t depth = rd_u32(packet + pos); pos += 4;   /* :64 */
  uint32_t ntrees = rd_u32(packet + pos); pos += 4;  /* :68 */
  if (depth > 16) return -1;
  int64_t leaves = (int64_t)go_pow(2, (int)depth);
  size_t per_tree = (size_t)(4 * leaves - 4) + (size_t)leaves * 4 + 4;
  if (len < 16 + (size_t)ntrees * per_tree) return -1;
  oracle_face *f = (oracle_face *)calloc(1, sizeof(*f));
  f->depth = depth; f->ntrees = ntrees; f->leaves = leaves;
  f->codes = (int8_t *)calloc((size_t)ntrees * 4 * leaves + 4, 1);
  f->preds = (float *)calloc((size_t)ntrees * leaves + 1, sizeof(float));
  f->thresh = (float *)calloc((size_t)ntrees + 1, sizeof(float));
  for (uint32_t t = 0; t < ntrees; t++) {
    int8_t *dst = f->codes + (size_t)t * 4 * leaves;
    dst[0] = dst[1] = dst[2] = dst[3] = 0;              /* :79 */
    memcpy(dst + 4, packet + pos, (size_t)(4 * leaves - 4)); /* :81-84 */
    pos += (size_t)(4 * leaves - 4);
    for (int64_t i = 0; i < leaves; i++) {              /* :89-95 */
      f->preds[(size_t)t * leaves + i] = rd_f32(packet + pos);
      pos += 4;
    }
    f->thresh[t] = rd_f32(packet + pos);                /* :96-100 */
    pos += 4;
  }
  *out = f;
  return 0;
}
void oracle_face_destroy(oracle_face *f) {
  if (!f) return;
  free(f->codes); free(f->preds); free(f->thresh); free(f);
}
void oracle_face_info(const oracle_face *f, uint32_t *depth, uint32_t *ntrees) {
  *depth = f->depth; *ntrees = f->ntrees;
}
/* raw table access for tests that cross-check the device tables */
const int8_t *oracle_face_codes(const oracle_face *f) { return f->codes; }
const float *oracle_face_preds(const oracle_face *f) { return f->preds; }
const float *oracle_face_thresh(const oracle_face *f) { return f->thresh; }

/* ---- core/pigo.go:113-147 classifyRegion ------------------------------- */
/* ntrees_evaluated (optional) receives how many trees were walked. */
static float face_classify(const oracle_face *pg, int64_t r, int64_t c, int64_t s,
                           const uint8_t *pixels, int64_t dim, int *ntrees_evaluated) {
  int64_t root = 0;
  float out = 0.0f;
  const int64_t treeDepth = pg->leaves;  /* RunCascade passes pow(2, depth), :216 */
  r = r * 256;                           /* :119 */
  c = c * 256;                           /* :120 */
  if (ntrees_evaluated) *ntrees_evaluated = 0;
  if (pg->ntrees > 0) {
    for (int64_t i = 0; i < (int64_t)pg->ntrees; i++) {
      int64_t idx = 1;
      for (uint32_t j = 0; j < pg->depth; j++) {
        int64_t x1 = ((r + (int64_t)pg->codes[root + 4 * idx + 0] * s) >> 8) * dim +
                     ((c + (int64_t)pg->codes[root + 4 * idx + 1] * s) >> 8);   /* :126 */
        int64_t x2 = ((r + (int64_t)pg->codes[root + 4 * idx + 2] * s) >> 8) * dim +
                     ((c + (int64_t)pg->codes[root + 4 * idx + 3] * s) >> 8);   /* :127 */
        idx = 2 * idx + (pixels[x1] <= pixels[x2] ? 1 : 0);                     /* :129-135 */
      }
      out += pg->preds[treeDepth * i + idx - treeDepth];                        /* :137 */
      if (ntrees_evaluated) (*ntrees_evaluated)++;
      if (out <= pg->thresh[i]) return -1.0f;                                   /* :139-141 */
      root += 4 * treeDepth;                                                    /* :142 */
    }
    return out - pg->thresh[pg->ntrees - 1];                                    /* :144 */
  }
  return 0.0f;
}

static const int64_t qCosTable[33] = {256, 251, 236, 212, 181, 142, 97, 49, 0, -49, -97, -142, -181, -212, -236, -251, -256,
                                      -251, -236, -212, -181, -142, -97, -49, 0, 49, 97, 142, 181, 212, 236, 251, 256};
static const int64_t qSinTable[33] = {0, 49, 97, 142, 181, 212, 236, 251, 256, 251, 236, 212, 181, 142, 97, 49, 0,
                                      -49, -97, -142, -181, -212, -236, -251, -256, -251, -236, -212, -181, -142, -97, -49, 0};

/* ---- core/pigo.go:150-191 classifyRotatedRegion ------------------------- */
/* NB (:168,:171): the COLUMN clamp uses nrows-1, ncols is unused. Kept. */
static float face_classify_rotated(const oracle_face *pg, int64_t r, int64_t c, int64_t s, double a,
                                   int64_t nrows, int64_t ncols, const uint8_t *pixels, int64_t dim,
                                   int *ntrees_evaluated) {
  (void)ncols;
  int64_t root = 0;
  float out = 0.0f;
  const int64_t treeDepth = pg->leaves;
  int64_t qsin = s * qSinTable[(int)(32.0 * a)];   /* :159 */
  int64_t qcos = s * qCosTable[(int)(32.0 * a)];   /* :160 */
  if (ntrees_evaluated) *ntrees_evaluated = 0;
  if (pg->ntrees > 0) {
    for (int64_t i = 0; i < (int64_t)pg->ntrees; i++) {
      int64_t idx = 1;
      for (uint32_t j = 0; j < pg->depth; j++) {
        const int8_t *cd = pg->codes + root + 4 * idx;
        int64_t r1 = go_abs(go_min(nrows - 1, go_max(0, 65536 * r + qcos * (int64_t)cd[0] - qsin * (int64_t)cd[1]) >> 16));
        int64_t c1 = go_abs(go_min(nrows - 1, go_max(0, 65536 * c + qsin * (int64_t)cd[0] + qcos * (int64_t)cd[1]) >> 16));
        int64_t r2 = go_abs(go_min(nrows - 1, go_max(0, 65536 * r + qcos * (int64_t)cd[2] - qsin * (int64_t)cd[3]) >> 16));
        int64_t c2 = go_abs(go_min(nrows - 1, go_max(0, 65536 * c + qsin * (int64_t)cd[2] + qcos * (int64_t)cd[3]) >> 16));
        idx = 2 * idx + (pixels[r1 * dim + c1] <= pixels[r2 * dim + c2] ? 1 : 0);  /* :179 */
      }
      out += pg->preds[treeDepth * i + idx - treeDepth];
      if (ntrees_evaluated) (*ntrees_evaluated)++;
      if (out <= pg->thresh[i]) return -1.0f;
      root += 4 * treeDepth;
    }
    return out - pg->thresh[pg->ntrees - 1];
  }
  return 0.0f;
}

float oracle_classify_region(const oracle_face *pg, int r, int c, int s, const uint8_t *pixels, int dim) {
  return face_classify(pg, r, c, s, pixels, dim, NULL);
}
float oracle_classify_rotated_region(const oracle_face *pg, int r, int c, int s, double a, int nrows, int ncols,
                                     const uint8_t *pixels, int dim) {
  return face_classify_rotated(pg, r, c, s, a, nrows, ncols, pixels, dim, NULL);
}

/* ---- scale ladder helpers, core/pigo.go:226-231,:255 ------------------- */
/* Fills scales[] (up to cap) and returns the number of ladder entries;
 * returns -1 if the ladder would not terminate within 1<<20 steps. */
int oracle_scale_ladder(int min_size, int max_size, double scale_factor, int *scales, int cap) {
  int64_t scale = min_size;
  int n = 0;
  while (scale <= max_size) {
    if (n < cap && scales) scales[n] = (int)scale;
    n++;
    if (n > (1 << 20)) return -1;
    scale = (int64_t)((double)scale + fmax(2, ((double)scale * scale_factor) - (double)scale)); /* :255 */
  }
  return n;
}

int64_t oracle_count_windows(int rows, int cols, int min_size, int max_size, double shift, double scale_factor) {
  int64_t scale = min_size, total = 0;
  while (scale <= max_size) {
    int64_t step = (int64_t)fmax(shift * (double)scale, 1);  /* :227 */
    int64_t offset = scale / 2 + 1;                            /* :228 */
    int64_t nr = 0, nc = 0;
    if (rows - offset >= offset) nr = (rows - offset - offset) / step + 1;
    if (cols - offset >= offset) nc = (cols - offset - offset) / step + 1;
    total += nr * nc;
    scale = (int64_t)((double)scale + fmax(2, ((double)scale * scale_factor) - (double)scale));
  }
  return total;
}

/* ---- core/pigo.go:212-258 RunCascade ------------------------------------ */
/* Returns the number of detections found (may exceed cap; only the first cap
 * are stored).  tree_hist (optional, ntrees+1 entries) counts windows by the
 * number of trees they walked -- used by DESIGN.md's workload statistics. */
int64_t oracle_run_cascade(const oracle_face *pg, const uint8_t *pixels, int rows, int cols, int dim,
                           int min_size, int max_size, double shift_factor, double scale_factor, double angle,
                           oracle_det *out, int64_t cap, int64_t *tree_hist) {
  int64_t ndet = 0;
  int64_t scale = min_size;                                       /* :219 */
  while (scale <= max_size) {                                     /* :226 */
    int64_t step = (int64_t)fmax(shift_factor * (double)scale, 1);  /* :227 */
    int64_t offset = (scale / 2 + 1);                              /* :228 */
    for (int64_t row = offset; row <= rows - offset; row += step) {       /* :230 */
      for (int64_t col = offset; col <= cols - offset; col += step) {     /* :231 */
        float q;
        int nt = 0;
        if (angle > 0.0) {                                         /* :232 */
          if (angle > 1.0) angle = 1.0;                            /* :233-235 */
          q = face_classify_rotated(pg, row, col, scale, angle, rows, cols, pixels, dim, tree_hist ? &nt : NULL);
        } else {
          q = face_classify(pg, row, col, scale, pixels, dim, tree_hist ? &nt : NULL);
        }
        if (tree_hist) tree_hist[nt]++;
        if (q > 0.0f) {                                            /* :246 */
          if (ndet < cap && out) {
            out[ndet].row = (int32_t)row; out[ndet].col = (int32_t)col;
            out[ndet].scale = (int32_t)scale; out[ndet].q = q;
          }
          ndet++;
        }
      }
    }
    scale = (int64_t)((double)scale + fmax(2, ((double)scale * scale_factor) - (double)scale)); /* :255 */
  }
  return ndet;
}

/* Frame-parallel batch driver used only as the CPU baseline in bench.py
 * (one frame per task, pthreads; the reference itself is single-goroutine, so
 * nthreads=1 is "the reference as shipped"; nthreads=N models N goroutines
 * each running RunCascade on its own frame). */
typedef struct {
  const oracle_face *pg; const uint8_t *frames; int nframes; size_t frame_stride;
  int rows, cols, dim, min_size, max_size; double shift_factor, scale_factor, angle;
  oracle_det *out; int64_t cap_per_frame; int64_t *n_out;
  int next; int64_t total; pthread_mutex_t mu;
} batch_job;

static void *batch_worker(void *arg) {
  batch_job *jb = (batch_job *)arg;
  for (;;) {
    pthread_mutex_lock(&jb->mu);
    int f = jb->next++;
    pthread_mutex_unlock(&jb->mu);
    if (f >= jb->nframes) break;
    int64_t n = oracle_run_cascade(jb->pg, jb->frames + (size_t)f * jb->frame_stride, jb->rows, jb->cols, jb->dim,
                                   jb->min_size, jb->max_size, jb->shift_factor, jb->scale_factor, jb->angle,
                                   jb->out ? jb->out + (size_t)f * jb->cap_per_frame : NULL, jb->cap_per_frame, NULL);
    if (jb->n_out) jb->n_out[f] = n;
    pthread_mutex_lock(&jb->mu);
    jb->total += n;
    pthread_mutex_unlock(&jb->mu);
  }
  return NULL;
}

int64_t oracle_run_cascade_batch(const oracle_face *pg, const uint8_t *frames, int nframes, size_t frame_stride,
                                 int rows, int cols, int dim, int min_size, int max_size, double shift_factor,
                                 double scale_factor, double angle, oracle_det *out, int64_t cap_per_frame,
                                 int64_t *n_out, int nthreads) {
  batch_job jb = {pg, frames, nframes, frame_stride, rows, cols, dim, min_size, max_size, shift_factor, scale_factor,
                  angle, out, cap_per_frame, n_out, 0, 0, PTHREAD_MUTEX_INITIALIZER};
  if (nthreads < 1) nthreads = 1;
  if (nthreads > 256) nthreads = 256;
  pthread_t th[256];
  for (int t = 1; t < nthreads; t++) pthread_create(&th[t], NULL, batch_worker, &jb);
  batch_worker(&jb);
  for (int t = 1; t < nthreads; t++) pthread_join(th[t], NULL);
  return jb.total;
}

/* ---- core/pigo.go:262-308 ClusterDetections ----------------------------- */
static double calc_iou(const oracle_det *d1, const oracle_det *d2) {  /* :268-278 */
  double r1 = (double)d1->row, c1 = (double)d1->col, s1 = (double)d1->scale;
  double r2 = (double)d2->row, c2 = (double)d2->col, s2 = (double)d2->scale;
  double overRow = fmax(0, fmin(r1 + s1 / 2, r2 + s2 / 2) - fmax(r1 - s1 / 2, r2 - s2 / 2));
  double overCol = fmax(0, fmin(c1 + s1 / 2, c2 + s2 / 2) - fmax(c1 - s1 / 2, c2 - s2 / 2));
  return overRow * overCol / (s1 * s1 + s2 * s2 - overRow * overCol);
}

/* Q as an unsigned key of the sort's order: ascending, -0 == +0, every NaN one above +inf. */
static uint32_t q_order_key(float q) {
  uint32_t b;
  if (isnan(q)) return UINT32_MAX;
  if (q == 0.0f) b = 0;
  else memcpy(&b, &q, sizeof b);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

/* Sorts dets IN PLACE (as the reference does, :264) -- stable, by q_order_key
 * ascending -- then greedy clustering.  Returns the number of clusters (may exceed cap). */
int64_t oracle_cluster(oracle_det *dets, int64_t n, double iou_threshold, oracle_det *out, int64_t cap) {
  /* stable bottom-up merge sort by q_order_key */
  if (n > 1) {
    oracle_det *tmp = (oracle_det *)malloc((size_t)n * sizeof(oracle_det));
    for (int64_t width = 1; width < n; width *= 2) {
      for (int64_t lo = 0; lo < n; lo += 2 * width) {
        int64_t mid = lo + width < n ? lo + width : n;
        int64_t hi = lo + 2 * width < n ? lo + 2 * width : n;
        int64_t i = lo, j = mid, k = lo;
        while (i < mid && j < hi) {
          if (q_order_key(dets[j].q) < q_order_key(dets[i].q)) tmp[k++] = dets[j++];
          else tmp[k++] = dets[i++];
        }
        while (i < mid) tmp[k++] = dets[i++];
        while (j < hi) tmp[k++] = dets[j++];
      }
      memcpy(dets, tmp, (size_t)n * sizeof(oracle_det));
    }
    free(tmp);
  }
  uint8_t *assignments = (uint8_t *)calloc((size_t)(n > 0 ? n : 1), 1);
  int64_t nclusters = 0;
  for (int64_t i = 0; i < n; i++) {
    if (!assignments[i]) {                                  /* :285 */
      int64_t r = 0, c = 0, s = 0, cnt = 0;
      float q = 0.0f;
      for (int64_t j = 0; j < n; j++) {
        if (calc_iou(&dets[i], &dets[j]) > iou_threshold) {  /* :293 */
          assignments[j] = 1;
          r += dets[j].row; c += dets[j].col; s += dets[j].scale;
          q += dets[j].q;
          cnt++;
        }
      }
      if (cnt > 0) {                                        /* :302 */
        if (nclusters < cap && out) {
          out[nclusters].row = (int32_t)(r / cnt);
          out[nclusters].col = (int32_t)(c / cnt);
          out[nclusters].scale = (int32_t)(s / cnt);
          out[nclusters].q = q;
        }
        nclusters++;
      }
    }
  }
  free(assignments);
  return nclusters;
}

/* ---- core/puploc.go:38-103 UnpackCascade -------------------------------- */
int oracle_puploc_create(const uint8_t *packet, size_t len, oracle_puploc **out) {
  if (len < 16) return -1;
  size_t pos = 0;
  uint32_t stages = rd_u32(packet + pos); pos += 4;   /* :51 */
  float scales = rd_f32(packet + pos); pos += 4;      /* :55-57 */
  uint32_t trees = rd_u32(packet + pos); pos += 4;    /* :61 */
  uint32_t depth = rd_u32(packet + pos); pos += 4;    /* :65 */
  if (depth > 16 || stages > 4096 || trees > 65536) return -1;
  int64_t leaves = (int64_t)go_pow(2, (int)depth);
  size_t ncode = (size_t)(4 * leaves - 4), npred = (size_t)leaves * 2;
  if (len < 16 + (size_t)stages * trees * (ncode + npred * 4)) return -1;
  oracle_puploc *p = (oracle_puploc *)calloc(1, sizeof(*p));
  p->stages = stages; p->trees = trees; p->depth = depth; p->scales = scales; p->leaves = leaves;
  p->codes = (int8_t *)calloc((size_t)stages * trees * ncode + 4, 1);
  p->preds = (float *)calloc((size_t)stages * trees * npred + 2, sizeof(float));
  size_t ci = 0, pi = 0;
  for (uint32_t s = 0; s < stages; s++) {
    for (uint32_t t = 0; t < trees; t++) {
      memcpy(p->codes + ci, packet + pos, ncode);   /* :75-78 */
      ci += ncode; pos += ncode;
      for (size_t i = 0; i < npred; i++) {          /* :83-91 */
        p->preds[pi++] = rd_f32(packet + pos);
        pos += 4;
      }
    }
  }
  *out = p;
  return 0;
}
void oracle_puploc_destroy(oracle_puploc *p) {
  if (!p) return;
  free(p->codes); free(p->preds); free(p);
}
void oracle_puploc_info(const oracle_puploc *p, uint32_t *stages, float *scales, uint32_t *trees, uint32_t *depth) {
  *stages = p->stages; *scales = p->scales; *trees = p->trees; *depth = p->depth;
}

/* int8 negation wraps (-(-128) == -128 in Go's int8): puploc.go:124-125 */
static inline int64_t neg_i8(int8_t v) { return (int64_t)(int8_t)(uint8_t)(0u - (uint8_t)v); }

/* Go's int(r) on amd64 (CVTTSS2SQ): truncation, and the int64 minimum for NaN and out-of-range values.  The products
 * 256*int(r) and 65536*int(r) below wrap like Go's int64 arithmetic, so that minimum samples like int(r) == 0. */
static inline int64_t go_int_f32(float v) {
  if (!(v > -9223372036854775808.0f && v < 9223372036854775808.0f)) return INT64_MIN;
  return (int64_t)v;
}
static inline int64_t go_mul_add(int64_t k, int64_t a, int64_t b) { return (int64_t)((uint64_t)k * (uint64_t)a + (uint64_t)b); }

/* ---- core/puploc.go:106-154 classifyRegion ------------------------------ */
static void puploc_classify(const oracle_puploc *plc, float r, float c, float s, int64_t nrows, int64_t ncols,
                            const uint8_t *pixels, int64_t dim, int flipV, float res[3]) {
  int64_t root = 0;
  const int64_t treeDepth = plc->leaves;  /* RunDetector passes pow(2, depth), :245 */
  for (int64_t i = 0; i < (int64_t)plc->stages; i++) {
    float dr = 0.0f, dc = 0.0f;
    for (int64_t j = 0; j < (int64_t)plc->trees; j++) {
      int64_t idx = 0;
      for (uint32_t k = 0; k < plc->depth; k++) {
        const int8_t *cd = plc->codes + root + 4 * idx;
        int64_t rs = (int64_t)go_math_round((double)s);
        int64_t r1 = go_min(nrows - 1, go_max(0, go_mul_add(256, go_int_f32(r), (int64_t)cd[0] * rs) >> 8));  /* :118 */
        int64_t r2 = go_min(nrows - 1, go_max(0, go_mul_add(256, go_int_f32(r), (int64_t)cd[2] * rs) >> 8));  /* :119 */
        int64_t c1, c2;
        if (flipV) {                                                                                 /* :123-129 */
          c1 = go_min(ncols - 1, go_max(0, go_mul_add(256, go_int_f32(c), neg_i8(cd[1]) * rs) >> 8));
          c2 = go_min(ncols - 1, go_max(0, go_mul_add(256, go_int_f32(c), neg_i8(cd[3]) * rs) >> 8));
        } else {
          c1 = go_min(ncols - 1, go_max(0, go_mul_add(256, go_int_f32(c), (int64_t)cd[1] * rs) >> 8));
          c2 = go_min(ncols - 1, go_max(0, go_mul_add(256, go_int_f32(c), (int64_t)cd[3] * rs) >> 8));
        }
        idx = 2 * idx + 1 + (pixels[r1 * dim + c1] > pixels[r2 * dim + c2] ? 1 : 0);                /* :130-136 */
      }
      int64_t lutIdx = 2 * ((int64_t)plc->trees * treeDepth * i + treeDepth * j + idx - (treeDepth - 1)); /* :138 */
      dr += plc->preds[lutIdx + 0];                                                                  /* :140 */
      if (flipV) dc += -plc->preds[lutIdx + 1];                                                      /* :141-145 */
      else dc += plc->preds[lutIdx + 1];
      root += 4 * treeDepth - 4;                                                                     /* :146 */
    }
    float t;
    t = dr * s; r += t;   /* :149  r += dr * s   (no FMA on amd64) */
    t = dc * s; c += t;   /* :150 */
    s *= plc->scales;     /* :151 */
  }
  res[0] = r; res[1] = c; res[2] = s;
}

static const float qCosTableF[33] = {256, 251, 236, 212, 181, 142, 97, 49, 0, -49, -97, -142, -181, -212, -236, -251, -256,
                                     -251, -236, -212, -181, -142, -97, -49, 0, 49, 97, 142, 181, 212, 236, 251, 256};
static const float qSinTableF[33] = {0, 49, 97, 142, 181, 212, 236, 251, 256, 251, 236, 212, 181, 142, 97, 49, 0,
                                     -49, -97, -142, -181, -212, -236, -251, -256, -251, -236, -212, -181, -142, -97, -49, 0};

/* ---- core/puploc.go:157-217 classifyRotatedRegion ----------------------- */
static void puploc_classify_rotated(const oracle_puploc *plc, float r, float c, float s, double a, int64_t nrows,
                                    int64_t ncols, const uint8_t *pixels, int64_t dim, int flipV, float res[3]) {
  int64_t root = 0;
  const int64_t treeDepth = plc->leaves;
  float qsin = s * qSinTableF[(int)(32.0 * a)];   /* :166 -- computed ONCE from the initial s */
  float qcos = s * qCosTableF[(int)(32.0 * a)];   /* :167 */
  for (int64_t i = 0; i < (int64_t)plc->stages; i++) {
    float dr = 0.0f, dc = 0.0f;
    for (int64_t j = 0; j < (int64_t)plc->trees; j++) {
      int64_t idx = 0;
      for (uint32_t k = 0; k < plc->depth; k++) {
        const int8_t *cd = plc->codes + root + 4 * idx;
        int64_t row1 = (int64_t)cd[0], row2 = (int64_t)cd[2], col1, col2;
        if (flipV) { col1 = neg_i8(cd[1]); col2 = neg_i8(cd[3]); }
        else { col1 = (int64_t)cd[1]; col2 = (int64_t)cd[3]; }
        int64_t iqc = (int64_t)qcos, iqs = (int64_t)qsin;
        int64_t r1 = go_min(nrows - 1, go_max(0, go_mul_add(65536, go_int_f32(r), iqc * row1 - iqs * col1)) >> 16);  /* :188 */
        int64_t c1 = go_min(ncols - 1, go_max(0, go_mul_add(65536, go_int_f32(c), iqs * row1 + iqc * col1)) >> 16);  /* :189 */
        int64_t r2 = go_min(nrows - 1, go_max(0, go_mul_add(65536, go_int_f32(r), iqc * row2 - iqs * col2)) >> 16);  /* :190 */
        int64_t c2 = go_min(ncols - 1, go_max(0, go_mul_add(65536, go_int_f32(c), iqs * row2 + iqc * col2)) >> 16);  /* :191 */
        idx = 2 * idx + 1 + (pixels[r1 * dim + c1] <= pixels[r2 * dim + c2] ? 1 : 0);                   /* :193-199 */
      }
      int64_t lutIdx = 2 * ((int64_t)plc->trees * treeDepth * i + treeDepth * j + idx - (treeDepth - 1));
      dr += plc->preds[lutIdx + 0];
      if (flipV) dc += -plc->preds[lutIdx + 1];
      else dc += plc->preds[lutIdx + 1];
      root += 4 * treeDepth - 4;
    }
    float t;
    t = dr * s; r += t;
    t = dc * s; c += t;
    s *= plc->scales;
  }
  res[0] = r; res[1] = c; res[2] = s;
}

void oracle_puploc_classify(const oracle_puploc *plc, float r, float c, float s, double angle, int nrows, int ncols,
                            const uint8_t *pixels, int dim, int flipV, float res[3]) {
  if (angle > 0.0) {
    if (angle > 1.0) angle = 1.0;
    puploc_classify_rotated(plc, r, c, s, angle, nrows, ncols, pixels, dim, flipV, res);
  } else {
    puploc_classify(plc, r, c, s, nrows, ncols, pixels, dim, flipV, res);
  }
}

/* Pool order of RunDetector's three sorts (:267-269), on (value, slot) pairs: numbers ascending (-0 == +0), every NaN
 * above every number, ties (NaNs among themselves too) by slot.  A total order, the same as the kernels' rank sorts:
 * with NaNs in the pool the order Go's sort.Sort leaves is an accident of its algorithm (DESIGN.md section 3.3). */
typedef struct { float v; int slot; } pool_entry;
static int cmp_f32(const void *a, const void *b) {
  const pool_entry *x = (const pool_entry *)a, *y = (const pool_entry *)b;
  const int nx = x->v != x->v, ny = y->v != y->v;
  if (nx != ny) return nx - ny;
  if (!nx && x->v != y->v) return (x->v > y->v) - (x->v < y->v);
  return (x->slot > y->slot) - (x->slot < y->slot);
}
static float pool_median(const float *pool, int mid) {
  pool_entry e[63];
  for (int i = 0; i < 63; i++) { e[i].v = pool[i]; e[i].slot = i; }
  qsort(e, 63, sizeof(pool_entry), cmp_f32);
  return e[mid].v;
}
/* int() of the picked row / col into the 32-bit field: truncation, saturated at the int32 range, NaN -> 0 (the CUDA
 * conversion; the reference's int is 64-bit and has no such bound) */
static int f32_to_i32(float v) {
  if (v != v) return 0;
  if (v >= 2147483648.0f) return INT32_MAX;
  if (v <= -2147483648.0f) return INT32_MIN;
  return (int)v;
}

/* ---- core/puploc.go:239-277 RunDetector --------------------------------- */
/* randoms: 3*perturbs float32 in [0,1), consumed in the reference's draw order
 * (row, col, scale per perturbation, :248-250).  Pool starts zeroed (:231-233).
 * Returns 0, or -1 when perturbs > 63 (the reference panics) or < 0. */
int oracle_puploc_run_detector(const oracle_puploc *plc, int row, int col, float scale, int perturbs,
                               const float *randoms, const uint8_t *pixels, int rows, int cols, int dim,
                               double angle, int flipV, int *out_row, int *out_col, float *out_scale) {
  float prow[63] = {0}, pcol[63] = {0}, pscale[63] = {0};
  if (perturbs > 63 || perturbs < 0) return -1;
  for (int i = 0; i < perturbs; i++) {
    float t1 = (float)scale * 0.15f;                                /* float32(pl.Scale)*0.15 */
    float rowf = (float)row + t1 * (0.5f - randoms[3 * i + 0]);       /* :248 */
    float colf = (float)col + t1 * (0.5f - randoms[3 * i + 1]);       /* :249 */
    float t2 = 0.15f * randoms[3 * i + 2];
    float sc = (float)scale * (0.925f + t2);                          /* :250 */
    float res[3];
    oracle_puploc_classify(plc, rowf, colf, sc, angle, rows, cols, pixels, dim, flipV, res);
    prow[i] = res[0]; pcol[i] = res[1]; pscale[i] = res[2];          /* :261-263 */
  }
  int mid = (int)go_math_round((double)perturbs / 2);   /* :273; :267-269 sort ALL 63 pooled slots */
  *out_row = f32_to_i32(pool_median(prow, mid));
  *out_col = f32_to_i32(pool_median(pcol, mid));
  *out_scale = pool_median(pscale, mid);
  return 0;
}

/* ---- core/flploc.go:36-57 GetLandmarkPoint (seed computation only) ------ */
void oracle_get_landmark_seed(int lrow, int lcol, int rrow, int rcol, int *row, int *col, float *scale) {
  int64_t dx = (int64_t)(lrow - rrow) * (lrow - rrow);   /* :37 */
  int64_t dy = (int64_t)(lcol - rcol) * (lcol - rcol);   /* :38 */
  double dist = sqrt((double)(dx + dy));                /* :39 */
  double r = (double)(lrow + rrow) / 2.0 + 0.25 * dist;  /* :41 */
  double c = (double)(lcol + rcol) / 2.0 + 0.15 * dist;  /* :42 */
  double s = 3.0 * dist;                                 /* :43 */
  *row = (int)r; *col = (int)c; *scale = (float)s;       /* :48-50 */
}

/* ---- core/grayscale.go:8-23 RgbToGrayscale on NRGBA (alpha ignored by the
 * formula; RGBA() of an opaque NRGBA pixel yields v*0x101) ---------------- */
void oracle_rgba_to_gray(const uint8_t *rgba, int64_t npix, uint8_t *gray) {
  for (int64_t i = 0; i < npix; i++) {
    uint32_t a = rgba[4 * i + 3];
    /* color.NRGBA.RGBA(): c = v*0x101; c = c*a16/0xffff with a16 = a*0x101 */
    uint32_t r = rgba[4 * i + 0] * 0x101u, g = rgba[4 * i + 1] * 0x101u, b = rgba[4 * i + 2] * 0x101u;
    uint32_t a16 = a * 0x101u;
    r = r * a16 / 0xffffu; g = g * a16 / 0xffffu; b = b * a16 / 0xffffu;
    gray[i] = (uint8_t)((0.299 * (double)r + 0.587 * (double)g + 0.114 * (double)b) / 256);
  }
}

/* ---- core/image.go:60-76 ImgToNRGBA, *image.YCbCr case -------------------
 * The per-pixel conversion is color.YCbCrToRGB of the Go standard library
 * (image/color/ycbcr.go, go1.22 per the reference's go.mod:3; NOT under the
 * reference tree), restated: 16.16 fixed point, yy1 = y*0x10101, and the
 * "bits 24..31 all zero ? >>16 : saturate" clamp.  The reference's own test
 * (core/image_test.go:118-138) restates the same constants with rounding and
 * accepts +-1; tests/test_oracle_pins.py checks this function against that
 * formula within +-1 for all six subsample ratios.
 * Offsets: image.YCbCr.YOffset / COffset relative to Rect.Min = (min_x, min_y),
 * min_x, min_y >= 0 (Go's x/2 truncates toward zero; a shift would not for
 * negative coordinates).  subsample = image.YCbCrSubsampleRatio (444, 422,
 * 420, 440, 411, 410 = 0..5). */
static uint8_t go_sat16(int32_t v) {
  if (((uint32_t)v & 0xff000000u) == 0) return (uint8_t)(v >> 16);
  return (uint8_t)(~(v >> 31));
}
void oracle_ycbcr_to_nrgba(const uint8_t *yp, const uint8_t *cbp, const uint8_t *crp, int y_stride, int c_stride,
                           int subsample, int min_x, int min_y, int width, int height, uint8_t *nrgba) {
  for (int dy = 0; dy < height; dy++) {
    for (int dx = 0; dx < width; dx++) {
      int x = min_x + dx, y = min_y + dy;
      int64_t siy = (int64_t)(y - min_y) * y_stride + (x - min_x);
      int64_t sic;
      switch (subsample) {
        case 1: sic = (int64_t)(y - min_y) * c_stride + (x / 2 - min_x / 2); break;
        case 2: sic = (int64_t)(y / 2 - min_y / 2) * c_stride + (x / 2 - min_x / 2); break;
        case 3: sic = (int64_t)(y / 2 - min_y / 2) * c_stride + (x - min_x); break;
        case 4: sic = (int64_t)(y - min_y) * c_stride + (x / 4 - min_x / 4); break;
        case 5: sic = (int64_t)(y / 2 - min_y / 2) * c_stride + (x / 4 - min_x / 4); break;
        default: sic = (int64_t)(y - min_y) * c_stride + (x - min_x); break;
      }
      int32_t yy1 = (int32_t)yp[siy] * 0x10101;
      int32_t cb1 = (int32_t)cbp[sic] - 128, cr1 = (int32_t)crp[sic] - 128;
      uint8_t *d = nrgba + 4 * ((int64_t)dy * width + dx);
      d[0] = go_sat16(yy1 + 91881 * cr1);
      d[1] = go_sat16(yy1 - 22554 * cb1 - 46802 * cr1);
      d[2] = go_sat16(yy1 + 116130 * cb1);
      d[3] = 0xff;
    }
  }
}
