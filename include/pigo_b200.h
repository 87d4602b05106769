/*
 * pigo_b200.h -- C-ABI of libpigo_b200.so, the H100 (sm_90a) drop-in for the
 * detection path of esimov/pigo (package "pigo", import github.com/esimov/pigo/core).
 *
 * Every entry point states the reference interface it replaces (file:line under the
 * reference tree).  The Go shim that binds these through cgo is go/pigo/ (see
 * INTEGRATION.md); the C++ mirror is include/pigo_b200.hpp; the Python/ctypes mirror used
 * by the tests and bench.py is pigo_b200/__init__.py.
 *
 * Conventions
 *  - plain pointers and sizes only; no CUDA/torch types (streams travel as void*).
 *  - every function returns a pigo_status (0 = ok, <0 = error); pigo_last_error() returns
 *    a thread-local message for the last failure on the calling thread.
 *  - the library NEVER falls back to a CPU path: without a usable sm_90 device every
 *    compute entry point fails with PIGO_E_NODEVICE / PIGO_E_CUDA.
 *  - the caller owns all input/output buffers.  Host buffers are copied inside the call
 *    (cgo rule: C keeps no Go pointer after return).  Handles own their device tables and
 *    are immutable after creation; compute calls on one handle may run concurrently from
 *    several OS threads (scratch comes from an internal per-handle pool).
 *  - frames handed over as HOST memory must hold (rows-1)*dim + cols bytes per frame (what the reference indexes);
 *    frames handed over as DEVICE memory (PIGO_FRAMES_DEVICE) must hold rows*dim bytes per frame.
 *  - pigo_last_error() is thread-local: a Go caller must fetch it on the OS thread that made the failing call
 *    (the shim brackets both with runtime.LockOSThread).
 *  - output capacity is supplied by the caller.  If more results exist than fit, the call
 *    sets *n_out / n_out[i] to the REQUIRED count and returns PIGO_E_CAP; the stored entries
 *    are then an unspecified subset (the scan emits unordered and sorts what fits), so the
 *    caller retries with a buffer of the reported size (all mirrors do).
 */
#ifndef PIGO_B200_H_
#define PIGO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

#define PIGO_B200_VERSION 200 /* 0.2.0 */

typedef enum {
  PIGO_OK = 0,
  PIGO_E_INVALID = -1,  /* bad argument / malformed cascade (the reference panics, core/pigo.go:64,81) */
  PIGO_E_CUDA = -2,     /* CUDA runtime failure; see pigo_last_error() */
  PIGO_E_CAP = -3,      /* output capacity too small; n_out holds the required count */
  PIGO_E_NOMEM = -4,
  PIGO_E_NODEVICE = -5  /* no sm_90 device visible: there is no CPU fallback */
} pigo_status;

/* Where the caller's frame / output buffers live. */
#define PIGO_MEM_HOST 0u          /* pageable or pinned host memory; copies happen inside the call */
#define PIGO_FRAMES_DEVICE 1u     /* `frames` is a device pointer on the active device            */
#define PIGO_OUT_DEVICE 2u        /* `out` and `n_out` are device pointers; the call is fully      */
                                  /* asynchronous on `stream` and returns without synchronising;   */
                                  /* PIGO_E_CAP is then NOT reported (check n_out[i] > cap later)  */

/* pigo.Detection (core/pigo.go:195-200): Row, Col, Scale int; Q float32.  16 bytes. */
typedef struct {
  int32_t row, col, scale;
  float q;
} pigo_det;

/* pigo.Puploc (core/puploc.go:14-19): Row, Col int; Scale float32; Perturbs int. */
typedef struct {
  int32_t row, col;
  float scale;
  int32_t perturbs;
} pigo_point;

typedef struct pigo_cascade pigo_cascade; /* pigo.Pigo          (core/pigo.go:37-43)   */
typedef struct pigo_puploc pigo_puploc;   /* pigo.PuplocCascade (core/puploc.go:23-30) */

/* ---- library -------------------------------------------------------------------------- */
const char *pigo_last_error(void);
int pigo_version(void);
/* Selects CUDA device `device` (verified to be compute capability 10.x) as the device of every
 * non-sharded entry point, process-wide; equivalent to pigo_init_devices(1u << device).  Called
 * implicitly with device 0 if omitted.  Each entry point binds its calling thread itself, so Go
 * callers need no runtime.LockOSThread for device affinity. */
int pigo_init(int device);
/* Multi-GPU (SURVEY.md section 8e; single process, no per-GPU host process needed): `device_mask` bit d
 * selects device d.  The *_sharded entry points split their frame batch over these devices
 * (shard g = frames [g*ceil(N/G), (g+1)*ceil(N/G)) on the g-th selected device); the lowest selected
 * device serves the non-sharded entry points.  Handles need no re-creation: their device tables are
 * replicated on a device at first use there.  Enables peer access between the selected devices. */
int pigo_init_devices(unsigned device_mask);
int pigo_device_count(void);
/* Waits for outstanding work and frees the library-owned scratch that belongs to no handle (handles stay valid). */
int pigo_shutdown(void);
/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
int64_t pigo_launch_count(void);
/* Pinned host memory for zero-staging H2D copies of frame batches. */
int pigo_alloc_pinned(void **ptr, size_t bytes);
int pigo_free_pinned(void *ptr);
/* Device buffers for callers that keep a frame batch resident across several calls (RunCascade, then RunDetector /
 * GetLandmarkPoint on the same frames) and pass it with PIGO_FRAMES_DEVICE. */
int pigo_device_alloc(void **ptr, size_t bytes);
int pigo_device_free(void *ptr);
int pigo_device_upload(void *dst_device, const void *src_host, size_t bytes);
int pigo_device_download(void *dst_host, const void *src_device, size_t bytes);

/* ---- face cascade: (*Pigo).Unpack, core/pigo.go:51-110 --------------------------------- */
/* Parses the `facefinder` binary layout (8 ignored bytes, u32 depth, u32 ntrees, then per
 * tree 4*2^d-4 int8 codes, 2^d f32 leaves, 1 f32 threshold) and uploads the device tables.
 * Returns PIGO_E_INVALID where the reference would panic on a short packet. */
int pigo_cascade_create(const uint8_t *packet, size_t len, pigo_cascade **out);
void pigo_cascade_destroy(pigo_cascade *c);
int pigo_cascade_info(const pigo_cascade *c, uint32_t *tree_depth, uint32_t *tree_num);

/* Scale ladder / grid arithmetic of RunCascade (core/pigo.go:226-231,:255), computed on the
 * host in float64 exactly as the reference does.  `scales` may be NULL. */
int pigo_scale_ladder(int min_size, int max_size, double scale_factor, int *scales, int cap, int *n_out);
int64_t pigo_count_windows(int rows, int cols, int min_size, int max_size, double shift_factor, double scale_factor);

/* ---- (*Pigo).RunCascade(cp CascadeParams, angle float64) []Detection, core/pigo.go:212-258
 * CascadeParams{ImageParams{Pixels,Rows,Cols,Dim},MinSize,MaxSize,ShiftFactor,ScaleFactor}
 * (core/pigo.go:16-34) is passed flattened.  Output order = the reference's emission order
 * (scale-major, then row, then col); Q is bit-identical to classifyRegion /
 * classifyRotatedRegion (core/pigo.go:113-191).  angle > 1 is clamped to 1 (:233-235). */
int pigo_run_cascade(const pigo_cascade *c, const uint8_t *pixels, int rows, int cols, int dim,
                     int min_size, int max_size, double shift_factor, double scale_factor, double angle,
                     pigo_det *out, int cap, int *n_out);

/* Additive batch form: `nframes` frames of identical geometry, `frame_stride` bytes apart.
 * out is [nframes][cap_per_frame], n_out is [nframes].  `flags` is a PIGO_* memory mask;
 * `stream` is a cudaStream_t (NULL = the library's own stream).  nframes <= 65535 per call; rows*dim < 2^31;
 * at most 2^31 windows per frame. */
int pigo_run_cascade_batch(const pigo_cascade *c, const uint8_t *frames, int nframes, size_t frame_stride,
                           int rows, int cols, int dim, int min_size, int max_size, double shift_factor,
                           double scale_factor, double angle, pigo_det *out, int cap_per_frame, int *n_out,
                           unsigned flags, void *stream);

/* Additive mixed-size form: `nimages` images of any geometry in one call (photos, thumbnails, several cameras).
 * pigo.ImageParams{Pixels,Rows,Cols,Dim} per image; the descriptor array itself always lives in host memory.
 * out is [nimages][cap_per_image], n_out is [nimages]; out[i][0..n_out[i]) is exactly what pigo_run_cascade returns
 * for image i alone (emission order, bit-equal Q, angle clamp).  The CascadeParams fields and `angle` are shared by
 * the whole call.  `flags` and `stream` as pigo_run_cascade_batch: with PIGO_FRAMES_DEVICE every `pixels` is a device
 * pointer holding rows*dim bytes, otherwise host memory holding (rows-1)*dim + cols bytes.  0 <= nimages <= 65535;
 * per image rows*dim < 2^31 and at most 2^31 windows.  Invalid arguments fail with PIGO_E_INVALID before any device
 * work; a stream that is being captured into a CUDA graph is rejected with PIGO_E_INVALID. */
typedef struct {
  const uint8_t *pixels;
  int32_t rows, cols, dim;
} pigo_image;

int pigo_run_cascade_images(const pigo_cascade *c, const pigo_image *images, int nimages, int min_size, int max_size,
                            double shift_factor, double scale_factor, double angle, pigo_det *out, int cap_per_image,
                            int *n_out, unsigned flags, void *stream);

/* Per-image angles: pigo_run_cascade_images with image i scanned at angles[i] (`angles` is a host array of nimages
 * doubles; > 0 rotates, > 1 is clamped to 1, <= 0 and NaN scan unrotated, as core/pigo.go:232-238).  out[i][0..n_out[i])
 * is byte for byte what pigo_run_cascade returns for image i alone at angles[i]; with every angle equal to a, the call
 * is pigo_run_cascade_images(..., a, ...).  An angle sweep is one call: list an image once per angle.  Host descriptors
 * that repeat (pixels, rows, cols, dim) are copied to the device once.  The rotated images keep one node table per
 * distinct int(32*a) on the device (at most 33, each nscales*ntrees*512 bytes over the call's longest ladder); past
 * 1 GiB of tables they run in several passes.  Everything else, including errors, as pigo_run_cascade_images; a null
 * `angles` with nimages > 0 fails with PIGO_E_INVALID. */
int pigo_run_cascade_images_angles(const pigo_cascade *c, const pigo_image *images, int nimages, const double *angles,
                                   int min_size, int max_size, double shift_factor, double scale_factor, pigo_det *out,
                                   int cap_per_image, int *n_out, unsigned flags, void *stream);

/* Multi-GPU form of the batch call: HOST frames (pinned memory from pigo_alloc_pinned recommended), sharded over
 * the devices of pigo_init_devices, one host thread and one stream per device, no data-path collective; every
 * device writes its frames' slices of `out` / `n_out`, so the result is identical to the single-GPU call.
 * PIGO_E_CAP is reported after all shards ran (every n_out[i] then holds the required count). */
int pigo_run_cascade_batch_sharded(const pigo_cascade *c, const uint8_t *frames, int nframes, size_t frame_stride,
                                   int rows, int cols, int dim, int min_size, int max_size, double shift_factor,
                                   double scale_factor, double angle, pigo_det *out, int cap_per_frame, int *n_out);

/* ---- (*Pigo).ClusterDetections(detections []Detection, iouThreshold float64) []Detection,
 * core/pigo.go:262-308.  Like the reference it SORTS `dets` in place by Q ascending (ties keep
 * their input order: a stable sort; Go's sort.Slice leaves tie order unspecified).  */
int pigo_cluster(pigo_det *dets, int n, double iou_threshold, pigo_det *out, int cap, int *n_out);
/* Batch form over the output layout of pigo_run_cascade_batch: dets is [nframes][cap_per_frame]
 * with n[i] valid entries (n[i] > cap_per_frame is treated as cap_per_frame). */
int pigo_cluster_batch(pigo_det *dets, const int *n, int nframes, int cap_per_frame, double iou_threshold,
                       pigo_det *out, int out_cap_per_frame, int *n_out, unsigned flags, void *stream);

/* ---- pupil / landmark cascades: (*PuplocCascade).UnpackCascade, core/puploc.go:38-103 --- */
int pigo_puploc_create(const uint8_t *packet, size_t len, pigo_puploc **out);
void pigo_puploc_destroy(pigo_puploc *p);
int pigo_puploc_info(const pigo_puploc *p, uint32_t *stages, float *scale_mul, uint32_t *trees, uint32_t *depth);

/* ---- (*PuplocCascade).RunDetector(pl Puploc, img ImageParams, angle float64, flipV bool) *Puploc,
 * core/puploc.go:239-277, for `nseeds` independent seeds on one image.
 * seeds[i].perturbs must be 0..63 (the reference panics above 63).  The reference draws
 * 3*perturbs values from the global math/rand stream (core/puploc.go:248-250), which is
 * auto-seeded and therefore not reproducible; here the caller either injects them
 * (`randoms` = [nseeds][63][3] float32 in [0,1), row/col/scale order) or passes NULL and the
 * library draws them from a counter-based generator keyed by (`rng_seed`, seed index).
 * Slots >= perturbs of the 63-entry pool are zero (fresh sync.Pool object, :228-236).
 * flipv: per-seed array (0/1) or NULL for all-false.  out[i].perturbs is 0 like the reference's. */
int pigo_puploc_run(const pigo_puploc *p, const pigo_point *seeds, int nseeds, const float *randoms,
                    uint64_t rng_seed, const uint8_t *pixels, int rows, int cols, int dim, double angle,
                    const uint8_t *flipv, pigo_point *out, unsigned flags, void *stream);

/* Additive batch form over several frames of identical geometry: seed i refines on frame seed_frame[i]
 * (frames `frame_stride` bytes apart; seed_frame may be NULL when nframes == 1). */
int pigo_puploc_run_frames(const pigo_puploc *p, const pigo_point *seeds, int nseeds, const int32_t *seed_frame,
                           const float *randoms, uint64_t rng_seed, const uint8_t *frames, int nframes,
                           size_t frame_stride, int rows, int cols, int dim, double angle, const uint8_t *flipv,
                           pigo_point *out, unsigned flags, void *stream);

/* Additive mixed-size form: seed i refines on images[seed_image[i]] (pigo_image as in pigo_run_cascade_images, each with
 * its own rows, cols, dim; seed_image may be NULL when nimages == 1).  The descriptor array lives in host memory; with
 * PIGO_FRAMES_DEVICE every `pixels` is a device pointer holding rows*dim bytes, otherwise host memory holding
 * (rows-1)*dim + cols bytes.  Everything else as pigo_puploc_run_frames.  1 <= nimages <= 65535, rows, cols >= 1. */
int pigo_puploc_run_images(const pigo_puploc *p, const pigo_point *seeds, int nseeds, const int32_t *seed_image,
                           const float *randoms, uint64_t rng_seed, const pigo_image *images, int nimages, double angle,
                           const uint8_t *flipv, pigo_point *out, unsigned flags, void *stream);

/* ---- (*PuplocCascade).GetLandmarkPoint(leftEye, rightEye *Puploc, img, perturb, flipV) *Puploc,
 * core/flploc.go:36-57: seed arithmetic in float64 on the host, then RunDetector(angle 0). */
int pigo_get_landmark_point(const pigo_puploc *p, const pigo_point *left_eye, const pigo_point *right_eye,
                            const uint8_t *pixels, int rows, int cols, int dim, int perturb, int flipv,
                            const float *randoms, uint64_t rng_seed, pigo_point *out);

/* ---- face -> ClusterDetections -> pupils -> landmarks for a frame batch, sequenced ON THE DEVICE (additive;
 * SURVEY.md section 8f row N1).  The reference's callers sequence these calls on the host, face by face:
 * core/flploc_test.go:75-154 and cmd/pigo/main.go:369-565.  Per frame: RunCascade(angle) -> ClusterDetections(iou) ->
 * for every cluster with Scale > min_face_scale: the two eye seeds (flploc_test.go:103-118), RunDetector(eye_perturbs,
 * angle, flipV=false) for each, then for call c = 0..ncalls-1 GetLandmarkPoint(leftEye, rightEye, flp_perturbs,
 * flp_flip[c]) on cascade flp[c] (the reference's sequence is 15 calls: lp46, lp44, lp42, lp38, lp312 each with flipV
 * false then true; lp93, lp84, lp82, lp81 with false; lp84 with true).
 * Outputs: faces[nframes][face_cap] = the clusters in the reference's order, n_faces[nframes] = number of clusters
 * (PIGO_E_CAP if one exceeds face_cap), points[nframes][face_cap][2 + ncalls] = left eye, right eye, then the landmark
 * calls in order; all-zero for clusters that were not refined (Scale <= min_face_scale).
 * Perturbation randoms: `randoms` = [nframes][face_cap][2 + ncalls][63][3] float32 (the parity tests inject them),
 * or NULL: counter-based generator keyed by (rng_seed, frame, cluster, call) -- so results do not depend on how a
 * batch is split over calls or devices.  flags: PIGO_FRAMES_DEVICE as usual; PIGO_OUT_DEVICE makes faces, n_faces,
 * points (and randoms) device pointers and the call asynchronous. */
typedef struct {
  int32_t min_size, max_size;
  double shift_factor, scale_factor, angle, iou_threshold;
  int32_t min_face_scale; /* 50 in the reference's callers */
  int32_t eye_perturbs;   /* 50 (tests) / 63 (CLI) */
  int32_t flp_perturbs;   /* 63 */
  int32_t det_cap;        /* raw detections kept per frame before clustering; 0 = 2048; PIGO_E_CAP if exceeded */
} pigo_pipeline_params;

int pigo_detect_batch(const pigo_cascade *face, const pigo_puploc *puploc, const pigo_puploc *const *flp,
                      const uint8_t *flp_flip, int ncalls, const uint8_t *frames, int nframes, size_t frame_stride,
                      int rows, int cols, int dim, const pigo_pipeline_params *params, const float *randoms,
                      uint64_t rng_seed, pigo_det *faces, int face_cap, int *n_faces, pigo_point *points,
                      unsigned flags, void *stream);
/* The same over the devices of pigo_init_devices (HOST buffers; frames sharded like pigo_run_cascade_batch_sharded,
 * every device runs the whole sequence on its frames, results land in the caller's arrays in frame order). */
int pigo_detect_batch_sharded(const pigo_cascade *face, const pigo_puploc *puploc, const pigo_puploc *const *flp,
                              const uint8_t *flp_flip, int ncalls, const uint8_t *frames, int nframes,
                              size_t frame_stride, int rows, int cols, int dim, const pigo_pipeline_params *params,
                              const float *randoms, uint64_t rng_seed, pigo_det *faces, int face_cap, int *n_faces,
                              pigo_point *points);

/* Additive mixed-size form of pigo_detect_batch: `nimages` images of any geometry (photos, thumbnails, several cameras)
 * in one call, frame f replaced by image i.  Outputs faces[nimages][face_cap], n_faces[nimages],
 * points[nimages][face_cap][2 + ncalls]; randoms (optional) [nimages][face_cap][2 + ncalls][63][3].  Image i's slices are
 * byte for byte what pigo_detect_batch(nframes = 1) returns for that image alone given its randoms slice; the library
 * generator's key is the same (slot = i*face_cap*(2+ncalls) + k*(2+ncalls) + call), so on images of one geometry both
 * calls agree byte for byte.  det_cap / face_cap, PIGO_E_CAP with the required counts, flags and stream as
 * pigo_detect_batch.  The descriptor array lives in host memory; pixels as pigo_run_cascade_images.  The CascadeParams
 * fields and angle of `params` are shared by every image.  0 <= nimages <= 65535, rows, cols >= 1 per image,
 * nimages*face_cap*(2+ncalls) <= 2^31-1.  Invalid arguments fail with PIGO_E_INVALID before any device work; a stream that
 * is being captured into a CUDA graph is rejected with PIGO_E_INVALID. */
int pigo_detect_images(const pigo_cascade *face, const pigo_puploc *puploc, const pigo_puploc *const *flp,
                       const uint8_t *flp_flip, int ncalls, const pigo_image *images, int nimages,
                       const pigo_pipeline_params *params, const float *randoms, uint64_t rng_seed, pigo_det *faces,
                       int face_cap, int *n_faces, pigo_point *points, unsigned flags, void *stream);

/* Per-image angles: pigo_detect_images with params->angle replaced by angles[i] for image i (`angles` is a host array of
 * nimages doubles, rules as pigo_run_cascade_images_angles; params->angle is ignored).  The scan and the eye RunDetector
 * of image i use angles[i]; the landmark calls stay at angle 0, as GetLandmarkPoint does.  The generator key is
 * pigo_detect_images' key, so with every angle equal both calls agree byte for byte.  Everything else as
 * pigo_detect_images; a null `angles` with nimages > 0 fails with PIGO_E_INVALID. */
int pigo_detect_images_angles(const pigo_cascade *face, const pigo_puploc *puploc, const pigo_puploc *const *flp,
                              const uint8_t *flp_flip, int ncalls, const pigo_image *images, int nimages,
                              const double *angles, const pigo_pipeline_params *params, const float *randoms,
                              uint64_t rng_seed, pigo_det *faces, int face_cap, int *n_faces, pigo_point *points,
                              unsigned flags, void *stream);

/* ---- Angle sweep merged per image (additive).  A caller who does not know a photo's tilt scans it at several angles and
 * wants one face list, each face with the angle it was found at.  Every image is scanned at every angle of the host
 * array angles[nangles] (rules as pigo_run_cascade_images_angles).  For image i:
 *   D_i = RunCascade(image i, angles[0]) ++ ... ++ RunCascade(image i, angles[nangles-1])   (each list in emission order)
 *   clusters of image i = ClusterDetections(D_i, iou_threshold)   (stable sort by Q: ties keep their order in D_i)
 *   angle_index[i][k] = index into `angles` of the member of cluster k with the largest Q (among equal Q the earliest in
 *                       D_i, so the angle listed first wins).
 * Listing two values of one orientation (0 and 1, say, or 0 and -0.5) scans it twice, and every face it finds is counted
 * twice in D_i; the clusters then weigh that orientation double.
 * det_cap (0 = 2048) bounds the raw detections of each (image, angle) entry: PIGO_E_CAP names the entry that exceeds it.
 * out[nimages][cap_per_image] / n_out[nimages] as pigo_run_cascade_images (PIGO_E_CAP with the required counts in n_out);
 * angle_index[nimages][cap_per_image] may be NULL.  With PIGO_OUT_DEVICE, out, angle_index and n_out are device pointers
 * and the call is asynchronous.  Host pixels of an image are copied to the device once.  Invalid arguments fail with
 * PIGO_E_INVALID before any device work: a null `angles`, nangles < 1, nimages*nangles > 65535,
 * nimages*nangles*det_cap > 2^31-1, and the checks of pigo_run_cascade_images; a stream that is being captured into a
 * CUDA graph is rejected with PIGO_E_INVALID. */
int pigo_run_cascade_images_sweep(const pigo_cascade *c, const pigo_image *images, int nimages, const double *angles, int nangles,
                                  int min_size, int max_size, double shift_factor, double scale_factor, double iou_threshold,
                                  int det_cap, pigo_det *out, int32_t *angle_index, int cap_per_image, int *n_out,
                                  unsigned flags, void *stream);

/* Pipeline form: the clusters of pigo_run_cascade_images_sweep (params->iou_threshold, params->det_cap per (image, angle)
 * entry; params->angle is ignored), then pigo_detect_images' per-face sequence on them, with the eye RunDetector of face k
 * of image i at angles[face_angle[i][k]] and the landmark calls at angle 0, as GetLandmarkPoint does.  Outputs, randoms
 * layout, generator key, face_cap, PIGO_E_CAP (n_faces then holds the required counts), flags and stream as
 * pigo_detect_images with nimages images; face_angle[nimages][face_cap] may be NULL.  With nangles == 1 the call returns
 * byte for byte what pigo_detect_images_angles returns with every angle equal to angles[0], and every face_angle is 0.
 * Invalid arguments as pigo_run_cascade_images_sweep and pigo_detect_images (nimages*face_cap*(2+ncalls) <= 2^31-1). */
int pigo_detect_images_sweep(const pigo_cascade *face, const pigo_puploc *puploc, const pigo_puploc *const *flp,
                             const uint8_t *flp_flip, int ncalls, const pigo_image *images, int nimages, const double *angles,
                             int nangles, const pigo_pipeline_params *params, const float *randoms, uint64_t rng_seed,
                             pigo_det *faces, int32_t *face_angle, int face_cap, int *n_faces, pigo_point *points,
                             unsigned flags, void *stream);

/* ---- RgbToGrayscale(src image.Image) []uint8, core/grayscale.go:8-23, for *image.NRGBA input (what GetImage returns,
 * core/image.go:13-33): gray = uint8((0.299 r + 0.587 g + 0.114 b) / 256) in float64 on the 16-bit, alpha-premultiplied
 * channels color.NRGBA.RGBA() yields.  rgba is [npixels][4] (R,G,B,A), gray is [npixels].  flags: PIGO_FRAMES_DEVICE /
 * PIGO_OUT_DEVICE say where rgba / gray live.  (SURVEY.md section 8f row N2: the stage just before the hot path.) */
int pigo_rgba_to_gray(const uint8_t *rgba, size_t npixels, uint8_t *gray, unsigned flags, void *stream);

/* ---- ImgToNRGBA(img image.Image) *image.NRGBA for *image.YCbCr sources, core/image.go:60-76 (what DecodeImage yields
 * for a JPEG; SURVEY.md section 8f row N3): per pixel color.YCbCrToRGB(Y[YOffset], Cb[COffset], Cr[COffset]) with
 * alpha 0xff, bit-exact with Go's 16.16 fixed-point conversion.  `subsample` is image.YCbCrSubsampleRatio (0..5 = 444,
 * 422, 420, 440, 411, 410); (min_x, min_y) = img.Rect.Min (>= 0), width/height = Rect size; the Y plane holds `height`
 * rows of y_stride bytes, the chroma planes c_stride bytes per chroma row.  Outputs (either may be NULL): nrgba
 * [height][width][4], gray [height][width] = RgbToGrayscale of the converted image (fused).  flags as pigo_rgba_to_gray. */
int pigo_ycbcr_to_nrgba(const uint8_t *y, const uint8_t *cb, const uint8_t *cr, int y_stride, int c_stride,
                        int subsample, int min_x, int min_y, int width, int height, uint8_t *nrgba, uint8_t *gray,
                        unsigned flags, void *stream);

/* ---- RgbToGrayscale(ImgToNRGBA(img)) for a batch of decoded images of any size (core/grayscale.go:8-23, core/image.go:35-90;
 * what cmd/pigo/main.go:281-286 feeds the detector), straight into device memory for the mixed-size calls.
 * Each pigo_decoded describes one decoded Go image at its rectangle's origin:
 *   PIGO_DECODED_YCBCR  *image.YCbCr: plane = Y[YOffset(Rect.Min):], Cb and Cr[COffset(Rect.Min):]; stride = YStride, CStride;
 *                       subsample = SubsampleRatio (0..5 = 444, 422, 420, 440, 411, 410); (min_x, min_y) = Rect.Min (>= 0)
 *   PIGO_DECODED_NRGBA  *image.NRGBA: plane[0] = Pix[PixOffset(Rect.Min):], stride[0] = Stride
 *   PIGO_DECODED_RGBA   *image.RGBA (alpha-premultiplied), laid out as NRGBA
 *   PIGO_DECODED_GRAY   *image.Gray: plane[0] = Pix[PixOffset(Rect.Min):], stride[0] = Stride
 *   PIGO_DECODED_GRAY16, _RGBA64, _NRGBA64, _CMYK, _PALETTED  *image.Gray16, RGBA64, NRGBA64, CMYK, Paletted:
 *                       plane[0] = Pix[PixOffset(Rect.Min):], stride[0] = Stride; 2, 8, 8, 4 and 1 bytes per pixel
 *                       (16-bit samples big-endian, as Go stores them).  Paletted only: plane[1] = the palette as
 *                       stride[1] (1..256) NRGBA entries of 4 bytes, entry i = color.NRGBAModel.Convert(Palette[i]).
 * width, height = Rect size.  Fields a format does not use are ignored, but take part in the repeat test below.
 * Output: `gray` is a device buffer of *gray_bytes bytes.  Source i gets a 256-byte-aligned slot of height rows of exactly
 * width bytes and images[i] = {slot, height, width, width} (dim == width: the rotated scan's column clamp,
 * core/pigo.go:168,171, reads past cols on some shapes, so a padded pitch would change results).  Pass `images` unchanged,
 * with PIGO_FRAMES_DEVICE, to pigo_run_cascade_images[_angles], pigo_detect_images[_angles] or pigo_puploc_run_images.
 * Slot bytes: YCbCr = the fused `gray` output of pigo_ycbcr_to_nrgba; NRGBA = pigo_rgba_to_gray of the pixels; RGBA =
 * the same after color.NRGBAModel (c*0xffff/a >> 8 in uint32, a == 0 -> 0; a channel above alpha wraps as in Go);
 * Gray = Y (luma(Y, Y, Y, 0xff) == Y for every Y).  The other types go through color.NRGBAModel (go1.22 image/color, all
 * arithmetic uint32; nrgbaModel(r, g, b, a) = a == 0xffff: c >> 8; a == 0: all zero; else uint8((c*0xffff/a) >> 8),
 * alpha uint8(a >> 8)) and then luma: Gray16 = the high byte of Y (nrgbaModel(Y, Y, Y, 0xffff)); RGBA64 =
 * nrgbaModel(R, G, B, A) of the stored channels (a channel above alpha wraps as in Go); NRGBA64 = nrgbaModel(C*A/0xffff
 * for each colour channel, A), keeping the precision that premultiplying loses; CMYK = w = 0xffff - K*0x101,
 * R = (0xffff - C*0x101)*w/0xffff (G from M, B from Y), alpha 0xffff; Paletted = luma(palette[index]).
 * One difference from the reference: a palette index at or past stride[1] gives gray 0 here, where Go's Paletted.At
 * would panic; Go's PNG decoder never makes such an index, since it extends a short palette with opaque black (gray 0).
 * Descriptors that are byte-identical share one slot and are converted once (an angle sweep of one photo costs one
 * conversion).  Required size = sum over distinct descriptors of round256(width*height).  If `gray` is NULL or
 * *gray_bytes is smaller, the call sets *gray_bytes to the required size and returns PIGO_E_CAP; that query, every
 * argument check and a call with n == 0 (PIGO_OK, required size 0) need no device.  PIGO_E_INVALID: n outside 0..65535, an unknown
 * format (4 is not assigned), subsample outside 0..5, a negative YCbCr origin, width or height < 1, width*height >= 2^31,
 * a stride below width * bytes per pixel (CStride: below the rectangle's chroma width), a null plane, a null palette or a
 * palette length outside 1..256, a null src / images / gray_bytes, or a stream that is being captured into a CUDA graph.
 * flags: PIGO_FRAMES_DEVICE = the planes are device pointers; on a caller's stream the call then returns without
 * synchronising.  Host planes are read only during the call: one copy per plane per distinct source, of the bytes the
 * rectangle covers.  With stream NULL the call synchronises before it returns. */
#define PIGO_DECODED_YCBCR 0
#define PIGO_DECODED_NRGBA 1
#define PIGO_DECODED_RGBA 2
#define PIGO_DECODED_GRAY 3
#define PIGO_DECODED_GRAY16 5
#define PIGO_DECODED_RGBA64 6
#define PIGO_DECODED_NRGBA64 7
#define PIGO_DECODED_CMYK 8
#define PIGO_DECODED_PALETTED 9
typedef struct {
  int32_t format, subsample, min_x, min_y, width, height;
  const uint8_t *plane[3];
  int32_t stride[2];
} pigo_decoded;

int pigo_gray_images(const pigo_decoded *src, int n, uint8_t *gray, size_t *gray_bytes, pigo_image *images, unsigned flags,
                     void *stream);

/* ---- Multi-GPU forms of the mixed-size and decoded calls: HOST inputs and HOST outputs, over the devices of
 * pigo_init_devices (the default device if none were selected), one host thread per shard, no data-path collective.
 * The entries are cut into contiguous ranges of the caller's order (an entry is never split) that balance a modelled
 * cost, count_windows x (rotated ? 1.4 : 1) + 4096 per entry, not the entry count (pigo_shard_plan); shard s writes its
 * entries' slices of the output arrays.  For any split, entry i's slices are byte for byte what the single-device call
 * returns:
 *   pigo_run_cascade_images_sharded  = pigo_run_cascade_images_angles (pigo_run_cascade_images at angle 0 when angles is NULL)
 *   pigo_detect_images_sharded       = pigo_detect_images_angles (angles NULL: params->angle for every image), with the same
 *                                      randoms ([nimages][face_cap][2+ncalls][63][3]) or the same rng_seed: a shard that
 *                                      starts at image lo keys its generator and reads its randoms as image lo of the call
 *   pigo_*_decoded_sharded           = pigo_gray_images of the sources, then the matching call above on its images; each
 *                                      device copies and converts its own sources (repeats within a shard share a slot)
 * Host images listed several times in a shard are copied to that shard's device once.  Argument checks are those of the
 * single-device calls (the decoded forms: pigo_gray_images' checks first) and need no device.  PIGO_E_CAP: the first
 * other error of a shard wins; otherwise, after every shard ran, every n_out[i] / n_faces[i] holds the required count.
 * Developer option "shard_split" = k > 0 cuts these calls into k shards, shard s on the (s mod G)-th device. */
int pigo_run_cascade_images_sharded(const pigo_cascade *c, const pigo_image *images, int nimages, const double *angles,
                                    int min_size, int max_size, double shift_factor, double scale_factor, pigo_det *out,
                                    int cap_per_image, int *n_out);
int pigo_detect_images_sharded(const pigo_cascade *face, const pigo_puploc *puploc, const pigo_puploc *const *flp,
                               const uint8_t *flp_flip, int ncalls, const pigo_image *images, int nimages,
                               const double *angles, const pigo_pipeline_params *params, const float *randoms,
                               uint64_t rng_seed, pigo_det *faces, int face_cap, int *n_faces, pigo_point *points);
int pigo_run_cascade_decoded_sharded(const pigo_cascade *c, const pigo_decoded *src, int n, const double *angles,
                                     int min_size, int max_size, double shift_factor, double scale_factor, pigo_det *out,
                                     int cap_per_image, int *n_out);
int pigo_detect_decoded_sharded(const pigo_cascade *face, const pigo_puploc *puploc, const pigo_puploc *const *flp,
                                const uint8_t *flp_flip, int ncalls, const pigo_decoded *src, int n, const double *angles,
                                const pigo_pipeline_params *params, const float *randoms, uint64_t rng_seed, pigo_det *faces,
                                int face_cap, int *n_faces, pigo_point *points);
/* The split the four calls above make (no device needed): first[0..n_used] are the shards' first entries, first[n_used] ==
 * nimages, n_used = min(shards, nimages) non-empty shards.  The largest shard's cost is the least any contiguous split
 * into that many shards reaches.  nshards = 0: the count the calls use (option shard_split, else one per selected
 * device); `first` may be NULL (n_used only) and otherwise holds n_used + 1 entries (nimages + 1 always suffice).
 * `angles` NULL: every entry unrotated.  Images are checked as in pigo_run_cascade_images; pixels are not read. */
int pigo_shard_plan(const pigo_image *images, int nimages, const double *angles, int min_size, int max_size,
                    double shift_factor, double scale_factor, int nshards, int *first, int *n_used);

/* ---- tuning / introspection (not part of the reference surface) ------------------------- */
/* Process-global developer knobs (kernel variants, group sizes, per-kernel timing): debugging and
 * benchmarking only, NOT per handle -- set them before the first compute call and leave them alone while
 * other threads are inside the library.  Names: pigo_b200/csrc/host.h (struct Options). */
int pigo_set_option(const char *name, int64_t value);
/* Host-only: JSON description of how RunCascade would be scheduled for this geometry (scale ladder, tile bands and
 * their shared-memory tile geometry, first ladder entry left to the gather role, tile role of the fused kernel, band
 * ratio), for a call of many frames.  Needs no device. */
int pigo_describe_plan(int rows, int cols, int min_size, int max_size, double shift_factor, double scale_factor,
                       char *json, size_t cap);
/* The same for a call of `nframes` frames of this geometry (>= 1): small calls plan narrower tile bands. */
int pigo_describe_plan_frames(int rows, int cols, int min_size, int max_size, double shift_factor, double scale_factor,
                              int nframes, char *json, size_t cap);
int64_t pigo_get_option(const char *name);
/* Copies the default device's block-interleaved copy of a depth-6 cascade (the table the unrotated deep kernel reads) to
 * dst and sets *bytes to its size; dst == NULL only sets *bytes (0: depth != 6, no such table). */
int pigo_cascade_block_table(pigo_cascade *c, uint8_t *dst, size_t *bytes);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* PIGO_B200_H_ */
