// host.h -- host-side declarations shared by the translation units of libpigo_b200.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"

namespace pigo {

int set_err(int code, const char* fmt, ...);
extern std::atomic<long long> g_launches;
// Makes kernel `fn` on the current device accept launches of `bytes` of dynamic shared memory.  The attribute is shared
// by every host thread, so it only ever grows: calls that run concurrently on one device (several threads on one handle,
// several shards of a sharded call) never lower it below another launch's request.
void raise_dyn_smem(const void* fn, int bytes);

// Per-kernel CUDA-event timing (enabled by option "timing"): every launch of kernel class `slot` is bracketed by an
// event pair on its stream; "t_<name>_ns" / "t_<name>_n" return the summed device time and the launch count.
enum TimeSlot { T_TILED = 0, T_GATHER, T_DEEP, T_FINALIZE, T_CLUSTER, T_PUPLOC, T_GRAY, T_SEEDS, T_ROTTAB, T_YCBCR, T_GRAY_IMAGES, T_MERGE, T_NSLOTS };
void timing_reset();
void walk_stats_reset();
long long walk_stats_query(int which);
unsigned long long* walk_stats_buffer(int dev);   // nullptr unless option walk_stats is on
long long timing_query(const std::string& key);
void timing_begin(int slot, cudaStream_t st);
void timing_end(int slot, cudaStream_t st);

struct Options {
  std::atomic<long long> scan_mode{0};      // 0 auto (fused + gather-v2 + deep), 1 universal gather kernel only, 3 gather-v2 + deep only
  std::atomic<long long> chunk{256};        // windows per work chunk of the universal gather kernel
  std::atomic<long long> gather_ctas_per_sm{0};   // CTAs per SM of the gather-v2 kernel (0 = auto: 2 unrotated, 4 rotated; capped at occupancy)
  std::atomic<long long> tile_max_scale{0}; // largest window size routed to the tile warps (0 = auto)
  std::atomic<long long> tile_warps{24};    // warps (= private tile buffers) per CTA of the fused kernel
  std::atomic<long long> tile_ni{1};        // item slots per lane of a tile warp
  std::atomic<long long> gather_warps{8};   // gather-role warps per CTA of the fused kernel (0 = separate gather launch)
  std::atomic<long long> tile_ks{48};       // cascade trees resident in shared memory (fused kernel)
  std::atomic<long long> gather_ks{32};     // cascade trees resident in shared memory (gather-v2 kernel)
  std::atomic<long long> gather_ni{1};      // windows per lane in the gather role / gather-v2 kernel
  std::atomic<long long> fused_smem_kb{0};  // cap on the fused kernel's shared memory (0 = all 227 KB)
  std::atomic<long long> tile_min_core{32};        // a band is tiled only if its core edge is at least this many pixels ...
  std::atomic<long long> tile_min_core_steps{3};   // ... and at least this many window steps of its largest scale
  std::atomic<long long> tile_prefetch{0};  // tile warps: child-pair prefetch (64-bit node loads) vs plain 32-bit node loads
  std::atomic<long long> gather_block{0};   // gather block edge in windows: 16, 8, or 0 = auto (8 for <= 4 frames)
  std::atomic<long long> deep_group{0};     // lanes (trees per step) per window in the deep kernel: 8, 16, 32; 0 = auto (32 for calls of <= 4 M windows: latency, else 8)
  std::atomic<long long> sub_batch{0};      // frames per pipeline group (0 = auto: 128 for resident frames; host frames: see host_first)
  std::atomic<long long> host_stream{1};    // host frames: 1 = the scan kernels start at once and wait IN-KERNEL for each frame's copy (a ready counter the copy
                                            // stream bumps after every chunk), so copy and scan overlap frame by frame; 0 = per-group copy events (round 1)
  std::atomic<long long> stream_taper{0};   // host_stream group sizes: 0 = uniform 128, 1 = 128 then half of the rest (>= 32), 2 = 1/8, 1/4, 3/8, 3/16, 1/16 of the batch
  std::atomic<long long> copy_chunk{8};     // host_stream: frames per H2D copy chunk
  std::atomic<long long> tile_tmap{1};      // tile fill: 1 = one TMA tensor copy per tile (cuTensorMapEncodeTiled descriptors), 0 = one bulk copy per tile row
  std::atomic<long long> walk_stats{0};     // 1 = count live lanes per walk iteration of the tile role ("walk_useful" / "walk_iters" read them back)
  std::atomic<long long> tile_core_cap{0};  // largest tile core edge in pixels; 0 = unlimited
  std::atomic<long long> deep_smem{0};      // deep kernel with the tree records in shared memory: 0 = auto, 1 = on, 2 = off; deep_smem_threads = CTA size
  std::atomic<long long> deep_smem_threads{256};
  std::atomic<long long> deep_smem_lo{24};   // first resident tree / number of resident trees of that kernel
  std::atomic<long long> deep_smem_k{128};
  std::atomic<long long> gather_limit{0};   // trees a gather-role window walks before it goes to the deep kernel; 0 = auto (8 for calls of <= 40 M windows, else 16; rotated and mixed-size scans see scan_driver.cu)
  std::atomic<long long> queue_cap{0};      // developer knob: cap of the deep queue in items (0 = sized from the window count)
  std::atomic<long long> tile_ptab{0};      // fused kernel, tile role: 1 = per-scale offset tables, scale-synchronous rounds (scan_ptab_kernel)
  std::atomic<long long> ptab_kt{16};       // trees per table of that kernel (survivors go to the deep queue)
  std::atomic<long long> ptab_ks{24};       // raw cascade trees its gather warps keep in shared memory
  std::atomic<long long> tile_head{0};      // fused kernel, tile role: 0 = classic lane refill from tree 0, N = dense head over the first N trees (scan_head_kernel)
  std::atomic<long long> head_back{12};     // dense head: generic phase parks its live windows and returns to the head below this many live lanes
  std::atomic<long long> deep_flat{0};      // deep kernel loop: 0 = groups of a warp fetch together (round 1), 1 = flat (fetch or step per iteration)
  std::atomic<long long> rot_mode{0};       // rotated scan: 0 = table-driven block kernel + deep kernel, 1 = universal gather kernel
  std::atomic<long long> puploc_stage{1};   // pair kernel: 0 = all global, 1 = the current stage's node codes staged in shared memory, 2 = + the stage's pixel patch when it fits
  std::atomic<long long> puploc_mode{0};    // RunDetector kernel: 0 = (perturbation, tree)-pair kernel, 1 = warp-per-perturbation kernel
  std::atomic<long long> lanes{1};          // internal streams the groups alternate between
  std::atomic<long long> tile_tail_min{6};  // tail policy threshold
  std::atomic<long long> tile_band_ratio{0};    // a band spans scales up to ratio/100 x its first scale; 0 = auto (200, or 140 for calls of <= 2 M windows)
  std::atomic<long long> timing{0};         // 1 = bracket every kernel with CUDA events (bench.py roofline pass)
  std::atomic<long long> shard_split{0};    // sharded mixed-size / decoded calls: 0 = one shard per selected device, k > 0 = k shards,
                                            // shard s on device s mod G (several shards share a device: the multi-shard path on one GPU)
  std::atomic<long long>* find(const std::string& k) {
    struct Entry { const char* name; std::atomic<long long> Options::*field; };
    static const Entry table[] = {
        {"scan_mode", &Options::scan_mode}, {"chunk", &Options::chunk}, {"gather_ctas_per_sm", &Options::gather_ctas_per_sm},
        {"tile_max_scale", &Options::tile_max_scale}, {"tile_warps", &Options::tile_warps}, {"tile_ni", &Options::tile_ni},
        {"gather_warps", &Options::gather_warps}, {"tile_ks", &Options::tile_ks}, {"gather_ks", &Options::gather_ks},
        {"gather_ni", &Options::gather_ni}, {"fused_smem_kb", &Options::fused_smem_kb}, {"tile_min_core", &Options::tile_min_core},
        {"tile_min_core_steps", &Options::tile_min_core_steps}, {"tile_prefetch", &Options::tile_prefetch},
         {"gather_block", &Options::gather_block}, {"deep_group", &Options::deep_group},
        {"sub_batch", &Options::sub_batch}, {"lanes", &Options::lanes}, {"tile_tail_min", &Options::tile_tail_min},
        {"tile_band_ratio", &Options::tile_band_ratio}, {"timing", &Options::timing}, {"host_stream", &Options::host_stream}, {"copy_chunk", &Options::copy_chunk}, {"stream_taper", &Options::stream_taper},
        {"deep_flat", &Options::deep_flat}, {"tile_head", &Options::tile_head}, {"tile_ptab", &Options::tile_ptab}, {"queue_cap", &Options::queue_cap}, {"ptab_kt", &Options::ptab_kt}, {"ptab_ks", &Options::ptab_ks}, {"tile_core_cap", &Options::tile_core_cap}, {"walk_stats", &Options::walk_stats}, {"tile_tmap", &Options::tile_tmap}, {"gather_limit", &Options::gather_limit}, {"deep_smem", &Options::deep_smem}, {"deep_smem_threads", &Options::deep_smem_threads}, {"deep_smem_lo", &Options::deep_smem_lo}, {"deep_smem_k", &Options::deep_smem_k}, {"head_back", &Options::head_back}, {"rot_mode", &Options::rot_mode}, {"puploc_mode", &Options::puploc_mode}, {"puploc_stage", &Options::puploc_stage}, {"shard_split", &Options::shard_split}};
    for (const Entry& e : table)
      if (k == e.name) return &(this->*e.field);
    return nullptr;
  }
  bool set(const std::string& k, long long v) {
    std::atomic<long long>* f = find(k);
    if (!f) return false;
    *f = v;
    if (f == &timing) timing_reset();
    if (f == &walk_stats) walk_stats_reset();
    return true;
  }
  long long get(const std::string& k) {
    if (k.rfind("t_", 0) == 0) return timing_query(k);
    if (k == "walk_useful") return walk_stats_query(0);
    if (k == "walk_iters") return walk_stats_query(1);
    std::atomic<long long>* f = find(k);
    return f ? f->load() : -1;
  }
};
extern Options g_opt;

struct PuplocTables {
  const int8_t* codes;  // [stages*trees][4*leaves]: 4 pad bytes, then the reference's 4*leaves-4 code bytes (core/puploc.go:75-80), so that node i
                        // sits at word i+1 and its two children (nodes 2i+1, 2i+2) at the 8-byte aligned word pair 2i+2, 2i+3
  const float* preds;   // [stages*trees][leaves][2]
  int32_t stages, trees, depth, leaves;
  float scales;
};

// Work list of the (perturbation, tree)-pair RunDetector kernel (puploc.cu): work item w in [0, nwork) is the RunDetector
// call of slot (w / span) * stride + first + w % span; position j = w % span selects the cascade tab[tab_of[j]] and the
// flip flag flip_of[j] (or flipv[slot] when given).  All pointers are device pointers.
constexpr int kMaxPupTabs = 12;
struct PupWork {
  const pigo_point* seeds;     // [slots]; perturbs < 0 marks an inactive slot
  pigo_point* out;             // [slots]
  const float* randoms;        // [slots][63][3] injected perturbation randoms, or nullptr (counter-based generator)
  uint64_t rng_seed;
  uint64_t slot_base;          // added to the slot index in the generator key (frame shards of one logical batch)
  const uint8_t* frames;
  size_t frame_stride;
  const int32_t* slot_frame;   // frame of each slot (nullptr = frame 0) unless slots_per_frame > 0
  const uint8_t* flipv;        // per-slot flip flags (nullptr: use flip_of[j])
  int32_t slots_per_frame;     // > 0: frame = slot / slots_per_frame
  int32_t nrows, ncols, dim, rot_slot;   // rot_slot: -1 unrotated; kRotSlotPerImage: images[frame].rot_slot; kRotSlotPerFace: face_rot[slot / stride]
  int32_t first, span, stride, nwork, ntabs;
  PuplocTables tab[kMaxPupTabs];
  uint8_t tab_of[32], flip_of[32];
  const ImageDesc* images;     // mixed-size call: the image table the frame indices refer to (frames .. dim unused); nullptr = uniform frames
  const int32_t* face_rot;     // angle sweep (rot_slot == kRotSlotPerFace, with images): rotation slot of face slot `slot / stride`
};

// Angle sweep merge (cluster.cu).  cluster_kernel<true> reads the sorted keys (position in D_i in the low 32 bits) and the
// per-position angle tags, and writes each cluster's tag and slot_of[tag] (either output may be nullptr).
struct SweepTags {
  const uint64_t* keys;
  const int32_t* tag;
  const int32_t* slot_of;
  int32_t* out_tag;
  int32_t* out_rot;
};
// Device scratch of launch_sweep_merge, per image a segment of nangles*det_cap entries.
struct SweepScratch {
  pigo_det* merged;
  pigo_det* tmp;
  int32_t* tag;
  int32_t* seeds;
  uint8_t* flags;
  uint64_t *keys_in, *keys_out;
  int32_t *seg_begin, *seg_end, *n_merged;
  void* sort_temp;
  size_t sort_bytes;
};

// Chroma subsampling of image.YCbCrSubsampleRatio `sub` (0..5 = 444, 422, 420, 440, 411, 410) as shifts of the luma
// coordinates: 422/420 halve x, 411/410 quarter it; 420/440/410 halve y.
__host__ __device__ __forceinline__ int chroma_xshift(int sub) { return (sub == 1 || sub == 2) ? 1 : ((sub == 4 || sub == 5) ? 2 : 0); }
__host__ __device__ __forceinline__ int chroma_yshift(int sub) { return (sub == 2 || sub == 3 || sub == 5) ? 1 : 0; }

// One distinct source of a pigo_gray_images call, all pointers on the device.  Work item q of the call's kernel is the
// 16-pixel chunk q - first[k] (row-major, ceil(width/16) chunks per row) of the source k with first[k] <= q < first[k+1].
struct GraySrc {
  const uint8_t* plane[3];   // pigo_decoded.plane, at the rectangle's origin
  uint8_t* dst;              // the source's slot in the arena: height rows of width bytes
  int32_t format, sub, min_x, min_y, width, height, stride0, stride1;
};

// The formats gray_images_kernel<true> converts: Gray16, RGBA64, NRGBA64, CMYK and Paletted.
__host__ __device__ __forceinline__ bool decoded_wide(int format) { return format >= PIGO_DECODED_GRAY16; }

// Bytes per pixel of plane 0 of a pigo_decoded format.
__host__ __device__ __forceinline__ int decoded_bpp(int format) {
  switch (format) {
    case PIGO_DECODED_NRGBA: case PIGO_DECODED_RGBA: case PIGO_DECODED_CMYK: return 4;
    case PIGO_DECODED_RGBA64: case PIGO_DECODED_NRGBA64: return 8;
    case PIGO_DECODED_GRAY16: return 2;
    default: return 1;
  }
}

// ---- workspace -----------------------------------------------------------------------------------------
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return PIGO_OK;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    if (cudaMalloc(&p, want) != cudaSuccess) {
      cudaGetLastError();
      return set_err(PIGO_E_NOMEM, "cudaMalloc(%zu) failed", want);
    }
    cap = want;
    return PIGO_OK;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

constexpr int kMaxLanes = 4;

struct Workspace {
  cudaStream_t stream = nullptr;
  DevBuf frames, raw, counters, out, nout, plan, tiles, scratch_a, scratch_b, scratch_c, rot_tab, ptab;
  std::vector<int> ptab_sig;                   // geometry the cached per-scale offset tables were built for (empty = none)
  int rot_slot = -1;                           // table slot the cached rotated node table was built for (-1 = none)
  DevBuf longq[kMaxLanes];                     // the deep queue Q2 per pipeline lane
  DevBuf longq_sorted[kMaxLanes], longq_aux[kMaxLanes];   // Q2 in image order, and the sort's bins and keys (launch_deep_sort)
  cudaStream_t lane_stream[kMaxLanes] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t ev_fork = nullptr, ev_join[kMaxLanes] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t busy = nullptr;                  // last asynchronous use of this workspace (device-output calls)
  bool busy_valid = false;
  cudaStream_t active_stream = nullptr;        // stream of the call that currently borrows this workspace (see WsGuard)
  bool active_stream_set = false;
  cudaStream_t copy_stream = nullptr;          // H2D copies of host frames, one event per pipeline group
  cudaEvent_t group_copied = nullptr;          // streamed host frames: the current group's "all chunks copied" event (run_scan orders
                                               // the kernels behind the polling fused kernel after it)
  std::vector<cudaEvent_t> copy_events;
  cudaEvent_t copy_event(int k) {
    while ((int)copy_events.size() <= k) {
      cudaEvent_t e;
      if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return nullptr;
      copy_events.push_back(e);
    }
    return copy_events[k];
  }
  int ensure_lanes(int n) {
    if (!ev_fork && cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming) != cudaSuccess) return set_err(PIGO_E_CUDA, "event creation failed");
    for (int l = 0; l < n && n > 1; ++l) {
      if (!lane_stream[l] && cudaStreamCreateWithFlags(&lane_stream[l], cudaStreamNonBlocking) != cudaSuccess)
        return set_err(PIGO_E_CUDA, "stream creation failed");
      if (!ev_join[l] && cudaEventCreateWithFlags(&ev_join[l], cudaEventDisableTiming) != cudaSuccess)
        return set_err(PIGO_E_CUDA, "event creation failed");
    }
    return PIGO_OK;
  }
  // cached plan
  std::vector<ScaleEntry> plan_host;
  uint64_t wins = 0;
  int p_rows = -1, p_cols = -1, p_min = 0, p_max = 0;
  int pad_first_untiled = -1;  // which gather-block prefix is currently stored in the device copy of the plan
  double p_shift = 0, p_scale = 0;
  // mixed-size calls keep their own device plan / image table and rotated node tables, so that they never disturb the
  // cached uniform plan above (plan_host, pad_first_untiled, rot_slot + rot_tab, ptab_sig)
  DevBuf img_tab, img_rot;
  DevBuf gray_arena;                           // a sharded decoded call's converted images on this device (pigo_*_decoded_sharded)
  DevBuf sweep;                                // an angle sweep's merge scratch and per-face outputs (pigo_*_images_sweep)
  std::vector<int> img_rot_slots;                           // what img_rot was built for: one table per slot, in order (empty = nothing)
  int img_rot_len = 0, img_rot_min = 0;
  double img_rot_scale = 0;
  void* pinned = nullptr;
  size_t pinned_cap = 0;
  unsigned int* seq = nullptr;                 // pinned 1, 2, 3, ...: source of the ready-counter updates (host_stream)
  ~Workspace() {
    frames.release(); raw.release(); counters.release(); out.release(); nout.release(); plan.release();
    for (int l = 0; l < kMaxLanes; ++l) {
      longq[l].release(); longq_sorted[l].release(); longq_aux[l].release();
      if (lane_stream[l]) cudaStreamDestroy(lane_stream[l]);
      if (ev_join[l]) cudaEventDestroy(ev_join[l]);
    }
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (busy) cudaEventDestroy(busy);
    for (auto e : copy_events) cudaEventDestroy(e);
    if (copy_stream) cudaStreamDestroy(copy_stream);
    tiles.release(); scratch_a.release(); scratch_b.release(); scratch_c.release(); rot_tab.release(); ptab.release();
    img_tab.release(); img_rot.release(); gray_arena.release(); sweep.release();
    if (pinned) cudaFreeHost(pinned);
    if (seq) cudaFreeHost(seq);
    if (stream) cudaStreamDestroy(stream);
  }
};

struct WorkspacePool {
  std::mutex mu;
  std::vector<Workspace*> free_list;
  Workspace* acquire() {
    {
      std::lock_guard<std::mutex> g(mu);
      if (!free_list.empty()) { Workspace* w = free_list.back(); free_list.pop_back(); return w; }
    }
    Workspace* w = new Workspace();
    if (cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking) != cudaSuccess) { delete w; return nullptr; }
    return w;
  }
  void release(Workspace* w) { std::lock_guard<std::mutex> g(mu); free_list.push_back(w); }
  ~WorkspacePool() { for (auto* w : free_list) delete w; }
};

// Borrow of a workspace for one API call.  Whatever way the call ends (device-output calls return while their kernels
// are still running; an error may return in the middle of queued work), the last stream the workspace was used on is
// marked with the `busy` event before the workspace goes back to the pool, and the next borrower waits on it (ws_enter).
struct WsGuard {
  WorkspacePool& pool; Workspace* w;
  WsGuard(WorkspacePool& p) : pool(p), w(p.acquire()) {}
  ~WsGuard() {
    if (!w) return;
    if (w->active_stream_set) {
      if (w->busy && cudaEventRecord(w->busy, w->active_stream) == cudaSuccess) w->busy_valid = true; else cudaGetLastError();
      w->active_stream_set = false;
    }
    pool.release(w);
  }
};


// ---- devices -------------------------------------------------------------------------------------------
// The library serves up to kMaxDevices GPUs from one process (SURVEY.md section 8e: single process, frames sharded over the
// devices of a mask).  Handles keep the parsed tables on the host and build one device replica per GPU on first use.
constexpr int kMaxDevices = 16;
int use_device(int dev);        // validates (sm_90) + cudaSetDevice on the calling thread
int default_device();           // device of the non-sharded entry points (pigo_init, implicit device 0)
int device_sms(int dev);
std::vector<int> shard_devices();   // devices of the mask given to pigo_init_devices, ascending

struct FaceReplica {            // device copy of one face cascade
  int device = 0, num_sms = 132;
  DevBuf codes, preds, thresh, tiled_tab, block_tab;
  FaceTables tab{};
  WorkspacePool pool;
  ~FaceReplica() { cudaSetDevice(device); codes.release(); preds.release(); thresh.release(); tiled_tab.release(); block_tab.release(); }
};
struct PuplocReplica {
  int device = 0, num_sms = 132;
  DevBuf codes, preds;
  PuplocTables tab{};
  WorkspacePool pool;
  ~PuplocReplica() { cudaSetDevice(device); codes.release(); preds.release(); }
};

}  // namespace pigo

struct pigo_cascade {
  uint32_t depth = 0, ntrees = 0, leaves = 0;
  std::vector<int8_t> h_codes;          // reference layout (core/pigo.go:79-86), see FaceTables
  std::vector<float> h_preds, h_thr;
  std::mutex mu;
  pigo::FaceReplica* rep[pigo::kMaxDevices] = {};
  ~pigo_cascade() { for (auto* r : rep) delete r; }
};

struct pigo_puploc {
  uint32_t stages = 0, trees = 0, depth = 0, leaves = 0;
  float scales = 0.f;
  std::vector<int8_t> h_codes;
  std::vector<float> h_preds;
  std::mutex mu;
  pigo::PuplocReplica* rep[pigo::kMaxDevices] = {};
  ~pigo_puploc() { for (auto* r : rep) delete r; }
};


namespace pigo {
// kernels / drivers implemented in the other .cu files
void launch_scan_gather(const ScanArgs& A, int grid, int max_scale, cudaStream_t st);
void launch_scan_tiled(const TiledArgs& A, const TileMaps& TM, int grid, int threads, size_t smem, int ni, cudaStream_t st);
int tiled_max_threads(int ni);
void launch_ptab_build(const FaceTables& T, const ScaleEntry* plan, const TiledArgs& A, int first_untiled, uint8_t* out, int grid, cudaStream_t st);
void launch_gray(const uint8_t* rgba, size_t npix, uint8_t* gray, int grid, cudaStream_t st);
void launch_ycbcr(const uint8_t* y, const uint8_t* cb, const uint8_t* cr, int y_stride, int c_stride, int subsample, int min_x, int min_y,
                  int width, int height, uint8_t* nrgba, uint8_t* gray, int grid, cudaStream_t st);
// wide: the sources are all Gray16, RGBA64, NRGBA64, CMYK or Paletted (else all YCbCr, NRGBA, RGBA or Gray).
void launch_gray_images(const GraySrc* src, const uint64_t* first, int nsrc, uint64_t total, bool wide, int grid, cudaStream_t st);
void launch_scan_gather2(const TiledArgs& A, int grid, size_t smem, cudaStream_t st);
int gather2_ctas_per_sm(size_t smem, int ng, bool rot, bool img = false);
void launch_rot_table(const FaceTables& T, const ScaleEntry* plan, int nscales, int slot, RotNode* out, int grid, cudaStream_t st);
void launch_deep(const ScanArgs& A, unsigned long long* counter, int num_sms, int group, bool ordered, cudaStream_t st);
size_t deep_sort_aux_bytes(int rows, int cols, int nframes, size_t qcap);
int launch_deep_sort(const ScanArgs& A, int rows, int cols, DeepItem* sorted, void* aux, int num_sms, cudaStream_t st);
void launch_deep_smem(const ScanArgs& A, unsigned long long* counter, const uint8_t* tab_tiled, int num_sms, int threads, int group, int t_lo, int k,
                      cudaStream_t st);
int gather_max_ctas_per_sm(int depth, bool rot);
void launch_finalize(const RawDet* raw, const int32_t* raw_count, int cap, const ScaleEntry* plan, int nscales, pigo_det* out,
                     int32_t* n_out, int nframes, cudaStream_t st);
void launch_finalize_images(const RawDet* raw, const int32_t* raw_count, int cap, const ScaleEntry* plan, const ImageDesc* images,
                            pigo_det* out, int32_t* n_out, int nimages, cudaStream_t st);
void launch_cluster(pigo_det* dets, const int32_t* n_in, int cap, double thr, pigo_det* tmp, uint8_t* flags, int32_t* seeds,
                    pigo_det* out, int out_cap, int32_t* n_out, int nframes, cudaStream_t st);
size_t sweep_sort_bytes(int nimages, int seg_cap);
int launch_sweep_merge(const pigo_det* raw, const int32_t* raw_count, int nimages, int nangles, int det_cap, double thr, const SweepScratch& S,
                       const int32_t* slot_of, pigo_det* out, int out_cap, int32_t* n_out, int32_t* out_tag, int32_t* out_rot, cudaStream_t st);
void launch_puploc(const PuplocTables& T, const pigo_point* seeds, int nseeds, const float* randoms, uint64_t rng_seed,
                   const uint8_t* frames, const int32_t* seed_frame, size_t frame_stride, int rows, int cols, int dim, int rot_slot,
                   const uint8_t* flipv, pigo_point* out, const ImageDesc* images, cudaStream_t st);
int launch_puploc_pairs(const PupWork& W, unsigned int* counter, int num_sms, cudaStream_t st);
void launch_eye_seeds(const pigo_det* clusters, const int32_t* ncl, int cl_cap, int nframes, int face_cap, int stride, int min_face,
                      int eye_perturbs, pigo_det* faces, int32_t* nfaces, pigo_point* seeds, cudaStream_t st);
void launch_landmark_seeds(const pigo_point* points, pigo_point* seeds, int nslots, int stride, int ncalls, int flp_perturbs, cudaStream_t st);
int build_tiled_tables(const FaceTables& tab, const std::vector<int8_t>& codes, const std::vector<float>& preds,
                       const std::vector<float>& thr, DevBuf& out);
int build_block_tables(const FaceTables& tab, const std::vector<int8_t>& codes, const std::vector<float>& preds,
                       const std::vector<float>& thr, DevBuf& out);
int describe_plan(const std::vector<ScaleEntry>& plan, uint64_t wins, int ntrees, int batch_frames, char* buf, size_t cap);
int run_scan(FaceReplica* c, Workspace* w, int lane, ScanArgs& A, unsigned long long* d_work, cudaStream_t st, int num_sms);
// Whether a scan of cascade c runs on the block/deep kernels rather than the universal gather kernel (scan_driver.cu).
bool block_path(const FaceReplica* c, bool rot, int max_scale, size_t rot_bytes);
struct ImagesSchedule {
  int gb_shift;       // log2 of the gather block edge in windows
  int gather_limit;   // trees a window walks in the gather-v2 kernel before it goes to the deep kernel
  int deep_group;     // lanes per window in the deep kernel
  bool deep_ordered;  // the deep kernel takes its queue in image order (launch_deep_sort)
};
ImagesSchedule images_schedule(uint64_t call_windows, bool rot, int large_limit);
int run_scan_images(FaceReplica* c, Workspace* w, ScanArgs& A, const ImagesSchedule& P, uint32_t group_blocks, uint64_t group_windows,
                    int max_rows, int max_cols, unsigned long long* d_work, cudaStream_t st, int num_sms);
FaceReplica* face_replica(pigo_cascade* c, int dev, int* rc);
PuplocReplica* puploc_replica(pigo_puploc* p, int dev, int* rc);
}  // namespace pigo
