// api.cu -- the C-ABI of libpigo_b200.so (include/pigo_b200.h): cascade parsing, scan planning on the
// host (float64 ladder arithmetic exactly as core/pigo.go:226-231,:255), scratch management and the
// kernel sequence of each entry point.  No CPU compute path exists: without a device the calls fail.
#include <cuda_runtime.h>

#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <algorithm>
#include <map>
#include <numeric>
#include <string>
#include <thread>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "host.h"

namespace pigo {

thread_local std::string g_err;
std::atomic<long long> g_launches{0};
static std::atomic<int> g_device{-1};
Options g_opt;

// ---- per-kernel event timing --------------------------------------------------------------------------------
struct TimingSlot {
  std::vector<cudaEvent_t> ev;  // begin/end pairs
  size_t used = 0;
};
static TimingSlot g_tslot[T_NSLOTS];
static std::mutex g_tmu;
static const char* kSlotNames[T_NSLOTS] = {"tiled", "gather", "deep", "finalize", "cluster", "puploc", "gray", "seeds", "rottab", "ycbcr", "gray_images", "merge"};

void timing_reset() {
  std::lock_guard<std::mutex> g(g_tmu);
  for (auto& s : g_tslot) s.used = 0;
}
static void timing_mark(int slot, cudaStream_t st) {
  if (!g_opt.timing.load()) return;
  std::lock_guard<std::mutex> g(g_tmu);
  TimingSlot& s = g_tslot[slot];
  if (s.used >= 1u << 16) return;
  if (s.used == s.ev.size()) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) { cudaGetLastError(); return; }
    s.ev.push_back(e);
  }
  cudaEventRecord(s.ev[s.used++], st);
}
void timing_begin(int slot, cudaStream_t st) { timing_mark(slot, st); }
void timing_end(int slot, cudaStream_t st) { timing_mark(slot, st); }
long long timing_query(const std::string& key) {
  std::lock_guard<std::mutex> g(g_tmu);
  for (int i = 0; i < T_NSLOTS; ++i) {
    const std::string base = std::string("t_") + kSlotNames[i];
    TimingSlot& s = g_tslot[i];
    if (key == base + "_n") return (long long)(s.used / 2);
    if (key == base + "_ns") {
      double total = 0;
      for (size_t k = 0; k + 1 < s.used; k += 2) {
        float ms = 0;
        if (cudaEventSynchronize(s.ev[k + 1]) != cudaSuccess || cudaEventElapsedTime(&ms, s.ev[k], s.ev[k + 1]) != cudaSuccess) {
          cudaGetLastError();
          return -2;
        }
        total += (double)ms * 1e6;
      }
      return (long long)total;
    }
  }
  return -1;
}

// A workspace can be handed to another caller (another thread / stream) while the asynchronous work of its previous
// user is still running on that user's stream: order every new user behind the last recorded use.
static bool stream_capturing(cudaStream_t st) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) { cudaGetLastError(); return false; }
  return cs == cudaStreamCaptureStatusActive;
}

static int ws_enter(Workspace* w, cudaStream_t st) {
  if (!w->busy && cudaEventCreateWithFlags(&w->busy, cudaEventDisableTiming) != cudaSuccess) return set_err(PIGO_E_CUDA, "event creation failed");
  if (stream_capturing(st)) {   // CUDA-graph capture of a device-output call: no events cross the capture boundary (see scan_batch_on)
    if (w->busy_valid) cudaEventSynchronize(w->busy);
    w->busy_valid = false;
    w->active_stream_set = false;
    return PIGO_OK;
  }
  if (w->busy_valid && cudaStreamWaitEvent(st, w->busy, 0) != cudaSuccess) return set_err(PIGO_E_CUDA, "cudaStreamWaitEvent failed");
  w->active_stream = st; w->active_stream_set = true;   // WsGuard records `busy` on it when the call ends, however it ends
  return PIGO_OK;
}
static int ws_leave_async(Workspace* w, cudaStream_t st) {
  if (stream_capturing(st)) { w->active_stream_set = false; return PIGO_OK; }
  if (cudaEventRecord(w->busy, st) != cudaSuccess) return set_err(PIGO_E_CUDA, "cudaEventRecord failed");
  w->busy_valid = true;
  w->active_stream_set = false;
  return PIGO_OK;
}

// One call's borrow of a workspace of `pool`, used as that Workspace*.  st = the caller's stream (or, stream_ NULL, the
// workspace's own), already ordered behind the workspace's last asynchronous use (ws_enter); rc = the borrow's result.
struct Borrow {
  WsGuard guard;
  Workspace* w = nullptr;
  cudaStream_t st = nullptr;
  int rc = PIGO_OK;
  Borrow(WorkspacePool& pool, void* stream_) : guard(pool), w(guard.w) {
    if (!w) { rc = set_err(PIGO_E_CUDA, "could not create a CUDA stream"); return; }
    st = stream_ ? (cudaStream_t)stream_ : w->stream;
    rc = ws_enter(w, st);
  }
  Workspace* operator->() const { return w; }
  operator Workspace*() const { return w; }
  void keep() { guard.w = nullptr; }   // the workspace never goes back to the pool (it belongs to a captured graph)
};

void raise_dyn_smem(const void* fn, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, int> granted;   // (device, kernel) -> the attribute's value
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return; }
  std::lock_guard<std::mutex> g(mu);
  int& cur = granted[{dev, fn}];
  if (bytes <= cur) return;
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess) cur = bytes;
  else cudaGetLastError();   // the launch that needs it fails and reports
}

int set_err(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

#define CUDA_TRY(expr)                                                                              \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) return set_err(PIGO_E_CUDA, "%s failed: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

// ---- devices ------------------------------------------------------------------------------------------------
static std::mutex g_dev_mu;
static int g_sms[kMaxDevices] = {};          // 0 = not validated yet
static std::atomic<unsigned> g_mask{0};

int device_sms(int dev) { return (dev >= 0 && dev < kMaxDevices && g_sms[dev] > 0) ? g_sms[dev] : 132; }

int use_device(int dev) {
  if (dev < 0 || dev >= kMaxDevices) return set_err(PIGO_E_INVALID, "device %d out of range", dev);
  if (g_sms[dev] == 0) {
    std::lock_guard<std::mutex> g(g_dev_mu);
    if (g_sms[dev] == 0) {
      int n = 0;
      cudaError_t e = cudaGetDeviceCount(&n);
      if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        return set_err(PIGO_E_NODEVICE, "no CUDA device visible (%s); libpigo_b200 has no CPU fallback",
                       e == cudaSuccess ? "count=0" : cudaGetErrorString(e));
      }
      if (dev >= n) return set_err(PIGO_E_INVALID, "device %d out of range (0..%d)", dev, n - 1);
      cudaDeviceProp prop;
      CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
      if (prop.major != 9 || prop.minor != 0)
        return set_err(PIGO_E_NODEVICE, "device %d is sm_%d%d; this library contains sm_90a code only", dev, prop.major, prop.minor);
      g_sms[dev] = prop.multiProcessorCount;
    }
  }
  CUDA_TRY(cudaSetDevice(dev));
  return PIGO_OK;
}

int default_device() {
  int dev = g_device.load();
  if (dev < 0) {
    if (pigo_init(0) != PIGO_OK) return -1;
    dev = g_device.load();
  }
  return dev;
}

std::vector<int> shard_devices() {
  std::vector<int> v;
  const unsigned m = g_mask.load();
  for (int d = 0; d < kMaxDevices; ++d)
    if (m & (1u << d)) v.push_back(d);
  return v;
}

static int ensure_device() {
  const int dev = default_device();
  if (dev < 0) return PIGO_E_NODEVICE;   // message set by pigo_init
  return use_device(dev);
}

// Device replicas of the handles: built on first use on a device, from the host copy of the parsed tables.
FaceReplica* face_replica(pigo_cascade* c, int dev, int* rc) {
  *rc = PIGO_OK;
  if (dev < 0 || dev >= kMaxDevices) { *rc = set_err(PIGO_E_INVALID, "device %d out of range", dev); return nullptr; }
  std::lock_guard<std::mutex> g(c->mu);
  if (c->rep[dev]) return c->rep[dev];
  if ((*rc = use_device(dev))) return nullptr;
  FaceReplica* r = new FaceReplica();
  r->device = dev; r->num_sms = device_sms(dev);
  if ((*rc = r->codes.reserve(c->h_codes.size())) || (*rc = r->preds.reserve(c->h_preds.size() * 4)) ||
      (*rc = r->thresh.reserve(c->h_thr.size() * 4))) { delete r; return nullptr; }
  cudaMemcpy(r->codes.p, c->h_codes.data(), c->h_codes.size(), cudaMemcpyHostToDevice);
  cudaMemcpy(r->preds.p, c->h_preds.data(), c->h_preds.size() * 4, cudaMemcpyHostToDevice);
  cudaError_t e = cudaMemcpy(r->thresh.p, c->h_thr.data(), c->h_thr.size() * 4, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { delete r; *rc = set_err(PIGO_E_CUDA, "table upload failed: %s", cudaGetErrorString(e)); return nullptr; }
  r->tab.codes = (const int8_t*)r->codes.p; r->tab.preds = (const float*)r->preds.p; r->tab.thresh = (const float*)r->thresh.p;
  r->tab.depth = (int)c->depth; r->tab.ntrees = (int)c->ntrees; r->tab.leaves = (int)c->leaves;
  if ((*rc = build_tiled_tables(r->tab, c->h_codes, c->h_preds, c->h_thr, r->tiled_tab))) { delete r; return nullptr; }
  if ((*rc = build_block_tables(r->tab, c->h_codes, c->h_preds, c->h_thr, r->block_tab))) { delete r; return nullptr; }
  r->tab.blocks = (const uint8_t*)r->block_tab.p;
  c->rep[dev] = r;
  return r;
}

PuplocReplica* puploc_replica(pigo_puploc* p, int dev, int* rc) {
  *rc = PIGO_OK;
  if (dev < 0 || dev >= kMaxDevices) { *rc = set_err(PIGO_E_INVALID, "device %d out of range", dev); return nullptr; }
  std::lock_guard<std::mutex> g(p->mu);
  if (p->rep[dev]) return p->rep[dev];
  if ((*rc = use_device(dev))) return nullptr;
  PuplocReplica* r = new PuplocReplica();
  r->device = dev; r->num_sms = device_sms(dev);
  // device layout of the codes: one pad word in front of every tree (see PuplocTables)
  const size_t nt = (size_t)p->stages * p->trees, ncode = 4 * (size_t)p->leaves - 4;
  std::vector<int8_t> padded(nt * (ncode + 4) + 16, 0);
  for (size_t t = 0; t < nt; ++t) memcpy(padded.data() + t * (ncode + 4) + 4, p->h_codes.data() + t * ncode, ncode);
  if ((*rc = r->codes.reserve(padded.size())) || (*rc = r->preds.reserve(p->h_preds.size() * 4))) { delete r; return nullptr; }
  cudaMemcpy(r->codes.p, padded.data(), padded.size(), cudaMemcpyHostToDevice);
  cudaError_t e = cudaMemcpy(r->preds.p, p->h_preds.data(), p->h_preds.size() * 4, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { delete r; *rc = set_err(PIGO_E_CUDA, "table upload failed: %s", cudaGetErrorString(e)); return nullptr; }
  r->tab.codes = (const int8_t*)r->codes.p; r->tab.preds = (const float*)r->preds.p;
  r->tab.stages = (int)p->stages; r->tab.trees = (int)p->trees; r->tab.depth = (int)p->depth; r->tab.leaves = (int)p->leaves;
  r->tab.scales = p->scales;
  p->rep[dev] = r;
  return r;
}

// ---- scale ladder / grid: core/pigo.go:226-231,:255 ---------------------------------------------------
static int build_plan(int rows, int cols, int min_size, int max_size, double shift, double scale_factor,
                      std::vector<ScaleEntry>& plan, uint64_t& total) {
  plan.clear();
  total = 0;
  long long scale = min_size;
  int guard = 0;
  while (scale <= max_size) {
    if (++guard > (1 << 16)) return set_err(PIGO_E_INVALID, "scale ladder longer than 65536 entries");
    if (scale < 0) return set_err(PIGO_E_INVALID, "negative window size %lld (the reference indexes out of bounds)", scale);
    {
      // scale == 0 is well defined in the reference: step 1, offset 1, every node compares a pixel with itself
      const long long step = (long long)std::fmax(shift * (double)scale, 1.0);  // :227
      const long long off = scale / 2 + 1;                                      // :228
      long long nr = 0, nc = 0;
      if (rows - off >= off) nr = (rows - off - off) / step + 1;                // :230
      if (cols - off >= off) nc = (cols - off - off) / step + 1;                // :231
      if (nr > 0 && nc > 0) {
        ScaleEntry e;
        e.s = (int)scale; e.step = (int)step; e.off = (int)off; e.nrows = (int)nr; e.ncols = (int)nc;
        e.wbase = (uint32_t)total; e.nwin = (uint32_t)(nr * nc); e.pad = 0;
        total += (uint64_t)(nr * nc);
        if (total > 0x7fffffffull) return set_err(PIGO_E_INVALID, "more than 2^31 windows per frame");
        plan.push_back(e);
      }
    }
    const double next = (double)scale + std::fmax(2.0, ((double)scale * scale_factor) - (double)scale);  // :255
    if (!(next < 9.0e15)) break;
    scale = (long long)next;
  }
  return PIGO_OK;
}

}  // namespace pigo

using namespace pigo;

// Frames per pipeline group of one batch call.  Resident frames: uniform groups of 128 (fewest kernel tails; the deferred
// queues of a group stay bounded).  Host frames: 64, with or without in-kernel waiting (host_stream): with it the fused kernel
// of a group is copy-bound and ends when the group's last chunk arrives, and the group's tail kernels then overlap the next
// group's copy.  When PCIe and the scan run at about the same rate, a step costs about  [time the scan idles behind the first copy chunks] + [scan]  and also at least
// [copy] + [tail kernels of the last group]; stream_taper = 1 (128, then half of the rest) shortens the second term but
// its small groups lengthen the first; stream_taper = 2 (1/8, 1/4, 3/8, 3/16, 1/16 of the batch)
// tries to shorten both.
static std::vector<int> group_schedule(int nframes, bool resident, bool streamed) {
  std::vector<int> g;
  long long sub = g_opt.sub_batch.load();
  const long long taper = g_opt.stream_taper.load();
  if (sub <= 0 && streamed && taper == 1) {
    for (int left = nframes; left > 0;) {
      const int n = std::min(left, std::min(128, std::max(32, (left + 1) / 2)));
      g.push_back(n);
      left -= n;
    }
    return g;
  }
  if (sub <= 0 && streamed && taper == 2 && nframes >= 64) {
    static const int sixteenths[5] = {2, 4, 6, 3, 1};
    int left = nframes;
    for (int k = 0; k < 5 && left > 0; ++k) {
      const int n = k == 4 ? left : std::min(left, std::min(128, std::max(8, nframes * sixteenths[k] / 16)));
      g.push_back(n);
      left -= n;
    }
    if (left > 0) g.push_back(left);
    return g;
  }
  const bool auto_sub = sub <= 0;
  if (sub <= 0) sub = resident ? 128 : 64;   // streamed host frames: 64 (a group's tail kernels overlap the next group's chunks)
  for (int left = nframes; left > 0; left -= (int)sub) g.push_back((int)std::min<long long>(sub, left));
  if (auto_sub && streamed && taper == 3 && g.size() >= 2 && g.back() >= 32) {
    // the step ends one group's tail kernels after the last chunk: halve the LAST group only
    const int n = g.back();
    g.back() = n - n / 2;
    g.push_back(n / 2);
  }
  return g;
}

// Host outputs of a scan: the counts, then only the used prefix of every frame's slice of d_out ([nframes][cap]) and, given
// `tags`, of the per-slot int32 d_tags ([nframes][cap]); PIGO_E_CAP if a frame has more detections than cap_per_frame.
// The counts are the lead + nframes int32 at d_cnt, copied at once: the frame counts come last, after `lead` others (an
// angle sweep's raw-list counts), and with lead > 0 all of them go to cnt and n_out receives the frame counts.
static int copy_results_to_host(const pigo_det* d_out, const int32_t* d_cnt, int cap, int nframes, pigo_det* out, int cap_per_frame,
                                int* n_out, cudaStream_t st, const int32_t* d_tags = nullptr, int32_t* tags = nullptr, int lead = 0,
                                int32_t* cnt = nullptr) {
  CUDA_TRY(cudaMemcpyAsync(lead > 0 ? cnt : n_out, d_cnt, (size_t)(lead + nframes) * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (lead > 0) std::copy(cnt + lead, cnt + lead + nframes, n_out);
  int need_more = 0;
  size_t max_n = 0;
  for (int f = 0; f < nframes; ++f) {
    if (n_out[f] > cap_per_frame) need_more = 1;
    size_t k = (size_t)std::min(n_out[f], cap_per_frame);
    if (k > max_n) max_n = k;
  }
  if (cap_per_frame > 0 && max_n > 0) {
    CUDA_TRY(cudaMemcpy2DAsync(out, (size_t)cap_per_frame * sizeof(pigo_det), d_out, (size_t)cap * sizeof(pigo_det),
                               max_n * sizeof(pigo_det), nframes, cudaMemcpyDeviceToHost, st));
    if (tags)
      CUDA_TRY(cudaMemcpy2DAsync(tags, (size_t)cap_per_frame * 4, d_tags, (size_t)cap * 4, max_n * 4, nframes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
  }
  if (need_more) return set_err(PIGO_E_CAP, "output capacity %d per frame too small", cap_per_frame);
  return PIGO_OK;
}

// Bytes of a host image the reference may index, (rows-1)*dim + cols (core/pigo.go:126 with Dim >= Cols): never read more
// than that from the caller's buffer.
static size_t readable_bytes(int rows, int cols, int dim) { return rows > 0 ? (size_t)(rows - 1) * dim + cols : 0; }

// Table slot of a rotated scan, core/pigo.go:159,:232-236: angle > 0 rotates, angle > 1 is clamped to 1, and angle <= 0
// or NaN scans unrotated (-1).
static int rot_slot_of(double angle) { return angle > 0.0 ? (int)(32.0 * (angle > 1.0 ? 1.0 : angle)) : -1; }

// ---- RunCascade on one device -----------------------------------------------------------------------------------
static int scan_batch_on(pigo_cascade* c, int dev, const uint8_t* frames, int nframes, size_t frame_stride, int rows, int cols, int dim,
                         int min_size, int max_size, double shift_factor, double scale_factor, double angle, pigo_det* out,
                         int cap_per_frame, int* n_out, unsigned flags, void* stream_, uint8_t* host_frames_dst = nullptr) {
  // host_frames_dst (optional, host frames only): device buffer of nframes * round256(rows*dim) bytes that receives the
  // frames instead of the call's own scratch -- the pipeline keeps them for the pupil / landmark stages that follow.
  int rc = PIGO_OK;
  FaceReplica* R = face_replica(c, dev, &rc);
  if (!R) return rc;
  if ((rc = use_device(dev))) return rc;
  const bool frames_dev = flags & PIGO_FRAMES_DEVICE, out_dev = flags & PIGO_OUT_DEVICE;

  Borrow w(R->pool, stream_);
  if (w.rc) return w.rc;
  cudaStream_t st = w.st;
  auto plan_cached = [&] {
    return w->p_rows == rows && w->p_cols == cols && w->p_min == min_size && w->p_max == max_size && w->p_shift == shift_factor &&
           w->p_scale == scale_factor;
  };
  // CUDA-graph capture (device frames + device outputs on the caller's capturing stream, after one un-captured warm-up call
  // with the same arguments): the captured kernels keep using this workspace's scratch on every replay, so the workspace
  // is taken out of the pool for good -- it belongs to the graph from now on.
  const bool capturing = stream_capturing(st);
  if (capturing) {
    if (!(flags & PIGO_FRAMES_DEVICE) || !(flags & PIGO_OUT_DEVICE)) return set_err(PIGO_E_INVALID, "stream capture needs device frames and device outputs");
    if (!plan_cached())
      return set_err(PIGO_E_INVALID, "stream capture: run the same call once outside the capture first (the plan upload synchronises)");
    w.keep();
  }

  // plan (cached per workspace)
  if (!plan_cached()) {
    rc = build_plan(rows, cols, min_size, max_size, shift_factor, scale_factor, w->plan_host, w->wins);
    if (rc) { w->p_rows = -1; return rc; }
    if ((rc = w->plan.reserve((w->plan_host.size() + 1) * sizeof(ScaleEntry)))) return rc;
    if (!w->plan_host.empty())
      CUDA_TRY(cudaMemcpyAsync(w->plan.p, w->plan_host.data(), w->plan_host.size() * sizeof(ScaleEntry), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));  // plan_host may be rebuilt by the next call before the copy ran
    w->pad_first_untiled = -1;
    w->rot_slot = -1;
    w->ptab_sig.clear();
    w->p_rows = rows; w->p_cols = cols; w->p_min = min_size; w->p_max = max_size; w->p_shift = shift_factor; w->p_scale = scale_factor;
  }
  const int nscales = (int)w->plan_host.size();
  const int cap = cap_per_frame > 0 ? cap_per_frame : 1;

  // device buffers.  A host frame is only guaranteed to hold its readable bytes.
  const uint8_t* d_frames = frames;
  const size_t frame_bytes = (size_t)rows * dim;
  const size_t frame_min = readable_bytes(rows, cols, dim);
  size_t d_stride = frame_stride;
  uint8_t* d_frames_w = host_frames_dst;
  if (!frames_dev) {
    d_stride = (frame_bytes + 255) & ~(size_t)255;
    if (!d_frames_w) {
      if ((rc = w->frames.reserve(d_stride * nframes + 256))) return rc;
      d_frames_w = (uint8_t*)w->frames.p;
    }
    d_frames = d_frames_w;
  }
  pigo_det* d_out = out;
  int32_t* d_nout = n_out;
  if (!out_dev) {
    if ((rc = w->out.reserve((size_t)nframes * cap * sizeof(pigo_det)))) return rc;
    if ((rc = w->nout.reserve((size_t)nframes * sizeof(int32_t)))) return rc;
    d_out = (pigo_det*)w->out.p;
    d_nout = (int32_t*)w->nout.p;
  }
  if ((rc = w->raw.reserve((size_t)nframes * cap * sizeof(RawDet)))) return rc;
  bool zero_out_staging = !out_dev;   // slots past a frame's count travel back to the host too: keep them defined (zero)

  // Sub-batch pipeline: the batch is cut into groups of frames (group_schedule) that alternate between `lanes` internal
  // streams.  (1) The deferred queue (Q2) of a group is bounded and consumed soon after they are filled;
  // (2) with host frames, the H2D copy of group k+1 overlaps the scan of group k.
  const int rot_slot = rot_slot_of(angle);
  // Host frames, streamed: the copy stream moves the frames up chunk by chunk and bumps a ready counter after each chunk;
  // the fused kernel (whose tile / block order is frame-major) waits in-kernel for the frame it is about to touch, so the
  // scan runs right behind the copy at frame granularity instead of group granularity.  Only the fused kernel polls: the
  // kernels queued behind it start after every frame of the group has arrived (stream wait on the group's last chunk).
  const bool fused_path = rot_slot < 0 && c->depth == 6 && g_opt.scan_mode.load() == 0 && g_opt.tile_warps.load() > 0;
  const bool streamed = !frames_dev && g_opt.host_stream.load() != 0 && fused_path;
  const std::vector<int> groups = group_schedule(nframes, frames_dev, streamed);
  const int nsub = (int)groups.size();
  int lanes = (int)std::min<long long>(std::max<long long>(1, g_opt.lanes.load()), kMaxLanes);
  if (nsub == 1 || rot_slot >= 0) lanes = 1;   // (the rotated node table is built once, on the first group's stream)
  if ((rc = w->ensure_lanes(lanes))) return rc;

  // counters: [0..nframes) raw counts | 8 x u64 work counters per sub-batch
  const size_t work_off = ((size_t)nframes * 4 + 15) & ~(size_t)15;
  const size_t cnt_bytes = work_off + (size_t)nsub * 64 + 128;
  if ((rc = w->counters.reserve(cnt_bytes))) return rc;
  CUDA_TRY(cudaMemsetAsync(w->counters.p, 0, cnt_bytes, st));
  int32_t* d_rawcount = (int32_t*)w->counters.p;
  unsigned long long* d_work = (unsigned long long*)((char*)w->counters.p + work_off);
  unsigned int* d_ready = (unsigned int*)((char*)w->counters.p + work_off + (size_t)nsub * 64 + 64);
  if (streamed && !w->seq) {
    CUDA_TRY(cudaHostAlloc((void**)&w->seq, 65536 * sizeof(unsigned int), cudaHostAllocDefault));
    for (unsigned i = 0; i < 65536; ++i) w->seq[i] = i + 1;
  }

  if (lanes > 1 || !frames_dev) {
    CUDA_TRY(cudaEventRecord(w->ev_fork, st));   // everything queued on `st` so far (previous results, memset) comes first
    for (int l = 0; l < lanes && lanes > 1; ++l) CUDA_TRY(cudaStreamWaitEvent(w->lane_stream[l], w->ev_fork, 0));
    if (!frames_dev) {
      if (!w->copy_stream && cudaStreamCreateWithFlags(&w->copy_stream, cudaStreamNonBlocking) != cudaSuccess)
        return set_err(PIGO_E_CUDA, "stream creation failed");
      CUDA_TRY(cudaStreamWaitEvent(w->copy_stream, w->ev_fork, 0));
    }
  }
  int f0 = 0;
  for (int k = 0; k < nsub; ++k) {
    const int nf = groups[k];
    const int lane = k % lanes;
    cudaStream_t ls = lanes > 1 ? w->lane_stream[lane] : st;
    cudaEvent_t ev_group = nullptr;
    if (!frames_dev) {
      // the copies run on the copy stream (pinned source memory) and overlap the scan
      cudaStream_t cs = w->copy_stream;
      const long long chunk = streamed ? std::max<long long>(1, g_opt.copy_chunk.load()) : nf;
      for (int c0 = 0; c0 < nf; c0 += (int)chunk) {
        const int cn = (int)std::min<long long>(chunk, nf - c0);
        uint8_t* dst = d_frames_w + (size_t)(f0 + c0) * d_stride;
        const uint8_t* src = frames + (size_t)(f0 + c0) * frame_stride;
        const bool last = f0 + c0 + cn == nframes;   // only the batch's last frame may be short; the others have a successor behind them
        if (frame_stride == d_stride || cn == 1) {
          CUDA_TRY(cudaMemcpyAsync(dst, src, d_stride * (size_t)(cn - 1) + (last ? frame_min : frame_bytes), cudaMemcpyHostToDevice, cs));
        } else {
          CUDA_TRY(cudaMemcpy2DAsync(dst, d_stride, src, frame_stride, frame_min, cn, cudaMemcpyHostToDevice, cs));
        }
        if (streamed) CUDA_TRY(cudaMemcpyAsync(d_ready, w->seq + (f0 + c0 + cn - 1), sizeof(unsigned int), cudaMemcpyHostToDevice, cs));
      }
      ev_group = w->copy_event(k);
      if (!ev_group) return set_err(PIGO_E_CUDA, "event creation failed");
      CUDA_TRY(cudaEventRecord(ev_group, cs));
      if (!streamed) CUDA_TRY(cudaStreamWaitEvent(ls, ev_group, 0));
    }
    if (nscales > 0 && c->ntrees > 0) {
      ScanArgs A{};
      A.tab = R->tab;
      A.frames = d_frames + (size_t)f0 * d_stride; A.frame_stride = d_stride; A.nframes = nf; A.rows = rows; A.cols = cols; A.dim = dim;
      A.plan = (const ScaleEntry*)w->plan.p; A.nscales = nscales; A.wins_per_frame = (uint32_t)w->wins;
      A.rot_slot = rot_slot; A.rot_tab = nullptr; A.batch_frames = nframes;
      A.raw = (RawDet*)w->raw.p + (size_t)f0 * cap; A.raw_count = d_rawcount + f0; A.cap = cap;
      A.frame_base = (uint32_t)f0; A.ready = streamed ? d_ready : nullptr;
      w->group_copied = streamed ? ev_group : nullptr;
      rc = run_scan(R, w, lane, A, d_work + 8 * (size_t)k, ls, R->num_sms);
      if (rc) return rc;
    }
    if (streamed && !(nscales > 0 && c->ntrees > 0)) CUDA_TRY(cudaStreamWaitEvent(ls, ev_group, 0));   // nothing polled: still order the stream behind the copy
    f0 += nf;
  }
  if (lanes > 1) {
    for (int l = 0; l < lanes; ++l) {
      CUDA_TRY(cudaEventRecord(w->ev_join[l], w->lane_stream[l]));
      CUDA_TRY(cudaStreamWaitEvent(st, w->ev_join[l], 0));
    }
  }
  if (zero_out_staging) CUDA_TRY(cudaMemsetAsync(d_out, 0, (size_t)nframes * cap * sizeof(pigo_det), st));
  timing_begin(T_FINALIZE, st);
  launch_finalize((const RawDet*)w->raw.p, d_rawcount, cap, (const ScaleEntry*)w->plan.p, nscales, d_out, d_nout, nframes, st);
  timing_end(T_FINALIZE, st);
  g_launches++;
  CUDA_TRY(cudaGetLastError());

  if (out_dev) return ws_leave_async(w, st);
  return copy_results_to_host(d_out, d_nout, cap, nframes, out, cap_per_frame, n_out, st);
}

static int check_batch_args(const pigo_cascade* c, const uint8_t* frames, int nframes, size_t frame_stride, int rows, int cols, int dim,
                            const pigo_det* out, int cap_per_frame, const int* n_out) {
  if (!c || !n_out || (!out && cap_per_frame > 0)) return set_err(PIGO_E_INVALID, "null argument");
  if (nframes < 0 || nframes > 65535) return set_err(PIGO_E_INVALID, "nframes must be 0..65535");
  if (rows < 0 || cols < 0 || dim < cols) return set_err(PIGO_E_INVALID, "bad geometry rows=%d cols=%d dim=%d", rows, cols, dim);
  if (cap_per_frame < 0) return set_err(PIGO_E_INVALID, "negative capacity");
  if ((uint64_t)rows * (uint64_t)dim > 0x7fffffffull) return set_err(PIGO_E_INVALID, "frames larger than 2^31 bytes are not supported");
  if (nframes > 0 && !frames) return set_err(PIGO_E_INVALID, "null frames");
  if (nframes > 1 && frame_stride < (size_t)rows * dim - (size_t)(dim - cols))
    return set_err(PIGO_E_INVALID, "frame_stride smaller than a frame");
  return PIGO_OK;
}

// ---- RunCascade over images of different sizes (pigo_run_cascade_images) -----------------------------------------------
// Windows per group of consecutive images: at most what a 128-frame group of 1080p frames holds at the test parameters
// (128 x 894,448), so that the deep queue of a group stays as bounded as the uniform path's.
static constexpr uint64_t kImagesGroupWindows = 128ull * 894448ull;

// Geometry of images[0..nimages): rows and cols at least min_edge (1 where images are refined on, which needs a pixel) and
// dim >= cols; with `pixels` also at most 2^31 bytes and non-null pixels.
static int check_image_geometry(const pigo_image* images, int nimages, int min_edge, bool pixels) {
  for (int i = 0; i < nimages; ++i) {
    const pigo_image& im = images[i];
    if (im.rows < min_edge || im.cols < min_edge || im.dim < im.cols)
      return set_err(PIGO_E_INVALID, "image %d: bad geometry rows=%d cols=%d dim=%d", i, im.rows, im.cols, im.dim);
    if (!pixels) continue;
    if ((uint64_t)im.rows * (uint64_t)im.dim > 0x7fffffffull) return set_err(PIGO_E_INVALID, "image %d: larger than 2^31 bytes", i);
    if (!im.pixels) return set_err(PIGO_E_INVALID, "image %d: null pixels", i);
  }
  return PIGO_OK;
}

static int check_images_args(const pigo_cascade* c, const pigo_image* images, int nimages, const pigo_det* out, int cap_per_image,
                             const int* n_out) {
  if (nimages < 0 || nimages > 65535) return set_err(PIGO_E_INVALID, "nimages must be 0..65535");
  if (nimages > 0 && !images) return set_err(PIGO_E_INVALID, "null images");
  if (!n_out) return set_err(PIGO_E_INVALID, "null n_out");
  if (cap_per_image < 0) return set_err(PIGO_E_INVALID, "negative capacity");
  if (!out && cap_per_image > 0) return set_err(PIGO_E_INVALID, "null out");
  const int rc = check_image_geometry(images, nimages, 0, true);
  if (rc) return rc;
  if (!c) return set_err(PIGO_E_INVALID, "null cascade");
  return PIGO_OK;
}

// The ladders of a mixed-size call's images (host only).  `longest` = the first image with the strictly longest ladder;
// every other ladder is a prefix of it (the rotated node table and the meaning of a ladder index are shared by the whole call).
struct ImagePlans {
  std::vector<std::vector<ScaleEntry>> plans;
  std::vector<uint64_t> wins;
  int longest = 0;
  // The ladders of entries [lo, lo+n), the shard of a sharded call that starts at entry lo.
  ImagePlans slice(int lo, int n) const {
    ImagePlans s;
    s.plans.assign(plans.begin() + lo, plans.begin() + lo + n);
    s.wins.assign(wins.begin() + lo, wins.begin() + lo + n);
    for (int i = 0; i < n; ++i)
      if (s.plans[i].size() > s.plans[s.longest].size()) s.longest = i;
    return s;
  }
};

static int build_image_plans(const pigo_image* images, int nimages, int min_size, int max_size, double shift, double scale_factor, ImagePlans& ip) {
  auto& plans = ip.plans;
  plans.assign(nimages, {});
  ip.wins.assign(nimages, 0);
  int& longest = ip.longest;
  longest = 0;
  for (int i = 0; i < nimages; ++i) {
    int rc = build_plan(images[i].rows, images[i].cols, min_size, max_size, shift, scale_factor, plans[i], ip.wins[i]);
    if (rc) return rc;
    if (plans[i].size() > plans[longest].size()) longest = i;
  }
  for (int i = 0; i < nimages; ++i)
    for (size_t k = 0; k < plans[i].size(); ++k) {
      const ScaleEntry &a = plans[i][k], &b = plans[longest][k];
      if (a.s != b.s || a.step != b.step || a.off != b.off)
        return set_err(PIGO_E_INVALID, "image %d: ladder entry %zu is not shared with the longest ladder", i, k);
    }
  return PIGO_OK;
}

// Bound on the rotated node tables one pass of a mixed-size call keeps on the device (one table per distinct slot, each
// over the call's longest ladder, at most 512 MB).  A call whose slots need more runs its rotated images in several passes.
static constexpr size_t kImagesRotBytes = (size_t)1 << 30;

// The items of a call in one arena of 256-byte-aligned slots of bytes(item) bytes.  Items whose key(item) repeats an earlier
// one share its slot, so a sweep that lists one photo once per angle copies (or converts) it once.
// off[i] = byte offset of item i's slot; first[i] = item i is the first to use that slot (its bytes are the ones written).
template <typename T, typename Key, typename Bytes>
static size_t arena_layout(const T* items, int n, Key key, Bytes bytes, std::vector<size_t>& off, std::vector<char>& first) {
  std::map<decltype(key(items[0])), size_t> seen;
  off.assign(n, 0);
  first.assign(n, 0);
  size_t total = 0;
  for (int i = 0; i < n; ++i) {
    const auto ins = seen.emplace(key(items[i]), total);
    off[i] = ins.first->second;
    if (ins.second) { first[i] = 1; total += (bytes(items[i]) + 255) & ~(size_t)255; }
  }
  return total;
}

// Host images of a mixed-size call: descriptors that repeat an earlier (pixels, rows, cols, dim) share its slot.
static size_t arena_layout(const pigo_image* images, int n, std::vector<size_t>& off, std::vector<char>& first) {
  return arena_layout(images, n, [](const pigo_image& im) { return std::make_tuple(im.pixels, im.rows, im.cols, im.dim); },
                      [](const pigo_image& im) { return (size_t)im.rows * im.dim; }, off, first);
}

// Host images into one arena in w->frames (arena_layout: each distinct image once), copying only their readable bytes;
// pixels[i] = image i's device copy.  Given `wins`, images without windows are not copied: a scan never reads them.
static int stage_pixels(Workspace* w, const pigo_image* images, int nimages, const std::vector<uint64_t>* wins, cudaStream_t st,
                        std::vector<const uint8_t*>& pixels) {
  std::vector<size_t> off;
  std::vector<char> first;
  const size_t total = arena_layout(images, nimages, off, first);
  const int rc = w->frames.reserve(total + 256);
  if (rc) return rc;
  pixels.resize(nimages);
  for (int i = 0; i < nimages; ++i) {
    uint8_t* dst = (uint8_t*)w->frames.p + off[i];
    pixels[i] = dst;
    if (!first[i] || (wins && (*wins)[i] == 0)) continue;   // a repeat, or never read
    const pigo_image& im = images[i];
    CUDA_TRY(cudaMemcpyAsync(dst, im.pixels, readable_bytes(im.rows, im.cols, im.dim), cudaMemcpyHostToDevice, st));
  }
  return PIGO_OK;
}

// Decoded images of pigo_gray_images: byte-identical descriptors share a slot of width*height gray bytes.
static size_t arena_layout(const pigo_decoded* src, int n, std::vector<size_t>& off, std::vector<char>& first) {
  return arena_layout(src, n,
                      [](const pigo_decoded& d) {
                        return std::make_tuple(d.format, d.subsample, d.min_x, d.min_y, d.width, d.height, d.plane[0], d.plane[1], d.plane[2],
                                               d.stride[0], d.stride[1]);
                      },
                      [](const pigo_decoded& d) { return (size_t)d.width * d.height; }, off, first);
}

// Image i is scanned at angles[i].  The rotated and the unrotated scan are different kernel variants, so the images run
// in passes: the unrotated images in caller order, then the rotated ones ordered by (slot, caller index), cut into
// passes of at most kImagesRotBytes of node tables.  That order does not depend on how the caller interleaves images and
// angles.  Each pass is grouped and scheduled from its own windows; finalize writes every image to its caller index.
static int scan_images_on(pigo_cascade* c, int dev, const pigo_image* images, int nimages, const ImagePlans& ip, int min_size, int max_size,
                          double shift_factor, double scale_factor, const double* angles, pigo_det* out, int cap_per_image, int* n_out,
                          unsigned flags, void* stream_) {
  int rc = PIGO_OK;
  FaceReplica* R = face_replica(c, dev, &rc);
  if (!R) return rc;
  if ((rc = use_device(dev))) return rc;
  const bool frames_dev = flags & PIGO_FRAMES_DEVICE, out_dev = flags & PIGO_OUT_DEVICE;
  std::vector<int> slot(nimages);
  bool any_rot = false;
  for (int i = 0; i < nimages; ++i) { slot[i] = rot_slot_of(angles[i]); any_rot |= slot[i] >= 0; }
  const int nlad = (int)ip.plans[ip.longest].size();
  const int max_scale = nlad > 0 ? ip.plans[ip.longest].back().s : 0;
  const size_t rot_bytes = (size_t)nlad * (size_t)R->tab.ntrees * 64 * sizeof(RotNode);
  if (!block_path(R, any_rot, max_scale, rot_bytes)) {
    // cascades of depth != 6 and the universal-kernel options: the single-image path, image by image at its own angle
    int rc_cap = PIGO_OK;
    for (int i = 0; i < nimages; ++i) {
      const pigo_image& im = images[i];
      rc = scan_batch_on(c, dev, im.pixels, 1, (size_t)im.rows * im.dim, im.rows, im.cols, im.dim, min_size, max_size, shift_factor,
                         scale_factor, angles[i], out ? out + (size_t)i * cap_per_image : nullptr, cap_per_image, n_out + i, flags, stream_);
      if (rc == PIGO_E_CAP) rc_cap = rc;
      else if (rc) return rc;
    }
    return rc_cap == PIGO_OK ? PIGO_OK : set_err(PIGO_E_CAP, "output capacity %d per image too small", cap_per_image);
  }

  Borrow w(R->pool, stream_);
  if (w.rc) return w.rc;
  cudaStream_t st = w.st;
  const int cap = cap_per_image > 0 ? cap_per_image : 1;

  // order[j] = caller index of the image at position j of the call's image table; passes are ranges of positions
  std::vector<int> order(nimages);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return slot[a] < slot[b]; });
  struct Pass { int first, n; std::vector<int> slots; };   // slots: the pass's node tables in order (empty = unrotated)
  std::vector<Pass> passes;
  const size_t slots_per_pass = std::max<size_t>(1, kImagesRotBytes / std::max<size_t>(rot_bytes, 1));
  for (int j = 0; j < nimages; ++j) {
    const int s = slot[order[j]];
    const bool new_slot = j == 0 || s != slot[order[j - 1]];
    if (j == 0 || (s >= 0 && slot[order[j - 1]] < 0) || (new_slot && s >= 0 && passes.back().slots.size() == slots_per_pass))
      passes.push_back(Pass{j, 0, {}});
    Pass& p = passes.back();
    if (new_slot && s >= 0) p.slots.push_back(s);
    p.n++;
  }
  size_t max_tables = 0;
  for (const Pass& p : passes) max_tables = std::max(max_tables, p.slots.size());

  // per pass: schedule from the pass's windows; block prefixes per image, groups of consecutive images
  std::vector<ImageDesc> desc(nimages);
  std::vector<ScaleEntry> plan_all;
  struct Group { int first, n; uint32_t blocks; uint64_t windows; int pass; };
  std::vector<Group> groups;
  std::vector<ImagesSchedule> sched(passes.size());
  const long long sub = g_opt.sub_batch.load();   // developer knob: at most this many images per group
  for (size_t pi = 0; pi < passes.size(); ++pi) {
    const Pass& p = passes[pi];
    uint64_t pass_windows = 0;
    for (int j = p.first; j < p.first + p.n; ++j) pass_windows += ip.wins[order[j]];
    // (gather-v2 is the whole scan here, as on the rotated path: large unrotated calls keep 24 trees, not run_scan's 16,
    // since the hand-over point was not re-measured for it)
    sched[pi] = images_schedule(pass_windows, !p.slots.empty(), 24);
    const int GB = 1 << sched[pi].gb_shift;
    // groups of about equal window counts (a uniform 1080p batch gets the uniform path's groups of 128)
    const uint64_t ngroups = std::max<uint64_t>(1, (pass_windows + kImagesGroupWindows - 1) / kImagesGroupWindows);
    const uint64_t group_target = (pass_windows + ngroups - 1) / ngroups;
    const size_t first_group = groups.size();
    for (int j = p.first; j < p.first + p.n; ++j) {
      const int i = order[j];
      if (groups.size() == first_group || (groups.back().windows > 0 && groups.back().windows + ip.wins[i] > group_target) ||
          (sub > 0 && groups.back().n >= sub))
        groups.push_back(Group{j, 0, 0, 0, (int)pi});
      Group& G = groups.back();
      ImageDesc& d = desc[j];
      d.rows = images[i].rows; d.cols = images[i].cols; d.dim = images[i].dim;
      d.nscales = (int)ip.plans[i].size();
      d.plan_off = (uint32_t)plan_all.size();
      d.block_base = G.blocks;
      d.rot_slot = slot[i];
      d.rot_off = 0;
      if (slot[i] >= 0)
        d.rot_off = (uint32_t)((std::find(p.slots.begin(), p.slots.end(), slot[i]) - p.slots.begin()) * (size_t)nlad * R->tab.ntrees);
      d.out_index = i;
      uint32_t nb = 0;
      for (ScaleEntry e : ip.plans[i]) {
        e.pad = nb;
        nb += (uint32_t)((e.ncols + GB - 1) / GB) * (uint32_t)((e.nrows + GB - 1) / GB);
        plan_all.push_back(e);
      }
      if ((uint64_t)G.blocks + nb > 0xffffffffull) return set_err(PIGO_E_INVALID, "image %d: too many windows", i);
      G.blocks += nb; G.windows += ip.wins[i]; G.n++;
    }
  }

  // pixels: device images in place, host images staged
  if (frames_dev) {
    for (int j = 0; j < nimages; ++j) desc[j].base = images[order[j]].pixels;
  } else {
    std::vector<const uint8_t*> pixels;
    if ((rc = stage_pixels(w, images, nimages, &ip.wins, st, pixels))) return rc;
    for (int j = 0; j < nimages; ++j) desc[j].base = pixels[order[j]];
  }

  // image table + concatenated plan (this call's own buffer: the workspace's cached uniform plan stays as it is)
  const size_t desc_bytes = ((size_t)nimages * sizeof(ImageDesc) + 255) & ~(size_t)255;
  const size_t plan_bytes = plan_all.size() * sizeof(ScaleEntry);
  std::vector<uint8_t> tab(desc_bytes + plan_bytes);
  memcpy(tab.data(), desc.data(), (size_t)nimages * sizeof(ImageDesc));
  if (plan_bytes) memcpy(tab.data() + desc_bytes, plan_all.data(), plan_bytes);
  if ((rc = w->img_tab.reserve(tab.size()))) return rc;
  CUDA_TRY(cudaMemcpyAsync(w->img_tab.p, tab.data(), tab.size(), cudaMemcpyHostToDevice, st));
  const ImageDesc* d_desc = (const ImageDesc*)w->img_tab.p;
  const ScaleEntry* d_plan = (const ScaleEntry*)((const uint8_t*)w->img_tab.p + desc_bytes);
  const int longest_pos = (int)(std::find(order.begin(), order.end(), ip.longest) - order.begin());
  // the node tables of a pass over the longest ladder, one per slot, cached per workspace by (slots, ladder)
  if (max_tables > 0 && nlad > 0) {
    const size_t cap0 = w->img_rot.cap;
    if ((rc = w->img_rot.reserve(max_tables * rot_bytes))) { w->img_rot_slots.clear(); return rc; }
    if (w->img_rot.cap != cap0) w->img_rot_slots.clear();   // a new buffer holds no tables
  }
  auto build_tables = [&](const std::vector<int>& slots) -> int {
    if (w->img_rot_slots == slots && w->img_rot_len == nlad && w->img_rot_min == min_size && w->img_rot_scale == scale_factor) return PIGO_OK;
    w->img_rot_slots.clear();
    timing_begin(T_ROTTAB, st);
    for (size_t k = 0; k < slots.size(); ++k) {
      launch_rot_table(R->tab, d_plan + desc[longest_pos].plan_off, nlad, slots[k], (RotNode*)w->img_rot.p + k * (size_t)nlad * R->tab.ntrees * 64,
                       R->num_sms * 8, st);
      g_launches++;
    }
    timing_end(T_ROTTAB, st);
    CUDA_TRY(cudaGetLastError());
    w->img_rot_slots = slots; w->img_rot_len = nlad; w->img_rot_min = min_size; w->img_rot_scale = scale_factor;
    return PIGO_OK;
  };

  // outputs and counters: [0..nimages) raw counts | 8 x u64 work counters per group
  pigo_det* d_out = out;
  int32_t* d_nout = n_out;
  if (!out_dev) {
    if ((rc = w->out.reserve((size_t)nimages * cap * sizeof(pigo_det)))) return rc;
    if ((rc = w->nout.reserve((size_t)nimages * sizeof(int32_t)))) return rc;
    d_out = (pigo_det*)w->out.p;
    d_nout = (int32_t*)w->nout.p;
  }
  if ((rc = w->raw.reserve((size_t)nimages * cap * sizeof(RawDet)))) return rc;
  const size_t work_off = ((size_t)nimages * 4 + 15) & ~(size_t)15;
  const size_t cnt_bytes = work_off + groups.size() * 64 + 64;
  if ((rc = w->counters.reserve(cnt_bytes))) return rc;
  CUDA_TRY(cudaMemsetAsync(w->counters.p, 0, cnt_bytes, st));
  int32_t* d_rawcount = (int32_t*)w->counters.p;
  unsigned long long* d_work = (unsigned long long*)((char*)w->counters.p + work_off);

  int tables_of = -1;   // pass whose node tables img_rot holds in this call
  for (size_t k = 0; k < groups.size(); ++k) {
    const Group& G = groups[k];
    if (G.windows == 0 || R->tab.ntrees == 0) continue;
    const Pass& p = passes[G.pass];
    if (!p.slots.empty() && tables_of != G.pass) {
      if ((rc = build_tables(p.slots))) return rc;
      tables_of = G.pass;
    }
    int first_live = G.first;
    while (ip.wins[order[first_live]] == 0) ++first_live;
    ScanArgs A{};
    A.tab = R->tab;
    A.frames = desc[first_live].base;   // a readable pixel for the idle lanes of the kernels
    A.nframes = G.n;
    A.plan = d_plan;
    // the images kernels read only whether the pass is rotated; each image's node table comes from its ImageDesc
    A.rot_slot = p.slots.empty() ? -1 : p.slots[0];
    A.rot_tab = p.slots.empty() ? nullptr : (const RotNode*)w->img_rot.p;
    A.batch_frames = nimages;
    A.raw = (RawDet*)w->raw.p + (size_t)G.first * cap; A.raw_count = d_rawcount + G.first; A.cap = cap;
    A.images = d_desc + G.first; A.nimages = G.n;
    int max_rows = 1, max_cols = 1;
    for (int j = G.first; j < G.first + G.n; ++j) { max_rows = std::max(max_rows, desc[j].rows); max_cols = std::max(max_cols, desc[j].cols); }
    if ((rc = run_scan_images(R, w, A, sched[G.pass], G.blocks, G.windows, max_rows, max_cols, d_work + 8 * k, st, R->num_sms))) return rc;
  }
  if (!out_dev) CUDA_TRY(cudaMemsetAsync(d_out, 0, (size_t)nimages * cap * sizeof(pigo_det), st));
  timing_begin(T_FINALIZE, st);
  launch_finalize_images((const RawDet*)w->raw.p, d_rawcount, cap, d_plan, d_desc, d_out, d_nout, nimages, st);
  timing_end(T_FINALIZE, st);
  g_launches++;
  CUDA_TRY(cudaGetLastError());
  if (out_dev) return ws_leave_async(w, st);
  return copy_results_to_host(d_out, d_nout, cap, nimages, out, cap_per_image, n_out, st);
}

// The devices of the sharded calls: those of pigo_init_devices, or the default device.  Empty if there is none.
static std::vector<int> sharded_devices() {
  std::vector<int> devs = shard_devices();
  if (devs.empty()) {
    const int d = default_device();
    if (d >= 0) devs.push_back(d);
  }
  return devs;
}

// Runs fn(shard index, device, first entry, entry count) for shard s = entries [first[s], first[s+1]) on devs[s % G], one
// host thread per non-empty shard.  Returns the first error, PIGO_E_CAP last (so that every shard's required counts are
// valid when the caller retries).
template <typename F>
static int for_each_shard(const std::vector<int>& devs, const std::vector<int>& first, F fn) {
  const int S = (int)first.size() - 1, G = (int)devs.size();
  std::vector<int> rcs(std::max(S, 0), PIGO_OK);
  std::vector<std::string> msgs(std::max(S, 0));
  std::vector<std::thread> th;
  for (int s = 0; s < S; ++s) {
    const int lo = first[s], hi = first[s + 1];
    if (hi <= lo) continue;
    th.emplace_back([&, s, lo, hi]() {
      rcs[s] = fn(s, devs[s % G], lo, hi - lo);
      if (rcs[s] != PIGO_OK) msgs[s] = g_err;   // g_err is thread-local: carry the worker's message back
    });
  }
  for (auto& t : th) t.join();
  int rc = PIGO_OK;
  for (int s = 0; s < S; ++s) {
    if (rcs[s] == PIGO_OK) continue;
    if (rc == PIGO_OK || (rc == PIGO_E_CAP && rcs[s] != PIGO_E_CAP)) { rc = rcs[s]; g_err = msgs[s]; }
  }
  return rc;
}

// The frame batches' split: one shard per device of the mask, frames [g*ceil(N/G), (g+1)*ceil(N/G)) like SURVEY.md section 8e.
template <typename F>
static int for_each_shard(int nframes, F fn) {
  const std::vector<int> devs = sharded_devices();
  if (devs.empty()) return PIGO_E_NODEVICE;
  const int G = (int)devs.size();
  const int per = (nframes + G - 1) / G;
  std::vector<int> first(G + 1);
  for (int g = 0; g <= G; ++g) first[g] = std::min(nframes, g * per);
  return for_each_shard(devs, first, fn);
}

// ---- the split of a sharded mixed-size call (pigo_shard_plan) -----------------------------------------------------------
// Modelled cost of an entry, in tenths of a window: count_windows x (rotated ? kRotCost : 10) + kImgCost.
// kRotCost / 10 = 1.4 is the ratio of the unrotated to the rotated windows/s of DESIGN.md section 5.  Those two rates come
// from different workloads and were never measured as a cost ratio; tools/ragged_bench.py --sections sharded sets modelled
// shard costs against measured shard times.  kImgCost stands for the fixed cost of an entry (descriptor, finalize, its
// share of the launches): 4096 windows, a guess of the same standing.
static constexpr uint64_t kRotCost = 14, kImgCost = 4096 * 10;

// first[0..S] of the cut of cost[] into S = min(nshards, n) contiguous non-empty ranges whose largest cost is the least
// any contiguous split into at most S ranges reaches (binary search on that bottleneck, then a greedy cut that also
// leaves one entry for every shard still to come).
static std::vector<int> cut_shards(const std::vector<uint64_t>& cost, int nshards) {
  const int n = (int)cost.size(), S = std::min(nshards, n);
  std::vector<int> first{0};
  if (S <= 0) return first;
  uint64_t lo = 0, hi = 0;
  for (uint64_t c : cost) { lo = std::max(lo, c); hi += c; }
  auto ranges_at = [&](uint64_t B) {   // ranges a greedy cut at bottleneck B needs
    int k = 1;
    uint64_t sum = 0;
    for (uint64_t c : cost) {
      if (sum + c > B) { ++k; sum = 0; }
      sum += c;
    }
    return k;
  };
  while (lo < hi) {
    const uint64_t mid = lo + (hi - lo) / 2;
    if (ranges_at(mid) <= S) hi = mid; else lo = mid + 1;
  }
  uint64_t sum = 0;
  for (int i = 0; i < n; ++i) {
    const int shards_left = S - (int)first.size();   // ranges still to start after the current one
    // cut before entry i when it does not fit under the bottleneck, or when entries i.. are just enough for those ranges
    if (i > 0 && shards_left > 0 && (sum + cost[i] > lo || n - i <= shards_left)) {
      first.push_back(i);
      sum = 0;
    }
    sum += cost[i];
  }
  first.push_back(n);
  return first;
}

// Shards of a sharded mixed-size call on G devices: option shard_split, or one per device.
static int shard_count(int G) {
  const long long k = g_opt.shard_split.load();
  return k > 0 ? (int)std::min<long long>(k, 65535) : G;
}

// The split of entries with window counts wins[] at angles[] (nullptr: all unrotated) into at most nshards shards.
static std::vector<int> plan_shards(const std::vector<uint64_t>& wins, const double* angles, int nshards) {
  std::vector<uint64_t> cost(wins.size());
  for (size_t i = 0; i < wins.size(); ++i) cost[i] = wins[i] * (angles && rot_slot_of(angles[i]) >= 0 ? kRotCost : 10) + kImgCost;
  return cut_shards(cost, nshards);
}

// ---- RunDetector over uniform frames or over an image table (pigo_puploc_run_frames / pigo_puploc_run_images) -----------
// Host seeds of a standalone RunDetector call: Perturbs range and frame / image index.  *wide = some seed lies outside the
// 32-bit envelope of the pair kernel (it then runs on the warp-per-perturbation kernel).
static int check_puploc_seeds(const pigo_point* seeds, int nseeds, const int32_t* seed_frame, int nframes, const char* unit, bool* wide) {
  for (int i = 0; i < nseeds; ++i) {
    if (seeds[i].perturbs < 0 || seeds[i].perturbs > 63)
      return set_err(PIGO_E_INVALID, "seed %d: Perturbs=%d outside 0..63 (the reference panics, core/puploc.go:261)", i, seeds[i].perturbs);
    if (seed_frame && (seed_frame[i] < 0 || seed_frame[i] >= nframes)) return set_err(PIGO_E_INVALID, "seed %d: %s index out of range", i, unit);
    if (!(std::fabs(seeds[i].scale) <= 16384.0f)) *wide = true;
  }
  return PIGO_OK;
}

// Pixels of a mixed-size call on the device.  Device images stay where they are; host images are staged, every one of
// them (the RunDetector stages read each image).  The call's ImageDesc table (pixels, rows, cols, pitch and, given `angles`,
// each image's rotation slot) goes to w->img_tab; `staged` receives the device descriptors of the images.
static int stage_images(Workspace* w, const pigo_image* images, int nimages, const double* angles, bool frames_dev, cudaStream_t st,
                        const ImageDesc** d_desc, std::vector<pigo_image>& staged) {
  int rc = PIGO_OK;
  staged.assign(images, images + nimages);
  if (!frames_dev) {
    std::vector<const uint8_t*> pixels;
    if ((rc = stage_pixels(w, images, nimages, nullptr, st, pixels))) return rc;
    for (int i = 0; i < nimages; ++i) staged[i].pixels = pixels[i];
  }
  std::vector<ImageDesc> desc(nimages);
  for (int i = 0; i < nimages; ++i) {
    desc[i] = ImageDesc{};
    desc[i].base = staged[i].pixels; desc[i].rows = staged[i].rows; desc[i].cols = staged[i].cols; desc[i].dim = staged[i].dim;
    desc[i].rot_slot = angles ? rot_slot_of(angles[i]) : -1;
    desc[i].out_index = i;
  }
  if ((rc = w->img_tab.reserve((size_t)nimages * sizeof(ImageDesc)))) return rc;
  CUDA_TRY(cudaMemcpyAsync(w->img_tab.p, desc.data(), (size_t)nimages * sizeof(ImageDesc), cudaMemcpyHostToDevice, st));
  *d_desc = (const ImageDesc*)w->img_tab.p;
  return PIGO_OK;
}

// Where the seeds' pixels are: `nframes` uniform frames `stride` bytes apart, or (images != nullptr) an image table of
// `nframes` entries.  Pointers are host or device memory as the call's flags say.
struct PuplocPixels {
  const uint8_t* frames;
  int nframes;
  size_t stride;
  int rows, cols, dim;
  const pigo_image* images;
};

static int puploc_run_on(pigo_puploc* p, const pigo_point* seeds, int nseeds, const int32_t* seed_frame, const float* randoms, uint64_t rng_seed,
                         const PuplocPixels& px, double angle, const uint8_t* flipv, pigo_point* out, bool wide, unsigned flags, void* stream_) {
  int rc = PIGO_OK;
  const int dev = default_device();
  PuplocReplica* R = puploc_replica(p, dev, &rc);
  if (!R) return rc;
  const bool frames_dev = flags & PIGO_FRAMES_DEVICE, out_dev = flags & PIGO_OUT_DEVICE;
  Borrow w(R->pool, stream_);
  if (w.rc) return w.rc;
  cudaStream_t st = w.st;
  const uint8_t* d_pix = px.frames;
  const ImageDesc* d_img = nullptr;
  if (px.images) {
    std::vector<pigo_image> staged;
    if ((rc = stage_images(w, px.images, px.nframes, nullptr, frames_dev, st, &d_img, staged))) return rc;
  } else if (!frames_dev) {
    const size_t bytes = px.stride * (size_t)(px.nframes - 1) + readable_bytes(px.rows, px.cols, px.dim);
    if ((rc = w->frames.reserve(px.stride * (size_t)(px.nframes - 1) + (size_t)px.rows * px.dim))) return rc;
    CUDA_TRY(cudaMemcpyAsync(w->frames.p, px.frames, bytes, cudaMemcpyHostToDevice, st));
    d_pix = (const uint8_t*)w->frames.p;
  }
  const int32_t* d_sf = seed_frame;
  const pigo_point* d_seeds = seeds;
  pigo_point* d_out = out;
  const float* d_rnd = randoms;
  const uint8_t* d_flip = flipv;
  if (!out_dev) {
    const size_t sb = (size_t)nseeds * sizeof(pigo_point), rb = (size_t)nseeds * 63 * 3 * sizeof(float);
    if ((rc = w->scratch_a.reserve(2 * sb))) return rc;
    d_seeds = (const pigo_point*)w->scratch_a.p;
    d_out = (pigo_point*)((char*)w->scratch_a.p + sb);
    CUDA_TRY(cudaMemcpyAsync(w->scratch_a.p, seeds, sb, cudaMemcpyHostToDevice, st));
    if (randoms) {
      if ((rc = w->scratch_b.reserve(rb))) return rc;
      CUDA_TRY(cudaMemcpyAsync(w->scratch_b.p, randoms, rb, cudaMemcpyHostToDevice, st));
      d_rnd = (const float*)w->scratch_b.p;
    }
    if (flipv) {
      if ((rc = w->scratch_c.reserve(nseeds))) return rc;
      CUDA_TRY(cudaMemcpyAsync(w->scratch_c.p, flipv, nseeds, cudaMemcpyHostToDevice, st));
      d_flip = (const uint8_t*)w->scratch_c.p;
    }
    if (seed_frame) {
      if ((rc = w->nout.reserve((size_t)nseeds * 4))) return rc;
      CUDA_TRY(cudaMemcpyAsync(w->nout.p, seed_frame, (size_t)nseeds * 4, cudaMemcpyHostToDevice, st));
      d_sf = (const int32_t*)w->nout.p;
    }
  }
  const int rot_slot = rot_slot_of(angle);  // core/puploc.go:252-256, :166
  bool done = false;
  timing_begin(T_PUPLOC, st);
  if (g_opt.puploc_mode.load() == 0 && !wide) {
    if ((rc = w->counters.reserve(64))) return rc;
    CUDA_TRY(cudaMemsetAsync(w->counters.p, 0, 64, st));
    PupWork W{};
    W.seeds = d_seeds; W.out = d_out; W.randoms = d_rnd; W.rng_seed = rng_seed; W.frames = d_pix; W.frame_stride = px.stride;
    W.slot_frame = d_sf; W.flipv = d_flip; W.slots_per_frame = 0; W.nrows = px.rows; W.ncols = px.cols; W.dim = px.dim; W.rot_slot = rot_slot;
    W.first = 0; W.span = 1; W.stride = 1; W.nwork = nseeds; W.ntabs = 1; W.tab[0] = R->tab; W.images = d_img;
    done = launch_puploc_pairs(W, (unsigned int*)w->counters.p, R->num_sms, st) == 0;
  }
  if (!done)
    launch_puploc(R->tab, d_seeds, nseeds, d_rnd, rng_seed, d_pix, d_sf, px.stride, px.rows, px.cols, px.dim, rot_slot, d_flip, d_out, d_img, st);
  timing_end(T_PUPLOC, st);
  g_launches++;
  CUDA_TRY(cudaGetLastError());
  if (out_dev) return ws_leave_async(w, st);
  CUDA_TRY(cudaMemcpyAsync(out, d_out, (size_t)nseeds * sizeof(pigo_point), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return PIGO_OK;
}

// =========================================================================================================
extern "C" {

const char* pigo_last_error(void) { return g_err.c_str(); }
int pigo_version(void) { return PIGO_B200_VERSION; }
int64_t pigo_launch_count(void) { return g_launches.load(); }

int pigo_init(int device) {
  int rc = use_device(device);
  if (rc) return rc;
  g_device.store(device);
  g_mask.store(1u << device);
  return PIGO_OK;
}

int pigo_init_devices(unsigned device_mask) {
  if (device_mask == 0 || device_mask >= (1u << kMaxDevices)) return set_err(PIGO_E_INVALID, "empty or out-of-range device mask 0x%x", device_mask);
  int first = -1;
  for (int d = kMaxDevices - 1; d >= 0; --d) {
    if (!(device_mask & (1u << d))) continue;
    int rc = use_device(d);
    if (rc) return rc;
    first = d;
  }
  // peer access between the devices of the mask: the device-output form of the sharded calls gathers over NVLink
  for (int a = 0; a < kMaxDevices; ++a)
    for (int b = 0; b < kMaxDevices; ++b) {
      if (a == b || !(device_mask & (1u << a)) || !(device_mask & (1u << b))) continue;
      int can = 0;
      if (cudaDeviceCanAccessPeer(&can, a, b) == cudaSuccess && can) {
        cudaSetDevice(a);
        cudaError_t e = cudaDeviceEnablePeerAccess(b, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        cudaGetLastError();
      }
    }
  CUDA_TRY(cudaSetDevice(first));
  g_device.store(first);
  g_mask.store(device_mask);
  return PIGO_OK;
}

int pigo_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int pigo_shutdown_impl(void);
int pigo_shutdown(void) { return pigo_shutdown_impl(); }

int pigo_alloc_pinned(void** ptr, size_t bytes) {
  if (!ptr) return set_err(PIGO_E_INVALID, "null ptr");
  int rc = ensure_device();
  if (rc) return rc;
  CUDA_TRY(cudaHostAlloc(ptr, bytes, cudaHostAllocPortable));
  return PIGO_OK;
}
int pigo_free_pinned(void* ptr) {
  if (ptr) CUDA_TRY(cudaFreeHost(ptr));
  return PIGO_OK;
}

int pigo_device_alloc(void** ptr, size_t bytes) {
  if (!ptr) return set_err(PIGO_E_INVALID, "null ptr");
  int rc = ensure_device();
  if (rc) return rc;
  if (cudaMalloc(ptr, bytes ? bytes : 1) != cudaSuccess) { cudaGetLastError(); return set_err(PIGO_E_NOMEM, "cudaMalloc(%zu) failed", bytes); }
  return PIGO_OK;
}
int pigo_device_free(void* ptr) {
  if (ptr) CUDA_TRY(cudaFree(ptr));
  return PIGO_OK;
}
int pigo_device_upload(void* dst, const void* src, size_t bytes) {
  if (bytes == 0) return PIGO_OK;
  if (!dst || !src) return set_err(PIGO_E_INVALID, "null argument");
  int rc = ensure_device();
  if (rc) return rc;
  CUDA_TRY(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
  return PIGO_OK;
}
int pigo_device_download(void* dst, const void* src, size_t bytes) {
  if (bytes == 0) return PIGO_OK;
  if (!dst || !src) return set_err(PIGO_E_INVALID, "null argument");
  int rc = ensure_device();
  if (rc) return rc;
  CUDA_TRY(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
  return PIGO_OK;
}

int pigo_set_option(const char* name, int64_t value) {
  if (!name) return set_err(PIGO_E_INVALID, "null option name");
  return g_opt.set(name, value) ? PIGO_OK : set_err(PIGO_E_INVALID, "unknown option '%s'", name);
}
int64_t pigo_get_option(const char* name) { return name ? g_opt.get(name) : -1; }

int pigo_cascade_block_table(pigo_cascade* c, uint8_t* dst, size_t* bytes) {
  if (!c || !bytes) return set_err(PIGO_E_INVALID, "null argument");
  int rc = ensure_device();
  if (rc) return rc;
  FaceReplica* R = face_replica(c, default_device(), &rc);
  if (!R) return rc;
  const size_t n = R->block_tab.p ? (size_t)((c->ntrees + kBlockTrees - 1) / kBlockTrees) * kBlockBytes : 0;
  if (dst) {
    if (*bytes < n) return set_err(PIGO_E_INVALID, "block table needs %zu bytes", n);
    if (n) CUDA_TRY(cudaMemcpy(dst, R->block_tab.p, n, cudaMemcpyDeviceToHost));
  }
  *bytes = n;
  return PIGO_OK;
}

// ---- (*Pigo).Unpack, core/pigo.go:51-110 ----------------------------------------------------------------
static uint32_t rd_u32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

int pigo_cascade_create(const uint8_t* packet, size_t len, pigo_cascade** out) {
  if (!packet || !out) return set_err(PIGO_E_INVALID, "null argument");
  if (len < 16) return set_err(PIGO_E_INVALID, "cascade packet shorter than its 16-byte header");
  const uint32_t depth = rd_u32(packet + 8);    // :64 (bytes 0..7 are skipped, :61)
  const uint32_t ntrees = rd_u32(packet + 12);  // :68
  if (depth < 1 || depth > 12) return set_err(PIGO_E_INVALID, "unsupported tree depth %u", depth);
  const size_t leaves = (size_t)1 << depth;
  const size_t per_tree = (4 * leaves - 4) + 4 * leaves + 4;
  if (ntrees > (1u << 20) || len < 16 + (size_t)ntrees * per_tree)
    return set_err(PIGO_E_INVALID, "cascade packet truncated: %zu bytes, need %zu", len, 16 + (size_t)ntrees * per_tree);
  int rc = ensure_device();
  if (rc) return rc;
  pigo_cascade* c = new pigo_cascade();
  c->depth = depth; c->ntrees = ntrees; c->leaves = (uint32_t)leaves;
  c->h_codes.assign((size_t)ntrees * 4 * leaves + 16, 0);
  c->h_preds.assign((size_t)ntrees * leaves + 4, 0.f);
  c->h_thr.assign(ntrees + 4, 0.f);
  size_t pos = 16;
  for (uint32_t t = 0; t < ntrees; ++t) {
    memcpy(c->h_codes.data() + (size_t)t * 4 * leaves + 4, packet + pos, 4 * leaves - 4);  // 4 zero bytes first, :79-86
    pos += 4 * leaves - 4;
    memcpy(c->h_preds.data() + (size_t)t * leaves, packet + pos, 4 * leaves);              // :89-95 (LE f32 bit copy)
    pos += 4 * leaves;
    memcpy(c->h_thr.data() + t, packet + pos, 4);                                          // :96-100
    pos += 4;
  }
  // device tables: on the default device now, on every other device of a sharded call at its first use there
  if (!face_replica(c, default_device(), &rc)) { delete c; return rc; }
  *out = c;
  return PIGO_OK;
}

void pigo_cascade_destroy(pigo_cascade* c) { delete c; }

int pigo_cascade_info(const pigo_cascade* c, uint32_t* tree_depth, uint32_t* tree_num) {
  if (!c) return set_err(PIGO_E_INVALID, "null cascade");
  if (tree_depth) *tree_depth = c->depth;
  if (tree_num) *tree_num = c->ntrees;
  return PIGO_OK;
}

int pigo_scale_ladder(int min_size, int max_size, double scale_factor, int* scales, int cap, int* n_out) {
  long long scale = min_size;
  int n = 0;
  while (scale <= max_size) {
    if (scales && n < cap) scales[n] = (int)scale;
    if (++n > (1 << 16)) return set_err(PIGO_E_INVALID, "scale ladder longer than 65536 entries");
    scale = (long long)((double)scale + std::fmax(2.0, ((double)scale * scale_factor) - (double)scale));
  }
  if (n_out) *n_out = n;
  return (scales && n > cap) ? set_err(PIGO_E_CAP, "ladder has %d entries", n) : PIGO_OK;
}

int64_t pigo_count_windows(int rows, int cols, int min_size, int max_size, double shift_factor, double scale_factor) {
  std::vector<ScaleEntry> plan;
  uint64_t total = 0;
  if (build_plan(rows, cols, min_size, max_size, shift_factor, scale_factor, plan, total) != PIGO_OK) return -1;
  return (int64_t)total;
}

int pigo_describe_plan_frames(int rows, int cols, int min_size, int max_size, double shift_factor, double scale_factor, int nframes,
                              char* json, size_t cap) {
  if (!json) return set_err(PIGO_E_INVALID, "null buffer");
  if (nframes < 1) return set_err(PIGO_E_INVALID, "nframes must be at least 1");
  std::vector<ScaleEntry> plan;
  uint64_t total = 0;
  int rc = build_plan(rows, cols, min_size, max_size, shift_factor, scale_factor, plan, total);
  if (rc) return rc;
  return describe_plan(plan, total, 468, nframes, json, cap);   // geometry of the stock 468-tree facefinder cascade
}
int pigo_describe_plan(int rows, int cols, int min_size, int max_size, double shift_factor, double scale_factor, char* json, size_t cap) {
  return pigo_describe_plan_frames(rows, cols, min_size, max_size, shift_factor, scale_factor, 1 << 20, json, cap);
}

// ---- RunCascade ------------------------------------------------------------------------------------------
int pigo_run_cascade_batch(const pigo_cascade* cc, const uint8_t* frames, int nframes, size_t frame_stride, int rows, int cols,
                           int dim, int min_size, int max_size, double shift_factor, double scale_factor, double angle,
                           pigo_det* out, int cap_per_frame, int* n_out, unsigned flags, void* stream_) {
  int rc = check_batch_args(cc, frames, nframes, frame_stride, rows, cols, dim, out, cap_per_frame, n_out);
  if (rc) return rc;
  if ((rc = ensure_device())) return rc;
  if (nframes == 0) return PIGO_OK;
  return scan_batch_on(const_cast<pigo_cascade*>(cc), default_device(), frames, nframes, frame_stride, rows, cols, dim, min_size, max_size,
                       shift_factor, scale_factor, angle, out, cap_per_frame, n_out, flags, stream_);
}

int pigo_run_cascade(const pigo_cascade* c, const uint8_t* pixels, int rows, int cols, int dim, int min_size, int max_size,
                     double shift_factor, double scale_factor, double angle, pigo_det* out, int cap, int* n_out) {
  return pigo_run_cascade_batch(c, pixels, 1, (size_t)rows * (size_t)dim, rows, cols, dim, min_size, max_size, shift_factor,
                                scale_factor, angle, out, cap, n_out, PIGO_MEM_HOST, nullptr);
}

}  // extern "C"

// The entry points whose host work synchronises refuse a caller's stream that is capturing a CUDA graph.
static int refuse_capture(const char* fn, void* stream_) {
  if (stream_ && stream_capturing((cudaStream_t)stream_)) return set_err(PIGO_E_INVALID, "%s does not support stream capture", fn);
  return PIGO_OK;
}

// `angles`, or when it is nullptr n copies of `angle`, held in `store`.
static const double* angles_or(const double* angles, double angle, int n, std::vector<double>& store) {
  if (angles) return angles;
  store.assign(n, angle);
  return store.data();
}

// The start of a mixed-size call after its argument checks: the ladders of its n scan entries (a sweep's expanded list),
// the default device and the refusal of stream capture (`fn` names the entry point).  With n == 0 nothing more is to do.
static int images_prologue(const char* fn, const pigo_image* images, int n, int min_size, int max_size, double shift_factor, double scale_factor,
                           void* stream_, ImagePlans& ip) {
  int rc = build_image_plans(images, n, min_size, max_size, shift_factor, scale_factor, ip);
  if (rc) return rc;
  if ((rc = ensure_device())) return rc;
  return refuse_capture(fn, stream_);
}

// pigo_run_cascade_images and pigo_run_cascade_images_angles: image i at angles[i] (nullptr: `angle` for every image).  `fn`
// names the entry point in messages.
static int run_cascade_images(const char* fn, const pigo_cascade* cc, const pigo_image* images, int nimages, const double* angles, double angle,
                              int min_size, int max_size, double shift_factor, double scale_factor, pigo_det* out, int cap_per_image, int* n_out,
                              unsigned flags, void* stream_) {
  int rc = check_images_args(cc, images, nimages, out, cap_per_image, n_out);
  if (rc) return rc;
  ImagePlans ip;
  std::vector<double> uniform;
  if ((rc = images_prologue(fn, images, nimages, min_size, max_size, shift_factor, scale_factor, stream_, ip)) || nimages == 0) return rc;
  return scan_images_on(const_cast<pigo_cascade*>(cc), default_device(), images, nimages, ip, min_size, max_size, shift_factor, scale_factor,
                        angles_or(angles, angle, nimages, uniform), out, cap_per_image, n_out, flags, stream_);
}

extern "C" {

int pigo_run_cascade_images(const pigo_cascade* cc, const pigo_image* images, int nimages, int min_size, int max_size, double shift_factor,
                            double scale_factor, double angle, pigo_det* out, int cap_per_image, int* n_out, unsigned flags, void* stream_) {
  return run_cascade_images("pigo_run_cascade_images", cc, images, nimages, nullptr, angle, min_size, max_size, shift_factor, scale_factor,
                            out, cap_per_image, n_out, flags, stream_);
}

int pigo_run_cascade_images_angles(const pigo_cascade* cc, const pigo_image* images, int nimages, const double* angles, int min_size,
                                   int max_size, double shift_factor, double scale_factor, pigo_det* out, int cap_per_image, int* n_out,
                                   unsigned flags, void* stream_) {
  if (nimages > 0 && !angles) return set_err(PIGO_E_INVALID, "null angles");
  return run_cascade_images("pigo_run_cascade_images_angles", cc, images, nimages, angles, 0.0, min_size, max_size, shift_factor, scale_factor,
                            out, cap_per_image, n_out, flags, stream_);
}

// Multi-GPU form (SURVEY.md section 8e): HOST frames are sharded over the devices of pigo_init_devices; every device
// scans its shard (no data-path collective), and the per-frame results land in the caller's arrays in frame order, so
// the output equals the single-GPU result exactly.
int pigo_run_cascade_batch_sharded(const pigo_cascade* cc, const uint8_t* frames, int nframes, size_t frame_stride, int rows, int cols,
                                   int dim, int min_size, int max_size, double shift_factor, double scale_factor, double angle,
                                   pigo_det* out, int cap_per_frame, int* n_out) {
  int rc = check_batch_args(cc, frames, nframes, frame_stride, rows, cols, dim, out, cap_per_frame, n_out);
  if (rc) return rc;
  if (nframes == 0) return ensure_device();
  pigo_cascade* c = const_cast<pigo_cascade*>(cc);
  return for_each_shard(nframes, [&](int, int dev, int lo, int n) {
    return scan_batch_on(c, dev, frames + (size_t)lo * frame_stride, n, frame_stride, rows, cols, dim, min_size, max_size, shift_factor,
                         scale_factor, angle, out ? out + (size_t)lo * cap_per_frame : nullptr, cap_per_frame, n_out + lo, PIGO_MEM_HOST, nullptr);
  });
}

// ---- ClusterDetections ---------------------------------------------------------------------------------
static WorkspacePool g_misc_pool[kMaxDevices];   // scratch of the handle-less entry points (cluster, grayscale, ycbcr), per device

// pigo_shutdown: waits for the devices in use and releases the library-owned scratch that is not tied to a handle (cached
// workspaces of the handle-less entry points).  Handles stay valid -- their own scratch goes with pigo_*_destroy -- and the
// library can be used again afterwards.
int pigo_shutdown_impl(void) {
  for (int d = 0; d < kMaxDevices; ++d) {
    if (g_misc_pool[d].free_list.empty()) continue;
    if (cudaSetDevice(d) != cudaSuccess) { cudaGetLastError(); continue; }
    cudaDeviceSynchronize();
    std::lock_guard<std::mutex> g(g_misc_pool[d].mu);
    for (auto* w : g_misc_pool[d].free_list) delete w;
    g_misc_pool[d].free_list.clear();
  }
  const int dev = g_device.load();
  if (dev >= 0) cudaSetDevice(dev);
  return PIGO_OK;
}

static int cluster_batch_on(int dev, pigo_det* dets, const int* n, int nframes, int cap_per_frame, double iou_threshold, pigo_det* out,
                            int out_cap_per_frame, int* n_out, unsigned flags, void* stream_) {
  int rc = use_device(dev);
  if (rc) return rc;
  const bool on_dev = (flags & PIGO_OUT_DEVICE) != 0;  // dets, n, out, n_out all on the device
  Borrow w(g_misc_pool[dev], stream_);
  if (w.rc) return w.rc;
  cudaStream_t st = w.st;
  const int cap = std::max(cap_per_frame, 1), ocap = std::max(out_cap_per_frame, 1);
  const size_t nd = (size_t)nframes * cap;
  if ((rc = w->scratch_a.reserve(nd * sizeof(pigo_det)))) return rc;
  if ((rc = w->scratch_b.reserve(nd))) return rc;
  if ((rc = w->scratch_c.reserve(nd * sizeof(int32_t)))) return rc;
  pigo_det *d_dets = dets, *d_out = out;
  const int32_t* d_n = n;
  int32_t* d_nout = n_out;
  if (!on_dev) {
    if ((rc = w->raw.reserve(nd * sizeof(pigo_det)))) return rc;
    if ((rc = w->out.reserve((size_t)nframes * ocap * sizeof(pigo_det)))) return rc;
    if ((rc = w->nout.reserve((size_t)nframes * 8))) return rc;
    d_dets = (pigo_det*)w->raw.p; d_out = (pigo_det*)w->out.p;
    d_nout = (int32_t*)w->nout.p;
    int32_t* dn = d_nout + nframes;
    d_n = dn;
    if (cap_per_frame > 0 && dets) CUDA_TRY(cudaMemcpyAsync(d_dets, dets, nd * sizeof(pigo_det), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(dn, n, (size_t)nframes * 4, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(d_out, 0, (size_t)nframes * ocap * sizeof(pigo_det), st));   // defined padding in the host copy
  }
  timing_begin(T_CLUSTER, st);
  launch_cluster(d_dets, d_n, cap, iou_threshold, (pigo_det*)w->scratch_a.p, (uint8_t*)w->scratch_b.p, (int32_t*)w->scratch_c.p,
                 d_out, ocap, d_nout, nframes, st);
  timing_end(T_CLUSTER, st);
  g_launches++;
  CUDA_TRY(cudaGetLastError());
  if (on_dev) return ws_leave_async(w, st);
  if (cap_per_frame > 0 && dets) CUDA_TRY(cudaMemcpyAsync(dets, d_dets, nd * sizeof(pigo_det), cudaMemcpyDeviceToHost, st));  // in-place sort
  CUDA_TRY(cudaMemcpyAsync(n_out, d_nout, (size_t)nframes * 4, cudaMemcpyDeviceToHost, st));
  if (out_cap_per_frame > 0 && out)
    CUDA_TRY(cudaMemcpyAsync(out, d_out, (size_t)nframes * ocap * sizeof(pigo_det), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  for (int f = 0; f < nframes; ++f)
    if (n_out[f] > out_cap_per_frame) return set_err(PIGO_E_CAP, "cluster capacity %d too small", out_cap_per_frame);
  return PIGO_OK;
}

int pigo_cluster_batch(pigo_det* dets, const int* n, int nframes, int cap_per_frame, double iou_threshold, pigo_det* out,
                       int out_cap_per_frame, int* n_out, unsigned flags, void* stream_) {
  if (!n || !n_out || nframes < 0) return set_err(PIGO_E_INVALID, "null argument");
  if (cap_per_frame < 0 || out_cap_per_frame < 0) return set_err(PIGO_E_INVALID, "negative capacity");
  int rc = ensure_device();
  if (rc) return rc;
  if (nframes == 0) return PIGO_OK;
  return cluster_batch_on(default_device(), dets, n, nframes, cap_per_frame, iou_threshold, out, out_cap_per_frame, n_out, flags, stream_);
}

int pigo_cluster(pigo_det* dets, int n, double iou_threshold, pigo_det* out, int cap, int* n_out) {
  if (n < 0) return set_err(PIGO_E_INVALID, "negative n");
  if (n == 0) { if (n_out) *n_out = 0; return ensure_device(); }
  return pigo_cluster_batch(dets, &n, 1, n, iou_threshold, out, cap, n_out, PIGO_MEM_HOST, nullptr);
}

// ---- UnpackCascade / RunDetector / GetLandmarkPoint --------------------------------------------------------
int pigo_puploc_create(const uint8_t* packet, size_t len, pigo_puploc** out) {
  if (!packet || !out) return set_err(PIGO_E_INVALID, "null argument");
  if (len < 16) return set_err(PIGO_E_INVALID, "puploc packet shorter than its 16-byte header");
  const uint32_t stages = rd_u32(packet + 0);   // core/puploc.go:51
  float scales; memcpy(&scales, packet + 4, 4); // :55-57
  const uint32_t trees = rd_u32(packet + 8);    // :61
  const uint32_t depth = rd_u32(packet + 12);   // :65
  if (depth < 1 || depth > 16 || stages > 4096 || trees > 65536) return set_err(PIGO_E_INVALID, "implausible puploc header");
  const size_t leaves = (size_t)1 << depth, ncode = 4 * leaves - 4, npred = 2 * leaves;
  const size_t nt = (size_t)stages * trees;
  if (len < 16 + nt * (ncode + npred * 4)) return set_err(PIGO_E_INVALID, "puploc packet truncated");
  int rc = ensure_device();
  if (rc) return rc;
  pigo_puploc* p = new pigo_puploc();
  p->stages = stages; p->trees = trees; p->depth = depth; p->leaves = (uint32_t)leaves; p->scales = scales;
  p->h_codes.resize(nt * ncode + 16);
  p->h_preds.resize(nt * npred + 4);
  size_t pos = 16;
  for (size_t t = 0; t < nt; ++t) {
    memcpy(p->h_codes.data() + t * ncode, packet + pos, ncode); pos += ncode;          // :75-80
    memcpy(p->h_preds.data() + t * npred, packet + pos, npred * 4); pos += npred * 4;  // :83-91
  }
  if (!puploc_replica(p, default_device(), &rc)) { delete p; return rc; }
  *out = p;
  return PIGO_OK;
}

void pigo_puploc_destroy(pigo_puploc* p) { delete p; }

int pigo_puploc_info(const pigo_puploc* p, uint32_t* stages, float* scale_mul, uint32_t* trees, uint32_t* depth) {
  if (!p) return set_err(PIGO_E_INVALID, "null cascade");
  if (stages) *stages = p->stages;
  if (scale_mul) *scale_mul = p->scales;
  if (trees) *trees = p->trees;
  if (depth) *depth = p->depth;
  return PIGO_OK;
}

int pigo_puploc_run(const pigo_puploc* pc, const pigo_point* seeds, int nseeds, const float* randoms, uint64_t rng_seed,
                    const uint8_t* pixels, int rows, int cols, int dim, double angle, const uint8_t* flipv, pigo_point* out,
                    unsigned flags, void* stream_) {
  return pigo_puploc_run_frames(pc, seeds, nseeds, nullptr, randoms, rng_seed, pixels, 1, (size_t)std::max(rows, 0) * (size_t)std::max(dim, 0),
                                rows, cols, dim, angle, flipv, out, flags, stream_);
}

int pigo_puploc_run_frames(const pigo_puploc* pc, const pigo_point* seeds, int nseeds, const int32_t* seed_frame, const float* randoms,
                           uint64_t rng_seed, const uint8_t* pixels, int nframes, size_t frame_stride, int rows, int cols, int dim,
                           double angle, const uint8_t* flipv, pigo_point* out, unsigned flags, void* stream_) {
  pigo_puploc* p = const_cast<pigo_puploc*>(pc);
  if (!p || !seeds || !out || !pixels) return set_err(PIGO_E_INVALID, "null argument");
  if (nseeds < 0 || rows <= 0 || cols <= 0 || dim < cols || nframes < 1) return set_err(PIGO_E_INVALID, "bad geometry");
  if (nframes > 1 && !seed_frame) return set_err(PIGO_E_INVALID, "seed_frame is required when nframes > 1");
  int rc = ensure_device();
  if (rc) return rc;
  if (nseeds == 0) return PIGO_OK;
  bool wide = false;
  if (!(flags & PIGO_OUT_DEVICE) && (rc = check_puploc_seeds(seeds, nseeds, seed_frame, nframes, "frame", &wide))) return rc;
  const PuplocPixels px{pixels, nframes, frame_stride, rows, cols, dim, nullptr};
  return puploc_run_on(p, seeds, nseeds, seed_frame, randoms, rng_seed, px, angle, flipv, out, wide, flags, stream_);
}

int pigo_puploc_run_images(const pigo_puploc* pc, const pigo_point* seeds, int nseeds, const int32_t* seed_image, const float* randoms,
                           uint64_t rng_seed, const pigo_image* images, int nimages, double angle, const uint8_t* flipv, pigo_point* out,
                           unsigned flags, void* stream_) {
  if (nseeds < 0) return set_err(PIGO_E_INVALID, "negative nseeds");
  if (!seeds) return set_err(PIGO_E_INVALID, "null seeds");
  if (!out) return set_err(PIGO_E_INVALID, "null out");
  if (nimages < 1 || nimages > 65535) return set_err(PIGO_E_INVALID, "nimages must be 1..65535");
  if (!images) return set_err(PIGO_E_INVALID, "null images");
  if (nimages > 1 && !seed_image) return set_err(PIGO_E_INVALID, "seed_image is required when nimages > 1");
  int rc = check_image_geometry(images, nimages, 1, true);
  if (rc) return rc;
  bool wide = false;
  if (!(flags & PIGO_OUT_DEVICE) && (rc = check_puploc_seeds(seeds, nseeds, seed_image, nimages, "image", &wide))) return rc;
  if (!pc) return set_err(PIGO_E_INVALID, "null cascade");
  if ((rc = ensure_device())) return rc;
  if (nseeds == 0) return PIGO_OK;
  const PuplocPixels px{nullptr, nimages, 0, 0, 0, 0, images};
  return puploc_run_on(const_cast<pigo_puploc*>(pc), seeds, nseeds, seed_image, randoms, rng_seed, px, angle, flipv, out, wide, flags, stream_);
}

int pigo_get_landmark_point(const pigo_puploc* p, const pigo_point* left_eye, const pigo_point* right_eye, const uint8_t* pixels,
                            int rows, int cols, int dim, int perturb, int flipv, const float* randoms, uint64_t rng_seed,
                            pigo_point* out) {
  if (!left_eye || !right_eye) return set_err(PIGO_E_INVALID, "null argument");
  // core/flploc.go:37-50 (float64 on the host)
  const long long dx = (long long)(left_eye->row - right_eye->row) * (left_eye->row - right_eye->row);
  const long long dy = (long long)(left_eye->col - right_eye->col) * (left_eye->col - right_eye->col);
  const double dist = std::sqrt((double)(dx + dy));
  const double row = (double)(left_eye->row + right_eye->row) / 2.0 + 0.25 * dist;
  const double col = (double)(left_eye->col + right_eye->col) / 2.0 + 0.15 * dist;
  const double scale = 3.0 * dist;
  pigo_point seed;
  seed.row = (int)row; seed.col = (int)col; seed.scale = (float)scale; seed.perturbs = perturb;
  const uint8_t fl = flipv ? 1 : 0;
  return pigo_puploc_run(p, &seed, 1, randoms, rng_seed, pixels, rows, cols, dim, 0.0, &fl, out, PIGO_MEM_HOST, nullptr);
}

}  // extern "C"

// ---- face -> cluster -> pupils -> landmarks on the device (SURVEY.md section 8f row N1) ----------------------------------
// The reference sequences these calls on the host (core/flploc_test.go:75-154, cmd/pigo/main.go:369-565); here one call
// runs RunCascade, ClusterDetections, the eye-seed arithmetic, RunDetector for both eyes of every face, the
// GetLandmarkPoint seed arithmetic and `ncalls` landmark RunDetector calls per face, stream-ordered on the device, with
// one D2H copy of the results at the end.  Only the pixel source differs between the uniform batch and the mixed-size
// call: `scan(w, st, dets, det_cap, cnt, W)` stages the pixels, runs RunCascade into dets[nframes][det_cap] / cnt[nframes]
// on `st`, points W's pixel fields (uniform frames, or the image table) at the pixels the RunDetector stages read and sets
// W.rot_slot to the eye stage's rotation (the call's slot, kRotSlotPerImage or kRotSlotPerFace).  `unit` names a frame in
// the capacity messages.  An angle sweep scans every frame at `nangles` angles: the scan writes nframes*nangles lists
// (frame-major), and `cluster(w, st, dets, det_cap, cnt, clusters, ncl, W, &tags)` turns them into clusters[nframes][face_cap]
// / ncl[nframes]; it may point `tags` at per-face device values that are copied to `face_tags` with the other results.
// ClusterFrames is the one-list-per-frame clustering.
struct ClusterFrames {
  int dev, nframes;
  double iou;
  int face_cap;
  int operator()(Workspace*, cudaStream_t st, pigo_det* d_dets, int det_cap, int32_t* d_cnt, pigo_det* d_clusters, int32_t* d_ncl, PupWork&,
                 int32_t**) const {
    return cluster_batch_on(dev, d_dets, d_cnt, nframes, det_cap, iou, d_clusters, face_cap, d_ncl, PIGO_OUT_DEVICE, st);
  }
};

template <typename ScanFn, typename ClusterFn>
static int detect_on(int dev, pigo_cascade* face, pigo_puploc* puploc, pigo_puploc* const* flp, const uint8_t* flp_flip, int ncalls, int nframes,
                     int nangles, const char* unit, const pigo_pipeline_params& P, const float* randoms, uint64_t rng_seed, uint64_t slot_base,
                     pigo_det* faces, int face_cap, int* n_faces, pigo_point* points, int32_t* face_tags, unsigned flags, void* stream_,
                     ScanFn scan, ClusterFn cluster) {
  int rc = PIGO_OK;
  FaceReplica* R = face_replica(face, dev, &rc);
  if (!R) return rc;
  PuplocReplica* PR = puploc_replica(puploc, dev, &rc);
  if (!PR) return rc;
  const int stride = 2 + ncalls;
  PupWork W{};
  W.ntabs = 1; W.tab[0] = PR->tab;
  std::vector<const pigo_puploc*> seen{puploc};
  for (int cidx = 0; cidx < ncalls; ++cidx) {
    size_t k = 0;
    while (k < seen.size() && seen[k] != flp[cidx]) ++k;
    if (k == seen.size()) {
      if ((int)k >= kMaxPupTabs) return set_err(PIGO_E_INVALID, "more than %d distinct landmark cascades", kMaxPupTabs - 1);
      PuplocReplica* r = puploc_replica(flp[cidx], dev, &rc);
      if (!r) return rc;
      seen.push_back(flp[cidx]);
      W.tab[k] = r->tab; W.ntabs = (int)k + 1;
    }
    W.tab_of[cidx] = (uint8_t)k; W.flip_of[cidx] = flp_flip && flp_flip[cidx] ? 1 : 0;
  }
  if ((rc = use_device(dev))) return rc;
  const bool out_dev = flags & PIGO_OUT_DEVICE;
  const int det_cap = P.det_cap > 0 ? P.det_cap : 2048;

  Borrow w(R->pool, stream_);
  if (w.rc) return w.rc;
  cudaStream_t st = w.st;

  const size_t nslots = (size_t)nframes * face_cap * stride, nscan = (size_t)nframes * nangles;
  // scratch: raw detections + counts, clusters + counts, seeds, points, faces, work counters
  const size_t b_dets = nscan * det_cap * sizeof(pigo_det), b_cl = (size_t)nframes * face_cap * sizeof(pigo_det);
  const size_t b_pts = nslots * sizeof(pigo_point);
  if ((rc = w->raw.reserve(b_dets)) || (rc = w->out.reserve(b_cl + b_cl)) || (rc = w->nout.reserve((nscan + 3 * (size_t)nframes) * 4 + 256)) ||
      (rc = w->scratch_a.reserve(b_pts)) || (rc = w->scratch_b.reserve(b_pts)) || (rc = w->counters.reserve(256))) return rc;
  pigo_det* d_dets = (pigo_det*)w->raw.p;
  pigo_det* d_clusters = (pigo_det*)w->out.p;
  pigo_det* d_faces = out_dev ? faces : (pigo_det*)((char*)w->out.p + b_cl);
  int32_t* d_cnt = (int32_t*)w->nout.p;
  int32_t* d_ncl = d_cnt + nscan;
  int32_t* d_nfaces = out_dev ? n_faces : d_ncl + nframes;
  pigo_point* d_seeds = (pigo_point*)w->scratch_a.p;
  pigo_point* d_points = out_dev ? points : (pigo_point*)w->scratch_b.p;
  const float* d_rnd = randoms;
  if (randoms && !out_dev) {
    const size_t rb = nslots * 63 * 3 * sizeof(float);
    if ((rc = w->scratch_c.reserve(rb))) return rc;
    CUDA_TRY(cudaMemcpyAsync(w->scratch_c.p, randoms, rb, cudaMemcpyHostToDevice, st));
    d_rnd = (const float*)w->scratch_c.p;
  }
  CUDA_TRY(cudaMemsetAsync(w->counters.p, 0, 256, st));
  CUDA_TRY(cudaMemsetAsync(d_points, 0, b_pts, st));

  if ((rc = scan(w, st, d_dets, det_cap, d_cnt, W))) return rc;
  int32_t* d_tags = nullptr;
  if ((rc = cluster(w, st, d_dets, det_cap, d_cnt, d_clusters, d_ncl, W, &d_tags))) return rc;
  timing_begin(T_SEEDS, st);
  launch_eye_seeds(d_clusters, d_ncl, face_cap, nframes, face_cap, stride, P.min_face_scale, P.eye_perturbs, d_faces, d_nfaces, d_seeds, st);
  timing_end(T_SEEDS, st);
  g_launches++;

  W.seeds = d_seeds; W.out = d_points; W.randoms = d_rnd; W.rng_seed = rng_seed; W.slot_base = slot_base;
  W.slot_frame = nullptr; W.flipv = nullptr;
  W.slots_per_frame = face_cap * stride;
  W.stride = stride;
  // (a) both eyes of every face slot, at the scan's angle (a sweep: the face's own angle): RunDetector(puploc, img, det.angle, false), main.go:422
  PupWork E = W;
  E.first = 0; E.span = 2; E.nwork = nframes * face_cap * 2;
  E.tab_of[0] = E.tab_of[1] = 0; E.flip_of[0] = E.flip_of[1] = 0;
  timing_begin(T_PUPLOC, st);
  if (launch_puploc_pairs(E, (unsigned int*)w->counters.p, R->num_sms, st) != 0) return set_err(PIGO_E_INVALID, "pupil cascade has too many trees per stage for the pipeline kernel");
  timing_end(T_PUPLOC, st);
  g_launches++;
  if (ncalls > 0) {
    // (b) landmark seeds from the two eye results (GetLandmarkPoint always passes angle 0.0, core/flploc.go:53-56)
    timing_begin(T_SEEDS, st);
    launch_landmark_seeds(d_points, d_seeds, nframes * face_cap, stride, ncalls, P.flp_perturbs, st);
    timing_end(T_SEEDS, st);
    g_launches++;
    PupWork Lm = W;
    Lm.rot_slot = -1; Lm.first = 2; Lm.span = ncalls; Lm.nwork = nframes * face_cap * ncalls;
    timing_begin(T_PUPLOC, st);
    if (launch_puploc_pairs(Lm, (unsigned int*)w->counters.p + 16, R->num_sms, st) != 0) return set_err(PIGO_E_INVALID, "landmark cascade has too many trees per stage for the pipeline kernel");
    timing_end(T_PUPLOC, st);
    g_launches++;
  }
  CUDA_TRY(cudaGetLastError());
  if (out_dev) return ws_leave_async(w, st);

  // one D2H round: counts (raw detections, clusters), faces, points (and the faces' tags)
  std::vector<int32_t> cnt(nscan + nframes);
  CUDA_TRY(cudaMemcpyAsync(cnt.data(), d_cnt, cnt.size() * 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(n_faces, d_nfaces, (size_t)nframes * 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(faces, d_faces, b_cl, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(points, d_points, b_pts, cudaMemcpyDeviceToHost, st));
  if (face_tags && d_tags) CUDA_TRY(cudaMemcpyAsync(face_tags, d_tags, (size_t)nframes * face_cap * 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  for (size_t e = 0; e < nscan; ++e) {
    if (cnt[e] <= det_cap) continue;
    if (nangles == 1) return set_err(PIGO_E_CAP, "%s %d has %d raw detections, det_cap is %d: raise pigo_pipeline_params.det_cap", unit, (int)e, cnt[e], det_cap);
    return set_err(PIGO_E_CAP, "%s %d at angle %d has %d raw detections, det_cap is %d: raise pigo_pipeline_params.det_cap", unit, (int)(e / nangles),
                   (int)(e % nangles), cnt[e], det_cap);
  }
  for (int f = 0; f < nframes; ++f)
    if (n_faces[f] > face_cap) return set_err(PIGO_E_CAP, "%s %d has %d faces, face_cap is %d", unit, f, n_faces[f], face_cap);
  return PIGO_OK;
}

static int detect_batch_on(int dev, pigo_cascade* face, pigo_puploc* puploc, pigo_puploc* const* flp, const uint8_t* flp_flip, int ncalls,
                           const uint8_t* frames, int nframes, size_t frame_stride, int rows, int cols, int dim, const pigo_pipeline_params& P,
                           const float* randoms, uint64_t rng_seed, uint64_t slot_base, pigo_det* faces, int face_cap, int* n_faces,
                           pigo_point* points, unsigned flags, void* stream_) {
  const bool frames_dev = flags & PIGO_FRAMES_DEVICE;
  auto scan = [&](Workspace* w, cudaStream_t st, pigo_det* d_dets, int det_cap, int32_t* d_cnt, PupWork& W) {
    int rc = PIGO_OK;
    W.frames = frames; W.frame_stride = frame_stride; W.nrows = rows; W.ncols = cols; W.dim = dim;
    W.rot_slot = rot_slot_of(P.angle);
    if (!frames_dev) {
      // the scan call streams the host frames into THIS buffer (chunked copy overlapped with the scan kernels); the
      // pupil / landmark stages gather from it afterwards
      W.frame_stride = ((size_t)rows * dim + 255) & ~(size_t)255;
      if ((rc = w->frames.reserve(W.frame_stride * nframes + 256))) return rc;
      W.frames = (const uint8_t*)w->frames.p;
    }
    return scan_batch_on(face, dev, frames, nframes, frame_stride, rows, cols, dim, P.min_size, P.max_size, P.shift_factor, P.scale_factor,
                         P.angle, d_dets, det_cap, d_cnt, (flags & PIGO_FRAMES_DEVICE) | PIGO_OUT_DEVICE, st,
                         frames_dev ? nullptr : (uint8_t*)w->frames.p);
  };
  return detect_on(dev, face, puploc, flp, flp_flip, ncalls, nframes, 1, "frame", P, randoms, rng_seed, slot_base, faces, face_cap, n_faces, points,
                   nullptr, flags, stream_, scan, ClusterFrames{dev, nframes, P.iou_threshold, face_cap});
}

// Mixed-size form: the images' pixels are staged once (stage_images) and both the images scan and the RunDetector stages
// read them; `ip` holds the call's ladders (build_image_plans).  Image i is scanned and its eyes are refined at angles[i]
// (P.angle is not used).  slot_base offsets the generator key as in detect_batch_on (a shard that starts at image lo of a
// larger call passes lo*face_cap*(2+ncalls)).
static int detect_images_on(int dev, pigo_cascade* face, pigo_puploc* puploc, pigo_puploc* const* flp, const uint8_t* flp_flip, int ncalls,
                            const pigo_image* images, int nimages, const double* angles, const ImagePlans& ip, const pigo_pipeline_params& P,
                            const float* randoms, uint64_t rng_seed, uint64_t slot_base, pigo_det* faces, int face_cap, int* n_faces,
                            pigo_point* points, unsigned flags, void* stream_) {
  const bool frames_dev = flags & PIGO_FRAMES_DEVICE;
  auto scan = [&](Workspace* w, cudaStream_t st, pigo_det* d_dets, int det_cap, int32_t* d_cnt, PupWork& W) {
    std::vector<pigo_image> staged;
    int rc = stage_images(w, images, nimages, angles, frames_dev, st, &W.images, staged);
    if (rc) return rc;
    W.rot_slot = kRotSlotPerImage;
    return scan_images_on(face, dev, staged.data(), nimages, ip, P.min_size, P.max_size, P.shift_factor, P.scale_factor, angles, d_dets,
                          det_cap, d_cnt, PIGO_FRAMES_DEVICE | PIGO_OUT_DEVICE, st);
  };
  return detect_on(dev, face, puploc, flp, flp_flip, ncalls, nimages, 1, "image", P, randoms, rng_seed, slot_base, faces, face_cap, n_faces, points,
                   nullptr, flags, stream_, scan, ClusterFrames{dev, nimages, P.iou_threshold, face_cap});
}

// ---- angle sweep: every image at every angle, merged per image (pigo_run_cascade_images_sweep, pigo_detect_images_sweep) ----
// Entry e = i*nangles + a of a sweep's expanded list is images[i] at angles[a]; the scan writes one raw list per entry.
static void sweep_entries(const pigo_image* images, int nimages, const double* angles, int nangles, std::vector<pigo_image>& ex,
                          std::vector<double>& ex_angles) {
  ex.clear(); ex_angles.clear();
  for (int i = 0; i < nimages; ++i)
    for (int a = 0; a < nangles; ++a) { ex.push_back(images[i]); ex_angles.push_back(angles[a]); }
}

// Image i's clusters of D_i = list(i, 0) ++ ... ++ list(i, nangles-1) (raw lists dets[e][det_cap], cnt[e]), as ClusterDetections
// computes them with a stable sort by Q: out[nimages][out_cap], n_out[nimages] (the required counts), and per cluster the index
// into `angles` of its largest-Q member (*tags: tags_dst if given, else scratch) and that angle's rotation slot (*rot).  All
// on the device, on `st`; the scratch is w->sweep.
static int sweep_merge(Workspace* w, cudaStream_t st, const pigo_det* d_dets, const int32_t* d_cnt, int nimages, const double* angles, int nangles,
                       int det_cap, double iou, pigo_det* d_out, int out_cap, int32_t* d_nout, int32_t* tags_dst, int32_t** tags, int32_t** rot) {
  const int seg_cap = nangles * det_cap;
  const size_t N = (size_t)nimages * seg_cap, nf = (size_t)nimages * out_cap;
  const size_t sort_bytes = sweep_sort_bytes(nimages, seg_cap);
  size_t total = 0;
  auto carve = [&](size_t bytes) { const size_t o = total; total += (bytes + 255) & ~(size_t)255; return o; };
  const size_t o_slot = carve((size_t)nangles * 4), o_seg = carve((size_t)nimages * 12), o_merged = carve(N * sizeof(pigo_det)),
               o_tmp = carve(N * sizeof(pigo_det)), o_tag = carve(N * 4), o_seeds = carve(N * 4), o_flags = carve(N), o_kin = carve(N * 8),
               o_kout = carve(N * 8), o_ftag = carve(nf * 4), o_rot = carve(nf * 4), o_sort = carve(sort_bytes);
  int rc = w->sweep.reserve(total);
  if (rc) return rc;
  uint8_t* b = (uint8_t*)w->sweep.p;
  std::vector<int32_t> slot_of(nangles);
  for (int a = 0; a < nangles; ++a) slot_of[a] = rot_slot_of(angles[a]);
  CUDA_TRY(cudaMemcpyAsync(b + o_slot, slot_of.data(), (size_t)nangles * 4, cudaMemcpyHostToDevice, st));
  SweepScratch S{};
  S.merged = (pigo_det*)(b + o_merged); S.tmp = (pigo_det*)(b + o_tmp); S.tag = (int32_t*)(b + o_tag); S.seeds = (int32_t*)(b + o_seeds);
  S.flags = b + o_flags; S.keys_in = (uint64_t*)(b + o_kin); S.keys_out = (uint64_t*)(b + o_kout);
  S.seg_begin = (int32_t*)(b + o_seg); S.seg_end = S.seg_begin + nimages; S.n_merged = S.seg_end + nimages;
  S.sort_temp = b + o_sort; S.sort_bytes = sort_bytes;
  *tags = tags_dst ? tags_dst : (int32_t*)(b + o_ftag);
  *rot = (int32_t*)(b + o_rot);
  timing_begin(T_MERGE, st);
  if (launch_sweep_merge(d_dets, d_cnt, nimages, nangles, det_cap, iou, S, (const int32_t*)(b + o_slot), d_out, out_cap, d_nout, *tags, *rot, st))
    return set_err(PIGO_E_CUDA, "segmented sort of the sweep failed");
  timing_end(T_MERGE, st);
  g_launches += 3;
  CUDA_TRY(cudaGetLastError());
  return PIGO_OK;
}

// Raw-list capacity of a sweep: entry e = i*nangles + a holds more than det_cap detections.
static int sweep_raw_cap(const int32_t* cnt, int nimages, int nangles, int det_cap, const char* what) {
  for (int e = 0; e < nimages * nangles; ++e)
    if (cnt[e] > det_cap)
      return set_err(PIGO_E_CAP, "image %d at angle %d has %d raw detections, det_cap is %d: raise %s", e / nangles, e % nangles, cnt[e], det_cap, what);
  return PIGO_OK;
}

// ex / ex_angles: the expanded list (sweep_entries), ip: its ladders.
static int sweep_scan_on(pigo_cascade* c, int dev, const pigo_image* ex, const double* ex_angles, int nimages, const double* angles, int nangles,
                         const ImagePlans& ip, int min_size, int max_size, double shift_factor, double scale_factor, double iou, int det_cap,
                         pigo_det* out, int32_t* angle_index, int cap_per_image, int* n_out, unsigned flags, void* stream_) {
  int rc = PIGO_OK;
  FaceReplica* R = face_replica(c, dev, &rc);
  if (!R) return rc;
  if ((rc = use_device(dev))) return rc;
  const bool out_dev = flags & PIGO_OUT_DEVICE;
  Borrow w(R->pool, stream_);
  if (w.rc) return w.rc;
  cudaStream_t st = w.st;
  const int E = nimages * nangles, ocap = std::max(cap_per_image, 1);
  if ((rc = w->raw.reserve((size_t)E * det_cap * sizeof(pigo_det))) || (rc = w->nout.reserve(((size_t)E + nimages) * 4))) return rc;
  pigo_det* d_raw = (pigo_det*)w->raw.p;
  int32_t* d_cnt = (int32_t*)w->nout.p;
  if ((rc = scan_images_on(c, dev, ex, E, ip, min_size, max_size, shift_factor, scale_factor, ex_angles, d_raw, det_cap, d_cnt,
                           (flags & PIGO_FRAMES_DEVICE) | PIGO_OUT_DEVICE, st)))
    return rc;
  pigo_det* d_out = out;
  int32_t* d_nout = n_out;
  if (!out_dev) {
    if ((rc = w->out.reserve((size_t)nimages * ocap * sizeof(pigo_det)))) return rc;
    d_out = (pigo_det*)w->out.p;
    d_nout = d_cnt + E;
    CUDA_TRY(cudaMemsetAsync(d_out, 0, (size_t)nimages * ocap * sizeof(pigo_det), st));   // defined padding in the host copy
  }
  int32_t *d_tags = nullptr, *d_rot = nullptr;
  if ((rc = sweep_merge(w, st, d_raw, d_cnt, nimages, angles, nangles, det_cap, iou, d_out, ocap, d_nout, out_dev ? angle_index : nullptr, &d_tags,
                        &d_rot)))
    return rc;
  if (out_dev) return ws_leave_async(w, st);
  // d_cnt holds the E raw-list counts, then (d_nout = d_cnt + E) the clusters': one copy brings both back.  The raw-list
  // error wins over the cluster-capacity error, whose message this function words itself.
  std::vector<int32_t> cnt((size_t)E + nimages);
  rc = copy_results_to_host(d_out, d_cnt, ocap, nimages, out, cap_per_image, n_out, st, d_tags, angle_index, E, cnt.data());
  if (rc != PIGO_OK && rc != PIGO_E_CAP) return rc;
  if ((rc = sweep_raw_cap(cnt.data(), nimages, nangles, det_cap, "det_cap"))) return rc;
  for (int i = 0; i < nimages; ++i)
    if (n_out[i] > cap_per_image) return set_err(PIGO_E_CAP, "image %d has %d clusters, cap_per_image is %d", i, n_out[i], cap_per_image);
  return PIGO_OK;
}

// Pipeline form: the images' pixels are staged once (stage_images); the scan reads them at every angle and the eye and
// landmark stages through the call's ImageDesc table.  The eyes of face k of image i are refined at angles[tag], tag being
// the face's angle index (kRotSlotPerFace); the generator key and randoms layout are pigo_detect_images'.
static int detect_sweep_on(int dev, pigo_cascade* face, pigo_puploc* puploc, pigo_puploc* const* flp, const uint8_t* flp_flip, int ncalls,
                           const pigo_image* images, int nimages, const double* angles, int nangles, const ImagePlans& ip,
                           const pigo_pipeline_params& P, const float* randoms, uint64_t rng_seed, pigo_det* faces, int face_cap, int* n_faces,
                           pigo_point* points, int32_t* face_angle, unsigned flags, void* stream_) {
  const bool frames_dev = flags & PIGO_FRAMES_DEVICE, out_dev = flags & PIGO_OUT_DEVICE;
  auto scan = [&](Workspace* w, cudaStream_t st, pigo_det* d_dets, int det_cap, int32_t* d_cnt, PupWork& W) {
    std::vector<pigo_image> staged, ex;
    std::vector<double> ex_angles;
    int rc = stage_images(w, images, nimages, nullptr, frames_dev, st, &W.images, staged);
    if (rc) return rc;
    W.rot_slot = kRotSlotPerFace;
    sweep_entries(staged.data(), nimages, angles, nangles, ex, ex_angles);
    return scan_images_on(face, dev, ex.data(), nimages * nangles, ip, P.min_size, P.max_size, P.shift_factor, P.scale_factor, ex_angles.data(),
                          d_dets, det_cap, d_cnt, PIGO_FRAMES_DEVICE | PIGO_OUT_DEVICE, st);
  };
  auto cluster = [&](Workspace* w, cudaStream_t st, pigo_det* d_dets, int det_cap, int32_t* d_cnt, pigo_det* d_clusters, int32_t* d_ncl, PupWork& W,
                     int32_t** d_tags) {
    int32_t* rot = nullptr;
    const int rc = sweep_merge(w, st, d_dets, d_cnt, nimages, angles, nangles, det_cap, P.iou_threshold, d_clusters, face_cap, d_ncl,
                               out_dev ? face_angle : nullptr, d_tags, &rot);
    W.face_rot = rot;
    return rc;
  };
  return detect_on(dev, face, puploc, flp, flp_flip, ncalls, nimages, nangles, "image", P, randoms, rng_seed, 0, faces, face_cap, n_faces, points,
                   face_angle, flags, stream_, scan, cluster);
}

// Extent of the planes image.YCbCr holds for Rect (min)-(min + size), min >= 0: bytes from the rectangle's origin to its
// last sample in the Y plane and in each chroma plane (COffset rows and columns per ratio), and the rectangle's chroma width.
struct YCbCrExtent {
  size_t y_bytes, c_bytes;
  int c_cols;
};
static YCbCrExtent ycbcr_extent(int subsample, int min_x, int min_y, int width, int height, int y_stride, int c_stride) {
  const int xs = chroma_xshift(subsample), ys = chroma_yshift(subsample);
  const int c_rows = ((min_y + height - 1) >> ys) - (min_y >> ys) + 1, c_cols = ((min_x + width - 1) >> xs) - (min_x >> xs) + 1;
  return YCbCrExtent{(size_t)(height - 1) * y_stride + width, (size_t)(c_rows - 1) * c_stride + c_cols, c_cols};
}

// Host bytes of plane k of a decoded source from its rectangle's origin to its last sample (0: the format has no plane k).
// A Paletted source's plane 1 is its palette of stride[1] 4-byte entries.
static size_t decoded_plane_bytes(const pigo_decoded& d, int k) {
  if (d.format == PIGO_DECODED_YCBCR) {
    const YCbCrExtent e = ycbcr_extent(d.subsample, d.min_x, d.min_y, d.width, d.height, d.stride[0], d.stride[1]);
    return k == 0 ? e.y_bytes : e.c_bytes;
  }
  if (d.format == PIGO_DECODED_PALETTED && k == 1) return (size_t)4 * d.stride[1];
  return k == 0 ? (size_t)(d.height - 1) * d.stride[0] + (size_t)d.width * decoded_bpp(d.format) : 0;
}

static int check_decoded(const pigo_decoded* src, int n) {
  for (int i = 0; i < n; ++i) {
    const pigo_decoded& d = src[i];
    if (d.format < PIGO_DECODED_YCBCR || d.format > PIGO_DECODED_PALETTED || d.format == 4)
      return set_err(PIGO_E_INVALID, "source %d: unknown format %d", i, d.format);
    if (d.width < 1 || d.height < 1) return set_err(PIGO_E_INVALID, "source %d: bad size %dx%d", i, d.width, d.height);
    if ((uint64_t)d.width * (uint64_t)d.height > 0x7fffffffull) return set_err(PIGO_E_INVALID, "source %d: 2^31 pixels or more", i);
    const bool ycc = d.format == PIGO_DECODED_YCBCR;
    if (ycc && (d.subsample < 0 || d.subsample > 5))
      return set_err(PIGO_E_INVALID, "source %d: unknown YCbCr subsample ratio %d (0..5 = 444, 422, 420, 440, 411, 410)", i, d.subsample);
    if (ycc && (d.min_x < 0 || d.min_y < 0)) return set_err(PIGO_E_INVALID, "source %d: negative rectangle origin", i);
    if (!d.plane[0] || (ycc && (!d.plane[1] || !d.plane[2]))) return set_err(PIGO_E_INVALID, "source %d: null plane", i);
    if ((int64_t)d.stride[0] < (int64_t)d.width * decoded_bpp(d.format)) return set_err(PIGO_E_INVALID, "source %d: stride %d below the row", i, d.stride[0]);
    if (ycc && d.stride[1] < ycbcr_extent(d.subsample, d.min_x, d.min_y, d.width, d.height, d.stride[0], d.stride[1]).c_cols)
      return set_err(PIGO_E_INVALID, "source %d: chroma stride %d below the chroma row", i, d.stride[1]);
    if (d.format == PIGO_DECODED_PALETTED && !d.plane[1]) return set_err(PIGO_E_INVALID, "source %d: null palette", i);
    if (d.format == PIGO_DECODED_PALETTED && (d.stride[1] < 1 || d.stride[1] > 256))
      return set_err(PIGO_E_INVALID, "source %d: palette length %d outside 1..256", i, d.stride[1]);
  }
  return PIGO_OK;
}

// The landmark cascade handles flp[0..ncalls) of a pipeline call.
static int check_landmarks(const pigo_puploc* const* flp, int ncalls) {
  for (int i = 0; i < ncalls; ++i)
    if (!flp[i]) return set_err(PIGO_E_INVALID, "null landmark cascade %d", i);
  return PIGO_OK;
}

// The pipeline parameters of the pigo_detect_* calls: ncalls, the flp array (and, with `handles`, its entries), face_cap and
// the Perturbs of prm (not null).
static int check_pipeline_params(int ncalls, const pigo_puploc* const* flp, bool handles, int face_cap, const pigo_pipeline_params& prm) {
  if (ncalls < 0 || ncalls > 30) return set_err(PIGO_E_INVALID, "ncalls must be 0..30");
  if (ncalls > 0 && !flp) return set_err(PIGO_E_INVALID, "null flp");
  int rc = PIGO_OK;
  if (handles && (rc = check_landmarks(flp, ncalls))) return rc;
  if (face_cap < 1 || face_cap > 4096) return set_err(PIGO_E_INVALID, "face_cap must be 1..4096");
  if (prm.eye_perturbs < 0 || prm.eye_perturbs > 63 || prm.flp_perturbs < 0 || prm.flp_perturbs > 63)
    return set_err(PIGO_E_INVALID, "Perturbs outside 0..63 (the reference panics, core/puploc.go:261)");
  return PIGO_OK;
}

extern "C" {

static int check_detect_args(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, int ncalls, const uint8_t* frames,
                             int nframes, size_t frame_stride, int rows, int cols, int dim, const pigo_pipeline_params* prm,
                             const pigo_det* faces, int face_cap, const int* n_faces, const pigo_point* points) {
  if (!face || !puploc || !prm || !faces || !n_faces || !points || (ncalls > 0 && !flp)) return set_err(PIGO_E_INVALID, "null argument");
  const int rc = check_pipeline_params(ncalls, flp, true, face_cap, *prm);
  if (rc) return rc;
  if (rows <= 0 || cols <= 0) return set_err(PIGO_E_INVALID, "bad geometry");
  return check_batch_args(face, frames, nframes, frame_stride, rows, cols, dim, faces, face_cap, n_faces);
}

int pigo_detect_batch(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, const uint8_t* flp_flip, int ncalls,
                      const uint8_t* frames, int nframes, size_t frame_stride, int rows, int cols, int dim, const pigo_pipeline_params* prm,
                      const float* randoms, uint64_t rng_seed, pigo_det* faces, int face_cap, int* n_faces, pigo_point* points,
                      unsigned flags, void* stream) {
  int rc = check_detect_args(face, puploc, flp, ncalls, frames, nframes, frame_stride, rows, cols, dim, prm, faces, face_cap, n_faces, points);
  if (rc) return rc;
  if ((rc = ensure_device())) return rc;
  if (nframes == 0) return PIGO_OK;
  return detect_batch_on(default_device(), const_cast<pigo_cascade*>(face), const_cast<pigo_puploc*>(puploc), (pigo_puploc* const*)flp, flp_flip,
                         ncalls, frames, nframes, frame_stride, rows, cols, dim, *prm, randoms, rng_seed, 0, faces, face_cap, n_faces, points, flags, stream);
}

int pigo_detect_batch_sharded(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, const uint8_t* flp_flip, int ncalls,
                              const uint8_t* frames, int nframes, size_t frame_stride, int rows, int cols, int dim, const pigo_pipeline_params* prm,
                              const float* randoms, uint64_t rng_seed, pigo_det* faces, int face_cap, int* n_faces, pigo_point* points) {
  int rc = check_detect_args(face, puploc, flp, ncalls, frames, nframes, frame_stride, rows, cols, dim, prm, faces, face_cap, n_faces, points);
  if (rc) return rc;
  if (nframes == 0) return ensure_device();
  const size_t per_frame = (size_t)face_cap * (2 + ncalls);
  return for_each_shard(nframes, [&](int, int dev, int lo, int n) {
    return detect_batch_on(dev, const_cast<pigo_cascade*>(face), const_cast<pigo_puploc*>(puploc), (pigo_puploc* const*)flp, flp_flip, ncalls,
                           frames + (size_t)lo * frame_stride, n, frame_stride, rows, cols, dim, *prm,
                           randoms ? randoms + (size_t)lo * per_frame * 189 : nullptr, rng_seed, (uint64_t)lo * per_frame,
                           faces + (size_t)lo * face_cap, face_cap, n_faces + lo, points + (size_t)lo * per_frame, PIGO_MEM_HOST, nullptr);
  });
}

// Mixed-size pipeline arguments: what check_images_args and check_detect_args check except the uniform geometry, with a
// message that names the argument; the cascade handles last, so that every other check is reachable without a device.
static int check_detect_images_args(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, int ncalls,
                                    const pigo_image* images, int nimages, const pigo_pipeline_params* prm, const pigo_det* faces, int face_cap,
                                    const int* n_faces, const pigo_point* points) {
  if (nimages < 0 || nimages > 65535) return set_err(PIGO_E_INVALID, "nimages must be 0..65535");
  if (nimages > 0 && !images) return set_err(PIGO_E_INVALID, "null images");
  if (!prm) return set_err(PIGO_E_INVALID, "null params");
  if (!faces) return set_err(PIGO_E_INVALID, "null faces");
  if (!n_faces) return set_err(PIGO_E_INVALID, "null n_faces");
  if (!points) return set_err(PIGO_E_INVALID, "null points");
  int rc = check_pipeline_params(ncalls, flp, false, face_cap, *prm);
  if (rc) return rc;
  if ((uint64_t)nimages * (uint64_t)face_cap * (uint64_t)(2 + ncalls) > 0x7fffffffull)
    return set_err(PIGO_E_INVALID, "nimages*face_cap*(2+ncalls) exceeds 2^31-1 pupil work items");
  if ((rc = check_image_geometry(images, nimages, 1, true))) return rc;
  if (!face) return set_err(PIGO_E_INVALID, "null cascade");
  if (!puploc) return set_err(PIGO_E_INVALID, "null pupil cascade");
  return check_landmarks(flp, ncalls);
}

// pigo_detect_images and pigo_detect_images_angles: image i at angles[i] (nullptr: prm->angle for every image).  `fn`
// names the entry point in messages.
static int detect_images(const char* fn, const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, const uint8_t* flp_flip,
                         int ncalls, const pigo_image* images, int nimages, const double* angles, const pigo_pipeline_params* prm,
                         const float* randoms, uint64_t rng_seed, pigo_det* faces, int face_cap, int* n_faces, pigo_point* points, unsigned flags,
                         void* stream) {
  int rc = check_detect_images_args(face, puploc, flp, ncalls, images, nimages, prm, faces, face_cap, n_faces, points);
  if (rc) return rc;
  ImagePlans ip;
  std::vector<double> uniform;
  if ((rc = images_prologue(fn, images, nimages, prm->min_size, prm->max_size, prm->shift_factor, prm->scale_factor, stream, ip)) || nimages == 0)
    return rc;
  return detect_images_on(default_device(), const_cast<pigo_cascade*>(face), const_cast<pigo_puploc*>(puploc), (pigo_puploc* const*)flp, flp_flip,
                          ncalls, images, nimages, angles_or(angles, prm->angle, nimages, uniform), ip, *prm, randoms, rng_seed, 0, faces, face_cap,
                          n_faces, points, flags, stream);
}

int pigo_detect_images(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, const uint8_t* flp_flip, int ncalls,
                       const pigo_image* images, int nimages, const pigo_pipeline_params* prm, const float* randoms, uint64_t rng_seed,
                       pigo_det* faces, int face_cap, int* n_faces, pigo_point* points, unsigned flags, void* stream) {
  return detect_images("pigo_detect_images", face, puploc, flp, flp_flip, ncalls, images, nimages, nullptr, prm, randoms, rng_seed, faces, face_cap,
                       n_faces, points, flags, stream);
}

int pigo_detect_images_angles(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, const uint8_t* flp_flip,
                              int ncalls, const pigo_image* images, int nimages, const double* angles, const pigo_pipeline_params* prm,
                              const float* randoms, uint64_t rng_seed, pigo_det* faces, int face_cap, int* n_faces, pigo_point* points,
                              unsigned flags, void* stream) {
  if (nimages > 0 && !angles) return set_err(PIGO_E_INVALID, "null angles");
  return detect_images("pigo_detect_images_angles", face, puploc, flp, flp_flip, ncalls, images, nimages, angles, prm, randoms, rng_seed, faces,
                       face_cap, n_faces, points, flags, stream);
}

// Sweep arguments checked before the per-image ones: the angle list and the size of the expanded list (det_cap > 0).
static int check_sweep_args(int nimages, const double* angles, int nangles) {
  if (!angles) return set_err(PIGO_E_INVALID, "null angles");
  if (nangles < 1) return set_err(PIGO_E_INVALID, "nangles must be >= 1");
  if (nimages > 0 && (uint64_t)nimages * (uint64_t)nangles > 65535)
    return set_err(PIGO_E_INVALID, "nimages*nangles = %llu scan entries exceeds 65535", (unsigned long long)nimages * nangles);
  return PIGO_OK;
}
static int check_sweep_merge(int nimages, int nangles, int det_cap) {
  if (nimages > 0 && (uint64_t)nimages * (uint64_t)nangles * (uint64_t)det_cap > 0x7fffffffull)
    return set_err(PIGO_E_INVALID, "nimages*nangles*det_cap exceeds 2^31-1 merged detections");
  return PIGO_OK;
}

int pigo_run_cascade_images_sweep(const pigo_cascade* cc, const pigo_image* images, int nimages, const double* angles, int nangles, int min_size,
                                  int max_size, double shift_factor, double scale_factor, double iou_threshold, int det_cap, pigo_det* out,
                                  int32_t* angle_index, int cap_per_image, int* n_out, unsigned flags, void* stream_) {
  int rc = check_sweep_args(nimages, angles, nangles);
  if (rc) return rc;
  if (det_cap < 0) return set_err(PIGO_E_INVALID, "negative det_cap");
  const int dcap = det_cap > 0 ? det_cap : 2048;
  if ((rc = check_sweep_merge(nimages, nangles, dcap))) return rc;
  if ((rc = check_images_args(cc, images, nimages, out, cap_per_image, n_out))) return rc;
  std::vector<pigo_image> ex;
  std::vector<double> ex_angles;
  sweep_entries(images, nimages, angles, nangles, ex, ex_angles);
  ImagePlans ip;
  if ((rc = images_prologue("pigo_run_cascade_images_sweep", ex.data(), (int)ex.size(), min_size, max_size, shift_factor, scale_factor, stream_,
                            ip)) || nimages == 0)
    return rc;
  return sweep_scan_on(const_cast<pigo_cascade*>(cc), default_device(), ex.data(), ex_angles.data(), nimages, angles, nangles, ip, min_size,
                       max_size, shift_factor, scale_factor, iou_threshold, dcap, out, angle_index, cap_per_image, n_out, flags, stream_);
}

int pigo_detect_images_sweep(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, const uint8_t* flp_flip, int ncalls,
                             const pigo_image* images, int nimages, const double* angles, int nangles, const pigo_pipeline_params* prm,
                             const float* randoms, uint64_t rng_seed, pigo_det* faces, int32_t* face_angle, int face_cap, int* n_faces,
                             pigo_point* points, unsigned flags, void* stream) {
  int rc = check_sweep_args(nimages, angles, nangles);
  if (rc) return rc;
  if (prm && (rc = check_sweep_merge(nimages, nangles, prm->det_cap > 0 ? prm->det_cap : 2048))) return rc;
  if ((rc = check_detect_images_args(face, puploc, flp, ncalls, images, nimages, prm, faces, face_cap, n_faces, points))) return rc;
  std::vector<pigo_image> ex;
  std::vector<double> ex_angles;
  sweep_entries(images, nimages, angles, nangles, ex, ex_angles);
  ImagePlans ip;
  if ((rc = images_prologue("pigo_detect_images_sweep", ex.data(), (int)ex.size(), prm->min_size, prm->max_size, prm->shift_factor,
                            prm->scale_factor, stream, ip)) || nimages == 0)
    return rc;
  return detect_sweep_on(default_device(), const_cast<pigo_cascade*>(face), const_cast<pigo_puploc*>(puploc), (pigo_puploc* const*)flp, flp_flip,
                         ncalls, images, nimages, angles, nangles, ip, *prm, randoms, rng_seed, faces, face_cap, n_faces, points, face_angle,
                         flags, stream);
}

// ---- RgbToGrayscale, core/grayscale.go:8-23 ----------------------------------------------------------------
int pigo_rgba_to_gray(const uint8_t* rgba, size_t npixels, uint8_t* gray, unsigned flags, void* stream_) {
  if (npixels == 0) return ensure_device();
  if (!rgba || !gray) return set_err(PIGO_E_INVALID, "null argument");
  int rc = ensure_device();
  if (rc) return rc;
  const int dev = default_device();
  Borrow w(g_misc_pool[dev], stream_);   // a device-output call returns while the kernel still reads the staging buffer
  if (w.rc) return w.rc;
  cudaStream_t st = w.st;
  const bool in_dev = flags & PIGO_FRAMES_DEVICE, out_dev = flags & PIGO_OUT_DEVICE;
  const uint8_t* d_in = rgba;
  uint8_t* d_out = gray;
  if (!in_dev) {
    if ((rc = w->frames.reserve(npixels * 4))) return rc;
    CUDA_TRY(cudaMemcpyAsync(w->frames.p, rgba, npixels * 4, cudaMemcpyHostToDevice, st));
    d_in = (const uint8_t*)w->frames.p;
  }
  if (!out_dev) {
    if ((rc = w->out.reserve(npixels))) return rc;
    d_out = (uint8_t*)w->out.p;
  }
  const size_t want = (npixels / 16 + 255) / 256 + 1;
  const int grid = (int)std::min<size_t>(want, (size_t)device_sms(dev) * 16);
  timing_begin(T_GRAY, st);
  launch_gray(d_in, npixels, d_out, grid, st);
  timing_end(T_GRAY, st);
  g_launches++;
  CUDA_TRY(cudaGetLastError());
  if (out_dev) return PIGO_OK;
  CUDA_TRY(cudaMemcpyAsync(gray, d_out, npixels, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return PIGO_OK;
}

// ---- ImgToNRGBA for *image.YCbCr, core/image.go:60-76 (section 8f row N3) ------------------------------------------------
int pigo_ycbcr_to_nrgba(const uint8_t* y, const uint8_t* cb, const uint8_t* cr, int y_stride, int c_stride, int subsample, int min_x, int min_y,
                        int width, int height, uint8_t* nrgba, uint8_t* gray, unsigned flags, void* stream_) {
  if (width < 0 || height < 0 || y_stride < 0 || c_stride < 0) return set_err(PIGO_E_INVALID, "bad geometry");
  if (subsample < 0 || subsample > 5) return set_err(PIGO_E_INVALID, "unknown YCbCr subsample ratio %d (0..5 = 444, 422, 420, 440, 411, 410)", subsample);
  if (min_x < 0 || min_y < 0) return set_err(PIGO_E_INVALID, "negative rectangle origin");
  const size_t npix = (size_t)width * height;
  if (npix == 0) return ensure_device();
  if (npix > 0x7fffffffull) return set_err(PIGO_E_INVALID, "images larger than 2^31 pixels are not supported");
  if (!y || !cb || !cr || (!nrgba && !gray)) return set_err(PIGO_E_INVALID, "null argument");
  int rc = ensure_device();
  if (rc) return rc;
  const int dev = default_device();
  Borrow w(g_misc_pool[dev], stream_);
  if (w.rc) return w.rc;
  cudaStream_t st = w.st;
  const bool in_dev = flags & PIGO_FRAMES_DEVICE, out_dev = flags & PIGO_OUT_DEVICE;
  const uint8_t *d_y = y, *d_cb = cb, *d_cr = cr;
  if (!in_dev) {
    const YCbCrExtent e = ycbcr_extent(subsample, min_x, min_y, width, height, y_stride, c_stride);
    const size_t y_bytes = e.y_bytes, c_bytes = e.c_bytes;
    const size_t yo = (y_bytes + 255) & ~(size_t)255, co = (c_bytes + 255) & ~(size_t)255;
    if ((rc = w->frames.reserve(yo + 2 * co))) return rc;
    uint8_t* b = (uint8_t*)w->frames.p;
    CUDA_TRY(cudaMemcpyAsync(b, y, y_bytes, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(b + yo, cb, c_bytes, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(b + yo + co, cr, c_bytes, cudaMemcpyHostToDevice, st));
    d_y = b; d_cb = b + yo; d_cr = b + yo + co;
  }
  uint8_t *d_rgba = nrgba, *d_gray = gray;
  if (!out_dev) {
    if ((rc = w->out.reserve(npix * 5 + 256))) return rc;
    d_rgba = nrgba ? (uint8_t*)w->out.p : nullptr;
    d_gray = gray ? (uint8_t*)w->out.p + ((npix * 4 + 255) & ~(size_t)255) : nullptr;
  }
  timing_begin(T_YCBCR, st);
  launch_ycbcr(d_y, d_cb, d_cr, y_stride, c_stride, subsample, min_x, min_y, width, height, d_rgba, d_gray, device_sms(dev) * 16, st);
  timing_end(T_YCBCR, st);
  g_launches++;
  CUDA_TRY(cudaGetLastError());
  if (out_dev) return PIGO_OK;
  if (nrgba) CUDA_TRY(cudaMemcpyAsync(nrgba, d_rgba, npix * 4, cudaMemcpyDeviceToHost, st));
  if (gray) CUDA_TRY(cudaMemcpyAsync(gray, d_gray, npix, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return PIGO_OK;
}

}  // extern "C"

// ---- RgbToGrayscale(ImgToNRGBA(img)) for a batch of decoded images, core/grayscale.go:8-23 + core/image.go:35-90 -----------
// The distinct sources of src (first[i], arena_layout) into their slots gray + off[i] on device dev: one kernel launch for
// the YCbCr, NRGBA, RGBA and Gray sources and one for the other formats, each made only when the call has such sources.
// With stream_ NULL the slots are complete on return; on a caller's stream only the host planes' copies are.
static int gray_images_on(int dev, const pigo_decoded* src, int n, const std::vector<size_t>& off, const std::vector<char>& first, uint8_t* gray,
                          unsigned flags, void* stream_) {
  int rc = use_device(dev);
  if (rc) return rc;
  Borrow w(g_misc_pool[dev], stream_);
  if (w.rc) return w.rc;
  cudaStream_t st = w.st;
  const bool in_dev = flags & PIGO_FRAMES_DEVICE;

  // the distinct sources, the ones gray_images_kernel<false> converts first (nnarrow of them); host planes go to one
  // staging buffer, each plane 256-byte aligned
  std::vector<int> who;
  for (int wide = 0; wide < 2; ++wide)
    for (int i = 0; i < n; ++i)
      if (first[i] && decoded_wide(src[i].format) == (wide == 1)) who.push_back(i);
  const int ns = (int)who.size();
  int nnarrow = 0;
  while (nnarrow < ns && !decoded_wide(src[who[nnarrow]].format)) ++nnarrow;
  std::vector<size_t> stage_off((size_t)ns * 3, 0);
  size_t stage_bytes = 0;
  if (!in_dev) {
    for (int k = 0; k < ns; ++k)
      for (int p = 0; p < 3; ++p) {
        stage_off[(size_t)k * 3 + p] = stage_bytes;
        stage_bytes += (decoded_plane_bytes(src[who[k]], p) + 255) & ~(size_t)255;
      }
    if ((rc = w->frames.reserve(stage_bytes + 256))) return rc;
  }
  std::vector<GraySrc> tab(ns);
  // each kernel's work range starts at 0: firsts[0..nnarrow] for the first kernel, firsts[nnarrow+1..ns+1] for the second
  std::vector<uint64_t> firsts(ns + 2, 0);
  for (int k = 0; k < ns; ++k) {
    const pigo_decoded& d = src[who[k]];
    GraySrc& t = tab[k];
    for (int p = 0; p < 3; ++p)
      t.plane[p] = !in_dev && decoded_plane_bytes(d, p) ? (const uint8_t*)w->frames.p + stage_off[(size_t)k * 3 + p] : d.plane[p];
    t.dst = gray + off[who[k]];
    t.format = d.format; t.sub = d.subsample; t.min_x = d.min_x; t.min_y = d.min_y; t.width = d.width; t.height = d.height;
    t.stride0 = d.stride[0]; t.stride1 = d.stride[1];
    const int at = k < nnarrow ? k : k + 1;
    firsts[at + 1] = firsts[at] + (uint64_t)d.height * (uint64_t)((d.width + 15) / 16);
  }
  const size_t tab_bytes = ((size_t)ns * sizeof(GraySrc) + 255) & ~(size_t)255;
  std::vector<uint8_t> blob(tab_bytes + firsts.size() * sizeof(uint64_t));
  memcpy(blob.data(), tab.data(), (size_t)ns * sizeof(GraySrc));
  memcpy(blob.data() + tab_bytes, firsts.data(), firsts.size() * sizeof(uint64_t));
  if ((rc = w->img_tab.reserve(blob.size()))) return rc;
  if (!in_dev) {
    for (int k = 0; k < ns; ++k)
      for (int p = 0; p < 3; ++p) {
        const size_t b = decoded_plane_bytes(src[who[k]], p);
        if (b) CUDA_TRY(cudaMemcpyAsync((uint8_t*)w->frames.p + stage_off[(size_t)k * 3 + p], src[who[k]].plane[p], b, cudaMemcpyHostToDevice, st));
      }
  }
  cudaEvent_t copied = nullptr;
  if (!in_dev && stream_) {   // host planes are the caller's again once their copies are done; the kernel may still run
    if (!(copied = w->copy_event(0))) return set_err(PIGO_E_CUDA, "event creation failed");
    CUDA_TRY(cudaEventRecord(copied, st));
  }
  CUDA_TRY(cudaMemcpyAsync(w->img_tab.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
  const GraySrc* d_tab = (const GraySrc*)w->img_tab.p;
  const uint64_t* d_first = (const uint64_t*)((const uint8_t*)w->img_tab.p + tab_bytes);
  timing_begin(T_GRAY_IMAGES, st);
  if (nnarrow > 0) {
    launch_gray_images(d_tab, d_first, nnarrow, firsts[nnarrow], false, device_sms(dev) * 16, st);
    g_launches++;
  }
  if (ns > nnarrow) {
    launch_gray_images(d_tab + nnarrow, d_first + nnarrow + 1, ns - nnarrow, firsts[ns + 1], true, device_sms(dev) * 16, st);
    g_launches++;
  }
  timing_end(T_GRAY_IMAGES, st);
  CUDA_TRY(cudaGetLastError());
  if (!stream_) CUDA_TRY(cudaStreamSynchronize(st));   // the library's own stream: the arena is complete on return
  else if (copied) CUDA_TRY(cudaEventSynchronize(copied));
  return PIGO_OK;
}

extern "C" {

// One slot per distinct source in the caller's device arena (arena_layout), converted by gray_images_on.
int pigo_gray_images(const pigo_decoded* src, int n, uint8_t* gray, size_t* gray_bytes, pigo_image* images, unsigned flags, void* stream_) {
  if (n < 0 || n > 65535) return set_err(PIGO_E_INVALID, "%d sources: outside 0..65535", n);
  if (!gray_bytes) return set_err(PIGO_E_INVALID, "null gray_bytes");
  if (n > 0 && (!src || !images)) return set_err(PIGO_E_INVALID, "null src or images");
  int rc = check_decoded(src, n);
  if (rc) return rc;
  std::vector<size_t> off;
  std::vector<char> first;
  const size_t total = arena_layout(src, n, off, first);
  if (!gray || *gray_bytes < total) {
    *gray_bytes = total;
    if (total > 0) return set_err(PIGO_E_CAP, "the gray arena needs %zu bytes", total);
  }
  if (n == 0) return PIGO_OK;
  if ((rc = ensure_device())) return rc;
  if ((rc = refuse_capture("pigo_gray_images", stream_))) return rc;
  for (int i = 0; i < n; ++i) images[i] = pigo_image{gray + off[i], src[i].height, src[i].width, src[i].width};
  return gray_images_on(default_device(), src, n, off, first, gray, flags, stream_);
}

}  // extern "C"

// ---- sharded mixed-size calls: contiguous ranges of entries over the devices (pigo_*_images_sharded, pigo_*_decoded_sharded) ----
// Geometry-only images of decoded sources (Dim = width, as pigo_gray_images gives them): the argument checks and ladders
// read no pixels, so every descriptor points at one placeholder byte.
static const uint8_t kNoPixels = 0;
static std::vector<pigo_image> decoded_geometry(const pigo_decoded* src, int n) {
  std::vector<pigo_image> v(n);
  for (int i = 0; i < n; ++i) v[i] = pigo_image{&kNoPixels, src[i].height, src[i].width, src[i].width};
  return v;
}

// Runs fn(device images, stream) for a decoded shard on device dev.  The sources are converted into the gray arena of a
// borrowed workspace (the layout pigo_gray_images gives them), and everything of the shard is ordered on the workspace's
// own stream: the copies and conversion, then the scan or pipeline that reads the arena.
template <typename F>
static int with_gray_shard(int dev, const pigo_decoded* src, int n, F fn) {
  int rc = use_device(dev);
  if (rc) return rc;
  Borrow w(g_misc_pool[dev], nullptr);
  if (w.rc) return w.rc;
  std::vector<size_t> off;
  std::vector<char> first;
  const size_t total = arena_layout(src, n, off, first);
  if ((rc = w->gray_arena.reserve(total + 256))) return rc;
  uint8_t* gray = (uint8_t*)w->gray_arena.p;
  std::vector<pigo_image> images(n);
  for (int i = 0; i < n; ++i) images[i] = pigo_image{gray + off[i], src[i].height, src[i].width, src[i].width};
  if ((rc = gray_images_on(dev, src, n, off, first, gray, PIGO_MEM_HOST, w.st))) return rc;
  return fn(images.data(), (void*)w.st);
}

// A sharded mixed-size call over `images` (host pixels, or with src the geometry of the decoded sources) at angles[]
// (nullptr: `angle` for every image): the call's ladders, its split over the devices, and for the shard of entries
// [lo, lo+n) on device dev fn(dev, images, n, lo, angles, ladders, flags, stream) over the shard's host images, or over
// the device images of its converted sources on the stream that converted them.
template <typename F>
static int run_sharded(const pigo_image* images, const pigo_decoded* src, int nimages, const double* angles, double angle, int min_size,
                       int max_size, double shift_factor, double scale_factor, F fn) {
  ImagePlans ip;
  int rc = build_image_plans(images, nimages, min_size, max_size, shift_factor, scale_factor, ip);
  if (rc) return rc;
  if (nimages == 0) return ensure_device();
  std::vector<double> uniform;
  angles = angles_or(angles, angle, nimages, uniform);
  const std::vector<int> devs = sharded_devices();
  if (devs.empty()) return PIGO_E_NODEVICE;   // message set by pigo_init
  const std::vector<int> first = plan_shards(ip.wins, angles, shard_count((int)devs.size()));
  return for_each_shard(devs, first, [&](int, int dev, int lo, int n) {
    const ImagePlans sp = ip.slice(lo, n);
    if (!src) return fn(dev, images + lo, n, lo, angles + lo, sp, PIGO_MEM_HOST, nullptr);
    return with_gray_shard(dev, src + lo, n, [&](const pigo_image* dimg, void* st) {
      return fn(dev, dimg, n, lo, angles + lo, sp, PIGO_FRAMES_DEVICE, st);
    });
  });
}

static int run_cascade_sharded(const pigo_cascade* cc, const pigo_image* images, const pigo_decoded* src, int nimages, const double* angles,
                               int min_size, int max_size, double shift_factor, double scale_factor, pigo_det* out, int cap_per_image, int* n_out) {
  pigo_cascade* c = const_cast<pigo_cascade*>(cc);
  return run_sharded(images, src, nimages, angles, 0.0, min_size, max_size, shift_factor, scale_factor,
                     [&](int dev, const pigo_image* im, int n, int lo, const double* a, const ImagePlans& sp, unsigned flags, void* st) {
                       return scan_images_on(c, dev, im, n, sp, min_size, max_size, shift_factor, scale_factor, a,
                                             out ? out + (size_t)lo * cap_per_image : nullptr, cap_per_image, n_out + lo, flags, st);
                     });
}

static int detect_sharded(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, const uint8_t* flp_flip, int ncalls,
                          const pigo_image* images, const pigo_decoded* src, int nimages, const double* angles, const pigo_pipeline_params* prm,
                          const float* randoms, uint64_t rng_seed, pigo_det* faces, int face_cap, int* n_faces, pigo_point* points) {
  const size_t per_image = (size_t)face_cap * (2 + ncalls);
  pigo_cascade* fc = const_cast<pigo_cascade*>(face);
  pigo_puploc* pc = const_cast<pigo_puploc*>(puploc);
  return run_sharded(images, src, nimages, angles, prm->angle, prm->min_size, prm->max_size, prm->shift_factor, prm->scale_factor,
                     [&](int dev, const pigo_image* im, int n, int lo, const double* a, const ImagePlans& sp, unsigned flags, void* st) {
                       // the shard's generator keys and injected randoms are those of images lo.. in the whole call
                       const float* rnd = randoms ? randoms + (size_t)lo * per_image * 189 : nullptr;
                       return detect_images_on(dev, fc, pc, (pigo_puploc* const*)flp, flp_flip, ncalls, im, n, a, sp, *prm, rnd, rng_seed,
                                               (uint64_t)lo * per_image, faces + (size_t)lo * face_cap, face_cap, n_faces + lo,
                                               points + (size_t)lo * per_image, flags, st);
                     });
}

// Arguments of the decoded forms: what pigo_gray_images checks, before the checks of the matching mixed-size call.
static int check_decoded_args(const pigo_decoded* src, int n) {
  if (n < 0 || n > 65535) return set_err(PIGO_E_INVALID, "%d sources: outside 0..65535", n);
  if (n > 0 && !src) return set_err(PIGO_E_INVALID, "null src");
  return check_decoded(src, n);
}

extern "C" {

int pigo_run_cascade_images_sharded(const pigo_cascade* c, const pigo_image* images, int nimages, const double* angles, int min_size, int max_size,
                                    double shift_factor, double scale_factor, pigo_det* out, int cap_per_image, int* n_out) {
  const int rc = check_images_args(c, images, nimages, out, cap_per_image, n_out);
  if (rc) return rc;
  return run_cascade_sharded(c, images, nullptr, nimages, angles, min_size, max_size, shift_factor, scale_factor, out, cap_per_image, n_out);
}

int pigo_detect_images_sharded(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, const uint8_t* flp_flip,
                               int ncalls, const pigo_image* images, int nimages, const double* angles, const pigo_pipeline_params* prm,
                               const float* randoms, uint64_t rng_seed, pigo_det* faces, int face_cap, int* n_faces, pigo_point* points) {
  const int rc = check_detect_images_args(face, puploc, flp, ncalls, images, nimages, prm, faces, face_cap, n_faces, points);
  if (rc) return rc;
  return detect_sharded(face, puploc, flp, flp_flip, ncalls, images, nullptr, nimages, angles, prm, randoms, rng_seed, faces, face_cap, n_faces,
                        points);
}

int pigo_run_cascade_decoded_sharded(const pigo_cascade* c, const pigo_decoded* src, int n, const double* angles, int min_size, int max_size,
                                     double shift_factor, double scale_factor, pigo_det* out, int cap_per_image, int* n_out) {
  int rc = check_decoded_args(src, n);
  if (rc) return rc;
  const std::vector<pigo_image> geo = decoded_geometry(src, n);
  if ((rc = check_images_args(c, geo.data(), n, out, cap_per_image, n_out))) return rc;
  return run_cascade_sharded(c, geo.data(), src, n, angles, min_size, max_size, shift_factor, scale_factor, out, cap_per_image, n_out);
}

int pigo_detect_decoded_sharded(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, const uint8_t* flp_flip,
                                int ncalls, const pigo_decoded* src, int n, const double* angles, const pigo_pipeline_params* prm,
                                const float* randoms, uint64_t rng_seed, pigo_det* faces, int face_cap, int* n_faces, pigo_point* points) {
  int rc = check_decoded_args(src, n);
  if (rc) return rc;
  const std::vector<pigo_image> geo = decoded_geometry(src, n);
  if ((rc = check_detect_images_args(face, puploc, flp, ncalls, geo.data(), n, prm, faces, face_cap, n_faces, points))) return rc;
  return detect_sharded(face, puploc, flp, flp_flip, ncalls, geo.data(), src, n, angles, prm, randoms, rng_seed, faces, face_cap, n_faces, points);
}

int pigo_shard_plan(const pigo_image* images, int nimages, const double* angles, int min_size, int max_size, double shift_factor,
                    double scale_factor, int nshards, int* first, int* n_used) {
  if (nimages < 0 || nimages > 65535) return set_err(PIGO_E_INVALID, "nimages must be 0..65535");
  if (nimages > 0 && !images) return set_err(PIGO_E_INVALID, "null images");
  if (!n_used) return set_err(PIGO_E_INVALID, "null n_used");
  if (nshards < 0) return set_err(PIGO_E_INVALID, "negative nshards");
  int rc = check_image_geometry(images, nimages, 0, false);
  if (rc) return rc;
  ImagePlans ip;
  if ((rc = build_image_plans(images, nimages, min_size, max_size, shift_factor, scale_factor, ip))) return rc;
  if (nshards == 0) nshards = shard_count(std::max(1, (int)shard_devices().size()));
  const std::vector<int> cut = plan_shards(ip.wins, angles, nshards);
  *n_used = (int)cut.size() - 1;
  if (first) std::copy(cut.begin(), cut.end(), first);
  return PIGO_OK;
}

}  // extern "C"
