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
#include <string>
#include <thread>
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
static const char* kSlotNames[T_NSLOTS] = {"tiled", "gather", "deep", "finalize", "cluster", "puploc", "gray", "seeds", "rottab", "ycbcr"};

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

  WsGuard g(R->pool);
  Workspace* w = g.w;
  if (!w) return set_err(PIGO_E_CUDA, "could not create a CUDA stream");
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : w->stream;
  if ((rc = ws_enter(w, st))) return rc;
  // CUDA-graph capture (device frames + device outputs on the caller's capturing stream, after one un-captured warm-up call
  // with the same arguments): the captured kernels keep using this workspace's scratch on every replay, so the workspace
  // is taken out of the pool for good -- it belongs to the graph from now on.
  const bool capturing = stream_capturing(st);
  if (capturing) {
    if (!(flags & PIGO_FRAMES_DEVICE) || !(flags & PIGO_OUT_DEVICE)) return set_err(PIGO_E_INVALID, "stream capture needs device frames and device outputs");
    if (w->p_rows != rows || w->p_cols != cols || w->p_min != min_size || w->p_max != max_size || w->p_shift != shift_factor ||
        w->p_scale != scale_factor)
      return set_err(PIGO_E_INVALID, "stream capture: run the same call once outside the capture first (the plan upload synchronises)");
    g.w = nullptr;
  }

  // plan (cached per workspace)
  if (w->p_rows != rows || w->p_cols != cols || w->p_min != min_size || w->p_max != max_size || w->p_shift != shift_factor ||
      w->p_scale != scale_factor) {
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

  // device buffers.  A host frame is only guaranteed to hold (rows-1)*dim + cols bytes (what the reference indexes,
  // core/pigo.go:126 with Dim >= Cols): never read more than that from the caller's buffer.
  const uint8_t* d_frames = frames;
  const size_t frame_bytes = (size_t)rows * dim;
  const size_t frame_min = rows > 0 ? (size_t)(rows - 1) * dim + cols : 0;
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
  // streams.  (1) The deferred queues (Q1/Q2) of a group are bounded and consumed soon after they are filled;
  // (2) with host frames, the H2D copy of group k+1 overlaps the scan of group k.
  int rot_slot = -1;
  if (angle > 0.0) {                      // core/pigo.go:232-236
    const double a = angle > 1.0 ? 1.0 : angle;
    rot_slot = (int)(32.0 * a);           // :159
  }
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
  CUDA_TRY(cudaMemcpyAsync(n_out, d_nout, (size_t)nframes * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  int need_more = 0;
  size_t max_n = 0;
  for (int f = 0; f < nframes; ++f) {
    if (n_out[f] > cap_per_frame) need_more = 1;
    size_t k = (size_t)std::min(n_out[f], cap_per_frame);
    if (k > max_n) max_n = k;
  }
  if (cap_per_frame > 0 && max_n > 0) {
    // copy only the used prefix of every frame's slice
    CUDA_TRY(cudaMemcpy2DAsync(out, (size_t)cap_per_frame * sizeof(pigo_det), d_out, (size_t)cap * sizeof(pigo_det),
                               max_n * sizeof(pigo_det), nframes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
  }
  if (need_more) return set_err(PIGO_E_CAP, "output capacity %d per frame too small", cap_per_frame);
  return PIGO_OK;
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

// Runs fn(shard index, device, first frame, frame count) on one host thread per device of the mask; frames are split
// [g*ceil(N/G), (g+1)*ceil(N/G)) like SURVEY.md section 8e.  Returns the first error, PIGO_E_CAP last (so that every
// shard's required counts are valid when the caller retries).
template <typename F>
static int for_each_shard(int nframes, F fn) {
  std::vector<int> devs = shard_devices();
  if (devs.empty()) {
    const int d = default_device();
    if (d < 0) return PIGO_E_NODEVICE;
    devs.push_back(d);
  }
  const int G = (int)devs.size();
  const int per = (nframes + G - 1) / G;
  std::vector<int> rcs(G, PIGO_OK);
  std::vector<std::string> msgs(G);
  std::vector<std::thread> th;
  for (int gidx = 0; gidx < G; ++gidx) {
    const int lo = std::min(nframes, gidx * per), hi = std::min(nframes, lo + per);
    if (hi <= lo) continue;
    th.emplace_back([&, gidx, lo, hi]() {
      rcs[gidx] = fn(gidx, devs[gidx], lo, hi - lo);
      if (rcs[gidx] != PIGO_OK) msgs[gidx] = g_err;   // g_err is thread-local: carry the worker's message back
    });
  }
  for (auto& t : th) t.join();
  int rc = PIGO_OK;
  for (int gidx = 0; gidx < G; ++gidx) {
    if (rcs[gidx] == PIGO_OK) continue;
    if (rc == PIGO_OK || (rc == PIGO_E_CAP && rcs[gidx] != PIGO_E_CAP)) { rc = rcs[gidx]; g_err = msgs[gidx]; }
  }
  return rc;
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

int pigo_describe_plan(int rows, int cols, int min_size, int max_size, double shift_factor, double scale_factor, char* json, size_t cap) {
  if (!json) return set_err(PIGO_E_INVALID, "null buffer");
  std::vector<ScaleEntry> plan;
  uint64_t total = 0;
  int rc = build_plan(rows, cols, min_size, max_size, shift_factor, scale_factor, plan, total);
  if (rc) return rc;
  return describe_plan(plan, total, 468, json, cap);   // geometry of the stock 468-tree facefinder cascade
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
  WsGuard g(g_misc_pool[dev]);
  Workspace* w = g.w;
  if (!w) return set_err(PIGO_E_CUDA, "could not create a CUDA stream");
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : w->stream;
  if ((rc = ws_enter(w, st))) return rc;
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
  const int dev = default_device();
  PuplocReplica* R = puploc_replica(p, dev, &rc);
  if (!R) return rc;
  const bool frames_dev = flags & PIGO_FRAMES_DEVICE, out_dev = flags & PIGO_OUT_DEVICE;
  bool wide = false;   // some seed outside the 32-bit envelope of the pair kernel (only checkable for host seeds)
  if (!out_dev)
    for (int i = 0; i < nseeds; ++i) {
      if (seeds[i].perturbs < 0 || seeds[i].perturbs > 63)
        return set_err(PIGO_E_INVALID, "seed %d: Perturbs=%d outside 0..63 (the reference panics, core/puploc.go:261)", i, seeds[i].perturbs);
      if (seed_frame && (seed_frame[i] < 0 || seed_frame[i] >= nframes)) return set_err(PIGO_E_INVALID, "seed %d: frame index out of range", i);
      if (!(std::fabs(seeds[i].scale) <= 16384.0f)) wide = true;
    }
  WsGuard g(R->pool);
  Workspace* w = g.w;
  if (!w) return set_err(PIGO_E_CUDA, "could not create a CUDA stream");
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : w->stream;
  if ((rc = ws_enter(w, st))) return rc;
  const uint8_t* d_pix = pixels;
  if (!frames_dev) {
    const size_t bytes = frame_stride * (size_t)(nframes - 1) + (size_t)(rows - 1) * dim + cols;   // what the reference may index
    if ((rc = w->frames.reserve(frame_stride * (size_t)(nframes - 1) + (size_t)rows * dim))) return rc;
    CUDA_TRY(cudaMemcpyAsync(w->frames.p, pixels, bytes, cudaMemcpyHostToDevice, st));
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
  int rot_slot = -1;
  if (angle > 0.0) rot_slot = (int)(32.0 * (angle > 1.0 ? 1.0 : angle));  // core/puploc.go:252-256, :166
  bool done = false;
  timing_begin(T_PUPLOC, st);
  if (g_opt.puploc_mode.load() == 0 && !wide) {
    if ((rc = w->counters.reserve(64))) return rc;
    CUDA_TRY(cudaMemsetAsync(w->counters.p, 0, 64, st));
    PupWork W{};
    W.seeds = d_seeds; W.out = d_out; W.randoms = d_rnd; W.rng_seed = rng_seed; W.frames = d_pix; W.frame_stride = frame_stride;
    W.slot_frame = d_sf; W.flipv = d_flip; W.slots_per_frame = 0; W.nrows = rows; W.ncols = cols; W.dim = dim; W.rot_slot = rot_slot;
    W.first = 0; W.span = 1; W.stride = 1; W.nwork = nseeds; W.ntabs = 1; W.tab[0] = R->tab;
    done = launch_puploc_pairs(W, (unsigned int*)w->counters.p, R->num_sms, st) == 0;
  }
  if (!done)
    launch_puploc(R->tab, d_seeds, nseeds, d_rnd, rng_seed, d_pix, d_sf, frame_stride, rows, cols, dim, rot_slot, d_flip, d_out, st);
  timing_end(T_PUPLOC, st);
  g_launches++;
  CUDA_TRY(cudaGetLastError());
  if (out_dev) return ws_leave_async(w, st);
  CUDA_TRY(cudaMemcpyAsync(out, d_out, (size_t)nseeds * sizeof(pigo_point), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return PIGO_OK;
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
// one D2H copy of the results at the end.
static int detect_batch_on(int dev, pigo_cascade* face, pigo_puploc* puploc, pigo_puploc* const* flp, const uint8_t* flp_flip, int ncalls,
                           const uint8_t* frames, int nframes, size_t frame_stride, int rows, int cols, int dim, const pigo_pipeline_params& P,
                           const float* randoms, uint64_t rng_seed, uint64_t slot_base, pigo_det* faces, int face_cap, int* n_faces,
                           pigo_point* points, unsigned flags, void* stream_) {
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
  const bool frames_dev = flags & PIGO_FRAMES_DEVICE, out_dev = flags & PIGO_OUT_DEVICE;
  const int det_cap = P.det_cap > 0 ? P.det_cap : 2048;

  WsGuard g(R->pool);
  Workspace* w = g.w;
  if (!w) return set_err(PIGO_E_CUDA, "could not create a CUDA stream");
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : w->stream;
  if ((rc = ws_enter(w, st))) return rc;

  const size_t frame_bytes = (size_t)rows * dim;
  const uint8_t* d_frames = frames;
  size_t d_stride = frame_stride;
  if (!frames_dev) {
    // the scan call below streams the host frames into THIS buffer (chunked copy overlapped with the scan kernels); the
    // pupil / landmark stages gather from it afterwards
    d_stride = (frame_bytes + 255) & ~(size_t)255;
    if ((rc = w->frames.reserve(d_stride * nframes + 256))) return rc;
    d_frames = (const uint8_t*)w->frames.p;
  }
  const size_t nslots = (size_t)nframes * face_cap * stride;
  // scratch: raw detections + counts, clusters + counts, seeds, points, faces, work counters
  const size_t b_dets = (size_t)nframes * det_cap * sizeof(pigo_det), b_cl = (size_t)nframes * face_cap * sizeof(pigo_det);
  const size_t b_pts = nslots * sizeof(pigo_point);
  if ((rc = w->raw.reserve(b_dets)) || (rc = w->out.reserve(b_cl + b_cl)) || (rc = w->nout.reserve((size_t)nframes * 16 + 256)) ||
      (rc = w->scratch_a.reserve(b_pts)) || (rc = w->scratch_b.reserve(b_pts)) || (rc = w->counters.reserve(256))) return rc;
  pigo_det* d_dets = (pigo_det*)w->raw.p;
  pigo_det* d_clusters = (pigo_det*)w->out.p;
  pigo_det* d_faces = out_dev ? faces : (pigo_det*)((char*)w->out.p + b_cl);
  int32_t* d_cnt = (int32_t*)w->nout.p;
  int32_t* d_ncl = d_cnt + nframes;
  int32_t* d_nfaces = out_dev ? n_faces : d_cnt + 2 * (size_t)nframes;
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

  if (frames_dev)
    rc = scan_batch_on(face, dev, d_frames, nframes, d_stride, rows, cols, dim, P.min_size, P.max_size, P.shift_factor, P.scale_factor, P.angle,
                       d_dets, det_cap, d_cnt, PIGO_FRAMES_DEVICE | PIGO_OUT_DEVICE, st);
  else
    rc = scan_batch_on(face, dev, frames, nframes, frame_stride, rows, cols, dim, P.min_size, P.max_size, P.shift_factor, P.scale_factor, P.angle,
                       d_dets, det_cap, d_cnt, PIGO_OUT_DEVICE, st, (uint8_t*)w->frames.p);
  if (rc) return rc;
  rc = cluster_batch_on(dev, d_dets, d_cnt, nframes, det_cap, P.iou_threshold, d_clusters, face_cap, d_ncl, PIGO_OUT_DEVICE, st);
  if (rc) return rc;
  timing_begin(T_SEEDS, st);
  launch_eye_seeds(d_clusters, d_ncl, face_cap, nframes, face_cap, stride, P.min_face_scale, P.eye_perturbs, d_faces, d_nfaces, d_seeds, st);
  timing_end(T_SEEDS, st);
  g_launches++;

  int rot_slot = -1;
  if (P.angle > 0.0) rot_slot = (int)(32.0 * (P.angle > 1.0 ? 1.0 : P.angle));   // RunDetector(puploc, img, det.angle, false), main.go:422
  W.seeds = d_seeds; W.out = d_points; W.randoms = d_rnd; W.rng_seed = rng_seed; W.slot_base = slot_base;
  W.frames = d_frames; W.frame_stride = d_stride; W.slot_frame = nullptr; W.flipv = nullptr;
  W.slots_per_frame = face_cap * stride; W.nrows = rows; W.ncols = cols; W.dim = dim;
  W.stride = stride;
  // (a) both eyes of every face slot
  PupWork E = W;
  E.rot_slot = rot_slot; E.first = 0; E.span = 2; E.nwork = nframes * face_cap * 2;
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

  // one D2H round: counts (raw detections, clusters), faces, points
  std::vector<int32_t> cnt(2 * (size_t)nframes);
  CUDA_TRY(cudaMemcpyAsync(cnt.data(), d_cnt, cnt.size() * 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(n_faces, d_nfaces, (size_t)nframes * 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(faces, d_faces, b_cl, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(points, d_points, b_pts, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  for (int f = 0; f < nframes; ++f)
    if (cnt[f] > det_cap) return set_err(PIGO_E_CAP, "frame %d has %d raw detections, det_cap is %d: raise pigo_pipeline_params.det_cap", f, cnt[f], det_cap);
  for (int f = 0; f < nframes; ++f)
    if (n_faces[f] > face_cap) return set_err(PIGO_E_CAP, "frame %d has %d faces, face_cap is %d", f, n_faces[f], face_cap);
  return PIGO_OK;
}

extern "C" {

static int check_detect_args(const pigo_cascade* face, const pigo_puploc* puploc, const pigo_puploc* const* flp, int ncalls, const uint8_t* frames,
                             int nframes, size_t frame_stride, int rows, int cols, int dim, const pigo_pipeline_params* prm,
                             const pigo_det* faces, int face_cap, const int* n_faces, const pigo_point* points) {
  if (!face || !puploc || !prm || !faces || !n_faces || !points || (ncalls > 0 && !flp)) return set_err(PIGO_E_INVALID, "null argument");
  if (ncalls < 0 || ncalls > 30) return set_err(PIGO_E_INVALID, "ncalls must be 0..30");
  for (int i = 0; i < ncalls; ++i)
    if (!flp[i]) return set_err(PIGO_E_INVALID, "null landmark cascade %d", i);
  if (face_cap < 1 || face_cap > 4096) return set_err(PIGO_E_INVALID, "face_cap must be 1..4096");
  if (prm->eye_perturbs < 0 || prm->eye_perturbs > 63 || prm->flp_perturbs < 0 || prm->flp_perturbs > 63)
    return set_err(PIGO_E_INVALID, "Perturbs outside 0..63 (the reference panics, core/puploc.go:261)");
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

// ---- RgbToGrayscale, core/grayscale.go:8-23 ----------------------------------------------------------------
int pigo_rgba_to_gray(const uint8_t* rgba, size_t npixels, uint8_t* gray, unsigned flags, void* stream_) {
  if (npixels == 0) return ensure_device();
  if (!rgba || !gray) return set_err(PIGO_E_INVALID, "null argument");
  int rc = ensure_device();
  if (rc) return rc;
  const int dev = default_device();
  WsGuard g(g_misc_pool[dev]);
  Workspace* w = g.w;
  if (!w) return set_err(PIGO_E_CUDA, "could not create a CUDA stream");
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : w->stream;
  if ((rc = ws_enter(w, st))) return rc;   // a device-output call returns while the kernel still reads the staging buffer
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
  WsGuard g(g_misc_pool[dev]);
  Workspace* w = g.w;
  if (!w) return set_err(PIGO_E_CUDA, "could not create a CUDA stream");
  cudaStream_t st = stream_ ? (cudaStream_t)stream_ : w->stream;
  if ((rc = ws_enter(w, st))) return rc;
  const bool in_dev = flags & PIGO_FRAMES_DEVICE, out_dev = flags & PIGO_OUT_DEVICE;
  // plane extents as image.YCbCr lays them out for Rect (min)-(min + size): COffset rows / columns per ratio
  const int cw_div = (subsample == 1 || subsample == 2) ? 2 : ((subsample == 4 || subsample == 5) ? 4 : 1);
  const int ch_div = (subsample == 2 || subsample == 3 || subsample == 5) ? 2 : 1;
  const int c_rows = (min_y + height - 1) / ch_div - min_y / ch_div + 1, c_cols = (min_x + width - 1) / cw_div - min_x / cw_div + 1;
  const size_t y_bytes = (size_t)(height - 1) * y_stride + width, c_bytes = (size_t)(c_rows - 1) * c_stride + c_cols;
  const uint8_t *d_y = y, *d_cb = cb, *d_cr = cr;
  if (!in_dev) {
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
