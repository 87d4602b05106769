// pigo_b200.hpp -- header-only C++ host-side mirror of the pigo Go API over the C-ABI (include/pigo_b200.h).
//
// The reference is compiled code (Go); its toolchain is absent from the build image, so the host side above the
// C-ABI is provided in C++ (this file), in Go for maintainers who have the toolchain (go/pigo/pigo.go) and in
// Python/ctypes for the tests (pigo_b200/__init__.py).  Names, argument meaning and failure behaviour follow
// core/pigo.go, core/puploc.go and core/flploc.go: methods that cannot fail in the reference throw
// std::runtime_error here where the reference would panic.
#pragma once
#include <cmath>
#include <cstdint>
#include <fstream>
#include <iterator>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "pigo_b200.h"

namespace pigo {

struct ImageParams {            // core/pigo.go:29-34
  const uint8_t* Pixels = nullptr;
  int Rows = 0, Cols = 0, Dim = 0;
};
struct CascadeParams {          // core/pigo.go:16-22
  ImageParams Image;
  int MinSize = 0, MaxSize = 0;
  double ShiftFactor = 0, ScaleFactor = 0;
};
struct Detection {              // core/pigo.go:195-200
  int Row = 0, Col = 0, Scale = 0;
  float Q = 0;
};
struct SweepDetection {         // additive: a cluster of an angle sweep and the listed angle it was found at
  Detection Det;
  double Angle = 0.0;
};
struct Puploc {                 // core/puploc.go:14-19
  int Row = 0, Col = 0;
  float Scale = 0;
  int Perturbs = 0;
};

namespace detail {
// the pigo_cascade_params of cps
inline std::vector<pigo_cascade_params> params_of(const std::vector<CascadeParams>& cps) {
  std::vector<pigo_cascade_params> prm;
  for (const CascadeParams& cp : cps) prm.push_back(pigo_cascade_params{cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor});
  return prm;
}
}  // namespace detail

inline void check(int rc) {
  if (rc != PIGO_OK) throw std::runtime_error(std::string("libpigo_b200: ") + pigo_last_error());
}

class Pigo {                    // core/pigo.go:37-43
 public:
  Pigo() = default;
  // (*Pigo).Unpack, core/pigo.go:51-110
  static Pigo Unpack(const std::vector<uint8_t>& packet) {
    Pigo p;
    pigo_cascade* h = nullptr;
    check(pigo_cascade_create(packet.data(), packet.size(), &h));
    p.h_.reset(h, pigo_cascade_destroy);
    return p;
  }
  // (*Pigo).RunCascade, core/pigo.go:212-258
  std::vector<Detection> RunCascade(const CascadeParams& cp, double angle) const {
    int cap = 1024, n = 0;
    for (;;) {
      std::vector<pigo_det> buf((size_t)cap);
      const int rc = pigo_run_cascade(h_.get(), cp.Image.Pixels, cp.Image.Rows, cp.Image.Cols, cp.Image.Dim, cp.MinSize, cp.MaxSize,
                                      cp.ShiftFactor, cp.ScaleFactor, angle, buf.data(), cap, &n);
      if (rc == PIGO_E_CAP) { cap = n; continue; }
      check(rc);
      std::vector<Detection> out((size_t)n);
      for (int i = 0; i < n; ++i) out[i] = Detection{buf[i].row, buf[i].col, buf[i].scale, buf[i].q};
      return out;
    }
  }
  // (*Pigo).ClusterDetections, core/pigo.go:262-308 -- sorts `detections` in place like the reference (:264)
  std::vector<Detection> ClusterDetections(std::vector<Detection>& detections, double iouThreshold) const {
    const int n = (int)detections.size();
    if (n == 0) return {};
    std::vector<pigo_det> in((size_t)n), out((size_t)n);
    for (int i = 0; i < n; ++i) in[i] = pigo_det{detections[i].Row, detections[i].Col, detections[i].Scale, detections[i].Q};
    int k = 0;
    check(pigo_cluster(in.data(), n, iouThreshold, out.data(), n, &k));
    for (int i = 0; i < n; ++i) detections[i] = Detection{in[i].row, in[i].col, in[i].scale, in[i].q};
    std::vector<Detection> res((size_t)k);
    for (int i = 0; i < k; ++i) res[i] = Detection{out[i].row, out[i].col, out[i].scale, out[i].q};
    return res;
  }
  // additive: RunCascade for a frame batch (host frames `stride` bytes apart); sharded = over the GPUs of InitDevices
  std::vector<std::vector<Detection>> RunCascadeBatch(const uint8_t* frames, int nframes, size_t stride, const CascadeParams& cp, double angle,
                                                      bool sharded = false) const {
    int cap = 256;
    for (;;) {
      std::vector<pigo_det> buf((size_t)cap * nframes);
      std::vector<int> cnt((size_t)nframes);
      const int rc = sharded ? pigo_run_cascade_batch_sharded(h_.get(), frames, nframes, stride, cp.Image.Rows, cp.Image.Cols, cp.Image.Dim, cp.MinSize,
                                                              cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor, angle, buf.data(), cap, cnt.data())
                           : pigo_run_cascade_batch(h_.get(), frames, nframes, stride, cp.Image.Rows, cp.Image.Cols, cp.Image.Dim, cp.MinSize, cp.MaxSize,
                                                    cp.ShiftFactor, cp.ScaleFactor, angle, buf.data(), cap, cnt.data(), PIGO_MEM_HOST, nullptr);
      if (rc == PIGO_E_CAP) { for (int c : cnt) cap = c > cap ? c : cap; continue; }
      check(rc);
      std::vector<std::vector<Detection>> out((size_t)nframes);
      for (int f = 0; f < nframes; ++f)
        for (int i = 0; i < cnt[f]; ++i) { const pigo_det& d = buf[(size_t)f * cap + i]; out[f].push_back(Detection{d.row, d.col, d.scale, d.q}); }
      return out;
    }
  }
  // additive: RunCascade for images of different sizes in one call (host pixels); result i is what RunCascade returns for
  // images[i] with cp's MinSize / MaxSize / ShiftFactor / ScaleFactor (cp.Image is not used)
  std::vector<std::vector<Detection>> RunCascadeImages(const std::vector<ImageParams>& images, const CascadeParams& cp, double angle) const {
    return RunCascadeImagesAngles(images, cp, std::vector<double>(images.size(), angle));
  }
  // additive: RunCascadeImages with images[i] scanned at angles[i] (one angle per image; an angle sweep lists an image once
  // per angle, and repeated pixels are copied to the device once)
  std::vector<std::vector<Detection>> RunCascadeImagesAngles(const std::vector<ImageParams>& images, const CascadeParams& cp,
                                                             const std::vector<double>& angles) const {
    if (angles.size() != images.size()) throw std::invalid_argument("RunCascadeImagesAngles needs one angle per image");
    return runImages(images, cp, angles, false);
  }
  // additive: RunCascadeImagesAngles over the GPUs of InitDevices (host pixels, contiguous shards of about equal modelled
  // cost); the result equals the single-GPU call's
  std::vector<std::vector<Detection>> RunCascadeImagesSharded(const std::vector<ImageParams>& images, const CascadeParams& cp,
                                                              const std::vector<double>& angles) const {
    if (angles.size() != images.size()) throw std::invalid_argument("RunCascadeImagesSharded needs one angle per image");
    return runImages(images, cp, angles, true);
  }
  // additive: every image scanned at every angle of `angles`, one merged list per image: the clusters of the concatenation
  // of its RunCascade lists over the angles, each with the listed angle of its largest-Q member (pigo_run_cascade_images_sweep).
  // PIGO_E_CAP is retried with the reported counts (or a larger det_cap).
  std::vector<std::vector<SweepDetection>> RunCascadeImagesSweep(const std::vector<ImageParams>& images, const CascadeParams& cp,
                                                                 const std::vector<double>& angles, double iou) const {
    const int n = (int)images.size();
    std::vector<pigo_image> desc((size_t)n);
    for (int i = 0; i < n; ++i) desc[i] = pigo_image{images[i].Pixels, images[i].Rows, images[i].Cols, images[i].Dim};
    int cap = 64, det_cap = 0;
    for (;;) {
      std::vector<pigo_det> buf((size_t)cap * (n > 0 ? n : 1));
      std::vector<int32_t> idx(buf.size());
      std::vector<int> cnt((size_t)(n > 0 ? n : 1));
      const int rc = pigo_run_cascade_images_sweep(h_.get(), desc.data(), n, angles.data(), (int)angles.size(), cp.MinSize, cp.MaxSize, cp.ShiftFactor,
                                                   cp.ScaleFactor, iou, det_cap, buf.data(), idx.data(), cap, cnt.data(), PIGO_MEM_HOST, nullptr);
      if (rc == PIGO_E_CAP) {
        bool grown = false;
        for (int c : cnt) if (c > cap) { cap = c; grown = true; }
        if (!grown) det_cap = 4 * (det_cap + 512);   // raw detections of an (image, angle) entry exceeded det_cap
        continue;
      }
      check(rc);
      std::vector<std::vector<SweepDetection>> out((size_t)n);
      for (int f = 0; f < n; ++f)
        for (int i = 0; i < cnt[f]; ++i) {
          const size_t k = (size_t)f * cap + i;
          out[f].push_back(SweepDetection{Detection{buf[k].row, buf[k].col, buf[k].scale, buf[k].q}, angles[(size_t)idx[k]]});
        }
      return out;
    }
  }
  // additive: the list of calls RunCascade(cps[i], angles[i]) as one call (pigo_run_cascade_images_params): each
  // CascadeParams carries its own Image, MinSize, MaxSize, ShiftFactor and ScaleFactor; result i is what that RunCascade
  // returns.  angles is empty (every image unrotated) or has one entry per image.
  std::vector<std::vector<Detection>> RunCascadeImagesParams(const std::vector<CascadeParams>& cps, const std::vector<double>& angles = {}) const {
    if (!angles.empty() && angles.size() != cps.size()) throw std::invalid_argument("RunCascadeImagesParams needs no angles or one angle per image");
    std::vector<ImageParams> images;
    for (const CascadeParams& cp : cps) images.push_back(cp.Image);
    const std::vector<pigo_cascade_params> prm = detail::params_of(cps);
    return runImages(images, CascadeParams{}, angles, false, prm.data());
  }
  const pigo_cascade* handle() const { return h_.get(); }

 private:
  // images with cp's parameters, or (params not null) image i with params[i]; angles empty = NULL
  std::vector<std::vector<Detection>> runImages(const std::vector<ImageParams>& images, const CascadeParams& cp, const std::vector<double>& angles,
                                                bool sharded, const pigo_cascade_params* params = nullptr) const {
    const int n = (int)images.size();
    std::vector<pigo_image> desc((size_t)n);
    for (int i = 0; i < n; ++i) desc[i] = pigo_image{images[i].Pixels, images[i].Rows, images[i].Cols, images[i].Dim};
    const double* ang = angles.empty() ? nullptr : angles.data();
    int cap = 256;
    for (;;) {
      std::vector<pigo_det> buf((size_t)cap * (n > 0 ? n : 1));
      std::vector<int> cnt((size_t)(n > 0 ? n : 1));
      const int rc = params ? pigo_run_cascade_images_params(h_.get(), desc.data(), n, params, ang, buf.data(), cap, cnt.data(), PIGO_MEM_HOST, nullptr)
                     : sharded ? pigo_run_cascade_images_sharded(h_.get(), desc.data(), n, ang, cp.MinSize, cp.MaxSize, cp.ShiftFactor,
                                                                 cp.ScaleFactor, buf.data(), cap, cnt.data())
                               : pigo_run_cascade_images_angles(h_.get(), desc.data(), n, ang, cp.MinSize, cp.MaxSize, cp.ShiftFactor,
                                                                cp.ScaleFactor, buf.data(), cap, cnt.data(), PIGO_MEM_HOST, nullptr);
      if (rc == PIGO_E_CAP) { for (int c : cnt) cap = c > cap ? c : cap; continue; }
      check(rc);
      std::vector<std::vector<Detection>> out((size_t)n);
      for (int f = 0; f < n; ++f)
        for (int i = 0; i < cnt[f]; ++i) { const pigo_det& d = buf[(size_t)f * cap + i]; out[f].push_back(Detection{d.row, d.col, d.scale, d.q}); }
      return out;
    }
  }
  std::shared_ptr<pigo_cascade> h_;
};
inline Pigo NewPigo() { return Pigo(); }   // core/pigo.go:46
inline void InitDevices(unsigned mask) { check(pigo_init_devices(mask)); }   // additive: GPUs of the sharded entry points

class PuplocCascade {            // core/puploc.go:23-30
 public:
  uint64_t Seed = 0;             // keys the library RNG (the reference uses the auto-seeded global math/rand)
  // (*PuplocCascade).UnpackCascade, core/puploc.go:38-103
  static PuplocCascade UnpackCascade(const std::vector<uint8_t>& packet) {
    PuplocCascade p;
    pigo_puploc* h = nullptr;
    check(pigo_puploc_create(packet.data(), packet.size(), &h));
    p.h_.reset(h, pigo_puploc_destroy);
    return p;
  }
  // (*PuplocCascade).UnpackFlp, core/flploc.go:27-33
  static PuplocCascade UnpackFlp(const std::string& cf) {
    std::ifstream f(cf, std::ios::binary);
    if (!f) throw std::runtime_error("cannot open " + cf);
    std::vector<uint8_t> bytes((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    return UnpackCascade(bytes);
  }
  // (*PuplocCascade).RunDetector, core/puploc.go:239-277; `randoms` (optional) = 63*3 floats in [0,1)
  Puploc RunDetector(const Puploc& pl, const ImageParams& img, double angle, bool flipV, const float* randoms = nullptr) {
    pigo_point seed{pl.Row, pl.Col, pl.Scale, pl.Perturbs}, out{};
    const uint8_t fl = flipV ? 1 : 0;
    check(pigo_puploc_run(h_.get(), &seed, 1, randoms, ++Seed, img.Pixels, img.Rows, img.Cols, img.Dim, angle, &fl, &out, PIGO_MEM_HOST, nullptr));
    return Puploc{out.row, out.col, out.scale, 0};
  }
  // (*PuplocCascade).GetLandmarkPoint, core/flploc.go:36-57
  Puploc GetLandmarkPoint(const Puploc& leftEye, const Puploc& rightEye, const ImageParams& img, int perturb, bool flipV,
                          const float* randoms = nullptr) {
    pigo_point le{leftEye.Row, leftEye.Col, leftEye.Scale, 0}, re{rightEye.Row, rightEye.Col, rightEye.Scale, 0}, out{};
    check(pigo_get_landmark_point(h_.get(), &le, &re, img.Pixels, img.Rows, img.Cols, img.Dim, perturb, flipV ? 1 : 0, randoms, ++Seed, &out));
    return Puploc{out.row, out.col, out.scale, 0};
  }
  const pigo_puploc* handle() const { return h_.get(); }

 private:
  std::shared_ptr<pigo_puploc> h_;
};

// additive: the face -> cluster -> pupils -> landmarks sequence of core/flploc_test.go:75-154 / cmd/pigo/main.go:369-565 for a frame
// batch in one library call (sequenced on the device); calls[c] = (landmark cascade, flipV).
struct FaceResult {
  Detection Face;
  bool Refined = false;          // Scale > min_face_scale: eyes and landmarks below are valid
  Puploc LeftEye, RightEye;
  std::vector<Puploc> Landmarks;
};
inline std::vector<std::vector<FaceResult>> DetectBatch(const Pigo& face, const PuplocCascade& plc,
                                                        const std::vector<std::pair<const PuplocCascade*, bool>>& calls, const uint8_t* frames,
                                                        int nframes, size_t stride, const CascadeParams& cp, double iou, int min_face_scale,
                                                        int eye_perturbs, int flp_perturbs, uint64_t rng_seed, bool sharded = false,
                                                        const float* randoms = nullptr, int face_cap = 32) {
  const int ncalls = (int)calls.size();
  std::vector<const pigo_puploc*> hs;
  std::vector<uint8_t> fl;
  for (auto& c : calls) { hs.push_back(c.first->handle()); fl.push_back(c.second ? 1 : 0); }
  pigo_pipeline_params prm{};
  prm.min_size = cp.MinSize; prm.max_size = cp.MaxSize; prm.shift_factor = cp.ShiftFactor; prm.scale_factor = cp.ScaleFactor; prm.angle = 0.0;
  prm.iou_threshold = iou; prm.min_face_scale = min_face_scale; prm.eye_perturbs = eye_perturbs; prm.flp_perturbs = flp_perturbs; prm.det_cap = 0;
  std::vector<pigo_det> faces((size_t)nframes * face_cap);
  std::vector<int> nfaces((size_t)nframes);
  std::vector<pigo_point> pts((size_t)nframes * face_cap * (2 + ncalls));
  check(sharded ? pigo_detect_batch_sharded(face.handle(), plc.handle(), hs.data(), fl.data(), ncalls, frames, nframes, stride, cp.Image.Rows, cp.Image.Cols,
                                            cp.Image.Dim, &prm, randoms, rng_seed, faces.data(), face_cap, nfaces.data(), pts.data())
                : pigo_detect_batch(face.handle(), plc.handle(), hs.data(), fl.data(), ncalls, frames, nframes, stride, cp.Image.Rows, cp.Image.Cols,
                                    cp.Image.Dim, &prm, randoms, rng_seed, faces.data(), face_cap, nfaces.data(), pts.data(), PIGO_MEM_HOST, nullptr));
  std::vector<std::vector<FaceResult>> out((size_t)nframes);
  for (int f = 0; f < nframes; ++f)
    for (int k = 0; k < nfaces[f]; ++k) {
      const pigo_det& d = faces[(size_t)f * face_cap + k];
      FaceResult r;
      r.Face = Detection{d.row, d.col, d.scale, d.q};
      if (d.scale > min_face_scale) {
        const pigo_point* p = &pts[((size_t)f * face_cap + k) * (2 + ncalls)];
        r.Refined = true;
        r.LeftEye = Puploc{p[0].row, p[0].col, p[0].scale, 0}; r.RightEye = Puploc{p[1].row, p[1].col, p[1].scale, 0};
        for (int c = 0; c < ncalls; ++c) r.Landmarks.push_back(Puploc{p[2 + c].row, p[2 + c].col, p[2 + c].scale, 0});
      }
      out[f].push_back(r);
    }
  return out;
}
namespace detail {
inline std::vector<std::vector<FaceResult>> detectImages(const Pigo& face, const PuplocCascade& plc,
                                                         const std::vector<std::pair<const PuplocCascade*, bool>>& calls,
                                                         const std::vector<ImageParams>& images, const CascadeParams& cp, double iou,
                                                         int min_face_scale, int eye_perturbs, int flp_perturbs, uint64_t rng_seed,
                                                         const std::vector<double>& angles, int face_cap, bool sharded,
                                                         const pigo_cascade_params* cparams = nullptr) {
  const int ncalls = (int)calls.size(), n = (int)images.size();
  std::vector<const pigo_puploc*> hs;
  std::vector<uint8_t> fl;
  for (auto& c : calls) { hs.push_back(c.first->handle()); fl.push_back(c.second ? 1 : 0); }
  std::vector<pigo_image> desc((size_t)n);
  for (int i = 0; i < n; ++i) desc[i] = pigo_image{images[i].Pixels, images[i].Rows, images[i].Cols, images[i].Dim};
  pigo_pipeline_params prm{};
  prm.min_size = cp.MinSize; prm.max_size = cp.MaxSize; prm.shift_factor = cp.ShiftFactor; prm.scale_factor = cp.ScaleFactor; prm.angle = 0.0;
  prm.iou_threshold = iou; prm.min_face_scale = min_face_scale; prm.eye_perturbs = eye_perturbs; prm.flp_perturbs = flp_perturbs; prm.det_cap = 0;
  for (;;) {
    std::vector<pigo_det> faces((size_t)(n > 0 ? n : 1) * face_cap);
    std::vector<int> nfaces((size_t)(n > 0 ? n : 1));
    std::vector<pigo_point> pts((size_t)(n > 0 ? n : 1) * face_cap * (2 + ncalls));
    const double* ang = angles.empty() ? nullptr : angles.data();
    const int rc = cparams ? pigo_detect_images_params(face.handle(), plc.handle(), hs.data(), fl.data(), ncalls, desc.data(), n, cparams, ang, &prm,
                                                       nullptr, rng_seed, faces.data(), face_cap, nfaces.data(), pts.data(), PIGO_MEM_HOST, nullptr)
                   : sharded ? pigo_detect_images_sharded(face.handle(), plc.handle(), hs.data(), fl.data(), ncalls, desc.data(), n, angles.data(), &prm,
                                                          nullptr, rng_seed, faces.data(), face_cap, nfaces.data(), pts.data())
                             : pigo_detect_images_angles(face.handle(), plc.handle(), hs.data(), fl.data(), ncalls, desc.data(), n, angles.data(), &prm,
                                                       nullptr, rng_seed, faces.data(), face_cap, nfaces.data(), pts.data(), PIGO_MEM_HOST, nullptr);
    if (rc == PIGO_E_CAP) {
      bool grown = false;
      for (int i = 0; i < n; ++i)
        if (nfaces[i] > face_cap) { face_cap = nfaces[i]; grown = true; }
      if (!grown) prm.det_cap = 4 * (prm.det_cap + 512);   // raw detections per image exceeded det_cap
      continue;
    }
    check(rc);
    std::vector<std::vector<FaceResult>> out((size_t)n);
    for (int f = 0; f < n; ++f)
      for (int k = 0; k < nfaces[f]; ++k) {
        const pigo_det& d = faces[(size_t)f * face_cap + k];
        FaceResult r;
        r.Face = Detection{d.row, d.col, d.scale, d.q};
        if (d.scale > min_face_scale) {
          const pigo_point* p = &pts[((size_t)f * face_cap + k) * (2 + ncalls)];
          r.Refined = true;
          r.LeftEye = Puploc{p[0].row, p[0].col, p[0].scale, 0}; r.RightEye = Puploc{p[1].row, p[1].col, p[1].scale, 0};
          for (int c = 0; c < ncalls; ++c) r.Landmarks.push_back(Puploc{p[2 + c].row, p[2 + c].col, p[2 + c].scale, 0});
        }
        out[f].push_back(r);
      }
    return out;
  }
}
}  // namespace detail

// additive: DetectImages with image i scanned and its eyes refined at angles[i] (one angle per image; the landmark calls stay
// at angle 0).  result[i] lists image i's clusters; on PIGO_E_CAP the call is retried with the reported face count (or a
// larger det_cap).
inline std::vector<std::vector<FaceResult>> DetectImagesAngles(const Pigo& face, const PuplocCascade& plc,
                                                               const std::vector<std::pair<const PuplocCascade*, bool>>& calls,
                                                               const std::vector<ImageParams>& images, const CascadeParams& cp, double iou,
                                                               int min_face_scale, int eye_perturbs, int flp_perturbs, uint64_t rng_seed,
                                                               const std::vector<double>& angles, int face_cap = 32) {
  if (angles.size() != images.size()) throw std::invalid_argument("DetectImagesAngles needs one angle per image");
  return detail::detectImages(face, plc, calls, images, cp, iou, min_face_scale, eye_perturbs, flp_perturbs, rng_seed, angles, face_cap, false);
}
// additive: DetectImagesAngles with every image's own CascadeParams (pigo_detect_images_params): image i is cps[i].Image, scanned
// with cps[i]'s MinSize, MaxSize, ShiftFactor and ScaleFactor and refined at angles[i] (empty: every image unrotated); iou, the
// face scale and the perturbs stay shared.  PIGO_E_CAP is retried as in DetectImagesAngles.
inline std::vector<std::vector<FaceResult>> DetectImagesParams(const Pigo& face, const PuplocCascade& plc,
                                                               const std::vector<std::pair<const PuplocCascade*, bool>>& calls,
                                                               const std::vector<CascadeParams>& cps, double iou, int min_face_scale, int eye_perturbs,
                                                               int flp_perturbs, uint64_t rng_seed, const std::vector<double>& angles = {},
                                                               int face_cap = 32) {
  if (!angles.empty() && angles.size() != cps.size()) throw std::invalid_argument("DetectImagesParams needs no angles or one angle per image");
  std::vector<ImageParams> images;
  for (const CascadeParams& cp : cps) images.push_back(cp.Image);
  const std::vector<pigo_cascade_params> prm = detail::params_of(cps);
  return detail::detectImages(face, plc, calls, images, CascadeParams{}, iou, min_face_scale, eye_perturbs, flp_perturbs, rng_seed, angles, face_cap,
                              false, prm.data());
}
// additive: DetectImagesAngles over the GPUs of InitDevices (host pixels, contiguous shards of about equal modelled cost); the
// result, generator keys included, equals the single-GPU call's
inline std::vector<std::vector<FaceResult>> DetectImagesSharded(const Pigo& face, const PuplocCascade& plc,
                                                                const std::vector<std::pair<const PuplocCascade*, bool>>& calls,
                                                                const std::vector<ImageParams>& images, const CascadeParams& cp, double iou,
                                                                int min_face_scale, int eye_perturbs, int flp_perturbs, uint64_t rng_seed,
                                                                const std::vector<double>& angles, int face_cap = 32) {
  if (angles.size() != images.size()) throw std::invalid_argument("DetectImagesSharded needs one angle per image");
  return detail::detectImages(face, plc, calls, images, cp, iou, min_face_scale, eye_perturbs, flp_perturbs, rng_seed, angles, face_cap, true);
}
// additive: DetectBatch for images of different sizes in one library call (host pixels; cp.Image is not used), every image at
// `angle`.  result[i] lists image i's clusters; PIGO_E_CAP is retried as in DetectImagesAngles.
inline std::vector<std::vector<FaceResult>> DetectImages(const Pigo& face, const PuplocCascade& plc,
                                                         const std::vector<std::pair<const PuplocCascade*, bool>>& calls,
                                                         const std::vector<ImageParams>& images, const CascadeParams& cp, double iou, int min_face_scale,
                                                         int eye_perturbs, int flp_perturbs, uint64_t rng_seed, double angle = 0.0, int face_cap = 32) {
  return DetectImagesAngles(face, plc, calls, images, cp, iou, min_face_scale, eye_perturbs, flp_perturbs, rng_seed,
                            std::vector<double>(images.size(), angle), face_cap);
}
// additive: DetectImages over an angle sweep (pigo_detect_images_sweep): every image scanned at every angle of `angles`, one
// merged face list per image, each face refined with its eyes at the angle it was found at (Angle, the listed value); the
// landmark calls stay at angle 0.  PIGO_E_CAP is retried as in DetectImagesAngles.
struct SweepFace {
  FaceResult Face;
  double Angle = 0.0;
};
inline std::vector<std::vector<SweepFace>> DetectImagesSweep(const Pigo& face, const PuplocCascade& plc,
                                                             const std::vector<std::pair<const PuplocCascade*, bool>>& calls,
                                                             const std::vector<ImageParams>& images, const CascadeParams& cp, double iou,
                                                             int min_face_scale, int eye_perturbs, int flp_perturbs, uint64_t rng_seed,
                                                             const std::vector<double>& angles, int face_cap = 32) {
  const int ncalls = (int)calls.size(), n = (int)images.size();
  std::vector<const pigo_puploc*> hs;
  std::vector<uint8_t> fl;
  for (auto& c : calls) { hs.push_back(c.first->handle()); fl.push_back(c.second ? 1 : 0); }
  std::vector<pigo_image> desc((size_t)n);
  for (int i = 0; i < n; ++i) desc[i] = pigo_image{images[i].Pixels, images[i].Rows, images[i].Cols, images[i].Dim};
  pigo_pipeline_params prm{};
  prm.min_size = cp.MinSize; prm.max_size = cp.MaxSize; prm.shift_factor = cp.ShiftFactor; prm.scale_factor = cp.ScaleFactor; prm.angle = 0.0;
  prm.iou_threshold = iou; prm.min_face_scale = min_face_scale; prm.eye_perturbs = eye_perturbs; prm.flp_perturbs = flp_perturbs; prm.det_cap = 0;
  for (;;) {
    std::vector<pigo_det> faces((size_t)(n > 0 ? n : 1) * face_cap);
    std::vector<int32_t> fangle(faces.size());
    std::vector<int> nfaces((size_t)(n > 0 ? n : 1));
    std::vector<pigo_point> pts((size_t)(n > 0 ? n : 1) * face_cap * (2 + ncalls));
    const int rc = pigo_detect_images_sweep(face.handle(), plc.handle(), hs.data(), fl.data(), ncalls, desc.data(), n, angles.data(), (int)angles.size(),
                                            &prm, nullptr, rng_seed, faces.data(), fangle.data(), face_cap, nfaces.data(), pts.data(), PIGO_MEM_HOST,
                                            nullptr);
    if (rc == PIGO_E_CAP) {
      bool grown = false;
      for (int i = 0; i < n; ++i)
        if (nfaces[i] > face_cap) { face_cap = nfaces[i]; grown = true; }
      if (!grown) prm.det_cap = 4 * (prm.det_cap + 512);   // raw detections of an (image, angle) entry exceeded det_cap
      continue;
    }
    check(rc);
    std::vector<std::vector<SweepFace>> out((size_t)n);
    for (int f = 0; f < n; ++f)
      for (int k = 0; k < nfaces[f]; ++k) {
        const size_t s = (size_t)f * face_cap + k;
        const pigo_det& d = faces[s];
        SweepFace r;
        r.Face.Face = Detection{d.row, d.col, d.scale, d.q};
        r.Angle = angles[(size_t)fangle[s]];
        if (d.scale > min_face_scale) {
          const pigo_point* p = &pts[s * (2 + ncalls)];
          r.Face.Refined = true;
          r.Face.LeftEye = Puploc{p[0].row, p[0].col, p[0].scale, 0}; r.Face.RightEye = Puploc{p[1].row, p[1].col, p[1].scale, 0};
          for (int c = 0; c < ncalls; ++c) r.Face.Landmarks.push_back(Puploc{p[2 + c].row, p[2 + c].col, p[2 + c].scale, 0});
        }
        out[f].push_back(r);
      }
    return out;
  }
}
inline PuplocCascade NewPuplocCascade() { return PuplocCascade(); }   // core/puploc.go:33

}  // namespace pigo
