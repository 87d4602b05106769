// The reference's landmark test (core/flploc_test.go:75-154: sample image -> one face with Scale > 50 -> both pupils -> 15
// landmark points, each with Row > 0 && Col > 0) on the sample swept at angles 0, 1/32 and 31/32 through DetectImagesSweep of
// the C++ mirror: one merged face list, whose face passes the reference's assertions, and RunCascadeImagesSweep lists the same
// clusters with the same angles; with the single angle 0 the sweep equals ClusterDetections of RunCascade.
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <vector>

#include "pigo_b200.hpp"

static std::vector<uint8_t> slurp(const std::string& p) {
  std::ifstream f(p, std::ios::binary);
  return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

int main(int argc, char** argv) {
  const std::string root = argc > 1 ? argv[1] : ".";
  const std::string cdir = root + "/pigo_b200/data/cascade/";
  const auto casc = slurp(cdir + "facefinder");
  const auto gray = slurp(root + "/tests/golden/sample_gray_400x320.u8");
  if (casc.empty() || gray.size() != 400 * 320) { std::fprintf(stderr, "fixtures missing\n"); return 2; }
  try {
    pigo::Pigo p = pigo::Pigo::Unpack(casc);
    pigo::PuplocCascade plc = pigo::PuplocCascade::UnpackCascade(slurp(cdir + "puploc"));
    std::vector<pigo::PuplocCascade> flp;
    const char* names[] = {"lp46", "lp44", "lp42", "lp38", "lp312", "lp93", "lp84", "lp82", "lp81"};
    for (const char* n : names) flp.push_back(pigo::PuplocCascade::UnpackFlp(cdir + "lps/" + n));
    std::vector<std::pair<const pigo::PuplocCascade*, bool>> calls;   // core/flploc_test.go:122-146
    for (int e = 0; e < 5; ++e) { calls.push_back({&flp[e], false}); calls.push_back({&flp[e], true}); }
    for (int m = 5; m < 9; ++m) calls.push_back({&flp[m], false});
    calls.push_back({&flp[6], true});
    const pigo::ImageParams sample{gray.data(), 400, 320, 320};
    std::vector<uint8_t> tiny(16, 0);
    const std::vector<pigo::ImageParams> images = {sample, pigo::ImageParams{tiny.data(), 4, 4, 4}};
    const std::vector<double> angles = {0.0, 1.0 / 32, 31.0 / 32};
    pigo::CascadeParams cp;
    cp.MinSize = 20; cp.MaxSize = 1000; cp.ShiftFactor = 0.2; cp.ScaleFactor = 1.1;   // core/pigo_test.go:44-50
    const auto all = pigo::DetectImagesSweep(p, plc, calls, images, cp, 0.1, 50, 50, 63, 7, angles);
    if (all.size() != images.size() || !all[1].empty()) return 1;
    int refined = 0;
    for (const auto& sf : all[0]) {
      if (sf.Face.Face.Scale <= 50) continue;
      ++refined;
      if (!sf.Face.Refined || sf.Face.Landmarks.size() != 15) return 1;
      for (const auto& lm : sf.Face.Landmarks)
        if (!(lm.Row > 0 && lm.Col > 0)) { std::printf("landmark (%d, %d) not inside the image\n", lm.Row, lm.Col); return 1; }
    }
    std::printf("sweep of the sample: %zu faces, %d refined\n", all[0].size(), refined);
    if (refined != 1) return 1;
    const auto dets = p.RunCascadeImagesSweep(images, cp, angles, 0.1);
    if (dets.size() != images.size() || dets[0].size() != all[0].size()) return 1;
    for (size_t k = 0; k < dets[0].size(); ++k) {
      const pigo::Detection& a = dets[0][k].Det;
      const pigo::Detection& b = all[0][k].Face.Face;
      if (std::memcmp(&a, &b, sizeof(a)) != 0 || dets[0][k].Angle != all[0][k].Angle) return 1;
    }
    pigo::CascadeParams one = cp;
    one.Image = sample;
    auto raw = p.RunCascade(one, 0.0);
    const auto cl = p.ClusterDetections(raw, 0.1);
    const auto single = p.RunCascadeImagesSweep({sample}, cp, {0.0}, 0.1);
    if (single[0].size() != cl.size()) return 1;
    for (size_t k = 0; k < cl.size(); ++k)
      if (std::memcmp(&single[0][k].Det, &cl[k], sizeof(pigo::Detection)) != 0 || single[0][k].Angle != 0.0) return 1;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "error: %s\n", e.what());
    return 1;
  }
  std::printf("OK\n");
  return 0;
}
