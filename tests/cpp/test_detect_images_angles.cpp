// The reference's landmark test (core/flploc_test.go:75-154: sample image -> one face with Scale > 50 -> both pupils -> 15
// landmark points, each with Row > 0 && Col > 0) on the sample placed in an angle sweep (angles 0, 0.1, 0.5) through
// DetectImagesAngles of the C++ mirror: the angle-0 entry passes the reference's assertions, and a RunCascadeImagesAngles
// sweep over the same list equals one RunCascade call per entry.
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
    const std::vector<pigo::ImageParams> images = {pigo::ImageParams{tiny.data(), 4, 4, 4}, sample, sample, sample};
    const std::vector<double> angles = {0.0, 0.0, 0.1, 0.5};
    pigo::CascadeParams cp;
    cp.MinSize = 20; cp.MaxSize = 1000; cp.ShiftFactor = 0.2; cp.ScaleFactor = 1.1;   // core/pigo_test.go:44-50
    const auto all = pigo::DetectImagesAngles(p, plc, calls, images, cp, 0.1, 50, 50, 63, 7, angles);
    if (all.size() != images.size()) return 1;
    int refined = 0;
    for (const auto& fr : all[1]) {
      if (fr.Face.Scale <= 50) continue;
      ++refined;
      if (!fr.Refined || fr.Landmarks.size() != 15) return 1;
      for (const auto& lm : fr.Landmarks)
        if (!(lm.Row > 0 && lm.Col > 0)) { std::printf("landmark (%d, %d) not inside the image\n", lm.Row, lm.Col); return 1; }
    }
    std::printf("sweep faces at 0 / 0.1 / 0.5: %zu %zu %zu, refined at 0: %d\n", all[1].size(), all[2].size(), all[3].size(), refined);
    if (refined != 1) return 1;
    const auto dets = p.RunCascadeImagesAngles(images, cp, angles);
    for (size_t i = 0; i < images.size(); ++i) {
      pigo::CascadeParams one = cp;
      one.Image = images[i];
      const auto e = p.RunCascade(one, angles[i]);
      if (e.size() != dets[i].size()) return 1;
      for (size_t k = 0; k < e.size(); ++k)
        if (std::memcmp(&e[k], &dets[i][k], sizeof(pigo::Detection)) != 0) return 1;
    }
    return 0;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
}
