// A list of RunCascade calls with different CascadeParams, as the reference's callers use them (cmd/pigo, the test suite,
// the puploc and facedet examples), through RunCascadeImagesParams of the C++ mirror: each entry equals one RunCascade call
// with its own parameters and angle.  Then DetectImagesParams on the sample under the test suite's parameters passes the
// reference's landmark assertions (core/flploc_test.go:75-154) next to a tiny image under other parameters.
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

static pigo::CascadeParams params(const pigo::ImageParams& im, int mn, int mx, double shift, double scale) {
  pigo::CascadeParams cp;
  cp.Image = im; cp.MinSize = mn; cp.MaxSize = mx; cp.ShiftFactor = shift; cp.ScaleFactor = scale;
  return cp;
}

int main(int argc, char** argv) {
  const std::string root = argc > 1 ? argv[1] : ".";
  const std::string cdir = root + "/pigo_b200/data/cascade/";
  const auto casc = slurp(cdir + "facefinder");
  const auto gray = slurp(root + "/tests/golden/sample_gray_400x320.u8");
  if (casc.empty() || gray.size() != 400 * 320) { std::fprintf(stderr, "fixtures missing\n"); return 2; }
  try {
    pigo::Pigo p = pigo::Pigo::Unpack(casc);
    const pigo::ImageParams sample{gray.data(), 400, 320, 320};
    std::vector<uint8_t> tiny(16, 0);
    const pigo::ImageParams small{tiny.data(), 4, 4, 4};
    const std::vector<pigo::CascadeParams> cps = {params(sample, 20, 1000, 0.2, 1.1), params(sample, 20, 1000, 0.15, 1.15),
                                                  params(sample, 60, 600, 0.1, 1.1), params(small, 20, 1000, 0.2, 1.1),
                                                  params(sample, 100, 600, 0.15, 1.1)};
    const std::vector<double> angles = {0.0, 0.1, 0.0, 0.0, 0.5};
    const auto dets = p.RunCascadeImagesParams(cps, angles);
    if (dets.size() != cps.size()) return 1;
    size_t found = 0;
    for (size_t i = 0; i < cps.size(); ++i) {
      const auto e = p.RunCascade(cps[i], angles[i]);
      if (e.size() != dets[i].size()) { std::printf("entry %zu: %zu vs %zu detections\n", i, dets[i].size(), e.size()); return 1; }
      for (size_t k = 0; k < e.size(); ++k)
        if (std::memcmp(&e[k], &dets[i][k], sizeof(pigo::Detection)) != 0) { std::printf("entry %zu differs at %zu\n", i, k); return 1; }
      found += e.size();
    }
    const auto unrotated = p.RunCascadeImagesParams(cps);
    for (size_t i = 0; i < cps.size(); ++i)
      if (unrotated[i].size() != p.RunCascade(cps[i], 0.0).size()) return 1;

    pigo::PuplocCascade plc = pigo::PuplocCascade::UnpackCascade(slurp(cdir + "puploc"));
    std::vector<pigo::PuplocCascade> flp;
    const char* names[] = {"lp46", "lp44", "lp42", "lp38", "lp312", "lp93", "lp84", "lp82", "lp81"};
    for (const char* n : names) flp.push_back(pigo::PuplocCascade::UnpackFlp(cdir + "lps/" + n));
    std::vector<std::pair<const pigo::PuplocCascade*, bool>> calls;   // core/flploc_test.go:122-146
    for (int e = 0; e < 5; ++e) { calls.push_back({&flp[e], false}); calls.push_back({&flp[e], true}); }
    for (int m = 5; m < 9; ++m) calls.push_back({&flp[m], false});
    calls.push_back({&flp[6], true});
    const std::vector<pigo::CascadeParams> pcs = {params(small, 60, 600, 0.1, 1.1), params(sample, 20, 1000, 0.2, 1.1)};
    const auto all = pigo::DetectImagesParams(p, plc, calls, pcs, 0.1, 50, 50, 63, 7);
    if (all.size() != pcs.size() || !all[0].empty()) return 1;
    int refined = 0;
    for (const auto& fr : all[1]) {
      if (fr.Face.Scale <= 50) continue;
      ++refined;
      if (!fr.Refined || fr.Landmarks.size() != 15) return 1;
      for (const auto& lm : fr.Landmarks)
        if (!(lm.Row > 0 && lm.Col > 0)) { std::printf("landmark (%d, %d) not inside the image\n", lm.Row, lm.Col); return 1; }
    }
    std::printf("%zu detections over %zu entries, sample faces %zu, refined %d\n", found, cps.size(), all[1].size(), refined);
    return refined == 1 && found > 0 ? 0 : 1;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
}
