// The sharded mixed-size calls through the C++ mirror: RunCascadeImagesSharded and DetectImagesSharded equal
// RunCascadeImagesAngles and DetectImagesAngles (same rng_seed: the generator keys must not depend on the split) for the
// shard count given on the command line (option shard_split), on the sample image placed among other images at mixed
// angles.  The sample entry also passes the reference's landmark assertions (core/flploc_test.go:75-154): one face with
// Scale > 50 and 15 landmark points inside the image.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <vector>

#include "pigo_b200.hpp"

static std::vector<uint8_t> slurp(const std::string& p) {
  std::ifstream f(p, std::ios::binary);
  return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

static bool same(const pigo::Puploc& a, const pigo::Puploc& b) {
  return a.Row == b.Row && a.Col == b.Col && std::memcmp(&a.Scale, &b.Scale, sizeof(float)) == 0;
}

int main(int argc, char** argv) {
  const std::string root = argc > 1 ? argv[1] : ".";
  const int split = argc > 2 ? std::atoi(argv[2]) : 3;
  const std::string cdir = root + "/pigo_b200/data/cascade/";
  const auto casc = slurp(cdir + "facefinder");
  const auto gray = slurp(root + "/tests/golden/sample_gray_400x320.u8");
  if (casc.empty() || gray.size() != 400 * 320) { std::fprintf(stderr, "fixtures missing\n"); return 2; }
  try {
    pigo::check(pigo_set_option("shard_split", split));
    pigo::Pigo p = pigo::Pigo::Unpack(casc);
    pigo::PuplocCascade plc = pigo::PuplocCascade::UnpackCascade(slurp(cdir + "puploc"));
    std::vector<pigo::PuplocCascade> flp;
    const char* names[] = {"lp46", "lp44", "lp42", "lp38", "lp312", "lp93", "lp84", "lp82", "lp81"};
    for (const char* n : names) flp.push_back(pigo::PuplocCascade::UnpackFlp(cdir + "lps/" + n));
    std::vector<std::pair<const pigo::PuplocCascade*, bool>> calls;   // core/flploc_test.go:122-146
    for (int e = 0; e < 5; ++e) { calls.push_back({&flp[e], false}); calls.push_back({&flp[e], true}); }
    for (int m = 5; m < 9; ++m) calls.push_back({&flp[m], false});
    calls.push_back({&flp[6], true});
    // the sample among other images: tiny, wide, odd-sized and a 1080p frame (pseudo-random pixels), some listed twice
    std::vector<uint8_t> tiny(16, 7), noise((size_t)1080 * 1921);
    unsigned x = 12345;
    for (auto& b : noise) { x = x * 1103515245u + 12345u; b = (uint8_t)(x >> 16); }
    const pigo::ImageParams sample{gray.data(), 400, 320, 320};
    const std::vector<pigo::ImageParams> images = {pigo::ImageParams{tiny.data(), 4, 4, 4}, pigo::ImageParams{noise.data(), 97, 333, 335},
                                                   sample, pigo::ImageParams{noise.data(), 1080, 1920, 1921}, sample,
                                                   pigo::ImageParams{noise.data(), 301, 1200, 1201}, sample};
    const std::vector<double> angles = {0.0, 0.0, 0.0, 0.25, 0.1, 0.5, 0.0};
    pigo::CascadeParams cp;
    cp.MinSize = 20; cp.MaxSize = 1000; cp.ShiftFactor = 0.2; cp.ScaleFactor = 1.1;   // core/pigo_test.go:44-50
    const auto d1 = p.RunCascadeImagesAngles(images, cp, angles), ds = p.RunCascadeImagesSharded(images, cp, angles);
    for (size_t i = 0; i < images.size(); ++i) {
      if (d1[i].size() != ds[i].size()) { std::printf("image %zu: %zu vs %zu detections\n", i, d1[i].size(), ds[i].size()); return 1; }
      for (size_t k = 0; k < d1[i].size(); ++k)
        if (std::memcmp(&d1[i][k], &ds[i][k], sizeof(pigo::Detection)) != 0) return 1;
    }
    const auto f1 = pigo::DetectImagesAngles(p, plc, calls, images, cp, 0.1, 50, 50, 63, 11, angles);
    const auto fs = pigo::DetectImagesSharded(p, plc, calls, images, cp, 0.1, 50, 50, 63, 11, angles);
    for (size_t i = 0; i < images.size(); ++i) {
      if (f1[i].size() != fs[i].size()) return 1;
      for (size_t k = 0; k < f1[i].size(); ++k) {
        const auto &a = f1[i][k], &b = fs[i][k];
        if (std::memcmp(&a.Face, &b.Face, sizeof(pigo::Detection)) != 0 || a.Refined != b.Refined || a.Landmarks.size() != b.Landmarks.size())
          return 1;
        if (a.Refined && (!same(a.LeftEye, b.LeftEye) || !same(a.RightEye, b.RightEye))) return 1;
        for (size_t c = 0; c < a.Landmarks.size(); ++c)
          if (!same(a.Landmarks[c], b.Landmarks[c])) return 1;
      }
    }
    int refined = 0;
    for (const auto& fr : fs[2]) {
      if (fr.Face.Scale <= 50) continue;
      ++refined;
      if (!fr.Refined || fr.Landmarks.size() != 15) return 1;
      for (const auto& lm : fr.Landmarks)
        if (!(lm.Row > 0 && lm.Col > 0)) { std::printf("landmark (%d, %d) not inside the image\n", lm.Row, lm.Col); return 1; }
    }
    std::printf("shard_split %d: sample faces %zu, refined %d\n", split, fs[2].size(), refined);
    return refined == 1 ? 0 : 1;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
}
