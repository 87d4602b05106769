// Replays the reference's landmark test (core/flploc_test.go:75-154: sample image -> face -> both pupils -> 15 landmark
// points, each with Row > 0 && Col > 0) with the sample image inside a mixed-size batch, through DetectImages of the C++
// mirror; a second call that starts from face_cap 1 must take the PIGO_E_CAP retry and find the same faces.
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

static bool same(const pigo::Puploc& a, const pigo::Puploc& b) { return a.Row == b.Row && a.Col == b.Col && a.Scale == b.Scale; }

int main(int argc, char** argv) {
  const std::string root = argc > 1 ? argv[1] : ".";
  const std::string cdir = root + "/pigo_b200/data/cascade/";
  const auto casc = slurp(cdir + "facefinder");
  const auto gray = slurp(root + "/tests/golden/sample_gray_400x320.u8");
  if (casc.empty() || gray.size() != 400 * 320) { std::fprintf(stderr, "fixtures missing\n"); return 2; }
  try {
    pigo::Pigo p = pigo::Pigo::Unpack(casc);
    pigo::PuplocCascade plc = pigo::PuplocCascade::UnpackCascade(slurp(cdir + "puploc"));
    // the reference's 15-call sequence (core/flploc_test.go:122-146)
    std::vector<pigo::PuplocCascade> flp;
    const char* names[] = {"lp46", "lp44", "lp42", "lp38", "lp312", "lp93", "lp84", "lp82", "lp81"};
    for (const char* n : names) flp.push_back(pigo::PuplocCascade::UnpackFlp(cdir + "lps/" + n));
    std::vector<std::pair<const pigo::PuplocCascade*, bool>> calls;
    for (int e = 0; e < 5; ++e) { calls.push_back({&flp[e], false}); calls.push_back({&flp[e], true}); }
    for (int m = 5; m < 9; ++m) calls.push_back({&flp[m], false});
    calls.push_back({&flp[6], true});
    // around the sample: a tiny image, a wide strided image tiled from the sample (two faces side by side), and noise
    const int WR = 420, WC = 700, WD = 720, NR = 120, NC = 90;
    std::vector<uint8_t> wide((size_t)WR * WD, 0), noise((size_t)NR * NC), tiny(16, 0);
    for (int y = 0; y < WR; ++y)
      for (int x = 0; x < WC; ++x) wide[(size_t)y * WD + x] = gray[(size_t)(y % 400) * 320 + (x % 350 < 320 ? x % 350 : 0)];
    uint32_t s = 12345;
    for (auto& v : noise) { s = s * 1664525u + 1013904223u; v = (uint8_t)(s >> 24); }
    const std::vector<pigo::ImageParams> images = {pigo::ImageParams{tiny.data(), 4, 4, 4}, pigo::ImageParams{wide.data(), WR, WC, WD},
                                                   pigo::ImageParams{gray.data(), 400, 320, 320}, pigo::ImageParams{noise.data(), NR, NC, NC}};
    pigo::CascadeParams cp;
    cp.MinSize = 20; cp.MaxSize = 1000; cp.ShiftFactor = 0.2; cp.ScaleFactor = 1.1;   // core/pigo_test.go:44-50
    const auto all = pigo::DetectImages(p, plc, calls, images, cp, 0.1, 50, 50, 63, 7);
    if (all.size() != images.size()) return 1;
    int refined = 0;
    for (const auto& fr : all[2]) {
      if (!fr.Refined) continue;
      ++refined;
      if (fr.Face.Scale <= 50 || fr.Landmarks.size() != 15) return 1;
      for (const auto& lm : fr.Landmarks)
        if (!(lm.Row > 0 && lm.Col > 0)) { std::printf("landmark (%d, %d) not inside the image\n", lm.Row, lm.Col); return 1; }
    }
    std::printf("images=%zu sample faces=%zu refined=%d wide faces=%zu\n", all.size(), all[2].size(), refined, all[1].size());
    if (refined != 1) return 1;
    // PIGO_E_CAP retry: the wide image holds more than one face.  The library generator's key includes face_cap (the slot
    // index), so the retried call's points come from other randoms: compare the faces, and the points of a third call with
    // the face_cap the retry settled on.
    if (all[1].size() < 2) return 1;
    const auto again = pigo::DetectImages(p, plc, calls, images, cp, 0.1, 50, 50, 63, 7, 0.0, 1);
    int need = 1;
    for (const auto& v : all) need = (int)v.size() > need ? (int)v.size() : need;
    const auto direct = pigo::DetectImages(p, plc, calls, images, cp, 0.1, 50, 50, 63, 7, 0.0, need);
    for (size_t i = 0; i < images.size(); ++i) {
      if (again[i].size() != all[i].size() || direct[i].size() != all[i].size()) return 1;
      for (size_t k = 0; k < all[i].size(); ++k) {
        const auto &a = all[i][k], &b = again[i][k], &d = direct[i][k];
        if (std::memcmp(&a.Face, &b.Face, sizeof(pigo::Detection)) != 0 || a.Refined != b.Refined) return 1;
        if (b.Refined && (!same(b.LeftEye, d.LeftEye) || !same(b.RightEye, d.RightEye))) return 1;
        for (size_t c = 0; c < b.Landmarks.size(); ++c)
          if (!same(b.Landmarks[c], d.Landmarks[c])) return 1;
      }
    }
    return 0;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
}
