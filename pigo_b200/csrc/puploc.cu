// puploc.cu -- PuplocCascade.RunDetector (core/puploc.go:239-277) for a batch of seeds on one image:
// one CTA per seed, one warp per perturbation, one lane per tree of a stage, then the three independent 63-slot sorts
// and the "median" pick of the reference.  classifyRegion / classifyRotatedRegion (core/puploc.go:106-217) walk
// stages x trees x depth pixel-pair tests with global-memory gathers; tables stay L2/L1-resident.
//
// float32 arithmetic uses explicit round-to-nearest intrinsics (and the library is built with
// -fmad=false): Go on amd64 never fuses r += dr*s (core/puploc.go:149-151).
#include <algorithm>
#include <climits>

#include "common.cuh"
#include "host.h"

namespace pigo {

__device__ __constant__ float c_qcosf[33] = {256, 251, 236, 212, 181, 142, 97, 49, 0, -49, -97, -142, -181, -212, -236, -251, -256,
                                             -251, -236, -212, -181, -142, -97, -49, 0, 49, 97, 142, 181, 212, 236, 251, 256};
__device__ __constant__ float c_qsinf[33] = {0, 49, 97, 142, 181, 212, 236, 251, 256, 251, 236, 212, 181, 142, 97, 49, 0,
                                             -49, -97, -142, -181, -212, -236, -251, -256, -251, -236, -212, -181, -142, -97, -49, 0};

// int8 negation wraps in Go: -int8(-128) == -128 (core/puploc.go:124-125, :181-182)
__device__ __forceinline__ int neg_i8(int v) { return (int)(int8_t)(-v); }

__device__ __forceinline__ uint32_t mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  x ^= x >> 31;
  return (uint32_t)(x >> 40);  // 24 random bits
}

// Rank order of the 63-slot pool sorts, a total order so that exactly
// one slot has each rank: numbers ascending (-0 == +0), every NaN above every number, ties (NaNs among themselves too)
// by slot index.  The reference's sort.Sort order is an accident of its algorithm once NaNs take part (DESIGN.md §3.3).
// rank_key maps a value to an unsigned key in that order; value j comes before value i when key j < key i, or when the keys
// are equal and j < i.
__device__ __forceinline__ unsigned rank_key(float v) {
  if (v != v) return 0xFFFFFFFFu;
  const unsigned b = __float_as_uint(v == 0.f ? 0.f : v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// One CTA (32 warps) per seed; one WARP per perturbation (two rounds cover the 63 slots) and one LANE per tree of the
// current stage: the trees of a stage are independent of each other (they all start from the stage's (r, c, s)), only
// the float32 sums dr, dc are order-sensitive -- lanes walk the trees in parallel, then the sums are formed in tree order
// with shuffles, exactly like the reference's sequential loop (core/puploc.go:112-151).  That turns the reference's
// stages*trees*depth = 1000-deep dependent gather chain into stages*depth = 50; the two children of a node are fetched
// together with the node's pixel pair (child-pair prefetch).
// IMG (mixed-size call): seed_frame indexes the image table `images`, whose entry gives the pixels, rows, cols and pitch;
// frames / frame_stride / nrows / ncols / dim are then unused, and rot_slot == kRotSlotPerImage takes the image's slot.
template <bool IMG = false>
__global__ void __launch_bounds__(1024, 1) puploc_kernel(PuplocTables T, const pigo_point* __restrict__ seeds, int nseeds,
                                                         const float* __restrict__ randoms, uint64_t rng_seed,
                                                         const uint8_t* __restrict__ frames, const int32_t* __restrict__ seed_frame,
                                                         size_t frame_stride, int frame_rows, int frame_cols, int frame_dim,
                                                         int rot_slot, const uint8_t* __restrict__ flipv_arr,
                                                         pigo_point* __restrict__ out, const ImageDesc* __restrict__ images) {
  const unsigned FULL = 0xffffffffu;
  const int sidx = blockIdx.x;
  const ImageDesc im = IMG ? images[seed_frame ? seed_frame[sidx] : 0] : ImageDesc{};
  const uint8_t* __restrict__ pixels = IMG ? im.base : frames + (seed_frame ? (size_t)seed_frame[sidx] * frame_stride : 0);
  const int nrows = IMG ? im.rows : frame_rows, ncols = IMG ? im.cols : frame_cols, dim = IMG ? im.dim : frame_dim;
  if (IMG && rot_slot == kRotSlotPerImage) rot_slot = im.rot_slot;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ float rows_[64], cols_[64], scal_[64];
  __shared__ unsigned krow_[64], kcol_[64], kscal_[64];   // their rank_key
  const pigo_point seed = seeds[sidx];
  if (seed.perturbs < 0) return;               // inactive seed (CTA-uniform): out[sidx] is left as it is, like the pair kernel's
  const int P = min(seed.perturbs, 63);        // device seeds are not checked on the host: Perturbs above 63 run as 63
  const bool flip = flipv_arr ? (flipv_arr[sidx] != 0) : false;
  const int L = T.leaves;
  const int tree_codes = 4 * L;   // device layout: one pad word, then the 4L-4 code bytes (node i at word i+1), see PuplocTables

  for (int i = warp; i < 63; i += 32) {       // warp-uniform: perturbation i (pool slot i)
    float r = 0.f, c = 0.f, s = 0.f;
    if (i < P) {
      float u0, u1, u2;
      if (randoms) {
        const float* rr = randoms + ((size_t)sidx * 63 + i) * 3;
        u0 = rr[0]; u1 = rr[1]; u2 = rr[2];
      } else {
        const uint64_t key = rng_seed * 0xD1342543DE82EF95ull + (uint64_t)sidx * 64 + i;
        u0 = mix64(key * 3 + 0) * (1.0f / 16777216.0f);
        u1 = mix64(key * 3 + 1) * (1.0f / 16777216.0f);
        u2 = mix64(key * 3 + 2) * (1.0f / 16777216.0f);
      }
      const float t1 = __fmul_rn(seed.scale, 0.15f);
      r = __fadd_rn((float)seed.row, __fmul_rn(t1, __fsub_rn(0.5f, u0)));   // core/puploc.go:248
      c = __fadd_rn((float)seed.col, __fmul_rn(t1, __fsub_rn(0.5f, u1)));   // :249
      s = __fmul_rn(seed.scale, __fadd_rn(0.925f, __fmul_rn(0.15f, u2)));   // :250
      int iqs = 0, iqc = 0;
      if (rot_slot >= 0) {
        iqs = (int)__fmul_rn(s, c_qsinf[rot_slot]);  // int(qsin), :166, :188 (from the INITIAL s)
        iqc = (int)__fmul_rn(s, c_qcosf[rot_slot]);
      }
      for (int st = 0; st < T.stages; ++st) {
        float dr = 0.f, dc = 0.f;
        const long long ir = (long long)r, ic = (long long)c;  // int(r): truncation toward zero
        const long long rs = llround((double)s);               // int(math.Round(float64(s)))
        for (int j0 = 0; j0 < T.trees; j0 += 32) {             // 32 trees of the stage at a time, one per lane
          const int j = min(j0 + lane, T.trees - 1);           // surplus lanes redo the last tree (ignored below)
          const size_t tg = (size_t)st * T.trees + j;
          const int* tc = reinterpret_cast<const int*>(T.codes + tg * tree_codes);   // 4-byte aligned: tree_codes % 4 == 0
          const float2* tp = reinterpret_cast<const float2*>(T.preds + tg * 2 * L);
          int idx = 0;
          int cw = __ldg(tc + 1);
          for (int k = 0; k < T.depth; ++k) {
            // children of node idx are nodes 2idx+1, 2idx+2 = words 2idx+2, 2idx+3: one aligned 64-bit load, in flight with this node's pixels
            int kl = 0, kr = 0;
            if (k + 1 < T.depth) { const int2 kk = __ldg(reinterpret_cast<const int2*>(tc) + idx + 1); kl = kk.x; kr = kk.y; }
            const int k0 = (int8_t)(cw), k2 = (int8_t)(cw >> 16);
            const int k1 = flip ? neg_i8((int8_t)(cw >> 8)) : (int)(int8_t)(cw >> 8);
            const int k3 = flip ? neg_i8(cw >> 24) : (cw >> 24);
            long long r1, c1, r2, c2;
            int bit;
            if (rot_slot < 0) {
              r1 = min((long long)nrows - 1, max(0ll, (256 * ir + k0 * rs) >> 8));   // :118
              r2 = min((long long)nrows - 1, max(0ll, (256 * ir + k2 * rs) >> 8));   // :119
              c1 = min((long long)ncols - 1, max(0ll, (256 * ic + k1 * rs) >> 8));   // :124/:127
              c2 = min((long long)ncols - 1, max(0ll, (256 * ic + k3 * rs) >> 8));
              bit = __ldg(pixels + r1 * dim + c1) > __ldg(pixels + r2 * dim + c2) ? 1 : 0;   // :130-136
            } else {
              r1 = min((long long)nrows - 1, max(0ll, 65536 * ir + (long long)iqc * k0 - (long long)iqs * k1) >> 16);  // :188
              c1 = min((long long)ncols - 1, max(0ll, 65536 * ic + (long long)iqs * k0 + (long long)iqc * k1) >> 16);  // :189
              r2 = min((long long)nrows - 1, max(0ll, 65536 * ir + (long long)iqc * k2 - (long long)iqs * k3) >> 16);  // :190
              c2 = min((long long)ncols - 1, max(0ll, 65536 * ic + (long long)iqs * k2 + (long long)iqc * k3) >> 16);  // :191
              bit = __ldg(pixels + r1 * dim + c1) <= __ldg(pixels + r2 * dim + c2) ? 1 : 0;  // :193-199
            }
            cw = bit ? kr : kl;
            idx = 2 * idx + 1 + bit;
          }
          const float2 leaf = __ldg(tp + (idx - (L - 1)));
          const int nv = min(32, T.trees - j0);
          for (int q = 0; q < nv; ++q) {                       // the reference's tree-ordered float32 sums, :140-145
            const float pr = __shfl_sync(FULL, leaf.x, q), pc = __shfl_sync(FULL, leaf.y, q);
            dr = __fadd_rn(dr, pr);
            dc = __fadd_rn(dc, flip ? -pc : pc);
          }
        }
        r = __fadd_rn(r, __fmul_rn(dr, s));   // :149
        c = __fadd_rn(c, __fmul_rn(dc, s));   // :150
        s = __fmul_rn(s, T.scales);           // :151
      }
    }
    // pool slots >= Perturbs stay 0 (fresh pool object, :228-236); all 63 slots are sorted (:267-269)
    if (lane == 0) { rows_[i] = r; cols_[i] = c; scal_[i] = s; krow_[i] = rank_key(r); kcol_[i] = rank_key(c); kscal_[i] = rank_key(s); }
  }
  __syncthreads();
  const int i = threadIdx.x;
  const int mid = (int)llround((double)P / 2);  // int(math.Round(float64(Perturbs)/2)), :273
  if (i < 63) {
    // rank sort of 63 values (rank_key, ties: index order); the thread whose rank == mid publishes it
    const unsigned vr = krow_[i], vc = kcol_[i], vs = kscal_[i];
    int kr = 0, kc = 0, ks = 0;
    for (int j = 0; j < 63; ++j) {
      kr += (krow_[j] < vr || (krow_[j] == vr && j < i)) ? 1 : 0;
      kc += (kcol_[j] < vc || (kcol_[j] == vc && j < i)) ? 1 : 0;
      ks += (kscal_[j] < vs || (kscal_[j] == vs && j < i)) ? 1 : 0;
    }
    if (kr == mid) out[sidx].row = (int)rows_[i];      // int() truncation, :273
    if (kc == mid) out[sidx].col = (int)cols_[i];
    if (ks == mid) out[sidx].scale = scal_[i];
    if (i == 0) out[sidx].perturbs = 0;          // the returned Puploc leaves Perturbs unset (:272-276)
  }
}

// ============================================================================================================
// Round 2 kernel: (perturbation, tree) PAIRS.  The trees of a stage are independent of each other and so are the
// perturbations, so a stage of one RunDetector call is P x trees independent tree walks (63 x 20 = 1260 for a landmark
// call): they are dealt to the threads of the CTA as a flat list -- every lane walks a real tree (the warp-per-perturbation
// kernel above keeps 20 of 32 lanes busy) -- the leaves go to shared memory, and one thread per perturbation forms the
// float32 sums dr, dc in TREE ORDER exactly like the reference's sequential loop (core/puploc.go:138-151).
// CTAs are persistent and pull work items (one RunDetector call each) from a global counter; an item is addressed as
// slot = (w / span) * stride + first + w % span, which lets one launch cover e.g. "the two eye seeds of every face slot"
// or "the 15 landmark calls of every face slot", each position j = w % span with its own cascade and flip flag.
// Inactive slots (seed.perturbs < 0) are skipped.  32-bit coordinate arithmetic, exact because
//   (256*int(r) + code*rs) >> 8  ==  int(r) + ((code*rs) >> 8)        (256*int(r) is a multiple of 256), and
//   max(0, 65536*int(r) + x) >> 16  ==  max(0, int(r) + (x >> 16))    (rotated variant, see RotNode in common.cuh);
// exact while |int(Round(s))| < 2^24 at every stage; the host leaves seeds with |Scale| * max(1, |scales|)^(stages-1) > 16384
// to the 64-bit kernel above (standalone calls) or refuses cascades whose scale grows by more than 512 (pipeline).
constexpr int kPairThreads = 512;
// Sample area of one perturbation in the coming stage: centre +- (|rs|/2 + 1) unrotated ((code*rs) >> 8 with |code| <= 128);
// rotated: the offsets are (iqc*k0 -+ iqs*k1) >> 16 with iqc, iqs fixed from the INITIAL scale of the perturbation (core/puploc.go:166),
// so the radius comes from them, not from the current scale.
__device__ __forceinline__ void box_add(int* box, int ir, int ic, int rs, bool rot, int iqs, int iqc) {
  const int a = rs < 0 ? -rs : rs;
  const int h = rot ? (((iqs < 0 ? -iqs : iqs) + (iqc < 0 ? -iqc : iqc)) >> 9) + 2 : (a >> 1) + 2;   // |iqc*k0 - iqs*k1| >> 16 <= (|iqc| + |iqs|) * 128 >> 16
  atomicMin(&box[0], ir - h); atomicMax(&box[1], ir + h);
  atomicMin(&box[2], ic - h); atomicMax(&box[3], ic + h);
}
// int(r) of core/puploc.go:118, kept inside +-2^30 so that adding a sample offset (|offset| <= |scale|/2 < 2^23, the host
// rejects larger scales) cannot wrap: anything beyond +-2^30 clamps to the same image border as the exact value would
__device__ __forceinline__ int clamp_coord(float v) { return max(-(1 << 30), min(1 << 30, (int)v)); }

// STAGED: the node codes of the CURRENT STAGE (trees x 4L bytes: 40 KB for a landmark cascade, 80 KB for the pupil cascade)
// are copied to shared memory with coalesced loads before the stage's walks, so that the per-level child fetch is a
// shared-memory load instead of a lane-divergent global one (the unstaged kernel is bound by L1TEX sectors); the shared copy skews consecutive trees by 8 bytes, otherwise every tree's node i would sit in the
// same bank.  The pixel pairs stay global gathers (a landmark seed's patch is up to ~100 KB).
// PATCH (with STAGED): before a stage whose sample area -- the bounding box of all perturbations' centres +- scale/2, clamped
// to the image -- fits `patch_cap` bytes, that area is copied to shared memory with coalesced 16-byte loads and the
// stage's pixel pairs become shared-memory loads too (a stage gathers 1260 x depth x 2 lane-divergent bytes from it; the
// scale shrinks by 0.7-0.8 per stage, so the later stages of a landmark call fit).  Stages that do not fit gather from global memory.
// IMG (mixed-size call): the slot's frame index selects an entry of the image table W.images, which gives the pixels, the
// clamps rows-1 / cols-1 and the row pitch (the patch's 16-byte path then needs that image's pitch and base aligned), and
// with W.rot_slot == kRotSlotPerImage the rotation table slot; with W.rot_slot == kRotSlotPerFace (angle sweep) the slot
// comes from W.face_rot of the slot's face, slot / W.stride.
template <bool STAGED, bool PATCH, bool IMG = false>
__global__ void __launch_bounds__(kPairThreads, PATCH ? 2 : 3) puploc_pair_kernel(const PupWork W, unsigned int* __restrict__ counter, int leaf_bytes,
                                                                                 int codes_bytes, int patch_cap) {
  extern __shared__ __align__(16) uint8_t s_dyn[];
  float2* s_leaf = reinterpret_cast<float2*>(s_dyn);     // [63][trees]
  uint8_t* s_codes = s_dyn + leaf_bytes;                 // STAGED: [trees][4L + 8]
  uint8_t* s_patch = s_codes + codes_bytes;              // PATCH: [rows][pitch]
  __shared__ int s_box[4];                               // PATCH: min row, max row, min col, max col over the perturbations
  __shared__ float s_r[64], s_c[64], s_s[64];
  __shared__ int s_ir[64], s_ic[64], s_rs[64], s_qs[64], s_qc[64];
  __shared__ unsigned s_item;
  const int tid = threadIdx.x, nt = blockDim.x;
  for (;;) {
    __syncthreads();
    if (tid == 0) {
      s_item = atomicAdd(counter, 1u);
      if (PATCH) { s_box[0] = INT_MAX; s_box[1] = INT_MIN; s_box[2] = INT_MAX; s_box[3] = INT_MIN; }
    }
    __syncthreads();
    const unsigned w = s_item;
    if (w >= (unsigned)W.nwork) break;
    const int j = (int)(w % (unsigned)W.span);
    const int slot = (int)(w / (unsigned)W.span) * W.stride + W.first + j;
    const pigo_point seed = W.seeds[slot];
    if (seed.perturbs < 0) continue;                       // inactive slot (CTA-uniform)
    const int P = min(seed.perturbs, 63);                  // device seeds are not checked on the host: Perturbs above 63 run as 63
    const PuplocTables T = W.tab[W.tab_of[j]];
    const bool flip = W.flipv ? (W.flipv[slot] != 0) : (W.flip_of[j] != 0);
    const int frame = W.slots_per_frame > 0 ? slot / W.slots_per_frame : (W.slot_frame ? W.slot_frame[slot] : 0);
    const uint8_t* __restrict__ pixels = IMG ? W.images[frame].base : W.frames + (size_t)frame * W.frame_stride;
    auto dim = [&]() { return IMG ? W.images[frame].dim : W.dim; };   // row pitch (read at each use, as W.dim was before IMG)
    const int L = T.leaves, tree_codes = 4 * L, rlim = (IMG ? W.images[frame].rows : W.nrows) - 1, clim = (IMG ? W.images[frame].cols : W.ncols) - 1;   // padded device layout, see PuplocTables
    const int rot_slot = (IMG && W.rot_slot == kRotSlotPerImage) ? W.images[frame].rot_slot
                         : (IMG && W.rot_slot == kRotSlotPerFace) ? W.face_rot[slot / W.stride] : W.rot_slot;
    const bool rot = rot_slot >= 0;
    const int sstride = tree_codes + 8;                    // shared-memory tree stride (bank skew)
    auto stage_codes = [&](int st) {
      const uint2* src = reinterpret_cast<const uint2*>(T.codes + (size_t)st * T.trees * tree_codes);
      const int per_tree = tree_codes / 8, total = per_tree * T.trees;
      for (int q = tid; q < total; q += nt) {
        const int t = q / per_tree, o = q - t * per_tree;
        *reinterpret_cast<uint2*>(s_codes + t * sstride + 8 * o) = __ldg(src + q);
      }
    };
    if (STAGED) stage_codes(0);

    if (tid < 64) {
      float r = 0.f, c = 0.f, s = 0.f;
      int qs = 0, qc = 0;
      if (tid < P && tid < 63) {
        float u0, u1, u2;
        if (W.randoms) {
          const float* rr = W.randoms + ((size_t)slot * 63 + tid) * 3;
          u0 = rr[0]; u1 = rr[1]; u2 = rr[2];
        } else {
          const uint64_t key = W.rng_seed * 0xD1342543DE82EF95ull + ((uint64_t)slot + W.slot_base) * 64 + tid;
          u0 = mix64(key * 3 + 0) * (1.0f / 16777216.0f);
          u1 = mix64(key * 3 + 1) * (1.0f / 16777216.0f);
          u2 = mix64(key * 3 + 2) * (1.0f / 16777216.0f);
        }
        const float t1 = __fmul_rn(seed.scale, 0.15f);
        r = __fadd_rn((float)seed.row, __fmul_rn(t1, __fsub_rn(0.5f, u0)));   // core/puploc.go:248
        c = __fadd_rn((float)seed.col, __fmul_rn(t1, __fsub_rn(0.5f, u1)));   // :249
        s = __fmul_rn(seed.scale, __fadd_rn(0.925f, __fmul_rn(0.15f, u2)));   // :250
        if (rot) {
          qs = (int)__fmul_rn(s, c_qsinf[rot_slot]);     // int(qsin), :166,:188 (from the INITIAL s)
          qc = (int)__fmul_rn(s, c_qcosf[rot_slot]);
        }
      }
      s_r[tid] = r; s_c[tid] = c; s_s[tid] = s; s_qs[tid] = qs; s_qc[tid] = qc;
      s_ir[tid] = clamp_coord(r); s_ic[tid] = clamp_coord(c); s_rs[tid] = (int)llround((double)s);   // int(r), int(math.Round(float64(s)))
      if (PATCH && tid < P) box_add(s_box, s_ir[tid], s_ic[tid], s_rs[tid], rot, qs, qc);
    }
    __syncthreads();
    // PATCH: geometry of the staged sample area of the coming stage (CTA-uniform), see load_patch
    int p_r0 = 0, p_c0 = 0, p_pitch = 0;
    bool p_use = false;
    auto load_patch = [&]() {
      p_use = false;
      if (!PATCH || P == 0) return;
      const int r0 = min(max(s_box[0], 0), rlim), r1 = min(max(s_box[1], 0), rlim);
      const int c0 = min(max(s_box[2], 0), clim) & ~15, c1 = min(max(s_box[3], 0), clim);
      const long long rows = (long long)r1 - r0 + 1, pitch = ((long long)c1 - c0 + 16) & ~15ll;
      if (rows <= 0 || pitch <= 0 || rows * pitch > patch_cap || (dim() & 15) || (reinterpret_cast<uintptr_t>(pixels) & 15)) return;
      p_use = true; p_r0 = r0; p_c0 = c0; p_pitch = (int)pitch;
      const int vec_per_row = (int)(pitch >> 4), total = (int)rows * vec_per_row;
      for (int q = tid; q < total; q += nt) {
        const int y = q / vec_per_row, x = q - y * vec_per_row;
        if (c0 + 16 * x + 16 <= dim())     // (vectors past the end of the row are never sampled: columns are clamped to ncols-1 < the pitch)
          *reinterpret_cast<uint4*>(s_patch + (size_t)y * pitch + 16 * x) =
              __ldg(reinterpret_cast<const uint4*>(pixels + (size_t)(r0 + y) * dim() + c0 + 16 * x));
      }
    };
    load_patch();
    if (PATCH) {
      __syncthreads();
      if (tid == 0) { s_box[0] = INT_MAX; s_box[1] = INT_MIN; s_box[2] = INT_MAX; s_box[3] = INT_MIN; }   // refilled after the stage's sums
    }

    const int npairs = P * T.trees;
    for (int st = 0; st < T.stages; ++st) {
      if (W.stats && tid == 0) atomicAdd(W.stats + ((PATCH && p_use) ? 2 : 3), 1ull);   // option walk_stats: patch / global stages
      for (int p = tid; p < npairs; p += nt) {
        const int i = p / T.trees, t = p - i * T.trees;
        const int ir = s_ir[i], ic = s_ic[i], rs = s_rs[i];
        const size_t tg = (size_t)st * T.trees + t;
        const int* tc = STAGED ? reinterpret_cast<const int*>(s_codes + t * sstride) : reinterpret_cast<const int*>(T.codes + tg * tree_codes);
        const int2* tc2 = reinterpret_cast<const int2*>(tc);
        const float2* tp = reinterpret_cast<const float2*>(T.preds + tg * 2 * L);
        int idx = 0;
        int cw = STAGED ? tc[1] : __ldg(tc + 1);
        if (!rot) {
          for (int k = 0; k < T.depth; ++k) {
            // children of node idx are nodes 2idx+1, 2idx+2 = words 2idx+2, 2idx+3 of the padded tree: ONE aligned 64-bit
            // load, in flight together with this node's pixels
            int kl = 0, kr = 0;
            if (k + 1 < T.depth) { const int2 kk = STAGED ? tc2[idx + 1] : __ldg(tc2 + idx + 1); kl = kk.x; kr = kk.y; }
            const int k0 = (int8_t)(cw), k2 = (int8_t)(cw >> 16);
            const int k1 = flip ? neg_i8((int8_t)(cw >> 8)) : (int)(int8_t)(cw >> 8);
            const int k3 = flip ? neg_i8(cw >> 24) : (cw >> 24);
            const int r1 = __vimin_s32_relu(ir + ((k0 * rs) >> 8), rlim), r2 = __vimin_s32_relu(ir + ((k2 * rs) >> 8), rlim);   // :118-119
            const int c1 = __vimin_s32_relu(ic + ((k1 * rs) >> 8), clim), c2 = __vimin_s32_relu(ic + ((k3 * rs) >> 8), clim);   // :124/:127
            const unsigned q1 = (PATCH && p_use) ? s_patch[(r1 - p_r0) * p_pitch + (c1 - p_c0)] : __ldg(pixels + (size_t)r1 * dim() + c1);
            const unsigned q2 = (PATCH && p_use) ? s_patch[(r2 - p_r0) * p_pitch + (c2 - p_c0)] : __ldg(pixels + (size_t)r2 * dim() + c2);
            const int bit = q1 > q2 ? 1 : 0;                                                                                     // :130-136
            cw = bit ? kr : kl;
            idx = 2 * idx + 1 + bit;
          }
        } else {
          const long long iqs = s_qs[i], iqc = s_qc[i];        // 64-bit products: int(256*s)*code leaves 32 bits for s > 2^15
          for (int k = 0; k < T.depth; ++k) {
            int kl = 0, kr = 0;
            if (k + 1 < T.depth) { const int2 kk = STAGED ? tc2[idx + 1] : __ldg(tc2 + idx + 1); kl = kk.x; kr = kk.y; }
            const int k0 = (int8_t)(cw), k2 = (int8_t)(cw >> 16);
            const int k1 = flip ? neg_i8((int8_t)(cw >> 8)) : (int)(int8_t)(cw >> 8);
            const int k3 = flip ? neg_i8(cw >> 24) : (cw >> 24);
            const int r1 = __vimin_s32_relu(ir + (int)((iqc * k0 - iqs * k1) >> 16), rlim);   // :188
            const int c1 = __vimin_s32_relu(ic + (int)((iqs * k0 + iqc * k1) >> 16), clim);   // :189
            const int r2 = __vimin_s32_relu(ir + (int)((iqc * k2 - iqs * k3) >> 16), rlim);   // :190
            const int c2 = __vimin_s32_relu(ic + (int)((iqs * k2 + iqc * k3) >> 16), clim);   // :191
            const unsigned q1 = (PATCH && p_use) ? s_patch[(r1 - p_r0) * p_pitch + (c1 - p_c0)] : __ldg(pixels + (size_t)r1 * dim() + c1);
            const unsigned q2 = (PATCH && p_use) ? s_patch[(r2 - p_r0) * p_pitch + (c2 - p_c0)] : __ldg(pixels + (size_t)r2 * dim() + c2);
            const int bit = q1 <= q2 ? 1 : 0;                                                                                    // :193-199
            cw = bit ? kr : kl;
            idx = 2 * idx + 1 + bit;
          }
        }
        s_leaf[p] = __ldg(tp + (idx - (L - 1)));
      }
      __syncthreads();
      if (STAGED && st + 1 < T.stages) stage_codes(st + 1);   // the sums below only read s_leaf
      if (tid < P) {
        float dr = 0.f, dc = 0.f;
        const float2* lf = s_leaf + tid * T.trees;
        for (int t = 0; t < T.trees; ++t) {                  // the reference's tree-ordered float32 sums, :140-145
          dr = __fadd_rn(dr, lf[t].x);
          dc = __fadd_rn(dc, flip ? -lf[t].y : lf[t].y);
        }
        const float s = s_s[tid];
        const float r = __fadd_rn(s_r[tid], __fmul_rn(dr, s));   // :149
        const float c = __fadd_rn(s_c[tid], __fmul_rn(dc, s));   // :150
        const float s2 = __fmul_rn(s, T.scales);                 // :151
        s_r[tid] = r; s_c[tid] = c; s_s[tid] = s2;
        s_ir[tid] = clamp_coord(r); s_ic[tid] = clamp_coord(c); s_rs[tid] = (int)llround((double)s2);
        if (PATCH) box_add(s_box, s_ir[tid], s_ic[tid], s_rs[tid], rot, s_qs[tid], s_qc[tid]);
      }
      __syncthreads();
      if (PATCH && st + 1 < T.stages) {
        load_patch();
        __syncthreads();
        if (tid == 0) { s_box[0] = INT_MAX; s_box[1] = INT_MIN; s_box[2] = INT_MAX; s_box[3] = INT_MIN; }
      }
    }
    // pool slots >= Perturbs stay 0 (fresh pool object, :228-236); all 63 slots are sorted (:267-269) by their rank_key,
    // which take the place of the integer coordinates (no longer read)
    unsigned* k_r = reinterpret_cast<unsigned*>(s_ir);
    unsigned* k_c = reinterpret_cast<unsigned*>(s_ic);
    unsigned* k_s = reinterpret_cast<unsigned*>(s_rs);
    if (tid < 63) { k_r[tid] = rank_key(s_r[tid]); k_c[tid] = rank_key(s_c[tid]); k_s[tid] = rank_key(s_s[tid]); }
    __syncthreads();
    if (tid < 63) {
      const int mid = (int)llround((double)P / 2);   // int(math.Round(float64(Perturbs)/2)), :273
      const unsigned vr = k_r[tid], vc = k_c[tid], vs = k_s[tid];
      int kr = 0, kc = 0, ks = 0;
      for (int q = 0; q < 63; ++q) {
        kr += (k_r[q] < vr || (k_r[q] == vr && q < tid)) ? 1 : 0;
        kc += (k_c[q] < vc || (k_c[q] == vc && q < tid)) ? 1 : 0;
        ks += (k_s[q] < vs || (k_s[q] == vs && q < tid)) ? 1 : 0;
      }
      if (kr == mid) W.out[slot].row = (int)s_r[tid];      // int() truncation, :273
      if (kc == mid) W.out[slot].col = (int)s_c[tid];
      if (ks == mid) W.out[slot].scale = s_s[tid];
      if (tid == 0) W.out[slot].perturbs = 0;        // the returned Puploc leaves Perturbs unset (:272-276)
    }
  }
}

template <bool IMG>
static void set_pair_smem(int bytes) {
  raise_dyn_smem((const void*)puploc_pair_kernel<true, true, IMG>, bytes);
  raise_dyn_smem((const void*)puploc_pair_kernel<true, false, IMG>, bytes);
  raise_dyn_smem((const void*)puploc_pair_kernel<false, false, IMG>, bytes);
}
// codes_bytes > 0: the stage's node codes are staged; patch_cap > 0 (with them): so is the stage's pixel patch
template <bool IMG>
static void launch_pair_variant(const PupWork& W, unsigned int* counter, int grid, size_t smem, int leaf, int codes_bytes, int patch_cap,
                                cudaStream_t st) {
  if (patch_cap > 0) puploc_pair_kernel<true, true, IMG><<<grid, kPairThreads, smem, st>>>(W, counter, leaf, codes_bytes, patch_cap);
  else if (codes_bytes > 0) puploc_pair_kernel<true, false, IMG><<<grid, kPairThreads, smem, st>>>(W, counter, leaf, codes_bytes, 0);
  else puploc_pair_kernel<false, false, IMG><<<grid, kPairThreads, smem, st>>>(W, counter, leaf, 0, 0);
}

int launch_puploc_pairs(const PupWork& W, unsigned int* counter, int num_sms, cudaStream_t st) {
  // shared memory is sized by the cascades THIS launch uses (positions first .. first+span-1), not by every table of the work list
  int trees_max = 0;
  size_t codes_max = 0;
  for (int j = 0; j < W.span && j < 32; ++j) {
    const PuplocTables& T = W.tab[W.tab_of[j]];
    trees_max = max(trees_max, T.trees);
    codes_max = std::max(codes_max, (size_t)T.trees * (4 * (size_t)T.leaves + 8));
  }
  const size_t leaf = ((size_t)63 * trees_max * sizeof(float2) + 15) & ~(size_t)15;
  if (leaf > 100 * 1024) return -1;                                   // caller falls back to the warp-per-perturbation kernel
  const size_t kBudget = 110 * 1024;                                  // two CTAs per SM at least
  codes_max = (codes_max + 15) & ~(size_t)15;
  const bool staged = g_opt.puploc_stage.load() != 0 && leaf + codes_max <= kBudget;
  size_t patch_cap = 0;
  if (staged && g_opt.puploc_stage.load() >= 2 && leaf + codes_max + 4096 <= kBudget) patch_cap = std::min<size_t>(48 * 1024, kBudget - leaf - codes_max);
  const size_t smem = leaf + (staged ? codes_max : 0) + patch_cap;
  static bool attr_set[kMaxDevices] = {};
  int dev = 0; cudaGetDevice(&dev);
  if (!attr_set[dev]) {
    set_pair_smem<false>((int)kBudget);
    set_pair_smem<true>((int)kBudget);
    attr_set[dev] = true;
  }
  const int grid = max(1, min(W.nwork, num_sms * 3));
  if (W.images) launch_pair_variant<true>(W, counter, grid, smem, (int)leaf, staged ? (int)codes_max : 0, (int)patch_cap, st);
  else launch_pair_variant<false>(W, counter, grid, smem, (int)leaf, staged ? (int)codes_max : 0, (int)patch_cap, st);
  return 0;
}

// ---- seeds of the face -> pupils -> landmarks sequence (the CALLER's arithmetic in the reference) -----------------------
// Eye seeds, core/flploc_test.go:103-118 == cmd/pigo/main.go:416-449 (float32 products, int() truncation):
//   Row = face.Row - int(0.075*float32(Scale)); Col = face.Col -/+ int(0.175|0.185*float32(Scale)); Scale = float32(Scale)*0.25
// One thread per (frame, face slot k).  Face slot layout: [frame][face_cap][stride], stride = 2 + ncalls.
__global__ void __launch_bounds__(256) eye_seed_kernel(const pigo_det* __restrict__ clusters, const int32_t* __restrict__ ncl, int cl_cap,
                                                       int nframes, int face_cap, int stride, int min_face, int eye_perturbs,
                                                       pigo_det* __restrict__ faces, int32_t* __restrict__ nfaces, pigo_point* __restrict__ seeds) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nframes * face_cap) return;
  const int f = i / face_cap, k = i - f * face_cap;
  const int n = ncl[f];
  if (k == 0) nfaces[f] = n;                              // required count (may exceed face_cap: the caller retries)
  pigo_point* sd = seeds + (size_t)i * stride;
  const pigo_point off = {0, 0, 0.f, -1};
  for (int j = 0; j < stride; ++j) sd[j] = off;
  pigo_det d = {0, 0, 0, 0.f};
  if (k < n && k < cl_cap) {
    d = clusters[(size_t)f * cl_cap + k];
    if (d.scale > min_face) {                             // core/flploc_test.go:102, cmd/pigo/main.go:404
      const float fs = (float)d.scale;
      const int row = d.row - (int)__fmul_rn(0.075f, fs);
      sd[0] = pigo_point{row, d.col - (int)__fmul_rn(0.175f, fs), __fmul_rn(fs, 0.25f), eye_perturbs};
      sd[1] = pigo_point{row, d.col + (int)__fmul_rn(0.185f, fs), __fmul_rn(fs, 0.25f), eye_perturbs};
    }
  }
  faces[i] = d;
}

// Landmark seeds, GetLandmarkPoint core/flploc.go:37-50 (float64): one thread per (face slot, call).
__global__ void __launch_bounds__(256) landmark_seed_kernel(const pigo_point* __restrict__ points, pigo_point* __restrict__ seeds, int nslots,
                                                            int stride, int ncalls, int flp_perturbs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nslots * ncalls) return;
  const int fs = i / ncalls, cidx = i - fs * ncalls;
  const size_t base = (size_t)fs * stride;
  if (seeds[base].perturbs < 0) return;                   // face without eye seeds
  const pigo_point le = points[base], re = points[base + 1];
  const long long dx = (long long)(le.row - re.row) * (le.row - re.row);
  const long long dy = (long long)(le.col - re.col) * (le.col - re.col);
  const double dist = __dsqrt_rn((double)(dx + dy));
  const double row = __dadd_rn((double)(le.row + re.row) / 2.0, __dmul_rn(0.25, dist));
  const double col = __dadd_rn((double)(le.col + re.col) / 2.0, __dmul_rn(0.15, dist));
  seeds[base + 2 + cidx] = pigo_point{(int)row, (int)col, (float)__dmul_rn(3.0, dist), flp_perturbs};
}

void launch_eye_seeds(const pigo_det* clusters, const int32_t* ncl, int cl_cap, int nframes, int face_cap, int stride, int min_face,
                      int eye_perturbs, pigo_det* faces, int32_t* nfaces, pigo_point* seeds, cudaStream_t st) {
  const int n = nframes * face_cap;
  eye_seed_kernel<<<(n + 255) / 256, 256, 0, st>>>(clusters, ncl, cl_cap, nframes, face_cap, stride, min_face, eye_perturbs, faces, nfaces, seeds);
}
void launch_landmark_seeds(const pigo_point* points, pigo_point* seeds, int nslots, int stride, int ncalls, int flp_perturbs, cudaStream_t st) {
  const int n = nslots * ncalls;
  if (n <= 0) return;
  landmark_seed_kernel<<<(n + 255) / 256, 256, 0, st>>>(points, seeds, nslots, stride, ncalls, flp_perturbs);
}

void launch_puploc(const PuplocTables& T, const pigo_point* seeds, int nseeds, const float* randoms, uint64_t rng_seed,
                   const uint8_t* frames, const int32_t* seed_frame, size_t frame_stride, int rows, int cols, int dim, int rot_slot,
                   const uint8_t* flipv, pigo_point* out, const ImageDesc* images, cudaStream_t st) {
  if (images)
    puploc_kernel<true><<<nseeds, 1024, 0, st>>>(T, seeds, nseeds, randoms, rng_seed, frames, seed_frame, frame_stride, rows, cols, dim,
                                                 rot_slot, flipv, out, images);
  else
    puploc_kernel<false><<<nseeds, 1024, 0, st>>>(T, seeds, nseeds, randoms, rng_seed, frames, seed_frame, frame_stride, rows, cols, dim,
                                                  rot_slot, flipv, out, nullptr);
}

}  // namespace pigo
