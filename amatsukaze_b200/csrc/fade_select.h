// fade_select.h -- AMTEraseLogo::CalcFade2's record choice and decision (LogoScan.hpp:1263-1315), one definition for the
// host (amtk_calc_fade2*, logo_host.cpp) and the device (the erase stream's fade kernel, logo_kernels.cuh).
// Both compilers build it without fast-math or contraction (_build.py), so host and device give the same bits.
#pragma once

#ifdef __CUDACC__
#define AMTK_HD __host__ __device__ __forceinline__
#else
#define AMTK_HD inline
#endif

namespace amtk {

// Index of the analyze record CalcFade2 reads for offset i in [-4, 4] around frame n.
AMTK_HD int calc_fade2_index(int num_records, int num_frames, int n, int i) {
  const int nblk = (num_records + 7) / 8;
  int nsrc = n + i;
  nsrc = nsrc < num_frames - 1 ? nsrc : num_frames - 1;
  nsrc = nsrc > 0 ? nsrc : 0;
  const int r = nsrc + i;                               // sic: offset applied twice (:1273-1275)
  int blk = r >> 3;                                     // AviSynth clamps GetFrame to the clip
  blk = blk < nblk - 1 ? blk : nblk - 1;
  blk = blk > 0 ? blk : 0;
  int idx = blk * 8 + (r & 7);                          // AMTAnalyzeLogo clamps (:1133)
  idx = idx < num_records - 1 ? idx : num_records - 1;
  return idx > 0 ? idx : 0;
}

// First minimum of 11 values (std::min_element's choice).
AMTK_HD int calc_fade2_first_min(const float* v) {
  int best = 0;
  for (int j = 1; j < 11; ++j)
    if (v[j] < v[best]) best = j;
  return best;
}

// The decision itself on the nine records -- all CalcFade2 ever looks at.  rec(i) points at the 33 floats of offset
// i - 4 (i = 0 .. 8), wherever they are stored.
template <typename Rec>
AMTK_HD void calc_fade2_decide(const Rec& rec, float* fadeT, float* fadeB) {
  constexpr int kDist = 4;
  int best[2 * kDist + 1];
  for (int i = 0; i < 2 * kDist + 1; ++i) best[i] = calc_fade2_first_min(rec(i));
  const float* centre = rec(kDist);
  const int bestT = calc_fade2_first_min(centre + 11), bestB = calc_fade2_first_min(centre + 22);
  float before = 0, after = 0;
  for (int i = 1; i <= 4; ++i) { before += best[kDist - i]; after += best[kDist + i]; }
  before /= 4 * 10; after /= 4 * 10;
  if ((before < 0.3 && after > 0.7) || (before > 0.7 && after < 0.3)) {   // abrupt switch: per field
    *fadeT = bestT / 10.0f; *fadeB = bestB / 10.0f;
  } else {
    *fadeT = *fadeB = best[kDist] / 10.0f;
  }
}

struct Rec9 {                // nine records back to back (offset order)
  const float* p;
  AMTK_HD const float* operator()(int i) const { return p + i * 33; }
};

AMTK_HD void calc_fade2_records(const float* rec9, float* fadeT, float* fadeB) { calc_fade2_decide(Rec9{ rec9 }, fadeT, fadeB); }

}  // namespace amtk
