// comb_stream.cuh -- field-difference / combing metric, streaming pass, round-2 kernel ("warp-streams").
//
// Same integer spec and the same arithmetic as comb_kernels.cuh (bytes as exact fp16 subnormals, HFMA2 stencil,
// HSET2 thresholds, VABSDIFF4 + SWAR compare + IDP.4A for the inter-frame difference, pair-coded mask sums); what
// changed is the decomposition, chosen from the round-1 profile (issue/ALU-pipe bound at 0.195 warp-inst/B, 0.40
// barrier stalls per issue, 78 % issue-active):
//
//   * ONE WARP = one tile stream.  A warp owns a tile of 128 bytes x 4R rows (4 runs of R rows, 8 lanes per
//     row) and streams its frames through its own 2-slot TMA ring (current frame + the one in flight; the previous
//     frame's rows stay in registers).  There is no block barrier and no empty-barrier:
//     the only synchronisation is the warp's own wait on the "full" mbarrier of the next slot, and lane 0 refilling
//     the slot the warp has just finished with.  Eight such warps share an SM, phase-decorrelated, so the two
//     half-rate pipes (FMA-heavy: HFMA2/IDP/IMAD; ALU: HSET2/PRMT/LOP3/VABSDIFF4/IADD3) see a mixed instruction stream.
//   * 16-byte strips per lane-row (LDS.128): half the shared-memory loads, prologue and loop overhead per pixel.
//   * no per-row threshold loads on edge tiles: every tile runs the plain body; the few rows the spec excludes
//     (y < 2, y >= H-2, and the zero-filled rows just below the plane) are re-evaluated by the affected lanes after
//     the main pass and their hits subtracted (integer counters: exact).
//   * counters: per-lane pair-coded sums -> REDUX -> six global RED per warp and tile-frame (no shared-memory stage).
//   * the 64-byte remainder columns of the U and V planes (chroma width 960 = 7.5 tiles) share ONE tile through a 4-D
//     tensor map (x, plane, y, frame): its box arrives in shared memory with the ordinary 128-byte pitch, so there is a
//     single copy of the row code (instruction footprint matters: eight phase-decorrelated warps share a 32 KB L1.5 I$).
//   * four warp streams form a CTA only so that the hardware places one on each SM sub-partition; they never
//     synchronise with each other.
// 8-bit clips run the BAND form of the same kernel (WtCfg / WbCfg, ws_bands): the warps of a CTA share one ring whose slots
// hold a 512-byte-wide band of one frame, warp w taking bytes [128c, 128c + 128) (c = w % 4) of its row group's rows with
// the same row code.
// Per warp-stream tile, a frame's box is 64 separate 128-byte pieces of 64 rows; the DRAM pages they open serve one piece
// each, and that access pattern, not the arithmetic, set the pace on H100 (DESIGN.md 3.1a).  A band box reads 512
// contiguous bytes per row.
#pragma once
#include <cuda_fp16.h>
#include "amtk_internal.h"
#include "tma_utils.cuh"
#include "comb_kernels.cuh"      // bytes_ge, decode_pair, CombSegment
#include "logo_kernels.cuh"      // scan_item (logo items of the band form)

namespace amtk {

constexpr int kWsTW = 128;               // tile width in bytes
constexpr int kWsRuns = 4;               // runs per warp (8 lanes x 16 bytes per row)
constexpr int kWsWarps = 4;              // default warp streams per CTA: one per SM sub-partition

template <int R_, int STAGES_, int WARPS_ = kWsWarps, int BPS_ = 1>
struct WsCfg {
  static constexpr int R = R_, STAGES = STAGES_, WARPS = WARPS_;
  static constexpr int BPS = BPS_;                          // 1: 8-bit samples; 2: 16-bit containers holding <= 10 bits (YUV420P10)
  static constexpr int TH = kWsRuns * R;                    // output rows per tile
  static constexpr int BOXH = TH + 4;                       // + 2 halo rows above and below
  static constexpr int STAGE_BYTES = kWsTW * BOXH;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;   // one warp's ring
  static constexpr int SMEM = WARPS * RING_BYTES + 128;     // + alignment slack
  static constexpr int FIT = (227 * 1024) / (SMEM + 1024 + 8 * WARPS * STAGES + 8);    // CTAs that fit in shared memory
  static constexpr int MIN_CTAS = FIT >= 4 ? 4 : FIT >= 3 ? 3 : FIT >= 2 ? 2 : 1;      // resident CTAs the register budget is set for
  static constexpr bool BAND = false;
};

// Band form (8-bit samples): the warps of a CTA share one ring of slots, each slot a 512-byte-wide band of one frame.
// A band is GROUPS row groups of 4R rows; warp w takes column w % 4 and row group w / 4.
constexpr int kWbW = 512;                // band width in bytes: four warps x 128 bytes
constexpr int kWbHalf = 256;             // a band is loaded as two TMA boxes of this width (256 elements is the box limit)
template <int R_, int STAGES_, int GROUPS_>
struct BandCfg {
  static constexpr int R = R_, STAGES = STAGES_, GROUPS = GROUPS_, WARPS = GROUPS * (kWbW / kWsTW), BPS = 1;
  static constexpr int TH = GROUPS * kWsRuns * R;           // output rows per band
  static constexpr int BOXH = TH + 4;
  static_assert(BOXH <= 256, "a TMA box is at most 256 rows");
  static constexpr int HALF_BYTES = kWbHalf * BOXH;         // one TMA box
  static constexpr int STAGE_BYTES = 2 * HALF_BYTES;        // one slot: the band's box of one frame
  static constexpr int SMEM = STAGES * STAGE_BYTES + 128;
  static constexpr int FIT = (227 * 1024) / (SMEM + 1024 + 12 * STAGES + 16);
  static constexpr int MIN_CTAS = FIT >= 4 ? 4 : FIT >= 3 ? 3 : FIT >= 2 ? 2 : 1;
  static constexpr bool BAND = true;
};
// 512 x 4R bands: three 4-warp CTAs per SM (AMTK_COMB_WS_BAND=1)
template <int R_, int STAGES_> using WbCfg = BandCfg<R_, STAGES_, 1>;
// Tall bands, 512 x 12R (the 8-bit default): the same twelve warps per SM in one CTA.  The 4 halo rows are re-read once
// per 12R rows instead of once per 4R (1080 luma rows: 1100 read instead of 1148).
constexpr int kWtGroups = 3;
template <int R_, int STAGES_> using WtCfg = BandCfg<R_, STAGES_, kWtGroups>;

// A tile class: all tiles of one class have the same shape and are numbered consecutively from tile0.
//   kind 0: a 128-byte wide tile (band form: a 512-byte wide band) of one plane (3-D map: x, y, frame).
//   kind 1: the remainder columns (<= 64 bytes) of U and V side by side in one tile -- a 4-D map (x, plane, y, frame)
//           whose box (64, 2, BOXH, 1) lands in shared memory as rows of [U 64 bytes | V 64 bytes], i.e. with the same
//           128-byte pitch as an ordinary tile, so the same code runs on it.
struct WsClass {
  int tile0, ntiles;
  int kind;
  int tilesX;                 // tiles per tile-row
  int map;                    // kind 0: index into WsArgs::map
  int x0;                     // kind 1: first sample of the remainder column
  int W;                      // plane width in bytes (band form: which columns hold samples)
  int H;                      // plane height in rows
  int cls;                    // 0 = Y, 1 = C (counts[] half)
  unsigned thM, thS, thL;     // encoded thresholds (see CombPlane)
};
constexpr int kWsMaxClasses = 4;
struct WsArgs {
  CUtensorMap map[3];         // 128-byte boxes of Y, U, V
  CUtensorMap map_uv;         // 4-D: the U|V remainder pair
  WsClass cl[kWsMaxClasses];
  int nclasses;
  const CombSegment* segs;    // work items (tile, frame range), in queue order; band form: tile < 0 = logo item (frame range)
  int nitems;
  int* queue;                 // global item counter (zeroed by the host before the launch)
  int* counts;                // [nframes_out][12]
  int out_frame0;
  int prefetch;               // > 0: tile loads are announced to L2 (cp.async.bulk.prefetch.tensor) this many steps before their slot frees
  ScanItemJob logo;           // band form: what the logo items evaluate (only read when the queue has some)
};

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

__device__ __forceinline__ void tma_prefetch_3d(const CUtensorMap* map, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];" ::"l"(map), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* map, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];" ::"l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

#ifndef AMTK_WS_RELOAD_PREV
#define AMTK_WS_RELOAD_PREV 1
#endif
constexpr bool kWsReloadPrev = AMTK_WS_RELOAD_PREV != 0;
#ifndef AMTK_WS_L_VIA_IDP
#define AMTK_WS_L_VIA_IDP 0
#endif
constexpr bool kWsLviaIdp = AMTK_WS_L_VIA_IDP != 0;        // large-threshold counter: 510 per hit instead of pair-coded
// an LDS.128 the compiler cannot merge with an earlier C++ load of the same address
__device__ __forceinline__ uint4 lds128(const uint8_t* p) {
  uint4 v;
  asm("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(smem_u32(p)));
  return v;
}

struct H8 { __half2 v[8]; };   // 16 pixels of one row as fp16x2

__device__ __forceinline__ H8 bytes16_to_half(const uint4 raw) {
  H8 r;
  const uint32_t w[4] = { raw.x, raw.y, raw.z, raw.w };
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t a = __byte_perm(w[i], 0, 0x4140), b = __byte_perm(w[i], 0, 0x4342);   // zero-extended bytes = exact fp16 subnormals
    r.v[2 * i] = *reinterpret_cast<__half2*>(&a); r.v[2 * i + 1] = *reinterpret_cast<__half2*>(&b);
  }
  return r;
}

struct WsCounts { uint32_t S[2], L[2], M[2]; };   // slot = row parity relative to the lane's first row; S/L pair-coded, M 128 per hit

// comb response masks of one 16-pixel row: acc -= mask (pair-coded)
__device__ __forceinline__ void ws_row_masks(const H8& h0, const H8& h1, const H8& h2, const H8& h3, const H8& h4,
                                             const __half2 thS, const __half2 thL, uint32_t& accS, uint32_t& accL) {
  const __half2 k4 = __float2half2_rn(4.0f), km3 = __float2half2_rn(-3.0f);
  uint32_t mS[8], mL[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    __half2 t = __hadd2(h0.v[q], h4.v[q]);
    t = __hfma2(k4, h2.v[q], t);
    const __half2 u = __hadd2(h1.v[q], h3.v[q]);
    const __half2 r = __habs2(__hfma2(km3, u, t));
    mS[q] = __hge2_mask(r, thS);
    mL[q] = __hge2_mask(r, thL);
  }
  // 8 masks + accumulator = 9 operands = four 3-input adds (ALU pipe) ...
  accS = accS - (mS[0] + mS[1]) - (mS[2] + mS[3] + mS[4]) - (mS[5] + mS[6] + mS[7]);
  if (kWsLviaIdp) {
    // ... or, for the large-threshold masks, eight IDP.4A on the FMA-heavy pipe, which has the slack: the loop is
    // ALU-pipe bound (HSET2/PRMT/LOP3/IADD3/VABSDIFF4 = 49 of 92 instructions per 16-pixel row).  A 0xFFFF lane is two
    // 0xFF bytes, so the byte sum grows by 510 per hit.
#pragma unroll
    for (int q = 0; q < 8; ++q) accL = __dp4a(mL[q], 0x01010101u, accL);
  } else {
    accL = accL - (mL[0] + mL[1]) - (mL[2] + mL[3] + mL[4]) - (mL[5] + mL[6] + mL[7]);
  }
}

// Main body: R rows of one lane's 16-byte strip.  cur points at smem row (run*R) of the box = global row y_first-2.
// P[j] holds the previous frame's bytes of output row j (kept in REGISTERS from the step before: the centre row of step
// k is exactly the "previous" row of step k+1, so the inter-frame difference costs neither a second shared-memory slot
// nor a second LDS); on return P holds this frame's rows.
// Per 16-pixel row: 32 HFMA2/HADD2 + 4 IDP + 4 IMAD.IADD on the FMA-heavy pipe; 16 HSET2 + 8 PRMT + 8 LOP3 + 8 IADD3 +
// 4 VABSDIFF4 on the ALU pipe; 2 LDS.128.  (ptxas reschedules the unrolled body on its own: three different source
// orders of this loop gave the identical SASS schedule.)
template <int R, int PITCH>
__device__ __forceinline__ WsCounts ws_rows(const uint8_t* __restrict__ cur, uint4 (&P)[R],
                                            const uint32_t kM, const uint32_t thS_bits, const uint32_t thL_bits) {
  const __half2 thS = *reinterpret_cast<const __half2*>(&thS_bits);
  const __half2 thL = *reinterpret_cast<const __half2*>(&thL_bits);
  WsCounts c = { { 0u, 0u }, { 0u, 0u }, { 0u, 0u } };
  H8 h0 = bytes16_to_half(*reinterpret_cast<const uint4*>(cur));
  H8 h1 = bytes16_to_half(*reinterpret_cast<const uint4*>(cur + PITCH));
  uint4 raw_c = *reinterpret_cast<const uint4*>(cur + 2 * PITCH);
  uint4 raw_n = *reinterpret_cast<const uint4*>(cur + 3 * PITCH);
  H8 h2 = bytes16_to_half(raw_c);
  H8 h3 = bytes16_to_half(raw_n);
#pragma unroll
  for (int j = 0; j < R; ++j) {
    const uint4 raw_nn = *reinterpret_cast<const uint4*>(cur + (j + 4) * PITCH);
    const uint4 pv = P[j];
    const int f = j & 1;
    const H8 h4 = bytes16_to_half(raw_nn);
    // inter-frame difference of the centre row: VABSDIFF4 + SWAR compare (ALU pipe), IDP.4A count (FMA pipe)
    c.M[f] = __dp4a(bytes_ge(__vabsdiffu4(raw_c.x, pv.x), kM), 0x01010101u, c.M[f]);
    c.M[f] = __dp4a(bytes_ge(__vabsdiffu4(raw_c.y, pv.y), kM), 0x01010101u, c.M[f]);
    c.M[f] = __dp4a(bytes_ge(__vabsdiffu4(raw_c.z, pv.z), kM), 0x01010101u, c.M[f]);
    c.M[f] = __dp4a(bytes_ge(__vabsdiffu4(raw_c.w, pv.w), kM), 0x01010101u, c.M[f]);
    // P[j] <- this frame's centre row.  Its bytes are in raw_c already, but raw_c's registers were allocated while the old
    // P[j] was still live, so "P[j] = raw_c" costs four register moves per row; loading the row a second time straight
    // into P[j]'s registers is one LDS.128 on the otherwise idle LSU pipe.
    if (kWsReloadPrev) P[j] = lds128(cur + (j + 2) * PITCH); else P[j] = raw_c;
    ws_row_masks(h0, h1, h2, h3, h4, thS, thL, c.S[f], c.L[f]);
    h0 = h1; h1 = h2; h2 = h3; h3 = h4; raw_c = raw_n; raw_n = raw_nn;
  }
  return c;
}


// Software-pipelined form of ws_rows: the thresholds / mask sums of row j-1 (ALU pipe) are written next to the stencil
// of row j (FMA-heavy pipe), per register pair, so that independent work for both half-rate pipes is adjacent in the
// instruction stream.  Same results (integer counters).
__device__ __forceinline__ void ws_masks_q(const __half2 r, const __half2 thS, const __half2 thL, uint32_t& mS, uint32_t& mL) {
  mS = __hge2_mask(__habs2(r), thS);
  mL = __hge2_mask(__habs2(r), thL);
}
template <int R, int PITCH>
__device__ __forceinline__ WsCounts ws_rows_sp(const uint8_t* __restrict__ cur, uint4 (&P)[R],
                                               const uint32_t kM, const uint32_t thS_bits, const uint32_t thL_bits) {
  const __half2 thS = *reinterpret_cast<const __half2*>(&thS_bits);
  const __half2 thL = *reinterpret_cast<const __half2*>(&thL_bits);
  const __half2 k4 = __float2half2_rn(4.0f), km3 = __float2half2_rn(-3.0f);
  WsCounts c = { { 0u, 0u }, { 0u, 0u }, { 0u, 0u } };
  H8 h0 = bytes16_to_half(*reinterpret_cast<const uint4*>(cur));
  H8 h1 = bytes16_to_half(*reinterpret_cast<const uint4*>(cur + PITCH));
  uint4 raw_c = *reinterpret_cast<const uint4*>(cur + 2 * PITCH);
  uint4 raw_n = *reinterpret_cast<const uint4*>(cur + 3 * PITCH);
  H8 h2 = bytes16_to_half(raw_c);
  H8 h3 = bytes16_to_half(raw_n);
  __half2 rp[8];                                              // responses of the previous row, not yet thresholded
#pragma unroll
  for (int j = 0; j <= R; ++j) {
    uint4 raw_nn = make_uint4(0u, 0u, 0u, 0u);
    H8 h4;
    if (j < R) {
      raw_nn = *reinterpret_cast<const uint4*>(cur + (j + 4) * PITCH);
      const uint4 pv = P[j];
      const int f = j & 1;
      h4 = bytes16_to_half(raw_nn);
      c.M[f] = __dp4a(bytes_ge(__vabsdiffu4(raw_c.x, pv.x), kM), 0x01010101u, c.M[f]);
      c.M[f] = __dp4a(bytes_ge(__vabsdiffu4(raw_c.y, pv.y), kM), 0x01010101u, c.M[f]);
      c.M[f] = __dp4a(bytes_ge(__vabsdiffu4(raw_c.z, pv.z), kM), 0x01010101u, c.M[f]);
      c.M[f] = __dp4a(bytes_ge(__vabsdiffu4(raw_c.w, pv.w), kM), 0x01010101u, c.M[f]);
      if (kWsReloadPrev) P[j] = lds128(cur + (j + 2) * PITCH); else P[j] = raw_c;
    }
    uint32_t mS[8], mL[8];
    __half2 rn[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      if (j < R) {
        __half2 t = __hadd2(h0.v[q], h4.v[q]);
        t = __hfma2(k4, h2.v[q], t);
        const __half2 u = __hadd2(h1.v[q], h3.v[q]);
        rn[q] = __hfma2(km3, u, t);
      }
      if (j > 0) ws_masks_q(rp[q], thS, thL, mS[q], mL[q]);
    }
    if (j > 0) {
      const int fp = (j - 1) & 1;
      c.S[fp] = c.S[fp] - (mS[0] + mS[1]) - (mS[2] + mS[3] + mS[4]) - (mS[5] + mS[6] + mS[7]);
      c.L[fp] = c.L[fp] - (mL[0] + mL[1]) - (mL[2] + mL[3] + mL[4]) - (mL[5] + mL[6] + mL[7]);
    }
    if (j < R) {
#pragma unroll
      for (int q = 0; q < 8; ++q) rp[q] = rn[q];
      h0 = h1; h1 = h2; h2 = h3; h3 = h4; raw_c = raw_n; raw_n = raw_nn;
    }
  }
  return c;
}

#ifndef AMTK_WS_SP
#define AMTK_WS_SP 0
#endif
// ---- YUV420P10 (16-bit containers, samples < 1024) --------------------------------------------------------------------
// A 10-bit sample in a 16-bit lane IS an exact fp16 bit pattern (k * 2^-24, k < 2048): no conversion at all.  The response
// needs 13 bits, so the stencil runs as 32-bit integer ops on the two 16-bit lanes at once (no lane ever leaves [0, 65535]:
// r' = r + 8192), |r| comes from one packed max (VIMNMX.U16x2 of r' and 16384 - r'), and the thresholds are HSET2 on the
// bit patterns (positive fp16 patterns below 0x7C00 order like integers).  The inter-frame difference is HADD2 + HSET2 |d|
// (|d| < 1024: exact).  16-byte strips = 8 pixels per lane-row; ~42 instructions per 8 pixels = 2.6 per BYTE (8-bit: 5.75).
struct W4 { uint32_t v[4]; };
__device__ __forceinline__ W4 w4(const uint4 r) { W4 x; x.v[0] = r.x; x.v[1] = r.y; x.v[2] = r.z; x.v[3] = r.w; return x; }
constexpr uint32_t kWs10Bias = 8192u * 0x00010001u;

__device__ __forceinline__ void ws_row_masks10(const W4& h0, const W4& h1, const W4& h2, const W4& h3, const W4& h4,
                                               const __half2 thS, const __half2 thL, uint32_t& accS, uint32_t& accL) {
  uint32_t mS[4], mL[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint32_t t = h2.v[q] * 4u + h0.v[q];
    t = t + h4.v[q] + kWs10Bias;
    const uint32_t u = h1.v[q] + h3.v[q];
    const uint32_t rp = t - 3u * u;                        // r + 8192 in both lanes
    const uint32_t m = __vmaxu2(rp, 2u * kWs10Bias - rp);  // 8192 + |r|
    const __half2 mh = *reinterpret_cast<const __half2*>(&m);
    mS[q] = __hge2_mask(mh, thS);
    mL[q] = __hge2_mask(mh, thL);
  }
  accS = accS - (mS[0] + mS[1]) - (mS[2] + mS[3]);
  accL = accL - (mL[0] + mL[1]) - (mL[2] + mL[3]);
}

template <int R, int PITCH>
__device__ __forceinline__ WsCounts ws_rows10(const uint8_t* __restrict__ cur, uint4 (&P)[R],
                                              const uint32_t kM, const uint32_t thS_bits, const uint32_t thL_bits) {
  const __half2 thS = *reinterpret_cast<const __half2*>(&thS_bits);
  const __half2 thL = *reinterpret_cast<const __half2*>(&thL_bits);
  const __half2 thM = *reinterpret_cast<const __half2*>(&kM);
  WsCounts c = { { 0u, 0u }, { 0u, 0u }, { 0u, 0u } };
  W4 h0 = w4(*reinterpret_cast<const uint4*>(cur));
  W4 h1 = w4(*reinterpret_cast<const uint4*>(cur + PITCH));
  W4 h2 = w4(*reinterpret_cast<const uint4*>(cur + 2 * PITCH));
  W4 h3 = w4(*reinterpret_cast<const uint4*>(cur + 3 * PITCH));
#pragma unroll
  for (int j = 0; j < R; ++j) {
    const W4 h4 = w4(*reinterpret_cast<const uint4*>(cur + (j + 4) * PITCH));
    const W4 pv = w4(P[j]);
    const int f = j & 1;
    uint32_t mM[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
      mM[q] = __hge2_mask(__habs2(__hsub2(*reinterpret_cast<const __half2*>(&h2.v[q]), *reinterpret_cast<const __half2*>(&pv.v[q]))), thM);
    c.M[f] = c.M[f] - (mM[0] + mM[1]) - (mM[2] + mM[3]);
    if (kWsReloadPrev) P[j] = lds128(cur + (j + 2) * PITCH); else P[j] = make_uint4(h2.v[0], h2.v[1], h2.v[2], h2.v[3]);
    ws_row_masks10(h0, h1, h2, h3, h4, thS, thL, c.S[f], c.L[f]);
    h0 = h1; h1 = h2; h2 = h3; h3 = h4;
  }
  return c;
}

template <int PITCH>
__device__ __noinline__ void ws_fixup10(const uint8_t* cur, uint32_t rows, uint32_t mine, uint32_t thS_bits, uint32_t thL_bits, WsCounts& c) {
  const __half2 thS = *reinterpret_cast<const __half2*>(&thS_bits);
  const __half2 thL = *reinterpret_cast<const __half2*>(&thL_bits);
  for (uint32_t m = rows; m; m &= m - 1) {
    const int j = __ffs(m) - 1;
    if (!((mine >> j) & 1u)) continue;
    const uint8_t* p = cur + j * PITCH;
    uint32_t dS = 0u, dL = 0u;
    ws_row_masks10(w4(*reinterpret_cast<const uint4*>(p)), w4(*reinterpret_cast<const uint4*>(p + PITCH)), w4(*reinterpret_cast<const uint4*>(p + 2 * PITCH)),
                   w4(*reinterpret_cast<const uint4*>(p + 3 * PITCH)), w4(*reinterpret_cast<const uint4*>(p + 4 * PITCH)), thS, thL, dS, dL);
    c.S[j & 1] -= dS; c.L[j & 1] -= dL;
  }
}

// Rows the spec excludes from the comb response but the plain body counted: y < 2, H-2 <= y < H (no full window) and
// the phantom rows H, H+1 (zero-filled by TMA; their windows still see the last two real rows).  The affected lanes
// re-evaluate exactly those rows and ADD the masks back (the body subtracted them).  Rare: edge tiles only, and then
// 2 to 4 rows; `rows` is the warp-wide union of row indices, `mine` this lane's own set.
template <int PITCH>
__device__ __noinline__ void ws_fixup(const uint8_t* cur, uint32_t rows, uint32_t mine, uint32_t thS_bits, uint32_t thL_bits, WsCounts& c) {
  const __half2 thS = *reinterpret_cast<const __half2*>(&thS_bits);
  const __half2 thL = *reinterpret_cast<const __half2*>(&thL_bits);
  for (uint32_t m = rows; m; m &= m - 1) {
    const int j = __ffs(m) - 1;
    if (!((mine >> j) & 1u)) continue;
    const uint8_t* p = cur + j * PITCH;
    const H8 h0 = bytes16_to_half(*reinterpret_cast<const uint4*>(p));
    const H8 h1 = bytes16_to_half(*reinterpret_cast<const uint4*>(p + PITCH));
    const H8 h2 = bytes16_to_half(*reinterpret_cast<const uint4*>(p + 2 * PITCH));
    const H8 h3 = bytes16_to_half(*reinterpret_cast<const uint4*>(p + 3 * PITCH));
    const H8 h4 = bytes16_to_half(*reinterpret_cast<const uint4*>(p + 4 * PITCH));
    uint32_t dS = 0u, dL = 0u;
    ws_row_masks(h0, h1, h2, h3, h4, thS, thL, dS, dL);      // what the body added for this row (mod 2^32)
    c.S[j & 1] -= dS; c.L[j & 1] -= dL;
  }
}

// Per-warp rings: every warp streams its own 128-byte tile (WsCfg).
template <typename Cfg>
__device__ __forceinline__ void ws_warp_streams(const WsArgs& a) {
  constexpr int S = Cfg::STAGES, R = Cfg::R;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bars[Cfg::WARPS][S];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* tiles = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u) + warp * Cfg::RING_BYTES;   // this warp's ring
  uint64_t* full_bar = full_bars[warp];
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < S; ++s) mbar_init(&full_bar[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  // warp streams are independent from here on: no block-level synchronisation, work comes from a global queue of
  // (tile, frame range) items (long items first, short ones last, so the warps finish within a short item of each other)
  uint32_t gload = 0;      // loads consumed so far by this warp (ring position of L_0 of the current item)
  const int strip = lane & 7, run = lane >> 3;
  const int lane_off = (run * R) * kWsTW + strip * 16;       // lane's byte offset inside a slot
  for (;;) {
    int item = 0;
    if (lane == 0) item = atomicAdd(a.queue, 1);
    item = __shfl_sync(0xFFFFFFFFu, item, 0);
    if (item >= a.nitems) break;
    const CombSegment seg = a.segs[item];
    int ci = 0;
#pragma unroll
    for (int k = 1; k < kWsMaxClasses; ++k) if (k < a.nclasses && seg.tile >= a.cl[k].tile0) ci = k;
    const WsClass& C = a.cl[ci];
    const int lt = seg.tile - C.tile0;
    const int ty = lt / C.tilesX, tx = lt - ty * C.tilesX;
    const int y0 = ty * Cfg::TH;
    const int y_first = y0 + run * R;
    const int nf = seg.fend - seg.fbegin;
    const int nloads = nf + 1;                               // L_0 = previous frame, L_k = frame fbegin+k-1
    const int fprev = seg.fbegin > 0 ? seg.fbegin - 1 : seg.fbegin;

    auto issue_at = [&](int j, int st) {                     // lane 0 only; st = (gload + j) % S
      const int fr = (j == 0) ? fprev : seg.fbegin + j - 1;
      mbar_expect_tx(&full_bar[st], Cfg::STAGE_BYTES);
      uint8_t* dst = tiles + st * Cfg::STAGE_BYTES;
      if (C.kind == 0) tma_load_3d(dst, &a.map[C.map], &full_bar[st], tx * kWsTW, y0 - 2, fr);
      else tma_load_4d(dst, &a.map_uv, &full_bar[st], C.x0, 0, y0 - 2, fr);
    };
    auto prefetch_at = [&](int j) {                          // lane 0 only: pull load j (a frame of this tile) into L2
      const int fr = seg.fbegin + j - 1;                     // j >= S >= 1
      if (C.kind == 0) tma_prefetch_3d(&a.map[C.map], tx * kWsTW, y0 - 2, fr);
      else tma_prefetch_4d(&a.map_uv, C.x0, 0, y0 - 2, fr);
    };
    const int pf = a.prefetch;
    if (lane == 0) {
      const int pro = nloads < S ? nloads : S;
      for (int j = 0; j < pro; ++j) issue_at(j, (int)((gload + (uint32_t)j) % S));
      for (int j = S; j < S + pf && j < nloads; ++j) prefetch_at(j);
    }
    // rows of this lane's run the spec excludes (bit j = row y_first + j)
    uint32_t fix_mine = 0u;
    if (y_first < 2) fix_mine |= (1u << (2 - y_first)) - 1u;
    {
      const int lo_j = max(C.H - 2 - y_first, 0), hi_j = min(C.H + 2 - y_first, R);     // rows H-2 .. H+1
      if (hi_j > lo_j) fix_mine |= ((1u << hi_j) - 1u) & ~((1u << lo_j) - 1u);
    }
    const uint32_t fix_rows = __reduce_or_sync(0xFFFFFFFFu, fix_mine);
    const int flip = y_first & 1;                            // slot 0 of this lane's run holds rows of this parity
    const uint32_t kM = C.thM, tS = C.thS, tL = C.thL;
    int* const crow = a.counts + C.cls * 6 + lane + ((long long)seg.fbegin - 1 - a.out_frame0) * 12;

    int st = (int)(gload % S);
    uint32_t ph = (gload / S) & 1u;
    mbar_wait(&full_bar[st], ph);                            // L_0: the frame before the first one of this item
    uint4 P[R];
    {
      const uint8_t* l0 = tiles + st * Cfg::STAGE_BYTES + lane_off;
#pragma unroll
      for (int j = 0; j < R; ++j) P[j] = *reinterpret_cast<const uint4*>(l0 + (j + 2) * kWsTW);
      __syncwarp();
      if (lane == 0 && S < nloads) issue_at(S, st);          // its slot is free again at once: the rows live in registers
      if (lane == 0 && pf > 0 && S + pf < nloads) prefetch_at(S + pf);
    }
    for (int k = 1; k <= nf; ++k) {
      if (++st == S) { st = 0; ph ^= 1u; }
      mbar_wait(&full_bar[st], ph);
      const uint8_t* cur = tiles + st * Cfg::STAGE_BYTES + lane_off;
      WsCounts c = Cfg::BPS == 2 ? ws_rows10<R, kWsTW>(cur, P, kM, tS, tL)
                                 : (AMTK_WS_SP ? ws_rows_sp<R, kWsTW>(cur, P, kM, tS, tL) : ws_rows<R, kWsTW>(cur, P, kM, tS, tL));
      if (fix_rows) {
        if (Cfg::BPS == 2) ws_fixup10<kWsTW>(cur, fix_rows, fix_mine, tS, tL, c); else ws_fixup<kWsTW>(cur, fix_rows, fix_mine, tS, tL, c);
        __syncwarp();
      }
      // slot -> field: lanes whose run starts on an odd row swap their two slots
      const uint32_t s0 = flip ? c.S[1] : c.S[0], s1 = flip ? c.S[0] : c.S[1];
      const uint32_t l0 = flip ? c.L[1] : c.L[0], l1 = flip ? c.L[0] : c.L[1];
      const uint32_t m0 = flip ? c.M[1] : c.M[0], m1 = flip ? c.M[0] : c.M[1];
      const uint32_t rM0 = __reduce_add_sync(0xFFFFFFFFu, m0), rS0 = __reduce_add_sync(0xFFFFFFFFu, s0), rL0 = __reduce_add_sync(0xFFFFFFFFu, l0);
      const uint32_t rM1 = __reduce_add_sync(0xFFFFFFFFu, m1), rS1 = __reduce_add_sync(0xFFFFFFFFu, s1), rL1 = __reduce_add_sync(0xFFFFFFFFu, l1);
      __syncwarp();                                          // every lane is past its shared-memory reads of this slot
      if (lane == 0 && (k + S) < nloads) issue_at(k + S, st);               // refill the slot that was just released
      if (lane == 0 && pf > 0 && (k + S + pf) < nloads) prefetch_at(k + S + pf);
      if (lane < 6) {                                        // lane = field*3 + metric = the counts[] layout of one class
        const int fld = lane >= 3, met = lane - 3 * fld;
        uint32_t v = met == 0 ? (fld ? rM1 : rM0) : met == 1 ? (fld ? rS1 : rS0) : (fld ? rL1 : rL0);
        v = (met == 0 && Cfg::BPS == 1) ? (v >> 7) : (met == 2 && kWsLviaIdp && Cfg::BPS == 1) ? v / 510u : decode_pair(v);
        if (v) atomicAdd(crow + (size_t)k * 12, (int)v);     // (an unconditional RED measured 3 % slower: hot counter lines)
      }
    }
    gload += (uint32_t)nloads;
  }
}

// Shared band ring: the warps of a CTA stream ONE band of 512 bytes x 4R x GROUPS rows of a plane (BandCfg).  Warp w runs
// the same row code as a warp stream on bytes [128c, 128c + 128) of the 4R rows of row group g (c = w % 4, g = w / 4); the
// slot holds the band's whole box, loaded as two 256-byte-wide TMA boxes (the box-dimension limit) side by side, each with
// a 256-byte pitch.  Against the plane's real size the 3-D map zero-fills the columns right of it and the rows below it; a
// zero column gives a zero response and a zero difference, below every threshold (>= 1), so ragged right edges need no
// tile class of their own, and rows from H + 2 on count nothing.  A warp whose column lies wholly right of the plane, or
// whose row group starts at or below row H + 2, skips the arithmetic but still waits and releases like the others.
// Ring protocol: full_bar[slot] completes when both boxes have landed (TMA complete_tx); each warp releases every load
// once it is done with it (lane 0 adds 1 to released[slot]), and the warp that makes the last (NW-th) release of a load
// refills that slot with load j + S.  No warp waits for another's release, so the only waits are on full_bar, each with a watchdog
// (mm_wait): a protocol error drains the launch instead of hanging the GPU, and the host fails the next call on the
// context (launch_comb_ws reads the watchdog record back).
template <typename Cfg>
__device__ __forceinline__ void ws_bands(const WsArgs& a) {
  constexpr int S = Cfg::STAGES, R = Cfg::R, NW = Cfg::WARPS;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[S];
  __shared__ uint32_t released[S];                           // warp releases per slot (every NW-th is the last of a load)
  __shared__ int item_s[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint8_t* slots = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < S; ++s) { mbar_init(&full_bar[s], 1); released[s] = 0u; }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  int* const dbg = a.queue + 16;                             // watchdog record (zeroed with the queue counter per launch)
  uint32_t gload = 0;                                        // loads consumed so far by the CTA (ring position of L_0 of the current item)
  const int strip = lane & 7, run = lane >> 3;
  const int col = (warp % 4) * kWsTW;                        // this warp's byte column inside the band
  const int grow = (warp / 4) * kWsRuns * R;                 // and the first row of its row group
  const int lane_off = (col / kWbHalf) * Cfg::HALF_BYTES + (grow + run * R) * kWbHalf + (col % kWbHalf) + strip * 16;
  for (int it = 0;; it ^= 1) {                               // item_s is double-buffered: one block barrier per item
    if (tid == 0) item_s[it] = atomicAdd(a.queue, 1);
    __syncthreads();
    const int item = item_s[it];
    if (item >= a.nitems) break;
    const CombSegment seg = a.segs[item];
    if (seg.tile < 0) {
      // Logo item: ScanFrame scores of frames [fbegin, fend) with the slots as scratch.  It neither waits on nor arrives at
      // any mbarrier and loads nothing through the ring, so gload and the ring phases carry over to the next item unchanged.
      scan_item<32 * NW>(a.logo, seg.fbegin, seg.fend, a.out_frame0, slots);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the slots' next writer is the TMA unit
      continue;                                              // (the block barrier at the top orders the scratch reads before it)
    }
    int ci = 0;
#pragma unroll
    for (int k = 1; k < kWsMaxClasses; ++k) if (k < a.nclasses && seg.tile >= a.cl[k].tile0) ci = k;
    const WsClass& C = a.cl[ci];
    const int lt = seg.tile - C.tile0;
    const int ty = lt / C.tilesX, tx = lt - ty * C.tilesX;
    const int y0 = ty * Cfg::TH, x0 = tx * kWbW;
    const int y_first = y0 + grow + run * R;
    const bool two = x0 + kWbHalf < C.W;                     // the right box has bytes in the plane
    const bool active = x0 + col < C.W && y0 + grow < C.H + 2;     // this warp's rows can count anything
    const int nf = seg.fend - seg.fbegin;
    const int nloads = nf + 1;                               // L_0 = previous frame, L_k = frame fbegin+k-1
    const int fprev = seg.fbegin > 0 ? seg.fbegin - 1 : seg.fbegin;
    const CUtensorMap* map = &a.map[C.map];

    auto issue_at = [&](int j, int st) {                     // one thread: load j into slot st
      const int fr = (j == 0) ? fprev : seg.fbegin + j - 1;
      uint8_t* dst = slots + st * Cfg::STAGE_BYTES;
      mbar_expect_tx(&full_bar[st], two ? 2 * Cfg::HALF_BYTES : Cfg::HALF_BYTES);
      tma_load_3d(dst, map, &full_bar[st], x0, y0 - 2, fr);
      if (two) tma_load_3d(dst + Cfg::HALF_BYTES, map, &full_bar[st], x0 + kWbHalf, y0 - 2, fr);
    };
    auto release = [&](int j, int st) {                      // this warp is done with load j (slot st)
      __syncwarp();
      if (lane == 0 && atomicAdd(&released[st], 1u) % NW == NW - 1 && j + S < nloads) issue_at(j + S, st);
    };
    // every slot is free here: each warp released each load of the previous item before the block barrier
    if (tid == 0) {
      const int pro = nloads < S ? nloads : S;
      for (int j = 0; j < pro; ++j) issue_at(j, (int)((gload + (uint32_t)j) % S));
    }
    // rows of this lane's run the spec excludes (bit j = row y_first + j)
    uint32_t fix_mine = 0u;
    if (y_first < 2) fix_mine |= (1u << (2 - y_first)) - 1u;
    {
      const int lo_j = max(C.H - 2 - y_first, 0), hi_j = min(C.H + 2 - y_first, R);     // rows H-2 .. H+1
      if (hi_j > lo_j) fix_mine |= ((1u << hi_j) - 1u) & ~((1u << lo_j) - 1u);
    }
    const uint32_t fix_rows = __reduce_or_sync(0xFFFFFFFFu, fix_mine);
    const int flip = y_first & 1;                            // slot 0 of this lane's run holds rows of this parity
    const uint32_t kM = C.thM, tS = C.thS, tL = C.thL;
    int* const crow = a.counts + C.cls * 6 + lane + ((long long)seg.fbegin - 1 - a.out_frame0) * 12;

    int st = (int)(gload % S);
    uint32_t ph = (gload / S) & 1u;
    mm_wait(&full_bar[st], ph, dbg, 1, 0);                   // L_0: the frame before the first one of this item
    uint4 P[R];
    if (active) {
      const uint8_t* l0 = slots + st * Cfg::STAGE_BYTES + lane_off;
#pragma unroll
      for (int j = 0; j < R; ++j) P[j] = *reinterpret_cast<const uint4*>(l0 + (j + 2) * kWbHalf);
    }
    release(0, st);                                          // the rows live in registers now
    for (int k = 1; k <= nf; ++k) {
      if (++st == S) { st = 0; ph ^= 1u; }
      mm_wait(&full_bar[st], ph, dbg, 2, k);
      if (!active) { release(k, st); continue; }
      const uint8_t* cur = slots + st * Cfg::STAGE_BYTES + lane_off;
      WsCounts c = ws_rows<R, kWbHalf>(cur, P, kM, tS, tL);
      if (fix_rows) {
        ws_fixup<kWbHalf>(cur, fix_rows, fix_mine, tS, tL, c);
        __syncwarp();
      }
      const uint32_t s0 = flip ? c.S[1] : c.S[0], s1 = flip ? c.S[0] : c.S[1];
      const uint32_t l0 = flip ? c.L[1] : c.L[0], l1 = flip ? c.L[0] : c.L[1];
      const uint32_t m0 = flip ? c.M[1] : c.M[0], m1 = flip ? c.M[0] : c.M[1];
      const uint32_t rM0 = __reduce_add_sync(0xFFFFFFFFu, m0), rS0 = __reduce_add_sync(0xFFFFFFFFu, s0), rL0 = __reduce_add_sync(0xFFFFFFFFu, l0);
      const uint32_t rM1 = __reduce_add_sync(0xFFFFFFFFu, m1), rS1 = __reduce_add_sync(0xFFFFFFFFu, s1), rL1 = __reduce_add_sync(0xFFFFFFFFu, l1);
      release(k, st);                                        // every lane is past its shared-memory reads of this slot
      if (lane < 6) {                                        // lane = field*3 + metric = the counts[] layout of one class
        const int fld = lane >= 3, met = lane - 3 * fld;
        uint32_t v = met == 0 ? (fld ? rM1 : rM0) : met == 1 ? (fld ? rS1 : rS0) : (fld ? rL1 : rL0);
        v = met == 0 ? (v >> 7) : (met == 2 && kWsLviaIdp) ? v / 510u : decode_pair(v);
        if (v) atomicAdd(crow + (size_t)k * 12, (int)v);
      }
    }
    gload += (uint32_t)nloads;
  }
}

template <typename Cfg>
__global__ void __launch_bounds__(32 * Cfg::WARPS, Cfg::MIN_CTAS) comb_ws_kernel(const __grid_constant__ WsArgs a) {
  if constexpr (Cfg::BAND) ws_bands<Cfg>(a); else ws_warp_streams<Cfg>(a);
}
}  // namespace amtk
