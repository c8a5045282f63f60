// tnr_kernels.cuh -- temporal noise reduction (the reference's TemporalNRFilter, VideoFilter.hpp:27-212) on the GPU.
//
// Output frame n of a clip of N frames averages the window w_i = clamp(n - d + i, 0, N - 1), i = 0..2d.  Per luma pixel:
// a window frame is "in" when |Y-Yi| + |U-Ui| + |V-Vi| <= thresh (the centre frame w_d always is, :177-180), k counts
// them, f = 1.0f / k (:183), and dY = 0.5f + f*Y_i over the in-frames in ascending i (:185-199), each product and sum
// rounded on its own (no FMA); out = (T)dY, which the x64 build truncates through a 32-bit signed integer (:202).  U and V
// take the same chain with the mask of the luma pixel that writes them (:204-208): (2cx, 2cy) progressive,
// (2cx, 4(cy>>1) + (cy&1)) interlaced.  DESIGN.md section 3.4 restates the spec line by line.
//
// Work unit ("group"): one chroma row cy and the two luma rows that share it (2cy, 2cy+1 progressive; 4(cy>>1)+(cy&1) and
// +2 interlaced; the first one writes the chroma), 16 bytes of each luma row and the 8 matching bytes of U and V.  There
// is no spatial stencil, so a thread walks a run of output frames down its column through time: tnr_kernel<Tin, Tout,
// D, ...> keeps the 2d+1 window in registers and loads frame n+d+1 while it filters frame n, so every input byte is read
// once per run (plus 2d halo frames) and every output byte is written once.  tnr_general_kernel<Tin, Tout, ...> covers
// d up to 63 by reading the window from memory for every output frame.
//
// RING = true instantiates the same kernels for amtk_tnr_stream: the source is a ring of `src_count` frame slots in HBM
// and frame f lives in slot f mod src_count, so a window that wraps past the end of the ring is only addresses.
//
// WIDEN = true filters source samples Tin at src_bits into Tout = uint16_t at dst_bits = src_bits + k (ConvertBits fused
// into the filter; DESIGN.md section 3.4): the output equals the filter at dst_bits on the samples src << k.  The masks
// are the ones built at src_bits (dist << k <= t << (dst_bits-8) exactly when dist <= t << (src_bits-8)), and because
// scaling by 2^k commutes with binary32 rounding here (no overflow, no subnormal product), dY starts at 2^-k * 0.5f, adds
// f*Y_i on the unshifted samples and is multiplied by 2^k before the truncation.  A group still covers 16 destination
// bytes per luma row, so from 8 bits it loads 8 source bytes per luma row and 4 per chroma row (TnrHalfGroup).
#pragma once
#include <type_traits>
#include "amtk_internal.h"

namespace amtk {

static constexpr int kTnrThreads = 128;
static constexpr int kTnrMaxD = 63;          // 2d+1 <= MAX_NFRAMES = 128 (VideoFilter.hpp:38-40,91)
static constexpr int kTnrMaxTemplD = 7;      // d <= this runs the register-window kernel

struct TnrArgs {
  const uint8_t* src;                 // frame `src_first` of the clip (frames [src_first, src_first+src_count) resident);
                                      // RING kernels: slot 0 of a ring of src_count slots (src_first is 0)
  long long src_stride, s_offu, s_offv;
  int s_pitchY, s_pitchUV;
  int src_first, src_count;
  uint8_t* dst;                       // destination of output frame `lo`
  long long dst_stride, d_offu, d_offv;
  int d_pitchY, d_pitchUV;
  int W, H, N;                        // luma size; clip length (the window clamps at 0 and N-1)
  int lo, hi, run;                    // output frames [lo, hi) of the clip, `run` consecutive frames per thread
  int thresh, interlaced;
  int vec;                            // 1: every group address is aligned to its load / store width
};

struct TnrWiden { float half, scale; };   // WIDEN kernels: 2^-k * 0.5f and 2^k

// 16 luma bytes of each of the two rows, 8 bytes of U and of V
struct TnrGroup { uint4 a, b; uint2 u, v; };
// the same pixels of an 8-bit source widened to 2-byte samples: 8 luma bytes of each row, 4 bytes of U and of V
struct TnrHalfGroup { uint2 a, b; uint1 u, v; };
template <typename Tin, typename Tout>
using TnrIn = typename std::conditional<sizeof(Tin) == sizeof(Tout), TnrGroup, TnrHalfGroup>::type;

__device__ __forceinline__ void tnr_ld(uint4& r, const uint8_t* p) { r = __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void tnr_ld(uint2& r, const uint8_t* p) { r = __ldg(reinterpret_cast<const uint2*>(p)); }
__device__ __forceinline__ void tnr_ld(uint1& r, const uint8_t* p) { r.x = __ldg(reinterpret_cast<const unsigned*>(p)); }

template <typename T> __device__ __forceinline__ uint32_t tnr_elem(const uint32_t* w, int j) {
  if (sizeof(T) == 1) return (w[j >> 2] >> ((j & 3) * 8)) & 0xFFu;
  return (w[j >> 1] >> ((j & 1) * 16)) & 0xFFFFu;
}
template <typename T> __device__ __forceinline__ void tnr_put(uint32_t* w, int j, uint32_t v) {
  if (sizeof(T) == 1) w[j >> 2] |= v << ((j & 3) * 8);
  else w[j >> 1] |= v << ((j & 1) * 16);
}

// exact float of an integer < 2^23: two full-rate instructions instead of a quarter-rate I2F
__device__ __forceinline__ float tnr_u2f(uint32_t v) { return __fsub_rn(__uint_as_float(0x4B000000u | v), 8388608.0f); }

struct TnrGeom {
  int ya, yb, cy, x0, cx0;            // luma rows, chroma row, first luma / chroma column of the group
  int nl, nc;                         // valid luma / chroma elements in this group
};

template <typename T> __device__ __forceinline__ TnrGeom tnr_geom(const TnrArgs& a, int gx, int cy) {
  constexpr int NL = 16 / sizeof(T);
  TnrGeom g;
  g.cy = cy;
  g.ya = a.interlaced ? 4 * (cy >> 1) + (cy & 1) : 2 * cy;
  g.yb = g.ya + (a.interlaced ? 2 : 1);
  g.x0 = gx * NL; g.cx0 = gx * (NL / 2);
  g.nl = min(NL, a.W - g.x0); g.nc = g.nl >> 1;
  return g;
}

// One group of source frame f, at the source's sample width; g is the geometry of the destination samples (Tout).
template <typename Tin, typename Tout, bool RING>
__device__ __forceinline__ TnrIn<Tin, Tout> tnr_load(const TnrArgs& a, const TnrGeom& g, int f, bool full) {
  const uint8_t* fr = a.src + (long long)(RING ? f % a.src_count : f - a.src_first) * a.src_stride;
  const uint8_t* ra = fr + (long long)g.ya * a.s_pitchY + g.x0 * (int)sizeof(Tin);
  const uint8_t* rb = fr + (long long)g.yb * a.s_pitchY + g.x0 * (int)sizeof(Tin);
  const uint8_t* ru = fr + a.s_offu + (long long)g.cy * a.s_pitchUV + g.cx0 * (int)sizeof(Tin);
  const uint8_t* rv = fr + a.s_offv + (long long)g.cy * a.s_pitchUV + g.cx0 * (int)sizeof(Tin);
  TnrIn<Tin, Tout> r;
  if (full) {
    tnr_ld(r.a, ra); tnr_ld(r.b, rb); tnr_ld(r.u, ru); tnr_ld(r.v, rv);
    return r;
  }
  r.a = r.b = decltype(r.a){}; r.u = r.v = decltype(r.u){};
  for (int j = 0; j < g.nl; ++j) {
    tnr_put<Tin>(&r.a.x, j, reinterpret_cast<const Tin*>(ra)[j]);
    tnr_put<Tin>(&r.b.x, j, reinterpret_cast<const Tin*>(rb)[j]);
  }
  for (int j = 0; j < g.nc; ++j) {
    tnr_put<Tin>(&r.u.x, j, reinterpret_cast<const Tin*>(ru)[j]);
    tnr_put<Tin>(&r.v.x, j, reinterpret_cast<const Tin*>(rv)[j]);
  }
  return r;
}

template <typename T>
__device__ __forceinline__ void tnr_store(const TnrArgs& a, const TnrGeom& g, int n, bool full, const TnrGroup& o) {
  uint8_t* fr = a.dst + (long long)(n - a.lo) * a.dst_stride;
  uint8_t* ra = fr + (long long)g.ya * a.d_pitchY + g.x0 * (int)sizeof(T);
  uint8_t* rb = fr + (long long)g.yb * a.d_pitchY + g.x0 * (int)sizeof(T);
  uint8_t* ru = fr + a.d_offu + (long long)g.cy * a.d_pitchUV + g.cx0 * (int)sizeof(T);
  uint8_t* rv = fr + a.d_offv + (long long)g.cy * a.d_pitchUV + g.cx0 * (int)sizeof(T);
  if (full) {
    *reinterpret_cast<uint4*>(ra) = o.a; *reinterpret_cast<uint4*>(rb) = o.b;
    *reinterpret_cast<uint2*>(ru) = o.u; *reinterpret_cast<uint2*>(rv) = o.v;
    return;
  }
  for (int j = 0; j < g.nl; ++j) {
    reinterpret_cast<T*>(ra)[j] = (T)tnr_elem<T>(&o.a.x, j);
    reinterpret_cast<T*>(rb)[j] = (T)tnr_elem<T>(&o.b.x, j);
  }
  for (int j = 0; j < g.nc; ++j) {
    reinterpret_cast<T*>(ru)[j] = (T)tnr_elem<T>(&o.u.x, j);
    reinterpret_cast<T*>(rv)[j] = (T)tnr_elem<T>(&o.v.x, j);
  }
}

// (T)dY of the x64 reference: truncation through int (cvttss2si), then the low bits
template <typename T> __device__ __forceinline__ uint32_t tnr_out(float v) { return (uint32_t)(T)__float2int_rz(v); }
// WIDEN: the sum was taken on unshifted samples from 2^-k * 0.5f; times 2^k it is the sum on the samples << k
template <typename T, bool WIDEN> __device__ __forceinline__ uint32_t tnr_out(float v, float scale) {
  return tnr_out<T>(WIDEN ? __fmul_rn(v, scale) : v);
}

// The 1/k table (VideoFilter.hpp:171-183: sumKernel adds 1.0f per in-frame, so it is exactly k; 1.f / k is IEEE division)
__device__ __forceinline__ void tnr_fill_rcp(float* rcp) {
  for (int k = threadIdx.x; k < 129; k += blockDim.x) rcp[k] = k ? __fdiv_rn(1.0f, (float)k) : 0.0f;
  __syncthreads();
}

// Filter one group of output frame n from the window held in registers (win[i] = frame w_i).
template <typename Tin, typename Tout, bool WIDEN, int NF>
__device__ __forceinline__ TnrGroup tnr_filter(const TnrIn<Tin, Tout> (&win)[NF], int thresh, const float* rcp, TnrWiden w) {
  constexpr int NL = 16 / sizeof(Tout), NC = NL / 2, D = NF / 2;
  const float d0 = WIDEN ? w.half : 0.5f;
  TnrGroup o;
  o.a = o.b = make_uint4(0, 0, 0, 0); o.u = o.v = make_uint2(0, 0);
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    const uint32_t Uc = tnr_elem<Tin>(&win[D].u.x, j), Vc = tnr_elem<Tin>(&win[D].v.x, j);
    int duv[NF];      // |U-Ui| + |V-Vi|, shared by the 2x2 luma pixels of this chroma sample
#pragma unroll
    for (int i = 0; i < NF; ++i) duv[i] = (int)__sad(Uc, tnr_elem<Tin>(&win[i].u.x, j), __sad(Vc, tnr_elem<Tin>(&win[i].v.x, j), 0u));
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int row = p >> 1, x = 2 * j + (p & 1);
      const uint32_t Yc = tnr_elem<Tin>(row ? &win[D].b.x : &win[D].a.x, x);
      uint32_t mask = 0;
#pragma unroll
      for (int i = 0; i < NF; ++i) {
        const int diff = (int)__sad(Yc, tnr_elem<Tin>(row ? &win[i].b.x : &win[i].a.x, x), (uint32_t)duv[i]);
        mask |= (diff <= thresh ? 1u : 0u) << i;
      }
      const float f = rcp[__popc(mask)];
      float dY = d0;
#pragma unroll
      for (int i = 0; i < NF; ++i) {        // an out-frame adds 0.0f * Y_i = +0: dY + 0 == dY exactly
        const float c = (mask >> i) & 1u ? f : 0.0f;
        dY = __fadd_rn(dY, __fmul_rn(c, tnr_u2f(tnr_elem<Tin>(row ? &win[i].b.x : &win[i].a.x, x))));
      }
      tnr_put<Tout>(row ? &o.b.x : &o.a.x, x, tnr_out<Tout, WIDEN>(dY, w.scale));
      if (p == 0) {                         // x even on the chroma-writing row
        float dU = d0, dV = d0;
#pragma unroll
        for (int i = 0; i < NF; ++i) {
          const float c = (mask >> i) & 1u ? f : 0.0f;
          dU = __fadd_rn(dU, __fmul_rn(c, tnr_u2f(tnr_elem<Tin>(&win[i].u.x, j))));
          dV = __fadd_rn(dV, __fmul_rn(c, tnr_u2f(tnr_elem<Tin>(&win[i].v.x, j))));
        }
        tnr_put<Tout>(&o.u.x, j, tnr_out<Tout, WIDEN>(dU, w.scale));
        tnr_put<Tout>(&o.v.x, j, tnr_out<Tout, WIDEN>(dV, w.scale));
      }
    }
  }
  return o;
}

__device__ __forceinline__ int tnr_clamp(int f, int N) { return f < 0 ? 0 : (f >= N ? N - 1 : f); }

// Register-window kernel for d = D <= kTnrMaxTemplD.  grid.x covers the groups of one frame, grid.y the runs of frames.
template <typename Tin, typename Tout, int D, bool RING, bool WIDEN>
__global__ void __launch_bounds__(kTnrThreads) tnr_kernel(const TnrArgs a, const TnrWiden wd) {
  static_assert(WIDEN || std::is_same<Tin, Tout>::value, "only the widening kernels change the sample format");
  constexpr int NF = 2 * D + 1, NL = 16 / sizeof(Tout);
  __shared__ float rcp[129];
  tnr_fill_rcp(rcp);
  const int ngx = (a.W + NL - 1) / NL, hc = a.H >> 1;
  const int gid = blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= ngx * hc) return;
  const int n0 = a.lo + blockIdx.y * a.run, n1 = min(a.hi, n0 + a.run);
  if (n0 >= n1) return;
  const TnrGeom g = tnr_geom<Tout>(a, gid % ngx, gid / ngx);
  const bool full = a.vec && g.nl == NL;
  TnrIn<Tin, Tout> win[NF];
#pragma unroll
  for (int i = 0; i < NF; ++i) win[i] = tnr_load<Tin, Tout, RING>(a, g, tnr_clamp(n0 - D + i, a.N), full);
  for (int n = n0; n < n1; ++n) {
    TnrIn<Tin, Tout> next;
    const bool more = n + 1 < n1;
    if (more) next = tnr_load<Tin, Tout, RING>(a, g, tnr_clamp(n + 1 + D, a.N), full);
    tnr_store<Tout>(a, g, n, full, tnr_filter<Tin, Tout, WIDEN, NF>(win, a.thresh, rcp, wd));
    if (more) {
#pragma unroll
      for (int i = 0; i + 1 < NF; ++i) win[i] = win[i + 1];
      win[NF - 1] = next;
    }
  }
}

// Any d in [0, 63]: the window is read from memory (L1/L2) for every output frame; pass 1 counts the in-frames of each
// pixel, pass 2 re-derives each inclusion and adds in frame order.
template <typename Tin, typename Tout, bool RING, bool WIDEN>
__global__ void __launch_bounds__(kTnrThreads) tnr_general_kernel(const TnrArgs a, int d, const TnrWiden wd) {
  static_assert(WIDEN || std::is_same<Tin, Tout>::value, "only the widening kernels change the sample format");
  constexpr int NL = 16 / sizeof(Tout), NC = NL / 2;
  __shared__ float rcp[129];
  tnr_fill_rcp(rcp);
  const int ngx = (a.W + NL - 1) / NL, hc = a.H >> 1;
  const int gid = blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= ngx * hc) return;
  const int n0 = a.lo + blockIdx.y * a.run, n1 = min(a.hi, n0 + a.run);
  const TnrGeom g = tnr_geom<Tout>(a, gid % ngx, gid / ngx);
  const bool full = a.vec && g.nl == NL;
  const int nf = 2 * d + 1;
  const float d0 = WIDEN ? wd.half : 0.5f;
  for (int n = n0; n < n1; ++n) {
    const TnrIn<Tin, Tout> c = tnr_load<Tin, Tout, RING>(a, g, tnr_clamp(n, a.N), full);
    TnrGroup o;
    o.a = o.b = make_uint4(0, 0, 0, 0); o.u = o.v = make_uint2(0, 0);
    int k[2 * NL];
#pragma unroll
    for (int p = 0; p < 2 * NL; ++p) k[p] = 0;
    for (int i = 0; i < nf; ++i) {
      const TnrIn<Tin, Tout> w = tnr_load<Tin, Tout, RING>(a, g, tnr_clamp(n - d + i, a.N), full);
#pragma unroll
      for (int p = 0; p < 2 * NL; ++p) {
        const int x = p % NL, j = x >> 1;
        const uint32_t duv = __sad(tnr_elem<Tin>(&c.u.x, j), tnr_elem<Tin>(&w.u.x, j), __sad(tnr_elem<Tin>(&c.v.x, j), tnr_elem<Tin>(&w.v.x, j), 0u));
        const uint32_t yc = tnr_elem<Tin>(p < NL ? &c.a.x : &c.b.x, x), yi = tnr_elem<Tin>(p < NL ? &w.a.x : &w.b.x, x);
        k[p] += (int)__sad(yc, yi, duv) <= a.thresh;
      }
    }
    float acc[2 * NL], accU[NC], accV[NC];
#pragma unroll
    for (int p = 0; p < 2 * NL; ++p) acc[p] = d0;
#pragma unroll
    for (int j = 0; j < NC; ++j) { accU[j] = d0; accV[j] = d0; }
    for (int i = 0; i < nf; ++i) {
      const TnrIn<Tin, Tout> w = tnr_load<Tin, Tout, RING>(a, g, tnr_clamp(n - d + i, a.N), full);
#pragma unroll
      for (int p = 0; p < 2 * NL; ++p) {
        const int x = p % NL, j = x >> 1;
        const uint32_t duv = __sad(tnr_elem<Tin>(&c.u.x, j), tnr_elem<Tin>(&w.u.x, j), __sad(tnr_elem<Tin>(&c.v.x, j), tnr_elem<Tin>(&w.v.x, j), 0u));
        const uint32_t yc = tnr_elem<Tin>(p < NL ? &c.a.x : &c.b.x, x), yi = tnr_elem<Tin>(p < NL ? &w.a.x : &w.b.x, x);
        const float f = (int)__sad(yc, yi, duv) <= a.thresh ? rcp[k[p]] : 0.0f;
        acc[p] = __fadd_rn(acc[p], __fmul_rn(f, tnr_u2f(yi)));
        if (p < NL && (x & 1) == 0) {
          accU[j] = __fadd_rn(accU[j], __fmul_rn(f, tnr_u2f(tnr_elem<Tin>(&w.u.x, j))));
          accV[j] = __fadd_rn(accV[j], __fmul_rn(f, tnr_u2f(tnr_elem<Tin>(&w.v.x, j))));
        }
      }
    }
#pragma unroll
    for (int p = 0; p < 2 * NL; ++p) tnr_put<Tout>(p < NL ? &o.a.x : &o.b.x, p % NL, tnr_out<Tout, WIDEN>(acc[p], wd.scale));
#pragma unroll
    for (int j = 0; j < NC; ++j) { tnr_put<Tout>(&o.u.x, j, tnr_out<Tout, WIDEN>(accU[j], wd.scale)); tnr_put<Tout>(&o.v.x, j, tnr_out<Tout, WIDEN>(accV[j], wd.scale)); }
    tnr_store<Tout>(a, g, n, full, o);
  }
}

}  // namespace amtk
