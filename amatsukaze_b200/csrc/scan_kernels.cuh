// scan_kernels.cuh -- LogoScan accumulation and logo erase on the GPU.
//
// LogoScan::AddFrame (LogoScan.hpp:594-659): per frame, the ROI border pixels decide whether the background is
// flat (max-min <= thy on Y, U and V) and give the background level (mean of the middle half of the sorted border
// values, :414-428); valid frames add f, bg, f^2, bg^2, f*bg to per-pixel accumulators (LogoColor::Add, :357-364).
// The reference accumulates ints in doubles; every partial sum is an exact integer < 2^53, so exact u64 integer
// accumulation is bit-identical after conversion.  A 256-bin histogram replaces the sort exactly.
#pragma once
#include "amtk_internal.h"
#include "exact_math.h"

namespace amtk {

struct ScanClip {
  const uint8_t* base; long long frame_stride; long long offU, offV;
  int pitchY, pitchUV;
  int scanx, scany, scanw, scanh, logUVx, logUVy, thy;
  int frame0, nframes;
};

// One CTA (256 threads) per frame: border histogram per plane -> {valid, bgY, bgU, bgV}.
__global__ void __launch_bounds__(256) scan_border_kernel(const ScanClip c, const uint8_t* __restrict__ select,
                                                          int4* __restrict__ frame_bg) {
  __shared__ unsigned int hist[3][256];
  __shared__ int res[3][2];
  const int f = blockIdx.x, tid = threadIdx.x;
  if (select && !select[f]) { if (tid == 0) frame_bg[f] = make_int4(0, 0, 0, 0); return; }
  for (int i = tid; i < 3 * 256; i += 256) (&hist[0][0])[i] = 0u;
  __syncthreads();
  const uint8_t* fr = c.base + (long long)(c.frame0 + f) * c.frame_stride;
  for (int pl = 0; pl < 3; ++pl) {
    const int w = pl ? (c.scanw >> c.logUVx) : c.scanw, h = pl ? (c.scanh >> c.logUVy) : c.scanh;
    const int pitch = pl ? c.pitchUV : c.pitchY;
    const uint8_t* p = fr + (pl == 0 ? 0 : (pl == 1 ? c.offU : c.offV)) +
                       (pl ? ((c.scanx >> c.logUVx) + (long long)(c.scany >> c.logUVy) * pitch)
                           : (c.scanx + (long long)c.scany * pitch));
    // border = rows 0 and h-1 (all x) + columns 0 and w-1 for y in [1,h-1)  (:616-635)
    const int nb = 2 * w + 2 * (h - 2);
    for (int i = tid; i < nb; i += 256) {
      int x, y;
      if (i < w) { x = i; y = 0; }
      else if (i < 2 * w) { x = i - w; y = h - 1; }
      else { const int k = i - 2 * w; y = 1 + (k >> 1); x = (k & 1) ? (w - 1) : 0; }
      atomicAdd(&hist[pl][p[x + (long long)y * pitch]], 1u);
    }
  }
  __syncthreads();
  if (tid < 3) {
    const int pl = tid;
    const int w = pl ? (c.scanw >> c.logUVx) : c.scanw, h = pl ? (c.scanh >> c.logUVy) : c.scanh;
    const int n = 2 * w + 2 * (h - 2);
    const int lo = n / 4, hi = n - n / 4;            // sorted ranks [lo, hi) are averaged (:421-423)
    int vmin = -1, vmax = 0, rank = 0;
    long long sum = 0;
    for (int v = 0; v < 256; ++v) {
      const int cnt = (int)hist[pl][v];
      if (cnt) {
        if (vmin < 0) vmin = v;
        vmax = v;
        const int a = max(rank, lo), b = min(rank + cnt, hi);
        if (b > a) sum += (long long)(b - a) * v;
        rank += cnt;
      }
    }
    const int nn = hi - lo;
    res[pl][0] = (vmax - vmin > c.thy) ? 0 : 1;      // abs(front-back) > thy rejects (:639-649)
    res[pl][1] = (int)((sum + nn / 2) / nn);         // (int)((t + nn/2)/nn) on exact integers (:425-427)
  }
  __syncthreads();
  if (tid == 0) frame_bg[f] = make_int4(res[0][0] & res[1][0] & res[2][0], res[0][1], res[1][1], res[2][1]);
}

// grid (pixel blocks, frame splits): thread per ROI pixel (Y then U then V), loops over its share of the frames.
// sums: [npix][3] u64 = sumF, sumF2, sumFB.  plane scalars bgsum[pl*2+{0,1}] = sumB, sumB2; bgsum[6] = nvalid.
__global__ void __launch_bounds__(256) scan_accumulate_kernel(const ScanClip c, const int4* __restrict__ frame_bg,
                                                              unsigned long long* __restrict__ sums,
                                                              unsigned long long* __restrict__ bgsum,
                                                              uint8_t* __restrict__ valid_out) {
  const int ny = c.scanw * c.scanh, wc = c.scanw >> c.logUVx, hc = c.scanh >> c.logUVy, nc = wc * hc;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int per = (c.nframes + gridDim.y - 1) / gridDim.y;
  const int f_lo = blockIdx.y * per, f_hi = min(c.nframes, f_lo + per);
  if (i < ny + 2 * nc) {
    int pl, x, y, pitch; long long off;
    if (i < ny) { pl = 0; y = i / c.scanw; x = i - y * c.scanw; pitch = c.pitchY; off = c.scanx + (long long)c.scany * pitch; }
    else {
      const int k = (i - ny) % nc; pl = 1 + (i - ny) / nc; y = k / wc; x = k - y * wc; pitch = c.pitchUV;
      off = (pl == 1 ? c.offU : c.offV) + (c.scanx >> c.logUVx) + (long long)(c.scany >> c.logUVy) * pitch;
    }
    const uint8_t* p = c.base + (long long)c.frame0 * c.frame_stride + off + x + (long long)y * pitch;
    unsigned long long sF = 0, sF2 = 0, sFB = 0;
    for (int f = f_lo; f < f_hi; ++f) {
      const int4 bg = frame_bg[f];
      if (bg.x) {
        const unsigned v = p[(long long)f * c.frame_stride];
        const unsigned b = (unsigned)(pl == 0 ? bg.y : (pl == 1 ? bg.z : bg.w));
        sF += v; sF2 += v * v; sFB += v * b;
      }
    }
    if (sF | sF2 | sFB) {
      atomicAdd(&sums[(size_t)i * 3 + 0], sF); atomicAdd(&sums[(size_t)i * 3 + 1], sF2); atomicAdd(&sums[(size_t)i * 3 + 2], sFB);
    }
  }
  // per-plane background sums + valid count: one thread per frame split
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned long long sb[3] = { 0, 0, 0 }, sb2[3] = { 0, 0, 0 }, nv = 0;
    for (int f = f_lo; f < f_hi; ++f) {
      const int4 bg = frame_bg[f];
      if (valid_out) valid_out[f] = (uint8_t)bg.x;
      if (bg.x) {
        ++nv;
        sb[0] += bg.y; sb2[0] += (unsigned long long)bg.y * bg.y;
        sb[1] += bg.z; sb2[1] += (unsigned long long)bg.z * bg.z;
        sb[2] += bg.w; sb2[2] += (unsigned long long)bg.w * bg.w;
      }
    }
    for (int pl = 0; pl < 3; ++pl) { atomicAdd(&bgsum[pl * 2], sb[pl]); atomicAdd(&bgsum[pl * 2 + 1], sb2[pl]); }
    atomicAdd(&bgsum[6], nv);
  }
}

// ---- LogoScan::AddFrame<uint16_t> (LogoScan.hpp:594-659) on 2-byte samples (9..16 bits) -------------------------
// The same two steps as above on uint16_t samples; pitches are in samples, offsets and the frame stride in bytes.
// The reference keeps the border samples in std::vector<short> (:406, :604-635), so at 16 bits a sample >= 32768 wraps
// negative in the range test, in the sort and in the background value, which can then be negative (reproduced; at up to
// 15 bits it cannot happen).  The sums are signed 64-bit integers kept in the same u64 buffers (two's complement).
//
// Border: the sort is replaced by two 256-bin passes over the order-preserving key k = short + 32768.  Pass 1 counts the
// high bytes (and sums the low bytes) of each bucket, which locates the sorted ranks [lo, hi) that med_average averages;
// pass 2 counts the low bytes of the (at most two) buckets that hold ranks lo and hi - 1.  Exact: every sum is an integer.
__global__ void __launch_bounds__(256) scan_border16_kernel(const ScanClip c, const uint8_t* __restrict__ select,
                                                            int4* __restrict__ frame_bg) {
  __shared__ unsigned int hist[3][256], lsum[3][256];      // per high byte: samples, sum of their low bytes
  __shared__ unsigned int hist2[3][2][256];                // low-byte counts of the buckets holding ranks lo and hi - 1
  __shared__ int edge[3][2], vmin[3], vmax[3];
  __shared__ int res[3][2];
  const int f = blockIdx.x, tid = threadIdx.x;
  if (select && !select[f]) { if (tid == 0) frame_bg[f] = make_int4(0, 0, 0, 0); return; }
  for (int i = tid; i < 3 * 256; i += 256) {
    (&hist[0][0])[i] = 0u; (&lsum[0][0])[i] = 0u; (&hist2[0][0][0])[i] = 0u; (&hist2[0][0][0])[3 * 256 + i] = 0u;
  }
  if (tid < 3) { vmin[tid] = INT_MAX; vmax[tid] = INT_MIN; }
  __syncthreads();
  const uint8_t* fr = c.base + (long long)(c.frame0 + f) * c.frame_stride;
  // key of border sample i of plane pl: rows 0 and h-1 (all x) + columns 0 and w-1 for y in [1,h-1)  (:616-635)
  auto border_key = [&](int pl, int i) -> int {
    const int w = pl ? (c.scanw >> c.logUVx) : c.scanw, h = pl ? (c.scanh >> c.logUVy) : c.scanh;
    const int pitch = pl ? c.pitchUV : c.pitchY;
    const uint16_t* p = reinterpret_cast<const uint16_t*>(fr + (pl == 0 ? 0 : (pl == 1 ? c.offU : c.offV))) +
                        (pl ? ((c.scanx >> c.logUVx) + (long long)(c.scany >> c.logUVy) * pitch)
                            : (c.scanx + (long long)c.scany * pitch));
    int x, y;
    if (i < w) { x = i; y = 0; }
    else if (i < 2 * w) { x = i - w; y = h - 1; }
    else { const int k = i - 2 * w; y = 1 + (k >> 1); x = (k & 1) ? (w - 1) : 0; }
    return (int)(short)p[x + (long long)y * pitch] + 32768;
  };
  auto border_count = [&](int pl) {
    const int w = pl ? (c.scanw >> c.logUVx) : c.scanw, h = pl ? (c.scanh >> c.logUVy) : c.scanh;
    return 2 * w + 2 * (h - 2);
  };
  for (int pl = 0; pl < 3; ++pl) {
    int lo_v = INT_MAX, hi_v = INT_MIN;
    for (int i = tid; i < border_count(pl); i += 256) {
      const int k = border_key(pl, i);
      atomicAdd(&hist[pl][k >> 8], 1u); atomicAdd(&lsum[pl][k >> 8], (unsigned)(k & 255));
      lo_v = min(lo_v, k); hi_v = max(hi_v, k);
    }
    atomicMin(&vmin[pl], lo_v); atomicMax(&vmax[pl], hi_v);
  }
  __syncthreads();
  if (tid < 3) {
    const int pl = tid, n = border_count(pl), lo = n / 4, hi = n - n / 4;
    int rank = 0;
    edge[pl][0] = edge[pl][1] = -1;
    for (int b = 0; b < 256; ++b) {
      const int cnt = (int)hist[pl][b];
      if (lo >= rank && lo < rank + cnt) edge[pl][0] = b;
      if (hi - 1 >= rank && hi - 1 < rank + cnt) edge[pl][1] = b;
      rank += cnt;
    }
  }
  __syncthreads();
  for (int pl = 0; pl < 3; ++pl) {
    for (int i = tid; i < border_count(pl); i += 256) {
      const int k = border_key(pl, i);
      if ((k >> 8) == edge[pl][0]) atomicAdd(&hist2[pl][0][k & 255], 1u);
      else if ((k >> 8) == edge[pl][1]) atomicAdd(&hist2[pl][1][k & 255], 1u);
    }
  }
  __syncthreads();
  if (tid < 3) {
    const int pl = tid, n = border_count(pl);
    const int lo = n / 4, hi = n - n / 4;            // sorted ranks [lo, hi) are averaged (:421-423)
    int rank = 0;
    long long sum = 0;                               // sum of the averaged samples (as short), exact
    for (int b = 0; b < 256; ++b) {
      const int cnt = (int)hist[pl][b];
      if (!cnt) continue;
      const int a = max(rank, lo), e = min(rank + cnt, hi);
      if (a == rank && e == rank + cnt) {            // the whole bucket is averaged
        sum += (long long)cnt * (b * 256 - 32768) + lsum[pl][b];
      } else if (e > a) {                            // a bucket that holds rank lo or hi - 1: resolve its low bytes
        const unsigned int* h2 = hist2[pl][b == edge[pl][0] ? 0 : 1];
        int r = rank;
        for (int l = 0; l < 256; ++l) {
          const int c2 = (int)h2[l];
          const int a2 = max(r, lo), e2 = min(r + c2, hi);
          if (e2 > a2) sum += (long long)(e2 - a2) * (b * 256 + l - 32768);
          r += c2;
        }
      }
      rank += cnt;
    }
    const int nn = hi - lo;
    res[pl][0] = (vmax[pl] - vmin[pl] > c.thy) ? 0 : 1;     // abs(front-back) > thy rejects (:639-649)
    // (int)((t + nn/2)/nn) (:425-427): the double quotient truncates toward zero, as integer division does
    res[pl][1] = nn > 0 ? (int)((sum + nn / 2) / nn) : 0;
  }
  __syncthreads();
  if (tid == 0) frame_bg[f] = make_int4(res[0][0] & res[1][0] & res[2][0], res[0][1], res[1][1], res[2][1]);
}

// LogoColor::Add(f, bg) (:357-364) for 2-byte samples: f*f and f*bg are int products as in the reference.  f*bg always fits
// an int (|bg| <= 32768); f*f does not at 16 bits (f >= 46341): it is taken as the reference's int arithmetic on the
// two's-complement machines it runs on produces it, wrapped to 32 bits.
__global__ void __launch_bounds__(256) scan_accumulate16_kernel(const ScanClip c, const int4* __restrict__ frame_bg,
                                                                unsigned long long* __restrict__ sums,
                                                                unsigned long long* __restrict__ bgsum,
                                                                uint8_t* __restrict__ valid_out) {
  const int ny = c.scanw * c.scanh, wc = c.scanw >> c.logUVx, hc = c.scanh >> c.logUVy, nc = wc * hc;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int per = (c.nframes + gridDim.y - 1) / gridDim.y;
  const int f_lo = blockIdx.y * per, f_hi = min(c.nframes, f_lo + per);
  if (i < ny + 2 * nc) {
    int pl, x, y, pitch; long long off, eoff;        // plane offset (bytes), ROI origin (samples)
    if (i < ny) { pl = 0; y = i / c.scanw; x = i - y * c.scanw; pitch = c.pitchY; off = 0; eoff = c.scanx + (long long)c.scany * pitch; }
    else {
      const int k = (i - ny) % nc; pl = 1 + (i - ny) / nc; y = k / wc; x = k - y * wc; pitch = c.pitchUV;
      off = pl == 1 ? c.offU : c.offV; eoff = (c.scanx >> c.logUVx) + (long long)(c.scany >> c.logUVy) * pitch;
    }
    const uint8_t* p = c.base + (long long)c.frame0 * c.frame_stride + off + 2 * (eoff + x + (long long)y * pitch);
    long long sF = 0, sF2 = 0, sFB = 0;
    for (int f = f_lo; f < f_hi; ++f) {
      const int4 bg = frame_bg[f];
      if (bg.x) {
        const int v = *reinterpret_cast<const uint16_t*>(p + (long long)f * c.frame_stride);
        const int b = pl == 0 ? bg.y : (pl == 1 ? bg.z : bg.w);
        sF += v; sF2 += (int)((unsigned)v * (unsigned)v); sFB += v * b;
      }
    }
    if (sF | sF2 | sFB) {
      atomicAdd(&sums[(size_t)i * 3 + 0], (unsigned long long)sF); atomicAdd(&sums[(size_t)i * 3 + 1], (unsigned long long)sF2);
      atomicAdd(&sums[(size_t)i * 3 + 2], (unsigned long long)sFB);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    long long sb[3] = { 0, 0, 0 }, sb2[3] = { 0, 0, 0 };
    unsigned long long nv = 0;
    for (int f = f_lo; f < f_hi; ++f) {
      const int4 bg = frame_bg[f];
      if (valid_out) valid_out[f] = (uint8_t)bg.x;
      if (bg.x) {
        ++nv;
        sb[0] += bg.y; sb2[0] += (long long)bg.y * bg.y;
        sb[1] += bg.z; sb2[1] += (long long)bg.z * bg.z;
        sb[2] += bg.w; sb2[2] += (long long)bg.w * bg.w;
      }
    }
    for (int pl = 0; pl < 3; ++pl) {
      atomicAdd(&bgsum[pl * 2], (unsigned long long)sb[pl]); atomicAdd(&bgsum[pl * 2 + 1], (unsigned long long)sb2[pl]);
    }
    atomicAdd(&bgsum[6], nv);
  }
}

// ---- InitialLogoCreator::onFrame's store (LogoScan.hpp:881-914) for one batch of a frame stream ------------------
// The batch holds n <= kScanStackBatch rectangles in CopyYV12 packing (Y, then U, then V), `stride` bytes apart (a multiple
// of 16); frame_bg is scan_border_kernel's verdict on them.  One CTA (256 threads) per frame ranks it among the valid
// frames of the batch in read order; the first `room` valid frames are appended to the stack (frame `rank` of `stack`)
// with 16-byte copies, the rest are past the cut-off.  result[0] = frames stored; the CTA of the frame that fills the
// last place writes its batch index to result[1] (the host sets it to -1 before the launch).
constexpr int kScanStackBatch = 200;         // the reference's callback cadence (readCount % 200, :905)
__global__ void __launch_bounds__(256) scan_stack_kernel(const uint8_t* __restrict__ batch, long long stride,
                                                         const int4* __restrict__ frame_bg, int n, int room,
                                                         uint8_t* __restrict__ stack, int* __restrict__ result) {
  const int f = blockIdx.x, tid = threadIdx.x;
  const int valid_t = tid < n ? frame_bg[tid].x : 0;
  const int rank = __syncthreads_count(tid < f && valid_t);       // valid frames before f in the batch
  if (f == 0) {
    const int total = __syncthreads_count(valid_t);
    if (tid == 0) result[0] = min(total, room);
  }
  if (!frame_bg[f].x || rank >= room) return;
  if (tid == 0 && rank == room - 1) result[1] = f;
  const uint4* src = reinterpret_cast<const uint4*>(batch + (long long)f * stride);
  uint4* dst = reinterpret_cast<uint4*>(stack + (long long)rank * stride);
  for (long long i = tid; i < stride / 16; i += 256) dst[i] = src[i];
}

// ---- AMTEraseLogo::Delogo (LogoScan.hpp:1248-1261) on the Y,U,V ROIs of each frame, in place -------------------
struct EraseJob {
  uint8_t* base; long long frame_stride; long long offU, offV;
  int pitchY, pitchUV;           // ELEMENTS
  int frame0, nframes;
  int w, h, logUVx, logUVy, imgx, imgy;
  int uvparity;                  // ((imgy / 2) % 2) of the logo's REAL frame position (the clip may be an ROI-only staging copy)
  const float *aY, *bY, *aU, *bU, *aV, *bV;
  const float* fades;            // [nframes][2] fadeT, fadeB (device)
  float maxv;
};

// Delogo of one sample at one fade (LogoScan.hpp:1248-1261): std::min(std::max(tmp + 0.5f, 0.0f), maxv).
__device__ __forceinline__ float delogo_sample(float srcv, float a, float b, float maxv, float fade) {
  const float tmp = remove_logo(srcv, a, b, maxv, fade, AMTK_FSUB(1.0f, fade));
  const float t = AMTK_FADD(tmp, 0.5f);
  const float m = (t > 0.0f) ? t : 0.0f;
  return (maxv < m) ? maxv : m;
}

// The fade Delogo applies to row y of a plane's logo rectangle of `rows` rows (pl 0: luma, else chroma), or -1 when the
// field passes leave that row untouched.  Equal fades: one frame pass (:1374).  Otherwise each field pass covers rows/2
// rows (:1380-1381, :1391-1395): luma rows of the top field take fadeT, chroma row y takes fadeT when (y & 1) == uvparity
// (:1385-1396).
__device__ __forceinline__ float delogo_row_fade(int pl, int y, int rows, float fadeT, float fadeB, int uvparity) {
  if (fadeT == fadeB) return fadeT;
  if (y >= 2 * (rows / 2)) return -1.0f;
  if (pl == 0) return (y & 1) ? fadeB : fadeT;
  return ((y & 1) == uvparity) ? fadeT : fadeB;
}

template <typename pixel_t>
__global__ void __launch_bounds__(256) erase_logo_kernel(const EraseJob j) {
  const int f = blockIdx.x;
  const float fadeT = j.fades[f * 2], fadeB = j.fades[f * 2 + 1];
  pixel_t* fr = reinterpret_cast<pixel_t*>(j.base + (long long)(j.frame0 + f) * j.frame_stride);
  const int wc = j.w >> j.logUVx, hc = j.h >> j.logUVy, ny = j.w * j.h, nc = wc * hc;
  for (int i = threadIdx.x; i < ny + 2 * nc; i += blockDim.x) {
    pixel_t* p; float a, b, fade;
    if (i < ny) {
      const int y = i / j.w, x = i - y * j.w;
      p = fr + j.imgx + x + (long long)(j.imgy + y) * j.pitchY;
      fade = delogo_row_fade(0, y, j.h, fadeT, fadeB, j.uvparity);
      a = j.aY[i]; b = j.bY[i];
    } else {
      const int k = (i - ny) % nc, pl = (i - ny) / nc;
      const int y = k / wc, x = k - y * wc;
      p = reinterpret_cast<pixel_t*>(reinterpret_cast<uint8_t*>(fr) + (pl == 0 ? j.offU : j.offV)) +
          (j.imgx >> j.logUVx) + x + (long long)((j.imgy >> j.logUVy) + y) * j.pitchUV;
      fade = delogo_row_fade(1, y, hc, fadeT, fadeB, j.uvparity);
      a = (pl == 0 ? j.aU : j.aV)[k]; b = (pl == 0 ? j.bU : j.bV)[k];
    }
    if (fade < 0.0f) continue;
    *p = (pixel_t)delogo_sample((float)*p, a, b, j.maxv, fade);
  }
}

// ---- amtk_erase_logo_clip out of place: dst frame k = source frame src0 + k with its logo rectangles erased ----------
// One pass writes every dst sample once: each thread moves one 16-byte piece of a row of one plane (grid: row pieces,
// plane, frames), and where the piece meets the plane's logo rectangle it replaces those samples by erase_logo_kernel's
// values (delogo_sample, delogo_row_fade) before the store.  VEC: every base, stride, plane offset and pitch of src and dst
// is a multiple of 16, so whole pieces move as one streaming 16-byte load and store; otherwise byte by byte, with the same
// values.  Only the row_bytes of each row are written (row padding stays untouched).
struct EraseCopyJob {
  const uint8_t* src; uint8_t* dst;
  long long sstride, dstride;
  long long s_off[3], d_off[3];   // plane offsets in a frame (Y: 0)
  int s_pitch[3], d_pitch[3];     // bytes
  int row_bytes[3], rows[3];
  int rx[3], ry[3], rw[3], rh[3]; // each plane's logo rectangle, samples
  const float* a[3]; const float* b[3];
  const float* fades;             // [nframes][2] fadeT, fadeB (device)
  int src0, nframes, pieces_y;    // pieces_y: 16-byte pieces of a luma row
  float maxv; int uvparity;
};

template <typename pixel_t, bool VEC>
__global__ void __launch_bounds__(256) erase_copy_kernel(const __grid_constant__ EraseCopyJob j) {
  constexpr int kPer = 16 / (int)sizeof(pixel_t);
  const int pl = blockIdx.y;
  const int rb = j.row_bytes[pl], pieces = (rb + 15) >> 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)j.rows[pl] * pieces) return;
  const int y = (int)(i / pieces), c = (int)(i - (long long)y * pieces);
  const int nbytes = min(16, rb - c * 16);
  const int ry = y - j.ry[pl], x0 = c * kPer;
  const bool in_rows = ry >= 0 && ry < j.rh[pl] && x0 < j.rx[pl] + j.rw[pl] && x0 + kPer > j.rx[pl];
  for (int k = blockIdx.z; k < j.nframes; k += gridDim.z) {
    const uint8_t* s = j.src + (long long)(j.src0 + k) * j.sstride + j.s_off[pl] + (long long)y * j.s_pitch[pl] + c * 16;
    uint8_t* d = j.dst + (long long)k * j.dstride + j.d_off[pl] + (long long)y * j.d_pitch[pl] + c * 16;
    union { uint4 v; uint8_t b[16]; pixel_t p[kPer]; } u;
    if (VEC && nbytes == 16) u.v = __ldcs(reinterpret_cast<const uint4*>(s));
    else for (int q = 0; q < nbytes; ++q) u.b[q] = s[q];
    if (in_rows) {
      const float fade = delogo_row_fade(pl, ry, j.rh[pl], j.fades[2 * k], j.fades[2 * k + 1], j.uvparity);
      if (fade >= 0.0f) {
        const int xa = max(x0, j.rx[pl]), xb = min(min(x0 + kPer, j.rx[pl] + j.rw[pl]), x0 + nbytes / (int)sizeof(pixel_t));
        const float* a = j.a[pl] + (long long)ry * j.rw[pl] - j.rx[pl];
        const float* b = j.b[pl] + (long long)ry * j.rw[pl] - j.rx[pl];
        for (int x = xa; x < xb; ++x) u.p[x - x0] = (pixel_t)delogo_sample((float)u.p[x - x0], a[x], b[x], j.maxv, fade);
      }
    }
    if (VEC && nbytes == 16) __stcs(reinterpret_cast<uint4*>(d), u.v);
    else for (int q = 0; q < nbytes; ++q) d[q] = u.b[q];
  }
}

// ---- AMTEraseLogo::CalcFade (LogoScan.hpp:1317-1341) for outputs [n0, n0 + count) of an erase stream -------------
// codes[n] (uploaded at create): 0 or 1 = the fade of a uniform logoframe window (both fields), 2 = CalcFade2 on the nine
// records calc_fade2_index picks, read from the record ring (frame f's record at row f % ring).  One thread per output.
struct RingRecords {
  const float* rec; int ring, N, n;
  __host__ __device__ const float* operator()(int i) const { return rec + (long long)(calc_fade2_index(N, N, n, i - 4) % ring) * 33; }
};

__global__ void __launch_bounds__(256) erase_fade_kernel(const uint8_t* __restrict__ codes, const float* __restrict__ rec,
                                                         int ring, int N, int n0, int count, float* __restrict__ fades) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  const int n = n0 + k, code = codes[n];
  float ft, fb;
  if (code < 2) ft = fb = (float)code;
  else calc_fade2_decide(RingRecords{ rec, ring, N, n }, &ft, &fb);
  fades[2 * k] = ft; fades[2 * k + 1] = fb;
}

// ---- LogoFrame::ScanFrame's input from one device frame of a logo scan stream (DESIGN.md section 3.3.3) -----------
// Copies each evaluated logo's luma rectangle into the frame's slot.  rects[blockIdx.y]: the rectangle's first byte xb and
// row y in the frame as addressed (row r at ybase + (y + r) * step), row_bytes x rows, and where its rows go in the slot
// (off, dpitch: multiples of 16).  Each thread moves one 16-byte column of a row: one vector copy when the source is
// 16-byte aligned, else the widest copies its alignment allows (logo x positions can be odd).
struct LogoRect { long long off; int xb, y, row_bytes, rows, dpitch; };

__global__ void __launch_bounds__(256) logo_rect_gather_kernel(const uint8_t* __restrict__ ybase, long long step,
                                                               uint8_t* __restrict__ slot, const LogoRect* __restrict__ rects) {
  const LogoRect r = rects[blockIdx.y];
  const int cols = (r.row_bytes + 15) >> 4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cols * r.rows; i += gridDim.x * blockDim.x) {
    const int y = i / cols, c = i - y * cols;
    const uint8_t* s = ybase + (long long)(r.y + y) * step + r.xb + c * 16;
    uint8_t* d = slot + r.off + (long long)y * r.dpitch + c * 16;
    const int n = min(16, r.row_bytes - c * 16);
    const unsigned a = (unsigned)reinterpret_cast<uintptr_t>(s);
    if (n == 16 && (a & 15) == 0) {
      *reinterpret_cast<uint4*>(d) = __ldg(reinterpret_cast<const uint4*>(s));
    } else if (n == 16 && (a & 7) == 0) {
      reinterpret_cast<uint2*>(d)[0] = __ldg(reinterpret_cast<const uint2*>(s));
      reinterpret_cast<uint2*>(d)[1] = __ldg(reinterpret_cast<const uint2*>(s) + 1);
    } else if ((a & 3) == 0 && (n & 3) == 0) {
      for (int k = 0; k < n; k += 4) *reinterpret_cast<unsigned*>(d + k) = __ldg(reinterpret_cast<const unsigned*>(s + k));
    } else if ((a & 1) == 0 && (n & 1) == 0) {
      for (int k = 0; k < n; k += 2) *reinterpret_cast<unsigned short*>(d + k) = __ldg(reinterpret_cast<const unsigned short*>(s + k));
    } else {
      for (int k = 0; k < n; ++k) d[k] = __ldg(s + k);
    }
  }
}

// ---- AMTSource::MergeField (AMTSource.hpp:291-355): weave two decoded frames, optional NV12 chroma split ------------
struct WeaveJob {
  const uint8_t* src; uint8_t* dst;
  long long sstride, dstride, s_offu, s_offv, d_offu, d_offv;
  int s_pitchY, s_pitchUV, d_pitchY, d_pitchUV;   // BYTES
  int row_bytes_y, row_bytes_c;                   // payload bytes per luma / chroma row (planar)
  int H, HC, bps, nv12;
  const int* top_idx; const int* bot_idx;         // device
  int dst_frame0;
};

// grid (row blocks, 3 planes, frames); each thread moves 16 bytes of a row (tail bytes one by one)
__global__ void __launch_bounds__(256) weave_kernel(const WeaveJob j) {
  const int k = blockIdx.z, pl = blockIdx.y;
  const int rows = pl ? j.HC : j.H;
  const int rb = pl ? j.row_bytes_c : j.row_bytes_y;
  const uint8_t* ft = j.src + (long long)j.top_idx[k] * j.sstride;
  const uint8_t* fb = j.src + (long long)j.bot_idx[k] * j.sstride;
  uint8_t* fd = j.dst + (long long)(j.dst_frame0 + k) * j.dstride;
  const int vec_per_row = (rb + 15) / 16;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)rows * vec_per_row;
       i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / vec_per_row), v = (int)(i - (long long)y * vec_per_row);
    const uint8_t* fs = (y & 1) ? fb : ft;             // even rows from `top`, odd rows from `bottom` (Copy1 :292-302)
    const int nbytes = min(16, rb - v * 16);
    if (pl == 0 || !j.nv12) {
      const uint8_t* s = fs + (pl == 0 ? 0 : (pl == 1 ? j.s_offu : j.s_offv)) + (long long)y * (pl ? j.s_pitchUV : j.s_pitchY) + v * 16;
      uint8_t* d = fd + (pl == 0 ? 0 : (pl == 1 ? j.d_offu : j.d_offv)) + (long long)y * (pl ? j.d_pitchUV : j.d_pitchY) + v * 16;
      if (nbytes == 16 && ((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d)) & 15) == 0)
        *reinterpret_cast<uint4*>(d) = *reinterpret_cast<const uint4*>(s);
      else
        for (int b = 0; b < nbytes; ++b) d[b] = s[b];
    } else {
      // NV12: interleaved UV row -> U (pl 1) or V (pl 2) samples (Copy2 :304-321)
      const uint8_t* s = fs + j.s_offu + (long long)y * j.s_pitchUV;
      uint8_t* d = fd + (pl == 1 ? j.d_offu : j.d_offv) + (long long)y * j.d_pitchUV + v * 16;
      const int comp = pl - 1;
      for (int b = 0; b < nbytes; b += j.bps) {
        const int xs = (v * 16 + b) / j.bps;           // sample index in the row
        for (int q = 0; q < j.bps; ++q) d[b + q] = s[(xs * 2 + comp) * j.bps + q];
      }
    }
  }
}

// ---- read-bandwidth probe: what a do-nothing streaming read achieves on this GPU ---------------------------------
__global__ void __launch_bounds__(256) read_probe_kernel(const uint4* __restrict__ p, size_t n16, unsigned* __restrict__ sink) {
  uint4 acc = make_uint4(0, 0, 0, 0);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < n16; i += 4 * stride) {          // 4 independent 16-byte loads in flight per thread
    const uint4 a = __ldcs(p + i), b = __ldcs(p + i + stride), c = __ldcs(p + i + 2 * stride), d = __ldcs(p + i + 3 * stride);
    acc.x ^= a.x ^ b.x ^ c.x ^ d.x; acc.y ^= a.y ^ b.y ^ c.y ^ d.y; acc.z ^= a.z ^ b.z ^ c.z ^ d.z; acc.w ^= a.w ^ b.w ^ c.w ^ d.w;
  }
  for (; i < n16; i += stride) { const uint4 a = __ldcs(p + i); acc.x ^= a.x; acc.y ^= a.y; acc.z ^= a.z; acc.w ^= a.w; }
  const unsigned v = acc.x ^ acc.y ^ acc.z ^ acc.w;
  if (v == 0x9E3779B9u) atomicAdd(sink, 1u);               // keeps the loads alive; practically never taken
}

}  // namespace amtk
