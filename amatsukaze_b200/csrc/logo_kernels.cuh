// logo_kernels.cuh -- logo-template correlation on the GPU.
//
// Replaces, per frame: DeintY/CopyY (LogoScan.hpp:763-790), LogoDataParam::EvaluateLogo (:231-255) and
// LogoDataParam::CorrelationScore (:288-318) incl. CalcCorrelation5x5_AVX (ComputeKernel.cpp:77-121).
//
// Structure (two launches per evaluation job):
//   logo_scores_kernel : grid (pixel slices, frame lanes).  Each thread OWNS up to PXT feature pixels of the logo
//                        and keeps their 25 zero-mean taps in registers for the whole launch, so the 129 KB tap
//                        table is read once per CTA instead of once per frame (it would otherwise need ~400 TB/s
//                        of L2 bandwidth at the frame rates the streaming pass reaches).  Per frame the CTA stages
//                        the ROI as float (deinterlaced or raw) in shared memory, and per fade level builds the
//                        logo-removed image `work` in shared memory and lets every thread emit the score of its
//                        pixels, using the exact AVX expression tree (exact_math.h).
//   logo_sum_kernel    : the reference adds the ~1.3k pixel scores of an evaluation SEQUENTIALLY in float
//                        (LogoScan.hpp:310).  That order is kept (bit-exact results), but one thread per
//                        (frame, fade) runs its chain, so all 32 lanes of a warp carry independent chains.
#pragma once
#include "amtk_internal.h"
#include "exact_math.h"
#include "tma_utils.cuh"

namespace amtk {

constexpr int kEvalThreads = 512;
constexpr int kMaxFades = 24;

struct EvalJob {
  const void* ybase;         // Y plane of frame 0 of the (device-resident) clip window
  long long frame_stride;    // bytes
  int pitch;                 // ELEMENTS
  int frame0, nframes;       // frames [frame0, frame0+nframes) of the window, or positions of frame_list
  const int* frame_list;     // null, or device list: lane frame f reads window frame frame_list[frame0 + f] - list_base
  int list_base;
  int imgx, imgy;            // ROI origin in the frame (full-frame coordinates)
  int roi_w, roi_h;          // staged ROI size (always the FULL logo rectangle, also for field logos)
  int src_mode;              // 0: DeintY, 1: CopyY
  int src_off, src_stride;   // view of the staged ROI this logo reads (field logos: off = 0|w, stride = 2w)
  LogoDev logo;              // logo.w x logo.h = evaluated size (h/2 for field logos)
  float maxv;
  int nfades;
  float fades[kMaxFades];
  float* scores;             // [nframes][nfades][countPad]
  int use_tma;               // 1: the ROI is fetched by TMA through roi_map (box roi_box_w x roi_h x 1 elements)
  int roi_box_w;             // row pitch of the staged raw ROI in ELEMENTS (multiple of 16 bytes)
  int roi_box_x;             // x of the box in the frame: imgx rounded DOWN to 16 bytes (TMA faults on unaligned starts)
  int ab_smem;               // 1: logo planes A,B are staged in shared memory; 0: read through L1 (large logos)
  int pair_fades;            // 1: two fade levels per pass (needs a second work image in shared memory)
  CUtensorMap roi_map;       // 3-D (x, y, frame) view of the Y plane as addressed with `pitch`
};

// Shared-memory layout of logo_scores_kernel (floats unless noted):
//   A[npx] B[npx]      logo planes, loaded once per CTA
//   src[roi_n]         the frame's ROI as float (DeintY or CopyY)
//   work[npx + 8] x2   logo-removed images of the current PAIR of fade levels
//   raw[2][box_w*roi_h] pixel_t: double-buffered ROI samples, filled by TMA one frame ahead (128-byte aligned)
__host__ __device__ inline size_t logo_scores_smem_bytes(int roi_n, int npx, int raw_bytes_one, int ab_smem, int pair_fades) {
  return ((size_t)(ab_smem ? 2 : 0) * ((npx + 3) & ~3) + ((roi_n + 3) & ~3) +
          (size_t)(pair_fades ? 2 : 1) * (((size_t)npx + 8 + 3) & ~(size_t)3)) * sizeof(float) +
         128 + 2 * (((size_t)raw_bytes_one + 127) & ~(size_t)127);
}

// CW > 0: logo width AND staged ROI width are the compile-time constant CW (the common 64-pixel logos): every 5x5 window
// address becomes an immediate and the index walkers lose their divisions (about half of the kernel's instructions were
// integer bookkeeping, profiles/r02h_logo_scores_kernel_ncu_full_summary.txt).  CW = 0: both widths at run time.
template <typename pixel_t, int PXT, int CW = 0, int CH = 0>        // CH > 0: logo height AND ROI height known as well (loops unroll)
__global__ void __launch_bounds__(kEvalThreads, 1) logo_scores_kernel(const __grid_constant__ EvalJob job) {
  extern __shared__ float smem_f[];
  __shared__ __align__(8) uint64_t roi_bar[2];
  const int tid = threadIdx.x;
  const LogoDev& lg = job.logo;
  const int w = CW ? CW : lg.w, npx = w * (CH ? CH : lg.h);
  const int roi_w = CW ? CW : job.roi_w;
  const int roi_h = CH ? CH : job.roi_h;
  const int roi_n = roi_w * roi_h;
  float* src = smem_f + (job.ab_smem ? 2 * ((npx + 3) & ~3) : 0);
  const float* sA = job.ab_smem ? smem_f : lg.A;                         // large logos read A,B through L1 instead
  const float* sB = job.ab_smem ? smem_f + ((npx + 3) & ~3) : lg.B;
  float* work = src + ((roi_n + 3) & ~3);
  float* work2 = work + ((npx + 8 + 3) & ~3);                            // second fade level of a pair (pair_fades only)
  uint8_t* raw_base = reinterpret_cast<uint8_t*>(work + (size_t)(job.pair_fades ? 2 : 1) * ((npx + 8 + 3) & ~3));
  raw_base += (128u - (smem_u32(raw_base) & 127u)) & 127u;
  const int raw_pitch = job.roi_box_w;                                   // elements per staged ROI row
  const uint32_t raw_bytes = (uint32_t)raw_pitch * roi_h * sizeof(pixel_t);
  const uint32_t raw_stride = (raw_bytes + 127u) & ~127u;

  // ---- one-time: logo planes to smem, adopt feature pixels, pull their taps into registers ----
  if (job.ab_smem)
    for (int i = tid; i < npx; i += kEvalThreads) { smem_f[i] = lg.A[i]; smem_f[((npx + 3) & ~3) + i] = lg.B[i]; }
  float taps[PXT][25];
  int pxy[PXT];
  int cidx[PXT];
#pragma unroll
  for (int p = 0; p < PXT; ++p) {
    const int c = (blockIdx.x * PXT + p) * kEvalThreads + tid;
    cidx[p] = c;
    if (c < lg.count) {
      const uint32_t v = lg.pix[c];
      pxy[p] = (int)((v & 0xFFFFu) - 2) + (int)((v >> 16) - 2) * w;     // top-left of the 5x5 window
#pragma unroll
      for (int t = 0; t < 25; ++t) taps[p][t] = lg.tapsT[(size_t)t * lg.countPad + c];
    } else {
      pxy[p] = 0;
#pragma unroll
      for (int t = 0; t < 25; ++t) taps[p][t] = 0.0f;
    }
  }
  // per-thread walk over image indices i = tid, tid+512, ... without divisions: (x,y) advance by (dx,dy)
  const int roi_dx = kEvalThreads % roi_w, roi_dy = kEvalThreads / roi_w;
  const int roi_y0 = tid / roi_w, roi_x0 = tid - roi_y0 * roi_w;
  const int lg_dx = kEvalThreads % w, lg_dy = kEvalThreads / w;
  const int lg_y0 = tid / w, lg_x0 = tid - lg_y0 * w;

  if (job.use_tma && tid == 0) {
    mbar_init(&roi_bar[0], 1); mbar_init(&roi_bar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto frame_at = [&](int f) { return job.frame_list ? job.frame_list[job.frame0 + f] - job.list_base : job.frame0 + f; };
  auto issue_roi = [&](int f, int buf) {          // thread 0: TMA box (roi_box_w x roi_h) of frame f -> raw[buf]
    mbar_expect_tx(&roi_bar[buf], raw_bytes);
    tma_load_3d(raw_base + buf * raw_stride, &job.roi_map, &roi_bar[buf], job.roi_box_x, job.imgy, frame_at(f));
  };
  int f = blockIdx.y;
  if (job.use_tma && tid == 0 && f < job.nframes) issue_roi(f, 0);
  for (int it = 0; f < job.nframes; f += gridDim.y, ++it) {
    const pixel_t* raw;
    if (job.use_tma) {
      // the other buffer was last read in the previous iteration, before several block barriers: free to refill
      if (tid == 0 && f + (int)gridDim.y < job.nframes) issue_roi(f + gridDim.y, (it + 1) & 1);
      mbar_wait(&roi_bar[it & 1], (uint32_t)(it >> 1) & 1u);
      raw = reinterpret_cast<const pixel_t*>(raw_base + (it & 1) * raw_stride) + (job.imgx - job.roi_box_x);
    } else {                                       // layouts TMA cannot describe: plain coalesced element loads
      const pixel_t* fr = reinterpret_cast<const pixel_t*>(
          reinterpret_cast<const uint8_t*>(job.ybase) + (long long)frame_at(f) * job.frame_stride);
      const pixel_t* roi = fr + job.imgx + (long long)job.imgy * job.pitch;
      pixel_t* dst = reinterpret_cast<pixel_t*>(raw_base);
      int x = roi_x0, y = roi_y0;
      for (int i = tid; i < roi_n; i += kEvalThreads) {
        dst[x + y * raw_pitch] = roi[x + (long long)y * job.pitch];
        x += roi_dx; y += roi_dy; if (x >= roi_w) { x -= roi_w; ++y; }
      }
      __syncthreads();
      raw = dst;
    }
    // ---- ROI as float: DeintY (:763-780) or CopyY (:782-790) ----
    {
      int x = roi_x0, y = roi_y0;
      for (int i = tid; i < roi_n; i += kEvalThreads) {
        const pixel_t* rp = raw + x + y * raw_pitch;
        float v;
        if (job.src_mode == 0 && y > 0 && y < roi_h - 1) {
          const int a = rp[-raw_pitch], b = rp[0], c = rp[raw_pitch];
          v = (float)(a + 2 * b + c + 2) / 4.0f;       // exact: integer < 2^24, division by 4
        } else {
          v = (float)rp[0];
        }
        src[i] = v;
        x += roi_dx; y += roi_dy; if (x >= roi_w) { x -= roi_w; ++y; }
      }
    }
    __syncthreads();

    // Fade levels are processed in PAIRS: both logo-removed images are built in one phase and every thread then scores
    // its pixels on both (6 independent dependency chains instead of 3, half as many block barriers per frame).
    const int fstep = job.pair_fades ? 2 : 1;
    for (int fi = 0; fi < job.nfades; fi += fstep) {
      const int nf2 = min(fstep, job.nfades - fi);
      const float fade0 = job.fades[fi], fade1 = job.fades[fi + nf2 - 1];
      const float omf0 = AMTK_FSUB(1.0f, fade0), omf1 = AMTK_FSUB(1.0f, fade1);
      // ---- logo removal at these fade levels (LogoScan.hpp:241-251) ----
      {
        int x = lg_x0, y = lg_y0;
        for (int i = tid; i < npx; i += kEvalThreads) {
          const float srcv = src[job.src_off + x + y * job.src_stride];
          const float av = sA[i], bv = sB[i];
          work[i] = remove_logo(srcv, av, bv, job.maxv, fade0, omf0);
          if (nf2 == 2) work2[i] = remove_logo(srcv, av, bv, job.maxv, fade1, omf1);
          x += lg_dx; y += lg_dy; if (x >= w) { x -= w; ++y; }
        }
      }
      __syncthreads();
      // ---- per-feature score (LogoScan.hpp:298-308) ----
      float* out0 = job.scores + ((size_t)f * job.nfades + fi) * lg.countPad;
      float sum[2][PXT]; int bin[2][PXT];
#pragma unroll
      for (int p = 0; p < PXT; ++p) {
        const float* wp = work + pxy[p];
        float avg;
        sum[0][p] = corr5x5_tree(taps[p], [&](int dy, int dx) { return wp[dy * w + dx]; }, &avg);
        bin[0][p] = scale_bin(avg);
        if (nf2 == 2) {
          const float* wq = work2 + pxy[p];
          sum[1][p] = corr5x5_tree(taps[p], [&](int dy, int dx) { return wq[dy * w + dx]; }, &avg);
          bin[1][p] = scale_bin(avg);
        }
      }
#pragma unroll
      for (int p = 0; p < PXT; ++p) {
        if (cidx[p] < lg.count) {
          const float2* sc = lg.scales + (size_t)cidx[p] * 32;
          const float2 s0 = __ldg(sc + bin[0][p]);
          out0[cidx[p]] = pixel_score(sum[0][p], s0.x, s0.y);
          if (nf2 == 2) {
            const float2 s1 = __ldg(sc + bin[1][p]);
            out0[lg.countPad + cidx[p]] = pixel_score(sum[1][p], s1.x, s1.y);
          }
        }
      }
      __syncthreads();     // `work`/`work2` are rewritten by the next pair / `src` by the next frame
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// scan_item: LogoFrame::ScanFrame scores (DeintY source, ROI = the logo rectangle, fades {0, 1}) of a few frames, run
// as a work item of the band-form comb kernel (comb_stream.cuh) between its streaming items.  The fused step used to run
// logo_scores_kernel + logo_sum_bulk_kernel after the comb kernel (6 % of the step on H100); a logo kernel of its own
// cannot run beside the comb kernel there (three comb CTAs take 61 440 of an SM's 65 536 registers).  The comb CTAs have
// issue slots to spare (load bound), so they take the logo work themselves.  The arithmetic is the exact_math.h code of
// logo_scores_kernel, so the bits are the same; the per-pixel scores of the item's frames stay in shared memory and 2F
// threads add them in the reference's order (LogoScan.hpp:310), as logo_sum_bulk_kernel does.
// The item runs while the memory system is saturated by the streaming items, so every global load waits long, and the
// comb kernel leaves the item few registers to keep loads in flight with: the ROI rows (in 16-byte pieces: the band
// form's layouts are 16-byte aligned) and the logo planes A, B (into the two work images, which are then rewritten in
// place) arrive by cp.async, all in flight at once; each feature pixel's 25 taps are read once for both fades; the
// score-scale lookups, which depend on the correlation, are consumed one pixel later; the ordered sums read their rows one
// 128-byte line ahead.  F comes from the ring of the band form that runs (scan_item_frames), up to kScanItemMaxFrames.
// Shared memory (the comb ring's slots, all free at an item boundary), floats unless noted:
//   work0[npx + 8] work1[npx + 8]   logo-removed images at fade 0 and fade 1
//   sc[F][2][countPad + 4]          per-pixel scores (row pitch 4 banks apart: the 2F summing lanes do not conflict)
//   raw[h][rpitch] u8               the frame's ROI rows from imgx rounded down to 16 bytes, rpitch <= (w + 30) & ~15
// ---------------------------------------------------------------------------------------------------------
struct ScanItemJob {
  const uint8_t* ybase;      // Y plane of frame 0 of the device window (8-bit samples, 16-byte aligned)
  long long frame_stride;    // bytes (multiple of 16)
  int pitch;                 // bytes (multiple of 16)
  int imgx, imgy;            // the logo rectangle's origin in the frame
  LogoDev logo;
  float maxv;
  int frames;                // F: frames per item (score rows kept in shared memory)
  float* scores;             // [frame - out_frame0][2] (one logo, fades 0 and 1)
};
constexpr int kScanItemMaxFrames = 16;
__host__ __device__ inline size_t scan_item_smem_bytes(int w, int h, int countPad, int frames) {
  return (2 * (((size_t)w * h + 8 + 3) & ~(size_t)3) + (size_t)frames * 2 * (countPad + 4)) * sizeof(float) + (size_t)((w + 30) & ~15) * h;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(src) : "memory");
}

template <int NT>
__device__ __forceinline__ void scan_item(const ScanItemJob& j, int fbegin, int fend, int out_frame0, uint8_t* smem) {
  const LogoDev& lg = j.logo;
  const int tid = threadIdx.x, w = lg.w, h = lg.h, npx = w * h, count = lg.count, spitch = lg.countPad + 4;
  float* work0 = reinterpret_cast<float*>(smem);
  float* work1 = work0 + ((npx + 8 + 3) & ~3);
  float* sc = work1 + ((npx + 8 + 3) & ~3);
  uint8_t* raw = reinterpret_cast<uint8_t*>(sc + (size_t)j.frames * 2 * spitch);     // 16-byte aligned
  const int xa = j.imgx & ~15, xo = j.imgx - xa;             // ROI rows are loaded from xa, in 16-byte pieces
  const int rpitch = (xo + w + 15) & ~15, cpr = rpitch >> 4, nchunks = cpr * h;
  const float omf0 = AMTK_FSUB(1.0f, 0.0f), omf1 = AMTK_FSUB(1.0f, 1.0f);
  // per-thread walk over pixel indices i = tid, tid+NT, ... without divisions: (x,y) advance by (dx,dy)
  const int dx = NT % w, dy = NT / w, y0 = tid / w, x0 = tid - y0 * w;
  for (int f = fbegin; f < fend; ++f) {
    __syncthreads();     // the work images of the previous frame are no longer read
    const uint8_t* roi = j.ybase + (long long)f * j.frame_stride + xa + (long long)j.imgy * j.pitch;
    for (int k = tid; k < nchunks; k += NT) {
      const int y = k / cpr;
      cp_async16(raw + 16 * k, roi + (long long)y * j.pitch + 16 * (k - y * cpr));
    }
    for (int q = tid; q < (npx >> 2); q += NT) { cp_async16(work0 + 4 * q, lg.A + 4 * q); cp_async16(work1 + 4 * q, lg.B + 4 * q); }
    for (int i = (npx & ~3) + tid; i < npx; i += NT) { cp_async4(work0 + i, lg.A + i); cp_async4(work1 + i, lg.B + i); }
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
    {
      int x = x0, y = y0;
      for (int i = tid; i < npx; i += NT) {
        const uint8_t* rp = raw + y * rpitch + xo + x;
        float v;                                             // DeintY (:763-780)
        if (y > 0 && y < h - 1) { const int a = rp[-rpitch], b = rp[0], c = rp[rpitch]; v = (float)(a + 2 * b + c + 2) / 4.0f; }
        else v = (float)rp[0];
        const float av = work0[i], bv = work1[i];            // A, B -> the logo-removed images, in place
        work0[i] = remove_logo(v, av, bv, j.maxv, 0.0f, omf0);
        work1[i] = remove_logo(v, av, bv, j.maxv, 1.0f, omf1);
        x += dx; y += dy; if (x >= w) { x -= w; ++y; }
      }
    }
    __syncthreads();
    // per-feature score (LogoScan.hpp:298-308), both fades from one read of the taps; the scale lookups of a pixel are
    // consumed after the next pixel's correlation
    float* s0 = sc + (size_t)(f - fbegin) * 2 * spitch;
    float2 kp0 = make_float2(0.0f, 0.0f), kp1 = kp0;
    int cp = -1;
#pragma unroll 1
    for (int c = tid; c < count; c += NT) {
      const uint32_t pv = __ldg(lg.pix + c);
      float taps[25];
#pragma unroll
      for (int t = 0; t < 25; ++t) taps[t] = __ldg(lg.tapsT + (size_t)t * lg.countPad + c);
      const int o = (int)((pv & 0xFFFFu) - 2) + (int)((pv >> 16) - 2) * w;
      float avg0, avg1;
      s0[c] = corr5x5_tree(taps, [&](int ry, int rx) { return work0[o + ry * w + rx]; }, &avg0);
      s0[spitch + c] = corr5x5_tree(taps, [&](int ry, int rx) { return work1[o + ry * w + rx]; }, &avg1);
      const float2 kn0 = __ldg(lg.scales + (size_t)c * 32 + scale_bin(avg0)), kn1 = __ldg(lg.scales + (size_t)c * 32 + scale_bin(avg1));
      if (cp >= 0) { s0[cp] = pixel_score(s0[cp], kp0.x, kp0.y); s0[spitch + cp] = pixel_score(s0[spitch + cp], kp1.x, kp1.y); }
      kp0 = kn0; kp1 = kn1; cp = c;
    }
    if (cp >= 0) { s0[cp] = pixel_score(s0[cp], kp0.x, kp0.y); s0[spitch + cp] = pixel_score(s0[spitch + cp], kp1.x, kp1.y); }
  }
  __syncthreads();
  // ordered sums (:252-254,310): thread t adds the score row of frame fbegin + t/2, fade t%2, its loads one 128-byte line
  // ahead of the dependent adds (the row has countPad >= count floats: the reads of the last line stay inside it)
  if (tid < 2 * (fend - fbegin)) {
    const float4* row = reinterpret_cast<const float4*>(sc + (size_t)tid * spitch);
    const int nlines = lg.countPad >> 5;
    float4 q[8];             // the next 8 float4 of the row: each one consumed is replaced by the one a line further on
#pragma unroll
    for (int k = 0; k < 8; ++k) q[k] = row[k];
    float r = 0.0f;
    int c = 0;
#pragma unroll 1
    for (int l = 0; l < nlines; ++l) {
      const bool more = l + 1 < nlines;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float4 v = q[k];
        if (more) q[k] = row[(l + 1) * 8 + k];
        if (c + 4 <= count) {
          r = AMTK_FADD(r, v.x); r = AMTK_FADD(r, v.y); r = AMTK_FADD(r, v.z); r = AMTK_FADD(r, v.w);
        } else {
          if (c < count) r = AMTK_FADD(r, v.x);
          if (c + 1 < count) r = AMTK_FADD(r, v.y);
          if (c + 2 < count) r = AMTK_FADD(r, v.z);
        }
        c += 4;
      }
    }
    j.scores[(size_t)(fbegin + (tid >> 1) - out_frame0) * 2 + (tid & 1)] = AMTK_FDIV(r, lg.blackScore);
  }
}

// One thread per (frame, fade): ordered float sum of the pixel scores, divided by blackScore (:252-254,310).
// out index = row*out_frame_stride + out_off + fade*out_fade_stride, row = out_rows[frame] (out_rows may be null: row =
// frame); take_abs for AMTAnalyzeLogo (:1152-1154).
// The chain of ~1.3k dependent FADDs is inherent (the order is the reference's); the loads are software-pipelined
// one 128-byte line ahead so the chain never waits on memory.  32-thread blocks spread the chains over all SMs.
constexpr int kSumThreads = 32;
__global__ void __launch_bounds__(kSumThreads) logo_sum_kernel(const float* __restrict__ scores, int count, int countPad,
                                                               int nframes, int nfades, float blackScore, int take_abs,
                                                               float* __restrict__ out, int out_frame_stride, int out_off,
                                                               int out_fade_stride, const int* __restrict__ out_rows) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nframes * nfades) return;
  const float4* row = reinterpret_cast<const float4*>(scores + (size_t)t * countPad);   // countPad % 32 == 0
  const int nlines = countPad >> 5;            // 32 floats (8 float4) per line; padding reads stay inside the row
  float4 cur[8], nxt[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) cur[k] = row[k];
  float r = 0.0f;
  int c = 0;
  for (int l = 0; l < nlines; ++l) {
    if (l + 1 < nlines) {
#pragma unroll
      for (int k = 0; k < 8; ++k) nxt[k] = row[(l + 1) * 8 + k];
    }
    if (c + 32 <= count) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        r = AMTK_FADD(r, cur[k].x); r = AMTK_FADD(r, cur[k].y); r = AMTK_FADD(r, cur[k].z); r = AMTK_FADD(r, cur[k].w);
      }
      c += 32;
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (c < count) r = AMTK_FADD(r, cur[k].x); ++c;
        if (c < count) r = AMTK_FADD(r, cur[k].y); ++c;
        if (c < count) r = AMTK_FADD(r, cur[k].z); ++c;
        if (c < count) r = AMTK_FADD(r, cur[k].w); ++c;
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) cur[k] = nxt[k];
  }
  float v = AMTK_FDIV(r, blackScore);
  if (take_abs) v = fabsf(v);
  const int f = t / nfades, fi = t - f * nfades;
  out[(size_t)(out_rows ? out_rows[f] : f) * out_frame_stride + out_off + (size_t)fi * out_fade_stride] = v;
}

// Same reduction with the 32 score rows of a warp brought into shared memory by 32 bulk copies (all in flight at
// once, ~168 KB for a 64x64 logo), after which each lane walks its row with conflict-free LDS.128 (row pitch
// countPad+4 floats = 4 banks apart per lane).  The dependent-add chain then runs at ALU latency instead of waiting
// on a global load every 128 bytes.
__global__ void __launch_bounds__(32) logo_sum_bulk_kernel(const float* __restrict__ scores, int count, int countPad,
                                                            int nframes, int nfades, float blackScore, int take_abs,
                                                            float* __restrict__ out, int out_frame_stride, int out_off,
                                                            int out_fade_stride, const int* __restrict__ out_rows) {
  extern __shared__ __align__(16) float sum_rows[];
  __shared__ __align__(8) uint64_t bar;
  const int lane = threadIdx.x, total = nframes * nfades;
  const int t0 = blockIdx.x * 32, nrows = min(32, total - t0);
  const int pitch = countPad + 4;
  const uint32_t row_bytes = (uint32_t)countPad * sizeof(float);
  if (lane == 0) { mbar_init(&bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncwarp();
  if (lane == 0) mbar_expect_tx(&bar, row_bytes * (uint32_t)nrows);
  __syncwarp();
  if (lane < nrows) bulk_load_1d(sum_rows + (size_t)lane * pitch, scores + (size_t)(t0 + lane) * countPad, row_bytes, &bar);
  mbar_wait(&bar, 0);
  if (lane >= nrows) return;
  const float4* row = reinterpret_cast<const float4*>(sum_rows + (size_t)lane * pitch);
  float r = 0.0f;
  const int n4 = count >> 2;
#pragma unroll 8
  for (int i = 0; i < n4; ++i) {
    const float4 v = row[i];
    r = AMTK_FADD(r, v.x); r = AMTK_FADD(r, v.y); r = AMTK_FADD(r, v.z); r = AMTK_FADD(r, v.w);
  }
  const float* tail = sum_rows + (size_t)lane * pitch;
  for (int c = n4 << 2; c < count; ++c) r = AMTK_FADD(r, tail[c]);
  float v = AMTK_FDIV(r, blackScore);
  if (take_abs) v = fabsf(v);
  const int t = t0 + lane;
  const int f = t / nfades, fi = t - f * nfades;
  out[(size_t)(out_rows ? out_rows[f] : f) * out_frame_stride + out_off + (size_t)fi * out_fade_stride] = v;
}

__global__ void fill_pairs_kernel(float* out, int nframes, int stride, int off, float v0, float v1) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < nframes) { out[(size_t)f * stride + off] = v0; out[(size_t)f * stride + off + 1] = v1; }
}

}  // namespace amtk
