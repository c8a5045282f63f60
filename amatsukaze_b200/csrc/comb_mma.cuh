// comb_mma.cuh -- field-difference / combing metric, streaming pass, tensor-core variant (8-bit samples).
//
// Why tensor cores in an HBM-streaming kernel: in the SIMT kernels (comb_kernels.cuh, comb_stream.cuh) the 5-tap vertical
// stencil costs ~6 issue slots per pixel (u8 -> fp16 conversion 0.5, stencil 2.0, thresholds 1.0, mask sums 0.5,
// inter-frame difference 1.25, loads/overhead), so the ALU pipe (HSET2/PRMT/LOP3/IADD3) rather than HBM can set the pace.
// The stencil is a product with a banded Toeplitz matrix -- exact in u8 x u8 -> s32 -- and the tensor pipe is otherwise
// idle, so here it does the stencil:
//
//     D[x][n] = sum_r  tile[r][x] * band[r][n]          M = 128 pixels of a tile row, K = 64 box rows, N = 128
//        n in [0,60):    pos(y0+n) = p[y-2] + 4 p[y] + p[y+2]        (band entries 1, 4, 1)
//        n in [64,124):  neg(y0+n) = 3 (p[y-1] + p[y+1])             (band entries 3, 3)
//
// as Hopper warpgroup MMAs: wgmma.mma_async m64n128k32 .s32.u8.u8, two M halves x two K steps per tile-frame, issued by
// the four consumer warps (one warpgroup).  8-bit wgmma reads its shared-memory operands K-major only, and the TMA-staged
// tile is row-major (x contiguous), so the tile is the A operand from registers: every thread gathers the bytes of its
// fragment (four box rows of one pixel column per register) from the swizzled slot.  The band matrix is the B operand,
// K-major in shared memory, built once per CTA.  Both halves are < 2048, so their low 16 bits are exact fp16 bit patterns
// (k * 2^-24): one PRMT packs the accumulators of rows y, y+1 (= the two fields) into a half2, and the rest is
//     r = HADD2(pos, -neg);  HSET2.GE(|r|, thS);  HSET2.GE(|r|, thL);  adds of the masks
// The inter-frame difference stays on the SIMT side (VABSDIFF4 + SWAR compare + IDP.4A on the raw bytes of the current
// and the previous slot).
//
// Same integer spec, same counters, bit-identical results (integer adds commute).  It is an opt-in experiment
// (AMTK_COMB_MMA=1|2), not the product path.  Every device-side wait has a watchdog (mm_wait): a protocol error fails the
// call, it cannot hang the GPU.
#pragma once
#include <cuda_fp16.h>
#include "amtk_internal.h"
#include "tma_utils.cuh"
#include "comb_stream.cuh"       // WsArgs / WsClass / CombSegment / bytes_ge

namespace amtk {

constexpr int kMmTW = 128;                       // tile width in bytes = MMA M (two m64 halves)
constexpr int kMmTH = 60;                        // output rows per tile
constexpr int kMmBoxH = 64;                      // + 2 halo rows above and below = MMA K (two k32 steps)
constexpr int kMmSlot = kMmTW * kMmBoxH;         // 8192 bytes
constexpr int kMmStages = 4;                     // previous frame, current frame, two frames in flight (power of two)
constexpr int kMmConsumerWarps = 4;              // = one warpgroup (warps 0..3)
constexpr int kMmThreads = 32 * (kMmConsumerWarps + 1);   // + the producer warp
constexpr int kMmBandBytes = 128 * kMmBoxH;      // N x K u8
constexpr int kMmSmemPerStream = kMmStages * kMmSlot;    // + kMmBandBytes + 1024 once per CTA (slack for the 1024-byte alignment the swizzle needs)
constexpr int kMmBandLBO = 2048, kMmBandSBO = 128;                   // band matrix: K-major, no swizzle, 8x16-byte core matrices

// ---- wgmma wrappers ---------------------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D (+)= A[registers] * B[smem desc], u8 x u8 -> s32, M64 N128 K32.  Fragment of thread (warp w, lane l) of the warpgroup:
// a[i] = A[16w + l/4 + 8(i&1)][16(i>>1) + 4(l&3) + 0..3] (lowest k in the low byte); d[4g + j] = D[16w + l/4 + 8(j>>1)][8g + 2(l&3) + (j&1)].
__device__ __forceinline__ void wg_mma_u8(uint32_t (&d)[64], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
      "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, "
      "%51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p;\n\t"
      "}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
        "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
        "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
        "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
        "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
        "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate)
      : "memory");
}

// wgmma shared-memory matrix descriptor (sm_90 format): start, leading / stride byte offsets, layout type in bits 62-63
// (0 = no swizzle)
__device__ __forceinline__ uint64_t mm_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}

// band[n][k], k = box row (global row y0 - 2 + k), n = output column of D
__device__ __forceinline__ uint32_t mm_band(int n, int k) {
  if (n < kMmTH) { const int d = k - n; return (d == 0 || d == 4) ? 1u : (d == 2 ? 4u : 0u); }
  if (n >= 64 && n < 64 + kMmTH) { const int d = k - (n - 64); return (d == 1 || d == 3) ? 3u : 0u; }
  return 0u;
}

// Roles: warps 0..3 = consumers (one warpgroup: A-fragment gathers, wgmma, thresholds; warp w holds pixel columns
// 16w..16w+15 of each 64-column half of a tile, and 15 of the 60 strip rows of the inter-frame difference); warp 4 =
// producer (TMA loads, counter flush).  With AMTK_COMB_MMA=2 a CTA streams TWO tiles at once (work items come in pairs with
// the same frame range), so the fixed per-step costs (barrier waits, loop and ring bookkeeping) are paid once per two
// tile-frames.
// Ring protocol: full_bar[slot] completes when a load has landed; empty_bar[slot] completes when every consumer warp is
// done with the load in that slot (used as the current frame of step j and as the previous frame of step j+1) AND has
// published the counters of its frame.  The producer waits for the release of load j before it flushes frame j and before
// it refills that slot, once per load and in load order, so no parity wait can fall two phases behind.
template <int NS>
__global__ void __launch_bounds__(kMmThreads, 2) comb_mma_kernel(const __grid_constant__ WsArgs a) {
  constexpr int kStageBytes = NS * kMmSlot;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMmStages];
  __shared__ __align__(8) uint64_t empty_bar[kMmStages];
  __shared__ int item_s;
  __shared__ uint32_t red[4][16];                            // [step & 3][stream * 8 + counter]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool producer = warp == kMmConsumerWarps;
  uint8_t* slots = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* band = slots + kMmStages * kStageBytes;

  // ---- one-time setup: band matrix, barriers ----
  for (int o = tid * 4; o < kMmBandBytes; o += kMmThreads * 4) {       // 4 consecutive k of one row n per store
    const int kc = o / kMmBandLBO, rem = o - kc * kMmBandLBO;
    const int ng = rem / kMmBandSBO, i = (rem % kMmBandSBO) >> 4, kk = rem & 15;
    const int n = ng * 8 + i, k = kc * 16 + kk;
    *reinterpret_cast<uint32_t*>(band + o) = mm_band(n, k) | (mm_band(n, k + 1) << 8) | (mm_band(n, k + 2) << 16) | (mm_band(n, k + 3) << 24);
  }
  if (tid < 64) red[tid >> 4][tid & 15] = 0u;
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kMmStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kMmConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");          // band matrix: generic-proxy stores -> async-proxy (wgmma) reads
  __syncthreads();
  int* const dbg = a.queue + 16;                             // watchdog record (64 bytes after the queue counter, zeroed per launch)
  const uint64_t descB0 = mm_desc(smem_u32(band), kMmBandLBO, kMmBandSBO);
  const uint64_t descB1 = mm_desc(smem_u32(band) + 2 * kMmBandLBO, kMmBandLBO, kMmBandSBO);

  // inter-frame difference: consumer thread t owns strip (t & 7) of the box rows b0, b0+8, b0+16, b0+24 with
  // b0 = 2 + (t >> 3) for t < 64 and 34 + ((t - 64) >> 3) for the rest (rows 2..61 = the 60 tile rows; the fourth row of
  // the last four row groups would be 62..65 and is skipped).  Rows 8 apart share (row & 7), so the swizzled 16-byte chunk
  // (chunk index ^ (row & 7)) is the same in all four: one address + immediates.  They also share the row parity = the field.
  const int mv_b0 = (tid < 64 ? 2 : 34) + ((tid & 63) >> 3);
  const int mv_toff = mv_b0 * kMmTW + (((tid & 7) ^ (mv_b0 & 7)) << 4);
  const bool mv_row3 = mv_b0 + 24 <= kMmTH + 1;
  const int mv_shift = (mv_b0 & 1) ? 16 : 0;                 // tile row = box row - 2: same parity; odd rows count in the high half
  // publishing lane i < 6 of a consumer warp owns counter i of counts[]' [field][move, shima, lshima] layout
  const uint32_t pub_selM = (lane == 0 || lane == 3) ? 0xFFFFFFFFu : 0u, pub_selS = (lane == 1 || lane == 4) ? 0xFFFFFFFFu : 0u;
  const uint32_t pub_selL = (lane == 2 || lane == 5) ? 0xFFFFFFFFu : 0u;
  const int pub_shift = (lane >= 3 && lane < 6) ? 16 : 0;
  uint32_t* const pub_red = &red[0][lane & 7];

  uint32_t gload = 0;          // loads consumed so far (ring position)
  int* pend_crow = nullptr;    // producer: counters of the last frame of the previous item still sit in red[]
  int pend_k = 0;
  for (;;) {
    if (tid == kMmConsumerWarps * 32) item_s = atomicAdd(a.queue, 1);
    __syncthreads();
    // Every consumer has published the last frame of the previous item before it reached this barrier: flush it now.
    if (producer && pend_k > 0) {
      if (lane < 8 * NS) {
        const uint32_t v = red[pend_k & 3][lane];
        red[pend_k & 3][lane] = 0u;
        if (pend_crow && v) atomicAdd(pend_crow + (size_t)pend_k * 12, (int)v);
      }
      pend_k = 0;
    }
    // warp-uniform by construction; the reduction tells the compiler so (uniform registers for all the bookkeeping)
    const int pair = (int)__reduce_max_sync(0xFFFFFFFFu, (unsigned)item_s);
    if (NS * pair >= a.nitems) break;
    int tileS[NS], fb = 0, fe = 0;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const CombSegment seg = a.segs[NS * pair + s];
      tileS[s] = (int)__reduce_max_sync(0xFFFFFFFFu, (unsigned)(seg.tile + 0x40000000)) - 0x40000000;   // < 0: filler stream, results dropped
      if (s == 0) { fb = (int)__reduce_max_sync(0xFFFFFFFFu, (unsigned)seg.fbegin); fe = (int)__reduce_max_sync(0xFFFFFFFFu, (unsigned)seg.fend); }
    }
    const int nf = fe - fb;
    const int nloads = nf + 1;                               // L_0 = previous frame, L_k = frame fb+k-1
    const int fprev = fb > 0 ? fb - 1 : fb;
    int ciS[NS], txS[NS], y0S[NS]; bool dropS[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      dropS[s] = tileS[s] < 0;
      const int tile = dropS[s] ? ~tileS[s] : tileS[s];
      int ci = 0;
#pragma unroll
      for (int k = 1; k < kWsMaxClasses; ++k) if (k < a.nclasses && tile >= a.cl[k].tile0) ci = k;
      const int lt = tile - a.cl[ci].tile0;
      const int ty = lt / a.cl[ci].tilesX;
      ciS[s] = ci; txS[s] = lt - ty * a.cl[ci].tilesX; y0S[s] = ty * kMmTH;
    }

    if (producer) {
      // =========================== producer warp ===========================
      auto wait_release = [&](uint32_t gl) {                 // every consumer warp is done with load gl
        mm_wait(&empty_bar[gl & (kMmStages - 1)], (gl / kMmStages) & 1u, dbg, 2, (int)gl, true);
      };
      auto issue_load = [&](int j) {                         // lane 0 only: both tiles of load j into one stage
        const uint32_t gl = gload + (uint32_t)j;
        const int st = (int)(gl & (kMmStages - 1));
        const int fr = (j == 0) ? fprev : fb + j - 1;
        mbar_expect_tx(&full_bar[st], kStageBytes);
#pragma unroll
        for (int s = 0; s < NS; ++s)
          tma_load_3d(slots + st * kStageBytes + s * kMmSlot, &a.map[a.cl[ciS[s]].map], &full_bar[st], txS[s] * kMmTW, y0S[s] - 2, fr);
      };
      const int fl_s = lane >> 3, fl_i = lane & 7;           // flush lane = (stream, counter)
      int* const crow = (lane < 8 * NS && fl_i < 6 && !dropS[fl_s & (NS - 1)])
                            ? a.counts + a.cl[ciS[fl_s & (NS - 1)]].cls * 6 + fl_i + ((long long)fb - 1 - a.out_frame0) * 12 : nullptr;
      auto flush = [&](int k) {                              // counters of frame k: shared -> global, slot cleared for reuse
        if (lane < 8 * NS) {
          const uint32_t v = red[k & 3][lane];
          red[k & 3][lane] = 0u;
          if (crow && v) atomicAdd(crow + (size_t)k * 12, (int)v);
        }
      };
      if (gload > 0) wait_release(gload - 1u);               // the last load of the previous item (every earlier one was waited for there)
      if (lane == 0) {
        const int pro = nloads < kMmStages ? nloads : kMmStages;
        for (int j = 0; j < pro; ++j) issue_load(j);
      }
      __syncwarp();
      for (int k = 1; k <= nf; ++k) {
        wait_release(gload + (uint32_t)(k - 1));             // frame k-1 is published; the slot of load k-1 is free
        if (k > 1) flush(k - 1);                             // before the refill: frame k+3 reuses red[(k-1) & 3]
        if (lane == 0 && (k + kMmStages - 1) < nloads) issue_load(k + kMmStages - 1);
        __syncwarp();
      }
      pend_crow = crow; pend_k = nf;                         // frame nf is flushed after the next block barrier
    } else {
      // =========================== consumer warps ===========================
      // rows of a tile the spec excludes although the plain pass counts them: y < 2 and H-2 <= y < H+2 (rows >= H are
      // zero-filled by TMA, but the windows of H, H+1 still see the last two real rows).  Bit n = tile row n.
      unsigned long long fixS[NS];
      uint32_t kMS[NS], tSS[NS], tLS[NS];
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        const WsClass& C = a.cl[ciS[s]];
        unsigned long long fix = 0ull;
        if (y0S[s] == 0) fix |= 3ull;
        const int lo = max(C.H - 2 - y0S[s], 0), hi = min(C.H + 2 - y0S[s], kMmTH);
        if (hi > lo) fix |= ((1ull << hi) - 1ull) & ~((1ull << lo) - 1ull);
        fixS[s] = fix; kMS[s] = C.thM; tSS[s] = C.thS; tLS[s] = C.thL;
      }
      const bool any_fix = (fixS[0] | fixS[NS - 1]) != 0ull;
      const int q2 = 2 * (lane & 3);                         // accumulator columns of this thread: 8g + q2 + {0, 1}
      // A fragment: pixel column x = 64 mh + 16 warp + lane/4 (+ 8) sits in 16-byte chunk 4 mh + warp of its box row
      const int a_col = lane >> 2, a_k = 4 * (lane & 3);

      // inter-frame difference of load j against load j-1, one tile: packed hits, low half = even rows, high = odd rows
      auto move_tile = [&](const uint8_t* cur, const uint8_t* prv, uint32_t kM) -> uint32_t {
        uint32_t m = 0u;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (i == 3 && !mv_row3) break;
          const uint4 c4 = *reinterpret_cast<const uint4*>(cur + mv_toff + i * 8 * kMmTW);
          const uint4 p4 = *reinterpret_cast<const uint4*>(prv + mv_toff + i * 8 * kMmTW);
          m = __dp4a(bytes_ge(__vabsdiffu4(c4.x, p4.x), kM), 0x01010101u, m);
          m = __dp4a(bytes_ge(__vabsdiffu4(c4.y, p4.y), kM), 0x01010101u, m);
          m = __dp4a(bytes_ge(__vabsdiffu4(c4.z, p4.z), kM), 0x01010101u, m);
          m = __dp4a(bytes_ge(__vabsdiffu4(c4.w, p4.w), kM), 0x01010101u, m);
        }
        return (m >> 7) << mv_shift;                           // <= 64 hits per lane, in the half of its field
      };
      auto move_step = [&](int j, uint32_t (&pend)[NS]) {
        const uint32_t gl = gload + (uint32_t)j;
        const int st = (int)(gl & (kMmStages - 1)), sp = (int)((gl - 1) & (kMmStages - 1));
        mm_wait(&full_bar[st], (gl / kMmStages) & 1u, dbg, 4, j);
#pragma unroll
        for (int s = 0; s < NS; ++s)
          pend[s] = move_tile(slots + st * kStageBytes + s * kMmSlot, slots + sp * kStageBytes + s * kMmSlot, kMS[s]);
      };
      auto release = [&](int j) {                            // this warp is done with load j (and has published its frame)
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[(gload + (uint32_t)j) & (kMmStages - 1)]);
      };
      // A fragment of k step ks of M half mh: a[i] = box rows 32 ks + 16 (i >> 1) + a_k + 0..3 of pixel column
      // 64 mh + 16 warp + a_col + 8 (i & 1), gathered byte by byte from the 128-byte-swizzled slot
      auto load_a = [&](const uint8_t* tile, int mh, int ks, uint32_t (&af)[4]) {
        const int chunk = 4 * mh + warp;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint32_t v = 0u;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int kr = 32 * ks + 16 * (i >> 1) + a_k + j;
            v |= (uint32_t)tile[kr * kMmTW + ((chunk ^ (kr & 7)) << 4) + a_col + 8 * (i & 1)] << (8 * j);
          }
          af[i] = v;
        }
      };

      {                                                      // L_0: the frame before the first one of this item
        const int st = (int)(gload & (kMmStages - 1));
        mm_wait(&full_bar[st], (gload / kMmStages) & 1u, dbg, 5, 0);
      }
      uint32_t pendM[NS];
      move_step(1, pendM);
      release(0);
      uint32_t d[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) d[i] = 0u;
      for (int k = 1; k <= nf; ++k) {
        const uint8_t* stage = slots + ((gload + (uint32_t)k) & (kMmStages - 1)) * kStageBytes;   // full since move_step(k)
#pragma unroll
        for (int s = 0; s < NS; ++s) {
          const __half2 thS = *reinterpret_cast<const __half2*>(&tSS[s]);
          const __half2 thL = *reinterpret_cast<const __half2*>(&tLS[s]);
          __half2 aS[4], aL[4];
#pragma unroll
          for (int c = 0; c < 4; ++c) { aS[c] = __float2half2_rn(0.0f); aL[c] = __float2half2_rn(0.0f); }
#pragma unroll
          for (int mh = 0; mh < 2; ++mh) {
            uint32_t a0[4], a1[4];
            load_a(stage + s * kMmSlot, mh, 0, a0);
            load_a(stage + s * kMmSlot, mh, 1, a1);
            wg_fence();
            wg_mma_u8(d, a0, descB0, 0u);                    // box rows 0..31
            wg_mma_u8(d, a1, descB1, 1u);                    // box rows 32..63
            wg_commit();
            wg_wait0();
            // thresholds: pos of tile row n in d[4g + j], neg in d[32 + 4g + j] (g = n / 8); j = 0, 1 and 2, 3 are rows n,
            // n+1 of two pixel columns.  HSET2.BF writes 1.0 per hit; the hits are counted with HADD2 -- exact, <= 32 per half.
#pragma unroll
            for (int g = 0; g < 8; ++g) {
              uint32_t keep = 0xFFFFFFFFu;                   // edge tiles: the excluded rows contribute r = 0 < th
              if (any_fix) {
                const uint32_t b = (uint32_t)(fixS[s] >> (8 * g + q2)) & 3u;
                keep = ((b & 1u) ? 0u : 0x0000FFFFu) | ((b & 2u) ? 0u : 0xFFFF0000u);
              }
#pragma unroll
              for (int hr = 0; hr < 2; ++hr) {
                const uint32_t pos = __byte_perm(d[4 * g + 2 * hr], d[4 * g + 2 * hr + 1], 0x5410) & keep;
                const uint32_t neg = __byte_perm(d[32 + 4 * g + 2 * hr], d[32 + 4 * g + 2 * hr + 1], 0x5410) & keep;
                const __half2 r = __habs2(__hsub2(*reinterpret_cast<const __half2*>(&pos), *reinterpret_cast<const __half2*>(&neg)));
                const int c = (2 * g + hr) & 3;
                aS[c] = __hadd2(aS[c], __hge2(r, thS));
                aL[c] = __hadd2(aL[c], __hge2(r, thL));
              }
            }
          }
          // One multiply by 2^-24 turns the fp16 counts into their integer bit patterns (k * 2^-24 is the subnormal with
          // bits k): low half = even rows (top field), high half = odd rows.
          const uint32_t one_ulp = 0x00010001u;
          const __half2 ulp = *reinterpret_cast<const __half2*>(&one_ulp);
          const __half2 sS = __hmul2(__hadd2(__hadd2(aS[0], aS[1]), __hadd2(aS[2], aS[3])), ulp);
          const __half2 sL = __hmul2(__hadd2(__hadd2(aL[0], aL[1]), __hadd2(aL[2], aL[3])), ulp);
          const uint32_t rS = __reduce_add_sync(0xFFFFFFFFu, *reinterpret_cast<const uint32_t*>(&sS));   // <= 32 x 32 per half
          const uint32_t rL = __reduce_add_sync(0xFFFFFFFFu, *reinterpret_cast<const uint32_t*>(&sL));
          const uint32_t rM = __reduce_add_sync(0xFFFFFFFFu, pendM[s]);
          const uint32_t v = (((rM & pub_selM) | (rS & pub_selS) | (rL & pub_selL)) >> pub_shift) & 0xFFFFu;
          if (lane < 6 && v) atomicAdd(pub_red + ((k & 3) * 16 + s * 8), v);
        }
        if (k < nf) move_step(k + 1, pendM);
        release(k);
      }
    }
    gload += (uint32_t)nloads;
  }
}

}  // namespace amtk
