// find_kernels.cuh -- per-pixel temporal sums of the luma plane for the logo finder (amtk_logo_find_*, DESIGN.md section
// 3.5): s1[y][x] += Y and s2[y][x] += Y*Y over every frame added, exact 64-bit integers.
//
// The work is the list of (tile, frame) pairs, tile-major: a tile is 256 bytes x 32 rows of the Y plane (256 8-bit or 128
// 16-bit samples wide).  Each CTA takes one contiguous share of that list, so every CTA streams the same number of tile
// frames whatever the tile count, and keeps its partial sums in registers while it stays on one tile.  It adds them to HBM
// with 64-bit atomic adds when the tile changes, at the end of its share and every kFindRunCap frames, so the totals are
// exact and do not depend on the order.  Thread t (of 512) owns the 16 bytes at column t & 15 of row t >> 4.
// Partials: 8-bit s1 and s2 in 32 bits (255 * 255 * 65536 < 2^32); 16-bit s1 in 32 bits, s2 in 64 bits.
#pragma once
#include <cuda.h>
#include <cstdint>
#include "tma_utils.cuh"

namespace amtk {

constexpr int kFindTileBytes = 256, kFindTileRows = 32, kFindThreads = 512;
constexpr int kFindStages = 8;                          // TMA ring: 8 x 8 KB in flight per CTA
constexpr int kFindRunCap = 65536;                      // frames a 32-bit partial may hold
constexpr int kFindSmemBytes = kFindStages * kFindTileBytes * kFindTileRows + 128;

struct FindArgs {
  const uint8_t* base;            // frame 0 of the window (plain-load kernel)
  long long frame_stride;
  int pitch;                      // bytes per row
  int width, height;              // luma size in samples
  int row_bytes;                  // width * bytes per sample
  int tiles_x, ntiles;
  int frame0, nframes;            // window frames [frame0, frame0 + nframes) (window numbering)
  unsigned long long* s1;         // [height][width]
  unsigned long long* s2;
};

template <int BPS> struct FindAcc;

template <> struct FindAcc<1> {
  uint32_t s1[16], s2[16];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int j = 0; j < 16; ++j) { s1[j] = 0; s2[j] = 0; }
  }
  __device__ __forceinline__ void add(const uint4& q) {
    const uint32_t w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const uint32_t v = (w[i] >> (8 * b)) & 0xFFu;
        s1[4 * i + b] += v;
        s2[4 * i + b] += v * v;
      }
  }
  __device__ __forceinline__ void flush(const FindArgs& a, int y, int xb) {
    if (y >= a.height) return;
    unsigned long long* p1 = a.s1 + (size_t)y * a.width;
    unsigned long long* p2 = a.s2 + (size_t)y * a.width;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int x = xb + j;
      if (x < a.width && s2[j]) { atomicAdd(p1 + x, (unsigned long long)s1[j]); atomicAdd(p2 + x, (unsigned long long)s2[j]); }
    }
  }
};

template <> struct FindAcc<2> {
  uint32_t s1[8]; unsigned long long s2[8];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int j = 0; j < 8; ++j) { s1[j] = 0; s2[j] = 0; }
  }
  __device__ __forceinline__ void add(const uint4& q) {
    const uint32_t w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t v = (w[i] >> (16 * h)) & 0xFFFFu;
        s1[2 * i + h] += v;
        s2[2 * i + h] += (unsigned long long)(v * v);      // < 2^32: exact in 32 bits, then widened
      }
  }
  __device__ __forceinline__ void flush(const FindArgs& a, int y, int xb) {
    if (y >= a.height) return;
    unsigned long long* p1 = a.s1 + (size_t)y * a.width;
    unsigned long long* p2 = a.s2 + (size_t)y * a.width;
    const int x0 = xb >> 1;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int x = x0 + j;
      if (x < a.width && s2[j]) { atomicAdd(p1 + x, (unsigned long long)s1[j]); atomicAdd(p2 + x, s2[j]); }
    }
  }
};

// Share of CTA b in the tile-major list of ntiles * nframes tile frames.
__device__ __forceinline__ void find_share(const FindArgs& a, long long* begin, long long* end) {
  const long long total = (long long)a.ntiles * a.nframes;
  *begin = total * blockIdx.x / gridDim.x;
  *end = total * (blockIdx.x + 1) / gridDim.x;
}

// Walks the CTA's share; load(p, tile, frame, q) fetches the thread's 16 bytes of list entry p, done(p) runs once they
// have been added.
template <int BPS, typename Load, typename Done>
__device__ __forceinline__ void find_walk(const FindArgs& a, long long begin, long long end, Load load, Done done) {
  const int col = (threadIdx.x & 15) * 16, row = threadIdx.x >> 4;
  FindAcc<BPS> acc; acc.zero();
  int tile = (int)(begin / a.nframes), f = (int)(begin % a.nframes), run = 0;
  for (long long p = begin; p < end; ++p) {
    uint4 q;
    load(p, tile, f, q);
    acc.add(q);
    done(p);
    ++run; ++f;
    const bool tile_ends = f == a.nframes;
    if (tile_ends || p + 1 == end || run == kFindRunCap) {
      const int ty = tile / a.tiles_x, tx = tile - ty * a.tiles_x;
      const int y = ty * kFindTileRows + row, xb = tx * kFindTileBytes + col;
      if (xb < a.row_bytes) acc.flush(a, y, xb);
      acc.zero(); run = 0;
      if (tile_ends) { ++tile; f = 0; }
    }
  }
}

// TMA form: base, pitch and frame stride multiples of 16 bytes.  map: 3-D uint8 map (row bytes, height, frames) with a
// 256 x 32 x 1 box; out-of-bounds bytes read as zeros and add nothing.
template <int BPS>
__global__ void __launch_bounds__(kFindThreads) find_sums_tma_kernel(const __grid_constant__ CUtensorMap map, FindArgs a) {
  extern __shared__ __align__(128) uint8_t find_smem[];
  // offset within the shared array (not a cast through an integer), so that the compiler keeps shared loads (LDS)
  uint8_t* ring = find_smem + ((128u - (smem_u32(find_smem) & 127u)) & 127u);
  __shared__ __align__(8) uint64_t full[kFindStages];
  constexpr uint32_t kBox = kFindTileBytes * kFindTileRows;
  long long begin, end;
  find_share(a, &begin, &end);
  if (begin >= end) return;
  // thread 0 issues the list entries in order: (itile, iframe) is the next one, advanced without a division
  int itile = (int)(begin / a.nframes), iframe = (int)(begin % a.nframes);
  auto issue = [&](int s) {
    const int ty = itile / a.tiles_x, tx = itile - ty * a.tiles_x;
    mbar_expect_tx(&full[s], kBox);
    tma_load_3d(ring + (size_t)s * kBox, &map, &full[s], tx * kFindTileBytes, ty * kFindTileRows, a.frame0 + iframe);
    if (++iframe == a.nframes) { iframe = 0; ++itile; }
  };
  if (threadIdx.x == 0) {
    for (int s = 0; s < kFindStages; ++s) mbar_init(&full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    for (int s = 0; s < kFindStages && begin + s < end; ++s) issue(s);
  }
  __syncthreads();
  const int off = (threadIdx.x >> 4) * kFindTileBytes + (threadIdx.x & 15) * 16;
  int slot = 0;                                        // ring slot of the current entry and the phase it completes
  uint32_t phase = 0;
  find_walk<BPS>(a, begin, end, [&](long long, int, int, uint4& q) {
    mbar_wait(&full[slot], phase);
    q = *reinterpret_cast<const uint4*>(ring + slot * (int)kBox + off);
  }, [&](long long p) {
    // every thread has added its bytes, so its shared-memory reads are complete: the slot may be refilled.  The TMA
    // write is an async-proxy access; the proxy fence orders it after the generic reads.
    __syncthreads();
    if (threadIdx.x == 0 && p + kFindStages < end) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      issue(slot);
    }
    if (++slot == kFindStages) { slot = 0; phase ^= 1u; }
  });
}

// Plain-load form for any other layout: byte loads (2-byte samples: even addresses, so 16-bit loads), zeros outside the
// plane, the same walk and the same sums.
template <int BPS>
__global__ void __launch_bounds__(kFindThreads) find_sums_plain_kernel(FindArgs a) {
  long long begin, end;
  find_share(a, &begin, &end);
  const int col = (threadIdx.x & 15) * 16, row = threadIdx.x >> 4;
  find_walk<BPS>(a, begin, end, [&](long long, int tile, int f, uint4& q) {
    const int ty = tile / a.tiles_x, tx = tile - ty * a.tiles_x;
    const int xb = tx * kFindTileBytes + col, y = ty * kFindTileRows + row;
    const uint8_t* r = a.base + (long long)(a.frame0 + f) * a.frame_stride + (long long)y * a.pitch;
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t v = 0;
      if (y < a.height) {
        if (BPS == 1) {
#pragma unroll
          for (int b = 0; b < 4; ++b) { const int x = xb + 4 * i + b; if (x < a.row_bytes) v |= (uint32_t)__ldg(r + x) << (8 * b); }
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int x = xb + 4 * i + 2 * h;
            if (x < a.row_bytes) v |= (uint32_t)__ldg(reinterpret_cast<const uint16_t*>(r + x)) << (16 * h);
          }
        }
      }
      w[i] = v;
    }
    q = make_uint4(w[0], w[1], w[2], w[3]);
  }, [](long long) {});
}

}  // namespace amtk
