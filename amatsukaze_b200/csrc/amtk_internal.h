// amtk_internal.h -- shared declarations of the CUDA translation unit (not part of the public ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <mutex>
#include <string>
#include <vector>
#include "../../include/amtk_b200.h"
#include "logo_host.h"

// cuTensorMapEncodeTiled is fetched through cudaGetDriverEntryPoint (no link-time dependency on libcuda.so).
typedef CUresult (*amtk_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                         const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                         CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

namespace amtk {

void set_error(const std::string& msg);
bool cuda_ok(cudaError_t e, const char* what);

#define AMTK_CUDA(call)                                          \
  do {                                                           \
    if (!::amtk::cuda_ok((call), #call)) return 0;               \
  } while (0)
#define AMTK_FAIL(msg)                                           \
  do {                                                           \
    ::amtk::set_error(msg);                                      \
    return 0;                                                    \
  } while (0)

// Move-only owner of one CUDA allocation, event or stream, released when the owner goes or takes another.  It converts
// to the raw handle; put() releases the current one and returns the slot an allocation call fills.
template <class P, auto Release> class CudaOwned {
 public:
  CudaOwned() = default;
  CudaOwned(CudaOwned&& o) noexcept : p_(o.release()) {}
  CudaOwned& operator=(CudaOwned&& o) noexcept { reset(o.release()); return *this; }
  ~CudaOwned() { reset(); }
  operator P() const { return p_; }
  P get() const { return p_; }
  P* put() { reset(); return &p_; }
  P release() { P p = p_; p_ = nullptr; return p; }
  void reset(P p = nullptr) { if (p_) Release(p_); p_ = p; }
 private:
  P p_ = nullptr;
};
template <class T> using DevBuf = CudaOwned<T*, cudaFree>;           // cudaMalloc
template <class T> using PinnedBuf = CudaOwned<T*, cudaFreeHost>;    // cudaHostAlloc
using EventHandle = CudaOwned<cudaEvent_t, cudaEventDestroy>;
using StreamHandle = CudaOwned<cudaStream_t, cudaStreamDestroy>;

// A device buffer grown on demand and reused across calls.  ensure(need) keeps it when it holds need bytes, else frees
// it and allocates max(need, 1 MiB); on failure it is empty, with capacity 0.
struct GrowBuf {
  DevBuf<uint8_t> buf;
  size_t cap = 0;
  bool ensure(size_t need) {
    if (cap >= need) return true;
    buf.reset(); cap = 0;
    const size_t sz = std::max(need, (size_t)1 << 20);
    uint8_t* p = nullptr;
    if (!cuda_ok(cudaMalloc(&p, sz), "cudaMalloc(scratch)")) return false;
    buf.reset(p); cap = sz;
    return true;
  }
  template <class T = uint8_t> T* at(size_t byte_off = 0) const { return reinterpret_cast<T*>(buf.get() + byte_off); }
};

// Evaluation tables of one logo as the kernels see them (all device pointers).
struct LogoDev {
  int w, h, count, countPad;      // countPad: kernel-tap row pitch (multiple of 32)
  float blackScore;
  const float* A;                 // w*h
  const float* B;                 // w*h
  const uint32_t* pix;            // count: x | y<<16, reference scan order
  const float* tapsT;             // 25 x countPad, tap-major (coalesced one-time load into registers)
  const float2* scales;           // count x 32 {scale, scale2}
};

}  // namespace amtk

struct amtk_ctx {
  // One context = one device + one stream + one set of scratch buffers.  Entry points serialise on this mutex (taken by
  // DevSelect), so concurrent calls on ONE context from several host threads (AviSynth Prefetch threads calling GetFrame
  // on MT_NICE_FILTER filters) are safe; calls on distinct contexts run concurrently.  Recursive: amtk_scan_logo calls
  // other entry points.
  mutable std::recursive_mutex mu;
  int device = 0;
  cudaStream_t stream = nullptr;            // borrowed: the caller's stream, or owned_stream
  amtk::StreamHandle owned_stream;          // a group context's own stream (null for contexts on a caller's stream)
  amtk::StreamHandle copy_stream;           // H2D staging for host-resident clips
  amtk::StreamHandle side_stream, side_stream2;   // GetFrame-sized AMTAnalyzeLogo calls: the three logo evaluations run side by side (main + two side streams)
  amtk::EventHandle ev_fork, ev_join1, ev_join2;
  amtk::EventHandle ev_copy[2];
  amtk::EventHandle ev_done[2];
  int sm_count = 0;
  int64_t launches = 0;
  long long h2d_bytes_last = 0;             // payload bytes the last host-clip call copied host->device
  // scratch (grown on demand, reused across calls)
  amtk::GrowBuf scratch;                    // per-pixel scores
  amtk::GrowBuf stage[2];                   // device staging of host clips
  amtk::GrowBuf small;                      // misc small device buffers (counters, segments)
  amtk::GrowBuf dout;                       // device-side outputs when the caller's are on the host
  amtk::GrowBuf dout2;
  amtk::GrowBuf erase_clip;                 // amtk_erase_logo_clip: records, fades, frame list and fade codes of one call
  amtk::PinnedBuf<void> hout; void* hout_dev = nullptr;     // small host outputs: pinned, device-mapped; the kernels write it directly (no D2H copy operation)
  amtk_encode_tiled_fn encode_tiled = nullptr;
  struct Knobs {            // kernel-variant selection; read from AMTK_* environment variables at context creation
    int eval_waves = 1;     // logo_scores_kernel CTAs per SM
    int eval_cw = 1;        // 1: 64-pixel-wide logos use the compile-time-width kernel variant
    int eval_par = 1;       // 1: AMTAnalyzeLogo calls of <= 16 frames run their three evaluations concurrently on three streams
    int comb_generic = 0;   // 1: force the plain-load comb kernel
    int comb_merge_uv = 1;  // U|V remainder columns share one tile
    int comb_part = -1;     // partition: -1 auto, 0 equal-share, 1 lock-step
    int comb_strip = 8, comb_stages = 3, comb_R = 0, comb_ctas = 0, comb_sync = 0, comb_l2 = 64;
    int comb_item = 0;        // frames per long work item of the warp-stream kernel (0 = auto)
    int comb_tail = 4;        // third tier of the work queue: items of this many frames over the last ~4 % of the range (0 = two tiers: +0.7 % kernel time on H100)
    int comb_ws_stages = 2;  // ring slots per warp stream
    int comb_mma = 0;        // 1|2: tensor-core streaming kernel (comb_mma.cuh) for 8-bit clips, NS tiles per CTA step
    int comb_ws10 = 0;       // 1: 16-bit containers with <= 10 significant bits run the warp-stream kernel's integer-lane form
                             // (0: the CTA-ring kernel, 1.94 vs 2.05 ms per 900 1080p frames on H100)
    int comb_ws_warps = 4;   // warp streams per CTA
    int comb_ws_prefetch = 0; // L2 prefetch distance of the warp streams' tile loads (steps ahead of the slot refill)
    int comb_ws_band = 2;    // 8-bit clips: 2 = 512 x 12R bands (12 warps per CTA), 1 = 512 x 4R bands (4 warps per CTA); 0 = one 128-byte tile per warp
    int comb_ws = 1;        // 1: round-2 warp-stream kernel for 8-bit clips (comb_stream.cuh); 0: round-1 CTA-ring kernel
  } knobs;
  // cached launch plan of the streaming comb kernel: work items on the device + occupancy, keyed by geometry, tile count,
  // range and logo-item layout.  The tile count is part of the key because the tile classes do not follow from the geometry
  // alone: the U|V pair class of the per-warp form depends on the plane order (off_v > off_u) and the plane distance.  The
  // logo-item count and frames per logo item are part of it so that a comb-only call never runs a fused call's list.
  struct CombPlanKey {                        // compared byte for byte: no padding (static_assert in amtk_b200.cu)
    const void* kernel;                       // the kernel variant the items are cut for
    int wY, hY, wC, hC, ntiles, nf, f0;
    int item, tail;                           // frames per long item (AMTK_COMB_ITEM) and per tail item (AMTK_COMB_TAIL)
    int ctas;
    int nlogo, logoF;                         // logo items of the band form (fused step) and frames per logo item
  };
  struct CombPlan {
    bool valid = false;
    CombPlanKey key{};
    amtk::GrowBuf dev;                        // [items][CombSegment] + queue counter
    int nitems = 0; size_t q_off = 0;
    int occ = 0; const void* occ_kernel = nullptr;
  } plan;
  // watchdog records of the last two band-form comb launches, used alternately (ws_watch[8 * k], k = watch_next ^ 1 is
  // the last launch's): a launch reads its record back into one while the previous launch's is checked
  amtk::PinnedBuf<int> ws_watch;            // 2 x 8 ints
  amtk::EventHandle ev_watch[2];            // recorded after each read-back
  bool watch_pending[2] = { false, false }; // that record has not been checked yet
  int watch_next = 0;                       // the record the next band-form launch reads back into
  // optional per-launch timing of the dominant (comb) kernel with CUDA events on the launching stream
  bool timing = false;
  std::vector<std::pair<amtk::EventHandle, amtk::EventHandle>> timing_events;   // recorded, not yet resolved
  std::vector<std::pair<amtk::EventHandle, amtk::EventHandle>> timing_pool;     // free pairs
  double timing_ms = 0.0; int64_t timing_count = 0;
};

struct amtk_logo {
  // Device the HBM copies live on (-1 = none yet).  Deliberately NOT a pointer to the context that first evaluated the
  // logo: logos are host objects that may outlive any context (ADVICE r1: use-after-free in destroy/ensure_device).
  int device = -1;
  amtk::HostLogo host;
  // device copies (valid after create_mask; A/B valid from creation)
  amtk::DevBuf<float> dA, dB;                     // Y planes
  amtk::DevBuf<float> dAU, dBU, dAV, dBV;
  amtk::DevBuf<uint32_t> dPix; amtk::DevBuf<float> dTapsT; amtk::DevBuf<float2> dScales;
  int countPad = 0;
  bool has_mask = false;
  bool tables_uploaded = false;
  std::mutex mu;
};

struct amtk_scan {
  amtk_ctx* ctx = nullptr;                 // used by add_frames/get_* only (the context must be alive for those calls)
  int device = 0;                          // amtk_scan_destroy needs nothing but the ordinal
  int scanw = 0, scanh = 0, logUVx = 1, logUVy = 1, thy = 0;
  int nvalid = 0;
  int bytes_per_sample = 0, bits = 0;      // sample format fixed by the first clip added (0: none yet; bits 8 for 1-byte)
  amtk::DevBuf<unsigned long long> dSums;  // [npix][3] u64: sumF, sumF2, sumFB  (exact integers; s64 for 2-byte samples)
  amtk::DevBuf<unsigned long long> dBg;    // [3 planes][2]: sumB, sumB2 (per plane scalars) + [6] = nvalid
  size_t npix = 0;
};
