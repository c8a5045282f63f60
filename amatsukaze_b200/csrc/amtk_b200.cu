// amtk_b200.cu -- the C ABI of libamtk_b200.so (include/amtk_b200.h) and all kernel launches.
// Host side of the drop-in boundary: validates arguments, moves host-resident clips through HBM staging buffers,
// builds TMA descriptors and the static work partition, launches the sm_90a kernels.  No CPU compute fallback.
#include "amtk_internal.h"
#include "logo_kernels.cuh"
#include "comb_kernels.cuh"
#include "comb_stream.cuh"
#include "comb_mma.cuh"
#include "scan_kernels.cuh"
#include "tnr_kernels.cuh"
#include "find_kernels.cuh"
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <type_traits>

extern "C" { static int logo_ensure_device(const amtk_logo* cl, amtk_ctx* ctx, bool need_tables); }

namespace amtk {

static thread_local std::string g_error;
static constexpr size_t kEvalSmemLimit = 226 * 1024;     // dynamic shared memory we ask for at most (227 KB per CTA on sm_90)
void set_error(const std::string& msg) { g_error = msg; }
bool cuda_ok(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return true;
  set_error(std::string("CUDA error: ") + cudaGetErrorString(e) + " in " + what);
  return false;
}

LogoDev logo_dev(const amtk_logo* l) {
  LogoDev d;
  d.w = l->host.w; d.h = l->host.h; d.count = l->host.count(); d.countPad = l->countPad;
  d.blackScore = l->host.blackScore; d.A = l->dA; d.B = l->dB; d.pix = l->dPix; d.tapsT = l->dTapsT; d.scales = l->dScales;
  return d;
}

struct DevSelect {   // RAII: make a device (the context's, or an ordinal) current for the duration of a call
  int prev = -1; bool ok = true;
  std::unique_lock<std::recursive_mutex> lock;     // held for the whole entry point when constructed from a context
  explicit DevSelect(const amtk_ctx* c) : DevSelect(c->device) { lock = std::unique_lock<std::recursive_mutex>(c->mu); }
  explicit DevSelect(int device) { ok = cuda_ok(cudaGetDevice(&prev), "cudaGetDevice") && cuda_ok(cudaSetDevice(device), "cudaSetDevice"); }
  ~DevSelect() { if (prev >= 0) cudaSetDevice(prev); }
};

static bool validate_clip(const amtk_clip* c, bool need_chroma) {
  if (!c || !c->base) { set_error("clip: null"); return false; }
  if (c->bytes_per_sample != 1 && c->bytes_per_sample != 2) { set_error("Unsupported pixel format"); return false; }
  if (c->width <= 0 || c->height <= 0 || c->num_frames <= 0) { set_error("clip: bad geometry"); return false; }
  if (c->pitch_y < c->width * c->bytes_per_sample) { set_error("clip: pitch_y smaller than a row"); return false; }
  if (need_chroma && c->pitch_uv < (c->width >> c->log_uvx) * c->bytes_per_sample) { set_error("clip: pitch_uv smaller than a row"); return false; }
  return true;
}

// A device-resident window of a clip: frames [first, first+count) of the clip are at dev_base + i*frame_stride
// (i = frame - first).
struct Window { const uint8_t* dev_base; int first; int count; };

// HBM staging budget per buffer (two buffers).  AMTK_STAGE_MB overrides it; read on every call, so that tests can force
// chunk boundaries on a context that already exists.
static size_t stage_budget() {
  const char* e = getenv("AMTK_STAGE_MB");
  return e ? (size_t)std::max(1, atoi(e)) << 20 : (size_t)256 << 20;
}

// Double-buffered H2D staging of a host clip's frames [frame0, frame0+nframes) in chunks of at most `per` frames, each
// staging buffer at least `need` bytes.  Per chunk [lo, hi): upload(w, lo, hi) enqueues on the copy stream the copies
// of what the chunk reads into w.dev_base (a staging buffer), sets w.first and w.count to the frames it staged (w comes
// as [lo, hi)) and returns the bytes it moved (< 0: failed); then run(w, lo, hi) enqueues the chunk's work on the
// context's stream.  A buffer is refilled only after the work of the chunk that last read it; the work waits for its own
// copies, so uploads overlap the kernels of the chunk before.  h2d_bytes_last becomes the total of the uploads.
// Returns once every upload has read the host memory (the caller may then reuse it); the work may still be in flight.
template <typename Upload, typename Run>
static int stage_chunks(amtk_ctx* ctx, int frame0, int nframes, int per, size_t need, Upload upload, Run run) {
  // the two buffers grow together: a failed growth leaves both empty, so both are reallocated by the next call
  if (!ctx->stage[0].ensure(need) || !ctx->stage[1].ensure(need)) { ctx->stage[0] = {}; ctx->stage[1] = {}; return 0; }
  long long h2d = 0;
  int chunk = 0;
  bool ok = true;
  for (int lo = frame0; ok && lo < frame0 + nframes; lo += per, ++chunk) {
    const int hi = std::min(frame0 + nframes, lo + per), b = chunk & 1;
    Window w{ ctx->stage[b].at(), lo, hi - lo };
    ok = cuda_ok(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_done[b], 0), "cudaStreamWaitEvent(stage)");   // previous user of this buffer
    const long long bytes = ok ? upload(w, lo, hi) : -1;
    ok = bytes >= 0 && cuda_ok(cudaEventRecord(ctx->ev_copy[b], ctx->copy_stream), "cudaEventRecord(stage)") &&
         cuda_ok(cudaStreamWaitEvent(ctx->stream, ctx->ev_copy[b], 0), "cudaStreamWaitEvent(stage)") && run(w, lo, hi) &&
         cuda_ok(cudaEventRecord(ctx->ev_done[b], ctx->stream), "cudaEventRecord(stage)");
    h2d += ok ? bytes : 0;
  }
  // Copies run in order on the copy stream, so the last chunk's copy event covers every upload.  A chunk k >= 2 upload
  // waits on the device for the work of chunk k-2, so without this wait a call could return while later chunks are still
  // queued to read the caller's (pinned) memory.  On a failure, wait for whatever was enqueued.
  if (!ok) { cudaStreamSynchronize(ctx->copy_stream); return 0; }
  if (chunk > 0) AMTK_CUDA(cudaEventSynchronize(ctx->ev_copy[(chunk - 1) & 1]));
  ctx->h2d_bytes_last = h2d;
  return 1;
}

// Upload of stage_chunks: frames [first, end) of a host clip in one copy.
static long long stage_frames(amtk_ctx* ctx, const amtk_clip* clip, Window& w, int first, int end) {
  const size_t fs = (size_t)clip->frame_stride, bytes = (size_t)(end - first) * fs;
  if (!cuda_ok(cudaMemcpyAsync(const_cast<uint8_t*>(w.dev_base), reinterpret_cast<const uint8_t*>(clip->base) + (size_t)first * fs,
                               bytes, cudaMemcpyHostToDevice, ctx->copy_stream), "cudaMemcpyAsync(stage)"))
    return -1;
  w.first = first; w.count = end - first;
  return (long long)bytes;
}

// Runs fn(window, lo, hi) so that frames [lo,hi) (clip numbering) are resident; with need_prev the frame lo-1 is
// resident too when lo > 0.  Device clips: one call, zero copies.  Host clips: stage_chunks of whole frames.
template <typename Fn>
static int for_each_window(amtk_ctx* ctx, const amtk_clip* clip, int frame0, int nframes, bool need_prev, Fn fn) {
  if (frame0 < 0 || nframes < 0 || frame0 + nframes > clip->num_frames) AMTK_FAIL("frame range outside the clip");
  if (nframes == 0) return 1;
  if (clip->on_device) {
    Window w{ reinterpret_cast<const uint8_t*>(clip->base), 0, clip->num_frames };
    return fn(w, frame0, frame0 + nframes);
  }
  const size_t fs = (size_t)clip->frame_stride;
  int per = (int)std::max<size_t>(1, std::min<size_t>((size_t)nframes, stage_budget() / fs));
  if (need_prev && per > 1) per -= 1;
  return stage_chunks(ctx, frame0, nframes, per, (size_t)(per + (need_prev ? 1 : 0)) * fs,
                      [&](Window& w, int lo, int hi) { return stage_frames(ctx, clip, w, need_prev && lo > 0 ? lo - 1 : lo, hi); }, fn);
}

// ROI-only staging of HOST clips for the entry points that read nothing but a rectangle of every frame
// (LogoFrame::ScanFrame, AMTAnalyzeLogo, ReMakeLogo's fade sweep, LogoScan::AddFrame, AMTEraseLogo -- the reference
// itself touches only the ROI there, LogoScan.hpp:1559-1566,1146-1155,606-635,1374-1397).  Instead of moving whole frames
// over PCIe (3.1 MB each for a 6 KB rectangle) the library copies the rectangle rows of Y (and U, V) into a compact
// clip in HBM with strided 3-D copies and runs the same kernels on that clip with shifted coordinates.
// fn(vclip, window, lo, hi, dx, dy): vclip describes the resident data; luma sample (x, y) of the real frame is at
// (x - dx, y - dy) in vclip (chroma: shifted by dx >> log_uvx, dy >> log_uvy).  write_back copies the rectangles back
// to the host frames after fn (in-place erase).
template <typename Fn>
static int for_each_roi_window(amtk_ctx* ctx, const amtk_clip* clip, int frame0, int nframes, int rx, int ry, int rw, int rh,
                               bool with_chroma, bool write_back, Fn fn) {
  if (frame0 < 0 || nframes < 0 || frame0 + nframes > clip->num_frames) AMTK_FAIL("frame range outside the clip");
  if (nframes == 0) return 1;
  if (clip->on_device) {
    Window w{ reinterpret_cast<const uint8_t*>(clip->base), 0, clip->num_frames };
    return fn(*clip, w, frame0, frame0 + nframes, 0, 0);
  }
  const int bps = clip->bytes_per_sample, lx = clip->log_uvx, ly = clip->log_uvy;
  const int A = 16 << lx;                                              // luma byte alignment that keeps chroma 16-byte aligned
  const int xb0 = ((rx * bps) / A) * A;
  const int xb1 = std::min(clip->pitch_y, (((rx + rw) * bps + A - 1) / A) * A);
  const int cp = ((xb1 - xb0 + A - 1) / A) * A;                        // compact luma pitch (bytes); chroma pitch = cp >> lx
  const int dy = ry & ~((1 << ly) - 1);
  const int y1 = std::min(clip->height, (ry + rh + (1 << ly) - 1) & ~((1 << ly) - 1));
  const int rowsY = y1 - dy, rowsC = with_chroma ? (rowsY >> ly) : 0;
  const int cpc = cp >> lx, spanY = xb1 - xb0;
  const int xc0 = xb0 >> lx, spanC = std::min(clip->pitch_uv - xc0, spanY >> lx);
  // plane offsets are whole rows of the luma pitch, so the frame stride is a multiple of both pitches (3-D copies)
  const int rows_u = rowsY, rows_c_as_y = (int)(((long long)cpc * rowsC + cp - 1) / cp);
  const long long offU = (long long)cp * rows_u, offV = offU + (long long)cp * rows_c_as_y;
  const long long fs = with_chroma ? offV + (long long)cp * rows_c_as_y : (long long)cp * rowsY;
  if (cp <= 0 || rowsY <= 0 || (with_chroma && spanC <= 0)) AMTK_FAIL("ROI staging: empty rectangle");
  const int per = (int)std::max<size_t>(1, std::min<size_t>((size_t)nframes, stage_budget() / (size_t)fs));
  amtk_clip v = *clip;
  v.frame_stride = fs; v.off_u = offU; v.off_v = offV;
  v.width = cp / bps; v.height = rowsY; v.pitch_y = cp; v.pitch_uv = cpc; v.on_device = 1;
  const uint8_t* hbase = reinterpret_cast<const uint8_t*>(clip->base);
  // one strided copy per plane and chunk (cudaMemcpy3D: x = bytes of a rectangle row, y = rows, z = frames); falls back
  // to one 2-D copy per frame when the frame stride is not a whole number of rows
  auto copy_plane = [&](int pl, uint8_t* dev, int first, int count, bool to_host, cudaStream_t st) -> bool {
    const long long hoff = pl == 0 ? 0 : (pl == 1 ? clip->off_u : clip->off_v);
    const int hp = pl ? clip->pitch_uv : clip->pitch_y, dp = pl ? cpc : cp;
    const int span = pl ? spanC : spanY, rows = pl ? rowsC : rowsY;
    const long long doff = pl == 0 ? 0 : (pl == 1 ? offU : offV);
    uint8_t* h = const_cast<uint8_t*>(hbase) + (long long)first * clip->frame_stride + hoff + (long long)(pl ? (dy >> ly) : dy) * hp + (pl ? xc0 : xb0);
    uint8_t* d = dev + doff;
    if (clip->frame_stride % hp == 0 && fs % dp == 0) {
      cudaMemcpy3DParms p3; memset(&p3, 0, sizeof(p3));
      const cudaPitchedPtr hptr = make_cudaPitchedPtr(h, (size_t)hp, (size_t)hp, (size_t)(clip->frame_stride / hp));
      const cudaPitchedPtr dptr = make_cudaPitchedPtr(d, (size_t)dp, (size_t)dp, (size_t)(fs / dp));
      p3.srcPtr = to_host ? dptr : hptr; p3.dstPtr = to_host ? hptr : dptr;
      p3.extent = make_cudaExtent((size_t)span, (size_t)rows, (size_t)count);
      p3.kind = to_host ? cudaMemcpyDeviceToHost : cudaMemcpyHostToDevice;
      return cuda_ok(cudaMemcpy3DAsync(&p3, st), "cudaMemcpy3DAsync(roi)");
    }
    for (int f = 0; f < count; ++f) {
      uint8_t* hf = h + (long long)f * clip->frame_stride; uint8_t* df = d + (long long)f * fs;
      if (!cuda_ok(to_host ? cudaMemcpy2DAsync(hf, hp, df, dp, span, rows, cudaMemcpyDeviceToHost, st)
                           : cudaMemcpy2DAsync(df, dp, hf, hp, span, rows, cudaMemcpyHostToDevice, st), "cudaMemcpy2DAsync(roi)")) return false;
    }
    return true;
  };
  const int nplanes = with_chroma ? 3 : 1;
  const long long payload = (long long)spanY * rowsY + (with_chroma ? 2LL * spanC * rowsC : 0);     // bytes per frame
  return stage_chunks(ctx, frame0, nframes, per, (size_t)per * (size_t)fs,
                      [&](Window& w, int lo, int hi) -> long long {
                        for (int pl = 0; pl < nplanes; ++pl)
                          if (!copy_plane(pl, const_cast<uint8_t*>(w.dev_base), lo, hi - lo, false, ctx->copy_stream)) return -1;
                        return (hi - lo) * payload;
                      },
                      [&](const Window& w, int lo, int hi) -> int {
                        v.base = w.dev_base; v.num_frames = hi - lo;
                        if (!fn(v, w, lo, hi, xb0 / bps, dy)) return 0;
                        if (write_back)
                          for (int pl = 0; pl < nplanes; ++pl)
                            if (!copy_plane(pl, const_cast<uint8_t*>(w.dev_base), lo, hi - lo, true, ctx->stream)) return 0;
                        return 1;
                      });
}

// ---------------------------------------------------------------------------------------------------------
// logo evaluation launches
// ---------------------------------------------------------------------------------------------------------
struct EvalSpec {
  const amtk_logo* logo;      // evaluated logo (mask built)
  int roi_x, roi_y;           // staged rectangle (the FULL logo rectangle, frame coordinates)
  int roi_w, roi_h;
  int src_mode, src_off, src_stride;
  int nfades; const float* fades;
  int take_abs;
  int out_off, out_fade_stride;     // where in an output row the values go
};

// cudaFuncAttributeMaxDynamicSharedMemorySize is sticky per (device, kernel), whichever context sets it: one table for the
// process, only ever raised, so that a small launch on one context never lowers the limit a larger one on another relies on
static bool want_smem(amtk_ctx* ctx, const void* fn, int bytes) {
  static std::mutex mu;
  static std::vector<std::pair<std::pair<int, const void*>, int>> table;     // ((device, kernel), limit set)
  std::lock_guard<std::mutex> lock(mu);
  for (auto& e : table) if (e.first.first == ctx->device && e.first.second == fn) {
    if (e.second >= bytes) return true;
    if (!cuda_ok(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes), "cudaFuncSetAttribute")) return false;
    e.second = bytes; return true;
  }
  if (!cuda_ok(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes), "cudaFuncSetAttribute")) return false;
  table.emplace_back(std::make_pair(ctx->device, fn), bytes);
  return true;
}

// A tiled TMA map with unit element strides, no interleave and no out-of-bounds fill.
static CUresult encode_map(const amtk_ctx* ctx, CUtensorMap* map, CUtensorMapDataType type, int rank, const void* base,
                           const cuuint64_t* gdim, const cuuint64_t* gstr, const cuuint32_t* box,
                           CUtensorMapSwizzle swizzle, CUtensorMapL2promotion promo) {
  const cuuint32_t estr[4] = { 1u, 1u, 1u, 1u };
  return ctx->encode_tiled(map, type, rank, const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           swizzle, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// Shared-memory plan of logo_scores_kernel: everything for logos up to ~100x100, A/B through L1 up to ~16k px, one fade
// per pass beyond.  box_bytes: the staged TMA box of one frame.  Fails with the reason when nothing fits.
static bool eval_plan(int roi_w, int roi_h, int logo_px, int box_bytes, int* ab_smem, int* pair_fades, size_t* smem) {
  *ab_smem = 1; *pair_fades = 1;
  *smem = logo_scores_smem_bytes(roi_w * roi_h, logo_px, box_bytes, *ab_smem, *pair_fades);
  if (*smem > kEvalSmemLimit) { *ab_smem = 0; *smem = logo_scores_smem_bytes(roi_w * roi_h, logo_px, box_bytes, *ab_smem, *pair_fades); }
  if (*smem > kEvalSmemLimit) { *pair_fades = 0; *smem = logo_scores_smem_bytes(roi_w * roi_h, logo_px, box_bytes, *ab_smem, *pair_fades); }
  if (*smem > kEvalSmemLimit) { set_error("logo too large for the shared-memory evaluation path (more than ~24k pixels)"); return false; }
  return true;
}

// Whether a w x h logo has a plan when its luma box is staged from rows padded to 16 bytes, as the frame streams' slots
// keep them (so that a stream can refuse the logo before any frame is sent).
static bool eval_plan_padded(int w, int h, int bytes_per_sample) {
  int ab, pf; size_t smem;
  return eval_plan(w, h, w * h, (int)((((long long)w * bytes_per_sample + 15) & ~15LL) * h), &ab, &pf, &smem);
}

// Evaluates sp's logo on frames [lo, hi) on stream `st`, with the per-pixel scores at byte offset scratch_off of
// ctx->scratch (analyze_impl runs three evaluations side by side, each on its own stream and slice).  With frame_list (a
// device list of clip frame indices), [lo, hi) are positions in the list, and the result of frame frame_list[p] goes to
// row frame_list[p] of dout (out_row0 is then 0).
static int launch_eval(amtk_ctx* ctx, const amtk_clip* clip, const Window& win, int lo, int hi, int pitch_elems,
                       const EvalSpec& sp, float* dout, int out_frame_stride, int out_row0, cudaStream_t st, size_t scratch_off,
                       const int* frame_list = nullptr) {
  const amtk::HostLogo& hl = sp.logo->host;
  if (!logo_ensure_device(sp.logo, ctx, true)) return 0;
  if (sp.nfades < 1 || sp.nfades > kMaxFades) AMTK_FAIL("too many fade levels");
  const int count = hl.count();
  const int bits = clip->bits_per_sample;
  const float maxv = (float)((1 << bits) - 1);
  if (count == 0) {   // degenerate logo: CorrelationScore is 0 -> 0/blackScore
    AMTK_FAIL("logo has no feature pixels");
  }
  const int countPad = sp.logo->countPad;
  // ROI staging: TMA box of (roi_w rounded up to 16 bytes) x roi_h samples per frame, when the layout allows it
  const int bps = clip->bytes_per_sample;
  // the box starts at imgx rounded down to 16 bytes: the TMA unit raises "illegal instruction" when the innermost
  // start address is not 16-byte aligned
  const int box_x = ((sp.roi_x * bps) & ~15) / bps;
  const int box_w = ((((sp.roi_x - box_x) + sp.roi_w) * bps + 15) & ~15) / bps;
  const long long pitch_bytes = (long long)pitch_elems * bps;
  const long long plane_rows = ((long long)clip->pitch_y * clip->height) / pitch_bytes;     // rows as addressed with pitch_elems
  // A row step above the plane's pitch (ScanFrame's byte pitch on 2-byte samples) can address rows whose start lies in
  // the plane's last, partial row step: the map's rows end before them, so such an ROI is read without TMA.
  const bool tma_ok = ctx->encode_tiled && box_w <= 256 && sp.roi_h <= 256 && (pitch_bytes & 15) == 0 &&
                      (clip->frame_stride & 15) == 0 && (reinterpret_cast<uintptr_t>(win.dev_base) & 15) == 0 &&
                      sp.roi_y + sp.roi_h <= plane_rows;
  int ab_smem, pair_fades;
  size_t smem;
  if (!eval_plan(sp.roi_w, sp.roi_h, hl.w * hl.h, box_w * sp.roi_h * bps, &ab_smem, &pair_fades, &smem)) return 0;
  CUtensorMap roi_map;
  memset(&roi_map, 0, sizeof(roi_map));
  if (tma_ok) {
    cuuint64_t gdim[3] = { (cuuint64_t)pitch_elems, (cuuint64_t)plane_rows, (cuuint64_t)win.count };
    cuuint64_t gstr[2] = { (cuuint64_t)pitch_bytes, (cuuint64_t)clip->frame_stride };
    cuuint32_t box[3] = { (cuuint32_t)box_w, (cuuint32_t)sp.roi_h, 1u };
    CUresult r = encode_map(ctx, &roi_map, bps == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, win.dev_base,
                            gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE);
    if (r != CUDA_SUCCESS) AMTK_FAIL("cuTensorMapEncodeTiled(roi) failed (" + std::to_string((int)r) + ")");
  }
  // frames per launch bounded by the score scratch (<= 96 MB)
  const size_t per_frame = (size_t)sp.nfades * countPad * sizeof(float);
  const int batch = (int)std::max<size_t>(1, std::min<size_t>((size_t)(hi - lo), ((size_t)96 << 20) / per_frame));
  if (!ctx->scratch.ensure(scratch_off + per_frame * batch)) return 0;
  for (int f0 = lo; f0 < hi; f0 += batch) {
    const int n = std::min(batch, hi - f0);
    EvalJob job;
    job.ybase = win.dev_base; job.frame_stride = clip->frame_stride; job.pitch = pitch_elems;
    job.frame0 = frame_list ? f0 : f0 - win.first; job.nframes = n;
    job.frame_list = frame_list; job.list_base = win.first;
    job.imgx = sp.roi_x; job.imgy = sp.roi_y;
    job.roi_w = sp.roi_w; job.roi_h = sp.roi_h;
    job.src_mode = sp.src_mode; job.src_off = sp.src_off; job.src_stride = sp.src_stride;
    job.logo = logo_dev(sp.logo); job.maxv = maxv; job.nfades = sp.nfades;
    for (int i = 0; i < sp.nfades; ++i) job.fades[i] = sp.fades[i];
    job.scores = ctx->scratch.at<float>(scratch_off);
    job.use_tma = tma_ok ? 1 : 0; job.roi_box_w = box_w; job.roi_box_x = box_x; job.roi_map = roi_map;
    job.ab_smem = ab_smem; job.pair_fades = pair_fades;
    const int slices3 = (count + kEvalThreads * 3 - 1) / (kEvalThreads * 3);
    int pxt = 3, slices = slices3;
    if (count <= kEvalThreads) { pxt = 1; slices = 1; }
    else if (count <= kEvalThreads * 2) { pxt = 2; slices = 1; }
    // one CTA per SM (the kernel needs the whole register file): a single wave, so the tap tables are loaded once per SM
    const int lanes = std::max(1, std::min(n, (ctx->sm_count * ctx->knobs.eval_waves) / slices));
    dim3 grid(slices, lanes);
    const bool u16 = clip->bytes_per_sample == 2;
    const bool w64 = hl.w == 64 && sp.roi_w == 64 && ctx->knobs.eval_cw;     // compile-time width variant
    const bool wh64 = w64 && hl.h == 64 && sp.roi_h == 64;                   // ... and height (LogoFrame::ScanFrame on 64x64 logos)
#define AMTK_LAUNCH_SCORES(T, P)                                                                              \
  do {                                                                                                        \
    void (*kfn)(const EvalJob) = wh64 ? logo_scores_kernel<T, P, 64, 64> : w64 ? logo_scores_kernel<T, P, 64, 0> : logo_scores_kernel<T, P, 0, 0>; \
    if (!want_smem(ctx, (const void*)kfn, (int)smem)) return 0;                                                \
    kfn<<<grid, kEvalThreads, smem, st>>>(job);                                                               \
  } while (0)
    if (!u16) { if (pxt == 1) AMTK_LAUNCH_SCORES(uint8_t, 1); else if (pxt == 2) AMTK_LAUNCH_SCORES(uint8_t, 2); else AMTK_LAUNCH_SCORES(uint8_t, 3); }
    else      { if (pxt == 1) AMTK_LAUNCH_SCORES(uint16_t, 1); else if (pxt == 2) AMTK_LAUNCH_SCORES(uint16_t, 2); else AMTK_LAUNCH_SCORES(uint16_t, 3); }
#undef AMTK_LAUNCH_SCORES
    AMTK_CUDA(cudaGetLastError());
    const int total = n * sp.nfades;
    float* sum_out = frame_list ? dout : dout + (size_t)(f0 - out_row0) * out_frame_stride;
    const int* rows = frame_list ? frame_list + f0 : nullptr;
    const size_t sum_smem = (size_t)32 * (countPad + 4) * sizeof(float);
    if (sum_smem <= 200 * 1024) {
      if (!want_smem(ctx, (const void*)logo_sum_bulk_kernel, (int)sum_smem)) return 0;
      logo_sum_bulk_kernel<<<(total + 31) / 32, 32, sum_smem, st>>>(
          job.scores, count, countPad, n, sp.nfades, hl.blackScore, sp.take_abs, sum_out, out_frame_stride, sp.out_off, sp.out_fade_stride, rows);
    } else {
      logo_sum_kernel<<<(total + kSumThreads - 1) / kSumThreads, kSumThreads, 0, st>>>(
          job.scores, count, countPad, n, sp.nfades, hl.blackScore, sp.take_abs, sum_out, out_frame_stride, sp.out_off, sp.out_fade_stride, rows);
    }
    AMTK_CUDA(cudaGetLastError());
    ctx->launches += 2;
  }
  return 1;
}

static bool roi_inside(const amtk::HostLogo& full, const amtk_clip* clip, int pitch_elems) {
  // the ROI rows must lie inside the frame allocation as addressed with pitch_elems
  if (full.imgx < 0 || full.imgy < 0) return false;
  const long long last = (long long)full.imgx + full.w - 1 + (long long)(full.imgy + full.h - 1) * pitch_elems;
  const long long plane_elems = (long long)clip->pitch_y / clip->bytes_per_sample * clip->height;
  return full.imgx + full.w <= pitch_elems && last < plane_elems;
}

// ---------------------------------------------------------------------------------------------------------
// comb launch
// ---------------------------------------------------------------------------------------------------------
static int comb_thresholds_ok(const amtk_comb_params* p, int bytes_per_sample) {
  if (bytes_per_sample == 2) {
    const int all[6] = { p->th_move_y, p->th_shima_y, p->th_lshima_y, p->th_move_c, p->th_shima_c, p->th_lshima_c };
    for (int v : all) if (v < 1) { set_error("comb: thresholds must be >= 1"); return 0; }
    if (p->th_move_y > 32768 || p->th_move_c > 32768) { set_error("comb: th_move must be in [1,32768] for 16-bit samples"); return 0; }
    return 1;
  }
  const int m[2] = { p->th_move_y, p->th_move_c };
  const int s[4] = { p->th_shima_y, p->th_lshima_y, p->th_shima_c, p->th_lshima_c };
  for (int v : m) if (v < 1 || v > 128) { set_error("comb: th_move must be in [1,128]"); return 0; }
  for (int v : s) if (v < 1 || v > 2047) { set_error("comb: th_shima/th_lshima must be in [1,2047]"); return 0; }
  return 1;
}

// Everything the host needs to know about one compiled comb-kernel variant.
struct CombVariant {
  int R, strip, stages, sync, TH, boxH, threads, smem;
  void (*kernel)(const CombArgs);        // 8-bit samples
  void (*kernel16)(const CombArgs);      // 16-bit samples (only for the default variants; else NULL)
};
template <typename Cfg> static CombVariant make_variant() {
  return CombVariant{ Cfg::R, Cfg::STRIP, Cfg::STAGES, Cfg::SYNC, Cfg::TH, Cfg::BOXH, Cfg::THREADS, Cfg::SMEM, comb_tma_kernel<Cfg, 1>, nullptr };
}
template <typename Cfg> static CombVariant make_variant16() {     // 8-byte strips: 8 px of u8 or 4 px of u16
  return CombVariant{ Cfg::R, Cfg::STRIP, Cfg::STAGES, Cfg::SYNC, Cfg::TH, Cfg::BOXH, Cfg::THREADS, Cfg::SMEM, comb_tma_kernel<Cfg, 1>, comb_tma_kernel<Cfg, 2> };
}
static const CombVariant* comb_variants(int* n) {
  static const CombVariant v[] = {
    // production: rows-per-run chosen per clip (pick_comb_R), 8-byte strips, 3-stage ring, block barrier per tile-frame
    make_variant16<CombCfg<15, 8, 3, 0>>(), make_variant16<CombCfg<16, 8, 3, 0>>(), make_variant16<CombCfg<17, 8, 3, 0>>(),
    // kept for tools/tune_comb.py: 2- and 4-stage rings, mbarrier 'release' sync (all measured below the production
    // variant; DESIGN.md section 6)
    make_variant<CombCfg<17, 8, 2, 0>>(), make_variant<CombCfg<17, 8, 4, 0>>(), make_variant<CombCfg<17, 8, 3, 1>>(),
  };
  *n = (int)(sizeof(v) / sizeof(v[0]));
  return v;
}

// rows per run: the R in {15,16,17} that wastes the fewest rows over luma + chroma (1080/540 -> 17, 720/360 -> 15)
static int pick_comb_R(int hY, int hC) {
  int best = 16; long long best_waste = -1;
  for (int R = 17; R >= 15; --R) {
    const int th = 8 * R;
    const long long waste = (long long)((hY + th - 1) / th) * th - hY + 2LL * (((hC + th - 1) / th) * th - hC) / 2;
    if (best_waste < 0 || waste < best_waste) { best_waste = waste; best = R; }
  }
  return best;
}

// ---- round-2 streaming kernel (comb_stream.cuh): independent warp streams, 8-bit samples ----------------------
struct WsVariant { int R, stages, warps, bps, TH, boxH, smem; bool band; void (*kernel)(const WsArgs); };
template <typename Cfg> static WsVariant make_ws() { return WsVariant{ Cfg::R, Cfg::STAGES, Cfg::WARPS, Cfg::BPS, Cfg::TH, Cfg::BOXH, Cfg::SMEM, Cfg::BAND, comb_ws_kernel<Cfg> }; }
static const WsVariant* ws_variants(int* n) {
  static const WsVariant v[] = { make_ws<WsCfg<17, 2>>(), make_ws<WsCfg<15, 2>>(), make_ws<WsCfg<16, 2>>(), make_ws<WsCfg<9, 2>>(), make_ws<WsCfg<15, 3>>(), make_ws<WsCfg<12, 2>>(), make_ws<WsCfg<10, 2>>(),
                                 make_ws<WsCfg<15, 2, 7>>(), make_ws<WsCfg<13, 2, 5>>(), make_ws<WsCfg<15, 2, 2>>(), make_ws<WsCfg<15, 3, 3>>(),
                                 // 16-bit containers with <= 10 significant bits (YUV420P10): integer-lane stencil, no conversion
                                 make_ws<WsCfg<15, 2, 4, 2>>(), make_ws<WsCfg<16, 2, 4, 2>>(), make_ws<WsCfg<17, 2, 4, 2>>(),
                                 // 8-bit 512 x 4R bands: four warps share one ring of 512-byte-wide slots
                                 make_ws<WbCfg<15, 2>>(), make_ws<WbCfg<16, 2>>(), make_ws<WbCfg<17, 2>>(), make_ws<WbCfg<15, 3>>(),
                                 // 8-bit tall bands (default): twelve warps share one ring of 512 x 12R slots (R = 17 spills
                                 // at the 168 registers of 384 threads per SM)
                                 make_ws<WtCfg<15, 2>>(), make_ws<WtCfg<16, 2>>() };
  *n = (int)(sizeof(v) / sizeof(v[0]));
  return v;
}
// rows per run for tiles of `runs` runs: fewest wasted rows over luma + chroma, ties to the larger R (less halo per row)
static int pick_ws_R(int hY, int hC, int runs = kWsRuns) {
  int best = 17; long long best_waste = -1;
  for (int R : { 17, 16, 15 }) {
    const int th = runs * R;
    const long long waste = 2LL * ((long long)((hY + th - 1) / th) * th - hY) + 2LL * ((long long)((hC + th - 1) / th) * th - hC);
    if (best_waste < 0 || waste < best_waste) { best_waste = waste; best = R; }
  }
  return best;
}

// Watchdog record k of the band-form launches (amtk_ctx::ws_watch), when it has not been checked: waits for its read-back
// and fails if a device-side wait of that launch timed out, which means the counters it returned are not valid.  A launch
// checks the previous launch's record after it has enqueued its own work, so the GPU never waits for the host here; a
// call that synchronises its stream anyway checks its own launch's record after that (ws_watchdog_synced).  So a
// timed-out wait fails the call that ran it when that call synchronises, and otherwise the next comb call on the context.
static int ws_watchdog_ok(amtk_ctx* ctx, int k) {
  if (!ctx->watch_pending[k]) return 1;
  AMTK_CUDA(cudaEventSynchronize(ctx->ev_watch[k]));
  ctx->watch_pending[k] = false;
  const int* d = ctx->ws_watch + 8 * k;
  if (d[0]) {
    char msg[256];
    snprintf(msg, sizeof(msg), "comb_ws (band form): a device-side wait timed out (wait %d, step %d, CTA %d, thread %d, parity %d); its counters are not valid",
             d[1], d[2], d[3], d[4], d[5]);
    AMTK_FAIL(msg);
  }
  return 1;
}
// After a synchronisation of the context's stream: checks both records (their read-backs are done, no wait), the older first.
static int ws_watchdog_synced(amtk_ctx* ctx) {
  return ws_watchdog_ok(ctx, ctx->watch_next) && ws_watchdog_ok(ctx, ctx->watch_next ^ 1);
}

// The watchdog record a band-form launch leaves on the device: 8 ints behind the work queue counter of the cached plan
// (args.queue + 16), valid until the next comb launch on the context resets the queue.
static const int* ws_watch_record(const amtk_ctx* ctx) {
  return ctx->plan.dev.at<const int>(ctx->plan.q_off) + 16;
}

// L2 promotion of the streaming comb kernels' tensor maps (AMTK_COMB_L2: 0, 64, 128 or 256 bytes)
static CUtensorMapL2promotion comb_l2_promotion(const amtk_ctx* ctx) {
  switch (ctx->knobs.comb_l2) {
    case 0: return CU_TENSOR_MAP_L2_PROMOTION_NONE;
    case 64: return CU_TENSOR_MAP_L2_PROMOTION_L2_64B;
    case 256: return CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
    default: return CU_TENSOR_MAP_L2_PROMOTION_L2_128B;
  }
}

// The tail of a streaming comb launch: zero the nf counter rows at `counts`, then launch() on the context's stream,
// between the two events of a timing pair when kernel timing is on.
template <typename Launch>
static int comb_launch(amtk_ctx* ctx, int* counts, int nf, Launch launch) {
  AMTK_CUDA(cudaMemsetAsync(counts, 0, (size_t)nf * 12 * sizeof(int), ctx->stream));
  std::pair<EventHandle, EventHandle> ev;
  if (ctx->timing) {
    if (!ctx->timing_pool.empty()) { ev = std::move(ctx->timing_pool.back()); ctx->timing_pool.pop_back(); }
    else { AMTK_CUDA(cudaEventCreate(ev.first.put())); AMTK_CUDA(cudaEventCreate(ev.second.put())); }
    AMTK_CUDA(cudaEventRecord(ev.first, ctx->stream));
  }
  launch();
  AMTK_CUDA(cudaGetLastError());
  if (ctx->timing) { AMTK_CUDA(cudaEventRecord(ev.second, ctx->stream)); ctx->timing_events.push_back(std::move(ev)); }
  ctx->launches += 1;
  return 1;
}

static_assert(std::has_unique_object_representations<amtk_ctx::CombPlanKey>::value, "plan keys are compared with memcmp");

// Points args at the cached work-item list of the queue kernels (warp-stream and wgmma forms), after building it with
// build() and uploading it when the cached list was made for another key; resets the queue counter behind it.
template <typename Build>
static int comb_plan(amtk_ctx* ctx, const amtk_ctx::CombPlanKey& key, WsArgs& args, Build build) {
  amtk_ctx::CombPlan& plan = ctx->plan;
  if (!plan.valid || memcmp(&plan.key, &key, sizeof(key)) != 0) {
    const std::vector<CombSegment> segs = build();
    const size_t seg_bytes = segs.size() * sizeof(CombSegment);
    plan.q_off = (seg_bytes + 255) & ~(size_t)255;
    plan.valid = false;
    if (!plan.dev.ensure(plan.q_off + 256)) return 0;
    AMTK_CUDA(cudaMemcpyAsync(plan.dev.at(), segs.data(), seg_bytes, cudaMemcpyHostToDevice, ctx->stream));
    AMTK_CUDA(cudaStreamSynchronize(ctx->stream));           // pageable source vector dies at the end of this scope
    plan.nitems = (int)segs.size(); plan.key = key; plan.valid = true;
  }
  AMTK_CUDA(cudaMemsetAsync(plan.dev.at(plan.q_off), 0, 256, ctx->stream));
  args.segs = plan.dev.at<const CombSegment>();
  args.nitems = plan.nitems;
  args.queue = plan.dev.at<int>(plan.q_off);
  return 1;
}

// The warp-stream kernel variant a clip runs (NULL: none compiled for the AMTK_COMB_* settings).  8-bit clips run the
// tall band form (AMTK_COMB_WS_BAND=2) when a variant has the rows per run and stages asked for, else the 512 x 4R band
// form; AMTK_COMB_WS_BAND=1 asks for the latter, =0 or another warp count for one 128-byte tile per warp.
// tall = false: the 512 x 4R band variant of a band-form clip, whichever band form it runs.
static const WsVariant* ws_variant(const amtk_ctx* ctx, const amtk_clip* clip, bool tall = true) {
  const int hY = clip->height, hC = clip->height >> clip->log_uvy;
  int nvar = 0; const WsVariant* vars = ws_variants(&nvar);
  const int bps = clip->bytes_per_sample;
  const bool band = bps == 1 && ctx->knobs.comb_ws_band && ctx->knobs.comb_ws_warps == kWsWarps;
  auto find = [&](int runs, int warps) -> const WsVariant* {
    const int R = ctx->knobs.comb_R ? ctx->knobs.comb_R : pick_ws_R(hY, hC, runs);
    for (int i = 0; i < nvar; ++i)
      if (vars[i].R == R && vars[i].stages == ctx->knobs.comb_ws_stages && vars[i].warps == warps && vars[i].bps == bps && vars[i].band == band) return &vars[i];
    return nullptr;
  };
  if (band && tall && ctx->knobs.comb_ws_band == 2)
    if (const WsVariant* V = find(kWtGroups * kWsRuns, kWtGroups * kWsWarps)) return V;
  return find(kWsRuns, ctx->knobs.comb_ws_warps);
}

// lj (band form only): the queue also gets logo items, ScanFrame scores of lj->frames frames each (fused step)
static int launch_comb_ws(amtk_ctx* ctx, const amtk_clip* clip, const Window& win, int lo, int hi,
                          const amtk_comb_params* prm, int* dcounts, int out_row0, const ScanItemJob* lj = nullptr) {
  const int hY = clip->height, hC = clip->height >> clip->log_uvy;
  const int wY = clip->width, wC = clip->width >> clip->log_uvx;
  const int bps = clip->bytes_per_sample;
  const WsVariant* V = ws_variant(ctx, clip);
  if (!V) AMTK_FAIL("comb: no warp-stream kernel variant for the requested AMTK_COMB_* settings");
  const bool band = V->band;
  if (lj && !band) AMTK_FAIL("comb: logo items need the band form");
  const int WW = V->warps;
  // the record a band-form launch reads back into was checked by the launch before the last one (this only waits when that
  // launch failed after enqueueing its kernel); the last one's is checked once this launch is queued
  if (!ws_watchdog_ok(ctx, ctx->watch_next)) return 0;
  const int prev = ctx->watch_next ^ 1;
  WsArgs args;
  memset(&args, 0, sizeof(args));
  const CUtensorMapL2promotion promo = comb_l2_promotion(ctx);
  for (int pl = 0; pl < 3; ++pl) {
    const long long off = pl == 0 ? 0 : (pl == 1 ? clip->off_u : clip->off_v);
    cuuint64_t gdim[3] = { (cuuint64_t)(pl ? wC : wY) * bps, (cuuint64_t)(pl ? hC : hY), (cuuint64_t)win.count };     // x in BYTES (u8 element type also for 16-bit containers)
    cuuint64_t gstr[2] = { (cuuint64_t)(pl ? clip->pitch_uv : clip->pitch_y), (cuuint64_t)clip->frame_stride };
    cuuint32_t box[3] = { (cuuint32_t)(band ? kWbHalf : kWsTW), (cuuint32_t)V->boxH, 1u };
    if (encode_map(ctx, &args.map[pl], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, win.dev_base + off, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_NONE, promo) != CUDA_SUCCESS)
      AMTK_FAIL("cuTensorMapEncodeTiled failed");
  }
  // chroma remainder columns of at most 64 bytes: U and V side by side in one tile through a 4-D map (x, plane, y, frame)
  const int remC = (wC * bps) % kWsTW;
  const long long uv_dist = clip->off_v - clip->off_u;
  const bool pair_uv = !band && ctx->knobs.comb_merge_uv && remC > 0 && remC <= kWsTW / 2 && uv_dist > 0 && (uv_dist & 15) == 0;
  if (pair_uv) {
    cuuint64_t gdim[4] = { (cuuint64_t)wC * bps, 2u, (cuuint64_t)hC, (cuuint64_t)win.count };
    cuuint64_t gstr[3] = { (cuuint64_t)uv_dist, (cuuint64_t)clip->pitch_uv, (cuuint64_t)clip->frame_stride };
    cuuint32_t box[4] = { (cuuint32_t)(kWsTW / 2), 2u, (cuuint32_t)V->boxH, 1u };
    if (encode_map(ctx, &args.map_uv, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, win.dev_base + clip->off_u, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_NONE, promo) != CUDA_SUCCESS)
      AMTK_FAIL("cuTensorMapEncodeTiled(uv pair) failed");
  }
  const int tyY = (hY + V->TH - 1) / V->TH, tyC = (hC + V->TH - 1) / V->TH;
  int tile0 = 0, nc = 0;
  auto thresholds = [&](WsClass& C, bool chroma) {
    C.cls = chroma ? 1 : 0; C.H = chroma ? hC : hY;
    const int tM = chroma ? prm->th_move_c : prm->th_move_y, tS = chroma ? prm->th_shima_c : prm->th_shima_y, tL = chroma ? prm->th_lshima_c : prm->th_lshima_y;
    if (bps == 1) {
      C.thM = (unsigned)(0x80 - tM) * 0x01010101u;
      C.thS = (unsigned)tS * 0x00010001u;     // integer k in [1,2047] IS the fp16 bit pattern of k*2^-24
      C.thL = (unsigned)tL * 0x00010001u;
    } else {                                   // <= 10-bit samples: |d| <= 1023, |r| <= 6138, r is compared as 8192 + |r| (bit patterns)
      C.thM = (unsigned)std::min(tM, 2047) * 0x00010001u;
      C.thS = (unsigned)(8192 + std::min(tS, 8191)) * 0x00010001u;
      C.thL = (unsigned)(8192 + std::min(tL, 8191)) * 0x00010001u;
    }
  };
  for (int pl = 0; pl < 3; ++pl) {                         // 128-byte tiles of Y, U, V
    WsClass& C = args.cl[nc];
    const int w = (pl ? wC : wY) * bps;                    // bytes
    C.kind = 0; C.map = pl; C.W = w; thresholds(C, pl != 0);
    C.tilesX = band ? (w + kWbW - 1) / kWbW : (pl && pair_uv) ? w / kWsTW : (w + kWsTW - 1) / kWsTW;
    C.tile0 = tile0; C.ntiles = C.tilesX * (pl ? tyC : tyY);
    if (C.ntiles == 0) continue;
    tile0 += C.ntiles; ++nc;
  }
  if (pair_uv) {
    WsClass& C = args.cl[nc];
    C.kind = 1; C.x0 = wC * bps - remC; C.tilesX = 1; thresholds(C, true);
    C.tile0 = tile0; C.ntiles = tyC; tile0 += C.ntiles; ++nc;
  }
  args.nclasses = nc;
  const int ntiles = tile0, nf = hi - lo;
  amtk_ctx::CombPlan& plan = ctx->plan;
  if (plan.occ_kernel != (const void*)V->kernel) {          // once per kernel variant, not per launch
    int occ = 0;
    AMTK_CUDA(cudaFuncSetAttribute(V->kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, V->smem));
    AMTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, V->kernel, 32 * WW, V->smem));
    if (occ < 1) AMTK_FAIL("comb kernel does not fit on an SM");
    plan.occ = occ; plan.occ_kernel = (const void*)V->kernel;
  }
  int occ = plan.occ;
  if (ctx->knobs.comb_ctas > 0) occ = std::min(occ, ctx->knobs.comb_ctas);
  // Work queue: every tile's frame range is cut into items; the warps pull items from a global counter.  Long items
  // (little halo overhead: one extra tile load per item) make up the first ~85 % of the work, short ones the rest, so
  // that all warps run dry within about one short item of each other.  The item list depends only on the tile count and
  // the frame range, so it stays on the device between calls (a 1-frame GetFrame call re-uses it without any copy).
  // A band CTA is one stream (its warps work on the same item); otherwise every warp is one.
  // Logo items (fused step) are spread evenly through the head tier: placed first they would start every CTA with
  // arithmetic and leave HBM idle, and in the short tail tiers they would upset the balance at the end of the kernel.
  const int logoF = lj ? lj->frames : 0, nlogo = lj ? (nf + logoF - 1) / logoF : 0;
  const long long total = (long long)ntiles * nf + nlogo;
  const int per_cta = band ? 1 : WW;
  const int nwarps = ctx->sm_count * occ * per_cta;
  const int grid = (int)std::min<long long>((long long)ctx->sm_count * occ, (total + per_cta - 1) / per_cta);
  const int f0 = lo - win.first;
  const amtk_ctx::CombPlanKey key{ (const void*)V->kernel, wY, hY, wC, hC, ntiles, nf, f0, ctx->knobs.comb_item, ctx->knobs.comb_tail,
                                   occ * WW, nlogo, logoF };
  if (!comb_plan(ctx, key, args, [&] {
    int big = ctx->knobs.comb_item > 0 ? ctx->knobs.comb_item : 64, small = std::max(4, big / 4);
    // each warp should see at least ~6 big items; shrink for short clips
    while (big > 8 && (long long)ntiles * (nf / big) < 6LL * nwarps) { big /= 2; small = std::max(4, big / 4); }
    const int tail_frames = std::min(nf, std::max(small, (int)(nf * 0.15)));
    const int head_frames = nf - tail_frames;
    // third tier (AMTK_COMB_TAIL = frames per item, 0 = off): the last ~4 % of the frames in very short items, so that the warps
    // run dry within one such item of each other (two tiers instead of three: +0.7 % kernel time on H100)
    const int tiny = ctx->knobs.comb_tail;
    const int end_frames = (tiny > 0 && tiny < small) ? std::min(tail_frames, std::max(tiny, (int)(nf * 0.04))) : 0;
    const int mid_end = nf - end_frames;
    std::vector<CombSegment> segs;
    segs.reserve((size_t)ntiles * (head_frames / big + tail_frames / small + (tiny > 0 ? end_frames / tiny : 0) + 3) + nlogo);
    // Warp streams: tile-major within each tier.  Bands: frame-block-major with x fastest, so that the bands of one row of
    // the picture are read at the same frames.
    auto tier = [&](int fa, int fz, int step) {
      if (band) {
        for (int f = fa; f < fz; f += step)
          for (int t = 0; t < ntiles; ++t) segs.push_back(CombSegment{ t, f0 + f, f0 + std::min(fz, f + step) });
      } else {
        for (int t = 0; t < ntiles; ++t)
          for (int f = fa; f < fz; f += step) segs.push_back(CombSegment{ t, f0 + f, f0 + std::min(fz, f + step) });
      }
    };
    tier(0, head_frames, big);
    if (nlogo > 0) {                                         // logo item k goes before head item (2k+1) * nhead / (2 * nlogo)
      const std::vector<CombSegment> head(segs);
      const long long nhead = (long long)head.size();
      segs.clear();
      int k = 0;
      for (long long i = 0; i <= nhead; ++i) {
        for (; k < nlogo && (2LL * k + 1) * nhead / (2LL * nlogo) <= i; ++k)
          segs.push_back(CombSegment{ -1, f0 + k * logoF, f0 + std::min(nf, (k + 1) * logoF) });
        if (i < nhead) segs.push_back(head[(size_t)i]);
      }
    }
    tier(head_frames, mid_end, small);
    if (tiny > 0) tier(mid_end, nf, tiny);
    return segs;
  }))
    return 0;
  args.counts = dcounts;
  args.out_frame0 = out_row0 - win.first;
  args.prefetch = ctx->knobs.comb_ws_prefetch;
  if (lj) args.logo = *lj;
  if (!comb_launch(ctx, dcounts + (size_t)(lo - out_row0) * 12, nf, [&] { V->kernel<<<grid, 32 * WW, V->smem, ctx->stream>>>(args); }))
    return 0;
  if (band) {
    // the band ring's watchdog record, read back without a synchronisation
    if (!ctx->ws_watch) {
      AMTK_CUDA(cudaHostAlloc(ctx->ws_watch.put(), 2 * 8 * sizeof(int), cudaHostAllocDefault));
      for (EventHandle& e : ctx->ev_watch) AMTK_CUDA(cudaEventCreateWithFlags(e.put(), cudaEventDisableTiming));
    }
    const int k = ctx->watch_next;
    AMTK_CUDA(cudaMemcpyAsync(ctx->ws_watch + 8 * k, ws_watch_record(ctx), 8 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    AMTK_CUDA(cudaEventRecord(ctx->ev_watch[k], ctx->stream));
    ctx->watch_pending[k] = true;
    ctx->watch_next = k ^ 1;
  }
  return ws_watchdog_ok(ctx, prev);
}

// ---- tensor-core streaming kernel (comb_mma.cuh): one CTA = one tile stream, stencil as four wgmma per tile-frame ----
static int launch_comb_mma(amtk_ctx* ctx, const amtk_clip* clip, const Window& win, int lo, int hi,
                           const amtk_comb_params* prm, int* dcounts, int out_row0) {
  const int hY = clip->height, hC = clip->height >> clip->log_uvy;
  const int wY = clip->width, wC = clip->width >> clip->log_uvx;
  WsArgs args;
  memset(&args, 0, sizeof(args));
  for (int pl = 0; pl < 3; ++pl) {
    const long long off = pl == 0 ? 0 : (pl == 1 ? clip->off_u : clip->off_v);
    cuuint64_t gdim[3] = { (cuuint64_t)(pl ? wC : wY), (cuuint64_t)(pl ? hC : hY), (cuuint64_t)win.count };
    cuuint64_t gstr[2] = { (cuuint64_t)(pl ? clip->pitch_uv : clip->pitch_y), (cuuint64_t)clip->frame_stride };
    cuuint32_t box[3] = { (cuuint32_t)kMmTW, (cuuint32_t)kMmBoxH, 1u };
    // 128-byte swizzle: the staged tile is the MN-major A operand of the MMA as it lands
    if (encode_map(ctx, &args.map[pl], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, win.dev_base + off, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_128B,
                   comb_l2_promotion(ctx)) != CUDA_SUCCESS)
      AMTK_FAIL("cuTensorMapEncodeTiled failed");
  }
  const int tyY = (hY + kMmTH - 1) / kMmTH, tyC = (hC + kMmTH - 1) / kMmTH;
  int tile0 = 0, nc = 0;
  for (int pl = 0; pl < 3; ++pl) {
    WsClass& C = args.cl[nc];
    const bool chroma = pl != 0;
    C.kind = 0; C.map = pl; C.cls = chroma ? 1 : 0; C.H = chroma ? hC : hY;
    C.thM = (unsigned)(0x80 - (chroma ? prm->th_move_c : prm->th_move_y)) * 0x01010101u;
    C.thS = (unsigned)(chroma ? prm->th_shima_c : prm->th_shima_y) * 0x00010001u;
    C.thL = (unsigned)(chroma ? prm->th_lshima_c : prm->th_lshima_y) * 0x00010001u;
    C.tilesX = ((chroma ? wC : wY) + kMmTW - 1) / kMmTW;
    C.tile0 = tile0; C.ntiles = C.tilesX * (chroma ? tyC : tyY);
    if (C.ntiles == 0) continue;
    tile0 += C.ntiles; ++nc;
  }
  args.nclasses = nc;
  const int ntiles = tile0, nf = hi - lo;
  amtk_ctx::CombPlan& plan = ctx->plan;
  // NS tiles per CTA step (AMTK_COMB_MMA = 1 or 2)
  const int NS = ctx->knobs.comb_mma == 2 ? 2 : 1;
  void (*kern)(const WsArgs) = NS == 2 ? comb_mma_kernel<2> : comb_mma_kernel<1>;
  const int smem = NS * kMmSmemPerStream + kMmBandBytes + 1024;
  if (plan.occ_kernel != (const void*)kern) {
    AMTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int occ_q = 0;
    AMTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_q, kern, kMmThreads, smem));
    if (occ_q < 1) AMTK_FAIL("comb_mma: kernel does not fit on an SM");
    plan.occ = occ_q; plan.occ_kernel = (const void*)kern;
  }
  int occ = plan.occ;
  if (ctx->knobs.comb_ctas > 0) occ = std::min(occ, ctx->knobs.comb_ctas);
  const int npairs_t = (ntiles + NS - 1) / NS;               // a CTA streams NS tiles at a time
  const long long total = (long long)npairs_t * nf;
  const int nstreams = ctx->sm_count * occ;
  const int grid = (int)std::min<long long>(nstreams, total);
  const int f0 = lo - win.first;
  const amtk_ctx::CombPlanKey key{ (const void*)kern, wY, hY, wC, hC, ntiles, nf, f0, ctx->knobs.comb_item, 0, occ, 0, 0 };
  if (!comb_plan(ctx, key, args, [&] {
    int big = ctx->knobs.comb_item > 0 ? ctx->knobs.comb_item : 64, small = std::max(4, big / 4);
    while (big > 8 && (long long)npairs_t * (nf / big) < 6LL * nstreams) { big /= 2; small = std::max(4, big / 4); }
    const int tail_frames = std::min(nf, std::max(small, (int)(nf * 0.15)));
    const int head_frames = nf - tail_frames;
    // Items come in PAIRS (2i, 2i+1) with the same frame range; an odd tile count is padded with a filler (tile = ~t: the
    // last tile once more, results dropped).  Frame-block-major order: CTAs running at the same time work on the same
    // frames of neighbouring tiles, so halo rows and straddled lines are shared through L2.
    std::vector<CombSegment> segs;
    segs.reserve((size_t)NS * npairs_t * (head_frames / big + tail_frames / small + 2));
    auto push_block = [&](int fa, int fz) {
      for (int t = 0; t < ntiles; t += NS) {
        segs.push_back(CombSegment{ t, fa, fz });
        if (NS == 2) segs.push_back(CombSegment{ t + 1 < ntiles ? t + 1 : ~t, fa, fz });
      }
    };
    for (int f = 0; f < head_frames; f += big) push_block(f0 + f, f0 + std::min(head_frames, f + big));
    for (int f = head_frames; f < nf; f += small) push_block(f0 + f, f0 + std::min(nf, f + small));
    return segs;
  }))
    return 0;
  args.counts = dcounts;
  args.out_frame0 = out_row0 - win.first;
  if (!comb_launch(ctx, dcounts + (size_t)(lo - out_row0) * 12, nf, [&] { kern<<<grid, kMmThreads, smem, ctx->stream>>>(args); }))
    return 0;
  // experimental kernel: read its watchdog record back (costs a stream synchronisation per launch)
  int dbg[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
  AMTK_CUDA(cudaMemcpyAsync(dbg, args.queue + 16, sizeof(dbg), cudaMemcpyDeviceToHost, ctx->stream));
  AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
  if (dbg[0]) {
    char msg[256];
    snprintf(msg, sizeof(msg), "comb_mma<%d>: a device-side wait timed out (wait %d, step %d, CTA %d, thread %d, parity %d); results discarded",
             NS, dbg[1], dbg[2], dbg[3], dbg[4], dbg[5]);
    AMTK_FAIL(msg);
  }
  return 1;
}

static bool comb_tma_layout(const amtk_ctx* ctx, const amtk_clip* clip, const Window& win) {
  return ctx->encode_tiled && !((clip->frame_stride & 15) || (clip->pitch_y & 15) || (clip->pitch_uv & 15) || (clip->off_u & 15) ||
                                (clip->off_v & 15) || (reinterpret_cast<uintptr_t>(win.dev_base) & 15));
}
// launch_comb runs the band form of the warp-stream kernel on this window
static bool comb_runs_band(const amtk_ctx* ctx, const amtk_clip* clip, const Window& win) {
  return comb_tma_layout(ctx, clip, win) && !ctx->knobs.comb_generic && !ctx->knobs.comb_mma && ctx->knobs.comb_ws &&
         clip->bytes_per_sample == 1 && ctx->knobs.comb_ws_band && ctx->knobs.comb_ws_warps == kWsWarps;
}

static int launch_comb(amtk_ctx* ctx, const amtk_clip* clip, const Window& win, int lo, int hi,
                       const amtk_comb_params* prm, int* dcounts, int out_row0) {
  if (!comb_tma_layout(ctx, clip, win) || ctx->knobs.comb_generic) {
    // generic kernel: any sample size / pitch (DESIGN.md 3.1 "fallback")
    CombGenericArgs g;
    g.base = win.dev_base; g.frame_stride = clip->frame_stride;
    g.off[0] = 0; g.off[1] = clip->off_u; g.off[2] = clip->off_v;
    const int bps = clip->bytes_per_sample;
    for (int pl = 0; pl < 3; ++pl) {
      g.pitch[pl] = (pl ? clip->pitch_uv : clip->pitch_y) / bps;
      g.W[pl] = pl ? (clip->width >> clip->log_uvx) : clip->width;
      g.H[pl] = pl ? (clip->height >> clip->log_uvy) : clip->height;
      g.thM[pl] = pl ? prm->th_move_c : prm->th_move_y;
      g.thS[pl] = pl ? prm->th_shima_c : prm->th_shima_y;
      g.thL[pl] = pl ? prm->th_lshima_c : prm->th_lshima_y;
    }
    g.first_frame = lo - win.first; g.prev_of_first = lo > 0 ? lo - 1 - win.first : lo - win.first;
    g.nframes = hi - lo; g.counts = dcounts + (size_t)(lo - out_row0) * 12;
    AMTK_CUDA(cudaMemsetAsync(g.counts, 0, (size_t)(hi - lo) * 12 * sizeof(int), ctx->stream));
    for (int f0 = 0; f0 < hi - lo; f0 += 16384) {            // gridDim.z limit
      CombGenericArgs gg = g;
      gg.first_frame = g.first_frame + f0; gg.prev_of_first = f0 ? gg.first_frame - 1 : g.prev_of_first;
      gg.nframes = std::min(16384, hi - lo - f0); gg.counts = g.counts + (size_t)f0 * 12;
      dim3 grid((g.W[0] + kGenTW - 1) / kGenTW, (g.H[0] + kGenTH - 1) / kGenTH, gg.nframes * 3);
      if (bps == 1) comb_generic_kernel<uint8_t><<<grid, 256, 0, ctx->stream>>>(gg);
      else comb_generic_kernel<uint16_t><<<grid, 256, 0, ctx->stream>>>(gg);
      AMTK_CUDA(cudaGetLastError());
      ctx->launches += 1;
    }
    return 1;
  }
  if (clip->bytes_per_sample == 1 && ctx->knobs.comb_mma) return launch_comb_mma(ctx, clip, win, lo, hi, prm, dcounts, out_row0);
  if (ctx->knobs.comb_ws && (clip->bytes_per_sample == 1 || (clip->bits_per_sample <= 10 && ctx->knobs.comb_ws10)))
    return launch_comb_ws(ctx, clip, win, lo, hi, prm, dcounts, out_row0);
  const int hY = clip->height, hC = clip->height >> clip->log_uvy;
  const int R = ctx->knobs.comb_R ? ctx->knobs.comb_R : pick_comb_R(hY, hC);
  int nvar = 0; const CombVariant* vars = comb_variants(&nvar); const CombVariant* V = nullptr;
  for (int i = 0; i < nvar; ++i) if (vars[i].R == R && vars[i].strip == ctx->knobs.comb_strip && vars[i].stages == ctx->knobs.comb_stages && vars[i].sync == ctx->knobs.comb_sync) V = &vars[i];
  if (!V) AMTK_FAIL("comb: no kernel variant for the requested AMTK_COMB_* settings");
  const int bps = clip->bytes_per_sample;
  if (bps == 2 && !V->kernel16) AMTK_FAIL("comb: the selected AMTK_COMB_* variant has no 16-bit kernel");
  const int twe = kCombTW / bps;                 // samples per tile row
  CombArgs args;
  memset(&args, 0, sizeof(args));
  // Chroma width 960 = 7.5 tiles: the 64-pixel remainders of U and V share ONE tile (two half-width TMA boxes)
  // instead of two half-empty ones.
  const int wC = clip->width >> clip->log_uvx;
  const int rem = wC % twe;
  const bool merge_uv = ctx->knobs.comb_merge_uv && rem > 0 && rem <= twe / 2 && (V->boxH * (kCombTW / 2)) % 128 == 0;
  int tile0 = 0;
  for (int pl = 0; pl < 4; ++pl) {
    CombPlane& P = args.plane[pl];
    const bool chroma = pl != 0;
    P.W = chroma ? wC : clip->width;
    P.H = chroma ? hC : hY;
    P.tilesX = (P.W + twe - 1) / twe; P.tilesY = (P.H + V->TH - 1) / V->TH;
    if (merge_uv && (pl == 1 || pl == 2)) P.tilesX -= 1;           // remainder column handled by the pseudo plane
    if (pl == 3) { P.tilesX = merge_uv ? 1 : 0; if (!merge_uv) P.tilesY = 0; }
    P.tile0 = tile0; tile0 += P.tilesX * P.tilesY;
    P.cls = chroma ? 1 : 0;
    const int thM = chroma ? prm->th_move_c : prm->th_move_y;
    const int thS = chroma ? prm->th_shima_c : prm->th_shima_y, thL = chroma ? prm->th_lshima_c : prm->th_lshima_y;
    if (bps == 1) {
      P.thM = (unsigned)(0x80 - thM) * 0x01010101u;
      P.thS = (unsigned)thS * 0x00010001u;       // integer k in [1,2047] IS the fp16 bit pattern of k*2^-24
      P.thL = (unsigned)thL * 0x00010001u;
    } else {
      P.thM = (unsigned)(0x8000 - thM) * 0x00010001u;
      const float fs = (float)thS, fl = (float)thL;
      memcpy(&P.thS, &fs, 4); memcpy(&P.thL, &fl, 4);
    }
    if (pl == 3) break;
    const long long off = pl == 0 ? 0 : (pl == 1 ? clip->off_u : clip->off_v);
    const int pitch = pl ? clip->pitch_uv : clip->pitch_y;
    cuuint64_t gdim[3] = { (cuuint64_t)P.W, (cuuint64_t)P.H, (cuuint64_t)win.count };
    cuuint64_t gstr[2] = { (cuuint64_t)pitch, (cuuint64_t)clip->frame_stride };
    for (int half = 0; half < (pl && merge_uv ? 2 : 1); ++half) {
      cuuint32_t box[3] = { (cuuint32_t)(half ? twe / 2 : twe), (cuuint32_t)V->boxH, 1u };
      CUtensorMap* m = half ? &args.map_half[pl - 1] : &args.map[pl];
      CUresult r = encode_map(ctx, m, bps == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, win.dev_base + off, gdim, gstr, box,
                              CU_TENSOR_MAP_SWIZZLE_NONE, comb_l2_promotion(ctx));
      if (r != CUDA_SUCCESS) AMTK_FAIL("cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
    }
  }
  args.half_x = wC - rem;
  const int ntiles = tile0;
  const int nf = hi - lo;
  // ---- static partition of (tile, frame) pairs over the resident CTAs: tile-major, frame-minor, equal shares.
  // A tile-frame costs the same wherever it lies (the kernel is issue/latency bound per warp, and tile shapes are
  // chosen so that bands are full), so equal counts = equal time; each CTA touches at most ~2 tiles.
  int occ = 0;
  void (*kern)(const CombArgs) = bps == 1 ? V->kernel : V->kernel16;
  AMTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, V->smem));
  AMTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, V->threads, V->smem));
  if (occ < 1) AMTK_FAIL("comb kernel does not fit on an SM");
  if (ctx->knobs.comb_ctas > 0) occ = std::min(occ, ctx->knobs.comb_ctas);
  const long long total = (long long)ntiles * nf;
  int grid = (int)std::min<long long>((long long)ctx->sm_count * occ, total);
  std::vector<CombSegment> segs;
  // "lock-step" partition: every tile is cut into the same C frame ranges, so neighbouring tiles stream the same
  // frames at the same time and share halo rows / straddled 128-byte lines through L2.  Used when the plane pitch
  // makes tile rows straddle lines (pitch % 128 != 0 on luma); costs a few idle CTA slots.
  const int chunks = std::max(1, std::min(nf, grid / std::max(1, ntiles)));
  // Since the tensor maps use 64-byte L2 promotion (straddled lines are no longer fetched whole) the equal-share
  // partition wins on every layout measured (tools/part_probe.py); lock-step stays available through the knob.
  const bool lockstep = ctx->knobs.comb_part == 1;
  if (lockstep) grid = chunks * ntiles;
  std::vector<int> seg_start((size_t)grid + 1, 0);
  if (lockstep) {
    for (int b = 0; b < grid; ++b) {                 // CTA b = (chunk c, tile t), tile-minor so that co-resident CTAs are neighbours
      const int c = b / ntiles, t = b % ntiles;
      const int f0 = (int)((long long)nf * c / chunks), f1 = (int)((long long)nf * (c + 1) / chunks);
      seg_start[b] = (int)segs.size();
      if (f1 > f0) segs.push_back(CombSegment{ t, lo - win.first + f0, lo - win.first + f1 });
    }
  } else
  for (int b = 0; b < grid; ++b) {
    const long long lo_i = total * b / grid, hi_i = total * (b + 1) / grid;     // [lo_i, hi_i) of the tile-major order
    seg_start[b] = (int)segs.size();
    long long i = lo_i;
    while (i < hi_i) {
      const int t = (int)(i / nf), f = (int)(i % nf);
      const int take = (int)std::min<long long>(nf - f, hi_i - i);
      segs.push_back(CombSegment{ t, lo - win.first + f, lo - win.first + f + take });
      i += take;
    }
  }
  seg_start[grid] = (int)segs.size();
  const size_t seg_bytes = segs.size() * sizeof(CombSegment), st_bytes = seg_start.size() * sizeof(int);
  const size_t st_off = (seg_bytes + 255) & ~(size_t)255;
  if (!ctx->small.ensure(st_off + st_bytes)) return 0;
  AMTK_CUDA(cudaMemcpyAsync(ctx->small.at(), segs.data(), seg_bytes, cudaMemcpyHostToDevice, ctx->stream));
  AMTK_CUDA(cudaMemcpyAsync(ctx->small.at(st_off), seg_start.data(), st_bytes, cudaMemcpyHostToDevice, ctx->stream));
  // pageable host vectors: the async copies above have completed their host reads on return
  args.segs = ctx->small.at<const CombSegment>();
  args.seg_start = ctx->small.at<const int>(st_off);
  args.counts = dcounts;
  args.out_frame0 = out_row0 - win.first;
  return comb_launch(ctx, dcounts + (size_t)(lo - out_row0) * 12, nf, [&] { kern<<<grid, V->threads, V->smem, ctx->stream>>>(args); });
}

// ---------------------------------------------------------------------------------------------------------
// temporal noise reduction launch
// ---------------------------------------------------------------------------------------------------------
// Byte span [lo, hi) a clip's frames touch (plane offsets may be negative or out of order: V-first layouts).
static void clip_span(const amtk_clip* c, uintptr_t* lo, uintptr_t* hi) {
  const int hc = c->height >> c->log_uvy, rowc = (c->width >> c->log_uvx) * c->bytes_per_sample;
  const long long ends[3] = { (long long)c->pitch_y * (c->height - 1) + (long long)c->width * c->bytes_per_sample,
                              c->off_u + (long long)c->pitch_uv * (hc - 1) + rowc, c->off_v + (long long)c->pitch_uv * (hc - 1) + rowc };
  const long long first = std::min<long long>(0, std::min(c->off_u, c->off_v));
  const long long last = std::max(ends[0], std::max(ends[1], ends[2])) + (long long)(c->num_frames - 1) * c->frame_stride;
  *lo = reinterpret_cast<uintptr_t>(c->base) + first; *hi = reinterpret_cast<uintptr_t>(c->base) + last;
}

// Filters output frames [lo, hi) of the clip from the resident window `win` into `dbase` (destination of frame lo, laid
// out like `dl`).  ring: `win` is a ring of win.count slots holding frame f in slot f mod win.count (amtk_tnr_stream).
// dl->bits_per_sample above src's widens the output by the difference (the widening kernels, with or without ring).
static int launch_tnr(amtk_ctx* ctx, const amtk_clip* src, const Window& win, const amtk_clip* dl, uint8_t* dbase,
                      int lo, int hi, const amtk_tnr_params* p, bool ring = false) {
  TnrArgs a;
  a.src = win.dev_base; a.src_stride = src->frame_stride; a.s_offu = src->off_u; a.s_offv = src->off_v;
  a.s_pitchY = src->pitch_y; a.s_pitchUV = src->pitch_uv; a.src_first = win.first; a.src_count = win.count;
  a.dst = dbase; a.dst_stride = dl->frame_stride; a.d_offu = dl->off_u; a.d_offv = dl->off_v;
  a.d_pitchY = dl->pitch_y; a.d_pitchUV = dl->pitch_uv;
  a.W = src->width; a.H = src->height; a.N = src->num_frames;
  a.lo = lo; a.hi = hi;
  a.thresh = p->threshold << (src->bits_per_sample - 8);      // VideoFilter.hpp:120; at src_bits also when widening
  a.interlaced = p->interlaced;
  const int bps = src->bytes_per_sample, obps = dl->bytes_per_sample, nl = 16 / obps;
  const int shift = dl->bits_per_sample - src->bits_per_sample;
  const TnrWiden wd{ ldexpf(0.5f, -shift), ldexpf(1.0f, shift) };
  const int sa = 16 * bps / obps;                              // source bytes of a group's luma row
  auto al = [](long long v, int m) { return (v & (m - 1)) == 0; };
  a.vec = al((long long)reinterpret_cast<uintptr_t>(win.dev_base), sa) && al(a.src_stride, sa) && al(a.s_pitchY, sa) &&
          al(a.s_offu, sa / 2) && al(a.s_offv, sa / 2) && al(a.s_pitchUV, sa / 2) &&
          al((long long)reinterpret_cast<uintptr_t>(dbase), 16) && al(a.dst_stride, 16) && al(a.d_pitchY, 16) &&
          al(a.d_offu, 8) && al(a.d_offv, 8) && al(a.d_pitchUV, 8);
  const long long groups = (long long)((a.W + nl - 1) / nl) * (a.H >> 1);
  // runs of frames per thread: enough threads for about two full waves of 2048 per SM; longer runs re-read fewer halos
  const long long want = (long long)ctx->sm_count * 2048 * 2;
  const int n = hi - lo;
  int nruns = (int)std::max<long long>(1, std::min<long long>({ (long long)n, (want + groups - 1) / groups, 65535LL }));
  a.run = (n + nruns - 1) / nruns;
  nruns = (n + a.run - 1) / a.run;
  const dim3 grid((unsigned)((groups + kTnrThreads - 1) / kTnrThreads), (unsigned)nruns);
  const int d = p->temporal_distance;
#define AMTK_TNR_CASE(TI, TO, RING, WIDEN)                                                                    \
  switch (d) {                                                                                                \
    case 0: tnr_kernel<TI, TO, 0, RING, WIDEN><<<grid, kTnrThreads, 0, ctx->stream>>>(a, wd); break;         \
    case 1: tnr_kernel<TI, TO, 1, RING, WIDEN><<<grid, kTnrThreads, 0, ctx->stream>>>(a, wd); break;         \
    case 2: tnr_kernel<TI, TO, 2, RING, WIDEN><<<grid, kTnrThreads, 0, ctx->stream>>>(a, wd); break;         \
    case 3: tnr_kernel<TI, TO, 3, RING, WIDEN><<<grid, kTnrThreads, 0, ctx->stream>>>(a, wd); break;         \
    case 4: tnr_kernel<TI, TO, 4, RING, WIDEN><<<grid, kTnrThreads, 0, ctx->stream>>>(a, wd); break;         \
    case 5: tnr_kernel<TI, TO, 5, RING, WIDEN><<<grid, kTnrThreads, 0, ctx->stream>>>(a, wd); break;         \
    case 6: tnr_kernel<TI, TO, 6, RING, WIDEN><<<grid, kTnrThreads, 0, ctx->stream>>>(a, wd); break;         \
    case 7: tnr_kernel<TI, TO, 7, RING, WIDEN><<<grid, kTnrThreads, 0, ctx->stream>>>(a, wd); break;         \
    default: tnr_general_kernel<TI, TO, RING, WIDEN><<<grid, kTnrThreads, 0, ctx->stream>>>(a, d, wd); break;     \
  }
  static_assert(kTnrMaxTemplD == 7, "the switch above lists every register-window kernel");
  if (shift == 0) {
    if (bps == 1) { if (ring) { AMTK_TNR_CASE(uint8_t, uint8_t, true, false) } else { AMTK_TNR_CASE(uint8_t, uint8_t, false, false) } }
    else { if (ring) { AMTK_TNR_CASE(uint16_t, uint16_t, true, false) } else { AMTK_TNR_CASE(uint16_t, uint16_t, false, false) } }
  } else {
    if (bps == 1) { if (ring) { AMTK_TNR_CASE(uint8_t, uint16_t, true, true) } else { AMTK_TNR_CASE(uint8_t, uint16_t, false, true) } }
    else { if (ring) { AMTK_TNR_CASE(uint16_t, uint16_t, true, true) } else { AMTK_TNR_CASE(uint16_t, uint16_t, false, true) } }
  }
#undef AMTK_TNR_CASE
  AMTK_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return 1;
}

// The filter parameters amtk_tnr_frames and the frame stream accept.
static bool tnr_params_ok(const amtk_tnr_params* p) {
  if (p->temporal_distance < 0 || p->temporal_distance > kTnrMaxD) { set_error("tnr: temporal_distance must be in [0,63]"); return false; }
  if (p->threshold < 0 || p->threshold > 65535) { set_error("tnr: threshold must be in [0,65535]"); return false; }
  if (p->interlaced != 0 && p->interlaced != 1) { set_error("tnr: interlaced must be 0 or 1"); return false; }
  return true;
}

// The source formats the filter accepts (c already passed validate_clip).
static bool tnr_format_ok(const amtk_clip* c, int interlaced) {
  if (c->log_uvx != 1 || c->log_uvy != 1) { set_error("tnr: only 4:2:0 clips are supported"); return false; }
  const int bits = c->bits_per_sample;
  if (!(c->bytes_per_sample == 1 ? bits == 8 : (bits == 10 || bits == 12 || bits == 14 || bits == 16))) {
    set_error("tnr: bits_per_sample must be 8 (1-byte samples) or 10, 12, 14, 16 (2-byte samples)"); return false;
  }
  if ((c->width & 1) || (c->height & 1)) { set_error("tnr: width and height must be even"); return false; }
  if (interlaced && (c->height & 3)) { set_error("tnr: interlaced clips need a height that is a multiple of 4"); return false; }
  return true;
}

// Per-plane 2-D copies of the sample bytes of one frame (row padding untouched), on `st`; host to host: row by row on the
// CPU, done on return.
static int copy_frame_planes(uint8_t* dst, const amtk_clip& dl, const uint8_t* src, const amtk_clip& sl, cudaMemcpyKind kind, cudaStream_t st) {
  const size_t rowY = (size_t)sl.width * sl.bytes_per_sample, rowC = (size_t)(sl.width >> sl.log_uvx) * sl.bytes_per_sample;
  const int hc = sl.height >> sl.log_uvy;
  if (kind == cudaMemcpyHostToHost) {
    // planes of equal pitch in one copy (rows and the padding between them): one large memcpy streams, where row-sized
    // ones ran at half the rate for 2-byte 1080p frames
    auto plane = [](uint8_t* d, int dp, const uint8_t* s, int sp, size_t row, int rows) {
      if (rows <= 0) return;
      if (dp == sp) { memcpy(d, s, (size_t)(rows - 1) * (size_t)dp + row); return; }
      for (int y = 0; y < rows; ++y) memcpy(d + (size_t)y * dp, s + (size_t)y * sp, row);
    };
    plane(dst, dl.pitch_y, src, sl.pitch_y, rowY, sl.height);
    plane(dst + dl.off_u, dl.pitch_uv, src + sl.off_u, sl.pitch_uv, rowC, hc);
    plane(dst + dl.off_v, dl.pitch_uv, src + sl.off_v, sl.pitch_uv, rowC, hc);
    return 1;
  }
  AMTK_CUDA(cudaMemcpy2DAsync(dst, dl.pitch_y, src, sl.pitch_y, rowY, sl.height, kind, st));
  AMTK_CUDA(cudaMemcpy2DAsync(dst + dl.off_u, dl.pitch_uv, src + sl.off_u, sl.pitch_uv, rowC, hc, kind, st));
  AMTK_CUDA(cudaMemcpy2DAsync(dst + dl.off_v, dl.pitch_uv, src + sl.off_v, sl.pitch_uv, rowC, hc, kind, st));
  return 1;
}

// One frame of c's size at the given sample format in a frame stream's own layout: 16-byte aligned pitches and planes and
// a 256-byte frame stride, so the kernels' vector and TMA paths run whatever the layout of the frames sent.
static amtk_clip stream_frame_layout(const amtk_clip& c, int bytes_per_sample, int bits_per_sample) {
  amtk_clip f = c;
  const int hc = f.height >> f.log_uvy;
  f.bytes_per_sample = bytes_per_sample; f.bits_per_sample = bits_per_sample;
  f.pitch_y = (f.width * bytes_per_sample + 15) & ~15;
  f.pitch_uv = ((f.width >> f.log_uvx) * bytes_per_sample + 15) & ~15;
  f.off_u = (int64_t)f.pitch_y * f.height;
  f.off_v = f.off_u + (int64_t)f.pitch_uv * hc;
  f.frame_stride = (f.off_v + (int64_t)f.pitch_uv * hc + 255) & ~(int64_t)255;
  f.base = nullptr; f.num_frames = 1; f.on_device = 1;
  return f;
}

// The Y, U and V rectangles of one frame packed into one slot, Y then U then V (CopyYV12's order, LogoScan.hpp:893-902):
// the frame streams keep only these bytes of each frame.  (x, y, w, h) is the luma rectangle; the chroma rectangles are
// (x >> lx, y >> ly, w >> lx, h >> ly).  Pitches and plane offsets are bytes inside the slot.  A luma-only slot (the logo
// scan stream: ScanFrame reads nothing else) holds the Y rectangle alone.
struct RectPack {
  int x = 0, y = 0, w = 0, h = 0, lx = 1, ly = 1, bps = 1;
  bool luma_only = false;
  long long pitchY = 0, pitchC = 0, offU = 0, offV = 0, stride = 0;      // stride: slot to slot (a multiple of 16)
  long long payload() const { return ((long long)w * h + (luma_only ? 0 : 2LL * (w >> lx) * (h >> ly))) * bps; }
};

// Slot layout with the given luma pitch alignment (bytes); chroma rows are packed tightly.
static RectPack rect_pack(int x, int y, int w, int h, int lx, int ly, int bps, int pitch_align, bool luma_only = false) {
  RectPack r;
  r.x = x; r.y = y; r.w = w; r.h = h; r.lx = lx; r.ly = ly; r.bps = bps; r.luma_only = luma_only;
  r.pitchY = ((long long)w * bps + pitch_align - 1) / pitch_align * pitch_align;
  r.pitchC = luma_only ? 0 : (long long)(w >> lx) * bps;
  r.offU = r.pitchY * h; r.offV = r.offU + r.pitchC * (h >> ly);
  r.stride = (r.offV + r.pitchC * (h >> ly) + 15) & ~15LL;
  return r;
}

// `nframes` packed rectangles, `stride` bytes apart from `base` in device memory, as a clip of frames of format `fmt`
// that hold the rectangle at (0, 0).  A luma-only pack gives a clip without chroma rows (pitch_uv 0) for the evaluation
// kernels, which read luma alone.
static amtk_clip slot_view(const amtk_clip& fmt, const RectPack& r, const uint8_t* base, long long stride, int nframes) {
  amtk_clip v = fmt;
  v.base = base; v.frame_stride = stride; v.off_u = r.offU; v.off_v = r.offV;
  v.width = (int)(r.pitchY / r.bps); v.height = r.h; v.pitch_y = (int)r.pitchY; v.pitch_uv = (int)r.pitchC;
  v.num_frames = nframes; v.on_device = 1;
  return v;
}

// Copies the rectangles of one-frame clip `frame` into the packed slot (to_slot) or back out of it.  Host frames: row by
// row on the CPU, so `slot` is host memory.  Device frames: 2-D copies on `st`, so `slot` is device memory.  row_step: the
// bytes from one luma row to the next as the frame is addressed (0: its pitch_y).
static int rect_copy(const RectPack& r, const amtk_clip* frame, uint8_t* slot, bool to_slot, cudaStream_t st, long long row_step = 0) {
  uint8_t* base = const_cast<uint8_t*>(reinterpret_cast<const uint8_t*>(frame->base));
  for (int p = 0; p < (r.luma_only ? 1 : 3); ++p) {
    const int rw = (p ? r.w >> r.lx : r.w) * r.bps, rh = p ? r.h >> r.ly : r.h;
    const long long fp = p ? frame->pitch_uv : (row_step > 0 ? row_step : frame->pitch_y), sp = p ? r.pitchC : r.pitchY;
    uint8_t* f = base + (p == 0 ? 0 : (p == 1 ? frame->off_u : frame->off_v)) +
                 (long long)(p ? r.y >> r.ly : r.y) * fp + (long long)(p ? r.x >> r.lx : r.x) * r.bps;
    uint8_t* s = slot + (p == 0 ? 0 : (p == 1 ? r.offU : r.offV));
    if (frame->on_device) {
      AMTK_CUDA(to_slot ? cudaMemcpy2DAsync(s, (size_t)sp, f, (size_t)fp, (size_t)rw, (size_t)rh, cudaMemcpyDeviceToDevice, st)
                        : cudaMemcpy2DAsync(f, (size_t)fp, s, (size_t)sp, (size_t)rw, (size_t)rh, cudaMemcpyDeviceToDevice, st));
    } else {
      for (int yy = 0; yy < rh; ++yy) {
        if (to_slot) memcpy(s + yy * sp, f + yy * fp, (size_t)rw);
        else memcpy(f + yy * fp, s + yy * sp, (size_t)rw);
      }
    }
  }
  return 1;
}

// Calls copy(k, e) for each run [k, e) of consecutive slots in [lo, hi) that host[] marks as filled from host memory, so
// a frame stream uploads each run in one copy.  Stops at the first copy that fails.
template <class Copy> static int for_each_host_run(const std::vector<uint8_t>& host, int lo, int hi, Copy copy) {
  for (int k = lo; k < hi;) {
    if (!host[(size_t)k]) { ++k; continue; }
    int e = k;
    while (e < hi && host[(size_t)e]) ++e;
    if (!copy(k, e)) return 0;
    k = e;
  }
  return 1;
}

// A frame stream's batch: a device buffer, its pinned twin (streams that download into one) and the event recorded after
// the batch's work.  The stream's batch type derives from it and adds its own fields.
struct StreamBatch { DevBuf<uint8_t> d; PinnedBuf<uint8_t> h; EventHandle done; };

// Batches whose outputs have all been received, kept for reuse.  Events are destroyed only with the pool, so raw event
// handles taken from its batches stay valid for the stream's life.
struct BatchPool {
  std::vector<StreamBatch> free;
  // A retired batch, or a new one of `bytes` (with a pinned twin when pinned_what names it); false on a CUDA error.
  bool take(StreamBatch* b, size_t bytes, const char* dev_what, const char* pinned_what) {
    if (!free.empty()) { *b = std::move(free.back()); free.pop_back(); return true; }
    StreamBatch n;
    if (!cuda_ok(cudaMalloc(n.d.put(), bytes), dev_what) ||
        (pinned_what && !cuda_ok(cudaHostAlloc(n.h.put(), bytes, cudaHostAllocDefault), pinned_what)) ||
        !cuda_ok(cudaEventCreateWithFlags(n.done.put(), cudaEventDisableTiming), "cudaEventCreate"))
      return false;
    *b = std::move(n);
    return true;
  }
  void give(StreamBatch&& b) { free.push_back(std::move(b)); }
};

static bool same_format(const amtk_clip& f, const amtk_clip* c) {
  return c->width == f.width && c->height == f.height && c->bytes_per_sample == f.bytes_per_sample &&
         c->bits_per_sample == f.bits_per_sample && c->log_uvx == f.log_uvx && c->log_uvy == f.log_uvy;
}

// A valid clip that describes exactly one frame, as every frame stream takes and returns them.
static bool one_frame(const amtk_clip* c, const char* stream, const char* what) {
  if (!validate_clip(c, true)) return false;
  if (c->num_frames != 1) { set_error(std::string(stream) + ": " + what + " must describe exactly one frame"); return false; }
  return true;
}

// `closed` is why a stream's calls fail (nullptr: open).  stream_open sets that reason as the error; stream_fail closes
// an open stream after a CUDA error.
static bool stream_open(const char* closed, const char* stream) {
  if (closed) set_error(std::string(stream) + ": closed (" + closed + ")");
  return !closed;
}
static int stream_fail(const char*& closed) {
  if (!closed) closed = "an earlier CUDA error";
  return 0;
}

// Deletes a frame stream when nothing of it can still be in flight: the context's stream (and `also`, a second stream it
// used) is idle.  When the device cannot be selected its work may still be running, and its memory is not freed.
template <class S> static void stream_destroy(S* s, cudaStream_t also = nullptr) {
  DevSelect ds(s->ctx);
  if (!ds.ok) return;
  if (also) cudaStreamSynchronize(also);
  cudaStreamSynchronize(s->ctx->stream);
  delete s;
}

static bool sample_bits_ok(const amtk_clip* c, const char* stream) {
  if (c->bytes_per_sample == 1 ? c->bits_per_sample == 8 : c->bits_per_sample > 8 && c->bits_per_sample <= 16) return true;
  set_error(std::string(stream) + ": bits_per_sample must be 8 for 1-byte samples and 9..16 for 2-byte samples");
  return false;
}

// The batches of the erase, logo scan and comb streams.  Frame f goes into slot f % B of batch buffer f / B; a batch buffer
// is `head` bytes (the batch's results, a multiple of 256, and what else the stream keeps before slot 0), then B slots
// `slot` bytes apart.  Host frames are written into the buffer's pinned twin and uploaded when the batch is launched,
// device frames into the buffer itself.  A launch ends in seal(): the download of a prefix of the buffer into the twin and
// the batch's event, the only thing a receive waits on.  Batch k may be received once batch k + 1 was launched (its
// download overlaps that batch's work) or once the input has ended, and goes back to the pool with its last output.
// After a CUDA error the stream is closed: every call but counts and destroy fails with the reason.
struct SlotBatch : StreamBatch { std::vector<uint8_t> host; };      // host[j]: slot j was filled from host memory

// Batch: SlotBatch, or a type derived from it that adds what the stream keeps per batch.
template <class Batch = SlotBatch> struct SlotStream {
  amtk_ctx* ctx = nullptr;
  const char* name;                         // "comb stream", ...: the prefix of its errors
  const char* batch_name;                   // "comb batch", ...: names the batch's CUDA calls in theirs
  int B = 1;
  const char* closed = nullptr;             // why every call but counts and destroy fails (nullptr: open)
  bool finished = false;                    // finish was called (streams that have one)
  bool have_fmt = false;
  amtk_clip fmt{};                          // the first frame's format
  size_t head = 0, slot = 0;                // bytes before slot 0; slot to slot
  std::deque<Batch> batches;                // batch first_batch, first_batch + 1, ... (not yet fully received)
  BatchPool pool;
  int first_batch = 0;
  int sent = 0, launched = 0, received = 0;
  int64_t h2d = 0, d2h = 0;
  SlotStream(const char* name_, const char* batch_name_) : name(name_), batch_name(batch_name_) {}

  // Sets the reason as the error when the stream is closed; the calls that take input are closed by finish as well.
  bool open(bool takes_input) const {
    return stream_open(closed, name) && stream_open(takes_input && finished ? "finished" : nullptr, name);
  }
  int fail() { return stream_fail(closed); }
  std::string cuda_call(const char* fn) const { return std::string(fn) + "(" + batch_name + ")"; }

  // The batch buffer of frame f (allocated, or taken from the pool, when f is its first frame); nullptr on a CUDA error.
  Batch* batch_of(int f) {
    const int k = f / B - first_batch;
    while ((int)batches.size() <= k) {
      Batch b;
      if (!pool.take(&b, head + (size_t)B * slot, cuda_call("cudaMalloc").c_str(), cuda_call("cudaHostAlloc").c_str())) return nullptr;
      b.host.assign((size_t)B, 0);
      batches.push_back(std::move(b));
    }
    return &batches[(size_t)k];
  }
  Batch& batch(int k) { return batches[(size_t)(k - first_batch)]; }
  size_t slot_at(int j) const { return head + (size_t)j * slot; }      // byte offset of slot j in a batch buffer

  // Uploads the host slots among slots [lo, hi) of b, one copy per run; `payload` of each slot's bytes are frame data.
  int upload(Batch& b, int lo, int hi, int64_t payload) {
    return for_each_host_run(b.host, lo, hi, [&](int j, int e) {
      const size_t off = slot_at(j);
      if (slot > 0) AMTK_CUDA(cudaMemcpyAsync(b.d + off, b.h + off, (size_t)(e - j) * slot, cudaMemcpyHostToDevice, ctx->stream));
      h2d += (int64_t)(e - j) * payload;
      return 1;
    });
  }

  // The end of a launch: downloads the first `bytes` of b (`counted` of them results) and records its event.
  int seal(Batch& b, size_t bytes, int64_t counted) {
    AMTK_CUDA(cudaMemcpyAsync(b.h, b.d, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    d2h += counted;
    AMTK_CUDA(cudaEventRecord(b.done, ctx->stream));
    launched += 1;
    return 1;
  }

  // How many of the stream's outputs may be received; `total` is all of them once the input has `ended`.
  int ready(bool ended, int total) const { return ended ? total : std::min(total, std::max(0, launched - 1) * B); }

  // The front batch with its work complete; nullptr, and the stream closed, on a CUDA error.
  Batch* front() {
    Batch& b = batches.front();
    if (!cuda_ok(cudaEventSynchronize(b.done), cuda_call("cudaEventSynchronize").c_str())) { fail(); return nullptr; }
    return &b;
  }

  // After outputs of the front batch were received: the batch goes back to the pool with the last of its `ready` ones.
  void retire(int ready) {
    if (received != std::min(ready, (first_batch + 1) * B)) return;
    pool.give(std::move(batches.front()));
    batches.pop_front();
    first_batch += 1;
  }

  void counts(int* sent_, int* received_, int64_t* h2d_bytes, int64_t* d2h_bytes) const {
    std::lock_guard<std::recursive_mutex> lock(ctx->mu);
    if (sent_) *sent_ = sent;
    if (received_) *received_ = received;
    if (h2d_bytes) *h2d_bytes = h2d;
    if (d2h_bytes) *d2h_bytes = d2h;
  }
};

static std::once_flag g_driver_once;
static amtk_encode_tiled_fn g_encode = nullptr;

}  // namespace amtk

using namespace amtk;

// =============================================================================================================
// C ABI
// =============================================================================================================
extern "C" {

const char* amtk_last_error(void) { return g_error.c_str(); }
int amtk_version(void) { return 100; }

int amtk_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int amtk_ctx_create(int device, void* cuda_stream, amtk_ctx** out) {
  if (!out) AMTK_FAIL("amtk_ctx_create: out is null");
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); AMTK_FAIL("no CUDA device: this library has no CPU fallback"); }
  if (device < 0 || device >= n) AMTK_FAIL("amtk_ctx_create: bad device ordinal");
  int prev = 0; AMTK_CUDA(cudaGetDevice(&prev));
  AMTK_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop; AMTK_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) { cudaSetDevice(prev); AMTK_FAIL("this build targets sm_90a (Hopper H100) only"); }
  amtk_ctx* c = new amtk_ctx();
  c->device = device; c->sm_count = prop.multiProcessorCount;
  // NULL selects the legacy default stream (which orders with every blocking stream, e.g. torch's default one)
  c->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
  bool ok = cuda_ok(cudaStreamCreateWithFlags(c->copy_stream.put(), cudaStreamNonBlocking), "cudaStreamCreate(copy)") &&
            cuda_ok(cudaStreamCreateWithFlags(c->side_stream.put(), cudaStreamNonBlocking), "cudaStreamCreate(side)") &&
            cuda_ok(cudaStreamCreateWithFlags(c->side_stream2.put(), cudaStreamNonBlocking), "cudaStreamCreate(side2)") &&
            cuda_ok(cudaEventCreateWithFlags(c->ev_fork.put(), cudaEventDisableTiming), "cudaEventCreate") &&
            cuda_ok(cudaEventCreateWithFlags(c->ev_join1.put(), cudaEventDisableTiming), "cudaEventCreate") &&
            cuda_ok(cudaEventCreateWithFlags(c->ev_join2.put(), cudaEventDisableTiming), "cudaEventCreate");
  for (int b = 0; b < 2 && ok; ++b) {
    ok = cuda_ok(cudaEventCreateWithFlags(c->ev_copy[b].put(), cudaEventDisableTiming), "cudaEventCreate") &&
         cuda_ok(cudaEventCreateWithFlags(c->ev_done[b].put(), cudaEventDisableTiming), "cudaEventCreate");
  }
  std::call_once(g_driver_once, [] {
    void* fn = nullptr; cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      g_encode = reinterpret_cast<amtk_encode_tiled_fn>(fn);
    else cudaGetLastError();
  });
  c->encode_tiled = g_encode;
  // per-context tuning knobs (defaults are the measured best, DESIGN.md section 6; env AMTK_* overrides them for tools/tune_comb.py)
  if (const char* e = getenv("AMTK_COMB_STRIP")) c->knobs.comb_strip = atoi(e);
  if (const char* e = getenv("AMTK_COMB_STAGES")) c->knobs.comb_stages = atoi(e);
  if (const char* e = getenv("AMTK_COMB_R")) c->knobs.comb_R = atoi(e);
  if (const char* e = getenv("AMTK_COMB_CTAS")) c->knobs.comb_ctas = atoi(e);
  if (const char* e = getenv("AMTK_COMB_SYNC")) c->knobs.comb_sync = atoi(e);
  if (const char* e = getenv("AMTK_COMB_GENERIC")) c->knobs.comb_generic = atoi(e);
  if (const char* e = getenv("AMTK_COMB_MERGE_UV")) c->knobs.comb_merge_uv = atoi(e);
  if (const char* e = getenv("AMTK_COMB_PART")) c->knobs.comb_part = atoi(e);
  if (const char* e = getenv("AMTK_EVAL_WAVES")) c->knobs.eval_waves = std::max(1, atoi(e));
  if (const char* e = getenv("AMTK_COMB_L2")) c->knobs.comb_l2 = atoi(e);
  if (const char* e = getenv("AMTK_COMB_WS")) c->knobs.comb_ws = atoi(e);
  if (const char* e = getenv("AMTK_COMB_WS_STAGES")) c->knobs.comb_ws_stages = atoi(e);
  if (const char* e = getenv("AMTK_COMB_ITEM")) c->knobs.comb_item = atoi(e);
  if (const char* e = getenv("AMTK_COMB_TAIL")) c->knobs.comb_tail = atoi(e);
  if (const char* e = getenv("AMTK_COMB_MMA")) c->knobs.comb_mma = atoi(e);
  if (const char* e = getenv("AMTK_COMB_WS10")) c->knobs.comb_ws10 = atoi(e);
  if (const char* e = getenv("AMTK_EVAL_CW")) c->knobs.eval_cw = atoi(e);
  if (const char* e = getenv("AMTK_EVAL_PAR")) c->knobs.eval_par = atoi(e);
  if (const char* e = getenv("AMTK_COMB_WS_WARPS")) c->knobs.comb_ws_warps = atoi(e);
  if (const char* e = getenv("AMTK_COMB_WS_PF")) c->knobs.comb_ws_prefetch = atoi(e);
  if (const char* e = getenv("AMTK_COMB_WS_BAND")) c->knobs.comb_ws_band = atoi(e);
  cudaSetDevice(prev);
  if (!ok) { amtk_ctx_destroy(c); return 0; }
  *out = c;
  return 1;
}

void amtk_ctx_destroy(amtk_ctx* c) {
  if (!c) return;
  int prev = 0; cudaGetDevice(&prev); cudaSetDevice(c->device);
  // nothing the context's buffers and events serve may still be in flight when they are released
  for (cudaStream_t s : { c->stream, c->copy_stream.get(), c->side_stream.get(), c->side_stream2.get() })
    if (s) cudaStreamSynchronize(s);
  delete c;
  cudaSetDevice(prev);
}

int amtk_ctx_synchronize(amtk_ctx* c) {
  if (!c) AMTK_FAIL("null context");
  DevSelect ds(c); if (!ds.ok) return 0;
  AMTK_CUDA(cudaStreamSynchronize(c->stream));
  return 1;
}
int64_t amtk_ctx_launch_count(const amtk_ctx* c) { return c ? c->launches : 0; }
int64_t amtk_ctx_last_h2d_bytes(const amtk_ctx* c) { return c ? c->h2d_bytes_last : 0; }

int amtk_ctx_set_kernel_timing(amtk_ctx* c, int enable) {
  if (!c) AMTK_FAIL("null context");
  c->timing = enable != 0;
  return 1;
}

int amtk_ctx_get_kernel_timing(amtk_ctx* c, double* ms_total, int64_t* launches, int reset) {
  if (!c) AMTK_FAIL("null context");
  DevSelect ds(c); if (!ds.ok) return 0;
  AMTK_CUDA(cudaStreamSynchronize(c->stream));
  for (auto& ev : c->timing_events) {
    float ms = 0.0f;
    AMTK_CUDA(cudaEventElapsedTime(&ms, ev.first, ev.second));
    c->timing_ms += ms; c->timing_count += 1;
    c->timing_pool.push_back(std::move(ev));
  }
  c->timing_events.clear();
  if (ms_total) *ms_total = c->timing_ms;
  if (launches) *launches = c->timing_count;
  if (reset) { c->timing_ms = 0.0; c->timing_count = 0; }
  return 1;
}

int amtk_probe_read_ms(amtk_ctx* c, const void* ptr, size_t bytes, int reps, double* ms_out) {
  if (!c || !ptr || !ms_out || reps < 1) AMTK_FAIL("amtk_probe_read_ms: bad argument");
  if (reinterpret_cast<uintptr_t>(ptr) & 15) AMTK_FAIL("amtk_probe_read_ms: pointer must be 16-byte aligned");
  DevSelect ds(c); if (!ds.ok) return 0;
  if (!c->small.ensure(256)) return 0;
  EventHandle e0, e1;
  AMTK_CUDA(cudaEventCreate(e0.put())); AMTK_CUDA(cudaEventCreate(e1.put()));
  const int grid = c->sm_count * 8;
  unsigned* sink = c->small.at<unsigned>();
  read_probe_kernel<<<grid, 256, 0, c->stream>>>(reinterpret_cast<const uint4*>(ptr), bytes / 16, sink);
  AMTK_CUDA(cudaEventRecord(e0, c->stream));
  for (int i = 0; i < reps; ++i) read_probe_kernel<<<grid, 256, 0, c->stream>>>(reinterpret_cast<const uint4*>(ptr), bytes / 16, sink);
  AMTK_CUDA(cudaEventRecord(e1, c->stream));
  AMTK_CUDA(cudaEventSynchronize(e1));
  float ms = 0; AMTK_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  AMTK_CUDA(cudaGetLastError());
  *ms_out = ms / reps;
  return 1;
}

int amtk_host_alloc(size_t bytes, void** out) {
  if (!out) AMTK_FAIL("amtk_host_alloc: out is null");
  AMTK_CUDA(cudaHostAlloc(out, bytes, cudaHostAllocDefault));
  return 1;
}
void amtk_host_free(void* p) { if (p) cudaFreeHost(p); }

int amtk_device_alloc(amtk_ctx* c, size_t bytes, void** out) {
  if (!c || !out) AMTK_FAIL("amtk_device_alloc: null argument");
  DevSelect ds(c); if (!ds.ok) return 0;
  AMTK_CUDA(cudaMalloc(out, bytes));
  return 1;
}
void amtk_device_free(amtk_ctx* c, void* p) {
  if (!c || !p) return;
  DevSelect ds(c);
  cudaStreamSynchronize(c->stream);
  cudaFree(p);
}
int amtk_memcpy_h2d(amtk_ctx* c, void* dst, const void* src, size_t bytes) {
  if (!c || !dst || !src) AMTK_FAIL("amtk_memcpy_h2d: null argument");
  DevSelect ds(c); if (!ds.ok) return 0;
  AMTK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->stream));
  AMTK_CUDA(cudaStreamSynchronize(c->stream));
  return 1;
}
int amtk_memcpy_d2d(amtk_ctx* c, void* dst, const void* src, size_t bytes) {
  if (!c || !dst || !src) AMTK_FAIL("amtk_memcpy_d2d: null argument");
  DevSelect ds(c); if (!ds.ok) return 0;
  AMTK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, c->stream));
  AMTK_CUDA(cudaStreamSynchronize(c->stream));
  return 1;
}
int amtk_memcpy_d2h(amtk_ctx* c, void* dst, const void* src, size_t bytes) {
  if (!c || !dst || !src) AMTK_FAIL("amtk_memcpy_d2h: null argument");
  DevSelect ds(c); if (!ds.ok) return 0;
  AMTK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
  AMTK_CUDA(cudaStreamSynchronize(c->stream));
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// logos
// ---------------------------------------------------------------------------------------------------------
// The two upload steps fill local buffers and hand them to the logo only once every copy has succeeded: a failed upload
// leaves the logo as it was, so the next evaluation tries again.
static int logo_upload_planes(amtk_logo* l) {
  amtk::HostLogo& h = l->host;
  const size_t ny = h.ySize() * sizeof(float), nc = h.cSize() * sizeof(float);
  const float* src[6] = { h.aY(), h.bY(), h.aU(), h.bU(), h.aV(), h.bV() };
  DevBuf<float> d[6];
  for (int i = 0; i < 6; ++i) {
    const size_t n = i < 2 ? ny : nc;
    AMTK_CUDA(cudaMalloc(d[i].put(), std::max<size_t>(n, 16)));
    AMTK_CUDA(cudaMemcpy(d[i], src[i], n, cudaMemcpyHostToDevice));
  }
  DevBuf<float>* dst[6] = { &l->dA, &l->dB, &l->dAU, &l->dBU, &l->dAV, &l->dBV };
  for (int i = 0; i < 6; ++i) *dst[i] = std::move(d[i]);
  return 1;
}

static int logo_upload_tables(amtk_logo* l) {
  amtk::HostLogo& h = l->host;
  const int count = h.count();
  DevBuf<uint32_t> pix; DevBuf<float> taps; DevBuf<float2> scales;
  if (count > 0) {
    std::vector<float> tapsT((size_t)25 * l->countPad, 0.0f);
    for (int c = 0; c < count; ++c) for (int t = 0; t < 25; ++t) tapsT[(size_t)t * l->countPad + c] = h.kernels[(size_t)c * 25 + t];
    AMTK_CUDA(cudaMalloc(pix.put(), (size_t)count * sizeof(uint32_t)));
    AMTK_CUDA(cudaMalloc(taps.put(), tapsT.size() * sizeof(float)));
    AMTK_CUDA(cudaMalloc(scales.put(), (size_t)count * 32 * sizeof(float2)));
    AMTK_CUDA(cudaMemcpy(pix, h.pix.data(), (size_t)count * sizeof(uint32_t), cudaMemcpyHostToDevice));
    AMTK_CUDA(cudaMemcpy(taps, tapsT.data(), tapsT.size() * sizeof(float), cudaMemcpyHostToDevice));
    AMTK_CUDA(cudaMemcpy(scales, h.scales.data(), (size_t)count * 32 * sizeof(float2), cudaMemcpyHostToDevice));
  }
  l->dPix = std::move(pix); l->dTapsT = std::move(taps); l->dScales = std::move(scales);
  l->tables_uploaded = true;
  return 1;
}

// Logos are host objects; their HBM copies are made on first use by a context (and stay on that device).
static int logo_ensure_device(const amtk_logo* cl, amtk_ctx* ctx, bool need_tables) {
  amtk_logo* l = const_cast<amtk_logo*>(cl);
  std::lock_guard<std::mutex> lock(l->mu);
  if (l->device >= 0 && l->dA && l->device != ctx->device) AMTK_FAIL("logo already resident on another device");
  l->device = ctx->device;
  if (!l->dA && !logo_upload_planes(l)) return 0;
  if (need_tables) {
    if (!l->has_mask) AMTK_FAIL("logo has no mask: call amtk_logo_create_mask first");
    if (!l->tables_uploaded && !logo_upload_tables(l)) return 0;
  }
  return 1;
}

static int logo_adopt(amtk_ctx* /*ctx: logos bind to a device on first use*/, amtk::HostLogo&& h, amtk_logo** out) {
  amtk_logo* l = new amtk_logo();
  l->host = std::move(h);
  *out = l;
  return 1;
}

int amtk_logo_create(amtk_ctx* ctx, const float* data, int w, int h, int lx, int ly, int imgw, int imgh, int imgx, int imgy, amtk_logo** out) {
  if (!data || !out) AMTK_FAIL("amtk_logo_create: null argument");   // ctx may be NULL: bound on first use
  if (w < 5 || h < 5 || w > 4096 || h > 4096 || lx < 0 || lx > 2 || ly < 0 || ly > 2) AMTK_FAIL("amtk_logo_create: bad logo geometry");
  amtk::HostLogo hl; hl.init(w, h, lx, ly, imgw, imgh, imgx, imgy);
  memcpy(hl.data.data(), data, hl.dataSize() * sizeof(float));
  return logo_adopt(ctx, std::move(hl), out);
}

int amtk_logo_load(amtk_ctx* ctx, const char* path, amtk_logo** out, void* header540) {
  if (!path || !out) AMTK_FAIL("amtk_logo_load: null argument");
  amtk::HostLogo hl; amtk::LgdHeader hdr; std::string err;
  if (!amtk::lgd_load(path, hl, &hdr, err)) AMTK_FAIL(err);
  if (header540) memcpy(header540, &hdr, sizeof(hdr));
  return logo_adopt(ctx, std::move(hl), out);
}

int amtk_logo_save(const amtk_logo* l, const char* path, const char* name, int service_id) {
  if (!l || !path) AMTK_FAIL("amtk_logo_save: null argument");
  std::string err;
  if (!amtk::lgd_save(l->host, path, name ? name : "No Name", service_id, err)) AMTK_FAIL(err);
  return 1;
}

void amtk_logo_destroy(amtk_logo* l) {
  if (!l) return;
  if (l->device >= 0 && l->dA) { DevSelect ds(l->device); delete l; }
  else delete l;
}

int amtk_logo_deint(const amtk_logo* src, amtk_logo** out) {
  if (!src || !out) AMTK_FAIL("amtk_logo_deint: null argument");
  amtk::HostLogo d; amtk::logo_deint(src->host, d);
  return logo_adopt(nullptr, std::move(d), out);
}

int amtk_logo_field(const amtk_logo* src, int bottom, amtk_logo** out) {
  if (!src || !out) AMTK_FAIL("amtk_logo_field: null argument");
  if (src->host.h / 2 < 5) AMTK_FAIL("amtk_logo_field: logo too small");
  amtk::HostLogo f; amtk::logo_field(src->host, bottom != 0, f);
  return logo_adopt(nullptr, std::move(f), out);
}

int amtk_logo_create_mask(amtk_logo* l, float maskratio) {
  if (!l) AMTK_FAIL("amtk_logo_create_mask: null logo");
  if (!(maskratio > 0.0f) || maskratio > 1.0f) AMTK_FAIL("amtk_logo_create_mask: maskratio must be in (0,1]");
  std::lock_guard<std::mutex> lock(l->mu);
  amtk::logo_create_mask(l->host, maskratio);
  l->countPad = std::max(32, (l->host.count() + 31) & ~31);
  l->has_mask = true;
  l->tables_uploaded = false;       // (re)uploaded by the next evaluation call
  return 1;
}

int amtk_logo_get_info(const amtk_logo* l, amtk_logo_info* o) {
  if (!l || !o) AMTK_FAIL("amtk_logo_get_info: null argument");
  const amtk::HostLogo& h = l->host;
  o->w = h.w; o->h = h.h; o->log_uvx = h.logUVx; o->log_uvy = h.logUVy;
  o->imgw = h.imgw; o->imgh = h.imgh; o->imgx = h.imgx; o->imgy = h.imgy;
  o->maskpixels = h.maskpixels; o->count = h.count(); o->black_score = h.blackScore;
  return 1;
}

int amtk_logo_get_tables(const amtk_logo* l, float* data, uint8_t* mask, float* kernels, float* scales) {
  if (!l) AMTK_FAIL("amtk_logo_get_tables: null logo");
  const amtk::HostLogo& h = l->host;
  if (data) memcpy(data, h.data.data(), h.dataSize() * sizeof(float));
  if ((mask || kernels || scales) && !l->has_mask) AMTK_FAIL("logo has no mask");
  if (mask) memcpy(mask, h.mask.data(), h.mask.size());
  if (kernels) memcpy(kernels, h.kernels.data(), h.kernels.size() * sizeof(float));
  if (scales) memcpy(scales, h.scales.data(), h.scales.size() * sizeof(float));
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// evaluation entry points
// ---------------------------------------------------------------------------------------------------------
// Small host outputs (a GetFrame-sized call returns 8 .. 1056 bytes): the result kernels write straight into a pinned, device-mapped
// buffer of the context, so the call ends with a stream synchronise and a CPU copy instead of a D2H copy operation and ITS
// completion (a third of a one-frame call's wall time).  Only for outputs that kernels write once (logo scores), never for the
// atomically accumulated combing counters.
constexpr size_t kHostOutBytes = 64 << 10;
static float* host_out_alias(amtk_ctx* ctx, size_t bytes) {
  if (bytes > kHostOutBytes) return nullptr;
  if (!ctx->hout) {
    void* h = nullptr;
    if (cudaHostAlloc(&h, kHostOutBytes, cudaHostAllocMapped) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    ctx->hout.reset(h);
    if (cudaHostGetDevicePointer(&ctx->hout_dev, ctx->hout, 0) != cudaSuccess) { cudaGetLastError(); ctx->hout.reset(); return nullptr; }
  }
  return reinterpret_cast<float*>(ctx->hout_dev);
}
// device buffer the result kernels of a host-output call write to: the mapped alias when the output is small, else ctx->dout
static float* host_out_buffer(amtk_ctx* ctx, size_t bytes) {
  if (float* a = host_out_alias(ctx, bytes)) return a;
  if (!ctx->dout.ensure(bytes)) return nullptr;
  return ctx->dout.at<float>();
}

static int finish_output(amtk_ctx* ctx, void* host_dst, const void* dev_src, size_t bytes, int out_on_device) {
  if (out_on_device) return 1;
  if (ctx->hout && dev_src == ctx->hout_dev) {
    AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
    memcpy(host_dst, ctx->hout, bytes);
    return 1;
  }
  AMTK_CUDA(cudaMemcpyAsync(host_dst, dev_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
  return 1;
}

// `real` is the caller's clip (frame size checks), `clip` the resident data (the same, or an ROI-only staging copy whose
// luma origin sits at (dx, dy) of the real frame).
static int scan_frames_impl(amtk_ctx* ctx, const amtk_clip* real, const amtk_clip* clip, int dx, int dy, amtk_logo* const* logos, int nlogos,
                            const Window& win, int lo, int hi, int pitch_override, float* dscores, int row0) {
  static const float kFades01[2] = { 0.0f, 1.0f };
  const int pitch = pitch_override > 0 ? pitch_override : clip->pitch_y / clip->bytes_per_sample;
  const int real_pitch = pitch_override > 0 ? pitch_override : real->pitch_y / real->bytes_per_sample;
  for (int i = 0; i < nlogos; ++i) {
    const amtk_logo* lg = logos[i];
    float* o = dscores + (size_t)(lo - row0) * nlogos * 2;
    if (!lg || lg->host.imgw != real->width || lg->host.imgh != real->height) {      // LogoScan.hpp:1551-1558
      fill_pairs_kernel<<<(hi - lo + 127) / 128, 128, 0, ctx->stream>>>(o, hi - lo, nlogos * 2, i * 2, 0.0f, -1.0f);
      AMTK_CUDA(cudaGetLastError()); ctx->launches += 1;
      continue;
    }
    if (!roi_inside(lg->host, real, real_pitch)) AMTK_FAIL("logo rectangle lies outside the frame");
    EvalSpec sp{ lg, lg->host.imgx - dx, lg->host.imgy - dy, lg->host.w, lg->host.h, 0, 0, lg->host.w, 2, kFades01, 0, i * 2, 1 };
    if (!launch_eval(ctx, clip, win, lo, hi, pitch, sp, dscores, nlogos * 2, row0, ctx->stream, 0)) return 0;
  }
  return 1;
}

// bounding box of the rectangles of all logos that will be evaluated on `clip` (false when there is none)
static bool logos_bbox(const amtk_clip* clip, amtk_logo* const* logos, int nlogos, int* rx, int* ry, int* rw, int* rh) {
  int x0 = 1 << 30, y0 = 1 << 30, x1 = -1, y1 = -1;
  for (int i = 0; i < nlogos; ++i) {
    const amtk_logo* lg = logos[i];
    if (!lg || lg->host.imgw != clip->width || lg->host.imgh != clip->height) continue;
    x0 = std::min(x0, lg->host.imgx); y0 = std::min(y0, lg->host.imgy);
    x1 = std::max(x1, lg->host.imgx + lg->host.w); y1 = std::max(y1, lg->host.imgy + lg->host.h);
  }
  if (x1 < 0 || x0 < 0 || y0 < 0 || x1 > clip->width || y1 > clip->height) return false;
  *rx = x0; *ry = y0; *rw = x1 - x0; *rh = y1 - y0;
  return true;
}

int amtk_logo_scan_frames(amtk_ctx* ctx, const amtk_clip* clip, amtk_logo* const* logos, int nlogos,
                          int frame0, int nframes, int pitch_override, float* out, int out_on_device) {
  if (ctx && nframes == 0) return 1;                                 // empty range: nothing to do
  if (!ctx || !logos || !out || nlogos < 1) AMTK_FAIL("amtk_logo_scan_frames: bad argument");
  if (!validate_clip(clip, false)) return 0;
  DevSelect ds(ctx); if (!ds.ok) return 0;
  const size_t bytes = (size_t)nframes * nlogos * 2 * sizeof(float);
  float* d = out;
  if (!out_on_device) { d = host_out_buffer(ctx, bytes); if (!d) return 0; }
  int rx, ry, rw, rh;
  if (!clip->on_device && pitch_override <= 0 && logos_bbox(clip, logos, nlogos, &rx, &ry, &rw, &rh)) {
    // host frames: only the logo rectangles cross PCIe (the reference reads nothing else, LogoScan.hpp:1559-1566)
    if (!for_each_roi_window(ctx, clip, frame0, nframes, rx, ry, rw, rh, false, false,
                             [&](const amtk_clip& v, const Window& w, int lo, int hi, int dx, int dy) {
          return scan_frames_impl(ctx, clip, &v, dx, dy, logos, nlogos, w, lo, hi, 0, d, frame0); }))
      return 0;
  } else if (!for_each_window(ctx, clip, frame0, nframes, false, [&](const Window& w, int lo, int hi) {
        return scan_frames_impl(ctx, clip, clip, 0, 0, logos, nlogos, w, lo, hi, pitch_override, d, frame0); }))
    return 0;
  return finish_output(ctx, out, d, bytes, out_on_device);
}

// AMTAnalyzeLogo's 33 values of frames [lo, hi) into rows lo - row0.. of dout; with frame_list (see launch_eval) of the
// frames at list positions [lo, hi) into rows frame_list[p].
static int analyze_impl(amtk_ctx* ctx, const amtk_clip* clip, int dx, int dy, const amtk_logo* dl, const amtk_logo* ft, const amtk_logo* fb,
                        const Window& win, int lo, int hi, float* dout, int row0, const int* frame_list = nullptr) {
  float fades[11];
  for (int f = 0; f <= 10; ++f) fades[f] = (float)f / 10.0f;             // LogoScan.hpp:1152
  const int pitch = clip->pitch_y / clip->bytes_per_sample;
  const int w = dl->host.w, h = dl->host.h;
  const int rx = dl->host.imgx - dx, ry = dl->host.imgy - dy;
  EvalSpec sp{ dl, rx, ry, w, h, 0, 0, w, 11, fades, 1, 0, 1 };                // p[f]: deint logo on DeintY
  EvalSpec st{ ft, rx, ry, w, h, 1, 0, 2 * w, 11, fades, 1, 11, 1 };           // t[f]: top field logo on CopyY, stride 2w
  EvalSpec sb{ fb, rx, ry, w, h, 1, w, 2 * w, 11, fades, 1, 22, 1 };           // b[f]: bottom field logo on CopyY + w
  const int n = hi - lo;
  if (!(ctx->knobs.eval_par && n <= 16 && ctx->side_stream && ctx->side_stream2))
    return launch_eval(ctx, clip, win, lo, hi, pitch, sp, dout, 33, row0, ctx->stream, 0, frame_list) &&
           launch_eval(ctx, clip, win, lo, hi, pitch, st, dout, 33, row0, ctx->stream, 0, frame_list) &&
           launch_eval(ctx, clip, win, lo, hi, pitch, sb, dout, 33, row0, ctx->stream, 0, frame_list);
  // GetFrame-sized call (AMTAnalyzeLogo::GetFrame = 8 source frames): each evaluation launches only n CTAs, so the three of them
  // run side by side on three streams, each with its own slice of the score scratch (115 -> ~70 us per call).
  const EvalSpec* specs[3] = { &sp, &st, &sb };
  size_t off[3], total = 0;
  for (int i = 0; i < 3; ++i) {
    if (!logo_ensure_device(specs[i]->logo, ctx, true)) return 0;                      // table uploads happen before the fork
    off[i] = total;
    total += (((size_t)n * 11 * specs[i]->logo->countPad * sizeof(float)) + 255) & ~(size_t)255;
  }
  if (!ctx->scratch.ensure(total)) return 0;                    // no reallocation once work is in flight
  cudaStream_t streams[3] = { ctx->stream, ctx->side_stream, ctx->side_stream2 };
  cudaEvent_t joins[3] = { nullptr, ctx->ev_join1, ctx->ev_join2 };
  AMTK_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
  int ok = 1;
  for (int i = 0; i < 3 && ok; ++i) {
    if (i) ok = cuda_ok(cudaStreamWaitEvent(streams[i], ctx->ev_fork, 0), "cudaStreamWaitEvent");
    ok = ok && launch_eval(ctx, clip, win, lo, hi, pitch, *specs[i], dout, 33, row0, streams[i], off[i], frame_list);
    if (i && ok) ok = cuda_ok(cudaEventRecord(joins[i], streams[i]), "cudaEventRecord") &&
                      cuda_ok(cudaStreamWaitEvent(ctx->stream, joins[i], 0), "cudaStreamWaitEvent");
  }
  if (!ok) { cudaStreamSynchronize(ctx->side_stream); cudaStreamSynchronize(ctx->side_stream2); }   // nothing of this call stays in flight
  return ok;
}

int amtk_logo_analyze_frames(amtk_ctx* ctx, const amtk_clip* clip, const amtk_logo* dl, const amtk_logo* ft, const amtk_logo* fb,
                             int frame0, int nframes, float* out, int out_on_device) {
  if (ctx && nframes == 0) return 1;
  if (!ctx || !dl || !ft || !fb || !out) AMTK_FAIL("amtk_logo_analyze_frames: bad argument");
  if (!validate_clip(clip, false)) return 0;
  if (ft->host.w != dl->host.w || fb->host.w != dl->host.w || ft->host.h != dl->host.h / 2 || fb->host.h != dl->host.h / 2)
    AMTK_FAIL("field logos do not match the deint logo");
  DevSelect ds(ctx); if (!ds.ok) return 0;
  const size_t bytes = (size_t)nframes * 33 * sizeof(float);
  float* d = out;
  if (!out_on_device) { d = host_out_buffer(ctx, bytes); if (!d) return 0; }
  if (!roi_inside(dl->host, clip, clip->pitch_y / clip->bytes_per_sample)) AMTK_FAIL("logo rectangle lies outside the frame");
  if (!for_each_roi_window(ctx, clip, frame0, nframes, dl->host.imgx, dl->host.imgy, dl->host.w, dl->host.h, false, false,
                           [&](const amtk_clip& v, const Window& w, int lo, int hi, int dx, int dy) {
        return analyze_impl(ctx, &v, dx, dy, dl, ft, fb, w, lo, hi, d, frame0); }))
    return 0;
  return finish_output(ctx, out, d, bytes, out_on_device);
}

int amtk_logo_eval_fades(amtk_ctx* ctx, const amtk_clip* clip, const amtk_logo* dl, const float* fades, int nfades,
                         int frame0, int nframes, float* out, int out_on_device) {
  if (ctx && nframes == 0) return 1;
  if (!ctx || !dl || !fades || !out) AMTK_FAIL("amtk_logo_eval_fades: bad argument");
  if (nfades < 1 || nfades > kMaxFades) AMTK_FAIL("amtk_logo_eval_fades: 1..24 fade levels");
  if (!validate_clip(clip, false)) return 0;
  DevSelect ds(ctx); if (!ds.ok) return 0;
  const size_t bytes = (size_t)nframes * nfades * sizeof(float);
  float* d = out;
  if (!out_on_device) { d = host_out_buffer(ctx, bytes); if (!d) return 0; }
  const int pitch = clip->pitch_y / clip->bytes_per_sample;
  if (!roi_inside(dl->host, clip, pitch)) AMTK_FAIL("logo rectangle lies outside the frame");
  if (!for_each_roi_window(ctx, clip, frame0, nframes, dl->host.imgx, dl->host.imgy, dl->host.w, dl->host.h, false, false,
                           [&](const amtk_clip& v, const Window& w, int lo, int hi, int dx, int dy) {
        EvalSpec sp{ dl, dl->host.imgx - dx, dl->host.imgy - dy, dl->host.w, dl->host.h, 0, 0, dl->host.w, nfades, fades, 0, 0, 1 };
        return launch_eval(ctx, &v, w, lo, hi, v.pitch_y / v.bytes_per_sample, sp, d, nfades, frame0, ctx->stream, 0); }))
    return 0;
  return finish_output(ctx, out, d, bytes, out_on_device);
}

// ---------------------------------------------------------------------------------------------------------
// combing metric + fused step
// ---------------------------------------------------------------------------------------------------------
void amtk_comb_default_params(amtk_comb_params* p) {
  if (!p) return;
  p->th_move_y = 20; p->th_shima_y = 12; p->th_lshima_y = 36;
  p->th_move_c = 24; p->th_shima_c = 16; p->th_lshima_c = 48;
}

// Frames per logo item of the fused step, or 0 for the serial path.  A logo runs fused when its item (scan_item_smem_bytes)
// holds one frame in the 512 x 4R band ring's slots, whichever band form runs, so which logos run fused does not depend on
// the form.  F then comes from the ring of the variant that runs: as many frames as its slots hold, at most
// kScanItemMaxFrames (the tall ring holds 13 for a 64x64 logo at maskratio 0.35, the 512 x 4R ring 2).
static int scan_item_frames(const amtk_logo* lg, const amtk_ctx* ctx, const amtk_clip* clip) {
  const WsVariant* V4 = ws_variant(ctx, clip, false);
  const WsVariant* V = ws_variant(ctx, clip);
  if (!V4 || !V) return 0;
  const int w = lg->host.w, h = lg->host.h;
  if (scan_item_smem_bytes(w, h, lg->countPad, 1) > (size_t)V4->smem - 128) return 0;   // the slots (SMEM = ring + alignment slack)
  int F = 0;
  while (F < kScanItemMaxFrames && scan_item_smem_bytes(w, h, lg->countPad, F + 1) <= (size_t)V->smem - 128) ++F;
  return F;
}

// The logo of a fused step that runs as logo items of the band-form comb kernel on `clip`'s window w (nullptr: the logo
// kernels run after the comb kernel), and its frames per item in *F.  One logo on an 8-bit clip (the headline case) runs
// fused; anything else (several logos, other sample sizes or comb kernels, logos whose item does not fit in the ring)
// runs serially.
static const amtk_logo* scan_comb_fused_logo(const amtk_ctx* ctx, const amtk_clip* clip, const Window& w, amtk_logo* const* logos,
                                             int nlogos, int* F) {
  const amtk_logo* lg0 = nlogos == 1 ? logos[0] : nullptr;
  const bool one_logo = lg0 && lg0->has_mask && lg0->host.count() > 0 &&
                        lg0->host.imgw == clip->width && lg0->host.imgh == clip->height && lg0->host.imgx >= 0 && lg0->host.imgy >= 0 &&
                        lg0->host.imgx + lg0->host.w <= clip->width && lg0->host.imgy + lg0->host.h <= clip->height;
  const WsVariant* V = one_logo && comb_runs_band(ctx, clip, w) ? ws_variant(ctx, clip) : nullptr;
  *F = V ? scan_item_frames(lg0, ctx, clip) : 0;
  return *F > 0 ? lg0 : nullptr;
}

// The fused step on frames [lo, hi) of the resident window w: scores into rows lo - row0.. of dscores (nlogos pairs per
// row), counters into rows lo - row0.. of dcounts.  Fused: one comb launch whose queue also holds the logo items.
// pitch_override > 0 addresses the Y plane of the logo evaluation with that element pitch (amtk_logo_scan_frames'
// pitch_elems_override); the logo kernels then run after the comb kernel.
static int scan_comb_window(amtk_ctx* ctx, const amtk_clip* clip, const Window& w, int lo, int hi, amtk_logo* const* logos, int nlogos,
                            const amtk_comb_params* prm, float* dscores, int* dcounts, int row0, int pitch_override) {
  int F = 0;
  if (const amtk_logo* lg0 = pitch_override > 0 ? nullptr : scan_comb_fused_logo(ctx, clip, w, logos, nlogos, &F)) {
    if (!logo_ensure_device(lg0, ctx, true)) return 0;
    ScanItemJob lj;
    lj.ybase = w.dev_base; lj.frame_stride = clip->frame_stride; lj.pitch = clip->pitch_y;
    lj.imgx = lg0->host.imgx; lj.imgy = lg0->host.imgy;
    lj.logo = logo_dev(lg0); lj.maxv = (float)((1 << clip->bits_per_sample) - 1);
    lj.frames = F; lj.scores = dscores;
    return launch_comb_ws(ctx, clip, w, lo, hi, prm, dcounts, row0, &lj);
  }
  return launch_comb(ctx, clip, w, lo, hi, prm, dcounts, row0) &&
         scan_frames_impl(ctx, clip, clip, 0, 0, logos, nlogos, w, lo, hi, pitch_override, dscores, row0);
}

// The fused step over frames [frame0, frame0 + nframes).  Without logos (amtk_comb_frames: with_logos false, nlogos 0) it
// is the combing pass alone: launch_comb per window, and with host outputs only the counters are downloaded.
static int scan_comb_frames_impl(amtk_ctx* ctx, const amtk_clip* clip, amtk_logo* const* logos, int nlogos, const amtk_comb_params* prm,
                                 int pitch_override, int frame0, int nframes, float* scores, int32_t* counts, int out_on_device,
                                 bool with_logos, const char* name) {
  if (ctx && nframes == 0) return 1;
  if (!ctx || !prm || !counts || (with_logos && (!scores || !logos || nlogos < 1))) AMTK_FAIL(std::string(name) + ": bad argument");
  if (!validate_clip(clip, true) || !comb_thresholds_ok(prm, clip->bytes_per_sample)) return 0;
  // the clip's own element pitch is no override: the call is then amtk_scan_comb_frames, launches included
  if (pitch_override == clip->pitch_y / clip->bytes_per_sample) pitch_override = 0;
  DevSelect ds(ctx); if (!ds.ok) return 0;
  const size_t sbytes = (size_t)nframes * nlogos * 2 * sizeof(float), cbytes = (size_t)nframes * 12 * sizeof(int32_t);
  float* ds_ = scores; int* dc = counts;
  if (!out_on_device) {
    if (!ctx->dout.ensure(sbytes) || !ctx->dout2.ensure(cbytes)) return 0;
    ds_ = ctx->dout.at<float>(); dc = ctx->dout2.at<int>();
  }
  if (!for_each_window(ctx, clip, frame0, nframes, true, [&](const Window& w, int lo, int hi) {
        return scan_comb_window(ctx, clip, w, lo, hi, logos, nlogos, prm, ds_, dc, frame0, pitch_override); }))
    return 0;
  if (out_on_device) return 1;
  if (sbytes) AMTK_CUDA(cudaMemcpyAsync(scores, ds_, sbytes, cudaMemcpyDeviceToHost, ctx->stream));
  AMTK_CUDA(cudaMemcpyAsync(counts, dc, cbytes, cudaMemcpyDeviceToHost, ctx->stream));
  // the stream is synchronised, so this call's own watchdog record is checked too
  AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
  return ws_watchdog_synced(ctx);
}

int amtk_comb_frames(amtk_ctx* ctx, const amtk_clip* clip, const amtk_comb_params* prm, int frame0, int nframes,
                     int32_t* counts, int out_on_device) {
  return scan_comb_frames_impl(ctx, clip, nullptr, 0, prm, 0, frame0, nframes, nullptr, counts, out_on_device, false, "amtk_comb_frames");
}

int amtk_scan_comb_frames(amtk_ctx* ctx, const amtk_clip* clip, amtk_logo* const* logos, int nlogos,
                          const amtk_comb_params* prm, int frame0, int nframes, float* scores, int32_t* counts, int out_on_device) {
  return scan_comb_frames_impl(ctx, clip, logos, nlogos, prm, 0, frame0, nframes, scores, counts, out_on_device, true,
                               "amtk_scan_comb_frames");
}

int amtk_scan_comb_frames_pitch(amtk_ctx* ctx, const amtk_clip* clip, amtk_logo* const* logos, int nlogos,
                                const amtk_comb_params* prm, int pitch_elems_override, int frame0, int nframes, float* scores,
                                int32_t* counts, int out_on_device) {
  return scan_comb_frames_impl(ctx, clip, logos, nlogos, prm, std::max(pitch_elems_override, 0), frame0, nframes, scores, counts,
                               out_on_device, true, "amtk_scan_comb_frames_pitch");
}

// ---------------------------------------------------------------------------------------------------------
// LogoScan accumulation
// ---------------------------------------------------------------------------------------------------------
// The sample formats LogoScan takes: 1-byte samples at up to 8 bits, 2-byte samples at 9..16 bits with even pitches,
// plane offsets and frame stride.  Returns the bits maxv is made of (8 for 1-byte samples), 0 with the error set.
static int scan_sample_bits(const amtk_clip* c) {
  if (c->bytes_per_sample == 1) {
    if (c->bits_per_sample <= 8) return 8;
  } else if (c->bits_per_sample > 8 && c->bits_per_sample <= 16) {
    if (((c->pitch_y | c->pitch_uv | c->off_u | c->off_v | c->frame_stride | (int64_t)reinterpret_cast<uintptr_t>(c->base)) & 1) == 0)
      return c->bits_per_sample;
    set_error("LogoScan: 2-byte clips need even pitches, plane offsets, frame stride and base");
    return 0;
  }
  set_error("LogoScan: bits_per_sample must be at most 8 for 1-byte samples and 9..16 for 2-byte samples");
  return 0;
}

int amtk_scan_create(amtk_ctx* ctx, int scanw, int scanh, int lx, int ly, int thy, amtk_scan** out) {
  if (!ctx || !out) AMTK_FAIL("amtk_scan_create: null argument");
  if (scanw < 4 || scanh < 4 || scanw > 4096 || scanh > 4096 || lx < 0 || lx > 2 || ly < 0 || ly > 2) AMTK_FAIL("amtk_scan_create: bad geometry");
  DevSelect ds(ctx); if (!ds.ok) return 0;
  std::unique_ptr<amtk_scan> s(new amtk_scan());
  s->ctx = ctx; s->device = ctx->device; s->scanw = scanw; s->scanh = scanh; s->logUVx = lx; s->logUVy = ly; s->thy = thy;
  s->npix = (size_t)scanw * scanh + 2 * (size_t)(scanw >> lx) * (scanh >> ly);
  // zeroed on the stream the accumulation kernels run on, so that they see the zeros
  if (!cuda_ok(cudaMalloc(s->dSums.put(), s->npix * 3 * sizeof(unsigned long long)), "cudaMalloc") ||
      !cuda_ok(cudaMalloc(s->dBg.put(), 8 * sizeof(unsigned long long)), "cudaMalloc") ||
      !cuda_ok(cudaMemsetAsync(s->dSums, 0, s->npix * 3 * sizeof(unsigned long long), ctx->stream), "cudaMemsetAsync") ||
      !cuda_ok(cudaMemsetAsync(s->dBg, 0, 8 * sizeof(unsigned long long), ctx->stream), "cudaMemsetAsync"))
    return 0;
  *out = s.release();
  return 1;
}

void amtk_scan_destroy(amtk_scan* s) {
  if (!s) return;
  DevSelect ds(s->device);
  delete s;
}

int amtk_scan_add_frames(amtk_scan* s, const amtk_clip* clip, int scanx, int scany, int frame0, int nframes,
                         const uint8_t* frame_select, uint8_t* valid_out) {
  if (!s) AMTK_FAIL("amtk_scan_add_frames: null scan");
  amtk_ctx* ctx = s->ctx;
  if (!validate_clip(clip, true)) return 0;
  const int bits = scan_sample_bits(clip);
  if (!bits) return 0;
  if (s->bytes_per_sample && (clip->bytes_per_sample != s->bytes_per_sample || bits != s->bits))
    AMTK_FAIL("LogoScan: the clip's sample format differs from the first clip's");
  if (clip->log_uvx != s->logUVx || clip->log_uvy != s->logUVy) AMTK_FAIL("chroma subsampling mismatch");
  if (scanx < 0 || scany < 0 || scanx + s->scanw > clip->width || scany + s->scanh > clip->height) AMTK_FAIL("scan rectangle outside the frame");
  if (frame0 < 0 || nframes < 0 || frame0 + nframes > clip->num_frames) AMTK_FAIL("frame range outside the clip");
  DevSelect ds(ctx); if (!ds.ok) return 0;
  s->bytes_per_sample = clip->bytes_per_sample; s->bits = bits;
  const bool wide = clip->bytes_per_sample == 2;
  // small per-frame buffers: int4 bg[n], u8 select[n], u8 valid[n]
  const size_t bg_bytes = (size_t)nframes * sizeof(int4), off_sel = (bg_bytes + 255) & ~(size_t)255;
  const size_t off_val = off_sel + (((size_t)nframes + 255) & ~(size_t)255);
  if (!ctx->dout.ensure(off_val + (size_t)nframes + 256)) return 0;
  uint8_t* base = ctx->dout.at();
  int4* dbg = reinterpret_cast<int4*>(base); uint8_t* dsel = base + off_sel; uint8_t* dval = base + off_val;
  if (frame_select) AMTK_CUDA(cudaMemcpyAsync(dsel, frame_select, (size_t)nframes, cudaMemcpyHostToDevice, ctx->stream));
  // host clips: only the scan rectangle (Y, U, V) is uploaded -- LogoScan::AddFrame reads nothing else (LogoScan.hpp:606-635)
  const int ok = for_each_roi_window(ctx, clip, frame0, nframes, scanx, scany, s->scanw, s->scanh, true, false,
                                     [&](const amtk_clip& v, const Window& w, int lo, int hi, int dx, int dy) {
    ScanClip c;
    c.base = w.dev_base; c.frame_stride = v.frame_stride; c.offU = v.off_u; c.offV = v.off_v;
    c.pitchY = v.pitch_y / v.bytes_per_sample; c.pitchUV = v.pitch_uv / v.bytes_per_sample;
    c.scanx = scanx - dx; c.scany = scany - dy; c.scanw = s->scanw; c.scanh = s->scanh; c.logUVx = s->logUVx; c.logUVy = s->logUVy; c.thy = s->thy;
    c.frame0 = lo - w.first; c.nframes = hi - lo;
    const int rel = lo - frame0;
    if (wide) scan_border16_kernel<<<hi - lo, 256, 0, ctx->stream>>>(c, frame_select ? dsel + rel : nullptr, dbg + rel);
    else scan_border_kernel<<<hi - lo, 256, 0, ctx->stream>>>(c, frame_select ? dsel + rel : nullptr, dbg + rel);
    AMTK_CUDA(cudaGetLastError());
    const int pixblocks = (int)((s->npix + 255) / 256);
    const int splits = std::max(1, std::min(hi - lo, (ctx->sm_count * 8) / pixblocks));
    if (wide) scan_accumulate16_kernel<<<dim3(pixblocks, splits), 256, 0, ctx->stream>>>(c, dbg + rel, s->dSums, s->dBg, dval + rel);
    else scan_accumulate_kernel<<<dim3(pixblocks, splits), 256, 0, ctx->stream>>>(c, dbg + rel, s->dSums, s->dBg, dval + rel);
    AMTK_CUDA(cudaGetLastError());
    ctx->launches += 2;
    return 1;
  });
  if (!ok) return 0;
  std::vector<uint8_t> tmp;
  unsigned long long nv = 0;
  if (valid_out) AMTK_CUDA(cudaMemcpyAsync(valid_out, dval, (size_t)nframes, cudaMemcpyDeviceToHost, ctx->stream));
  AMTK_CUDA(cudaMemcpyAsync(&nv, s->dBg + 6, sizeof(nv), cudaMemcpyDeviceToHost, ctx->stream));
  AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
  s->nvalid = (int)nv;
  return 1;
}

int amtk_scan_num_valid(const amtk_scan* s) { return s ? s->nvalid : 0; }

int amtk_scan_get_sums(amtk_scan* s, double* out) {
  if (!s || !out) AMTK_FAIL("amtk_scan_get_sums: null argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  std::vector<unsigned long long> h(s->npix * 3), bg(8);
  AMTK_CUDA(cudaStreamSynchronize(s->ctx->stream));
  AMTK_CUDA(cudaMemcpy(h.data(), s->dSums, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  AMTK_CUDA(cudaMemcpy(bg.data(), s->dBg, bg.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  const size_t ny = (size_t)s->scanw * s->scanh, nc = (size_t)(s->scanw >> s->logUVx) * (s->scanh >> s->logUVy);
  for (size_t i = 0; i < s->npix; ++i) {
    const int pl = i < ny ? 0 : (i < ny + nc ? 1 : 2);
    // two's-complement s64 (2-byte samples can make sumB, sumFB and sumF2 negative); exact while |sum| < 2^53
    out[i * 5 + 0] = (double)(long long)h[i * 3 + 0];        // sumF
    out[i * 5 + 1] = (double)(long long)bg[pl * 2 + 0];      // sumB
    out[i * 5 + 2] = (double)(long long)h[i * 3 + 1];        // sumF2
    out[i * 5 + 3] = (double)(long long)bg[pl * 2 + 1];      // sumB2
    out[i * 5 + 4] = (double)(long long)h[i * 3 + 2];        // sumFB
  }
  s->nvalid = (int)bg[6];
  return 1;
}

int amtk_scan_get_logo(amtk_scan* s, int maxv, int clean, float* data) {
  if (!s || !data) AMTK_FAIL("amtk_scan_get_logo: null argument");
  std::vector<double> sums(s->npix * 5);
  if (!amtk_scan_get_sums(s, sums.data())) return 0;
  if (!amtk::scan_finalize(sums.data(), s->nvalid, s->scanw, s->scanh, s->logUVx, s->logUVy, maxv, clean != 0, data))
    AMTK_FAIL("Insufficient logo frames");
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// ScanLogo pipeline (LogoScan.hpp:794-1098)
// ---------------------------------------------------------------------------------------------------------
namespace {
struct ScanGuard { amtk_scan* s = nullptr; ~ScanGuard() { if (s) amtk_scan_destroy(s); } };
struct LogoGuard { amtk_logo* l = nullptr; ~LogoGuard() { if (l) amtk_logo_destroy(l); } };

// The frames MakeInitialLogo stored (the reference's UtVideo work file): frames [0, nframes) of clip with select[i] != 0
// (select == nullptr: all of them), the scan rectangle at (x, y) of each; numFrames of them are stored.
struct StoredFrames {
  const amtk_clip* clip;
  int x, y, nframes;
  const uint8_t* select;
  int numFrames;
  bool stored(int i) const { return !select || select[i]; }
};

// The second half of LogoAnalyzer::ScanLogo (LogoScan.hpp:1058-1079) over the stored frames: GetLogo(false) of their sums
// (:845-849), ReMakeLogo twice (:923-1036), the final callback and LogoData::Save with the header of :1076-1078 (imgw, imgh:
// the source's frame size; imgx, imgy: the scan rectangle).  amtk_scan_logo runs it on the clip it was given, the frame
// stream on its HBM stack of rectangles; integer sums do not depend on the order frames are added, and the fade sweep reads
// nothing but the rectangle, so both write the same bytes for the same stored frames.
int scan_logo_from_stored(amtk_ctx* ctx, const StoredFrames& st, int w, int h, int thy, int imgw, int imgh, int imgx, int imgy,
                          int service_id, const char* dstpath, amtk_logo_analyze_cb cb) {
  DevSelect ds(ctx); if (!ds.ok) return 0;
  const amtk_clip* clip = st.clip;
  const int lx = clip->log_uvx, ly = clip->log_uvy, numFrames = st.numFrames, n = st.nframes;
  // the reference's three 255s (:845, :968, :1030) at the clip's depth; the sweep takes its maxv from the clip too
  const int maxv = clip->bytes_per_sample == 1 ? 255 : (1 << clip->bits_per_sample) - 1;
  const size_t ndata = ((size_t)w * h + 2 * (size_t)(w >> lx) * (h >> ly)) * 2;
  std::vector<float> logodata(ndata);
  {
    ScanGuard init;
    if (!amtk_scan_create(ctx, w, h, lx, ly, thy, &init.s)) return 0;
    if (n > 0 && !amtk_scan_add_frames(init.s, clip, st.x, st.y, 0, n, st.select, nullptr)) return 0;
    if (!amtk_scan_get_logo(init.s, maxv, 0, logodata.data())) return 0;     // "Insufficient logo frames"
  }
  // ---- ReMakeLogo x2 (:923-1036): 20-fade sweep over the STORED frames into HBM, read back once per round; every 100 of
  //      them the callback gets (i / numFrames * 25 + progressbase, i, numFrames, numFrames) (:977-982); frames whose best
  //      fade index is > 8 are accumulated again (:1018-1021).  Only frames [0, n) are touched. ----
  float fades[20];
  for (int fi = 0; fi < 20; ++fi) fades[fi] = 0.1f * fi;                      // :967
  const int kBlock = 128;                                                      // frames per sweep call
  DevBuf<float> dsweep;
  AMTK_CUDA(cudaMalloc(dsweep.put(), (size_t)n * 20 * sizeof(float)));
  float* dsw = dsweep;
  std::vector<float> sweep((size_t)n * 20);
  for (int round = 0; round < 2; ++round) {
    const float progressbase = 50.0f + 25.0f * round;                          // :1064-1068
    LogoGuard raw, deint;
    if (!amtk_logo_create(ctx, logodata.data(), w, h, lx, ly, w, h, st.x, st.y, &raw.l)) return 0;
    if (!amtk_logo_deint(raw.l, &deint.l) || !amtk_logo_create_mask(deint.l, 0.1f)) return 0;      // :929-931
    for (int f0 = 0; f0 < n; f0 += kBlock) {
      const int blk = std::min(kBlock, n - f0);
      bool any = false;
      for (int i = f0; i < f0 + blk; ++i) any = any || st.stored(i);
      if (any && !amtk_logo_eval_fades(ctx, clip, deint.l, fades, 20, f0, blk, dsw + (size_t)f0 * 20, 1)) return 0;
    }
    AMTK_CUDA(cudaMemcpyAsync(sweep.data(), dsw, sweep.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
    std::vector<uint8_t> sel2((size_t)n, 0);
    int stored = 0;                                                            // the reference's i: index among the stored frames
    for (int i = 0; i < n; ++i) {
      if (!st.stored(i)) continue;
      float best = FLT_MAX; int bi = 0;                                        // :964-975, first strict minimum of |score|
      for (int fi = 0; fi < 20; ++fi) { const float r = std::fabs(sweep[(size_t)i * 20 + fi]); if (r < best) { best = r; bi = fi; } }
      sel2[i] = bi > 8;                                                        // :1018-1021
      if ((stored % 100) == 0 && cb && !cb((float)stored / (float)numFrames * 25.0f + progressbase, stored, numFrames, numFrames))
        AMTK_FAIL("Cancel requested");
      ++stored;
    }
    ScanGuard acc;
    if (!amtk_scan_create(ctx, w, h, lx, ly, thy, &acc.s)) return 0;
    if (!amtk_scan_add_frames(acc.s, clip, st.x, st.y, 0, n, sel2.data(), nullptr)) return 0;
    if (!amtk_scan_get_logo(acc.s, maxv, 1, logodata.data())) return 0;       // :1030-1035
  }
  if (cb && !cb(1.0f, numFrames, numFrames, numFrames)) AMTK_FAIL("Cancel requested");     // :1071-1073
  LogoGuard fin;                                                                // :1075-1078
  if (!amtk_logo_create(nullptr, logodata.data(), w, h, lx, ly, imgw, imgh, imgx, imgy, &fin.l)) return 0;
  return amtk_logo_save(fin.l, dstpath, "No Name", service_id);
}
}  // namespace

int amtk_scan_logo(amtk_ctx* ctx, const amtk_clip* clip, int service_id, const char* dstpath,
                   int imgx, int imgy, int w, int h, int thy, int max_frames, amtk_logo_analyze_cb cb) {
  if (!ctx || !dstpath) AMTK_FAIL("amtk_scan_logo: null argument");
  if (!validate_clip(clip, true) || !scan_sample_bits(clip)) return 0;
  const int n = clip->num_frames;
  // ---- MakeInitialLogo (:917-921): frames are offered in reading order until max_frames valid ones were gathered (:884);
  //      every 200 frames read the callback gets (position/size * 50, readCount, 0, numFrames) and may cancel (:905-910).
  //      The clip replaces the decoder, so "position / file size" is frames read / frames in the clip. ----
  std::vector<uint8_t> valid((size_t)n), select((size_t)n, 0);
  int numFrames = 0, nread = 0;
  {
    ScanGuard probe;                       // validity only; the accumulation proper runs once the cut-off frame is known
    if (!amtk_scan_create(ctx, w, h, clip->log_uvx, clip->log_uvy, thy, &probe.s)) return 0;
    while (nread < n && numFrames < max_frames) {
      const int blk = std::min(200, n - nread);
      if (!amtk_scan_add_frames(probe.s, clip, imgx, imgy, nread, blk, nullptr, valid.data() + nread)) return 0;
      int i = nread;
      for (; i < nread + blk && numFrames < max_frames; ++i) if (valid[i]) { select[i] = 1; ++numFrames; }
      // the frame on which the limit is reached is the last one processed (onFrame returns false on the NEXT call, :884)
      nread = (numFrames >= max_frames) ? i : nread + blk;
      if ((nread % 200) == 0 && cb && !cb(50.0f * (float)nread / (float)std::max(1, n), nread, 0, numFrames)) AMTK_FAIL("Cancel requested");
    }
  }
  const StoredFrames st{ clip, imgx, imgy, nread, select.data(), numFrames };
  return scan_logo_from_stored(ctx, st, w, h, thy, clip->width, clip->height, imgx, imgy, service_id, dstpath, cb);
}

// ---------------------------------------------------------------------------------------------------------
// ScanLogo fed one decoded frame at a time (InitialLogoCreator::onFrame, LogoScan.hpp:881-914; DESIGN.md section 3.3.1)
// ---------------------------------------------------------------------------------------------------------
// Frames are gathered into a batch of at most 200 rectangles (CopyYV12 packing, `S` bytes apart): host frames row by row
// into a pinned buffer, uploaded in one copy when the batch is resolved; device frames with 2-D copies on the context's
// stream.  A batch is resolved at every read count that is a multiple of 200 and at finish: scan_border_kernel decides
// validity, scan_stack_kernel ranks and appends the accepted rectangles to the HBM stack, and one wait reads back how many
// were stored and where the cut-off fell.
struct amtk_scan_logo_stream {
  amtk_ctx* ctx = nullptr;
  int imgx = 0, imgy = 0, w = 0, h = 0, thy = 0, max_frames = 0;
  amtk_logo_analyze_cb cb = nullptr;
  const char* closed = nullptr;             // why send and finish fail (nullptr: open)
  bool have_fmt = false;
  int imgw = 0, imgh = 0, lx = 1, ly = 1;   // fixed by the first frame (onFirstFrame, :852-880)
  int bps = 1, bits = 8;                    // sample format, fixed by the first frame
  RectPack rp;                              // Y, U, V rectangles of a slot (CopyYV12 packing at bps bytes per sample)
  long long payload = 0, S = 0;             // rectangle bytes per frame; stride in the batch and the stack (16-byte multiple)
  PinnedBuf<uint8_t> hbatch;                // kScanStackBatch slots
  DevBuf<uint8_t> dbatch;                   // kScanStackBatch slots
  std::vector<uint8_t> slot_host;           // slot k of the open batch came from host memory
  int nbatch = 0;                           // frames in the open batch
  int64_t last_pos = 0, last_size = 1;      // pos and size sent with the newest frame
  DevBuf<int4> dbg;                         // scan_border_kernel's verdicts on the batch
  PinnedBuf<int> hres; int* dres = nullptr; // mapped: frames stored, cut-off index in the batch
  DevBuf<uint8_t> stack; int stack_cap = 0; // stored rectangles (frames), grown on demand (stream-ordered)
  int sent = 0;                             // frames sent, including those after the cut-off
  int reads = 0;                            // frames taken in while *more was 1 (the reference's readCount)
  int cutoff = -1;                          // read count of the cut-off frame (-1: not reached)
  int ngather = 0;                          // numFrames
  int64_t h2d = 0;
  bool more() const { return cutoff < 0; }
};

namespace {

bool scan_stream_check_frame(const amtk_scan_logo_stream* s, const amtk_clip* c, int64_t size) {
  if (!one_frame(c, "scan logo stream", "the frame clip")) return false;
  if (size < 1) { set_error("scan logo stream: size must be >= 1"); return false; }
  if (!sample_bits_ok(c, "scan logo stream")) return false;
  if (s->have_fmt) {
    if (c->width != s->imgw || c->height != s->imgh) { set_error("scan logo stream: the frame's size differs from the first frame's"); return false; }
    if (c->bytes_per_sample != s->bps || c->bits_per_sample != s->bits) {
      set_error("scan logo stream: the frame's sample format differs from the first frame's"); return false;
    }
    if (c->log_uvx != s->lx || c->log_uvy != s->ly) { set_error("chroma subsampling mismatch"); return false; }
  } else if (c->log_uvx < 0 || c->log_uvx > 2 || c->log_uvy < 0 || c->log_uvy > 2) {
    set_error("scan logo stream: bad chroma subsampling"); return false;
  }
  if (s->imgx + s->w > c->width || s->imgy + s->h > c->height) { set_error("scan rectangle outside the frame"); return false; }
  return true;
}

// Grows the stack to hold `need` frames (stream-ordered: the old contents move on the context's stream).
int scan_stream_reserve(amtk_scan_logo_stream* s, int need) {
  if (need <= s->stack_cap) return 1;
  const int cap = std::min(s->max_frames, std::max(need, std::max(2 * s->stack_cap, 256)));
  cudaStream_t st = s->ctx->stream;
  void* p = nullptr;
  AMTK_CUDA(cudaMallocAsync(&p, (size_t)cap * (size_t)s->S, st));
  if (s->stack) {
    AMTK_CUDA(cudaMemcpyAsync(p, s->stack, (size_t)s->ngather * (size_t)s->S, cudaMemcpyDeviceToDevice, st));
    AMTK_CUDA(cudaFreeAsync(s->stack, st));
    s->stack.release();
  }
  s->stack.reset(reinterpret_cast<uint8_t*>(p)); s->stack_cap = cap;
  return 1;
}

// Resolves the open batch: validity, ranks, cut-off, store; then the 200-frame callback when the batch closed on one.
int scan_stream_resolve(amtk_scan_logo_stream* s) {
  amtk_ctx* ctx = s->ctx;
  const int n = s->nbatch;
  if (n == 0) return 1;
  s->nbatch = 0;
  const int ok = for_each_host_run(s->slot_host, 0, n, [&](int k, int e) {   // one per batch unless frames were mixed
    AMTK_CUDA(cudaMemcpy2DAsync(s->dbatch + (size_t)k * s->S, (size_t)s->S, s->hbatch + (size_t)k * s->S, (size_t)s->S,
                                (size_t)s->payload, (size_t)(e - k), cudaMemcpyHostToDevice, ctx->stream));
    s->h2d += (int64_t)(e - k) * s->payload;
    return 1;
  });
  if (!ok) return 0;
  const int room = s->max_frames - s->ngather;
  if (!scan_stream_reserve(s, s->ngather + std::min(n, room))) return 0;
  ScanClip c;
  c.base = s->dbatch; c.frame_stride = s->S; c.offU = s->rp.offU; c.offV = s->rp.offV;
  c.pitchY = s->w; c.pitchUV = s->w >> s->lx;
  c.scanx = 0; c.scany = 0; c.scanw = s->w; c.scanh = s->h; c.logUVx = s->lx; c.logUVy = s->ly; c.thy = s->thy;
  c.frame0 = 0; c.nframes = n;
  s->hres[0] = 0; s->hres[1] = -1;
  if (s->bps == 2) scan_border16_kernel<<<n, 256, 0, ctx->stream>>>(c, nullptr, s->dbg);
  else scan_border_kernel<<<n, 256, 0, ctx->stream>>>(c, nullptr, s->dbg);
  AMTK_CUDA(cudaGetLastError());
  scan_stack_kernel<<<n, 256, 0, ctx->stream>>>(s->dbatch, s->S, s->dbg, n, room, s->stack + (size_t)s->ngather * s->S, s->dres);
  AMTK_CUDA(cudaGetLastError());
  ctx->launches += 2;
  AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
  const int stored = reinterpret_cast<volatile int*>(s->hres.get())[0], cut = reinterpret_cast<volatile int*>(s->hres.get())[1];
  s->ngather += stored;
  if (cut >= 0) s->cutoff = s->reads - n + cut + 1;
  const int r = s->reads;
  if (r % kScanStackBatch == 0 && (s->cutoff < 0 || r <= s->cutoff) && s->cb) {
    const float progress = (float)s->last_pos / (float)s->last_size * 50.0f;     // (float)currentPos / filesize * 50 (:907)
    if (!s->cb(progress, r, 0, s->ngather)) { s->closed = "cancelled"; AMTK_FAIL("Cancel requested"); }
  }
  return 1;
}

}  // namespace

int amtk_scan_logo_stream_create(amtk_ctx* ctx, int imgx, int imgy, int w, int h, int thy, int max_frames,
                                 amtk_logo_analyze_cb cb, amtk_scan_logo_stream** out) {
  if (!ctx || !out) AMTK_FAIL("amtk_scan_logo_stream_create: null argument");
  if (w < 4 || h < 4 || w > 4096 || h > 4096) AMTK_FAIL("amtk_scan_create: bad geometry");
  if (imgx < 0 || imgy < 0) AMTK_FAIL("amtk_scan_logo_stream_create: negative scan position");
  if (max_frames < 0) AMTK_FAIL("amtk_scan_logo_stream_create: negative max_frames");
  amtk_scan_logo_stream* s = new amtk_scan_logo_stream();
  s->ctx = ctx; s->imgx = imgx; s->imgy = imgy; s->w = w; s->h = h; s->thy = thy; s->max_frames = max_frames; s->cb = cb;
  if (max_frames == 0) s->cutoff = 0;        // onFrame returns false on the first frame (:885)
  *out = s;
  return 1;
}

void amtk_scan_logo_stream_destroy(amtk_scan_logo_stream* s) {
  if (s) stream_destroy(s);                  // the stack is a stream-ordered allocation: the stream is idle when it goes
}

int amtk_scan_logo_stream_send(amtk_scan_logo_stream* s, const amtk_clip* frame, int64_t pos, int64_t size, int* more) {
  if (!s || !frame) AMTK_FAIL("amtk_scan_logo_stream_send: null argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  amtk_ctx* ctx = s->ctx;
  if (!stream_open(s->closed, "scan logo stream") || !scan_stream_check_frame(s, frame, size)) return 0;
  if (s->sent == INT32_MAX) AMTK_FAIL("scan logo stream: too many frames");
  if (!s->more()) {                          // past the cut-off: accepted, not copied, not counted (:884-885)
    s->sent += 1;
    if (more) *more = 0;
    return 1;
  }
  if (!s->have_fmt) {                        // the first frame fixes the format and sizes the batch buffers
    const RectPack rp = rect_pack(s->imgx, s->imgy, s->w, s->h, frame->log_uvx, frame->log_uvy, frame->bytes_per_sample, 1);
    const long long payload = rp.payload(), S = rp.stride;
    void* dr = nullptr;     // a failed allocation leaves have_fmt false: the next frame allocates all of them again
    if (!cuda_ok(cudaHostAlloc(s->hbatch.put(), (size_t)kScanStackBatch * S, cudaHostAllocDefault), "cudaHostAlloc(batch)") ||
        !cuda_ok(cudaMalloc(s->dbatch.put(), (size_t)kScanStackBatch * S), "cudaMalloc(batch)") ||
        !cuda_ok(cudaMalloc(s->dbg.put(), (size_t)kScanStackBatch * sizeof(int4)), "cudaMalloc(batch)") ||
        !cuda_ok(cudaHostAlloc(s->hres.put(), 2 * sizeof(int), cudaHostAllocMapped), "cudaHostAlloc(result)") ||
        !cuda_ok(cudaHostGetDevicePointer(&dr, s->hres, 0), "cudaHostGetDevicePointer"))
      return 0;
    s->dres = reinterpret_cast<int*>(dr);
    s->rp = rp; s->payload = payload; s->S = S; s->slot_host.assign(kScanStackBatch, 0);
    s->imgw = frame->width; s->imgh = frame->height; s->lx = frame->log_uvx; s->ly = frame->log_uvy;
    s->bps = frame->bytes_per_sample; s->bits = frame->bits_per_sample;
    s->have_fmt = true;
  }
  // the rectangle rows of Y, U and V into slot k (CopyYV12, :893-902)
  const int k = s->nbatch;
  if (!rect_copy(s->rp, frame, (frame->on_device ? s->dbatch.get() : s->hbatch.get()) + (size_t)k * s->S, true, ctx->stream))
    return stream_fail(s->closed);
  s->slot_host[k] = frame->on_device ? 0 : 1;
  s->nbatch += 1; s->sent += 1; s->reads += 1;
  s->last_pos = pos; s->last_size = size;
  if (s->reads % kScanStackBatch == 0 && !scan_stream_resolve(s)) return stream_fail(s->closed);
  if (more) *more = s->more() ? 1 : 0;
  return 1;
}

int amtk_scan_logo_stream_finish(amtk_scan_logo_stream* s, int service_id, const char* dstpath) {
  if (!s || !dstpath) AMTK_FAIL("amtk_scan_logo_stream_finish: null argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  if (!stream_open(s->closed, "scan logo stream")) return 0;
  s->closed = "finished";
  if (s->sent == 0) AMTK_FAIL("scan logo stream: finish without any frame sent (there is no first frame to take the format from)");
  if (!scan_stream_resolve(s)) return 0;
  amtk_clip stack{};
  stack.base = s->stack; stack.frame_stride = s->S;
  stack.off_u = s->rp.offU; stack.off_v = s->rp.offV;
  stack.width = s->w; stack.height = s->h; stack.pitch_y = (int)s->rp.pitchY; stack.pitch_uv = (int)s->rp.pitchC;
  stack.log_uvx = s->lx; stack.log_uvy = s->ly; stack.bytes_per_sample = s->bps; stack.bits_per_sample = s->bits;
  stack.num_frames = s->ngather; stack.on_device = 1;
  const StoredFrames st{ &stack, 0, 0, s->ngather, nullptr, s->ngather };
  return scan_logo_from_stored(s->ctx, st, s->w, s->h, s->thy, s->imgw, s->imgh, s->imgx, s->imgy, service_id, dstpath, s->cb);
}

int amtk_scan_logo_stream_counts(const amtk_scan_logo_stream* s, int* nread, int* ngather, int64_t* h2d_bytes) {
  if (!s) AMTK_FAIL("amtk_scan_logo_stream_counts: null stream");
  std::lock_guard<std::recursive_mutex> lock(s->ctx->mu);
  if (nread) *nread = s->cutoff >= 0 ? std::min(s->reads, s->cutoff) : s->reads;
  if (ngather) *ngather = s->ngather;
  if (h2d_bytes) *h2d_bytes = s->h2d;
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// erase
// ---------------------------------------------------------------------------------------------------------
// Delogo of frames [lo, hi) of the resident clip v (window w; the logo rectangle at (imgx - dx, imgy - dy)) with the device
// fades of frame lo at `fades`.
static int launch_erase(amtk_ctx* ctx, const amtk_logo* logo, const amtk_clip& v, const Window& w, int lo, int hi, int dx, int dy,
                        const float* fades) {
  const amtk::HostLogo& h = logo->host;
  EraseJob j;
  j.base = const_cast<uint8_t*>(w.dev_base); j.frame_stride = v.frame_stride;
  j.offU = v.off_u; j.offV = v.off_v;
  j.pitchY = v.pitch_y / v.bytes_per_sample; j.pitchUV = v.pitch_uv / v.bytes_per_sample;
  j.frame0 = lo - w.first; j.nframes = hi - lo;
  j.w = h.w; j.h = h.h; j.logUVx = h.logUVx; j.logUVy = h.logUVy; j.imgx = h.imgx - dx; j.imgy = h.imgy - dy;
  j.uvparity = (h.imgy / 2) % 2;                                             // LogoScan.hpp:1385, real frame position
  j.aY = logo->dA; j.bY = logo->dB; j.aU = logo->dAU; j.bU = logo->dBU; j.aV = logo->dAV; j.bV = logo->dBV;
  j.fades = fades;
  j.maxv = (float)((1 << v.bits_per_sample) - 1);
  if (v.bytes_per_sample == 1) erase_logo_kernel<uint8_t><<<hi - lo, 256, 0, ctx->stream>>>(j);
  else erase_logo_kernel<uint16_t><<<hi - lo, 256, 0, ctx->stream>>>(j);
  AMTK_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return 1;
}

int amtk_erase_logo_frames(amtk_ctx* ctx, const amtk_clip* clip, const amtk_logo* logo, int frame0, int nframes, const float* fades) {
  if (!ctx || !logo || !fades) AMTK_FAIL("amtk_erase_logo_frames: bad argument");
  if (!validate_clip(clip, true)) return 0;
  const amtk::HostLogo& h = logo->host;
  if (h.imgx < 0 || h.imgy < 0 || h.imgx + h.w > clip->width || h.imgy + h.h > clip->height) AMTK_FAIL("logo rectangle lies outside the frame");
  if (frame0 < 0 || nframes < 0 || frame0 + nframes > clip->num_frames) AMTK_FAIL("frame range outside the clip");
  if (nframes == 0) return 1;
  DevSelect ds(ctx); if (!ds.ok) return 0;
  if (!logo_ensure_device(logo, ctx, false)) return 0;
  if (!ctx->dout.ensure((size_t)nframes * 2 * sizeof(float))) return 0;
  AMTK_CUDA(cudaMemcpyAsync(ctx->dout.at(), fades, (size_t)nframes * 2 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  // Device clips are edited in place in HBM.  Host clips (the IClip::GetFrame surface: one MakeWritable'd CPU frame) move
  // only the three logo rectangles: up, Delogo kernel, back down -- not the reference's full-frame copy (LogoScan.hpp:1347).
  const int ok = for_each_roi_window(ctx, clip, frame0, nframes, h.imgx, h.imgy, h.w, h.h, true, true,
                                     [&](const amtk_clip& v, const Window& w, int lo, int hi, int dx, int dy) {
    return launch_erase(ctx, logo, v, w, lo, hi, dx, dy, ctx->dout.at<const float>() + (size_t)(lo - frame0) * 2);
  });
  if (!ok) return 0;
  AMTK_CUDA(cudaStreamSynchronize(ctx->stream));    // `fades` staging buffer is reused by later calls; host frames are complete
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// AMTEraseLogo(AMTAnalyzeLogo(...)) fed one decoded frame at a time (DESIGN.md section 3.3.2)
// ---------------------------------------------------------------------------------------------------------
// Frame f's three logo rectangles go into slot f % B of batch buffer f / B (RectPack layout, luma rows padded to 16 bytes
// so the evaluation kernels' TMA path runs): host frames row by row into the buffer's pinned twin, device frames with 2-D
// copies on the context's stream.  A batch buffer holds the fades of its B outputs, then its B slots.  The send that makes
// S >= min(N, (k+1)B + 8) launches batch k: one upload of the host slots sent since the last launch (per batch buffer
// touched), the evaluation kernels over the analysed frames among them (records into a ring of B + 16 rows: output n
// reads frames in [n - 8, n + 8] only, see the header), erase_fade_kernel for the batch's outputs, erase_logo_kernel on
// its slots, one download of the fades and slots into the pinned twin, and an event.  recv waits on that event only.
// CalcFade (LogoScan.hpp:1317-1341) of outputs [n0, n1) of a clip of N frames: code[n] = the fade of a uniform logoframe
// window (0 or 1), or 2 = CalcFade2 (outputs outside [n0, n1) get 2); analysed[f] = 1 for the frames whose records some
// CalcFade2 among them reads.  Returns how many frames that is.
static int erase_fade_plan(int N, const uint8_t* frame_result, int max_fade_length, int n0, int n1,
                           std::vector<uint8_t>& code, std::vector<uint8_t>& analysed) {
  code.assign((size_t)N, 2); analysed.assign((size_t)N, 0);
  int n_analysed = 0;
  for (int n = n0; n < n1; ++n) {
    if (frame_result) {
      const int half = max_fade_length >> 1;
      const uint8_t first = frame_result[std::max(0, std::min(N - 1, n - half))];
      bool uniform = true;
      for (int i = -half + 1; i <= half && uniform; ++i) uniform = frame_result[std::max(0, std::min(N - 1, n + i))] == first;
      if (uniform) code[(size_t)n] = frame_result[(size_t)n] == 2 ? 1 : 0;
    }
    if (code[(size_t)n] == 2)
      for (int i = -4; i <= 4; ++i) {
        const int f = calc_fade2_index(N, N, n, i);
        n_analysed += analysed[(size_t)f] ? 0 : 1;
        analysed[(size_t)f] = 1;
      }
  }
  return n_analysed;
}

struct amtk_erase_logo_stream : SlotStream<> {      // head: the fades of the batch's B outputs; slot: rp.stride
  amtk_erase_logo_stream() : SlotStream("erase logo stream", "erase batch") {}
  amtk_logo* logo = nullptr;                // the stream's own copy of the raw logo (Delogo's tables)
  amtk_logo *deint = nullptr, *fieldT = nullptr, *fieldB = nullptr;   // AMTAnalyzeLogo's logos, masks built
  int N = 0, ring = 0;
  std::vector<uint8_t> analysed;            // per frame: some CalcFade2 reads its record
  DevBuf<uint8_t> dcode;                    // per output: 0 / 1 = uniform logoframe window, 2 = CalcFade2
  DevBuf<float> drec;                       // record ring, frame f at row f % ring (null when nothing is analysed)
  RectPack rp;                              // slot layout
  int n_analysed = 0;                       // frames in the analysed set
  int uploaded = 0, n_analysed_done = 0;
};

namespace {

// One frame of a format the stream can take (the first frame's, once one was sent); sets the reason otherwise.
bool erase_stream_check_frame(const amtk_erase_logo_stream* s, const amtk_clip* c, const char* what) {
  if (!one_frame(c, "erase logo stream", what)) return false;
  if (s->have_fmt) {
    if (!same_format(s->fmt, c)) { set_error("erase logo stream: " + std::string(what) + "'s format differs from the first frame's"); return false; }
    return true;
  }
  if (!sample_bits_ok(c, "erase logo stream")) return false;
  const amtk::HostLogo& h = s->logo->host;
  if (c->log_uvx != h.logUVx || c->log_uvy != h.logUVy) { set_error("chroma subsampling mismatch"); return false; }
  if (h.imgx + h.w > c->width || h.imgy + h.h > c->height) { set_error("logo rectangle lies outside the frame"); return false; }
  return s->n_analysed == 0 || eval_plan_padded(h.w, h.h, c->bytes_per_sample);      // the plan at this sample size
}

// Launches batch k (outputs [kB, min(N, (k+1)B))); every frame it reads has been sent.
int erase_stream_launch(amtk_erase_logo_stream* s, int k) {
  amtk_ctx* ctx = s->ctx;
  const RectPack& rp = s->rp;
  const int lo = k * s->B, hi = std::min(s->N, lo + s->B);
  // upload: the host slots of frames [uploaded, sent), one copy per run of host slots in a batch buffer
  for (int f = s->uploaded; f < s->sent; f = (f / s->B + 1) * s->B) {
    const int first = f / s->B * s->B;
    if (!s->upload(s->batch(f / s->B), f - first, std::min(s->sent - first, s->B), rp.payload())) return 0;
  }
  // analysis: AMTAnalyzeLogo's records of the analysed frames among them, in runs inside one buffer and one ring turn
  for (int f = s->uploaded; f < s->sent;) {
    if (!s->analysed[(size_t)f]) { ++f; continue; }
    int e = f + 1;
    while (e < s->sent && s->analysed[(size_t)e] && e % s->B != 0 && e % s->ring != 0) ++e;
    const amtk_clip v = slot_view(s->fmt, rp, s->batch(f / s->B).d + s->head, rp.stride, s->B);
    const Window w{ reinterpret_cast<const uint8_t*>(v.base), f / s->B * s->B, s->B };
    const amtk::HostLogo& dh = s->deint->host;
    if (!analyze_impl(ctx, &v, dh.imgx, dh.imgy, s->deint, s->fieldT, s->fieldB, w, f, e, s->drec + (size_t)(f % s->ring) * 33, f)) return 0;
    s->n_analysed_done += e - f;
    f = e;
  }
  s->uploaded = s->sent;
  // fades, erase, download
  SlotBatch& b = s->batch(k);
  float* dfades = reinterpret_cast<float*>(b.d.get());
  erase_fade_kernel<<<(hi - lo + 255) / 256, 256, 0, ctx->stream>>>(s->dcode, s->drec, s->ring, s->N, lo, hi - lo, dfades);
  AMTK_CUDA(cudaGetLastError());
  const amtk::HostLogo& h = s->logo->host;
  EraseJob j;
  j.base = b.d + s->head; j.frame_stride = rp.stride; j.offU = rp.offU; j.offV = rp.offV;
  j.pitchY = (int)(rp.pitchY / rp.bps); j.pitchUV = (int)(rp.pitchC / rp.bps);
  j.frame0 = 0; j.nframes = hi - lo;
  j.w = h.w; j.h = h.h; j.logUVx = h.logUVx; j.logUVy = h.logUVy; j.imgx = 0; j.imgy = 0;
  j.uvparity = (h.imgy / 2) % 2;                                             // LogoScan.hpp:1385, real frame position
  j.aY = s->logo->dA; j.bY = s->logo->dB; j.aU = s->logo->dAU; j.bU = s->logo->dBU; j.aV = s->logo->dAV; j.bV = s->logo->dBV;
  j.fades = dfades;
  j.maxv = (float)((1 << s->fmt.bits_per_sample) - 1);
  if (rp.bps == 1) erase_logo_kernel<uint8_t><<<hi - lo, 256, 0, ctx->stream>>>(j);
  else erase_logo_kernel<uint16_t><<<hi - lo, 256, 0, ctx->stream>>>(j);
  AMTK_CUDA(cudaGetLastError());
  ctx->launches += 2;
  return s->seal(b, s->head + (size_t)(hi - lo) * s->slot, (int64_t)(hi - lo) * (rp.payload() + 2 * (int64_t)sizeof(float)));
}

}  // namespace

int amtk_erase_logo_stream_create(amtk_ctx* ctx, const amtk_logo* logo, float maskratio, int num_frames,
                                  const uint8_t* frame_result, int max_fade_length, int batch_size,
                                  amtk_erase_logo_stream** out) {
  if (!ctx || !logo || !out) AMTK_FAIL("amtk_erase_logo_stream_create: null argument");
  if (num_frames < 1) AMTK_FAIL("erase logo stream: num_frames must be >= 1");
  if (max_fade_length < 0) AMTK_FAIL("erase logo stream: max_fade_length must be >= 0");
  if (batch_size < 1 || batch_size > 256) AMTK_FAIL("erase logo stream: batch_size must be in [1,256]");
  if (!(maskratio > 0.0f) || maskratio > 1.0f) AMTK_FAIL("amtk_logo_create_mask: maskratio must be in (0,1]");
  if (logo->host.imgx < 0 || logo->host.imgy < 0) AMTK_FAIL("logo rectangle lies outside the frame");
  if (frame_result)
    for (int i = 0; i < num_frames; ++i)
      if (frame_result[i] > 2) AMTK_FAIL("erase logo stream: frame_result values must be 0, 1 or 2");
  const int N = num_frames;
  std::vector<uint8_t> code, analysed;
  const int n_analysed = erase_fade_plan(N, frame_result, max_fade_length, 0, N, code, analysed);
  std::unique_ptr<amtk_erase_logo_stream, void (*)(amtk_erase_logo_stream*)> s(new amtk_erase_logo_stream(), amtk_erase_logo_stream_destroy);
  s->ctx = ctx; s->N = N; s->B = batch_size; s->ring = batch_size + 16;
  s->analysed = std::move(analysed); s->n_analysed = n_analysed;
  amtk::HostLogo copy = logo->host;
  if (!logo_adopt(ctx, std::move(copy), &s->logo)) return 0;
  if (!amtk_logo_deint(logo, &s->deint) || !amtk_logo_create_mask(s->deint, maskratio) ||       // AMTAnalyzeLogo (:1177-1185)
      !amtk_logo_field(logo, 0, &s->fieldT) || !amtk_logo_create_mask(s->fieldT, maskratio) ||
      !amtk_logo_field(logo, 1, &s->fieldB) || !amtk_logo_create_mask(s->fieldB, maskratio))
    return 0;
  if (n_analysed > 0) {                     // what amtk_logo_analyze_frames refuses, before any frame is sent
    const amtk::HostLogo& dh = s->deint->host;
    if (dh.count() == 0 || s->fieldT->host.count() == 0 || s->fieldB->host.count() == 0) AMTK_FAIL("logo has no feature pixels");
    if (!eval_plan_padded(dh.w, dh.h, 1)) return 0;
  }
  DevSelect ds(ctx); if (!ds.ok) return 0;
  if (!logo_ensure_device(s->logo, ctx, false)) return 0;
  AMTK_CUDA(cudaMalloc(s->dcode.put(), (size_t)N));
  AMTK_CUDA(cudaMemcpy(s->dcode, code.data(), (size_t)N, cudaMemcpyHostToDevice));
  if (n_analysed > 0) AMTK_CUDA(cudaMalloc(s->drec.put(), (size_t)s->ring * 33 * sizeof(float)));
  *out = s.release();
  return 1;
}

void amtk_erase_logo_stream_destroy(amtk_erase_logo_stream* s) {
  if (!s) return;
  amtk_logo* logos[] = { s->logo, s->deint, s->fieldT, s->fieldB };
  stream_destroy(s);
  for (amtk_logo* l : logos) amtk_logo_destroy(l);
}

int amtk_erase_logo_stream_send(amtk_erase_logo_stream* s, const amtk_clip* frame) {
  if (!s || !frame) AMTK_FAIL("amtk_erase_logo_stream_send: null argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  amtk_ctx* ctx = s->ctx;
  if (!s->open(true)) return 0;
  if (s->sent >= s->N) AMTK_FAIL("erase logo stream: all num_frames frames were sent");
  if (!erase_stream_check_frame(s, frame, "the frame")) return 0;
  if (!s->have_fmt) {                        // the first frame fixes the format and the slot layout
    const amtk::HostLogo& h = s->logo->host;
    s->fmt = *frame; s->fmt.base = nullptr; s->fmt.num_frames = 1;
    s->rp = rect_pack(h.imgx, h.imgy, h.w, h.h, h.logUVx, h.logUVy, frame->bytes_per_sample, 16);
    s->slot = (size_t)s->rp.stride;
    s->head = ((size_t)s->B * 2 * sizeof(float) + 255) & ~(size_t)255;
    s->have_fmt = true;
  }
  const int f = s->sent;
  SlotBatch* b = s->batch_of(f);
  if (!b) return s->fail();
  if (!rect_copy(s->rp, frame, (frame->on_device ? b->d.get() : b->h.get()) + s->slot_at(f % s->B), true, ctx->stream)) return s->fail();
  b->host[(size_t)(f % s->B)] = frame->on_device ? 0 : 1;
  s->sent += 1;
  while ((long long)s->launched * s->B < s->N && s->sent >= std::min<long long>(s->N, (long long)(s->launched + 1) * s->B + 8))
    if (!erase_stream_launch(s, s->launched)) return s->fail();
  return 1;
}

int amtk_erase_logo_stream_recv(amtk_erase_logo_stream* s, const amtk_clip* dst, int* n, int* got, float* fades) {
  if (!s || !dst) AMTK_FAIL("amtk_erase_logo_stream_recv: null argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  amtk_ctx* ctx = s->ctx;
  if (!s->open(false) || !erase_stream_check_frame(s, dst, "dst")) return 0;
  if (got) *got = 0;
  const int ready = s->ready(s->sent == s->N, s->N);
  if (s->received >= ready) return 1;
  SlotBatch* b = s->front();
  if (!b) return 0;
  const int slot = s->received - s->first_batch * s->B;
  const size_t off = s->slot_at(slot);
  if (dst->on_device) {
    if (!rect_copy(s->rp, dst, b->d + off, false, ctx->stream) ||
        !cuda_ok(cudaStreamSynchronize(ctx->stream), "cudaStreamSynchronize")) return s->fail();
  } else if (!rect_copy(s->rp, dst, b->h + off, false, ctx->stream)) {
    return s->fail();
  }
  if (fades) { memcpy(fades, b->h + (size_t)slot * 2 * sizeof(float), 2 * sizeof(float)); }
  if (n) *n = s->received;
  if (got) *got = 1;
  s->received += 1;
  s->retire(ready);
  return 1;
}

int amtk_erase_logo_stream_counts(const amtk_erase_logo_stream* s, int* sent, int* received, int* analyzed,
                                  int64_t* h2d_bytes, int64_t* d2h_bytes) {
  if (!s) AMTK_FAIL("amtk_erase_logo_stream_counts: null stream");
  std::lock_guard<std::recursive_mutex> lock(s->ctx->mu);
  s->counts(sent, received, h2d_bytes, d2h_bytes);
  if (analyzed) *analyzed = s->n_analysed_done;
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// AMTEraseLogo(AMTAnalyzeLogo(...)) over a whole clip in one call (DESIGN.md section 3.3.4)
// ---------------------------------------------------------------------------------------------------------
// The records of the frames some output's CalcFade2 reads are computed by one analysis pass over a device list of those
// frames (three evaluations, records at row f of an N x 33 buffer), erase_fade_kernel decides every output's fades from
// them with ring = N, and then erase_logo_kernel edits the rectangles in place or erase_copy_kernel writes whole frames
// to dst.  Host clips in place: the ROI rows of the frames the records span are staged for the analysis, and the output
// range is staged, erased and written back as amtk_erase_logo_frames does.
namespace {

struct OwnedLogo {
  amtk_logo* l = nullptr;
  ~OwnedLogo() { amtk_logo_destroy(l); }
};

int launch_erase_copy(amtk_ctx* ctx, const amtk_clip* src, const amtk_clip* dst, const amtk_logo* logo, int frame0, int nframes,
                      const float* dfades) {
  const amtk::HostLogo& h = logo->host;
  const int bps = src->bytes_per_sample, lx = src->log_uvx, ly = src->log_uvy;
  const int wc = src->width >> lx, hc = src->height >> ly;
  EraseCopyJob j;
  j.src = reinterpret_cast<const uint8_t*>(src->base); j.dst = reinterpret_cast<uint8_t*>(const_cast<void*>(dst->base));
  j.sstride = src->frame_stride; j.dstride = dst->frame_stride;
  const long long so[3] = { 0, src->off_u, src->off_v }, d_o[3] = { 0, dst->off_u, dst->off_v };
  const int sp[3] = { src->pitch_y, src->pitch_uv, src->pitch_uv }, dp[3] = { dst->pitch_y, dst->pitch_uv, dst->pitch_uv };
  bool vec = ((reinterpret_cast<uintptr_t>(src->base) | reinterpret_cast<uintptr_t>(dst->base)) & 15) == 0 &&
             ((src->frame_stride | dst->frame_stride) & 15) == 0;
  for (int p = 0; p < 3; ++p) {
    j.s_off[p] = so[p]; j.d_off[p] = d_o[p]; j.s_pitch[p] = sp[p]; j.d_pitch[p] = dp[p];
    j.row_bytes[p] = (p ? wc : src->width) * bps; j.rows[p] = p ? hc : src->height;
    j.rx[p] = p ? h.imgx >> lx : h.imgx; j.ry[p] = p ? h.imgy >> ly : h.imgy;
    j.rw[p] = p ? h.w >> lx : h.w;       j.rh[p] = p ? h.h >> ly : h.h;
    vec = vec && ((so[p] | d_o[p] | sp[p] | dp[p]) & 15) == 0;
  }
  j.a[0] = logo->dA; j.a[1] = logo->dAU; j.a[2] = logo->dAV;
  j.b[0] = logo->dB; j.b[1] = logo->dBU; j.b[2] = logo->dBV;
  j.fades = dfades; j.src0 = frame0; j.nframes = nframes;
  j.pieces_y = (src->width * bps + 15) >> 4;
  j.maxv = (float)((1 << src->bits_per_sample) - 1);
  j.uvparity = (h.imgy / 2) % 2;                                             // LogoScan.hpp:1385
  const dim3 grid((unsigned)(((long long)src->height * j.pieces_y + 255) / 256), 3, (unsigned)std::min(nframes, 65535));
  if (bps == 1) { if (vec) erase_copy_kernel<uint8_t, true><<<grid, 256, 0, ctx->stream>>>(j); else erase_copy_kernel<uint8_t, false><<<grid, 256, 0, ctx->stream>>>(j); }
  else { if (vec) erase_copy_kernel<uint16_t, true><<<grid, 256, 0, ctx->stream>>>(j); else erase_copy_kernel<uint16_t, false><<<grid, 256, 0, ctx->stream>>>(j); }
  AMTK_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return 1;
}

}  // namespace

int amtk_erase_logo_clip(amtk_ctx* ctx, const amtk_clip* src, const amtk_clip* dst, const amtk_logo* logo, float maskratio,
                         const uint8_t* frame_result, int max_fade_length, int frame0, int nframes, float* fades_out) {
  if (!ctx || !src || !logo) AMTK_FAIL("amtk_erase_logo_clip: null argument");
  if (!validate_clip(src, true) || !sample_bits_ok(src, "amtk_erase_logo_clip")) return 0;
  const int N = src->num_frames;
  if (max_fade_length < 0) AMTK_FAIL("amtk_erase_logo_clip: max_fade_length must be >= 0");
  if (!(maskratio > 0.0f) || maskratio > 1.0f) AMTK_FAIL("amtk_logo_create_mask: maskratio must be in (0,1]");
  const amtk::HostLogo& h = logo->host;
  if (src->log_uvx != h.logUVx || src->log_uvy != h.logUVy) AMTK_FAIL("chroma subsampling mismatch");
  if (h.imgx < 0 || h.imgy < 0 || h.imgx + h.w > src->width || h.imgy + h.h > src->height) AMTK_FAIL("logo rectangle lies outside the frame");
  if (frame0 < 0 || nframes < 0 || frame0 > N - nframes) AMTK_FAIL("frame range outside the clip");
  if (frame_result)
    for (int i = 0; i < N; ++i)
      if (frame_result[i] > 2) AMTK_FAIL("amtk_erase_logo_clip: frame_result values must be 0, 1 or 2");
  if (dst) {
    if (!validate_clip(dst, true)) return 0;
    if (!dst->on_device) AMTK_FAIL("amtk_erase_logo_clip: dst must be device resident");
    if (!src->on_device) AMTK_FAIL("amtk_erase_logo_clip: an out-of-place call needs a device-resident src");
    if (!same_format(*src, dst)) AMTK_FAIL("amtk_erase_logo_clip: dst's format differs from src's");
    if (dst->num_frames < nframes) AMTK_FAIL("amtk_erase_logo_clip: dst holds fewer than nframes frames");
    uintptr_t s0, s1, d0, d1;
    clip_span(src, &s0, &s1); clip_span(dst, &d0, &d1);
    if (s0 < d1 && d0 < s1) AMTK_FAIL("amtk_erase_logo_clip: dst overlaps src");
  }
  // the outputs' CalcFade and the frames whose records they read (ascending)
  std::vector<uint8_t> code, analysed;
  const int M = erase_fade_plan(N, frame_result, max_fade_length, frame0, frame0 + nframes, code, analysed);
  std::vector<int> list;
  list.reserve((size_t)M);
  for (int f = 0; f < N; ++f) if (analysed[(size_t)f]) list.push_back(f);
  OwnedLogo deint, fieldT, fieldB;                                              // AMTAnalyzeLogo (:1177-1185)
  if (!amtk_logo_deint(logo, &deint.l) || !amtk_logo_create_mask(deint.l, maskratio) ||
      !amtk_logo_field(logo, 0, &fieldT.l) || !amtk_logo_create_mask(fieldT.l, maskratio) ||
      !amtk_logo_field(logo, 1, &fieldB.l) || !amtk_logo_create_mask(fieldB.l, maskratio))
    return 0;
  if (M > 0) {                              // what amtk_logo_analyze_frames refuses, before any launch
    if (deint.l->host.count() == 0 || fieldT.l->host.count() == 0 || fieldB.l->host.count() == 0) AMTK_FAIL("logo has no feature pixels");
    if (!eval_plan_padded(h.w, h.h, src->bytes_per_sample)) return 0;
  }
  if (nframes == 0) return 1;
  DevSelect ds(ctx); if (!ds.ok) return 0;
  if (!logo_ensure_device(logo, ctx, false)) return 0;
  // one buffer: records [N][33] (when some frame is analysed), fades [nframes][2], the frame list, the fade codes
  auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t rec_b = M > 0 ? (size_t)N * 33 * sizeof(float) : 0, fad_b = (size_t)nframes * 2 * sizeof(float);
  const size_t list_b = (size_t)M * sizeof(int), off_f = up(rec_b), off_l = off_f + up(fad_b), off_c = off_l + up(list_b);
  if (!ctx->erase_clip.ensure(off_c + (size_t)N)) return 0;
  float* drec = ctx->erase_clip.at<float>();
  float* dfades = ctx->erase_clip.at<float>(off_f);
  int* dlist = ctx->erase_clip.at<int>(off_l);
  uint8_t* dcode = ctx->erase_clip.at(off_c);
  AMTK_CUDA(cudaMemcpyAsync(dcode, code.data(), (size_t)N, cudaMemcpyHostToDevice, ctx->stream));
  if (M > 0) AMTK_CUDA(cudaMemcpyAsync(dlist, list.data(), list_b, cudaMemcpyHostToDevice, ctx->stream));
  long long h2d = 0;
  // 1. analysis of the listed frames, before anything is written
  if (M > 0) {
    const amtk::HostLogo& dh = deint.l->host;
    if (src->on_device) {
      const Window w{ reinterpret_cast<const uint8_t*>(src->base), 0, N };
      if (!analyze_impl(ctx, src, 0, 0, deint.l, fieldT.l, fieldB.l, w, 0, M, drec, 0, dlist)) return 0;
    } else {
      if (!for_each_roi_window(ctx, src, list.front(), list.back() - list.front() + 1, dh.imgx, dh.imgy, dh.w, dh.h, false, false,
                               [&](const amtk_clip& v, const Window& w, int lo, int hi, int dx, int dy) {
            const int plo = (int)(std::lower_bound(list.begin(), list.end(), lo) - list.begin());
            const int phi = (int)(std::lower_bound(list.begin(), list.end(), hi) - list.begin());
            return plo == phi ? 1 : analyze_impl(ctx, &v, dx, dy, deint.l, fieldT.l, fieldB.l, w, plo, phi, drec, 0, dlist); }))
        return 0;
      h2d += ctx->h2d_bytes_last;
    }
  }
  // 2. fades of every output (frame f's record at row f)
  erase_fade_kernel<<<(nframes + 255) / 256, 256, 0, ctx->stream>>>(dcode, drec, N, N, frame0, nframes, dfades);
  AMTK_CUDA(cudaGetLastError());
  ctx->launches += 1;
  // 3. erase
  if (dst) {
    if (!launch_erase_copy(ctx, src, dst, logo, frame0, nframes, dfades)) return 0;
  } else if (src->on_device) {
    const Window w{ reinterpret_cast<const uint8_t*>(src->base), 0, N };
    if (!launch_erase(ctx, logo, *src, w, frame0, frame0 + nframes, 0, 0, dfades)) return 0;
  } else {
    if (!for_each_roi_window(ctx, src, frame0, nframes, h.imgx, h.imgy, h.w, h.h, true, true,
                             [&](const amtk_clip& v, const Window& w, int lo, int hi, int dx, int dy) {
          return launch_erase(ctx, logo, v, w, lo, hi, dx, dy, dfades + (size_t)(lo - frame0) * 2); }))
      return 0;
    h2d += ctx->h2d_bytes_last;
  }
  if (!src->on_device) ctx->h2d_bytes_last = h2d;
  if (fades_out) AMTK_CUDA(cudaMemcpyAsync(fades_out, dfades, fad_b, cudaMemcpyDeviceToHost, ctx->stream));
  AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// LogoFrame::ScanFrame fed one decoded frame at a time (DESIGN.md section 3.3.3)
// ---------------------------------------------------------------------------------------------------------
// Frame f goes into slot f % B of batch buffer f / B.  A slot holds the luma rectangle of every evaluated logo (one
// luma-only RectPack each, rows as the frame is addressed, padded to 16 bytes so the evaluation kernels' TMA path runs):
// host frames row by row into the buffer's pinned twin, device frames by logo_rect_gather_kernel on the context's stream.
// A batch buffer holds the results of its B frames, then its B slots.  Launching batch k uploads each run of host slots in
// one copy, runs launch_eval per evaluated logo over the slots (rectangle at (0, 0)), downloads the result rows into the
// pinned twin and records an event; recv waits on that event only.
struct amtk_logo_scan_stream : SlotStream<> {       // head: the result rows of the batch's B frames
  amtk_logo_scan_stream() : SlotStream("logo scan stream", "logo scan batch") {}
  std::vector<amtk_logo*> logos;            // the stream's own copies (nullptr: an invalid logo)
  bool reference_pitch = false;
  std::vector<uint8_t> evaluated;           // per logo: evaluated on frames of this format
  std::vector<int> eval;                    // the evaluated logos
  std::vector<RectPack> rp;                 // per evaluated logo: its rectangle in a slot ...
  std::vector<long long> rect_off;          // ... at this byte offset
  long long payload = 0;                    // rectangle bytes per frame
  DevBuf<LogoRect> drects;                  // logo_rect_gather_kernel's table
  int gather_blocks = 0;
  int nlogos() const { return (int)logos.size(); }
};

namespace {

bool logo_scan_evaluates(const amtk_logo* lg, const amtk_clip* c) {      // LogoScan.hpp:1551-1558
  return lg && lg->host.imgw == c->width && lg->host.imgh == c->height;
}

// Luma elements from one addressed row to the next: the byte pitch itself for 2-byte samples under reference_pitch.
int logo_scan_pitch(const amtk_logo_scan_stream* s, const amtk_clip* c) {
  return s->reference_pitch && c->bytes_per_sample == 2 ? c->pitch_y : c->pitch_y / c->bytes_per_sample;
}

// One frame the stream can take; sets the reason otherwise.
bool logo_scan_check_frame(const amtk_logo_scan_stream* s, const amtk_clip* c) {
  if (!one_frame(c, "logo scan stream", "the frame")) return false;
  if (s->have_fmt && !same_format(s->fmt, c)) { set_error("logo scan stream: the frame's format differs from the first frame's"); return false; }
  if (!sample_bits_ok(c, "logo scan stream")) return false;
  const int pitch = logo_scan_pitch(s, c);
  for (const amtk_logo* lg : s->logos) {
    if (!logo_scan_evaluates(lg, c)) continue;
    if (!roi_inside(lg->host, c, pitch)) { set_error("logo rectangle lies outside the frame"); return false; }
    if (!s->have_fmt && !eval_plan_padded(lg->host.w, lg->host.h, c->bytes_per_sample)) return false;      // the plan at this sample size
  }
  return true;
}

// The first frame fixes the format, the evaluated logos, the slot layout and the gather table.
int logo_scan_layout(amtk_logo_scan_stream* s, const amtk_clip* c) {
  const int bps = c->bytes_per_sample;
  std::vector<LogoRect> table;
  s->evaluated.assign((size_t)s->nlogos(), 0);
  long long off = 0;
  for (int i = 0; i < s->nlogos(); ++i) {
    if (!logo_scan_evaluates(s->logos[(size_t)i], c)) continue;
    const amtk::HostLogo& h = s->logos[(size_t)i]->host;
    const RectPack r = rect_pack(h.imgx, h.imgy, h.w, h.h, c->log_uvx, c->log_uvy, bps, 16, true);
    s->evaluated[(size_t)i] = 1;
    s->eval.push_back(i); s->rp.push_back(r); s->rect_off.push_back(off);
    table.push_back(LogoRect{ off, h.imgx * bps, h.imgy, h.w * bps, h.h, (int)r.pitchY });
    s->gather_blocks = std::max(s->gather_blocks, ((h.w * bps + 15) / 16 * h.h + 255) / 256);
    s->payload += r.payload();
    off += r.stride;
  }
  s->slot = (size_t)off;
  s->head = ((size_t)s->B * s->nlogos() * 2 * sizeof(float) + 255) & ~(size_t)255;
  if (!table.empty()) {
    AMTK_CUDA(cudaMalloc(s->drects.put(), table.size() * sizeof(LogoRect)));
    AMTK_CUDA(cudaMemcpy(s->drects, table.data(), table.size() * sizeof(LogoRect), cudaMemcpyHostToDevice));
  }
  s->fmt = *c; s->fmt.base = nullptr; s->fmt.num_frames = 1;
  s->have_fmt = true;
  return 1;
}

// Launches batch k (frames [kB, min(S, (k+1)B))); all of them have been sent.
int logo_scan_launch(amtk_logo_scan_stream* s, int k) {
  static const float kFades01[2] = { 0.0f, 1.0f };
  amtk_ctx* ctx = s->ctx;
  SlotBatch& b = s->batch(k);
  const int n = std::min(s->sent - k * s->B, s->B);
  if (!s->upload(b, 0, n, s->payload)) return 0;
  float* dres = reinterpret_cast<float*>(b.d.get());
  for (size_t j = 0; j < s->eval.size(); ++j) {
    const int i = s->eval[j];
    const amtk_logo* lg = s->logos[(size_t)i];
    // the slots as a clip of n frames holding this logo's rectangle at (0, 0)
    const amtk_clip v = slot_view(s->fmt, s->rp[j], b.d + s->head + s->rect_off[j], (long long)s->slot, n);
    const Window w{ reinterpret_cast<const uint8_t*>(v.base), 0, n };
    EvalSpec sp{ lg, 0, 0, lg->host.w, lg->host.h, 0, 0, lg->host.w, 2, kFades01, 0, i * 2, 1 };
    if (!launch_eval(ctx, &v, w, 0, n, v.width, sp, dres, s->nlogos() * 2, 0, ctx->stream, 0)) return 0;
  }
  const size_t res = (size_t)n * (size_t)s->nlogos() * 2 * sizeof(float);
  return s->seal(b, res, (int64_t)res);
}

}  // namespace

// The logos of a stream that evaluates ScanFrame: what amtk_logo_scan_frames refuses, checked before any frame is sent.
static int stream_logos_ok(amtk_logo* const* logos, int nlogos) {
  for (int i = 0; i < nlogos; ++i) {
    const amtk_logo* lg = logos[i];
    if (!lg) continue;
    if (!lg->has_mask) AMTK_FAIL("logo has no mask: call amtk_logo_create_mask first");
    const amtk::HostLogo& h = lg->host;
    if (h.count() == 0) AMTK_FAIL("logo has no feature pixels");
    if (!eval_plan_padded(h.w, h.h, 1)) return 0;
  }
  return 1;
}

// A stream's own copies of checked logos (nullptr stays nullptr), in HBM; the caller may destroy its logos afterwards.
static int stream_logos_copy(amtk_ctx* ctx, amtk_logo* const* logos, int nlogos, std::vector<amtk_logo*>* dst) {
  dst->assign((size_t)nlogos, nullptr);
  for (int i = 0; i < nlogos; ++i) {
    amtk_logo* src = logos[i];
    if (!src) continue;
    std::lock_guard<std::mutex> lock(src->mu);
    amtk::HostLogo copy = src->host;
    logo_adopt(ctx, std::move(copy), &(*dst)[(size_t)i]);
    (*dst)[(size_t)i]->countPad = src->countPad;
    (*dst)[(size_t)i]->has_mask = true;
  }
  DevSelect ds(ctx); if (!ds.ok) return 0;
  for (amtk_logo* l : *dst)
    if (l && !logo_ensure_device(l, ctx, true)) return 0;
  return 1;
}

int amtk_logo_scan_stream_create(amtk_ctx* ctx, amtk_logo* const* logos, int nlogos, int batch_size,
                                 int reference_pitch, amtk_logo_scan_stream** out) {
  if (!ctx || !logos || !out || nlogos < 1) AMTK_FAIL("amtk_logo_scan_stream_create: bad argument");
  if (batch_size < 1 || batch_size > 256) AMTK_FAIL("logo scan stream: batch_size must be in [1,256]");
  if (!stream_logos_ok(logos, nlogos)) return 0;
  std::unique_ptr<amtk_logo_scan_stream, void (*)(amtk_logo_scan_stream*)> s(new amtk_logo_scan_stream(), amtk_logo_scan_stream_destroy);
  s->ctx = ctx; s->B = batch_size; s->reference_pitch = reference_pitch != 0;
  if (!stream_logos_copy(ctx, logos, nlogos, &s->logos)) return 0;
  *out = s.release();
  return 1;
}

void amtk_logo_scan_stream_destroy(amtk_logo_scan_stream* s) {
  if (!s) return;
  const std::vector<amtk_logo*> logos = s->logos;
  stream_destroy(s);
  for (amtk_logo* l : logos) amtk_logo_destroy(l);
}

int amtk_logo_scan_stream_send(amtk_logo_scan_stream* s, const amtk_clip* frame) {
  if (!s || !frame) AMTK_FAIL("amtk_logo_scan_stream_send: null argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  amtk_ctx* ctx = s->ctx;
  if (!s->open(true) || !logo_scan_check_frame(s, frame)) return 0;
  if (!s->have_fmt && !logo_scan_layout(s, frame)) return s->fail();
  const int f = s->sent;
  SlotBatch* b = s->batch_of(f);
  if (!b) return s->fail();
  const size_t off = s->slot_at(f % s->B);
  const long long step = (long long)logo_scan_pitch(s, frame) * frame->bytes_per_sample;
  if (frame->on_device) {
    if (!s->eval.empty()) {
      logo_rect_gather_kernel<<<dim3(s->gather_blocks, (unsigned)s->eval.size()), 256, 0, ctx->stream>>>(
          reinterpret_cast<const uint8_t*>(frame->base), step, b->d + off, s->drects);
      if (!cuda_ok(cudaGetLastError(), "logo_rect_gather_kernel")) return s->fail();
      ctx->launches += 1;
    }
  } else {
    for (size_t j = 0; j < s->eval.size(); ++j)
      if (!rect_copy(s->rp[j], frame, b->h + off + s->rect_off[j], true, ctx->stream, step)) return s->fail();
  }
  b->host[(size_t)(f % s->B)] = frame->on_device ? 0 : 1;
  s->sent += 1;
  if (s->sent % s->B == 0 && !logo_scan_launch(s, s->launched)) return s->fail();
  return 1;
}

int amtk_logo_scan_stream_finish(amtk_logo_scan_stream* s) {
  if (!s) AMTK_FAIL("amtk_logo_scan_stream_finish: null stream");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  if (!s->open(true)) return 0;
  if (s->sent > s->launched * s->B && !logo_scan_launch(s, s->launched)) return s->fail();
  s->finished = true;
  return 1;
}

int amtk_logo_scan_stream_recv(amtk_logo_scan_stream* s, float* out, int max_frames, int* got) {
  if (!s || !out || !got || max_frames < 0) AMTK_FAIL("amtk_logo_scan_stream_recv: bad argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  if (!s->open(false)) return 0;
  *got = 0;
  const int ready = s->ready(s->finished, s->sent);
  const int L = s->nlogos();
  while (*got < max_frames && s->received < ready) {
    const SlotBatch* b = s->front();
    if (!b) return 0;
    const int lo = s->first_batch * s->B, hi = std::min(ready, lo + s->B);
    const int take = std::min(max_frames - *got, hi - s->received);
    const float* res = reinterpret_cast<const float*>(b->h.get());
    for (int r = 0; r < take; ++r) {
      const float* src = res + (size_t)(s->received + r - lo) * L * 2;
      float* dst = out + (size_t)(*got + r) * L * 2;
      for (int i = 0; i < L; ++i) {
        dst[2 * i] = s->evaluated[(size_t)i] ? src[2 * i] : 0.0f;
        dst[2 * i + 1] = s->evaluated[(size_t)i] ? src[2 * i + 1] : -1.0f;
      }
    }
    s->received += take; *got += take;
    s->retire(ready);
  }
  return 1;
}

int amtk_logo_scan_stream_counts(const amtk_logo_scan_stream* s, int* sent, int* received, int64_t* h2d_bytes, int64_t* d2h_bytes) {
  if (!s) AMTK_FAIL("amtk_logo_scan_stream_counts: null stream");
  s->counts(sent, received, h2d_bytes, d2h_bytes);
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// the fused step fed one decoded frame at a time, and the comb stream: the same without logos (DESIGN.md sections 3.1d
// and 3.1e)
// ---------------------------------------------------------------------------------------------------------
// Frame f goes into frame slot f % B of batch buffer f / B.  A batch buffer holds the batch's n counter rows, then its n
// score rows (so that one download carries both), then, at a fixed offset, the watchdog record (res_off bytes in all);
// then one halo slot, then B frame slots; every slot is one frame in the stream's layout (stream_frame_layout of the first
// frame).  Host frames are copied into the buffer's pinned twin, device frames into the buffer on the context's stream.
// Launching batch k uploads each run of host slots in one copy, copies batch k-1's last slot into the halo slot, runs
// scan_comb_window over the slots as a device clip (halo, then frames kB..), downloads the result rows into the pinned twin
// and records an event; recv waits on that event only.  The logo items, or the logo kernels after the comb kernel, read
// the rectangles from the slots; without logos scan_comb_window is launch_comb alone.
// watched: the launch ran the band form and left its watchdog record after the rows; n: the batch's frames (its result rows)
struct ScanCombBatch : SlotBatch { bool watched = false; int n = 0; };

namespace {
constexpr size_t kCombRow = 12 * sizeof(int32_t);      // one frame's counters
}  // namespace

struct amtk_scan_comb_stream : SlotStream<ScanCombBatch> {   // fmt: one slot, the first frame's format in the stream's layout
  explicit amtk_scan_comb_stream(const char* name_ = "scan comb stream", const char* batch_name_ = "scan comb batch")
      : SlotStream(name_, batch_name_) {}
  virtual ~amtk_scan_comb_stream() = default;      // a comb stream is destroyed as this type
  amtk_comb_params prm{};
  std::vector<amtk_logo*> logos;            // the stream's own copies (nullptr: an invalid logo); none in a comb stream
  bool reference_pitch = false;             // 2-byte Y planes addressed with ScanFrame's byte-pitch row step
  size_t res_off = 0;                       // bytes before the halo slot
  int nlogos() const { return (int)logos.size(); }
  size_t row_bytes() const { return kCombRow + logos.size() * 2 * sizeof(float); }      // one frame's results
};

struct amtk_comb_stream : amtk_scan_comb_stream {
  amtk_comb_stream() : amtk_scan_comb_stream("comb stream", "comb batch") {}
};

namespace {

// Whether the logo kernels of s address frames of c's format with ScanFrame's byte-pitch row step.
bool scan_comb_byte_step(const amtk_scan_comb_stream* s, const amtk_clip* c) {
  return s->reference_pitch && c->bytes_per_sample == 2;
}

// One frame the stream can take; sets the reason otherwise.  The first frame is checked as amtk_scan_comb_frames checks a
// clip, and every evaluated logo's rectangle must lie inside it.  Under the byte-pitch row step every frame is checked as
// the logo scan stream checks it: the rectangle, as addressed, must lie inside the frame's Y plane.
bool scan_comb_check_frame(const amtk_scan_comb_stream* s, const amtk_clip* c) {
  if (!one_frame(c, s->name, "the frame")) return false;
  if (s->have_fmt && !same_format(s->fmt, c)) {
    set_error(std::string(s->name) + ": the frame's format differs from the first frame's");
    return false;
  }
  if (!s->have_fmt) {
    if (!comb_thresholds_ok(&s->prm, c->bytes_per_sample)) return false;
    for (const amtk_logo* lg : s->logos) {
      if (!logo_scan_evaluates(lg, c)) continue;
      const amtk::HostLogo& h = lg->host;
      if (h.imgx < 0 || h.imgy < 0 || h.imgx + h.w > c->width || h.imgy + h.h > c->height) {
        set_error("logo rectangle lies outside the frame");
        return false;
      }
      if (!eval_plan_padded(h.w, h.h, c->bytes_per_sample)) return false;      // the plan at this sample size
    }
  }
  if (scan_comb_byte_step(s, c))
    for (const amtk_logo* lg : s->logos)
      if (logo_scan_evaluates(lg, c) && !roi_inside(lg->host, c, c->pitch_y)) {
        set_error("logo rectangle lies outside the frame");
        return false;
      }
  return true;
}

// Launches batch k (frames [kB, min(S, (k+1)B))); all of them have been sent, and batch k-1 is still held.
int scan_comb_launch(amtk_scan_comb_stream* s, int k) {
  amtk_ctx* ctx = s->ctx;
  ScanCombBatch& b = s->batch(k);
  const int lo = k * s->B, n = std::min(s->sent - lo, s->B);
  if (!s->upload(b, 0, n, (int64_t)s->slot)) return 0;
  if (k > 0)             // the frame before the batch: batch k-1's last slot, in HBM since that batch's launch
    AMTK_CUDA(cudaMemcpyAsync(b.d + s->res_off, s->batch(k - 1).d + s->slot_at(s->B - 1), s->slot, cudaMemcpyDeviceToDevice, ctx->stream));
  // the slots as a device clip of frames [kB - 1, kB + n) (batch 0: [0, n), so that frame 0 is its own previous frame)
  const uint8_t* base = b.d + (k > 0 ? s->res_off : s->head);
  amtk_clip v = s->fmt;
  v.base = base; v.num_frames = n + (k > 0 ? 1 : 0);
  const Window w{ base, k > 0 ? lo - 1 : 0, v.num_frames };
  b.n = n;
  b.watched = comb_runs_band(ctx, &v, w);
  int* dcounts = reinterpret_cast<int*>(b.d.get());
  float* dscores = reinterpret_cast<float*>(b.d + (size_t)n * kCombRow);
  // the byte-pitch row step on the slots: the slot's byte pitch as element pitch (DESIGN.md section 3.1e)
  const int pitch_override = scan_comb_byte_step(s, &v) ? v.pitch_y : 0;
  if (!scan_comb_window(ctx, &v, w, lo, lo + n, s->logos.data(), s->nlogos(), &s->prm, dscores, dcounts, lo, pitch_override)) return 0;
  if (b.watched)
    AMTK_CUDA(cudaMemcpyAsync(b.h + (size_t)s->B * s->row_bytes(), ws_watch_record(ctx), 8 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  return s->seal(b, (size_t)n * s->row_bytes(), (int64_t)n * (int64_t)s->row_bytes());
}

// Sets up s, a new stream, over nlogos logos (none: a comb stream, which makes no CUDA call here); deletes s on a refusal.
int scan_comb_stream_make(amtk_scan_comb_stream* s, amtk_ctx* ctx, amtk_logo* const* logos, int nlogos,
                          const amtk_comb_params* params, int batch_size, bool reference_pitch) {
  std::unique_ptr<amtk_scan_comb_stream> owned(s);        // nothing of CUDA's until the logos are copied
  if (batch_size < 1 || batch_size > 256) AMTK_FAIL(std::string(s->name) + ": batch_size must be in [1,256]");
  const int all[6] = { params->th_move_y, params->th_shima_y, params->th_lshima_y, params->th_move_c, params->th_shima_c, params->th_lshima_c };
  for (int v : all) if (v < 1) AMTK_FAIL("comb: thresholds must be >= 1");      // the rest depends on the sample size
  if (!stream_logos_ok(logos, nlogos)) return 0;
  s->ctx = ctx; s->prm = *params; s->B = batch_size; s->reference_pitch = reference_pitch;
  owned.release();
  if (nlogos > 0 && !stream_logos_copy(ctx, logos, nlogos, &s->logos)) { amtk_scan_comb_stream_destroy(s); return 0; }
  return 1;
}

// Up to max_frames result rows: counters into counts, and scores into scores when the stream has logos.
int scan_comb_recv(amtk_scan_comb_stream* s, float* scores, int32_t* counts, int max_frames, int* got) {
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  if (!s->open(false)) return 0;
  *got = 0;
  const int ready = s->ready(s->finished, s->sent);
  const size_t srow = (size_t)s->nlogos() * 2 * sizeof(float);
  while (*got < max_frames && s->received < ready) {
    const ScanCombBatch* b = s->front();
    if (!b) return 0;
    const int lo = s->first_batch * s->B, hi = std::min(ready, lo + s->B);
    const uint8_t* res = b->h.get();
    const int32_t* wd = reinterpret_cast<const int32_t*>(res + (size_t)s->B * s->row_bytes());
    if (b->watched && wd[0]) {           // this batch's own record: no other comb call on the context can have consumed it
      char msg[256];
      snprintf(msg, sizeof(msg), "%s: a device-side wait of the batch of frames %d.. timed out (wait %d, step %d, CTA %d, thread %d, parity %d); its %s are not valid",
               s->name, lo, wd[1], wd[2], wd[3], wd[4], wd[5], srow ? "results" : "counters");
      set_error(msg);
      s->closed = "a device-side wait timed out";
      return 0;
    }
    const int take = std::min(max_frames - *got, hi - s->received), r = s->received - lo;
    memcpy(counts + (size_t)*got * 12, res + (size_t)r * kCombRow, (size_t)take * kCombRow);
    if (srow)
      memcpy(reinterpret_cast<uint8_t*>(scores) + (size_t)*got * srow, res + (size_t)b->n * kCombRow + (size_t)r * srow, (size_t)take * srow);
    s->received += take; *got += take;
    s->retire(ready);
  }
  return 1;
}

}  // namespace

static int scan_comb_stream_create_impl(amtk_ctx* ctx, amtk_logo* const* logos, int nlogos, const amtk_comb_params* params,
                                        int batch_size, bool reference_pitch, amtk_scan_comb_stream** out, const char* name) {
  if (!ctx || !logos || !params || !out || nlogos < 1) AMTK_FAIL(std::string(name) + ": bad argument");
  amtk_scan_comb_stream* s = new amtk_scan_comb_stream();
  if (!scan_comb_stream_make(s, ctx, logos, nlogos, params, batch_size, reference_pitch)) return 0;
  *out = s;
  return 1;
}

int amtk_scan_comb_stream_create(amtk_ctx* ctx, amtk_logo* const* logos, int nlogos, const amtk_comb_params* params,
                                 int batch_size, amtk_scan_comb_stream** out) {
  return scan_comb_stream_create_impl(ctx, logos, nlogos, params, batch_size, false, out, "amtk_scan_comb_stream_create");
}

int amtk_scan_comb_stream_create_pitch(amtk_ctx* ctx, amtk_logo* const* logos, int nlogos, const amtk_comb_params* params,
                                       int batch_size, int reference_pitch, amtk_scan_comb_stream** out) {
  return scan_comb_stream_create_impl(ctx, logos, nlogos, params, batch_size, reference_pitch != 0, out,
                                      "amtk_scan_comb_stream_create_pitch");
}

void amtk_scan_comb_stream_destroy(amtk_scan_comb_stream* s) {
  if (!s) return;
  const std::vector<amtk_logo*> logos = s->logos;
  stream_destroy(s);
  for (amtk_logo* l : logos) amtk_logo_destroy(l);
}

int amtk_scan_comb_stream_send(amtk_scan_comb_stream* s, const amtk_clip* frame) {
  if (!s || !frame) AMTK_FAIL("amtk_scan_comb_stream_send: null argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  if (!s->open(true) || !scan_comb_check_frame(s, frame)) return 0;
  if (s->sent == INT32_MAX) AMTK_FAIL(std::string(s->name) + ": too many frames");
  if (!s->have_fmt) {    // the first frame fixes the slot layout
    s->fmt = stream_frame_layout(*frame, frame->bytes_per_sample, frame->bits_per_sample);
    s->res_off = ((size_t)s->B * s->row_bytes() + 8 * sizeof(int) + 255) & ~(size_t)255;
    s->slot = (size_t)s->fmt.frame_stride;
    s->head = s->res_off + s->slot;          // frame slot 0 follows the halo slot
    s->have_fmt = true;
  }
  const int f = s->sent;
  ScanCombBatch* b = s->batch_of(f);
  if (!b) return s->fail();
  const uint8_t* src = reinterpret_cast<const uint8_t*>(frame->base);
  if (!copy_frame_planes((frame->on_device ? b->d.get() : b->h.get()) + s->slot_at(f % s->B), s->fmt, src, *frame,
                         frame->on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToHost, s->ctx->stream))
    return s->fail();
  b->host[(size_t)(f % s->B)] = frame->on_device ? 0 : 1;
  s->sent += 1;
  if (s->sent % s->B == 0 && !scan_comb_launch(s, s->launched)) return s->fail();
  return 1;
}

int amtk_scan_comb_stream_finish(amtk_scan_comb_stream* s) {
  if (!s) AMTK_FAIL("amtk_scan_comb_stream_finish: null stream");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  if (!s->open(true)) return 0;
  if (s->sent > s->launched * s->B && !scan_comb_launch(s, s->launched)) return s->fail();
  s->finished = true;
  return 1;
}

int amtk_scan_comb_stream_recv(amtk_scan_comb_stream* s, float* scores, int32_t* counts, int max_frames, int* got) {
  if (!s || !scores || !counts || !got || max_frames < 0) AMTK_FAIL("amtk_scan_comb_stream_recv: bad argument");
  return scan_comb_recv(s, scores, counts, max_frames, got);
}

int amtk_scan_comb_stream_counts(const amtk_scan_comb_stream* s, int* sent, int* received, int64_t* h2d_bytes, int64_t* d2h_bytes) {
  if (!s) AMTK_FAIL("amtk_scan_comb_stream_counts: null stream");
  s->counts(sent, received, h2d_bytes, d2h_bytes);
  return 1;
}

int amtk_comb_stream_create(amtk_ctx* ctx, const amtk_comb_params* params, int batch_size, amtk_comb_stream** out) {
  if (!ctx || !params || !out) AMTK_FAIL("amtk_comb_stream_create: bad argument");
  amtk_comb_stream* s = new amtk_comb_stream();
  if (!scan_comb_stream_make(s, ctx, nullptr, 0, params, batch_size, false)) return 0;
  *out = s;
  return 1;
}

void amtk_comb_stream_destroy(amtk_comb_stream* s) { amtk_scan_comb_stream_destroy(s); }

int amtk_comb_stream_send(amtk_comb_stream* s, const amtk_clip* frame) {
  if (!s || !frame) AMTK_FAIL("amtk_comb_stream_send: null argument");
  return amtk_scan_comb_stream_send(s, frame);
}

int amtk_comb_stream_finish(amtk_comb_stream* s) {
  if (!s) AMTK_FAIL("amtk_comb_stream_finish: null stream");
  return amtk_scan_comb_stream_finish(s);
}

int amtk_comb_stream_recv(amtk_comb_stream* s, int32_t* counts, int max_frames, int* got) {
  if (!s || !counts || !got || max_frames < 0) AMTK_FAIL("amtk_comb_stream_recv: bad argument");
  return scan_comb_recv(s, nullptr, counts, max_frames, got);
}

int amtk_comb_stream_counts(const amtk_comb_stream* s, int* sent, int* received, int64_t* h2d_bytes, int64_t* d2h_bytes) {
  if (!s) AMTK_FAIL("amtk_comb_stream_counts: null stream");
  return amtk_scan_comb_stream_counts(s, sent, received, h2d_bytes, d2h_bytes);
}

int amtk_weave_frames(amtk_ctx* ctx, const amtk_clip* src, const amtk_clip* dst, int dst_frame0,
                      const int32_t* top_idx, const int32_t* bottom_idx, int n, int src_is_nv12) {
  if (!ctx || !top_idx || !bottom_idx) AMTK_FAIL("amtk_weave_frames: null argument");
  if (!validate_clip(src, true) || !validate_clip(dst, true)) return 0;
  if (!src->on_device || !dst->on_device) AMTK_FAIL("amtk_weave_frames: clips must be device resident");
  if (src->width != dst->width || src->height != dst->height || src->bytes_per_sample != dst->bytes_per_sample ||
      src->log_uvx != dst->log_uvx || src->log_uvy != dst->log_uvy)
    AMTK_FAIL("amtk_weave_frames: source and destination formats differ");
  if (n < 0 || dst_frame0 < 0 || dst_frame0 + n > dst->num_frames) AMTK_FAIL("frame range outside the clip");
  for (int k = 0; k < n; ++k)
    if (top_idx[k] < 0 || top_idx[k] >= src->num_frames || bottom_idx[k] < 0 || bottom_idx[k] >= src->num_frames)
      AMTK_FAIL("amtk_weave_frames: source frame index outside the clip");
  if (n == 0) return 1;
  DevSelect ds(ctx); if (!ds.ok) return 0;
  if (!ctx->dout.ensure((size_t)n * 2 * sizeof(int))) return 0;
  int* didx = ctx->dout.at<int>();
  AMTK_CUDA(cudaMemcpyAsync(didx, top_idx, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  AMTK_CUDA(cudaMemcpyAsync(didx + n, bottom_idx, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  WeaveJob j;
  j.src = reinterpret_cast<const uint8_t*>(src->base); j.dst = const_cast<uint8_t*>(reinterpret_cast<const uint8_t*>(dst->base));
  j.sstride = src->frame_stride; j.dstride = dst->frame_stride;
  j.s_offu = src->off_u; j.s_offv = src->off_v; j.d_offu = dst->off_u; j.d_offv = dst->off_v;
  j.s_pitchY = src->pitch_y; j.s_pitchUV = src->pitch_uv; j.d_pitchY = dst->pitch_y; j.d_pitchUV = dst->pitch_uv;
  j.bps = src->bytes_per_sample; j.nv12 = src_is_nv12 ? 1 : 0;
  j.H = src->height; j.HC = src->height >> src->log_uvy;
  j.row_bytes_y = src->width * j.bps; j.row_bytes_c = (src->width >> src->log_uvx) * j.bps;
  j.top_idx = didx; j.bot_idx = didx + n; j.dst_frame0 = dst_frame0;
  for (int k0 = 0; k0 < n; k0 += 32768) {
    WeaveJob jj = j; jj.top_idx += k0; jj.bot_idx += k0; jj.dst_frame0 += k0;
    const int nn = std::min(32768, n - k0);
    const long long work = (long long)j.H * ((j.row_bytes_y + 15) / 16);
    dim3 grid((unsigned)std::min<long long>((work + 255) / 256, 4096), 3, nn);
    weave_kernel<<<grid, 256, 0, ctx->stream>>>(jj);
    AMTK_CUDA(cudaGetLastError());
    ctx->launches += 1;
  }
  AMTK_CUDA(cudaStreamSynchronize(ctx->stream));      // index staging buffer is reused by later calls
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// temporal noise reduction
// ---------------------------------------------------------------------------------------------------------
void amtk_tnr_default_params(amtk_tnr_params* p) {
  if (!p) return;
  p->temporal_distance = 3; p->threshold = 1; p->interlaced = 0;
}

int amtk_tnr_frames(amtk_ctx* ctx, const amtk_clip* src, const amtk_clip* dst, int dst_frame0,
                    const amtk_tnr_params* p, int frame0, int nframes) {
  if (!ctx || !src || !dst || !p) AMTK_FAIL("amtk_tnr_frames: null argument");
  if (!tnr_params_ok(p)) return 0;
  if (!validate_clip(src, true) || !validate_clip(dst, true) || !tnr_format_ok(src, p->interlaced)) return 0;
  const int bits = src->bits_per_sample;
  if (dst->width != src->width || dst->height != src->height || dst->log_uvx != 1 || dst->log_uvy != 1)
    AMTK_FAIL("tnr: source and destination formats differ");
  if (dst->bytes_per_sample != src->bytes_per_sample || dst->bits_per_sample != bits) {     // widening (ConvertBits fused)
    if (dst->bytes_per_sample == 1 && src->bytes_per_sample == 2)
      AMTK_FAIL("tnr: a 1-byte destination cannot hold a 2-byte source");
    if (dst->bytes_per_sample != 2 || dst->bits_per_sample == 8)
      AMTK_FAIL("tnr: source and destination formats differ (a 2-byte destination must be at 10, 12, 14 or 16 bits)");
    if (dst->bits_per_sample < bits)
      AMTK_FAIL("tnr: the destination has fewer bits than the source; only widening is provided (narrowing is dither arithmetic)");
    if (!(dst->bits_per_sample == 10 || dst->bits_per_sample == 12 || dst->bits_per_sample == 14 || dst->bits_per_sample == 16))
      AMTK_FAIL("tnr: bits_per_sample must be 8 (1-byte samples) or 10, 12, 14, 16 (2-byte samples)");
  }
  if (frame0 < 0 || nframes < 0 || frame0 + nframes > src->num_frames) AMTK_FAIL("frame range outside the clip");
  if (dst_frame0 < 0 || dst_frame0 + nframes > dst->num_frames) AMTK_FAIL("tnr: destination frame range outside the clip");
  if (src->on_device == dst->on_device) {
    uintptr_t s0, s1, d0, d1;
    clip_span(src, &s0, &s1); clip_span(dst, &d0, &d1);
    if (s0 < d1 && d0 < s1) AMTK_FAIL("tnr: source and destination overlap");
  }
  if (nframes == 0) return 1;
  DevSelect ds(ctx); if (!ds.ok) return 0;
  const int d = p->temporal_distance, N = src->num_frames;
  const size_t sfs = (size_t)src->frame_stride, dfs = (size_t)dst->frame_stride;
  const size_t budget = stage_budget();
  int per = nframes;
  if (!src->on_device) per = (int)std::max<long long>(1, std::min<long long>(per, (long long)(budget / sfs) - 2LL * d));
  if (!dst->on_device) per = (int)std::max<size_t>(1, std::min<size_t>((size_t)per, budget / dfs));
  // host destinations: the kernel writes a chunk into ctx->dout laid out like dst (shifted so that a plane placed before
  // the Y plane stays inside the buffer), then the rows are copied out
  size_t dshift = 0;
  if (!dst->on_device) {
    amtk_clip one = *dst; one.num_frames = 1; one.base = nullptr;
    uintptr_t f0, f1; clip_span(&one, &f0, &f1);
    dshift = (size_t)(0 - f0);
    if (!ctx->dout.ensure((size_t)(per - 1) * dfs + (size_t)(f1 - f0))) return 0;
  }
  auto run = [&](const Window& w, int lo, int hi) -> int {
    uint8_t* hdst = const_cast<uint8_t*>(reinterpret_cast<const uint8_t*>(dst->base)) + (size_t)(dst_frame0 + lo - frame0) * dfs;
    uint8_t* dbase = dst->on_device ? hdst : ctx->dout.at(dshift);
    if (!launch_tnr(ctx, src, w, dst, dbase, lo, hi, p)) return 0;
    if (!dst->on_device)         // the sample bytes of every row, nothing of the row padding
      for (int k = 0; k < hi - lo; ++k)
        if (!copy_frame_planes(hdst + (size_t)k * dfs, *dst, dbase + (size_t)k * dfs, *dst, cudaMemcpyDeviceToHost, ctx->stream)) return 0;
    return 1;
  };
  if (src->on_device) {          // chunks of the host destination's budget, or the whole range at once
    const Window w{ reinterpret_cast<const uint8_t*>(src->base), 0, N };
    for (int lo = frame0; lo < frame0 + nframes; lo += per)
      if (!run(w, lo, std::min(frame0 + nframes, lo + per))) return 0;
  } else if (!stage_chunks(ctx, frame0, nframes, per, (size_t)(per + 2 * d) * sfs,     // frames [lo-d, hi+d) clamped to the clip:
                           [&](Window& w, int lo, int hi) {                           // every window frame of outputs [lo, hi)
                             return stage_frames(ctx, src, w, std::max(0, lo - d), std::min(N, hi + d)); }, run))
    return 0;
  AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// temporal noise reduction, one frame at a time (cudaTNRCreate / SendFrame / RecvFrame / Finish)
// ---------------------------------------------------------------------------------------------------------
// Frames go into a ring of R = 2d + 2B slots in HBM (frame f in slot f mod R): the 2d + B window of the batch in flight
// plus the B frames sent for the next one.  Batch k (outputs [kB, (k+1)B)) is launched by the send that makes
// S >= (k+1)B + d, when its whole window has arrived; finish() launches the rest over windows clamped at the last frame.
// Each batch writes into its own output buffer of B frames, which goes back to a free list once every output in it has
// been received.  Host memory moves on the context's copy stream, so uploads and downloads overlap the kernel in flight;
// device memory is copied on the context's stream, in order with the caller's own work there.
// out_bits > 0 widens (ConvertBits fused, DESIGN.md section 3.4): the ring keeps the frames as sent and the outputs are
// 2-byte samples at out_bits, filtered by the ring + widening kernels.
struct amtk_tnr_stream {
  amtk_ctx* ctx = nullptr;
  amtk_tnr_params p{};
  int B = 1, R = 0;
  int out_bits = 0;                         // 0: outputs in the source's format
  bool ref_emission = false, finished = false;
  bool have_fmt = false;
  amtk_clip fmt{};                          // format of the first frame, in the ring's own layout (base unset)
  amtk_clip ofmt{};                         // format of the outputs, in the output buffers' layout (fmt unless widening)
  DevBuf<uint8_t> ring;
  std::vector<cudaEvent_t> slot_reader;     // per slot: completion event of the last batch that read it (nullptr: none)
  std::vector<int32_t> tags;                // tag of every frame sent
  int sent = 0, launched = 0, delivered = 0;   // frames sent (S), batches launched, outputs received or dropped
  struct Batch : StreamBatch { int lo = 0, hi = 0; };     // d: outputs [lo, hi)
  std::deque<Batch> batches;                // launched and not yet fully received, oldest first
  BatchPool pool;
};

namespace {

// Launches output frames [lo, hi) as one batch.
int tnr_stream_launch(amtk_tnr_stream* s, int lo, int hi) {
  amtk_ctx* ctx = s->ctx;
  amtk_tnr_stream::Batch b;
  if (!s->pool.take(&b, (size_t)s->B * (size_t)s->ofmt.frame_stride, "cudaMalloc(tnr batch)", nullptr)) return 0;
  amtk_clip rc = s->fmt;
  rc.base = s->ring; rc.num_frames = s->sent; rc.on_device = 1;      // the window clamps at the last frame sent
  const Window w{ s->ring, 0, s->R };
  const bool ok = launch_tnr(ctx, &rc, w, &s->ofmt, b.d, lo, hi, &s->p, true) &&
                  cuda_ok(cudaEventRecord(b.done, ctx->stream), "cudaEventRecord");
  if (!ok) { s->pool.give(std::move(b)); return 0; }
  const int d = s->p.temporal_distance;
  for (int f = std::max(0, lo - d); f < std::min(s->sent, hi + d); ++f) s->slot_reader[f % s->R] = b.done;
  b.lo = lo; b.hi = hi;
  s->batches.push_back(std::move(b));
  s->launched += 1;
  return 1;
}

// The reference's CPU queue (VideoFilter.hpp:45-89) drops frames N-d .. d-1 of a clip of N < 2d frames.
bool tnr_stream_dropped(const amtk_tnr_stream* s, int n) {
  const int d = s->p.temporal_distance, N = s->sent;
  return s->ref_emission && s->finished && N < 2 * d && n >= N - d && n <= d - 1;
}

// Skips dropped outputs and releases the batches whose outputs have all been received.
void tnr_stream_retire(amtk_tnr_stream* s) {
  while (s->delivered < s->sent && tnr_stream_dropped(s, s->delivered)) s->delivered += 1;
  while (!s->batches.empty() && s->batches.front().hi <= s->delivered) {
    s->pool.give(std::move(s->batches.front()));
    s->batches.pop_front();
  }
}

}  // namespace

int amtk_tnr_stream_create(amtk_ctx* ctx, const amtk_tnr_params* p, int batch_size, int reference_emission,
                           amtk_tnr_stream** out) {
  return amtk_tnr_stream_create_widening(ctx, p, 0, batch_size, reference_emission, out);
}

int amtk_tnr_stream_create_widening(amtk_ctx* ctx, const amtk_tnr_params* p, int out_bits, int batch_size,
                                    int reference_emission, amtk_tnr_stream** out) {
  if (!ctx || !p || !out) AMTK_FAIL("amtk_tnr_stream_create: null argument");
  if (out_bits != 0 && out_bits != 10 && out_bits != 12 && out_bits != 14 && out_bits != 16)
    AMTK_FAIL("tnr stream: out_bits must be 0 (the source's format) or 10, 12, 14, 16 (2-byte samples)");
  if (!tnr_params_ok(p)) return 0;
  if (batch_size < 1 || batch_size > 256) AMTK_FAIL("tnr stream: batch_size must be in [1,256]");
  if (reference_emission != 0 && reference_emission != 1) AMTK_FAIL("tnr stream: reference_emission must be 0 or 1");
  amtk_tnr_stream* s = new amtk_tnr_stream();
  s->ctx = ctx; s->p = *p; s->B = batch_size; s->ref_emission = reference_emission != 0; s->out_bits = out_bits;
  s->R = 2 * p->temporal_distance + 2 * batch_size;
  *out = s;
  return 1;
}

void amtk_tnr_stream_destroy(amtk_tnr_stream* s) {
  if (s) stream_destroy(s, s->ctx->copy_stream);     // host frames move on the copy stream
}

int amtk_tnr_stream_send(amtk_tnr_stream* s, const amtk_clip* frame, int32_t frame_index) {
  if (!s || !frame) AMTK_FAIL("amtk_tnr_stream_send: null argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  amtk_ctx* ctx = s->ctx;
  if (s->finished) AMTK_FAIL("tnr stream: send after finish");
  if (!one_frame(frame, "tnr stream", "frame") || !tnr_format_ok(frame, s->p.interlaced)) return 0;
  if (s->have_fmt && !same_format(s->fmt, frame))
    AMTK_FAIL("tnr stream: the frame's size or sample format differs from the first frame's");
  if (s->sent == INT32_MAX) AMTK_FAIL("tnr stream: too many frames");
  if (!s->have_fmt) {    // the first frame fixes the ring's format and the outputs'
    if (s->out_bits && s->out_bits < frame->bits_per_sample)
      AMTK_FAIL("tnr: the destination has fewer bits than the source; only widening is provided (narrowing is dither arithmetic)");
    const amtk_clip f = stream_frame_layout(*frame, frame->bytes_per_sample, frame->bits_per_sample);
    const amtk_clip o = s->out_bits && s->out_bits != frame->bits_per_sample ? stream_frame_layout(*frame, 2, s->out_bits) : f;
    uint8_t* ring = nullptr;
    AMTK_CUDA(cudaMalloc(reinterpret_cast<void**>(&ring), (size_t)s->R * (size_t)f.frame_stride));
    s->ring.reset(ring); s->fmt = f; s->ofmt = o; s->have_fmt = true;
    s->slot_reader.assign((size_t)s->R, nullptr);
  }
  const int slot = s->sent % s->R;
  uint8_t* dst = s->ring + (size_t)slot * (size_t)s->fmt.frame_stride;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(frame->base);
  if (frame->on_device) {
    if (!copy_frame_planes(dst, s->fmt, src, *frame, cudaMemcpyDeviceToDevice, ctx->stream)) return 0;
    AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->h2d_bytes_last = 0;
  } else {
    if (s->slot_reader[slot]) AMTK_CUDA(cudaStreamWaitEvent(ctx->copy_stream, s->slot_reader[slot], 0));
    if (!copy_frame_planes(dst, s->fmt, src, *frame, cudaMemcpyHostToDevice, ctx->copy_stream)) return 0;
    AMTK_CUDA(cudaStreamSynchronize(ctx->copy_stream));
    ctx->h2d_bytes_last = (long long)frame->width * frame->height * frame->bytes_per_sample * 3 / 2;
  }
  s->tags.push_back(frame_index);
  s->sent += 1;
  const int d = s->p.temporal_distance;
  while ((long long)(s->launched + 1) * s->B + d <= s->sent)
    if (!tnr_stream_launch(s, s->launched * s->B, (s->launched + 1) * s->B)) return 0;
  return 1;
}

int amtk_tnr_stream_finish(amtk_tnr_stream* s) {
  if (!s) AMTK_FAIL("amtk_tnr_stream_finish: null argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  if (s->finished) AMTK_FAIL("tnr stream: finish called twice");
  s->finished = true;
  while ((long long)s->launched * s->B < s->sent)
    if (!tnr_stream_launch(s, s->launched * s->B, (int)std::min<long long>((long long)(s->launched + 1) * s->B, s->sent))) return 0;
  tnr_stream_retire(s);
  return 1;
}

int amtk_tnr_stream_recv(amtk_tnr_stream* s, const amtk_clip* dst, int32_t* frame_index, int* got) {
  if (!s || !dst) AMTK_FAIL("amtk_tnr_stream_recv: null argument");
  DevSelect ds(s->ctx); if (!ds.ok) return 0;
  amtk_ctx* ctx = s->ctx;
  if (!one_frame(dst, "tnr stream", "dst") || !tnr_format_ok(dst, s->p.interlaced)) return 0;
  if (s->have_fmt && !same_format(s->ofmt, dst))
    AMTK_FAIL(s->ofmt.bits_per_sample == s->fmt.bits_per_sample
                  ? "tnr stream: dst's size or sample format differs from the frames sent"
                  : "tnr stream: dst's size or sample format differs from the stream's output format (2-byte samples at out_bits)");
  if (got) *got = 0;
  tnr_stream_retire(s);
  // before finish the newest launched batch is held back, so that its kernel runs while the one before it is received
  const long long ready = s->finished ? s->sent : (long long)std::max(0, s->launched - 1) * s->B;
  if (s->delivered >= ready) return 1;
  const amtk_tnr_stream::Batch& b = s->batches.front();
  const uint8_t* src = b.d + (size_t)(s->delivered - b.lo) * (size_t)s->ofmt.frame_stride;
  uint8_t* d = const_cast<uint8_t*>(reinterpret_cast<const uint8_t*>(dst->base));
  if (dst->on_device) {
    if (!copy_frame_planes(d, *dst, src, s->ofmt, cudaMemcpyDeviceToDevice, ctx->stream)) return 0;
    AMTK_CUDA(cudaStreamSynchronize(ctx->stream));
  } else {
    AMTK_CUDA(cudaStreamWaitEvent(ctx->copy_stream, b.done, 0));
    if (!copy_frame_planes(d, *dst, src, s->ofmt, cudaMemcpyDeviceToHost, ctx->copy_stream)) return 0;
    AMTK_CUDA(cudaStreamSynchronize(ctx->copy_stream));
  }
  if (frame_index) *frame_index = s->tags[(size_t)s->delivered];
  if (got) *got = 1;
  s->delivered += 1;
  tnr_stream_retire(s);
  return 1;
}

// ---------------------------------------------------------------------------------------------------------
// Logo finder: per-pixel temporal luma sums (DESIGN.md section 3.5)
// ---------------------------------------------------------------------------------------------------------
struct amtk_logo_find {
  amtk_ctx* ctx = nullptr;
  int device = 0;
  int width = 0, height = 0, bytes_per_sample = 0, bits = 0;     // fixed by the first clip (0: none yet)
  int64_t nframes = 0;
  DevBuf<unsigned long long> dSums;                                // s1 [height][width], then s2 [height][width]
};

int amtk_logo_find_create(amtk_ctx* ctx, amtk_logo_find** out) {
  if (!ctx || !out) AMTK_FAIL("amtk_logo_find_create: null argument");
  amtk_logo_find* f = new amtk_logo_find();
  f->ctx = ctx; f->device = ctx->device;
  *out = f;
  return 1;
}

void amtk_logo_find_destroy(amtk_logo_find* f) {
  if (!f) return;
  DevSelect ds(f->device);
  delete f;
}

int amtk_logo_find_add_frames(amtk_logo_find* f, const amtk_clip* clip, int frame0, int nframes) {
  if (!f) AMTK_FAIL("amtk_logo_find_add_frames: null finder");
  if (!validate_clip(clip, false)) return 0;
  const int bits = scan_sample_bits(clip);
  if (!bits) return 0;
  if (clip->width < 16 || clip->height < 16 || clip->width > 8192 || clip->height > 8192)
    AMTK_FAIL("amtk_logo_find_add_frames: width and height must be in [16, 8192]");
  if (f->bytes_per_sample && (clip->width != f->width || clip->height != f->height ||
                              clip->bytes_per_sample != f->bytes_per_sample || bits != f->bits))
    AMTK_FAIL("amtk_logo_find_add_frames: the clip's size or sample format differs from the first clip's");
  if (frame0 < 0 || nframes < 0 || frame0 + nframes > clip->num_frames) AMTK_FAIL("frame range outside the clip");
  amtk_ctx* ctx = f->ctx;
  DevSelect ds(ctx); if (!ds.ok) return 0;
  const size_t npix = (size_t)clip->width * clip->height;
  if (!f->dSums) {
    AMTK_CUDA(cudaMalloc(f->dSums.put(), 2 * npix * sizeof(unsigned long long)));
    AMTK_CUDA(cudaMemsetAsync(f->dSums, 0, 2 * npix * sizeof(unsigned long long), ctx->stream));
    f->width = clip->width; f->height = clip->height; f->bytes_per_sample = clip->bytes_per_sample; f->bits = bits;
  }
  ctx->h2d_bytes_last = 0;
  if (nframes == 0) return 1;
  const int bps = clip->bytes_per_sample, row_bytes = clip->width * bps;
  FindArgs a;
  a.width = clip->width; a.height = clip->height; a.row_bytes = row_bytes;
  a.tiles_x = (row_bytes + kFindTileBytes - 1) / kFindTileBytes;
  a.ntiles = a.tiles_x * ((clip->height + kFindTileRows - 1) / kFindTileRows);
  a.s1 = f->dSums; a.s2 = f->dSums + npix;
  // one launch over the window's frames [lo, hi): TMA when the resident layout allows it, else plain loads
  auto launch = [&](const uint8_t* base, long long stride, int pitch, int lo, int hi) -> int {
    a.base = base; a.frame_stride = stride; a.pitch = pitch; a.frame0 = lo; a.nframes = hi - lo;
    const bool tma = ctx->encode_tiled && ((reinterpret_cast<uintptr_t>(base) | (uintptr_t)stride | (uintptr_t)pitch) & 15) == 0;
    const void* kern = tma ? (bps == 1 ? (const void*)find_sums_tma_kernel<1> : (const void*)find_sums_tma_kernel<2>)
                           : (bps == 1 ? (const void*)find_sums_plain_kernel<1> : (const void*)find_sums_plain_kernel<2>);
    const int smem = tma ? kFindSmemBytes : 0;
    if (tma && !want_smem(ctx, kern, smem)) return 0;
    int occ = 0;
    AMTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kFindThreads, smem));
    const long long work = (long long)a.ntiles * a.nframes;
    const int grid = (int)std::max<long long>(1, std::min<long long>(work, (long long)std::max(occ, 1) * ctx->sm_count));
    if (tma) {
      CUtensorMap map;
      const cuuint64_t gdim[3] = { (cuuint64_t)row_bytes, (cuuint64_t)clip->height, (cuuint64_t)hi };
      const cuuint64_t gstr[2] = { (cuuint64_t)pitch, (cuuint64_t)stride };
      const cuuint32_t box[3] = { (cuuint32_t)kFindTileBytes, (cuuint32_t)kFindTileRows, 1u };
      if (encode_map(ctx, &map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, base, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_NONE,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B) != CUDA_SUCCESS)
        AMTK_FAIL("amtk_logo_find_add_frames: cuTensorMapEncodeTiled failed");
      if (bps == 1) find_sums_tma_kernel<1><<<grid, kFindThreads, smem, ctx->stream>>>(map, a);
      else find_sums_tma_kernel<2><<<grid, kFindThreads, smem, ctx->stream>>>(map, a);
    } else {
      if (bps == 1) find_sums_plain_kernel<1><<<grid, kFindThreads, 0, ctx->stream>>>(a);
      else find_sums_plain_kernel<2><<<grid, kFindThreads, 0, ctx->stream>>>(a);
    }
    AMTK_CUDA(cudaGetLastError());
    ctx->launches += 1;
    return 1;
  };
  int ok;
  if (clip->on_device) {
    ok = launch(reinterpret_cast<const uint8_t*>(clip->base), clip->frame_stride, clip->pitch_y, frame0, frame0 + nframes);
  } else {
    // host clips: only the Y rows cross PCIe, into a compact layout whose pitch and frame stride are multiples of 16
    const int cp = (row_bytes + 15) & ~15;
    const size_t fs = (size_t)cp * clip->height;
    const int per = (int)std::max<size_t>(1, std::min<size_t>((size_t)nframes, stage_budget() / fs));
    const uint8_t* hbase = reinterpret_cast<const uint8_t*>(clip->base);
    ok = stage_chunks(ctx, frame0, nframes, per, (size_t)per * fs,
                      [&](Window& w, int lo, int hi) -> long long {
                        uint8_t* d = const_cast<uint8_t*>(w.dev_base);
                        const uint8_t* h = hbase + (long long)lo * clip->frame_stride;
                        if (clip->frame_stride % clip->pitch_y == 0) {
                          cudaMemcpy3DParms p3; memset(&p3, 0, sizeof(p3));
                          p3.srcPtr = make_cudaPitchedPtr(const_cast<uint8_t*>(h), (size_t)clip->pitch_y, (size_t)clip->pitch_y,
                                                          (size_t)(clip->frame_stride / clip->pitch_y));
                          p3.dstPtr = make_cudaPitchedPtr(d, (size_t)cp, (size_t)cp, (size_t)clip->height);
                          p3.extent = make_cudaExtent((size_t)row_bytes, (size_t)clip->height, (size_t)(hi - lo));
                          p3.kind = cudaMemcpyHostToDevice;
                          if (!cuda_ok(cudaMemcpy3DAsync(&p3, ctx->copy_stream), "cudaMemcpy3DAsync(find)")) return -1;
                        } else {
                          for (int i = 0; i < hi - lo; ++i)
                            if (!cuda_ok(cudaMemcpy2DAsync(d + (size_t)i * fs, cp, h + (long long)i * clip->frame_stride, clip->pitch_y,
                                                           row_bytes, clip->height, cudaMemcpyHostToDevice, ctx->copy_stream),
                                         "cudaMemcpy2DAsync(find)"))
                              return -1;
                        }
                        w.first = lo; w.count = hi - lo;
                        return (long long)(hi - lo) * row_bytes * clip->height;
                      },
                      [&](const Window& w, int lo, int hi) -> int { return launch(w.dev_base, (long long)fs, cp, lo - w.first, hi - w.first); });
  }
  if (!ok) return 0;
  f->nframes += nframes;
  return 1;
}

int amtk_logo_find_get_sums(amtk_logo_find* f, uint64_t* s1, uint64_t* s2, int64_t* nframes) {
  if (!f) AMTK_FAIL("amtk_logo_find_get_sums: null finder");
  if (nframes) *nframes = f->nframes;
  if (!f->dSums || (!s1 && !s2)) return 1;
  DevSelect ds(f->ctx); if (!ds.ok) return 0;
  const size_t npix = (size_t)f->width * f->height;
  if (s1) AMTK_CUDA(cudaMemcpyAsync(s1, f->dSums, npix * sizeof(uint64_t), cudaMemcpyDeviceToHost, f->ctx->stream));
  if (s2) AMTK_CUDA(cudaMemcpyAsync(s2, f->dSums + npix, npix * sizeof(uint64_t), cudaMemcpyDeviceToHost, f->ctx->stream));
  AMTK_CUDA(cudaStreamSynchronize(f->ctx->stream));
  return 1;
}

void amtk_logo_find_default_params(amtk_logo_find_params* p) {
  if (!p) return;
  p->block = 8; p->var_ratio = 0.5f; p->mean_delta = 6.0f; p->margin = 8; p->min_blocks = 4;
}

int amtk_logo_find_rects(const uint64_t* s1, const uint64_t* s2, int64_t nframes, int width, int height, int bits,
                         const amtk_logo_find_params* p, int max_rects, int32_t* rects, float* scores, int* n) {
  if (!s1 || !s2 || !p || !n || (!rects && max_rects > 0)) AMTK_FAIL("amtk_logo_find_rects: null argument");
  *n = 0;
  if (p->block < 2) AMTK_FAIL("amtk_logo_find_rects: block must be at least 2");
  if (width < 16 || height < 16 || width > 8192 || height > 8192) AMTK_FAIL("amtk_logo_find_rects: width and height must be in [16, 8192]");
  if (bits < 8 || bits > 16) AMTK_FAIL("amtk_logo_find_rects: bits must be in 8..16");
  if (max_rects < 0) AMTK_FAIL("amtk_logo_find_rects: max_rects < 0");
  std::vector<amtk::FoundRect> found;
  amtk::find_logo_rects(s1, s2, nframes, width, height, bits, p->block, p->var_ratio, p->mean_delta, p->margin, p->min_blocks, &found);
  const int cnt = std::min<int>(max_rects, (int)found.size());
  for (int i = 0; i < cnt; ++i) {
    rects[4 * i + 0] = found[i].x; rects[4 * i + 1] = found[i].y; rects[4 * i + 2] = found[i].w; rects[4 * i + 3] = found[i].h;
    if (scores) scores[i] = found[i].score;
  }
  *n = cnt;
  return 1;
}

void amtk_calc_fade2(const float* records, int num_records, int num_frames, int n, float* ft, float* fb) {
  amtk::calc_fade2(records, num_records, num_frames, n, ft, fb);
}
int amtk_calc_fade2_index(int num_records, int num_frames, int n, int i) { return amtk::calc_fade2_index(num_records, num_frames, n, i); }
void amtk_calc_fade2_records(const float* rec9, float* ft, float* fb) { amtk::calc_fade2_records(rec9, ft, fb); }

}  // extern "C"

#include "group.cuh"
