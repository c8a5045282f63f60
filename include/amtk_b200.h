/* include/amtk_b200.h -- C ABI of libamtk_b200.so: the H100-native (sm_90a) implementation of Amatsukaze's
 * per-frame pixel-analysis hot path (logo-template correlation, LogoScan accumulation, logo erase, and the
 * field-difference / combing metric).
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch types.  Every entry point names the
 * reference interface it replaces (paths relative to the reference's Amatsukaze/ directory).  A reference-side
 * binding (what a maintainer would add to LogoScan.hpp / FilteredSource.hpp) is shown in INTEGRATION.md.
 *
 * Conventions (mirroring the reference's C exports, StreamUtils.hpp:1037-1039 + LogoScan.hpp:1083-1098):
 *   - every function returns 1 on success, 0 on failure; after a failure amtk_last_error() returns the
 *     message for the calling thread (the reference: `return false` after ctx->setError(); text fetched with
 *     AMTContext_GetError()).
 *   - handles are opaque, owned by the caller, released with the matching *_destroy().
 *   - a context is bound to ONE CUDA device and ONE stream; calls on distinct contexts run concurrently, calls on the
 *     SAME context from several host threads are safe and serialise on the context (the reference filters answer
 *     CACHE_GET_MTMODE with MT_NICE_FILTER, LogoScan.hpp:1220-1225,1500-1505: AviSynth may call GetFrame from several
 *     Prefetch threads at once).
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with an error.
 */
#ifndef AMTK_B200_H
#define AMTK_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define AMTK_API __attribute__((visibility("default")))

typedef struct amtk_ctx amtk_ctx;
typedef struct amtk_logo amtk_logo;
typedef struct amtk_scan amtk_scan;

/* ---------------------------------------------------------------------------------------------
 * Context / errors   (replaces AMTContext_Create / ATMContext_Delete / AMTContext_GetError,
 *                     StreamUtils.hpp:1037-1039, for this path)
 * ------------------------------------------------------------------------------------------- */
AMTK_API const char* amtk_last_error(void);
AMTK_API int amtk_version(void);
/* number of CUDA devices visible (0 when there is no driver/GPU; never fails) */
AMTK_API int amtk_device_count(void);
/* device: CUDA ordinal.  stream: the cudaStream_t every kernel of this context is launched on (e.g. torch's
 * current stream); NULL = the legacy default stream. */
AMTK_API int amtk_ctx_create(int device, void* cuda_stream, amtk_ctx** out);
AMTK_API void amtk_ctx_destroy(amtk_ctx* ctx);
AMTK_API int amtk_ctx_synchronize(amtk_ctx* ctx);
/* kernels launched by this context since creation (bench.py reports it as gpu_launches) */
AMTK_API int64_t amtk_ctx_launch_count(const amtk_ctx* ctx);
/* payload bytes the last call on a HOST clip copied host->device (whole frames for the combing pass, only the logo /
 * scan rectangle rows for the logo entry points -- what the reference reads there, LogoScan.hpp:1559-1566) */
AMTK_API int64_t amtk_ctx_last_h2d_bytes(const amtk_ctx* ctx);

/* Per-launch timing of the dominant streaming kernel (comb) with CUDA events recorded on the context's stream
 * around each launch; get() synchronizes the stream, returns the accumulated milliseconds and launch count. */
AMTK_API int amtk_ctx_set_kernel_timing(amtk_ctx* ctx, int enable);
AMTK_API int amtk_ctx_get_kernel_timing(amtk_ctx* ctx, double* ms_total, int64_t* launches, int reset);

/* Measurement helper: a trivial streaming read (uint4 loads, XOR-reduced) over [ptr, ptr+bytes) on the context's
 * stream, timed with CUDA events; returns the average milliseconds of `reps` passes after one warm-up pass.
 * bench.py reports bytes/ms as the read-only HBM ceiling next to the roofline numbers. */
AMTK_API int amtk_probe_read_ms(amtk_ctx* ctx, const void* device_ptr, size_t bytes, int reps, double* ms_out);

/* Pinned host memory for the host-buffer entry points (optional; pageable memory works, only slower). */
AMTK_API int amtk_host_alloc(size_t bytes, void** out);
AMTK_API void amtk_host_free(void* p);
/* HBM buffers for device-resident clips (what AMTSource keeps its decoded frames in, replacing the reference's CPU
 * frame cache, AMTSource.hpp:419-425) and synchronous copies on the context's stream. */
AMTK_API int amtk_device_alloc(amtk_ctx* ctx, size_t bytes, void** out);
AMTK_API void amtk_device_free(amtk_ctx* ctx, void* p);
AMTK_API int amtk_memcpy_h2d(amtk_ctx* ctx, void* dst_device, const void* src_host, size_t bytes);
AMTK_API int amtk_memcpy_d2h(amtk_ctx* ctx, void* dst_host, const void* src_device, size_t bytes);
AMTK_API int amtk_memcpy_d2d(amtk_ctx* ctx, void* dst_device, const void* src_device, size_t bytes);   /* MakeWritable of a device frame */

/* ---------------------------------------------------------------------------------------------
 * Clip descriptor: a run of planar YUV frames, either resident in HBM or in host memory.
 * Describes what the reference's filters read through PVideoFrame::GetReadPtr/GetPitch(PLANAR_Y|U|V)
 * (LogoScan.hpp:1138-1145, AMTSource.hpp:357-408).
 * ------------------------------------------------------------------------------------------- */
typedef struct amtk_clip {
  const void* base;        /* first byte of frame 0 (its Y plane)                                  */
  int64_t frame_stride;    /* bytes from one frame to the next                                     */
  int64_t off_u, off_v;    /* byte offsets of the U and V planes inside a frame                    */
  int32_t width, height;   /* luma size in pixels                                                  */
  int32_t pitch_y, pitch_uv; /* bytes per row.  When base, frame_stride, off_u/off_v and the pitches are  */
                             /* all multiples of 16 bytes the TMA streaming kernels run; any other layout */
                             /* takes slower plain-load kernels with identical results                    */
  int32_t log_uvx, log_uvy;  /* chroma subsampling shifts (1,1 for YV12 / YUV420P10)               */
  int32_t bytes_per_sample;  /* 1 (YV12) or 2 (YUV420P10/P12/P16, little endian)                   */
  int32_t bits_per_sample;   /* 8, 10, 12 or 16: maxv = (1<<bits)-1 (LogoScan.hpp:1130,1575); every sample must be
                              * <= maxv (the 10-bit combing path relies on it, as the reference's 10-bit formats do).
                              * amtk_tnr_frames also accepts 14 (the product filters after ConvertBits(14)), and a
                              * destination at more bits than its source (it widens as it filters) */
  int32_t num_frames;
  int32_t on_device;         /* 1: base is a device pointer on the context's device; 0: host pointer */
} amtk_clip;

/* Host memory and when a call returns.  A call that takes host memory (a host clip or frame, or a host array such as
 * fades, frame_result, frame_select or top_idx/bottom_idx) returns only when it no longer reads that memory: the caller
 * may overwrite or free it at once, pinned or pageable.  Host outputs (results, a host dst, host clips erased in place)
 * are complete when it returns.  A call on device clips with device outputs may return once its work is enqueued: order
 * later work on the context's stream, or call amtk_ctx_synchronize. */

/* ---------------------------------------------------------------------------------------------
 * Logos   (replaces logo::LogoData / logo::LogoDataParam, AMTLogo.hpp:49-280, LogoScan.hpp:61-334)
 * ------------------------------------------------------------------------------------------- */
typedef struct amtk_logo_info {
  int32_t w, h, log_uvx, log_uvy;
  int32_t imgw, imgh, imgx, imgy;
  int32_t maskpixels;      /* min(w*h,(int)(w*h*maskratio)), LogoScan.hpp:172; 0 before create_mask */
  int32_t count;           /* mask pixels the y,x in [2,dim-2) scan visits (= kernels/scales rows)   */
  float black_score;       /* LogoScan.hpp:227-228                                                   */
} amtk_logo_info;

/* data: aY,bY,aU,bU,aV,bV contiguous floats -- LogoData's own layout (AMTLogo.hpp:203-212).
 * Logos are host objects: ctx may be NULL; the HBM copy of a logo's tables is made by the first context that
 * evaluates it (and the logo then belongs to that device). */
AMTK_API int amtk_logo_create(amtk_ctx* ctx, const float* data, int w, int h, int log_uvx, int log_uvy,
                              int imgw, int imgh, int imgx, int imgy, amtk_logo** out);
/* LogoData::Load (AMTLogo.hpp:257-279): reads a .lgd, skipping the AviUtl base part; header540 (may be NULL)
 * receives the raw 540-byte LogoHeader (AMTLogo.hpp:19-47). */
AMTK_API int amtk_logo_load(amtk_ctx* ctx, const char* path, amtk_logo** out, void* header540);
/* LogoData::Save (AMTLogo.hpp:239-255) incl. the AviUtl-compatible base part (ToOutLGP, :96-167). */
AMTK_API int amtk_logo_save(const amtk_logo* logo, const char* path, const char* name, int service_id);
AMTK_API void amtk_logo_destroy(amtk_logo* logo);
/* DeintLogo (LogoScan.hpp:734-761): vertical [1 2 1]/4 of the Y planes, same image placement. */
AMTK_API int amtk_logo_deint(const amtk_logo* src, amtk_logo** out);
/* LogoDataParam::MakeFieldLogo (LogoScan.hpp:257-283). */
AMTK_API int amtk_logo_field(const amtk_logo* src, int bottom, amtk_logo** out);
/* LogoDataParam::CreateLogoMask (LogoScan.hpp:112-229): mask, kernels, scale tables, blackScore; uploads the
 * evaluation tables to HBM on next use.  Must be called before the logo is used by scan/analyze entry points.
 * (Setup-time host code, once per logo -- exactly where the reference runs it; the per-frame path is CUDA.) */
AMTK_API int amtk_logo_create_mask(amtk_logo* logo, float maskratio);
AMTK_API int amtk_logo_get_info(const amtk_logo* logo, amtk_logo_info* out);
/* Copies out host tables (any pointer may be NULL): data (LogoData layout), mask w*h, kernels count*25,
 * scales count*32*2 {scale,scale2}. */
AMTK_API int amtk_logo_get_tables(const amtk_logo* logo, float* data, uint8_t* mask, float* kernels, float* scales);

/* ---------------------------------------------------------------------------------------------
 * Logo evaluation
 * ------------------------------------------------------------------------------------------- */
/* LogoFrame::ScanFrame over frames [frame0, frame0+nframes) (LogoScan.hpp:1543-1589; the CMAnalyze entry,
 * CMAnalyze.hpp:291-292).  logos[i] are DEINT logos with masks.  out: float[nframes][nlogos][2] = corr0,corr1
 * (EvalResult, :1532-1535); a logo whose imgw/imgh differ from the clip yields (0,-1) (:1551-1558).
 * pitch_elems_override: 0 = use clip.pitch_y/bytes_per_sample; >0 = element pitch to use for addressing the Y
 * plane (the reference passes the BYTE pitch even for 16-bit samples, :1547,1561 -- see INTEGRATION.md).
 * out_on_device: 1 = out is a device pointer (stays in HBM), 0 = host pointer. */
AMTK_API int amtk_logo_scan_frames(amtk_ctx* ctx, const amtk_clip* clip, amtk_logo* const* logos, int nlogos,
                                   int frame0, int nframes, int pitch_elems_override, float* out, int out_on_device);
/* AMTAnalyzeLogo::GetFrameT body per SOURCE frame (LogoScan.hpp:1119-1161): out float[nframes][33] =
 * LogoAnalyzeFrame{p[11],t[11],b[11]} (:1100-1103) for source frames frame0.. (the caller groups 8 per output
 * frame and clamps, :1133). */
AMTK_API int amtk_logo_analyze_frames(amtk_ctx* ctx, const amtk_clip* clip, const amtk_logo* deint_logo,
                                      const amtk_logo* field_top, const amtk_logo* field_bottom,
                                      int frame0, int nframes, float* out, int out_on_device);
/* General form used by LogoAnalyzer::ReMakeLogo's 20-fade sweep (LogoScan.hpp:955-975): evaluates
 * EvaluateLogo(DeintY(roi), maxv, fades[i]) for every frame; out float[nframes][nfades] (signed scores). */
AMTK_API int amtk_logo_eval_fades(amtk_ctx* ctx, const amtk_clip* clip, const amtk_logo* deint_logo,
                                  const float* fades, int nfades, int frame0, int nframes, float* out, int out_on_device);

/* ---------------------------------------------------------------------------------------------
 * Field-difference / combing metric (the telecine pre-pass the reference drives through
 * AMTFilterSource::FilterPass/ReadAllFrames, FilteredSource.hpp:232-238,417-439,519-544, and computes in the
 * external KFM plugin).  Integer spec: DESIGN.md section 4; 8-bit and 16-bit (YUV420P10/12/16) samples.
 * counts int32[nframes][12] = [plane class Y,C][field top,bottom][move, shima, lshima].
 * Thresholds: 8-bit th_move in [1,128], th_shima/th_lshima in [1,2047]; 16-bit th_move in [1,32768], others >= 1.
 * ------------------------------------------------------------------------------------------- */
typedef struct amtk_comb_params {
  int32_t th_move_y, th_shima_y, th_lshima_y;   /* defaults 20, 12, 36 */
  int32_t th_move_c, th_shima_c, th_lshima_c;   /* defaults 24, 16, 48 */
} amtk_comb_params;
AMTK_API void amtk_comb_default_params(amtk_comb_params* p);
/* prev(frame0) is frame0-1 when frame0 > 0 (halo frame for range-sharded clips), else frame0 itself. */
AMTK_API int amtk_comb_frames(amtk_ctx* ctx, const amtk_clip* clip, const amtk_comb_params* params,
                              int frame0, int nframes, int32_t* counts, int out_on_device);

/* The fused hot-path step of BASELINE.json's headline metric: one pass over frames [frame0, frame0+nframes)
 * producing BOTH the ScanFrame scores (as amtk_logo_scan_frames) and the combing counters (as amtk_comb_frames). */
AMTK_API int amtk_scan_comb_frames(amtk_ctx* ctx, const amtk_clip* clip, amtk_logo* const* logos, int nlogos,
                                   const amtk_comb_params* params, int frame0, int nframes,
                                   float* scores, int32_t* counts, int out_on_device);
/* The same step with amtk_logo_scan_frames' pitch_elems_override, so that LogoFrame::ScanFrame's byte-pitch row step on
 * 2-byte samples (pitch_elems_override = clip.pitch_y) runs in the same call as the combing counters.  scores equal
 * amtk_logo_scan_frames(ctx, clip, logos, nlogos, frame0, nframes, pitch_elems_override, ...) bit for bit, with its
 * refusals and messages; counts equal amtk_comb_frames.  pitch_elems_override <= 0, or equal to
 * clip.pitch_y / bytes_per_sample, is amtk_scan_comb_frames exactly, launches included; any other value runs the comb
 * kernel, then the logo kernels with that element pitch (the launches of amtk_comb_frames plus amtk_logo_scan_frames on
 * the same clip).  Host clips are staged as amtk_scan_comb_frames stages them. */
AMTK_API int amtk_scan_comb_frames_pitch(amtk_ctx* ctx, const amtk_clip* clip, amtk_logo* const* logos, int nlogos,
                                         const amtk_comb_params* params, int pitch_elems_override,
                                         int frame0, int nframes, float* scores, int32_t* counts, int out_on_device);

/* ---------------------------------------------------------------------------------------------
 * LogoScan accumulation (replaces logo::LogoScan, LogoScan.hpp:398-660; the ScanLogo C export's inner loop,
 * :1083-1098 -> :881-914)
 * ------------------------------------------------------------------------------------------- */
AMTK_API int amtk_scan_create(amtk_ctx* ctx, int scanw, int scanh, int log_uvx, int log_uvy, int thy, amtk_scan** out);
AMTK_API void amtk_scan_destroy(amtk_scan* s);
/* LogoScan::AddFrame for every frame in [frame0, frame0+nframes) with the ROI at (scanx, scany) (:594-659);
 * valid_out (may be NULL; host pointer) receives 1/0 per frame = AddFrame's return value.
 * Samples: 1-byte at up to 8 bits (AddFrame<uint8_t>) or 2-byte at 9..16 bits (AddFrame<uint16_t>, even pitches, plane
 * offsets, frame stride and base).  The first clip added fixes the sample size and depth; a clip of another one is
 * refused.  thy is in sample units at every depth, as in the reference.  2-byte samples follow the reference's int
 * arithmetic: the border samples are shorts (:406), so at 16 bits a sample >= 32768 counts as negative in the range
 * test, the sort and the background value, and f*f (:361) wraps to 32 bits for f >= 46341.  The sums are exact 64-bit
 * integers, equal to the reference's doubles while they stay below 2^53: at 16 bits, up to 2^21 valid frames.
 * frame_select (may be NULL; host pointer, nframes bytes): only frames with a non-zero byte are offered
 * (ReMakeLogo's `minFades[i] > 8` filter, :1018-1021). */
AMTK_API int amtk_scan_add_frames(amtk_scan* s, const amtk_clip* clip, int scanx, int scany, int frame0, int nframes,
                                  const uint8_t* frame_select, uint8_t* valid_out);
AMTK_API int amtk_scan_num_valid(const amtk_scan* s);
/* raw accumulators as doubles, plane-major Y,U,V, 5 per pixel {sumF,sumB,sumF2,sumB2,sumFB} (LogoColor, :346) */
AMTK_API int amtk_scan_get_sums(amtk_scan* s, double* out);
/* LogoScan::Normalize(maxv) + GetLogo(clean) (:471-566): fills data (LogoData layout); maxv comes from the caller
 * ((1 << bits) - 1 for the scan's depth gives ScanLogo's logo); returns 0 with error
 * "Insufficient logo frames" when the reference would return nullptr (:847-849).  With clean and an odd scanw or
 * scanh (4:2:0), luma pixels of the last column or row whose chroma index falls past the chroma planes skip their
 * chroma reads and writes; the reference reaches outside its planes there, so no result is pinned at those sizes. */
AMTK_API int amtk_scan_get_logo(amtk_scan* s, int maxv, int clean, float* data);

/* The whole logo-generation pipeline of the reference's ScanLogo C export (LogoScan.hpp:1083-1098 ->
 * LogoAnalyzer::ScanLogo :1058-1079): MakeInitialLogo (:917-921, AddFrame on every frame until max_frames valid ones),
 * ReMakeLogo twice (:923-1036: deint logo, mask 0.1, 20-fade sweep per valid frame, re-accumulate frames whose best
 * fade index is > 8, GetLogo(clean)), then LogoData::Save.  The clip stands where the reference decodes `srcpath`;
 * the valid ROI frames stay in HBM instead of the UtVideo work file.  cb (may be NULL) has the reference's
 * LOGO_ANALYZE_CB signature (:792): bool(float progress, int nread, int total, int ngather); returning 0 cancels
 * ("Cancel requested", :908-910).  Samples as for amtk_scan_add_frames: at 9..16 bits the pipeline runs with
 * maxv = (1 << bits) - 1 where the reference has 255 (:845, :968, :1030; its work file is 8-bit only, :812). */
typedef int (*amtk_logo_analyze_cb)(float progress, int nread, int total, int ngather);
AMTK_API int amtk_scan_logo(amtk_ctx* ctx, const amtk_clip* clip, int service_id, const char* dstpath,
                            int imgx, int imgy, int w, int h, int thy, int max_frames, amtk_logo_analyze_cb cb);

/* The same pipeline fed one decoded frame at a time, as the reference's SimpleVideoReader::readAll drives
 * InitialLogoCreator::onFrame (LogoScan.hpp:671-727,881-914): one call per reference call.  Only the scan rectangle of
 * each valid frame is kept, in an HBM stack that grows with the frames gathered.  Spec: DESIGN.md section 3.3.1.
 *   - The first frame fixes width, height and chroma subsampling (onFirstFrame, :852-880); later frames must match them,
 *     in any layout, host or device.  It also fixes the sample format: 1-byte samples at 8 bits or 2-byte samples at
 *     9..16 bits (maxv = (1 << bits) - 1, as amtk_scan_logo); a frame of another size or depth is refused.  The rectangle
 *     must lie inside the frame.  A rejected frame leaves the stream as it was.
 *   - Frame r (1-based read count) is offered to LogoScan::AddFrame unless max_frames valid frames were gathered before
 *     it; the frame that brings the count to max_frames is the cut-off.  Frames sent after the cut-off are accepted and
 *     ignored (not copied, not counted, no callback).
 *   - Frames are resolved in batches ending at every r that is a multiple of 200 and at finish, before the send that
 *     closes the batch returns; then, if r % 200 == 0 and r <= the cut-off, cb((float)pos / (float)size * 50, r, 0,
 *     numFrames) with the pos and size sent with frame r.  *more = 0 from the send that resolves the batch holding the
 *     cut-off (max_frames = 0: from the first send).
 *   - Host frames: only the rectangle rows are copied, into a pinned batch buffer (send returns once the frame may be
 *     reused), one upload per batch.  Device frames are copied on the device, in order on the context's stream.
 *   - A cancel (cb returns 0, "Cancel requested"), a CUDA error or any finish closes the stream: afterwards only counts
 *     and destroy succeed.  destroy is valid at any point and waits for the stream's device work.  Calls serialise on
 *     the context; streams on one context are independent. */
typedef struct amtk_scan_logo_stream amtk_scan_logo_stream;
/* LogoAnalyzer(ctx, ..., imgx, imgy, w, h, thy, numMaxFrames, cb) (:1039-1056); cb may be NULL.  Refused: w or h outside
 * [4, 4096], a negative imgx, imgy or max_frames, a null ctx or out. */
AMTK_API int amtk_scan_logo_stream_create(amtk_ctx* ctx, int imgx, int imgy, int w, int h, int thy, int max_frames,
                                          amtk_logo_analyze_cb cb, amtk_scan_logo_stream** out);
AMTK_API void amtk_scan_logo_stream_destroy(amtk_scan_logo_stream* s);
/* InitialLogoCreator::onFrame (:881-914).  frame: ONE frame (host or device); pos, size: SimpleVideoReader::currentPos and
 * the source's size (size >= 1).  *more (may be NULL) = 0: stop decoding (onFrame returned false, :885) */
AMTK_API int amtk_scan_logo_stream_send(amtk_scan_logo_stream* s, const amtk_clip* frame, int64_t pos, int64_t size, int* more);
/* end of input: GetLogo(false) (:845-849), ReMakeLogo twice, the final callback, LogoData::Save (:1058-1079); the file
 * equals what amtk_scan_logo writes for a clip of the same frames.  Fails when no frame was sent (the reference would
 * dereference a null LogoScan there). */
AMTK_API int amtk_scan_logo_stream_finish(amtk_scan_logo_stream* s, int service_id, const char* dstpath);
/* frames read up to the cut-off, frames gathered (numFrames, as of the last resolved batch), payload bytes uploaded
 * host->device so far: the Y, U and V rectangles at bytes_per_sample per sample, per host frame (any pointer may be
 * NULL) */
AMTK_API int amtk_scan_logo_stream_counts(const amtk_scan_logo_stream* s, int* nread, int* ngather, int64_t* h2d_bytes);

/* ---------------------------------------------------------------------------------------------
 * Frame ingest: field weave + NV12 split on the device (replaces AMTSource::MergeField / Copy1 / Copy2,
 * AMTSource.hpp:291-355, used by MakeFrame :357-366 for half-delay (BFF / repeat-field) sources,
 * StreamReform.hpp:890-903).  dst frame k (k = 0..n-1, starting at dst_frame0) takes its EVEN rows (luma and chroma)
 * from src frame top_idx[k] and its ODD rows from src frame bottom_idx[k]; with src_is_nv12 the source chroma is one
 * interleaved UV plane at off_u (pitch_uv bytes per row) that is split into dst's U and V planes.
 * Both clips must be device resident, same size and sample format.  top_idx/bottom_idx are host pointers.
 * ------------------------------------------------------------------------------------------- */
AMTK_API int amtk_weave_frames(amtk_ctx* ctx, const amtk_clip* src, const amtk_clip* dst, int dst_frame0,
                               const int32_t* top_idx, const int32_t* bottom_idx, int n, int src_is_nv12);

/* ---------------------------------------------------------------------------------------------
 * Temporal noise reduction (the reference's TemporalNRFilter, VideoFilter.hpp:27-212, and the GPU twin it declares as
 * CudaTemporalNRFilter, :214-267, over cudaTNRCreate / cudaTNRSendFrame / cudaTNRRecvFrame / cudaTNRFinish, whose
 * CudaFilter.h is not in the reference tree).  The server's EnableTemporalNR profile option writes KTemporalNR(3, 1)
 * after ConvertBits(14) (AmatsukazeServer/Server/Misc.cs:1403-1428): the defaults below.  Bit-exact against the
 * reference's TemporalNRFilter; the arithmetic of the external KTemporalNR plugin is not in the reference tree.
 *
 * Destination frame dst_frame0+k receives source frame frame0+k filtered over the window
 * w_i = clamp(frame0+k - d + i, 0, src->num_frames - 1), i = 0..2d: the window clamps at the ends of the CLIP, never at
 * frame0.  (For clips shorter than 2d frames the reference's onFrame/finish queue, :45-89, drops frames; this entry point
 * returns every frame.)  Spec: DESIGN.md section 3.4.
 *   - 4:2:0 only (log_uvx = log_uvy = 1), 1-byte samples at 8 bits or 2-byte samples at 10, 12, 14 or 16 bits; width and
 *     height even; interlaced also needs height % 4 == 0 (the reference reads and writes one chroma row past the plane
 *     otherwise).  src and dst have the same size; their layouts (pitches, plane offsets) may differ.
 *   - dst has src's sample format, or it widens: 2-byte samples at dst bits in {10, 12, 14, 16} above src's bits,
 *     k = dst bits - src bits.  dst then receives the filter at dst's bits (threshold << (dst bits - 8)) applied to the
 *     source frames shifted left by k, bit-exact against TemporalNRFilter on those frames: ConvertBits(14) then
 *     KTemporalNR(3, 1) on a limited-range clip (AviSynth+'s widening is that shift) in one pass that reads the source
 *     at its own size.  Host sources are staged at the source's size.  Refused, each with its reason: narrowing (dst
 *     bits below src's), a 1-byte dst for a 2-byte src, a 2-byte dst at 8 bits.
 *   - src and dst may each be device resident or host memory; host sources are staged through HBM in chunks with d halo
 *     frames on each side.  Only the sample bytes of each dst row are written (row padding stays untouched).
 *   - src and dst must not overlap.  Returns when dst is complete.
 * ------------------------------------------------------------------------------------------- */
typedef struct amtk_tnr_params {
  int32_t temporal_distance;   /* d in [0, 63]: 2d+1 frames (MAX_NFRAMES = 128, VideoFilter.hpp:38-40,91)  */
  int32_t threshold;           /* in [0, 65535]; compared as threshold << (bits - 8) (:120)                */
  int32_t interlaced;          /* 0 or 1: chroma row of luma row y is ((y>>1)&~1)|(y&1) (:164)             */
} amtk_tnr_params;
AMTK_API void amtk_tnr_default_params(amtk_tnr_params* p);      /* (3, 1, 0): KTemporalNR(3, 1) */
AMTK_API int amtk_tnr_frames(amtk_ctx* ctx, const amtk_clip* src, const amtk_clip* dst, int dst_frame0,
                             const amtk_tnr_params* params, int frame0, int nframes);

/* The same filter fed one frame at a time, as a decoder produces them: the reference's cudaTNRCreate / cudaTNRSendFrame /
 * cudaTNRRecvFrame / cudaTNRFinish (driven by CudaTemporalNRFilter, VideoFilter.hpp:214-267).  Each frame is uploaded
 * once into a ring of 2d + 2*batch_size frame slots in HBM and each output is downloaded once.  Spec: DESIGN.md 3.4.
 *   - Pixels: output n equals amtk_tnr_frames' output n for the clip of all N frames sent before finish (window
 *     clamp(n - d + i, 0, N - 1)), byte for byte.
 *   - Which outputs: reference_emission = 0 returns every frame in send order (the frame count CudaTemporalNRFilter's
 *     finish checks, :243-261).  reference_emission = 1 follows the CPU TemporalNRFilter queue (:45-89): the same for
 *     N >= 2d; for N < 2d frames N-d .. d-1 are dropped (d = 3: N = 5 gives 0, 1, 3, 4; N = 4 gives 0, 3; N <= 3 none).
 *   - send takes a tag (the reference's frameIndex_); recv returns the tag of the frame it delivers.
 *   - When outputs can be received, with S the number of frames sent and batch k = outputs [kB, (k+1)B), B = batch_size:
 *     batch k is launched by the send that makes S >= (k+1)B + d, and finish launches the rest (the last batch may be
 *     short).  Before finish, recv delivers the outputs of batch k only once batch k+1 has been launched, so that the
 *     download of batch k overlaps the kernel of batch k+1; after finish every remaining output can be received.  recv
 *     waits for the device only for an output it may deliver; otherwise it returns 1 with *got = 0.  This rule does not
 *     depend on timing.
 *   - Outputs not yet received stay in HBM (one frame each, allocated in batches), so "send everything, finish, receive
 *     everything" works at that cost.
 *   - send returns once the frame's bytes have been copied (host, pinned or pageable, or device memory); recv returns once
 *     dst is written.  Only the sample bytes of each dst row are written.  frame and dst are one-frame clips; host memory
 *     is copied on the context's copy stream, device memory in order on the context's stream.
 *   - The first frame fixes the format (size, bits, sample size; the amtk_tnr_frames formats); later frames and every dst
 *     must match it, in any layout.  Rejected, leaving the stream as it was: d outside [0, 63], t outside [0, 65535],
 *     batch_size outside [1, 256], an unsupported or changed format, send after finish, a second finish.
 *   - Calls serialise on the context like every entry point; streams on one context are independent.  Destroy a stream
 *     before its context; destroy may come at any point of the clip. */
typedef struct amtk_tnr_stream amtk_tnr_stream;
AMTK_API int amtk_tnr_stream_create(amtk_ctx* ctx, const amtk_tnr_params* params, int batch_size,
                                    int reference_emission, amtk_tnr_stream** out);     /* cudaTNRCreate    */
/* The same stream, widening as it filters (ConvertBits fused, as amtk_tnr_frames does for a 2-byte dst above the source's
 * bits): out_bits = 0 is amtk_tnr_stream_create; out_bits in {10, 12, 14, 16} makes every output 2-byte samples at
 * out_bits, the filter at out_bits on the frames sent shifted left by out_bits - their bits (equal bits: no shift).
 * Frames are sent and uploaded at their own size (an 8-bit frame moves 8-bit bytes) and every dst takes the output
 * format.  Rejected: out_bits outside {0, 10, 12, 14, 16} at create; a first frame with more bits than out_bits
 * (narrowing) at its send, which fixes no format, so a valid frame may follow.  The receive rule, the tags and
 * reference_emission are those of amtk_tnr_stream_create. */
AMTK_API int amtk_tnr_stream_create_widening(amtk_ctx* ctx, const amtk_tnr_params* params, int out_bits, int batch_size,
                                             int reference_emission, amtk_tnr_stream** out);
AMTK_API void amtk_tnr_stream_destroy(amtk_tnr_stream* s);
AMTK_API int amtk_tnr_stream_send(amtk_tnr_stream* s, const amtk_clip* frame, int32_t frame_index);   /* cudaTNRSendFrame */
AMTK_API int amtk_tnr_stream_recv(amtk_tnr_stream* s, const amtk_clip* dst, int32_t* frame_index,
                                  int* got);                                            /* cudaTNRRecvFrame */
AMTK_API int amtk_tnr_stream_finish(amtk_tnr_stream* s);                                 /* cudaTNRFinish    */

/* ---------------------------------------------------------------------------------------------
 * Logo erase (replaces AMTEraseLogo::Delogo on Y,U,V, LogoScan.hpp:1248-1261,1374-1397), in place on a
 * device-resident or host clip.  fades float[nframes][2] = fadeT,fadeB per frame (host pointer).
 * ------------------------------------------------------------------------------------------- */
AMTK_API int amtk_erase_logo_frames(amtk_ctx* ctx, const amtk_clip* clip, const amtk_logo* logo,
                                    int frame0, int nframes, const float* fades);
/* AMTEraseLogo::CalcFade2 (LogoScan.hpp:1263-1315) on host records (float[num_records][33]). */
AMTK_API void amtk_calc_fade2(const float* records, int num_records, int num_frames, int n, float* fade_t, float* fade_b);
/* The same decision without materialising every record of the clip: CalcFade2 reads nine records around frame n
 * (offsets i = -4..4, with the reference's double offset, :1273-1275).  _index gives the record each offset reads,
 * _records decides from those nine (float[9][33], offset order). */
AMTK_API int amtk_calc_fade2_index(int num_records, int num_frames, int n, int i);
AMTK_API void amtk_calc_fade2_records(const float* rec9, float* fade_t, float* fade_b);

/* The eraser chain the encoder runs whenever a logo is configured, AMTEraseLogo(AMTAnalyzeLogo(src, logo), logo, logof,
 * maxfade) (FilteredSource.hpp:441-475), fed one decoded frame at a time and read back in frame order.  Each frame is sent
 * once, only its logo rectangles cross PCIe, each frame is analysed at most once, and the fade decision and Delogo run
 * batched on the device.  Spec: DESIGN.md section 3.3.2.
 *   - Pixels: with C the N frames sent, output n is source frame n with its Y, U and V logo rectangles replaced by what
 *     amtk_erase_logo_frames(ctx, C, logo, n, 1, fades_n) writes, byte for byte.  fades_n is AMTEraseLogo::CalcFade(n)
 *     (LogoScan.hpp:1317-1341): with a frame_result, the window of max_fade_length >> 1 frames on each side (clamped to
 *     [0, N-1]) decides fade 1 (all 2) or 0 (all 0 or all 1) when it is uniform; otherwise, and always without a
 *     frame_result, CalcFade2 over the amtk_logo_analyze_frames records of C, reading the records
 *     amtk_calc_fade2_index(N, N, n, i), i = -4..4.  The fades equal the host's bit for bit.  Mode 0 only (no debug label).
 *   - Lookahead: output n reads records of frames in [n-8, min(N-1, n+8)] only (the negative offsets of the (nsrc + i)
 *     quirk, :1273-1275, map into frames 4..7 of outputs 0..7).  Frame k is analysed, once, exactly when some output that
 *     takes CalcFade2 reads its record; that set follows from frame_result at create.  A uniform frame_result analyses
 *     nothing and launches no evaluation kernel.
 *   - Receive rule, with S the frames sent and batch k = outputs [kB, min(N, (k+1)B)), B = batch_size: the send that makes
 *     S >= min(N, (k+1)B + 8) launches batch k, so the N-th send launches every remaining batch (there is no finish).
 *     Batch k's outputs can be received once batch k+1 was launched, or once S = N; outputs come in frame order.  recv
 *     waits on the device only for an output it delivers; otherwise it returns 1 with *got = 0.  The rule does not depend
 *     on timing.
 *   - Format: the first frame fixes size, bits, sample size and subsampling (1-byte samples at 8 bits or 2-byte samples at
 *     9..16 bits; the logo's subsampling); later frames and every dst must match it, in any layout (host pinned or
 *     pageable, or device; any plane order or padding).  The logo rectangle must lie inside the frame.
 *   - Host frames: send copies the rectangle rows into a pinned batch buffer and returns; the slots are uploaded when a
 *     batch is launched.  Device frames are copied on the device, in order on the context's stream.  h2d_bytes grows by
 *     (w*h + 2*(w>>lx)*(h>>ly)) * bytes_per_sample per host frame, d2h_bytes by that plus 8 (its fades) per output.
 *   - Rejected, leaving the stream as it was: a frame of another format, more than N sends, a clip that is not one frame,
 *     a first frame whose sample size the evaluation plan refuses.  A CUDA error closes the stream (then only counts and
 *     destroy succeed).  destroy is valid at any point and waits for the stream's device work.  Calls serialise on the
 *     context; streams on one context are independent.
 *   - HBM: the rectangles and fades of outputs not yet received (buffers of B frames, reused), a ring of B + 16 records
 *     when some frame is analysed, and N bytes of fade codes. */
typedef struct amtk_erase_logo_stream amtk_erase_logo_stream;
/* logo: the raw logo (amtk_logo_load's); the stream keeps its own copies and builds the deint and field logos with masks at
 * maskratio as the AMTAnalyzeLogo constructor does (LogoScan.hpp:1164-1201).  num_frames: N, the clip length CalcFade and
 * CalcFade2 clamp with.  frame_result: NULL (no logoframe file) or N values in {0, 1, 2} (ReadLogoFrameFile's frameResult,
 * :1421-1461).  Refused with the reason: N < 1, max_fade_length < 0, batch_size outside [1, 256], maskratio outside
 * (0, 1], a frame_result value above 2, a logo too small for field logos, and -- when some frame is analysed -- a logo
 * the evaluation plan refuses (amtk_logo_analyze_frames' message). */
AMTK_API int amtk_erase_logo_stream_create(amtk_ctx* ctx, const amtk_logo* logo, float maskratio, int num_frames,
                                           const uint8_t* frame_result, int max_fade_length, int batch_size,
                                           amtk_erase_logo_stream** out);
AMTK_API void amtk_erase_logo_stream_destroy(amtk_erase_logo_stream* s);
/* frame: ONE frame, source frame S (0-based) */
AMTK_API int amtk_erase_logo_stream_send(amtk_erase_logo_stream* s, const amtk_clip* frame);
/* Writes the next output's three erased logo rectangles into dst and nothing else of dst: dst must hold source frame n's
 * pixels (the caller keeps its frames).  *n = the output's frame index; fades (may be NULL) = {fadeT, fadeB}. */
AMTK_API int amtk_erase_logo_stream_recv(amtk_erase_logo_stream* s, const amtk_clip* dst, int* n, int* got, float* fades);
/* frames sent, outputs received, frames analysed so far, payload bytes host->device and device->host (any may be NULL) */
AMTK_API int amtk_erase_logo_stream_counts(const amtk_erase_logo_stream* s, int* sent, int* received, int* analyzed,
                                           int64_t* h2d_bytes, int64_t* d2h_bytes);

/* The same eraser chain over a whole clip in one call, for clips already resident in HBM (or in host memory, in place).
 * Spec: DESIGN.md section 3.3.4.
 *   - Clip length: N = src->num_frames is the clip length CalcFade and CalcFade2 clamp with.
 *   - logo, maskratio, frame_result (NULL or N values in {0, 1, 2}) and max_fade_length mean what they mean at
 *     amtk_erase_logo_stream_create; the call builds the deint and field logos as the AMTAnalyzeLogo constructor does, with
 *     the same refusals and messages.
 *   - Pixels: for k in [0, nframes), output k is source frame n = frame0 + k with its Y, U and V logo rectangles replaced by
 *     what amtk_erase_logo_frames(ctx, src, logo, n, 1, fades_n) writes, byte for byte.  fades_n is AMTEraseLogo::CalcFade(n)
 *     over the AMTAnalyzeLogo records of src, the records amtk_erase_logo_stream uses for the same N frames: output n equals
 *     the stream's output n, and the fades equal the host's (amtk_calc_fade2, amtk_calc_fade2_records) bit for bit.
 *   - Records are read from src as it is when the call starts, including frames outside [frame0, frame0 + nframes): output
 *     n reads frames n-8 .. n+8.  Every frame some output's CalcFade2 reads is analysed exactly once per call, and all
 *     analysis is done before anything is written.  A uniform or absent need (a uniform frame_result) analyses nothing and
 *     launches no evaluation kernel.
 *   - dst == NULL: in place on src, logo rectangles only.  src may be device resident, or in host memory with the rectangle
 *     rows staged as amtk_erase_logo_frames does (amtk_ctx_last_h2d_bytes counts the rectangles the analysis and the erase
 *     moved).  Ranges split across several in-place calls are exact only if no call's record window (frame0 - 8 ..
 *     frame0 + nframes + 7) reaches frames an earlier call erased: erase out of place, or in one call.
 *   - dst != NULL: a device-resident clip of src's size and sample format in any layout, holding at least nframes frames and
 *     not overlapping src, which must be device resident too.  Frame k of dst receives the whole of output k; only the
 *     sample bytes of each row are written (row padding stays untouched, as amtk_tnr_frames).  src is not modified.
 *   - fades_out (may be NULL; host pointer): float[nframes][2] = {fadeT, fadeB}.
 *   - Refused with the reason, before anything is written: what amtk_erase_logo_stream_create refuses; a frame range outside
 *     the clip; a logo rectangle outside the frame; a chroma subsampling mismatch; when some frame is analysed, a sample
 *     size the evaluation plan refuses; a dst that is on the host, of another format, too short or overlapping src; a host
 *     src with a dst.
 *   - Launches (device-resident src): 6 per evaluation pass when some frame is analysed (three evaluations of two kernels;
 *     one pass holds 96 MiB / (44 * countPad) analysed frames, ~545 for a 64x64 logo of 4096 feature pixels), plus
 *     erase_fade_kernel and one erase kernel (erase_logo_kernel in place, erase_copy_kernel out of place).  The count does
 *     not grow with nframes while the analysed frames fit one pass.
 *   - HBM: N * 33 floats of records when some frame is analysed, 8 bytes of fades per output and N bytes of fade codes,
 *     kept by the context for its next call; the deint and field logos' tables while the call runs. */
AMTK_API int amtk_erase_logo_clip(amtk_ctx* ctx, const amtk_clip* src, const amtk_clip* dst, const amtk_logo* logo,
                                  float maskratio, const uint8_t* frame_result, int max_fade_length,
                                  int frame0, int nframes, float* fades_out);

/* LogoFrame(ctx, logofiles, maskratio) and its IterateFrames loop (LogoScan.hpp:1570-1630), the logo detection CMAnalyze
 * runs over a whole recording, fed one decoded frame at a time and read back in frame order.  Only the luma rectangles of
 * the evaluated logos cross PCIe, and the evaluations of B frames run as one batch.  Spec: DESIGN.md section 3.3.3.
 *   - Results: the result for sent frame n equals amtk_logo_scan_frames(ctx, frame_n, logos, nlogos, 0, 1, p, out, 0) bit
 *     for bit, with p = frame_n.pitch_y when reference_pitch is set and samples are 2 bytes, else 0.  A NULL logo, or a
 *     logo whose imgw/imgh differ from the frame's size, gives (0, -1) and costs no device work.
 *   - Format: the first frame fixes width, height, bits and sample size (1-byte samples at 8 bits or 2-byte samples at
 *     9..16 bits) and chroma subsampling.  Later frames must match, in any layout (pitches, plane order), from host memory
 *     (pinned or pageable) or device memory.  Each frame is addressed with its own pitch, including the reference_pitch row
 *     step (the byte pitch in elements: rows two physical rows apart at 16 bits).
 *   - Rejected, leaving the stream as it was: a clip of other than one frame, a frame of another format, a frame on which an
 *     evaluated logo's rectangle, as addressed, leaves the Y plane ("logo rectangle lies outside the frame", as
 *     amtk_logo_scan_frames refuses it), and a first frame whose sample size the evaluation plan refuses.
 *   - Receive rule, with S the frames sent, B = batch_size and batch k = frames [kB, (k+1)B): the send that makes
 *     S = (k+1)B launches batch k; finish launches the open partial batch, if any, and closes the stream to sends
 *     ("closed (finished)").  Batch k's results can be received once batch k+1 was launched, or after finish; they come in
 *     frame order.  recv waits on the device only for batches it delivers from; otherwise it returns 1 with *got = 0.  The
 *     rule does not depend on timing.
 *   - Host frames: send copies the rectangle rows into a pinned batch buffer and returns; the caller may reuse the frame.
 *     Each launch uploads one copy per run of host slots.  Device frames are gathered on the device by one kernel launch.
 *   - Counts: h2d_bytes grows by the sum over evaluated logos of w*h*bytes_per_sample per host frame, d2h_bytes by
 *     8*nlogos per result.  amtk_ctx_launch_count grows by 2 per evaluated logo per batch and by 1 per device frame.
 *   - A CUDA error closes the stream (then only counts and destroy succeed).  destroy is valid at any point and waits for
 *     the stream's device work.  Calls serialise on the context; streams on one context are independent.
 *   - HBM: per batch not yet received, B slots of the evaluated rectangles and B*nlogos result pairs. */
typedef struct amtk_logo_scan_stream amtk_logo_scan_stream;
/* logos[i]: DEINT logos with masks, or NULL (an invalid logo -> (0, -1), :1551-1558).  The stream keeps its own copies: the
 * caller may destroy its logos after create.  reference_pitch = 1: 2-byte Y planes are addressed with the byte pitch as
 * ScanFrame does (:1547,1561).  Refused with the reason: null ctx or out, nlogos < 1, batch_size outside [1, 256], a logo
 * without a mask, a logo with no feature pixels, a logo the evaluation plan refuses at 1-byte samples.  These checks apply to
 * every non-NULL logo, also one whose imgw/imgh will not match the frames (which amtk_logo_scan_frames never looks at); a
 * caller that knows the frame size passes NULL for such a logo, since it gives (0, -1) either way. */
AMTK_API int amtk_logo_scan_stream_create(amtk_ctx* ctx, amtk_logo* const* logos, int nlogos, int batch_size,
                                          int reference_pitch, amtk_logo_scan_stream** out);
AMTK_API void amtk_logo_scan_stream_destroy(amtk_logo_scan_stream* s);
/* frame: ONE frame, frame S (0-based) of the recording */
AMTK_API int amtk_logo_scan_stream_send(amtk_logo_scan_stream* s, const amtk_clip* frame);
/* end of input */
AMTK_API int amtk_logo_scan_stream_finish(amtk_logo_scan_stream* s);
/* up to max_frames results in frame order: out float[*got][nlogos][2] = EvalResult{corr0, corr1} (:1532-1535) */
AMTK_API int amtk_logo_scan_stream_recv(amtk_logo_scan_stream* s, float* out, int max_frames, int* got);
/* frames sent, results received, payload bytes host->device and device->host (any may be NULL) */
AMTK_API int amtk_logo_scan_stream_counts(const amtk_logo_scan_stream* s, int* sent, int* received,
                                          int64_t* h2d_bytes, int64_t* d2h_bytes);

/* The combing / field-difference counters (amtk_comb_frames) of the telecine pre-pass (KFM pass 1 under
 * AMTFilterSource::ReadAllFrames, FilteredSource.hpp:417-439) over a recording fed one decoded frame at a time and read
 * back in frame order.  Each frame crosses PCIe once: the frame before a batch reaches the batch's halo slot by a
 * device-to-device copy.  Spec: DESIGN.md section 3.1d.
 *   - Results: with C the clip of all frames sent, the 12 counters of sent frame n equal row n of
 *     amtk_comb_frames(ctx, C, params, 0, N, ...): the previous frame of frame 0 is frame 0 itself, of frame n frame n-1.
 *     They are integers and identical, not close.
 *   - Format: the first frame fixes width, height, bits, sample size and chroma subsampling, and must be a frame
 *     amtk_comb_frames accepts; the thresholds are checked for its sample size then (comb_thresholds_ok's messages), and a
 *     refused first frame fixes no format.  Later frames must match, in any layout (pitches, plane order), from host
 *     memory (pinned or pageable) or device memory.  The frames are kept in the stream's own layout (16-byte aligned
 *     pitches and planes), so the TMA kernels run whatever the frames' own layout.
 *   - Rejected, leaving the stream as it was: a clip of other than one frame, a frame of another format, a send after
 *     finish ("closed (finished)") and a second finish.
 *   - Receive rule, with S the frames sent, B = batch_size and batch k = frames [kB, (k+1)B): the send that makes
 *     S = (k+1)B launches batch k; finish launches the open partial batch, if any.  Batch k's rows can be received once
 *     batch k+1 was launched, or after finish; they come in frame order.  recv waits on the device only for batches it
 *     delivers from; otherwise it returns 1 with *got = 0.  The rule does not depend on timing.
 *   - Host frames: send copies the three planes into a pinned batch buffer and returns; the caller may reuse the frame.
 *     Each launch uploads one copy per run of host slots.  Device frames are copied on the context's stream, in order with
 *     the caller's work there.
 *   - Counts: h2d_bytes grows by one slot frame (the stream layout's frame_stride) per host frame, d2h_bytes by 48 per
 *     result.  amtk_ctx_launch_count and the kernel timing grow by one comb launch per batch.
 *   - Watchdog: each band-form batch keeps its own copy of the kernel's watchdog record; recv checks it before delivering
 *     that batch's rows, so another comb call on the context in between cannot hide a timed-out wait.  (As for any comb
 *     call, the context's next comb launch also checks the last launch's record and fails if its wait timed out.)
 *   - A CUDA error closes the stream (then only counts and destroy succeed).  destroy is valid at any point and waits for
 *     the stream's device work.  Calls serialise on the context; streams on one context are independent.  Other comb calls
 *     on the context in between are correct, but the cached launch plan is then rebuilt.
 *   - Memory: per batch not yet received, one device buffer and its pinned twin of 48*B bytes + (B+1) slot frames. */
typedef struct amtk_comb_stream amtk_comb_stream;
/* Refused with the reason: null ctx, params or out, batch_size outside [1, 256], a threshold < 1. */
AMTK_API int amtk_comb_stream_create(amtk_ctx* ctx, const amtk_comb_params* params, int batch_size, amtk_comb_stream** out);
AMTK_API void amtk_comb_stream_destroy(amtk_comb_stream* s);
/* frame: ONE frame, frame S (0-based) of the recording */
AMTK_API int amtk_comb_stream_send(amtk_comb_stream* s, const amtk_clip* frame);
/* end of input */
AMTK_API int amtk_comb_stream_finish(amtk_comb_stream* s);
/* up to max_frames rows in frame order: counts int32[*got][12], as amtk_comb_frames */
AMTK_API int amtk_comb_stream_recv(amtk_comb_stream* s, int32_t* counts, int max_frames, int* got);
/* frames sent, rows received, payload bytes host->device and device->host (any may be NULL) */
AMTK_API int amtk_comb_stream_counts(const amtk_comb_stream* s, int* sent, int* received, int64_t* h2d_bytes, int64_t* d2h_bytes);

/* The fused step (amtk_scan_comb_frames: the ScanFrame scores of LogoFrame and the combing counters of the telecine
 * pre-pass) over a recording fed one decoded frame at a time and read back in frame order, so that CMAnalyze's logo
 * detection and the pre-pass share one decode.  Each frame crosses PCIe once; the logo rectangles are read from the frames
 * kept in HBM, and the frame before a batch reaches the batch's halo slot by a device-to-device copy.  Spec: DESIGN.md
 * section 3.1e.
 *   - Results: with C the clip of all N frames sent, the results of sent frame n equal row n of
 *     amtk_scan_comb_frames(ctx, C, logos, nlogos, params, 0, N, ...) bit for bit: nlogos score pairs and 12 counters.  The
 *     previous frame of frame 0 is frame 0 itself, of frame n frame n-1.  A NULL logo, or a logo whose imgw/imgh differ from
 *     the frame's size, gives (0, -1).
 *   - Format: the first frame fixes width, height, bits, sample size and chroma subsampling, and must be a frame
 *     amtk_scan_comb_frames accepts; the thresholds are checked for its sample size then (comb_thresholds_ok's messages),
 *     every evaluated logo's rectangle must lie inside it ("logo rectangle lies outside the frame") and have an evaluation
 *     plan at its sample size; a refused first frame fixes no format.  Later frames must match, in any layout (pitches,
 *     plane order), from host memory (pinned or pageable) or device memory.  The frames are kept in the comb stream's slot
 *     layout (16-byte aligned pitches and planes), so the TMA kernels run whatever the frames' own layout.
 *   - Rejected, leaving the stream as it was: a clip of other than one frame, a frame of another format, a first frame as
 *     above, a send after finish ("closed (finished)") and a second finish.
 *   - Receive rule, with S the frames sent, B = batch_size and batch k = frames [kB, (k+1)B): the send that makes
 *     S = (k+1)B launches batch k; finish launches the open partial batch, if any.  Batch k's results can be received once
 *     batch k+1 was launched, or after finish; they come in frame order.  recv waits on the device only for batches it
 *     delivers from; otherwise it returns 1 with *got = 0.  The rule does not depend on timing.
 *   - Host frames: send copies the three planes into a pinned batch buffer and returns; the caller may reuse the frame.
 *     Each launch uploads one copy per run of host slots.  Device frames are copied on the context's stream, in order with
 *     the caller's work there.
 *   - Counts: h2d_bytes grows by one slot frame (the stream layout's frame_stride) per host frame, d2h_bytes by
 *     48 + 8*nlogos per result.  amtk_ctx_launch_count grows per batch by exactly the launches amtk_scan_comb_frames makes
 *     on a device clip of the batch's frames: 1 when the batch runs fused (8-bit frames, nlogos = 1, an evaluated logo
 *     whose logo item fits in the band-form comb kernel's ring: the scores come from that one launch's logo items), else
 *     1 comb launch + 2 per evaluated logo + 1 per other logo.
 *   - Watchdog: each band-form batch keeps its own copy of the kernel's watchdog record; recv checks it before delivering
 *     that batch's results, as the comb stream does.
 *   - A CUDA error closes the stream (then only counts and destroy succeed).  destroy is valid at any point and waits for
 *     the stream's device work.  Calls serialise on the context; streams on one context are independent.  Other comb or
 *     logo calls on the context in between are correct, but the cached launch plan is then rebuilt.
 *   - Memory: per batch not yet received, one device buffer and its pinned twin of (48 + 8*nlogos)*B bytes + (B+1) slot
 *     frames. */
typedef struct amtk_scan_comb_stream amtk_scan_comb_stream;
/* logos[i]: DEINT logos with masks, or NULL; the stream keeps its own copies.  Refused with the reason: null ctx, logos,
 * params or out, nlogos < 1, batch_size outside [1, 256], a threshold < 1, a logo without a mask, a logo with no feature
 * pixels, a logo the evaluation plan refuses at 1-byte samples (as amtk_logo_scan_stream_create). */
AMTK_API int amtk_scan_comb_stream_create(amtk_ctx* ctx, amtk_logo* const* logos, int nlogos, const amtk_comb_params* params,
                                          int batch_size, amtk_scan_comb_stream** out);
/* The same stream with ScanFrame's byte-pitch row step (as amtk_logo_scan_stream_create's reference_pitch):
 * reference_pitch = 0 is amtk_scan_comb_stream_create.  reference_pitch = 1 addresses 2-byte Y planes with the byte pitch
 * as element pitch, so element row r of the logo evaluation is luma row 2r of the frame: the results of sent frame n then
 * equal row n of amtk_scan_comb_frames_pitch(ctx, C, logos, nlogos, params, C.pitch_y, 0, N, ...) on a resident clip C
 * of the frames sent, the scores those of amtk_logo_scan_stream with reference_pitch = 1 and the counters the comb
 * stream's.  Every 2-byte frame is then also refused, leaving the stream as it was, when an evaluated logo's rectangle as
 * addressed leaves the frame's Y plane ("logo rectangle lies outside the frame"; on even heights: imgy + h > height / 2).
 * The logo kernels read the rectangles from the slots with the slot's byte pitch as element pitch, which addresses the
 * same samples whatever the frame's own pitch.  Per batch the launches of amtk_scan_comb_frames_pitch on a device clip of
 * the batch's slots (2-byte frames: 1 comb launch + 2 per evaluated logo + 1 per other logo); 1-byte frames run as
 * amtk_scan_comb_stream_create's.  Everything else as amtk_scan_comb_stream_create. */
AMTK_API int amtk_scan_comb_stream_create_pitch(amtk_ctx* ctx, amtk_logo* const* logos, int nlogos,
                                                const amtk_comb_params* params, int batch_size, int reference_pitch,
                                                amtk_scan_comb_stream** out);
AMTK_API void amtk_scan_comb_stream_destroy(amtk_scan_comb_stream* s);
/* frame: ONE frame, frame S (0-based) of the recording */
AMTK_API int amtk_scan_comb_stream_send(amtk_scan_comb_stream* s, const amtk_clip* frame);
/* end of input */
AMTK_API int amtk_scan_comb_stream_finish(amtk_scan_comb_stream* s);
/* up to max_frames results in frame order: scores float[*got][nlogos][2] (corr0, corr1) and counts int32[*got][12], as
 * amtk_scan_comb_frames */
AMTK_API int amtk_scan_comb_stream_recv(amtk_scan_comb_stream* s, float* scores, int32_t* counts, int max_frames, int* got);
/* frames sent, results received, payload bytes host->device and device->host (any may be NULL) */
AMTK_API int amtk_scan_comb_stream_counts(const amtk_scan_comb_stream* s, int* sent, int* received, int64_t* h2d_bytes,
                                          int64_t* d2h_bytes);

/* ---------------------------------------------------------------------------------------------
 * Logo finder: where the logo rectangle is, the imgx, imgy, w, h that amtk_scan_logo and amtk_scan_logo_stream take (the
 * reference's GUI has the user draw it on a preview frame, LogoGUISupport.hpp:15-177).  Spec: DESIGN.md section 3.5.
 * ------------------------------------------------------------------------------------------- */
typedef struct amtk_logo_find amtk_logo_find;
AMTK_API int amtk_logo_find_create(amtk_ctx* ctx, amtk_logo_find** out);
AMTK_API void amtk_logo_find_destroy(amtk_logo_find* f);
/* Adds frames [frame0, frame0+nframes) of clip: for every luma sample Y, s1[y][x] += Y and s2[y][x] += Y*Y, exact 64-bit
 * integers whatever the order or split of the frames.  Only the Y plane is read.  The clip may be in host memory (pinned
 * or pageable; only the Y rows are copied, width * height * bytes_per_sample per frame, amtk_ctx_last_h2d_bytes) or
 * device memory, in any layout; one-frame clips are welcome.  The first clip fixes width, height, bits and sample size:
 * 1-byte samples at 8 bits or 2-byte samples at 9..16 bits (as amtk_scan_add_frames takes them); width and height in
 * [16, 8192].  Refused with the reason, leaving the sums as they were: a clip of another format, a frame range outside the
 * clip.  One kernel launch per call on a device clip, one per staged chunk on a host clip.  HBM: 16 bytes per pixel. */
AMTK_API int amtk_logo_find_add_frames(amtk_logo_find* f, const amtk_clip* clip, int frame0, int nframes);
/* s1, s2: host uint64[height][width] (either may be NULL); *nframes (may be NULL) = frames added so far.  The only
 * device-to-host copy of the finder. */
AMTK_API int amtk_logo_find_get_sums(amtk_logo_find* f, uint64_t* s1, uint64_t* s2, int64_t* nframes);

/* The rectangles, from the sums alone (host code, no device needed).  A logo is what stays put while the picture moves
 * under it: over many frames it lowers the variance of the pixels it covers (by (1 - alpha)^2 where it is always shown),
 * and its edges stay sharp in the temporal mean, where moving content blurs into a smooth field.  The rule (DESIGN.md
 * section 3.5), in double, with n = nframes, maxv = (1 << bits) - 1, per pixel mean m = s1 / n, variance s2 / n - m^2
 * and edge strength |m(x+1, y) - m(x, y)| + |m(x, y+1) - m(x, y)| (a neighbour outside the frame counts 0), over the
 * blocks of block x block pixels that lie wholly inside the frame:
 *   1. Per block, the mean of its pixels' variances and of their edge strengths; the medians of both over all blocks.
 *   2. A block is "held" when its variance <= var_ratio * the median variance, or its edge strength >= the median edge
 *      strength + mean_delta * maxv / 255.  Blocks in the outermost row or column of blocks are never held.
 *   3. Held blocks are joined into 8-connected components.  Components of fewer than min_blocks blocks are dropped, and
 *      so are letterbox and pillarbox bars: components that reach from the second column of blocks to the second-to-last,
 *      or from the second row to the second-to-last.
 *   4. Each component's bounding box grows by margin pixels on each side and is clipped to the frame; the left and top
 *      edges are rounded down and the right and bottom edges up to even values within the frame's even size, and w and h
 *      are clamped to [4, 4096] (amtk_scan_logo_stream_create's limits), moving imgx, imgy back inside the frame.
 *   5. Score = the sum over its held blocks of max(0, 1 - variance / median variance) + max(0, edge strength - median
 *      edge strength) / (mean_delta * maxv / 255).  Rectangles come best first; equal scores in raster order.
 * Fewer than 2 frames, or a median block variance of 0 (a still picture), give *n = 0 without error.  Refused: null s1,
 * s2, p or n, a null rects with max_rects > 0, block < 2, width or height outside [16, 8192], bits outside 8..16,
 * max_rects < 0.  At most max_rects rectangles are written; *n is the number written. */
typedef struct amtk_logo_find_params {
  int32_t block;          /* block edge in pixels, default 8                                                           */
  float   var_ratio;      /* a block is "held" when its variance <= var_ratio * the frame's median block variance, default 0.5 */
  float   mean_delta;     /* ... or when its edge strength in the temporal mean >= the median + mean_delta * (maxv / 255),
                           * default 6 */
  int32_t margin;         /* pixels added on each side of a component, default 8                                       */
  int32_t min_blocks;     /* components smaller than this are dropped, default 4                                       */
} amtk_logo_find_params;
AMTK_API void amtk_logo_find_default_params(amtk_logo_find_params* p);
/* rects int32[*n][4] = imgx, imgy, w, h, best first; scores float[*n] (may be NULL) */
AMTK_API int amtk_logo_find_rects(const uint64_t* s1, const uint64_t* s2, int64_t nframes, int width, int height, int bits,
                                  const amtk_logo_find_params* p, int max_rects, int32_t* rects, float* scores, int* n);

/* ---------------------------------------------------------------------------------------------
 * Multi-GPU (SURVEY.md 8(e)): ONE process drives several devices -- a context, a stream and a host thread per device
 * (each thread pinned to the CPUs next to its GPU), NCCL over NVLink only for the final gather of the small per-frame
 * result blocks and for the exact integer all-reduce of a frame-sharded LogoScan.  This is what the reference's
 * job-per-GPU scheduler (AmatsukazeServer/Server/ResourceManager.cs:81-85, Amatsukaze/InterProcessComm.hpp:87-95) would
 * drive from C++/C#.  NCCL is loaded with dlopen on first use; one device needs no NCCL at all.
 * ------------------------------------------------------------------------------------------- */
typedef struct amtk_group amtk_group;
/* devices: CUDA ordinals (NULL = 0..ndev-1) */
AMTK_API int amtk_group_create(int ndev, const int* devices, amtk_group** out);
AMTK_API void amtk_group_destroy(amtk_group* g);
AMTK_API int amtk_group_size(const amtk_group* g);
/* the context of member i: create logos / scans / device buffers for that device through it */
AMTK_API amtk_ctx* amtk_group_ctx(amtk_group* g, int i);
/* CPUs member i's host thread was bound to (0 = not bound), NCCL version in use (0 = none) */
AMTK_API int amtk_group_numa_cpus(const amtk_group* g, int i);
AMTK_API int amtk_group_nccl_version(const amtk_group* g);
/* pinned host memory allocated and first-touched by member i's thread (NUMA-local to its GPU) */
AMTK_API int amtk_group_host_alloc(amtk_group* g, int i, size_t bytes, void** out);
/* BASELINE configs[4]: clips[i] (host or device resident, all with >= nframes frames) is analysed on member i with logos[i]
 * (amtk_scan_comb_frames semantics, frames [0, nframes)), then ONE ncclAllGather of the per-member result blocks.
 * Device clips: returns when the work is enqueued (asynchronous); host clips: returns when the staging is done. */
AMTK_API int amtk_group_scan_comb_streams(amtk_group* g, const amtk_clip* clips, amtk_logo* const* logos,
                                          const amtk_comb_params* params, int nframes);
/* gathered results of the last pass as held by member `from`: scores float[ndev][nframes][2], counts int32[ndev][nframes][12] */
AMTK_API int amtk_group_fetch_results(amtk_group* g, int from, int nframes, float* scores, int32_t* counts);
AMTK_API int amtk_group_synchronize(amtk_group* g);
/* device-side timing: mark = one CUDA event per member after everything enqueued so far (compute and collective);
 * elapsed = milliseconds between two marks per member (take the maximum) */
AMTK_API int amtk_group_mark(amtk_group* g, int slot);
AMTK_API int amtk_group_elapsed_ms(amtk_group* g, int slot_a, int slot_b, double* ms_per_member);
/* frame-sharded LogoScan: member i adds frames [frame0[i], frame0[i]+nframes[i]) of clips[i] to scans[i] (created on
 * amtk_group_ctx(g, i)), then ONE ncclAllReduce(ncclSum, ncclUint64) leaves the whole-clip sums in every scans[i]. */
AMTK_API int amtk_group_scan_add_frames(amtk_group* g, amtk_scan* const* scans, const amtk_clip* clips, int scanx, int scany,
                                        const int* frame0, const int* nframes);

#ifdef __cplusplus
}
#endif
#endif /* AMTK_B200_H */
