// oracle/ref_tnr_stream_glue.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles the reference's own VideoFilter and CudaTemporalNRFilter (VideoFilter.hpp:9-25,214-267, extracted verbatim by
// oracle/build_ref_tnr_stream.sh into _ref/ref_tnr_stream.inc) against stand-ins for FFmpeg's frames and the reference's
// CoreUtils, with oracle/ref_tnr_stream/CudaFilter.h mapping its cudaTNR* calls onto the library's amtk_tnr_stream_*.
// The library is loaded from the path the caller passes.  One entry point for the tests:
//   ref_tnr_stream_run: init, onFrame for frames 0..N-1 (frameIndex_ = n), finish; the frames and frameIndex_ values the
//                       filter emits.
// Frames go in and out as packed planar 4:2:0 (Y W*H, U and V (W/2)*(H/2), `bps` bytes a sample).
#include <dlfcn.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <deque>
#include <memory>
#include <string>
#include <utility>
#include <vector>

struct NonCopyable {
  NonCopyable() {}
  NonCopyable(const NonCopyable&) = delete;
  NonCopyable& operator=(const NonCopyable&) = delete;
};
struct InvalidOperationException {};
struct RuntimeException {};
#define THROW(type, msg) throw type()

enum AVPixelFormat { AV_PIX_FMT_YUV420P, AV_PIX_FMT_YUV420P10LE, AV_PIX_FMT_YUV420P12LE, AV_PIX_FMT_YUV420P14LE, AV_PIX_FMT_YUV420P16LE };
static int bits_of(int format) { static const int b[5] = { 8, 10, 12, 14, 16 }; return b[format]; }

// FFmpeg's reference-counted frame: data points into a shared buffer; copying the AVFrame (av_frame_ref) shares it.
struct AVFrame {
  uint8_t* data[4] = { nullptr, nullptr, nullptr, nullptr };
  int linesize[4] = { 0, 0, 0, 0 };
  int format = 0, width = 0, height = 0;
  std::shared_ptr<std::vector<uint8_t>> buf;
};
static void av_frame_copy_props(AVFrame*, const AVFrame*) {}
static void av_frame_unref(AVFrame* f) {
  f->buf.reset();
  for (int p = 0; p < 4; ++p) { f->data[p] = nullptr; f->linesize[p] = 0; }
}
// a new buffer, rows padded to `align` bytes, as FFmpeg's allocator does
static int av_frame_get_buffer(AVFrame* f, int align) {
  const int bps = f->format == AV_PIX_FMT_YUV420P ? 1 : 2;
  const int ly = (f->width * bps + align - 1) / align * align, lc = ((f->width / 2) * bps + align - 1) / align * align;
  const size_t ysz = (size_t)ly * f->height, csz = (size_t)lc * (f->height / 2);
  f->buf = std::make_shared<std::vector<uint8_t>>(ysz + 2 * csz, 0);
  f->linesize[0] = ly; f->linesize[1] = f->linesize[2] = lc;
  f->data[0] = f->buf->data(); f->data[1] = f->data[0] + ysz; f->data[2] = f->data[1] + csz;
  return 0;
}
namespace av {
class Frame {
public:
  int frameIndex_;
  explicit Frame(int frameIndex = -1) : frameIndex_(frameIndex), frame_(new AVFrame()) {}
  Frame(const Frame& o) : frameIndex_(o.frameIndex_), frame_(new AVFrame(*o.frame_)) {}    // shares the buffer
  AVFrame* operator()() { return frame_.get(); }
private:
  std::unique_ptr<AVFrame> frame_;
};
}  // namespace av

#include "CudaFilter.h"
#include "ref_tnr_stream.inc"

namespace {
AVPixelFormat fmt_of(int bits) {
  switch (bits) { case 10: return AV_PIX_FMT_YUV420P10LE; case 12: return AV_PIX_FMT_YUV420P12LE;
                  case 14: return AV_PIX_FMT_YUV420P14LE; case 16: return AV_PIX_FMT_YUV420P16LE; default: return AV_PIX_FMT_YUV420P; }
}
size_t frame_bytes(int W, int H, int bps) { return ((size_t)W * H + 2 * (size_t)(W / 2) * (H / 2)) * bps; }

std::unique_ptr<av::Frame> make_frame(const uint8_t* packed, int W, int H, int bps, int bits, int index) {
  std::unique_ptr<av::Frame> fr(new av::Frame(index));
  AVFrame* f = (*fr)();
  f->format = fmt_of(bits); f->width = W; f->height = H;
  av_frame_get_buffer(f, 64);
  const int rows[3] = { H, H / 2, H / 2 }, rb[3] = { W * bps, (W / 2) * bps, (W / 2) * bps };
  for (int p = 0; p < 3; ++p)
    for (int y = 0; y < rows[p]; ++y) memcpy(f->data[p] + (size_t)y * f->linesize[p], packed, rb[p]), packed += rb[p];
  return fr;
}
void read_frame(AVFrame* f, int W, int H, int bps, uint8_t* packed) {
  const int rows[3] = { H, H / 2, H / 2 }, rb[3] = { W * bps, (W / 2) * bps, (W / 2) * bps };
  for (int p = 0; p < 3; ++p)
    for (int y = 0; y < rows[p]; ++y) memcpy(packed, f->data[p] + (size_t)y * f->linesize[p], rb[p]), packed += rb[p];
}

class Collect : public VideoFilter {
public:
  std::vector<std::unique_ptr<av::Frame>> frames;
  void start() override {}
  void onFrame(std::unique_ptr<av::Frame>&& frame) override { frames.push_back(std::move(frame)); }
  void finish() override {}
};

template <typename F> bool sym(void* h, const char* name, F* out) {
  *out = reinterpret_cast<F>(dlsym(h, name));
  return *out != nullptr;
}
void set_msg(char* err, int errlen, const std::string& m) {
  if (err && errlen > 0) snprintf(err, (size_t)errlen, "%s", m.c_str());
}
}  // namespace

extern "C" {

// Runs the reference's CudaTemporalNRFilter (init(d, threshold, batch, interlaced), onFrame for frames 0..N-1 with
// frameIndex_ = n, finish) on the library at `libpath`, device 0.  Writes up to out_cap emitted frames to out and their
// frameIndex_ to out_idx; returns how many the filter emitted, or -1 if it threw (err receives the library's last error).
int ref_tnr_stream_run(const char* libpath, const void* frames, int N, int W, int H, int bps, int bits, int d, int threshold,
                       int interlaced, int batch, void* out, int32_t* out_idx, int out_cap, char* err, int errlen) {
  set_msg(err, errlen, "");
  void* h = dlopen(libpath, RTLD_NOW | RTLD_LOCAL);
  if (!h) { set_msg(err, errlen, dlerror()); return -1; }
  int (*ctx_create)(int, void*, amtk_ctx**) = nullptr;
  void (*ctx_destroy)(amtk_ctx*) = nullptr;
  const char* (*last_error)(void) = nullptr;
  if (!sym(h, "amtk_ctx_create", &ctx_create) || !sym(h, "amtk_ctx_destroy", &ctx_destroy) ||
      !sym(h, "amtk_last_error", &last_error) || !sym(h, "amtk_tnr_stream_create", &g_amtk.stream_create) ||
      !sym(h, "amtk_tnr_stream_destroy", &g_amtk.stream_destroy) || !sym(h, "amtk_tnr_stream_send", &g_amtk.stream_send) ||
      !sym(h, "amtk_tnr_stream_recv", &g_amtk.stream_recv) || !sym(h, "amtk_tnr_stream_finish", &g_amtk.stream_finish)) {
    set_msg(err, errlen, "missing amtk_* symbol");
    dlclose(h);
    return -1;
  }
  if (!ctx_create(0, nullptr, &g_amtk.ctx)) { set_msg(err, errlen, last_error()); dlclose(h); return -1; }
  int m = -1;
  try {
    CudaTemporalNRFilter f;
    Collect c;
    f.nextFilter = &c;
    f.init(d, threshold, batch, interlaced);
    f.start();
    const size_t fs = frame_bytes(W, H, bps);
    for (int n = 0; n < N; ++n) f.onFrame(make_frame((const uint8_t*)frames + (size_t)n * fs, W, H, bps, bits, n));
    f.finish();
    m = (int)c.frames.size();
    for (int k = 0; k < m && k < out_cap; ++k) {
      read_frame((*c.frames[k])(), W, H, bps, (uint8_t*)out + (size_t)k * fs);
      out_idx[k] = c.frames[k]->frameIndex_;
    }
  } catch (...) {
    set_msg(err, errlen, last_error());
    m = -1;
  }
  for (CudaTNRFilter t : g_tnr_handles) { g_amtk.stream_destroy(t->s); delete t; }
  g_tnr_handles.clear();
  ctx_destroy(g_amtk.ctx);
  g_amtk.ctx = nullptr;
  dlclose(h);
  return m;
}

}  // extern "C"
