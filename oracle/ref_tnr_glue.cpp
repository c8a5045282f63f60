// oracle/ref_tnr_glue.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles the reference's VideoFilter / TemporalNRFilter (VideoFilter.hpp:9-212, extracted verbatim by
// oracle/build_ref_tnr.sh into _ref/ref_tnr.inc) against minimal stand-ins for what those lines use from FFmpeg and the
// reference's CoreUtils / Transcode headers, and exports two entry points for the tests:
//   ref_tnr_sequence: the filter's own onFrame/finish queue over a whole clip (which frames it emits, and their pixels);
//   ref_tnr_window:   TNRFilter (and so filterKernel) on an explicit window of 2d+1 frames.
// Nothing here is algorithmic: frames go in and out as packed planar 4:2:0 (Y W*H, U and V (W/2)*(H/2), `bps` bytes a sample).
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <memory>
#include <utility>
#include <vector>

struct NonCopyable {
  NonCopyable() {}
  NonCopyable(const NonCopyable&) = delete;
  NonCopyable& operator=(const NonCopyable&) = delete;
};
struct InvalidOperationException {};
struct FormatException {};
struct RuntimeException {};
#define THROW(type, msg) throw type()

enum AVPixelFormat { AV_PIX_FMT_YUV420P, AV_PIX_FMT_YUV420P10LE, AV_PIX_FMT_YUV420P12LE, AV_PIX_FMT_YUV420P14LE, AV_PIX_FMT_YUV420P16LE };
struct AVComponentDescriptor { int depth; };
struct AVPixFmtDescriptor { AVComponentDescriptor comp[4]; };
static const AVPixFmtDescriptor* av_pix_fmt_desc_get(AVPixelFormat f) {
  static const AVPixFmtDescriptor d[5] = { { { { 8 } } }, { { { 10 } } }, { { { 12 } } }, { { { 14 } } }, { { { 16 } } } };
  return &d[f];
}
struct AVFrame {
  uint8_t* data[4] = { nullptr, nullptr, nullptr, nullptr };
  int linesize[4] = { 0, 0, 0, 0 };
  int format = 0, width = 0, height = 0;
  std::vector<uint8_t> buf;
};
static void av_frame_copy_props(AVFrame*, const AVFrame*) {}
// rows padded to `align` bytes, as FFmpeg's allocator does
static int av_frame_get_buffer(AVFrame* f, int align) {
  const int bps = f->format == AV_PIX_FMT_YUV420P ? 1 : 2;
  const int ly = (f->width * bps + align - 1) / align * align, lc = ((f->width / 2) * bps + align - 1) / align * align;
  const size_t ysz = (size_t)ly * f->height, csz = (size_t)lc * (f->height / 2);
  f->buf.assign(ysz + 2 * csz, 0);
  f->linesize[0] = ly; f->linesize[1] = f->linesize[2] = lc;
  f->data[0] = f->buf.data(); f->data[1] = f->data[0] + ysz; f->data[2] = f->data[1] + csz;
  return 0;
}
namespace av {
class Frame {
public:
  int frameIndex_;
  explicit Frame(int frameIndex = -1) : frameIndex_(frameIndex), frame_(new AVFrame()) {}
  AVFrame* operator()() { return frame_.get(); }
private:
  std::unique_ptr<AVFrame> frame_;
};
}  // namespace av

// the tests call the filter's private TNRFilter directly (ref_tnr_window)
#define private public
#include "ref_tnr.inc"
#undef private

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
  for (int p = 0; p < 3; ++p) {
    for (int y = 0; y < rows[p]; ++y) memcpy(f->data[p] + (size_t)y * f->linesize[p], packed, rb[p]), packed += rb[p];
  }
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
}  // namespace

extern "C" {

// init(d, t, interlaced), onFrame for frames 0..N-1 (frameIndex_ = n), finish.  Writes the emitted frames to out (room for
// N frames) and their frameIndex_ to out_idx; returns how many were emitted, -1 if the filter threw.
int ref_tnr_sequence(const void* frames, int N, int W, int H, int bps, int bits, int d, int threshold, int interlaced,
                     void* out, int32_t* out_idx) {
  try {
    TemporalNRFilter f;
    Collect c;
    f.nextFilter = &c;
    f.init(d, threshold, interlaced != 0);
    f.start();
    const size_t fs = frame_bytes(W, H, bps);
    for (int n = 0; n < N; ++n) f.onFrame(make_frame((const uint8_t*)frames + (size_t)n * fs, W, H, bps, bits, n));
    f.finish();
    const int m = (int)c.frames.size();
    for (int k = 0; k < m && k < N; ++k) {
      read_frame((*c.frames[k])(), W, H, bps, (uint8_t*)out + (size_t)k * fs);
      out_idx[k] = c.frames[k]->frameIndex_;
    }
    return m;
  } catch (...) {
    return -1;
  }
}

// TNRFilter on the explicit window win[0..nf-1] (nf = 2d+1).  Returns 0 if the filter threw.
int ref_tnr_window(const void* const* win, int nf, int W, int H, int bps, int bits, int threshold, int interlaced, void* out) {
  try {
    TemporalNRFilter f;
    f.init((nf - 1) / 2, threshold, interlaced != 0);
    std::vector<std::unique_ptr<av::Frame>> keep;
    AVFrame* frames[128];
    for (int i = 0; i < nf; ++i) {
      keep.push_back(make_frame((const uint8_t*)win[i], W, H, bps, bits, i));
      frames[i] = (*keep.back())();
    }
    std::unique_ptr<av::Frame> r = f.TNRFilter(frames, 0);
    read_frame((*r)(), W, H, bps, (uint8_t*)out);
    return 1;
  } catch (...) {
    return 0;
  }
}

}  // extern "C"
