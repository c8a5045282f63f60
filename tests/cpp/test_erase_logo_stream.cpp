// tests/cpp/test_erase_logo_stream.cpp -- AMTEraseLogo of the host-side mirror over a child that is not device resident:
// MakeSource's chain AMTEraseLogo(AMTAnalyzeLogo(src, logo), logo, logof, maxfade) served from the frame stream for
// in-order reads and from the per-frame path for the others, on a host clip that counts the GetFrame calls per frame.
// usage: test_erase_logo_stream order <raw> <logo.lgd> <logo2.lgd|-> <logof|-> <maxfade> <orders.bin> <out.bin> <tnr 0|1>
//        (driven by tests/test_gpu_erase_logo_stream_filter.py)
#include "../../amatsukaze_b200/host/filters.hpp"
#include <string>

static void dump(const std::string& path, const std::vector<uint8_t>& v) {
  FILE* fp = fopen(path.c_str(), "wb");
  if (!fp) { fprintf(stderr, "cannot write %s\n", path.c_str()); exit(2); }
  fwrite(v.data(), 1, v.size(), fp); fclose(fp);
}
static void pack(const PVideoFrame& f, std::vector<uint8_t>& out) {      // CPU frame -> tight planar bytes
  const int pl[3] = { PLANAR_Y, PLANAR_U, PLANAR_V };
  for (int p = 0; p < 3; ++p)
    for (int y = 0; y < f->GetHeight(pl[p]); ++y)
      out.insert(out.end(), f->GetReadPtr(pl[p]) + (size_t)y * f->GetPitch(pl[p]), f->GetReadPtr(pl[p]) + (size_t)y * f->GetPitch(pl[p]) + f->GetRowSize(pl[p]));
}

// A CPU-only source (not an IDeviceClip) over an AMTSRAW1 file of packed 4:2:0 pictures at 8 bits; calls[n] counts the
// requests for frame n.
class CountingClip : public IClip {
  VideoInfo vi_;
  std::vector<uint8_t> data_;
  size_t fsz_ = 0;
public:
  std::vector<int> calls;
  explicit CountingClip(const std::string& path) {
    FILE* fp = fopen(path.c_str(), "rb");
    char magic[8]; int32_t h[6];
    if (!fp || fread(magic, 1, 8, fp) != 8 || fread(h, 4, 6, fp) != 6 || h[2] != 8) throw AvisynthError("CountingClip: bad file " + path);
    vi_.width = h[0]; vi_.height = h[1]; vi_.num_frames = h[3]; vi_.pixel_type = VideoInfo::CS_YV12;
    fsz_ = (size_t)vi_.width * vi_.height * 3 / 2;
    data_.resize(fsz_ * vi_.num_frames);
    const bool ok = fread(data_.data(), 1, data_.size(), fp) == data_.size();
    fclose(fp);
    if (!ok) throw AvisynthError("CountingClip: truncated " + path);
    calls.assign(vi_.num_frames, 0);
  }
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    n = std::max(0, std::min(vi_.num_frames - 1, n));
    calls[n] += 1;
    PVideoFrame f = env->NewVideoFrame(vi_);
    const uint8_t* src = data_.data() + fsz_ * (size_t)n;
    const int planes[3] = { PLANAR_Y, PLANAR_U, PLANAR_V };
    for (int p = 0; p < 3; ++p) {
      const int rows = f->GetHeight(planes[p]), rb = f->GetRowSize(planes[p]);
      for (int y = 0; y < rows; ++y, src += rb) memcpy(f->GetWritePtr(planes[p]) + (size_t)y * f->GetPitch(planes[p]), src, rb);
    }
    return f;
  }
  bool __stdcall GetParity(int) override { return true; }
  void __stdcall GetAudio(void*, int64_t, int64_t, IScriptEnvironment*) override {}
  int __stdcall SetCacheHints(int, int) override { return 0; }
  const VideoInfo& __stdcall GetVideoInfo() override { return vi_; }
};

static AVSValue Call(IScriptEnvironment* env, const char* name, std::vector<AVSValue> args) { return env->Invoke(name, AVSValue(args)); }

// MakeSource's eraser lines (FilteredSource.hpp:441-475) over `src`: the logo, then the extra erase logo if any
static PClip Erasers(IScriptEnvironment* env, PClip src, const std::vector<std::string>& logos, const std::string& logof, int maxfade,
                     std::vector<PClip>& erasers) {
  PClip last = src;
  for (const auto& lg : logos) {
    PClip ana = Call(env, "AMTAnalyzeLogo", { AVSValue(last), AVSValue(lg), AVSValue(35) }).AsClip();
    last = Call(env, "AMTEraseLogo", { AVSValue(last), AVSValue(ana), AVSValue(lg), logof.empty() ? AVSValue() : AVSValue(logof),
                                       AVSValue(0), AVSValue(maxfade) }).AsClip();
    erasers.push_back(last);
  }
  return last;
}

static std::vector<int> ReadOrder(const std::string& path) {
  std::vector<int> v;
  FILE* fp = fopen(path.c_str(), "rb");
  if (!fp) throw AvisynthError("cannot read " + path);
  int32_t x;
  while (fread(&x, 4, 1, fp) == 1) v.push_back(x);
  fclose(fp);
  return v;
}

int main(int argc, char** argv) {
  if (argc != 10 || std::string(argv[1]) != "order") { fprintf(stderr, "usage: test_erase_logo_stream order ...\n"); return 2; }
  amtk_ctx* actx = nullptr;
  if (!amtk_ctx_create(0, nullptr, &actx)) { fprintf(stderr, "ctx: %s\n", amtk_last_error()); return 3; }
  int rc = 0;
  try {
    IScriptEnvironment2 env;
    BindDevice(&env, actx, DEV_TYPE_CPU);
    av::AddBuiltins(&env);
    AvisynthPluginInit3(&env, nullptr);
    std::vector<std::string> logos = { argv[3] };
    if (std::string(argv[4]) != "-") logos.push_back(argv[4]);
    const std::string logof = std::string(argv[5]) == "-" ? "" : argv[5];
    const int maxfade = atoi(argv[6]);
    const bool tnr = atoi(argv[9]) != 0;
    // orders.bin: int32 frame numbers, patterns separated by -1; each pattern is served by a new chain over a new clip
    const std::vector<int> all = ReadOrder(argv[7]);
    std::vector<uint8_t> packed;
    int k = 0;
    for (size_t i = 0; i < all.size(); ++k) {
      std::vector<int> order;
      for (; i < all.size() && all[i] >= 0; ++i) order.push_back(all[i]);
      ++i;
      auto* cc = new CountingClip(argv[2]);
      PClip src(cc);
      std::vector<PClip> erasers;
      PClip out = Erasers(&env, src, logos, logof, maxfade, erasers);
      if (tnr) out = Call(&env, "KTemporalNR", { AVSValue(out), AVSValue(3), AVSValue(1), AVSValue(false) }).AsClip();
      for (int n : order) pack(out->GetFrame(n, &env), packed);
      int mx = 0, total = 0, zero = 0;
      for (int c : cc->calls) { mx = std::max(mx, c); total += c; zero += c == 0; }
      printf("order %d: reads=%zu", k, order.size());
      for (size_t e = 0; e < erasers.size(); ++e) {
        const auto* er = dynamic_cast<const logo::AMTEraseLogo*>(erasers[e].get());
        printf(" sent%zu=%d streams%zu=%d", e, er->FramesSent(), e, er->StreamsStarted());
      }
      printf(" child_max=%d child_total=%d child_unasked=%d\n", mx, total, zero);
    }
    dump(argv[8], packed);
  } catch (const AvisynthError& e) {
    fprintf(stderr, "AvisynthError: %s\n", e.msg.c_str()); rc = 4;
  } catch (const std::exception& e) {
    fprintf(stderr, "exception: %s\n", e.what()); rc = 5;
  }
  amtk_ctx_destroy(actx);
  printf(rc == 0 ? "OK\n" : "FAILED\n");
  return rc;
}
