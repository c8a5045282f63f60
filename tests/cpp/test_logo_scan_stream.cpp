// tests/cpp/test_logo_scan_stream.cpp -- logo::LogoFrame of the host-side mirror over a CPU-frame source that counts the
// frames it is asked for (the frame stream) and over the device-resident AMTSource of the same frames (one batched call),
// then CMAnalyze's logo analysis over each of them.
// usage: test_logo_scan_stream <raw> <logo1.lgd> <logo2.lgd> [<more.lgd> ...] <outdir>
//        (driven by tests/test_gpu_logo_scan_stream_filter.py; <raw> is an AMTSRAW1 file of packed 4:2:0 frames at 8 or
//        10 bits whose rows need no padding at 64 bytes; <outdir>/cpu and <outdir>/dev must exist).  The logos are
//        logo1, a file that does not exist, logo2 and the others; CMAnalyze matches the first two and erases the rest.
#include "../../amatsukaze_b200/host/filters.hpp"
#include <string>

static void dump(const std::string& path, const void* p, size_t n) {
  FILE* fp = fopen(path.c_str(), "wb");
  if (!fp) { fprintf(stderr, "cannot write %s\n", path.c_str()); exit(2); }
  fwrite(p, 1, n, fp); fclose(fp);
}

static void copy_file(const std::string& from, const std::string& to) {
  FILE* a = fopen(from.c_str(), "rb"); FILE* b = fopen(to.c_str(), "wb");
  if (!a || !b) throw AvisynthError("cannot copy " + from + " to " + to);
  std::vector<char> buf(1 << 20); size_t n;
  while ((n = fread(buf.data(), 1, buf.size(), a)) > 0) fwrite(buf.data(), 1, n, b);
  fclose(a); fclose(b);
}

// A CPU-only source (not an IDeviceClip) over an AMTSRAW1 file; calls[n] counts the requests for frame n and `order`
// records them.
class CountingClip : public IClip {
  VideoInfo vi_;
  std::vector<uint8_t> data_;
  size_t fsz_ = 0;
public:
  std::vector<int> calls, order;
  explicit CountingClip(const std::string& path) {
    FILE* fp = fopen(path.c_str(), "rb");
    char magic[8]; int32_t h[6];
    if (!fp || fread(magic, 1, 8, fp) != 8 || fread(h, 4, 6, fp) != 6) throw AvisynthError("CountingClip: bad file " + path);
    vi_.width = h[0]; vi_.height = h[1]; vi_.num_frames = h[3];
    vi_.pixel_type = h[2] == 8 ? VideoInfo::CS_YV12 : VideoInfo::CS_YUV420P10;
    vi_.fps_numerator = (unsigned)h[4]; vi_.fps_denominator = (unsigned)h[5];
    fsz_ = (size_t)vi_.width * vi_.height * 3 / 2 * vi_.ComponentSize();
    data_.resize(fsz_ * vi_.num_frames);
    const bool ok = fread(data_.data(), 1, data_.size(), fp) == data_.size();
    fclose(fp);
    if (!ok) throw AvisynthError("CountingClip: truncated " + path);
    calls.assign(vi_.num_frames, 0);
  }
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    n = std::max(0, std::min(vi_.num_frames - 1, n));
    calls[n] += 1; order.push_back(n);
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

static std::string g_raw;
static PClip g_counting;                      // the CPU source CMAnalyze opened (kept alive to read its counts)

int main(int argc, char** argv) {
  if (argc < 5) { fprintf(stderr, "usage: test_logo_scan_stream <raw> <logo1.lgd> <logo2.lgd> [<more.lgd> ...] <outdir>\n"); return 2; }
  g_raw = argv[1];
  const std::string out = argv[argc - 1];
  std::vector<tstring> logos = { argv[2], out + "/does-not-exist.lgd" };
  for (int i = 3; i < argc - 1; ++i) logos.push_back(argv[i]);
  amtk_ctx* actx = nullptr;
  if (!amtk_ctx_create(0, nullptr, &actx)) { fprintf(stderr, "ctx: %s\n", amtk_last_error()); return 3; }
  int rc = 0;
  try {
    IScriptEnvironment2 env;
    BindDevice(&env, actx, DEV_TYPE_CPU);
    AvisynthPluginInit3(&env, nullptr);
    AMTContext ctx;
    for (const std::string kind : { "cpu", "dev" }) {
      // ---- LogoFrame::scanFrames / selectLogo / writeResult ----
      PClip clip;
      CountingClip* cc = nullptr;
      if (kind == "cpu") clip = PClip(cc = new CountingClip(g_raw));
      else clip = env.Invoke("AMTSource", AVSValue(std::vector<AVSValue>{ AVSValue(g_raw) })).AsClip();
      const int N = clip->GetVideoInfo().num_frames;
      logo::LogoFrame logof(ctx, logos, 0.35f);
      logof.scanFrames(clip, &env);
      logof.selectLogo();
      logof.writeResult(out + "/" + kind + "/logof.txt");
      dump(out + "/" + kind + "/eval.bin", logof.results(), sizeof(float) * 2 * logos.size() * N);
      printf("%s: best=%d ratio=%.6f", kind.c_str(), logof.getBestLogo(), logof.getLogoRatio());
      if (cc) {
        int mx = 0, zero = 0; bool in_order = (int)cc->order.size() == N;
        for (int c : cc->calls) { mx = std::max(mx, c); zero += c == 0; }
        for (size_t i = 0; in_order && i < cc->order.size(); ++i) in_order = cc->order[i] == (int)i;
        printf(" asked=%zu child_max=%d child_unasked=%d in_order=%d", cc->order.size(), mx, zero, in_order ? 1 : 0);
      }
      printf("\n");
      // ---- CMAnalyze ctor -> logoFrame (CMAnalyze.hpp:25-47,273-317): two match logos, the rest erase logos ----
      ConfigWrapper setting;
      setting.tmpDir = out + "/" + kind;
      setting.logoPath = { logos[0], logos[1] };
      setting.eraseLogoPath.assign(logos.begin() + 2, logos.end());
      copy_file(g_raw, setting.getTmpAMTSourcePath(0));
      if (kind == "cpu")                     // AMTSource replaced by the counting CPU source
        env.AddFunction("AMTSource", "s[filter]s[outqp]b", [](AVSValue, void*, IScriptEnvironment*) -> AVSValue {
          g_counting = PClip(new CountingClip(g_raw));
          return AVSValue(g_counting); }, nullptr);
      else
        env.AddFunction("AMTSource", "s[filter]s[outqp]b", av::CreateAMTSource, nullptr);
      CMAnalyze cma(ctx, setting, 0, N, &env);
      printf("%s cmanalyze: logopath=%s ratio=%.6f", kind.c_str(), cma.getLogoPath().c_str(), cma.getLogoRatio());
      if (kind == "cpu") {
        const auto* counted = static_cast<const CountingClip*>(g_counting.get());
        int mx = 0;
        for (int c : counted->calls) mx = std::max(mx, c);
        printf(" asked=%zu child_max=%d", counted->order.size(), mx);
        g_counting = nullptr;
      }
      printf("\n");
    }
  } catch (const AvisynthError& e) {
    fprintf(stderr, "AvisynthError: %s\n", e.msg.c_str()); rc = 4;
  } catch (const std::exception& e) {
    fprintf(stderr, "exception: %s\n", e.what()); rc = 5;
  }
  amtk_ctx_destroy(actx);
  printf(rc == 0 ? "OK\n" : "FAILED\n");
  return rc;
}
