// tests/cpp/test_scan_comb_pitch.cpp -- CMAnalyze of the host-side mirror with and without its combing-stats path over
// 8- or 10-bit sources: a CPU-frame source that counts the frames it is asked for (one fused frame stream with ScanFrame's
// byte-pitch row step) and the device-resident AMTSource of the same frames (one amtk_scan_comb_frames_pitch call), next
// to AMTCombAnalyze's stats file of the same source.  The driver defines the library's stream-creating and whole-clip
// entry points itself, counting each call and passing it on to the library's, so that it can report which the mirror
// made in each run.
// usage: test_scan_comb_pitch <raw> <logo1.lgd> <logo2.lgd> [<more.lgd> ...] <outdir>
//        (driven by tests/test_gpu_scan_comb_pitch.py; <raw> is an AMTSRAW1 file of packed 4:2:0 frames at 8 or 10 bits;
//        <outdir>/{cpu,dev}/{plain,fused} must exist).  CMAnalyze matches logo1 and logo2 and erases the rest.  Writes
//        <outdir>/<kind>/plain/logof*.txt (no stats path), <outdir>/<kind>/fused/logof*.txt and combstat.txt (stats path)
//        and <outdir>/<kind>/combstat_ref.txt (AMTCombAnalyze under ReadAllFrames).  Prints one line per CMAnalyze run:
//        "<kind> <how>: logopath=.. ratio=.. [asked=..] calls=<entry>=<n>,..."
#include "../../amatsukaze_b200/host/filters.hpp"
#include <dlfcn.h>
#include <map>
#include <string>

// ---- the counted entry points -------------------------------------------------------------------------------------
static std::map<std::string, int> g_calls;

template <typename Fn> static Fn next_fn(const char* name) {
  void* p = dlsym(RTLD_NEXT, name);
  if (!p) { fprintf(stderr, "dlsym(%s) failed\n", name); abort(); }
  return reinterpret_cast<Fn>(p);
}

#define AMTK_COUNTED(ret, name, params, args)                                     \
  extern "C" ret name params {                                                    \
    g_calls[#name] += 1;                                                          \
    static ret (*fn) params = next_fn<ret (*) params>(#name);                     \
    return fn args;                                                               \
  }
AMTK_COUNTED(int, amtk_scan_comb_stream_create, (amtk_ctx* c, amtk_logo* const* l, int n, const amtk_comb_params* p, int b, amtk_scan_comb_stream** o),
             (c, l, n, p, b, o))
AMTK_COUNTED(int, amtk_scan_comb_stream_create_pitch, (amtk_ctx* c, amtk_logo* const* l, int n, const amtk_comb_params* p, int b, int r, amtk_scan_comb_stream** o),
             (c, l, n, p, b, r, o))
AMTK_COUNTED(int, amtk_logo_scan_stream_create, (amtk_ctx* c, amtk_logo* const* l, int n, int b, int r, amtk_logo_scan_stream** o),
             (c, l, n, b, r, o))
AMTK_COUNTED(int, amtk_comb_stream_create, (amtk_ctx* c, const amtk_comb_params* p, int b, amtk_comb_stream** o), (c, p, b, o))
AMTK_COUNTED(int, amtk_scan_comb_frames, (amtk_ctx* c, const amtk_clip* k, amtk_logo* const* l, int n, const amtk_comb_params* p, int f0, int nf, float* s, int32_t* cn, int d),
             (c, k, l, n, p, f0, nf, s, cn, d))
AMTK_COUNTED(int, amtk_scan_comb_frames_pitch, (amtk_ctx* c, const amtk_clip* k, amtk_logo* const* l, int n, const amtk_comb_params* p, int po, int f0, int nf, float* s, int32_t* cn, int d),
             (c, k, l, n, p, po, f0, nf, s, cn, d))
AMTK_COUNTED(int, amtk_logo_scan_frames, (amtk_ctx* c, const amtk_clip* k, amtk_logo* const* l, int n, int f0, int nf, int po, float* o, int d),
             (c, k, l, n, f0, nf, po, o, d))
AMTK_COUNTED(int, amtk_comb_frames, (amtk_ctx* c, const amtk_clip* k, const amtk_comb_params* p, int f0, int nf, int32_t* cn, int d),
             (c, k, p, f0, nf, cn, d))
#undef AMTK_COUNTED

// calls=<entry>=<n>,... (the counted entry points called since the last Calls(), by name)
static std::string Calls() {
  std::string s = "calls=";
  for (const auto& kv : g_calls) s += kv.first + "=" + std::to_string(kv.second) + ",";
  g_calls.clear();
  return s;
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

// asked=<requests> child_max=<most requests of one frame> child_unasked=<frames never asked for> in_order=<asked 0, 1, ...>
static std::string Asked(const CountingClip& cc) {
  int mx = 0, zero = 0; bool in_order = cc.order.size() == cc.calls.size();
  for (int c : cc.calls) { mx = std::max(mx, c); zero += c == 0; }
  for (size_t i = 0; in_order && i < cc.order.size(); ++i) in_order = cc.order[i] == (int)i;
  char buf[160];
  snprintf(buf, sizeof(buf), "asked=%zu child_max=%d child_unasked=%d in_order=%d", cc.order.size(), mx, zero, in_order ? 1 : 0);
  return buf;
}

static std::string g_raw;
static PClip g_counting;                      // the CPU source CMAnalyze opened (kept alive to read its counts)

int main(int argc, char** argv) {
  if (argc < 5) { fprintf(stderr, "usage: test_scan_comb_pitch <raw> <logo1.lgd> <logo2.lgd> [<more.lgd> ...] <outdir>\n"); return 2; }
  g_raw = argv[1];
  const std::string out = argv[argc - 1];
  std::vector<tstring> logos;
  for (int i = 2; i < argc - 1; ++i) logos.push_back(argv[i]);
  amtk_ctx* actx = nullptr;
  if (!amtk_ctx_create(0, nullptr, &actx)) { fprintf(stderr, "ctx: %s\n", amtk_last_error()); return 3; }
  int rc = 0;
  try {
    IScriptEnvironment2 env;
    BindDevice(&env, actx, DEV_TYPE_CPU);
    AvisynthPluginInit3(&env, nullptr);
    AMTContext ctx;
    for (const std::string kind : { "cpu", "dev" }) {
      if (kind == "cpu")                     // AMTSource replaced by the counting CPU source
        env.AddFunction("AMTSource", "s[filter]s[outqp]b", [](AVSValue, void*, IScriptEnvironment*) -> AVSValue {
          g_counting = PClip(new CountingClip(g_raw));
          return AVSValue(g_counting); }, nullptr);
      else
        env.AddFunction("AMTSource", "s[filter]s[outqp]b", av::CreateAMTSource, nullptr);
      for (const std::string how : { "plain", "fused" }) {
        ConfigWrapper setting;
        setting.tmpDir = out + "/" + kind + "/" + how;
        setting.logoPath = { logos[0], logos[1] };
        setting.eraseLogoPath.assign(logos.begin() + 2, logos.end());
        copy_file(g_raw, setting.getTmpAMTSourcePath(0));
        const int N = env.Invoke("AMTSource", AVSValue(std::vector<AVSValue>{ AVSValue(g_raw) })).AsClip()->GetVideoInfo().num_frames;
        g_counting = nullptr;
        g_calls.clear();
        CMAnalyze cma(ctx, setting, 0, N, &env, how == "fused" ? setting.tmpDir + "/combstat.txt" : tstring());
        printf("%s %s: logopath=%s ratio=%.6f", kind.c_str(), how.c_str(), cma.getLogoPath().c_str(), cma.getLogoRatio());
        if (kind == "cpu") printf(" %s", Asked(*static_cast<const CountingClip*>(g_counting.get())).c_str());
        printf(" %s\n", Calls().c_str());
        g_counting = nullptr;
      }
      // AMTCombAnalyze's stats file of the same source, pulled by ReadAllFrames (FilteredSource.hpp:417-439)
      PClip src = kind == "cpu" ? PClip(new CountingClip(g_raw))
                                : env.Invoke("AMTSource", AVSValue(std::vector<AVSValue>{ AVSValue(g_raw) })).AsClip();
      PClip comb = env.Invoke("AMTCombAnalyze", AVSValue(std::vector<AVSValue>{ AVSValue(src), AVSValue(out + "/" + kind + "/combstat_ref.txt") })).AsClip();
      ReadAllFrames(comb, &env);
    }
  } catch (const AvisynthError& e) {
    fprintf(stderr, "AvisynthError: %s\n", e.msg.c_str()); rc = 4;
  } catch (const std::exception& e) {
    fprintf(stderr, "exception: %s\n", e.what()); rc = 5;
  }
  g_counting = nullptr;
  amtk_ctx_destroy(actx);
  printf(rc == 0 ? "OK\n" : "FAILED\n");
  return rc;
}
