// tests/cpp/test_comb_stream.cpp -- AMTCombAnalyze of the host-side mirror over a CPU-frame source that counts the frames
// it is asked for (the frame stream) and over the device-resident AMTSource of the same frames (one launch), alone and as
// KFM pass 1 under AMTFilterSource.
// usage: test_comb_stream filter <raw> <outdir>         (<outdir>/cpu and <outdir>/dev must exist)
//        test_comb_stream passes <tmpdir> <vfr|cfr> <cpu|dev>   (the clip at <tmpdir>/amts0.dat)
//        (driven by tests/test_gpu_comb_stream_filter.py; <raw> is an AMTSRAW1 file of packed 4:2:0 frames at 8 or 10 bits)
#include "../../amatsukaze_b200/host/filters.hpp"
#include <string>

static void dump(const std::string& path, const std::vector<int32_t>& v) {
  FILE* fp = fopen(path.c_str(), "wb");
  if (!fp) { fprintf(stderr, "cannot write %s\n", path.c_str()); exit(2); }
  fwrite(v.data(), sizeof(int32_t), v.size(), fp); fclose(fp);
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
    f->SetProperty("SourceFrame", (double)n);
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
static std::vector<PClip> g_sources;          // the CPU sources the passes opened, in order

static void CpuSourceHook(IScriptEnvironment* env) {      // AMTSource replaced by the counting CPU source
  env->AddFunction("AMTSource", "s[filter]s[outqp]b", [](AVSValue, void*, IScriptEnvironment*) -> AVSValue {
    g_sources.push_back(PClip(new CountingClip(g_raw)));
    return AVSValue(g_sources.back()); }, nullptr);
}

int main(int argc, char** argv) {
  if (argc < 4) { fprintf(stderr, "usage: test_comb_stream filter <raw> <outdir> | passes <tmpdir> <vfr|cfr> <cpu|dev>\n"); return 2; }
  const std::string mode = argv[1];
  amtk_ctx* actx = nullptr;
  if (!amtk_ctx_create(0, nullptr, &actx)) { fprintf(stderr, "ctx: %s\n", amtk_last_error()); return 3; }
  int rc = 0;
  try {
    if (mode == "filter" && argc == 4) {
      g_raw = argv[2];
      const std::string out = argv[3];
      IScriptEnvironment2 env;
      BindDevice(&env, actx, DEV_TYPE_CPU);
      AvisynthPluginInit3(&env, nullptr);
      for (const std::string kind : { "cpu", "dev" }) {
        // ReadAllFrames over KFMDeint pass 1 (FilteredSource.hpp:417-439)
        CountingClip* cc = nullptr;
        PClip src = kind == "cpu" ? PClip(cc = new CountingClip(g_raw))
                                  : env.Invoke("AMTSource", AVSValue(std::vector<AVSValue>{ AVSValue(g_raw) })).AsClip();
        const int N = src->GetVideoInfo().num_frames;
        PClip comb = env.Invoke("AMTCombAnalyze", AVSValue(std::vector<AVSValue>{ AVSValue(src), AVSValue(out + "/" + kind + "/combstat.txt") })).AsClip();
        int same = 0;
        for (int i = 0; i < N; ++i) {
          PVideoFrame f = comb->GetFrame(i, &env);
          if (cc) same += f->GetProperty("SourceFrame", -1) == i;
        }
        printf("%s:", kind.c_str());
        if (cc) printf(" %s frames_returned=%d", Asked(*cc).c_str(), same);
        printf("\n");
        if (!cc) continue;
        // Counts() after a partial pull, and after an out-of-order GetFrame first
        for (const std::string how : { "partial", "seek" }) {
          auto* c2 = new CountingClip(g_raw);
          PClip s2(c2);
          auto* a = new AMTCombAnalyze(s2, "", &env);
          PClip hold(a);
          PVideoFrame f;
          if (how == "partial") for (int i = 0; i < N / 3; ++i) f = a->GetFrame(i, &env);
          else f = a->GetFrame(N / 2, &env);
          const int got = (int)f->GetProperty("SourceFrame", -1);
          dump(out + "/cpu/counts_" + how + ".bin", a->Counts(&env));
          printf("%s: %s returned=%d\n", how.c_str(), Asked(*c2).c_str(), got);
        }
      }
    } else if (mode == "passes" && argc == 5) {
      ConfigWrapper setting; setting.tmpDir = argv[2];
      g_raw = setting.getTmpAMTSourcePath(0);
      const bool cpu = std::string(argv[4]) == "cpu";
      AMTContext ctx;
      AMTFilterSource fs(ctx, setting, actx, 0, EncodeFileKey{ 0 }, "", std::string(argv[3]) == "cfr" ? KFMCfrScript : KFMVfrScript,
                         nullptr, cpu ? DEV_TYPE_CPU : DEV_TYPE_CUDA, cpu ? FilterScript(CpuSourceHook) : FilterScript());
      printf("passes: preproc=%zu out_frames=%d timecodes=%zu\n", fs.getPasses().size(), fs.getVideoInfo().num_frames, fs.getTimeCodes().size());
      if (cpu) printf("pass0: %s\n", Asked(*static_cast<const CountingClip*>(g_sources.at(0).get())).c_str());
      g_sources.clear();
    } else {
      fprintf(stderr, "unknown mode\n"); rc = 2;
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
