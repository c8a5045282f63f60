// tests/cpp/test_tnr_widen.cpp -- the server's two lines `ConvertBits(14)` then `KTemporalNR(3, 1)` (Misc.cs:1403-1428) as
// the output pass of AMTFilterSource, on a device-resident source (one fused widening call, no widened intermediate) and
// on a CPU source; the mirror's ConvertBits on its own; AMTEraseLogo chained in place on the fused filter's IDeviceClip.
// usage: test_tnr_widen <mode> ...   (driven by tests/test_gpu_tnr_widen.py)
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

// a CPU-only source: the frames of an AMTSRAW1 file (8-bit), served as host frames; not an IDeviceClip
class HostRawClip : public IClip {
  VideoInfo vi_;
  std::vector<uint8_t> data_;
public:
  explicit HostRawClip(const std::string& path) {
    FILE* fp = fopen(path.c_str(), "rb");
    char magic[8]; int32_t h[6];
    if (!fp || fread(magic, 1, 8, fp) != 8 || fread(h, 4, 6, fp) != 6) throw AvisynthError("HostRawClip: bad file " + path);
    vi_.width = h[0]; vi_.height = h[1]; vi_.num_frames = h[3]; vi_.pixel_type = VideoInfo::CS_YV12;
    data_.resize((size_t)vi_.width * vi_.height * 3 / 2 * vi_.num_frames);
    const bool ok = fread(data_.data(), 1, data_.size(), fp) == data_.size();
    fclose(fp);
    if (!ok) throw AvisynthError("HostRawClip: truncated " + path);
  }
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    PVideoFrame f = env->NewVideoFrame(vi_);
    const uint8_t* src = data_.data() + (size_t)vi_.width * vi_.height * 3 / 2 * n;
    const int planes[3] = { PLANAR_Y, PLANAR_U, PLANAR_V };
    for (int p = 0; p < 3; ++p) {
      const int rows = f->GetHeight(planes[p]), rb = f->GetRowSize(planes[p]);
      for (int y = 0; y < rows; ++y, src += rb) memcpy(f->GetWritePtr(planes[p]) + (size_t)y * f->GetPitch(planes[p]), src, rb);
    }
    f->SetProperty("FrameType", (double)(n % 3 + 1));
    return f;
  }
  bool __stdcall GetParity(int) override { return true; }
  void __stdcall GetAudio(void*, int64_t, int64_t, IScriptEnvironment*) override {}
  int __stdcall SetCacheHints(int, int) override { return 0; }
  const VideoInfo& __stdcall GetVideoInfo() override { return vi_; }
};

static std::string g_raw;
static PClip g_convert;          // the ConvertBits filter of the last script run

static AVSValue Call(IScriptEnvironment* env, const char* name, std::vector<AVSValue> args) { return env->Invoke(name, AVSValue(args)); }

// the lines the server writes with EnableTemporalNR: ConvertBits(14) then KTemporalNR(3, 1), as the output pass
static void WidenTnrScript(IScriptEnvironment* env) {
  g_convert = Call(env, "ConvertBits", { env->GetVar("AMT_SOURCE"), AVSValue(14) }).AsClip();
  env->SetVar("last", Call(env, "KTemporalNR", { AVSValue(g_convert), AVSValue(3), AVSValue(1) }));
}
static void ConvertScript(IScriptEnvironment* env) {
  g_convert = Call(env, "ConvertBits", { env->GetVar("AMT_SOURCE"), AVSValue(14) }).AsClip();
  env->SetVar("last", AVSValue(g_convert));
}
static FilterScript CpuSourceHook(bool cpu) {           // AMTSource replaced by a CPU-frame source
  if (!cpu) return nullptr;
  return [](IScriptEnvironment* env) {
    env->AddFunction("AMTSource", "s[filter]s[outqp]b", [](AVSValue, void*, IScriptEnvironment*) -> AVSValue {
      return AVSValue(PClip(new HostRawClip(g_raw))); }, nullptr);
  };
}
static std::string Error(IScriptEnvironment* env, const char* name, std::vector<AVSValue> args) {
  try { Call(env, name, args); } catch (const AvisynthError& e) { return e.msg; }
  return "none";
}

int main(int argc, char** argv) {
  if (argc < 3) { fprintf(stderr, "usage: test_tnr_widen <mode> ...\n"); return 2; }
  const std::string mode = argv[1];
  amtk_ctx* actx = nullptr;
  if (!amtk_ctx_create(0, nullptr, &actx)) { fprintf(stderr, "ctx: %s\n", amtk_last_error()); return 3; }
  int rc = 0;
  try {
    if ((mode == "pass" || mode == "convert") && argc == 5) {     // tmpdir dev|cpu out.bin   (clip at <tmpdir>/amts0.dat)
      ConfigWrapper setting; setting.tmpDir = argv[2];
      const bool cpu = std::string(argv[3]) == "cpu";
      g_raw = setting.getTmpAMTSourcePath(0);
      AMTContext ctx;
      AMTFilterSource fs(ctx, setting, actx, 0, EncodeFileKey{ 0 }, "", mode == "pass" ? WidenTnrScript : ConvertScript, nullptr,
                         cpu ? DEV_TYPE_CPU : DEV_TYPE_CUDA, CpuSourceHook(cpu));
      PClip clip = fs.getClip();
      IScriptEnvironment* env = fs.getEnv();
      const long long l0 = amtk_ctx_launch_count(actx);
      amtk_clip dc;
      IDeviceClip* d = dynamic_cast<IDeviceClip*>(clip.get());
      const bool resident = d && d->GetDeviceClip(&dc);
      PClip cpuclip(new av::OnCPU(clip));
      std::vector<uint8_t> packed;
      int ndev = 0, types = 0;
      for (int n = 0; n < fs.getVideoInfo().num_frames; ++n) {
        PVideoFrame raw = clip->GetFrame(n, env);
        ndev += raw->IsDevice();
        types += raw->GetProperty("FrameType", 0) != 0;
        pack(cpuclip->GetFrame(n, env), packed);
      }
      const long long launches = amtk_ctx_launch_count(actx) - l0;
      printf("%s: frames=%d bits=%d resident=%d device_frames=%d typed=%d launches=%lld materialized=%d\n", mode.c_str(),
             fs.getVideoInfo().num_frames, fs.getVideoInfo().BitsPerComponent(), (int)resident, ndev, types, launches,
             (int)static_cast<av::ConvertBits*>(g_convert.get())->Materialized());
      if (mode == "convert") {
        const AVSValue none;
        printf("narrow10: %s\n", Error(env, "ConvertBits", { AVSValue(clip), AVSValue(10), none, AVSValue(0) }).c_str());
        printf("narrow8: %s\n", Error(env, "ConvertBits", { AVSValue(clip), AVSValue(8) }).c_str());
        printf("dither: %s\n", Error(env, "ConvertBits", { env->GetVar("AMT_SOURCE"), AVSValue(14), none, AVSValue(0) }).c_str());
        PClip same = Call(env, "ConvertBits", { AVSValue(clip), AVSValue(14) }).AsClip();
        IScriptEnvironment2 plugin_only;
        AvisynthPluginInit3(&plugin_only, nullptr);
        printf("same_bits_is_child=%d builtin=%d plugin_registers=%d\n", (int)(same == clip),
               (int)env->FunctionExists("ConvertBits"), (int)plugin_only.FunctionExists("ConvertBits"));
      }
      dump(argv[4], packed);
    } else if (mode == "erase" && argc == 6) {            // tmpdir logo.lgd per_frame.bin in_place.bin
      ConfigWrapper setting; setting.tmpDir = argv[2];
      AMTContext ctx;
      AMTFilterSource fs(ctx, setting, actx, 0, EncodeFileKey{ 0 }, "", WidenTnrScript);
      PClip tnr = fs.getClip();
      IScriptEnvironment* env = fs.getEnv();
      const int n = fs.getVideoInfo().num_frames;
      const std::string logo = argv[3];
      PClip ana = Call(env, "AMTAnalyzeLogo", { AVSValue(tnr), AVSValue(logo), AVSValue(35) }).AsClip();
      PClip er = Call(env, "AMTEraseLogo", { AVSValue(tnr), AVSValue(ana), AVSValue(logo), AVSValue(), AVSValue(0), AVSValue(16) }).AsClip();
      std::vector<uint8_t> per_frame, in_place;
      PClip erc(new av::OnCPU(er));
      for (int i = 0; i < n; ++i) pack(erc->GetFrame(i, env), per_frame);         // copy-on-write device frames
      dynamic_cast<logo::AMTEraseLogo*>(er.get())->EraseInPlace(0, n, env);         // one launch on the filter's HBM clip
      PClip tc(new av::OnCPU(tnr));
      for (int i = 0; i < n; ++i) pack(tc->GetFrame(i, env), in_place);
      printf("erase: frames=%d bits=%d identical=%d materialized=%d\n", n, fs.getVideoInfo().BitsPerComponent(),
             (int)(per_frame == in_place), (int)static_cast<av::ConvertBits*>(g_convert.get())->Materialized());
      dump(argv[4], per_frame);
      dump(argv[5], in_place);
    } else {
      fprintf(stderr, "unknown mode\n"); rc = 2;
    }
  } catch (const AvisynthError& e) {
    fprintf(stderr, "AvisynthError: %s\n", e.msg.c_str()); rc = 4;
  } catch (const AviSynthException& e) {
    fprintf(stderr, "AviSynthException: %s\n", e.what()); rc = 4;
  } catch (const std::exception& e) {
    fprintf(stderr, "exception: %s\n", e.what()); rc = 5;
  }
  g_convert.reset();
  amtk_ctx_destroy(actx);
  printf(rc == 0 ? "OK\n" : "FAILED\n");
  return rc;
}
