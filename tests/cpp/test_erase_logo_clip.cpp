// tests/cpp/test_erase_logo_clip.cpp -- AMTEraseLogo of the host-side mirror over a device-resident child: MakeSource's chain
// AMTEraseLogo(AMTAnalyzeLogo(src, logo), logo, logof, maxfade) over an AMTSource, served from one amtk_erase_logo_clip
// call, against the same chain served by the per-frame path (an analyze clip over a second AMTSource of the same file) and
// by the frame stream (a CPU source); EraseInPlace over its own chain and over the per-frame composition; KTemporalNR over
// the resident eraser.
// usage: test_erase_logo_clip <raw> <logo.lgd> <logof|-> <maxfade> <outdir>   (driven by tests/test_gpu_erase_logo_clip_filter.py)
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
static std::vector<uint8_t> packAll(PClip c, IScriptEnvironment* env) {
  PClip cpu(new av::OnCPU(c));
  std::vector<uint8_t> v;
  for (int n = 0; n < c->GetVideoInfo().num_frames; ++n) pack(cpu->GetFrame(n, env), v);
  return v;
}

// A CPU-only source (not an IDeviceClip) over an AMTSRAW1 file of packed 4:2:0 pictures at 8 bits.
class CpuClip : public IClip {
  VideoInfo vi_;
  std::vector<uint8_t> data_;
  size_t fsz_ = 0;
public:
  explicit CpuClip(const std::string& path) {
    FILE* fp = fopen(path.c_str(), "rb");
    char magic[8]; int32_t h[6];
    if (!fp || fread(magic, 1, 8, fp) != 8 || fread(h, 4, 6, fp) != 6 || h[2] != 8) throw AvisynthError("CpuClip: bad file " + path);
    vi_.width = h[0]; vi_.height = h[1]; vi_.num_frames = h[3]; vi_.pixel_type = VideoInfo::CS_YV12;
    fsz_ = (size_t)vi_.width * vi_.height * 3 / 2;
    data_.resize(fsz_ * vi_.num_frames);
    const bool ok = fread(data_.data(), 1, data_.size(), fp) == data_.size();
    fclose(fp);
    if (!ok) throw AvisynthError("CpuClip: truncated " + path);
  }
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    n = std::max(0, std::min(vi_.num_frames - 1, n));
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

// AMTEraseLogo(AMTAnalyzeLogo(analysed, logo), logo, logof, maxfade) over `src`
static PClip Eraser(IScriptEnvironment* env, PClip src, PClip analysed, const std::string& lg, const std::string& logof, int maxfade) {
  PClip ana = Call(env, "AMTAnalyzeLogo", { AVSValue(analysed), AVSValue(lg), AVSValue(35) }).AsClip();
  return Call(env, "AMTEraseLogo", { AVSValue(src), AVSValue(ana), AVSValue(lg), logof.empty() ? AVSValue() : AVSValue(logof),
                                     AVSValue(0), AVSValue(maxfade) }).AsClip();
}
static logo::AMTEraseLogo* AsEraser(PClip c) { return dynamic_cast<logo::AMTEraseLogo*>(c.get()); }
static bool IsResident(PClip c) { amtk_clip dc; IDeviceClip* d = dynamic_cast<IDeviceClip*>(c.get()); return d && d->GetDeviceClip(&dc); }

int main(int argc, char** argv) {
  if (argc != 6) { fprintf(stderr, "usage: test_erase_logo_clip <raw> <logo.lgd> <logof|-> <maxfade> <outdir>\n"); return 2; }
  amtk_ctx* actx = nullptr;
  if (!amtk_ctx_create(0, nullptr, &actx)) { fprintf(stderr, "ctx: %s\n", amtk_last_error()); return 3; }
  int rc = 0;
  try {
    const std::string raw = argv[1], lg = argv[2], logof = std::string(argv[3]) == "-" ? "" : argv[3], out = argv[5];
    const int maxfade = atoi(argv[4]);
    IScriptEnvironment2 envObj; IScriptEnvironment* env = &envObj;
    BindDevice(env, actx, DEV_TYPE_CPU);
    av::AddBuiltins(env);
    AvisynthPluginInit3(env, nullptr);
    auto source = [&]() { return Call(env, "AMTSource", { AVSValue(raw) }).AsClip(); };
    // the resident chain: one out-of-place call, the source untouched
    PClip src = source();
    const std::vector<uint8_t> before = packAll(src, env);
    PClip er = Eraser(env, src, src, lg, logof, maxfade);
    const int N = er->GetVideoInfo().num_frames;
    const long long l0 = amtk_ctx_launch_count(actx);
    const std::vector<uint8_t> resident = packAll(er, env);
    const long long launches = amtk_ctx_launch_count(actx) - l0;
    std::vector<float> fades((size_t)N * 2), pfades((size_t)N * 2);
    for (int n = 0; n < N; ++n) AsEraser(er)->GetFades(n, fades[2 * n], fades[2 * n + 1], env);
    // the per-frame path: the analyze clip reads a second AMTSource of the same file
    PClip src2 = source(), src2b = source();
    PClip per = Eraser(env, src2, src2b, lg, logof, maxfade);
    const std::vector<uint8_t> per_frame = packAll(per, env);
    for (int n = 0; n < N; ++n) AsEraser(per)->GetFades(n, pfades[2 * n], pfades[2 * n + 1], env);
    // the frame stream over a CPU source
    PClip cpu(new CpuClip(raw));
    PClip st = Eraser(env, cpu, cpu, lg, logof, maxfade);
    const std::vector<uint8_t> stream = packAll(st, env);
    // EraseInPlace over its own chain (one call) and over the per-frame composition
    PClip src3 = source(), src4 = source(), src4b = source();
    AsEraser(Eraser(env, src3, src3, lg, logof, maxfade))->EraseInPlace(0, N, env);
    AsEraser(Eraser(env, src4, src4b, lg, logof, maxfade))->EraseInPlace(0, N, env);
    dynamic_cast<av::AMTSource*>(src3.get())->SyncHostFromDevice(env);
    dynamic_cast<av::AMTSource*>(src4.get())->SyncHostFromDevice(env);
    const std::vector<uint8_t> in_place = packAll(src3, env), in_place_per_frame = packAll(src4, env);
    // KTemporalNR over the resident eraser (its one-call path) and over the per-frame eraser (its host path)
    PClip tnr = Call(env, "KTemporalNR", { AVSValue(er), AVSValue(3), AVSValue(1), AVSValue(false) }).AsClip();
    PClip tnr_per = Call(env, "KTemporalNR", { AVSValue(per), AVSValue(3), AVSValue(1), AVSValue(false) }).AsClip();
    const std::vector<uint8_t> t1 = packAll(tnr, env), t2 = packAll(tnr_per, env);
    // device frames for a CUDA consumer
    IScriptEnvironment2 denvObj; IScriptEnvironment* denv = &denvObj;
    BindDevice(denv, actx, DEV_TYPE_CUDA);
    av::AddBuiltins(denv);
    AvisynthPluginInit3(denv, nullptr);
    PClip dsrc = Call(denv, "AMTSource", { AVSValue(raw) }).AsClip();
    PClip der = Eraser(denv, dsrc, dsrc, lg, logof, maxfade);
    int ndev = 0;
    for (int n = 0; n < N; ++n) ndev += der->GetFrame(n, denv)->IsDevice();
    const std::vector<uint8_t> dev_frames = packAll(der, denv);
    printf("erase_clip: frames=%d resident=%d per_frame_resident=%d launches=%lld device_frames=%d\n", N, (int)IsResident(er),
           (int)IsResident(per), launches, ndev);
    printf("identical: per_frame=%d stream=%d fades=%d source_untouched=%d in_place=%d in_place_per_frame=%d tnr=%d "
           "tnr_resident=%d device=%d\n",
           (int)(resident == per_frame), (int)(resident == stream), (int)(memcmp(fades.data(), pfades.data(), fades.size() * 4) == 0),
           (int)(packAll(src, env) == before), (int)(in_place == resident), (int)(in_place_per_frame == resident), (int)(t1 == t2),
           (int)IsResident(tnr), (int)(dev_frames == resident));
    dump(out + "/resident.bin", resident);
    FILE* fp = fopen((out + "/fades.bin").c_str(), "wb");
    fwrite(fades.data(), 4, fades.size(), fp); fclose(fp);
  } catch (const AvisynthError& e) {
    fprintf(stderr, "AvisynthError: %s\n", e.msg.c_str()); rc = 4;
  } catch (const std::exception& e) {
    fprintf(stderr, "exception: %s\n", e.what()); rc = 5;
  }
  amtk_ctx_destroy(actx);
  printf(rc == 0 ? "OK\n" : "FAILED\n");
  return rc;
}
