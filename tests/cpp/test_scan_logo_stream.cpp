// tests/cpp/test_scan_logo_stream.cpp -- logo::LogoAnalyzer of the host-side mirror over a CPU-frame source that records
// the frames it is asked for, and over a device-resident source holding the same frames.
// usage: test_scan_logo_stream <raw> <imgx> <imgy> <w> <h> <thy> <max_frames> <service_id> <out_cpu.lgd> <out_dev.lgd>
//        (driven by tests/test_gpu_scan_logo_stream.py; <raw> is an AMTSRAW1 file of packed 8-bit 4:2:0 frames)
#include "../../amatsukaze_b200/host/filters.hpp"
#include <string>

struct RawFrames {
  VideoInfo vi;
  std::vector<uint8_t> data;
  size_t fsz = 0;
  explicit RawFrames(const std::string& path) {
    FILE* fp = fopen(path.c_str(), "rb");
    char magic[8]; int32_t h[6];
    if (!fp || fread(magic, 1, 8, fp) != 8 || fread(h, 4, 6, fp) != 6 || h[2] != 8) throw AvisynthError("RawFrames: bad file " + path);
    vi.width = h[0]; vi.height = h[1]; vi.num_frames = h[3]; vi.pixel_type = VideoInfo::CS_YV12;
    fsz = (size_t)vi.width * vi.height * 3 / 2;
    data.resize(fsz * vi.num_frames);
    const bool ok = fread(data.data(), 1, data.size(), fp) == data.size();
    fclose(fp);
    if (!ok) throw AvisynthError("RawFrames: truncated " + path);
  }
};

// CPU frames; `asked` lists the requests in order.
class RecordingClip : public IClip {
  const RawFrames& raw_;
public:
  std::vector<int> asked;
  explicit RecordingClip(const RawFrames& raw) : raw_(raw) {}
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    asked.push_back(n);
    PVideoFrame f = env->NewVideoFrame(raw_.vi);
    const uint8_t* src = raw_.data.data() + raw_.fsz * (size_t)n;
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
  const VideoInfo& __stdcall GetVideoInfo() override { return raw_.vi; }
};

// The same frames resident in HBM (packed 4:2:0), handed out through IDeviceClip.
class ResidentClip : public IClip, public IDeviceClip {
  const RawFrames& raw_;
  amtk_ctx* ctx_;
  void* mem_ = nullptr;
public:
  int frames_asked = 0;
  ResidentClip(const RawFrames& raw, amtk_ctx* ctx) : raw_(raw), ctx_(ctx) {
    if (!amtk_device_alloc(ctx, raw.data.size(), &mem_) || !amtk_memcpy_h2d(ctx, mem_, raw.data.data(), raw.data.size()))
      throw AvisynthError(amtk_last_error());
  }
  ~ResidentClip() { amtk_device_free(ctx_, mem_); }
  bool GetDeviceClip(amtk_clip* out) override { *out = PackedDeviceClip(raw_.vi, mem_); return true; }
  PVideoFrame __stdcall GetFrame(int, IScriptEnvironment*) override { ++frames_asked; throw AvisynthError("ResidentClip: GetFrame"); }
  bool __stdcall GetParity(int) override { return true; }
  void __stdcall GetAudio(void*, int64_t, int64_t, IScriptEnvironment*) override {}
  int __stdcall SetCacheHints(int, int) override { return 0; }
  const VideoInfo& __stdcall GetVideoInfo() override { return raw_.vi; }
};

int main(int argc, char** argv) {
  if (argc != 11) { fprintf(stderr, "usage: test_scan_logo_stream <raw> <imgx> <imgy> <w> <h> <thy> <max_frames> <service_id> <cpu.lgd> <dev.lgd>\n"); return 2; }
  amtk_ctx* actx = nullptr;
  if (!amtk_ctx_create(0, nullptr, &actx)) { fprintf(stderr, "ctx: %s\n", amtk_last_error()); return 3; }
  int rc = 0;
  try {
    const RawFrames raw(argv[1]);
    const int imgx = atoi(argv[2]), imgy = atoi(argv[3]), w = atoi(argv[4]), h = atoi(argv[5]), thy = atoi(argv[6]);
    const int maxf = atoi(argv[7]), sid = atoi(argv[8]);
    IScriptEnvironment2 env;
    BindDevice(&env, actx, DEV_TYPE_CPU);
    AMTContext actxlog;
    {
      auto* rc_clip = new RecordingClip(raw);
      PClip src(rc_clip);
      logo::LogoAnalyzer analyzer(actxlog, imgx, imgy, w, h, thy, maxf, nullptr);
      analyzer.ScanLogo(src, sid, argv[9], &env);
      bool in_order = true;
      for (size_t i = 0; i < rc_clip->asked.size(); ++i) in_order = in_order && rc_clip->asked[i] == (int)i;
      printf("cpu: asked=%zu in_order=%d\n", rc_clip->asked.size(), in_order ? 1 : 0);
    }
    {
      auto* dev_clip = new ResidentClip(raw, actx);
      PClip src(dev_clip);
      logo::LogoAnalyzer analyzer(actxlog, imgx, imgy, w, h, thy, maxf, nullptr);
      analyzer.ScanLogo(src, sid, argv[10], &env);
      printf("device: frames_asked=%d\n", dev_clip->frames_asked);
    }
  } catch (const AvisynthError& e) {
    fprintf(stderr, "error: %s\n", e.msg.c_str());
    rc = 1;
  }
  amtk_ctx_destroy(actx);
  return rc;
}
