// tests/cpp/test_scan_logo_stream_deep.cpp -- logo::LogoAnalyzer of the host-side mirror on 10- and 12-bit sources: a
// YUV420P10/P12 av::AMTSource (device resident) and a CPU-frame source that records the frames it is asked for, both over
// the same decoded pictures.
// usage: test_scan_logo_stream_deep <raw> <imgx> <imgy> <w> <h> <thy> <max_frames> <service_id> <out_cpu.lgd> <out_src.lgd>
//        (driven by tests/test_gpu_logoscan_2byte.py; <raw> is an AMTSRAW1 file of packed 10- or 12-bit 4:2:0 frames)
#include "../../amatsukaze_b200/host/filters.hpp"
#include <string>

struct RawFrames {
  VideoInfo vi;
  std::vector<uint8_t> data;
  size_t fsz = 0;
  explicit RawFrames(const std::string& path) {
    FILE* fp = fopen(path.c_str(), "rb");
    char magic[8]; int32_t h[6];
    if (!fp || fread(magic, 1, 8, fp) != 8 || fread(h, 4, 6, fp) != 6 || (h[2] != 10 && h[2] != 12)) throw AvisynthError("RawFrames: bad file " + path);
    vi.width = h[0]; vi.height = h[1]; vi.num_frames = h[3];
    vi.pixel_type = h[2] == 10 ? VideoInfo::CS_YUV420P10 : VideoInfo::CS_YUV420P12;
    fsz = (size_t)vi.width * vi.height * 3 / 2 * 2;
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

int main(int argc, char** argv) {
  if (argc != 11) { fprintf(stderr, "usage: test_scan_logo_stream_deep <raw> <imgx> <imgy> <w> <h> <thy> <max_frames> <service_id> <cpu.lgd> <src.lgd>\n"); return 2; }
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
      auto* source = new av::AMTSource(argv[1], &env);
      PClip src(source);
      amtk_clip dc;
      printf("source: bits=%d resident=%d\n", src->GetVideoInfo().BitsPerComponent(), source->GetDeviceClip(&dc) ? 1 : 0);
      logo::LogoAnalyzer analyzer(actxlog, imgx, imgy, w, h, thy, maxf, nullptr);
      analyzer.ScanLogo(src, sid, argv[10], &env);
    }
  } catch (const AvisynthError& e) {
    fprintf(stderr, "error: %s\n", e.msg.c_str());
    rc = 1;
  }
  amtk_ctx_destroy(actx);
  return rc;
}
