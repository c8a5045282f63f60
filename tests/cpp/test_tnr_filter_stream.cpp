// tests/cpp/test_tnr_filter_stream.cpp -- KTemporalNR of the host-side mirror over a child that is not device resident:
// the frame stream for in-order reads, the gather for the others, and ConvertBits(14) fused into the stream, on a host
// clip that counts the GetFrame calls it receives per frame.
// usage: test_tnr_filter_stream <mode> ...   (driven by tests/test_gpu_tnr_filter_stream.py and
//                                            tools/bench_tnr_filter_stream.py)
#include "../../amatsukaze_b200/host/filters.hpp"
#include <dlfcn.h>
#include <malloc.h>
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

// A CPU-only source (not an IDeviceClip): num_frames frames, frame n being picture n % P of an AMTSRAW1 file of P packed
// 4:2:0 pictures at 8, 10, 12 or 14 bits.  Every frame carries SourceFrame = n; calls[n] counts the requests for frame n.
class CountingClip : public IClip {
  VideoInfo vi_;
  std::vector<uint8_t> data_;
  int pictures_ = 0;
  size_t fsz_ = 0;
public:
  std::vector<int> calls;
  CountingClip(const std::string& path, int num_frames) {
    FILE* fp = fopen(path.c_str(), "rb");
    char magic[8]; int32_t h[6];
    if (!fp || fread(magic, 1, 8, fp) != 8 || fread(h, 4, 6, fp) != 6) throw AvisynthError("CountingClip: bad file " + path);
    vi_.width = h[0]; vi_.height = h[1]; pictures_ = h[3];
    vi_.pixel_type = h[2] == 8 ? VideoInfo::CS_YV12 : h[2] == 10 ? VideoInfo::CS_YUV420P10 : h[2] == 12 ? VideoInfo::CS_YUV420P12 : VideoInfo::CS_YUV420P14;
    vi_.num_frames = num_frames > 0 ? num_frames : pictures_;
    fsz_ = (size_t)vi_.width * vi_.height * 3 / 2 * vi_.ComponentSize();
    data_.resize(fsz_ * pictures_);
    const bool ok = fread(data_.data(), 1, data_.size(), fp) == data_.size();
    fclose(fp);
    if (!ok) throw AvisynthError("CountingClip: truncated " + path);
    calls.assign(vi_.num_frames, 0);
  }
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    n = std::max(0, std::min(vi_.num_frames - 1, n));
    calls[n] += 1;
    PVideoFrame f = env->NewVideoFrame(vi_);
    const uint8_t* src = data_.data() + fsz_ * (size_t)(n % pictures_);
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

static AVSValue Call(IScriptEnvironment* env, const char* name, std::vector<AVSValue> args) { return env->Invoke(name, AVSValue(args)); }

// [ConvertBits(widen) then] KTemporalNR(d, t, interlaced) over `src`
static PClip Tnr(IScriptEnvironment* env, PClip src, int widen, int d, int t, bool il, PClip* convert) {
  PClip c = widen ? Call(env, "ConvertBits", { AVSValue(src), AVSValue(widen) }).AsClip() : src;
  if (convert) *convert = widen ? c : nullptr;
  return Call(env, "KTemporalNR", { AVSValue(c), AVSValue(d), AVSValue(t), AVSValue(il) }).AsClip();
}

static std::string Counters(const CountingClip& cc, const PClip& tnr, const PClip& convert) {
  const auto* k = dynamic_cast<const KTemporalNR*>(tnr.get());
  const auto* cb = dynamic_cast<const av::ConvertBits*>(convert.get());
  int mx = 0, total = 0, zero = 0;
  for (int c : cc.calls) { mx = std::max(mx, c); total += c; zero += c == 0; }
  char buf[256];
  snprintf(buf, sizeof(buf), "sent=%d gathered=%d host_widened=%d child_max=%d child_total=%d child_unasked=%d",
           k->FramesSent(), k->FramesGathered(), cb ? cb->HostWidenedFrames() : 0, mx, total, zero);
  return buf;
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

// free device memory through the driver API (the library's context is current on this thread after its calls)
static size_t DeviceFree() {
  typedef int (*MemGetInfo)(size_t*, size_t*);
  static MemGetInfo fn = nullptr;
  if (!fn) {
    void* h = dlopen("libcuda.so.1", RTLD_NOW);
    fn = h ? reinterpret_cast<MemGetInfo>(dlsym(h, "cuMemGetInfo_v2")) : nullptr;
    if (!fn) throw AvisynthError("cuMemGetInfo_v2 not found");
  }
  size_t f = 0, t = 0;
  if (fn(&f, &t) != 0) throw AvisynthError("cuMemGetInfo_v2 failed");
  return f;
}

static double Now() { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec + 1e-9 * t.tv_nsec; }

static std::string g_raw;
static int g_frames = 0, g_widen = 0;
static PClip g_source, g_convert;

static void OutputScript(IScriptEnvironment* env) {       // the server's lines as the output pass
  env->SetVar("last", AVSValue(Tnr(env, env->GetVar("AMT_SOURCE").AsClip(), g_widen, 3, 1, false, &g_convert)));
}
static void CpuSourceHook(IScriptEnvironment* env) {      // AMTSource replaced by the counting CPU source
  env->AddFunction("AMTSource", "s[filter]s[outqp]b", [](AVSValue, void*, IScriptEnvironment*) -> AVSValue {
    g_source = PClip(new CountingClip(g_raw, g_frames));
    return AVSValue(g_source); }, nullptr);
}

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: test_tnr_filter_stream <mode> ...\n"); return 2; }
  const std::string mode = argv[1];
  amtk_ctx* actx = nullptr;
  if (!amtk_ctx_create(0, nullptr, &actx)) { fprintf(stderr, "ctx: %s\n", amtk_last_error()); return 3; }
  int rc = 0;
  try {
    if (mode == "order" && argc == 9) {            // raw widen d t interlaced orders.bin out.bin
      // orders.bin: int32 frame numbers, patterns separated by -1; each pattern is served by a new filter over a new clip
      IScriptEnvironment2 env;
      BindDevice(&env, actx, DEV_TYPE_CPU);
      av::AddBuiltins(&env);
      AvisynthPluginInit3(&env, nullptr);
      const std::vector<int> all = ReadOrder(argv[7]);
      std::vector<uint8_t> packed;
      int k = 0;
      for (size_t i = 0; i < all.size(); ++k) {
        std::vector<int> order;
        for (; i < all.size() && all[i] >= 0; ++i) order.push_back(all[i]);
        ++i;
        auto* cc = new CountingClip(argv[2], 0);
        PClip src(cc), convert;
        PClip tnr = Tnr(&env, src, atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]) != 0, &convert);
        int typed = 0;
        for (int n : order) {
          PVideoFrame f = tnr->GetFrame(n, &env);
          if (f->IsDevice()) throw AvisynthError("a device frame from a host child");
          typed += f->GetProperty("SourceFrame", -1) == n;
          pack(f, packed);
        }
        printf("order %d: reads=%zu bits=%d typed=%d %s\n", k, order.size(), tnr->GetVideoInfo().BitsPerComponent(), typed,
               Counters(*cc, tnr, convert).c_str());
      }
      dump(argv[8], packed);
    } else if (mode == "pass" && argc == 4) {      // tmpdir out.bin: ConvertBits(14) + KTemporalNR(3, 1) on a CPU source
      ConfigWrapper setting; setting.tmpDir = argv[2];
      g_raw = setting.getTmpAMTSourcePath(0); g_frames = 0; g_widen = 14;
      AMTContext ctx;
      AMTFilterSource fs(ctx, setting, actx, 0, EncodeFileKey{ 0 }, "", OutputScript, nullptr, DEV_TYPE_CPU, CpuSourceHook);
      PClip clip = fs.getClip();
      IScriptEnvironment* env = fs.getEnv();
      PClip cpuclip(new av::OnCPU(clip));
      std::vector<uint8_t> packed;
      int ndev = 0, typed = 0;
      long long h2d_max = 0;
      for (int n = 0; n < fs.getVideoInfo().num_frames; ++n) {     // as the existing drivers read: twice per frame
        PVideoFrame raw = clip->GetFrame(n, env);
        h2d_max = std::max<long long>(h2d_max, amtk_ctx_last_h2d_bytes(actx));
        ndev += raw->IsDevice();
        typed += raw->GetProperty("SourceFrame", -1) == n;
        pack(cpuclip->GetFrame(n, env), packed);
      }
      printf("pass: frames=%d bits=%d device_frames=%d typed=%d h2d_max=%lld %s\n", fs.getVideoInfo().num_frames,
             fs.getVideoInfo().BitsPerComponent(), ndev, typed, h2d_max,
             Counters(*static_cast<CountingClip*>(g_source.get()), clip, g_convert).c_str());
      dump(argv[3], packed);
    } else if (mode == "release" && argc == 3) {   // raw: filters destroyed mid-clip, 40 times
      IScriptEnvironment2 env;
      BindDevice(&env, actx, DEV_TYPE_CPU);
      av::AddBuiltins(&env);
      AvisynthPluginInit3(&env, nullptr);
      size_t live = 0;
      auto one = [&](int k) {
        PClip src(new CountingClip(argv[2], 40));
        PClip tnr = Tnr(&env, src, 14, 3, 1, false, nullptr);
        for (int n = 0; n < 20 + k % 7; ++n) tnr->GetFrame(n, &env);
        live = DeviceFree();
      };                                           // the filter goes here: ring and batches in flight, outputs pending
      one(0);
      amtk_ctx_synchronize(actx);
      const size_t free0 = DeviceFree();
      for (int k = 0; k < 40; ++k) one(k);
      amtk_ctx_synchronize(actx);
      const size_t free1 = DeviceFree();
      printf("release: free0=%zu live=%zu free1=%zu\n", free0, live, free1);
    } else if (mode == "bench" && argc == 10) {    // tmpdir frames widen fwd|rev count dump.bin n1,n2,... pool|fresh
      // pool: freed frames are reused by malloc (as AviSynth+ reuses frames from its cache) instead of being returned to
      // the kernel and faulted in again, zeroed, on the next allocation
      if (std::string(argv[9]) == "pool") { mallopt(M_MMAP_THRESHOLD, 32 << 20); mallopt(M_TRIM_THRESHOLD, 1 << 30); }
      ConfigWrapper setting; setting.tmpDir = argv[2];
      g_raw = setting.getTmpAMTSourcePath(0); g_frames = atoi(argv[3]); g_widen = atoi(argv[4]);
      const bool rev = std::string(argv[5]) == "rev";
      const int count = atoi(argv[6]);
      std::vector<int> keep;
      for (char* p = argv[8]; *p;) { keep.push_back((int)strtol(p, &p, 10)); if (*p == ',') ++p; }
      AMTContext ctx;
      AMTFilterSource fs(ctx, setting, actx, 0, EncodeFileKey{ 0 }, "", OutputScript, nullptr, DEV_TYPE_CPU, CpuSourceHook);
      PClip clip = fs.getClip();
      IScriptEnvironment* env = fs.getEnv();
      const int N = fs.getVideoInfo().num_frames;
      std::vector<PVideoFrame> kept;
      const double t0 = Now();                      // every GetFrame ends in a synchronous receive or copy
      for (int i = 0; i < count; ++i) {
        const int n = rev ? N - 1 - i : i;
        PVideoFrame f = clip->GetFrame(n, env);
        if (std::find(keep.begin(), keep.end(), n) != keep.end()) kept.push_back(f);
      }
      const double dt = Now() - t0;
      const std::string counters = Counters(*static_cast<CountingClip*>(g_source.get()), clip, g_convert);
      const double t1 = Now();                      // the CPU source alone, the same frames in the same order
      for (int i = 0; i < count; ++i) g_source->GetFrame(rev ? N - 1 - i : i, env);
      const double ds = Now() - t1;
      std::vector<uint8_t> packed;                  // in the order read
      for (const auto& f : kept) pack(f, packed);
      printf("bench: frames=%d bits=%d seconds=%.6f fps=%.2f source_seconds=%.6f h2d_last=%lld %s\n", count,
             fs.getVideoInfo().BitsPerComponent(), dt, count / dt, ds, (long long)amtk_ctx_last_h2d_bytes(actx), counters.c_str());
      dump(argv[7], packed);
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
  g_source.reset(); g_convert.reset();
  amtk_ctx_destroy(actx);
  printf(rc == 0 ? "OK\n" : "FAILED\n");
  return rc;
}
