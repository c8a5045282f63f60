// filters.hpp -- host-side (C++) mirror of the reference's filter / in-process interface for the hot path, written
// against avs_compat.h and calling the CUDA library ONLY through the C ABI (include/amtk_b200.h).
//
//   av::AMTSource          frame provider behind IClip::GetFrame           (reference AMTSource.hpp:721-830,873-882)
//   logo::AMTAnalyzeLogo   8 x LogoAnalyzeFrame{p,t,b} per output frame    (reference LogoScan.hpp:1100-1236)
//   logo::AMTEraseLogo     CalcFade / CalcFade2 / Delogo                   (reference LogoScan.hpp:1238-1519)
//   logo::LogoFrame        scanFrames / selectLogo / writeResult           (reference LogoScan.hpp:1521-1836;
//                                                                            the CMAnalyze entry, CMAnalyze.hpp:291-311)
//   logo::LogoAnalyzer     ScanLogo over a clip read frame by frame        (reference LogoScan.hpp:794-1080)
//   AMTCombAnalyze + ReadAllFrames   the telecine pre-pass pull loop       (reference FilteredSource.hpp:417-439,519-544;
//                                                                            the arithmetic lives in the external KFM plugin)
//   KTemporalNR            the reference's TemporalNRFilter under the plugin filter's name (reference VideoFilter.hpp:27-212;
//                                                                            the server's script line, Misc.cs:1403-1428)
//   av::ConvertBits        AviSynth+'s built-in ConvertBits, widening only, as a built-in of the mirror environment
//                                                                            (AddBuiltins; the line before KTemporalNR)
//   AvisynthPluginInit3    registration with the reference's names/arg specs (reference Amatsukaze.cpp:43-66)
//
// Same names, argument meaning and error behaviour as the reference; the bodies are new: frames live in HBM, every
// per-pixel loop is a CUDA kernel, and whole-clip passes are single batched calls instead of per-frame loops.
#pragma once
#include <algorithm>
#include <cmath>
#include <ctime>
#include <deque>
#include <memory>
#include <mutex>
#include <numeric>
#include <regex>
#include <stdexcept>
#include "avs_compat.h"
#include "../../include/amtk_b200.h"

// ---------------------------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------------------------
typedef std::string tstring;

struct AMTContext {                                      // logging subset of StreamUtils.hpp:343-511
  bool quiet = true;
  void infoF(const char* fmt, ...) const { if (quiet) return; va_list ap; va_start(ap, fmt); fprintf(stderr, "AMT [info] "); vfprintf(stderr, fmt, ap); fputc('\n', stderr); va_end(ap); }
  void debugF(const char* fmt, ...) const { if (quiet) return; va_list ap; va_start(ap, fmt); fprintf(stderr, "AMT [debug] "); vfprintf(stderr, fmt, ap); fputc('\n', stderr); va_end(ap); }
  void info(const char* s) const { if (!quiet) fprintf(stderr, "AMT [info] %s\n", s); }
};

struct IOException : std::runtime_error { using std::runtime_error::runtime_error; };

inline void amtk_check(int ok, IScriptEnvironment* env) {      // C-ABI failure -> AvisynthError, like env->ThrowError
  if (!ok) env->ThrowError("%s", amtk_last_error());
}
inline int nblocks(int n, int block) { return (n + block - 1) / block; }

// A clip whose frames are resident in HBM can hand filters a descriptor for batched processing.
class IDeviceClip {
public:
  virtual ~IDeviceClip() {}
  virtual bool GetDeviceClip(amtk_clip* out) = 0;
};

inline amtk_clip HostFrameClip(const PVideoFrame& f, const VideoInfo& vi) {     // one frame (CPU, or a device view) as a 1-frame clip
  amtk_clip c; memset(&c, 0, sizeof(c));
  c.base = f->Base(); c.frame_stride = (int64_t)((f->TotalBytes() + 15) & ~(size_t)15);
  c.off_u = (int64_t)f->GetOffset(PLANAR_U); c.off_v = (int64_t)f->GetOffset(PLANAR_V);
  c.width = vi.width; c.height = vi.height; c.pitch_y = f->GetPitch(PLANAR_Y); c.pitch_uv = f->GetPitch(PLANAR_U);
  c.log_uvx = c.log_uvy = 1; c.bytes_per_sample = vi.ComponentSize(); c.bits_per_sample = vi.BitsPerComponent();
  c.num_frames = 1; c.on_device = f->IsDevice() ? 1 : 0;
  return c;
}

// A clip of tightly packed 4:2:0 frames (Y, U, V back to back) at `base` in HBM.
inline amtk_clip PackedDeviceClip(const VideoInfo& vi, void* base) {
  const size_t ysz = (size_t)vi.width * vi.height * vi.ComponentSize(), csz = (size_t)(vi.width / 2) * (vi.height / 2) * vi.ComponentSize();
  amtk_clip c; memset(&c, 0, sizeof(c));
  c.base = base; c.frame_stride = (int64_t)(ysz + 2 * csz); c.off_u = (int64_t)ysz; c.off_v = (int64_t)(ysz + csz);
  c.width = vi.width; c.height = vi.height; c.pitch_y = vi.width * vi.ComponentSize(); c.pitch_uv = (vi.width / 2) * vi.ComponentSize();
  c.log_uvx = c.log_uvy = 1; c.bytes_per_sample = vi.ComponentSize(); c.bits_per_sample = vi.BitsPerComponent();
  c.num_frames = vi.num_frames; c.on_device = 1;
  return c;
}

// Frame n of a PackedDeviceClip owned by `mem`: a zero-copy view for a CUDA consumer (AviSynthNeo device frame), a CPU
// copy otherwise.
inline PVideoFrame PackedDeviceFrame(const VideoInfo& vi, const std::shared_ptr<void>& mem, int n, IScriptEnvironment* env) {
  const amtk_clip c = PackedDeviceClip(vi, mem.get());
  const size_t fsz = (size_t)c.frame_stride;
  const uint8_t* base = static_cast<const uint8_t*>(mem.get()) + fsz * n;
  if (env->GetDeviceType() == DEV_TYPE_CUDA) {
    const size_t off[3] = { 0, (size_t)c.off_u, (size_t)c.off_v };
    const int pitch[3] = { c.pitch_y, c.pitch_uv, c.pitch_uv };
    return std::make_shared<VideoFrame>(vi, const_cast<uint8_t*>(base), fsz, off, pitch, mem);
  }
  std::vector<uint8_t> tmp(fsz);
  amtk_check(amtk_memcpy_d2h(env->GetAmtkContext(), tmp.data(), base, tmp.size()), env);
  PVideoFrame f = env->NewVideoFrame(vi);
  const int planes[3] = { PLANAR_Y, PLANAR_U, PLANAR_V };
  size_t off = 0;
  for (int p = 0; p < 3; ++p) {
    const int rows = f->GetHeight(planes[p]), rb = f->GetRowSize(planes[p]);
    for (int y = 0; y < rows; ++y) memcpy(f->GetWritePtr(planes[p]) + (size_t)y * f->GetPitch(planes[p]), tmp.data() + off + (size_t)y * rb, rb);
    off += (size_t)rows * rb;
  }
  return f;
}

// Binds a script environment to a device context: frames made writable on the device get a private HBM copy.
inline void BindDevice(IScriptEnvironment* env, amtk_ctx* ctx, AvsDeviceType consumer = DEV_TYPE_CPU) {
  env->SetAmtkContext(ctx);
  env->SetDeviceType(consumer);
  env->MakeWritableDevice = [env, ctx](PVideoFrame* pvf) -> bool {
    const PVideoFrame& f = *pvf;
    void* p = nullptr;
    if (!amtk_device_alloc(ctx, f->TotalBytes(), &p)) env->ThrowError("%s", amtk_last_error());
    std::shared_ptr<void> own(p, [ctx](void* q) { amtk_device_free(ctx, q); });
    if (!amtk_memcpy_d2d(ctx, p, f->Base(), f->TotalBytes())) env->ThrowError("%s", amtk_last_error());
    PVideoFrame w = std::make_shared<VideoFrame>(*f);     // copies geometry + properties, then re-points at the new memory
    w->Rebase(static_cast<uint8_t*>(p), own);
    *pvf = w;
    return true;
  };
}

namespace av {

// Picture structure of a decoded frame (StreamUtils.hpp:577-586) and the source-frame list built from it
// (StreamReform.hpp:145-154,874-904): which decoded picture feeds which OUTPUT frame, and whether the output frame is
// half a frame period late (bottom-field-first pictures), in which case its top field comes from the PREVIOUS decoded
// picture (AMTSource.hpp:524-551 OnFrameDecoded).
enum PICTURE_TYPE { PIC_FRAME = 0, PIC_FRAME_DOUBLING, PIC_FRAME_TRIPLING, PIC_TFF, PIC_BFF, PIC_TFF_RFF, PIC_BFF_RFF, MAX_PIC_TYPE };

struct FilterSourceFrame {
  bool halfDelay;
  int decoded;               // index of the decoded picture (the reference keys this by framePTS)
  double pts;                // in frame periods (the reference: 90 kHz clock)
};

inline std::vector<FilterSourceFrame> MakeFilterSourceFrames(const std::vector<uint8_t>& pics) {   // StreamReform.hpp:874-904
  std::vector<FilterSourceFrame> list;
  for (int d = 0; d < (int)pics.size(); ++d) {
    FilterSourceFrame f{ false, d, (double)list.size() };
    switch (pics[d]) {
      case PIC_FRAME: case PIC_TFF: case PIC_TFF_RFF: list.push_back(f); break;
      case PIC_FRAME_DOUBLING: list.push_back(f); f.pts += 1; list.push_back(f); break;
      case PIC_FRAME_TRIPLING: list.push_back(f); f.pts += 1; list.push_back(f); f.pts += 1; list.push_back(f); break;
      case PIC_BFF: f.halfDelay = true; f.pts -= 0.5; list.push_back(f); break;
      case PIC_BFF_RFF: f.halfDelay = true; f.pts -= 0.5; list.push_back(f); f.halfDelay = false; f.pts += 1; list.push_back(f); break;
      default: list.push_back(f); break;
    }
  }
  return list;
}

// Field plan of every output frame: (top, bottom) decoded-picture indices, exactly what OnFrameDecoded + GetFrame produce
// (AMTSource.hpp:524-551,721-780): no delay -> MakeFrame(cur, cur); halfDelay -> MakeFrame(prev, cur) when the previous
// decoded picture exists, otherwise no frame is made and GetFrame serves the next cached frame (ForceGetFrame's
// lower_bound, :567-577) -- an output frame without its own picture takes the plan of the next one that has.
inline void MakeFieldPlan(const std::vector<FilterSourceFrame>& frames, std::vector<int32_t>& top, std::vector<int32_t>& bottom) {
  const int n = (int)frames.size();
  top.assign(n, -1); bottom.assign(n, -1);
  for (int k = 0; k < n; ++k) {
    const int d = frames[k].decoded;
    if (!frames[k].halfDelay) { top[k] = bottom[k] = d; }
    else if (d > 0) { top[k] = d - 1; bottom[k] = d; }
  }
  int next_t = -1, next_b = -1;
  for (int k = n - 1; k >= 0; --k) {                       // ForceGetFrame: first cached frame at or after k ...
    if (top[k] >= 0) { next_t = top[k]; next_b = bottom[k]; }
    else { top[k] = next_t; bottom[k] = next_b; }
  }
  for (int k = 0; k < n; ++k)                               // ... or, past the last one, the last cached frame
    if (top[k] < 0) { top[k] = k ? top[k - 1] : 0; bottom[k] = k ? bottom[k - 1] : 0; }
}

// ---------------------------------------------------------------------------------------------------------------
// AMTSource: frame provider.  The reference decodes MPEG2/H.264 with FFmpeg into CPU frames on demand
// (AMTSource.hpp:585-780); decode is out of scope here, so the source is a file of DECODED pictures (the stand-in for the
// `amts%d.dat` artefact, AMTSource.hpp:835-871) that is uploaded ONCE and stays resident in HBM.  Everything after the
// decoder is reproduced: the picture-structure -> source-frame list, the half-delay field weave (MergeField on the
// device, amtk_weave_frames), NV12 chroma split, the FrameType frame property, GetParity, MT mode.
//   "AMTSRAW1" + int32 {width,height,bits,num_frames,fps_num,fps_den} + planar 4:2:0 frames            (all PIC_FRAME)
//   "AMTSRAW2" + the same six int32 + int32 {nv12} + num x {uint8 pic_struct, uint8 pict_type} + decoded pictures
// ---------------------------------------------------------------------------------------------------------------
class AMTSource : public IClip, public IDeviceClip {
  VideoInfo vi;
  amtk_ctx* ctx;
  std::vector<uint8_t> host;          // CPU copy of the OUTPUT frames, made lazily (only CPU consumers need it)
  bool host_valid = false;
  std::shared_ptr<void> dev;          // HBM: output frames (what filters read)
  std::vector<uint8_t> pict_type;     // per OUTPUT frame: AV_PICTURE_TYPE of the picture that supplies its top field
  std::vector<FilterSourceFrame> frames_;
  bool interlaced = true;
  size_t ysz() const { return (size_t)vi.width * vi.height * vi.ComponentSize(); }
  size_t csz() const { return (size_t)(vi.width / 2) * (vi.height / 2) * vi.ComponentSize(); }
  size_t fsz() const { return ysz() + 2 * csz(); }
  static std::shared_ptr<void> DevAlloc(amtk_ctx* ctx, size_t bytes, IScriptEnvironment* env) {
    void* p = nullptr;
    amtk_check(amtk_device_alloc(ctx, bytes, &p), env);
    return std::shared_ptr<void>(p, [ctx](void* q) { amtk_device_free(ctx, q); });
  }
  amtk_clip Desc(void* base, int nframes, bool nv12 = false) const {
    amtk_clip c; memset(&c, 0, sizeof(c));
    c.base = base; c.frame_stride = (int64_t)fsz(); c.off_u = (int64_t)ysz(); c.off_v = (int64_t)(ysz() + csz());
    c.width = vi.width; c.height = vi.height; c.pitch_y = vi.width * vi.ComponentSize();
    c.pitch_uv = (nv12 ? vi.width : vi.width / 2) * vi.ComponentSize();
    c.log_uvx = c.log_uvy = 1; c.bytes_per_sample = vi.ComponentSize(); c.bits_per_sample = vi.BitsPerComponent();
    c.num_frames = nframes; c.on_device = 1;
    return c;
  }
  void EnsureHost(IScriptEnvironment* env) {
    if (host_valid) return;
    host.resize(fsz() * vi.num_frames);
    amtk_check(amtk_memcpy_d2h(ctx, host.data(), dev.get(), host.size()), env);
    host_valid = true;
  }
public:
  AMTSource(const tstring& path, IScriptEnvironment* env) : ctx(env->GetAmtkContext()) {
    FILE* fp = fopen(path.c_str(), "rb");
    if (!fp) env->ThrowError("AMTSource: failed to open %s", path.c_str());
    char magic[8]; int32_t h[6]; int32_t nv12 = 0;
    if (fread(magic, 1, 8, fp) != 8 || (memcmp(magic, "AMTSRAW1", 8) != 0 && memcmp(magic, "AMTSRAW2", 8) != 0) || fread(h, 4, 6, fp) != 6) {
      fclose(fp); env->ThrowError("AMTSource: bad header in %s", path.c_str());
    }
    const bool v2 = magic[7] == '2';
    const int ndec = h[3];
    vi.width = h[0]; vi.height = h[1]; vi.fps_numerator = (unsigned)h[4]; vi.fps_denominator = (unsigned)h[5];
    switch (h[2]) {                                       // AMTSource.hpp:428-442
      case 8: vi.pixel_type = VideoInfo::CS_YV12; break;
      case 10: vi.pixel_type = VideoInfo::CS_YUV420P10; break;
      case 12: vi.pixel_type = VideoInfo::CS_YUV420P12; break;
      default: fclose(fp); env->ThrowError("AMTSource: unsupported bit depth %d", h[2]);
    }
    std::vector<uint8_t> pics((size_t)ndec, (uint8_t)PIC_FRAME), ptype((size_t)ndec, 1);
    if (v2) {
      std::vector<uint8_t> meta((size_t)ndec * 2);
      if (fread(&nv12, 4, 1, fp) != 1 || fread(meta.data(), 1, meta.size(), fp) != meta.size()) { fclose(fp); env->ThrowError("AMTSource: truncated file %s", path.c_str()); }
      for (int d = 0; d < ndec; ++d) { pics[d] = meta[2 * d]; ptype[d] = meta[2 * d + 1]; if (pics[d] >= MAX_PIC_TYPE) { fclose(fp); env->ThrowError("AMTSource: bad picture structure"); } }
    }
    if (!ctx) { fclose(fp); env->ThrowError("AMTSource: no device bound to the script environment"); }
    // decoded pictures: pinned staging -> HBM
    const size_t dec_bytes = fsz() * (size_t)ndec;
    void* pinned = nullptr;
    amtk_check(amtk_host_alloc(std::max<size_t>(dec_bytes, 16), &pinned), env);
    const bool ok = fread(pinned, 1, dec_bytes, fp) == dec_bytes;
    fclose(fp);
    if (!ok) { amtk_host_free(pinned); env->ThrowError("AMTSource: truncated file %s", path.c_str()); }
    std::shared_ptr<void> decoded = DevAlloc(ctx, std::max<size_t>(dec_bytes, 16), env);
    const int up = amtk_memcpy_h2d(ctx, decoded.get(), pinned, dec_bytes);
    amtk_host_free(pinned);
    amtk_check(up, env);
    frames_ = MakeFilterSourceFrames(pics);
    vi.num_frames = (int)frames_.size();
    std::vector<int32_t> top, bottom;
    MakeFieldPlan(frames_, top, bottom);
    bool identity = !nv12 && vi.num_frames == ndec;
    for (int k = 0; k < vi.num_frames && identity; ++k) identity = top[k] == k && bottom[k] == k;
    if (identity) dev = decoded;                          // progressive / TFF material: the decoded pictures ARE the frames
    else {                                                // MakeFrame for every output frame, on the device (AMTSource.hpp:357-366)
      dev = DevAlloc(ctx, fsz() * (size_t)vi.num_frames, env);
      const amtk_clip src = Desc(decoded.get(), ndec, nv12 != 0), dst = Desc(dev.get(), vi.num_frames);
      amtk_check(amtk_weave_frames(ctx, &src, &dst, 0, top.data(), bottom.data(), vi.num_frames, nv12 != 0), env);
    }
    pict_type.resize(vi.num_frames);
    for (int k = 0; k < vi.num_frames; ++k) pict_type[k] = ptype[top[k]];          // ret->SetProperty("FrameType", top->pict_type) :369
  }

  const std::vector<FilterSourceFrame>& SourceFrames() const { return frames_; }

  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    n = std::max(0, std::min(vi.num_frames - 1, n));
    PVideoFrame f;
    if (env->GetDeviceType() == DEV_TYPE_CUDA) {          // zero-copy view of the resident frame (AviSynthNeo device frame)
      const size_t off[3] = { 0, ysz(), ysz() + csz() };
      const int pitch[3] = { vi.width * vi.ComponentSize(), (vi.width / 2) * vi.ComponentSize(), (vi.width / 2) * vi.ComponentSize() };
      f = std::make_shared<VideoFrame>(vi, static_cast<uint8_t*>(dev.get()) + fsz() * n, fsz(), off, pitch, dev);
    } else {
      EnsureHost(env);
      f = env->NewVideoFrame(vi);
      const uint8_t* src = host.data() + fsz() * n;
      const int planes[3] = { PLANAR_Y, PLANAR_U, PLANAR_V };
      size_t off = 0;
      for (int p = 0; p < 3; ++p) {
        const int rows = f->GetHeight(planes[p]), rb = f->GetRowSize(planes[p]);
        for (int y = 0; y < rows; ++y) memcpy(f->GetWritePtr(planes[p]) + (size_t)y * f->GetPitch(planes[p]), src + off + (size_t)y * rb, rb);
        off += (size_t)rows * rb;
      }
    }
    f->SetProperty("FrameType", (double)pict_type[n]);
    return f;
  }
  bool GetDeviceClip(amtk_clip* c) override { *c = Desc(dev.get(), vi.num_frames); return true; }
  // device frames edited in place by a batched filter become visible to CPU GetFrame after this
  void SyncHostFromDevice(IScriptEnvironment*) { host_valid = false; }
  void __stdcall GetAudio(void*, int64_t, int64_t, IScriptEnvironment*) override {}
  const VideoInfo& __stdcall GetVideoInfo() override { return vi; }
  bool __stdcall GetParity(int) override { return interlaced; }                         // AMTSource.hpp:821-823
  int __stdcall SetCacheHints(int cachehints, int) override {                             // :825-830 + Neo device hooks
    if (cachehints == CACHE_GET_MTMODE) return MT_NICE_FILTER;
    if (cachehints == CACHE_GET_DEV_TYPE) return DEV_TYPE_CPU | DEV_TYPE_CUDA;
    return 0;
  }
};

inline AVSValue __cdecl CreateAMTSource(AVSValue args, void*, IScriptEnvironment* env) {     // AMTSource.hpp:873-882
  // [filter]s [outqp]b are decode options: ignored.  A clip already opened by an earlier pass of the same job is shared.
  const std::string path = args[0].AsString();
  if (auto* shared = env->SharedClips()) {
    auto it = shared->find("AMTSource:" + path);
    if (it != shared->end()) return AVSValue(it->second);
    PClip c(new AMTSource(path, env));
    (*shared)["AMTSource:" + path] = c;
    return AVSValue(c);
  }
  return AVSValue(PClip(new AMTSource(path, env)));
}

// OnCPU (AviSynthNeo): downloads device frames so that a CPU consumer can read them.
class OnCPU : public GenericVideoFilter {
public:
  explicit OnCPU(PClip c) : GenericVideoFilter(c) {}
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    PVideoFrame f = child->GetFrame(n, env);
    if (!f->IsDevice()) return f;
    PVideoFrame h = env->NewVideoFrame(vi);
    std::vector<uint8_t> tmp(f->TotalBytes());
    amtk_check(amtk_memcpy_d2h(env->GetAmtkContext(), tmp.data(), f->Base(), tmp.size()), env);
    const int planes[3] = { PLANAR_Y, PLANAR_U, PLANAR_V };
    for (int p = 0; p < 3; ++p)
      for (int y = 0; y < h->GetHeight(planes[p]); ++y)
        memcpy(h->GetWritePtr(planes[p]) + (size_t)y * h->GetPitch(planes[p]),
               tmp.data() + f->GetOffset(planes[p]) + (size_t)y * f->GetPitch(planes[p]), h->GetRowSize(planes[p]));
    h->CopyPropertiesFrom(*f);
    return h;
  }
  int __stdcall SetCacheHints(int cachehints, int) override {
    if (cachehints == CACHE_GET_MTMODE) return MT_NICE_FILTER;
    if (cachehints == CACHE_GET_DEV_TYPE) return DEV_TYPE_CPU;
    if (cachehints == CACHE_GET_CHILD_DEV_TYPE) return DEV_TYPE_CUDA | DEV_TYPE_CPU;
    return 0;
  }
};

// ConvertBits (AviSynth+ built-in) stand-in, widening only.  The server writes ConvertBits(14) before KTemporalNR
// (Misc.cs:1403-1428) on a limited-range YUV clip (AMTSource sets no _ColorRange, the line passes no fulls), for which
// AviSynth+ widens by a left shift of k = bits - source bits on every plane.  That shift is AviSynth+'s arithmetic, not
// code in the reference tree.  Narrowing is AviSynth+'s dither arithmetic, which is not in the reference, so it throws.
// It is a built-in of the mirror environment (AddBuiltins), the way OnCPU stands in for AviSynthNeo's, and is never
// registered by AvisynthPluginInit3: the real plugin must not shadow AviSynth+'s own ConvertBits.
//  - device-resident child: an IDeviceClip; the widened clip is made in HBM by one amtk_tnr_frames call at d = 0 (exactly
//    the shift) when a consumer first asks for it.  KTemporalNR over it filters the child with one widening call instead,
//    so on that path the widened clip is never made;
//  - any other child: each frame is widened on the host when a consumer asks for it.  KTemporalNR over it reads the
//    child's frames instead and widens inside its own calls, so on that path no frame is widened on the host.
class ConvertBits : public GenericVideoFilter, public IDeviceClip {
  amtk_ctx* ctx;
  int shift;
  std::shared_ptr<void> dev;          // widened clip in HBM, made on first use (device-resident child only)
  int host_widened = 0;               // frames widened on the host
  bool Resident() {
    if (dev) return true;
    amtk_clip src;
    if (!SourceDeviceClip(&src)) return false;
    void* p = nullptr;
    const amtk_clip probe = PackedDeviceClip(vi, nullptr);
    if (!amtk_device_alloc(ctx, (size_t)probe.frame_stride * vi.num_frames, &p)) throw AvisynthError(amtk_last_error());
    amtk_ctx* c = ctx;
    std::shared_ptr<void> own(p, [c](void* q) { amtk_device_free(c, q); });
    const amtk_clip out = PackedDeviceClip(vi, p);
    amtk_tnr_params prm{ 0, 0, 0 };                       // d = 0: every frame is its own window, the output is src << k
    if (!amtk_tnr_frames(ctx, &src, &out, 0, &prm, 0, vi.num_frames)) throw AvisynthError(amtk_last_error());
    dev = own;
    return true;
  }
  PVideoFrame HostWidened(int n, IScriptEnvironment* env) {
    PVideoFrame s = child->GetFrame(n, env);
    if (s->IsDevice()) env->ThrowError("ConvertBits: device frames of a clip that is not device resident are not provided");
    PVideoFrame d = env->NewVideoFrame(vi);
    const bool wide = child->GetVideoInfo().ComponentSize() == 2;
    const int planes[3] = { PLANAR_Y, PLANAR_U, PLANAR_V };
    for (int p = 0; p < 3; ++p)
      for (int y = 0; y < d->GetHeight(planes[p]); ++y) {
        const uint8_t* sr = s->GetReadPtr(planes[p]) + (size_t)y * s->GetPitch(planes[p]);
        uint16_t* dr = reinterpret_cast<uint16_t*>(d->GetWritePtr(planes[p]) + (size_t)y * d->GetPitch(planes[p]));
        const int w = d->GetRowSize(planes[p]) / 2;
        for (int x = 0; x < w; ++x) dr[x] = (uint16_t)((wide ? reinterpret_cast<const uint16_t*>(sr)[x] : sr[x]) << shift);
      }
    d->CopyPropertiesFrom(*s);
    ++host_widened;
    return d;
  }
public:
  ConvertBits(PClip clip, int bits, IScriptEnvironment* env) : GenericVideoFilter(clip), ctx(env->GetAmtkContext()) {
    shift = bits - vi.BitsPerComponent();
    switch (bits) {
      case 10: vi.pixel_type = VideoInfo::CS_YUV420P10; break;
      case 12: vi.pixel_type = VideoInfo::CS_YUV420P12; break;
      case 14: vi.pixel_type = VideoInfo::CS_YUV420P14; break;
      default: vi.pixel_type = VideoInfo::CS_YUV420P16; break;
    }
  }
  // the child's device clip, not widened (KTemporalNR widens inside its own call); false when the child is not resident
  bool SourceDeviceClip(amtk_clip* c) {
    IDeviceClip* d = dynamic_cast<IDeviceClip*>(child.get());
    return d && d->GetDeviceClip(c);
  }
  const PClip& Child() const { return child; }
  bool Materialized() const { return dev != nullptr; }
  int HostWidenedFrames() const { return host_widened; }
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    n = std::max(0, std::min(vi.num_frames - 1, n));
    if (!Resident()) return HostWidened(n, env);
    PVideoFrame f = PackedDeviceFrame(vi, dev, n, env);
    f->CopyPropertiesFrom(*child->GetFrame(n, env));
    return f;
  }
  bool GetDeviceClip(amtk_clip* c) override {
    if (!Resident()) return false;
    *c = PackedDeviceClip(vi, dev.get());
    return true;
  }
  int __stdcall SetCacheHints(int cachehints, int) override {
    if (cachehints == CACHE_GET_MTMODE) return MT_NICE_FILTER;
    if (cachehints == CACHE_GET_DEV_TYPE) return DEV_TYPE_CPU | DEV_TYPE_CUDA;
    return 0;
  }
  // AviSynth+'s spec: ConvertBits(clip, int bits, bool truerange, int dither, int dither_bits, bool fulls, bool fulld)
  static constexpr const char* kParams = "c[bits]i[truerange]b[dither]i[dither_bits]i[fulls]b[fulld]b";
  static AVSValue __cdecl Create(AVSValue args, void*, IScriptEnvironment* env) {
    PClip clip = args[0].AsClip();
    const VideoInfo& svi = clip->GetVideoInfo();
    const int bits = args[1].AsInt(svi.BitsPerComponent()), from = svi.BitsPerComponent();
    if (!svi.IsPlanar()) env->ThrowError("ConvertBits: only 4:2:0 YUV clips are provided");
    if (bits < from || args[3].Defined() || args[4].Defined())
      env->ThrowError("ConvertBits: only widening is provided; narrowing is AviSynth+'s dither arithmetic, which is not in the reference");
    if (args[2].Defined() || args[5].Defined() || args[6].Defined())
      env->ThrowError("ConvertBits: only the limited-range widening is provided (no truerange, fulls or fulld)");
    if (bits != 10 && bits != 12 && bits != 14 && bits != 16 && bits != from) env->ThrowError("ConvertBits: bits must be 10, 12, 14 or 16");
    if (bits == from) return AVSValue(clip);                // AviSynth+ returns the clip itself
    if (!env->GetAmtkContext()) env->ThrowError("ConvertBits: no device bound to the script environment");
    return AVSValue(PClip(new ConvertBits(clip, bits, env)));
  }
};

// The functions the mirror environment provides itself, as AviSynth+ does, rather than the plugin.
inline void AddBuiltins(IScriptEnvironment* env) {
  env->AddFunction("ConvertBits", ConvertBits::kParams, ConvertBits::Create, 0);
}

}  // namespace av

namespace logo {

struct LogoAnalyzeFrame { float p[11], t[11], b[11]; };              // LogoScan.hpp:1100-1103
static_assert(sizeof(LogoAnalyzeFrame) == 132, "LogoAnalyzeFrame layout");

struct LogoHandle {                                                     // RAII over amtk_logo
  amtk_logo* h = nullptr;
  LogoHandle() {}
  explicit LogoHandle(amtk_logo* p) : h(p) {}
  LogoHandle(LogoHandle&& o) : h(o.h) { o.h = nullptr; }
  LogoHandle& operator=(LogoHandle&& o) { if (this != &o) { reset(); h = o.h; o.h = nullptr; } return *this; }
  ~LogoHandle() { reset(); }
  void reset() { if (h) amtk_logo_destroy(h); h = nullptr; }
  bool valid() const { return h != nullptr; }
};

// ---------------------------------------------------------------------------------------------------------------
// AMTAnalyzeLogo (LogoScan.hpp:1106-1236)
// ---------------------------------------------------------------------------------------------------------------
class AMTAnalyzeLogo : public GenericVideoFilter {
  VideoInfo srcvi;
  LogoHandle logo, deintLogo, fieldLogoT, fieldLogoB;
  float maskratio;
  tstring logoPath;
public:
  AMTAnalyzeLogo(PClip clip, const tstring& logoPath, float maskratio, IScriptEnvironment* env)
      : GenericVideoFilter(clip), srcvi(vi), maskratio(maskratio), logoPath(logoPath) {
    amtk_logo* p = nullptr;
    if (!amtk_logo_load(env->GetAmtkContext(), logoPath.c_str(), &p, nullptr))
      env->ThrowError("Failed to read logo file (%s)", logoPath.c_str());                 // :1173-1175
    logo = LogoHandle(p);
    amtk_check(amtk_logo_deint(logo.h, &p), env); deintLogo = LogoHandle(p);             // :1177-1180
    amtk_check(amtk_logo_create_mask(deintLogo.h, maskratio), env);
    amtk_check(amtk_logo_field(logo.h, 0, &p), env); fieldLogoT = LogoHandle(p);         // :1182-1185
    amtk_check(amtk_logo_create_mask(fieldLogoT.h, maskratio), env);
    amtk_check(amtk_logo_field(logo.h, 1, &p), env); fieldLogoB = LogoHandle(p);
    amtk_check(amtk_logo_create_mask(fieldLogoB.h, maskratio), env);
    const int out_bytes = (int)sizeof(LogoAnalyzeFrame) * 8;                              // :1195-1200
    vi.pixel_type = VideoInfo::CS_BGR32;
    vi.width = 64;
    vi.height = nblocks(out_bytes, vi.width * 4);
    vi.num_frames = nblocks(vi.num_frames, 8);
  }

  // records of SOURCE frames [first, first+count) (count <= srcvi.num_frames - first), batched on the device
  void AnalyzeSourceFrames(int first, int count, LogoAnalyzeFrame* out, IScriptEnvironment* env) {
    amtk_ctx* ctx = env->GetAmtkContext();
    amtk_clip dc;
    IDeviceClip* d = dynamic_cast<IDeviceClip*>(child.get());
    if (d && d->GetDeviceClip(&dc)) {       // HBM-resident source: one batched call, results returned to the host
      amtk_check(amtk_logo_analyze_frames(ctx, &dc, deintLogo.h, fieldLogoT.h, fieldLogoB.h, first, count,
                                          reinterpret_cast<float*>(out), 0), env);
      return;
    }
    for (int i = 0; i < count; ++i) {                                                      // any other IClip: frame by frame
      PVideoFrame f = child->GetFrame(first + i, env);
      amtk_clip hc = HostFrameClip(f, srcvi);
      amtk_check(amtk_logo_analyze_frames(ctx, &hc, deintLogo.h, fieldLogoT.h, fieldLogoB.h, 0, 1, reinterpret_cast<float*>(out + i), 0), env);
    }
  }

  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    const int pixelSize = srcvi.ComponentSize();
    if (pixelSize != 1 && pixelSize != 2) env->ThrowError("[AMTAnalyzeLogo] Unsupported pixel format");   // :1213-1215
    PVideoFrame dst = env->NewVideoFrame(vi);
    LogoAnalyzeFrame* pDst = reinterpret_cast<LogoAnalyzeFrame*>(dst->GetWritePtr());
    const int first = std::min(srcvi.num_frames - 1, n * 8);
    const int count = std::max(1, std::min(8, srcvi.num_frames - n * 8));
    AnalyzeSourceFrames(first, count, pDst, env);
    for (int i = count; i < 8; ++i) pDst[i] = pDst[count - 1];        // nsrc clamps to the last source frame (:1133)
    return dst;
  }
  int __stdcall SetCacheHints(int cachehints, int) override { return cachehints == CACHE_GET_MTMODE ? MT_NICE_FILTER : 0; }   // :1220-1225
  // what AMTEraseLogo's frame stream needs to recognise the MakeSource chain
  const PClip& Source() const { return child; }
  const tstring& LogoPath() const { return logoPath; }
  float MaskRatio() const { return maskratio; }

  static AVSValue __cdecl Create(AVSValue args, void*, IScriptEnvironment* env) {         // :1227-1235
    return AVSValue(PClip(new AMTAnalyzeLogo(args[0].AsClip(), args[1].AsString(), (float)args[2].AsFloat(35) / 100.0f, env)));
  }
};

// ---------------------------------------------------------------------------------------------------------------
// AMTEraseLogo (LogoScan.hpp:1238-1519)
// ---------------------------------------------------------------------------------------------------------------
// The MakeSource chain AMTEraseLogo(AMTAnalyzeLogo(child, logo), logo, ...) in mode 0 is served by the library, which
// computes the analyze records itself; the analyze clip is then never asked for a frame:
//  - device-resident child (IDeviceClip): on first use the whole clip is erased into the filter's own HBM clip by ONE
//    amtk_erase_logo_clip call (DESIGN.md section 3.3.4), out of place, so the child (shared across passes) stays as it
//    is.  Frames are served as device views (CUDA consumer) or copies (CPU consumer), GetFades from that call's fades, and
//    the filter is an IDeviceClip itself, so KTemporalNR, AMTCombAnalyze and LogoFrame downstream take their one-call
//    resident paths;
//  - any other child: in-order reads are served from a frame stream (amtk_erase_logo_stream, DESIGN.md section 3.3.2):
//    each child frame is asked for once, in order; any other read drops the stream and takes the per-frame path below.
// Any other analyze clip, or mode != 0, takes the per-frame path.
class AMTEraseLogo : public GenericVideoFilter, public IDeviceClip {
  PClip analyzeclip;
  std::vector<int> frameResult;
  LogoHandle logo;
  int mode, maxFadeLength;
  std::string lastDebugLabel;
  tstring logoPath;
  // frame stream state, guarded by streamMu (GetFrame may come from several threads: MT_NICE_FILTER)
  static constexpr int kStreamBatch = 16;
  struct StreamRelease { void operator()(amtk_erase_logo_stream* s) const { amtk_erase_logo_stream_destroy(s); } };
  std::mutex streamMu;
  int streamable = -1;                      // -1: not decided yet
  std::unique_ptr<amtk_erase_logo_stream, StreamRelease> stream;
  std::deque<PVideoFrame> held;             // frames sent and not yet served, oldest first (output streamNext first)
  int streamNext = 0, streamSent = 0;
  int lastServed = -1; PVideoFrame lastFrame;
  int framesSent = 0, streamsStarted = 0;
  // resident path state, guarded by devMu
  amtk_ctx* actx;
  std::mutex devMu;
  std::shared_ptr<void> dev;                // the erased clip in HBM
  amtk_clip out;                            // ... and its descriptor
  std::vector<float> devFades;              // [N][2] fades of that call

  // mode 0 over AMTAnalyzeLogo(child, the same logo): the records are the library's own to compute
  bool OwnChain() const {
    const AMTAnalyzeLogo* a = dynamic_cast<const AMTAnalyzeLogo*>(analyzeclip.get());
    return mode == 0 && a && a->Source().get() == child.get() && a->LogoPath() == logoPath;
  }
  float MaskRatio() const { return dynamic_cast<const AMTAnalyzeLogo*>(analyzeclip.get())->MaskRatio(); }
  bool ChildDeviceClip(amtk_clip* dc) {
    IDeviceClip* d = dynamic_cast<IDeviceClip*>(child.get());
    return d && d->GetDeviceClip(dc);
  }
  // erases the whole device-resident child into the filter's HBM clip once; false when this is not such a chain
  bool Resident() {
    std::lock_guard<std::mutex> lock(devMu);
    if (dev) return true;
    amtk_clip src;
    if (!OwnChain() || !ChildDeviceClip(&src)) return false;
    auto check = [](int ok) { if (!ok) throw AvisynthError(amtk_last_error()); };
    void* p = nullptr;
    check(amtk_device_alloc(actx, (size_t)PackedDeviceClip(vi, nullptr).frame_stride * vi.num_frames, &p));
    amtk_ctx* c = actx;
    std::shared_ptr<void> own(p, [c](void* q) { amtk_device_free(c, q); });
    out = PackedDeviceClip(vi, p);
    std::vector<uint8_t> fr(frameResult.begin(), frameResult.end());
    std::vector<float> fades((size_t)vi.num_frames * 2);
    check(amtk_erase_logo_clip(actx, &src, &out, logo.h, MaskRatio(), fr.empty() ? nullptr : fr.data(), maxFadeLength, 0,
                               vi.num_frames, fades.data()));
    devFades = std::move(fades);
    dev = own;
    return true;
  }

  bool Streamable(IScriptEnvironment* env) {
    if (streamable < 0) {
      amtk_clip dc;
      IDeviceClip* d = dynamic_cast<IDeviceClip*>(child.get());
      const AMTAnalyzeLogo* a = dynamic_cast<const AMTAnalyzeLogo*>(analyzeclip.get());
      streamable = mode == 0 && !(d && d->GetDeviceClip(&dc)) && a && a->Source().get() == child.get() && a->LogoPath() == logoPath;
    }
    return streamable == 1;
  }
  void DropStream() { stream.reset(); held.clear(); streamNext = streamSent = 0; }
  bool StartStream(IScriptEnvironment* env) {
    std::vector<uint8_t> fr(frameResult.begin(), frameResult.end());
    amtk_erase_logo_stream* s = nullptr;
    if (!amtk_erase_logo_stream_create(env->GetAmtkContext(), logo.h, dynamic_cast<const AMTAnalyzeLogo*>(analyzeclip.get())->MaskRatio(),
                                       vi.num_frames, fr.empty() ? nullptr : fr.data(), maxFadeLength, kStreamBatch, &s)) {
      streamable = 0;                       // refused (a logo too large for the evaluation plan, ...): the per-frame path
      return false;
    }
    stream.reset(s);
    streamsStarted += 1;
    return true;
  }
  // The stream's next output: send the child's next frames until it can be received.
  PVideoFrame ServeNext(IScriptEnvironment* env) {
    for (;;) {
      if (!held.empty()) {
        amtk_clip dst = HostFrameClip(held.front(), vi);
        int got = 0, idx = -1;
        amtk_check(amtk_erase_logo_stream_recv(stream.get(), &dst, &idx, &got, nullptr), env);
        if (got) {
          PVideoFrame f = held.front();
          held.pop_front();
          streamNext += 1;
          return f;
        }
      }
      PVideoFrame f = child->GetFrame(streamSent, env);
      env->MakeWritable(&f);
      amtk_clip c = HostFrameClip(f, vi);
      amtk_check(amtk_erase_logo_stream_send(stream.get(), &c), env);
      held.push_back(f);
      streamSent += 1; framesSent += 1;
    }
  }

  void CalcFade2(int n, float& fadeT, float& fadeB, IScriptEnvironment* env) {           // :1263-1315
    // CalcFade2 looks at nine analyze records around n; they sit in at most three analyze frames (8 records each), which
    // are fetched through the analyze clip's GetFrame exactly like the reference does -- nothing proportional to the clip
    // length is allocated or cleared here.
    const int nrec = vi.num_frames;
    float rec9[9 * 33];
    PVideoFrame held; int held_blk = -1;
    for (int i = -4; i <= 4; ++i) {
      const int src = amtk_calc_fade2_index(nrec, vi.num_frames, n, i);
      const int blk = src >> 3;
      if (blk != held_blk) { held = analyzeclip->GetFrame(blk, env); held_blk = blk; }
      memcpy(rec9 + (size_t)(i + 4) * 33, reinterpret_cast<const LogoAnalyzeFrame*>(held->GetReadPtr()) + (src & 7), sizeof(LogoAnalyzeFrame));
    }
    amtk_calc_fade2_records(rec9, &fadeT, &fadeB);
  }
  void CalcFade(int n, float& fadeT, float& fadeB, IScriptEnvironment* env) {            // :1317-1341
    if (frameResult.empty()) { CalcFade2(n, fadeT, fadeB, env); return; }
    const int halfWidth = maxFadeLength >> 1;
    bool uniform = true; int first = 0;
    for (int i = -halfWidth; i <= halfWidth; ++i) {
      const int v = frameResult[std::max(0, std::min(vi.num_frames - 1, n + i))];
      if (i == -halfWidth) first = v; else if (v != first) uniform = false;
    }
    if (uniform) fadeT = fadeB = (frameResult[std::max(0, std::min(vi.num_frames - 1, n))] == 2) ? 1.0f : 0.0f;
    else CalcFade2(n, fadeT, fadeB, env);
  }
  void ReadLogoFrameFile(const tstring& path, IScriptEnvironment* env) {                  // :1421-1461
    struct Elem { bool isStart; int best, start, end; };
    std::vector<Elem> el;
    FILE* fp = fopen(path.c_str(), "r");
    if (!fp) env->ThrowError("Failed to read dat file (%s)", path.c_str());
    std::regex re("^\\s*(\\d+)\\s+(\\S)\\s+(\\d+)\\s+(\\S+)\\s+(\\d+)\\s+(\\d+)");
    char line[512];
    while (fgets(line, sizeof(line), fp)) {
      std::cmatch m;
      if (std::regex_search(line, m, re))
        el.push_back(Elem{ std::tolower(m[2].str()[0]) == 's', std::stoi(m[1].str()), std::stoi(m[5].str()), std::stoi(m[6].str()) });
    }
    fclose(fp);
    frameResult.assign(vi.num_frames, 0);
    auto fill = [&](int a, int b, int v) { std::fill(frameResult.begin() + std::min(vi.num_frames, a), frameResult.begin() + std::min(vi.num_frames, std::max(a, b)), v); };
    for (size_t i = 0; i + 1 < el.size() || i < el.size(); i += 2) {
      if (i + 1 >= el.size() || !el[i].isStart || el[i + 1].isStart)
        env->ThrowError("Invalid logoframe file. Start and End must be cyclic.");
      fill(el[i].start, el[i].end + 1, 1);
      fill(el[i].end, el[i + 1].start + 1, 2);
      fill(el[i + 1].start + 1, el[i + 1].end + 1, 1);
    }
  }
public:
  AMTEraseLogo(PClip clip, PClip analyzeclip, const tstring& logoPath, const tstring& logofPath, int mode, int maxFadeLength, IScriptEnvironment* env)
      : GenericVideoFilter(clip), analyzeclip(analyzeclip), mode(mode), maxFadeLength(maxFadeLength), logoPath(logoPath),
        actx(env->GetAmtkContext()) {
    amtk_logo* p = nullptr;
    if (!amtk_logo_load(env->GetAmtkContext(), logoPath.c_str(), &p, nullptr))
      env->ThrowError("Failed to read logo file (%s)", logoPath.c_str());                 // :1471-1477
    logo = LogoHandle(p);
    if (logofPath.size() > 0) ReadLogoFrameFile(logofPath, env);
  }
  void GetFades(int n, float& fadeT, float& fadeB, IScriptEnvironment* env) {
    if (Resident()) { fadeT = devFades[(size_t)n * 2]; fadeB = devFades[(size_t)n * 2 + 1]; return; }
    CalcFade(n, fadeT, fadeB, env);
  }

  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {               // :1343-1419
    const int pixelSize = vi.ComponentSize();
    if (pixelSize != 1 && pixelSize != 2) env->ThrowError("[AMTEraseLogo] Unsupported pixel format");
    if (Resident()) {
      n = std::max(0, std::min(vi.num_frames - 1, n));
      PVideoFrame f = PackedDeviceFrame(vi, dev, n, env);
      f->CopyPropertiesFrom(*child->GetFrame(n, env));
      return f;
    }
    if (std::lock_guard<std::mutex> lock(streamMu); Streamable(env)) {
      if (n == lastServed && lastFrame) return lastFrame;
      if (!stream && n == 0) StartStream(env);
      if (stream && n == streamNext) {
        try {
          lastFrame = ServeNext(env);
        } catch (...) {
          DropStream();
          throw;
        }
        lastServed = n;
        return lastFrame;
      }
      DropStream();                          // any other read: the per-frame path
    }
    PVideoFrame frame = child->GetFrame(n, env);
    env->MakeWritable(&frame);
    float fades[2];
    CalcFade(n, fades[0], fades[1], env);
    if (mode != 0) {                       // logo-frame debug mode (:1400-1418): the frame is returned with a text label
      lastDebugLabel = DebugLabel(fades[0], fades[1]);      // drawn by the reference's DrawText (TextOut.cpp, out of scope); the
      return frame;                                          // label itself is available through GetDebugLabel()
    }
    // The CPU frame is edited in place; the library moves only the three logo rectangles through HBM (Delogo kernel),
    // with no per-frame device allocation and no full-frame copy.
    amtk_clip c = HostFrameClip(frame, vi);
    amtk_check(amtk_erase_logo_frames(env->GetAmtkContext(), &c, logo.h, 0, 1, fades), env);
    return frame;
  }
  static std::string DebugLabel(float fadeT, float fadeB) {                               // :1404-1414
    const char* str = (fadeT == fadeB) ? ((fadeT < 0.5) ? "X" : "O") : ((fadeT < fadeB) ? "BTM" : "TOP");
    char buf[200];
    snprintf(buf, sizeof(buf), "%s %.1f vs %.1f", str, fadeT, fadeB);
    return buf;
  }
  const std::string& GetDebugLabel() const { return lastDebugLabel; }
  int FramesSent() const { return framesSent; }             // child frames the frame streams took in
  int StreamsStarted() const { return streamsStarted; }
  // Batched form for an HBM-resident source: every frame of [first, first+count) erased in place.  Over its own analyze
  // chain one amtk_erase_logo_clip call decides the fades on the device; otherwise the fades come from the analyze clip.
  void EraseInPlace(int first, int count, IScriptEnvironment* env) {
    amtk_clip dc;
    if (!ChildDeviceClip(&dc)) env->ThrowError("[AMTEraseLogo] EraseInPlace needs a device-resident source");
    if (OwnChain()) {
      std::vector<uint8_t> fr(frameResult.begin(), frameResult.end());
      amtk_check(amtk_erase_logo_clip(env->GetAmtkContext(), &dc, nullptr, logo.h, MaskRatio(), fr.empty() ? nullptr : fr.data(),
                                      maxFadeLength, first, count, nullptr), env);
      return;
    }
    std::vector<float> fades((size_t)count * 2);
    for (int i = 0; i < count; ++i) CalcFade(first + i, fades[2 * i], fades[2 * i + 1], env);
    amtk_check(amtk_erase_logo_frames(env->GetAmtkContext(), &dc, logo.h, first, count, fades.data()), env);
  }
  bool GetDeviceClip(amtk_clip* c) override {
    if (!Resident()) return false;
    *c = out;
    return true;
  }
  int __stdcall SetCacheHints(int cachehints, int) override { return cachehints == CACHE_GET_MTMODE ? MT_NICE_FILTER : 0; }   // :1500-1505

  static AVSValue __cdecl Create(AVSValue args, void*, IScriptEnvironment* env) {         // :1507-1518
    return AVSValue(PClip(new AMTEraseLogo(args[0].AsClip(), args[1].AsClip(), args[2].AsString(), args[3].AsString(""),
                                           args[4].AsInt(0), args[5].AsInt(16), env)));
  }
};

// ---------------------------------------------------------------------------------------------------------------
// LogoFrame (LogoScan.hpp:1521-1836): whole-clip logo scan used by CMAnalyze::logoFrame (CMAnalyze.hpp:273-317)
// ---------------------------------------------------------------------------------------------------------------
class LogoFrame {
  AMTContext& ctx;
  int numLogos;
  std::vector<LogoHandle> logoArr, deintArr;
  int numFrames = 0, framesPerSec = 30;
  VideoInfo vi;
  struct EvalResult { float corr0, corr1; };
  std::vector<EvalResult> evalResults;
  static constexpr int kStreamBatch = 64;                               // frames per launch of the frame stream
  static constexpr int kCombBatch = 16;                                 // ... of the streams that run the combing pass (as AMTCombAnalyze)
  const float THRESH = 0.2f;                                            // |score| below this is "unknown" (:1538)
  int bestLogo = -1;
  float logoRatio = 0.0f;
public:
  LogoFrame(AMTContext& ctx, const std::vector<tstring>& logofiles, float maskratio) : ctx(ctx) {   // :1592-1616
    numLogos = (int)logofiles.size();
    logoArr.resize(numLogos); deintArr.resize(numLogos);
    for (int i = 0; i < numLogos; ++i) {
      amtk_logo* p = nullptr;
      if (!amtk_logo_load(nullptr, logofiles[i].c_str(), &p, nullptr)) continue;          // load errors are ignored (:1612-1614)
      logoArr[i] = LogoHandle(p);
      if (amtk_logo_deint(logoArr[i].h, &p)) { deintArr[i] = LogoHandle(p); amtk_logo_create_mask(deintArr[i].h, maskratio); }
    }
  }

  void scanFrames(PClip clip, IScriptEnvironment2* env) {                                   // :1618-1630
    vi = clip->GetVideoInfo();
    const int pixelSize = vi.ComponentSize();
    if (pixelSize != 1 && pixelSize != 2) env->ThrowError("[LogoFrame] Unsupported pixel format");
    amtk_ctx* actx = env->GetAmtkContext();
    std::vector<amtk_logo*> hs(numLogos);
    for (int i = 0; i < numLogos; ++i) hs[i] = deintArr[i].h;          // invalid logos stay NULL -> (0,-1) (:1551-1558)
    evalResults.assign((size_t)vi.num_frames * numLogos, EvalResult{ 0, -1 });
    // the reference passes the BYTE pitch as element pitch also for 16-bit clips (:1547,1561); kept for parity
    amtk_clip dc;
    IDeviceClip* d = dynamic_cast<IDeviceClip*>(clip.get());
    if (d && d->GetDeviceClip(&dc)) {                                    // one batched call for the whole clip
      const int quirk = pixelSize == 2 ? dc.pitch_y : 0;
      amtk_check(amtk_logo_scan_frames(actx, &dc, hs.data(), numLogos, 0, vi.num_frames, quirk,
                                       reinterpret_cast<float*>(evalResults.data()), 0), env);
    } else {
      // generic IClip: the reference's pull loop (:1577-1579) feeding the frame stream (DESIGN.md section 3.3.3), which
      // moves only the logo rectangles and evaluates kStreamBatch frames per launch
      struct StreamRelease { void operator()(amtk_logo_scan_stream* s) const { amtk_logo_scan_stream_destroy(s); } };
      // create checks every logo it is given; one made for another frame size gives (0,-1) whatever it holds, so it is
      // passed as NULL, as the per-frame and batched calls never look at it either
      std::vector<amtk_logo*> evaluated(hs);
      for (amtk_logo*& lg : evaluated) {
        amtk_logo_info li;
        if (lg && (!amtk_logo_get_info(lg, &li) || li.imgw != vi.width || li.imgh != vi.height)) lg = nullptr;
      }
      amtk_logo_scan_stream* s = nullptr;
      amtk_check(amtk_logo_scan_stream_create(actx, evaluated.data(), numLogos, kStreamBatch, 1, &s), env);
      std::unique_ptr<amtk_logo_scan_stream, StreamRelease> stream(s);
      int received = 0;
      auto drain = [&]() {
        int got = 0;
        amtk_check(amtk_logo_scan_stream_recv(stream.get(), reinterpret_cast<float*>(evalResults.data() + (size_t)received * numLogos),
                                              vi.num_frames - received, &got), env);
        received += got;
      };
      for (int n = 0; n < vi.num_frames; ++n) {
        PVideoFrame f = clip->GetFrame(n, env);
        amtk_clip hc = HostFrameClip(f, vi);
        amtk_check(amtk_logo_scan_stream_send(stream.get(), &hc), env);
        drain();
        if ((n % 5000) == 0) ctx.infoF("%6d/%d", n, vi.num_frames);
      }
      amtk_check(amtk_logo_scan_stream_finish(stream.get()), env);
      drain();
    }
    numFrames = vi.num_frames;
    framesPerSec = (int)std::round((float)vi.fps_numerator / vi.fps_denominator);
    ctx.info("Finished");
  }

  // scanFrames, and the combing counters of the same frames (AMTCombAnalyze's, int32[num_frames][12]) from the same pass,
  // so that the logo detection and the telecine pre-pass share one decode.  The scores equal scanFrames(clip, env)'s: on
  // 2-byte samples both keep ScanFrame's byte-pitch row step.
  //  - device-resident clip: one amtk_scan_comb_frames_pitch call.
  //  - any other clip: each child frame is asked for once, in order, and sent to the fused frame stream (DESIGN.md section
  //    3.1e) with the byte-pitch row step.
  void scanFrames(PClip clip, IScriptEnvironment2* env, const amtk_comb_params& prm, std::vector<int32_t>& counts) {
    vi = clip->GetVideoInfo();
    const int pixelSize = vi.ComponentSize();
    if (pixelSize != 1 && pixelSize != 2) env->ThrowError("[LogoFrame] Unsupported pixel format");
    amtk_ctx* actx = env->GetAmtkContext();
    const int N = vi.num_frames;
    std::vector<amtk_logo*> hs(numLogos);
    for (int i = 0; i < numLogos; ++i) hs[i] = deintArr[i].h;          // invalid logos stay NULL -> (0,-1) (:1551-1558)
    evalResults.assign((size_t)N * numLogos, EvalResult{ 0, -1 });
    counts.assign((size_t)N * 12, 0);
    float* scores = reinterpret_cast<float*>(evalResults.data());
    amtk_clip dc;
    IDeviceClip* d = dynamic_cast<IDeviceClip*>(clip.get());
    if (d && d->GetDeviceClip(&dc)) {
      const int quirk = pixelSize == 2 ? dc.pitch_y : 0;
      amtk_check(amtk_scan_comb_frames_pitch(actx, &dc, hs.data(), numLogos, &prm, quirk, 0, N, scores, counts.data(), 0), env);
    } else {
      // logos made for another frame size give (0,-1) whatever they hold; the stream checks every logo it is given
      std::vector<amtk_logo*> evaluated(hs);
      for (amtk_logo*& lg : evaluated) {
        amtk_logo_info li;
        if (lg && (!amtk_logo_get_info(lg, &li) || li.imgw != vi.width || li.imgh != vi.height)) lg = nullptr;
      }
      struct FusedRelease { void operator()(amtk_scan_comb_stream* s) const { amtk_scan_comb_stream_destroy(s); } };
      amtk_scan_comb_stream* s = nullptr;
      amtk_check(amtk_scan_comb_stream_create_pitch(actx, evaluated.data(), numLogos, &prm, kCombBatch, 1, &s), env);
      std::unique_ptr<amtk_scan_comb_stream, FusedRelease> fused(s);
      int received = 0;
      auto drain = [&]() {
        int got = 0;
        amtk_check(amtk_scan_comb_stream_recv(fused.get(), scores + (size_t)received * numLogos * 2, counts.data() + (size_t)received * 12,
                                              N - received, &got), env);
        received += got;
      };
      for (int n = 0; n < N; ++n) {
        PVideoFrame f = clip->GetFrame(n, env);
        amtk_clip hc = HostFrameClip(f, vi);
        amtk_check(amtk_scan_comb_stream_send(fused.get(), &hc), env);
        drain();
        if ((n % 5000) == 0) ctx.infoF("%6d/%d", n, N);
      }
      amtk_check(amtk_scan_comb_stream_finish(fused.get()), env);
      drain();
    }
    numFrames = N;
    framesPerSec = (int)std::round((float)vi.fps_numerator / vi.fps_denominator);
    ctx.info("Finished");
  }

  const float* results() const { return reinterpret_cast<const float*>(evalResults.data()); }
  // Offline re-analysis of saved scores: float[nframes][numLogos][2] as scanFrames produces them (the reference can only
  // dump them, dumpResult :1632-1645).  Lets selectLogo / writeResult run without a device.
  void setResults(const float* corr, int nframes, unsigned fps_numerator, unsigned fps_denominator) {
    evalResults.resize((size_t)nframes * numLogos);
    memcpy(evalResults.data(), corr, evalResults.size() * sizeof(EvalResult));
    numFrames = nframes;
    framesPerSec = (int)std::round((float)fps_numerator / fps_denominator);
  }

  // choose the logo that is detected most often with the least residue after removal (:1647-1682)
  void selectLogo(int numCandidates = -1) {
    if (numCandidates < 0) numCandidates = numLogos;
    struct Summary { float cost = 0; int numFrames = 0; };
    std::vector<Summary> sum(numCandidates);
    for (int n = 0; n < numFrames; ++n)
      for (int i = 0; i < numCandidates; ++i) {
        const EvalResult& r = evalResults[(size_t)n * numLogos + i];
        if (r.corr0 > THRESH && std::abs(r.corr1) < THRESH) { sum[i].numFrames++; sum[i].cost += std::abs(r.corr1); }
      }
    std::vector<float> score(numCandidates);
    for (int i = 0; i < numCandidates; ++i) {
      const Summary& s = sum[i];
      score[i] = (s.numFrames == 0) ? INFINITY : (s.cost / s.numFrames) * (numFrames / (float)s.numFrames);
      ctx.debugF("logo%d: %f * %f = %f", i + 1, (s.cost / s.numFrames), (numFrames / (float)s.numFrames), score[i]);
    }
    bestLogo = (int)(std::min_element(score.begin(), score.end()) - score.begin());
    logoRatio = (float)sum[bestLogo].numFrames / numFrames;
  }

  // logoframe file for join_logo_scp / AMTEraseLogo::ReadLogoFrameFile (:1686-1827)
  void writeResult(const tstring& outpath, int logoIndex = -1) {
    if (logoIndex < 0) { if (bestLogo < 0) selectLogo(); logoIndex = bestLogo; }
    const float threshL = 0.5f, avgDur = 1.0f, medianDur = 0.5f;
    const int halfAvg = int(framesPerSec * avgDur / 2 + 0.5f), aveFrames = halfAvg * 2 + 1;
    const int halfMed = int(framesPerSec * medianDur / 2 + 0.5f), medFrames = halfMed * 2 + 1;
    const int win = std::max(aveFrames, medFrames), halfWin = win / 2;
    const int N = numFrames;
    // raw score per frame (negative corr0 and positive corr1 are noise), edge-padded by half a window
    std::vector<float> padded((size_t)N + win);
    float* raw = padded.data() + halfWin;
    for (int n = 0; n < N; ++n) {
      const EvalResult& r = evalResults[(size_t)n * numLogos + logoIndex];
      raw[n] = std::max(0.0f, r.corr0) + std::min(0.0f, r.corr1);
    }
    std::fill(padded.data(), raw, raw[0]);
    std::fill(raw + N, padded.data() + padded.size(), raw[N - 1]);

    struct FR { int result; float score; };
    std::vector<FR> fr(N);
    std::vector<float> med(medFrames);
    for (int i = 0; i < N; ++i) {
      // min of the maxima before and after: rescues frames where motion washes the logo out
      const float beforeMax = *std::max_element(raw + i - halfAvg, raw + i);
      const float afterMax = *std::max_element(raw + i + 1, raw + i + 1 + halfAvg);
      const float mm = std::min(beforeMax, afterMax);
      const int mmRes = (std::abs(mm) < threshL) ? 1 : (mm < 0.0f) ? 0 : 2;
      const float avg = std::accumulate(raw + i - halfAvg, raw + i + halfAvg + 1, 0.0f) / aveFrames;
      const int avgRes = (std::abs(avg) < THRESH) ? 1 : (avg < 0.0f) ? 0 : 2;
      fr[i].result = (mmRes != avgRes) ? 1 : mmRes;
      std::copy(raw + i - halfMed, raw + i + halfMed + 1, med.begin());
      std::sort(med.begin(), med.end());
      fr[i].score = med[halfMed];
    }
    // unknown runs bounded by equal states take that state
    for (int it = 0; it != N;) {
      int first1 = it; while (first1 < N && fr[first1].result != 1) ++first1;
      it = first1; while (it < N && fr[it].result == 1) ++it;
      const int prev = (first1 == 0) ? 0 : fr[first1 - 1].result;
      const int next = (it == N) ? 0 : fr[it].result;
      if (prev == next) for (int k = first1; k < it; ++k) fr[k].result = prev;
    }
    // emit logo sections, refining the boundaries on the median-filtered score
    std::string out;
    auto last_before = [&](int hi, int lo, auto pred, int none) {        // reverse find in [lo,hi): index+1 of the hit, else `none`
      for (int k = hi - 1; k >= lo; --k) if (pred(fr[k])) return k + 1;
      return none;
    };
    auto first_from = [&](int lo, int hi, auto pred) { for (int k = lo; k < hi; ++k) if (pred(fr[k])) return k; return hi; };
    for (int it = 0; it != N;) {
      const int sEnd0 = first_from(it, N, [](const FR& r) { return r.result == 2; });
      const int eEnd0 = first_from(sEnd0, N, [](const FR& r) { return r.result == 0; });
      int sEnd = sEnd0, eEnd = eEnd0;
      if (sEnd != N) {
        if (fr[sEnd].score >= THRESH) sEnd = last_before(sEnd, 0, [&](const FR& r) { return r.score < THRESH; }, 0);
        else sEnd = first_from(sEnd, N, [&](const FR& r) { return r.score >= THRESH; });
      }
      if (eEnd != N) {
        if (fr[eEnd].score <= -THRESH) eEnd = last_before(eEnd, sEnd, [&](const FR& r) { return r.score > -THRESH; }, sEnd);
        else eEnd = first_from(eEnd, N, [&](const FR& r) { return r.score <= -THRESH; });
      }
      const int sStart = last_before(sEnd, it, [&](const FR& r) { return r.score <= -THRESH; }, it);
      const int eStart = last_before(eEnd, sEnd, [&](const FR& r) { return r.score >= THRESH; }, sEnd);
      const int sBest = first_from(sStart, sEnd, [](const FR& r) { return r.score > 0; });
      const int eBest = last_before(eEnd, eStart, [](const FR& r) { return r.score > 0; }, eStart);
      if (sEnd != eEnd) {
        char buf[128];
        snprintf(buf, sizeof(buf), "%6d S 0 ALL %6d %6d\n", sBest, sStart, sEnd); out += buf;
        snprintf(buf, sizeof(buf), "%6d E 0 ALL %6d %6d\n", eBest - 1, eStart - 1, eEnd - 1); out += buf;
      }
      it = eEnd0;
    }
    FILE* fp = fopen(outpath.c_str(), "w");
    if (!fp) throw IOException("failed to open " + outpath);
    fwrite(out.data(), 1, out.size(), fp);
    fclose(fp);
  }
  int getBestLogo() const { return bestLogo; }
  float getLogoRatio() const { return logoRatio; }
};

// ---------------------------------------------------------------------------------------------------------------
// LogoAnalyzer (LogoScan.hpp:794-1080): logo generation from a clip read frame by frame, as the reference's
// SimpleVideoReader drives InitialLogoCreator::onFrame, over amtk_scan_logo_stream.  The constructor takes the reference's
// parameters minus the decoder's path, the service id and the work file (the rectangles stay in HBM); the service id
// comes with ScanLogo, as for LogoData::Save.
// ---------------------------------------------------------------------------------------------------------------
typedef bool (*LOGO_ANALYZE_CB)(float progress, int nread, int total, int ngather);     // LogoScan.hpp:792

class LogoAnalyzer {
  AMTContext& ctx;
  int scanx, scany, scanw, scanh, thy, numMaxFrames;
  LOGO_ANALYZE_CB cb;
  static LOGO_ANALYZE_CB& current() { static thread_local LOGO_ANALYZE_CB c = nullptr; return c; }
  static int trampoline(float progress, int nread, int total, int ngather) { return current()(progress, nread, total, ngather) ? 1 : 0; }
  struct Stream {                                                       // RAII over amtk_scan_logo_stream
    amtk_scan_logo_stream* s = nullptr;
    ~Stream() { if (s) amtk_scan_logo_stream_destroy(s); }
  };
public:
  LogoAnalyzer(AMTContext& ctx, int imgx, int imgy, int w, int h, int thy, int numMaxFrames, LOGO_ANALYZE_CB cb)
      : ctx(ctx), scanx(imgx), scany(imgy), scanw(w), scanh(h), thy(thy), numMaxFrames(numMaxFrames), cb(cb) {}

  // Reads source's frames in order (device frames when the source is device resident) until the stream answers
  // more == 0 or the clip ends, then GetLogo, ReMakeLogo x2 and Save (:1058-1079).  A clip's "file position" is the
  // number of frames read and its "file size" the number of frames (progress = (n + 1) / num_frames * 50).
  void ScanLogo(PClip source, int serviceid, const tstring& dstpath, IScriptEnvironment* env) {
    const VideoInfo& vi = source->GetVideoInfo();
    Stream st;
    current() = cb;
    amtk_check(amtk_scan_logo_stream_create(env->GetAmtkContext(), scanx, scany, scanw, scanh, thy, numMaxFrames,
                                            cb ? &LogoAnalyzer::trampoline : nullptr, &st.s), env);
    amtk_clip dclip;
    IDeviceClip* dev = dynamic_cast<IDeviceClip*>(source.get());
    const bool resident = dev && dev->GetDeviceClip(&dclip);
    for (int n = 0; n < vi.num_frames; ++n) {
      int more = 1;
      if (resident) {
        amtk_clip f = dclip;
        f.base = static_cast<const uint8_t*>(dclip.base) + (int64_t)n * dclip.frame_stride;
        f.num_frames = 1;
        amtk_check(amtk_scan_logo_stream_send(st.s, &f, n + 1, vi.num_frames, &more), env);
      } else {
        PVideoFrame frame = source->GetFrame(n, env);
        const amtk_clip f = HostFrameClip(frame, vi);
        amtk_check(amtk_scan_logo_stream_send(st.s, &f, n + 1, vi.num_frames, &more), env);
      }
      if (!more) break;
    }
    amtk_check(amtk_scan_logo_stream_finish(st.s, serviceid, dstpath.c_str()), env);
  }
};

}  // namespace logo

// ---------------------------------------------------------------------------------------------------------------
// Telecine pre-pass.  In the product the script calls KFMDeint(..., pass=..., filepath=AMT_TMP) from an external plugin
// and AMTFilterSource pulls every frame and discards it (FilteredSource.hpp:417-439,519-544).  AMTCombAnalyze is that
// pre-pass filter for the field-difference / combing counters; GetFrame returns the source frame untouched (pre-process
// semantics), results go to <AMT_TMP>.combstat.txt (one line per frame: 12 integers) when a path is given.
//  - device-resident child: the whole clip is analysed by ONE streaming launch on first use.
//  - any other child: the frame stream (DESIGN.md section 3.1d).  A GetFrame of the next frame in order pulls that child
//    frame once, sends it and returns it, so ReadAllFrames decodes every frame once; once the last frame is sent the rows
//    are received and the file is written.  Any other request, and Counts() before the end, first completes the pass by
//    pulling the remaining frames in order through the stream.
// ---------------------------------------------------------------------------------------------------------------
// The combing-stats file of the telecine pre-pass: one line per frame, its 12 counters (int32[num_frames][12]) as decimal
// integers separated by single spaces.  `who` names the writer in the error.
inline void WriteCombStats(const tstring& path, const std::vector<int32_t>& counts, int num_frames, const char* who, IScriptEnvironment* env) {
  FILE* fp = fopen(path.c_str(), "w");
  if (!fp) env->ThrowError("%s: failed to write %s", who, path.c_str());
  for (int n = 0; n < num_frames; ++n) {
    for (int k = 0; k < 12; ++k) fprintf(fp, k ? " %d" : "%d", counts[(size_t)n * 12 + k]);
    fputc('\n', fp);
  }
  fclose(fp);
}

class AMTCombAnalyze : public GenericVideoFilter {
  static constexpr int kStreamBatch = 16;          // frames per launch of the frame stream: faster than 64 (DESIGN.md 6.6)
  struct StreamRelease { void operator()(amtk_comb_stream* s) const { amtk_comb_stream_destroy(s); } };
  std::vector<int32_t> counts;
  tstring outpath;
  amtk_comb_params prm;
  bool started = false, done = false;
  std::unique_ptr<amtk_comb_stream, StreamRelease> stream;              // null: device-resident child, or the pass is done
  int sent = 0, received = 0;
  // First use: a device-resident child is analysed at once; any other gets a frame stream.
  void Start(IScriptEnvironment* env) {
    if (started) return;
    amtk_ctx* ctx = env->GetAmtkContext();
    counts.assign((size_t)vi.num_frames * 12, 0);
    amtk_clip dc;
    IDeviceClip* d = dynamic_cast<IDeviceClip*>(child.get());
    if (d && d->GetDeviceClip(&dc)) {
      amtk_check(amtk_comb_frames(ctx, &dc, &prm, 0, vi.num_frames, counts.data(), 0), env);
      started = true;
      Write(env);
      return;
    }
    amtk_comb_stream* s = nullptr;
    amtk_check(amtk_comb_stream_create(ctx, &prm, kStreamBatch, &s), env);
    stream.reset(s);
    started = true;
    if (vi.num_frames == 0) End(env);
  }
  void Receive(IScriptEnvironment* env) {
    int got = 0;
    amtk_check(amtk_comb_stream_recv(stream.get(), counts.data() + (size_t)received * 12, vi.num_frames - received, &got), env);
    received += got;
  }
  // Pulls the next child frame once, sends it and returns it; the last one ends the pass.
  PVideoFrame Send(IScriptEnvironment* env) {
    PVideoFrame f = child->GetFrame(sent, env);
    const amtk_clip c = HostFrameClip(f, vi);
    amtk_check(amtk_comb_stream_send(stream.get(), &c), env);
    sent += 1;
    Receive(env);
    if (sent == vi.num_frames) End(env);
    return f;
  }
  void End(IScriptEnvironment* env) {
    amtk_check(amtk_comb_stream_finish(stream.get()), env);
    Receive(env);
    stream.reset();
    Write(env);
  }
  void Complete(IScriptEnvironment* env) {
    Start(env);
    while (!done) Send(env);
  }
  void Write(IScriptEnvironment* env) {
    if (!outpath.empty()) WriteCombStats(outpath, counts, vi.num_frames, "AMTCombAnalyze", env);
    done = true;
  }
public:
  AMTCombAnalyze(PClip clip, const tstring& outpath, IScriptEnvironment*) : GenericVideoFilter(clip), outpath(outpath) { amtk_comb_default_params(&prm); }
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    Start(env);
    if (!done && n == sent) return Send(env);
    Complete(env);
    return child->GetFrame(n, env);
  }
  const std::vector<int32_t>& Counts(IScriptEnvironment* env) { Complete(env); return counts; }
  int __stdcall SetCacheHints(int cachehints, int) override { return cachehints == CACHE_GET_MTMODE ? MT_SERIALIZED : 0; }
  static AVSValue __cdecl Create(AVSValue args, void*, IScriptEnvironment* env) {
    return AVSValue(PClip(new AMTCombAnalyze(args[0].AsClip(), args[1].AsString(""), env)));
  }
};

// AMTFilterSource::ReadAllFrames (FilteredSource.hpp:417-439): pull every frame of a pre-process pass and discard it.
inline void ReadAllFrames(PClip clip, IScriptEnvironment* env) {
  const int n = clip->GetVideoInfo().num_frames;
  for (int i = 0; i < n; ++i) clip->GetFrame(i, env);
}

// ---------------------------------------------------------------------------------------------------------------
// Telecine side files and their consumers (SURVEY 8 f3)
// ---------------------------------------------------------------------------------------------------------------
// AMTDecimate (FilteredSource.hpp:637-676): <tmp>.duration.txt holds one integer per OUTPUT frame = how many source
// frames it lasts; output frame i shows source frame sum(durations[0..i)).
class AMTDecimate : public GenericVideoFilter {
  std::vector<int> durations, framesMap;
public:
  AMTDecimate(PClip source, const std::string& duration, IScriptEnvironment* env) : GenericVideoFilter(source) {
    FILE* fp = fopen(duration.c_str(), "r");
    if (!fp) env->ThrowError("[AMTDecimate] failed to open %s", duration.c_str());
    char line[256];
    while (fgets(line, sizeof(line), fp)) durations.push_back(std::atoi(line));
    fclose(fp);
    const int numSourceFrames = std::accumulate(durations.begin(), durations.end(), 0);
    if (vi.num_frames != numSourceFrames)
      env->ThrowError("[AMTDecimate] # of frames does not match. %d(%s) vs %d(source clip)", numSourceFrames, duration.c_str(), vi.num_frames);
    vi.num_frames = (int)durations.size();
    framesMap.assign(durations.size(), 0);
    for (size_t i = 0; i + 1 < durations.size(); ++i) framesMap[i + 1] = framesMap[i] + durations[i];
  }
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    return child->GetFrame(framesMap[std::max(0, std::min(n, vi.num_frames - 1))], env);
  }
  int SourceFrame(int n) const { return framesMap[std::max(0, std::min(n, (int)framesMap.size() - 1))]; }
  static AVSValue __cdecl Create(AVSValue args, void*, IScriptEnvironment* env) {
    return AVSValue(PClip(new AMTDecimate(args[0].AsClip(), args[1].AsString(), env)));
  }
};

// AMTFilterSource::readTimecodeFile + readTimecode (FilteredSource.hpp:163-212): timestamps in ms, one per line,
// '#' comments, optional "# total: <seconds>"; the end time is extrapolated when absent; the VFR base rate is the one
// of 60/120/240 (x1000/1001) whose grid fits the timestamps best.
struct TimecodeFile {
  std::vector<double> timeCodes;
  int vfrTimingFps = 0;
  bool read(const std::string& path) {
    FILE* fp = fopen(path.c_str(), "r");
    if (!fp) return false;
    std::regex re("#\\s*total:\\s*([+-]?([0-9]*[.])?[0-9]+).*");
    char line[512];
    timeCodes.clear();
    bool total = false;
    while (!total && fgets(line, sizeof(line), fp)) {
      std::string str(line);
      while (!str.empty() && (str.back() == '\n' || str.back() == '\r')) str.pop_back();
      if (str.empty()) continue;
      std::smatch m;
      if (std::regex_search(str, m, re)) { timeCodes.push_back(std::atof(m[1].str().c_str()) * 1000); total = true; }
      else if (str[0] != '#') timeCodes.push_back(std::atoi(str.c_str()));
    }
    fclose(fp);
    if (!total) {
      const size_t n = timeCodes.size();
      if (n >= 2) timeCodes.push_back(timeCodes[n - 1] * 2 - timeCodes[n - 2]);
      else if (n == 1) timeCodes.push_back(timeCodes[0] + 1000.0 / 60.0);
    }
    if (timeCodes.empty()) return true;
    double minDiff = timeCodes.back();
    const double epsilon = timeCodes.size() * 10e-10;
    for (int fps : { 60, 120, 240 }) {
      const double mult = fps / 1001.0, inv = 1.0 / mult;
      double diff = 0;
      for (double ts : timeCodes) diff += std::abs(inv * std::round(ts * mult) - ts);
      if (diff < minDiff - epsilon) { vfrTimingFps = fps; minDiff = diff; }
    }
    return true;
  }
};

// Pulldown classification from the combing counters (this repo's heuristic; the reference delegates the decision to
// the external KFM plugin).  3:2 telecine shows up as two adjacent combed frames in every 5-frame cycle.  The cycle
// phase is taken from the whole clip (the frame pair position with the largest summed comb response); a cycle whose
// pair stands out by `ratio` against its other three frames becomes 4 film frames (durations 1,1,2,1: the film frame
// that straddles the combed pair lasts two video frames), any other cycle passes through as 5 x 1.
// Writes <base>.duration.txt (AMTDecimate) and <base>.timecode.txt (ms per output frame, "# total:" trailer).
// Returns the number of film cycles, -1 on I/O error.
inline int WriteTelecineFiles(const std::vector<int32_t>& counts, int num_frames, unsigned fps_num, unsigned fps_den,
                              const std::string& base, double ratio = 2.0) {
  // the large-threshold response ("lshima", Y top+bottom) separates real combing from vertical detail best
  auto shima = [&](int n) { return (long long)counts[(size_t)n * 12 + 2] + counts[(size_t)n * 12 + 5]; };
  int phase = 0; long long best = -1;
  for (int p = 0; p < 5; ++p) {
    long long acc = 0;
    for (int n = p; n + 1 < num_frames; n += 5) acc += std::min(shima(n), shima(n + 1));
    if (acc > best) { best = acc; phase = p; }
  }
  const int start = (phase + 3) % 5;                      // cycles begin two frames before the combed pair
  std::vector<int> durations;
  int film_cycles = 0, n = 0;
  for (; n < start && n < num_frames; ++n) durations.push_back(1);
  for (; n + 5 <= num_frames; n += 5) {
    const long long pair = std::min(shima(n + 2), shima(n + 3));
    const long long rest = std::max(std::max(shima(n), shima(n + 1)), shima(n + 4));
    if ((double)pair > ratio * (double)std::max<long long>(rest, 1)) {
      ++film_cycles;
      const int d[4] = { 1, 1, 2, 1 };
      durations.insert(durations.end(), d, d + 4);
    } else {
      durations.insert(durations.end(), 5, 1);
    }
  }
  for (; n < num_frames; ++n) durations.push_back(1);
  FILE* fd = fopen((base + ".duration.txt").c_str(), "w");
  FILE* ft = fopen((base + ".timecode.txt").c_str(), "w");
  if (!fd || !ft) { if (fd) fclose(fd); if (ft) fclose(ft); return -1; }
  fprintf(ft, "# timecode format v2\n");
  const double frame_ms = 1000.0 * fps_den / fps_num;
  int src = 0;
  for (int d : durations) { fprintf(fd, "%d\n", d); fprintf(ft, "%d\n", (int)std::round(src * frame_ms)); src += d; }
  fprintf(ft, "# total: %.6f\n", src * frame_ms / 1000.0);
  fclose(fd); fclose(ft);
  return film_cycles;
}

// ConfigWrapper is reduced to the accessors logoFrame() and AMTFilterSource read.
struct ConfigWrapper {
  std::vector<tstring> logoPath, eraseLogoPath;          // --logo / --erase-logo (AmatsukazeCLI.hpp:358-366)
  bool looseLogoDetection = false;                       // --loose-logo-detection (:370)
  tstring tmpDir = ".";
  const std::vector<tstring>& getLogoPath() const { return logoPath; }
  const std::vector<tstring>& getEraseLogoPath() const { return eraseLogoPath; }
  bool isLooseLogoDetection() const { return looseLogoDetection; }
  bool noDelogo = false;                                 // --no-delogo
  int maxFadeLength = 16;                                // --max-fade-length
  bool isNoDelogo() const { return noDelogo; }
  int getMaxFadeLength() const { return maxFadeLength; }
  tstring getAvsTmpPath(int v) const { return tmpDir + "/v" + std::to_string(v) + "-0-0.avstmp"; }             // TranscodeSetting.hpp:875-880 (format, div = 0)
  tstring getAvsDurationPath(int v) const { return getAvsTmpPath(v) + ".duration.txt"; }                       // :882-885
  tstring getAvsTimecodePath(int v) const { return getAvsTmpPath(v) + ".timecode.txt"; }                       // :887-890
  tstring getTmpAMTSourcePath(int v) const { return tmpDir + "/amts" + std::to_string(v) + ".dat"; }            // TranscodeSetting.hpp:926-928
  tstring getTmpLogoFramePath(int v, int logoIndex = -1) const {                                               // :934-939
    return tmpDir + "/logof" + std::to_string(v) + (logoIndex == -1 ? std::string() : "-" + std::to_string(logoIndex)) + ".txt";
  }
};

struct AviSynthException : std::runtime_error { using std::runtime_error::runtime_error; };

// AMTTelecineDecide: the second pre-process pass.  Reads the counters the first pass left in <AMT_TMP>.combstat.txt and
// writes <AMT_TMP>.duration.txt / .timecode.txt (consumed by AMTDecimate and readTimecodeFile) on first use; GetFrame
// hands the source frame through, like every pre-process filter.
class AMTTelecineDecide : public GenericVideoFilter {
  tstring base;
  bool done = false;
  int film_cycles = -1;
  void Run(IScriptEnvironment* env) {
    if (done) return;
    FILE* fp = fopen((base + ".combstat.txt").c_str(), "r");
    if (!fp) env->ThrowError("AMTTelecineDecide: pass 1 results missing (%s.combstat.txt)", base.c_str());
    std::vector<int32_t> counts((size_t)vi.num_frames * 12, 0);
    size_t got = 0;
    for (; got < counts.size(); ++got) if (fscanf(fp, "%d", &counts[got]) != 1) break;
    fclose(fp);
    if (got != counts.size()) env->ThrowError("AMTTelecineDecide: %s.combstat.txt does not match the clip (%d frames)", base.c_str(), vi.num_frames);
    film_cycles = WriteTelecineFiles(counts, vi.num_frames, vi.fps_numerator, vi.fps_denominator, base);
    if (film_cycles < 0) env->ThrowError("AMTTelecineDecide: failed to write %s.duration.txt", base.c_str());
    done = true;
  }
public:
  AMTTelecineDecide(PClip clip, const tstring& base, IScriptEnvironment*) : GenericVideoFilter(clip), base(base) {}
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override { Run(env); return child->GetFrame(n, env); }
  int FilmCycles(IScriptEnvironment* env) { Run(env); return film_cycles; }
  int __stdcall SetCacheHints(int cachehints, int) override { return cachehints == CACHE_GET_MTMODE ? MT_SERIALIZED : 0; }
};

// KFMDeint stand-in: the reference's scripts call `dsrc.KFMDeint(mode=.., pass=pass, ..., dev=AMT_DEV, filepath=AMT_TMP)`
// from the external KFM plugin (Misc.cs:1297-1323).  Only its PASS PROTOCOL is reproduced here, on this repo's combing
// metric: pass 1 = counters (pre-process), pass 2 = pulldown decision -> duration/timecode files (pre-process),
// pass 3 = the clip handed to the encoder (AMTFilterSource then appends AMTDecimate because the duration file exists).
inline AVSValue __cdecl CreateKFMDeint(AVSValue args, void*, IScriptEnvironment* env) {
  PClip clip = args[0].AsClip();
  const int pass = args[2].AsInt(0);
  const tstring base = args[3].AsString("");
  if (pass == 1) return AVSValue(PClip(new AMTCombAnalyze(clip, base.empty() ? tstring() : base + ".combstat.txt", env)));
  if (pass == 2) { if (base.empty()) env->ThrowError("KFMDeint: pass 2 needs filepath"); return AVSValue(PClip(new AMTTelecineDecide(clip, base, env))); }
  return AVSValue(clip);
}

// ---------------------------------------------------------------------------------------------------------------
// KTemporalNR stand-in: with EnableTemporalNR the server's filter script reads `ConvertBits(14)` then `KTemporalNR(3, 1)`
// (Misc.cs:1403-1428), a filter of the external CUDA plugin that also provides KFM.  That plugin's arithmetic is not in
// the reference tree, so this filter runs the reference's own TemporalNRFilter (VideoFilter.hpp:27-212) through
// amtk_tnr_frames -- bit-exact against that filter, parity with the external plugin unpinned -- under the plugin's name
// and argument spec, so the generated line runs unchanged.  Output frame n averages the 2d+1 frames clamp(n-d+i, 0, N-1).
//  - device-resident child (IDeviceClip): the whole clip is filtered into HBM by ONE call on first use; frames are served
//    as device views (CUDA consumer) or downloaded (CPU consumer), and the filter is an IDeviceClip itself, so later
//    device filters (AMTEraseLogo::EraseInPlace, ...) chain on its output;
//  - the mirror's ConvertBits over a device-resident clip (the server's two lines): the same ONE call, made on the clip
//    ConvertBits would widen, with the destination at ConvertBits' depth, so amtk_tnr_frames widens inside the filter and
//    the widened intermediate is never made.  The output VideoInfo is ConvertBits' (14-bit).  This path exists only in
//    the mirror: under AviSynth+ the built-in ConvertBits stays in charge and hands this filter CPU frames, so there
//    only amtk_tnr_frames' widening is new, reachable from a filter that receives the 8-bit clip;
//  - any other child (under AviSynth+ always: its ConvertBits hands this filter CPU frames at 14 bits): frames are served
//    as new CPU frames, each request choosing by the access pattern.  An encoder pulls frames strictly in order, and the
//    C++ drivers read each frame twice (through the clip and through OnCPU):
//      * the frame served last, asked again: the same frame;
//      * n is the next output of the live frame stream (amtk_tnr_stream, batch kStreamBatch): received from it, sending
//        the child's next frames until it can be received (each child frame is asked for once; finish after the last);
//      * n is the frame after the one served last (so also frame 0 first) without a live stream: a stream starts at
//        s0 = max(0, n - d) and its outputs s0 .. n-1 are received and dropped.  That is exact: stream output j is frame
//        s0 + j with its window clamped to [s0, N-1], the clip's own clamp whenever s0 = 0 or j >= d, and before finish
//        a batch only launches once its whole window has been sent;
//      * any other frame: the 2d+1 window frames are gathered into one pinned (or HBM) buffer and filtered by a one-frame
//        call, and the stream is dropped (its HBM freed).  A random read costs 2d+1 uploads this way; a stream restart
//        costs about 2d+2B.
//    Under the mirror's ConvertBits the frames come from ConvertBits' child and the stream (or the gather call) widens
//    them, so the host never widens a frame and each upload is at the source's size.  Under AviSynth+ the built-in
//    ConvertBits stays in charge and this filter streams the 14-bit frames it receives.
// ---------------------------------------------------------------------------------------------------------------
class KTemporalNR : public GenericVideoFilter, public IDeviceClip {
  amtk_ctx* ctx;
  amtk_tnr_params prm;
  std::shared_ptr<void> dev;          // filtered clip in HBM (device-resident child only)
  amtk_clip out;                      // ... and its descriptor
  bool fused = false;                 // dev was filtered from the clip under the child ConvertBits
  PClip src;                          // host path: the clip whose frames are filtered (ConvertBits' child under it)
  VideoInfo svi;                      // ... and its format
  std::shared_ptr<void> win;          // gather buffer of the generic path: 2d+1 frames
  size_t win_frame = 0; bool win_dev = false;
  static constexpr int kStreamBatch = 16;
  struct StreamRelease { void operator()(amtk_tnr_stream* s) const { amtk_tnr_stream_destroy(s); } };
  std::unique_ptr<amtk_tnr_stream, StreamRelease> stream;
  int next_send = 0, next_out = 0;    // clip frames: the next one to send to the stream, the next one it delivers
  std::deque<PVideoFrame> props;      // frame properties (no pixels) of the frames next_out .. next_send-1
  int last_n = -1;                    // the frame served last, and that frame
  PVideoFrame last;
  int sent = 0, gathered = 0;
  static void check(int ok) { if (!ok) throw AvisynthError(amtk_last_error()); }
  // filters the whole device-resident child once; false when the child is not device resident
  bool Resident() {
    if (dev) return true;
    amtk_clip src;
    av::ConvertBits* cb = dynamic_cast<av::ConvertBits*>(child.get());
    const bool widen = cb && cb->SourceDeviceClip(&src);
    if (!widen) {
      IDeviceClip* d = dynamic_cast<IDeviceClip*>(child.get());
      if (!d || !d->GetDeviceClip(&src)) return false;
    }
    void* p = nullptr;
    check(amtk_device_alloc(ctx, (size_t)PackedDeviceClip(vi, nullptr).frame_stride * vi.num_frames, &p));
    amtk_ctx* c = ctx;
    std::shared_ptr<void> own(p, [c](void* q) { amtk_device_free(c, q); });
    out = PackedDeviceClip(vi, p);
    check(amtk_tnr_frames(ctx, &src, &out, 0, &prm, 0, vi.num_frames));
    dev = own; fused = widen;
    return true;
  }
  PVideoFrame GatheredFrame(int n, IScriptEnvironment* env) {
    const int d = prm.temporal_distance, nf = 2 * d + 1;
    const PVideoFrame centre = src->GetFrame(n, env);
    const bool on_dev = centre->IsDevice();
    const size_t fb = (centre->TotalBytes() + 15) & ~(size_t)15;
    if (!win || win_frame != fb || win_dev != on_dev) {
      void* p = nullptr;
      amtk_check(on_dev ? amtk_device_alloc(ctx, fb * nf, &p) : amtk_host_alloc(fb * nf, &p), env);
      amtk_ctx* c = ctx;
      win = on_dev ? std::shared_ptr<void>(p, [c](void* q) { amtk_device_free(c, q); }) : std::shared_ptr<void>(p, [](void* q) { amtk_host_free(q); });
      win_frame = fb; win_dev = on_dev;
    }
    uint8_t* buf = static_cast<uint8_t*>(win.get());
    for (int i = 0; i < nf; ++i) {
      const int f = std::max(0, std::min(vi.num_frames - 1, n - d + i));
      PVideoFrame fr = f == n ? centre : src->GetFrame(f, env);
      if (fr->IsDevice() != on_dev || fr->TotalBytes() != centre->TotalBytes()) env->ThrowError("KTemporalNR: frames of the child differ in layout");
      if (on_dev) amtk_check(amtk_memcpy_d2d(ctx, buf + (size_t)i * fb, fr->Base(), fr->TotalBytes()), env);
      else memcpy(buf + (size_t)i * fb, fr->Base(), fr->TotalBytes());
    }
    amtk_clip sc = HostFrameClip(centre, svi);
    sc.base = buf; sc.frame_stride = (int64_t)fb; sc.num_frames = nf;
    PVideoFrame dst = env->NewVideoFrame(vi);
    amtk_clip dc = HostFrameClip(dst, vi);
    amtk_check(amtk_tnr_frames(ctx, &sc, &dc, 0, &prm, d, 1), env);    // window frame d is frame n; widens to vi's bits
    dst->CopyPropertiesFrom(*centre);
    ++gathered;
    return dst;
  }
  // A new stream whose next output is frame n: it starts at s0 = max(0, n - d) and outputs s0 .. n-1 are dropped.
  void StartStream(int n, IScriptEnvironment* env) {
    DropStream();
    const int out_bits = svi.BitsPerComponent() != vi.BitsPerComponent() ? vi.BitsPerComponent() : 0;
    amtk_tnr_stream* s = nullptr;
    amtk_check(amtk_tnr_stream_create_widening(ctx, &prm, out_bits, kStreamBatch, 0, &s), env);
    stream.reset(s);
    next_send = next_out = std::max(0, n - prm.temporal_distance);
    while (next_out < n) Pull(env);
  }
  void DropStream() { stream.reset(); props.clear(); }
  // The stream's next output (frame next_out) in a new CPU frame, sending the source's next frames until it comes.
  PVideoFrame Pull(IScriptEnvironment* env) {
    PVideoFrame dst = env->NewVideoFrame(vi);
    const amtk_clip dc = HostFrameClip(dst, vi);
    for (;;) {
      int32_t tag = -1; int got = 0;
      amtk_check(amtk_tnr_stream_recv(stream.get(), &dc, &tag, &got), env);
      if (got) {
        if (tag != next_out) env->ThrowError("KTemporalNR: the frame stream delivered frame %d for frame %d", (int)tag, next_out);
        break;
      }
      if (next_send >= vi.num_frames) env->ThrowError("KTemporalNR: the frame stream delivered no frame %d", next_out);
      const PVideoFrame f = src->GetFrame(next_send, env);
      const amtk_clip fc = HostFrameClip(f, svi);
      amtk_check(amtk_tnr_stream_send(stream.get(), &fc, next_send), env);
      PVideoFrame p = std::make_shared<VideoFrame>(VideoInfo());       // the properties, not the pixels
      p->CopyPropertiesFrom(*f);
      props.push_back(p);
      ++next_send; ++sent;
      if (next_send == vi.num_frames) amtk_check(amtk_tnr_stream_finish(stream.get()), env);
    }
    dst->CopyPropertiesFrom(*props.front());
    props.pop_front();
    ++next_out;
    return dst;
  }
  PVideoFrame HostFrame(int n, IScriptEnvironment* env) {
    if (last && n == last_n) return last;
    try {
      PVideoFrame f;
      if (stream && n == next_out) f = Pull(env);
      else if (n == last_n + 1) { StartStream(n, env); f = Pull(env); }
      else { DropStream(); f = GatheredFrame(n, env); }
      last_n = n; last = f;
      return f;
    } catch (...) {                   // a failed call leaves no half-fed stream behind
      DropStream(); last_n = -1; last.reset();
      throw;
    }
  }
public:
  KTemporalNR(PClip clip, int dist, int thresh, bool interlaced, IScriptEnvironment* env)
      : GenericVideoFilter(clip), ctx(env->GetAmtkContext()) {
    if (!ctx) env->ThrowError("KTemporalNR: no device bound to the script environment");
    prm.temporal_distance = dist; prm.threshold = thresh; prm.interlaced = interlaced ? 1 : 0;
    if (dist < 0 || dist > 63) env->ThrowError("KTemporalNR: dist must be in [0,63]");
    if (thresh < 0 || thresh > 65535) env->ThrowError("KTemporalNR: thresh must be in [0,65535]");
    av::ConvertBits* cb = dynamic_cast<av::ConvertBits*>(child.get());
    src = cb ? cb->Child() : child;
    svi = src->GetVideoInfo();
  }
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override {
    n = std::max(0, std::min(vi.num_frames - 1, n));
    if (!Resident()) return HostFrame(n, env);
    // fused: the properties come from the source frame, which ConvertBits would copy, so its widened clip is never made
    PVideoFrame s = fused ? static_cast<av::ConvertBits*>(child.get())->Child()->GetFrame(n, env) : child->GetFrame(n, env);
    PVideoFrame f = PackedDeviceFrame(vi, dev, n, env);
    f->CopyPropertiesFrom(*s);
    return f;
  }
  int FramesSent() const { return sent; }            // host path: frames sent to a frame stream
  int FramesGathered() const { return gathered; }    // host path: frames filtered from a gathered window
  bool GetDeviceClip(amtk_clip* c) override {
    if (!Resident()) return false;
    *c = out;
    return true;
  }
  int __stdcall SetCacheHints(int cachehints, int) override {
    if (cachehints == CACHE_GET_MTMODE) return MT_SERIALIZED;
    if (cachehints == CACHE_GET_DEV_TYPE) return DEV_TYPE_CPU | DEV_TYPE_CUDA;
    return 0;
  }
  static AVSValue __cdecl Create(AVSValue args, void*, IScriptEnvironment* env) {
    return AVSValue(PClip(new KTemporalNR(args[0].AsClip(), args[1].AsInt(3), args[2].AsInt(1), args[3].AsBool(false), env)));
  }
};

// ---------------------------------------------------------------------------------------------------------------
// AMTFilterSource (FilteredSource.hpp:214-300,417-544): the multi-pass filter driver.  Up to four passes; every pass
// builds a FRESH script environment (InitEnv), defines MakeSource(), sets AMT_SOURCE / AMT_TMP / AMT_PASS / AMT_DEV,
// runs the main filter script and asks whether it declared itself a pre-process (AMT_PRE_PROC); a pre-process pass is
// pulled frame by frame and discarded (ReadAllFrames), the first non-pre-process pass is the output.  Afterwards
// AMTDecimate is appended when the passes left a duration file, and the timecode file is read.
// AviSynth script text is replaced by a C++ callable with the same contract (reads the AMT_* variables, may set
// AMT_PRE_PROC, leaves the result in `last`); KFMVfrScript / KFMCfrScript are the two scripts Misc.cs generates.
// What is new on the GPU: the decoded clip is uploaded ONCE -- the environments of all passes share it through
// SharedClips -- where the reference re-opens and re-decodes the source in every pass (:441-447, InitEnv per pass).
// ---------------------------------------------------------------------------------------------------------------
struct EncodeFileKey { int video = 0; };
typedef std::function<void(IScriptEnvironment*)> FilterScript;

inline void KFMVfrScript(IScriptEnvironment* env) {                                       // Misc.cs:1305-1307,1315-1323
  const int AMT_PASS = env->GetVar("AMT_PASS").AsInt();
  static const int sel[3] = { 1, 2, 3 };
  const int pass = sel[std::max(0, std::min(2, AMT_PASS))];                              // pass = Select(AMT_PASS, 1, 2, 3)
  env->SetVar("AMT_PRE_PROC", AVSValue(AMT_PASS < 2));
  env->SetVar("last", env->Invoke("KFMDeint", AVSValue(std::vector<AVSValue>{ env->GetVar("AMT_SOURCE"), AVSValue(4), AVSValue(pass),
                                  AVSValue(std::string(env->GetVar("AMT_TMP").AsString())), env->GetVar("AMT_DEV") })));
}
inline void KFMCfrScript(IScriptEnvironment* env) {                                       // Misc.cs:1311-1313
  const int AMT_PASS = env->GetVar("AMT_PASS").AsInt();
  static const int sel[2] = { 1, 3 };
  const int pass = sel[std::max(0, std::min(1, AMT_PASS))];                              // pass = Select(AMT_PASS, 1, 3)
  env->SetVar("AMT_PRE_PROC", AVSValue(AMT_PASS < 1));
  env->SetVar("last", env->Invoke("KFMDeint", AVSValue(std::vector<AVSValue>{ env->GetVar("AMT_SOURCE"), AVSValue(2), AVSValue(pass),
                                  AVSValue(std::string(env->GetVar("AMT_TMP").AsString())), env->GetVar("AMT_DEV") })));
}

extern "C" inline const char* __stdcall AvisynthPluginInit3(IScriptEnvironment* env, const AVS_Linkage* const);

class AMTFilterSource {
public:
  struct PassInfo { int pass; bool preproc; int frames; double seconds; };

  AMTFilterSource(AMTContext& ctx, const ConfigWrapper& setting, amtk_ctx* device, int gpuIndex, EncodeFileKey key,
                  const tstring& logopath, FilterScript mainScript, FilterScript postScript = nullptr,
                  AvsDeviceType consumer = DEV_TYPE_CUDA, FilterScript envHook = nullptr)
      : ctx(ctx), setting_(setting), device_(device), consumer_(consumer), envHook_(envHook) {
    try {
      int pass = 0;
      for (; pass < 4; ++pass) {                                                         // :232-238
        if (!FilterPass(pass, gpuIndex, key, logopath, mainScript)) break;
        ReadAllFrames(pass);
      }
      // (after four pre-process passes the reference keeps the environment of the last one as the output, :257-275)
      if (postScript) { env_->SetVar("AMT_SOURCE", env_->GetVar("last")); postScript(env_.get()); }   // :257-261
      const tstring durationpath = setting_.getAvsDurationPath(key.video);               // :263-267
      if (FileExists(durationpath))
        env_->SetVar("last", env_->Invoke("AMTDecimate", AVSValue(std::vector<AVSValue>{ env_->GetVar("last"), AVSValue(durationpath) })));
      readTimecode(key);                                                                 // :269
      filter_ = env_->GetVar("last").AsClip();
      MakeOutFormat();
    } catch (const AvisynthError& avserror) {
      throw AviSynthException(avserror.msg);                                             // :289-295
    }
  }
  const PClip& getClip() const { return filter_; }
  IScriptEnvironment2* getEnv() const { return env_.get(); }
  const VideoInfo& getVideoInfo() const { return outvi_; }
  const std::vector<double>& getTimeCodes() const { return timeCodes_; }
  int getVfrTimingFps() const { return vfrTimingFps_; }
  const std::vector<PassInfo>& getPasses() const { return passes_; }
  int numSourceUploads() const { return (int)shared_.size(); }        // clips opened over ALL passes (1 = uploaded once)

private:
  AMTContext& ctx;
  const ConfigWrapper& setting_;
  amtk_ctx* device_;
  AvsDeviceType consumer_;
  FilterScript envHook_;                                // runs at the end of InitEnv (tests: replace AMTSource by a CPU clip)
  std::unique_ptr<IScriptEnvironment2> env_;
  std::map<std::string, PClip> shared_;                 // HBM-resident clips shared by the environments of all passes
  PClip filter_;
  VideoInfo outvi_;
  std::vector<double> timeCodes_;
  int vfrTimingFps_ = 0;
  std::vector<PassInfo> passes_;
  tstring logopath_;
  int video_ = 0;

  static bool FileExists(const tstring& p) { FILE* f = fopen(p.c_str(), "rb"); if (f) fclose(f); return f != nullptr; }

  void InitEnv() {                                                                       // :389-415
    env_.reset(new IScriptEnvironment2());
    BindDevice(env_.get(), device_, consumer_);
    env_->SetSharedClips(&shared_);
    av::AddBuiltins(env_.get());                         // what AviSynth+ itself provides (ConvertBits)
    AvisynthPluginInit3(env_.get(), nullptr);            // LoadPlugin(Amatsukaze.dll) :414
    if (envHook_) envHook_(env_.get());
  }

  // function MakeSource(bool "mt") (:441-475): AMTSource + the logo erasers; Prefetch and Trim belong to AviSynth / the
  // stream-reform stage and are not reproduced.
  static AVSValue __cdecl MakeSourceThunk(AVSValue, void* self, IScriptEnvironment* env) { return static_cast<AMTFilterSource*>(self)->MakeSource(env); }
  AVSValue MakeSource(IScriptEnvironment* env) {
    AVSValue last = env->Invoke("AMTSource", AVSValue(std::vector<AVSValue>{ AVSValue(setting_.getTmpAMTSourcePath(video_)) }));
    auto eraseLogo = [&](const tstring& logo, const tstring& logoFramePath, bool forceEnable) {
      if (!(forceEnable || FileExists(logoFramePath))) return;
      AVSValue analyze = env->Invoke("AMTAnalyzeLogo", AVSValue(std::vector<AVSValue>{ last, AVSValue(logo), AVSValue() }));
      last = env->Invoke("AMTEraseLogo", AVSValue(std::vector<AVSValue>{ last, analyze, AVSValue(logo), AVSValue(logoFramePath), AVSValue(),
                                                                          AVSValue(setting_.getMaxFadeLength()) }));
    };
    if (!setting_.isNoDelogo() && logopath_.size() > 0) eraseLogo(logopath_, setting_.getTmpLogoFramePath(video_), true);
    const auto& el = setting_.getEraseLogoPath();
    for (int i = 0; i < (int)el.size(); ++i) eraseLogo(el[i], setting_.getTmpLogoFramePath(video_, i), false);
    return last;
  }

  // returns: was this pass a pre-process?                                               (:519-544)
  bool FilterPass(int pass, int gpuIndex, EncodeFileKey key, const tstring& logopath, const FilterScript& mainScript) {
    InitEnv();
    logopath_ = logopath; video_ = key.video;
    env_->AddFunction("MakeSource", "[mt]b", MakeSourceThunk, this);
    env_->SetVar("AMT_SOURCE", env_->Invoke("MakeSource", AVSValue(true)));
    env_->SetVar("AMT_TMP", AVSValue(setting_.getAvsTmpPath(key.video)));
    env_->SetVar("AMT_PASS", AVSValue(pass));
    env_->SetVar("AMT_DEV", AVSValue(gpuIndex));
    env_->SetVar("last", env_->GetVar("AMT_SOURCE"));
    if (mainScript) mainScript(env_.get());
    return env_->GetVarDef("AMT_PRE_PROC", AVSValue(false)).AsBool();
  }

  void ReadAllFrames(int pass) {                                                         // :417-439
    PClip clip = env_->GetVar("last").AsClip();
    const VideoInfo vi = clip->GetVideoInfo();
    ctx.infoF("filter pass %d: %d frames", pass + 1, vi.num_frames);
    struct timespec t0, t1; clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int i = 0; i < vi.num_frames; ++i) PVideoFrame frame = clip->GetFrame(i, env_.get());
    clock_gettime(CLOCK_MONOTONIC, &t1);
    passes_.push_back(PassInfo{ pass, true, vi.num_frames, (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec) });
  }

  void readTimecode(EncodeFileKey key) {                                                 // :189-212
    const tstring timecodepath = setting_.getAvsTimecodePath(key.video);
    if (!FileExists(timecodepath)) return;
    TimecodeFile tc;
    if (tc.read(timecodepath)) { timeCodes_ = tc.timeCodes; vfrTimingFps_ = tc.vfrTimingFps; }
  }
  void MakeOutFormat() { outvi_ = filter_->GetVideoInfo(); }                             // :600-612 (format bookkeeping only)
};

// ---------------------------------------------------------------------------------------------------------------
// CMAnalyze (CMAnalyze.hpp:22-317) -- the logo-analysis half only: the constructor runs logoFrame() when logos are
// configured and exposes getLogoPath().  chapter_exe / join_logo_scp subprocesses, Trim/zone parsing (:319-679) are
// out of scope (SURVEY section 8).  ConfigWrapper is reduced to the accessors logoFrame() reads.
// ---------------------------------------------------------------------------------------------------------------


class CMAnalyze {
public:
  // env must have the plugin registered (AvisynthPluginInit3) and an amtk context bound; the reference creates its
  // own script environment and loads itself as a plugin (:275-280) -- on the GPU build the caller owns the device.
  // combStatsPath: empty (the default) runs the logo analysis alone.  Otherwise the same pass over the source also makes
  // the combing counters of the telecine pre-pass (LogoFrame::scanFrames with counts) and writes them to that file, in
  // AMTCombAnalyze's format: one decode serves both.  The logoframe files are the same either way.
  CMAnalyze(AMTContext& ctx, const ConfigWrapper& setting, int videoFileIndex, int /*numFrames*/, IScriptEnvironment2* env,
            const tstring& combStatsPath = tstring())
      : ctx(ctx), setting_(setting), combStatsPath_(combStatsPath) {
    if (setting_.getLogoPath().size() > 0 || setting_.getEraseLogoPath().size() > 0) {                        // :34
      ctx.info("[logo analysis]");
      logoFrame(videoFileIndex, env);
      if (logopath.size() > 0) ctx.infoF("matched logo: %s", logopath.c_str());
    }
  }
  const tstring& getLogoPath() const { return logopath; }
  float getLogoRatio() const { return logoRatio; }
private:
  AMTContext& ctx;
  const ConfigWrapper& setting_;
  const tstring combStatsPath_;
  tstring logopath;
  float logoRatio = 0.0f;

  void logoFrame(int videoFileIndex, IScriptEnvironment2* env) {                                              // :273-317
    try {
      PClip clip = env->Invoke("AMTSource", AVSValue(std::vector<AVSValue>{ AVSValue(setting_.getTmpAMTSourcePath(videoFileIndex)) })).AsClip();
      const VideoInfo vi = clip->GetVideoInfo();
      const int duration = (int)((int64_t)vi.num_frames * vi.fps_denominator / vi.fps_numerator);
      const auto& logoPath = setting_.getLogoPath();
      const auto& eraseLogoPath = setting_.getEraseLogoPath();
      std::vector<tstring> allLogoPath = logoPath;
      allLogoPath.insert(allLogoPath.end(), eraseLogoPath.begin(), eraseLogoPath.end());
      logo::LogoFrame logof(ctx, allLogoPath, 0.35f);
      if (combStatsPath_.empty()) {
        logof.scanFrames(clip, env);                     // ONE batched device pass for all logos
      } else {                                           // ... that also makes the pre-pass's combing counters
        amtk_comb_params prm;
        amtk_comb_default_params(&prm);
        std::vector<int32_t> counts;
        logof.scanFrames(clip, env, prm, counts);
        WriteCombStats(combStatsPath_, counts, vi.num_frames, "CMAnalyze", env);
      }
      if (logoPath.size() > 0) {
        logof.selectLogo((int)logoPath.size());
        logof.writeResult(setting_.getTmpLogoFramePath(videoFileIndex));
        logoRatio = logof.getLogoRatio();
        const float threshold = setting_.isLooseLogoDetection() ? 0.03f : (duration <= 60 * 7) ? 0.03f : 0.1f;
        if (logoRatio < threshold) ctx.info("no logo matched in this section");
        else logopath = setting_.getLogoPath()[logof.getBestLogo()];
      }
      for (int i = 0; i < (int)eraseLogoPath.size(); ++i)
        logof.writeResult(setting_.getTmpLogoFramePath(videoFileIndex, i), (int)logoPath.size() + i);
    } catch (const AvisynthError& avserror) {
      throw AviSynthException(avserror.msg);                                                                  // :314-316
    }
  }
};

// Registration with the reference's names and argument specs (Amatsukaze.cpp:43-66).
extern "C" inline const char* __stdcall AvisynthPluginInit3(IScriptEnvironment* env, const AVS_Linkage* const) {
  env->AddFunction("AMTSource", "s[filter]s[outqp]b", av::CreateAMTSource, 0);
  env->AddFunction("AMTAnalyzeLogo", "cs[maskratio]i", logo::AMTAnalyzeLogo::Create, 0);
  env->AddFunction("AMTEraseLogo", "ccs[logof]s[mode]i[maxfade]i", logo::AMTEraseLogo::Create, 0);
  env->AddFunction("AMTDecimate", "c[duration]s", AMTDecimate::Create, 0);
  env->AddFunction("AMTCombAnalyze", "c[filepath]s", AMTCombAnalyze::Create, 0);
  env->AddFunction("KFMDeint", "c[mode]i[pass]i[filepath]s[dev]i", CreateKFMDeint, 0);      // pass protocol only (see CreateKFMDeint)
  env->AddFunction("KTemporalNR", "c[dist]i[thresh]i[interlaced]b", KTemporalNR::Create, 0); // the reference's TemporalNRFilter (see KTemporalNR)
  return "Amatsukaze plugin (H100 hot path)";
}
