// avs_compat.h -- a Linux-compilable, signature-compatible SUBSET of the AviSynth(Neo) filter interface the
// reference's filters are written against (reference: include/avisynth.h -- IClip :1120-1136, PClip, PVideoFrame
// :987-1007, VideoInfo, GenericVideoFilter :1288-1299, IScriptEnvironment :1400-1470, AVSValue, AvisynthError :127-134).
//
// The reference's header is MSVC-only (__int64, __stdcall, baked AVS_Linkage thunks) and there is no AviSynth
// runtime on Linux, so the GPU filters (filters.hpp) are written against this subset: same class and method names,
// argument order and error behaviour, so the filter sources read like reference-compatible plugins.
// Independent implementation; nothing here is copied from avisynth.h.
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#ifndef __stdcall
#define __stdcall
#endif
#ifndef __cdecl
#define __cdecl
#endif

struct amtk_ctx;

enum { PLANAR_Y = 1 << 0, PLANAR_U = 1 << 1, PLANAR_V = 1 << 2 };
enum { CACHE_GET_MTMODE = 509,                         // the requests the reference's filters answer ...
       CACHE_GET_DEV_TYPE = 518,                       // ... plus AviSynthNeo's device hooks (include/avisynth.h:1112-1113):
       CACHE_GET_CHILD_DEV_TYPE = 519 };               // which device a filter returns frames on / accepts frames from
enum AvsDeviceType { DEV_TYPE_NONE = 0, DEV_TYPE_CPU = 1, DEV_TYPE_CUDA = 2, DEV_TYPE_ANY = 0xFFFF };   // include/avisynth.h:137-141
enum MtMode { MT_INVALID = 0, MT_NICE_FILTER = 1, MT_MULTI_INSTANCE = 2, MT_SERIALIZED = 3 };

struct AvisynthError {                                  // thrown by IScriptEnvironment::ThrowError
  std::string msg;
  explicit AvisynthError(const std::string& m) : msg(m) {}
};

struct VideoInfo {
  enum { CS_UNKNOWN = 0, CS_YV12 = 1, CS_YUV420P10 = 2, CS_YUV420P12 = 3, CS_YUV420P16 = 4, CS_BGR32 = 5, CS_YUV420P14 = 6 };
  int width = 0, height = 0;
  unsigned fps_numerator = 30000, fps_denominator = 1001;
  int num_frames = 0;
  int pixel_type = CS_UNKNOWN;
  bool HasVideo() const { return width != 0; }
  bool IsPlanar() const { return (pixel_type >= CS_YV12 && pixel_type <= CS_YUV420P16) || pixel_type == CS_YUV420P14; }
  int BitsPerComponent() const {
    switch (pixel_type) {
      case CS_YUV420P10: return 10; case CS_YUV420P12: return 12; case CS_YUV420P14: return 14; case CS_YUV420P16: return 16;
      default: return 8;
    }
  }
  int ComponentSize() const { return pixel_type == CS_BGR32 ? 1 : (BitsPerComponent() > 8 ? 2 : 1); }
  int GetPlaneWidthSubsampling(int plane) const { return (plane == PLANAR_Y || !IsPlanar()) ? 0 : 1; }
  int GetPlaneHeightSubsampling(int plane) const { return (plane == PLANAR_Y || !IsPlanar()) ? 0 : 1; }
  int BytesFromPixels(int pixels) const { return pixel_type == CS_BGR32 ? pixels * 4 : pixels * ComponentSize(); }
};

// One frame: planar Y,U,V (or a single packed plane for CS_BGR32).  Either in host memory (rows 64-byte aligned, owned)
// or -- the AviSynthNeo DEV_TYPE_CUDA case, include/avisynth.h:1651-1652 NewVideoFrame(vi, device) -- a VIEW of memory in
// HBM (IsDevice(): the pointers returned by GetReadPtr/GetWritePtr are device pointers; `owner` keeps the allocation
// alive).  Frame properties (SetProperty/GetProperty, include/avisynth.h:1009-1017) carry FrameType etc.
class VideoFrame {
  std::vector<uint8_t> buf_;
  uint8_t* dev_ = nullptr;                 // non-null: device frame (view)
  size_t dev_bytes_ = 0;
  std::shared_ptr<void> owner_;
  std::map<std::string, double> props_;
  int pitch_[3] = { 0, 0, 0 }, rowsize_[3] = { 0, 0, 0 }, height_[3] = { 0, 0, 0 };
  size_t off_[3] = { 0, 0, 0 };
  static int idx(int plane) { return plane == PLANAR_U ? 1 : (plane == PLANAR_V ? 2 : 0); }
public:
  // device view: tightly described by per-plane offsets and pitches inside [base, base + bytes)
  VideoFrame(const VideoInfo& vi, uint8_t* dev_base, size_t bytes, const size_t off[3], const int pitch[3], std::shared_ptr<void> owner)
      : dev_(dev_base), dev_bytes_(bytes), owner_(owner) {
    for (int p = 0; p < 3; ++p) {
      const int w = p ? vi.width >> 1 : vi.width, h = p ? vi.height >> 1 : vi.height;
      rowsize_[p] = vi.BytesFromPixels(w); pitch_[p] = pitch[p]; height_[p] = h; off_[p] = off[p];
    }
  }
  bool IsDevice() const { return dev_ != nullptr; }
  void Rebase(uint8_t* dev_base, std::shared_ptr<void> owner) { dev_ = dev_base; owner_ = owner; }   // same geometry, other memory
  void SetProperty(const char* key, double v) { props_[key] = v; }
  double GetProperty(const char* key, double def) const { auto it = props_.find(key); return it == props_.end() ? def : it->second; }
  int GetProperty(const char* key, int def) const { auto it = props_.find(key); return it == props_.end() ? def : (int)it->second; }
  void CopyPropertiesFrom(const VideoFrame& o) { props_ = o.props_; }
  explicit VideoFrame(const VideoInfo& vi) {
    const int planes = vi.IsPlanar() ? 3 : 1;
    size_t total = 0;
    for (int p = 0; p < planes; ++p) {
      const int w = p ? vi.width >> 1 : vi.width, h = p ? vi.height >> 1 : vi.height;
      rowsize_[p] = vi.BytesFromPixels(w);
      pitch_[p] = (rowsize_[p] + 63) & ~63;
      height_[p] = h;
      off_[p] = total;
      total += (size_t)pitch_[p] * h;
    }
    buf_.assign(total + 64, 0);
  }
  int GetPitch(int plane = PLANAR_Y) const { return pitch_[idx(plane)]; }
  int GetRowSize(int plane = PLANAR_Y) const { return rowsize_[idx(plane)]; }
  int GetHeight(int plane = PLANAR_Y) const { return height_[idx(plane)]; }
  const uint8_t* GetReadPtr(int plane = PLANAR_Y) const { return Base() + off_[idx(plane)]; }
  uint8_t* GetWritePtr(int plane = PLANAR_Y) { return const_cast<uint8_t*>(Base()) + off_[idx(plane)]; }
  size_t GetOffset(int plane) const { return off_[idx(plane)]; }
  const uint8_t* Base() const { return dev_ ? dev_ : buf_.data(); }
  size_t TotalBytes() const { return dev_ ? dev_bytes_ : buf_.size() - 64; }
};
typedef std::shared_ptr<VideoFrame> PVideoFrame;

class IScriptEnvironment;
class AVSValue;

class IClip {                                            // base class of all filters (include/avisynth.h:1120-1136)
public:
  virtual ~IClip() {}
  virtual PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) = 0;
  virtual bool __stdcall GetParity(int n) = 0;
  virtual void __stdcall GetAudio(void* buf, int64_t start, int64_t count, IScriptEnvironment* env) = 0;
  virtual int __stdcall SetCacheHints(int cachehints, int frame_range) = 0;
  virtual const VideoInfo& __stdcall GetVideoInfo() = 0;
};
typedef std::shared_ptr<IClip> PClip;

class GenericVideoFilter : public IClip {                // include/avisynth.h:1288-1299
protected:
  PClip child;
  VideoInfo vi;
public:
  explicit GenericVideoFilter(PClip c) : child(c), vi(c->GetVideoInfo()) {}
  PVideoFrame __stdcall GetFrame(int n, IScriptEnvironment* env) override { return child->GetFrame(n, env); }
  void __stdcall GetAudio(void* buf, int64_t start, int64_t count, IScriptEnvironment* env) override { child->GetAudio(buf, start, count, env); }
  const VideoInfo& __stdcall GetVideoInfo() override { return vi; }
  bool __stdcall GetParity(int n) override { return child->GetParity(n); }
  int __stdcall SetCacheHints(int, int) override { return 0; }
};

class AVSValue {                                         // tagged value passed to filter factories
  char type_ = 'v';
  PClip clip_; std::string str_; int i_ = 0; double f_ = 0; std::vector<AVSValue> arr_;
public:
  AVSValue() {}
  AVSValue(PClip c) : type_('c'), clip_(c) {}
  AVSValue(IClip* c) : type_('c'), clip_(c) {}
  AVSValue(const char* s) : type_('s'), str_(s) {}
  AVSValue(const std::string& s) : type_('s'), str_(s) {}
  AVSValue(int i) : type_('i'), i_(i) {}
  AVSValue(bool b) : type_('b'), i_(b) {}
  AVSValue(double f) : type_('f'), f_(f) {}
  AVSValue(const std::vector<AVSValue>& a) : type_('a'), arr_(a) {}
  bool Defined() const { return type_ != 'v'; }
  bool IsClip() const { return type_ == 'c'; }
  bool IsString() const { return type_ == 's'; }
  bool IsArray() const { return type_ == 'a'; }
  PClip AsClip() const { return clip_; }
  const char* AsString() const { return str_.c_str(); }
  const char* AsString(const char* def) const { return type_ == 's' ? str_.c_str() : def; }
  int AsInt() const { return type_ == 'f' ? (int)f_ : i_; }
  int AsInt(int def) const { return (type_ == 'i' || type_ == 'b') ? i_ : (type_ == 'f' ? (int)f_ : def); }
  double AsFloat() const { return type_ == 'f' ? f_ : (double)i_; }
  double AsFloat(double def) const { return type_ == 'f' ? f_ : ((type_ == 'i') ? (double)i_ : def); }
  bool AsBool() const { return i_ != 0; }
  bool AsBool(bool def) const { return type_ == 'b' || type_ == 'i' ? i_ != 0 : def; }
  int ArraySize() const { return type_ == 'a' ? (int)arr_.size() : 1; }
  const AVSValue& operator[](int i) const { static const AVSValue none; return type_ == 'a' ? (i < (int)arr_.size() ? arr_[i] : none) : *this; }
};

class IScriptEnvironment {
public:
  typedef AVSValue(__cdecl* ApplyFunc)(AVSValue args, void* user_data, IScriptEnvironment* env);
  virtual ~IScriptEnvironment() {}
  void ThrowError(const char* fmt, ...) {
    char buf[1024];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    throw AvisynthError(buf);
  }
  virtual PVideoFrame NewVideoFrame(const VideoInfo& vi) { return std::make_shared<VideoFrame>(vi); }
  virtual bool MakeWritable(PVideoFrame* pvf) {
    if ((*pvf)->IsDevice()) return MakeWritableDevice(pvf);
    if (pvf->use_count() == 1) return false;
    *pvf = std::make_shared<VideoFrame>(**pvf);         // full-frame copy, as AviSynth does (LogoScan.hpp:1347)
    return true;
  }
  // device frames: a private HBM copy (device-to-device), provided by the binding layer (filters.hpp)
  std::function<bool(PVideoFrame*)> MakeWritableDevice = [](PVideoFrame*) { return false; };
  // AviSynthNeo: which device the consumer of this environment's frames runs on (INeoEnv::GetDeviceType,
  // include/avisynth.h:1700).  DEV_TYPE_CUDA lets device-resident sources hand out zero-copy frame views.
  virtual AvsDeviceType GetDeviceType() const { return dev_type_; }
  void SetDeviceType(AvsDeviceType t) { dev_type_ = t; }
  // Clips that outlive one script environment (AMTFilterSource builds a fresh environment per pass,
  // FilteredSource.hpp:519-523; the decoded clip stays resident in HBM across passes through this table).
  std::map<std::string, std::shared_ptr<IClip>>* SharedClips() { return shared_clips_; }
  void SetSharedClips(std::map<std::string, std::shared_ptr<IClip>>* m) { shared_clips_ = m; }
  // name, parameter spec ("cs[maskratio]i" ...), factory, user data -- Amatsukaze.cpp:55-63
  virtual void AddFunction(const char* name, const char* params, ApplyFunc apply, void* user_data) {
    funcs_[name] = Func{ params, apply, user_data };
  }
  virtual bool FunctionExists(const char* name) { return funcs_.count(name) != 0; }
  virtual const char* FunctionParams(const char* name) { auto it = funcs_.find(name); return it == funcs_.end() ? nullptr : it->second.params.c_str(); }
  virtual AVSValue Invoke(const char* name, const AVSValue args) {
    auto it = funcs_.find(name);
    if (it == funcs_.end()) ThrowError("Script error: there is no function named '%s'", name);
    return it->second.apply(args, it->second.user_data, this);
  }
  // script variables (AMT_SOURCE, AMT_TMP, AMT_PASS, AMT_DEV ... FilteredSource.hpp:530-540)
  virtual bool SetVar(const char* name, const AVSValue& v) { vars_[name] = v; return true; }
  virtual AVSValue GetVarDef(const char* name, const AVSValue& def = AVSValue()) { auto it = vars_.find(name); return it == vars_.end() ? def : it->second; }
  virtual AVSValue GetVar(const char* name) { auto it = vars_.find(name); if (it == vars_.end()) ThrowError("Script error: no variable named '%s'", name); return it->second; }
  // device binding: analogue of INeoEnv::GetDevice/GetDeviceStream (include/avisynth.h:1698-1706)
  virtual amtk_ctx* GetAmtkContext() { return amtk_; }
  void SetAmtkContext(amtk_ctx* c) { amtk_ = c; }
private:
  struct Func { std::string params; ApplyFunc apply; void* user_data; };
  std::map<std::string, Func> funcs_;
  std::map<std::string, AVSValue> vars_;
  amtk_ctx* amtk_ = nullptr;
  AvsDeviceType dev_type_ = DEV_TYPE_CPU;
  std::map<std::string, std::shared_ptr<IClip>>* shared_clips_ = nullptr;
};
typedef IScriptEnvironment IScriptEnvironment2;

struct AVS_Linkage;   // opaque; present only so that AvisynthPluginInit3 keeps its signature (Amatsukaze.cpp:43)
