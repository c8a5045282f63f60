// logo_host.h -- host-side logo model: what logo::LogoData / logo::LogoDataParam hold on the CPU in the reference
// (AMTLogo.hpp:49-280, LogoScan.hpp:61-334).  Setup-time only (once per logo); the per-frame work is on the GPU.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace amtk {

struct LgdHeader {          // logo::LogoHeader, AMTLogo.hpp:19-47 (540 bytes, no padding)
  int32_t magic, version;
  int32_t w, h, logUVx, logUVy;
  int32_t imgw, imgh, imgx, imgy;
  char name[255];
  // 1 byte of natural padding follows name[] so that serviceId is 4-aligned
  int32_t serviceId;
  int32_t reserved[60];
};
static_assert(sizeof(LgdHeader) == 540, "LgdHeader must match the reference's LogoHeader");

struct HostLogo {
  int w = 0, h = 0, logUVx = 1, logUVy = 1;
  int imgw = 0, imgh = 0, imgx = 0, imgy = 0;
  std::vector<float> data;          // aY,bY,aU,bU,aV,bV
  // evaluation tables (empty until create_mask)
  std::vector<uint8_t> mask;        // w*h
  int maskpixels = 0;
  std::vector<uint32_t> pix;        // visited mask pixels in scan order: x | y<<16
  std::vector<float> kernels;       // count*25 zero-mean taps
  std::vector<float> scales;        // count*32*{scale,scale2}
  float blackScore = 0.0f;

  int wUV() const { return w >> logUVx; }
  int hUV() const { return h >> logUVy; }
  size_t ySize() const { return (size_t)w * h; }
  size_t cSize() const { return (size_t)wUV() * hUV(); }
  size_t dataSize() const { return (ySize() + 2 * cSize()) * 2; }
  float* aY() { return data.data(); }
  float* bY() { return aY() + ySize(); }
  float* aU() { return bY() + ySize(); }
  float* bU() { return aU() + cSize(); }
  float* aV() { return bU() + cSize(); }
  float* bV() { return aV() + cSize(); }
  const float* aY() const { return data.data(); }
  const float* bY() const { return aY() + ySize(); }
  const float* aU() const { return bY() + ySize(); }
  const float* bU() const { return aU() + cSize(); }
  const float* aV() const { return bU() + cSize(); }
  const float* bV() const { return aV() + cSize(); }
  int count() const { return (int)pix.size(); }

  void init(int w_, int h_, int lx, int ly, int iw, int ih, int ix, int iy);
};

void logo_deint(const HostLogo& src, HostLogo& dst);                 // DeintLogo, LogoScan.hpp:734-761
void logo_field(const HostLogo& src, bool bottom, HostLogo& dst);    // MakeFieldLogo, LogoScan.hpp:257-283
void logo_create_mask(HostLogo& l, float maskratio);                 // CreateLogoMask, LogoScan.hpp:112-229
float logo_corr_score_host(const HostLogo& l, const float* work);    // CorrelationScore, LogoScan.hpp:288-318
bool lgd_load(const std::string& path, HostLogo& out, LgdHeader* hdr, std::string& err);   // AMTLogo.hpp:257-279
bool lgd_save(const HostLogo& l, const std::string& path, const std::string& name, int serviceId, std::string& err);  // :239-255

// LogoColor::Normalize + GetAB over all pixels, LogoScan::GetLogo incl. `clean` (LogoScan.hpp:367-395,471-566).
// sums: plane-major Y,U,V, 5 doubles per pixel.  Returns false when the reference returns nullptr.
// With `clean` and a scanw or scanh that is not a multiple of the subsampling, the last luma column or row maps to a
// chroma index past the chroma planes; those pixels skip their chroma reads and writes (the reference reads and writes
// outside its planes there), so nothing past out_data's end is touched.
bool scan_finalize(const double* sums, int nframes, int scanw, int scanh, int logUVx, int logUVy,
                   int maxv, bool clean, float* out_data);

// AMTEraseLogo::CalcFade2 (LogoScan.hpp:1263-1315); calc_fade2_index / calc_fade2_records come from fade_select.h
void calc_fade2(const float* records, int num_records, int num_frames, int n, float* fadeT, float* fadeB);

// The logo finder's rectangle rule (DESIGN.md section 3.5) on per-pixel sums s1 = sum Y, s2 = sum Y*Y over nframes
// frames of a width x height luma plane at `bits` bits; best first.
struct FoundRect { int x, y, w, h; float score; };
void find_logo_rects(const uint64_t* s1, const uint64_t* s2, int64_t nframes, int width, int height, int bits, int block,
                     float var_ratio, float mean_delta, int margin, int min_blocks, std::vector<FoundRect>* out);

}  // namespace amtk

#include "fade_select.h"
