// logo_host.cpp -- host-side logo preparation (compiled with -ffp-contract=off, no fast-math).
// Everything here runs once per logo (or once per finished scan); the per-frame hot path is CUDA.
#include "logo_host.h"
#include "exact_math.h"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>

namespace amtk {

namespace {
constexpr int kTaps = 25;     // 5x5 window (LogoDataParam::KLEN, LogoScan.hpp:63-66)
constexpr int kBins = 32;     // 256 >> 3 flat-background bins (CLEN, LogoScan.hpp:67-68)

struct PlaneView {            // row accessor handed to corr5x5_tree
  const float* base; int stride;
  float operator()(int dy, int dx) const { return base[dy * stride + dx]; }
};

// 5x5 neighbourhood of (x,y), mean removed: the "logo kernel" of one feature pixel (LogoScan.hpp:135-147).
void zero_mean_window(const float* img, int stride, int x, int y, float* k) {
  int t = 0;
  for (int dy = -2; dy <= 2; ++dy)
    for (int dx = -2; dx <= 2; ++dx) k[t++] = img[(x + dx) + (y + dy) * stride];
  float s = 0.0f;
  for (int i = 0; i < kTaps; ++i) s = s + k[i];
  const float mean = s / kTaps;
  for (int i = 0; i < kTaps; ++i) k[i] = k[i] - mean;
}
}  // namespace

void HostLogo::init(int w_, int h_, int lx, int ly, int iw, int ih, int ix, int iy) {
  w = w_; h = h_; logUVx = lx; logUVy = ly; imgw = iw; imgh = ih; imgx = ix; imgy = iy;
  data.assign(dataSize(), 0.0f);
  mask.clear(); pix.clear(); kernels.clear(); scales.clear(); maskpixels = 0; blackScore = 0.0f;
}

void logo_deint(const HostLogo& s, HostLogo& d) {
  d.init(s.w, s.h, s.logUVx, s.logUVy, s.imgw, s.imgh, s.imgx, s.imgy);
  const int w = s.w, h = s.h;
  const float* srcs[2] = { s.aY(), s.bY() };
  float* dsts[2] = { d.aY(), d.bY() };
  for (int p = 0; p < 2; ++p) {
    const float* in = srcs[p]; float* out = dsts[p];
    std::copy(in, in + w, out);                                             // first row
    std::copy(in + (size_t)(h - 1) * w, in + (size_t)h * w, out + (size_t)(h - 1) * w);   // last row
    for (int y = 1; y < h - 1; ++y)
      for (int x = 0; x < w; ++x)
        out[x + y * w] = (in[x + (y - 1) * w] + 2 * in[x + y * w] + in[x + (y + 1) * w]) / 4.0f;
  }
  // chroma of a deint logo is never read by the evaluation path (the reference leaves it uninitialised)
}

void logo_field(const HostLogo& s, bool bottom, HostLogo& f) {
  f.init(s.w, s.h / 2, s.logUVx, s.logUVy, s.imgw, s.imgh / 2, s.imgx, s.imgy / 2);
  const int w = s.w, b = bottom ? 1 : 0;
  for (int y = 0; y < f.h; ++y) {
    std::copy(s.aY() + (size_t)(b + 2 * y) * w, s.aY() + (size_t)(b + 2 * y + 1) * w, f.aY() + (size_t)y * w);
    std::copy(s.bY() + (size_t)(b + 2 * y) * w, s.bY() + (size_t)(b + 2 * y + 1) * w, f.bY() + (size_t)y * w);
  }
  const int uvOff = b ^ (f.imgy % 2);
  const int wc = f.wUV(), hc = f.hUV();
  const float* cs[4] = { s.aU(), s.bU(), s.aV(), s.bV() };
  float* cd[4] = { f.aU(), f.bU(), f.aV(), f.bV() };
  for (int p = 0; p < 4; ++p)
    for (int y = 0; y < hc; ++y)
      std::copy(cs[p] + (size_t)(uvOff + 2 * y) * wc, cs[p] + (size_t)(uvOff + 2 * y + 1) * wc, cd[p] + (size_t)y * wc);
}

float logo_corr_score_host(const HostLogo& l, const float* work) {
  float total = 0.0f;
  const int n = l.count();
  for (int c = 0; c < n; ++c) {
    const int x = (int)(l.pix[c] & 0xFFFFu), y = (int)(l.pix[c] >> 16);
    float avg;
    PlaneView v{ work + (x - 2) + (size_t)(y - 2) * l.w, l.w };
    const float sum = corr5x5_tree(&l.kernels[(size_t)c * kTaps], v, &avg);
    const float* sc = &l.scales[((size_t)c * kBins + scale_bin(avg)) * 2];
    total = total + pixel_score(sum, sc[0], sc[1]);      // sequential float sum (LogoScan.hpp:310)
  }
  return total;
}

void logo_create_mask(HostLogo& l, float maskratio) {
  const int w = l.w, h = l.h, npx = w * h;
  // 32 flat backgrounds (grey = bin<<3) with the logo painted on: Y = (Y - b*255)/a where a>0
  // (LogoScan.hpp:128-133 + AddLogo :320-333).
  std::vector<float> slices((size_t)npx * kBins + 8, 0.0f);
  const float* A = l.aY(); const float* B = l.bY();
  const int maxv = 255;
  for (int bin = 0; bin < kBins; ++bin) {
    float* sl = &slices[(size_t)bin * npx];
    const float grey = (float)(bin << 3);
    for (int i = 0; i < npx; ++i) {
      float v = grey;
      if (A[i] > 0) v = (v - B[i] * maxv) / A[i];
      sl[i] = v;
    }
  }
  // feature strength = energy of the zero-mean 5x5 window on the mid-grey slice (LogoScan.hpp:152-163)
  struct Cand { float energy; int index; };
  std::vector<Cand> cand((size_t)npx);
  for (int i = 0; i < npx; ++i) cand[i] = { 0.0f, i };
  const float* mid = &slices[(size_t)(kBins / 2) * npx];
  for (int y = 2; y < h - 2; ++y)
    for (int x = 2; x < w - 2; ++x) {
      float k[kTaps];
      zero_mean_window(mid, w, x, y, k);
      float e = 0.0f;
      for (int i = 0; i < kTaps; ++i) e = e + k[i] * k[i];
      cand[x + y * w].energy = e;
    }
  // strongest first; ties resolved towards the HIGHER pixel index (std::greater<pair<float,int>>, :169)
  std::sort(cand.begin(), cand.end(), [](const Cand& a, const Cand& b) {
    if (a.energy != b.energy) return a.energy > b.energy;
    return a.index > b.index;
  });
  l.maskpixels = std::min(npx, (int)(npx * maskratio));
  l.mask.assign((size_t)npx, 0);
  for (int i = 0; i < l.maskpixels; ++i) l.mask[cand[i].index] = 1;

  // per-feature kernels (from the black slice) and their response on every flat background (:188-200)
  l.pix.clear(); l.kernels.clear(); l.scales.clear();
  float corrTotal = 0.0f;
  for (int y = 2; y < h - 2; ++y)
    for (int x = 2; x < w - 2; ++x) {
      if (!l.mask[x + y * w]) continue;
      float k[kTaps];
      zero_mean_window(slices.data(), w, x, y, k);
      l.pix.push_back((uint32_t)x | ((uint32_t)y << 16));
      l.kernels.insert(l.kernels.end(), k, k + kTaps);
      for (int bin = 0; bin < kBins; ++bin) {
        float avg;
        PlaneView v{ &slices[(size_t)bin * npx] + (x - 2) + (size_t)(y - 2) * w, w };
        const float r = std::fabs(corr5x5_tree(k, v, &avg));
        l.scales.push_back(r);       // raw response for now
        l.scales.push_back(0.0f);
        corrTotal += r;
      }
    }
  // NOTE the divisor is maskpixels, not the number of visited features (LogoScan.hpp:202)
  const float corrMean = corrTotal / (l.maskpixels * kBins);
  const float corrFloor = corrMean * 0.2f;                 // corrLowerLimit, :121,204
  for (size_t i = 0; i < l.scales.size(); i += 2) {
    const float r = l.scales[i];
    l.scales[i] = (r > 0) ? (1.0f / r) : 0.0f;             // normalising scale (:207)
    l.scales[i + 1] = std::min(1.0f, r / corrFloor);       // cap for weak features (:208)
  }
  // response of the bare logo on a near-black (16) background is the unit of all scores (:227-228)
  l.blackScore = logo_corr_score_host(l, &slices[(size_t)(16 >> 3) * npx]);
}

// ---------------------------------------------------------------------------------------------------
// .lgd files (include/logo.h:31-89 + AMTLogo.hpp:169-279)
// ---------------------------------------------------------------------------------------------------
namespace {
#pragma pack(push, 1)
struct LgdFileHeader { char tag[28]; uint8_t count_be[4]; };                      // LOGO_FILE_HEADER (32 B)
struct LgdBaseHeader { char name[32]; int16_t x, y, h, w, fi, fo, st, ed; };      // LOGO_HEADER (48 B)
struct LgdBasePixel { int16_t dp_y, y, dp_cb, cb, dp_cr, cr; };                    // LOGO_PIXEL (12 B)
#pragma pack(pop)
static_assert(sizeof(LgdFileHeader) == 32 && sizeof(LgdBaseHeader) == 48 && sizeof(LgdBasePixel) == 12, "lgd layout");
const char kLgdTag[] = "<logo data file ver0.1>";
constexpr int kMaxDp = 1000;                                                       // LOGO_MAX_DP

// YV12 <-> AviUtl YC48 conversions used only to derive the AviUtl-compatible base part (AMTLogo.hpp:58-94)
float yc48_from_yv12_y(float y) { return float(((int(y * 255) * 1197) >> 6) - 299); }
float yc48_from_yv12_c(float u) { return float(((int(u * 255) - 128) * 4681 + 164) >> 8); }
float yv12_from_yc48_y(float y) { return float(((((int)y * 219 + 383) >> 12) + 16) / 255.0f); }
float yv12_from_yc48_c(float u) { return float((((((int)u + 2048) * 7 + 66) >> 7) + 16) / 255.0f); }

template <typename ToYV12, typename ToYC48>
void ab_to_yc48(float& A, float& B, ToYV12 toYV12, ToYC48 toYC48) {
  // line through the images of 0 and 2048 (AMTLogo.hpp:72-94)
  const float x0 = toYV12(0.0f), x1 = toYV12(2048.0f);
  const float y0 = toYC48((x0 - B) / A), y1 = toYC48((x1 - B) / A);
  B = y0;
  A = (y1 - y0) / 2048.0f;
}
void base_component(float A, float B, int16_t& color, int16_t& dp) {
  // AMTLogo.hpp:105-124 (same for the three components)
  color = 0; dp = 0;
  if (A == 1) return;
  float t = B / (1 - A) + 0.5f;
  if (!(std::fabs(t) < 0x7FFF)) return;
  const int16_t c = (int16_t)t;
  t = (1 - A) * kMaxDp + 0.5f;
  if (std::fabs(t) > 0x3FFF || (int16_t)t == 0) return;
  color = c; dp = (int16_t)t;
}
}  // namespace

bool lgd_load(const std::string& path, HostLogo& out, LgdHeader* hdr, std::string& err) {
  FILE* fp = fopen(path.c_str(), "rb");
  if (!fp) { err = "Failed to read logo file (" + path + ")"; return false; }
  bool ok = false;
  LgdFileHeader fh; LgdBaseHeader bh; LgdHeader eh;
  do {
    if (fread(&fh, sizeof(fh), 1, fp) != 1 || fread(&bh, sizeof(bh), 1, fp) != 1) break;
    if (fseek(fp, (long)bh.h * bh.w * (long)sizeof(LgdBasePixel), SEEK_CUR) != 0) break;   // skip base part
    if (fread(&eh, sizeof(eh), 1, fp) != 1) break;
    // the reference does not validate magic/version (AMTLogo.hpp:268); sanity-check sizes only
    if (eh.w <= 0 || eh.h <= 0 || eh.w > 4096 || eh.h > 4096 || eh.logUVx < 0 || eh.logUVx > 2 || eh.logUVy < 0 || eh.logUVy > 2) break;
    out.init(eh.w, eh.h, eh.logUVx, eh.logUVy, eh.imgw, eh.imgh, eh.imgx, eh.imgy);
    if (fread(out.data.data(), sizeof(float), out.dataSize(), fp) != out.dataSize()) break;
    ok = true;
  } while (0);
  fclose(fp);
  if (!ok) { err = "Failed to read logo file (" + path + ")"; return false; }
  if (hdr) *hdr = eh;
  return true;
}

bool lgd_save(const HostLogo& l, const std::string& path, const std::string& name, int serviceId, std::string& err) {
  FILE* fp = fopen(path.c_str(), "wb");
  if (!fp) { err = "failed to open for write: " + path; return false; }
  LgdFileHeader fh; memset(&fh, 0, sizeof(fh));
  memcpy(fh.tag, kLgdTag, sizeof(kLgdTag) - 1);
  fh.count_be[3] = 1;                                   // big-endian 1 (SWAP_ENDIAN(1), AMTLogo.hpp:173)
  LgdBaseHeader bh; memset(&bh, 0, sizeof(bh));
  strncpy(bh.name, name.c_str(), sizeof(bh.name) - 1);
  bh.x = (int16_t)l.imgx; bh.y = (int16_t)l.imgy; bh.w = (int16_t)l.w; bh.h = (int16_t)l.h;
  std::vector<LgdBasePixel> base((size_t)l.w * l.h);
  const int wc = l.wUV();
  for (int y = 0; y < l.h; ++y)
    for (int x = 0; x < l.w; ++x) {
      const int o = x + y * l.w, oc = (x >> l.logUVx) + (y >> l.logUVy) * wc;
      LgdBasePixel& p = base[o];
      float A = l.aY()[o], B = l.bY()[o];
      ab_to_yc48(A, B, yv12_from_yc48_y, yc48_from_yv12_y); base_component(A, B, p.y, p.dp_y);
      A = l.aU()[oc]; B = l.bU()[oc];
      ab_to_yc48(A, B, yv12_from_yc48_c, yc48_from_yv12_c); base_component(A, B, p.cb, p.dp_cb);
      A = l.aV()[oc]; B = l.bV()[oc];
      ab_to_yc48(A, B, yv12_from_yc48_c, yc48_from_yv12_c); base_component(A, B, p.cr, p.dp_cr);
    }
  LgdHeader eh; memset(&eh, 0, sizeof(eh));
  eh.magic = 0x12345; eh.version = 1;
  eh.w = l.w; eh.h = l.h; eh.logUVx = l.logUVx; eh.logUVy = l.logUVy;
  eh.imgw = l.imgw; eh.imgh = l.imgh; eh.imgx = l.imgx; eh.imgy = l.imgy;
  // the reference copies at most sizeof(std::string)-1 = 31 characters here (`sizeof(name) - 1` names the
  // std::string parameter, AMTLogo.hpp:45), so longer names are truncated the same way
  strncpy(eh.name, name.c_str(), 31);
  eh.serviceId = serviceId;
  bool ok = fwrite(&fh, sizeof(fh), 1, fp) == 1 && fwrite(&bh, sizeof(bh), 1, fp) == 1 &&
            fwrite(base.data(), sizeof(LgdBasePixel), base.size(), fp) == base.size() &&
            fwrite(&eh, sizeof(eh), 1, fp) == 1 &&
            fwrite(l.data.data(), sizeof(float), l.dataSize(), fp) == l.dataSize();
  fclose(fp);
  if (!ok) err = "failed to write to file: " + path;
  return ok;
}

// ---------------------------------------------------------------------------------------------------
// LogoScan finalisation (LogoScan.hpp:336-395, 471-566) -- microseconds of double arithmetic, host side
// ---------------------------------------------------------------------------------------------------
namespace {
void fit_line(int n, double sx, double sy, double sxx, double sxy, double& a, double& b) {
  const double det = (double)n * sxx - sx * sx;          // NaN/Inf on degenerate input is intended (:338)
  a = ((double)n * sxy - sx * sy) / det;
  b = (sxx * sy - sx * sxy) / det;
}
bool pixel_ab(const double* s, int maxv, int n, float& A, float& B) {
  const double mv = (double)maxv, mv2 = (double)maxv * maxv;
  const double F = s[0] / mv, Bg = s[1] / mv, F2 = s[2] / mv2, B2 = s[3] / mv2, FB = s[4] / mv2;
  double a1, b1, a2, b2;
  fit_line(n, F, Bg, F2, FB, a1, b1);                    // background as a function of foreground
  fit_line(n, Bg, F, B2, FB, a2, b2);                    // and the other way round; average both (:384-389)
  A = (float)((a1 + (1 / a2)) / 2);
  B = (float)((b1 + (-b2 / a2)) / 2);
  return !(std::isnan(A) || std::isnan(B) || std::isinf(A) || std::isinf(B) || A == 0);
}
float ab_distance(float a, float b) { return (1.0f / 3.0f) * (a - 1) * (a - 1) + (a - 1) * b + b * b; }
}  // namespace

bool scan_finalize(const double* sums, int nframes, int scanw, int scanh, int logUVx, int logUVy,
                   int maxv, bool clean, float* out) {
  const int wc = scanw >> logUVx, hc = scanh >> logUVy, ny = scanw * scanh, nc = wc * hc;
  float* aY = out; float* bY = aY + ny; float* aU = bY + ny; float* bU = aU + nc; float* aV = bU + nc; float* bV = aV + nc;
  const double* sY = sums; const double* sU = sY + (size_t)ny * 5; const double* sV = sU + (size_t)nc * 5;
  for (int i = 0; i < ny; ++i) if (!pixel_ab(sY + (size_t)i * 5, maxv, nframes, aY[i], bY[i])) return false;
  for (int i = 0; i < nc; ++i) {
    if (!pixel_ab(sU + (size_t)i * 5, maxv, nframes, aU[i], bU[i])) return false;
    if (!pixel_ab(sV + (size_t)i * 5, maxv, nframes, aV[i], bV[i])) return false;
  }
  if (clean) {
    // Pixels whose (a,b) is indistinguishable from "no logo" are reset to identity (:536-561).  The reference's
    // three maxfilter() passes write only a scratch buffer (:434-454,544-546), i.e. have no effect; none here.
    // When scanw or scanh is not a multiple of the subsampling, the last luma column or row maps to a chroma index
    // oc >= nc, past the chroma planes (the reference indexes the same way and reads and writes outside them): such
    // pixels take their distance from Y alone and reset only Y, so nothing outside `out` is touched.
    std::vector<float> dist((size_t)ny);
    for (int y = 0; y < scanh; ++y)
      for (int x = 0; x < scanw; ++x) {
        const int o = x + y * scanw, oc = (x >> logUVx) + (y >> logUVy) * wc;
        float d = ab_distance(aY[o], bY[o]);
        if (oc < nc) { d += ab_distance(aU[oc], bU[oc]); d += ab_distance(aV[oc], bV[oc]); }   // (Y + U) + V, the reference's order
        d *= 1000;
        dist[o] = d;
      }
    for (int y = 0; y < scanh; ++y)
      for (int x = 0; x < scanw; ++x) {
        const int o = x + y * scanw, oc = (x >> logUVx) + (y >> logUVy) * wc;
        if (dist[o] < 0.3f) {
          aY[o] = 1; bY[o] = 0;
          if (oc < nc) { aU[oc] = 1; bU[oc] = 0; aV[oc] = 1; bV[oc] = 0; }
        }
      }
  }
  return true;
}

// ---------------------------------------------------------------------------------------------------
// AMTEraseLogo::CalcFade2 (LogoScan.hpp:1263-1315): pick the fade(s) for frame n from analyze records
// ---------------------------------------------------------------------------------------------------
// calc_fade2_index and calc_fade2_records are in fade_select.h (shared with the device).
void calc_fade2(const float* records, int num_records, int num_frames, int n, float* fadeT, float* fadeB) {
  float rec9[9 * 33];
  for (int i = -4; i <= 4; ++i)
    memcpy(rec9 + (size_t)(i + 4) * 33, records + (size_t)calc_fade2_index(num_records, num_frames, n, i) * 33, 33 * sizeof(float));
  calc_fade2_records(rec9, fadeT, fadeB);
}

// The logo finder's rule, DESIGN.md section 3.5.  Every sum is taken in a fixed order (pixels of a block row-major) so
// that a restatement in another language gets the same doubles.
void find_logo_rects(const uint64_t* s1, const uint64_t* s2, int64_t nframes, int width, int height, int bits, int block,
                     float var_ratio, float mean_delta, int margin, int min_blocks, std::vector<FoundRect>* out) {
  out->clear();
  const int B = block, bw = width / B, bh = height / B;
  if (nframes < 2 || bw < 3 || bh < 3) return;
  const double n = (double)nframes, maxv = (double)((1 << bits) - 1);
  auto mean = [&](int x, int y) { return (double)s1[(size_t)y * width + x] / n; };
  // per block: the mean of its pixels' temporal variances and of their edge strengths in the temporal mean
  std::vector<double> bv((size_t)bw * bh), be((size_t)bw * bh);
  for (int by = 0; by < bh; ++by)
    for (int bx = 0; bx < bw; ++bx) {
      double sv = 0.0, se = 0.0;
      for (int y = by * B; y < (by + 1) * B; ++y)
        for (int x = bx * B; x < (bx + 1) * B; ++x) {
          const double m = mean(x, y);
          sv += (double)s2[(size_t)y * width + x] / n - m * m;
          se += (x + 1 < width ? std::fabs(mean(x + 1, y) - m) : 0.0) + (y + 1 < height ? std::fabs(mean(x, y + 1) - m) : 0.0);
        }
      bv[(size_t)by * bw + bx] = sv / (double)(B * B);
      be[(size_t)by * bw + bx] = se / (double)(B * B);
    }
  auto median = [](std::vector<double> v) {
    std::nth_element(v.begin(), v.begin() + (v.size() - 1) / 2, v.end());
    return v[(v.size() - 1) / 2];
  };
  const double vmed = median(bv), emed = median(be);
  if (!(vmed > 0.0)) return;
  const double vlim = (double)var_ratio * vmed, dlim = (double)mean_delta * maxv / 255.0;
  // held blocks and their strength: how far they pass the two tests
  std::vector<double> strength((size_t)bw * bh, 0.0);
  std::vector<uint8_t> held((size_t)bw * bh, 0);
  for (int by = 1; by < bh - 1; ++by)
    for (int bx = 1; bx < bw - 1; ++bx) {
      const size_t k = (size_t)by * bw + bx;
      if (bv[k] <= vlim || be[k] - emed >= dlim) {
        held[k] = 1;
        strength[k] = std::max(1.0 - bv[k] / vmed, 0.0) + std::max(be[k] - emed, 0.0) / dlim;
      }
    }
  std::vector<uint8_t> seen((size_t)bw * bh, 0);
  std::vector<int> stack;
  for (int by = 0; by < bh; ++by)
    for (int bx = 0; bx < bw; ++bx) {
      const size_t k0 = (size_t)by * bw + bx;
      if (!held[k0] || seen[k0]) continue;
      int x0 = bx, y0 = by, x1 = bx, y1 = by, count = 0;
      double sum = 0.0;
      stack.assign(1, (int)k0); seen[k0] = 1;
      while (!stack.empty()) {                       // depth first; strengths are added in the order blocks leave the stack
        const int k = stack.back(); stack.pop_back();
        const int cy = k / bw, cx = k % bw;
        ++count; sum += strength[(size_t)k];
        x0 = std::min(x0, cx); x1 = std::max(x1, cx); y0 = std::min(y0, cy); y1 = std::max(y1, cy);
        for (int dy = -1; dy <= 1; ++dy)
          for (int dx = -1; dx <= 1; ++dx) {
            const int ny = cy + dy, nx = cx + dx;
            if (ny < 0 || nx < 0 || ny >= bh || nx >= bw) continue;
            const size_t kk = (size_t)ny * bw + nx;
            if (held[kk] && !seen[kk]) { seen[kk] = 1; stack.push_back((int)kk); }
          }
      }
      if (count < min_blocks) continue;
      if ((y0 == 1 && y1 == bh - 2) || (x0 == 1 && x1 == bw - 2)) continue;     // pillarbox and letterbox bars
      const int W2 = width & ~1, H2 = height & ~1;
      const int rx0 = std::max(0, x0 * B - margin) & ~1, ry0 = std::max(0, y0 * B - margin) & ~1;
      const int rx1 = std::min(W2, ((x1 + 1) * B + margin + 1) & ~1), ry1 = std::min(H2, ((y1 + 1) * B + margin + 1) & ~1);
      FoundRect r;
      r.w = std::min(4096, std::max(4, rx1 - rx0)); r.h = std::min(4096, std::max(4, ry1 - ry0));
      r.x = std::min(rx0, W2 - r.w); r.y = std::min(ry0, H2 - r.h);
      r.score = (float)sum;
      out->push_back(r);
    }
  // best first; equal scores keep the raster order of the components' first blocks
  std::stable_sort(out->begin(), out->end(), [](const FoundRect& a, const FoundRect& b) { return a.score > b.score; });
}

}  // namespace amtk
