/* oracle/tnr_oracle.c -- TEST INFRASTRUCTURE ONLY.
 * Plain-C restatement of the reference's TemporalNRFilter (Amatsukaze/VideoFilter.hpp:27-212), line-cited.  Frames are
 * packed planar 4:2:0: Y (H rows of W samples), U and V (H/2 rows of W/2 samples), samples of `bps` bytes.
 * Compiled with -ffp-contract=off: every float product and sum is rounded on its own, as in the reference's x64 build. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static unsigned get(const void* p, int bps, size_t i) { return bps == 1 ? ((const uint8_t*)p)[i] : ((const uint16_t*)p)[i]; }
static void put(void* p, int bps, size_t i, float v) {
  const int t = (int)v;                                   /* (T)dY: cvttss2si to int32, then the low bits (:202,206-207) */
  if (bps == 1) ((uint8_t*)p)[i] = (uint8_t)t; else ((uint16_t*)p)[i] = (uint16_t)t;
}

/* TNRFilter + filterKernel (:99-211) for one output frame; win[i] = frame w_i, nf = 2d+1 (NFRAMES_, :34) */
void or_tnr_frame(const void* const* win, int nf, int W, int H, int bps, int bits, int threshold, int interlaced, void* out) {
  const int thresh = threshold << (bits - 8);             /* :120 */
  const int mid = nf / 2;                                 /* :158 */
  const size_t ysz = (size_t)W * H, csz = (size_t)(W / 2) * (H / 2);
  const int cw = W / 2;
  float kernel[128];
  for (int i = 0; i < nf; ++i) kernel[i] = 1;             /* :122-125 */
  for (int y = 0; y < H; ++y) {
    for (int x = 0; x < W; ++x) {
      const int cy = interlaced ? (((y >> 1) & ~1) | (y & 1)) : (y >> 1);     /* :164 */
      const int cx = x >> 1;                                                  /* :165 */
      const size_t iy = (size_t)y * W + x, ic = (size_t)cy * cw + cx;
      const int Y = get(win[mid], bps, iy), U = get(win[mid], bps, ysz + ic), V = get(win[mid], bps, ysz + csz + ic);
      float sumKernel = 0.0f;                                                 /* :171-181 */
      for (int i = 0; i < nf; ++i) {
        const int diff = abs(Y - (int)get(win[i], bps, iy)) + abs(U - (int)get(win[i], bps, ysz + ic)) +
                         abs(V - (int)get(win[i], bps, ysz + csz + ic));      /* calcDiff, :148-153 */
        if (diff <= thresh) sumKernel += kernel[i];
      }
      const float factor = 1.f / sumKernel;                                   /* :183 */
      float dY = 0.5f, dU = 0.5f, dV = 0.5f;                                  /* :185-187 */
      for (int i = 0; i < nf; ++i) {                                          /* :188-200 */
        const int rY = get(win[i], bps, iy), rU = get(win[i], bps, ysz + ic), rV = get(win[i], bps, ysz + csz + ic);
        const int diff = abs(Y - rY) + abs(U - rU) + abs(V - rV);
        if (diff <= thresh) {
          const float coef = kernel[i] * factor;
          dY += coef * rY;
          dU += coef * rU;
          dV += coef * rV;
        }
      }
      put(out, bps, iy, dY);                                                  /* :202 */
      if ((x & 1) == 0 && ((interlaced ? (y >> 1) : y) & 1) == 0) {           /* :204-208 */
        put(out, bps, ysz + ic, dU);
        put(out, bps, ysz + csz + ic, dV);
      }
    }
  }
}

/* The library's definition: output k = frame frame0+k over w_i = clamp(frame0+k - d + i, 0, N-1). */
void or_tnr_clip(const void* frames, int N, int W, int H, int bps, int bits, int d, int threshold, int interlaced,
                 int frame0, int nframes, void* out) {
  const size_t fs = ((size_t)W * H + 2 * (size_t)(W / 2) * (H / 2)) * bps;
  const void* win[128];
  for (int k = 0; k < nframes; ++k) {
    const int n = frame0 + k;
    for (int i = 0; i <= 2 * d; ++i) {
      int f = n - d + i;
      f = f < 0 ? 0 : (f > N - 1 ? N - 1 : f);
      win[i] = (const uint8_t*)frames + (size_t)f * fs;
    }
    or_tnr_frame(win, 2 * d + 1, W, H, bps, bits, threshold, interlaced, (uint8_t*)out + (size_t)k * fs);
  }
}
