"""oracle/pyscan16.py -- TEST INFRASTRUCTURE ONLY: the checkers of LogoScan on 2-byte samples (9..16 bits).

  * RefScan16        -- the reference's own LogoScan with AddFrame<uint16_t> (oracle/_ref/libamtk_ref.so)
  * PyScan16         -- the same accumulation restated on exact integers, for where oracle/_ref was not built
  * compose_scan_logo -- the ScanLogo pipeline (LogoScan.hpp:845-1031) at maxv, from the oracle's pieces

Only tests/ may import this; the product package never does.
"""
import numpy as np

from oracle.pyoracle import (OracleLogo, OracleScan, RefScan, _p, c_float_p, c_u8_p, c_u16_p, oracle_lib,
                             ref_available)


class RefScan16(RefScan):
    """The reference's own LogoScan, with AddFrame<uint16_t> (LogoScan.hpp:594-659) next to the 8-bit add_frame."""

    def add_frame_u16(self, y, u, v, pitchY=None, pitchUV=None):
        y, u, v = [np.ascontiguousarray(p, np.uint16) for p in (y, u, v)]
        return self.R.ref_scan_add_frame_u16(self.ptr, _p(y, c_u16_p), _p(u, c_u16_p), _p(v, c_u16_p),
                                             y.shape[1] if pitchY is None else pitchY,
                                             u.shape[1] if pitchUV is None else pitchUV)


def _wrap32(a):
    return ((a + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


class PyScan16:
    """LogoScan::AddFrame<uint16_t> (LogoScan.hpp:594-659) restated on exact integers, for where oracle/_ref was not built:
    the border samples live in a std::vector<short> (:406), so at 16 bits a sample >= 32768 wraps negative in the range
    test, the sort and med_average (:414-428); LogoColor::Add (:357-364) takes int products, so f*f wraps to 32 bits at
    16 bits.  The sums are int64 and equal the reference's doubles while they stay below 2^53.  Normalize + GetLogo run in
    the C port (OracleScan), which tests/test_oracle.py pins to the reference."""

    def __init__(self, scanw, scanh, thy, logUVx=1, logUVy=1):
        self.w, self.h, self.thy, self.lx, self.ly = scanw, scanh, thy, logUVx, logUVy
        self.ny = scanw * scanh
        self.nc = (scanw >> logUVx) * (scanh >> logUVy)
        self.acc = np.zeros((self.ny + 2 * self.nc, 5), np.int64)
        self.nframes = 0

    @staticmethod
    def _med_average(s):
        n = len(s)
        lo, hi = n // 4, n - n // 4
        nn = hi - lo
        return int((float(s[lo:hi].sum()) + nn // 2) / nn)        # (int)((t + nn/2) / nn) in double, t exact

    def add_frame_u16(self, y, u, v):
        dims = [(self.w, self.h), (self.w >> self.lx, self.h >> self.ly), (self.w >> self.lx, self.h >> self.ly)]
        planes = [np.asarray(p, np.uint16)[:ph, :pw].astype(np.int64) for p, (pw, ph) in zip((y, u, v), dims)]
        bgs = []
        for P, (pw, ph) in zip(planes, dims):
            tmp = []
            for x in range(pw):                                            # :616-635, the reference's push order
                tmp += [P[0, x], P[ph - 1, x]]
            for yy in range(1, ph - 1):
                tmp += [P[yy, 0], P[yy, pw - 1]]
            s = np.sort(np.array(tmp, np.int64).astype(np.uint16).view(np.int16).astype(np.int64))
            if abs(int(s[0]) - int(s[-1])) > self.thy:
                return 0
            bgs.append(self._med_average(s))
        rows = []
        for P, b in zip(planes, bgs):
            f = P.ravel()
            rows.append(np.stack([f, np.full_like(f, b), _wrap32(f * f), np.full_like(f, b * b), f * b], axis=1))
        self.acc += np.concatenate(rows)
        self.nframes += 1
        return 1

    def sums(self):
        return self.acc.astype(np.float64)

    def get_logo(self, maxv, clean=False):
        sc = OracleScan(self.w, self.h, self.thy, self.lx, self.ly)
        sc.set_sums(self.sums(), self.nframes)
        return sc.get_logo(maxv, clean)


def scan16_class():
    """The LogoScan the 2-byte tests compare against: the reference's own (oracle/_ref), else PyScan16."""
    return RefScan16 if ref_available() else PyScan16


def compose_scan_logo(Y, U, V, w, h, thy, max_frames, maxv, logUVx=1, logUVy=1, scan_class=None):
    """LogoAnalyzer::ScanLogo (LogoScan.hpp:845-1031) on per-frame scan rectangles Y[i], U[i], V[i] (uint8 or uint16),
    with maxv in place of the reference's three 255s (:845, :968, :1030): MakeInitialLogo up to max_frames valid frames,
    GetLogo(false), then twice: DeintLogo + CreateLogoMask(0.1), DeintY + EvaluateLogo at 20 fades per stored frame,
    re-accumulate the frames whose best fade index is > 8, GetLogo(true).  Returns (logo data or None for "Insufficient
    logo frames", indices of the stored frames)."""
    wide = np.asarray(Y[0]).dtype != np.uint8
    if scan_class is None:
        scan_class = scan16_class() if wide else (RefScan if ref_available() else OracleScan)
    add = "add_frame_u16" if wide else "add_frame"
    sc = scan_class(w, h, thy, logUVx, logUVy)
    stored = []
    for i in range(len(Y)):
        if len(stored) >= max_frames:
            break
        if getattr(sc, add)(Y[i], U[i], V[i]):
            stored.append(i)
    data = sc.get_logo(maxv, False)
    if data is None:
        return None, stored
    L = oracle_lib()
    deint = L.amtk_or_deint_y_u16 if wide else L.amtk_or_deint_y_u8
    ptr_t = c_u16_p if wide else c_u8_p
    for _ in range(2):
        de = OracleLogo.create(data, w, h, w, h, 0, 0, logUVx, logUVy).deint().create_mask(0.1)
        keep = []
        for i in stored:
            ry = np.ascontiguousarray(Y[i])
            dd = np.zeros(w * h + 8, np.float32)
            deint(_p(dd, c_float_p), ry.ctypes.data_as(ptr_t), w, w, h)
            res = [abs(np.float32(de.evaluate(dd, float(maxv), np.float32(0.1) * np.float32(fi)))) for fi in range(20)]
            if int(np.argmin(res)) > 8:
                keep.append(i)
        sc2 = scan_class(w, h, thy, logUVx, logUVy)
        for i in keep:
            getattr(sc2, add)(Y[i], U[i], V[i])
        data = sc2.get_logo(maxv, True)
        if data is None:
            return None, stored
    return data, stored
