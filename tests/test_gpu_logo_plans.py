"""Logo evaluation at every launch plan of launch_eval (csrc/amtk_b200.cu), bit for bit against the reference's own code
(oracle/_ref) where it was built, else the C port that tests/test_oracle.py pins to it.

launch_eval picks, per call: pixels per thread and pixel slices from the feature count, whether the logo planes A/B and
a second fade image fit in shared memory, TMA or plain loads for the ROI, the bulk or plain score sum, and how many
frame batches the 96 MB score scratch needs.  eval_plan() below restates that choice; a CPU test checks that the cases
of this file reach every value of every plan dimension, so moving a threshold cannot silently drop a path from the
suite.  Every GPU case walks at least three frames per CTA lane, so the TMA double buffer wraps on every CTA.
"""
import functools
import zlib

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from test_gpu_erase import logo_data

# ---- restatement of launch_eval's plan choice (amtk_b200.cu:238-253,283-286,305-306; logo_kernels.cuh:54-58) ----------
K_EVAL_THREADS = 512
K_SMEM_LIMIT = 226 * 1024
K_SUM_BULK_LIMIT = 200 * 1024
K_SCRATCH = 96 << 20
K_LITE_LIMIT = 29 * 1024
SM_H100 = 132


def _smem_bytes(roi_n, npx, raw_bytes_one, ab_smem, pair_fades):
    r4 = lambda v: (v + 3) & ~3
    return ((2 if ab_smem else 0) * r4(npx) + r4(roi_n) + (2 if pair_fades else 1) * r4(npx + 8)) * 4 + 128 + \
        2 * ((raw_bytes_one + 127) & ~127)


def lite_smem_bytes(w, h, bps):
    """logo_lite_smem_bytes (logo_kernels.cuh): the fused step runs the small-footprint kernel when this is <= 29 KB."""
    return ((w * h + 8 + 3) & ~3) * 4 + ((w * h * bps + 15) & ~15) + 16


def eval_plan(count, logo_w, logo_h, roi_x, roi_w, roi_h, bps, pitch_bytes, frame_stride, nfades, nframes,
              sm_count=SM_H100, eval_cw=True):
    """The launch plan of one launch_eval call on a device clip (the ROI is the logo rectangle)."""
    npx = logo_w * logo_h
    count_pad = max(32, (count + 31) & ~31)
    if count <= K_EVAL_THREADS:
        pxt, slices = 1, 1
    elif count <= 2 * K_EVAL_THREADS:
        pxt, slices = 2, 1
    else:
        pxt, slices = 3, (count + 3 * K_EVAL_THREADS - 1) // (3 * K_EVAL_THREADS)
    box_x = ((roi_x * bps) & ~15) // bps
    box_w = ((((roi_x - box_x) + roi_w) * bps + 15) & ~15) // bps
    tma = box_w <= 256 and roi_h <= 256 and pitch_bytes % 16 == 0 and frame_stride % 16 == 0
    raw = box_w * roi_h * bps
    ab_smem, pair = 1, 1
    if _smem_bytes(roi_w * roi_h, npx, raw, ab_smem, pair) > K_SMEM_LIMIT:
        ab_smem = 0
    if _smem_bytes(roi_w * roi_h, npx, raw, ab_smem, pair) > K_SMEM_LIMIT:
        pair = 0
    fits = _smem_bytes(roi_w * roi_h, npx, raw, ab_smem, pair) <= K_SMEM_LIMIT
    batch = max(1, min(nframes, K_SCRATCH // (nfades * count_pad * 4)))
    lanes = max(1, min(batch, sm_count // slices))
    w64 = logo_w == 64 and roi_w == 64 and eval_cw
    return {
        "pxt": pxt, "slices": slices, "multi_slice": slices > 1, "ab_smem": ab_smem, "pair_fades": pair, "fits": fits,
        "load": "tma" if tma else "plain", "sum": "bulk" if 32 * (count_pad + 4) * 4 <= K_SUM_BULK_LIMIT else "plain",
        "batches": (nframes + batch - 1) // batch, "lanes": lanes,
        "cw": "64x64" if (w64 and logo_h == 64 and roi_h == 64) else ("64" if w64 else "runtime"),
        "bits16": bps == 2,
    }


# ---- cases -------------------------------------------------------------------------------------------------------------
def _bisect_ratio(raw, threshold):
    """(r_lo, r_hi): mask ratios whose deint feature counts are the largest <= threshold and the smallest > threshold."""
    lo, hi = 0.0, 1.0
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        if raw.deint().create_mask(mid).info().count > threshold:
            hi = mid
        else:
            lo = mid
    return lo, hi


# name: (bits, logo w, h, seed, ratio or ("<=", T) / (">", T), imgx, imgy, frame W, H)
CASES = {
    "pxt1_cw64x64_8":   (8, 64, 64, 1, ("<=", 512), 160, 40, 320, 160),
    "pxt2_cw64x64_16":  (16, 64, 64, 2, (">", 512), 163, 40, 320, 160),
    "pxt2_runtime_8":   (8, 48, 40, 6, ("<=", 1024), 161, 33, 320, 128),
    "pxt3_runtime_12":  (12, 48, 40, 6, (">", 1024), 0, 20, 256, 96),                # left edge
    "pxt3_cw64_8":      (8, 64, 48, 3, ("<=", 1536), 175, 0, 320, 128),              # top edge, imgx % 16 = 15
    "slices2_cw64x64_8": (8, 64, 64, 1, (">", 1536), 256, 64, 320, 128),            # right and bottom edge
    "slices2_10":       (10, 96, 64, 2, 0.35, 104, 30, 256, 128),
    "ab0_bulk_8":       (8, 128, 96, 5, 0.1, 32, 32, 320, 128),                     # bottom edge
    "ab0_plainsum_12":  (12, 128, 96, 5, 0.2, 96, 20, 256, 128),                    # right edge
    "ab0_pair0_wide_8": (8, 256, 60, 10, 0.05, 1, 0, 320, 96),                      # box wider than 256 -> plain loads
    "ab0_pair0_16":     (16, 160, 112, 7, 0.05, 40, 8, 224, 128),
    "ab0_pair0_plain_8": (8, 256, 90, 10, 0.3, 32, 6, 320, 96),
    "wide_plain_16":    (16, 250, 64, 9, 0.05, 7, 16, 272, 96),                     # 16-bit box of 264 elements
    "wide_tma_16":      (16, 250, 64, 9, 0.05, 3, 16, 272, 96),                     # ... and of exactly 256
    "pitch_plain_10":   (10, 48, 40, 6, 0.35, 100, 30, 204, 80),                    # 408-byte rows: TMA cannot describe them
    "pitch_plain_8":    (8, 64, 64, 1, 0.35, 60, 10, 200, 96),
}


def _bps(bits):
    return 1 if bits == 8 else 2


@functools.lru_cache(maxsize=None)
def _ratio(name):
    bits, w, h, seed, r, imgx, imgy, W, H = CASES[name]
    if not isinstance(r, tuple):
        return r
    raw = ab.Logo.create(synth.make_logo(w, h, seed=seed)["data"], w, h, W, H, imgx, imgy)
    lo, hi = _bisect_ratio(raw, r[1])
    return lo if r[0] == "<=" else hi


def _plan(name, nfades=2, nframes=None, sm_count=SM_H100):
    bits, w, h, seed, _, imgx, imgy, W, H = CASES[name]
    raw = ab.Logo.create(synth.make_logo(w, h, seed=seed)["data"], w, h, W, H, imgx, imgy)
    count = raw.deint().create_mask(_ratio(name)).info().count
    bps = _bps(bits)
    p = eval_plan(count, w, h, imgx, w, h, bps, W * bps, W * H * 3 // 2 * bps, nfades, nframes or 1, sm_count)
    p["count"] = count
    return p


# eval_fades call that needs several score batches: 24 fades x ~6.1 k feature pixels (countPad 6112) -> 171 frames each
BATCH_CASE = ("ab0_bulk_8", 0.5, 360)


def test_plan_table_covers_every_launch_path(native_lib):
    """Every value of every plan dimension is reached by a case of this file (no GPU needed: logos and masks are host
    objects).  Fails when a threshold in launch_eval moves and a path drops out of the suite."""
    plans = {n: _plan(n) for n in CASES}
    for name, (bits, w, h, seed, r, *_rest) in CASES.items():
        if isinstance(r, tuple):                                    # the searched ratios land right next to the threshold
            c = plans[name]["count"]
            assert (c <= r[1]) if r[0] == "<=" else (c > r[1]), (name, c)
            assert abs(c - r[1]) <= 16, (name, c)
        assert plans[name]["fits"], name
    want = {"pxt": {1, 2, 3}, "multi_slice": {False, True}, "load": {"tma", "plain"}, "sum": {"bulk", "plain"},
            "cw": {"64x64", "64", "runtime"}}
    for dim, values in want.items():
        assert {p[dim] for p in plans.values()} == values, dim
    for bits16 in (False, True):                                    # shared-memory plans and both sums at 8 AND 16 bits
        sub = [p for p in plans.values() if p["bits16"] == bits16]
        for dim in ("ab_smem", "pair_fades"):
            assert {p[dim] for p in sub} == {0, 1}, (dim, bits16)
        assert {p["sum"] for p in sub} == {"bulk", "plain"}, bits16
    assert {CASES[n][0] for n in CASES} == {8, 10, 12, 16}
    assert {CASES[n][5] % 16 for n in CASES if CASES[n][0] == 8} >= {0, 1, 15}
    assert {CASES[n][5] % 8 for n in CASES if CASES[n][0] != 8} >= {0, 3}
    edges = set()
    for bits, w, h, seed, r, x, y, W, H in CASES.values():
        edges |= {e for e, hit in (("l", x == 0), ("t", y == 0), ("r", x + w == W), ("b", y + h == H)) if hit}
    assert edges == {"l", "t", "r", "b"}
    # the multi-batch eval_fades call
    name, ratio, n = BATCH_CASE
    bits, w, h, seed, _, imgx, imgy, W, H = CASES[name]
    raw = ab.Logo.create(synth.make_logo(w, h, seed=seed)["data"], w, h, W, H, imgx, imgy)
    count = raw.deint().create_mask(ratio).info().count
    assert eval_plan(count, w, h, imgx, w, h, 1, W, W * H * 3 // 2, 24, n)["batches"] >= 3
    assert eval_plan(count, w, h, imgx, w, h, 1, W, W * H * 3 // 2, 2, n)["batches"] == 1
    # the scan-lite limit: 96x61 / 80x61 fit at 8 / 16 bits, one row more does not
    assert lite_smem_bytes(96, 61, 1) <= K_LITE_LIMIT < lite_smem_bytes(96, 62, 1)
    assert lite_smem_bytes(80, 61, 2) <= K_LITE_LIMIT < lite_smem_bytes(80, 62, 2)
    # a logo that fits at 8 bits is too large at 16 (the "too large" rejection below)
    assert eval_plan(4000, 256, 90, 0, 256, 90, 1, 640, 640 * 288 * 3 // 2, 2, 1)["fits"]
    assert not eval_plan(4000, 256, 90, 0, 256, 90, 2, 1280, 1280 * 288 * 3 // 2, 2, 1)["fits"]


# ---- GPU side ------------------------------------------------------------------------------------------------------------
def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def make_clip_frames(n, W, H, bits, logo=None, imgx=0, imgy=0, seed=0):
    """(n, W*H*3/2) packed 4:2:0 frames of `bits`-bit samples (uint8 or uint16) spread over [0, maxv]: a moving ramp plus
    noise, with 0 and maxv patches, and the logo composited on most frames (off on every fifth)."""
    maxv = (1 << bits) - 1
    rng = np.random.default_rng(seed)
    dt = np.uint8 if bits == 8 else np.uint16
    ysz, csz = W * H, (W // 2) * (H // 2)
    yy, xx = np.mgrid[0:H, 0:W]
    out = np.empty((n, ysz + 2 * csz), dt)
    for i in range(n):
        ramp = ((xx * 7 + yy * 5 + i * 11) % 256) * (maxv + 1) // 256
        Y = np.clip(ramp + rng.integers(-maxv // 16 - 1, maxv // 16 + 2, (H, W)), 0, maxv)
        if i % 3 == 0:
            Y[(yy // 7 + xx // 9 + i) % 5 == 0] = maxv
        if i % 3 == 1:
            Y[(yy // 5 + xx // 11 + i) % 4 == 0] = 0
        if logo is not None and i % 5:
            al = logo["alpha8"].astype(np.int64)
            lh, lw = al.shape
            roi = Y[imgy:imgy + lh, imgx:imgx + lw]
            Y[imgy:imgy + lh, imgx:imgx + lw] = (roi * (256 - al) + al * (maxv * 9 // 10)) >> 8
        out[i, :ysz] = Y.ravel()
        out[i, ysz:] = rng.integers(0, maxv + 1, 2 * csz)
    return out


def to_device(a):
    t = torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a)
    return t.cuda()


def y_planes(a, W, H):
    return a[:, :W * H].reshape(a.shape[0], H, W)


def _bits_of(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


class Oracle:
    """Reference logo evaluation: the reference's own code when oracle/_ref exists, else the C port."""

    def __init__(self, po, data, w, h, W, H, imgx, imgy):
        self.po, self.w, self.h, self.x, self.y = po, w, h, imgx, imgy
        self.ref = po.ref_available()
        mk = po.RefLogo.create if self.ref else po.OracleLogo.create
        self.raw = mk(data, w, h, W, H, imgx, imgy)

    def deint(self, ratio):
        return self.raw.deint().create_mask(ratio)

    def fields(self, ratio):
        return self.raw.field(0).create_mask(ratio), self.raw.field(1).create_mask(ratio)

    def scan(self, de, plane, maxv):
        if self.ref:
            return self.po.ref_scan_frame(de, plane, maxv=maxv)
        return de.scan_frame(plane, maxv=maxv)

    def analyze(self, de, top, bot, plane, maxv):
        f = self.po.ref_analyze_frame if self.ref else self.po.or_analyze_frame
        return f(de, top, bot, plane, maxv=maxv)

    def deint_roi(self, plane):
        """DeintY of the logo rectangle (LogoScan.hpp:763-780)."""
        roi = np.ascontiguousarray(plane[self.y:self.y + self.h, self.x:self.x + self.w])
        if self.ref:
            return self.po.ref_deint_y(roi, self.w, self.h)
        L = self.po.oracle_lib()
        out = np.zeros(self.w * self.h + 8, np.float32)
        fn = L.amtk_or_deint_y_u8 if roi.dtype == np.uint8 else L.amtk_or_deint_y_u16
        fn(out.ctypes.data_as(self.po.c_float_p), roi.ctypes.data_as(self.po.c_u8_p if roi.dtype == np.uint8 else self.po.c_u16_p),
           self.w, self.w, self.h)
        return out

    def fades(self, de, plane, maxv, fades):
        src = self.deint_roi(plane)
        return np.array([de.evaluate(src, maxv, np.float32(f)) for f in fades], np.float32)


def _setup(po, name, n):
    bits, w, h, seed, _, imgx, imgy, W, H = CASES[name]
    lg = synth.make_logo(w, h, seed=seed)
    ratio = _ratio(name)
    host = make_clip_frames(n, W, H, bits, logo=lg, imgx=imgx, imgy=imgy, seed=zlib.crc32(name.encode()))
    P = ab.Logo.create(lg["data"], w, h, W, H, imgx, imgy).deint().create_mask(ratio)
    O = Oracle(po, lg["data"], w, h, W, H, imgx, imgy)
    return bits, (1 << bits) - 1, W, H, host, P, O, O.deint(ratio), lg, ratio


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(CASES))
def test_scan_frames_every_plan(ctx, oracle, name):
    """LogoFrame::ScanFrame scores at every plan; the clip is long enough that every CTA lane walks >= 3 frames."""
    plan = _plan(name)
    n = 3 * max(1, _sm_count() // plan["slices"]) + 5
    bits, maxv, W, H, host, P, O, de, lg, _ = _setup(oracle, name, n)
    assert _plan(name, nframes=n, sm_count=_sm_count())["lanes"] * 3 <= n
    assert P.info().count == plan["count"]
    dev = to_device(host)                                       # the descriptor holds only its address
    clip = ab.yv12_clip(dev, W, H, n, True, bits)
    got = ctx.scan_frames(clip, [P]).cpu().numpy()[:, 0]
    Y = y_planes(host, W, H)
    ref = np.stack([O.scan(de, Y[i], float(maxv)) for i in range(n)])
    assert np.array_equal(_bits_of(got), _bits_of(ref)), (name, np.argwhere(_bits_of(got) != _bits_of(ref))[:4])
    assert ref[:, 0].max() > ref[:, 0].min()                          # the scores are not all one value
    # frame-range calls (frame0 > 0) give the same rows
    a, b = n // 3, n - 3
    part = ctx.scan_frames(clip, [P], frame0=a, nframes=b - a).cpu().numpy()[:, 0]
    assert np.array_equal(_bits_of(part), _bits_of(ref[a:b])), name


@pytest.mark.gpu
def test_too_large_at_16_bits(ctx):
    """A 256x90 logo fits the shared-memory plan at 8 bits (two-byte samples need 46 KB more): rejected at 16."""
    lg = synth.make_logo(256, 90, seed=10)
    W, H = 320, 96
    p = ab.Logo.create(lg["data"], 256, 90, W, H, 32, 6).deint().create_mask(0.3)
    fr = to_device(make_clip_frames(2, W, H, 10))
    with pytest.raises(ab.AmtkError, match="too large"):
        ctx.scan_frames(ab.yv12_clip(fr, W, H, 2, True, 10), [p])
    fr8 = to_device(make_clip_frames(2, W, H, 8))
    ctx.scan_frames(ab.yv12_clip(fr8, W, H, 2, True, 8), [p])        # the same logo at 8 bits is fine


FADE_SETS = {
    1: np.array([1.9], np.float32),
    7: np.array([0.0, 1.0, 1.9, 0.5, 0.1, 1.3, 0.7], np.float32),
    24: np.concatenate([np.float32(0.1) * np.arange(20, dtype=np.float32), np.array([1.0, 0.25, 1.95, 0.05], np.float32)]),
}


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["pxt1_cw64x64_8", "pxt3_runtime_12", "ab0_pair0_16", "wide_plain_16", "pitch_plain_10"])
@pytest.mark.parametrize("nf", [1, 7, 24])
def test_eval_fades_every_plan(ctx, oracle, name, nf):
    """ReMakeLogo's fade sweep (LogoScan.hpp:964-975) with 1, 7 (odd: the last pass of a fade pair is single) and 24 fade
    levels, over a range that starts at frame0 > 0 and is long enough to wrap the ROI ring on every lane."""
    n = 3 * max(1, _sm_count() // _plan(name)["slices"]) + 9
    bits, maxv, W, H, host, P, O, de, lg, ratio = _setup(oracle, name, n)
    fades = FADE_SETS[nf]
    dev = to_device(host)                                       # the descriptor holds only its address
    clip = ab.yv12_clip(dev, W, H, n, True, bits)
    f0 = 4
    got = ctx.eval_fades(clip, P, fades, frame0=f0, nframes=n - f0).cpu().numpy()
    Y = y_planes(host, W, H)
    ref = np.stack([O.fades(de, Y[i], float(maxv), fades) for i in range(f0, n)])
    assert np.array_equal(_bits_of(got), _bits_of(ref)), (name, nf, np.argwhere(_bits_of(got) != _bits_of(ref))[:4])


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_eval_fades_several_batches(ctx, oracle):
    """24 fades x 6.1 k feature pixels: the 96 MB score scratch holds 171 frames, so a 360-frame call runs 3 batches; each
    batch's sums must land on its own rows (frame0 > 0 shifts them all)."""
    name, ratio, n = BATCH_CASE
    bits, w, h, seed, _, imgx, imgy, W, H = CASES[name]
    lg = synth.make_logo(w, h, seed=seed)
    f0, total = 5, n + 9
    host = make_clip_frames(total, W, H, bits, logo=lg, imgx=imgx, imgy=imgy, seed=77)
    P = ab.Logo.create(lg["data"], w, h, W, H, imgx, imgy).deint().create_mask(ratio)
    cnt = P.info().count
    assert eval_plan(cnt, w, h, imgx, w, h, 1, W, W * H * 3 // 2, 24, n)["batches"] >= 3
    O = Oracle(oracle, lg["data"], w, h, W, H, imgx, imgy)
    de = O.deint(ratio)
    fades = FADE_SETS[24]
    dev = to_device(host)                                       # the descriptor holds only its address
    clip = ab.yv12_clip(dev, W, H, total, True, bits)
    got = ctx.eval_fades(clip, P, fades, frame0=f0, nframes=n).cpu().numpy()
    Y = y_planes(host, W, H)
    ref = np.stack([O.fades(de, Y[i], 255.0, fades) for i in range(f0, f0 + n)])
    assert np.array_equal(_bits_of(got), _bits_of(ref)), np.argwhere(_bits_of(got) != _bits_of(ref))[:4]


ANALYZE_CASES = [(8, 64, 48, 3, 0.35, 160, 34, 320, 128), (12, 96, 64, 2, 0.2, 17, 30, 256, 128), (16, 64, 64, 1, 0.5, 64, 0, 192, 96)]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", ANALYZE_CASES, ids=lambda c: "%dbit_%dx%d" % c[:3])
def test_analyze_parallel_and_serial_agree(ctx, oracle, case):
    """AMTAnalyzeLogo records: calls of <= 16 frames run their three evaluations on three streams, longer ones serially;
    both equal the reference."""
    bits, w, h, seed, ratio, imgx, imgy, W, H = case
    maxv = (1 << bits) - 1
    lg = synth.make_logo(w, h, seed=seed)
    n = 3 * _sm_count() + 5
    host = make_clip_frames(n, W, H, bits, logo=lg, imgx=imgx, imgy=imgy, seed=bits)
    raw = ab.Logo.create(lg["data"], w, h, W, H, imgx, imgy)
    de, top, bot = raw.deint().create_mask(ratio), raw.field(0).create_mask(ratio), raw.field(1).create_mask(ratio)
    dev = to_device(host)                                       # the descriptor holds only its address
    clip = ab.yv12_clip(dev, W, H, n, True, bits)
    serial = ctx.analyze_frames(clip, de, top, bot).cpu().numpy()
    par = np.concatenate([ctx.analyze_frames(clip, de, top, bot, frame0=a, nframes=min(16, n - a)).cpu().numpy()
                          for a in range(0, 48, 16)])
    assert np.array_equal(_bits_of(par), _bits_of(serial[:48]))
    O = Oracle(oracle, lg["data"], w, h, W, H, imgx, imgy)
    ode = O.deint(ratio)
    ot, ob = O.fields(ratio)
    Y = y_planes(host, W, H)
    ref = np.stack([O.analyze(ode, ot, ob, Y[i], float(maxv)) for i in range(n)])
    assert np.array_equal(_bits_of(serial), _bits_of(ref)), np.argwhere(_bits_of(serial) != _bits_of(ref))[:4]


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_runtime_width_knob_matches_templates(ctx, oracle, monkeypatch):
    """AMTK_EVAL_CW=0 runs the run-time-width kernel on 64x64 and 64x48 logos: the same bits as the compile-time 64x64 and
    64-wide templates the default context picks."""
    monkeypatch.setenv("AMTK_EVAL_CW", "0")
    c0 = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    monkeypatch.delenv("AMTK_EVAL_CW")
    try:
        for (h, seed, imgx, imgy, bits) in ((64, 1, 128, 32, 8), (48, 3, 131, 17, 16)):
            W, H, n = 256, 128, 3 * _sm_count() + 4
            lg = synth.make_logo(64, h, seed=seed)
            host = make_clip_frames(n, W, H, bits, logo=lg, imgx=imgx, imgy=imgy, seed=h)
            raw = ab.Logo.create(lg["data"], 64, h, W, H, imgx, imgy)
            de, top, bot = raw.deint().create_mask(0.35), raw.field(0).create_mask(0.35), raw.field(1).create_mask(0.35)
            dev = to_device(host)                                       # the descriptor holds only its address
            clip = ab.yv12_clip(dev, W, H, n, True, bits)
            for fn in (lambda c: c.scan_frames(clip, [de]), lambda c: c.eval_fades(clip, de, FADE_SETS[7], frame0=3),
                       lambda c: c.analyze_frames(clip, de, top, bot, nframes=40)):
                a, b = fn(ctx).cpu().numpy(), fn(c0).cpu().numpy()
                assert np.array_equal(_bits_of(a), _bits_of(b)), h
            O = Oracle(oracle, lg["data"], 64, h, W, H, imgx, imgy)
            ode = O.deint(0.35)
            Y = y_planes(host, W, H)
            ref = np.stack([O.scan(ode, Y[i], float((1 << bits) - 1)) for i in range(n)])
            assert np.array_equal(_bits_of(c0.scan_frames(clip, [de]).cpu().numpy()[:, 0]), _bits_of(ref)), h
    finally:
        c0.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [8, 10, 16])
def test_flat_rois(ctx, oracle, bits):
    """Constant frames (0, maxv, mid): zero-variance windows, whose score sums are +0 or -0; the sign must match too."""
    maxv = (1 << bits) - 1
    W, H, w, h, imgx, imgy = 256, 128, 64, 48, 96, 40
    lg = synth.make_logo(w, h, seed=3)
    vals = [0, maxv, maxv // 2 + 1, 1]
    n = len(vals)
    dt = np.uint8 if bits == 8 else np.uint16
    host = np.stack([np.full(W * H * 3 // 2, v, dt) for v in vals])
    raw = ab.Logo.create(lg["data"], w, h, W, H, imgx, imgy)
    de = raw.deint().create_mask(0.35)
    dev = to_device(host)                                       # the descriptor holds only its address
    clip = ab.yv12_clip(dev, W, H, n, True, bits)
    O = Oracle(oracle, lg["data"], w, h, W, H, imgx, imgy)
    ode = O.deint(0.35)
    Y = y_planes(host, W, H)
    got = ctx.scan_frames(clip, [de]).cpu().numpy()[:, 0]
    ref = np.stack([O.scan(ode, Y[i], float(maxv)) for i in range(n)])
    assert np.array_equal(_bits_of(got), _bits_of(ref)), (_bits_of(got), _bits_of(ref))
    fades = FADE_SETS[24]
    got = ctx.eval_fades(clip, de, fades).cpu().numpy()
    ref = np.stack([O.fades(ode, Y[i], float(maxv), fades) for i in range(n)])
    assert np.array_equal(_bits_of(got), _bits_of(ref))


LITE_CASES = [(8, 48, 40, 0.35, 101, 30), (8, 96, 61, 0.35, 64, 20), (8, 96, 62, 0.35, 64, 20),
              (16, 48, 40, 0.35, 101, 30), (16, 80, 61, 0.35, 160, 7), (16, 80, 62, 0.35, 160, 7)]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("mode", ["1", "2"])
def test_scan_lite_sizes(oracle, monkeypatch, mode):
    """AMTK_SCAN_LITE=1 (small-footprint kernel under the comb kernel) and 2 (on its own) on non-64 logos and on logos just
    under and just over the kernel's 29 KB shared-memory limit (those take the serial path): all equal the reference."""
    monkeypatch.setenv("AMTK_SCAN_LITE", mode)
    c = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    monkeypatch.delenv("AMTK_SCAN_LITE")
    try:
        W, H, n = 320, 128, 40
        prm = ab.default_comb_params()
        for (bits, w, h, ratio, imgx, imgy) in LITE_CASES:
            bb = 10 if bits == 16 else 8
            data = logo_data(w, h, seed=w + h)                       # odd heights: synth.make_logo needs even ones
            host = make_clip_frames(n, W, H, bb, seed=h)
            de = ab.Logo.create(data, w, h, W, H, imgx, imgy).deint().create_mask(ratio)
            dev = to_device(host)                                   # the descriptor holds only its address
            s, cnt = c.scan_comb_frames(ab.yv12_clip(dev, W, H, n, True, bb), [de], prm)
            O = Oracle(oracle, data, w, h, W, H, imgx, imgy)
            ode = O.deint(ratio)
            Y = y_planes(host, W, H)
            ref = np.stack([O.scan(ode, Y[i], float((1 << bb) - 1)) for i in range(n)])
            assert np.array_equal(_bits_of(s.cpu().numpy()[:, 0]), _bits_of(ref)), (bits, w, h)
            ysz, csz = W * H, (W // 2) * (H // 2)
            U = host[:, ysz:ysz + csz].reshape(n, H // 2, W // 2)
            V = host[:, ysz + csz:].reshape(n, H // 2, W // 2)
            assert np.array_equal(cnt.cpu().numpy(), oracle.or_comb_clip(Y, U, V, prm.as_list())), (bits, w, h)
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_host_clip_several_logos(ctx, oracle, monkeypatch):
    """Host clips with 3 logos: one bounding-box ROI staged per chunk (1 MiB staging -> many chunks), one evaluation per
    logo at its offset inside the box; plus a logo of another frame size (corr1 = -1)."""
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    for bits in (8, 12):
        W, H, n = 720, 480, 150
        specs = [(64, 64, 1, 0.35, 600, 20), (48, 40, 6, 0.5, 33, 301), (96, 64, 2, 0.2, 301, 416)]
        host = make_clip_frames(n, W, H, bits, seed=bits)
        Y = y_planes(host, W, H)
        logos, refs = [], []
        for (w, h, seed, ratio, x, y) in specs:
            lg = synth.make_logo(w, h, seed=seed)
            logos.append(ab.Logo.create(lg["data"], w, h, W, H, x, y).deint().create_mask(ratio))
            O = Oracle(oracle, lg["data"], w, h, W, H, x, y)
            ode = O.deint(ratio)
            refs.append(np.stack([O.scan(ode, Y[i], float((1 << bits) - 1)) for i in range(n)]))
        other = ab.Logo.create(synth.make_logo(32, 32)["data"], 32, 32, 1920, 1080, 0, 0).deint().create_mask(0.35)
        clip = ab.yv12_clip(host, W, H, n, False, bits)
        got = ctx.scan_frames(clip, logos[:1] + [other] + logos[1:], frame0=3, nframes=n - 3)
        assert np.all(got[:, 1, 0] == 0.0) and np.all(got[:, 1, 1] == -1.0)
        for k, j in enumerate((0, 2, 3)):
            assert np.array_equal(_bits_of(got[:, j]), _bits_of(refs[k][3:])), (bits, k)
        dbuf = to_device(host)
        dev = ctx.scan_frames(ab.yv12_clip(dbuf, W, H, n, True, bits), logos).cpu().numpy()
        for k in range(3):
            assert np.array_equal(_bits_of(dev[:, k]), _bits_of(refs[k])), (bits, k)


@pytest.mark.gpu
def test_small_launch_does_not_lower_shared_memory_limit(ctx, oracle, monkeypatch):
    """The dynamic shared-memory limit of a kernel belongs to the device, not to a context: a small-logo scan-lite call
    (its score sum needs little shared memory) on another context, and on this one, must not break the next large-logo
    call here.  It used to fail with "invalid argument" at launch."""
    W, H, n = 320, 128, 6
    host = make_clip_frames(n, W, H, 8, seed=5)
    dev = to_device(host)                                       # the descriptor holds only its address
    clip = ab.yv12_clip(dev, W, H, n, True, 8)
    big = synth.make_logo(64, 64, seed=1)
    pb = ab.Logo.create(big["data"], 64, 64, W, H, 128, 32).deint().create_mask(0.35)    # 1433 features: a 185 KB bulk sum
    small = synth.make_logo(32, 32, seed=2)
    ps = ab.Logo.create(small["data"], 32, 32, W, H, 16, 16).deint().create_mask(0.35)
    O = Oracle(oracle, big["data"], 64, 64, W, H, 128, 32)
    ode = O.deint(0.35)
    Y = y_planes(host, W, H)
    ref = np.stack([O.scan(ode, Y[i], 255.0) for i in range(n)])
    monkeypatch.setenv("AMTK_SCAN_LITE", "2")
    lite = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    monkeypatch.delenv("AMTK_SCAN_LITE")
    try:
        for c in (ctx, lite):
            assert np.array_equal(_bits_of(c.scan_frames(clip, [pb]).cpu().numpy()[:, 0]), _bits_of(ref))
            lite.scan_comb_frames(clip, [ps])                         # small bulk-sum launch on the lite context
            assert np.array_equal(_bits_of(c.scan_frames(clip, [pb]).cpu().numpy()[:, 0]), _bits_of(ref))
    finally:
        lite.close()
