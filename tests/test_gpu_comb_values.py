"""The combing counters at their edges: thresholds hit exactly, and every counter at its maximum at once.

Each kernel form compares responses with thresholds in its own way: byte tricks and fp16 bit patterns at 8 bits, biased
fp16 bit patterns behind an `8192 + min(t, 8191)` clamp in the 10-bit warp-stream form, fp32 in the CTA ring, plain
integers in the generic kernel; the 8-bit and 10-bit forms add pair-coded mask sums that stay valid only below 65536 per
tile-frame.  Random frames rarely put a pixel exactly on a threshold, so a `>=` that became `>` or a clamp one too low
would pass them.  Here every one of the 12 counters has many pixels exactly at its threshold and at threshold - 1 (a CPU
test proves it: the spec's counts for th and th + 1 differ for every counter), and saturated frames put every counter
at its closed-form maximum."""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from test_gpu_comb_plans import _ctx

FORMS = {8: {"band": {}, "warp": {"AMTK_COMB_WS_BAND": "0"}, "cta": {"AMTK_COMB_WS": "0"}, "mma": {"AMTK_COMB_MMA": "1"},
             "generic": {"AMTK_COMB_GENERIC": "1"}},
         10: {"cta": {}, "ws10": {"AMTK_COMB_WS10": "1"}, "generic": {"AMTK_COMB_GENERIC": "1"}},
         12: {"cta": {}, "generic": {"AMTK_COMB_GENERIC": "1"}},
         16: {"cta": {}, "generic": {"AMTK_COMB_GENERIC": "1"}}}
MAXR = {8: 1530, 10: 6138, 12: 24570, 16: 393210}           # 6 * maxv: the largest response

# (thM, thS, thL) luma, chroma.  "ramp": frames built around the thresholds (every counter discriminates);
# "edge": near-saturated frames (responses 6*maxv, 6*maxv - 1 and a few below; moves maxv and maxv - 1).
THRESHOLDS = {
    8: [("ramp", (7, 100, 701), (13, 64, 1000)), ("ramp", (128, 300, 601), (1, 1, 2)), ("ramp", (127, 6, 7), (64, 1, 455)),
        ("edge", (128, 1530, 1529), (128, 1529, 1530))],
    10: [("ramp", (40, 900, 3001), (1, 1, 2)), ("ramp", (600, 1500, 2400), (300, 77, 1201)),
         ("edge", (1023, 6138, 6137), (1022, 6137, 6138)), ("edge", (1024, 6139, 8191), (2048, 8192, 100000))],
    12: [("ramp", (100, 5000, 12001), (3, 9, 20000)), ("ramp", (2048, 7, 6001), (3900, 600, 601)),
         ("edge", (4095, 24570, 24569), (4094, 24569, 24570))],
    16: [("ramp", (32768, 90000, 150001), (5, 77, 300001)), ("ramp", (1, 1, 2), (30000, 120000, 120001)),
         ("edge", (32768, 393210, 393209), (32767, 393209, 393210))],
}


def _ramp_plane(rng, n, h, w, th, maxv):
    """Rows alternating L + D and L per column (response 6D at every row of both fields), D ramping around thS/6 in even
    columns and thL/6 in odd ones, +-2 of noise per sample; odd frames add thM (moves thM + -4..4)."""
    thM, thS, thL = th
    T = np.where(np.arange(w) % 2 == 0, thS, thL)
    D = np.maximum(0, np.round(T / 6).astype(np.int64) + (np.arange(w) // 2) % 3 - 1)
    L = np.clip((maxv - D - thM) // 2, 2, None)
    even = (np.arange(h) % 2 == 0)[:, None]
    out = np.empty((n, h, w), np.int64)
    for k in range(n):
        out[k] = L[None, :] + D[None, :] * even + rng.integers(-2, 3, (h, w)) + (thM if k % 2 else 0)
    return np.clip(out, 0, maxv)


def _edge_plane(rng, n, h, w, maxv):
    """Rows alternating 0 / maxv, inverted every frame, with 3 % of the samples one step inside the range."""
    rows = (np.arange(h)[None, :, None] + np.arange(n)[:, None, None]) % 2
    out = np.broadcast_to(rows * maxv, (n, h, w)).astype(np.int64)
    hit = rng.random((n, h, w)) < 0.03
    return np.where(hit, np.where(out == 0, 1, maxv - 1), out)


def make_frames(bits, kind, th_y, th_c, W=200, H=70, n=6, seed=1):
    """Packed planes (Y, U, V) as (n, rows, cols) arrays of uint8 / uint16."""
    maxv = (1 << bits) - 1
    rng = np.random.default_rng(seed + bits)
    dt = np.uint8 if bits == 8 else np.uint16
    if kind == "ramp":
        planes = [_ramp_plane(rng, n, H, W, th_y, maxv), _ramp_plane(rng, n, H // 2, W // 2, th_c, maxv),
                  _ramp_plane(rng, n, H // 2, W // 2, th_c, maxv)]
    else:
        planes = [_edge_plane(rng, n, H, W, maxv), _edge_plane(rng, n, H // 2, W // 2, maxv), _edge_plane(rng, n, H // 2, W // 2, maxv)]
    return [p.astype(dt) for p in planes]


def _counts(po, planes, th6):
    return po.or_comb_clip(*planes, list(th6))


def _pack(planes):
    n = planes[0].shape[0]
    return np.concatenate([p.reshape(n, -1) for p in planes], axis=1)


def _cases():
    return [(bits, i) for bits in sorted(THRESHOLDS) for i in range(len(THRESHOLDS[bits]))]


@pytest.mark.parametrize("bits,i", _cases())
def test_frames_put_pixels_on_every_threshold(oracle, bits, i):
    """th and th + 1 give different counts for every counter (for edge sets: every counter whose threshold a sample can
    reach), so a kernel that compares one step off cannot match the spec."""
    kind, ty, tc = THRESHOLDS[bits][i]
    planes = make_frames(bits, kind, ty, tc)
    th6 = ty + tc
    a = _counts(oracle, planes, th6)
    b = _counts(oracle, planes, [t + 1 for t in th6])
    maxv = (1 << bits) - 1
    top = lambda j: maxv if j % 3 == 0 else MAXR[bits]            # the largest move / response
    reach = [top(j) - 1 <= th6[j] <= top(j) for j in range(6)]     # edge frames put samples on these two values only
    for c in range(12):
        j = (c // 6) * 3 + c % 3
        if kind == "ramp" or reach[j]:
            assert a[1:, c].sum() != b[1:, c].sum(), (bits, th6, c)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("bits,form", [(b, f) for b in sorted(FORMS) for f in FORMS[b]])
def test_exact_thresholds(oracle, monkeypatch, bits, form):
    c = _ctx(monkeypatch, FORMS[bits][form])
    try:
        for kind, ty, tc in THRESHOLDS[bits]:
            for (W, H, n) in ((200, 70, 6), (320, 136, 5)):
                planes = make_frames(bits, kind, ty, tc, W, H, n)
                prm = ab.default_comb_params()
                prm.th_move_y, prm.th_shima_y, prm.th_lshima_y = ty
                prm.th_move_c, prm.th_shima_c, prm.th_lshima_c = tc
                ref = _counts(oracle, planes, ty + tc)
                f = _pack(planes)
                buf = torch.from_numpy(f.view(np.int16) if f.dtype == np.uint16 else f).cuda()
                clip = ab.yv12_clip(buf, W, H, n, True, bits)
                got = c.comb_frames(clip, prm).cpu().numpy()
                assert np.array_equal(got, ref), (form, bits, ty, tc, W, np.argwhere(got != ref)[:5])
                part = np.concatenate([c.comb_frames(clip, prm, 0, 2).cpu().numpy(), c.comb_frames(clip, prm, 2, n - 2).cpu().numpy()])
                assert np.array_equal(part, ref), (form, bits, ty, tc, W, "ranges")
    finally:
        c.close()


def saturated(bits, W, H, n):
    maxv = (1 << bits) - 1
    planes = []
    for (h, w) in ((H, W), (H // 2, W // 2), (H // 2, W // 2)):
        rows = (np.arange(h)[None, :, None] + np.arange(n)[:, None, None]) % 2
        planes.append(np.broadcast_to(rows * maxv, (n, h, w)).astype(np.uint8 if bits == 8 else np.uint16))
    return planes


def saturated_counts(W, H, n):
    """Closed form: every sample moves by maxv on every frame after the first, every row in [2, H-2) responds 6*maxv."""
    out = np.zeros((n, 12), np.int64)
    for base, (w, h, k) in ((0, (W, H, 1)), (6, (W // 2, H // 2, 2))):
        for f in (0, 1):
            rows = len(range(f, h, 2))
            inner = len([y for y in range(2, h - 2) if y % 2 == f])
            out[1:, base + 3 * f] = k * w * rows
            out[:, base + 3 * f + 1] = out[:, base + 3 * f + 2] = k * w * inner
    return out


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("bits,form", [(b, f) for b in sorted(FORMS) for f in FORMS[b]])
def test_saturated_counters(oracle, monkeypatch, bits, form):
    """Every counter at its maximum at once (the pair-coded sums nearest their limit), and zero one step above it."""
    W, H, n = 1024, 272, 3
    maxv = (1 << bits) - 1
    thM = min(maxv, 128 if bits == 8 else 32768)
    planes = saturated(bits, W, H, n)
    f = _pack(planes)
    want = saturated_counts(W, H, n)
    c = _ctx(monkeypatch, FORMS[bits][form])
    try:
        buf = torch.from_numpy(f.view(np.int16) if f.dtype == np.uint16 else f).cuda()
        clip = ab.yv12_clip(buf, W, H, n, True, bits)
        for above in (0, 1):
            prm = ab.default_comb_params()
            m = maxv + 1 if above and maxv + 1 <= (128 if bits == 8 else 32768) else thM
            s = MAXR[bits] + above
            prm.th_move_y, prm.th_shima_y, prm.th_lshima_y, prm.th_move_c, prm.th_shima_c, prm.th_lshima_c = m, s, s, m, s, s
            ref = _counts(oracle, planes, prm.as_list())
            exp = want.copy()
            if above:
                exp[:, [1, 2, 4, 5, 7, 8, 10, 11]] = 0
                if m > maxv:
                    exp[:, [0, 3, 6, 9]] = 0
            assert np.array_equal(ref, exp), (bits, above)
            got = c.comb_frames(clip, prm).cpu().numpy()
            assert np.array_equal(got, exp), (form, bits, above, np.argwhere(got != exp)[:5])
    finally:
        c.close()
