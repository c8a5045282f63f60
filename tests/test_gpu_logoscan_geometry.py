"""LogoScan accumulation and logo generation (amtk_scan_*, amtk_scan_logo, amtk_scan_logo_stream) across scan rectangles,
validity thresholds and frame splits, against the reference's own LogoScan::AddFrame, Normalize and GetLogo
(oracle.pyoracle.RefScan, compiled into oracle/_ref; the C port OracleScan where that was not built).

scan_border_kernel and scan_accumulate_kernel (csrc/scan_kernels.cuh) branch on the rectangle's size and on the frame
count of each add_frames call: the border loop runs more than one pass when a plane's border has over 256 pixels, the
median cut [n/4, n - n/4) falls between ranks when n is 2 mod 4, and amtk_scan_add_frames splits a call's frames over
`splits` rows of CTAs, `per` frames each (amtk_b200.cu).  The frames here are built so that every such branch decides
something: each plane's border has a chosen spread max - min (thy, thy + 1, ...), runs of equal values straddle the
median cut or not, the middle sum lands on .5 of the rounding or not, and a synthetic logo is blended over a background
that changes from frame to frame.

4:2:0 only, rectangles of even size (what the reference's GUI makes, LogoAnalyzeModel.cs rounds x, y, w and h to even).
Odd rectangles are tested for one thing only: GetLogo(clean) must not write past the caller's buffer."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth

H100_SMS = 132
THY = 12


# ---------------------------------------------------------------------------------------------------------------------
# the launch arithmetic of amtk_scan_add_frames and scan_border_kernel, restated
# ---------------------------------------------------------------------------------------------------------------------
def npix(w, h):
    return w * h + 2 * (w >> 1) * (h >> 1)


def max_splits(w, h, sms):
    """Frame splits of a call with enough frames: (8 * SMs) / pixel blocks, at least 1 (amtk_scan_add_frames)."""
    return max(1, (sms * 8) // ((npix(w, h) + 255) // 256))


def split_of(n, w, h, sms):
    """(splits, per, splits that get frames) for one add_frames call of n frames."""
    s = max(1, min(n, max_splits(w, h, sms)))
    per = -(-n // s)
    return s, per, -(-n // per)


def border_n(w, h):
    """Border pixels of a w x h plane: rows 0 and h - 1, columns 0 and w - 1 between them (scan_border_kernel's nb)."""
    return 2 * w + 2 * (h - 2)


def call_regimes(n, w, h, sms):
    s, per, used = split_of(n, w, h, sms)
    out = set()
    if per == 1:
        out.add("per=1")
    if per > 1 and used < s:
        out.add("per>1, empty trailing splits")
    if per > 1 and n % per:
        out.add("uneven last split")
    if s == 1 and n > 1:
        out.add("splits=1")
    return out


def shape_regimes(w, h):
    out = set()
    wc, hc = w >> 1, h >> 1
    if border_n(w, h) > 256:
        out.add("luma border loop > 256")
    if border_n(wc, hc) > 256:
        out.add("chroma border loop > 256")
    if border_n(wc, hc) % 4 == 2:
        out.add("chroma n = 2 mod 4")
    if (wc - 2) * (hc - 2) <= 0:
        out.add("every chroma pixel on the border")
    return out


def call_plan(w, h, sms):
    """Frame counts of the add_frames calls a sweep case makes: per = 1, per > 1 with empty trailing splits, per > 1
    with a short last split; a rectangle with one split gets three frames, then five."""
    s = max_splits(w, h, sms)
    return [3, 5] if s == 1 else [s, s + 1, 2 * s - 1]


# (frame W, H, scan x, y, w, h)
GEOMETRIES = {
    "4x4": (32, 16, 10, 6, 4, 4),
    "6x4": (32, 16, 12, 8, 6, 4),
    "64x50": (128, 96, 34, 22, 64, 50),
    "96x48": (160, 64, 40, 8, 96, 48),
    "272x64": (320, 96, 24, 16, 272, 64),
    "320x288": (352, 320, 16, 16, 320, 288),
    "1920x1080": (1920, 1080, 0, 0, 1920, 1080),
    "64x50-left": (128, 96, 0, 20, 64, 50),
    "64x50-top": (128, 96, 30, 0, 64, 50),
    "64x50-right": (128, 96, 64, 20, 64, 50),
    "64x50-bottom": (128, 96, 30, 46, 64, 50),
}

REGIMES = {"per=1", "per>1, empty trailing splits", "uneven last split", "splits=1", "luma border loop > 256",
           "chroma border loop > 256", "chroma n = 2 mod 4", "every chroma pixel on the border"}


def sweep_regimes(sms):
    got = set()
    for W, H, x, y, w, h in GEOMETRIES.values():
        got |= shape_regimes(w, h)
        for n in call_plan(w, h, sms):
            got |= call_regimes(n, w, h, sms)
    return got


def edges_touched():
    out = set()
    for W, H, x, y, w, h in GEOMETRIES.values():
        out |= {e for e, hit in (("left", x == 0), ("top", y == 0), ("right", x + w == W), ("bottom", y + h == H)) if hit}
    return out


def test_launch_arithmetic_restated():
    """The restatement against hand-computed values, then: the sweep reaches every regime on a 132-SM H100."""
    assert border_n(64, 48) == 220 and border_n(32, 24) == 108                  # the geometry the older tests use
    assert max_splits(64, 48, H100_SMS) == 58 and max_splits(320, 288, H100_SMS) == 1
    assert border_n(32, 25) % 4 == 2 and border_n(96, 48) > 256 and border_n(136, 32) > 256
    assert split_of(100, 64, 48, H100_SMS) == (58, 2, 50)
    assert all(border_n(w, h) % 2 == 0 for w in range(2, 300) for h in range(2, 40))     # n is always even
    assert sweep_regimes(H100_SMS) == REGIMES
    assert edges_touched() == {"left", "top", "right", "bottom"}
    for name, (W, H, x, y, w, h) in GEOMETRIES.items():
        assert w % 2 == 0 and h % 2 == 0 and x % 2 == 0 and y % 2 == 0 and x + w <= W and y + h <= H, name
        assert sum(call_plan(w, h, H100_SMS)) * (W * H * 3 // 2) < 64 << 20, name                  # a few MB each
    # the rectangle that gives one split reaches it through its pixel blocks (about 540 or more)
    assert (npix(320, 288) + 255) // 256 == 540


# ---------------------------------------------------------------------------------------------------------------------
# frames
# ---------------------------------------------------------------------------------------------------------------------
def border_index(w, h):
    """(rows, cols) of a plane's border in scan_border_kernel's order."""
    ys = np.concatenate([np.zeros(w, int), np.full(w, h - 1), np.repeat(np.arange(1, h - 1), 2)])
    xs = np.concatenate([np.arange(w), np.arange(w), np.tile([0, w - 1], max(0, h - 2))])
    return ys, xs


def border_multiset(rng, n, vmin, d, straddle, half):
    """n sorted border values in [vmin, vmin + d] with both ends present.  straddle: equal values on both sides of the
    cuts n/4 - 1 | n/4 and n - n/4 - 1 | n - n/4.  half: the sum of ranks [n/4, n - n/4) is nn/2 mod nn, i.e. the
    rounded mean sits on .5 (best effort: a narrow spread may leave no room)."""
    lo, hi = n // 4, n - n // 4
    nn = hi - lo
    if straddle or d < 2:
        s = np.sort(rng.integers(vmin, vmin + d + 1, n))
    else:                   # three bands of values, so that the ranks on each side of a cut differ
        b1, b2 = vmin + d // 3, vmin + 2 * d // 3
        s = np.concatenate([rng.integers(vmin, b1 + 1, lo), rng.integers(b1 + 1, b2 + 1, nn), rng.integers(b2 + 1, vmin + d + 1, n - hi)])
    s[0], s[-1] = vmin, vmin + d
    s.sort()
    if straddle and lo >= 1:
        s[lo] = s[lo - 1]
        s[hi - 1] = s[hi]
    if half:
        k = int((nn // 2 - int(s[lo:hi].sum())) % nn)
        j = hi - 2 if straddle else hi - 1
        while k and j >= lo + (1 if straddle else 0):
            top = (s[j + 1] - (0 if straddle or j < hi - 1 or d < 2 else 1)) if j + 1 < n else vmin + d
            step = min(k, max(0, int(top) - int(s[j])))
            s[j] += step
            k -= step
            j -= 1
    return s


class Gen:
    """Deterministic 4:2:0 frames: noise outside the rectangle; inside it each plane's border is a chosen multiset and
    the interior is a fixed synthetic logo blended over the frame's background level in about three frames of four."""

    def __init__(self, W, H, x, y, w, h, seed):
        self.W, self.H, self.x, self.y, self.w, self.h = W, H, x, y, w, h
        self.rng = np.random.default_rng(seed)
        self.planes = [(w, h), (w >> 1, h >> 1), (w >> 1, h >> 1)]
        # synth.make_logo's opacity blob (Y at 230, chroma at half strength towards 128); none in odd rectangles
        self.alpha = [np.zeros((ph, pw)) for pw, ph in self.planes]
        self.color = [230.0, 128.0, 128.0]
        if w % 2 == 0 and h % 2 == 0:
            lg = synth.make_logo(w, h, seed=seed & 7)
            self.alpha = [lg["alpha8"] / 256.0, lg["alphaC"] / 256.0, lg["alphaC"] / 256.0]

    def frames(self, spreads, levels=None, logo=True, straddle=None, half=None):
        """spreads: (n, 3) border max - min per frame and plane (clamped to 0..255); levels: (n, 3) border minima or None
        (random); straddle, half: (n, 3) bools or None (random)."""
        W, H, rng = self.W, self.H, self.rng
        n = len(spreads)
        ysz, csz = W * H, (W >> 1) * (H >> 1)
        out = rng.integers(0, 256, (n, ysz + 2 * csz), dtype=np.uint8)
        d = np.clip(np.asarray(spreads), 0, 255)
        straddle = rng.random((n, 3)) < 0.5 if straddle is None else straddle
        half = rng.random((n, 3)) < 0.6 if half is None else half
        on = (rng.random(n) < 0.75) & logo                  # the logo shows in about three frames of four
        for i in range(n):
            for p, (pw, ph) in enumerate(self.planes):
                if p == 0:
                    plane = out[i, :ysz].reshape(H, W)[self.y:self.y + ph, self.x:self.x + pw]
                else:
                    o = ysz + (p - 1) * csz
                    plane = out[i, o:o + csz].reshape(H >> 1, W >> 1)[self.y >> 1:(self.y >> 1) + ph,
                                                                      self.x >> 1:(self.x >> 1) + pw]
                dp = int(d[i, p])
                vmin = int(levels[i, p]) if levels is not None else int(rng.integers(0, 256 - dp))
                ys, xs = border_index(pw, ph)
                s = border_multiset(rng, len(ys), vmin, dp, bool(straddle[i, p]), bool(half[i, p]))
                lo, hi = len(s) // 4, len(s) - len(s) // 4
                inner = np.full((ph, pw), float(s[lo:hi].mean()))          # the background level AddFrame finds
                if on[i]:
                    inner = inner * (1 - self.alpha[p]) + self.alpha[p] * self.color[p]
                plane[:] = np.clip(np.rint(inner), 0, 255).astype(np.uint8)
                plane[ys, xs] = rng.permutation(s)
        return out

    def sweep_spreads(self, n):
        """Every fifth frame at exactly THY in every plane; frames 1, 2, 3 of every seven one over THY in Y, U, V; the
        rest between 2 and THY (a spread of 2 or more leaves room for the .5 rounding)."""
        d = self.rng.integers(2, THY + 1, (n, 3))
        d[::5] = THY
        for i in range(n):
            if 1 <= i % 7 <= 3:
                d[i, i % 7 - 1] = THY + 1
        return d

    def random_spreads(self, n, thy):
        """Mostly valid frames (spread <= thy in every plane), some at exactly thy, about one in six with one plane
        at thy + 1."""
        rng = self.rng
        d = rng.integers(0, max(0, thy) + 1, (n, 3))
        d[rng.random((n, 3)) < 0.25] = thy
        bad = rng.random(n) < 0.17
        d[bad, rng.integers(0, 3, int(bad.sum()))] = thy + 1
        return d


def pattern(n, k):
    """(n, 3) bools, False where (frame + plane) % k == 0: both values in every plane even for a few frames."""
    i = np.arange(n)[:, None] + np.arange(3)[None, :]
    return i % k != 0


def rois(frames, W, H, x, y, w, h):
    n = frames.shape[0]
    ysz, csz = W * H, (W >> 1) * (H >> 1)
    Y = frames[:, :ysz].reshape(n, H, W)[:, y:y + h, x:x + w]
    U = frames[:, ysz:ysz + csz].reshape(n, H >> 1, W >> 1)[:, y >> 1:(y >> 1) + (h >> 1), x >> 1:(x >> 1) + (w >> 1)]
    V = frames[:, ysz + csz:].reshape(n, H >> 1, W >> 1)[:, y >> 1:(y >> 1) + (h >> 1), x >> 1:(x >> 1) + (w >> 1)]
    return Y, U, V


def border_facts(frames, W, H, x, y, w, h):
    """Per frame and plane: (max - min, equal values straddle a cut, the rounded mean sits on .5)."""
    out = []
    for P, (pw, ph) in zip(rois(frames, W, H, x, y, w, h), [(w, h), (w >> 1, h >> 1), (w >> 1, h >> 1)]):
        ys, xs = border_index(pw, ph)
        s = np.sort(P[:, ys, xs].astype(np.int64), axis=1)
        n = s.shape[1]
        lo, hi = n // 4, n - n // 4
        spread = s[:, -1] - s[:, 0]
        strad = (s[:, lo - 1] == s[:, lo]) | (s[:, hi - 1] == s[:, hi]) if lo >= 1 else np.zeros(len(s), bool)
        half = 2 * (s[:, lo:hi].sum(axis=1) % (hi - lo)) == hi - lo
        out.append((spread, strad, half))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the oracle and the comparison
# ---------------------------------------------------------------------------------------------------------------------
def scan_class(po):
    return po.RefScan if po.ref_available() else po.OracleScan


def oracle_scan(po, frames, geom, thy, select=None):
    W, H, x, y, w, h = geom
    sc = scan_class(po)(w, h, thy)
    Y, U, V = rois(frames, W, H, x, y, w, h)
    valid = []
    for i in range(frames.shape[0]):
        valid.append(0 if select is not None and not select[i] else int(sc.add_frame(Y[i], U[i], V[i])))
    return sc, valid


def assert_same(acc, valid, sc, ref_valid, where):
    assert list(map(int, valid)) == ref_valid, where
    assert acc.num_valid == sc.nframes == sum(ref_valid), where
    assert np.array_equal(acc.sums(), sc.sums()), where                  # exact integers in doubles
    got = []
    for clean in (False, True):
        a, b = acc.get_logo(255, clean), sc.get_logo(255, clean)
        assert (a is None) == (b is None), (where, clean)
        if a is not None:
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (where, clean)
        got.append(a)
    return got


def device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def clip_of(frames, W, H, on_device=True):
    return ab.yv12_clip(frames, W, H, frames.shape[0], on_device)


# ---------------------------------------------------------------------------------------------------------------------
# 2: the geometry sweep
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_sweep_reaches_every_regime_on_this_device():
    sms = device_sms()
    assert sweep_regimes(sms) == REGIMES, sms


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GEOMETRIES))
def test_scan_geometry_matches_reference(ctx, oracle, name):
    geom = GEOMETRIES[name]
    W, H, x, y, w, h = geom
    sms = device_sms()
    plan = call_plan(w, h, sms)
    n = sum(plan)
    g = Gen(W, H, x, y, w, h, seed=zlib.crc32(name.encode()))
    frames = g.frames(g.sweep_spreads(n), straddle=pattern(n, 2), half=pattern(n, 3))
    # the frames do what they are for: valid and invalid frames, straddled cuts and .5 rounding in every plane
    facts = border_facts(frames, *geom)
    for p, (spread, strad, half) in enumerate(facts):
        assert (spread == THY).any() and (spread == THY + 1).any(), (name, p)
        assert strad.any() and (~strad).any() and half.any() and (~half).any(), (name, p)
    dev = torch.from_numpy(frames).cuda()
    clip = clip_of(dev, W, H)
    acc = ctx.logo_scan(w, h, THY)
    valid, f0 = [], 0
    for k in plan:
        valid.append(acc.add_frames(clip, x, y, f0, k))
        f0 += k
    sc, rv = oracle_scan(oracle, frames, geom, THY)
    assert 0 < sum(rv) < n
    logos = assert_same(acc, np.concatenate(valid), sc, rv, name)
    assert logos[0] is not None and logos[1] is not None, name      # the fit is not degenerate


# ---------------------------------------------------------------------------------------------------------------------
# 3: validity
# ---------------------------------------------------------------------------------------------------------------------
VGEOM = (128, 96, 34, 22, 64, 50)


def threshold_spreads(g, thy, n=72):
    """Frame i has plane i % 3 at spread thy + (i // 3) % 2 (exactly thy, or one over), the others at most thy."""
    rng = g.rng
    top = min(max(thy, 0), 255)
    d = rng.integers(0, top + 1, (n, 3))
    for i in range(n):
        d[i, i % 3] = thy + (i // 3) % 2
    return np.clip(d, 0, 255)


@pytest.mark.gpu
@pytest.mark.parametrize("thy", [-1, 0, 1, 12, 254, 255])
def test_threshold_edges(ctx, oracle, thy):
    W, H, x, y, w, h = VGEOM
    g = Gen(*VGEOM, seed=1000 + thy)
    d = threshold_spreads(g, thy)
    frames = g.frames(d)
    want = [int(all(int(v) <= thy for v in row)) for row in d]         # max - min > thy rejects (:639-649)
    dev = torch.from_numpy(frames).cuda()
    acc = ctx.logo_scan(w, h, thy)
    valid = acc.add_frames(clip_of(dev, W, H), x, y)
    assert valid.tolist() == want
    if 0 <= thy < 255:                   # frames exactly at thy pass and one over fails, in Y, U and V each
        for p in range(3):
            at = [i for i in range(len(d)) if i % 3 == p and (i // 3) % 2 == 0]
            over = [i for i in range(len(d)) if i % 3 == p and (i // 3) % 2 == 1]
            assert all(want[i] for i in at) and not any(want[i] for i in over), p
    sc, rv = oracle_scan(oracle, frames, VGEOM, thy)
    logos = assert_same(acc, valid, sc, rv, thy)
    if thy < 0:
        assert sum(rv) == 0 and logos == [None, None]                    # no valid frames: "Insufficient logo frames"


@pytest.mark.gpu
def test_frame_select(ctx, oracle):
    W, H, x, y, w, h = VGEOM
    g = Gen(*VGEOM, seed=77)
    n = 150
    frames = g.frames(g.random_spreads(n, THY))
    clip = clip_of(torch.from_numpy(frames).cuda(), W, H)
    rng = np.random.default_rng(5)
    for what, sel in (("none", np.zeros(n, np.uint8)), ("all", np.ones(n, np.uint8)),
                      ("random", (rng.random(n) < 0.5).astype(np.uint8))):
        acc = ctx.logo_scan(w, h, THY)
        valid = np.concatenate([acc.add_frames(clip, x, y, 0, 61, select=sel[:61]),
                                acc.add_frames(clip, x, y, 61, n - 61, select=sel[61:])])
        sc, rv = oracle_scan(oracle, frames, VGEOM, THY, select=sel)
        assert_same(acc, valid, sc, rv, what)
        if what == "none":
            assert acc.get_logo(255) is None and not valid.any()
        else:
            assert sum(rv) > 0


def constant_background_frames(g, n, levels):
    """Every frame has the same border multiset in every plane (so the same background), the interior varies."""
    rng = np.random.default_rng(9)
    frames = g.frames(np.full((n, 3), 6), levels=np.tile(levels, (n, 1)), straddle=np.ones((n, 3), bool),
                      half=np.zeros((n, 3), bool))
    W, H, x, y, w, h = g.W, g.H, g.x, g.y, g.w, g.h
    # one border multiset for all frames: copy frame 0's rectangle borders, keep each frame's own interior
    Y, U, V = rois(frames, W, H, x, y, w, h)
    for P, (pw, ph) in zip((Y, U, V), g.planes):
        ys, xs = border_index(pw, ph)
        for i in range(1, n):
            P[i, ys, xs] = rng.permutation(P[0, ys, xs])
    return frames


@pytest.mark.gpu
def test_insufficient_logo_frames(ctx, oracle, tmp_path):
    """GetLogo returns nullptr (:847-849) when no frame is valid, and when every valid frame has the same background
    (the fit of foreground on background has no determinant); amtk_scan_logo fails with the reference's message."""
    W, H, x, y, w, h = VGEOM
    g = Gen(*VGEOM, seed=31)
    n = 40
    cases = {"no valid frame": (g.frames(np.full((n, 3), THY + 1)), THY),
             "constant background": (constant_background_frames(g, n, [100, 128, 140]), THY)}
    for what, (frames, thy) in cases.items():
        dev = torch.from_numpy(frames).cuda()
        acc = ctx.logo_scan(w, h, thy)
        valid = acc.add_frames(clip_of(dev, W, H), x, y)
        sc, rv = oracle_scan(oracle, frames, VGEOM, thy)
        assert assert_same(acc, valid, sc, rv, what) == [None, None], what
        assert sum(rv) == (0 if what == "no valid frame" else n), what
        with pytest.raises(ab.AmtkError, match="Insufficient logo frames"):
            ctx.scan_logo(clip_of(dev, W, H), str(tmp_path / "x.lgd"), x, y, w, h, thy, 100000)


# ---------------------------------------------------------------------------------------------------------------------
# 4: host clips staged through many ROI windows
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("rect", [(37, 23, 272, 64), (50, 30, 320, 288), (368, 296, 272, 64)])
def test_staged_host_clips_equal_device_clip(ctx, oracle, monkeypatch, rect):
    """AMTK_STAGE_MB=1 cuts many ROI windows; rectangles at x, y off the window alignment (32 luma bytes, 2 rows), and
    one against the right and bottom edges of the frame."""
    W, H = 640, 360
    x, y, w, h = rect
    geom = (W, H, x, y, w, h)
    g = Gen(*geom, seed=x * 1000 + y)
    n = 130
    frames = g.frames(g.random_spreads(n, THY))
    dev = torch.from_numpy(frames).cuda()

    def run(clip):
        acc = ctx.logo_scan(w, h, THY)
        valid = np.concatenate([acc.add_frames(clip, x, y, 0, 57), acc.add_frames(clip, x, y, 57, n - 57)])
        return valid, acc.num_valid, acc.sums(), [acc.get_logo(255, c) for c in (False, True)]

    want = run(clip_of(dev, W, H))
    assert want[1] > 0
    sc, rv = oracle_scan(oracle, frames, geom, THY)
    acc = ctx.logo_scan(w, h, THY)
    assert_same(acc, acc.add_frames(clip_of(dev, W, H), x, y), sc, rv, rect)
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    pinned = torch.from_numpy(frames.copy()).pin_memory()
    for kind, buf in (("pageable", frames), ("pinned", pinned)):
        before = ctx.launches
        got = run(clip_of(buf, W, H, on_device=False))
        assert (ctx.launches - before) // 2 >= 4, kind        # two kernels per ROI window: two or more per call
        assert got[0].tolist() == want[0].tolist() and got[1] == want[1], kind
        assert np.array_equal(got[2], want[2]), kind
        for a, b in zip(got[3], want[3]):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), kind


# ---------------------------------------------------------------------------------------------------------------------
# 5: the whole pipeline and the frame stream
# ---------------------------------------------------------------------------------------------------------------------
def compose_pipeline(po, frames, geom, thy, maxf):
    """ScanLogo (LogoScan.hpp:1058-1098) composed from the oracle's pieces, as test_scan_logo_pipeline: MakeInitialLogo
    up to maxf valid frames, ReMakeLogo twice, the final data (None: "Insufficient logo frames")."""
    W, H, x, y, w, h = geom
    Y, U, V = rois(frames, W, H, x, y, w, h)
    sc = scan_class(po)(w, h, thy)
    stored = []
    for i in range(frames.shape[0]):
        if len(stored) >= maxf:
            break
        if sc.add_frame(Y[i], U[i], V[i]):
            stored.append(i)
    data = sc.get_logo(255, False)
    if data is None:
        return None, stored
    for _ in range(2):
        de = po.OracleLogo.create(data, w, h, w, h, 0, 0).deint().create_mask(0.1)
        keep = []
        for i in stored:
            ry = np.ascontiguousarray(Y[i])
            dd = np.zeros(w * h + 8, np.float32)
            po.oracle_lib().amtk_or_deint_y_u8(dd.ctypes.data_as(po.c_float_p), ry.ctypes.data_as(po.c_u8_p), w, w, h)
            res = [abs(np.float32(de.evaluate(dd, 255.0, np.float32(0.1) * np.float32(fi)))) for fi in range(20)]
            if int(np.argmin(res)) > 8:
                keep.append(i)
        sc2 = scan_class(po)(w, h, thy)
        for i in keep:
            sc2.add_frame(Y[i], U[i], V[i])
        data = sc2.get_logo(255, True)
        if data is None:
            return None, stored
    return data, stored


PIPELINE = {"64x50": ((128, 96, 34, 22, 64, 50), 300, "inside a stack batch"),
            "96x48": ((160, 64, 40, 8, 96, 48), 150, 60),
            "272x64": ((320, 96, 24, 16, 272, 64), 120, 100000)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PIPELINE))
def test_pipeline_and_stream(ctx, oracle, tmp_path, name):
    geom, n, maxf = PIPELINE[name]
    W, H, x, y, w, h = geom
    g = Gen(*geom, seed=len(name) * 7919)
    frames = g.frames(g.random_spreads(n, THY))
    _, rv = oracle_scan(oracle, frames, geom, THY)
    if maxf == "inside a stack batch":
        # the cut-off frame is read inside the second batch of 200 (scan_stack_kernel), not at its end
        cut = next(r for r in range(241, 290) if rv[r - 1])
        maxf = sum(rv[:cut])
    want, stored = compose_pipeline(oracle, frames, geom, THY, maxf)
    assert want is not None and len(stored) == min(maxf, sum(rv))
    if isinstance(PIPELINE[name][2], str):
        assert 200 < stored[-1] + 1 < 300 and stored[-1] < n - 10
    dev = torch.from_numpy(frames).cuda()
    whole = str(tmp_path / "whole.lgd")
    ctx.scan_logo(clip_of(dev, W, H), whole, x, y, w, h, THY, maxf, service_id=21)
    got = ab.Logo.load(whole)
    gi = got.info()
    assert (gi.w, gi.h, gi.imgw, gi.imgh, gi.imgx, gi.imgy) == (w, h, W, H, x, y)
    assert np.array_equal(got.tables()["data"].view(np.uint32), want.view(np.uint32))
    s = ctx.scan_logo_stream(x, y, w, h, THY, maxf)
    for i in range(n):
        s.send(ab.yv12_clip(dev[i:i + 1], W, H, 1, True), i + 1, n)
    streamed = str(tmp_path / "stream.lgd")
    s.finish(streamed, 21)
    assert s.counts()[1] == len(stored)
    s.close()
    assert open(streamed, "rb").read() == open(whole, "rb").read()


# ---------------------------------------------------------------------------------------------------------------------
# odd rectangles: GetLogo(clean) stays inside the caller's buffer
# ---------------------------------------------------------------------------------------------------------------------
def odd_frames(W, H, x, y, w, h, n):
    """Flat Y, U and V rectangles whose level changes per frame (every pixel fits a = 1, b = 0), except chroma pixel
    (0, 0): in U it is 255 - background (a = -1, b = 1), in V it swings over 0..253 with a background of 254 or 255
    (a about 0.007, b about 0.995).  The luma pixels of an odd rectangle's last row (or column) map to chroma index
    nc, past the chroma planes; read from this layout, U's b and V's a and b of pixel 0 sit at aU[nc], bU[nc] and
    aV[nc], and the float after the data at bV[nc].  With that float near 0 the pixel looks like "no logo", so a
    finaliser that indexes past the planes resets it and writes 0 there."""
    rng = np.random.default_rng(w * 16 + h)
    ysz, csz = W * H, (W >> 1) * (H >> 1)
    out = rng.integers(0, 256, (n, ysz + 2 * csz), dtype=np.uint8)
    wc, hc = w >> 1, h >> 1
    for i in range(n):
        Y = out[i, :ysz].reshape(H, W)
        U = out[i, ysz:ysz + csz].reshape(H >> 1, W >> 1)
        V = out[i, ysz + csz:].reshape(H >> 1, W >> 1)
        by, bu, bv = 40 + (37 * i) % 150, 100 + (13 * i) % 50, 254 + (i * 5 // 3) % 2
        Y[y:y + h, x:x + w] = by
        U[y >> 1:(y >> 1) + hc, x >> 1:(x >> 1) + wc] = bu
        V[y >> 1:(y >> 1) + hc, x >> 1:(x >> 1) + wc] = bv
        U[y >> 1, x >> 1] = 255 - bu
        V[y >> 1, x >> 1] = rng.integers(128, 254) if bv == 255 else rng.integers(0, 128)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(7, 5), (9, 6), (6, 7)])
def test_odd_rectangle_get_logo_stays_in_buffer(ctx, w, h):
    """amtk_scan_get_logo on an odd rectangle into a buffer with a sentinel tail: the tail must be untouched, with
    clean false and true.  The sentinel is a tiny float (1e-30), which reads as b = 0 (see odd_frames)."""
    W, H, x, y, n = 32, 16, 4, 4, 24
    clip = clip_of(torch.from_numpy(odd_frames(W, H, x, y, w, h, n)).cuda(), W, H)
    acc = ctx.logo_scan(w, h, 255)
    assert acc.add_frames(clip, x, y).all()
    tail = 64
    sentinel = np.float32(1e-30).view(np.uint32)
    for clean in (0, 1):
        buf = np.full(acc.ndata + tail, sentinel, np.uint32)
        ok = ctx.L.amtk_scan_get_logo(acc.h, 255, clean, buf.ctypes.data_as(C.POINTER(C.c_float)))
        assert ok, ctx.L.amtk_last_error().decode()
        assert (buf[acc.ndata:] == sentinel).all(), (clean, np.flatnonzero(buf[acc.ndata:] != sentinel))
        assert np.isfinite(buf[:acc.ndata].view(np.float32)).all()
