"""Every entry point on frames in AviSynth's own plane order: Y, then V, then U.

AviSynth's YV12 and its generic 4:2:0 formats are "V plane first" (avisynth.h, CS_VPlaneFirst), so a frame handed over by a
real filter chain has off_v < off_u, while a clip built by `yv12_clip` has U first.  The kernels must take U and V from the
descriptor's offsets wherever they lie: the combing pass's U|V pair class (per-warp form), which reads both remainder
columns through one 4-D tensor map whose plane stride is off_v - off_u, must switch off; ROI staging of host clips must move
each plane from its own offset and write erased rectangles back to the same place; weave must read and write the planes it
is told.  Every result here must equal the U-first clip's result and the oracle's, on packed frames and on frames with
64-byte-padded rows, gaps between the planes and a frame stride that is not a whole number of rows; padding and gaps are
poisoned and must stay untouched."""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from test_gpu_erase import erase_reference, logo_data
from test_gpu_frame_layouts import COMB_SETTINGS, Layout, _dev, _knob_ctx, _np, _packed_clip, _to10, _bits_of
from test_gpu_logo_plans import Oracle

pytestmark = pytest.mark.gpu


class VFirst(Layout):
    """Layout with the V plane before the U plane.  packed: pitches = row bytes, no gaps, frame stride = payload."""

    def __init__(self, W, H, bits, pitch_y=None, pitch_uv=None, gap=0, packed=False):
        bps = 1 if bits == 8 else 2
        if packed:
            pitch_y, pitch_uv, gap = W * bps, (W // 2) * bps, 0
        super().__init__(W, H, bits, pitch_y, pitch_uv, gap)
        self.off_u, self.off_v = self.off_v, self.off_u              # the frame stride already ends after the later plane
        if packed:
            self.fs = self.off_u + self.puv * (H // 2)
        assert self.off_v < self.off_u


# (W, H, pitch_y, pitch_uv, gap) in samples of 8-bit clips (doubled at 16-bit containers); None = row rounded up to 64 bytes.
# 320x120: 160-byte chroma rows end 32 bytes past a 128-byte tile (64 at 10 bits), so the per-warp form pairs U and V of a
# U-first clip.  200x100_row8: rows 8 bytes longer than 16-byte multiples, no TMA (generic kernel, plain loads).
GEOMS = {
    "320x120": (320, 120, None, None, 0),
    "720x480": (720, 480, None, None, 32),
    "1440x1080": (1440, 1080, None, None, 0),
    "200x100_row8": (200, 100, 208, 108, 0),
}


def _frames(W, H, n, **kw):
    return synth.make_frames(2, n, W, H, device="cpu", logo_period=10, **kw).numpy()


def _layouts(name, bits):
    W, H, py, puv, gap = GEOMS[name]
    s = 1 if bits == 8 else 2
    return [VFirst(W, H, bits, packed=True), VFirst(W, H, bits, py * s if py else None, puv * s if puv else None, gap)]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(GEOMS))
def test_comb_on_v_first_frames(ctx, oracle, monkeypatch, name):
    """On ONE context per setting: U-first, then V-first packed and padded, then U-first again, whole clips and range calls
    with a halo frame -- so a launch plan cached for one plane order is offered to the other."""
    W, H = GEOMS[name][:2]
    n = 4 if W > 1000 else 9
    f8 = _frames(W, H, n, mode="telecine")
    prm = ab.default_comb_params()
    p10 = ab.default_comb_params()
    p10.th_move_y, p10.th_shima_y, p10.th_lshima_y, p10.th_move_c, p10.th_shima_c, p10.th_lshima_c = 80, 48, 144, 96, 64, 192
    data = {}
    for bits in (8, 10):
        f = f8 if bits == 8 else _to10(f8)
        Y, U, V = [p.view(f.dtype) for p in Layout(W, H, bits).planes(f)]
        ref = oracle.or_comb_clip(Y, U, V, (prm if bits == 8 else p10).as_list())
        assert ref[:, 6:].sum() > 0
        data[bits] = (f, ref, [(L, L.pack(f)) for L in _layouts(name, bits)])
    for env, bits in COMB_SETTINGS:
        f, ref, lays = data[bits]
        p = prm if bits == 8 else p10
        c = _knob_ctx(monkeypatch, env)
        try:
            pclip, pbuf = _packed_clip(f, W, H, bits, True)
            assert np.array_equal(_np(c.comb_frames(pclip, p)), ref), (env, bits, "U first")
            for L, buf in lays:
                dbuf = _dev(buf)
                d = L.desc(dbuf, True)
                got = _np(c.comb_frames(d, p))
                assert np.array_equal(got, ref), (env, bits, L.py, np.argwhere(got != ref)[:4])
                part = np.concatenate([_np(c.comb_frames(d, p, 0, 3)), _np(c.comb_frames(d, p, 3, n - 3))])
                assert np.array_equal(part, ref), (env, bits, L.py, "ranges")
                assert np.array_equal(_np(dbuf), buf)
            assert np.array_equal(_np(c.comb_frames(pclip, p)), ref), (env, bits, "U first again")
        finally:
            c.close()
    for bits in (8, 10):                                                # host clips: whole-frame staging in small chunks
        f, ref, lays = data[bits]
        monkeypatch.setenv("AMTK_STAGE_MB", "1" if W < 1000 else "8")
        for L, buf in lays:
            host = buf.copy()
            got = _np(ctx.comb_frames(L.desc(host, False), prm if bits == 8 else p10, 1, n - 1))
            assert np.array_equal(got, ref[1:]), (bits, L.py, "host")
            assert np.array_equal(host, buf)
        monkeypatch.delenv("AMTK_STAGE_MB")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("name", sorted(GEOMS))
def test_logo_entry_points_on_v_first_frames(ctx, oracle, monkeypatch, name, bits):
    """scan, analyze, eval_fades and the fused step on device clips and on host clips staged in ROI chunks."""
    W, H = GEOMS[name][:2]
    w, h = (64, 48) if W > 300 else (48, 40)
    imgx, imgy = W - w - 3, H - h - 1
    n = 6 if W > 1000 else 14
    lg = synth.make_logo(w, h, seed=5)
    f8 = _frames(W, H, n, mode="telecine", logo=lg, imgx=imgx, imgy=imgy)
    f = f8 if bits == 8 else _to10(f8)
    maxv = float((1 << bits) - 1)
    raw = ab.Logo.create(lg["data"], w, h, W, H, imgx, imgy)
    de, top, bot = raw.deint().create_mask(0.35), raw.field(0).create_mask(0.35), raw.field(1).create_mask(0.35)
    O = Oracle(oracle, lg["data"], w, h, W, H, imgx, imgy)
    ode = O.deint(0.35)
    ot, ob = O.fields(0.35)
    Y, U, V = [p.view(f.dtype) for p in Layout(W, H, bits).planes(f)]
    fades = np.float32(0.1) * np.arange(12, dtype=np.float32)
    r_scan = np.stack([O.scan(ode, Y[i], maxv) for i in range(n)])
    r_an = np.stack([O.analyze(ode, ot, ob, Y[i], maxv) for i in range(n)])
    r_fd = np.stack([O.fades(ode, Y[i], maxv, fades) for i in range(n)])
    prm = ab.default_comb_params()
    r_comb = oracle.or_comb_clip(Y, U, V, prm.as_list())
    pclip, pbuf = _packed_clip(f, W, H, bits, True)
    u_sc, u_cc = ctx.scan_comb_frames(pclip, [de], prm)
    assert np.array_equal(_bits_of(_np(u_sc)[:, 0]), _bits_of(r_scan)) and np.array_equal(_np(u_cc), r_comb)
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    for L in _layouts(name, bits):
        buf = L.pack(f)
        dbuf = _dev(buf)
        for on_dev in (True, False):
            hbuf = dbuf if on_dev else buf.copy()
            clip = L.desc(hbuf, on_dev)
            where = ("device" if on_dev else "host", L.py)
            assert np.array_equal(_bits_of(_np(ctx.scan_frames(clip, [de]))[:, 0]), _bits_of(r_scan)), where
            assert np.array_equal(_bits_of(_np(ctx.analyze_frames(clip, de, top, bot, 1, n - 1))), _bits_of(r_an[1:])), where
            assert np.array_equal(_bits_of(_np(ctx.eval_fades(clip, de, fades, 2, n - 2))), _bits_of(r_fd[2:])), where
            sc, cc = ctx.scan_comb_frames(clip, [de], prm)
            assert np.array_equal(_bits_of(_np(sc)[:, 0]), _bits_of(r_scan)) and np.array_equal(_np(cc), r_comb), where
            if not on_dev:
                assert np.array_equal(hbuf, buf)
        assert np.array_equal(_np(dbuf), buf)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(GEOMS))
def test_logoscan_on_v_first_frames(ctx, oracle, monkeypatch, name, tmp_path):
    """LogoScan accumulation reads the U and V rectangles: each must come from its own plane.  amtk_scan_logo (the whole
    ScanLogo pipeline) must write the same logo file as on the U-first clip."""
    W, H = GEOMS[name][:2]
    sw, sh = 48, 32
    sx, sy = W - sw - 5, H - sh - 2
    n = 40
    lg = synth.make_logo(sw, sh, seed=4)
    f = _frames(W, H, n, logo=lg, imgx=sx, imgy=sy, mode="flat")
    Y, U, V = Layout(W, H, 8).planes(f)
    o = oracle.OracleScan(sw, sh, 12)
    ov = [o.add_frame(Y[i][sy:sy + sh, sx:sx + sw], U[i][sy // 2:(sy + sh) // 2, sx // 2:(sx + sw) // 2],
                      V[i][sy // 2:(sy + sh) // 2, sx // 2:(sx + sw) // 2]) for i in range(n)]
    assert 0 < sum(ov)
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    pclip, pbuf = _packed_clip(f, W, H, 8, True)
    maxf = max(2, sum(ov) - 1)

    def scan_logo(clip, path):                                         # the logo data, or the pipeline's error message
        try:
            ctx.scan_logo(clip, path, sx, sy, sw, sh, 12, maxf)
        except ab.AmtkError as e:
            return str(e)
        return ab.Logo.load(path).tables()["data"].view(np.uint32)
    want = scan_logo(pclip, str(tmp_path / "u_first.lgd"))
    for L in _layouts(name, 8):
        buf = L.pack(f)
        for on_dev in (True, False):
            hbuf = _dev(buf) if on_dev else buf.copy()
            acc = ctx.logo_scan(sw, sh, 12)
            valid = acc.add_frames(L.desc(hbuf, on_dev), sx, sy)
            assert valid.tolist() == ov and np.array_equal(acc.sums(), o.sums()), (on_dev, L.py)
            got = scan_logo(L.desc(hbuf, on_dev), str(tmp_path / ("v_first_%d_%d.lgd" % (on_dev, L.py))))
            assert type(got) is type(want) and np.array_equal(got, want), (on_dev, L.py, got if isinstance(got, str) else "")
            assert np.array_equal(_np(hbuf), buf)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("name", sorted(GEOMS))
def test_erase_on_v_first_frames(ctx, oracle, monkeypatch, name, bits):
    """U's logo planes and fades go to the U plane and V's to V, wherever the descriptor puts them: the logo's U and V
    parameters differ, so a swap changes the samples."""
    W, H = GEOMS[name][:2]
    w, h = 46, 41
    imgx, imgy = W - w - 1, H - h - 4
    n = 4 if W > 1000 else 10
    maxv = (1 << bits) - 1
    rng = np.random.default_rng(bits + W + 1)
    f = rng.integers(0, maxv + 1, (n, W * H * 3 // 2)).astype(np.uint8 if bits == 8 else np.uint16)
    d = logo_data(w, h, seed=W + 1)
    logo = ab.Logo.create(d, w, h, W, H, imgx, imgy)
    fades = np.array([[1, 1], [0, 1], [0.5, 0.5], [0.3, 0.7], [1, 0]] * 2, np.float32)[:n]
    exp = f.copy()
    for i in range(n):
        Yp, Up, Vp = [p.view(f.dtype) for p in Layout(W, H, bits).planes(exp[i:i + 1])]
        erase_reference(oracle, oracle.OracleLogo.create(d, w, h, W, H, imgx, imgy).data(), w, h, imgx, imgy,
                        Yp[0], Up[0], Vp[0], fades[i, 0], fades[i, 1], float(maxv))
    assert not np.array_equal(exp, f)
    f0 = 1
    pclip, pbuf = _packed_clip(f, W, H, bits, True)
    ctx.erase_logo(pclip, logo, fades[f0:], frame0=f0, nframes=n - f0)
    u_first = _np(pbuf).view(f.dtype)
    assert np.array_equal(u_first[f0:], exp[f0:]) and np.array_equal(u_first[:f0], f[:f0])
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    for L in _layouts(name, bits):
        want = L.pack(exp)
        want[:f0] = L.pack(f[:f0])
        dbuf = _dev(L.pack(f))
        ctx.erase_logo(L.desc(dbuf, True), logo, fades[f0:], frame0=f0, nframes=n - f0)
        assert np.array_equal(_np(dbuf), want), ("device", L.py, np.argwhere(_np(dbuf) != want)[:4])
        host = L.pack(f)
        ctx.erase_logo(L.desc(host, False), logo, fades[f0:], frame0=f0, nframes=n - f0)
        assert np.array_equal(host, want), ("host", L.py, np.argwhere(host != want)[:4])


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(GEOMS))
@pytest.mark.parametrize("case", ["vfirst_to_vfirst", "ufirst_to_vfirst", "vfirst_to_ufirst", "nv12_to_vfirst", "nv12_16_to_vfirst"])
def test_weave_with_v_first_frames(ctx, name, case):
    """AMTSource::MergeField with V-first planar sources and V-first destinations: every woven plane lands on the plane of
    the same name, and nothing outside the woven frames' samples changes."""
    W, H, py, puv, gap = GEOMS[name]
    bits = 16 if case == "nv12_16_to_vfirst" else 8
    s = 1 if bits == 8 else 2
    n = 3 if W > 1000 else 5
    rng = np.random.default_rng(W + bits + len(case))
    f = rng.integers(0, (1 << bits), (n, W * H * 3 // 2)).astype(np.uint8 if bits == 8 else np.uint16)
    nv12 = case.startswith("nv12")
    pad = lambda: (py * s if py else None, puv * s if puv else None, gap)
    if nv12:
        Ls = Layout(W, H, bits, py * s if py else None, None, gap, nv12=True)
    elif case.startswith("vfirst"):
        Ls = VFirst(W, H, bits, *pad())
    else:
        Ls = Layout(W, H, bits, *pad())
    Ld = Layout(W, H, bits, *pad()) if case.endswith("ufirst") else VFirst(W, H, bits, *pad())
    top = np.array([0, 1, 2, 2][:n - 1], np.int32) % n
    bot = np.array([1, 2, 2, 3][:n - 1], np.int32) % n
    k0 = 1
    dst = np.full((n + 2, Ld.fs), 0xFF, np.uint8)
    exp_frames = np.zeros((len(top), W * H * 3 // 2), f.dtype)
    for k in range(len(top)):
        for (o, rows, cols) in ((0, H, W), (W * H, H // 2, W // 2), (W * H + (W // 2) * (H // 2), H // 2, W // 2)):
            e = f[top[k], o:o + rows * cols].reshape(rows, cols).copy()
            e[1::2] = f[bot[k], o:o + rows * cols].reshape(rows, cols)[1::2]
            exp_frames[k, o:o + rows * cols] = e.ravel()
    want = dst.copy()
    want[k0:k0 + len(top)] = Ld.pack(exp_frames)
    sbuf, dbuf = _dev(Ls.pack(f)), _dev(dst)
    ctx.weave_frames(Ls.desc(sbuf, True), Ld.desc(dbuf, True), top, bot, dst_frame0=k0, src_is_nv12=nv12)
    got = _np(dbuf)
    assert np.array_equal(got, want), (name, case, np.argwhere(got != want)[:4])
