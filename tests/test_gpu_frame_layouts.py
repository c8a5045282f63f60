"""Every entry point on AviSynth-shaped frames: padded rows and planes, poisoned padding.

The product's own filter surface hands the kernels frames whose rows are padded: VideoFrame rounds every row up to 64
bytes (host/avs_compat.h), HostFrameClip rounds the frame stride up to 16 (host/filters.hpp) -- 1440x1080 gets a luma pitch
of 1472 and a chroma pitch of 768.  Here every byte that is not a sample is 0xFF (0xFFFF at 16 bits, above maxv), and the
frame stride carries a 16-byte tail so that it is not a whole number of rows, which sends host-clip ROI staging down its
per-frame 2-D copy path.  A kernel, tensor map or ROI copy that used the pitch where it should use the width would count
or overwrite padding; each result must equal the one on the packed clip, the reference's, and leave the padding alone."""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from test_gpu_erase import erase_reference, logo_data
from test_gpu_logo_plans import Oracle

pytestmark = pytest.mark.gpu


def _rup(v, a):
    return (v + a - 1) // a * a


class Layout:
    """Planar 4:2:0 frame layout (or Y + interleaved UV when nv12) with padded pitches, optional gaps between planes and a
    16-byte frame tail."""

    def __init__(self, W, H, bits, pitch_y=None, pitch_uv=None, gap=0, nv12=False):
        self.W, self.H, self.bits, self.nv12 = W, H, bits, nv12
        self.bps = 1 if bits == 8 else 2
        self.row_y = W * self.bps
        self.row_c = (W // 2) * self.bps * (2 if nv12 else 1)
        self.py = pitch_y or _rup(self.row_y, 64)
        self.puv = pitch_uv or _rup(self.row_c, 64)
        self.off_u = self.py * H + gap
        self.off_v = self.off_u if nv12 else self.off_u + self.puv * (H // 2) + gap
        self.fs = _rup(self.off_v + self.puv * (H // 2), 16) + 16
        while self.fs % self.py == 0 or self.fs % self.puv == 0:      # never a whole number of rows
            self.fs += 16

    def planes(self, packed):
        """Byte views (n, rows, row bytes) of Y, U, V of packed frames (n, W*H*3/2) of uint8/uint16."""
        b = np.ascontiguousarray(packed).view(np.uint8)
        n, W, H, s = b.shape[0], self.W, self.H, self.bps
        ysz, csz = W * H * s, (W // 2) * (H // 2) * s
        return (b[:, :ysz].reshape(n, H, W * s), b[:, ysz:ysz + csz].reshape(n, H // 2, (W // 2) * s),
                b[:, ysz + csz:].reshape(n, H // 2, (W // 2) * s))

    def pack(self, packed, stripes=False):
        """Frames in this layout; padding 0xFF, or with stripes rows of padding alternating 0x00 / 0xFF and flipping from
        frame to frame (a combing kernel that read them would count them as combed and moving)."""
        n = packed.shape[0]
        Y, U, V = self.planes(packed)
        buf = np.full((n, self.fs), 0xFF, np.uint8)
        H2 = self.H // 2
        if stripes:
            for off, pitch, rows in ((0, self.py, self.H), (self.off_u, self.puv, H2), (self.off_v, self.puv, H2)):
                par = (np.arange(rows)[None, :, None] + np.arange(n)[:, None, None]) & 1
                buf[:, off:off + pitch * rows].reshape(n, rows, pitch)[:] = (par * 0xFF).astype(np.uint8)
        buf[:, :self.py * self.H].reshape(n, self.H, self.py)[:, :, :self.row_y] = Y
        if self.nv12:
            s = self.bps
            uv = np.stack([U.reshape(n, H2, -1, s), V.reshape(n, H2, -1, s)], axis=3).reshape(n, H2, self.row_c)
            buf[:, self.off_u:self.off_u + self.puv * H2].reshape(n, H2, self.puv)[:, :, :self.row_c] = uv
        else:
            for off, P in ((self.off_u, U), (self.off_v, V)):
                buf[:, off:off + self.puv * H2].reshape(n, H2, self.puv)[:, :, :self.row_c] = P
        return buf

    def desc(self, buf, on_device):
        d = ab.ClipDesc()
        d.base = buf.data_ptr() if isinstance(buf, torch.Tensor) else buf.ctypes.data
        d.frame_stride, d.off_u, d.off_v = self.fs, self.off_u, self.off_v
        d.width, d.height, d.pitch_y, d.pitch_uv = self.W, self.H, self.py, self.puv
        d.log_uvx = d.log_uvy = 1
        d.bytes_per_sample, d.bits_per_sample = self.bps, self.bits
        d.num_frames, d.on_device = buf.shape[0], 1 if on_device else 0
        return d


# (W, H, pitch_y, pitch_uv, gap): None = row bytes rounded up to 64 (VideoFrame)
GEOMS = {
    "1440x1080": (1440, 1080, None, None, 0),          # 1472 / 768
    "720x480": (720, 480, None, None, 32),             # 768 / 384, 32-byte gaps between the planes
    "720x480_luma720": (720, 480, 720, 384, 0),        # 720 / 384
    "200x100": (200, 100, None, None, 0),              # 256 / 128
    "200x100_plus64": (200, 100, 320, 192, 16),        # another 64 bytes per row
    "200x100_row8": (200, 100, 208, 108, 0),           # rows 8 bytes longer: no TMA, the generic comb kernel
}


def _frames8(name, n, logo=None, imgx=0, imgy=0, mode="telecine"):
    W, H = GEOMS[name][:2]
    return synth.make_frames(2, n, W, H, device="cpu", mode=mode, logo=logo, imgx=imgx, imgy=imgy, logo_period=10).numpy()


def _to10(f8):
    f = f8.astype(np.uint16)
    return (f * 4 + (f & 3)).astype(np.uint16)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _packed_clip(a, W, H, bits, on_device):
    a = np.ascontiguousarray(a)
    buf = _dev(a.view(np.int16) if a.dtype == np.uint16 else a) if on_device else a
    return ab.yv12_clip(buf, W, H, a.shape[0], on_device, bits), buf


def _knob_ctx(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    c = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    for k in env:
        monkeypatch.delenv(k)
    return c


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _bits_of(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


COMB_SETTINGS = [({}, 8), ({"AMTK_COMB_WS_BAND": "0"}, 8), ({"AMTK_COMB_WS": "0"}, 8), ({"AMTK_COMB_MMA": "1"}, 8),
                 ({"AMTK_COMB_GENERIC": "1"}, 8), ({}, 10), ({"AMTK_COMB_WS10": "1"}, 10), ({"AMTK_COMB_GENERIC": "1"}, 10)]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(GEOMS))
def test_comb_on_padded_frames(ctx, oracle, monkeypatch, name):
    W, H, py, puv, gap = GEOMS[name]
    n = 4 if W > 1000 else 9
    f8 = _frames8(name, n)
    prm = ab.default_comb_params()
    p10 = ab.default_comb_params()
    p10.th_move_y, p10.th_shima_y, p10.th_lshima_y, p10.th_move_c, p10.th_shima_c, p10.th_lshima_c = 80, 48, 144, 96, 64, 192
    data = {}
    for bits in (8, 10):
        f = f8 if bits == 8 else _to10(f8)
        Y, U, V = [p.view(f.dtype) for p in Layout(W, H, bits).planes(f)]
        ref = oracle.or_comb_clip(Y, U, V, (prm if bits == 8 else p10).as_list())
        assert ref[:, [1, 4]].sum() > 0
        L = Layout(W, H, bits, py * (1 if bits == 8 else 2) if py else None, puv * (1 if bits == 8 else 2) if puv else None, gap)
        data[bits] = (f, L, L.pack(f), ref)
    for (env, bits), stripes in [(e, False) for e in COMB_SETTINGS] + [(e, True) for e in COMB_SETTINGS[:3] + COMB_SETTINGS[5:6]]:
        f, L, padded, ref = data[bits]
        padded = L.pack(f, stripes=True) if stripes else padded
        p = prm if bits == 8 else p10
        c = _knob_ctx(monkeypatch, env)
        try:
            dbuf = _dev(padded)
            got = _np(c.comb_frames(L.desc(dbuf, True), p))
            assert np.array_equal(got, ref), (env, bits, stripes, np.argwhere(got != ref)[:4])
            pclip, pbuf = _packed_clip(f, W, H, bits, True)
            assert np.array_equal(_np(c.comb_frames(pclip, p)), ref), (env, bits, "packed")
            # range calls with a halo frame
            part = np.concatenate([_np(c.comb_frames(L.desc(dbuf, True), p, 0, 2)), _np(c.comb_frames(L.desc(dbuf, True), p, 2, 1)),
                                   _np(c.comb_frames(L.desc(dbuf, True), p, 3, n - 3))])
            assert np.array_equal(part, ref), (env, bits, "ranges")
            assert np.array_equal(_np(dbuf), padded)                    # read-only: nothing written anywhere
        finally:
            c.close()
    for bits in (8, 10):                                                # host copy: whole-frame staging of padded frames
        f, L, padded, ref = data[bits]
        monkeypatch.setenv("AMTK_STAGE_MB", "1" if W < 1000 else "8")
        host = padded.copy()
        got = _np(ctx.comb_frames(L.desc(host, False), prm if bits == 8 else p10, 1, n - 1))
        monkeypatch.delenv("AMTK_STAGE_MB")
        assert np.array_equal(got, ref[1:]), (bits, "host")


def _logo_geom(name):
    W, H = GEOMS[name][:2]
    w, h = (64, 48) if W > 300 else (48, 40)
    return w, h, W - w - 3, H - h - 1                                  # near the right and bottom edges, odd imgx


@pytest.mark.timeout(900)
@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("name", sorted(GEOMS))
def test_logo_entry_points_on_padded_frames(ctx, oracle, monkeypatch, name, bits):
    W, H, py, puv, gap = GEOMS[name]
    w, h, imgx, imgy = _logo_geom(name)
    n = 6 if W > 1000 else 20
    lg = synth.make_logo(w, h, seed=5)
    f8 = _frames8(name, n, logo=lg, imgx=imgx, imgy=imgy)
    f = f8 if bits == 8 else _to10(f8)
    maxv = float((1 << bits) - 1)
    s = 1 if bits == 8 else 2
    L = Layout(W, H, bits, py * s if py else None, puv * s if puv else None, gap)
    padded = L.pack(f)
    raw = ab.Logo.create(lg["data"], w, h, W, H, imgx, imgy)
    de, top, bot = raw.deint().create_mask(0.35), raw.field(0).create_mask(0.35), raw.field(1).create_mask(0.35)
    O = Oracle(oracle, lg["data"], w, h, W, H, imgx, imgy)
    ode = O.deint(0.35)
    ot, ob = O.fields(0.35)
    Y = L.planes(f)[0].view(f.dtype)
    fades = np.float32(0.1) * np.arange(20, dtype=np.float32)
    r_scan = np.stack([O.scan(ode, Y[i], maxv) for i in range(n)])
    r_an = np.stack([O.analyze(ode, ot, ob, Y[i], maxv) for i in range(n)])
    r_fd = np.stack([O.fades(ode, Y[i], maxv, fades) for i in range(n)])
    prm = ab.default_comb_params()
    U, V = [p.view(f.dtype) for p in L.planes(f)[1:]]
    r_comb = oracle.or_comb_clip(Y, U, V, prm.as_list())
    dbuf = _dev(padded)
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    for on_dev in (True, False):
        hbuf = dbuf if on_dev else padded.copy()                       # the descriptor holds only its address
        clip = L.desc(hbuf, on_dev)
        where = "device" if on_dev else "host"
        assert np.array_equal(_bits_of(_np(ctx.scan_frames(clip, [de]))[:, 0]), _bits_of(r_scan)), where
        assert np.array_equal(_bits_of(_np(ctx.analyze_frames(clip, de, top, bot, 1, n - 1))), _bits_of(r_an[1:])), where
        assert np.array_equal(_bits_of(_np(ctx.eval_fades(clip, de, fades, 2, n - 2))), _bits_of(r_fd[2:])), where
        sc, cc = ctx.scan_comb_frames(clip, [de], prm)
        assert np.array_equal(_bits_of(_np(sc)[:, 0]), _bits_of(r_scan)) and np.array_equal(_np(cc), r_comb), where
    pclip, pbuf = _packed_clip(f, W, H, bits, True)
    assert np.array_equal(_bits_of(_np(ctx.scan_frames(pclip, [de]))[:, 0]), _bits_of(r_scan))
    lite = _knob_ctx(monkeypatch, {"AMTK_SCAN_LITE": "1"})
    try:
        sc, cc = lite.scan_comb_frames(L.desc(dbuf, True), [de], prm)
        assert np.array_equal(_bits_of(_np(sc)[:, 0]), _bits_of(r_scan)) and np.array_equal(_np(cc), r_comb), "lite"
    finally:
        lite.close()
    assert np.array_equal(_np(dbuf), padded)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(GEOMS))
def test_logoscan_accumulate_on_padded_frames(ctx, oracle, monkeypatch, name):
    W, H, py, puv, gap = GEOMS[name]
    sw, sh = 48, 32
    sx, sy = W - sw - 5, H - sh - 2
    n = 8 if W > 1000 else 30
    lg = synth.make_logo(sw, sh, seed=4)
    f = _frames8(name, n, logo=lg, imgx=sx, imgy=sy, mode="flat")
    L = Layout(W, H, 8, py, puv, gap)
    padded = L.pack(f)
    Y, U, V = L.planes(f)
    o = oracle.OracleScan(sw, sh, 12)
    ov = [o.add_frame(Y[i][sy:sy + sh, sx:sx + sw], U[i][sy // 2:(sy + sh) // 2, sx // 2:(sx + sw) // 2],
                      V[i][sy // 2:(sy + sh) // 2, sx // 2:(sx + sw) // 2]) for i in range(n)]
    assert 0 < sum(ov)
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    for on_dev in (True, False):
        acc = ctx.logo_scan(sw, sh, 12)
        hbuf = _dev(padded) if on_dev else padded.copy()               # the descriptor holds only its address
        valid = acc.add_frames(L.desc(hbuf, on_dev), sx, sy)
        assert valid.tolist() == ov and np.array_equal(acc.sums(), o.sums()), on_dev


@pytest.mark.timeout(900)
@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("name", sorted(GEOMS))
def test_erase_on_padded_frames(ctx, oracle, monkeypatch, name, bits):
    """Device clips are edited in place; host clips move the three logo rectangles up and back with one 2-D copy per frame
    (the frame stride is not a whole number of rows).  Padding and every sample outside the logo stay unchanged."""
    W, H, py, puv, gap = GEOMS[name]
    w, h = 46, 41
    imgx, imgy = W - w - 1, H - h - 4                                  # chroma parity depends on H; odd imgx
    n = 4 if W > 1000 else 12
    maxv = (1 << bits) - 1
    rng = np.random.default_rng(bits + W)
    f = rng.integers(0, maxv + 1, (n, W * H * 3 // 2)).astype(np.uint8 if bits == 8 else np.uint16)
    s = 1 if bits == 8 else 2
    L = Layout(W, H, bits, py * s if py else None, puv * s if puv else None, gap)
    d = logo_data(w, h, seed=W)
    logo = ab.Logo.create(d, w, h, W, H, imgx, imgy)
    fades = np.array([[1, 1], [0, 1], [0.5, 0.5], [0.3, 0.7], [1, 0], [0, 0]] * 3, np.float32)[:n]
    exp = f.copy()
    for i in range(n):
        Yp, Up, Vp = [p.view(f.dtype) for p in Layout(W, H, bits).planes(exp[i:i + 1])]
        erase_reference(oracle, oracle.OracleLogo.create(d, w, h, W, H, imgx, imgy).data(), w, h, imgx, imgy,
                        Yp[0], Up[0], Vp[0], fades[i, 0], fades[i, 1], float(maxv))
    want = L.pack(exp)
    f0 = 1
    want[0] = L.pack(f[:1])[0]                                         # frame 0 lies outside the erased range
    dbuf = _dev(L.pack(f))
    ctx.erase_logo(L.desc(dbuf, True), logo, fades[f0:], frame0=f0, nframes=n - f0)
    assert np.array_equal(_np(dbuf), want), ("device", np.argwhere(_np(dbuf) != want)[:4])
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    host = L.pack(f)
    ctx.erase_logo(L.desc(host, False), logo, fades[f0:], frame0=f0, nframes=n - f0)
    assert np.array_equal(host, want), ("host", np.argwhere(host != want)[:4])
    pclip, pbuf = _packed_clip(f, W, H, bits, True)
    ctx.erase_logo(pclip, logo, fades[f0:], frame0=f0, nframes=n - f0)
    assert np.array_equal(L.pack(_np(pbuf).view(f.dtype)), want)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", ["1440x1080", "720x480", "200x100_plus64", "200x100_row8"])
@pytest.mark.parametrize("src", ["planar8", "nv12_8", "nv12_16"])
def test_weave_on_padded_frames(ctx, name, src):
    """AMTSource::MergeField into a poisoned padded destination from a padded planar or NV12 (P010-style at 16 bits)
    source, at dst_frame0 > 0: only the samples of the woven frames change."""
    W, H, py, puv, gap = GEOMS[name]
    bits = 16 if src == "nv12_16" else 8
    n = 3 if W > 1000 else 6
    rng = np.random.default_rng(W + bits)
    f = rng.integers(0, (1 << bits), (n, W * H * 3 // 2)).astype(np.uint8 if bits == 8 else np.uint16)
    s = 1 if bits == 8 else 2
    nv12 = src.startswith("nv12")
    Ls = Layout(W, H, bits, (py * s if py else None), None if nv12 else (puv * s if puv else None), gap, nv12=nv12)
    Ld = Layout(W, H, bits, (py * s if py else None), puv * s if puv else None, gap)
    top = np.array([0, 1, 2, 2, 4, 5][:n - 1], np.int32) % n
    bot = np.array([1, 2, 2, 3, 5, 5][:n - 1], np.int32) % n
    k0 = 1
    m = n + 2
    dst = np.full((m, Ld.fs), 0xFF, np.uint8)
    exp_frames = np.zeros((len(top), W * H * 3 // 2), f.dtype)
    for k in range(len(top)):
        for (o, rows, cols) in ((0, H, W), (W * H, H // 2, W // 2), (W * H + (W // 2) * (H // 2), H // 2, W // 2)):
            t = f[top[k], o:o + rows * cols].reshape(rows, cols)
            b = f[bot[k], o:o + rows * cols].reshape(rows, cols)
            e = t.copy()
            e[1::2] = b[1::2]
            exp_frames[k, o:o + rows * cols] = e.ravel()
    want = dst.copy()
    want[k0:k0 + len(top)] = Ld.pack(exp_frames)
    sbuf, dbuf = _dev(Ls.pack(f)), _dev(dst)
    ctx.weave_frames(Ls.desc(sbuf, True), Ld.desc(dbuf, True), top, bot, dst_frame0=k0, src_is_nv12=nv12)
    got = _np(dbuf)
    assert np.array_equal(got, want), (name, src, np.argwhere(got != want)[:4])
