"""amtk_tnr_frames widening the clip as it filters it (ConvertBits(14) fused into KTemporalNR(3, 1)): an 8-, 10-, 12- or
14-bit source into a 2-byte destination at more bits must equal the filter at the destination's depth on the frames
shifted left by the difference, byte for byte against the C port (and the reference's compiled TemporalNRFilter where
oracle/_ref is built).  Also the layouts and staging of the clip path, the rejections, and the host-side mirror's
ConvertBits + KTemporalNR through tests/cpp/test_tnr_widen.cpp."""
import os
import re
import struct
import subprocess

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth, _build
from oracle import pytnr as pt
from test_gpu_tnr import POISON, _desc, _layout, _pack, _padding_untouched, _unpack

pytestmark = pytest.mark.gpu

PAIRS = ((8, 10), (8, 14), (8, 16), (10, 14), (12, 16), (14, 16))
DS = (0, 1, 3, 7, 8, 20)                 # register-window kernels (0..7) and the general kernel (8, 20)


class Mem:
    """A clip buffer in device memory, pinned host memory or pageable host memory, with its descriptor."""

    def __init__(self, raw, L, N, kind):
        self.kind = kind
        if kind == "dev":
            self.mem = torch.from_numpy(raw).cuda()
        elif kind == "pinned":
            self.mem = torch.from_numpy(raw).pin_memory()
        else:
            self.mem = raw
        ptr = self.mem.ctypes.data if kind == "host" else self.mem.data_ptr()
        self.desc = _desc(ptr, L, N, kind == "dev")

    def raw(self):
        torch.cuda.synchronize()
        if self.kind == "dev":
            return self.mem.cpu().numpy()
        return self.mem.numpy().copy() if self.kind == "pinned" else self.mem.copy()


def shifted(frames, sb, db):
    return frames.astype(np.uint16) << (db - sb)


def expect(frames, sb, db, d, t, il, W, H):
    """The definition: the filter at dst_bits on the clip widened by a left shift."""
    return pt.or_tnr_clip(shifted(frames, sb, db), W, H, db, d, t, il)


def run(ctx, frames, sb, db, d, t, il, W, H, frame0=0, nframes=None, src="dev", dst="dev", lsrc=None, ldst=None,
        dst_frames=None, dst_frame0=0):
    N = frames.shape[0]
    n = N - frame0 if nframes is None else nframes
    lsrc = lsrc or _layout(W, H, sb)
    ldst = ldst or _layout(W, H, db)
    nd = dst_frames if dst_frames is not None else n
    s = Mem(_pack(frames, lsrc), lsrc, N, src)
    o = Mem(np.full(nd * ldst["fs"], POISON, np.uint8), ldst, nd, dst)
    ctx.tnr_frames(s.desc, o.desc, ab.tnr_params(d, t, il), frame0, n, dst_frame0)
    raw = o.raw()
    return _unpack(raw, ldst, nd), raw


@pytest.mark.parametrize("sb,db", PAIRS)
@pytest.mark.parametrize("d", DS)
@pytest.mark.parametrize("il", [0, 1])
def test_pixels(ctx, sb, db, d, il):
    """Element-wise groups (76-pixel packed rows), vector groups with a ragged last group (76 pixels, rows padded to 64
    bytes) and vector groups only (128 pixels); thresholds 0, 1, a middle value and the largest."""
    H = 12
    N = 2 * d + 3                        # >= 2d: the reference's queue emits every frame
    for W, pad in ((76, False), (76, True), (128, False)):
        ls, ld = _layout(W, H, sb, pad=pad), _layout(W, H, db, pad=pad)
        fr = synth.noisy_clip(7000 + 31 * d + 3 * sb + db + il + W + pad, N, W, H, sb)
        for t in (0, 1, 127, 65535):
            got, raw = run(ctx, fr, sb, db, d, t, il, W, H, lsrc=ls, ldst=ld)
            assert np.array_equal(got, expect(fr, sb, db, d, t, il, W, H)), (W, pad, t)
            assert _padding_untouched(raw, ld, N)
            if pt.ref_available() and W == 76 and not pad:
                idx, ref = pt.ref_tnr_sequence(shifted(fr, sb, db), W, H, db, d, t, il)
                assert np.array_equal(idx, np.arange(N)) and np.array_equal(got, ref), (t,)


@pytest.mark.parametrize("sb,db", PAIRS)
@pytest.mark.parametrize("il", [0, 1])
def test_threshold_edges_and_maximum(ctx, sb, db, il):
    """Luma exactly on t << (src_bits-8) and one above it in every window frame, so the inclusion is tested at its edge;
    then all-maximum clips, so the sum is tested at maxv << k."""
    W, H, d, t = 40, 8, 3, 3
    th, maxv = t << (sb - 8), (1 << sb) - 1
    N = 2 * d + 4
    fr = synth.noisy_clip(41 + sb + db, N, W, H, sb).astype(np.int64)
    ysz = W * H
    c = fr[d].copy()
    for n in range(N):
        if n == d:
            continue
        delta = np.where(np.arange(ysz) % 4 < 2, th, th + 1) * np.where(np.arange(ysz) % 2 == 0, 1, -1)
        fr[n, :ysz] = np.clip(c[:ysz] + delta, 0, maxv)
        fr[n, ysz:] = c[ysz:]
    fr = fr.astype(np.uint8 if sb == 8 else np.uint16)
    got, _ = run(ctx, fr, sb, db, d, t, il, W, H)
    assert np.array_equal(got, expect(fr, sb, db, d, t, il, W, H))
    for dd in (3, 8):
        full = np.full_like(fr, maxv)
        got, _ = run(ctx, full, sb, db, dd, 0, il, W, H)
        assert np.array_equal(got, shifted(full, sb, db)), dd


@pytest.mark.parametrize("sb,db", [(8, 14), (10, 16)])
@pytest.mark.parametrize("src", ["dev", "pinned", "host"])
@pytest.mark.parametrize("dst", ["dev", "pinned", "host"])
def test_memory_pairings(ctx, sb, db, src, dst):
    W, H, d, N = 48, 16, 3, 11
    fr = synth.noisy_clip(500 + sb, N, W, H, sb)
    got, _ = run(ctx, fr, sb, db, d, 1, 0, W, H, src=src, dst=dst)
    assert np.array_equal(got, expect(fr, sb, db, d, 1, 0, W, H))
    if src != "dev":                      # every frame staged once, at the source's size
        assert ctx.last_h2d_bytes == N * _layout(W, H, sb)["fs"]


@pytest.mark.parametrize("sb,db", [(8, 14), (12, 16)])
@pytest.mark.parametrize("d", [3, 8])
@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("vfirst", [False, True])
def test_padded_and_v_first_layouts(ctx, sb, db, d, il, vfirst):
    """Rows padded to 64 bytes with poisoned padding, V before U, a 50-pixel (ragged) width and a frame stride that is not
    a whole number of rows, on either side or both."""
    W, H = 50, 16
    N = 2 * d + 3
    fr = synth.noisy_clip(66 + d + sb, N, W, H, sb)
    ref = expect(fr, sb, db, d, 2, il, W, H)
    ls = _layout(W, H, sb, pad=True, vfirst=vfirst, extra=24)
    ld = _layout(W, H, db, pad=True, vfirst=vfirst, extra=24)
    for src_l, dst_l in ((ls, ld), (None, ld), (ls, None)):
        for src, dst in (("dev", "dev"), ("host", "host")):
            got, raw = run(ctx, fr, sb, db, d, 2, il, W, H, lsrc=src_l, ldst=dst_l, src=src, dst=dst)
            assert np.array_equal(got, ref), (src, dst)
            assert _padding_untouched(raw, dst_l or _layout(W, H, db), N)


@pytest.mark.parametrize("sb,db", [(8, 14), (14, 16)])
@pytest.mark.parametrize("d", [1, 3, 8])
@pytest.mark.parametrize("where", ["h2d", "d2h", "h2h"])
def test_host_staging_across_chunks(ctx, monkeypatch, sb, db, d, where):
    """AMTK_STAGE_MB=1 with 256x256 frames: a few frames per chunk, each needing halo frames from its neighbours."""
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    W, H, N = 256, 256, 2 * d + 20
    fr = synth.noisy_clip(123 + d + sb, N, W, H, sb)
    full = expect(fr, sb, db, d, 1, 1, W, H)
    src, dst = {"h2d": ("host", "dev"), "d2h": ("dev", "host"), "h2h": ("host", "host")}[where]
    got, _ = run(ctx, fr, sb, db, d, 1, 1, W, H, src=src, dst=dst)
    assert np.array_equal(got, full)
    got, _ = run(ctx, fr, sb, db, d, 1, 1, W, H, frame0=d + 3, nframes=11, src=src, dst=dst)
    assert np.array_equal(got, full[d + 3:d + 14])


@pytest.mark.parametrize("sb,db", [(8, 14), (12, 16)])
@pytest.mark.parametrize("d", [1, 3, 8])
def test_range_calls_clamp_at_the_clip_ends(ctx, sb, db, d):
    W, H, N = 36, 8, 30
    fr = synth.noisy_clip(88 + sb, N, W, H, sb)
    full = expect(fr, sb, db, d, 4, 0, W, H)
    L = _layout(W, H, db)
    for frame0, n in ((5, 7), (0, 3), (N - 4, 4), (d + 1, 1), (13, 17)):
        for src in ("dev", "host"):
            got, raw = run(ctx, fr, sb, db, d, 4, 0, W, H, frame0=frame0, nframes=n, dst_frames=n + 3, dst_frame0=2, src=src)
            assert np.array_equal(got[2:2 + n], full[frame0:frame0 + n]), (frame0, n, src)
            assert (raw[:2 * L["fs"]] == POISON).all() and (raw[(2 + n) * L["fs"]:] == POISON).all()


@pytest.mark.parametrize("bits", [8, 10, 12, 14, 16])
def test_same_format_is_the_clip_call(ctx, bits):
    """src_bits == dst_bits (widening by 0) is the clip call; d = 0 widening is exactly the shift (what the mirror's
    ConvertBits materialises)."""
    W, H, N = 76, 12, 9
    fr = synth.noisy_clip(900 + bits, N, W, H, bits)
    got, _ = run(ctx, fr, bits, bits, 3, 1, 0, W, H)
    assert np.array_equal(got, pt.or_tnr_clip(fr, W, H, bits, 3, 1, 0))
    for db in (b for b in (10, 12, 14, 16) if b > bits):
        got, _ = run(ctx, fr, bits, db, 0, 0, 0, W, H)
        assert np.array_equal(got, shifted(fr, bits, db)), db


def _expect_error(ctx, src, dst, text):
    with pytest.raises(ab.AmtkError, match=text):
        ctx.tnr_frames(src, dst, ab.tnr_params(3, 1), 0, src.num_frames)


def test_rejections(ctx):
    W, H, N = 32, 16, 4
    bufs = {}
    for bits in (8, 10, 14, 16):
        L = _layout(W, H, bits)
        bufs[bits] = (Mem(np.zeros(N * L["fs"], np.uint8), L, N, "dev"), L)
    s8, s10, s14, s16 = (bufs[b][0].desc for b in (8, 10, 14, 16))
    o8 = Mem(np.zeros(N * bufs[8][1]["fs"], np.uint8), bufs[8][1], N, "dev")
    ctx.tnr_frames(s8, o8.desc)                                                 # 8 -> 8: unchanged
    ctx.tnr_frames(s8, s14)                                                     # 8 -> 14: accepted
    _expect_error(ctx, s16, s14, "fewer bits than the source; only widening")   # narrowing
    _expect_error(ctx, s14, s10, "fewer bits than the source; only widening")
    d8 = _desc(s8.base, bufs[8][1], N, True)
    _expect_error(ctx, s10, d8, "1-byte destination cannot hold a 2-byte source")
    two8 = _desc(s10.base, bufs[10][1], N, True)
    two8.bits_per_sample = 8                                                    # 2-byte samples at 8 bits
    _expect_error(ctx, s8, two8, "2-byte destination must be at 10, 12, 14 or 16 bits")
    odd = _desc(s14.base, bufs[14][1], N, True)
    odd.bits_per_sample = 11
    _expect_error(ctx, s8, odd, "bits_per_sample must be")
    small = _desc(s14.base, bufs[14][1], N, True)
    small.width = W - 2
    _expect_error(ctx, s8, small, "formats differ")
    _expect_error(ctx, s10, s10, "overlap")                                     # rejected today, still rejected
    with pytest.raises(ab.AmtkError, match="temporal_distance"):
        ctx.tnr_frames(s8, s14, ab.tnr_params(64, 1))


# ---------------------------------------------------------------------------------------------------------------
# the host-side mirror: ConvertBits(14) then KTemporalNR(3, 1)
# ---------------------------------------------------------------------------------------------------------------
W, H, IMGX, IMGY = 256, 128, 160, 32


@pytest.fixture(scope="module")
def exe():
    return _build.build_tnr_widen_test() if os.path.exists("/usr/bin/g++") else _build.TNR_WIDEN_TEST


def _write_raw1(path, frames):
    with open(path, "wb") as f:
        f.write(b"AMTSRAW1" + struct.pack("<6i", W, H, 8, frames.shape[0], 30000, 1001))
        f.write(frames.tobytes())


def _drive(exe, *args):
    r = subprocess.run([exe, *map(str, args)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


@pytest.mark.parametrize("source", ["dev", "cpu"])
def test_convertbits_then_ktemporalnr_output_pass(exe, tmp_path, source):
    n = 17
    frames = synth.noisy_clip(4343, n, W, H, 8)
    _write_raw1(tmp_path / "amts0.dat", frames)
    out = _drive(exe, "pass", tmp_path, source, tmp_path / "out.bin")
    assert "pass: frames=%d bits=14" % n in out
    if source == "dev":        # one fused call from the 8-bit clip, no widened intermediate, device views
        assert "resident=1 device_frames=%d" % n in out
        assert "launches=1 materialized=0" in out
    else:                      # ConvertBits widens each CPU frame, KTemporalNR gathers 14-bit windows
        assert "resident=0 device_frames=0" in out and "materialized=0" in out
    assert "typed=%d" % n in out
    got = np.fromfile(tmp_path / "out.bin", np.uint16).reshape(n, -1)
    assert np.array_equal(got, pt.or_tnr_clip(frames.astype(np.uint16) << 6, W, H, 14, 3, 1, 0))


@pytest.mark.parametrize("source", ["dev", "cpu"])
def test_convertbits_alone(exe, tmp_path, source):
    n = 9
    frames = synth.noisy_clip(4444, n, W, H, 8)
    _write_raw1(tmp_path / "amts0.dat", frames)
    out = _drive(exe, "convert", tmp_path, source, tmp_path / "out.bin")
    assert "convert: frames=%d bits=14" % n in out
    if source == "dev":        # materialised by one d = 0 call when first asked for
        assert "resident=1 device_frames=%d" % n in out and "launches=1 materialized=1" in out
    else:
        assert "resident=0 device_frames=0" in out and "launches=0 materialized=0" in out
    narrowing = "ConvertBits: only widening is provided; narrowing is AviSynth\\+'s dither arithmetic, which is not in the reference"
    for what in ("narrow10", "narrow8", "dither"):
        assert any(l.startswith(what + ": ") and re.search(narrowing, l) for l in out.splitlines()), what
    assert "same_bits_is_child=1 builtin=1 plugin_registers=0" in out
    got = np.fromfile(tmp_path / "out.bin", np.uint16).reshape(n, -1)
    assert np.array_equal(got, frames.astype(np.uint16) << 6)


def test_erase_in_place_on_the_fused_filters_device_clip(exe, tmp_path):
    n = 24
    lg = synth.make_logo(64, 64, seed=1)
    frames = synth.make_frames(35, n, W, H, logo=lg, imgx=IMGX, imgy=IMGY, logo_period=16).numpy()
    _write_raw1(tmp_path / "amts0.dat", frames)
    logo_path = str(tmp_path / "logo.lgd")
    ab.Logo.create(lg["data"], 64, 64, W, H, IMGX, IMGY).save(logo_path)
    out = _drive(exe, "erase", tmp_path, logo_path, tmp_path / "per_frame.bin", tmp_path / "in_place.bin")
    assert "erase: frames=%d bits=14 identical=1 materialized=0" % n in out
    per_frame = np.fromfile(tmp_path / "per_frame.bin", np.uint16).reshape(n, -1)
    tnr = pt.or_tnr_clip(frames.astype(np.uint16) << 6, W, H, 14, 3, 1, 0)
    assert not np.array_equal(per_frame, tnr)                 # the logo was erased from the filtered frames ...
    ysz = W * H
    Y = per_frame[:, :ysz].reshape(n, H, W)
    T = tnr[:, :ysz].reshape(n, H, W)
    outside = np.ones((H, W), bool)
    outside[IMGY:IMGY + 64, IMGX:IMGX + 64] = False
    assert np.array_equal(Y[:, outside], T[:, outside])       # ... and nothing outside its rectangle changed
