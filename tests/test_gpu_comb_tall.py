"""The tall band form of the 8-bit warp-stream kernel (comb_stream.cuh, WtCfg): one 12-warp CTA per SM streams a band of
512 bytes x 12R rows, warp w running the row code on column w % 4 of row group w / 4.  It is the default for 8-bit clips
(AMTK_COMB_WS_BAND=2); when no tall variant has the rows per run and stages asked for, the clip runs the 512 x 4R band form
instead.  Counters must equal the spec oracle's bit for bit on ragged widths, heights whose last band has idle row groups,
edge rows inside a middle row group, extreme thresholds, range calls, other layouts, staged host clips, the fused step
and the comb stream.

The CPU tests restate the tall form's rows per run, tile counts and the rows it reads per frame."""
import re

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from test_gpu_comb_plans import SHAPES, SRC, _check, _ctx, _frames, _oracle_counts, _params, pick_ws_R
from test_gpu_frame_layouts import Layout

TALL = {"AMTK_COMB_WS_BAND": "2"}
BAND = {"AMTK_COMB_WS_BAND": "1"}


def tables():
    """(tall, band) variants compiled into ws_variants(): lists of (R, stages)."""
    body = re.search(r"static const WsVariant\* ws_variants\(int\* n\) \{(.*?)\n\}", open(SRC).read(), re.S).group(1)
    get = lambda kind: [tuple(int(x) for x in a.split(",")) for a in re.findall(r"make_ws<%s<([^>]*)>>\(\)" % kind, body)]
    return get("WtCfg"), get("WbCfg")


def pick_tall_R(hY, hC):
    """pick_ws_R's rule with 12R-row bands: fewest wasted rows over luma + chroma, ties to the larger R."""
    best, bw = 17, None
    for R in (17, 16, 15):
        th = 12 * R
        w = 2 * (-(-hY // th) * th - hY) + 2 * (-(-hC // th) * th - hC)
        if bw is None or w < bw:
            best, bw = R, w
    return best


def tall_runs(H):
    """Whether a default-knob context runs an 8-bit clip of height H in the tall form, and with which R."""
    R = pick_tall_R(H, H // 2)
    return (R, 2) in tables()[0], R


def rows_read(H, TH):
    """Rows a band's box reads from a plane of H rows, summed over its bands: TH rows + 2 halo rows above and below,
    clipped to the plane (TMA fills the rest with zeros without reading)."""
    return sum(min(y0 + TH + 2, H) - max(y0 - 2, 0) for y0 in range(0, H, TH))


def ntiles(W, H, TH):
    return sum(-(-w // 512) * -(-h // TH) for w, h in ((W, H), (W // 2, H // 2), (W // 2, H // 2)))


# ---- CPU -------------------------------------------------------------------------------------------------------------
def test_tall_variants_fall_back_to_bands():
    tall, band = tables()
    assert sorted(tall) == [(15, 2), (16, 2)]
    assert all(v in band for v in tall)                        # every tall variant has a band variant to fall back on
    assert (17, 2) not in tall and (15, 3) not in tall         # AMTK_COMB_R=17 and AMTK_COMB_WS_STAGES=3 run bands


def test_tall_geometry():
    assert tall_runs(1080) == (True, 15) and tall_runs(720) == (True, 15) and pick_ws_R(1080, 540) == 15
    assert tall_runs(204) == (False, 17)                       # 204 = 12 x 17: no tall R = 17, the band form runs
    assert ntiles(1920, 1080, 180) == 4 * 6 + 2 * 2 * 3 == 36 and ntiles(1440, 1080, 180) == 3 * 6 + 2 * 2 * 3 == 30
    assert ntiles(1920, 1080, 60) == 4 * 18 + 2 * 2 * 9
    # rows read per frame: luma 1100 (tall) against 1148 (bands), chroma 548 against 572
    assert (rows_read(1080, 180), rows_read(540, 180)) == (1100, 548)
    assert (rows_read(1080, 60), rows_read(540, 60)) == (1148, 572)
    per_frame = lambda W, TH: W * rows_read(1080, TH) + 2 * (W // 2) * rows_read(540, TH)
    assert per_frame(1920, 180) == 3164160 and per_frame(1920, 60) == 3302400
    assert per_frame(1440, 180) < per_frame(1440, 60)
    # every test height below leaves the last band with idle row groups or edge rows inside a row group
    for H in (34, 120, 136, 272, 1100, 100):
        R = pick_tall_R(H, H // 2)
        assert tall_runs(H)[0] and H % (12 * R), H


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _counts(c, fr, W, H, prm):
    return c.comb_frames(ab.yv12_clip(fr, W, H, fr.shape[0], True), prm).cpu().numpy()


# (W, H, n): ragged widths (one partial box, 3 bands + 416 bytes, 3.75 bands, a 64-byte chroma plane in a 512-byte band);
# heights whose last band has idle row groups (34, 272, 1100), a row group that starts at H (120: chroma 60) and rows
# H-2 .. H+1 inside a middle row group (100, 136 chroma 68)
TALL_SHAPES = ((160, 34, 3), (1952, 136, 2), (1920, 120, 3), (128, 1100, 2), (320, 272, 5), (320, 100, 9), (640, 360, 9))


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_tall_form_is_bit_exact(oracle, monkeypatch):
    c = _ctx(monkeypatch, TALL)
    try:
        for (W, H, n) in TALL_SHAPES:
            f = _frames(W, H, n, 8, seed=W + H)
            for prm in (_params(8), ab.default_comb_params()):      # extreme thresholds, then the defaults
                _check(c, oracle, f, W, H, 8, prm, what="tall")
            _check(c, oracle, f, W, H, 8, _params(8), vfirst=True, what="tall vfirst")
            L = Layout(W, H, 8, W + 64, W // 2 + 32, 48)             # padded pitches, gaps between the planes
            ref = _oracle_counts(oracle, f, W, H, _params(8))
            buf = torch.from_numpy(L.pack(f)).cuda()
            got = c.comb_frames(L.desc(buf, True), _params(8)).cpu().numpy()
            assert np.array_equal(got, ref), ("padded", W, H)
        # maximum response everywhere: alternating 0 / 255 rows, every row group of the band busy (360) or not (128)
        for h in (128, 360):
            w = 512
            fr = torch.zeros((2, w * h * 3 // 2), dtype=torch.uint8, device="cuda")
            fr[:, : w * h].view(2, h, w)[:, 0::2, :] = 255
            p2 = ab.default_comb_params()
            p2.th_shima_y, p2.th_lshima_y = 1530, 1531
            out = _counts(c, fr, w, h, p2)
            assert out[0, 1] + out[0, 4] == (h - 4) * w and out[0, 2] + out[0, 5] == 0 and out[:, 0].sum() == 0, h
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_tall_form_on_staged_host_chunks(oracle, monkeypatch):
    c = _ctx(monkeypatch, TALL)
    try:
        w, h, n = 640, 360, 17
        fr = synth.make_frames(0, n, w, h, device="cuda", mode="telecine")
        prm = ab.default_comb_params()
        Y, U, V = synth.split_planes(fr, w, h)
        ref = oracle.or_comb_clip(Y, U, V, prm.as_list())
        monkeypatch.setenv("AMTK_STAGE_MB", "1")                 # 1 MiB staging -> a few frames per chunk, one launch each
        hbuf = fr.cpu().numpy()
        got = c.comb_frames(ab.yv12_clip(hbuf, w, h, n, False), prm)
        got = got.cpu().numpy() if hasattr(got, "cpu") else np.asarray(got)
        assert np.array_equal(got, ref)
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("W", [1920, 1440])
def test_tall_equals_bands_at_1080(oracle, monkeypatch, W):
    H, n = 1080, 6
    fr = synth.make_frames(W, n, W, H, device="cuda", mode="telecine")
    prm = ab.default_comb_params()
    got = {}
    for name, env in (("tall", TALL), ("band", BAND)):
        c = _ctx(monkeypatch, env)
        try:
            got[name] = _counts(c, fr, W, H, prm)
        finally:
            c.close()
    Y, U, V = synth.split_planes(fr, W, H)
    assert np.array_equal(got["tall"], got["band"])
    assert np.array_equal(got["tall"], oracle.or_comb_clip(Y, U, V, prm.as_list()))


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("form", ["tall", "band"])
def test_every_band_variant(oracle, monkeypatch, form):
    """Every compiled variant of both band forms, reached through AMTK_COMB_R and AMTK_COMB_WS_STAGES (with the tall form
    the default, the 512 x 4R variants that have a tall twin need AMTK_COMB_WS_BAND=1)."""
    tall, band = tables()
    for R, S in (tall if form == "tall" else band):
        c = _ctx(monkeypatch, dict(TALL if form == "tall" else BAND, AMTK_COMB_R=str(R), AMTK_COMB_WS_STAGES=str(S)))
        try:
            for (W, H, n) in SHAPES[8]:
                _check(c, oracle, _frames(W, H, n, 8), W, H, 8, _params(8), what=(form, R, S))
        finally:
            c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_one_context_alternates_forms(oracle, monkeypatch):
    """One default-knob context (plus AMTK_COMB_WS10=1, so that 10-bit clips run the per-warp form) alternating the tall
    form (height 120), the 512 x 4R band form (height 204: the tall rule picks R = 17, which has no tall variant) and the
    per-warp form, with comb-only and fused calls: the cached plan and the kernel's shared-memory setting follow the form."""
    from test_gpu_fused_step import _check as fused_check
    from test_gpu_logo_plans import make_clip_frames
    assert tall_runs(120)[0] and not tall_runs(204)[0]
    c = _ctx(monkeypatch, {"AMTK_COMB_WS10": "1"})
    try:
        f8 = {H: _frames(320, H, 9, 8, seed=H) for H in (120, 204)}
        f10 = _frames(224, 136, 7, 10)
        logo = {H: make_clip_frames(12, 320, H, 8, seed=H) for H in (120, 204)}
        for _ in range(2):
            for H in (120, 204):
                _check(c, oracle, f8[H], 320, H, 8, _params(8), what=("alternate", H))
                _check(c, oracle, f10, 224, 136, 10, _params(10), what="alternate ws10")
                fused_check(c, oracle, logo[H], 320, H, (40, 32, 101, 30, H), fused=True)
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_fused_step_at_1080_runs_tall(oracle, monkeypatch):
    """The headline geometry: one launch per call, 13 frames per logo item (the tall R = 15 ring's budget), scores
    bit-exact."""
    from test_gpu_fused_item_plans import Plan, plan
    from test_gpu_fused_step import _check as fused_check, _logo
    from test_gpu_logo_plans import make_clip_frames
    _, P = _logo(64, 64, 1920, 1080, 1700, 60, seed=1)
    assert plan(1920, 1080, 64, 64, P.info().count) == Plan("tall", 15, 2, 384, 13)
    c = _ctx(monkeypatch, TALL)
    try:
        packed = make_clip_frames(12, 1920, 1080, 8, seed=1080)
        fused_check(c, oracle, packed, 1920, 1080, (64, 64, 1700, 60, 1), fused=True)
        fused_check(c, oracle, packed, 1920, 1080, (64, 64, 1700, 60, 1), frame0=5, n=6, fused=True)
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_comb_stream_runs_tall(oracle, monkeypatch):
    from test_gpu_comb_stream import make_frames, resident, run
    c = _ctx(monkeypatch, TALL)
    try:
        B, w, h = 16, 640, 360
        fr = make_frames(3 * B + 5, w, h, 8, seed=16)
        rows, _, _ = run(c, fr, w, h, 8, B, ab.default_comb_params())
        exp = resident(c, fr, w, h, 8, ab.default_comb_params())
        assert np.array_equal(rows, exp)
        assert np.array_equal(exp, _oracle_counts(oracle, fr, w, h, ab.default_comb_params()))
    finally:
        c.close()
