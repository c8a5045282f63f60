"""The fused step and the combing counters where a slightly wrong kernel would still pass the broader suites: every call
writes into outputs filled beforehand with values no kernel computes (0x7FC00001, a NaN, for scores; 0x7F7F7F7F for
counters), so a score row or a counter row left unwritten fails even when the caching allocator hands back a block that
already holds the right numbers.

Scores are compared bit for bit with the reference's ScanFrame (the C port where oracle/_ref is absent); counters with the
combing spec's vectorised form over the whole clip and its scalar form on a few frames.  The cases put the previous frame
at an item's start on window frame 1, make the work list's three tiers meet inside the call, end the logo items with a
short one, put the spec-excluded rows at several positions of the last band, and set the 10-bit thresholds on and around
the largest response a 10-bit stencil can give.  The mutants of tools/mutants.py that a test is there to kill are named in
its docstring."""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from test_gpu_comb_plans import _ctx, _tiers
from test_gpu_comb_tall import ntiles, pick_tall_R, tall_runs
from test_gpu_frame_layouts import Layout
from test_gpu_fused_item_plans import plan
from test_gpu_fused_step import MASKRATIO, _logo
from test_gpu_logo_plans import Oracle, _bits_of, make_clip_frames, to_device, y_planes

pytestmark = pytest.mark.gpu

SCORE_POISON = 0x7FC00001
COUNT_POISON = 0x7F7F7F7F


def poisoned(n, nlogos=0):
    """(scores, counts) device outputs filled with the poison patterns."""
    s = torch.full((n, max(nlogos, 1), 2), SCORE_POISON, dtype=torch.int32, device="cuda").view(torch.float32)
    c = torch.full((n, 12), COUNT_POISON, dtype=torch.int32, device="cuda")
    return s, c


def planes(packed, W, H):
    ysz, csz = W * H, (W // 2) * (H // 2)
    return (y_planes(packed, W, H), packed[:, ysz:ysz + csz].reshape(-1, H // 2, W // 2),
            packed[:, ysz + csz:].reshape(-1, H // 2, W // 2))


def spec_counts(oracle, packed, W, H, prm, frame0, n, scalar=(0, -1)):
    """Counters of frames [frame0, frame0 + n) by the spec (previous of frame 0 = itself): the vectorised form (8-bit) or the
    scalar loop for every frame, and the scalar loop again on the frames at the offsets `scalar` (negative: from the end)."""
    Y, U, V = planes(packed, W, H)
    th = prm.as_list()
    impl = "avx2" if packed.dtype == np.uint8 else "scalar"
    out = np.stack([oracle.or_comb_frame((Y[i], U[i], V[i]), (Y[max(i - 1, 0)], U[max(i - 1, 0)], V[max(i - 1, 0)]), th, impl)
                    for i in range(frame0, frame0 + n)])
    for k in scalar:
        i = frame0 + (k % n)
        j = max(i - 1, 0)
        assert np.array_equal(out[i - frame0], oracle.or_comb_frame((Y[i], U[i], V[i]), (Y[j], U[j], V[j]), th, "scalar")), i
    return out


def ref_scores(oracle, packed, W, H, data, spec, frame0, n):
    w, h, imgx, imgy, _ = spec
    O = Oracle(oracle, data, w, h, W, H, imgx, imgy)
    de = O.deint(MASKRATIO)
    Y = y_planes(packed, W, H)
    return np.stack([O.scan(de, Y[i], 255.0) for i in range(frame0, frame0 + n)])


def fused(c, oracle, packed, W, H, spec, frame0, n, fused_expected=True):
    """One poisoned amtk_scan_comb_frames call on a device clip, checked against both oracles."""
    data, P = _logo(*spec[:2], W, H, *spec[2:])
    buf = to_device(packed)
    clip = ab.yv12_clip(buf, W, H, packed.shape[0], True)
    s, cnt = poisoned(n, 1)
    l0 = c.launches
    c.scan_comb_frames(clip, [P], ab.default_comb_params(), frame0=frame0, nframes=n, scores=s, counts=cnt)
    torch.cuda.synchronize()
    assert (c.launches - l0 == 1) == fused_expected, c.launches - l0
    got_s, got_c = s.cpu().numpy()[:, 0], cnt.cpu().numpy()
    want_c = spec_counts(oracle, packed, W, H, ab.default_comb_params(), frame0, n)
    bad = np.argwhere(got_c != want_c)
    assert bad.size == 0, ("counters", W, H, frame0, n, bad[:6].tolist())
    want_s = ref_scores(oracle, packed, W, H, data, spec, frame0, n)
    bad = np.argwhere(_bits_of(got_s) != _bits_of(want_s))
    assert bad.size == 0, ("scores", W, H, spec, frame0, n, bad[:6].tolist())


# (W, H, frames in the clip, logo (w, h, imgx, imgy, seed), frame0, nframes).  Heights: 120 and 136 leave rows H-2..H+1
# inside the last band's runs at different offsets, 178 gives odd-height chroma planes, 100 puts the plane's end inside
# the first band's middle row group; R = 15 runs start on odd rows.  frame0 = 1: the first items start at window frame 1.
CASES = {
    "320x120_from1": (320, 120, 41, (48, 40, 101, 30, 4), 1, 39),
    "320x120_from0_short_last_item": (320, 120, 37, (48, 40, 101, 30, 4), 0, 37),
    "640x136_from1": (640, 136, 30, (40, 32, 280, 88, 7), 1, 27),
    "576x178_oddchroma": (576, 178, 26, (33, 27, 0, 150, 8), 2, 23),
    "1952x100_from1": (1952, 100, 21, (64, 64, 1952 - 64, 30, 3), 1, 20),
}


def test_cases_reach_their_plans():
    """Every case runs fused in the tall form with R = 15 (runs on odd rows) and ends its logo items with a short one."""
    for name, (W, H, nclip, (w, h, x, y, seed), frame0, n) in CASES.items():
        assert tall_runs(H) == (True, 15), name
        assert frame0 + n <= nclip


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(CASES))
def test_fused_poisoned(ctx, oracle, name):
    """Kills band_top_mask, band_lo_j, band_hi_j, band_flip_off, band_flip_move_only, band_prev_window_frame1,
    band_prev_first_next, ws_move_encoding, ws_shima_gt, item_fade_order, item_last_row_unwritten, item_row_behind,
    item_black_mul, item_sum_tail, logo_item_end, logo_item_last_frame."""
    W, H, nclip, spec, frame0, n = CASES[name]
    packed = make_clip_frames(nclip, W, H, 8, seed=len(name))
    w, h = spec[:2]
    _, P = _logo(w, h, W, H, *spec[2:])
    p = plan(W, H, w, h, P.info().count)
    assert p != "serial" and n % p.F != 0, (name, p)          # the last logo item is short
    fused(ctx, oracle, packed, W, H, spec, frame0, n)


def _long_clip(W, H, n, seed):
    """n frames cycling through 13 random ones (so every frame differs from the one before it)."""
    base = make_clip_frames(13, W, H, 8, seed=seed)
    return base[np.arange(n) % 13]


def _three_tier_frames(W, H):
    """Frames per call at which the band queue of a W x H clip has a head, a middle and an end tier (one tall CTA per SM)."""
    R = pick_tall_R(H, H // 2)
    tiles = ntiles(W, H, 12 * R)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 64
    while _tiers(tiles, n, sms, 0, 4) < 3:
        n += 64
    return n + 37                                                    # a ragged last item in every tier


@pytest.mark.timeout(1200)
def test_three_tiers_meet(ctx, oracle):
    """The first frames of the middle and end tiers, and the last of the head tier, are counted once each, in a fused call
    and a comb-only call that both start at window frame 1.  Kills tier_mid_skip, tier_mid_twice, tier_end_skip,
    logo_item_end, logo_item_last_frame, band_prev_window_frame1."""
    W, H = 4096, 34
    n = _three_tier_frames(W, H)
    packed = _long_clip(W, H, n + 1, seed=21)
    prm = ab.default_comb_params()
    buf = to_device(packed)
    clip = ab.yv12_clip(buf, W, H, n + 1, True)
    _, cnt = poisoned(n)
    ctx.comb_frames(clip, prm, 1, n, out=cnt)
    want = spec_counts(oracle, packed, W, H, prm, 1, n, scalar=(0, n // 2, -1))
    got = cnt.cpu().numpy()
    assert np.array_equal(got, want), np.argwhere(got != want)[:6].tolist()
    fused(ctx, oracle, packed, W, H, (40, 16, 2000, 9, 5), 1, n)


# ---- 2-byte samples ------------------------------------------------------------------------------------------------------
def _saturated_10bit(W, H, n, seed):
    """10-bit frames with rows alternating 1023 / 0 in part of every plane (|response| = 6 x 1023 = 6138, the largest a
    10-bit stencil gives) and random samples elsewhere; the stripes move from frame to frame."""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 1024, (n, W * H * 3 // 2)).astype(np.uint16)
    for k, (off, w, h) in enumerate(((0, W, H), (W * H, W // 2, H // 2), (W * H + (W // 2) * (H // 2), W // 2, H // 2))):
        p = f[:, off:off + w * h].reshape(n, h, w)
        for i in range(n):
            stripe = (np.arange(h) % 2 == (i + k) % 2) * 1023
            p[i, :, : w // 2] = stripe[:, None]
        f[:, off:off + w * h] = p.reshape(n, w * h)
    return f


FORMS10 = {"cta": {}, "ws10": {"AMTK_COMB_WS10": "1"}, "generic": {"AMTK_COMB_GENERIC": "1"}}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("form", sorted(FORMS10))
@pytest.mark.parametrize("th", [(1, 6138, 6138), (2, 6137, 6139), (1023, 6139, 8191), (512, 8191, 9000)])
def test_10bit_thresholds_at_the_largest_response(oracle, monkeypatch, form, th):
    """Small and large thresholds on, just below and above the largest 10-bit response, in every form a 10-bit clip can
    run, from window frame 1, into poisoned counters.  Kills ws10_lshima_clamp, u16_exact_float, u16_shima_gt,
    generic_rows, generic_prev_self."""
    W, H, n = 160, 70, 6
    f = _saturated_10bit(W, H, n, seed=sum(th))
    prm = ab.default_comb_params()
    prm.th_move_y, prm.th_shima_y, prm.th_lshima_y = th
    prm.th_move_c, prm.th_shima_c, prm.th_lshima_c = th[0], th[2], th[1]
    c = _ctx(monkeypatch, FORMS10[form])
    buf = torch.from_numpy(f.view(np.int16)).cuda()
    clip = ab.yv12_clip(buf, W, H, n, True, 10)
    _, cnt = poisoned(n - 1)
    c.comb_frames(clip, prm, 1, n - 1, out=cnt)
    want = spec_counts(oracle, f, W, H, prm, 1, n - 1)
    got = cnt.cpu().numpy()
    c.close()
    assert np.array_equal(got, want), (form, th, np.argwhere(got != want)[:6].tolist())
    assert want[:, [2, 5, 8, 11]].any() or th[1] > 6138       # the large-threshold counters hit where they can


@pytest.mark.timeout(900)
def test_generic_layout_range_calls(ctx, oracle):
    """An 8-bit clip whose pitch TMA cannot describe runs the generic kernel: range calls from frames 1 and 3 into
    poisoned counters.  Kills generic_rows, generic_prev_self."""
    W, H, n = 200, 58, 9
    packed = make_clip_frames(n, W, H, 8, seed=5)
    L = Layout(W, H, 8, pitch_y=W + 3, pitch_uv=W // 2 + 5)
    buf = torch.from_numpy(L.pack(packed)).cuda()
    clip = L.desc(buf, True)
    prm = ab.default_comb_params()
    for frame0 in (1, 3):
        _, cnt = poisoned(n - frame0)
        ctx.comb_frames(clip, prm, frame0, n - frame0, out=cnt)
        want = spec_counts(oracle, packed, W, H, prm, frame0, n - frame0)
        got = cnt.cpu().numpy()
        assert np.array_equal(got, want), (frame0, np.argwhere(got != want)[:6].tolist())
