"""How the fused step plans its logo items, restated, and the logo items run on every band variant at every frames-per-item
regime its ring allows.

amtk_scan_comb_frames with one logo on an 8-bit clip hands the band-form comb kernel logo items of F frames (scan_item in
csrc/logo_kernels.cuh, queued by launch_comb_ws in csrc/amtk_b200.cu).  F is not observable from outside the library, so
the restatement below is the only record of which variant and which F a case runs; the CPU tests pin it to the numbers
DESIGN.md 3.1a / 3.2 state, and every GPU case asserts the (variant, F) it stands for, so a change of the rings or the plan
fails an assertion instead of silently moving a case to another regime.  The GPU cases compare the scores bit for bit with
the reference's ScanFrame and the counters with the combing spec (the helpers of test_gpu_fused_step.py), on frame ranges
that end at every position of an item, logos at the ring budget of several F and at the eligibility edge, ROI offsets,
widths and heights at the edges of scan_item's loops, feature counts at the edges of its ordered sums, and staged host
clips."""
import functools
import os
import re
from collections import namedtuple

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from test_gpu_comb_plans import _ctx, pick_ws_R
from test_gpu_comb_tall import pick_tall_R, tables
from test_gpu_fused_step import _logo, _refs, _run
from test_gpu_frame_layouts import Layout
from test_gpu_logo_plans import _bits_of, make_clip_frames, to_device

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "amatsukaze_b200", "csrc")


def _constant(fname, name):
    m = re.search(r"constexpr int %s = (\d+);" % name, open(os.path.join(CSRC, fname)).read())
    assert m, (fname, name)
    return int(m.group(1))


# ---- restatement of the plan ---------------------------------------------------------------------------------------------
MAX_FRAMES = _constant("logo_kernels.cuh", "kScanItemMaxFrames")
RUNS = _constant("comb_stream.cuh", "kWsRuns")            # runs of R rows per warp
TALL_GROUPS = _constant("comb_stream.cuh", "kWtGroups")   # row groups of a tall band
HALF = _constant("comb_stream.cuh", "kWbHalf")            # a slot is two TMA boxes of this width

Plan = namedtuple("Plan", "form R stages threads F")
KNOBS = {"AMTK_COMB_WS_BAND": "2", "AMTK_COMB_R": "0", "AMTK_COMB_WS_STAGES": "2"}


def ring_bytes(form, R, stages):
    """BandCfg::SMEM less its 128 bytes of alignment slack: STAGES slots of two boxes of HALF x (GROUPS x 4R + 4) rows."""
    groups = TALL_GROUPS if form == "tall" else 1
    return stages * 2 * HALF * (groups * RUNS * R + 4)


def ws_variant(H, env=None, tall=True):
    """ws_variant of an 8-bit 4:2:0 clip of height H: ("tall" | "band", R, stages), None when none is compiled.  The tall
    form runs when AMTK_COMB_WS_BAND=2 (the default) and a tall variant has the R and stages; else the 512 x 4R form.
    tall=False: the 512 x 4R variant, whichever form runs."""
    k = dict(KNOBS, **(env or {}))
    band, R, S = int(k["AMTK_COMB_WS_BAND"]), int(k["AMTK_COMB_R"]), int(k["AMTK_COMB_WS_STAGES"])
    if not band:
        return None
    talls, bands = tables()
    if tall and band == 2:
        Rt = R or pick_tall_R(H, H // 2)
        if (Rt, S) in talls:
            return ("tall", Rt, S)
    R4 = R or pick_ws_R(H, H // 2)
    return ("band", R4, S) if (R4, S) in bands else None


def count_pad(count):
    return max(32, (count + 31) & ~31)


def item_bytes(w, h, count, F):
    """scan_item_smem_bytes: two fade images, F x 2 score rows, the raw ROI rows."""
    return (2 * ((w * h + 8 + 3) & ~3) + F * 2 * (count_pad(count) + 4)) * 4 + ((w + 30) & ~15) * h


def plan(W, H, w, h, count, env=None):
    """What amtk_scan_comb_frames runs for one w x h logo with `count` feature pixels on a W x H 8-bit clip of a
    TMA-describable layout: Plan(form, R, stages, threads per CTA, F), or "serial".  scan_item_frames: the logo runs fused
    when its item holds one frame in the 512 x 4R ring; F is then as many frames as the ring that runs holds, at most
    kScanItemMaxFrames."""
    V, V4 = ws_variant(H, env), ws_variant(H, env, tall=False)
    if V is None or V4 is None or count < 1 or w > W or h > H or item_bytes(w, h, count, 1) > ring_bytes(*V4):
        return "serial"
    F = 0
    while F < MAX_FRAMES and item_bytes(w, h, count, F + 1) <= ring_bytes(*V):
        F += 1
    return Plan(V[0], V[1], V[2], 32 * RUNS * (TALL_GROUPS if V[0] == "tall" else 1), F)


def slack(H, w, h, count, env=None):
    """Bytes of the running ring left free by the item at its F."""
    p = plan(10 ** 4, H, w, h, count, env)
    return ring_bytes(p.form, p.R, p.stages) - item_bytes(w, h, count, p.F)


# ---- logos that sit where a case claims ----------------------------------------------------------------------------------
W = 320                                                    # frame width of the matrix and most geometry cases
WIDTHS = (16, 24, 32, 40, 48, 64, 80, 96, 112)                    # logo widths searched for budget edges (seed = logo height)


@functools.lru_cache(maxsize=None)
def feature_count(w, h, seed):
    return _logo(w, h, w, h, 0, 0, seed)[1].info().count


def budget_edge(H, env, F):
    """(under, over, free): of the w x h logos (seed h, w in WIDTHS) that get F frames per item while the next taller one
    gets fewer, the one that leaves the fewest bytes of the running ring free, and that next one.  F = 0: the eligibility
    edge -- the largest logo whose one-frame item fits in the 512 x 4R ring, and the next, which takes the serial path
    (free = bytes of the 512 x 4R ring left)."""
    V4 = ring_bytes(*ws_variant(H, env, tall=False))
    best = None
    for w in WIDTHS:
        prev = None
        for h in range(8, min(H, 192) - 2):
            c = feature_count(w, h, h)
            p = plan(W, H, w, h, c, env)
            f = 0 if p == "serial" else p.F
            if prev is not None:
                (ph, pc, pf) = prev
                hit = pf >= 1 and f == 0 if F == 0 else pf == F and f < F
                if hit:
                    free = V4 - item_bytes(w, ph, pc, 1) if F == 0 else slack(H, w, ph, pc, env)
                    if best is None or free < best[2]:
                        best = ((w, ph, pc), (w, h, c), free)
                    break
            prev = (h, c, f)
    return best


def count_case(pred):
    """The first small logo (w x h, seed h) whose feature count satisfies pred."""
    for h in range(7, 31):
        for w in range(9, 48):
            c = feature_count(w, h, h)
            if c > 0 and pred(c):
                return w, h, c
    return None


# The band variants that run logo items: name -> (frame height, knobs, ws_variant).  Heights pick R by default where one
# does (578..600 is the first run of heights whose tall R is 17 and 4R R is 15); no height picks the 4R R = 16 variant while
# the tall form is on, and no height picks 3 stages.  136: the tall form at R = 15, eligibility from the R = 17 4R ring.
VARIANTS = {
    "WtCfg<15,2>": (120, {}, ("tall", 15, 2)),
    "WtCfg<16,2>": (192, {}, ("tall", 16, 2)),
    "WbCfg<15,2>": (600, {}, ("band", 15, 2)),
    "WbCfg<16,2>": (192, {"AMTK_COMB_WS_BAND": "1"}, ("band", 16, 2)),
    "WbCfg<17,2>": (204, {}, ("band", 17, 2)),
    "WbCfg<15,3>": (120, {"AMTK_COMB_WS_STAGES": "3"}, ("band", 15, 3)),
    "WtCfg<15,2>@136": (136, {}, ("tall", 15, 2)),
}
# Budget edges per form: the 512 x 4R rings give F = 1 at the eligibility edge, F = 2 and F = 8 at theirs; an eligible
# logo's one-frame item takes at most a 4R ring and its score rows at most half of that, so the tall rings give every
# eligible logo at least F = 4 (the eligibility edge is their smallest F) -- F = 13 is the headline logo's.  F = 16 is
# the cap (kScanItemMaxFrames): the largest logo that gets it, and a small logo far below the ring's end.
EDGES = {"tall": (0, 13, 16), "band": (0, 2, 8, 16)}
# Bytes a budget-edge case may leave free: a few hundred; at F = 16 the item grows in steps of 16 x 2 x 32 score floats
# (countPad is a multiple of 32), and on the R = 17 and 3-stage 4R rings no searched logo gets closer than 1-3 kB.
FREE_MAX = {16: 16 * 2 * 32 * 4}


def regime_logos(variant, regime):
    """[(spec, plan)] of a matrix case; spec = (w, h, imgx, imgy, seed).  Asserts that each logo gets the (variant, F) the
    case stands for."""
    H, env, V = VARIANTS[variant]
    assert ws_variant(H, env) == V, (variant, ws_variant(H, env))
    place = lambda w, h, c: ((w, h, (W - w) // 2 - 3, (H - h) // 2, h), plan(W, H, w, h, c, env))
    if regime == "small":
        spec, p = place(16, 16, feature_count(16, 16, 16))
        assert p.F == MAX_FRAMES and slack(H, 16, 16, feature_count(16, 16, 16), env) > 16 * 1024, (variant, p)
        return [(spec, p)]
    F = int(regime[1:]) if regime != "edge" else 0
    found = budget_edge(H, env, F)
    assert found is not None, (variant, regime)
    (uw, uh, uc), (ow, oh, oc), free = found
    assert 0 <= free <= FREE_MAX.get(F, 512), (variant, regime, found)
    under, over = place(uw, uh, uc), place(ow, oh, oc)
    assert under[1] != "serial" and under[1][:3] == V, (variant, regime, under)
    if F == 0:
        assert over[1] == "serial", (variant, over)
        assert V[0] == "tall" or under[1].F == 1                 # on a 4R ring the eligibility edge is the F = 1 edge
    else:
        assert under[1].F == F and (over[1] == "serial" or over[1].F < F), (variant, regime, under, over)
    return [under, over]


MATRIX = [(v, r) for v in VARIANTS for r in ["edge"] + ["F%d" % f for f in EDGES[VARIANTS[v][2][0]][1:]] + ["small"]]


# ---- CPU: the restatement against the numbers DESIGN.md states ----------------------------------------------------------
def test_compiled_tables_and_cap():
    tall, band = tables()
    assert sorted(tall) == [(15, 2), (16, 2)]
    assert sorted(band) == [(15, 2), (15, 3), (16, 2), (17, 2)]
    assert MAX_FRAMES == 16
    assert (RUNS, TALL_GROUPS, HALF) == (4, 3, 256)


def test_ring_sizes():
    assert [ring_bytes("tall", R, 2) for R in (15, 16)] == [188416, 200704]
    assert [ring_bytes("band", R, 2) for R in (15, 16, 17)] == [65536, 69632, 73728]
    assert ring_bytes("band", 15, 3) == 98304


def test_headline_plan(native_lib):
    """64x64 at maskratio 0.35 (1433 features) on 1080p: WtCfg<15,2> at F = 13 with 288 bytes free, F = 2 in WbCfg<15,2>;
    720x576 runs WtCfg<16,2> at F = 14."""
    _, P = _logo(64, 64, 1920, 1080, 1700, 60, seed=1)
    c = P.info().count
    assert c == 1433 and count_pad(c) == 1440
    assert plan(1920, 1080, 64, 64, c) == Plan("tall", 15, 2, 384, 13)
    assert slack(1080, 64, 64, c) == 288 and item_bytes(64, 64, c, 13) == 188416 - 288
    assert plan(1920, 1080, 64, 64, c, {"AMTK_COMB_WS_BAND": "1"}) == Plan("band", 15, 2, 128, 2)
    assert plan(720, 576, 64, 64, c) == Plan("tall", 16, 2, 384, 14)
    assert plan(1920, 1080, 64, 64, c, {"AMTK_COMB_WS_BAND": "0"}) == "serial"


def test_variant_choice():
    assert ws_variant(1080) == ("tall", 15, 2) and ws_variant(120) == ("tall", 15, 2)
    assert ws_variant(192) == ws_variant(576) == ("tall", 16, 2)               # 12R-row bands: R = 16
    assert ws_variant(204) == ws_variant(204, tall=False) == ("band", 17, 2)   # tall R = 17 is not compiled
    assert ws_variant(136) == ("tall", 15, 2) and ws_variant(136, tall=False) == ("band", 17, 2)
    assert ws_variant(600) == ("band", 15, 2)
    assert ws_variant(120, {"AMTK_COMB_WS_STAGES": "3"}) == ("band", 15, 3)    # no tall variant has 3 stages
    assert ws_variant(120, {"AMTK_COMB_R": "17"}) == ("band", 17, 2)
    assert ws_variant(120, {"AMTK_COMB_WS_BAND": "1"}) == ("band", 15, 2)
    assert ws_variant(120, {"AMTK_COMB_R": "11"}) is None


def test_cap_and_eligibility_follow_the_rings():
    """A small logo gets the cap on every ring; a logo whose one-frame item needs more than 65 536 but at most 73 728 bytes
    runs fused at height 136 (eligibility from the R = 17 4R ring), in the tall form, and not at height 120."""
    for H, env, _ in VARIANTS.values():
        assert plan(W, H, 16, 16, 60, env).F == 16
    w, h, c = 96, 64, 2000
    assert item_bytes(w, h, c, 1) == 72544
    assert plan(W, 120, w, h, c) == "serial"
    assert plan(W, 136, w, h, c) == Plan("tall", 15, 2, 384, 8)


@pytest.mark.parametrize("variant,regime", MATRIX, ids=["%s-%s" % m for m in MATRIX])
def test_matrix_logos_sit_where_they_claim(native_lib, variant, regime):
    regime_logos(variant, regime)


def test_geometry_cases_sit_where_they_claim(native_lib):
    for form in GEOM_FORMS:
        for kind in GEOM_KINDS:
            geometry_logos(form, kind)


# ---- item geometry cases -------------------------------------------------------------------------------------------------
# The tall form (384 threads per CTA) and the 512 x 4R form (128 threads), both at R = 15 on 120-row frames.
GEOM_FORMS = {"tall": ({}, ("tall", 15, 2)), "band": ({"AMTK_COMB_WS_BAND": "1"}, ("band", 15, 2))}
GEOM_KINDS = ("offsets", "right_edge", "wide", "short", "counts")
GH = 120


def geometry_logos(form, kind):
    """[(frame width, spec, plan)] of a geometry case, each asserted to run fused on the form's variant.
    offsets: imgx % 16 in {0, 1, 15}, with (imgx % 16) + w one under, on and one over 48 (the ROI rows are loaded from imgx
             rounded down to 16 bytes, in 16-byte pieces);
    right_edge: logos ending at the right edge of 328-wide frames (8 mod 16; the 16-byte pieces of the last one reach into
             the pitch's padding);
    wide: logos 127, 128, 129, 383, 384 and 400 wide, as tall as stays eligible (the pixel walk steps NT % w columns and
             NT / w rows: one row and one column, exactly one row, no row);
    short: the shortest logos with feature pixels (features sit 2 rows inside the logo, so 5 rows), where DeintY's edge rows
             are 2 of 5;
    counts: feature counts with count % 4 = 0, 1, 2, 3 (the ordered sums add 4 scores at a time while c + 4 <= count), a
             multiple of 32 (countPad == count: the read-ahead ends on the row's last line) and one under 32."""
    env, V = GEOM_FORMS[form]
    specs = []                                             # (frame width, w, h, imgx, seed)
    if kind == "offsets":
        specs = [(W, s - xo, 30, 64 + xo, s) for xo in (0, 1, 15) for s in (47, 48, 49)]
    elif kind == "right_edge":
        specs = [(328, w, 40, 328 - w, w) for w in (40, 37, 47)]
    elif kind == "wide":
        for w in (127, 128, 129, 383, 384, 400):
            h = max(h for h in range(5, 60) if plan(416, GH, w, h, feature_count(w, h, h), env) != "serial")
            specs.append((416, w, h, (416 - w) // 2, h))
    elif kind == "short":
        specs = [(W, 41, 5, 17, 5), (W, 40, 5, 200, 6), (W, 41, 6, 90, 7), (W, 33, 7, 250, 8)]
    elif kind == "counts":
        preds = [lambda c, r=r: c > 32 and c % 32 and c % 4 == r for r in range(4)]
        preds += [lambda c: c >= 64 and c % 32 == 0, lambda c: c < 32]
        for k, pred in enumerate(preds):
            w, h, c = count_case(pred)
            assert pred(c), (k, w, h, c)
            specs.append((W, w, h, 30 + 40 * k, h))
    out = []
    for Wf, w, h, imgx, seed in specs:
        c = feature_count(w, h, seed)
        assert c > 0, (kind, w, h)
        p = plan(Wf, GH, w, h, c, env)
        assert p != "serial" and p[:3] == V, (form, kind, w, h, p)
        out.append((Wf, (w, h, imgx, (GH - h) // 3, seed), p))
    if kind == "counts":
        counts = [feature_count(w, h, sd) for _, (w, h, _, _, sd), _ in out]
        assert {c % 4 for c in counts} == {0, 1, 2, 3} and any(c % 32 == 0 for c in counts) and min(counts) < 32
    return out


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def item_ranges(F):
    """Frame ranges ending at every position of an item: n in {1, F - 1, F, F + 1, 2F + 1} from frame 0, and 2F + 1 frames
    from frame 3 (a clip of 2F + 4 frames)."""
    return sorted({(0, n) for n in (1, F - 1, F, F + 1, 2 * F + 1) if n > 0} | {(3, 2 * F + 1)})


def _run_ranges(c, oracle, packed, Wf, H, spec, p, clip):
    """One logo over item_ranges of its F: scores bit-equal to the reference's ScanFrame, counters to the spec, one launch
    per call when it runs fused and more when it takes the serial path."""
    w, h, imgx, imgy, seed = spec
    data, P = _logo(w, h, Wf, H, imgx, imgy, seed)
    assert P.info().count == feature_count(w, h, seed)
    rs, rc = _refs(oracle, packed, Wf, H, data, w, h, imgx, imgy, 0, packed.shape[0])
    fused = p != "serial"
    for frame0, n in item_ranges(p.F if fused else 1):
        s, cnt = _run(c, clip, P, frame0, n, fused)
        assert np.array_equal(_bits_of(s), _bits_of(rs[frame0:frame0 + n])), (Wf, H, spec, p, frame0, n)
        assert np.array_equal(cnt, rc[frame0:frame0 + n]), (Wf, H, spec, p, frame0, n)


def _max_F(logos):
    return max([p.F for *_, p in logos if p != "serial"] + [1])


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("variant,regime", MATRIX, ids=["%s-%s" % m for m in MATRIX])
def test_items_on_every_variant(oracle, monkeypatch, variant, regime):
    """Every band variant that runs logo items, at the eligibility edge (the last logo runs fused in one launch, the next
    takes the serial path), at the ring's end for several F (the largest logo that gets F and the next size up) and at the
    cap."""
    H, env, _ = VARIANTS[variant]
    logos = regime_logos(variant, regime)
    packed = make_clip_frames(2 * _max_F(logos) + 4, W, H, 8, seed=H + len(regime))
    buf = to_device(packed)
    clip = ab.yv12_clip(buf, W, H, packed.shape[0], True)
    c = _ctx(monkeypatch, env)
    try:
        for spec, p in logos:
            _run_ranges(c, oracle, packed, W, H, spec, p, clip)
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("form", sorted(GEOM_FORMS))
@pytest.mark.parametrize("kind", GEOM_KINDS)
def test_item_geometry(oracle, monkeypatch, form, kind):
    logos = geometry_logos(form, kind)
    c = _ctx(monkeypatch, GEOM_FORMS[form][0])
    try:
        for Wf in sorted({Wf for Wf, _, _ in logos}):
            packed = make_clip_frames(2 * _max_F(logos) + 4, Wf, GH, 8, seed=Wf + len(kind))
            if kind == "right_edge":                       # pitch 384, padding 0xFF: a score that read it would change
                L = Layout(Wf, GH, 8)
                assert Wf % 16 == 8 and L.py % 16 == 0 and L.puv % 16 == 0
                buf = torch.from_numpy(L.pack(packed)).cuda()
                clip = L.desc(buf, True)
            else:
                buf = to_device(packed)
                clip = ab.yv12_clip(buf, Wf, GH, packed.shape[0], True)
            for W2, spec, p in logos:
                if W2 == Wf:
                    _run_ranges(c, oracle, packed, Wf, GH, spec, p, clip)
    finally:
        c.close()


def stage_windows(fs, frame0, n, mb=1):
    """for_each_window's chunks of a host clip with need_prev: frames per window."""
    per = max(1, min(n, (mb << 20) // fs))
    per = per - 1 if per > 1 else per
    return [min(per, frame0 + n - lo) for lo in range(frame0, frame0 + n, per)]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("form", sorted(GEOM_FORMS))
def test_staged_windows_not_a_multiple_of_F(oracle, monkeypatch, form):
    """Host clips through 1 MiB staging buffers: windows of 17 frames and ragged last windows, none a multiple of F; one
    fused launch per window."""
    env, V = GEOM_FORMS[form]
    c = _ctx(monkeypatch, env)
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    try:
        n = 41
        packed = make_clip_frames(n, W, GH, 8, seed=41)
        hclip = ab.yv12_clip(packed, W, GH, n, False)
        for spec in ((64, 64, 100, 30, 14), (48, 40, 203, 61, 15)):
            w, h, imgx, imgy, seed = spec
            data, P = _logo(w, h, W, GH, imgx, imgy, seed)
            p = plan(W, GH, w, h, P.info().count, env)
            assert p != "serial" and p[:3] == V and p.F > 1, (form, spec, p)
            rs, rc = _refs(oracle, packed, W, GH, data, w, h, imgx, imgy, 0, n)
            for frame0, m in ((0, n), (5, 30), (40, 1), (2, p.F + 1)):
                wins = stage_windows(hclip.frame_stride, frame0, m)
                assert any(k % p.F for k in wins), (wins, p.F)
                l0 = c.launches
                s, cnt = _run(c, hclip, P, frame0, m, None)
                assert c.launches - l0 == len(wins), (spec, frame0, m, wins)
                assert np.array_equal(_bits_of(s), _bits_of(rs[frame0:frame0 + m])), (spec, p, frame0, m)
                assert np.array_equal(cnt, rc[frame0:frame0 + m]), (spec, p, frame0, m)
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_720x576_runs_tall_r16(oracle, monkeypatch):
    """A realistic size on WtCfg<16,2>: 720x576 (576 = 3 x 192), a 64x64 logo at F = 14, device and host clips, against the
    reference and against a per-warp-form context, which takes the serial path on the same frames.  The rows are padded to
    64 bytes as decoders deliver them: packed 720-wide frames have a 360-byte chroma pitch, which no tensor map describes,
    so they take the serial path."""
    Wf, H, n = 720, 576, 42
    L = Layout(Wf, H, 8)
    assert (L.py, L.puv) == (768, 384)
    spec = (64, 64, 600, 40, 1)
    data, P = _logo(*spec[:2], Wf, H, *spec[2:])
    assert plan(Wf, H, 64, 64, P.info().count) == Plan("tall", 16, 2, 384, 14)
    assert plan(Wf, H, 64, 64, P.info().count, {"AMTK_COMB_WS_BAND": "0"}) == "serial"
    packed = make_clip_frames(n, Wf, H, 8, seed=576)
    rs, rc = _refs(oracle, packed, Wf, H, data, *spec[:4], 0, n)
    host = L.pack(packed)
    buf = torch.from_numpy(host).cuda()
    clips = {"device": L.desc(buf, True), "host": L.desc(host, False)}
    c = _ctx(monkeypatch, {})
    warp = _ctx(monkeypatch, {"AMTK_COMB_WS_BAND": "0"})
    try:
        for where, clip in clips.items():
            for frame0, m in ((0, n), (0, 14), (1, 15), (5, 29), (41, 1)):
                # host clips: one fused launch per staging window (a clip that fits is staged as m - 1 frames and 1)
                l0 = c.launches
                s, cnt = _run(c, clip, P, frame0, m, True if where == "device" else None)
                if where == "host":
                    assert c.launches - l0 == len(stage_windows(L.fs, frame0, m, 256)), (frame0, m)
                assert np.array_equal(_bits_of(s), _bits_of(rs[frame0:frame0 + m])), (where, frame0, m)
                assert np.array_equal(cnt, rc[frame0:frame0 + m]), (where, frame0, m)
                s2, cnt2 = _run(warp, clip, P, frame0, m, False)
                assert np.array_equal(_bits_of(s2), _bits_of(s)) and np.array_equal(cnt2, cnt), (where, frame0, m)
    finally:
        c.close()
        warp.close()
