"""Launch plans of the combing pass: which kernel form runs, every compiled variant, every knob, and the cached plan.

The combing pass has six forms: the band and per-warp forms of the warp-stream kernel (8-bit), its 10-bit form
(AMTK_COMB_WS10=1), the CTA-ring kernel (10/12/16-bit by default, AMTK_COMB_WS=0), the tensor-core kernel (AMTK_COMB_MMA)
and the generic plain-load kernel (layouts a tensor map cannot describe, AMTK_COMB_GENERIC=1).  The warp-stream and
tensor-core forms keep their work items on the device between calls (amtk_ctx::CombPlan), so a call must never run on the
items of another call whose tile classes differ.  Every result is compared with the spec oracle (oracle/amtk_oracle.c)
exactly.

The CPU tests parse the compiled variant tables out of csrc/amtk_b200.cu and restate how the host picks rows per run, the
U|V pair and merge classes, the tile counts and the work-queue tiers, so that a new variant or a moved threshold cannot
leave a path untested."""
import os
import re

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from test_gpu_frame_layouts import Layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "amatsukaze_b200", "csrc", "amtk_b200.cu")
SM_H100 = 132                      # H100 SXM
WS_OCC = 3                         # resident CTAs per SM of the warp-stream forms (DESIGN.md 3.1a)

# Every compiled variant.  Warp-stream: (form, R, stages, warps, bytes per sample); CTA ring: (R, strip, stages, sync,
# has a 16-bit kernel).
WS_SWEEP = [("warp", 17, 2, 4, 1), ("warp", 15, 2, 4, 1), ("warp", 16, 2, 4, 1), ("warp", 9, 2, 4, 1), ("warp", 15, 3, 4, 1),
            ("warp", 12, 2, 4, 1), ("warp", 10, 2, 4, 1), ("warp", 15, 2, 7, 1), ("warp", 13, 2, 5, 1), ("warp", 15, 2, 2, 1),
            ("warp", 15, 3, 3, 1), ("warp", 15, 2, 4, 2), ("warp", 16, 2, 4, 2), ("warp", 17, 2, 4, 2),
            ("band", 15, 2, 4, 1), ("band", 16, 2, 4, 1), ("band", 17, 2, 4, 1), ("band", 15, 3, 4, 1)]
CTA_SWEEP = [(15, 8, 3, 0, True), (16, 8, 3, 0, True), (17, 8, 3, 0, True), (17, 8, 2, 0, False), (17, 8, 4, 0, False),
             (17, 8, 3, 1, False)]


def compiled_tables():
    s = open(SRC).read()
    body = re.search(r"static const WsVariant\* ws_variants\(int\* n\) \{(.*?)\n\}", s, re.S).group(1)
    ws = []
    for kind, args in re.findall(r"make_ws<(WsCfg|WbCfg)<([^>]*)>>\(\)", body):
        a = [int(x) for x in args.split(",")]
        ws.append(("band", a[0], a[1], 4, 1) if kind == "WbCfg" else ("warp",) + tuple(a + [4, 1][len(a) - 2:]))
    body = re.search(r"static const CombVariant\* comb_variants\(int\* n\) \{(.*?)\n\}", s, re.S).group(1)
    cta = []
    for fn, args in re.findall(r"(make_variant16|make_variant)<CombCfg<([^>]*)>>\(\)", body):
        a = [int(x) for x in args.split(",")]
        cta.append(tuple(a + [0][len(a) - 3:]) + (fn == "make_variant16",))
    return ws, cta


def ws_env(v):
    kind, R, S, W, B = v
    e = {"AMTK_COMB_R": str(R), "AMTK_COMB_WS_STAGES": str(S)}
    if kind == "warp":
        e["AMTK_COMB_WS_WARPS"] = str(W)
        if W == 4 and B == 1:
            e["AMTK_COMB_WS_BAND"] = "0"
        if B == 2:
            e["AMTK_COMB_WS10"] = "1"
    return e


def cta_env(v):
    R, strip, stages, sync, _ = v
    return {"AMTK_COMB_WS": "0", "AMTK_COMB_R": str(R), "AMTK_COMB_STRIP": str(strip), "AMTK_COMB_STAGES": str(stages),
            "AMTK_COMB_SYNC": str(sync)}


# ---- restatement of the host's plan choice (csrc/amtk_b200.cu: pick_ws_R, pick_comb_R, launch_comb_ws, launch_comb,
# launch_comb_mma) ----------------------------------------------------------------------------------------------------
def pick_ws_R(hY, hC):
    best, bw = 17, None
    for R in (17, 16, 15):
        th = 4 * R
        w = 2 * (-(-hY // th) * th - hY) + 2 * (-(-hC // th) * th - hC)
        if bw is None or w < bw:
            best, bw = R, w
    return best


def pick_comb_R(hY, hC):
    best, bw = 16, None
    for R in (17, 16, 15):
        th = 8 * R
        w = -(-hY // th) * th - hY + 2 * (-(-hC // th) * th - hC) // 2
        if bw is None or w < bw:
            best, bw = R, w
    return best


def _tiers(ntiles, nf, nwarps, item, tail):
    big = item if item > 0 else 64
    small = max(4, big // 4)
    while big > 8 and ntiles * (nf // big) < 6 * nwarps:
        big //= 2
        small = max(4, big // 4)
    tail_frames = min(nf, max(small, int(nf * 0.15)))
    head = nf - tail_frames
    end = min(tail_frames, max(tail, int(nf * 0.04))) if 0 < tail < small else 0
    return int(head > 0) + int(nf - end > head) + int(end > 0)


def plan(case):
    """The plan features a case reaches: form, R, pair/merge, band boxes, tile count parity, work-queue tiers."""
    W, H, bits, env, n, vfirst = case["W"], case["H"], case["bits"], case["env"], case["n"], case.get("vfirst", False)
    bps = 1 if bits == 8 else 2
    wC, hC = W // 2, H // 2
    k = lambda name, d: int(env.get(name, d))
    out = {}
    if k("AMTK_COMB_GENERIC", 0):
        out["form"] = "generic"
    elif bps == 1 and k("AMTK_COMB_MMA", 0):
        NS = 2 if k("AMTK_COMB_MMA", 0) == 2 else 1
        ntiles = sum(-(-w // 128) * -(-h // 60) for w, h in ((W, H), (wC, hC), (wC, hC)))
        out.update(form="mma%d" % NS, odd=ntiles % 2 == 1)
    elif k("AMTK_COMB_WS", 1) and (bps == 1 or (bits <= 10 and k("AMTK_COMB_WS10", 0))):
        R = k("AMTK_COMB_R", 0) or pick_ws_R(H, hC)
        band = bps == 1 and k("AMTK_COMB_WS_BAND", 1) == 1 and k("AMTK_COMB_WS_WARPS", 4) == 4
        rem = (wC * bps) % 128
        pair = not band and k("AMTK_COMB_MERGE_UV", 1) == 1 and 0 < rem <= 64 and not vfirst
        ty = lambda h: -(-h // (4 * R))
        ntiles = 0
        for pl, (w, h) in enumerate(((W * bps, H), (wC * bps, hC), (wC * bps, hC))):
            ntiles += (-(-w // 512) if band else (w // 128 if pl and pair else -(-w // 128))) * ty(h)
        ntiles += ty(hC) if pair else 0
        occ = min(WS_OCC, k("AMTK_COMB_CTAS", 0) or WS_OCC)
        nwarps = SM_H100 * occ * (1 if band else k("AMTK_COMB_WS_WARPS", 4))
        out.update(form="band" if band else "ws10" if bps == 2 else "warp", wsR=R, pair=pair,
                   tiers=_tiers(ntiles, n, nwarps, k("AMTK_COMB_ITEM", 0), k("AMTK_COMB_TAIL", 4)))
        if band:
            out["boxes"] = {1 if (w % 512 or 512) <= 256 else 2 for w in (W, wC)}
    else:
        R = k("AMTK_COMB_R", 0) or pick_comb_R(H, hC)
        twe = 128 // bps
        rem = wC % twe
        out.update(form="cta", ctaR=R, merge=k("AMTK_COMB_MERGE_UV", 1) == 1 and 0 < rem <= twe // 2)
    return out


def _c(W, H, bits, env, n, **kw):
    return dict(W=W, H=H, bits=bits, env=env, n=n, **kw)


BAND0 = {"AMTK_COMB_WS_BAND": "0"}
WS10 = {"AMTK_COMB_WS10": "1"}
CTA = {"AMTK_COMB_WS": "0"}
PLAN_CASES = {
    "band_R15": _c(320, 120, 8, {}, 9), "band_R16": _c(320, 128, 8, {}, 5), "band_R17_1952": _c(1952, 136, 8, {}, 3),
    "band_vfirst": _c(320, 120, 8, {}, 9, vfirst=True), "band_tiny": _c(160, 34, 8, {}, 3),
    "band_tail0": _c(320, 120, 8, {"AMTK_COMB_TAIL": "0"}, 40), "band_tail2": _c(320, 120, 8, {"AMTK_COMB_TAIL": "2"}, 40),
    "band_tail1_item256": _c(640, 360, 8, {"AMTK_COMB_TAIL": "1", "AMTK_COMB_ITEM": "256"}, 40),
    "band_ctas1_pf1": _c(640, 360, 8, {"AMTK_COMB_CTAS": "1", "AMTK_COMB_WS_PF": "1"}, 12),
    "band_l2_0": _c(1440, 120, 8, {"AMTK_COMB_L2": "0"}, 5), "band_l2_256": _c(1440, 120, 8, {"AMTK_COMB_L2": "256"}, 5),
    "warp_pair": _c(320, 120, 8, BAND0, 9), "warp_vfirst": _c(320, 120, 8, BAND0, 9, vfirst=True),
    "warp_pair64_R17": _c(384, 136, 8, BAND0, 5), "warp_nopair": _c(512, 128, 8, BAND0, 5),
    "warp_merge0": _c(320, 120, 8, dict(BAND0, AMTK_COMB_MERGE_UV="0"), 9),
    "warp_item8_tail2": _c(320, 120, 8, dict(BAND0, AMTK_COMB_ITEM="8", AMTK_COMB_TAIL="2"), 40),
    "warp_ctas2_pf2": _c(640, 360, 8, dict(BAND0, AMTK_COMB_CTAS="2", AMTK_COMB_WS_PF="2"), 12),
    "warp_l2_128": _c(1920, 64, 8, dict(BAND0, AMTK_COMB_L2="128"), 3),
    "ws10_pair": _c(320, 120, 10, WS10, 9), "ws10_vfirst": _c(320, 120, 10, WS10, 9, vfirst=True),
    "ws10_nopair": _c(224, 136, 10, WS10, 7), "ws10_tail0_pf1": _c(320, 128, 10, dict(WS10, AMTK_COMB_TAIL="0", AMTK_COMB_WS_PF="1"), 40),
    "cta_R15_merge": _c(320, 240, 8, CTA, 5), "cta_R16": _c(512, 256, 8, CTA, 5), "cta_R17": _c(320, 272, 8, CTA, 5),
    "cta_merge0": _c(320, 240, 8, dict(CTA, AMTK_COMB_MERGE_UV="0"), 5),
    "cta_part1": _c(640, 360, 8, dict(CTA, AMTK_COMB_PART="1"), 9), "cta_ctas7": _c(640, 360, 8, dict(CTA, AMTK_COMB_CTAS="7"), 9),
    "cta_l2_256": _c(320, 240, 8, dict(CTA, AMTK_COMB_L2="256"), 5),
    "cta10": _c(320, 240, 10, {}, 5), "cta10_part1": _c(224, 136, 10, {"AMTK_COMB_PART": "1"}, 7),
    "cta12": _c(320, 272, 12, {}, 5), "cta16": _c(1920, 64, 16, {}, 3), "cta16_vfirst": _c(320, 120, 16, {}, 5, vfirst=True),
    "mma1": _c(320, 120, 8, {"AMTK_COMB_MMA": "1"}, 9), "mma2_odd": _c(128, 60, 8, {"AMTK_COMB_MMA": "2"}, 9),
    "mma2_even": _c(320, 120, 8, {"AMTK_COMB_MMA": "2", "AMTK_COMB_ITEM": "8", "AMTK_COMB_CTAS": "1"}, 12),
    "generic8": _c(200, 100, 8, {"AMTK_COMB_GENERIC": "1"}, 5), "generic16": _c(200, 100, 16, {"AMTK_COMB_GENERIC": "1"}, 5),
}


def test_sweep_lists_equal_the_compiled_tables():
    ws, cta = compiled_tables()
    assert len(ws) >= 18 and len(cta) >= 6
    assert sorted(ws) == sorted(WS_SWEEP)
    assert sorted(cta) == sorted(CTA_SWEEP)


def test_plan_cases_reach_every_plan_dimension():
    p = {name: plan(c) for name, c in PLAN_CASES.items()}
    get = lambda key: {v[key] for v in p.values() if key in v}
    assert {15, 16, 17} <= get("wsR") and {15, 16, 17} <= get("ctaR")
    assert get("pair") == {True, False} and get("merge") == {True, False}
    assert set().union(*[v["boxes"] for v in p.values() if "boxes" in v]) == {1, 2}
    assert True in {v["odd"] for v in p.values() if v["form"] == "mma2"} and False in {v["odd"] for v in p.values() if v["form"] == "mma2"}
    assert get("tiers") == {1, 2, 3}
    assert {v["form"] for v in p.values()} == {"band", "warp", "ws10", "cta", "mma1", "mma2", "generic"}
    for form in ("band", "warp"):                             # both 8-bit queue orders with 1, 2 and 3 tiers
        assert {v["tiers"] for v in p.values() if v["form"] == form} == {1, 2, 3}, form
    assert p["warp_vfirst"]["pair"] is False and p["warp_pair"]["pair"] is True and p["ws10_pair"]["pair"] is True


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _ctx(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    c = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    for k in env:
        monkeypatch.delenv(k)
    return c


def _frames(W, H, n, bits, seed=3, mode="interlaced"):
    """(n, W*H*3/2) packed U-first frames; 10/12/16-bit samples spread from 8-bit content, with the largest legal sample
    scattered over the frame."""
    f8 = synth.make_frames(seed, n, W, H, device="cpu", mode=mode).numpy()
    if bits == 8:
        return f8
    a = f8.astype(np.uint32)
    f = (a * 257 if bits == 16 else (a << (bits - 8)) | (a & ((1 << (bits - 8)) - 1))).astype(np.uint16)
    f[:, ::7] = (1 << bits) - 1
    return f


def _oracle_counts(po, f, W, H, prm):
    Y, U, V = [p.view(f.dtype) for p in Layout(W, H, 8 if f.dtype == np.uint8 else 16).planes(f)]
    return po.or_comb_clip(Y, U, V, prm.as_list())


def _vfirst(W, H, bits):
    from test_gpu_plane_order import VFirst
    return VFirst(W, H, bits, packed=True)


def _dclip(f, W, H, bits, vfirst=False, layout=None):
    """(descriptor, device buffer) of frames f: packed U-first, packed V-first or any Layout."""
    L = layout or (_vfirst(W, H, bits) if vfirst else None)
    if L is None:
        buf = torch.from_numpy(f.view(np.int16) if f.dtype == np.uint16 else f).cuda()
        return ab.yv12_clip(buf, W, H, f.shape[0], True, bits), buf
    buf = torch.from_numpy(L.pack(f)).cuda()
    return L.desc(buf, True), buf


def _params(bits):
    p = ab.default_comb_params()
    p.th_move_y, p.th_shima_y, p.th_lshima_y, p.th_move_c, p.th_shima_c, p.th_lshima_c = {
        8: (1, 1, 2047, 128, 700, 701), 10: (80, 48, 3000, 200, 1, 6138), 12: (320, 192, 12000, 800, 1, 24570),
        16: (20000, 3000, 100000, 32768, 1, 393210)}[bits]
    return p


def _check(c, po, f, W, H, bits, prm, vfirst=False, what=""):
    ref = _oracle_counts(po, f, W, H, prm)
    clip, buf = _dclip(f, W, H, bits, vfirst)
    got = c.comb_frames(clip, prm).cpu().numpy()
    assert np.array_equal(got, ref), (what, W, H, bits, vfirst, np.argwhere(got != ref)[:5])
    n = f.shape[0]
    if n > 4:                                                  # range calls with a halo frame
        part = np.concatenate([c.comb_frames(clip, prm, 0, 3).cpu().numpy(), c.comb_frames(clip, prm, 3, 1).cpu().numpy(),
                               c.comb_frames(clip, prm, 4, n - 4).cpu().numpy()])
        assert np.array_equal(part, ref), (what, W, H, bits, "ranges")
    return ref


SHAPES = {8: ((160, 34, 3), (128, 272, 5), (1952, 36, 2), (32, 1100, 2), (640, 360, 9), (320, 120, 9), (1920, 64, 3)),
          10: ((224, 136, 7), (320, 150, 5), (96, 62, 3), (1920, 64, 2), (64, 1100, 2), (320, 120, 9)),
          12: ((224, 136, 7), (320, 120, 5), (1920, 64, 2)),
          16: ((224, 136, 7), (320, 120, 5), (96, 62, 3))}


def _sweep_ids():
    return ["ws_%s_R%d_S%d_W%d_B%d" % v for v in WS_SWEEP] + ["cta_R%d_X%d_S%d_Y%d_%d" % v for v in CTA_SWEEP]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("v", WS_SWEEP + CTA_SWEEP, ids=_sweep_ids())
def test_every_compiled_variant(oracle, monkeypatch, v):
    """Each variant on ragged shapes (partial tiles and bands, planes narrower than a tile, the U|V pair and merge
    classes), extreme thresholds and range calls with a halo frame; the CTA-ring variants without a 16-bit kernel refuse
    16-bit containers with their message."""
    ws = isinstance(v[0], str)
    env = ws_env(v) if ws else cta_env(v)
    bitss = ([10] if v[4] == 2 else [8]) if ws else ([8, 10, 12, 16] if v[4] else [8])
    c = _ctx(monkeypatch, env)
    try:
        for bits in bitss:
            for (W, H, n) in SHAPES[bits]:
                _check(c, oracle, _frames(W, H, n, bits), W, H, bits, _params(bits), what=str(v))
        if not ws and not v[4]:
            f = _frames(224, 136, 3, 10)
            with pytest.raises(ab.AmtkError, match="has no 16-bit kernel"):
                c.comb_frames(_dclip(f, 224, 136, 10)[0], _params(10))
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(PLAN_CASES))
def test_plan_case(oracle, monkeypatch, name):
    """The cases that reach every plan dimension (see test_plan_cases_reach_every_plan_dimension), each against the spec."""
    cs = PLAN_CASES[name]
    W, H, bits, n = cs["W"], cs["H"], cs["bits"], cs["n"]
    c = _ctx(monkeypatch, cs["env"])
    try:
        ref = _check(c, oracle, _frames(W, H, n, bits, seed=n), W, H, bits, _params(bits), cs.get("vfirst", False), name)
        assert ref.sum() > 0
    finally:
        c.close()


def _probe(monkeypatch, env, clip, prm):
    """Which form a context with AMTK_COMB_R=11 (no compiled variant has R = 11) runs: the warp-stream and CTA-ring
    launchers refuse before any launch, the generic and tensor-core forms do not use R and run."""
    c = _ctx(monkeypatch, dict(env, AMTK_COMB_R="11"))
    try:
        c.comb_frames(clip, prm)
        return "runs"
    except ab.AmtkError as e:
        msg = str(e)
        if "no warp-stream kernel variant" in msg:
            return "ws"
        if "comb: no kernel variant" in msg:
            return "cta"
        raise
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_dispatch(monkeypatch):
    W, H = 320, 120
    clips = {}
    keep = []
    for bits in (8, 10, 12, 16):
        f = _frames(W, H, 3, bits)
        for vf in (False, True):
            d, b = _dclip(f, W, H, bits, vf)
            clips[(bits, vf)] = d
            keep.append(b)
    f = _frames(W, H, 3, 8)                                   # off_u 8 bytes past a 16-byte boundary: no tensor map
    mis = Layout(W, H, 8, W, W // 2, 8)
    d, b = _dclip(f, W, H, 8, layout=mis)
    clips["mis"] = d
    keep.append(b)
    expect = {   # env -> {clip: form}
        (): {(8, False): "ws", (8, True): "ws", "mis": "runs", (10, False): "cta", (10, True): "cta", (12, False): "cta",
             (16, False): "cta", (16, True): "cta"},
        (("AMTK_COMB_WS_BAND", "0"),): {(8, False): "ws", (8, True): "ws", "mis": "runs"},
        (("AMTK_COMB_WS_WARPS", "2"),): {(8, False): "ws"},
        (("AMTK_COMB_WS10", "1"),): {(8, False): "ws", (10, False): "ws", (10, True): "ws", (12, False): "cta", (16, False): "cta"},
        (("AMTK_COMB_WS", "0"),): {(8, False): "cta", (8, True): "cta", (10, False): "cta", "mis": "runs"},
        (("AMTK_COMB_WS", "0"), ("AMTK_COMB_WS10", "1")): {(10, False): "cta"},
        (("AMTK_COMB_MMA", "1"),): {(8, False): "runs", (8, True): "runs", (10, False): "cta", "mis": "runs"},
        (("AMTK_COMB_MMA", "2"),): {(8, False): "runs", (16, False): "cta"},
        (("AMTK_COMB_GENERIC", "1"),): {(8, False): "runs", (8, True): "runs", (10, False): "runs", (12, False): "runs",
                                        (16, True): "runs"},
    }
    for env, want in expect.items():
        for key, form in want.items():
            bits = 8 if key == "mis" else key[0]
            got = _probe(monkeypatch, dict(env), clips[key], _params(bits))
            assert got == form, (env, key, got)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("form", ["band", "warp", "ws10", "mma", "cta"])
def test_cached_plan_reuse(oracle, monkeypatch, form):
    """One context, a sequence of calls that each change one input of the launch plan: plane order (U-first -> V-first ->
    U-first: the per-warp forms pair U and V only on U-first clips, so the tile count changes while the geometry does not),
    frame count, first frame, geometry, bit depth, pitch, frame stride, host clips.  Every call must equal the spec."""
    env = {"band": {}, "warp": BAND0, "ws10": WS10, "mma": {"AMTK_COMB_MMA": "2"}, "cta": CTA}[form]
    bits = 10 if form == "ws10" else 8
    other = 8 if bits == 10 else 10
    c = _ctx(monkeypatch, env)
    cache = {}

    def prm(b):                                                # every chroma sample counts: no tile may go unread
        p = _params(b)
        p.th_move_c = p.th_shima_c = 1
        return p

    def data(W, H, b, n=9):
        if (W, H, b, n) not in cache:
            f = _frames(W, H, n, b, seed=W + H + b)
            ref = _oracle_counts(oracle, f, W, H, prm(b))
            assert ref[:, [7, 10]].min() > 0
            cache[(W, H, b, n)] = (f, ref)
        return cache[(W, H, b, n)]

    def call(W, H, b, f0=0, nf=None, vfirst=False, layout=None, host=False, n=9):
        f, ref = data(W, H, b, n)
        nf = f.shape[0] - f0 if nf is None else nf
        L = layout or (_vfirst(W, H, b) if vfirst else Layout(W, H, b, W * (1 if b == 8 else 2), (W // 2) * (1 if b == 8 else 2)))
        if host:
            buf = L.pack(f)
            got = c.comb_frames(L.desc(buf, False), prm(b), f0, nf)
            got = got.cpu().numpy() if hasattr(got, "cpu") else np.asarray(got)
        else:
            clip, buf = _dclip(f, W, H, b, layout=L)
            got = c.comb_frames(clip, prm(b), f0, nf).cpu().numpy()
        assert np.array_equal(got, ref[f0:f0 + nf]), (form, W, H, b, f0, nf, vfirst, host, np.argwhere(got != ref[f0:f0 + nf])[:5])

    try:
        call(320, 120, bits, 0, 5)
        call(320, 120, bits)                                  # frame count
        call(320, 120, bits, vfirst=True)                     # same geometry and range, other plane order
        call(320, 120, bits)
        call(320, 120, bits, vfirst=True)
        call(320, 120, bits, 0, 5)                            # frame count
        call(320, 120, bits, 2, 5)                            # first frame
        call(320, 120, bits, 2, 5, vfirst=True)
        call(352, 120, bits)                                  # width (176-byte chroma rows: still a pair at 8 bits)
        call(320, 136, bits)                                  # height
        call(320, 120, other)                                 # bit depth
        call(320, 120, bits)
        s = 1 if bits == 8 else 2
        call(320, 120, bits, layout=Layout(320, 120, bits, 384 * s, 192 * s))          # pitch
        call(320, 120, bits, layout=Layout(320, 120, bits, 384 * s, 192 * s, 32))      # frame stride and plane distance
        from test_gpu_plane_order import VFirst
        call(320, 120, bits, layout=VFirst(320, 120, bits, 384 * s, 192 * s, 32))
        monkeypatch.setenv("AMTK_STAGE_MB", "1")
        call(320, 120, bits, 1, 60, host=True, n=64)          # host clip: staged windows of a few frames each
        call(320, 120, bits, 1, 60, vfirst=True, host=True, n=64)
        monkeypatch.delenv("AMTK_STAGE_MB")
        call(320, 120, bits, n=64)
        call(320, 120, bits)
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_generic_kernel_past_16384_frames(ctx, oracle):
    """The generic kernel launches at most 16384 frames at a time (gridDim.z = 3 planes x frames).  Each later launch takes
    the frame before its own first frame as the previous one -- the last frame of the launch before it."""
    W, H = 64, 36
    L = Layout(W, H, 8, W, W // 2, 8)                          # off_u 8 bytes past a 16-byte boundary: no tensor map
    n = 2 * 16384 + 5
    rng = np.random.default_rng(16384)
    f = rng.integers(0, 256, (n, W * H * 3 // 2), dtype=np.uint8)
    prm = ab.default_comb_params()
    ref = _oracle_counts(oracle, f, W, H, prm)
    assert ref[1:, 0].min() > 0                                # every frame moves against its predecessor
    buf = torch.from_numpy(L.pack(f)).cuda()
    clip = L.desc(buf, True)
    got = ctx.comb_frames(clip, prm).cpu().numpy()
    assert np.array_equal(got, ref), np.argwhere(got != ref)[:5]
    f0, nf = 7, 16384 + 3
    got = ctx.comb_frames(clip, prm, f0, nf).cpu().numpy()
    assert np.array_equal(got, ref[f0:f0 + nf]), np.argwhere(got != ref[f0:f0 + nf])[:5]
