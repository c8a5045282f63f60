"""amtk_logo_find_rects (the logo finder's rectangle rule, DESIGN.md section 3.5) without a device: a numpy restatement of
the rule agrees with the library on constructed sum maps, rectangles, order and scores; refusals; the header compiles as
C99 with the new names."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import amatsukaze_b200 as ab

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUNCS = ["amtk_logo_find_create", "amtk_logo_find_destroy", "amtk_logo_find_add_frames", "amtk_logo_find_get_sums",
         "amtk_logo_find_default_params", "amtk_logo_find_rects"]


def rule(s1, s2, n, bits, block=8, var_ratio=0.5, mean_delta=6.0, margin=8, min_blocks=4):
    """The rule of DESIGN.md section 3.5, restated.  Sums are taken in the order the library takes them, so the doubles
    are the same."""
    H, W = s1.shape
    B, bw, bh = block, W // block, H // block
    if n < 2 or bw < 3 or bh < 3:
        return [], []
    m = s1.astype(np.float64) / float(n)
    v = s2.astype(np.float64) / float(n) - m * m
    ex = np.zeros_like(m)
    ey = np.zeros_like(m)
    ex[:, :-1] = np.abs(m[:, 1:] - m[:, :-1])
    ey[:-1, :] = np.abs(m[1:, :] - m[:-1, :])
    sv = np.zeros((bh, bw))
    se = np.zeros((bh, bw))
    for dy in range(B):
        for dx in range(B):
            sv = sv + v[dy:bh * B:B, dx:bw * B:B]
            se = se + (ex[dy:bh * B:B, dx:bw * B:B] + ey[dy:bh * B:B, dx:bw * B:B])
    bv, be = sv / float(B * B), se / float(B * B)
    vmed = np.sort(bv.ravel())[(bv.size - 1) // 2]
    emed = np.sort(be.ravel())[(be.size - 1) // 2]
    if not vmed > 0:
        return [], []
    vlim = float(np.float32(var_ratio)) * vmed
    dlim = float(np.float32(mean_delta)) * float((1 << bits) - 1) / 255.0
    held = np.zeros((bh, bw), bool)
    strength = np.zeros((bh, bw))
    iv, ie = bv[1:-1, 1:-1], be[1:-1, 1:-1]
    h = (iv <= vlim) | (ie - emed >= dlim)
    held[1:-1, 1:-1] = h
    strength[1:-1, 1:-1] = np.where(h, np.maximum(1.0 - iv / vmed, 0.0) + np.maximum(ie - emed, 0.0) / dlim, 0.0)
    seen = np.zeros((bh, bw), bool)
    out = []
    W2, H2 = W & ~1, H & ~1
    for by in range(bh):
        for bx in range(bw):
            if not held[by, bx] or seen[by, bx]:
                continue
            members, stack = [], [(by, bx)]
            seen[by, bx] = True
            while stack:
                cy, cx = stack.pop()
                members.append((cy, cx))
                for dy in (-1, 0, 1):
                    for dx in (-1, 0, 1):
                        ny, nx = cy + dy, cx + dx
                        if 0 <= ny < bh and 0 <= nx < bw and held[ny, nx] and not seen[ny, nx]:
                            seen[ny, nx] = True
                            stack.append((ny, nx))
            if len(members) < min_blocks:
                continue
            ys = [p[0] for p in members]
            xs = [p[1] for p in members]
            if (min(ys) == 1 and max(ys) == bh - 2) or (min(xs) == 1 and max(xs) == bw - 2):
                continue                                   # bars
            total = 0.0
            for p in members:                              # in the order the blocks leave the depth-first stack
                total += strength[p]
            rx0 = max(0, min(xs) * B - margin) & ~1
            ry0 = max(0, min(ys) * B - margin) & ~1
            rx1 = min(W2, ((max(xs) + 1) * B + margin + 1) & ~1)
            ry1 = min(H2, ((max(ys) + 1) * B + margin + 1) & ~1)
            w = min(4096, max(4, rx1 - rx0))
            hh = min(4096, max(4, ry1 - ry0))
            out.append(((min(rx0, W2 - w), min(ry0, H2 - hh), w, hh), np.float32(total)))
    out.sort(key=lambda r: -float(r[1]))          # stable: equal scores keep raster order
    return [r[0] for r in out], [r[1] for r in out]


def background(H, W, seed, bits=8):
    """Mean and variance maps (float64) of moving content after many frames: a smooth mean with a little per-pixel noise,
    and a variance around (maxv / 8)^2."""
    rng = np.random.default_rng(seed)
    k = ((1 << bits) - 1) / 255.0
    y, x = np.mgrid[0:H, 0:W]
    m = k * (110 + 20 * np.sin(x / 37.0) * np.cos(y / 29.0) + rng.normal(0, 0.3, (H, W)))
    v = (k * 32) ** 2 * (1 + 0.1 * rng.random((H, W)))
    return m, v


def texture(h, w):
    """A logo's own pattern: 4 x 4 cells of 1 and 0.4."""
    y, x = np.mgrid[0:h, 0:w]
    return np.where((x // 4 + y // 4) % 2 == 0, 1.0, 0.4)


def add_logo(m, v, x, y, w, h, shift=0.0, var_scale=1.0):
    """A logo at (x, y, w, h): its pattern times `shift` added to the mean, the variance scaled by var_scale."""
    m = m.copy()
    v = v.copy()
    roi = m[y:y + h, x:x + w]
    roi += shift * texture(*roi.shape)
    v[y:y + h, x:x + w] *= var_scale
    return m, v


def sums_of(m, v, n):
    """Exact-integer sum maps (uint64) of n frames with per-pixel mean m and variance v."""
    s1 = np.rint(m * n)
    mm = s1 / n
    s2 = np.rint((v + mm * mm) * n)
    return s1.astype(np.uint64), s2.astype(np.uint64)


def check(s1, s2, n, bits, params=None, **kw):
    p = params if params is not None else ab.default_logo_find_params()
    rects, scores = ab.logo_find_rects(s1, s2, n, bits, p, max_rects=64)
    want_r, want_s = rule(s1, s2, n, bits, p.block, p.var_ratio, p.mean_delta, p.margin, p.min_blocks)
    assert [tuple(r) for r in rects.tolist()] == [tuple(r) for r in want_r[:64]]
    assert np.array_equal(np.asarray(scores, np.float32).view(np.uint32), np.asarray(want_s[:64], np.float32).view(np.uint32))
    return [tuple(r) for r in rects.tolist()], scores


def covers(rect, x, y, w, h, slack):
    rx, ry, rw, rh = rect
    return (rx <= x and ry <= y and rx + rw >= x + w and ry + rh >= y + h and
            x - rx <= slack and y - ry <= slack and rx + rw - (x + w) <= slack and ry + rh - (y + h) <= slack)


def test_defaults():
    p = ab.default_logo_find_params()
    assert (p.block, p.var_ratio, p.mean_delta, p.margin, p.min_blocks) == (8, 0.5, 6.0, 8, 4)


def test_lowered_variance_only():
    m, v = background(96, 160, 1)
    m, v = add_logo(m, v, 96, 16, 32, 24, var_scale=0.3)
    s1, s2 = sums_of(m, v, 600)
    rects, scores = check(s1, s2, 600, 8)
    assert len(rects) == 1 and covers(rects[0], 96, 16, 32, 24, 16)


def test_shifted_mean_only():
    m, v = background(96, 160, 2)
    m, v = add_logo(m, v, 24, 40, 32, 24, shift=40)
    s1, s2 = sums_of(m, v, 600)
    rects, _ = check(s1, s2, 600, 8)
    assert len(rects) == 1 and covers(rects[0], 24, 40, 32, 24, 16)


@pytest.mark.parametrize("bits", [8, 10, 12, 16])
def test_both_signs_at_every_depth(bits):
    k = ((1 << bits) - 1) / 255.0
    m, v = background(128, 192, 3, bits)
    m, v = add_logo(m, v, 130, 20, 40, 32, shift=30 * k, var_scale=0.45)
    s1, s2 = sums_of(m, v, 1800)
    rects, scores = check(s1, s2, 1800, bits)
    assert len(rects) == 1 and covers(rects[0], 130, 20, 40, 32, 16)


@pytest.mark.parametrize("kind", ["letterbox", "pillarbox"])
def test_bars_are_not_reported(kind):
    m, v = background(120, 200, 4)
    m, v = add_logo(m, v, 112, 40, 32, 32, shift=40, var_scale=0.5)
    bars = (np.s_[:20, :], np.s_[-20:, :]) if kind == "letterbox" else (np.s_[:, :40], np.s_[:, -40:])
    for b in bars:
        m[b], v[b] = 16.0, 0.0
    s1, s2 = sums_of(m, v, 300)
    rects, _ = check(s1, s2, 300, 8)
    assert len(rects) == 1 and covers(rects[0], 112, 40, 32, 32, 16)


def test_still_picture_and_too_few_frames():
    m, v = background(64, 64, 5)
    s1, s2 = sums_of(m, v * 0, 30)
    assert check(s1, s2, 30, 8)[0] == []                       # median block variance 0
    m, v = add_logo(*background(64, 64, 6), 24, 24, 16, 16, shift=50, var_scale=0.2)
    s1, s2 = sums_of(m, v, 1)
    assert check(s1, s2, 1, 8)[0] == []
    assert check(s1, s2, 0, 8)[0] == []
    s1, s2 = sums_of(m, v, 2)
    assert len(check(s1, s2, 2, 8)[0]) == 1


@pytest.mark.parametrize("H,W", [(67, 91), (17, 16), (101, 153), (35, 4099)])
def test_odd_frame_sizes(H, W):
    m, v = background(H, W, 7)
    x, y = (W // 2) & ~7, max(8, (H // 3) & ~7)
    m, v = add_logo(m, v, x, y, 16, 8, shift=50, var_scale=0.3)
    s1, s2 = sums_of(m, v, 100)
    rects, _ = check(s1, s2, 100, 8)
    for rx, ry, rw, rh in rects:
        assert rx % 2 == 0 and ry % 2 == 0 and rw % 2 == 0 and rh % 2 == 0
        assert rx + rw <= W and ry + rh <= H and 4 <= rw <= 4096 and 4 <= rh <= 4096


def test_wide_components_are_clamped():
    m, v = background(64, 4400, 11)
    m, v = add_logo(m, v, 16, 24, 4300, 16, shift=50, var_scale=0.3)
    s1, s2 = sums_of(m, v, 100)
    rects, _ = check(s1, s2, 100, 8)
    assert rects and rects[0][2] == 4096


def test_corners_and_frame_edges():
    H, W = 144, 256
    m0, v0 = background(H, W, 8)
    spots = [(8, 8), (W - 40, 8), (8, H - 40), (W - 40, H - 40)]
    m, v = m0, v0
    for i, (x, y) in enumerate(spots):
        m, v = add_logo(m, v, x, y, 32, 32, shift=30 + 10 * i, var_scale=0.4)
    s1, s2 = sums_of(m, v, 500)
    rects, scores = check(s1, s2, 500, 8)
    assert len(rects) == 4 and list(scores) == sorted(scores, reverse=True)
    for x, y in spots:
        assert sum(covers(r, x + 8, y + 8, 16, 16, 32) for r in rects) == 1
    # a logo reaching the frame's edge: its edge blocks are never held, the rectangle is clipped to the frame
    m, v = add_logo(m0, v0, 0, 0, 48, 40, shift=40, var_scale=0.3)
    s1, s2 = sums_of(m, v, 500)
    rects, _ = check(s1, s2, 500, 8)
    assert len(rects) == 1 and rects[0][0] == 0 and rects[0][1] == 0


@pytest.mark.parametrize("block,margin,min_blocks", [(2, 0, 1), (4, 3, 2), (16, 8, 1), (8, 100, 4), (5, 7, 3)])
def test_other_parameters(block, margin, min_blocks):
    m, v = background(128, 160, 9)
    m, v = add_logo(m, v, 64, 48, 40, 32, shift=-40, var_scale=0.6)
    s1, s2 = sums_of(m, v, 200)
    p = ab.default_logo_find_params()
    p.block, p.margin, p.min_blocks = block, margin, min_blocks
    check(s1, s2, 200, 8, p)
    p.var_ratio, p.mean_delta = 0.9, 2.5
    check(s1, s2, 200, 8, p)


def test_max_rects_and_null_scores():
    H, W = 144, 256
    m, v = background(H, W, 8)
    for x, y in [(16, 16), (W - 48, 16), (16, H - 48)]:
        m, v = add_logo(m, v, x, y, 32, 32, shift=40, var_scale=0.4)
    s1, s2 = sums_of(m, v, 300)
    full, _ = ab.logo_find_rects(s1, s2, 300, 8, max_rects=16)
    part, _ = ab.logo_find_rects(s1, s2, 300, 8, max_rects=2)
    assert len(full) == 3 and np.array_equal(part, full[:2])
    L = ab.lib()
    rects, n = np.zeros((4, 4), np.int32), C.c_int()
    p = ab.default_logo_find_params()
    assert L.amtk_logo_find_rects(s1.ctypes.data, s2.ctypes.data, 300, W, H, 8, C.byref(p), 4,
                                  rects.ctypes.data_as(ab.capi.c_i32_p), None, C.byref(n)) == 1
    assert n.value == 3 and np.array_equal(rects[:3], full)


def test_refusals():
    L = ab.lib()
    s = np.zeros((32, 32), np.uint64)
    p = ab.default_logo_find_params()
    rects, n = np.zeros((4, 4), np.int32), C.c_int()
    rp = rects.ctypes.data_as(ab.capi.c_i32_p)

    def call(s1, s2, w, h, bits, pp, r=rp, nn=C.byref(n)):
        return L.amtk_logo_find_rects(s1, s2, 10, w, h, bits, pp, 4, r, None, nn)

    assert call(None, s.ctypes.data, 32, 32, 8, C.byref(p)) == 0
    assert b"null argument" in L.amtk_last_error()
    assert call(s.ctypes.data, None, 32, 32, 8, C.byref(p)) == 0
    assert call(s.ctypes.data, s.ctypes.data, 32, 32, 8, None) == 0
    assert call(s.ctypes.data, s.ctypes.data, 32, 32, 8, C.byref(p), r=None) == 0
    assert call(s.ctypes.data, s.ctypes.data, 32, 32, 8, C.byref(p), nn=None) == 0
    for b in (1, 0, -3):
        q = ab.default_logo_find_params()
        q.block = b
        assert call(s.ctypes.data, s.ctypes.data, 32, 32, 8, C.byref(q)) == 0
        assert b"block must be at least 2" in L.amtk_last_error()
    for w, h in ((15, 32), (32, 15), (8193, 32), (32, 8193), (0, 0)):
        assert call(s.ctypes.data, s.ctypes.data, w, h, 8, C.byref(p)) == 0
        assert b"width and height must be in [16, 8192]" in L.amtk_last_error()
    assert call(s.ctypes.data, s.ctypes.data, 32, 32, 17, C.byref(p)) == 0
    assert call(s.ctypes.data, s.ctypes.data, 32, 32, 8, C.byref(p)) == 1 and n.value == 0


def test_finder_without_a_context_is_refused():
    L = ab.lib()
    out = C.c_void_p()
    assert L.amtk_logo_find_create(None, C.byref(out)) == 0
    assert b"amtk_logo_find_create: null argument" in L.amtk_last_error()
    assert L.amtk_logo_find_add_frames(None, None, 0, 1) == 0
    assert L.amtk_logo_find_get_sums(None, None, None, None) == 0
    L.amtk_logo_find_destroy(None)


def test_header_compiles_as_c99_with_the_new_symbols(tmp_path):
    src = tmp_path / "use.c"
    src.write_text('#include "amtk_b200.h"\n'
                   "int (*create)(amtk_ctx*, amtk_logo_find**) = amtk_logo_find_create;\n"
                   "void (*destroy)(amtk_logo_find*) = amtk_logo_find_destroy;\n"
                   "int (*add)(amtk_logo_find*, const amtk_clip*, int, int) = amtk_logo_find_add_frames;\n"
                   "int (*sums)(amtk_logo_find*, uint64_t*, uint64_t*, int64_t*) = amtk_logo_find_get_sums;\n"
                   "void (*defaults)(amtk_logo_find_params*) = amtk_logo_find_default_params;\n"
                   "int (*rects)(const uint64_t*, const uint64_t*, int64_t, int, int, int, const amtk_logo_find_params*, int,\n"
                   "             int32_t*, float*, int*) = amtk_logo_find_rects;\n")
    r = subprocess.run(["cc", "-std=c99", "-pedantic", "-Werror", "-c", str(src), "-I", os.path.join(ROOT, "include"),
                        "-o", str(tmp_path / "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_ctypes_sees_the_symbols():
    names = [s[0] for s in ab.SIGNATURES]
    L = ab.lib()
    for f in FUNCS:
        assert f in names and hasattr(L, f), f
