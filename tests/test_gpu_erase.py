"""AMTEraseLogo (erase_logo_kernel) at every bit depth and chroma field parity, against a reference built in the test from
the eight Delogo calls of AMTEraseLogo::GetFrameT (LogoScan.hpp:1356-1397) with the reference's own offsets, run through
the reference's own Delogo (oracle/_ref) where it was built, else the C port.

Frame mode (fadeT == fadeB) erases the whole logo rectangle; field mode erases h/2 rows per field, so an odd h (or an odd
hUV) leaves the last row untouched, and the chroma rows of the top field start at (imgy/2) % 2.  Everything outside the
three logo rectangles must stay as it was."""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab

FADES = np.array([[1, 1], [0, 0], [0.5, 0.5], [1, 0], [0, 1], [0.3, 0.7]], np.float32)


def logo_data(w, h, seed):
    """LogoData planes aY,bY,aU,bU,aV,bV of any size (odd ones too) under the model bg = a*src + b*maxv (LogoScan.hpp:247):
    a = 1/(1-alpha), b = -alpha*L*a, with opacity 0..0.6 and logo level L 0..1."""
    rng = np.random.default_rng(seed)
    out = []
    for n in (w * h, (w >> 1) * (h >> 1), (w >> 1) * (h >> 1)):
        alpha = rng.integers(0, 154, n) / 256.0
        alpha[rng.random(n) < 0.2] = 0.0
        lev = rng.integers(0, 256, n) / 255.0
        a = 1.0 / (1.0 - alpha)
        out += [a, -alpha * lev * a]
    return np.concatenate(out).astype(np.float32)


def _delogo(po):
    return po.ref_delogo if po.ref_has_erase() else po.or_delogo


def erase_reference(po, logo_data, w, h, imgx, imgy, Y, U, V, fadeT, fadeB, maxv):
    """AMTEraseLogo::GetFrameT, mode 0, on 2-D planes (edited in place); logUVx = logUVy = 1."""
    delogo = _delogo(po)
    wUV, hUV = w >> 1, h >> 1
    ny, nc = w * h, wUV * hUV
    d = np.asarray(logo_data, np.float32)
    aY, bY = d[:ny], d[ny:2 * ny]
    aU, bU = d[2 * ny:2 * ny + nc], d[2 * ny + nc:2 * ny + 2 * nc]
    aV, bV = d[2 * ny + 2 * nc:2 * ny + 3 * nc], d[2 * ny + 3 * nc:2 * ny + 4 * nc]
    pitchY, pitchUV = Y.shape[1], U.shape[1]
    off = imgx + imgy * pitchY
    offUV = (imgx >> 1) + (imgy >> 1) * pitchUV
    fy, fu, fv = Y.reshape(-1), U.reshape(-1), V.reshape(-1)

    def run(flat, o, ww, hh, lp, ip, A, B, fade):
        # Delogo(dst + o, ...): the reference pointer arithmetic on a flat view of the plane
        view = flat[o:]
        rows = (hh - 1) * ip + ww if hh > 0 else 0
        if rows <= 0:
            return
        buf = np.ascontiguousarray(view[:rows])
        delogo(buf, A, B, fade, maxv, logopitch=lp, imgpitch=ip, w=ww, h=hh)
        view[:rows] = buf

    if fadeT == fadeB:
        run(fy, off, w, h, w, pitchY, aY, bY, fadeT)
        run(fu, offUV, wUV, hUV, wUV, pitchUV, aU, bU, fadeT)
        run(fv, offUV, wUV, hUV, wUV, pitchUV, aV, bV, fadeT)
    else:
        run(fy, off, w, h // 2, w * 2, pitchY * 2, aY, bY, fadeT)
        run(fy, off + pitchY, w, h // 2, w * 2, pitchY * 2, aY[w:], bY[w:], fadeB)
        uvparity = (imgy // 2) % 2
        tuvoff, buvoff = uvparity * pitchUV, (1 - uvparity) * pitchUV
        tuvoffl, buvoffl = uvparity * wUV, (1 - uvparity) * wUV
        run(fu, offUV + tuvoff, wUV, hUV // 2, wUV * 2, pitchUV * 2, aU[tuvoffl:], bU[tuvoffl:], fadeT)
        run(fv, offUV + tuvoff, wUV, hUV // 2, wUV * 2, pitchUV * 2, aV[tuvoffl:], bV[tuvoffl:], fadeT)
        run(fu, offUV + buvoff, wUV, hUV // 2, wUV * 2, pitchUV * 2, aU[buvoffl:], bU[buvoffl:], fadeB)
        run(fv, offUV + buvoff, wUV, hUV // 2, wUV * 2, pitchUV * 2, aV[buvoffl:], bV[buvoffl:], fadeB)


def logo_rect_mask(W, H, w, h, imgx, imgy):
    """True on every sample of a packed frame that lies inside one of the three logo rectangles."""
    m = np.zeros(W * H * 3 // 2, bool)
    m[:W * H].reshape(H, W)[imgy:imgy + h, imgx:imgx + w] = True
    cw, ch = W // 2, H // 2
    for o in (W * H, W * H + cw * ch):
        m[o:o + cw * ch].reshape(ch, cw)[imgy >> 1:(imgy >> 1) + (h >> 1), imgx >> 1:(imgx >> 1) + (w >> 1)] = True
    return m


def _frames(n, W, H, bits, seed):
    maxv = (1 << bits) - 1
    rng = np.random.default_rng(seed)
    a = rng.integers(0, maxv + 1, (n, W * H * 3 // 2))
    a[:, ::7] = maxv
    a[:, 3::11] = 0
    return a.astype(np.uint8 if bits == 8 else np.uint16)


def _expected(po, data, w, h, imgx, imgy, frames, W, H, fades, maxv):
    exp = frames.copy()
    for i in range(exp.shape[0]):
        Y = exp[i, :W * H].reshape(H, W)
        U = exp[i, W * H:W * H + (W // 2) * (H // 2)].reshape(H // 2, W // 2)
        V = exp[i, W * H + (W // 2) * (H // 2):].reshape(H // 2, W // 2)
        erase_reference(po, data, w, h, imgx, imgy, Y, U, V, fades[i, 0], fades[i, 1], maxv)
    return exp


@pytest.mark.parametrize("geom", [(64, 64, 160, 32), (48, 41, 33, 34), (50, 42, 17, 35), (46, 46, 1, 2), (42, 43, 213, 84)])
def test_erase_composition_matches_port(oracle, geom):
    """The composition above equals the C port's AMTEraseLogo::GetFrameT (or_erase_frame) on 8-bit frames, in frame and
    field mode, at both chroma parities and with odd h / odd hUV."""
    po = oracle
    w, h, imgx, imgy = geom
    W, H = 256, 128
    O = po.OracleLogo.create(logo_data(w, h, seed=w), w, h, W, H, imgx, imgy)
    fr = _frames(len(FADES), W, H, 8, seed=h)
    for i, (ft, fb) in enumerate(FADES):
        a = fr[i].copy()
        Y = np.ascontiguousarray(a[:W * H].reshape(H, W))
        U = np.ascontiguousarray(a[W * H:W * H + W * H // 4].reshape(H // 2, W // 2))
        V = np.ascontiguousarray(a[W * H + W * H // 4:].reshape(H // 2, W // 2))
        po.or_erase_frame(O, Y, U, V, ft, fb)
        b = fr[i:i + 1].copy()
        got = _expected(po, O.data(), w, h, imgx, imgy, b, W, H, FADES[i:i + 1], 255.0)[0]
        assert np.array_equal(got, np.concatenate([Y.ravel(), U.ravel(), V.ravel()])), (geom, ft, fb)
        assert np.array_equal(got[~logo_rect_mask(W, H, w, h, imgx, imgy)], fr[i][~logo_rect_mask(W, H, w, h, imgx, imgy)])


# (w, h, imgx, imgy): chroma parity (imgy/2)%2 = 0 | 1, odd imgx, odd h, odd hUV
ERASE_GEOMS = [(64, 64, 160, 32), (48, 41, 33, 34), (50, 42, 17, 35), (46, 46, 1, 2), (42, 43, 213, 84)]


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [8, 10, 12, 16])
def test_erase_every_depth_and_parity(ctx, oracle, bits, monkeypatch):
    po = oracle
    maxv = float((1 << bits) - 1)
    W, H = 256, 128
    n = 2 * len(FADES) + 2
    fades = np.concatenate([FADES, FADES[::-1], FADES[:2]])
    for gi, (w, h, imgx, imgy) in enumerate(ERASE_GEOMS):
        d = logo_data(w, h, seed=w + gi)
        logo = ab.Logo.create(d, w, h, W, H, imgx, imgy)
        data = po.OracleLogo.create(d, w, h, W, H, imgx, imgy).data()
        orig = _frames(n, W, H, bits, seed=bits * 10 + gi)
        exp = _expected(po, data, w, h, imgx, imgy, orig, W, H, fades, maxv)
        outside = ~logo_rect_mask(W, H, w, h, imgx, imgy)
        assert np.array_equal(exp[:, outside], orig[:, outside])
        # device clip, whole range
        dev = torch.from_numpy(orig.view(np.int16) if bits > 8 else orig).cuda()
        ctx.erase_logo(ab.yv12_clip(dev, W, H, n, True, bits), logo, fades)
        got = dev.cpu().numpy().view(orig.dtype)
        assert np.array_equal(got, exp), (bits, gi, np.argwhere(got != exp)[:4])
        # host clip in 1 MiB staging chunks, range starting at frame0 > 0: earlier frames stay untouched
        monkeypatch.setenv("AMTK_STAGE_MB", "1")
        host = orig.copy()
        f0 = 3
        ctx.erase_logo(ab.yv12_clip(host, W, H, n, False, bits), logo, fades[f0:], frame0=f0, nframes=n - f0)
        monkeypatch.delenv("AMTK_STAGE_MB")
        exp_h = orig.copy()
        exp_h[f0:] = _expected(po, data, w, h, imgx, imgy, orig[f0:], W, H, fades[f0:], maxv)
        assert np.array_equal(host, exp_h), (bits, gi, "host", np.argwhere(host != exp_h)[:4])
