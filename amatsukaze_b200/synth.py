"""Deterministic synthetic clips and logos (integer-only, identical on CPU and CUDA).

Used by tests/, bench.py and __graft_entry__.smoke() to feed BOTH the CUDA path and the CPU oracle the same
bytes (SURVEY.md section 8(d) "Synthetic inputs").  All pixel arithmetic is integer torch ops, so a tensor made on
`cuda:0` equals the one made on `cpu` bit for bit.  Nothing here touches oracle/.

Frame layout produced: tightly packed YV12 -- Y (H x W), U (H/2 x W/2), V (H/2 x W/2), one frame after the other
(frame stride W*H*3/2 bytes), i.e. exactly what amtk_clip_desc describes with pitchY=W, pitchUV=W/2.
"""
import numpy as np
import torch

M32 = 0xFFFFFFFF


def _hash32(x, y, n, plane, seed):
    """32-bit avalanche hash of (x, y, n, plane, seed) evaluated in int64 with masking (portable, exact)."""
    h = (x * 0x9E3779B1 + y * 0x85EBCA77 + n * 0xC2B2AE3D + (plane * 0x27D4EB2F + seed)) & M32
    h = h ^ (h >> 15)
    h = (h * 0x2C1B3C6D) & M32
    h = h ^ (h >> 12)
    h = (h * 0x297A2D39) & M32
    h = h ^ (h >> 15)
    return h


def make_logo(w=64, h=64, seed=1, L8=230):
    """Opacity-blob logo.  Returns dict with alpha8 (h,w) uint8, alphaC (h/2,w/2), L8, and `data`: float32 LogoData
    layout aY,bY,aU,bU,aV,bV (AMTLogo.hpp:206-212) following the reference model bg = a*src + b*maxv
    (LogoScan.hpp:247), i.e. a = 1/(1-alpha), b = -alpha*L/(1-alpha)."""
    yy, xx = np.mgrid[0:h, 0:w]
    cx, cy = w * 0.5, h * 0.5
    r = ((xx - cx) / (w * 0.36)) ** 2 + ((yy - cy) / (h * 0.30)) ** 2
    alpha8 = np.zeros((h, w), np.int64)
    alpha8[r < 1.0] = 128
    chk = ((xx // 4 + yy // 3 + seed) % 2 == 0) & (r < 1.0)
    alpha8[chk] = 38
    ring = (r >= 1.0) & (r < 1.25)
    alpha8[ring] = 64
    alpha8[:3, :] = 0
    alpha8[-3:, :] = 0
    alpha8[:, :3] = 0
    alpha8[:, -3:] = 0
    alphaC = (alpha8[0::2, 0::2] + alpha8[1::2, 0::2] + alpha8[0::2, 1::2] + alpha8[1::2, 1::2]) // 8  # half strength
    aY = 1.0 / (1.0 - alpha8 / 256.0)
    bY = -(alpha8 / 256.0) * (L8 / 255.0) * aY
    aC = 1.0 / (1.0 - alphaC / 256.0)
    bC = -(alphaC / 256.0) * (128 / 255.0) * aC
    data = np.concatenate([aY.ravel(), bY.ravel(), aC.ravel(), bC.ravel(), aC.ravel(), bC.ravel()]).astype(np.float32)
    return {"w": w, "h": h, "alpha8": alpha8.astype(np.uint8), "alphaC": alphaC.astype(np.uint8), "L8": L8, "data": data}


def logo_fade256(n, period=200):
    """Logo visibility schedule (0..256) per frame index tensor n: off for the first quarter of each period,
    linear fade-in over period/20 frames, on, fade-out ending at 85 % of the period, off."""
    p = n % period
    ramp = max(1, period // 20)
    up = torch.clamp(((p - period // 4) * 256) // ramp, 0, 256)
    down = torch.clamp((((period * 17) // 20 - p) * 256) // ramp, 0, 256)
    return torch.minimum(up, down)


_TC_TOP = (0, 1, 1, 2, 3)
_TC_BOT = (0, 1, 2, 3, 3)


def _field_time(n, parity, mode):
    if mode == "telecine":   # 24p -> 60i 3:2 pulldown: fields At Ab | Bt Bb | Bt Cb | Ct Db | Dt Db
        m = n % 5
        tt = torch.zeros_like(n)
        tb = torch.zeros_like(n)
        for i in range(5):
            tt = torch.where(m == i, torch.full_like(n, _TC_TOP[i]), tt)
            tb = torch.where(m == i, torch.full_like(n, _TC_BOT[i]), tb)
        k = (n // 5) * 4 + torch.where(parity == 0, tt, tb)
        return k * 2
    return n * 2 + parity    # true interlaced: every field has its own sampling time


def _plane(n, H, W, plane, seed, mode, speed):
    """n: int64 tensor (N,1,1).  Returns int64 (N,H,W) pixel values before logo compositing."""
    dev = n.device
    y = torch.arange(H, device=dev, dtype=torch.int64).view(1, H, 1)
    x = torch.arange(W, device=dev, dtype=torch.int64).view(1, 1, W)
    noise = (_hash32(x, y, n, plane, seed) & 3) - 1          # -1..2: below the default combing thresholds
    if mode == "flat":
        g = 40 + (_hash32(n, n * 0 + 7, n * 0, 3, seed) % 160) if plane == 0 else 128 + ((_hash32(n, n * 0 + 9, n * 0, plane, seed) & 15) - 8)
        bad = (_hash32(n, n * 0 + 11, n * 0, 5, seed) % 10) < 3          # ~30 % of frames get a gradient -> fail thy
        v = g + ((_hash32(x, y, n, plane, seed) & 3) - 2)
        if plane == 0:
            v = v + torch.where(bad, x & 63, torch.zeros_like(x))      # sawtooth: any ROI >= 32 px wide fails thy
        return v
    par = y & 1
    t = _field_time(n, par, mode)                                        # (N,H,1)
    if plane == 0:
        tri = (3 * x + 5 * y) & 127                      # triangular ramp: continuous, so only real motion combs
        v = 64 + torch.where(tri < 64, tri, 127 - tri)
        bx = (speed * 4 * t) % (W + 128) - 128
        inbar = (x >= bx) & (x < bx + 128)
        v = torch.where(inbar, 180 + ((x - bx) & 15), v)
        ty0, ty1, tx0, tx1 = H // 3, (2 * H) // 3, W // 4, (3 * W) // 4
        intex = (y >= ty0) & (y < ty1) & (x >= tx0) & (x < tx1)
        tex = 48 + (_hash32((x - speed * t) >> 2, y >> 3, n * 0, 9, seed) & 127)     # 4x8-pixel blocks moving horizontally
        v = torch.where(intex, tex, v)
        v = v + noise
        return torch.clamp(v, 16, 235)
    v = 128 + noise
    ty0, ty1, tx0, tx1 = H // 3, (2 * H) // 3, W // 4, (3 * W) // 4
    intex = (y >= ty0) & (y < ty1) & (x >= tx0) & (x < tx1)
    tex = 112 + (_hash32((x - (speed * t) // 2) >> 2, y >> 2, n * 0, 9 + plane, seed) & 31)
    v = torch.where(intex, tex + noise, v)
    return torch.clamp(v, 16, 240)


def make_frames(n0, count, W, H, seed=0x5EED0001, device="cpu", mode="interlaced", logo=None, imgx=0, imgy=0,
                speed=2, logo_period=200, out=None):
    """Frames n0..n0+count-1 as a uint8 tensor (count, W*H*3/2) in packed YV12 order.

    mode: "interlaced" (every field its own time -> combing on motion), "telecine" (3:2 pulldown of a 24p source:
    2 of every 5 frames are combed), "flat" (flat grey + noise, for LogoScan accumulation).
    logo: dict from make_logo() composited at (imgx, imgy) with the logo_fade256 schedule."""
    dev = torch.device(device)
    n = torch.arange(n0, n0 + count, device=dev, dtype=torch.int64).view(count, 1, 1)
    planes = []
    for plane, (ph, pw) in enumerate(((H, W), (H // 2, W // 2), (H // 2, W // 2))):
        v = _plane(n, ph, pw, plane, seed, mode, speed)
        if logo is not None:
            if plane == 0:
                al = torch.from_numpy(logo["alpha8"].astype(np.int64)).to(dev)
                Lv, lx, ly = logo["L8"], imgx, imgy
            else:
                al = torch.from_numpy(logo["alphaC"].astype(np.int64)).to(dev)
                Lv, lx, ly = 128, imgx // 2, imgy // 2
            lh, lw = al.shape
            fade = logo_fade256(n, logo_period) if mode != "flat" else torch.where((_hash32(n, n * 0 + 13, n * 0, 6, seed) & 3) != 0, 256, 0)
            a = (al.view(1, lh, lw) * fade) >> 8
            roi = v[:, ly:ly + lh, lx:lx + lw]
            v[:, ly:ly + lh, lx:lx + lw] = (roi * (256 - a) + a * Lv + 128) >> 8
        planes.append(v.to(torch.uint8).reshape(count, -1))
    res = torch.cat(planes, dim=1)
    if out is not None:
        out.copy_(res)
        return out
    return res


def noisy_clip(seed, count, W, H, bits=8, n0=0):
    """Frames n0..n0+count-1 of a seeded noisy 4:2:0 clip for the temporal noise reduction: numpy (count, W*H*3/2) of
    uint8 (bits 8) or uint16, packed Y, U, V.  A smooth picture plus per-frame noise of +-(3 << (bits-8)), so thresholds of
    a few steps split each window; about one frame in six jumps away (a cut), and a block of samples sits at the maximum.
    Integer-only numpy, identical on every platform."""
    maxv = (1 << bits) - 1
    s = bits - 8
    n = np.arange(n0, n0 + count, dtype=np.int64).reshape(count, 1, 1)
    cut = (_hash32(n, n * 0 + 3, n * 0, 7, seed) % 6) == 0
    planes = []
    for plane, (ph, pw) in enumerate(((H, W), (H // 2, W // 2), (H // 2, W // 2))):
        y = np.arange(ph, dtype=np.int64).reshape(1, ph, 1)
        x = np.arange(pw, dtype=np.int64).reshape(1, 1, pw)
        base = ((60 + 5 * x + 3 * y + 40 * plane) % 160 + 40) << s
        amp = 3 << s
        v = base + (_hash32(x, y, n, plane, seed) % (2 * amp + 1)) - amp
        v = np.where(cut, v + (50 << s), v)
        v = np.where((x < max(1, pw // 4)) & (y < max(1, ph // 4)), maxv, v)
        planes.append(np.clip(v, 0, maxv).reshape(count, -1))
    return np.concatenate(planes, axis=1).astype(np.uint8 if bits == 8 else np.uint16)


def scan_frames16(seed, n, W, H, x, y, w, h, bits, thy, log_uvx=1, log_uvy=1):
    """n packed frames for LogoScan on 2-byte samples: numpy (n, W*H + 2*(W>>log_uvx)*(H>>log_uvy)) uint16 at `bits` bits,
    Y, U, V back to back.  Outside the scan rectangle (x, y, w, h): noise over the whole range.  Inside it, per frame and
    plane, the border takes values in [L, L + d] with both ends present: d is at most thy, exactly thy in about one frame
    of four, thy + 1 in one plane of about one frame of six; L is anywhere in [0, maxv - d] and sits at maxv - d (samples at
    maxv) in about one frame of eight.  The interior is the border's middle mean blended with a logo blob (colour maxv
    in Y, maxv / 4 in U, 3 maxv / 4 in V) in about three frames of four."""
    rng = np.random.default_rng(seed)
    maxv = (1 << bits) - 1
    W2, H2, w2, h2 = W >> log_uvx, H >> log_uvy, w >> log_uvx, h >> log_uvy
    ysz, csz = W * H, W2 * H2
    out = rng.integers(0, maxv + 1, (n, ysz + 2 * csz), dtype=np.int64)
    d = rng.integers(0, max(thy, 0) + 1, (n, 3))
    d[rng.random((n, 3)) < 0.25] = thy
    bad = rng.random(n) < 0.17
    d[bad, rng.integers(0, 3, int(bad.sum()))] = thy + 1
    d = np.clip(d, 0, maxv)
    top = rng.random((n, 3)) < 0.125
    on = rng.random(n) < 0.75
    planes = [(w, h, x, y, W, H, 0, maxv), (w2, h2, x >> log_uvx, y >> log_uvy, W2, H2, ysz, maxv // 4),
              (w2, h2, x >> log_uvx, y >> log_uvy, W2, H2, ysz + csz, 3 * maxv // 4)]
    for p, (pw, ph, px, py, PW, PH, off, color) in enumerate(planes):
        yy, xx = np.mgrid[0:ph, 0:pw]
        r = np.hypot((xx - (pw - 1) / 2) / max(pw / 2, 1), (yy - (ph - 1) / 2) / max(ph / 2, 1))
        alpha = np.clip(1.2 - 1.5 * r, 0, 0.8)
        ys = np.concatenate([np.zeros(pw, int), np.full(pw, ph - 1), np.repeat(np.arange(1, ph - 1), 2)])
        xs = np.concatenate([np.arange(pw), np.arange(pw), np.tile([0, pw - 1], max(0, ph - 2))])
        nb = len(ys)
        for i in range(n):
            dp = int(d[i, p])
            lo = maxv - dp if top[i, p] else int(rng.integers(0, maxv - dp + 1))
            s = rng.integers(lo, lo + dp + 1, nb)
            s[0], s[-1] = lo, lo + dp
            bg = float(np.sort(s)[nb // 4:nb - nb // 4].mean())
            inner = np.full((ph, pw), bg)
            if on[i]:
                inner = inner * (1 - alpha) + alpha * color
            plane = out[i, off:off + PW * PH].reshape(PH, PW)[py:py + ph, px:px + pw]
            plane[:] = np.clip(np.rint(inner), 0, maxv)
            plane[ys, xs] = rng.permutation(s)
    return out.astype(np.uint16)


def scan_rects(frames, W, H, x, y, w, h, log_uvx=1, log_uvy=1):
    """Packed frames (as scan_frames16 makes them) -> the Y, U, V scan rectangles, numpy (n, rows, cols) views each."""
    n = frames.shape[0]
    W2, H2 = W >> log_uvx, H >> log_uvy
    ysz, csz = W * H, W2 * H2
    cx, cy, cw, ch = x >> log_uvx, y >> log_uvy, w >> log_uvx, h >> log_uvy
    Y = frames[:, :ysz].reshape(n, H, W)[:, y:y + h, x:x + w]
    U = frames[:, ysz:ysz + csz].reshape(n, H2, W2)[:, cy:cy + ch, cx:cx + cw]
    V = frames[:, ysz + csz:ysz + 2 * csz].reshape(n, H2, W2)[:, cy:cy + ch, cx:cx + cw]
    return Y, U, V


def split_planes(frames, W, H):
    """(N, W*H*3/2) uint8 tensor/array -> (Y (N,H,W), U (N,H/2,W/2), V) numpy views."""
    a = frames.cpu().numpy() if isinstance(frames, torch.Tensor) else frames
    n = a.shape[0]
    ysz, csz = W * H, (W // 2) * (H // 2)
    Y = a[:, :ysz].reshape(n, H, W)
    U = a[:, ysz:ysz + csz].reshape(n, H // 2, W // 2)
    V = a[:, ysz + csz:].reshape(n, H // 2, W // 2)
    return Y, U, V
