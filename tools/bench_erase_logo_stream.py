"""Erase logo stream (amtk_erase_logo_stream) vs the per-frame path, on pinned 1080p YV12 frames.

The per-frame path is what the host mirror's logo::AMTEraseLogo runs on a child that is not device resident: per output
frame, CalcFade2 fetches up to three analyze frames, each made of 8 one-frame amtk_logo_analyze_frames calls (there is no
frame cache), then one amtk_erase_logo_frames call on the frame.  The stream sends every frame once and receives each
output once.

    python tools/bench_erase_logo_stream.py [--frames 600] [--baseline-frames 96]

Prints one JSON line: frames/s of each case, H2D / D2H payload bytes per frame, frames analysed, the card's name, power
limit and SM clock.  Sampled outputs are checked against the C oracle's CalcFade2 and the per-frame path's pixels.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import amatsukaze_b200 as ab  # noqa: E402
from amatsukaze_b200 import synth  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

W, H = 1920, 1080
FSZ = W * H * 3 // 2


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smmax = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smmax}
    except Exception as e:           # the measurement still stands; say what is missing
        return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": "unavailable (%s)" % type(e).__name__}


def frame_desc(buf, i):
    d = ab.yv12_clip(buf, W, H, 1, False)
    d.base = buf.data_ptr() + (i % buf.shape[0]) * FSZ
    return d


def table(N, every, maxfade):
    """frame_result with a logo section change every `every` frames (0 = no table)."""
    if not every:
        return None
    fr = np.zeros(N, np.uint8)
    for k, s in enumerate(range(0, N, every)):
        fr[s:s + every] = 2 if k % 2 else 0
    return fr


def run_stream(ctx, logo, frames, N, fr, maxfade, B, keep=()):
    """Returns (seconds, counts, {n: (output rect bytes, fades)} for n in keep)."""
    dst = torch.empty(FSZ, dtype=torch.uint8).pin_memory()
    kept = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s = ctx.erase_logo_stream(logo, N, fr, maxfade, B)
    got, held = 0, -1
    for i in range(N):
        s.send(frame_desc(frames, i))
        while True:
            if held != got:                                 # dst holds source frame n's pixels (MakeWritable's copy)
                dst.copy_(frames[got % frames.shape[0]])
                held = got
            d = ab.yv12_clip(dst, W, H, 1, False)
            r = s.recv(d)
            if r is None:
                break
            if r[0] in keep:
                kept[r[0]] = (dst.numpy().copy(), r[1])
            got += 1
    dt = time.perf_counter() - t0
    c = s.counts()
    s.close()
    assert got == N
    return dt, c, kept


def per_frame(ctx, logo, deint, ft, fb, frames, N, fr, maxfade, keep=()):
    """The mirror's per-frame AMTEraseLogo::GetFrame on a host child: CalcFade(2) with analyze frames rebuilt from 8
    one-frame analyze calls each, then one erase call."""
    dst = torch.empty(FSZ, dtype=torch.uint8).pin_memory()
    rec = np.zeros((8, 33), np.float32)
    kept = {}
    half = maxfade >> 1
    t0 = time.perf_counter()
    for n in range(N):
        uniform = fr is not None and all(fr[max(0, min(N - 1, n + i))] == fr[max(0, min(N - 1, n - half))] for i in range(-half, half + 1))
        if uniform:
            fades = (1.0, 1.0) if fr[n] == 2 else (0.0, 0.0)
        else:
            rec9 = np.zeros((9, 33), np.float32)
            held = -1
            for i in range(-4, 5):
                src = ab.lib().amtk_calc_fade2_index(N, N, n, i)
                if src >> 3 != held:
                    held = src >> 3
                    for j in range(8):
                        k = min(N - 1, held * 8 + j)
                        ctx.analyze_frames(frame_desc(frames, k), deint, ft, fb, out=rec[j:j + 1])
                rec9[i + 4] = rec[src & 7]
            ft_, fb_ = C_fades(rec9)
            fades = (ft_, fb_)
        dst.copy_(frames[n % frames.shape[0]])
        ctx.erase_logo(ab.yv12_clip(dst, W, H, 1, False), logo, np.array([fades], np.float32))
        if n in keep:
            kept[n] = (dst.numpy().copy(), fades)
    return time.perf_counter() - t0, kept


def C_fades(rec9):
    import ctypes as C
    r = np.ascontiguousarray(rec9, np.float32)
    a, b = C.c_float(), C.c_float()
    ab.lib().amtk_calc_fade2_records(r.ctypes.data_as(C.POINTER(C.c_float)), C.byref(a), C.byref(b))
    return a.value, b.value


def oracle_fades(frames, olog, N, n):
    """The C oracle's AMTAnalyzeLogo records for the nine frames CalcFade2 reads, then its CalcFade2."""
    dl, ft, fb = olog
    rec = np.zeros((N, 33), np.float32)
    for i in range(-4, 5):
        k = ab.lib().amtk_calc_fade2_index(N, N, n, i)
        Y = frames[k % frames.shape[0]].numpy()[:W * H].reshape(H, W)
        rec[k] = po.or_analyze_frame(dl, ft, fb, Y, 255.0)
    return po.or_calc_fade2(rec, N, n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=600)
    ap.add_argument("--baseline-frames", type=int, default=96)
    ap.add_argument("--distinct", type=int, default=48, help="distinct source frames, cycled")
    ap.add_argument("--maxfade", type=int, default=16)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU: there is no CPU fallback"
    torch.cuda.set_device(0)
    ctx = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    po.oracle_lib()
    logos = {"64x64": (synth.make_logo(64, 64), 64, 64, 1600, 60), "192x96": (synth.make_logo(192, 96), 192, 96, 1680, 48)}
    res = {"metric": "erase_logo_stream", "width": W, "height": H, "frames": a.frames, "maxfade": a.maxfade, "cases": []}
    res.update(gpu_info())
    N = a.frames
    every = max(1, round((a.maxfade + 1) / 0.05))          # about 5 % of frames within maxfade/2 of a transition
    for lname, (lg, lw, lh, ix, iy) in logos.items():
        frames = synth.make_frames(0, a.distinct, W, H, seed=11, mode="interlaced", logo=lg, imgx=ix, imgy=iy,
                                   logo_period=40).pin_memory()
        logo = ab.Logo.create(lg["data"], lw, lh, W, H, ix, iy)
        deint, ft, fb = logo.deint().create_mask(0.35), logo.field(0).create_mask(0.35), logo.field(1).create_mask(0.35)
        olog = tuple(x.create_mask(0.35) for x in (lambda r: (r.deint(), r.field(0), r.field(1)))(
            po.OracleLogo.create(lg["data"], lw, lh, W, H, ix, iy)))
        for tname, fr in (("table5pct", table(N, every, a.maxfade)), ("no_table", None)):
            keep = (0, 1, N // 2, N - 1)
            run_stream(ctx, logo, frames, min(N, 64), None if fr is None else fr[:min(N, 64)], a.maxfade, 16)   # warm-up
            nb = min(N, a.baseline_frames if fr is None else 2 * every)     # the table case needs its transitions
            fr_b = table(nb, every, a.maxfade) if fr is not None else None
            tb, kb = per_frame(ctx, logo, deint, ft, fb, frames, nb, fr_b, a.maxfade, keep=(0, 1, nb - 1))
            # the stream over the same nb frames must give the per-frame path's pixels and fades
            _, _, ks = run_stream(ctx, logo, frames, nb, fr_b, a.maxfade, 16, keep=(0, 1, nb - 1))
            for n in kb:
                assert np.array_equal(ks[n][0], kb[n][0]) and tuple(np.float32(ks[n][1])) == tuple(np.float32(kb[n][1])), n
            case = {"logo": lname, "table": tname, "per_frame_fps": nb / tb, "per_frame_frames": nb, "stream": []}
            for B in (1, 4, 16, 64):
                dt, c, kept = run_stream(ctx, logo, frames, N, fr, a.maxfade, B, keep=keep)
                for n in keep:
                    if fr is None or not all(fr[max(0, min(N - 1, n + i))] == fr[max(0, min(N - 1, n - (a.maxfade >> 1)))]
                                             for i in range(-(a.maxfade >> 1), (a.maxfade >> 1) + 1)):
                        exp = oracle_fades(frames, olog, N, n)
                        assert tuple(np.float32(kept[n][1])) == tuple(np.float32(exp)), (lname, tname, B, n, kept[n][1], exp)
                case["stream"].append({"B": B, "fps": N / dt, "h2d_per_frame": c[3] / N, "d2h_per_frame": c[4] / N,
                                       "analysed": c[2]})
            res["cases"].append(case)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
