"""Whole-clip logo erase (amtk_erase_logo_clip) on 1800 resident 1080p YV12 frames, against the other ways to run the
eraser chain AMTEraseLogo(AMTAnalyzeLogo(src, logo), logo, logof, maxfade) on a clip already in HBM:

  - clip_in_place / clip_out_of_place: one amtk_erase_logo_clip call (dst = NULL / a second HBM clip);
  - per_frame: the mirror's previous composition, rebuilt from the C ABI: per output, the 8-frame amtk_logo_analyze_frames
    blocks CalcFade2 reads (AMTAnalyzeLogo::GetFrame, no frame cache), amtk_calc_fade2_records, and a one-frame
    amtk_erase_logo_frames;
  - stream: amtk_erase_logo_stream fed the device frames one at a time, each output received into its frame.

    python tools/bench_erase_logo_clip.py [--frames 1800] [--rounds 2]

The cases alternate within each round.  Every case's output clip and fades must be identical to clip_in_place's.  Times
are host clocks around work that ends in a device synchronise.  Prints one JSON line with frames/s per case and round,
the card's name, power limit and SM clock read in the same run.
"""
import argparse
import ctypes as C
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

W, H = 1920, 1080
FSZ = W * H * 3 // 2
IMGX, IMGY, LW, LH = 1600, 60, 64, 64


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smmax = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smmax}
    except Exception as e:           # the measurement still stands; say what is missing
        return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": "unavailable (%s)" % type(e).__name__}


def table(N, every):
    """frame_result with a logo section change every `every` frames."""
    fr = np.zeros(N, np.uint8)
    for k, s in enumerate(range(0, N, every)):
        fr[s:s + every] = 2 if k % 2 else 0
    return fr


def one(clip_t, n):
    d = ab.yv12_clip(clip_t, W, H, 1, True)
    d.base = clip_t.data_ptr() + n * FSZ
    return d


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def per_frame(ctx, src, work, logo, deint, ft, fb, N, fr, maxfade):
    L = ab.lib()
    fades = np.zeros((N, 2), np.float32)
    half = maxfade >> 1
    blk = torch.empty((8, 33), dtype=torch.float32).pin_memory().numpy()
    sclip = ab.yv12_clip(src, W, H, N, True)
    wclip = ab.yv12_clip(work, W, H, N, True)
    for n in range(N):
        if fr is not None and all(fr[max(0, min(N - 1, n + i))] == fr[max(0, min(N - 1, n - half))] for i in range(-half, half + 1)):
            fades[n] = 1.0 if fr[n] == 2 else 0.0
        else:
            rec9 = np.zeros((9, 33), np.float32)
            held = -1
            for i in range(-4, 5):
                k = L.amtk_calc_fade2_index(N, N, n, i)
                if k >> 3 != held:                         # AMTAnalyzeLogo::GetFrame(k >> 3): one 8-frame call
                    held = k >> 3
                    first, cnt = min(N - 1, held * 8), max(1, min(8, N - held * 8))
                    ctx.analyze_frames(sclip, deint, ft, fb, first, cnt, out=blk[:cnt])
                    blk[cnt:] = blk[cnt - 1]
                rec9[i + 4] = blk[k & 7]
            a, b = C.c_float(), C.c_float()
            L.amtk_calc_fade2_records(rec9.ctypes.data_as(C.POINTER(C.c_float)), C.byref(a), C.byref(b))
            fades[n] = (a.value, b.value)
        ctx.erase_logo(wclip, logo, fades[n:n + 1], n, 1)
    return fades


def stream(ctx, src, work, logo, N, fr, maxfade, B=16):
    s = ctx.erase_logo_stream(logo, N, fr, maxfade, B)
    fades = np.zeros((N, 2), np.float32)
    got = 0
    for i in range(N):
        s.send(one(src, i))
        while True:
            r = s.recv(one(work, got)) if got < N else None
            if r is None:
                break
            fades[r[0]] = r[1]
            got += 1
    s.close()
    assert got == N
    return fades


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1800)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--distinct", type=int, default=60, help="distinct source frames, cycled")
    ap.add_argument("--maxfade", type=int, default=16)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU: there is no CPU fallback"
    torch.cuda.set_device(0)
    ctx = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    N = a.frames
    lg = synth.make_logo(LW, LH)
    base = synth.make_frames(0, a.distinct, W, H, seed=11, mode="interlaced", logo=lg, imgx=IMGX, imgy=IMGY, logo_period=40)
    src = base.cuda().repeat((N + a.distinct - 1) // a.distinct, 1)[:N].contiguous()
    work, dst = torch.empty_like(src), torch.empty_like(src)
    logo = ab.Logo.create(lg["data"], LW, LH, W, H, IMGX, IMGY)
    deint, ft, fb = logo.deint().create_mask(0.35), logo.field(0).create_mask(0.35), logo.field(1).create_mask(0.35)
    sclip = ab.yv12_clip(src, W, H, N, True)
    res = {"metric": "erase_logo_clip", "width": W, "height": H, "frames": N, "logo": "%dx%d" % (LW, LH),
           "maxfade": a.maxfade, "cases": []}
    res.update(gpu_info())
    every = max(1, round((a.maxfade + 1) / 0.05))          # about 5 % of frames within maxfade/2 of a transition
    for tname, fr in (("no_table", None), ("table5pct", table(N, every))):
        # warm-up of every shape, then the reference output
        work.copy_(src)
        ref_fades = ctx.erase_logo_clip(ab.yv12_clip(work, W, H, N, True), logo, None, fr, a.maxfade)
        ref = work.clone()
        ctx.erase_logo_clip(sclip, logo, ab.yv12_clip(dst, W, H, N, True), fr, a.maxfade, 0, 64)
        case = {"table": tname, "rounds": []}
        for _ in range(a.rounds):
            rnd = {}
            work.copy_(src)
            t, f = timed(lambda: ctx.erase_logo_clip(ab.yv12_clip(work, W, H, N, True), logo, None, fr, a.maxfade))
            assert torch.equal(work, ref) and np.array_equal(f.view(np.uint32), ref_fades.view(np.uint32)), "clip_in_place"
            rnd["clip_in_place_fps"] = N / t
            dst.zero_()
            t, f = timed(lambda: ctx.erase_logo_clip(sclip, logo, ab.yv12_clip(dst, W, H, N, True), fr, a.maxfade))
            assert torch.equal(dst, ref) and np.array_equal(f.view(np.uint32), ref_fades.view(np.uint32)), "clip_out_of_place"
            rnd["clip_out_of_place_fps"] = N / t
            work.copy_(src)
            t, f = timed(lambda: per_frame(ctx, src, work, logo, deint, ft, fb, N, fr, a.maxfade))
            assert torch.equal(work, ref) and np.array_equal(f.view(np.uint32), ref_fades.view(np.uint32)), "per_frame"
            rnd["per_frame_fps"] = N / t
            work.copy_(src)
            t, f = timed(lambda: stream(ctx, src, work, logo, N, fr, a.maxfade))
            assert torch.equal(work, ref) and np.array_equal(f.view(np.uint32), ref_fades.view(np.uint32)), "stream"
            rnd["stream_device_frames_fps"] = N / t
            case["rounds"].append(rnd)
        case["identical"] = True
        res["cases"].append(case)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
