"""The logo finder's accumulation (amtk_logo_find_add_frames) on resident clips and on a pinned host clip:

  - yv12_1080p: 1800 device-resident 1080p YV12 frames (8-bit Y planes, the TMA kernel), one call;
  - p10_1080p: 900 device-resident 1080p YUV420P10 frames (2-byte Y planes), one call;
  - host_pinned: 480 1080p YV12 frames in pinned host memory, one call (only the Y rows cross PCIe).

    python tools/bench_logo_find.py [--reps 5]

Each case runs once to warm up and is then timed `reps` times with CUDA events on the context's stream; the best and
the median are reported.  Bandwidth is the Y-plane bytes the call must read over its time, next to the read-only
ceiling measured in the same run by amtk_probe_read_ms over as many bytes.  The sums of every case are checked against a
torch reduction of the same frames before timing.  Prints one JSON line with the card's name, power limit and SM clock.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import amatsukaze_b200 as ab  # noqa: E402

W, H = 1920, 1080


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smmax = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smmax}
    except Exception as e:           # the measurement still stands; say what is missing
        return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": "unavailable (%s)" % type(e).__name__}


def frames(n, bits, device):
    """n packed 4:2:0 frames of random samples at `bits` bits: uint8 (bytes per frame) of the given device."""
    g = torch.Generator(device=device).manual_seed(bits)
    ysz, csz = W * H, (W // 2) * (H // 2)
    if bits == 8:
        return torch.randint(0, 256, (n, ysz + 2 * csz), dtype=torch.uint8, device=device, generator=g)
    v = torch.randint(0, 1 << bits, (n, ysz + 2 * csz), dtype=torch.int16, device=device, generator=g)
    return v.view(torch.uint8).view(n, -1)


def check_sums(fd, fr, n, bits):
    """The finder's sums against a torch reduction (int64) of the Y planes, on the device."""
    s1, s2, got = fd.sums()
    assert got == n
    bps = 1 if bits == 8 else 2
    w1 = torch.zeros(H * W, dtype=torch.int64, device="cuda")
    w2 = torch.zeros(H * W, dtype=torch.int64, device="cuda")
    for i in range(0, n, 100):
        blk = fr[i:i + 100, :W * H * bps]
        if fr.device.type != "cuda":
            blk = blk.cuda()
        y = (blk if bps == 1 else blk.contiguous().view(torch.int16)).to(torch.int64)
        if bps == 2:
            y = y & 0xFFFF
        w1 += y.sum(0)
        w2 += (y * y).sum(0)
    assert np.array_equal(s1.astype(np.int64).ravel(), w1.cpu().numpy()), "s1 differs"
    assert np.array_equal(s2.view(np.int64).ravel(), w2.cpu().numpy()), "s2 differs"


def case(ctx, name, fr, n, bits, on_device, reps):
    clip = ab.yv12_clip(fr, W, H, n, on_device, bits)
    fd = ctx.logo_find()
    fd.add_frames(clip)
    check_sums(fd, fr, n, bits)
    st = torch.cuda.current_stream()
    ms = []
    for _ in range(reps):
        fd = ctx.logo_find()
        fd.add_frames(clip, 0, 1)                 # allocates the sums outside the timed window
        ctx.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        launches = ctx.launches
        a.record(st)
        fd.add_frames(clip, 1, n - 1)
        b.record(st)
        b.synchronize()
        ms.append(a.elapsed_time(b))
        launches = ctx.launches - launches
    ybytes = (n - 1) * W * H * (1 if bits == 8 else 2)
    best, med = min(ms), float(np.median(ms))
    out = {"frames": n - 1, "ms_best": round(best, 3), "ms_median": round(med, 3),
           "frames_per_s": round((n - 1) / (best * 1e-3), 1), "y_bytes_per_ms": round(ybytes / best),
           "launches": launches}
    if on_device:
        probe = C.c_double()
        ab.capi.check(ctx.L.amtk_probe_read_ms(ctx.h, C.c_void_p(fr.data_ptr()), ybytes - ybytes % 16, reps, C.byref(probe)))
        out["probe_read_bytes_per_ms"] = round((ybytes - ybytes % 16) / probe.value)
        out["share_of_probe"] = round(out["y_bytes_per_ms"] / out["probe_read_bytes_per_ms"], 3)
    else:
        out["h2d_bytes"] = ctx.last_h2d_bytes
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    ctx = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    res = {"bench": "logo_find", **gpu_info()}
    fr = frames(1800, 8, "cuda")
    res["yv12_1080p"] = case(ctx, "yv12_1080p", fr, 1800, 8, True, args.reps)
    del fr
    torch.cuda.empty_cache()
    fr = frames(900, 10, "cuda")
    res["p10_1080p"] = case(ctx, "p10_1080p", fr, 900, 10, True, args.reps)
    del fr
    torch.cuda.empty_cache()
    host = frames(480, 8, "cuda").cpu().pin_memory()
    res["host_pinned_1080p"] = case(ctx, "host_pinned", host, 480, 8, False, max(2, args.reps // 2))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
