"""What the logo evaluation adds to the fused step: comb-only, ScanFrame-only and fused calls on resident clips.

    python tools/bench_fused_step.py [--rounds 5] [--calls 10]

Two resident 1800-frame clips, 1920x1080 (logo 64x64 at (1700, 60), the bench.py headline) and 1440x1080 (logo at
(1300, 60)).  Rounds alternate amtk_comb_frames, amtk_logo_scan_frames and amtk_scan_comb_frames on each clip, each
timed with CUDA events over --calls back-to-back calls; the medians over the rounds are reported with the fused-minus-
comb-only cost, which is what the logo evaluation costs inside the fused step.  Prints one JSON line with the card name,
its power limit and the SM clock read after the timed rounds (numbers are only comparable at the same clock).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import amatsukaze_b200 as ab  # noqa: E402
from amatsukaze_b200 import synth  # noqa: E402

FRAMES = 1800
CLIPS = {"1920x1080": (1920, 1080, 1700, 60), "1440x1080": (1440, 1080, 1300, 60)}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim, sm, smax = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock": sm, "sm_clock_max": smax}
    except Exception as e:      # the timing stands without it
        return {"name": torch.cuda.get_device_name(0), "nvidia_smi": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100: there is no CPU fallback"
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    ctx = ab.Context(0, stream.cuda_stream)
    prm = ab.default_comb_params()
    lg = synth.make_logo(64, 64)
    res = {}
    for name, (W, H, imgx, imgy) in CLIPS.items():
        fs = W * H * 3 // 2
        buf = torch.empty((FRAMES, fs), dtype=torch.uint8, device="cuda")
        for n0 in range(0, FRAMES, 20):
            n = min(20, FRAMES - n0)
            synth.make_frames(n0, n, W, H, seed=7, device="cuda", mode="interlaced", logo=lg, imgx=imgx, imgy=imgy, out=buf[n0:n0 + n])
        torch.cuda.synchronize()
        clip = ab.yv12_clip(buf, W, H, FRAMES, True)
        logo = ab.Logo.create(lg["data"], 64, 64, W, H, imgx, imgy).deint().create_mask(0.35)
        scores = torch.empty((FRAMES, 1, 2), dtype=torch.float32, device="cuda")
        counts = torch.empty((FRAMES, 12), dtype=torch.int32, device="cuda")
        calls = {
            "comb_frames": lambda: ctx.comb_frames(clip, prm, out=counts),
            "scan_frames": lambda: ctx.scan_frames(clip, [logo], out=scores),
            "scan_comb_frames": lambda: ctx.scan_comb_frames(clip, [logo], prm, scores=scores, counts=counts),
        }
        ms = {k: [] for k in calls}
        with torch.cuda.stream(stream):
            for fn in calls.values():                      # warm-up: plans, tables, shared-memory attributes
                fn(); fn()
            stream.synchronize()
            for _ in range(args.rounds):
                for k, fn in calls.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    for _ in range(args.calls):
                        fn()
                    e1.record(stream)
                    e1.synchronize()
                    ms[k].append(e0.elapsed_time(e1) / args.calls)
        med = {k: float(np.median(v)) for k, v in ms.items()}
        res[name] = {"ms_per_call_median": med, "ms_per_call_all": ms,
                     "fused_minus_comb_ms": med["scan_comb_frames"] - med["comb_frames"],
                     "fused_frames_per_s": FRAMES / (med["scan_comb_frames"] * 1e-3)}
        del buf
    print(json.dumps({"tool": "bench_fused_step", "frames": FRAMES, "rounds": args.rounds, "calls_per_round": args.calls,
                      "gpu": gpu_info(), "results": res}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
