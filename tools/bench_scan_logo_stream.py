"""Logo generation fed one frame at a time (amtk_scan_logo_stream) on 1080p YV12 (or YUV420P10/P12) frames.

    python tools/bench_scan_logo_stream.py [--frames 20000] [--distinct 300] [--bits 8|10|12] [--out DIR] [--tiny]

Sources: pinned host frames, pageable host frames and device frames.  The host and device sources replay `--distinct`
seeded frames (tens of thousands of distinct 1080p frames do not fit in memory); 30 % of them carry a bright pixel on the
corner both scan rectangles share, which makes them invalid (the background rejects some of the others).  Rectangles 64x64 and 256x128, thy 12, max_frames
`--frames`.  For every (rectangle, source): send rate (frames/s over the sends up to `more == 0`, ending in a device
synchronise), H2D payload bytes per host frame, and `finish` time for the stored frames.  For comparison, amtk_scan_logo
on a device-resident clip of the first `--compare` frames of the same sequence, timed, with its file checked against the
stream's at the same max_frames.  The card's name, power limit and SM clock are read in the same run.  One JSON line on
stdout (and in DIR/bench_scan_logo_stream.json with --out).

--bits 10 or 12 widens the same frames to 2-byte samples (shifted left by bits - 8) and scales thy with them
(12 << (bits - 8)), so the same frames are valid at every depth; the samples per frame are the same, the bytes twice.

--tiny rehearses the whole script at 320x192 and a few hundred frames; without a GPU it stops where it needs one.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import amatsukaze_b200 as ab                     # noqa: E402
from amatsukaze_b200 import synth                # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"
    except Exception:            # noqa: BLE001 -- recorded as unknown
        return "unknown"


def make_frames(distinct, w, h, x0, y0, seed=0x5EED0100):
    """distinct packed YV12 frames (CPU, uint8) and their intended validity: flat noisy background, every frame with
    index % 10 in {3, 6, 9} gets a 255 pixel at (x0, y0), the corner shared by both scan rectangles."""
    gen = "cuda" if torch.cuda.is_available() else "cpu"
    fr = torch.cat([synth.make_frames(i, min(25, distinct - i), w, h, seed=seed, device=gen, mode="flat").cpu()
                    for i in range(0, distinct, 25)])
    bad = (np.arange(distinct) % 10) % 3 == 0
    bad[np.arange(distinct) % 10 == 0] = False
    fr[torch.from_numpy(bad), y0 * w + x0] = 255
    return fr, ~bad


def run_stream(ctx, src, n_distinct, w, h, rect, maxf, cap, thy):
    x0, y0, sw, sh = rect
    s = ctx.scan_logo_stream(x0, y0, sw, sh, thy, maxf)
    clips = [src(i) for i in range(n_distinct)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sent = 0
    while sent < cap:
        more = s.send(clips[sent % n_distinct], sent + 1, cap)
        sent += 1
        if not more:
            break
    ctx.synchronize()
    t1 = time.perf_counter()
    data, err = None, None
    with tempfile.TemporaryDirectory() as d:
        dst = os.path.join(d, "s.lgd")
        try:
            s.finish(dst, 1)
            data = open(dst, "rb").read()
        except ab.AmtkError as e:        # rectangles beyond the fade sweep's shared-memory plan (amtk_scan_logo alike)
            err = str(e)
        ctx.synchronize()
        t2 = time.perf_counter()
    nread, ngather, h2d = s.counts()
    s.close()
    return {"sent": sent, "nread": nread, "ngather": ngather, "send_fps": sent / (t1 - t0),
            "finish_s": t2 - t1 if err is None else None, "finish_error": err,
            "h2d_bytes": h2d, "h2d_per_frame": h2d / sent}, (data, err)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20000)
    ap.add_argument("--distinct", type=int, default=300)
    ap.add_argument("--compare", type=int, default=1500, help="frames of the resident clip amtk_scan_logo runs on")
    ap.add_argument("--bits", type=int, default=8, choices=(8, 10, 12))
    ap.add_argument("--out", default=None)
    ap.add_argument("--tiny", action="store_true")
    a = ap.parse_args()
    w, h = (320, 192) if a.tiny else (1920, 1080)
    if a.tiny:
        a.frames, a.distinct, a.compare = min(a.frames, 300), min(a.distinct, 20), min(a.compare, 120)
    x0, y0 = w - 320, 32
    rects = [(x0, y0, 64, 64), (x0, y0, 256, 128)]
    host, intended = make_frames(a.distinct, w, h, x0, y0)
    thy = 12 << (a.bits - 8)
    if a.bits > 8:          # int16 holds the widened samples (the library reads bytes; torch gathers int16 on the GPU)
        host = host.to(torch.int16) << (a.bits - 8)
    print("frames: %d distinct %dx%d, %.0f %% without the border pixel" % (a.distinct, w, h, 100 * intended.mean()), file=sys.stderr)
    if not torch.cuda.is_available():
        raise SystemExit("bench_scan_logo_stream: no CUDA device (timings need an H100; nothing is reported without one)")
    ctx = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    dev = host.to("cuda")
    pinned = host.pin_memory()
    page = host.numpy().copy()
    sources = {
        "pinned": lambda i: ab.yv12_clip(pinned[i:i + 1], w, h, 1, False, bits=a.bits),
        "pageable": lambda i: ab.yv12_clip(page[i:i + 1], w, h, 1, False, bits=a.bits),
        "device": lambda i: ab.yv12_clip(dev[i:i + 1], w, h, 1, True, bits=a.bits),
    }
    cap = 3 * a.frames + 1000
    res = {"card": card(), "frame": "%dx%d %s" % (w, h, "YV12" if a.bits == 8 else "YUV420P%d" % a.bits), "bits": a.bits,
           "thy": thy, "max_frames": a.frames, "distinct": a.distinct, "runs": []}
    for rect in rects:
        # warm-up of every shape the timed runs use
        run_stream(ctx, sources["device"], a.distinct, w, h, rect, min(a.frames, 400), cap, thy)
        for name, src in sources.items():
            r, _ = run_stream(ctx, src, a.distinct, w, h, rect, a.frames, cap, thy)
            r.update({"rect": "%dx%d" % rect[2:], "source": name})
            res["runs"].append(r)
            print(json.dumps(r), file=sys.stderr)
        # amtk_scan_logo on a resident clip of the first `compare` frames of the sequence, same max_frames for both
        nclip = a.compare
        clip_t = dev[torch.arange(nclip, device="cuda") % a.distinct].contiguous()
        maxc = int(nclip * 0.5)
        sr, sout = run_stream(ctx, sources["device"], a.distinct, w, h, rect, maxc, nclip, thy)
        wout = (None, None)
        with tempfile.TemporaryDirectory() as d:
            dst = os.path.join(d, "w.lgd")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            try:
                ctx.scan_logo(ab.yv12_clip(clip_t, w, h, nclip, True, bits=a.bits), dst, rect[0], rect[1], rect[2], rect[3], thy, maxc,
                              service_id=1)
                wout = (open(dst, "rb").read(), None)
            except ab.AmtkError as e:
                wout = (None, str(e))
            ctx.synchronize()
            t1 = time.perf_counter()
        del clip_t
        res["runs"].append({"rect": "%dx%d" % rect[2:], "source": "resident clip, amtk_scan_logo", "frames": nclip, "max_frames": maxc,
                            "scan_logo_s": t1 - t0 if wout[1] is None else None, "scan_logo_error": wout[1],
                            "stream_send_plus_finish_s": sr["sent"] / sr["send_fps"] + (sr["finish_s"] or 0.0),
                            "same_result": sout == wout})
        print(json.dumps(res["runs"][-1]), file=sys.stderr)
        if sout != wout:
            raise SystemExit("bench_scan_logo_stream: the stream's result differs from amtk_scan_logo's")
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_scan_logo_stream.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
