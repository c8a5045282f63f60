"""Generates tests/golden/logoscan16_golden.json by running the REFERENCE'S OWN LogoScan::AddFrame<uint16_t>, Normalize and
GetLogo (oracle/_ref/libamtk_ref.so, built from the reference sources by oracle/build_ref.sh) on seeded 2-byte frames
(amatsukaze_b200.synth.scan_frames16) at 10, 12 and 16 bits, and the ScanLogo composition at maxv
(oracle.pyscan16.compose_scan_logo) on them at 10 and 12 bits.  Run where oracle/_ref has been built:

    python tests/golden/gen_logoscan16_golden.py

Pinned per case: a digest of the input frames, AddFrame's verdict per frame, a digest of the accumulators (float64
bytes, plane-major Y, U, V, {sumF, sumB, sumF2, sumB2, sumFB} per pixel) and of GetLogo(false) / GetLogo(true) at
maxv = (1 << bits) - 1 (float32 bytes; null: "Insufficient logo frames")."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from amatsukaze_b200 import synth          # noqa: E402
from oracle import pyoracle as po          # noqa: E402
from oracle import pyscan16 as ps          # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "logoscan16_golden.json")

# name: (seed, frames, W, H, x, y, w, h, bits, thy, log_uvx, log_uvy)
SCAN_CASES = {
    "10bit-420-32x24": (101, 48, 64, 48, 10, 6, 32, 24, 10, 48, 1, 1),
    "12bit-422-30x20": (102, 48, 64, 40, 8, 4, 30, 20, 12, 192, 1, 0),
    "16bit-444-16x12": (103, 48, 40, 32, 6, 8, 16, 12, 16, 3072, 0, 0),
    "16bit-420-6x4": (104, 64, 32, 16, 12, 8, 6, 4, 16, 3072, 1, 1),
    "16bit-420-72x40-thy0": (105, 32, 96, 64, 12, 10, 72, 40, 16, 0, 1, 1),
}
# name: (scan case, max_frames)
PIPELINE_CASES = {"10bit-420-32x24": ("10bit-420-32x24", 40), "12bit-422-30x20": ("12bit-422-30x20", 100000)}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def case_frames(c):
    seed, n, W, H, x, y, w, h, bits, thy, lx, ly = c
    fr = synth.scan_frames16(seed, n, W, H, x, y, w, h, bits, thy, lx, ly)
    return fr, synth.scan_rects(fr, W, H, x, y, w, h, lx, ly)


def run_scan(scan_class, c):
    seed, n, W, H, x, y, w, h, bits, thy, lx, ly = c
    fr, (Y, U, V) = case_frames(c)
    sc = scan_class(w, h, thy, lx, ly)
    valid = [int(sc.add_frame_u16(Y[i], U[i], V[i])) for i in range(n)]
    logos = [sc.get_logo((1 << bits) - 1, clean) for clean in (False, True)]
    return {"frames": digest(fr), "valid": valid, "sums": digest(sc.sums()),
            "logo": [None if lg is None else digest(lg) for lg in logos],
            "negative_sums": bool((sc.sums() < 0).any()), "samples_from_32768": bool((fr >= 32768).any())}


def run_pipeline(scan_class, c, maxf):
    seed, n, W, H, x, y, w, h, bits, thy, lx, ly = c
    _, (Y, U, V) = case_frames(c)
    data, stored = ps.compose_scan_logo(Y, U, V, w, h, thy, maxf, (1 << bits) - 1, lx, ly, scan_class=scan_class)
    return {"stored": len(stored), "data": None if data is None else digest(data)}


def main():
    if not po.ref_available():
        sys.exit("gen_logoscan16_golden.py: oracle/_ref/libamtk_ref.so is missing (run oracle/build_ref.sh)")
    out = {"scan": {k: run_scan(ps.RefScan16, c) for k, c in SCAN_CASES.items()},
           "pipeline": {k: run_pipeline(ps.RefScan16, SCAN_CASES[s], m) for k, (s, m) in PIPELINE_CASES.items()}}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
