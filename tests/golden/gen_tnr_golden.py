"""Regenerate tests/golden/tnr_golden.json from the reference's own TemporalNRFilter (oracle/_ref/libamtk_ref_tnr.so,
built by oracle/build_ref_tnr.sh where the reference tree is present).

    python tests/golden/gen_tnr_golden.py

Each case runs the reference on a seeded synth.noisy_clip and records, for the filter's own onFrame/finish queue, the
frameIndex_ values it emits and a sha256 of the emitted frames; and a sha256 of TNRFilter over the window clamped at the
clip's ends for every frame (the library's definition).  Only hashes of outputs are stored, no reference source.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from amatsukaze_b200 import synth  # noqa: E402
from oracle import pytnr as pt  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tnr_golden.json")
W, H = 12, 8          # not a multiple of 16; H % 4 == 0 so both interlace modes apply


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def clamped_windows(N, d):
    return [[min(max(n - d + i, 0), N - 1) for i in range(2 * d + 1)] for n in range(N)]


def cases():
    out = []
    for bits in (8, 10, 12, 14, 16):                      # the threshold / interlace matrix at N = 2d+2
        for d in (0, 1, 3, 7, 63):
            for t in (0, 1, 4, 65535):
                for il in (0, 1):
                    out.append((bits, d, t, il, 2 * d + 2))
    for bits in (8, 16):                                  # short clips: N from 1 to 2d+2
        for il in (0, 1):
            for d in (0, 1, 3, 7):
                for N in range(1, 2 * d + 3):
                    out.append((bits, d, 4, il, N))
            for N in (1, 2, 63, 64, 65, 126, 127, 128):
                out.append((bits, 63, 4, il, N))
    return sorted(set(out))


def seed_of(bits, d, t, il, N):
    return (bits * 1000003 + d * 10007 + (t & 0xFFFF) * 31 + il * 7 + N) & 0x7FFFFFFF


def main():
    if not pt.build_ref():
        sys.exit("the reference TemporalNRFilter is not built (oracle/build_ref_tnr.sh needs the reference tree)")
    rows = []
    for bits, d, t, il, N in cases():
        seed = seed_of(bits, d, t, il, N)
        fr = synth.noisy_clip(seed, N, W, H, bits)
        idx, seq = pt.ref_tnr_sequence(fr, W, H, bits, d, t, il)
        full = np.stack([pt.ref_tnr_frame([fr[i] for i in win], W, H, bits, t, il) for win in clamped_windows(N, d)])
        rows.append([bits, d, t, il, N, seed, idx.tolist(), sha(seq), sha(full)])
    doc = {"about": "reference TemporalNRFilter (VideoFilter.hpp:27-212) on synth.noisy_clip(seed, N, W, H, bits); "
                    "row = [bits, d, t, interlaced, N, seed, emitted frameIndex_, sha256[:16] of the emitted frames, "
                    "sha256[:16] of every frame over its clamped window]",
           "W": W, "H": H, "cases": rows}
    with open(OUT, "w") as f:
        json.dump(doc, f, separators=(",", ":"))
        f.write("\n")
    print("wrote %d cases to %s" % (len(rows), OUT))


if __name__ == "__main__":
    main()
