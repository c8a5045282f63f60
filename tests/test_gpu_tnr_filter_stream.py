"""KTemporalNR of the host-side mirror over a child that is not device resident (tests/cpp/test_tnr_filter_stream.cpp): in-order
reads are served from a frame stream that asks the child for each frame once, other reads from a gathered window, and
under the mirror's ConvertBits the stream widens the 8-bit frames itself.  Every served frame must equal the C port of
the reference's TemporalNRFilter over the whole clip and carry the properties of its own source frame."""
import os
import struct
import subprocess

import numpy as np
import pytest

from amatsukaze_b200 import synth, _build
from oracle import pytnr as pt

pytestmark = pytest.mark.gpu

W, H = 48, 16                          # H % 4 == 0: interlaced clips are accepted


@pytest.fixture(scope="module")
def exe():
    return _build.build_tnr_filter_stream_test() if os.path.exists("/usr/bin/g++") else _build.TNR_FILTER_STREAM_TEST


def _write_raw(path, frames, bits, w=W, h=H):
    with open(path, "wb") as f:
        f.write(b"AMTSRAW1" + struct.pack("<6i", w, h, bits, frames.shape[0], 30000, 1001))
        f.write(frames.tobytes())


def _drive(exe, *args):
    r = subprocess.run([exe, *map(str, args)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def _stats(line):
    return {k: int(v) for k, v in (kv.split("=") for kv in line.split(": ", 1)[1].split())}


def patterns(N):
    """name -> the frames read, in order."""
    rng = np.random.default_rng(1000 + N)
    ordered = list(range(N))
    h, q = N // 2, N // 4
    return {
        "in_order": ordered,
        "in_order_twice": [n for n in ordered for _ in range(2)],
        "seeks": list(range(0, h)) + list(range(min(N - 1, h + q), N)) + list(range(q, min(N, h + 2))),
        "reverse": ordered[::-1],
        "random": [int(x) for x in rng.integers(0, N, 2 * N)],
        "from_the_end": list(range(max(0, N - 3), N)),
    }


@pytest.mark.parametrize("source", ["8", "14", "8to14"])
@pytest.mark.parametrize("d", [0, 1, 3, 9])
@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("N", [1, 5, 17, 75])
def test_access_patterns(exe, tmp_path, source, d, il, N):
    sb = 14 if source == "14" else 8
    ob = 8 if source == "8" else 14
    t = 2
    frames = synth.noisy_clip(5150 + 7 * d + N + sb + il, N, W, H, sb)
    _write_raw(tmp_path / "src.dat", frames, sb)
    want = pt.or_tnr_clip(frames.astype(np.uint16) << (ob - sb) if ob != sb else frames, W, H, ob, d, t, il)
    pats = patterns(N)
    orders = np.concatenate([np.array(p + [-1], np.int32) for p in pats.values()])
    orders.tofile(tmp_path / "orders.bin")
    out = _drive(exe, "order", tmp_path / "src.dat", 14 if source == "8to14" else 0, d, t, il, tmp_path / "orders.bin",
                 tmp_path / "out.bin")
    lines = [l for l in out.splitlines() if l.startswith("order ")]
    assert len(lines) == len(pats)
    got = np.fromfile(tmp_path / "out.bin", np.uint8 if ob == 8 else np.uint16).reshape(-1, frames.shape[1])
    pos = 0
    for (name, order), line in zip(pats.items(), lines):
        s = _stats(line)
        served = got[pos:pos + len(order)]
        pos += len(order)
        assert np.array_equal(served, want[order]), name
        assert s["reads"] == len(order) and s["bits"] == ob and s["typed"] == len(order), (name, line)
        assert s["host_widened"] == 0, (name, line)          # a fused ConvertBits never widens on the host
        if name in ("in_order", "in_order_twice"):            # every child frame asked for exactly once
            assert s["sent"] == N and s["gathered"] == 0, (name, line)
            assert s["child_max"] == 1 and s["child_total"] == N and s["child_unasked"] == 0, (name, line)
        if name == "reverse" and N > 1:                       # no read follows the one before it: all gathered
            assert s["gathered"] == N and s["sent"] == 0, (name, line)
        if name == "from_the_end" and N > 3:                  # one gather, then a stream from max(0, N-2-d)
            assert s["gathered"] == 1 and s["sent"] == N - max(0, N - 2 - d), (name, line)
    assert pos == got.shape[0]


def test_convertbits_then_ktemporalnr_output_pass(exe, tmp_path):
    """The server's two lines as AMTFilterSource's output pass on a CPU source: the stream widens, uploading 8-bit bytes."""
    n, w, h = 17, 256, 128
    frames = synth.noisy_clip(4343, n, w, h, 8)
    _write_raw(tmp_path / "amts0.dat", frames, 8, w, h)
    out = _drive(exe, "pass", tmp_path, tmp_path / "out.bin")
    s = _stats(next(l for l in out.splitlines() if l.startswith("pass: ")))
    assert s["frames"] == n and s["bits"] == 14 and s["device_frames"] == 0 and s["typed"] == n
    assert s["host_widened"] == 0 and s["sent"] == n and s["gathered"] == 0
    assert s["child_max"] == 1 and s["child_total"] == n
    assert s["h2d_max"] == w * h * 3 // 2                     # one 8-bit frame per upload
    got = np.fromfile(tmp_path / "out.bin", np.uint16).reshape(n, -1)
    assert np.array_equal(got, pt.or_tnr_clip(frames.astype(np.uint16) << 6, w, h, 14, 3, 1, 0))


def test_filter_destroyed_mid_clip_returns_its_device_memory(exe, tmp_path):
    w, h = 1920, 1080
    _write_raw(tmp_path / "src.dat", synth.noisy_clip(3, 4, w, h, 8), 8, w, h)
    out = _drive(exe, "release", tmp_path / "src.dat")
    s = _stats(next(l for l in out.splitlines() if l.startswith("release: ")))
    assert s["live"] < s["free0"] - (100 << 20), out          # the stream held its ring and batches ...
    assert abs(s["free1"] - s["free0"]) <= 0.01 * s["free0"], out     # ... and 40 filters gave them back
