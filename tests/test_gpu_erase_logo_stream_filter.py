"""AMTEraseLogo of the host-side mirror over a child that is not device resident (tests/cpp/test_erase_logo_stream.cpp):
MakeSource's chain AMTEraseLogo(AMTAnalyzeLogo(src, logo), logo, logof, maxfade) pulled in order is served from the frame
stream, which asks the child for each frame once and never reads the analyze clip; reverse and random reads take the
per-frame path.  Every served frame must equal the reference composition (tests/test_gpu_erase_logo_stream.py)."""
import os
import struct
import subprocess

import numpy as np
import pytest

import amatsukaze_b200 as ab
from amatsukaze_b200 import _build
from test_gpu_erase_logo_stream import H, LOGO, LOGOF, W, Reference, make_clip, write_logof

pytestmark = pytest.mark.gpu

IMGX, IMGY = 100, 42
FSZ = W * H * 3 // 2


@pytest.fixture(scope="module")
def exe():
    return _build.build_erase_logo_stream_test() if os.path.exists("/usr/bin/g++") else _build.ERASE_LOGO_STREAM_TEST


def _drive(exe, *args):
    r = subprocess.run([exe, *map(str, args)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    return [l for l in r.stdout.splitlines() if l.startswith("order")]


def _stats(line):
    return {k: int(v) for k, v in (kv.split("=") for kv in line.split(": ", 1)[1].split())}


def _setup(tmp_path, N, logof_kind):
    frames = make_clip(N, 8, IMGX, IMGY, seed=5)
    raw = tmp_path / "clip.raw"
    with open(raw, "wb") as f:
        f.write(b"AMTSRAW1" + struct.pack("<6i", W, H, 8, N, 30000, 1001))
        f.write(frames.tobytes())
    lgd = str(tmp_path / "logo.lgd")
    ab.Logo.create(LOGO["data"], 64, 64, W, H, IMGX, IMGY).save(lgd)
    logof = write_logof(tmp_path / "logof.txt", LOGOF[logof_kind]) if logof_kind else "-"
    return frames, str(raw), lgd, logof


def _orders(tmp_path, orders):
    p = tmp_path / "orders.bin"
    np.array([x for o in orders for x in list(o) + [-1]], np.int32).tofile(p)
    return str(p)


@pytest.mark.parametrize("logof_kind,maxfade", [(None, 16), ("close", 16), ("middle", 31)])
def test_in_order_equals_reference_and_per_frame_path(exe, oracle, tmp_path, logof_kind, maxfade):
    N = 100
    frames, raw, lgd, logof = _setup(tmp_path, N, logof_kind)
    rng = np.random.default_rng(3)
    orders = {"in_order": list(range(N)), "in_order_twice": [n for n in range(N) for _ in range(2)],
              "reverse": list(range(N))[::-1], "random": [int(x) for x in rng.integers(0, N, 60)]}
    out = tmp_path / "out.bin"
    lines = _drive(exe, "order", raw, lgd, "-", logof, maxfade, _orders(tmp_path, orders.values()), out, 0)
    got = np.fromfile(out, np.uint8).reshape(-1, FSZ)
    ref = Reference(oracle, 8, IMGX, IMGY)
    fades, _ = ref.fades(ref.records(frames), N, None if logof == "-" else logof, maxfade)
    exp = ref.pixels(frames, fades)
    pos = 0
    for (name, order), line in zip(orders.items(), lines):
        st = _stats(line)
        assert np.array_equal(got[pos:pos + len(order)], exp[order]), name
        pos += len(order)
        if name.startswith("in_order"):
            assert (st["child_max"], st["child_total"], st["child_unasked"]) == (1, N, 0), line     # analyze clip never asked
            assert st["sent0"] == N and st["streams0"] == 1
        elif name == "reverse":                       # per frame until the last read (frame 0), which starts a stream
            assert st["streams0"] == 1 and st["child_max"] > 1, line


def test_chained_erasers_and_tnr_over_them(exe, oracle, tmp_path):
    """Two erasers (the logo and an extra erase logo) each run their own stream and in-order reads pass down the chain;
    KTemporalNR pulled over them still asks each source frame once."""
    N = 60
    frames, raw, lgd, logof = _setup(tmp_path, N, None)
    lgd2 = str(tmp_path / "logo2.lgd")
    ab.Logo.create(LOGO["data"], 64, 64, W, H, 16, 20).save(lgd2)
    orders = _orders(tmp_path, [list(range(N)), list(range(N))[::-1]])
    out = tmp_path / "out.bin"
    lines = _drive(exe, "order", raw, lgd, lgd2, "-", 16, orders, out, 0)
    st = _stats(lines[0])
    assert (st["child_max"], st["child_total"], st["sent0"], st["sent1"]) == (1, N, N, N), lines[0]
    got = np.fromfile(out, np.uint8).reshape(-1, FSZ)
    assert np.array_equal(got[:N], got[N:][::-1]), "stream and per-frame path differ"
    out2 = tmp_path / "out2.bin"
    lines = _drive(exe, "order", raw, lgd, lgd2, "-", 16, _orders(tmp_path, [list(range(N))]), out2, 1)
    st = _stats(lines[0])
    assert (st["child_max"], st["child_total"], st["sent0"], st["sent1"]) == (1, N, N, N), lines[0]
