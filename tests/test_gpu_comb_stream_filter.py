"""AMTCombAnalyze of the host-side mirror over a source that is not device resident (tests/cpp/test_comb_stream.cpp): it
feeds the frame stream, asks for each child frame once and in order under ReadAllFrames, and its combstat.txt -- and the
duration and timecode files KFMVfrScript / KFMCfrScript make from it under AMTFilterSource -- are byte-identical to those
of the same frames on a device-resident AMTSource."""
import os
import struct
import subprocess

import numpy as np
import pytest

import amatsukaze_b200 as ab
from amatsukaze_b200 import _build, synth
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

W, H = 256, 160
N = 150          # many batches of the mirror's 16 frames, the last one partial


@pytest.fixture(scope="module")
def exe():
    return _build.build_comb_stream_test() if os.path.exists("/usr/bin/g++") else _build.COMB_STREAM_TEST


def _frames(bits):
    fr = synth.make_frames(0, N, W, H, seed=0x5EED0500, mode="telecine").numpy()
    if bits == 10:
        low = np.random.default_rng(1).integers(0, 4, fr.shape)
        fr = ((fr.astype(np.int64) << 2) | low).astype(np.uint16)
    return fr


def _write_raw(path, fr, bits):
    with open(path, "wb") as f:
        f.write(b"AMTSRAW1" + struct.pack("<6i", W, H, bits, N, 30000, 1001))
        f.write(fr.tobytes())


@pytest.mark.parametrize("bits", [8, 10])
def test_cpu_source_equals_device_resident(exe, tmp_path, bits):
    fr = _frames(bits)
    raw = tmp_path / "clip.raw"
    _write_raw(raw, fr, bits)
    for kind in ("cpu", "dev"):
        (tmp_path / kind).mkdir()
    r = subprocess.run([exe, "filter", str(raw), str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = {l.split(":")[0]: l for l in r.stdout.splitlines() if ":" in l}
    assert "cpu: asked=%d child_max=1 child_unasked=0 in_order=1 frames_returned=%d" % (N, N) in lines["cpu"], lines["cpu"]
    c, d = (tmp_path / "cpu" / "combstat.txt").read_bytes(), (tmp_path / "dev" / "combstat.txt").read_bytes()
    assert c == d
    got = np.loadtxt(tmp_path / "cpu" / "combstat.txt", dtype=np.int64).astype(np.int32)
    assert got.shape == (N, 12) and (got != 0).any(axis=0).all()
    if bits == 8:                                  # the counters are the metric itself
        ysz, csz = W * H, (W // 2) * (H // 2)
        Y = fr[:, :ysz].reshape(-1, H, W)
        U = fr[:, ysz:ysz + csz].reshape(-1, H // 2, W // 2)
        V = fr[:, ysz + csz:].reshape(-1, H // 2, W // 2)
        assert np.array_equal(got, po.or_comb_clip(Y, U, V, ab.default_comb_params().as_list()))
    # Counts() after a partial pull, and after an out-of-order GetFrame: the pass is completed in order, the same rows
    for how, returned in (("partial", N // 3 - 1), ("seek", N // 2)):
        assert np.array_equal(np.fromfile(tmp_path / "cpu" / ("counts_%s.bin" % how), np.int32).reshape(N, 12), got), how
        line = lines[how]
        assert "child_max=%d" % (2 if how == "seek" else 1) in line and "child_unasked=0" in line, line
        assert line.rstrip().endswith("returned=%d" % returned), line


@pytest.mark.parametrize("script", ["vfr", "cfr"])
@pytest.mark.parametrize("bits", [8, 10])
def test_telecine_passes_on_a_cpu_source(exe, tmp_path, script, bits):
    fr = _frames(bits)
    files = {}
    for kind in ("cpu", "dev"):
        d = tmp_path / kind
        d.mkdir()
        _write_raw(d / "amts0.dat", fr, bits)
        r = subprocess.run([exe, "passes", str(d), script, kind], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        if kind == "cpu":
            assert "pass0: asked=%d child_max=1 child_unasked=0 in_order=1" % N in r.stdout, r.stdout
        files[kind] = {p.name: p.read_bytes() for p in d.glob("v0-0-0.avstmp*")}
    names = {"v0-0-0.avstmp.combstat.txt"} | ({"v0-0-0.avstmp.duration.txt", "v0-0-0.avstmp.timecode.txt"} if script == "vfr" else set())
    assert set(files["cpu"]) == set(files["dev"]) == names
    for name in names:
        assert files["cpu"][name] == files["dev"][name], name
