"""logo::LogoFrame and CMAnalyze of the host-side mirror over a source that is not device resident
(tests/cpp/test_logo_scan_stream.cpp): scanFrames feeds the frame stream, asks for each frame once and in order, and its
results, the logoframe file writeResult makes and what CMAnalyze picks and writes are byte-identical to those of the same
frames on a device-resident AMTSource."""
import os
import struct
import subprocess

import numpy as np
import pytest

import amatsukaze_b200 as ab
from amatsukaze_b200 import _build, synth
from test_gpu_erase_logo_stream import H, W

pytestmark = pytest.mark.gpu

N = 150          # more than two batches of the mirror's 64 frames, the last one partial


@pytest.fixture(scope="module")
def exe():
    return _build.build_logo_scan_stream_test() if os.path.exists("/usr/bin/g++") else _build.LOGO_SCAN_STREAM_TEST


def _setup(tmp_path, bits):
    """A clip where logo 1 shows in sections and logo 2 never does; both logos lie in the upper half, so the byte-pitch
    row step of 10-bit frames keeps them inside the plane.  Logo 3 is made for 1920x1080 and is too large for the
    evaluation plan: it gives (0, -1) on these frames on both branches, without being checked."""
    lg = synth.make_logo(64, 64, seed=3)
    fr = synth.make_frames(0, N, W, H, seed=0x5EED0300, logo=lg, imgx=37, imgy=5, logo_period=60).numpy()
    if bits == 10:
        low = np.random.default_rng(1).integers(0, 4, fr.shape)
        fr = ((fr.astype(np.int64) << 2) | low).astype(np.uint16)
    raw = tmp_path / "clip.raw"
    with open(raw, "wb") as f:
        f.write(b"AMTSRAW1" + struct.pack("<6i", W, H, bits, N, 30000, 1001))
        f.write(fr.tobytes())
    l1, l2, l3 = str(tmp_path / "logo1.lgd"), str(tmp_path / "logo2.lgd"), str(tmp_path / "logo3.lgd")
    ab.Logo.create(lg["data"], 64, 64, W, H, 37, 5).save(l1)
    ab.Logo.create(synth.make_logo(48, 40, seed=5)["data"], 48, 40, W, H, 181, 9).save(l2)
    ab.Logo.create(synth.make_logo(256, 128, seed=9)["data"], 256, 128, 1920, 1080, 100, 100).save(l3)
    for kind in ("cpu", "dev"):
        (tmp_path / kind).mkdir()
    return str(raw), l1, l2, l3


@pytest.mark.parametrize("bits", [8, 10])
def test_cpu_source_equals_device_resident(exe, tmp_path, bits):
    raw, l1, l2, l3 = _setup(tmp_path, bits)
    r = subprocess.run([exe, raw, l1, l2, l3, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = {l.split(":")[0]: l for l in r.stdout.splitlines() if ":" in l}
    cpu = dict(kv.split("=") for kv in lines["cpu"].split(": ", 1)[1].split())
    assert (cpu["asked"], cpu["child_max"], cpu["child_unasked"], cpu["in_order"]) == (str(N), "1", "0", "1"), lines["cpu"]
    assert lines["cpu"].split(" asked")[0].split(": ")[1] == lines["dev"].split(": ")[1]          # best logo and ratio
    c, d = tmp_path / "cpu", tmp_path / "dev"
    ev = np.fromfile(c / "eval.bin", np.float32).reshape(N, 4, 2)
    assert (c / "eval.bin").read_bytes() == (d / "eval.bin").read_bytes()
    assert np.all(ev[:, 1] == np.array([0.0, -1.0], np.float32))              # the unreadable logo
    assert np.all(ev[:, 3] == np.array([0.0, -1.0], np.float32))              # the logo of another frame size
    if bits == 8:              # (at 10 bits the byte-pitch row step reads every other row: the logo does not match there)
        assert ev[:, 0, 0].max() > 0.5 and ev[:, 0, 0].min() < 0.2
    assert (c / "logof.txt").read_bytes() == (d / "logof.txt").read_bytes()
    cm_cpu, cm_dev = lines["cpu cmanalyze"], lines["dev cmanalyze"]
    assert cm_cpu.split(": ", 1)[1].split(" asked")[0] == cm_dev.split(": ", 1)[1]               # logo path and ratio
    assert cm_cpu.rstrip().endswith("asked=%d child_max=1" % N), cm_cpu
    for name in ("logof0.txt", "logof0-0.txt", "logof0-1.txt"):
        assert (c / name).read_bytes() == (d / name).read_bytes(), name
