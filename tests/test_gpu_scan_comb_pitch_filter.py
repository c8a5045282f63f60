"""CMAnalyze of the host-side mirror with its combing-stats path at every depth (tests/cpp/test_scan_comb_pitch.cpp): over a
YUV420P10 (and a YV12) source that is not device resident it asks for each frame once and in order and creates exactly
one stream, the fused stream with ScanFrame's byte-pitch row step; over the device-resident AMTSource of the same frames
it makes exactly one amtk_scan_comb_frames_pitch call.  Both write logoframe files byte-identical to those CMAnalyze
writes without the stats path (LogoFrame::scanFrames(clip, env), which this change leaves as it was), and a stats file
byte-identical to AMTCombAnalyze's over the same source."""
import os
import struct
import subprocess

import numpy as np
import pytest

import amatsukaze_b200 as ab
from amatsukaze_b200 import _build, synth

pytestmark = pytest.mark.gpu

W, H = 256, 160
N = 150          # many batches of the fused stream's 16 frames, the last one partial
STREAMS = ("amtk_scan_comb_stream_create", "amtk_scan_comb_stream_create_pitch", "amtk_logo_scan_stream_create",
           "amtk_comb_stream_create")
CLIP_CALLS = ("amtk_scan_comb_frames", "amtk_scan_comb_frames_pitch", "amtk_logo_scan_frames", "amtk_comb_frames")


@pytest.fixture(scope="module")
def exe():
    return _build.build_scan_comb_pitch_test() if os.path.exists("/usr/bin/g++") else _build.SCAN_COMB_PITCH_TEST


def _setup(tmp_path, bits):
    """3:2 pulldown frames where logo 1 shows in sections (inside the rows the byte-pitch step reads) and logo 2 never
    does; logo 3 (erased) is made for 1920x1080."""
    lg = synth.make_logo(64, 64, seed=3)
    fr = synth.make_frames(0, N, W, H, seed=0x5EED0800, mode="telecine", logo=lg, imgx=37, imgy=5, logo_period=60).numpy()
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
        for how in ("plain", "fused"):
            (tmp_path / kind / how).mkdir(parents=True)
    return str(raw), l1, l2, l3


def _calls(line):
    """The counted entry points a run called: {name: count}."""
    field = line.split(" calls=", 1)[1]
    return {k: int(v) for k, v in (kv.split("=") for kv in field.split(",") if kv)}


@pytest.mark.parametrize("bits", [10, 8])
def test_one_path_at_every_depth(exe, tmp_path, bits):
    raw, l1, l2, l3 = _setup(tmp_path, bits)
    r = subprocess.run([exe, raw, l1, l2, l3, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = {l.split(":")[0]: l.split(": ", 1)[1] for l in r.stdout.splitlines() if ":" in l}
    for kind in ("cpu", "dev"):
        plain, fused = lines[kind + " plain"], lines[kind + " fused"]
        assert plain.split(" asked")[0].split(" calls=")[0] == fused.split(" asked")[0].split(" calls=")[0], (plain, fused)
        calls = _calls(fused)
        if kind == "cpu":
            assert " asked=%d child_max=1 child_unasked=0 in_order=1 " % N in fused, fused
            assert sum(calls.get(f, 0) for f in STREAMS) == 1 and calls.get("amtk_scan_comb_stream_create_pitch") == 1, calls
            assert not any(calls.get(f) for f in CLIP_CALLS), calls
        else:
            assert not any(calls.get(f) for f in STREAMS), calls
            assert sum(calls.get(f, 0) for f in CLIP_CALLS) == 1 and calls.get("amtk_scan_comb_frames_pitch") == 1, calls
        d = tmp_path / kind
        names = sorted(p.name for p in (d / "plain").iterdir() if p.name.startswith("logof"))
        assert names == ["logof0-0.txt", "logof0.txt"], names
        for name in names:
            assert (d / "plain" / name).read_bytes() == (d / "fused" / name).read_bytes(), (kind, name)
        assert (d / "fused" / "combstat.txt").read_bytes() == (d / "combstat_ref.txt").read_bytes(), kind
    assert (tmp_path / "cpu" / "fused" / "combstat.txt").read_bytes() == (tmp_path / "dev" / "fused" / "combstat.txt").read_bytes()
    got = np.loadtxt(tmp_path / "cpu" / "fused" / "combstat.txt", dtype=np.int64)
    assert got.shape == (N, 12) and (got != 0).any(axis=0).all()
