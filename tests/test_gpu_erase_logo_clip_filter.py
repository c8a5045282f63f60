"""AMTEraseLogo of the host-side mirror over a device-resident AMTSource (tests/cpp/test_erase_logo_clip.cpp): MakeSource's
chain is served from one amtk_erase_logo_clip call into the filter's own HBM clip.  Its frames and fades must equal the
per-frame path's and the frame stream's over a CPU source, leave the source untouched, and equal the reference
composition; EraseInPlace gives the same pixels over its own chain and over the per-frame composition; KTemporalNR over
the eraser runs its resident path with the output of the host path."""
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


@pytest.fixture(scope="module")
def exe():
    return _build.build_erase_logo_clip_test() if os.path.exists("/usr/bin/g++") else _build.ERASE_LOGO_CLIP_TEST


@pytest.mark.parametrize("logof_kind,maxfade", [(None, 16), ("close", 16), ("middle", 31)])
def test_resident_chain(exe, oracle, tmp_path, logof_kind, maxfade):
    N = 100
    frames = make_clip(N, 8, IMGX, IMGY, seed=5)
    raw = tmp_path / "clip.raw"
    with open(raw, "wb") as f:
        f.write(b"AMTSRAW1" + struct.pack("<6i", W, H, 8, N, 30000, 1001))
        f.write(frames.tobytes())
    lgd = str(tmp_path / "logo.lgd")
    ab.Logo.create(LOGO["data"], 64, 64, W, H, IMGX, IMGY).save(lgd)
    logof = write_logof(tmp_path / "logof.txt", LOGOF[logof_kind]) if logof_kind else "-"
    r = subprocess.run([exe, str(raw), lgd, logof, str(maxfade), str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "erase_clip: frames=%d resident=1 per_frame_resident=0" % N in r.stdout, r.stdout
    assert "device_frames=%d" % N in r.stdout, r.stdout
    assert ("identical: per_frame=1 stream=1 fades=1 source_untouched=1 in_place=1 in_place_per_frame=1 tnr=1 "
            "tnr_resident=1 device=1") in r.stdout, r.stdout
    launches = int(r.stdout.split("launches=")[1].split()[0])
    assert launches == 8                    # one analysis pass, the fade kernel and the copy-and-erase kernel
    got = np.fromfile(tmp_path / "resident.bin", np.uint8).reshape(N, -1)
    fades = np.fromfile(tmp_path / "fades.bin", np.float32).reshape(N, 2)
    ref = Reference(oracle, 8, IMGX, IMGY)
    rf, _ = ref.fades(ref.records(frames), N, None if logof == "-" else logof, maxfade)
    assert np.array_equal(fades.view(np.uint32), rf.view(np.uint32))
    assert np.array_equal(got, ref.pixels(frames, rf))
