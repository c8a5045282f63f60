"""CPU tests of the 2-byte LogoScan checker: PyScan16 (oracle/pyscan16.py, the restatement of the reference's
LogoScan::AddFrame<uint16_t> used where oracle/_ref was not built) and the ScanLogo composition at maxv must reproduce the
golden vectors the reference's own code produced (tests/golden/logoscan16_golden.json, written by
tests/golden/gen_logoscan16_golden.py) at 10, 12 and 16 bits, including 16-bit borders with samples >= 32768, which the
reference's std::vector<short> wraps negative.  Where oracle/_ref was built the reference's own code is checked too."""
import json
import os
import sys

import numpy as np
import pytest

from oracle import pyoracle as po
from oracle import pyscan16 as ps

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import gen_logoscan16_golden as gen          # noqa: E402

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "logoscan16_golden.json")))


def scan_classes():
    return [ps.PyScan16] + ([ps.RefScan16] if po.ref_available() else [])


def test_golden_covers_every_depth_and_the_16_bit_wrap():
    bits = {c[8] for c in gen.SCAN_CASES.values()}
    assert bits == {10, 12, 16}
    assert {(c[10], c[11]) for c in gen.SCAN_CASES.values()} == {(1, 1), (1, 0), (0, 0)}
    for name, g in GOLD["scan"].items():
        assert 0 < sum(g["valid"]) < len(g["valid"]), name           # valid and rejected frames in every case
        assert all(lg is not None for lg in g["logo"]), name          # the fit is not degenerate
        wide = gen.SCAN_CASES[name][8] == 16
        assert g["samples_from_32768"] == wide and g["negative_sums"] == wide, name
    assert {gen.SCAN_CASES[s][8] for s, _ in gen.PIPELINE_CASES.values()} == {10, 12}


@pytest.mark.parametrize("name", list(gen.SCAN_CASES))
def test_scan_reproduces_golden(name):
    for cls in scan_classes():
        assert gen.run_scan(cls, gen.SCAN_CASES[name]) == GOLD["scan"][name], (cls.__name__, name)


@pytest.mark.parametrize("name", list(gen.PIPELINE_CASES))
def test_scan_logo_composition_reproduces_golden(name):
    scan, maxf = gen.PIPELINE_CASES[name]
    for cls in scan_classes():
        got = gen.run_pipeline(cls, gen.SCAN_CASES[scan], maxf)
        assert got == GOLD["pipeline"][name], (cls.__name__, name)
    assert GOLD["pipeline"][name]["data"] is not None


def test_pyscan16_takes_the_reference_int_arithmetic():
    """Two frames whose every sample is 50000 and 40000 at 16 bits: the border's short is 50000 - 65536, its middle mean
    -15535.5 truncates to -15535; f*f wraps to 32 bits; f*bg fits an int."""
    sc = ps.PyScan16(8, 8, 1 << 20, 1, 1)
    for v in (50000, 40000):
        assert sc.add_frame_u16(np.full((8, 8), v), np.full((4, 4), v), np.full((4, 4), v))
    s = sc.sums()[0]
    bg = [-15535, -25535]
    assert s.tolist() == [90000.0, float(sum(bg)), float(50000 ** 2 - 2 ** 32 + 40000 ** 2),
                          float(bg[0] ** 2 + bg[1] ** 2), float(50000 * bg[0] + 40000 * bg[1])]
