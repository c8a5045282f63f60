"""The mutation table of tools/mutants.py stays applicable and inside its safety rule: every mutant's `before` snippet occurs
exactly once in its file, no mutant touches block barriers, mbarriers, TMA or bulk copies, atomics, the work queue or the
watchdog, every equivalent mutant carries its argument, and every mutant the GPU tests name as killed is in the table."""
import glob
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mutants  # noqa: E402


@pytest.mark.parametrize("m", mutants.MUTANTS, ids=lambda m: m["name"])
def test_before_occurs_once(m):
    with open(os.path.join(ROOT, m["file"])) as f:
        src = f.read()
    assert src.count(m["before"]) == 1
    assert m["after"] != m["before"]
    assert mutants.apply(src, m).count(m["after"]) >= 1


@pytest.mark.parametrize("m", mutants.MUTANTS, ids=lambda m: m["name"])
def test_no_forbidden_token(m):
    for tok in mutants.FORBIDDEN:
        assert tok not in m["before"] and tok not in m["after"], tok


def test_table_is_well_formed():
    names = [m["name"] for m in mutants.MUTANTS]
    assert len(names) == len(set(names))
    for m in mutants.MUTANTS:
        assert m["what"] and m["tests"], m["name"]
        assert m["equivalent"] is None or len(m["equivalent"]) > 40, m["name"]
        for t in m["tests"]:
            assert os.path.exists(os.path.join(ROOT, t.split("::")[0])), (m["name"], t)


def test_named_kills_are_in_the_table():
    """Mutant names in the 'Kills ...' sentences of the tests' docstrings are all entries of the table, and every mutant
    that is not equivalent is named by some test."""
    named = set()
    for path in glob.glob(os.path.join(ROOT, "tests", "test_gpu_*.py")):
        with open(path) as f:
            for block in re.findall(r"Kills ([^.]*)\.", f.read()):
                named.update(re.findall(r"[a-z0-9_]+", block))
    table = {m["name"] for m in mutants.MUTANTS}
    assert named <= table, sorted(named - table)
    assert {m["name"] for m in mutants.MUTANTS if not m["equivalent"]} - named <= {
        "generic_split_prev"}, sorted({m["name"] for m in mutants.MUTANTS if not m["equivalent"]} - named)
