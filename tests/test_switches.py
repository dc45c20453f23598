"""The library's environment switches exist so that the tests can run a second path on the same input: every switch the
CUDA sources name must be set by some test, and only host_util.cu reads the environment at all (so DCR_B200_TUNING
gates every switch)."""
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "dcr_b200" / "csrc"


def _sources():
    return sorted(p for p in CSRC.iterdir() if p.suffix in (".cu", ".cuh", ".h"))


def test_every_switch_is_set_by_a_test():
    # every quoted DCR_* name, not only tuning_flag("...") / tuning_int("...") arguments: a wrapper around those
    # must not hide a switch
    switches, hooks = set(), set()
    for src in _sources():
        txt = src.read_text()
        switches |= set(re.findall(r'"(DCR_[A-Z0-9_]+)"', txt))
        hooks |= set(re.findall(r'tuning_(?:flag|int)\("([A-Z0-9_]+)"', txt))
    switches.discard("DCR_B200_TUNING")
    assert hooks and hooks <= switches
    tests = "\n".join(p.read_text() for p in sorted((ROOT / "tests").glob("test_*.py")) if p.name != Path(__file__).name)
    unset = sorted(s for s in switches if not re.search(r"""setenv\(\s*["']%s["']""" % s, tests))
    assert not unset, f"switches no test sets: {unset}"


def test_only_host_util_reads_the_environment():
    readers = sorted(src.name for src in _sources() if "getenv" in src.read_text())
    assert readers == ["host_util.cu"], readers
