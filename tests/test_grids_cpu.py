"""The CPU twin of the affine-row coder (scripts/rows6_model.cpp: the arithmetic of k_rows6 / k_pop6 from rows6_core.cuh, the
row classification of k_row_meta) on every family of endpoint grid discretize() can build: off-centre, float16-extreme, far
from zero and narrow, tiny spans, coarse grids at the plan's dt limit, and rows off the affine line by up to the
classification tolerance.  Every integer pmf must be the exact function's, the pop search must reproduce a search of the
full table, and the worst screening error of a trusted bin must stay below a quarter of its window -- the margin that
catches an under-sized window even where no integer happens to flip."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TWIN = os.path.join(ROOT, "scripts", "rows6_model.cpp")
FAMILIES = {1: "off-centre", 2: "float16 extrema", 3: "far and narrow", 4: "tiny span", 5: "dt near 64", 6: "perturbed"}


@pytest.fixture(scope="module")
def twin(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ is not installed: the CPU twin of the affine-row coder cannot be compiled")
    exe = str(tmp_path_factory.mktemp("rows6") / "rows6_model")
    r = subprocess.run([gxx, "-O2", "-std=c++17", "-o", exe, TWIN, "-lm"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _run(exe, rows, seed, S, family):
    r = subprocess.run([exe, str(rows), str(seed), str(S), str(family)], capture_output=True, text=True, timeout=300)
    out = r.stdout
    print(out)
    m = re.search(r"mismatches (\d+) \(in dead zones \d+\)  pop-search mismatches (\d+)  worst trusted err [\d.]+ units "
                  r"\(([\d.]+) of its window\)", out)
    fix = re.search(r"wide fix-word mismatches (\d+)", out)
    share = re.search(r"exact-path \d+ \(([\d.]+)% of evaluated\)", out)
    assert m and fix and share, out
    return r.returncode, int(m.group(1)), int(m.group(2)), int(fix.group(1)), float(m.group(3)), float(share.group(1))


def _check(res, what):
    rc, mism, popbad, fixbad, worst, share = res
    print(f"{what}: exact path {share:.2f} % of evaluated bins, worst trusted error {worst:.3f} of its window")
    assert (rc, mism, popbad, fixbad) == (0, 0, 0, 0), f"{what}: exit {rc}, {mism} mismatches, {popbad} pop-search and " \
                                                       f"{fixbad} fix-word mismatches"
    assert worst <= 0.25, f"{what}: worst trusted error {worst} of its window"


@pytest.mark.parametrize("family", list(FAMILIES))
def test_twin_every_grid_family_on_mixed_supports(twin, family):
    """8000 rows of family `family` at the mix of 1024 / 256 / 64 bins."""
    _check(_run(twin, 8000, 11 + family, 0, family), FAMILIES[family])


@pytest.mark.parametrize("S", [2048, 4096])
@pytest.mark.parametrize("family", [1, 3, 4])
def test_twin_grid_families_at_wide_supports(twin, family, S):
    """quantbits 11 and 12 (chains re-anchored every 256 bins, the wide fix word) on the off-centre, far-and-narrow and
    tiny-span grids."""
    _check(_run(twin, 600, 21 + family, S, family), f"{FAMILIES[family]} at S = {S}")


def test_twin_default_rows_are_unchanged(twin):
    """Family 0 is the grid family the kernels were tuned on (spans about -6.5 .. 6.5): still exact, and the family
    argument does not disturb its draws."""
    _check(_run(twin, 8000, 5, 0, 0), "default grids")
    plain = subprocess.run([twin, "3000", "7"], capture_output=True, text=True).stdout
    fam0 = subprocess.run([twin, "3000", "7", "0", "0"], capture_output=True, text=True).stdout
    assert fam0.startswith(plain) and fam0[len(plain):].startswith("family 0:")
