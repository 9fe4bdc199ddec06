"""CPU-only checks of the tensor-core conv kernel's instantiations in the built library (cuobjdump -res-usage): the
narrow tile of padded-width-64 models compiles within the launch shape the conv path relies on, and adding it left the
wide and head instantiations at their resource counts."""
import re
import subprocess

import pytest

from bitswap_b200 import _lib

# k_conv_wg runs 384 threads under __maxnreg__(128): 48 K registers, so a coder CTA still fits beside a conv CTA
# (DESIGN 5.2).  SHARED is the static part only; the stages and hand-off tile are dynamic.
WIDE_AND_HEADS = {"TcArgs": {"REG": 128, "SHARED": 1024, "LOCAL": 0, "STACK": 0},
                  "HeadArgs": {"REG": 128, "SHARED": 1024, "LOCAL": 0, "STACK": 0}}


@pytest.fixture(scope="module")
def usage():
    so = _lib.build()
    out = subprocess.run(["cuobjdump", "-res-usage", so], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True).stdout
    res = {}
    for args, line in re.findall(r"Function \S*k_conv_wgIN\S*?\d+(\w+?)EEEv\S*:\s*\n\s*(REG:.*)", out):
        res[args] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    assert res, "no k_conv_wg instantiation found in the library"
    return res


def test_narrow_instantiation_fits_the_launch_shape(usage):
    assert "NarrowArgs" in usage, sorted(usage)
    u = usage["NarrowArgs"]
    assert u["REG"] <= 128, u
    assert u["LOCAL"] == 0 and u["STACK"] == 0, f"the narrow tile spills: {u}"


@pytest.mark.parametrize("args", sorted(WIDE_AND_HEADS))
def test_wide_and_head_instantiations_unchanged(usage, args):
    assert args in usage, sorted(usage)
    got = {k: usage[args][k] for k in WIDE_AND_HEADS[args]}
    assert got == WIDE_AND_HEADS[args]
