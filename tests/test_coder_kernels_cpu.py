"""CPU-only check of the coder instantiations in the built library (cuobjdump -res-usage).

The generic two-phase coder (k_rows / k_rows_wide, k_pop_coarse, k_push_pairs), the shared-table prior pop (k_pop_full),
the affine-row coder (k_rows6 / k_pop6) and the fused coder (k_logistic_push / k_logistic_pop) must be instantiated
exactly for the supports their dispatchers accept, and nothing else: a support missing from a dispatcher, or a kernel
variant left behind, changes the set.  Every coder kernel must fit its __launch_bounds__ without spilling.
"""
import re
import subprocess

import pytest

from bitswap_b200 import _lib

NBS = [1, 2, 4, 8, 16, 32, 64, 128]                      # bins per lane: S = 32 * NB = 32 ... 4096
FUSED_NBS = [nb for nb in NBS if nb <= 32]


def _expected():
    want = set()
    for nb in NBS:
        for flag in (0, 1):
            want.add(("k_rows", (nb, flag)) if nb <= 32 else ("k_rows_wide", (nb // 32, flag)))    # POP
            want.add(("k_pop_coarse", (nb, flag)))                                                 # MASK
    for nb in FUSED_NBS:
        for mask in (0, 1):
            want.add(("k_logistic_push", (nb, mask)))
            want.add(("k_logistic_pop", (nb, mask)))
    want |= {("k_pop_full", (nb,)) for nb in (4, 8, 16, 32)}
    want |= {("k_push_pairs", (m,)) for m in (0, 1)}
    for pop in (0, 1):
        for verify, lpr in ((0, 2), (0, 4), (0, 8), (0, 32), (1, 4), (1, 32)):
            for wide in (0, 1):
                want.add(("k_rows6", (pop, verify, lpr, wide)))
    want |= {("k_pop6", (mask, wide)) for mask in (0, 1) for wide in (0, 1)}
    return want


CODER = {name for name, _ in _expected()} | {"k_pop_coarse_wide"}
# registers per thread allowed by each kernel's __launch_bounds__: 512 threads x 2 CTAs per SM for the row-table kernels,
# 128-thread CTAs (no minimum) for the serial and fused ones
MAX_REG = {"k_rows": 64, "k_rows_wide": 64, "k_rows6": 64}


def _parse(mangled):
    """(kernel name, integral template arguments) of a mangled kernel name, or None."""
    for m in re.finditer(r"(\d+)k_", mangled):
        digits, at = m.group(1), m.end(1)
        for k in range(1, len(digits) + 1):                # the length prefix may follow other digits (anonymous namespace)
            n = int(digits[-k:])
            name = mangled[at:at + n]
            if n > 2 and re.fullmatch(r"k_\w+", name) and mangled[at + n:at + n + 1] in ("I", "E", "v"):
                targs = re.match(r"I((?:L[a-z]\d+E)+)", mangled[at + n:])      # Li16E, Lb1E, ...
                return name, tuple(int(v) for v in re.findall(r"L[a-z](\d+)E", targs.group(1))) if targs else ()
    return None


@pytest.fixture(scope="module")
def usage():
    so = _lib.build()
    out = subprocess.run(["cuobjdump", "-res-usage", so], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True).stdout
    res = {}
    for mangled, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out):
        key = _parse(mangled)
        if key and key[0] in CODER:
            assert key not in res, key
            res[key] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    return res


def test_coder_instantiations_are_exactly_the_supported_ones(usage):
    want = _expected()
    assert sorted(set(usage) - want) == [], "unexpected coder kernels"
    assert sorted(want - set(usage)) == [], "coder kernels missing from the library"


def test_coder_kernels_fit_their_launch_bounds(usage):
    for (name, args), u in sorted(usage.items()):
        assert u["LOCAL"] == 0, f"{name}{args} uses local memory: {u}"
        assert u["REG"] <= MAX_REG.get(name, 255), f"{name}{args}: {u}"
