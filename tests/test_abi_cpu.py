"""CPU-only checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, and exports
every symbol include/bitswap_b200.h declares (no compute calls without a GPU)."""
import ctypes
import os
import re

import pytest

from bitswap_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def so():
    return _lib.build()


def test_header_symbols_are_exported(so):
    hdr = open(os.path.join(ROOT, "include", "bitswap_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)             # drop comments
    declared = sorted(set(re.findall(r"\b(bsw_[a-z0-9_]+)\s*\(", hdr)))
    assert declared, "no declarations parsed"
    L = ctypes.CDLL(so)
    missing = [n for n in declared if not hasattr(L, n)]
    assert not missing, f"declared in the header but not exported: {missing}"
    assert sorted(_lib.EXPORTS) == declared


def test_library_is_sm90a_only(so):
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", so], stdout=subprocess.PIPE, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_product_does_not_import_the_oracle():
    pkg = os.path.join(ROOT, "bitswap_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert "oracle" not in src.replace("no oracle", ""), f"{f} mentions the oracle"


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "SO_PATH", str(tmp_path / "nope.so"))
    monkeypatch.setattr(_lib, "_lib", None)
    with pytest.raises(_lib.BswError):
        _lib.lib()
