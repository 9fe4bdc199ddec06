"""CPU-only checks for models of any kernel size (1, 3, 5, 7) and padded width (64, 128, ..., 512):

1. the conv instantiations in the built library (cuobjdump -res-usage): exactly one k_conv_wg tile per padded width and
   one per head kind and no other, each within the launch shape (<= 128 registers, no spills), the width-256 dense tile and the
   non-folding head at their pinned counts; k_conv_simt at kernel sizes 1 and 7 without spills;
2. config validation: an even kernel size, or one outside 1..7, is refused before any device work, by CodecConfig and
   Model (ValueError) and by bsw_model_create (BSW_E_INVALID);
3. the float32 / float64 model oracle against the reference Model's outputs for --kernel 5 / 1 / 7 models
   (tests/golden/make_golden_kw.py).
"""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from bitswap_b200 import _lib, synthetic
from bitswap_b200.config import CodecConfig
from bitswap_b200.model import Model, _Desc
from codec_harness import KW_MODELS, golden_model, model_oracle_vs_golden
from oracle import oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def usage():
    so = _lib.build()
    out = subprocess.run(["cuobjdump", "-res-usage", so], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True).stdout
    res = {}
    for name, line in re.findall(r"Function (\S*(?:k_conv_wg|k_conv_simt)I\S*):\s*\n\s*(REG:.*)", out):
        res[name] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    return res


# Every k_conv_wg instantiation, as (test id, mangled template argument): the dense tile at each padded width and the
# heads without and with the per-tap fold.
CONV_WG_TILES = [(f"dense{w}", f"DenseArgsILi{w}E") for w in (64, 128, 192, 256, 320, 384, 448, 512)] + \
                [("head", "HeadArgsILb0E"), ("head_fold", "HeadArgsILb1E")]
# k_conv_wg runs 384 threads under __maxnreg__(128): 48 K registers, so a coder CTA still fits beside a conv CTA
# (DESIGN 5.2).  SHARED is the static part only; the stages and hand-off tile are dynamic.
PINNED_USAGE = {"dense256": {"REG": 128, "SHARED": 1024, "LOCAL": 0, "STACK": 0},
                "head": {"REG": 128, "SHARED": 1024, "LOCAL": 0, "STACK": 0}}


def _is_tile(name, args):
    return re.search(rf"k_conv_wgINS_\d+{args}EEEEv", name) is not None


def test_conv_wg_instantiations_are_exactly_the_tiles(usage):
    """The library holds one k_conv_wg per padded width and head kind, and no other: a width missing from the
    dispatcher, or a tile type left behind, changes the set."""
    names = [k for k in usage if "k_conv_wg" in k]
    tiles = [t for n in names for t, args in CONV_WG_TILES if _is_tile(n, args)]
    assert len(tiles) == len(names), names
    assert sorted(tiles) == sorted(t for t, _ in CONV_WG_TILES), names


@pytest.mark.parametrize("tile,args", CONV_WG_TILES, ids=[t for t, _ in CONV_WG_TILES])
def test_conv_wg_tiles_fit_the_launch_shape(usage, tile, args):
    u = [v for k, v in usage.items() if _is_tile(k, args)]
    assert len(u) == 1, sorted(usage)
    assert u[0]["REG"] <= 128, u[0]
    assert u[0]["LOCAL"] == 0 and u[0]["STACK"] == 0, f"{tile} spills: {u[0]}"
    if tile in PINNED_USAGE:
        assert {k: u[0][k] for k in PINNED_USAGE[tile]} == PINNED_USAGE[tile]


@pytest.mark.parametrize("ks,tco", [(1, 2), (1, 8), (7, 2), (7, 8)])
def test_simt_kernel_sizes_1_and_7_do_not_spill(usage, ks, tco):
    u = [v for k, v in usage.items() if f"k_conv_simtILi{ks}ELi{tco}EE" in k]
    assert len(u) == 1, sorted(usage)
    assert u[0]["LOCAL"] == 0 and u[0]["STACK"] == 0, f"k_conv_simt<{ks}, {tco}> spills: {u[0]}"


@pytest.mark.parametrize("ks", [1, 3, 5, 7])
def test_config_accepts_odd_kernels_up_to_7(ks):
    assert CodecConfig(kernel_size=ks).kernel_size == ks


@pytest.mark.parametrize("ks", [-1, 0, 2, 4, 6, 8, 9, 11])
def test_config_and_model_refuse_other_kernels(ks):
    with pytest.raises(ValueError):
        CodecConfig(kernel_size=ks)
    with pytest.raises(ValueError):
        Model(xs=(3, 32, 32), nz=2, zchannels=8, kernel_size=ks, reswidth=100)


@pytest.mark.parametrize("ks,rc", [(4, 4), (9, 4), (0, 4)])
def test_model_create_refuses_other_kernels(ks, rc):
    """The descriptor check comes before any allocation: BSW_E_INVALID, no device needed."""
    h = ctypes.c_void_p()
    d = _Desc(3, 2, 8, 1, ks, 2, 100, 0, 1, 1)
    assert _lib.lib().bsw_model_create(ctypes.byref(h), ctypes.byref(d)) == rc
    assert not h.value
    assert "kernel_size" in _lib.lib().bsw_last_error().decode()


@pytest.mark.parametrize("name", KW_MODELS)
def test_kw_model_oracle_matches_reference(name):
    """The oracle builds --kernel 5 / 1 / 7 models as the reference does: float32 within 2e-6 absolute of the golden
    outputs (measured: identical), float64 within 2e-5 relative to max(1, |output|).  The golden outputs carry the
    reference's float32 rounding, which grows with the taps summed: measured 9.6e-7 (1x1), 3.2e-6 (5x5) and 6.9e-6
    (7x7) absolute against the float64 oracle."""
    cfg, _ = golden_model(name)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    for dtype, tol in ((torch.float32, lambda want: 2e-6), (torch.float64, lambda want: 2e-5 * np.maximum(1.0, np.abs(want)))):
        orc = O.ModelOracle(cfg, sd, dtype=dtype)
        model_oracle_vs_golden(name, lambda kind, i, g: (orc.infer(i) if kind == "infer" else orc.generate(i))(g), tol)
