"""CPU-only checks for models wider than 256 channels (reswidth 257..512, padded widths 320, 384, 448, 512); the
k_conv_wg instantiations at these widths are checked with the others in test_kernel_width_cpu.py:

1. synthetic.state_dict_spec at these widths: key layout and shapes of the reference's ResNet blocks, in-convs and heads;
2. the float32 / float64 model oracle against the reference Model's outputs at widths 320 and 512
   (tests/golden/make_golden_wide.py).
"""
import re

import numpy as np
import pytest
import torch

from bitswap_b200 import synthetic
from bitswap_b200.config import CodecConfig
from oracle import oracle as O
from codec_harness import WIDE_MODELS, golden_model, model_oracle_vs_golden


@pytest.mark.parametrize("W,ks", [(257, 3), (320, 5), (448, 1), (512, 7)])
def test_state_dict_spec_at_wide_widths(W, ks):
    cfg = CodecConfig(xs=(3, 32, 32), nz=3, zchannels=8, nprocessing=1, kernel_size=ks, resdepth=3, reswidth=W)
    spec = {k: shape for k, shape, _ in synthetic.state_dict_spec(cfg)}
    assert spec["infer_in.1.v"] == (W, 12, 5, 5)
    assert spec[f"infer_res0.0.res{W}layer1.conv1.v"] == (W, W, 5, 5)
    for p in ("infer_res1.0", "deepinfer_res.0.0", "deepgen_res.1.0", "gen_res1.0"):
        assert spec[f"{p}.res{W}layer1.conv1.v"] == (W, W, ks, ks)
        assert spec[f"{p}.res{W}layer1.conv2.gain"] == (W,)
    assert spec["deepgen_in.1.0.v"] == (W, 8, ks, ks)
    assert spec["deepinfer_mu.0.0.v"] == spec["deepgen_std.1.0.v"] == (8, W, ks, ks)
    assert spec["gen_mu.0.v"] == (12, W, ks, ks)
    assert not [k for k in spec if re.search(r"res\d+layer", k) and f"res{W}layer" not in k]


@pytest.mark.parametrize("name", WIDE_MODELS)
def test_wide_model_oracle_matches_reference(name):
    """The oracle builds width-320 and width-512 models as the reference does: float32 within 2e-6 absolute of the golden
    outputs, float64 within 2e-5 relative to max(1, |output|)."""
    cfg, _ = golden_model(name)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    for dtype, tol in ((torch.float32, lambda want: 2e-6), (torch.float64, lambda want: 2e-5 * np.maximum(1.0, np.abs(want)))):
        orc = O.ModelOracle(cfg, sd, dtype=dtype)
        model_oracle_vs_golden(name, lambda kind, i, g: (orc.infer(i) if kind == "infer" else orc.generate(i))(g), tol)
