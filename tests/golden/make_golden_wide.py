"""Generates the wide-model golden files by running the REFERENCE's own Model (same recipe as make_golden_kw.py).

Run in the build container only (needs the reference checkout, read-only; BITSWAP_REFERENCE overrides its path):
    python tests/golden/make_golden_wide.py
The outputs are committed; nothing at test time reads the reference.

What is pinned, for two models the reference's training scripts build with --width above 256:
  model_wide_*.npz  the reference Model's infer(i) / generate(i) mu and scale on fixed inputs, with weights from the
                    seeded synthetic generator loaded with load_state_dict(strict=True) -- which also pins the key layout
                    and shapes of synthetic.state_dict_spec at these widths.  The weights are not stored: tests
                    regenerate them from the seed.  The config is stored as JSON under "cfg".
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_kw import model_golden                         # noqa: E402

from bitswap_b200.config import CodecConfig                     # noqa: E402

MODELS = {
    "wide_k3_w320": CodecConfig(xs=(3, 32, 32), nz=2, zchannels=2, nprocessing=1, kernel_size=3, resdepth=2, reswidth=320),
    "wide_k7_w512": CodecConfig(xs=(3, 32, 32), nz=2, zchannels=2, nprocessing=1, kernel_size=7, resdepth=2, reswidth=512,
                                cond_xscale=True),
}


if __name__ == "__main__":
    torch.set_num_threads(4)
    for name, cfg in MODELS.items():
        model_golden(name, cfg)
    print("wide golden files written to", os.path.dirname(os.path.abspath(__file__)))
