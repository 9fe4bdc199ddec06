"""Generates the kernel-size / width golden files by running the REFERENCE's own Model (same recipe as make_golden.py).

Run in the build container only (needs the reference checkout, read-only; BITSWAP_REFERENCE overrides its path):
    python tests/golden/make_golden_kw.py
The outputs are committed; nothing at test time reads the reference.

What is pinned, for three models the reference's training scripts build with --kernel 5 / 1 / 7:
  model_kw_*.npz    the reference Model's infer(i) / generate(i) mu and scale on fixed inputs, with weights from the
                    seeded synthetic generator loaded with load_state_dict(strict=True) -- which also pins the key layout
                    and shapes of synthetic.state_dict_spec for these flags.  The weights are not stored: tests
                    regenerate them from the seed.  The config is stored as JSON under "cfg".
"""
import json
import os
import sys
from dataclasses import asdict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import ImageBins, OUT, ref_model                # noqa: E402  (reference classes + shared helpers)

from bitswap_b200.config import CodecConfig                     # noqa: E402
from bitswap_b200 import synthetic                              # noqa: E402

SEED = 50
MODELS = {
    "kw_k5_w100": CodecConfig(xs=(3, 32, 32), nz=2, zchannels=2, nprocessing=1, kernel_size=5, resdepth=2, reswidth=100),
    "kw_k1_w12": CodecConfig(xs=(1, 32, 32), nz=2, zchannels=1, nprocessing=1, kernel_size=1, resdepth=2, reswidth=12),
    "kw_k7_w16": CodecConfig(xs=(3, 32, 32), nz=3, zchannels=2, nprocessing=1, kernel_size=7, resdepth=3, reswidth=16,
                             cond_xscale=True),
}


def model_golden(name, cfg):
    sd = synthetic.synthetic_state_dict(cfg, seed=SEED, varied=True)
    m = ref_model(cfg, sd)
    _, zcen = synthetic.synthetic_bins(cfg, seed=0)
    rs = np.random.RandomState(3)
    out = {"cfg": np.array(json.dumps(asdict(cfg)))}
    x = synthetic.synthetic_images(cfg, 1, seed=9)[0].reshape(-1).astype(np.int64)
    xcen = ImageBins(torch.float64, "cpu", cfg.xdim).centres()
    given = xcen[torch.arange(cfg.xdim), torch.from_numpy(x)]
    out["x"] = x.astype(np.uint8)
    with torch.no_grad():
        for i in range(cfg.nz):
            if i > 0:
                sym = rs.randint(0, cfg.zsupport, cfg.zdim)
                out[f"zsym_in_infer{i}"] = sym.astype(np.int16)
                given = zcen[i - 1, torch.arange(cfg.zdim), torch.from_numpy(sym)]
            mu, sc = m.infer(i)(given=given)
            out[f"infer{i}_mu"], out[f"infer{i}_scale"] = mu.numpy(), sc.numpy()
            sym = rs.randint(0, cfg.zsupport, cfg.zdim)
            out[f"zsym_in_gen{i}"] = sym.astype(np.int16)
            z = zcen[i, torch.arange(cfg.zdim), torch.from_numpy(sym)]
            mu, sc = m.generate(i)(given=z)
            out[f"gen{i}_mu"], out[f"gen{i}_scale"] = mu.numpy(), sc.numpy()
    np.savez_compressed(os.path.join(OUT, f"model_{name}.npz"), **out)


if __name__ == "__main__":
    torch.set_num_threads(4)
    for name, cfg in MODELS.items():
        model_golden(name, cfg)
    print("kernel-size / width golden files written to", OUT)
