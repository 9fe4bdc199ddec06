"""The dense convs and in-convs run as one four-CTA cluster per image that share their operand loads by TMA multicast.
Every CTA still computes the same tile with the same k order and MMAs, so mu/sigma must be bit-identical to the
single-CTA launches (conv mode bit 8) on both grids."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from conv_harness import conv_mode, outputs_in_conv_modes   # noqa: E402
from bitswap_b200 import synthetic                   # noqa: E402
from bitswap_b200.config import CodecConfig          # noqa: E402
from bitswap_b200.model import Model                 # noqa: E402

NO_MULTICAST = 8


@pytest.mark.parametrize("B", [170, 1])
def test_multicast_clusters_equal_single_cta_convs(B):
    """Per-tile grid (mode 0) and persistent grid (mode 7), each with and without multicast, over every conv shape on the
    path: in-convs with 1 and 25 taps, dense 3x3, 5x5 and the heads.  B = 170 leaves some clusters of the persistent grid
    one image more than others; B = 1 is a single cluster."""
    cfg = CodecConfig(xs=(3, 32, 32), nz=2, zchannels=8, nprocessing=1, resdepth=1, reswidth=252)
    out = outputs_in_conv_modes(cfg, B, (0, NO_MULTICAST, 7, 7 | NO_MULTICAST), seed=5)
    for grid in (0, 7):
        for a, b in zip(out[grid], out[grid | NO_MULTICAST]):
            assert torch.equal(a, b), f"conv mode {grid} with and without multicast"
        assert all(torch.isfinite(t).all() for t in out[grid])


def test_default_multicast_grid_vs_float64_oracle():
    """The default grid (mode 7: persistent four-CTA clusters with multicast, several images per cluster at B = 170)
    against an independent reference: the float64 oracle, within the 1e-4 bar on mu/sigma."""
    from oracle import oracle as O
    B = 170
    cfg = CodecConfig(xs=(3, 32, 32), nz=2, zchannels=8, nprocessing=1, resdepth=1, reswidth=252)
    sd = synthetic.synthetic_state_dict(cfg, seed=61, varied=True)
    m = Model.from_config(cfg, max_batch=B, use_tensor_cores=True).load_state_dict(sd)
    m.compress()
    orc = O.ModelOracle(cfg, sd, dtype=torch.float64, device="cuda")
    rs = np.random.RandomState(6)
    gx = torch.from_numpy((rs.randint(0, 256, (B, cfg.xdim)) - 127.5) / 127.5).cuda()
    gz = torch.from_numpy(rs.uniform(-5, 5, (B, cfg.zdim))).cuda()
    worst = 0.0
    with conv_mode(7):
        for i in range(cfg.nz):
            for kind, g in (("infer", gx if i == 0 else gz), ("generate", gz)):
                mu, sc = (m.infer(i) if kind == "infer" else m.generate(i))(g)
                mu_o, sc_o = (orc.infer(i) if kind == "infer" else orc.generate(i))(g)
                worst = max(worst, (mu - mu_o).abs().max().item(), (sc - sc_o).abs().max().item())
    print(f"mode 7, B = {B}: max |err| vs torch-f64 oracle {worst:.2e}")
    assert worst < 1e-4, worst

