"""Models of any kernel size (1, 3, 5, 7) and of padded width 128 or 192 on the tensor cores.

1. P3c per layer: every conv kind on its own against float64, with the harness of conv_harness.py (same inputs, value
   sets, bars tau = 2^-13 / 2^-14 and exact checks), on [2, MAXB, 256, Wp] plane buffers: widths 65..192 at kernel 3,
   kernels 1 / 5 / 7 at widths 61, 128, 192 and 252.  Conv modes 8 / 15 must be bit-identical to 0 / 7.  The worst
   normalised error is reported per (path, conv kind, kernel size, padded width).
2. Whole nets against the float64 oracle (1e-4) and the SIMT path, batch invariance, persistent == per-tile grid.
3. The reference pin: Model against the reference's outputs (tests/golden/model_kw_*.npz) within 1e-4.
4. The Bit-Swap recursion through PipelinedCodec defaults against the oracle, exact round trips, and edge-coded
   containers, for a padded-width-128 and a padded-width-192 model with kernel sizes 5 and 7.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from codec_harness import KW_MODELS, TOL, golden_model, gpu_oracle, model_oracle_vs_golden, tc_case   # noqa: E402
from conv_harness import VALUES, Case, conv_cfg, outputs_in_conv_modes, worst_report   # noqa: E402
from oracle import oracle as O                                         # noqa: E402
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200.model import Model                                   # noqa: E402
from bitswap_b200.codec import Bins, PipelinedCodec                    # noqa: E402
from bitswap_b200.container import compress_images, decompress_images  # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402

# (tensor cores?, config).  zchannels <= 32 run the in-conv on the tensor cores, 40 the SIMT in-conv + split; heads of
# <= 32 outputs run on the tensor cores, 40 and 80 on k_conv_simt after a tensor-core trunk.
MODELS = {
    # padded width 128 / 192 at kernel 3
    "tc k3 W65 zc1 C3": (True, conv_cfg(3, 1, 65, 3)),
    "tc k3 W100 zc20 C3": (True, conv_cfg(3, 20, 100, 3)),
    "tc k3 W128 zc40 C1 cond": (True, conv_cfg(1, 40, 128, 3, cond=True)),
    "tc k3 W129 zc2 C1 cond": (True, conv_cfg(1, 2, 129, 3, cond=True)),
    "tc k3 W150 zc40 C3": (True, conv_cfg(3, 40, 150, 3)),
    "tc k3 W192 zc16 C1": (True, conv_cfg(1, 16, 192, 3)),
    # kernel sizes 1 / 5 / 7 at padded widths 64, 128, 192, 256
    "tc k1 W61 zc8 C3": (True, conv_cfg(3, 8, 61, 1)),
    "tc k1 W128 zc20 C1 cond": (True, conv_cfg(1, 20, 128, 1, cond=True)),
    "tc k1 W192 zc1 C3": (True, conv_cfg(3, 1, 192, 1)),
    "tc k1 W252 zc40 C1": (True, conv_cfg(1, 40, 252, 1)),
    "tc k5 W61 zc40 C1": (True, conv_cfg(1, 40, 61, 5)),
    "tc k5 W128 zc2 C3 cond": (True, conv_cfg(3, 2, 128, 5, cond=True)),
    "tc k5 W192 zc20 C3": (True, conv_cfg(3, 20, 192, 5)),
    "tc k5 W252 zc8 C1": (True, conv_cfg(1, 8, 252, 5)),
    "tc k7 W61 zc20 C3": (True, conv_cfg(3, 20, 61, 7)),
    "tc k7 W128 zc8 C1": (True, conv_cfg(1, 8, 128, 7)),
    "tc k7 W192 zc40 C3 cond": (True, conv_cfg(3, 40, 192, 7, cond=True)),
    "tc k7 W252 zc2 C1 cond": (True, conv_cfg(1, 2, 252, 7, cond=True)),
    # the float32 SIMT path at kernel sizes 1 and 7 (dense convs too)
    "simt k1 W100 zc20 C1": (False, conv_cfg(1, 20, 100, 1)),
    "simt k7 W63 zc2 C3 cond": (False, conv_cfg(3, 2, 63, 7, cond=True)),
}
MINE = {}                                    # ("k{ks} Wp{Wp}", path, kind) -> worst normalised error
_report = worst_report("P3c per kernel size and padded width: worst |out - f(y)| / s (beyond the ELU/rounding allowance)",
                       MINE)


@pytest.mark.parametrize("vs", VALUES)
@pytest.mark.parametrize("name", list(MODELS))
def test_kernel_width_conv_kernels_vs_float64(name, vs):
    Case(MODELS, name, vs, seed_base=9000, worst=MINE, compare_modes=True, per_kernel_width=True).run()


NETS = {
    "k3 W100 nz2": conv_cfg(3, 8, 100, 3),
    "k3 W150 nz3 cond": conv_cfg(3, 8, 150, 3, True, nz=3),
    "k5 W128 nz2": conv_cfg(3, 8, 128, 5),
    "k7 W192 nz2 zc40": conv_cfg(3, 40, 192, 7),
    "k1 W252 nz4": conv_cfg(3, 8, 252, 1, nz=4),
    "k1 W65 nz3 zc20": conv_cfg(1, 20, 65, 1, nz=3),
    "k7 W61 nz2 cond": conv_cfg(3, 2, 61, 7, True),
}


@pytest.mark.parametrize("name", list(NETS))
def test_kernel_width_nets_vs_f64_oracle_and_simt(name):
    """Whole nets on the tensor cores: mu / sigma of every infer(i) / generate(i) within 1e-4 of the float64 oracle and
    of the SIMT path; a row alone equals the same row in the batch, bit for bit."""
    worst_o, worst_s = tc_case(NETS[name], 3, dtype=torch.float64)
    print(f"tensor cores {name}: max |err| vs torch-f64 oracle {worst_o:.2e}, vs SIMT f32 path {worst_s:.2e}")
    assert worst_o < TOL and worst_s < TOL


@pytest.mark.parametrize("name", ["k7 W128", "k1 W192"])
def test_kernel_width_persistent_grid_equals_per_tile_grid(name):
    """B = 170: 340 (Wp 128) / 1020 (Wp 192) tiles per dense conv, several per CTA on the persistent grid; in-convs with
    1 / 49 and 25 taps, dense convs, heads.  Bit-identical mu and sigma."""
    cfg = {"k7 W128": conv_cfg(3, 8, 128, 7, nz=3), "k1 W192": conv_cfg(1, 2, 192, 1, True, nz=3)}[name]
    out = outputs_in_conv_modes(cfg, 170, (0, 7))
    for a, b in zip(out[0], out[7]):
        assert torch.equal(a, b), "conv mode 7"
    assert all(torch.isfinite(t).all() for t in out[7])


@pytest.mark.parametrize("tc", [True, False], ids=["tc", "simt"])
@pytest.mark.parametrize("name", KW_MODELS)
def test_kernel_width_model_matches_reference(name, tc):
    """Model (tensor cores and SIMT) within 1e-4 of the reference Model's outputs for --kernel 5 / 1 / 7."""
    cfg, _ = golden_model(name)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    m = Model.from_config(cfg, max_batch=1, use_tensor_cores=tc).load_state_dict(sd)
    m.compress()
    worst = model_oracle_vs_golden(name, lambda kind, i, g: (m.infer(i) if kind == "infer" else m.generate(i))(g.cuda()),
                                   lambda want: TOL)
    print(f"{name} {'tensor cores' if tc else 'SIMT'}: max |err| vs the reference {worst:.2e}")


RECURSION = {"k5 W100": conv_cfg(3, 8, 100, 5), "k7 W150": conv_cfg(3, 8, 150, 7, nz=3)}


@pytest.mark.parametrize("name", list(RECURSION))
def test_kernel_width_recursion_vs_oracle_and_roundtrip(name):
    """PipelinedCodec with its defaults (tensor-core nets), 256 streams over 4 lanes:
    (a) sampled streams == the oracle recursion driven with the same GPU nets and torch-CUDA float64 pmfs;
    (b) exact pixel round trip, initial states restored."""
    B, nsample = 256, 6
    cfg = RECURSION[name]
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    bins = Bins(cfg, zend, zcen)
    pc = PipelinedCodec(cfg, sd, bins, B)
    assert pc.lanes == 4
    imgs = synthetic.synthetic_images(cfg, B, seed=78)
    ss = StreamSet(B, 8192)
    w, head = synthetic.initial_words(4096, seed=100)
    ss.fill(w, head)
    init = ss.export_lists()
    pc.encode(ss, torch.from_numpy(imgs).cuda())
    torch.cuda.synchronize()
    ss.raise_on_error()
    got = ss.export_lists()
    m = pc.models[0]
    orc = gpu_oracle(cfg, m, sd, zend, zcen, cls=O.BitSwapOracle)
    for b in sorted(set(int(v) for v in np.linspace(0, B - 1, nsample).round())):
        want = orc.encode_image(O.CState(w, head), imgs[b]).to_list()
        assert got[b] == want, f"{name}: stream {b} differs from the oracle"
    out = pc.decode(ss, B)
    torch.cuda.synchronize()
    ss.raise_on_error()
    assert np.array_equal(out.cpu().numpy(), imgs) and ss.export_lists() == init


def test_kernel_width_containers_edge_coded_roundtrip():
    """Odd-sized RGB images through a tensor-core PipelinedCodec of a kernel-7, padded-width-192 model: exact round trip."""
    cfg = RECURSION["k7 W150"]
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    rs = np.random.RandomState(9)
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(28, 28), (1, 1), (33, 5), (40, 70), (64, 31)]]
    pc = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), 16, lanes=2, free_running=True)
    conts = compress_images(pc, images, excess_state_len=3000, edges="code")
    back = decompress_images(pc, conts, channels=3)
    for img, rec in zip(images, back):
        assert rec.shape == img.shape and np.array_equal(rec, img), img.shape
