"""Models wider than 256 channels (reswidth 257..512, padded widths 320, 384, 448, 512) on the tensor cores and on SIMT.

1. P3c per layer: every conv kind on its own against float64, with the harness of conv_harness.py (same inputs, value
   sets, bars tau = 2^-13 / 2^-14 and exact checks) and the per-kernel-size bookkeeping of test_kernel_width_gpu.py, on
   [2, MAXB, 256, Wp] plane buffers: widths 257..512 at kernel 3, kernels 1 / 5 / 7 at widths 320, 384 and 512 (7x7 at
   512 is the longest sum of any model), and the float32 SIMT path at widths 320 and 512.  Conv modes 8 / 15 must be
   bit-identical to 0 / 7.  The worst normalised error is reported per (path, conv kind, kernel size, padded width).
2. Whole nets against the float64 oracle (1e-4) and the SIMT path, batch invariance, persistent == per-tile grid.
3. The reference pin: Model against the reference's outputs (tests/golden/model_wide_*.npz) within 1e-4.
4. Bit-Swap and BB-ANS through PipelinedCodec defaults against the oracle recursion, exact round trips, and an
   edge-coded container.
5. Widths above 512 are refused on the tensor cores with a message that names the supported range.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from codec_harness import TOL, WIDE_MODELS, golden_model, gpu_oracle, model_oracle_vs_golden, tc_case   # noqa: E402
from conv_harness import VALUES, Case, conv_cfg, outputs_in_conv_modes, worst_report   # noqa: E402
from oracle import oracle as O                                         # noqa: E402
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200.model import Model                                   # noqa: E402
from bitswap_b200.codec import Bins, PipelinedCodec, BITSWAP, BBANS    # noqa: E402
from bitswap_b200.container import compress_images, decompress_images  # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402
from bitswap_b200._lib import BswError                                 # noqa: E402

# (tensor cores?, config).  zchannels <= 32 run the in-conv on the tensor cores, 40 the SIMT in-conv + split; heads of
# <= 32 outputs run on the tensor cores, 40 and 80 on k_conv_simt after a wide tensor-core trunk.
MODELS = {
    # padded widths 320 .. 512 at kernel 3
    "tc k3 W257 zc1 C3": (True, conv_cfg(3, 1, 257, 3)),
    "tc k3 W300 zc20 C1": (True, conv_cfg(1, 20, 300, 3)),
    "tc k3 W320 zc40 C3 cond": (True, conv_cfg(3, 40, 320, 3, cond=True)),
    "tc k3 W384 zc2 C1 cond": (True, conv_cfg(1, 2, 384, 3, cond=True)),
    "tc k3 W400 zc16 C3": (True, conv_cfg(3, 16, 400, 3)),
    "tc k3 W448 zc8 C1": (True, conv_cfg(1, 8, 448, 3)),
    "tc k3 W500 zc32 C3": (True, conv_cfg(3, 32, 500, 3)),
    "tc k3 W512 zc40 C1": (True, conv_cfg(1, 40, 512, 3)),
    # kernel sizes 1 / 5 / 7 at padded widths 320, 384, 512
    "tc k1 W320 zc8 C3": (True, conv_cfg(3, 8, 320, 1)),
    "tc k1 W384 zc40 C1 cond": (True, conv_cfg(1, 40, 384, 1, cond=True)),
    "tc k1 W512 zc2 C3": (True, conv_cfg(3, 2, 512, 1)),
    "tc k5 W320 zc2 C1": (True, conv_cfg(1, 2, 320, 5)),
    "tc k5 W384 zc20 C3 cond": (True, conv_cfg(3, 20, 384, 5, cond=True)),
    "tc k5 W512 zc8 C3": (True, conv_cfg(3, 8, 512, 5)),
    "tc k7 W320 zc16 C3 cond": (True, conv_cfg(3, 16, 320, 7, cond=True)),
    "tc k7 W384 zc1 C1": (True, conv_cfg(1, 1, 384, 7)),
    "tc k7 W512 zc2 C3 cond": (True, conv_cfg(3, 2, 512, 7, cond=True)),
    # the float32 SIMT path above 256 (dense convs too)
    "simt k3 W320 zc8 C3": (False, conv_cfg(3, 8, 320, 3)),
    "simt k3 W512 zc20 C1 cond": (False, conv_cfg(1, 20, 512, 3, cond=True)),
    "simt k7 W320 zc2 C1 cond": (False, conv_cfg(1, 2, 320, 7, cond=True)),
    "simt k7 W512 zc40 C3": (False, conv_cfg(3, 40, 512, 7)),
}
MINE = {}                                    # ("k{ks} Wp{Wp}", path, kind) -> worst normalised error
_report = worst_report("P3c wide models: worst |out - f(y)| / s (beyond the ELU/rounding allowance)", MINE)


@pytest.mark.parametrize("vs", VALUES)
@pytest.mark.parametrize("name", list(MODELS))
def test_wide_conv_kernels_vs_float64(name, vs):
    Case(MODELS, name, vs, seed_base=12000, worst=MINE, compare_modes=True, per_kernel_width=True).run()


NETS = {
    "k3 W320 nz2": conv_cfg(3, 8, 320, 3),
    "k5 W384 nz3 cond": conv_cfg(3, 8, 384, 5, True, nz=3),
    "k1 W448 nz2 zc20": conv_cfg(1, 20, 448, 1),
    "k7 W512 nz2 zc40": conv_cfg(3, 40, 512, 7),
    "k3 W257 nz2 cond": conv_cfg(3, 2, 257, 3, True),
}


@pytest.mark.parametrize("name", list(NETS))
def test_wide_nets_vs_f64_oracle_and_simt(name):
    """Whole nets on the tensor cores: mu / sigma of every infer(i) / generate(i) within 1e-4 of the float64 oracle and
    of the SIMT path; a row alone equals the same row in the batch, bit for bit."""
    worst_o, worst_s = tc_case(NETS[name], 3, dtype=torch.float64)
    print(f"tensor cores {name}: max |err| vs torch-f64 oracle {worst_o:.2e}, vs SIMT f32 path {worst_s:.2e}")
    assert worst_o < TOL and worst_s < TOL


@pytest.mark.parametrize("name", ["k5 W384", "k3 W512"])
def test_wide_persistent_grid_equals_per_tile_grid(name):
    """B = 170: 2040 (Wp 384) / 2720 (Wp 512) tiles per dense conv, many per CTA on the persistent grid; in-convs, dense
    convs with the per-tap fold, heads.  Bit-identical mu and sigma in modes 0, 7, 8 and 15."""
    cfg = {"k5 W384": conv_cfg(3, 8, 384, 5, nz=3), "k3 W512": conv_cfg(1, 2, 512, 3, True, nz=3)}[name]
    out = outputs_in_conv_modes(cfg, 170, (0, 7, 8, 15))
    for mode in (7, 8, 15):
        for a, b in zip(out[0], out[mode]):
            assert torch.equal(a, b), f"conv mode {mode}"
    assert all(torch.isfinite(t).all() for t in out[0])


@pytest.mark.parametrize("tc", [True, False], ids=["tc", "simt"])
@pytest.mark.parametrize("name", WIDE_MODELS)
def test_wide_model_matches_reference(name, tc):
    """Model (tensor cores and SIMT) within 1e-4 of the reference Model's outputs at widths 320 and 512."""
    cfg, _ = golden_model(name)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    m = Model.from_config(cfg, max_batch=1, use_tensor_cores=tc).load_state_dict(sd)
    m.compress()
    worst = model_oracle_vs_golden(name, lambda kind, i, g: (m.infer(i) if kind == "infer" else m.generate(i))(g.cuda()),
                                   lambda want: TOL)
    print(f"{name} {'tensor cores' if tc else 'SIMT'}: max |err| vs the reference {worst:.2e}")


RECURSION = {"k5 W320": conv_cfg(3, 8, 320, 5), "k3 W512": conv_cfg(3, 8, 512, 3, nz=3)}


@pytest.mark.parametrize("scheme", [BITSWAP, BBANS], ids=["bitswap", "bbans"])
@pytest.mark.parametrize("name", list(RECURSION))
def test_wide_recursion_vs_oracle_and_roundtrip(name, scheme):
    """PipelinedCodec with its defaults (tensor-core nets), 256 streams over 4 lanes:
    (a) sampled streams == the oracle recursion driven with the same GPU nets and torch-CUDA float64 pmfs;
    (b) exact pixel round trip, initial states restored."""
    B, nsample = 256, 6
    cfg = RECURSION[name]
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    pc = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), B)
    assert pc.lanes == 4
    imgs = synthetic.synthetic_images(cfg, B, seed=78)
    ss = StreamSet(B, 8192)
    w, head = synthetic.initial_words(4096, seed=100)
    ss.fill(w, head)
    init = ss.export_lists()
    pc.encode(ss, torch.from_numpy(imgs).cuda(), scheme=scheme)
    torch.cuda.synchronize()
    ss.raise_on_error()
    got = ss.export_lists()
    m = pc.models[0]
    orc = gpu_oracle(cfg, m, sd, zend, zcen, cls=O.BitSwapOracle)
    enc = orc.encode_image if scheme == BITSWAP else orc.encode_image_bbans
    for b in sorted(set(int(v) for v in np.linspace(0, B - 1, nsample).round())):
        want = enc(O.CState(w, head), imgs[b]).to_list()
        assert got[b] == want, f"{name}: stream {b} differs from the oracle"
    out = pc.decode(ss, B, scheme=scheme)
    torch.cuda.synchronize()
    ss.raise_on_error()
    assert np.array_equal(out.cpu().numpy(), imgs) and ss.export_lists() == init


def test_wide_containers_edge_coded_roundtrip():
    """Odd-sized RGB images through a tensor-core PipelinedCodec of a kernel-5, padded-width-320 model: exact round trip."""
    cfg = RECURSION["k5 W320"]
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    rs = np.random.RandomState(9)
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(28, 28), (1, 1), (33, 5), (40, 70), (64, 31)]]
    pc = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), 16, lanes=2, free_running=True)
    conts = compress_images(pc, images, excess_state_len=3000, edges="code")
    back = decompress_images(pc, conts, channels=3)
    for img, rec in zip(images, back):
        assert rec.shape == img.shape and np.array_equal(rec, img), img.shape


def test_wide_width_above_512_is_refused_on_the_tensor_cores():
    cfg = conv_cfg(3, 2, 513, 3)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    with pytest.raises(BswError, match=r"reswidth 1\.\.512"):
        Model.from_config(cfg, max_batch=1, use_tensor_cores=True).load_state_dict(sd)
    Model.from_config(cfg, max_batch=1, use_tensor_cores=False).load_state_dict(sd)      # SIMT takes any width
