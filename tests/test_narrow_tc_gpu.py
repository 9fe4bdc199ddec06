"""Tensor-core convs of models of padded width 64 (reswidth 1..64: the MNIST models) -- the narrow k_conv_wg tile.

1. P3c on the narrow tile: every conv kind on its own against float64, with the harness of conv_harness.py (same
   inputs, value sets, bar tau = 2^-13 and exact checks), on [2, MAXB, 256, 64] plane buffers; conv modes 8 / 15 (no
   multicast, which narrow launches never use) must be bit-identical to 0 / 7.
2. Whole nets of mnist2/4/8 against the float64 oracle and the SIMT path, batch invariance, persistent == per-tile grid.
3. The Bit-Swap recursion of mnist2 / mnist8 through PipelinedCodec with its defaults (tensor cores) against the oracle.
4. compress_images(edges="code") on 28x28 digits and odd sizes with a tensor-core mnist2 codec: exact round trip.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from codec_harness import TOL, gpu_oracle, tc_case                     # noqa: E402
from conv_harness import VALUES, Case, conv_cfg, outputs_in_conv_modes, worst_report   # noqa: E402
from oracle import oracle as O                                         # noqa: E402
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200.config import preset                                 # noqa: E402
from bitswap_b200.model import Model                                   # noqa: E402
from bitswap_b200.codec import BitSwapCodec, Bins, PipelinedCodec      # noqa: E402
from bitswap_b200.container import compress_images, decompress_images  # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402

# (tensor cores?, config).  zchannels <= 32 run the in-conv on the narrow tile, 40 the SIMT in-conv + split into 64-wide
# planes; heads of <= 32 outputs run on the tensor cores (cchunks = 2), 40 and 80 on k_conv_simt after a narrow trunk.
MODELS = {
    "tc W64 zc1 C1": (True, conv_cfg(1, 1, 64)),                   # MNIST default width
    "tc W61 zc1 C1": (True, conv_cfg(1, 1, 61)),                   # mnist8
    "tc W63 zc2 C3 cond": (True, conv_cfg(3, 2, 63, cond=True)),
    "tc W15 zc8 C3": (True, conv_cfg(3, 8, 15)),                   # 49 padded channels
    "tc W62 zc16 C1": (True, conv_cfg(1, 16, 62)),                 # 32-output tensor-core heads
    "tc W20 zc20 C3": (True, conv_cfg(3, 20, 20)),                 # SIMT heads; the z in-convs have the W -> W shape
    "tc W64 zc40 C1": (True, conv_cfg(1, 40, 64)),                 # SIMT in-conv + split into narrow planes
}
WP = 64
WORST = {}                                   # (path, kind) -> worst normalised error
_report = worst_report("P3c on the narrow tile (padded width 64): worst |out - f(y)| / s (beyond the ELU/rounding allowance)",
                       WORST)


@pytest.mark.parametrize("vs", VALUES)
@pytest.mark.parametrize("name", list(MODELS))
def test_narrow_conv_kernels_vs_float64(name, vs):
    case = Case(MODELS, name, vs, seed_base=5000, worst=WORST, compare_modes=True)
    assert case.Wp == WP
    case.run()


@pytest.mark.parametrize("name", ["mnist2", "mnist4", "mnist8"])
def test_narrow_nets_vs_f64_oracle_and_simt(name):
    """Whole nets on the tensor cores: mu / sigma of every infer(i) / generate(i) within 1e-4 of the float64 oracle and
    of the SIMT path; a row alone equals the same row in the batch, bit for bit."""
    worst_o, worst_s = tc_case(preset(name), 3, dtype=torch.float64)
    print(f"tensor cores {name}: max |err| vs torch-f64 oracle {worst_o:.2e}, vs SIMT f32 path {worst_s:.2e}")
    assert worst_o < TOL and worst_s < TOL


def test_narrow_persistent_grid_equals_per_tile_grid():
    """B = 170: 340 half-image tiles per narrow conv, up to three per CTA on the persistent grid; in-convs with 1 and
    25 taps, dense 3x3 and 5x5, heads.  Bit-identical mu and sigma."""
    out = outputs_in_conv_modes(preset("mnist8"), 170, (0, 7))
    for a, b in zip(out[0], out[7]):
        assert torch.equal(a, b), "conv mode 7"
    assert all(torch.isfinite(t).all() for t in out[7])


@pytest.mark.parametrize("name", ["mnist2", "mnist8"])
def test_narrow_recursion_vs_oracle_and_batch_roundtrip(name):
    """PipelinedCodec with its defaults (tensor-core nets), 256 streams over 4 lanes:
    (a) sampled streams == the oracle recursion driven with the same GPU nets and torch-CUDA float64 pmfs;
    (b) the same images coded by a differently-sized single-lane codec leave identical streams;
    (c) exact pixel round trip, initial states restored."""
    B, nsample = 256, 8
    cfg = preset(name)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    bins = Bins(cfg, zend, zcen)
    pc = PipelinedCodec(cfg, sd, bins, B)
    assert pc.lanes == 4
    imgs = synthetic.synthetic_images(cfg, B, seed=78)
    imgs[1] = imgs[0]
    ss = StreamSet(B, 8192)
    w, head = synthetic.initial_words(4096, seed=100)
    ss.fill(w, head)
    init = ss.export_lists()
    pc.encode(ss, torch.from_numpy(imgs).cuda())
    torch.cuda.synchronize()
    ss.raise_on_error()
    got = ss.export_lists()
    assert got[0] == got[1] and got[0] != got[2]
    sample = sorted(set(int(v) for v in np.linspace(0, B - 1, nsample).round()))
    m = pc.models[0]
    orc = gpu_oracle(cfg, m, sd, zend, zcen, cls=O.BitSwapOracle)
    for b in sample:
        want = orc.encode_image(O.CState(w, head), imgs[b]).to_list()
        assert got[b] == want, f"{name}: stream {b} differs from the oracle"
    m2 = Model.from_config(cfg, max_batch=len(sample), use_tensor_cores=True).load_state_dict(sd)
    m2.compress()
    c2 = BitSwapCodec(cfg, m2, bins, len(sample))
    ss2 = StreamSet(len(sample), 8192)
    ss2.fill(w, head)
    c2.encode(ss2, torch.from_numpy(np.ascontiguousarray(imgs[sample])).cuda())
    torch.cuda.synchronize()
    ss2.raise_on_error()
    assert ss2.export_lists() == [got[b] for b in sample]
    out = pc.decode(ss, B)
    torch.cuda.synchronize()
    ss.raise_on_error()
    assert np.array_equal(out.cpu().numpy(), imgs) and ss.export_lists() == init


def test_narrow_containers_edge_coded_roundtrip():
    """28 x 28 single-channel digits (one partial block each, no Pad(2)) and odd sizes through a tensor-core mnist2
    PipelinedCodec: exact round trip."""
    cfg = preset("mnist2")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    bins = Bins(cfg, zend, zcen)
    rs = np.random.RandomState(9)
    sizes = [(28, 28)] * 4 + [(1, 1), (33, 5), (40, 70), (64, 31)]
    images = []
    for h, w in sizes:
        im = np.zeros((h, w, 1), np.uint8)
        im[h // 5:h - h // 5, w // 4:w - w // 4] = rs.randint(128, 256, (h - 2 * (h // 5), w - 2 * (w // 4), 1))
        images.append(im)
    pc = PipelinedCodec(cfg, sd, bins, 16, lanes=2, free_running=True)
    conts = compress_images(pc, images, excess_state_len=3000, edges="code")
    back = decompress_images(pc, conts, channels=1)
    for img, rec in zip(images, back):
        assert rec.shape == img.shape and np.array_equal(rec, img), img.shape
