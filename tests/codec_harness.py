"""Models, codecs, containers and the oracle recursion driven by the GPU nets -- TEST INFRASTRUCTURE.

`setup` builds the synthetic model, bins and codec of a preset; `gpu_oracle` is the oracle recursion (torch-CUDA float64
pmfs, the C coder) with the GPU nets injected, so that its states are comparable bit for bit with the device's; the chain
helpers run the reference demo procedure (demo_compress.py:113-162) on the oracle and a lone chain on the device.  Imports
without a GPU."""
import collections
import json
import os

import numpy as np
import torch

from edge_oracle import EdgeOracle
from oracle import oracle as O
from bitswap_b200 import synthetic
from bitswap_b200.codec import BitSwapCodec, Bins, BITSWAP
from bitswap_b200.config import CodecConfig, preset, with_
from bitswap_b200.container import extract_edge_blocks
from bitswap_b200.model import Model
from bitswap_b200.rand import ImageBins
from bitswap_b200.streams import StreamSet

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-4          # north_star: per-latent mu/sigma within 1e-4 of the reference torch model

Setup = collections.namedtuple("Setup", "cfg model sd zend zcen bins codec")


def model(cfg, max_batch, tc=False):
    """The synthetic model of cfg (state dict seed 50), loaded and compressed: (model, state dict)."""
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    m = Model.from_config(cfg, max_batch=max_batch, use_tensor_cores=tc).load_state_dict(sd)
    m.compress()
    return m, sd


def setup(name, B, *, q=None, tc=False):
    """Preset `name` (at quantbits q if given): its model, the synthetic bins (seed 0) and a BitSwapCodec of max_batch B."""
    cfg = preset(name) if q is None else with_(preset(name), quantbits=q)
    m, sd = model(cfg, B, tc)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    bins = Bins(cfg, zend, zcen)
    return Setup(cfg, m, sd, zend, zcen, bins, BitSwapCodec(cfg, m, bins, B))


def random_images(C, sizes, seed):
    """Random uint8 HWC images of the given (h, w) and C channels."""
    rs = np.random.RandomState(seed)
    return [rs.randint(0, 256, (h, w, C)).astype(np.uint8) for h, w in sizes]


# ---- the oracle recursion on the GPU nets -----------------------------------------------------------------------------------
def gpu_oracle(cfg, m, sd, zend, zcen, cls=EdgeOracle, record=None):
    """The oracle recursion (cls: EdgeOracle or O.BitSwapOracle) with model m's nets in place of its own and the reference's
    float64 table expression on torch-CUDA: its states are the device's, bit for bit.  record: the oracle's per-chain
    bookkeeping (restbits, excess_state_len, push lengths)."""
    orc = cls(cfg, O.ModelOracle(cfg, sd), zend, zcen, coder="c", pmf="cuda", record=record)

    def gpu_net(kind, level, given):
        f = m.infer(level) if kind == "infer" else m.generate(level)
        mu, sc = f(given.cuda())
        return mu.cpu(), sc.cpu()
    orc._net = gpu_net
    return orc


def oracle_chain(orc, blocks, extents, scheme, n_init=3000):
    """The reference demo procedure (demo_compress.py:113-162) run by the oracle on one chain's blocks, from the seeded
    initial state: (the words above the lowest depth any pop reached, head)."""
    wds, head = synthetic.initial_words(n_init, seed=100)
    st = O.CState(wds, head)
    low = st.n
    pops = []
    orc.trace = pops
    enc = orc.encode_image if scheme == BITSWAP else orc.encode_image_bbans
    for k, b in enumerate(blocks):
        st = enc(st, b.transpose(2, 0, 1), extent=None if extents is None else (int(extents[k][0]), int(extents[k][1])))
    orc.trace = None
    low = min([ln - 1 for tag, ln, _ in pops if tag.startswith("pop")] + [low])
    return np.asarray(st.words[low:st.n], dtype=np.uint32), int(st.head)


def demo_oracle_container(orc, img, n_init):
    """The reference demo procedure (demo_compress.py:113-162,268-284) run by the oracle on one image, with extents: the
    edge-coded single-chain container."""
    blocks, extents, h, w = extract_edge_blocks(img)
    words, head = oracle_chain(orc, blocks, extents, BITSWAP, n_init)
    tail = np.array([head & 0xffffffff, head >> 32, len(blocks), h, w], dtype=np.uint64)
    return np.concatenate([words, tail.astype(np.uint32)])


def lone_chain(codec, blocks, extents, scheme, n_init=4000):
    """One chain coded on a stream set of its own, one block per call: (the words above the lowest depth, head).  The
    blocks and extents stay on the device until the lanes are joined: a free-running codec reads them on its own streams."""
    wds, head = synthetic.initial_words(n_init, seed=100)
    ss = StreamSet(1, n_init + 1400 * len(blocks) + 64, device=codec.device)
    ss.fill(wds, head)
    x = torch.from_numpy(np.ascontiguousarray(blocks.transpose(0, 3, 1, 2))).cuda()
    e = None if extents is None else torch.from_numpy(np.ascontiguousarray(extents, dtype=np.int16)).cuda()
    for k in range(len(blocks)):
        codec.encode(ss, x[k:k + 1], scheme=scheme, extent=None if e is None else e[k:k + 1])
    if hasattr(codec, "join"):
        codec.join()
    torch.cuda.synchronize()
    ss.raise_on_error()
    words, offs, heads, _ = ss.export()
    return words[ss.min_words()[0]:offs[1]], int(heads[0])


def chains_of(unpacked):
    """[(words, head, nblocks)] of an unpacked container or archive (unpack_container / unpack_archive), in block order."""
    words, offs, heads, nblocks = unpacked[:4]
    return [(words[offs[k]:offs[k + 1]], int(heads[k]), int(nblocks[k])) for k in range(len(heads))]


# ---- codec stand-ins --------------------------------------------------------------------------------------------------------
class Counting:
    """Codec proxy counting decode calls and the blocks they pop."""

    def __init__(self, codec):
        self.codec, self.calls, self.blocks = codec, 0, 0

    def __getattr__(self, name):
        return getattr(self.codec, name)

    def decode(self, ss, count, **kw):
        self.calls += 1
        self.blocks += count
        return self.codec.decode(ss, count, **kw)


class NoDevice:
    """A codec stand-in that fails the test if anything on it is touched."""

    def __getattr__(self, name):
        raise AssertionError(f"codec.{name} touched")


# ---- the nets ---------------------------------------------------------------------------------------------------------------
def tc_case(cfg, B, seed=4, dtype=torch.float32):
    """Every infer(i) / generate(i) of cfg's synthetic nets on the tensor cores against the torch oracle (dtype) and the SIMT
    path, with a row alone bit-identical to the same row in the batch: (worst error vs the oracle, vs SIMT)."""
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    m_tc = Model.from_config(cfg, max_batch=B, use_tensor_cores=True).load_state_dict(sd)
    m_si = Model.from_config(cfg, max_batch=B, use_tensor_cores=False).load_state_dict(sd)
    m_tc.compress(); m_si.compress()
    orc = O.ModelOracle(cfg, sd, dtype=dtype)
    rs = np.random.RandomState(seed)
    worst_o = worst_s = 0.0
    for i in range(cfg.nz):
        gx = torch.from_numpy((rs.randint(0, 256, (B, cfg.xdim)) - 127.5) / 127.5) if i == 0 else \
            torch.from_numpy(rs.uniform(-5, 5, (B, cfg.zdim)))
        gz = torch.from_numpy(rs.uniform(-5, 5, (B, cfg.zdim)))
        for kind, g in (("infer", gx), ("generate", gz)):
            f = lambda mm: (mm.infer(i) if kind == "infer" else mm.generate(i))     # noqa: E731
            mu, sc = f(m_tc)(g.cuda())
            mu_s, sc_s = f(m_si)(g.cuda())
            mu_o, sc_o = f(orc)(g)
            worst_o = max(worst_o, (mu.cpu() - mu_o).abs().max().item(), (sc.cpu() - sc_o).abs().max().item())
            worst_s = max(worst_s, (mu - mu_s).abs().max().item(), (sc - sc_s).abs().max().item())
            mu1, sc1 = f(m_tc)(g[B - 1:].cuda())           # batch invariance: last row alone, bit-identical
            assert torch.equal(mu1[0], mu[B - 1]) and torch.equal(sc1[0], sc[B - 1])
    return worst_o, worst_s


# ---- golden files -----------------------------------------------------------------------------------------------------------
def bitswap_golden(name):
    """The reference-classes Bit-Swap run of preset `name` (tests/golden/bitswap_{name}.json)."""
    return json.load(open(os.path.join(GOLDEN, f"bitswap_{name}.json")))


def golden_model(name):
    """(config, arrays) of the reference Model's outputs tests/golden/model_{name}.npz."""
    g = np.load(os.path.join(GOLDEN, f"model_{name}.npz"))
    c = json.loads(str(g["cfg"]))
    c["xs"] = tuple(c["xs"])
    return CodecConfig(**c), g


def model_oracle_vs_golden(name, net, tol):
    """Runs net(kind, level, given [1, dim] float64) -> (mu, scale) on the golden inputs of `name`; every output within
    tol(want) of the reference's."""
    cfg, g = golden_model(name)
    _, zcen = synthetic.synthetic_bins(cfg, seed=0)
    xcen = ImageBins(torch.float64, "cpu", cfg.xdim).centres()
    zr = torch.arange(cfg.zdim)
    worst = 0.0
    for i in range(cfg.nz):
        if i == 0:
            given = xcen[torch.arange(cfg.xdim), torch.from_numpy(g["x"].astype(np.int64))]
        else:
            given = zcen[i - 1, zr, torch.from_numpy(g[f"zsym_in_infer{i}"].astype(np.int64))]
        z = zcen[i, zr, torch.from_numpy(g[f"zsym_in_gen{i}"].astype(np.int64))]
        for kind, inp, key in (("infer", given, f"infer{i}"), ("generate", z, f"gen{i}")):
            mu, sc = net(kind, i, inp.unsqueeze(0))
            for got, want in ((mu, g[key + "_mu"]), (sc, g[key + "_scale"])):
                err = np.abs(got[0].detach().cpu().double().numpy() - want)
                worst = max(worst, float(err.max()))
                assert np.all(err < tol(want)), f"{name} {key}: max |err| {err.max():.3e}"
    return worst


KW_MODELS = ["kw_k5_w100", "kw_k1_w12", "kw_k7_w16"]       # tests/golden/make_golden_kw.py
WIDE_MODELS = ["wide_k3_w320", "wide_k7_w512"]             # tests/golden/make_golden_wide.py
