"""The single-pass bf16 arithmetic of the tensor-core convs (Model(..., tc_precision="bf16")).

1. Per layer: every tensor-core conv kind against the float64 conv of its RNE-rounded bf16 operands (conv_harness with
   precision="bf16"): dense 3x3 / 5x5 in the four epilogue forms, the x and z in-convs (the SIMT in-conv + split at
   zchannels 40), the three heads (folding at padded widths >= 320) and SIMT heads after a bf16 trunk; padded widths 64,
   128, 192, 256, 320 and 512, kernels 1 / 3 / 5 / 7; conv modes 0 / 7 / 8 / 15, n in {1, 5, 170}, the four value
   sets.  Bar tau = 2^-13 of the tensor-core path.  Exact: the hi plane is RNE of the epilogue output, the lo plane is
   never written, padded channels are 0, rows >= n are untouched.
2. Invariance: modes 8 / 15 equal 0 / 7 and the persistent grid equals the per-tile grid at B = 170; outputs do not
   depend on batch size or position; switching a model to bf16 and back gives its split outputs bit for bit; bf16 and
   split outputs differ.
3. Whole nets against the float64 oracle: cifar8, mnist2 and the cifar8 layout at W 384 (kernel 3) and W 512 (kernel 7).
4. Codec: Bit-Swap and BB-ANS through PipelinedCodec(tc_precision="bf16") against the oracle recursion driven by the same
   GPU nets, exact round trips, edge-coded containers with chain_blocks, an archive, and an archive decoded in the other
   arithmetic failing its initial-state check.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from codec_harness import gpu_oracle                                   # noqa: E402
from conv_harness import (A, A_ELU, CONV1, CONV2_FORMS, IN_FORM, MAXB, RESID, T, T_ELU, VALUES, Case, Checker,   # noqa: E402
                          _bf16, _canary, _elu, _given, _hidden, _nchw, _nhwc, _softplus, _split, _untouched, conv_cfg,
                          conv_mode, worst_report)
from oracle import oracle as O                                         # noqa: E402
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200._lib import lib, check                               # noqa: E402
from bitswap_b200.config import preset, with_                          # noqa: E402
from bitswap_b200.model import Model                                   # noqa: E402
from bitswap_b200.codec import Bins, PipelinedCodec, BITSWAP, BBANS    # noqa: E402
from bitswap_b200.container import compress_archive, compress_images, decompress_archive, decompress_images   # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402

BSW_TC_SPLIT, BSW_TC_BF16 = 0, 1
BF16_REL = 2.0 ** -8                         # RNE to bf16 (8 significant bits): half an ulp, relative


def _rne(t):
    """float32 values (or float64 holding float32 values) rounded to nearest even bf16, as float64."""
    return t.float().to(torch.bfloat16).double()


class Bf16Case(Case):
    """conv_harness.Case on a model in the bf16 arithmetic.  The reference of a conv that runs on the tensor cores is the
    float64 conv of its RNE-rounded bf16 input and folded weights, the operands its one MMA multiplies; convs on the SIMT
    kernel keep the float32 reference.  The next-conv input a tensor-core conv writes is the hi plane alone: RNE of the
    epilogue output, within half a bf16 ulp of the reference, while the lo plane keeps its 0xffff fill.  Everything else
    (inputs, weights, value sets, grid modes, batches, the checks of T and of untouched rows) is the shared harness's."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.m = None                            # the harness's split model, freed before the bf16 one is built
        self.m = Model.from_config(self.cfg, max_batch=MAXB, use_tensor_cores=True,
                                   tc_precision="bf16").load_state_dict(self.sd)
        assert self.tc
        self._planes_ref = None

    def _conv(self, kind, x, w, b):
        if self.path(kind) == "tc":
            x, w = _rne(x), _rne(w)
        return O.conv_f64(x, w, b)

    def in_conv(self, kind, prefix, n, rs):
        inp = torch.from_numpy(_given(self.vs, kind, self.cfg, n, rs)).cuda()
        x = inp.double().view(n, self.cfg.xs[0], 32, 32) if kind == "in_x" else inp.double().view(n, -1, 16, 16)
        if kind == "in_x":
            x = O._squeeze2(x)
        y, s = self._conv(kind, x, *O.fold_wn(self.sd, prefix))
        self.hidden(kind, prefix, IN_FORM, inp, n, _nhwc(y), _nhwc(s), None, True)

    def dense(self, kind, prefix, n, rs):
        W = self.W
        inp = torch.from_numpy(_hidden(self.vs, n, W, rs)).cuda()
        resid = torch.from_numpy(_hidden(self.vs, n, W, rs, elu=False)[..., :W]).cuda().double()
        x = _nchw(inp.double(), W)
        for conv, forms in ((".conv1", {"conv1": CONV1}), (".conv2", CONV2_FORMS)):
            y, s = self._conv(kind, x, *O.fold_wn(self.sd, prefix + conv, loggain=conv == ".conv1"))
            for flags in forms.values():
                self.hidden(kind, prefix + conv, flags, inp, n, _nhwc(y), _nhwc(s), resid, bool(flags & A))

    def head(self, kind, prefix, n, rs):
        cfg, W = self.cfg, self.W
        inp = torch.from_numpy(_hidden(self.vs, n, W, rs)).cuda()
        x = _nchw(inp.double(), W)
        std = {"head_infer": "infer_std", "head_deepgen": "deepgen_std.0.0", "head_x": "gen_std.0"}[kind]
        has_sc = kind != "head_x" or cfg.cond_xscale
        y_mu, s_mu = self._conv(kind, x, *O.fold_wn(self.sd, prefix))
        if has_sc:
            y_sc, s_sc = self._conv(kind, x, *O.fold_wn(self.sd, std))
            f = {"head_infer": lambda r: 0.1 + 0.9 * torch.sigmoid(r + 2.0),
                 "head_deepgen": lambda r: 0.1 + 0.9 * _softplus(r + float(np.log(np.exp(1.0) - 1.0))),
                 "head_x": lambda r: (2.0 / 255.0) / 8.0 + _softplus(r)}[kind]
        dim = cfg.xdim if kind == "head_x" else cfg.zdim

        def latent(t):              # flat CHW output rows -> [n, 256, C]
            t = t.view(n, cfg.xs[0], 32, 32) if kind == "head_x" else t.view(n, -1, 16, 16)
            return _nhwc(O._squeeze2(t) if kind == "head_x" else t)

        def run(label):
            label = f"{label} / {kind} {prefix} / n={n}"
            ck = Checker(self, self.path(kind), kind, label)
            mu, sc = _canary((n + 3, dim)), _canary((n + 3, dim))
            self.hook(prefix, inp, n, 0, mu=mu, sc=sc)
            torch.cuda.synchronize()
            _untouched(mu[n:], label + " mu rows >= n")
            _untouched(sc[n:], label + " scale rows >= n")
            ck.bound("mu", latent(mu[:n]), _nhwc(y_mu), _nhwc(s_mu), 0)
            if has_sc:
                ck.bound("scale", latent(sc[:n]), _nhwc(f(y_sc)), _nhwc(s_sc), 1)
            else:
                _untouched(sc[:n], label + " scale (mu-only head)")
        self.each_mode(run)

    def hidden(self, kind, prefix, flags, inp, n, y, s, resid, out_planes_written):
        """The shared checks of T, A and untouched rows; the hi plane of a tensor-core conv is checked in hook()."""
        if out_planes_written and self.path(kind) == "tc":
            self._planes_ref = (kind, prefix, flags, y, s, resid)
            out_planes_written = False
        try:
            super().hidden(kind, prefix, flags, inp, n, y, s, resid, out_planes_written)
        finally:
            self._planes_ref = None

    def hook(self, prefix, inp, n, flags, Tb=None, Ab=None, planes=None, mu=None, sc=None):
        super().hook(prefix, inp, n, flags, Tb, Ab, planes, mu, sc)
        if self._planes_ref is None:
            return
        kind, _, flags, y, s, resid = self._planes_ref
        W = self.W
        label = f"{self.name} / {self.vs} / {kind} {prefix} / n={n} flags={flags}"
        r, s2 = (y + resid, (s * s + resid * resid).sqrt()) if flags & RESID else (y, s)
        t_true = _elu(r) if flags & T_ELU else r
        a_true = _elu(t_true) if flags & A_ELU else t_true
        n_a = (1 if flags & T_ELU else 0) + (1 if flags & A_ELU else 0)
        ck = Checker(self, "tc", kind, label)
        torch.cuda.synchronize()
        hi, lo = self.planes[0], self.planes[1]
        assert bool((hi[n:] == -1).all()), f"{label}: planes written at rows >= n"
        assert bool((lo == -1).all()), f"{label}: the bf16 arithmetic wrote the lo plane"
        val = _bf16(hi[:n])
        assert bool((val[..., W:] == 0).all()), f"{label}: padded plane channels not zero"
        ck.bound("planes", val[..., :W], a_true, s2, n_a, rel=BF16_REL)
        if (flags & T) and not (flags & A_ELU):          # the planes are the trunk: hi = RNE(T) bit for bit
            assert torch.equal(hi[:n], _split(Tb[:n])[0]), f"{label}: hi plane is not RNE(T)"
        elif flags & T:                                 # hi = RNE(ELU(T)), the ELU by the hardware ex2
            e = _elu(Tb[:n].double())
            ck.bound("planes from T", val[..., :W], e[..., :W], torch.zeros_like(s2), 1, rel=BF16_REL)

# (tensor cores?, config).  zchannels 40: SIMT in-conv + split; heads of more than 32 outputs (2 zchannels > 32) run on
# k_conv_simt after the bf16 trunk.
MODELS = {
    "k3 W64 zc8 C1": (True, conv_cfg(1, 8, 64, 3)),
    "k5 W100 zc40 C3 cond": (True, conv_cfg(3, 40, 100, 5, cond=True)),
    "k1 W192 zc16 C3": (True, conv_cfg(3, 16, 192, 1)),
    "k3 W252 zc8 C3": (True, conv_cfg(3, 8, 252, 3)),
    "k7 W256 zc20 C1 cond": (True, conv_cfg(1, 20, 256, 7, cond=True)),
    "k3 W320 zc2 C3": (True, conv_cfg(3, 2, 320, 3)),
    "k5 W512 zc32 C1 cond": (True, conv_cfg(1, 32, 512, 5, cond=True)),
}
MINE = {}                                    # ("k{ks} Wp{Wp}", path, kind) -> worst normalised error
_report = worst_report("bf16 tensor cores: worst |out - f(y)| / s against the rounded-operand float64 conv", MINE)


@pytest.mark.parametrize("vs", VALUES)
@pytest.mark.parametrize("name", list(MODELS))
def test_bf16_conv_kernels_vs_rounded_operand_float64(name, vs):
    Bf16Case(MODELS, name, vs, seed_base=15000, worst=MINE, compare_modes=True, per_kernel_width=True).run()


@pytest.mark.parametrize("name", ["cifar8", "k5 W384"])
def test_bf16_persistent_grid_equals_per_tile_grid(name):
    """B = 170, bf16: mu and sigma of every net bit-identical in conv modes 0, 7, 8 and 15 (four-CTA clusters with the
    bf16 box split at W 252, folding tiles at W 384)."""
    cfg = preset("cifar8") if name == "cifar8" else conv_cfg(3, 8, 384, 5, nz=3)
    sd = synthetic.synthetic_state_dict(cfg, seed=61, varied=True)
    m = Model.from_config(cfg, max_batch=170, use_tensor_cores=True, tc_precision="bf16").load_state_dict(sd)
    m.compress()
    gx, gz = _inputs(cfg, 170)
    out = {}
    for mode in (0, 7, 8, 15):
        with conv_mode(mode):
            out[mode] = _nets(m, cfg, gx, gz)
    for mode in (7, 8, 15):
        for a, b in zip(out[0], out[mode]):
            assert torch.equal(a, b), f"conv mode {mode}"
    assert all(torch.isfinite(t).all() for t in out[0])


def _nets(m, cfg, gx, gz):
    res = []
    for i in range(cfg.nz):
        for f, g in ((m.infer(i), gx if i == 0 else gz), (m.generate(i), gz)):
            mu, sc = f(g)
            res += [mu.clone(), sc.clone()]
    torch.cuda.synchronize()
    return res


def _inputs(cfg, B, seed=4):
    rs = np.random.RandomState(seed)
    gx = torch.from_numpy((rs.randint(0, 256, (B, cfg.xdim)) - 127.5) / 127.5).cuda()
    gz = torch.from_numpy(rs.uniform(-5, 5, (B, cfg.zdim))).cuda()
    return gx, gz


@pytest.mark.parametrize("name", ["cifar8", "mnist2"])
def test_bf16_batch_position_and_switching(name):
    """Rows do not depend on batch size or position; bf16 -> split -> bf16 on one model reproduces each arithmetic bit
    for bit, and the two arithmetics differ."""
    cfg = preset(name)
    B = 9
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    m = Model.from_config(cfg, max_batch=B, use_tensor_cores=True, tc_precision="bf16").load_state_dict(sd)
    m.compress()
    assert m.tc_precision == "bf16"
    gx, gz = _inputs(cfg, B)
    bf = _nets(m, cfg, gx, gz)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(3)).cuda()
    shuffled = _nets(m, cfg, gx[perm], gz[perm])
    alone = _nets(m, cfg, gx[4:5], gz[4:5])
    for a, s, o in zip(bf, shuffled, alone):
        assert torch.equal(a[perm], s), "a row depends on its position in the batch"
        assert torch.equal(a[4:5], o), "a row depends on the batch size"
    check(lib().bsw_model_set_tc_precision(m.handle, BSW_TC_SPLIT))
    sp = _nets(m, cfg, gx, gz)
    check(lib().bsw_model_set_tc_precision(m.handle, BSW_TC_BF16))
    again = _nets(m, cfg, gx, gz)
    m_split = Model.from_config(cfg, max_batch=B, use_tensor_cores=True).load_state_dict(sd)
    m_split.compress()
    want = _nets(m_split, cfg, gx, gz)
    assert all(torch.equal(a, b) for a, b in zip(sp, want)), "split outputs after bf16 differ from a split model's"
    assert all(torch.equal(a, b) for a, b in zip(again, bf)), "bf16 outputs after split differ from the first bf16 run"
    assert any(not torch.equal(a, b) for a, b in zip(bf, sp)), "bf16 and split arithmetic gave identical outputs"


# Whole nets: the bar is 0.1 on the |mu|, |sigma| deviations from the float64 oracle.  bf16 operands carry up to 2^-9
# relative error per multiply, and it compounds over the in-conv, up to 2 x 8 ResNet convs and the head of a net: on an
# H100 the worst deviation over every output of the four nets below was 2.7e-2 (mu) and 1.3e-2 (sigma), against 7e-5
# for the split arithmetic (DESIGN 5.2).  The bar leaves 3.6x to that and is still far below what a net with a dropped
# tap or a lost k16 half produces (the conv loses a ninth to a half of its sum); the per-layer tests above are the
# tight ones.
NET_BAR = 0.1
NETS = {
    "cifar8": preset("cifar8"),
    "mnist2": preset("mnist2"),
    "cifar8 W384 k3": with_(preset("cifar8"), reswidth=384, kernel_size=3),
    "cifar8 W512 k7": with_(preset("cifar8"), reswidth=512, kernel_size=7),
}


@pytest.mark.parametrize("name", list(NETS))
def test_bf16_nets_vs_float64_oracle(name):
    cfg = NETS[name]
    B = 2
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    m = Model.from_config(cfg, max_batch=B, use_tensor_cores=True, tc_precision="bf16").load_state_dict(sd)
    m_split = Model.from_config(cfg, max_batch=B, use_tensor_cores=True).load_state_dict(sd)
    m.compress(); m_split.compress()
    orc = O.ModelOracle(cfg, sd, dtype=torch.float64, device="cuda")
    gx, gz = _inputs(cfg, B)
    worst_mu = worst_sc = worst_split = 0.0
    for i in range(cfg.nz):
        for kind, g in (("infer", gx if i == 0 else gz), ("generate", gz)):
            f = lambda mm: (mm.infer(i) if kind == "infer" else mm.generate(i))     # noqa: E731
            mu, sc = f(m)(g)
            mu_s, sc_s = f(m_split)(g)
            mu_o, sc_o = f(orc)(g)
            worst_mu = max(worst_mu, (mu.double() - mu_o.to(mu.device)).abs().max().item())
            worst_sc = max(worst_sc, (sc.double() - sc_o.to(sc.device)).abs().max().item())
            worst_split = max(worst_split, (mu_s.double() - mu_o.to(mu.device)).abs().max().item(),
                              (sc_s.double() - sc_o.to(sc.device)).abs().max().item())
    print(f"bf16 {name}: max |mu - oracle| {worst_mu:.3e}, max |sigma - oracle| {worst_sc:.3e} "
          f"(split: {worst_split:.3e})")
    assert worst_mu < NET_BAR and worst_sc < NET_BAR
    assert worst_split < 1e-4


def _pipelined(cfg, B, **kw):
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    return sd, zend, zcen, PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), B, **kw)


@pytest.mark.parametrize("scheme", [BITSWAP, BBANS], ids=["bitswap", "bbans"])
@pytest.mark.parametrize("name", ["cifar8", "tiny3"])
def test_bf16_recursion_vs_oracle_and_roundtrip(name, scheme):
    """PipelinedCodec defaults in bf16, 256 streams over 4 lanes: sampled streams equal the oracle recursion driven by the
    same bf16 GPU nets, and the round trip restores pixels and initial states."""
    B, nsample = 256, 6
    cfg = preset(name)
    sd, zend, zcen, pc = _pipelined(cfg, B, tc_precision="bf16")
    assert pc.lanes == 4 and all(m.tc_precision == "bf16" for m in pc.models)
    imgs = synthetic.synthetic_images(cfg, B, seed=78)
    ss = StreamSet(B, 1 << 15)
    w, head = synthetic.initial_words(20000, seed=100)      # BB-ANS pops all eight cifar8 levels before it pushes
    ss.fill(w, head)
    init = ss.export_lists()
    pc.encode(ss, torch.from_numpy(imgs).cuda(), scheme=scheme)
    torch.cuda.synchronize()
    ss.raise_on_error()
    got = ss.export_lists()
    orc = gpu_oracle(cfg, pc.models[0], sd, zend, zcen, cls=O.BitSwapOracle)
    enc = orc.encode_image if scheme == BITSWAP else orc.encode_image_bbans
    for b in sorted(set(int(v) for v in np.linspace(0, B - 1, nsample).round())):
        assert got[b] == enc(O.CState(w, head), imgs[b]).to_list(), f"{name}: stream {b} differs from the oracle"
    out = pc.decode(ss, B, scheme=scheme)
    torch.cuda.synchronize()
    ss.raise_on_error()
    assert np.array_equal(out.cpu().numpy(), imgs) and ss.export_lists() == init


def test_bf16_containers_archives_and_the_other_arithmetic():
    """Edge-coded multi-chain containers and an archive round-trip exactly in bf16; an archive decoded with a model of the
    other arithmetic fails the initial-state check, both ways."""
    cfg = preset("tiny3")
    rs = np.random.RandomState(9)
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(28, 28), (1, 1), (33, 65), (100, 70), (64, 31)]]
    sd, zend, zcen, bf = _pipelined(cfg, 16, lanes=2, free_running=True, tc_precision="bf16")
    split = PipelinedCodec(cfg, sd, bf.bins, 16, lanes=2)
    conts = compress_images(bf, images, excess_state_len=3000, edges="code", chain_blocks=2)
    for img, rec in zip(images, decompress_images(bf, conts, channels=3)):
        assert rec.shape == img.shape and np.array_equal(rec, img), img.shape
    archives = {}
    for tag, pc in (("bf16", bf), ("split", split)):
        archives[tag] = compress_archive(pc, images, chain_blocks=3, excess_state_len=3000)
        back = decompress_archive(pc, archives[tag])
        assert all(np.array_equal(b, im) for b, im in zip(back, images)), tag
    assert not np.array_equal(archives["bf16"], archives["split"])
    with pytest.raises(ValueError, match="decoded to a state other than the initial one"):
        decompress_archive(split, archives["bf16"])
    with pytest.raises(ValueError, match="decoded to a state other than the initial one"):
        decompress_archive(bf, archives["split"])
