"""The per-layer float64 harness (P3c) of the conv suites -- TEST INFRASTRUCTURE.

`bsw_selftest_conv` runs one conv of a loaded model through the dispatch the nets use (tensor-core dense conv, in-conv or
head; SIMT in-conv + bf16 split; SIMT head; the SIMT path of a float32 model), fed float32 inputs made here.  The
reference is the same conv in float64 on those inputs, with the weights folded as the product folds them at load.

For every output element, with y the float64 pre-activation and s = sqrt(sum_k (a_k w_k)^2 + b^2 (+ residual^2)) the
l2 norm of the terms summed into it, a `Case` asserts

    |out - f(y)| <= tau * s + TAU_ABS * (ELUs applied) + REL * |f(y)|

f is the epilogue (ELU, the scale transforms, the identity).  TAU_ABS covers the hardware-ex2 ELU of the tensor-core
epilogue (2.4e-7, DESIGN 5.2); REL is the float32 rounding of the result itself.  tau is set per path from measurement
(DESIGN 3, P3c).  Exact checks: the bf16 planes are the RNE split of the trunk where A = T; padded channels are exact
zeros; rows >= n of every output buffer keep their fill and every row < n is written.

`conv_mode` is the one place that sets the process-global conv mode; it restores the default however the block ends.
Imports without a GPU.
"""
import contextlib

import numpy as np
import pytest
import torch

from oracle import oracle as O
from bitswap_b200 import synthetic
from bitswap_b200.config import CodecConfig
from bitswap_b200.model import Model
from bitswap_b200._lib import lib, check, cuda_stream_ptr

RESID, T, T_ELU, A, A_ELU = 1, 2, 4, 8, 16          # BSW_CONV_* of include/bitswap_b200.h
CONV1 = A | A_ELU                                    # conv1: A = ELU(raw)
CONV2_FORMS = {
    "conv2 mid-block": RESID | T | A | A_ELU,         # trunk += raw in place, A = ELU(T)
    "conv2 block end": RESID | T | T_ELU | A | A_ELU,   # T = ELU(trunk + raw), A = ELU(T)
    "conv2 before a tensor-core head": RESID | T | T_ELU | A,   # planes = the ELU'd trunk itself
    "conv2 before a SIMT head": RESID | T | T_ELU,    # no next-conv input
}
IN_FORM = T | T_ELU | A | A_ELU                      # in-conv of a net with ResNet layers

# Bars, normalised by s, over the whole matrix on an H100 80GB HBM3 (DESIGN 3, P3c): tensor cores measured 2^-14.3
# (dense 5x5), bar 2^-13 -- a margin of 2.5, not 4, because 2^-12 would leave the head constant log(e - 1) truncated
# to 0.5413f undetected; SIMT measured 2^-15.8 (dense 5x5, 6400 sequential FMAs), bar 2^-14.  The inputs are seeded
# and the kernels deterministic, so the measured worst is reproducible bit for bit.
TAU = {"tc": 2.0 ** -13, "simt": 2.0 ** -14}
TAU_ABS = 2.0 ** -21
REL = 2.0 ** -22
SPLIT_REL = 2.0 ** -17                               # hi + lo represents a float32 value to 2^-18 relative

MODES = (0, 7, 8, 15)                                # per-tile / persistent grids, with and without TMA multicast
BATCHES = (1, 5, 170)                                # 170: several images per persistent cluster, uneven clusters
MAXB = 173                                           # three rows beyond the largest batch stay untouched
CANARY = 0x7FC5A5A5                                  # quiet-NaN fill of every output buffer
# net-like | wide dynamic range | cancelling channel pairs | head biases across [-30, 30]
VALUES = ("netlike", "wide", "cancel", "saturate")


def conv_cfg(C, zc, W, ks=3, cond=False, nz=2):
    return CodecConfig(xs=(C, 32, 32), nz=nz, zchannels=zc, nprocessing=1, resdepth=2, reswidth=W, kernel_size=ks,
                       cond_xscale=cond)


@contextlib.contextmanager
def conv_mode(mode):
    """Run the block in conv mode `mode` (-1: the default), then restore the default."""
    check(lib().bsw_set_conv_mode(mode))
    try:
        yield
    finally:
        check(lib().bsw_set_conv_mode(-1))


def outputs_in_conv_modes(cfg, B, modes, seed=4):
    """A tensor-core model of cfg (synthetic weights, seed 61) at max_batch B: mu and sigma of every infer(i) and
    generate(i) on seeded pixel and latent inputs, in each conv mode -> {mode: [tensors]}."""
    sd = synthetic.synthetic_state_dict(cfg, seed=61, varied=True)
    m = Model.from_config(cfg, max_batch=B, use_tensor_cores=True).load_state_dict(sd)
    m.compress()
    rs = np.random.RandomState(seed)
    gx = torch.from_numpy((rs.randint(0, 256, (B, cfg.xdim)) - 127.5) / 127.5).cuda()
    gz = torch.from_numpy(rs.uniform(-5, 5, (B, cfg.zdim))).cuda()
    out = {}
    for mode in modes:
        with conv_mode(mode):
            res = []
            for i in range(cfg.nz):
                mu, sc = m.infer(i)(gx if i == 0 else gz)
                res += [mu.clone(), sc.clone()]
                mu, sc = m.generate(i)(gz)
                res += [mu.clone(), sc.clone()]
            torch.cuda.synchronize()
            out[mode] = res
    return out


def worst_report(title, worst):
    """A module-scoped fixture that prints `worst` ({([tag,] path, kind): worst normalised error}) under `title` once
    the module's tests are done."""
    @pytest.fixture(scope="module", autouse=True)
    def _report(request):
        yield
        tr = request.config.pluginmanager.getplugin("terminalreporter")
        capman = request.config.pluginmanager.getplugin("capturemanager")
        if tr is None or capman is None or not worst:
            return
        with capman.global_and_fixture_disabled():
            tr.write_line("")
            tr.write_line(title)
            for (*tag, path, kind), v in sorted(worst.items()):
                tr.write_line("  " + "".join(f"{t:10s} " for t in tag) + f"{path:4s} {kind:16s} {v:.3e}  "
                              f"(2^{np.log2(v) if v > 0 else float('-inf'):.1f}, bar 2^{np.log2(TAU[path]):.0f})")
    return _report


# ---------------------------------------------------------------------------------------------------------------
# inputs and weights
# ---------------------------------------------------------------------------------------------------------------
def _bits_mix(x, rs):
    """Some exact zeros, some bf16-exact values (lo = 0), some whose low 16 bits sit on the bf16 split's RNE tie."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).copy()
    u = rs.uniform(size=b.shape)
    b[u < 0.1] = 0
    m = (u >= 0.1) & (u < 0.2)
    b[m] &= np.uint32(0xFFFF0000)
    m = (u >= 0.2) & (u < 0.3)
    b[m] = (b[m] & np.uint32(0xFFFF0000)) | np.uint32(0x8000)
    return b.view(np.float32)


def _wide_scales(rs, shape):
    """Per-(image, channel) scales 2^U(-10, 6); every fourth image is quiet (2^-10 more), so its outputs have small s."""
    sc = np.exp2(rs.uniform(-10, 6, shape))
    sc[3::4] *= 2.0 ** -10
    return sc


def _hidden(vs, n, W, rs, elu=True):
    """float32 NHWC [n, 256, 256-padded] activations (elu) or trunk values, distinct per image, padded channels zero."""
    x = rs.standard_normal((n, 256, W))
    if elu:
        x = np.where(x > 0, x, np.expm1(x))
    if vs == "wide":
        x = _bits_mix(x * _wide_scales(rs, (n, 1, W)), rs)
    elif vs == "cancel":
        if not elu:
            x = np.zeros_like(x)                   # the residual would dominate s
        x[:, :, 1::2] = x[:, :, 0:2 * (W // 2):2]  # channel pairs equal, their weights nearly opposite
    out = np.zeros((n, 256, -(-W // 64) * 64), np.float32)
    out[..., :W] = x
    return out


def _given(vs, kind, cfg, n, rs):
    """flat CHW `given` of an in-conv: pixel centres (x) or latents in [-5, 5] (z)."""
    if kind == "in_x":
        C = cfg.xs[0]
        g = (rs.randint(0, 256, (n, C, 1024)) - 127.5) / 127.5
        if vs == "wide":
            g = _bits_mix(rs.standard_normal((n, C, 1024)) * _wide_scales(rs, (n, C, 1)), rs)
        elif vs == "cancel":
            g = g.reshape(n, C, 32, 32)
            g[..., 1::2] = g[..., 0::2]            # Squeeze2d channel pairs (fw = 0, 1) equal
    else:
        zc = cfg.zchannels
        g = rs.uniform(-5, 5, (n, zc, 256))
        if vs == "wide":
            g = _bits_mix(rs.standard_normal((n, zc, 256)) * _wide_scales(rs, (n, zc, 1)), rs)
        elif vs == "cancel":
            g[:, 1::2] = g[:, 0:2 * (zc // 2):2]
    return np.ascontiguousarray(np.asarray(g, np.float32).reshape(n, -1))


def _state_dict(cfg, vs, seed):
    """Synthetic weights (v ~ N(0, 0.05), the production gain ranges), then per value set: per-output-channel weight
    scales 2^[-6, 6] (wide), input-channel pairs with nearly opposite weights and no bias (cancel), head biases
    U(-30, 30) (saturate)."""
    sd = synthetic.synthetic_state_dict(cfg, seed=seed, varied=True)
    rs = np.random.RandomState(seed + 1)
    for key in [k for k in sd if k.endswith(".v")]:
        p = key[:-2]
        v, g, b = sd[key].numpy().astype(np.float64), sd[p + ".gain"].numpy().astype(np.float64), sd[p + ".b"].numpy().astype(np.float64)
        if vs == "wide":
            k = rs.randint(-6, 7, size=g.shape)
            if p.endswith(".conv2"):
                g = g * 2.0 ** k
            else:                                  # softplus(gain) * 2^k, through the inverse softplus
                g = np.log(np.expm1(np.logaddexp(0.0, g) * 2.0 ** k))
        elif vs == "cancel":
            I = v.shape[1]
            v[:, 1::2] = -v[:, 0:2 * (I // 2):2] * (1 + 2.0 ** -8 * rs.standard_normal(v[:, 1::2].shape))
            b[:] = 0
        elif vs == "saturate" and ("_mu" in p or "_std" in p):
            b = rs.uniform(-30, 30, b.shape)
        for name, a in ((".v", v), (".gain", g), (".b", b)):
            sd[p + name] = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    return sd


# ---------------------------------------------------------------------------------------------------------------
# checking
# ---------------------------------------------------------------------------------------------------------------
def _nhwc(t):                      # [n, C, 16, 16] -> [n, 256, C]
    return t.permute(0, 2, 3, 1).reshape(t.shape[0], 256, t.shape[1])


def _nchw(t, W):                   # [n, 256, >= W] -> [n, W, 16, 16]
    return t[..., :W].permute(0, 2, 1).reshape(t.shape[0], W, 16, 16)


def _elu(x):
    return torch.where(x > 0, x, torch.expm1(x))


def _softplus(x):
    return -torch.nn.functional.logsigmoid(-x)


def _where(q):
    """Where the worst normalised error of q [n, 256, C] sits: image, pixel row/column, channel, 32-channel chunk."""
    i = int(torch.argmax(q))
    img, rest = divmod(i, q.shape[1] * q.shape[2])
    p, ch = divmod(rest, q.shape[2])
    r, c = divmod(p, 16)
    edge = "border" if r in (0, 15) or c in (0, 15) else "interior"
    return f"image {img}, pixel row {r} col {c} ({edge}, pixel half {r // 8}), channel {ch} (chunk {ch // 32})"


class Checker:
    def __init__(self, case, path, kind, label):
        self.case, self.path, self.kind, self.label = case, path, kind, label

    def bound(self, what, out, ref, s, elus, rel=REL):
        """out ~ ref within tau * s (+ allowances); all [n, 256, C]."""
        err = (out.double() - ref).abs() - elus * TAU_ABS - rel * ref.abs()
        q = err.clamp_min(0) / s.clamp_min(1e-300)
        q = torch.where(torch.isfinite(out), q, torch.full_like(q, float("inf")))
        w = float(q.max())
        if bool((s > 0).any()):                     # not the absolute-only checks (s = 0)
            self.case.note(self.path, self.kind, w)
        assert w <= TAU[self.path], (f"{self.label} {what}: normalised error {w:.3e} > bar {TAU[self.path]:.3e} at "
                                     f"{_where(q)}")


def _canary(shape):
    return torch.full(shape, CANARY, dtype=torch.int32, device="cuda").view(torch.float32)


def _untouched(t, label):
    assert bool((t.view(torch.int32) == CANARY).all()), f"{label}: written where nothing may be"


def _split(x):
    """The RNE bf16 hi/lo split of float32 x, as uint16 bit patterns."""
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi.view(torch.int16), lo.view(torch.int16)


def _bf16(bits):
    return bits.view(torch.bfloat16).float().double()


# ---------------------------------------------------------------------------------------------------------------
# one model x one value set: every conv kind on it, every form, grid mode and batch
# ---------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


class Case:
    """Model `name` of `models` ({name: (tensor cores?, config)}) on value set `vs`, weights seeded from seed_base and its
    place in the tables.  Its worst normalised errors go into `worst`, keyed (path, kind), or with per_kernel_width
    ("k{ks} Wp{Wp}", path, kind) where the dense conv of the kernel-size blocks ("dense3") is reported as "dense k{ks}".
    plane_width: width of the bf16 plane buffers (default: the padded width).  compare_modes: every output of conv modes
    8 / 15 must be bit-identical to the same run in modes 0 / 7."""

    def __init__(self, models, name, vs, *, seed_base, worst, plane_width=None, compare_modes=False,
                 per_kernel_width=False):
        self.tc, self.cfg = models[name]
        self.name, self.vs = name, vs
        self.seed = seed_base + 17 * list(models).index(name) + VALUES.index(vs)
        self.sd = _state_dict(self.cfg, vs, self.seed)
        self.m = Model.from_config(self.cfg, max_batch=MAXB, use_tensor_cores=self.tc).load_state_dict(self.sd)
        self.W, self.Wp = self.cfg.reswidth, -(-self.cfg.reswidth // 64) * 64
        self.planes = torch.empty((2, MAXB, 256, plane_width or self.Wp), dtype=torch.int16, device="cuda")
        self.modes = MODES if self.tc else (-1,)
        self.worst, self.compare_modes, self.per_kernel_width = worst, compare_modes, per_kernel_width
        self._outs = None

    def note(self, path, kind, w):
        key = (path, kind)
        if self.per_kernel_width:
            ks = self.cfg.kernel_size
            key = (f"k{ks} Wp{self.Wp}", path, f"dense k{ks}" if kind == "dense3" else kind)
        self.worst[key] = max(self.worst.get(key, 0.0), w)

    def path(self, kind):
        if not self.tc:
            return "simt"
        if kind == "in_z" and self.cfg.zchannels > 32:
            return "simt"                           # SIMT in-conv, then the split into the first layer's planes
        if kind.startswith("head") and self.head_outs(kind) > 32:
            return "simt"                           # SIMT head on the float32 trunk
        return "tc"

    def head_outs(self, kind):
        zc, C = self.cfg.zchannels, self.cfg.xs[0]
        return (8 * C if self.cfg.cond_xscale else 4 * C) if kind == "head_x" else 2 * zc

    def hook(self, prefix, inp, n, flags, Tb=None, Ab=None, planes=None, mu=None, sc=None):
        p = lambda t: None if t is None else t.data_ptr()     # noqa: E731
        check(lib().bsw_selftest_conv(self.m.handle, prefix.encode(), inp.data_ptr(), n, flags, p(Tb), p(Ab), p(planes),
                                      p(mu), p(sc), cuda_stream_ptr()))
        if self._outs is not None:
            self._outs.append([t.clone() for t in (Tb, Ab, planes, mu, sc) if t is not None])

    def each_mode(self, fn):
        outs = {}
        for mode in self.modes:
            self._outs = [] if self.compare_modes else None
            with conv_mode(mode):
                fn(f"{self.name} / {self.vs} / mode {mode}")
            outs[mode] = self._outs
        self._outs = None
        if self.compare_modes:
            for a, b in ((0, 8), (7, 15)):
                if a in outs and b in outs:
                    for x, y in zip(sum(outs[a], []), sum(outs[b], [])):
                        assert torch.equal(_bits(x), _bits(y)), f"{self.name} / {self.vs}: mode {b} differs from mode {a}"

    # ---- in-convs and dense convs: NHWC outputs T (float32), A (float32 on SIMT, bf16 planes on the tensor cores) ----
    def hidden(self, kind, prefix, flags, inp, n, y, s, resid, out_planes_written):
        W, Wp = self.W, self.Wp
        path = self.path(kind)
        r, s2 = (y + resid, (s * s + resid * resid).sqrt()) if flags & RESID else (y, s)
        t_true = _elu(r) if flags & T_ELU else r
        a_true = _elu(t_true) if flags & A_ELU else t_true
        n_t = 1 if flags & T_ELU else 0
        n_a = n_t + (1 if flags & A_ELU else 0)

        def run(label):
            label = f"{label} / {kind} {prefix} / n={n} flags={flags}"
            ck = Checker(self, path, kind, label)
            Tb = _canary((n + 3, 256, Wp))
            if flags & RESID:
                Tb[:n, :, :W] = resid.float()
                Tb[:n, :, W:] = 0
            Ab = _canary((n + 3, 256, Wp))
            self.hook(prefix, inp, n, flags, Tb, Ab, self.planes)
            torch.cuda.synchronize()
            _untouched(Tb[n:], label + " T rows >= n")
            _untouched(Ab[n:], label + " A rows >= n")
            if flags & T:
                assert bool((Tb[:n, :, W:] == 0).all()), f"{label}: padded trunk channels not zero"
                ck.bound("T", Tb[:n, :, :W], t_true, s2, n_t)
            else:
                _untouched(Tb[:n], label + " T (not an output)")
            simt_a = (flags & A) and (path == "simt")
            if simt_a:
                assert bool((Ab[:n, :, W:] == 0).all()), f"{label}: padded A channels not zero"
                ck.bound("A", Ab[:n, :, :W], a_true, s2, n_a)
                if flags & T:                       # A from the float32 T, up to the ELU
                    tw = Tb[:n, :, :W].double()
                    ck.bound("A from T", Ab[:n, :, :W], _elu(tw) if flags & A_ELU else tw, torch.zeros_like(s2),
                             1 if flags & A_ELU else 0)
            else:
                _untouched(Ab[:n], label + " A (not written on this path)")
            if out_planes_written:
                hi, lo = self.planes[0], self.planes[1]
                assert bool((hi[n:] == -1).all() and (lo[n:] == -1).all()), f"{label}: planes written at rows >= n"
                val = _bf16(hi[:n]) + _bf16(lo[:n])
                assert bool((val[..., W:] == 0).all()), f"{label}: padded plane channels not zero"
                ck.bound("planes", val[..., :W], a_true, s2, n_a, rel=SPLIT_REL)
                src = Ab[:n] if simt_a else (Tb[:n] if (flags & T) and not (flags & A_ELU) else None)
                if src is not None:                 # planes = the RNE split of a float32 tensor we hold: bit for bit
                    h, l = _split(src)
                    assert torch.equal(hi[:n], h) and torch.equal(lo[:n], l), f"{label}: planes are not the RNE split"
                else:                               # planes = split(ELU(T)): lo within half a bf16 ulp of hi, value within
                    # the ELU bound.  (hi == RNE(hi + lo) need not hold: lo may round up to exactly half an ulp.)
                    assert bool((_bf16(lo[:n]).abs() <= 2.0 ** -8 * _bf16(hi[:n]).abs()).all()), f"{label}: |lo| > ulp(hi) / 2"
                    if flags & T:
                        e = _elu(Tb[:n].double())
                        ck.bound("planes from T", val[..., :W], e[..., :W], torch.zeros_like(s2), 1, rel=SPLIT_REL)
        self.each_mode(run)

    def in_conv(self, kind, prefix, n, rs):
        g = _given(self.vs, kind, self.cfg, n, rs)
        inp = torch.from_numpy(g).cuda()
        x = inp.double().view(n, self.cfg.xs[0], 32, 32) if kind == "in_x" else inp.double().view(n, -1, 16, 16)
        if kind == "in_x":
            x = O._squeeze2(x)
        w, b = O.fold_wn(self.sd, prefix)
        y, s = O.conv_f64(x, w, b)
        self.hidden(kind, prefix, IN_FORM, inp, n, _nhwc(y), _nhwc(s), None, self.tc)

    def dense(self, kind, prefix, n, rs):
        W = self.W
        inp = torch.from_numpy(_hidden(self.vs, n, W, rs)).cuda()
        resid = torch.from_numpy(_hidden(self.vs, n, W, rs, elu=False)[..., :W]).cuda().double()
        x = _nchw(inp.double(), W)
        for conv, forms in ((".conv1", {"conv1": CONV1}), (".conv2", CONV2_FORMS)):
            w, b = O.fold_wn(self.sd, prefix + conv, loggain=conv == ".conv1")
            y, s = O.conv_f64(x, w, b)
            y, s = _nhwc(y), _nhwc(s)
            for flags in forms.values():
                self.hidden(kind, prefix + conv, flags, inp, n, y, s, resid, self.tc and bool(flags & A))

    # ---- heads: mu / scale in flat CHW, compared in the latent NHWC layout ----
    def head(self, kind, prefix, n, rs):
        cfg, W = self.cfg, self.W
        inp = torch.from_numpy(_hidden(self.vs, n, W, rs)).cuda()
        x = _nchw(inp.double(), W)
        std = {"head_infer": "infer_std", "head_deepgen": "deepgen_std.0.0", "head_x": "gen_std.0"}[kind]
        has_sc = kind != "head_x" or cfg.cond_xscale
        y_mu, s_mu = O.conv_f64(x, *O.fold_wn(self.sd, prefix))
        if has_sc:
            y_sc, s_sc = O.conv_f64(x, *O.fold_wn(self.sd, std))
            f = {"head_infer": lambda r: 0.1 + 0.9 * torch.sigmoid(r + 2.0),
                 "head_deepgen": lambda r: 0.1 + 0.9 * _softplus(r + float(np.log(np.exp(1.0) - 1.0))),
                 "head_x": lambda r: (2.0 / 255.0) / 8.0 + _softplus(r)}[kind]
            sc_true = _nhwc(f(y_sc))
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
                ck.bound("scale", latent(sc[:n]), sc_true, _nhwc(s_sc), 1)
            else:
                _untouched(sc[:n], label + " scale (mu-only head)")
        self.each_mode(run)

    def run(self):
        rs = np.random.RandomState(self.seed)
        W = self.W
        convs = [("in_x", "infer_in.1", self.in_conv), ("in_z", "deepgen_in.0.0", self.in_conv),
                 ("dense5", f"infer_res0.0.res{W}layer1", self.dense), ("dense3", f"gen_res1.0.res{W}layer1", self.dense),
                 ("head_infer", "infer_mu", self.head), ("head_deepgen", "deepgen_mu.0.0", self.head),
                 ("head_x", "gen_mu.0", self.head)]
        for n in BATCHES:
            for kind, prefix, fn in convs:
                if self.vs == "saturate" and not kind.startswith("head"):
                    continue                        # only the heads' biases change in this value set
                fn(kind, prefix, n, rs)


