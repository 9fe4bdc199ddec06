"""oracle/oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement of the reference's Bit-Swap hot path (fhkingma/bitswap @
dfe0bf7d): the rANS coder, the logistic table construction, the inference-time
VAE forward and the sender/receiver recursions.  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module; bitswap_b200/ never does.

Parity status: PINNED against the reference itself.  tests/golden/make_golden.py
ran the reference's own classes (ANS, logistic_cdf, Model) in the build container
and wrote tests/golden/*; tests/test_oracle.py checks every function here
against those files (SURVEY.md 8c: the reference ships no golden vectors).

Two implementations of the integer coder live side by side:
  * `AnsPort`   -- literal Python/NumPy port, same data structures as the
                   reference (Python list state, per-symbol loop).  This is the
                   "reference's own CPU ANS" that bench.py times.
  * `liborc.so` -- oracle/ans_oracle.c, same arithmetic in C, used by the tests
                   for sizes where Python loops would take minutes.
"""
import ctypes
import os
import subprocess

import numpy as np
import torch
import torch.nn.functional as F

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build():
    """Compile oracle/ans_oracle.c -> oracle/liborc.so (idempotent)."""
    so = os.path.join(_HERE, "liborc.so")
    src = os.path.join(_HERE, "ans_oracle.c")
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "liborc.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        c_i64, c_p = ctypes.c_int64, ctypes.c_void_p
        L.orc_logistic_pmfs.argtypes = [c_p, c_p, c_p, c_i64, c_i64, c_i64, c_p]
        L.orc_logistic_pmfs.restype = None
        L.orc_tables.argtypes = [c_p, c_i64, c_i64, ctypes.c_int, ctypes.c_int, c_p, c_p]
        L.orc_push.argtypes = [c_p, c_p, c_i64, c_p, c_p, c_p, c_p, c_i64, c_i64, ctypes.c_int]
        L.orc_pop.argtypes = [c_p, c_p, c_p, c_p, c_p, c_p, c_i64, c_i64, ctypes.c_int]
        _LIB = L
    return _LIB


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ----------------------------------------------------------------------------------------------
# Float side: logistic pmfs (cifar_compress.py:182-184, rand.py:67-68)
# ----------------------------------------------------------------------------------------------

def logistic_pmfs_torch(endpoints, mu, scale):
    """Exactly the reference's tensor expression, on torch CPU float64.
    endpoints [L,S-1]; mu, scale [L] or [1] -> pmfs [L,S]."""
    cdfs = torch.sigmoid((endpoints.t() - mu) / scale).t()
    pmfs = cdfs[:, 1:] - cdfs[:, :-1]
    return torch.cat((cdfs[:, 0].unsqueeze(1), pmfs, 1. - cdfs[:, -1].unsqueeze(1)), dim=1)


def logistic_pmfs_c(endpoints, mu, scale):
    """Same, through ans_oracle.c (libm exp).  numpy f64 in/out."""
    e = np.ascontiguousarray(endpoints, dtype=np.float64)
    mu = np.ascontiguousarray(mu, dtype=np.float64)
    scale = np.ascontiguousarray(scale, dtype=np.float64)
    L, S = e.shape[0], e.shape[1] + 1
    out = np.empty((L, S), dtype=np.float64)
    lib().orc_logistic_pmfs(_ptr(e), _ptr(mu), _ptr(scale), 1 if mu.size > 1 else 0, L, S, _ptr(out))
    return out


# ----------------------------------------------------------------------------------------------
# Integer side: ANS.__init__ / encode / decode (cifar_compress.py:12-67)
# ----------------------------------------------------------------------------------------------

def tables_np(pmfs, bits=31, quantbits=8):
    """ANS.__init__ (cifar_compress.py:25-46) in NumPy.  pmfs f64 [L,S] ->
    (P int64 [L,S], C int64 [L,S+1])."""
    pmfs = np.asarray(pmfs, dtype=np.float64)
    L, S = pmfs.shape
    mult = (1 << bits) - (1 << quantbits)                       # :28
    P = (pmfs * mult).astype(np.int64)                          # :29  .long() truncates toward zero
    P += 1                                                      # :32
    am = np.argmax(P, axis=1)                                   # :35  first maximum, like torch CPU
    P[np.arange(L), am] += (1 << bits) - P.sum(axis=1)
    C = np.zeros((L, S + 1), dtype=np.int64)                    # :38-39
    np.cumsum(P, axis=1, out=C[:, 1:])
    assert np.all(C[:, -1] == (1 << bits))                      # :46
    return P, C


def tables_c(pmfs, bits=31, quantbits=8):
    pmfs = np.ascontiguousarray(pmfs, dtype=np.float64)
    L, S = pmfs.shape
    P = np.empty((L, S), dtype=np.int64)
    C = np.empty((L, S + 1), dtype=np.int64)
    rc = lib().orc_tables(_ptr(pmfs), L, S, bits, quantbits, _ptr(P), _ptr(C))
    if rc:
        raise AssertionError("bad table")
    return P, C


class AnsPort:
    """Literal port of the reference `ANS` class: same constructor, same Python
    list state (words bottom-first, head last), same per-symbol loops."""

    def __init__(self, pmfs, bits=31, quantbits=8):
        self.bits, self.mask = bits, (1 << bits) - 1
        self.seq_len, self.support = pmfs.shape
        self.pmfs, self.cdfs = tables_np(pmfs.detach().cpu().numpy() if torch.is_tensor(pmfs) else pmfs,
                                         bits, quantbits)

    def encode(self, x, symbols):                                # :48-55
        bits = self.bits
        for i, s in enumerate(np.asarray(symbols).tolist()):
            p = int(self.pmfs[i, s])
            if x[-1] >= (((1 << 32) >> bits) << 32) * p:                 # :51
                x.append(x[-1] >> 32)
                x[-2] &= 0xffffffff
            x[-1] = ((x[-1] // p) << bits) + (x[-1] % p) + int(self.cdfs[i, s])
        return x

    def decode(self, x):                                         # :57-67
        seq = np.zeros(self.seq_len, dtype=np.int64)
        for i in range(self.seq_len - 1, -1, -1):
            m = x[-1] & self.mask
            s = int(np.searchsorted(self.cdfs[i, :-1], m, 'right')) - 1
            seq[i] = s
            x[-1] = int(self.pmfs[i, s]) * (x[-1] >> self.bits) + m - int(self.cdfs[i, s])
            if x[-1] < (1 << 32):
                x[-1] = (x[-1] << 32) | x.pop(-2)               # IndexError when the stack is empty
        return x, torch.from_numpy(seq)


class AnsC:
    """Same interface on the C oracle.  State = (words uint32 array with spare
    capacity, n, head) wrapped in `CState`."""

    def __init__(self, pmfs=None, bits=31, quantbits=8, tables=None):
        self.bits = bits
        if tables is None:
            pm = pmfs.detach().cpu().numpy() if torch.is_tensor(pmfs) else pmfs
            tables = tables_c(pm, bits, quantbits)
        self.P, self.C = (np.ascontiguousarray(t, dtype=np.int64) for t in tables)
        self.seq_len, self.support = self.P.shape

    def encode(self, st, symbols):
        sym = np.ascontiguousarray(np.asarray(symbols), dtype=np.int64)
        n = ctypes.c_int64(st.n)
        head = ctypes.c_uint64(st.head)
        rc = lib().orc_push(_ptr(st.words), ctypes.byref(n), st.words.size, ctypes.byref(head),
                            _ptr(self.P), _ptr(self.C), _ptr(sym), self.seq_len, self.support, self.bits)
        if rc:
            raise OverflowError("oracle stack capacity")
        st.n, st.head = n.value, head.value
        return st

    def decode(self, st):
        sym = np.empty(self.seq_len, dtype=np.int64)
        n = ctypes.c_int64(st.n)
        head = ctypes.c_uint64(st.head)
        rc = lib().orc_pop(_ptr(st.words), ctypes.byref(n), ctypes.byref(head),
                           _ptr(self.P), _ptr(self.C), _ptr(sym), self.seq_len, self.support, self.bits)
        st.n, st.head = n.value, head.value
        if rc:
            raise IndexError("pop from empty ANS stack")
        return st, sym


class CState:
    def __init__(self, words, head, cap=None):
        words = np.asarray(words, dtype=np.uint32)
        cap = cap or max(2 * words.size, words.size + (1 << 16))
        self.words = np.zeros(cap, dtype=np.uint32)
        self.words[:words.size] = words
        self.n, self.head = int(words.size), int(head)

    @classmethod
    def from_list(cls, x, cap=None):
        return cls(np.array(x[:-1], dtype=np.uint64).astype(np.uint32), x[-1], cap)

    def to_list(self):
        return [int(w) for w in self.words[:self.n]] + [int(self.head)]

    def copy(self):
        c = CState(self.words[:self.n], self.head, self.words.size)
        return c

    def digest(self):
        return state_digest(self.words[:self.n], self.head)


def state_digest(words, head):
    """First 16 hex of sha256(uint32 words || uint64 head) (SURVEY.md 8c)."""
    import hashlib
    b = np.asarray(words, dtype=np.uint32).tobytes() + np.array([head], dtype=np.uint64).tobytes()
    return hashlib.sha256(b).hexdigest()[:16]


# ----------------------------------------------------------------------------------------------
# Model forward, inference-time only (model/cifar_train.py:315-438, utils/torch/modules.py:98-241)
# ----------------------------------------------------------------------------------------------

def _wn(sd, prefix, loggain=True):
    """Weight-normalised kernel (modules.py:98-105)."""
    v, gain = sd[prefix + ".v"], sd[prefix + ".gain"]
    g = -F.logsigmoid(-gain) if loggain else gain                 # softplus, modules.py:112-114
    vnorm = v.view(v.shape[0], -1).norm(p=2, dim=1)
    return v * (g / (vnorm + 1e-10)).view(-1, 1, 1, 1), sd[prefix + ".b"]


def _conv(sd, prefix, x, loggain=True):
    w, b = _wn(sd, prefix, loggain)
    return F.conv2d(x, w, b, stride=1, padding=(w.shape[-1] - 1) // 2)


def _resblock(sd, prefix, x, W, n):
    """ResNetBlock of n ResNetLayers: x + conv2(ELU(conv1(ELU(x)))) (modules.py:229-241)."""
    for l in range(1, n + 1):
        p = f"{prefix}.res{W}layer{l}"
        c1 = F.elu(_conv(sd, p + ".conv1", F.elu(x)))
        x = x + _conv(sd, p + ".conv2", c1, loggain=False)
    return x


def _squeeze2(x):      # modules.py:175-186  out ch = c*4 + fh*2 + fw
    n, c, h, w = x.shape
    return x.view(n, c, h // 2, 2, w // 2, 2).permute(0, 1, 3, 5, 2, 4).reshape(n, c * 4, h // 2, w // 2)


def _unsqueeze2(x):    # modules.py:198-208
    n, c, h, w = x.shape
    return x.view(n, c // 4, 2, 2, h, w).permute(0, 1, 4, 2, 5, 3).reshape(n, c // 4, h * 2, w * 2)


def fold_wn(sd, prefix, loggain=True):
    """The float32 kernel and bias the product folds at load (bsw_model_load_conv): ||v|| summed in float64 and rounded
    to float32, g = softplus(gain) in float64 rounded to float32, then w = v * (g / (||v|| + 1e-10)) in float32."""
    v = sd[prefix + ".v"].detach().cpu().numpy().astype(np.float32)
    gain = sd[prefix + ".gain"].detach().cpu().numpy().astype(np.float32)
    vnorm = np.sqrt((v.reshape(v.shape[0], -1).astype(np.float64) ** 2).sum(1)).astype(np.float32)
    g = gain.astype(np.float64)
    g = (np.maximum(g, 0.0) + np.log1p(np.exp(-np.abs(g)))).astype(np.float32) if loggain else gain
    scale = g / (vnorm + np.float32(1e-10))
    w = v * scale.astype(np.float32)[:, None, None, None]
    return torch.from_numpy(w.astype(np.float32)), sd[prefix + ".b"].detach().cpu().float()


def conv_f64(x, w, b=None):
    """One "same" convolution in float64, and the l2 norm of its products: (y, s) with y = conv(x, w) + b and
    s = sqrt(sum_k (x_k w_k)^2 + b^2) per output element, the scale a correctly rounded float32-accurate conv is held to
    (normalising by s rather than |y| keeps outputs where the terms cancel testable)."""
    x, w = x.double(), w.double().to(x.device)
    pad = (w.shape[-1] - 1) // 2
    y = F.conv2d(x, w, None, padding=pad)
    s2 = F.conv2d(x * x, w * w, None, padding=pad)
    if b is not None:
        b = b.double().to(x.device).view(1, -1, 1, 1)
        y, s2 = y + b, s2 + b * b
    return y, s2.sqrt()


class ModelOracle:
    """infer(i)(given) / generate(i)(given) of the reference Model in
    compressing mode, batched over a leading dimension: given [B, dim] (any
    float dtype, flat CHW) -> (mu, scale) float64 [B, dim_out].

    dtype is the arithmetic: float32 (default, the reference's own) or float64, a reference for the float32 kernels
    whose own error is far below theirs.  The input is first rounded to float32, as `given.float()` in the reference
    and the product do.  device places the computation (and the outputs), e.g. "cuda" for large float64 batches."""

    def __init__(self, cfg, state_dict, dtype=torch.float32, device="cpu"):
        self.cfg, self.dtype, self.device = cfg, dtype, torch.device(device)
        self.sd = {k: v.float().to(device=self.device, dtype=dtype) for k, v in state_dict.items()}

    def _given(self, given):
        return given.float().to(device=self.device, dtype=self.dtype)

    @torch.no_grad()
    def infer(self, i):
        cfg, sd, W = self.cfg, self.sd, self.cfg.reswidth
        rd = cfg.level_resdepth

        def distribution(given):
            h = self._given(given)
            if i == 0:                                           # cifar_train.py:326-349
                h = h.view((-1,) + tuple(cfg.xs))
                h = F.elu(_conv(sd, "infer_in.1", _squeeze2(h)))
                if cfg.nprocessing > 0:
                    h = F.elu(_resblock(sd, "infer_res0.0", h, W, cfg.nprocessing))
                if rd[0] > 0:
                    h = F.elu(_resblock(sd, "infer_res1.0", h, W, rd[0]))
                mu = _conv(sd, "infer_mu", h)
                scale = 0.1 + 0.9 * torch.sigmoid(_conv(sd, "infer_std", h) + 2.)
            else:                                                # :352-368
                h = h.view(-1, cfg.zchannels, 16, 16)
                h = F.elu(_conv(sd, f"deepinfer_in.{i-1}.0", h))
                if rd[i] > 0:
                    h = F.elu(_resblock(sd, f"deepinfer_res.{i-1}.0", h, W, rd[i]))
                mu = _conv(sd, f"deepinfer_mu.{i-1}.0", h)
                scale = 0.1 + 0.9 * torch.sigmoid(_conv(sd, f"deepinfer_std.{i-1}.0", h) + 2.)
            B = mu.shape[0]
            return mu.reshape(B, -1).double(), scale.reshape(B, -1).double()     # :375-376
        return distribution

    @torch.no_grad()
    def generate(self, i):
        cfg, sd, W = self.cfg, self.sd, self.cfg.reswidth
        rd = cfg.level_resdepth

        def distribution(given):
            h = self._given(given).view(-1, cfg.zchannels, 16, 16)    # :391-393
            if i == 0:                                           # :396-411
                h = F.elu(_conv(sd, "gen_in.0", h))
                if rd[0] > 0:
                    h = F.elu(_resblock(sd, "gen_res1.0", h, W, rd[0]))
                if cfg.nprocessing > 0:
                    h = F.elu(_resblock(sd, "gen_res0.0", h, W, cfg.nprocessing))
                mu = _unsqueeze2(_conv(sd, "gen_mu.0", h))
                if cfg.cond_xscale:                              # imagenetcrop_train.py:306-315,417
                    pre = _unsqueeze2(_conv(sd, "gen_std.0", h))
                else:
                    pre = sd["gen_std"].unsqueeze(0).expand(mu.shape)
                scale = ((2. / 255.) / 8.) + (-F.logsigmoid(-pre))
            else:                                                # :414-426
                h = F.elu(_conv(sd, f"deepgen_in.{i-1}.0", h))
                if rd[i] > 0:
                    h = F.elu(_resblock(sd, f"deepgen_res.{i-1}.0", h, W, rd[i]))
                mu = _conv(sd, f"deepgen_mu.{i-1}.0", h)
                pre = _conv(sd, f"deepgen_std.{i-1}.0", h) + float(np.log(np.exp(1.) - 1.))
                scale = 0.1 + 0.9 * (-F.logsigmoid(-pre))
            B = mu.shape[0]
            return mu.reshape(B, -1).double(), scale.reshape(B, -1).double()     # :434-435
        return distribution


# ----------------------------------------------------------------------------------------------
# Bits-back schedules (cifar_compress.py:175-250 sender, :283-352 receiver)
# ----------------------------------------------------------------------------------------------

class BitSwapOracle:
    """One chain (= one reference 'experiment'): images are pushed one after
    another onto a single ANS state.  `coder` is AnsPort (list state) or AnsC
    (CState); pmf = "torch" (the reference's expression on torch CPU), "cuda" (the same
    expression on torch CUDA -- how the reference itself runs it) or "c" (libm, ans_oracle.c).

    record: optional dict, the reference's per-chain bookkeeping, filled by every encode of the chain.  All lengths are
    len(state) of the reference's list (words + head, = CState.n + 1):
      init_len    length of the state the chain's first image was coded onto (len(initialstate), cifar_compress.py:159)
      rest_len    len(restbits): the length after the first image's first pop for Bit-Swap (:190-192), after the last of
                  its nz pops for BB-ANS (:224-226); None before that point
      excess_len  demo_compress.py:137 `excess_state_len`: the least length after any pop, starting from init_len
      push_lens   [(trace tag, length)] after every push, in order: the chain's peak depth and the push that reaches it
      images      images coded so far"""

    def __init__(self, cfg, model, zendpoints, zcentres, coder="c", pmf="torch", trace=None, record=None):
        self.cfg, self.model = cfg, model
        self.zend, self.zcen = zendpoints.double(), zcentres.double()
        # ImageBins (utils/torch/rand.py:146-152): 255 inner endpoints, 256 centres, identical for every dimension
        k = torch.arange(1, 256, dtype=torch.float64)
        self.xend = (((k - 127.5) / 127.5) - 1. / 255.)[None,].expand([cfg.xdim, -1])
        k = torch.arange(0, 256, dtype=torch.float64)
        self.xcen = ((k - 127.5) / 127.5)[None,].expand([cfg.xdim, -1])
        self.coder_kind, self.pmf_kind, self.trace, self.record = coder, pmf, trace, record
        self.zr, self.xr = torch.arange(cfg.zdim), torch.arange(cfg.xdim)
        self.mu_hook = None     # optional: callable(kind, level, mu, scale) -> (mu, scale) to inject GPU nets
        self.timers = None      # optional dict: seconds per phase {net, cdf, tables, pop, push} (bench.py's 5-way split, BASELINE.md 3)

    # -- helpers ------------------------------------------------------------------------------
    def _timed(self, name, fn, *a):
        if self.timers is None:
            return fn(*a)
        import time
        t0 = time.perf_counter()
        r = fn(*a)
        self.timers[name] = self.timers.get(name, 0.0) + time.perf_counter() - t0
        return r

    def _pop(self, endpoints, mu, sc, q, state):
        """tables + decode of one level: float64 pmfs (:182-184), ANS.__init__ (:13-46), ANS.decode (:57-67)."""
        pm = self._timed("cdf", self._pmfs, endpoints, mu, sc)
        coder = self._timed("tables", self._coder, pm, q)
        return self._timed("pop", coder.decode, state)

    def _push(self, endpoints, mu, sc, q, state, symbols):
        pm = self._timed("cdf", self._pmfs, endpoints, mu, sc)
        coder = self._timed("tables", self._coder, pm, q)
        return self._timed("push", coder.encode, state, symbols)

    def _pmfs(self, endpoints, mu, scale):
        if self.pmf_kind == "torch":
            return logistic_pmfs_torch(endpoints, mu, scale).numpy()
        if self.pmf_kind == "cuda":
            # the reference's tensor expression evaluated where the reference evaluates it: on the GPU (device=f"cuda:{gpu}",
            # cifar_compress.py:77,182-184).  torch-CUDA's float64 sigmoid is what the product's float64 cdf is bit-matched
            # to, so with this kind EVERY stream must be bit-identical (no 1-ulp libm/Sleef bin flips, SURVEY.md H2).
            return logistic_pmfs_torch(endpoints.cuda(), mu.cuda(), scale.cuda()).cpu().numpy()
        return logistic_pmfs_c(endpoints.numpy(), mu.numpy(), scale.numpy())

    def _coder(self, pmfs, q):
        bits = self.cfg.ansbits
        return AnsPort(pmfs, bits, q) if self.coder_kind == "port" else AnsC(pmfs, bits, q)

    def _net(self, kind, level, given):
        return self._timed("net", self._net_raw, kind, level, given)

    def _net_raw(self, kind, level, given):
        f = self.model.infer(level) if kind == "infer" else self.model.generate(level)
        mu, sc = f(given.unsqueeze(0))
        mu, sc = mu[0], sc[0]
        if self.mu_hook is not None:
            mu, sc = self.mu_hook(kind, level, mu, sc)
        return mu, sc

    def _note(self, tag, st, rest=False):
        """Trace entry and accounting after one pop or push.  rest: this pop is where the reference takes restbits if the
        chain has not taken it yet."""
        n = len(st) if isinstance(st, list) else st.n + 1
        if self.trace is not None:
            if isinstance(st, list):
                self.trace.append((tag, n, state_digest(np.array(st[:-1], dtype=np.uint64).astype(np.uint32), st[-1])))
            else:
                self.trace.append((tag, n, st.digest()))
        r = self.record
        if r is not None:
            if tag.startswith("pop"):
                r["excess_len"] = min(r["excess_len"], n)
                if rest and r["rest_len"] is None:
                    r["rest_len"] = n
            else:
                r["push_lens"].append((tag, n))

    def _begin(self, st):
        """A chain's first encode sets up its record (see the class docstring)."""
        r = self.record
        if r is not None and "init_len" not in r:
            n = len(st) if isinstance(st, list) else st.n + 1
            r.update(init_len=n, rest_len=None, excess_len=n, push_lens=[], images=0)

    def _end(self):
        if self.record is not None:
            self.record["images"] += 1

    def _prior(self):
        c = self.cfg
        return self._pmfs(self.zend[-1], torch.zeros(1, dtype=torch.float64), torch.ones(1, dtype=torch.float64))

    # -- Bit-Swap sender, one image (cifar_compress.py:175-204,244-250) ----------------------------
    def encode_image(self, state, x):
        c = self.cfg
        x = torch.as_tensor(np.asarray(x).reshape(-1).astype(np.int64))
        q = c.quantbits
        zsym = None
        self._begin(state)
        for zi in range(c.nz):
            given = self.zcen[zi - 1, self.zr, zsym] if zi > 0 else self.xcen[self.xr, x]           # :180
            mu, sc = self._net("infer", zi, given)                                                  # :181
            state, zsymtop = self._pop(self.zend[zi], mu, sc, q, state)                             # :182-187
            zsymtop = torch.as_tensor(np.asarray(zsymtop))
            self._note(f"pop z{zi+1}", state, rest=zi == 0)                                         # :190-192 restbits
            z = self.zcen[zi, self.zr, zsymtop]                                                     # :195
            mu, sc = self._net("generate", zi, z)                                                   # :196
            ends = self.zend[zi - 1] if zi > 0 else self.xend                                       # :197
            state = self._push(ends, mu, sc, q if zi > 0 else 8, state, (zsym if zi > 0 else x).numpy())   # :202
            self._note(f"push {'z%d' % zi if zi > 0 else 'x'}", state)
            zsym = zsymtop                                                                          # :204
        state = self._timed("push", self._timed("tables", self._coder, self._timed("cdf", self._prior), q).encode, state, zsym.numpy())   # :245-250
        self._note("push prior", state)
        self._end()
        return state

    # -- Bit-Swap receiver, one image (cifar_compress.py:283-317) -------------------------------
    def decode_image(self, state):
        c = self.cfg
        q = c.quantbits
        state, zsymtop = self._timed("pop", self._timed("tables", self._coder, self._timed("cdf", self._prior), q).decode, state)   # :284-289
        zsymtop = torch.as_tensor(np.asarray(zsymtop))
        for zi in reversed(range(c.nz)):                                                            # :294
            z = self.zcen[zi, self.zr, zsymtop]
            mu, sc = self._net("generate", zi, z)                                                   # :296-297
            ends = self.zend[zi - 1] if zi > 0 else self.xend
            state, sym = self._pop(ends, mu, sc, q if zi > 0 else 8, state)                         # :303
            sym = torch.as_tensor(np.asarray(sym))
            given = self.zcen[zi - 1, self.zr, sym] if zi > 0 else self.xcen[self.xr, sym]          # :306
            mu, sc = self._net("infer", zi, given)                                                  # :307
            state = self._push(self.zend[zi], mu, sc, q, state, zsymtop.numpy())                    # :313
            zsymtop = sym                                                                           # :315
        return state, zsymtop.numpy().astype(np.uint8)

    # -- BB-ANS sender/receiver (cifar_compress.py:205-242, :319-352) ------------------------------
    def encode_image_bbans(self, state, x):
        c = self.cfg
        x = torch.as_tensor(np.asarray(x).reshape(-1).astype(np.int64))
        q = c.quantbits
        zs, zsym = [], None
        self._begin(state)
        for zi in range(c.nz):                                                                      # :209-221
            given = self.zcen[zi - 1, self.zr, zsym] if zi > 0 else self.xcen[self.xr, x]
            mu, sc = self._net("infer", zi, given)
            state, zsym = self._coder(self._pmfs(self.zend[zi], mu, sc), q).decode(state)
            zsym = torch.as_tensor(np.asarray(zsym))
            zs.append(zsym)
            self._note(f"pop z{zi+1}", state, rest=zi == c.nz - 1)                                 # :224-226 restbits
        zsym = None
        for zi in range(c.nz):                                                                      # :228-240
            zsymtop = zs[zi]
            z = self.zcen[zi, self.zr, zsymtop]
            mu, sc = self._net("generate", zi, z)
            ends = self.zend[zi - 1] if zi > 0 else self.xend
            state = self._coder(self._pmfs(ends, mu, sc), q if zi > 0 else 8).encode(
                state, (zsym if zi > 0 else x).numpy())
            self._note(f"push {'z%d' % zi if zi > 0 else 'x'}", state)
            zsym = zsymtop
        state = self._coder(self._prior(), q).encode(state, zsym.numpy())                          # :245-250
        self._note("push prior", state)
        self._end()
        return state

    def decode_image_bbans(self, state):
        c = self.cfg
        q = c.quantbits
        state, top = self._coder(self._prior(), q).decode(state)
        top = torch.as_tensor(np.asarray(top))
        zs = [top]
        for zi in reversed(range(c.nz)):                                                            # :323-334
            z = self.zcen[zi, self.zr, zs[-1]]
            mu, sc = self._net("generate", zi, z)
            ends = self.zend[zi - 1] if zi > 0 else self.xend
            state, sym = self._coder(self._pmfs(ends, mu, sc), q if zi > 0 else 8).decode(state)
            zs.append(torch.as_tensor(np.asarray(sym)))
        # zs = [z_nz, z_{nz-1}, ..., z_1, x]
        for zi in reversed(range(c.nz)):                                                            # :337-350
            sym = zs[c.nz - zi]                     # the variable one level below z_{zi+1}
            given = self.zcen[zi - 1, self.zr, sym] if zi > 0 else self.xcen[self.xr, sym]
            mu, sc = self._net("infer", zi, given)
            state = self._coder(self._pmfs(self.zend[zi], mu, sc), q).encode(state, zs[c.nz - zi - 1].numpy())
        return state, zs[-1].numpy().astype(np.uint8)
