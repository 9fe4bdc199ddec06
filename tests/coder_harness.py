"""The latent coder through the C ABI, and a numpy restatement of the reference coder -- TEST INFRASTRUCTURE.

Row generators, initial states, the two-phase, fused and push-then-pop runners, the oracle side (our exported float64 pmfs
-> ANS.__init__ -> the reference coder), the q = 12 known-answer test, and the vectorised numpy ANS coder with the head
builder of the bin-edge tests.  `coder_paths` is the one place that sets the process-global coder switches (rows mode,
k_rows6 verify mode, k_rows6 lanes per row); it restores their defaults however the block ends, so a failing test cannot
leave the next one on the kernel family it forced.  Imports without a GPU."""
import contextlib
import json
import os

import numpy as np
import torch

from oracle import oracle as O
from bitswap_b200 import synthetic
from bitswap_b200.streams import StreamSet
from bitswap_b200._lib import lib, check, cuda_stream_ptr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
dev = "cuda"


@contextlib.contextmanager
def coder_paths(rows_mode=None, verify=None, lanes_per_row=None):
    """Set the given coder switches for the block, then restore each one to its default (rows mode -1: classify the rows;
    verify off; lanes per row 0: the library's choice)."""
    try:
        if rows_mode is not None:
            check(lib().bsw_set_rows_mode(rows_mode))
        if verify is not None:
            check(lib().bsw_rows6_set_verify(verify))
        if lanes_per_row is not None:
            check(lib().bsw_rows6_set_lanes_per_row(lanes_per_row))
        yield
    finally:
        if rows_mode is not None:
            check(lib().bsw_set_rows_mode(-1))
        if verify is not None:
            check(lib().bsw_rows6_set_verify(0))
        if lanes_per_row is not None:
            check(lib().bsw_rows6_set_lanes_per_row(0))


# ---- inputs ---------------------------------------------------------------------------------------------------------------
def pad_big(ends):
    """Endpoints [L, S - 1] padded to [L, S] with 1e300, the row layout the logistic coder entry points read."""
    L, Sm1 = ends.shape
    out = np.full((L, Sm1 + 1), 1e300)
    out[:, :Sm1] = ends
    return out


def initial_states(B, seed, n=3000, step=7):
    """B initial state lists: stream b holds n + step * b seeded words (seed + b) and its head."""
    out = []
    for b in range(B):
        w, head = synthetic.initial_words(n + step * b, seed=seed + b)
        out.append([int(v) for v in w] + [head])
    return out


def hostile_rows(L, S, q, B, seed, affine=True):
    """One level's rows (ends [L, S - 1], mu, sigma [B, L]) and symbols [B, L]: ordinary, needle-sharp, all-bins-live and
    off-grid rows, symbols in the edge bins.  affine: uniform grids; else the top level's equal-mass bins."""
    rs = np.random.RandomState(seed)
    if affine:
        lo, hi = -6 - rs.uniform(0, 1, L), 6 + rs.uniform(0, 1, L)
        ends = np.linspace(lo, hi, S + 1, axis=1)[:, 1:-1].copy()
    else:                                                   # the top level: equal-mass logistic bins, float32
        from bitswap_b200.rand import Bins as RBins
        ends = RBins(torch.zeros((1, 1, L)), torch.ones((1, 1, L)), q).endpoints().numpy().reshape(L, S - 1).astype(np.float64)
    mu = rs.normal(0, 1.5, (B, L)).astype(np.float32)
    sc = rs.uniform(0.1, 1.0, (B, L)).astype(np.float32)
    sc[:, 0::5] = np.float32(1e-4)                          # needle-sharp: a few bins live
    sc[:, 1::5] = rs.uniform(3.0, 6.0, sc[:, 1::5].shape).astype(np.float32)    # wide: every bin live (chunks of S/32)
    mu[:, 2::7] = rs.choice([-25.0, 25.0], size=mu[:, 2::7].shape).astype(np.float32)   # mass beyond the grid
    sym = rs.randint(0, S, size=(B, L)).astype(np.int16)
    sym[:, :6] = [0, S - 1, 1, S - 2, S // 2, 0]
    return ends, mu, sc, sym


def level_case(L, S, q, B, seed, affine=True, sc_lo=0.1):
    """One level's rows (ends, mu, sigma) with sigma in [sc_lo, 1]; the callers add their own special rows."""
    rs = np.random.RandomState(seed)
    if affine:
        lo, hi = -6 - rs.uniform(0, 1, L), 6 + rs.uniform(0, 1, L)
        ends = np.linspace(lo, hi, S + 1, axis=1)[:, 1:-1].copy()
    else:                                                   # the top level: equal-mass logistic bins, float32 (discretization.py:25-27)
        from bitswap_b200.rand import Bins
        ends = Bins(torch.zeros((1, 1, L)), torch.ones((1, 1, L)), q).endpoints().numpy().reshape(L, S - 1).astype(np.float64)
    mu = rs.normal(0, 1.5, (B, L)).astype(np.float32)
    sc = rs.uniform(sc_lo, 1.0, (B, L)).astype(np.float32)
    return ends, mu, sc


# ---- the endpoint grids discretize() can build (test_grids_gpu.py) --------------------------------------------------------
def half(x):
    """Nearest float16 value, saturating at +-65504 (discretize() takes the extrema of float16 samples)."""
    return np.clip(np.asarray(x, dtype=np.float64), -65504.0, 65504.0).astype(np.float16).astype(np.float64)


def linspace_rows(lo, hi, S):
    """Rows of np.linspace(lo, hi, S + 1) without their two ends: the S - 1 endpoints of an S-bin uniform grid."""
    return np.linspace(lo, hi, S + 1, axis=1)[:, 1:-1].copy()


def _family_extrema(family, L, rs):
    u = lambda a, b: rs.uniform(a, b, L)                                       # noqa: E731
    sgn = rs.choice([-1.0, 1.0], L)
    if family == 1:                                           # off-centre: centre within +-1000, span 1 .. 21
        c, w = u(-1000, 1000), u(1, 21)
        lo = half(c - w * u(0.2, 0.8))
        return lo, half(lo + w)
    if family == 2:                                           # float16 extrema at or near +-65504, possibly asymmetric
        k = rs.randint(0, 4, L)
        lo = np.where(k == 0, -65504.0, half(-u(30000, 65504)))
        hi = np.where(k == 1, 65504.0, np.where(k == 2, half(u(-1000, 60000)), half(u(30000, 65504))))
        lo[k == 3], hi[k == 3] = -65504.0, 65504.0
        return lo, hi
    if family == 3:                                           # far from zero and narrow: |centre| in 30000 .. 60000, span <= 1
        c, w = sgn * u(30000, 60000), u(1e-3, 1)
        lo = c - w * u(0.2, 0.8)
        return lo, lo + w
    if family == 4:                                           # tiny spans 2^-20 .. 2^-24, at 0 and at 1000
        c, w = rs.choice([0.0, 1000.0], L), np.ldexp(1.0, -rs.randint(20, 25, L))
        lo = c - w * u(0.2, 0.8)
        return lo, lo + w
    if family == 5:                                           # ordinary spans; sigma puts dt at the plan's limit of 64
        lo = half(u(-10, 5))
        return lo, half(lo + u(0.5, 20))
    lo = u(-300, 300)                                         # 6: perturbed off the affine line (below)
    return lo, lo + np.exp(u(np.log(0.5), np.log(100.0)))


def draw(lo, hi, S, B, rs, family=0):
    """mu, sigma [B, L] (float32) relative to each row's centre c, half-width h and bin width d: a few bins live, many live,
    mass just beyond the grid, or anything in between.  Constant rows (d = 0) get sigma in [0.1, 1] around their value."""
    L = lo.shape[0]
    c, h = 0.5 * (lo + hi), 0.5 * (hi - lo)
    d = (hi - lo) / S
    u = lambda a, b: rs.uniform(a, b, (B, L))                                  # noqa: E731
    kind = rs.randint(0, 4, (B, L))
    sc = np.select([kind == 0, kind == 1, kind == 2],
                   [d * 10 ** u(-1.5, 0.5), h * u(0.05, 0.6), d * 10 ** u(-1, 1.5)],
                   d * 10 ** (u(0, 1) * np.log10(np.maximum(1.0, h / np.where(d > 0, d, 1.0)))))
    mu = np.where(kind == 2, c + rs.choice([-1.0, 1.0], (B, L)) * (h + sc * u(0, 12)), c + h * u(-1.2, 1.2))
    if family == 5:
        sc = d / (64.0 * u(0.97, 1.03))
        mu = c + h * u(-1, 1)
    flat = np.broadcast_to(d <= 0, (B, L))
    sc = np.where(flat, u(0.1, 1.0), sc)
    mu = np.where(flat, c + u(-1, 1), mu)
    return mu.astype(np.float32), np.maximum(sc.astype(np.float32), np.float32(1e-38))


def family_case(family, L, S, B, seed):
    rs = np.random.RandomState(seed)
    lo, hi = _family_extrema(family, L, rs)
    ends = linspace_rows(lo, hi, S)
    mu, sc = draw(lo, hi, S, B, rs, family)
    if family == 6:                     # every interior endpoint off the line by up to dv, one of them by exactly dv:
        emax = np.maximum(np.abs(lo), np.abs(hi))              # dv up to the classification tolerance 1e-13 max(1, emax)
        dv = 1e-13 * np.maximum(1.0, emax) * 10 ** rs.uniform(-6, 0, L)
        ends[:, 1:-1] += dv[:, None] * rs.uniform(-1, 1, (L, S - 3))
        ends[np.arange(L), rs.randint(1, S - 2, L)] += rs.choice([-1.0, 1.0], L) * dv
    return ends, mu, sc


# ---- runners --------------------------------------------------------------------------------------------------------------
def run_2p(ends, mu, sc, S, q, states, sym, mode, cap=1 << 15):
    """pop then push of one level through the two-phase ABI in rows mode `mode`, on streams of capacity `cap`; returns
    (states after pop, popped symbols, states after push)."""
    B, L = mu.shape
    with coder_paths(rows_mode=mode):
        e_pad = torch.from_numpy(pad_big(ends)).to(dev)
        dmu, dsc, dsym = torch.from_numpy(mu).to(dev), torch.from_numpy(sc).to(dev), torch.from_numpy(sym).to(dev)
        nbytes = int(lib().bsw_logistic_scratch_bytes(B, L, S, 0))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        ss = StreamSet(B, cap)
        ss.import_lists(states)
        out = torch.zeros((B, L), dtype=torch.int16, device=dev)
        check(lib().bsw_logistic_pop_2p(ss.handle, 0, B, dmu.data_ptr(), L, dsc.data_ptr(), L, e_pad.data_ptr(), S, out.data_ptr(),
                                        L, S, 31, q, scratch.data_ptr(), nbytes, cuda_stream_ptr()))
        ss.raise_on_error()
        a, popped = ss.export_lists(), out.cpu().numpy().copy()
        check(lib().bsw_logistic_push_2p(ss.handle, 0, B, dmu.data_ptr(), L, dsc.data_ptr(), L, e_pad.data_ptr(), S, dsym.data_ptr(),
                                         L, S, 31, q, scratch.data_ptr(), nbytes, cuda_stream_ptr()))
        ss.raise_on_error()
        return a, popped, ss.export_lists()


def run_fused(ends, mu, sc, S, q, states, sym, cap=1 << 15):
    """run_2p through the fused one-warp-per-stream kernels (up to 1024 bins)."""
    B, L = mu.shape
    e_pad = torch.from_numpy(pad_big(ends)).to(dev)
    dmu, dsc, dsym = torch.from_numpy(mu).to(dev), torch.from_numpy(sc).to(dev), torch.from_numpy(sym).to(dev)
    ss = StreamSet(B, cap)
    ss.import_lists(states)
    out = torch.zeros((B, L), dtype=torch.int16, device=dev)
    check(lib().bsw_logistic_pop(ss.handle, 0, B, dmu.data_ptr(), L, dsc.data_ptr(), L, e_pad.data_ptr(), S, out.data_ptr(), L, S,
                                 31, q, cuda_stream_ptr()))
    ss.raise_on_error()
    a, popped = ss.export_lists(), out.cpu().numpy().copy()
    check(lib().bsw_logistic_push(ss.handle, 0, B, dmu.data_ptr(), L, dsc.data_ptr(), L, e_pad.data_ptr(), S, dsym.data_ptr(), L,
                                  S, 31, q, cuda_stream_ptr()))
    ss.raise_on_error()
    return a, popped, ss.export_lists()


def push_pop(ends, mu, sc, S, q, states, sym, coder):
    """push `sym`, then pop them again, through coder "generic", "classified", "affine" (two-phase, rows mode 0, -1, 1) or
    "fused"; returns (states after push, popped symbols, states after pop)."""
    B, L = mu.shape
    e_pad = torch.from_numpy(pad_big(ends)).to(dev)
    dmu, dsc, dsym = torch.from_numpy(mu).to(dev), torch.from_numpy(sc).to(dev), torch.from_numpy(sym).to(dev)
    nbytes = int(lib().bsw_logistic_scratch_bytes(B, L, S, 0))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    ss = StreamSet(B, 1 << 15)
    ss.import_lists(states)
    out = torch.zeros((B, L), dtype=torch.int16, device=dev)
    args = (dmu.data_ptr(), L, dsc.data_ptr(), L, e_pad.data_ptr(), S)
    with coder_paths(rows_mode={"generic": 0, "classified": -1, "affine": 1, "fused": -1}[coder]):
        if coder == "fused":
            check(lib().bsw_logistic_push(ss.handle, 0, B, *args, dsym.data_ptr(), L, S, 31, q, cuda_stream_ptr()))
            ss.raise_on_error()
            pushed = ss.export_lists()
            check(lib().bsw_logistic_pop(ss.handle, 0, B, *args, out.data_ptr(), L, S, 31, q, cuda_stream_ptr()))
        else:
            check(lib().bsw_logistic_push_2p(ss.handle, 0, B, *args, dsym.data_ptr(), L, S, 31, q, scratch.data_ptr(), nbytes,
                                             cuda_stream_ptr()))
            ss.raise_on_error()
            pushed = ss.export_lists()
            check(lib().bsw_logistic_pop_2p(ss.handle, 0, B, *args, out.data_ptr(), L, S, 31, q, scratch.data_ptr(), nbytes,
                                            cuda_stream_ptr()))
        ss.raise_on_error()
        return pushed, out.cpu().numpy().copy(), ss.export_lists()


# ---- the oracle side ------------------------------------------------------------------------------------------------------
def ref_pmfs_cuda(ends, mu, sc):
    """The reference's tensor expression (cifar_compress.py:182-184) evaluated by torch ON THE GPU, as the
    reference itself runs it (device = cuda, cifar_compress.py:77)."""
    cdfs = torch.sigmoid((ends.t() - mu) / sc).t()
    pmfs = cdfs[:, 1:] - cdfs[:, :-1]
    return torch.cat((cdfs[:, 0].unsqueeze(1), pmfs, 1. - cdfs[:, -1].unsqueeze(1)), dim=1)


def oracle_tables(ends, mu, sc, S, q):
    """Per stream b, ANS.__init__'s integer tables (O.tables_c) of our exported pmfs (bsw_logistic_pmfs) of row set b."""
    e_raw = torch.from_numpy(np.ascontiguousarray(ends)).to(dev)
    tabs = []
    for b in range(mu.shape[0]):
        pm = torch.empty((mu.shape[1], S), dtype=torch.float64, device=dev)
        m64 = torch.from_numpy(mu[b]).double().to(dev).contiguous()
        s64 = torch.from_numpy(sc[b]).double().to(dev).contiguous()
        check(lib().bsw_logistic_pmfs(e_raw.data_ptr(), S - 1, m64.data_ptr(), s64.data_ptr(), 1, mu.shape[1], S, pm.data_ptr(),
                                      cuda_stream_ptr()))
        torch.cuda.synchronize()
        tabs.append(O.tables_c(pm.cpu().numpy(), 31, q))
    return tabs


def check_vs_oracle(res, tabs, states, sym, check_streams):
    """A run_2p result against the reference coder on `tabs`, for the streams in check_streams."""
    after_pop, popped, after_push = res
    for b in check_streams:
        a = O.AnsC(tables=tabs[b])
        st, s_ = a.decode(O.CState.from_list(states[b]))
        assert np.array_equal(popped[b], s_), f"stream {b}: popped symbols differ"
        assert after_pop[b] == st.to_list(), f"stream {b}: state after pop differs"
        assert after_push[b] == a.encode(st, sym[b].astype(np.int64)).to_list(), f"stream {b}: state after push differs"


# ---- the q = 12 known-answer test (tests/golden/make_golden_q12.py) -------------------------------------------------------
KAT = json.load(open(os.path.join(GOLDEN, "ans_kat_q12.json")))[0]


def kat_inputs():
    rs = np.random.RandomState(KAT["seed"])
    pm = rs.dirichlet(np.ones(KAT["S"]) * 0.5, size=KAT["L"])
    sym = rs.randint(0, KAT["S"], size=KAT["L"])
    w, head = synthetic.initial_words(KAT["N"], seed=100)
    return pm, sym, w, head


# ---- the vectorised reference coder (cifar_compress.py:48-67 for N streams at once) ---------------------------------------
# A pop reads mm = x & (2^31 - 1) and picks the bin with searchsorted(C[:-1], mm, 'right') - 1; a head drawn at random sits on
# a given bin edge with probability 2^-31, so the head builder below puts heads exactly on the edges and on the
# renormalisation thresholds (x < 2^32 after a pop, x >= 2^33 P[s] before a push).
BITS = 31
U64 = np.uint64
TWO32 = 1 << 32
POP_KINDS = ("lower", "upper", "renorm 2^32-1", "renorm 2^32", "random")
PUSH_KINDS = ("lim-1", "lim", "kmax*p-1", "kmax*p", "kmin*p-1", "kmin*p", "kmid*p", "random")


class RowTables:
    """Integer tables of R rows, P [R, S] and C [R, S + 1] (int64, as O.tables_np returns them), and the key searchsorted runs
    on: row r's C[r, :-1] offset by r * 2^32, so one call searches every stream in its own row."""

    def __init__(self, P, C):
        self.P, self.C = np.ascontiguousarray(P, dtype=np.int64), np.ascontiguousarray(C, dtype=np.int64)
        self.R, self.S = self.P.shape
        self.key = ((np.arange(self.R, dtype=np.int64)[:, None] << 32) + self.C[:, :-1]).ravel()

    def search(self, rows, mm, side="right"):
        """searchsorted(C[rows[j], :-1], mm[j], side) - 1 for every stream j (the reference's ANS.decode with 'right')."""
        q = (rows << 32) + mm.astype(np.int64)
        return np.searchsorted(self.key, q, side) - 1 - rows * self.S


class Stacks:
    """N reference states: words [N, cap] uint32 bottom-first with n [N] of them in use, and the heads x [N] uint64."""

    def __init__(self, words, n, x):
        self.w, self.n, self.x = words, np.asarray(n, dtype=np.int64).copy(), np.asarray(x, dtype=U64).copy()

    @classmethod
    def from_packed(cls, words, offsets, heads, cap):
        offsets = np.asarray(offsets, dtype=np.int64)
        n = np.diff(offsets)
        w = np.zeros((len(n), cap), dtype=np.uint32)
        w[np.arange(cap)[None, :] < n[:, None]] = words
        return cls(w, n, heads)

    @classmethod
    def from_lists(cls, states, cap):
        n = np.array([len(s) - 1 for s in states], dtype=np.int64)
        w = np.zeros((len(states), cap), dtype=np.uint32)
        for j, s in enumerate(states):
            w[j, :n[j]] = np.array(s[:-1], dtype=np.uint64).astype(np.uint32)
        return cls(w, n, np.array([s[-1] for s in states], dtype=U64))

    def packed(self):
        """(words uint32 [sum n], offsets int64 [N + 1], heads uint64 [N]), the layout of StreamSet.export."""
        offs = np.zeros(self.n.size + 1, dtype=np.int64)
        np.cumsum(self.n, out=offs[1:])
        return self.w[np.arange(self.w.shape[1])[None, :] < self.n[:, None]], offs, self.x.copy()

    def to_lists(self):
        return [[int(v) for v in self.w[j, :self.n[j]]] + [int(self.x[j])] for j in range(self.n.size)]


def _rows_for(rows, N):
    rows = np.asarray(rows, dtype=np.int64)
    return np.broadcast_to(rows, (N, rows.shape[-1]))


def pop(tab, rows, st, side="right", bits=BITS):
    """ANS.decode of len(rows) rows for every stream in `st` (in place), rows descending; rows [L] (shared) or [N, L].
    Returns the symbols [N, L].  side='left' is a deliberately wrong search the harness must catch."""
    N = st.x.size
    rows = _rows_for(rows, N)
    sym = np.empty(rows.shape, dtype=np.int64)
    mask = U64((1 << bits) - 1)
    for i in range(rows.shape[1] - 1, -1, -1):
        r = rows[:, i]
        mm = st.x & mask                                                            # :60
        s = tab.search(r, mm, side)                                                 # :61
        p, c = tab.P[r, s].astype(U64), tab.C[r, s].astype(U64)
        x = p * (st.x >> U64(bits)) + mm - c                                        # :63
        need = np.flatnonzero(x < U64(TWO32))                                       # :64
        if (st.n[need] <= 0).any():
            raise IndexError("pop from empty ANS stack")
        st.n[need] -= 1
        x[need] = (x[need] << U64(32)) | st.w[need, st.n[need]].astype(U64)         # :65
        st.x = x
        sym[:, i] = s
    return sym


def push(tab, rows, st, sym, bits=BITS):
    """ANS.encode of len(rows) rows for every stream in `st` (in place), rows ascending; sym [N, L]."""
    N = st.x.size
    rows = _rows_for(rows, N)
    sym = np.asarray(sym, dtype=np.int64)
    for i in range(rows.shape[1]):
        r, s = rows[:, i], sym[:, i]
        p, c = tab.P[r, s].astype(U64), tab.C[r, s].astype(U64)
        lim = U64(((TWO32 >> bits) << 32)) * p                                      # :51
        big = np.flatnonzero(st.x >= lim)
        if (st.n[big] >= st.w.shape[1]).any():
            raise OverflowError("stack capacity")
        st.w[big, st.n[big]] = (st.x[big] & U64(0xffffffff)).astype(np.uint32)     # :52-53
        st.n[big] += 1
        st.x[big] >>= U64(32)
        st.x = ((st.x // p) << U64(bits)) + st.x % p + c                           # :54
    return st


def assert_same(label, got_sym, got_packed, want_sym, want, top=None):
    """Popped symbols (optional), then heads, word counts and word stacks, all as packed numpy arrays.  top: index of the
    view's top row, whose symbol is checked (and reported) first."""
    words, offs, heads = got_packed[:3]
    w_words, w_offs, w_heads = want.packed()
    if want_sym is not None:
        got_sym = np.asarray(got_sym).astype(np.int64)
        if top is not None:
            bad = np.flatnonzero(got_sym[:, top] != want_sym[:, top])
            assert bad.size == 0, f"{label}: top-row symbol of {bad.size} streams, first {bad[:6].tolist()}: " \
                                  f"got {got_sym[bad[:6], top].tolist()}, want {want_sym[bad[:6], top].tolist()}"
        bad = np.flatnonzero((got_sym != want_sym).any(axis=1))
        assert bad.size == 0, f"{label}: symbols of {bad.size} streams differ, first {bad[:6].tolist()}"
    bad = np.flatnonzero(np.asarray(heads, dtype=U64) != w_heads)
    assert bad.size == 0, f"{label}: heads of {bad.size} streams differ, first {bad[:6].tolist()}"
    bad = np.flatnonzero(np.diff(offs) != np.diff(w_offs))
    assert bad.size == 0, f"{label}: word counts of {bad.size} streams differ, first {bad[:6].tolist()}"
    assert np.array_equal(np.asarray(words, dtype=np.uint32), w_words), f"{label}: word stacks differ"


# ---- the head builder -----------------------------------------------------------------------------------------------------
def pop_heads(p, c, kind, rs, bits=BITS):
    """Heads x in [2^32, 2^64) for a pop of bins with integer pmf p and cdf c (int64 arrays, one entry per head): mm = x & mask
    on the bin's lower edge C[s] or upper edge C[s + 1] - 1, or such that the decoded value p (x >> 31) + mm - c is exactly
    2^32 - 1 (a word is read) or 2^32 (none is), or mm anywhere in the bin under a random upper part.  Returns (x uint64, ok):
    ok is False where no mm inside the bin gives the kind (the renormalisation targets need x >> 31 >= 2)."""
    p, c = np.asarray(p, dtype=np.int64), np.asarray(c, dtype=np.int64)
    n = p.size
    hi = rs.randint(2, 1 << (64 - bits), n, dtype=np.int64)
    ok = np.ones(n, dtype=bool)
    if kind == "lower":
        mm = c
    elif kind == "upper":
        mm = c + p - 1
    elif kind in ("renorm 2^32-1", "renorm 2^32"):
        T = TWO32 - (1 if kind == "renorm 2^32-1" else 0)
        hi, d = T // p, T % p
        ok = hi >= 2
        hi = np.where(ok, hi, 2)
        mm = c + np.where(ok, d, 0)
    elif kind == "random":
        hi = rs.randint(1 << (63 - bits), 1 << (64 - bits), n, dtype=np.int64)
        mm = c + (rs.random_sample(n) * p).astype(np.int64)
    else:
        raise ValueError(kind)
    return (hi.astype(U64) << U64(bits)) | mm.astype(U64), ok


def push_heads(p, kind, rs, bits=BITS):
    """Heads x in [2^32, 2^64) for a push of bins with integer pmf p: x = lim - 1 and lim with lim = 2^33 p (the
    renormalisation threshold), x = k p - 1 and k p for the largest k with k p < lim, the smallest with k p - 1 >= 2^32 and one
    in between (the quotient steps of the division the kernels replace with a reciprocal), or any x.  Returns (x, ok)."""
    p = np.asarray(p, dtype=np.int64)
    n = p.size
    lim = p.astype(object) * ((TWO32 >> bits) << 32)
    kmax = (lim - 1) // p.astype(object)
    kmin = (TWO32 + 1 + p.astype(object) - 1) // p.astype(object)
    if kind in ("lim-1", "lim"):
        x = lim - (1 if kind == "lim-1" else 0)
    elif kind.startswith("k"):
        k = {"kmax": kmax, "kmin": kmin}.get(kind[:4])
        if k is None:
            k = kmin + (np.array([int(v) for v in (kmax - kmin)], dtype=object) * rs.random_sample(n)).astype(np.int64)
        x = k * p.astype(object) - (1 if kind.endswith("-1") else 0)
    elif kind == "random":
        x = np.array([int(v) for v in rs.randint(1, 1 << 32, n, dtype=np.int64)], dtype=object) << 32
        x = x | np.array([int(v) for v in rs.randint(0, 1 << 32, n, dtype=np.int64)], dtype=object)
    else:
        raise ValueError(kind)
    x = np.array([int(v) for v in x], dtype=object)
    ok = (x >= TWO32) & (x < (1 << 64))
    return np.array([int(v) if o else TWO32 for v, o in zip(x, ok)], dtype=U64), ok.astype(bool)


def check_pop_heads(x, rows_tab, r, s, kind, bits=BITS):
    """Each head lands where it claims: its bin is s, and the kind's edge or decoded value holds."""
    tab = rows_tab
    mm = (x & U64((1 << bits) - 1)).astype(np.int64)
    assert (x >= U64(TWO32)).all()
    assert np.array_equal(tab.search(r, mm), s), kind
    if kind == "lower":
        assert np.array_equal(mm, tab.C[r, s])
    elif kind == "upper":
        assert np.array_equal(mm, tab.C[r, s + 1] - 1)
    elif kind.startswith("renorm"):
        y = tab.P[r, s].astype(U64) * (x >> U64(bits)) + mm.astype(U64) - tab.C[r, s].astype(U64)
        assert (y == U64(TWO32 - (1 if kind == "renorm 2^32-1" else 0))).all(), kind


def check_push_heads(x, p, kind, bits=BITS):
    lim = [int(v) * ((TWO32 >> bits) << 32) for v in p]
    xs = [int(v) for v in x]
    assert all(TWO32 <= v < (1 << 64) for v in xs)
    if kind == "lim-1":
        assert all(v == m - 1 for v, m in zip(xs, lim))
    elif kind == "lim":
        assert all(v == m for v, m in zip(xs, lim))
    elif kind.startswith("k"):
        d = 1 if kind.endswith("-1") else 0
        assert all((v + d) % int(q) == 0 and v + d < m for v, q, m in zip(xs, p, lim)), kind
        if kind.startswith("kmax"):
            assert all(v + d + int(q) >= m for v, q, m in zip(xs, p, lim))
        if kind.startswith("kmin"):
            assert all(v + d - int(q) - 1 < TWO32 for v, q in zip(xs, p))
