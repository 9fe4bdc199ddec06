"""Bin edges and renormalisation thresholds of the ANS coder: the harness the GPU edge tests (test_bin_edges_gpu.py) run on,
pinned here without a GPU.

A pop reads mm = x & (2^31 - 1) and picks the bin with searchsorted(C[:-1], mm, 'right') - 1; a head drawn at random sits on a
given bin edge with probability 2^-31, so random states say nothing about the comparisons that decide edges (`<=` against
`<`) or the renormalisation thresholds (x < 2^32 after a pop, x >= 2^33 P[s] before a push).  The head builder below puts a
head exactly on those values, and the vectorised coder below is the reference's ANS.encode / ANS.decode (cifar_compress.py
:48-67) for N streams at once, checked here against the literal port (AnsPort) and the C oracle (AnsC)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle as O                                                      # noqa: E402

BITS = 31
U64 = np.uint64
TWO32 = 1 << 32
POP_KINDS = ("lower", "upper", "renorm 2^32-1", "renorm 2^32", "random")
PUSH_KINDS = ("lim-1", "lim", "kmax*p-1", "kmax*p", "kmin*p-1", "kmin*p", "kmid*p", "random")


# ---- the vectorised coder ---------------------------------------------------------------------------------------------------
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


# ---- the head builder -------------------------------------------------------------------------------------------------------
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


# ---- tables with the shapes where searches go wrong -------------------------------------------------------------------------
def edge_pmfs(S, R, rs):
    """R pmf rows of S bins: dead bins (pmf 0, so P = 1), argmax ties (the remnant goes to the first maximum), the remnant
    bin at 0 and at S - 1, one bin holding almost all the mass, and ordinary random rows."""
    pm = rs.dirichlet(np.full(S, 0.3), size=R)
    for r in range(R):
        k = r % 6
        if k == 0:                                               # dead bins on both sides of a live middle
            lo, hi = sorted(rs.randint(0, S, 2))
            pm[r, :lo] = 0
            pm[r, hi + 1:] = 0
        elif k == 1 and S >= 2:                                  # tied maxima, the first of them somewhere random
            a, b = sorted(rs.choice(S, 2, replace=False))
            pm[r, a] = pm[r, b] = pm[r].max() * 1.5
        elif k == 2:                                             # remnant at bin 0
            pm[r, 0] = pm[r].sum()
        elif k == 3:                                             # remnant at bin S - 1
            pm[r, -1] = pm[r].sum()
        elif k == 4:                                             # nearly all the mass in one bin, the rest dead or tiny
            pm[r] = rs.choice([0.0, 1e-12], S)
            pm[r, rs.randint(S)] = 1.0
        pm[r] /= pm[r].sum()
    return pm


def _q(S):
    return max(1, (S - 1).bit_length())


SUPPORTS = [2, 3, 5, 16, 31, 32, 33, 100, 256, 1000, 1024, 2048, 4096]


def _case(S, R, seed):
    rs = np.random.RandomState(seed)
    pm = edge_pmfs(S, R, rs)
    P, C = O.tables_np(pm, BITS, _q(S))
    return rs, pm, RowTables(P, C)


@pytest.mark.parametrize("S", SUPPORTS)
def test_tables_have_the_shapes_they_claim(S):
    rs, pm, tab = _case(S, 12, S)
    Pc, Cc = O.tables_c(pm, BITS, _q(S))
    assert np.array_equal(Pc, tab.P) and np.array_equal(Cc, tab.C)
    am = tab.P.argmax(axis=1)
    assert (tab.P == 1).any()                                                      # dead bins
    assert 0 in am and S - 1 in am                                                 # the remnant at both ends
    assert (tab.P.max(axis=1) > (1 << BITS) - (1 << BITS) // 1000 - S).any()        # one bin with almost all the mass
    if S >= 3:                                                                     # a tie before the remnant: first maximum
        r = 1
        pre = (pm[r] * ((1 << BITS) - (1 << _q(S)))).astype(np.int64) + 1
        assert (pre == pre.max()).sum() >= 2 and am[r] == np.argmax(pre)


@pytest.mark.parametrize("S", SUPPORTS)
def test_heads_land_where_they_claim(S):
    rs, pm, tab = _case(S, 12, 100 + S)
    for r in range(tab.R):
        s = np.arange(S)
        rr = np.full(S, r)
        for kind in POP_KINDS:
            x, ok = pop_heads(tab.P[r], tab.C[r, :-1], kind, rs)
            check_pop_heads(x[ok], tab, rr[ok], s[ok], kind)
            if kind in ("lower", "upper", "random"):
                assert ok.all()
        for kind in PUSH_KINDS:
            x, ok = push_heads(tab.P[r], kind, rs)
            assert ok.all() or kind == "lim"
            check_push_heads(x[ok], tab.P[r][ok], kind)
    # the renormalisation targets exist wherever a bin is narrow enough: every bin with P < 2^31
    x, ok = pop_heads(np.array([1, 2, 3, 1 << 30, (1 << 31) - 1]), np.zeros(5, dtype=np.int64), "renorm 2^32", rs)
    assert ok.tolist() == [True, True, True, True, True]


def _edge_states(tab, S, top, rs, n_words, kinds=POP_KINDS):
    """For each kind, one stream per bin of row `top`, its head on that kind, n_words random words below it."""
    heads, want_bins = [], []
    for kind in kinds:
        x, ok = pop_heads(tab.P[top], tab.C[top, :-1], kind, rs)
        heads.append(x[ok])
        want_bins.append(np.arange(S)[ok])
    x = np.concatenate(heads)
    N = x.size
    words = rs.randint(0, 1 << 32, (N, n_words), dtype=np.int64).astype(np.uint32)
    return Stacks(np.concatenate([words, np.zeros((N, 4 * n_words + 8), np.uint32)], axis=1), np.full(N, n_words), x), \
        np.concatenate(want_bins)


@pytest.mark.parametrize("S", SUPPORTS)
def test_vectorised_coder_equals_the_reference_coders(S):
    """Pop every bin's edges and thresholds at the top row, then the rows below, and push a Latin pattern of symbols from
    push-threshold heads: the vectorised coder equals AnsPort (the literal port of the reference class) and AnsC."""
    R = 7
    rs, pm, tab = _case(S, R, 200 + S)
    rows = np.arange(R)
    st, bins = _edge_states(tab, S, R - 1, rs, n_words=R + 1)
    states = st.to_lists()
    sym = pop(tab, rows, st)
    assert np.array_equal(sym[:, -1], bins)
    port = O.AnsPort(pm, BITS, _q(S))
    ac = O.AnsC(tables=(tab.P, tab.C))
    pick = np.unique(np.r_[np.arange(0, len(states), max(1, len(states) // 40)), len(states) - 1])
    got = st.to_lists()
    for j in pick:
        x, s = port.decode(list(states[j]))
        assert x == got[j] and np.array_equal(s.numpy(), sym[j]), j
        cs, s2 = ac.decode(O.CState.from_list(states[j]))
        assert cs.to_list() == got[j] and np.array_equal(s2, sym[j]), j
    # a push round trip restores the states
    push(tab, rows, st, sym)
    assert st.to_lists() == states
    # push from every threshold head, symbol (j + 7 r) mod S at row r
    N = S * len(PUSH_KINDS)
    j = np.arange(N)
    psym = (j[:, None] + 7 * rows[None, :]) % S
    x = np.concatenate([push_heads(tab.P[0], k, rs)[0] for k in PUSH_KINDS])
    st = Stacks(np.zeros((N, R + 4), np.uint32), np.zeros(N, np.int64), x)
    st.w[:, 0] = 12345
    st.n[:] = 1
    before = st.to_lists()
    push(tab, rows, st, psym)
    got = st.to_lists()
    pick = np.unique(np.r_[np.arange(0, N, max(1, N // 60)), np.arange(S - 2, N, S)] % N)
    for j in pick:
        assert port.encode(list(before[j]), psym[j]) == got[j], j
        assert ac.encode(O.CState.from_list(before[j]), psym[j]).to_list() == got[j], j


def test_harness_catches_a_left_side_search():
    """A decode that searches with side='left' (the `<` for `<=` slip) differs from the reference exactly at lower edges:
    the harness's comparison must fail on edge heads, while random heads at these sizes do not notice."""
    S, R = 256, 5
    rs, pm, tab = _case(S, R, 7)
    rows = np.arange(R)
    st, _ = _edge_states(tab, S, R - 1, rs, n_words=R + 1, kinds=("lower", "upper"))
    want = Stacks(st.w.copy(), st.n, st.x)
    want_sym = pop(tab, rows, want)
    wrong = Stacks(st.w.copy(), st.n, st.x)
    wrong_sym = pop(tab, rows, wrong, side="left")
    with pytest.raises(AssertionError, match="top-row symbol"):
        assert_same("side=left", wrong_sym, wrong.packed(), want_sym, want, top=R - 1)
    x = (rs.randint(1 << 32, 1 << 63, st.x.size, dtype=np.int64).astype(U64) << U64(1)) | U64(1)   # heads as the suite draws them
    want = Stacks(st.w.copy(), st.n, x)
    want_sym = pop(tab, rows, want)
    wrong = Stacks(st.w.copy(), st.n, x)
    assert_same("random heads", pop(tab, rows, wrong, side="left"), wrong.packed(), want_sym, want, top=R - 1)
