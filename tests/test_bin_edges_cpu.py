"""Bin edges and renormalisation thresholds of the ANS coder: the harness the GPU edge tests (test_bin_edges_gpu.py) run on,
pinned here without a GPU.

A pop reads mm = x & (2^31 - 1) and picks the bin with searchsorted(C[:-1], mm, 'right') - 1; a head drawn at random sits on a
given bin edge with probability 2^-31, so random states say nothing about the comparisons that decide edges (`<=` against
`<`) or the renormalisation thresholds (x < 2^32 after a pop, x >= 2^33 P[s] before a push).  The head builder of
coder_harness.py puts a head exactly on those values, and its vectorised coder is the reference's ANS.encode / ANS.decode
(cifar_compress.py:48-67) for N streams at once, checked here against the literal port (AnsPort) and the C oracle (AnsC)."""
import numpy as np
import pytest

from coder_harness import (BITS, POP_KINDS, PUSH_KINDS, U64, RowTables, Stacks, assert_same, check_pop_heads,
                           check_push_heads, pop, pop_heads, push, push_heads)
from oracle import oracle as O


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
