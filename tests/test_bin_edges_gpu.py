"""Every pop and push kernel at both edges of every bin and at both renormalisation thresholds, against the reference's
integer tables.

A pop is asked, with a chosen head, which bin holds mm at the one value where the answer changes: for a target row t the
kernels get a view of L' rows ending at t (mu, sigma and endpoints offset by whole rows, stream strides 0, so every stream
reads the same rows), and stream j's head sits on one edge of bin s_j of row t, or makes the decoded value 2^32 - 1 or 2^32
(coder_harness.pop_heads).  The view's top row i = L' - 1 is popped first; the rows below pop random words.  L' cycles
over 1, 2, 31, 32, 33, 64 and 65, so the target row sits on lane i & 31 = 0, 1, 30 or 31 of the first 32-row block the kernels
load, alone in its block or with whole blocks below it that are adopted through the one-block-ahead preload (only the random
heads of the rows below meet that path).  A push codes every (row, symbol) pair once (stream j pushes (j + 7 r) mod S at
row r) from heads on the push threshold 2^33 P[s] and on the quotient steps of the division the kernels replace with a
reciprocal.

Everything is compared with the vectorised reference coder of coder_harness.py on tables built from the reference's
own expression evaluated on this GPU (torch.sigmoid, float64) and ANS.__init__: popped symbols (the top row's first), heads,
word counts and word stacks."""
import os
import sys
import time
from collections import Counter

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from coder_harness import (POP_KINDS, PUSH_KINDS, RowTables, Stacks, assert_same, check_pop_heads,   # noqa: E402
                           check_push_heads, coder_paths, dev, family_case, linspace_rows, pad_big, pop, pop_heads,
                           push, push_heads, ref_pmfs_cuda)
from oracle import oracle as O                                                                  # noqa: E402
from bitswap_b200.streams import StreamSet                                                      # noqa: E402
from bitswap_b200._lib import lib, check, cuda_stream_ptr                                       # noqa: E402
VIEWS = (1, 2, 31, 32, 33, 64, 65)
# two-phase paths: (rows mode, k_rows6 lanes per row); mode -1 classifies the rows (k_rows6 / k_pop6 when every row is a
# uniform grid), 1 forces the affine kernels (non-uniform rows take the exact path for every bin), 0 is k_rows /
# k_rows_wide + k_pop_coarse
TWO_PHASE = {"classified": (-1, 0), "classified lpr32": (-1, 32), "affine": (1, 0), "affine lpr32": (1, 32), "generic": (0, 0)}
ALL = ("classified", "classified lpr32", "affine", "generic", "fused", "table")


class Level:
    """One level's rows: endpoints [R, S - 1] (or one row read with row stride 0), mu and sigma per row (every stream reads
    the same ones), their device copies, and the reference's integer tables of every row."""

    def __init__(self, ends, mu, sc, S, q, shared_row=False):
        self.S, self.q, self.R = S, q, mu.size
        self.ers = 0 if shared_row else S
        self.e_pad = torch.from_numpy(pad_big(ends)).to(dev)
        self.mu = torch.from_numpy(np.ascontiguousarray(mu, dtype=np.float32)).to(dev)
        self.sc = torch.from_numpy(np.ascontiguousarray(sc, dtype=np.float32)).to(dev)
        e = torch.from_numpy(np.ascontiguousarray(ends, dtype=np.float64)).to(dev)
        if shared_row:
            e = e.expand(self.R, -1)
        pm = torch.cat([ref_pmfs_cuda(e[r:r + 256], self.mu[r:r + 256].double(), self.sc[r:r + 256].double()).cpu()
                        for r in range(0, self.R, 256)]).numpy()
        P, C = O.tables_np(pm, 31, q)
        self.tab = RowTables(P, C)
        self.P32 = torch.from_numpy(P.astype(np.uint32).view(np.int32)).to(dev)
        self.C32 = torch.from_numpy(C.astype(np.uint32).view(np.int32)).to(dev)


def _code(fam, push_, lv, ss, N, r0, L, sym=None, mu=None, sc=None):
    """One launch of family `fam` over rows r0 .. r0 + L - 1 of `lv` for streams 0 .. N - 1.  mu, sc: per-stream rows
    [N, L] on the device (stride L) instead of the level's shared ones (stride 0).  Returns the popped symbols (pop)."""
    S, q, st = lv.S, lv.q, cuda_stream_ptr()
    if mu is None:
        mu_p, mss, sc_p, sss = lv.mu.data_ptr() + 4 * r0, 0, lv.sc.data_ptr() + 4 * r0, 0
    else:
        mu_p, mss, sc_p, sss = mu.data_ptr(), L, sc.data_ptr(), L
    e_p = lv.e_pad.data_ptr() + 8 * r0 * lv.ers
    if fam == "table":
        P_p, C_p = lv.P32.data_ptr() + 4 * r0 * S, lv.C32.data_ptr() + 4 * r0 * (S + 1)
        if push_:
            s32 = torch.from_numpy(sym.astype(np.int32)).to(dev)
            check(lib().bsw_ans_push(ss.handle, 0, N, P_p, C_p, 0, 0, s32.data_ptr(), L, S, 31, st))
            return None
        out = torch.zeros((N, L), dtype=torch.int32, device=dev)
        check(lib().bsw_ans_pop(ss.handle, 0, N, P_p, C_p, 0, 0, out.data_ptr(), L, S, 31, st))
        return out.cpu().numpy()
    s16 = torch.from_numpy(sym.astype(np.int16)).to(dev) if push_ else torch.zeros((N, L), dtype=torch.int16, device=dev)
    args = (ss.handle, 0, N, mu_p, mss, sc_p, sss, e_p, lv.ers, s16.data_ptr(), L, S, 31, q)
    if fam == "fused":
        check((lib().bsw_logistic_push if push_ else lib().bsw_logistic_pop)(*args, st))
    else:
        nbytes = int(lib().bsw_logistic_scratch_bytes(N, L, S, 0))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        mode, lpr = TWO_PHASE[fam]
        with coder_paths(rows_mode=mode, lanes_per_row=lpr):
            check((lib().bsw_logistic_push_2p if push_ else lib().bsw_logistic_pop_2p)(*args, scratch.data_ptr(), nbytes, st))
    return None if push_ else s16.cpu().numpy()


def _edge_heads(tab, rows, rs):
    """Pop heads on every kind for every bin of each target row in `rows` (one row per stream group).  Returns (x, row)."""
    xs, rr = [], []
    S = tab.S
    for t in np.atleast_1d(rows):
        for kind in POP_KINDS:
            x, ok = pop_heads(tab.P[t], tab.C[t, :-1], kind, rs)
            s = np.arange(S)[ok]
            check_pop_heads(x[ok], tab, np.full(s.size, t), s, kind)
            xs.append(x[ok])
            rr.append(np.full(s.size, t))
    return np.concatenate(xs), np.concatenate(rr)


def _pop_rows(lv, targets, fams, label, seed, counts):
    """One launch per target row and family; streams: every bin x every head kind of the target row."""
    rs = np.random.RandomState(seed)
    S = lv.S
    ss = StreamSet(S * len(POP_KINDS), 128)
    for k, t in enumerate(targets):
        Lp = min(VIEWS[k % len(VIEWS)], t + 1)
        r0 = t - Lp + 1
        x, _ = _edge_heads(lv.tab, t, rs)
        N = x.size
        st = Stacks(rs.randint(0, 1 << 32, (N, Lp), dtype=np.int64).astype(np.uint32), np.full(N, Lp), x)
        packed = st.packed()
        want_sym = pop(lv.tab, np.arange(r0, t + 1), st)
        for fam in fams:
            ss.import_packed(*packed)
            got_sym = _code(fam, False, lv, ss, N, r0, Lp)
            ss.raise_on_error()
            assert_same(f"{label} {fam} row {t} L'={Lp}", got_sym, ss.export(0, N), want_sym, st, top=Lp - 1)
            counts[fam] += N


def _push_rows(lv, r0, L, fams, label, seed, counts, kinds=PUSH_KINDS):
    """S streams per push-head kind over rows r0 .. r0 + L - 1: stream j pushes (j + 7 r) mod S at row r, its head on that
    kind for its first symbol."""
    rs = np.random.RandomState(seed)
    S = lv.S
    N = S * len(kinds)
    j = np.arange(N)
    sym = (j[:, None] + 7 * np.arange(L)[None, :]) % S
    p0 = lv.tab.P[r0, j % S]
    x = np.empty(N, dtype=np.uint64)
    for g, kind in enumerate(kinds):
        xg, ok = push_heads(p0[g * S:(g + 1) * S], kind, rs)
        assert ok.all(), kind
        check_push_heads(xg, p0[g * S:(g + 1) * S], kind)
        x[g * S:(g + 1) * S] = xg
    st = Stacks(np.zeros((N, L + 1), np.uint32), np.ones(N, np.int64), x)
    st.w[:, 0] = rs.randint(0, 1 << 32, N, dtype=np.int64).astype(np.uint32)
    packed = st.packed()
    push(lv.tab, np.arange(r0, r0 + L), st, sym)
    ss = StreamSet(N, L + 64)
    for fam in fams:
        ss.import_packed(*packed)
        _code(fam, True, lv, ss, N, r0, L, sym=sym)
        ss.raise_on_error()
        assert_same(f"{label} {fam} push rows {r0}..{r0 + L - 1}", None, ss.export(0, N), None, st)
        counts[fam] += N * L


def _report(label, counts, t0):
    print(f"{label}: " + ", ".join(f"{f} {n}" for f, n in counts.items()) + f" targets checked in {time.time() - t0:.1f} s")


# ---- levels -----------------------------------------------------------------------------------------------------------------
SPECIAL = ("needle", "every bin live", "off grid left", "off grid right", "on an edge", "on a centre", "sigma 0.1")


def _special_level(S, R, seed, dyadic=True):
    """R uniform-grid rows whose kind cycles through SPECIAL and three ordinary rows: needle-sharp sigma (dead bins on both
    sides), sigma wide enough that every bin is live (chunks of 32 bins, 128 above 1024), mu beyond either end of the grid,
    mu exactly on a bin edge and on a bin centre (the grid is +-8 with dyadic endpoints where S is a power of two, so float32
    mu equals the float64 endpoint or centre), sigma at the 0.1 floor."""
    rs = np.random.RandomState(seed)
    lo, hi = -6 - rs.uniform(0, 1, R), 6 + rs.uniform(0, 1, R)
    kind = np.arange(R) % (len(SPECIAL) + 3)
    ex = (kind == 4) | (kind == 5)
    lo[ex], hi[ex] = -8.0, 8.0
    ends = linspace_rows(lo, hi, S)
    mu = rs.normal(0, 1.5, R)
    sc = rs.uniform(0.1, 1.0, R)
    sc[kind == 0] = 1e-4
    sc[kind == 1] = rs.uniform(4.0, 6.0, (kind == 1).sum())
    mu[kind == 2], mu[kind == 3] = -25.0, 25.0
    for r in np.flatnonzero(ex):
        k = rs.randint(S // 4, 3 * S // 4)
        mu[r] = ends[r, k] if kind[r] == 4 else 0.5 * (ends[r, k] + ends[r, k + 1])
        sc[r] = rs.choice([1e-3, 0.05, 0.3])
    sc[kind == 6] = 0.1
    return ends, mu.astype(np.float32), sc.astype(np.float32)


def _check_special(lv, ends, mu):
    """The edge and centre rows really put mu where they claim (float32 mu equal to the float64 endpoint / centre)."""
    S = lv.S
    if S & (S - 1):
        return
    kind = np.arange(lv.R) % (len(SPECIAL) + 3)
    for r in np.flatnonzero((kind == 4) | (kind == 5)):
        e = ends[r]
        at = np.flatnonzero(e == float(mu[r])) if kind[r] == 4 else np.flatnonzero(0.5 * (e[:-1] + e[1:]) == float(mu[r]))
        assert at.size == 1, r


# Target rows are sampled so that each case costs about the same: a launch's phase A evaluates (bins x streams x view rows)
# ~ S^2 L', so a case gets about LAUNCH_BUDGET / (S x families) target rows, never fewer than its ten special rows.
LAUNCH_BUDGET = 40 * 1024


def _targets(R, S, nfams, cap=128, special_every=10):
    """Target rows of R: the first `special_every` (one of each kind of special row), the last, and an even spread."""
    n = min(cap, max(special_every, LAUNCH_BUDGET // (S * nfams)))
    step = max(1, R // n)
    return sorted(set(range(0, R, step)) | set(range(min(R, special_every))) | {R - 1})


POW2 = [1 << q for q in range(5, 13)]


@pytest.mark.parametrize("S", POW2)
def test_pop_edges_sampled_rows_every_family(S):
    """About 128 target rows of a level of special and ordinary rows, at every power of two from 32 to 4096 bins, through
    every pop kernel: k_pop6 (classified, lanes per row 4 and 32, forced affine), k_pop_coarse, the fused k_logistic_pop
    (up to 1024 bins) and k_pop_tables on the reference's own tables."""
    q = S.bit_length() - 1
    t0 = time.time()
    R = 130
    ends, mu, sc = _special_level(S, R, seed=S)
    lv = Level(ends, mu, sc, S, q)
    _check_special(lv, ends, mu)
    assert (lv.tab.P[np.arange(R) % 10 == 0] == 1).any(axis=1).all()                  # the needle rows have dead bins
    assert (lv.tab.P[np.arange(R) % 10 == 1] > 1).all()                               # every bin live
    fams = [f for f in ALL if f != "fused" or S <= 1024]
    counts = Counter()
    _pop_rows(lv, _targets(R, S, len(fams)), fams, f"S={S}", S, counts)
    _report(f"pop S={S}", counts, t0)


@pytest.mark.parametrize("S", [8, 12, 20, 100, 1020])
def test_pop_edges_affine_kernels_at_supports_that_are_not_powers_of_two(S):
    q = max(3, (S - 1).bit_length())
    t0 = time.time()
    R = 130
    ends, mu, sc = _special_level(S, R, seed=S + 1)
    lv = Level(ends, mu, sc, S, q)
    counts = Counter()
    fams = ("affine", "affine lpr32", "table")
    _pop_rows(lv, _targets(R, S, len(fams)), fams, f"S={S}", S, counts)
    _report(f"pop S={S}", counts, t0)


@pytest.mark.parametrize("family", [3, 4, 5, 6])
@pytest.mark.parametrize("S", [1024, 2048])
def test_pop_edges_on_hostile_grid_families(family, S):
    """Far-narrow grids, tiny spans, dt near 64 and rows perturbed within the classification tolerance (the grid families
    of test_grids_gpu.py): forced affine kernels (rows outside the rule take the exact path), the classification path and
    the generic kernels."""
    q = S.bit_length() - 1
    t0 = time.time()
    R = 130
    ends, mu, sc = family_case(family, R, S, 1, seed=4000 + 10 * family + S)
    lv = Level(ends, mu[0], sc[0], S, q)
    counts = Counter()
    fams = ("affine", "classified", "generic")
    _pop_rows(lv, _targets(R, S, len(fams), special_every=5), fams, f"family {family} S={S}", family + S, counts)
    _report(f"pop family {family} S={S}", counts, t0)


def _full_uniform_level():
    ends, mu, sc = _special_level(1024, 2048, seed=2048)
    return Level(ends, mu, sc, 1024, 10)


FULL_ROWS = range(0, 2048, 31)          # 67 rows spread over a full-size level, and its last row below


def test_pop_edges_rows_of_a_full_size_uniform_level():
    """Rows of a 2048-row level at 1024 bins (q = 10) through k_pop6 (classified) and k_pop_coarse."""
    t0 = time.time()
    lv = _full_uniform_level()
    counts = Counter()
    _pop_rows(lv, list(FULL_ROWS) + [lv.R - 1], ("classified", "generic"), "full uniform level", 11, counts)
    _report("pop, rows of a full-size uniform level", counts, t0)


def _equal_mass_level(R, S, q, seed):
    from bitswap_b200.rand import Bins as RBins
    rs = np.random.RandomState(seed)
    m0 = torch.from_numpy(rs.normal(0, 0.5, (1, 1, R)).astype(np.float32))
    s0 = torch.from_numpy(rs.uniform(0.5, 2.0, (1, 1, R)).astype(np.float32))
    ends = RBins(m0, s0, q).endpoints().numpy().reshape(R, S - 1).astype(np.float64)
    mu = rs.normal(0, 1.5, R).astype(np.float32)
    sc = rs.uniform(0.1, 1.0, R).astype(np.float32)
    sc[0::5] = np.float32(1e-4)
    sc[1::5] = np.float32(0.1)
    mu[2::7] = rs.choice([-25.0, 25.0], size=mu[2::7].shape).astype(np.float32)
    return Level(ends, mu, sc, S, q)


def test_pop_edges_rows_of_a_top_level_equal_mass_level():
    """Rows of a 2048-row equal-mass level (rand.Bins, 1024 bins), the level the generic kernels code in production."""
    t0 = time.time()
    lv = _equal_mass_level(2048, 1024, 10, seed=5)
    counts = Counter()
    _pop_rows(lv, list(FULL_ROWS) + [lv.R - 1], ("generic",), "equal-mass level", 12, counts)
    _report("pop, rows of an equal-mass level", counts, t0)


def _pixel_level(seed):
    """The pixel rows of one 3x32x32 block: ImageBins (256 bins, one endpoint row for every dim, read with row stride 0),
    mu in [-1.1, 1.1] as the x head gives it, sigma from (2/255)/8 to 1."""
    from bitswap_b200.rand import ImageBins
    rs = np.random.RandomState(seed)
    R = 3 * 32 * 32
    ends = ImageBins(torch.float64, "cpu", 1).endpoints().numpy()
    mu = rs.uniform(-1.1, 1.1, R).astype(np.float32)
    sc = ((2.0 / 255.0) / 8.0 * np.exp(rs.uniform(0, np.log(8 * 255 / 2.0), R))).astype(np.float32)
    sc[::97] = np.float32((2.0 / 255.0) / 8.0)
    return Level(ends, mu, sc, 256, 8, shared_row=True)


def test_pop_edges_every_pixel_dim_of_a_block():
    """Every dim of a 3x32x32 block's pixel rows.  The endpoint row is shared, so each stream gets its own mu/sigma rows
    (stride L') and one launch covers many dims: per dim, the bins around the mode, the first and last live bins and their
    dead neighbours, bins 0 and 255, each on every head kind; k_pop6, k_pop_coarse and the fused pop."""
    t0 = time.time()
    lv = _pixel_level(21)
    tab, S, R = lv.tab, lv.S, lv.R
    rs = np.random.RandomState(22)
    counts = Counter()
    lp_of = np.array(VIEWS)[np.arange(R) % len(VIEWS)]
    short = lp_of - 1 > np.arange(R)                      # dims too low for their view: popped with L' = 1 instead
    for v, Lp in enumerate(VIEWS):
        dims = np.flatnonzero(((np.arange(R) % len(VIEWS) == v) & ~short) | (short if Lp == 1 else False))
        xs, rows, bins = [], [], []
        for t in dims:
            live = np.flatnonzero(tab.P[t] > 1)
            am = int(tab.P[t].argmax())
            b = np.unique(np.clip([0, S - 1, am - 1, am, am + 1, live[0] - 1, live[0], live[-1], live[-1] + 1], 0, S - 1))
            for kind in POP_KINDS:
                x, ok = pop_heads(tab.P[t, b], tab.C[t, b], kind, rs)
                check_pop_heads(x[ok], tab, np.full(ok.sum(), t), b[ok], kind)
                xs.append(x[ok])
                rows.append(np.full(ok.sum(), t))
                bins.append(b[ok])
        x, top = np.concatenate(xs), np.concatenate(rows)
        N = x.size
        view = top[:, None] + np.arange(-Lp + 1, 1)[None, :]
        st = Stacks(rs.randint(0, 1 << 32, (N, Lp), dtype=np.int64).astype(np.uint32), np.full(N, Lp), x)
        packed = st.packed()
        want_sym = pop(tab, view, st)
        assert np.array_equal(want_sym[:, -1], np.concatenate(bins))
        mu = torch.from_numpy(lv.mu.cpu().numpy()[view]).to(dev)
        sc = torch.from_numpy(lv.sc.cpu().numpy()[view]).to(dev)
        ss = StreamSet(N, 128)
        for fam in ("classified", "generic", "fused"):
            ss.import_packed(*packed)
            got_sym = _code(fam, False, lv, ss, N, 0, Lp, mu=mu, sc=sc)
            ss.raise_on_error()
            assert_same(f"pixel {fam} L'={Lp}", got_sym, ss.export(0, N), want_sym, st, top=Lp - 1)
            counts[fam] += N
    _report("pop, every pixel dim", counts, t0)


# ---- push -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", POW2 + [8, 12, 20, 100, 1020])
def test_push_every_row_symbol_pair(S):
    """Every (row, symbol) pair of 130 rows, from every push-threshold head, through k_rows6 + k_push_pairs, k_rows +
    k_push_pairs, the fused push and the table-driven push."""
    q = max(3, (S - 1).bit_length())
    t0 = time.time()
    ends, mu, sc = _special_level(S, 130, seed=S + 2)
    lv = Level(ends, mu, sc, S, q)
    if S >= 32 and not S & (S - 1):                   # the generic and fused kernels code powers of two from 32 bins
        fams = [f for f in ALL if f != "fused" or S <= 1024]
    else:
        fams = ["affine", "affine lpr32", "table"]
    counts = Counter()
    _push_rows(lv, 0, 130, fams, f"S={S}", S + 3, counts)
    _report(f"push S={S}", counts, t0)


@pytest.mark.parametrize("level", ["uniform", "equal-mass", "pixel"])
def test_push_every_row_symbol_pair_of_full_levels(level):
    t0 = time.time()
    if level == "uniform":
        lv, fams = _full_uniform_level(), ("classified", "generic", "fused", "table")
    elif level == "equal-mass":
        lv, fams = _equal_mass_level(2048, 1024, 10, seed=6), ("generic", "fused", "table")
    else:
        lv, fams = _pixel_level(23), ("classified", "generic", "fused", "table")
    counts = Counter()
    _push_rows(lv, 0, lv.R, fams, level, 7, counts, kinds=("lim-1", "lim"))
    _report(f"push, every (row, symbol) of the {level} level", counts, t0)
