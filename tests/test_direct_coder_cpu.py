"""The direct-cdf quantiser on the CPU: its tables are valid on hostile rows and on perturbed cdf values, it codes at the
reference quantiser's rate, a numpy push-then-pop round trip on its tables is exact, and the `coder=` argument is
validated before any device work.  Runs without a GPU."""
import types

import numpy as np
import pytest

import coder_harness as H
from direct_harness import direct_tables
from oracle import oracle as O
from bitswap_b200.codec import BitSwapCodec, PipelinedCodec
from bitswap_b200.config import preset


def cdfs(e, mu, sc):
    """Logistic cdf values [L, S - 1] of rows e ([S - 1] shared, or [L, S - 1]) at mu, sc [L]."""
    e = np.broadcast_to(e, (mu.size, np.shape(e)[-1]))
    with np.errstate(over="ignore", invalid="ignore"):
        return 1.0 / (1.0 + np.exp(-((e - mu[:, None]) / sc[:, None])))


def assert_valid(P, C):
    S = P.shape[1]
    assert (P >= 1).all(), f"a bin of zero mass (min P {P.min()})"
    assert (P.sum(axis=1) == 1 << 31).all()
    assert (np.diff(C, axis=1) > 0).all() and (C[:, 0] == 0).all() and (C[:, S] == 1 << 31).all()
    assert (P[:, 0] >= 2).all() and (P[:, -1] >= 2).all()


def hostile_cdfs(S, rs):
    """Needle, constant, tiny-span, off-grid, every-bin-live and beyond-the-grid rows at S bins."""
    grid = np.linspace(-6.5, 6.5, S + 1)[1:-1]
    rows = [
        cdfs(grid, rs.normal(0, 1, 8), np.full(8, 1e-6)),                                   # needle
        cdfs(np.full(S - 1, 0.25), rs.normal(0, 1, 4), rs.uniform(0.1, 1, 4)),               # constant row
        cdfs(np.sort(rs.uniform(-1e-6, 1e-6, S - 1)) + 1000.0, np.array([1000.0] * 4), np.full(4, 1e-7)),   # tiny span
        cdfs(grid + rs.uniform(-0.3, 0.3, S - 1) * 13 / S, rs.normal(0, 2, 8), rs.uniform(0.05, 2, 8)),      # off-grid
        cdfs(grid, rs.normal(0, 1, 4), rs.uniform(5, 50, 4)),                                # every bin live
        cdfs(grid, np.array([-40.0, 40.0, -6.5, 6.5]), np.full(4, 0.3)),                     # beyond either end, on an edge
        np.sort(np.repeat(rs.uniform(0, 1, (4, (S - 1 + 3) // 4)), 4, axis=1)[:, :S - 1], axis=1),            # runs of equal cdf
    ]
    return np.concatenate([np.clip(np.nan_to_num(r, nan=0.0), 0.0, 1.0) for r in rows])


@pytest.mark.parametrize("S", [32, 256, 1024, 4096])
def test_tables_valid_on_hostile_and_perturbed_rows(S):
    rs = np.random.RandomState(S)
    F = hostile_cdfs(S, rs)
    assert_valid(*direct_tables(F))
    # an evaluation error of a few ulps, independently per value, can make F fall between neighbours
    for _ in range(4):
        Fp = np.clip(F + rs.randint(-4, 5, F.shape) * np.spacing(F), 0.0, 1.0)
        assert_valid(*direct_tables(Fp))
    P, C = direct_tables(np.full((2, S - 1), np.nan))          # NaN mu or sigma: every F counts as 0
    assert_valid(P, C)
    assert (C[:, 1:S] == 2 * np.arange(1, S)).all()


def _excess(pmf, P):
    """Expected code length under pmf minus the entropy, bits/symbol, per row."""
    with np.errstate(divide="ignore", invalid="ignore"):
        H_ = -np.where(pmf > 0, pmf * np.log2(np.where(pmf > 0, pmf, 1.0)), 0.0).sum(axis=1)
    return -(pmf * np.log2(P / 2.0 ** 31)).sum(axis=1) - H_


@pytest.mark.parametrize("kind", ["ordinary", "sharp", "pixel", "wide"])
def test_rate_matches_the_reference_quantiser(kind):
    """Expected code length within 1e-5 bits/symbol of the reference quantiser's (ANS.__init__) on the same cdf values."""
    rs = np.random.RandomState(7)
    if kind == "pixel":
        S, q, n = 256, 8, 1000
        e = ((np.arange(1, 256) - 127.5) / 127.5) - 1 / 255
        F = cdfs(e, rs.uniform(-1, 1, n), rs.uniform(0.01, 0.2, n))
    else:
        S, q, n = (4096, 12, 200) if kind == "wide" else (1024, 10, 800)
        e = np.linspace(-6.5, 6.5, S + 1)[1:-1]
        F = cdfs(e, rs.normal(0, 1, n), np.full(n, 0.01) if kind == "sharp" else rs.uniform(0.1, 2, n))
    pmf = np.diff(np.concatenate([np.zeros((n, 1)), F, np.ones((n, 1))], axis=1), axis=1)
    P_ref, _ = O.tables_np(pmf, 31, q)
    P_dir, _ = direct_tables(F)
    d = np.abs(_excess(pmf, P_ref) - _excess(pmf, P_dir))
    print(f"{kind}: max |direct - reference| {d.max():.2e} bits/symbol, mean excess over entropy "
          f"{_excess(pmf, P_dir).mean():.2e} (direct) {_excess(pmf, P_ref).mean():.2e} (reference)")
    assert d.max() < 1e-5


@pytest.mark.parametrize("S", [32, 1024, 4096])
def test_numpy_round_trip_on_direct_tables(S):
    """Push symbols onto seeded states with the numpy reference coder on direct tables, pop them back: symbols and states
    return exactly.  Includes the edge and threshold heads of the bin-edge tests."""
    rs = np.random.RandomState(S + 1)
    F = hostile_cdfs(S, rs)
    tab = H.RowTables(*direct_tables(F))
    R = tab.R
    N, L = 64, 24
    rows = rs.randint(0, R, (N, L))
    sym = rs.randint(0, S, (N, L))
    sym[:, :4] = [0, S - 1, 1, S - 2]
    st = H.Stacks.from_lists(H.initial_states(N, seed=3, n=200), cap=4096)
    before = st.to_lists()
    H.push(tab, rows, st, sym)
    got = H.pop(tab, rows, st)
    assert np.array_equal(got, sym) and st.to_lists() == before
    for kind in H.POP_KINDS:                       # heads exactly on the bin edges and the renormalisation points
        r = rs.randint(0, R, 256)
        s = rs.randint(0, S, 256)
        x, ok = H.pop_heads(tab.P[r, s], tab.C[r, s], kind, rs)
        x, r, s = x[ok], r[ok], s[ok]
        H.check_pop_heads(x, tab, r, s, kind)
        st = H.Stacks(np.ones((x.size, 4), np.uint32), np.full(x.size, 4), x)
        assert np.array_equal(H.pop(tab, r[:, None], st)[:, 0], s), kind


def test_coder_argument_is_validated_before_device_work():
    nothing = types.SimpleNamespace(device=0)     # never touched: the coder is checked first
    for bad in ("Direct", "fused", None, 1):
        with pytest.raises(ValueError, match="coder must be one of"):
            BitSwapCodec(preset("tiny3"), nothing, nothing, 4, coder=bad)
        with pytest.raises(ValueError, match="coder must be one of"):
            PipelinedCodec(preset("tiny3"), {}, nothing, 4, coder=bad)
