"""The latent coder on every endpoint grid discretize() can build, bin by bin against the exact function.

discretize() fits each latent dimension with np.linspace between the float16 extrema of its samples, so a level's rows can
be off-centre, narrow, far from zero, as wide as +-65504, a few float16 ulps wide, or constant.  The affine-row coder
(k_rows6 / k_pop6) leans on two things there: the rounding term of the row fit (k_row_meta) and the window widening by the
endpoint deviation (r6_plan).  These tests pin the row classification to its rule, run full-size levels of every grid family
through the verify build of k_rows6, run degenerate rows (zero-width bins) through the generic and fused coders, hold the
exported pmfs to the reference expression on the same grids, and run the codec on discretize()'s own tables with a constant
latent dimension -- all against the oracle coder on our pmfs."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from coder_harness import (check_vs_oracle, coder_paths, dev, draw, family_case, half, initial_states,   # noqa: E402
                           linspace_rows, oracle_tables, push_pop, ref_pmfs_cuda, run_2p, run_fused)
from codec_harness import gpu_oracle                                                # noqa: E402
from oracle import oracle as O                                                      # noqa: E402
from bitswap_b200 import synthetic                                                  # noqa: E402
from bitswap_b200.config import CodecConfig, preset, with_                          # noqa: E402
from bitswap_b200.model import Model                                                # noqa: E402
from bitswap_b200.codec import BitSwapCodec, Bins, BITSWAP, BBANS                  # noqa: E402
from bitswap_b200.streams import StreamSet                                          # noqa: E402
from bitswap_b200._lib import lib, check, cuda_stream_ptr                           # noqa: E402

FAMILIES = {1: "off-centre", 2: "float16 extrema", 3: "far and narrow", 4: "tiny span", 5: "dt near 64", 6: "perturbed"}


def _affine_rule(ends):
    """k_row_meta's classification restated: the line through the first and last endpoint, its worst deviation plus the
    rounding term emax * 2.3e-16; affine iff d > 0, dev <= 1e-13 max(1, emax) and emax < 1e6."""
    n = ends.shape[-1]
    a = ends[..., :1]
    d = (ends[..., -1:] - a) / (n - 1)
    dev = np.abs(ends - (np.arange(n) * d + a)).max(-1)
    emax = np.abs(ends).max(-1)
    dev = dev + emax * 2.3e-16
    return (d[..., 0] > 0) & (dev <= 1e-13 * np.maximum(1.0, emax)) & (emax < 1e6)


def _symbols(B, L, S, rs):
    sym = rs.randint(0, S, size=(B, L)).astype(np.int16)
    sym[:, :6] = [0, S - 1, 1, S - 2, S // 2, 0]
    return sym


# ---- the row classification ---------------------------------------------------------------------------------------------
def _special_rows(S):
    """One row per level, each a grid discretize() can build or a row just either side of the rule."""
    def lin(lo, hi):
        return linspace_rows(np.array([lo]), np.array([hi]), S)[0]

    def perturbed(f):
        e = lin(-300.0, 200.0)
        e[S // 3] += f * 1e-13 * 300.0
        return e
    return {
        "float16 +-65504": lin(-65504.0, 65504.0),
        "float16 -65504 .. 1234": lin(-65504.0, float(half(1234.3))),
        "one float16 ulp at 1000": lin(1000.0, 1000.5),
        "one float16 ulp at -2": lin(-2.0, -2.0 + 2.0 ** -10),
        "one float16 ulp at 0 (subnormal)": lin(0.0, 2.0 ** -24),
        "far and narrow": lin(45000.0, 45000.5),
        "0.5 x tolerance off the line": perturbed(0.5),
        "2 x tolerance off the line": perturbed(2.0),
        "constant": np.full(S - 1, 0.375),
        "emax >= 1e6": lin(1e6, 1e6 + 100.0),
    }


@pytest.mark.parametrize("q", [8, 12])
def test_row_classification_matches_the_rule_and_every_level_codes_exactly(q):
    """Bins over levels that are ordinary uniform grids except for one special row each: level_is_uniform equals the rule
    restated in numpy, and every level codes (classification on) exactly as the generic kernels and the oracle."""
    S = 1 << q
    special = _special_rows(S)
    cfg = CodecConfig(xs=(1, 32, 32), nz=len(special), zchannels=1, quantbits=q)
    L = cfg.zdim
    rs = np.random.RandomState(q)
    lo, hi = -6 - rs.uniform(0, 1, (cfg.nz, L)), 6 + rs.uniform(0, 1, (cfg.nz, L))
    zend = np.stack([linspace_rows(lo[i], hi[i], S) for i in range(cfg.nz)])
    at = [(37 * i + 5) % L for i in range(cfg.nz)]
    for i, row in enumerate(special.values()):
        zend[i, at[i]] = row
    zcen = np.zeros((cfg.nz, L, S))
    bins = Bins(cfg, zend, zcen)
    want = _affine_rule(zend).all(axis=1)
    got = np.array([bins.level_is_uniform(i) for i in range(cfg.nz)])
    names = list(special)
    assert np.array_equal(got, want), [(names[i], bool(got[i]), bool(want[i])) for i in np.flatnonzero(got != want)]
    assert not want[names.index("constant")] and not want[names.index("2 x tolerance off the line")]
    assert not want[names.index("emax >= 1e6")] and want[names.index("0.5 x tolerance off the line")]
    B = 3
    for i, name in enumerate(names):
        ends = zend[i]
        elo, ehi = ends[:, 0] - (ends[:, -1] - ends[:, 0]) / (S - 2), ends[:, -1] + (ends[:, -1] - ends[:, 0]) / (S - 2)
        mu, sc = draw(elo, ehi, S, B, rs)
        sym = _symbols(B, L, S, rs)
        states = initial_states(B, seed=40 + i, n=1500)
        res = run_2p(ends, mu, sc, S, q, states, sym, mode=-1)
        gen = run_2p(ends, mu, sc, S, q, states, sym, mode=0)
        assert gen[0] == res[0] and np.array_equal(gen[1], res[1]) and gen[2] == res[2], name
        check_vs_oracle(res, oracle_tables(ends, mu, sc, S, q), states, sym, range(B))


# ---- full-size levels of every grid family in verify mode ------------------------------------------------------------------
VERIFY_CASES = [(f, S) for f in FAMILIES for S in (32, 256, 1024, 4096)] + [(1, 2048), (3, 2048)]


@pytest.mark.parametrize("family,S", VERIFY_CASES)
def test_affine_rows_verified_on_every_grid_family(family, S):
    """2048 rows x B = 4 streams of one grid family through k_rows6 / k_pop6 in verify mode (every bin also evaluated with
    the exact function on the real endpoints): 0 disagreements, the worst trusted screening error at most a quarter of
    its window, and the same streams and symbols as the classification path and the oracle.  The affine kernels are forced
    so that a level with some rows outside the rule still runs them (those rows take the exact path for every bin)."""
    q = S.bit_length() - 1
    L, B = 2048, 4
    ends, mu, sc = family_case(family, L, S, B, seed=1000 * family + S)
    sym = _symbols(B, L, S, np.random.RandomState(S + family))
    states = initial_states(B, seed=70 * family, n=6000)
    stats = np.zeros(4, dtype=np.uint64)
    with coder_paths(verify=1):
        got = run_2p(ends, mu, sc, S, q, states, sym, mode=1)
        check(lib().bsw_rows6_verify_read(stats.ctypes.data))
    mism, worst, checked, exact_path = (int(v) for v in stats)
    n_aff = int(_affine_rule(ends).sum())
    print(f"{FAMILIES[family]} S={S}: {n_aff} of {L} rows affine, {checked} bins evaluated of {2 * B * L * S}, exact path "
          f"{100.0 * exact_path / max(checked, 1):.2f} % of evaluated, worst trusted error {worst / 10:.1f} % of the window, "
          f"{mism} mismatches")
    assert checked > 0 and mism == 0
    assert worst <= 250, worst
    if n_aff == L:                                        # the classification picks these kernels by itself
        cls = run_2p(ends, mu, sc, S, q, states, sym, mode=-1)
        assert got[0] == cls[0] and np.array_equal(got[1], cls[1]) and got[2] == cls[2]
    _check_picked_vs_oracle(got, ends, mu, sc, S, q, states, sym)


def _check_picked_vs_oracle(res, ends, mu, sc, S, q, states, sym, picks=(0, 3)):
    picks = list(picks)
    sub = ([res[0][b] for b in picks], res[1][picks], [res[2][b] for b in picks])
    check_vs_oracle(sub, oracle_tables(ends, mu[picks], sc[picks], S, q), [states[b] for b in picks], sym[picks],
                     range(len(picks)))


@pytest.mark.parametrize("family,S", VERIFY_CASES)
def test_generic_kernels_on_every_grid_family(family, S):
    """The same levels through the generic two-phase kernels (the path a whole level takes when one of its rows is outside
    the affine rule): streams and symbols equal to the oracle's."""
    q = S.bit_length() - 1
    L, B = 2048, 4
    ends, mu, sc = family_case(family, L, S, B, seed=1000 * family + S)
    sym = _symbols(B, L, S, np.random.RandomState(S + family))
    states = initial_states(B, seed=70 * family, n=6000)
    _check_picked_vs_oracle(run_2p(ends, mu, sc, S, q, states, sym, mode=0), ends, mu, sc, S, q, states, sym)


# ---- degenerate rows on the generic and fused coders -----------------------------------------------------------------------
def _degenerate_case(L, S, B, seed):
    """Constant rows, rows with runs of equal endpoints (a fine grid rounded to float16), tiny spans, and ordinary rows."""
    rs = np.random.RandomState(seed)
    lo, hi = -6 - rs.uniform(0, 1, L), 6 + rs.uniform(0, 1, L)
    kind = np.arange(L) % 6
    lo[kind == 0] = hi[kind == 0] = rs.choice([0.0, 0.375, -20.0, 65504.0, -3e-5], (kind == 0).sum())
    lo[kind == 1], hi[kind == 1] = -3.0, 3.0                            # rounded to float16 below: runs of equal endpoints
    lo[kind == 2] = rs.choice([0.0, 1000.0], (kind == 2).sum())
    hi[kind == 2] = lo[kind == 2] + np.ldexp(1.0, -rs.randint(20, 25, (kind == 2).sum()))
    lo[kind == 3], hi[kind == 3] = 1.0, 1.0 + 2.0 ** -10                # one float16 ulp: S - 1 endpoints in [1, 1 + 2^-10]
    ends = linspace_rows(lo, hi, S)
    ends[kind == 1] = half(ends[kind == 1])
    ends[kind == 4] = np.repeat(ends[kind == 4][:, ::8], 8, axis=1)[:, :S - 1]    # equal in runs of 8
    mu, sc = draw(lo, hi, S, B, rs)
    return ends, mu, sc


@pytest.mark.parametrize("coder", ["generic", "classified", "affine", "fused"])
@pytest.mark.parametrize("S", [32, 1024, 4096])
def test_degenerate_rows_on_the_generic_and_fused_coders(S, coder):
    """Rows with zero-width bins (constant rows, runs of equal endpoints) and tiny spans: pop, then push, through the generic
    kernels, the classification path (these rows send the level to the generic kernels), the forced affine kernels and
    (up to 1024 bins) the fused coder -- each against the oracle on our pmfs."""
    if coder == "fused" and S > 1024:
        pytest.skip("the fused coder codes up to 1024 bins")
    q = S.bit_length() - 1
    L, B = 300, 6
    ends, mu, sc = _degenerate_case(L, S, B, seed=S)
    assert (np.diff(ends, axis=1) == 0).any(axis=1).sum() >= L // 3
    sym = _symbols(B, L, S, np.random.RandomState(S + 1))
    states = initial_states(B, seed=S, n=2000)
    tabs = oracle_tables(ends, mu, sc, S, q)
    if coder == "fused":
        res = run_fused(ends, mu, sc, S, q, states, sym)
    else:
        res = run_2p(ends, mu, sc, S, q, states, sym, {"generic": 0, "classified": -1, "affine": 1}[coder])
    check_vs_oracle(res, tabs, states, sym, range(B))


ROUNDTRIP_CASES = [("tiny span", S) for S in (32, 256, 1024)] + [("degenerate", S) for S in (32, 1024, 4096)]


@pytest.mark.parametrize("coder", ["generic", "classified", "affine", "fused"])
@pytest.mark.parametrize("rows,S", ROUNDTRIP_CASES)
def test_push_then_pop_round_trip_on_tiny_and_degenerate_rows(rows, S, coder):
    """push every row's symbol (edge bins included), then pop: the symbols and the initial states come back, and the
    pushed states are the oracle's.  The generic kernels' push takes its integers from k_rows and their pop re-evaluates
    the chunk from k_rows' bases, so a wrong k_rows integer breaks this round trip, not only the agreement with the
    reference."""
    if coder == "fused" and S > 1024:
        pytest.skip("the fused coder codes up to 1024 bins")
    q = S.bit_length() - 1
    B = 4
    if rows == "tiny span":
        ends, mu, sc = family_case(4, 1024, S, B, seed=5000 + S)
    else:
        ends, mu, sc = _degenerate_case(300, S, B, seed=S + 9)
    L = ends.shape[0]
    sym = _symbols(B, L, S, np.random.RandomState(S + 2))
    states = initial_states(B, seed=S + 3, n=500)
    pushed, popped, back = push_pop(ends, mu, sc, S, q, states, sym, coder)
    assert np.array_equal(popped, sym) and back == states
    tabs = oracle_tables(ends, mu, sc, S, q)
    for b in range(B):
        assert pushed[b] == O.AnsC(tables=tabs[b]).encode(O.CState.from_list(states[b]), sym[b].astype(np.int64)).to_list()


# ---- the exact function on these grids -------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", list(FAMILIES) + ["degenerate"])
def test_exported_pmfs_equal_the_reference_expression_on_every_grid_family(family):
    """bsw_logistic_pmfs (the pmfs the oracle's tables are built from) is bit-identical to the reference's float64 torch
    expression evaluated on this GPU, on every grid family."""
    for S in (256, 4096):
        L = 512
        if family == "degenerate":
            ends, mu, sc = _degenerate_case(L, S, 1, seed=S + 3)
        else:
            ends, mu, sc = family_case(family, L, S, 1, seed=77 * family + S)
        e = torch.from_numpy(np.ascontiguousarray(ends)).to(dev)
        m = torch.from_numpy(mu[0]).double().to(dev)
        s = torch.from_numpy(sc[0]).double().to(dev)
        out = torch.empty((L, S), dtype=torch.float64, device=dev)
        check(lib().bsw_logistic_pmfs(e.data_ptr(), S - 1, m.data_ptr(), s.data_ptr(), 1, L, S, out.data_ptr(), cuda_stream_ptr()))
        ref = ref_pmfs_cuda(e, m, s)
        assert torch.equal(out, ref), f"S={S}: {(out != ref).sum().item()} of {out.numel()} pmfs differ from torch-CUDA"


# ---- the real path: discretize()'s own tables, one constant dimension ------------------------------------------------------
_DISC = {}


def _discretized(name, q):
    """discretize() on the synthetic model, then dimension 5 of level 0 replaced by the row discretize() builds for a
    dimension whose samples are all equal (bsw_discretize_fold on constant float16 samples, then bsw_discretize_edges)."""
    if (name, q) not in _DISC:
        from bitswap_b200.discretization import discretize
        cfg = with_(preset(name), quantbits=q)
        sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
        m = Model.from_config(cfg, max_batch=128).load_state_dict(sd)
        m.compress()
        imgs = torch.from_numpy(synthetic.synthetic_images(cfg, 512, seed=17, kind="smooth"))
        zend, zcen = discretize(cfg.nz, q, torch.float64, "cpu", m, "synthetic", images=imgs, ppb=2)
        S = 1 << q
        mm = torch.empty(2, dtype=torch.int32, device=dev)
        samples = torch.full((64, 1), 0.8125, dtype=torch.float16, device=dev)
        ze = torch.empty(S - 1, dtype=torch.float64, device=dev)
        zc = torch.empty(S, dtype=torch.float64, device=dev)
        check(lib().bsw_discretize_reset(mm.data_ptr(), 1, cuda_stream_ptr()))
        check(lib().bsw_discretize_fold(samples.data_ptr(), mm.data_ptr(), 64, 1, cuda_stream_ptr()))
        check(lib().bsw_discretize_edges(mm.data_ptr(), 1, q, ze.data_ptr(), S - 1, zc.data_ptr(), S, cuda_stream_ptr()))
        torch.cuda.synchronize()
        assert torch.all(ze == 0.8125) and torch.all(zc == 0.8125)
        zend[0, 5], zcen[0, 5] = ze.cpu(), zc.cpu()
        m.compress()
        _DISC[(name, q)] = (cfg, m, sd, zend, zcen)
    return _DISC[(name, q)]


@pytest.mark.parametrize("scheme", [BITSWAP, BBANS])
@pytest.mark.parametrize("name,q", [("tiny", 8), ("tiny", 10), ("tiny", 12), ("tiny3", 8), ("tiny3", 12)])
def test_codec_on_discretized_bins_with_a_constant_dimension_vs_oracle(name, q, scheme):
    """The codec on the tables discretize() builds, with one constant latent dimension (which moves its level to the
    generic kernels): every stream equals the oracle recursion driven with the same nets, and decoding restores the
    images and the initial states."""
    cfg, m, sd, zend, zcen = _discretized(name, q)
    bins = Bins(cfg, zend, zcen)
    rule = _affine_rule(zend.numpy()).all(axis=1)
    assert not rule[0] and rule[1:cfg.nz - 1].all()
    assert [bins.level_is_uniform(i) for i in range(cfg.nz - 1)] == list(rule[:cfg.nz - 1])
    B, nimg = 4, 2
    codec = BitSwapCodec(cfg, m, bins, B)
    ss = StreamSet(B, 1 << 15)
    imgs = synthetic.synthetic_images(cfg, B * nimg, seed=31, kind="smooth").reshape(nimg, B, *cfg.xs)
    states = initial_states(B, seed=200, n=4000)
    ss.import_lists(states)
    for xi in range(nimg):
        codec.encode(ss, torch.from_numpy(imgs[xi]).cuda(), scheme=scheme)
    ss.raise_on_error()
    got = ss.export_lists()
    for b in range(B):
        orc = gpu_oracle(cfg, m, sd, zend, zcen, cls=O.BitSwapOracle)
        st = O.CState.from_list(states[b])
        for xi in range(nimg):
            st = (orc.encode_image if scheme == BITSWAP else orc.encode_image_bbans)(st, imgs[xi, b])
        assert got[b] == st.to_list(), f"stream {b} differs from the oracle"
    for xi in reversed(range(nimg)):
        out = codec.decode(ss, B, scheme=scheme)
        assert np.array_equal(out.cpu().numpy(), imgs[xi])
    ss.raise_on_error()
    assert ss.export_lists() == states
