"""Pins oracle/ (the CPU restatement) against the golden vectors that
tests/golden/make_golden.py produced from the reference's own classes."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O
from bitswap_b200.config import preset
from bitswap_b200 import synthetic
from bitswap_b200.rand import Bins, ImageBins

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def _kat_inputs(k):
    rs = np.random.RandomState(k["seed"])
    pm = rs.dirichlet(np.ones(k["S"]) * 0.5, size=k["L"])
    sym = rs.randint(0, k["S"], size=k["L"])
    w, head = synthetic.initial_words(k["N"], seed=100)
    return pm, sym, w, head


KATS = json.load(open(os.path.join(GOLDEN, "ans_kat.json")))


@pytest.mark.parametrize("k", KATS, ids=[k["name"] for k in KATS])
def test_ans_kat_c(k):
    pm, sym, w, head = _kat_inputs(k)
    assert O.state_digest(w, head) == k["init_sha"]
    P, C = O.tables_c(pm, 31, k["q"])
    P2, C2 = O.tables_np(pm, 31, k["q"])
    assert np.array_equal(P, P2) and np.array_equal(C, C2)
    assert [int(v) for v in P[0, :6]] == k["P_row0_head"]
    assert _sha(P) == k["P_sha"] and _sha(C) == k["C_sha"]
    a = O.AnsC(tables=(P, C))
    st = a.encode(O.CState(w, head), sym)
    assert (st.n + 1, hex(st.head), st.digest()) == (k["push_len"], k["push_head"], k["push_sha"])
    st2, psym = a.decode(O.CState(w, head))
    assert (st2.n + 1, hex(st2.head), st2.digest()) == (k["pop_len"], k["pop_head"], k["pop_sha"])
    assert [int(v) for v in psym[:6]] == k["pop_syms_head"] and _sha(psym.astype(np.int64)) == k["pop_syms_sha"]
    # inverse property both ways (reference round-trip, make_golden.py asserts the same)
    st3, rsym = a.decode(st)
    assert np.array_equal(rsym, sym) and st3.digest() == k["init_sha"]
    assert a.encode(st2, psym).digest() == k["init_sha"]


def test_ans_kat_port_literal():
    k = KATS[0]
    pm, sym, w, head = _kat_inputs(k)
    a = O.AnsPort(pm, 31, k["q"])
    init = [int(v) for v in w] + [head]
    pushed = a.encode(init.copy(), sym)
    assert (len(pushed), hex(pushed[-1])) == (k["push_len"], k["push_head"])
    assert O.CState.from_list(pushed).digest() == k["push_sha"]
    popped, ps = a.decode(init.copy())
    assert (len(popped), hex(popped[-1])) == (k["pop_len"], k["pop_head"])
    assert [int(v) for v in ps[:6]] == k["pop_syms_head"]


def test_underflow_is_indexerror():
    k = KATS[1]
    assert k["underflow_N512"] == "IndexError"
    pm, sym, _, _ = _kat_inputs(k)
    w, head = synthetic.initial_words(512, seed=100)
    a = O.AnsC(pm, 31, k["q"])
    with pytest.raises(IndexError):
        a.decode(O.CState(w, head))
    with pytest.raises(IndexError):
        O.AnsPort(pm[-600:], 31, k["q"]).decode([int(v) for v in w[:40]] + [head])


def test_tables_small_incl_ties():
    g = np.load(os.path.join(GOLDEN, "tables_small.npz"))
    for tag, q in (("a", 4), ("b", 8)):
        for fn in (O.tables_c, O.tables_np):
            P, C = fn(g["pm_" + tag], 31, q)
            assert np.array_equal(P, g["P_" + tag]) and np.array_equal(C, g["C_" + tag])


def test_pmfs_small():
    g = np.load(os.path.join(GOLDEN, "pmfs_small.npz"))
    t = torch.from_numpy
    # torch path is the reference's own expression on this host: bit-exact
    assert np.array_equal(O.logistic_pmfs_torch(t(g["ends"]), t(g["mu"]), t(g["sc"])).numpy(), g["pm"])
    assert np.array_equal(O.logistic_pmfs_torch(t(g["xe"]), t(g["xmu"]), t(g["xsc"])).numpy(), g["xpm"])
    one, zero = torch.ones(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
    assert np.array_equal(O.logistic_pmfs_torch(t(g["ends"]), zero, one).numpy(), g["prior"])
    # libm path: <= 1 ulp of cdf (SURVEY.md H2)
    assert np.abs(O.logistic_pmfs_c(g["ends"], g["mu"], g["sc"]) - g["pm"]).max() <= 4e-16
    assert np.abs(O.logistic_pmfs_c(g["xe"], g["xmu"], g["xsc"]) - g["xpm"]).max() <= 4e-16
    assert np.abs(O.logistic_pmfs_c(g["ends"], np.zeros(1), np.ones(1)) - g["prior"]).max() <= 4e-16


def test_bins_match_reference():
    g = np.load(os.path.join(GOLDEN, "bins.npz"))
    b = Bins(torch.zeros((1, 1, 4)), torch.ones((1, 1, 4)), 6)
    assert b.endpoints().dtype == torch.float32          # the top-level table is float32 (SURVEY.md 3.5)
    assert np.array_equal(b.endpoints().numpy(), g["top_end"]) and np.array_equal(b.centres().numpy(), g["top_cen"])
    ib = ImageBins(torch.float64, "cpu", 3)
    assert np.array_equal(ib.endpoints().numpy(), g["img_end"]) and np.array_equal(ib.centres().numpy(), g["img_cen"])
    b64 = Bins(torch.zeros(2, dtype=torch.float64) + 0.25, torch.ones(2, dtype=torch.float64) * 0.5, 4)
    assert np.array_equal(b64.endpoints().numpy(), g["b64_end"]) and np.array_equal(b64.centres().numpy(), g["b64_cen"])


def _model_oracle_vs_golden(name, dtype, tol):
    cfg = preset(name)
    g = np.load(os.path.join(GOLDEN, f"model_{name}.npz"))
    m = O.ModelOracle(cfg, synthetic.synthetic_state_dict(cfg, seed=50, varied=True), dtype=dtype)
    _, zcen = synthetic.synthetic_bins(cfg, seed=0)
    xcen = ImageBins(torch.float64, "cpu", cfg.xdim).centres()
    zr = torch.arange(cfg.zdim)

    def close(got, key):
        want = g[key]
        return bool(np.all(np.abs(got[0].numpy() - want) < tol(want)))

    for i in range(cfg.nz):
        if i == 0:
            given = xcen[torch.arange(cfg.xdim), torch.from_numpy(g["x"].astype(np.int64))]
        else:
            given = zcen[i - 1, zr, torch.from_numpy(g[f"zsym_in_infer{i}"].astype(np.int64))]
        mu, sc = m.infer(i)(given.unsqueeze(0))
        assert close(mu, f"infer{i}_mu") and close(sc, f"infer{i}_scale")
        z = zcen[i, zr, torch.from_numpy(g[f"zsym_in_gen{i}"].astype(np.int64))]
        mu, sc = m.generate(i)(z.unsqueeze(0))
        assert close(mu, f"gen{i}_mu") and close(sc, f"gen{i}_scale")


@pytest.mark.parametrize("name", ["tiny", "tiny3"])
def test_model_oracle_matches_reference(name):
    """The float32 oracle repeats the reference's operations: within 2e-6 absolute of the golden outputs."""
    _model_oracle_vs_golden(name, torch.float32, lambda want: 2e-6)


@pytest.mark.parametrize("name", ["tiny", "tiny3"])
def test_model_oracle_float64_matches_reference(name):
    """The float64 oracle computes the reference model too (squeeze maps, scale transforms): it is the reference the
    per-layer and whole-net float64 GPU tests hold the kernels to.  The golden outputs are the reference's float32
    arithmetic, so it is held to 2e-6 relative to max(1, |output|) (measured: 2.5e-6 at |mu| = 5.3, 5e-7 relative)."""
    _model_oracle_vs_golden(name, torch.float64, lambda want: 2e-6 * np.maximum(1.0, np.abs(want)))


@pytest.mark.parametrize("name", ["tiny", "tiny3"])
@pytest.mark.parametrize("coder", ["c", "port"])
def test_bitswap_oracle_trace(name, coder):
    """Sender trace (len + sha after every op) equals the reference-classes run; receiver restores
    the initial state and the pixels."""
    g = json.load(open(os.path.join(GOLDEN, f"bitswap_{name}.json")))
    cfg = preset(name)
    torch.set_num_threads(4)
    m = O.ModelOracle(cfg, synthetic.synthetic_state_dict(cfg, seed=50, varied=True))
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    trace = []
    bs = O.BitSwapOracle(cfg, m, zend, zcen, coder=coder, pmf="torch", trace=trace)
    imgs = synthetic.synthetic_images(cfg, g["nimg"], seed=7)
    w, head = synthetic.initial_words(g["nwords"], seed=100)
    st = ([int(v) for v in w] + [head]) if coder == "port" else O.CState(w, head)
    for xi in range(g["nimg"]):
        st = bs.encode_image(st, imgs[xi])
    got = [(ln, sha) for _, ln, sha in trace]
    want = [(ln, sha) for _, ln, sha in g["trace"][1:]]
    assert got == want
    bs.trace = None
    for xi in reversed(range(g["nimg"])):
        st, x = bs.decode_image(st)
        assert np.array_equal(x, imgs[xi].reshape(-1))
    final = O.CState.from_list(st).digest() if coder == "port" else st.digest()
    assert final == g["trace"][0][2]


def test_bbans_oracle_roundtrip():
    cfg = preset("tiny")
    m = O.ModelOracle(cfg, synthetic.synthetic_state_dict(cfg, seed=50, varied=True))
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    bs = O.BitSwapOracle(cfg, m, zend, zcen, coder="c", pmf="c")
    imgs = synthetic.synthetic_images(cfg, 2, seed=7)
    w, head = synthetic.initial_words(900, seed=100)
    st = O.CState(w, head)
    init = st.digest()
    for xi in range(2):
        st = bs.encode_image_bbans(st, imgs[xi])
    for xi in reversed(range(2)):
        st, x = bs.decode_image_bbans(st)
        assert np.array_equal(x, imgs[xi].reshape(-1))
    assert st.digest() == init
