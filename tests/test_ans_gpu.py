"""GPU parity of the coder kernels against the oracle (through the C ABI, ctypes).

Parity ladder (SURVEY.md 8c):
  P0  integer coder on injected integer tables      -> state lists bit-identical to the oracle
  P1  table quantiser on injected float64 pmfs      -> P, C bit-identical to ANS.__init__
  P2  float64 logistic pmfs                         -> == torch-CUDA's own sigmoid expression bit for bit,
                                                       <= 4e-16 from the torch-CPU golden; and feeding OUR
                                                       pmfs to the oracle coder reproduces OUR fused-kernel
                                                       state bit for bit.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from coder_harness import (check_vs_oracle, coder_paths, initial_states, level_case, oracle_tables, pad_big,   # noqa: E402
                           ref_pmfs_cuda, run_2p, run_fused)
from oracle import oracle as O                      # noqa: E402  (checker only)
from bitswap_b200 import synthetic                   # noqa: E402
from bitswap_b200._lib import lib, check, cuda_stream_ptr   # noqa: E402
from bitswap_b200.ans import ANS                     # noqa: E402
from bitswap_b200.streams import StreamSet           # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KATS = json.load(open(os.path.join(GOLDEN, "ans_kat.json")))
dev = "cuda"


def _kat_inputs(k):
    rs = np.random.RandomState(k["seed"])
    pm = rs.dirichlet(np.ones(k["S"]) * 0.5, size=k["L"])
    sym = rs.randint(0, k["S"], size=k["L"])
    w, head = synthetic.initial_words(k["N"], seed=100)
    return pm, sym, [int(v) for v in w] + [head]


@pytest.mark.parametrize("k", KATS, ids=[k["name"] for k in KATS])
def test_kat_dropin_ans(k):
    """The reference's own call sequence on the drop-in class reproduces the reference's states."""
    pm, sym, st0 = _kat_inputs(k)
    a = ANS(torch.from_numpy(pm).to(dev), 31, k["q"])
    assert [int(v) for v in a.pmfs[0, :6]] == k["P_row0_head"]
    pushed = a.encode(st0.copy(), torch.from_numpy(sym).to(dev))
    assert (len(pushed), hex(pushed[-1])) == (k["push_len"], k["push_head"])
    assert O.CState.from_list(pushed).digest() == k["push_sha"]
    popped, psym = a.decode(st0.copy())
    assert psym.dtype == torch.int64 and psym.device.type == "cuda"
    assert (len(popped), hex(popped[-1])) == (k["pop_len"], k["pop_head"])
    assert O.CState.from_list(popped).digest() == k["pop_sha"]
    assert [int(v) for v in psym[:6].cpu()] == k["pop_syms_head"]
    back, rsym = a.decode(pushed.copy())
    assert back == st0 and np.array_equal(rsym.cpu().numpy(), sym)
    assert a.encode(popped.copy(), psym) == st0


def test_underflow_and_overflow_map_to_reference_exceptions():
    k = KATS[1]
    pm, sym, _ = _kat_inputs(k)
    w, head = synthetic.initial_words(512, seed=100)
    a = ANS(torch.from_numpy(pm).to(dev), 31, k["q"])
    with pytest.raises(IndexError):
        a.decode([int(v) for v in w] + [head])
    # overflow: a stream set with too little capacity
    ss = StreamSet(1, 32)
    ss.fill(w[:20], head)
    s32 = torch.from_numpy(sym.astype(np.int32)).to(dev)
    check(lib().bsw_ans_push(ss.handle, 0, 1, a._P.data_ptr(), a._C.data_ptr(), 0, 0, s32.data_ptr(),
                             a.seq_len, a.support, 31, cuda_stream_ptr()))
    with pytest.raises(OverflowError):
        ss.raise_on_error()


def test_out_of_range_symbols_raise_index_error_like_the_reference():
    """ADVICE r1: the reference indexes self.pmfs[i, s] (cifar_compress.py:50) -- a symbol outside the support or a symbol
    vector of the wrong length is an IndexError there; here it must neither read device memory out of bounds nor
    silently corrupt the stream."""
    k = KATS[0]
    pm, sym, st = _kat_inputs(k)
    a = ANS(torch.from_numpy(pm).cuda(), 31, k["q"])
    bad = sym.copy(); bad[3] = k["S"]
    with pytest.raises(IndexError):
        a.encode(list(st), torch.from_numpy(bad))
    with pytest.raises(IndexError):
        a.encode(list(st), torch.from_numpy(sym[:-1]))
    bad[3] = -1
    with pytest.raises(IndexError):
        a.encode(list(st), torch.from_numpy(bad))
    # device-side check of the batched entry points: the stream is flagged, nothing is read out of bounds
    S, L, B = k["S"], k["L"], 3
    P, C = O.tables_c(pm, 31, k["q"])
    dP, dC = torch.from_numpy(P.astype(np.uint32).view(np.int32)).cuda(), torch.from_numpy(C.astype(np.uint32).view(np.int32)).cuda()
    s32 = torch.from_numpy(np.tile(sym, (B, 1)).astype(np.int32)).cuda()
    s32[1, 7] = S + 5
    ss = StreamSet(B, 4096)
    ss.import_lists([st] * B)
    check(lib().bsw_ans_push(ss.handle, 0, B, dP.data_ptr(), dC.data_ptr(), 0, 0, s32.data_ptr(), L, S, 31, cuda_stream_ptr()))
    _, _, f = ss.sizes()
    assert f.tolist() == [0, 4, 0]
    with pytest.raises(IndexError):
        ss.raise_on_error()
    for mode in (0, 1):                                       # two-phase push, generic and affine-row kernels
        ends = np.linspace(-6.5, 6.5, 65)[None, 1:-1].repeat(L, 0)
        mu = np.zeros((B, L), dtype=np.float32); sc = np.full((B, L), 0.5, dtype=np.float32)
        s16 = np.tile((sym % 64).astype(np.int16), (B, 1)); s16[2, 5] = 64
        with pytest.raises(IndexError):
            run_2p(ends, mu, sc, 64, 6, [st] * B, s16, mode, cap=1 << 14)


def test_bad_arguments_are_rejected():
    ss = StreamSet(2, 64)
    rc = lib().bsw_ans_push(ss.handle, 1, 2, None, None, 0, 0, None, 4, 4, 31, None)
    assert rc == 4 and b"range" in lib().bsw_last_error()


@pytest.mark.parametrize("L,S,q", [(8, 16, 4), (12, 16, 4), (300, 100, 6), (512, 256, 8), (256, 1024, 10), (40, 3000, 10),
                                   (64, 2, 1), (64, 4, 2), (64, 8, 3), (48, 2048, 11), (24, 4096, 12)])
def test_p1_tables_bit_identical(L, S, q):
    g = np.load(os.path.join(GOLDEN, "tables_small.npz"))
    rs = np.random.RandomState(L + S)
    if (L, S) == (12, 16):
        pm, Pw, Cw = g["pm_a"], g["P_a"], g["C_a"]          # includes tied-argmax rows (reference tie rule)
    else:
        pm = rs.dirichlet(np.ones(S) * rs.choice([0.05, 0.5, 5.0]), size=L)
        pm[0] = 1.0 / S                                       # exact tie across the whole row
        Pw, Cw = O.tables_c(pm, 31, q)
    a = ANS(torch.from_numpy(pm).to(dev), 31, q)
    assert np.array_equal(a.pmfs, Pw) and np.array_equal(a.cdfs, Cw)


@pytest.mark.parametrize("B,L,S,shared", [(37, 200, 16, False), (64, 333, 100, False), (33, 512, 256, True), (16, 700, 1024, False)])
def test_p0_batched_coder_vs_oracle(B, L, S, shared):
    """Injected integer tables + symbols + initial words: every stream's exported list == oracle's."""
    rs = np.random.RandomState(B * 7 + S)
    q = 4
    T = 1 if shared else B
    pm = rs.dirichlet(np.ones(S) * 0.3, size=(T, L))
    tabs = [O.tables_c(pm[t], 31, q) for t in range(T)]
    P = torch.from_numpy(np.stack([t[0] for t in tabs]).astype(np.uint32).view(np.int32)).to(dev)
    C = torch.from_numpy(np.stack([t[1] for t in tabs]).astype(np.uint32).view(np.int32)).to(dev)
    sym = rs.randint(0, S, size=(B, L)).astype(np.int32)
    states = initial_states(B, seed=100, n=400, step=13)
    ss = StreamSet(B, 4096)
    ss.import_lists(states)
    pss, css = (0, 0) if shared else (L * S, L * (S + 1))
    dsym = torch.from_numpy(sym).to(dev)
    # push, compare; then pop everything back, compare symbols and the restored state
    check(lib().bsw_ans_push(ss.handle, 0, B, P.data_ptr(), C.data_ptr(), pss, css, dsym.data_ptr(), L, S, 31, cuda_stream_ptr()))
    ss.raise_on_error()
    got = ss.export_lists()
    for b in range(B):
        a = O.AnsC(tables=tabs[0 if shared else b])
        want = a.encode(O.CState.from_list(states[b]), sym[b]).to_list()
        assert got[b] == want, f"stream {b} differs after push"
    out = torch.zeros((B, L), dtype=torch.int32, device=dev)
    check(lib().bsw_ans_pop(ss.handle, 0, B, P.data_ptr(), C.data_ptr(), pss, css, out.data_ptr(), L, S, 31, cuda_stream_ptr()))
    ss.raise_on_error()
    assert np.array_equal(out.cpu().numpy(), sym)
    assert ss.export_lists() == states
    # pop-first (bits-back direction) on a sub-range of streams only
    first, cnt = 3, B - 5
    check(lib().bsw_ans_pop(ss.handle, first, cnt, P.data_ptr() + (0 if shared else first * L * S * 4),
                            C.data_ptr() + (0 if shared else first * L * (S + 1) * 4), pss, css, out.data_ptr(), L, S, 31,
                            cuda_stream_ptr()))
    ss.raise_on_error()
    got = ss.export_lists()
    o = out.cpu().numpy()
    for b in range(B):
        if first <= b < first + cnt:
            a = O.AnsC(tables=tabs[0 if shared else b])
            st, s = a.decode(O.CState.from_list(states[b]))
            assert got[b] == st.to_list() and np.array_equal(o[b - first], s)
        else:
            assert got[b] == states[b]


def test_p2_logistic_pmfs():
    g = np.load(os.path.join(GOLDEN, "pmfs_small.npz"))
    for ends, mu, sc, want in ((g["ends"], g["mu"], g["sc"], g["pm"]), (g["xe"], g["xmu"], g["xsc"], g["xpm"]),
                               (g["ends"], np.zeros(1), np.ones(1), g["prior"])):
        L, S = want.shape
        e, m, s = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (ends, mu, sc))
        out = torch.empty((L, S), dtype=torch.float64, device=dev)
        check(lib().bsw_logistic_pmfs(e.data_ptr(), S - 1, m.data_ptr(), s.data_ptr(), 1 if m.numel() > 1 else 0, L, S,
                                      out.data_ptr(), cuda_stream_ptr()))
        assert np.abs(out.cpu().numpy() - want).max() <= 4e-16          # vs torch-CPU (reference classes) golden
        assert torch.equal(out, ref_pmfs_cuda(e, m, s))                  # vs the reference expression on this GPU
    # a full-size level: 2048 x 1024, bit-exact against torch-CUDA
    rs = np.random.RandomState(1)
    L, S = 2048, 1024
    lo, hi = -6 - rs.uniform(0, 1, L), 6 + rs.uniform(0, 1, L)
    e = torch.from_numpy(np.linspace(lo, hi, S + 1, axis=1)[:, 1:-1].copy()).to(dev)
    m = torch.from_numpy(rs.normal(0, 2, L).astype(np.float32)).double().to(dev)
    s = torch.from_numpy(rs.uniform(0.1, 1.0, L).astype(np.float32)).double().to(dev)
    out = torch.empty((L, S), dtype=torch.float64, device=dev)
    check(lib().bsw_logistic_pmfs(e.data_ptr(), S - 1, m.data_ptr(), s.data_ptr(), 1, L, S, out.data_ptr(), cuda_stream_ptr()))
    ref = ref_pmfs_cuda(e, m, s)
    assert torch.equal(out, ref), f"{(out != ref).sum().item()} of {out.numel()} pmfs differ from torch-CUDA"


def _pad_inf(ends):
    L, Sm1 = ends.shape
    out = np.full((L, Sm1 + 1), np.inf)
    out[:, :Sm1] = ends
    return out


@pytest.mark.parametrize("B,L,S,q,kind", [(9, 100, 64, 6, "z"), (20, 256, 128, 7, "z"), (33, 3072, 256, 8, "x"),
                                         (17, 2048, 1024, 10, "z"), (5, 515, 512, 9, "z"), (6, 64, 32, 5, "z")])
def test_p2_fused_logistic_coder_vs_oracle_on_our_pmfs(B, L, S, q, kind):
    """Fused kernels (table in registers, reciprocal-division shortcut) vs: our exported float64 pmfs (true
    division) -> oracle ANS.__init__ -> oracle coder.  Bit-identical states and symbols for every stream."""
    rs = np.random.RandomState(B + L + S)
    if kind == "x":      # ImageBins: one endpoint row shared by all dims, scale shared by all streams
        from bitswap_b200.rand import ImageBins
        ends = ImageBins(torch.float64, "cpu", 1).endpoints().numpy()          # [1, 255]
        ends_rows = np.repeat(ends, L, axis=0)
        mu = rs.uniform(-1, 1, (B, L)).astype(np.float32)
        sc = np.repeat(rs.uniform(0.003, 0.7, (1, L)).astype(np.float32), B, axis=0)
        ers, sss = 0, 0
    else:
        lo, hi = -6 - rs.uniform(0, 1, L), 6 + rs.uniform(0, 1, L)
        ends_rows = np.linspace(lo, hi, S + 1, axis=1)[:, 1:-1].copy()
        ends = ends_rows
        mu = rs.normal(0, 2, (B, L)).astype(np.float32)
        sc = rs.uniform(0.1, 1.0, (B, L)).astype(np.float32)
        ers, sss = S, L
    e_pad = torch.from_numpy(_pad_inf(ends)).to(dev)
    e_raw = torch.from_numpy(np.ascontiguousarray(ends_rows)).to(dev)
    dmu, dsc = torch.from_numpy(mu).to(dev), torch.from_numpy(sc).to(dev)
    dsc_arg = dsc[:1].contiguous() if kind == "x" else dsc
    states = initial_states(B, seed=100, n=1500)
    ss = StreamSet(B, 1 << 14)
    ss.import_lists(states)
    tabs = oracle_tables(ends_rows, mu, sc, S, q)                   # oracle side, on OUR pmfs
    # pop first (bits-back), then push other symbols
    out = torch.zeros((B, L), dtype=torch.int16, device=dev)
    check(lib().bsw_logistic_pop(ss.handle, 0, B, dmu.data_ptr(), L, dsc_arg.data_ptr(), sss, e_pad.data_ptr(), ers,
                                 out.data_ptr(), L, S, 31, q, cuda_stream_ptr()))
    ss.raise_on_error()
    got = ss.export_lists()
    o = out.cpu().numpy()
    ost = []
    for b in range(B):
        st, s = O.AnsC(tables=tabs[b]).decode(O.CState.from_list(states[b]))
        assert np.array_equal(o[b], s), f"stream {b}: popped symbols differ"
        assert got[b] == st.to_list(), f"stream {b}: state differs after pop"
        ost.append(st)
    sym = rs.randint(0, S, size=(B, L)).astype(np.int16)
    sym[:, :4] = [0, S - 1, S // 2, 1]                       # edge bins
    dsym = torch.from_numpy(sym).to(dev)
    check(lib().bsw_logistic_push(ss.handle, 0, B, dmu.data_ptr(), L, dsc_arg.data_ptr(), sss, e_pad.data_ptr(), ers,
                                  dsym.data_ptr(), L, S, 31, q, cuda_stream_ptr()))
    ss.raise_on_error()
    got = ss.export_lists()
    for b in range(B):
        want = O.AnsC(tables=tabs[b]).encode(ost[b], sym[b].astype(np.int64)).to_list()
        assert got[b] == want, f"stream {b}: state differs after push"
    # inverse: popping again returns the pushed symbols and the post-pop state
    check(lib().bsw_logistic_pop(ss.handle, 0, B, dmu.data_ptr(), L, dsc_arg.data_ptr(), sss, e_pad.data_ptr(), ers,
                                 out.data_ptr(), L, S, 31, q, cuda_stream_ptr()))
    assert np.array_equal(out.cpu().numpy(), sym)
    # materialised-table kernel == quantiser on our pmfs
    P = torch.empty((L, S), dtype=torch.int32, device=dev)
    C = torch.empty((L, S + 1), dtype=torch.int32, device=dev)
    mu64, sc64 = dmu[0].double().contiguous(), dsc[0].double().contiguous()
    check(lib().bsw_logistic_tables(e_raw.data_ptr(), S - 1, mu64.data_ptr(), sc64.data_ptr(), 1, L, S, 31, q,
                                    P.data_ptr(), C.data_ptr(), cuda_stream_ptr()))
    assert np.array_equal(P.cpu().numpy().view(np.uint32).astype(np.int64), tabs[0][0])
    assert np.array_equal(C.cpu().numpy().view(np.uint32).astype(np.int64), tabs[0][1])


def test_fused_underflow_flags_stream():
    L, S, q = 512, 256, 8
    rs = np.random.RandomState(0)
    from bitswap_b200.rand import ImageBins
    e_pad = torch.from_numpy(_pad_inf(ImageBins(torch.float64, "cpu", 1).endpoints().numpy())).to(dev)
    mu = torch.from_numpy(rs.uniform(-1, 1, (2, L)).astype(np.float32)).to(dev)
    sc = torch.full((1, L), 0.5, dtype=torch.float32, device=dev)
    ss = StreamSet(2, 4096)
    w, head = synthetic.initial_words(2000, seed=100)
    ss.import_lists([[int(v) for v in w[:10]] + [head], [int(v) for v in w] + [head]])
    out = torch.zeros((2, L), dtype=torch.int16, device=dev)
    check(lib().bsw_logistic_pop(ss.handle, 0, 2, mu.data_ptr(), L, sc.data_ptr(), 0, e_pad.data_ptr(), 0,
                                 out.data_ptr(), L, S, 31, q, cuda_stream_ptr()))
    _, _, flags = ss.sizes()
    assert flags.tolist() == [1, 0]
    with pytest.raises(IndexError):
        ss.raise_on_error()


def test_cdf_fast_equals_exact():
    """The lean float64 cdf of the two-phase kernels (hand-inlined libdevice exp + Newton reciprocal, no range
    branches) against the exact one (IEEE division + exp()) on 2^27 random triples incl. far tails."""
    import ctypes
    bad = ctypes.c_int64(-1)
    ex = (ctypes.c_double * 5)()
    check(lib().bsw_selftest_cdf(1 << 27, 12345, ctypes.byref(bad), ex))
    assert bad.value == 0, f"{bad.value} mismatches, e.g. (e, mu, sigma, fast, exact) = {list(ex)}"


def test_packed_export_import_roundtrip():
    """Device gather/scatter serialisation == the per-stream export, and import restores every stream."""
    B = 37
    ss = StreamSet(B, 512)
    rs = np.random.RandomState(3)
    states = []
    for b in range(B):
        n = int(rs.randint(0, 500))
        states.append([int(v) for v in rs.randint(0, 1 << 32, size=n, dtype=np.uint64)] + [int(rs.randint(1 << 32, 1 << 62))])
    ss.import_lists(states)
    w, o, h = ss.export_packed()
    w2, o2, h2, _ = ss.export()
    assert np.array_equal(w, w2) and np.array_equal(o, o2) and np.array_equal(h, h2)
    w, o, h = w.copy(), o.copy(), h.copy()
    ss2 = StreamSet(B, 512)
    ss2.import_packed_fast(w, o, h)
    torch.cuda.synchronize()
    assert ss2.export_lists() == states
    sub_w, sub_o, sub_h = ss.export_packed(first=5, count=9)
    assert np.array_equal(sub_o, o[5:15] - o[5]) and np.array_equal(sub_w, w[o[5]:o[14]])


@pytest.mark.parametrize("S,q,mode", [(1024, 10, 0), (1024, 10, -1), (1024, 10, 1), (256, 8, 0), (256, 8, -1), (128, 7, -1), (128, 7, 0),
                                      (64, 6, 0), (64, 6, -1), (32, 5, 0), (32, 5, -1), (512, 9, 0), (512, 9, -1), (512, 9, 1),
                                      (16, 4, -1), (16, 4, 1), (8, 3, -1), (8, 3, 1)])
def test_two_phase_abi_extreme_tables_vs_fused_and_oracle(S, q, mode):
    """Two-phase coder through the C ABI against the fused kernels and the oracle (fed our exact pmfs), on hostile rows:
    sigma at the x-level minimum (2/255/8) so that almost every bin is a saturated tail (P = 1, huge remnant), means far
    outside the bin range, symbols in the dead tails, plus ordinary rows.  mode 0 = generic kernels (k_rows/k_pop_coarse),
    -1 = classify the rows (uniform grids here -> the affine-row kernels k_rows6/k_pop6), 1 = affine kernels forced.
    S = 8 and 16 exist for the affine kernels only (the generic and fused ones own S/32 bins per lane): oracle alone."""
    rs = np.random.RandomState(S)
    B, L = 9, 96
    lo, hi = -6 - rs.uniform(0, 1, L), 6 + rs.uniform(0, 1, L)
    ends = np.linspace(lo, hi, S + 1, axis=1)[:, 1:-1].copy()
    mu = rs.normal(0, 2, (B, L)).astype(np.float32)
    sc = rs.uniform(0.1, 1.0, (B, L)).astype(np.float32)
    sc[:, 0::4] = np.float32((2. / 255.) / 8.)                 # needle-sharp rows
    mu[:, 1::8] = rs.choice([-25.0, 25.0, -7.5, 7.5], size=mu[:, 1::8].shape).astype(np.float32)    # mass outside the bins
    states = initial_states(B, seed=500, n=3000, step=1)
    tabs = oracle_tables(ends, mu, sc, S, q)
    sym = rs.randint(0, S, size=(B, L)).astype(np.int16)
    sym[:, :6] = [0, S - 1, 1, S - 2, S // 2, 0]
    res = run_2p(ends, mu, sc, S, q, states, sym, mode, cap=1 << 14)
    if S >= 32:
        fused = run_fused(ends, mu, sc, S, q, states, sym, cap=1 << 14)
        assert res[0] == fused[0] and np.array_equal(res[1], fused[1]) and res[2] == fused[2]
    check_vs_oracle(res, tabs, states, sym, range(B))


@pytest.mark.parametrize("mode", [0, -1, 1])
@pytest.mark.parametrize("bits,q", [(32, 10), (31, 31), (10, 12)])
def test_two_phase_abi_refuses_bits_out_of_range(bits, q, mode):
    """The two-phase coder codes 1 <= bits <= 31 and 0 <= quantbits < bits, like the fused one: anything else is
    BSW_E_INVALID before any coder kernel runs, for every kernel family, and the streams are left as they were."""
    B, L, S = 3, 40, 1024
    rs = np.random.RandomState(7)
    ends = np.linspace(-6, 6, S + 1)[1:-1]
    e_pad = torch.from_numpy(pad_big(np.tile(ends, (L, 1)))).to(dev)
    dmu = torch.from_numpy(rs.normal(0, 1, (B, L)).astype(np.float32)).to(dev)
    dsc = torch.from_numpy(rs.uniform(0.1, 1.0, (B, L)).astype(np.float32)).to(dev)
    sym = torch.from_numpy(rs.randint(0, S, size=(B, L)).astype(np.int16)).to(dev)
    nbytes = int(lib().bsw_logistic_scratch_bytes(B, L, S, 0))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    states = initial_states(B, seed=40, n=500, step=1)
    ss = StreamSet(B, 1 << 12)
    ss.import_lists(states)
    with coder_paths(rows_mode=mode):
        for fn, s_ in ((lib().bsw_logistic_push_2p, sym), (lib().bsw_logistic_pop_2p, sym.clone())):
            rc = fn(ss.handle, 0, B, dmu.data_ptr(), L, dsc.data_ptr(), L, e_pad.data_ptr(), S, s_.data_ptr(), L, S, bits, q,
                    scratch.data_ptr(), nbytes, cuda_stream_ptr())
            assert rc == 4, (fn, rc)
            assert b"out of range" in lib().bsw_last_error()
        torch.cuda.synchronize()
    assert ss.export_lists() == states
    assert not ss.sizes()[2].any()


def test_screening_cdf_error_is_far_inside_the_window():
    """k_rows trusts bsw_cdf_apx only when the scaled pmf is >= 64 units (2^-51 each) away from a truncation boundary;
    the pmf error is at most twice the cdf error, so the cdf error must stay below 32 units.  Measured worst case over
    2^27 arguments (bulk, steep part, far tails, sigma down to the x-level minimum) has to be below 8."""
    worst = ctypes.c_double(0)
    check(lib().bsw_selftest_cdf_apx(1 << 27, 777, ctypes.byref(worst)))
    print("worst |apx - exact| =", worst.value, "units of 2^-51")
    assert worst.value < 8.0


def test_affine_rows_full_size_level_every_bin_verified_against_the_exact_function():
    """VERDICT r1 weak #3: the screened table kernels are sound only if every integer they emit is the exact function's.
    A full-size latent level (2048 rows x 1024 bins, q = 10, sigma down to the 0.1 floor) is run through k_rows6 in
    verify mode, which evaluates the exact function (bsw_cdf_fast on the real endpoints) for EVERY bin next to the
    screened value: 0 disagreements, the worst screening error of a trusted bin below a quarter of its window, and the
    streams equal what the generic kernels leave."""
    L, S, q, B = 2048, 1024, 10, 16
    ends, mu, sc = level_case(L, S, q, B, seed=3)
    sc[:, ::7] = np.float32(0.1)
    mu[:, ::11] *= 3
    rs = np.random.RandomState(5)
    sym = rs.randint(0, S, size=(B, L)).astype(np.int16)
    states = initial_states(B, seed=700, n=6000, step=1)
    stats = np.zeros(4, dtype=np.uint64)
    with coder_paths(verify=1):
        got = run_2p(ends, mu, sc, S, q, states, sym, mode=-1, cap=1 << 14)
        check(lib().bsw_rows6_verify_read(stats.ctypes.data))
    mism, worst, checked, exact_path = (int(v) for v in stats)
    print(f"verify: {checked} bins evaluated of {2 * B * L * S}, {exact_path} took the exact path, worst trusted error "
          f"{worst / 10:.1f} % of the window, {mism} mismatches")
    assert checked > 0.25 * 2 * B * L * S and mism == 0
    assert worst <= 250, worst                            # a trusted bin's error must stay below a quarter of its window
    ref = run_2p(ends, mu, sc, S, q, states, sym, mode=0, cap=1 << 14)
    assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and got[2] == ref[2]


def test_affine_kernels_forced_on_non_uniform_rows_fall_back_to_the_exact_function():
    """mode 1 pushes the equal-mass top-level rows (not a uniform grid) through k_rows6/k_pop6: the plan refuses to
    vouch for them (mask = 0) and every bin takes the exact path -- same streams as the generic kernels."""
    L, S, q, B = 96, 1024, 10, 5
    ends, mu, sc = level_case(L, S, q, B, seed=9, affine=False)
    sym = np.random.RandomState(1).randint(0, S, size=(B, L)).astype(np.int16)
    states = initial_states(B, seed=800, n=3000, step=1)
    a = run_2p(ends, mu, sc, S, q, states, sym, mode=1, cap=1 << 14)
    b = run_2p(ends, mu, sc, S, q, states, sym, mode=0, cap=1 << 14)
    c = run_2p(ends, mu, sc, S, q, states, sym, mode=-1, cap=1 << 14)       # classification -> generic
    assert a[0] == b[0] == c[0] and np.array_equal(a[1], b[1]) and a[2] == b[2] == c[2]


@pytest.mark.parametrize("L,S,q", [(2048, 1024, 10), (3072, 256, 8), (93, 64, 6), (300, 512, 9), (93, 32, 5), (93, 16, 4),
                                   (93, 8, 3)])
def test_affine_rows_mapping_does_not_change_the_integers(L, S, q):
    """k_rows6 deals a warp to 32/LPR rows (LPR lanes per row, 32/LPR chunks per lane one after the other).  A chunk's
    arithmetic does not depend on the mapping, so LPR = 2, 4, 8 and 32 (the one-row-per-warp kernel of the first version)
    must leave identical streams and symbols -- including a row count that is not a multiple of the rows per warp, dead
    tails (needle-sharp rows) and symbols in them.  The reference is the generic kernels' run; at S = 8 and 16, which only
    the affine kernels code, it is the oracle coder on our exported pmfs."""
    B = 5
    ends, mu, sc = level_case(L, S, q, B, seed=17)
    sc[:, ::5] = np.float32((2. / 255.) / 8.)
    mu[:, 1::9] *= 4
    rs = np.random.RandomState(23)
    sym = rs.randint(0, S, size=(B, L)).astype(np.int16)
    sym[:, :4] = [0, S - 1, 1, S // 2]
    states = initial_states(B, seed=900, n=7000, step=1)
    res = {}
    for lpr in (32, 8, 4, 2):
        with coder_paths(lanes_per_row=lpr):
            res[lpr] = run_2p(ends, mu, sc, S, q, states, sym, mode=1, cap=1 << 14)
    if S >= 32:
        ref = run_2p(ends, mu, sc, S, q, states, sym, mode=0, cap=1 << 14)
    else:
        ref = res[32]
        check_vs_oracle(ref, oracle_tables(ends, mu, sc, S, q), states, sym, range(B))
    for lpr, got in res.items():
        assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and got[2] == ref[2], f"lanes per row = {lpr}"
