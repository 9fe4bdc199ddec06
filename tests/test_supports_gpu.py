"""Latent supports below the default precision on the GPU: the affine-row kernels at supports that are not powers of two
and below 32 bins, their verify mode at every power of two from 8 to 1024, the refusals of each kernel family, the codec
at quantbits 5, 8 and 9 on the fused coder and on PipelinedCodec, the refusal of quantbits 1-4, and the discretisation
kernels (sampling, extrema, uniform fit) bit for bit against numpy.  The coder oracle is the one of the P2a and q12
tests: our exported float64 pmfs (bsw_logistic_pmfs) -> ANS.__init__ (O.tables_c) -> the reference coder (O.AnsC)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from coder_harness import (check_vs_oracle, coder_paths, dev, hostile_rows, initial_states, oracle_tables, pad_big,   # noqa: E402
                           run_2p)
from codec_harness import gpu_oracle, setup                            # noqa: E402
from oracle import oracle as O                                         # noqa: E402
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200.config import preset, with_                          # noqa: E402
from bitswap_b200.codec import Bins, PipelinedCodec, BITSWAP, BBANS    # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402
from bitswap_b200._lib import lib, check, cuda_stream_ptr              # noqa: E402


def _q_of(S):
    """quantbits handed to the coder with a support S that is not a power of two: the smallest q with 2^q >= S."""
    return (S - 1).bit_length()


# ---- affine-row kernels at supports the generic family does not take ---------------------------------------------------
@pytest.mark.parametrize("S", [8, 12, 20, 100, 1020])
@pytest.mark.parametrize("mode", [-1, 1])
def test_affine_supports_not_powers_of_two_vs_oracle(S, mode):
    """bsw_rows6_launch takes any multiple of 4 in [8, 1024].  Pop then push of one level (B = 16 streams, L = 77 rows) on the
    hostile rows of _rows -- needle-sharp rows, rows where every bin is live, mass beyond the grid, symbols in the edge
    bins -- must leave every stream and symbol bit-identical to the oracle.  mode -1 classifies the rows (uniform grids:
    the affine kernels), mode 1 forces the affine kernels; the generic kernels would refuse these supports."""
    B, L, q = 16, 77, _q_of(S)
    ends, mu, sc, sym = hostile_rows(L, S, q, B, seed=1000 + S)
    states = initial_states(B, seed=40 + S)
    res = run_2p(ends, mu, sc, S, q, states, sym, mode)
    check_vs_oracle(res, oracle_tables(ends, mu, sc, S, q), states, sym, range(B))


@pytest.mark.parametrize("S", [8, 16, 32, 64, 128, 256, 512, 1024])
def test_affine_verify_mode_at_every_power_of_two(S):
    """A full-size level (2048 rows, sigma down to 0.1, every-bin-live and off-grid rows) through k_rows6 in verify mode,
    which evaluates the exact function next to every screened bin: 0 disagreements and the worst trusted error under a
    quarter of the window.  The streams equal the generic kernels' (S >= 32) or the oracle's (S < 32)."""
    L, q, B = 2048, S.bit_length() - 1, 4
    rs = np.random.RandomState(S)
    lo, hi = -6 - rs.uniform(0, 1, L), 6 + rs.uniform(0, 1, L)
    ends = np.linspace(lo, hi, S + 1, axis=1)[:, 1:-1].copy()
    mu = rs.normal(0, 1.5, (B, L)).astype(np.float32)
    sc = rs.uniform(0.1, 1.0, (B, L)).astype(np.float32)
    sc[:, ::7] = np.float32(0.1)
    sc[:, 3::7] = np.float32(4.0)
    mu[:, ::11] *= 3
    mu[:, 5::13] = np.float32(20.0)
    sym = rs.randint(0, S, size=(B, L)).astype(np.int16)
    states = initial_states(B, seed=700 + S, n=6000)
    stats = np.zeros(4, dtype=np.uint64)
    with coder_paths(verify=1):
        got = run_2p(ends, mu, sc, S, q, states, sym, mode=-1)
        check(lib().bsw_rows6_verify_read(stats.ctypes.data))
    mism, worst, checked, exact_path = (int(v) for v in stats)
    print(f"verify S={S}: {checked} bins evaluated of {2 * B * L * S}, {exact_path} exact path, worst trusted error "
          f"{worst / 10:.1f} % of the window, {mism} mismatches")
    assert checked > 0 and mism == 0
    assert worst <= 250, worst
    if S >= 32:
        ref = run_2p(ends, mu, sc, S, q, states, sym, mode=0)
        assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and got[2] == ref[2]
    else:
        check_vs_oracle(got, oracle_tables(ends, mu, sc, S, q), states, sym, range(B))


# ---- refusals ------------------------------------------------------------------------------------------------------------
def _abi_2p_rc(S, q, mode, B=2, L=4):
    ends = np.linspace(-6.0, 6.0, S + 1)[None, 1:-1].repeat(L, 0)
    e_pad = torch.from_numpy(pad_big(ends)).to(dev)
    mu = torch.zeros((B, L), dtype=torch.float32, device=dev)
    sc = torch.ones((B, L), dtype=torch.float32, device=dev)
    sym = torch.zeros((B, L), dtype=torch.int16, device=dev)
    nbytes = int(lib().bsw_logistic_scratch_bytes(B, L, S, 0))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    ss = StreamSet(B, 4096)
    ss.import_lists(initial_states(B, seed=3))
    with coder_paths(rows_mode=mode):
        rcs = [fn(ss.handle, 0, B, mu.data_ptr(), L, sc.data_ptr(), L, e_pad.data_ptr(), S, sym.data_ptr(), L, S, 31, q,
                  scratch.data_ptr(), nbytes, cuda_stream_ptr()) for fn in (lib().bsw_logistic_pop_2p, lib().bsw_logistic_push_2p)]
    torch.cuda.synchronize()
    assert ss.export_lists() == initial_states(B, seed=3)                 # a refused call leaves the streams alone
    return rcs


def _fused_rc(S, q, B=2, L=4):
    e_pad = torch.full((L, S), 1e300, dtype=torch.float64, device=dev)
    mu = torch.zeros((B, L), dtype=torch.float32, device=dev)
    sc = torch.ones((B, L), dtype=torch.float32, device=dev)
    sym = torch.zeros((B, L), dtype=torch.int16, device=dev)
    ss = StreamSet(B, 4096)
    ss.import_lists(initial_states(B, seed=3))
    return [fn(ss.handle, 0, B, mu.data_ptr(), L, sc.data_ptr(), L, e_pad.data_ptr(), S, sym.data_ptr(), L, S, 31, q,
               cuda_stream_ptr()) for fn in (lib().bsw_logistic_pop, lib().bsw_logistic_push)]


@pytest.mark.parametrize("S,q", [(16, 4), (8, 3), (4, 2), (2, 1)])
def test_generic_and_fused_kernels_refuse_supports_below_32(S, q):
    """Every generic and fused kernel owns S/32 bins per lane: the generic two-phase ABI (mode 0) and the fused ABI return
    BSW_E_INVALID below 32 bins, naming the supports they take."""
    assert _abi_2p_rc(S, q, mode=0) == [4, 4]
    assert b"32,64" in lib().bsw_last_error()
    assert _fused_rc(S, q) == [4, 4]
    assert b"32,64" in lib().bsw_last_error()


@pytest.mark.parametrize("S", [10, 14, 30, 1022, 4])
def test_affine_kernels_refuse_supports_not_a_multiple_of_4(S):
    """The affine ABI (mode 1) codes 4-bin groups: a support that is not a multiple of 4 (or below 8) is BSW_E_INVALID."""
    assert _abi_2p_rc(S, _q_of(S), mode=1) == [4, 4]
    msg = lib().bsw_last_error()
    assert b"multiple of 4" in msg or b"32,64" in msg, msg


def test_quantbits_below_5_are_refused_before_device_work():
    """A quantbits 4 model builds equal-mass top-level bins of 16 entries, which no kernel that codes the top level (generic
    or fused) takes.  Bins refuses it with ValueError before anything reaches the device, rather than letting the
    codec fail at its first encode."""
    cfg = with_(preset("tiny"), quantbits=4)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    assert zend.shape == (cfg.nz, cfg.zdim, 15)
    with pytest.raises(ValueError, match=r"\[5, 12\]"):
        Bins(cfg, zend, zcen)
    h = ctypes.c_void_p()
    ze = np.ascontiguousarray(zend.numpy(), dtype=np.float64)
    zc = np.ascontiguousarray(zcen.numpy(), dtype=np.float64)
    assert lib().bsw_bins_create(ctypes.byref(h), cfg.nz, cfg.zdim, 4, cfg.xdim, ze.ctypes.data, zc.ctypes.data) == 4
    assert b"[5, 12]" in lib().bsw_last_error() and not h.value


# ---- the codec at quantbits 5, 8 and 9 -------------------------------------------------------------------------------------
@pytest.mark.parametrize("q", [5, 8, 9])
@pytest.mark.parametrize("name,scheme", [("tiny3", BITSWAP), ("tiny", BBANS)])
def test_fused_coder_equals_two_phase_at_low_quantbits(name, scheme, q):
    """set_two_phase(False) codes every level with the fused one-warp-per-stream kernels (launch_fused<S/32>): the streams
    must be bit-identical to the two-phase coder's, and the fused decode must restore images and states."""
    B, nimg = 4, 2
    cfg, m, sd, zend, zcen, bins, codec = setup(name, B, q=q)
    imgs = synthetic.synthetic_images(cfg, B * nimg, seed=13).reshape(nimg, B, *cfg.xs)
    states = initial_states(B, seed=200, n=4000)
    res = {}
    for two_phase in (True, False):
        codec.set_two_phase(two_phase)
        ss = StreamSet(B, 1 << 15)
        ss.import_lists(states)
        for xi in range(nimg):
            codec.encode(ss, torch.from_numpy(imgs[xi]).cuda(), scheme=scheme)
        ss.raise_on_error()
        res[two_phase] = ss.export_lists()
    assert res[False] == res[True]
    for xi in reversed(range(nimg)):                              # the fused coder decodes what it encoded
        out = codec.decode(ss, B, scheme=scheme)
        assert np.array_equal(out.cpu().numpy(), imgs[xi])
    ss.raise_on_error()
    assert ss.export_lists() == states
    codec.set_two_phase(True)


def test_pipelined_codec_overlap_mode_q9_vs_oracle():
    """PipelinedCodec, 2 lanes in overlap mode, at quantbits 9 (512 bins: k_rows<16>, k_rows6 at S = 512, the prior pop
    k_pop_full<16>): every stream equals the oracle recursion driven with its lane's nets, equals program order, and decodes
    back exactly."""
    B = 6
    cfg = with_(preset("tiny3"), quantbits=9)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    pc = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), B, lanes=2, use_tensor_cores=False)
    ss = StreamSet(B, 1 << 15)
    imgs = synthetic.synthetic_images(cfg, 2 * B, seed=29).reshape(2, B, *cfg.xs)
    states = initial_states(B, seed=600, n=5000)
    res = []
    for mode in (1, 0):
        pc.set_dual_stream(mode)
        ss.import_lists(states)
        for xi in range(2):
            pc.encode(ss, torch.from_numpy(imgs[xi]).cuda())
        torch.cuda.synchronize()
        ss.raise_on_error()
        res.append(ss.export_lists())
    assert res[0] == res[1]
    for b in range(B):
        orc = gpu_oracle(cfg, pc.models[b // pc.per], sd, zend, zcen, cls=O.BitSwapOracle)
        st = O.CState.from_list(states[b])
        for xi in range(2):
            st = orc.encode_image(st, imgs[xi, b])
        assert res[0][b] == st.to_list(), f"stream {b} differs from the oracle"
    pc.set_dual_stream(1)
    for xi in (1, 0):
        out = pc.decode(ss, B)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), imgs[xi])
    ss.raise_on_error()
    assert ss.export_lists() == states


# ---- discretisation kernels, bit for bit ------------------------------------------------------------------------------------
def _ord2f(o):
    """Inverse of the kernels' order-preserving float -> uint32 map (the running extrema are integer atomics)."""
    o = np.asarray(o).view(np.uint32)
    u = np.where(o & 0x80000000, o & 0x7fffffff, ~o).astype(np.uint32)
    return u.view(np.float32)


def _extrema(mm, dim):
    h = mm.cpu().numpy()
    return _ord2f(h[:dim]), _ord2f(h[dim:])


def _check_fit(mm, dim, lo, hi):
    """bsw_discretize_edges at every quantbits 5-12 == np.linspace(lo, hi, 2^q + 1) per dimension (endpoints: the inner
    points; centres: discretize_kbins's (e[:-1] + e[1:]) / 2 of the whole edge vector), bit for bit."""
    for q in range(5, 13):
        n = 1 << q
        ze = torch.full((dim, n - 1), np.nan, dtype=torch.float64, device=dev)
        zc = torch.full((dim, n), np.nan, dtype=torch.float64, device=dev)
        check(lib().bsw_discretize_edges(mm.data_ptr(), dim, q, ze.data_ptr(), n - 1, zc.data_ptr(), n, cuda_stream_ptr()))
        torch.cuda.synchronize()
        ge, gc = ze.cpu().numpy(), zc.cpu().numpy()
        for d in range(dim):
            edges = np.linspace(float(lo[d]), float(hi[d]), n + 1)
            cen = (edges[:-1] + edges[1:]) / 2
            assert np.array_equal(ge[d].view(np.uint64), edges[1:-1].view(np.uint64)), (q, d, lo[d], hi[d])
            assert np.array_equal(gc[d].view(np.uint64), cen.view(np.uint64)), (q, d, lo[d], hi[d])


@pytest.mark.parametrize("rows,dim,stride", [(1000, 300, "dim"), (77, 130, 0)])
def test_discretize_sample_extrema_and_fit_are_bit_exact(rows, dim, stride):
    """k_sample_logistic, k_minmax_half and k_uniform_edges against numpy on the same uniforms.  Rows not a multiple of the
    64-row strip (one above 64, so several CTAs' atomics meet on one dimension), dim not a multiple of 128, scale row stride
    dim or 0, uniforms below the clamp bound and above 1 - bound.  eps = log(u) - log1p(-u) in float32 on CUDA, as the
    reference draws it; z = float64 mu + float64 sigma * eps cast straight to float16, as the reference's assignment does.
    Samples compare as uint16, extrema equal min / max, and the fit is checked at every quantbits 5-12."""
    rs = np.random.RandomState(rows + dim)
    bound = float(np.float32(1e-5))
    mu = rs.normal(0, 2, (rows, dim)).astype(np.float32)
    sc_rows = 1 if stride == 0 else rows
    sc = rs.uniform(0.05, 3.0, (sc_rows, dim)).astype(np.float32)
    u = rs.random_sample((rows, dim)).astype(np.float32)
    u[0, :5] = [0.0, 1e-7, 1e-6, 1.0 - 1e-7, np.float32(0.99999994)]
    u[rows - 1, -3:] = [0.0, np.float32(0.99999994), 5e-6]
    u[:, 7] = np.where(np.arange(rows) % 2, np.float32(0.99999994), np.float32(1e-8))      # a dimension of clamped draws
    du, dmu, dsc = (torch.from_numpy(a).to(dev) for a in (u, mu, sc))
    out = torch.zeros((rows, dim), dtype=torch.float16, device=dev)
    mm = torch.empty(2 * dim, dtype=torch.int32, device=dev)
    check(lib().bsw_discretize_reset(mm.data_ptr(), dim, cuda_stream_ptr()))
    check(lib().bsw_discretize_sample(dmu.data_ptr(), dsc.data_ptr(), 0 if stride == 0 else dim, du.data_ptr(), bound,
                                      out.data_ptr(), mm.data_ptr(), rows, dim, cuda_stream_ptr()))
    uc = torch.clamp(du, min=bound, max=1 - bound)
    eps = (torch.log(uc) - torch.log1p(-uc)).cpu().numpy()
    assert eps.dtype == np.float32 and np.isfinite(eps).all()
    z = mu.astype(np.float64) + np.broadcast_to(sc, (rows, dim)).astype(np.float64) * eps.astype(np.float64)
    want = z.astype(np.float16)
    got = out.cpu().numpy()
    bad = int((got.view(np.uint16) != want.view(np.uint16)).sum())
    assert bad == 0, f"{bad} of {rows * dim} float16 samples differ"
    lo, hi = _extrema(mm, dim)
    assert np.array_equal(lo, want.min(axis=0).astype(np.float32)) and np.array_equal(hi, want.max(axis=0).astype(np.float32))
    # a zero row folded in afterwards, as discretize() does when the batches do not fill the sample array
    zero = torch.zeros((1, dim), dtype=torch.float16, device=dev)
    check(lib().bsw_discretize_fold(zero.data_ptr(), mm.data_ptr(), 1, dim, cuda_stream_ptr()))
    lo, hi = _extrema(mm, dim)
    assert np.array_equal(lo, np.minimum(want.min(axis=0), 0).astype(np.float32))
    assert np.array_equal(hi, np.maximum(want.max(axis=0), 0).astype(np.float32))
    _check_fit(mm, dim, lo.astype(np.float64), hi.astype(np.float64))


def test_discretize_fold_and_fit_at_extreme_extrema():
    """Extrema folded in by bsw_discretize_fold from float16 samples (70 rows: two strips meet in the atomics): the largest
    finite span (-65504, 65504), the smallest (0, 2^-24, one subnormal step), a constant dimension, one-sided and ordinary
    ones.  The extrema equal min / max and the fit equals np.linspace at every quantbits 5-12."""
    rows, dim = 70, 9
    rs = np.random.RandomState(8)
    s = (rs.normal(0, 3, (rows, dim))).astype(np.float16)
    s[:, 0] = 0; s[3, 0] = -65504; s[66, 0] = 65504
    s[:, 1] = 0; s[69, 1] = np.float16(2.0 ** -24)
    s[:, 2] = np.float16(1.5)
    s[:, 3] = np.float16(-7.25); s[65, 3] = np.float16(-65504)
    s[:, 4] = np.abs(s[:, 4]) + np.float16(60000); s[10, 4] = np.float16(65504)
    s[:, 5] = np.float16(-2.0 ** -24); s[0, 5] = np.float16(-0.0)
    hs = torch.from_numpy(s).to(dev)
    mm = torch.empty(2 * dim, dtype=torch.int32, device=dev)
    check(lib().bsw_discretize_reset(mm.data_ptr(), dim, cuda_stream_ptr()))
    check(lib().bsw_discretize_fold(hs.data_ptr(), mm.data_ptr(), 64, dim, cuda_stream_ptr()))           # two calls, as
    check(lib().bsw_discretize_fold(hs[64:].contiguous().data_ptr(), mm.data_ptr(), rows - 64, dim, cuda_stream_ptr()))
    lo, hi = _extrema(mm, dim)
    assert np.array_equal(lo, s.min(axis=0).astype(np.float32)) and np.array_equal(hi, s.max(axis=0).astype(np.float32))
    assert (lo[0], hi[0], hi[1], lo[2], hi[2]) == (-65504, 65504, 2.0 ** -24, 1.5, 1.5)
    _check_fit(mm, dim, lo.astype(np.float64), hi.astype(np.float64))
