"""quantbits 11 and 12 on the GPU: latent supports of 2048 and 4096 bins through every coder kernel family, the codec, the
containers and discretize(), bit-identical to the oracle (ANS.__init__ + the reference coder) on our own pmfs."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from edge_oracle import EdgeOracle                                     # noqa: E402
from oracle import oracle as O                                         # noqa: E402
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200.ans import ANS                                       # noqa: E402
from bitswap_b200.config import preset, with_                          # noqa: E402
from bitswap_b200.model import Model                                   # noqa: E402
from bitswap_b200.codec import BitSwapCodec, Bins, PipelinedCodec, BITSWAP, BBANS   # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402
from bitswap_b200._lib import lib, check, cuda_stream_ptr, BswError   # noqa: E402
from test_quantbits_cpu import KAT, kat_inputs                         # noqa: E402

dev = "cuda"
WIDE = [(2048, 11), (4096, 12)]


def test_kat_q12_dropin_ans():
    pm, sym, w, head = kat_inputs()
    st0 = [int(v) for v in w] + [head]
    a = ANS(torch.from_numpy(pm).to(dev), 31, 12)
    assert [int(v) for v in a.pmfs[0, :6]] == KAT["P_row0_head"]
    pushed = a.encode(st0.copy(), torch.from_numpy(sym).to(dev))
    assert (len(pushed), hex(pushed[-1])) == (KAT["push_len"], KAT["push_head"])
    assert O.CState.from_list(pushed).digest() == KAT["push_sha"]
    popped, psym = a.decode(st0.copy())
    assert (len(popped), hex(popped[-1])) == (KAT["pop_len"], KAT["pop_head"])
    assert O.CState.from_list(popped).digest() == KAT["pop_sha"]
    assert [int(v) for v in psym[:6].cpu()] == KAT["pop_syms_head"]
    back, rsym = a.decode(pushed.copy())
    assert back == st0 and np.array_equal(rsym.cpu().numpy(), sym)
    assert a.encode(popped.copy(), psym) == st0


def _pad_big(ends):
    L, Sm1 = ends.shape
    out = np.full((L, Sm1 + 1), 1e300)
    out[:, :Sm1] = ends
    return out


def _states(B, seed, n=3000):
    out = []
    for b in range(B):
        w, head = synthetic.initial_words(n + 7 * b, seed=seed + b)
        out.append([int(v) for v in w] + [head])
    return out


def _rows(L, S, q, B, seed, affine=True):
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


def _run_2p(ends, mu, sc, S, q, states, sym, mode):
    B, L = mu.shape
    check(lib().bsw_set_rows_mode(mode))
    try:
        e_pad = torch.from_numpy(_pad_big(ends)).to(dev)
        dmu, dsc, dsym = torch.from_numpy(mu).to(dev), torch.from_numpy(sc).to(dev), torch.from_numpy(sym).to(dev)
        nbytes = int(lib().bsw_logistic_scratch_bytes(B, L, S, 0))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        ss = StreamSet(B, 1 << 15)
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
    finally:
        check(lib().bsw_set_rows_mode(-1))


def _oracle_tables(ends, mu, sc, S, q):
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


def _check_vs_oracle(res, tabs, states, sym, check_streams):
    after_pop, popped, after_push = res
    for b in check_streams:
        a = O.AnsC(tables=tabs[b])
        st, s_ = a.decode(O.CState.from_list(states[b]))
        assert np.array_equal(popped[b], s_), f"stream {b}: popped symbols differ"
        assert after_pop[b] == st.to_list(), f"stream {b}: state after pop differs"
        assert after_push[b] == a.encode(st, sym[b].astype(np.int64)).to_list(), f"stream {b}: state after push differs"


@pytest.mark.parametrize("S,q", WIDE)
@pytest.mark.parametrize("family", ["generic", "affine", "forced_affine"])
def test_two_phase_wide_support_vs_oracle(S, q, family):
    """pop then push of one level through bsw_logistic_pop_2p / push_2p, against our exported pmfs -> oracle ANS.__init__ ->
    oracle coder.  generic = k_rows_wide / k_pop_coarse_wide, affine = k_rows6 / k_pop6 on uniform grids, forced_affine =
    the affine kernels on the equal-mass top-level rows (every bin takes the exact path).  B = 64 streams, L = 99 rows (not
    a multiple of the 8 rows per warp); ordinary, needle-sharp, all-bins-live and off-grid rows."""
    B, L = 64, 99
    ends, mu, sc, sym = _rows(L, S, q, B, seed=S + len(family), affine=family != "forced_affine")
    mode = {"generic": 0, "affine": -1, "forced_affine": 1}[family]
    states = _states(B, seed=300)
    res = _run_2p(ends, mu, sc, S, q, states, sym, mode)
    tabs = _oracle_tables(ends, mu, sc, S, q)
    _check_vs_oracle(res, tabs, states, sym, range(B))
    if family == "affine":
        gen = _run_2p(ends, mu, sc, S, q, states, sym, 0)
        assert gen[0] == res[0] and np.array_equal(gen[1], res[1]) and gen[2] == res[2]


def test_affine_rows_q12_full_size_level_verified_against_the_exact_function():
    """A full-size cifar level at quantbits 12 (2048 rows x 4096 bins, sigma down to 0.1) through k_rows6 in verify mode: every
    bin is also evaluated with the exact function.  0 disagreements and the worst trusted error under a quarter of the
    window (the bar of the q = 10 test), with the chains re-anchored every 256 bins."""
    L, S, q, B = 2048, 4096, 12, 8
    rs = np.random.RandomState(3)
    lo, hi = -6 - rs.uniform(0, 1, L), 6 + rs.uniform(0, 1, L)
    ends = np.linspace(lo, hi, S + 1, axis=1)[:, 1:-1].copy()
    mu = rs.normal(0, 1.5, (B, L)).astype(np.float32)
    sc = rs.uniform(0.1, 1.0, (B, L)).astype(np.float32)
    sc[:, ::7] = np.float32(0.1)
    sc[:, 3::7] = np.float32(4.0)                          # every bin live: m = 128, four anchors per lane
    mu[:, ::11] *= 3
    sym = rs.randint(0, S, size=(B, L)).astype(np.int16)
    states = _states(B, seed=700, n=6000)
    check(lib().bsw_rows6_set_verify(1))
    stats = np.zeros(4, dtype=np.uint64)
    try:
        got = _run_2p(ends, mu, sc, S, q, states, sym, mode=-1)
        check(lib().bsw_rows6_verify_read(stats.ctypes.data))
    finally:
        check(lib().bsw_rows6_set_verify(0))
    mism, worst, checked, exact_path = (int(v) for v in stats)
    print(f"verify q=12: {checked} bins evaluated of {2 * B * L * S}, {exact_path} exact path, worst trusted error "
          f"{worst / 10:.1f} % of the window, {mism} mismatches")
    assert checked > 0.2 * 2 * B * L * S and mism == 0
    assert worst <= 250, worst
    ref = _run_2p(ends, mu, sc, S, q, states, sym, mode=0)
    assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and got[2] == ref[2]


def test_affine_lanes_per_row_do_not_change_the_streams_at_4096():
    S, q, B, L = 4096, 12, 5, 93
    ends, mu, sc, sym = _rows(L, S, q, B, seed=17)
    states = _states(B, seed=900, n=7000)
    res = {}
    try:
        for lpr in (32, 8, 4, 2):
            check(lib().bsw_rows6_set_lanes_per_row(lpr))
            res[lpr] = _run_2p(ends, mu, sc, S, q, states, sym, mode=1)
    finally:
        check(lib().bsw_rows6_set_lanes_per_row(0))
    ref = _run_2p(ends, mu, sc, S, q, states, sym, mode=0)
    for lpr, got in res.items():
        assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and got[2] == ref[2], f"lanes per row = {lpr}"


def _setup(name, q, B, tc=False):
    cfg = with_(preset(name), quantbits=q)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    m = Model.from_config(cfg, max_batch=B, use_tensor_cores=tc).load_state_dict(sd)
    m.compress()
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    bins = Bins(cfg, zend, zcen)
    return cfg, m, sd, zend, zcen, bins, BitSwapCodec(cfg, m, bins, B)


def _oracle_with(cfg, m, sd, zend, zcen, cls=O.BitSwapOracle):
    orc = cls(cfg, O.ModelOracle(cfg, sd), zend, zcen, coder="c", pmf="cuda")

    def _net(kind, level, given):
        f = m.infer(level) if kind == "infer" else m.generate(level)
        mu, sc = f(given.cuda())
        return mu.cpu(), sc.cpu()
    orc._net = _net
    return orc


@pytest.mark.parametrize("q", [11, 12])
@pytest.mark.parametrize("name,scheme", [("tiny", BITSWAP), ("tiny3", BITSWAP), ("tiny", BBANS), ("tiny3", BBANS)])
def test_p4_wide_support_vs_oracle_with_injected_nets(name, scheme, q):
    B, nimg = 4, 2
    cfg, m, sd, zend, zcen, bins, codec = _setup(name, q, B)
    assert cfg.zsupport == 1 << q
    ss = StreamSet(B, 1 << 15)
    imgs = synthetic.synthetic_images(cfg, B * nimg, seed=11).reshape(nimg, B, *cfg.xs)
    states = _states(B, seed=100, n=4000)
    ss.import_lists(states)
    for xi in range(nimg):
        codec.encode(ss, torch.from_numpy(imgs[xi]).cuda(), scheme=scheme)
    ss.raise_on_error()
    got = ss.export_lists()
    for b in range(B):
        orc = _oracle_with(cfg, m, sd, zend, zcen)
        st = O.CState.from_list(states[b])
        for xi in range(nimg):
            st = (orc.encode_image if scheme == BITSWAP else orc.encode_image_bbans)(st, imgs[xi, b])
        assert got[b] == st.to_list(), f"stream {b} differs from the oracle"
    for xi in reversed(range(nimg)):
        out = codec.decode(ss, B, scheme=scheme)
        assert np.array_equal(out.cpu().numpy(), imgs[xi])
    ss.raise_on_error()
    assert ss.export_lists() == states


def test_cifar8_q12_tensor_cores_full_width():
    """cifar8 at quantbits 12 on the tensor-core nets, B = 256 over 4 lanes: sampled streams equal the oracle driven with
    the same nets, and the batch decodes back exactly."""
    B = 256
    cfg = with_(preset("cifar8"), quantbits=12)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    pc = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), B, lanes=4, use_tensor_cores=True)
    ss = StreamSet(B, 1 << 14)
    imgs = synthetic.synthetic_images(cfg, B, seed=21)
    states = _states(B, seed=1000, n=5000)
    ss.import_lists(states)
    pc.encode(ss, torch.from_numpy(imgs).cuda())
    torch.cuda.synchronize()
    ss.raise_on_error()
    got = ss.export_lists()
    for b in (0, 77, 255):
        lane = b // pc.per
        m = pc.models[lane]
        orc = _oracle_with(cfg, m, sd, zend, zcen)
        st = orc.encode_image(O.CState.from_list(states[b]), imgs[b])
        assert got[b] == st.to_list(), f"stream {b} differs from the oracle"
    out = pc.decode(ss, B)
    torch.cuda.synchronize()
    ss.raise_on_error()
    assert np.array_equal(out.cpu().numpy(), imgs) and ss.export_lists() == states


def test_overlap_mode_equals_program_order_q12():
    B = 6
    cfg = with_(preset("tiny3"), quantbits=12)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    pc = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), B, lanes=2, use_tensor_cores=False)
    ss = StreamSet(B, 1 << 15)
    imgs = synthetic.synthetic_images(cfg, 3 * B, seed=43).reshape(3, B, *cfg.xs)
    states = _states(B, seed=400, n=5000)
    res = []
    for mode in (0, 1):
        pc.set_dual_stream(mode)
        ss.import_lists(states)
        for xi in range(3):
            pc.encode(ss, torch.from_numpy(imgs[xi]).cuda(), scheme=BBANS)
        torch.cuda.synchronize()
        ss.raise_on_error()
        res.append(ss.export_lists())
    assert res[0] == res[1]
    for xi in (2, 1, 0):
        out = pc.decode(ss, B, scheme=BBANS)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), imgs[xi])
    assert ss.export_lists() == states


def _demo_oracle_container(orc, img, n_init):
    from bitswap_b200.container import extract_edge_blocks
    blocks, extents, h, w = extract_edge_blocks(img)
    wds, head = synthetic.initial_words(n_init, seed=100)
    st = O.CState(wds, head)
    low = st.n
    pops = []
    orc.trace = pops
    for b, e in zip(blocks, extents):
        st = orc.encode_image(st, b.transpose(2, 0, 1), extent=(int(e[0]), int(e[1])))
    orc.trace = None
    low = min([ln - 1 for tag, ln, _ in pops if tag.startswith("pop")] + [low])
    return np.concatenate([st.words[low:st.n], np.array([st.head & 0xffffffff, st.head >> 32, len(blocks), h, w],
                                                         dtype=np.uint64)]).astype(np.uint32)


def test_edge_coded_containers_q12():
    from bitswap_b200.container import compress_images, decompress_images
    sizes = [(40, 70), (20, 20), (33, 1)]
    rs = np.random.RandomState(5)
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    cfg, m, sd, zend, zcen, bins, codec = _setup("tiny3", 12, len(images))
    for edges in ("code", "crop"):
        conts = compress_images(codec, images[:1] if edges == "crop" else images, excess_state_len=3000, edges=edges)
        back = decompress_images(codec, conts)
        if edges == "crop":
            assert np.array_equal(back[0], images[0][:32, :64])
    conts = compress_images(codec, images, excess_state_len=3000, edges="code")
    back = decompress_images(codec, conts)
    for img, rec in zip(images, back):
        assert rec.shape == img.shape and np.array_equal(rec, img)
    orc = _oracle_with(cfg, m, sd, zend, zcen, cls=EdgeOracle)
    for img, cont in zip(images, conts):
        assert np.array_equal(cont, _demo_oracle_container(orc, img, 3000)), img.shape


def test_gpu_discretize_q12_then_codec_roundtrip():
    from bitswap_b200.discretization import discretize
    cfg = with_(preset("tiny3"), quantbits=12)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    m = Model.from_config(cfg, max_batch=128).load_state_dict(sd)
    m.compress()
    imgs = torch.from_numpy(synthetic.synthetic_images(cfg, 512, seed=17, kind="smooth"))
    zend, zcen = discretize(cfg.nz, 12, torch.float64, "cpu", m, "synthetic", images=imgs, ppb=2)
    assert zend.shape == (cfg.nz, cfg.zdim, 4095) and zcen.shape == (cfg.nz, cfg.zdim, 4096)
    assert torch.all(zend[:, :, 1:] > zend[:, :, :-1])
    bins = Bins(cfg, zend, zcen)
    assert all(bins.level_is_uniform(i) for i in range(cfg.nz - 1)) and not bins.level_is_uniform(cfg.nz - 1)
    B = 4
    codec = BitSwapCodec(cfg, m, bins, B)
    ss = StreamSet(B, 1 << 14)
    wds, head = synthetic.initial_words(4000, seed=100)
    ss.fill(wds, head)
    init = ss.export_lists()
    x = imgs[:B].cuda()
    codec.encode(ss, x)
    out = codec.decode(ss, B)
    ss.raise_on_error()
    assert torch.equal(out, x) and ss.export_lists() == init


def test_fused_coder_is_refused_above_1024_bins():
    cfg, m, sd, zend, zcen, bins, codec = _setup("tiny", 12, 2)
    with pytest.raises(ValueError, match="1024"):
        codec.set_two_phase(False)
    rc = lib().bsw_codec_set_two_phase(codec._h, 0)
    assert rc == 4 and b"1024" in lib().bsw_last_error()
    pc = PipelinedCodec(cfg, sd, bins, 2, lanes=1, use_tensor_cores=False)
    with pytest.raises(ValueError, match="1024"):
        pc.set_two_phase(False)
    codec.set_two_phase(True)                                  # the two-phase coder stays available
    # the fused entry points themselves refuse S > 1024
    ss = StreamSet(1, 1 << 13)
    ss.import_lists(_states(1, seed=5))
    e = torch.full((4, 4096), 1e300, dtype=torch.float64, device=dev)
    mu = torch.zeros((1, 4), dtype=torch.float32, device=dev)
    sc = torch.ones((1, 4), dtype=torch.float32, device=dev)
    out = torch.zeros((1, 4), dtype=torch.int16, device=dev)
    rc = lib().bsw_logistic_pop(ss.handle, 0, 1, mu.data_ptr(), 4, sc.data_ptr(), 4, e.data_ptr(), 4096, out.data_ptr(), 4, 4096,
                                31, 12, cuda_stream_ptr())
    assert rc == 4 and b"1024" in lib().bsw_last_error()


def test_q13_bins_are_refused():
    cfg = with_(preset("tiny"), quantbits=13)
    with pytest.raises(ValueError):
        Bins(cfg, np.zeros((2, 256, 8191)), np.zeros((2, 256, 8192)))
    cfg12 = with_(preset("tiny"), quantbits=12)
    zend, zcen = synthetic.synthetic_bins(cfg12, seed=0)
    import ctypes
    h = ctypes.c_void_p()
    ze = np.ascontiguousarray(zend.numpy(), dtype=np.float64)
    zc = np.ascontiguousarray(zcen.numpy(), dtype=np.float64)
    assert lib().bsw_bins_create(ctypes.byref(h), cfg12.nz, cfg12.zdim, 13, cfg12.xdim, ze.ctypes.data, zc.ctypes.data) == 4
    with pytest.raises(BswError):
        check(lib().bsw_bins_create(ctypes.byref(h), cfg12.nz, cfg12.zdim, 13, cfg12.xdim, ze.ctypes.data, zc.ctypes.data))
