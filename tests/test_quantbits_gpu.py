"""quantbits 11 and 12 on the GPU: latent supports of 2048 and 4096 bins through every coder kernel family, the codec, the
containers and discretize(), bit-identical to the oracle (ANS.__init__ + the reference coder) on our own pmfs."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from coder_harness import (KAT, check_vs_oracle, coder_paths, dev, hostile_rows, initial_states, kat_inputs,   # noqa: E402
                           oracle_tables, run_2p)
from codec_harness import demo_oracle_container, gpu_oracle, setup   # noqa: E402
from oracle import oracle as O                                         # noqa: E402
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200.ans import ANS                                       # noqa: E402
from bitswap_b200.config import preset, with_                          # noqa: E402
from bitswap_b200.model import Model                                   # noqa: E402
from bitswap_b200.codec import BitSwapCodec, Bins, PipelinedCodec, BITSWAP, BBANS   # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402
from bitswap_b200._lib import lib, check, cuda_stream_ptr, BswError   # noqa: E402

WIDE = [(1 << q, q) for q in range(5, 13)]              # every support the codec codes: 32 ... 4096 bins


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


@pytest.mark.parametrize("S,q", WIDE)
@pytest.mark.parametrize("family", ["generic", "affine", "forced_affine"])
def test_two_phase_wide_support_vs_oracle(S, q, family):
    """pop then push of one level through bsw_logistic_pop_2p / push_2p, against our exported pmfs -> oracle ANS.__init__ ->
    oracle coder, at every power of two from 32 to 4096 bins.  generic = k_rows<S/32> / k_pop_coarse<S/32> (k_rows_wide<S/1024>
    above 1024), affine = k_rows6 / k_pop6 on uniform grids, forced_affine =
    the affine kernels on the equal-mass top-level rows (every bin takes the exact path).  B = 64 streams, L = 99 rows (not
    a multiple of the 8 rows per warp); ordinary, needle-sharp, all-bins-live and off-grid rows."""
    B, L = 64, 99
    ends, mu, sc, sym = hostile_rows(L, S, q, B, seed=S + len(family), affine=family != "forced_affine")
    mode = {"generic": 0, "affine": -1, "forced_affine": 1}[family]
    states = initial_states(B, seed=300)
    res = run_2p(ends, mu, sc, S, q, states, sym, mode)
    tabs = oracle_tables(ends, mu, sc, S, q)
    check_vs_oracle(res, tabs, states, sym, range(B))
    if family == "affine":
        gen = run_2p(ends, mu, sc, S, q, states, sym, 0)
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
    states = initial_states(B, seed=700, n=6000)
    stats = np.zeros(4, dtype=np.uint64)
    with coder_paths(verify=1):
        got = run_2p(ends, mu, sc, S, q, states, sym, mode=-1)
        check(lib().bsw_rows6_verify_read(stats.ctypes.data))
    mism, worst, checked, exact_path = (int(v) for v in stats)
    print(f"verify q=12: {checked} bins evaluated of {2 * B * L * S}, {exact_path} exact path, worst trusted error "
          f"{worst / 10:.1f} % of the window, {mism} mismatches")
    assert checked > 0.2 * 2 * B * L * S and mism == 0
    assert worst <= 250, worst
    ref = run_2p(ends, mu, sc, S, q, states, sym, mode=0)
    assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and got[2] == ref[2]


def test_affine_lanes_per_row_do_not_change_the_streams_at_4096():
    S, q, B, L = 4096, 12, 5, 93
    ends, mu, sc, sym = hostile_rows(L, S, q, B, seed=17)
    states = initial_states(B, seed=900, n=7000)
    res = {}
    for lpr in (32, 8, 4, 2):
        with coder_paths(lanes_per_row=lpr):
            res[lpr] = run_2p(ends, mu, sc, S, q, states, sym, mode=1)
    ref = run_2p(ends, mu, sc, S, q, states, sym, mode=0)
    for lpr, got in res.items():
        assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and got[2] == ref[2], f"lanes per row = {lpr}"


@pytest.mark.parametrize("q", [5, 8, 9, 11, 12])
@pytest.mark.parametrize("name,scheme", [("tiny", BITSWAP), ("tiny3", BITSWAP), ("tiny", BBANS), ("tiny3", BBANS)])
def test_p4_wide_support_vs_oracle_with_injected_nets(name, scheme, q):
    """The codec end to end at quantbits 5, 8, 9, 11 and 12 (q = 6, 7 and 10 are the presets' own): every stream equals the
    oracle recursion driven with the same nets, and decoding restores images and states.  The prior pop on the shared
    table (k_pop_full<S/32>, and the cdf-table pop at S = 32) runs only here and in the tests of test_supports_gpu.py."""
    B, nimg = 4, 2
    cfg, m, sd, zend, zcen, bins, codec = setup(name, B, q=q)
    assert cfg.zsupport == 1 << q
    ss = StreamSet(B, 1 << 15)
    imgs = synthetic.synthetic_images(cfg, B * nimg, seed=11).reshape(nimg, B, *cfg.xs)
    states = initial_states(B, seed=100, n=4000)
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
    states = initial_states(B, seed=1000, n=5000)
    ss.import_lists(states)
    pc.encode(ss, torch.from_numpy(imgs).cuda())
    torch.cuda.synchronize()
    ss.raise_on_error()
    got = ss.export_lists()
    for b in (0, 77, 255):
        lane = b // pc.per
        m = pc.models[lane]
        orc = gpu_oracle(cfg, m, sd, zend, zcen, cls=O.BitSwapOracle)
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
    states = initial_states(B, seed=400, n=5000)
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


def test_edge_coded_containers_q12():
    from bitswap_b200.container import compress_images, decompress_images
    sizes = [(40, 70), (20, 20), (33, 1)]
    rs = np.random.RandomState(5)
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", len(images), q=12)
    for edges in ("code", "crop"):
        conts = compress_images(codec, images[:1] if edges == "crop" else images, excess_state_len=3000, edges=edges)
        back = decompress_images(codec, conts)
        if edges == "crop":
            assert np.array_equal(back[0], images[0][:32, :64])
    conts = compress_images(codec, images, excess_state_len=3000, edges="code")
    back = decompress_images(codec, conts)
    for img, rec in zip(images, back):
        assert rec.shape == img.shape and np.array_equal(rec, img)
    orc = gpu_oracle(cfg, m, sd, zend, zcen)
    for img, cont in zip(images, conts):
        assert np.array_equal(cont, demo_oracle_container(orc, img, 3000)), img.shape


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
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny", 2, q=12)
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
    ss.import_lists(initial_states(1, seed=5))
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
