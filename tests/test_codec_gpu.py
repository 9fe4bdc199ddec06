"""GPU parity of the nets (P3) and of the device-resident recursion (P4), through the C ABI."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from coder_harness import initial_states                           # noqa: E402
from codec_harness import GOLDEN, TOL, bitswap_golden, gpu_oracle, model, setup, tc_case   # noqa: E402
from conv_harness import outputs_in_conv_modes      # noqa: E402
from oracle import oracle as O                      # noqa: E402  (checker only)
from bitswap_b200 import synthetic                   # noqa: E402
from bitswap_b200.config import CodecConfig, preset  # noqa: E402
from bitswap_b200.model import Model                 # noqa: E402
from bitswap_b200.codec import BitSwapCodec, Bins, BITSWAP, BBANS   # noqa: E402
from bitswap_b200.streams import StreamSet           # noqa: E402
from bitswap_b200.rand import ImageBins              # noqa: E402


@pytest.mark.parametrize("name", ["tiny", "tiny3"])
def test_p3_nets_vs_reference_golden(name):
    """mu/scale of every infer(i)/generate(i) against outputs of the REFERENCE Model (golden file)."""
    cfg = preset(name)
    g = np.load(os.path.join(GOLDEN, f"model_{name}.npz"))
    m, _ = model(cfg, 4)
    _, zcen = synthetic.synthetic_bins(cfg, seed=0)
    xcen = ImageBins(torch.float64, "cpu", cfg.xdim).centres()
    zr = torch.arange(cfg.zdim)
    worst = 0.0
    for i in range(cfg.nz):
        if i == 0:
            given = xcen[torch.arange(cfg.xdim), torch.from_numpy(g["x"].astype(np.int64))]
        else:
            given = zcen[i - 1, zr, torch.from_numpy(g[f"zsym_in_infer{i}"].astype(np.int64))]
        mu, sc = m.infer(i)(given=given.cuda())            # reference call shape: flat float64 in, flat float64 out
        assert mu.dtype == torch.float64 and mu.shape == (cfg.zdim,)
        worst = max(worst, np.abs(mu.cpu().numpy() - g[f"infer{i}_mu"]).max(), np.abs(sc.cpu().numpy() - g[f"infer{i}_scale"]).max())
        z = zcen[i, zr, torch.from_numpy(g[f"zsym_in_gen{i}"].astype(np.int64))]
        mu, sc = m.generate(i)(given=z.cuda())
        assert mu.shape == ((cfg.xdim,) if i == 0 else (cfg.zdim,))
        worst = max(worst, np.abs(mu.cpu().numpy() - g[f"gen{i}_mu"]).max(), np.abs(sc.cpu().numpy() - g[f"gen{i}_scale"]).max())
    assert worst < TOL, worst


@pytest.mark.parametrize("name,B", [("mnist2", 3), ("cifar8", 2)])
def test_p3_nets_vs_oracle_full_width(name, B):
    """Reference-sized nets (W=63 / W=252) against the torch float32 oracle, batched, batch-invariant."""
    cfg = preset(name)
    m, sd = model(cfg, B)
    orc = O.ModelOracle(cfg, sd)
    rs = np.random.RandomState(4)
    _, zcen = synthetic.synthetic_bins(cfg, seed=0)
    worst = 0.0
    for i in range(cfg.nz):
        if i == 0:
            given = torch.from_numpy((rs.randint(0, 256, (B, cfg.xdim)) - 127.5) / 127.5)
        else:
            given = torch.from_numpy(rs.uniform(-5, 5, (B, cfg.zdim)))
        for kind in ("infer", "generate"):
            gv = given if (kind == "infer") else torch.from_numpy(rs.uniform(-5, 5, (B, cfg.zdim)))
            f_gpu = m.infer(i) if kind == "infer" else m.generate(i)
            f_cpu = orc.infer(i) if kind == "infer" else orc.generate(i)
            mu, sc = f_gpu(gv.cuda())
            mu_o, sc_o = f_cpu(gv)
            worst = max(worst, (mu.cpu() - mu_o).abs().max().item(), (sc.cpu() - sc_o).abs().max().item())
            # batch invariance / determinism (H3): row 1 alone gives bit-identical outputs
            mu1, sc1 = f_gpu(gv[1:2].cuda())
            assert torch.equal(mu1[0], mu[1]) and torch.equal(sc1[0], sc[1])
    assert worst < TOL, worst


@pytest.mark.parametrize("name", ["tiny", "tiny3"])
def test_p4_bitswap_vs_reference_trace(name):
    """Own nets + own tables on the inputs of the reference-classes golden run.  Bits-back pops SAMPLE the
    latents from the low bits of the ANS head, so a 1e-7 difference in one mu (float32 conv summation order vs
    torch-CPU) re-draws every later latent: the states cannot be compared word for word (that comparison is
    made with injected nets in test_p4_vs_oracle_with_injected_nets).  What must hold: the code length agrees
    statistically (bits/dim), identical streams stay identical, and decoding restores pixels and the initial
    state exactly."""
    g = bitswap_golden(name)
    B = 3
    cfg, m, sd, zend, zcen, bins, codec = setup(name, B)
    ss = StreamSet(B, 8192)
    imgs = synthetic.synthetic_images(cfg, g["nimg"], seed=7)
    w, head = synthetic.initial_words(g["nwords"], seed=100)
    ss.fill(w, head)
    init = ss.export_lists()
    for xi in range(g["nimg"]):
        x = torch.from_numpy(np.repeat(imgs[xi][None], B, axis=0)).cuda()
        codec.encode(ss, x)
    ss.raise_on_error()
    final = ss.export_lists()
    assert final[0] == final[1] == final[2]                      # identical streams stay identical
    bpd = 32.0 * (len(final[0]) - len(init[0])) / (cfg.xdim * g["nimg"])
    print(f"{name}: net bits/dim ours {bpd:.4f} reference-classes run {g['net_bits_per_dim']:.4f}")
    assert abs(bpd - g["net_bits_per_dim"]) < 0.25              # 2 images of random-weight nets: sampling noise
    for xi in reversed(range(g["nimg"])):
        out = codec.decode(ss, B)
        assert np.array_equal(out.cpu().numpy(), np.repeat(imgs[xi][None], B, axis=0))
    ss.raise_on_error()
    assert ss.export_lists() == init


@pytest.mark.parametrize("name,scheme", [("tiny", BITSWAP), ("tiny3", BITSWAP), ("tiny", BBANS), ("tiny3", BBANS)])
def test_p4_vs_oracle_with_injected_nets(name, scheme):
    """Oracle recursion driven with OUR mu/sigma and the reference's float64 table expression evaluated by torch on the
    GPU (where the reference evaluates it): EVERY stream's state list is bit-identical, for distinct images/streams."""
    B, nimg = 4, 2
    cfg, m, sd, zend, zcen, bins, codec = setup(name, B)
    ss = StreamSet(B, 1 << 14)
    imgs = synthetic.synthetic_images(cfg, B * nimg, seed=11).reshape(nimg, B, *cfg.xs)
    states = initial_states(B, seed=100, n=3000, step=11)
    ss.import_lists(states)
    for xi in range(nimg):
        codec.encode(ss, torch.from_numpy(imgs[xi]).cuda(), scheme=scheme)
    ss.raise_on_error()
    got = ss.export_lists()
    n_ident = 0
    for b in range(B):
        orc = gpu_oracle(cfg, m, sd, zend, zcen, cls=O.BitSwapOracle)
        st = O.CState.from_list(states[b])
        for xi in range(nimg):
            st = (orc.encode_image if scheme == BITSWAP else orc.encode_image_bbans)(st, imgs[xi, b])
        want = st.to_list()
        assert len(got[b]) == len(want), f"stream {b}: word count differs"
        n_ident += int(got[b] == want)
    print(f"{name}/{'bitswap' if scheme == BITSWAP else 'bbans'}: {n_ident}/{B} streams bit-identical to the oracle")
    assert n_ident == B
    for xi in reversed(range(nimg)):
        out = codec.decode(ss, B, scheme=scheme)
        assert np.array_equal(out.cpu().numpy(), imgs[xi])
    ss.raise_on_error()
    assert ss.export_lists() == states


def test_p4_roundtrip_sub_range_and_chain_independence():
    """Coding streams [2,6) leaves the others untouched; a stream's result does not depend on its neighbours."""
    B = 8
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny", B)
    ss = StreamSet(B, 8192)
    w, head = synthetic.initial_words(1200, seed=100)
    ss.fill(w, head)
    init = ss.export_lists()
    imgs = synthetic.synthetic_images(cfg, 4, seed=3)
    codec.encode(ss, torch.from_numpy(imgs).cuda(), first=2)
    after = ss.export_lists()
    assert after[:2] == init[:2] and after[6:] == init[6:]
    ss2 = StreamSet(1, 8192)
    ss2.fill(w, head)
    codec.encode(ss2, torch.from_numpy(imgs[2:3]).cuda())
    assert ss2.export_lists()[0] == after[4]
    out = codec.decode(ss, 4, first=2)
    assert np.array_equal(out.cpu().numpy(), imgs) and ss.export_lists() == init


# ---------------------------------------------------------------------------------------------------
# tensor-core path (conv_tc.cu): bf16 hi/lo split, three wgmma per k-step, float32 register accumulation
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("label,cfg", [
    ("one 3x3 layer", CodecConfig(xs=(3, 32, 32), nz=1, zchannels=8, nprocessing=0, resdepth=1, reswidth=252)),
    ("one 5x5 layer", CodecConfig(xs=(3, 32, 32), nz=1, zchannels=8, nprocessing=1, resdepth=0, reswidth=252)),
    ("width 256 crop", CodecConfig(xs=(3, 32, 32), nz=2, zchannels=8, nprocessing=1, resdepth=2, reswidth=256, cond_xscale=True)),
])
def test_p3_tc_single_layers(label, cfg):
    worst_o, worst_s = tc_case(cfg, 3)
    print(f"tensor cores {label}: max |err| vs torch-f32 oracle {worst_o:.2e}, vs SIMT f32 path {worst_s:.2e}")
    assert worst_o < TOL and worst_s < TOL


@pytest.mark.parametrize("label,cfg", [
    ("zchannels 20: SIMT heads after a tensor-core trunk",
     CodecConfig(xs=(3, 32, 32), nz=2, zchannels=20, nprocessing=1, resdepth=2, reswidth=252)),
    ("zchannels 40: SIMT in-conv + k_split_planes, SIMT heads",
     CodecConfig(xs=(3, 32, 32), nz=2, zchannels=40, nprocessing=1, resdepth=2, reswidth=252)),
    ("nz 4, resdepth 2: levels without ResNet layers",
     CodecConfig(xs=(3, 32, 32), nz=4, zchannels=8, nprocessing=1, resdepth=2, reswidth=252)),
    ("width 193", CodecConfig(xs=(3, 32, 32), nz=2, zchannels=8, nprocessing=1, resdepth=2, reswidth=193)),
    ("width 255", CodecConfig(xs=(3, 32, 32), nz=2, zchannels=8, nprocessing=1, resdepth=2, reswidth=255, cond_xscale=True)),
])
def test_p3_tc_dispatch_seams_vs_f64_oracle(label, cfg):
    """Whole nets at the dispatch seams of run_net on a tensor-core model, against the float64 oracle."""
    worst_o, worst_s = tc_case(cfg, 3, dtype=torch.float64)
    print(f"tensor cores {label}: max |err| vs torch-f64 oracle {worst_o:.2e}, vs SIMT f32 path {worst_s:.2e}")
    assert worst_o < TOL and worst_s < TOL


def test_p3_tc_persistent_kernel_equals_per_tile_kernels():
    """k_conv_wg on the persistent grid (one CTA per SM walking half-image tiles, the TMA ring prefetching across tile
    boundaries; the default) against the per-tile grid (one CTA per tile): same k-block and MMA order per accumulator,
    same epilogue arithmetic -> bit-identical mu and sigma.  B = 170 gives 680 half-image tiles per conv, i.e. up to
    six tiles per CTA on 132 SMs: accumulators and stages are reused across tiles; every conv shape on the path
    (in-convs with 1 and 25 taps, dense 3x3, 5x5, heads)."""
    cfg = CodecConfig(xs=(3, 32, 32), nz=2, zchannels=8, nprocessing=1, resdepth=1, reswidth=252)
    out = outputs_in_conv_modes(cfg, 170, (0, 7))
    for a, b in zip(out[0], out[7]):
        assert torch.equal(a, b), "conv mode 7"
    assert all(torch.isfinite(t).all() for t in out[7])


def test_p3_tc_cifar8_full():
    cfg = preset("cifar8")
    worst_o, worst_s = tc_case(cfg, 2)
    print(f"tensor cores cifar8: max |err| vs torch-f32 oracle {worst_o:.2e}, vs SIMT f32 path {worst_s:.2e}")
    assert worst_o < TOL and worst_s < TOL


def test_p4_tc_roundtrip_cifar8():
    """Encoder and decoder regenerate bit-identical tables from the tensor-core nets: exact round trip, with a
    different batch split on the decode side (H3: results do not depend on batch size or position)."""
    B = 6
    cfg, m, sd, zend, zcen, bins, codec = setup("cifar8", B, tc=True)
    ss = StreamSet(B, 8192)
    w, head = synthetic.initial_words(4096, seed=100)
    ss.fill(w, head)
    init = ss.export_lists()
    imgs = synthetic.synthetic_images(cfg, B, seed=21)
    codec.encode(ss, torch.from_numpy(imgs).cuda())
    ss.raise_on_error()
    n, _, _ = ss.sizes()
    print("cifar8 tensor cores: net bits/dim", 32.0 * (n.mean() - 4095) / cfg.xdim)
    out_a = codec.decode(ss, 2, first=0)                  # decode in two differently-sized calls
    out_b = codec.decode(ss, 4, first=2)
    ss.raise_on_error()
    assert np.array_equal(torch.cat([out_a, out_b]).cpu().numpy(), imgs)
    assert ss.export_lists() == init


@pytest.mark.parametrize("name,scheme", [("tiny3", BITSWAP), ("tiny", BBANS), ("mnist2", BITSWAP)])
def test_two_phase_coder_equals_fused_coder(name, scheme):
    """ans_rows.cu (parallel row tables + serial coder) and the fused one-warp-per-stream kernels must leave
    bit-identical streams and symbols."""
    B = 5
    cfg, m, sd, zend, zcen, bins, codec = setup(name, B)
    ss = StreamSet(B, 1 << 14)
    imgs = synthetic.synthetic_images(cfg, B, seed=31)
    states = initial_states(B, seed=200, n=5000, step=3)
    res = []
    for two_phase in (True, False):
        codec.set_two_phase(two_phase)
        ss.import_lists(states)
        codec.encode(ss, torch.from_numpy(imgs).cuda(), scheme=scheme)
        ss.raise_on_error()
        res.append(ss.export_lists())
        out = codec.decode(ss, B, scheme=scheme)
        assert np.array_equal(out.cpu().numpy(), imgs) and ss.export_lists() == states
    assert res[0] == res[1]
    # cross: encode with one variant, decode with the other
    codec.set_two_phase(True)
    codec.encode(ss, torch.from_numpy(imgs).cuda(), scheme=scheme)
    codec.set_two_phase(False)
    out = codec.decode(ss, B, scheme=scheme)
    assert np.array_equal(out.cpu().numpy(), imgs) and ss.export_lists() == states


def test_config0_mnist_b1_state_identical_at_every_level():
    """BASELINE.json configs[0]: MNIST 32x32x1 (28x28 zero-padded), 2-latent VAE, batch = 1.  The reference's own
    loop shape (cifar_compress.py:175-250) driven level by level through the drop-in pieces -- model.infer /
    generate, the fused logistic coder, the prior table -- must leave the ANS state bit-identical to the CPU
    oracle after EVERY pop and push (oracle fed the same GPU mu/sigma), for a 2-image chain."""
    import ctypes
    from bitswap_b200._lib import lib, check, cuda_stream_ptr
    cfg = preset("mnist2")
    m, sd = model(cfg, 1)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    bins = Bins(cfg, zend, zcen)
    S, q = cfg.zsupport, cfg.quantbits

    def ptrs(level):
        a, b, c = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        check(lib().bsw_bins_device_ptrs(bins.handle, level, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)))
        return a.value, c.value

    # oracle trace with the GPU nets injected
    trace = []
    orc = gpu_oracle(cfg, m, sd, zend, zcen, cls=O.BitSwapOracle)
    orc.trace = trace
    imgs = np.zeros((2, 1, 32, 32), dtype=np.uint8)
    imgs[:, :, 2:30, 2:30] = synthetic.synthetic_images(cfg, 2, seed=13)[:, :, 2:30, 2:30]     # Pad(2), mnist_compress.py:129
    w, head = synthetic.initial_words(1500, seed=100)
    st = O.CState(w, head)
    for xi in range(2):
        st = orc.encode_image(st, imgs[xi])
    want = [(ln, sha) for _, ln, sha in trace]

    ss = StreamSet(1, 1 << 14)
    ss.fill(w, head)
    got = []

    def note():
        lst = ss.export_lists()[0]
        got.append((len(lst), O.CState.from_list(lst).digest()))
    zr = torch.arange(cfg.zdim)
    P = torch.empty((cfg.zdim, S), dtype=torch.int32, device="cuda")
    C = torch.empty((cfg.zdim, S + 1), dtype=torch.int32, device="cuda")
    zero, one = torch.zeros(1, dtype=torch.float64, device="cuda"), torch.ones(1, dtype=torch.float64, device="cuda")
    e_top = zend[-1].contiguous().cuda()
    check(lib().bsw_logistic_tables(e_top.data_ptr(), S - 1, zero.data_ptr(), one.data_ptr(), 0, cfg.zdim, S, 31, q,
                                    P.data_ptr(), C.data_ptr(), cuda_stream_ptr()))
    for xi in range(2):
        x = torch.from_numpy(imgs[xi].reshape(-1).astype(np.int64))
        zsym = None
        for zi in range(cfg.nz):
            given = zcen[zi - 1, zr, zsym.long().cpu()] if zi > 0 else (x.double() - 127.5) / 127.5
            mu, sc = m.infer(zi)(given.cuda())
            mu32, sc32 = mu.float().contiguous(), sc.float().contiguous()
            out = torch.zeros(cfg.zdim, dtype=torch.int16, device="cuda")
            ze, xe = ptrs(zi)
            check(lib().bsw_logistic_pop(ss.handle, 0, 1, mu32.data_ptr(), cfg.zdim, sc32.data_ptr(), cfg.zdim, ze, S,
                                         out.data_ptr(), cfg.zdim, S, 31, q, cuda_stream_ptr()))
            note()
            mu, sc = m.generate(zi)(zcen[zi, zr, out.long().cpu()].cuda())
            mu32, sc32 = mu.float().contiguous(), sc.float().contiguous()
            if zi > 0:
                zl, _ = ptrs(zi - 1)
                sy = zsym.to(torch.int16).contiguous()
                check(lib().bsw_logistic_push(ss.handle, 0, 1, mu32.data_ptr(), cfg.zdim, sc32.data_ptr(), cfg.zdim, zl, S,
                                              sy.data_ptr(), cfg.zdim, S, 31, q, cuda_stream_ptr()))
            else:
                sy = x.to(torch.int16).cuda().contiguous()
                check(lib().bsw_logistic_push(ss.handle, 0, 1, mu32.data_ptr(), cfg.xdim, sc32.data_ptr(), cfg.xdim, xe, 0,
                                              sy.data_ptr(), cfg.xdim, 256, 31, 8, cuda_stream_ptr()))
            note()
            zsym = out
        s32 = zsym.to(torch.int32).contiguous()
        check(lib().bsw_ans_push(ss.handle, 0, 1, P.data_ptr(), C.data_ptr(), 0, 0, s32.data_ptr(), cfg.zdim, S, 31,
                                 cuda_stream_ptr()))
        note()
    ss.raise_on_error()
    assert got == want


def test_pipelined_codec_equals_single_codec():
    """PipelinedCodec (sub-batches on separate CUDA streams) leaves exactly the streams a single codec leaves."""
    from bitswap_b200.codec import PipelinedCodec
    B = 7
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", B)
    ss = StreamSet(B, 1 << 14)
    pc = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), B, lanes=3, use_tensor_cores=False)
    imgs = synthetic.synthetic_images(cfg, 2 * B, seed=41).reshape(2, B, *cfg.xs)
    states = initial_states(B, seed=300, n=4000, step=1)
    res = []
    for c in (codec, pc):
        ss.import_lists(states)
        for xi in range(2):
            c.encode(ss, torch.from_numpy(imgs[xi]).cuda())
        torch.cuda.synchronize()
        ss.raise_on_error()
        res.append(ss.export_lists())
    assert res[0] == res[1]
    for xi in (1, 0):
        out = pc.decode(ss, B)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), imgs[xi])
    assert ss.export_lists() == states


@pytest.mark.parametrize("name,tc,scheme,lanes", [("cifar8", True, BITSWAP, 2), ("tiny3", False, BBANS, 1), ("imagenetcrop4", True, BITSWAP, 1)])
def test_overlap_mode_equals_program_order(name, tc, scheme, lanes):
    """bsw_codec_set_dual_stream(1) enqueues the recursion as a dependency graph on three internal streams (nets / float64
    table kernels / serial coder kernels) so that one chain's tensor-pipe and FP64-pipe work overlap.  It must leave
    exactly the streams the plain program order leaves -- three chained images per stream, so every buffer is reused
    across images -- and decode them back, with the overlap on in both directions."""
    from bitswap_b200.codec import PipelinedCodec
    B = 6
    cfg = preset(name)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    pc = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), B, lanes=lanes, use_tensor_cores=tc)
    ss = StreamSet(B, 1 << 15)
    imgs = synthetic.synthetic_images(cfg, 3 * B, seed=43).reshape(3, B, *cfg.xs)
    states = initial_states(B, seed=400, n=5000, step=1)
    res = []
    for mode in (0, 1):
        pc.set_dual_stream(mode)
        ss.import_lists(states)
        for xi in range(3):
            pc.encode(ss, torch.from_numpy(imgs[xi]).cuda(), scheme=scheme)
        torch.cuda.synchronize()
        ss.raise_on_error()
        res.append(ss.export_lists())
    assert res[0] == res[1]
    for xi in (2, 1, 0):
        out = pc.decode(ss, B, scheme=scheme)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), imgs[xi])
    assert ss.export_lists() == states


def test_container_variable_size_images_vs_oracle_demo_procedure():
    """BASELINE config 5 shape: variable-size images, each ONE chain over its 32x32 blocks, many images at once.
    The containers must equal what the reference's demo procedure (demo_compress.py:113-162,268-284) yields when the
    oracle runs it per image with the same (GPU) nets, and decompress_images must restore the cropped images."""
    from bitswap_b200.container import compress_images, decompress_images, extract_blocks
    cfg = preset("tiny3")                 # RGB, conditional x-scale: the imagenetcrop model family
    sizes = [(64, 96), (32, 32), (100, 70), (40, 129)]
    rs = np.random.RandomState(5)
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    _, m, sd, zend, zcen, _, codec = setup("tiny3", len(images))
    conts = compress_images(codec, images, excess_state_len=3000)
    # oracle: the reference demo loop, one image at a time
    orc = gpu_oracle(cfg, m, sd, zend, zcen, cls=O.BitSwapOracle)
    for img, cont in zip(images, conts):
        blocks, h, w = extract_blocks(img)
        wds, head = synthetic.initial_words(3000, seed=100)
        st = O.CState(wds, head)
        low = st.n
        # track the lowest stack depth like demo_compress.py:137 (after every pop)
        pops = []
        orc.trace = pops
        for b in blocks:
            st = orc.encode_image(st, b.transpose(2, 0, 1))
        low = min([ln - 1 for tag, ln, _ in pops if tag.startswith("pop")] + [low])
        want = np.concatenate([st.words[low:st.n], np.array([st.head & 0xffffffff, st.head >> 32, len(blocks), h, w], dtype=np.uint64)]).astype(np.uint32)
        assert np.array_equal(cont, want)
    back = decompress_images(codec, conts)
    for img, rec in zip(images, back):
        h, w = img.shape[0] - img.shape[0] % 32, img.shape[1] - img.shape[1] % 32
        assert np.array_equal(rec, img[:h, :w])
    # the same through a free-running multi-lane codec (what `bench.py --config crop` runs): identical containers
    from bitswap_b200.codec import PipelinedCodec
    pc = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), len(images), lanes=3, use_tensor_cores=False, free_running=True)
    conts_pc = compress_images(pc, images, excess_state_len=3000)
    assert all(np.array_equal(a, b) for a, b in zip(conts, conts_pc))
    back_pc = decompress_images(pc, conts_pc)
    assert all(np.array_equal(a, b) for a, b in zip(back, back_pc))


def test_gpu_discretize_builds_usable_bins():
    """discretize() with the reference's signature on the GPU nets: table layout, float32 top level, uniform
    lower levels covering every sample -- and the codec round-trips with the tables it built."""
    from bitswap_b200.discretization import discretize
    cfg = preset("tiny3")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    m = Model.from_config(cfg, max_batch=128).load_state_dict(sd)
    m.compress()
    imgs = torch.from_numpy(synthetic.synthetic_images(cfg, 512, seed=17, kind="smooth"))
    zend, zcen = discretize(cfg.nz, cfg.quantbits, torch.float64, "cpu", m, "synthetic", images=imgs, ppb=8)
    S = cfg.zsupport
    assert zend.shape == (cfg.nz, cfg.zdim, S - 1) and zcen.shape == (cfg.nz, cfg.zdim, S) and zend.dtype == torch.float64
    assert torch.all(zend[:, :, 1:] > zend[:, :, :-1])                                   # strictly increasing endpoints
    ref_e, _ = synthetic.synthetic_bins(cfg, seed=0)
    assert torch.equal(zend[-1], ref_e[-1])                                              # top level == rand.Bins (float32)
    w = zend[0, :, 1:] - zend[0, :, :-1]
    assert (w.max(dim=1).values - w.min(dim=1).values).max() < 1e-9                     # uniform width per dimension
    B = 4
    codec = BitSwapCodec(cfg, m, Bins(cfg, zend, zcen), B)
    ss = StreamSet(B, 8192)
    wds, head = synthetic.initial_words(3000, seed=100)
    ss.fill(wds, head)
    x = imgs[:B].cuda()
    codec.encode(ss, x)
    out = codec.decode(ss, B)
    ss.raise_on_error()
    assert torch.equal(out, x)


def test_gpu_discretize_vs_oracle_nets_on_identical_noise():
    """f3: the sampler is pinned, not just the table layout.  The same U(0,1) draws go through (a) discretize() on the GPU
    nets with the sampling / extrema / linspace kernels of csrc/discretize.cu and (b) the reference procedure
    (discretization.py:59-83,105-118) restated in torch-CPU over the oracle nets with float16 storage and the sklearn-
    equivalent fit.  Endpoints must agree to float16 storage accuracy: a net difference of 1e-6 can flip the float16
    rounding of an extreme sample (one float16 ulp = 2^-10 relative), so the bar is: 99 % of all endpoints within 1e-3 and
    every endpoint within 4 float16 ulps of the range."""
    from bitswap_b200.discretization import discretize, uniform_bins
    cfg = preset("tiny3")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    bs, ppb, q = 64, 8, cfg.quantbits
    m = Model.from_config(cfg, max_batch=bs).load_state_dict(sd)
    m.compress()
    orc = O.ModelOracle(cfg, sd)
    imgs = torch.from_numpy(synthetic.synthetic_images(cfg, 1024, seed=19, kind="smooth"))
    rs = np.random.RandomState(77)
    bank = {}

    def uniforms(tag, shape):
        if tag not in bank:
            bank[tag] = torch.from_numpy(rs.random_sample(shape).astype(np.float32))
        return bank[tag].cuda()
    zend, zcen = discretize(cfg.nz, q, torch.float64, "cpu", m, "synthetic", images=imgs, ppb=ppb, bs=bs, uniforms=uniforms)

    # (b) the reference procedure on the CPU nets, same noise
    nz, zdim, nbins = cfg.nz, cfg.zdim, 1 << q
    nsamples = ppb * nbins
    batches = nsamples // bs

    def eps_of(tag, shape):
        u = torch.clamp(bank[tag] if tag in bank else uniforms(tag, shape).cpu(), min=1e-30, max=1 - 1e-30)
        return torch.log(u) - torch.log1p(-u)
    x = (imgs.float().reshape(imgs.shape[0], -1) - 127.5) / 127.5
    while x.shape[0] < nsamples:
        x = torch.cat([x, x])
    gen_s = torch.zeros((nz, nsamples, zdim), dtype=torch.float16)
    inf_s = torch.zeros((nz, nsamples, zdim), dtype=torch.float16)
    gen_s[-1] = eps_of(("top",), (nsamples, zdim)).half()
    for zi in reversed(range(1, nz)):
        for bi in range(batches):
            sl = slice(bi * bs, bi * bs + bs)
            mu, sc = orc.generate(zi)(gen_s[zi][sl].float())
            gen_s[zi - 1][sl] = (mu.double() + sc.double() * eps_of(("gen", zi, bi), mu.shape).double()).half()
        lvl = nz - zi - 1
        for bi in range(batches):
            sl = slice(bi * bs, bi * bs + bs)
            mu, sc = orc.infer(lvl)(x[sl] if lvl == 0 else inf_s[lvl - 1][sl].float())
            inf_s[lvl][sl] = (mu.double() + sc.double() * eps_of(("inf", lvl, bi), mu.shape).double()).half()
    worst, close, total = 0.0, 0, 0
    for zi in range(nz - 1):
        e_ref, c_ref = uniform_bins(torch.cat([gen_s[zi], inf_s[zi]], dim=0), q)
        span = (e_ref[:, -1] - e_ref[:, 0]).abs().max().item()
        d = (zend[zi] - e_ref).abs()
        worst = max(worst, d.max().item() / max(span, 1e-9))
        close += int((d <= 1e-3).sum()); total += d.numel()
        assert (zcen[zi] - c_ref).abs().max().item() <= d.max().item() + 1e-12
    print(f"discretize on identical noise: {100.0 * close / total:.2f} % of endpoints within 1e-3, worst {worst:.2e} of the range")
    assert close >= 0.99 * total and worst <= 4 * 2.0 ** -10
    # the top level is rand.Bins on float32 zeros / ones, no sampling: exact.  (The sampling, extrema and fit kernels are
    # pinned bit for bit on their own, through the C ABI, in test_supports_gpu.py.)
    ref_top, _ = synthetic.synthetic_bins(cfg, seed=0)
    assert torch.equal(zend[-1], ref_top[-1])


def test_elbo_on_gpu_nets_matches_oracle_nets():
    """Batched ELBO (model/cifar_train.py:441-490) on the GPU nets vs the same assembly on the torch oracle with the
    same noise: bits/dim within 1e-3; and it is the quantity the code length tracks (reported, not asserted: random-init
    nets make both far from trained values)."""
    from bitswap_b200.elbo import elbo
    cfg = preset("tiny3")
    B = 4
    m, sd = model(cfg, B)
    orc = O.ModelOracle(cfg, sd)
    x = torch.from_numpy(synthetic.synthetic_images(cfg, B, seed=19, kind="smooth"))
    gen = torch.Generator().manual_seed(7)
    u = [torch.rand(B, cfg.zdim, generator=gen, dtype=torch.float64).clamp_(1e-5, 1 - 1e-5) for _ in range(cfg.nz)]
    eps = [torch.log(v) - torch.log1p(-v) for v in u]
    a = elbo(m, x.cuda(), eps=eps)
    b = elbo(orc, x, cfg=cfg, eps=eps)
    assert (a["elbo_bits_per_dim"].cpu() - b["elbo_bits_per_dim"]).abs().max() < 1e-3
    print("ELBO bits/dim (random-init tiny3):", a["elbo_bits_per_dim"].cpu().numpy().round(3))


@pytest.mark.parametrize("name,B,lanes,nsample", [("cifar8", 1024, 4, 8), ("imagenet4", 96, 2, 8), ("imagenetcrop4", 24, 1, 4)])
def test_p4_full_size_configs_vs_oracle_and_batch_roundtrip(name, B, lanes, nsample):
    """BASELINE.json configs at full model size, tensor-core nets, pipelined codec:
      cifar8        configs[1] in the exact shape bench.py times: 1024 streams, 4 lanes of 256
      imagenet4     configs[2]'s model (W = 254, resdepth [2]*4)
      imagenetcrop4 configs[4]'s model (W = 256, conditional x-scale head)
    (a) `nsample` streams spread over the lanes == the oracle recursion driven with the same GPU nets and the reference's
        float64 table expression on torch-CUDA, state list for state list (cifar8: 35 840 symbol-ops per stream);
    (b) H3 / SURVEY 8e "the result must not depend on the batch": the same images coded by a small single-lane codec
        (other batch size, other positions) leave identical streams;
    (c) size-independent properties on the whole batch: identical inputs -> identical streams, exact pixel round trip,
        initial states restored, per-stream flags clean."""
    from bitswap_b200.codec import PipelinedCodec
    cfg = preset(name)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    bins = Bins(cfg, zend, zcen)
    pc = PipelinedCodec(cfg, sd, bins, B, lanes=lanes, use_tensor_cores=True)
    imgs = synthetic.synthetic_images(cfg, B, seed=77)
    imgs[1] = imgs[0]                                           # streams 0 and 1: same image, same initial state
    ss = StreamSet(B, 8192)
    w, head = synthetic.initial_words(4096, seed=100)
    ss.fill(w, head)
    init = ss.export_lists()
    pc.encode(ss, torch.from_numpy(imgs).cuda())
    torch.cuda.synchronize()
    ss.raise_on_error()
    got = ss.export_lists()
    assert got[0] == got[1] and got[0] != got[2]
    sample = sorted(set(int(v) for v in np.linspace(0, B - 1, nsample).round()))
    orc = gpu_oracle(cfg, pc.models[0], sd, zend, zcen, cls=O.BitSwapOracle)
    for b in sample:
        want = orc.encode_image(O.CState(w, head), imgs[b]).to_list()
        assert got[b] == want, f"{name}: stream {b} differs from the oracle"
    # (b) another batch composition
    m2 = Model.from_config(cfg, max_batch=len(sample), use_tensor_cores=True).load_state_dict(sd)
    m2.compress()
    c2 = BitSwapCodec(cfg, m2, bins, len(sample))
    ss2 = StreamSet(len(sample), 8192)
    ss2.fill(w, head)
    c2.encode(ss2, torch.from_numpy(np.ascontiguousarray(imgs[sample])).cuda())
    torch.cuda.synchronize()
    ss2.raise_on_error()
    assert ss2.export_lists() == [got[b] for b in sample]
    out = pc.decode(ss, B)
    torch.cuda.synchronize()
    ss.raise_on_error()
    assert np.array_equal(out.cpu().numpy(), imgs) and ss.export_lists() == init
