"""Partial edge blocks on the GPU: bsw_codec_encode_ext / bsw_codec_decode_ext against the extent-aware oracle, across
every coder variant, and compress_images(edges="code") end to end."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from coder_harness import coder_paths, initial_states                 # noqa: E402
from codec_harness import demo_oracle_container, gpu_oracle, setup     # noqa: E402
from edge_oracle import pad_block                                      # noqa: E402
from oracle import oracle as O                                         # noqa: E402
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200.config import preset                                 # noqa: E402
from bitswap_b200.codec import Bins, PipelinedCodec, BITSWAP, BBANS    # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402

MIXED = [(1, 1), (1, 32), (32, 1), (17, 29), (32, 32), (5, 7)]


def _ext(extents):
    return torch.tensor(extents, dtype=torch.int16, device="cuda")


def _code(codec, ss, states, imgs, exts, scheme):
    """Encode len(imgs) chained batches, export, decode them back; returns (states after encode, decoded batches)."""
    ss.import_lists(states)
    for x, e in zip(imgs, exts):
        codec.encode(ss, torch.from_numpy(x).cuda(), scheme=scheme, extent=None if e is None else _ext(e))
    torch.cuda.synchronize()
    ss.raise_on_error()
    enc = ss.export_lists()
    dec = []
    for x, e in reversed(list(zip(imgs, exts))):
        out = codec.decode(ss, x.shape[0], scheme=scheme, extent=None if e is None else _ext(e))
        torch.cuda.synchronize()
        dec.append(out.cpu().numpy())
    ss.raise_on_error()
    return enc, dec[::-1]


@pytest.mark.parametrize("name,scheme", [("tiny", BITSWAP), ("tiny3", BITSWAP), ("tiny", BBANS), ("tiny3", BBANS)])
def test_ext_vs_oracle_with_injected_nets(name, scheme):
    """Mixed extents in one batch, on a sub-range of the stream set: every stream's state list equals the oracle's after
    encode; decode restores the valid pixels (edge-padded) and the initial states; the streams outside the range stay put."""
    B, first = len(MIXED), 2
    cfg, m, sd, zend, zcen, bins, codec = setup(name, B)
    imgs = synthetic.synthetic_images(cfg, 2 * B, seed=11).reshape(2, B, *cfg.xs)
    exts = [MIXED, MIXED[::-1]]
    ss = StreamSet(B + first + 1, 1 << 14)
    states = initial_states(B + first + 1, 500)
    ss.import_lists(states)
    for x, e in zip(imgs, exts):
        codec.encode(ss, torch.from_numpy(x).cuda(), first=first, scheme=scheme, extent=_ext(e))
    torch.cuda.synchronize()
    ss.raise_on_error()
    got = ss.export_lists()
    assert got[:first] == states[:first] and got[first + B:] == states[first + B:]
    orc = gpu_oracle(cfg, m, sd, zend, zcen)
    enc = orc.encode_image if scheme == BITSWAP else orc.encode_image_bbans
    for b in range(B):
        st = O.CState.from_list(states[first + b])
        for x, e in zip(imgs, exts):
            st = enc(st, x[b], extent=e[b])
        assert got[first + b] == st.to_list(), f"stream {b}, extents {exts[0][b]}, {exts[1][b]}"
    for x, e in reversed(list(zip(imgs, exts))):
        out = codec.decode(ss, B, first=first, scheme=scheme, extent=_ext(e)).cpu().numpy()
        for b in range(B):
            assert np.array_equal(out[b].reshape(-1), pad_block(x[b].reshape(-1), e[b]).astype(np.uint8))
    ss.raise_on_error()
    assert ss.export_lists() == states


@pytest.mark.parametrize("scheme", [BITSWAP, BBANS])
def test_full_extents_equal_the_plain_calls(scheme):
    B = 5
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", B)
    imgs = list(synthetic.synthetic_images(cfg, 2 * B, seed=13).reshape(2, B, *cfg.xs))
    ss = StreamSet(B, 1 << 14)
    states = initial_states(B, 600)
    a = _code(codec, ss, states, imgs, [None, None], scheme)
    b = _code(codec, ss, states, imgs, [[(32, 32)] * B] * 2, scheme)
    assert a[0] == b[0]
    assert all(np.array_equal(x, y) for x, y in zip(a[1], b[1]))
    assert all(np.array_equal(x, y) for x, y in zip(a[1], imgs))


@pytest.mark.parametrize("scheme", [BITSWAP, BBANS])
def test_masked_calls_agree_across_coder_variants(scheme):
    """Two-phase on/off, generic (rows mode 0) and affine (rows mode 1) pixel kernels, overlap mode on/off and a
    PipelinedCodec with 1 and 3 lanes leave identical streams and decode identical blocks."""
    B = len(MIXED)
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", B)
    imgs = list(synthetic.synthetic_images(cfg, 2 * B, seed=17).reshape(2, B, *cfg.xs))
    exts = [MIXED, MIXED[::-1]]
    ss = StreamSet(B, 1 << 14)
    states = initial_states(B, 700)
    want = _code(codec, ss, states, imgs, exts, scheme)
    variants = []
    codec.set_two_phase(False)
    variants.append(("fused", _code(codec, ss, states, imgs, exts, scheme)))
    codec.set_two_phase(True)
    for mode in (0, 1):
        with coder_paths(rows_mode=mode):
            variants.append((f"rows mode {mode}", _code(codec, ss, states, imgs, exts, scheme)))
    codec.set_dual_stream(True)
    variants.append(("overlap", _code(codec, ss, states, imgs, exts, scheme)))
    codec.set_dual_stream(False)
    for lanes in (1, 3):
        pc = PipelinedCodec(cfg, sd, bins, B, lanes=lanes, use_tensor_cores=False)
        variants.append((f"{lanes} lanes", _code(pc, ss, states, imgs, exts, scheme)))
    for label, got in variants:
        assert got[0] == want[0], label
        assert all(np.array_equal(x, y) for x, y in zip(got[1], want[1])), label


def test_pad_area_does_not_change_the_bitstream():
    B = len(MIXED)
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", B)
    x = synthetic.synthetic_images(cfg, B, seed=19)
    y = x.copy()
    rs = np.random.RandomState(3)
    for b, (vh, vw) in enumerate(MIXED):
        noise = rs.randint(0, 256, y[b].shape).astype(np.uint8)
        keep = np.zeros(y[b].shape, bool)
        keep[:, :vh, :vw] = True
        y[b] = np.where(keep, y[b], noise)
    ss = StreamSet(B, 1 << 14)
    states = initial_states(B, 800)
    a = _code(codec, ss, states, [x], [MIXED], BITSWAP)
    b = _code(codec, ss, states, [y], [MIXED], BITSWAP)
    assert a[0] == b[0] and np.array_equal(a[1][0], b[1][0])


def test_invalid_extent_flags_only_that_stream():
    B = 4
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", B)
    x = synthetic.synthetic_images(cfg, B, seed=23)
    states = initial_states(B, 900)
    ss = StreamSet(B, 1 << 14)
    ss.import_lists(states)
    codec.encode(ss, torch.from_numpy(x).cuda(), extent=_ext([(32, 32), (0, 5), (33, 1), (7, 7)]))
    _, _, flags = ss.sizes()
    assert flags.tolist() == [0, 4, 4, 0]
    with pytest.raises(IndexError, match="block extent"):
        ss.raise_on_error()
    got = ss.export_lists()
    assert got[1] == states[1] and got[2] == states[2]
    ref = StreamSet(B, 1 << 14)
    ref.import_lists(states)
    codec.encode(ref, torch.from_numpy(x).cuda(), extent=_ext([(32, 32), (32, 32), (32, 32), (7, 7)]))
    want = ref.export_lists()
    assert got[0] == want[0] and got[3] == want[3]
    # decode: a bad extent is flagged before the first pop
    ref.raise_on_error()
    out = codec.decode(ref, B, extent=_ext([(32, 32), (32, 32), (1, 0), (7, 7)])).cpu().numpy()
    _, _, flags = ref.sizes()
    assert flags.tolist() == [0, 0, 4, 0]
    assert np.array_equal(out[0], x[0])
    assert np.array_equal(out[3].reshape(-1), pad_block(x[3].reshape(-1), (7, 7)).astype(np.uint8))


def test_container_edges_code_vs_oracle_demo_procedure():
    from bitswap_b200.container import compress_images, decompress_images
    sizes = [(100, 70), (20, 20), (33, 1), (64, 96), (225, 224)]
    rs = np.random.RandomState(5)
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", len(images))
    conts = compress_images(codec, images, excess_state_len=3000, edges="code")
    back = decompress_images(codec, conts)
    for img, rec in zip(images, back):
        assert rec.shape == img.shape and np.array_equal(rec, img)
    crop = compress_images(codec, [images[3]], excess_state_len=3000)
    assert np.array_equal(crop[0], conts[3])                  # whole blocks: byte-identical to the crop mode
    orc = gpu_oracle(cfg, m, sd, zend, zcen)
    for img, cont in zip(images, conts):
        assert np.array_equal(cont, demo_oracle_container(orc, img, 3000)), img.shape
    pc = PipelinedCodec(cfg, sd, bins, len(images), lanes=3, use_tensor_cores=False, free_running=True)
    conts_pc = compress_images(pc, images, excess_state_len=3000, edges="code")
    assert all(np.array_equal(a, b) for a, b in zip(conts, conts_pc))
    back_pc = decompress_images(pc, conts_pc)
    assert all(np.array_equal(a, b) for a, b in zip(images, back_pc))


def test_imagenetcrop4_tensor_cores_partial_blocks():
    """The config-5 model on tensor cores: images with partial blocks round-trip exactly; one image's container equals the
    oracle's demo procedure driven by the same GPU nets."""
    from bitswap_b200.container import compress_images, decompress_images
    cfg = preset("imagenetcrop4")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    bins = Bins(cfg, zend, zcen)
    sizes = [(40, 70), (33, 33), (64, 31)]
    rs = np.random.RandomState(8)
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    pc = PipelinedCodec(cfg, sd, bins, len(images), lanes=2, use_tensor_cores=True, free_running=True)
    conts = compress_images(pc, images, excess_state_len=4000, edges="code")
    back = decompress_images(pc, conts)
    assert all(np.array_equal(a, b) for a, b in zip(images, back))
    orc = gpu_oracle(cfg, pc.models[0], sd, zend, zcen)
    assert np.array_equal(conts[2], demo_oracle_container(orc, images[2], 4000))
