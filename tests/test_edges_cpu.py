"""Partial edge blocks without a GPU: the extent-aware oracle recursions, the tiling with extents, and the container
header rules for edge-coded images."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from edge_oracle import EdgeOracle, pad_block           # noqa: E402
from oracle import oracle as O                            # noqa: E402
from bitswap_b200 import synthetic                        # noqa: E402
from bitswap_b200.config import preset                    # noqa: E402
from bitswap_b200.container import (block_extents, decompress_images, extract_blocks, extract_edge_blocks,   # noqa: E402
                                    unextract_edge_blocks)

ENCODE = {"bitswap": "encode_image", "bbans": "encode_image_bbans"}
DECODE = {"bitswap": "decode_image", "bbans": "decode_image_bbans"}


def _oracle(name):
    cfg = preset(name)
    torch.set_num_threads(4)
    m = O.ModelOracle(cfg, synthetic.synthetic_state_dict(cfg, seed=50, varied=True))
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    return cfg, EdgeOracle(cfg, m, zend, zcen, coder="c", pmf="torch")


@pytest.mark.parametrize("name", ["tiny", "tiny3"])
@pytest.mark.parametrize("scheme", ["bitswap", "bbans"])
def test_oracle_with_extents_round_trips_valid_pixels_and_state(name, scheme):
    """A chain of three partial blocks: decoding returns each block's valid pixels, edge-padded, and the initial state."""
    cfg, orc = _oracle(name)
    imgs = synthetic.synthetic_images(cfg, 3, seed=7)
    extents = [(17, 29), (1, 32), (32, 1)]
    w, head = synthetic.initial_words(1500, seed=100)
    st = O.CState(w, head)
    init = st.digest()
    for x, e in zip(imgs, extents):
        st = getattr(orc, ENCODE[scheme])(st, x, extent=e)
    for x, e in reversed(list(zip(imgs, extents))):
        st, got = getattr(orc, DECODE[scheme])(st, extent=e)
        assert np.array_equal(got, pad_block(x.reshape(-1), e).astype(np.uint8))
    assert st.digest() == init


@pytest.mark.parametrize("scheme", ["bitswap", "bbans"])
def test_full_extent_equals_unmasked_oracle(scheme):
    cfg, orc = _oracle("tiny3")
    x = synthetic.synthetic_images(cfg, 1, seed=9)[0]
    w, head = synthetic.initial_words(1500, seed=100)
    a = getattr(orc, ENCODE[scheme])(O.CState(w, head), x)
    b = getattr(orc, ENCODE[scheme])(O.CState(w, head), x, extent=(32, 32))
    assert a.to_list() == b.to_list()


def test_masked_pixels_cost_no_bits_and_pad_area_is_ignored():
    """A (1, 1) block pushes 3 pixel symbols instead of 3072: far fewer words; garbage outside the extent changes nothing."""
    cfg, orc = _oracle("tiny3")
    x = synthetic.synthetic_images(cfg, 1, seed=9)[0]
    y = x.copy()
    y[:, 1:, :] = 255 - y[:, 1:, :]
    y[:, :, 1:] = 0
    w, head = synthetic.initial_words(1500, seed=100)
    full = orc.encode_image(O.CState(w, head), x)
    one = orc.encode_image(O.CState(w, head), x, extent=(1, 1))
    assert one.n < full.n
    assert orc.encode_image(O.CState(w, head), y, extent=(1, 1)).to_list() == one.to_list()


def test_oracle_rejects_bad_extents():
    cfg, orc = _oracle("tiny")
    x = synthetic.synthetic_images(cfg, 1, seed=9)[0]
    w, head = synthetic.initial_words(900, seed=100)
    for e in [(0, 5), (5, 0), (33, 1), (1, 33)]:
        with pytest.raises(ValueError):
            orc.encode_image(O.CState(w, head), x, extent=e)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 40), (40, 1), (20, 20), (33, 1), (32, 32), (64, 96), (100, 70), (225, 224)])
def test_edge_tiling_roundtrip_and_extents(h, w):
    rs = np.random.RandomState(h * 1000 + w)
    img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    blocks, ext, hh, ww = extract_edge_blocks(img)
    gh, gw = -(-h // 32), -(-w // 32)
    assert (hh, ww) == (h, w) and blocks.shape == (gh * gw, 32, 32, 3) and ext.shape == (gh * gw, 2) and ext.dtype == np.int16
    for k, (vh, vw) in enumerate(ext):
        by, bx = divmod(k, gw)
        assert (vh, vw) == (min(32, h - 32 * by), min(32, w - 32 * bx))
        # valid region = the image, the rest = edge replication (np.pad "edge" of the block's valid region)
        assert np.array_equal(blocks[k, :vh, :vw], img[32 * by:32 * by + vh, 32 * bx:32 * bx + vw])
        chw = blocks[k].transpose(2, 0, 1).reshape(-1)
        assert np.array_equal(pad_block(chw, (vh, vw)), chw.astype(np.int64))
    assert np.array_equal(unextract_edge_blocks(blocks, h, w), img)
    if h % 32 == 0 and w % 32 == 0:                          # whole blocks: the same tiling as the crop mode
        assert np.array_equal(blocks, extract_blocks(img)[0]) and (ext == 32).all()
    assert np.array_equal(block_extents(h, w), ext)


def test_edge_coded_headers_are_parsed_and_checked_before_any_device_work():
    """Tails of edge-coded containers carry the true H, W and nblocks = ceil(H/32) * ceil(W/32).  Inconsistent ones are a
    ValueError while the headers are parsed, before any codec is touched (so None stands in for it)."""
    good = [np.array([7, 7, 1, 0, 8, 64, 100], np.uint32),      # 2 x 4 blocks
            np.array([7, 1, 0, 1, 1, 1], np.uint32),            # a single pixel
            np.array([1, 0, 2, 33, 1], np.uint32)]              # 2 x 1 blocks
    bad = [np.array([7, 7, 1, 0, 6, 64, 100], np.uint32),       # 64 x 100 needs 8 blocks
           np.array([7, 1, 0, 2, 1, 1], np.uint32),             # one pixel is one block
           np.array([1, 0, 1, 33, 1], np.uint32),
           np.array([1, 0, 0, 0, 5], np.uint32)]
    for c in bad:
        with pytest.raises(ValueError):
            decompress_images(None, good + [c])
    # well-formed headers get past parsing and only then need the codec
    with pytest.raises(AttributeError):
        decompress_images(None, good)
    # the HWC quirk has no edge-coded form
    with pytest.raises(ValueError):
        decompress_images(None, [good[0]], hwc_quirk=True)


def test_compress_rejects_edge_coding_with_hwc_quirk_and_unknown_modes():
    from bitswap_b200.container import compress_images
    img = np.zeros((40, 40, 3), np.uint8)
    with pytest.raises(ValueError):
        compress_images(None, [img], hwc_quirk=True, edges="code")
    with pytest.raises(ValueError):
        compress_images(None, [img], edges="pad")
