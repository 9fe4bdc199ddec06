"""Images coded as several chains on the GPU: exact round trips, every chain against the oracle's demo procedure on its
blocks, the calls split into sub-ranges of max_batch streams, and mixed single- and multi-chain containers."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from codec_harness import chains_of, gpu_oracle, lone_chain, oracle_chain, random_images, setup   # noqa: E402
from bitswap_b200 import synthetic                                         # noqa: E402
from bitswap_b200.config import preset                                     # noqa: E402
from bitswap_b200.codec import BitSwapCodec, Bins, PipelinedCodec, BITSWAP, BBANS   # noqa: E402
from bitswap_b200.container import (chain_sizes, compress_images, decompress_images, extract_blocks,   # noqa: E402
                                    extract_edge_blocks, unpack_container)

N_INIT = 3000


def _tiles(img, edges):
    """(blocks [n, 32, 32, C], extents [n, 2] or None) of an image as compress_images tiles it."""
    if edges == "code":
        blocks, ext, _, _ = extract_edge_blocks(img)
        return blocks, ext
    return extract_blocks(img)[0], None


CASES = [("tiny", BITSWAP, "crop"), ("tiny", BBANS, "code"), ("tiny3", BITSWAP, "code"), ("tiny3", BBANS, "crop")]


@pytest.mark.parametrize("name,scheme,edges", CASES)
def test_round_trips_and_every_chain_equals_the_oracle(name, scheme, edges):
    """Odd-sized images at chain_blocks 1, 2, 3 and 7 round-trip exactly; every chain of every container holds what the
    oracle's demo procedure writes for that chain's blocks, driven by the same GPU nets."""
    sizes = [(100, 70), (33, 65), (64, 96), (97, 40)] if edges == "code" else [(100, 70), (64, 96), (130, 33), (32, 32)]
    cfg, m, sd, zend, zcen, bins, codec = setup(name, 16)
    C = cfg.xs[0]
    images = random_images(C, sizes, seed=31)
    want = images if edges == "code" else [im[:im.shape[0] // 32 * 32, :im.shape[1] // 32 * 32] for im in images]
    orc = gpu_oracle(cfg, m, sd, zend, zcen)
    checked = 0
    for L in (1, 2, 3, 7):
        conts = compress_images(codec, images, excess_state_len=N_INIT, scheme=scheme, edges=edges, chain_blocks=L)
        back = decompress_images(codec, conts, channels=C, scheme=scheme)
        for img, rec in zip(want, back):
            assert rec.shape == img.shape and np.array_equal(rec, img), (L, img.shape)
        for img, cont in zip(images, conts):
            blocks, ext = _tiles(img, edges)
            chains = chains_of(unpack_container(cont))
            assert [nb for _, _, nb in chains] == chain_sizes(len(blocks), L)
            if L not in (1, 3) and img is not images[0]:        # the oracle is slow: every chain of two splits, one image of the others
                continue
            s = 0
            for ws, hd, nb in chains:
                ow, oh = oracle_chain(orc, blocks[s:s + nb], None if ext is None else ext[s:s + nb], scheme)
                assert np.array_equal(ws, ow) and hd == oh, (L, img.shape, s)
                s += nb
                checked += 1
    assert checked > 0


def test_no_split_writes_the_reference_container():
    """chain_blocks=None and any chain_blocks >= an image's block count write the same arrays as a call without it."""
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", 4)
    images = random_images(3, [(100, 70), (64, 96), (33, 1)], seed=37)          # 4 x 3, 2 x 3 and 2 x 1 blocks
    for edges in ("crop", "code"):
        imgs = images[:2] if edges == "crop" else images
        plain = compress_images(codec, imgs, excess_state_len=N_INIT, edges=edges)
        for L in (None, 12, 13, 1000):
            got = compress_images(codec, imgs, excess_state_len=N_INIT, edges=edges, chain_blocks=L)
            assert all(a.dtype == b.dtype and np.array_equal(a, b) for a, b in zip(plain, got)), (edges, L)
    # an image of at most L blocks keeps the reference layout next to an image that is split
    mixed = compress_images(codec, images, excess_state_len=N_INIT, edges="code", chain_blocks=6)
    assert len(chains_of(unpack_container(mixed[0]))) == 2 and np.array_equal(mixed[1], plain[1]) and np.array_equal(mixed[2], plain[2])


@pytest.mark.parametrize("scheme", [BITSWAP, BBANS])
def test_more_chains_than_max_batch(scheme):
    """24 chains through a codec of max_batch 8 (three calls per step) write the containers a codec of max_batch 24 writes
    (one call per step); so does a free-running 4-lane PipelinedCodec of max_batch 8, whose lanes must see every stream
    at the same lane at every step."""
    cfg, m, sd, zend, zcen, bins, big = setup("tiny3", 24)
    images = random_images(3, [(150, 390), (33, 65)], seed=41)                 # 5 x 13 and 2 x 3 blocks, edge-coded
    small = BitSwapCodec(cfg, m, bins, 8)
    pc = PipelinedCodec(cfg, sd, bins, 8, lanes=4, use_tensor_cores=False, free_running=True)
    kw = dict(excess_state_len=N_INIT, scheme=scheme, edges="code", chain_blocks=3)
    want = compress_images(big, images, **kw)
    assert [[nb for _, _, nb in chains_of(unpack_container(c))] for c in want] == [[3] * 21 + [2], [3, 3]]   # 24 streams, 23 at the last step
    for codec in (small, pc):
        got = compress_images(codec, images, **kw)
        assert all(np.array_equal(a, b) for a, b in zip(want, got))
        back = decompress_images(codec, got, scheme=scheme)
        assert all(np.array_equal(a, b) for a, b in zip(images, back))


def test_one_call_decodes_single_and_multi_chain_containers():
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", 12)
    images = random_images(3, [(100, 70), (20, 20), (64, 96), (130, 33)], seed=43)
    single = compress_images(codec, images, excess_state_len=N_INIT, edges="code")
    multi = compress_images(codec, images, excess_state_len=N_INIT, edges="code", chain_blocks=3)
    assert [len(chains_of(unpack_container(c))) for c in multi] == [4, 1, 2, 4]
    mix = [multi[0], single[1], single[2], multi[2], multi[3], single[0]]
    back = decompress_images(codec, mix)
    for rec, img in zip(back, [images[0], images[1], images[2], images[2], images[3], images[0]]):
        assert np.array_equal(rec, img)


def test_imagenetcrop4_tensor_cores_each_chain_equals_a_lone_chain():
    """The config-5 model on tensor cores through a free-running 2-lane PipelinedCodec: chain k of an edge-coded image
    holds exactly what a lone single-chain encode of its blocks leaves, and the containers round-trip."""
    cfg = preset("imagenetcrop4")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
    pc = PipelinedCodec(cfg, sd, bins, 8, lanes=2, use_tensor_cores=True, free_running=True)
    images = random_images(3, [(100, 130), (64, 31)], seed=47)                  # 4 x 5 and 2 x 1 blocks
    conts = compress_images(pc, images, excess_state_len=4000, edges="code", chain_blocks=6)
    back = decompress_images(pc, conts)
    assert all(np.array_equal(a, b) for a, b in zip(images, back))
    blocks, ext = _tiles(images[0], "code")
    chains = chains_of(unpack_container(conts[0]))
    assert [nb for _, _, nb in chains] == [5, 5, 5, 5]
    s = 0
    for ws, hd, nb in chains:
        lw, lh = lone_chain(pc, blocks[s:s + nb], ext[s:s + nb], BITSWAP)
        assert np.array_equal(ws, lw) and hd == lh, s
        s += nb
    assert np.array_equal(conts[1], compress_images(pc, images[1:], excess_state_len=4000, edges="code")[0])
