"""Archives on the GPU: exact round trips, every chain against the oracle's demo procedure on its run of the global block
sequence (across image boundaries), a one-image archive against compress_images, region decodes against crops of the
full decode with exactly the planned pops, and the initial-state check."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from codec_harness import Counting, chains_of, gpu_oracle, lone_chain, oracle_chain, random_images, setup   # noqa: E402
from bitswap_b200 import container, synthetic                              # noqa: E402
from bitswap_b200.config import preset                                     # noqa: E402
from bitswap_b200.model import Model                                       # noqa: E402
from bitswap_b200.codec import BitSwapCodec, Bins, PipelinedCodec, BITSWAP, BBANS   # noqa: E402
from bitswap_b200.container import (chain_sizes, compress_archive, compress_images, decompress_archive,   # noqa: E402
                                    extract_edge_blocks, plan_archive, unpack_archive, unpack_container)

N_INIT = 3000
SIZES = [(1, 1), (100, 70), (28, 28), (33, 65), (5, 40), (64, 31)]          # 1 + 12 + 1 + 6 + 2 + 2 = 24 blocks


def _sequence(images):
    """(blocks [n, 32, 32, C], extents [n, 2]) of the archive's global block sequence."""
    tiles = [extract_edge_blocks(im) for im in images]
    return np.concatenate([t[0] for t in tiles]), np.concatenate([t[1] for t in tiles])


def _planned_calls(plan, max_batch):
    return sum(-(-n // max_batch) for n in container._active(sorted([d for d in plan.depth.tolist() if d], reverse=True)))


@pytest.mark.parametrize("name,scheme", [("tiny", BITSWAP), ("tiny", BBANS), ("tiny3", BITSWAP), ("tiny3", BBANS)])
def test_round_trips_and_every_chain_equals_the_oracle(name, scheme):
    cfg, m, sd, zend, zcen, bins, codec = setup(name, 16)
    images = random_images(cfg.xs[0], SIZES, seed=71)
    blocks, ext = _sequence(images)
    orc = gpu_oracle(cfg, m, sd, zend, zcen)
    for L in (None, 1, 3, 7):
        a = compress_archive(codec, images, chain_blocks=L, scheme=scheme, excess_state_len=N_INIT)
        back = decompress_archive(codec, a)
        assert len(back) == len(images)
        assert all(b.shape == im.shape and np.array_equal(b, im) for b, im in zip(back, images)), L
        chains = chains_of(unpack_archive(a))
        assert [nb for _, _, nb in chains] == chain_sizes(len(blocks), L)
        s = 0
        for k, (ws, hd, nb) in enumerate(chains):
            ow, oh = oracle_chain(orc, blocks[s:s + nb], ext[s:s + nb], scheme)
            assert np.array_equal(ws, ow) and hd == oh, (L, k)
            s += nb


@pytest.mark.parametrize("L", [None, 1, 4, 5])
def test_an_archive_of_one_image_holds_the_containers_chains(L):
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", 8)
    img = random_images(3, [(100, 130)], seed=73)                                     # 4 x 5 blocks
    a = compress_archive(codec, img, chain_blocks=L, excess_state_len=N_INIT)
    (c,) = compress_images(codec, img, excess_state_len=N_INIT, edges="code", chain_blocks=L)
    want = chains_of(unpack_container(c))
    got = chains_of(unpack_archive(a))
    assert len(got) == len(want) and all(np.array_equal(g[0], w[0]) and g[1:] == w[1:] for g, w in zip(got, want))


def test_regions_equal_crops_of_the_full_decode_with_the_planned_pops():
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny", 8)
    images = random_images(1, SIZES + [(90, 40), (1, 100)], seed=75)
    rs = np.random.RandomState(76)
    for L in (None, 3, 5):
        a = compress_archive(codec, images, chain_blocks=L, scheme=BBANS, excess_state_len=N_INIT)
        full = decompress_archive(codec, a)
        n = len(images)
        singles = [[(i, 0, 0) + images[i].shape[:2]] for i in range(n)]
        windows = []
        for _ in range(6):
            i = rs.randint(n)
            h, w = images[i].shape[:2]
            bh, bw = rs.randint(1, h + 1), rs.randint(1, w + 1)
            windows.append((i, rs.randint(0, h - bh + 1), rs.randint(0, w - bw + 1), bh, bw))
        repeated = [windows[0], windows[0], (1, 0, 0, 100, 70), (1, 40, 30, 60, 40), (n - 1, 0, 99, 1, 1), (0, 0, 0, 1, 1)]
        for regions in singles + [[r] for r in windows] + [windows, repeated]:
            counting = Counting(codec)
            got = decompress_archive(counting, a, regions)
            assert len(got) == len(regions)
            for (i, y, x, h, w), g in zip(regions, got):
                want = full[i][y:y + h, x:x + w]
                assert g.dtype == np.uint8 and g.flags.c_contiguous and np.array_equal(g, want), (L, i, y, x, h, w)
            plan = plan_archive(a, regions)
            assert counting.blocks == int(plan.depth.sum()), (L, regions)
            assert counting.calls == _planned_calls(plan, codec.max_batch), (L, regions)


@pytest.mark.parametrize("scheme", [BITSWAP, BBANS])
def test_more_chains_than_max_batch_and_a_free_running_pipelined_codec(scheme):
    """25 chains through max_batch 24 (two calls per step), max_batch 8 (four) and a free-running 2-lane PipelinedCodec of
    max_batch 8 write the same archive and decode it exactly."""
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", 24)
    images = random_images(3, [(150, 390), (33, 65), (1, 1), (28, 28)], seed=77)       # 65 + 6 + 1 + 1 = 73 blocks
    kw = dict(chain_blocks=3, scheme=scheme, excess_state_len=N_INIT)
    want = compress_archive(codec, images, **kw)
    assert len(chains_of(unpack_archive(want))) == 25
    pc = PipelinedCodec(cfg, sd, bins, 8, lanes=2, use_tensor_cores=False, free_running=True)
    for codec in (BitSwapCodec(cfg, m, bins, 8), pc):
        got = compress_archive(codec, images, **kw)
        assert np.array_equal(got, want)
        assert all(np.array_equal(a, b) for a, b in zip(decompress_archive(codec, got), images))
        counting = Counting(codec)
        regions = [(0, 100, 300, 50, 90), (3, 0, 0, 28, 28), (1, 10, 10, 1, 1)]
        got_r = decompress_archive(counting, got, regions)
        assert all(np.array_equal(g, images[i][y:y + h, x:x + w]) for (i, y, x, h, w), g in zip(regions, got_r))
        assert counting.blocks == int(plan_archive(got, regions).depth.sum())


def test_imagenetcrop4_tensor_cores_each_chain_equals_a_lone_chain():
    cfg = preset("imagenetcrop4")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
    pc = PipelinedCodec(cfg, sd, bins, 8, lanes=2, use_tensor_cores=True, free_running=True)
    rs = np.random.RandomState(79)
    sizes = [(int(rs.randint(1, 70)), int(rs.randint(1, 70))) for _ in range(30)]
    images = random_images(3, sizes, seed=80)
    blocks, ext = _sequence(images)
    a = compress_archive(pc, images, chain_blocks=8, excess_state_len=4000)
    back = decompress_archive(pc, a)
    assert all(np.array_equal(b, im) for b, im in zip(back, images))
    chains = chains_of(unpack_archive(a))
    assert [nb for _, _, nb in chains] == chain_sizes(len(blocks), 8) and len(chains) >= 4
    s = 0
    for k, (ws, hd, nb) in enumerate(chains):
        lw, lh = lone_chain(pc, blocks[s:s + nb], ext[s:s + nb], BITSWAP)
        assert np.array_equal(ws, lw) and hd == lh, k
        s += nb


def _flip_head_lo(a, k):
    """The archive with bit 0 of chain k's head_lo flipped."""
    K, N = int(a[-6]), int(a[-5])
    a = a.copy()
    a[len(a) - 6 - 2 * N - 4 * K + 4 * k + 1] ^= 1
    return a


def test_the_initial_state_check():
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny3", 8)
    images = random_images(3, SIZES, seed=81)
    a = compress_archive(codec, images, chain_blocks=5, excess_state_len=N_INIT)     # 24 blocks: chains of 5, 5, 5, 5, 4
    assert [nb for _, _, nb in chains_of(unpack_archive(a))] == [5, 5, 5, 5, 4]
    # a codec built from other weights decodes other symbols: a chain does not come back to its initial state (or, checked
    # first, the stream flags report a pop past its stack or a symbol outside its table)
    sd51 = synthetic.synthetic_state_dict(cfg, seed=51, varied=True)
    m51 = Model.from_config(cfg, max_batch=8, use_tensor_cores=False).load_state_dict(sd51)
    m51.compress()
    with pytest.raises((ValueError, IndexError)):
        decompress_archive(BitSwapCodec(cfg, m51, bins, 8), a)
    # a corrupt head names its chain, whole or through a region that reaches the chain's first block
    for k in (0, 2, 4):
        bad = _flip_head_lo(a, k)
        with pytest.raises(ValueError, match=f"chain {k} "):
            decompress_archive(codec, bad)
        first_block = 5 * k                                                    # the chain's first block in the sequence
        with pytest.raises(ValueError, match=f"chain {k} "):
            decompress_archive(codec, bad, [_region_of_block(images, first_block)])
    # a region decode that leaves the corrupt chain partly popped does not check it: the last block of chain 2 (block 14,
    # image 3's first block) is reached by popping one block
    assert _region_of_block(images, 14) == (3, 0, 0, 1, 1) and _region_of_block(images, 10) == (1, 96, 0, 1, 1)
    plan = plan_archive(a, [(3, 0, 0, 1, 1)])
    assert plan.depth.tolist() == [0, 0, 1, 0, 0]
    got = decompress_archive(codec, _flip_head_lo(a, 2), [(3, 0, 0, 1, 1)])
    assert got[0].shape == (1, 1, 3)
    assert np.array_equal(decompress_archive(codec, a, [(3, 0, 0, 1, 1)])[0], images[3][:1, :1])


def _region_of_block(images, b):
    """The top-left pixel of block b of the global sequence, as a region."""
    for i, im in enumerate(images):
        gh, gw = -(-im.shape[0] // 32), -(-im.shape[1] // 32)
        if b < gh * gw:
            return (i, 32 * (b // gw), 32 * (b % gw), 1, 1)
        b -= gh * gw
    raise IndexError(b)
