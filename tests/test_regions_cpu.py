"""Decoding regions of containers, without a GPU: the plan (which chains, and how deep) against hand-computed chains, and
every invalid request refused before any device work."""
import numpy as np
import pytest

from codec_harness import NoDevice
from bitswap_b200.container import (block_grid, chain_sizes, decompress_images, decompress_regions, pack_container,
                                    plan_regions)


def _container(h, w, L=None, seed=0):
    """A container whose headers describe an h x w image coded as chain_sizes(blocks, L) (the words are random: only the
    plan reads it)."""
    rs = np.random.RandomState(seed)
    sizes = chain_sizes(int(np.prod(block_grid(h, w))), L)
    return pack_container([(rs.randint(0, 1 << 32, 5, dtype=np.uint64).astype(np.uint32), 12345, nb) for nb in sizes], h, w)


def _plan(h, w, L, boxes):
    (p,) = plan_regions([_container(h, w, L)], [(0,) + b for b in boxes])
    return p.first.tolist(), p.depth.tolist(), np.flatnonzero(p.needed).tolist()


def test_single_chain():
    # 64 x 96: 2 x 3 blocks, one chain of 6; decoding starts at block 5
    assert _plan(64, 96, None, [(0, 0, 64, 96)]) == ([0], [6], [0, 1, 2, 3, 4, 5])
    assert _plan(64, 96, None, [(63, 95, 1, 1)]) == ([5], [1], [5])               # bottom-right pixel
    assert _plan(64, 96, None, [(0, 0, 1, 1)]) == ([0], [6], [0])                 # top-left pixel: the whole chain
    assert _plan(64, 96, None, [(40, 31, 10, 2)]) == ([3], [3], [3, 4])           # straddles a block column
    assert _plan(64, 96, None, [(32, 64, 32, 32), (40, 40, 1, 1)]) == ([4], [2], [4, 5])


def test_multi_chain_edge_coded():
    # 100 x 70, edge-coded: 4 x 3 blocks, chain_blocks 5 -> chains of 4, 4, 4 blocks: [0..3], [4..7], [8..11]
    assert chain_sizes(12, 5) == [4, 4, 4]
    assert _plan(100, 70, 5, [(0, 0, 100, 70)]) == ([0, 0, 0], [4, 4, 4], list(range(12)))
    assert _plan(100, 70, 5, [(99, 69, 1, 1)]) == ([4, 4, 3], [0, 0, 1], [11])    # the partial corner block
    assert _plan(100, 70, 5, [(0, 0, 1, 1)]) == ([0, 4, 4], [4, 0, 0], [0])
    # rows 1-2, columns 1-2: blocks 4, 5, 7, 8 -> chain 0 skipped, chain 1 from its block 0, chain 2 from its block 0
    assert _plan(100, 70, 5, [(40, 40, 40, 30)]) == ([4, 0, 0], [0, 4, 4], [4, 5, 7, 8])
    # block 3 only (row 1, column 0): the last block of chain 0; one box straddling chains 0 and 1 (blocks 2 and 5)
    assert _plan(100, 70, 5, [(32, 0, 32, 32)]) == ([3, 4, 4], [1, 0, 0], [3])
    assert _plan(100, 70, 5, [(31, 64, 2, 6)]) == ([2, 1, 4], [2, 3, 0], [2, 5])
    # several boxes: the union, each chain to its earliest block
    assert _plan(100, 70, 5, [(99, 0, 1, 1), (0, 64, 1, 6), (50, 33, 1, 1)]) == ([2, 0, 1], [2, 4, 3], [2, 4, 9])


def test_crop_container_and_several_containers():
    # a crop-mode container of 128 x 160 (4 x 5 blocks), chain_blocks 3: 7 chains [3, 3, 3, 3, 3, 3, 2]
    c = _container(128, 160, 3)
    single = _container(33, 65)                                                    # 2 x 3 blocks, one chain
    plans = plan_regions([single, c, single], [(1, 96, 128, 32, 32), (1, 64, 0, 1, 160), (2, 0, 64, 1, 1)])
    assert [len(p.first) for p in plans] == [1, 7, 1]
    assert plans[0].depth.tolist() == [0] and plans[0].first.tolist() == [6] and not plans[0].needed.any()
    # blocks 10..14 (row 2) and 19 (the last): chains 3 (9..11), 4 (12..14), 6 (18, 19)
    assert plans[1].first.tolist() == [3, 3, 3, 1, 0, 3, 1]
    assert plans[1].depth.tolist() == [0, 0, 0, 2, 3, 0, 1]
    assert np.flatnonzero(plans[1].needed).tolist() == [10, 11, 12, 13, 14, 19]
    assert plans[2].first.tolist() == [2] and plans[2].depth.tolist() == [4]
    # plan_regions matches a brute force over every chain of random boxes
    rs = np.random.RandomState(3)
    for h, w, L in [(130, 97, 4), (2048, 1536, 32), (33, 1, None), (224, 225, 7)]:
        gh, gw = block_grid(h, w)
        sizes = chain_sizes(gh * gw, L)
        boxes = []
        for _ in range(3):
            bh, bw = rs.randint(1, h + 1), rs.randint(1, w + 1)
            boxes.append((rs.randint(0, h - bh + 1), rs.randint(0, w - bw + 1), bh, bw))
        want = np.zeros((gh, gw), bool)
        for y, x, bh, bw in boxes:
            for yy in range(y, y + bh):
                want[yy // 32, x // 32:(x + bw - 1) // 32 + 1] = True
        first, depth, needed = _plan(h, w, L, boxes)
        assert needed == np.flatnonzero(want).tolist()
        s = 0
        for k, nb in enumerate(sizes):
            hit = np.flatnonzero(want.reshape(-1)[s:s + nb])
            assert first[k] == (hit[0] if hit.size else nb) and depth[k] == nb - first[k]
            s += nb


@pytest.mark.parametrize("region", [
    (0, 0, 0, 0, 10), (0, 0, 0, 10, 0), (0, 0, 0, -1, 10),                        # empty
    (0, 0, 0, 65, 10), (0, 0, 0, 10, 97), (0, 60, 0, 5, 1), (0, 0, 90, 1, 7),     # past the bottom or the right
    (0, -1, 0, 1, 1), (0, 0, -1, 1, 1),                                           # before the top or the left
    (0, 0.0, 0, 1, 1), (0, 0, 0, 1.5, 1), (0, "0", 0, 1, 1), (True, 0, 0, 1, 1), (0, 0, 0, 1, None),   # not ints
    (2, 0, 0, 1, 1), (-1, 0, 0, 1, 1), (7, 0, 0, 1, 1),                            # no such container
    (0, 0, 0, 1), (0, 0, 0, 1, 1, 1), 5, None])                                     # not five fields
def test_invalid_regions_are_refused_before_any_device_work(region):
    conts = [_container(64, 96, 2), _container(100, 70)]
    with pytest.raises(ValueError):
        plan_regions(conts, [(1, 0, 0, 100, 70), region])
    with pytest.raises(ValueError):
        decompress_regions(NoDevice(), conts, [(1, 0, 0, 100, 70), region])


def test_malformed_containers_are_refused_before_any_device_work():
    good = _container(64, 96, 2)
    for bad in [np.zeros(4, np.uint32), np.array([7, 7, 1, 0, 5, 64, 96], np.uint32), good[1:]]:
        with pytest.raises(ValueError):
            plan_regions([good, bad], [(0, 0, 0, 1, 1)])
        with pytest.raises(ValueError):
            decompress_regions(NoDevice(), [good, bad], [(0, 0, 0, 1, 1)])
    with pytest.raises(ValueError):                                                # edge-coded: no hwc_quirk form
        decompress_regions(NoDevice(), [_container(100, 70)], [(0, 0, 0, 1, 1)], hwc_quirk=True)


def test_good_requests_reach_the_codec():
    conts = [_container(64, 96, 2), _container(100, 70)]
    for regions in ([(0, 63, 95, 1, 1)], [(np.int64(1), np.int32(0), 0, 100, 70)], [np.array([0, 0, 0, 64, 96])]):
        with pytest.raises(AssertionError, match="touched"):
            decompress_regions(NoDevice(), conts, regions)
    with pytest.raises(AssertionError, match="touched"):
        decompress_images(NoDevice(), conts)
    assert decompress_regions(NoDevice(), conts, []) == []
