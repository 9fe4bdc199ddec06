"""Archives of many images whose chains run across images, without a GPU: the chain runs over the global block sequence,
the archive layout and every check of its parser, and the decode plan against a brute force."""
import types

import numpy as np
import pytest

from codec_harness import NoDevice
from bitswap_b200 import container
from bitswap_b200.codec import BBANS, BITSWAP
from bitswap_b200.container import (ARCHIVE_MARK, CHAIN_MARK, MAX_BLOCKS, block_grid, chain_sizes, compress_archive,
                                    decompress_archive, extract_edge_blocks, pack_archive, plan_archive, unpack_archive,
                                    unpack_container)


def _blocks(h, w):
    return int(np.prod(block_grid(h, w)))


def _archive(shapes, L, seed=0, n_init=3000, s=100, scheme=BITSWAP):
    """An archive whose tables describe images of the given (h, w) coded as chain_sizes(total, L) (the words are random:
    only the parser and the plan read it)."""
    rs = np.random.RandomState(seed)
    sizes = chain_sizes(sum(_blocks(h, w) for h, w in shapes), L)
    chains = [(rs.randint(0, 1 << 32, rs.randint(0, 30), dtype=np.uint64).astype(np.uint32),
               int(rs.randint(1 << 32, 1 << 63, dtype=np.uint64)), nb) for nb in sizes]
    return pack_archive(chains, shapes, n_init, s, scheme), chains


def _recording(monkeypatch):
    """compress_archive on a codec stub: the encoder records the block sequence and chains it is given and returns empty
    chains, so the split and the layout are checked without a device."""
    seen = {}

    def fake(codec, blocks, extents, chains, scheme, n_init, seed, wpb):
        seen.update(blocks=blocks, extents=extents, chains=chains)
        return [(np.zeros(0, np.uint32), 5, nb) for _, nb in chains]
    monkeypatch.setattr(container, "_encode", fake)
    return seen, types.SimpleNamespace(cfg=types.SimpleNamespace(xs=[3]))


@pytest.mark.parametrize("L", [None, 1, 3, 7, 16, 64])
def test_chains_run_over_the_global_block_sequence(L, monkeypatch):
    seen, codec = _recording(monkeypatch)
    rs = np.random.RandomState(1)
    shapes = [(1, 1), (100, 70), (28, 28), (33, 65), (32, 32), (64, 31)]               # 1, 12, 1, 6, 1, 2 blocks
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    a = compress_archive(codec, images, chain_blocks=L)
    total = sum(_blocks(h, w) for h, w in shapes)
    sizes = chain_sizes(total, L)
    assert [nb for _, nb in seen["chains"]] == sizes
    assert max(sizes) - min(sizes) <= 1 and sizes == sorted(sizes, reverse=True)
    assert [s for s, _ in seen["chains"]] == (np.cumsum(sizes) - sizes).tolist()
    # the sequence is every image's edge-coded blocks in turn, in the model's CHW layout
    tiles = [extract_edge_blocks(im) for im in images]
    assert np.array_equal(seen["blocks"], np.concatenate([t[0] for t in tiles]).transpose(0, 3, 1, 2))
    assert np.array_equal(seen["extents"], np.concatenate([t[1] for t in tiles]))
    ends = set(np.cumsum([_blocks(h, w) for h, w in shapes]).tolist())
    if L in (3, 7):                                                                    # some chain crosses an image boundary
        assert any(not {s + d for d in range(1, nb)}.isdisjoint(ends) for s, nb in seen["chains"])
    _, _, _, nblocks, got, n_init, seed, scheme = unpack_archive(a)
    assert nblocks.tolist() == sizes and got.tolist() == [list(s) for s in shapes] and (n_init, seed, scheme) == (10000, 100, 0)


@pytest.mark.parametrize("shapes,L", [([(1, 1)], None), ([(100, 70), (28, 28)], 3), ([(28, 28)] * 50, 16),
                                      ([(2048, 1536), (1, 700)], 64), ([(5, 5)] * 3, 1)])
def test_writer_and_parser_round_trip(shapes, L):
    a, chains = _archive(shapes, L, seed=len(shapes), n_init=77, s=12345, scheme=BBANS)
    assert a.dtype == np.uint32 and a.ndim == 1 and a[-1] == ARCHIVE_MARK
    K, N = len(chains), len(shapes)
    assert a.tolist()[-6:] == [K, N, 77, 12345, BBANS, ARCHIVE_MARK]
    assert len(a) == sum(len(c[0]) for c in chains) + 4 * K + 2 * N + 6
    words, offs, heads, nblocks, got, n_init, seed, scheme = unpack_archive(a)
    assert got.tolist() == [list(s) for s in shapes] and (n_init, seed, scheme) == (77, 12345, BBANS)
    for k, (ws, hd, nb) in enumerate(chains):
        assert np.array_equal(words[offs[k]:offs[k + 1]], ws) and int(heads[k]) == hd and int(nblocks[k]) == nb


def _tweak(a, pos, value):
    a = a.copy()
    a[pos] = value
    return a


def _malformed():
    shapes = [(64, 96), (1, 1), (33, 40)]                                              # 6 + 1 + 4 blocks
    good, chains = _archive(shapes, 3)                                                 # chains of 3, 3, 3, 2
    K, N = len(chains), len(shapes)
    tbl = len(good) - 6 - 2 * N - 4 * K
    shp = len(good) - 6 - 2 * N

    def field(k, f):
        return tbl + 4 * k + f
    big = pack_archive([(np.zeros(0, np.uint32), 1, 1 << 20)] * 17, [(32 << 10, 32 << 10)] * 17, 10, 0, 0)
    return good, [
        good[:5], np.zeros(0, np.uint32), good[-6:], good[1:], np.concatenate([[5], good]).astype(np.uint32),
        _tweak(good, -1, CHAIN_MARK), _tweak(good, -1, 0),                             # not the mark
        _tweak(good, -6, 0), _tweak(good, -5, 0),                                      # K = 0, N = 0
        _tweak(good, -6, 1 << 30), _tweak(good, -5, 1 << 31),                          # tables beyond the length
        _tweak(good, shp, 0), _tweak(good, shp + 3, 0),                                # h = 0, w = 0
        _tweak(good, shp, 32 << 10), _tweak(_tweak(good, shp, 32 << 11), shp + 1, 32 << 10),   # > MAX_BLOCKS blocks
        _tweak(good, field(1, 3), 2), _tweak(good, field(3, 3), 3),                    # chains hold 10, 12 blocks
        _tweak(good, shp + 3, 40),                                                     # images hold 12 blocks
        _tweak(_tweak(good, field(3, 3), 0), field(0, 3), 5),                          # a chain of no blocks
        _tweak(good, field(0, 0), good[field(0, 0)] + 1),                              # words claimed > words held
        _tweak(good, field(0, 0), good[field(0, 0)] - 1) if good[field(0, 0)] else _tweak(good, field(1, 0), 1 << 20),
        _tweak(good, -4, 1), _tweak(good, -4, 0), _tweak(good, -4, (1 << 24) + 1),     # excess_state_len
        _tweak(good, -2, 2), _tweak(good, -2, 1 << 31),                                # scheme
        big,                                                                           # consistent, > 2^24 blocks
        np.zeros((2, 8), np.uint32)]


def test_malformed_archives_are_refused_before_any_device_work():
    good, bad = _malformed()
    assert len(plan_archive(good).first) == 4
    for a in bad:
        with pytest.raises(ValueError):
            unpack_archive(a)
        with pytest.raises(ValueError):
            plan_archive(a)
        with pytest.raises(ValueError):
            decompress_archive(NoDevice(), a)
    with pytest.raises(AssertionError, match="touched"):                              # well-formed: then the codec is needed
        decompress_archive(NoDevice(), good)
    assert unpack_archive(_tweak(good, -4, 2))[5] == 2 and unpack_archive(_tweak(good, -4, 1 << 24))[5] == 1 << 24


@pytest.mark.parametrize("shapes,L", [([(1, 1)], None), ([(100, 70), (28, 28)], 3), ([(28, 28)] * 40, 16),
                                      ([(2048, 1536)], 64), ([(2048, 1536)], None)])
@pytest.mark.parametrize("scheme", [BITSWAP, BBANS])
def test_unpack_container_refuses_an_archive(shapes, L, scheme):
    a = _archive(shapes, L, scheme=scheme)[0]
    assert int(a[-1]) != CHAIN_MARK
    nblocks, h, w = (int(v) for v in a[-3:])                                           # read as a reference tail
    assert w >= 1 << 31 and (h == 0 or np.prod(block_grid(h, w)) > MAX_BLOCKS)        # h is the scheme
    with pytest.raises(ValueError):
        unpack_container(a)


def _brute(shapes, sizes, regions):
    """(first, depth, needed) by walking every pixel of every region."""
    offs = np.cumsum([0] + [_blocks(h, w) for h, w in shapes])
    needed = np.zeros(offs[-1], bool)
    for i, y, x, h, w in regions:
        gw = block_grid(*shapes[i])[1]
        for yy in range(y, y + h):
            for xx in range(x, x + w):
                needed[offs[i] + yy // 32 * gw + xx // 32] = True
    first, s = [], 0
    for nb in sizes:
        hit = np.flatnonzero(needed[s:s + nb])
        first.append(int(hit[0]) if hit.size else nb)
        s += nb
    return first, [nb - f for nb, f in zip(sizes, first)], needed


def test_plan_archive_matches_a_brute_force():
    rs = np.random.RandomState(5)
    for trial in range(12):
        n = rs.randint(1, 9)
        shapes = [(1, 1) if rs.rand() < 0.2 else (int(rs.randint(1, 130)), int(rs.randint(1, 130))) for _ in range(n)]
        L = [None, 1, 2, 3, 5, 7][trial % 6]
        a = _archive(shapes, L, seed=trial)[0]
        sizes = chain_sizes(sum(_blocks(h, w) for h, w in shapes), L)
        regions = [(0, 0, 0, 1, 1), (n - 1, shapes[-1][0] - 1, shapes[-1][1] - 1, 1, 1)]   # the first and last images
        for _ in range(rs.randint(0, 5)):
            i = rs.randint(n)
            h, w = shapes[i]
            bh, bw = rs.randint(1, h + 1), rs.randint(1, w + 1)
            regions.append((i, rs.randint(0, h - bh + 1), rs.randint(0, w - bw + 1), bh, bw))
        for rg in (regions, regions[1:], regions[2:] or [(0, 0, 0) + shapes[0]]):
            p = plan_archive(a, rg)
            first, depth, needed = _brute(shapes, sizes, rg)
            assert p.first.tolist() == first and p.depth.tolist() == depth and np.array_equal(p.needed, needed), (trial, rg)
        p = plan_archive(a)                                                            # None: every image, every chain whole
        assert p.first.tolist() == [0] * len(sizes) and p.depth.tolist() == sizes and p.needed.all()


def test_an_image_straddling_two_chains():
    # images of 6, 1, 4 blocks as chains 3, 3, 3, 2 over blocks [0..2], [3..5], [6..8], [9, 10]
    a = _archive([(64, 96), (1, 1), (33, 40)], 3)[0]
    assert plan_archive(a, [(1, 0, 0, 1, 1)]).depth.tolist() == [0, 0, 3, 0]          # the one-block image: chain 2 whole
    p = plan_archive(a, [(2, 0, 0, 1, 1)])                                             # image 2's first block is block 7
    assert p.first.tolist() == [3, 3, 1, 2] and p.depth.tolist() == [0, 0, 2, 0]
    p = plan_archive(a, [(2, 0, 0, 33, 40)])                                           # blocks 7..10: a chain and a bit
    assert p.first.tolist() == [3, 3, 1, 0] and p.depth.tolist() == [0, 0, 2, 2]
    p = plan_archive(a, [(0, 32, 64, 1, 1)])                                           # image 0's last block: block 5
    assert p.first.tolist() == [3, 2, 3, 2] and p.depth.tolist() == [0, 1, 0, 0]


@pytest.mark.parametrize("region", [
    (0, 0, 0, 0, 10), (0, 0, 0, 10, 0), (0, 0, 0, -1, 10),                            # empty
    (0, 0, 0, 65, 10), (0, 0, 0, 10, 97), (0, 60, 0, 5, 1), (0, 0, 90, 1, 7),         # past the bottom or the right
    (0, -1, 0, 1, 1), (0, 0, -1, 1, 1),                                               # before the top or the left
    (0, 0.0, 0, 1, 1), (0, 0, 0, 1.5, 1), (0, "0", 0, 1, 1), (True, 0, 0, 1, 1), (0, 0, 0, 1, None),   # not ints
    (3, 0, 0, 1, 1), (-1, 0, 0, 1, 1), (7, 0, 0, 1, 1),                               # no such image
    (1, 0, 0, 1, 2), (0, 0, 0, 1), (0, 0, 0, 1, 1, 1), 5, None])                      # off the 1 x 1 image; not five
def test_invalid_regions_are_refused_before_any_device_work(region):
    a = _archive([(64, 96), (1, 1), (33, 40)], 3)[0]
    with pytest.raises(ValueError):
        plan_archive(a, [(2, 0, 0, 33, 40), region])
    with pytest.raises(ValueError):
        decompress_archive(NoDevice(), a, [(2, 0, 0, 33, 40), region])


def test_good_regions_reach_the_codec():
    a = _archive([(64, 96), (1, 1), (33, 40)], 3)[0]
    for regions in (None, [(1, 0, 0, 1, 1)], [(np.int64(2), np.int32(0), 0, 33, 40)], [np.array([0, 0, 0, 64, 96])]):
        with pytest.raises(AssertionError, match="touched"):
            decompress_archive(NoDevice(), a, regions)
    assert decompress_archive(NoDevice(), a, []) == []


@pytest.mark.parametrize("kw", [dict(chain_blocks=0), dict(chain_blocks=2.0), dict(scheme=2), dict(excess_state_len=1),
                                dict(excess_state_len=(1 << 24) + 1), dict(seed=-1), dict(seed=1 << 32), dict(seed=1.0)])
def test_compress_archive_arguments_are_checked_before_any_device_work(kw):
    with pytest.raises(ValueError):
        compress_archive(NoDevice(), [np.zeros((4, 4, 3), np.uint8)], **kw)


@pytest.mark.parametrize("images", [[], [np.zeros((4, 4, 1), np.uint8)], [np.zeros((4, 4), np.uint8)],
                                    [np.zeros((0, 4, 3), np.uint8)], [np.zeros((4, 4, 3), np.float32)],
                                    [np.zeros((4, 4, 3), np.uint8), np.zeros((4, 0, 3), np.uint8)]])
def test_bad_images_are_refused_before_the_encoder(images, monkeypatch):
    seen, codec = _recording(monkeypatch)
    with pytest.raises(ValueError):
        compress_archive(codec, images)
    assert not seen
