"""Images coded as several chains, without a GPU: the split policy, the multi-chain container layout and its checks."""
import numpy as np
import pytest

from bitswap_b200.container import (CHAIN_MARK, block_grid, chain_sizes, compress_images, decompress_images, pack_container,
                                    unpack_container)


@pytest.mark.parametrize("n", [1, 2, 3, 7, 16, 49, 100, 256, 3072, 11750])
@pytest.mark.parametrize("L", [1, 2, 3, 7, 16, 32, 64, 5000])
def test_split_policy(n, L):
    sizes = chain_sizes(n, L)
    assert len(sizes) == -(-n // L) and sum(sizes) == n
    assert max(sizes) - min(sizes) <= 1 and sizes == sorted(sizes, reverse=True) and min(sizes) >= 1
    assert max(sizes) <= L
    assert chain_sizes(n, None) == [n] and chain_sizes(n, n) == [n]


def _chains(rs, sizes):
    return [(rs.randint(0, 1 << 32, rs.randint(0, 40), dtype=np.uint64).astype(np.uint32),
             int(rs.randint(1 << 32, 1 << 63, dtype=np.uint64)), nb) for nb in sizes]


@pytest.mark.parametrize("h,w,L", [(64, 96, 1), (64, 96, 4), (100, 70, 3), (33, 1, 1), (225, 224, 7), (2048, 1536, 32)])
def test_writer_and_parser_round_trip(h, w, L):
    rs = np.random.RandomState(h * 7 + w + L)
    n = int(np.prod(block_grid(h, w)))
    chains = _chains(rs, chain_sizes(n, L))
    c = pack_container(chains, h, w)
    assert c.dtype == np.uint32 and c.ndim == 1
    words, offs, heads, nblocks, hh, ww = unpack_container(c)
    assert (hh, ww) == (h, w) and len(heads) == len(chains)
    for k, (ws, hd, nb) in enumerate(chains):
        assert np.array_equal(words[offs[k]:offs[k + 1]], ws) and int(heads[k]) == hd and int(nblocks[k]) == nb
    if len(chains) == 1:                                        # the reference layout, word for word
        ws, hd, nb = chains[0]
        assert np.array_equal(c, np.concatenate([ws, np.array([hd & 0xffffffff, hd >> 32, nb, h, w], np.uint32)]))
    else:
        K = len(chains)
        assert c[-1] == CHAIN_MARK and list(c[-4:-1]) == [K, h, w] and len(c) == sum(len(x[0]) for x in chains) + 4 * K + 4


def _multi(h=64, w=96, sizes=(2, 2, 1, 1), seed=0):
    return pack_container(_chains(np.random.RandomState(seed), sizes), h, w)


def _tweak(c, pos, value):
    c = c.copy()
    c[pos] = value
    return c


def _table(c, k, field):
    """Index of field (0 nwords, 1 head_lo, 2 head_hi, 3 nblocks) of chain k in the table of container c."""
    K = int(c[-4])
    return len(c) - 4 * K - 4 + 4 * k + field


def test_malformed_multi_chain_tails_are_rejected_before_any_device_work():
    """Every inconsistent trailer is a ValueError while the headers are parsed, before a stream set is sized from them (so
    no codec is needed); good containers, single- and multi-chain, get past parsing and only then need the codec."""
    chains = [(np.arange(5, dtype=np.uint32), 1 << 40, 2), (np.arange(3, dtype=np.uint32), 7, 2),
              (np.zeros(0, np.uint32), 9, 1), (np.arange(4, dtype=np.uint32), 11 << 32, 1)]
    good = pack_container(chains, 64, 96)                           # 2 x 3 blocks as 2 + 2 + 1 + 1
    single = np.array([7, 7, 1, 0, 6, 64, 96], np.uint32)
    nw0 = _table(good, 0, 0)
    bad = [good[-11:],                                              # too short for its own table
           _tweak(good, -4, 1),                                     # K = 1 in the multi-chain layout
           _tweak(good, -4, 0),
           _tweak(good, -4, 1 << 30),                               # K far beyond the length
           np.array([0] * 12 + [3, 64, 96, CHAIN_MARK], np.uint32), # chains of no blocks
           _tweak(good, _table(good, 2, 3), 0),                     # one chain with no blocks
           _tweak(good, _table(good, 2, 3), 2),                     # nblocks sum to 7, 64 x 96 has 6
           _tweak(good, -3, 96),                                    # h: 96 x 96 has 9 blocks
           _tweak(good, -3, 0),                                     # empty image
           _tweak(good, -2, 100),                                   # 64 x 100 has 8 blocks
           _tweak(good, nw0, 6),                                    # words claimed > words held
           _tweak(good, nw0, 4),                                    # words claimed < words held
           np.concatenate([[5], good]).astype(np.uint32),           # one stray word
           good[1:],                                                # one word missing
           pack_container([(np.zeros(0, np.uint32), 1, 1)] * 3, 32, 64),        # 3 chains of one block, 2 blocks
           pack_container([(np.zeros(0, np.uint32), 1, 1 << 20)] * 3, 32 << 11, 32 << 10)]   # consistent, absurdly large
    for c in bad:
        with pytest.raises(ValueError):
            decompress_images(None, [good, single, c])
    with pytest.raises(AttributeError):                             # well-formed: parsing passes, then the codec is needed
        decompress_images(None, [good, single])
    # the HWC quirk rules hold for multi-chain containers too: whole blocks only
    with pytest.raises(ValueError):
        decompress_images(None, [_multi(40, 96, (2, 2, 1, 1))], hwc_quirk=True)
    with pytest.raises(AttributeError):
        decompress_images(None, [good], hwc_quirk=True)


def test_single_chain_tails_are_still_rejected():
    """The single-chain rules are untouched: the tails the container tests reject stay rejected, next to a multi-chain
    container."""
    good = _multi()
    for c in [np.zeros(4, np.uint32), np.array([7, 7, 1, 0, 5, 64, 96], np.uint32), np.array([7, 7, 1, 0, 6, 64, 100], np.uint32),
              np.array([7, 7, 1, 0, 0, 0, 96], np.uint32), np.array([7, 7, 1, 0, 1 << 21, 32 << 11, 32 << 10], np.uint32),
              np.zeros((2, 8), np.uint32), np.array([1, 0, 1, 33, 1], np.uint32)]:
        with pytest.raises(ValueError):
            decompress_images(None, [good, c])


@pytest.mark.parametrize("h,w,sizes", [(64, 96, (2, 2, 1, 1)), (33, 1, (1, 1)), (2048, 1536, (32,) * 96),
                                       (32 << 5, 32 << 5, (512, 512))])
def test_multi_chain_tail_fails_the_single_chain_header_rule(h, w, sizes):
    """Read as a reference-layout tail, the last five words of a multi-chain container give (nblocks, h, w) =
    (h, w, CHAIN_MARK): a width of 2^31 or more, whose block count no 32-bit nblocks matches."""
    c = _multi(h, w, sizes)
    nblocks, hh, ww = (int(v) for v in c[-3:])
    assert (nblocks, hh, ww) == (h, w, CHAIN_MARK)
    assert nblocks != np.prod(block_grid(hh, ww)) or nblocks > (1 << 20)
    assert np.prod(block_grid(hh, ww)) > (1 << 20)


@pytest.mark.parametrize("bad", [0, -1, -32, 1.0, 2.5, "16", True, False, [4]])
def test_chain_blocks_argument_is_checked_before_any_device_work(bad):
    img = np.zeros((64, 64, 3), np.uint8)
    with pytest.raises(ValueError):
        compress_images(None, [img], chain_blocks=bad)
    with pytest.raises(ValueError):
        compress_images(None, [img], edges="code", chain_blocks=bad)


def test_good_chain_blocks_get_past_the_checks():
    img = np.zeros((64, 64, 3), np.uint8)
    for ok in (None, 1, 3, np.int64(2), 10 ** 6):
        with pytest.raises(AttributeError):                         # only then is the codec needed
            compress_images(None, [img], chain_blocks=ok)
