"""Checked containers and archives without a GPU: the block digest definition pinned by known answers and a literal walk,
the check trailer through every writer and reader (with and without a stamp), every malformed trailer refused before any
device work, plans of checked arrays equal to the unchecked ones, and the C ABI's refusals of bad tables."""
import types

import numpy as np
import pytest

from checksum_harness import block_digest_scalar, block_digests, kernel_twin
from codec_harness import NoDevice
from bitswap_b200 import container
from bitswap_b200._lib import lib
from bitswap_b200.codec import BBANS, BITSWAP, Fingerprint
from bitswap_b200.container import (ARCHIVE_MARK, CHECK_MARK, CHECK_VERSION, STAMP_MARK, compress_archive,
                                    compress_images, decompress_archive, decompress_images, decompress_regions,
                                    plan_archive, plan_regions, read_stamp, unpack_archive, unpack_container)

BSW_E_INVALID = 4
FP = Fingerprint(1, 3, 8, 8, 1, 3, 8, 252, False, 10, True, "split", True, "reference",
                 "0123456789abcdef00112233445566ff", "fedcba98765432100f1e2d3c4b5a6978")


def _ramp(C):
    return (np.arange(C * 1024) % 251).astype(np.uint8).reshape(C, 32, 32)


def _random(C, seed):
    return np.random.RandomState(seed).randint(0, 256, (C, 32, 32)).astype(np.uint8)


# bsw_block_digest of these slots: pins the definition in include/bitswap_b200.h (the GPU tests hold the kernel to the twin)
KNOWN = {"zero C3": (np.zeros((3, 32, 32), np.uint8), 0, 32, 32, 0x35F90A2B),
         "ramp C3": (_ramp(3), 0, 32, 32, 0x8BB373DC),
         "ramp C3 block 7": (_ramp(3), 7, 32, 32, 0xF10F3B0F),
         "ramp C1 edge 5x17": (_ramp(1), 12, 5, 17, 0xBD91BD56),
         "random C4 edge 1x1": (_random(4, 1), 1 << 24, 1, 1, 0x4F7F3BE3)}


@pytest.mark.parametrize("case", sorted(KNOWN))
def test_block_digest_known_answers(case):
    slot, i, vh, vw, want = KNOWN[case]
    assert block_digest_scalar(slot, i, vh, vw) == want
    assert int(block_digests(slot[None], [i], [[vh, vw]])[0]) == want


EDGES = [(vh, vw) for vh in (1, 2, 16, 31, 32) for vw in (1, 2, 16, 31, 32)]


@pytest.mark.parametrize("C", [1, 2, 3, 4])
def test_vectorised_twin_walks_the_definition(C):
    slots = np.stack([np.zeros((C, 32, 32), np.uint8), _ramp(C)] + [_random(C, C * 100 + k) for k in range(len(EDGES))])
    ext = [(32, 32), (32, 32)] + EDGES
    index = [0, 5] + list(range(3, 3 + 7 * len(EDGES), 7))
    got = block_digests(slots, index, ext)
    assert got.dtype == np.uint32
    assert [int(v) for v in got] == [block_digest_scalar(s, i, vh, vw) for s, i, (vh, vw) in zip(slots, index, ext)]


def test_quirk_slots_are_full_extent_slots_in_slot_order():
    """A hwc_quirk slot holds the block's HWC bytes flat in the C*1024 bytes; its digest is the full-extent one of them."""
    hwc = np.random.RandomState(7).randint(0, 256, (32, 32, 3)).astype(np.uint8)
    slot = hwc.reshape(3, 32, 32)                                              # what the tile kernel stores
    assert int(block_digests(slot[None], [4])[0]) == block_digest_scalar(slot, 4, 32, 32)
    assert block_digest_scalar(slot, 4) != block_digest_scalar(hwc.transpose(2, 0, 1), 4)


@pytest.mark.parametrize("C,vh,vw", [(1, 32, 32), (3, 32, 32), (3, 17, 5), (2, 1, 32), (4, 32, 1)])
def test_one_flipped_byte_inside_the_extent_always_changes_the_digest(C, vh, vw):
    base = _random(C, 11 + vh + vw)
    pos = [(c, r, col) for c in range(C) for r in range(vh) for col in range(vw)]
    slots = np.repeat(base[None], len(pos), axis=0)
    for k, (c, r, col) in enumerate(pos):
        slots[k, c, r, col] ^= 1 << (k % 8)
    want = int(block_digests(base[None], [9], [[vh, vw]])[0])
    got = block_digests(slots, [9] * len(pos), [[vh, vw]] * len(pos))
    assert (got != want).all()


def test_bytes_outside_the_extent_are_not_read_and_the_seed_counts():
    base = _random(3, 21)
    other = base.copy()
    other[:, 20:, :] = 0
    other[:, :, 9:] = 255
    assert block_digest_scalar(base, 3, 20, 9) == block_digest_scalar(other, 3, 20, 9)
    seen = {block_digest_scalar(base, i, vh, vw) for i, vh, vw in [(3, 20, 9), (4, 20, 9), (3, 21, 9), (3, 20, 10),
                                                                    (1 << 20, 20, 9), (0, 20, 9)]}
    assert len(seen) == 6


def test_kernel_twin_seeds_each_block_with_its_index_in_its_own_sequence():
    rs = np.random.RandomState(2)
    x = rs.randint(0, 256, (3, 4, 1, 32, 32)).astype(np.uint8)
    block = np.array([[0, 5, 2, -1], [1, 4, -1, -1], [3, -1, -1, 6]])
    offs = np.array([0, 2, 2, 7])                                            # sequences of 2, 0 and 5 blocks
    out = kernel_twin(x, block, offs)
    for (t, j), g in np.ndenumerate(block):
        if g >= 0:
            i = g - (0 if g < 2 else 2)
            assert out[g] == block_digest_scalar(x[t, j], i)


# ---- writers and readers on a stand-in codec -------------------------------------------------------------------------------
def _fake_encoders(monkeypatch, seed=9):
    """Encoders that replay the same random chains and digests for every writer call (only the layout is checked)."""
    def chains(chains):
        rs = np.random.RandomState(seed)
        return [(rs.randint(0, 1 << 32, rs.randint(0, 40), dtype=np.uint64).astype(np.uint32),
                 int(rs.randint(1 << 32, 1 << 62, dtype=np.uint64)), nb) for _, nb in chains]

    def plain(codec, blocks, extents, ch, scheme, n_init, seed_, wpb):
        return chains(ch)

    def checked(codec, blocks, extents, ch, scheme, n_init, seed_, wpb, seq_offsets):
        total = int(seq_offsets[-1])
        return chains(ch), np.random.RandomState(seed + 1).randint(0, 1 << 32, total, dtype=np.uint64).astype(np.uint32)
    monkeypatch.setattr(container, "_encode", plain)
    monkeypatch.setattr(container, "_encode_checked", checked)
    return types.SimpleNamespace(cfg=types.SimpleNamespace(xs=[3]), fingerprint=lambda: FP)


def _images():
    rs = np.random.RandomState(4)
    return [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(64, 96), (33, 70), (32, 32), (100, 130)]]


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, np.ndarray):
            assert np.array_equal(x, y)
        else:
            assert x == y


def _nblocks(img, kw):
    h, w = img.shape[:2]
    return -(-h // 32) * -(-w // 32) if kw.get("edges") == "code" else (h // 32) * (w // 32)


@pytest.mark.parametrize("stamp", [False, True])
@pytest.mark.parametrize("kw", [dict(), dict(chain_blocks=2), dict(edges="code"), dict(edges="code", chain_blocks=3),
                                dict(hwc_quirk=True, scheme=BBANS, excess_state_len=77, seed=5)])
def test_containers_round_trip_through_the_check_trailer(monkeypatch, kw, stamp):
    codec = _fake_encoders(monkeypatch)
    plain = compress_images(codec, _images(), stamp=stamp, **kw)
    checked = compress_images(codec, _images(), stamp=stamp, checksums=True, **kw)
    ref = compress_images(codec, _images(), **kw)
    digests = container._encode_checked(None, None, None, [(0, 1)], 0, 0, 0, 0, np.array([0, 10 ** 4]))[1]
    off = 0
    quirk = kw.get("hwc_quirk", False)
    for img, r, p, c in zip(_images(), ref, plain, checked):
        n = _nblocks(img, kw)
        body = c[:c.size - 29] if stamp else c
        assert c.dtype == np.uint32 and body.size == r.size + n + 3
        assert np.array_equal(body[:r.size], r) and np.array_equal(body[r.size:r.size + n], digests[off:off + n])
        assert list(body[-3:]) == [n, CHECK_VERSION, CHECK_MARK]
        if stamp:
            assert np.array_equal(c[body.size:], p[r.size:]) and read_stamp(c) == read_stamp(p)
        _same(unpack_container(c, quirk), unpack_container(r, quirk))
        off += n
    if not quirk:
        regions = [(0, 3, 5, 40, 50), (3, 60, 100, 10, 10), (1, 0, 0, 1, 1)]
        for a, b in zip(plan_regions(checked, regions), plan_regions(ref, regions)):
            _same(a, b)


@pytest.mark.parametrize("stamp", [False, True])
@pytest.mark.parametrize("kw", [dict(), dict(chain_blocks=None), dict(chain_blocks=3, scheme=BBANS, excess_state_len=2,
                                                                         seed=(1 << 32) - 1)])
def test_archives_round_trip_through_the_check_trailer(monkeypatch, kw, stamp):
    codec = _fake_encoders(monkeypatch)
    ref = compress_archive(codec, _images(), **kw)
    p = compress_archive(codec, _images(), stamp=stamp, **kw)
    c = compress_archive(codec, _images(), stamp=stamp, checksums=True, **kw)
    n = sum(_nblocks(im, dict(edges="code")) for im in _images())
    body = c[:c.size - 29] if stamp else c
    assert ref[-1] == ARCHIVE_MARK and body.size == ref.size + n + 3 and np.array_equal(body[:ref.size], ref)
    assert list(body[-3:]) == [n, CHECK_VERSION, CHECK_MARK]
    if stamp:
        assert np.array_equal(c[body.size:], p[ref.size:]) and c[-1] == STAMP_MARK
    _same(unpack_archive(c), unpack_archive(ref))
    regions = [(1, 5, 5, 20, 60), (3, 0, 0, 100, 130)]
    _same(plan_archive(c, regions), plan_archive(ref, regions))
    _same(plan_archive(c), plan_archive(ref))


def test_checksums_are_made_only_on_request(monkeypatch):
    codec = _fake_encoders(monkeypatch)
    monkeypatch.setattr(container, "_encode_checked", lambda *a: (_ for _ in ()).throw(AssertionError("digested")))
    assert all(c[-1] != CHECK_MARK for c in compress_images(codec, _images()))
    assert compress_archive(codec, _images())[-1] == ARCHIVE_MARK


# ---- malformed trailers ----------------------------------------------------------------------------------------------------
def _arrays(monkeypatch):
    """A checked single-chain container, multi-chain container and archive, unstamped."""
    codec = _fake_encoders(monkeypatch)
    ims = _images()
    single = compress_images(codec, ims[:1], checksums=True)[0]
    multi = compress_images(codec, ims[3:], edges="code", chain_blocks=4, checksums=True)[0]
    return dict(single=single, multi=multi, archive=compress_archive(codec, ims, chain_blocks=5, checksums=True))


def _trailer_edits(a):
    """Malformed variants of a checked array a: name -> array."""
    n = int(a[-3])
    inner, digests = a[:a.size - 3 - n], a[a.size - 3 - n:a.size - 3]
    tr = lambda m, v=CHECK_VERSION: np.array([m, v, CHECK_MARK], dtype=np.uint32)       # noqa: E731
    cat = lambda *p: np.concatenate([np.asarray(x, dtype=np.uint32) for x in p])         # noqa: E731
    return {
        "version 0": cat(inner, digests, tr(n, 0)),
        "version 2": cat(inner, digests, tr(n, 2)),
        "version 2^32-1": cat(inner, digests, tr(n, 0xFFFFFFFF)),
        "more blocks than words": cat(inner, digests, tr(a.size)),
        "more than any array": cat(inner, digests, tr(container.MAX_ARCHIVE_BLOCKS + 1)),
        "nblocks 2^32-1": cat(inner, digests, tr(0xFFFFFFFF)),
        "one digest short": cat(inner, digests[:-1], tr(n - 1)),
        "one digest extra": cat(inner, digests, [7], tr(n + 1)),
        "no digests": cat(inner, tr(0)),
        "count one low": cat(inner, digests, tr(n - 1)),
        "count one high": cat(inner, digests, tr(n + 1)),
        "trailer alone": tr(0),
        "trailer of one": cat([5], tr(0)),
        "nested trailer": cat(a, digests, tr(n)),
        "stamp inside": cat(inner, [0] * 26, [26, 1, STAMP_MARK], digests, tr(n)),
        "truncated digests": cat(a[:inner.size + n // 2], tr(n)),
        "mark only": np.array([CHECK_MARK], dtype=np.uint32),
    }


CASES = sorted(_trailer_edits(np.array([1, 2, 3, 4, 5, 9, 9, 1, 1, CHECK_MARK], dtype=np.uint32)))


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("layout", ["single", "multi", "archive"])
def test_malformed_trailers_are_refused_before_any_device_work(monkeypatch, layout, case):
    bad = _trailer_edits(_arrays(monkeypatch)[layout])[case]
    monkeypatch.setattr(container, "StreamSet", lambda *a, **k: (_ for _ in ()).throw(AssertionError("StreamSet built")))
    if layout == "archive":
        calls = [lambda: unpack_archive(bad), lambda: plan_archive(bad), lambda: decompress_archive(NoDevice(), bad)]
    else:
        calls = [lambda: unpack_container(bad), lambda: plan_regions([bad], [(0, 0, 0, 1, 1)]),
                 lambda: decompress_images(NoDevice(), [bad]), lambda: decompress_regions(NoDevice(), [bad], [(0, 0, 0, 1, 1)])]
    for call in calls:
        with pytest.raises(ValueError):
            call()


def test_a_stamp_wraps_the_check_trailer_and_nothing_else(monkeypatch):
    arrays = _arrays(monkeypatch)
    codec = _fake_encoders(monkeypatch)
    both = compress_images(codec, _images()[:1], checksums=True, stamp=True)[0]
    assert both[-1] == STAMP_MARK and np.array_equal(both[:arrays["single"].size], arrays["single"])
    _same(unpack_container(both), unpack_container(arrays["single"]))
    with pytest.raises(ValueError):                              # a checked archive is not a container, nor the reverse
        unpack_container(arrays["archive"])
    with pytest.raises(ValueError):
        unpack_archive(arrays["single"])


# ---- the C ABI's refusals ---------------------------------------------------------------------------------------------------
FAKE = 1 << 40                               # never dereferenced: every call below is refused before anything is enqueued


def _abi(which, block=(0, 1, -1, 2), offs=(0, 3), channels=3, n_slots=None, n_seqs=None, null=()):
    block = np.ascontiguousarray(block, dtype=np.int64)
    offs = np.ascontiguousarray(offs, dtype=np.int64)
    p = dict(blocks=FAKE, ext=None, block=block.ctypes.data, offs=offs.ctypes.data, out=FAKE, expected=FAKE, result=FAKE)
    for k in null:
        p[k] = None
    n_slots = block.size if n_slots is None else n_slots
    n_seqs = offs.size - 1 if n_seqs is None else n_seqs
    if which == "digests":
        return lib().bsw_block_digests(p["blocks"], p["ext"], channels, n_slots, p["block"], p["offs"], n_seqs, p["out"], None)
    return lib().bsw_block_digests_check(p["blocks"], p["ext"], channels, n_slots, p["block"], p["offs"], n_seqs,
                                         p["expected"], p["result"], None)


ABI_BAD = {"channels 0": dict(channels=0), "channels 5": dict(channels=5), "no slots": dict(n_slots=0),
           "negative slots": dict(n_slots=-1), "no sequences": dict(n_seqs=0), "block past the end": dict(block=(0, 3)),
           "block -2": dict(block=(0, -2)), "block twice": dict(block=(1, 0, 1)), "offsets not from 0": dict(offs=(1, 3)),
           "offsets decrease": dict(offs=(0, 3, 2)), "offsets past 2^31": dict(offs=(0, 1 << 31)),
           "null blocks": dict(null=("blocks",)), "null table": dict(null=("block",)), "null offsets": dict(null=("offs",)),
           "null output": dict(null=("out", "expected", "result"))}


@pytest.mark.parametrize("which", ["digests", "check"])
@pytest.mark.parametrize("case", sorted(ABI_BAD))
def test_the_abi_refuses_bad_tables(which, case):
    assert _abi(which, **ABI_BAD[case]) == BSW_E_INVALID
    assert "bsw_block_digests" in lib().bsw_last_error().decode()


def test_the_check_result_is_refused_without_its_own_buffers():
    assert _abi("check", null=("result",)) == BSW_E_INVALID
    assert _abi("check", null=("expected",)) == BSW_E_INVALID
    assert _abi("digests", null=("out",)) == BSW_E_INVALID
