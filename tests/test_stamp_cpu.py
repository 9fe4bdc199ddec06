"""Stamped containers and archives without a GPU: the digest definition pinned by known answers, the stamp layout through
every writer and reader, every malformed stamp refused, and the refusal rule of the decoders against a stand-in codec."""
import types

import numpy as np
import pytest

from codec_harness import NoDevice
from stamp_harness import digest, digest_scalar, hexdigest
from bitswap_b200 import container
from bitswap_b200.codec import BBANS, BITSWAP, Fingerprint
from bitswap_b200.container import (ARCHIVE_MARK, CHAIN_MARK, STAMP_MARK, STAMP_VERSION, Stamp, compress_archive,
                                    compress_images, decompress_archive, decompress_images, decompress_regions,
                                    plan_archive, plan_regions, read_stamp, unpack_archive, unpack_container)

FP = Fingerprint(1, 3, 8, 8, 1, 3, 8, 252, False, 10, True, "split", True, "reference",
                 "0123456789abcdef00112233445566ff", "fedcba98765432100f1e2d3c4b5a6978")


def _pattern(n):
    return (bytes(range(256)) * (n // 256 + 1))[:n]


# bsw_digest of _pattern(n): pins the definition in include/bitswap_b200.h (the GPU tests hold the kernel to the twin)
KNOWN = {0: "50f10553f9e45a74693d993520f0ca99", 1: "44c8716ba655866465f868980f27a253",
         7: "70a6ffd26f0dceb56cd83e31e9063a1c", 8: "3554420d996b36d630e724bbd6db2b0c",
         9: "7ca1a70fe32ba1fc67d614be54880dc5", 65535: "9ab1bb2cfe6c5781d24ff63833e82d7d",
         65536: "670aabcb554f68ecb855d224ae7a45cd", 65537: "a860360f7ea469c0ac0df373402637f6"}


@pytest.mark.parametrize("n", sorted(KNOWN))
def test_digest_known_answers(n):
    assert hexdigest(digest(_pattern(n))) == KNOWN[n]


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 255, 8 * 8192 - 1, 8 * 8192, 8 * 8192 + 1, 16 * 8192 + 13])
def test_vectorised_twin_walks_the_definition(n):
    data = np.random.RandomState(n).randint(0, 256, n).astype(np.uint8).tobytes()
    assert digest(data) == digest_scalar(data)


def test_digest_sees_every_word_and_the_length():
    base = np.random.RandomState(3).randint(0, 256, 3 * 65536 + 5).astype(np.uint8)
    seen = {hexdigest(digest(base.tobytes()))}
    for pos in (0, 7, 8, 65535, 65536, 131071, base.size - 1):
        b = base.copy()
        b[pos] ^= 1
        seen.add(hexdigest(digest(b.tobytes())))
    seen.add(hexdigest(digest(base.tobytes() + b"\0")))                  # zero padding is not the same as a zero byte
    assert len(seen) == 9


# ---- writers and readers on a stand-in codec -------------------------------------------------------------------------------
def _recording(monkeypatch, fp=FP):
    """A codec stand-in with a fingerprint, and an encoder that returns random chains (only the layout is checked)."""
    rs = np.random.RandomState(9)

    def fake(codec, blocks, extents, chains, scheme, n_init, seed, wpb):
        return [(rs.randint(0, 1 << 32, rs.randint(0, 40), dtype=np.uint64).astype(np.uint32),
                 int(rs.randint(1 << 32, 1 << 62, dtype=np.uint64)), nb) for _, nb in chains]
    monkeypatch.setattr(container, "_encode", fake)
    return types.SimpleNamespace(cfg=types.SimpleNamespace(xs=[3]), fingerprint=lambda: fp)


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


def _writes(monkeypatch, write, **kw):
    """(unstamped, stamped) output of one writer call each, the encoder replaying the same random chains."""
    codec = _recording(monkeypatch)
    plain = write(codec, _images(), **kw)
    codec = _recording(monkeypatch)
    return plain, write(codec, _images(), stamp=True, **kw)


@pytest.mark.parametrize("kw", [dict(), dict(chain_blocks=2), dict(edges="code"), dict(edges="code", chain_blocks=3),
                                dict(hwc_quirk=True, scheme=BBANS, excess_state_len=77, seed=5)])
def test_containers_round_trip_through_the_stamp(monkeypatch, kw):
    plain, stamped = _writes(monkeypatch, compress_images, **kw)
    regions = [(0, 3, 5, 40, 50), (3, 60, 100, 10, 10), (1, 0, 0, 1, 1)]
    for p, s in zip(plain, stamped):
        assert s.dtype == np.uint32 and s[-1] == STAMP_MARK and s[-2] == STAMP_VERSION and s[-3] == 26
        assert np.array_equal(s[:p.size], p) and s.size == p.size + 29
        st = read_stamp(s)
        assert st == Stamp(FP, kw.get("scheme", BITSWAP), kw.get("hwc_quirk", False), kw.get("excess_state_len", 10000),
                           kw.get("seed", 100))
        assert read_stamp(p) is None
        _same(unpack_container(s, kw.get("hwc_quirk", False)), unpack_container(p, kw.get("hwc_quirk", False)))
    if not kw.get("hwc_quirk"):
        for a, b in zip(plan_regions(stamped, regions), plan_regions(plain, regions)):
            _same(a, b)


@pytest.mark.parametrize("kw", [dict(), dict(chain_blocks=None), dict(chain_blocks=3, scheme=BBANS, excess_state_len=2,
                                                                         seed=(1 << 32) - 1)])
def test_archives_round_trip_through_the_stamp(monkeypatch, kw):
    p, s = _writes(monkeypatch, compress_archive, **kw)
    assert np.array_equal(s[:p.size], p) and s.size == p.size + 29 and p[-1] == ARCHIVE_MARK
    assert read_stamp(s) == Stamp(FP, kw.get("scheme", BITSWAP), False, kw.get("excess_state_len", 10000), kw.get("seed", 100))
    _same(unpack_archive(s), unpack_archive(p))
    regions = [(1, 5, 5, 20, 60), (3, 0, 0, 100, 130)]
    _same(plan_archive(s, regions), plan_archive(p, regions))
    _same(plan_archive(s), plan_archive(p))


def test_a_stamp_is_made_only_on_request(monkeypatch):
    codec = _recording(monkeypatch, fp=None)
    codec.fingerprint = lambda: (_ for _ in ()).throw(AssertionError("fingerprint taken"))
    assert read_stamp(compress_images(codec, _images())[0]) is None
    assert read_stamp(compress_archive(codec, _images())) is None


@pytest.mark.parametrize("kw", [dict(excess_state_len=1), dict(excess_state_len=(1 << 24) + 1), dict(seed=-1),
                                dict(seed=1 << 32), dict(scheme=2)])
def test_stamped_writer_arguments_are_checked_before_any_device_work(kw):
    with pytest.raises(ValueError):
        compress_images(NoDevice(), _images(), stamp=True, **kw)


# ---- malformed stamps ------------------------------------------------------------------------------------------------------
def _stamped(monkeypatch):
    (c,), (cs,) = (x[:1] for x in _writes(monkeypatch, compress_images, chain_blocks=2))
    a, a_s = _writes(monkeypatch, compress_archive, chain_blocks=3)
    return c, cs, a, a_s


def _tweak(a, pos, value):
    a = a.copy()
    a[pos] = value
    return a


def _field(name):
    """Position of a stamp field counted from the end of a stamped array."""
    order = list(Fingerprint._fields[:14]) + [f"model_digest{i}" for i in range(4)] + [f"bins_digest{i}" for i in range(4)] \
        + ["scheme", "hwc_quirk", "excess_state_len", "seed"]
    return order.index(name) - 26 - 3


def _bad_stamps(s):
    return [
        s[-3:], s[-29:], s[-28:],                                                          # nothing or no room before it
        _tweak(s, -3, 25), _tweak(s, -3, 27), _tweak(s, -3, 1 << 31),                      # nfields
        _tweak(s, -2, 0), _tweak(s, -2, 2), _tweak(s, -2, 1 << 31),                        # unknown version
        _tweak(s, _field("cond_xscale"), 2), _tweak(s, _field("kernel_size"), 2), _tweak(s, _field("kernel_size"), 9),
        _tweak(s, _field("quantbits"), 4), _tweak(s, _field("quantbits"), 13), _tweak(s, _field("use_tensor_cores"), 2),
        _tweak(s, _field("tc_precision"), 2), _tweak(s, _field("tc_heads"), 7), _tweak(s, _field("coder"), 2),
        _tweak(s, _field("scheme"), 2), _tweak(s, _field("hwc_quirk"), 2),
        _tweak(s, _field("excess_state_len"), 1), _tweak(s, _field("excess_state_len"), (1 << 24) + 1),
        np.concatenate([s, s[-29:]]),                                                      # a stamp inside a stamp
    ]


def test_malformed_stamps_are_refused_before_any_device_work(monkeypatch):
    c, cs, a, a_s = _stamped(monkeypatch)
    for bad in _bad_stamps(cs):
        for f in (read_stamp, unpack_container, lambda x: plan_regions([x], [(0, 0, 0, 1, 1)]),
                  lambda x: decompress_images(NoDevice(), [c, x]), lambda x: decompress_regions(NoDevice(), [x], [])):
            with pytest.raises(ValueError):
                f(bad)
    for bad in _bad_stamps(a_s) + [_tweak(a_s, _field("scheme"), BBANS), _tweak(a_s, _field("excess_state_len"), 9999),
                                   _tweak(a_s, _field("seed"), 101), _tweak(a_s, _field("hwc_quirk"), 1)]:
        for f in (unpack_archive, plan_archive, lambda x: decompress_archive(NoDevice(), x)):
            with pytest.raises(ValueError):
                f(bad)


def test_a_reader_of_the_unstamped_layouts_refuses_a_stamped_array(monkeypatch):
    c, cs, a, a_s = _stamped(monkeypatch)
    for s in (cs, a_s):
        nblocks, h, w = (int(v) for v in s[-3:])                                           # read as a reference tail
        assert (nblocks, h, w) == (26, STAMP_VERSION, STAMP_MARK) and w >= 1 << 31
        with pytest.raises(ValueError):
            container._check_header(nblocks, h, w, False)
        assert int(s[-1]) not in (CHAIN_MARK, ARCHIVE_MARK)
    with pytest.raises(ValueError):
        unpack_archive(cs)                                                                 # a stamped container is no archive
    with pytest.raises(ValueError):
        unpack_container(a_s)                                                              # nor a stamped archive a container


# ---- the refusal rule ------------------------------------------------------------------------------------------------------
class _Codec:
    """A stand-in codec of a given fingerprint whose decoder must not run."""

    def __init__(self, fp):
        self.fp, self.device, self.cfg = fp, 0, types.SimpleNamespace(xs=(fp.xc, 32, 32), nz=fp.nz, zdim=2048)

    def fingerprint(self):
        return self.fp

    def decode(self, *a, **k):
        raise AssertionError("decode called")


@pytest.mark.parametrize("field,value", [("coder", "direct"), ("tc_precision", "bf16"), ("use_tensor_cores", False),
                                         ("tc_heads", False), ("reswidth", 256), ("quantbits", 12), ("revision", 2),
                                         ("model_digest", "0" * 32), ("bins_digest", "1" * 32)])
def test_each_mismatch_is_named_before_any_stream_is_made(monkeypatch, field, value):
    c, cs, a, a_s = _stamped(monkeypatch)
    monkeypatch.setattr(container, "StreamSet", lambda *a, **k: (_ for _ in ()).throw(AssertionError("StreamSet built")))
    codec = _Codec(FP._replace(**{field: value}))
    calls = [lambda: decompress_images(codec, [c, cs]), lambda: decompress_regions(codec, [cs], [(0, 0, 0, 1, 1)]),
             lambda: decompress_archive(codec, a_s)]
    for call in calls:
        with pytest.raises(ValueError, match=rf"{field}: stamped {getattr(FP, field)!r}, here {value!r}"):
            call()


def test_arguments_are_compared_too(monkeypatch):
    c, cs, a, a_s = _stamped(monkeypatch)
    codec = _Codec(FP)
    with pytest.raises(ValueError, match="scheme: stamped 0, here 1") as e:
        decompress_images(codec, [cs], scheme=BBANS, hwc_quirk=True, channels=1)
    assert "hwc_quirk: stamped False, here True" in str(e.value) and "channels: stamped 3, here 1" in str(e.value)
    monkeypatch.setattr(container, "StreamSet", lambda *a, **k: (_ for _ in ()).throw(AssertionError("StreamSet built")))
    for call in (lambda: decompress_images(codec, [cs]), lambda: decompress_archive(codec, a_s),
                 lambda: decompress_images(codec, [c])):                                   # matching: on to the streams
        with pytest.raises(AssertionError, match="StreamSet built"):
            call()


def test_unstamped_arrays_never_ask_for_a_fingerprint(monkeypatch):
    c, cs, a, a_s = _stamped(monkeypatch)
    with pytest.raises(AssertionError, match="touched"):
        decompress_images(NoDevice(), [c])
    with pytest.raises(AssertionError, match="codec.fingerprint touched"):
        decompress_images(NoDevice(), [c, cs])
    with pytest.raises(AssertionError, match="codec.fingerprint touched"):
        decompress_archive(NoDevice(), a_s)
