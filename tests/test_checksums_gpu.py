"""Checked containers and archives on the device: the digest kernel against its numpy twin, checked = unchecked + trailer
for every writer mode and kind of codec with verified round trips, a flipped digest caught by every decoder that pops its
block and by none that does not, and a container decoded with another coder or arithmetic than the encoder's."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from checksum_harness import block_digests, kernel_twin                                           # noqa: E402
from codec_harness import random_images, setup                                                    # noqa: E402
from bitswap_b200 import synthetic                                                                # noqa: E402
from bitswap_b200._lib import lib                                                                 # noqa: E402
from bitswap_b200.codec import BBANS, BITSWAP, Bins, BitSwapCodec, PipelinedCodec                 # noqa: E402
from bitswap_b200.config import preset                                                            # noqa: E402
from bitswap_b200.container import (CHECK_MARK, CHECK_VERSION, TILE_CODE, TILE_CROP, TILE_QUIRK, _Blocks,  # noqa: E402
                                    block_extents, compress_archive, compress_images, decompress_archive,
                                    decompress_images, decompress_regions)
from bitswap_b200.model import Model                                                              # noqa: E402

SENTINEL = 0x5A5A5A5A


# ---- the kernel against the twin --------------------------------------------------------------------------------------------
def _case(rs, S, J, C, ragged, offs):
    x = rs.randint(0, 256, (S, J, C, 32, 32)).astype(np.uint8)
    total = int(offs[-1])
    block = np.full(S * J, -1, dtype=np.int64)
    live = rs.rand(S * J) < 0.7
    block[np.flatnonzero(live)[:total]] = rs.permutation(total)[:min(total, int(live.sum()))]
    ext = rs.randint(1, 33, (S, J, 2)).astype(np.int16) if ragged else None
    if ragged:
        ext[0, 0] = (32, 32)
    return x, block.reshape(S, J), ext


@pytest.mark.parametrize("C", [1, 3, 4])
@pytest.mark.parametrize("ragged", [False, True])
def test_kernel_equals_the_twin(C, ragged):
    rs = np.random.RandomState(C + 10 * ragged)
    offs = np.array([0, 5, 5, 19, 40], dtype=np.int64)
    x, block, ext = _case(rs, 6, 9, C, ragged, offs)
    xd = torch.from_numpy(x).cuda()
    ed = None if ext is None else torch.from_numpy(ext).cuda()
    out = torch.full((int(offs[-1]) + 64,), SENTINEL, dtype=torch.int32, device="cuda")
    tab = np.ascontiguousarray(block.reshape(-1))
    st = torch.cuda.current_stream().cuda_stream
    assert lib().bsw_block_digests(xd.data_ptr(), None if ed is None else ed.data_ptr(), C, tab.size, tab.ctypes.data,
                                   offs.ctypes.data, len(offs) - 1, out[32:].data_ptr(), st) == 0
    got = out.cpu().numpy().view(np.uint32)
    want = kernel_twin(x, block, offs, ext, np.full(int(offs[-1]), SENTINEL, dtype=np.uint32))
    assert (got[:32] == SENTINEL).all() and (got[-32:] == SENTINEL).all()
    assert np.array_equal(got[32:-32], want)
    # the compare step: every block equal, then two digests changed
    res = torch.empty(2, dtype=torch.int64, device="cuda")
    for flip in ([], [17, 3]):
        exp = want.copy()
        live = set(block[block >= 0].tolist())
        flip = [g for g in flip if g in live]
        for g in flip:
            exp[g] ^= 1 << 7
        ed_ = torch.from_numpy(exp.view(np.int32)).cuda()
        assert lib().bsw_block_digests_check(xd.data_ptr(), None if ed is None else ed.data_ptr(), C, tab.size,
                                             tab.ctypes.data, offs.ctypes.data, len(offs) - 1, ed_.data_ptr(),
                                             res.data_ptr(), st) == 0
        bad, first = res.cpu().tolist()
        assert bad == len(flip) and (first == min(flip) if flip else first == (1 << 63) - 1)


def test_kernel_on_quirk_slots_and_a_large_buffer():
    """Full-extent slots (what a hwc_quirk buffer holds) and 2 x 2048 slots of 3 channels, one sequence."""
    rs = np.random.RandomState(3)
    x = rs.randint(0, 256, (2048, 2, 3, 32, 32)).astype(np.uint8)
    block = np.arange(4096, dtype=np.int64)[::-1].copy()
    offs = np.array([0, 4096], dtype=np.int64)
    out = torch.zeros(4096, dtype=torch.int32, device="cuda")
    xd = torch.from_numpy(x).cuda()
    assert lib().bsw_block_digests(xd.data_ptr(), None, 3, 4096, block.ctypes.data, offs.ctypes.data, 1, out.data_ptr(),
                                   torch.cuda.current_stream().cuda_stream) == 0
    want = np.empty(4096, dtype=np.uint32)
    want[block] = block_digests(x.reshape(-1, 3, 32, 32), block)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want)


# ---- writers and round trips --------------------------------------------------------------------------------------------------
def _codec(kind, B=8):
    if kind.startswith("tiny"):
        return setup(kind, B).codec
    name = {"imagenetcrop4": "imagenetcrop4", "mnist2": "mnist2", "direct": "tiny3", "bf16": "mnist2"}[kind]
    cfg = preset(name)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
    if kind == "direct":
        m = Model.from_config(cfg, max_batch=B, use_tensor_cores=False).load_state_dict(sd)
        m.compress()
        return BitSwapCodec(cfg, m, bins, B, coder="direct")
    m = Model.from_config(cfg, max_batch=B, use_tensor_cores=True, tc_precision="bf16" if kind == "bf16" else "split")
    m.load_state_dict(sd)
    m.compress()
    return BitSwapCodec(cfg, m, bins, B)


def _twin_digests(codec, img, mode, first=0):
    """The digests of one image's row-major blocks, by the reference tiling and the numpy twin, its first block being block
    `first` of the sequence the digests are seeded over (a container: its image; an archive: all its images)."""
    blocks = np.asarray(_Blocks(codec, [img], mode, strict=False))
    ext = block_extents(*img.shape[:2]) if mode == TILE_CODE else None
    return block_digests(blocks, first + np.arange(len(blocks)), ext)


def _split(c, stamped):
    body = c[:c.size - 29] if stamped else c
    n = int(body[-3])
    assert list(body[-2:]) == [CHECK_VERSION, CHECK_MARK]
    return body[:body.size - 3 - n], body[body.size - 3 - n:body.size - 3]


@pytest.mark.parametrize("kind,scheme", [("tiny", BITSWAP), ("tiny", BBANS), ("tiny3", BITSWAP), ("tiny3", BBANS),
                                         ("imagenetcrop4", BITSWAP), ("mnist2", BITSWAP), ("direct", BITSWAP),
                                         ("bf16", BITSWAP)])
def test_checked_arrays_are_the_unchecked_ones_plus_the_trailer_and_verify(kind, scheme):
    codec = _codec(kind)
    C = codec.cfg.xs[0]
    host = random_images(C, [(33, 65), (64, 96), (100, 70), (32, 32), (28, 28), (1, 40)], seed=41)
    big = [im for im in host if min(im.shape[:2]) >= 32]
    kw = dict(scheme=scheme, excess_state_len=3000)
    for args in (dict(), dict(edges="code", chain_blocks=3), dict(hwc_quirk=True), dict(edges="code", stamp=True)):
        ims = host if args.get("edges") == "code" else big
        mode = TILE_CODE if args.get("edges") == "code" else TILE_QUIRK if args.get("hwc_quirk") else TILE_CROP
        plain = compress_images(codec, ims, **kw, **args)
        cuda = [torch.from_numpy(im).cuda() for im in ims]
        for images in (ims, cuda):
            checked = compress_images(codec, images, checksums=True, **kw, **args)
            for img, p, c in zip(ims, plain, checked):
                inner, digests = _split(c, args.get("stamp", False))
                assert np.array_equal(inner, p[:inner.size]) and np.array_equal(digests, _twin_digests(codec, img, mode))
                if args.get("stamp"):
                    assert np.array_equal(c[-29:], p[-29:]) and c.size == p.size + digests.size + 3
        q = args.get("hwc_quirk", False)
        out = decompress_images(codec, checked, channels=C, scheme=scheme, hwc_quirk=q)
        want = decompress_images(codec, plain, channels=C, scheme=scheme, hwc_quirk=q)
        assert all(np.array_equal(a, b) for a, b in zip(out, want))
        if args.get("edges") == "code":
            assert all(np.array_equal(a, b) for a, b in zip(out, ims))
    a_plain = compress_archive(codec, host, chain_blocks=3, **kw)
    a = compress_archive(codec, host, chain_blocks=3, checksums=True, **kw)
    assert np.array_equal(a[:a_plain.size], a_plain)
    first = np.cumsum([0] + [-(-im.shape[0] // 32) * -(-im.shape[1] // 32) for im in host])
    assert np.array_equal(a[a_plain.size:-3], np.concatenate([_twin_digests(codec, im, TILE_CODE, int(f))
                                                              for im, f in zip(host, first)]))
    assert all(np.array_equal(x, y) for x, y in zip(decompress_archive(codec, a), host))


# ---- a flipped digest ---------------------------------------------------------------------------------------------------------
def _flip(c, k):
    """c with the digest of its block k changed (unstamped)."""
    c = c.copy()
    n = int(c[-3])
    c[c.size - 3 - n + k] ^= 1
    return c


def test_a_flipped_digest_is_caught_by_every_decode_that_pops_its_block():
    codec = setup("tiny3", 8).codec
    host = random_images(3, [(40, 40), (100, 130)], seed=43)
    conts = compress_images(codec, host, edges="code", chain_blocks=3, excess_state_len=3000, checksums=True)
    # image 1: 4 x 5 blocks in chains [0-2, 3-5, 6-8, 9-11, 12-14, 15-17, 18-19]; block 7 is row 1, column 2, chain 2
    bad = [conts[0], _flip(conts[1], 7)]
    for call in (lambda: decompress_images(codec, bad), lambda: decompress_images(codec, bad, as_tensors=True),
                 lambda: decompress_regions(codec, bad, [(1, 32, 32, 5, 5)]),                 # block 6: pops 8, 7, 6
                 lambda: decompress_regions(codec, bad, [(1, 40, 70, 1, 1)])):                # block 7 itself
        with pytest.raises(ValueError, match=r"1 decoded block differs .* image 1, block row 1, column 2, in chain 2 of "
                                             r"container 1"):
            call()
    # windows that never pop block 7: block 8 (chain 2's last), block 19, all of image 0
    for regions in ([(1, 32, 96, 32, 32)], [(1, 96, 128, 4, 2)], [(0, 0, 0, 40, 40)]):
        got = decompress_regions(codec, bad, regions)
        assert all(np.array_equal(g, host[i][y:y + h, x:x + w]) for g, (i, y, x, h, w) in zip(got, regions))
    assert all(np.array_equal(a, b) for a, b in zip(decompress_images(codec, bad, verify=False), host))
    # an archive: 4 + 20 blocks, chains of 3; block 11 of the sequence is image 1's block 7 again, in chain 3
    a = compress_archive(codec, host, chain_blocks=3, excess_state_len=3000, checksums=True)
    a_bad = _flip(a, 11)
    with pytest.raises(ValueError, match=r"image 1, block row 1, column 2, in chain 3 of the archive"):
        decompress_archive(codec, a_bad)
    assert np.array_equal(decompress_archive(codec, a_bad, [(0, 0, 0, 40, 40)])[0], host[0])
    assert all(np.array_equal(x, y) for x, y in zip(decompress_archive(codec, a_bad, verify=False), host))


# ---- another coder or arithmetic than the encoder's ---------------------------------------------------------------------------
def _other(kind):
    """(encoder, decoder) codecs that differ in coder (tiny3, SIMT) or in tc_precision (mnist2, tensor cores)."""
    if kind == "coder":
        cfg = preset("tiny3")
        sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
        bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
        out = []
        for coder in ("reference", "direct"):
            m = Model.from_config(cfg, max_batch=8, use_tensor_cores=False).load_state_dict(sd)
            m.compress()
            out.append(BitSwapCodec(cfg, m, bins, 8, coder=coder))
        return out
    return [_codec("mnist2"), _codec("bf16")]


def _outcome(call):
    try:
        return "returned", call()
    except (IndexError, OverflowError) as e:
        return f"stream error {type(e).__name__}", None
    except ValueError as e:
        return "ValueError", str(e)


@pytest.mark.parametrize("kind", ["coder", "tc_precision"])
def test_another_coder_or_arithmetic_is_caught_by_the_digests(kind, record_property):
    enc, dec = _other(kind)
    C = enc.cfg.xs[0]
    host = random_images(C, [(64, 64), (33, 65), (28, 28)], seed=47)
    kw = dict(edges="code", excess_state_len=3000)
    plain = compress_images(enc, host, **kw)
    what, got = _outcome(lambda: decompress_images(dec, plain, channels=C))
    if what == "returned":                                # unchecked: wrong pixels come back without a word
        wrong = sum(not np.array_equal(a, b) for a, b in zip(got, host))
        what = f"returned, {wrong} of {len(host)} images wrong"
        assert wrong > 0
    record_property("unchecked", what)
    print(f"{kind}: unchecked container decoded with the other codec: {what}")
    assert what.startswith(("returned", "stream error"))
    checked = compress_images(enc, host, checksums=True, **kw)
    what_c, msg = _outcome(lambda: decompress_images(dec, checked, channels=C))
    record_property("checked", what_c)
    print(f"{kind}: checked container decoded with the other codec: {what_c} {msg or ''}")
    assert what_c == "ValueError" or what_c.startswith("stream error")
    if what_c == "ValueError":
        assert "differ" in msg and "image" in msg
    assert all(np.array_equal(a, b) for a, b in zip(decompress_images(enc, checked, channels=C), host))


# ---- max_batch, lanes and as_tensors -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pipelined", [False, True])
def test_checked_decodes_through_sub_batches_lanes_and_tensors(pipelined):
    s = setup("tiny3", 24)
    codec = PipelinedCodec(s.cfg, s.sd, s.bins, 8, lanes=2, use_tensor_cores=False, free_running=True) if pipelined \
        else BitSwapCodec(s.cfg, s.model, s.bins, 8)                                    # max_batch 8 < the chains below
    host = random_images(3, [(150, 390), (33, 65), (1, 1), (28, 28), (64, 64)], seed=49)
    plain = compress_images(codec, host, edges="code", chain_blocks=3, excess_state_len=3000)
    conts = compress_images(codec, [torch.from_numpy(im).cuda() for im in host], edges="code", chain_blocks=3,
                            excess_state_len=3000, checksums=True)
    assert all(np.array_equal(c[:p.size], p) for c, p in zip(conts, plain))
    for got in (decompress_images(codec, conts), decompress_images(codec, conts, as_tensors=True)):
        assert all(np.array_equal(g.cpu().numpy() if torch.is_tensor(g) else g, h) for g, h in zip(got, host))
    regions = [(0, 100, 300, 50, 90), (0, 0, 0, 1, 1), (1, 0, 0, 33, 65), (4, 5, 5, 20, 20)]
    got = decompress_regions(codec, conts, regions, as_tensors=True)
    assert all(np.array_equal(g.cpu().numpy(), host[i][y:y + h, x:x + w]) for g, (i, y, x, h, w) in zip(got, regions))
    a = compress_archive(codec, host, chain_blocks=3, excess_state_len=3000, checksums=True)
    assert all(np.array_equal(g.cpu().numpy(), h) for g, h in zip(decompress_archive(codec, a, as_tensors=True), host))
    # image 0 is 5 x 13 blocks; block 40 is row 3, column 1
    bad = [_flip(conts[0], 40)] + conts[1:]
    with pytest.raises(ValueError, match=r"image 0, block row 3, column 1"):
        decompress_images(codec, bad, as_tensors=True)
    mixed = [plain[0], conts[1], plain[2], conts[3], conts[4]]                          # checked and unchecked in one call
    assert all(np.array_equal(g, h) for g, h in zip(decompress_images(codec, mixed), host))
