"""Images in and out as CUDA tensors: the tile and untile kernels against their numpy twin on every kind of strided input,
with the bytes around their outputs untouched; CUDA input writing the same containers and archives as numpy input on every
kind of codec; as_tensors decodes equal to the numpy ones; invalid CUDA input refused before any device work."""
import os
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from codec_harness import random_images, setup                                                   # noqa: E402
from device_io_harness import tile_twin, untile_twin                                              # noqa: E402
from bitswap_b200 import container, synthetic                                                     # noqa: E402
from bitswap_b200._lib import lib                                                                 # noqa: E402
from bitswap_b200.codec import BBANS, BITSWAP, Bins, BitSwapCodec, PipelinedCodec                 # noqa: E402
from bitswap_b200.config import preset                                                            # noqa: E402
from bitswap_b200.container import (TILE_CODE, TILE_CROP, TILE_QUIRK, _Blocks, _chain_runs,         # noqa: E402
                                    compress_archive, compress_images, decompress_archive, decompress_images,
                                    decompress_regions)
from bitswap_b200.model import Model                                                              # noqa: E402

SIZES = [(1, 1), (1, 33), (31, 32), (32, 32), (33, 65), (28, 28), (100, 70)]
PAD = 4096


def _stub(C, device=0):
    return types.SimpleNamespace(cfg=types.SimpleNamespace(xs=[C]), device=device)


def _strided(C, rs):
    """CUDA images of every stride pattern, with their host copies: contiguous, CHW permuted, a crop view, a channel slice,
    an expanded (stride 0) tensor."""
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()           # noqa: E731
    big = cuda(rs.randint(0, 256, (80, 90, C)).astype(np.uint8))
    chw = cuda(rs.randint(0, 256, (C, 70, 45)).astype(np.uint8))
    rgba = cuda(rs.randint(0, 256, (40, 100, C + 1)).astype(np.uint8))
    row = cuda(rs.randint(0, 256, (1, 66, C)).astype(np.uint8))
    ims = [cuda(rs.randint(0, 256, (h, w, C)).astype(np.uint8)) for h, w in SIZES]
    ims += [chw.permute(1, 2, 0), big[5:38, 7:40], big[40:, ::2], rgba[..., :C], row.expand(35, 66, C)]
    return ims


def _tile_abi(blocks, cnb, stream, steps, ragged):
    """bsw_tile_blocks into buffers with PAD sentinel bytes on both sides: (blocks, extents, sentinels intact)."""
    K, C = len(cnb), blocks.C
    x = torch.full((2 * PAD + steps * K * C * 1024,), 0xAB, dtype=torch.uint8, device="cuda")
    e = torch.full((2 * PAD + steps * K * 2,), -1, dtype=torch.int16, device="cuda")
    views, keep = blocks.views(_stub(C))
    assert lib().bsw_tile_blocks(views.ctypes.data, len(views), C, blocks.mode, cnb.ctypes.data, stream.ctypes.data, K,
                                 steps, x[PAD:].data_ptr(), e[PAD:].data_ptr() if ragged else None,
                                 torch.cuda.current_stream().cuda_stream) == 0
    x, e = x.cpu().numpy(), e.cpu().numpy()
    intact = (x[:PAD] == 0xAB).all() and (x[-PAD:] == 0xAB).all() and (e[:PAD] == -1).all() and (e[-PAD:] == -1).all()
    return x[PAD:-PAD].reshape(steps, K, C, 32, 32), e[PAD:-PAD].reshape(steps, K, 2), intact


@pytest.mark.parametrize("mode", [TILE_CROP, TILE_CODE, TILE_QUIRK])
@pytest.mark.parametrize("C", [1, 3])
def test_tile_equals_the_twin_on_every_stride_pattern(mode, C):
    rs = np.random.RandomState(5 + mode + C)
    ims = _strided(C, rs)
    ims = [im for im in ims if mode == TILE_CODE or min(im.shape[:2]) >= 32]
    host = [np.ascontiguousarray(im.cpu().numpy()) for im in ims]
    batch = torch.from_numpy(rs.randint(0, 256, (5, 33, 65, C)).astype(np.uint8)).cuda()
    for images, twin_images in ((ims, host), (host, host), (batch, list(batch.cpu().numpy())),
                                (batch.cpu().numpy(), list(batch.cpu().numpy())), (host[:2] + ims[2:], host)):
        blocks = _Blocks(_stub(C), images, mode, strict=False)
        gh, gw = container._grid(blocks.shapes, mode)
        for L in (None, 1, 3, 7, 32):
            _, cnb = _chain_runs(gh * gw, L)
            order = np.argsort(-cnb, kind="stable")
            stream = np.empty(len(cnb), dtype=np.int32)
            stream[order] = np.arange(len(cnb))
            steps = int(cnb.max())
            want_x, want_e = tile_twin(twin_images, mode, cnb, stream, steps)
            got_x, got_e, intact = _tile_abi(blocks, cnb, stream, steps, mode == TILE_CODE)
            assert intact and np.array_equal(got_x, want_x), (mode, C, L)
            if mode == TILE_CODE:
                assert np.array_equal(got_e, want_e)


@pytest.mark.parametrize("quirk", [False, True])
@pytest.mark.parametrize("C", [1, 3])
def test_untile_equals_the_twin(quirk, C):
    rs = np.random.RandomState(9 + C)
    shapes = [(32, 64), (96, 32), (64, 64)] if quirk else SIZES + [(150, 390)]
    mode = TILE_QUIRK if quirk else TILE_CODE
    nb = np.array([-(-h // 32) * -(-w // 32) for h, w in shapes], dtype=np.int64)
    for L in (None, 1, 3, 7, 32):
        cnb = np.array(container.chain_sizes(int(nb.sum()), L), dtype=np.int64)
        stream = np.arange(len(cnb), dtype=np.int32)[::-1].copy()
        steps = int(cnb.max())
        x = rs.randint(0, 256, (steps, len(cnb), C, 32, 32)).astype(np.uint8)
        regions = [(i, 0, 0, h, w) for i, (h, w) in enumerate(shapes)]
        for i, (h, w) in enumerate(shapes):
            regions += [(i, h - 1, w - 1, 1, 1), (i, min(31, h - 1), 0, 1, 1), (i, 0, 0, min(h, 3), min(w, 3)),
                        (i, 0, 0, 1, 1), (i, h // 2, w // 3, h - h // 2, w - w // 3)]
        total = sum(h * w for _, _, _, h, w in regions) * C
        out = torch.full((2 * PAD + total,), 0xCD, dtype=torch.uint8, device="cuda")
        sh = np.ascontiguousarray(shapes, dtype=np.int32)
        regs = np.ascontiguousarray(regions, dtype=np.int32)
        xd = torch.from_numpy(x).cuda()
        assert lib().bsw_untile_regions(sh.ctypes.data, len(sh), C, mode, cnb.ctypes.data, stream.ctypes.data, len(cnb),
                                        len(cnb), steps, xd.data_ptr(), regs.ctypes.data, len(regs), out[PAD:].data_ptr(),
                                        torch.cuda.current_stream().cuda_stream) == 0
        got = out.cpu().numpy()
        assert (got[:PAD] == 0xCD).all() and (got[-PAD:] == 0xCD).all()
        assert np.array_equal(got[PAD:-PAD], untile_twin(shapes, mode, cnb, stream.astype(np.int64), x, regions)), L


# ---- containers and archives: CUDA input writes what numpy input writes ---------------------------------------------------
def _codec(kind):
    if kind.startswith("tiny"):
        return setup(kind, 8).codec
    name = {"imagenetcrop4": "imagenetcrop4", "mnist2": "mnist2", "direct": "tiny3", "bf16": "mnist2"}[kind]
    cfg = preset(name)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
    if kind == "direct":
        m = Model.from_config(cfg, max_batch=8, use_tensor_cores=False).load_state_dict(sd)
        m.compress()
        return BitSwapCodec(cfg, m, bins, 8, coder="direct")
    m = Model.from_config(cfg, max_batch=8, use_tensor_cores=True, tc_precision="bf16" if kind == "bf16" else "split")
    m.load_state_dict(sd)
    m.compress()
    return BitSwapCodec(cfg, m, bins, 8)


def _variants(host):
    """The same images as CUDA tensors: contiguous, CHW permuted, and as views into one wider tensor."""
    cont = [torch.from_numpy(im).cuda() for im in host]
    perm = [torch.from_numpy(np.ascontiguousarray(im.transpose(2, 0, 1))).cuda().permute(1, 2, 0) for im in host]
    wide = []
    for im in host:
        h, w, C = im.shape
        t = torch.zeros((h + 3, w + 5, C + 1), dtype=torch.uint8, device="cuda")
        t[2:2 + h, 1:1 + w, :C] = torch.from_numpy(im).cuda()
        wide.append(t[2:2 + h, 1:1 + w, :C])
    return [cont, perm, wide]


@pytest.mark.parametrize("kind,scheme", [("tiny", BITSWAP), ("tiny", BBANS), ("tiny3", BITSWAP), ("tiny3", BBANS),
                                         ("imagenetcrop4", BITSWAP), ("mnist2", BITSWAP), ("direct", BITSWAP),
                                         ("bf16", BITSWAP)])
def test_cuda_input_writes_the_bytes_numpy_input_writes(kind, scheme):
    codec = _codec(kind)
    C = codec.cfg.xs[0]
    host = random_images(C, [(33, 65), (64, 96), (100, 70), (32, 32), (28, 28), (1, 40)], seed=31)
    big = [im for im in host if min(im.shape[:2]) >= 32]
    kw = dict(scheme=scheme, excess_state_len=3000)
    for args in (dict(), dict(edges="code", chain_blocks=3), dict(hwc_quirk=True), dict(edges="code", stamp=True)):
        ims = host if args.get("edges") == "code" else big
        want = compress_images(codec, ims, **kw, **args)
        for variant in _variants(ims):
            got = compress_images(codec, variant, **kw, **args)
            assert len(got) == len(want) and all(g.dtype == np.uint32 and np.array_equal(g, w) for g, w in zip(got, want)), args
    same = [im[:28, :28] for im in big]
    want = compress_images(codec, same, edges="code", **kw)
    assert all(np.array_equal(g, w) for g, w in zip(compress_images(codec, torch.from_numpy(np.stack(same)).cuda(),
                                                                     edges="code", **kw), want))
    for stamp in (False, True):
        want = compress_archive(codec, host, chain_blocks=3, stamp=stamp, **kw)
        for variant in _variants(host):
            assert np.array_equal(compress_archive(codec, variant, chain_blocks=3, stamp=stamp, **kw), want)
        assert np.array_equal(compress_archive(codec, torch.from_numpy(np.stack(same)).cuda(), chain_blocks=3, stamp=stamp, **kw),
                              compress_archive(codec, np.stack(same), chain_blocks=3, stamp=stamp, **kw))


def _same_tensors(got, want):
    for g, w in zip(got, want):
        assert torch.is_tensor(g) and g.is_cuda and g.dtype == torch.uint8 and g.is_contiguous()
        assert tuple(g.shape) == w.shape and np.array_equal(g.cpu().numpy(), w)
    assert len(got) == len(want)


@pytest.mark.parametrize("pipelined", [False, True])
def test_as_tensors_decodes_equal_the_numpy_ones(pipelined):
    s = setup("tiny3", 24)
    codec = PipelinedCodec(s.cfg, s.sd, s.bins, 8, lanes=2, use_tensor_cores=False, free_running=True) if pipelined \
        else BitSwapCodec(s.cfg, s.model, s.bins, 8)                                    # max_batch 8 < the chains below
    host = random_images(3, [(150, 390), (33, 65), (1, 1), (28, 28), (64, 64)], seed=33)
    conts = compress_images(codec, [torch.from_numpy(im).cuda() for im in host], edges="code", chain_blocks=3,
                            excess_state_len=3000)
    full = decompress_images(codec, conts)
    assert all(np.array_equal(a, b) for a, b in zip(full, host))
    _same_tensors(decompress_images(codec, conts, as_tensors=True), host)
    regions = [(0, 100, 300, 50, 90), (0, 0, 0, 1, 1), (0, 31, 31, 2, 2), (1, 10, 10, 1, 1), (1, 0, 0, 33, 65), (4, 5, 5, 20, 20)]
    want = decompress_regions(codec, conts, regions)
    assert all(np.array_equal(w, host[i][y:y + h, x:x + w_]) for (i, y, x, h, w_), w in zip(regions, want))
    _same_tensors(decompress_regions(codec, conts, regions, as_tensors=True), want)
    a = compress_archive(codec, host, chain_blocks=3, excess_state_len=3000)
    _same_tensors(decompress_archive(codec, a, as_tensors=True), host)
    want = decompress_archive(codec, a, regions)
    _same_tensors(decompress_archive(codec, a, regions, as_tensors=True), want)
    q = compress_images(codec, [im for im in host if min(im.shape[:2]) >= 32], hwc_quirk=True, excess_state_len=3000)
    _same_tensors(decompress_images(codec, q, hwc_quirk=True, as_tensors=True), decompress_images(codec, q, hwc_quirk=True))


# ---- invalid CUDA input ---------------------------------------------------------------------------------------------------
class _Untouchable:
    """A codec stand-in with a config and a device; any call on it fails the test."""

    def __init__(self, C, device):
        self.cfg, self.device = types.SimpleNamespace(xs=[C]), device

    def __getattr__(self, name):
        raise AssertionError(f"codec.{name} touched")


BAD = {"float": lambda ok: [ok.float()], "int16": lambda ok: [ok.short()], "2-D": lambda ok: [ok[..., 0]],
       "4-D in a list": lambda ok: [ok[None]], "channels": lambda ok: [ok[..., :2]], "empty": lambda ok: [ok[:0]],
       "no columns": lambda ok: [ok[:, :0]], "batch of floats": lambda ok: ok[None].float(),
       "batch channels": lambda ok: ok[None, ..., :1], "second image bad": lambda ok: [ok, ok.int()]}


@pytest.mark.parametrize("case", sorted(BAD))
@pytest.mark.parametrize("writer", ["images crop", "images code", "archive"])
def test_invalid_cuda_input_is_refused_before_any_device_work(case, writer, monkeypatch):
    monkeypatch.setattr(container, "StreamSet", lambda *a, **k: (_ for _ in ()).throw(AssertionError("StreamSet built")))
    codec = _Untouchable(3, torch.cuda.current_device())
    images = BAD[case](torch.zeros((40, 40, 3), dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        if writer == "archive":
            compress_archive(codec, images)
        else:
            compress_images(codec, images, edges=writer.split()[1])


@pytest.mark.parametrize("writer", ["images crop", "images code", "archive"])
def test_small_or_foreign_cuda_images_are_refused_before_any_device_work(writer, monkeypatch):
    monkeypatch.setattr(container, "StreamSet", lambda *a, **k: (_ for _ in ()).throw(AssertionError("StreamSet built")))
    dev = torch.cuda.current_device()
    ok = torch.zeros((40, 40, 3), dtype=torch.uint8, device="cuda")
    call = (lambda c, ims: compress_archive(c, ims)) if writer == "archive" else \
        (lambda c, ims: compress_images(c, ims, edges=writer.split()[1]))
    with pytest.raises(ValueError, match="cuda:"):
        call(_Untouchable(3, dev + 1), [ok])                                       # the codec is on another device
    with pytest.raises(ValueError, match="cuda:"):
        call(_Untouchable(3, dev + 1), ok[None])
    if writer == "images crop":
        for small in ([ok[:31]], [ok[:, :20]], ok[None, :31]):
            with pytest.raises(ValueError, match=">= 32"):
                call(_Untouchable(3, dev), small)
