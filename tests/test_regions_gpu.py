"""Decoding regions of containers on the GPU: every region equals the crop of the whole decoded image, the codec pops
exactly the planned blocks, and a chain stopped part-way holds the encoder's state before its earliest wanted block."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from codec_harness import Counting, random_images, setup                   # noqa: E402
from bitswap_b200 import container, synthetic                              # noqa: E402
from bitswap_b200.config import preset                                     # noqa: E402
from bitswap_b200.codec import Bins, PipelinedCodec, BITSWAP, BBANS                 # noqa: E402
from bitswap_b200.streams import StreamSet                                 # noqa: E402
from bitswap_b200.container import (block_grid, chain_sizes, compress_images, decompress_images,   # noqa: E402
                                    decompress_regions, extract_blocks, extract_edge_blocks, plan_regions)

N_INIT = 3000


def _regions(rs, shapes, count):
    """Corner pixels, whole images, one-pixel rows and `count` random boxes over images of the given (h, w)."""
    out = []
    for i, (h, w) in enumerate(shapes):
        out += [(i, 0, 0, h, w), (i, h - 1, w - 1, 1, 1), (i, 0, 0, 1, 1), (i, h - 1, 0, 1, w)]
    for _ in range(count):
        i = rs.randint(len(shapes))
        h, w = shapes[i]
        bh, bw = rs.randint(1, h + 1), rs.randint(1, w + 1)
        out.append((i, rs.randint(0, h - bh + 1), rs.randint(0, w - bw + 1), bh, bw))
    return out


def _check(codec, conts, regions, full, **kw):
    got = decompress_regions(codec, conts, regions, **kw)
    assert len(got) == len(regions)
    for (i, y, x, h, w), g in zip(regions, got):
        want = full[i][y:y + h, x:x + w]
        assert g.dtype == np.uint8 and g.flags.c_contiguous and g.shape == want.shape, (i, y, x, h, w)
        assert np.array_equal(g, want), (i, y, x, h, w)


CASES = [("tiny", BITSWAP, "crop"), ("tiny", BBANS, "code"), ("tiny3", BITSWAP, "code"), ("tiny3", BBANS, "crop")]


@pytest.mark.parametrize("name,scheme,edges", CASES)
def test_regions_equal_crops_of_the_whole_image(name, scheme, edges):
    """Many regions in one call and one region per call, at chain_blocks None, 3 and 5; the codec pops exactly the
    planned blocks."""
    cfg, _, sd, _, _, bins, codec = setup(name, 8)
    C = cfg.xs[0]
    sizes = [(33, 65), (70, 100), (97, 40), (130, 33)] if edges == "code" else [(70, 100), (64, 96), (130, 33)]
    images = random_images(C, sizes, seed=61)
    rs = np.random.RandomState(62)
    for L in (None, 3, 5):
        conts = compress_images(codec, images, excess_state_len=N_INIT, scheme=scheme, edges=edges, chain_blocks=L)
        full = decompress_images(codec, conts, channels=C, scheme=scheme)
        shapes = [f.shape[:2] for f in full]
        regions = _regions(rs, shapes, 12)
        counting = Counting(codec)
        _check(counting, conts, regions, full, channels=C, scheme=scheme)
        plans = plan_regions(conts, regions)
        assert counting.blocks == sum(int(p.depth.sum()) for p in plans)
        assert counting.calls == sum(-(-n // codec.max_batch) for n in container._active(
            sorted([d for p in plans for d in p.depth.tolist() if d], reverse=True)))
        for r in _regions(rs, shapes, 4)[-6:]:
            counting = Counting(codec)
            _check(counting, conts, [r], full, channels=C, scheme=scheme)
            assert counting.blocks == sum(int(p.depth.sum()) for p in plan_regions(conts, [r]))


def test_mixed_repeated_and_more_chains_than_max_batch():
    """Single- and multi-chain containers mixed and repeated, more streams than max_batch (three calls per step), through
    a BitSwapCodec and a free-running 2-lane PipelinedCodec; then an hwc_quirk crop container."""
    cfg, _, sd, _, _, bins, codec = setup("tiny3", 4)
    images = random_images(3, [(150, 130), (33, 65), (70, 100)], seed=63)             # 5 x 5, 2 x 3 and 3 x 4 blocks
    single = compress_images(codec, images, excess_state_len=N_INIT, edges="code")
    multi = compress_images(codec, images, excess_state_len=N_INIT, edges="code", chain_blocks=2)
    conts = [multi[0], single[1], multi[2], single[0], multi[0], single[2]]
    full = [images[0], images[1], images[2], images[0], images[0], images[2]]
    rs = np.random.RandomState(64)
    regions = _regions(rs, [f.shape[:2] for f in full], 16)
    plans = plan_regions(conts, regions)
    assert sum(int((p.depth > 0).sum()) for p in plans) > 3 * 4                 # more than three calls' worth of streams
    pc = PipelinedCodec(cfg, sd, bins, 4, lanes=2, use_tensor_cores=False, free_running=True)
    for c in (codec, pc):
        _check(c, conts, regions, full)
    quirk = compress_images(codec, images[:1], excess_state_len=N_INIT, hwc_quirk=True, chain_blocks=3)
    qfull = decompress_images(codec, quirk, hwc_quirk=True)
    assert qfull[0].shape == (128, 128, 3)
    _check(pc, quirk, _regions(rs, [(128, 128)], 6), qfull, hwc_quirk=True)


def test_imagenetcrop4_tensor_cores():
    cfg = preset("imagenetcrop4")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
    pc = PipelinedCodec(cfg, sd, bins, 8, lanes=2, use_tensor_cores=True, free_running=True)
    images = random_images(3, [(100, 200)], seed=65)                                   # 4 x 7 blocks: chains of 7, 7, 7, 7
    conts = compress_images(pc, images, excess_state_len=4000, edges="code", chain_blocks=8)
    full = decompress_images(pc, conts)
    assert np.array_equal(full[0], images[0])
    regions = [(0, 40, 50, 30, 100), (0, 99, 0, 1, 200), (0, 0, 190, 5, 10), (0, 10, 10, 80, 40)]
    counting = Counting(pc)
    _check(counting, conts, regions, full)
    assert counting.blocks == sum(int(p.depth.sum()) for p in plan_regions(conts, regions))


def _lone_states(codec, blocks, extents, scheme, n_init):
    """One chain encoded alone, one block per call: (its state list before each block and after the last, the lowest word
    count it reached)."""
    wds, head = synthetic.initial_words(n_init, seed=100)
    ss = StreamSet(1, n_init + 1400 * len(blocks) + 64, device=codec.device)
    ss.fill(wds, head)
    x = torch.from_numpy(np.ascontiguousarray(blocks.transpose(0, 3, 1, 2))).cuda()
    e = None if extents is None else torch.from_numpy(np.ascontiguousarray(extents, dtype=np.int16)).cuda()
    states = [ss.export_lists()[0]]
    for k in range(len(blocks)):
        codec.encode(ss, x[k:k + 1], scheme=scheme, extent=None if e is None else e[k:k + 1])
        torch.cuda.synchronize()
        states.append(ss.export_lists()[0])
    ss.raise_on_error()
    return states, int(ss.min_words()[0])


@pytest.mark.parametrize("scheme,edges", [(BITSWAP, "code"), (BBANS, "crop")])
def test_a_chain_stopped_part_way_holds_the_encoders_state(scheme, edges, monkeypatch):
    """After decoding a chain down to its earliest wanted block j, its stream holds the state the encoder had before block
    j, less the never-borrowed initial words the container trims."""
    cfg, _, sd, _, _, bins, codec = setup("tiny", 8)
    img = random_images(1, [(130, 97)], seed=66)[0]                                    # 5 x 4 blocks (4 x 3 cropped)
    L = 4
    conts = compress_images(codec, [img], excess_state_len=N_INIT, scheme=scheme, edges=edges, chain_blocks=L)
    if edges == "code":
        blocks, ext, h, w = extract_edge_blocks(img)
    else:
        (blocks, h, w), ext = extract_blocks(img), None
    sizes = chain_sizes(len(blocks), L)
    assert len(sizes) >= 3
    made = []

    class Recorded(StreamSet):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)
    monkeypatch.setattr(container, "StreamSet", Recorded)
    gw = block_grid(h, w)[1]
    regions = [(0, 33, 64, 1, 1), (0, 64, 32, 1, 1), (0, h - 1, w - 1, 1, 1)]   # blocks gw + 2, 2 gw + 1 and the last
    (plan,) = plan_regions(conts, regions)
    assert np.flatnonzero(plan.needed).tolist() == [gw + 2, 2 * gw + 1, len(blocks) - 1]
    decompress_regions(codec, conts, regions, channels=1, scheme=scheme)
    got = made[-1].export_lists()
    streams = [k for k in np.argsort(-plan.depth, kind="stable") if plan.depth[k]]
    assert len(got) == len(streams) and len(streams) >= 2 and any(0 < plan.first[k] for k in streams)
    starts = np.cumsum(sizes) - sizes
    for j, k in enumerate(streams):
        s, nb = int(starts[k]), sizes[k]
        states, lo = _lone_states(codec, blocks[s:s + nb], None if ext is None else ext[s:s + nb], scheme, N_INIT)
        assert got[j] == states[int(plan.first[k])][lo:], (k, int(plan.first[k]))
