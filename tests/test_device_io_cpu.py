"""Images in and out of the block buffers, without a GPU: a numpy twin of the tile and untile kernels' index math (binary
searches over the image, chain and region offsets the C side builds from its host tables) reproduces the placement the
writers and readers made with the reference tiling, row by row and pixel by pixel, and the C ABI refuses every malformed
table field with BSW_E_INVALID before anything reaches the device."""
import ctypes

import numpy as np
import pytest

from device_io_harness import _grid, _ioff, tile_rows, tile_twin, untile_twin
from bitswap_b200 import container
from bitswap_b200._lib import lib
from bitswap_b200.container import (MAX_BLOCKS, TILE_CODE, TILE_CROP, TILE_QUIRK, _VIEW, _blocks_to_model, _chain_runs,
                                    _Job, _plan, _sequence_extents, block_extents, chain_sizes, extract_blocks,
                                    extract_edge_blocks)

SIZES = [(1, 1), (1, 33), (31, 32), (32, 32), (33, 65), (28, 28), (100, 70)]
BSW_E_INVALID = 4


# ---- the placement before the kernels: the reference tiling, laid out and cut on the host ---------------------------------
def host_tiling(images, mode):
    tiles = [extract_edge_blocks(im) if mode == TILE_CODE else extract_blocks(im)[:1] + (None,) for im in images]
    blocks = np.concatenate([_blocks_to_model(t[0], mode == TILE_QUIRK) for t in tiles])
    return blocks, (np.concatenate([t[1] for t in tiles]) if mode == TILE_CODE else None)


def host_placement(blocks, extents, chains, order):
    """[t, j] = block t of the j-th largest chain, as the encoder placed it (written rows only: a mask)."""
    steps = max(nb for _, nb in chains)
    x = np.zeros((steps, len(order)) + blocks.shape[1:], dtype=np.uint8)
    e = np.full((steps, len(order), 2), 32, dtype=np.int16)
    mask = np.zeros((steps, len(order)), dtype=bool)
    for j, c in enumerate(order):
        s, nb = chains[c]
        x[:nb, j] = blocks[s:s + nb]
        if extents is not None:
            e[:nb, j] = extents[s:s + nb]
        mask[:nb, j] = True
    return x, e, mask


def host_cut(job, regions, x, quirk):
    """The regions as the decoder cut them from x: gather the needed blocks, untile them, crop."""
    regions, plan = _plan(job, regions)
    order = np.argsort(-plan.depth, kind="stable")[:np.count_nonzero(plan.depth)]
    n, C = len(order), x.shape[2]
    stream = np.full(len(job.cnb), -1, dtype=np.int64)
    stream[order] = np.arange(n)
    b = np.flatnonzero(plan.needed)
    c = np.searchsorted(job.cstart + job.cnb, b, side="right")
    pos = np.full(plan.needed.size, -1, dtype=np.int64)
    pos[b] = np.arange(b.size)
    got = x.reshape(-1, C, 32, 32)[(job.cstart[c] + job.cnb[c] - 1 - b) * n + stream[c]]
    host = got.reshape(-1, 32, 32, C) if quirk else got.transpose(0, 2, 3, 1)
    out = []
    for i, y, x0, h, w in regions:
        gw = -(-job.shapes[i][1] // 32)
        by, bx = np.arange(y // 32, (y + h - 1) // 32 + 1), np.arange(x0 // 32, (x0 + w - 1) // 32 + 1)
        sel = host[pos[job.ioff[i] + by[:, None] * gw + bx[None, :]].reshape(-1)]
        tile = sel.reshape(by.size, bx.size, 32, 32, C).swapaxes(1, 2).reshape(32 * by.size, 32 * bx.size, C)
        out.append(tile[y - 32 * by[0]:y - 32 * by[0] + h, x0 - 32 * bx[0]:x0 - 32 * bx[0] + w])
    return out, order, stream


def _layout(shapes, mode, L, archive):
    """(chains [(start, nb)] in sequence order, cnb, stream, order) as compress_images / compress_archive cut them."""
    nb = np.array([int(np.prod(_grid(h, w, mode))) for h, w in shapes], dtype=np.int64)
    cnb = np.array(chain_sizes(int(nb.sum()), L), dtype=np.int64) if archive else _chain_runs(nb, L)[1]
    order = np.argsort(-cnb, kind="stable")
    stream = np.empty(len(cnb), dtype=np.int32)
    stream[order] = np.arange(len(cnb))
    return list(zip((np.cumsum(cnb) - cnb).tolist(), cnb.tolist())), cnb, stream, order


CASES = [(mode, C, L, archive) for mode in (TILE_CROP, TILE_CODE, TILE_QUIRK) for C in (1, 3)
         for L in (None, 1, 3, 7, 32) for archive in ((False, True) if mode == TILE_CODE else (False,))]


@pytest.mark.parametrize("mode,C,L,archive", CASES)
def test_the_tile_twin_places_every_row_as_the_encoder_did(mode, C, L, archive):
    rs = np.random.RandomState(C + 7 * (L or 0))
    images = [rs.randint(0, 256, (h, w, C)).astype(np.uint8) for h, w in SIZES]
    chains, cnb, stream, order = _layout(SIZES, mode, L, archive)
    if archive and L in (3, 7):                                        # some chain crosses an image boundary
        ends = set(_ioff(SIZES, mode)[1:].tolist())
        assert any(not {s + d for d in range(1, nb)}.isdisjoint(ends) for s, nb in chains)
    blocks, extents = host_tiling(images, mode)
    want, want_e, mask = host_placement(blocks, extents, chains, order)
    got, got_e = tile_twin(images, mode, cnb, stream, int(cnb.max()))
    assert np.array_equal(got[mask], want[mask])
    assert (got[~mask] == 0xAB).all()                                   # rows past a chain's end are not written
    if mode == TILE_CODE:
        assert np.array_equal(got_e[mask], want_e[mask])
        assert np.array_equal(_sequence_extents(np.array(SIZES, dtype=np.int64)),
                              np.concatenate([block_extents(h, w) for h, w in SIZES]))
    assert np.array_equal(container._Blocks(_Stub(C), images, mode, strict=False).__array__(), blocks)


@pytest.mark.parametrize("L", [None, 1, 32])
def test_the_tile_rows_of_a_2048_x_1536_image_and_its_neighbours(L):
    shapes = [(33, 65), (1536, 2048), (1, 1)]
    chains, cnb, stream, order = _layout(shapes, TILE_CODE, L, archive=True)
    t, j, i, by, bx, vh, vw = tile_rows(shapes, TILE_CODE, cnb, stream)
    chain_of = np.argsort(stream)
    seq = np.array([chains[c][0] for c in chain_of])[j] + t                # the encoder's row (t, j): block start + t
    gws = np.array([_grid(*s, TILE_CODE)[1] for s in shapes])
    assert np.array_equal(_ioff(shapes, TILE_CODE)[i] + by * gws[i] + bx, seq)
    assert sorted(seq.tolist()) == list(range(int(cnb.sum())))           # every block exactly once
    assert np.array_equal(np.stack([vh, vw], -1)[np.argsort(seq)], _sequence_extents(np.array(shapes, dtype=np.int64)))


def _regions(shapes, rs):
    regs = [(i, 0, 0, h, w) for i, (h, w) in enumerate(shapes)]
    for i, (h, w) in enumerate(shapes):
        for y, x in ((0, 0), (min(31, h - 1), min(31, w - 1)), (min(32, h - 1), min(32, w - 1)), (h - 1, w - 1),
                     (0, min(31, w - 1))):
            regs.append((i, y, x, 1, 1))                                   # 1 x 1 at block corners
        regs += [(i, 0, 0, min(h, 7), min(w, 5)), (i, 1, 2, min(h - 1, 3) or 1, min(w - 2, 30) if w > 2 else 1)]
        bh, bw = rs.randint(1, h + 1), rs.randint(1, w + 1)
        regs.append((i, rs.randint(0, h - bh + 1), rs.randint(0, w - bw + 1), bh, bw))
    return [r for r in regs if r[1] + r[3] <= shapes[r[0]][0] and r[2] + r[4] <= shapes[r[0]][1]]


@pytest.mark.parametrize("quirk,C,L,archive", [(q, C, L, a) for q in (False, True) for C in (1, 3) for L in (None, 1, 3, 7, 32)
                                               for a in ((False, True) if not q else (False,))])
def test_the_untile_twin_cuts_every_region_as_the_decoder_did(quirk, C, L, archive):
    rs = np.random.RandomState(11 + C + (L or 0))
    shapes = [(32, 64), (96, 32), (64, 64)] if quirk else SIZES
    chains, cnb, stream, order = _layout(shapes, TILE_CODE, L, archive)
    cstart = np.cumsum(cnb) - cnb
    job = _Job(None, None, cstart, cnb, shapes, _ioff(shapes, TILE_CODE))
    regions = _regions(shapes, rs)
    for regs in [regions, regions[len(shapes):len(shapes) + 6], [regions[-1]]]:   # partial decodes skip and shorten chains
        plan = _plan(job, regs)[1]
        depth = int(plan.depth.max())
        n = int(np.count_nonzero(plan.depth))
        x = rs.randint(0, 256, (depth, n, C, 32, 32)).astype(np.uint8)
        want, order, stream = host_cut(job, regs, x, quirk)
        got = untile_twin(shapes, TILE_QUIRK if quirk else TILE_CODE, cnb, stream.astype(np.int64), x, regs)
        assert np.array_equal(got, np.concatenate([w.reshape(-1) for w in want]))


# ---- the C ABI's host validation ------------------------------------------------------------------------------------------
FAKE = 1 << 40                               # never dereferenced: every call below is refused before anything is enqueued


class _Stub:
    def __init__(self, C):
        self.cfg = type("cfg", (), {"xs": [C]})()


def _tile_call(views=None, n_images=None, channels=3, mode=TILE_CODE, cnb=None, stream=None, n_chains=None, steps=7,
               blocks=FAKE, ext=FAKE, null=()):
    if views is None:
        views = np.zeros(2, dtype=_VIEW)
        views["pixels"] = FAKE
        views["h"], views["w"] = (33, 100), (65, 70)                     # 2 x 3 + 4 x 3 = 18 blocks
        views["sy"], views["sx"], views["sc"] = (65 * 3, 70 * 3), 3, 1
    cnb = np.array([7, 6, 5], dtype=np.int64) if cnb is None else np.asarray(cnb, dtype=np.int64)
    stream = np.array([0, 1, 2], dtype=np.int32) if stream is None else np.asarray(stream, dtype=np.int32)
    args = dict(images=views.ctypes.data, cnb=cnb.ctypes.data, stream=stream.ctypes.data, blocks=blocks)
    for k in null:
        args[k] = None
    return lib().bsw_tile_blocks(args["images"], len(views) if n_images is None else n_images, channels, mode, args["cnb"],
                                 args["stream"], len(cnb) if n_chains is None else n_chains, steps, args["blocks"], ext, None)


def _views(**change):
    v = np.zeros(2, dtype=_VIEW)
    v["pixels"] = FAKE
    v["h"], v["w"] = (33, 100), (65, 70)
    v["sy"], v["sx"], v["sc"] = (65 * 3, 70 * 3), 3, 1
    for k, val in change.items():
        v[k][1] = val
    return v


TILE_BAD = {
    "no images": dict(n_images=0), "no chains": dict(n_chains=0), "no steps": dict(steps=0),
    "channels 0": dict(channels=0), "channels 5": dict(channels=5), "mode": dict(mode=3),
    "null images": dict(null=("images",)), "null chain blocks": dict(null=("cnb",)), "null streams": dict(null=("stream",)),
    "null buffer": dict(null=("blocks",)), "null pixels": dict(views=_views(pixels=0)), "h 0": dict(views=_views(h=0)),
    "w 0": dict(views=_views(w=0)), "h < 0": dict(views=_views(h=-5)), "sy < 0": dict(views=_views(sy=-1)),
    "sx < 0": dict(views=_views(sx=-3)), "sc < 0": dict(views=_views(sc=-1)),
    "too many blocks": dict(views=_views(h=32 * 1025, w=32 * 1024)),
    "negative chain": dict(cnb=[7, 6, -1, 6]), "chains short": dict(cnb=[7, 6, 4]), "chains long": dict(cnb=[7, 6, 6]),
    "chains past the end": dict(cnb=[7, 6, 5, 1]), "stream repeated": dict(stream=[0, 1, 1]),
    "stream out of range": dict(stream=[0, 1, 3]), "stream negative": dict(stream=[0, -1, 2]),
    "chain longer than steps": dict(steps=6),
}


@pytest.mark.parametrize("case", sorted(TILE_BAD))
def test_tile_refuses_a_malformed_table(case):
    assert _tile_call(**TILE_BAD[case]) == BSW_E_INVALID


def test_tile_refuses_crop_blocks_over_the_limit():
    assert _tile_call(views=_views(h=32 * 1025 + 31, w=32 * 1024 + 31), mode=TILE_CROP) == BSW_E_INVALID
    assert MAX_BLOCKS == 1 << 20


def _untile_call(shapes=((33, 65), (100, 70)), channels=3, mode=TILE_CODE, cnb=(7, 6, 5), stream=(0, 1, 2), n_streams=3,
                 steps=7, regions=((0, 0, 0, 33, 65), (1, 5, 5, 10, 10)), n_images=None, n_chains=None, n_regions=None,
                 null=()):
    shapes = np.ascontiguousarray(shapes, dtype=np.int32).reshape(-1, 2)
    cnb = np.ascontiguousarray(cnb, dtype=np.int64)
    stream = np.ascontiguousarray(stream, dtype=np.int32)
    regions = np.ascontiguousarray(regions, dtype=np.int32).reshape(-1, 5)
    p = dict(shapes=shapes.ctypes.data, cnb=cnb.ctypes.data, stream=stream.ctypes.data, blocks=FAKE,
             regions=regions.ctypes.data, out=FAKE)
    for k in null:
        p[k] = None
    return lib().bsw_untile_regions(p["shapes"], len(shapes) if n_images is None else n_images, channels, mode, p["cnb"],
                                    p["stream"], len(cnb) if n_chains is None else n_chains, n_streams, steps, p["blocks"],
                                    p["regions"], len(regions) if n_regions is None else n_regions, p["out"], None)


UNTILE_BAD = {
    "no images": dict(n_images=0), "no chains": dict(n_chains=0), "no streams": dict(n_streams=0), "no steps": dict(steps=0),
    "no regions": dict(n_regions=0), "channels 0": dict(channels=0), "channels 5": dict(channels=5), "mode": dict(mode=-1),
    "null shapes": dict(null=("shapes",)), "null chain blocks": dict(null=("cnb",)), "null streams": dict(null=("stream",)),
    "null buffer": dict(null=("blocks",)), "null regions": dict(null=("regions",)), "null out": dict(null=("out",)),
    "h 0": dict(shapes=((0, 65), (100, 70))), "w 0": dict(shapes=((33, 65), (100, 0))),
    "too many blocks": dict(shapes=((33, 65), (32 * 1025, 32 * 1024))), "chains short": dict(cnb=(7, 6, 4)),
    "chains long": dict(cnb=(7, 6, 6)), "negative chain": dict(cnb=(7, 6, -1, 6), stream=(0, 1, 2, 2)),
    "stream < -1": dict(stream=(0, -2, 2)), "stream >= n_streams": dict(stream=(0, 1, 3)),
    "region of no image": dict(regions=((2, 0, 0, 1, 1),)), "region of image -1": dict(regions=((-1, 0, 0, 1, 1),)),
    "region h 0": dict(regions=((0, 0, 0, 0, 1),)), "region w 0": dict(regions=((0, 0, 0, 1, 0),)),
    "region y < 0": dict(regions=((0, -1, 0, 1, 1),)), "region x < 0": dict(regions=((0, 0, -1, 1, 1),)),
    "region leaves the bottom": dict(regions=((0, 30, 0, 4, 1),)), "region leaves the right": dict(regions=((1, 0, 69, 1, 2),)),
    "region outside the crop": dict(mode=TILE_CROP, cnb=(3, 3, 2), steps=3,
                                    regions=((0, 32, 0, 1, 1),)),
    "region of an undecoded chain": dict(stream=(0, -1, 2), regions=((1, 0, 32, 1, 1),)),
    "region below the decoded steps": dict(steps=3, regions=((0, 0, 0, 1, 1),)),
}


@pytest.mark.parametrize("case", sorted(UNTILE_BAD))
def test_untile_refuses_a_malformed_table(case):
    assert _untile_call(**UNTILE_BAD[case]) == BSW_E_INVALID


def test_the_abi_declares_the_view_as_the_python_records_lay_it_out():
    assert _VIEW.itemsize == 40 and [_VIEW.fields[f][1] for f in _VIEW.names] == [0, 8, 12, 16, 24, 32]
    assert ctypes.sizeof(ctypes.c_void_p) == 8
