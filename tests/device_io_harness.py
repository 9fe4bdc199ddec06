"""A numpy twin of the tile and untile kernels (bitswap_b200/csrc/tiles.cu) -- TEST INFRASTRUCTURE: the same binary searches
over the image, chain and region offsets the C side builds from its host tables, element by element."""
import numpy as np

from bitswap_b200.container import TILE_CODE, TILE_QUIRK


def _grid(h, w, mode):
    return (-(-h // 32), -(-w // 32)) if mode == TILE_CODE else (h // 32, w // 32)


def _ioff(shapes, mode):
    return np.concatenate([[0], np.cumsum([int(np.prod(_grid(h, w, mode))) for h, w in shapes])]).astype(np.int64)


# ---- the kernels' index math, in numpy ---------------------------------------------------------------------------------------
def tile_rows(shapes, mode, cnb, stream):
    """Rows k_tile_blocks writes: (t, j, image i, block row by, block column bx, vh, vw) per coded block, one CTA each."""
    ioff, K = _ioff(shapes, mode), len(cnb)
    chain_of = np.argsort(stream)                                       # stream j holds chain chain_of[j]
    cum = np.concatenate([[0], np.cumsum(cnb[chain_of])])
    sstart = (np.cumsum(cnb) - cnb)[chain_of]
    q = np.arange(cum[-1])
    j = np.searchsorted(cum[:K], q, side="right") - 1
    t = q - cum[j]
    g = sstart[j] + t
    i = np.searchsorted(ioff[:-1], g, side="right") - 1
    h, w = np.asarray(shapes, dtype=np.int64)[i].T
    gw = np.array([_grid(*s, mode)[1] for s in shapes], dtype=np.int64)[i]
    b = g - ioff[i]
    by, bx = b // gw, b % gw
    return t, j, i, by, bx, np.minimum(32, h - 32 * by), np.minimum(32, w - 32 * bx)


def tile_twin(images, mode, cnb, stream, steps):
    """What bsw_tile_blocks writes: blocks [steps, K, C, 32, 32] and extents [steps, K, 2]; unwritten rows keep 0xAB / -1."""
    C = images[0].shape[2]
    x = np.full((steps, len(cnb), C, 32, 32), 0xAB, dtype=np.uint8)
    ext = np.full((steps, len(cnb), 2), -1, dtype=np.int16)
    ar = np.arange(32)
    for t, j, i, by, bx, vh, vw in zip(*tile_rows([im.shape[:2] for im in images], mode, cnb, stream)):
        blk = images[i][32 * by + np.minimum(ar, vh - 1)[:, None], 32 * bx + np.minimum(ar, vw - 1)[None, :]]    # [32, 32, C]
        x[t, j] = blk.reshape(C, 32, 32) if mode == TILE_QUIRK else blk.transpose(2, 0, 1)
        ext[t, j] = (vh, vw)
    return x, ext


def untile_twin(shapes, mode, cnb, stream, x, regions):
    """What bsw_untile_regions writes: every region as contiguous HWC, in turn, in one flat buffer."""
    S, n, C = x.shape[:3]
    ioff, K = _ioff(shapes, mode), len(cnb)
    gws = np.array([_grid(h, w, mode)[1] for h, w in shapes], dtype=np.int64)
    cstart = np.concatenate([[0], np.cumsum(cnb)])
    regs = np.asarray(regions, dtype=np.int64).reshape(-1, 5)
    roff = np.concatenate([[0], np.cumsum(regs[:, 3] * regs[:, 4])])
    p = np.arange(roff[-1])
    r = np.searchsorted(roff[:-1], p, side="right") - 1
    i, y, x0, _, w = regs[r].T
    loc = p - roff[r]
    Y, X = y + loc // w, x0 + loc % w
    g = ioff[i] + (Y >> 5) * gws[i] + (X >> 5)
    c = np.searchsorted(cstart[:K], g, side="right") - 1
    base = ((cstart[c + 1] - 1 - g) * n + stream[c]) * C * 1024
    pix = (Y & 31) * 32 + (X & 31)
    ch = np.arange(C)
    idx = base[:, None] + (pix[:, None] * C + ch if mode == TILE_QUIRK else ch * 1024 + pix[:, None])
    return x.reshape(-1)[idx].reshape(-1)
