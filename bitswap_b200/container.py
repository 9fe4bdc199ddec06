"""Variable-size images as chained 32x32 block streams + the reference's demo container format.

Reference: block tiling `extract_blocks` / `unextract_blocks` (benchmark_compress.py:20-39), the demo codec
(demo_compress.py:72-162 compress, :268-284 file format; demo_decompress.py:69-148, :216-227).  One image =
ONE ANS chain over its blocks (imagenetcrop_compress.py:127-210); different images are independent chains, so
a set of images is coded as a StreamSet with one stream per image: step t codes block t of every image that
has more than t blocks (images are ordered by block count so the active streams are always a prefix).

Container (np.uint32 array, what demo_compress.py saves with np.save):
    [ words that were actually borrowed or produced ..., head_lo, head_hi, nblocks, h, w ]
Blocks are fed CHW like the demo path does (demo_compress.py:120).  `hwc_quirk=True` reproduces
imagenetcrop_compress.py:130 instead, which flattens each [32,32,3] HWC block straight into the CHW model's input
(`torch.from_numpy(x).view(xdim)`) -- the layout behind the README's ImageNet-crop numbers.

Edges: the reference crops every image down to multiples of 32 (`edges="crop"`, the default).  `edges="code"` keeps the
whole image: it is tiled into ceil(H/32) x ceil(W/32) blocks, and a block on the bottom or right edge codes only the
pixels inside its valid extent (vh, vw) = (min(32, H - 32 by), min(32, W - 32 bx)) (bsw_codec_encode_ext).  The tail then
holds the true H and W; an image whose sides are multiples of 32 gives the same container in both modes, and a header
with a side off a multiple of 32 (which the crop mode never writes) is what marks an edge-coded container.
"""
import numpy as np
import torch

from .codec import BITSWAP
from .streams import StreamSet
from .synthetic import initial_words


def extract_blocks(arr, block_size=(32, 32)):
    """HWC uint8 image -> (blocks [n, 32, 32, C] row-major over the block grid, h, w) with h, w cropped down to
    multiples of the block size (benchmark_compress.py:20-31)."""
    bh, bw = block_size
    h, w, c = arr.shape
    h -= h % bh
    w -= w % bw
    arr = arr[:h, :w]
    blocks = arr.reshape(h // bh, bh, w // bw, bw, c).swapaxes(1, 2).reshape(-1, bh, bw, c)
    return blocks, h, w


def unextract_blocks(blocks, h, w):
    """Inverse of extract_blocks (benchmark_compress.py:35-39)."""
    n, bh, bw, c = blocks.shape
    return blocks.reshape(h // bh, w // bw, bh, bw, c).swapaxes(1, 2).reshape(h, w, c)


def block_grid(h, w):
    """Blocks per column and per row of an h x w image tiled with partial edge blocks."""
    return -(-h // 32), -(-w // 32)


def block_extents(h, w):
    """int16 [n, 2] valid extents (vh, vw) of the row-major blocks of an h x w image tiled with partial edge blocks."""
    gh, gw = block_grid(h, w)
    vh = np.minimum(32, h - 32 * np.arange(gh))
    vw = np.minimum(32, w - 32 * np.arange(gw))
    return np.stack(np.broadcast_arrays(vh[:, None], vw[None, :]), axis=-1).reshape(-1, 2).astype(np.int16)


def extract_edge_blocks(arr):
    """HWC uint8 image (any H, W >= 1) -> (blocks [n, 32, 32, C] row-major over the ceil(H/32) x ceil(W/32) grid,
    extents int16 [n, 2], h, w).  Pixels outside a block's extent are edge-replicated here for definiteness; the codec
    ignores them and applies the same rule itself."""
    h, w, c = arr.shape
    gh, gw = block_grid(h, w)
    padded = np.pad(arr, ((0, 32 * gh - h), (0, 32 * gw - w), (0, 0)), mode="edge")
    blocks, _, _ = extract_blocks(padded)
    return blocks, block_extents(h, w), h, w


def unextract_edge_blocks(blocks, h, w):
    """Inverse of extract_edge_blocks: the h x w image from its (padded) blocks."""
    gh, gw = block_grid(h, w)
    return np.ascontiguousarray(unextract_blocks(blocks, 32 * gh, 32 * gw)[:h, :w])


def _blocks_to_model(blocks, hwc_quirk):
    """[n,32,32,C] HWC blocks -> [n,C,32,32] model input."""
    n, bh, bw, c = blocks.shape
    return blocks.reshape(n, c, bh, bw) if hwc_quirk else blocks.transpose(0, 3, 1, 2)


def _model_to_blocks(x, hwc_quirk):
    n, c, bh, bw = x.shape
    return np.ascontiguousarray(x).reshape(n, bh, bw, c) if hwc_quirk else np.ascontiguousarray(x.transpose(0, 2, 3, 1))


def compress_images(codec, images, excess_state_len=10000, seed=100, scheme=BITSWAP, hwc_quirk=False, words_per_block=1400,
                    edges="crop"):
    """images: list of HWC uint8 arrays.  Returns one container array per image.
    Every chain starts from the reference's initial state: `excess_state_len` random words drawn with
    np.random.seed(100) (demo_compress.py:113-115, :202).
    edges="crop" (the reference's behaviour): every image is cropped down to multiples of 32 and must be at least 32x32.
    edges="code": the whole image (any H, W >= 1) is coded, with partial blocks at the bottom and right edges;
    decompress_images returns it exactly."""
    if edges not in ("crop", "code"):
        raise ValueError(f"edges must be 'crop' or 'code', got {edges!r}")
    if edges == "code" and hwc_quirk:
        raise ValueError("edges='code' needs the CHW block layout: hwc_quirk scrambles the rows and columns the extents refer to")
    images = [np.asarray(im) for im in images]
    if edges == "code":
        tiled = [extract_edge_blocks(im) for im in images]
    else:
        tiled = [(b, None, h, w) for b, h, w in (extract_blocks(im) for im in images)]
    order = sorted(range(len(images)), key=lambda i: (-tiled[i][0].shape[0], i))
    nblk = [tiled[i][0].shape[0] for i in order]
    n = len(images)
    w, head = initial_words(excess_state_len, seed=seed)
    # capacity: `words_per_block` words per 32x32 block (1400 = 14.6 bits/dim; 8 bits/dim of raw pixels is 768).  A chain
    # that still overflows is retried with twice the room instead of failing after the whole chain was coded.
    for attempt in range(4):
        ss = StreamSet(n, excess_state_len + (words_per_block << attempt) * max(nblk) + 64, device=codec.device)
        ss.fill(w, head)
        try:
            return _compress_chains(codec, ss, tiled, order, nblk, scheme, hwc_quirk)
        except OverflowError:
            if attempt == 3:
                raise
    raise AssertionError("unreachable")


def _compress_chains(codec, ss, tiled, order, nblk, scheme, hwc_quirk):
    n = len(order)
    # all blocks to the device once: [step t, stream j] = block t of the j-th largest image (CHW, demo_compress.py:120)
    C = tiled[order[0]][0].shape[-1]
    host = np.zeros((max(nblk), n, C, 32, 32), dtype=np.uint8)
    for j, i in enumerate(order):
        host[:nblk[j], j] = _blocks_to_model(tiled[i][0], hwc_quirk)
    dev = torch.from_numpy(host).to(torch.device("cuda", codec.device))
    ext = _extents_to_device(codec, [tiled[i][1] for i in order], nblk)
    for t in range(max(nblk)):
        active = sum(1 for b in nblk if b > t)
        codec.encode(ss, dev[t, :active].contiguous(), first=0, scheme=scheme,
                     extent=None if ext is None else ext[t, :active].contiguous())
    torch.cuda.synchronize()
    ss.raise_on_error()
    words, offs, heads, _ = ss.export()
    lo = ss.min_words()                                       # never-borrowed initial words (demo_compress.py:137,160)
    out = [None] * n
    for j, i in enumerate(order):
        ws = words[offs[j] + lo[j]:offs[j + 1]]
        hd = int(heads[j])
        _, _, h, wd = tiled[i]
        tail = np.array([hd & 0xffffffff, hd >> 32, nblk[j], h, wd], dtype=np.uint32)           # demo_compress.py:272-279
        out[i] = np.concatenate([ws.astype(np.uint32), tail])
    return out


def _extents_to_device(codec, extents, nblk):
    """[step t, stream j] block extents as one int16 device tensor, or None when every block is full (then the plain
    calls run, which code exactly what full extents would)."""
    if all(e is None or (e == 32).all() for e in extents):
        return None
    host = np.full((max(nblk), len(nblk), 2), 32, dtype=np.int16)
    for j, e in enumerate(extents):
        if e is not None:
            host[:nblk[j], j] = e
    return torch.from_numpy(host).to(torch.device("cuda", codec.device))


def decompress_images(codec, containers, channels=3, scheme=BITSWAP, hwc_quirk=False, headroom_words=None):
    """Inverse of compress_images: list of container arrays -> list of HWC uint8 images (the cropped size for a crop-mode
    container, the full size for an edge-coded one: a header whose h or w is not a multiple of 32)."""
    meta = []
    for c in containers:
        c = np.asarray(c, dtype=np.uint32)
        if c.ndim != 1 or c.size < 5:
            raise ValueError(f"container too short ({c.size} words): needs at least head_lo, head_hi, nblocks, h, w")
        nblocks, h, w = int(c[-3]), int(c[-2]), int(c[-1])                                      # demo_decompress.py:216-219
        if h <= 0 or w <= 0 or nblocks != np.prod(block_grid(h, w)) or nblocks > (1 << 20):
            raise ValueError(f"inconsistent container header: nblocks={nblocks}, h={h}, w={w}")
        if hwc_quirk and (h % 32 or w % 32):
            raise ValueError(f"edge-coded container (h={h}, w={w}) cannot be decoded with hwc_quirk")
        head = (int(c[-4]) << 32) | int(c[-5])                                                  # :222
        meta.append((c[:-5], head, nblocks, h, w))
    order = sorted(range(len(containers)), key=lambda i: (-meta[i][2], i))
    nblk = [meta[i][2] for i in order]
    n = len(containers)
    # The receiver pushes too (it returns the borrowed bits, cifar_compress.py:306-313): one block's worth of latents,
    # nz * zdim symbols at <= 31 bits each, can sit on the stack above the container's own length.
    if headroom_words is None:
        headroom_words = codec.cfg.nz * codec.cfg.zdim + 64
    ss = StreamSet(n, max(len(meta[i][0]) for i in order) + headroom_words, device=codec.device)
    ss.import_lists([[int(v) for v in meta[i][0]] + [meta[i][1]] for i in order])
    dev = torch.zeros((max(nblk), n, channels, 32, 32), dtype=torch.uint8, device=torch.device("cuda", codec.device))
    ext = _extents_to_device(codec, [block_extents(meta[i][3], meta[i][4]) for i in order], nblk)
    for t in reversed(range(max(nblk))):
        active = sum(1 for b in nblk if b > t)
        codec.decode(ss, active, first=0, scheme=scheme, out=dev[t, :active],
                     extent=None if ext is None else ext[t, :active].contiguous())
    if hasattr(codec, "join"):                                             # (free-running multi-lane codec: lanes -> current stream)
        codec.join()
    host = dev.cpu().numpy()                                               # one transfer for every block of every image
    blocks = [_model_to_blocks(host[:nblk[j], j], hwc_quirk) for j in range(n)]
    ss.raise_on_error()
    out = [None] * n
    for j, i in enumerate(order):
        out[i] = unextract_edge_blocks(blocks[j], meta[i][3], meta[i][4])
    return out
