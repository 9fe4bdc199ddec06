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

Chains: one chain is serial (block t+1 starts from the state block t left), so coding time grows with an image's block
count.  `chain_blocks=L` splits an image of n blocks into K = ceil(n / L) contiguous runs of its row-major blocks and codes
each run as its own chain from the reference's seeded initial state; the K chains run side by side as K streams.  Each
chain is exactly what the demo procedure writes for its run of blocks, and each keeps its own borrowed initial words, so
more chains cost more bits.  K = 1 is the reference layout above; K >= 2 is written as
    [ words_0 ... | ... | words_{K-1} ... | (nwords_k, head_lo_k, head_hi_k, nblocks_k) for k < K | K, h, w, CHAIN_MARK ]
CHAIN_MARK >= 2^31 sits where the reference layout has w, so a reader of that layout alone sees an impossible header.

Regions: a chain is a stack, so decoding pops its blocks last to first; to reach block j of a chain of n blocks the decoder
pops n - j blocks and no further, and a chain none of whose blocks is wanted is not imported at all.  decompress_regions
decodes only that (plan_regions says how much), and decompress_images is the same path with one whole-image region per
container.
"""
import collections
import numbers

import numpy as np
import torch

from .codec import BITSWAP
from .streams import StreamSet
from .synthetic import initial_words

CHAIN_MARK = 0x8043484E                  # bit 31 | "CHN": last word of a multi-chain container
MAX_BLOCKS = 1 << 20                     # blocks per image a container may declare


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


def chain_sizes(nblocks, chain_blocks=None):
    """Block counts of the chains an image of `nblocks` row-major blocks is coded as, in block order: K = ceil(nblocks /
    chain_blocks) contiguous runs whose sizes differ by at most one, larger runs first.  None, or chain_blocks >= nblocks:
    one chain (the reference layout)."""
    if chain_blocks is None or chain_blocks >= nblocks:
        return [nblocks]
    k = -(-nblocks // chain_blocks)
    q, r = divmod(nblocks, k)
    return [q + 1] * r + [q] * (k - r)


def _check_chain_blocks(chain_blocks):
    if chain_blocks is None:
        return None
    if isinstance(chain_blocks, bool) or not isinstance(chain_blocks, numbers.Integral) or chain_blocks < 1:
        raise ValueError(f"chain_blocks must be None or a positive int, got {chain_blocks!r}")
    return int(chain_blocks)


def _sub_ranges(active, max_batch):
    """(first, count) calls covering streams [0, active) with at most max_batch streams each.  The boundaries are multiples
    of max_batch whatever `active` is, so a stream always lands at the same offset of a call: a free-running
    PipelinedCodec then codes it on the same lane at every step."""
    return [(b, min(max_batch, active - b)) for b in range(0, active, max_batch)]


def _active(nblk):
    """Streams still coding at each step t, for block counts sorted largest first: the active streams are a prefix."""
    return np.searchsorted(-np.asarray(nblk), -np.arange(max(nblk)), side="left")


def compress_images(codec, images, excess_state_len=10000, seed=100, scheme=BITSWAP, hwc_quirk=False, words_per_block=1400,
                    edges="crop", chain_blocks=None):
    """images: list of HWC uint8 arrays.  Returns one container array per image.
    Every chain starts from the reference's initial state: `excess_state_len` random words drawn with
    np.random.seed(100) (demo_compress.py:113-115, :202).
    edges="crop" (the reference's behaviour): every image is cropped down to multiples of 32 and must be at least 32x32.
    edges="code": the whole image (any H, W >= 1) is coded, with partial blocks at the bottom and right edges;
    decompress_images returns it exactly.
    chain_blocks: None (the reference's one chain per image) or a positive int L: an image of n > L blocks is coded as
    ceil(n / L) chains of contiguous blocks (chain_sizes), which run side by side.  Fewer serial steps, more initial bits."""
    if edges not in ("crop", "code"):
        raise ValueError(f"edges must be 'crop' or 'code', got {edges!r}")
    if edges == "code" and hwc_quirk:
        raise ValueError("edges='code' needs the CHW block layout: hwc_quirk scrambles the rows and columns the extents refer to")
    chain_blocks = _check_chain_blocks(chain_blocks)
    images = [np.asarray(im) for im in images]
    if edges == "code":
        tiled = [extract_edge_blocks(im) for im in images]
    else:
        tiled = [(b, None, h, w) for b, h, w in (extract_blocks(im) for im in images)]
    # chains (image, first block, blocks) in image and block order; streams hold them largest first
    chains = []
    for i, t in enumerate(tiled):
        sizes = chain_sizes(t[0].shape[0], chain_blocks)
        chains += [(i, s, nb) for s, nb in zip(np.cumsum([0] + sizes[:-1]).tolist(), sizes)]
    order = sorted(range(len(chains)), key=lambda c: (-chains[c][2], c))
    nblk = [chains[c][2] for c in order]
    w, head = initial_words(excess_state_len, seed=seed)
    # capacity: `words_per_block` words per 32x32 block of the longest chain (1400 = 14.6 bits/dim; 8 bits/dim of raw pixels
    # is 768).  A chain that still overflows is retried with twice the room instead of failing after it was coded.
    for attempt in range(4):
        ss = StreamSet(len(chains), excess_state_len + (words_per_block << attempt) * max(nblk) + 64, device=codec.device)
        ss.fill(w, head)
        try:
            return _compress_chains(codec, ss, tiled, chains, order, nblk, scheme, hwc_quirk)
        except OverflowError:
            if attempt == 3:
                raise
    raise AssertionError("unreachable")


def _compress_chains(codec, ss, tiled, chains, order, nblk, scheme, hwc_quirk):
    n = len(order)
    # all blocks to the device once: [step t, stream j] = block t of the j-th largest chain (CHW, demo_compress.py:120)
    C = tiled[chains[order[0]][0]][0].shape[-1]
    host = np.zeros((max(nblk), n, C, 32, 32), dtype=np.uint8)
    model = [_blocks_to_model(t[0], hwc_quirk) for t in tiled]
    for j, c in enumerate(order):
        i, s, nb = chains[c]
        host[:nb, j] = model[i][s:s + nb]
    dev = torch.from_numpy(host).to(torch.device("cuda", codec.device))
    ext = _extents_to_device(codec, [None if tiled[i][1] is None else tiled[i][1][s:s + nb] for i, s, nb in
                                     (chains[c] for c in order)], nblk)
    active = _active(nblk)
    for t in range(max(nblk)):
        for b, cnt in _sub_ranges(int(active[t]), codec.max_batch):
            codec.encode(ss, dev[t, b:b + cnt], first=b, scheme=scheme, extent=None if ext is None else ext[t, b:b + cnt])
    torch.cuda.synchronize()
    ss.raise_on_error()
    words, offs, heads, _ = ss.export()
    lo = ss.min_words()                                       # never-borrowed initial words (demo_compress.py:137,160)
    mine = [[] for _ in tiled]                                # each image's streams, in block order
    stream = np.empty(n, dtype=np.int64)
    stream[order] = np.arange(n)
    for c, (i, _, _) in enumerate(chains):
        mine[i].append(int(stream[c]))
    return [pack_container([(words[offs[j] + lo[j]:offs[j + 1]], int(heads[j]), nblk[j]) for j in js], h, wd)
            for js, (_, _, h, wd) in zip(mine, tiled)]


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


def pack_container(chains, h, w):
    """One image's container from its chains in block order, [(words uint32 [m], head int, nblocks)]: the reference layout
    for one chain (demo_compress.py:272-279), the multi-chain layout (module docstring) for two or more."""
    if len(chains) == 1:
        ws, hd, nb = chains[0]
        return np.concatenate([np.asarray(ws, dtype=np.uint32),
                               np.array([hd & 0xffffffff, hd >> 32, nb, h, w], dtype=np.uint32)])
    table = np.array([(len(ws), hd & 0xffffffff, hd >> 32, nb) for ws, hd, nb in chains], dtype=np.uint32)
    return np.concatenate([np.asarray(ws, dtype=np.uint32) for ws, _, _ in chains]
                          + [table.reshape(-1), np.array([len(chains), h, w, CHAIN_MARK], dtype=np.uint32)])


def _check_header(nblocks, h, w, hwc_quirk):
    if h <= 0 or w <= 0 or nblocks != np.prod(block_grid(h, w)) or nblocks > MAX_BLOCKS:
        raise ValueError(f"inconsistent container header: nblocks={nblocks}, h={h}, w={w}")
    if hwc_quirk and (h % 32 or w % 32):
        raise ValueError(f"edge-coded container (h={h}, w={w}) cannot be decoded with hwc_quirk")


def unpack_container(c, hwc_quirk=False):
    """Inverse of pack_container: (words uint32, offsets int64 [K+1], heads uint64 [K], nblocks int64 [K], h, w), chain k's
    words being words[offsets[k]:offsets[k+1]].  Every field is checked here, before anything is sized from it: a truncated
    or inconsistent container is a ValueError."""
    c = np.asarray(c, dtype=np.uint32)
    if c.ndim != 1 or c.size < 5:
        raise ValueError(f"container too short ({c.size} words): needs at least head_lo, head_hi, nblocks, h, w")
    if int(c[-1]) != CHAIN_MARK:
        nblocks, h, w = int(c[-3]), int(c[-2]), int(c[-1])                                      # demo_decompress.py:216-219
        _check_header(nblocks, h, w, hwc_quirk)
        head = (int(c[-4]) << 32) | int(c[-5])                                                  # :222
        return (c[:-5], np.array([0, c.size - 5], dtype=np.int64), np.array([head], dtype=np.uint64),
                np.array([nblocks], dtype=np.int64), h, w)
    k, h, w = int(c[-4]), int(c[-3]), int(c[-2])
    if k < 2 or c.size < 4 * k + 4:
        raise ValueError(f"multi-chain container of {c.size} words cannot hold the table of its {k} chains")
    table = c[c.size - 4 * k - 4:-4].reshape(k, 4).astype(np.int64)
    nwords, nblocks = table[:, 0], table[:, 3]
    if (nblocks < 1).any():
        raise ValueError("multi-chain container: a chain with no blocks")
    _check_header(int(nblocks.sum()), h, w, hwc_quirk)                 # (so also K <= blocks, as each chain has one)
    body = c.size - 4 * k - 4
    if int(nwords.sum()) != body:
        raise ValueError(f"multi-chain container: the chains claim {int(nwords.sum())} words, the container holds {body}")
    offsets = np.zeros(k + 1, dtype=np.int64)
    np.cumsum(nwords, out=offsets[1:])
    heads = (table[:, 2].astype(np.uint64) << np.uint64(32)) | table[:, 1].astype(np.uint64)
    return c[:body], offsets, heads, nblocks, h, w


RegionPlan = collections.namedtuple("RegionPlan", "first depth needed")
RegionPlan.__doc__ = """What decoding a container's regions costs.  first, depth: int64 [K], per chain in block order, the
earliest block the regions need counted from the chain's first block (the chain's block count when it holds none of them)
and the blocks to pop to reach it, nblocks - first (0: the chain is skipped).  needed: bool [nblocks], the row-major
blocks the regions cover."""


def _check_region(r, parsed):
    try:
        fields = tuple(r)
    except TypeError:
        raise ValueError(f"a region is (i, y, x, h, w), got {r!r}") from None
    if len(fields) != 5 or not all(isinstance(v, numbers.Integral) and not isinstance(v, bool) for v in fields):
        raise ValueError(f"a region is five ints (i, y, x, h, w), got {r!r}")
    i, y, x, h, w = (int(v) for v in fields)
    if not 0 <= i < len(parsed):
        raise ValueError(f"region {r!r}: no container {i} among {len(parsed)}")
    H, W = parsed[i][4], parsed[i][5]
    if h < 1 or w < 1 or y < 0 or x < 0 or y + h > H or x + w > W:
        raise ValueError(f"region {r!r} is empty or leaves the {H} x {W} image of container {i}")
    return i, y, x, h, w


def _plan(parsed, regions):
    """(regions as int tuples, one RegionPlan per container) for unpack_container results.  Every region is checked here."""
    regions = [_check_region(r, parsed) for r in regions]
    boxes = collections.defaultdict(list)
    for i, y, x, h, w in regions:
        boxes[i].append((y, x, h, w))
    plans = []
    for i, (_, _, _, nblocks, H, W) in enumerate(parsed):
        gw = block_grid(H, W)[1]
        needed = np.zeros(int(nblocks.sum()), dtype=bool)
        grid = needed.reshape(-1, gw)
        for y, x, h, w in boxes[i]:
            grid[y // 32:(y + h - 1) // 32 + 1, x // 32:(x + w - 1) // 32 + 1] = True
        starts = np.cumsum(nblocks) - nblocks
        earliest = np.minimum.reduceat(np.where(needed, np.arange(needed.size), needed.size), starts)
        first = np.minimum(earliest - starts, nblocks)
        plans.append(RegionPlan(first, nblocks - first, needed))
    return regions, plans


def plan_regions(containers, regions, hwc_quirk=False):
    """The decode plan of decompress_regions, computed on the host alone: one RegionPlan per container.  regions: list of
    (i, y, x, h, w) in pixels of container i's decoded image (the cropped size for a crop-mode container).  A malformed
    container, or a region that is empty, leaves the image, has a non-int field or names no container, is a ValueError."""
    parsed = [unpack_container(c, hwc_quirk) for c in containers]
    return _plan(parsed, regions)[1]


def decompress_regions(codec, containers, regions, channels=3, scheme=BITSWAP, hwc_quirk=False, headroom_words=None):
    """regions: list of (i, y, x, h, w) -> one HWC uint8 array per region, equal to decompress_images(...)[i][y:y+h, x:x+w].
    Only the chains holding a wanted block are imported, and each is popped only down to the earliest block any region on
    its container wants (plan_regions): a chain of n blocks whose earliest wanted block is j costs n - j block decodes.
    Blocks are row-major, so a window near an image's bottom is cheapest, and a single-chain container gains only there."""
    parsed = [unpack_container(c, hwc_quirk) for c in containers]
    return _decode_regions(codec, parsed, regions, channels, scheme, hwc_quirk, headroom_words)


def decompress_images(codec, containers, channels=3, scheme=BITSWAP, hwc_quirk=False, headroom_words=None):
    """Inverse of compress_images: list of container arrays -> list of HWC uint8 images (the cropped size for a crop-mode
    container, the full size for an edge-coded one: a header whose h or w is not a multiple of 32).  Single- and
    multi-chain containers can be mixed in one call."""
    parsed = [unpack_container(c, hwc_quirk) for c in containers]
    return _decode_regions(codec, parsed, [(i, 0, 0, p[4], p[5]) for i, p in enumerate(parsed)], channels, scheme,
                           hwc_quirk, headroom_words)


def _decode_regions(codec, parsed, regions, channels, scheme, hwc_quirk, headroom_words):
    regions, plans = _plan(parsed, regions)
    if not regions:
        return []
    # chains in image and block order: image, index within the image, first block, blocks, blocks to pop
    cimg = np.concatenate([np.full(len(p[3]), i) for i, p in enumerate(parsed)])
    ck = np.concatenate([np.arange(len(p[3])) for p in parsed])
    cstart = np.concatenate([np.cumsum(p[3]) - p[3] for p in parsed])
    cnb = np.concatenate([p[3] for p in parsed])
    cdepth = np.concatenate([pl.depth for pl in plans])
    order = np.argsort(-cdepth, kind="stable")[:np.count_nonzero(cdepth)]   # streams: deepest chain first, skipped ones out
    pieces = [parsed[i][0][parsed[i][1][k]:parsed[i][1][k + 1]] for i, k in zip(cimg[order], ck[order])]
    depth = cdepth[order].tolist()
    n = len(depth)
    # The receiver pushes too (it returns the borrowed bits, cifar_compress.py:306-313): one block's worth of latents,
    # nz * zdim symbols at <= 31 bits each, can sit on the stack above the chain's own length.
    if headroom_words is None:
        headroom_words = codec.cfg.nz * codec.cfg.zdim + 64
    ss = StreamSet(n, max(len(p) for p in pieces) + headroom_words, device=codec.device)
    offs = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(p) for p in pieces], out=offs[1:])
    ss.import_packed(np.concatenate(pieces), offs, np.array([parsed[i][2][k] for i, k in zip(cimg[order], ck[order])],
                                                              dtype=np.uint64))
    # Steps are aligned at the chains' ends: step s pops block n - 1 - s of every stream deeper than s, so the active
    # streams stay a prefix and [s, stream] holds that block, in the output and in the extents alike.
    dev = torch.empty((max(depth), n, channels, 32, 32), dtype=torch.uint8, device=torch.device("cuda", codec.device))
    extents = [block_extents(p[4], p[5]) for p in parsed]
    ext = _extents_to_device(codec, [extents[i][s + nb - d:s + nb][::-1] for i, s, nb, d in
                                     zip(cimg[order], cstart[order], cnb[order], depth)], depth)
    active = _active(depth)
    for s in range(max(depth)):
        for b, cnt in _sub_ranges(int(active[s]), codec.max_batch):
            codec.decode(ss, cnt, first=b, scheme=scheme, out=dev[s, b:b + cnt],
                         extent=None if ext is None else ext[s, b:b + cnt])
    if hasattr(codec, "join"):                                             # (free-running multi-lane codec: lanes -> current stream)
        codec.join()
    # the needed blocks of every image, gathered on the device into one transfer; pos[i][b]: block b's row in it
    stream = np.full(len(cnb), -1, dtype=np.int64)
    stream[order] = np.arange(n)
    first_chain = np.cumsum([0] + [len(p[3]) for p in parsed])
    rows, pos, m = [], [], 0
    for i, (p, pl) in enumerate(zip(parsed, plans)):
        b = np.flatnonzero(pl.needed)
        c = first_chain[i] + np.searchsorted(np.cumsum(p[3]), b, side="right")
        rows.append((cstart[c] + cnb[c] - 1 - b) * n + stream[c])
        pos.append(np.full(pl.needed.size, -1, dtype=np.int64))
        pos[i][b] = m + np.arange(b.size)
        m += b.size
    idx = torch.from_numpy(np.concatenate(rows)).to(dev.device)
    host = _model_to_blocks(dev.view(-1, channels, 32, 32).index_select(0, idx).cpu().numpy(), hwc_quirk)
    ss.raise_on_error()
    out = []
    for i, y, x, h, w in regions:
        gw = block_grid(parsed[i][4], parsed[i][5])[1]
        by, bx = np.arange(y // 32, (y + h - 1) // 32 + 1), np.arange(x // 32, (x + w - 1) // 32 + 1)
        tile = unextract_blocks(host[pos[i][by[:, None] * gw + bx[None, :]].reshape(-1)], 32 * by.size, 32 * bx.size)
        out.append(np.ascontiguousarray(tile[y - 32 * by[0]:y - 32 * by[0] + h, x - 32 * bx[0]:x - 32 * bx[0] + w]))
    return out
