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

Archives: a set of images as one array whose chains run across images.  Each chain borrows its first latent samples from
the initial words and keeps them, so one chain per small image pays them per image; compress_archive tiles every image as
edges="code" does, lays their row-major blocks end to end in the order given and cuts that one sequence into
chain_sizes(total blocks, chain_blocks) runs, each a chain from the seeded initial state.  Layout:
    [ words_0 ... words_{K-1} | (nwords_k, head_lo_k, head_hi_k, nblocks_k) for k < K | (h_i, w_i) for i < N
    | K, N, excess_state_len, seed, scheme, ARCHIVE_MARK ]
Read as a reference tail its width is ARCHIVE_MARK >= 2^31 and as a multi-chain container its last word is not CHAIN_MARK,
so unpack_container refuses it.  Decoding an image pops, in each chain holding its blocks, from the chain's end down to its
first block there; a chain popped to its first block must come back to the seeded initial state (cifar_compress.py:356).
Containers and archives share one encode loop (_encode) and one decode loop (_decode_regions) over a block sequence.

Stamps (opt-in: stamp=True): any of the three layouts above may carry, after its last word, what the codec that wrote it was
    [ inner array, byte-identical to the unstamped one | fields (uint32) | nfields, STAMP_VERSION, STAMP_MARK ]
with the fields of version 1, in order: the Fingerprint (revision, xc, nz, zchannels, nprocessing, kernel_size, resdepth,
reswidth, cond_xscale, quantbits, use_tensor_cores, tc_precision 0 split / 1 bf16, tc_heads, coder 0 reference / 1 direct,
model digest [4], bins digest [4]), then scheme, hwc_quirk, excess_state_len and seed.  STAMP_MARK >= 2^31 sits where the
reference layout has w and the archive its ARCHIVE_MARK, so a reader of the unstamped layouts refuses a stamped array.  The
decoders compare a stamp with codec.fingerprint() and their own scheme, hwc_quirk and channels before any stream is
created, and refuse it naming every field that differs; a stamped container also gets the archives' initial-state check.

Checksums (opt-in: checksums=True): any of the three layouts may carry a 32-bit digest of every coded block's pixels,
    [ inner array, byte-identical to the unchecked one | digest per block, in block-sequence order | nblocks, CHECK_VERSION,
      CHECK_MARK ]
the block sequence being the image's row-major blocks for a container and the archive's global sequence for an archive;
a stamp, when there is one too, goes after this trailer.  The digest (bsw_block_digest, include/bitswap_b200.h) covers the
block's valid extent as the coding buffer holds it and is seeded with the block's index in its sequence and its extent.
The writers digest the tiled buffer on the device; the decoders digest every block they decode (including blocks popped
on the way to a window) and compare on the device, then raise ValueError naming the first mismatching block after the
stream flags.  CHECK_MARK >= 2^31 sits where the unchecked layouts have their last word, so a reader of those refuses a
checked array.
"""
import collections
import numbers

import numpy as np
import torch

from ._lib import check, cuda_stream_ptr, lib, on_device
from .codec import BBANS, BITSWAP, CODERS, Fingerprint
from .model import TC_PRECISIONS
from .streams import StreamSet
from .synthetic import initial_words

CHAIN_MARK = 0x8043484E                  # bit 31 | "CHN": last word of a multi-chain container
MAX_BLOCKS = 1 << 20                     # blocks per image a container may declare
ARCHIVE_MARK = 0x80415243                # bit 31 | "ARC": last word of an archive
MAX_ARCHIVE_BLOCKS = 1 << 24             # blocks an archive may declare in all
MAX_INITIAL_WORDS = 1 << 24              # largest excess_state_len an archive may declare
STAMP_MARK = 0x80535450                  # bit 31 | "STP": last word of a stamped container or archive
STAMP_VERSION = 1
_STAMP_NFIELDS = {1: 26}                 # per version: 14 fingerprint words, two 4-word digests, 4 coding arguments
CHECK_MARK = 0x80434B53                  # bit 31 | "CKS": last word of a checked container or archive
CHECK_VERSION = 1

Stamp = collections.namedtuple("Stamp", "fingerprint scheme hwc_quirk excess_state_len seed")
Stamp.__doc__ = """What a stamped container or archive records about its writer: the codec's Fingerprint, the scheme (BITSWAP /
BBANS), hwc_quirk and the seeded initial state (excess_state_len, seed) every chain started from."""


def _stamp_words(fp, scheme, hwc_quirk, excess_state_len, seed):
    """The stamp appended to an array: fields, nfields, STAMP_VERSION, STAMP_MARK."""
    f = list(fp[:14])
    f[Fingerprint._fields.index("tc_precision")] = TC_PRECISIONS[fp.tc_precision]
    f[Fingerprint._fields.index("coder")] = CODERS[fp.coder]
    digests = [np.frombuffer(bytes.fromhex(d), dtype="<u4") for d in (fp.model_digest, fp.bins_digest)]
    fields = np.concatenate([np.array([int(v) for v in f], dtype=np.uint32)] + digests
                            + [np.array([scheme, int(hwc_quirk), excess_state_len, seed], dtype=np.uint32)])
    return np.concatenate([fields, np.array([fields.size, STAMP_VERSION, STAMP_MARK], dtype=np.uint32)])


def _check_stamp_args(scheme, excess_state_len, seed):
    if scheme not in (BITSWAP, BBANS):
        raise ValueError(f"scheme must be BITSWAP or BBANS, got {scheme!r}")
    for name, v, lo, hi in (("excess_state_len", excess_state_len, 2, MAX_INITIAL_WORDS), ("seed", seed, 0, (1 << 32) - 1)):
        if isinstance(v, bool) or not isinstance(v, numbers.Integral) or not lo <= v <= hi:
            raise ValueError(f"{name} must be an int in [{lo}, {hi}], got {v!r}")


def _split_stamp(a):
    """(inner array, Stamp) of a stamped array, (a, None) of any other.  Every stamp field is checked here, before anything
    is sized from it: a truncated or malformed stamp is a ValueError."""
    if a.ndim != 1 or a.size < 3 or int(a[-1]) != STAMP_MARK:
        return a, None
    nfields, version = int(a[-3]), int(a[-2])
    if version not in _STAMP_NFIELDS:
        raise ValueError(f"stamp of unknown version {version} (this reader knows {sorted(_STAMP_NFIELDS)})")
    if nfields != _STAMP_NFIELDS[version]:
        raise ValueError(f"stamp version {version} has {_STAMP_NFIELDS[version]} fields, this one claims {nfields}")
    if a.size < nfields + 4:
        raise ValueError(f"stamped array of {a.size} words cannot hold its {nfields} stamp fields and a stamped array")
    f = [int(v) for v in a[a.size - 3 - nfields:-3]]
    inner = a[:a.size - 3 - nfields]
    if int(inner[-1]) == STAMP_MARK:
        raise ValueError("a stamp inside a stamp")
    n = len(Fingerprint._fields) - 2
    head, digests, (scheme, hwc_quirk, excess_state_len, seed) = f[:n], f[n:n + 8], f[n + 8:]
    names = Fingerprint._fields
    for name, ok in (("cond_xscale", (0, 1)), ("kernel_size", (1, 3, 5, 7)), ("quantbits", range(5, 13)),
                     ("use_tensor_cores", (0, 1)), ("tc_precision", TC_PRECISIONS.values()), ("tc_heads", (0, 1)),
                     ("coder", CODERS.values())):
        if head[names.index(name)] not in ok:
            raise ValueError(f"stamp: {name} = {head[names.index(name)]} is out of range")
    if scheme not in (BITSWAP, BBANS) or hwc_quirk not in (0, 1):
        raise ValueError(f"stamp: scheme = {scheme}, hwc_quirk = {hwc_quirk} out of range")
    if not 2 <= excess_state_len <= MAX_INITIAL_WORDS:
        raise ValueError(f"stamp: excess_state_len {excess_state_len} outside [2, {MAX_INITIAL_WORDS}]")
    precision = {v: k for k, v in TC_PRECISIONS.items()}
    coders = {v: k for k, v in CODERS.items()}
    for name, conv in (("cond_xscale", bool), ("use_tensor_cores", bool), ("tc_precision", precision.get),
                       ("tc_heads", bool), ("coder", coders.get)):
        head[names.index(name)] = conv(head[names.index(name)])
    fp = Fingerprint(*head, *(np.asarray(digests[k:k + 4], dtype="<u4").tobytes().hex() for k in (0, 4)))
    return inner, Stamp(fp, scheme, bool(hwc_quirk), excess_state_len, seed)


def read_stamp(array):
    """The Stamp of a stamped container or archive, None for an unstamped one; on the host only, so that a user can see
    which codec decodes it before building one.  A malformed stamp is a ValueError."""
    return _split_stamp(np.asarray(array, dtype=np.uint32))[1]


def _check_stamps(codec, stamps, scheme, hwc_quirk, channels, what):
    """ValueError naming every field in which a stamp differs from this codec and these arguments (stamps: one Stamp or
    None per array).  The codec is asked for its fingerprint only when some array is stamped."""
    if all(st is None for st in stamps):
        return
    fp = codec.fingerprint()
    for i, st in enumerate(stamps):
        if st is None:
            continue
        want = list(zip(Fingerprint._fields, st.fingerprint, fp)) + [("scheme", st.scheme, scheme),
                                                                    ("hwc_quirk", st.hwc_quirk, bool(hwc_quirk))]
        if channels is not None:
            want.append(("channels", st.fingerprint.xc, channels))
        diff = [f"{name}: stamped {a!r}, here {b!r}" for name, a, b in want if a != b]
        if diff:
            raise ValueError(f"{what} {i} was written by a different codec or with other arguments; it cannot be decoded "
                             f"here: " + "; ".join(diff))


def _check_words(digests):
    """The check trailer appended to an array whose blocks have these digests (uint32, block-sequence order)."""
    return np.concatenate([np.asarray(digests, dtype=np.uint32),
                           np.array([len(digests), CHECK_VERSION, CHECK_MARK], dtype=np.uint32)])


def _split_check(a):
    """(inner array, digests uint32 [nblocks]) of a checked array, (a, None) of any other.  The trailer is checked here,
    before anything is sized from it; that nblocks matches the inner header is the caller's check (_check_count)."""
    if a.ndim != 1 or a.size < 3 or int(a[-1]) != CHECK_MARK:
        return a, None
    nblocks, version = int(a[-3]), int(a[-2])
    if version != CHECK_VERSION:
        raise ValueError(f"check trailer of unknown version {version} (this reader knows {CHECK_VERSION})")
    if nblocks > MAX_ARCHIVE_BLOCKS:
        raise ValueError(f"check trailer: {nblocks} blocks, more than any array holds ({MAX_ARCHIVE_BLOCKS})")
    if a.size < nblocks + 4:
        raise ValueError(f"checked array of {a.size} words cannot hold its {nblocks} digests and a checked array")
    inner = a[:a.size - 3 - nblocks]
    if int(inner[-1]) == CHECK_MARK:
        raise ValueError("a check trailer inside a check trailer")
    if int(inner[-1]) == STAMP_MARK:
        raise ValueError("a stamp inside a check trailer (a stamp goes after the check trailer)")
    return inner, a[inner.size:a.size - 3]


def _check_count(digests, nblocks, what):
    if digests is not None and digests.size != nblocks:
        raise ValueError(f"{what}: the check trailer holds {digests.size} digests, the header {nblocks} blocks")


# What a decode job verifies: its block sequence as the sequences the digests were computed over (offsets int64 [n + 1]:
# a container's image each, or one for an archive), the stored digests over the job's sequence (expected uint32) and which
# blocks have one (checked bool: an unchecked container's blocks have none); archive: how an error names the chain.
_Checks = collections.namedtuple("_Checks", "offsets expected checked archive")


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


# bsw_image_view and the tiling modes of bsw_tile_blocks / bsw_untile_regions (include/bitswap_b200.h)
_VIEW = np.dtype([("pixels", "<u8"), ("h", "<i4"), ("w", "<i4"), ("sy", "<i8"), ("sx", "<i8"), ("sc", "<i8")])
TILE_CROP, TILE_CODE, TILE_QUIRK = 0, 1, 2


def _is_cuda(x):
    return torch.is_tensor(x) and x.is_cuda


def _grid(shapes, mode):
    """Block grid (gh, gw) int64 [N] of images of these (h, w) [N, 2]: floor in crop and quirk mode, ceil in code mode."""
    h, w = shapes[:, 0], shapes[:, 1]
    return (-(-h // 32), -(-w // 32)) if mode == TILE_CODE else (h // 32, w // 32)


class _Blocks:
    """The block sequence of a writer call, still as the images it was given: the tile kernel lays it out on the device
    (_tile).  images: a list of HWC arrays, CPU tensors or CUDA tensors, or one [N, H, W, C] array or tensor.  CUDA images
    are checked here, before any device work (ValueError); host images too when `strict`, else as far as tiling needs.
    np.asarray of it is the same sequence by the reference tiling, [n, C, 32, 32] in the model's layout."""

    def __init__(self, codec, images, mode, strict):
        C = codec.cfg.xs[0]
        side = 1 if mode == TILE_CODE else 32
        self.mode = mode
        self.batch = (torch.is_tensor(images) or isinstance(images, np.ndarray)) and images.ndim == 4
        if self.batch:
            self.images = images if _is_cuda(images) else np.asarray(images)
            n, H, W = self.images.shape[:3]
            if _is_cuda(images):
                _check_cuda_image(codec, "images", images[0] if n else images.reshape(-1), C, side)
            elif strict:
                _check_host_image("images", self.images[0] if n else self.images.reshape(-1), C)
            self.shapes = np.tile(np.array([[H, W]], dtype=np.int64), (n, 1))
            self.C = int(self.images.shape[3])
            return
        self.images = [im if _is_cuda(im) else np.asarray(im) for im in images]
        for i, im in enumerate(self.images):
            if _is_cuda(im):
                _check_cuda_image(codec, f"image {i}", im, C, side)
            elif strict:
                _check_host_image(f"image {i}", im, C)
            elif im.ndim != 3:
                raise ValueError(f"image {i}: expected an H x W x C array, got shape {im.shape}")
        chans = {int(im.shape[2]) for im in self.images}
        if len(chans) > 1:
            raise ValueError(f"the images have different channel counts {sorted(chans)}")
        self.C = chans.pop() if chans else C
        self.shapes = np.array([im.shape[:2] for im in self.images], dtype=np.int64).reshape(-1, 2)

    def views(self, codec):
        """(bsw_image_view records on the codec's device, the tensors they point into).  Host images go up as one flat
        copy on the current stream."""
        dev = torch.device("cuda", codec.device)
        v = np.zeros(len(self.shapes), dtype=_VIEW)
        v["h"], v["w"] = self.shapes[:, 0], self.shapes[:, 1]
        if self.batch:
            t = self.images if _is_cuda(self.images) else torch.from_numpy(np.ascontiguousarray(self.images, np.uint8)).to(dev)
            s0, v["sy"], v["sx"], v["sc"] = t.stride()
            v["pixels"] = np.uint64(t.data_ptr()) + np.uint64(s0) * np.arange(len(v), dtype=np.uint64)
            return v, [t]
        keep = []
        host = [k for k, im in enumerate(self.images) if not _is_cuda(im)]
        if host:
            t = torch.from_numpy(np.concatenate([np.ascontiguousarray(self.images[k], np.uint8).reshape(-1) for k in host])).to(dev)
            keep.append(t)
            n = self.shapes[host, 0] * self.shapes[host, 1] * self.C
            v["pixels"][host] = np.uint64(t.data_ptr()) + (np.cumsum(n) - n).astype(np.uint64)
            v["sy"][host], v["sx"][host], v["sc"][host] = self.shapes[host, 1] * self.C, self.C, 1
        for k, im in enumerate(self.images):
            if _is_cuda(im):
                v[k] = (im.data_ptr(), im.shape[0], im.shape[1]) + tuple(im.stride())
                keep.append(im)
        return v, keep

    def __array__(self, dtype=None, copy=None):
        ims = [np.asarray(im.cpu()) if torch.is_tensor(im) else np.asarray(im) for im in self.images]
        tiles = [extract_edge_blocks(im)[0] if self.mode == TILE_CODE else extract_blocks(im)[0] for im in ims]
        a = np.concatenate([_blocks_to_model(t, self.mode == TILE_QUIRK) for t in tiles])
        return a if dtype is None else a.astype(dtype)


def _check_cuda_image(codec, what, t, C, side):
    if (t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != C or t.shape[0] < side or t.shape[1] < side
            or t.device.index != codec.device):
        raise ValueError(f"{what}: expected an H x W x {C} uint8 CUDA tensor on cuda:{codec.device} with H, W >= {side}, "
                         f"got {t.dtype} {tuple(t.shape)} on {t.device}")
    if np.prod(block_grid(*t.shape[:2])) > MAX_BLOCKS:
        raise ValueError(f"{what} of {t.shape[0]} x {t.shape[1]} has more than {MAX_BLOCKS} blocks")


def _check_host_image(what, im, C):
    if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != C or im.shape[0] < 1 or im.shape[1] < 1:
        raise ValueError(f"{what}: expected an H x W x {C} uint8 array with H, W >= 1, got {im.dtype} {im.shape}")
    if np.prod(block_grid(*im.shape[:2])) > MAX_BLOCKS:
        raise ValueError(f"{what} of {im.shape[0]} x {im.shape[1]} has more than {MAX_BLOCKS} blocks")


def _sequence_extents(shapes):
    """int16 [n, 2]: block_extents of images of these (h, w) in turn, without a step per image."""
    gh, gw = _grid(shapes, TILE_CODE)
    nb = gh * gw
    img = np.repeat(np.arange(len(nb)), nb)
    b = np.arange(int(nb.sum())) - np.repeat(np.cumsum(nb) - nb, nb)
    by, bx = b // gw[img], b % gw[img]
    return np.stack([np.minimum(32, shapes[img, 0] - 32 * by), np.minimum(32, shapes[img, 1] - 32 * bx)], -1).astype(np.int16)


def _chain_runs(nb, chain_blocks):
    """chain_sizes of every image of nb blocks, without a step per image: (chains per image, block counts in turn)."""
    k = np.ones_like(nb) if chain_blocks is None else np.where(chain_blocks >= nb, 1, -(-nb // chain_blocks))
    img = np.repeat(np.arange(len(nb)), k)
    pos = np.arange(int(k.sum())) - np.repeat(np.cumsum(k) - k, k)
    q, r = nb // k, nb % k
    return k, q[img] + (pos < r[img])


def compress_images(codec, images, excess_state_len=10000, seed=100, scheme=BITSWAP, hwc_quirk=False, words_per_block=1400,
                    edges="crop", chain_blocks=None, stamp=False, checksums=False):
    """images: list of HWC uint8 images -- numpy arrays, CPU tensors, or CUDA tensors of any strides on the codec's device
    -- or one [N, H, W, C] array or tensor.  Returns one container array per image (numpy uint32, the same bytes whatever
    the images were held in).  The images are tiled into blocks on the device; host images go up in one copy.
    Every chain starts from the reference's initial state: `excess_state_len` random words drawn with
    np.random.seed(100) (demo_compress.py:113-115, :202).
    edges="crop" (the reference's behaviour): every image is cropped down to multiples of 32 and must be at least 32x32.
    edges="code": the whole image (any H, W >= 1) is coded, with partial blocks at the bottom and right edges;
    decompress_images returns it exactly.
    chain_blocks: None (the reference's one chain per image) or a positive int L: an image of n > L blocks is coded as
    ceil(n / L) chains of contiguous blocks (chain_sizes), which run side by side.  Fewer serial steps, more initial bits.
    stamp=True: every container is followed by a stamp of codec.fingerprint() and these arguments (module docstring),
    which decompress_images checks; the container before it is unchanged.
    checksums=True: every container is followed by a 32-bit digest of each of its blocks' pixels (module docstring),
    against which every decoder checks each block it decodes; the container before it is unchanged, and a stamp goes
    after the digests.
    A CUDA image that is not a uint8 H x W x C tensor with the codec's C, is on another device, or is empty (under 32 x 32
    with edges="crop") is a ValueError before any device work."""
    if edges not in ("crop", "code"):
        raise ValueError(f"edges must be 'crop' or 'code', got {edges!r}")
    if edges == "code" and hwc_quirk:
        raise ValueError("edges='code' needs the CHW block layout: hwc_quirk scrambles the rows and columns the extents refer to")
    chain_blocks = _check_chain_blocks(chain_blocks)
    if stamp:
        _check_stamp_args(scheme, excess_state_len, seed)
        tail = _stamp_words(codec.fingerprint(), scheme, hwc_quirk, excess_state_len, seed)
    mode = TILE_CODE if edges == "code" else TILE_QUIRK if hwc_quirk else TILE_CROP
    blocks = _Blocks(codec, images, mode, strict=False)
    if not len(blocks.shapes):
        raise ValueError("no images")
    gh, gw = _grid(blocks.shapes, mode)
    hw = blocks.shapes if mode == TILE_CODE else 32 * np.stack([gh, gw], -1)     # what the containers record
    # one block sequence of every image in turn; each image's chains are runs inside its own blocks
    per_image, sizes = _chain_runs(gh * gw, chain_blocks)
    chains = list(zip((np.cumsum(sizes) - sizes).tolist(), sizes.tolist()))
    extents = None if mode != TILE_CODE else _sequence_extents(blocks.shapes)
    ioff = np.concatenate([[0], np.cumsum(gh * gw)]).astype(np.int64)
    if checksums:
        coded, digests = _encode_checked(codec, blocks, extents, chains, scheme, excess_state_len, seed, words_per_block, ioff)
    else:
        coded = _encode(codec, blocks, extents, chains, scheme, excess_state_len, seed, words_per_block)
    out, k = [], 0
    for i, (K, (h, w)) in enumerate(zip(per_image.tolist(), hw.tolist())):
        out.append(pack_container(coded[k:k + K], h, w))
        if checksums:
            out[-1] = np.concatenate([out[-1], _check_words(digests[ioff[i]:ioff[i + 1]])])
        if stamp:
            out[-1] = np.concatenate([out[-1], tail])
        k += K
    return out


def _encode(codec, blocks, extents, chains, scheme, excess_state_len, seed, words_per_block):
    """Codes a block sequence (blocks: a _Blocks; extents int16 [n, 2] or None) as the chains (start, nblocks) given, each a
    run of it, from the seeded initial state.  Returns [(words above the lowest depth, head, nblocks)] in chain order.
    Streams hold the chains largest first, so the active streams at each step are a prefix."""
    return _encode_checked(codec, blocks, extents, chains, scheme, excess_state_len, seed, words_per_block, None)[0]


def _encode_checked(codec, blocks, extents, chains, scheme, excess_state_len, seed, words_per_block, seq_offsets):
    """_encode's chains and the block digests: None when seq_offsets is None, else uint32 [blocks], the digest of every
    block in sequence order as tiled, seeded over the sequences seq_offsets (int64) lays end to end (bsw_block_digests)."""
    cnb = np.array([nb for _, nb in chains], dtype=np.int64)
    order = np.argsort(-cnb, kind="stable")
    nblk = cnb[order]
    stream = np.empty(len(cnb), dtype=np.int32)
    stream[order] = np.arange(len(cnb))
    x, ext = _tile(codec, blocks, cnb, stream, int(nblk[0]), extents is not None and not (extents == 32).all())
    digests = None
    if seq_offsets is not None:
        # slot [t, j] holds block t of the chain on stream j, at sequence index start + t
        start = np.array([s for s, _ in chains], dtype=np.int64)[order]
        t = np.arange(int(nblk[0]), dtype=np.int64)[:, None]
        digests = _digest_blocks(codec, x, ext, np.where(t < nblk[None, :], start[None, :] + t, -1), seq_offsets)
    w, head = initial_words(excess_state_len, seed=seed)
    # capacity: `words_per_block` words per 32x32 block of the longest chain (1400 = 14.6 bits/dim; 8 bits/dim of raw pixels
    # is 768).  A chain that still overflows is retried with twice the room instead of failing after it was coded.
    for attempt in range(4):
        ss = StreamSet(len(cnb), excess_state_len + (words_per_block << attempt) * int(nblk[0]) + 64, device=codec.device)
        ss.fill(w, head)
        try:
            words, offs, heads = _compress_chains(codec, ss, x, ext, nblk, scheme)
        except OverflowError:
            if attempt == 3:
                raise
            continue
        coded = [(words[offs[j]:offs[j + 1]], int(heads[j]), nb) for j, nb in zip(stream.tolist(), cnb.tolist())]
        return coded, None if digests is None else digests.cpu().numpy().view(np.uint32)
    raise AssertionError("unreachable")


def _digest_blocks(codec, x, ext, block, seq_offsets):
    """The digests of the blocks in x [step, stream, C, 32, 32] (extents ext [step, stream, 2] or None: full), on the
    device, on the current stream (bsw_block_digests): an int32 CUDA tensor [total blocks], in sequence order.  block:
    int64 [step, stream], each slot's block in the sequence (-1: none); seq_offsets: int64, the sequences' offsets."""
    seq_offsets = np.ascontiguousarray(seq_offsets, dtype=np.int64)
    block = np.ascontiguousarray(block, dtype=np.int64).reshape(-1)
    out = torch.zeros(int(seq_offsets[-1]), dtype=torch.int32, device=x.device)
    if block.size:
        with on_device(codec.device):
            check(lib().bsw_block_digests(x.data_ptr(), None if ext is None else ext.data_ptr(), x.shape[2], block.size,
                                          block.ctypes.data, seq_offsets.ctypes.data, len(seq_offsets) - 1,
                                          out.data_ptr(), cuda_stream_ptr()))
    return out


def _tile(codec, blocks, cnb, stream, steps, ragged):
    """The coding buffer [step t, stream j, C, 32, 32] (block t of the chain on stream j; CHW, demo_compress.py:120) and,
    when `ragged`, the int16 extents [t, j, 2], tiled on the device on the current stream (bsw_tile_blocks).  cnb: int64
    block counts of the chains in sequence order; stream: int32, the stream of each chain."""
    dev = torch.device("cuda", codec.device)
    x = torch.empty((steps, len(cnb), blocks.C, 32, 32), dtype=torch.uint8, device=dev)
    ext = torch.empty((steps, len(cnb), 2), dtype=torch.int16, device=dev) if ragged else None
    if steps:
        views, keep = blocks.views(codec)
        with on_device(codec.device):
            check(lib().bsw_tile_blocks(views.ctypes.data, len(views), blocks.C, blocks.mode, cnb.ctypes.data,
                                        stream.ctypes.data, len(cnb), steps, x.data_ptr(),
                                        None if ext is None else ext.data_ptr(), cuda_stream_ptr()))
    return x, ext


def _compress_chains(codec, ss, x, ext, nblk, scheme):
    """Codes x [step, stream] onto the streams (nblk: their block counts, largest first) and reads back only the words above
    each stream's lowest depth (the never-borrowed initial words stay, demo_compress.py:137,160): (words uint32, offsets
    int64 [n + 1], heads uint64 [n]) in stream order."""
    active = _active(nblk)
    for t in range(int(nblk[0])):
        for b, cnt in _sub_ranges(int(active[t]), codec.max_batch):
            codec.encode(ss, x[t, b:b + cnt], first=b, scheme=scheme, extent=None if ext is None else ext[t, b:b + cnt])
    torch.cuda.synchronize()
    ss.raise_on_error()
    words_d, offs_d, heads_d, _ = ss.pack_device(trim=True)
    offs = offs_d.cpu().numpy()
    return words_d[:int(offs[-1])].cpu().numpy().view(np.uint32), offs, heads_d.cpu().numpy().view(np.uint64)


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
    or inconsistent container is a ValueError.  A stamped or checked container is accepted: its stamp and check trailer
    are checked and stripped."""
    return _unpack_container(c, hwc_quirk)[:-1]


def _unpack_container(c, hwc_quirk):
    """unpack_container's tuple and the container's block digests (None for an unchecked container)."""
    c, digests = _split_check(_split_stamp(np.asarray(c, dtype=np.uint32))[0])
    if c.ndim != 1 or c.size < 5:
        raise ValueError(f"container too short ({c.size} words): needs at least head_lo, head_hi, nblocks, h, w")
    if int(c[-1]) != CHAIN_MARK:
        nblocks, h, w = int(c[-3]), int(c[-2]), int(c[-1])                                      # demo_decompress.py:216-219
        _check_header(nblocks, h, w, hwc_quirk)
        _check_count(digests, nblocks, "container")
        head = (int(c[-4]) << 32) | int(c[-5])                                                  # :222
        return (c[:-5], np.array([0, c.size - 5], dtype=np.int64), np.array([head], dtype=np.uint64),
                np.array([nblocks], dtype=np.int64), h, w, digests)
    k, h, w = int(c[-4]), int(c[-3]), int(c[-2])
    if k < 2 or c.size < 4 * k + 4:
        raise ValueError(f"multi-chain container of {c.size} words cannot hold the table of its {k} chains")
    table = c[c.size - 4 * k - 4:-4].reshape(k, 4).astype(np.int64)
    nwords, nblocks = table[:, 0], table[:, 3]
    if (nblocks < 1).any():
        raise ValueError("multi-chain container: a chain with no blocks")
    _check_header(int(nblocks.sum()), h, w, hwc_quirk)                 # (so also K <= blocks, as each chain has one)
    _check_count(digests, int(nblocks.sum()), "multi-chain container")
    body = c.size - 4 * k - 4
    if int(nwords.sum()) != body:
        raise ValueError(f"multi-chain container: the chains claim {int(nwords.sum())} words, the container holds {body}")
    offsets = np.zeros(k + 1, dtype=np.int64)
    np.cumsum(nwords, out=offsets[1:])
    heads = (table[:, 2].astype(np.uint64) << np.uint64(32)) | table[:, 1].astype(np.uint64)
    return c[:body], offsets, heads, nblocks, h, w, digests


RegionPlan = collections.namedtuple("RegionPlan", "first depth needed")
RegionPlan.__doc__ = """What decoding a container's regions costs.  first, depth: int64 [K], per chain in block order, the
earliest block the regions need counted from the chain's first block (the chain's block count when it holds none of them)
and the blocks to pop to reach it, nblocks - first (0: the chain is skipped).  needed: bool [nblocks], the row-major
blocks the regions cover."""

# A decode job: a block sequence of images, each image's row-major blocks in turn (image i owns blocks ioff[i] to
# ioff[i + 1]), and the chains that code it, contiguous runs in sequence order (chain k: pieces[k] and heads[k], blocks
# cstart[k] to cstart[k] + cnb[k]).  A container is one image whose chains stay inside it; an archive lets them run across.
_Job = collections.namedtuple("_Job", "pieces heads cstart cnb shapes ioff")


def _containers_job(parsed):
    """The decode job of unpack_container results: the containers' images in turn, each with its own chains."""
    nb = [int(p[3].sum()) for p in parsed]
    ioff = np.zeros(len(parsed) + 1, dtype=np.int64)
    np.cumsum(nb, out=ioff[1:])
    cnb = np.concatenate([p[3] for p in parsed]) if parsed else np.zeros(0, np.int64)
    return _Job([p[0][p[1][k]:p[1][k + 1]] for p in parsed for k in range(len(p[3]))],
                np.concatenate([p[2] for p in parsed]) if parsed else np.zeros(0, np.uint64),
                np.cumsum(cnb) - cnb, cnb, [(p[4], p[5]) for p in parsed], ioff)


def _check_region(r, shapes):
    try:
        fields = tuple(r)
    except TypeError:
        raise ValueError(f"a region is (i, y, x, h, w), got {r!r}") from None
    if len(fields) != 5 or not all(isinstance(v, numbers.Integral) and not isinstance(v, bool) for v in fields):
        raise ValueError(f"a region is five ints (i, y, x, h, w), got {r!r}")
    i, y, x, h, w = (int(v) for v in fields)
    if not 0 <= i < len(shapes):
        raise ValueError(f"region {r!r}: no image {i} among {len(shapes)}")
    H, W = shapes[i]
    if h < 1 or w < 1 or y < 0 or x < 0 or y + h > H or x + w > W:
        raise ValueError(f"region {r!r} is empty or leaves the {H} x {W} image {i}")
    return i, y, x, h, w


def _plan(job, regions):
    """(regions as int tuples, RegionPlan over the job's chains and block sequence).  Every region is checked here."""
    regions = [_check_region(r, job.shapes) for r in regions]
    needed = np.zeros(int(job.ioff[-1]), dtype=bool)
    for i, y, x, h, w in regions:
        grid = needed[job.ioff[i]:job.ioff[i + 1]].reshape(-1, block_grid(*job.shapes[i])[1])
        grid[y // 32:(y + h - 1) // 32 + 1, x // 32:(x + w - 1) // 32 + 1] = True
    if not len(job.cnb):
        return regions, RegionPlan(job.cnb.copy(), job.cnb.copy(), needed)
    earliest = np.minimum.reduceat(np.where(needed, np.arange(needed.size), needed.size), job.cstart)
    first = np.minimum(earliest - job.cstart, job.cnb)
    return regions, RegionPlan(first, job.cnb - first, needed)


def plan_regions(containers, regions, hwc_quirk=False):
    """The decode plan of decompress_regions, computed on the host alone: one RegionPlan per container.  regions: list of
    (i, y, x, h, w) in pixels of container i's decoded image (the cropped size for a crop-mode container).  A malformed
    container, or a region that is empty, leaves the image, has a non-int field or names no container, is a ValueError."""
    job = _containers_job([unpack_container(c, hwc_quirk) for c in containers])
    plan = _plan(job, regions)[1]
    k = np.searchsorted(job.cstart, job.ioff)                     # container i's chains: k[i] to k[i + 1]
    return [RegionPlan(plan.first[k[i]:k[i + 1]], plan.depth[k[i]:k[i + 1]], plan.needed[job.ioff[i]:job.ioff[i + 1]])
            for i in range(len(job.shapes))]


def _stamped_job(codec, containers, channels, scheme, hwc_quirk):
    """The decode job of a list of containers, every stamp checked against the codec and the arguments; each chain's
    seeded initial state (words, head) where its container is stamped (None where it is not; None alone when no
    container is stamped); and the job's _Checks (None when no container is checked)."""
    split = [_split_stamp(np.asarray(c, dtype=np.uint32)) for c in containers]
    parsed = [_unpack_container(inner, hwc_quirk) for inner, _ in split]
    _check_stamps(codec, [st for _, st in split], scheme, hwc_quirk, channels, "container")
    states, initial = {}, []
    for (_, st), p in zip(split, parsed):
        if st is not None and (st.excess_state_len, st.seed) not in states:
            states[st.excess_state_len, st.seed] = initial_words(st.excess_state_len, seed=st.seed)
        initial += [None if st is None else states[st.excess_state_len, st.seed]] * len(p[3])
    job = _containers_job(parsed)
    checks = None
    if any(p[6] is not None for p in parsed):
        nb = np.diff(job.ioff)
        checks = _Checks(job.ioff, np.concatenate([np.zeros(n, np.uint32) if p[6] is None else p[6] for p, n in zip(parsed, nb)]),
                         np.repeat([p[6] is not None for p in parsed], nb), False)
    return job, initial if states else None, checks


def decompress_regions(codec, containers, regions, channels=3, scheme=BITSWAP, hwc_quirk=False, headroom_words=None,
                       as_tensors=False, verify=True):
    """regions: list of (i, y, x, h, w) -> one HWC uint8 array per region, equal to decompress_images(...)[i][y:y+h, x:x+w].
    Only the chains holding a wanted block are imported, and each is popped only down to the earliest block any region on
    its container wants (plan_regions): a chain of n blocks whose earliest wanted block is j costs n - j block decodes.
    Blocks are row-major, so a window near an image's bottom is cheapest, and a single-chain container gains only there.
    A stamped container must match the codec's fingerprint, scheme, hwc_quirk and channels (ValueError naming every field
    that differs, before any decoding), and each of its chains popped down to its first block must come back to the
    stamp's initial state.
    A checked container (compress_images(checksums=True)) has every block decoded here, including the blocks popped on
    the way to a window, compared with its stored digest on the device; after the stream flags (IndexError,
    OverflowError), a mismatch is a ValueError naming how many blocks differ and the first one's image, block row and
    column, and chain.  verify=False skips that comparison.
    as_tensors=True: contiguous torch.uint8 [h, w, C] tensors on the codec's device instead, the same pixels; no pixel
    crosses PCIe.  Either way the regions are cut on the device and the decode is complete when this returns."""
    job, initial, checks = _stamped_job(codec, containers, channels, scheme, hwc_quirk)
    return _decode_regions(codec, job, regions, channels, scheme, hwc_quirk, headroom_words, initial, as_tensors,
                           checks if verify else None)


def decompress_images(codec, containers, channels=3, scheme=BITSWAP, hwc_quirk=False, headroom_words=None, as_tensors=False,
                      verify=True):
    """Inverse of compress_images: list of container arrays -> list of HWC uint8 images (the cropped size for a crop-mode
    container, the full size for an edge-coded one: a header whose h or w is not a multiple of 32).  Single- and
    multi-chain containers can be mixed in one call, and so can stamped and unstamped, checked and unchecked ones (see
    decompress_regions; verify=False skips the block digests).
    as_tensors=True: contiguous torch.uint8 [h, w, C] CUDA tensors on the codec's device instead of numpy arrays."""
    job, initial, checks = _stamped_job(codec, containers, channels, scheme, hwc_quirk)
    return _decode_regions(codec, job, [(i, 0, 0, h, w) for i, (h, w) in enumerate(job.shapes)], channels, scheme,
                           hwc_quirk, headroom_words, initial, as_tensors, checks if verify else None)


def _decode_regions(codec, job, regions, channels, scheme, hwc_quirk, headroom_words, initial=None, as_tensors=False,
                   checks=None):
    """Decodes the job's regions.  channels None: the codec's.  initial: per chain, None or the seeded initial state
    (words, head) it started from; such a chain popped down to its first block must then hold its top words and head, or
    ValueError.  as_tensors: CUDA tensors instead of numpy arrays.  checks: None or the job's _Checks; every decoded block
    that has a stored digest must then match it, or ValueError."""
    regions, plan = _plan(job, regions)
    if not regions:
        return []
    if channels is None:
        channels = codec.cfg.xs[0]
    cstart, cnb = job.cstart, job.cnb
    order = np.argsort(-plan.depth, kind="stable")[:np.count_nonzero(plan.depth)]  # streams: deepest first, skipped ones out
    pieces = [job.pieces[c] for c in order]
    depth = plan.depth[order]
    n = len(depth)
    # The receiver pushes too (it returns the borrowed bits, cifar_compress.py:306-313): one block's worth of latents,
    # nz * zdim symbols at <= 31 bits each, can sit on the stack above the chain's own length.
    if headroom_words is None:
        headroom_words = codec.cfg.nz * codec.cfg.zdim + 64
    ss = StreamSet(n, max(len(p) for p in pieces) + headroom_words, device=codec.device)
    offs = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(p) for p in pieces], out=offs[1:])
    ss.import_packed(np.concatenate(pieces), offs, job.heads[order])
    # Steps are aligned at the chains' ends: step s pops block n - 1 - s of every stream deeper than s, so the active
    # streams stay a prefix and [s, stream] holds that block, in the output and in the extents alike.
    dev = torch.empty((int(depth[0]), n, channels, 32, 32), dtype=torch.uint8, device=torch.device("cuda", codec.device))
    ext = _decode_extents(codec, job, (cstart + cnb)[order], depth)
    active = _active(depth)
    for s in range(int(depth[0])):
        for b, cnt in _sub_ranges(int(active[s]), codec.max_batch):
            codec.decode(ss, cnt, first=b, scheme=scheme, out=dev[s, b:b + cnt],
                         extent=None if ext is None else ext[s, b:b + cnt])
    if hasattr(codec, "join"):                                             # (free-running multi-lane codec: lanes -> current stream)
        codec.join()
    stream = np.full(len(cnb), -1, dtype=np.int32)
    stream[order] = np.arange(n)
    out = _untile(codec, job, regions, stream, dev, TILE_QUIRK if hwc_quirk else TILE_CODE)
    if checks is not None:
        # slot [s, j] holds block cend_j - 1 - s of the sequence for s < depth_j; blocks without a digest are skipped
        g = (cstart + cnb)[order][None, :] - 1 - np.arange(int(depth[0]), dtype=np.int64)[:, None]
        live = (g >= (cstart + cnb - plan.depth)[order][None, :])
        block = np.where(live & checks.checked[np.where(live, g, 0)], g, -1)
        result = _verify_blocks(codec, dev, ext, block, checks)
    ss.raise_on_error()                                                    # (synchronises the device)
    if checks is not None:
        _raise_on_mismatch(job, checks, *result.cpu().tolist())
    if initial is not None:
        _check_initial_state(ss, order, plan.first[order] == 0, initial)
    size = np.array([h * w * channels for _, _, _, h, w in regions], dtype=np.int64)
    start = (np.cumsum(size) - size).tolist()
    if not as_tensors:
        out = out.cpu().numpy()
    return [out[o:o + m].view(h, w, channels) if as_tensors else out[o:o + m].reshape(h, w, channels)
            for o, m, (_, _, _, h, w) in zip(start, size.tolist(), regions)]


def _verify_blocks(codec, x, ext, block, checks):
    """bsw_block_digests_check of the decoded blocks in x [step, stream, C, 32, 32] on the current stream: an int64 CUDA
    tensor (blocks that differ from their stored digest, the lowest such index in the job's sequence)."""
    block = np.ascontiguousarray(block, dtype=np.int64).reshape(-1)
    offsets = np.ascontiguousarray(checks.offsets, dtype=np.int64)
    expected = torch.from_numpy(np.ascontiguousarray(checks.expected, dtype=np.uint32).view(np.int32)).to(x.device)
    result = torch.empty(2, dtype=torch.int64, device=x.device)
    with on_device(codec.device):
        check(lib().bsw_block_digests_check(x.data_ptr(), None if ext is None else ext.data_ptr(), x.shape[2], block.size,
                                            block.ctypes.data, offsets.ctypes.data, len(offsets) - 1, expected.data_ptr(),
                                            result.data_ptr(), cuda_stream_ptr()))
    return result


def _raise_on_mismatch(job, checks, bad, g):
    """ValueError naming the first of `bad` decoded blocks whose digest differs (g: its index in the job's sequence)."""
    if not bad:
        return
    i = int(np.searchsorted(job.ioff, g, side="right")) - 1
    by, bx = divmod(g - int(job.ioff[i]), block_grid(*job.shapes[i])[1])
    k = int(np.searchsorted(job.cstart, g, side="right")) - 1
    where = f"chain {k} of the archive" if checks.archive else \
        f"chain {k - int(np.searchsorted(job.cstart, job.ioff[i]))} of container {i}"
    raise ValueError(f"{bad} decoded block{'s' if bad > 1 else ''} differ{'' if bad > 1 else 's'} from the stored digest: "
                     f"the first is image {i}, block row {by}, column {bx}, in {where}.  The codec is not the encoder's "
                     f"(coder, tc_precision, conv path, weights, bins or build), or the array is corrupt")


def _decode_extents(codec, job, cend, depth):
    """[step s, stream j] int16 extents of block cend_j - 1 - s on the device, or None when every decoded block is full (then
    the plain calls run, which code exactly what full extents would).  Rows past a stream's depth hold (32, 32)."""
    s = np.arange(int(depth[0]))[:, None]
    live = s < depth[None, :]
    seq = _sequence_extents(np.asarray(job.shapes, dtype=np.int64).reshape(-1, 2))
    host = np.where(live[..., None], seq[np.where(live, cend[None, :] - 1 - s, 0)], np.int16(32))
    if (host == 32).all():
        return None
    return torch.from_numpy(np.ascontiguousarray(host, dtype=np.int16)).to(torch.device("cuda", codec.device))


def _untile(codec, job, regions, stream, x, mode):
    """The regions cut out of the decoder's buffer x [step, stream, C, 32, 32] on the device, on the current stream
    (bsw_untile_regions): one flat uint8 CUDA tensor holding each region as contiguous HWC, the regions in turn.  stream:
    int32 per chain of the job, the stream that decoded it (-1: none)."""
    shapes = np.ascontiguousarray(np.asarray(job.shapes, dtype=np.int64).reshape(-1, 2), dtype=np.int32)
    regs = np.ascontiguousarray(regions, dtype=np.int32).reshape(-1, 5)
    cnb = np.ascontiguousarray(job.cnb, dtype=np.int64)
    C = x.shape[2]
    out = torch.empty(int((regs[:, 3].astype(np.int64) * regs[:, 4]).sum()) * C, dtype=torch.uint8, device=x.device)
    with on_device(codec.device):
        check(lib().bsw_untile_regions(shapes.ctypes.data, len(shapes), C, mode, cnb.ctypes.data, stream.ctypes.data,
                                       len(cnb), x.shape[1], x.shape[0], x.data_ptr(), regs.ctypes.data, len(regs),
                                       out.data_ptr(), cuda_stream_ptr()))
    return out


def _check_initial_state(ss, order, done, initial):
    """A chain popped down to its first block holds what it started from: the top words of the seeded initial stack and
    its head (cifar_compress.py:356).  done: bool per stream, the streams popped that far; order: each stream's chain;
    initial: per chain, its (words, head) or None (not checked)."""
    got, offs, heads, _ = ss.export()
    for j in np.flatnonzero(done).tolist():
        if initial[order[j]] is None:
            continue
        words, head = initial[order[j]]
        m = int(offs[j + 1] - offs[j])
        if not (m <= words.size and int(heads[j]) == head and np.array_equal(got[offs[j]:offs[j + 1]], words[words.size - m:])):
            raise ValueError(f"chain {int(order[j])} decoded to a state other than the initial one it was coded from: a "
                             f"different model, bins or conv path than the encoder's, or a corrupt archive or container")


def pack_archive(chains, shapes, excess_state_len, seed, scheme):
    """An archive from its chains in block-sequence order, [(words uint32 [m], head int, nblocks)], and its images' (h, w):
    [ words_0 ... words_{K-1} | (nwords_k, head_lo_k, head_hi_k, nblocks_k) for k < K | (h_i, w_i) for i < N
    | K, N, excess_state_len, seed, scheme, ARCHIVE_MARK ]."""
    table = np.array([(len(ws), hd & 0xffffffff, hd >> 32, nb) for ws, hd, nb in chains], dtype=np.uint32).reshape(-1)
    return np.concatenate([np.asarray(ws, dtype=np.uint32) for ws, _, _ in chains]
                          + [table, np.asarray(shapes, dtype=np.uint32).reshape(-1),
                             np.array([len(chains), len(shapes), excess_state_len, seed, scheme, ARCHIVE_MARK], dtype=np.uint32)])


def unpack_archive(a):
    """Inverse of pack_archive: (words uint32, offsets int64 [K+1], heads uint64 [K], nblocks int64 [K], shapes int64 [N, 2],
    excess_state_len, seed, scheme), chain k's words being words[offsets[k]:offsets[k+1]].  Every field is checked here,
    before anything is sized from it: a truncated or inconsistent archive is a ValueError.  A stamped archive is accepted:
    its stamp is checked, must agree with the header's scheme and initial state, and is stripped; so is a checked
    archive's check trailer."""
    return _unpack_archive(a)[:-2]


def _unpack_archive(a):
    """unpack_archive's tuple, the archive's Stamp (or None) and its block digests (or None)."""
    a, stamp = _split_stamp(np.asarray(a, dtype=np.uint32))
    a, digests = _split_check(a)
    if a.ndim != 1 or a.size < 6 or int(a[-1]) != ARCHIVE_MARK:
        raise ValueError("not an archive: it must be a 1-D uint32 array ending in ARCHIVE_MARK")
    k, n, n_init, seed, scheme = (int(v) for v in a[-6:-1])
    if k < 1 or n < 1 or a.size < 6 + 4 * k + 2 * n:
        raise ValueError(f"archive of {a.size} words cannot hold the tables of its {k} chains and {n} images")
    body = a.size - 6 - 4 * k - 2 * n
    table = a[body:body + 4 * k].reshape(k, 4).astype(np.int64)
    shapes = a[body + 4 * k:-6].reshape(n, 2).astype(np.int64)
    if (shapes < 1).any():
        raise ValueError("archive: an image with no pixels")
    blocks = -(-shapes[:, 0] // 32) * -(-shapes[:, 1] // 32)
    if (blocks > MAX_BLOCKS).any():
        raise ValueError(f"archive: an image of more than {MAX_BLOCKS} blocks")
    nwords, nblocks = table[:, 0], table[:, 3]
    if (nblocks < 1).any():
        raise ValueError("archive: a chain with no blocks")
    if int(nblocks.sum()) != int(blocks.sum()) or int(blocks.sum()) > MAX_ARCHIVE_BLOCKS:
        raise ValueError(f"archive: the chains hold {int(nblocks.sum())} blocks, the images {int(blocks.sum())} "
                         f"(at most {MAX_ARCHIVE_BLOCKS})")
    _check_count(digests, int(blocks.sum()), "archive")
    if int(nwords.sum()) != body:
        raise ValueError(f"archive: the chains claim {int(nwords.sum())} words, the archive holds {body}")
    if not 2 <= n_init <= MAX_INITIAL_WORDS:
        raise ValueError(f"archive: excess_state_len {n_init} outside [2, {MAX_INITIAL_WORDS}]")
    if scheme not in (BITSWAP, BBANS):
        raise ValueError(f"archive: unknown scheme {scheme}")
    if stamp is not None and (stamp.scheme, stamp.excess_state_len, stamp.seed) != (scheme, n_init, seed):
        raise ValueError(f"archive: the stamp's scheme, excess_state_len and seed "
                         f"{(stamp.scheme, stamp.excess_state_len, stamp.seed)} disagree with the header's {(scheme, n_init, seed)}")
    if stamp is not None and stamp.hwc_quirk:
        raise ValueError("archive: the stamp has hwc_quirk set, which archives never use")
    offsets = np.zeros(k + 1, dtype=np.int64)
    np.cumsum(nwords, out=offsets[1:])
    heads = (table[:, 2].astype(np.uint64) << np.uint64(32)) | table[:, 1].astype(np.uint64)
    return a[:body], offsets, heads, nblocks, shapes, n_init, seed, scheme, stamp, digests


def _archive_job(a):
    """The decode job of an archive, its header's initial state and scheme, its Stamp and its _Checks (or None)."""
    words, offsets, heads, nblocks, shapes, n_init, seed, scheme, stamp, digests = _unpack_archive(a)
    ioff = np.zeros(len(shapes) + 1, dtype=np.int64)
    np.cumsum(-(-shapes[:, 0] // 32) * -(-shapes[:, 1] // 32), out=ioff[1:])
    job = _Job([words[offsets[k]:offsets[k + 1]] for k in range(len(heads))], heads, np.cumsum(nblocks) - nblocks, nblocks,
               [(int(h), int(w)) for h, w in shapes], ioff)
    checks = None if digests is None else \
        _Checks(np.array([0, ioff[-1]], dtype=np.int64), digests, np.ones(digests.size, dtype=bool), True)
    return job, n_init, seed, scheme, stamp, checks


def compress_archive(codec, images, chain_blocks=64, scheme=BITSWAP, excess_state_len=10000, seed=100, words_per_block=1400,
                     stamp=False, checksums=False):
    """images: a sequence of HWC uint8 images of any sizes (H, W >= 1, C = the model's) -- numpy arrays, CPU tensors, or CUDA
    tensors of any strides on the codec's device -- or one [N, H, W, C] array or tensor -> one np.uint32 archive.
    Each image is tiled as compress_images(edges="code") tiles it; the row-major blocks of all images, in the order given,
    form one sequence, cut into chain_sizes(total blocks, chain_blocks) contiguous runs, each coded as a chain from the seeded
    initial state.  A chain may start or end inside an image, so the initial words are paid once per chain, not once per
    image.  chain_blocks None: one chain over everything (the reference's experiment layout, cifar_compress.py).
    stamp=True: the archive is followed by a stamp of codec.fingerprint() and these arguments (module docstring), which
    decompress_archive checks; the archive before it is unchanged.
    checksums=True: the archive is followed by a 32-bit digest of each block's pixels, in the archive's block sequence
    (module docstring), against which decompress_archive checks each block it decodes; a stamp goes after the digests."""
    chain_blocks = _check_chain_blocks(chain_blocks)
    if not (torch.is_tensor(images) or isinstance(images, np.ndarray)):
        images = list(images)
    if not len(images):
        raise ValueError("an archive holds at least one image")
    _check_stamp_args(scheme, excess_state_len, seed)
    blocks = _Blocks(codec, images, TILE_CODE, strict=True)
    gh, gw = _grid(blocks.shapes, TILE_CODE)
    total = int((gh * gw).sum())
    if total > MAX_ARCHIVE_BLOCKS:
        raise ValueError(f"the images hold {total} blocks, an archive at most {MAX_ARCHIVE_BLOCKS}")
    sizes = chain_sizes(total, chain_blocks)
    chains = list(zip(np.cumsum([0] + sizes[:-1]).tolist(), sizes))
    tail = _stamp_words(codec.fingerprint(), scheme, False, int(excess_state_len), int(seed)) if stamp else None
    args = (codec, blocks, _sequence_extents(blocks.shapes), chains, scheme, int(excess_state_len), int(seed), words_per_block)
    if checksums:
        coded, digests = _encode_checked(*args, np.array([0, total], dtype=np.int64))
    else:
        coded = _encode(*args)
    a = pack_archive(coded, blocks.shapes, int(excess_state_len), int(seed), scheme)
    if checksums:
        a = np.concatenate([a, _check_words(digests)])
    return a if tail is None else np.concatenate([a, tail])


def plan_archive(archive, regions=None):
    """The decode plan of decompress_archive, on the host alone: one RegionPlan over the archive's chains and its block
    sequence (every image's row-major blocks in turn).  regions None: every image whole."""
    job = _archive_job(archive)[0]
    return _plan(job, _all_images(job) if regions is None else regions)[1]


def decompress_archive(codec, archive, regions=None, as_tensors=False, verify=True):
    """regions None -> every image of the archive, exactly as given; else a list of (i, y, x, h, w) over image i -> one HWC
    uint8 array per region, byte-identical to the crop of the full decode.  Each chain holding a wanted block is popped
    from its end down to the earliest wanted block in it (plan_archive).  Every chain popped down to its first block must
    come back to the seeded initial state it was coded from; otherwise ValueError naming the chain.  A stamped archive must
    match the codec's fingerprint (ValueError naming every field that differs, before any decoding).  Every block a
    checked archive has decoded here must match its stored digest (ValueError naming the first that does not, after the
    stream flags; verify=False skips it).  as_tensors=True: contiguous torch.uint8 [h, w, C] CUDA tensors on the codec's
    device instead of numpy arrays."""
    job, n_init, seed, scheme, stamp, checks = _archive_job(archive)
    regions = _all_images(job) if regions is None else regions
    _check_stamps(codec, [stamp], scheme, False, None, "archive")
    return _decode_regions(codec, job, regions, None, scheme, False, None,
                           initial=[initial_words(n_init, seed=seed)] * len(job.cnb), as_tensors=as_tensors,
                           checks=checks if verify else None)


def _all_images(job):
    return [(i, 0, 0, h, w) for i, (h, w) in enumerate(job.shapes)]
