"""The block digest of include/bitswap_b200.h (bsw_block_digest) in numpy -- TEST INFRASTRUCTURE.  `block_digests`
vectorises over slots and lanes; `block_digest_scalar` walks the definition byte by byte with Python ints; `kernel_twin`
is what bsw_block_digests writes for a block buffer and its per-slot table.  Imports without a GPU."""
import numpy as np

SEED = 0x424C4F434B534551
P = 0x9E3779B1
M32, M64 = (1 << 32) - 1, (1 << 64) - 1


def _mix64(z):
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _fmix32(h):
    h = np.asarray(h, dtype=np.uint32)
    with np.errstate(over="ignore"):
        h = h ^ (h >> np.uint32(16))
        h = h * np.uint32(0x85EBCA6B)
        h = h ^ (h >> np.uint32(13))
        h = h * np.uint32(0xC2B2AE35)
    return h ^ (h >> np.uint32(16))


def block_digests(slots, index, extents=None):
    """bsw_block_digest of every slot: slots uint8 [n, C, 32, 32], index int [n] (each block's index in its own sequence),
    extents int [n, 2] (vh, vw) or None (full) -> uint32 [n]."""
    slots = np.asarray(slots, dtype=np.uint8)
    n, C = slots.shape[:2]
    ext = np.full((n, 2), 32, dtype=np.int64) if extents is None else np.asarray(extents, dtype=np.int64).reshape(n, 2)
    vh, vw = ext[:, 0], ext[:, 1]
    key = (np.asarray(index, dtype=np.uint64) << np.uint64(16)) | (vh.astype(np.uint64) << np.uint64(8)) | vw.astype(np.uint64)
    s = _mix64(key ^ np.uint64(SEED))
    lane = np.arange(32, dtype=np.uint64)
    with np.errstate(over="ignore"):
        a = (_mix64(s[:, None] + lane[None, :] + np.uint64(1)) & np.uint64(M32)).astype(np.uint32)
        cols = lane[None, :].astype(np.int64) < vw[:, None]
        for c in range(C):
            for r in range(32):
                live = cols & (r < vh)[:, None]
                x = a ^ slots[:, c, r, :].astype(np.uint32)
                step = ((x << np.uint32(13)) | (x >> np.uint32(19))) * np.uint32(P)
                a = np.where(live, step, a)
        h = (s >> np.uint64(32)).astype(np.uint32)
        for l in range(32):
            h = _fmix32(h ^ a[:, l])
    return h


def _mix64_int(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def _fmix32_int(h):
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M32
    return h ^ (h >> 16)


def block_digest_scalar(slot, index, vh=32, vw=32):
    """The definition, literally: one slot uint8 [C, 32, 32], its block's index in its sequence, its extent."""
    slot = np.asarray(slot, dtype=np.uint8)
    index, vh, vw = int(index), int(vh), int(vw)
    s = _mix64_int(((index << 16) | (vh << 8) | vw) ^ SEED)
    h = s >> 32
    for lane in range(32):
        a = _mix64_int((s + lane + 1) & M64) & M32
        if lane < vw:
            for c in range(slot.shape[0]):
                for r in range(vh):
                    x = a ^ int(slot[c, r, lane])
                    a = ((((x << 13) | (x >> 19)) & M32) * P) & M32
        h = _fmix32_int(h ^ a)
    return h


def kernel_twin(x, block, seq_offsets, extents=None, out=None):
    """What bsw_block_digests writes: x uint8 [..., C, 32, 32] slots, block int64 [...] (sequence index per slot, -1 none),
    seq_offsets int64 [n + 1], extents int16 [..., 2] or None; out uint32 [total] (zeros if None) receives them."""
    x = np.asarray(x, dtype=np.uint8)
    C = x.shape[-3]
    slots, block = x.reshape(-1, C, 32, 32), np.asarray(block, dtype=np.int64).reshape(-1)
    offs = np.asarray(seq_offsets, dtype=np.int64)
    out = np.zeros(int(offs[-1]), dtype=np.uint32) if out is None else out
    live = block >= 0
    g = block[live]
    index = g - offs[np.searchsorted(offs[:-1], g, side="right") - 1]
    ext = None if extents is None else np.asarray(extents).reshape(-1, 2)[live]
    out[g] = block_digests(slots[live], index, ext)
    return out
