"""The digest definition of include/bitswap_b200.h (bsw_digest) in numpy -- TEST INFRASTRUCTURE.  `digest` vectorises
over chunks and lanes; `digest_scalar` walks the definition word by word for short inputs.  Imports without a GPU."""
import numpy as np

CHUNK = 8192
PA, PB = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xC2B2AE3D27D4EB4F)
CA, CB = 0x5354414D50484131, 0x5354414D50484232
DA, DB = 0x4449474553544131, 0x4449474553544232
M64 = (1 << 64) - 1


def mix(z):
    """splitmix64 finaliser on uint64 arrays (wrapping)."""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def rotl(x, r):
    return (x << np.uint64(r)) | (x >> np.uint64(64 - r))


def _words(data):
    data = bytes(data)
    return np.frombuffer(data + b"\0" * (-len(data) % 8), dtype="<u8").astype(np.uint64), len(data)


def _finish(n, ha, hb):
    da, db = mix(np.uint64(n ^ DA)), mix(np.uint64((n + DB) & M64))
    for a, b in zip(ha.tolist(), hb.tolist()):
        da = mix(da ^ np.uint64(a))
        with np.errstate(over="ignore"):
            db = mix(db + np.uint64(b))
    da, db = int(da), int(db)
    return [da & 0xffffffff, da >> 32, db & 0xffffffff, db >> 32]


def digest(data):
    """bsw_digest of `data` (bytes-like) as four uint32."""
    w, n = _words(data)
    nch = -(-w.size // CHUNK)
    if nch == 0:
        return _finish(n, np.zeros(0, np.uint64), np.zeros(0, np.uint64))
    padded = np.zeros(nch * CHUNK, dtype=np.uint64)
    padded[:w.size] = w
    W = padded.reshape(nch, CHUNK // 32, 32)                   # [chunk, step j, lane]: word 32 j + lane of the chunk
    c = np.arange(nch, dtype=np.uint64)[:, None]
    lane = np.arange(32, dtype=np.uint64)[None, :]
    a = mix((c << np.uint64(6)) | (np.uint64(2) * lane))
    b = mix((c << np.uint64(6)) | (np.uint64(2) * lane + np.uint64(1)))
    index = c * np.uint64(CHUNK) + lane
    with np.errstate(over="ignore"):
        for j in range(CHUNK // 32):
            live = index + np.uint64(32 * j) < np.uint64(w.size)
            x = W[:, j, :]
            a = np.where(live, rotl(a ^ x, 29) * PA, a)
            b = np.where(live, (rotl(b, 23) + x) * PB, b)
        ha, hb = mix(c[:, 0] ^ np.uint64(CA)), mix(c[:, 0] + np.uint64(CB))
        for l in range(32):
            ha, hb = mix(ha ^ a[:, l]), mix(hb + b[:, l])
    return _finish(n, ha, hb)


def _mix_int(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def digest_scalar(data):
    """The same definition with Python ints, one word at a time (slow: for short inputs)."""
    w, n = _words(data)
    w = [int(v) for v in w]
    rot = lambda x, r: ((x << r) | (x >> (64 - r))) & M64                    # noqa: E731
    da, db = _mix_int(n ^ DA), _mix_int((n + DB) & M64)
    for c in range(-(-len(w) // CHUNK)):
        chunk = w[c * CHUNK:(c + 1) * CHUNK]
        ha, hb = _mix_int(c ^ CA), _mix_int((c + CB) & M64)
        for lane in range(32):
            a, b = _mix_int((c << 6) | (2 * lane)), _mix_int((c << 6) | (2 * lane + 1))
            for x in chunk[lane::32]:
                a = (rot(a ^ x, 29) * int(PA)) & M64
                b = ((rot(b, 23) + x) * int(PB)) & M64
            ha, hb = _mix_int(ha ^ a), _mix_int((hb + b) & M64)
        da, db = _mix_int(da ^ ha), _mix_int((db + hb) & M64)
    return [da & 0xffffffff, da >> 32, db & 0xffffffff, db >> 32]


def hexdigest(out4):
    """Four uint32 as the 32 hex digits the package reports (bitswap_b200._lib.digest_hex)."""
    return np.asarray(out4, dtype="<u4").tobytes().hex()
