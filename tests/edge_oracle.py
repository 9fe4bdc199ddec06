"""The oracle recursions for partial edge blocks -- TEST INFRASTRUCTURE.

`EdgeOracle` is `oracle.BitSwapOracle` with an `extent=(vh, vw)` argument on the four image calls.  The latent levels and
the prior are the parent class's, untouched.  At the pixel level only the dims (c, r, col) with r < vh and col < vw are
coded, with the tables those rows get in a full call, in the same order (push ascending, pop descending): in reference
terms `ANS(pmfs[valid], 31, 8).encode(state, x[valid])` and its inverse.  The block the nets see is the valid region
edge-padded with numpy (`np.pad(mode="edge")`), written here independently of the device's pad kernel so that it checks
it.

Mechanism: every pixel-level table goes through `_pmfs(self.xend, ...)` and then `_coder(...)` (push, pop, Bit-Swap and
BB-ANS alike), so those two hooks select the valid rows and wrap the coder so that it encodes x[valid] and decodes into
the padded block.
"""
import numpy as np
import torch

from oracle import oracle as O


class _MaskedCoder:
    def __init__(self, coder, orc):
        self.coder, self.orc = coder, orc

    def encode(self, state, symbols):
        return self.coder.encode(state, np.asarray(symbols)[self.orc._mask])

    def decode(self, state):
        state, sym = self.coder.decode(state)
        full = np.zeros(self.orc.cfg.xdim, dtype=np.int64)
        full[self.orc._mask] = np.asarray(sym)
        return state, torch.as_tensor(pad_block(full, self.orc._extent))


def x_mask(xdim, extent):
    """Flat CHW bool mask of the coded dims of a block with valid extent (vh, vw)."""
    vh, vw = int(extent[0]), int(extent[1])
    if not (1 <= vh <= 32 and 1 <= vw <= 32):
        raise ValueError(f"block extent {(vh, vw)} outside [1, 32] x [1, 32]")
    m = np.zeros((xdim // 1024, 32, 32), dtype=bool)
    m[:, :vh, :vw] = True
    return m.reshape(-1)


def pad_block(x, extent):
    """The padding rule: the valid region of the flat CHW block, edge-replicated to 32 x 32 (int64, flat)."""
    vh, vw = int(extent[0]), int(extent[1])
    v = np.asarray(x).reshape(-1, 32, 32)[:, :vh, :vw]
    return np.pad(v, ((0, 0), (0, 32 - vh), (0, 32 - vw)), mode="edge").reshape(-1).astype(np.int64)


class EdgeOracle(O.BitSwapOracle):
    _mask = None
    _extent = None
    _x_next = False

    def _pmfs(self, endpoints, mu, scale):
        if endpoints is self.xend and self._mask is not None:
            m = torch.from_numpy(self._mask)
            self._x_next = True
            return super()._pmfs(self.xend[m], mu[m], scale[m])
        return super()._pmfs(endpoints, mu, scale)

    def _coder(self, pmfs, q):
        coder = super()._coder(pmfs, q)
        if self._x_next:
            self._x_next = False
            return _MaskedCoder(coder, self)
        return coder

    def _with_extent(self, fn, state, extent, x=None):
        if extent is None:
            return fn(state) if x is None else fn(state, x)
        self._mask, self._extent = x_mask(self.cfg.xdim, extent), extent
        try:
            if x is None:
                return fn(state)
            return fn(state, pad_block(np.asarray(x).reshape(-1), extent))
        finally:
            self._mask = self._extent = None
            self._x_next = False

    def encode_image(self, state, x, extent=None):
        return self._with_extent(super().encode_image, state, extent, x)

    def decode_image(self, state, extent=None):
        return self._with_extent(super().decode_image, state, extent)

    def encode_image_bbans(self, state, x, extent=None):
        return self._with_extent(super().encode_image_bbans, state, extent, x)

    def decode_image_bbans(self, state, extent=None):
        return self._with_extent(super().decode_image_bbans, state, extent)
