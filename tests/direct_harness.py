"""The direct-cdf quantiser in numpy, its oracle recursion and its level runners -- TEST INFRASTRUCTURE.

`direct_tables` is the format's definition restated on float64 cdf values (bsw_direct_push in include/bitswap_b200.h);
`DirectOracle` is the oracle recursion (`EdgeOracle`, GPU nets injected by `codec_harness.gpu_oracle`) with every level, the
pixels and the prior quantised by it from torch-CUDA's float64 sigmoid; `direct_level` runs one level's pop or push through
the C ABI.  Imports without a GPU."""
import numpy as np
import torch

from edge_oracle import EdgeOracle, _MaskedCoder
from oracle import oracle as O
from bitswap_b200.streams import StreamSet
from bitswap_b200._lib import lib, check, cuda_stream_ptr

TOTAL = 1 << 31


def direct_tables(F):
    """P [L, S] and C [L, S + 1] (int64) of the direct quantiser from the float cdf values F [L, S - 1] at the endpoints:
    C_0 = 0, C_S = 2^31, C_k = floor(RN(F_{k-1} (2^31 - 2S))) + 2k; a NaN F counts as 0."""
    F = np.asarray(F, dtype=np.float64)
    F = np.where(np.isnan(F), 0.0, F)
    L, S = F.shape[0], F.shape[1] + 1
    C = np.zeros((L, S + 1), dtype=np.int64)
    C[:, 1:S] = np.floor(F * float(TOTAL - 2 * S)).astype(np.int64) + 2 * np.arange(1, S, dtype=np.int64)
    C[:, S] = TOTAL
    return np.diff(C, axis=1), C


def torch_cdfs(ends, mu, sc):
    """torch.sigmoid((e - mu) / sigma) in float64 on the GPU, rows [L, S - 1]; mu, sc [L] or [1] (float32 values up-cast)."""
    e = torch.from_numpy(np.array(ends, dtype=np.float64)).cuda()
    m = torch.as_tensor(np.asarray(mu)).double().cuda()
    s = torch.as_tensor(np.asarray(sc)).double().cuda()
    return torch.sigmoid((e.t() - m) / s).t().cpu().numpy()


class DirectOracle(EdgeOracle):
    """The oracle recursion with the direct quantiser: `_pmfs` hands on the cdf values of the reference's expression on
    torch-CUDA (what the kernels' float64 cdf is bit-matched to) instead of pmfs, and `_coder` quantises them directly."""

    def _pmfs(self, endpoints, mu, scale):
        if endpoints is self.xend and self._mask is not None:
            m = torch.from_numpy(self._mask)
            self._x_next = True
            endpoints, mu, scale = self.xend[m], mu[m], scale[m]
        return torch.sigmoid((endpoints.cuda().t() - mu.cuda()) / scale.cuda()).t().cpu().numpy()

    def _coder(self, cdfs, q):
        coder = O.AnsC(tables=direct_tables(cdfs))
        if self._x_next:                  # the pixel level of a partial block (EdgeOracle)
            self._x_next = False
            return _MaskedCoder(coder, self)
        return coder


def _level_args(ends_pad, mu, sc, ers):
    e = torch.from_numpy(np.ascontiguousarray(ends_pad)).cuda()
    dmu, dsc = torch.from_numpy(np.ascontiguousarray(mu)).cuda(), torch.from_numpy(np.ascontiguousarray(sc)).cuda()
    return e, dmu, dsc


def direct_level(pop, ends_pad, mu, sc, S, states, sym=None, ers=None, mss=None, sss=None, cap=1 << 15):
    """One direct pop (pop=True) or push of a level through bsw_direct_pop / bsw_direct_push on streams holding `states`.
    ends_pad: [L, S] padded rows, or one [S] row with ers = 0.  Returns (the StreamSet, popped symbols [B, L] or None)."""
    B, L = mu.shape
    ers = S if ers is None else ers
    e, dmu, dsc = _level_args(ends_pad, mu, sc, ers)
    nbytes = int(lib().bsw_logistic_scratch_bytes(B, L, S, 0))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    ss = StreamSet(B, cap)
    ss.import_lists(states)
    args = (ss.handle, 0, B, dmu.data_ptr(), L if mss is None else mss, dsc.data_ptr(), L if sss is None else sss,
            e.data_ptr(), ers)
    if pop:
        out = torch.zeros((B, L), dtype=torch.int16, device="cuda")
        check(lib().bsw_direct_pop(*args, out.data_ptr(), L, S, 31, 0, scratch.data_ptr(), nbytes, cuda_stream_ptr()))
    else:
        out = torch.from_numpy(np.ascontiguousarray(sym, dtype=np.int16)).cuda()
        check(lib().bsw_direct_push(*args, out.data_ptr(), L, S, 31, 0, scratch.data_ptr(), nbytes, cuda_stream_ptr()))
    torch.cuda.synchronize()
    return ss, (out.cpu().numpy().astype(np.int64) if pop else None)
