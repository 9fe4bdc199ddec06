"""Batched, device-resident Bit-Swap / BB-ANS codec (host-side handle of `bsw_codec`).

Replaces the sender/receiver loop bodies of the reference's compress()
(cifar_compress.py:175-250 and :283-352): one call codes one image per stream for
a whole batch of independent chains; the ANS state never leaves the GPU between
latent levels.  Chain more images onto the same streams by calling again.
"""
import collections
import ctypes

import numpy as np
import torch

from ._lib import lib, check, cuda_stream_ptr, device_index, digest_hex, on_device
from .config import CodecConfig
from .model import TC_PRECISIONS, Model
from .streams import StreamSet

BITSWAP, BBANS = 0, 1
MIN_QUANTBITS = 5           # narrowest latent support of the device codec: 32 bins (every coder kernel owns S/32 bins per lane)
MAX_QUANTBITS = 12          # widest latent support of the device codec: 4096 bins
FUSED_MAX_SUPPORT = 1024    # the fused coder keeps a row table in one warp's registers
# Quantiser of the coder (BSW_CODER_REFERENCE / BSW_CODER_DIRECT of include/bitswap_b200.h)
CODERS = {"reference": 0, "direct": 1}


Fingerprint = collections.namedtuple(
    "Fingerprint", "revision xc nz zchannels nprocessing kernel_size resdepth reswidth cond_xscale quantbits "
                   "use_tensor_cores tc_precision tc_heads coder model_digest bins_digest")
Fingerprint.__doc__ = """Everything that decides a codec's bitstreams (bsw_codec_fingerprint): the bitstream revision of the library, the
model's architecture, quantbits, the conv path (use_tensor_cores, tc_precision "split" / "bf16", tc_heads: whether the heads
run on the tensor cores), the coder ("reference" / "direct") and 32-hex-digit digests of the folded weights and of the bin
tables the kernels read.  Two codecs with equal fingerprints write and read the same bitstreams."""


class _Fp(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in Fingerprint._fields[:14]] + [("model_digest", ctypes.c_uint32 * 4),
                                                                          ("bins_digest", ctypes.c_uint32 * 4)]


def device_digest(t):
    """bsw_digest of a contiguous CUDA tensor's bytes, as 32 hex digits (see include/bitswap_b200.h for the definition)."""
    assert t.is_cuda and t.is_contiguous()
    out = (ctypes.c_uint32 * 4)()
    with on_device(t.device.index):
        check(lib().bsw_digest(ctypes.c_void_p(t.data_ptr()), t.numel() * t.element_size(), out, cuda_stream_ptr()))
    return digest_hex(out)


def check_coder(coder):
    """ValueError unless `coder` is "reference" or "direct" (raised before any device work)."""
    if not (isinstance(coder, str) and coder in CODERS):
        raise ValueError(f"coder must be one of {sorted(CODERS)}, got {coder!r}")


def check_quantbits(q):
    """ValueError unless MIN_QUANTBITS <= q <= MAX_QUANTBITS (raised before any device work)."""
    if not (isinstance(q, (int, np.integer)) and MIN_QUANTBITS <= int(q) <= MAX_QUANTBITS):
        raise ValueError(f"quantbits must be an integer in [{MIN_QUANTBITS}, {MAX_QUANTBITS}], got {q!r}: the top latent level "
                         f"is coded by kernels that own 2^quantbits / 32 bins per lane, so 32 bins is the narrowest support "
                         f"the codec codes and 4096 the widest")


class Bins:
    """Device copy of the discretisation tables (zendpoints [nz,zdim,2^q-1], zcentres [nz,zdim,2^q],
    the layout discretize() returns, discretization.py:99).  quantbits 5 to 12: 32 to 4096 bins per latent dimension
    (at 12, cifar8's bins take 1.07 GB of device memory); any other quantbits raises ValueError here."""

    def __init__(self, cfg: CodecConfig, zendpoints, zcentres, device=None):
        check_quantbits(cfg.quantbits)
        self.device = device_index(device)
        ze = np.ascontiguousarray(zendpoints.detach().cpu().numpy() if torch.is_tensor(zendpoints) else zendpoints, dtype=np.float64)
        zc = np.ascontiguousarray(zcentres.detach().cpu().numpy() if torch.is_tensor(zcentres) else zcentres, dtype=np.float64)
        assert ze.shape == (cfg.nz, cfg.zdim, cfg.zsupport - 1) and zc.shape == (cfg.nz, cfg.zdim, cfg.zsupport)
        self._h = ctypes.c_void_p()
        with on_device(self.device):
            check(lib().bsw_bins_create(ctypes.byref(self._h), cfg.nz, cfg.zdim, cfg.quantbits, cfg.xdim, ze.ctypes.data, zc.ctypes.data))

    def level_is_uniform(self, level):
        """True if every endpoint row of latent level `level` (-1: the pixel row) is a uniform grid (affine-row kernels)."""
        return bool(lib().bsw_bins_level_is_uniform(self._h, int(level)))

    @property
    def handle(self):
        return self._h

    def digest(self):
        """Digest of these bin tables as stored on the device (bsw_bins_digest), 32 hex digits; computed once."""
        out = (ctypes.c_uint32 * 4)()
        with on_device(self.device):
            check(lib().bsw_bins_digest(self._h, out, cuda_stream_ptr()))
        return digest_hex(out)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                lib().bsw_bins_destroy(h)
            except Exception:
                pass
            self._h = None


class BitSwapCodec:
    """coder: "reference" (default) quantises every level as the reference's ANS.__init__ does, so its bitstreams are the
    reference's; "direct" quantises each bin's cdf on its own (see bsw_direct_push), which needs no whole-row table and
    codes faster at the same rate, with its own bitstreams: a stream decodes only with the coder that encoded it."""

    def __init__(self, cfg: CodecConfig, model: Model, bins: Bins, max_batch: int, coder: str = "reference"):
        check_coder(coder)
        self.cfg, self.model, self.bins, self.max_batch = cfg, model, bins, int(max_batch)
        self.device = model.device
        if bins.device != self.device:
            raise ValueError(f"model is on cuda:{model.device} but the bin tables are on cuda:{bins.device}")
        self._h = ctypes.c_void_p()
        with on_device(self.device):
            check(lib().bsw_codec_create(ctypes.byref(self._h), model.handle, bins.handle, self.max_batch))
            check(lib().bsw_codec_set_coder(self._h, CODERS[coder]))
        self._coder = coder

    @property
    def coder(self):
        """The quantiser this codec codes with: "reference" or "direct"."""
        return self._coder

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                lib().bsw_codec_destroy(h)
            except Exception:
                pass
            self._h = None

    def encode(self, streams: StreamSet, x: torch.Tensor, first=0, scheme=BITSWAP, extent=None):
        """x: uint8 CUDA tensor [count, C, 32, 32]; pushes one image onto each of `count` streams. Async.
        extent: None (full blocks) or an int16 CUDA tensor [count, 2] of valid block extents (vh, vw) in [1, 32]: only the
        pixels inside the extent are coded, the rest of the block is ignored (see bsw_codec_encode_ext)."""
        assert x.is_cuda and x.dtype == torch.uint8 and x.is_contiguous()
        self._same_device(streams, x)
        count = x.shape[0]
        with on_device(self.device):
            if extent is None:
                check(lib().bsw_codec_encode(self._h, streams.handle, first, count, x.data_ptr(), scheme, cuda_stream_ptr()))
            else:
                ext = self._extent(extent, count)
                check(lib().bsw_codec_encode_ext(self._h, streams.handle, first, count, x.data_ptr(), ext.data_ptr(), scheme,
                                                 cuda_stream_ptr()))

    def _extent(self, extent, count):
        if not (torch.is_tensor(extent) and extent.is_cuda and extent.dtype == torch.int16 and extent.is_contiguous()
                and tuple(extent.shape) == (count, 2)):
            raise ValueError(f"extent: need a contiguous int16 CUDA tensor of shape ({count}, 2)")
        if extent.device.index != self.device:
            raise ValueError(f"codec is on cuda:{self.device}, extents on {extent.device}")
        return extent

    def _same_device(self, streams, x=None):
        if streams.device != self.device or (x is not None and x.device.index != self.device):
            raise ValueError(f"codec is on cuda:{self.device}; streams on cuda:{streams.device}"
                             + (f", pixels on {x.device}" if x is not None else ""))

    def decode(self, streams: StreamSet, count: int, first=0, scheme=BITSWAP, out=None, extent=None):
        """Pops one image from each stream; returns uint8 CUDA tensor [count, C, 32, 32]. Async.
        extent: the tensor the images were encoded with (None = full blocks); pixels outside it come back edge-padded."""
        if out is None:
            out = torch.empty((count,) + tuple(self.cfg.xs), dtype=torch.uint8, device=torch.device("cuda", self.device))
        if not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.numel() >= count * int(np.prod(self.cfg.xs))):
            raise ValueError("decode(out=...): need a contiguous uint8 CUDA tensor with room for `count` images")
        self._same_device(streams, out)
        with on_device(self.device):
            if extent is None:
                check(lib().bsw_codec_decode(self._h, streams.handle, first, count, out.data_ptr(), scheme, cuda_stream_ptr()))
            else:
                ext = self._extent(extent, count)
                check(lib().bsw_codec_decode_ext(self._h, streams.handle, first, count, out.data_ptr(), ext.data_ptr(), scheme,
                                                 cuda_stream_ptr()))
        return out

    @property
    def last_launches(self):
        return int(lib().bsw_codec_last_launches(self._h))

    def fingerprint(self):
        """The Fingerprint of this codec as it is now (the coder it was last set to).  The digests are computed on the
        device the first time and kept with the model and the bins."""
        f = _Fp()
        with on_device(self.device):
            check(lib().bsw_codec_fingerprint(self._h, ctypes.byref(f), cuda_stream_ptr()))
        precision = {v: k for k, v in TC_PRECISIONS.items()}
        coders = {v: k for k, v in CODERS.items()}
        return Fingerprint(f.revision, f.xc, f.nz, f.zchannels, f.nprocessing, f.kernel_size, f.resdepth, f.reswidth,
                           bool(f.cond_xscale), f.quantbits, bool(f.use_tensor_cores), precision[f.tc_precision],
                           bool(f.tc_heads), coders[f.coder], digest_hex(f.model_digest), digest_hex(f.bins_digest))

    CATEGORIES = ("misc", "conv_in", "conv_dense3x3", "conv_dense5x5", "conv_head", "pop_z", "push_z", "pop_x",
                  "push_x", "prior", "rows_z", "rows_x")

    def set_dual_stream(self, on=True):
        """True: overlap mode -- the recursion is enqueued as a dependency graph on three internal streams (nets, float64
        table kernels, serial coder kernels), so that the tensor-pipe and the FP64-pipe work of one chain share the SMs;
        False (default): plain program order on the caller's stream.  Same results either way."""
        check(lib().bsw_codec_set_dual_stream(self._h, int(on)))

    def set_two_phase(self, on=True):
        """True (default): parallel row-table kernel + serial coder; False: fused one-warp-per-stream kernels, which hold a
        row's table in registers and so take at most 1024 bins (quantbits <= 10): ValueError above that.  The switch picks
        between reference coders: ValueError on a direct codec."""
        if not on and self._coder != "reference":
            raise ValueError("set_two_phase(False): the direct coder has only its two-phase kernels; the fused coder is a "
                             "reference coder")
        if not on and self.cfg.zsupport > FUSED_MAX_SUPPORT:
            raise ValueError(f"set_two_phase(False): the fused coder takes at most {FUSED_MAX_SUPPORT} bins per row, these bins "
                             f"have {self.cfg.zsupport} (quantbits {self.cfg.quantbits}); keep the two-phase coder")
        check(lib().bsw_codec_set_two_phase(self._h, int(on)))

    def profile(self, enable=-1):
        """Per-kernel-category device time since profiling was enabled: {name: (ms, launches)}.
        enable: True/False resets and starts/stops, -1 just reads."""
        ms = np.zeros(12, dtype=np.float64)
        n = np.zeros(12, dtype=np.int64)
        check(lib().bsw_codec_profile(self._h, int(enable), ms.ctypes.data, n.ctypes.data))
        return {k: (float(ms[i]), int(n[i])) for i, k in enumerate(self.CATEGORIES)}


class PipelinedCodec:
    """`lanes` BitSwapCodecs, each coding a contiguous sub-range of the streams on its own CUDA stream.

    The coder's row-table kernel is FP64-pipe bound and the dense convs are tensor-pipe bound; chains of
    different sub-batches drift apart in phase, so their kernels share SMs and the two pipes overlap
    (4 lanes by default).  Results are identical to a single BitSwapCodec: every stream is independent and every kernel is
    batch-invariant.  Each lane owns a model replica (activations are per-lane anyway).  tc_precision: the arithmetic of
    every lane's tensor-core convs ("split" or "bf16", see Model); coder: the quantiser of every lane ("reference" or
    "direct", see BitSwapCodec).  Both change the bitstreams."""

    def __init__(self, cfg: CodecConfig, state_dict, bins: Bins, max_batch: int, lanes: int = 4, use_tensor_cores=True, lane_size: int = 0,
                 free_running: bool = False, tc_precision: str = "split", coder: str = "reference"):
        check_coder(coder)
        self.cfg, self.bins, self.max_batch = cfg, bins, int(max_batch)
        self.device = bins.device
        self.lanes = max(1, min(int(lanes), self.max_batch))
        self.per = -(-self.max_batch // self.lanes)
        if lane_size > 0:             # explicit sub-batch size (the last lane takes the remainder), e.g. a multiple of SMs/2
            self.per = min(int(lane_size), self.max_batch)
            self.lanes = -(-self.max_batch // self.per)
        self.models, self.codecs, self.streams = [], [], []
        self.serial = False          # True: run the lanes back to back on the current stream (clean per-kernel timing)
        # free_running: calls fork the lanes from the current stream but do NOT join them back -- consecutive encode()/
        # decode() calls then chain per lane (a lane may be decoding while its neighbour still encodes), and the caller orders
        # later work after the codec with join().  (A start offset between the lanes was tried -- all lanes run the same
        # program, so their latency-bound serial coder phases could coincide -- and measured no effect: they drift apart on
        # their own within a step.)
        self.free_running = bool(free_running)
        for _ in range(self.lanes):
            m = Model.from_config(cfg, max_batch=self.per, use_tensor_cores=use_tensor_cores, device=self.device,
                                  tc_precision=tc_precision).load_state_dict(state_dict)
            m.compress()
            self.models.append(m)
            self.codecs.append(BitSwapCodec(cfg, m, bins, self.per, coder=coder))
            self.streams.append(torch.cuda.Stream(device=self.device))

    def _ranges(self, count):
        out, b = [], 0
        while b < count:
            out.append((b, min(self.per, count - b)))
            b += self.per
        return out

    def _fan(self, count, fn):
        if self.serial:
            for i, (b, n) in enumerate(self._ranges(count)):
                fn(self.codecs[i], b, n)
            return
        cur = torch.cuda.current_stream(self.device)
        ev = torch.cuda.Event()
        ev.record(cur)
        for i, (b, n) in enumerate(self._ranges(count)):
            st = self.streams[i]
            st.wait_event(ev)
            with torch.cuda.stream(st):
                fn(self.codecs[i], b, n)
        if not self.free_running:
            self.join()

    def join(self):
        """The current stream waits for everything the lanes have been given so far."""
        cur = torch.cuda.current_stream(self.device)
        for st in self.streams:
            cur.wait_stream(st)

    def encode(self, streams: StreamSet, x: torch.Tensor, first=0, scheme=BITSWAP, extent=None):
        assert x.is_cuda and x.dtype == torch.uint8 and x.is_contiguous() and x.shape[0] <= self.max_batch
        self._fan(x.shape[0], lambda c, b, n: c.encode(streams, x[b:b + n], first=first + b, scheme=scheme,
                                                       extent=None if extent is None else extent[b:b + n]))

    def decode(self, streams: StreamSet, count: int, first=0, scheme=BITSWAP, out=None, extent=None):
        if out is None:
            out = torch.empty((count,) + tuple(self.cfg.xs), dtype=torch.uint8, device=torch.device("cuda", self.device))
        self._fan(count, lambda c, b, n: c.decode(streams, n, first=first + b, scheme=scheme, out=out[b:b + n],
                                                  extent=None if extent is None else extent[b:b + n]))
        return out

    @property
    def coder(self):
        return self.codecs[0].coder

    def fingerprint(self):
        """The lanes' common Fingerprint; RuntimeError if two lanes would write different bitstreams."""
        fps = [c.fingerprint() for c in self.codecs]
        for i, f in enumerate(fps[1:], 1):
            if f != fps[0]:
                raise RuntimeError(f"lane {i} of this PipelinedCodec has fingerprint {f}, lane 0 {fps[0]}")
        return fps[0]

    def set_two_phase(self, on=True):
        if not on and self.coder != "reference":
            raise ValueError("set_two_phase(False): the direct coder has only its two-phase kernels; the fused coder is a "
                             "reference coder")
        if not on and self.cfg.zsupport > FUSED_MAX_SUPPORT:
            raise ValueError(f"set_two_phase(False): the fused coder takes at most {FUSED_MAX_SUPPORT} bins per row, these bins "
                             f"have {self.cfg.zsupport} (quantbits {self.cfg.quantbits}); keep the two-phase coder")
        for c in self.codecs:
            c.set_two_phase(on)

    def set_dual_stream(self, on=True):
        for c in self.codecs:
            c.set_dual_stream(on)

    @property
    def last_launches(self):
        return sum(c.last_launches for c in self.codecs)

    def profile(self, enable=-1):
        tot = {}
        for c in self.codecs:
            for k, (ms, n) in c.profile(enable).items():
                a = tot.get(k, (0.0, 0))
                tot[k] = (a[0] + ms, a[1] + n)
        return tot
