"""Drop-in inference-time `Model` with the reference's call surface.

Reference: class Model, model/cifar_train.py:17-438 (identical in mnist_train /
imagenet_train; imagenetcrop_train differs by the conditional x-scale head,
:306-315,417).  Only the compression-time surface is provided -- the constructor
arguments, load_state_dict(), eval(), compress(), infer(i)(given) and
generate(i)(given); training (loss/sample/train/test) is out of scope.

The forward passes run in csrc/nets.cu (+ conv_tc.cu) through the C ABI
(bsw_model_* / bsw_vae_*); weight normalisation is folded once at load.
"""
import ctypes

import numpy as np
import torch

from ._lib import lib, check, cuda_stream_ptr, device_index, digest_hex, on_device
from .config import CodecConfig
from .synthetic import state_dict_spec


class _Desc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("xc", "nz", "zchannels", "nprocessing", "kernel_size", "resdepth",
                                              "reswidth", "cond_xscale", "max_batch", "use_tensor_cores")]


# Arithmetic of the tensor-core convs (BSW_TC_SPLIT / BSW_TC_BF16 of include/bitswap_b200.h)
TC_PRECISIONS = {"split": 0, "bf16": 1}


class Model:
    """tc_precision (tensor-core models only): "split" (default) runs every multiply-add as three bf16 MMAs on hi/lo
    operand planes, mu/sigma within 1e-4 of the float32 reference model; "bf16" runs one MMA on the RNE-rounded bf16
    operands, faster, mu/sigma a few 1e-3 off.  The two arithmetics give different bitstreams: a stream decodes only with
    a model of the arithmetic that encoded it."""

    def __init__(self, xs=(3, 32, 32), nz=1, zchannels=16, nprocessing=1, kernel_size=3, resdepth=2, reswidth=256,
                 dropout_p=0., tag='', root_process=True, cond_xscale=False, max_batch=1, use_tensor_cores=False, device=None,
                 tc_precision="split"):
        # the config validates the architecture (kernel_size: ValueError) before any device work
        self.cfg = CodecConfig(xs=tuple(xs), nz=nz, zchannels=zchannels, nprocessing=nprocessing, kernel_size=kernel_size,
                               resdepth=resdepth, reswidth=reswidth, cond_xscale=cond_xscale)
        if tc_precision not in TC_PRECISIONS:
            raise ValueError(f"tc_precision must be one of {sorted(TC_PRECISIONS)}, got {tc_precision!r}")
        if tc_precision != "split" and not use_tensor_cores:
            raise ValueError(f"tc_precision={tc_precision!r} needs use_tensor_cores=True: the float32 SIMT path has one "
                             "arithmetic")
        self._tc_precision = tc_precision
        if not torch.cuda.is_available():
            raise RuntimeError("bitswap_b200.Model needs a CUDA device (no CPU fallback)")
        assert tuple(xs[1:]) == (32, 32), "blocks are always 32x32 (latents 16x16)"
        self.xs, self.nz, self.zchannels = tuple(xs), nz, zchannels
        self.zdim = (zchannels, 16, 16)
        self.compressing = False
        self.max_batch = int(max_batch)
        self._desc = _Desc(xs[0], nz, zchannels, nprocessing, kernel_size, resdepth, reswidth, int(cond_xscale), self.max_batch,
                           int(use_tensor_cores))
        self.device = device_index(device)
        self._h = ctypes.c_void_p()
        self._sd = None
        self._create()

    def _create(self):
        self._destroy()
        with on_device(self.device):
            check(lib().bsw_model_create(ctypes.byref(self._h), ctypes.byref(self._desc)))
            if self._desc.use_tensor_cores:
                check(lib().bsw_model_set_tc_precision(self._h, TC_PRECISIONS[self._tc_precision]))
        self._loaded = False

    def _destroy(self):
        if getattr(self, "_h", None):
            try:
                with on_device(self.device):
                    lib().bsw_model_destroy(self._h)
            except Exception:
                pass
            self._h = ctypes.c_void_p()

    @classmethod
    def from_config(cls, cfg: CodecConfig, **kw):
        return cls(xs=cfg.xs, nz=cfg.nz, zchannels=cfg.zchannels, nprocessing=cfg.nprocessing,
                   kernel_size=cfg.kernel_size, resdepth=cfg.resdepth, reswidth=cfg.reswidth,
                   cond_xscale=cfg.cond_xscale, **kw)

    def __del__(self):
        self._destroy()

    @property
    def handle(self):
        return self._h

    def digest(self):
        """Digest of the folded weights the kernels read (bsw_model_digest), 32 hex digits: equal for every instance of
        one state dict, whatever its max_batch, conv path or tc_precision.  Computed once per loaded handle, so
        load_state_dict() and to(), which re-create it, start afresh."""
        assert self._loaded, "load_state_dict() first"
        out = (ctypes.c_uint32 * 4)()
        with on_device(self.device):
            check(lib().bsw_model_digest(self._h, out, cuda_stream_ptr()))
        return digest_hex(out)

    @property
    def tc_precision(self):
        """"split" or "bf16": the arithmetic of the tensor-core convs (fixed at construction)."""
        return self._tc_precision

    # -- nn.Module-shaped no-ops the compression scripts call ---------------------------------------
    def to(self, device=None, *a, **k):
        """nn.Module.to(device): the handle (weights, activations) lives on ONE device; moving re-creates it there and
        reloads the weights.  The reference scripts call Model(...).to(f"cuda:{gpu}") before load_state_dict."""
        if device is None or isinstance(device, torch.dtype):
            return self
        idx = device_index(device)
        if idx != self.device:
            sd = self._sd
            self._destroy()
            self.device = idx
            self._create()
            if sd is not None:
                self.load_state_dict(sd)
        return self

    def eval(self):
        return self

    def compress(self, compress=True):          # model/cifar_train.py:311-312
        self.compressing = compress

    def load_state_dict(self, sd, strict=True):
        """Accepts the reference checkpoint layout (SURVEY.md A2)."""
        spec = state_dict_spec(self.cfg)
        keys = [k for k, _, _ in spec]
        if strict:
            missing, extra = [k for k in keys if k not in sd], [k for k in sd if k not in keys]
            if missing or extra:
                raise RuntimeError(f"state_dict mismatch: missing {missing[:4]} unexpected {extra[:4]}")
        f32 = lambda t: np.ascontiguousarray(t.detach().cpu().numpy(), dtype=np.float32)   # noqa: E731
        self._sd = sd
        if self._loaded:
            self._create()
        with on_device(self.device):
            self._load(sd, spec, f32)
        self._loaded = True
        return self

    def _load(self, sd, spec, f32):
        for key, shape, kind in spec:
            if kind == "gen_std":
                a = f32(sd[key])
                assert a.shape == shape
                check(lib().bsw_model_load_gen_std(self._h, a.ctypes.data))
            elif kind == "v":
                prefix = key[:-2]
                v, g, b = f32(sd[key]), f32(sd[prefix + ".gain"]), f32(sd[prefix + ".b"])
                assert v.shape == shape, (key, v.shape, shape)
                loggain = 0 if prefix.endswith(".conv2") else 1          # modules.py:223-227
                check(lib().bsw_model_load_conv(self._h, prefix.encode(), v.ctypes.data, g.ctypes.data, b.ctypes.data,
                                                shape[0], shape[1], shape[2], loggain))
        check(lib().bsw_model_finalize(self._h))

    # -- infer / generate -----------------------------------------------------------------------------
    def _run(self, infer, i, given):
        assert self._loaded, "load_state_dict() first"
        assert self.compressing, "only compressing mode is provided (model.compress())"
        in_dtype = given.dtype
        flat_in = given.dim() == 1
        cfg = self.cfg
        dim_in = cfg.xdim if (infer and i == 0) else cfg.zdim
        dim_out = cfg.xdim if (not infer and i == 0) else cfg.zdim
        dev = torch.device("cuda", self.device)
        g = given.to(device=dev, dtype=torch.float32).reshape(-1, dim_in).contiguous()    # h.float(), :324,:392
        n = g.shape[0]
        assert n <= self.max_batch, f"batch {n} > max_batch {self.max_batch}"
        mu = torch.empty((n, dim_out), dtype=torch.float32, device=dev)
        sc = torch.empty((n, dim_out), dtype=torch.float32, device=dev)
        with on_device(self.device):
            if infer:
                check(lib().bsw_vae_infer(self._h, i, g.data_ptr(), n, mu.data_ptr(), sc.data_ptr(), cuda_stream_ptr()))
            else:
                check(lib().bsw_vae_generate(self._h, i, g.data_ptr(), n, mu.data_ptr(), sc.data_ptr(), 1, cuda_stream_ptr()))
        if flat_in:
            mu, sc = mu.view(-1), sc.view(-1)
        return mu.to(in_dtype), sc.to(in_dtype)                       # .type(type), :375-376,:434-435

    def infer(self, i):
        return lambda given: self._run(True, i, given)

    def generate(self, i):
        return lambda given: self._run(False, i, given)
