"""Codec / model hyper-parameters of the Bit-Swap hot path.

Mirrors the constructor arguments the reference's compression scripts use
(reference: cifar_compress.py:71-87,106; mnist_compress.py:72-88,107;
imagenet_compress.py:81-88,107; imagenetcrop_compress.py:89,100).
"""
import re
from dataclasses import dataclass, replace
from typing import Tuple


@dataclass(frozen=True)
class CodecConfig:
    xs: Tuple[int, int, int] = (3, 32, 32)   # image block shape (C,H,W); always 32x32
    nz: int = 8                              # number of latent levels
    zchannels: int = 8                       # latent channels (latents are zchannels x 16 x 16)
    nprocessing: int = 4                     # 5x5 ResNet layers on the x side
    kernel_size: int = 3
    resdepth: int = 8                        # total 3x3 ResNet layers, round-robin over levels
    reswidth: int = 252
    quantbits: int = 10                      # latent discretisation precision (2^q bins)
    ansbits: int = 31                        # rANS probability precision (cifar_compress.py:75)
    cond_xscale: bool = False                # imagenetcrop: x-scale is a conv head, not a parameter

    def __post_init__(self):
        # the reference's --kernel: ResNet blocks, z in-convs and heads; "same" padding needs it odd, and the device
        # convs are built for 1, 3, 5 and 7
        if self.kernel_size not in (1, 3, 5, 7):
            raise ValueError(f"kernel_size must be 1, 3, 5 or 7 (odd, at most 7), got {self.kernel_size!r}")

    @property
    def zdim(self) -> int:
        return self.zchannels * 16 * 16

    @property
    def xdim(self) -> int:
        return self.xs[0] * self.xs[1] * self.xs[2]

    @property
    def zsupport(self) -> int:
        return 1 << self.quantbits

    @property
    def level_resdepth(self):
        """Round-robin distribution of the 3x3 ResNet layers (model/cifar_train.py:66-72)."""
        d = [0] * self.nz
        i = 0
        for _ in range(self.resdepth):
            i = 0 if i == self.nz else i
            d[i] += 1
            i += 1
        return d

    @property
    def symbol_ops_per_image(self) -> int:
        return 2 * self.nz * self.zdim + self.xdim


def _cifar_width(nz):
    return {8: 252, 4: 254, 2: 255}.get(nz, 256)


def _mnist_width(nz):
    return {8: 61, 4: 62, 2: 63}.get(nz, 64)


def preset(name: str) -> CodecConfig:
    """Named configurations: cifar{1,2,4,8}, imagenet{...}, mnist{...}, imagenetcrop4, tiny*."""
    m = re.fullmatch(r"(cifar|imagenet)(\d+)", name)
    if m:
        nz = int(m.group(2))
        return CodecConfig(xs=(3, 32, 32), nz=nz, zchannels=8, reswidth=_cifar_width(nz))
    if name.startswith("mnist"):
        nz = int(name[5:])
        return CodecConfig(xs=(1, 32, 32), nz=nz, zchannels=1, reswidth=_mnist_width(nz))
    if name == "imagenetcrop4":
        return CodecConfig(xs=(3, 32, 32), nz=4, zchannels=8, reswidth=256, cond_xscale=True)
    if name == "tiny":      # small odd-width net for fast parity tests (not a reference config)
        return CodecConfig(xs=(1, 32, 32), nz=2, zchannels=1, nprocessing=2, resdepth=2, reswidth=15, quantbits=6)
    if name == "tiny3":     # RGB, 3 levels, conditional x-scale
        return CodecConfig(xs=(3, 32, 32), nz=3, zchannels=2, nprocessing=1, resdepth=3, reswidth=20,
                           quantbits=7, cond_xscale=True)
    raise KeyError(name)


with_ = replace
