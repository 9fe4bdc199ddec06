"""bitswap_b200 -- H100-native Bit-Swap hot path (rANS over discretised-logistic
tables + hierarchical-VAE mu/sigma nets) behind the reference's Python call
surface.  See DESIGN.md / INTEGRATION.md."""
from .config import CodecConfig, preset  # noqa: F401
