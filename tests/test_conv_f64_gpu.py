"""P3c: every conv kernel on its own against a float64 evaluation of the same conv, with the harness of conv_harness.py
(inputs, value sets, the bound |out - f(y)| <= tau * s + allowances, exact checks) on [2, MAXB, 256, 256] plane buffers."""
import pytest

pytestmark = pytest.mark.gpu

from conv_harness import VALUES, Case, conv_cfg, worst_report      # noqa: E402

# (tensor cores?, config).  zchannels 1..32 run the in-conv on the tensor cores, 40 the SIMT in-conv + split; heads of
# 2 * zc <= 32 outputs run on the tensor cores, 20 and 32 (TCO = 8 variant at 64 outputs) and 40 on k_conv_simt.
MODELS = {
    "tc W252 zc1 C3": (True, conv_cfg(3, 1, 252)),
    "tc W193 zc2 C1 cond": (True, conv_cfg(1, 2, 193, cond=True)),
    "tc W255 zc8 C3 cond": (True, conv_cfg(3, 8, 255, cond=True)),
    "tc W256 zc16 C1": (True, conv_cfg(1, 16, 256)),
    "tc W252 zc20 C3": (True, conv_cfg(3, 20, 252)),
    "tc W193 zc32 C1": (True, conv_cfg(1, 32, 193)),
    "tc W255 zc40 C3 cond": (True, conv_cfg(3, 40, 255, cond=True)),
    "simt W15 zc1 C1": (False, conv_cfg(1, 1, 15)),
    "simt W20 zc2 C3 cond": (False, conv_cfg(3, 2, 20, cond=True)),
    "simt W63 zc32 C1": (False, conv_cfg(1, 32, 63)),
    "simt W252 zc20 C3": (False, conv_cfg(3, 20, 252)),
}
WORST = {}                                           # (path, kind) -> worst normalised error, reported at the end
_report = worst_report("P3c per-layer float64 parity: worst |out - f(y)| / s (beyond the ELU/rounding allowance)", WORST)


@pytest.mark.parametrize("vs", VALUES)
@pytest.mark.parametrize("name", list(MODELS))
def test_conv_kernels_vs_float64(name, vs):
    Case(MODELS, name, vs, seed_base=1000, worst=WORST, plane_width=256).run()
