"""Models wider than 256 channels on the float32 SIMT convs and on the tensor cores (the k_conv_wg tiles of padded widths
384 / 512, which fold the main accumulator once per tap), measured alternately in one process with the protocol and
report of scripts/bench_widths.py: the cifar8 layout (nz 8, zchannels 8, kernel 3, 4 5x5 + 8 ResNet layers) at reswidth
384 and 512.  One JSON line per (model, arm) with Mpixel/s, the per-category profile, bits/dim, round-trip status, and
the card name, power limit and median SM clock read in the same run; then a summary line.

    python scripts/bench_widths_wide.py --steps 2 --warmup 1 --rounds 3
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_widths                                                    # noqa: E402
from bitswap_b200.config import preset, with_                          # noqa: E402

bench_widths.MODELS = {
    "cifar8 W384": with_(preset("cifar8"), reswidth=384),
    "cifar8 W512": with_(preset("cifar8"), reswidth=512),
}

if __name__ == "__main__":
    bench_widths.main()
