"""The two arithmetics of the tensor-core convs, split (three bf16 MMAs per multiply-add) and bf16 (one), measured
alternately round by round in one process with the protocol and report of scripts/bench_widths.py.  Workloads: cifar8
(B = 1024, 4 free-running lanes), mnist2, and the cifar8 layout at reswidth 384.  One JSON line per (model, arm) with
Mpixel/s (median and range over the rounds), the per-category device time of one serial encode+decode, bits/dim,
round-trip status, and the card name, power limit and median SM clock read in the same run; then a summary line.
Random weights: bits/dim is a proxy, the rate cost of bf16 on trained models is not measured here.

    python scripts/bench_precision.py --steps 3 --warmup 1 --rounds 3
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench_widths                                                    # noqa: E402
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200.codec import Bins, PipelinedCodec                    # noqa: E402
from bitswap_b200.config import preset, with_                          # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402

MODELS = {
    "cifar8": preset("cifar8"),
    "mnist2": preset("mnist2"),
    "cifar8 W384": with_(preset("cifar8"), reswidth=384),
}
PRECISIONS = ("split", "bf16")


class Arm(bench_widths.Arm):
    def __init__(self, model, precision, B, lanes):
        self.model, self.precision, self.B = model, precision, B
        self.cfg = cfg = MODELS[model]
        sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
        zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
        self.bins = Bins(cfg, zend, zcen)
        self.codec = PipelinedCodec(cfg, sd, self.bins, B, lanes=lanes, free_running=True, tc_precision=precision)
        self.x = torch.from_numpy(synthetic.synthetic_images(cfg, B, seed=7)).cuda()
        self.ss = StreamSet(B, 1 << 13)
        w, head = synthetic.initial_words(2000, seed=100)
        self.ss.fill(w, head)
        self.init = self.ss.export_lists()
        self.exact = True

    @property
    def label(self):
        return f"{self.model} {self.precision}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--lanes", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--models", nargs="+", default=list(MODELS), choices=list(MODELS))
    args = ap.parse_args()
    name, limit = torch.cuda.get_device_name(), bench_widths.smi("power.limit")
    arms = [Arm(mdl, p, args.batch, args.lanes) for mdl in args.models for p in PRECISIONS]
    for a in arms:
        for _ in range(args.warmup):
            a.step()
    rates = {a.label: [] for a in arms}
    clocks = []
    for _ in range(args.rounds):                          # alternate the arms so that clock drift hits all of them
        for a in arms:
            ms = sum(a.step() for _ in range(args.steps))
            clocks.append(bench_widths.smi("clocks.sm"))
            rates[a.label].append(args.steps * args.batch * 1024 / (ms * 1e-3) / 1e6)
    clocks = [c for c in clocks if c is not None]
    sm_mhz = float(np.median(clocks)) if clocks else None
    res = {}
    for a in arms:
        r = dict(model=a.model, arm=a.precision, reswidth=a.cfg.reswidth, kernel_size=a.cfg.kernel_size, batch=args.batch,
                 lanes=args.lanes, Mpixel_s_median=round(float(np.median(rates[a.label])), 4),
                 Mpixel_s_range=[round(min(rates[a.label]), 4), round(max(rates[a.label]), 4)],
                 profile_ms_launches=a.profile(), bits_per_dim=round(a.bits_per_dim(), 4), roundtrip_exact=a.exact,
                 card=name, power_limit_w=limit, sm_clock_mhz_median=sm_mhz)
        res[a.label] = r
        print(json.dumps(r), flush=True)
    print(json.dumps({"summary": {m: {
        "bf16_vs_split_Mpixel_s": round(res[f"{m} bf16"]["Mpixel_s_median"] / res[f"{m} split"]["Mpixel_s_median"], 3),
        "roundtrip_exact": res[f"{m} bf16"]["roundtrip_exact"] and res[f"{m} split"]["roundtrip_exact"]}
        for m in args.models}, "card": name, "power_limit_w": limit, "sm_clock_mhz_median": sm_mhz}), flush=True)


if __name__ == "__main__":
    main()
