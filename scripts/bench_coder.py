"""The reference and direct coders (BitSwapCodec coder="reference" / "direct"), measured alternately round by round in one
process with the protocol and report of scripts/bench_widths.py.  Workloads: cifar8 with split and with bf16 nets at
quantbits 10 and 12 (B = 1024, 4 free-running lanes), and mnist2.  One JSON line per (workload, coder) with Mpixel/s
(median and range over the rounds), the per-category device time of one serial encode+decode (rows_* = the parallel
kernels, pop_*/push_* = the serial ones), bits/dim, round-trip status, and the card name, power limit and median SM clock
read in the same run; then a summary line with the direct/reference ratios.  Random weights: bits/dim is a proxy.

    python scripts/bench_coder.py --steps 3 --warmup 1 --rounds 3
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

# workload -> (config, tensor-core arithmetic)
WORKLOADS = {
    "cifar8 split q10": (preset("cifar8"), "split"),
    "cifar8 split q12": (with_(preset("cifar8"), quantbits=12), "split"),
    "cifar8 bf16 q10": (preset("cifar8"), "bf16"),
    "cifar8 bf16 q12": (with_(preset("cifar8"), quantbits=12), "bf16"),
    "mnist2": (preset("mnist2"), "split"),
}
CODERS = ("reference", "direct")


class Arm(bench_widths.Arm):
    def __init__(self, workload, coder, B, lanes, bins):
        self.model, self.coder, self.B = workload, coder, B
        self.cfg = cfg = WORKLOADS[workload][0]
        sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
        self.bins = bins
        self.codec = PipelinedCodec(cfg, sd, bins, B, lanes=lanes, free_running=True, tc_precision=WORKLOADS[workload][1],
                                    coder=coder)
        self.x = torch.from_numpy(synthetic.synthetic_images(cfg, B, seed=7)).cuda()
        self.ss = StreamSet(B, 1 << 13)
        w, head = synthetic.initial_words(2000, seed=100)
        self.ss.fill(w, head)
        self.init = self.ss.export_lists()
        self.exact = True

    @property
    def label(self):
        return f"{self.model} {self.coder}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--lanes", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    args = ap.parse_args()
    name, limit = torch.cuda.get_device_name(), bench_widths.smi("power.limit")
    bins = {}                                              # one device copy of the bins per config (1.07 GB at cifar8 q12)
    arms = []
    for wl in args.workloads:
        cfg = WORKLOADS[wl][0]
        if cfg not in bins:
            zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
            bins[cfg] = Bins(cfg, zend, zcen)
        arms += [Arm(wl, c, args.batch, args.lanes, bins[cfg]) for c in CODERS]
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
        r = dict(workload=a.model, coder=a.coder, quantbits=a.cfg.quantbits, tc_precision=WORKLOADS[a.model][1],
                 batch=args.batch, lanes=args.lanes, Mpixel_s_median=round(float(np.median(rates[a.label])), 4),
                 Mpixel_s_range=[round(min(rates[a.label]), 4), round(max(rates[a.label]), 4)],
                 profile_ms_launches=a.profile(), bits_per_dim=round(a.bits_per_dim(), 5), roundtrip_exact=a.exact,
                 card=name, power_limit_w=limit, sm_clock_mhz_median=sm_mhz)
        res[a.label] = r
        print(json.dumps(r), flush=True)
    print(json.dumps({"summary": {w: {
        "direct_vs_reference_Mpixel_s": round(res[f"{w} direct"]["Mpixel_s_median"] / res[f"{w} reference"]["Mpixel_s_median"], 3),
        "bits_per_dim_direct_minus_reference": round(res[f"{w} direct"]["bits_per_dim"] - res[f"{w} reference"]["bits_per_dim"], 5),
        "roundtrip_exact": res[f"{w} direct"]["roundtrip_exact"] and res[f"{w} reference"]["roundtrip_exact"]}
        for w in args.workloads}, "card": name, "power_limit_w": limit, "sm_clock_mhz_median": sm_mhz}), flush=True)


if __name__ == "__main__":
    main()
