"""Models of padded width 128 and 192, and a kernel-size-5 model, on the float32 SIMT convs and on the tensor cores (the
k_conv_wg tiles of padded widths 128 / 192 / 256), measured alternately in one process with the protocol of bench.py
(synthetic weights, bins and images resident in HBM, warm-up steps, then timed encode+decode steps of B images on
free-running lanes, CUDA events around each step).  Models: the cifar8 layout (nz 8, zchannels 8, 4 5x5 + 8 ResNet
layers) at reswidth 128 and 192, and at its own reswidth 252 with kernel_size 5.

Prints one JSON line per (model, arm) and a summary line: encode+decode Mpixel/s (median and range over the rounds), the
per-category device time of one serial encode+decode of the B images (ms summed over its launches), net bits/dim of the
synthetic images, whether every step restored its pixels and the streams their initial states, and the card name, power
limit and median SM clock read in the same run (nvidia-smi --query-gpu, read-only).  Random weights: bits/dim moves by
sampling noise only, it is no statement about the rate of trained models.  The two arms code different bitstreams (the
tensor-core nets are not bit-identical to the SIMT nets), so their bits/dim differ by noise too.

    python scripts/bench_widths.py --steps 3 --warmup 1 --rounds 3
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200.codec import Bins, PipelinedCodec                    # noqa: E402
from bitswap_b200.config import preset, with_                          # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402


# name -> CodecConfig: the cifar8 layout at the widths of the padded-width-128 / -192 tiles, and with 5x5 kernels
MODELS = {
    "cifar8 W128": with_(preset("cifar8"), reswidth=128),
    "cifar8 W192": with_(preset("cifar8"), reswidth=192),
    "cifar8 k5": with_(preset("cifar8"), kernel_size=5),
}


def smi(field):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


class Arm:
    def __init__(self, model, tc, B, lanes):
        self.model, self.tc, self.B = model, tc, B
        self.cfg = cfg = MODELS[model]
        sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
        zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
        self.bins = Bins(cfg, zend, zcen)
        self.codec = PipelinedCodec(cfg, sd, self.bins, B, lanes=lanes, use_tensor_cores=tc, free_running=True)
        self.x = torch.from_numpy(synthetic.synthetic_images(cfg, B, seed=7)).cuda()
        self.ss = StreamSet(B, 1 << 13)
        w, head = synthetic.initial_words(2000, seed=100)
        self.ss.fill(w, head)
        self.init = self.ss.export_lists()
        self.exact = True

    @property
    def label(self):
        return f"{self.model} {'tensor cores' if self.tc else 'SIMT'}"

    def step(self):
        """one encode+decode of B images; returns ms"""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        self.codec.encode(self.ss, self.x)
        out = self.codec.decode(self.ss, self.B)
        self.codec.join()
        e1.record()
        e1.synchronize()
        self.exact &= bool(torch.equal(out, self.x))
        return e0.elapsed_time(e1)

    def bits_per_dim(self):
        self.codec.encode(self.ss, self.x)
        self.codec.join()
        torch.cuda.synchronize()
        n1 = self.ss.export_lists()
        bpd = float(np.mean([32.0 * (len(b) - len(a)) / self.cfg.xdim for a, b in zip(self.init, n1)]))
        out = self.codec.decode(self.ss, self.B)
        self.codec.join()
        torch.cuda.synchronize()
        self.exact &= bool(torch.equal(out, self.x)) and self.ss.export_lists() == self.init
        return bpd

    def profile(self):
        self.codec.free_running = False
        self.codec.serial = True
        self.codec.profile(True)
        self.codec.encode(self.ss, self.x)
        out = self.codec.decode(self.ss, self.B)
        torch.cuda.synchronize()
        prof = self.codec.profile(False)
        self.codec.serial = False
        self.codec.free_running = True
        self.exact &= bool(torch.equal(out, self.x))
        return {k: [round(ms, 3), n] for k, (ms, n) in prof.items() if n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--lanes", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--models", nargs="+", default=list(MODELS), choices=list(MODELS))
    args = ap.parse_args()
    name, limit = torch.cuda.get_device_name(), smi("power.limit")
    arms = [Arm(mdl, tc, args.batch, args.lanes) for mdl in args.models for tc in (False, True)]
    for a in arms:
        for _ in range(args.warmup):
            a.step()
    rates = {a.label: [] for a in arms}
    clocks = []
    for _ in range(args.rounds):                          # alternate the arms so that clock drift hits all of them
        for a in arms:
            ms = sum(a.step() for _ in range(args.steps))
            clocks.append(smi("clocks.sm"))              # right after the timed steps, while the card is still warm
            rates[a.label].append(args.steps * args.batch * 1024 / (ms * 1e-3) / 1e6)     # bench.py's unit: B*1024 pixels per step
    clocks = [c for c in clocks if c is not None]
    sm_mhz = float(np.median(clocks)) if clocks else None
    res = {}
    for a in arms:
        r = dict(model=a.model, arm="tc" if a.tc else "simt", reswidth=a.cfg.reswidth,
                 kernel_size=a.cfg.kernel_size, batch=args.batch, lanes=args.lanes,
                 Mpixel_s_median=round(float(np.median(rates[a.label])), 4),
                 Mpixel_s_range=[round(min(rates[a.label]), 4), round(max(rates[a.label]), 4)],
                 profile_ms_launches=a.profile(), bits_per_dim=round(a.bits_per_dim(), 4), roundtrip_exact=a.exact,
                 card=name, power_limit_w=limit, sm_clock_mhz_median=sm_mhz)
        res[a.label] = r
        print(json.dumps(r), flush=True)
    print(json.dumps({"summary": {m: {
        "tc_vs_simt_Mpixel_s": round(res[f"{m} tensor cores"]["Mpixel_s_median"] / res[f"{m} SIMT"]["Mpixel_s_median"], 3),
        "roundtrip_exact": res[f"{m} tensor cores"]["roundtrip_exact"] and res[f"{m} SIMT"]["roundtrip_exact"]}
        for m in args.models}, "card": name, "power_limit_w": limit, "sm_clock_mhz_median": sm_mhz}), flush=True)


if __name__ == "__main__":
    main()
