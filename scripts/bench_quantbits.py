"""Cost of finer latent bins: cifar8 at quantbits 10, 11 and 12 (1024, 2048 and 4096 bins per latent dimension), measured
alternately in one process with the protocol of bench.py (synthetic weights and images resident in HBM, warm-up steps,
then timed encode+decode steps of B images on free-running lanes, CUDA events around each step).

Prints one JSON line per quantbits and a summary line: encode+decode Mpixel/s (median and range over the rounds), the
per-category device time per 256-stream kernel launch (rows_z, pop_z, push_z, prior), net bits/dim of the synthetic
images, the device memory of the bins and of the coder scratch, and the card name and power limit read in the same run.
Random weights: bits/dim moves by sampling noise only, it is no statement about the rate of trained models.

    python scripts/bench_quantbits.py --steps 5 --warmup 2 --rounds 3
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


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        limit = float(out.strip().splitlines()[0])
    except Exception:
        limit = None
    return name, limit


class Arm:
    def __init__(self, q, B, lanes):
        self.q, self.B = q, B
        self.cfg = cfg = with_(preset("cifar8"), quantbits=q)
        sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
        zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
        self.bins = Bins(cfg, zend, zcen)
        self.codec = PipelinedCodec(cfg, sd, self.bins, B, lanes=lanes, use_tensor_cores=True, free_running=True)
        self.x = torch.from_numpy(synthetic.synthetic_images(cfg, B, seed=7)).cuda()
        self.ss = StreamSet(B, 1 << 14)
        w, head = synthetic.initial_words(2000, seed=100)
        self.ss.fill(w, head)
        per = self.codec.per
        pop_row = 136                                     # bsw_rows_scratch_bytes: 32 chunk bases + fix per (stream, row)
        self.mem = {"bins_bytes": 16 * cfg.nz * cfg.zdim * cfg.zsupport,
                    "scratch_bytes": self.codec.lanes * (per * max(cfg.zdim, cfg.xdim) * (pop_row + 16)),
                    "prior_tables_bytes": self.codec.lanes * cfg.zdim * (2 * cfg.zsupport + 1) * 4}

    def step(self):
        """one encode+decode of B images; returns ms"""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        self.codec.encode(self.ss, self.x)
        out = self.codec.decode(self.ss, self.B)
        self.codec.join()
        e1.record()
        e1.synchronize()
        assert torch.equal(out, self.x)
        return e0.elapsed_time(e1)

    def bits_per_dim(self):
        n0 = self.ss.export_lists()
        self.codec.encode(self.ss, self.x)
        self.codec.join()
        torch.cuda.synchronize()
        n1 = self.ss.export_lists()
        bpd = float(np.mean([32.0 * (len(b) - len(a)) / self.cfg.xdim for a, b in zip(n0, n1)]))
        self.codec.decode(self.ss, self.B)
        self.codec.join()
        torch.cuda.synchronize()
        return bpd

    def profile(self):
        self.codec.free_running = False
        self.codec.serial = True
        self.codec.profile(True)
        self.codec.encode(self.ss, self.x)
        self.codec.decode(self.ss, self.B)
        torch.cuda.synchronize()
        prof = self.codec.profile(False)
        self.codec.serial = False
        self.codec.free_running = True
        return {k: round(ms / n, 4) for k, (ms, n) in prof.items() if n and k in ("rows_z", "pop_z", "push_z", "prior")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--lanes", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--quantbits", type=int, nargs="+", default=[10, 11, 12])
    args = ap.parse_args()
    name, limit = card()
    arms = [Arm(q, args.batch, args.lanes) for q in args.quantbits]
    for a in arms:
        for _ in range(args.warmup):
            a.step()
    rates = {a.q: [] for a in arms}
    for _ in range(args.rounds):                          # alternate the arms so that clock drift hits all of them
        for a in arms:
            ms = sum(a.step() for _ in range(args.steps))
            rates[a.q].append(args.steps * args.batch * 1024 / (ms * 1e-3) / 1e6)     # bench.py's unit: B*1024 pixels per step
    res = []
    for a in arms:
        r = dict(quantbits=a.q, support=a.cfg.zsupport, batch=args.batch, lanes=args.lanes,
                 Mpixel_s_median=round(float(np.median(rates[a.q])), 4),
                 Mpixel_s_range=[round(min(rates[a.q]), 4), round(max(rates[a.q]), 4)],
                 ms_per_256_stream_launch=a.profile(), bits_per_dim=round(a.bits_per_dim(), 4), **a.mem,
                 card=name, power_limit_w=limit)
        res.append(r)
        print(json.dumps(r), flush=True)
    base = res[0]
    print(json.dumps({"summary": {f"q{r['quantbits']}": {
        "Mpixel_s_vs_first": round(r["Mpixel_s_median"] / base["Mpixel_s_median"], 3),
        "rows_z_vs_first": round(r["ms_per_256_stream_launch"].get("rows_z", 0) / max(base["ms_per_256_stream_launch"].get("rows_z", 1e-9), 1e-9), 3)}
        for r in res}, "card": name, "power_limit_w": limit}), flush=True)


if __name__ == "__main__":
    main()
