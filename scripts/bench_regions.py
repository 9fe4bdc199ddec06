"""Decoding windows of images: `python scripts/bench_regions.py [--rounds 3 --warmup 1 --big-rounds 2]`.

decompress_regions pops a chain only down to the earliest block a window needs and skips chains the windows miss
(plan_regions), so what a window costs depends on the chain layout.  Two workloads, every setting alternated round by
round in one process after `--warmup` rounds of the crop settings:
  photo  one 2048 x 1536 synthetic_photo (3072 blocks) at chain_blocks None and 32: the full decode against 1, 16 and 64
         seeded random 256 x 256 windows per call (`--big-rounds` rounds, fresh windows each round);
  crop   the BASELINE config-5 images (synthetic_crop_images(100, seed=0)) at chain_blocks None and 32: one seeded random
         224 x 224 crop per image against the full decode (`--rounds` rounds).
imagenetcrop4 on the tensor cores, edges="code", one PipelinedCodec per (workload, chain_blocks) sized to its chain count
with up to `--lanes` free-running lanes, as bench_chains.py runs it; the containers are written once per setting, by the
same codec.  Per setting: seconds per call (host clock around the call, which ends in a device transfer), the blocks
decoded and the blocks the windows cover by plan_regions next to the blocks and calls the codec saw, the serial depth (the
deepest chain's pops), delivered Mpixel/s (pixels returned / seconds) and whether every window equals the crop of the full
decode.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from scripts.bench_chains import synthetic_photo              # noqa: E402
from scripts.bench_crop import synthetic_crop_images          # noqa: E402
from scripts.bench_edges import card                          # noqa: E402


class Counting:
    """Codec proxy counting decode calls and the blocks they pop."""

    def __init__(self, codec):
        self.codec = codec
        self.reset()

    def __getattr__(self, name):
        return getattr(self.codec, name)

    def reset(self):
        self.calls, self.blocks = 0, 0

    def decode(self, ss, count, **kw):
        self.calls += 1
        self.blocks += count
        return self.codec.decode(ss, count, **kw)


def windows(rs, shapes, per_image, side):
    """`per_image` random side x side windows (i, y, x, h, w) on each image of the given (h, w)."""
    return [(i, int(rs.randint(0, h - side + 1)), int(rs.randint(0, w - side + 1)), side, side)
            for i, (h, w) in enumerate(shapes) for _ in range(per_image)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--big-rounds", type=int, default=2)
    ap.add_argument("--lanes", type=int, default=4)
    args = ap.parse_args()
    from bitswap_b200 import synthetic
    from bitswap_b200.config import preset
    from bitswap_b200.codec import PipelinedCodec, Bins
    from bitswap_b200.container import (chain_sizes, compress_images, decompress_images, decompress_regions,
                                        extract_edge_blocks, plan_regions)

    assert torch.cuda.is_available(), "bench_regions.py needs a GPU"
    torch.cuda.set_device(0)
    cfg = preset("imagenetcrop4")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))

    # workload -> (images, chain_blocks settings, modes: name -> windows per image (None: full decode), window side, rounds)
    workloads = {"crop": (synthetic_crop_images(args.images, seed=0), [None, 32], {"full": None, "1 crop/image": 1}, 224,
                          args.rounds),
                 "photo": ([synthetic_photo(1536, 2048, seed=0)], [None, 32],
                           {"full": None, "1 window": 1, "16 windows": 16, "64 windows": 64}, 256, args.big_rounds)}
    setups, results = {}, {}
    for wl, (images, settings, modes, _, _) in workloads.items():
        nblocks = [extract_edge_blocks(im)[0].shape[0] for im in images]
        for L in settings:
            chains = len([s for n in nblocks for s in chain_sizes(n, L)])
            codec = Counting(PipelinedCodec(cfg, sd, bins, chains, lanes=min(args.lanes, chains), use_tensor_cores=True,
                                            free_running=True))
            t0 = time.perf_counter()
            conts = compress_images(codec, images, edges="code", chain_blocks=L)
            print(f"{wl} chain_blocks={L}: {chains} chains written in {time.perf_counter() - t0:.2f} s", file=sys.stderr,
                  flush=True)
            setups[wl, L] = dict(codec=codec, conts=conts, chains=chains, full=None)
            for mode in modes:
                results[wl, L, mode] = dict(s=[], decoded=[], needed=[], depth=[], calls=[], popped=[], px=[], exact=True)

    def one_call(wl, L, mode, rnd):
        images, _, modes, side, _ = workloads[wl]
        st = setups[wl, L]
        codec, conts = st["codec"], st["conts"]
        per = modes[mode]
        regions = (None if per is None else
                   windows(np.random.RandomState(1000 * rnd + per), [im.shape[:2] for im in images], per, side))
        codec.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = decompress_images(codec, conts) if regions is None else decompress_regions(codec, conts, regions)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if regions is None:
            regions = [(i, 0, 0) + im.shape[:2] for i, im in enumerate(images)]
            exact = all(np.array_equal(a, b) for a, b in zip(images, out))
            st["full"] = out
        else:
            exact = all(np.array_equal(o, st["full"][i][y:y + h, x:x + w]) for o, (i, y, x, h, w) in zip(out, regions))
        plans = plan_regions(conts, regions)
        return dict(s=dt, decoded=sum(int(p.depth.sum()) for p in plans), needed=sum(int(p.needed.sum()) for p in plans),
                    depth=max(int(p.depth.max()) for p in plans), calls=codec.calls, popped=codec.blocks,
                    px=sum(h * w for _, _, _, h, w in regions)), exact

    for _ in range(args.warmup):
        for L in workloads["crop"][1]:
            for mode in workloads["crop"][2]:
                one_call("crop", L, mode, 0)
    for wl, (images, settings, modes, _, rounds) in workloads.items():
        for rnd in range(rounds):
            for L in settings:
                for mode in modes:                            # "full" first: the windows are checked against it
                    got, exact = one_call(wl, L, mode, rnd + 1)
                    r = results[wl, L, mode]
                    for k, v in got.items():
                        r[k].append(v)
                    r["exact"] &= exact
                    print(f"{wl} chain_blocks={L} {mode}: {got['s']:.3f} s, {got['decoded']} blocks decoded "
                          f"({got['needed']} needed), depth {got['depth']}, exact {exact}", file=sys.stderr, flush=True)

    out = {"card": card(), "workload": {
        "crop": f"{args.images} synthetic_crop_images(seed=0), edges='code', imagenetcrop4, tensor cores, up to {args.lanes} "
                f"free-running lanes; one random 224 x 224 crop per image; {args.rounds} alternated rounds",
        "photo": f"one 2048 x 1536 synthetic_photo(seed=0), same model and lanes; 1, 16 and 64 random 256 x 256 windows per "
                 f"call; {args.big_rounds} alternated rounds, fresh windows each round"}}
    for (wl, L, mode), r in results.items():
        s = np.array(r["s"])
        out[f"{wl} chain_blocks={L} {mode}"] = {
            "chains": setups[wl, L]["chains"], "s_per_call_median": float(np.median(s)), "s_per_call_range": [float(s.min()),
                                                                                                         float(s.max())],
            "blocks_decoded_mean": float(np.mean(r["decoded"])), "blocks_needed_mean": float(np.mean(r["needed"])),
            "codec_blocks_mean": float(np.mean(r["popped"])), "codec_calls_mean": float(np.mean(r["calls"])),
            "plan_is_what_ran": r["decoded"] == r["popped"],
            "serial_depth_mean": float(np.mean(r["depth"])), "serial_depth_max": int(max(r["depth"])),
            "Mpixel_s": float(np.sum(r["px"]) / np.sum(s) / 1e6), "exact": bool(r["exact"])}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
