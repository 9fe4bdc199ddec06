"""Images coded as several chains: `python scripts/bench_chains.py [--rounds 3 --warmup 1 --big-rounds 2]`.

A chain is serial, so the time to code an image grows with its block count.  compress_images(chain_blocks=L) splits an
image of n blocks into ceil(n / L) chains that run side by side, at the price of each chain's borrowed initial words.
Two workloads, each setting alternated round by round in one process after `--warmup` rounds of each:
  crop   the BASELINE config-5 images of scripts/bench_edges.py (synthetic_crop_images(100, seed=0), imagenetcrop4 on the
         tensor cores, 4 free-running lanes, edges="code") at chain_blocks None, 64, 32 and 16;
  photo  one 2048 x 1536 image of the same generator formula (3072 blocks) at chain_blocks None and 32 (`--big-rounds`
         rounds; its warm-up is the crop workload's, which runs the same kernels).
Every setting gets a PipelinedCodec sized to its stream count (max_batch = chains), as bench_edges.py sizes its codec to
the image count.  A round is compress + decompress of every image.  Per setting: chains and serial depth (the longest
chain's blocks); encode and decode seconds and their host time outside device work (the call's wall time outside the span
from its first coder call to the end of its last coder kernel: staging, stream-set set-up, export, container packing and
parsing); Mpixel/s; bits/dim over all container words; the initial-bit overhead sum(start - min words) over the chains
and its share of the container words; whether the round trip was exact.  The card's name and power limit are read in
the same run.
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

from scripts.bench_crop import synthetic_crop_images       # noqa: E402
from scripts.bench_edges import card                         # noqa: E402


def synthetic_photo(h, w, seed=0):
    """One HWC uint8 image of synthetic_crop_images' formula at a given size."""
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    img = np.stack([128 + 60 * np.sin(xx * rs.uniform(0.01, 0.1) + yy * rs.uniform(0.01, 0.1) + rs.uniform(0, 6)) +
                    rs.normal(0, 6, (h, w)) for _ in range(3)], axis=-1)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


class DeviceSpan:
    """Codec proxy: CUDA events from the first coder call of a compress/decompress call to the end of its last coder
    kernel on every lane."""

    def __init__(self, codec):
        self.codec = codec
        self.lanes = getattr(codec, "streams", None)
        self.reset()

    def __getattr__(self, name):
        return getattr(self.codec, name)

    def reset(self):
        self.start, self.ends = None, {}

    def _span(self, fn, *a, **k):
        if self.start is None:
            torch.cuda.synchronize()                        # the staging enqueued before the first call is host-side time
            self.start = torch.cuda.Event(enable_timing=True)
            self.start.record()
        out = fn(*a, **k)
        for i, st in enumerate(self.lanes or [torch.cuda.current_stream()]):
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(st)
            self.ends[i] = ev
        return out

    def encode(self, *a, **k):
        return self._span(self.codec.encode, *a, **k)

    def decode(self, *a, **k):
        return self._span(self.codec.decode, *a, **k)

    def seconds(self):
        return max(self.start.elapsed_time(e) for e in self.ends.values()) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--big-rounds", type=int, default=2)
    ap.add_argument("--lanes", type=int, default=4)
    args = ap.parse_args()
    from bitswap_b200 import container, synthetic
    from bitswap_b200.config import preset
    from bitswap_b200.codec import PipelinedCodec, Bins
    from bitswap_b200.container import chain_sizes, compress_images, decompress_images, extract_edge_blocks
    from bitswap_b200.streams import StreamSet

    assert torch.cuda.is_available(), "bench_chains.py needs a GPU"
    torch.cuda.set_device(0)
    cfg = preset("imagenetcrop4")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
    excess = 10000                                          # compress_images' default initial state: excess - 1 words + head

    made = []

    class Recorded(StreamSet):                              # keeps the encoder's stream set for its min_words()
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)
    container.StreamSet = Recorded

    workloads = {"crop": (synthetic_crop_images(args.images, seed=0), [None, 64, 32, 16], args.rounds),
                 "photo": ([synthetic_photo(1536, 2048, seed=0)], [None, 32], args.big_rounds)}
    setups = {}
    for wl, (images, settings, _) in workloads.items():
        nblocks = [extract_edge_blocks(im)[0].shape[0] for im in images]
        for L in settings:
            sizes = [s for n in nblocks for s in chain_sizes(n, L)]
            codec = PipelinedCodec(cfg, sd, bins, len(sizes), lanes=min(args.lanes, len(sizes)), use_tensor_cores=True,
                                   free_running=True)
            setups[wl, L] = dict(codec=DeviceSpan(codec), chains=len(sizes), depth=max(sizes), enc=[], dec=[], enc_host=[],
                                 dec_host=[], exact=True)

    def one_round(wl, L):
        images = workloads[wl][0]
        s = setups[wl, L]
        codec = s["codec"]
        made.clear()
        codec.reset()
        t0 = time.perf_counter()
        conts = compress_images(codec, images, edges="code", chain_blocks=L)
        torch.cuda.synchronize()
        te = time.perf_counter() - t0
        enc_dev = codec.seconds()
        ss = made[-1]
        borrowed = int(np.sum(excess - 1 - ss.min_words()))
        codec.reset()
        t0 = time.perf_counter()
        back = decompress_images(codec, conts)
        torch.cuda.synchronize()
        td = time.perf_counter() - t0
        dec_dev = codec.seconds()
        return conts, back, te, td, te - enc_dev, td - dec_dev, borrowed

    for _ in range(args.warmup):
        for L in workloads["crop"][1]:
            one_round("crop", L)
    for wl, (images, settings, rounds) in workloads.items():
        for _ in range(rounds):
            for L in settings:
                conts, back, te, td, he, hd, borrowed = one_round(wl, L)
                print(f"{wl} chain_blocks={L}: encode {te:.2f} s, decode {td:.2f} s (host {he:.2f} + {hd:.2f} s)",
                      file=sys.stderr, flush=True)
                s = setups[wl, L]
                s["enc"].append(te)
                s["dec"].append(td)
                s["enc_host"].append(he)
                s["dec_host"].append(hd)
                s["exact"] &= all(np.array_equal(a, b) for a, b in zip(images, back))
                s["words"] = int(sum(len(c) for c in conts))
                s["borrowed"] = borrowed

    out = {"card": card(), "workload": {
        "crop": f"{args.images} synthetic_crop_images(seed=0), edges='code', imagenetcrop4, tensor cores, up to {args.lanes} "
                f"free-running lanes, {args.rounds} alternated rounds per setting",
        "photo": f"one 2048 x 1536 synthetic_photo(seed=0), edges='code', same model and lanes, {args.big_rounds} alternated "
                 f"rounds per setting"}}
    for (wl, L), s in setups.items():
        images = workloads[wl][0]
        dims = sum(im.size for im in images)
        px = dims / 3
        steps = np.array(s["enc"]) + np.array(s["dec"])
        out[f"{wl} chain_blocks={L}"] = {
            "chains": s["chains"], "serial_depth_blocks": s["depth"],
            "encode_s_median": float(np.median(s["enc"])), "decode_s_median": float(np.median(s["dec"])),
            "encode_host_s_median": float(np.median(s["enc_host"])), "decode_host_s_median": float(np.median(s["dec_host"])),
            "Mpixel_s_median": px / float(np.median(steps)) / 1e6,
            "Mpixel_s_range": [px / float(steps.max()) / 1e6, px / float(steps.min()) / 1e6],
            "bits_per_dim": 32.0 * s["words"] / dims, "initial_words": s["borrowed"],
            "initial_share": s["borrowed"] / s["words"], "roundtrip_ok": bool(s["exact"])}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
