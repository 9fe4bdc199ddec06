"""Small images as one archive: `python scripts/bench_archive.py [--images 4096 --rounds 3 --warmup 1 --draws 16]`.

compress_archive lays the blocks of many images end to end and cuts that sequence into chains of about chain_blocks blocks,
so the initial words each chain borrows are paid once per chain instead of once per image.  Two workloads:
  cifar  4096 synthetic 32 x 32 RGB images (synthetic_images(kind="smooth")) on cifar8;
  mnist  4096 synthetic 28 x 28 single-channel images (the same generator at 32 x 32, cropped) on mnist2;
both on the tensor cores with up to 4 free-running lanes.  Settings: per-image containers (compress_images(edges="code"),
one chain per image: the default chain_blocks=None) and archives at chain_blocks 16, 64 and 256.  Every setting gets a
PipelinedCodec sized to its chain count (max_batch = chains).  After `--warmup` rounds of each setting, the settings
alternate round by round in one process; a round is compress + decompress of every image.  Per setting: chains; total
words and bits/dim over everything stored (trailers and tables included); the initial words, sum(start - min words) over
the chains, and their share of the stored words; encode and decode seconds and their host time outside device work (as in
bench_chains.py); Mpixel/s; the median seconds and blocks popped to decode one random image, over `--draws` draws (a
single-image decode call for containers, a one-region decompress_archive for archives); whether every round trip and every
single-image decode was exact.  The card's name and power limit are read in the same run.
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

from scripts.bench_chains import DeviceSpan                # noqa: E402
from scripts.bench_edges import card                         # noqa: E402


class Popped(DeviceSpan):
    """DeviceSpan that also counts the blocks decode calls pop."""

    def reset(self):
        super().reset()
        self.blocks = 0

    def decode(self, ss, count, **k):
        self.blocks += count
        return super().decode(ss, count, **k)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--draws", type=int, default=16)
    ap.add_argument("--lanes", type=int, default=4)
    args = ap.parse_args()
    from bitswap_b200 import container, synthetic
    from bitswap_b200.config import preset
    from bitswap_b200.codec import PipelinedCodec, Bins
    from bitswap_b200.container import (chain_sizes, compress_archive, compress_images, decompress_archive,
                                        decompress_images)
    from bitswap_b200.streams import StreamSet

    assert torch.cuda.is_available(), "bench_archive.py needs a GPU"
    torch.cuda.set_device(0)
    excess = 10000                                          # the default initial state: excess - 1 words + head

    made = []

    class Recorded(StreamSet):                              # keeps the encoder's stream set for its min_words()
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)
    container.StreamSet = Recorded

    settings = [None, 16, 64, 256]                          # None: per-image containers
    models = {"cifar": ("cifar8", 32), "mnist": ("mnist2", 28)}
    workloads, setups = {}, {}

    def set_up(wl):
        """The workload's images and one codec per setting (one workload's codecs are alive at a time)."""
        name, side = models[wl]
        cfg = preset(name)
        sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
        bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
        imgs = synthetic.synthetic_images(cfg, args.images, seed=7, kind="smooth")[:, :, :side, :side]
        workloads[wl] = [np.ascontiguousarray(im.transpose(1, 2, 0)) for im in imgs]
        for L in settings:
            chains = args.images if L is None else len(chain_sizes(args.images, L))
            codec = PipelinedCodec(cfg, sd, bins, chains, lanes=min(args.lanes, chains), use_tensor_cores=True,
                                   free_running=True)
            setups[wl, L] = dict(codec=Popped(codec), chains=chains, enc=[], dec=[], enc_host=[], dec_host=[],
                                 one_s=[], one_blocks=[], exact=True)

    def one_round(wl, L):
        images = workloads[wl]
        s = setups[wl, L]
        codec = s["codec"]
        made.clear()
        codec.reset()
        t0 = time.perf_counter()
        stored = (compress_images(codec, images, edges="code") if L is None else compress_archive(codec, images, chain_blocks=L))
        torch.cuda.synchronize()
        te = time.perf_counter() - t0
        enc_dev = codec.seconds()
        borrowed = int(np.sum(excess - 1 - made[-1].min_words()))
        codec.reset()
        t0 = time.perf_counter()
        back = decompress_images(codec, stored, channels=images[0].shape[2]) if L is None else decompress_archive(codec, stored)
        torch.cuda.synchronize()
        td = time.perf_counter() - t0
        return stored, back, te, td, te - enc_dev, td - codec.seconds(), borrowed

    def one_image(wl, L, i):
        images = workloads[wl]
        codec = setups[wl, L]["codec"]
        codec.reset()
        t0 = time.perf_counter()
        if L is None:
            (got,) = decompress_images(codec, [setups[wl, L]["stored"][i]], channels=images[0].shape[2])
        else:
            (got,) = decompress_archive(codec, setups[wl, L]["stored"], [(i, 0, 0) + images[i].shape[:2]])
        torch.cuda.synchronize()
        return time.perf_counter() - t0, codec.blocks, np.array_equal(got, images[i])

    for wl in models:
        set_up(wl)
        images = workloads[wl]
        for _ in range(args.warmup):
            for L in settings:
                one_round(wl, L)
        for _ in range(args.rounds):
            for L in settings:
                stored, back, te, td, he, hd, borrowed = one_round(wl, L)
                print(f"{wl} chain_blocks={L}: encode {te:.2f} s, decode {td:.2f} s (host {he:.2f} + {hd:.2f} s)",
                      file=sys.stderr, flush=True)
                s = setups[wl, L]
                s["enc"].append(te)
                s["dec"].append(td)
                s["enc_host"].append(he)
                s["dec_host"].append(hd)
                s["exact"] &= all(np.array_equal(a, b) for a, b in zip(images, back))
                s["stored"] = stored
                s["words"] = int(sum(len(c) for c in stored)) if L is None else int(len(stored))
                s["borrowed"] = borrowed
        for i in np.random.RandomState(11).randint(len(images), size=args.draws):
            for L in settings:
                sec, blocks, ok = one_image(wl, L, int(i))
                s = setups[wl, L]
                s["one_s"].append(sec)
                s["one_blocks"].append(blocks)
                s["exact"] &= ok
        for L in settings:                                  # free this workload's codecs and stored data
            del setups[wl, L]["codec"], setups[wl, L]["stored"]
        torch.cuda.empty_cache()

    out = {"card": card(), "workload": {
        wl: f"{args.images} synthetic_images(kind='smooth', seed=7) at {workloads[wl][0].shape}, {name}, tensor cores, up to "
            f"{args.lanes} free-running lanes, {args.rounds} alternated rounds per setting, {args.draws} single-image draws"
        for wl, (name, _) in models.items()}}
    for (wl, L), s in setups.items():
        images = workloads[wl]
        dims = sum(im.size for im in images)
        px = dims / images[0].shape[2]
        steps = np.array(s["enc"]) + np.array(s["dec"])
        out[f"{wl} " + ("per-image containers" if L is None else f"archive chain_blocks={L}")] = {
            "chains": s["chains"], "words": s["words"], "bits_per_dim": 32.0 * s["words"] / dims,
            "initial_words": s["borrowed"], "initial_share": s["borrowed"] / s["words"],
            "encode_s_median": float(np.median(s["enc"])), "decode_s_median": float(np.median(s["dec"])),
            "encode_host_s_median": float(np.median(s["enc_host"])), "decode_host_s_median": float(np.median(s["dec_host"])),
            "Mpixel_s_median": px / float(np.median(steps)) / 1e6,
            "Mpixel_s_range": [px / float(steps.max()) / 1e6, px / float(steps.min()) / 1e6],
            "one_image_s_median": float(np.median(s["one_s"])), "one_image_blocks_median": float(np.median(s["one_blocks"])),
            "roundtrip_ok": bool(s["exact"])}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
