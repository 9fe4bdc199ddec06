"""Cropped vs edge-coded variable-size images: `python scripts/bench_edges.py [--images 100 --rounds 3 --warmup 1]`.

The BASELINE config-5 workload of scripts/bench_crop.py (the same synthetic_crop_images(100, seed=0), the imagenetcrop4
model on tensor cores, a free-running 4-lane PipelinedCodec on one GPU) coded two ways, alternated in one process:
  crop  compress_images(edges="crop"): every image cropped down to multiples of 32 (the reference's demo behaviour);
  code  compress_images(edges="code"): the whole image, partial edge blocks coding only their valid pixels.
A round is compress + decompress of every image; the modes alternate round by round after `--warmup` rounds of each.
Per mode it prints Mpixel/s over the pixels that mode returns, bits/dim over those dims (counted as bench_crop.py does:
32 bits per container word minus the 3-word tail), whether the round trip returned those pixels exactly, and the
host compressors on the full images.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from scripts.bench_crop import host_compressors, synthetic_crop_images     # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--lanes", type=int, default=4)
    args = ap.parse_args()
    from bitswap_b200 import synthetic
    from bitswap_b200.config import preset
    from bitswap_b200.codec import PipelinedCodec, Bins
    from bitswap_b200.container import compress_images, decompress_images

    assert torch.cuda.is_available(), "bench_edges.py needs a GPU"
    torch.cuda.set_device(0)
    cfg = preset("imagenetcrop4")
    images = synthetic_crop_images(args.images, seed=0)
    want = {"crop": [im[:im.shape[0] - im.shape[0] % 32, :im.shape[1] - im.shape[1] % 32] for im in images], "code": images}
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    codec = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), len(images), lanes=min(args.lanes, len(images)),
                           use_tensor_cores=True, free_running=True)

    def one_round(mode):
        t0 = time.perf_counter()
        conts = compress_images(codec, images, edges=mode)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        back = decompress_images(codec, conts)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        return conts, back, t1 - t0, t2 - t1

    for _ in range(args.warmup):
        for mode in ("crop", "code"):
            one_round(mode)
    res = {m: {"enc_s": [], "dec_s": [], "roundtrip_ok": True} for m in ("crop", "code")}
    for _ in range(args.rounds):
        for mode in ("crop", "code"):
            conts, back, te, td = one_round(mode)
            print(f"{mode}: encode {te:.2f} s, decode {td:.2f} s", file=sys.stderr, flush=True)
            r = res[mode]
            r["enc_s"].append(te)
            r["dec_s"].append(td)
            r["roundtrip_ok"] &= all(np.array_equal(a, b) for a, b in zip(want[mode], back))
            r["words"] = sum(len(c) - 3 for c in conts)
            r["blocks"] = int(sum(int(c[-3]) for c in conts))
            r["serial_depth_blocks"] = int(max(int(c[-3]) for c in conts))
    out = {"card": card(), "workload": f"{len(images)} synthetic_crop_images(seed=0), imagenetcrop4, tensor cores, "
                                        f"{codec.lanes} free-running lanes, {args.rounds} alternated rounds per mode"}
    for mode, r in res.items():
        dims = sum(im.size for im in want[mode])
        px = dims / 3
        steps = np.array(r["enc_s"]) + np.array(r["dec_s"])
        out[mode] = {"pixels": int(px), "blocks": r["blocks"], "serial_depth_blocks": r["serial_depth_blocks"],
                     "Mpixel_s_median": px / float(np.median(steps)) / 1e6,
                     "Mpixel_s_range": [px / float(steps.max()) / 1e6, px / float(steps.min()) / 1e6],
                     "encode_s_median": float(np.median(r["enc_s"])), "decode_s_median": float(np.median(r["dec_s"])),
                     "bits_per_dim": 32.0 * r["words"] / dims, "roundtrip_ok": bool(r["roundtrip_ok"])}
    out["host_compressors_full_images"] = host_compressors(images)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
