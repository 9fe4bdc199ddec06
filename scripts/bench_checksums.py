"""What per-block checksums cost: `python scripts/bench_checksums.py [--images 4096 --rounds 3 --warmup 1 --lanes 4]`.

Workloads (synthetic weights, tensor cores, a PipelinedCodec of up to `--lanes` free-running lanes sized to the chain count):
bench_archive.py's cifar8 (32 x 32 x 3) and mnist2 (28 x 28 x 1) sets of `--images` synthetic_images(kind="smooth"), each as
per-image containers (compress_images(edges="code")) and as an archive at chain_blocks=16, and bench_chains.py's 2048 x 1536
synthetic photo at chain_blocks=32 on imagenetcrop4.  Per workload, checksums=False and checksums=True alternate round by
round after `--warmup` rounds of each; a round is the writer call plus the full decode, both ended by a device synchronise.
Reported per arm: median encode and decode seconds, stored words and the words the digests add, and whether every round trip
was exact and the checked arrays were the unchecked ones plus their trailers.  One more checked round per workload runs under
torch.profiler (traces in a temporary directory, or `--out`): the device time of k_block_digests, encode and decode, against
the HBM bound of reading every digested slot once (blocks x C x 1024 bytes at 3.35 TB/s, the H100 SXM data-sheet figure).
The card's name and power limit are read in the same run.
"""
import argparse
import glob
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from scripts.bench_chains import synthetic_photo                 # noqa: E402
from scripts.bench_edges import card                             # noqa: E402

HBM_BYTES_S = 3.35e12


def _digest_kernels(trace):
    """(device seconds, launches) of k_block_digests in a chrome trace torch.profiler wrote."""
    ev = json.load(open(trace))["traceEvents"]
    ks = [e["dur"] / 1e6 for e in ev if e.get("cat") == "kernel" and "k_block_digests" in e["name"]]
    return float(sum(ks)), len(ks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--lanes", type=int, default=4)
    ap.add_argument("--out", default=None, help="directory for the profiler traces (default: a temporary one)")
    args = ap.parse_args()
    from bitswap_b200 import synthetic
    from bitswap_b200.config import preset
    from bitswap_b200.codec import PipelinedCodec, Bins
    from bitswap_b200.container import (CHECK_MARK, chain_sizes, compress_archive, compress_images, decompress_archive,
                                        decompress_images)

    assert torch.cuda.is_available(), "bench_checksums.py needs a GPU"
    torch.cuda.set_device(0)
    out_dir = args.out or tempfile.mkdtemp(prefix="bench_checksums_")
    os.makedirs(out_dir, exist_ok=True)

    def codec_for(name, chains):
        cfg = preset(name)
        sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
        bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
        return PipelinedCodec(cfg, sd, bins, chains, lanes=min(args.lanes, chains), use_tensor_cores=True, free_running=True)

    def small(name, side):
        imgs = synthetic.synthetic_images(preset(name), args.images, seed=7, kind="smooth")[:, :, :side, :side]
        return [np.ascontiguousarray(im.transpose(1, 2, 0)) for im in imgs]

    jobs = []
    for name, side in (("cifar8", 32), ("mnist2", 28)):
        host = small(name, side)
        C = host[0].shape[2]
        jobs.append(dict(name=f"{name} per-image containers", model=name, chains=args.images, images=host,
                         write=lambda c, ims, k: compress_images(c, ims, edges="code", checksums=k),
                         read=lambda c, s, C=C: decompress_images(c, s, channels=C)))
        jobs.append(dict(name=f"{name} archive chain_blocks=16", model=name, chains=len(chain_sizes(args.images, 16)),
                         images=host, write=lambda c, ims, k: compress_archive(c, ims, chain_blocks=16, checksums=k),
                         read=lambda c, s: decompress_archive(c, s)))
    photo = [synthetic_photo(1536, 2048, seed=0)]
    jobs.append(dict(name="photo 2048 x 1536 chain_blocks=32", model="imagenetcrop4", chains=96, images=photo,
                     write=lambda c, ims, k: compress_images(c, ims, edges="code", chain_blocks=32, checksums=k),
                     read=lambda c, s: decompress_images(c, s)))

    out = {"card": card(), "workload": f"{args.images} synthetic_images(kind='smooth', seed=7) per set, the photo of "
                                       f"bench_chains.py; tensor cores, up to {args.lanes} free-running lanes; "
                                       f"{args.rounds} alternated rounds per arm after {args.warmup} warm-up"}
    for job in jobs:
        codec = codec_for(job["model"], job["chains"])
        stored = {}

        def one_round(checked):
            t0 = time.perf_counter()
            s = job["write"](codec, job["images"], checked)
            torch.cuda.synchronize()
            te = time.perf_counter() - t0
            t0 = time.perf_counter()
            back = job["read"](codec, s)
            torch.cuda.synchronize()
            td = time.perf_counter() - t0
            stored[checked] = s
            return te, td, len(back) == len(job["images"]) and all(np.array_equal(b, w) for b, w in zip(back, job["images"]))

        res = {k: dict(enc=[], dec=[], exact=True) for k in (False, True)}
        for r in range(args.warmup + args.rounds):
            for checked in (False, True):
                te, td, ok = one_round(checked)
                res[checked]["exact"] &= ok
                if r >= args.warmup:
                    res[checked]["enc"].append(te)
                    res[checked]["dec"].append(td)
                    print(f"{job['name']} checksums={checked}: encode {te:.3f} s, decode {td:.3f} s", file=sys.stderr,
                          flush=True)
        plain, checked = stored[False], stored[True]
        plain, checked = ([plain], [checked]) if isinstance(plain, np.ndarray) else (plain, checked)
        blocks = sum(int(c[-3]) for c in checked)
        layout_ok = all(c[-1] == CHECK_MARK and c.size == p.size + int(c[-3]) + 3 and np.array_equal(c[:p.size], p)
                        for p, c in zip(plain, checked))
        words = [sum(a.size for a in plain), sum(a.size for a in checked)]
        tdir = os.path.join(out_dir, f"trace_{len(out)}")
        os.makedirs(tdir, exist_ok=True)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA],
                                    on_trace_ready=torch.profiler.tensorboard_trace_handler(tdir)):
            one_round(True)
        sec, launches = _digest_kernels(sorted(glob.glob(os.path.join(tdir, "*.json")))[-1])
        C = job["images"][0].shape[2]
        moved = 2 * blocks * C * 1024                                   # every slot read once by the encoder and the decoder
        out[job["name"]] = {
            "blocks": blocks, "words_unchecked": words[0], "words_checked": words[1],
            "words_added_percent": 100.0 * (words[1] - words[0]) / words[0],
            **{("checked" if k else "unchecked"): {
                "encode_s_median": float(np.median(r["enc"])), "decode_s_median": float(np.median(r["dec"])),
                "encode_s": r["enc"], "decode_s": r["dec"], "roundtrip_ok": bool(r["exact"])} for k, r in res.items()},
            "checked_is_unchecked_plus_trailer": bool(layout_ok),
            "k_block_digests": {"device_s": sec, "launches": launches, "bytes_min": moved, "hbm_bound_s": moved / HBM_BYTES_S,
                                "fraction_of_hbm_bound": moved / HBM_BYTES_S / sec if sec else None}}
        print(json.dumps({job["name"]: out[job["name"]]}), file=sys.stderr, flush=True)
        del codec
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
