"""What a stamp costs: `python scripts/bench_stamp.py [--reps 3 --images 4096 --rounds 3 --warmup 1]`.

A stamp holds the codec's fingerprint, whose model and bins digests are computed on the device once per model and bins
(bsw_model_digest, bsw_bins_digest) and kept with them.  Two measurements, the card's name and power limit read in the same
run:
  digests  the first digest() of freshly loaded models (cifar8 and imagenetcrop4 on the tensor cores) and of fresh cifar8
           bins at quantbits 10 and 12, `--reps` times each: host clock around a call that ends in a stream synchronise;
  archive  the cifar8 workload of bench_archive.py at chain_blocks=16 (`--images` synthetic 32 x 32 images, a PipelinedCodec
           of up to 4 free-running lanes sized to the chain count), compress_archive + decompress_archive, stamped and
           unstamped alternated round by round after `--warmup` rounds of each (the first stamped warm-up round pays the
           one-off digests).  Per setting: median encode and decode seconds, and whether every round trip was exact and the
           stamped archive was the unstamped one plus 29 words.
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

from scripts.bench_edges import card                         # noqa: E402


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--images", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--lanes", type=int, default=4)
    args = ap.parse_args()
    from bitswap_b200 import synthetic
    from bitswap_b200.config import preset, with_
    from bitswap_b200.codec import Bins, PipelinedCodec
    from bitswap_b200.container import chain_sizes, compress_archive, decompress_archive
    from bitswap_b200.model import Model

    assert torch.cuda.is_available(), "bench_stamp.py needs a GPU"
    torch.cuda.set_device(0)
    out = {"card": card()}

    digests = {}
    for name in ("cifar8", "imagenetcrop4"):
        cfg = preset(name)
        sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
        ts = []
        for _ in range(args.reps):
            m = Model.from_config(cfg, max_batch=1, use_tensor_cores=True).load_state_dict(sd)
            ts.append(timed(m.digest))
            del m
        digests[f"{name} model"] = ts
    for q in (10, 12):
        cfg = with_(preset("cifar8"), quantbits=q)
        zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
        ts = []
        for _ in range(args.reps):
            b = Bins(cfg, zend, zcen)
            ts.append(timed(b.digest))
            del b
            torch.cuda.empty_cache()
        digests[f"cifar8 bins quantbits={q}"] = ts
        del zend, zcen
    out["digest_ms"] = {k: {"median": 1e3 * float(np.median(v)), "all": [1e3 * t for t in v]} for k, v in digests.items()}
    print(json.dumps(out), file=sys.stderr, flush=True)

    cfg = preset("cifar8")
    L = 16
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
    imgs = synthetic.synthetic_images(cfg, args.images, seed=7, kind="smooth")
    images = [np.ascontiguousarray(im.transpose(1, 2, 0)) for im in imgs]
    chains = len(chain_sizes(args.images, L))
    codec = PipelinedCodec(cfg, sd, bins, chains, lanes=min(args.lanes, chains), use_tensor_cores=True, free_running=True)
    res = {s: dict(enc=[], dec=[], exact=True) for s in (False, True)}
    last = {}

    def one_round(stamp):
        t0 = time.perf_counter()
        a = compress_archive(codec, images, chain_blocks=L, stamp=stamp)
        torch.cuda.synchronize()
        te = time.perf_counter() - t0
        t0 = time.perf_counter()
        back = decompress_archive(codec, a)
        torch.cuda.synchronize()
        td = time.perf_counter() - t0
        last[stamp] = a
        return te, td, all(np.array_equal(x, y) for x, y in zip(back, images))

    first = {}
    for w in range(args.warmup):
        for stamp in (False, True):
            te, td, ok = one_round(stamp)
            if w == 0:
                first[stamp] = (te, td)
            res[stamp]["exact"] &= ok
    for _ in range(args.rounds):
        for stamp in (False, True):
            te, td, ok = one_round(stamp)
            print(f"stamp={stamp}: encode {te:.2f} s, decode {td:.2f} s", file=sys.stderr, flush=True)
            res[stamp]["enc"].append(te)
            res[stamp]["dec"].append(td)
            res[stamp]["exact"] &= ok
    layout_ok = last[False].size + 29 == last[True].size and np.array_equal(last[True][:last[False].size], last[False])
    out["archive"] = {
        "workload": f"cifar8, {args.images} synthetic_images(kind='smooth', seed=7), chain_blocks={L} ({chains} chains), "
                    f"tensor cores, {codec.lanes} free-running lanes, {args.rounds} alternated rounds after {args.warmup} "
                    f"warm-up round(s)",
        **{("stamped" if s else "unstamped"): {
            "encode_s_median": float(np.median(r["enc"])), "decode_s_median": float(np.median(r["dec"])),
            "encode_s": r["enc"], "decode_s": r["dec"], "first_warmup_round_s": list(first.get(s, ())),
            "roundtrip_ok": bool(r["exact"])} for s, r in res.items()},
        "stamped_is_unstamped_plus_29_words": bool(layout_ok)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
