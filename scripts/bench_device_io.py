"""Images in and out as CUDA tensors: `python scripts/bench_device_io.py [--images 4096 --rounds 3 --warmup 1 --out DIR]`.

Two arms, alternated round by round in one process after `--warmup` rounds of each:
  numpy  a list of HWC numpy arrays in, numpy arrays out (what bench_archive.py runs);
  cuda   one [N, H, W, C] CUDA tensor in (a CUDA image for the photo), as_tensors=True out.
Workloads: bench_archive.py's cifar8 (4096 32 x 32 RGB) and mnist2 (4096 28 x 28) sets, as per-image containers
(compress_images(edges="code")) and as an archive at chain_blocks 16; the 2048 x 1536 synthetic photo of bench_chains.py on
imagenetcrop4 at chain_blocks 32; and a training batch: 256 random images of the cifar8 archive decoded in one
decompress_archive call.  All on the tensor cores with up to 4 free-running lanes, one PipelinedCodec sized to the chains.
Per workload and arm: encode and decode seconds, their host time (wall time outside the span from the first coder call to
the end of the last coder kernel, scripts/bench_chains.py's DeviceSpan) and Mpixel/s, medians over the rounds; the host
time split by phase, from a cProfile run of one round of its own (cumulative seconds of the container's phases); and, from a
torch.profiler run of one more round, the bytes copied host to device and device to host and the tile / untile kernels'
device time against the HBM bound of the bytes they move (3.35 TB/s, the H100 SXM data sheet).  Every round trip is checked
exact.  The card's name and power limit are read in the same run.
"""
import argparse
import cProfile
import glob
import json
import os
import pstats
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from scripts.bench_chains import DeviceSpan, synthetic_photo     # noqa: E402
from scripts.bench_edges import card                             # noqa: E402

HBM_BYTES_S = 3.35e12
PHASES = {                                                       # cProfile function name (container.py / streams.py) -> phase
    "__init__": "images: check and describe", "views": "images: upload", "_tile": "tile (with upload)",
    "_sequence_extents": "extents and chain table", "_chain_runs": "extents and chain table",
    "fill": "stream set: create and fill", "import_packed": "stream set: import", "raise_on_error": "stream flags (sync)",
    "pack_device": "readback: pack", "_compress_chains": "encode loop, sync and readback", "pack_container": "pack containers",
    "pack_archive": "pack archive", "_stamped_job": "parse containers", "_archive_job": "parse archive", "_plan": "plan",
    "_decode_extents": "decode extents", "_untile": "untile", "_check_initial_state": "initial-state check",
    "_decode_regions": "decode (all of it)", "_encode": "encode (all of it)"}


def _phases(prof):
    st = pstats.Stats(prof)
    out = {}
    for (fn, _, name), (_, _, _, cum, _) in st.stats.items():
        if name in PHASES and os.path.basename(fn) in ("container.py", "streams.py"):
            key = PHASES[name] + (" [StreamSet]" if name == "__init__" and fn.endswith("streams.py") else "")
            out[key] = out.get(key, 0.0) + cum
    return {k: round(v, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def _transfers(trace):
    """(HtoD bytes, DtoH bytes, {kernel: (device seconds, launches)}) of a chrome trace torch.profiler wrote."""
    ev = json.load(open(trace))["traceEvents"]
    htod = sum(e["args"].get("bytes", 0) for e in ev if e.get("cat") == "gpu_memcpy" and "HtoD" in e["name"])
    dtoh = sum(e["args"].get("bytes", 0) for e in ev if e.get("cat") == "gpu_memcpy" and "DtoH" in e["name"])
    ks = {}
    for e in ev:
        if e.get("cat") == "kernel" and ("k_tile_blocks" in e["name"] or "k_untile_regions" in e["name"]):
            k = "k_tile_blocks" if "k_tile_blocks" in e["name"] else "k_untile_regions"
            s, n = ks.get(k, (0.0, 0))
            ks[k] = (s + e["dur"] / 1e6, n + 1)
    return htod, dtoh, ks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--lanes", type=int, default=4)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default=None, help="directory for the profiler traces (default: a temporary one)")
    args = ap.parse_args()
    from bitswap_b200 import synthetic
    from bitswap_b200.config import preset
    from bitswap_b200.codec import PipelinedCodec, Bins
    from bitswap_b200.container import (chain_sizes, compress_archive, compress_images, decompress_archive,
                                        decompress_images)

    assert torch.cuda.is_available(), "bench_device_io.py needs a GPU"
    torch.cuda.set_device(0)
    out_dir = args.out or tempfile.mkdtemp(prefix="bench_device_io_")
    os.makedirs(out_dir, exist_ok=True)

    def model(name):
        cfg = preset(name)
        return cfg, synthetic.synthetic_state_dict(cfg, seed=50, varied=False), Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))

    def codec_for(m, chains):
        cfg, sd, bins = m
        return DeviceSpan(PipelinedCodec(cfg, sd, bins, chains, lanes=min(args.lanes, chains), use_tensor_cores=True,
                                         free_running=True))

    def small(name, side):
        cfg = preset(name)
        imgs = synthetic.synthetic_images(cfg, args.images, seed=7, kind="smooth")[:, :, :side, :side]
        return [np.ascontiguousarray(im.transpose(1, 2, 0)) for im in imgs]

    def arms(host):
        dev = torch.from_numpy(np.stack(host)).cuda() if len(host) > 1 else torch.from_numpy(host[0]).cuda()
        return {"numpy": host, "cuda": dev if len(host) > 1 else [dev]}

    rs = np.random.RandomState(11)
    jobs = []                     # dict(name, codec, inputs per arm, want, write, read, source: the job whose output it reads)
    for wl, (name, side) in {"cifar": ("cifar8", 32), "mnist": ("mnist2", 28)}.items():
        m, host = model(name), small(name, side)
        C = host[0].shape[2]
        jobs.append(dict(name=f"{wl} per-image containers", codec=codec_for(m, args.images), inputs=arms(host), want=host,
                         write=lambda c, ims: compress_images(c, ims, edges="code"),
                         read=lambda c, s, t, C=C: decompress_images(c, s, channels=C, as_tensors=t)))
        arch = dict(name=f"{wl} archive chain_blocks=16", codec=codec_for(m, len(chain_sizes(args.images, 16))),
                    inputs=arms(host), want=host, write=lambda c, ims: compress_archive(c, ims, chain_blocks=16),
                    read=lambda c, s, t: decompress_archive(c, s, as_tensors=t))
        jobs.append(arch)
        if wl == "cifar":
            pick = rs.choice(args.images, args.batch, replace=False)
            regions = [(int(i), 0, 0, side, side) for i in pick]
            jobs.append(dict(name=f"cifar training batch of {args.batch} from the archive", codec=arch["codec"],
                             want=[host[i] for i in pick], source=arch["name"],
                             read=lambda c, s, t, r=regions: decompress_archive(c, s, r, as_tensors=t)))
    photo = [synthetic_photo(1536, 2048, seed=0)]
    jobs.append(dict(name="photo 2048 x 1536 chain_blocks=32", codec=codec_for(model("imagenetcrop4"), 96), inputs=arms(photo),
                     want=photo, write=lambda c, ims: compress_images(c, ims, edges="code", chain_blocks=32),
                     read=lambda c, s, t: decompress_images(c, s, as_tensors=t)))

    stored = {}

    def one_round(job, arm):
        codec, te, he = job["codec"], 0.0, 0.0
        if "source" in job:
            s = stored[job["source"], arm]
        else:
            codec.reset()
            t0 = time.perf_counter()
            s = stored[job["name"], arm] = job["write"](codec, job["inputs"][arm])
            torch.cuda.synchronize()
            te = time.perf_counter() - t0
            he = te - codec.seconds()
        codec.reset()
        t0 = time.perf_counter()
        back = job["read"](codec, s, arm == "cuda")
        torch.cuda.synchronize()
        td = time.perf_counter() - t0
        ok = len(back) == len(job["want"]) and all(np.array_equal(b.cpu().numpy() if torch.is_tensor(b) else b, w)
                                                   for b, w in zip(back, job["want"]))
        return te, td, he, td - codec.seconds(), ok

    res = {}
    for job in jobs:
        name = job["name"]
        for _ in range(args.warmup):
            for arm in ("numpy", "cuda"):
                one_round(job, arm)
        for _ in range(args.rounds):
            for arm in ("numpy", "cuda"):
                te, td, he, hd, ok = one_round(job, arm)
                r = res.setdefault((name, arm), dict(enc=[], dec=[], enc_host=[], dec_host=[], exact=True, want=job["want"]))
                r["enc"].append(te)
                r["dec"].append(td)
                r["enc_host"].append(he)
                r["dec_host"].append(hd)
                r["exact"] &= ok
                print(f"{name} [{arm}]: encode {te:.3f} s, decode {td:.3f} s (host {he:.3f} + {hd:.3f} s)", file=sys.stderr,
                      flush=True)
        for arm in ("numpy", "cuda"):
            r = res[name, arm]
            prof = cProfile.Profile()
            prof.enable()
            one_round(job, arm)
            prof.disable()
            r["phases"] = _phases(prof)
            tdir = os.path.join(out_dir, f"trace_{len(res)}_{arm}")
            os.makedirs(tdir, exist_ok=True)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA],
                                        on_trace_ready=torch.profiler.tensorboard_trace_handler(tdir)):
                one_round(job, arm)
            r["htod"], r["dtoh"], r["kernels"] = _transfers(sorted(glob.glob(os.path.join(tdir, "*.json")))[-1])
        if "source" in job or not any(j.get("source") == name for j in jobs):
            del job["codec"]                                    # free the codecs no later job decodes with
            torch.cuda.empty_cache()

    out = {"card": card(), "workload": f"{args.images} synthetic_images(kind='smooth', seed=7) per set, the photo of "
                                       f"bench_chains.py; tensor cores, up to {args.lanes} free-running lanes; "
                                       f"{args.rounds} alternated rounds per arm after {args.warmup} warm-up"}
    for (name, arm), r in res.items():
        want = r["want"]
        px = sum(im.shape[0] * im.shape[1] for im in want)
        pix_bytes = sum(im.size for im in want)
        steps = np.array(r["enc"]) + np.array(r["dec"])
        kern = {}
        for k, (sec, n) in r["kernels"].items():
            moved = 2 * pix_bytes                                     # each pixel byte read once and written once (at least)
            kern[k] = {"device_s": sec, "launches": n, "bytes_min": moved, "hbm_bound_s": moved / HBM_BYTES_S,
                       "fraction_of_hbm_bound": moved / HBM_BYTES_S / sec if sec else None}
        out[f"{name} [{arm}]"] = {
            "encode_s_median": float(np.median(r["enc"])), "decode_s_median": float(np.median(r["dec"])),
            "encode_host_s_median": float(np.median(r["enc_host"])), "decode_host_s_median": float(np.median(r["dec_host"])),
            "Mpixel_s_median": px / float(np.median(steps)) / 1e6, "htod_bytes_per_round": r["htod"],
            "dtoh_bytes_per_round": r["dtoh"], "pixel_bytes": pix_bytes, "tile_untile_kernels": kern,
            "host_phases_s (cProfile, one round)": r["phases"], "roundtrip_ok": bool(r["exact"])}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
