"""BASELINE.json configs[4]: 100 variable-size images as chained 32x32 block streams over the GPUs of one box, next to
gzip / bz2 / lzma / PNG / WebP on the host -- `python bench.py --config crop [--gpus N]` (torchrun for N > 1).

Reference: imagenetcrop_compress.py:127-210 -- every image is ONE ANS chain over its blocks (fresh initial state per image,
:122), coded with the imagenetcrop model (nz = 4, W = 256, conditional x-scale head); benchmark_compress.py:64-103 for the
host compressors.  Here the chains are dealt to the ranks by `parallel.shard_by_cost` (greedy longest-first over block
counts, SURVEY.md 8e), every rank codes its chains as one StreamSet (one stream per image, step t = block t of every
image that has one), and rank 0 gathers the demo-format containers (demo_compress.py:268-284).

A chain is strictly sequential in its blocks (the whole point of bits-back chaining), so this configuration is
latency-bound by construction: ~13 streams per GPU x up to 256 dependent steps of ~45 kernel launches.  Synthetic smooth
images and random-init weights: the rates are NOT the paper's; the path, its exactness and its throughput are the point.
"""
import bz2
import gzip
import io
import json
import lzma
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def synthetic_crop_images(n, seed=0):
    """n HWC uint8 images with H, W ~ U{224..512} (49..256 blocks of 32x32 after cropping, SURVEY.md 8d config 5)."""
    rs = np.random.RandomState(seed)
    images = []
    for _ in range(n):
        h, w = rs.randint(224, 513, 2)
        yy, xx = np.mgrid[0:h, 0:w]
        img = np.stack([128 + 60 * np.sin(xx * rs.uniform(0.01, 0.1) + yy * rs.uniform(0.01, 0.1) + rs.uniform(0, 6)) +
                        rs.normal(0, 6, (h, w)) for _ in range(3)], axis=-1)
        images.append(np.clip(np.rint(img), 0, 255).astype(np.uint8))
    return images


def host_compressors(crops):
    """bits/dim of the host compressors the reference compares with (benchmark_compress.py:64-103)."""
    dims = sum(c.size for c in crops)
    raw = [c.tobytes() for c in crops]
    res = {"gzip": sum(8 * len(gzip.compress(r)) for r in raw) / dims,
           "bz2": sum(8 * len(bz2.compress(r)) for r in raw) / dims,
           "lzma": sum(8 * len(lzma.compress(r)) for r in raw) / dims}
    try:
        import PIL.Image as pimg
        from PIL.PngImagePlugin import getchunks

        def png_idat(c):                                      # IDAT chunks only, as benchmark_compress.py:80-84
            return 8 * sum(len(d) for t, d, _ in getchunks(pimg.fromarray(c), optimize=True) if t == b"IDAT")

        def webp(c):
            b = io.BytesIO()
            pimg.fromarray(c).save(b, format="WebP", lossless=True, quality=100)
            return 8 * len(b.getvalue())
        res["png"] = sum(png_idat(c) for c in crops) / dims
        res["webp"] = sum(webp(c) for c in crops) / dims
    except Exception as e:                                    # noqa: BLE001
        res["pil"] = str(e)
    return res


def run_crop(args, rank, world, local):
    import torch.distributed as dist
    from bitswap_b200 import synthetic, parallel
    from bitswap_b200.config import preset
    from bitswap_b200.model import Model
    from bitswap_b200.codec import PipelinedCodec, Bins
    from bitswap_b200.container import compress_images, decompress_images

    assert torch.cuda.is_available(), "bench.py needs a GPU (no CPU fallback for the product path)"
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = torch.device("cuda", local)
    cfg = preset("imagenetcrop4")
    n = args.crop_images
    images = synthetic_crop_images(n, seed=0)                 # every rank builds the same list; it codes only its shard
    crops = [im[:im.shape[0] - im.shape[0] % 32, :im.shape[1] - im.shape[1] % 32] for im in images]
    costs = [c.shape[0] * c.shape[1] // 1024 for c in crops]
    shards = parallel.shard_by_cost(costs, world)
    mine = shards[rank]
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    # a chain is sequential in its blocks, so one step of one lane is a string of small latency-bound kernels (<= 100 images:
    # less than one wave of conv CTAs); the lanes of a free-running PipelinedCodec code disjoint groups of chains concurrently
    lanes = max(1, min(args.lanes if args.lanes > 0 else 4, len(mine)))
    codec = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), max(1, len(mine)), lanes=lanes, use_tensor_cores=True, free_running=True)
    my_images = [images[i] for i in mine]

    def sync():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    def one_step():
        t0 = time.perf_counter()
        conts = compress_images(codec, my_images, hwc_quirk=args.hwc_quirk) if my_images else []
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        gathered = [conts]
        if world > 1:                                         # every rank receives every container (the "gather the final bitstreams" step):
            # one device buffer of container words + lengths per rank, NCCL all_gather_into_tensor (parallel.gather_packed)
            flat = np.concatenate(conts).view(np.int32) if conts else np.zeros(0, np.int32)
            words_t = torch.from_numpy(flat.copy()).to(dev) if flat.size else torch.zeros(1, dtype=torch.int32, device=dev)
            lens_t = torch.tensor([len(c) for c in conts], dtype=torch.int64, device=dev)
            W, M, counts = parallel.gather_packed(words_t, lens_t, torch.zeros_like(lens_t))
            Wh, Mh, ch = W.cpu().numpy().view(np.uint32), M.cpu().numpy(), counts.cpu().numpy()
            gathered = []
            for r in range(world):
                off = np.concatenate([[0], np.cumsum(Mh[r, 0, :int(ch[r, 1])])]).astype(np.int64)
                gathered.append([Wh[r, off[i]:off[i + 1]].copy() for i in range(int(ch[r, 1]))])
        t2 = time.perf_counter()
        back = decompress_images(codec, conts, hwc_quirk=args.hwc_quirk) if my_images else []
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        return conts, gathered, back, (t1 - t0, t2 - t1, t3 - t2)

    for _ in range(max(args.warmup, 1)):
        one_step()
    sync()
    enc = gat = dec = 0.0
    launches = 0
    for _ in range(args.steps):
        conts, gathered, back, (a, b, c) = one_step()
        enc += a; gat += b; dec += c
        launches += 2 * max(costs[i] for i in mine) * codec.last_launches if mine else 0
    sync()
    assert all(np.array_equal(crops[i], r) for i, r in zip(mine, back)), "round trip failed"
    t = torch.tensor([enc, gat, dec], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    enc, gat, dec = t.tolist()
    dims = sum(c.size for c in crops)
    px = dims / 3
    value = px * args.steps / (enc + gat + dec) / 1e6
    if rank == 0:
        by_index = {}
        for r, g in enumerate(gathered):
            for i, c in zip(shards[r], g):
                by_index[i] = c
        assert sorted(by_index) == list(range(n)), "rank 0 did not receive every container"
        bits = sum(32 * (len(by_index[i]) - 3) for i in range(n))
        line = {"metric": "Mpixels/sec encode+decode (Bit-Swap, variable-size images as chained 32x32 block streams)", "value": value,
                "unit": "Mpixel/s", "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 1),
                "ms_per_step": 1e3 * (enc + gat + dec) / args.steps, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
                "dtype": "f64 tables / int64 coder / bf16x3 split wgmma convs", "data": "synthetic",
                "config": {"workload": f"BASELINE configs[4]: {n} variable-size images (H, W ~ U{{224..512}}, {sum(costs)} blocks of 32x32x3), each "
                                       f"image ONE chain over its blocks, imagenetcrop model (nz=4, W=256, conditional x-scale), chains dealt to "
                                       f"{world} GPU(s) by block count; step = compress every chain + gather the containers on rank 0 + decompress",
                           "chains_per_gpu": [len(s) for s in shards], "blocks_per_gpu": [sum(costs[i] for i in s) for s in shards],
                           "serial_depth_blocks": max(costs), "lanes_per_gpu": lanes, "layout": "HWC quirk of imagenetcrop_compress.py:130" if args.hwc_quirk else "CHW (demo_compress.py:120)",
                           "note": "latency-bound by construction: a chain is sequential in its blocks; timed through the public API with host "
                                   "images in and host containers/images out (this IS the end-to-end number)"},
                "encode_Mpixel_s": px * args.steps / enc / 1e6, "decode_Mpixel_s": px * args.steps / dec / 1e6,
                "container_gather_ms": 1e3 * gat / args.steps,
                "bits_per_dim": {"bitswap_incl_borrowed_initial_bits": bits / dims, **host_compressors(crops)},
                "roundtrip_ok": True, "gpu_launches": int(launches),
                "e2e": {"value": value, "unit": "Mpixel/s", "h2d_bytes_per_step": int(dims), "d2h_bytes_per_step": int(dims + bits // 8)},
                "roofline": None, "cpu_baseline": None}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    print("run through bench.py: python bench.py --config crop [--gpus N --steps K --warmup W]")
