"""Host corpora against attached corpus images (Corpus.share / Corpus.attach) on the same requests.

Two workloads, each over a host corpus (Corpus(memory="host"), a private cudaHostAlloc copy) and over an attached
image of the same index on /dev/shm (its pages registered with cudaHostRegister), alternated over `--rounds` rounds:

1. bench_corpus.py's: 8 C2-shaped files, crop batches of 256 crops of 176 400 samples, f32, requests drawn beforehand
   on the device;
2. bench_packed.py's: 96 C2-shaped files of 1-30 s, packed batches of whole files filling T = 8.4 M samples.

Device time per call comes from CUDA events around all draws back to back.  The bytes each call gathers are computed on
the host from the plan, and over the call's time and over the gather kernel's own time (a torch.profiler run of its
own) give the gather rate from each kind of pinned memory.  Every draw is checked bit for bit between the two corpora
first.  Also: the time Corpus.share takes to write an image and attach it, and the time clx_corpus_attach takes (check,
registration, index upload) per GB of image, on an image of `--attach-gb` GB made of the crop workload's files repeated
(capped at half of /dev/shm's free space).  The card's name, power limit and SM clock are read in the same run.  One
JSON line.

    python tools/bench_shared_corpus.py
    python tools/bench_shared_corpus.py --rounds 3 --attach-gb 2
"""
from __future__ import annotations

import argparse
import json
import mmap
import os
import sys
import time
import uuid

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import claxon_b200 as cb  # noqa: E402
from tools import bench_corpus, bench_packed  # noqa: E402
from tools.bench_crops import make_files  # noqa: E402
from tools.bench_out_modes import gpu_info  # noqa: E402


def shm_path(tag):
    return os.path.join("/dev/shm", f"clx-bench-{tag}-{os.getpid()}-{uuid.uuid4().hex[:8]}.clxc")


def device_ms(call, items):
    import torch
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for x in items:
        call(x)
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / len(items)


def timed_share(idx, path, ctx):
    t0 = time.perf_counter()
    corpus = cb.Corpus.share(idx, path, ctx)
    return corpus, time.perf_counter() - t0


def attach_seconds(path, ctx, reps):
    """Seconds per Corpus.attach of an already mapped image (the mapping is made once, outside the clock)."""
    with open(path, "r+b") as f:
        mm = mmap.mmap(f.fileno(), 0)
    per = []
    for _ in range(reps):
        t0 = time.perf_counter()
        c = cb.Corpus.attach(mm, ctx)
        per.append(time.perf_counter() - t0)
        c.close()
        del c
    return float(np.median(per)), len(mm)


def main():
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=50, help="crop-batch draws")
    ap.add_argument("--packed-draws", type=int, default=20)
    ap.add_argument("--attach-gb", type=float, default=4.0, help="size of the image attach is timed on")
    ap.add_argument("--attach-reps", type=int, default=3)
    ap.add_argument("--profile-calls", type=int, default=10)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    ctx = cb.Context(device=0)
    paths = []
    try:
        # 1. crops
        n, B = 176400, 256
        idx = cb.index(make_files(8, 800))
        host = cb.Corpus(idx, ctx, memory="host")
        paths.append(shm_path("crops"))
        att, crop_share_s = timed_share(idx, paths[-1], ctx)
        hb, ab = host.crops(B, n, dtype=torch.float32), att.crops(B, n, dtype=torch.float32)
        lens = torch.tensor([f.length for f in idx.files], device="cuda")
        gen = torch.Generator(device="cuda").manual_seed(7)
        draws = []
        for _ in range(args.calls):
            fi = torch.randint(0, len(idx), (B,), device="cuda", generator=gen)
            off = (torch.rand(B, device="cuda", generator=gen) * (lens[fi] - n + 1).double()).long()
            draws.append((fi, off))
        exact = True
        for fi, off in draws:
            ho = hb(fi, off)[0].view(torch.int32).clone()
            exact &= bool(torch.equal(ab(fi, off)[0].view(torch.int32), ho))
        crop_bytes = float(np.mean([bench_corpus.gathered_bytes(host, fi, off, n) for fi, off in draws]))

        # 2. packed
        T = 8_400_000
        rng = np.random.default_rng(2025)
        pidx = cb.index(bench_packed.make_files(96, rng))
        pdraws = [bench_packed.draw(pidx, T, rng) for _ in range(args.packed_draws)]
        PB = max(len(d) for d in pdraws)
        phost = cb.Corpus(pidx, ctx, memory="host")
        paths.append(shm_path("packed"))
        patt, packed_share_s = timed_share(pidx, paths[-1], ctx)
        hp, ap_ = phost.packed(PB, T), patt.packed(PB, T)
        for d in pdraws:
            ho = hp(d)[0].view(torch.int32).clone()
            exact &= bool(torch.equal(ap_(d)[0].view(torch.int32), ho))
        packed_bytes = float(np.mean([bench_packed.span_bytes(phost, d) for d in pdraws]))

        calls = {"crops_host": lambda x: hb(*x, check=False), "crops_attached": lambda x: ab(*x, check=False),
                 "packed_host": lambda d: hp(d, check=False), "packed_attached": lambda d: ap_(d, check=False)}
        items = {"crops": draws, "packed": pdraws}
        for name, call in calls.items():
            for x in items[name.split("_")[0]][:3]:
                call(x)
        ms = {k: [] for k in calls}
        for _ in range(args.rounds):
            for name, call in calls.items():
                ms[name].append(device_ms(call, items[name.split("_")[0]]))
        info = gpu_info()
        kernels_us = {name: bench_corpus.profile_kernels(call, items[name.split("_")[0]][:args.profile_calls],
                                                         "excerpt_") for name, call in calls.items()}
        gbps = {}
        for name in calls:
            nbytes = crop_bytes if name.startswith("crops") else packed_bytes
            gather = kernels_us[name].get("excerpt_gather_kernel")
            gbps[name] = {"over_call": round(nbytes / (float(np.median(ms[name])) * 1e6), 2),
                          "over_gather_kernel": round(nbytes / (gather * 1e3), 2) if gather else None}
        del hb, ab, hp, ap_
        att.close()
        patt.close()

        # 3. attach (registration) cost on a large image: the crop files repeated
        free = os.statvfs("/dev/shm")
        free_gb = free.f_bavail * free.f_frsize / 1e9
        per_copy = sum(f.data.size for f in idx.files)
        copies = max(1, int(min(args.attach_gb, free_gb / 2) * 1e9 / per_copy))
        big = cb.FlacIndex([f for _ in range(copies) for f in idx.files])
        paths.append(shm_path("attach"))
        c, big_share_s = timed_share(big, paths[-1], ctx)
        c.close()
        del c
        attach_s, image_bytes = attach_seconds(paths[-1], ctx, args.attach_reps)
        small_attach_s, small_bytes = attach_seconds(paths[0], ctx, args.attach_reps)
        attach = {"image_bytes": image_bytes, "attach_s": round(attach_s, 4),
                  "attach_s_per_GB": round(attach_s / (image_bytes / 1e9), 4),
                  "share_s": round(big_share_s, 3), "share_s_per_GB": round(big_share_s / (image_bytes / 1e9), 3),
                  "small_image_bytes": small_bytes, "small_attach_s": round(small_attach_s, 4),
                  "dev_shm_free_GB": round(free_gb, 1)}
        row = {"bench": "shared_corpus", "rounds": args.rounds, "bit_exact_attached_vs_host": exact,
               "crops": {"batch": B, "num_frames": n, "files": 8, "draws": args.calls, "gathered_bytes_per_call": int(crop_bytes),
                         "image_bytes": os.path.getsize(paths[0]), "share_s": round(crop_share_s, 3)},
               "packed": {"T": T, "files": 96, "draws": args.packed_draws, "gathered_bytes_per_call": int(packed_bytes),
                          "image_bytes": os.path.getsize(paths[1]), "share_s": round(packed_share_s, 3)},
               "ms_per_call": {k: bench_corpus.stats(v) for k, v in ms.items()},
               "ms_rounds": {k: [round(x, 4) for x in v] for k, v in ms.items()},
               "gather_GBps": gbps, "kernels_us_per_call": kernels_us, "attach": attach, "gpu": info}
        line = json.dumps(row)
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")
    finally:
        for p in paths:
            if os.path.lexists(p):
                os.unlink(p)
    ctx.close()


if __name__ == "__main__":
    main()
