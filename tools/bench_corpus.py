"""Crops of a device-resident corpus (Corpus / CropBatch) against load_crops() and the resident windowed batch.

bench_crops.py's workload: C2-shaped files (16-bit stereo, 4096-sample frames), B = 256 excerpts of 176 400 samples
(4 s at 44.1 kHz), f32.  In one process, alternated over `--rounds` rounds:

1. crop-batch calls back to back, requests drawn beforehand on the device with torch.randint, check=False: device time
   per call from CUDA events on torch's stream around `--calls` calls (the request copies, the graph, the waits);
2. the same calls with check=True (one sync each), host clock per call;
3. load_crops() calls, host clock per call;
4. bench_crops.py's part 1: resident windowed batches of the same shape, Context.run_steps over `--streams` streams;
5. part 1 over a host corpus (Corpus(memory="host")) of the same files, the same draws: each call also gathers the
   crops' spans of frames from pinned host memory over PCIe.

Every crop-batch draw of parts 1 and 5 is checked bit for bit against load_crops() of the same requests once (and the
two batches against each other), before the timed rounds.  A separate torch.profiler run of `--profile-calls` host-corpus
calls gives the gather kernel's own time and the planner kernels'; the bytes each call gathers are computed on the host
from the plan (plan_range over every crop of every draw), and over the gather's time give its PCIe rate.  The card's
name, power limit and SM clock are read in the same run; memory of the crop batches is reported (corpus bytes and the
device memory of each corpus, planar scratch, output, the host-corpus batch's staging buffer).  One JSON line.

    python tools/bench_corpus.py
    python tools/bench_corpus.py --rounds 3 --calls 100
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import claxon_b200 as cb  # noqa: E402
from tools.bench_crops import excerpts, gather, make_files  # noqa: E402
from tools.bench_out_modes import gpu_info  # noqa: E402


def stats(v):
    med = float(np.median(v))
    return {"median": round(med, 4), "min": round(float(np.min(v)), 4),
            "spread": round((float(np.max(v)) - float(np.min(v))) / med, 4) if med else 0.0}


def gathered_bytes(corpus, fi, off, n):
    """Bytes the gather copies for one call: per crop, from its first planned frame's start to its last one's end."""
    total = 0
    for f, o in zip(fi.tolist(), off.tolist()):
        x = corpus.index[f]
        sel, _, _ = cb.plan_range(x.descs, o, min(o + n, x.length), starts=x.starts)
        if sel.size:
            total += int(x.descs["byte_offset"][sel[-1]]) + int(x.descs["byte_len"][sel[-1]]) - int(x.descs["byte_offset"][sel[0]])
    return total


def profile_kernels(call, items, match):
    """Device time per call(x), x in items, of each kernel whose name contains `match` (us), from a torch.profiler run
    of its own.  Kernels are named without namespace and template arguments: "void clx::k<clx::CropLayout>(...)" is k."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for x in items:
            call(x)
        torch.cuda.synchronize()
    us = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = getattr(e, "cuda_time_total", 0) if t is None else t
        if t and match in e.key:
            name = e.key.split("(")[0].split("<")[0].split("::")[-1].split()[-1]
            us[name] = round(us.get(name, 0.0) + t / len(items), 2)
    return us


def main():
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--files", type=int, default=8)
    ap.add_argument("--frames", type=int, default=800, help="frames per file (4096 samples each)")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--num-frames", type=int, default=176400)
    ap.add_argument("--calls", type=int, default=50, help="crop-batch calls per round (parts 1 and 2)")
    ap.add_argument("--load-crops-calls", type=int, default=3, help="load_crops() calls per round")
    ap.add_argument("--units", type=int, default=4, help="resident windowed batches of part 4")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--streams", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-calls", type=int, default=20, help="host-corpus calls in the torch.profiler run")
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    n, B = args.num_frames, args.batch
    ctx = cb.Context(device=0, n_streams=args.streams)
    idx = cb.index(make_files(args.files, args.frames))
    rng = np.random.default_rng(2024)

    corpus = cb.Corpus(idx, ctx)
    batch = corpus.crops(B, n, dtype=torch.float32)
    slots = B * corpus.frames_bound(n)
    slot_elems = (max(192, int((corpus.descs["n_channels"].astype(np.int64) * corpus.descs["block_size"]).max())) + 3) & ~3
    host = cb.Corpus(idx, ctx, memory="host")
    hbatch = host.crops(B, n, dtype=torch.float32)
    span_stride = (host.bytes_bound(n) + 30) & ~15
    memory = {"corpus_bytes": corpus.nbytes, "slots": slots, "planar_scratch_bytes": slots * slot_elems * 4,
              "output_bytes": B * corpus.channels * n * 4, "trash_rows_bytes": corpus.channels * n * 4,
              "device_corpus_device_bytes": corpus.device_bytes, "host_corpus_device_bytes": host.device_bytes,
              "host_batch_staging_bytes": B * span_stride, "crop_bytes_bound": host.bytes_bound(n)}

    # requests drawn on the device; the largest offset keeps every crop whole, as in bench_crops.py
    lens = torch.tensor([f.length for f in idx.files], device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(7)
    draws = []
    for _ in range(args.calls):
        fi = torch.randint(0, len(idx), (B,), device="cuda", generator=gen)
        off = (torch.rand(B, device="cuda", generator=gen) * (lens[fi] - n + 1).double()).long()
        draws.append((fi, off))
    exact, host_exact = True, True
    for fi, off in draws[:3]:
        out, lengths = batch(fi, off)
        exp, elen = cb.load_crops(idx, fi.tolist(), off.tolist(), n, ctx=ctx)
        exact &= bool(torch.equal(out.view(torch.int32), exp.view(torch.int32)) and torch.equal(lengths.cpu(), elen))
        out_d = out.clone()
        out, lengths = hbatch(fi, off)
        host_exact &= bool(torch.equal(out.view(torch.int32), exp.view(torch.int32)) and torch.equal(lengths.cpu(), elen)
                           and torch.equal(out.view(torch.int32), out_d.view(torch.int32)))
    per_call = [gathered_bytes(host, fi, off, n) for fi, off in draws]
    gathered = {"mean_per_call": int(np.mean(per_call)), "min": int(np.min(per_call)), "max": int(np.max(per_call))}

    win = []
    for _ in range(args.units):
        files, offsets = excerpts(idx, B, n, rng)
        data, descs, w = gather(idx, files, offsets, n, 2)
        win.append(ctx.upload(data, descs, mode=cb.OUT_CHANNELS_F32, channels=2 * B, channel_stride=n, windows=w))
    ctx.run_steps(win, args.units * 2, args.streams)
    for fi, off in draws[:5]:
        batch(fi, off, check=False)
        hbatch(fi, off, check=False)
    torch.cuda.synchronize()

    def device_ms(b):  # device time per call, back to back over every draw
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for fi, off in draws:
            b(fi, off, check=False)
        stop.record()
        stop.synchronize()
        return start.elapsed_time(stop) / len(draws)

    ms = {"crop_batch_device": [], "host_corpus_crop_batch_device": [], "crop_batch_checked_host": [],
          "load_crops_host": [], "windowed_resident_device": []}
    for _ in range(args.rounds):
        ms["crop_batch_device"].append(device_ms(batch))
        ms["host_corpus_crop_batch_device"].append(device_ms(hbatch))
        per = []
        for fi, off in draws:
            t0 = time.perf_counter()
            batch(fi, off, check=True)
            per.append((time.perf_counter() - t0) * 1e3)
        ms["crop_batch_checked_host"].append(float(np.median(per)))
        per = []
        for _ in range(args.load_crops_calls):
            files, offsets = excerpts(idx, B, n, rng)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            cb.load_crops(idx, files, offsets, n, ctx=ctx)
            torch.cuda.synchronize()
            per.append((time.perf_counter() - t0) * 1e3)
        ms["load_crops_host"].append(float(np.median(per)))
        ms["windowed_resident_device"].append(ctx.run_steps(win, args.steps, args.streams) / args.steps)
    info = gpu_info()
    for dev in win:
        dev.close()
    kernels_us = profile_kernels(lambda d: hbatch(*d, check=False), draws[:args.profile_calls], "excerpt_")
    prof_bytes = float(np.mean(per_call[:args.profile_calls]))
    gather_us = kernels_us.get("excerpt_gather_kernel")
    host_ms = float(np.median(ms["host_corpus_crop_batch_device"]))
    gathered.update({"gather_kernel_GBps": round(prof_bytes / (gather_us * 1e3), 2) if gather_us else None,
                     "over_whole_call_GBps": round(gathered["mean_per_call"] / (host_ms * 1e6), 2)})
    row = {"bench": "corpus_crops", "batch": B, "num_frames": n, "files": args.files, "frames_per_file": args.frames,
           "rounds": args.rounds, "calls": args.calls, "bit_exact_vs_load_crops": exact,
           "host_corpus_bit_exact_vs_load_crops_and_device_corpus": host_exact,
           "ms_per_call": {k: stats(v) for k, v in ms.items()}, "ms_rounds": {k: [round(x, 4) for x in v] for k, v in ms.items()},
           "host_corpus_kernels_us_per_call": kernels_us, "gathered_bytes": gathered, "memory": memory, "gpu": info}
    line = json.dumps(row)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    del batch, hbatch
    corpus = host = None
    ctx.close()


if __name__ == "__main__":
    main()
