"""Packed batches of whole files (Corpus.packed / PackedBatch) against load() and a padded CropBatch.

C2-shaped files (16-bit stereo, 4096-sample frames) of random length from 1 to 30 s made with synth.make_file.  Each
draw is a random choice of whole files that fills T (8.4 M samples by default) along the columns of one [C, T] tensor.
Every draw is checked bit for bit against load() of the same files once.  Then, alternated over `--rounds` rounds:

1. packed-batch calls back to back over a device corpus, check=False: device time per call from CUDA events on torch's
   stream around every draw;
2. the same over a host corpus (Corpus(memory="host")): each call also gathers the files' frames over PCIe;
3. load() of the same files (their bytes; it demuxes them too), host clock per call;
4. a CropBatch with L = the longest file of any draw, B = the most files of a draw and offsets 0 (files past a draw's
   end get offset = length, so no frames): the padded layout, device time per call.

A torch.profiler run gives each excerpt_* kernel's own time per call (the planner's cost).  Memory of each (output,
planar scratch, staging) and the byte bound against the bytes actually gathered are reported, with the card's name,
power limit and SM clock read in the same run.  One JSON line.

    python tools/bench_packed.py
    python tools/bench_packed.py --rounds 3 --samples 4200000
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
from claxon_b200 import synth  # noqa: E402
from tools.bench_corpus import profile_kernels, stats  # noqa: E402
from tools.bench_out_modes import gpu_info  # noqa: E402


def make_files(n_files, rng):
    out = []
    for i in range(n_files):
        cfg = synth.workload_config("c2", int(rng.integers(11, 324)))  # 1 to 30 s of 4096-sample frames at 44.1 kHz
        cfg.seed = cfg.seed + 7919 * (i + 1)
        b = synth.generate(cfg)
        out.append(np.frombuffer(synth.make_file(b, 0, b.n_frames), np.uint8).copy())
    return out


def draw(idx, T, rng):
    """Whole files in random order while their columns fit in T."""
    files, at = [], 0
    for f in rng.permutation(len(idx)):
        n = idx[int(f)].length
        if at + n > T:
            break
        files.append(int(f))
        at += (n + 3) & ~3
    return files


def span_bytes(corpus, files):
    return sum(int(corpus.index[f].descs["byte_offset"][-1]) + int(corpus.index[f].descs["byte_len"][-1])
               - int(corpus.index[f].descs["byte_offset"][0]) for f in files)


def main():
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--files", type=int, default=96)
    ap.add_argument("--samples", type=int, default=8_400_000, help="T, the columns of one call")
    ap.add_argument("--draws", type=int, default=20)
    ap.add_argument("--load-calls", type=int, default=2, help="load() calls per round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    T = args.samples
    rng = np.random.default_rng(2025)
    srcs = make_files(args.files, rng)
    ctx = cb.Context(device=0)
    idx = cb.index(srcs)
    draws = [draw(idx, T, rng) for _ in range(args.draws)]
    B = max(len(d) for d in draws)
    longest = max(idx[f].length for d in draws for f in d)

    corpus, host = cb.Corpus(idx, ctx), cb.Corpus(idx, ctx, memory="host")
    packed, hpacked = corpus.packed(B, T), host.packed(B, T)
    crops = corpus.crops(B, longest)
    slot_elems = (max(192, int((corpus.descs["n_channels"].astype(np.int64) * corpus.descs["block_size"]).max())) + 3) & ~3
    C_ = corpus.channels
    memory = {
        "files": args.files, "corpus_bytes": corpus.nbytes, "max_excerpts": B, "T": T, "longest_file": longest,
        "packed": {"output_bytes": C_ * packed.stride * 4, "slots": corpus.packed_frames_bound(B, T),
                   "planar_scratch_bytes": corpus.packed_frames_bound(B, T) * slot_elems * 4,
                   "host_staging_bytes": host.packed_bytes_bound(B, T)},
        "crop_batch_padded": {"output_bytes": (B + 1) * C_ * longest * 4, "slots": B * corpus.frames_bound(longest),
                              "planar_scratch_bytes": B * corpus.frames_bound(longest) * slot_elems * 4}}
    gathered = [span_bytes(corpus, d) for d in draws]
    bytes_bound = {"bound": host.packed_bytes_bound(B, T), "gathered_mean": int(np.mean(gathered)),
                   "gathered_max": int(np.max(gathered))}

    exact = True
    for d in draws:
        out, starts, lengths = packed(d)
        hout, _, _ = hpacked(d)
        views = cb.load([srcs[f] for f in d], ctx=ctx)
        for (v, _), s, n in zip(views, starts.tolist(), lengths.tolist()):
            exact &= bool(n == v.shape[1] and torch.equal(out[:v.shape[0], s:s + n].view(torch.int32), v.view(torch.int32)))
        exact &= bool(torch.equal(out.view(torch.int32), hout.view(torch.int32)))

    def crop_args(d):
        files = d + [0] * (B - len(d))
        return files, [0] * len(d) + [idx[0].length] * (B - len(d))

    crop_draws = [crop_args(d) for d in draws]

    def device_ms(call, items):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for x in items:
            call(x)
        stop.record()
        stop.synchronize()
        return start.elapsed_time(stop) / len(items)

    for d, c in zip(draws[:3], crop_draws[:3]):
        packed(d, check=False)
        hpacked(d, check=False)
        crops(*c, check=False)
    ms = {"packed_device": [], "packed_host_corpus_device": [], "load_host": [], "crop_batch_padded_device": []}
    for r in range(args.rounds):
        ms["packed_device"].append(device_ms(lambda d: packed(d, check=False), draws))
        ms["packed_host_corpus_device"].append(device_ms(lambda d: hpacked(d, check=False), draws))
        per = []
        for d in draws[r % len(draws):][:args.load_calls]:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            cb.load([srcs[f] for f in d], ctx=ctx)
            torch.cuda.synchronize()
            per.append((time.perf_counter() - t0) * 1e3)
        ms["load_host"].append(float(np.median(per)))
        ms["crop_batch_padded_device"].append(device_ms(lambda c: crops(*c, check=False), crop_draws))
    info = gpu_info()
    kernels_us = {"device": profile_kernels(lambda d: packed(d, check=False), draws[:10], "excerpt_"),
                  "host_corpus": profile_kernels(lambda d: hpacked(d, check=False), draws[:10], "excerpt_")}
    samples = float(np.mean([sum(idx[f].length for f in d) for d in draws]))
    row = {"bench": "packed", "T": T, "draws": args.draws, "rounds": args.rounds, "files_per_draw_mean": float(np.mean([len(d) for d in draws])),
           "samples_per_draw_mean": samples, "bit_exact_vs_load_and_host_corpus": exact,
           "ms_per_call": {k: stats(v) for k, v in ms.items()}, "ms_rounds": {k: [round(x, 4) for x in v] for k, v in ms.items()},
           "packed_kernels_us_per_call": kernels_us, "bytes_bound": bytes_bound, "memory": memory, "gpu": info}
    line = json.dumps(row)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    del packed, hpacked, crops
    corpus = host = None
    ctx.close()


if __name__ == "__main__":
    main()
