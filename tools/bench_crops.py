"""Excerpts of FLAC files on the device: windowed channels-first batches and load_crops().

The workload of a training loader: C2-shaped files (16-bit stereo, 4096-sample frames) long enough to hold many
excerpts, and B = 256 excerpts of 176 400 samples (4 s at 44.1 kHz) at seeded random offsets.

1. Steady state over resident batches (Context.run_steps, CUDA events, bench_out_modes.py's method): `--units`
   windowed batches of such excerpts ([B * C, 176 400] rows, only the frames that overlap an excerpt, the first and last
   of each clipped), against channels batches of the same frames unclipped (two rows, every frame whole, back to back),
   timed alternately `--rounds` times.  Gsamples/s of decoded samples (every sample of every frame in the batch) and of
   stored samples (the windows' samples; unclipped: the same as decoded).
2. Whole load_crops() calls, the time split into planning and gather on the host, batch creation (upload, host CRC-16,
   graph instantiation), decode, and the copy into the [B, C, 176 400] tensor, with the phases of
   claxon_b200._decode_excerpts timed one by one (the call itself is timed too).

The card's name, power limit and SM clock are read in the same run.  One JSON line per part.

    python tools/bench_crops.py
    python tools/bench_crops.py --files 8 --frames 800 --units 4 --steps 200
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
from tools.bench_out_modes import gpu_info  # noqa: E402


def make_files(n_files, frames):
    out = []
    for i in range(n_files):
        cfg = synth.workload_config("c2", frames)
        cfg.seed = cfg.seed + 7919 * (i + 1)
        b = synth.generate(cfg)
        out.append(np.frombuffer(synth.make_file(b, 0, b.n_frames), np.uint8).copy())
    return out


def excerpts(idx, B, n, rng):
    files = rng.integers(0, len(idx), B)
    offsets = np.array([int(rng.integers(0, idx[f].length - n + 1)) for f in files])
    return files, offsets


def gather(idx, files, offsets, n, C_):
    """What load_crops() uploads: the frames overlapping each excerpt, their bytes, windows and columns."""
    chunks, parts, wins, at = [], [], [], 0
    for b, (fi, o) in enumerate(zip(files, offsets)):
        f = idx[int(fi)]
        sel, w, cols = cb.plan_range(f.descs, int(o), min(int(o) + n, f.length), column=0, row=b * C_, starts=f.starts)
        d = f.descs[sel]
        b0, b1 = int(d["byte_offset"][0]), int(d["byte_offset"][-1]) + int(d["byte_len"][-1])
        chunks.append(f.data[b0:b1])
        d["byte_offset"] = d["byte_offset"] - np.uint64(b0) + np.uint64(at)
        d["out_offset"] = cols
        parts.append(d)
        wins.append(w)
        at += b1 - b0
    return np.concatenate(chunks), np.concatenate(parts), np.concatenate(wins)


def part1(ctx, idx, args, rng):
    n, B = args.num_frames, args.batch
    win, full = [], []
    decoded = stored = 0
    for _ in range(args.units):
        files, offsets = excerpts(idx, B, n, rng)
        data, descs, w = gather(idx, files, offsets, n, 2)
        win.append(ctx.upload(data, descs, mode=cb.OUT_CHANNELS_F32, channels=2 * B, channel_stride=n, windows=w))
        d = descs.copy()
        bs = d["block_size"].astype(np.uint64)
        d["out_offset"] = np.concatenate([[0], np.cumsum(bs)[:-1]]).astype(np.uint64)
        full.append(ctx.upload(data, d, mode=cb.OUT_CHANNELS_F32, channels=2, channel_stride=int(bs.sum())))
        decoded += int((d["n_channels"].astype(np.int64) * d["block_size"]).sum())
        stored += int((d["n_channels"].astype(np.int64) * w["count"]).sum())
    ok = True
    for dev in win[:1] + full[:1]:
        dev.decode(0)
        ok &= bool((dev.results()["status"] == 0).all())
    for v in (win, full):
        ctx.run_steps(v, max(args.warmup, args.units), args.streams)
    ms = {"windowed": [], "unclipped": []}
    for _ in range(args.rounds):
        ms["windowed"].append(ctx.run_steps(win, args.steps, args.streams))
        ms["unclipped"].append(ctx.run_steps(full, args.steps, args.streams))
    info = gpu_info()
    rows = {}
    for k, v in ms.items():
        med = float(np.median(v))
        per_s = args.steps / args.units / (med * 1e-3)
        rows[k] = {"gsamples_decoded_per_s": round(decoded * per_s / 1e9, 3),
                   "gsamples_stored_per_s": round((stored if k == "windowed" else decoded) * per_s / 1e9, 3),
                   "ms_per_batch": round(med / args.steps, 4),
                   "spread": round((max(v) - min(v)) / med, 4), "ms_rounds": [round(x, 3) for x in v]}
    for dev in win + full:
        dev.close()
    return {"part": "steady_state", "batch": B, "num_frames": n, "units": args.units, "steps": args.steps,
            "streams": args.streams, "rounds": args.rounds, "frames_per_batch": int(descs.size),
            "decoded_samples_per_batch": decoded // args.units, "stored_samples_per_batch": stored // args.units,
            "all_ok": ok, "modes": rows, "gpu": info}


def part2(ctx, idx, args, rng):
    import torch
    n, B = args.num_frames, args.batch
    phases = {"plan_gather": [], "create": [], "decode": [], "copy": [], "load_crops_call": []}
    for it in range(args.calls + 1):
        files, offsets = excerpts(idx, B, n, rng)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        data, descs, w = gather(idx, files, offsets, n, 2)
        t1 = time.perf_counter()
        dev = ctx.upload(data, descs, mode=cb.OUT_CHANNELS_F32, channels=2 * B, channel_stride=n, windows=w)
        t2 = time.perf_counter()
        dev.decode(0)
        res = dev.results()
        t3 = time.perf_counter()
        out = torch.empty((B, 2, n), dtype=torch.float32, device="cuda")
        out.view(2 * B, n).copy_(dev.tensor())
        torch.cuda.current_stream().synchronize()
        t4 = time.perf_counter()
        dev.close()
        assert (res["status"] == 0).all()
        t5 = time.perf_counter()
        t, _ = cb.load_crops(idx, files, offsets, n, ctx=ctx)
        torch.cuda.synchronize()
        t6 = time.perf_counter()
        assert torch.equal(t, out)
        if it == 0:
            continue  # first call: allocator and module warm-up
        for k, v in zip(phases, (t1 - t0, t2 - t1, t3 - t2, t4 - t3, t6 - t5)):
            phases[k].append(v * 1e3)
    info = gpu_info()
    return {"part": "load_crops", "batch": B, "num_frames": n, "calls": args.calls,
            "ms_median": {k: round(float(np.median(v)), 3) for k, v in phases.items()},
            "ms_min": {k: round(float(np.min(v)), 3) for k, v in phases.items()},
            "output_gsamples_per_s": round(B * 2 * n / (np.median(phases["load_crops_call"]) * 1e-3) / 1e9, 3),
            "gpu": info}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--files", type=int, default=8)
    ap.add_argument("--frames", type=int, default=800, help="frames per file (4096 samples each)")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--num-frames", type=int, default=176400)
    ap.add_argument("--units", type=int, default=4, help="resident batches of part 1")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--streams", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10, help="load_crops calls of part 2")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    ctx = cb.Context(device=0, n_streams=args.streams)
    idx = cb.index(make_files(args.files, args.frames))
    rng = np.random.default_rng(2024)
    for fn in (part1, part2):
        line = json.dumps(fn(ctx, idx, args, rng))
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
