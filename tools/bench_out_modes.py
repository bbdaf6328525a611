"""Steady-state throughput of device-resident batches per output mode (planar i32 / interleaved i32 / i16 /
channels-first i32 / f32).

The method of bench.py's steady state: `--units` resident batches of one workload, every one decoded once before
timing, then `--steps` steps round-robin over `--streams` streams through Context.run_steps (CUDA events).  The
modes are timed alternately in one process, `--rounds` times each; the median and the spread (max - min over the
median) are reported per mode, with the output bytes per sample, whether one batch per mode equals the generator's
PCM byte for byte, and the card's name, power limit and SM clock read in the same run.  A channels-first batch holds
one unit as rows of its samples per channel, the frames' columns packed back to back.

    python tools/bench_out_modes.py                      # C2, C3, C4: planar, their interleaved modes, channels i32 / f32
    python tools/bench_out_modes.py --workloads c2 --steps 1000
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import claxon_b200 as cb  # noqa: E402
from claxon_b200 import synth  # noqa: E402

CH_I32, CH_F32 = cb.OUT_CHANNELS_I32, cb.OUT_CHANNELS_F32
ESIZE = {cb.OUT_PLANAR_I32: 4, cb.OUT_INTERLEAVED_I32: 4, cb.OUT_INTERLEAVED_I16: 2, CH_I32: 4, CH_F32: 4}
NAMES = {cb.OUT_PLANAR_I32: "planar_i32", cb.OUT_INTERLEAVED_I32: "interleaved_i32", cb.OUT_INTERLEAVED_I16: "interleaved_i16",
         CH_I32: "channels_i32", CH_F32: "channels_f32"}
PLAN = {  # workload -> (frames per unit, units, modes)
    "c2": (1024, 128, (cb.OUT_PLANAR_I32, cb.OUT_INTERLEAVED_I16, cb.OUT_INTERLEAVED_I32, CH_I32, CH_F32)),
    "c3": (8192, 8, (cb.OUT_PLANAR_I32, cb.OUT_INTERLEAVED_I32, CH_I32, CH_F32)),
    "c4": (1100, 128, (cb.OUT_PLANAR_I32, cb.OUT_INTERLEAVED_I16, CH_I32, CH_F32)),
}


def channels_layout(descs):
    """(descs with out_offset = column, rows, stride): the unit's frames back to back along each row."""
    d = descs.copy()
    bs = d["block_size"].astype(np.uint64)
    d["out_offset"] = np.concatenate([[0], np.cumsum(bs)[:-1]]).astype(np.uint64)
    return d, int(d["n_channels"].max()), int(bs.sum())


def upload(ctx, b, descs, out_elems, mode):
    if mode in (CH_I32, CH_F32):
        d, rows, stride = channels_layout(descs)
        assert rows * stride == out_elems  # one shape per unit: every element is a sample
        return ctx.upload(b.data, d, mode=mode, channels=rows, channel_stride=stride)
    return ctx.upload(b.data, descs, out_elems, mode=mode)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        row = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in row.split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"nvidia-smi": "unavailable"}


def expected_bytes(b, descs, out_elems, mode):
    """The generator's PCM in the mode's layout (planar i32, or interleaved little-endian elements)."""
    if mode == cb.OUT_PLANAR_I32:
        return b.pcm[:out_elems].astype("<i4").tobytes()
    if mode in (CH_I32, CH_F32):
        rows = np.concatenate([b.pcm[int(b.pcm_offsets[i]):int(b.pcm_offsets[i + 1])].reshape(int(descs[i]["n_channels"]), -1)
                               for i in range(b.n_frames)], axis=1)
        if mode == CH_F32:
            rows = rows.astype(np.float32) * np.float32(2.0 ** -(int(descs[0]["bits_per_sample"]) - 1))  # one width per workload
        return rows.astype("<f4" if mode == CH_F32 else "<i4").tobytes()
    parts = []
    for i in range(b.n_frames):
        nch = int(descs[i]["n_channels"])
        parts.append(synth.interleaved_le_bytes(b.pcm[int(b.pcm_offsets[i]):int(b.pcm_offsets[i + 1])], nch, 8 * ESIZE[mode]))
    return b"".join(parts)


def run_workload(ctx, name, units, steps, streams, rounds, warmup):
    frames, default_units, modes = PLAN[name]
    units = units or default_units
    batches = {m: [] for m in modes}
    samples = 0
    first = None
    for u in range(units):
        cfg = synth.workload_config(name, frames)
        cfg.seed = cfg.seed + 1000003 * u  # bench.py's units: same shape, own content
        b = synth.generate(cfg)
        descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
        assert out_elems == b.n_samples  # frames back to back: every output byte is a sample
        for m in modes:
            batches[m].append(upload(ctx, b, descs, out_elems, m))
        samples += b.n_samples
        if u == 0:
            first = (b, descs, out_elems)
    exact = {}
    b, descs, out_elems = first
    for m in modes:
        dev = batches[m][0]
        dev.decode(0)
        out, res = dev.read()
        got = out.reshape(-1).view(np.uint8)[:out_elems * ESIZE[m]].tobytes()
        exact[NAMES[m]] = bool((res["status"] == 0).all()) and got == expected_bytes(b, descs, out_elems, m)
    for m in modes:  # every batch once, every graph warm
        ctx.run_steps(batches[m], max(warmup, units), streams)
    ms = {m: [] for m in modes}
    for _ in range(rounds):
        for m in modes:
            ms[m].append(ctx.run_steps(batches[m], steps, streams))
    info = gpu_info()  # read in the same run, right after the timed region
    per_step = samples / units
    rows = {}
    for m in modes:
        med = float(np.median(ms[m]))
        rows[NAMES[m]] = {
            "msamples_per_s": round(per_step * steps / (med * 1e-3) / 1e6, 1),
            "ms_median": round(med, 3),
            "spread": round((max(ms[m]) - min(ms[m])) / med, 4),
            "ms_rounds": [round(x, 3) for x in ms[m]],
            "out_bytes_per_sample": ESIZE[m],
            "bit_exact": exact[NAMES[m]],
        }
    for v in batches.values():
        for d in v:
            d.close()
    return {"workload": name, "frames_per_unit": frames, "units": units, "steps": steps, "streams": streams,
            "rounds": rounds, "modes": rows, "gpu": info}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", default="c2,c3,c4")
    ap.add_argument("--units", type=int, default=0, help="resident batches per workload (0: the plan's)")
    ap.add_argument("--steps", type=int, default=4000)
    ap.add_argument("--streams", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    ctx = cb.Context(device=0, n_streams=args.streams)
    for name in args.workloads.split(","):
        line = json.dumps(run_workload(ctx, name, args.units, args.steps, args.streams, args.rounds, args.warmup))
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
