"""Resampled packed batches (Corpus.packed(..., sample_rate=R)) against a PackedBatch of the same source spans and
against load() plus torchaudio.functional.resample per file.

96 C2-shaped files (16-bit stereo, 4096-sample frames) of 1 to 30 s, half at 44.1 kHz and half at 48 kHz, made with
synth.make_file.  Each draw is whole files in random order, as many as fill T = 300 s at R = 16 kHz (4.8 M columns).
Two baselines: a PackedBatch at the corpus's rates of exactly the source spans (for whole files, the whole files: the
work the resampled batch runs before its filter kernel), and today's route, load() of the same files into CUDA tensors
followed by torchaudio.functional.resample of each file on the GPU.  Device time per call from CUDA events on torch's
stream around every draw, alternated over `--rounds` rounds (for load(), the events also take its host planning, which
the stream waits for).  A torch.profiler run gives resample_packed_kernel's own time per call and its bytes (source
samples staged, every output element written).  A few excerpts of one draw are checked against tests/spec_resample.py
(float64) of their files.  Memory from torch.cuda.mem_get_info around each batch's creation.  The card's name, power
limit and SM clock are read in the same run.  One JSON line.

    python tools/bench_resampled_packed.py
    python tools/bench_resampled_packed.py --rounds 3 --seconds 120
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import claxon_b200 as cb  # noqa: E402
from claxon_b200 import synth  # noqa: E402
from tests import spec_resample as S  # noqa: E402
from tools.bench_corpus import stats  # noqa: E402
from tools.bench_out_modes import gpu_info  # noqa: E402
from tools.bench_resampled_crops import created, profile_kernels  # noqa: E402


def make_files(n_files, rng):
    out = []
    for i in range(n_files):
        cfg = synth.workload_config("c2", int(rng.integers(11, 324)))  # 1 to 30 s of 4096-sample frames
        cfg.seed = cfg.seed + 7919 * (i + 1)
        cfg.sample_rate_code = 9 if i % 2 == 0 else 10  # 44.1 kHz, 48 kHz
        b = synth.generate(cfg)
        out.append(np.frombuffer(synth.make_file(b, 0, b.n_frames), np.uint8).copy())
    return out


def draw(idx, T, R, rng):
    """Whole files in random order while their columns at R fit in T."""
    files, at = [], 0
    for f in rng.permutation(len(idx)):
        nt = S.out_len(idx[int(f)].length, idx[int(f)].info.sample_rate, R)
        if at + nt > T:
            break
        files.append(int(f))
        at += (nt + 3) & ~3
    return files


def main():
    import torch
    import torchaudio.functional as F
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--files", type=int, default=96)
    ap.add_argument("--seconds", type=float, default=300.0)
    ap.add_argument("--rate", type=int, default=16000)
    ap.add_argument("--draws", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    R = args.rate
    T = int(args.seconds * R)
    rng = np.random.default_rng(2026)
    srcs = make_files(args.files, rng)
    ctx = cb.Context(device=0)
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, ctx)
    draws = [draw(idx, T, R, rng) for _ in range(args.draws)]
    B = max(len(d) for d in draws)
    T_plain = max(sum((idx[f].length + 3) & ~3 for f in d) for d in draws)

    resampled, mem_resampled = created(lambda: corpus.packed(B, T, sample_rate=R))
    packed, mem_packed = created(lambda: corpus.packed(B, T_plain, dtype=torch.float32))

    # correctness: a few excerpts of the first draw against the float64 reference of their whole files
    out, starts, lengths = resampled(draws[0])
    worst = 0.0
    for b in range(0, len(draws[0]), max(1, len(draws[0]) // 5)):
        f = draws[0][b]
        x = cb.load(srcs[f], ctx=ctx)[0].double().cpu().numpy()
        y = S.resample(x, idx[f].info.sample_rate, R)
        s, n = int(starts[b]), int(lengths[b])
        worst = max(worst, float(np.abs(out[:y.shape[0], s:s + n].double().cpu().numpy() - y).max()))

    def device_ms(call, items):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for x in items:
            call(x)
        stop.record()
        stop.synchronize()
        return start.elapsed_time(stop) / len(items)

    def today(d):
        views = cb.load([srcs[f] for f in d], ctx=ctx)
        return [F.resample(v, r, R) for v, r in views]

    call_r = lambda d: resampled(d, check=False)  # noqa: E731
    call_p = lambda d: packed(d, check=False)  # noqa: E731
    for d in draws[:2]:
        call_r(d)
        call_p(d)
        today(d)
    ms = {"resampled_packed_device": [], "packed_batch_source_spans_device": [], "load_plus_torchaudio_resample": []}
    for _ in range(args.rounds):
        ms["resampled_packed_device"].append(device_ms(call_r, draws))
        ms["packed_batch_source_spans_device"].append(device_ms(call_p, draws))
        ms["load_plus_torchaudio_resample"].append(device_ms(today, draws))
    info = gpu_info()
    kernels = profile_kernels(call_r, draws, "resample")
    # resample_packed_kernel's traffic: every source sample of every span staged once per row (tiles overlap by 2w + o),
    # every element of the [C, stride] output written once
    C_ = corpus.channels
    src_samples = float(np.mean([sum(idx[f].length for f in d) for d in draws])) * C_
    traffic = {"source_bytes_read": int(src_samples * 4), "output_bytes_written": C_ * resampled.stride * 4,
               "decoded_source_samples_per_call": int(src_samples)}
    rk = kernels.get("resample_packed_kernel")
    if rk:
        traffic["resample_packed_kernel_GB_per_s"] = round(
            (traffic["source_bytes_read"] + traffic["output_bytes_written"]) / (rk * 1e3), 1)
    row = {"bench": "resampled_packed", "T": T, "rate": R, "files": args.files, "file_rates": [44100, 48000],
           "files_per_draw": [len(d) for d in draws], "max_excerpts": B,
           "source_columns": corpus.resample_packed_source_bound(B, T, R), "draws": args.draws, "rounds": args.rounds,
           "max_abs_err_vs_float64_reference": worst,
           "ms_per_call": {k: stats(v) for k, v in ms.items()},
           "ms_rounds": {k: [round(x, 4) for x in v] for k, v in ms.items()},
           "resample_kernels_us_per_call": kernels, "traffic": traffic,
           "memory_bytes": {"resampled_packed_batch": int(mem_resampled), "packed_batch_source_spans": int(mem_packed)},
           "gpu": info}
    line = json.dumps(row)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    del resampled, packed, out, starts, lengths
    corpus = None
    ctx.close()


if __name__ == "__main__":
    main()
