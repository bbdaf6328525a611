"""Resampled crop batches (Corpus.crops(..., sample_rate=R)) against a CropBatch of the same source spans.

C2-shaped files (16-bit stereo, 4096-sample frames) of 20 to 40 s, half at 44.1 kHz and half at 48 kHz, made with
synth.make_file.  Each draw is B = 256 crops of L = 10 s at R = 16 kHz (160 000 samples) from random files and offsets.
Two baselines decode the same source spans without the filter: a CropBatch at the corpus's rates whose crops start at
the spans (num_frames = the largest source bound, so its crops reach a little past the shorter spans), and a
PackedBatch of exactly the spans, which is the work the resampled batch runs before its filter kernel.
A few crops of one draw are checked against tests/spec_resample.py (float64) applied to load() of their files.  Then,
alternated over `--rounds` rounds, device time per call from CUDA events on torch's stream around every draw.  A
torch.profiler run gives resample_kernel's own time per call and its bytes (source samples staged, outputs written)
over that time.  Memory is taken from torch.cuda.mem_get_info around each batch's creation.  The card's name, power
limit and SM clock are read in the same run.  One JSON line.

    python tools/bench_resampled_crops.py
    python tools/bench_resampled_crops.py --rounds 3 --batch 64
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
from tools.bench_corpus import profile_kernels, stats  # noqa: E402
from tools.bench_out_modes import gpu_info  # noqa: E402


def make_files(n_files, rng):
    out = []
    for i in range(n_files):
        cfg = synth.workload_config("c2", int(rng.integers(216, 431)))  # 20 to 40 s of 4096-sample frames
        cfg.seed = cfg.seed + 7919 * (i + 1)
        cfg.sample_rate_code = 9 if i % 2 == 0 else 10  # 44.1 kHz, 48 kHz
        b = synth.generate(cfg)
        out.append(np.frombuffer(synth.make_file(b, 0, b.n_frames), np.uint8).copy())
    return out


def draw(idx, B, L, R, rng):
    files = rng.integers(0, len(idx), B)
    offs = [int(rng.integers(0, S.out_len(idx[int(f)].length, idx[int(f)].info.sample_rate, R) - L + 1)) for f in files]
    spans = [S.source_span(idx[int(f)].length, idx[int(f)].info.sample_rate, R, o, L) for f, o in zip(files, offs)]
    return [int(f) for f in files], offs, [lo for lo, _ in spans], [hi - lo for lo, hi in spans]


def created(make):
    """(batch, device bytes its creation took)."""
    import torch
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    batch = make()
    torch.cuda.synchronize()
    return batch, free0 - torch.cuda.mem_get_info()[0]


def main():
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--files", type=int, default=64)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--rate", type=int, default=16000)
    ap.add_argument("--draws", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    B, R = args.batch, args.rate
    L = int(args.seconds * R)
    rng = np.random.default_rng(2026)
    srcs = make_files(args.files, rng)
    ctx = cb.Context(device=0)
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, ctx)
    draws = [draw(idx, B, L, R, rng) for _ in range(args.draws)]
    src_L = corpus.resample_source_bound(L, R)

    resampled, mem_resampled = created(lambda: corpus.crops(B, L, sample_rate=R))
    crops, mem_crops = created(lambda: corpus.crops(B, src_L, dtype=torch.float32))
    packed, mem_packed = created(lambda: corpus.packed(B, B * ((src_L + 3) & ~3), dtype=torch.float32))

    # correctness: a few crops of the first draw against the float64 reference of their whole files
    files, offs, los, lens = draws[0]
    out, lengths = resampled(files, offs)
    worst = 0.0
    for b in range(0, B, max(1, B // 6)):
        x = cb.load(srcs[files[b]], ctx=ctx)[0].double().cpu().numpy()
        y = S.resample(x, idx[files[b]].info.sample_rate, R)[:, offs[b]:offs[b] + L]
        worst = max(worst, float(np.abs(out[b, :y.shape[0], :y.shape[1]].double().cpu().numpy() - y).max()))

    def device_ms(call, items):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for x in items:
            call(x)
        stop.record()
        stop.synchronize()
        return start.elapsed_time(stop) / len(items)

    call_r = lambda d: resampled(d[0], d[1], check=False)  # noqa: E731
    call_c = lambda d: crops(d[0], d[2], check=False)  # noqa: E731
    call_p = lambda d: packed(d[0], d[2], d[3], check=False)  # noqa: E731
    for d in draws[:2]:
        call_r(d)
        call_c(d)
        call_p(d)
    ms = {"resampled_device": [], "crop_batch_source_spans_device": [], "packed_batch_source_spans_device": []}
    for _ in range(args.rounds):
        ms["resampled_device"].append(device_ms(call_r, draws))
        ms["crop_batch_source_spans_device"].append(device_ms(call_c, draws))
        ms["packed_batch_source_spans_device"].append(device_ms(call_p, draws))
    info = gpu_info()
    kernels = profile_kernels(call_r, draws, "resample")
    # resample_kernel's traffic: every source sample of every span staged once per row (tiles overlap by 2w + o), every
    # output element written once
    C_ = corpus.channels
    src_samples = float(np.mean([sum(d[3]) for d in draws])) * C_
    traffic = {"source_bytes_read": int(src_samples * 4), "output_bytes_written": B * C_ * L * 4,
               "decoded_source_samples_per_call": int(src_samples)}
    rk = kernels.get("resample_kernel")
    if rk:
        traffic["resample_kernel_GB_per_s"] = round((traffic["source_bytes_read"] + traffic["output_bytes_written"]) / (rk * 1e3), 1)
    row = {"bench": "resampled_crops", "B": B, "L": L, "rate": R, "files": args.files, "file_rates": [44100, 48000],
           "source_bound": src_L, "draws": args.draws, "rounds": args.rounds,
           "max_abs_err_vs_float64_reference": worst,
           "ms_per_call": {k: stats(v) for k, v in ms.items()}, "ms_rounds": {k: [round(x, 4) for x in v] for k, v in ms.items()},
           "resample_kernels_us_per_call": kernels, "traffic": traffic,
           "memory_bytes": {"resampled_batch": int(mem_resampled), "crop_batch_source_spans": int(mem_crops),
                            "packed_batch_source_spans": int(mem_packed)}, "gpu": info}
    line = json.dumps(row)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    del resampled, crops, packed, out, lengths
    corpus = None
    ctx.close()


if __name__ == "__main__":
    main()
