"""Mel crop batches (Corpus.mel_crops) against a resampled crop batch alone and against a resampled crop batch followed
by torchaudio's MelSpectrogram and a log on the GPU.

The workload of bench_resampled_crops.py: C2-shaped files (16-bit stereo, 4096-sample frames) of 20 to 40 s, half at
44.1 kHz and half at 48 kHz; each draw is B = 256 crops of 10 s at 16 kHz from random files and offsets.  The features
are Whisper-sized: n_fft 400, hop 160, 128 mels (HTK), ln(max(mel, 1e-10)).  Three arms, alternated over `--rounds`
rounds, device time per call from CUDA events on torch's stream around every draw: the mel crop batch, the resampled
crop batch alone, and the resampled crop batch + torchaudio.transforms.MelSpectrogram(...).cuda() + clamp_min().log().
Peak device memory of each arm: torch.cuda.mem_get_info around the batch's creation, plus the torch allocator's peak
during one call.  A torch.profiler run gives mel_kernel's time per call; its traffic (the inner output read once, the
features written once) and FLOPs (the FFTs at 5 N log2 N per N-point complex FFT, the split and power, the mel sums
over the non-zero weights) are computed from shapes.  Four crops of one draw are checked against tests/spec_mel.py
(float64) applied to the resampled crop batch's output, and the whole draw against torchaudio's features.  The card's
name, power limit and SM clock are read in the same run.  One JSON line.

    python tools/bench_mel_crops.py
    python tools/bench_mel_crops.py --rounds 3 --batch 64
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import claxon_b200 as cb  # noqa: E402
from tests import spec_mel as S  # noqa: E402
from tools.bench_corpus import stats  # noqa: E402
from tools.bench_out_modes import gpu_info  # noqa: E402
from tools.bench_resampled_crops import created, draw, make_files, profile_kernels  # noqa: E402


def main():
    import torch
    import torchaudio
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
    n_fft, hop, n_mels, floor = 400, 160, 128, 1e-10
    rng = np.random.default_rng(2026)
    srcs = make_files(args.files, rng)
    ctx = cb.Context(device=0)
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, ctx)
    draws = [draw(idx, B, L, R, rng)[:2] for _ in range(args.draws)]

    mel, mem_mel = created(lambda: corpus.mel_crops(B, L, R, n_fft=n_fft, hop_length=hop, n_mels=n_mels, log_floor=floor))
    crops, mem_crops = created(lambda: corpus.crops(B, L, sample_rate=R))
    ta, mem_ta = created(lambda: torchaudio.transforms.MelSpectrogram(R, n_fft=n_fft, hop_length=hop, n_mels=n_mels).cuda())

    call_m = lambda d: mel(d[0], d[1], check=False)  # noqa: E731
    call_c = lambda d: crops(d[0], d[1], check=False)  # noqa: E731

    def call_t(d):
        x, _ = crops(d[0], d[1], check=False)
        return ta(x).clamp_min(floor).log()

    # correctness: four crops against the float64 reference of the crop output, the draw against torchaudio's features
    files, offs = draws[0]
    x = call_c(draws[0])[0].cpu().numpy()
    feats = call_m(draws[0])[0].cpu().numpy()
    rows = [0, B // 3, B // 2, B - 1]
    ref = S.mel(x[rows], n_fft, hop, mel.window, mel.fbank, True, floor)
    delta = S.bound(x[rows], n_fft, hop, mel.window, mel.fbank, True)
    worst_ratio = S.check(feats[rows], ref, delta, floor)
    ta_feats = call_t(draws[0]).cpu().numpy()
    vs_ta = float(np.abs(ta_feats - feats).max())

    def peak_bytes(call):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        call(draws[0])
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    memory = {"mel_crop_batch": int(mem_mel) + peak_bytes(call_m),
              "resampled_crop_batch": int(mem_crops) + peak_bytes(call_c),
              "resampled_crop_batch_plus_torchaudio": int(mem_crops) + int(mem_ta) + peak_bytes(call_t)}

    def device_ms(call, items):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for d in items:
            call(d)
        stop.record()
        stop.synchronize()
        return start.elapsed_time(stop) / len(items)

    arms = {"mel_crop_batch": call_m, "resampled_crop_batch": call_c, "resampled_crop_batch_plus_torchaudio": call_t}
    for d in draws[:2]:
        for call in arms.values():
            call(d)
    ms = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, call in arms.items():
            ms[k].append(device_ms(call, draws))
    info = gpu_info()
    kernels = profile_kernels(call_m, draws, "_kernel")
    mk = kernels.get("mel_kernel")
    rows_, F, N = B * corpus.channels, mel.n_frames, n_fft // 2
    nz = int(sum(np.count_nonzero(mel.fbank[:, m]) for m in range(n_mels)))
    traffic = {"bytes_read": rows_ * L * 4, "bytes_written": rows_ * n_mels * F * 4,
               "flops": int(rows_ * F * (5 * N * math.log2(N) + 12 * (N + 1) + 2 * nz)), "nonzero_weights": nz}
    if mk:
        traffic["mel_kernel_GB_per_s"] = round((traffic["bytes_read"] + traffic["bytes_written"]) / (mk * 1e3), 1)
        traffic["mel_kernel_GFLOP_per_s"] = round(traffic["flops"] / (mk * 1e3), 1)
    row = {"bench": "mel_crops", "B": B, "L": L, "rate": R, "files": args.files, "file_rates": [44100, 48000],
           "n_fft": n_fft, "hop": hop, "n_mels": n_mels, "log_floor": floor, "frames": F, "draws": args.draws,
           "rounds": args.rounds, "worst_error_to_bound_ratio": round(worst_ratio, 4),
           "max_abs_diff_vs_torchaudio_log": vs_ta,
           "ms_per_call": {k: stats(v) for k, v in ms.items()}, "ms_rounds": {k: [round(x, 4) for x in v] for k, v in ms.items()},
           "kernels_us_per_call": kernels, "traffic": traffic, "peak_memory_bytes": memory, "gpu": info}
    line = json.dumps(row)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    del mel, crops, ta
    corpus = None
    ctx.close()


if __name__ == "__main__":
    main()
