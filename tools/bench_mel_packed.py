"""Mel packed batches (Corpus.mel_packed) against the resampled packed batch alone, against that batch followed by
torchaudio's MelSpectrogram and a log per excerpt slice, and against mel_crops with one crop per file padded to the
longest file.

The workload of tools/bench_resampled_packed.py: 96 C2-shaped files (16-bit stereo, 4096-sample frames) of 1 to 30 s,
half at 44.1 kHz and half at 48 kHz; each draw is whole files in random order, as many as fill T = 300 s at R = 16 kHz
(4.8 M columns).  n_fft 400, hop 160, 128 HTK mels, log floor 1e-10.  Device time per call from CUDA events on torch's
stream around every draw, the arms alternated over `--rounds` rounds.  Peak device memory per arm: the memory its
creation took plus the peak allocated during one call.  A torch.profiler run gives mel_packed_kernel's and the planner's
own time per call, with bytes and FLOPs computed from shapes (as tools/bench_mel_crops.py counts them).  Every excerpt of
one draw is checked against tests/spec_mel.py (float64) of its slice of the resampled packed output.  The card's name,
power limit and SM clock are read in the same run.  One JSON line.

    python tools/bench_mel_packed.py
    python tools/bench_mel_packed.py --rounds 3 --seconds 120
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
from tests import spec_resample as SR  # noqa: E402
from tools.bench_corpus import stats  # noqa: E402
from tools.bench_out_modes import gpu_info  # noqa: E402
from tools.bench_resampled_crops import created, profile_kernels  # noqa: E402
from tools.bench_resampled_packed import draw, make_files  # noqa: E402


def main():
    import torch
    import torchaudio
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--files", type=int, default=96)
    ap.add_argument("--seconds", type=float, default=300.0)
    ap.add_argument("--rate", type=int, default=16000)
    ap.add_argument("--draws", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    R, n_fft, hop, n_mels, floor = args.rate, 400, 160, 128, 1e-10
    T = int(args.seconds * R)
    rng = np.random.default_rng(2026)
    srcs = make_files(args.files, rng)
    ctx = cb.Context(device=0)
    idx = cb.index(srcs)
    corpus = cb.Corpus(idx, ctx)
    draws = [draw(idx, T, R, rng) for _ in range(args.draws)]
    B = max(len(d) for d in draws)
    Lmax = max(SR.out_len(f.length, f.info.sample_rate, R) for f in idx.files)
    kw = dict(n_fft=n_fft, hop_length=hop, n_mels=n_mels, log_floor=floor)

    mel, mem_mel = created(lambda: corpus.mel_packed(B, T, R, **kw))
    packed, mem_packed = created(lambda: corpus.packed(B, T, sample_rate=R))
    ta, mem_ta = created(lambda: torchaudio.transforms.MelSpectrogram(R, n_fft=n_fft, hop_length=hop,
                                                                      n_mels=n_mels).cuda())
    crops, mem_crops = created(lambda: corpus.mel_crops(B, Lmax, R, **kw))

    call_m = lambda d: mel(d, check=False)  # noqa: E731
    call_p = lambda d: packed(d, check=False)  # noqa: E731
    call_c = lambda d: crops(d + [0] * (B - len(d)), [0] * B, check=False)  # noqa: E731

    def call_t(d):
        x, starts, lengths = packed(d, check=False)
        return [ta(x[:, s:s + n]).clamp_min(floor).log() for s, n in zip(starts.tolist(), lengths.tolist())]

    # correctness: every excerpt of the first draw against the float64 reference of its slice of the packed output
    x, s, n = call_p(draws[0])
    x, s, n = x.cpu().numpy(), s.cpu().numpy(), n.cpu().numpy()
    feats, starts, frames, _ = call_m(draws[0])
    feats, starts, frames = feats.cpu().numpy(), starts.cpu().numpy(), frames.cpu().numpy()
    worst_ratio = 0.0
    for b in range(len(draws[0])):
        seg = x[:, s[b]:s[b] + n[b]]
        ref = S.mel(seg, n_fft, hop, mel.window, mel.fbank, True, floor)
        delta = S.bound(seg, n_fft, hop, mel.window, mel.fbank, True)
        worst_ratio = max(worst_ratio, S.check(feats[:, :, starts[b]:starts[b] + frames[b]], ref, delta, floor))

    def peak_bytes(call):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        call(draws[0])
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    memory = {"mel_packed_batch": int(mem_mel) + peak_bytes(call_m),
              "resampled_packed_batch": int(mem_packed) + peak_bytes(call_p),
              "resampled_packed_batch_plus_torchaudio": int(mem_packed) + int(mem_ta) + peak_bytes(call_t),
              "mel_crops_padded_to_longest": int(mem_crops) + peak_bytes(call_c)}

    def device_ms(call, items):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for d in items:
            call(d)
        stop.record()
        stop.synchronize()
        return start.elapsed_time(stop) / len(items)

    arms = {"mel_packed_batch": call_m, "resampled_packed_batch": call_p,
            "resampled_packed_batch_plus_torchaudio": call_t, "mel_crops_padded_to_longest": call_c}
    for d in draws[:2]:
        for call in arms.values():
            call(d)
    ms = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, call in arms.items():
            ms[k].append(device_ms(call, draws))
    info = gpu_info()
    kernels = profile_kernels(call_m, draws, "mel_packed")
    mk = kernels.get("mel_packed_kernel")
    # mel_packed_kernel over the mean draw: each frame reads n_fft samples per row, every element of the features is
    # written, and each (row, frame) costs the FFT, the power and the mel sums
    C_, N = corpus.channels, n_fft // 2
    frames_per_call = float(np.mean([sum(1 + SR.out_len(idx[f].length, idx[f].info.sample_rate, R) // hop for f in d)
                                     for d in draws]))
    nz = int(sum(np.count_nonzero(mel.fbank[:, m]) for m in range(n_mels)))
    pairs = C_ * frames_per_call
    traffic = {"row_frame_pairs": int(pairs), "feature_columns": mel.stride,
               "bytes_read": int(pairs * n_fft * 4), "bytes_written": C_ * n_mels * mel.stride * 4,
               "flops": int(pairs * (5 * N * math.log2(N) + 12 * (N + 1) + 2 * nz)), "nonzero_weights": nz}
    if mk:
        traffic["mel_packed_kernel_GB_per_s"] = round((traffic["bytes_read"] + traffic["bytes_written"]) / (mk * 1e3), 1)
        traffic["mel_packed_kernel_GFLOP_per_s"] = round(traffic["flops"] / (mk * 1e3), 1)
        traffic["mel_packed_kernel_ns_per_row_frame"] = round(mk * 1e3 / pairs, 3)
    row = {"bench": "mel_packed", "T": T, "rate": R, "files": args.files, "file_rates": [44100, 48000],
           "files_per_draw": [len(d) for d in draws], "max_excerpts": B, "longest_file_at_rate": Lmax,
           "n_fft": n_fft, "hop": hop, "n_mels": n_mels, "log_floor": floor, "draws": args.draws,
           "rounds": args.rounds, "worst_error_to_bound_ratio": round(worst_ratio, 4),
           "ms_per_call": {k: stats(v) for k, v in ms.items()},
           "ms_rounds": {k: [round(v, 4) for v in vs] for k, vs in ms.items()},
           "kernels_us_per_call": kernels, "traffic": traffic, "peak_memory_bytes": memory, "gpu": info}
    line = json.dumps(row)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    del mel, packed, crops, ta
    corpus = None
    ctx.close()


if __name__ == "__main__":
    main()
