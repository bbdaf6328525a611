"""Normalised mel batches (normalize="whisper" / "per_feature") against the unnormalised batch and against the
unnormalised batch's data followed by the same normalisation in torch on the GPU.

Crops: the files of tools/bench_resampled_crops.py (C2-shaped, 16-bit stereo, 20 to 40 s, half at 44.1 kHz and half at
48 kHz); each draw is B = 256 crops of 30 s at 16 kHz from random files and offsets (past the file's end reads zeros,
as Whisper pads), n_fft 400, hop 160, 80 Slaney mels with Slaney norm, log floor 1e-10: Whisper's front end.  Arms:
  * whisper_mel_crop_batch: mel_crops(..., normalize="whisper");
  * log_mel_crop_batch: the same without normalize (3001 frames, no map);
  * resampled_crop_batch_plus_torch_whisper: the resampled crop batch, then Whisper's features in torch on the GPU
    (torch.stft, the batch's filterbank, log10 of the clamp, the last frame dropped, max - 8, (l + 4) / 4): what
    transformers.WhisperFeatureExtractor's torch path does on a CUDA device.
WhisperFeatureExtractor's default path on the CPU is timed on a few rows, per crop row.
Packed: the workload of tools/bench_mel_packed.py (96 files of 1 to 30 s at 44.1 / 48 kHz, whole files filling 300 s at
16 kHz, n_fft 400, hop 160, 128 HTK mels, log floor 1e-10).  Arms: mel_packed(normalize="per_feature"), mel_packed
alone, and mel_packed followed by a torch loop that normalises each excerpt's slice (mean, unbiased std, NaN to 0,
(x - mean) / (std + 1e-5)).

Device time per call from CUDA events on torch's stream around every draw, the arms alternated over `--rounds`
rounds.  A torch.profiler run of its own gives mel_norm_kernel's time per call; its bytes are one read and one write of
the normalised features (the traffic the pass needs; its second and third walks are meant to hit L1 / L2), computed
from shapes.  Each normalised arm is checked against its torch arm on one draw.  The card's name, power limit and SM
clock are read in the same run.  One JSON line.

    python tools/bench_mel_norm.py
    python tools/bench_mel_norm.py --rounds 3 --batch 64
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import claxon_b200 as cb  # noqa: E402
from tests import spec_resample as SR  # noqa: E402
from tools.bench_corpus import profile_kernels, stats  # noqa: E402
from tools.bench_out_modes import gpu_info  # noqa: E402
from tools.bench_resampled_crops import make_files as crop_files  # noqa: E402
from tools.bench_resampled_packed import draw as packed_draw, make_files as packed_files  # noqa: E402


def device_ms(call, items):
    import torch
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for d in items:
        call(d)
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / len(items)


def alternate(arms, draws, rounds):
    for d in draws[:2]:
        for call in arms.values():
            call(d)
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, call in arms.items():
            ms[k].append(device_ms(call, draws))
    return ms


def crops_part(ctx, args, rng):
    import torch
    B, R, L = args.batch, 16000, 480000
    n_fft, hop, n_mels, floor = 400, 160, 80, 1e-10
    idx = cb.index(crop_files(args.files, rng))
    corpus = cb.Corpus(idx, ctx)
    nt = [SR.out_len(f.length, f.info.sample_rate, R) for f in idx.files]
    draws = []
    for _ in range(args.draws):
        files = [int(f) for f in rng.integers(0, len(idx), B)]
        draws.append((files, [int(rng.integers(0, max(1, nt[f] - L // 2))) for f in files]))
    kw = dict(n_fft=n_fft, hop_length=hop, n_mels=n_mels, mel_scale="slaney", norm="slaney", log_floor=floor)
    whisper = corpus.mel_crops(B, L, R, normalize="whisper", **kw)
    plain = corpus.mel_crops(B, L, R, **kw)
    crops = corpus.crops(B, L, sample_rate=R)
    window = torch.hann_window(n_fft, device="cuda")
    filters = torch.from_numpy(whisper.fbank.T.copy()).cuda()  # [n_mels, n_fft // 2 + 1]

    def torch_whisper(x):  # x [B, C, L] -> [B, C, n_mels, F - 1]
        st = torch.stft(x.reshape(-1, L), n_fft, hop, window=window, return_complex=True)
        mag = st[..., :-1].abs() ** 2
        l = torch.clamp(filters @ mag, min=floor).log10()
        l = torch.maximum(l, l.amax(dim=(-2, -1), keepdim=True) - 8.0)
        return ((l + 4.0) / 4.0).reshape(B, -1, n_mels, mag.shape[-1])

    call_w = lambda d: whisper(*d, check=False)  # noqa: E731
    call_p = lambda d: plain(*d, check=False)  # noqa: E731
    call_t = lambda d: torch_whisper(crops(*d, check=False)[0])  # noqa: E731
    vs_torch = float((call_w(draws[0])[0] - call_t(draws[0])).abs().max())
    ms = alternate({"whisper_mel_crop_batch": call_w, "log_mel_crop_batch": call_p,
                    "resampled_crop_batch_plus_torch_whisper": call_t}, draws, args.rounds)
    # WhisperFeatureExtractor (its default path, on the CPU) on a few crop rows
    fe_ms = None
    try:
        import transformers
        fe = transformers.WhisperFeatureExtractor(feature_size=n_mels)
        x = crops(*draws[0], check=False)[0][:4, 0].cpu().numpy()
        fe(x[0], sampling_rate=R, return_tensors="np")
        t0 = time.perf_counter()
        for row in x:
            fe(row, sampling_rate=R, return_tensors="np")
        fe_ms = (time.perf_counter() - t0) * 1e3 / len(x)
    except ImportError:
        pass
    us = profile_kernels(call_w, draws, "mel_")
    elems = B * corpus.channels * n_mels * whisper.n_frames
    out = {"B": B, "L": L, "rate": R, "n_mels": n_mels, "frames": whisper.n_frames, "files": args.files,
           "max_abs_diff_vs_torch_whisper": vs_torch, "ms_per_call": {k: stats(v) for k, v in ms.items()},
           "ms_rounds": {k: [round(x, 4) for x in v] for k, v in ms.items()}, "kernels_us_per_call": us,
           "whisper_feature_extractor_cpu_ms_per_crop_row": None if fe_ms is None else round(fe_ms, 2)}
    mk = us.get("mel_norm_kernel")
    if mk:
        out["mel_norm_kernel_bytes"] = 2 * 4 * elems
        out["mel_norm_kernel_GB_per_s"] = round(2 * 4 * elems / (mk * 1e3), 1)
    del whisper, plain, crops
    return out


def packed_part(ctx, args, rng):
    import torch
    R, T = 16000, int(300 * 16000)
    n_fft, hop, n_mels, floor = 400, 160, 128, 1e-10
    idx = cb.index(packed_files(96, rng))
    corpus = cb.Corpus(idx, ctx)
    draws = [packed_draw(idx, T, R, rng) for _ in range(args.draws)]
    B = max(len(d) for d in draws)
    kw = dict(n_fft=n_fft, hop_length=hop, n_mels=n_mels, log_floor=floor)
    norm = corpus.mel_packed(B, T, R, normalize="per_feature", **kw)
    plain = corpus.mel_packed(B, T, R, **kw)

    def torch_norm(d):
        feats, starts, frames, _ = plain(d, check=False)
        out = []
        for s, F in zip(starts.tolist(), frames.tolist()):
            seg = feats[:, :, s:s + F]
            mu = seg.mean(-1, keepdim=True)
            sd = torch.nan_to_num(seg.std(-1, keepdim=True), nan=0.0)
            out.append((seg - mu) / (sd + 1e-5))
        return out

    call_n = lambda d: norm(d, check=False)  # noqa: E731
    call_p = lambda d: plain(d, check=False)  # noqa: E731
    feats, starts, frames, _ = call_n(draws[0])
    ref = torch_norm(draws[0])
    vs_torch = max(float((feats[:, :, s:s + F] - r).abs().max()) for s, F, r in zip(starts.tolist(), frames.tolist(), ref))
    ms = alternate({"per_feature_mel_packed_batch": call_n, "mel_packed_batch": call_p,
                    "mel_packed_batch_plus_torch_per_slice": torch_norm}, draws, args.rounds)
    us = profile_kernels(call_n, draws, "mel_")
    frames_per_call = float(np.mean([sum(1 + SR.out_len(idx[f].length, idx[f].info.sample_rate, R) // hop for f in d)
                                     for d in draws]))
    elems = corpus.channels * n_mels * frames_per_call
    out = {"T": T, "rate": R, "n_mels": n_mels, "max_excerpts": B, "files_per_draw": [len(d) for d in draws],
           "frames_per_call": frames_per_call, "max_abs_diff_vs_torch_per_slice": vs_torch,
           "ms_per_call": {k: stats(v) for k, v in ms.items()},
           "ms_rounds": {k: [round(x, 4) for x in v] for k, v in ms.items()}, "kernels_us_per_call": us}
    mk = us.get("mel_norm_kernel")
    if mk:
        out["mel_norm_kernel_bytes"] = int(2 * 4 * elems)
        out["mel_norm_kernel_GB_per_s"] = round(2 * 4 * elems / (mk * 1e3), 1)
    del norm, plain
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--files", type=int, default=64)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--draws", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    rng = np.random.default_rng(2026)
    ctx = cb.Context(device=0)
    row = {"bench": "mel_norm", "draws": args.draws, "rounds": args.rounds,
           "crops": crops_part(ctx, args, rng), "packed": packed_part(ctx, args, rng), "gpu": gpu_info()}
    line = json.dumps(row)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
