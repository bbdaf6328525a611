"""The resampler and mel kernels element by element, on designed signals (-m gpu).

Resampler.  A linear kernel is described by its impulse responses.  Files of zeros with impulses of 2^(bps - 2) (x =
0.5 exactly), spaced more than 2w + o apart and stepping through the residues mod o, give outputs that each see one
impulse or none: exactly f32(h[ph, k]) / 2, within 2^-25 |h| of tests/spec_resample.py's tap, or exactly 0
(tests/spec_signal.py).  So every tap of every phase lands where it should, through crop batches (responses cut by crop
starts and ends and by tile boundaries, one batch of more than 65 535 crops) and resampled packed batches (many short
excerpts of different rates in one tile).  Full-scale noise files are held to the FIR's per-element bound.

Mel.  The batch's window and filterbank are replaced (claxon_b200._mel_tables, which both batch kinds call) by a window
with zeros inside it and slices of the identity of at most 512 columns, so the features are |X_t[k]|^2 itself, bin by
bin, 0 and n_fft / 2 included, for every n_fft the batches accept, both center modes, crop and packed batches, with F
past the tile.  Each bin is held to spec_signal.bin_bound; silence gives exactly 0.  Non-triangular filterbanks (edge
bins, negative weights, an empty column, a column over every bin, zeros inside a band) are checked with and without the
log.
"""
import math

import numpy as np
import pytest

import claxon_b200 as cb
from tests import pcm_flac as P
from tests import spec_mel as SM
from tests import spec_resample as SR
from tests import spec_signal as S
from tests.test_mel_host import supported

gpu = pytest.mark.gpu
WORST = {}


def note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), ratio)


@pytest.fixture(scope="module")
def rctx():
    c = cb.Context(device=0)
    yield c
    c.close()


def r4(v):
    return (v + 3) & ~3


# --------------------------------------------------------------------------- signals

def impulse_pcm(r, R, C_, bps, seed):
    """Impulses of +-2^(bps - 2) every S > 2w + o samples, gcd(S, o) = 1 (at most 48 a channel once o is large), each
    channel shifted; channel 0 also at samples 0 and N - 1, channel 1 % C at 1 and N - 2."""
    o, _, _, w = SR.params(r, R)
    K = 2 * w + o
    S_ = K + 1
    while math.gcd(S_, o) != 1:
        S_ += 1
    n_imp = min(max(o, 64), 48 if o > 1000 else 1 << 30)
    N = (n_imp + 1) * S_ + 7 * C_ + K + 3
    amp = 1 << (bps - 2)
    sign = np.random.default_rng(seed).choice([-1, 1], (C_, n_imp))
    pcm = np.zeros((C_, N), np.int64)
    for c in range(C_):
        pcm[c, S_ + 7 * c + S_ * np.arange(n_imp)] = amp * sign[c]
    pcm[0, [0, N - 1]] = amp
    pcm[1 % C_, [1, N - 2]] = -amp
    return pcm


def noise_pcm(r, R, C_, bps, seed):
    o, _, _, w = SR.params(r, R)
    N = 3 * (2 * w + o) + 501
    return np.random.default_rng(seed).integers(-(1 << (bps - 1)), 1 << (bps - 1), (C_, N))


# target R: (source rate, channels, bps) of its impulse files; each rate also has a noise file
RESAMPLE_CASES = {
    16000: [(48000, 4, 16), (44100, 2, 24), (22050, 1, 12), (16000, 2, 16)],
    48000: [(16000, 4, 20)],
    44100: [(8000, 2, 8)],
    1000: [(96000, 2, 16)],
    50: [(96000, 1, 24)],
}
_cache = {}


class RateCorpus:
    """The impulse and noise files of one target rate, their float64 signals and each file's reference at R."""

    def __init__(self, R, ctx):
        self.R = R
        pcms, self.rates, self.bps = [], [], []
        for i, (r, C_, bps) in enumerate(RESAMPLE_CASES[R]):
            pcms += [impulse_pcm(r, R, C_, bps, i), noise_pcm(r, R, 2, 16, 100 + i)]
            self.rates += [r, r]
            self.bps += [bps, 16]
        self.kind = ["impulse", "noise"] * (len(pcms) // 2)
        self.x = [p / float(1 << (b - 1)) for p, b in zip(pcms, self.bps)]
        bs = [128 if k == "impulse" else 1024 for k in self.kind]
        self.idx = cb.index([P.flac_from_pcm(p, b, r, s) for p, b, r, s in zip(pcms, self.bps, self.rates, bs)])
        self.corpus = cb.Corpus(self.idx, ctx)
        self.nt = [SR.out_len(x.shape[1], r, R) for x, r in zip(self.x, self.rates)]
        self.ref = [S.fir_ref_bound(x, r, R) for x, r in zip(self.x, self.rates)]
        # resample_tables' tile: halved from 1024 until every rate's staged span fits 8192 samples (32 at least)
        self.tile = 1024
        for r in set(self.rates) - {R}:
            o, n, _, w = SR.params(r, R)
            while self.tile > 32 and ((self.tile + 3 * n - 1) // n + 2) * o + 2 * w > 8192:
                self.tile //= 2

    def padded(self, fi, L):
        ref, bound = self.ref[fi]
        z = np.zeros((ref.shape[0], L))
        return np.concatenate([ref, z], 1), np.concatenate([bound, z], 1)

    def responses(self, fi):
        """The first and last output of each impulse's response (impulse files), else a few spread outputs."""
        x, r = self.x[fi], self.rates[fi]
        if r == self.R:
            s = np.flatnonzero(x.any(0))
            return list(zip(s, s))
        o, n, _, w = SR.params(r, self.R)
        s = np.flatnonzero(x.any(0))
        return [(-(-(t - w - o + 1) // o) * n, (t + w) // o * n + n - 1) for t in s]


def rate_corpus(R, ctx):
    if R not in _cache:
        _cache[R] = RateCorpus(R, ctx)
    return _cache[R]


def check_crops(rc, batch, files, offsets, key):
    out, lengths = batch(files, offsets)
    out, lengths = out.cpu().numpy(), lengths.cpu().numpy()
    files, offsets = np.asarray(files), np.asarray(offsets)
    L = batch.num_frames
    for fi in np.unique(files):
        sel = np.flatnonzero(files == fi)
        ref, bound = rc.padded(fi, L)
        cols = offsets[sel, None] + np.arange(L)[None, :]
        ch = ref.shape[0]
        want = np.minimum(L, rc.nt[fi] - offsets[sel])
        assert np.array_equal(lengths[sel], want), (key, fi)
        dev = out[sel]
        assert not dev[:, ch:].any(), (key, fi, "rows the file lacks")
        ratio = S.check_fir(dev[:, :ch].transpose(1, 0, 2), ref[:, cols], bound[:, cols], f"{key} file {fi}")
        note(f"resample {rc.kind[fi]}", ratio)


def crop_offsets(rc, L, rng):
    files, offsets = [], []
    T = rc.tile
    for fi, Nt in enumerate(rc.nt):
        resp = rc.responses(fi)
        pick = [resp[i] for i in rng.choice(len(resp), min(len(resp), 6), replace=False)]
        cand = {0, 1, max(0, Nt - 1), Nt, max(0, Nt - L // 2)}
        for a, b in pick:
            mid = (a + b) // 2
            cand |= {a + 1, mid, b - L + 2, mid - T, mid - 2 * T + 1, mid - L // 2}  # cut by crop and tile edges
        cand |= set(int(v) for v in rng.integers(0, Nt + 1, 3))
        for o in sorted(c for c in cand if 0 <= c <= Nt):
            files.append(fi)
            offsets.append(o)
    return files, offsets


@gpu
@pytest.mark.parametrize("R", sorted(RESAMPLE_CASES))
def test_resampled_crops_impulse_responses(rctx, R):
    rc = rate_corpus(R, rctx)
    rng = np.random.default_rng(R)
    T = rc.tile
    for L in sorted({1, 7, T - 1, T + 3, 3 * T + 5}):
        files, offsets = crop_offsets(rc, L, rng)
        check_crops(rc, rc.corpus.crops(len(files), L, sample_rate=R), files, offsets, f"R {R} L {L}")
    print(f"tile {T}; worst error / bound so far: {WORST}")


@gpu
@pytest.mark.parametrize("R", sorted(RESAMPLE_CASES))
def test_resampled_packed_impulse_responses(rctx, R):
    """Whole files, excerpts across responses and tiles, and runs of excerpts of 1 to 9 outputs from every file."""
    rc = rate_corpus(R, rctx)
    rng = np.random.default_rng(R + 1)
    files, offsets, lengths = [], [], []
    for fi, Nt in enumerate(rc.nt):
        files.append(fi), offsets.append(0), lengths.append(-1)
        for a, b in rc.responses(fi)[:: max(1, len(rc.responses(fi)) // 5)]:
            files.append(fi), offsets.append(max(0, a - 3)), lengths.append(b - a + 7)
            files.append(fi), offsets.append(max(0, min(a + 1, Nt))), lengths.append(2 * rc.tile + 3)
    for _ in range(120):
        fi = int(rng.integers(0, len(rc.nt)))
        a, b = rc.responses(fi)[int(rng.integers(0, len(rc.responses(fi))))]
        files.append(fi), offsets.append(max(0, min(int(rng.integers(a, b + 1)), rc.nt[fi])))
        lengths.append(int(rng.integers(1, 10)))
    n = [min(rc.nt[f] - o, rc.nt[f] if ln == -1 else ln) for f, o, ln in zip(files, offsets, lengths)]
    T = sum(r4(v) for v in n) + 8
    pk = rc.corpus.packed(len(files), T, sample_rate=R)
    out, starts, got_n = pk(files, offsets, lengths)
    out, starts, got_n = out.cpu().numpy(), starts.cpu().numpy(), got_n.cpu().numpy()
    assert got_n.tolist() == n
    ref = np.zeros(out.shape)
    bound = np.zeros(out.shape)
    for fi, o, s, m in zip(files, offsets, starts, n):
        r, bd = rc.ref[fi]
        ref[:r.shape[0], s:s + m] = r[:, o:o + m]
        bound[:r.shape[0], s:s + m] = bd[:, o:o + m]
    note("resample packed", S.check_fir(out, ref, bound, f"packed R {R}"))


@gpu
def test_more_than_65535_crops(rctx):
    """70 000 crops: the crop loop of resample_kernel takes a second trip over gridDim.y."""
    R = 16000
    rc = rate_corpus(R, rctx)
    rng = np.random.default_rng(65536)
    B, L = 70000, 5
    files = rng.integers(0, len(rc.nt), B)
    offsets = np.array([int(rng.integers(0, rc.nt[f] + 1)) for f in files])
    check_crops(rc, rc.corpus.crops(B, L, sample_rate=R), files, offsets, "70000 crops")


# --------------------------------------------------------------------------- mel, bin by bin

MEL_RATE, MEL_N = 16000, 12000


def mel_pcm():
    """16-bit rows: cosines of periods 4, 6, 10 and 16; DC, a full-scale alternation, impulses and a full-scale
    square wave; silence and full-scale noise; cosines of periods 30 and 8 together."""
    t = np.arange(MEL_N)
    rng = np.random.default_rng(44)
    imp = np.zeros(MEL_N, np.int64)
    imp[5::97] = 16384
    return [
        np.stack([np.round(30000 * np.cos(2 * np.pi * t / p)) for p in (4, 6, 10, 16)]).astype(np.int64),
        np.stack([np.full(MEL_N, 32767), np.where(t % 2, -32768, 32767), imp, np.where((t // 6) % 2, -32767, 32767)]),
        np.stack([np.zeros(MEL_N, np.int64), rng.integers(-32768, 32768, MEL_N)]),
        np.round(16000 * np.cos(2 * np.pi * t / 30) + 16000 * np.cos(2 * np.pi * t / 8)).astype(np.int64)[None],
    ]


_mel = {}


def mel_corpus(ctx):
    if "c" not in _mel:
        pcms = mel_pcm()
        idx = cb.index([P.flac_from_pcm(p, 16, MEL_RATE, 1024) for p in pcms])
        _mel["c"] = (cb.Corpus(idx, ctx), [p / 32768.0 for p in pcms])
    return _mel["c"]


def mel_tile(n_fft):
    t = 32
    while t > 1 and 2 * t * (n_fft // 2) * 8 > 65536:
        t //= 2
    return t


def mel_shape(n_fft, center):
    """(window, hop, L): a window of win_length n_fft - 1 (center) or n_fft - 3 with zeros inside it, and L giving F =
    2 * tile - 1 frames (past the tile, a partial last tile)."""
    win = n_fft - 1 if center else n_fft - 3
    w = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(win) / win) + 0.25).astype(np.float32)
    w[3::7] = 0.0
    hop = max(1, n_fft // 3)
    F = max(2, 2 * mel_tile(n_fft) - 1)
    L = (F - 1) * hop + (hop - 1) // 2 if center else n_fft + (F - 1) * hop + hop // 2
    assert SM.n_frames(L, n_fft, hop, center) == F
    return w, hop, L


_MEL_TABLES = cb._mel_tables


def patched(monkeypatch, window, fbank):
    def tables(*args, **kw):
        params, _, _ = _MEL_TABLES(*args, **kw)
        return params, window, fbank

    monkeypatch.setattr(cb, "_mel_tables", tables)


def slices(K):
    for k0 in range(0, K, 512):
        fb = np.zeros((K, min(512, K - k0)), np.float32)
        fb[k0 + np.arange(fb.shape[1]), np.arange(fb.shape[1])] = 1.0
        yield k0, fb


def power_ref(seg, n_fft, hop, window, center):
    u = SM.frames(seg, n_fft, hop, window, center)
    return np.abs(np.fft.rfft(u, axis=-1)) ** 2, S.frames_energy(u, n_fft)


def crop_rows(xs, files, offsets, L, C_):
    x = np.zeros((len(files), C_, L))
    for b, (f, o) in enumerate(zip(files, offsets)):
        seg = xs[f][:, o:o + L]
        x[b, :seg.shape[0], :seg.shape[1]] = seg
    return x


@gpu
@pytest.mark.parametrize("center", [True, False])
def test_mel_bins_every_n_fft(rctx, monkeypatch, center):
    corpus, xs = mel_corpus(rctx)
    C_ = corpus.channels
    for n_fft in supported():
        window, hop, L = mel_shape(n_fft, center)
        files, offsets = [], []
        for fi in range(len(xs)):
            for o in (0, MEL_N // 2 + 3, MEL_N - L // 2):
                files.append(fi), offsets.append(o)
        x = crop_rows(xs, files, offsets, L, C_)
        ref, E = power_ref(x, n_fft, hop, window, center)          # [B, C, F, K], [B, C, F]
        # packed: excerpts of L samples, of the shortest length with a frame, and of a middling one
        shortest = n_fft // 2 + 1 if center else n_fft
        pf, po, pl = [], [], []
        for fi in range(len(xs)):
            for o, n in ((7, L), (MEL_N - shortest, shortest), (101, shortest + 2 * hop + 1), (0, L // 2 + shortest)):
                pf.append(fi), po.append(o), pl.append(n)
        T = sum(r4(n) for n in pl)
        kw = dict(n_fft=n_fft, win_length=window.size, hop_length=hop, center=center)
        for k0, fb in slices(n_fft // 2 + 1):
            patched(monkeypatch, window, fb)
            K = fb.shape[1]
            mb = corpus.mel_crops(len(files), L, n_mels=K, **kw)
            feats, _ = mb(files, offsets)
            dev = feats.cpu().numpy().transpose(0, 1, 3, 2)              # [B, C, F, K]
            note("mel crops", S.check_bins(dev, ref[..., k0:k0 + K], E, n_fft, f"crops n_fft {n_fft} bins {k0}+"))
            assert not dev[E == 0].any()
            mp = corpus.mel_packed(len(pf), T, n_mels=K, **kw)
            out, starts, frames, lengths = mp(pf, po, pl)
            out, starts, frames = out.cpu().numpy(), starts.cpu().numpy(), frames.cpu().numpy()
            covered = np.zeros(out.shape, bool)
            for b, (fi, o, n) in enumerate(zip(pf, po, pl)):
                F = SM.n_frames(n, n_fft, hop, center)
                assert frames[b] == F
                seg = np.zeros((C_, n))
                seg[:xs[fi].shape[0]] = xs[fi][:, o:o + n]
                pr, pe = power_ref(seg, n_fft, hop, window, center)
                d = out[:, :, starts[b]:starts[b] + F].transpose(0, 2, 1)
                note("mel packed", S.check_bins(d, pr[..., k0:k0 + K], pe, n_fft, f"packed n_fft {n_fft} excerpt {b}"))
                covered[:, :, starts[b]:starts[b] + F] = True
            assert not out[~covered].any(), n_fft
            del mb, mp, feats, out
    print(f"worst error / bound so far: {WORST}")


NONTRI = 7


def nontriangular(K):
    """Columns: bins 0 and N only; negative weights; all zero; every bin; zeros inside a band; alternating signs over
    every bin; bin N alone."""
    fb = np.zeros((K, NONTRI), np.float32)
    fb[0, 0], fb[K - 1, 0] = 1.0, 0.5
    fb[3:11, 1] = -1.0
    fb[:, 3] = 0.25
    fb[5, 4], fb[8, 4] = 1.0, 2.0
    fb[:, 5] = np.where(np.arange(K) % 2, -1.0, 1.0)
    fb[K - 1, 6] = 3.0
    return fb


@gpu
@pytest.mark.parametrize("n_fft", [30, 400])
def test_mel_nontriangular_filterbanks(rctx, monkeypatch, n_fft):
    """Power within sum_k |fb_k| (bin bound_k) plus the band's n fmaf roundings; with the log, exactly the floor's
    float32(ln) where even the upper bound is at or below the floor (silence, negative and empty columns), else
    ln(mel) within the same bound and logf's rounding."""
    corpus, xs = mel_corpus(rctx)
    C_, K = corpus.channels, n_fft // 2 + 1
    window, hop, L = mel_shape(n_fft, True)
    files, offsets = [0, 1, 2, 3, 1], [0, 11, 5000, MEL_N - L // 2, 3]
    x = crop_rows(xs, files, offsets, L, C_)
    P_, E = power_ref(x, n_fft, hop, window, True)
    fb = nontriangular(K)
    fb64 = fb.astype(np.float64)
    nz = fb != 0
    band = np.array([np.ptp(np.flatnonzero(c)) + 1 if c.any() else 0 for c in nz.T])
    ref = P_ @ fb64                                                     # [B, C, F, M]
    bb = S.bin_bound(P_, E, n_fft) @ np.abs(fb64)
    bound = bb + band * S.U * (1 + 2.0 ** -20) * ((P_ + S.bin_bound(P_, E, n_fft)) @ np.abs(fb64))
    patched(monkeypatch, window, fb)
    floor = 2.0 ** -30
    for log_floor in (None, floor):
        mb = corpus.mel_crops(len(files), L, n_mels=NONTRI, n_fft=n_fft, win_length=window.size, hop_length=hop,
                              log_floor=log_floor)
        dev = mb(files, offsets)[0].cpu().numpy().transpose(0, 1, 3, 2).astype(np.float64)
        if log_floor is None:
            note("mel non-triangular", S.check_fir(dev, ref, bound, f"n_fft {n_fft}"))
            assert (dev[..., 2] == 0).all() and (dev[E == 0] == 0).all()
            assert (dev[..., 1][ref[..., 1] + bound[..., 1] < 0] < 0).all()
            continue
        at_floor = np.float32(np.log(np.float64(np.float32(floor))))
        low = ref + bound <= floor
        assert (dev[low] == at_floor).all() and low[..., 2].all() and low[E == 0].all()
        high = ref - bound > floor
        lo_ = np.where(high, ref - bound, 1.0)
        tol = np.log(np.where(high, ref, 1.0) / lo_) + 2.0 ** -22 * np.maximum(1.0, np.abs(np.log(np.where(high, ref, 1.0))))
        err = np.abs(dev - np.log(np.where(high, ref, 1.0)))
        assert (err[high] <= tol[high]).all(), (err[high] / tol[high]).max()
        mid = ~low & ~high
        assert (dev[mid] >= at_floor).all() and (dev[mid] <= np.log(np.maximum(ref + bound, floor))[mid] + 1e-6).all()


@gpu
def test_report_worst_ratios():
    """Runs last in this module: the worst ratio of error to bound of each check above."""
    print(f"worst error / bound: {WORST}")
    assert all(v <= 1.0 for v in WORST.values())
