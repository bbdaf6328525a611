"""Every excerpt batch kind past one scan block: thousands of excerpts per call against tests/spec_excerpts.py (-m gpu).

The planners (excerpt_scan_kernel, resample_map_kernel, mel_packed_plan_kernel) walk a call's excerpts 1024 at a time
and carry their running sums between chunks.  So each call here has B in {1023, 1024, 1025, 2049, 5000}, invalid
requests at 1023 / 1024 and 2047 / 2048, empty and 1-sample excerpts at the chunk edges, and T chosen so that the first
excerpt that does not fit is 1024 or 2049.  Every output is held whole, [C, T] or [B, C, L] or [C, n_mels, T_f], to the
restated plan: starts, lengths, statuses and the error word exactly, the samples bit for bit against load() (float64
resampler and mel references within their bounds), and every element outside an excerpt exactly 0.

Beyond the planners: owner_of over the slot and gather-chunk scans past 1024 excerpts (emit, host gather, several
chunks per long span), the binary searches of resample_packed_kernel and mel_packed_kernel, excerpt_zero_kernel's
grid-stride ((B + 1) C > 32768 rows), a short call after a long one, and mel_norm_kernel's second trip over its
2^20 CTAs x 16 warps (n C n_mels > 2^24 segments), with a Whisper crop batch of more than 65 535 rows.  Wherever a
pass must clear what an earlier call wrote (a crop's tail and missing rows, a packed excerpt's alignment pad and
missing rows, the unused excerpts past the count), the batch is first called with requests that fill those places.

The error word, and the lengths and statuses of the unused excerpts past the count, have no public view: like the
other batch tests, these read the batches' `_error`, `_lengths` and `_status` views of the library's buffers.
"""
import gc

import numpy as np
import pytest

import claxon_b200 as cb
from tests import edge_frames as E
from tests import pcm_flac as P
from tests import spec_excerpts as X
from tests import spec_mel as SM
from tests import spec_mel_norm as MN
from tests import spec_signal as SS

gpu = pytest.mark.gpu
R = 16000
FLOOR = 1e-10
MEL = dict(n_fft=8, hop_length=4, log_floor=FLOOR)  # excerpts of 5 samples and more have frames
WORST = {}


def note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratios():
    """After the module's tests: the worst ratio of error to bound each kind reached (for the normalisations, the
    error in float32 ulps of the map applied to the unnormalised features).  Each checker asserts its own bound."""
    yield
    print(f"\nworst error / bound: {WORST}")


# --------------------------------------------------------------------------- the corpus

def variable_flac(pcm, bps, rate, sizes):
    """pcm as a variable-blocking stream: block sizes cycling through `sizes` (the last one cut at the end)."""
    C_, N = pcm.shape
    head = bytearray(P.streaminfo(C_, N, bps, rate, max(sizes), P.md5_of(pcm, bps)))
    head[8:10] = min(sizes).to_bytes(2, "big")  # STREAMINFO's minimum block size
    parts, at, i = [bytes(head)], 0, 0
    while at < N:
        bs = min(sizes[i % len(sizes)], N - at)
        subs = [E.Sub("constant", [int(r[0])]) if r.min() == r.max() else E.Sub("verbatim", r.tolist())
                for r in pcm[:, at:at + bs]]
        parts.append(E.write(E.Frame(bps, subs, block_size=bs, number=at, variable=True,
                                     sr_code=P.RATE_CODES.get(rate, 0)))[0])
        at, i = at + bs, i + 1
    return np.frombuffer(b"".join(parts), np.uint8).copy()


# (channels, bits, rate, block size or a cycle of variable sizes, samples)
PLAIN = [(1, 16, R, 1024, 30000), (2, 12, R, 192, 4000), (4, 24, R, [256, 100, 37, 211], 6000),
         (2, 16, R, [512, 77, 300], 6000), (1, 8, R, 16, 500), (2, 20, R, 512, 3)]
OTHER = [(2, 16, 48000, 1024, 20000), (1, 16, 24000, [333, 512, 64], 9000), (4, 16, 48000, 256, 3000)]

def make_file(i, spec):
    C_, bps, rate, bs, N = spec
    rng = np.random.default_rng(100 + i)
    pcm = rng.integers(-(1 << (bps - 1)), 1 << (bps - 1), (C_, N))
    pcm[:, N // 3:N // 3 + 700] = np.arange(C_)[:, None] - 1  # constant subframes
    data = variable_flac(pcm, bps, rate, bs) if isinstance(bs, list) else P.flac_from_pcm(pcm, bps, rate, bs)
    return data, pcm


class Files:
    """A corpus of designed files: their bytes, PCM, load() rows (checked against the PCM) and lengths at R."""

    def __init__(self, specs, ctx):
        import torch
        made = [make_file(i, s) for i, s in enumerate(specs)]
        self.srcs = [d for d, _ in made]
        self.idx = cb.index(self.srcs)
        self.i32 = [cb.load(s, dtype=torch.int32, ctx=ctx)[0].cpu().numpy() for s in self.srcs]
        self.f32 = [cb.load(s, dtype=torch.float32, ctx=ctx)[0].cpu().numpy() for s in self.srcs]
        for (_, pcm), a, b, s in zip(made, self.i32, self.f32, specs):
            assert np.array_equal(a, pcm) and np.array_equal(b, (pcm / float(1 << (s[1] - 1))).astype(np.float32))
        self.rates = [s[2] for s in specs]
        self.N = [s[4] for s in specs]
        self.Nt = [X.length_at(n, r, R) for n, r in zip(self.N, self.rates)]
        self.C = max(s[0] for s in specs)
        self._refs = None
        self.corpora = {}

    def corpus(self, memory, ctx):
        if memory not in self.corpora:
            self.corpora[memory] = cb.Corpus(self.idx, ctx, memory=memory)
        return self.corpora[memory]

    def refs(self):
        """spec_signal.fir_ref_bound of each whole file at R (the float64 resampler and its per-output bound)."""
        if self._refs is None:
            self._refs = [SS.fir_ref_bound(x.astype(np.float64), r, R) for x, r in zip(self.f32, self.rates)]
        return self._refs


@pytest.fixture(scope="module")
def rctx():
    c = cb.Context(device=0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def plain(rctx):
    """1, 2 and 4 channel files at 16 kHz, fixed and variable blocking (C = 4)."""
    return Files(PLAIN, rctx)


@pytest.fixture(scope="module")
def mixed(rctx):
    """The same files and three more at 48 and 24 kHz."""
    return Files(PLAIN + OTHER, rctx)


# --------------------------------------------------------------------------- requests

def invalid_request(k, n_files, N):
    return [(n_files, 0, 1), (0, -1, 3), (0, 0, 0), (0, 0, -2), (0, N + 1, 1), (1 << 32, 0, 1)][k % 6]


def requests(B, Ns, seed, invalid=(), empty=(), ones=(), long=()):
    """B requests, mostly 1 to 9 samples (some to the file's end, some cut by it), with the given indices invalid,
    empty (offset N), of one sample, or long (20 000 samples and more of file 0, many frames and gather chunks)."""
    rng = np.random.default_rng(seed)
    files, offsets, lengths = [], [], []
    for b in range(B):
        f = int(rng.integers(0, len(Ns)))
        N = Ns[f]
        u = rng.random()
        if u < 0.05:
            o, ln = N - int(rng.integers(0, min(N, 9) + 1)), -1
        elif u < 0.1:
            o, ln = N - int(rng.integers(1, min(N, 4) + 1)), 9
        else:
            ln = min(int(rng.integers(1, 10)), N)
            o = int(rng.integers(0, N - ln + 1))
        files.append(f), offsets.append(o), lengths.append(ln)
    for b in ones:
        f = int(rng.integers(0, len(Ns)))
        files[b], offsets[b], lengths[b] = f, int(rng.integers(0, Ns[f])), 1
    for b in empty:
        f = int(rng.integers(0, len(Ns)))
        files[b], offsets[b], lengths[b] = f, Ns[f], (-1, 3)[b % 2]
    for k, b in enumerate(long):
        files[b], offsets[b], lengths[b] = 0, 11 * k, (-1, 20000 + k)[k % 2]
    for k, b in enumerate(invalid):
        files[b], offsets[b], lengths[b] = invalid_request(k, len(Ns), Ns[0])
    return files, offsets, lengths


def t_cut(files, offsets, lengths, Ns, k):
    """T at which excerpt k (valid, n_k >= 1) is the first that does not fit: one column short of its end."""
    p = X.packed_plan(files, offsets, lengths, Ns, 1 << 40)
    assert p.lengths[k] >= 1
    return p.starts[k] + p.lengths[k] - 1


def t_all(files, offsets, lengths, Ns):
    p = X.packed_plan(files, offsets, lengths, Ns, 1 << 40)
    return sum(X.r4(n) for n in p.lengths) + 13


EDGES = (1023, 1024, 2047, 2048, 3071, 3072, 4095, 4096)


def calls(Ns):
    """(name, max_excerpts, requests, T, count) of the calls every packed kind runs."""
    out = []
    r = requests(1023, Ns, 1, invalid=(5, 1022), empty=(1021,), ones=(1020,))
    out.append(("B 1023", 1023, r, t_all(*r, Ns), None))
    r = requests(1024, Ns, 2, invalid=(1023,), empty=(1021,), ones=(1022,), long=(3,))
    out.append(("B 1024", 1024, r, t_all(*r, Ns), None))
    r = requests(1025, Ns, 3, invalid=(1023,), empty=(1022,), ones=(1021,))
    r[0][1024], r[1][1024], r[2][1024] = 0, 5, 4
    out.append(("B 1025, first non-fit 1024", 1025, r, t_cut(*r, Ns, 1024), None))
    r = requests(2100, Ns, 4, invalid=(1023, 1024, 2047, 2048), empty=(1025, 2046), ones=(1022, 2045),
                 long=(100, 1500))
    out.append(("count 2049 of 2100", 2100, r, t_all(*r, Ns), 2049))
    r = requests(2050, Ns, 5, invalid=(2047, 2048), empty=(1023, 1024), ones=(1025,), long=(7, 1030))
    r[0][2049], r[1][2049], r[2][2049] = 0, 0, 7
    out.append(("B 2050, first non-fit 2049", 2050, r, t_cut(*r, Ns, 2049), None))
    r = requests(5000, Ns, 6, invalid=EDGES, empty=(1022, 2049, 3070), ones=(1025, 2046, 4097),
                 long=(10, 1100, 2500, 4000))
    out.append(("B 5000", 5000, r, t_all(*r, Ns), None))
    return out


def subset(r, count):
    return tuple(v[:count] for v in r) if count is not None else r


# --------------------------------------------------------------------------- packed batches

def run_packed(batch, fs, r, count, ref_rows, what):
    """One call of a plain packed batch against the plan and the load() rows: the used excerpts' starts, and the
    lengths and statuses of all max_excerpts of them (the unused ones 0).  Returns (plan, out, expected out)."""
    files, offsets, lengths = subset(r, count)
    plan = X.packed_plan(files, offsets, lengths, fs.N, batch.max_samples, max_excerpts=batch.max_excerpts)
    out, starts, _ = batch(files, offsets, lengths, check=False)
    out = out.cpu().numpy()
    X.check_plan(plan, starts.cpu().numpy(), batch._lengths.cpu().numpy(), batch._status.cpu().numpy(),
                 batch._error.item(), what)
    want = X.expected_packed(plan, files, offsets, ref_rows, fs.C, batch.max_samples, out.dtype)
    X.check_exact(out, want, what)
    return plan, out, want


def short_after(r, plan, n=300):
    """The first n requests of a long call, each valid excerpt with samples replaced by one of the 1-channel file 0,
    3 samples shorter (at least 1): the layout moves little, and the long call's samples are left in the short
    call's alignment pads and in the rows file 0 lacks, which the short call must clear."""
    files, offsets, lengths = (list(v[:n]) for v in r)
    for b in range(n):
        if plan.lengths[b]:
            files[b], offsets[b], lengths[b] = 0, 37 * b % 29000, max(1, plan.lengths[b] - 3)
    return files, offsets, lengths


@gpu
@pytest.mark.parametrize("memory", ["device", "host"])
@pytest.mark.parametrize("dtype_name", ["int32", "float32"])
def test_packed(rctx, plain, memory, dtype_name):
    import torch
    dtype = getattr(torch, dtype_name)
    corpus = plain.corpus(memory, rctx)
    rows = plain.i32 if dtype_name == "int32" else plain.f32
    for name, B, r, T, count in calls(plain.N):
        batch = corpus.packed(B, T, dtype=dtype)
        what = f"{memory} {dtype_name} {name}"
        if count is not None:  # every excerpt first, so that the unused ones have lengths and statuses to clear
            run_packed(batch, plain, r, None, rows, f"{what}, all {B}")
        long_plan, long_out, _ = run_packed(batch, plain, r, count, rows, what)
        if B == 5000:  # a short call after the long one, against the plan and a fresh batch
            short = short_after(r, long_plan)
            plan, out, want = run_packed(batch, plain, short, None, rows, f"{what}, then 300")
            assert plan.end < long_plan.end and long_out[:, plan.end:long_plan.end].any()
            stale = (long_out[:, :plan.end] != 0) & (want[:, :plan.end] == 0)  # what the per-excerpt zeroing clears
            assert stale[0].any() and stale[1:].any()
            fresh = corpus.packed(B, T, dtype=dtype)(*short, check=False)[0].cpu().numpy()
            X.check_exact(out, fresh, "fresh batch")
        del batch
        gc.collect()


# --------------------------------------------------------------------------- resampled packed batches

@gpu
def test_resampled_packed(rctx, mixed):
    corpus = mixed.corpus("device", rctx)
    refs = mixed.refs()
    for name, B, r, T, count in calls(mixed.Nt):
        files, offsets, lengths = subset(r, count)
        plan = X.packed_plan(files, offsets, lengths, mixed.Nt, T)
        batch = corpus.packed(B, T, sample_rate=R)
        out, starts, lens = batch(files, offsets, lengths, check=False)
        X.check_plan(plan, starts.cpu().numpy(), lens.cpu().numpy(), batch.status.cpu().numpy(),
                     batch._error.item(), f"resampled {name}")
        ref, bound = X.expected_resampled(plan, files, offsets, refs, mixed.C, T)
        note("resample", X.check_bound(out.cpu().numpy(), ref, bound, f"resampled {name}"))
        del batch
        gc.collect()


# --------------------------------------------------------------------------- mel packed batches

def check_mel_packed(feats, x, plan, mplan, window, fbank, what):
    """Features [C, M, T_f] against spec_mel of each excerpt's samples x[:, s_b : s_b + n_b] (the same requests'
    float32 packed output), excerpts of one length together; every other column exactly 0."""
    starts, lens = np.asarray(plan.starts), np.asarray(plan.lengths)
    fst, frames = np.asarray(mplan.starts), np.asarray(mplan.lengths)
    covered = np.zeros(feats.shape[-1], bool)
    for n in np.unique(lens[frames > 0]):
        sel = np.flatnonzero((lens == n) & (frames > 0))
        F = int(frames[sel[0]])
        seg = x[:, starts[sel][:, None] + np.arange(n)].transpose(1, 0, 2).astype(np.float64)   # [k, C, n]
        ref = SM.mel(seg, 8, 4, window, fbank, True, FLOOR)                                     # [k, C, M, F]
        delta = SM.bound(seg, 8, 4, window, fbank, True)
        cols = fst[sel][:, None] + np.arange(F)
        dev = feats[:, :, cols].transpose(2, 0, 1, 3)
        note("mel", SM.check(dev, ref, delta, FLOOR))
        covered[cols.ravel()] = True
    rest = feats[:, :, ~covered]
    assert not rest.any(), (what, "outside the excerpts' frames", np.argwhere(rest != 0)[:4].tolist())


@gpu
@pytest.mark.parametrize("resampled", [False, True])
def test_mel_packed(rctx, plain, mixed, resampled):
    fs = mixed if resampled else plain
    corpus = fs.corpus("device", rctx)
    rate = R if resampled else None
    Ns = fs.Nt if resampled else fs.N
    for name, B, r, T, count in calls(Ns):
        files, offsets, lengths = subset(r, count)
        plan = X.packed_plan(files, offsets, lengths, Ns, T)
        mplan = X.mel_plan(plan, 8, 4)
        pk = corpus.packed(B, T, sample_rate=rate)
        x = pk(files, offsets, lengths, check=False)[0].cpu().numpy()
        del pk
        mb = corpus.mel_packed(B, T, rate, n_mels=8, **MEL)
        nb = corpus.mel_packed(B, T, rate, n_mels=8, normalize="per_feature", **MEL)
        y0, st, fr, ln = mb(files, offsets, lengths, check=False)
        X.check_plan(mplan, st.cpu().numpy(), fr.cpu().numpy(), mb.status.cpu().numpy(), mb._error.item(), name)
        assert ln.cpu().tolist() == plan.lengths
        y0 = y0.cpu().numpy()
        check_mel_packed(y0, x, plan, mplan, mb.window, mb.fbank, f"mel {name}")
        y, st, fr, ln = nb(files, offsets, lengths, check=False)
        X.check_plan(mplan, st.cpu().numpy(), fr.cpu().numpy(), nb.status.cpu().numpy(), nb._error.item(), name)
        note("mel-norm (ulps)", X.per_feature_packed(y.cpu().numpy(), y0, mplan.starts, mplan.lengths))
        del mb, nb
        gc.collect()


# --------------------------------------------------------------------------- crop batches

@gpu
@pytest.mark.parametrize("memory", ["device", "host"])
def test_crops(rctx, plain, memory):
    """B 1025 and 8200 crops, invalid ones at the chunk edges: (8200 + 1) x 4 rows > 32768, so the zero pass
    grid-strides, and rows 32 768 and up (crops 8192 .. 8199) are cleared on its second trip.  Each batch is first
    called with every crop full (L samples of the 4-channel file), then with short, empty, 1-channel and invalid
    crops at the chunk edges and past crop 8192: a zero range the pass misses keeps the first call's samples."""
    import torch
    corpus = plain.corpus(memory, rctx)
    N2 = plain.N[2]
    for B, L, invalid in ((1025, 9, (1023, 1024)), (8200, 7, EDGES + (8191, 8192, 8199))):
        at = [b for b in (1021, 1022, 1025, 2046, 2049) if b < B]
        files, offsets, _ = requests(B, plain.N, B, empty=at[1::2], ones=at[0::2])
        if B == 8200:  # past row 32768: short, empty and 1-channel crops
            for b, (f, o) in zip(range(8193, 8199), ((2, N2 - 3), (2, N2), (0, 5), (1, 0), (2, N2 - 1), (4, 499))):
                files[b], offsets[b] = f, o
        for b in invalid:  # what a crop request can get wrong: the file, the offset
            files[b], offsets[b] = ((len(plain.N), 0), (0, -1), (1 << 32, 0), (2, N2 + 1))[b % 4]
        plan = X.crop_plan(files, offsets, L, plain.N)
        batch = corpus.crops(B, L, dtype=torch.int32)
        fill = batch([2] * B, [(97 * b) % (N2 - L) for b in range(B)])[0].cpu().numpy()
        want = X.expected_crops(plan, files, offsets, plain.i32, plain.C, L)
        assert ((fill != 0) & (want == 0))[B - 8:].any()  # the first call's samples where the second must clear
        out, lens = batch(files, offsets, check=False)
        X.check_plan(plan, None, lens.cpu().numpy(), batch.status.cpu().numpy(), batch._error.item(),
                     f"{memory} crops {B}")
        X.check_exact(out.cpu().numpy(), want, f"{memory} crops {B}")
        assert (B + 1) * plain.C > 32768 or B == 1025
        del batch
        gc.collect()


# --------------------------------------------------------------------------- mel_norm_kernel past 2^24 segments

_MEL_TABLES = cb._mel_tables


@pytest.fixture
def dense_fbank(monkeypatch):
    """Every batch made in the test gets a dense positive [5, n_mels] filterbank, so that no (row, mel) segment is
    constant and every one of them normalises to something other than 0; the same one for every batch of a shape."""

    def tables(*args, **kw):
        params, window, fbank = _MEL_TABLES(*args, **kw)
        return params, window, np.random.default_rng(9).uniform(0.1, 1.0, fbank.shape).astype(np.float32)

    monkeypatch.setattr(cb, "_mel_tables", tables)


@gpu
def test_mel_norm_past_2_24_segments(rctx, plain, dense_fbank):
    """66 000 crops / excerpts x C 2 x 128 mels = 16 896 000 segments: mel_norm_kernel's 2^20 CTAs of 16 warps cover
    2^24 of them, the rest (crops 65 536 and up) on its second trip.  Then Whisper over 33 000 crops: 66 000 rows."""
    two = Files([PLAIN[1], PLAIN[4]], rctx)  # 2 and 1 channels, blocks of 192 and 16 samples
    corpus = two.corpus("device", rctx)
    assert two.C == 2
    B, L, M = 66000, 8, 128
    assert B * two.C * M > 1 << 24 and -(-B * two.C * M // 16) > 1 << 20  # past mel_norm_kernel's grid
    files, offsets, _ = requests(B, two.N, 7)
    for b in range(65540, 65549):  # 0 to 8 samples: inner rows past 32 768 the zero pass clears on its second trip
        files[b], offsets[b] = b % 2, two.N[b % 2] - (b - 65540)
    for b in (1023, 65535, 65536, 65999):
        files[b], offsets[b] = 2, 0
    kw = dict(n_mels=M, **MEL)
    # crops: F = 3, v_b = 1 + n_b // 4; each batch called first with every crop 8 samples of the 2-channel file
    plan = X.crop_plan(files, offsets, L, two.N)
    nb, mb = corpus.mel_crops(B, L, normalize="per_feature", **kw), corpus.mel_crops(B, L, **kw)
    full = ([0] * B, [(13 * b) % (two.N[0] - L) for b in range(B)])
    nb(*full), mb(*full)
    y, lens = nb(files, offsets, check=False)
    X.check_plan(plan, None, lens.cpu().numpy(), nb.status.cpu().numpy(), nb._error.item(), "mel crops 66000")
    x = mb(files, offsets, check=False)[0].cpu().numpy()
    valid = [1 + n // 4 if n else 0 for n in plan.lengths]
    note("mel-norm (ulps)", X.per_feature_crops(y.cpu().numpy(), x, valid))
    rows = sorted({0, 1023, 65534, 65535, 65536, 65537, 65998, 65999} | set(range(65500, 65600)))
    assert {plan.lengths[b] for b in rows} >= set(range(9))
    crops = np.zeros((len(rows), two.C, L))
    for i, b in enumerate(rows):
        n = plan.lengths[b]
        if n:
            src = two.f32[files[b]]
            crops[i, :src.shape[0], :n] = src[:, offsets[b]:offsets[b] + n]
    ref = SM.mel(crops, 8, 4, mb.window, mb.fbank, True, FLOOR)
    note("mel", SM.check(x[rows], ref, SM.bound(crops, 8, 4, mb.window, mb.fbank, True), FLOOR))
    del nb, mb, y, x
    gc.collect()
    # packed: 66 000 excerpts of 5 to 9 samples, F_b 2 or 3
    rng = np.random.default_rng(8)
    lengths = rng.integers(5, 10, B).tolist()
    files = rng.integers(0, 2, B)
    offsets = [int(rng.integers(0, two.N[f] - n + 1)) for f, n in zip(files, lengths)]
    T = sum(X.r4(n) for n in lengths)
    plan = X.packed_plan(files, offsets, lengths, two.N, T)
    mplan = X.mel_plan(plan, 8, 4)
    nb, mb = corpus.mel_packed(B, T, normalize="per_feature", **kw), corpus.mel_packed(B, T, **kw)
    y, st, fr, _ = nb(files, offsets, lengths, check=False)
    X.check_plan(mplan, st.cpu().numpy(), fr.cpu().numpy(), nb.status.cpu().numpy(), nb._error.item(), "packed")
    x = mb(files, offsets, lengths, check=False)[0].cpu().numpy()
    note("mel-norm (ulps)", X.per_feature_packed(y.cpu().numpy(), x, mplan.starts, mplan.lengths))
    del nb, mb, y, x
    gc.collect()
    # Whisper: one CTA per row, 66 000 rows
    Bw = 33000
    files, offsets = files[:Bw].tolist(), offsets[:Bw]
    wb, mb = corpus.mel_crops(Bw, L, normalize="whisper", **kw), corpus.mel_crops(Bw, L, **kw)
    assert Bw * two.C > 65535
    y = wb(files, offsets, check=False)[0].cpu().numpy()
    x = mb(files, offsets, check=False)[0].cpu().numpy()
    for a in range(0, Bw, 4096):
        note("whisper (ulps)", X.ulp_ratio(y[a:a + 4096], MN.whisper(x[a:a + 4096, ..., :-1])))


# --------------------------------------------------------------------------- device-drawn requests

@gpu
def test_device_drawn_requests(rctx, plain):
    """3000 requests from torch.randint (invalid files, offsets and lengths among them), check=False, T short enough
    that the excerpts stop fitting part way: the outputs against the same requests planned on the host."""
    import torch
    corpus = plain.corpus("device", rctx)
    B, T = 3000, 9000
    gen = torch.Generator(device="cuda").manual_seed(12)
    batch = corpus.packed(B, T, dtype=torch.int32)
    for _ in range(2):
        files = torch.randint(0, len(plain.N) + 1, (B,), device="cuda", generator=gen)
        offsets = torch.randint(-1, 40, (B,), device="cuda", generator=gen)
        lengths = torch.randint(0, 10, (B,), device="cuda", generator=gen)
        out, starts, lens = batch(files, offsets, lengths, check=False)
        f, o, ln = files.cpu().numpy(), offsets.cpu().numpy(), lengths.cpu().numpy()
        plan = X.packed_plan(f, o, ln, plain.N, T)
        X.check_plan(plan, starts.cpu().numpy(), lens.cpu().numpy(), batch.status.cpu().numpy(),
                     batch._error.item(), "device-drawn")
        X.check_exact(out.cpu().numpy(), X.expected_packed(plan, f, o, plain.i32, plain.C, T), "device-drawn")
        fits = [b for b, s in enumerate(plan.status) if s == 0 and plan.lengths[b]]
        assert fits[-1] > 1024 and plan.starts[-1] > T  # the excerpts stop fitting past the first chunk

