"""Normalised mel batches: normalize="per_feature" / "whisper" on Corpus.mel_crops and Corpus.mel_packed (-m gpu).

1. The pass alone: a normalised batch must equal tests/spec_mel_norm.py's float64 map applied to the unnormalised
   batch's features for the same requests, within one float32 ulp.  This isolates mel_norm_kernel from the mel's own
   error.
2. End to end: within spec_mel_norm's tolerance of the map applied to tests/spec_mel.py's float64 features of the crop
   or packed output, and against transformers.WhisperFeatureExtractor on 30 s crops at 16 kHz.
3. Determinism, device-drawn requests, host corpora, launch counts and the C ABI refusals.
"""
import ctypes as C
import gc

import numpy as np
import pytest

import claxon_b200 as cb
from tests import spec_mel as S
from tests import spec_mel_norm as N
from tests import spec_resample as SR
from tests.test_gpu_mel_crops import GRID, edge_requests, mel_args, single_rate_files
from tests.test_gpu_mel_packed import lengths_at, requests, span
from tests.test_gpu_resampled_crops import mixed_files

gpu = pytest.mark.gpu
FLOOR = 1e-10
WORST = [0.0]  # the largest end-to-end error-to-bound ratio seen


@pytest.fixture(scope="module")
def rctx():
    c = cb.Context(device=0)
    yield c
    c.close()


def crop_valid(lengths, hop):
    """v_b = 1 + n_b // hop, 0 for n_b = 0."""
    return [1 + int(n) // hop if n > 0 else 0 for n in lengths]


def crops_pair(corpus, B, L, R, normalize, **kw):
    kw = {"log_floor": FLOOR, **kw}
    return (corpus.mel_crops(B, L, R, normalize=normalize, **kw), corpus.mel_crops(B, L, R, **kw))


def check_crops_pass(nb, plain, files, offsets):
    """One call of the normalised crop batch and of its unnormalised twin: the map of the twin's features, within an
    ulp; status, lengths and the error word equal.  Returns (features, lengths) of the normalised batch."""
    import torch
    x, lengths = plain(files, offsets, check=False)
    y, ly = nb(files, offsets, check=False)
    assert torch.equal(ly, lengths) and torch.equal(nb.status, plain.status) and torch.equal(nb._error, plain._error)
    x, y = x.cpu().numpy(), y.cpu().numpy()
    if nb.normalize == "whisper":
        assert y.shape == x[..., :-1].shape and nb.n_frames == plain.n_frames - 1
        ref = N.whisper(x[..., :-1])
    else:
        assert y.shape == x.shape
        v = crop_valid(lengths.tolist(), nb.params.hop_length)
        ref = np.stack([N.per_feature(x[b], vb) for b, vb in enumerate(v)])
    N.within_ulp(y, ref)
    return y, lengths.cpu().numpy()


def check_crops_end_to_end(nb, crops, files, offsets, rows=None):
    """The normalised crop batch against the map of spec_mel's features of the crop output, within spec_mel_norm's
    tolerance."""
    x, lengths = crops(files, offsets, check=False)
    y, _ = nb(files, offsets, check=False)
    x, y, lengths = x.cpu().numpy(), y.cpu().numpy(), lengths.tolist()
    p = nb.params
    rows = range(nb.batch) if rows is None else rows
    for b in rows:
        ref = S.mel(x[b], p.n_fft, p.hop_length, nb.window, nb.fbank, True, FLOOR)
        D = N.log_bound(ref, S.bound(x[b], p.n_fft, p.hop_length, nb.window, nb.fbank, True), FLOOR)
        if nb.normalize == "whisper":
            ref, D = ref[..., :-1], D[..., :-1]
            want = N.whisper(ref)
            tol = N.whisper_tol(want, D.max(axis=(-2, -1), keepdims=True))
        else:
            v = crop_valid([lengths[b]], p.hop_length)[0]
            want = N.per_feature(ref, v)
            _, sigma = N.stats(ref, v)
            tol = N.per_feature_tol(want, D[..., :max(v, 1)].max(-1, keepdims=True), sigma)
        WORST[0] = max(WORST[0], N.check(y[b], want, tol))


def check_packed_pass(nb, plain, files, offsets=None, lengths=None):
    """As check_crops_pass for packed batches: each excerpt's F_b frames mapped, every other element exactly 0."""
    import torch
    x, s, f, n = plain(files, offsets, lengths, check=False)
    y, sy, fy, ny = nb(files, offsets, lengths, check=False)
    assert torch.equal(sy, s) and torch.equal(fy, f) and torch.equal(ny, n) and torch.equal(nb.status, plain.status)
    x, y = x.cpu().numpy(), y.cpu().numpy()
    ref = np.zeros(x.shape)
    for st, F in zip(s.tolist(), f.tolist()):
        ref[:, :, st:st + F] = N.per_feature(x[:, :, st:st + F], F)
    N.within_ulp(y, ref)  # (exact zeros where ref is 0)
    return y, s.cpu().numpy(), f.cpu().numpy()


# --------------------------------------------------------------------------- 1. the pass alone

@gpu
@pytest.mark.parametrize("normalize", ["per_feature", "whisper"])
def test_plain_crops_pass(ctx, normalize):
    """A corpus of 1, 2 and 4 channel files (C = 4), every decode path: edge crops, past the file's end included."""
    idx = cb.index(single_rate_files())
    corpus = cb.Corpus(idx, ctx)
    L = 4000
    files, offsets = edge_requests(idx, L)
    nb, plain = crops_pair(corpus, len(files), L, None, normalize, n_fft=400, hop_length=160, n_mels=80)
    y, lengths = check_crops_pass(nb, plain, files, offsets)
    v = crop_valid(lengths, 160)
    assert min(v) < nb.n_frames and min(lengths) == 0  # crops past the file's end, and an empty one
    if normalize == "per_feature":
        for b, vb in enumerate(v):
            assert (y[b, :, :, vb:] == 0).all()
        mono = [b for b, f in enumerate(files) if idx[f].info.channels == 1 and v[b] > 0]
        assert mono and (y[mono, 1:] == 0).all()  # rows the file lacks: constant features, exactly 0


@gpu
@pytest.mark.parametrize("g", [g for g in range(len(GRID)) if GRID[g][3]])
def test_resampled_crops_grid_pass(rctx, g):
    """The mixed-rate corpus at 16 kHz over the centred entries of the mel grid: n_fft 8 to 4096, both maps."""
    *args, L = GRID[g]
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    files, offsets = edge_requests(idx, L, 16000)
    kw = mel_args(*args, log_floor=FLOOR)
    plain = corpus.mel_crops(len(files), L, 16000, **kw)
    for normalize in ("per_feature", "whisper"):
        if normalize == "whisper" and plain.n_frames < 2:
            continue
        check_crops_pass(corpus.mel_crops(len(files), L, 16000, normalize=normalize, **kw), plain, files, offsets)


@gpu
def test_invalid_requests_and_short_crops(rctx):
    """Invalid requests: per_feature all 0, whisper the constant (ln(floor) / ln 10 + 4) / 4.  Crops of one frame's
    samples or fewer (v_b = 1) and a full one."""
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    L, R = 3000, 16000
    files, offsets = edge_requests(idx, L, R)
    bad = {1: (len(idx), 0), 4: (0, -1), 9: ((1 << 32) + 1, 0)}
    for b, (f, o) in bad.items():
        files[b], offsets[b] = f, o
    Nt = SR.out_len(idx[0].length, idx[0].info.sample_rate, R)
    files += [0, 0, 0]
    offsets += [Nt - 1, Nt - 159, Nt - 160]  # v_b = 1, 1, 2
    for normalize in ("per_feature", "whisper"):
        nb, plain = crops_pair(corpus, len(files), L, R, normalize, hop_length=160, n_mels=64)
        y, lengths = check_crops_pass(nb, plain, files, offsets)
        assert crop_valid(lengths[-3:], 160) == [1, 1, 2]
        for b in bad:
            assert lengths[b] == 0
            if normalize == "per_feature":
                assert (y[b] == 0).all()
            else:
                want = np.float32((float(np.float32(np.log(FLOOR))) / N.LN10 + 4) / 4)
                assert (np.abs(y[b] - want) <= abs(np.spacing(want))).all()


@gpu
def test_packed_pass(ctx):
    """Plain packed batches over the 1 / 2 / 4 channel corpus, every decode path, whole files and excerpts."""
    idx = cb.index(single_rate_files())
    corpus = cb.Corpus(idx, ctx)
    rng = np.random.default_rng(5)
    files, offsets, lengths = requests(idx, lambda r: int(r.integers(150, 9000)), rng)
    T = span(idx, files, offsets, lengths)
    kw = dict(n_fft=400, hop_length=160, n_mels=80, log_floor=FLOOR)
    nb = corpus.mel_packed(len(files), T, normalize="per_feature", **kw)
    plain = corpus.mel_packed(len(files), T, **kw)
    assert nb.stride == plain.stride
    check_packed_pass(nb, plain, files, offsets, lengths)


@gpu
@pytest.mark.parametrize("g", [g for g in range(len(GRID)) if GRID[g][3]])
def test_resampled_packed_grid_pass(rctx, g):
    *args, L = GRID[g]
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    rng = np.random.default_rng(g)
    files, offsets, lengths = requests(idx, lambda r: int(r.integers(1, 3 * L)), rng, R)
    T = span(idx, files, offsets, lengths, R)
    kw = mel_args(*args, log_floor=FLOOR)
    check_packed_pass(corpus.mel_packed(len(files), T, R, normalize="per_feature", **kw),
                      corpus.mel_packed(len(files), T, R, **kw), files, offsets, lengths)
    gc.collect()


@gpu
def test_packed_excerpts_of_0_1_2_frames(rctx):
    """n_fft 64, hop 100: excerpts of 0 frames (<= 32 samples), 1 (33 to 99) and 2 (100 to 199), among longer ones,
    with invalid requests and unused slots (max_excerpts above the count)."""
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    Ns = lengths_at(idx, R)
    files = [0, 1, 2, 3, 4, 5, 6, 0, 1, 4, len(idx), 2]
    offsets = [0, 5, 0, 100, 0, 7, 0, Ns[0] - 40, 0, 0, 0, Ns[2] + 1]
    lengths = [20, 33, 99, 100, 199, 32, 1, -1, 5000, -1, 10, 10]
    T = span(idx, files[:10], offsets[:10], lengths[:10], R) + 64
    kw = dict(n_fft=64, hop_length=100, n_mels=16, log_floor=FLOOR)
    nb = corpus.mel_packed(16, T, R, normalize="per_feature", **kw)
    plain = corpus.mel_packed(16, T, R, **kw)
    _, _, f = check_packed_pass(nb, plain, files, offsets, lengths)
    assert f[:7].tolist() == [0, 1, 1, 2, 2, 0, 0] and f[10] == 0 and f[11] == 0


# --------------------------------------------------------------------------- 2. end to end

@gpu
def test_crops_end_to_end(rctx):
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    L, R = 5000, 16000
    files, offsets = edge_requests(idx, L, R)
    crops = corpus.crops(len(files), L, sample_rate=R)
    for normalize in ("per_feature", "whisper"):
        nb = corpus.mel_crops(len(files), L, R, n_fft=400, hop_length=160, n_mels=80, mel_scale="slaney",
                              norm="slaney", log_floor=FLOOR, normalize=normalize)
        check_crops_end_to_end(nb, crops, files, offsets)
    print(f"worst error / bound: {WORST[0]:.3g}")


@gpu
def test_packed_end_to_end(rctx):
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    rng = np.random.default_rng(11)
    files, offsets, lengths = requests(idx, lambda r: int(r.integers(150, 6000)), rng, R)
    T = span(idx, files, offsets, lengths, R)
    pk = corpus.packed(len(files), T, sample_rate=R)
    nb = corpus.mel_packed(len(files), T, R, n_fft=400, hop_length=160, n_mels=80, log_floor=FLOOR,
                           normalize="per_feature")
    x, s, n = pk(files, offsets, lengths, check=False)
    y, st, fr, _ = nb(files, offsets, lengths, check=False)
    x, y, p = x.cpu().numpy(), y.cpu().numpy(), nb.params
    for b, F in enumerate(fr.tolist()):
        if not F:
            continue
        seg = x[:, s[b]:s[b] + n[b]]
        ref = S.mel(seg, p.n_fft, p.hop_length, nb.window, nb.fbank, True, FLOOR)
        D = N.log_bound(ref, S.bound(seg, p.n_fft, p.hop_length, nb.window, nb.fbank, True), FLOOR)
        want = N.per_feature(ref, F)
        _, sigma = N.stats(ref, F)
        WORST[0] = max(WORST[0], N.check(y[:, :, st[b]:st[b] + F], want,
                                         N.per_feature_tol(want, D.max(-1, keepdims=True), sigma)))
    print(f"worst error / bound: {WORST[0]:.3g}")


@gpu
@pytest.mark.parametrize("n_mels", [80, 128])
def test_whisper_against_feature_extractor(rctx, n_mels):
    """30 s crops at 16 kHz (mostly past their file's end: Whisper's zero padding) against WhisperFeatureExtractor on
    each row of the crop output: within twice the Whisper tolerance, once for the batch's float32 STFT and once for the
    extractor's own (tests/test_mel_norm_spec.py)."""
    tf = pytest.importorskip("transformers")
    fe = tf.WhisperFeatureExtractor(feature_size=n_mels)
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    R, L = 16000, 480000
    files, offsets = [0, 3, 4, 6], [0, 1000, 0, 17]
    crops = corpus.crops(len(files), L, sample_rate=R)
    nb = corpus.mel_crops(len(files), L, R, n_fft=400, hop_length=160, n_mels=n_mels, mel_scale="slaney",
                          norm="slaney", log_floor=FLOOR, normalize="whisper")
    assert nb.n_frames == 3000
    x, _ = crops(files, offsets)
    y, _ = nb(files, offsets)
    x, y, p = x.cpu().numpy(), y.cpu().numpy(), nb.params
    for b in range(len(files)):
        for c in range(idx[files[b]].info.channels):
            hf = fe(x[b, c], sampling_rate=R, return_tensors="np")["input_features"][0]
            ref = S.mel(x[b, c], p.n_fft, p.hop_length, nb.window, nb.fbank, True, FLOOR)
            D = N.log_bound(ref, S.bound(x[b, c], p.n_fft, p.hop_length, nb.window, nb.fbank, True), FLOOR)
            tol = 2 * N.whisper_tol(hf, D[:, :-1].max())  # the batch's float32 STFT, and the extractor's
            err = np.abs(y[b, c].astype(np.float64) - hf)
            assert (err <= tol).all(), (b, c, float((err / tol).max()))


# --------------------------------------------------------------------------- 3. determinism, requests, corpora, launches

@gpu
def test_bit_identical_calls(rctx):
    import torch
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    L, R = 8000, 16000
    files, offsets = edge_requests(idx, L, R)
    rng = np.random.default_rng(2)
    pf, po, pl = requests(idx, lambda r: int(r.integers(100, 9000)), rng, R)
    T = span(idx, pf, po, pl, R)
    for make, args in ((lambda nz: corpus.mel_crops(len(files), L, R, log_floor=FLOOR, normalize=nz),
                        (files, offsets)),
                       (lambda nz: corpus.mel_packed(len(pf), T, R, log_floor=FLOOR, normalize=nz), (pf, po, pl))):
        for normalize in (("per_feature", "whisper") if len(args) == 2 else ("per_feature",)):
            nb = make(normalize)
            a = nb(*args)[0].clone()
            assert torch.equal(nb(*args)[0].view(torch.int32), a.view(torch.int32))
            nb(*[v[::-1] for v in args])
            assert torch.equal(nb(*args)[0].view(torch.int32), a.view(torch.int32))
            assert torch.equal(make(normalize)(*args)[0].view(torch.int32), a.view(torch.int32))


@gpu
def test_device_drawn_requests_without_sync(rctx):
    """Requests drawn on the GPU, check=False under sync debug mode "error", crop and packed batches interleaved."""
    import torch
    idx = cb.index(mixed_files())
    corpus = cb.Corpus(idx, rctx)
    R = 16000
    nt = torch.tensor(lengths_at(idx, R), device="cuda")
    pairs = [crops_pair(corpus, 12, 20000, R, "per_feature"), crops_pair(corpus, 9, 777, R, "whisper", n_fft=512,
                                                                           hop_length=100, n_mels=40)]
    packed = (corpus.mel_packed(10, 60000, R, log_floor=FLOOR, normalize="per_feature"),
              corpus.mel_packed(10, 60000, R, log_floor=FLOOR))
    gen = torch.Generator(device="cuda").manual_seed(7)
    draws = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            for nb, _ in pairs:
                fi = torch.randint(0, len(idx), (nb.batch,), device="cuda", generator=gen)
                off = torch.minimum((torch.rand(nb.batch, device="cuda", generator=gen) * (nt[fi] + 1)).long(), nt[fi])
                nb(fi, off, check=False)
                draws.append((nb, fi, off, nb.out.clone()))
            fi = torch.randint(0, len(idx), (10,), device="cuda", generator=gen)
            ln = torch.randint(1, 6000, (10,), device="cuda", generator=gen)
            y = packed[0](fi, None, ln, check=False)[0].clone()
            draws.append((packed[0], fi, ln, y))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for nb, fi, arg, y in draws:
        if nb is packed[0]:
            z = packed[1](fi, None, arg, check=False)
            x, s, f = z[0].cpu().numpy(), z[1].tolist(), z[2].tolist()
            ref = np.zeros(x.shape)
            for st, F in zip(s, f):
                ref[:, :, st:st + F] = N.per_feature(x[:, :, st:st + F], F)
            N.within_ulp(y.cpu().numpy(), ref)
            continue
        plain = next(p for n, p in pairs if n is nb)
        x, lengths = plain(fi, arg, check=False)
        x = x.cpu().numpy()
        if nb.normalize == "whisper":
            ref = N.whisper(x[..., :-1])
        else:
            hop = nb.params.hop_length
            ref = np.stack([N.per_feature(x[b], v) for b, v in enumerate(crop_valid(lengths.tolist(), hop))])
        N.within_ulp(y.cpu().numpy(), ref)


@gpu
def test_host_corpus(rctx):
    """A host corpus gives a device corpus's normalised features bit for bit."""
    import torch
    idx = cb.index(mixed_files())
    L, R = 5000, 16000
    files, offsets = edge_requests(idx, L, R)
    rng = np.random.default_rng(4)
    pf, po, pl = requests(idx, lambda r: int(r.integers(100, 9000)), rng, R)
    T = span(idx, pf, po, pl, R)
    got = []
    for memory in ("device", "host"):
        c = cb.Corpus(idx, rctx, memory=memory)
        got.append([c.mel_crops(len(files), L, R, log_floor=FLOOR, normalize=nz)(files, offsets)[0].clone()
                    for nz in ("per_feature", "whisper")]
                   + [c.mel_packed(len(pf), T, R, log_floor=FLOOR, normalize="per_feature")(pf, po, pl)[0].clone()])
        gc.collect()
    for a, b in zip(*got):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@gpu
def test_launch_counts(rctx):
    """A normalised call launches what the unnormalised one launches, plus mel_norm_kernel."""
    idx = cb.index(mixed_files())

    def per_call(batch, *args):
        batch(*args, check=False)
        n0 = rctx.launch_count
        batch(*args, check=False)
        return rctx.launch_count - n0

    B, L = 7, 5000
    for c in (cb.Corpus(idx, rctx), cb.Corpus(idx, rctx, memory="host")):
        req = (list(range(B)), [0] * B)
        base = per_call(c.mel_crops(B, L, 16000, log_floor=FLOOR), *req)
        for nz in ("per_feature", "whisper"):
            assert per_call(c.mel_crops(B, L, 16000, log_floor=FLOOR, normalize=nz), *req) == base + 1
        preq = (list(range(B)), None, [3000] * B)
        base = per_call(c.mel_packed(B, 30000, 16000, log_floor=FLOOR), *preq)
        assert per_call(c.mel_packed(B, 30000, 16000, log_floor=FLOOR, normalize="per_feature"), *preq) == base + 1


# --------------------------------------------------------------------------- 4. refusals

@gpu
def test_refusals(rctx):
    Lb = rctx._L
    idx = cb.index(mixed_files()[:3])
    corpus = cb.Corpus(idx, rctx)
    rates = np.array([f.info.sample_rate for f in idx.files], np.uint32)
    CL = cb.MEL_CENTER | cb.MEL_LOG
    PF, WH = cb.MEL_NORM_PER_FEATURE, cb.MEL_NORM_WHISPER
    b = C.c_void_p()

    def create(packed=False, flags=CL | PF, log_floor=FLOOR, n_fft=400, hop=160, n_mels=80, L=1000, n=4):
        mp = cb._lib.MelParams(n_fft, n_fft, hop, n_mels, flags, log_floor)
        w = np.ones(n_fft, np.float32)
        fb = np.ones((n_fft // 2 + 1, n_mels), np.float32)
        fn = Lb.clx_batch_create_mel_packed if packed else Lb.clx_batch_create_mel_crops
        rc = fn(rctx._h, corpus._h, rates.ctypes.data, 3, n, L, 16000, C.byref(mp), w.ctypes.data, fb.ctypes.data,
                C.byref(b))
        if rc == 0:
            Lb.clx_batch_destroy(rctx._h, b)
        else:
            assert not b.value
        return rc

    for packed in (False, True):
        assert create(packed) == 0
        for kw in (dict(flags=PF, log_floor=0.0), dict(flags=cb.MEL_CENTER | PF, log_floor=0.0),
                   dict(flags=cb.MEL_LOG | PF), dict(flags=cb.MEL_LOG | WH), dict(flags=WH, log_floor=0.0),
                   dict(flags=CL | PF | WH), dict(flags=CL | 16)):
            assert create(packed, **kw) == 90, (packed, kw)
    assert create(flags=CL | WH) == 0
    assert create(True, flags=CL | WH) == 90  # Whisper on a packed batch
    assert create(flags=CL | WH, n_fft=400, hop=160, L=201) == 0  # F = 2: one frame left
    assert create(flags=CL | WH, n_fft=400, hop=400, L=399) == 90  # F = 1
    assert create(flags=CL | PF, n_fft=400, hop=400, L=399) == 0
    assert create(flags=CL | PF, n_mels=512, n=1 << 22, L=1000) == 90  # 2^32 (crop, row, mel) segments
    assert create(True, flags=CL | PF, n_mels=512, n=1 << 22, L=1000) == 90
    with pytest.raises(ValueError, match="log_floor"):
        corpus.mel_crops(4, 1000, 16000, normalize="per_feature")
    with pytest.raises(ValueError, match="center"):
        corpus.mel_crops(4, 1000, 16000, log_floor=FLOOR, center=False, normalize="whisper")
    with pytest.raises(ValueError, match="normalize must be"):
        corpus.mel_packed(4, 1000, 16000, log_floor=FLOOR, normalize="whisper_v3")
    with pytest.raises(ValueError, match="crop batches"):
        corpus.mel_packed(4, 1000, 16000, log_floor=FLOOR, normalize="whisper")
