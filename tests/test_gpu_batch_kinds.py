"""Every kind of batch through the C ABI: what each accessor returns for it, and corpus lifetime (-m gpu).

A batch is one of seven kinds: a batch of frames (clx_batch_create_to), or one of the six corpus kinds.  Wrappers
(resampled and mel batches) run an inner batch, and some accessors of a wrapper return the inner batch's buffer.  A
mel batch wraps a resampled batch, or with the "_plain" suffix a crop or packed batch.  The table below is the header's
contract; each kind is created over a device corpus and a host corpus, every accessor is checked against it, and the
batches are destroyed.
"""
import ctypes as C

import numpy as np
import pytest

import claxon_b200 as cb
from tests.test_gpu_resampled_crops import mixed_files

gpu = pytest.mark.gpu
B, T, R = 4, 4000, 16000
MEL = dict(n_fft=400, win_length=400, hop_length=160, n_mels=80, flags=cb.MEL_CENTER, log_floor=0.0)

# "own": the batch's buffer, "inner": its inner batch's, None: NULL; the stride: 0, or how it is computed.
ACCESSORS = ("crop_requests", "crop_status", "crop_error", "crop_lengths", "packed_requests", "packed_count",
             "packed_starts", "mel_frames")
TABLE = {
    #                   requests status  error    lengths  p.req    p.count  p.starts mel_frames  stride
    "frames":          (None,   None,    None,    None,    None,    None,    None,    None,       "zero"),
    "crops":           ("own",  "own",   "own",   "own",   None,    None,    None,    None,       "zero"),
    "packed":          (None,   "own",   "own",   "own",   "own",   "own",   "own",   None,       "rows"),
    "resampled_crops": ("own",  "inner", "inner", "own",   None,    None,    None,    None,       "zero"),
    "resampled_packed": (None,  "inner", "inner", "own",   "own",   "own",   "own",   None,       "r4"),
    "mel_crops":       ("inner", "inner", "inner", "inner", None,   None,    None,    None,       "zero"),
    "mel_packed":      (None,   "inner", "inner", "inner", "inner", "inner", "own",   "own",      "frames"),
    "mel_crops_plain": ("inner", "inner", "inner", "inner", None,   None,    None,    None,       "zero"),
    "mel_packed_plain": (None,  "inner", "inner", "inner", "inner", "inner", "own",   "own",      "frames"),
}
WRAPPERS = ("resampled_crops", "resampled_packed", "mel_crops", "mel_packed", "mel_crops_plain", "mel_packed_plain")


@pytest.fixture(scope="module")
def rctx():
    c = cb.Context(device=0)
    yield c
    c.close()


def r4(n):
    return (n + 3) // 4 * 4


def create(ctx, corpus, kind, out):
    """Creates one batch of `kind` over `corpus` into `out`; returns the status."""
    L = ctx._L
    rates = np.array([f.info.sample_rate for f in corpus.index.files], np.uint32)
    mp = cb._lib.MelParams(*MEL.values())
    w = np.hanning(MEL["win_length"]).astype(np.float32)
    fb = np.full((MEL["n_fft"] // 2 + 1, MEL["n_mels"]), 0.01, np.float32)
    common = (ctx._h, corpus._h, rates.ctypes.data, len(rates))
    mel = (C.byref(mp), w.ctypes.data, fb.ctypes.data, C.byref(out))
    if kind == "frames":  # the first file's frames, planar
        f = corpus.index.files[0]
        descs = f.descs.copy()
        elems = descs["n_channels"].astype(np.uint64) * descs["block_size"]
        descs["out_offset"] = np.cumsum(elems) - elems
        return L.clx_batch_create_to(ctx._h, f.data.ctypes.data, f.data.size, descs.ctypes.data, descs.size,
                                     int(elems.sum()), 0, cb.OUT_PLANAR_I32, C.byref(out))
    if kind == "crops":
        return L.clx_batch_create_crops(ctx._h, corpus._h, B, T, cb.OUT_CHANNELS_F32, C.byref(out))
    if kind == "packed":
        return L.clx_batch_create_packed(ctx._h, corpus._h, B, T, cb.OUT_CHANNELS_F32, C.byref(out))
    if kind == "resampled_crops":
        return L.clx_batch_create_resampled_crops(*common, B, T, R, C.byref(out))
    if kind == "resampled_packed":
        return L.clx_batch_create_resampled_packed(*common, B, T, R, C.byref(out))
    rate = 0 if kind.endswith("_plain") else R  # mel batches over a crop / packed batch, or a resampled one
    if kind.startswith("mel_crops"):
        return L.clx_batch_create_mel_crops(*common, B, T, rate, *mel)
    return L.clx_batch_create_mel_packed(*common, B, T, rate, *mel)


def want_stride(ctx, corpus, how):
    if how == "zero":
        return 0
    if how == "r4":
        return r4(T)
    if how == "frames":
        mp = cb._lib.MelParams(*MEL.values())
        return int(ctx._L.clx_mel_packed_frames_bound(C.byref(mp), B, T))
    largest = max([192] + [int(f.descs["block_size"].max()) for f in corpus.index.files])  # the filler frame's too
    return r4(T) + r4(min(T, largest))


@gpu
@pytest.mark.parametrize("memory", ["device", "host"])
def test_accessors(rctx, memory):
    """Every accessor of every kind against TABLE: NULL where it says so, and otherwise a buffer of its own,
    distinct from every other buffer the batch hands out; the packed stride; the frame bytes (the corpus's own over a
    device corpus, the batch's staging buffer over a host corpus, NULL for a wrapper)."""
    L = rctx._L
    corpus = cb.Corpus(cb.index(mixed_files()), rctx, memory=memory)
    corpus_bytes, alive = set(), []  # (all alive at once, so that no address is reused)
    for kind, row in TABLE.items():
        b = C.c_void_p()
        alive.append(b)
        assert create(rctx, corpus, kind, b) == 0, kind
        got = {name: getattr(L, f"clx_batch_{name}")(b) for name in ACCESSORS}
        for name, want in zip(ACCESSORS, row):
            assert (got[name] is None) == (want is None), (kind, name, got[name])
        ptrs = [p for p in got.values() if p] + [L.clx_batch_device_out(b)]
        assert all(ptrs) and len(set(ptrs)) == len(ptrs), (kind, got)
        assert L.clx_batch_packed_stride(b) == want_stride(rctx, corpus, row[-1]), kind
        nbytes = L.clx_batch_device_bytes(b)
        if kind in WRAPPERS:
            assert nbytes is None, kind
        else:
            assert nbytes, kind
            if kind != "frames":
                corpus_bytes.add(nbytes)
    for b in alive:
        L.clx_batch_destroy(rctx._h, b)
    # crops and packed: one borrowed buffer over a device corpus, a staging buffer each over a host corpus
    assert len(corpus_bytes) == (1 if memory == "device" else 2)
    for name in ACCESSORS:
        assert getattr(L, f"clx_batch_{name}")(None) is None
    assert L.clx_batch_packed_stride(None) == 0 and L.clx_batch_device_bytes(None) is None
    corpus.close()


@gpu
@pytest.mark.parametrize("memory", ["device", "host"])
def test_corpus_outlives_its_batches(rctx, memory):
    """clx_corpus_destroy refuses while any batch of the corpus is alive, a wrapper and its inner batches included,
    and succeeds once they are destroyed."""
    L = rctx._L
    corpus = cb.Corpus(cb.index(mixed_files()), rctx, memory=memory)
    for kind in TABLE:
        if kind == "frames":
            continue
        b = C.c_void_p()
        assert create(rctx, corpus, kind, b) == 0, kind
        assert L.clx_corpus_destroy(rctx._h, corpus._h) == 90, kind
        L.clx_batch_destroy(rctx._h, b)
    # two wrappers at once, destroyed in creation order
    first, second = C.c_void_p(), C.c_void_p()
    assert create(rctx, corpus, "mel_packed", first) == 0 and create(rctx, corpus, "resampled_crops", second) == 0
    L.clx_batch_destroy(rctx._h, first)
    assert L.clx_corpus_destroy(rctx._h, corpus._h) == 90
    L.clx_batch_destroy(rctx._h, second)
    corpus.close()  # raises unless clx_corpus_destroy succeeds
    assert corpus._h is None
