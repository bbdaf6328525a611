"""The normalised log-mel spec (tests/spec_mel_norm.py) against the implementations it restates, the Python refusals
of normalize=, and clx_mel_packed_frames_bound with the normalisation flags (CPU only).

* Whisper: spec_mel.mel of the zero-padded 30 s input, its last frame dropped, then spec_mel_norm.whisper, against
  transformers.WhisperFeatureExtractor (skipped when transformers is absent).  That extractor computes its STFT in
  float32, the spec in float64, so they agree within the tolerance the device batch is held to: spec_mel_norm's
  Whisper bound from spec_mel's float32 power bound (about 1e-6 to 2e-5 measured, against a range of about 2).
* Per feature: spec_mel_norm.per_feature against a torch float64 restatement of NeMo's normalize_batch(x, seq_len,
  "per_feature") followed by NeMo's zero fill of the frames past seq_len.
"""

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import _lib
from tests import spec_mel as S
from tests import spec_mel_norm as N
from tests.test_mel_packed_bound import bound, params


# --------------------------------------------------------------------------- 1. Whisper

def whisper_features(x, n_mels):
    """The spec's Whisper features of one waveform x (at most 30 s at 16 kHz), [n_mels, 3000], and their tolerance
    for a float32 STFT."""
    import torch
    xp = np.zeros((1, 480000), np.float32)
    xp[0, :x.size] = x
    fb = cb.melscale_fbanks(201, 0.0, 8000.0, n_mels, 16000, "slaney", "slaney")
    w = torch.hann_window(400).numpy()
    ref = S.mel(xp, 400, 160, w, fb, True, 1e-10)[0][:, :-1]
    D = N.log_bound(ref, S.bound(xp, 400, 160, w, fb, True)[0][:, :-1], 1e-10)
    y = N.whisper(ref)
    return y, N.whisper_tol(y, D.max())


@pytest.mark.parametrize("n_mels", [80, 128])
def test_whisper_map_matches_whisper_feature_extractor(n_mels):
    tf = pytest.importorskip("transformers")
    fe = tf.WhisperFeatureExtractor(feature_size=n_mels)
    rng = np.random.default_rng(n_mels)
    signals = [(rng.standard_normal(480000) * 0.1).astype(np.float32),  # a full window
               (rng.standard_normal(16000 * 3 + 77) * 0.5).astype(np.float32),  # short files, zero-padded to 30 s
               np.sin(np.arange(4000) * 0.3).astype(np.float32) * 0.01,
               np.zeros(1000, np.float32)]  # silence: a constant row
    for x in signals:
        hf = fe(x, sampling_rate=16000, return_tensors="np")["input_features"][0]
        y, tol = whisper_features(x, n_mels)
        assert y.shape == hf.shape == (n_mels, 3000)
        N.check(hf, y, tol)


def test_whisper_map_edges():
    """The clamp sits 8 below the row's maximum in log10, each row on its own; a constant row maps to (l + 4) / 4."""
    x = np.full((2, 3, 4), np.log(1e-10))
    x[0, 1, 2] = np.log(1e3)
    y = N.whisper(x)
    assert y[0, 1, 2] == pytest.approx((3 + 4) / 4) and np.allclose(np.delete(y[0].ravel(), 6), (3 - 8 + 4) / 4)
    assert np.allclose(y[1], (-10 + 4) / 4)


# --------------------------------------------------------------------------- 2. per feature

def nemo_normalize_batch(x, seq_len):
    """NeMo's normalize_batch(x, seq_len, "per_feature") over x [B, n_mels, T], then the zero fill of the frames past
    seq_len that NeMo's filterbank applies after it, in torch float64."""
    import torch
    B, T = x.shape[0], x.shape[2]
    valid = torch.arange(T).unsqueeze(0).expand(B, T) < seq_len.unsqueeze(1)
    den = valid.sum(axis=1)
    mean = torch.where(valid.unsqueeze(1), x, 0.0).sum(axis=2) / den.unsqueeze(1)
    std = torch.sqrt(torch.sum(torch.where(valid.unsqueeze(1), x - mean.unsqueeze(2), 0.0) ** 2, axis=2)
                     / (den.unsqueeze(1) - 1.0))
    std = std.masked_fill(std.isnan(), 0.0) + 1e-5
    y = (x - mean.unsqueeze(2)) / std.unsqueeze(2)
    return y.masked_fill(~valid.unsqueeze(1), 0.0)


def test_per_feature_map_matches_nemo():
    import torch
    rng = np.random.default_rng(3)
    T = 37
    lens = [T, 1, 2, 17, 36]
    x = rng.standard_normal((len(lens), 5, T)) * 3.0 - 10.0
    x[2, 1] = -23.0  # a constant feature: exactly 0
    want = nemo_normalize_batch(torch.from_numpy(x), torch.tensor(lens)).numpy()
    for b, v in enumerate(lens):
        got = N.per_feature(x[b], v)
        np.testing.assert_allclose(got, want[b], rtol=1e-12, atol=1e-12)
        assert (got[:, v:] == 0).all()
    assert (N.per_feature(x[2], 2)[1] == 0).all() and (N.per_feature(x[0], 0) == 0).all()


# --------------------------------------------------------------------------- 3. refusals, the frames bound

def test_python_refusals():
    args = (16000, 400, None, 160, 0.0, None, 80, None, None)
    for kw, msg in ((dict(center=True, log_floor=None, normalize="per_feature"), "log_floor"),
                    (dict(center=False, log_floor=1e-10, normalize="whisper"), "center"),
                    (dict(center=True, log_floor=1e-10, normalize="nemo"), "normalize must be"),
                    (dict(center=True, log_floor=1e-10, normalize="PER_FEATURE"), "normalize must be")):
        with pytest.raises(ValueError, match=msg):
            cb._mel_tables(*args, kw["center"], "slaney", "slaney", kw["log_floor"], kw["normalize"])
    for normalize, flag in ((None, 0), ("per_feature", cb.MEL_NORM_PER_FEATURE), ("whisper", cb.MEL_NORM_WHISPER)):
        p, _, _ = cb._mel_tables(*args, True, "slaney", "slaney", 1e-10, normalize)
        assert p.flags == cb.MEL_CENTER | cb.MEL_LOG | flag
    with pytest.raises(ValueError, match="crop batches"):
        cb.MelPackedBatch(None, 4, 1000, log_floor=1e-10, normalize="whisper")
    assert (_lib.MEL_NORM_PER_FEATURE, _lib.MEL_NORM_WHISPER) == (4, 8)


def test_frames_bound_with_each_flag():
    lib = _lib.load()
    LOG, CEN = _lib.MEL_LOG, _lib.MEL_CENTER
    PF, WH = _lib.MEL_NORM_PER_FEATURE, _lib.MEL_NORM_WHISPER
    for B, T in ((4, 201), (25, 4_800_000), (3, 1000)):
        plain = bound(lib, params(flags=LOG | CEN, log_floor=1e-10), B, T)
        assert plain > 0
        assert bound(lib, params(flags=LOG | CEN | PF, log_floor=1e-10), B, T) == plain
        assert bound(lib, params(flags=LOG | CEN | WH, log_floor=1e-10), B, T) == 0
    for flags, floor in ((PF, 0.0), (WH, 0.0), (CEN | PF, 0.0), (CEN | WH, 0.0), (LOG | PF, 1e-10), (LOG | WH, 1e-10),
                         (LOG | CEN | PF | WH, 1e-10), (CEN | LOG | 16, 1e-10), (PF, 1e-10)):
        assert bound(lib, params(flags=flags, log_floor=floor), 4, 1000) == 0, flags
