"""The mel crop batch's reference and host side (CPU): tests/spec_mel.py against torchaudio's MelSpectrogram in float64,
the package's filterbank against torchaudio's melscale_fbanks, and the arguments MelCropBatch refuses before it reaches
the device."""
import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import synth
from tests import spec_mel as S

GRID = [  # n_fft, win_length, hop, center, n_mels, f_min, f_max, mel_scale, norm
    (8, 8, 1, True, 1, 0.0, None, "htk", None),
    (8, 5, 9, False, 1, 0.0, None, "slaney", "slaney"),
    (30, 27, 7, True, 1, 100.0, None, "htk", "slaney"),
    (320, 300, 160, True, 80, 0.0, 7600.0, "slaney", "slaney"),
    (400, 400, 160, True, 128, 0.0, None, "htk", None),
    (400, 301, 400, False, 80, 20.0, None, "htk", None),
    (400, 400, 160, True, 128, 0.0, 8000.0, "slaney", "slaney"),
    (512, 511, 777, True, 128, 0.0, None, "slaney", None),
    (2048, 1024, 512, False, 80, 30.0, 7000.0, "htk", "slaney"),
    (4096, 4096, 4096, True, 128, 0.0, None, "htk", None),
]


@pytest.mark.parametrize("n_fft,win,hop,center,n_mels,f_min,f_max,scale,norm", GRID)
def test_spec_matches_torchaudio(n_fft, win, hop, center, n_mels, f_min, f_max, scale, norm):
    torch = pytest.importorskip("torch")
    T = pytest.importorskip("torchaudio")
    rate = 16000
    rng = np.random.default_rng(n_fft + win + hop)
    L = max(n_fft // 2 + 1, n_fft) + 2 * hop + 13
    x = rng.standard_normal((2, 3, L))
    x[1, 2, L // 2:] = 0.0  # zero columns are transformed like any others
    ms = T.transforms.MelSpectrogram(rate, n_fft=n_fft, win_length=win, hop_length=hop, f_min=f_min, f_max=f_max,
                                     n_mels=n_mels, window_fn=torch.hann_window, center=center, norm=norm,
                                     mel_scale=scale, wkwargs={"dtype": torch.float64}).double()
    with torch.no_grad():
        ref = ms(torch.from_numpy(x)).numpy()
    fb = ms.mel_scale.fb.numpy()
    window = torch.hann_window(win, dtype=torch.float64).numpy()
    got = S.mel(x, n_fft, hop, window, fb, center)
    assert got.shape == ref.shape == (2, 3, n_mels, S.n_frames(L, n_fft, hop, center))
    assert np.allclose(got, ref, rtol=1e-9, atol=1e-9 * ref.max())
    lg = S.mel(x, n_fft, hop, window, fb, center, log_floor=1e-10)
    assert np.allclose(lg, np.log(np.maximum(ref, 1e-10)), rtol=1e-9, atol=1e-9)
    assert (S.bound(x, n_fft, hop, window, fb, center) >= 0).all()


def test_reflect_needs_more_than_half_a_frame():
    torch = pytest.importorskip("torch")
    x = np.ones((1, 200))
    with pytest.raises(ValueError):
        S.frames(x, 400, 160, np.ones(400), True)
    with pytest.raises(RuntimeError):
        torch.stft(torch.ones(1, 200), 400, 160, window=torch.ones(400), center=True, pad_mode="reflect",
                   return_complex=True)
    assert S.frames(np.ones((1, 201)), 400, 160, np.ones(400), True).shape == (1, 2, 400)


@pytest.mark.parametrize("scale", ["htk", "slaney"])
@pytest.mark.parametrize("norm", [None, "slaney"])
@pytest.mark.parametrize("n_freqs,f_min,f_max,n_mels,rate", [(201, 0.0, 8000.0, 128, 16000), (257, 20.0, 7600.0, 80, 16000),
                                                             (1025, 0.0, 22050.0, 128, 44100), (5, 0.0, 4000.0, 1, 8000),
                                                             (2049, 50.0, 11025.0, 512, 22050)])
def test_filterbank_matches_torchaudio(scale, norm, n_freqs, f_min, f_max, n_mels, rate):
    """Against torchaudio computing in float64 (its float32 filterbank is within about 1e-5 of both)."""
    torch = pytest.importorskip("torch")
    F = pytest.importorskip("torchaudio.functional")
    import warnings
    default = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = F.melscale_fbanks(n_freqs, f_min, f_max, n_mels, rate, norm, scale).numpy()
            ref32 = F.melscale_fbanks(n_freqs, f_min, f_max, n_mels, rate, norm, scale).float().numpy()
    finally:
        torch.set_default_dtype(default)
    got = cb.melscale_fbanks(n_freqs, f_min, f_max, n_mels, rate, norm, scale)
    assert got.shape == ref.shape and got.dtype == np.float64
    assert np.allclose(got, ref, rtol=1e-6, atol=1e-6 * np.abs(ref).max())
    assert np.array_equal(got.astype(np.float32), ref32)


def test_python_refusals():
    pytest.importorskip("torch")
    args = dict(n_fft=400, win_length=None, hop_length=None, f_min=0.0, f_max=None, n_mels=128, window_fn=None,
                wkwargs=None, center=True, norm=None, mel_scale="htk", log_floor=None)
    params, window, fbank = cb._mel_tables(16000, **args)
    assert (params.n_fft, params.win_length, params.hop_length, params.n_mels) == (400, 400, 200, 128)
    assert params.flags == cb.MEL_CENTER and params.log_floor == 0.0
    assert window.dtype == np.float32 and window.shape == (400,) and fbank.shape == (201, 128)
    assert fbank.dtype == np.float32 and fbank.flags.c_contiguous
    p, _, _ = cb._mel_tables(16000, **{**args, "log_floor": 1e-10, "center": False})
    assert p.flags == cb.MEL_LOG and p.log_floor == np.float32(1e-10)
    for bad in ({"mel_scale": "kaldi"}, {"norm": "max"}, {"log_floor": 0.0}, {"log_floor": -1.0},
                {"log_floor": float("inf")}, {"log_floor": float("nan")}, {"n_mels": 0}, {"hop_length": 0},
                {"win_length": 0}, {"window_fn": lambda n, **k: np.ones(n + 1)}):
        with pytest.raises(ValueError):
            cb._mel_tables(16000, **{**args, **bad})


def test_filterbank_rate():
    """The filterbank's rate: sample_rate when given, else the corpus's one rate; mixed rates need sample_rate."""
    def flac(rate_code, seed):
        cfg = synth.workload_config("c2", 3, seed)
        cfg.sample_rate_code = rate_code
        b = synth.generate(cfg)
        return np.frombuffer(synth.make_file(b, 0, b.n_frames), np.uint8).copy()
    one = cb.index([flac(9, 1), flac(9, 2)])
    mixed = cb.index([flac(9, 1), flac(10, 2)])
    assert cb._mel_rate(one, None) == 44100 and cb._mel_rate(one, 16000) == 16000
    assert cb._mel_rate(mixed, 16000) == 16000
    with pytest.raises(ValueError, match="2 sample rates"):
        cb._mel_rate(mixed, None)
