"""tests/spec_excerpts.py: the restated excerpt plan on hand-worked cases, and its checkers against mutated outputs.

The GPU tests of tests/test_gpu_many_excerpts.py hold whole outputs of thousands of excerpts to these checkers; the
mutations below are the mistakes a dropped or doubled carry between the planners' 1024-excerpt chunks would make, and
each one must be rejected, so that those GPU checks cannot pass vacuously.
"""
import numpy as np
import pytest

from tests import spec_excerpts as X
from tests import spec_mel_norm as MN

INV = X.ERR_INVALID


def word(b, status=INV, kind=0):
    return (kind << 62) | (b << 32) | status


# --------------------------------------------------------------------------- the restatement, by hand

def test_exact_fit_and_one_sample_over():
    Ns = [10, 7]
    files, offsets, lengths = [0, 1, 2, 0, 1], [0, 2, 0, 10, 0], [5, -1, 3, 3, 3]
    # starts: 0; 0 + r4(5) = 8; invalid (file 2) takes nothing: 16; empty at N: 16; 16
    p = X.packed_plan(files, offsets, lengths, Ns, T=19)
    assert p.starts == [0, 8, 16, 16, 16]
    assert p.lengths == [5, 5, 0, 0, 3] and p.status == [0, 0, INV, 0, 0]
    assert p.error == word(2) and p.end == 19  # min(16 + 4, T)
    p = X.packed_plan(files, offsets, lengths, Ns, T=18)  # the last one ends one column past T
    assert p.starts == [0, 8, 16, 16, 16]
    assert p.lengths == [5, 5, 0, 0, 0] and p.status == [0, 0, INV, 0, INV]
    assert p.error == word(2) and p.end == 16


def test_non_fit_refuses_every_later_excerpt():
    """Excerpts that fit are a prefix of the valid ones: after a non-fit even an empty or a 1-sample one is refused,
    and the non-fitting ones still advance the starts."""
    Ns = [100]
    p = X.packed_plan([0, 0, 0, 0], [0, 0, 0, 100], [8, 5, 1, 1], Ns, T=10)
    assert p.starts == [0, 8, 16, 20]
    assert p.lengths == [8, 0, 0, 0] and p.status == [0, INV, INV, INV] and p.error == word(1)
    assert p.end == 8


def test_invalid_requests_between_valid_ones():
    Ns = [10, 7]
    files = [0, 1 << 32, 0, 0, 0, 1, 0, 2, -1, 1]
    offsets = [1, 0, -1, 0, 0, 8, 11, 0, 0, 7]
    lengths = [2, 1, 1, 0, -2, 1, 1, 1, 1, -1]
    p = X.packed_plan(files, offsets, lengths, Ns, T=100)
    bad = [1, 2, 3, 4, 5, 6, 7, 8]  # reserved bits, offset -1, length 0, length -2, offset past N (twice), files
    assert [b for b, s in enumerate(p.status) if s] == bad
    assert p.lengths == [2] + [0] * 8 + [0]  # the last one: the empty excerpt at N, valid
    assert p.starts == [0] + [4] * 9 and p.error == word(1)


def test_count_below_max_excerpts():
    Ns = [10]
    files, offsets, lengths = [0] * 6, [0] * 6, [3, 3, 3, 3, 99, 99]
    p = X.packed_plan(files, offsets, lengths, Ns, T=8, count=2)
    assert p.starts == [0, 4] and p.lengths == [3, 3] and p.status == [0, 0]
    assert p.error == X.NO_ERROR and p.end == 8
    # the unused excerpts 2 .. 5 of a batch of 6: length 0 and status 0, whatever the requests there say
    q = X.packed_plan(files, offsets, lengths, Ns, T=8, count=2, max_excerpts=6)
    assert q.starts == [0, 4] and q.lengths == [3, 3, 0, 0, 0, 0] and q.status == [0] * 6 and q.error == p.error
    X.check_plan(q, [0, 4], [3, 3, 0, 0, 0, 0], [0] * 6, -1)
    with pytest.raises(AssertionError, match="lengths"):  # what a full call left in an unused excerpt
        X.check_plan(q, [0, 4], [3, 3, 0, 3, 0, 0], [0] * 6, -1)
    with pytest.raises(AssertionError, match="status"):
        X.check_plan(q, [0, 4], [3, 3, 0, 0, 0, 0], [0, 0, 0, 0, INV, 0], -1)


def test_rates_crops_and_mel_frames():
    assert X.length_at(10, 48000, 16000) == 4 and X.length_at(10, 24000, 16000) == 7
    assert X.length_at(10, 16000, 16000) == 10 and X.length_at(10, 44100, None) == 10
    c = X.crop_plan([0, 1, 0, 3], [8, 7, 11, 0], 5, [10, 7])
    assert c.lengths == [2, 0, 0, 0] and c.status == [0, 0, INV, INV] and c.error == word(2)
    # n_fft 8, hop 4, centred: a frame needs n > 4
    m = X.mel_plan(X.Plan([0] * 5, [5, 0, 9, 4, 1], [0] * 5, X.NO_ERROR), 8, 4)
    assert m.lengths == [2, 0, 3, 0, 0] and m.starts == [0, 4, 4, 8, 8] and m.end == 8
    assert X.mel_frame_count(8, 8, 4, False) == 1 and X.mel_frame_count(7, 8, 4, False) == 0


def test_error_word_order():
    assert X.error_word([(0, 2048, INV), (0, 1023, INV)]) == word(1023)
    assert X.error_word([(1, 3, -3), (0, 2000, INV)]) == word(2000)
    assert X.error_word([]) == X.NO_ERROR


# --------------------------------------------------------------------------- the checkers reject mutated outputs

def many(B=2100, seed=0):
    """A packed call of B excerpts of 1 to 9 samples of three small files, invalid ones at the chunk edges 1023 and
    2048, excerpts 1500 and 1501 of equal length from different files; its plan, PCM and the correct output."""
    rng = np.random.default_rng(seed)
    pcm = [rng.integers(-1000, 1000, (c, 50)).astype(np.int32) for c in (1, 2, 4)]
    Ns = [50, 50, 50]
    files = rng.integers(0, 3, B)
    lengths = rng.integers(1, 10, B)
    offsets = np.array([int(rng.integers(0, 50 - n + 1)) for n in lengths])
    files[[1023, 2048]] = 7
    files[1500], files[1501], lengths[1500], lengths[1501] = 1, 2, 5, 5
    T = sum(X.r4(int(n)) for n in lengths) + 8
    p = X.packed_plan(files, offsets, lengths, Ns, T)
    out = X.expected_packed(p, files, offsets, pcm, 4, T)
    return p, files, offsets, lengths, pcm, Ns, T, out


def test_correct_output_passes():
    p, files, offsets, lengths, pcm, Ns, T, out = many()
    X.check_plan(p, p.starts, p.lengths, p.status, word(1023))
    X.check_plan(X.packed_plan([], [], [], Ns, T), [], [], [], -1)  # no failure: all ones, read as int64 -1
    X.check_exact(out.copy(), out)


def test_starts_shifted_from_1024_rejected():
    p, files, offsets, lengths, pcm, Ns, T, out = many()
    shifted = X.Plan(p.starts[:1024] + [s + 4 for s in p.starts[1024:]], p.lengths, p.status, p.error)
    dev = X.expected_packed(shifted, files, offsets, pcm, 4, T)
    with pytest.raises(AssertionError, match="starts"):
        X.check_plan(p, shifted.starts, p.lengths, p.status, p.error)
    with pytest.raises(AssertionError):
        X.check_exact(dev, out)


def test_swapped_neighbours_in_second_chunk_rejected():
    p, files, offsets, lengths, pcm, Ns, T, out = many()
    f, o = files.copy(), offsets.copy()
    f[[1500, 1501]], o[[1500, 1501]] = f[[1501, 1500]], o[[1501, 1500]]
    dev = X.expected_packed(p, f, o, pcm, 4, T)  # same starts and lengths, each other's samples
    with pytest.raises(AssertionError):
        X.check_exact(dev, out)


def test_zero_column_past_previous_end_rejected():
    """A long call, then a short one: the short one's output must be 0 from its end to the long one's."""
    p, files, offsets, lengths, pcm, Ns, T, out = many()
    short = X.packed_plan(files[:40], offsets[:40], lengths[:40], Ns, T)
    assert short.end < p.end
    want = X.expected_packed(short, files[:40], offsets[:40], pcm, 4, T)
    dev = want.copy()
    dev[0, (short.end + p.end) // 2] = out[0, (short.end + p.end) // 2] or 1  # what the long call left there
    with pytest.raises(AssertionError):
        X.check_exact(dev, want)


def test_error_word_naming_the_later_failure_rejected():
    p, *_ = many()
    assert p.error == word(1023)
    with pytest.raises(AssertionError, match="error word"):
        X.check_plan(p, p.starts, p.lengths, p.status, word(2048))


def test_lengths_and_status_mutations_rejected():
    p, *_ = many()
    lens, st = list(p.lengths), list(p.status)
    lens[1030] += 1
    st[2049] = INV
    with pytest.raises(AssertionError, match="lengths"):
        X.check_plan(p, p.starts, lens, p.status, p.error)
    with pytest.raises(AssertionError, match="status"):
        X.check_plan(p, p.starts, p.lengths, st, p.error)


def test_stale_crop_tail_past_row_32768_rejected():
    """8200 crops x C 4: the zero pass's rows (b C + c) of crops 8192 and up are past its 32 768 CTAs, cleared on
    its second trip.  A crop there that is short, empty, invalid or of a 1-channel file keeps samples of an earlier
    call wherever that trip is missing; each such stale element must be rejected."""
    rng = np.random.default_rng(5)
    pcm = [rng.integers(-1000, 1000, (c, 50)).astype(np.int32) for c in (1, 2, 4)]
    Ns, B, L, C_ = [50, 50, 50], 8200, 7, 4
    files = rng.integers(0, 3, B)
    offsets = rng.integers(0, 44, B)
    files[8192:8196], offsets[8192:8196] = [2, 2, 0, 9], [47, 50, 3, 0]  # short, empty, 1 channel, invalid
    assert (B + 1) * C_ > 32768
    p = X.crop_plan(files, offsets, L, Ns)
    assert p.lengths[8192:8196] == [3, 0, 7, 0] and p.status[8195] == INV
    want = X.expected_crops(p, files, offsets, pcm, C_, L)
    X.check_exact(want.copy(), want)
    full = X.expected_crops(X.crop_plan([2] * B, [0] * B, L, Ns), [2] * B, [0] * B, pcm, C_, L)  # an earlier call
    for b, c, t in ((8192, 1, 5), (8193, 0, 0), (8194, 3, 2), (8195, 2, 6)):
        assert want[b, c, t] == 0 and full[b, c, t] != 0
        dev = want.copy()
        dev[b, c, t] = full[b, c, t]
        with pytest.raises(AssertionError):
            X.check_exact(dev, want)


def test_unnormalised_segment_past_2_24_rejected():
    """Crop features of 65 537 crops x 1 row x 256 mels x 2 frames: segment (b C + c) n_mels + m of crop 65 536 is
    past 2^24.  The correct map passes; that one segment left as it was does not."""
    rng = np.random.default_rng(3)
    B, M, F = 65537, 256, 2
    x = rng.uniform(-20.0, -5.0, (B, 1, M, F)).astype(np.float32)
    mu, sigma = MN.stats(x, F)
    y = ((x - mu) / (sigma + MN.EPS)).astype(np.float32)
    valid = np.full(B, F)
    X.per_feature_crops(y, x, valid)
    seg = (B - 1) * M + 3
    assert seg >= 1 << 24
    y[B - 1, 0, 3] = x[B - 1, 0, 3]
    with pytest.raises(AssertionError):
        X.per_feature_crops(y, x, valid)


def test_packed_norm_checker_rejects_mutations():
    rng = np.random.default_rng(4)
    frames = rng.integers(0, 6, 1500)
    frames[1100] = 3
    starts = np.cumsum([0] + [X.r4(int(f)) for f in frames[:-1]])
    Tf = int(starts[-1] + X.r4(int(frames[-1])) + 4)
    x = rng.uniform(-20.0, -5.0, (2, 8, Tf)).astype(np.float32)
    y = np.zeros_like(x)
    for s, f in zip(starts, frames):
        if f:
            y[:, :, s:s + f] = MN.per_feature(x[:, :, s:s + f], int(f)).astype(np.float32)
    X.per_feature_packed(y, x, starts, frames)
    bad = y.copy()
    s = int(starts[1100])
    bad[1, 5, s:s + 3] = x[1, 5, s:s + 3]  # one excerpt's segment left unnormalised
    with pytest.raises(AssertionError):
        X.per_feature_packed(bad, x, starts, frames)
    bad = y.copy()
    bad[0, 0, Tf - 1] = 1.0  # a column after every excerpt
    with pytest.raises(AssertionError, match="outside"):
        X.per_feature_packed(bad, x, starts, frames)


def test_resampled_bound_rejects_a_shift():
    """check_bound with expected_resampled: 0 bound outside excerpts, so a value one column late is caught."""
    refs = [(np.linspace(0.1, 0.5, 20)[None], np.full((1, 20), 1e-7))]
    p = X.packed_plan([0, 0], [0, 5], [5, 6], [20], 20)
    ref, bound = X.expected_resampled(p, [0, 0], [0, 5], refs, 1, 20)
    assert X.check_bound(ref + np.where(bound > 0, 5e-8, 0.0), ref, bound) < 0.6
    with pytest.raises(AssertionError):
        X.check_bound(np.roll(ref, 1, axis=1), ref, bound)
