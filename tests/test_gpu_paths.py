"""Which kernel decoded each frame (-m gpu).

The parity suite runs the product's launch sequence, in which the generic kernel re-decodes whatever a fast path
declined and the i64 second chance redoes what the i32 accumulator could not vouch for: it proves "fast path or
fallback".  Here the fallbacks are switched off (Context(no_generic=True, no_wide=True)), so every verdict of the
lane-per-frame path (clx_fused.cu) and the warp-per-frame path (clx_coop.cu) is seen as it is, and checked against
the rule of tests/fastpath.py: a valid frame that keeps its nominal width is decoded by the fast path itself,
bit-exact; anything it declines is accounted for.
"""
import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import synth
from oracle import oracle as O
from tests import fastpath as F
from tests.test_gpu_parity import SYNTH_CASES

pytestmark = pytest.mark.gpu

PATHS = {"seq": dict(lane_per_frame=True), "warp": dict(warp_per_frame=True)}


@pytest.fixture(scope="module", params=sorted(PATHS))
def fast(request):
    """(path, context without fallbacks, context with the i64 second chance but no generic kernel)"""
    c = cb.Context(device=0, no_generic=True, no_wide=True, **PATHS[request.param])
    c2 = cb.Context(device=0, no_generic=True, **PATHS[request.param])
    yield request.param, c, c2
    c.close()
    c2.close()


def oracle(data, descs, lengths, out_elems, verify=True):
    bad, st, ref = O.decode_batch(data, descs["byte_offset"], lengths, descs["out_offset"], out_elems, n_threads=8,
                                  verify_crc=verify)
    return st, ref


def run_both_ways(path, ctx, data, descs, lengths, out_elems, wide_ran=False):
    """The rule through a host-buffer call and through a resident batch; returns the verdict counts of the latter."""
    st, ref = oracle(data, descs, lengths, out_elems)
    out, res = ctx.decode_frames(data, descs, out_elems=out_elems)
    F.check_fast_path(path, data, descs, lengths, res, out, st, ref, wide_ran)
    dev = ctx.upload(data, descs, out_elems)
    dev.decode(0)
    out2, res2 = dev.read()
    dev.close()
    return F.check_fast_path(path, data, descs, lengths, res2, out2, st, ref, wide_ran)


def run_batch(path, ctx, b, wide_ran=False):
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    return run_both_ways(path, ctx, b.data, descs, b.frame_lengths, out_elems, wide_ran)


@pytest.mark.parametrize("case", sorted(SYNTH_CASES))
def test_fast_path_decodes_synthetic_cases_alone(fast, case):
    path, c, _ = fast
    run_batch(path, c, synth.generate(SYNTH_CASES[case]))


@pytest.mark.parametrize("seed", range(6))
def test_fast_path_decodes_random_configs_alone(fast, seed):
    """The six configurations of test_random_configs_vs_oracle (same seeds)."""
    rng = np.random.default_rng(1000 + seed)
    nch = int(rng.integers(1, 9))
    cfg = synth.SynthConfig(
        seed=int(rng.integers(1, 2**31)), n_frames=int(rng.integers(1, 200)),
        block_size=int(rng.choice([16, 192, 576, 1000, 1152, 2304, 4096, 4608, int(rng.integers(1, 9000))])),
        n_channels=nch, bps=int(rng.choice([8, 12, 16, 20, 24])), stereo_mode=-1 if nch == 2 else 0,
        type_mask=int(rng.integers(1, 16)), lpc_min_order=1, lpc_max_order=int(rng.integers(1, 33)),
        qlp_precision=0, rice_mode=int(rng.choice([-1, -2])), rice_kmin=0, rice_kmax=14,
        max_porder=int(rng.integers(0, 8)), rice2=int(rng.integers(0, 3)), wasted_max=int(rng.integers(0, 6)),
        long_unary_per_mille=int(rng.choice([0, 50])))
    path, c, _ = fast
    run_batch(path, c, synth.generate(cfg))


def test_fast_path_decodes_golden_frames_alone(fast, golden):
    """The frames of the reference's test streams (fixed-4, LPC up to order 20 in non_subset, Rice2, wasted bits)."""
    path, c, _ = fast
    for name in ("pop", "short", "wasted_bits", "non_subset", "empty_vorbis_comment", "repeated_vorbis_comment"):
        data = golden[f"{name}__bytes"]
        rows = [r for r in golden[f"{name}__frames"] if r[1] == 0 and r[3] > 0]
        offs = np.array([int(r[0]) for r in rows], np.uint64)
        lens = np.array([int(r[3]) for r in rows], np.uint32)
        descs, out_elems = cb.descs_from_offsets(data, offs, lens)
        run_both_ways(path, c, data, descs, lens, out_elems)


def test_fast_path_decodes_c2_full_size_alone(fast):
    path, c, _ = fast
    v = run_batch(path, c, synth.workload("c2"))
    assert v.declined == 0 and v.out_of_width == 0


def test_fast_path_c4_slice_out_of_width_frames(fast):
    """C4's forced Rice parameters code some 16-bit samples outside 16 bits: those frames may be declined, every
    other one must not be."""
    path, c, c2 = fast
    b = synth.workload("c4", 1100)
    v = run_batch(path, c, b)
    assert v.out_of_width > 0  # the slice really holds such frames
    run_batch(path, c2, b, wide_ran=True)


def test_fast_paths_never_accept_what_the_oracle_rejects(fast):
    """The 600-frame corruption corpus of test_corrupted_frames_status_parity under no_generic + no_wide, with and
    without CRC checks: a fast path either declines a damaged frame or reports the oracle's own status."""
    path = fast[0]
    base = synth.generate(synth.SynthConfig(n_frames=40, block_size=576, n_channels=2, bps=16, stereo_mode=-1,
                                           type_mask=15, lpc_min_order=1, lpc_max_order=32, qlp_precision=0,
                                           rice_mode=-1, max_porder=4, rice2=2, wasted_max=4))
    rng = np.random.default_rng(42)
    frames = []
    for trial in range(600):
        i = int(rng.integers(0, base.n_frames))
        f = base.data[int(base.frame_offsets[i]):int(base.frame_offsets[i + 1])].copy()
        kind = trial % 3
        if kind == 0:
            for _ in range(int(rng.integers(1, 4))):
                p = int(rng.integers(5, min(f.size, 60)))
                f[p] ^= 1 << int(rng.integers(0, 8))
        elif kind == 1:
            for _ in range(int(rng.integers(1, 3))):
                f[int(rng.integers(5, f.size))] ^= 1 << int(rng.integers(0, 8))
        else:
            f = f[: int(rng.integers(6, f.size))]
        st, d = cb.parse_frame_header(f)
        if st != 0:
            continue
        frames.append(f)
    data = np.concatenate(frames)
    lengths = np.array([f.size for f in frames], dtype=np.uint32)
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.uint64)
    rejected = 0
    for verify in (False, True):
        c = cb.Context(device=0, verify_crc=verify, no_generic=True, no_wide=True, **PATHS[path])
        descs, out_elems = cb.descs_from_offsets(data, offsets, lengths, flags=0 if verify else 1)
        st, ref = oracle(data, descs, lengths, out_elems, verify)
        # a damaged frame the oracle still accepts may end before the bytes it was given
        consumed = np.array([O.decode_frame(f, verify_crc=verify).info.consumed if s == 0 else 0
                             for f, s in zip(frames, st)], dtype=np.uint32)
        out, res = c.decode_frames(data, descs, out_elems=out_elems)
        v = F.check_fast_path(path, data, descs, consumed, res, out, st, ref, wide_ran=False)
        assert v.declined > 0
        rejected += int((st != 0).sum())
        c.close()
    assert rejected > 100


OVERFLOW_CONFIGS = {
    # test_wrapping_arithmetic_parity: 24-bit, every stereo mode, Rice2 residuals near 2^28: samples wrap i32
    "wrapping": synth.SynthConfig(n_frames=24, block_size=512, n_channels=2, bps=24, stereo_mode=-1, type_mask=12,
                                  lpc_min_order=1, lpc_max_order=12, qlp_precision=15, rice_mode=-2, rice_kmin=26,
                                  rice_kmax=29, rice2=1, residual_mean=3.0e8, max_porder=2),
    # test_narrow_accumulator_shortcut_is_verified: small coefficients pick the i32 accumulator, samples beyond 2^29
    "narrow-shortcut": synth.SynthConfig(n_frames=16, block_size=1024, n_channels=2, bps=16, stereo_mode=0, type_mask=8,
                                         lpc_min_order=1, lpc_max_order=8, qlp_precision=5, rice_mode=-2, rice_kmin=26,
                                         rice_kmax=29, rice2=1, residual_mean=2.0e8, max_porder=1),
}


@pytest.mark.parametrize("name", sorted(OVERFLOW_CONFIGS))
def test_wide_second_chance_output(name):
    """The i64 second chance (decode_subframes_kernel<*, true>) on its own.  "narrow-shortcut": the first pass must
    hand some frames to it (-3); with it running and the generic kernel still off, each of those frames must come
    back 0 and bit-exact from the WIDE instances — or -2 when a mid/side subframe signal reaches 2^29.
    "wrapping": its 15-bit LPC coefficients send every warp straight to the i64 body, so the first pass leaves
    nothing to the second chance; what it declines is exactly the mid/side frames at the 2^29 bound."""
    b = synth.generate(OVERFLOW_CONFIGS[name])
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    st, ref = oracle(b.data, descs, b.frame_lengths, out_elems)
    assert (st == 0).all()
    c1 = cb.Context(device=0, lane_per_frame=True, no_generic=True, no_wide=True)
    c2 = cb.Context(device=0, lane_per_frame=True, no_generic=True)
    for resident in (False, True):
        got = []
        for c in (c1, c2):
            if resident:
                dev = c.upload(b.data, descs, out_elems)
                dev.decode(0)
                got.append(dev.read())
                dev.close()
            else:
                got.append(c.decode_frames(b.data, descs, out_elems=out_elems))
        (out1, res1), (out2, res2) = got
        F.check_fast_path("seq", b.data, descs, b.frame_lengths, res1, out1, st, ref, wide_ran=False)
        F.check_fast_path("seq", b.data, descs, b.frame_lengths, res2, out2, st, ref, wide_ran=True)
        bound = np.array([F.mid_side_beyond_bound(d, F.subframe_signals(b.data, d)) for d in descs])
        wide = np.nonzero(res1["status"] == F.NEED_WIDE)[0]
        if name == "wrapping":
            assert wide.size == 0 and bound.any(), (name, resident, res1["status"])
            assert np.array_equal(res1["status"], np.where(bound, F.NEED_GENERIC, 0)), (name, resident)
            continue
        assert wide.size > 0, (name, resident, res1["status"])
        for i in wide:
            assert int(res2["status"][i]) == (F.NEED_GENERIC if bound[i] else 0), (name, resident, i)
        assert (res2["status"][wide] == 0).any()  # the WIDE instances' own output was compared
    c1.close()
    c2.close()
