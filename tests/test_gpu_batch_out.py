"""Output modes of device-resident batches (-m gpu, except the symbol check).

A resident batch (clx_batch_create_to) keeps its output planar i32 or interleaved little-endian i32 / i24 / i16, the
forms of clx_decode_frames_to.  On the lane-per-frame path the decode kernel writes I32 and I16 itself; the frames
the generic kernel takes over are converted afterwards, and every other path (and I24) converts all frames inside the
batch's graph.  Everything is compared byte for byte with the oracle's or the generator's PCM, laid out on the host,
and with the host-buffer call in the same mode.
"""
import ctypes as C
import hashlib

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import _lib, synth
from oracle import oracle as O
from tests import fastpath as F
from tests.test_gpu_mixed import NARROW_PARTS, PARTS
from tests.test_gpu_parity import SYNTH_CASES

gpu = pytest.mark.gpu

ESIZE = {cb.OUT_INTERLEAVED_I32: 4, cb.OUT_INTERLEAVED_I24: 3, cb.OUT_INTERLEAVED_I16: 2}
MODE_NAMES = {cb.OUT_INTERLEAVED_I32: "i32", cb.OUT_INTERLEAVED_I24: "i24", cb.OUT_INTERLEAVED_I16: "i16"}


def modes_for(descs):
    """The interleaved modes a batch of these frames may use."""
    bps = int(descs["bits_per_sample"].max())
    return [m for m, lim in ((cb.OUT_INTERLEAVED_I32, 32), (cb.OUT_INTERLEAVED_I24, 24), (cb.OUT_INTERLEAVED_I16, 16))
            if bps <= lim]


def expected_bytes(descs, planar, out_elems, mode, frames=None):
    """(bytes, mask): planar i32 samples (caller's layout) re-laid out per frame as interleaved little-endian
    elements of the mode's size (truncated like `sample as i16`), and which bytes belong to a frame."""
    es = ESIZE[mode]
    exp = np.zeros(out_elems * es, np.uint8)
    live = np.zeros(out_elems * es, bool)
    for i in range(descs.size) if frames is None else frames:
        d = descs[i]
        o, nch, bs = int(d["out_offset"]), int(d["n_channels"]), int(d["block_size"])
        exp[o * es:(o + nch * bs) * es] = np.frombuffer(
            synth.interleaved_le_bytes(planar[o:o + nch * bs], nch, 8 * es), np.uint8)
        live[o * es:(o + nch * bs) * es] = True
    return exp, live


def raw(out, out_elems, mode):
    return out.view(np.uint8)[:out_elems * ESIZE[mode]]


def resident(c, data, descs, out_elems, mode, stream=0):
    dev = c.upload(data, descs, out_elems, mode=mode)
    dev.decode(stream)
    out, res = dev.read()
    dev.close()
    return out, res


_oracle_cache = {}


def oracle_of(key, data, descs, lengths, out_elems):
    if key not in _oracle_cache:
        bad, st, ref = O.decode_batch(data, descs["byte_offset"], lengths, descs["out_offset"], out_elems, n_threads=8)
        _oracle_cache[key] = (st, ref)
    return _oracle_cache[key]


def random_config(seed):
    """The six configurations of test_random_configs_vs_oracle (same seeds)."""
    rng = np.random.default_rng(1000 + seed)
    nch = int(rng.integers(1, 9))
    return synth.SynthConfig(
        seed=int(rng.integers(1, 2**31)), n_frames=int(rng.integers(1, 200)),
        block_size=int(rng.choice([16, 192, 576, 1000, 1152, 2304, 4096, 4608, int(rng.integers(1, 9000))])),
        n_channels=nch, bps=int(rng.choice([8, 12, 16, 20, 24])), stereo_mode=-1 if nch == 2 else 0,
        type_mask=int(rng.integers(1, 16)), lpc_min_order=1, lpc_max_order=int(rng.integers(1, 33)),
        qlp_precision=0, rice_mode=int(rng.choice([-1, -2])), rice_kmin=0, rice_kmax=14,
        max_porder=int(rng.integers(0, 8)), rice2=int(rng.integers(0, 3)), wasted_max=int(rng.integers(0, 6)),
        long_unary_per_mille=int(rng.choice([0, 50])))


CASES = {**SYNTH_CASES, **{f"random-{s}": random_config(s) for s in range(6)}}
_streams = {}


def stream(name):
    if name not in _streams:
        _streams[name] = synth.generate(CASES[name])
    return _streams[name]


# --------------------------------------------------------------------------- 1. every path, every mode, every shape

@gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_resident_modes_match_oracle_and_host_call(ctx, case):
    b = stream(case)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    st, ref = oracle_of(case, b.data, descs, b.frame_lengths, out_elems)
    assert (st == 0).all()
    for mode in modes_for(descs):
        exp, live = expected_bytes(descs, ref, out_elems, mode)
        out, res = resident(ctx, b.data, descs, out_elems, mode)
        assert (res["status"] == 0).all() and np.array_equal(res["consumed"], b.frame_lengths), MODE_NAMES[mode]
        got = raw(out, out_elems, mode)
        assert np.array_equal(got[live], exp[live]), (MODE_NAMES[mode], np.nonzero(got != exp)[0][:8])
        host, hres = ctx.decode_frames(b.data, descs, out_elems=out_elems, mode=mode)
        assert (hres["status"] == 0).all()
        assert np.array_equal(raw(host, out_elems, mode)[live], got[live]), MODE_NAMES[mode]


# --------------------------------------------------------------------------- 2. mixed batches, caller layouts

def layout(descs, kind):
    """out_offsets packed back to back from 0, packed from an odd element, or each frame on an 8-element boundary
    (16 bytes in i16)."""
    descs = descs.copy()
    sizes = descs["n_channels"].astype(np.uint64) * descs["block_size"].astype(np.uint64)
    if kind == "aligned-8":
        sizes = (sizes + np.uint64(7)) & ~np.uint64(7)
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.uint64)
    offs += np.uint64({"packed": 0, "odd": 3, "aligned-8": 8}[kind])
    descs["out_offset"] = offs
    ends = offs + descs["n_channels"].astype(np.uint64) * descs["block_size"].astype(np.uint64)
    return descs, int(ends.max())


@gpu
@pytest.mark.parametrize("kind", ["packed", "odd", "aligned-8"])
def test_mixed_batch_every_mode_and_layout(ctx, kind):
    """Frames of 1 to 8 channels, 8 to 24 bits, wasted bits and every stereo mode side by side (shape_order, idle
    rows, the general flush), against the generator's PCM; I16 for the mixture of 8 to 16 bits."""
    for parts, modes in ((PARTS, (cb.OUT_INTERLEAVED_I32, cb.OUT_INTERLEAVED_I24)),
                         (NARROW_PARTS, (cb.OUT_INTERLEAVED_I16,))):
        b = F.mix(parts, seed=2024)
        descs, _ = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
        descs, out_elems = layout(descs, kind)
        planar = np.zeros(out_elems, np.int32)
        for i in range(b.n_frames):
            o, n = int(descs[i]["out_offset"]), int(descs[i]["n_channels"]) * int(descs[i]["block_size"])
            planar[o:o + n] = b.pcm[int(b.pcm_offsets[i]):int(b.pcm_offsets[i + 1])]
        for mode in modes:
            exp, live = expected_bytes(descs, planar, out_elems, mode)
            out, res = resident(ctx, b.data, descs, out_elems, mode, stream=1)
            assert (res["status"] == 0).all(), MODE_NAMES[mode]
            got = raw(out, out_elems, mode)
            assert np.array_equal(got[live], exp[live]), (MODE_NAMES[mode], np.nonzero(got != exp)[0][:8])
            host, _ = ctx.decode_frames(b.data, descs, out_elems=out_elems, mode=mode)
            assert np.array_equal(raw(host, out_elems, mode)[live], got[live]), MODE_NAMES[mode]


# --------------------------------------------------------------------------- 3. the fused writes alone

def fused_alone_matches_planar(c, data, descs, lengths, out_elems, key):
    """An interleaved resident batch gives the planar batch's statuses, and every frame it accepts is bit-exact."""
    st, ref = oracle_of(key, data, descs, lengths, out_elems)
    _, pres = resident(c, data, descs, out_elems, cb.OUT_PLANAR_I32)
    accepted = 0
    for mode in (cb.OUT_INTERLEAVED_I32, cb.OUT_INTERLEAVED_I16):
        if mode not in modes_for(descs):
            continue
        out, res = resident(c, data, descs, out_elems, mode)
        assert np.array_equal(res["status"], pres["status"]), MODE_NAMES[mode]
        good = [i for i in range(descs.size) if res["status"][i] == 0]
        exp, live = expected_bytes(descs, ref, out_elems, mode, frames=good)
        got = raw(out, out_elems, mode)
        assert np.array_equal(got[live], exp[live]), (MODE_NAMES[mode], np.nonzero((got != exp) & live)[0][:8])
        accepted += len(good)
    return accepted


@gpu
@pytest.mark.parametrize("case", ["c2-ms", "c2-indep", "c4-files", "all-types-wasted-rice2", "tiny-blocks-8bit",
                                  "8ch-12bit-fixed", "mixed", "mixed-narrow"])
def test_fused_path_alone(case):
    c = cb.Context(device=0, lane_per_frame=True, no_generic=True, no_wide=True)
    b = F.mix(PARTS if case == "mixed" else NARROW_PARTS, seed=2024) if case.startswith("mixed") else stream(case)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    assert fused_alone_matches_planar(c, b.data, descs, b.frame_lengths, out_elems, "alone-" + case) > 0
    c.close()


NARROW_SHORTCUT = synth.SynthConfig(n_frames=16, block_size=1024, n_channels=2, bps=16, stereo_mode=0, type_mask=8,
                                    lpc_min_order=1, lpc_max_order=8, qlp_precision=5, rice_mode=-2, rice_kmin=26,
                                    rice_kmax=29, rice2=1, residual_mean=2.0e8, max_porder=1)


@gpu
def test_wide_instances_write_interleaved():
    """The small-coefficient stream of test_wide_second_chance_output: the first pass hands frames to the i64 second
    chance, which rewrites them in the batch's mode."""
    c = cb.Context(device=0, lane_per_frame=True, no_generic=True)
    c1 = cb.Context(device=0, lane_per_frame=True, no_generic=True, no_wide=True)
    b = synth.generate(NARROW_SHORTCUT)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    _, res1 = resident(c1, b.data, descs, out_elems, cb.OUT_INTERLEAVED_I16)
    wide = np.nonzero(res1["status"] == F.NEED_WIDE)[0]
    assert wide.size > 0
    fused_alone_matches_planar(c, b.data, descs, b.frame_lengths, out_elems, "narrow-shortcut")
    _, res2 = resident(c, b.data, descs, out_elems, cb.OUT_INTERLEAVED_I16)
    assert (res2["status"][wide] == 0).any()  # the WIDE instances' own interleaved output was compared
    c.close()
    c1.close()


# --------------------------------------------------------------------------- 4. frames the fused path writes, then declines

def corruption_corpus():
    """The 600-trial corpus of test_corrupted_frames_status_parity."""
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
    return data, offsets, lengths


# test_wrapping_arithmetic_parity's stream at 16 bits, so that I16 applies too: mid/side frames beyond 2^29
WRAPPING_16 = synth.SynthConfig(n_frames=24, block_size=512, n_channels=2, bps=16, stereo_mode=-1, type_mask=12,
                                lpc_min_order=1, lpc_max_order=12, qlp_precision=15, rice_mode=-2, rice_kmin=26,
                                rice_kmax=29, rice2=1, residual_mean=3.0e8, max_porder=2)


def overwrite_case(name):
    if name == "corrupted":
        data, offsets, lengths = corruption_corpus()
        return data, cb.descs_from_offsets(data, offsets, lengths)
    b = synth.generate(WRAPPING_16)
    return b.data, cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)


@gpu
@pytest.mark.parametrize("name", ["wrapping-mid-side", "corrupted"])
def test_fallback_frames_are_overwritten(ctx, name):
    """Every region of an interleaved batch — failed frames included — equals the planar batch's output laid out on
    the host, with the planar batch's statuses; every frame that decodes equals the host call's output in the same
    mode.  (A failed frame's region holds what the generic kernel produced before it stopped, which depends on the
    bytes after the frame's end: the host call stages a chunk's bytes in scratch memory, so there it may differ.)"""
    data, (descs, out_elems) = overwrite_case(name)
    if name == "wrapping-mid-side":  # the stream really has frames the fused path declines after writing them
        assert any(F.mid_side_beyond_bound(d, F.subframe_signals(data, d)) for d in descs)
    pout, pres = resident(ctx, data, descs, out_elems, cb.OUT_PLANAR_I32)
    if name == "corrupted":
        assert (pres["status"] != 0).sum() > 50
    for mode in (cb.OUT_INTERLEAVED_I32, cb.OUT_INTERLEAVED_I16):
        out, res = resident(ctx, data, descs, out_elems, mode)
        assert np.array_equal(res["status"], pres["status"]), MODE_NAMES[mode]
        got = raw(out, out_elems, mode)
        exp, live = expected_bytes(descs, pout, out_elems, mode)
        assert np.array_equal(got[live], exp[live]), (MODE_NAMES[mode], np.nonzero((got != exp) & live)[0][:8])
        host, hres = ctx.decode_frames(data, descs, out_elems=out_elems, mode=mode)
        assert np.array_equal(hres["status"], res["status"]), MODE_NAMES[mode]
        _, good = expected_bytes(descs, pout, out_elems, mode, frames=np.nonzero(res["status"] == 0)[0])
        assert np.array_equal(raw(host, out_elems, mode)[good], got[good]), MODE_NAMES[mode]


# --------------------------------------------------------------------------- 5. independent golden: STREAMINFO MD5

@gpu
def test_resident_i16_md5_of_reference_fixtures(ctx, golden):
    for name in ("pop", "short", "wasted_bits"):
        data = golden[f"{name}__bytes"]
        si, first = cb.open_stream(data)
        descs, nxt, total, stop = cb.demux_frames(data, first)
        assert stop == 1 and si.bits_per_sample == 16
        out, res = resident(ctx, data, descs, total, cb.OUT_INTERLEAVED_I16)
        assert out.dtype == np.int16 and (res["status"] == 0).all()
        md5 = hashlib.md5()
        for d in descs:
            o, n = int(d["out_offset"]), int(d["n_channels"]) * int(d["block_size"])
            md5.update(out[o:o + n].astype("<i2").tobytes())
        assert md5.digest() == si.md5sum, name


# --------------------------------------------------------------------------- 6. full size, many decodes

@gpu
@pytest.mark.parametrize("name,mode", [("c2", cb.OUT_INTERLEAVED_I16), ("c3", cb.OUT_INTERLEAVED_I32)])
def test_full_size_equals_generator(name, mode):
    c = cb.Context(device=0, lane_per_frame=True)
    b = synth.workload(name)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    exp, live = expected_bytes(descs, b.pcm, out_elems, mode)
    assert live.all()
    dev = c.upload(b.data, descs, out_elems, mode=mode)
    assert dev.mode == mode and dev.device_out_ptr != 0
    dev.decode(0)
    out, res = dev.read()
    assert (res["status"] == 0).all() and np.array_equal(res["consumed"], b.frame_lengths)
    assert hashlib.sha1(raw(out, out_elems, mode).tobytes()).digest() == hashlib.sha1(exp.tobytes()).digest()
    c.run_steps([dev], 50, 2)
    out2, res2 = dev.read()
    assert np.array_equal(out2, out) and np.array_equal(res2, res)
    dev.close()
    c.close()


# --------------------------------------------------------------------------- 7. bytes in device memory

@gpu
def test_adopted_i16_batch_checks_crc_on_device():
    import torch
    c = cb.Context(device=0)
    b = synth.workload("c2", 200)
    data = b.data.copy()
    victim = 77
    data[int(b.frame_offsets[victim]) + int(b.frame_lengths[victim]) - 3] ^= 0x01  # last data byte before the CRC-16
    descs, out_elems = cb.descs_from_offsets(data, b.frame_offsets[:-1], b.frame_lengths)
    t = torch.from_numpy(data).cuda()
    dev = c.adopt(t.data_ptr(), t.numel(), descs, out_elems, mode=cb.OUT_INTERLEAVED_I16)
    dev.decode(0)
    out, res = dev.read()
    dev.close()
    c.close()
    assert res["status"][victim] == 23  # "frame CRC mismatch"
    good = [i for i in range(b.n_frames) if i != victim]
    assert (res["status"][good] == 0).all()
    exp, live = expected_bytes(descs, b.pcm, out_elems, cb.OUT_INTERLEAVED_I16, frames=good)
    assert np.array_equal(raw(out, out_elems, cb.OUT_INTERLEAVED_I16)[live], exp[live])


# --------------------------------------------------------------------------- 8. rejections

@gpu
def test_invalid_batches_and_reads_are_refused(ctx):
    b = synth.generate(SYNTH_CASES["ragged-3ch-24bit"])
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    with pytest.raises(cb.Error) as e:  # a 24-bit frame does not fit an I16 batch
        ctx.upload(b.data, descs, out_elems, mode=cb.OUT_INTERLEAVED_I16)
    assert e.value.status == 90
    with pytest.raises(cb.Error) as e:
        ctx.upload(b.data, descs, out_elems, mode=4)
    assert e.value.status == 90
    dev = ctx.upload(b.data, descs, out_elems, mode=cb.OUT_INTERLEAVED_I24)  # 24 bits fit I24
    dev.decode(0)
    dev.close()
    b = synth.workload("c2", 8)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    dev = ctx.upload(b.data, descs, out_elems, mode=cb.OUT_INTERLEAVED_I16)
    dev.decode(0)
    out = np.empty(out_elems, np.int32)
    results = np.zeros(descs.size, dtype=cb.RESULT_DTYPE)
    # clx_batch_read hands out int32: refused for an I16 batch
    assert ctx._L.clx_batch_read(ctx._h, dev._h, out.ctypes.data, out.size, results.ctypes.data) == 90
    out16, res = dev.read()
    assert (res["status"] == 0).all()
    dev.close()


def test_batch_output_mode_entry_points_are_exported():
    """(CPU) clx_batch_create_to and clx_batch_read_to are in the library's dynamic symbol table."""
    lib = C.CDLL(_lib.load()._name)
    for name in ("clx_batch_create_to", "clx_batch_read_to"):
        assert hasattr(lib, name), name
        assert name in _lib.SYMBOLS
