"""Kernels launched per decode, on every path and in every output mode (-m gpu).

`Context.launch_count` counts the kernels a decode enqueues (bench.py reports it as `gpu_launches`).  The numbers
below follow from the launch sequence: the path's fast kernels (lane per frame: the index pass and the decode
instances, two of them plus two i64 ones unless `no_wide`; warp per frame: entropy + prediction), then, unless
`no_generic`, the 12-tap and 32-tap generic instances, then the device CRC-16 where it runs, then the conversion to an
interleaved mode.  A resident batch on the lane-per-frame path writes interleaved i32 / i16 in its decode pass and
instead marks and converts the frames the generic kernel took over (two more kernels, both gated).
"""
import pytest

import claxon_b200 as cb
from claxon_b200 import synth

gpu = pytest.mark.gpu

PLANAR, I32, I24, I16 = cb.OUT_PLANAR_I32, cb.OUT_INTERLEAVED_I32, cb.OUT_INTERLEAVED_I24, cb.OUT_INTERLEAVED_I16

CONFIGS = {
    "lane": dict(lane_per_frame=True),
    "lane-no-wide": dict(lane_per_frame=True, no_wide=True),
    "lane-no-generic": dict(lane_per_frame=True, no_generic=True),
    "warp": dict(warp_per_frame=True),
    "generic": dict(generic_only=True),
}

# kernels per decode of a batch built from host bytes: planar, interleaved i32, i24, i16
BATCH = {
    "lane": {PLANAR: 7, I32: 9, I24: 8, I16: 9},
    "lane-no-wide": {PLANAR: 5, I32: 7, I24: 6, I16: 7},
    "lane-no-generic": {PLANAR: 5, I32: 5, I24: 6, I16: 5},
    "warp": {PLANAR: 4, I32: 5, I24: 5, I16: 5},
    "generic": {PLANAR: 2, I32: 3, I24: 3, I16: 3},
}

# decode kernels of one host-buffer call (one chunk), without CRC-16 and conversion: never fused
HOST_DECODE = {"lane": 7, "lane-no-wide": 5, "lane-no-generic": 5, "warp": 4, "generic": 2}

MODES = {"planar": PLANAR, "i32": I32, "i24": I24, "i16": I16}


@pytest.fixture(scope="module")
def batch():
    b = synth.workload("c2", 64)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    return b, descs, out_elems


def launches_of(c, fn):
    n0 = c.launch_count
    fn()
    return c.launch_count - n0


@gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_batch_launches(batch, config, mode):
    b, descs, out_elems = batch
    c = cb.Context(device=0, **CONFIGS[config])
    dev = c.upload(b.data, descs, out_elems, mode=MODES[mode])
    assert launches_of(c, lambda: dev.decode(0)) == BATCH[config][MODES[mode]]
    assert launches_of(c, lambda: dev.decode(1)) == BATCH[config][MODES[mode]]
    _, res = dev.read()
    dev.close()
    c.close()
    if config != "lane-no-generic":
        assert (res["status"] == 0).all()


@gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_adopted_batch_adds_device_crc(batch, config, mode):
    import torch
    b, descs, out_elems = batch
    c = cb.Context(device=0, **CONFIGS[config])
    t = torch.from_numpy(b.data.copy()).cuda()
    dev = c.adopt(t.data_ptr(), t.numel(), descs, out_elems, mode=MODES[mode])
    assert launches_of(c, lambda: dev.decode(0)) == BATCH[config][MODES[mode]] + 1
    dev.sync()
    dev.close()
    c.close()


@gpu
@pytest.mark.parametrize("verify_crc", [True, False])
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_host_call_launches(batch, config, mode, verify_crc):
    b, descs, out_elems = batch
    c = cb.Context(device=0, verify_crc=verify_crc, **CONFIGS[config])
    n = launches_of(c, lambda: c.decode_frames(b.data, descs, out_elems=out_elems, mode=MODES[mode]))
    c.close()
    assert n == HOST_DECODE[config] + int(verify_crc) + int(MODES[mode] != PLANAR)


@gpu
def test_small_host_call_takes_warp_per_frame_path(batch):
    """A host-buffer call of at most 4096 frames runs the warp-per-frame path unless lane_per_frame is set; a
    resident batch runs the lane-per-frame path."""
    b, descs, out_elems = batch
    c = cb.Context(device=0)
    assert launches_of(c, lambda: c.decode_frames(b.data, descs, out_elems=out_elems)) == HOST_DECODE["warp"] + 1
    dev = c.upload(b.data, descs, out_elems)
    assert launches_of(c, lambda: dev.decode(0)) == BATCH["lane"][PLANAR]
    dev.sync()
    dev.close()
    c.close()


@gpu
def test_warp_per_frame_wins_over_lane_per_frame(batch):
    b, descs, out_elems = batch
    c = cb.Context(device=0, warp_per_frame=True, lane_per_frame=True)
    dev = c.upload(b.data, descs, out_elems)
    assert launches_of(c, lambda: dev.decode(0)) == BATCH["warp"][PLANAR]
    dev.sync()
    dev.close()
    c.close()
