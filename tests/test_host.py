"""Host-side logic of the product (no GPU): C ABI surface, header parse, CRC, metadata walk,
demuxer, claxon-shaped Block API, error contract.  The oracle is used only as the checker."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import _lib, synth, shard
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KAT = json.load(open(os.path.join(ROOT, "tests", "golden", "kat.json")))


def test_library_exports_every_declared_symbol():
    """The C-ABI library loads and exports exactly the functions include/claxon_b200.h declares."""
    header = open(os.path.join(ROOT, "include", "claxon_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(clx_[a-z0-9_]+)\s*\(", header))
    L = _lib.load()
    for name in declared:
        assert hasattr(L, name), f"{name} declared in the header but not exported"
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    assert L.clx_abi_version() == 1
    # the CUDA kernels are in the same library (sm_90a SASS present)
    out = subprocess.run(["cuobjdump", "-lelf", _lib._build.LIB], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_product_does_not_import_the_oracle():
    pkg = os.path.join(ROOT, "claxon_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cpp", ".c", ".h")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "claxon_oracle" not in text and "from oracle" not in text and "import oracle" not in text, f


def test_no_device_fails_loudly():
    """Without a GPU the decode path must raise, not fall back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(cb.Error) as e:
        cb.Context()
    assert e.value.status == 92


def test_status_strings_match_claxon():
    # SURVEY.md Appendix B: verbatim strings, compared by string in the reference (src/error.rs:34-45)
    expect = {3: "frame sync code missing", 9: "frame header CRC mismatch", 16: "invalid partition order",
              18: "unencoded binary is not yet implemented", 23: "frame CRC mismatch",
              10: "header without bits per sample info", 14: "subframe has no non-wasted bits",
              22: "a negative quantized linear predictor coefficient shift is not supported, please file a bug.",
              43: "vendor string too long", 30: "invalid stream header"}
    for k, v in expect.items():
        assert cb.status_str(k) == v
    L = _lib.load()
    assert L.clx_status_kind(10) == cb.KIND_UNSUPPORTED and L.clx_status_kind(18) == cb.KIND_UNSUPPORTED
    assert L.clx_status_kind(2) == cb.KIND_IO and L.clx_status_kind(23) == cb.KIND_FORMAT


def test_error_equality_semantics():
    assert cb.Error(23) == cb.Error(23) and cb.Error(23) != cb.Error(9)
    assert cb.Error(2) != cb.Error(2)  # (&IoError(_), _) => false
    assert cb.Error(10).variant == "Unsupported" and cb.Error(16).variant == "FormatError"


def test_crc_against_oracle_and_vectors():
    L = _lib.load()
    for data, exp in KAT["crc8"]["cases"]:
        assert L.clx_crc8(bytes(data), len(data)) == exp
    for data, exp in KAT["crc16"]["cases"]:
        assert L.clx_crc16(bytes(data), len(data)) == exp
    rng = np.random.default_rng(0)
    for n in (0, 1, 7, 8, 9, 63, 64, 1000, 6157):
        buf = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert L.clx_crc16(buf, n) == O.lib().clxo_crc16(buf, n)
        assert L.clx_crc8(buf, n) == O.lib().clxo_crc8(buf, n)


def _hdr_tuple_cb(d):
    return (d.block_size, d.sample_rate, d.n_channels, d.channel_assignment, d.bits_per_sample, d.flags & 1,
            d.number, d.header_len)


def _hdr_tuple_o(h):
    return (h.block_size, h.sample_rate, h.n_channels, h.channel_assignment, h.bits_per_sample,
            h.variable_blocking, h.number, h.header_len)


def test_frame_header_parse_matches_oracle_on_mutations():
    b = synth.generate(synth.SynthConfig(n_frames=6, block_size=1000, n_channels=2, stereo_mode=-1, force_bs16=1,
                                         variable_blocking=1))
    rng = np.random.default_rng(5)
    base = b.data[:16].copy()
    n_ok = 0
    for trial in range(4000):
        buf = base.copy()
        for _ in range(rng.integers(0, 3)):
            buf[rng.integers(0, 12)] = rng.integers(0, 256)
        n = int(rng.integers(0, 17))
        st_o, h = O.read_frame_header(buf[:n].copy() if n else np.zeros(0, np.uint8))
        st_c, d = cb.parse_frame_header(buf[:n].copy() if n else np.zeros(0, np.uint8))
        assert st_o == st_c, (trial, st_o, st_c, buf[:n].tolist())
        if st_o == 0:
            n_ok += 1
            assert _hdr_tuple_cb(d) == _hdr_tuple_o(h)
    assert n_ok > 50


def _check_against_spec(buf, st_c, d, st_o=None, h=None):
    """Product (and oracle) against the plain-Python statement of the reference in tests/spec_header.py."""
    from tests import spec_header as S
    kind, val = S.parse(bytes(buf))
    if kind == "eof":
        assert st_c == 1 and (st_o is None or st_o == 1)
    elif kind == "err":
        want = "UnexpectedEof" if val == S.EOF_MSG else val
        assert cb.status_str(st_c) == want, (bytes(buf).hex(), cb.status_str(st_c), want)
        assert st_o is None or st_o == st_c
    else:
        assert st_c == 0, (bytes(buf).hex(), cb.status_str(st_c))
        want = (val["block_size"], val["sample_rate"], val["n_channels"], val["channel_assignment"],
                val["bits_per_sample"], val["variable"], val["number"], val["header_len"])
        assert _hdr_tuple_cb(d) == want, (bytes(buf).hex(), _hdr_tuple_cb(d), want)
        if h is not None:
            assert _hdr_tuple_o(h) == want


def test_frame_header_parse_matches_independent_spec_on_mutations():
    """The C++ parser and the C oracle share an author; tests/spec_header.py is a third statement of
    src/frame.rs:131-316 (bitwise CRC-8, the reference's own control flow and error strings) that both must match."""
    b = synth.generate(synth.SynthConfig(n_frames=6, block_size=1000, n_channels=2, stereo_mode=-1, force_bs16=1,
                                         variable_blocking=1))
    L = _lib.load()
    rng = np.random.default_rng(11)
    base = b.data[:16].copy()
    kinds = set()
    for trial in range(3000):
        buf = base.copy()
        for _ in range(rng.integers(0, 3)):
            buf[rng.integers(0, 12)] = rng.integers(0, 256)
        if trial % 3 == 0:  # a mutated header whose CRC-8 is right again: the field checks decide, not the checksum
            st0, d0 = cb.parse_frame_header(buf.copy(), flags=cb.OPT_NO_VERIFY_CRC if hasattr(cb, "OPT_NO_VERIFY_CRC") else 1)
            if st0 == 0:
                buf[d0.header_len - 1] = L.clx_crc8(buf[: d0.header_len - 1].tobytes(), d0.header_len - 1)
        n = int(rng.integers(0, 17))
        cut = buf[:n].copy() if n else np.zeros(0, np.uint8)
        st_o, h = O.read_frame_header(cut)
        st_c, d = cb.parse_frame_header(cut)
        _check_against_spec(cut, st_c, d, st_o, h)
        kinds.add(st_c)
    assert len(kinds) >= 6  # ok, eof, unexpected eof and several distinct format errors were all exercised


def test_frame_header_all_codes():
    # every block-size / sample-rate / channel / bps code, CRC fixed up so only the codes decide
    L = _lib.load()
    for bs_code in range(16):
        for sr_code in range(16):
            for cb_byte in range(0, 256, 1):
                hdr = bytearray([0xff, 0xf8, (bs_code << 4) | sr_code, cb_byte, 0x05])
                if bs_code == 6: hdr += b"\x20"
                if bs_code == 7: hdr += b"\x12\x34"
                if sr_code == 12: hdr += b"\x2c"
                if sr_code in (13, 14): hdr += b"\xac\x44"
                hdr.append(L.clx_crc8(bytes(hdr), len(hdr)))
                st_o, h = O.read_frame_header(np.frombuffer(bytes(hdr), np.uint8))
                st_c, d = cb.parse_frame_header(bytes(hdr))
                assert st_o == st_c, (bs_code, sr_code, cb_byte)
                if st_o == 0:
                    assert _hdr_tuple_cb(d) == _hdr_tuple_o(h)
                _check_against_spec(bytes(hdr), st_c, d)
            if sr_code > 1 and bs_code > 1:
                break  # the full cross product is only needed for a couple of rows


def test_var_length_int_in_header():
    L = _lib.load()
    for number in (0, 127, 128, 2047, 2048, 65535, 65536, (1 << 21) - 1, 1 << 21, (1 << 26) - 1, 1 << 26,
                   (1 << 31) - 1, 1 << 31, (1 << 36) - 1):
        b = synth.generate(synth.SynthConfig(n_frames=1, block_size=192, n_channels=1, variable_blocking=1))
        # rebuild the header with our own varint of `number` (sample number: up to 36 bits)
        def varint(v):
            if v < 0x80: return bytes([v])
            extra = 1
            while extra < 6 and v >= (1 << (6 * extra + 6 - extra)): extra += 1
            first = (0xff << (7 - extra)) & 0xff | (v >> (6 * extra))
            return bytes([first]) + bytes(0x80 | ((v >> (6 * i)) & 0x3f) for i in range(extra - 1, -1, -1))
        hdr = bytearray(b.data[:4].tobytes()) + varint(number)
        hdr.append(L.clx_crc8(bytes(hdr), len(hdr)))
        st, d = cb.parse_frame_header(bytes(hdr))
        st_o, h = O.read_frame_header(np.frombuffer(bytes(hdr), np.uint8))
        assert st == 0 and st_o == 0 and d.number == number == h.number
    k = KAT["var_length_int"]  # src/frame.rs:107-129 through the oracle-independent product parser
    hdr0 = bytes([0xff, 0xf9, 0x19, 0x08])
    at = 0
    for exp in k["values"]:
        st, d = cb.parse_frame_header(hdr0 + bytes(k["bytes"][at:]) + b"\0" * 4, flags=cb.OPT_NO_VERIFY_CRC)
        assert st == 0 and d.number == exp
        at += d.header_len - 5
    assert cb.parse_frame_header(hdr0 + bytes(k["bytes"][at:]), flags=1)[0] == 6


def test_open_stream_matches_golden(golden):
    for name in golden["names"]:
        name = str(name)
        meta = golden[f"{name}__meta"]
        data = golden[f"{name}__bytes"]
        try:
            si, first = cb.open_stream(data)
            st = 0
        except cb.Error as e:
            st = e.status
        assert st == meta[0], name
        if st == 0:
            assert first == meta[1] and si.channels == meta[2] and si.bits_per_sample == meta[3]
            assert (si.samples or 0) == meta[4]
            assert si.md5sum == bytes(golden[f"{name}__md5"])
    # reference tests/testsamples.rs:404-426
    with pytest.raises(cb.Error) as e:
        cb.open_stream(golden["large_vendor_string__bytes"])
    assert e.value == cb.Error(43)
    with pytest.raises(cb.Error) as e:
        cb.open_stream(golden["large_vorbis_comment_block__bytes"])
    assert e.value.variant == "Unsupported"


@pytest.mark.parametrize("cfgname", ["c2", "c3", "c4", "c5"])
def test_demux_finds_every_frame(cfgname):
    n = {"c2": 40, "c3": 40, "c4": 44, "c5": 3}[cfgname]
    b = synth.workload(cfgname, n)
    descs, nxt, total, stop = cb.demux_frames(b.data)
    assert stop == cb.EOF and nxt == b.data.size and descs.size == b.n_frames
    assert np.array_equal(descs["byte_offset"], b.frame_offsets[:-1])
    assert np.array_equal(descs["byte_len"], b.frame_lengths)
    assert (descs["flags"] & cb.FRAME_CRC16_VERIFIED).all()
    assert (descs["out_offset"] % 4 == 0).all() and total >= b.n_samples


def test_demux_false_sync_inside_residual_is_rejected():
    # plant sync-looking bytes inside frame payloads: the CRC-16 condition must reject them
    b = synth.workload("c2", 12)
    data = b.data.copy()
    hits = 0
    for i in range(b.n_frames):
        lo, hi = int(b.frame_offsets[i]) + 16, int(b.frame_offsets[i + 1]) - 4
        seg = data[lo:hi]
        idx = np.nonzero((seg[:-1] == 0xff) & ((seg[1:] & 0xfe) == 0xf8))[0]
        hits += idx.size
    descs, nxt, total, stop = cb.demux_frames(data)
    assert descs.size == b.n_frames and np.array_equal(descs["byte_len"], b.frame_lengths)
    # damaged frame: boundary unknown -> last descriptor is unverified and spans the rest
    data[int(b.frame_offsets[3]) + 100] ^= 0x10
    descs, nxt, total, stop = cb.demux_frames(data)
    assert descs.size >= 3 and not (descs["flags"][-1] & cb.FRAME_CRC16_VERIFIED) or descs.size == b.n_frames


def _same_demux(a, b):
    return a[0].size == b[0].size and np.array_equal(a[0], b[0]) and tuple(a[1:]) == tuple(b[1:])


def test_demux_on_several_threads_equals_sequential():
    """clx_demux_frames_mt (parts of the byte range on host threads, stitched by CRC-16-confirmed chains) returns
    descriptor for descriptor what clx_demux_frames returns: clean streams of every workload shape, a metadata prefix,
    planted sync codes with a valid-looking header, damaged frames (unknown boundary: the last descriptor), garbage
    between frames (stop status), truncation, and the max_frames limit."""
    L = _lib.load()
    rng = np.random.default_rng(31)
    cases = []
    for wl, n in (("c2", 96), ("c3", 64), ("c4", 110), ("c5", 6)):
        b = synth.workload(wl, n)
        cases.append((f"{wl} clean", b.data.copy(), 0))
        d = b.data.copy()
        d[int(b.frame_offsets[n // 2]) + 40] ^= 0x20             # a damaged frame in the middle
        cases.append((f"{wl} damaged", d, 0))
        cases.append((f"{wl} truncated", b.data[: int(b.frame_offsets[n - 2]) + 11].copy(), 0))
        d = np.concatenate([b.data[: int(b.frame_offsets[n // 3])], np.frombuffer(b"\x00garbage\xff\xf8\x00\x00", np.uint8),
                            b.data[int(b.frame_offsets[n // 3]):]])
        cases.append((f"{wl} garbage between frames", d, 0))
        # planted false starts: a real frame header (so sync, codes and CRC-8 are all right) copied into residual data
        d = b.data.copy()
        hdr = d[int(b.frame_offsets[1]): int(b.frame_offsets[1]) + 8].copy()
        for i in range(2, n, 3):
            at = int(b.frame_offsets[i]) + int(b.frame_lengths[i]) // 2
            d[at: at + hdr.size] = hdr
            # keep the frame intact as far as its CRC-16 goes: patch the footer
            f0, f1 = int(b.frame_offsets[i]), int(b.frame_offsets[i + 1])
            c = L.clx_crc16(d[f0: f1 - 2].tobytes(), f1 - 2 - f0)
            d[f1 - 2], d[f1 - 1] = c >> 8, c & 0xff
        cases.append((f"{wl} planted headers", d, 0))
    fb = synth.workload("c4", 44)
    file_bytes = np.frombuffer(synth.make_file(fb, 0, 44, padding=300), np.uint8)
    si, first = cb.open_stream(file_bytes)
    cases.append(("file with metadata", file_bytes.copy(), first))
    for name, data, start in cases:
        ref = cb.demux_frames(data, start=start)
        assert ref[0].size > 0, name
        for th in (2, 3, 5, 8, 13):
            got = cb.demux_frames(data, start=start, threads=th)
            assert _same_demux(ref, got), (name, th, ref[0].size, got[0].size, ref[1:], got[1:])
        for cap in (1, 7, ref[0].size):
            a = cb.demux_frames(data, start=start, max_frames=cap)
            g = cb.demux_frames(data, start=start, max_frames=cap, threads=4)
            assert _same_demux(a, g), (name, "max_frames", cap)
    # parts smaller than a frame, parts that start inside the last frame, a start offset past the end
    b = synth.workload("c5", 3)
    ref = cb.demux_frames(b.data)
    assert _same_demux(ref, cb.demux_frames(b.data, threads=8))
    assert cb.demux_frames(b.data, start=b.data.size + 5, threads=4)[0].size == 0


def test_block_api_matches_reference_unit_tests():
    k = KAT["block_sample"]
    blk = cb.Block(0, k["block_size"], np.array(k["buffer"], dtype=np.int32))
    assert blk.channels() == k["channels"] and blk.len() == 15 and blk.duration() == 5
    for ch, i, exp in k["checks"]:
        assert blk.sample(ch, i) == exp
    assert blk.channel(1).tolist() == [13, 17, 19, 23, 29]
    k = KAT["stereo_samples"]
    blk = cb.Block(0, k["block_size"], np.array(k["buffer"], dtype=np.int32))
    assert list(blk.stereo_samples()) == [tuple(p) for p in k["pairs"]]
    with pytest.raises(RuntimeError):
        cb.Block(0, 5, np.zeros(15, np.int32)).stereo_samples()
    e = cb.Block.empty()
    assert e.len() == 0 and e.channels() == 0 and e.time() == 0


def test_ensure_buffer_len():
    # src/frame.rs:639-648: result has exactly new_len elements for every capacity
    for cap in range(10):
        for new_len in range(10):
            buf = np.empty(cap, dtype=np.int32)
            r = cb._ensure_buffer_len(buf, new_len)
            assert r.size == new_len
    big = np.zeros(100, dtype=np.int32)
    r = cb._ensure_buffer_len(big[:10], 50)
    assert r.base is big or r.base is big.base or np.shares_memory(r, big)  # capacity reused


def test_shard_plan_partitions_and_balances():
    b = synth.workload("c4", 220)
    descs, out_elems = cb.descs_from_offsets(b.data, b.frame_offsets[:-1], b.frame_lengths)
    for world in (1, 2, 4, 8):
        plan = shard.plan_shards(descs, world)
        assert plan[0][0] == 0 and plan[-1][1] == descs.size
        assert all(plan[i][1] == plan[i + 1][0] for i in range(world - 1))
        costs = [float(shard.frame_costs(descs[lo:hi]).sum()) for lo, hi in plan]
        assert max(costs) <= 1.15 * (sum(costs) / world) + float(shard.frame_costs(descs).max())
        for lo, hi in plan:
            d, b0, b1, o0, o1 = shard.localize(descs, lo, hi)
            if d.size:
                st, hd = cb.parse_frame_header(b.data[b0:b1], int(d["byte_offset"][0]))
                assert st == 0 and hd.block_size == d["block_size"][0]


# --------------------------------------------------------------------------- FlacReaderOptions / tags (SURVEY.md §8 f3)

def test_flac_reader_tags_like_the_reference(golden):
    """The reference's own metadata tests (tests/testsamples.rs:319-352, :428-446) on its own fixtures."""
    mo = cb.FlacReaderOptions(metadata_only=True, read_vorbis_comment=True)
    r = cb.FlacReader.new_ext(golden["repeated_vorbis_comment__bytes"], mo)
    assert r.get_tag("FOO") == ["bar", "baz"] and r.get_tag("foo") == ["bar", "baz"] and r.get_tag("foobar") == []
    r = cb.FlacReader.new_ext(golden["empty_vorbis_comment__bytes"], mo)
    assert r.tags() == [("FOO", "bar"), ("X", "Y")]  # the zero-length comment is skipped
    # metadata_only_still_reads_vorbis_comment_block / no_read_vorbis_comment_block_does_not_contain_vendor_string
    r = cb.FlacReader.new_ext(golden["short__bytes"], mo)
    assert r.vendor() == "reference libFLAC 1.3.2 20170101"
    r = cb.FlacReader.new_ext(golden["short__bytes"], cb.FlacReaderOptions(metadata_only=True, read_vorbis_comment=False))
    assert r.vendor() is None and r.tags() == [] and r.streaminfo().samples == 4
    # a metadata-only reader cannot decode (the reference panics)
    for what in ("blocks", "samples", "into_samples"):
        with pytest.raises(RuntimeError):
            getattr(r, what)()
    assert cb.FlacReader.new_ext(golden["pop__bytes"], mo).vendor() is None or True  # pop.flac has no tags at all
    assert cb.FlacReader.new_ext(golden["pop__bytes"], mo).tags() == []


def test_open_stream_ex_stops_early(golden):
    """metadata_only + no tags wanted: the walk ends one block after STREAMINFO (src/lib.rs:275-279), so damage
    further on is not looked at; the default walk still reports it."""
    data = golden["short__bytes"].copy()   # STREAMINFO, SEEKTABLE, VORBIS_COMMENT, frames
    si, first = cb.open_stream(data)
    assert first == 108
    vc_header = 4 + 4 + 34 + 4 + 18       # 'fLaC', STREAMINFO block, SEEKTABLE block -> VORBIS_COMMENT header
    assert data[vc_header] & 0x7f == 4
    data[vc_header + 4] = 0xff             # vendor length now absurd
    with pytest.raises(cb.Error) as e:
        cb.open_stream(data)
    assert e.value.status == 43            # "vendor string too long"
    r = cb.FlacReader.new_ext(data, cb.FlacReaderOptions(metadata_only=True, read_vorbis_comment=False))
    assert r.streaminfo().bits_per_sample == 16


def test_open_stream_matches_independent_spec_on_mutations(golden):
    """Stream open (magic, metadata block walk, STREAMINFO checks, VORBIS_COMMENT validation, tags) of the product AND
    of the oracle against tests/spec_metadata.py — a third statement of src/lib.rs:186-307 and
    src/metadata.rs:212-545 — on the reference fixtures, a synthetic file, and thousands of byte mutations and
    truncations of their metadata: same claxon error string, or same first frame offset / stream info / vendor / tags."""
    from tests import spec_metadata as M
    seeds = [golden[f"{n}__bytes"] for n in ("pop", "short", "wasted_bits", "empty_vorbis_comment",
                                            "repeated_vorbis_comment", "non_subset")]
    b = synth.workload("c4", 22)
    seeds.append(np.frombuffer(synth.make_file(b, 0, 11, padding=64), np.uint8))
    rng = np.random.default_rng(23)
    seen = set()

    def check(buf):
        kind, val = M.open_stream(buf.tobytes())
        try:
            si, first = cb.open_stream(buf)
            got = None
        except cb.Error as e:
            got = e.message
        st_o = O.open_stream(buf)[0]
        if kind == "err":
            want = "UnexpectedEof" if val == M.EOF_MSG else val
            assert got == want, (got, want)
            assert cb.status_str(st_o) == want
            seen.add(want)
            return
        assert got is None and st_o == 0, (got, st_o)
        assert first == val["first_frame"]
        assert (si.min_block_size, si.max_block_size, si.sample_rate, si.channels, si.bits_per_sample) == (
            val["min_block_size"], val["max_block_size"], val["sample_rate"], val["channels"], val["bits_per_sample"])
        assert (si.samples or 0) == val["samples"] and si.md5sum == val["md5sum"]
        assert (si.min_frame_size or 0) == val["min_frame_size"] and (si.max_frame_size or 0) == val["max_frame_size"]
        r = cb.FlacReader.new_ext(buf, cb.FlacReaderOptions(metadata_only=True))
        assert r.vendor() == val["vendor"]
        assert r.tags() == [(c[:i], c[i + 1:]) for c, i in val["comments"]]
        seen.add("ok")

    for seed in seeds:
        seed = np.asarray(seed, dtype=np.uint8)
        kind, val = M.open_stream(seed.tobytes())
        assert kind == "ok"
        meta_end = val["first_frame"]
        check(seed)
        for trial in range(400):
            buf = seed[: meta_end + 64].copy()
            for _ in range(int(rng.integers(1, 4))):
                at = int(rng.integers(0, meta_end))
                # bias towards the bytes that steer the walk: small values, high bits, '=' and friends
                buf[at] = rng.choice([0, 1, 4, 0x7F, 0x80, 0x84, 0xFF, 0x3D, int(rng.integers(0, 256))])
            if trial % 4 == 0:
                buf = buf[: int(rng.integers(0, meta_end + 1))]
            check(buf)
    assert "ok" in seen and len(seen) >= 12, sorted(seen)  # a dozen distinct outcomes at least


# --------------------------------------------------------------------------- container feeds (SURVEY.md §8 f4)

def _check_container_descs(b, frame_bytes, descs, total, si):
    from oracle import oracle as O
    assert descs.size == b.n_frames and si.channels == b.config.n_channels and si.bits_per_sample == b.config.bps
    assert np.array_equal(descs["byte_len"], b.frame_lengths)  # exact extents, straight from the container
    bad, st, pcm = O.decode_batch(frame_bytes, descs["byte_offset"], descs["byte_len"], descs["out_offset"], total, n_threads=4)
    assert bad == 0
    for i in range(b.n_frames):
        o = int(descs[i]["out_offset"]); lo, hi = int(b.pcm_offsets[i]), int(b.pcm_offsets[i + 1])
        assert np.array_equal(pcm[o:o + hi - lo], b.pcm[lo:hi])


def test_ogg_packets_become_frame_descriptors():
    """examples/decode_ogg.rs: header packets skipped, one frame per packet, packets spanning pages reassembled, the
    empty last packet and a foreign logical stream ignored, page CRCs verified."""
    from tests import containers
    b = synth.workload("c3", 9)      # ~12 KB frames: every one spans several pages of 40 segments
    ogg = np.frombuffer(containers.flac_in_ogg(b), dtype=np.uint8)
    si, frames, descs, total = cb.ogg_frames(ogg)
    assert si.samples == b.n_samples // 2 and frames.size == b.data.size
    _check_container_descs(b, frames, descs, total, si)
    damaged = ogg.copy()
    damaged[len(damaged) // 2] ^= 1    # a flipped payload bit: the page checksum catches it
    with pytest.raises(cb.Error) as e:
        cb.ogg_frames(damaged)
    assert e.value.status == 93
    assert cb.ogg_frames(damaged, flags=cb.OPT_NO_VERIFY_CRC)[2].size == 9  # ... unless told not to look
    with pytest.raises(cb.Error):
        cb.ogg_frames(b.data)          # not an Ogg file at all


@pytest.mark.parametrize("co64", [False, True])
def test_mp4_sample_tables_become_frame_descriptors(co64):
    """examples/decode_mp4.rs: the first 'fLaC' track (another track comes first in the file), STREAMINFO from dfLa,
    frame extents from stsz + stsc runs + stco / co64; the descriptors index the file itself."""
    from tests import containers
    b = synth.workload("c4", 22)
    mp4 = np.frombuffer(containers.flac_in_mp4(b, co64=co64), dtype=np.uint8)
    si, descs, total = cb.mp4_frames(mp4)
    _check_container_descs(b, mp4, descs, total, si)
    assert not np.array_equal(np.diff(descs["byte_offset"].astype(np.int64)), b.frame_lengths[:-1])  # chunks are apart
    with pytest.raises(cb.Error) as e:
        cb.mp4_frames(mp4[: mp4.size // 3])  # sample tables point past the end
    assert e.value.status == 93


def test_bench_reference_arm_prints_one_json_line():
    """`bench.py --impl reference` (the CPU arm the driver runs first) needs no GPU: one JSON line on stdout with the
    contract's keys, bit-exact against the generator's PCM."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1",
                          "--frames", "64"], capture_output=True, text=True, timeout=300, cwd=root)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    line = json.loads(lines[0])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert key in line, key
    assert line["impl"] == "reference" and line["bit_exact"] is True and line["value"] > 0
    assert line["cpu_baseline"]["kind"] == "port" and line["e2e"]["h2d_bytes_per_step"] == 0
