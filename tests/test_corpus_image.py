"""Corpus images on the host (no GPU): clx_corpus_image_check against the plain-Python statement of the layout in
tests/spec_image.py.  Well-formed images of golden, synthetic, empty and one-frame corpora are accepted; every field
changed alone is refused.  The GPU half (the writer, attach, batches over attached images) is
tests/test_gpu_shared_corpus.py."""
import ctypes as C
import struct

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import _lib, synth
from tests import spec_image as S
from tests.test_gpu_corpus import c4ch_config, flac_of, variable_config


def check(img) -> int:
    img = np.ascontiguousarray(img, dtype=np.uint8)
    return int(_lib.load().clx_corpus_image_check(img.ctypes.data if img.size else None, img.size))


def files_of(srcs):
    return [(f.data, f.info, f.descs) for f in cb.index(srcs).files]


def spec_image(files, tails=None):
    frame, desc = S.filler_of(_lib.load())
    return S.image(files, frame, desc, tails)


def one_frame_file():
    b = synth.generate(synth.workload_config("c2", 1))
    return np.frombuffer(synth.make_file(b, 0, 1), np.uint8).copy()


def corpora(golden):
    return {
        "golden": files_of([golden[f"{n}__bytes"] for n in ("pop", "short", "wasted_bits")]),
        "synthetic": files_of([flac_of(synth.workload_config("c2", 9)), flac_of(c4ch_config()), flac_of(variable_config())]),
        "empty": [],
        "one_frame": files_of([one_frame_file()]),
    }


@pytest.mark.parametrize("name", ["golden", "synthetic", "empty", "one_frame"])
def test_spec_images_are_accepted(golden, name):
    files = corpora(golden)[name]
    img, lay = spec_image(files)
    assert img.size % 64 == 0 and lay["bytes_offset"] % S.ALIGN == 0
    assert check(img) == 0
    # the size the library computes for the same index
    descs = np.concatenate([d for _, _, d in files]) if files else np.zeros(0, cb.DESC_DTYPE)
    ff = np.concatenate([[0], np.cumsum([d.size for _, _, d in files])]).astype(np.uint32)
    sizes = np.array([len(x) for x, _, _ in files] or [0], dtype=np.uintp)
    L = _lib.load()
    assert L.clx_corpus_image_bytes(sizes.ctypes.data, descs.ctypes.data, descs.size, ff.ctypes.data, len(files)) == img.size


def test_files_without_frames_and_unconfirmed_ends(golden):
    tail = np.concatenate([flac_of(synth.workload_config("c2", 6)), np.frombuffer(b"\xff\xf8junk!", np.uint8)])
    idx = cb.index([golden["short__bytes"], tail])
    assert not idx[1].end_confirmed
    empty = (np.zeros(0, np.uint8), idx[0].info, np.zeros(0, cb.DESC_DTYPE))
    files = [empty] + files_of([golden["short__bytes"], tail]) + [empty]
    for verdict in (0, 2, 5, 10):  # OK or a frame header status
        assert check(spec_image(files, [0, 0, verdict, 0])[0]) == 0, verdict
    for verdict in (1, 11, 23, 90, -1):  # EOF, statuses a header never gives
        assert check(spec_image(files, [0, 0, verdict, 0])[0]) == 90, verdict
    for at in (0, 1, 3):  # a verdict on a file whose end is confirmed, or that has no frames
        tails = [0, 0, 0, 0]
        tails[at] = 5
        assert check(spec_image(files, tails)[0]) == 90, at


# --------------------------------------------------------------------------- one field at a time

def put(img, offset, fmt, value):
    img = img.copy()
    img[offset:offset + struct.calcsize(fmt)] = np.frombuffer(struct.pack(fmt, value), np.uint8)
    return img


def get(img, offset, fmt):
    return struct.unpack_from(fmt, img.tobytes(), offset)[0]


def record(lay, i, field):
    """Offset of a field of file record i."""
    at = {"byte_base": 56, "byte_count": 64, "first_frame": 72, "n_frames": 76, "flags": 80, "tail": 84}[field]
    return lay["files_offset"] + i * S.FILE.size + at


def desc(lay, f, field):
    at = {"byte_offset": 0, "byte_len": 8, "n_channels": 16, "flags": 19, "out_offset": 32}[field]
    return lay["descs_offset"] + f * S.DESC.size + at


@pytest.fixture(scope="module")
def clean(golden):
    files = files_of([golden["pop__bytes"], flac_of(synth.workload_config("c2", 9)), golden["short__bytes"]])
    img, lay = spec_image(files)
    assert check(img) == 0
    return img, lay, files


@pytest.mark.parametrize("field", ["magic", "version", "header_bytes", *S.HEADER_FIELDS])
def test_each_header_field_is_checked(clean, field):
    img, lay, _ = clean
    at = S.HEADER_OFFSETS[field]
    fmt = "<I" if field in ("version", "header_bytes") else "<Q"
    v = get(img, at, fmt)
    for bad in {v + 1, v - 1 if v else 1 << 40, v ^ (1 << 31), v + 4096}:
        assert check(put(img, at, fmt, bad)) == 90, (field, bad)


def test_size_and_alignment(clean):
    img, lay, _ = clean
    assert check(img[:-1]) == 90 and check(img[:S.HEADER.size]) == 90 and check(img[:0]) == 90
    assert check(np.concatenate([img, np.zeros(64, np.uint8)])) == 90
    # the same sections with the bytes region at a 64-byte boundary short of the page: every size consistent
    b, gap = lay["bytes_offset"], 64
    shifted = np.concatenate([img[:b - gap], img[b:]])
    shifted = put(shifted, S.HEADER_OFFSETS["bytes_offset"], "<Q", b - gap)
    shifted = put(shifted, S.HEADER_OFFSETS["total_bytes"], "<Q", lay["total_bytes"] - gap)
    assert check(shifted) == 90


def test_gaps_padding_and_filler(clean):
    img, lay, _ = clean
    region, n = lay["bytes_offset"], lay["nbytes"]
    for at in (S.HEADER.size, lay["files_offset"] + lay["files_bytes"], lay["descs_offset"] + lay["descs_bytes"],
               region + n, region + n + 11, lay["total_bytes"] - 1,  # filler frame, padding
               lay["files_offset"] + 28):  # a record's STREAMINFO padding
        assert check(put(img, at, "<B", img[at] ^ 0x20)) == 90, at
    f = lay["n_frames"]  # the filler's descriptor
    for field in ("byte_offset", "byte_len", "flags", "out_offset"):
        fmt = {"byte_offset": "<Q", "byte_len": "<I", "flags": "<B", "out_offset": "<Q"}[field]
        assert check(put(img, desc(lay, f, field), fmt, get(img, desc(lay, f, field), fmt) + 1)) == 90, field
    # the files' bytes themselves are not checked: they are what the frames decode to
    assert check(put(img, region + 100, "<B", img[region + 100] ^ 0x20)) == 0


def test_descriptors(clean):
    img, lay, files = clean
    n = lay["n_frames"]
    first_of_2 = files[0][2].size
    last = n - 1
    assert check(put(img, desc(lay, last, "byte_len"), "<I", get(img, desc(lay, last, "byte_len"), "<I") + 1)) == 90
    assert check(put(img, desc(lay, 3, "byte_offset"), "<Q", lay["nbytes"])) == 90  # past the bytes
    assert check(put(img, desc(lay, first_of_2 - 1, "byte_len"), "<I",  # into the next file's bytes
                     get(img, desc(lay, first_of_2 - 1, "byte_len"), "<I") + 1)) == 90
    # frames out of byte order within a file
    a, b = desc(lay, 4, "byte_offset"), desc(lay, 5, "byte_offset")
    swapped = img.copy()
    swapped[a:a + 40], swapped[b:b + 40] = img[b:b + 40], img[a:a + 40]
    assert check(swapped) == 90
    assert check(put(img, desc(lay, 2, "n_channels"), "<B", get(img, desc(lay, 2, "n_channels"), "<B") + 1)) == 90
    assert check(put(img, desc(lay, 2, "n_channels"), "<B", 9)) == 90
    assert check(put(img, desc(lay, 2, "flags"), "<B", get(img, desc(lay, 2, "flags"), "<B") | 4)) == 90
    assert check(put(img, desc(lay, 2, "out_offset"), "<Q", 4)) == 90
    # a first frame that does not start its file's bytes
    assert check(put(img, desc(lay, first_of_2, "byte_offset"), "<Q",
                     get(img, desc(lay, first_of_2, "byte_offset"), "<Q") + 1)) == 90


def test_file_records(clean):
    img, lay, files = clean
    for i in range(len(files)):
        for field in ("byte_base", "byte_count", "first_frame", "n_frames"):
            fmt = "<Q" if field.startswith("byte") else "<I"
            v = get(img, record(lay, i, field), fmt)
            for bad in {v + 1, v - 1 if v else 7}:
                assert check(put(img, record(lay, i, field), fmt, bad)) == 90, (i, field, bad)
        for flags in (0, 2, 3, 1 << 31):
            assert check(put(img, record(lay, i, "flags"), "<I", flags)) == 90, (i, flags)
    # frame ranges that decrease: file 1 takes one frame from file 0, with consistent counts
    n0 = get(img, record(lay, 0, "n_frames"), "<I")
    bad = put(img, record(lay, 0, "n_frames"), "<I", n0 - 1)
    bad = put(bad, record(lay, 1, "first_frame"), "<I", n0 - 1)
    bad = put(bad, record(lay, 1, "n_frames"), "<I", get(img, record(lay, 1, "n_frames"), "<I") + 1)
    assert check(bad) == 90


def test_writer_and_attach_refuse_without_a_context(clean):
    img, _, _ = clean
    L = _lib.load()
    h = C.c_void_p()
    assert L.clx_corpus_attach(None, img.ctypes.data, img.size, C.byref(h)) == 90 and not h.value
    assert L.clx_corpus_image_write(None, None, None, None, 0, None, 0, None, img.ctypes.data, img.size) == 90
    ff = np.array([0, 5, 3], np.uint32)  # decreasing file_frames
    sizes = np.array([100, 100], np.uintp)
    d = np.zeros(3, cb.DESC_DTYPE)
    assert L.clx_corpus_image_bytes(sizes.ctypes.data, d.ctypes.data, 3, ff.ctypes.data, 2) == 0


def test_shared_entry_points_are_exported():
    lib = C.CDLL(_lib.load()._name)
    for name in ("clx_corpus_image_bytes", "clx_corpus_image_write", "clx_corpus_image_check", "clx_corpus_attach"):
        assert hasattr(lib, name) and name in _lib.SYMBOLS, name
    assert struct.pack("<Q", _lib.IMAGE_MAGIC) == S.MAGIC and _lib.IMAGE_ALIGN == S.ALIGN


def test_share_refuses_an_existing_path(golden, tmp_path):
    p = tmp_path / "corpus.clxc"
    p.write_bytes(b"x")
    with pytest.raises(FileExistsError):
        cb.Corpus.share(cb.index(golden["short__bytes"]), p, ctx=object())
    assert p.read_bytes() == b"x" and sorted(x.name for x in tmp_path.iterdir()) == ["corpus.clxc"]
