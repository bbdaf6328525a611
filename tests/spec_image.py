"""The corpus image layout (include/claxon_b200.h, "Shared host corpora") restated in plain Python from the header's
documentation: what clx_corpus_image_write must produce byte for byte, and what clx_corpus_image_check must accept.

Nothing here calls the library's image code.  The inputs are what the writer gets: each file's bytes, its STREAMINFO
and its frame descriptors (byte_offset into that file's bytes), plus the trailing-bytes verdict of each file (the
writer decodes an unconfirmed last frame to get it; here it is given).  The filler frame and its descriptor are
inputs too (the library exposes the frame as clx_crop_filler_frame)."""
import struct

import numpy as np

MAGIC = b"CLXCORP1"
VERSION = 1
ALIGN = 4096
END_CONFIRMED = 1
CRC16_VERIFIED = 2
HEADER = struct.Struct("<8sII10Q")          # magic, version, header_bytes, then ten u64 fields
FILE = struct.Struct("<7I4xQ16sQQIIIi")     # STREAMINFO (4 pad bytes before samples), base, count, range, flags, tail
DESC = struct.Struct("<QIHHBBBBIQQ")
HEADER_FIELDS = ("n_files", "n_frames", "files_offset", "files_bytes", "descs_offset", "descs_bytes", "bytes_offset",
                 "bytes_size", "nbytes", "total_bytes")
assert HEADER.size == 96 and FILE.size == 88 and DESC.size == 40

# where each header field sits: magic 0, version 8, header_bytes 12, then the u64 fields from 16 on
HEADER_OFFSETS = {"magic": 0, "version": 8, "header_bytes": 12, **{n: 16 + 8 * i for i, n in enumerate(HEADER_FIELDS)}}


def up(x, a):
    return (x + a - 1) // a * a


def layout(n_files, n_frames, nbytes, filler_len):
    files_offset = 128
    files_bytes = n_files * FILE.size
    descs_offset = up(files_offset + files_bytes, 64)
    descs_bytes = (n_frames + 1) * DESC.size
    bytes_offset = up(descs_offset + descs_bytes, ALIGN)
    bytes_size = up(nbytes + filler_len, 64) + 128
    return dict(n_files=n_files, n_frames=n_frames, files_offset=files_offset, files_bytes=files_bytes,
                descs_offset=descs_offset, descs_bytes=descs_bytes, bytes_offset=bytes_offset, bytes_size=bytes_size,
                nbytes=nbytes, total_bytes=bytes_offset + bytes_size)


def pack_desc(d, byte_offset):
    return DESC.pack(byte_offset, int(d["byte_len"]), int(d["header_len"]), int(d["block_size"]), int(d["n_channels"]),
                     int(d["channel_assignment"]), int(d["bits_per_sample"]), int(d["flags"]), int(d["sample_rate"]),
                     int(d["number"]), 0)


def image(files, filler, filler_desc, tails=None):
    """files: (data, info, descs) per file, `info` with claxon_b200.StreamInfo's fields.  Returns (image as a uint8
    array, the header's fields as a dict)."""
    tails = tails or [0] * len(files)
    records, descs, chunks = [], [], []
    base = frame = 0
    for (data, info, d), tail in zip(files, tails):
        data = np.asarray(data, dtype=np.uint8)
        if d.size:
            first = int(d["byte_offset"][0])
            chunk = data[first:].tobytes()
            descs += [pack_desc(x, int(x["byte_offset"]) - first + base) for x in d]
            confirmed = bool(int(d["flags"][-1]) & CRC16_VERIFIED)
        else:
            chunk, confirmed = b"", True
        records.append(FILE.pack(info.min_block_size, info.max_block_size, info.min_frame_size or 0,
                                 info.max_frame_size or 0, info.sample_rate, info.channels, info.bits_per_sample,
                                 info.samples or 0, bytes(info.md5sum), base, len(chunk), frame, d.size,
                                 END_CONFIRMED if confirmed else 0, tail))
        chunks.append(chunk)
        base += len(chunk)
        frame += d.size
    lay = layout(len(files), frame, base, len(filler))
    descs.append(pack_desc(filler_desc, base))
    out = bytearray(lay["total_bytes"])
    out[:HEADER.size] = HEADER.pack(MAGIC, VERSION, HEADER.size, *(lay[n] for n in HEADER_FIELDS))
    out[lay["files_offset"]:lay["files_offset"] + lay["files_bytes"]] = b"".join(records)
    out[lay["descs_offset"]:lay["descs_offset"] + lay["descs_bytes"]] = b"".join(descs)
    region = lay["bytes_offset"]
    out[region:region + base] = b"".join(chunks)
    out[region + base:region + base + len(filler)] = filler
    return np.frombuffer(bytes(out), dtype=np.uint8).copy(), lay


def filler_of(lib):
    """The filler frame's bytes (clx_crop_filler_frame) and its descriptor as the header documents it: the frame's
    parsed header, its exact byte_len, flags CRC16_VERIFIED, out_offset 0 (byte_offset is set by image())."""
    import ctypes as C
    import claxon_b200 as cb
    buf = (C.c_uint8 * 64)()
    n = lib.clx_crop_filler_frame(buf, 64)
    frame = bytes(buf[:n])
    st, d = cb.parse_frame_header(frame)
    assert st == 0
    desc = np.frombuffer(bytes(d), dtype=cb.DESC_DTYPE)[0].copy()
    desc["byte_len"] = n
    desc["flags"] |= CRC16_VERIFIED
    return frame, desc
