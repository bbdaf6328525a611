"""A FLAC file that holds given PCM exactly (test helper, no tests here).

    flac_from_pcm(pcm [C, N] ints, bps, sample_rate, block_size=1024) -> np.ndarray of uint8

Designed signals (impulses, tones, full-scale alternations, silence) reach the device kernels that run after the decode
only through FLAC files.  The frames are written by tests/edge_frames.write: a block whose samples are all equal in a
channel is a `constant` subframe, every other one `verbatim`, so long and mostly silent files stay cheap to write in
Python.  Channels are independent, blocking is fixed (the last block may be shorter), and the STREAMINFO carries the
MD5 of the interleaved little-endian samples.  The frame header names the sample rate by its code where the format has
one, else by code 0 ("from STREAMINFO"), which every decoder here takes.
"""
from __future__ import annotations

import hashlib

import numpy as np

from tests import edge_frames as E

RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10,
              96000: 11}


def md5_of(pcm: np.ndarray, bps: int) -> bytes:
    """The STREAMINFO MD5: the samples interleaved, little-endian, in (bps + 7) // 8 bytes each."""
    nb = (bps + 7) // 8
    raw = np.ascontiguousarray(pcm.T).astype("<i4").view(np.uint8).reshape(-1, 4)[:, :nb]
    return hashlib.md5(raw.tobytes()).digest()


def streaminfo(C_: int, N: int, bps: int, sample_rate: int, block_size: int, md5: bytes) -> bytes:
    w = E.BitWriter()
    w.put(block_size, 16)
    w.put(block_size, 16)
    w.put(0, 24)  # frame sizes unknown
    w.put(0, 24)
    w.put(sample_rate, 20)
    w.put(C_ - 1, 3)
    w.put(bps - 1, 5)
    w.put(N, 36)
    body = w.to_bytes()[0] + md5
    assert len(body) == 34
    return b"fLaC" + bytes([0x80, 0, 0, 34]) + body  # the last metadata block, STREAMINFO, 34 bytes


def flac_from_pcm(pcm, bps: int, sample_rate: int, block_size: int = 1024) -> np.ndarray:
    pcm = np.atleast_2d(np.asarray(pcm, dtype=np.int64))
    C_, N = pcm.shape
    if bps not in E.BPS_CODE or not 1 <= C_ <= 8 or N < 1 or not 16 <= block_size <= 65535:
        raise ValueError("bps in {8, 12, 16, 20, 24}, 1 to 8 channels, N >= 1, block size 16 to 65535")
    if not 1 <= sample_rate <= 655350:
        raise ValueError("sample rate 1 to 655350")
    if pcm.min() < E.lo(bps) or pcm.max() > E.hi(bps):
        raise ValueError(f"samples outside {bps} bits")
    parts = [streaminfo(C_, N, bps, sample_rate, block_size, md5_of(pcm, bps))]
    sr_code = RATE_CODES.get(sample_rate, 0)
    for i, at in enumerate(range(0, N, block_size)):
        blk = pcm[:, at:at + block_size]
        subs = []
        for row in blk:
            v = row.tolist()
            subs.append(E.Sub("constant", [v[0]]) if row.min() == row.max() else E.Sub("verbatim", v))
        parts.append(E.write(E.Frame(bps, subs, block_size=blk.shape[1], number=i, sr_code=sr_code))[0])
    return np.frombuffer(b"".join(parts), np.uint8).copy()
