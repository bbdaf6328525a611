"""Packed batches' host-side bounds and exports (CPU only).

clx_packed_frames_bound must be at least the most frames any set of excerpts that fits in T columns can overlap, and
clx_packed_bytes_bound at least the most span bytes they can select plus 16 per excerpt.  Both are checked against a
brute force: for each excerpt length n, the most frames (or span bytes) plan_range() gives over every offset, then a DP
over every split of at most T samples into at most B excerpts.
"""
import ctypes as C

import numpy as np

import claxon_b200 as cb
from claxon_b200 import _lib
from tests.test_gpu_corpus import blocks_desc, brute_force
from tests.test_gpu_host_corpus import real_spans


def group_args(group):
    descs = np.concatenate(group) if group else np.zeros(0, dtype=cb.DESC_DTYPE)
    ff = np.concatenate([[0], np.cumsum([d.size for d in group])]).astype(np.uint32)
    return descs, ff


def frames_bound(group, B, T):
    descs, ff = group_args(group)
    return int(_lib.load().clx_packed_frames_bound(descs.ctypes.data, descs.size, ff.ctypes.data, len(group), B, T))


def bytes_bound(group, B, T):
    descs, ff = group_args(group)
    return int(_lib.load().clx_packed_bytes_bound(descs.ctypes.data, descs.size, ff.ctypes.data, len(group), B, T))


def best_split(per_n, B, T):
    """The largest sum of per_n[n_j] over at most B excerpts of n_j >= 1 samples, sum n_j <= T."""
    best = np.zeros(T + 1, dtype=np.int64)  # 0 excerpts
    top = 0
    for _ in range(B):
        nxt = best.copy()
        for t in range(1, T + 1):
            n = np.arange(1, t + 1)
            nxt[t] = max(nxt[t], int((best[t - n] + per_n[n]).max()))
        best = np.maximum.accumulate(nxt)
        top = max(top, int(best[T]))
    return top


def groups():
    rng = np.random.default_rng(3)
    return [
        [blocks_desc([64] * 6 + [17])],
        [blocks_desc(rng.integers(16, 90, 10).tolist() + [5]), blocks_desc([40])],
        [blocks_desc([1, 1, 3, 1, 1, 2])],  # 1-sample blocks
        [blocks_desc([50]), blocks_desc([7])],  # 1-frame files only
        [blocks_desc([32] * 4 + [1]), blocks_desc(rng.integers(1, 40, 12).tolist())],
    ]


def test_packed_frames_bound_brute_force():
    for group in groups():
        for T in (1, 2, 3, 5, 17, 64, 150):
            per_n = np.zeros(T + 1, dtype=np.int64)
            for n in range(1, T + 1):
                per_n[n] = max(brute_force(d, n) for d in group)
            for B in (1, 2, 3, 7):
                got = frames_bound(group, B, T)
                assert got >= best_split(per_n, B, T), (T, B, got)
    # the documented formula on a fixed-block corpus, and the refusals
    g = [blocks_desc([4096] * 20 + [1001])]
    assert frames_bound(g, 64, 8_400_000) == min((8_400_000 - 128) // 4096 + 128, 64 * 21)
    assert frames_bound(g, 0, 100) == frames_bound(g, 3, 0) == 0
    assert frames_bound([blocks_desc([5000]), blocks_desc([9])], 5, 10 ** 6) == 5  # no file with two frames


def with_gaps(d, rng):
    """Descriptors with random frame lengths and random gaps between frames."""
    d = d.copy()
    d["byte_len"] = rng.integers(11, 400, d.size)
    gaps = rng.integers(0, 300, d.size)
    d["byte_offset"] = int(rng.integers(0, 100)) + np.concatenate([[0], np.cumsum((d["byte_len"] + gaps)[:-1].astype(np.int64))])
    return d


def test_packed_bytes_bound_brute_force_with_gaps():
    rng = np.random.default_rng(8)
    for group in groups():
        group = [with_gaps(d, rng) for d in group]
        for T in (1, 3, 17, 64, 150):
            per_n = np.zeros(T + 1, dtype=np.int64)
            for n in range(1, T + 1):
                per_n[n] = max(real_spans(d, n) for d in group)
            for B in (1, 2, 5):
                got = bytes_bound(group, B, T)
                assert got >= best_split(per_n, B, T) + 16 * B, (T, B, got)
    assert bytes_bound(groups()[0], 0, 10) == 0


def test_packed_entry_points_are_exported():
    lib = C.CDLL(_lib.load()._name)
    for name in ("clx_batch_create_packed", "clx_packed_frames_bound", "clx_packed_bytes_bound",
                 "clx_batch_packed_requests", "clx_batch_packed_count", "clx_batch_packed_starts",
                 "clx_batch_packed_stride"):
        assert hasattr(lib, name) and name in _lib.SYMBOLS, name
    assert "PackedBatch" in cb.__all__
