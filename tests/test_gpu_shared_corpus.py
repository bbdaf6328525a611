"""Shared host corpora: corpus images written by Corpus.share() and attached by Corpus.attach() (-m gpu).

An attached corpus is a host corpus whose pinned bytes are the pages of an image file on /dev/shm, registered with
cudaHostRegister, instead of a private copy.  Every call is compared with the same call over a host corpus and a device
corpus of the same index: out, lengths, starts, status and the error word.  The host corpus takes the same gather path
over the same bytes, so it must agree bit for bit everywhere, failed crops included; the device corpus everywhere but
the rows of failed crops (which are unspecified).  Images are removed in `finally`.
"""
import contextlib
import gc
import mmap
import os
import uuid

import numpy as np
import pytest

import claxon_b200 as cb
from claxon_b200 import _lib, synth
from tests import spec_image as S
from tests.test_gpu_batch_out import corruption_corpus
from tests.test_gpu_corpus import bits, damaged_index, files_1_2_4, flac_of, requests_of

gpu = pytest.mark.gpu


@contextlib.contextmanager
def image_path():
    p = os.path.join("/dev/shm", f"clx-test-{os.getpid()}-{uuid.uuid4().hex}.clxc")
    try:
        yield p
    finally:
        if os.path.lexists(p):
            os.unlink(p)


def crop_call(batch, files, offsets):
    out, lengths = batch(files, offsets, check=False)
    return [bits(out).clone(), lengths.clone(), batch.status.clone(), batch._error.clone()]


def packed_call(batch, files, offsets, lengths):
    out, starts, ln = batch(files, offsets, lengths, check=False)
    return [bits(out).clone(), starts.clone(), ln.clone(), batch.status.clone(), batch._error.clone()]


def agree(att, host, dev, crops=True):
    """att and host equal in everything; att and dev in all but the output of failed crops / excerpts."""
    import torch
    assert all(torch.equal(a, h) for a, h in zip(att, host))
    assert all(torch.equal(a, d) for a, d in zip(att[1:], dev[1:]))
    status = att[-2]
    if crops:  # compare the rows of the crops that decoded
        ok = (status == 0).nonzero().flatten()
        assert torch.equal(att[0][ok], dev[0][ok])
    elif not status.any():
        assert torch.equal(att[0], dev[0])
    return status.cpu().tolist()


def three(idx, ctx, path):
    return cb.Corpus.share(idx, path, ctx), cb.Corpus(idx, ctx, memory="host"), cb.Corpus(idx, ctx)


def index_bytes(corpus):
    nf, nfiles = corpus.descs.size, len(corpus.index)
    return (nf + 1) * 40 + max(nf, 1) * 8 + (nfiles + 1) * 4 + max(nfiles, 1) * (8 + 4 + 4)


# --------------------------------------------------------------------------- 1. the image and the rebuilt index

@gpu
def test_written_image_equals_the_statement(ctx, golden):
    idx = cb.index([golden["pop__bytes"], flac_of(synth.workload_config("c2", 9)), golden["short__bytes"]])
    with image_path() as p:
        att = cb.Corpus.share(idx, p, ctx)
        with open(p, "rb") as f:
            written = np.frombuffer(f.read(), np.uint8)
        frame, desc = S.filler_of(_lib.load())
        expect, lay = S.image([(f.data, f.info, f.descs) for f in idx.files], frame, desc)
        assert written.size == expect.size and lay["bytes_offset"] % 4096 == 0
        assert np.array_equal(written, expect), np.nonzero(written != expect)[0][:8]
        assert att.memory == "shared" and att.path == p
        att.close()
        assert not [x for x in os.listdir("/dev/shm") if x.startswith(f".{os.path.basename(p)}")]  # no temporary left


@gpu
def test_rebuilt_index_and_load_crops(ctx, golden):
    import torch
    idx = cb.index(files_1_2_4(golden))
    with image_path() as p:
        att, host, _ = three(idx, ctx, p)
        assert np.array_equal(att.descs, host.descs) and np.array_equal(att.file_frames, host.file_frames)
        assert att.nbytes == host.nbytes and att.channels == host.channels
        for a, f in zip(att.index.files, idx.files):
            first = int(f.descs["byte_offset"][0])
            assert a.info == f.info and a.length == f.length and a.end_confirmed == f.end_confirmed
            assert np.array_equal(a.starts, f.starts) and not a.data.flags.writeable
            assert np.array_equal(a.data, f.data[first:])
            d = f.descs.copy()
            d["byte_offset"] -= np.uint64(first)
            d["out_offset"] = 0
            assert np.array_equal(a.descs, d)
        files, offsets = requests_of(idx)
        for dtype in (torch.float32, torch.int32):
            exp, el = cb.load_crops(idx, files, offsets, 1000, dtype=dtype, ctx=ctx)
            got, gl = cb.load_crops(att.index, files, offsets, 1000, dtype=dtype, ctx=ctx)
            assert torch.equal(bits(exp), bits(got)) and torch.equal(el, gl)
        assert att.device_bytes == host.device_bytes == index_bytes(att)
        assert att.frames_bound(5000) == host.frames_bound(5000) and att.bytes_bound(5000) == host.bytes_bound(5000)
        assert att.packed_bytes_bound(8, 50000) == host.packed_bytes_bound(8, 50000)


# --------------------------------------------------------------------------- 2. crops and packed batches

@gpu
@pytest.mark.parametrize("dtype_name", ["float32", "int32"])
def test_crops_and_packed_agree(ctx, golden, dtype_name):
    import torch
    dtype = getattr(torch, dtype_name)
    idx = cb.index(files_1_2_4(golden))
    files, offsets = requests_of(idx)
    B, n = len(files), len(idx)
    longest = max(f.length for f in idx.files)
    with image_path() as p:
        corpora = three(idx, ctx, p)
        for L in (1, 37, 3 * 4096 + 5, longest + 3):
            batches = [c.crops(B, L, dtype=dtype) for c in corpora]
            for f, o in (([b % n for b in range(B)], [0] * B), (files, offsets)):  # long spans, then short ones
                assert agree(*[crop_call(b, f, o) for b in batches]) == [0] * len(f)
            del batches
        T = sum((f.length + 3) & ~3 for f in idx.files)
        batches = [c.packed(2 * n, T, dtype=dtype) for c in corpora]
        rng = np.random.default_rng(3)
        whole = (list(range(n)), None, None)
        excerpts = ([int(x) for x in rng.integers(0, n, 2 * n)], None, None)
        excerpts = (excerpts[0], [int(rng.integers(0, idx[f].length)) for f in excerpts[0]],
                    [int(rng.integers(1, 30000)) for _ in excerpts[0]])
        for f, o, ln in (whole, excerpts, whole):
            st = agree(*[packed_call(b, f, o, ln) for b in batches], crops=False)
            assert st == [0] * len(f) or f is excerpts[0]  # (excerpts may not all fit)


@gpu
@pytest.mark.parametrize("dtype_name", ["float32", "int32"])
def test_damaged_files(ctx, golden, dtype_name):
    """Failed frames, a CRC-16 mismatch and trailing bytes after an unconfirmed last frame: the verdict is the image's."""
    import torch
    dtype = getattr(torch, dtype_name)
    idx = damaged_index(golden)
    s0 = int(idx[0].starts[16])
    files = [3, 0, 0, 1, 2, 2, 0, 3, 1, 2]
    offsets = [0, 0, s0 + 4086, int(idx[1].starts[9]) + 5, 0, idx[2].length - 100, s0 + 10, 50, 0, idx[2].length - 1]
    with image_path() as p:
        corpora = three(idx, ctx, p)
        batches = [c.crops(len(files), 3000, dtype=dtype) for c in corpora]
        agree(*[crop_call(b, [b_ % 4 for b_ in range(len(files))], [0] * len(files)) for b in batches])
        st = agree(*[crop_call(b, files, offsets) for b in batches])
        assert st[2] != 0 and st[3] == 23 and st[5] != 0 and st[0] == st[4] == 0
        with pytest.raises(cb.Error) as e_att:
            batches[0](files, offsets)
        with pytest.raises(cb.Error) as e_host:
            batches[1](files, offsets)
        assert str(e_att.value) == str(e_host.value)
        packed = [c.packed(8, 400000, dtype=dtype) for c in corpora]
        for f, o, ln in (([0, 1, 2, 3], None, None), ([2, 0, 1], [idx[2].length - 100, s0, 0], [100, 9000, 50000])):
            agree(*[packed_call(b, f, o, ln) for b in packed], crops=False)


@gpu
def test_corruption_corpus(ctx):
    import torch
    data, offsets, lengths = corruption_corpus()
    descs, _ = cb.descs_from_offsets(data, offsets, lengths)
    files = []
    for i in range(0, descs.size, 4):
        o, n = int(offsets[i]), int(lengths[i])
        d = descs[i:i + 1].copy()
        d["byte_offset"], d["out_offset"] = 0, 0
        info = cb.StreamInfo(576, 576, None, None, 44100, int(d["n_channels"][0]), int(d["bits_per_sample"][0]), None,
                             bytes(16))
        files.append(cb.IndexedFile(data[o:o + n].copy(), info, d, cb.frame_starts(d), int(d["block_size"][0]), False))
    idx = cb.FlacIndex(files)
    fs = list(range(len(files)))
    with image_path() as p:
        corpora = three(idx, ctx, p)
        batches = [c.crops(len(fs), 300, dtype=torch.int32) for c in corpora]
        agree(*[crop_call(b, fs, [0] * len(fs)) for b in batches])
        st = agree(*[crop_call(b, fs, [min(i % 5 * 100, files[i].length) for i in fs]) for b in batches])
        assert len(set(st)) >= 4, sorted(set(st))
        packed = [c.packed(len(fs), 300 * len(fs), dtype=torch.int32) for c in corpora]
        agree(*[packed_call(b, fs, None, [200] * len(fs)) for b in packed], crops=False)


# --------------------------------------------------------------------------- 3. another process

def seeded_requests(idx, seed):
    rng = np.random.default_rng(seed)
    files = [int(x) for x in rng.integers(0, len(idx), 48)]
    offsets = [int(rng.integers(0, idx[f].length + 1)) for f in files]
    pf = [int(x) for x in rng.integers(0, len(idx), 6)]
    po = [int(rng.integers(0, idx[f].length)) for f in pf]
    pl = [int(rng.integers(1, 40000)) for _ in pf]
    return files, offsets, pf, po, pl


def run_seeded(corpus, seed):
    import torch
    files, offsets, pf, po, pl = seeded_requests(corpus.index, seed)
    res = []
    for dtype in (torch.float32, torch.int32):
        res += [t.cpu().numpy() for t in crop_call(corpus.crops(len(files), 5000, dtype=dtype), files, offsets)]
        res += [t.cpu().numpy() for t in packed_call(corpus.packed(8, 200000, dtype=dtype), pf, po, pl)]
    return res


def _child(path, q):
    try:
        import claxon_b200 as cb_
        corpus = cb_.Corpus.attach(path, cb_.Context(device=0))
        q.put(("ok", corpus.device_bytes, index_bytes(corpus), run_seeded(corpus, 11)))
    except BaseException as e:  # reported to the parent, which fails at once instead of at its timeout
        import traceback
        q.put(("error", repr(e), traceback.format_exc(), None))


@gpu
def test_second_process_attaches_the_same_image(ctx, golden):
    import torch.multiprocessing as mp
    idx = cb.index(files_1_2_4(golden)[:5])
    with image_path() as p:
        att = cb.Corpus.share(idx, p, ctx)
        mine = run_seeded(att, 11)
        spawn = mp.get_context("spawn")
        q = spawn.Queue()
        proc = spawn.Process(target=_child, args=(p, q))
        proc.start()
        try:
            kind, dev_bytes, want, theirs = q.get(timeout=300)
            assert kind == "ok", (dev_bytes, want)
            proc.join(timeout=120)
            assert proc.exitcode == 0
        finally:
            if proc.is_alive():
                proc.terminate()
                proc.join(timeout=30)
        assert dev_bytes == want == att.device_bytes
        assert len(theirs) == len(mine) and all(np.array_equal(a, b) for a, b in zip(mine, theirs))
        assert not any(a.any() for a in mine[2::9])  # (every crop of the first call decoded)


# --------------------------------------------------------------------------- 4. registration, refusals, lifetime

@gpu
def test_one_mapping_attached_twice_destroyed_in_either_order(ctx, golden):
    import torch
    idx = cb.index(files_1_2_4(golden)[:4])
    files, offsets = requests_of(idx)
    with image_path() as p:
        host = cb.Corpus(idx, ctx, memory="host")
        want = crop_call(host.crops(len(files), 3000, dtype=torch.int32), files, offsets)
        cb.Corpus.share(idx, p, ctx).close()
        ctx2 = cb.Context(device=0)
        with open(p, "r+b") as f:
            mm = mmap.mmap(f.fileno(), 0)
        try:
            def use(c):
                got = crop_call(c.crops(len(files), 3000, dtype=torch.int32), files, offsets)
                assert all(torch.equal(a, b) for a, b in zip(got, want))
            for first_closed in (0, 1):
                pair = [cb.Corpus.attach(mm, ctx), cb.Corpus.attach(mm, ctx2)]
                use(pair[0])
                use(pair[1])
                pair[first_closed].close()
                use(pair[1 - first_closed])
                pair[1 - first_closed].close()
            # a refused attach of the same mapping registers nothing: the next attach still registers it afresh
            img = np.frombuffer(mm, np.uint8)
            import ctypes as C
            h = C.c_void_p()
            assert ctx._L.clx_corpus_attach(ctx._h, img.ctypes.data, img.size - 1, C.byref(h)) == 90 and not h.value
            del img
            again = cb.Corpus.attach(mm, ctx)
            use(again)
            batch = again.crops(4, 100, dtype=torch.float32)
            with pytest.raises(cb.Error) as e:
                again.close()
            assert e.value.status == 90
            use(again)  # still attached
            del batch
            gc.collect()
            again.close()
        finally:
            ctx2.close()  # (the mapping goes with the last view of it)


@gpu
def test_collected_in_one_cycle_with_its_batches(ctx, golden):
    """A corpus collected in one garbage cycle with its batches (its finalizer may run first, while they are alive)
    still detaches before its mapping goes: later images, mapped wherever the old ones were, attach and decode."""
    import torch
    idx = cb.index(files_1_2_4(golden)[:3])
    files, offsets = requests_of(idx)
    want = crop_call(cb.Corpus(idx, ctx, memory="host").crops(len(files), 3000, dtype=torch.int32), files, offsets)
    for _ in range(4):
        with image_path() as p:
            att = cb.Corpus.share(idx, p, ctx)
            batch = att.crops(len(files), 3000, dtype=torch.int32)
            got = crop_call(batch, files, offsets)
            assert all(torch.equal(a, b) for a, b in zip(got, want))
            cycle = [att, batch, att.packed(4, 10000)]
            cycle.append(cycle)
            del att, batch, cycle
            gc.collect()


@gpu
def test_refused_images_and_unlink_while_attached(ctx, golden):
    import torch
    idx = cb.index(files_1_2_4(golden)[:4])
    files, offsets = requests_of(idx)
    with image_path() as p, image_path() as bad:
        cb.Corpus.share(idx, p, ctx).close()
        with open(p, "rb") as f:
            good = bytearray(f.read())
        for mutate in (lambda b: b.__setitem__(0, b[0] ^ 1), lambda b: b.__setitem__(slice(16, 24), bytes(8))):
            b = bytearray(good)
            mutate(b)
            with open(bad, "wb") as f:
                f.write(b)
            with pytest.raises(cb.Error) as e:
                cb.Corpus.attach(bad, ctx)
            assert e.value.status == 90
            os.unlink(bad)
        with pytest.raises(FileExistsError):
            cb.Corpus.share(idx, p, ctx)
        att = cb.Corpus.attach(p, ctx)
        host = cb.Corpus(idx, ctx, memory="host")
        ab, hb = att.crops(len(files), 2000, dtype=torch.float32), host.crops(len(files), 2000, dtype=torch.float32)
        first = crop_call(ab, files, offsets)
        os.unlink(p)  # the pages stay while the corpus maps them
        for _ in range(2):
            got, want = crop_call(ab, files, offsets), crop_call(hb, files, offsets)
            assert all(torch.equal(a, b) for a, b in zip(got, want)) and torch.equal(got[0], first[0])
        packed = att.packed(4, 100000, dtype=torch.float32)
        out, starts, lengths = packed([0, 1, 2, 3], None, [5000] * 4)
        exp, _ = cb.load_crops(idx, [0, 1, 2, 3], [0] * 4, 5000, dtype=torch.float32, ctx=ctx)
        for b in range(4):
            assert torch.equal(bits(out[:, starts[b]:starts[b] + 5000][:exp.shape[1]]),
                               bits(exp[b, :out.shape[0]]))


@gpu
def test_two_devices_attach_one_mapping(golden):
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip(f"needs two GPUs (contexts on devices 0 and 1 attaching one mapping); this machine has {n}")
    idx = cb.index(files_1_2_4(golden)[:4])
    files, offsets = requests_of(idx)
    with image_path() as p:
        cb.Corpus.share(idx, p, cb.Context(device=0)).close()
        with open(p, "r+b") as f:
            mm = mmap.mmap(f.fileno(), 0)
        try:
            results = []
            for dev in (0, 1):
                with torch.cuda.device(dev):
                    c = cb.Corpus.attach(mm, cb.Context(device=dev))
                    results.append([t.cpu() for t in crop_call(c.crops(len(files), 3000, dtype=torch.int32), files,
                                                                offsets)])
                    torch.cuda.synchronize()
            assert all(torch.equal(a, b) for a, b in zip(*results)) and not results[0][2].any()
        finally:
            gc.collect()
