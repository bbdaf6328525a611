"""claxon_b200 — H100-native batched FLAC frame decoder behind claxon's API surface.

Host-side mirror of the reference interface for the per-frame decode path:

    claxon::FlacReader              -> claxon_b200.FlacReader       (reference src/lib.rs:217-470)
    claxon::frame::FrameReader      -> claxon_b200.FrameReader      (src/frame.rs:650-785)
    claxon::frame::Block            -> claxon_b200.Block            (src/frame.rs:402-529)
    claxon::Error                   -> claxon_b200.Error            (src/error.rs:18-32)

plus the batched entry points the GPU wants (`Context.decode_frames`, `demux_frames`).
All sample arithmetic happens in the CUDA library (`libclaxon_b200.so`); this package is
plumbing.  Nothing here imports the test oracle.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np

from . import _lib
from ._lib import (OPEN_METADATA_ONLY, OPEN_NO_VORBIS_COMMENT)
from ._lib import (FrameDesc, FrameResult, FrameWindow, OPT_NO_VERIFY_CRC, OPT_GENERIC_KERNEL_ONLY, OPT_WARP_PER_FRAME, OPT_LANE_PER_FRAME,
                   OPT_NO_GENERIC, OPT_NO_WIDE, FRAME_VARIABLE_BLOCKING, FRAME_CRC16_VERIFIED,
                   OUT_PLANAR_I32, OUT_INTERLEAVED_I32, OUT_INTERLEAVED_I16, OUT_INTERLEAVED_I24,
                   OUT_CHANNELS_I32, OUT_CHANNELS_F32, MEL_CENTER, MEL_LOG, MEL_NORM_PER_FEATURE,
                   MEL_NORM_WHISPER)

__all__ = ["Error", "Block", "FrameReader", "FlacReader", "FlacReaderOptions", "StreamInfo", "Context", "DeviceBatch",
           "parse_frame_header", "demux_frames", "open_stream", "ogg_frames", "mp4_frames", "status_str", "DESC_DTYPE", "RESULT_DTYPE", "load", "plan_columns",
           "WINDOW_DTYPE", "index", "FlacIndex", "IndexedFile", "load_crops", "plan_range", "frame_starts", "Corpus",
           "CropBatch", "PackedBatch", "MelCropBatch", "MelPackedBatch", "melscale_fbanks"]

# numpy views of the C structs (same layout; asserted below)
DESC_DTYPE = np.dtype([
    ("byte_offset", "<u8"), ("byte_len", "<u4"), ("header_len", "<u2"), ("block_size", "<u2"),
    ("n_channels", "u1"), ("channel_assignment", "u1"), ("bits_per_sample", "u1"), ("flags", "u1"),
    ("sample_rate", "<u4"), ("number", "<u8"), ("out_offset", "<u8")], align=True)
RESULT_DTYPE = np.dtype([("status", "<i4"), ("consumed", "<u4")], align=True)
WINDOW_DTYPE = np.dtype([("row", "<u4"), ("first", "<u4"), ("count", "<u4"), ("reserved", "<u4")], align=True)
assert DESC_DTYPE.itemsize == C.sizeof(FrameDesc) and RESULT_DTYPE.itemsize == C.sizeof(FrameResult)
assert WINDOW_DTYPE.itemsize == C.sizeof(FrameWindow)

KIND_NONE, KIND_IO, KIND_FORMAT, KIND_UNSUPPORTED, KIND_LIBRARY = range(5)
OK, EOF = 0, 1


def status_str(status: int) -> str:
    return _lib.load().clx_status_str(int(status)).decode()


class Error(Exception):
    """claxon::Error — compares by variant + message like the reference (src/error.rs:34-45)."""

    def __init__(self, status: int, detail: str = ""):
        self.status = int(status)
        self.kind = _lib.load().clx_status_kind(self.status)
        self.message = status_str(self.status)
        super().__init__(self.message + (f" ({detail})" if detail else ""))

    @property
    def variant(self) -> str:
        return {KIND_IO: "IoError", KIND_FORMAT: "FormatError", KIND_UNSUPPORTED: "Unsupported"}.get(
            self.kind, "LibraryError")

    def __eq__(self, other):
        if not isinstance(other, Error):
            return NotImplemented
        if self.kind == KIND_IO or other.kind == KIND_IO:
            return False  # (&IoError(_), _) => false
        return self.kind == other.kind and self.message == other.message

    __hash__ = Exception.__hash__


def _check(status: int, ctx: "Context | None" = None):
    if status != OK:
        detail = ""
        if ctx is not None and status == 91:
            detail = _lib.load().clx_ctx_last_error(ctx._h).decode()
        raise Error(status, detail)


def _as_u8(data) -> np.ndarray:
    if isinstance(data, np.ndarray):
        if data.dtype != np.uint8 or not data.flags.c_contiguous:
            data = np.ascontiguousarray(data, dtype=np.uint8)
        return data
    return np.frombuffer(bytes(data) if not isinstance(data, (bytes, bytearray, memoryview)) else data,
                         dtype=np.uint8)


# ---------------------------------------------------------------------------
# host-side parsing
# ---------------------------------------------------------------------------

@dataclass
class StreamInfo:  # claxon::metadata::StreamInfo (src/metadata.rs:29-54)
    min_block_size: int
    max_block_size: int
    min_frame_size: int | None
    max_frame_size: int | None
    sample_rate: int
    channels: int
    bits_per_sample: int
    samples: int | None
    md5sum: bytes

    @staticmethod
    def _from_c(si) -> "StreamInfo":
        return StreamInfo(si.min_block_size, si.max_block_size, si.min_frame_size or None,
                          si.max_frame_size or None, si.sample_rate, si.channels, si.bits_per_sample,
                          si.samples or None, bytes(si.md5sum))


def parse_frame_header(data, offset: int = 0, flags: int = 0):
    """read_frame_header_or_eof (src/frame.rs:131-316). Returns (status, FrameDesc)."""
    buf = _as_u8(data)
    d = FrameDesc()
    st = _lib.load().clx_parse_frame_header(buf.ctypes.data + offset, buf.size - offset, C.byref(d), flags)
    return st, d


def open_stream(data):
    """FlacReader::new's metadata walk. Returns (StreamInfo, first_frame_offset); raises Error."""
    buf = _as_u8(data)
    si = _lib.StreamInfoC()
    first = C.c_uint64(0)
    _check(_lib.load().clx_open_stream(buf.ctypes.data, buf.size, C.byref(si), C.byref(first)))
    return StreamInfo._from_c(si), first.value


def demux_frames(data, start: int = 0, max_frames: int = 1 << 20, flags: int = 0, threads: int = 1):
    """Finds frame boundaries without decoding. Returns (descs ndarray, next_offset, out_elems, stop_status).
    `threads` != 1: clx_demux_frames_mt on that many host threads (0 = all), same results."""
    buf = _as_u8(data)
    cap = min(max_frames, max(16, (buf.size - start) // 16 + 1))
    while True:
        descs = np.empty(cap, dtype=DESC_DTYPE)  # (filled by the call; zeroing 40 bytes per possible frame costs more than the scan)
        nxt, total, stop = C.c_uint64(0), C.c_uint64(0), C.c_int(0)
        if threads == 1:
            n = _lib.load().clx_demux_frames(buf.ctypes.data, buf.size, start, descs.ctypes.data, cap,
                                             C.byref(nxt), C.byref(total), C.byref(stop), flags)
        else:
            n = _lib.load().clx_demux_frames_mt(buf.ctypes.data, buf.size, start, descs.ctypes.data, cap,
                                                C.byref(nxt), C.byref(total), C.byref(stop), flags, threads)
        if n < cap or cap >= max_frames:
            return descs[:n].copy(), nxt.value, total.value, stop.value
        cap = min(max_frames, cap * 4)


def ogg_frames(data, flags: int = 0):
    """Frames of an in-memory Ogg FLAC file (examples/decode_ogg.rs): (StreamInfo, frame bytes, descs, out_elems);
    the descriptors index the returned byte array (packets may span pages in the file)."""
    buf = _as_u8(data)
    si = _lib.StreamInfoC()
    frames = np.zeros(max(16, buf.size), dtype=np.uint8)
    descs = np.zeros(max(16, buf.size // 8), dtype=DESC_DTYPE)
    n, used, total = C.c_size_t(0), C.c_size_t(0), C.c_uint64(0)
    _check(_lib.load().clx_ogg_frames(buf.ctypes.data, buf.size, C.byref(si), frames.ctypes.data, frames.size,
                                      descs.ctypes.data, descs.size, C.byref(n), C.byref(used), C.byref(total), flags))
    return StreamInfo._from_c(si), frames[: used.value].copy(), descs[: n.value].copy(), int(total.value)


def mp4_frames(data, flags: int = 0):
    """Frames of an in-memory MP4 file with a 'fLaC' track (examples/decode_mp4.rs): (StreamInfo, descs, out_elems);
    the descriptors index `data` itself."""
    buf = _as_u8(data)
    si = _lib.StreamInfoC()
    descs = np.zeros(max(16, buf.size // 8), dtype=DESC_DTYPE)
    n, total = C.c_size_t(0), C.c_uint64(0)
    _check(_lib.load().clx_mp4_frames(buf.ctypes.data, buf.size, C.byref(si), descs.ctypes.data, descs.size, C.byref(n),
                                      C.byref(total), flags))
    return StreamInfo._from_c(si), descs[: n.value].copy(), int(total.value)


def descs_from_offsets(data, offsets, lengths=None, flags: int = 0) -> tuple[np.ndarray, int]:
    """Builds descriptors for frames at known byte offsets (container-provided boundaries,
    cf. reference examples/decode_ogg.rs:107-113). Returns (descs, out_elems)."""
    buf = _as_u8(data)
    offsets = np.asarray(offsets, dtype=np.uint64)
    descs = np.zeros(offsets.size, dtype=DESC_DTYPE)
    L = _lib.load()
    out_at = 0
    d = FrameDesc()
    for i, off in enumerate(offsets):
        off = int(off)
        ln = int(lengths[i]) if lengths is not None else buf.size - off
        st = L.clx_parse_frame_header(buf.ctypes.data + off, ln, C.byref(d), flags)
        if st != OK:
            raise Error(st, f"frame {i}")
        d.byte_offset, d.byte_len, d.out_offset = off, ln, out_at
        descs[i] = np.frombuffer(bytes(d), dtype=DESC_DTYPE)[0]
        out_at += (d.n_channels * d.block_size + 3) & ~3
    return descs, out_at


# ---------------------------------------------------------------------------
# device context
# ---------------------------------------------------------------------------

class Context:
    """clx_ctx: one per host thread / GPU. Raises Error(NO_DEVICE) without a usable GPU."""

    def __init__(self, device: int = 0, verify_crc: bool = True, n_streams: int = 2, generic_only: bool = False,
                 warp_per_frame: bool = False, lane_per_frame: bool = False, host_threads: int = 0,
                 no_generic: bool = False, no_wide: bool = False):
        """Default: device-resident batches and large calls use the lane-per-frame index pass + lane-per-subframe
        decode pass (csrc/clx_fused.cu); small synchronous host-buffer calls (latency regime) use the
        warp-per-frame path (csrc/clx_coop.cu).  `warp_per_frame` / `lane_per_frame` force one of them everywhere,
        `generic_only` bypasses both (testing, A/B measurements).  `no_generic` / `no_wide` (testing) switch off
        the kernels that take over what a fast path declined: such frames then come back with status -2 (the
        generic kernel would have decoded them) or -3 (the lane-per-frame path's i64 second chance would have)."""
        self._L = _lib.load()
        flags = ((0 if verify_crc else OPT_NO_VERIFY_CRC) | (OPT_GENERIC_KERNEL_ONLY if generic_only else 0)
                 | (OPT_WARP_PER_FRAME if warp_per_frame else 0) | (OPT_LANE_PER_FRAME if lane_per_frame else 0)
                 | (OPT_NO_GENERIC if no_generic else 0) | (OPT_NO_WIDE if no_wide else 0))
        opts = _lib.Options(device, flags, n_streams, host_threads)
        h = C.c_void_p()
        _check(self._L.clx_ctx_create(C.byref(opts), C.byref(h)))
        self._h = h
        self.verify_crc = verify_crc

    def close(self):
        if getattr(self, "_h", None):
            self._L.clx_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launch_count(self) -> int:
        return int(self._L.clx_ctx_launch_count(self._h))

    def decode_frames(self, data, descs: np.ndarray, out: np.ndarray | None = None,
                      out_elems: int | None = None, mode: int = OUT_PLANAR_I32):
        """End-to-end host-buffer decode. Returns (out ndarray, results ndarray).  `mode`: OUT_PLANAR_I32 (claxon's
        Block layout, int32) or an interleaved little-endian form: OUT_INTERLEAVED_I32 (int32), _I16 (int16),
        _I24 (uint8, 3 bytes per sample); out_offset / out_elems count samples in every mode."""
        buf = _as_u8(data)
        descs = np.ascontiguousarray(descs, dtype=DESC_DTYPE)
        if out_elems is None:
            ends = descs["out_offset"] + descs["n_channels"].astype(np.uint64) * descs["block_size"]
            out_elems = int(ends.max()) if descs.size else 0
        if out is None:
            out = _out_array(out_elems, mode)
        results = np.zeros(descs.size, dtype=RESULT_DTYPE)
        _check(self._L.clx_decode_frames_to(self._h, buf.ctypes.data, buf.size, descs.ctypes.data, descs.size,
                                            out.ctypes.data, max(1, out_elems), results.ctypes.data, mode), self)
        return out, results

    def decode_frames_raw(self, bytes_ptr: int, nbytes: int, descs_ptr: int, n: int, out_ptr: int,
                          out_elems: int, results_ptr: int, mode: int = OUT_PLANAR_I32):
        """Same call on raw host addresses (pinned buffers owned by the caller)."""
        _check(self._L.clx_decode_frames_to(self._h, bytes_ptr, nbytes, descs_ptr, n, out_ptr, out_elems,
                                            results_ptr, mode), self)

    def run_steps(self, batches: list["DeviceBatch"], steps: int, n_streams: int) -> float:
        """Decodes `steps` batches round-robin over `n_streams` streams; returns device ms (CUDA events)."""
        arr = (C.c_void_p * len(batches))(*[b._h for b in batches])
        ms = C.c_float(0)
        _check(self._L.clx_ctx_run_steps(self._h, arr, len(batches), steps, n_streams, C.byref(ms)), self)
        return float(ms.value)

    def host_alloc(self, nbytes: int) -> np.ndarray:
        """Pinned host buffer as a uint8 ndarray (freed with host_free)."""
        p = self._L.clx_host_alloc(nbytes)
        if not p:
            raise MemoryError("cudaHostAlloc failed")
        return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p))

    def host_free(self, arr: np.ndarray):
        self._L.clx_host_free(arr.ctypes.data)

    def upload(self, data, descs: np.ndarray, out_elems: int | None = None, mode: int = OUT_PLANAR_I32,
               channels: int | None = None, channel_stride: int | None = None,
               windows: np.ndarray | None = None) -> "DeviceBatch":
        """A device-resident batch.  `mode`: the form its output is kept in, as for decode_frames (out_offset and
        out_elems count samples in every mode), or channels-first OUT_CHANNELS_I32 / _F32: a [channels,
        channel_stride] buffer in which out_offset is each frame's column (out_elems omitted, or their product).
        `windows` (channel modes; WINDOW_DTYPE, one per frame): frame i stores only samples [first, first + count)
        of each channel c, on row `row + c`, from column out_offset on (clx_batch_create_windows); `channels` is
        then the number of rows and has no cap of 8."""
        return DeviceBatch(self, data, descs, out_elems, mode=mode, channels=channels, channel_stride=channel_stride,
                           windows=windows)

    def adopt(self, device_ptr: int, nbytes: int, descs: np.ndarray, out_elems: int | None = None,
              mode: int = OUT_PLANAR_I32, channels: int | None = None, channel_stride: int | None = None,
              windows: np.ndarray | None = None) -> "DeviceBatch":
        """A batch whose frame bytes already sit in this GPU's memory at `device_ptr` (e.g. a torch tensor's
        data_ptr() after the NCCL scatter of claxon_b200.shard.scatter_batch): copied device to device."""
        return DeviceBatch(self, None, descs, out_elems, device_ptr=device_ptr, nbytes=nbytes, mode=mode,
                           channels=channels, channel_stride=channel_stride, windows=windows)


def _out_array(out_elems: int, mode: int) -> np.ndarray:
    """A host array for `out_elems` samples in output mode `mode`: int16, 3 bytes per sample as uint8, or int32."""
    n = max(1, out_elems)
    return (np.empty(n, dtype=np.int16) if mode == OUT_INTERLEAVED_I16 else
            np.empty(3 * n, dtype=np.uint8) if mode == OUT_INTERLEAVED_I24 else np.empty(n, dtype=np.int32))


_CHANNEL_MODES = (OUT_CHANNELS_I32, OUT_CHANNELS_F32)


class _Batch:
    """Owns a clx_batch: the one place that decodes, times and destroys one.  `keep`: what must outlive the batch (a
    crop batch's corpus).  The tensors that view the batch's buffers hold this handle, not the DeviceBatch or CropBatch
    around it, so the batch lives as long as the last of them."""

    def __init__(self, ctx: Context, h, keep=None):
        self.ctx, self.h, self.keep = ctx, h, keep

    def decode(self, stream: int):
        _check(self.ctx._L.clx_batch_decode(self.ctx._h, self.h, stream), self.ctx)

    def kernel_ms(self) -> float:
        ms = C.c_float(0)
        _check(self.ctx._L.clx_batch_last_kernel_ms(self.ctx._h, self.h, C.byref(ms)), self.ctx)
        return float(ms.value)

    def tensor(self, ptr: int, shape: tuple, typestr: str):
        """A zero-copy torch CUDA tensor over device memory of the batch; it keeps the batch alive."""
        import torch
        return torch.as_tensor(_DeviceView(self, ptr, shape, typestr), device="cuda")

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "_h", None):
            self.ctx._L.clx_batch_destroy(self.ctx._h, self.h)
        self.h = None
        if getattr(self.keep, "_close_pending", False):  # (see Corpus.__del__)
            try:
                self.keep.close()
            except Exception:  # another batch of it is still alive: the last one closes it
                pass

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _DeviceView:
    """__cuda_array_interface__ of device memory owned by `owner`, which it keeps alive while a tensor views it."""

    def __init__(self, owner, ptr: int, shape: tuple, typestr: str):
        self.owner = owner
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (int(ptr), False), "strides": None,
                                         "version": 2}


class DeviceBatch:
    """clx_batch: frames resident in HBM; decode() launches the kernels only."""

    def __init__(self, ctx: Context, data, descs: np.ndarray, out_elems: int | None, device_ptr: int | None = None,
                 nbytes: int = 0, mode: int = OUT_PLANAR_I32, channels: int | None = None,
                 channel_stride: int | None = None, windows: np.ndarray | None = None):
        self.ctx = ctx
        self.descs = np.ascontiguousarray(descs, dtype=DESC_DTYPE)
        self.mode = int(mode)
        self.channels = self.channel_stride = None
        self._stream = None  # internal stream of the last decode()
        # (a channel mode without its layout goes to clx_batch_create_to, which refuses it like any unknown mode)
        if channels is not None or channel_stride is not None:
            if self.mode not in _CHANNEL_MODES or channels is None or channel_stride is None:
                raise ValueError("channels= and channel_stride= go together, with a channel mode")
            self.channels, self.channel_stride = int(channels), int(channel_stride)
            if out_elems is not None and int(out_elems) != self.channels * self.channel_stride:
                raise ValueError("out_elems must equal channels * channel_stride")
            out_elems = self.channels * self.channel_stride
        if windows is not None:
            if self.channels is None:
                raise ValueError("windows= needs a channel mode with channels= and channel_stride=")
            windows = np.ascontiguousarray(windows, dtype=WINDOW_DTYPE)
            if windows.size != self.descs.size:
                raise ValueError("one window per frame")
        self.windows = windows
        if out_elems is None:
            raise ValueError("out_elems is required")
        self.out_elems = int(out_elems)
        on_device = device_ptr is not None
        if on_device:
            ptr, self.nbytes = device_ptr, int(nbytes)
        else:
            buf = _as_u8(data)
            ptr, self.nbytes = buf.ctypes.data, int(buf.size)
        flags = _lib.BATCH_BYTES_ON_DEVICE if on_device else 0
        h = C.c_void_p()
        if windows is not None:
            _check(ctx._L.clx_batch_create_windows(ctx._h, ptr, self.nbytes, self.descs.ctypes.data, windows.ctypes.data,
                                                   self.descs.size, self.channels, self.channel_stride, flags, self.mode,
                                                   C.byref(h)), ctx)
        elif self.channels is not None:
            _check(ctx._L.clx_batch_create_channels(ctx._h, ptr, self.nbytes, self.descs.ctypes.data, self.descs.size,
                                                    self.channels, self.channel_stride, flags, self.mode, C.byref(h)), ctx)
        else:
            _check(ctx._L.clx_batch_create_to(ctx._h, ptr, self.nbytes, self.descs.ctypes.data, self.descs.size,
                                              self.out_elems, flags, self.mode, C.byref(h)), ctx)
        self._batch = _Batch(ctx, h)

    @property
    def _h(self):
        return self._batch.h

    def decode(self, stream: int = 0):
        self._batch.decode(stream)
        self._stream = stream

    def sync(self):
        _check(self.ctx._L.clx_batch_sync(self.ctx._h, self._h), self.ctx)

    def kernel_ms(self) -> float:
        return self._batch.kernel_ms()

    def read(self):
        """Returns (out, results); `out` is in the batch's mode: int32, int16, or uint8 with 3 bytes per sample; in a
        channel mode an int32 / float32 array of shape (channels, channel_stride)."""
        if self.channels is not None:
            out = np.empty((self.channels, self.channel_stride),
                           dtype=np.float32 if self.mode == OUT_CHANNELS_F32 else np.int32)
        else:
            out = _out_array(self.out_elems, self.mode)
        results = np.zeros(self.descs.size, dtype=RESULT_DTYPE)
        _check(self.ctx._L.clx_batch_read_to(self.ctx._h, self._h, out.ctypes.data, max(1, self.out_elems),
                                             results.ctypes.data), self.ctx)
        return out, results

    def results(self):
        """The per-frame results of the last decode (waits for it), without copying the samples."""
        results = np.zeros(self.descs.size, dtype=RESULT_DTYPE)
        _check(self.ctx._L.clx_batch_read_to(self.ctx._h, self._h, None, 0, results.ctypes.data), self.ctx)
        return results

    def tensor(self):
        """A zero-copy torch CUDA tensor [channels, channel_stride] (float32 or int32) over the batch's output, for the
        channel modes.  It keeps the batch alive and shows whatever the batch's latest decode wrote; torch's current
        stream is made to wait for the last decode() first, so it may be read on that stream without a sync.
        (close() frees the memory under it.)"""
        import torch
        if self.channels is None:
            raise ValueError("tensor() needs a batch in a channel mode")
        if self._stream is not None:
            ptr = self.ctx._L.clx_ctx_stream(self.ctx._h, self._stream)
            torch.cuda.current_stream().wait_stream(torch.cuda.ExternalStream(ptr))
        return self._batch.tensor(self.device_out_ptr, (self.channels, self.channel_stride),
                                  "<f4" if self.mode == OUT_CHANNELS_F32 else "<i4")

    @property
    def device_out_ptr(self) -> int:
        return int(self.ctx._L.clx_batch_device_out(self._h) or 0)

    def close(self):
        self._batch.close()


_default_ctx: Context | None = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context()
    return _default_ctx


# ---------------------------------------------------------------------------
# claxon-shaped API
# ---------------------------------------------------------------------------

class Block:
    """claxon::frame::Block (src/frame.rs:402-529): planar samples, channel-major."""

    def __init__(self, time: int, block_size: int, buffer: np.ndarray):
        self._time = int(time)
        self._bs = int(block_size)
        self._buffer = buffer
        self._channels = (buffer.size // block_size) if block_size else 0  # src/frame.rs:418

    @staticmethod
    def empty() -> "Block":
        return Block(0, 0, np.zeros(0, dtype=np.int32))

    def time(self) -> int:
        return self._time

    def len(self) -> int:
        return self._bs * self._channels

    __len__ = len

    def duration(self) -> int:
        return self._bs

    def channels(self) -> int:
        return self._channels

    def channel(self, ch: int) -> np.ndarray:
        if not 0 <= ch < self._channels:
            raise IndexError("channel out of range")  # the reference panics
        return self._buffer[ch * self._bs:(ch + 1) * self._bs]

    def sample(self, ch: int, sample: int) -> int:
        return int(self._buffer[ch * self._bs + sample])

    def into_buffer(self) -> np.ndarray:
        return self._buffer

    def stereo_samples(self):
        if self._channels != 2:
            raise RuntimeError("stereo_samples() must only be called for blocks with two channels.")
        left, right = self.channel(0), self.channel(1)
        return ((int(l), int(r)) for l, r in zip(left, right))


def _ensure_buffer_len(buffer: np.ndarray | None, new_len: int) -> np.ndarray:
    """ensure_buffer_len (src/frame.rs:616-637): exact length, capacity reused when sufficient."""
    if buffer is None:
        return np.zeros(new_len, dtype=np.int32)
    base = buffer.base if isinstance(buffer.base, np.ndarray) and buffer.base.dtype == np.int32 else buffer
    if base.size >= new_len:
        return base[:new_len]
    return np.zeros(new_len, dtype=np.int32)


class FrameReader:
    """claxon::frame::FrameReader over an in-memory byte span positioned at a frame header."""

    def __init__(self, input, ctx: Context | None = None, _flac: bool = False):
        self._ctx = ctx or default_context()
        self._buf = _as_u8(input)
        L = self._ctx._L
        h = C.c_void_p()
        opener = L.clx_reader_open_flac if _flac else L.clx_reader_open_frames
        _check(opener(self._ctx._h, self._buf.ctypes.data, self._buf.size, C.byref(h)), self._ctx)
        self._h = h

    def read_next_or_eof(self, buffer: np.ndarray | None = None) -> Block | None:
        """Decodes the next frame; None at end of stream; raises Error on malformed input."""
        L = self._ctx._L
        st, d = parse_frame_header(self._buf, self.position(), 0 if self._ctx.verify_crc else OPT_NO_VERIFY_CRC)
        if st == EOF:
            return None
        _check(st)
        buffer = _ensure_buffer_len(buffer, d.n_channels * d.block_size)
        bs, ch, t = C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)
        st = L.clx_reader_next(self._h, buffer.ctypes.data, buffer.size, C.byref(bs), C.byref(ch), C.byref(t))
        if st == EOF:
            return None
        _check(st, self._ctx)
        return Block(t.value, bs.value, buffer)

    def read_batch(self, max_frames: int, buffer: np.ndarray | None = None) -> list[Block]:
        """Batched extension: demux + decode up to max_frames frames in one device pass."""
        L = self._ctx._L
        nf, need = C.c_size_t(0), C.c_uint64(0)
        st = L.clx_reader_plan_batch(self._h, max_frames, C.byref(nf), C.byref(need))  # demux ahead: exact buffer size
        if st == EOF:
            return []
        _check(st, self._ctx)
        descs = np.zeros(max_frames, dtype=DESC_DTYPE)
        cap = max(1, int(need.value))
        if buffer is None or buffer.size < cap:
            buffer = np.empty(cap, dtype=np.int32)
        n = C.c_size_t(0)
        st = L.clx_reader_next_batch(self._h, max_frames, buffer.ctypes.data, buffer.size, descs.ctypes.data,
                                     C.byref(n))
        if st == EOF:
            return []
        _check(st, self._ctx)
        blocks = []
        for i in range(n.value):
            d = descs[i]
            o, cnt = int(d["out_offset"]), int(d["n_channels"]) * int(d["block_size"])
            blocks.append(Block(int(d["number"]), int(d["block_size"]), buffer[o:o + cnt]))
        return blocks

    def position(self) -> int:
        return int(self._ctx._L.clx_reader_position(self._h))

    def into_inner(self):
        return self._buf

    def close(self):
        if getattr(self, "_h", None):
            self._ctx._L.clx_reader_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@dataclass
class FlacReaderOptions:
    """claxon::FlacReaderOptions (src/lib.rs:123-151)."""
    metadata_only: bool = False
    read_vorbis_comment: bool = True


def _parse_vorbis_comment(body: np.ndarray):
    """(vendor, [(comment, separator index)]) of a validated VORBIS_COMMENT body (src/metadata.rs:402-513)."""
    raw = body.tobytes()
    at = 4 + int.from_bytes(raw[0:4], "little")
    vendor = raw[4:at].decode("utf-8")
    count = int.from_bytes(raw[at:at + 4], "little")
    at += 4
    comments = []
    while len(raw) - at >= 4 and len(comments) < count:
        n = int.from_bytes(raw[at:at + 4], "little")
        at += 4
        if n == 0:  # zero-length comments occur in the wild and are skipped
            count -= 1
            continue
        c = raw[at:at + n]
        at += n
        comments.append((c.decode("utf-8"), c.index(b"=")))
    return vendor, comments


class FlacReader:
    """claxon::FlacReader (src/lib.rs:207-470) for in-memory streams / files."""

    def __init__(self, data, ctx: Context | None = None, options: FlacReaderOptions | None = None):
        self._options = options or FlacReaderOptions()
        buf = _as_u8(data)
        flags = ((OPEN_METADATA_ONLY if self._options.metadata_only else 0)
                 | (0 if self._options.read_vorbis_comment else OPEN_NO_VORBIS_COMMENT))
        si = _lib.StreamInfoC()
        first, vc_off, vc_len = C.c_uint64(0), C.c_uint64(0), C.c_uint32(0)
        _check(_lib.load().clx_open_stream_ex(buf.ctypes.data, buf.size, flags, C.byref(si), C.byref(first),
                                              C.byref(vc_off), C.byref(vc_len)))
        self._si = StreamInfo._from_c(si)
        self._vendor, self._comments = None, []
        if vc_len.value:
            self._vendor, self._comments = _parse_vorbis_comment(buf[vc_off.value:vc_off.value + vc_len.value])
        # FlacReaderState::Full / MetadataOnly (src/lib.rs:96-104)
        self._frames = None if self._options.metadata_only else FrameReader(buf, ctx, _flac=True)

    @classmethod
    def new(cls, data, ctx: Context | None = None) -> "FlacReader":
        return cls(data, ctx)

    @classmethod
    def new_ext(cls, data, options: FlacReaderOptions, ctx: Context | None = None) -> "FlacReader":
        return cls(data, ctx, options)

    @classmethod
    def open(cls, path, ctx: Context | None = None) -> "FlacReader":
        with open(path, "rb") as f:
            return cls(f.read(), ctx)

    @classmethod
    def open_ext(cls, path, options: FlacReaderOptions, ctx: Context | None = None) -> "FlacReader":
        with open(path, "rb") as f:
            return cls(f.read(), ctx, options)

    def streaminfo(self) -> StreamInfo:
        return self._si

    def vendor(self) -> str | None:
        """Vendor string of the Vorbis comment block, if present (src/lib.rs:318-325)."""
        return self._vendor

    def tags(self):
        """(name, value) pairs of the Vorbis comments, names as stored (src/lib.rs:327-345)."""
        return [(c[:i], c[i + 1:]) for c, i in self._comments]

    def get_tag(self, tag_name: str):
        """Values of every comment whose name equals tag_name ASCII-case-insensitively (src/lib.rs:347-360)."""
        def lower(t):
            return "".join(chr(ord(ch) + 32) if "A" <= ch <= "Z" else ch for ch in t)
        return [c[i + 1:] for c, i in self._comments if lower(c[:i]) == lower(tag_name)]

    def _full(self, what: str) -> FrameReader:
        if self._frames is None:  # the reference panics
            raise RuntimeError(f"FlacReaderOptions::metadata_only must be false to be able to use FlacReader::{what}()")
        return self._frames

    def blocks(self) -> FrameReader:
        return self._full("blocks")

    def samples(self, batch_frames: int = 256):
        """FlacSamples (src/lib.rs:473-519): interleaved samples, channel by channel for each inter-channel
        sample; an error surfaces once, where the bad frame starts, after every sample before it.  Frames are
        decoded `batch_frames` at a time on the device."""
        return self._iter_samples(self._full("samples"), batch_frames)

    def into_samples(self, batch_frames: int = 256):
        """FlacIntoSamples (src/lib.rs:412-435): as samples(), taking the reader with it."""
        frames, self._frames = self._full("into_samples"), None
        return self._iter_samples(frames, batch_frames)

    @staticmethod
    def _iter_samples(frames: FrameReader, batch_frames: int):
        while True:
            blocks = frames.read_batch(batch_frames)  # raises if the very next frame is bad
            if not blocks:
                return
            for block in blocks:
                ch, bs = block.channels(), block.duration()
                yield from block.into_buffer().reshape(ch, bs).T.reshape(-1).tolist()

    def into_inner(self):
        return self._frames.into_inner() if self._frames is not None else None


# ---------------------------------------------------------------------------
# FLAC files -> torch tensors
# ---------------------------------------------------------------------------

def frame_starts(descs: np.ndarray) -> np.ndarray:
    """Each frame's first sample (int64): the running sum of the block sizes before it, in stream order."""
    bs = descs["block_size"].astype(np.int64)
    return np.concatenate([[0], np.cumsum(bs)[:-1]]).astype(np.int64) if bs.size else bs


def plan_range(descs: np.ndarray, lo: int, hi: int, column: int = 0, row: int = 0, starts: np.ndarray | None = None):
    """The frames of one stream that overlap its samples [lo, hi), and where they go.  Returns (idx, windows, cols):
    the indices of those frames in `descs` (consecutive, in stream order), their windows (WINDOW_DTYPE: `row`, and
    the first sample and count of each frame inside the range) and each window's column, so that sample lo of the
    stream lands at column `column`.  `starts`: frame_starts(descs), if already known.  An empty range (or one past
    the end) has no frames."""
    if starts is None:
        starts = frame_starts(descs)
    bs = descs["block_size"].astype(np.int64)
    i0 = int(np.searchsorted(starts + bs, lo, side="right"))  # the first frame that ends after lo
    i1 = int(np.searchsorted(starts, hi, side="left")) if hi > lo else i0  # the frames that start before hi
    idx = np.arange(i0, max(i0, i1), dtype=np.int64)
    s0, b = starts[idx], bs[idx]
    first = np.maximum(lo - s0, 0)
    count = np.minimum(s0 + b, hi) - s0 - first
    windows = np.zeros(idx.size, dtype=WINDOW_DTYPE)
    windows["row"], windows["first"], windows["count"] = row, first, count
    cols = (column + s0 + first - lo).astype(np.uint64)
    return idx, windows, cols


def plan_columns(files_descs: list[np.ndarray]):
    """Column layout of several files' frames in one channels-first batch.  Returns (descs, starts, lengths, rows,
    stride): the files' descriptors concatenated with out_offset = each frame's column (its file's start plus the
    block sizes of the frames before it), each file's first column (a multiple of 4), each file's sample count per
    channel, the largest channel count, and the row length (the end of the last file rounded up to a multiple of 4)."""
    starts, lengths, parts = [], [], []
    at, rows = 0, 0
    for d in files_descs:
        d = np.array(d, dtype=DESC_DTYPE)
        n = int(d["block_size"].astype(np.int64).sum())
        idx, _, cols = plan_range(d, 0, n, column=at)  # the whole file: every frame, full windows
        d = d[idx]
        d["out_offset"] = cols
        starts.append(at)
        lengths.append(n)
        parts.append(d)
        rows = max(rows, int(d["n_channels"].max()) if d.size else 0)
        at = (at + n + 3) & ~3
    descs = np.concatenate(parts) if parts else np.zeros(0, dtype=DESC_DTYPE)
    return descs, starts, lengths, rows, at


@dataclass
class IndexedFile:
    """One stream of a FlacIndex: its bytes, STREAMINFO, frame descriptors (byte_offset into `data`), each frame's
    first sample, its length in samples per channel, and whether the end of its last frame was confirmed by the
    demuxer (False: the decode of that frame gives the verdict on what follows it, as in FlacReader)."""
    data: np.ndarray
    info: StreamInfo
    descs: np.ndarray
    starts: np.ndarray
    length: int
    end_confirmed: bool


class FlacIndex:
    """Frame indexes of FLAC streams, demuxed once: what load_crops() plans excerpts from."""

    def __init__(self, files: list[IndexedFile]):
        self.files = files

    def __len__(self) -> int:
        return len(self.files)

    def __getitem__(self, i: int) -> IndexedFile:
        return self.files[i]


def _read_source(src) -> np.ndarray:
    if isinstance(src, (bytes, bytearray, memoryview, np.ndarray)):
        return _as_u8(src)
    with open(src, "rb") as f:
        return np.frombuffer(f.read(), dtype=np.uint8)


def _map_source(src) -> np.ndarray:
    """A path as a read-only np.memmap (an empty file as an empty array); bytes as they are."""
    if isinstance(src, (bytes, bytearray, memoryview, np.ndarray)):
        return _as_u8(src)
    import os
    if os.path.getsize(src) == 0:
        return np.zeros(0, dtype=np.uint8)
    return np.memmap(src, dtype=np.uint8, mode="r")


def _index_one(buf: np.ndarray, i: int, threads: int) -> IndexedFile:
    si, first = open_stream(buf)
    descs, _, _, stop = demux_frames(buf, first, threads=threads)
    # OK: the last frame's end could not be confirmed (damage, or bytes after it); its decode gives the verdict
    if stop not in (OK, EOF):
        raise Error(stop, f"file {i}")
    if descs.size and (descs["n_channels"] != si.channels).any():
        raise ValueError(f"file {i}: a frame's channel count differs from STREAMINFO's ({si.channels})")
    starts = frame_starts(descs)
    n = int(starts[-1]) + int(descs["block_size"][-1]) if descs.size else 0
    return IndexedFile(buf, si, descs, starts, n, not (stop == OK and descs.size > 0))


def index(src, threads: int = 0) -> FlacIndex:
    """Opens and demuxes FLAC stream(s) once: `src` is a path or the file's bytes, or a list of them (paths are
    memory-mapped).  Raises what load() raises at demux time: the metadata error, a frame-header error where
    demuxing stopped, or ValueError for a frame whose channel count differs from STREAMINFO's."""
    many = isinstance(src, (list, tuple))
    return FlacIndex([_index_one(_map_source(s), i, threads) for i, s in enumerate(src if many else [src])])


def _torch_dtype(dtype):
    import torch
    dtype = torch.float32 if dtype is None else dtype
    if dtype not in (torch.float32, torch.int32):
        raise ValueError("dtype must be torch.float32 or torch.int32")
    return dtype


def _channels_mode(dtype) -> int:  # of a dtype _torch_dtype() accepted
    import torch
    return OUT_CHANNELS_F32 if dtype == torch.float32 else OUT_CHANNELS_I32


def _decode_excerpts(idx: FlacIndex, excerpts, rows: int, stride: int, out, ctx: Context | None, where):
    """Decodes excerpts of indexed files in one windowed batch into `out`, a torch tensor viewing [rows, stride].
    `excerpts`: (file, lo, hi, column, row) per excerpt: samples [lo, hi) of the file go to row `row` + c from
    column `column` on.  Only the frames overlapping an excerpt are gathered, uploaded and decoded.  where(k) names
    excerpt k in errors."""
    import torch
    chunks, parts, wins, owner, at = [], [], [], [], 0
    for k, (fi, lo, hi, column, row) in enumerate(excerpts):
        f = idx.files[fi]
        sel, w, cols = plan_range(f.descs, lo, hi, column=column, row=row, starts=f.starts)
        if not sel.size:
            continue
        d = f.descs[sel]
        b0 = int(d["byte_offset"][0])
        b1 = int(d["byte_offset"][-1]) + int(d["byte_len"][-1])
        chunks.append(f.data[b0:b1])
        d["byte_offset"] = d["byte_offset"] - np.uint64(b0) + np.uint64(at)
        d["out_offset"] = cols
        parts.append(d)
        wins.append(w)
        owner.append(np.full(sel.size, k, np.int64))
        at += b1 - b0
    if not parts:
        out.zero_()
        return
    descs, windows, owner = np.concatenate(parts), np.concatenate(wins), np.concatenate(owner)
    ctx = ctx or default_context()
    dev = ctx.upload(np.concatenate(chunks), descs, mode=_channels_mode(out.dtype), channels=rows, channel_stride=stride,
                     windows=windows)
    try:
        dev.decode(0)
        res = dev.results()
        bad = np.nonzero(res["status"] != OK)[0]
        if bad.size:
            raise Error(int(res["status"][bad[0]]), where(int(owner[bad[0]])))
        # an excerpt that contains a file's unconfirmed last frame: what follows that frame
        for j in np.nonzero(np.r_[owner[1:] != owner[:-1], True])[0]:
            k = int(owner[j])
            f = idx.files[excerpts[k][0]]
            last = f.descs[-1]
            if f.end_confirmed or excerpts[k][2] <= int(f.starts[-1]):
                continue
            if res["consumed"][j] < last["byte_len"]:
                st, _ = parse_frame_header(f.data, int(last["byte_offset"]) + int(res["consumed"][j]))
                if st != EOF:
                    raise Error(st, where(k))
        out.copy_(dev.tensor())
        torch.cuda.current_stream().synchronize()  # the copy has completed: nothing of the batch is needed
    finally:
        dev.close()


def load(src, dtype=None, ctx: Context | None = None, threads: int = 0, frame_offset: int = 0, num_frames: int = -1):
    """FLAC file(s) -> (tensor [channels, samples], sample_rate) on the GPU, channels first like torchaudio.load.

    `src`: a path or the file's bytes, or a list of them (then a list of results).  `dtype`: torch.float32 (the
    default: samples * 2^-(bits_per_sample - 1), in [-1, 1)) or torch.int32.  `frame_offset` / `num_frames` as in
    torchaudio: each file gives its samples [frame_offset, frame_offset + num_frames), cut at its end (num_frames -1:
    to the end), so [C_i, min(num_frames, N_i - frame_offset)]; only the frames that overlap that range are decoded.
    Every file is demuxed on `threads` host threads (0 = all) and all of them are decoded in one device-resident
    batch; each result is a view of one tensor.  Raises what FlacReader would: the metadata error, a frame-header error
    where demuxing stopped, or the first decoded frame that failed (naming the file); ValueError for a frame whose
    channel count differs from STREAMINFO's, and for frame_offset < 0 or past a file's end or num_frames < -1."""
    import torch
    dtype = _torch_dtype(dtype)
    if frame_offset < 0 or num_frames < -1:
        raise ValueError("frame_offset must be >= 0 and num_frames >= -1")
    many = isinstance(src, (list, tuple))
    idx = FlacIndex([_index_one(_read_source(s), i, threads) for i, s in enumerate(src if many else [src])])
    excerpts, spans, at, rows = [], [], 0, 0
    for i, f in enumerate(idx.files):
        if frame_offset > f.length:
            raise ValueError(f"file {i}: frame_offset {frame_offset} is past its end ({f.length} samples)")
        hi = f.length if num_frames < 0 else min(f.length, frame_offset + num_frames)
        excerpts.append((i, frame_offset, hi, at, 0))
        spans.append((at, hi - frame_offset))
        rows = max(rows, f.info.channels if f.descs.size else 0)
        at = (at + hi - frame_offset + 3) & ~3
    # (the batch's buffer reads 0 wherever no frame wrote, so one copy of it fills every element)
    out = torch.empty((max(rows, 1), at), dtype=dtype, device="cuda")
    _decode_excerpts(idx, excerpts, max(rows, 1), at, out, ctx, lambda k: f"file {k}")
    views = [(out[:f.info.channels, s:s + n], f.info.sample_rate) for f, (s, n) in zip(idx.files, spans)]
    return views if many else views[0]


def load_crops(index: FlacIndex, files, offsets, num_frames: int, dtype=None, ctx: Context | None = None):
    """Excerpts of indexed FLAC files as one [B, C, num_frames] CUDA tensor, the batch a training loader wants.

    Excerpt b is samples [offsets[b], offsets[b] + num_frames) of file files[b]; C is the largest channel count among
    the chosen files.  Columns past a file's end, and rows a file does not have, read 0.  Returns (tensor, lengths):
    lengths[b] = min(num_frames, N - offsets[b]) (a torch.int64 CPU tensor).  `dtype`: torch.float32 (the default, the
    rule of load()) or torch.int32.  Only the frames that overlap an excerpt are gathered into one host buffer,
    uploaded and decoded, in one batch whose rows are copied into the tensor once.  So errors of frames outside every
    excerpt are not reported: raises Error(status, "file i, crop b") for the first failed frame inside an excerpt, or
    for what follows a file's last frame (load()'s trailing-bytes check) when an excerpt contains that frame; ValueError
    for an offset < 0 or past the file's end, num_frames < 1, a file index out of range, or another dtype."""
    import torch
    dtype = _torch_dtype(dtype)
    files = [int(f) for f in np.asarray(files).reshape(-1)]
    offsets = [int(o) for o in np.asarray(offsets).reshape(-1)]
    num_frames = int(num_frames)
    if len(files) != len(offsets):
        raise ValueError("files and offsets must have the same length")
    if num_frames < 1:
        raise ValueError("num_frames must be >= 1")
    for b, (fi, o) in enumerate(zip(files, offsets)):
        if not 0 <= fi < len(index):
            raise ValueError(f"crop {b}: file index {fi} out of range")
        if not 0 <= o <= index[fi].length:
            raise ValueError(f"crop {b}: offset {o} outside file {fi} ({index[fi].length} samples)")
    B = len(files)
    C_ = max([index[fi].info.channels for fi in files], default=1)
    out = torch.empty((B, C_, num_frames), dtype=dtype, device="cuda")
    excerpts = [(fi, o, min(o + num_frames, index[fi].length), 0, b * C_) for b, (fi, o) in enumerate(zip(files, offsets))]
    lengths = torch.tensor([hi - lo for _, lo, hi, _, _ in excerpts], dtype=torch.int64)
    if B:
        _decode_excerpts(index, excerpts, B * C_, num_frames, out.view(B * C_, num_frames), ctx,
                         lambda k: f"file {files[k]}, crop {k}")
    return out, lengths


# ---------------------------------------------------------------------------
# device-resident corpora: crops planned on the device
# ---------------------------------------------------------------------------

class Corpus:
    """The compressed frames of a FlacIndex's files, copied once with their frame index (clx_corpus_create_ex), for
    CropBatch: crops whose frames, windows and columns are planned on the device.  Each file's bytes from its first
    frame to its end are copied; the trailing-bytes verdict of a file whose last frame's end is unconfirmed is taken
    once here.  `index` is kept for error messages.

    `memory`: where the bytes live.  "device" (the default) uploads them to the GPU.  "host" keeps them in pinned host
    memory the GPU reads directly, and only the frame index (about 48 bytes per frame) on the GPU: for corpora that
    should not take GPU memory from the model.  Every call of a crop batch of a host corpus then copies the frames its
    crops selected over PCIe first (about the crops' span bytes x B per call), so it is slower than over a device
    corpus; the results are the same.  `device_bytes` is the GPU memory the corpus holds.  For data-parallel jobs,
    Corpus.share() and Corpus.attach() give a host corpus whose pinned bytes exist once per machine (memory "shared")."""

    def __init__(self, index: FlacIndex, ctx: Context | None = None, memory: str = "device"):
        if memory not in ("device", "host"):
            raise ValueError('memory must be "device" or "host"')
        self.index = index
        self.memory = memory
        self.ctx = ctx or default_context()
        chunks, parts, file_frames, at = [], [], [0], 0
        for f in index.files:
            if f.descs.size:
                b0 = int(f.descs["byte_offset"][0])
                chunks.append(np.asarray(f.data[b0:]))
                d = f.descs.copy()
                d["byte_offset"] = d["byte_offset"] - np.uint64(b0) + np.uint64(at)
                d["out_offset"] = 0
                parts.append(d)
                at += f.data.size - b0
            file_frames.append(file_frames[-1] + f.descs.size)
        data = np.concatenate(chunks) if chunks else np.zeros(0, np.uint8)
        self.descs = np.concatenate(parts) if parts else np.zeros(0, dtype=DESC_DTYPE)
        self.file_frames = np.array(file_frames, dtype=np.uint32)
        self.nbytes = int(data.size)
        self.channels = max([int(self.descs["n_channels"].max())] if self.descs.size else [1])
        h = C.c_void_p()
        flags = _lib.CORPUS_HOST if memory == "host" else 0
        _check(self.ctx._L.clx_corpus_create_ex(self.ctx._h, data.ctypes.data, data.size, self.descs.ctypes.data,
                                                self.descs.size, self.file_frames.ctypes.data, len(index), flags,
                                                C.byref(h)), self.ctx)
        self._h = h

    @property
    def device_bytes(self) -> int:
        """clx_corpus_device_bytes: the GPU memory the corpus holds (its bytes too for a device corpus)."""
        return int(self.ctx._L.clx_corpus_device_bytes(self._h))

    def frames_bound(self, num_frames: int) -> int:
        """clx_crop_frames_bound: the most frames num_frames consecutive samples of one file can overlap."""
        return int(self.ctx._L.clx_crop_frames_bound(self.descs.ctypes.data, self.descs.size, self.file_frames.ctypes.data,
                                                     len(self.index), int(num_frames)))

    def bytes_bound(self, num_frames: int) -> int:
        """clx_crop_bytes_bound: the most compressed bytes a crop of num_frames samples can span."""
        return int(self.ctx._L.clx_crop_bytes_bound(self.descs.ctypes.data, self.descs.size, self.file_frames.ctypes.data,
                                                    len(self.index), int(num_frames)))

    def crops(self, batch: int, num_frames: int, dtype=None, sample_rate: int | None = None) -> "CropBatch":
        """A CropBatch of `batch` crops of `num_frames` samples; its CUDA graph is instantiated here.  Over a host
        corpus, the batch also holds a GPU staging buffer of about batch x bytes_bound(num_frames) bytes, and each call
        reads the selected crops' span bytes (about span bytes x batch) from host memory over PCIe.  With `sample_rate`
        R, every crop is at rate R whatever its file's rate: offsets and num_frames count samples at R (see CropBatch)."""
        return CropBatch(self, batch, num_frames, dtype, sample_rate)

    def mel_crops(self, batch: int, num_frames: int, sample_rate: int | None = None, *, n_fft: int = 400,
                  win_length: int | None = None, hop_length: int | None = None, f_min: float = 0.0,
                  f_max: float | None = None, n_mels: int = 128, window_fn=None, wkwargs: dict | None = None,
                  center: bool = True, norm: str | None = None, mel_scale: str = "htk",
                  log_floor: float | None = None, normalize: str | None = None) -> "MelCropBatch":
        """A MelCropBatch: the mel spectrogram of each crop of a crop batch of `batch` crops of `num_frames` samples
        (resampled to `sample_rate` when given), computed on the device.  The keywords are those of
        torchaudio.transforms.MelSpectrogram (window_fn None is torch.hann_window); log_floor None gives the power,
        a float ln(max(mel, log_floor)); normalize None, "per_feature" or "whisper" (see MelCropBatch)."""
        return MelCropBatch(self, batch, num_frames, sample_rate, n_fft=n_fft, win_length=win_length,
                            hop_length=hop_length, f_min=f_min, f_max=f_max, n_mels=n_mels, window_fn=window_fn,
                            wkwargs=wkwargs, center=center, norm=norm, mel_scale=mel_scale, log_floor=log_floor,
                            normalize=normalize)

    def resample_source_bound(self, num_frames: int, sample_rate: int) -> int:
        """The most source samples a crop of num_frames samples at `sample_rate` reads from one file of the corpus
        (clx_resample_source_bound, the largest over the files' rates)."""
        L = self.ctx._L
        return max([int(L.clx_resample_source_bound(f.info.sample_rate, int(sample_rate), int(num_frames)))
                    for f in self.index.files] or [0])

    def packed_frames_bound(self, max_excerpts: int, max_samples: int) -> int:
        """clx_packed_frames_bound: the most frames the excerpts of one packed call can overlap together."""
        return int(self.ctx._L.clx_packed_frames_bound(self.descs.ctypes.data, self.descs.size, self.file_frames.ctypes.data,
                                                       len(self.index), int(max_excerpts), int(max_samples)))

    def packed_bytes_bound(self, max_excerpts: int, max_samples: int) -> int:
        """clx_packed_bytes_bound: the staging bytes of a packed batch over a host corpus."""
        return int(self.ctx._L.clx_packed_bytes_bound(self.descs.ctypes.data, self.descs.size, self.file_frames.ctypes.data,
                                                      len(self.index), int(max_excerpts), int(max_samples)))

    def packed(self, max_excerpts: int, max_samples: int, dtype=None, sample_rate: int | None = None) -> "PackedBatch":
        """A PackedBatch of up to `max_excerpts` excerpts laid out along `max_samples` columns; its CUDA graph is
        instantiated here.  With `sample_rate` R, every excerpt is at rate R whatever its file's rate: offsets, lengths,
        max_samples and the starts count samples at R (see PackedBatch)."""
        return PackedBatch(self, max_excerpts, max_samples, dtype, sample_rate)

    def mel_packed(self, max_excerpts: int, max_samples: int, sample_rate: int | None = None, *, n_fft: int = 400,
                   win_length: int | None = None, hop_length: int | None = None, f_min: float = 0.0,
                   f_max: float | None = None, n_mels: int = 128, window_fn=None, wkwargs: dict | None = None,
                   center: bool = True, norm: str | None = None, mel_scale: str = "htk",
                   log_floor: float | None = None, normalize: str | None = None) -> "MelPackedBatch":
        """A MelPackedBatch: the mel spectrogram of each excerpt of a packed batch of up to `max_excerpts` excerpts
        along `max_samples` columns (resampled to `sample_rate` when given), packed along frames, computed on the
        device.  The keywords are mel_crops()'s, but normalize is None or "per_feature"."""
        return MelPackedBatch(self, max_excerpts, max_samples, sample_rate, n_fft=n_fft, win_length=win_length,
                              hop_length=hop_length, f_min=f_min, f_max=f_max, n_mels=n_mels, window_fn=window_fn,
                              wkwargs=wkwargs, center=center, norm=norm, mel_scale=mel_scale, log_floor=log_floor,
                              normalize=normalize)

    def mel_packed_frames_bound(self, max_excerpts: int, max_samples: int, *, n_fft: int = 400,
                                win_length: int | None = None, hop_length: int | None = None,
                                center: bool = True) -> int:
        """clx_mel_packed_frames_bound: the frame columns T_f of a MelPackedBatch with these parameters, which hold
        the frames of any excerpts that fit in max_samples columns (about max_samples / hop_length + 4 per excerpt)."""
        win_length = int(n_fft) if win_length is None else int(win_length)
        hop_length = win_length // 2 if hop_length is None else int(hop_length)
        params = _lib.MelParams(int(n_fft), win_length, hop_length, 1, MEL_CENTER if center else 0, 0.0)
        return int(self.ctx._L.clx_mel_packed_frames_bound(C.byref(params), int(max_excerpts), int(max_samples)))

    def resample_packed_source_bound(self, max_excerpts: int, max_samples: int, sample_rate: int) -> int:
        """clx_resample_packed_source_bound: the columns of the packed batch that decodes the source spans of a
        resampled PackedBatch (about max_samples x r / R for the corpus's highest rate r)."""
        return int(self.ctx._L.clx_resample_packed_source_bound(self._file_rates().ctypes.data, len(self.index),
                                                                int(sample_rate), int(max_excerpts), int(max_samples)))

    def _file_rates(self) -> np.ndarray:
        """Each file's STREAMINFO sample rate, uint32 (one 0 for a corpus without files, so that it has an address)."""
        return np.array([f.info.sample_rate for f in self.index.files] or [0], dtype=np.uint32)

    @classmethod
    def share(cls, index: FlacIndex, path, ctx: Context | None = None) -> "Corpus":
        """Writes `index` as a corpus image at `path` (clx_corpus_image_write) and attaches it (Corpus.attach).

        An image holds the frame index and the compressed bytes of a host corpus in one file that every process and
        GPU of a machine can attach, so a data-parallel job pins the bytes once per machine instead of once per rank.
        Put it on a tmpfs such as /dev/shm: its pages are the pinned memory.  Each file's bytes are copied straight
        from its own buffer (the index's memory map), with no concatenated copy; the trailing-bytes verdicts are taken
        once here.  The image is written under a temporary name in the same directory and linked to `path` when
        complete, so attachers see all of it or nothing; its size is reserved first (posix_fallocate), so a tmpfs that
        is too small raises OSError before anything is copied.  A `path` that exists is refused (FileExistsError).

        The usual pattern, one process per GPU::

            if rank == 0:
                corpus = Corpus.share(index, "/dev/shm/train.clxc")
            barrier()
            if rank != 0:
                corpus = Corpus.attach("/dev/shm/train.clxc")
            barrier()
            if rank == 0:
                os.unlink("/dev/shm/train.clxc")  # optional: the pages live until the last mapping goes

        Removing the file is the caller's job; the memory is freed when it is unlinked and the last process has
        closed its corpus (or exited)."""
        import mmap
        import os
        import secrets
        ctx = ctx or default_context()
        path = os.fspath(path)
        if os.path.lexists(path):
            raise FileExistsError(17, "corpus image exists", path)
        L, n = ctx._L, len(index)
        datas = [_as_u8(f.data) for f in index.files]
        descs = (np.ascontiguousarray(np.concatenate([f.descs for f in index.files]), dtype=DESC_DTYPE) if n else
                 np.zeros(0, dtype=DESC_DTYPE))
        file_frames = np.concatenate([[0], np.cumsum([f.descs.size for f in index.files])]).astype(np.uint32)
        ptrs = (C.c_void_p * max(n, 1))(*[d.ctypes.data for d in datas])
        sizes = np.array([d.size for d in datas] or [0], dtype=np.uintp)
        infos = (_lib.StreamInfoC * max(n, 1))()
        for i, f in enumerate(index.files):
            s = f.info
            infos[i] = _lib.StreamInfoC(s.min_block_size, s.max_block_size, s.min_frame_size or 0, s.max_frame_size or 0,
                                        s.sample_rate, s.channels, s.bits_per_sample, s.samples or 0,
                                        (C.c_uint8 * 16)(*s.md5sum))
        size = int(L.clx_corpus_image_bytes(sizes.ctypes.data, descs.ctypes.data, descs.size, file_frames.ctypes.data, n))
        if size == 0:
            raise Error(90, "the index cannot be written as a corpus image")
        folder, name = os.path.split(os.path.abspath(path))
        tmp = os.path.join(folder, f".{name}.{os.getpid()}.{secrets.token_hex(4)}.tmp")
        fd = os.open(tmp, os.O_RDWR | os.O_CREAT | os.O_EXCL, 0o666)
        mm = None
        try:
            os.posix_fallocate(fd, 0, size)
            mm = mmap.mmap(fd, size, mmap.MAP_SHARED, mmap.PROT_READ | mmap.PROT_WRITE)
            img = np.frombuffer(mm, dtype=np.uint8)
            st = L.clx_corpus_image_write(ctx._h, ptrs, sizes.ctypes.data, descs.ctypes.data, descs.size,
                                          file_frames.ctypes.data, n, infos, img.ctypes.data, size)
            del img
            _check(st, ctx)
            os.link(tmp, path)  # (not rename: a path created meanwhile is refused, never replaced)
        except BaseException:
            if mm is not None:
                mm.close()
            os.unlink(tmp)
            raise
        finally:
            os.close(fd)
        os.unlink(tmp)
        return cls._attach_map(mm, path, ctx)

    @classmethod
    def attach(cls, source, ctx: Context | None = None) -> "Corpus":
        """A host corpus over a corpus image (clx_corpus_attach): `source` is the image's path, which is mapped shared
        and read-write (the driver pins pages writable; the library never writes to them), or an mmap.mmap of one that
        the caller keeps open for as long as the corpus lives (then several attaches share that one mapping).

        The image is checked in full, its bytes region is registered as pinned memory with cudaHostRegister and only its
        frame index is copied to the GPU: `device_bytes` is the index alone, and every process and GPU that attaches the
        image shares the same physical pages.  Crops, packed batches and the bounds work as for Corpus(memory="host"),
        with the same results.  `memory` is "shared" and `path` the image's path (None for a mapping).  `descs`,
        `file_frames` and `channels` come from the image, and `index` is a FlacIndex rebuilt from it: each file's
        StreamInfo, length, frame starts and end_confirmed as written, its `data` a read-only zero-copy view of its
        bytes in the image (from its first frame to its end), so its descriptors' byte_offset count from there (and
        out_offset is 0).  close() detaches; the mapping is closed once nothing views it.  The file may be unlinked
        while attached.  Raises Error(90) for a file that is not a well-formed image."""
        import mmap
        import os
        ctx = ctx or default_context()
        if isinstance(source, mmap.mmap):
            return cls._attach_map(source, None, ctx, own=False)
        path = os.fspath(source)
        fd = os.open(path, os.O_RDWR)
        try:
            size = os.fstat(fd).st_size
            if size == 0:
                raise Error(90, f"{path} is empty, not a corpus image")
            mm = mmap.mmap(fd, size, mmap.MAP_SHARED, mmap.PROT_READ | mmap.PROT_WRITE)
        finally:
            os.close(fd)
        return cls._attach_map(mm, path, ctx)

    @classmethod
    def _attach_map(cls, mm, path, ctx: Context, own: bool = True) -> "Corpus":
        self = cls.__new__(cls)
        self.ctx, self.memory, self.path = ctx, "shared", path
        img = np.frombuffer(mm, dtype=np.uint8)
        h = C.c_void_p()
        st = ctx._L.clx_corpus_attach(ctx._h, img.ctypes.data, img.size, C.byref(h))
        if st != OK:
            del img
            if own:
                mm.close()
            _check(st, ctx)
        self._h, self._map, self._own_map = h, mm, own
        img.flags.writeable = False
        hd = _lib.ImageHeader.from_buffer_copy(img[:C.sizeof(_lib.ImageHeader)])
        recs = (_lib.ImageFile * hd.n_files).from_buffer_copy(img, hd.files_offset)
        self.descs = np.frombuffer(img, dtype=DESC_DTYPE, count=hd.n_frames, offset=hd.descs_offset).copy()
        self.file_frames = np.array([r.first_frame for r in recs] + [hd.n_frames], dtype=np.uint32)
        self.nbytes = int(hd.nbytes)
        self.channels = max([int(self.descs["n_channels"].max())] if self.descs.size else [1])
        region = img[hd.bytes_offset:hd.bytes_offset + hd.bytes_size]
        files = []
        for i, r in enumerate(recs):
            d = self.descs[self.file_frames[i]:self.file_frames[i + 1]].copy()
            d["byte_offset"] -= np.uint64(r.byte_base)
            files.append(IndexedFile(region[r.byte_base:r.byte_base + r.byte_count], StreamInfo._from_c(r.info), d,
                                     frame_starts(d), int(d["block_size"].astype(np.int64).sum()),
                                     bool(r.flags & _lib.IMAGE_END_CONFIRMED)))
        self.index = FlacIndex(files)
        return self

    def close(self):
        """Frees the corpus's copy of the bytes and its index; raises Error while a CropBatch of the corpus is alive.
        An attached corpus drops its registration of the image instead, then closes the mapping it opened (at once, or
        when the last view of it, such as index[i].data, is gone); the image file itself is left as it is."""
        if getattr(self, "_h", None) and getattr(self.ctx, "_h", None):
            _check(self.ctx._L.clx_corpus_destroy(self.ctx._h, self._h), self.ctx)
            self._h = None
        if getattr(self, "_h", None) and getattr(self, "_map", None) is not None:
            _still_registered.append(self._map)  # its context is gone: the pages stay registered, so stay mapped
            self._own_map = False
        self._h = None
        if getattr(self, "_own_map", False):
            self._own_map = False
            try:
                self._map.close()
            except BufferError:  # views of the image are alive: the mapping goes with the last of them
                pass

    def __del__(self):
        try:
            self.close()
        except Exception:
            # Finalized in one garbage cycle with batches of it that are not yet destroyed: the last of them detaches
            # it (_Batch.close), before the cycle's mapping of the image can be unmapped.
            self._close_pending = getattr(self, "memory", None) == "shared"


# Mappings of images whose corpus could not be detached (its context was closed first): kept mapped for the life of the
# process, so that no new mapping takes the address range the driver still has registered.
_still_registered = []


def _first_failure(error) -> tuple[int, int, int] | None:
    """The error word of a crop or packed batch, read with the call's one sync: None, or the first failed excerpt's
    (kind, index, status), kind 0 being an invalid or non-fitting request."""
    err = int(error.item()) & ((1 << 64) - 1)
    if err == (1 << 64) - 1:
        return None
    st = err & 0xffffffff
    return err >> 62, (err >> 32) & ((1 << 30) - 1), st - (1 << 32) if st >= 1 << 31 else st


def _length_at(f: IndexedFile, rate: int | None) -> tuple[int, str]:
    """File f's length in samples at `rate`, ceil(N * R / r), and " at R Hz"; N and "" at its own rate or None."""
    if rate is None or f.info.sample_rate == rate:
        return f.length, ""
    g = math.gcd(f.info.sample_rate, rate)
    return -(-f.length * (rate // g) // (f.info.sample_rate // g)), f" at {rate} Hz"


class CropBatch:
    """`batch` excerpts of `num_frames` samples of a Corpus's files per call, as one [B, C, L] CUDA tensor
    (clx_batch_create_crops): the crops' frames, windows and columns are planned on the device inside the batch's CUDA
    graph, so a call is two small device-to-device copies and one graph launch, and the offsets may be CUDA tensors
    (drawn with torch.randint on the device, no sync).  C is the corpus's largest channel count.

    Crop b is samples [offsets[b], offsets[b] + L) of file files[b], cut at the file's end: columns past it and rows the
    file does not have read 0, as in load_crops(), whose results a call reproduces bit for bit.  `out` and `lengths`
    (and `status`, an int32 CUDA tensor of per-crop statuses) are views of the batch's own buffers, overwritten by the
    next call; the next call waits for what torch's current stream has enqueued before it, so reading them on that stream
    is safe, clone() them to keep them.  Unlike load_crops(), a float32 batch is refused when any frame of the corpus
    has more than 24 bits (load_crops() refuses only the frames a call selects).

    Over a host corpus (Corpus(memory="host")), each call first copies every crop's span of frames from pinned host
    memory into a GPU staging buffer, one more kernel in the graph: about span bytes x B cross PCIe per call.  Results
    are the same as over a device corpus.

    With `sample_rate` R (clx_batch_create_resampled_crops; float32 only), files of any rate give crops at rate R:
    offsets and L count samples at R, and crop b is resample(x, r, R)[:, offsets[b] : offsets[b] + L], x the whole file
    as load() gives it and r its STREAMINFO rate, resample being torchaudio.functional.resample with its defaults (so
    the samples near a crop's edges are those of the resampled file, not of a resampled excerpt).  lengths[b] =
    min(L, N_t - offsets[b]) with N_t = ceil(N * R / r) the file's length at R; an offset past N_t is invalid.  Files
    already at R are copied, bit for bit what a batch without sample_rate gives.  A crop's status is that of its source
    span, the samples its outputs read.  Each call decodes every crop's source span with a packed batch of
    B x round_up_4(resample_source_bound(L, R)) columns (about L x r / R samples per crop and row) and filters them on
    the device."""

    def __init__(self, corpus: Corpus, batch: int, num_frames: int, dtype=None, sample_rate: int | None = None):
        mode = self._args(corpus, batch, num_frames, dtype, sample_rate)
        L = self.ctx._L
        h = C.c_void_p()
        if self.sample_rate is None:
            _check(L.clx_batch_create_crops(self.ctx._h, corpus._h, self.batch, self.num_frames, mode, C.byref(h)),
                   self.ctx)
        else:
            _check(L.clx_batch_create_resampled_crops(self.ctx._h, corpus._h, corpus._file_rates().ctypes.data,
                                                      len(corpus.index), self.batch, self.num_frames, self.sample_rate,
                                                      C.byref(h)), self.ctx)
        self.channels = corpus.channels
        self._attach(h, (self.batch, self.channels, self.num_frames), "<f4" if mode == OUT_CHANNELS_F32 else "<i4")

    def _args(self, corpus: Corpus, batch: int, num_frames: int, dtype, sample_rate: int | None) -> int:
        """Checks and keeps the arguments of every crop batch; returns the output mode."""
        import torch
        self.corpus, self.ctx = corpus, corpus.ctx
        self.batch, self.num_frames, self.dtype = int(batch), int(num_frames), _torch_dtype(dtype)
        self.sample_rate = None if sample_rate is None else int(sample_rate)
        if self.batch < 1 or self.num_frames < 1:
            raise ValueError("batch and num_frames must be >= 1")
        if self.sample_rate is not None and self.dtype != torch.float32:
            raise ValueError("a resampled crop batch is float32 only")
        return _channels_mode(self.dtype)

    def _attach(self, h, out_shape: tuple, typestr: str):
        """Takes ownership of the created batch `h` and views its buffers: out, lengths, status, requests, error."""
        import torch
        L = self.ctx._L
        self._batch = _Batch(self.ctx, h, keep=self.corpus)
        B, view = self.batch, self._batch.tensor
        self.out = view(L.clx_batch_device_out(h), out_shape, typestr)
        self.lengths = view(L.clx_batch_crop_lengths(h), (B,), "<i8")
        self.status = view(L.clx_batch_crop_status(h), (B,), "<i4")
        self._requests = view(L.clx_batch_crop_requests(h), (B, 2), "<i8")  # {u32 file, u32 reserved} as one i64, offset
        self._error = view(L.clx_batch_crop_error(h), (1,), "<i8")
        self._stream = torch.cuda.ExternalStream(L.clx_ctx_stream(self.ctx._h, 0))

    def __call__(self, files, offsets, check: bool = True):
        """Decodes crop b = samples [offsets[b], offsets[b] + L) of file files[b] for every b.  Returns (out [B, C, L],
        lengths [B] int64), both on the GPU.  The requests are copied on torch's current stream, the batch's stream
        waits for it, and torch's stream waits for the decode: nothing syncs with the host unless `check`.  check=True
        syncs once and raises what load_crops() would: ValueError for the first crop whose file index or offset is out
        of range, else Error(status, "file i, crop b") for the first crop with a failed frame, else for the first crop
        that contains an unconfirmed last frame followed by something other than the end of the stream.  With
        check=False nothing is raised; `status` holds each crop's outcome (CLX_ERR_INVALID_ARGUMENT, 90, for a request
        out of range, whose rows are zero and length 0) and a failed crop's rows are unspecified."""
        import torch
        files = _request_column(files, self.batch, "files", "a batch of {}")
        offsets = _request_column(offsets, self.batch, "offsets", "a batch of {}")
        self._requests[:, 0].copy_(files)
        self._requests[:, 1].copy_(offsets)
        self._stream.wait_stream(torch.cuda.current_stream())
        self._batch.decode(0)
        torch.cuda.current_stream().wait_stream(self._stream)
        if check:
            self._raise()
        return self.out, self.lengths

    def _raise(self):
        failure = _first_failure(self._error)
        if failure is None:
            return
        kind, b, st = failure
        fi, o = (int(v) for v in self._requests[b].tolist())
        if kind == 0:
            if not 0 <= fi < len(self.corpus.index):
                raise ValueError(f"crop {b}: file index {fi} out of range")
            N, at = _length_at(self.corpus.index[fi], self.sample_rate)
            raise ValueError(f"crop {b}: offset {o} outside file {fi} ({N} samples{at})")
        raise Error(st, f"file {fi}, crop {b}")

    def kernel_ms(self) -> float:
        """Device time of the last call's graph (CUDA events), planner and status pass included."""
        return self._batch.kernel_ms()


def _hz_to_mel(f, mel_scale: str):
    f = np.asarray(f, dtype=np.float64)
    if mel_scale == "htk":
        return 2595.0 * np.log10(1.0 + f / 700.0)
    f_sp, min_log_hz, logstep = 200.0 / 3, 1000.0, math.log(6.4) / 27.0
    with np.errstate(divide="ignore"):
        return np.where(f >= min_log_hz, min_log_hz / f_sp + np.log(f / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m, mel_scale: str):
    m = np.asarray(m, dtype=np.float64)
    if mel_scale == "htk":
        return 700.0 * (10.0 ** (m / 2595.0) - 1.0)
    f_sp, min_log_hz, logstep = 200.0 / 3, 1000.0, math.log(6.4) / 27.0
    min_log_mel = min_log_hz / f_sp
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def melscale_fbanks(n_freqs: int, f_min: float, f_max: float, n_mels: int, sample_rate: int, norm: str | None = None,
                    mel_scale: str = "htk") -> np.ndarray:
    """torchaudio.functional.melscale_fbanks in float64 numpy: the [n_freqs, n_mels] triangular filterbank over the
    bins linspace(0, sample_rate // 2, n_freqs), its corners equally spaced on the HTK or Slaney mel scale from f_min to
    f_max; norm "slaney" divides each triangle by half its width in Hz."""
    if norm not in (None, "slaney"):
        raise ValueError('norm must be None or "slaney"')
    if mel_scale not in ("htk", "slaney"):
        raise ValueError('mel_scale must be "htk" or "slaney"')
    all_freqs = np.linspace(0.0, float(int(sample_rate) // 2), int(n_freqs))
    m_pts = np.linspace(float(_hz_to_mel(f_min, mel_scale)), float(_hz_to_mel(f_max, mel_scale)), int(n_mels) + 2)
    f_pts = _mel_to_hz(m_pts, mel_scale)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts[None, :] - all_freqs[:, None]
    fb = np.maximum(0.0, np.minimum(-slopes[:, :-2] / f_diff[:-1], slopes[:, 2:] / f_diff[1:]))
    if norm == "slaney":
        fb *= (2.0 / (f_pts[2:n_mels + 2] - f_pts[:n_mels]))[None, :]
    return fb


def _mel_rate(index: FlacIndex, sample_rate: int | None) -> int:
    """The filterbank's rate: `sample_rate` when given, else the corpus's one STREAMINFO rate."""
    if sample_rate is not None:
        return int(sample_rate)
    rates = {f.info.sample_rate for f in index.files}
    if len(rates) != 1:
        raise ValueError(f"a corpus of {len(rates)} sample rates needs sample_rate= for its mel spectrogram")
    return rates.pop()


_MEL_NORMALIZE = {None: 0, "per_feature": MEL_NORM_PER_FEATURE, "whisper": MEL_NORM_WHISPER}


def _mel_tables(sample_rate: int, n_fft: int, win_length, hop_length, f_min: float, f_max, n_mels: int, window_fn,
                wkwargs, center: bool, norm, mel_scale: str, log_floor, normalize=None):
    """MelSpectrogram's arguments and `normalize` as (clx_mel_params, window [win_length] float32, fbank [n_fft // 2 +
    1, n_mels] float32); the C ABI checks the ranges."""
    import torch
    if normalize not in _MEL_NORMALIZE:
        raise ValueError('normalize must be None, "per_feature" or "whisper"')
    if normalize is not None and (log_floor is None or not center):
        raise ValueError(f'normalize="{normalize}" works on log features of centred frames: it needs log_floor and '
                         'center=True')
    n_fft, n_mels = int(n_fft), int(n_mels)
    win_length = n_fft if win_length is None else int(win_length)
    hop_length = win_length // 2 if hop_length is None else int(hop_length)
    f_max = float(sample_rate // 2) if f_max is None else float(f_max)
    flags = MEL_CENTER if center else 0
    if log_floor is not None:
        log_floor = float(log_floor)
        if not (math.isfinite(log_floor) and log_floor > 0):
            raise ValueError("log_floor must be finite and > 0")
        flags |= MEL_LOG
    if min(n_fft, win_length, hop_length, n_mels) < 1:
        raise ValueError("n_fft, win_length, hop_length and n_mels must be >= 1")
    window = (torch.hann_window if window_fn is None else window_fn)(win_length, **(wkwargs or {}))
    window = np.ascontiguousarray(torch.as_tensor(window).detach().cpu().numpy(), dtype=np.float32).reshape(-1)
    if window.size != win_length:
        raise ValueError(f"window_fn gave {window.size} values for win_length {win_length}")
    fbank = np.ascontiguousarray(melscale_fbanks(n_fft // 2 + 1, f_min, f_max, n_mels, sample_rate, norm, mel_scale),
                                 dtype=np.float32)
    params = _lib.MelParams(n_fft, win_length, hop_length, n_mels, flags | _MEL_NORMALIZE[normalize],
                            0.0 if log_floor is None else log_floor)
    return params, window, fbank


class MelCropBatch(CropBatch):
    """The mel spectrogram of every crop of a crop batch, computed on the device inside the batch's CUDA graph
    (clx_batch_create_mel_crops): a call returns (features [B, C, n_mels, F] float32, lengths [B] int64), with the
    requests, `status`, check, stream and sync rules of CropBatch.

    features = MelSpectrogram(x), x the [B, C, L] float32 output of the equivalent CropBatch (the resampled one with
    `sample_rate`) for the same requests, MelSpectrogram being torchaudio.transforms.MelSpectrogram(rate, n_fft=...,
    ...) with power 2, pad_mode "reflect", applied to x as a tensor: each crop is reflect-padded with its own samples,
    and its zero columns and rows are transformed like any others.  F = 1 + L // hop_length with center, else 1 + (L -
    n_fft) // hop_length.  With log_floor, features = ln(max(mel, log_floor)).  An invalid request's features are 0
    (ln(log_floor) with the log); a failed crop's are unspecified.  lengths and status are the crop batch's, lengths in
    samples at the crop's rate.  The filterbank's rate is `sample_rate`, else the corpus's single rate (ValueError for
    a corpus of mixed rates).  n_fft must be even, 8 to 4096, with n_fft / 2 a product of 2, 3 and 5; n_mels at most
    512; L above n_fft / 2 with center, at least n_fft without (Error 90 otherwise).

    `normalize` (log_floor and center required, else ValueError) normalises the log features on the device, in the
    same graph, each statistic and map in float64 rounded once to float32; calls stay bit-identical.
    * "per_feature": for each (crop b, row, mel), over its first v_b = 1 + n_b // hop_length frames (n_b = lengths[b];
      v_b = 0 when n_b = 0), y = (x - mean) / (std + 1e-5) with the unbiased std (0 for one frame): NeMo's per_feature
      normalize_batch, with torch.stft's frame count of the crop's valid samples.  Frames from v_b on read exactly 0,
      and so does every frame of an invalid crop and of a row the file lacks.
    * "whisper": transformers.WhisperFeatureExtractor's log-mel of each crop row as its (zero-padded) input: F - 1
      frames (n_frames; Whisper drops the last STFT frame), l = x / ln 10 and y = (max(l, M - 8) + 4) / 4 with M the
      row's largest l.  Whisper's own features come from mel_crops(B, 480000, 16000, n_fft=400, hop_length=160,
      n_mels=80 (or 128 for large-v3), mel_scale="slaney", norm="slaney", log_floor=1e-10, normalize="whisper"): 30 s
      at 16 kHz, 3000 frames."""

    def __init__(self, corpus: Corpus, batch: int, num_frames: int, sample_rate: int | None = None, *,
                 n_fft: int = 400, win_length: int | None = None, hop_length: int | None = None, f_min: float = 0.0,
                 f_max: float | None = None, n_mels: int = 128, window_fn=None, wkwargs: dict | None = None,
                 center: bool = True, norm: str | None = None, mel_scale: str = "htk", log_floor: float | None = None,
                 normalize: str | None = None):
        self._args(corpus, batch, num_frames, None, sample_rate)
        params, window, fbank = _mel_tables(_mel_rate(corpus.index, self.sample_rate), n_fft, win_length, hop_length,
                                            f_min, f_max, n_mels, window_fn, wkwargs, center, norm, mel_scale,
                                            log_floor, normalize)
        self.normalize = normalize
        self.params, self.fbank, self.window = params, fbank, window
        L = self.ctx._L
        h = C.c_void_p()
        _check(L.clx_batch_create_mel_crops(self.ctx._h, corpus._h, corpus._file_rates().ctypes.data, len(corpus.index),
                                            self.batch, self.num_frames, self.sample_rate or 0, C.byref(params),
                                            window.ctypes.data, fbank.ctypes.data, C.byref(h)), self.ctx)
        self.channels, self.n_mels = corpus.channels, params.n_mels
        self.n_frames = (1 + self.num_frames // params.hop_length if center else
                         1 + (self.num_frames - params.n_fft) // params.hop_length) - (normalize == "whisper")
        self._attach(h, (self.batch, self.channels, self.n_mels, self.n_frames), "<f4")


def _request_column(x, n: int | None, what: str, of_n: str = "{} files"):
    """A request column as an int64 CUDA tensor (integers only; CPU values are copied through pinned memory) of n values
    unless n is None; `of_n` names n in the error."""
    import torch
    if isinstance(x, torch.Tensor):
        if x.dtype.is_floating_point or x.dtype.is_complex or x.dtype == torch.bool:
            raise TypeError(f"{what} must hold integers")
        t = x.reshape(-1)
    else:
        t = torch.from_numpy(np.asarray(x, dtype=np.int64).reshape(-1))
    if n is not None and t.numel() != n:
        raise ValueError(f"{what}: {t.numel()} values for {of_n.format(n)}")
    if not t.is_cuda:
        t = t.to(torch.int64).pin_memory().to("cuda", non_blocking=True)
    return t


class PackedBatch:
    """Whole files or excerpts of different lengths of a Corpus's files, packed along the columns of one [C, T] CUDA
    tensor per call (clx_batch_create_packed), the layout of load(): excerpt b starts at column starts[b], each start a
    multiple of 4, start_{b+1} = start_b + round_up_4(n_b).  As for CropBatch, the frames, windows and columns are planned
    on the device inside the batch's CUDA graph, so a call is a few small device copies and one graph launch, and the
    requests may be CUDA tensors.  C is the corpus's largest channel count, T = max_samples.

    Excerpt b is samples [offsets[b], offsets[b] + n_b) of file files[b], n_b = min(lengths[b], N - offsets[b]) (to the
    file's end for a length of -1, the default; offsets default to 0).  Channel c goes to row c; every other element of
    the [C, T] output reads 0.  An excerpt whose columns would pass T does not fit: it gets length 0 and status 90, like
    an invalid request (the excerpts that fit are a prefix of the valid ones).  `out`, `starts`, `lengths` and `status`
    are views of the batch's own buffers, overwritten by the next call; the next call waits for what torch's current
    stream has enqueued before it.  A float32 batch is refused when any frame of the corpus has more than 24 bits.
    Memory: C x (T + the trash columns) output elements and a planar scratch of the corpus's largest frame for each of
    packed_frames_bound(max_excerpts, T) slots; over a host corpus also a staging buffer of packed_bytes_bound() bytes,
    and each call reads the selected spans over PCIe.

    With `sample_rate` R (clx_batch_create_resampled_packed; float32 only), files of any rate give excerpts at rate R,
    with the filter of CropBatch's `sample_rate`.  Everything counts samples at R: offsets, lengths, T, the starts and
    the returned lengths.  Excerpt b is resample(x, r, R)[:, offsets[b] : offsets[b] + n_b], x the whole file as load()
    gives it and r its STREAMINFO rate, with n_b = min(lengths[b], N_t - offsets[b]) and N_t = ceil(N * R / r) the
    file's length at R; so the samples near an excerpt's edges are those of the resampled file, not zero-padded.  An
    offset past N_t is invalid, one at N_t the valid empty excerpt; the layout and the fit rule are those above.  Files
    already at R are copied: over a corpus whose files are all at R, a call gives what a float32 batch without
    sample_rate gives, bit for bit.  An excerpt's status is that of its source span, the samples its outputs read.
    Memory: the [C, round_up_4(T)] output, and an inner packed batch of T_src = resample_packed_source_bound(max_excerpts,
    T, R) columns that decodes every excerpt's source span (about C x T_src float32 plus its slot scratch, so about T x
    r / R samples per row for the highest rate r: 6 x T for 96 kHz to 16 kHz)."""

    def __init__(self, corpus: Corpus, max_excerpts: int, max_samples: int, dtype=None, sample_rate: int | None = None):
        mode = self._args(corpus, max_excerpts, max_samples, dtype, sample_rate)
        L = self.ctx._L
        h = C.c_void_p()
        if self.sample_rate is None:
            _check(L.clx_batch_create_packed(self.ctx._h, corpus._h, self.max_excerpts, self.max_samples, mode,
                                             C.byref(h)), self.ctx)
        else:
            _check(L.clx_batch_create_resampled_packed(self.ctx._h, corpus._h, corpus._file_rates().ctypes.data,
                                                       len(corpus.index), self.max_excerpts, self.max_samples,
                                                       self.sample_rate, C.byref(h)), self.ctx)
        self.channels = corpus.channels
        self._attach(h, (self.channels,), "<f4" if mode == OUT_CHANNELS_F32 else "<i4")
        self.out = self.out[:, :self.max_samples]

    def _args(self, corpus: Corpus, max_excerpts: int, max_samples: int, dtype, sample_rate: int | None) -> int:
        """Checks and keeps the arguments of every packed batch; returns the output mode."""
        import torch
        self.corpus, self.ctx = corpus, corpus.ctx
        self.max_excerpts, self.max_samples, self.dtype = int(max_excerpts), int(max_samples), _torch_dtype(dtype)
        self.sample_rate = None if sample_rate is None else int(sample_rate)
        if self.max_excerpts < 1 or self.max_samples < 1:
            raise ValueError("max_excerpts and max_samples must be >= 1")
        if self.sample_rate is not None and self.dtype != torch.float32:
            raise ValueError("a resampled packed batch is float32 only")
        return _channels_mode(self.dtype)

    def _attach(self, h, out_shape: tuple, typestr: str):
        """Takes ownership of the created batch `h` and views its buffers: out (out_shape, then the batch's stride),
        starts, lengths, status, requests, count, error."""
        import torch
        L = self.ctx._L
        self._batch = _Batch(self.ctx, h, keep=self.corpus)
        self.stride = int(L.clx_batch_packed_stride(h))
        B, view = self.max_excerpts, self._batch.tensor
        self.out = view(L.clx_batch_device_out(h), (*out_shape, self.stride), typestr)
        self._starts = view(L.clx_batch_packed_starts(h), (B,), "<i8")
        self._lengths = view(L.clx_batch_crop_lengths(h), (B,), "<i8")
        self._status = view(L.clx_batch_crop_status(h), (B,), "<i4")
        self._requests = view(L.clx_batch_packed_requests(h), (B, 3), "<i8")  # {u32 file, u32 reserved}, offset, length
        self._count = view(L.clx_batch_packed_count(h), (1,), "<i4")
        self._error = view(L.clx_batch_crop_error(h), (1,), "<i8")
        self._stream = torch.cuda.ExternalStream(L.clx_ctx_stream(self.ctx._h, 0))
        self._n = 0

    @property
    def status(self):
        """Each excerpt's status of the last call (an int32 CUDA tensor view)."""
        return self._status[:self._n]

    def __call__(self, files, offsets=None, lengths=None, check: bool = True):
        """Decodes excerpt b = samples [offsets[b], offsets[b] + lengths[b]) of file files[b], cut at the file's end,
        for each of the n <= max_excerpts files.  Returns (out [C, T], starts [n] int64, lengths [n] int64), on the GPU.
        The requests are copied and the count set on torch's current stream, the batch's stream waits for it and torch's
        stream waits for the decode: nothing syncs with the host unless `check`.  check=True syncs once and raises, for
        the first excerpt in order that has one: ValueError for an invalid request or an excerpt that does not fit, else
        Error(status, "file i, excerpt b") for a failed frame or what follows a file's unconfirmed last frame.  With
        check=False nothing is raised and `status` holds each excerpt's outcome (90 for an invalid or non-fitting one)."""
        import torch
        files = _request_column(files, None, "files")
        n = files.numel()
        if n > self.max_excerpts:
            raise ValueError(f"{n} excerpts for a batch of at most {self.max_excerpts}")
        req = self._requests[:n]
        req[:, 0].copy_(files)
        if offsets is None:
            req[:, 1].zero_()
        else:
            req[:, 1].copy_(_request_column(offsets, n, "offsets"))
        if lengths is None:
            req[:, 2].fill_(-1)
        else:
            req[:, 2].copy_(_request_column(lengths, n, "lengths"))
        self._count.fill_(n)
        self._n = n
        self._stream.wait_stream(torch.cuda.current_stream())
        self._batch.decode(0)
        torch.cuda.current_stream().wait_stream(self._stream)
        if check:
            self._raise()
        return self.out, self._starts[:n], self._lengths[:n]

    def _raise(self):
        failure = _first_failure(self._error)
        if failure is None:
            return
        kind, b, st = failure
        fi, o, ln = (int(v) for v in self._requests[b].tolist())
        if kind == 0:
            if not 0 <= fi < len(self.corpus.index):
                raise ValueError(f"excerpt {b}: file index {fi} out of range")
            N, at = _length_at(self.corpus.index[fi], self.sample_rate)
            if not 0 <= o <= N:
                raise ValueError(f"excerpt {b}: offset {o} outside file {fi} ({N} samples{at})")
            if ln == 0 or ln < -1:
                raise ValueError(f"excerpt {b}: length {ln} (must be >= 1, or -1 for the rest of the file)")
            start = self._sample_start(b)
            n = N - o if ln == -1 else min(ln, N - o)
            raise ValueError(f"excerpt {b}: needs columns [{start}, {start + n}){at}, past max_samples "
                             f"{self.max_samples}")
        raise Error(st, f"file {fi}, excerpt {b}")

    def _sample_start(self, b: int) -> int:
        """Excerpt b's first column (one sync)."""
        return int(self._starts[b].item())

    def kernel_ms(self) -> float:
        """Device time of the last call's graph (CUDA events), planner and status pass included."""
        return self._batch.kernel_ms()


class MelPackedBatch(PackedBatch):
    """The mel spectrogram of every excerpt of a packed batch, packed along frames and computed on the device inside
    the batch's CUDA graph (clx_batch_create_mel_packed): a call returns (features [C, n_mels, T_f] float32, starts [n]
    int64, frames [n] int64, lengths [n] int64), all views of the batch's own buffers, with the requests, `status`,
    check, stream and sync rules of PackedBatch, and its raises (offsets, lengths and columns in samples at the
    batch's rate).  The parameters are MelCropBatch's.

    Take x [C, T], s_b and n_b the output, sample starts and lengths of the equivalent float32 PackedBatch (the
    resampled one with `sample_rate`) for the same requests.  Excerpt b's F_b frames are MelSpectrogram(x[:, s_b : s_b +
    n_b]), as MelCropBatch computes it: each excerpt is reflect-padded with its own samples at its own two edges, as
    torchaudio does on what load(file, frame_offset=o, num_frames=n) returns, and rows its file does not have are zeros
    transformed like any others (exactly 0, or ln(log_floor)).  F_b = 1 + n_b // hop_length with center when n_b >
    n_fft / 2, 1 + (n_b - n_fft) // hop_length without when n_b >= n_fft, else 0: invalid, non-fitting, empty and too
    short excerpts have no frames (a too short one keeps status 0 and its length in samples).  Excerpt b's frames are
    columns [starts[b], starts[b] + frames[b]) of every (row, mel), starts[0] = 0 and starts[b + 1] = starts[b] +
    round_up_4(frames[b]); every other element of the features reads exactly 0 after every call, with or without the
    log.  T_f = Corpus.mel_packed_frames_bound(max_excerpts, max_samples, ...) holds the frames of any excerpts that fit
    in max_samples columns, so only the packed batch's fit rule applies.  Calls are bit-identical.  Memory: the packed
    batch and C x n_mels x T_f float32.

    normalize="per_feature" (log_floor and center required) normalises each (excerpt b, row, mel) over its F_b frames
    as MelCropBatch does a crop's valid frames: y = (x - mean) / (std + 1e-5), unbiased std, 0 for one frame; the
    layout, starts and frame counts are unchanged and every other element still reads 0.  "whisper" is refused
    (ValueError): Whisper's input is a fixed 30 s window, and per-excerpt maxima match no reference."""

    def __init__(self, corpus: Corpus, max_excerpts: int, max_samples: int, sample_rate: int | None = None, *,
                 n_fft: int = 400, win_length: int | None = None, hop_length: int | None = None, f_min: float = 0.0,
                 f_max: float | None = None, n_mels: int = 128, window_fn=None, wkwargs: dict | None = None,
                 center: bool = True, norm: str | None = None, mel_scale: str = "htk", log_floor: float | None = None,
                 normalize: str | None = None):
        if normalize == "whisper":
            raise ValueError('normalize="whisper" is for crop batches (Whisper reads fixed 30 s windows)')
        self._args(corpus, max_excerpts, max_samples, None, sample_rate)
        params, window, fbank = _mel_tables(_mel_rate(corpus.index, self.sample_rate), n_fft, win_length, hop_length,
                                            f_min, f_max, n_mels, window_fn, wkwargs, center, norm, mel_scale,
                                            log_floor, normalize)
        self.normalize = normalize
        self.params, self.fbank, self.window = params, fbank, window
        L = self.ctx._L
        h = C.c_void_p()
        _check(L.clx_batch_create_mel_packed(self.ctx._h, corpus._h, corpus._file_rates().ctypes.data,
                                             len(corpus.index), self.max_excerpts, self.max_samples,
                                             self.sample_rate or 0, C.byref(params), window.ctypes.data,
                                             fbank.ctypes.data, C.byref(h)), self.ctx)
        self.channels, self.n_mels = corpus.channels, params.n_mels
        self._attach(h, (self.channels, self.n_mels), "<f4")  # stride: T_f
        self._frames = self._batch.tensor(L.clx_batch_mel_frames(h), (self.max_excerpts,), "<i8")

    def __call__(self, files, offsets=None, lengths=None, check: bool = True):
        """Computes the features of excerpt b = samples [offsets[b], offsets[b] + lengths[b]) of file files[b], cut at
        the file's end, for each of the n <= max_excerpts files, as PackedBatch.__call__ decodes them.  Returns
        (features [C, n_mels, T_f], starts [n], frames [n], lengths [n]): frame starts and counts, lengths in samples."""
        out, starts, lengths = super().__call__(files, offsets, lengths, check)
        return out, starts, self._frames[:self._n], lengths

    def _sample_start(self, b: int) -> int:
        """Excerpt b's first sample column in the packed batch, for the first excerpt the error word reports: the ones
        before it are valid and fit, so it is the sum of their round_up_4(length) (one sync)."""
        return int(((self._lengths[:b] + 3) // 4 * 4).sum().item())
