"""ctypes binding of the C ABI declared in include/claxon_b200.h.

The shared library is the product; this module only loads it.  There is no Python or
CPU fallback for the decode path: if the library cannot be loaded, or no CUDA device is
usable, the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

from . import _build


class FrameDesc(C.Structure):
    _fields_ = [
        ("byte_offset", C.c_uint64), ("byte_len", C.c_uint32), ("header_len", C.c_uint16),
        ("block_size", C.c_uint16), ("n_channels", C.c_uint8), ("channel_assignment", C.c_uint8),
        ("bits_per_sample", C.c_uint8), ("flags", C.c_uint8), ("sample_rate", C.c_uint32),
        ("number", C.c_uint64), ("out_offset", C.c_uint64),
    ]


class FrameResult(C.Structure):
    _fields_ = [("status", C.c_int32), ("consumed", C.c_uint32)]


class StreamInfoC(C.Structure):
    _fields_ = [
        ("min_block_size", C.c_uint32), ("max_block_size", C.c_uint32),
        ("min_frame_size", C.c_uint32), ("max_frame_size", C.c_uint32),
        ("sample_rate", C.c_uint32), ("channels", C.c_uint32), ("bits_per_sample", C.c_uint32),
        ("samples", C.c_uint64), ("md5sum", C.c_uint8 * 16),
    ]


class FrameWindow(C.Structure):
    _fields_ = [("row", C.c_uint32), ("first", C.c_uint32), ("count", C.c_uint32), ("reserved", C.c_uint32)]


class Options(C.Structure):
    _fields_ = [("device", C.c_int32), ("flags", C.c_uint32), ("n_streams", C.c_uint32),
                ("host_threads", C.c_uint32)]


class ImageHeader(C.Structure):  # clx_image_header: the header of a corpus image
    _fields_ = [("magic", C.c_uint64), ("version", C.c_uint32), ("header_bytes", C.c_uint32),
                ("n_files", C.c_uint64), ("n_frames", C.c_uint64), ("files_offset", C.c_uint64), ("files_bytes", C.c_uint64),
                ("descs_offset", C.c_uint64), ("descs_bytes", C.c_uint64), ("bytes_offset", C.c_uint64),
                ("bytes_size", C.c_uint64), ("nbytes", C.c_uint64), ("total_bytes", C.c_uint64)]


class ImageFile(C.Structure):  # clx_image_file: one file's record in a corpus image
    _fields_ = [("info", StreamInfoC), ("byte_base", C.c_uint64), ("byte_count", C.c_uint64),
                ("first_frame", C.c_uint32), ("n_frames", C.c_uint32), ("flags", C.c_uint32), ("tail", C.c_int32)]


class MelParams(C.Structure):  # clx_mel_params
    _fields_ = [("n_fft", C.c_uint32), ("win_length", C.c_uint32), ("hop_length", C.c_uint32), ("n_mels", C.c_uint32),
                ("flags", C.c_uint32), ("log_floor", C.c_float)]


assert C.sizeof(FrameDesc) == 40 and C.sizeof(FrameResult) == 8 and C.sizeof(FrameWindow) == 16
assert C.sizeof(StreamInfoC) == 56 and C.sizeof(ImageHeader) == 96 and C.sizeof(ImageFile) == 88
assert C.sizeof(MelParams) == 24

OPT_NO_VERIFY_CRC = 1
OPT_GENERIC_KERNEL_ONLY = 2
OPT_WARP_PER_FRAME = 4
OPT_LANE_PER_FRAME = 8
OPT_NO_GENERIC = 16
OPT_NO_WIDE = 32
OPEN_METADATA_ONLY, OPEN_NO_VORBIS_COMMENT = 1, 2
BATCH_BYTES_ON_DEVICE = 1
CORPUS_HOST = 1
MEL_CENTER, MEL_LOG = 1, 2
MEL_NORM_PER_FEATURE, MEL_NORM_WHISPER = 4, 8
IMAGE_MAGIC, IMAGE_VERSION, IMAGE_ALIGN, IMAGE_END_CONFIRMED = 0x3150524F43584C43, 1, 4096, 1
OUT_PLANAR_I32, OUT_INTERLEAVED_I32, OUT_INTERLEAVED_I16, OUT_INTERLEAVED_I24 = 0, 1, 2, 3
OUT_CHANNELS_I32, OUT_CHANNELS_F32 = 4, 5
FRAME_VARIABLE_BLOCKING = 1
FRAME_CRC16_VERIFIED = 2

# every exported symbol of include/claxon_b200.h: (restype, argtypes)
_vp, _sz, _u8p = C.c_void_p, C.c_size_t, C.c_void_p
SYMBOLS = {
    "clx_status_str": (C.c_char_p, [C.c_int]),
    "clx_status_kind": (C.c_int, [C.c_int]),
    "clx_abi_version": (C.c_uint32, []),
    "clx_parse_frame_header": (C.c_int, [_u8p, _sz, C.POINTER(FrameDesc), C.c_uint32]),
    "clx_open_stream": (C.c_int, [_u8p, _sz, C.POINTER(StreamInfoC), C.POINTER(C.c_uint64)]),
    "clx_open_stream_ex": (C.c_int, [_u8p, _sz, C.c_uint32, C.POINTER(StreamInfoC), C.POINTER(C.c_uint64),
                                     C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]),
    "clx_demux_frames": (_sz, [_u8p, _sz, C.c_uint64, _vp, _sz, C.POINTER(C.c_uint64),
                               C.POINTER(C.c_uint64), C.POINTER(C.c_int), C.c_uint32]),
    "clx_demux_frames_mt": (_sz, [_u8p, _sz, C.c_uint64, _vp, _sz, C.POINTER(C.c_uint64),
                                  C.POINTER(C.c_uint64), C.POINTER(C.c_int), C.c_uint32, C.c_uint32]),
    "clx_ogg_frames": (C.c_int, [_u8p, _sz, C.POINTER(StreamInfoC), _vp, _sz, _vp, _sz, C.POINTER(_sz), C.POINTER(_sz),
                                 C.POINTER(C.c_uint64), C.c_uint32]),
    "clx_mp4_frames": (C.c_int, [_u8p, _sz, C.POINTER(StreamInfoC), _vp, _sz, C.POINTER(_sz), C.POINTER(C.c_uint64), C.c_uint32]),
    "clx_crc8": (C.c_uint8, [_u8p, _sz]),
    "clx_crc16": (C.c_uint16, [_u8p, _sz]),
    "clx_ctx_create": (C.c_int, [C.POINTER(Options), C.POINTER(_vp)]),
    "clx_ctx_destroy": (None, [_vp]),
    "clx_ctx_last_error": (C.c_char_p, [_vp]),
    "clx_decode_frames": (C.c_int, [_vp, _u8p, _sz, _vp, _sz, _vp, _sz, _vp]),
    "clx_decode_frames_to": (C.c_int, [_vp, _u8p, _sz, _vp, _sz, _vp, _sz, _vp, C.c_uint32]),
    "clx_batch_create": (C.c_int, [_vp, _u8p, _sz, _vp, _sz, _sz, C.POINTER(_vp)]),
    "clx_batch_create_ex": (C.c_int, [_vp, _u8p, _sz, _vp, _sz, _sz, C.c_uint32, C.POINTER(_vp)]),
    "clx_batch_create_to": (C.c_int, [_vp, _u8p, _sz, _vp, _sz, _sz, C.c_uint32, C.c_uint32, C.POINTER(_vp)]),
    "clx_batch_create_channels": (C.c_int, [_vp, _u8p, _sz, _vp, _sz, C.c_uint32, _sz, C.c_uint32, C.c_uint32,
                                            C.POINTER(_vp)]),
    "clx_batch_create_windows": (C.c_int, [_vp, _u8p, _sz, _vp, _vp, _sz, C.c_uint32, _sz, C.c_uint32, C.c_uint32,
                                           C.POINTER(_vp)]),
    "clx_corpus_create": (C.c_int, [_vp, _u8p, _sz, _vp, _sz, _vp, _sz, C.POINTER(_vp)]),
    "clx_corpus_create_ex": (C.c_int, [_vp, _u8p, _sz, _vp, _sz, _vp, _sz, C.c_uint32, C.POINTER(_vp)]),
    "clx_corpus_destroy": (C.c_int, [_vp, _vp]),
    "clx_corpus_device_bytes": (_sz, [_vp]),
    "clx_crop_frames_bound": (_sz, [_vp, _sz, _vp, _sz, _sz]),
    "clx_crop_bytes_bound": (_sz, [_vp, _sz, _vp, _sz, _sz]),
    "clx_batch_create_crops": (C.c_int, [_vp, _vp, _sz, _sz, C.c_uint32, C.POINTER(_vp)]),
    "clx_batch_crop_requests": (_vp, [_vp]),
    "clx_batch_crop_status": (_vp, [_vp]),
    "clx_batch_crop_lengths": (_vp, [_vp]),
    "clx_batch_crop_error": (_vp, [_vp]),
    "clx_crop_filler_frame": (_sz, [_vp, _sz]),
    "clx_batch_create_packed": (C.c_int, [_vp, _vp, _sz, _sz, C.c_uint32, C.POINTER(_vp)]),
    "clx_packed_frames_bound": (_sz, [_vp, _sz, _vp, _sz, _sz, _sz]),
    "clx_packed_bytes_bound": (_sz, [_vp, _sz, _vp, _sz, _sz, _sz]),
    "clx_corpus_image_bytes": (_sz, [_vp, _vp, _sz, _vp, _sz]),
    "clx_corpus_image_write": (C.c_int, [_vp, _vp, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _sz]),
    "clx_corpus_image_check": (C.c_int, [_vp, _sz]),
    "clx_corpus_attach": (C.c_int, [_vp, _vp, _sz, C.POINTER(_vp)]),
    "clx_batch_packed_requests": (_vp, [_vp]),
    "clx_batch_packed_count": (_vp, [_vp]),
    "clx_batch_packed_starts": (_vp, [_vp]),
    "clx_batch_packed_stride": (_sz, [_vp]),
    "clx_batch_create_resampled_crops": (C.c_int, [_vp, _vp, _vp, _sz, _sz, _sz, C.c_uint32, C.POINTER(_vp)]),
    "clx_resample_source_bound": (_sz, [C.c_uint32, C.c_uint32, _sz]),
    "clx_batch_create_resampled_packed": (C.c_int, [_vp, _vp, _vp, _sz, _sz, _sz, C.c_uint32, C.POINTER(_vp)]),
    "clx_resample_packed_source_bound": (_sz, [_vp, _sz, C.c_uint32, _sz, _sz]),
    "clx_batch_create_mel_crops": (C.c_int, [_vp, _vp, _vp, _sz, _sz, _sz, C.c_uint32, _vp, _vp, _vp, C.POINTER(_vp)]),
    "clx_batch_create_mel_packed": (C.c_int, [_vp, _vp, _vp, _sz, _sz, _sz, C.c_uint32, _vp, _vp, _vp, C.POINTER(_vp)]),
    "clx_mel_packed_frames_bound": (_sz, [_vp, _sz, _sz]),
    "clx_batch_mel_frames": (_vp, [_vp]),
    "clx_batch_decode": (C.c_int, [_vp, _vp, C.c_uint32]),
    "clx_batch_sync": (C.c_int, [_vp, _vp]),
    "clx_batch_read": (C.c_int, [_vp, _vp, _vp, _sz, _vp]),
    "clx_batch_read_to": (C.c_int, [_vp, _vp, _vp, _sz, _vp]),
    "clx_batch_destroy": (None, [_vp, _vp]),
    "clx_batch_device_out": (_vp, [_vp]),
    "clx_batch_device_bytes": (_vp, [_vp]),
    "clx_batch_last_kernel_ms": (C.c_int, [_vp, _vp, C.POINTER(C.c_float)]),
    "clx_ctx_run_steps": (C.c_int, [_vp, C.POINTER(_vp), _sz, C.c_uint32, C.c_uint32, C.POINTER(C.c_float)]),
    "clx_ctx_launch_count": (C.c_uint64, [_vp]),
    "clx_ctx_stream": (_vp, [_vp, C.c_uint32]),
    "clx_host_alloc": (_vp, [_sz]),
    "clx_host_free": (None, [_vp]),
    "clx_reader_open_frames": (C.c_int, [_vp, _u8p, _sz, C.POINTER(_vp)]),
    "clx_reader_open_flac": (C.c_int, [_vp, _u8p, _sz, C.POINTER(_vp)]),
    "clx_reader_streaminfo": (C.c_int, [_vp, C.POINTER(StreamInfoC)]),
    "clx_reader_next": (C.c_int, [_vp, _vp, _sz, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                  C.POINTER(C.c_uint64)]),
    "clx_reader_plan_batch": (C.c_int, [_vp, _sz, C.POINTER(_sz), C.POINTER(C.c_uint64)]),
    "clx_reader_next_batch": (C.c_int, [_vp, _sz, _vp, _sz, _vp, C.POINTER(_sz)]),
    "clx_reader_position": (C.c_uint64, [_vp]),
    "clx_reader_close": (None, [_vp]),
}

_lib = None


def load():
    """Loads (building first if the sources are newer) libclaxon_b200.so."""
    global _lib
    if _lib is None:
        path = _build.build_lib()
        L = C.CDLL(path, mode=os.RTLD_GLOBAL if hasattr(os, "RTLD_GLOBAL") else 0)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the library does not export the symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib
