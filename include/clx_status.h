/* clx_status.h — per-frame / per-stream status codes of the claxon_b200 C ABI.
 *
 * One value per row of claxon's error catalogue on the frame-decode path
 * (SURVEY.md Appendix B).  claxon reports errors as
 *   Error::{IoError, FormatError(&'static str), Unsupported(&'static str)}
 * (reference src/error.rs:18-32) and compares them BY STRING
 * (src/error.rs:34-45); `clx_status_str()` returns that exact string and
 * `clx_status_kind()` the variant, so a binding can rebuild the Rust value.
 *
 * This header is shared by the product library and by the test oracle so the
 * two can be compared status-for-status.  It contains no code from claxon.
 */
#ifndef CLX_STATUS_H
#define CLX_STATUS_H

#ifdef __cplusplus
extern "C" {
#endif

/* Two negative values appear only under the test options of claxon_b200.h, which switch off the kernels
 * that would otherwise take a frame over: -2 (CLX_OPT_NO_GENERIC: a fast path declined the frame, the generic
 * kernel would have decoded it) and -3 (CLX_OPT_NO_WIDE: the frame needed the lane-per-frame path's i64 second
 * chance).  No other call ever returns a negative status. */
typedef enum clx_status {
    CLX_OK = 0,
    /* Ok(None): end of stream while reading the first two header bytes
     * (src/frame.rs:140-143). */
    CLX_EOF = 1,
    /* Error::IoError(UnexpectedEof): any other read past the end of input
     * (src/input.rs:139-142, :242). */
    CLX_ERR_IO_UNEXPECTED_EOF = 2,

    /* --- frame header (src/frame.rs:131-316) --- */
    CLX_ERR_SYNC_MISSING = 3,            /* :148 */
    CLX_ERR_FRAME_HEADER_RESERVED = 4,   /* :157 :177 :224 :236 :241 */
    CLX_ERR_FRAME_HEADER_INVALID = 5,    /* :210 */
    CLX_ERR_VARINT_INVALID = 6,          /* :82 :98 */
    CLX_ERR_FRAME_NUMBER_TOO_LARGE = 7,  /* :255 */
    CLX_ERR_BLOCK_SIZE_65535 = 8,        /* :273 */
    CLX_ERR_HEADER_CRC_MISMATCH = 9,     /* :300 */
    CLX_ERR_NO_BPS_IN_HEADER = 10,       /* :691 (Unsupported) */

    /* --- subframe (src/subframe.rs) --- */
    CLX_ERR_SUBFRAME_HEADER_INVALID = 11,   /* :32  */
    CLX_ERR_SUBFRAME_HEADER_RESERVED = 12,  /* :47 :55 */
    CLX_ERR_WASTED_BITS_GT_31 = 13,         /* :83  */
    CLX_ERR_NO_NON_WASTED_BITS = 14,        /* :199 */
    CLX_ERR_RESIDUAL_RESERVED = 15,         /* :245 */
    CLX_ERR_PARTITION_ORDER_INVALID = 16,   /* :263 */
    CLX_ERR_RESIDUAL_INVALID = 17,          /* :276 */
    CLX_ERR_UNENCODED_BINARY = 18,          /* :318 :366 (Unsupported) */
    CLX_ERR_FIXED_ORDER_GT_BLOCK = 19,      /* :500 */
    CLX_ERR_LPC_ORDER_GT_BLOCK = 20,        /* :663 */
    CLX_ERR_QLP_PRECISION_INVALID = 21,     /* :674 */
    CLX_ERR_NEGATIVE_QLP_SHIFT = 22,        /* :688-690 (Unsupported) */

    /* --- frame footer (src/frame.rs:752-763) --- */
    CLX_ERR_FRAME_CRC_MISMATCH = 23,        /* :761 */

    /* --- stream / metadata level, host only (src/lib.rs, src/metadata.rs) --- */
    CLX_ERR_STREAM_HEADER_INVALID = 30,     /* lib.rs:200 */
    CLX_ERR_STREAM_HEADER_ID3 = 31,         /* lib.rs:198 */
    CLX_ERR_STREAMINFO_MISSING = 32,        /* lib.rs:247 */
    CLX_ERR_SECOND_VORBIS_COMMENT = 33,     /* lib.rs:259 */
    CLX_ERR_SECOND_STREAMINFO = 34,         /* lib.rs:268 */
    CLX_ERR_STREAMINFO_LENGTH = 35,         /* metadata.rs:272 */
    CLX_ERR_METADATA_BLOCK_TYPE = 36,       /* metadata.rs:304 */
    CLX_ERR_BLOCK_SIZE_BOUNDS = 37,         /* metadata.rs:360 */
    CLX_ERR_BLOCK_SIZE_LT_16 = 38,          /* metadata.rs:363 */
    CLX_ERR_FRAME_SIZE_BOUNDS = 39,         /* metadata.rs:366 */
    CLX_ERR_SAMPLE_RATE_INVALID = 40,       /* metadata.rs:372 */
    CLX_ERR_VORBIS_TOO_SHORT = 41,          /* metadata.rs:406 */
    CLX_ERR_VORBIS_TOO_LARGE = 42,          /* metadata.rs:423 (Unsupported) */
    CLX_ERR_VENDOR_TOO_LONG = 43,           /* metadata.rs:431 */
    CLX_ERR_VORBIS_TOO_MANY = 44,           /* metadata.rs:446 */
    CLX_ERR_VORBIS_COMMENT_TOO_LONG = 45,   /* metadata.rs:461 */
    CLX_ERR_VORBIS_NAME_INVALID = 46,       /* metadata.rs:488 */
    CLX_ERR_VORBIS_NO_EQUALS = 47,          /* metadata.rs:495 */
    CLX_ERR_VORBIS_EXCESS_DATA = 48,        /* metadata.rs:500 */
    CLX_ERR_VORBIS_WRONG_COUNT = 49,        /* metadata.rs:504 */
    CLX_ERR_APPLICATION_TOO_SHORT = 50,     /* metadata.rs:527 */
    CLX_ERR_APPLICATION_TOO_LARGE = 51,     /* metadata.rs:535 (Unsupported) */
    CLX_ERR_UTF8_INVALID = 52,              /* String::from_utf8 failure, error.rs From<FromUtf8Error> */

    /* --- library level (no claxon counterpart) --- */
    CLX_ERR_INVALID_ARGUMENT = 90,
    CLX_ERR_CUDA = 91,
    CLX_ERR_NO_DEVICE = 92,
    CLX_ERR_CONTAINER = 93      /* malformed / unsupported Ogg or MP4 wrapper (the reference leaves containers to other crates) */
} clx_status;

/* Error variant of a status, mirroring claxon::Error. */
typedef enum clx_error_kind {
    CLX_KIND_NONE = 0,         /* CLX_OK / CLX_EOF */
    CLX_KIND_IO = 1,           /* Error::IoError */
    CLX_KIND_FORMAT = 2,       /* Error::FormatError */
    CLX_KIND_UNSUPPORTED = 3,  /* Error::Unsupported */
    CLX_KIND_LIBRARY = 4       /* not a claxon error */
} clx_error_kind;

static inline const char* clx_status_str_inline(int s) {
    switch (s) {
    case CLX_OK: return "ok";
    case CLX_EOF: return "end of stream";
    case CLX_ERR_IO_UNEXPECTED_EOF: return "UnexpectedEof";
    case CLX_ERR_SYNC_MISSING: return "frame sync code missing";
    case CLX_ERR_FRAME_HEADER_RESERVED: return "invalid frame header, encountered reserved value";
    case CLX_ERR_FRAME_HEADER_INVALID: return "invalid frame header";
    case CLX_ERR_VARINT_INVALID: return "invalid variable-length integer";
    case CLX_ERR_FRAME_NUMBER_TOO_LARGE: return "invalid frame header, frame number too large";
    case CLX_ERR_BLOCK_SIZE_65535: return "invalid block size, exceeds 65535";
    case CLX_ERR_HEADER_CRC_MISMATCH: return "frame header CRC mismatch";
    case CLX_ERR_NO_BPS_IN_HEADER: return "header without bits per sample info";
    case CLX_ERR_SUBFRAME_HEADER_INVALID: return "invalid subframe header";
    case CLX_ERR_SUBFRAME_HEADER_RESERVED: return "invalid subframe header, encountered reserved value";
    case CLX_ERR_WASTED_BITS_GT_31: return "wasted bits per sample must not exceed 31";
    case CLX_ERR_NO_NON_WASTED_BITS: return "subframe has no non-wasted bits";
    case CLX_ERR_RESIDUAL_RESERVED: return "invalid residual, encountered reserved value";
    case CLX_ERR_PARTITION_ORDER_INVALID: return "invalid partition order";
    case CLX_ERR_RESIDUAL_INVALID: return "invalid residual";
    case CLX_ERR_UNENCODED_BINARY: return "unencoded binary is not yet implemented";
    case CLX_ERR_FIXED_ORDER_GT_BLOCK: return "invalid fixed subframe, order is larger than block size";
    case CLX_ERR_LPC_ORDER_GT_BLOCK: return "invalid LPC subframe, lpc order is larger than block size";
    case CLX_ERR_QLP_PRECISION_INVALID: return "invalid subframe, qlp precision value invalid";
    case CLX_ERR_NEGATIVE_QLP_SHIFT:
        return "a negative quantized linear predictor coefficient shift is not supported, please file a bug.";
    case CLX_ERR_FRAME_CRC_MISMATCH: return "frame CRC mismatch";
    case CLX_ERR_STREAM_HEADER_INVALID: return "invalid stream header";
    case CLX_ERR_STREAM_HEADER_ID3: return "stream starts with ID3 header rather than FLAC header";
    case CLX_ERR_STREAMINFO_MISSING: return "streaminfo block missing";
    case CLX_ERR_SECOND_VORBIS_COMMENT: return "encountered second Vorbis comment block";
    case CLX_ERR_SECOND_STREAMINFO: return "encountered second streaminfo block";
    case CLX_ERR_STREAMINFO_LENGTH: return "invalid streaminfo metadata block length";
    case CLX_ERR_METADATA_BLOCK_TYPE: return "invalid metadata block type";
    case CLX_ERR_BLOCK_SIZE_BOUNDS: return "inconsistent bounds, min block size > max block size";
    case CLX_ERR_BLOCK_SIZE_LT_16: return "invalid block size, must be at least 16";
    case CLX_ERR_FRAME_SIZE_BOUNDS: return "inconsistent bounds, min frame size > max frame size";
    case CLX_ERR_SAMPLE_RATE_INVALID: return "invalid sample rate";
    case CLX_ERR_VORBIS_TOO_SHORT: return "Vorbis comment block is too short";
    case CLX_ERR_VORBIS_TOO_LARGE: return "Vorbis comment blocks larger than 10 MiB are not supported";
    case CLX_ERR_VENDOR_TOO_LONG: return "vendor string too long";
    case CLX_ERR_VORBIS_TOO_MANY: return "too many entries for Vorbis comment block";
    case CLX_ERR_VORBIS_COMMENT_TOO_LONG: return "Vorbis comment too long for Vorbis comment block";
    case CLX_ERR_VORBIS_NAME_INVALID: return "Vorbis comment field name contains invalid byte";
    case CLX_ERR_VORBIS_NO_EQUALS: return "Vorbis comment does not contain '='";
    case CLX_ERR_VORBIS_EXCESS_DATA: return "Vorbis comment block has excess data";
    case CLX_ERR_VORBIS_WRONG_COUNT: return "Vorbis comment block contains wrong number of entries";
    case CLX_ERR_APPLICATION_TOO_SHORT: return "application block length must be at least 4 bytes";
    case CLX_ERR_APPLICATION_TOO_LARGE: return "application blocks larger than 10 MiB are not supported";
    case CLX_ERR_UTF8_INVALID: return "Vorbis comment or vendor string is not valid UTF-8";
    case CLX_ERR_INVALID_ARGUMENT: return "claxon_b200: invalid argument";
    case CLX_ERR_CUDA: return "claxon_b200: CUDA error";
    case CLX_ERR_NO_DEVICE: return "claxon_b200: no CUDA device / extension not available";
    case CLX_ERR_CONTAINER: return "claxon_b200: malformed or unsupported container";
    default: return "claxon_b200: unknown status";
    }
}

static inline int clx_status_kind_inline(int s) {
    switch (s) {
    case CLX_OK: case CLX_EOF: return CLX_KIND_NONE;
    case CLX_ERR_IO_UNEXPECTED_EOF: return CLX_KIND_IO;
    case CLX_ERR_NO_BPS_IN_HEADER: case CLX_ERR_UNENCODED_BINARY: case CLX_ERR_NEGATIVE_QLP_SHIFT:
    case CLX_ERR_VORBIS_TOO_LARGE: case CLX_ERR_APPLICATION_TOO_LARGE:
        return CLX_KIND_UNSUPPORTED;
    case CLX_ERR_INVALID_ARGUMENT: case CLX_ERR_CUDA: case CLX_ERR_NO_DEVICE: case CLX_ERR_CONTAINER:
        return CLX_KIND_LIBRARY;
    default:
        return (s >= 3 && s < 90) ? CLX_KIND_FORMAT : CLX_KIND_LIBRARY;
    }
}

#ifdef __cplusplus
}
#endif
#endif /* CLX_STATUS_H */
