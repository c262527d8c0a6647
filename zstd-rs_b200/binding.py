"""ctypes binding of libb200zstd.so + Python mirrors of ruzstd's FrameDecoder / StreamingDecoder.

Reference interface mirrored (all paths relative to ruzstd/src/decoding/):
  FrameDecoder            frame_decoder.rs:80-84, 154-627
  BlockDecodingStrategy   frame_decoder.rs:96-100
  StreamingDecoder        streaming_decoder.rs:45-156
Everything here is plumbing over the C ABI; no decoding happens in Python.
"""
import ctypes as C
import io
import os
import re
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libb200zstd.so")
_HEADER = os.path.join(_HERE, "..", "include", "b200zstd.h")

READ_FN = C.CFUNCTYPE(C.c_long, C.c_void_p, C.POINTER(C.c_uint8), C.c_size_t)
WRITE_FN = C.CFUNCTYPE(C.c_long, C.c_void_p, C.POINTER(C.c_uint8), C.c_size_t)
READ_AT_FN = C.CFUNCTYPE(C.c_long, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint8), C.c_size_t)

ALL, UPTO_BLOCKS, UPTO_BYTES = 0, 1, 2
MEM_HOST, MEM_DEVICE = 0, 1
ERR_SKIP_FRAME = 8
ERR_INVALID_ARGUMENT = 220
ERR_SEEKABLE_TABLE, ERR_SEEKABLE_FRAME_SIZE, ERR_SEEKABLE_IO = 240, 241, 242   # EXTENSION: seekable archives
FLAG_CHECKSUM = 1
FLAG_PROFILE = 2
FLAG_DICT_TABLES = 4
FLAG_DICT_LONG = 8   # EXTENSION (B200Z_FLAG_DICT_LONG): long matches into the dictionary's last 2^27 bytes (libzstd's --patch-from)
HUF_DEBUG_BYTES, FSE_DEBUG_BYTES = 3088, 1040   # B200Z_DEBUG_HUF_BYTES / B200Z_DEBUG_FSE_BYTES: one raw huff0 / FSE table
UNCOMPRESSED, FASTEST = 0, 1   # CompressionLevel (ruzstd encoding/mod.rs:24-67); Default / Better / Best are not implemented there
LAZY = 5   # EXTENSION (B200Z_LEVEL_LAZY): a deeper parse with a lazy choice and repeat offsets; not ruzstd's output
OPT = 7    # EXTENSION (B200Z_LEVEL_OPT): a price-based parse over full-window match chains; not ruzstd's output
ULTRA = 10  # EXTENSION (B200Z_LEVEL_ULTRA): OPT's parse with far matches from the frame's whole window (window_log > 17)


class FrameIO(C.Structure):
    _fields_ = [("src_off", C.c_uint64), ("src_size", C.c_uint64), ("out_off", C.c_uint64), ("out_cap", C.c_uint64)]


class FrameResult(C.Structure):
    _fields_ = [("out_size", C.c_uint64), ("bytes_read", C.c_uint64), ("content_size", C.c_uint64), ("window_size", C.c_uint64),
                ("status", C.c_int32), ("stage", C.c_int32), ("blocks_decoded", C.c_uint32), ("error_block", C.c_uint32),
                ("has_checksum", C.c_uint32), ("checksum_from_data", C.c_uint32), ("has_dict_id", C.c_uint32), ("dict_id", C.c_uint32),
                ("has_calculated_checksum", C.c_uint32), ("calculated_checksum", C.c_uint32)]


FRAME_IO_DTYPE = np.dtype([("src_off", "<u8"), ("src_size", "<u8"), ("out_off", "<u8"), ("out_cap", "<u8")])
BLOCK_DESC_DTYPE = np.dtype([("src_off", "<u8"), ("content_size", "<u4"), ("block_type", "<u4"), ("decompressed_size", "<u4"), ("last_block", "<u4"),
                             ("literals_type", "<u4"), ("regenerated_size", "<u4"), ("compressed_size", "<u4"), ("num_streams", "<u4"),
                             ("num_sequences", "<u4"), ("modes", "<u4")])
BLOCK_FRAME_DTYPE = np.dtype([("out_off", "<u8"), ("out_cap", "<u8"), ("window_size", "<u8"), ("dict", "<u8"), ("first_block", "<u4"), ("num_blocks", "<u4")])
BLOCK_STATUS_DTYPE = np.dtype([("status", "<i4"), ("stage", "<i4"), ("out_size", "<u4"), ("reserved", "<u4")])
BLOCK_NOT_REACHED = -1
FRAME_RESULT_DTYPE = np.dtype([("out_size", "<u8"), ("bytes_read", "<u8"), ("content_size", "<u8"), ("window_size", "<u8"),
                               ("status", "<i4"), ("stage", "<i4"), ("blocks_decoded", "<u4"), ("error_block", "<u4"),
                               ("has_checksum", "<u4"), ("checksum_from_data", "<u4"), ("has_dict_id", "<u4"), ("dict_id", "<u4"),
                               ("has_calculated_checksum", "<u4"), ("calculated_checksum", "<u4")])
ALL_RESULT_DTYPE = np.dtype([("written", "<u8"), ("frames", "<u8"), ("skippable_frames", "<u8"), ("error_offset", "<u8"), ("status", "<i4"),
                             ("stage", "<i4"), ("error_frame", "<i4"), ("reserved", "<u4")])
COMPRESS_IO_DTYPE = np.dtype([("src_off", "<u8"), ("src_size", "<u8"), ("dst_off", "<u8"), ("dst_cap", "<u8")])
COMPRESS_RESULT_DTYPE = np.dtype([("dst_size", "<u8"), ("status", "<i4"), ("blocks", "<u4"), ("raw_blocks", "<u4"), ("rle_blocks", "<u4"),
                                  ("has_checksum", "<u4"), ("checksum", "<u4")])
DICT_SEGMENT_DTYPE = np.dtype([("src_off", "<u8"), ("score", "<u8"), ("epoch", "<u4"), ("size", "<u4")])
assert FRAME_IO_DTYPE.itemsize == C.sizeof(FrameIO) and FRAME_RESULT_DTYPE.itemsize == C.sizeof(FrameResult)


def lib_path():
    return _SO


def build(force=False):
    """Compile libb200zstd.so for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    srcs = [os.path.join(_HERE, "csrc", f) for f in os.listdir(os.path.join(_HERE, "csrc"))] + [_HEADER, os.path.join(_HERE, "Makefile")]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
        subprocess.check_call(["make", "-s", "-C", _HERE])
    return _SO


_lib = None


def lib():
    """The loaded library.  Raises if it was not built -- there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        raise RuntimeError(f"{_SO} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)")
    L = C.CDLL(_SO)
    vp, sz, u8p = C.c_void_p, C.c_size_t, C.POINTER(C.c_uint8)
    pp = C.POINTER(vp)
    sig = {
        "b200z_error_name": (C.c_char_p, [C.c_int]),
        "b200z_abi_version": (C.c_int, []),
        "b200z_ctx_create": (C.c_int, [C.c_int, pp]),
        "b200z_ctx_destroy": (None, [vp]),
        "b200z_ctx_last_error_message": (C.c_char_p, [vp]),
        "b200z_ctx_stream": (vp, [vp]),
        "b200z_ctx_kernel_launches": (C.c_uint64, [vp]),
        "b200z_debug_held_bytes": (None, [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
        "b200z_ctx_set_flags": (None, [vp, C.c_uint32]),
        "b200z_ctx_flags": (C.c_uint32, [vp]),
        "b200z_dict_create": (C.c_int, [vp, vp, sz, pp]),
        "b200z_dict_create_raw_content": (C.c_int, [vp, C.c_uint32, vp, sz, pp]),
        "b200z_dict_id": (C.c_uint32, [vp]),
        "b200z_dict_offset_history": (C.c_int, [vp, C.POINTER(C.c_uint32)]),
        "b200z_dict_content_size": (sz, [vp]),
        "b200z_dict_destroy": (None, [vp]),
        "b200z_decode_frames_batch": (C.c_int, [vp, vp, sz, C.c_int, vp, sz, pp, sz, vp, C.c_uint64, vp, sz, C.c_int, vp]),
        "b200z_decode_blocks_batch": (C.c_int, [vp, vp, sz, vp, sz, vp, sz, C.c_int, vp, sz, C.c_int, vp, vp]),
        "b200z_batch_prepare": (C.c_int, [vp, vp, sz, C.c_int, vp, sz, pp, sz, vp, C.c_uint64, pp]),
        "b200z_batch_run": (C.c_int, [vp, vp, sz]),
        "b200z_batch_finish": (C.c_int, [vp, vp]),
        "b200z_batch_run_profile": (C.c_int, [vp, vp, sz, C.POINTER(C.c_float), sz]),
        "b200z_batch_run_timeline": (C.c_int, [vp, vp, sz, C.POINTER(C.c_float), sz]),
        "b200z_num_stages": (C.c_int, []),
        "b200z_stage_kernel_name": (C.c_char_p, [C.c_int]),
        "b200z_batch_info": (C.c_int, [vp, C.POINTER(C.c_uint64)]),
        "b200z_batch_debug_literals": (C.c_int, [vp, C.c_uint32, vp, sz, C.POINTER(sz)]),
        "b200z_batch_debug_sequences": (C.c_int, [vp, C.c_uint32, vp, sz, C.POINTER(sz)]),
        "b200z_batch_debug_block_flags": (C.c_int, [vp, C.c_uint32, C.POINTER(C.c_uint32)]),
        "b200z_batch_debug_sched": (C.c_int, [vp, C.POINTER(C.c_uint32)]),
        "b200z_batch_debug_waves": (C.c_int, [vp, C.POINTER(C.c_uint32)]),
        "b200z_batch_debug_tables": (C.c_int, [vp, C.c_uint32, vp, vp, C.POINTER(C.c_uint32)]),
        "b200z_debug_route_frames": (C.c_int, [vp, vp, sz, C.c_uint32, vp, C.POINTER(sz)]),
        "b200z_debug_fse_order": (C.c_int, [vp, vp, vp, sz, vp, sz, vp, C.POINTER(sz)]),
        "b200z_batch_destroy": (None, [vp]),
        "b200z_decode_all_prepare": (C.c_int, [vp, vp, sz, C.c_int, pp, sz, vp, C.c_uint64, pp]),
        "b200z_decode_all_finish": (C.c_int, [vp, vp, vp]),
        "b200z_decode_all_batch": (C.c_int, [vp, vp, sz, C.c_int, pp, sz, vp, C.c_uint64, vp, sz, C.c_int, vp]),
        "b200z_debug_decode_all_chain": (C.c_int, [vp, sz, C.c_int, vp, sz, C.POINTER(sz)]),
        "b200z_decode_all_stream": (C.c_int, [vp, READ_FN, vp, WRITE_FN, vp, pp, sz, vp, C.c_uint64, vp]),
        "b200z_debug_stream_cut": (C.c_int, [vp, sz, C.c_uint64, vp, sz, C.POINTER(sz), vp]),
        "b200z_frame_decoder_new": (C.c_int, [vp, pp]),
        "b200z_frame_decoder_free": (None, [vp]),
        "b200z_frame_decoder_set_max_window_size": (None, [vp, C.c_uint64]),
        "b200z_frame_decoder_max_window_size": (C.c_uint64, [vp]),
        "b200z_frame_decoder_init": (C.c_int, [vp, READ_FN, vp]),
        "b200z_frame_decoder_reset": (C.c_int, [vp, READ_FN, vp]),
        "b200z_frame_decoder_skip_frame_length": (C.c_uint32, [vp]),
        "b200z_frame_decoder_add_dict": (C.c_int, [vp, vp, sz]),
        "b200z_frame_decoder_add_raw_content_dict": (C.c_int, [vp, C.c_uint32, vp, sz]),
        "b200z_frame_decoder_force_dict": (C.c_int, [vp, C.c_uint32]),
        "b200z_frame_decoder_decode_blocks": (C.c_int, [vp, READ_FN, vp, C.c_int, sz, C.POINTER(C.c_int)]),
        "b200z_frame_decoder_read": (C.c_long, [vp, vp, sz]),
        "b200z_frame_decoder_collect_to_writer": (C.c_long, [vp, WRITE_FN, vp]),
        "b200z_frame_decoder_can_collect": (sz, [vp]),
        "b200z_frame_decoder_is_finished": (C.c_int, [vp]),
        "b200z_frame_decoder_blocks_decoded": (sz, [vp]),
        "b200z_frame_decoder_bytes_read_from_source": (C.c_uint64, [vp]),
        "b200z_frame_decoder_content_size": (C.c_uint64, [vp]),
        "b200z_frame_decoder_get_checksum_from_data": (C.c_int, [vp, C.POINTER(C.c_uint32)]),
        "b200z_frame_decoder_get_calculated_checksum": (C.c_int, [vp, C.POINTER(C.c_uint32)]),
        "b200z_frame_decoder_decode_from_to": (C.c_int, [vp, vp, sz, vp, sz, C.POINTER(sz), C.POINTER(sz)]),
        "b200z_frame_decoder_decode_all": (C.c_int, [vp, vp, sz, vp, sz, C.POINTER(sz)]),
        "b200z_frame_decoder_last_stage": (C.c_int, [vp]),
        "b200z_frame_decoder_last_error_message": (C.c_char_p, [vp]),
        "b200z_streaming_decoder_new": (C.c_int, [vp, READ_FN, vp, pp]),
        "b200z_streaming_decoder_new_with_decoder": (C.c_int, [READ_FN, vp, vp, pp]),
        "b200z_streaming_decoder_new_with_max_window_size": (C.c_int, [vp, READ_FN, vp, C.c_uint64, pp]),
        "b200z_streaming_decoder_read": (C.c_long, [vp, vp, sz, C.POINTER(C.c_int)]),
        "b200z_streaming_decoder_frame_decoder": (vp, [vp]),
        "b200z_streaming_decoder_into_frame_decoder": (vp, [vp]),
        "b200z_streaming_decoder_free": (None, [vp]),
        "b200z_xxh64": (C.c_uint64, [vp, sz]),
        "b200z_compress_bound": (sz, [sz]),
        "b200z_compress_frames_batch": (C.c_int, [vp, vp, sz, C.c_int, vp, sz, C.c_int, C.c_int, vp, sz, C.c_int, vp]),
        "b200z_compress_frames_batch_dict": (C.c_int, [vp, vp, sz, C.c_int, vp, sz, C.c_int, C.c_int, vp, vp, sz, C.c_int, vp]),
        "b200z_compress_bound_dict": (sz, [sz, vp]),
        "b200z_compress_frames_batch_long": (C.c_int, [vp, vp, sz, C.c_int, vp, sz, C.c_int, C.c_int, vp, C.c_int, vp, sz, C.c_int, vp]),
        "b200z_compress_num_stages": (C.c_int, []),
        "b200z_compress_stage_name": (C.c_char_p, [C.c_int]),
        "b200z_compress_last_profile": (C.c_int, [vp, C.POINTER(C.c_float), sz]),
        "b200z_frame_compressor_new": (C.c_int, [vp, C.c_int, C.c_int, pp]),
        "b200z_frame_compressor_free": (None, [vp]),
        "b200z_frame_compressor_set_compression_level": (C.c_int, [vp, C.c_int]),
        "b200z_frame_compressor_compression_level": (C.c_int, [vp]),
        "b200z_frame_compressor_set_window_log": (C.c_int, [vp, C.c_int]),
        "b200z_frame_compressor_window_log": (C.c_int, [vp]),
        "b200z_frame_compressor_compress": (C.c_int, [vp, READ_FN, vp, WRITE_FN, vp, vp]),
        "b200z_dict_train_raw": (C.c_int, [vp, vp, sz, C.c_int, vp, sz, sz, sz, vp, sz, C.POINTER(sz), vp, sz, C.POINTER(sz)]),
        "b200z_dict_finalize": (C.c_int, [vp, vp, sz, vp, sz, C.c_int, vp, sz, C.c_uint32, vp, sz, C.POINTER(sz)]),
        "b200z_debug_dict_from_counts": (C.c_int, [vp, vp, sz, C.c_uint32, vp, sz, C.POINTER(sz)]),
        "b200z_seekable_bound": (sz, [sz, sz, C.c_int, vp]),
        "b200z_compress_seekable": (C.c_int, [vp, vp, sz, C.c_int, sz, C.c_int, C.c_int, vp, vp, sz, C.c_int, C.POINTER(sz)]),
        "b200z_compress_seekable_stream": (C.c_int, [vp, READ_FN, vp, WRITE_FN, vp, sz, C.c_int, C.c_int, vp, vp]),
        "b200z_seekable_open": (C.c_int, [vp, vp, sz, C.c_int, pp]),
        "b200z_seekable_open_source": (C.c_int, [vp, READ_AT_FN, vp, C.c_uint64, pp]),
        "b200z_seekable_num_frames": (C.c_uint64, [vp]),
        "b200z_seekable_content_size": (C.c_uint64, [vp]),
        "b200z_seekable_frame": (C.c_int, [vp, C.c_uint64, vp]),
        "b200z_seekable_close": (None, [vp]),
        "b200z_seekable_read_ranges": (C.c_int, [vp, vp, sz, pp, sz, vp, C.c_uint64, vp, sz, C.c_int, vp]),
        "b200z_debug_seekable_plan": (C.c_int, [vp, sz, vp, sz, vp, sz, C.POINTER(sz), vp, sz, C.POINTER(sz), C.POINTER(C.c_uint64)]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)          # AttributeError here == a symbol the header declares is not exported
        fn.restype = res
        fn.argtypes = args
    L._declared = sorted(sig)
    _lib = L
    return L


def declared_symbols():
    """Every function include/b200zstd.h declares (parsed from the header)."""
    txt = open(_HEADER).read()
    return sorted(set(re.findall(r"\b(b200z_[a-z0-9_]+)\s*\(", txt)))


def error_names():
    txt = open(_HEADER).read()
    return {int(v): k for k, v in re.findall(r"(B200Z_(?:OK|ERR_[A-Z0-9_]+))\s*=\s*(\d+)", txt)}


class B200ZError(Exception):
    """Mirror of ruzstd's FrameDecoderError: .code is the leaf variant, .stage the nesting path."""

    def __init__(self, code, stage=0, msg=""):
        self.code, self.stage = code, stage
        super().__init__(f"{lib().b200z_error_name(code).decode()} (stage {stage}) {msg}")


def held_bytes():
    """b200z_debug_held_bytes: (device bytes, pinned host bytes) the library's allocations hold now, over the whole process."""
    d, p = C.c_uint64(), C.c_uint64()
    lib().b200z_debug_held_bytes(C.byref(d), C.byref(p))
    return d.value, p.value


def xxh64(data):
    b = bytes(data)
    return lib().b200z_xxh64(b, len(b))


def route_frames(work, eligible, sms=132):
    """Host-only: the frames k_exec_cta would take (largest first) -- route_exec_frames, csrc/plan.cpp."""
    w = np.ascontiguousarray(work, dtype=np.uint64)
    el = np.ascontiguousarray(eligible, dtype=np.uint8)
    out = np.zeros(max(len(w), 1), dtype=np.uint32)
    n = C.c_size_t()
    rc = lib().b200z_debug_route_frames(w.ctypes.data, el.ctypes.data, len(w), sms, out.ctypes.data, C.byref(n))
    if rc:
        raise B200ZError(rc, 0, "b200z_debug_route_frames")
    return out[:n.value].copy()


def fse_order(first_block, nblocks, on_cta, nseq):
    """Host-only: the order in which k_fse takes the blocks (empty = descriptor order) -- build_fse_order, csrc/plan.cpp."""
    fb = np.ascontiguousarray(first_block, dtype=np.uint32)
    nb = np.ascontiguousarray(nblocks, dtype=np.uint32)
    oc = np.ascontiguousarray(on_cta, dtype=np.uint8)
    ns = np.ascontiguousarray(nseq, dtype=np.uint32)
    out = np.zeros(max(len(ns), 1), dtype=np.uint32)
    n = C.c_size_t()
    rc = lib().b200z_debug_fse_order(fb.ctypes.data, nb.ctypes.data, oc.ctypes.data, len(fb), ns.ctypes.data, len(ns), out.ctypes.data, C.byref(n))
    if rc:
        raise B200ZError(rc, 0, "b200z_debug_fse_order")
    return out[:n.value].copy()


def _ptr(x):
    """(address, nbytes, keepalive) of bytes / numpy / torch tensor (host or device)."""
    if x is None:
        return None, 0, None
    if isinstance(x, (bytes, bytearray)):
        a = np.frombuffer(x, dtype=np.uint8)
        return a.ctypes.data, a.nbytes, a
    if isinstance(x, np.ndarray):
        a = np.ascontiguousarray(x)
        return a.ctypes.data, a.nbytes, a
    if hasattr(x, "data_ptr"):  # torch tensor
        return x.data_ptr(), x.numel() * x.element_size(), x
    raise TypeError(type(x))


def _is_device(x):
    return hasattr(x, "is_cuda") and x.is_cuda


class Context:
    """One per GPU: pins the device, owns the stream (b200z_ctx)."""

    def __init__(self, device=0):
        self.L = lib()
        h = C.c_void_p()
        e = self.L.b200z_ctx_create(device, C.byref(h))
        if e:
            raise B200ZError(e, 0, "b200z_ctx_create: no usable CUDA device; this library has no CPU path")
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.L.b200z_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def stream(self):
        return self.L.b200z_ctx_stream(self.h)

    def kernel_launches(self):
        return self.L.b200z_ctx_kernel_launches(self.h)

    def set_flags(self, flags):
        """FLAG_CHECKSUM = 1: the batch entry also computes each frame's XXH64 content checksum on the GPU."""
        self.L.b200z_ctx_set_flags(self.h, flags)

    def _chk(self, e):
        if e:
            raise B200ZError(e, 0, self.L.b200z_ctx_last_error_message(self.h).decode())


class Dictionary:
    """Mirror of ruzstd::decoding::Dictionary (dictionary.rs:12-37); decode_dict == Dictionary.decode_dict."""

    def __init__(self, ctx, handle):
        self.ctx, self.h = ctx, handle

    @classmethod
    def decode_dict(cls, ctx, raw):
        h = C.c_void_p()
        b = bytes(raw)
        e = ctx.L.b200z_dict_create(ctx.h, b, len(b), C.byref(h))
        if e:
            raise B200ZError(e, 8)
        return cls(ctx, h)

    @classmethod
    def raw_content(cls, ctx, dict_id, content):
        h = C.c_void_p()
        b = bytes(content)
        ctx._chk(ctx.L.b200z_dict_create_raw_content(ctx.h, dict_id, b, len(b), C.byref(h)))
        return cls(ctx, h)

    @property
    def id(self):
        return self.ctx.L.b200z_dict_id(self.h)

    @property
    def offset_hist(self):
        a = (C.c_uint32 * 3)()
        self.ctx.L.b200z_dict_offset_history(self.h, a)
        return list(a)

    @property
    def content_size(self):
        return self.ctx.L.b200z_dict_content_size(self.h)

    def __del__(self):
        try:
            if self.h and self.ctx.h:
                self.ctx.L.b200z_dict_destroy(self.h)
        except Exception:
            pass


def _frames_array(frames):
    a = np.ascontiguousarray(frames, dtype=FRAME_IO_DTYPE) if not (isinstance(frames, np.ndarray) and frames.dtype == FRAME_IO_DTYPE) else np.ascontiguousarray(frames)
    return a


def _dict_args(dicts, forced):
    dicts = list(dicts or [])
    arr = (C.c_void_p * max(len(dicts), 1))(*[d.h for d in dicts])
    return arr, len(dicts), (forced.h if forced is not None else None)


def decode_blocks(ctx, blocks, frames, compressed, output):
    """b200z_decode_blocks_batch: the block-level entry (what replaces BlockDecoder::decompress_block, block_decoder.rs:97-197).
    blocks: BLOCK_DESC_DTYPE array, frames: BLOCK_FRAME_DTYPE array ('dict' = Dictionary or 0 per frame via `set_frame_dicts`).
    Returns (block status array, per-frame output sizes)."""
    blocks = np.ascontiguousarray(blocks, dtype=BLOCK_DESC_DTYPE)
    frames = np.ascontiguousarray(frames, dtype=BLOCK_FRAME_DTYPE)
    st = np.zeros(len(blocks), dtype=BLOCK_STATUS_DTYPE)
    fo = np.zeros(len(frames), dtype=np.uint64)
    ip, il, _k1 = _ptr(compressed)
    op, ol, _k2 = _ptr(output)
    e = ctx.L.b200z_decode_blocks_batch(ctx.h, blocks.ctypes.data, len(blocks), frames.ctypes.data, len(frames), ip, il,
                                        MEM_DEVICE if _is_device(compressed) else MEM_HOST, op, ol, MEM_DEVICE if _is_device(output) else MEM_HOST,
                                        st.ctypes.data, fo.ctypes.data)
    ctx._chk(e)
    return st, fo


def decode_frames(ctx, input, frames, output, dicts=None, forced_dict=None, max_window_size=0):
    """b200z_decode_frames_batch: one-shot batch decode.  input/output: bytes, numpy or torch (host or cuda)."""
    fr = _frames_array(frames)
    res = np.zeros(len(fr), dtype=FRAME_RESULT_DTYPE)
    ip, il, _k1 = _ptr(input)
    op, ol, _k2 = _ptr(output)
    darr, nd, forced = _dict_args(dicts, forced_dict)
    e = ctx.L.b200z_decode_frames_batch(ctx.h, ip, il, MEM_DEVICE if _is_device(input) else MEM_HOST, fr.ctypes.data, len(fr),
                                        darr, nd, forced, max_window_size, op, ol, MEM_DEVICE if _is_device(output) else MEM_HOST,
                                        res.ctypes.data)
    ctx._chk(e)
    return res


def _summary(a):
    return {k: int(a[0][k]) for k in ALL_RESULT_DTYPE.names if k != "reserved"}


def decode_all(ctx, input, output, dicts=None, forced_dict=None, max_window_size=0):
    """b200z_decode_all_prepare / b200z_batch_run / b200z_decode_all_finish: FrameDecoder::decode_all (frame_decoder.rs:541-577) of a
    buffer of concatenated zstd and skippable frames in one GPU submission, the plaintexts back to back at the start of `output`.
    input/output: bytes, numpy or torch (host or cuda).  `forced_dict` (a Dictionary) is an extension: it is applied to every frame.
    Returns (summary dict: written, frames, skippable_frames, error_offset, status, stage, error_frame; FRAME_RESULT_DTYPE rows, one
    per zstd frame of the chain).  Errors are reported in the summary, not raised."""
    b = AllBatch(ctx, input, dicts, forced_dict, max_window_size)
    try:
        if _is_device(output):
            b.run(output)
        else:
            import torch
            op, ol, _k = _ptr(output)
            dev = torch.empty(ol + 16, dtype=torch.uint8, device=f"cuda:{ctx.device}")
            b.run(dev[:ol])
            summary, res = b.finish()
            if summary["written"]:
                host = dev[:summary["written"]].cpu().numpy()   # kept alive until the copy is done
                C.memmove(op, host.ctypes.data, summary["written"])
            return summary, res
        return b.finish()
    finally:
        b.close()


class AllBatch:
    """Prepared decode_all submission (b200z_decode_all_prepare): the frames of `input` found and planned; run() decodes them into a
    device buffer, back to back by decoded size; finish() gives (summary dict, FRAME_RESULT_DTYPE rows).  Mirrors Batch."""

    def __init__(self, ctx, input, dicts=None, forced_dict=None, max_window_size=0):
        self.ctx = ctx
        ip, il, self._k = _ptr(input)
        darr, nd, forced = _dict_args(dicts, forced_dict)
        self._dicts = (dicts, forced_dict)
        h = C.c_void_p()
        ctx._chk(ctx.L.b200z_decode_all_prepare(ctx.h, ip, il, MEM_DEVICE if _is_device(input) else MEM_HOST, darr, nd, forced, max_window_size,
                                                C.byref(h)))
        self.h = h

    def run(self, d_output):
        op, ol, _k = _ptr(d_output)
        assert _is_device(d_output), "AllBatch.run writes into device memory"
        self.ctx._chk(self.ctx.L.b200z_batch_run(self.h, op, ol))

    def finish(self):
        res = np.zeros(self.info()["frames"], dtype=FRAME_RESULT_DTYPE)
        s = np.zeros(1, dtype=ALL_RESULT_DTYPE)
        self.ctx._chk(self.ctx.L.b200z_decode_all_finish(self.h, s.ctypes.data, res.ctypes.data))
        return _summary(s), res

    def info(self):
        """As Batch.info; "frames" is the number of zstd frames found."""
        a = (C.c_uint64 * 8)()
        self.ctx.L.b200z_batch_info(self.h, a)
        k = ["frames", "blocks", "compressed_blocks", "planned_bytes", "literal_scratch_bytes", "sequences", "launches_per_run"]
        return dict(zip(k, list(a)))

    def close(self):
        if getattr(self, "h", None) and self.ctx.h:
            self.ctx.L.b200z_batch_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def decode_all_batch(ctx, input, output, dicts=None, forced_dict=None, max_window_size=0):
    """b200z_decode_all_batch, the one-shot form of decode_all: returns the summary dict only."""
    ip, il, _k1 = _ptr(input)
    op, ol, _k2 = _ptr(output)
    darr, nd, forced = _dict_args(dicts, forced_dict)
    s = np.zeros(1, dtype=ALL_RESULT_DTYPE)
    ctx._chk(ctx.L.b200z_decode_all_batch(ctx.h, ip, il, MEM_DEVICE if _is_device(input) else MEM_HOST, darr, nd, forced, max_window_size, op, ol,
                                          MEM_DEVICE if _is_device(output) else MEM_HOST, s.ctypes.data))
    return _summary(s)


def decode_all_chain(data, by_candidates=False):
    """Host-only: the input offsets of the frames decode_all visits -- the host-input walk, or (by_candidates) the device-input
    selection through every magic-number candidate, with the scan and the walks done on the host."""
    b = np.frombuffer(bytes(data), dtype=np.uint8)
    n = C.c_size_t()
    cap = len(b) // 4 + 2
    out = np.zeros(cap, dtype=np.uint64)
    rc = lib().b200z_debug_decode_all_chain(b.ctypes.data if len(b) else None, len(b), 1 if by_candidates else 0, out.ctypes.data, cap, C.byref(n))
    if rc:
        raise B200ZError(rc, 0, "b200z_debug_decode_all_chain")
    return [int(x) for x in out[:n.value]]


STREAM_RESULT_DTYPE = np.dtype([("all", ALL_RESULT_DTYPE), ("delivered", "<u8"), ("submissions", "<u8"), ("checksum_frames", "<u8"),
                                ("checksum_mismatches", "<u8"), ("first_mismatch_frame", "<i8")])
STREAM_CUT_DTYPE = np.dtype([("start", "<u8"), ("end", "<u8"), ("in_bytes", "<u8"), ("out_bound", "<u8"), ("nblocks", "<u8"), ("nseq", "<u8"),
                             ("nframes", "<u4"), ("flags", "<u4")])
STREAM_CUT_END_DTYPE = np.dtype([("error_offset", "<u8"), ("skippable_frames", "<u8"), ("peak_buffered", "<u8"), ("status", "<i4"), ("stage", "<i4"),
                                 ("error_frame", "<i4"), ("reserved", "<u4")])


def decode_all_stream(ctx, source, drain, dicts=None, forced_dict=None, max_window_size=0):
    """b200z_decode_all_stream: FrameDecoder::decode_all of everything `source` holds (bytes, or an object with read(n)) to `drain` (an
    object with write(b), or a bytearray, which the plaintext is appended to), chunk by chunk through the GPU in bounded memory
    (B200Z_PIPELINE_CHUNK_BYTES per chunk).  Returns a dict: the decode_all summary (written, frames, skippable_frames, error_offset,
    status, stage, error_frame) and delivered, submissions, checksum_frames, checksum_mismatches, first_mismatch_frame.  Errors in the
    stream, a source that raises (it ends the source) and a drain that raises or returns 0 (FAILED_TO_DRAIN_DECODEBUFFER) are reported
    in the dict, not raised."""
    src = _Reader(source).src

    def _read(_user, buf, n):
        try:
            b = src.read(n)
            if b:
                C.memmove(buf, b, len(b))
            return len(b)
        except Exception:
            return -1

    def _write(_user, buf, n):
        try:
            if isinstance(drain, bytearray):
                drain.extend(C.string_at(buf, n))
                return n
            r = drain.write(C.string_at(buf, n))
            return n if r is None else r
        except Exception:
            return -1

    rd, wr = READ_FN(_read), WRITE_FN(_write)
    darr, nd, forced = _dict_args(dicts, forced_dict)
    res = np.zeros(1, dtype=STREAM_RESULT_DTYPE)
    ctx._chk(ctx.L.b200z_decode_all_stream(ctx.h, rd, None, wr, None, darr, nd, forced, max_window_size, res.ctypes.data))
    out = _summary(res["all"])
    out.update({k: int(res[0][k]) for k in STREAM_RESULT_DTYPE.names if k != "all"})
    return out


def stream_cut(data, chunk):
    """Host-only: how decode_all_stream cuts `data` at chunk size `chunk` -- (STREAM_CUT_DTYPE rows, one per submission; the end
    record as a dict: error_offset, skippable_frames, peak_buffered, status, stage, error_frame)."""
    b = np.frombuffer(bytes(data), dtype=np.uint8)
    n = C.c_size_t()
    end = np.zeros(1, dtype=STREAM_CUT_END_DTYPE)
    cap = 64
    while True:
        cuts = np.zeros(cap, dtype=STREAM_CUT_DTYPE)
        rc = lib().b200z_debug_stream_cut(b.ctypes.data if len(b) else None, len(b), chunk, cuts.ctypes.data, cap, C.byref(n), end.ctypes.data)
        if rc:
            raise B200ZError(rc, 0, "b200z_debug_stream_cut")
        if n.value <= cap:
            return cuts[:n.value], {k: int(end[0][k]) for k in STREAM_CUT_END_DTYPE.names if k != "reserved"}
        cap = n.value


WINDOW_LOG_MIN, WINDOW_LOG_MAX = 17, 27   # B200Z_WINDOW_LOG_MIN / _MAX


def compress_bound(n, dict=None):
    """b200z_compress_bound (b200z_compress_bound_dict with a Dictionary): the largest frame compress_frames can write for n input
    bytes."""
    return lib().b200z_compress_bound(n) if dict is None else lib().b200z_compress_bound_dict(n, dict.h)


def compress_frames(ctx, input, io, output, level=FASTEST, checksum=True, dict=None, dict_tables=False, window_log=WINDOW_LOG_MIN,
                    dict_long=False):
    """b200z_compress_frames_batch_long: one zstd frame per COMPRESS_IO_DTYPE row (src_off, src_size, dst_off, dst_cap), every block
    of every frame compressed at once, against `dict` (a Dictionary of this context) when given.  dict_tables=True sets
    FLAG_DICT_TABLES for the call: a formatted dictionary's entropy tables may then code each frame's first block.  window_log in
    [17, 27]: above 17, frames larger than 128 KiB also take long-distance matches up to 2^window_log bytes back (17 is
    b200z_compress_frames_batch_dict's output).  dict_long=True sets FLAG_DICT_LONG for the call: with `dict` and window_log > 17
    the long matches of every frame also reach into the dictionary's last 2^27 bytes, and each frame's window covers the
    dictionary (compress_patch_from).  input/output: bytes, numpy or torch (host or cuda).  Returns COMPRESS_RESULT_DTYPE rows."""
    fr = np.ascontiguousarray(io, dtype=COMPRESS_IO_DTYPE)
    res = np.zeros(len(fr), dtype=COMPRESS_RESULT_DTYPE)
    ip, il, _k1 = _ptr(input)
    op, ol, _k2 = _ptr(output)
    flags = ctx.L.b200z_ctx_flags(ctx.h)
    if dict_tables or dict_long:
        ctx.L.b200z_ctx_set_flags(ctx.h, flags | (FLAG_DICT_TABLES if dict_tables else 0) | (FLAG_DICT_LONG if dict_long else 0))
    try:
        e = ctx.L.b200z_compress_frames_batch_long(ctx.h, ip, il, MEM_DEVICE if _is_device(input) else MEM_HOST, fr.ctypes.data, len(fr),
                                                   level, 1 if checksum else 0, dict.h if dict is not None else None, window_log, op, ol,
                                                   MEM_DEVICE if _is_device(output) else MEM_HOST, res.ctypes.data)
    finally:
        ctx.L.b200z_ctx_set_flags(ctx.h, flags)
    ctx._chk(e)
    return res


def compress_to_vec(ctx, data, level=FASTEST, checksum=True, dict=None, dict_tables=False, window_log=WINDOW_LOG_MIN, dict_long=False):
    """Mirror of ruzstd::encoding::compress_to_vec (encoding/mod.rs): one frame holding `data`, as bytes (against `dict` when given,
    with its entropy tables when dict_tables=True; long-distance matches up to 2^window_log back, into the dictionary too when
    dict_long=True, see compress_frames)."""
    src = bytes(data)
    cap = compress_bound(len(src), dict)
    out = np.zeros(cap, dtype=np.uint8)
    io = np.array([(0, len(src), 0, cap)], dtype=COMPRESS_IO_DTYPE)
    res = compress_frames(ctx, src, io, out, level, checksum, dict, dict_tables, window_log, dict_long)
    return out[:int(res[0]["dst_size"])].tobytes()


def patch_window_log(reference_size, data_size):
    """The window_log compress_patch_from uses: min(27, max(17, ceil(log2(reference_size + data_size))))."""
    return min(WINDOW_LOG_MAX, max(WINDOW_LOG_MIN, (reference_size + data_size - 1).bit_length()))


def compress_patch_from(ctx, reference, data, level=FASTEST, checksum=True):
    """What `zstd --patch-from=reference` does: one frame of `data` compressed against `reference` as a raw-content dictionary, with
    long-distance matches into all of it (the last 2^27 bytes of a larger one) at window_log patch_window_log(len(reference),
    len(data)), as bytes.  The frame carries no dictionary ID, so it is decoded with the reference forced and a window limit of at
    least the frame's window (2^window_log):

        R = Dictionary.raw_content(ctx, 0, reference)
        decode_frames(ctx, frame, io, out, forced_dict=R, max_window_size=1 << 27)      # or decode_all(..., forced_dict=R, ...)
        d = FrameDecoder(ctx); d.add_raw_content_dict(1, reference); d.force_dict(1); d.set_max_window_size(1 << 27)
        d.decode_all(frame, len(data))

    libzstd decodes the same frame with ZSTD_decompress_usingDict (the reference as raw content) or ZSTD_DCtx_refPrefix, with
    ZSTD_d_windowLogMax at least the frame's window_log."""
    ref = bytes(reference)
    D = Dictionary.raw_content(ctx, 0, ref)
    try:
        return compress_to_vec(ctx, data, level, checksum, D, window_log=patch_window_log(len(ref), len(data)), dict_long=True)
    finally:
        del D


# ---- seekable archives (EXTENSION: zstd's seekable format; include/b200zstd.h, DESIGN.md section 4.10)
SEEKABLE_GROUP_BLOCKS = 2048   # B200Z_SEEKABLE_GROUP_BLOCKS
SEEKABLE_MAX_FRAME_SIZE = 1 << 30
SEEK_FRAME_DTYPE = np.dtype([("c_off", "<u8"), ("c_size", "<u8"), ("d_off", "<u8"), ("d_size", "<u8"), ("has_checksum", "<u4"),
                             ("checksum", "<u4")])
RANGE_DTYPE = np.dtype([("offset", "<u8"), ("length", "<u8"), ("out_off", "<u8")])
RANGE_RESULT_DTYPE = np.dtype([("status", "<i4"), ("stage", "<i4"), ("error_frame", "<i8"), ("frames", "<u8"), ("checksum_mismatches", "<u8")])
SEEK_PLAN_FRAME_DTYPE = np.dtype([("frame", "<u8"), ("dst_off", "<u8"), ("range", "<i8")])
SEEK_PLAN_PIECE_DTYPE = np.dtype([("dst_off", "<u8"), ("src_off", "<u8"), ("len", "<u8"), ("from_scratch", "<u4"), ("range", "<u4")])


def seekable_bound(n, frame_size=131072, checksum=True, dict=None):
    """b200z_seekable_bound: the largest archive compress_seekable can write for n input bytes (0 for a frame_size out of range)."""
    return lib().b200z_seekable_bound(n, frame_size, 1 if checksum else 0, dict.h if dict is not None else None)


def compress_seekable(ctx, input, output=None, frame_size=131072, level=FASTEST, checksum=True, dict=None, dict_tables=False):
    """b200z_compress_seekable: a seekable archive of `input` -- frames of frame_size bytes, each what compress_frames writes for that
    piece, back to back, then the seek table.  input/output: bytes, numpy or torch (host or cuda).  Returns the archive (bytes for a
    host input, a uint8 CUDA tensor for a device one) when output is None, else the archive's size in bytes."""
    ip, il, _k1 = _ptr(input)
    ret = output is None
    if ret:
        cap = max(seekable_bound(il, frame_size, checksum, dict), 1)
        if _is_device(input):
            import torch
            output = torch.empty(cap, dtype=torch.uint8, device=input.device)
        else:
            output = np.empty(cap, dtype=np.uint8)
    op, ol, _k2 = _ptr(output)
    written = C.c_size_t()
    flags = ctx.L.b200z_ctx_flags(ctx.h)
    if dict_tables:
        ctx.L.b200z_ctx_set_flags(ctx.h, flags | FLAG_DICT_TABLES)
    try:
        e = ctx.L.b200z_compress_seekable(ctx.h, ip, il, MEM_DEVICE if _is_device(input) else MEM_HOST, frame_size, level, 1 if checksum else 0,
                                          dict.h if dict is not None else None, op, ol, MEM_DEVICE if _is_device(output) else MEM_HOST,
                                          C.byref(written))
    finally:
        ctx.L.b200z_ctx_set_flags(ctx.h, flags)
    ctx._chk(e)
    if not ret:
        return written.value
    return output[:written.value] if _is_device(output) else output[:written.value].tobytes()


SEEKABLE_STREAM_RESULT_DTYPE = np.dtype([("read", "<u8"), ("written", "<u8"), ("frames", "<u8"), ("groups", "<u8")])


def compress_seekable_stream(ctx, source, drain, frame_size=131072, level=FASTEST, checksum=True, dict=None, dict_tables=False):
    """b200z_compress_seekable_stream: the archive compress_seekable writes for everything `source` holds, from the source to `drain`
    in groups of whole frames (B200Z_PIPELINE_CHUNK_BYTES each), in bounded memory.  Sources and drains as FrameCompressor takes them.
    Returns the SEEKABLE_STREAM_RESULT_DTYPE row (read, written, frames, groups).  A source or drain that fails raises
    B200ZError(ERR_SEEKABLE_IO), from the exception it raised."""
    rd, wr, failure = _source_drain_callbacks(source, drain)
    res = np.zeros(1, dtype=SEEKABLE_STREAM_RESULT_DTYPE)
    flags = ctx.L.b200z_ctx_flags(ctx.h)
    if dict_tables:
        ctx.L.b200z_ctx_set_flags(ctx.h, flags | FLAG_DICT_TABLES)
    try:
        e = ctx.L.b200z_compress_seekable_stream(ctx.h, rd, None, wr, None, frame_size, level, 1 if checksum else 0,
                                                 dict.h if dict is not None else None, res.ctypes.data)
    finally:
        ctx.L.b200z_ctx_set_flags(ctx.h, flags)
    _raise_chained(ctx, e, failure)
    return res[0]


def _ranges_array(ranges):
    if isinstance(ranges, np.ndarray) and ranges.dtype == RANGE_DTYPE:
        return np.ascontiguousarray(ranges)
    return np.array([tuple(r) for r in ranges], dtype=RANGE_DTYPE) if len(ranges) else np.zeros(0, dtype=RANGE_DTYPE)


class SeekableArchive:
    """An open seekable archive (b200z_seekable_open): its table, parsed and checked.  It borrows `archive` (bytes, numpy or torch, host
    or cuda) and keeps a reference to it.  .num_frames, .content_size, .frames (SEEK_FRAME_DTYPE rows), .read(offset, length) and
    .read_ranges(ranges, output).  A context manager; close() releases the handle."""

    def __init__(self, ctx, archive):
        self.ctx = ctx
        self.h = None
        self._file = None
        self._failure = []
        ap, al, self._k = _ptr(archive)
        self._archive = archive
        h = C.c_void_p()
        ctx._chk(ctx.L.b200z_seekable_open(ctx.h, ap, al, MEM_DEVICE if _is_device(archive) else MEM_HOST, C.byref(h)))
        self.h = h

    @classmethod
    def from_source(cls, ctx, f, length=None):
        """An archive behind a positional-read callback (b200z_seekable_open_source): `f` is a path or a binary file object, read with
        os.pread on its descriptor when it has one, else with seek() and read().  length: the archive's size, by default the file's.
        Only the footer and the table are read here, and only the touched frames by read_ranges.  A failed or short read raises
        B200ZError(ERR_SEEKABLE_IO), from the exception the file raised if any."""
        self = cls.__new__(cls)
        self.ctx, self.h, self._k, self._archive, self._failure = ctx, None, None, None, []
        self._file = open(f, "rb") if isinstance(f, (str, os.PathLike)) else None
        src = self._file if self._file is not None else f
        try:
            fd = src.fileno()
        except (AttributeError, OSError, io.UnsupportedOperation):
            fd = None
        if length is None:
            length = os.fstat(fd).st_size if fd is not None else src.seek(0, io.SEEK_END)

        def _read_at(_user, offset, buf, n):
            try:
                if fd is not None:
                    b = os.pread(fd, n, offset)
                else:
                    src.seek(offset)
                    b = src.read(n)
                if b:
                    C.memmove(buf, b, len(b))
                return len(b)
            except Exception as e:
                failure.append(e)
                return -1

        failure = self._failure
        self._read_at = READ_AT_FN(_read_at)
        h = C.c_void_p()
        try:
            self._chk(ctx.L.b200z_seekable_open_source(ctx.h, self._read_at, None, length, C.byref(h)))
        except BaseException:
            self.close()
            raise
        self.h = h
        return self

    def _chk(self, e):
        failure = list(self._failure)
        self._failure.clear()
        _raise_chained(self.ctx, e, failure)

    @property
    def num_frames(self):
        return self.ctx.L.b200z_seekable_num_frames(self.h)

    @property
    def content_size(self):
        return self.ctx.L.b200z_seekable_content_size(self.h)

    @property
    def frames(self):
        out = np.zeros(self.num_frames, dtype=SEEK_FRAME_DTYPE)
        for i in range(len(out)):
            self.ctx._chk(self.ctx.L.b200z_seekable_frame(self.h, i, out[i:].ctypes.data))
        return out

    def read_ranges(self, ranges, output, dicts=None, forced_dict=None, max_window_size=0):
        """b200z_seekable_read_ranges: RANGE_DTYPE rows (or (offset, length, out_off) tuples) into `output` (numpy or torch, host or
        cuda).  Returns RANGE_RESULT_DTYPE rows; a range that could not be read is reported there, not raised."""
        rg = _ranges_array(ranges)
        res = np.zeros(len(rg), dtype=RANGE_RESULT_DTYPE)
        op, ol, _k = _ptr(output)
        darr, nd, forced = _dict_args(dicts, forced_dict)
        self._chk(self.ctx.L.b200z_seekable_read_ranges(self.h, rg.ctypes.data, len(rg), darr, nd, forced, max_window_size, op, ol,
                                                        MEM_DEVICE if _is_device(output) else MEM_HOST, res.ctypes.data))
        return res

    def read(self, offset, length, dicts=None, forced_dict=None):
        """Plaintext [offset, offset + length) as bytes; raises B200ZError when a frame it needs fails."""
        out = np.zeros(max(length, 1), dtype=np.uint8)
        r = self.read_ranges([(offset, length, 0)], out, dicts, forced_dict)
        if r[0]["status"]:
            raise B200ZError(int(r[0]["status"]), int(r[0]["stage"]), f"frame {int(r[0]['error_frame'])}")
        return out[:length].tobytes()

    def close(self):
        if getattr(self, "h", None) and self.ctx.h:
            self.ctx.L.b200z_seekable_close(self.h)
        self.h = None
        if getattr(self, "_file", None) is not None:
            self._file.close()
            self._file = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def seekable_plan(archive, ranges):
    """Host-only: the read plan b200z_seekable_read_ranges follows for `ranges` on the host archive -- (SEEK_PLAN_FRAME_DTYPE rows,
    SEEK_PLAN_PIECE_DTYPE rows, scratch bytes).  Raises B200ZError for a corrupt table or invalid ranges."""
    a = np.frombuffer(bytes(archive), dtype=np.uint8)
    rg = _ranges_array(ranges)
    nf, npc, scr = C.c_size_t(), C.c_size_t(), C.c_uint64()
    fcap, pcap = 16, 16
    while True:
        fr = np.zeros(fcap, dtype=SEEK_PLAN_FRAME_DTYPE)
        pc = np.zeros(pcap, dtype=SEEK_PLAN_PIECE_DTYPE)
        rc = lib().b200z_debug_seekable_plan(a.ctypes.data if len(a) else None, len(a), rg.ctypes.data if len(rg) else None, len(rg), fr.ctypes.data,
                                             fcap, C.byref(nf), pc.ctypes.data, pcap, C.byref(npc), C.byref(scr))
        if rc == 0:
            return fr[:nf.value], pc[:npc.value], scr.value
        if rc == ERR_INVALID_ARGUMENT and (nf.value > fcap or npc.value > pcap):
            fcap, pcap = max(fcap, nf.value), max(pcap, npc.value)
            continue
        raise B200ZError(rc, 0, "b200z_debug_seekable_plan")


class FrameCompressor:
    """GPU-backed mirror of ruzstd::encoding::FrameCompressor (frame_compressor.rs:75-276): compress() reads the source to its end
    and writes one frame to the drain, chunk by chunk, in memory bounded by the chunk size (b200z_frame_compressor, see
    include/b200zstd.h).  Sources: bytes or file-likes with read(); drains: file-likes with write(), or a bytearray, which the
    frame is appended to.  An exception raised by the source or the drain fails the call as the reference's unwrap() would,
    with B200ZError(REFERENCE_WOULD_PANIC) raised from it."""

    def __init__(self, ctx, level=FASTEST, checksum=True, window_log=WINDOW_LOG_MIN):
        self.ctx, self.L = ctx, ctx.L
        self.h = None
        h = C.c_void_p()
        ctx._chk(self.L.b200z_frame_compressor_new(ctx.h, level, 1 if checksum else 0, C.byref(h)))
        self.h = h
        self._source = self._drain = None
        if window_log != WINDOW_LOG_MIN:
            self.set_window_log(window_log)

    def __del__(self):
        try:
            if self.h and self.ctx.h:
                self.L.b200z_frame_compressor_free(self.h)
        except Exception:
            pass

    def set_source(self, source):
        old, self._source = self._source, source
        return old

    def set_drain(self, drain):
        old, self._drain = self._drain, drain
        return old

    def source(self): return self._source
    def drain(self): return self._drain

    def take_source(self):
        s, self._source = self._source, None
        return s

    def take_drain(self):
        d, self._drain = self._drain, None
        return d

    def set_compression_level(self, level):
        """Returns the previous level, as the reference does."""
        old = self.compression_level()
        self.ctx._chk(self.L.b200z_frame_compressor_set_compression_level(self.h, level))
        return old

    def compression_level(self): return self.L.b200z_frame_compressor_compression_level(self.h)

    def set_window_log(self, window_log):
        """EXTENSION: long-distance matches up to 2^window_log back from the next compress() on (17: none).  Returns the previous
        value."""
        old = self.window_log()
        self.ctx._chk(self.L.b200z_frame_compressor_set_window_log(self.h, window_log))
        return old

    def window_log(self): return self.L.b200z_frame_compressor_window_log(self.h)

    def compress(self):
        """One frame from the source to the drain.  Returns the COMPRESS_RESULT_DTYPE row: dst_size = bytes written, blocks,
        raw / RLE blocks, checksum."""
        panic = [k for k, v in error_names().items() if v == "B200Z_ERR_REFERENCE_WOULD_PANIC"][0]
        if self._source is None or self._drain is None:
            raise B200ZError(panic, 0, "FrameCompressor::compress: no source or no drain set")
        rd, wr, failure = _source_drain_callbacks(self._source, self._drain)
        res = np.zeros(1, dtype=COMPRESS_RESULT_DTYPE)
        e = self.L.b200z_frame_compressor_compress(self.h, rd, None, wr, None, res.ctypes.data)
        _raise_chained(self.ctx, e, failure)
        return res[0]


def _source_drain_callbacks(source, drain):
    """(READ_FN, WRITE_FN, failures) over a source (bytes or a file-like with read()) and a drain (a file-like with write(), or a
    bytearray, which the bytes are appended to).  An exception either raises makes the callback fail; it is kept in `failures`."""
    src = _Reader(source).src
    failure = []

    def _read(_user, buf, n):
        try:
            b = src.read(n)
            if b:
                C.memmove(buf, b, len(b))
            return len(b)
        except Exception as e:
            failure.append(e)
            return -1

    def _write(_user, buf, n):
        try:
            if isinstance(drain, bytearray):
                drain.extend(C.string_at(buf, n))
                return n
            r = drain.write(C.string_at(buf, n))
            return n if r is None else r
        except Exception as e:
            failure.append(e)
            return -1

    return READ_FN(_read), WRITE_FN(_write), failure


def _raise_chained(ctx, e, failure):
    """Raises B200ZError for a nonzero code, from the first exception a callback raised."""
    if e:
        raise B200ZError(e, 0, ctx.L.b200z_ctx_last_error_message(ctx.h).decode()) from (failure[0] if failure else None)


def compress(ctx, source, target, level=FASTEST, checksum=True, window_log=WINDOW_LOG_MIN):
    """Mirror of ruzstd::encoding::compress (encoding/mod.rs): one frame from `source` (bytes or a reader) to `target` (a writer
    or a bytearray) through a FrameCompressor (with long-distance matches up to 2^window_log back).  Returns its result row."""
    fc = FrameCompressor(ctx, level, checksum, window_log)
    fc.set_source(source)
    fc.set_drain(target)
    return fc.compress()


def compress_profile(ctx):
    """{kernel name: ms} of the last compress_frames call made with FLAG_PROFILE set on the context."""
    L = ctx.L
    n = L.b200z_compress_num_stages()
    ms = (C.c_float * n)()
    ctx._chk(L.b200z_compress_last_profile(ctx.h, ms, n))
    return {L.b200z_compress_stage_name(i).decode(): ms[i] for i in range(n)}


def raw_dict_bounds(n, dict_size):
    """(dictionary bytes, segment records) that always hold what b200z_dict_train_raw writes for n sample bytes: n itself below
    16 bytes, else min(dict_size, n), because the segments lie in disjoint epochs; and max(1, n // 10000) records, because every
    epoch but a lone one is at least 10,000 bytes long (tests/test_dict_train_model.py checks both against the epoch rule)."""
    return (n if n < 16 else min(dict_size, n)), max(1, n // 10000)


def create_raw_dict(ctx, samples, dict_size, sample_sizes=None, segment_size=2048, segments=False):
    """b200z_dict_train_raw: a raw-content dictionary of at most `dict_size` bytes trained on the GPU (an extension in place of
    ruzstd::dictionary; DESIGN.md section 4.5).  samples: bytes, numpy or torch (host or cuda), cut into samples by
    `sample_sizes` (None: one sample), or a list of bytes-likes, one sample each.  Returns the dictionary as bytes, or (bytes,
    DICT_SEGMENT_DTYPE rows in epoch order) with segments=True."""
    if isinstance(samples, (list, tuple)):
        parts = [bytes(x) for x in samples]
        if sample_sizes is None:
            sample_sizes = [len(x) for x in parts]
        samples = b"".join(parts)
    ip, n, _k = _ptr(samples)
    sizes = None if sample_sizes is None else np.ascontiguousarray(sample_sizes, dtype=np.uint64)
    cap, nseg_cap = raw_dict_bounds(n, dict_size)
    out = np.zeros(max(cap, 1), dtype=np.uint8)
    segs = np.zeros(nseg_cap, dtype=DICT_SEGMENT_DTYPE)
    dlen, nseg = C.c_size_t(), C.c_size_t()
    ctx._chk(ctx.L.b200z_dict_train_raw(ctx.h, ip, n, MEM_DEVICE if _is_device(samples) else MEM_HOST,
                                        None if sizes is None else sizes.ctypes.data, 0 if sizes is None else len(sizes), dict_size,
                                        segment_size, out.ctypes.data, cap, C.byref(dlen), segs.ctypes.data if segments else None,
                                        len(segs), C.byref(nseg)))
    d = out[:dlen.value].tobytes()
    return (d, segs[:nseg.value].copy()) if segments else d


def create_raw_dict_from_source(ctx, source, source_size, output, dict_size):
    """ruzstd::dictionary::create_raw_dict_from_source (dictionary/mod.rs:127): reads `source` (a reader or bytes) to its end and
    writes a raw-content dictionary of at most `dict_size` bytes to `output` (anything with write()).  The training runs on the
    bytes read, so `source_size`, the reference's estimate of them, is not used."""
    data = bytes(source) if isinstance(source, (bytes, bytearray, memoryview)) else source.read()
    output.write(create_raw_dict(ctx, data, dict_size))


def create_raw_dict_from_dir(ctx, path, output, dict_size):
    """ruzstd::dictionary::create_raw_dict_from_dir (dictionary/mod.rs:76): every file under `path`, subdirectories included, is
    one sample.  Deviation: the files are taken in sorted path order, where the reference chains them in read_dir order (which
    the file system decides), so the dictionary does not depend on the file system."""
    files = []
    for dirpath, _, names in os.walk(path):
        files += [os.path.join(dirpath, f) for f in names]
    parts = []
    for f in sorted(files):
        with open(f, "rb") as fh:
            parts.append(fh.read())
    output.write(create_raw_dict(ctx, parts, dict_size))


DICT_HEADER_MAX = 328   # B200Z_DICT_HEADER_MAX: an upper bound on a finalized dictionary's header


def _samples_arg(samples, sample_sizes):
    """(samples buffer, sample sizes as u64 or None): a list of bytes-likes is one sample each; a buffer without sizes is one sample."""
    if isinstance(samples, (list, tuple)):
        parts = [bytes(x) for x in samples]
        if sample_sizes is None:
            sample_sizes = [len(x) for x in parts]
        samples = b"".join(parts)
    return samples, None if sample_sizes is None else np.ascontiguousarray(sample_sizes, dtype=np.uint64)


def finalize_dict(ctx, content, samples, sample_sizes=None, dict_id=0, dict_cap=None):
    """b200z_dict_finalize: `content` (bytes) as a zstd-format dictionary whose entropy tables come from the statistics of
    `samples` on the GPU (an extension, the counterpart of ZDICT_finalizeDictionary; DESIGN.md section 4.6).  samples: bytes,
    numpy or torch (host or cuda), cut by `sample_sizes` (None: one sample), or a list of bytes-likes, one sample each; an empty
    list gives the tables of flat counts.  dict_id 0 derives libzstd's ID from the content.  dict_cap: the largest dictionary
    wanted (None: room for all of the content); the content's last bytes are kept when it does not fit.  Returns bytes."""
    c = bytes(content)
    samples, sizes = _samples_arg(samples, sample_sizes)
    ip, n, _k = _ptr(samples)
    if sizes is None:
        sizes = np.array([n], dtype=np.uint64)
    cap = DICT_HEADER_MAX + len(c) if dict_cap is None else dict_cap
    out = np.zeros(max(cap, 1), dtype=np.uint8)
    dlen = C.c_size_t()
    ctx._chk(ctx.L.b200z_dict_finalize(ctx.h, c, len(c), ip, n, MEM_DEVICE if _is_device(samples) else MEM_HOST, sizes.ctypes.data, len(sizes),
                                       dict_id, out.ctypes.data, cap, C.byref(dlen)))
    return out[:dlen.value].tobytes()


def create_dict(ctx, samples, dict_size, sample_sizes=None, segment_size=2048, dict_id=0):
    """A zstd-format dictionary of at most `dict_size` bytes: create_raw_dict's content, finalized on the same samples
    (finalize_dict), its first bytes giving way to the header."""
    samples, sizes = _samples_arg(samples, sample_sizes)
    content = create_raw_dict(ctx, samples, dict_size, sample_sizes=sizes, segment_size=segment_size)
    return finalize_dict(ctx, content, samples, sizes, dict_id=dict_id, dict_cap=dict_size)


def dict_from_counts(counts, content, dict_id=0, dict_cap=None):
    """Host-only: what finalize_dict writes for the statistics counts[377] (literal bytes, LL, ML, OF codes) -- dict_from_counts,
    csrc/dict_format.cpp."""
    cnt = np.ascontiguousarray(counts, dtype=np.uint64)
    assert cnt.shape == (377,)
    c = bytes(content)
    cap = DICT_HEADER_MAX + len(c) if dict_cap is None else dict_cap
    out = np.zeros(max(cap, 1), dtype=np.uint8)
    dlen = C.c_size_t()
    rc = lib().b200z_debug_dict_from_counts(cnt.ctypes.data, c, len(c), dict_id, out.ctypes.data, cap, C.byref(dlen))
    if rc:
        raise B200ZError(rc, 0, "b200z_debug_dict_from_counts")
    return out[:dlen.value].tobytes()


class Batch:
    """Prepared submission: plan + descriptors + input resident in HBM; run() launches kernels only."""

    def __init__(self, ctx, input, frames, dicts=None, forced_dict=None, max_window_size=0):
        self.ctx = ctx
        self.frames = _frames_array(frames)
        ip, il, self._k = _ptr(input)
        darr, nd, forced = _dict_args(dicts, forced_dict)
        self._dicts = (dicts, forced_dict)
        h = C.c_void_p()
        ctx._chk(ctx.L.b200z_batch_prepare(ctx.h, ip, il, MEM_DEVICE if _is_device(input) else MEM_HOST, self.frames.ctypes.data,
                                           len(self.frames), darr, nd, forced, max_window_size, C.byref(h)))
        self.h = h

    def run(self, d_output):
        op, ol, _k = _ptr(d_output)
        assert _is_device(d_output), "Batch.run writes into device memory"
        self.ctx._chk(self.ctx.L.b200z_batch_run(self.h, op, ol))

    def run_profile(self, d_output):
        """{kernel name: device ms} for one pass, measured with CUDA events between the kernels."""
        op, ol, _k = _ptr(d_output)
        n = self.ctx.L.b200z_num_stages()
        ms = (C.c_float * n)()
        self.ctx._chk(self.ctx.L.b200z_batch_run_profile(self.h, op, ol, ms, n))
        return {self.ctx.L.b200z_stage_kernel_name(i).decode(): float(ms[i]) for i in range(n)}

    def run_timeline(self, d_output):
        """Completion time (ms from the start of the pass) of each kernel in the overlapped launch."""
        op, ol, _k = _ptr(d_output)
        ms = (C.c_float * 4)()
        self.ctx._chk(self.ctx.L.b200z_batch_run_timeline(self.h, op, ol, ms, 4))
        return {"k_setup+k_huf": float(ms[1]), "k_fse+k_exec": float(ms[2]), "k_exec_cta+k_exec": float(ms[3])}

    def finish(self):
        res = np.zeros(len(self.frames), dtype=FRAME_RESULT_DTYPE)
        self.ctx._chk(self.ctx.L.b200z_batch_finish(self.h, res.ctypes.data))
        return res

    def info(self):
        """Facts about the plan; launches_per_run is the kernels the most recent run() launched (0 before it)."""
        a = (C.c_uint64 * 8)()
        self.ctx.L.b200z_batch_info(self.h, a)
        k = ["frames", "blocks", "compressed_blocks", "planned_bytes", "literal_scratch_bytes", "sequences", "launches_per_run"]
        return dict(zip(k, list(a)))

    def debug_literals(self, block, cap=1 << 20):
        buf = np.empty(cap, dtype=np.uint8)
        n = C.c_size_t()
        self.ctx._chk(self.ctx.L.b200z_batch_debug_literals(self.h, block, buf.ctypes.data, cap, C.byref(n)))
        return buf[:n.value].tobytes()

    def debug_sequences(self, block, cap=100000):
        buf = np.empty((cap, 3), dtype=np.uint32)
        n = C.c_size_t()
        self.ctx._chk(self.ctx.L.b200z_batch_debug_sequences(self.h, block, buf.ctypes.data, cap, C.byref(n)))
        return buf[:n.value].copy()

    def debug_sched(self):
        a = (C.c_uint32 * 4)()
        self.ctx._chk(self.ctx.L.b200z_batch_debug_sched(self.h, a))
        return {"cta_frames": a[0], "handed_back_frames": a[1], "reasons": a[2], "handed_back_blocks": a[3]}

    def debug_waves(self):
        a = (C.c_uint32 * 4)()
        self.ctx._chk(self.ctx.L.b200z_batch_debug_waves(self.h, a))
        return {"k_huf": a[0], "k_fse": a[1], "k_huf_ctas_per_sm": a[2], "k_fse_ctas_per_sm": a[3]}

    def debug_block_flags(self, block):
        v = C.c_uint32()
        self.ctx._chk(self.ctx.L.b200z_batch_debug_block_flags(self.h, block, C.byref(v)))
        return v.value

    def debug_tables(self, block):
        """{"huf", "ll", "of", "ml"} tables block `block` decodes with (None = absent).  huf: {"max_bits", "entries": 2^max_bits
        (symbol, nb)}; ll/of/ml: {"log", "valid", "is_rle", "entries": 2^log (symbol, nb, baseline)} unpacked from fse_pack16."""
        huf = np.zeros(HUF_DEBUG_BYTES, dtype=np.uint8)
        fse = np.zeros(3 * FSE_DEBUG_BYTES, dtype=np.uint8)
        present = (C.c_uint32 * 4)()
        self.ctx._chk(self.ctx.L.b200z_batch_debug_tables(self.h, block, huf.ctypes.data, fse.ctypes.data, present))
        out = {"huf": None, "ll": None, "of": None, "ml": None}
        if present[0]:
            mb = int(huf[:4].view(np.uint32)[0])
            sym, nb4 = huf[16:16 + 2048], huf[16 + 2048:]
            n = 1 << mb if mb else 0
            out["huf"] = {"max_bits": mb, "entries": [(int(sym[i]), int(nb4[i >> 1] >> (4 * (i & 1))) & 15) for i in range(n)]}
        for k, name in enumerate(("ll", "of", "ml")):
            if not present[1 + k]:
                continue
            t = fse[k * FSE_DEBUG_BYTES:(k + 1) * FSE_DEBUG_BYTES]
            log, valid, is_rle = (int(x) for x in t[:12].view(np.uint32))
            ents = []
            for e in t[16:].view(np.uint16)[:1 << log] if log <= 9 else []:
                f, s = int(e) & 0x3FF, int(e) >> 10
                nb = log - (f.bit_length() - 1) if f else 0
                ents.append((s, nb, (f - (1 << (f.bit_length() - 1))) << nb if f else 0))
            out[name] = {"log": log, "valid": valid, "is_rle": is_rle, "entries": ents}
        return out

    def close(self):
        if getattr(self, "h", None) and self.ctx.h:
            self.ctx.L.b200z_batch_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _Reader:
    """io::Read adaptor over bytes or a Python file-like; keeps the ctypes callback alive."""

    def __init__(self, src):
        if isinstance(src, (bytes, bytearray, memoryview)):
            src = io.BytesIO(bytes(src))
        self.src = src

        def _cb(_user, buf, n):
            b = self.src.read(n)
            if b:
                C.memmove(buf, b, len(b))
            return len(b)
        self.cb = READ_FN(_cb)


class FrameDecoder:
    """GPU-backed mirror of ruzstd::decoding::FrameDecoder (frame_decoder.rs:154-627)."""

    def __init__(self, ctx, _handle=None):
        self.ctx, self.L = ctx, ctx.L
        if _handle is None:
            h = C.c_void_p()
            ctx._chk(self.L.b200z_frame_decoder_new(ctx.h, C.byref(h)))
            _handle = h
        self.h = _handle

    def __del__(self):
        try:
            if self.h and self.ctx.h:
                self.L.b200z_frame_decoder_free(self.h)
        except Exception:
            pass

    def _chk(self, e):
        if e:
            raise B200ZError(e, self.L.b200z_frame_decoder_last_stage(self.h), self.L.b200z_frame_decoder_last_error_message(self.h).decode())

    def set_max_window_size(self, n): self.L.b200z_frame_decoder_set_max_window_size(self.h, n)
    def max_window_size(self): return self.L.b200z_frame_decoder_max_window_size(self.h)

    def reset(self, reader):
        if not isinstance(reader, _Reader):
            reader = _Reader(reader)
        self._chk(self.L.b200z_frame_decoder_reset(self.h, reader.cb, None))
        return reader
    init = reset

    def skip_frame_length(self): return self.L.b200z_frame_decoder_skip_frame_length(self.h)

    def add_dict(self, raw):
        b = bytes(raw)
        self._chk(self.L.b200z_frame_decoder_add_dict(self.h, b, len(b)))

    def add_raw_content_dict(self, dict_id, content):
        b = bytes(content)
        self._chk(self.L.b200z_frame_decoder_add_raw_content_dict(self.h, dict_id, b, len(b)))

    def force_dict(self, dict_id): self._chk(self.L.b200z_frame_decoder_force_dict(self.h, dict_id))

    def decode_blocks(self, reader, strategy=ALL, n=0):
        fin = C.c_int(0)
        self._chk(self.L.b200z_frame_decoder_decode_blocks(self.h, reader.cb, None, strategy, n, C.byref(fin)))
        return bool(fin.value)

    def read(self, n):
        buf = np.empty(max(n, 1), dtype=np.uint8)
        r = self.L.b200z_frame_decoder_read(self.h, buf.ctypes.data, n)
        if r < 0:
            raise B200ZError(16, 9)
        return buf[:r].tobytes()

    def collect(self):
        """FrameDecoder::collect (frame_decoder.rs:381-389)."""
        out = bytearray()
        while True:
            n = self.can_collect()
            if n == 0:
                return bytes(out)
            out += self.read(n)

    def collect_to_writer(self, writer):
        def _cb(_user, buf, n):
            return writer.write(C.string_at(buf, n)) or 0
        cb = WRITE_FN(_cb)
        r = self.L.b200z_frame_decoder_collect_to_writer(self.h, cb, None)
        if r < 0:
            raise B200ZError(16, 9)
        return r

    def can_collect(self): return self.L.b200z_frame_decoder_can_collect(self.h)
    def is_finished(self): return bool(self.L.b200z_frame_decoder_is_finished(self.h))
    def blocks_decoded(self): return self.L.b200z_frame_decoder_blocks_decoded(self.h)
    def bytes_read_from_source(self): return self.L.b200z_frame_decoder_bytes_read_from_source(self.h)
    def content_size(self): return self.L.b200z_frame_decoder_content_size(self.h)

    def get_checksum_from_data(self):
        v = C.c_uint32()
        return v.value if self.L.b200z_frame_decoder_get_checksum_from_data(self.h, C.byref(v)) else None

    def get_calculated_checksum(self):
        v = C.c_uint32()
        return v.value if self.L.b200z_frame_decoder_get_calculated_checksum(self.h, C.byref(v)) else None

    def decode_from_to(self, source, target_len):
        src = bytes(source)
        buf = np.empty(max(target_len, 1), dtype=np.uint8)
        r, w = C.c_size_t(), C.c_size_t()
        self._chk(self.L.b200z_frame_decoder_decode_from_to(self.h, src, len(src), buf.ctypes.data, target_len, C.byref(r), C.byref(w)))
        return r.value, buf[:w.value].tobytes()

    def decode_all(self, data, out_cap):
        src = bytes(data)
        buf = np.empty(max(out_cap, 1), dtype=np.uint8)
        w = C.c_size_t()
        self._chk(self.L.b200z_frame_decoder_decode_all(self.h, src, len(src), buf.ctypes.data, out_cap, C.byref(w)))
        return buf[:w.value].tobytes()

    def decode_all_to_vec(self, data, capacity):
        """decode_all_to_vec (frame_decoder.rs:591-610): `capacity` plays the Vec's spare capacity."""
        return self.decode_all(data, capacity)


class StreamingDecoder:
    """GPU-backed mirror of ruzstd::decoding::StreamingDecoder (streaming_decoder.rs:45-156)."""

    def __init__(self, ctx, source, decoder=None, max_window_size=None):
        self.ctx, self.L = ctx, ctx.L
        self.source = _Reader(source)
        h = C.c_void_p()
        self._borrowed = decoder
        if decoder is not None:        # new_with_decoder
            e = self.L.b200z_streaming_decoder_new_with_decoder(self.source.cb, None, decoder.h, C.byref(h))
            if e:
                raise B200ZError(e, self.L.b200z_frame_decoder_last_stage(decoder.h))
        elif max_window_size is not None:
            e = self.L.b200z_streaming_decoder_new_with_max_window_size(ctx.h, self.source.cb, None, max_window_size, C.byref(h))
            if e:
                raise B200ZError(e, 1)
        else:
            e = self.L.b200z_streaming_decoder_new(ctx.h, self.source.cb, None, C.byref(h))
            if e:
                raise B200ZError(e, 1)
        self.h = h

    def read(self, n):
        buf = np.empty(max(n, 1), dtype=np.uint8)
        err = C.c_int(0)
        r = self.L.b200z_streaming_decoder_read(self.h, buf.ctypes.data, n, C.byref(err))
        if r < 0:
            raise B200ZError(err.value or 16)
        return buf[:r].tobytes()

    def read_to_end(self, chunk=1 << 16):
        out = bytearray()
        while True:
            b = self.read(chunk)
            if not b:
                return bytes(out)
            out += b

    def into_frame_decoder(self):
        if self._borrowed is not None:
            self.L.b200z_streaming_decoder_free(self.h); self.h = None
            return self._borrowed
        dh = self.L.b200z_streaming_decoder_into_frame_decoder(self.h)
        self.h = None
        return FrameDecoder(self.ctx, C.c_void_p(dh))

    def __del__(self):
        try:
            if self.h and self.ctx.h:
                self.L.b200z_streaming_decoder_free(self.h)
        except Exception:
            pass
