"""zstd-rs_b200 -- GPU-native (H100, sm_90a) zstd block decompressor behind ruzstd's FrameDecoder / StreamingDecoder API,
a batch compressor at ruzstd's Uncompressed and Fastest levels and extension levels LAZY, OPT and ULTRA (compress_frames / compress_to_vec; with
long-distance matches up to 2^27 bytes back through window_log, as the stream compressor), a stream compressor behind
ruzstd's FrameCompressor / encoding::compress API (FrameCompressor, compress), and a raw-content
dictionary trainer in place of ruzstd::dictionary (create_raw_dict, create_raw_dict_from_source, create_raw_dict_from_dir)
and a finalizer that turns its content into a zstd-format dictionary (finalize_dict, create_dict).  decode_all_stream decodes a
source of concatenated frames to a drain chunk by chunk through the GPU, in bounded memory.  compress_seekable writes zstd's
seekable format (independent frames behind a seek table), compress_seekable_stream writes it from a reader to a writer in bounded
memory, and SeekableArchive reads byte ranges of such an archive on the GPU, from memory or, with from_source, from a file.

The product is the C-ABI library ``libb200zstd.so`` (include/b200zstd.h, sources in csrc/).  This package is the
Python host-side mirror of the reference interface (same names, argument meaning and error behaviour as
ruzstd::decoding::{FrameDecoder, StreamingDecoder, BlockDecodingStrategy}) over that ABI via ctypes.

There is no CPU decode path: every decode call needs a CUDA device and fails loudly without one.
Import name: ``zstd_rs_b200`` (the directory name has a hyphen; see ``_pkg.py`` at the repo root).
"""
from .binding import (  # noqa: F401
    ALL, FASTEST, LAZY, OPT, ULTRA, UNCOMPRESSED, UPTO_BLOCKS, UPTO_BYTES, AllBatch, B200ZError, Batch, Context, Dictionary, FrameCompressor, FrameDecoder,
    SeekableArchive, StreamingDecoder, build, compress, compress_bound, compress_frames, compress_patch_from, compress_profile, compress_seekable, compress_seekable_stream, compress_to_vec, create_dict, create_raw_dict,
    create_raw_dict_from_dir,
    create_raw_dict_from_source, decode_all, decode_all_batch, decode_all_stream, decode_blocks, decode_frames,
    dict_from_counts, patch_window_log, error_names, finalize_dict, lib, lib_path, seekable_bound, seekable_plan, xxh64,
)
from . import binding  # noqa: F401
