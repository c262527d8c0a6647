/*
 * b200zstd.h -- C ABI of the GPU-native (H100, sm_90a) zstd block decompressor (libb200zstd.so).
 *
 * Drop-in boundary for the decode hot path of ruzstd (KillingSpark/zstd-rs @ eb7e03cc, crate ruzstd 0.9.1).
 * Everything below replaces work that the reference does inside
 *     BlockDecoder::decompress_block            ruzstd/src/decoding/block_decoder.rs:97-197
 * called from the block loops of
 *     FrameDecoder::decode_blocks               ruzstd/src/decoding/frame_decoder.rs:309-377
 *     FrameDecoder::decode_from_to              ruzstd/src/decoding/frame_decoder.rs:439-529
 * i.e. decode_literals (literals_section_decoder.rs:12), decode_sequences (sequence_section_decoder.rs:14),
 * execute_sequences (sequence_execution.rs:5) and DecodeBuffer::{push,repeat} (decode_buffer.rs:74,79), with
 * HuffmanTable / FSETable (huff0_decoder.rs:57, fse_decoder.rs:59) built and kept on the GPU.
 *
 * Plain C: opaque handles, pointers and sizes only.  No torch / CUDA types in any signature (a stream is passed
 * as void*).  No process-global state; a handle may migrate between threads but is used by one at a time
 * (the reference's FrameDecoder is Send + Sync, tests/mod.rs:37-45).  Nothing here ever falls back to a CPU
 * decoder: if no CUDA device is usable, b200z_ctx_create fails with B200Z_ERR_NO_DEVICE and every other entry
 * point needs a ctx.
 *
 * Error convention: int return, 0 = ok, >0 = b200z_error (one code per leaf of the reference's nested error
 * enums, decoding/errors.rs; numbering shared with the test oracle).  b200z_*_last_stage tells which stage
 * raised it (the nesting path in the reference).
 */
#ifndef B200ZSTD_H
#define B200ZSTD_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200Z_ABI_VERSION 1

typedef enum b200z_error {

    B200Z_OK = 0,
    /* ReadFrameHeaderError (errors.rs:95-104) */
    B200Z_ERR_MAGIC_NUMBER_READ = 1,
    B200Z_ERR_BAD_MAGIC_NUMBER = 2,
    B200Z_ERR_FRAME_DESCRIPTOR_READ = 3,
    B200Z_ERR_INVALID_FRAME_DESCRIPTOR = 4,
    B200Z_ERR_WINDOW_DESCRIPTOR_READ = 5,
    B200Z_ERR_DICTIONARY_ID_READ = 6,
    B200Z_ERR_FRAME_CONTENT_SIZE_READ = 7,
    B200Z_ERR_SKIP_FRAME = 8,
    /* FrameHeaderError (errors.rs:34-42) / FrameDecoderError (errors.rs:472-486) */
    B200Z_ERR_WINDOW_TOO_BIG = 10,
    B200Z_ERR_WINDOW_TOO_SMALL = 11,
    B200Z_ERR_WINDOW_SIZE_TOO_BIG = 12,
    B200Z_ERR_DICT_NOT_PROVIDED = 13,
    B200Z_ERR_NOT_YET_INITIALIZED = 14,
    B200Z_ERR_FAILED_TO_READ_CHECKSUM = 15,
    B200Z_ERR_FAILED_TO_DRAIN_DECODEBUFFER = 16,
    B200Z_ERR_FAILED_TO_SKIP_FRAME = 17,
    B200Z_ERR_TARGET_TOO_SMALL = 18,
    /* BlockHeaderReadError (errors.rs:156-161) */
    B200Z_ERR_BLOCK_HEADER_READ = 20,
    B200Z_ERR_FOUND_RESERVED_BLOCK = 21,
    B200Z_ERR_BLOCK_SIZE_TOO_LARGE = 22,
    /* DecodeBlockContentError / DecompressBlockError (errors.rs:345-350, 256-267) */
    B200Z_ERR_DECODER_STATE_IS_FAILED = 30,
    B200Z_ERR_EXPECTED_HEADER_OF_PREVIOUS_BLOCK = 31,
    B200Z_ERR_BLOCK_BODY_READ = 32,
    B200Z_ERR_BLOCK_CONTENT_READ = 33,
    B200Z_ERR_MALFORMED_SECTION_HEADER = 34,
    /* LiteralsSectionParseError / SequencesHeaderParseError (errors.rs:816-820, 870-872) */
    B200Z_ERR_LITSEC_ILLEGAL_TYPE = 40,
    B200Z_ERR_LITSEC_GET_BITS = 41,
    B200Z_ERR_LITSEC_NOT_ENOUGH_BYTES = 42,
    B200Z_ERR_SEQHDR_NOT_ENOUGH_BYTES = 45,
    /* DecompressLiteralsError (errors.rs:586-598) */
    B200Z_ERR_LIT_MISSING_COMPRESSED_SIZE = 50,
    B200Z_ERR_LIT_MISSING_NUM_STREAMS = 51,
    B200Z_ERR_LIT_GET_BITS = 52,
    B200Z_ERR_LIT_UNINITIALIZED_HUFFMAN_TABLE = 55,
    B200Z_ERR_LIT_MISSING_BYTES_FOR_JUMP_HEADER = 56,
    B200Z_ERR_LIT_MISSING_BYTES_FOR_LITERALS = 57,
    B200Z_ERR_LIT_EXTRA_PADDING = 58,
    B200Z_ERR_LIT_BITSTREAM_READ_MISMATCH = 59,
    B200Z_ERR_LIT_DECODED_LITERAL_COUNT_MISMATCH = 60,
    /* HuffmanTableError (errors.rs:991-1028) */
    B200Z_ERR_HUF_GET_BITS = 70,
    B200Z_ERR_HUF_FSE_DECODER = 71,
    B200Z_ERR_HUF_SOURCE_IS_EMPTY = 72,
    B200Z_ERR_HUF_NOT_ENOUGH_BYTES_FOR_WEIGHTS = 73,
    B200Z_ERR_HUF_EXTRA_PADDING = 74,
    B200Z_ERR_HUF_TOO_MANY_WEIGHTS = 75,
    B200Z_ERR_HUF_MISSING_WEIGHTS = 76,
    B200Z_ERR_HUF_LEFTOVER_NOT_POWER_OF_2 = 77,
    B200Z_ERR_HUF_NOT_ENOUGH_BYTES_TO_DECOMPRESS_WEIGHTS = 78,
    B200Z_ERR_HUF_FSE_TABLE_USED_TOO_MANY_BYTES = 79,
    B200Z_ERR_HUF_NOT_ENOUGH_BYTES_IN_SOURCE = 80,
    B200Z_ERR_HUF_WEIGHT_BIGGER_THAN_MAX_NUM_BITS = 81,
    B200Z_ERR_HUF_MAX_BITS_TOO_HIGH = 82,
    /* FSETableError (errors.rs:892-908); the same leaf can surface under Huffman weights, sequence
     * tables or a dictionary -- the code is the leaf, zo_last_error_stage() tells where. */
    B200Z_ERR_FSE_ACC_LOG_IS_ZERO = 90,
    B200Z_ERR_FSE_ACC_LOG_TOO_BIG = 91,
    B200Z_ERR_FSE_GET_BITS = 92,
    B200Z_ERR_FSE_PROBABILITY_COUNTER_MISMATCH = 93,
    B200Z_ERR_FSE_TOO_MANY_SYMBOLS = 94,
    B200Z_ERR_FSE_TABLE_IS_UNINITIALIZED = 95, /* FSEDecoderError::TableIsUninitialized (errors.rs:957-960) */
    /* DecodeSequenceError (errors.rs:726-739) */
    B200Z_ERR_SEQ_EXTRA_PADDING = 100,
    B200Z_ERR_SEQ_UNSUPPORTED_OFFSET = 101,
    B200Z_ERR_SEQ_ZERO_OFFSET = 102,
    B200Z_ERR_SEQ_NOT_ENOUGH_BYTES_FOR_NUM_SEQUENCES = 103,
    B200Z_ERR_SEQ_EXTRA_BITS = 104,
    B200Z_ERR_SEQ_MISSING_COMPRESSION_MODE = 105,
    B200Z_ERR_SEQ_MISSING_BYTE_FOR_RLE_LL_TABLE = 106,
    B200Z_ERR_SEQ_MISSING_BYTE_FOR_RLE_OF_TABLE = 107,
    B200Z_ERR_SEQ_MISSING_BYTE_FOR_RLE_ML_TABLE = 108,
    /* ExecuteSequencesError / DecodeBufferError (errors.rs:683-687, 393-396) */
    B200Z_ERR_EXEC_NOT_ENOUGH_BYTES_FOR_SEQUENCE = 110,
    B200Z_ERR_EXEC_ZERO_OFFSET = 111,
    B200Z_ERR_EXEC_NOT_ENOUGH_BYTES_IN_DICTIONARY = 112,
    B200Z_ERR_EXEC_OFFSET_TOO_BIG = 113,
    /* DictionaryDecodeError (errors.rs:419-424) */
    B200Z_ERR_DICT_NOT_ENOUGH_BYTES = 120,
    B200Z_ERR_DICT_BAD_MAGIC_NUM = 121,
    /* Places where the reference would panic (assert!/unreachable!/index out of bounds) instead of
     * returning an error; SURVEY.md Appendix B.8.  Never produced by spec-valid input. */
    B200Z_ERR_REFERENCE_WOULD_PANIC = 200,
    /* Resource limits of this build (documented deviations, never hit by spec-valid input). */
    B200Z_ERR_BLOCK_OUTPUT_LIMIT = 210,
    B200Z_ERR_INVALID_ARGUMENT = 220,
    B200Z_ERR_OUT_OF_MEMORY = 221
    ,
    /* this build only */
    B200Z_ERR_NO_DEVICE = 230,
    B200Z_ERR_CUDA = 231,
    /* EXTENSION, seekable archives (b200z_seekable_*): the seek table breaks one of the format's rules (the message names it) */
    B200Z_ERR_SEEKABLE_TABLE = 240,
    /* EXTENSION, seekable archives: a frame decoded to a size other than its seek-table entry's Decompressed_Size */
    B200Z_ERR_SEEKABLE_FRAME_SIZE = 241,
    /* EXTENSION, seekable archives from and to callbacks: a read, positional read or write callback failed or came up short (the
     * message names the callback and the archive offset) */
    B200Z_ERR_SEEKABLE_IO = 242
} b200z_error;

/* stage that raised the error == nesting path of the reference's FrameDecoderError (errors.rs:472-486) */
typedef enum b200z_stage {
    B200Z_STAGE_NONE = 0,
    B200Z_STAGE_FRAME_HEADER = 1, /* ReadFrameHeaderError / FrameHeaderError                          */
    B200Z_STAGE_BLOCK_HEADER = 2, /* FailedToReadBlockHeader(BlockHeaderReadError)                    */
    B200Z_STAGE_BLOCK_BODY = 3,   /* FailedToReadBlockBody(DecodeBlockContentError / section headers) */
    B200Z_STAGE_LITERALS = 4,     /* ... DecompressLiteralsError                                      */
    B200Z_STAGE_SEQUENCES = 5,    /* ... DecodeSequenceError                                          */
    B200Z_STAGE_EXECUTE = 6,      /* ... ExecuteSequencesError                                        */
    B200Z_STAGE_CHECKSUM = 7,     /* FailedToReadChecksum                                             */
    B200Z_STAGE_DICTIONARY = 8,   /* DictionaryDecodeError                                            */
    B200Z_STAGE_DRAIN = 9         /* FailedToDrainDecodebuffer                                        */
} b200z_stage;

const char *b200z_error_name(int code);
int b200z_abi_version(void);

/* ------------------------------------------------------------------------------------------------------------
 * Device context: pins one CUDA device, owns its stream(s) and scratch pools.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200z_ctx b200z_ctx;
int b200z_ctx_create(int device_ordinal, b200z_ctx **out);
void b200z_ctx_destroy(b200z_ctx *ctx);
const char *b200z_ctx_last_error_message(const b200z_ctx *ctx);
/* the CUDA stream (cudaStream_t as void*) all work of this ctx is enqueued on; for event timing by callers */
void *b200z_ctx_stream(const b200z_ctx *ctx);
/* Context flags.  B200Z_FLAG_CHECKSUM: the batch entry also computes every frame's content checksum on the GPU (XXH64 seed 0 over
 * the plaintext, the hash the reference feeds while draining, decode_buffer.rs:225-226,290,301) and returns it in
 * b200z_frame_result.calculated_checksum -- like the reference it is reported, never enforced (frame_decoder.rs:253-270).
 * Device output buffers must be readable 8 bytes past their end when this flag is set. */
#define B200Z_FLAG_CHECKSUM 1u
void b200z_ctx_set_flags(b200z_ctx *ctx, uint32_t flags);
uint32_t b200z_ctx_flags(const b200z_ctx *ctx);
/* number of this library's kernel launches since ctx creation (bench.py's gpu_launches) */
uint64_t b200z_ctx_kernel_launches(const b200z_ctx *ctx);
/* Bytes of device memory and of pinned host memory the library holds right now, over every context and handle of the process:
 * exactly what its allocations asked for (each cudaMalloc / cudaMallocHost it made and has not freed), not the driver's rounding.
 * For tests of what a call keeps, which a card-wide reading cannot isolate on a shared device. */
void b200z_debug_held_bytes(uint64_t *device, uint64_t *pinned);

/* ------------------------------------------------------------------------------------------------------------
 * Dictionaries (device resident).  Replaces Dictionary::decode_dict (decoding/dictionary.rs:45-126) +
 * FrameDecoder::add_dict (frame_decoder.rs:224-227); tables are expanded on the GPU.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200z_dict b200z_dict;
int b200z_dict_create(b200z_ctx *ctx, const uint8_t *raw, size_t len, b200z_dict **out);
/* EXTENSION (not in the reference, SURVEY.md 8c gap): raw-content dictionary = content only, offset history
 * [1,4,8], no entropy tables.  Frames compressed against it carry no dict id; select it with force_dict /
 * the `forced_dict` argument. */
int b200z_dict_create_raw_content(b200z_ctx *ctx, uint32_t id, const uint8_t *content, size_t len, b200z_dict **out);
uint32_t b200z_dict_id(const b200z_dict *d);
int b200z_dict_offset_history(const b200z_dict *d, uint32_t out[3]);
size_t b200z_dict_content_size(const b200z_dict *d);
void b200z_dict_destroy(b200z_dict *d);

/* ------------------------------------------------------------------------------------------------------------
 * Tier 1 -- batch entry: many independent frames in one submission (the throughput path; frames shard
 * across GPUs by giving each rank's ctx its own sub-list).  For each frame this does what
 *   FrameDecoder::reset + [force_dict] + decode_blocks(BlockDecodingStrategy::All) + read
 * does in the reference (tests/decode_corpus.rs:76-100), for all frames at once.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200z_frame_io {
    uint64_t src_off;  /* byte offset of the frame (magic number first) inside `input`          */
    uint64_t src_size; /* bytes available for this frame (may exceed the frame; see bytes_read) */
    uint64_t out_off;  /* where this frame's plaintext goes inside `output`                     */
    uint64_t out_cap;  /* room reserved there; TargetTooSmall if the frame needs more           */
} b200z_frame_io;

typedef struct b200z_frame_result {
    uint64_t out_size;       /* plaintext bytes produced at out_off                                        */
    uint64_t bytes_read;     /* FrameDecoder::bytes_read_from_source (frame_decoder.rs:273)                */
    uint64_t content_size;   /* FrameDecoder::content_size (frame_decoder.rs:246)                          */
    uint64_t window_size;    /* FrameHeader::window_size (frame.rs:116)                                    */
    int32_t status;          /* 0 or b200z_error                                                           */
    int32_t stage;           /* b200z_stage of the error                                                   */
    uint32_t blocks_decoded; /* FrameDecoder::blocks_decoded (frame_decoder.rs:297)                        */
    uint32_t error_block;    /* index of the block that failed (when status != 0 in stages 2..6)           */
    uint32_t has_checksum;   /* frame carries a content checksum                                           */
    uint32_t checksum_from_data;  /* get_checksum_from_data (frame_decoder.rs:254)                         */
    uint32_t has_dict_id;
    uint32_t dict_id;        /* FrameHeader::dictionary_id (frame.rs:142)                                  */
    uint32_t has_calculated_checksum; /* 1 when the context ran the GPU checksum stage (B200Z_FLAG_CHECKSUM)   */
    uint32_t calculated_checksum;     /* get_calculated_checksum (frame_decoder.rs:262): XXH64(seed 0) low 32 bits */
} b200z_frame_result;

#define B200Z_MEM_HOST 0
#define B200Z_MEM_DEVICE 1

/* One-shot: plan on the host, copy in (if host memory), run the kernels, copy out (if host memory), fill
 * `results[nframes]`.  Returns 0 if the submission ran (per-frame outcome in results[i].status) or a
 * b200z_error for a submission-level failure.  `dicts`/`ndicts`: dictionaries selectable by frame dict id
 * (FrameDecoder::add_dict); `forced_dict`: applied to every frame after init (FrameDecoder::force_dict,
 * frame_decoder.rs:229) or NULL.  `max_window_size` 0 = the reference default 128 MiB (frame_decoder.rs:25). */
int b200z_decode_frames_batch(b200z_ctx *ctx, const uint8_t *input, size_t input_len, int input_mem,
                              const b200z_frame_io *frames, size_t nframes, const b200z_dict *const *dicts,
                              size_t ndicts, const b200z_dict *forced_dict, uint64_t max_window_size,
                              uint8_t *output, size_t output_cap, int output_mem, b200z_frame_result *results);

/* Split form of the same call, for device-resident pipelines and for timing the kernels alone:
 *   prepare: host plan (frame/block/section header walk) + upload of input and descriptors into HBM
 *   run:     ONLY kernel launches on the ctx stream (async), input/descriptors/tables/output all in HBM
 *   finish:  synchronise and fetch per-frame results */
typedef struct b200z_batch b200z_batch;
int b200z_batch_prepare(b200z_ctx *ctx, const uint8_t *input, size_t input_len, int input_mem,
                        const b200z_frame_io *frames, size_t nframes, const b200z_dict *const *dicts, size_t ndicts,
                        const b200z_dict *forced_dict, uint64_t max_window_size, b200z_batch **out);
int b200z_batch_run(b200z_batch *b, uint8_t *d_output, size_t output_cap);
int b200z_batch_finish(b200z_batch *b, b200z_frame_result *results);
/* b200z_batch_run with a CUDA event between kernels: synchronises and returns each kernel's device milliseconds
 * (stage_ms[i] for kernel b200z_stage_kernel_name(i), i < b200z_num_stages()).  Profiling aid for bench.py. */
int b200z_batch_run_profile(b200z_batch *b, uint8_t *d_output, size_t output_cap, float *stage_ms, size_t nstages);
/* one pass exactly as b200z_batch_run launches it, with events on the stream: out_ms[0..3] = completion time, relative to the
 * start of the pass, of k_setup, of k_huf, of the pair k_fse + k_exec (k_exec runs beside k_fse as its programmatic dependent)
 * and of k_exec_cta + the k_exec launch that takes what it handed back (n >= 4) */
int b200z_batch_run_timeline(b200z_batch *b, uint8_t *d_output, size_t output_cap, float *out_ms, size_t n);
int b200z_num_stages(void);
const char *b200z_stage_kernel_name(int stage);
/* facts about a prepared batch: [0] frames [1] blocks [2] compressed blocks [3] input bytes planned
 * [4] literal-scratch bytes [5] sequences [6] kernels the most recent b200z_batch_run launched, k_xxh64 included (0 before the
 * first run) */
int b200z_batch_info(const b200z_batch *b, uint64_t out[8]);
/* per-stage device pointers for kernel-level parity tests (tests/ only): literals scratch and sequence
 * scratch of the LAST run, laid out exactly as the oracle's trace (oracle/ruzstd_oracle.h zo_block_trace) */
int b200z_batch_debug_literals(b200z_batch *b, uint32_t block, uint8_t *host_out, size_t cap, size_t *len);
int b200z_batch_debug_sequences(b200z_batch *b, uint32_t block, uint32_t *host_out_ll_ml_of, size_t cap_seqs, size_t *nseq);
/* bit 0: the block's `of` column holds raw offset_values; otherwise offsets after do_offset_history
 * (sequence_execution.rs:59-118), symbolic where they depend on the repeat-offset history at the block's start:
 * tag << 30 | decrements, tag 1..3 = history slot + 1 */
int b200z_batch_debug_block_flags(b200z_batch *b, uint32_t block, uint32_t *flags);
/* the entropy tables block `block` decodes with, as the planner resolved them (the defining block's table for Treeless
 * literals and Repeat modes, the predefined tables, a dictionary's tables), copied raw: the huff0 table into huf_out
 * (B200Z_DEBUG_HUF_BYTES: u32 max_bits, u32 status, 8 bytes padding, u8 symbol[2048], 4-bit code length nb4[1024]) and the
 * LL, OF and ML tables into fse_out (3 x B200Z_DEBUG_FSE_BYTES: u32 log, u32 valid, u32 is_rle, u32 padding, u16 entry[512],
 * entry = (1 << (log - nb) | base >> nb) | symbol << 10).  present[0..3] (huf, ll, of, ml) = 0 where the block has no table. */
#define B200Z_DEBUG_HUF_BYTES 3088
#define B200Z_DEBUG_FSE_BYTES 1040
int b200z_batch_debug_tables(b200z_batch *b, uint32_t block, uint8_t *huf_out, uint8_t *fse_out, uint32_t present[4]);
/* execution scheduling counters of the last run (tests / profiling): [0] frames given to k_exec_cta (block assembled in
 * shared memory), [1] frames it handed back to k_exec (one warp per frame), [2] OR of the reasons, [3] blocks handed back */
int b200z_batch_debug_sched(b200z_batch *b, uint32_t out[4]);
/* waves the literal and sequence kernels take for this batch's blocks on its device (a wave = every CTA resident at once):
 * [0] k_huf, [1] k_fse, [2] k_huf's resident CTAs per SM with the bit-reader ring it takes for this batch, [3] k_fse's */
int b200z_batch_debug_waves(b200z_batch *b, uint32_t out[4]);
/* Host-only views of a submission's scheduling decisions (no context, no device; for CPU tests of the host logic).
 * b200z_debug_route_frames: which frames k_exec_cta would take (largest first) given each frame's work (sequences + compressed
 * bytes / 16) and whether it is eligible (>= 2 blocks, >= 4096 compressed bytes, no dictionary); cta_frames has room for nframes.
 * b200z_debug_fse_order: the order in which k_fse takes the blocks (row by row across the warp kernel's frames, by decreasing
 * sequence count inside a row, k_exec_cta's frames last); *n_order = 0 means descriptor order; order has room for nblocks_total. */
int b200z_debug_route_frames(const uint64_t *work, const uint8_t *eligible, size_t nframes, uint32_t sms, uint32_t *cta_frames, size_t *n_cta);
int b200z_debug_fse_order(const uint32_t *first_block, const uint32_t *nblocks, const uint8_t *on_cta, size_t nframes, const uint32_t *nseq,
                          size_t nblocks_total, uint32_t *order, size_t *n_order);
void b200z_batch_destroy(b200z_batch *b);

/* ------------------------------------------------------------------------------------------------------------
 * Tier 1c -- decode_all on the batch path: one buffer of frames back to back (zstd and skippable frames, as in multi-frame .zst
 * files), decoded in one GPU submission.  Does what FrameDecoder::decode_all / decode_all_to_vec (frame_decoder.rs:541-610) does,
 * without the caller knowing where a frame starts or where its plaintext goes:
 *   prepare: finds the frames -- from offset 0, each frame's header walk says where the next one starts; on device input every
 *            byte offset is tested for a magic number on the GPU first (k_find_frames) and only the candidates' header digests
 *            come back -- and plans them as one submission.  b200z_batch_info[0] = the zstd frames found.
 *   run:     b200z_batch_run on such a batch decodes every frame and places the plaintexts back to back in `d_output` by the size
 *            each frame decodes to (never by Frame_Content_Size, which the reference does not check either), clamped to output_cap.
 *            b200z_batch_run_profile / _timeline return B200Z_ERR_INVALID_ARGUMENT for it.
 *   finish:  the outcome, with the first error in stream order as decode_all raises it (frame header, FailedToSkipFrame, block,
 *            literals, sequences, execution, checksum read or TargetTooSmall).
 * The chain of frames ends at the end of the input, at a break in it (no magic number: BadMagicNumber, or MagicNumberRead with
 * fewer than 4 bytes left), at a skippable frame that runs past the input (FailedToSkipFrame) or at a frame whose walk stopped
 * (frame header error, truncated block, missing checksum), which is reported as the planner reports it.
 * Differences from the reference: frames after the failing one may have been decoded too (they are not counted); on an error,
 * `written` still says how many bytes the frames before the failing one wrote, and output past them is unspecified.  When a
 * frame does not fit, the reference's UptoBytes(1 MiB) loop is replayed from the frame's block sizes to tell TargetTooSmall from
 * a later error of the same frame; an execution error in a block that no longer fits is not seen (that block is not executed).
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200z_all_result {
    uint64_t written;          /* plaintext bytes of the frames before the failing one (all of them without an error)        */
    uint64_t frames;           /* zstd frames decoded before the failing one                                                  */
    uint64_t skippable_frames; /* skippable frames passed before the failing one                                              */
    uint64_t error_offset;     /* input offset of the failing frame (input_len without an error)                              */
    int32_t status;            /* 0 or the b200z_error decode_all returns                                                    */
    int32_t stage;             /* b200z_stage of the error (0 for TargetTooSmall, as the reference reports them)               */
    int32_t error_frame;       /* index of the failing zstd frame in `results`, -1 when the failure is not a zstd frame's     */
    uint32_t reserved;
} b200z_all_result;

/* `dicts` and `max_window_size` as for b200z_decode_frames_batch.  `forced_dict` is an EXTENSION: decode_all calls init per frame
 * and never forces a dictionary; a non-NULL forced_dict is applied to every zstd frame (raw-content dictionary frames, which
 * carry no dictionary id).  NULL gives the reference's behaviour. */
int b200z_decode_all_prepare(b200z_ctx *ctx, const uint8_t *input, size_t input_len, int input_mem, const b200z_dict *const *dicts,
                             size_t ndicts, const b200z_dict *forced_dict, uint64_t max_window_size, b200z_batch **out);
/* synchronises; `results` is NULL or has room for b200z_batch_info[0] entries, one per zstd frame of the chain in stream order */
int b200z_decode_all_finish(b200z_batch *b, b200z_all_result *summary, b200z_frame_result *results);
/* one-shot form: prepare, run, finish; with host output the `written` bytes are copied back */
int b200z_decode_all_batch(b200z_ctx *ctx, const uint8_t *input, size_t input_len, int input_mem, const b200z_dict *const *dicts,
                           size_t ndicts, const b200z_dict *forced_dict, uint64_t max_window_size, uint8_t *output, size_t output_cap,
                           int output_mem, b200z_all_result *summary);
/* Host-only view of how prepare finds the frames (no context, no device; for CPU tests): the input offsets of the frames of the
 * chain, the one where it ends included.  by_candidates = 0: the host-input walk, frame to frame.  by_candidates = 1: the
 * device-input selection -- every byte offset tested for a magic number, every candidate walked with the bytes left from it, the
 * chain followed through the sorted candidates -- with the scan and the walks done on the host.  `at` has room for `cap` offsets;
 * *n = the chain's length. */
int b200z_debug_decode_all_chain(const uint8_t *input, size_t input_len, int by_candidates, uint64_t *at, size_t cap, size_t *n);

/* Reader and writer callbacks (io::Read::read / io::Write::write semantics), for tiers 1d and 2 and the stream compressor */
typedef long (*b200z_read_fn)(void *user, uint8_t *buf, size_t len);        /* bytes read, 0 = EOF, <0 = error */
typedef long (*b200z_write_fn)(void *user, const uint8_t *buf, size_t len); /* bytes written, 0 = full, <0 = error */

/* ------------------------------------------------------------------------------------------------------------
 * Tier 1d -- decode_all from a reader to a writer, chunk by chunk, in bounded memory.  Decodes a source of any length (a .zst
 * file of concatenated zstd and skippable frames, pzstd output, the stream compressor's single frame of unknown size) at GPU
 * speed without holding the whole input or output anywhere.  Rules:
 *   Output:    the drain receives what FrameDecoder::decode_all (frame_decoder.rs:541-577) writes for the source's bytes with
 *              unlimited output: the zstd frames' plaintexts back to back, skippable frames skipped -- decode_all's rule, not
 *              StreamingDecoder's single frame -- whatever the chunk size and however the source splits its reads.
 *   Errors:    `all` is what b200z_decode_all_batch reports for the same bytes with enough output room; TargetTooSmall cannot occur.
 *              After an error nothing more is written: the drain ends with the failing frame's output up to its first failing block
 *              (`delivered`).  The source may have been read up to one chunk past the failing frame.
 *   Read / write failures: a read returning < 0 (or more than asked for) ends the source, as the tier-2 reader treats it, and the
 *              frame in progress fails with the reference's read leaf (BLOCK_HEADER_READ, BLOCK_CONTENT_READ, ...).  A write returning
 *              <= 0 is B200Z_ERR_FAILED_TO_DRAIN_DECODEBUFFER at B200Z_STAGE_DRAIN (collect_to_writer's leaf).  Nothing is left in
 *              flight either way, and the context stays usable.
 *   Checksums: EXTENSION, with B200Z_FLAG_CHECKSUM: every frame's XXH64 is computed on the GPU, frames that span submissions
 *              included, and compared with the checksum the frame carries.  As in the reference (frame_decoder.rs:253-270) it is
 *              reported, never enforced.
 *   Dictionaries: as decode_all: `dicts` selected by frame dictionary ID; `forced_dict` the tier-1c extension for raw-content frames.
 *   History:   documented deviation, for frames RFC 8878 does not allow.  A frame that continues into a submission reaches back
 *              window_size bytes (at least 32) before the submission's first byte of that frame; inside a submission it reaches all of
 *              the frame's earlier output.  An offset past the window, which the reference accepts only when its undrained buffer
 *              happens to hold more, may therefore fail or not depending on where a chunk boundary falls.  Likewise a submission's
 *              output room is the sum of its blocks' bounds, min(128 KiB, window) for a Compressed block: a Compressed block that
 *              decodes to more may overrun it, depending on the other blocks of its submission and so on the chunk size.  Its frame
 *              then fails with B200Z_ERR_BLOCK_OUTPUT_LIMIT (B200Z_STAGE_EXECUTE) where decode_all_batch may decode it.  Spec-valid
 *              frames never depend on either.
 * Chunking: the source is read into a pinned buffer and cut at block ends into submissions.  With C = B200Z_PIPELINE_CHUNK_BYTES
 * (read by each call; 64 MiB by default) a submission holds whole blocks and at most C bytes of input (frame headers, blocks,
 * checksums and the skippable frames between its frames), a decoded size bound of 4 * C (a Raw or RLE block counts its size, a
 * Compressed block min(128 KiB, window)), C / 16384 blocks and C / 4 sequences -- or exactly one block, whatever C is.  Skippable
 * frames in front of a submission are read and dropped, never buffered.  While submission k decodes, the calling thread reads and
 * cuts k + 1 and writes k - 1; a frame that runs past a cut continues from its state, tables and window tail, carried device to
 * device (k_carry); the host reads back only each submission's frame states and then exactly the plaintext it writes.
 * Memory, allocated by the first call (again when C changes) and kept by the context, depends on C and on the largest window W
 * seen only.  Device, per each of two slots: C + 2 * 131097 input, max(W, 32) + max(4 * C, 131072) output, 4 * C + 32 * C / 16384
 * literals, 12 * (C / 4 + C / 4096) sequence scratch and 6.2 KB of tables per block (C / 16384 blocks): in all about
 * 2 * (12.4 * C + W), 1.7 GB at 64 MiB.  Pinned host: 2 * (C + 2 * 131097) input and max(4 * C, 131072) output.
 * Returns 0 when the call ran to an outcome, which `result` reports (an error in the stream, a failed drain); otherwise a b200z_error
 * (B200Z_ERR_INVALID_ARGUMENT, B200Z_ERR_OUT_OF_MEMORY, B200Z_ERR_CUDA) and `result` says what was delivered before it.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200z_stream_result {
    b200z_all_result all;          /* what b200z_decode_all_batch reports for the same bytes with unlimited output           */
    uint64_t delivered;            /* bytes handed to write_cb: all.written, plus on an error the failing frame's output of
                                      every block before its first failing block                                             */
    uint64_t submissions;          /* GPU submissions (chunks) the call ran                                                    */
    uint64_t checksum_frames;      /* B200Z_FLAG_CHECKSUM: frames that carry a checksum and were compared                      */
    uint64_t checksum_mismatches;
    int64_t first_mismatch_frame;  /* index among the zstd frames, -1 when none                                               */
} b200z_stream_result;

int b200z_decode_all_stream(b200z_ctx *ctx, b200z_read_fn read_cb, void *read_user, b200z_write_fn write_cb, void *write_user,
                            const b200z_dict *const *dicts, size_t ndicts, const b200z_dict *forced_dict, uint64_t max_window_size,
                            b200z_stream_result *result);

/* Host-only view of how b200z_decode_all_stream cuts a byte string into submissions at chunk size `chunk` (no context, no device;
 * for CPU tests).  One record per submission that holds a frame: [start, end) its stream bytes (skippable frames dropped in front
 * of it excluded), in_bytes = end - start, the decoded size bound, blocks, sequences and frames it holds; flags bit 0: its first
 * frame continues from the one before, bit 1: its last frame continues into the next.  `end`: where the cutter stopped -- the error
 * it can see from the headers it reads (frame header, skipped bytes, block header, truncated block or checksum), at which frame
 * (error_offset = the frame's stream offset, the source's length without an error), the skippable frames passed and the most
 * bytes it held in its buffer.  `cuts` has room for `cap` records; *n = the number of records. */
typedef struct b200z_stream_cut {
    uint64_t start, end, in_bytes, out_bound, nblocks, nseq;
    uint32_t nframes, flags;
} b200z_stream_cut;
typedef struct b200z_stream_cut_end {
    uint64_t error_offset, skippable_frames, peak_buffered;
    int32_t status, stage, error_frame;
    uint32_t reserved;
} b200z_stream_cut_end;
int b200z_debug_stream_cut(const uint8_t *input, size_t input_len, uint64_t chunk, b200z_stream_cut *cuts, size_t cap, size_t *n,
                           b200z_stream_cut_end *end);

/* ------------------------------------------------------------------------------------------------------------
 * Tier 1b -- block-level batch entry: the thin FFI for a host that keeps the reference's OWN frame / block /
 * section header parsing (frame.rs:6-85, block_decoder.rs:201-247, literals_section.rs:117-223,
 * sequence_section.rs:108-167) and ships compressed blocks.  It replaces the one call site of the hot path,
 * BlockDecoder::decompress_block (block_decoder.rs:97-197, called at :140-145 / :176-183), for many blocks of many
 * frames at once.  A descriptor carries what decompress_block has in hand when it calls decode_literals /
 * decode_sequences / execute_sequences.  The entropy tables are built on the GPU from the descriptions inside the
 * block content, so the "table pool" is implicit: Repeat / Treeless modes refer to the tables of the previous block
 * of the same frame (blocks of a frame are consecutive and in order), or to the frame's dictionary.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200z_block_desc {
    uint64_t src_off;             /* offset of the block CONTENT (after the 3-byte header) in `compressed`            */
    uint32_t content_size;        /* BlockHeader::content_size (block.rs:31-43)                                        */
    uint32_t block_type;          /* 0 Raw, 1 RLE, 2 Compressed                                                        */
    uint32_t decompressed_size;   /* BlockHeader::decompressed_size (Raw / RLE blocks)                                 */
    uint32_t last_block;
    /* what LiteralsSection::parse_from_header gave (literals_section.rs:9-28); checked against the content */
    uint32_t literals_type;       /* 0 Raw, 1 RLE, 2 Compressed, 3 Treeless                                            */
    uint32_t regenerated_size;
    uint32_t compressed_size;     /* 0 for Raw / RLE literals                                                          */
    uint32_t num_streams;         /* 1 or 4 (Compressed / Treeless), else 0                                            */
    /* what SequencesHeader::parse_from_header gave (sequence_section.rs:10-19) */
    uint32_t num_sequences;
    uint32_t modes;               /* the compression-modes byte (0 when num_sequences == 0)                            */
} b200z_block_desc;

typedef struct b200z_block_frame {
    uint64_t out_off;             /* where the frame's byte 0 goes inside `output`                                     */
    uint64_t out_cap;
    uint64_t window_size;         /* FrameHeader::window_size (frame.rs:116)                                           */
    const b200z_dict *dict;       /* dictionary in use (initial tables, offset history, content) or NULL               */
    uint32_t first_block;         /* index of the frame's first descriptor                                             */
    uint32_t num_blocks;
} b200z_block_frame;

typedef struct b200z_block_status {
    int32_t status;               /* 0, a b200z_error, or B200Z_BLOCK_NOT_REACHED (an earlier block of the frame failed) */
    int32_t stage;
    uint32_t out_size;            /* bytes this block added to the frame's output                                      */
    uint32_t reserved;
} b200z_block_status;
#define B200Z_BLOCK_NOT_REACHED (-1)

/* Decodes `nblocks` blocks of `nframes` frames.  `compressed` / `output` are host or device memory (B200Z_MEM_*).
 * Returns 0 when the submission ran; per-block outcomes in status[nblocks], per-frame totals in frame_out_size[nframes]
 * (either may be NULL).  B200Z_ERR_INVALID_ARGUMENT when a descriptor disagrees with the section headers found in the
 * block content. */
int b200z_decode_blocks_batch(b200z_ctx *ctx, const b200z_block_desc *blocks, size_t nblocks, const b200z_block_frame *frames,
                              size_t nframes, const uint8_t *compressed, size_t compressed_len, int compressed_mem, uint8_t *output,
                              size_t output_cap, int output_mem, b200z_block_status *status, uint64_t *frame_out_size);

/* ------------------------------------------------------------------------------------------------------------
 * Tier 2 -- mirror of ruzstd's FrameDecoder (decoding/frame_decoder.rs:154-627), GPU-backed.
 * Same names, argument meaning and error behaviour; `read_cb` has io::Read::read semantics.
 * ---------------------------------------------------------------------------------------------------------- */

/* BlockDecodingStrategy (frame_decoder.rs:96-100) */
#define B200Z_STRATEGY_ALL 0
#define B200Z_STRATEGY_UPTO_BLOCKS 1
#define B200Z_STRATEGY_UPTO_BYTES 2
#define B200Z_DEFAULT_MAX_WINDOW_SIZE (1024ull * 1024ull * 128ull) /* frame_decoder.rs:25 */

typedef struct b200z_frame_decoder b200z_frame_decoder;
int b200z_frame_decoder_new(b200z_ctx *ctx, b200z_frame_decoder **out);                    /* FrameDecoder::new :158 */
void b200z_frame_decoder_free(b200z_frame_decoder *d);
void b200z_frame_decoder_set_max_window_size(b200z_frame_decoder *d, uint64_t n);          /* :175 */
uint64_t b200z_frame_decoder_max_window_size(const b200z_frame_decoder *d);                /* :180 */
int b200z_frame_decoder_init(b200z_frame_decoder *d, b200z_read_fn read_cb, void *user);   /* init :190 */
int b200z_frame_decoder_reset(b200z_frame_decoder *d, b200z_read_fn read_cb, void *user);  /* reset :200 */
/* on B200Z_ERR_SKIP_FRAME from init/reset: the SkipFrame{length} payload (frame.rs:15-23) */
uint32_t b200z_frame_decoder_skip_frame_length(const b200z_frame_decoder *d);
/* a dictionary replaces the one of its ID for the frames reset after the call: the frame in progress keeps the one it started with */
int b200z_frame_decoder_add_dict(b200z_frame_decoder *d, const uint8_t *raw, size_t len);  /* decode_dict + add_dict :224 */
int b200z_frame_decoder_add_raw_content_dict(b200z_frame_decoder *d, uint32_t id, const uint8_t *content, size_t len); /* EXTENSION */
int b200z_frame_decoder_force_dict(b200z_frame_decoder *d, uint32_t dict_id);              /* :229 */
/* Deviation: after an error, decode_blocks (and decode_from_to, and a StreamingDecoder's read) returns that error again until the
 * decoder is reset.  The reference keeps no failed state and reads on from the next block header, with whatever tables the failed
 * block left half built; some such frames make it panic (tests/errcraft.py, reentries()). */
int b200z_frame_decoder_decode_blocks(b200z_frame_decoder *d, b200z_read_fn read_cb, void *user, int strategy,
                                      size_t n, int *finished);                            /* :309 */
long b200z_frame_decoder_read(b200z_frame_decoder *d, uint8_t *buf, size_t len);           /* impl Read :615 */
long b200z_frame_decoder_collect_to_writer(b200z_frame_decoder *d, b200z_write_fn write_cb, void *user); /* :393 */
size_t b200z_frame_decoder_can_collect(const b200z_frame_decoder *d);                      /* :409 */
int b200z_frame_decoder_is_finished(const b200z_frame_decoder *d);                         /* :284 */
size_t b200z_frame_decoder_blocks_decoded(const b200z_frame_decoder *d);                   /* :297 */
uint64_t b200z_frame_decoder_bytes_read_from_source(const b200z_frame_decoder *d);         /* :273 */
uint64_t b200z_frame_decoder_content_size(const b200z_frame_decoder *d);                   /* :246 */
int b200z_frame_decoder_get_checksum_from_data(const b200z_frame_decoder *d, uint32_t *out);  /* :254; 1 = Some */
int b200z_frame_decoder_get_calculated_checksum(const b200z_frame_decoder *d, uint32_t *out); /* :262; 1 = Some */
int b200z_frame_decoder_decode_from_to(b200z_frame_decoder *d, const uint8_t *src, size_t src_len, uint8_t *dst,
                                       size_t dst_len, size_t *read, size_t *written);     /* :439 */
int b200z_frame_decoder_decode_all(b200z_frame_decoder *d, const uint8_t *input, size_t input_len, uint8_t *output,
                                   size_t output_cap, size_t *written);                    /* :541 */
int b200z_frame_decoder_last_stage(const b200z_frame_decoder *d);
const char *b200z_frame_decoder_last_error_message(const b200z_frame_decoder *d);

/* ------------------------------------------------------------------------------------------------------------
 * Mirror of ruzstd's StreamingDecoder (decoding/streaming_decoder.rs:45-156): owns a source callback and a
 * frame decoder (its own, or a borrowed one = new_with_decoder).
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200z_streaming_decoder b200z_streaming_decoder;
int b200z_streaming_decoder_new(b200z_ctx *ctx, b200z_read_fn read_cb, void *user, b200z_streaming_decoder **out); /* :61 */
int b200z_streaming_decoder_new_with_decoder(b200z_read_fn read_cb, void *user, b200z_frame_decoder *dec,
                                             b200z_streaming_decoder **out);               /* :51 */
int b200z_streaming_decoder_new_with_max_window_size(b200z_ctx *ctx, b200z_read_fn read_cb, void *user,
                                                     uint64_t max_window_size, b200z_streaming_decoder **out); /* :72 */
long b200z_streaming_decoder_read(b200z_streaming_decoder *s, uint8_t *buf, size_t len, int *error); /* impl Read :118 */
b200z_frame_decoder *b200z_streaming_decoder_frame_decoder(b200z_streaming_decoder *s);    /* get at .decoder :46 */
/* into_frame_decoder :113 -- destroys the wrapper, returns the decoder (caller frees it unless it was borrowed) */
b200z_frame_decoder *b200z_streaming_decoder_into_frame_decoder(b200z_streaming_decoder *s);
void b200z_streaming_decoder_free(b200z_streaming_decoder *s);

/* ------------------------------------------------------------------------------------------------------------
 * Batch compressor -- ruzstd's encoding::{compress, compress_to_vec, FrameCompressor::compress} (encoding/mod.rs:24-67,
 * frame_compressor.rs:131-224) for many independent frames in one submission, every block of every frame encoded at once.
 * Frames are standard zstd: Single_Segment = 0, a 128 KiB window, Frame_Content_Size always present (smallest legal field;
 * the reference writes none), 128 KiB blocks, an optional content checksum (XXH64 seed 0, low 32 bits).  Blocks are RLE when
 * all their bytes are equal, else Compressed when that is smaller, else Raw; a Compressed block never refers to another
 * block's tables (no Treeless / Repeat modes, no repeat offsets).  The output need not equal the reference's byte for byte.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200z_compress_io {
    uint64_t src_off;   /* the frame's plaintext inside `input`                                  */
    uint64_t src_size;
    uint64_t dst_off;   /* where the frame goes inside `output`                                  */
    uint64_t dst_cap;   /* room reserved there; must be >= b200z_compress_bound(src_size)         */
} b200z_compress_io;

typedef struct b200z_compress_result {
    uint64_t dst_size;  /* bytes of the frame written at dst_off                                 */
    int32_t status;     /* 0 or b200z_error                                                      */
    uint32_t blocks;    /* blocks in the frame                                                   */
    uint32_t raw_blocks, rle_blocks;
    uint32_t has_checksum, checksum;
} b200z_compress_result;

/* CompressionLevel (encoding/mod.rs:24-67): Default = 2, Better = 3, Best = 4 are unimplemented!() in the reference */
#define B200Z_LEVEL_UNCOMPRESSED 0
#define B200Z_LEVEL_FASTEST 1
/* EXTENSION (not a ruzstd level; its output is not ruzstd's): the value after the reference's Best = 4.  Same framing, window,
 * blocks, compress bound and kernels as Fastest; a deeper parse and repeat offsets.  The parse keeps Fastest's blocks, 8 segments
 * per block, rounds of 32 positions and 5-byte minimum match, and adds per segment a table of the 6 most recent positions per
 * hash (seeded from 32 KiB before the segment), the segment's three most recent distinct offsets as candidates at every
 * position, and a lazy choice: the first position with a match competes with the next four, each candidate scored
 * 4 * length - floor(log2 offset) (a repeat scores 4 * length) less 3 per byte it starts later.  Each Compressed block codes an
 * offset as a repeat code where the decoder's offset history, tracked from the block's start with all three slots unknown,
 * names it; so no block depends on another block's encoding.  DESIGN.md section 4.4 states the rules and tests/clazy.py models
 * them byte for byte.  Accepted by the batch entries (with or without a dictionary and B200Z_FLAG_DICT_TABLES) and the stream
 * compressor; b200z_dict_finalize keeps the Fastest parse. */
#define B200Z_LEVEL_LAZY 5
/* context flag: b200z_compress_frames_batch records a CUDA event between its kernels and keeps each kernel's milliseconds
 * for b200z_compress_last_profile (profiling aid for bench.py; it synchronises anyway) */
#define B200Z_FLAG_PROFILE 2u
/* context flag: b200z_compress_frames_batch_dict with a formatted dictionary uses the dictionary's entropy tables in every frame's
 * first block: Treeless literals with its Huffman codes and Repeat for each of the LL / OF / ML tables, each only where it is
 * smaller (estimated, for the sequence tables) than the block's own tables.  Later blocks keep their own tables, so no block
 * depends on another's encoding.  Without the flag, or with a raw-content dictionary, the output is what it is without it.  The
 * encoder's view of the tables is built on the host by the dictionary's first use with the flag (no kernel launch) and kept
 * until b200z_dict_destroy. */
#define B200Z_FLAG_DICT_TABLES 4u

/* the largest frame b200z_compress_frames_batch can write for src_size bytes: src_size + 14 + 3 * max(1, ceil(src_size / 131072)) + 4 */
size_t b200z_compress_bound(size_t src_size);
/* Compresses `nframes` frames.  `input` / `output` are host or device memory (B200Z_MEM_*); `checksum` != 0 appends the
 * content checksum.  Returns 0 when the submission ran (results[nframes] filled).  Checked before any launch:
 * B200Z_ERR_INVALID_ARGUMENT for a range outside `input` / `output`, dst_cap < b200z_compress_bound(src_size), overlapping
 * destination ranges or an unknown level; B200Z_ERR_REFERENCE_WOULD_PANIC for the levels the reference does not implement.
 * Levels: Uncompressed, Fastest and the extension B200Z_LEVEL_LAZY. */
int b200z_compress_frames_batch(b200z_ctx *ctx, const uint8_t *input, size_t input_len, int input_mem,
                                const b200z_compress_io *frames, size_t nframes, int level, int checksum,
                                uint8_t *output, size_t output_cap, int output_mem, b200z_compress_result *results);
/* EXTENSION (ruzstd's FrameCompressor writes no dictionary ID and matches against no dictionary): compression against one
 * dictionary per submission.  The first 128 KiB of every frame may also match the last 128 KiB of the dictionary's content
 * (offsets stay within the 128 KiB window); the content checksum covers the frame's own plaintext.  A formatted dictionary's ID
 * goes into every frame header in the smallest field that holds it; a raw-content dictionary writes no ID (libzstd's
 * convention), so such frames are decoded with it forced (`forced_dict`, force_dict).  The encoder uses a formatted dictionary's
 * entropy tables only with B200Z_FLAG_DICT_TABLES, and never its repeat offsets.  The dictionary's match table is built on the ctx stream by its first use here
 * (one more kernel launch) and kept until b200z_dict_destroy.  dict == NULL writes exactly what b200z_compress_frames_batch
 * writes.  Besides that entry's checks: B200Z_ERR_INVALID_ARGUMENT for a dictionary created on another ctx and for
 * dst_cap < b200z_compress_bound_dict(src_size, dict), before any launch. */
int b200z_compress_frames_batch_dict(b200z_ctx *ctx, const uint8_t *input, size_t input_len, int input_mem,
                                     const b200z_compress_io *frames, size_t nframes, int level, int checksum, const b200z_dict *dict,
                                     uint8_t *output, size_t output_cap, int output_mem, b200z_compress_result *results);
/* b200z_compress_bound(src_size) + the size of the dictionary ID field the frame carries with `dict` (0, 1, 2 or 4 bytes) */
size_t b200z_compress_bound_dict(size_t src_size, const b200z_dict *dict);
/* EXTENSION: long-distance matching (libzstd's --long).  window_log lies in [B200Z_WINDOW_LOG_MIN, B200Z_WINDOW_LOG_MAX]; 17 is the
 * 128 KiB window every other entry writes. */
#define B200Z_WINDOW_LOG_MIN 17
#define B200Z_WINDOW_LOG_MAX 27
/* b200z_compress_frames_batch_dict with a window of 2^window_log bytes for long matches (EXTENSION; DESIGN.md section 4.11,
 * tests/cldm.py states the rule).  The regular parse keeps its 128 KiB reach; in every frame larger than 131072 bytes, content-defined
 * anchors (a gear hash of 64 bytes, about 1 in 128 positions, at most 1 in 16) find the nearest earlier anchor of the same frame
 * with the same 64-byte hash, and where its offset lies in (131072, 2^window_log] and 64 or more bytes match inside the anchor's
 * block, that match is forced into the parse.  Long matches never reach into the dictionary.  Each frame's Window_Descriptor
 * carries min(window_log, max(17, ceil(log2 src_size))), so a frame of 131072 bytes or fewer is exactly what window_log 17
 * writes, and window_log 17 is exactly b200z_compress_frames_batch_dict.  The compress bound is b200z_compress_bound_dict.  Besides
 * that entry's checks: B200Z_ERR_INVALID_ARGUMENT, before any launch, for window_log outside [17, 27] and for a window_log
 * above 17 at B200Z_LEVEL_UNCOMPRESSED.  Accepted at Fastest and LAZY.  With a frame larger than 131072 bytes and window_log > 17
 * the submission first runs the long-match kernels (k_lanchor twice, k_lscan, four k_lhist / k_lscan / k_lscatter passes of the
 * key sort, k_lcand, k_lblock: 17 launches, 3 when no anchor is found; counted in b200z_ctx_kernel_launches, not in
 * b200z_compress_last_profile's four stages), synchronising once to size the anchors' buffers: 44 bytes per anchor (at most one per 16 input bytes of those frames,
 * about one per 128 on typical data), 1 KiB per block of those frames and 8 bytes per block, kept with the context. */
int b200z_compress_frames_batch_long(b200z_ctx *ctx, const uint8_t *input, size_t input_len, int input_mem,
                                     const b200z_compress_io *frames, size_t nframes, int level, int checksum, const b200z_dict *dict,
                                     int window_log, uint8_t *output, size_t output_cap, int output_mem, b200z_compress_result *results);
int b200z_compress_num_stages(void);
const char *b200z_compress_stage_name(int stage);
/* each kernel's device milliseconds in the last b200z_compress_frames_batch run with B200Z_FLAG_PROFILE set */
int b200z_compress_last_profile(const b200z_ctx *ctx, float *stage_ms, size_t n);

/* ------------------------------------------------------------------------------------------------------------
 * Stream compressor -- mirror of ruzstd's FrameCompressor (encoding/frame_compressor.rs:75-276): one frame from a source of
 * unknown length (`read_cb`, io::Read::read semantics) to a drain (`write_cb`, io::Write::write_all over it), in bounded memory.
 * The frame is the reference's framing: magic, FHD 0x04 with the checksum or 0x00 without, Window_Descriptor 0x38 (128 KiB), no
 * Frame_Content_Size, 128 KiB blocks; a block is last only when a read returned 0 before it filled, so a source whose length is
 * a multiple of 128 KiB (0 included) ends with an empty last Raw block (01 00 00); then the low 32 bits of XXH64 (seed 0) of the
 * plaintext when the checksum is on.  Level Uncompressed writes Raw blocks, byte for byte the reference's frame, on the host
 * only (no kernel, no device copy).  Level Fastest writes every block's type and body as b200z_compress_frames_batch does for the
 * same block of the same input compressed as one frame, and so does level LAZY (EXTENSION) at LAZY.
 * The source is read into chunks of whole blocks: B200Z_PIPELINE_CHUNK_BYTES (read by _new) rounded down to a multiple of
 * 131072, at least 131072; 64 MiB by default.  At Fastest (and LAZY) each non-empty chunk is uploaded and compressed by three kernels
 * (k_cmatch, k_cenc, k_cassemble) on the ctx stream, counted in b200z_ctx_kernel_launches, while the host reads and hashes the
 * next chunk and writes the previous one: one write_cb pass per chunk (header in the first, trailer in the last), not per block.
 * Memory, allocated by the first Fastest compress and kept until _free, depends on the chunk C only.  Device: 2 * (C + 131072)
 * input, 2 * (C + 3 * C / 131072) output, and the compressor's staging for C / 131072 blocks (about 0.9 MB per block); about
 * 0.7 GB at 64 MiB.  Pinned host: 2 * C input and 2 * (C + 3 * C / 131072) output.
 * Errors: a read returning < 0 (or more than asked for), or a write returning <= 0, is an unwrap() panic in the reference; here
 * compress returns B200Z_ERR_REFERENCE_WOULD_PANIC (message in b200z_ctx_last_error_message), bytes already written stay
 * written, and the compressor stays usable.  Hashing and matching state reset with every compress.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200z_frame_compressor b200z_frame_compressor;
/* FrameCompressor::new :77.  B200Z_ERR_INVALID_ARGUMENT for a level outside 0-4 and B200Z_LEVEL_LAZY */
int b200z_frame_compressor_new(b200z_ctx *ctx, int level, int checksum, b200z_frame_compressor **out);
void b200z_frame_compressor_free(b200z_frame_compressor *fc);
int b200z_frame_compressor_set_compression_level(b200z_frame_compressor *fc, int level);   /* :263; 0-4 or LAZY, else INVALID_ARGUMENT */
int b200z_frame_compressor_compression_level(const b200z_frame_compressor *fc);            /* :273 */
/* EXTENSION: long-distance matches up to 2^window_log bytes back (b200z_compress_frames_batch_long's rule) from the next compress
 * on; window_log in [17, 27], else B200Z_ERR_INVALID_ARGUMENT.  The frame's Window_Descriptor is 2^window_log (its size is unknown
 * when the header is written).  Every block is what b200z_compress_frames_batch_long writes for the same block of the whole
 * input compressed as one frame at the same level and window_log, at any chunk size.  compress returns B200Z_ERR_INVALID_ARGUMENT,
 * before any read, for a window_log above 17 at level Uncompressed.  Above 17 each chunk goes to the device behind the last
 * H = 2^window_log + 128 bytes before it (a device-to-device copy from the other slot), and the long-match kernels run on the
 * spans of that history and the chunk (S = ceil(H / 131072) + C / 131072 of them) before k_cmatch.  Memory at window_log > 17,
 * allocated by the first compress that needs it and kept until _free: device input 2 * (H + C) in place of 2 * (C + 131072),
 * the anchors' buffers at the density bound, 44 * 8192 * S bytes, 1028 * S + 8 * C / 131072 bytes of counts, and 32 * S bytes
 * of spans per descriptor slot (two on the device, two pinned); about 0.83 GB more device memory than at 17 for window_log 27 and C = 64 MiB. */
int b200z_frame_compressor_set_window_log(b200z_frame_compressor *fc, int window_log);
int b200z_frame_compressor_window_log(const b200z_frame_compressor *fc);
/* compress :131-224: one frame from read_cb to write_cb.  B200Z_ERR_REFERENCE_WOULD_PANIC for levels 2-4 before any read, write
 * or launch.  result (may be NULL): dst_size = bytes written, blocks (the trailing empty block included), raw / RLE blocks
 * (the empty block is Raw), has_checksum, checksum */
int b200z_frame_compressor_compress(b200z_frame_compressor *fc, b200z_read_fn read_cb, void *read_user, b200z_write_fn write_cb,
                                    void *write_user, b200z_compress_result *result);

/* ------------------------------------------------------------------------------------------------------------
 * Raw-content dictionary trainer -- EXTENSION in place of ruzstd::dictionary::create_raw_dict_from_source /
 * create_raw_dict_from_dir (dictionary/mod.rs:76,127, feature dict_builder).  The reference cannot serve as the model: its
 * reservoir sample reads the whole source to EOF (reservoir.rs:83-104), so its epoch loop (mod.rs:171-188) reads nothing and
 * every source of 16 bytes or more gives an empty dictionary; pick_best_segment (cover.rs:71-95) also ignores its epoch.  This
 * entry implements what the reference's comments describe, exactly (DESIGN.md section 4.5): the local-maximum-coverage
 * method over 16-byte k-mers with every k-mer of the collection counted (2^22 hashed slots), epochs as compute_epoch_info with
 * the collection's byte count, the best segment of every epoch scored by the distinct k-mers it holds (a k-mer that leaves its
 * sample counts nothing), the counts of a chosen segment's k-mers zeroed for later epochs, and the segments concatenated by
 * ascending score (ties by epoch), the last dict_size bytes kept.  n < 16 returns the input itself; dict_size == 0 returns
 * nothing.  The result does not depend on the schedule.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200z_dict_segment {
    uint64_t src_off;   /* the segment's first byte in `samples`                                  */
    uint64_t score;     /* sum of the counts of its distinct k-mers when it was chosen            */
    uint32_t epoch;
    uint32_t size;      /* bytes: min(segment_size, samples_len, the epoch's length)              */
} b200z_dict_segment;

/* Trains on `samples` (host or device memory, B200Z_MEM_*), cut into nsamples samples of sample_sizes[] bytes (NULL: one
 * sample; nsamples is then ignored), and writes the dictionary to the host buffer `dict` (*dict_len bytes) and, when `segments`
 * is not NULL, one record per epoch in epoch order (*nsegments).  segment_size 0 means 2048, the reference's default.  Checked
 * before any launch, B200Z_ERR_INVALID_ARGUMENT: segment_size outside [16, 65536], sample sizes that do not sum to samples_len,
 * samples_len >= 2^32, dict_cap below what will be written (samples_len when it is below 16, else min(dict_size, the sum of the
 * epochs' segment sizes)), or segments_cap below the number of epochs.  Kernels: k_dtcount, k_dtprev, then one k_dtepoch per
 * epoch, all on the ctx stream and counted in b200z_ctx_kernel_launches. */
int b200z_dict_train_raw(b200z_ctx *ctx, const uint8_t *samples, size_t samples_len, int samples_mem, const size_t *sample_sizes,
                         size_t nsamples, size_t dict_size, size_t segment_size, uint8_t *dict, size_t dict_cap, size_t *dict_len,
                         b200z_dict_segment *segments, size_t segments_cap, size_t *nsegments);

/* ------------------------------------------------------------------------------------------------------------
 * Dictionary finalizer -- EXTENSION, the counterpart of libzstd's ZDICT_finalizeDictionary (ruzstd has none): turns dictionary
 * content (for instance b200z_dict_train_raw's) into a zstd-format dictionary that carries an ID and entropy tables, which
 * Dictionary::decode_dict (b200z_dict_create), ruzstd and libzstd load.  The statistics come from the GPU: the first block (at
 * most 128 KiB) of every sample is parsed against the content by the compressor's own parse (k_cmatch, with the content's match
 * table from k_cdict), and k_dstats counts the literal bytes and the LL / ML / OF codes of every block that is not RLE (u64
 * totals, integer atomics: the result does not depend on the schedule).  The samples go through in submissions of a bounded
 * number of blocks.  On the host, every symbol gets a count of at least 1 (literals 0-255, LL 0-35, ML 0-52, OF 0 up to
 * floor(log2(content_len + 131072))), and the tables are written at accuracy logs OF 8, ML 9, LL 9 with Huffman codes of at
 * most 11 bits.  Layout: magic 0xEC30A437, ID, Huffman description, OF, ML, LL descriptions, repeat offsets 1, 4, 8, content.
 * When the header and the content exceed dict_cap, the content's LAST bytes are kept (the trainer puts its best segments
 * last).  dict_id 0 derives the ID as libzstd does: (XXH64(content written, seed 0) mod (2^31 - 32768)) + 32768.
 * ---------------------------------------------------------------------------------------------------------- */
/* an upper bound on the header (everything before the content) b200z_dict_finalize writes */
#define B200Z_DICT_HEADER_MAX 328
/* Finalizes `content` (host memory) on `samples` (host or device memory, B200Z_MEM_*) cut into nsamples samples of
 * sample_sizes[] bytes; nsamples == 0 is legal and gives the tables of flat counts.  Writes the dictionary to the host buffer
 * `dict` (*dict_len bytes).  Checked before any launch, B200Z_ERR_INVALID_ARGUMENT: content_len below 8 or >= 2^31, dict_cap below
 * B200Z_DICT_HEADER_MAX + 8, sample sizes that do not sum to samples_len, dict_id >= 2^31 (the format reserves those IDs; libzstd
 * and ruzstd accept them, so this library does not write them).  Kernels: k_cdict once, then k_cmatch and k_dstats per
 * submission, all on the ctx stream and counted in b200z_ctx_kernel_launches.  Device memory: the compressor's per-block staging
 * for min(nsamples, 2048) blocks (about 0.9 MB per block whatever the samples' sizes, so up to about 1.8 GB), a copy of host samples,
 * and 0.5 MB for the content's match table; all of it stays with the ctx (reused by later compressions) until b200z_ctx_destroy. */
int b200z_dict_finalize(b200z_ctx *ctx, const uint8_t *content, size_t content_len,
                        const uint8_t *samples, size_t samples_len, int samples_mem, const size_t *sample_sizes, size_t nsamples,
                        uint32_t dict_id, uint8_t *dict, size_t dict_cap, size_t *dict_len);
/* Host only: what b200z_dict_finalize writes for the statistics counts[377] (literal bytes 0-255, LL codes 0-35, ML codes 0-52,
 * OF codes 0-31, in that order), with the same argument checks */
int b200z_debug_dict_from_counts(const uint64_t counts[377], const uint8_t *content, size_t content_len, uint32_t dict_id,
                                 uint8_t *dict, size_t dict_cap, size_t *dict_len);

/* ------------------------------------------------------------------------------------------------------------
 * Seekable archives -- EXTENSION (ruzstd has no seekable support): the zstd seekable format of zstd's contrib/seekable_format.
 * An archive is independent zstd frames back to back followed by one skippable frame that holds the seek table:
 *   Skippable_Magic_Number u32 LE 0x184D2A5E, Frame_Size u32 LE = n * (8 or 12) + 9, then per frame Compressed_Size u32,
 *   Decompressed_Size u32 and, with the Checksum_Flag, the low 32 bits of XXH64 (seed 0) of its plaintext; then the footer
 *   Number_Of_Frames u32 n, Seek_Table_Descriptor u8 (bit 7 Checksum_Flag, bits 6-2 reserved, must be 0) and
 *   Seekable_Magic_Number u32 LE 0x8F92EAB1, the archive's last 9 bytes.
 * Every zstd decoder reads an archive as concatenated frames and a skippable frame (decode_all, tiers 1c and 1d); a reader that
 * knows the table decodes only the frames a byte range touches (b200z_seekable_read_ranges).  DESIGN.md section 4.10.
 * ---------------------------------------------------------------------------------------------------------------------------- */
/* blocks (128 KiB each, a frame's last one shorter) b200z_compress_seekable compresses per submission: a group holds whole frames,
 * as many as fit in this many blocks, or one frame when a frame alone has more.  The device memory the call holds depends on it
 * (and on frame_size when one frame has more blocks), not on the archive: the compressor's staging of about 0.9 MB per block of the
 * largest group -- at most 2048 blocks (1.8 GB), and never more than the input's own blocks -- and with host memory that group's
 * input (up to 256 MiB) and its frames' bounds (b200z_compress_bound_dict each). */
#define B200Z_SEEKABLE_GROUP_BLOCKS 2048
#define B200Z_SEEKABLE_MAX_FRAME_SIZE (1u << 30)

/* b200z_compress_bound_dict of every frame (frame_size bytes each, the last one shorter) plus the seek table (17 bytes and 8 per
 * frame, 12 with `checksum`); 0 when frame_size is 0 or above B200Z_SEEKABLE_MAX_FRAME_SIZE */
size_t b200z_seekable_bound(size_t src_size, size_t frame_size, int checksum, const b200z_dict *dict);
/* Compresses `input` into a seekable archive at `output` (host or device memory, B200Z_MEM_*); *written = the archive's bytes.
 * The input is cut into frames of frame_size bytes (the last one shorter; an empty input gives no frame, and the archive is the
 * table alone).  Every frame is byte for byte what b200z_compress_frames_batch_dict writes for that piece with the same level,
 * checksum, dictionary and B200Z_FLAG_DICT_TABLES; the frames lie back to back from output[0], the table behind them.  With
 * `checksum` the table carries each frame's checksum (the one its trailer holds) and sets the Checksum_Flag.  The frames go
 * through in groups of whole frames (B200Z_SEEKABLE_GROUP_BLOCKS); host input is uploaded and host output downloaded group by
 * group.  Kernels per group: those of b200z_compress_frames_batch_dict (k_cmatch, k_cenc, k_cxxh64 with `checksum`, k_cassemble;
 * none of the first two at Uncompressed) plus k_cscan; then one k_cseek; all counted in b200z_ctx_kernel_launches.  Checked before
 * any launch: what b200z_compress_frames_batch_dict checks (levels, dictionary), and B200Z_ERR_INVALID_ARGUMENT for frame_size 0 or
 * above B200Z_SEEKABLE_MAX_FRAME_SIZE, more than 2^32 - 1 frames, or output_cap < b200z_seekable_bound. */
int b200z_compress_seekable(b200z_ctx *ctx, const uint8_t *input, size_t input_len, int input_mem, size_t frame_size, int level,
                            int checksum, const b200z_dict *dict, uint8_t *output, size_t output_cap, int output_mem, size_t *written);

/* A seekable archive from a reader to a writer, for sources too large to hold.
 *   Output:  write_cb receives exactly what b200z_compress_seekable writes for the whole source with the same frame_size, level,
 *            checksum, dictionary and B200Z_FLAG_DICT_TABLES, whatever the chunk size and however the source splits its reads: a
 *            frame's bytes depend on its piece and the dictionary only, and the table is written by one k_cseek at the end.
 *   Source:  read_cb as the stream compressor reads it: a frame is cut after frame_size bytes or where a read returns 0 (the end of
 *            the source, so only the last frame is shorter); an empty source gives the table alone.
 *   Groups:  with C = B200Z_PIPELINE_CHUNK_BYTES (read by each call; 64 MiB by default) a group is the most whole frames that hold
 *            at most C bytes and at most B200Z_SEEKABLE_GROUP_BLOCKS blocks, or one frame when a frame alone is larger: G =
 *            max(1, min(C / frame_size, B200Z_SEEKABLE_GROUP_BLOCKS / blocks per frame)) * frame_size <= max(C, frame_size) bytes.
 *            Two slots: while group k compresses on the ctx stream, the calling thread reads group k + 1 and writes group k - 1;
 *            uploads go on one copy stream and downloads on another.  Each group's frames are packed from its slot's byte 0 by
 *            k_cscan behind a running-size word of the slot's own; the host learns the packed size from that word's download.
 *   Kernels: per group, those of a b200z_compress_seekable group (k_cmatch, k_cenc, k_cxxh64 with `checksum`, k_cscan,
 *            k_cassemble; none of the first two at Uncompressed); then one k_cseek; all counted in b200z_ctx_kernel_launches.
 *   Memory:  kept by the context and sized by the first group, the largest one the source has.  Device: per slot G input, the
 *            bounds of G's frames (b200z_compress_bound_dict each) and 32 bytes per frame and 24 per block of descriptors; shared,
 *            the compressor's staging of about 0.9 MB per block of G.  Pinned host: per slot G input and the bounds of G's frames.
 *            What grows with the source is the seek table.  With E = 8 bytes per frame (12 with `checksum`): the entries on the
 *            device, in an array doubled when full, so at most 2 * E per frame after the call; during it the outgrown arrays are
 *            kept until it ends (freeing one earlier would wait for the whole device), so at most 4 * E per frame, each array its
 *            own allocation.  At the end the table frame (17 bytes + E per frame) is written on the device, into a buffer the
 *            context keeps (up to 1.5 times that size, as the compressor's output staging grows), and copied to pageable host
 *            memory of its size while it is written.  Each group's download takes its frames' bounds (about the group's input),
 *            not only their packed bytes, so that no host wait stands between the packed size and the bytes.
 *   Checks:  before any read, write or launch, as b200z_compress_seekable checks them: B200Z_ERR_REFERENCE_WOULD_PANIC for levels
 *            2-4; B200Z_ERR_INVALID_ARGUMENT for other unknown levels, a dictionary of another context, no callback, and frame_size
 *            0 or above B200Z_SEEKABLE_MAX_FRAME_SIZE.  A source that gives more than 2^32 - 1 frames fails with
 *            B200Z_ERR_INVALID_ARGUMENT when it gets there.
 *   Errors:  a read returning < 0 or more than asked for, or a write returning <= 0, is B200Z_ERR_SEEKABLE_IO, with a message
 *            naming the callback and the archive offset.  Bytes already written stay written, nothing is left in flight, and the
 *            context stays usable.  `result` (may be NULL) says what was read and written either way. */
typedef struct b200z_seekable_stream_result {
    uint64_t read;      /* plaintext bytes taken from the source             */
    uint64_t written;   /* archive bytes handed to write_cb (table included) */
    uint64_t frames;    /* frames in the archive                             */
    uint64_t groups;    /* GPU submissions the call ran                      */
} b200z_seekable_stream_result;
int b200z_compress_seekable_stream(b200z_ctx *ctx, b200z_read_fn read_cb, void *read_user, b200z_write_fn write_cb, void *write_user,
                                   size_t frame_size, int level, int checksum, const b200z_dict *dict,
                                   b200z_seekable_stream_result *result);

/* An open archive: its table, parsed and checked.  It borrows the archive (host or device memory), which the caller keeps alive and
 * unchanged until b200z_seekable_close; of a device archive only the table is copied to the host.  B200Z_ERR_SEEKABLE_TABLE, with
 * the rule in b200z_ctx_last_error_message, when the footer magic, the reserved bits, the skippable magic or Frame_Size is wrong,
 * when the table does not lie inside the archive, or when the entries' Compressed_Size do not add up to the table's offset. */
typedef struct b200z_seekable b200z_seekable;
typedef struct b200z_seek_frame {
    uint64_t c_off, c_size;   /* the frame's bytes in the archive                                                      */
    uint64_t d_off, d_size;   /* its plaintext in the archive's content (the Decompressed_Size before it, summed)      */
    uint32_t has_checksum;    /* the table carries checksums                                                           */
    uint32_t checksum;
} b200z_seek_frame;
int b200z_seekable_open(b200z_ctx *ctx, const uint8_t *archive, size_t len, int mem, b200z_seekable **out);
/* pread semantics: up to len bytes of the archive at offset into buf; returns the bytes read (0 at the end), < 0 on error */
typedef long (*b200z_read_at_fn)(void *user, uint64_t offset, uint8_t *buf, size_t len);
/* An archive of `len` bytes behind a positional-read callback (a file too large to hold, for instance).  Open reads the archive's
 * last 9 bytes (the footer), the table frame's 8-byte header (checked against the footer before anything of the table's size is
 * allocated or read) and then the table frame, nothing else, and checks them as b200z_seekable_open does, with the same
 * B200Z_ERR_SEEKABLE_TABLE messages; B200Z_ERR_OUT_OF_MEMORY when a well-formed table does not fit in host memory.  read_at and `user` must stay valid until b200z_seekable_close.  The handle works with
 * _num_frames, _content_size, _frame and b200z_seekable_read_ranges as a host archive's does: the same plan, one batch submission,
 * k_range_gather and launch counts, and the same results.  The only difference is where the touched frames' bytes come from: each
 * run of touched frames adjacent in the archive is fetched by one read_at call (partial reads are retried until a read returns 0)
 * into the pinned buffer a host archive's frames are gathered to.  A call holds what a host-archive call holds (the touched
 * frames' compressed bytes in pinned memory, the slots and the scratch), never the archive.  A read_at that fails (< 0, or more
 * than asked for) or comes up short is B200Z_ERR_SEEKABLE_IO, at open or before any launch of read_ranges; the handle stays
 * usable. */
int b200z_seekable_open_source(b200z_ctx *ctx, b200z_read_at_fn read_at, void *user, uint64_t len, b200z_seekable **out);
uint64_t b200z_seekable_num_frames(const b200z_seekable *s);
uint64_t b200z_seekable_content_size(const b200z_seekable *s);
int b200z_seekable_frame(const b200z_seekable *s, uint64_t i, b200z_seek_frame *out);
void b200z_seekable_close(b200z_seekable *s);

/* one range: plaintext [offset, offset + length) of the archive's content, written at output + out_off */
typedef struct b200z_range {
    uint64_t offset, length, out_off;
} b200z_range;
typedef struct b200z_range_result {
    int32_t status;                /* 0, the b200z_error of the first failing frame it needs (in content order), or
                                      B200Z_ERR_SEEKABLE_FRAME_SIZE when that frame decoded to another size than its entry */
    int32_t stage;                 /* b200z_stage of the error                                                            */
    int64_t error_frame;           /* the archive frame that failed, -1 when none                                          */
    uint64_t frames;               /* archive frames the range touches                                                     */
    uint64_t checksum_mismatches;  /* B200Z_FLAG_CHECKSUM: touched frames whose GPU checksum differs from their table entry
                                      or from their own trailer (reported, never enforced)                                 */
} b200z_range_result;
/* Reads `n` ranges into `output` (host or device memory).  Checked before any work, B200Z_ERR_INVALID_ARGUMENT: a range that
 * reaches past the content size or past output_cap, and ranges whose output slots overlap (ranges may overlap in the content).
 * Every frame the ranges touch is decoded once, in one submission of the batch decoder (b200z_batch_prepare / _run with
 * b200z_frame_io built from the table; `dicts`, `forced_dict` and `max_window_size` as for b200z_decode_frames_batch) with
 * out_cap = its Decompressed_Size: a frame that lies wholly inside a range is decoded in place, in the first such range's slot (the
 * decoder writes a frame's [out_off, out_off + out_cap) only); any other touched frame -- at most two per range -- into device
 * scratch.  k_range_gather then copies each range's other bytes from scratch or from another range's slot.  Host archives: only
 * the touched frames' bytes are gathered and uploaded.  Host output: the ranges' slots are staged on the device and copied to
 * their out_off; no other byte of `output` is written.  With B200Z_FLAG_CHECKSUM, device output must be readable 8 bytes past a
 * slot that ends at output_cap.  Kernels: the batch pass (b200z_batch_info[6]; with a device archive also the planner's two k_walk
 * launches), and one k_range_gather when some range has bytes outside its in-place frames; none when no range touches a frame.
 * Returns 0 when the call ran (outcomes in results[n]). */
int b200z_seekable_read_ranges(b200z_seekable *s, const b200z_range *ranges, size_t n, const b200z_dict *const *dicts, size_t ndicts,
                               const b200z_dict *forced_dict, uint64_t max_window_size, uint8_t *output, size_t output_cap, int output_mem,
                               b200z_range_result *results);

/* Host-only view of the read plan (no context, no device; for CPU tests): the archive's table (host memory, checked as by
 * b200z_seekable_open) and the ranges (checked as by b200z_seekable_read_ranges, with no output_cap).  plan_frames: every touched
 * frame once, by ascending frame index; range = the range it is decoded in place for (dst_off in the output), or -1 (dst_off in
 * scratch: the frames that are not in place, by ascending index, each at a multiple of 16).  pieces: per range in call order, per
 * touched frame by ascending index that is not in place for that range, the bytes it takes from the frame: len bytes from src_off
 * (scratch, or the output when the frame is in place for another range) to dst_off in the output.  *scratch_bytes: the scratch's
 * size.  *nframes / *npieces are set even when the caps are too small (then nothing is written; B200Z_ERR_INVALID_ARGUMENT). */
typedef struct b200z_seek_plan_frame {
    uint64_t frame, dst_off;
    int64_t range;
} b200z_seek_plan_frame;
typedef struct b200z_seek_plan_piece {
    uint64_t dst_off, src_off, len;
    uint32_t from_scratch, range;
} b200z_seek_plan_piece;
int b200z_debug_seekable_plan(const uint8_t *archive, size_t len, const b200z_range *ranges, size_t n, b200z_seek_plan_frame *frames,
                              size_t frames_cap, size_t *nframes, b200z_seek_plan_piece *pieces, size_t pieces_cap, size_t *npieces,
                              uint64_t *scratch_bytes);

/* XXH64(seed 0) of a host buffer -- the content-checksum hash the reference feeds on drain
 * (decode_buffer.rs:42,225,290,301); exposed so bindings can verify checksums like tests/decode_corpus.rs:61-74 */
uint64_t b200z_xxh64(const uint8_t *data, size_t len);

#ifdef __cplusplus
}
#endif
#endif /* B200ZSTD_H */
