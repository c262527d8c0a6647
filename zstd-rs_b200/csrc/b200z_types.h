// b200z_types.h -- POD layouts shared by the host planner and the CUDA kernels.
//
// Data layout in HBM (DESIGN.md section 3):
//   input      : all frames of a submission, byte-for-byte as on the wire (never re-packed)
//   BlockDesc  : one 128-byte descriptor per zstd block, written by the host planner (plan.cpp)
//   HufSlot    : GPU-resident huff0 LUT (ruzstd huff0::HuffmanTable.decode, huff0_decoder.rs:57-74)
//   FseTab     : GPU-resident FSE LUT (ruzstd fse::FSETable.decode, fse_decoder.rs:59-83), one per LL/OF/ML
//   literals   : scratch, regenerated literals of every Compressed/Treeless literals section
//   sequences  : scratch, 3 x u32 per sequence (ruzstd blocks::sequence_section::Sequence {ll, ml, of}) in PREFIX form:
//                {out_end, lit_end, of}: out_end = sum of (ll + ml), lit_end = sum of ll over the block's sequences up to and
//                including this one (mod 2^32), of = the offset after do_offset_history, symbolic when it depends on the
//                repeat-offset history at the block's start (seq_sym_* below); or the raw offset_value when the block is
//                flagged AUX_RAW_OFFSETS
//   output     : plaintext, each frame at the caller's out_off
#pragma once
#include <stdint.h>

// functions compiled for both the device and the host (tables.cuh, framing.cuh)
#ifdef __CUDACC__
#define B200Z_HD __host__ __device__ __forceinline__
#define B200Z_HDN __host__ __device__
#else
#define B200Z_HD inline
#define B200Z_HDN
#endif

namespace b200z {

// ---- block types / literal types as on the wire (block_decoder.rs:259-268, literals_section.rs:226-235)
enum : uint32_t { BT_RAW = 0, BT_RLE = 1, BT_COMPRESSED = 2 };
enum : uint32_t { LT_RAW = 0, LT_RLE = 1, LT_COMPRESSED = 2, LT_TREELESS = 3 };
// sequence compression modes (blocks/sequence_section.rs:49-63)
enum : uint32_t { MODE_PREDEFINED = 0, MODE_RLE = 1, MODE_FSE = 2, MODE_REPEAT = 3 };

constexpr uint32_t HUF_MAX_BITS = 11;         // huff0_decoder.rs:9
constexpr uint32_t HUF_TABLE_ENTRIES = 2048;  // 1 << 11
constexpr uint32_t FSE_MAX_ENTRIES = 512;

// ---- symbolic offsets.  k_fse decodes every block independently, so the repeat-offset history at a block's start
// (scratch.rs:22,44; carried from the previous block of the frame) is unknown to it: do_offset_history
// (sequence_execution.rs:59-118) runs on SYMBOLS.  A 32-bit value is either a concrete offset (< 2^30) or
//   tag << 30 | d   (tag 1..3): "history slot (tag - 1) at the start of this block, minus d, saturating at 0"
// (the only arithmetic the reference does on a history value is the saturating `- 1` of sequence_execution.rs:74).
// The execution kernels resolve symbols with the frame's actual history in O(1) per sequence, in parallel.
// A block that contains an offset code >= 30 (concrete values would collide with the tags) is decoded by the exact
// path, which emits raw offset_values and flags the block AUX_RAW_OFFSETS.
constexpr uint32_t SEQ_SYM_SHIFT = 30;
constexpr uint32_t SEQ_SYM_DMASK = (1u << SEQ_SYM_SHIFT) - 1u;
__host__ __device__ inline uint32_t seq_sym_resolve(uint32_t v, uint32_t h0, uint32_t h1, uint32_t h2) {
    const uint32_t tag = v >> SEQ_SYM_SHIFT;
    if (tag == 0) return v;
    const uint32_t h = tag == 1 ? h0 : (tag == 2 ? h1 : h2), d = v & SEQ_SYM_DMASK;
    return h > d ? h - d : 0u;
}
// BlockAux.flags
constexpr uint32_t AUX_RAW_OFFSETS = 1u;   // `of` holds raw offset_values (exact path of k_fse); hist_after is not valid
constexpr uint32_t AUX_WIDE = 2u;          // a prefix sum reached 2^31: positions are only meaningful as differences
constexpr uint32_t RESUME_SKIP = 0xFFFFFFFFu;   // resume[f]: nothing (left) for k_exec in this frame

// huff0 LUT, split so that it costs 3 KiB of shared memory per block instead of 4 (occupancy: every block of a
// 1 GiB submission is in flight at once): sym[i] = symbol, nb4[i >> 1] holds the 4-bit code length of entries
// 2k (low nibble) and 2k+1 (high nibble).   (huff0_decoder.rs:389-394 Entry{symbol,num_bits})
struct alignas(16) HufSlot {
    uint32_t max_bits;  // 0 = uninitialised (literals_section_decoder.rs:61-63)
    uint32_t status;    // build error (b200z_error) or 0
    uint32_t pad[2];
    uint8_t sym[HUF_TABLE_ENTRIES];
    uint8_t nb4[HUF_TABLE_ENTRIES / 2];
};
__host__ __device__ inline void huf_set(HufSlot *s, uint32_t i, uint32_t symbol, uint32_t nb) {
    s->sym[i] = (uint8_t)symbol;
    uint8_t o = s->nb4[i >> 1];
    s->nb4[i >> 1] = (i & 1u) ? (uint8_t)((o & 0x0Fu) | (nb << 4)) : (uint8_t)((o & 0xF0u) | nb);
}
__host__ __device__ inline uint32_t huf_nb(const uint8_t *nb4, uint32_t i) { return (nb4[i >> 1] >> ((i & 1u) * 4u)) & 15u; }

// FSE LUT, 16 bits per state so that LL + ML + OF of one block cost 2.5 KiB of shared memory:
//   entry = f | symbol << 10,   f = (1 << (log - num_bits)) | (base_line >> num_bits)
// base_line is always a multiple of 2^num_bits (fse_decoder.rs:340-366: baselines are whole slices), so
//   num_bits = log - floor(log2 f),  base_line = (f - 2^floor(log2 f)) << num_bits     (fse_decoder.rs:312-320 Entry)
// An RLE mode is stored as log = 0, e[0] = {f = 1, symbol}: reading 0 bits always lands on entry 0, which is
// what decode_sequences_with_rle does by substituting the constant code (sequence_section_decoder.rs:74-88).
struct alignas(16) FseTab {
    uint32_t log;     // accuracy_log, 0 for RLE
    uint32_t valid;   // 0 = never built (FSEDecoderError::TableIsUninitialized, fse_decoder.rs:33-35)
    uint32_t is_rle;
    uint32_t pad;
    uint16_t e[FSE_MAX_ENTRIES];
};
struct alignas(16) FseSlot { FseTab ll, of, ml; };

__host__ __device__ inline uint16_t fse_pack16(uint32_t log, uint32_t base, uint32_t nb, uint32_t sym) {
    return (uint16_t)(((1u << (log - nb)) | (base >> nb)) | (sym << 10));
}
__host__ __device__ inline uint32_t fse_pack(uint32_t base, uint32_t nb, uint32_t sym) { return base | (nb << 16) | (sym << 24); }

// One descriptor per block; everything the reference derives in decompress_block before calling the three hot
// stages (block_decoder.rs:97-181): literals header fields, sequence header fields, where each payload starts,
// and which table every section decodes with (Treeless / Repeat resolved to the defining slot by the planner).
struct alignas(16) BlockDesc {
    uint64_t src_off;        // offset of the block CONTENT in the input buffer (after the 3-byte header)
    uint64_t lit_buf_off;    // offset into the literals scratch (Compressed/Treeless literals only)
    uint64_t seq_buf_off;    // offset into the sequence scratch, in sequences
    uint32_t src_size;       // Block_Size (content bytes; 1 for RLE)
    uint32_t frame;          // index of the owning frame in this submission
    uint32_t btype;          // BT_*
    uint32_t raw_size;       // Raw/RLE: decompressed size
    uint32_t lit_type;       // LT_*
    uint32_t nstreams;       // 1 or 4 (Compressed/Treeless)
    uint32_t regen_size;     // literals regenerated size
    uint32_t lit_comp_size;  // literals compressed size (incl. tree description and jump table)
    uint32_t lit_off;        // offset of the literals payload inside the block content
    uint32_t seq_off;        // offset of the sequences payload (after the 1-4 byte header) inside the block content
    uint32_t nseq;           // number of sequences
    uint32_t modes;          // compression modes byte
    uint32_t host_status;    // error the planner found for this block (host_status()), 0 = none
    uint32_t block_in_frame; // ordinal of the block inside its frame
    uint32_t last;           // last block of the frame
    uint32_t pad0[5];
    const HufSlot *huf;      // table the literals decode with (own slot when lit_type == LT_COMPRESSED)
    HufSlot *huf_build;      // where a new Huffman table is built, or null
    const FseTab *ll, *of, *ml;  // tables the sequences decode with (null = uninitialised)
    FseSlot *fse_build;      // where new LL/OF/ML tables (FSE or RLE modes) are built, or null
};

// Per-block results written by the kernels
struct alignas(16) BlockAux {
    uint32_t status;         // literals-stage status (mk_status), 0 = ok
    uint32_t out_size;       // decompressed size of the block (known after sequence decode)
    uint32_t lit_streams_off;// offset inside the block content where the jump table / single stream starts
    uint32_t seq_bits_off;   // offset inside the block content where the sequence bitstream starts
    uint32_t sum_ll;         // sum of literal lengths over the block's sequences (mod 2^32)
    uint32_t seq_status;     // sequence-stage status (mk_status), 0 = ok; valid once `ready` is set
    uint32_t hist_after[3];  // offset history after the block (symbolic, seq_sym_*), unless AUX_RAW_OFFSETS
    uint32_t flags;          // AUX_*
    uint32_t ready;          // 1 once the block's sequence stage is over (k_fse): k_exec, launched as k_fse's programmatic
                             // dependent, starts a frame's block as soon as this is set (block-granular hand-off)
    uint32_t progress;       // sequences whose records k_fse's fast path has published so far (monotone; k_exec consumes them as they
                             // appear).  If the fast path gives the block up afterwards, the exact path rewrites the records with
                             // raw offsets and sets AUX_RAW_OFFSETS: k_exec then rolls the block back and runs it again.
};

// Per-frame state: carried between submissions for the streaming mirror, fresh for batch frames.
// offset_hist: scratch.rs:22,44 ; total_output_counter: decode_buffer.rs:14 ; produced/drained give
// DecodeBuffer::len() (decode_buffer.rs:58) = produced - drained.
struct alignas(16) FrameState {
    uint32_t hist[3];
    uint32_t status;          // first error: code | stage << 16
    uint64_t produced;        // bytes of this frame written to the output buffer so far
    uint64_t drained;         // bytes the host already drained (streaming); offsets reach back to `drained`
    uint64_t counter;         // total_output_counter (quirk: Raw/RLE blocks and fully-in-dict matches not counted)
    uint32_t error_block;     // block_in_frame of the failing block
    uint32_t blocks_done;     // blocks fully executed
    uint64_t xxh64;           // XXH64(seed 0) of the plaintext, when the checksum stage ran
    uint64_t pad;
};

// What the stream decoder (tier 1d) carries on the device into a submission whose first frame continues from the one before:
// the frame's plaintext bytes before the submission (k_carry), and, with the checksum, its XXH64 accumulators after `stripes`
// whole 32-byte stripes (k_xxh64_stream).  The carried tail of the frame's output holds the bytes hashed after those stripes.
struct alignas(16) StreamCarry {
    uint64_t v[4];
    uint64_t stripes;
    uint64_t total;
};

struct alignas(16) FrameDesc {
    uint64_t out_off;         // where the frame's byte 0 lives in the output buffer
    uint64_t out_cap;         // room at out_off
    uint64_t window_size;
    const uint8_t *dict;      // dictionary content (device) or null
    uint64_t dict_len;
    uint32_t first_block;
    uint32_t nblocks;
    uint32_t host_status;     // planner error that ends the frame after `nblocks` blocks (code | stage << 16)
    uint32_t pad;
};

// ---- status words: code | stage << 16 (b200z_error, B200Z_STAGE_*), 0 = ok
__host__ __device__ inline uint32_t mk_status(uint32_t code, uint32_t stage) { return code | (stage << 16); }
__host__ __device__ inline uint32_t status_code(uint32_t s) { return s & 0xffffu; }
__host__ __device__ inline uint32_t status_stage(uint32_t s) { return (s >> 16) & 0xffu; }
// BlockDesc::host_status adds where the planner's error lies relative to the literals stage (bits 24..31), so that the device can
// report a block's first error in the reference's order (block_first_error)
constexpr uint32_t HS_BEFORE_LITERALS = 1, HS_AFTER_LITERALS = 2;
__host__ __device__ inline uint32_t host_status(uint32_t code, uint32_t stage, uint32_t pos) { return mk_status(code, stage) | (pos << 24); }
__host__ __device__ inline uint32_t host_status_pos(uint32_t hs) { return hs >> 24; }
__host__ __device__ inline uint32_t host_status_word(uint32_t hs) { return hs & 0x00ffffffu; }
// The first error of a block in the reference's order: a planner error before the literals stage, the literals stage
// (BlockAux::status), any other planner error (sequences header), the sequence stage (BlockAux::seq_status).  0 = none.
__host__ __device__ inline uint32_t block_first_error(uint32_t host_st, uint32_t lit_st, uint32_t seq_st) {
    if (host_status_pos(host_st) == HS_BEFORE_LITERALS) return host_status_word(host_st);
    if (lit_st) return lit_st;
    if (host_st) return host_status_word(host_st);
    return seq_st;
}

}  // namespace b200z
