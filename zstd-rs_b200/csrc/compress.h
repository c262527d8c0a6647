// compress.h -- launch interface between the host library (api.cpp) and the compressor's kernels (compress.cu)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200zstd.h"
#include "encode.cuh"

namespace b200z {

constexpr uint32_t CM_WARPS = 8;                                          // segments (warps) per block in k_cmatch
constexpr uint32_t CSEG_SEQS = (ENC_BLOCK / CM_WARPS) / ENC_MIN_MATCH + 1;  // sequences one segment can hold
constexpr uint32_t CBLOCK_SEQS = CM_WARPS * CSEG_SEQS;

struct CFrame {        // one output frame
    uint64_t src_off, src_size, dst_off;
    uint32_t first_block, nblocks;
};
struct CBlock {        // one 128 KiB (or shorter last) block of a frame's input
    uint64_t src_off;  // in `input`
    uint32_t size;
    uint32_t back;     // bytes of the same frame before the block (matches may reach that far, up to the window)
    uint32_t frame;
    uint32_t pad;
};
struct CBlockInfo {    // k_cmatch: literals, sequences, type 1 when all bytes are equal; k_cenc: + block type and content size
    uint32_t nlit, nseq, type, csize;
};

struct LForced {       // a forced match of a block: [start, start + len) at offset off, block-relative
    uint32_t start, len, off;
};

struct FBlock {        // one block of a k_copt<..., true, true> launch
    uint32_t vbase;    // its first byte's virtual position; FAR_NONE: no far walk (its frame's window is 131072)
    uint32_t back;     // the frame's bytes before the block that repeats and far matches may reach: min(its offset in the frame, wf)
    uint32_t wf;       // its frame's window (131072 when vbase is FAR_NONE)
    uint32_t pad;
};

struct CompressArgs {
    const CFrame *frames;
    const CBlock *blocks;
    const uint8_t *input;
    uint8_t *output;
    uint8_t *lit_stage;   // [nblocks * ENC_BLOCK], reused as the encoded blocks' staging (`enc`) once k_cmatch is done
    SeqRec *seq_stage;    // [nblocks * CBLOCK_SEQS]
    uint8_t *lits;        // [nblocks * ENC_BLOCK]
    SeqRec *seqs;         // [nblocks * CBLOCK_SEQS]
    uint8_t *enc;
    CBlockInfo *info, *res;
    uint64_t *csum;       // [nframes]
    b200z_compress_result *results;
    uint32_t nframes, nblocks;
    int level, checksum;
    // the submission's dictionary (EXTENSION: ruzstd's FrameCompressor writes no dictionary ID and uses none).  dict_id goes into
    // every frame header (0: no field); dict / dtab are null when there is nothing to match against
    const uint8_t *dict;    // the last dict_len <= ENC_WINDOW bytes of its content (device): all a match can reach
    const uint32_t *dtab;   // [1 << CD_LOG] from k_cdict
    uint32_t dict_len, dict_id;
    const EncDict *etab;    // a formatted dictionary's tables for the frames' first blocks (B200Z_FLAG_DICT_TABLES), else null
    // long-distance matches (window_log > 17; ldm.cu): block b's forced matches are lforced[lf_off[b], + lf_cnt[b]); lf_cnt null: none,
    // and k_cmatch is the plain kernel.  window_log (0 counts as 17) sets each frame's Window_Descriptor
    const LForced *lforced;
    const uint32_t *lf_off, *lf_cnt;
    uint32_t window_log;
    // OPT (EXTENSION): k_copt's chain of the block it works on, one OPT_SPAN slot per CTA of its grid (opt_ctas())
    int32_t *opt_prev;
    // ULTRA (EXTENSION): a group's far stage (ldm.cu) for k_copt<..., true, true>: fblk[nblocks] per block, the sorted pairs and the
    // walks' starts; fblk null: k_copt is OPT's kernel (no block of the submission has a window beyond 131072)
    const FBlock *fblk;
    const uint32_t *fkeys, *fvals, *fstart;
    // B200Z_FLAG_DICT_LONG (ldm.cu): long matches reach into the dictionary's whole content ldict[ldict_len] (device), and each
    // frame's Window_Descriptor covers ldict_len + its size; ldict_len 0 and ldict null: they do not
    const uint8_t *ldict;
    uint64_t ldict_len;
};

// ---- OPT (compress.cu): a CTA's chain covers the block and the ENC_WINDOW bytes before it
constexpr uint32_t OPT_SPAN = ENC_WINDOW + ENC_BLOCK;
// k_copt's grid: the CTAs resident on the device at once (after init_compress_kernels); the CTAs stride over the blocks
uint32_t opt_ctas();

// ---- long-distance matches (ldm.cu; DESIGN.md section 4.11, tests/cldm.py)
constexpr uint32_t LDM_LEN = 64;          // bytes hashed at an anchor (the 64 ending at it), verified, and the least a kept match holds
constexpr uint32_t LDM_MASK_SHIFT = 57;   // a position passes when its gear hash's top 7 bits are 0: about 1 in 128
constexpr uint32_t LDM_QUIET = 15;        // an anchor passes and no position in the 15 before it does: at most 1 anchor in 16
constexpr uint32_t LDM_MARGIN = 128;      // bytes before the 2^window_log a stream chunk keeps: >= LDM_LEN - 1 + LDM_QUIET
constexpr uint32_t LDM_THREADS = 256, LDM_SPAN = ENC_BLOCK / LDM_THREADS;   // k_lanchor: positions per thread
constexpr uint32_t LDM_SPAN_CAP = LDM_THREADS * (LDM_SPAN / (LDM_QUIET + 1));   // the most anchors a span can hold
constexpr uint32_t LDM_TILE = 4096;       // pairs per CTA of the key sort
constexpr uint32_t LDM_NO_BLOCK = 0xffffffffu;
struct LSpan {         // up to ENC_BLOCK bytes whose anchors k_lanchor lists: a block of a long frame, or history before a stream chunk
    uint64_t off;      // in `input`
    uint64_t lo;       // the first byte of its frame in `input` (a stream chunk: of the history kept before it)
    uint32_t size, frame;
    uint32_t block;    // its CBlock, whose forced matches k_lblock writes; LDM_NO_BLOCK for history
    uint32_t pad;
};
// B200Z_FLAG_DICT_LONG: the dictionary's anchors, built once per dictionary (launch_ldm_dict) and kept with it, for k_lcand<true>;
// its content for k_lblock<true>, whose sources lie in the virtual stream D || X
constexpr uint64_t LDM_DICT_REACH = 1ull << B200Z_WINDOW_LOG_MAX;   // the dictionary bytes, from its end, whose anchors are listed
struct LDict {
    const uint32_t *keys;   // [n] the anchors' keys, ascending; equal keys in position order
    const uint32_t *dist;   // [n] |D| minus each anchor's position in D (1 .. 2^27)
    uint32_t n;
    const CFrame *frames;   // the submission's frames: an anchor's position in its frame is its input offset less src_off
};
struct LDictSrc {
    const uint8_t *d;       // D's content (device), allocated with 16 bytes of padding
    uint64_t len;           // |D|
};
struct LdmArgs {
    const uint8_t *input;
    const LSpan *spans;        // [nspans], in input order within each frame, the frames in submission order
    uint32_t nspans, window_log;
    uint32_t *tcount;          // [nspans * LDM_THREADS]: anchors per k_lanchor thread
    uint32_t *scount;          // [nspans + 1]: anchors per span, then their exclusive prefix sum and the total
    uint32_t cap;              // anchors the buffers below hold: the total, or (stream) the density bound; grids are sized by it
    uint32_t *keys[2], *vals[2], *hist;   // the sort's ping-pong pairs [cap] and its digit counts [256 * ceil(cap / LDM_TILE) + 1]
    uint64_t *apos;            // [cap] input offset of each anchor
    uint32_t *aframe, *cand;   // [cap] its frame, its candidate offset (0: none)
    LForced *forced;           // [cap]
    uint32_t *lf_off, *lf_cnt; // [blocks]: each span's CBlock's share of `forced`; lf_cnt zeroed by the host
    bool dict_long;            // B200Z_FLAG_DICT_LONG: k_lcand<true> and k_lblock<true> over ld and ds
    LDict ld;
    LDictSrc ds;
};
// k_lanchor<false> and k_lscan: tcount, scount and the total; adds the kernels it enqueued to *launched
int launch_ldm_count(const LdmArgs &a, cudaStream_t s, uint64_t *launched);
// with the buffers sized for a.cap >= the total: k_lanchor<true>, the sort, k_lcand and k_lblock
int launch_ldm_match(const LdmArgs &a, cudaStream_t s, uint64_t *launched);
// a dictionary's anchors (B200Z_FLAG_DICT_LONG), after launch_ldm_count over the spans of D's last min(|D|, 2^27) bytes (input: D,
// a.cap >= their total > 0): k_lanchor<true>, the sort and k_ldict, which writes the sorted keys[a.cap] and dist[a.cap] of |D| = dlen
constexpr uint32_t LDM_DICT_LAUNCHES = 16;   // launch_ldm_count's 2, then k_lanchor<true>, four sort passes of three and k_ldict
int launch_ldm_dict(const LdmArgs &a, uint64_t dlen, uint32_t *keys, uint32_t *dist, cudaStream_t s, uint64_t *launched);

// ---- ULTRA's far stage (ldm.cu; DESIGN.md section 4.4, tests/cultra.py): per group of whole blocks (at most
// B200Z_PIPELINE_CHUNK_BYTES of them, or a stream chunk) and the Wf bytes of its frame before its first block, the keyed positions'
// (key8, virtual position) pairs sorted by key (the LDM sort), then where each position's far walk starts in the sorted pairs.
// A group's positions are numbered in a virtual space: each frame's part (its history, then its blocks) is contiguous in it, so a
// distance in the virtual space is a distance in the frame.
constexpr uint32_t FAR_DEPTH = 8;          // D_F: far entries a position visits, collisions counted
constexpr uint32_t FAR_KEY = 8;            // bytes key8 hashes; a position is keyed when they end inside its 128 KiB block
constexpr uint32_t FAR_NONE = 0xffffffffu;
constexpr uint32_t FAR_LAUNCHES = 14;      // kernels per group: k_fkey, four sort passes of three, k_fstart
struct FPiece {        // one 128 KiB (or shorter last) block of a frame in a group, history or the group's own
    uint64_t off;      // in `input`
    uint32_t vbase;    // its first byte's virtual position
    uint32_t pbase;    // its first pair
    uint32_t size;     // bytes; the first size - 7 (if any) are keyed
    uint32_t pad;
};
struct FarArgs {
    const uint8_t *input;
    const FPiece *pieces;
    uint32_t npieces, npairs;
    uint32_t *total;                       // [1]: npairs, written by k_fkey for the sort
    uint32_t *keys[2], *vals[2], *hist;    // the sort's ping-pong pairs [npairs] and its digit counts [256 * ceil(npairs / LDM_TILE) + 1]
    uint32_t *start;                       // [virtual positions]: the sorted index a position's far walk starts at, or FAR_NONE
};
// the group's far stage: k_fkey, the sort, k_fstart (FAR_LAUNCHES kernels); adds the kernels it enqueued to *launched
int launch_far_stage(const FarArgs &f, cudaStream_t s, uint64_t *launched);

// the dictionary match table: 5-byte hash of a position in the dictionary's last ENC_WINDOW bytes -> that position + 1 (0 = none)
constexpr uint32_t CD_LOG = 17;

int init_compress_kernels();
// fills dtab[1 << CD_LOG] for the device content dict[len], len <= ENC_WINDOW (a memset and k_cdict, on stream s); adds the kernels
// it enqueued to *launched
int launch_dict_table(const uint8_t *dict, uint32_t len, uint32_t *dtab, cudaStream_t s, uint64_t *launched);
// dictionary statistics (b200z_dict_finalize): literal bytes, LL, ML and OF code counts, in that order, in one u64 array
constexpr uint32_t DS_LIT = 0, DS_LL = 256, DS_ML = DS_LL + 36, DS_OF = DS_ML + 53, DS_BINS = DS_OF + 32;   // 377 bins
constexpr uint32_t DS_THREADS = 256;
constexpr uint32_t DS_BLOCKS = 2048;   // blocks per statistics submission: the compressor's staging of that many blocks (~1.8 GB)
// k_cmatch<true> over a.blocks[a.nblocks] against a.dict / a.dtab, then k_dstats, which adds every non-RLE block's histograms to
// counts[DS_BINS]; adds the kernels it enqueued to *launched
int launch_dict_stats(const CompressArgs &a, unsigned long long *counts, cudaStream_t s, uint64_t *launched);
// dict_format.cpp (host): the argument rule of b200z_dict_finalize that needs no counts, and the dictionary from counts[DS_BINS]
int dict_check_args(size_t content_len, uint32_t dict_id, size_t dict_cap);
int dict_from_counts(const uint64_t *counts, const uint8_t *content, size_t content_len, uint32_t dict_id, uint8_t *dict, size_t dict_cap,
                     size_t *dict_len);
constexpr int kCompressStages = 4;
extern const char *const kCompressStageNames[kCompressStages];
int launch_compress_stage(const CompressArgs &a, int stage, cudaStream_t s, uint64_t *launched);   // adds the kernels it enqueued to *launched
// one chunk of a streamed frame (b200z_frame_compressor, Fastest): k_cmatch, k_cenc, k_cassemble<true> over a.blocks[a.nblocks],
// which all belong to a.frames[0] (the chunk); no dictionary, no checksum kernel.  Adds the kernels it enqueued to *launched
int launch_compress_chunk(const CompressArgs &a, cudaStream_t s, uint64_t *launched);

// ---- seekable archives (seekable.cu; EXTENSION, the zstd seekable format)
constexpr uint32_t SEEK_SKIPPABLE_MAGIC = 0x184D2A5Eu;
constexpr uint32_t SEEK_FOOTER_MAGIC = 0x8F92EAB1u;
constexpr uint32_t SEEK_FOOTER = 9;                 // Number_Of_Frames, Seek_Table_Descriptor, Seekable_Magic_Number
constexpr uint32_t SEEK_TABLE_FIXED = 8 + SEEK_FOOTER;   // the skippable frame's header and the footer
// k_cscan over a.blocks[a.nblocks] (a group of whole frames, after k_cenc and k_cxxh64): every a.frames[f].dst_off becomes the
// frame's packed archive offset less `origin`, *total (device) moves past the group, and frame f's table entry goes to
// entries[(first_frame + f) * (a.checksum ? 12 : 8)].  Adds the kernels it enqueued to *launched
int launch_seek_scan(const CompressArgs &a, uint64_t *total, uint64_t origin, uint8_t *entries, uint64_t first_frame, cudaStream_t s,
                     uint64_t *launched);
// k_cseek: the table frame of the n entries at output + (*total - origin)
int launch_seek_table(const uint8_t *entries, uint64_t n, int checksum, const uint64_t *total, uint64_t origin, uint8_t *output, cudaStream_t s,
                      uint64_t *launched);
// one copy piece of the read plan: len <= GATHER_CHUNK bytes from base + src to base + dst
struct GatherPiece {
    uint64_t src, dst;
    uint32_t len, pad;
};
constexpr uint32_t GATHER_CHUNK = 65536;
// k_range_gather: one CTA per piece
int launch_range_gather(const GatherPiece *pieces, uint32_t n, uint8_t *base, cudaStream_t s, uint64_t *launched);

}  // namespace b200z
