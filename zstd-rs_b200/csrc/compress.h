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
};

// the dictionary match table: 5-byte hash of a position in the dictionary's last ENC_WINDOW bytes -> that position + 1 (0 = none)
constexpr uint32_t CD_LOG = 17;

int init_compress_kernels();
// fills dtab[1 << CD_LOG] for the device content dict[len], len <= ENC_WINDOW (a memset and k_cdict, on stream s); adds the kernels
// it enqueued to *launched
int launch_dict_table(const uint8_t *dict, uint32_t len, uint32_t *dtab, cudaStream_t s, uint64_t *launched);
constexpr int kCompressStages = 4;
extern const char *const kCompressStageNames[kCompressStages];
int launch_compress_stage(const CompressArgs &a, int stage, cudaStream_t s, uint64_t *launched);   // adds the kernels it enqueued to *launched

}  // namespace b200z
