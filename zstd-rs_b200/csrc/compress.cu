// compress.cu -- sm_90a kernels of the batch compressor (ruzstd's encoding::compress at CompressionLevel::Fastest).
//
//   k_cmatch    : one CTA per 128 KiB block: greedy LZ77 parse into literals + sequences (two-table parallel parse)
//                 (<DICT, true>: the LAZY level's parse, an extension: K-way tables, repeat candidates, a lazy choice;
//                  <DICT, LAZY, true>: with the long-distance matches of ldm.cu forced into the parse, window_log > 17)
//   k_copt      : OPT (an extension): in k_cmatch's place, a grid of the resident CTAs striding over the blocks: per block a hash chain
//                 over the block and the 128 KiB before it, then one warp per segment parses it by a price-based forward DP
//                 (<DICT, LONG>: as k_cmatch's; <DICT, true, true>: ULTRA, with the far walk over ldm.cu's far stage)
//   k_cenc      : one warp per block: Huffman literals, FSE sequences, the Raw / RLE / Compressed decision (encode.cuh)
//                 (<TABLES, true>: LAZY and OPT, repeat-offset codes within each block first)
//   k_cxxh64    : content checksum of every frame's input (xxh64.cuh; four serial chains per frame)
//   k_cassemble : one CTA per block: frame header, the block at its prefix-summed offset, the checksum, per-frame results
//                 (<true, false>: one chunk of a streamed frame, blocks only; the host writes header, trailer and checksum;
//                 <false, true>: B200Z_FLAG_DICT_LONG, the Window_Descriptor covers the dictionary's content and the frame)
//   k_cdict     : not a stage: the match table of a dictionary, built once the first time the dictionary is used (EXTENSION)
//   k_dstats    : not a stage: literal and sequence-code histograms of k_cmatch's parse, for b200z_dict_finalize (EXTENSION)
//
// Every block is encoded from its own literals and sequences only (repeat offsets only at LAZY, within the block; Repeat / Treeless modes only in a frame's
// first block with a formatted dictionary's tables, which the format makes that block's previous tables), so all
// blocks of all frames -- including the blocks of one huge frame -- run at the same time.  Matches may still reach back into
// the previous block: the input is all there from the start.  With a dictionary (an extension: ruzstd's encoder has none), the
// first ENC_WINDOW bytes of every frame may also match the dictionary's content, which lies before the frame's first byte.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include <algorithm>

#include "compress.h"
#include "encode.cuh"
#include "xxh64.cuh"

namespace b200z {

constexpr uint32_t CM_THREADS = CM_WARPS * 32;
constexpr uint32_t CM_T1_LOG = 14;   // block-wide first-occurrence table
constexpr uint32_t CM_TP_LOG = 12;   // per-warp most-recent table
constexpr uint32_t CM_SEED = 16384;  // bytes before its segment a warp's private table starts from
constexpr uint32_t CM_CAP = 16;      // match bytes a lane verifies before the warp extends the chosen match together
constexpr uint32_t CM_SMEM = (4u << CM_T1_LOG) + CM_WARPS * (4u << CM_TP_LOG);
constexpr uint32_t CE_WARPS = 4;
// the LAZY parse (tests/clazy.py states it rule by rule)
constexpr uint32_t LZ_T1_LOG = 15;     // its t1 is twice Fastest's
constexpr uint32_t LZ_TAB_LOG = 10;    // buckets of a warp's table
constexpr uint32_t LZ_WAYS = 6;        // positions per bucket, u16 relative to the seed base, newest first (3 words)
constexpr uint32_t LZ_SEED = 32768;    // bytes before its segment a warp's table starts from (stream chunks keep 128 KiB in front)
constexpr uint32_t LZ_CAP = 32;        // match bytes a lane verifies before the warp extends the chosen match together
constexpr uint32_t LZ_DEPTH = 4;       // lanes after the first match that compete with it
constexpr int32_t LZ_LANE_COST = 3;    // gain a later lane gives up per byte it starts later
constexpr uint32_t LZ_EMPTY = 0xffffu;
constexpr uint32_t LZ_SMEM = (4u << LZ_T1_LOG) + CM_WARPS * (2u * LZ_WAYS << LZ_TAB_LOG);   // 224 KiB
static_assert(LZ_SEED + ENC_BLOCK / CM_WARPS < LZ_EMPTY, "a table entry must fit below the empty mark");
static_assert(LZ_WAYS == 6, "lz_push shifts three words");
// the OPT parse (tests/copt.py states it rule by rule)
constexpr uint32_t OPT_HASH_LOG = 13;   // H: the chain's hash
constexpr uint32_t OPT_DEPTH = 24;      // D: chain entries a position visits
constexpr uint32_t OPT_CANDS = 4;       // M: candidates kept per position
constexpr uint32_t OPT_SUFF = 32;       // bytes a candidate is verified for; a candidate this long is taken at once
constexpr uint32_t OPT_WIN = 256;       // W: nodes one DP spans before it closes
constexpr uint32_t OPT_NODES = OPT_WIN + OPT_SUFF;      // node a + k for k < OPT_NODES: a DP's reach
constexpr uint32_t OPT_PATH = OPT_WIN / ENC_MIN_MATCH + 1;   // the most matches a closed DP's path holds
constexpr uint32_t OPT_INF = 1u << 30;
constexpr uint32_t OPT_MATCH_W = 1024, OPT_OF_W = 512, OPT_REP_W0 = 256, OPT_REP_W1 = 512, OPT_REP_W2 = 768;   // prices in 1/256 bit
constexpr int32_t OPT_NONE = INT_MIN, OPT_FIX = INT_MIN + 1;   // prev: no earlier position; none in the stripe (resolved next)
constexpr uint32_t OPT_SMEM = CM_WARPS * (2u << OPT_HASH_LOG);  // the stripes' u16 heads (128 KiB), then the warps' DP state
struct OptWarp {       // one warp's DP state (k_copt's second phase)
    uint32_t cost[OPT_NODES], link[OPT_NODES], off[OPT_NODES], rep[3][OPT_NODES];   // link: from | length << 16 (0: a literal)
    uint32_t cand[32 * OPT_CANDS];                                                  // the chunk's lists (cand_pack)
    uint32_t path_pos[OPT_PATH], path_ml[OPT_PATH], path_off[OPT_PATH];
};
static_assert(CM_WARPS * sizeof(OptWarp) <= OPT_SMEM, "the DP state reuses the heads' shared memory");
static_assert(OPT_SPAN / CM_WARPS <= 0xffffu, "a stripe position must fit below the empty head");
static_assert(OPT_SUFF == 32 && OPT_SUFF - 1 <= 34, "one lane per length, and no length below OPT_SUFF has ML extra bits");

__device__ __forceinline__ uint64_t load5(const uint8_t *p) {
    return (uint64_t)__ldg(p) | ((uint64_t)__ldg(p + 1) << 8) | ((uint64_t)__ldg(p + 2) << 16) | ((uint64_t)__ldg(p + 3) << 24) |
           ((uint64_t)__ldg(p + 4) << 32);
}
__device__ __forceinline__ uint32_t hash5(const uint8_t *p, uint32_t log) { return (uint32_t)(((load5(p) << 24) * 889523592379ull) >> (64 - log)); }
__device__ __forceinline__ uint32_t match_len(const uint8_t *a, const uint8_t *b, uint32_t lim) {
    uint32_t n = 0;
    while (n < lim && __ldg(a + n) == __ldg(b + n)) n++;
    return n;
}

// LAZY: pushes u16 entry v into a bucket held as three words, slot 0 (the newest) in the low half of w0
__device__ __forceinline__ void lz_push(uint32_t &w0, uint32_t &w1, uint32_t &w2, uint32_t v) {
    w2 = (w2 << 16) | (w1 >> 16);
    w1 = (w1 << 16) | (w0 >> 16);
    w0 = (w0 << 16) | v;
}

// LAZY: inserts positions q0 + lane (the lanes with `valid`) into the warp's table in position order.  Lanes of one bucket form
// a group; its last lane pushes the group's last LZ_WAYS positions, oldest first, so the table does not depend on the schedule.
__device__ __forceinline__ void lz_insert(uint32_t *tab, const uint8_t *src, int32_t q0, bool valid, int32_t base, uint32_t lane) {
    const uint32_t h = valid ? hash5(src + q0 + (int32_t)lane, LZ_TAB_LOG) : (1u << LZ_TAB_LOG) + lane;   // invalid: a group alone
    const uint32_t grp = __match_any_sync(0xffffffffu, h);
    if (valid && lane == 31u - __clz(grp)) {
        uint32_t *bk = tab + 3 * h;
        uint32_t w0 = bk[0], w1 = bk[1], w2 = bk[2], m = grp;
        for (uint32_t c = __popc(grp); c > LZ_WAYS; c--) m &= m - 1;
        for (; m; m &= m - 1) lz_push(w0, w1, w2, (uint32_t)(q0 + __ffs(m) - 1 - base));
        bk[0] = w0; bk[1] = w1; bk[2] = w2;
    }
    __syncwarp();
}

// LAZY: extends the chosen match at qj (offset off, ml bytes verified) 32 bytes at a time, up to lim, as the Fastest loop does
// inline (kept there as it is so that the Fastest kernels compile to the same SASS)
template <bool DICT>
__device__ __forceinline__ uint32_t extend_match(const uint8_t *src, uint32_t qj, uint32_t off, uint32_t ml, uint32_t lim, uint32_t back,
                                                 const uint8_t *dict, uint32_t dict_len, uint32_t lane) {
    const uint32_t fpos = back + qj;   // an offset beyond the frame's start points into the dictionary
    const uint8_t *ref = DICT && off > fpos ? dict + dict_len - (off - fpos) : src + qj - off;
    while (ml < lim) {
        const uint32_t i = ml + lane;
        const bool stop = i >= lim || __ldg(src + qj + i) != __ldg(ref + i);
        const uint32_t sm = __ballot_sync(0xffffffffu, stop);
        if (sm) { ml += __ffs(sm) - 1; break; }
        ml += 32;
    }
    return min(ml, lim);
}

// long-distance matches: the forced pieces of one segment, in order -- the block's forced matches (ldm.cu) clipped to [s, e),
// pieces shorter than ENC_MIN_MATCH left to the regular parse.  has: a piece [cs, ce) at offset off is next.
struct LCursor {
    const LForced *f;
    uint32_t k, n, s, e, cs, ce, off;
    bool has;
    __device__ __forceinline__ void next() {
        has = false;
        while (k < n) {
            const LForced x = f[k++];
            if (x.start >= e) { k = n; break; }
            cs = max(x.start, s);
            ce = min(x.start + x.len, e);
            if (ce >= cs + ENC_MIN_MATCH) { off = x.off; has = true; break; }
        }
    }
};

// LAZY: one warp's parse of segment [s, e) (see k_cmatch); writes the segment's sequences and literals to its staging and its
// counts to *nseq_out, *nlit_out, *trail_out
// (LONG: the gaps between the segment's forced pieces, each piece one sequence, as in k_cmatch)
template <bool DICT, bool LONG>
__device__ __forceinline__ void cmatch_lazy(const CBlock &blk, const uint8_t *src, uint32_t s, uint32_t e, const uint32_t *t1, uint32_t *tab,
                                            int32_t base, uint32_t lane, const uint8_t *dict, const uint32_t *dtab, uint32_t dict_len,
                                            SeqRec *stage, uint8_t *lstage, uint32_t *nseq_out, uint32_t *nlit_out, uint32_t *trail_out,
                                            LCursor &lc) {
    uint32_t p = s, anchor = s, nseq = 0, nlit = 0;
    uint32_t r0 = 0, r1 = 0, r2 = 0;   // the segment's three most recent distinct offsets (0: none yet)
    uint32_t ee = e;                   // where the regular parse stops: the segment's end, or the next forced piece
    if constexpr (LONG) { lc.next(); if (lc.has) ee = lc.cs; }
    while (true) {   // once without LONG; with it, once per forced piece and once after the last (the body keeps its indentation)
    while (p + ENC_MIN_MATCH <= ee) {
        const uint32_t q = p + lane;
        const bool valid = q + ENC_MIN_MATCH <= ee;
        int32_t gain = INT_MIN;   // INT_MIN: no candidate of >= 5 bytes
        uint32_t len = 0, cand = 0, xlim = ee - q;
        if (valid) {
            const uint32_t lim = min(LZ_CAP, ee - q), fpos = blk.back + q;
            auto take = [&](uint32_t o, const uint8_t *ref, uint32_t l, int32_t cost) {
                const int32_t g = 4 * (int32_t)l - cost;
                if (l >= ENC_MIN_MATCH && g > gain) { gain = g; len = l; cand = o; return true; }
                return false;
            };
            auto rep = [&](uint32_t o) {   // the source must lie in the frame and the window
                if (o && o <= fpos && o <= ENC_WINDOW) take(o, src + q - o, match_len(src + q, src + q - o, lim), 0);
            };
            rep(r0); rep(r1); rep(r2);
            const uint32_t c1 = t1[hash5(src + q, LZ_T1_LOG)];
            if (c1 < q) take(q - c1, src + c1, match_len(src + q, src + c1, lim), 31 - __clz(q - c1));
            const uint32_t *bk = tab + 3 * hash5(src + q, LZ_TAB_LOG);
            const uint32_t w[3] = {bk[0], bk[1], bk[2]};
#pragma unroll
            for (uint32_t k = 0; k < LZ_WAYS; k++) {   // newest first
                const uint32_t rel = (w[k >> 1] >> (16 * (k & 1))) & 0xffffu;
                const int32_t c = base + (int32_t)rel;
                if (rel != LZ_EMPTY && c < (int32_t)q) {
                    const uint32_t o = (uint32_t)((int32_t)q - c);
                    take(o, src + c, match_len(src + q, src + c, lim), 31 - __clz(o));
                }
            }
            if (DICT && fpos < ENC_WINDOW) {
                const uint32_t c3 = __ldg(dtab + hash5(src + q, CD_LOG));
                const uint32_t off3 = fpos + dict_len - (c3 - 1);
                if (c3 && off3 <= ENC_WINDOW) {
                    const uint32_t rest = dict_len - (c3 - 1);   // dictionary bytes from the source to the dictionary's end
                    if (take(off3, dict + (c3 - 1), match_len(src + q, dict + (c3 - 1), min(lim, rest)), 31 - __clz(off3))) xlim = min(xlim, rest);
                }
            }
        }
        const uint32_t m = __ballot_sync(0xffffffffu, gain != INT_MIN);
        lz_insert(tab, src, (int32_t)p, valid, base, lane);   // after every lane's lookup (the ballot), before the next round's
        if (!m) { p += 32; continue; }
        // the lazy choice: lanes j .. j + LZ_DEPTH with a match score gain - LZ_LANE_COST * (lane - j); the highest wins, the
        // earlier lane on a tie (a score lies in [-9, 128], so score + 64 fits 8 bits above the lane's 5)
        const uint32_t j = __ffs(m) - 1, d = lane - j;
        const bool comp = gain != INT_MIN && lane >= j && d <= LZ_DEPTH;
        const uint32_t key = comp ? ((uint32_t)(gain - LZ_LANE_COST * (int32_t)d + 64) << 5) | (31 - lane) : 0u;
        const uint32_t win = 31 - (__reduce_max_sync(0xffffffffu, key) & 31);
        const uint32_t qj = p + win, off = __shfl_sync(0xffffffffu, cand, win);
        uint32_t ml = __shfl_sync(0xffffffffu, len, win);
        const uint32_t lim = __shfl_sync(0xffffffffu, xlim, win);
        if (ml == LZ_CAP) ml = extend_match<DICT>(src, qj, off, ml, DICT ? lim : ee - qj, blk.back, dict, dict_len, lane);
        for (uint32_t i = anchor + lane; i < qj; i += 32) lstage[nlit + i - anchor] = __ldg(src + i);
        if (lane == 0) stage[nseq] = SeqRec{qj - anchor, ml, off};
        nlit += qj - anchor;
        nseq++;
        anchor = p = qj + ml;
        if (off == r1) { r1 = r0; r0 = off; }   // off moves to the front
        else if (off != r0) { r2 = r1; r1 = r0; r0 = off; }
        __syncwarp();
    }
    if constexpr (!LONG) break;
    else {
        if (!lc.has) break;
        const uint32_t qj = lc.cs, ml = lc.ce - lc.cs, off = lc.off;   // the forced piece, taken as any match is
        for (uint32_t i = anchor + lane; i < qj; i += 32) lstage[nlit + i - anchor] = __ldg(src + i);
        if (lane == 0) stage[nseq] = SeqRec{qj - anchor, ml, off};
        nlit += qj - anchor;
        nseq++;
        anchor = p = qj + ml;
        if (off == r1) { r1 = r0; r0 = off; }
        else if (off != r0) { r2 = r1; r1 = r0; r0 = off; }
        lc.next();
        ee = lc.has ? lc.cs : e;
        __syncwarp();
    }
    }
    for (uint32_t i = anchor + lane; i < e; i += 32) lstage[nlit + i - anchor] = __ldg(src + i);
    if (lane == 0) { *nseq_out = nseq; *nlit_out = nlit + (e - anchor); *trail_out = e - anchor; }
}

// ------------------------------------------------------------------------------------------------------------
// k_cmatch.  The CTA first builds a first-occurrence table of the block (5-byte hash -> smallest position, shared-memory
// atomicMin: deterministic).  Warp w then parses segment w of the block greedily, 32 positions at a time: every lane looks
// its position up in the first-occurrence table and in the warp's private most-recent table (seeded with the CM_SEED bytes
// before the segment, which may lie in the previous block), keeps the longer verified candidate (candidate < position, offset
// <= 128 KiB, inside the frame), and the first lane with a match of >= 5 bytes wins.  A match never crosses its segment's end.
// With DICT, a lane whose position is fewer than ENC_WINDOW bytes into the frame also looks up the dictionary's table (k_cdict)
// when that source is within the window, and verifies it against the dictionary's content; the longest candidate wins, the
// smaller offset on a tie.  A dictionary match stops at the dictionary's end.  Without DICT the code is the plain parse.
// Sequences and literals go to per-segment staging; the CTA then packs them, the trailing literals of a segment joining the
// first sequence after them.  tests/cparse.py states this parse rule by rule; the GPU must produce exactly its sequences.
// LAZY (an extension, B200Z_LEVEL_LAZY) keeps the blocks, segments, rounds, dictionary lookup and packing, with a t1 over 2^15
// hashes.  The private table holds the LZ_WAYS most recent positions per hash (seeded from LZ_SEED bytes back, filled in position
// order); each lane also tries the segment's three most recent distinct offsets; every candidate scores 4 ml - floor(log2 off)
// (a repeat costs 0), and the first lane with a match competes with the next LZ_DEPTH lanes at LZ_LANE_COST per byte of delay.
// tests/clazy.py states it rule by rule.
// ------------------------------------------------------------------------------------------------------------
// LONG (window_log > 17, ldm.cu): each segment's forced pieces (LCursor) are taken as sequences, with the literals since the last
// match; the regular parse runs in the gaps between them exactly as it runs up to a segment's end, so no regular match crosses
// the next forced start.  tests/cldm.py states it.
template <bool DICT, bool LAZY, bool LONG = false>
__global__ void __launch_bounds__(CM_THREADS, 1)
k_cmatch(const CBlock *__restrict__ blocks, const uint8_t *__restrict__ input, uint8_t *__restrict__ lit_stage, SeqRec *__restrict__ seq_stage,
         uint8_t *__restrict__ lits, SeqRec *__restrict__ seqs, CBlockInfo *__restrict__ info, const uint8_t *__restrict__ dict,
         const uint32_t *__restrict__ dtab, uint32_t dict_len, const LForced *__restrict__ lforced = nullptr,
         const uint32_t *__restrict__ lf_off = nullptr, const uint32_t *__restrict__ lf_cnt = nullptr) {
    extern __shared__ __align__(16) uint8_t smem_cm[];
    uint32_t *t1 = reinterpret_cast<uint32_t *>(smem_cm);
    int32_t *tp_all = reinterpret_cast<int32_t *>(smem_cm + (4u << CM_T1_LOG));
    __shared__ uint32_t s_nseq[CM_WARPS], s_nlit[CM_WARPS], s_trail[CM_WARPS], s_add[CM_WARPS], s_soff[CM_WARPS], s_loff[CM_WARPS];
    const uint32_t b = blockIdx.x, tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
    const CBlock blk = blocks[b];
    const uint8_t *src = input + blk.src_off;
    const uint32_t n = blk.size;
    bool same = true;
    for (uint32_t i = tid; i < n; i += CM_THREADS) same &= __ldg(src + i) == __ldg(src);
    same = __syncthreads_and(same);
    if (n == 0 || same) {
        if (tid == 0) info[b] = CBlockInfo{n, 0, n ? 1u : 0u, 0};
        return;
    }
    constexpr uint32_t T1_LOG = LAZY ? LZ_T1_LOG : CM_T1_LOG;
    for (uint32_t i = tid; i < (1u << T1_LOG); i += CM_THREADS) t1[i] = 0xffffffffu;
    if constexpr (LAZY) {
        uint32_t *tab_all = reinterpret_cast<uint32_t *>(smem_cm + (4u << LZ_T1_LOG));
        for (uint32_t i = tid; i < CM_WARPS * (3u << LZ_TAB_LOG); i += CM_THREADS) tab_all[i] = 0xffffffffu;
    } else {
        for (uint32_t i = tid; i < CM_WARPS << CM_TP_LOG; i += CM_THREADS) tp_all[i] = INT_MIN;
    }
    __syncthreads();
    for (uint32_t q = tid; q + ENC_MIN_MATCH <= n; q += CM_THREADS) atomicMin(&t1[hash5(src + q, T1_LOG)], q);
    int32_t *tp = tp_all + (w << CM_TP_LOG);
    const uint32_t seglen = (n + CM_WARPS - 1) / CM_WARPS;
    const uint32_t s = min(n, w * seglen), e = min(n, s + seglen);
    LCursor lc{};
    if constexpr (LONG) lc = LCursor{lforced + lf_off[b], 0, lf_cnt[b], s, e, 0, 0, 0, false};
    if constexpr (LAZY) {
        SeqRec *stage = seq_stage + ((size_t)b * CM_WARPS + w) * CSEG_SEQS;
        uint8_t *lstage = lit_stage + (size_t)b * ENC_BLOCK + s;
        uint32_t *tab = reinterpret_cast<uint32_t *>(smem_cm + (4u << LZ_T1_LOG)) + w * (3u << LZ_TAB_LOG);
        const int32_t base = (int32_t)s - (int32_t)LZ_SEED;   // entries hold q - base
        const int32_t seed_lo = max(base, -(int32_t)blk.back), seed_hi = min((int32_t)s, (int32_t)n - (int32_t)ENC_MIN_MATCH + 1);
        for (int32_t q0 = seed_lo; q0 < seed_hi; q0 += 32) lz_insert(tab, src, q0, q0 + (int32_t)lane < seed_hi, base, lane);
        __syncthreads();
        cmatch_lazy<DICT, LONG>(blk, src, s, e, t1, tab, base, lane, dict, dtab, dict_len, stage, lstage, s_nseq + w, s_nlit + w, s_trail + w, lc);
    } else {
        const int32_t seed_lo = max((int32_t)s - (int32_t)CM_SEED, -(int32_t)min(blk.back, CM_SEED));
        for (int32_t q = seed_lo + (int32_t)lane; q < (int32_t)s && q + (int32_t)ENC_MIN_MATCH <= (int32_t)n; q += 32)   // inside the frame
            atomicMax(&tp[hash5(src + q, CM_TP_LOG)], q);
        __syncthreads();
        SeqRec *stage = seq_stage + ((size_t)b * CM_WARPS + w) * CSEG_SEQS;
        uint8_t *lstage = lit_stage + (size_t)b * ENC_BLOCK + s;
        uint32_t p = s, anchor = s, nseq = 0, nlit = 0;
        uint32_t ee = e;   // where the regular parse stops: the segment's end, or the next forced piece
        if constexpr (LONG) { lc.next(); if (lc.has) ee = lc.cs; }
        while (true) {   // as in cmatch_lazy
        while (p + ENC_MIN_MATCH <= ee) {
            const uint32_t q = p + lane;
            const bool valid = q + ENC_MIN_MATCH <= ee;
            uint32_t len = 0, cand = 0, h2 = 0, xlim = ee - q;   // xlim: how far the match may be extended
            if (valid) {
                const uint32_t lim = min(CM_CAP, ee - q);
                const uint32_t c1 = t1[hash5(src + q, CM_T1_LOG)];
                h2 = hash5(src + q, CM_TP_LOG);
                const int32_t c2 = tp[h2];
                if (c1 < q) { len = match_len(src + q, src + c1, lim); cand = q - c1; }
                // the window check cannot fail: c2 >= s - CM_SEED and q < s + seglen <= s + CM_SEED, so a tp offset is below 32 KiB
                // (offsets up to 128 KiB come from t1 only)
                if (c2 != INT_MIN && c2 < (int32_t)q && (int32_t)q - c2 <= (int32_t)ENC_WINDOW) {
                    const uint32_t l2 = match_len(src + q, src + c2, lim);
                    if (l2 > len || (l2 == len && (uint32_t)((int32_t)q - c2) < cand)) { len = l2; cand = (uint32_t)((int32_t)q - c2); }
                }
                const uint32_t fpos = blk.back + q;   // back < ENC_WINDOW means it is the block's position in the frame
                if (DICT && fpos < ENC_WINDOW) {
                    const uint32_t c3 = __ldg(dtab + hash5(src + q, CD_LOG));
                    const uint32_t off3 = fpos + dict_len - (c3 - 1);
                    if (c3 && off3 <= ENC_WINDOW) {
                        const uint32_t rest = dict_len - (c3 - 1);   // dictionary bytes from the source to the dictionary's end
                        const uint32_t l3 = match_len(src + q, dict + (c3 - 1), min(lim, rest));
                        if (l3 > len || (l3 == len && off3 < cand)) { len = l3; cand = off3; xlim = min(xlim, rest); }
                    }
                }
            }
            __syncwarp();
            if (valid) atomicMax(&tp[h2], (int32_t)q);
            const uint32_t m = __ballot_sync(0xffffffffu, len >= ENC_MIN_MATCH);
            if (!m) { p += 32; __syncwarp(); continue; }
            const uint32_t j = __ffs(m) - 1;
            const uint32_t qj = p + j, off = __shfl_sync(0xffffffffu, cand, j);
            uint32_t ml = __shfl_sync(0xffffffffu, len, j);
            if (ml == CM_CAP) {   // extend the chosen match 32 bytes at a time
                const uint32_t lim = DICT ? __shfl_sync(0xffffffffu, xlim, j) : ee - qj;
                const uint32_t fpos = blk.back + qj;   // an offset beyond the frame's start points into the dictionary
                const uint8_t *ref = DICT && off > fpos ? dict + dict_len - (off - fpos) : src + qj - off;
                while (ml < lim) {
                    const uint32_t i = ml + lane;
                    const bool stop = i >= lim || __ldg(src + qj + i) != __ldg(ref + i);
                    const uint32_t sm = __ballot_sync(0xffffffffu, stop);
                    if (sm) { ml += __ffs(sm) - 1; break; }
                    ml += 32;
                }
                ml = min(ml, lim);
            }
            for (uint32_t i = anchor + lane; i < qj; i += 32) lstage[nlit + i - anchor] = __ldg(src + i);
            if (lane == 0) stage[nseq] = SeqRec{qj - anchor, ml, off};
            nlit += qj - anchor;
            nseq++;
            anchor = p = qj + ml;
            __syncwarp();
        }
        if constexpr (!LONG) break;
        else {
            if (!lc.has) break;
            const uint32_t qj = lc.cs;   // the forced piece
            for (uint32_t i = anchor + lane; i < qj; i += 32) lstage[nlit + i - anchor] = __ldg(src + i);
            if (lane == 0) stage[nseq] = SeqRec{qj - anchor, lc.ce - qj, lc.off};
            nlit += qj - anchor;
            nseq++;
            anchor = p = lc.ce;
            lc.next();
            ee = lc.has ? lc.cs : e;
            __syncwarp();
        }
        }
        for (uint32_t i = anchor + lane; i < e; i += 32) lstage[nlit + i - anchor] = __ldg(src + i);
        if (lane == 0) { s_nseq[w] = nseq; s_nlit[w] = nlit + (e - anchor); s_trail[w] = e - anchor; }
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t carry = 0, so = 0, lo = 0;
        for (uint32_t v = 0; v < CM_WARPS; v++) {
            s_soff[v] = so; s_loff[v] = lo;
            so += s_nseq[v]; lo += s_nlit[v];
            if (s_nseq[v]) { s_add[v] = carry; carry = s_trail[v]; }
            else { s_add[v] = 0; carry += s_trail[v]; }
        }
        info[b] = CBlockInfo{lo, so, 0, 0};
    }
    __syncthreads();
    SeqRec *stage = seq_stage + ((size_t)b * CM_WARPS + w) * CSEG_SEQS;   // the segments' staging, packed below
    uint8_t *lstage = lit_stage + (size_t)b * ENC_BLOCK + s;
    SeqRec *out = seqs + (size_t)b * CBLOCK_SEQS + s_soff[w];
    for (uint32_t i = lane; i < s_nseq[w]; i += 32) {
        SeqRec r = stage[i];
        if (i == 0) r.ll += s_add[w];
        out[i] = r;
    }
    uint8_t *lo = lits + (size_t)b * ENC_BLOCK + s_loff[w];
    for (uint32_t i = lane; i < s_nlit[w]; i += 32) lo[i] = lstage[i];
}

// ------------------------------------------------------------------------------------------------------------
// k_copt (OPT, an extension, B200Z_LEVEL_OPT): the price-based parse.  The CTAs stride over the blocks; for each block:
//   chain  prev[q] for every position q in [-min(back, 131072), n - 4) is the nearest earlier position of the frame with the same
//          hash5(q, OPT_HASH_LOG), in the CTA's global slot.  Warp w builds stripe w of that range in position order 32 positions at
//          a time (__match_any_sync finds a lane's predecessor inside the round, a u16 head table per stripe the one before), then
//          the positions without one in their stripe take the last occurrence of the nearest earlier stripe's table.
//   prices the block's byte histogram prices a literal; a match pays OPT_MATCH_W plus its offset's code bits, or a repeat's weight.
//   parse  warp w parses segment w as a forward DP (opt_segment) over its parts between forced pieces.
// The packing is k_cmatch's.  tests/copt.py states the rule; the GPU must produce exactly its sequences.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t opt_log2(uint32_t x) {   // 256 floor(log2 x) + the 8 bits after the leading one (x >= 1)
    const uint32_t k = 31 - __clz(x);
    return 256 * k + ((k <= 8 ? x << (8 - k) : x >> (k - 8)) & 255u);
}

// a finder candidate in one word (0: none): length << 18 | offset at OPT (offsets <= 131072); at ULTRA (FAR) (length - 1) << 27 |
// (offset - 1), which holds offsets up to 2^27 and lengths 5..32
template <bool FAR> __device__ __forceinline__ uint32_t cand_pack(uint32_t ln, uint32_t o) { return FAR ? (ln - 1) << 27 | (o - 1) : ln << 18 | o; }
template <bool FAR> __device__ __forceinline__ uint32_t cand_len(uint32_t c) { return FAR ? (c >> 27) + 1 : c >> 18; }   // FAR: 1 for none
template <bool FAR> __device__ __forceinline__ uint32_t cand_off(uint32_t c) { return FAR ? (c & 0x7ffffffu) + 1 : c & 0x3ffffu; }

// ULTRA's far walk: the group's sorted (key8, virtual position) pairs and, per virtual position, where its walk starts (ldm.cu)
struct FarView {
    FBlock fb;
    const uint32_t *keys, *vals, *start;
};

// the finder's list of each position cb + lane (q + 5 <= stop), lengths increasing, into wk.cand
template <bool DICT, bool FAR>
__device__ __forceinline__ void opt_chunk(OptWarp &wk, const int32_t *prev, int32_t lo, const CBlock &blk, const uint8_t *src, uint32_t cb,
                                          uint32_t stop, const uint8_t *dict, const uint32_t *dtab, uint32_t dict_len, const FarView &fv,
                                          uint32_t lane) {
    const uint32_t q = cb + lane;
    uint32_t k0 = 0, k1 = 0, k2 = 0, k3 = 0, cnt = 0;
    auto push = [&](uint32_t v) {
        if (cnt == OPT_CANDS) { k0 = k1; k1 = k2; k2 = k3; cnt--; }   // the shortest drops out
        if (cnt == 0) k0 = v; else if (cnt == 1) k1 = v; else if (cnt == 2) k2 = v; else k3 = v;
        cnt++;
    };
    if (q + ENC_MIN_MATCH <= stop) {
        const uint32_t lim = min(OPT_SUFF, stop - q);
        uint32_t best = ENC_MIN_MATCH - 1;
        bool full = false;   // a verification reached its limit
        int32_t c = prev[(int32_t)q - lo];
        for (uint32_t seen = 0; c >= lo && (int32_t)q - c <= (int32_t)ENC_WINDOW && seen < OPT_DEPTH; seen++) {
            const uint32_t ln = match_len(src + q, src + c, lim);
            if (ln > best) {
                push(cand_pack<FAR>(ln, (uint32_t)((int32_t)q - c)));
                best = ln;
                if (ln == lim) { full = true; break; }
            }
            c = prev[c - lo];
        }
        // ULTRA: the same key8's earlier positions beyond 131072, nearest first, consecutive sorted pairs read backwards
        if (FAR && !full && fv.fb.vbase != FAR_NONE) {
            const uint32_t vq = fv.fb.vbase + q;
            uint32_t k = fv.start[vq];
            if (k != FAR_NONE) {
                const uint32_t key = fv.keys[k], reach = min(fv.fb.wf, fv.fb.back + q);
                for (uint32_t seen = 0; seen < FAR_DEPTH; seen++) {
                    const uint32_t d = vq - fv.vals[k];
                    if (d > reach) break;
                    const uint32_t ln = match_len(src + q, src + q - d, lim);
                    if (ln > best) {
                        push(cand_pack<FAR>(ln, d));
                        best = ln;
                        if (ln == lim) break;
                    }
                    if (k == 0 || fv.keys[--k] != key) break;
                }
            }
        }
        const uint32_t fpos = blk.back + q;
        if (DICT && fpos < ENC_WINDOW) {
            const uint32_t c3 = __ldg(dtab + hash5(src + q, CD_LOG));
            const uint32_t off3 = fpos + dict_len - (c3 - 1);
            if (c3 && off3 <= ENC_WINDOW) {
                const uint32_t ln = match_len(src + q, dict + (c3 - 1), min(lim, dict_len - (c3 - 1)));
                if (ln > best) push(cand_pack<FAR>(ln, off3));
            }
        }
    }
    uint32_t *out = wk.cand + lane * OPT_CANDS;
    out[0] = cnt > 0 ? k0 : 0u; out[1] = cnt > 1 ? k1 : 0u; out[2] = cnt > 2 ? k2 : 0u; out[3] = cnt > 3 ? k3 : 0u;
    __syncwarp();
}

// the length of repeat o at i (>= 5, else 0), verified for min(OPT_SUFF, stop - i) bytes; the source must lie in the frame and in
// the window wf (131072 at OPT, the frame's at ULTRA)
__device__ __forceinline__ uint32_t opt_rep(const uint8_t *src, uint32_t i, uint32_t o, uint32_t lim, uint32_t back, uint32_t wf, uint32_t lane) {
    const bool ok = o && o <= back + i && o <= wf;
    const bool stop = !ok || lane >= lim || __ldg(src + i + lane) != __ldg(src + i + lane - o);
    const uint32_t m = __ballot_sync(0xffffffffu, stop);
    const uint32_t ln = m ? __ffs(m) - 1 : 32u;
    return ok && ln >= ENC_MIN_MATCH ? ln : 0u;
}

// one warp's parse of segment [s, e) (see k_copt): the DPs of each part, forced pieces between them; staging as cmatch_lazy's
template <bool DICT, bool LONG, bool FAR>
__device__ __forceinline__ void opt_segment(OptWarp &wk, const int32_t *prev, int32_t lo, const uint32_t *lit, const CBlock &blk, const uint8_t *src,
                                            uint32_t s, uint32_t e, const uint8_t *dict, const uint32_t *dtab, uint32_t dict_len, SeqRec *stage,
                                            uint8_t *lstage, uint32_t *nseq_out, uint32_t *nlit_out, uint32_t *trail_out, LCursor &lc,
                                            const FarView &fv, uint32_t lane) {
    // the frame before the block that repeats may reach, and their window: at ULTRA the far stage's (up to Wf), else 131072
    const uint32_t rback = FAR ? fv.fb.back : blk.back, rwf = FAR ? fv.fb.wf : ENC_WINDOW;
    uint32_t p = s, anchor = s, nseq = 0, nlit = 0;
    uint32_t r0 = 0, r1 = 0, r2 = 0;   // the reps at p (0: none yet)
    auto push_rep = [&](uint32_t o) {
        if (o == r1) { r1 = r0; r0 = o; }
        else if (o != r0) { r2 = r1; r1 = r0; r0 = o; }
    };
    auto emit = [&](uint32_t q, uint32_t ml, uint32_t off) {
        for (uint32_t i = anchor + lane; i < q; i += 32) lstage[nlit + i - anchor] = __ldg(src + i);
        if (lane == 0) stage[nseq] = SeqRec{q - anchor, ml, off};
        nlit += q - anchor;
        nseq++;
        anchor = q + ml;
    };
    uint32_t stop = e;
    if constexpr (LONG) { lc.next(); if (lc.has) stop = lc.cs; }
    while (true) {
        while (p < stop) {   // one DP from a = p
            const uint32_t a = p;
            uint32_t end = min(stop, a + OPT_WIN);
            for (uint32_t k = lane; k < OPT_NODES; k += 32) wk.cost[k] = OPT_INF;
            __syncwarp();
            if (lane == 0) { wk.cost[0] = 0; wk.rep[0][0] = r0; wk.rep[1][0] = r1; wk.rep[2][0] = r2; }
            uint32_t cb = a;
            opt_chunk<DICT, FAR>(wk, prev, lo, blk, src, cb, stop, dict, dtab, dict_len, fv, lane);
            uint32_t tml = 0, toff = 0;   // a match taken at once at `end`
            for (uint32_t i = a; i < end; i++) {
                if (i >= cb + 32) { cb = i; opt_chunk<DICT, FAR>(wk, prev, lo, blk, src, cb, stop, dict, dtab, dict_len, fv, lane); }
                const uint32_t k = i - a, ci = wk.cost[k], x0 = wk.rep[0][k], x1 = wk.rep[1][k], x2 = wk.rep[2][k];
                const uint32_t *cl = wk.cand + (i - cb) * OPT_CANDS;
                const uint32_t c0 = cl[0], c1 = cl[1], c2 = cl[2], c3 = cl[3];
                uint32_t l0 = 0, l1 = 0, l2 = 0;
                if (i + ENC_MIN_MATCH <= stop) {
                    const uint32_t lim = min(OPT_SUFF, stop - i);
                    l0 = opt_rep(src, i, x0, lim, rback, rwf, lane);
                    l1 = opt_rep(src, i, x1, lim, rback, rwf, lane);
                    l2 = opt_rep(src, i, x2, lim, rback, rwf, lane);
                }
                // a candidate of OPT_SUFF bytes closes the DP: the longest, the first of rep0, rep1, rep2, the finder's on a tie
                const uint32_t ctop = c3 ? c3 : c2 ? c2 : c1 ? c1 : c0;
                if (l0 >= OPT_SUFF && l0 > tml) { tml = l0; toff = x0; }
                if (l1 >= OPT_SUFF && l1 > tml) { tml = l1; toff = x1; }
                if (l2 >= OPT_SUFF && l2 > tml) { tml = l2; toff = x2; }
                if (cand_len<FAR>(ctop) >= OPT_SUFF && cand_len<FAR>(ctop) > tml) { tml = cand_len<FAR>(ctop); toff = cand_off<FAR>(ctop); }
                if (tml) { end = i; break; }
                // lane l relaxes node i + l: the literal (l = 1), a match of l bytes (l >= 5)
                uint32_t c = OPT_INF, off = 0;
                if (lane == 1) c = ci + lit[__ldg(src + i)];
                else if (lane >= ENC_MIN_MATCH) {
                    uint32_t best = OPT_INF;
                    if (l0 >= lane) { best = OPT_REP_W0; off = x0; }
                    if (l1 >= lane && OPT_REP_W1 < best) { best = OPT_REP_W1; off = x1; }
                    if (l2 >= lane && OPT_REP_W2 < best) { best = OPT_REP_W2; off = x2; }
                    uint32_t f;   // the first finder candidate of >= lane bytes (OPT's expression kept as it was: the same SASS)
                    if constexpr (FAR) f = cand_len<FAR>(c0) >= lane ? c0 : cand_len<FAR>(c1) >= lane ? c1 : cand_len<FAR>(c2) >= lane ? c2 : cand_len<FAR>(c3) >= lane ? c3 : 0u;
                    else f = (c0 >> 18) >= lane ? c0 : (c1 >> 18) >= lane ? c1 : (c2 >> 18) >= lane ? c2 : (c3 >> 18) >= lane ? c3 : 0u;
                    if (f) {
                        const uint32_t o = cand_off<FAR>(f), pr = 256 * (31 - __clz(o + 3)) + OPT_OF_W;
                        if (pr < best) { best = pr; off = o; }
                    }
                    if (best != OPT_INF) c = ci + OPT_MATCH_W + best;
                }
                const uint32_t t = k + lane;
                if (c != OPT_INF && c < wk.cost[t]) {
                    wk.cost[t] = c;
                    wk.link[t] = k | (lane == 1 ? 0u : lane << 16);
                    wk.off[t] = off;
                    if (lane == 1 || off == x0) { wk.rep[0][t] = x0; wk.rep[1][t] = x1; wk.rep[2][t] = x2; }
                    else if (off == x1) { wk.rep[0][t] = off; wk.rep[1][t] = x0; wk.rep[2][t] = x2; }
                    else { wk.rep[0][t] = off; wk.rep[1][t] = x0; wk.rep[2][t] = x1; }
                }
                __syncwarp();
            }
            // close at `end`: the path's matches (lane 0 walks it back), then the taken match
            uint32_t np = 0;
            if (lane == 0) {
                for (uint32_t k = end - a; k;) {
                    const uint32_t lk = wk.link[k], f = lk & 0xffffu;
                    if (lk >> 16) { wk.path_pos[np] = a + f; wk.path_ml[np] = lk >> 16; wk.path_off[np] = wk.off[k]; np++; }
                    k = f;
                }
            }
            np = __shfl_sync(0xffffffffu, np, 0);
            __syncwarp();
            for (uint32_t j = np; j-- > 0;) emit(wk.path_pos[j], wk.path_ml[j], wk.path_off[j]);
            r0 = wk.rep[0][end - a]; r1 = wk.rep[1][end - a]; r2 = wk.rep[2][end - a];
            p = end;
            if (tml) {
                const uint32_t fpos = rback + end;
                const uint32_t xlim = DICT && toff > fpos ? min(stop - end, toff - fpos) : stop - end;   // a dictionary source: to its end
                const uint32_t ml = extend_match<DICT>(src, end, toff, tml, xlim, rback, dict, dict_len, lane);
                emit(end, ml, toff);
                push_rep(toff);
                p = end + ml;
            }
            __syncwarp();
        }
        if constexpr (!LONG) break;
        else {
            if (!lc.has) break;
            emit(lc.cs, lc.ce - lc.cs, lc.off);   // the forced piece, taken as any match is
            push_rep(lc.off);
            p = lc.ce;
            lc.next();
            stop = lc.has ? lc.cs : e;
            __syncwarp();
        }
    }
    for (uint32_t i = anchor + lane; i < e; i += 32) lstage[nlit + i - anchor] = __ldg(src + i);
    if (lane == 0) { *nseq_out = nseq; *nlit_out = nlit + (e - anchor); *trail_out = e - anchor; }
}

template <bool DICT, bool LONG, bool FAR = false>
__global__ void __launch_bounds__(CM_THREADS, 1)
k_copt(const CBlock *__restrict__ blocks, uint32_t nblocks, const uint8_t *__restrict__ input, uint8_t *__restrict__ lit_stage,
       SeqRec *__restrict__ seq_stage, uint8_t *__restrict__ lits, SeqRec *__restrict__ seqs, CBlockInfo *__restrict__ info,
       const uint8_t *__restrict__ dict, const uint32_t *__restrict__ dtab, uint32_t dict_len, int32_t *opt_prev,
       const LForced *__restrict__ lforced, const uint32_t *__restrict__ lf_off, const uint32_t *__restrict__ lf_cnt,
       const FBlock *__restrict__ fblk, const uint32_t *__restrict__ fkeys, const uint32_t *__restrict__ fvals,
       const uint32_t *__restrict__ fstart) {
    extern __shared__ __align__(16) uint8_t smem_co[];
    __shared__ uint32_t s_nseq[CM_WARPS], s_nlit[CM_WARPS], s_trail[CM_WARPS], s_add[CM_WARPS], s_soff[CM_WARPS], s_loff[CM_WARPS];
    __shared__ uint32_t s_lit[256];
    const uint32_t tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
    int32_t *prev = opt_prev + (size_t)blockIdx.x * OPT_SPAN;
    uint16_t *heads = reinterpret_cast<uint16_t *>(smem_co);
    OptWarp &wk = reinterpret_cast<OptWarp *>(smem_co)[w];
    for (uint32_t b = blockIdx.x; b < nblocks; b += gridDim.x) {
        const CBlock blk = blocks[b];
        const uint8_t *src = input + blk.src_off;
        const uint32_t n = blk.size;
        bool same = true;
        for (uint32_t i = tid; i < n; i += CM_THREADS) same &= __ldg(src + i) == __ldg(src);
        same = __syncthreads_and(same);
        if (n == 0 || same) {
            if (tid == 0) info[b] = CBlockInfo{n, 0, n ? 1u : 0u, 0};
            continue;
        }
        // prices: the block's byte histogram
        for (uint32_t i = tid; i < 256; i += CM_THREADS) s_lit[i] = 0;
        for (uint32_t i = tid; i < CM_WARPS << OPT_HASH_LOG; i += CM_THREADS) heads[i] = 0xffffu;
        __syncthreads();
        for (uint32_t i = tid; i < n; i += CM_THREADS) atomicAdd(&s_lit[__ldg(src + i)], 1u);
        // the chain, stripe w
        const int32_t lo = -(int32_t)min(blk.back, ENC_WINDOW), hi = (int32_t)n - 4;
        const int32_t slen = (hi - lo + (int32_t)CM_WARPS - 1) / (int32_t)CM_WARPS;
        const int32_t s0 = lo + (int32_t)w * slen, s1 = min(hi, s0 + slen);
        uint16_t *hd = heads + (w << OPT_HASH_LOG);
        for (int32_t c0 = s0; c0 < s1; c0 += 32) {
            const int32_t q = c0 + (int32_t)lane;
            const bool valid = q < s1;
            const uint32_t h = valid ? hash5(src + q, OPT_HASH_LOG) : (1u << OPT_HASH_LOG) + lane;
            const uint32_t grp = __match_any_sync(0xffffffffu, h), lower = grp & ((1u << lane) - 1);
            int32_t pv = OPT_FIX;
            if (lower) pv = c0 + 31 - __clz(lower);
            else if (valid && hd[h] != 0xffffu) pv = s0 + hd[h];
            __syncwarp();
            if (valid && lane == 31 - __clz(grp)) hd[h] = (uint16_t)(q - s0);
            if (valid) prev[q - lo] = pv;
            __syncwarp();
        }
        __syncthreads();
        if (tid < 256) s_lit[tid] = s_lit[tid] ? opt_log2(n) - opt_log2(s_lit[tid]) : OPT_INF;
        for (int32_t q = s0 + (int32_t)lane; q < s1; q += 32) {
            if (prev[q - lo] != OPT_FIX) continue;
            const uint32_t h = hash5(src + q, OPT_HASH_LOG);
            int32_t pv = OPT_NONE;
            for (int32_t v = (int32_t)w - 1; v >= 0; v--) {
                const uint32_t r = heads[((uint32_t)v << OPT_HASH_LOG) + h];
                if (r != 0xffffu) { pv = lo + v * slen + (int32_t)r; break; }
            }
            prev[q - lo] = pv;
        }
        __syncthreads();   // the chain is complete; the heads' memory becomes the warps' DP state
        const uint32_t seglen = (n + CM_WARPS - 1) / CM_WARPS;
        const uint32_t s = min(n, w * seglen), e = min(n, s + seglen);
        LCursor lc{};
        if constexpr (LONG) lc = LCursor{lforced + lf_off[b], 0, lf_cnt[b], s, e, 0, 0, 0, false};
        FarView fv{};
        if constexpr (FAR) fv = FarView{fblk[b], fkeys, fvals, fstart};
        {
            SeqRec *stage = seq_stage + ((size_t)b * CM_WARPS + w) * CSEG_SEQS;
            uint8_t *lstage = lit_stage + (size_t)b * ENC_BLOCK + s;
            opt_segment<DICT, LONG, FAR>(wk, prev, lo, s_lit, blk, src, s, e, dict, dtab, dict_len, stage, lstage, s_nseq + w, s_nlit + w, s_trail + w, lc,
                                         fv, lane);
        }
        __syncthreads();
        if (tid == 0) {   // k_cmatch's packing
            uint32_t carry = 0, so = 0, lo2 = 0;
            for (uint32_t v = 0; v < CM_WARPS; v++) {
                s_soff[v] = so; s_loff[v] = lo2;
                so += s_nseq[v]; lo2 += s_nlit[v];
                if (s_nseq[v]) { s_add[v] = carry; carry = s_trail[v]; }
                else { s_add[v] = 0; carry += s_trail[v]; }
            }
            info[b] = CBlockInfo{lo2, so, 0, 0};
        }
        __syncthreads();
        SeqRec *stage = seq_stage + ((size_t)b * CM_WARPS + w) * CSEG_SEQS;
        uint8_t *lstage = lit_stage + (size_t)b * ENC_BLOCK + s;
        SeqRec *out = seqs + (size_t)b * CBLOCK_SEQS + s_soff[w];
        for (uint32_t i = lane; i < s_nseq[w]; i += 32) {
            SeqRec r = stage[i];
            if (i == 0) r.ll += s_add[w];
            out[i] = r;
        }
        uint8_t *lout = lits + (size_t)b * ENC_BLOCK + s_loff[w];
        for (uint32_t i = lane; i < s_nlit[w]; i += 32) lout[i] = lstage[i];
        __syncthreads();   // before the next block's histogram, heads and counts
    }
}

// ------------------------------------------------------------------------------------------------------------
// k_cenc: one warp per block encodes its literals and sequences (encode_block) into the block's staging slot and decides the
// block type: RLE when all bytes are equal, Compressed when smaller than the input block, else Raw.  A formatted dictionary's
// tables (dt, B200Z_FLAG_DICT_TABLES) go to a frame's first block only (back == 0); without them (TABLES = false) encode_block gets
// a constant nullptr, so the plain path carries none of that code.
// With REPS (LAZY) the warp first writes the block's records with repeat-offset codes to rseqs (rep_pass) and encodes those.
// ------------------------------------------------------------------------------------------------------------
// LAZY: the decoder's offset history (RFC 8878 3.1.2.5) over one block's sequences, from three unknown slots (0; an offset is
// >= 1), so no block depends on another's encoding.  A sequence whose offset a known slot can name gets that Offset_Value
// (LL > 0: rep0 / rep1 / rep2 -> 1 / 2 / 3; LL = 0: rep1 / rep2 / rep0 - 1 -> 1 / 2 / 3), any other offset o is coded raw (o + 3);
// out[i].of = Offset_Value - 3 (mod 2^32), which encode_block codes as that Offset_Value.  The warp loads 32 records at a time
// and every lane runs the (uniform) history over them, keeping its own record's code.
__device__ __forceinline__ void rep_pass(const SeqRec *in, uint32_t nseq, SeqRec *out, uint32_t lane) {
    uint32_t h0 = 0, h1 = 0, h2 = 0;
    for (uint32_t b0 = 0; b0 < nseq; b0 += 32) {
        const uint32_t i = b0 + lane, cnt = min(32u, nseq - b0);
        const SeqRec r = i < nseq ? in[i] : SeqRec{0, 0, 0};
        uint32_t mine = 0;
        for (uint32_t k = 0; k < cnt; k++) {
            const uint32_t ll = __shfl_sync(0xffffffffu, r.ll, k), o = __shfl_sync(0xffffffffu, r.of, k);
            uint32_t ov;
            if (ll) ov = h0 == o ? 1u : h1 == o ? 2u : h2 == o ? 3u : o + 3;
            else ov = h1 == o ? 1u : h2 == o ? 2u : h0 && h0 - 1 == o ? 3u : o + 3;
            const uint32_t rep = ov > 3 ? 4u : ov - 1 + (ll == 0);   // 4: raw
            if (rep == 1) { h1 = h0; h0 = o; }
            else if (rep == 2) { h2 = h1; h1 = h0; h0 = o; }
            else if (rep >= 3) { h2 = h1; h1 = h0; h0 = o; }
            if (k == lane) mine = ov;
        }
        if (i < nseq) out[i] = SeqRec{r.ll, r.ml, mine - 3};
    }
    __syncwarp();
}

template <bool TABLES, bool REPS>
__global__ void __launch_bounds__(CE_WARPS * 32)
k_cenc(const CBlock *__restrict__ blocks, uint32_t nblocks, const CBlockInfo *__restrict__ info, const uint8_t *__restrict__ lits,
       const SeqRec *__restrict__ seqs, uint8_t *__restrict__ enc, CBlockInfo *__restrict__ res, const EncDict *__restrict__ dt,
       SeqRec *__restrict__ rseqs) {
    __shared__ EncScratch scratch[CE_WARPS];
    const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.x * CE_WARPS + w;
    if (b >= nblocks) return;
    const CBlockInfo in = info[b];
    const uint32_t n = blocks[b].size;
    const EncDict *bdt = TABLES && blocks[b].back == 0 ? dt : nullptr;
    uint32_t type = 0, csize = n;
    if (in.type == 1) { type = 1; csize = 1; }
    else if (n) {
        if (REPS) rep_pass(seqs + (size_t)b * CBLOCK_SEQS, in.nseq, rseqs + (size_t)b * CBLOCK_SEQS, lane);
        const uint32_t size = encode_block(scratch[w], lits + (size_t)b * ENC_BLOCK, in.nlit, REPS ? rseqs + (size_t)b * CBLOCK_SEQS : seqs + (size_t)b * CBLOCK_SEQS, in.nseq,
                                           enc + (size_t)b * ENC_BLOCK, ENC_BLOCK, lane, 32, TABLES ? bdt : nullptr);
        if (size < n) { type = 2; csize = size; }
    }
    if (lane == 0) res[b] = CBlockInfo{in.nlit, in.nseq, type, csize};
}

__global__ void k_cxxh64(const CFrame *__restrict__ frames, const uint8_t *__restrict__ input, uint64_t *__restrict__ csum, uint32_t nframes) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t f = t >> 2, k = t & 3;
    if (f >= nframes) return;
    const uint64_t h = xxh64_group(input + frames[f].src_off, frames[f].src_size, k);
    if (k == 0) csum[f] = h;
}

// ------------------------------------------------------------------------------------------------------------
// k_cassemble: one CTA per block.  Its offset inside the frame is the sum of the sizes of the blocks before it (read by the
// whole CTA); the first block also writes the frame header, the last one the checksum and the frame's result.
// With STREAM (b200z_frame_compressor) a CFrame is one chunk of a frame whose header, trailing empty block and checksum the host
// writes: the blocks are packed from the chunk's dst_off, and only a chunk that ends inside a block (the source ended there)
// sets the last-block bit on its last block.  Its result holds the chunk's packed size and block counts.  With DLONG
// (B200Z_FLAG_DICT_LONG) the Window_Descriptor is frame_window_log of src_size + ldict_len.
// ------------------------------------------------------------------------------------------------------------
template <bool STREAM, bool DLONG>
__global__ void __launch_bounds__(256)
k_cassemble(const CFrame *__restrict__ frames, const CBlock *__restrict__ blocks, const CBlockInfo *__restrict__ res, const uint8_t *__restrict__ enc,
            const uint8_t *__restrict__ input, const uint64_t *__restrict__ csum, uint8_t *__restrict__ output, b200z_compress_result *__restrict__ results,
            int level, int checksum, uint32_t dict_id, uint32_t window_log, uint64_t ldict_len) {
    __shared__ uint64_t s_red[3][8];
    const uint32_t b = blockIdx.x, tid = threadIdx.x;
    const CBlock blk = blocks[b];
    const CFrame fr = frames[blk.frame];
    const bool end = b == fr.first_block + fr.nblocks - 1;   // the CFrame's last block
    const bool last = end && (!STREAM || fr.src_size % ENC_BLOCK != 0);
    uint64_t before = 0, nraw = 0, nrle = 0;
    for (uint32_t i = fr.first_block + tid; i < b + (end ? 1u : 0u); i += 256) {
        const uint32_t t = level == 0 ? 0u : res[i].type;
        const uint32_t sz = 3 + (t == 0 ? blocks[i].size : t == 1 ? 1u : res[i].csize);
        if (i < b) before += sz;
        nraw += t == 0;
        nrle += t == 1;
    }
    for (int o = 16; o; o >>= 1) {
        before += __shfl_xor_sync(0xffffffffu, before, o);
        nraw += __shfl_xor_sync(0xffffffffu, nraw, o);
        nrle += __shfl_xor_sync(0xffffffffu, nrle, o);
    }
    if ((tid & 31) == 0) { s_red[0][tid >> 5] = before; s_red[1][tid >> 5] = nraw; s_red[2][tid >> 5] = nrle; }
    __syncthreads();
    before = nraw = nrle = 0;
    for (int i = 0; i < 8; i++) { before += s_red[0][i]; nraw += s_red[1][i]; nrle += s_red[2][i]; }
    const uint32_t hdr = STREAM ? 0u : frame_header_size(fr.src_size, dict_id);
    uint8_t *dst = output + fr.dst_off + hdr + before;
    const uint32_t type = level == 0 ? 0u : res[b].type;
    const uint32_t csize = type == 0 ? blk.size : type == 1 ? 1u : res[b].csize;
    const uint8_t *from = type == 2 ? enc + (size_t)b * ENC_BLOCK : input + blk.src_off;
    if (tid == 0) {
        const uint32_t bh = (last ? 1u : 0u) | (type << 1) | ((type == 1 ? blk.size : csize) << 3);
        dst[0] = (uint8_t)bh; dst[1] = (uint8_t)(bh >> 8); dst[2] = (uint8_t)(bh >> 16);
        if (!STREAM && b == fr.first_block)
            write_frame_header(output + fr.dst_off, fr.src_size, checksum != 0, dict_id,
                               frame_window_log(DLONG ? fr.src_size + ldict_len : fr.src_size, window_log));
    }
    for (uint32_t i = tid; i < csize; i += 256) dst[3 + i] = from[i];
    if (end && tid == 0) {
        const bool sum = !STREAM && checksum;
        const uint32_t c = sum ? (uint32_t)csum[blk.frame] : 0u;
        uint64_t size = hdr + before + 3 + csize;
        if (sum) { for (int i = 0; i < 4; i++) dst[3 + csize + i] = (uint8_t)(c >> (8 * i)); size += 4; }
        b200z_compress_result r;
        r.dst_size = size; r.status = 0; r.blocks = fr.nblocks; r.raw_blocks = (uint32_t)nraw; r.rle_blocks = (uint32_t)nrle;
        r.has_checksum = sum ? 1u : 0u; r.checksum = c;
        results[blk.frame] = r;
    }
}

// ------------------------------------------------------------------------------------------------------------
// k_cdict: the dictionary's match table.  The host hands it the dictionary's last ENC_WINDOW bytes (nothing further back can be
// referenced); every position with 5 bytes before their end goes under its 5-byte hash, the most recent position winning
// (atomicMax, so the table does not depend on the schedule).  Entries hold position + 1 over a zeroed table.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_cdict(const uint8_t *__restrict__ dict, uint32_t end, uint32_t *__restrict__ dtab) {
    const uint32_t d = blockIdx.x * 256 + threadIdx.x;
    if (d < end) atomicMax(&dtab[hash5(dict + d, CD_LOG)], d + 1);
}

// ------------------------------------------------------------------------------------------------------------
// k_dstats: the entropy statistics of a dictionary's training samples (b200z_dict_finalize).  One CTA per parsed block (k_cmatch
// against the dictionary's content): the histograms of its literal bytes and of its sequences' LL / ML / OF codes, as the
// encoder codes them (offsets raw as offset + 3), in shared memory, then added to the u64 totals.  RLE blocks are left out:
// the encoder writes no literals or sequences for them.  Integer atomics only, so the totals do not depend on the schedule.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(DS_THREADS)
k_dstats(const CBlockInfo *__restrict__ info, const uint8_t *__restrict__ lits, const SeqRec *__restrict__ seqs,
         unsigned long long *__restrict__ counts) {
    __shared__ uint32_t h[DS_BINS];
    const uint32_t b = blockIdx.x, tid = threadIdx.x;
    const CBlockInfo in = info[b];
    if (in.type == 1) return;
    for (uint32_t i = tid; i < DS_BINS; i += DS_THREADS) h[i] = 0;
    __syncthreads();
    const uint8_t *l = lits + (size_t)b * ENC_BLOCK;
    for (uint32_t i = tid; i < in.nlit; i += DS_THREADS) atomicAdd(&h[DS_LIT + __ldg(l + i)], 1u);
    const SeqRec *q = seqs + (size_t)b * CBLOCK_SEQS;
    for (uint32_t i = tid; i < in.nseq; i += DS_THREADS) {
        const SeqRec r = q[i];
        atomicAdd(&h[DS_LL + ll_code(r.ll)], 1u);
        atomicAdd(&h[DS_ML + ml_code(r.ml)], 1u);
        atomicAdd(&h[DS_OF + of_code(r.of)], 1u);
    }
    __syncthreads();
    for (uint32_t i = tid; i < DS_BINS; i += DS_THREADS)
        if (h[i]) atomicAdd(&counts[i], (unsigned long long)h[i]);
}

static uint32_t g_opt_ctas = 1;   // init_compress_kernels: the SMs times k_copt's CTAs per SM

static uint32_t cdiv_u(uint64_t a, uint32_t b) { return (uint32_t)((a + b - 1) / b); }

int launch_dict_stats(const CompressArgs &a, unsigned long long *counts, cudaStream_t s, uint64_t *launched) {
    if (!a.nblocks) return 0;
    k_cmatch<true, false><<<a.nblocks, CM_THREADS, CM_SMEM, s>>>(a.blocks, a.input, a.lit_stage, a.seq_stage, a.lits, a.seqs, a.info, a.dict, a.dtab, a.dict_len);
    int e = (int)cudaGetLastError();
    if (e) return e;
    ++*launched;
    k_dstats<<<a.nblocks, DS_THREADS, 0, s>>>(a.info, a.lits, a.seqs, counts);
    e = (int)cudaGetLastError();
    if (!e) ++*launched;
    return e;
}

int init_compress_kernels() {
    cudaError_t e = cudaFuncSetAttribute(k_cmatch<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CM_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cmatch<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CM_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cmatch<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LZ_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cmatch<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LZ_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cmatch<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CM_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cmatch<true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CM_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cmatch<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LZ_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_cmatch<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LZ_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_copt<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OPT_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_copt<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OPT_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_copt<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OPT_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_copt<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OPT_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_copt<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OPT_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_copt<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OPT_SMEM);
    int dev = 0, sms = 0, per = 0;
    if (e == cudaSuccess) e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_copt<true, true>, CM_THREADS, OPT_SMEM);
    if (e == cudaSuccess) g_opt_ctas = (uint32_t)std::max(1, sms * per);
    return (int)e;
}

uint32_t opt_ctas() { return g_opt_ctas; }

int launch_dict_table(const uint8_t *dict, uint32_t len, uint32_t *dtab, cudaStream_t s, uint64_t *launched) {
    int e = (int)cudaMemsetAsync(dtab, 0, sizeof(uint32_t) << CD_LOG, s);
    if (e || len < ENC_MIN_MATCH) return e;
    const uint32_t end = len - ENC_MIN_MATCH + 1;
    k_cdict<<<cdiv_u(end, 256), 256, 0, s>>>(dict, end, dtab);
    e = (int)cudaGetLastError();
    if (!e) ++*launched;
    return e;
}

const char *const kCompressStageNames[kCompressStages] = {"k_cmatch", "k_cenc", "k_cxxh64", "k_cassemble"};

int launch_compress_stage(const CompressArgs &a, int stage, cudaStream_t s, uint64_t *launched) {
    const bool lazy = a.level == B200Z_LEVEL_LAZY, opt = a.level == B200Z_LEVEL_OPT || a.level == B200Z_LEVEL_ULTRA;
    switch (stage) {
    case 0:
        if (!a.level || !a.nblocks) return 0;
        if (opt && a.fblk) {   // ULTRA with a far stage (always with the long-distance matches: both need window_log > 17)
            if (!a.lf_cnt) return (int)cudaErrorInvalidValue;
            auto k = a.dtab ? k_copt<true, true, true> : k_copt<false, true, true>;
            k<<<std::min(a.nblocks, g_opt_ctas), CM_THREADS, OPT_SMEM, s>>>(a.blocks, a.nblocks, a.input, a.lit_stage, a.seq_stage, a.lits, a.seqs, a.info,
                                                                         a.dict, a.dtab, a.dict_len, a.opt_prev, a.lforced, a.lf_off, a.lf_cnt,
                                                                         a.fblk, a.fkeys, a.fvals, a.fstart);
        } else if (opt) {
            auto k = a.lf_cnt ? (a.dtab ? k_copt<true, true> : k_copt<false, true>) : (a.dtab ? k_copt<true, false> : k_copt<false, false>);
            k<<<std::min(a.nblocks, g_opt_ctas), CM_THREADS, OPT_SMEM, s>>>(a.blocks, a.nblocks, a.input, a.lit_stage, a.seq_stage, a.lits, a.seqs, a.info,
                                                                         a.dict, a.dtab, a.dict_len, a.opt_prev, a.lforced, a.lf_off, a.lf_cnt,
                                                                         nullptr, nullptr, nullptr, nullptr);
        } else if (a.lf_cnt) {
            const uint32_t smem = lazy ? LZ_SMEM : CM_SMEM;
            auto k = lazy ? (a.dtab ? k_cmatch<true, true, true> : k_cmatch<false, true, true>) : (a.dtab ? k_cmatch<true, false, true> : k_cmatch<false, false, true>);
            k<<<a.nblocks, CM_THREADS, smem, s>>>(a.blocks, a.input, a.lit_stage, a.seq_stage, a.lits, a.seqs, a.info, a.dict, a.dtab, a.dict_len,
                                                  a.lforced, a.lf_off, a.lf_cnt);
        } else if (lazy) {
            if (a.dtab) k_cmatch<true, true><<<a.nblocks, CM_THREADS, LZ_SMEM, s>>>(a.blocks, a.input, a.lit_stage, a.seq_stage, a.lits, a.seqs, a.info, a.dict, a.dtab, a.dict_len);
            else k_cmatch<false, true><<<a.nblocks, CM_THREADS, LZ_SMEM, s>>>(a.blocks, a.input, a.lit_stage, a.seq_stage, a.lits, a.seqs, a.info, nullptr, nullptr, 0);
        } else if (a.dtab) k_cmatch<true, false><<<a.nblocks, CM_THREADS, CM_SMEM, s>>>(a.blocks, a.input, a.lit_stage, a.seq_stage, a.lits, a.seqs, a.info, a.dict, a.dtab, a.dict_len);
        else k_cmatch<false, false><<<a.nblocks, CM_THREADS, CM_SMEM, s>>>(a.blocks, a.input, a.lit_stage, a.seq_stage, a.lits, a.seqs, a.info, nullptr, nullptr, 0);
        break;
    case 1:   // LAZY's, OPT's and ULTRA's repeat-offset records go to seq_stage, free once k_cmatch / k_copt is done
        if (!a.level || !a.nblocks) return 0;
        if (lazy || opt) {
            if (a.etab) k_cenc<true, true><<<cdiv_u(a.nblocks, CE_WARPS), CE_WARPS * 32, 0, s>>>(a.blocks, a.nblocks, a.info, a.lits, a.seqs, a.enc, a.res, a.etab, a.seq_stage);
            else k_cenc<false, true><<<cdiv_u(a.nblocks, CE_WARPS), CE_WARPS * 32, 0, s>>>(a.blocks, a.nblocks, a.info, a.lits, a.seqs, a.enc, a.res, nullptr, a.seq_stage);
        } else if (a.etab) k_cenc<true, false><<<cdiv_u(a.nblocks, CE_WARPS), CE_WARPS * 32, 0, s>>>(a.blocks, a.nblocks, a.info, a.lits, a.seqs, a.enc, a.res, a.etab, nullptr);
        else k_cenc<false, false><<<cdiv_u(a.nblocks, CE_WARPS), CE_WARPS * 32, 0, s>>>(a.blocks, a.nblocks, a.info, a.lits, a.seqs, a.enc, a.res, nullptr, nullptr);
        break;
    case 2: if (!a.checksum || !a.nframes) return 0; k_cxxh64<<<cdiv_u((uint64_t)a.nframes * 4, 128), 128, 0, s>>>(a.frames, a.input, a.csum, a.nframes); break;
    case 3:
        if (!a.nblocks) return 0;
        if (a.ldict_len) k_cassemble<false, true><<<a.nblocks, 256, 0, s>>>(a.frames, a.blocks, a.res, a.enc, a.input, a.csum, a.output, a.results, a.level, a.checksum, a.dict_id, a.window_log, a.ldict_len);
        else k_cassemble<false, false><<<a.nblocks, 256, 0, s>>>(a.frames, a.blocks, a.res, a.enc, a.input, a.csum, a.output, a.results, a.level, a.checksum, a.dict_id, a.window_log, 0);
        break;
    default: return (int)cudaErrorInvalidValue;
    }
    const int e = (int)cudaGetLastError();
    if (!e) ++*launched;
    return e;
}

int launch_compress_chunk(const CompressArgs &a, cudaStream_t s, uint64_t *launched) {
    if (!a.nblocks) return 0;
    for (int st = 0; st < 2; st++)
        if (int e = launch_compress_stage(a, st, s, launched)) return e;
    k_cassemble<true, false><<<a.nblocks, 256, 0, s>>>(a.frames, a.blocks, a.res, a.enc, a.input, nullptr, a.output, a.results, a.level, 0, 0, 0, 0);
    const int e = (int)cudaGetLastError();
    if (!e) ++*launched;
    return e;
}

}  // namespace b200z
