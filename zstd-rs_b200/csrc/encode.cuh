// encode.cuh -- zstd block encoding (the format half of the compressor), compiled for BOTH device and host.
//
// k_cenc runs encode_block with one warp per block (lane = 0..31); the host unit test (tests/host/encode_test.cpp) runs the
// same function with a single lane.  What it writes follows ruzstd's compress_block (encoding/blocks/compressed.rs):
//   literals   Raw when there are <= 1024 of them or Huffman does not pay, else Compressed with 4 streams and a fresh table
//              (never Treeless); code lengths <= 11, weights in the direct 4-bit form when legal, FSE-compressed otherwise
//   sequences  offsets coded raw as offset + 3 (no repeat offsets, compressed.rs:27); per table FSE_Compressed with an
//              accuracy log <= 9 / 8 / 9 for LL / OF / ML (compressed.rs:55-72), RLE when the block has a single code;
//              never Repeat
// No block depends on another block's encoding, which is what lets every block of every frame be encoded at once.
// With a formatted dictionary's tables (EncDict, B200Z_FLAG_DICT_TABLES; k_cenc passes them for a frame's first block only, the
// one block where the format makes them the "previous" tables) encode_block may also choose Treeless literals with the
// dictionary's Huffman codes and, per sequence table, Repeat with the dictionary's FSE table; without them it writes the above.
#pragma once
#include <stdint.h>

#include "tables.cuh"

#ifdef __CUDA_ARCH__
#define B200Z_ENC_ADD(p, v) atomicAdd((p), (v))
#define B200Z_ENC_SYNC() __syncwarp()
#else
#define B200Z_ENC_ADD(p, v) (*(p) += (v))
#define B200Z_ENC_SYNC() ((void)0)
#endif

namespace b200z {

constexpr uint32_t ENC_BLOCK = 131072;       // MAX_BLOCK_SIZE
constexpr uint32_t ENC_WINDOW = 131072;      // MatchGeneratorDriver::new(1024 * 128, 1), frame_compressor.rs:83
constexpr uint32_t ENC_MIN_MATCH = 5;        // match_generator.rs:15
constexpr uint32_t ENC_HUF_MAX_BITS = 11;
constexpr uint32_t ENC_RAW_LITERALS_MAX = 1024;
constexpr uint32_t ENC_LL = 0, ENC_OF = 1, ENC_ML = 2;

struct SeqRec { uint32_t ll, ml, of; };   // literal length, match length (>= 3), offset (>= 1)

B200Z_HD uint32_t flog2(uint32_t x) { return hbs(x) - 1u; }   // floor(log2 x), x > 0
B200Z_HD uint32_t enc_max_log(uint32_t t) { return t == ENC_OF ? 8u : 9u; }
B200Z_HD uint32_t enc_max_sym(uint32_t t) { return t == ENC_LL ? 35u : t == ENC_OF ? 31u : 52u; }

// code of a value and its number of extra bits; the baselines are multiples of 2^bits, so the extra bits are the value's
// low bits (same tables as c_ll_base / c_ml_base in kernels.cu)
B200Z_HD uint32_t ll_code(uint32_t ll) {
    if (ll < 16) return ll;
    if (ll < 24) return 16 + ((ll - 16) >> 1);
    if (ll < 32) return 20 + ((ll - 24) >> 2);
    if (ll < 48) return 22 + ((ll - 32) >> 3);
    if (ll < 64) return 24;
    return flog2(ll) + 19;
}
B200Z_HD uint32_t ll_bits(uint32_t c) { return c < 16 ? 0 : c < 20 ? 1 : c < 22 ? 2 : c < 24 ? 3 : c == 24 ? 4 : c - 19; }
B200Z_HD uint32_t ml_code(uint32_t ml) {
    const uint32_t b = ml - 3;
    if (b < 32) return b;
    if (b < 40) return 32 + ((b - 32) >> 1);
    if (b < 48) return 36 + ((b - 40) >> 2);
    if (b < 64) return 38 + ((b - 48) >> 3);
    if (b < 96) return 40 + ((b - 64) >> 4);
    if (b < 128) return 42;
    return flog2(b) + 36;
}
B200Z_HD uint32_t ml_bits(uint32_t c) { return c < 32 ? 0 : c < 36 ? 1 : c < 38 ? 2 : c < 40 ? 3 : c < 42 ? 4 : c == 42 ? 5 : c - 36; }
B200Z_HD uint32_t of_code(uint32_t of) { return flog2(of + 3); }

// ---- forward LSB-first bit writer; bytes past `cap` are counted but not stored (the caller compares `pos` with its budget)
struct BitW {
    uint8_t *dst;
    uint32_t cap, pos;
    uint64_t acc;
    uint32_t n;
    B200Z_HD void put(uint32_t v, uint32_t nb) {   // nb <= 32
        acc |= (uint64_t)(v & (uint32_t)((1ull << nb) - 1ull)) << n;
        n += nb;
        while (n >= 8) { if (pos < cap) dst[pos] = (uint8_t)acc; pos++; acc >>= 8; n -= 8; }
    }
    B200Z_HD void pad() { if (n) put(0, 8 - n); }
    B200Z_HD void close() { put(1, 1); pad(); }    // end marker, then zero padding to the byte
};
B200Z_HD void put_byte(uint8_t *dst, uint32_t cap, uint32_t pos, uint32_t v) { if (pos < cap) dst[pos] = (uint8_t)v; }
B200Z_HD void put_le(uint8_t *dst, uint32_t cap, uint32_t pos, uint64_t v, uint32_t nbytes) {
    for (uint32_t i = 0; i < nbytes; i++) put_byte(dst, cap, pos + i, (uint32_t)(v >> (8 * i)) & 0xffu);
}

// ---- FSE ----------------------------------------------------------------------------------------------------
// normalised counts summing to 2^log; a symbol too rare for one cell gets -1 ("less than 1" probability).
// Needs at least one symbol and no more distinct symbols than 2^log.
B200Z_HDN inline void fse_normalize(const uint32_t *cnt, uint32_t maxsym, uint32_t total, uint32_t log, int16_t *norm) {
    const int32_t size = 1 << log;
    int32_t sum = 0, best = -1;
    uint32_t largest = 0;
    for (uint32_t s = 0; s <= maxsym; s++) {
        const uint64_t c = cnt[s];
        if (!c) { norm[s] = 0; continue; }
        if ((c << log) < total) { norm[s] = -1; sum += 1; continue; }
        int32_t v = (int32_t)(((c << log) + total / 2) / total);
        if (v < 1) v = 1;
        norm[s] = (int16_t)v;
        sum += v;
        if (v > best) { best = v; largest = s; }
    }
    int32_t diff = size - sum;
    if (diff > 0) norm[largest] = (int16_t)(norm[largest] + diff);
    while (diff < 0) {   // take cells from the most probable symbol, one at a time
        uint32_t m = 0;
        for (uint32_t s = 1; s <= maxsym; s++) if (norm[s] > norm[m]) m = s;
        norm[m]--;
        diff++;
    }
}

// the table description (FSE_writeNCount layout, read by fse_read_probabilities); returns its byte length
B200Z_HDN inline uint32_t fse_write_ncount(const int16_t *norm, uint32_t maxsym, uint32_t log, uint8_t *dst, uint32_t cap) {
    BitW w{dst, cap, 0, 0, 0};
    const uint32_t alpha = maxsym + 1;
    int32_t remaining = (1 << log) + 1, threshold = 1 << log;
    uint32_t nbits = log + 1, s = 0;
    bool prev0 = false;
    w.put(log - 5, 4);
    while (s < alpha && remaining > 1) {
        if (prev0) {
            uint32_t start = s;
            while (s < alpha && !norm[s]) s++;
            while (s >= start + 24) { start += 24; w.put(0xFFFFu, 16); }
            while (s >= start + 3) { start += 3; w.put(3, 2); }
            w.put(s - start, 2);
        }
        int32_t count = norm[s++];
        const int32_t max = (2 * threshold - 1) - remaining;
        remaining -= count < 0 ? -count : count;
        count++;
        if (count >= threshold) count += max;
        w.put((uint32_t)count, nbits - (count < max ? 1u : 0u));
        prev0 = count == 1;
        while (remaining < threshold) { nbits--; threshold >>= 1; }
    }
    w.pad();
    return w.pos;
}

// encoder table (FSE_buildCTable): the spread is fse_build_table's, so states decode to the same symbols
struct FseCT {
    uint16_t state[512];
    int32_t dnb[64];   // deltaNbBits
    int32_t dfs[64];   // deltaFindState
    uint32_t log;
};
B200Z_HDN inline void fse_build_ctable(const int16_t *norm, uint32_t maxsym, uint32_t log, FseCT &ct) {
    const uint32_t size = 1u << log, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    uint8_t sym[512];
    uint32_t cumul[65];
    uint32_t high = size - 1;
    cumul[0] = 0;
    for (uint32_t s = 0; s <= maxsym; s++) {
        if (norm[s] == -1) { cumul[s + 1] = cumul[s] + 1; sym[high--] = (uint8_t)s; }
        else cumul[s + 1] = cumul[s] + (uint32_t)(norm[s] > 0 ? norm[s] : 0);
    }
    uint32_t pos = 0;
    for (uint32_t s = 0; s <= maxsym; s++)
        for (int32_t k = 0; k < norm[s]; k++) {
            sym[pos] = (uint8_t)s;
            do pos = (pos + step) & mask; while (pos > high);
        }
    for (uint32_t u = 0; u < size; u++) ct.state[cumul[sym[u]]++] = (uint16_t)(size + u);
    int32_t total = 0;
    for (uint32_t s = 0; s <= maxsym; s++) {
        const int32_t p = norm[s];
        if (p == 0) { ct.dnb[s] = (int32_t)(((log + 1) << 16) - size); ct.dfs[s] = 0; }
        else if (p == -1 || p == 1) { ct.dnb[s] = (int32_t)((log << 16) - size); ct.dfs[s] = total - 1; total++; }
        else {
            const uint32_t max_out = log - flog2((uint32_t)p - 1);
            ct.dnb[s] = (int32_t)(max_out << 16) - (p << max_out);
            ct.dfs[s] = total - p;
            total += p;
        }
    }
    ct.log = log;
}
B200Z_HD uint32_t fse_init_state(const FseCT &ct, uint32_t s) {
    const uint32_t nb = (uint32_t)(ct.dnb[s] + (1 << 15)) >> 16;
    const uint32_t value = (nb << 16) - (uint32_t)ct.dnb[s];
    return ct.state[(int32_t)(value >> nb) + ct.dfs[s]];
}
B200Z_HD void fse_encode(BitW &w, const FseCT &ct, uint32_t &st, uint32_t s) {
    const uint32_t nb = (uint32_t)((int32_t)st + ct.dnb[s]) >> 16;
    w.put(st, nb);
    st = ct.state[(int32_t)(st >> nb) + ct.dfs[s]];
}

// accuracy log for `n` coded symbols (FSE_optimalTableLog's rule), at least 5 and enough for `distinct` symbols
B200Z_HD uint32_t fse_pick_log(uint32_t n, uint32_t maxsym, uint32_t distinct, uint32_t max_log) {
    uint32_t log = n > 1 ? flog2(n - 1) : 0;
    log = log > 2 ? log - 2 : 0;
    if (log > max_log) log = max_log;
    uint32_t min_log = flog2(n) + 1, m2 = flog2(maxsym) + 2;
    if (m2 < min_log) min_log = m2;
    if (log < min_log) log = min_log;
    if (log < 5) log = 5;
    while ((1u << log) < distinct) log++;
    return log > max_log ? max_log : log;
}

// ---- Huffman ------------------------------------------------------------------------------------------------
// code lengths of an optimal prefix code, limited to ENC_HUF_MAX_BITS and completed (Kraft sum exactly 1, which the
// implicit last weight requires).  Needs >= 2 symbols.  Returns the longest length.
B200Z_HDN inline uint32_t huf_lengths(const uint32_t *cnt, uint8_t *len) {
    uint32_t w[511];
    uint16_t sym[256], parent[511];
    uint8_t depth[511];
    uint32_t n = 0;
    for (uint32_t s = 0; s < 256; s++) {
        len[s] = 0;
        if (!cnt[s]) continue;
        uint32_t i = n++;   // insertion sort by (count, symbol)
        while (i > 0 && w[i - 1] > cnt[s]) { w[i] = w[i - 1]; sym[i] = sym[i - 1]; i--; }
        w[i] = cnt[s]; sym[i] = (uint16_t)s;
    }
    uint32_t a = 0, b = n;   // two queues: leaves [a, n), internal nodes [b, k)
    for (uint32_t k = n; k < 2 * n - 1; k++) {
        uint32_t pick[2];
        for (int t = 0; t < 2; t++) pick[t] = (a < n && (b >= k || w[a] <= w[b])) ? a++ : b++;
        w[k] = w[pick[0]] + w[pick[1]];
        parent[pick[0]] = parent[pick[1]] = (uint16_t)k;
    }
    depth[2 * n - 2] = 0;
    for (int32_t k = (int32_t)(2 * n) - 3; k >= 0; k--) depth[k] = depth[parent[k]] + 1;
    int32_t kraft = 0;   // in units of 2^-ENC_HUF_MAX_BITS
    for (uint32_t i = 0; i < n; i++) {
        uint32_t l = depth[i] > ENC_HUF_MAX_BITS ? ENC_HUF_MAX_BITS : depth[i];
        len[sym[i]] = (uint8_t)l;
        kraft += 1 << (ENC_HUF_MAX_BITS - l);
    }
    const int32_t one = 1 << ENC_HUF_MAX_BITS;
    while (kraft > one) {   // lengthen the longest code that can still grow (rarest first)
        uint32_t m = 256;
        for (uint32_t i = 0; i < n; i++) {
            const uint32_t s = sym[i];
            if (len[s] < ENC_HUF_MAX_BITS && (m == 256 || len[s] > len[m])) m = s;
        }
        len[m]++;
        kraft -= 1 << (ENC_HUF_MAX_BITS - len[m]);
    }
    while (kraft < one) {   // shorten the longest code (most frequent first); its gain always fits
        uint32_t m = 256;
        for (int32_t i = (int32_t)n - 1; i >= 0; i--) {
            const uint32_t s = sym[i];
            if (m == 256 || len[s] > len[m]) m = s;
        }
        kraft += 1 << (ENC_HUF_MAX_BITS - len[m]);
        len[m]--;
    }
    uint32_t maxb = 0;
    for (uint32_t s = 0; s < 256; s++) if (len[s] > maxb) maxb = len[s];
    return maxb;
}

// canonical codes in the decoder's order (huf_build_table: longest codes first, symbols ascending)
B200Z_HDN inline void huf_codes(const uint8_t *len, uint32_t maxb, uint16_t *code) {
    uint32_t rank_count[ENC_HUF_MAX_BITS + 2] = {0}, next[ENC_HUF_MAX_BITS + 2];
    for (uint32_t s = 0; s < 256; s++) rank_count[len[s]]++;
    next[maxb] = 0;
    for (uint32_t b = maxb; b >= 1; b--) next[b - 1] = next[b] + rank_count[b] * (1u << (maxb - b));
    for (uint32_t s = 0; s < 256; s++) {
        const uint32_t b = len[s];
        code[s] = 0;
        if (!b) continue;
        code[s] = (uint16_t)(next[b] >> (maxb - b));
        next[b] += 1u << (maxb - b);
    }
}

// Huffman tree description; 0 when it cannot be written (FSE-compressed weights needing >= 128 bytes, or one weight value only)
B200Z_HDN inline uint32_t huf_write_weights(const uint8_t *len, uint32_t maxb, uint8_t *dst, uint32_t cap) {
    uint32_t last = 0;
    for (uint32_t s = 0; s < 256; s++) if (len[s]) last = s;
    const uint32_t nw = last;   // the last symbol's weight is implicit
    uint8_t wt[256];
    for (uint32_t s = 0; s < nw; s++) wt[s] = (uint8_t)(len[s] ? maxb + 1 - len[s] : 0);
    if (nw <= 128) {
        put_byte(dst, cap, 0, 127 + nw);
        for (uint32_t i = 0; i < nw; i += 2) put_byte(dst, cap, 1 + i / 2, (uint32_t)(wt[i] << 4) | (i + 1 < nw ? wt[i + 1] : 0u));
        return 1 + (nw + 1) / 2;
    }
    uint32_t cnt[16] = {0}, maxw = 0, distinct = 0;
    for (uint32_t i = 0; i < nw; i++) { if (!cnt[wt[i]]++) distinct++; if (wt[i] > maxw) maxw = wt[i]; }
    if (distinct < 2) return 0;   // every state would read 0 bits and the decoder could not find the end
    int16_t norm[16];
    fse_normalize(cnt, maxw, nw, 6, norm);
    FseCT ct;
    fse_build_ctable(norm, maxw, 6, ct);
    const uint32_t hdr = fse_write_ncount(norm, maxw, 6, dst + 1, cap > 1 ? cap - 1 : 0);
    BitW w{dst + 1 + hdr, cap > 1 + hdr ? cap - 1 - hdr : 0, 0, 0, 0};
    uint32_t i = nw, s1, s2;   // two interleaved states: even weights on state 1, odd ones on state 2
    if (nw & 1) { s1 = fse_init_state(ct, wt[--i]); s2 = fse_init_state(ct, wt[--i]); fse_encode(w, ct, s1, wt[--i]); }
    else { s2 = fse_init_state(ct, wt[--i]); s1 = fse_init_state(ct, wt[--i]); }
    while (i > 0) { fse_encode(w, ct, s2, wt[--i]); fse_encode(w, ct, s1, wt[--i]); }
    w.put(s2, 6);
    w.put(s1, 6);
    w.close();
    const uint32_t size = hdr + w.pos;
    if (size >= 128) return 0;
    put_byte(dst, cap, 0, size);
    return 1 + size;
}

// ---- a formatted dictionary's tables, as the encoder uses them -------------------------------------------------------
struct EncDict {
    uint16_t huf_code[256];
    uint8_t huf_len[256];      // 0: the byte has no code in the dictionary's table
    FseCT ct[3];               // by ENC_LL / ENC_OF / ENC_ML
    int16_t norm[3][64];       // normalized counts, 0 past the table's last symbol
};
// From the dictionary's Huffman weights (nweights explicit ones; the last symbol's weight is implied) and its three FSE tables'
// normalized counts (nprobs[t] of them at accuracy log logs[t]), as Dictionary::decode_dict parsed them, so both are valid.
B200Z_HDN inline void enc_dict_build(const uint8_t *weights, uint32_t nweights, const int16_t *const probs[3], const uint32_t nprobs[3],
                                     const uint32_t logs[3], EncDict &d) {
    uint32_t sum = 0;
    for (uint32_t i = 0; i < nweights; i++) sum += weights[i] ? 1u << (weights[i] - 1) : 0u;
    const uint32_t maxb = hbs(sum), last = hbs((1u << maxb) - sum);
    for (uint32_t i = 0; i < 256; i++) {
        const uint32_t w = i < nweights ? weights[i] : i == nweights ? last : 0u;
        d.huf_len[i] = (uint8_t)(w ? maxb + 1 - w : 0);
    }
    huf_codes(d.huf_len, maxb, d.huf_code);
    for (uint32_t t = 0; t < 3; t++) {
        for (uint32_t c = 0; c < 64; c++) d.norm[t][c] = c < nprobs[t] ? probs[t][c] : 0;
        fse_build_ctable(d.norm[t], nprobs[t] - 1, logs[t], d.ct[t]);
    }
}

// log2(p) in 8-bit fixed point, p >= 1, in integers only (so the host and the GPU agree): the integer part from the highest set
// bit, the fraction bit by bit by squaring the mantissa
B200Z_HD uint32_t log2_q8(uint32_t p) {
    const uint32_t hb = flog2(p);
    uint64_t x = ((uint64_t)p << 16) >> hb;   // mantissa in [1, 2), 16 fraction bits
    uint32_t r = hb << 8;
    for (int i = 7; i >= 0; i--) {
        x = (x * x) >> 16;
        if (x >= (2u << 16)) { x >>= 1; r |= 1u << i; }
    }
    return r;
}
// estimated bits (8-bit fixed point) of coding cnt[0..maxsym] with normalized counts norm at accuracy log `log`: log - log2(p) per
// symbol (a "less than 1" count costs as 1)
B200Z_HD uint64_t fse_cost_q8(const uint32_t *cnt, uint32_t maxsym, const int16_t *norm, uint32_t log) {
    uint64_t c = 0;
    for (uint32_t s = 0; s <= maxsym; s++)
        if (cnt[s]) c += (uint64_t)cnt[s] * ((log << 8) - log2_q8(norm[s] > 0 ? (uint32_t)norm[s] : 1u));
    return c;
}

// ---- block ----------------------------------------------------------------------------------------------------
struct EncScratch {   // per warp (shared memory on the GPU)
    uint32_t lit_cnt[256];
    uint32_t cnt[3][64];          // LL / OF / ML code histograms
    uint16_t huf_code[256];
    uint8_t huf_len[256];
    FseCT ct[3];
    int16_t norm[3][64];
    uint32_t mode[3], maxsym[3];
    uint32_t stream_bits[4], stream_off[4];
    uint32_t use_huf, lit_end, total;
    uint32_t use_dict, dict_bits[4];   // Treeless literals with the dictionary's codes
};

B200Z_HD uint32_t raw_literals_header_size(uint32_t n) { return n < 32 ? 1 : n < 4096 ? 2 : 3; }
B200Z_HD uint32_t raw_literals_header(uint8_t *dst, uint32_t cap, uint32_t n) {
    if (n < 32) { put_byte(dst, cap, 0, n << 3); return 1; }
    if (n < 4096) { put_le(dst, cap, 0, (1u << 2) | (n << 4), 2); return 2; }
    put_le(dst, cap, 0, (3u << 2) | (n << 4), 3);
    return 3;
}

// Encodes one block's literals and sequences as the content of a Compressed block into dst[0, cap) and returns its size
// (which may exceed cap: then only the first cap bytes were stored).  Every lane of the group calls it; nlanes = 32 on the
// GPU, 1 on the host.  The trailing literals after the last sequence are the literals not consumed by any sequence.
// dt: a formatted dictionary's tables when the block is a frame's first block, else nullptr (then the output is exactly what it
// is without this argument).  With them:
//   literals   Treeless (the dictionary's codes; 1 stream below 1024 literals, else 4) when every literal byte has a code and it
//              is strictly smaller than what the rule above chooses (own Huffman or Raw)
//   sequences  per table, Repeat when the block has more than one code, every code has a nonzero count in the dictionary's
//              table, and its estimated cost is at most the table's own description plus its own estimated cost (fse_cost_q8)
B200Z_HDN inline uint32_t encode_block(EncScratch &s, const uint8_t *lits, uint32_t nlit, const SeqRec *seqs, uint32_t nseq,
                                      uint8_t *dst, uint32_t cap, uint32_t lane, uint32_t nlanes, const EncDict *dt = nullptr) {
    for (uint32_t i = lane; i < 256; i += nlanes) s.lit_cnt[i] = 0;
    for (uint32_t i = lane; i < 3 * 64; i += nlanes) s.cnt[i / 64][i % 64] = 0;
    for (uint32_t i = lane; i < 4; i += nlanes) { s.stream_bits[i] = 0; if (dt) s.dict_bits[i] = 0; }
    B200Z_ENC_SYNC();
    for (uint32_t i = lane; i < nlit; i += nlanes) B200Z_ENC_ADD(&s.lit_cnt[lits[i]], 1u);
    for (uint32_t i = lane; i < nseq; i += nlanes) {
        const SeqRec q = seqs[i];
        B200Z_ENC_ADD(&s.cnt[ENC_LL][ll_code(q.ll)], 1u);
        B200Z_ENC_ADD(&s.cnt[ENC_OF][of_code(q.of)], 1u);
        B200Z_ENC_ADD(&s.cnt[ENC_ML][ml_code(q.ml)], 1u);
    }
    B200Z_ENC_SYNC();
    // -- Huffman table (one lane); the description goes right after the widest literals header (5 bytes) and moves
    // back by one byte when the 4-byte header suffices
    const uint32_t seg = (nlit + 3) / 4;
    if (lane == 0) {
        s.use_huf = 0;
        uint32_t distinct = 0;
        for (uint32_t i = 0; i < 256; i++) distinct += s.lit_cnt[i] != 0;
        if (nlit > ENC_RAW_LITERALS_MAX && distinct >= 2) {
            const uint32_t maxb = huf_lengths(s.lit_cnt, s.huf_len);
            huf_codes(s.huf_len, maxb, s.huf_code);
            const uint32_t tree = huf_write_weights(s.huf_len, maxb, dst + 5, cap > 5 ? cap - 5 : 0);
            if (tree) { s.use_huf = 1; s.lit_end = tree; }
        }
        if (dt) {
            s.use_dict = nlit >= 2;
            for (uint32_t i = 0; i < 256; i++) if (s.lit_cnt[i] && !dt->huf_len[i]) s.use_dict = 0;
        }
    }
    B200Z_ENC_SYNC();
    const uint32_t dstreams = nlit < 1024 ? 1 : 4;   // streams of Treeless literals
    const bool try_dict = dt && s.use_dict;           // (dt is a constant nullptr in the plain path: all of this folds away)
    if (s.use_huf || try_dict) {
        uint32_t b[4] = {0, 0, 0, 0}, db[4] = {0, 0, 0, 0};
        if (s.use_huf) for (uint32_t i = lane; i < nlit; i += nlanes) b[i / seg] += s.huf_len[lits[i]];
        if (try_dict) for (uint32_t i = lane; i < nlit; i += nlanes) db[dstreams == 1 ? 0 : i / seg] += dt->huf_len[lits[i]];
        for (uint32_t k = 0; k < 4; k++) if (b[k]) B200Z_ENC_ADD(&s.stream_bits[k], b[k]);
        for (uint32_t k = 0; k < 4; k++) if (db[k]) B200Z_ENC_ADD(&s.dict_bits[k], db[k]);
        B200Z_ENC_SYNC();
        if (lane == 0) {
            const uint32_t tree = s.lit_end;
            uint32_t csize = tree + 6;
            for (uint32_t k = 0; k < 4; k++) csize += (s.stream_bits[k] + 8) / 8;   // + the end marker bit
            const uint32_t hsize = (nlit < 16384 && csize < 16384) ? 4 : 5;
            if (s.use_huf && hsize + csize >= nlit + 3) s.use_huf = 0;   // Huffman does not pay (compressed.rs:367-371)
            if (try_dict) {   // Treeless only when strictly smaller than the choice above
                uint32_t dsize = dstreams == 1 ? 0 : 6;
                for (uint32_t k = 0; k < dstreams; k++) dsize += (s.dict_bits[k] + 8) / 8;
                const uint32_t dh = dstreams == 1 ? 3 : (nlit < 16384 && dsize < 16384) ? 4 : 5;
                const uint32_t today = s.use_huf ? hsize + csize : raw_literals_header_size(nlit) + nlit;
                if ((dstreams == 1 && dsize >= 1024) || dh + dsize >= today) s.use_dict = 0;
                else {
                    s.use_huf = 0;
                    if (dh == 3) put_le(dst, cap, 0, 3u | (nlit << 4) | (dsize << 14), 3);
                    else if (dh == 4) put_le(dst, cap, 0, 3u | (2u << 2) | (nlit << 4) | ((uint64_t)dsize << 18), 4);
                    else put_le(dst, cap, 0, 3u | (3u << 2) | ((uint64_t)nlit << 4) | ((uint64_t)dsize << 22), 5);
                    uint32_t off = dh + (dstreams == 1 ? 0 : 6);
                    for (uint32_t k = 0; k < dstreams; k++) {
                        const uint32_t sz = (s.dict_bits[k] + 8) / 8;
                        if (dstreams == 4 && k < 3) put_le(dst, cap, dh + 2 * k, sz, 2);
                        s.stream_off[k] = off;
                        off += sz;
                    }
                    s.lit_end = off;
                }
            }
            if (s.use_huf) {
                if (hsize == 4) for (uint32_t i = 0; i < tree; i++) put_byte(dst, cap, 4 + i, 5 + i < cap ? dst[5 + i] : 0u);
                if (hsize == 4) put_le(dst, cap, 0, 2u | (2u << 2) | (nlit << 4) | ((uint64_t)csize << 18), 4);
                else put_le(dst, cap, 0, 2u | (3u << 2) | ((uint64_t)nlit << 4) | ((uint64_t)csize << 22), 5);
                uint32_t off = hsize + tree + 6;
                for (uint32_t k = 0; k < 4; k++) {
                    const uint32_t sz = (s.stream_bits[k] + 8) / 8;
                    if (k < 3) put_le(dst, cap, hsize + tree + 2 * k, sz, 2);
                    s.stream_off[k] = off;
                    off += sz;
                }
                s.lit_end = off;
            }
        }
        B200Z_ENC_SYNC();
    }
    const bool dict_lits = dt && s.use_dict;
    if (s.use_huf || dict_lits) {
        const uint16_t *code = dict_lits ? dt->huf_code : s.huf_code;
        const uint8_t *len = dict_lits ? dt->huf_len : s.huf_len;
        const uint32_t ns = dict_lits ? dstreams : 4;
        for (uint32_t k = lane; k < ns; k += nlanes) {   // each stream is written backwards: the decoder reads it from the end
            const uint32_t lo = ns == 1 ? 0 : k * seg, hi = k == ns - 1 ? nlit : lo + seg, off = s.stream_off[k];
            BitW w{dst + off, cap > off ? cap - off : 0, 0, 0, 0};
            for (uint32_t i = hi; i > lo; i--) w.put(code[lits[i - 1]], len[lits[i - 1]]);
            w.close();
        }
    } else {
        const uint32_t h = raw_literals_header(dst, cap, nlit);
        for (uint32_t i = lane; i < nlit; i += nlanes) put_byte(dst, cap, h + i, lits[i]);
        if (lane == 0) s.lit_end = h + nlit;
    }
    B200Z_ENC_SYNC();
    // -- sequences section (one lane: the bitstream is one serial chain of three FSE states)
    if (lane == 0) {
        uint32_t p = s.lit_end;
        if (nseq < 128) put_byte(dst, cap, p++, nseq);
        else if (nseq < 0x7F00) { put_byte(dst, cap, p++, (nseq >> 8) + 128); put_byte(dst, cap, p++, nseq & 0xffu); }
        else { put_byte(dst, cap, p++, 255); put_le(dst, cap, p, nseq - 0x7F00, 2); p += 2; }
        if (nseq) {
            const uint32_t pmodes = p++;
            uint32_t modes = 0;
            const FseCT *ct[3] = {&s.ct[0], &s.ct[1], &s.ct[2]};
            for (uint32_t t = 0; t < 3; t++) {
                uint32_t distinct = 0, maxsym = 0;
                for (uint32_t c = 0; c <= enc_max_sym(t); c++) if (s.cnt[t][c]) { distinct++; maxsym = c; }
                s.maxsym[t] = maxsym;
                if (distinct == 1) { s.mode[t] = 1; put_byte(dst, cap, p++, maxsym); }
                else {
                    s.mode[t] = 2;
                    const uint32_t log = fse_pick_log(nseq, maxsym, distinct, enc_max_log(t));
                    fse_normalize(s.cnt[t], maxsym, nseq, log, s.norm[t]);
                    fse_build_ctable(s.norm[t], maxsym, log, s.ct[t]);
                    const uint32_t desc = fse_write_ncount(s.norm[t], maxsym, log, dst + p, cap > p ? cap - p : 0);
                    bool rep = dt != nullptr;
                    for (uint32_t c = 0; rep && c <= maxsym; c++) if (s.cnt[t][c] && !dt->norm[t][c]) rep = false;
                    if (rep && fse_cost_q8(s.cnt[t], maxsym, dt->norm[t], dt->ct[t].log) <=
                                   ((uint64_t)desc << 11) + fse_cost_q8(s.cnt[t], maxsym, s.norm[t], log)) {
                        s.mode[t] = 3;   // Repeat: the dictionary's table, no description
                        ct[t] = &dt->ct[t];
                    } else {
                        p += desc;
                    }
                }
            }
            modes = (s.mode[ENC_LL] << 6) | (s.mode[ENC_OF] << 4) | (s.mode[ENC_ML] << 2);
            put_byte(dst, cap, pmodes, modes);
            BitW w{dst + p, cap > p ? cap - p : 0, 0, 0, 0};
            // the decoder reads LL, OF, ML states first and updates LL, ML, OF: the writer goes the other way round
            const uint32_t kEncOrder[3] = {ENC_OF, ENC_ML, ENC_LL}, kFlushOrder[3] = {ENC_ML, ENC_OF, ENC_LL};
            uint32_t st[3] = {0, 0, 0};
            const SeqRec q = seqs[nseq - 1];
            const uint32_t c0[3] = {ll_code(q.ll), of_code(q.of), ml_code(q.ml)};
            for (uint32_t t = 0; t < 3; t++) if (s.mode[t] >= 2) st[t] = fse_init_state(*ct[t], c0[t]);   // no bits: order is free
            w.put(q.ll, ll_bits(c0[ENC_LL]));
            w.put(q.ml - 3, ml_bits(c0[ENC_ML]));
            w.put(q.of + 3, c0[ENC_OF]);
            for (uint32_t n = nseq - 1; n-- > 0;) {
                const SeqRec r = seqs[n];
                const uint32_t c[3] = {ll_code(r.ll), of_code(r.of), ml_code(r.ml)};
                for (uint32_t t : kEncOrder) if (s.mode[t] >= 2) fse_encode(w, *ct[t], st[t], c[t]);
                w.put(r.ll, ll_bits(c[ENC_LL]));
                w.put(r.ml - 3, ml_bits(c[ENC_ML]));
                w.put(r.of + 3, c[ENC_OF]);
            }
            for (uint32_t t : kFlushOrder) if (s.mode[t] >= 2) w.put(st[t], ct[t]->log);
            w.close();
            p += w.pos;
        }
        s.total = p;
    }
    B200Z_ENC_SYNC();
    return s.total;
}

// frame header for a frame of `n` bytes: Single_Segment = 0, a 2^wlog window (128 KiB unless long matches are on), the dictionary ID in the smallest field that holds
// it (none for ID 0, as ruzstd's minify_val sizes it, encoding/frame_header.rs), Frame_Content_Size in the smallest legal field
B200Z_HD uint32_t dict_id_field_size(uint32_t dict_id) { return dict_id == 0 ? 0 : dict_id <= 0xffu ? 1 : dict_id <= 0xffffu ? 2 : 4; }
B200Z_HD uint32_t frame_header_size(uint64_t n, uint32_t dict_id) {
    return 6 + dict_id_field_size(dict_id) + ((n >= 256 && n <= 65791) ? 2 : (n >> 32) ? 8 : 4);
}
// the Window_Descriptor's exponent of a frame of n bytes compressed at window_log (0 counts as 17): min(window_log,
// max(17, ceil(log2 n))), so a frame never advertises more window than its content can use
B200Z_HD uint32_t frame_window_log(uint64_t n, uint32_t window_log) {
    if (window_log <= 17) return 17;
    uint32_t c = 17;
    while (c < window_log && (1ull << c) < n) c++;
    return c;
}
B200Z_HD uint32_t write_frame_header(uint8_t *dst, uint64_t n, bool checksum, uint32_t dict_id, uint32_t wlog = 17) {
    const uint32_t did = dict_id_field_size(dict_id), fcs = frame_header_size(n, dict_id) - 6 - did;
    const uint32_t flag = fcs == 2 ? 1 : fcs == 4 ? 2 : 3;
    put_le(dst, 4, 0, 0xFD2FB528u, 4);
    dst[4] = (uint8_t)((flag << 6) | (checksum ? 4u : 0u) | (did == 4 ? 3u : did));
    dst[5] = (uint8_t)((wlog - 10) << 3);
    for (uint32_t i = 0; i < did; i++) dst[6 + i] = (uint8_t)(dict_id >> (8 * i));
    const uint64_t v = fcs == 2 ? n - 256 : n;
    for (uint32_t i = 0; i < fcs; i++) dst[6 + did + i] = (uint8_t)(v >> (8 * i));
    return 6 + did + fcs;
}

}  // namespace b200z
