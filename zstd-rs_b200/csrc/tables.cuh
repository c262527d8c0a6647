// tables.cuh -- entropy-table parsing and LUT expansion, compiled for BOTH device and host.
//
// These run on the GPU for every block of a submission (kernel k_setup) so that the host only walks headers;
// the same code runs on the host once per dictionary (Dictionary::decode_dict needs the byte length of each
// table description to find the content).  What they must produce is defined by the reference:
//   FSETable::read_probabilities        ruzstd/src/fse/fse_decoder.rs:224-307
//   FSETable::build_decoding_table      ruzstd/src/fse/fse_decoder.rs:141-220 (+ :334-366)
//   HuffmanTable::read_weights          ruzstd/src/huff0/huff0_decoder.rs:132-278
//   HuffmanTable::build_table_from_weights  ruzstd/src/huff0/huff0_decoder.rs:284-377
// The algorithms are restated for a GPU thread (fixed-size local arrays, packed u16/u32 LUT entries, no heap);
// the results (LUT contents, byte counts, error kinds and their order) are the reference's.
#pragma once
#include <stdint.h>

#include "../../include/b200zstd.h"
#include "b200z_types.h"

namespace b200z {

B200Z_HD uint32_t hbs(uint32_t x) {  // "highest_bit_set": 32 - clz, x > 0  (fse_decoder.rs:326-329)
#ifdef __CUDA_ARCH__
    return 32u - (uint32_t)__clz((int)x);
#else
    return 32u - (uint32_t)__builtin_clz(x);
#endif
}

// ---- forward, LSB-first bit reader over a byte slice (bit_io/bit_reader.rs:28-91); only used on table
// descriptions (tens of bytes), so it assembles byte-wise.
struct FwdBits {
    const uint8_t *src;
    uint32_t len;
    uint32_t idx;  // bits read
    B200Z_HD bool get(uint32_t n, uint32_t &out) {  // n <= 24
        if (len * 8u - idx < n) return false;
        out = 0;
        if (n) {   // the n bits starting at bit idx, LSB first: at most 4 bytes, all inside the slice
            const uint32_t b0 = idx >> 3, sh = idx & 7u, nbytes = (sh + n + 7u) >> 3;
            uint32_t w = src[b0];
            if (nbytes > 1) w |= (uint32_t)src[b0 + 1] << 8;
            if (nbytes > 2) w |= (uint32_t)src[b0 + 2] << 16;
            if (nbytes > 3) w |= (uint32_t)src[b0 + 3] << 24;
            out = (w >> sh) & ((1u << n) - 1u);
        }
        idx += n;
        return true;
    }
};

// ---- reversed reader over a tiny slice (Huffman weight stream, <= 127 bytes): position based, zero-extended
// below bit 0, signed remaining -- the observable behaviour of BitReaderReversed (bit_reader_reverse.rs:27-113).
struct RevBitsSmall {
    const uint8_t *src;
    int32_t p;  // bits remaining (may go negative)
    B200Z_HD uint32_t get(uint32_t n) {  // n <= 16: bits [p - n, p) of the slice read as one little-endian number, bit p - 1 first
        uint32_t v = 0;
        if (n && p > 0) {
            const int32_t lo = p - (int32_t)n;
            if (lo >= 0) {
                const uint32_t b0 = (uint32_t)lo >> 3, sh = (uint32_t)lo & 7u, nbytes = (sh + n + 7u) >> 3;   // <= 3 bytes
                uint32_t w = src[b0];
                if (nbytes > 1) w |= (uint32_t)src[b0 + 1] << 8;
                if (nbytes > 2) w |= (uint32_t)src[b0 + 2] << 16;
                v = (w >> sh) & ((1u << n) - 1u);
            } else {   // only p (< n) real bits are left; zeros below bit 0
                const uint32_t m = (uint32_t)p;
                uint32_t w = src[0];
                if (m > 8) w |= (uint32_t)src[1] << 8;
                v = (w & ((1u << m) - 1u)) << (n - m);
            }
        }
        p -= (int32_t)n;
        return v;
    }
};

// ---- FSE --------------------------------------------------------------------------------------------------
// read_probabilities: probs[] gets the first min(nprobs, 256) entries; nprobs is the reference's
// symbol_probabilities.len() (it can exceed 256 through zero-run flags before TooManySymbols is raised).
B200Z_HDN inline int fse_read_probabilities(const uint8_t *src, uint32_t len, uint32_t max_log, uint32_t max_symbol,
                                            int16_t *probs, uint32_t &nprobs, uint32_t &acc_log, uint32_t &bytes_read) {
    FwdBits br{src, len, 0};
    uint32_t v;
    nprobs = 0;
    if (!br.get(4, v)) return B200Z_ERR_FSE_GET_BITS;
    acc_log = 5 + v;
    if (acc_log > max_log) return B200Z_ERR_FSE_ACC_LOG_TOO_BIG;
    uint32_t sum = 1u << acc_log, counter = 0;
    while (counter < sum) {
        uint32_t max_remaining = sum - counter + 1;
        uint32_t bits = hbs(max_remaining);
        if (!br.get(bits, v)) return B200Z_ERR_FSE_GET_BITS;
        uint32_t low_threshold = ((1u << bits) - 1u) - max_remaining;
        uint32_t mask = (1u << (bits - 1)) - 1u;
        uint32_t small = v & mask, value;
        if (small < low_threshold) { br.idx -= 1; value = small; }
        else if (v > mask) value = v - low_threshold;
        else value = v;
        int32_t prob = (int32_t)value - 1;
        if (nprobs < 256) probs[nprobs] = (int16_t)prob;
        nprobs++;
        if (prob != 0) counter += prob > 0 ? (uint32_t)prob : 1u;
        else {
            for (;;) {
                if (!br.get(2, v)) return B200Z_ERR_FSE_GET_BITS;
                for (uint32_t k = 0; k < v; k++) { if (nprobs < 256) probs[nprobs] = 0; nprobs++; }
                if (v != 3) break;
            }
        }
    }
    if (counter != sum) return B200Z_ERR_FSE_PROBABILITY_COUNTER_MISMATCH;
    if (nprobs > max_symbol + 1) return B200Z_ERR_FSE_TOO_MANY_SYMBOLS;
    bytes_read = (br.idx + 7u) >> 3;
    return 0;
}

// build_decoding_table into packed entries.  `out` may be global memory; it is used as its own scratch
// (pass 1 stores the symbol, pass 2 rewrites each entry with base_line/num_bits).
// `counter` = scratch for 256 u16 (callers on the GPU pass shared memory: per-thread local arrays of this size spill to L2)
B200Z_HDN inline int fse_build_table(const int16_t *probs, uint32_t nprobs, uint32_t acc_log, uint32_t max_symbol, uint32_t *out, uint16_t *counter) {
    if (nprobs > max_symbol + 1) return B200Z_ERR_FSE_TOO_MANY_SYMBOLS;
    const uint32_t size = 1u << acc_log;
    uint32_t negative_idx = size;
    for (uint32_t s = 0; s < nprobs; s++)
        if (probs[s] == -1) {
            if (negative_idx == 0) return B200Z_ERR_REFERENCE_WOULD_PANIC;
            negative_idx--;
            out[negative_idx] = fse_pack(0, acc_log, s);
        }
    const uint32_t step = (size >> 1) + (size >> 3) + 3, msk = size - 1;
    uint32_t pos = 0;
    for (uint32_t s = 0; s < nprobs; s++) {
        int32_t pr = probs[s];
        for (int32_t k = 0; k < pr; k++) {
            out[pos] = s;
            pos = (pos + step) & msk;
            uint32_t guard = 0;
            while (pos >= negative_idx) {
                pos = (pos + step) & msk;
                if (++guard > size) return B200Z_ERR_REFERENCE_WOULD_PANIC;  // the reference would spin forever
            }
        }
    }
    for (uint32_t s = 0; s < nprobs && s < 256; s++) counter[s] = 0;
    for (uint32_t i = 0; i < negative_idx; i++) {
        uint32_t sym = out[i] & 0xffu;  // unwritten entries read as whatever pass 1 left: all get written when sum == size
        if (sym >= nprobs) sym = 0;
        uint32_t prob = (uint32_t)(int32_t)probs[sym], cnt = counter[sym]++;
        // calc_baseline_and_numbits (fse_decoder.rs:340-366)
        uint32_t bl = 0, nb = 0;
        if (prob != 0) {
            uint32_t h = hbs(prob);
            uint32_t slices = ((1u << (h - 1)) == prob) ? prob : (1u << h);
            uint32_t n_double = slices - prob, n_single = prob - n_double;
            uint32_t width = size / slices;
            uint32_t b = hbs(width) - 1;
            if (cnt < n_double) { bl = n_single * width + cnt * width * 2; nb = b + 1; }
            else { bl = (cnt - n_double) * width; nb = b; }
        }
        out[i] = fse_pack(bl, nb, sym);
    }
    return 0;
}

// {base_line | num_bits << 16 | symbol << 24} -> the 16-bit resident form (b200z_types.h)
B200Z_HDN inline void fse_compact(const uint32_t *wide, uint32_t log, FseTab *tab) {
    for (uint32_t i = 0; i < (1u << log); i++) tab->e[i] = fse_pack16(log, wide[i] & 0xffffu, (wide[i] >> 16) & 0xffu, wide[i] >> 24);
    tab->log = log; tab->valid = 1; tab->is_rle = 0;
}

// FSETable::build_decoder (fse_decoder.rs:116-123) into an FseTab
B200Z_HDN inline int fse_build_decoder(const uint8_t *src, uint32_t len, uint32_t max_log, uint32_t max_symbol, FseTab *tab, uint32_t &bytes_read) {
    int16_t probs[256];
    uint32_t nprobs, acc_log;
    int e = fse_read_probabilities(src, len, max_log, max_symbol, probs, nprobs, acc_log, bytes_read);
    if (e) return e;
    uint32_t wide[FSE_MAX_ENTRIES];
    uint16_t counter[256];
    e = fse_build_table(probs, nprobs, acc_log, max_symbol, wide, counter);
    if (e) return e;
    fse_compact(wide, acc_log, tab);
    return 0;
}

// predefined distributions (sequence_section_decoder.rs:413-442)
B200Z_HDN inline int fse_build_predefined(uint32_t kind /*0 ll,1 of,2 ml*/, FseTab *tab) {
    const int8_t LL[36] = {4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1};
    const int8_t ML[53] = {1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1};
    const int8_t OF[29] = {1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1};
    int16_t probs[64];
    uint32_t n, log, maxsym;
    if (kind == 0) { n = 36; log = 6; maxsym = 35; for (uint32_t i = 0; i < n; i++) probs[i] = LL[i]; }
    else if (kind == 1) { n = 29; log = 5; maxsym = 31; for (uint32_t i = 0; i < n; i++) probs[i] = OF[i]; }
    else { n = 53; log = 6; maxsym = 52; for (uint32_t i = 0; i < n; i++) probs[i] = ML[i]; }
    uint32_t wide[64];
    uint16_t counter[64];
    int e = fse_build_table(probs, n, log, maxsym, wide, counter);
    if (e) return e;
    fse_compact(wide, log, tab);
    return 0;
}

// ---- Huffman ----------------------------------------------------------------------------------------------
// read_weights: weights[] (capacity 260), nweights, bytes_read.
// probs[256], tab[64], counter[256]: scratch (shared memory on the GPU)
B200Z_HDN inline int huf_read_weights_scratch(const uint8_t *src, uint32_t len, uint8_t *weights, uint32_t &nweights, uint32_t &bytes_read,
                                              int16_t *probs, uint32_t *tab, uint16_t *counter) {
    if (len == 0) return B200Z_ERR_HUF_SOURCE_IS_EMPTY;
    const uint32_t header = src[0];
    uint32_t bits_read = 8;
    if (header < 128) {
        const uint8_t *fs = src + 1;
        const uint32_t fs_len = len - 1;
        if (header > fs_len) return B200Z_ERR_HUF_NOT_ENOUGH_BYTES_FOR_WEIGHTS;
        uint32_t nprobs, acc_log, used;
        int e = fse_read_probabilities(fs, fs_len, 6, 255, probs, nprobs, acc_log, used);
        if (e) return e;
        e = fse_build_table(probs, nprobs, acc_log, 255, tab, counter);
        if (e) return e;
        if (used > header) return B200Z_ERR_HUF_FSE_TABLE_USED_TOO_MANY_BYTES;
        const uint32_t clen = header - used;
        if (fs_len - used < clen) return B200Z_ERR_HUF_NOT_ENOUGH_BYTES_TO_DECOMPRESS_WEIGHTS;
        bits_read += (used + clen) * 8;
        const uint8_t *cs = fs + used;
        // skip padding: up to 8 zero bits then the 1 marker (huff0_decoder.rs:188-200)
        if (clen == 0 || cs[clen - 1] == 0) return B200Z_ERR_HUF_EXTRA_PADDING;
        RevBitsSmall br{cs, (int32_t)((clen - 1) * 8 + hbs(cs[clen - 1]) - 1)};
        uint32_t s1 = tab[br.get(acc_log)];
        uint32_t s2 = tab[br.get(acc_log)];
        nweights = 0;
        for (;;) {  // :208-234
            weights[nweights++] = (uint8_t)(s1 >> 24);
            s1 = tab[(s1 & 0xffffu) + br.get((s1 >> 16) & 0xffu)];
            if (br.p <= -1) { weights[nweights++] = (uint8_t)(s2 >> 24); break; }
            weights[nweights++] = (uint8_t)(s2 >> 24);
            s2 = tab[(s2 & 0xffffu) + br.get((s2 >> 16) & 0xffu)];
            if (br.p <= -1) { weights[nweights++] = (uint8_t)(s1 >> 24); break; }
            if (nweights > 255) return B200Z_ERR_HUF_TOO_MANY_WEIGHTS;
        }
    } else {
        const uint32_t n = header - 127;
        const uint32_t need = (n + 1) >> 1;
        nweights = n;
        if (len - 1 < need) return B200Z_ERR_HUF_NOT_ENOUGH_BYTES_IN_SOURCE;
        for (uint32_t i = 0; i < n; i++) {
            uint32_t b = src[1 + (i >> 1)];
            weights[i] = (uint8_t)((i & 1u) ? (b & 0xFu) : (b >> 4));
        }
        bits_read += n * 4;
    }
    bytes_read = (bits_read + 7u) >> 3;
    return 0;
}

B200Z_HDN inline int huf_read_weights(const uint8_t *src, uint32_t len, uint8_t *weights, uint32_t &nweights, uint32_t &bytes_read) {
    int16_t probs[256];
    uint32_t tab[64];
    uint16_t counter[256];
    return huf_read_weights_scratch(src, len, weights, nweights, bytes_read, probs, tab, counter);
}

// build_table_from_weights into a HufSlot (serial form: dictionaries on the host; the per-block GPU form is in setup.cuh)
B200Z_HDN inline int huf_build_table(const uint8_t *weights, uint32_t nweights, HufSlot *slot, uint32_t &max_bits_out) {
    uint32_t weight_sum = 0;
    for (uint32_t i = 0; i < nweights; i++) {
        uint32_t w = weights[i];
        if (w > HUF_MAX_BITS) return B200Z_ERR_HUF_WEIGHT_BIGGER_THAN_MAX_NUM_BITS;
        weight_sum += w > 0 ? 1u << (w - 1) : 0u;
    }
    if (weight_sum == 0) return B200Z_ERR_HUF_MISSING_WEIGHTS;
    const uint32_t max_bits = hbs(weight_sum);
    const uint32_t left_over = (1u << max_bits) - weight_sum;
    if (left_over == 0 || (left_over & (left_over - 1))) return B200Z_ERR_HUF_LEFTOVER_NOT_POWER_OF_2;
    const uint32_t last_weight = hbs(left_over);
    if (max_bits > HUF_MAX_BITS) return B200Z_ERR_HUF_MAX_BITS_TOO_HIGH;
    // rank counts per code length (bit_ranks, :328-332); code length = max_bits + 1 - weight
    uint32_t rank_count[HUF_MAX_BITS + 2];
    for (uint32_t b = 0; b <= max_bits; b++) rank_count[b] = 0;
    for (uint32_t i = 0; i < nweights; i++) rank_count[weights[i] ? max_bits + 1 - weights[i] : 0]++;
    rank_count[max_bits + 1 - last_weight]++;
    // starting index per code length: longest codes first (:344-351)
    uint32_t rank_idx[HUF_MAX_BITS + 2];
    rank_idx[max_bits] = 0;
    for (uint32_t b = max_bits; b >= 1; b--) rank_idx[b - 1] = rank_idx[b] + rank_count[b] * (1u << (max_bits - b));
    // fill in symbol order (:360-374); the implicit last symbol is index nweights (wraps to u8 like `symbol as u8`)
    for (uint32_t s = 0; s <= nweights; s++) {
        uint32_t w = s < nweights ? weights[s] : last_weight;
        if (w == 0) continue;
        uint32_t b = max_bits + 1 - w, n = 1u << (max_bits - b), base = rank_idx[b];
        rank_idx[b] += n;
        for (uint32_t i = 0; i < n; i++) huf_set(slot, base + i, s & 0xffu, b);
    }
    max_bits_out = max_bits;
    return 0;
}

// HuffmanTable::build_decoder (huff0_decoder.rs:117-123) into a HufSlot
B200Z_HDN inline int huf_build_decoder(const uint8_t *src, uint32_t len, HufSlot *slot, uint32_t &bytes_read) {
    uint8_t weights[260];
    uint32_t nweights;
    int e = huf_read_weights(src, len, weights, nweights, bytes_read);
    if (e) return e;
    uint32_t mb;
    e = huf_build_table(weights, nweights, slot, mb);
    if (e) return e;
    slot->max_bits = mb;
    return 0;
}

}  // namespace b200z
