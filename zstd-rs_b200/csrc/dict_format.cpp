// dict_format.cpp -- the zstd dictionary writer of b200z_dict_finalize and b200z_debug_dict_from_counts (host only): entropy
// tables from symbol counts, then the layout Dictionary::decode_dict reads (dictionary.rs:45-126, RFC 8878 section 5):
//   magic 0xEC30A437 | ID | Huffman description | OF, ML, LL FSE descriptions | repeat offsets 1, 4, 8 | content
// The tables are written with the encoder's own writers (encode.cuh) at ZDICT's accuracy logs (OF 8, ML 9, LL 9).
#include <string.h>

#include <algorithm>

#include "compress.h"
#include "plan.h"

namespace b200z {

namespace {

constexpr size_t kMinContent = 8;   // the largest repeat offset of the header: the content must be at least that long

// floor(log2 x), x > 0 (ZSTD_highbit32)
uint32_t highbit64(uint64_t x) { return 63u - (uint32_t)__builtin_clzll(x); }

// one histogram as u32 counts: scaled down (by a power of two, a nonzero count staying >= 1) until its total is below 2^30, so
// that the table builders' u32 sums cannot overflow; every symbol in [0, need] then gets at least 1, as ZDICT does, so the
// table can code anything the encoder may meet
void scaled_counts(const uint64_t *in, uint32_t n, uint32_t need, uint32_t *out) {
    uint64_t total = 0;
    for (uint32_t s = 0; s < n; s++) total += in[s];
    uint32_t shift = 0;
    while ((total >> shift) >= (1ull << 30) - 512) shift++;
    for (uint32_t s = 0; s < n; s++) {
        const uint64_t v = in[s] >> shift;
        out[s] = (uint32_t)(v ? v : in[s] ? 1 : 0);
        if (s <= need && !out[s]) out[s] = 1;
    }
}

}  // namespace

int dict_check_args(size_t content_len, uint32_t dict_id, size_t dict_cap) {
    if (content_len < kMinContent || content_len >= (1ull << 31) || dict_id >= (1u << 31) || dict_cap < B200Z_DICT_HEADER_MAX + kMinContent)
        return B200Z_ERR_INVALID_ARGUMENT;
    return 0;
}

int dict_from_counts(const uint64_t *counts, const uint8_t *content, size_t content_len, uint32_t dict_id, uint8_t *dict, size_t dict_cap,
                     size_t *dict_len) {
    if (!counts || !dict || !dict_len || !content) return B200Z_ERR_INVALID_ARGUMENT;
    if (int e = dict_check_args(content_len, dict_id, dict_cap)) return e;
    uint8_t hdr[B200Z_DICT_HEADER_MAX];
    size_t h = 8;
    // ---- Huffman: lengths <= 11 bits over all 256 byte values.  huf_write_weights writes nothing when every length is the
    // same (all 8 bits: flat counts) or the description would reach 128 bytes; the table is then the fixed near-flat code
    // 7 bits for 0x00, 9 bits for 0xFE and 0xFF, 8 bits for the rest (Kraft sum 1: 2^-7 + 2 * 2^-9 = 3 * 2^-8)
    uint32_t lit[256];
    scaled_counts(counts + DS_LIT, 256, 255, lit);
    uint8_t len[256];
    uint32_t maxb = huf_lengths(lit, len);
    uint32_t tree = huf_write_weights(len, maxb, hdr + h, 128);
    if (!tree) {
        memset(len, 8, sizeof len);
        len[0] = 7;
        len[254] = len[255] = 9;
        maxb = 9;
        tree = huf_write_weights(len, maxb, hdr + h, 128);
        if (!tree) return B200Z_ERR_INVALID_ARGUMENT;   // cannot happen: that description is a few bytes long
    }
    h += tree;
    // ---- FSE: OF, ML, LL.  Every OF code a match into the content can need gets a count (libzstd checks codes up to
    // highbit32(content size + 128 KiB) when it compresses with the dictionary)
    struct { uint32_t lo, n, log, need; } order[3] = {
        {DS_OF, 32, 8, std::min<uint32_t>(31u, highbit64((uint64_t)content_len + 131072))}, {DS_ML, 53, 9, 52}, {DS_LL, 36, 9, 35}};
    for (const auto &o : order) {
        uint32_t cnt[64];
        scaled_counts(counts + o.lo, o.n, o.need, cnt);
        uint32_t maxsym = 0, total = 0;
        for (uint32_t s = 0; s < o.n; s++) if (cnt[s]) { maxsym = s; total += cnt[s]; }
        int16_t norm[64];
        fse_normalize(cnt, maxsym, total, o.log, norm);
        h += fse_write_ncount(norm, maxsym, o.log, hdr + h, (uint32_t)(sizeof hdr - h));
    }
    for (uint32_t r : {1u, 4u, 8u}) { put_le(hdr, sizeof hdr, (uint32_t)h, r, 4); h += 4; }
    // ---- the content's last bytes that fit, and the ID (libzstd's rule for a derived one, over the content written)
    const size_t keep = std::min(content_len, dict_cap - h);
    const uint8_t *tail = content + (content_len - keep);
    if (!dict_id) {
        XXH64State x;
        x.reset();
        x.update(tail, keep);
        dict_id = (uint32_t)(x.digest() % ((1ull << 31) - 32768)) + 32768;
    }
    put_le(hdr, sizeof hdr, 0, 0xEC30A437u, 4);
    put_le(hdr, sizeof hdr, 4, dict_id, 4);
    memcpy(dict, hdr, h);
    memmove(dict + h, tail, keep);
    *dict_len = h + keep;
    return 0;
}

}  // namespace b200z
