/*
 * ruzstd_oracle.c -- CPU restatement (plain C) of ruzstd's decode path; see ruzstd_oracle.h.
 * TEST INFRASTRUCTURE ONLY: never linked into or called from the product path.
 *
 * Every function cites the reference file:line it follows (relative to /root/reference/ruzstd/src/).
 * The loop structure is the reference's (single-threaded, block by block, one sequence at a time); the
 * growable RingBuffer (decoding/ringbuffer.rs) is replaced by a flat vector + head index with identical
 * observable behaviour (len(), extend, extend_from_within, drop_first_n, as_slices order).
 */
#include "ruzstd_oracle.h"

#include <pthread.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ small vector helpers */
typedef struct { uint8_t *p; size_t len, cap; } bytevec;

static int bv_reserve(bytevec *v, size_t extra) {
    if (v->len + extra <= v->cap) return 0;
    size_t ncap = v->cap ? v->cap : 4096;
    while (ncap < v->len + extra) ncap *= 2;
    uint8_t *np = (uint8_t *)realloc(v->p, ncap);
    if (!np) return -1;
    v->p = np; v->cap = ncap;
    return 0;
}
static int bv_push(bytevec *v, const uint8_t *d, size_t n) {
    if (bv_reserve(v, n)) return -1;
    if (n) memcpy(v->p + v->len, d, n);
    v->len += n;
    return 0;
}
static void bv_free(bytevec *v) { free(v->p); v->p = NULL; v->len = v->cap = 0; }

/* ------------------------------------------------------------------ XXH64 (seed 0)
 * The reference uses twox_hash::XxHash64::with_seed(0) (decode_buffer.rs:42) fed on drain
 * (decode_buffer.rs:225-226, 290, 301); `finish() as u32` is the content checksum (frame_decoder.rs:262-270). */
#define XP1 0x9E3779B185EBCA87ULL
#define XP2 0xC2B2AE3D27D4EB4FULL
#define XP3 0x165667B19E3779F9ULL
#define XP4 0x85EBCA77C2B2AE63ULL
#define XP5 0x27D4EB2F165667C5ULL
typedef struct { uint64_t v[4]; uint64_t total; uint8_t mem[32]; uint32_t memsize; } xxh64_state;
static uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static uint64_t rd64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }
static uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint64_t xxh_round(uint64_t acc, uint64_t in) { acc += in * XP2; acc = rotl64(acc, 31); return acc * XP1; }
static uint64_t xxh_merge(uint64_t acc, uint64_t v) { v = xxh_round(0, v); acc ^= v; return acc * XP1 + XP4; }
static void xxh64_reset(xxh64_state *s) {
    s->v[0] = XP1 + XP2; s->v[1] = XP2; s->v[2] = 0; s->v[3] = 0ULL - XP1; s->total = 0; s->memsize = 0;
}
static void xxh64_update(xxh64_state *s, const uint8_t *p, size_t len) {
    s->total += len;
    if (s->memsize + len < 32) { if (len) memcpy(s->mem + s->memsize, p, len); s->memsize += (uint32_t)len; return; }
    const uint8_t *end = p + len;
    if (s->memsize) {
        size_t fill = 32 - s->memsize;
        memcpy(s->mem + s->memsize, p, fill);
        for (int i = 0; i < 4; i++) s->v[i] = xxh_round(s->v[i], rd64(s->mem + 8 * i));
        p += fill; s->memsize = 0;
    }
    while (p + 32 <= end) { for (int i = 0; i < 4; i++) s->v[i] = xxh_round(s->v[i], rd64(p + 8 * i)); p += 32; }
    if (p < end) { memcpy(s->mem, p, (size_t)(end - p)); s->memsize = (uint32_t)(end - p); }
}
static uint64_t xxh64_digest(const xxh64_state *s) {
    uint64_t h;
    if (s->total >= 32) {
        h = rotl64(s->v[0], 1) + rotl64(s->v[1], 7) + rotl64(s->v[2], 12) + rotl64(s->v[3], 18);
        for (int i = 0; i < 4; i++) h = xxh_merge(h, s->v[i]);
    } else h = s->v[2] + XP5;
    h += s->total;
    const uint8_t *p = s->mem, *end = s->mem + s->memsize;
    while (p + 8 <= end) { h ^= xxh_round(0, rd64(p)); h = rotl64(h, 27) * XP1 + XP4; p += 8; }
    if (p + 4 <= end) { h ^= (uint64_t)rd32(p) * XP1; h = rotl64(h, 23) * XP2 + XP3; p += 4; }
    while (p < end) { h ^= (*p) * XP5; h = rotl64(h, 11) * XP1; p++; }
    h ^= h >> 33; h *= XP2; h ^= h >> 29; h *= XP3; h ^= h >> 32;
    return h;
}
uint64_t zo_xxh64(const uint8_t *data, size_t len) { xxh64_state s; xxh64_reset(&s); xxh64_update(&s, data, len); return xxh64_digest(&s); }

/* ------------------------------------------------------------------ forward BitReader (bit_io/bit_reader.rs) */
typedef struct { size_t idx; const uint8_t *src; size_t len; } bitreader;
static size_t br_bits_left(const bitreader *b) { return b->len * 8 - b->idx; }               /* :13-15 */
/* get_bits :28-91 -- LSB-first; returns -1 for NotEnoughRemainingBits / TooManyBits */
static int br_get_bits(bitreader *b, size_t n, uint64_t *out) {
    if (n > 64) return -1;
    if (br_bits_left(b) < n) return -1;
    uint64_t v = 0;
    for (size_t i = 0; i < n; i++) {                       /* same result as the byte-chunked loop :44-86 */
        size_t bit = b->idx + i;
        v |= (uint64_t)((b->src[bit >> 3] >> (bit & 7)) & 1) << i;
    }
    b->idx += n;
    *out = v;
    return 0;
}
static void br_return_bits(bitreader *b, size_t n) { b->idx -= n; }                            /* :21-26 */

/* ------------------------------------------------------------------ BitReaderReversed (bit_io/bit_reader_reverse.rs)
 * Restated with the same fields.  refill :43-87, get_bits :92-100, peek_bits :105-113, get_bits_triple :151-162,
 * bits_remaining :27-29. */
typedef struct {
    size_t index; uint8_t bits_consumed; size_t extra_bits; const uint8_t *src; size_t len; uint64_t container;
} brr;
static void brr_new(brr *r, const uint8_t *src, size_t len) {                                  /* :31-39 */
    r->index = len; r->bits_consumed = 64; r->src = src; r->len = len; r->container = 0; r->extra_bits = 0;
}
static long brr_bits_remaining(const brr *r) {                                                 /* :27-29 */
    return (long)r->index * 8 + (64 - (long)r->bits_consumed) - (long)r->extra_bits;
}
static void brr_refill(brr *r) {                                                               /* :43-87 */
    size_t bytes_consumed = r->bits_consumed / 8;
    if (bytes_consumed == 0) return;
    if (r->index >= bytes_consumed) {
        r->index -= bytes_consumed;
        r->bits_consumed &= 7;
        r->container = rd64(r->src + r->index);           /* source[index..][..8]; index+8 <= len holds, see header note */
    } else if (r->index > 0) {
        if (r->len >= 8) r->container = rd64(r->src);
        else { uint8_t v[8] = {0}; memcpy(v, r->src, r->len); r->container = rd64(v); }
        r->bits_consumed = (uint8_t)(r->bits_consumed - 8 * (uint8_t)r->index);
        r->index = 0;
        r->container <<= r->bits_consumed;                /* bits_consumed < 64 here */
        r->extra_bits += r->bits_consumed;
        r->bits_consumed = 0;
    } else if (r->bits_consumed < 64) {
        r->container <<= r->bits_consumed;
        r->extra_bits += r->bits_consumed;
        r->bits_consumed = 0;
    } else {
        r->extra_bits += r->bits_consumed;
        r->bits_consumed = 0;
        r->container = 0;
    }
}
static uint64_t brr_peek(const brr *r, uint8_t n) {                                            /* :105-113 */
    if (n == 0) return 0;
    uint64_t mask = (n >= 64) ? ~0ULL : ((1ULL << n) - 1);
    return (r->container >> (64 - r->bits_consumed - n)) & mask;
}
static uint64_t brr_get_bits(brr *r, uint8_t n) {                                              /* :92-100 */
    if ((unsigned)r->bits_consumed + n > 64) brr_refill(r);
    uint64_t v = brr_peek(r, n);
    r->bits_consumed = (uint8_t)(r->bits_consumed + n);
    return v;
}
static void brr_get_bits_triple(brr *r, uint8_t n1, uint8_t n2, uint8_t n3, uint64_t *v1, uint64_t *v2, uint64_t *v3) { /* :151-162 */
    unsigned sum = (unsigned)n1 + n2 + n3;
    if (sum <= 56) {
        brr_refill(r);
        if (sum == 0) { *v1 = *v2 = *v3 = 0; return; }                                         /* peek_bits_triple :118-140 */
        uint64_t all = r->container >> (64 - r->bits_consumed - sum);
        *v1 = (all >> (n3 + n2)) & ((1ULL << n1) - 1);
        *v2 = (all >> n3) & ((1ULL << n2) - 1);
        *v3 = all & ((1ULL << n3) - 1);
        r->bits_consumed = (uint8_t)(r->bits_consumed + sum);
        return;
    }
    *v1 = brr_get_bits(r, n1); *v2 = brr_get_bits(r, n2); *v3 = brr_get_bits(r, n3);
}
/* the "skip padding, drop the first 1" loop shared by literals_section_decoder.rs:97-109,
 * sequence_section_decoder.rs:28-40 and huff0_decoder.rs:188-200; returns skipped_bits */
static int brr_skip_padding(brr *r) {
    int skipped = 0;
    for (;;) { uint64_t v = brr_get_bits(r, 1); skipped++; if (v == 1 || skipped > 8) break; }
    return skipped;
}

/* ------------------------------------------------------------------ FSE (fse/fse_decoder.rs) */
typedef struct { uint32_t base_line; uint8_t num_bits; uint8_t symbol; } fse_entry;       /* Entry :312-320 */
#define FSE_MAX_TABLE 512
#define FSE_MAX_PROBS 320
typedef struct {
    uint8_t max_symbol;
    fse_entry decode[FSE_MAX_TABLE]; size_t decode_len;
    uint8_t accuracy_log;
    int32_t probs[FSE_MAX_PROBS]; size_t nprobs;       /* nprobs may exceed FSE_MAX_PROBS (only counted then) */
} fse_table;

static void fse_new(fse_table *t, uint8_t max_symbol) { memset(t, 0, sizeof *t); t->max_symbol = max_symbol; } /* :87-95 */
static void fse_reset(fse_table *t) { t->nprobs = 0; t->decode_len = 0; t->accuracy_log = 0; }      /* :108-113 */
static void fse_reinit_from(fse_table *t, const fse_table *o) { uint8_t ms = t->max_symbol; *t = *o; t->max_symbol = ms; } /* :98-105 */
static uint32_t highest_bit_set(uint32_t x) { return 32 - (uint32_t)__builtin_clz(x); }             /* :326-329 (x>0) */
static size_t fse_next_position(size_t p, size_t table_size) {                                      /* :334-338 */
    p += (table_size >> 1) + (table_size >> 3) + 3; p &= table_size - 1; return p;
}
static void fse_calc_baseline_and_numbits(uint32_t total, uint32_t nsym, uint32_t state_number, uint32_t *bl, uint8_t *nb) { /* :340-366 */
    if (nsym == 0) { *bl = 0; *nb = 0; return; }
    uint32_t slices = ((1u << (highest_bit_set(nsym) - 1)) == nsym) ? nsym : (1u << highest_bit_set(nsym));
    uint32_t n_double = slices - nsym;
    uint32_t n_single = nsym - n_double;
    uint32_t slice_width = total / slices;
    uint32_t num_bits = highest_bit_set(slice_width) - 1;
    if (state_number < n_double) { *bl = n_single * slice_width + state_number * slice_width * 2; *nb = (uint8_t)(num_bits + 1); }
    else { *bl = (state_number - n_double) * slice_width; *nb = (uint8_t)num_bits; }
}
/* build_decoding_table :141-220 */
static int fse_build_decoding_table(fse_table *t) {
    if (t->nprobs > (size_t)t->max_symbol + 1) return ZO_ERR_FSE_TOO_MANY_SYMBOLS;
    size_t table_size = (size_t)1 << t->accuracy_log;
    if (table_size > FSE_MAX_TABLE) return ZO_ERR_REFERENCE_WOULD_PANIC; /* unreachable: logs are capped by callers */
    memset(t->decode, 0, sizeof(fse_entry) * table_size);
    t->decode_len = table_size;
    size_t negative_idx = table_size;
    for (size_t s = 0; s < t->nprobs; s++)
        if (t->probs[s] == -1) {
            if (negative_idx == 0) return ZO_ERR_REFERENCE_WOULD_PANIC;   /* index underflow in the reference */
            negative_idx--;
            t->decode[negative_idx].symbol = (uint8_t)s;
            t->decode[negative_idx].base_line = 0;
            t->decode[negative_idx].num_bits = t->accuracy_log;
        }
    size_t position = 0;
    for (size_t idx = 0; idx < t->nprobs; idx++) {
        if (t->probs[idx] <= 0) continue;
        for (int32_t k = 0; k < t->probs[idx]; k++) {
            t->decode[position].symbol = (uint8_t)idx;
            position = fse_next_position(position, table_size);
            size_t guard = 0;
            while (position >= negative_idx) {
                position = fse_next_position(position, table_size);
                if (++guard > table_size) return ZO_ERR_REFERENCE_WOULD_PANIC; /* reference would spin forever */
            }
        }
    }
    uint32_t counter[256]; memset(counter, 0, sizeof counter);
    for (size_t idx = 0; idx < negative_idx; idx++) {
        uint8_t sym = t->decode[idx].symbol;
        int32_t prob = (sym < t->nprobs) ? t->probs[sym] : 0;
        uint32_t bl; uint8_t nb;
        fse_calc_baseline_and_numbits((uint32_t)table_size, (uint32_t)prob, counter[sym], &bl, &nb);
        if (nb > t->accuracy_log) return ZO_ERR_REFERENCE_WOULD_PANIC;       /* assert :213 */
        counter[sym]++;
        t->decode[idx].base_line = bl; t->decode[idx].num_bits = nb;
    }
    return 0;
}
/* read_probabilities :224-307; *bytes_read on success */
static int fse_read_probabilities(fse_table *t, const uint8_t *src, size_t len, uint8_t max_log, size_t *bytes_read) {
    t->nprobs = 0;
    bitreader br = {0, src, len};
    uint64_t v;
    if (br_get_bits(&br, 4, &v)) return ZO_ERR_FSE_GET_BITS;
    t->accuracy_log = (uint8_t)(5 + v);
    if (t->accuracy_log > max_log) return ZO_ERR_FSE_ACC_LOG_TOO_BIG;
    if (t->accuracy_log == 0) return ZO_ERR_FSE_ACC_LOG_IS_ZERO;
    uint32_t probability_sum = 1u << t->accuracy_log, probability_counter = 0;
    while (probability_counter < probability_sum) {
        uint32_t max_remaining = probability_sum - probability_counter + 1;
        uint32_t bits_to_read = highest_bit_set(max_remaining);
        if (br_get_bits(&br, bits_to_read, &v)) return ZO_ERR_FSE_GET_BITS;
        uint32_t unchecked = (uint32_t)v;
        uint32_t low_threshold = ((1u << bits_to_read) - 1) - max_remaining;
        uint32_t mask = (1u << (bits_to_read - 1)) - 1;
        uint32_t small = unchecked & mask;
        uint32_t value;
        if (small < low_threshold) { br_return_bits(&br, 1); value = small; }
        else if (unchecked > mask) value = unchecked - low_threshold;
        else value = unchecked;
        int32_t prob = (int32_t)value - 1;
        if (t->nprobs < FSE_MAX_PROBS) t->probs[t->nprobs] = prob;
        t->nprobs++;
        if (prob != 0) {
            probability_counter += (prob > 0) ? (uint32_t)prob : 1u;
        } else {
            for (;;) {
                if (br_get_bits(&br, 2, &v)) return ZO_ERR_FSE_GET_BITS;
                for (uint64_t k = 0; k < v; k++) { if (t->nprobs < FSE_MAX_PROBS) t->probs[t->nprobs] = 0; t->nprobs++; }
                if (v != 3) break;
            }
        }
    }
    if (probability_counter != probability_sum) return ZO_ERR_FSE_PROBABILITY_COUNTER_MISMATCH;
    if (t->nprobs > (size_t)t->max_symbol + 1) return ZO_ERR_FSE_TOO_MANY_SYMBOLS;
    *bytes_read = (br.idx % 8 == 0) ? br.idx / 8 : br.idx / 8 + 1;
    return 0;
}
/* build_decoder :116-123 */
static int fse_build_decoder(fse_table *t, const uint8_t *src, size_t len, uint8_t max_log, size_t *bytes_read) {
    t->accuracy_log = 0;
    int e = fse_read_probabilities(t, src, len, max_log, bytes_read);
    if (e) return e;
    return fse_build_decoding_table(t);
}
/* build_from_probabilities :126-137 */
static int fse_build_from_probabilities(fse_table *t, uint8_t acc_log, const int32_t *probs, size_t n) {
    if (acc_log == 0) return ZO_ERR_FSE_ACC_LOG_IS_ZERO;
    t->nprobs = n;
    for (size_t i = 0; i < n && i < FSE_MAX_PROBS; i++) t->probs[i] = probs[i];
    t->accuracy_log = acc_log;
    return fse_build_decoding_table(t);
}
/* FSEDecoder :5-51: the state IS the current Entry */
typedef struct { fse_entry state; const fse_table *table; } fse_decoder;
static void fsed_new(fse_decoder *d, const fse_table *t) {                                        /* :14-23 */
    d->table = t;
    if (t->decode_len) d->state = t->decode[0]; else { d->state.base_line = 0; d->state.num_bits = 0; d->state.symbol = 0; }
}
static int fsed_init_state(fse_decoder *d, brr *bits) {                                           /* :32-40 */
    if (d->table->accuracy_log == 0) return ZO_ERR_FSE_TABLE_IS_UNINITIALIZED;
    uint64_t s = brr_get_bits(bits, d->table->accuracy_log);
    /* decode[new_state] (:37) past the cells: a description that failed after setting accuracy_log (AccLogTooBig, :230-237)
     * leaves the previous cells, or none; decode_blocks called again after that error reaches it through a Repeat mode */
    if (s >= d->table->decode_len) return ZO_ERR_REFERENCE_WOULD_PANIC;
    d->state = d->table->decode[s];
    return 0;
}
static int fsed_update_state(fse_decoder *d, brr *bits) {                                         /* :43-51 */
    uint64_t add = brr_get_bits(bits, d->state.num_bits);
    uint32_t ns = d->state.base_line + (uint32_t)add;
    if (ns >= d->table->decode_len) return ZO_ERR_REFERENCE_WOULD_PANIC;   /* cannot happen for tables built above */
    d->state = d->table->decode[ns];
    return 0;
}

/* ------------------------------------------------------------------ Huffman (huff0/huff0_decoder.rs) */
typedef struct { uint8_t symbol, num_bits; } huf_entry;                                          /* Entry :389-394 */
typedef struct {
    huf_entry decode[2048]; size_t decode_len;
    uint8_t weights[260]; size_t nweights;
    uint8_t max_num_bits;
    uint8_t bits[260]; size_t nbits;
    fse_table fse;
} huf_table;
static void huf_new(huf_table *h) { memset(h, 0, sizeof *h); fse_new(&h->fse, 255); }            /* :78-89 */
static void huf_reset(huf_table *h) { h->decode_len = 0; h->nweights = 0; h->max_num_bits = 0; h->nbits = 0; fse_reset(&h->fse); } /* :104-112 */
/* read_weights :132-278 */
static int huf_read_weights(huf_table *h, const uint8_t *src, size_t len, uint32_t *bytes_read) {
    if (len == 0) return ZO_ERR_HUF_SOURCE_IS_EMPTY;
    uint8_t header = src[0];
    size_t bits_read = 8;
    if (header < 128) {
        const uint8_t *fse_stream = src + 1; size_t fse_len = len - 1;
        if ((size_t)header > fse_len) return ZO_ERR_HUF_NOT_ENOUGH_BYTES_FOR_WEIGHTS;
        size_t used = 0;
        int e = fse_build_decoder(&h->fse, fse_stream, fse_len, 6, &used);
        if (e) return e;                                           /* HuffmanTableError::FSETableError(leaf) */
        if (used > (size_t)header) return ZO_ERR_HUF_FSE_TABLE_USED_TOO_MANY_BYTES;
        fse_decoder dec1, dec2; fsed_new(&dec1, &h->fse); fsed_new(&dec2, &h->fse);
        size_t clen = (size_t)header - used;
        if (fse_len - used < clen) return ZO_ERR_HUF_NOT_ENOUGH_BYTES_TO_DECOMPRESS_WEIGHTS;
        brr br; brr_new(&br, fse_stream + used, clen);
        bits_read += (used + clen) * 8;
        int skipped = brr_skip_padding(&br);
        if (skipped > 8) return ZO_ERR_HUF_EXTRA_PADDING;
        if ((e = fsed_init_state(&dec1, &br))) return ZO_ERR_HUF_FSE_DECODER;
        if ((e = fsed_init_state(&dec2, &br))) return ZO_ERR_HUF_FSE_DECODER;
        h->nweights = 0;
        for (;;) {                                                                                /* :208-234 */
            h->weights[h->nweights++] = dec1.state.symbol;
            if (fsed_update_state(&dec1, &br)) return ZO_ERR_REFERENCE_WOULD_PANIC;
            if (brr_bits_remaining(&br) <= -1) { h->weights[h->nweights++] = dec2.state.symbol; break; }
            h->weights[h->nweights++] = dec2.state.symbol;
            if (fsed_update_state(&dec2, &br)) return ZO_ERR_REFERENCE_WOULD_PANIC;
            if (brr_bits_remaining(&br) <= -1) { h->weights[h->nweights++] = dec1.state.symbol; break; }
            if (h->nweights > 255) return ZO_ERR_HUF_TOO_MANY_WEIGHTS;
        }
    } else {
        const uint8_t *raw = src + 1; size_t raw_len = len - 1;
        unsigned num_weights = (unsigned)header - 127;
        size_t bytes_needed = (num_weights % 2 == 0) ? num_weights / 2 : num_weights / 2 + 1;
        h->nweights = num_weights; memset(h->weights, 0, num_weights);
        if (raw_len < bytes_needed) return ZO_ERR_HUF_NOT_ENOUGH_BYTES_IN_SOURCE;
        for (unsigned i = 0; i < num_weights; i++) {
            h->weights[i] = (i % 2 == 0) ? (uint8_t)(raw[i / 2] >> 4) : (uint8_t)(raw[i / 2] & 0xF);
            bits_read += 4;
        }
    }
    *bytes_read = (uint32_t)((bits_read % 8 == 0) ? bits_read / 8 : bits_read / 8 + 1);
    return 0;
}
/* build_table_from_weights :284-377 */
static int huf_build_table_from_weights(huf_table *h) {
    h->nbits = h->nweights + 1;
    memset(h->bits, 0, h->nbits);
    uint32_t weight_sum = 0;
    for (size_t i = 0; i < h->nweights; i++) {
        uint8_t w = h->weights[i];
        if (w > 11) return ZO_ERR_HUF_WEIGHT_BIGGER_THAN_MAX_NUM_BITS;
        weight_sum += w > 0 ? 1u << (w - 1) : 0;
    }
    if (weight_sum == 0) return ZO_ERR_HUF_MISSING_WEIGHTS;
    uint8_t max_bits = (uint8_t)highest_bit_set(weight_sum);
    uint32_t left_over = (1u << max_bits) - weight_sum;
    if (left_over == 0 || (left_over & (left_over - 1))) return ZO_ERR_HUF_LEFTOVER_NOT_POWER_OF_2;
    uint8_t last_weight = (uint8_t)highest_bit_set(left_over);
    for (size_t s = 0; s < h->nweights; s++) h->bits[s] = h->weights[s] > 0 ? (uint8_t)(max_bits + 1 - h->weights[s]) : 0;
    h->bits[h->nweights] = (uint8_t)(max_bits + 1 - last_weight);
    h->max_num_bits = max_bits;
    if (max_bits > 11) return ZO_ERR_HUF_MAX_BITS_TOO_HIGH;
    uint32_t bit_ranks[13] = {0};
    for (size_t i = 0; i < h->nbits; i++) bit_ranks[h->bits[i]]++;
    h->decode_len = (size_t)1 << max_bits;
    memset(h->decode, 0, sizeof(huf_entry) * h->decode_len);
    size_t rank_indexes[13] = {0};
    rank_indexes[max_bits] = 0;
    for (int b = max_bits; b >= 1; b--) rank_indexes[b - 1] = rank_indexes[b] + (size_t)bit_ranks[b] * ((size_t)1 << (max_bits - b));
    if (rank_indexes[0] != h->decode_len) return ZO_ERR_REFERENCE_WOULD_PANIC;                    /* assert :353 */
    for (size_t s = 0; s < h->nbits; s++) {
        uint8_t b = h->bits[s];
        if (b != 0) {
            size_t base = rank_indexes[b], n = (size_t)1 << (max_bits - b);
            rank_indexes[b] += n;
            for (size_t i = 0; i < n; i++) { h->decode[base + i].symbol = (uint8_t)s; h->decode[base + i].num_bits = b; }
        }
    }
    return 0;
}
/* build_decoder :117-123 */
static int huf_build_decoder(huf_table *h, const uint8_t *src, size_t len, uint32_t *bytes_used) {
    h->decode_len = 0;
    int e = huf_read_weights(h, src, len, bytes_used);
    if (e) return e;
    return huf_build_table_from_weights(h);
}

/* ------------------------------------------------------------------ DecodeBuffer (decoding/decode_buffer.rs) */
typedef struct {
    bytevec buf; size_t head;        /* RingBuffer stand-in: live bytes are buf.p[head..buf.len) */
    bytevec dict_content;
    size_t window_size;
    uint64_t total_output_counter;
    xxh64_state hash;
} decode_buffer;
static size_t db_len(const decode_buffer *b) { return b->buf.len - b->head; }                   /* :58-60 */
static void db_reset(decode_buffer *b, size_t window_size) {                                     /* :46-56 */
    b->window_size = window_size; b->buf.len = 0; b->head = 0; b->dict_content.len = 0;
    b->total_output_counter = 0; xxh64_reset(&b->hash);
}
static int db_push(decode_buffer *b, const uint8_t *d, size_t n) {                               /* :74-77 */
    if (bv_push(&b->buf, d, n)) return ZO_ERR_OUT_OF_MEMORY;
    b->total_output_counter += n; return 0;
}
static int db_extend_from_within(decode_buffer *b, size_t start_idx, size_t n) {                 /* ringbuffer.rs:283-454 */
    if (bv_reserve(&b->buf, n)) return ZO_ERR_OUT_OF_MEMORY;
    memcpy(b->buf.p + b->buf.len, b->buf.p + b->head + start_idx, n);   /* caller guarantees start+n <= len */
    b->buf.len += n; return 0;
}
static int db_repeat(decode_buffer *b, size_t offset, size_t match_length);
static int db_repeat_from_dict(decode_buffer *b, size_t offset, size_t match_length) {           /* :143-179 */
    if (b->total_output_counter <= (uint64_t)b->window_size) {
        size_t bytes_from_dict = offset - db_len(b);
        if (bytes_from_dict > b->dict_content.len) return ZO_ERR_EXEC_NOT_ENOUGH_BYTES_IN_DICTIONARY;
        if (bytes_from_dict < match_length) {
            if (bv_push(&b->buf, b->dict_content.p + b->dict_content.len - bytes_from_dict, bytes_from_dict)) return ZO_ERR_OUT_OF_MEMORY;
            b->total_output_counter += bytes_from_dict;
            return db_repeat(b, db_len(b), match_length - bytes_from_dict);
        } else {
            size_t low = b->dict_content.len - bytes_from_dict;
            if (bv_push(&b->buf, b->dict_content.p + low, match_length)) return ZO_ERR_OUT_OF_MEMORY;
        }
        return 0;
    }
    return ZO_ERR_EXEC_OFFSET_TOO_BIG;
}
static int db_repeat(decode_buffer *b, size_t offset, size_t match_length) {                     /* :79-111 */
    if (offset > db_len(b)) return db_repeat_from_dict(b, offset, match_length);
    size_t buf_len = db_len(b), start_idx = buf_len - offset, end_idx = start_idx + match_length;
    if (end_idx > buf_len) {                                                                     /* repeat_in_chunks :113-141 */
        size_t left = match_length;
        while (left > 0) {
            size_t chunk = offset < left ? offset : left;
            int e = db_extend_from_within(b, start_idx, chunk); if (e) return e;
            left -= chunk; start_idx += chunk;
        }
    } else { int e = db_extend_from_within(b, start_idx, match_length); if (e) return e; }
    b->total_output_counter += match_length;
    return 0;
}
static int db_can_drain_to_window_size(const decode_buffer *b, size_t *n) {                      /* :182-188 */
    if (db_len(b) > b->window_size) { *n = db_len(b) - b->window_size; return 1; } return 0;
}
static void db_drop_first_n(decode_buffer *b, size_t n) {
    b->head += n;
    if (b->head == b->buf.len) { b->head = 0; b->buf.len = 0; }
    else if (b->head > (1u << 20) && b->head > b->buf.len / 2) {   /* compaction: not observable */
        memmove(b->buf.p, b->buf.p + b->head, b->buf.len - b->head); b->buf.len -= b->head; b->head = 0;
    }
}
/* drain_to :256-314 with a write callback; one slice (the flat buffer never wraps).  Returns bytes written
 * or a negative value if the sink failed (bytes accepted before the failure are still dropped+hashed, as
 * the DrainGuard does :265-281). */
static long db_drain_to(decode_buffer *b, size_t amount, zo_write_fn write, void *user, uint8_t *target) {
    if (amount == 0) return 0;
    size_t n1 = db_len(b) < amount ? db_len(b) : amount;
    const uint8_t *slice = b->buf.p + b->head;
    size_t written = 0; int failed = 0;
    if (target) { memcpy(target, slice, n1); written = n1; }
    else {
        while (written < n1) {                                                                   /* write_all_bytes :318-328 */
            long w = write(user, slice + written, n1 - written);
            if (w == 0) break;
            if (w < 0) { failed = 1; break; }
            written += (size_t)w;
        }
    }
    xxh64_update(&b->hash, slice, written);
    db_drop_first_n(b, written);
    return failed ? -1 : (long)written;
}

/* ------------------------------------------------------------------ scratch / dictionary / decoder state */
typedef struct { uint32_t ll, ml, of; } sequence;                                               /* blocks/sequence_section.rs:21-37 */
typedef struct {
    uint32_t id; fse_table of, ml, ll; int of_rle, ml_rle, ll_rle; huf_table huf;
    bytevec content; uint32_t offset_hist[3];
} dictionary;                                                                                    /* dictionary.rs:12-37 */

typedef struct {                                                                                 /* scratch.rs:15-27 */
    huf_table huf;
    fse_table offsets, literal_lengths, match_lengths; int of_rle, ll_rle, ml_rle;              /* FSEScratch :99-106; -1 = None */
    decode_buffer buffer;
    uint32_t offset_hist[3];
    bytevec literals_buffer;
    sequence *sequences; size_t nseq, seq_cap;
    bytevec block_content_buffer;
} scratch;

struct zo_decoder {
    int has_state;
    /* FrameHeader (frame.rs:88-111) */
    uint8_t descriptor, window_descriptor; int has_dict_id; uint32_t dict_id; uint64_t frame_content_size;
    scratch sc;
    int frame_finished; size_t block_counter; uint64_t bytes_read_counter; int has_check_sum; uint32_t check_sum;
    int using_dict; uint32_t using_dict_id;
    dictionary **dicts; size_t ndicts;
    uint64_t max_window_size;
    int last_stage;
    uint32_t skip_length;             /* SkipFrame{length} of the last init */
    /* trace */
    int trace_on; zo_block_trace *tb; size_t ntb, tb_cap; bytevec tlits; zo_seq_trace *tseq; size_t ntseq, tseq_cap;
    uint64_t trace_out_pos;
};

#define MAGIC_NUM 0xFD2FB528u                              /* common/mod.rs:6 */
#define MIN_WINDOW_SIZE 1024ULL                            /* common/mod.rs:10 */
#define MAX_WINDOW_SIZE ((1ULL << 41) + 7 * (1ULL << 38))  /* common/mod.rs:14 */
#define MAX_BLOCK_SIZE (128u * 1024u)                      /* common/mod.rs:21 */
#define DEFAULT_MAX_WINDOW_SIZE (1024ULL * 1024 * 128)     /* frame_decoder.rs:25 */
#define MAX_LITERAL_LENGTH_CODE 35
#define MAX_MATCH_LENGTH_CODE 52
#define MAX_OFFSET_CODE 31

static void scratch_init(scratch *s, size_t window) {                                            /* scratch.rs:30-50 */
    memset(s, 0, sizeof *s);
    huf_new(&s->huf);
    fse_new(&s->offsets, MAX_OFFSET_CODE); fse_new(&s->literal_lengths, MAX_LITERAL_LENGTH_CODE); fse_new(&s->match_lengths, MAX_MATCH_LENGTH_CODE);
    s->of_rle = s->ll_rle = s->ml_rle = -1;
    db_reset(&s->buffer, window);
    s->offset_hist[0] = 1; s->offset_hist[1] = 4; s->offset_hist[2] = 8;
}
static void scratch_reset(scratch *s, size_t window) {                                           /* scratch.rs:52-68 */
    s->offset_hist[0] = 1; s->offset_hist[1] = 4; s->offset_hist[2] = 8;
    s->literals_buffer.len = 0; s->nseq = 0; s->block_content_buffer.len = 0;
    db_reset(&s->buffer, window);
    fse_reset(&s->literal_lengths); fse_reset(&s->match_lengths); fse_reset(&s->offsets);
    s->ll_rle = s->ml_rle = s->of_rle = -1;
    huf_reset(&s->huf);
}
static int scratch_init_from_dict(scratch *s, const dictionary *d) {                             /* scratch.rs:70-78 */
    fse_reinit_from(&s->offsets, &d->of); fse_reinit_from(&s->literal_lengths, &d->ll); fse_reinit_from(&s->match_lengths, &d->ml);
    s->of_rle = d->of_rle; s->ll_rle = d->ll_rle; s->ml_rle = d->ml_rle;
    { fse_table keep = s->huf.fse; (void)keep; s->huf = d->huf; }                                /* huff0_decoder.rs:93-101 */
    memcpy(s->offset_hist, d->offset_hist, sizeof s->offset_hist);
    s->buffer.dict_content.len = 0;
    if (bv_push(&s->buffer.dict_content, d->content.p, d->content.len)) return ZO_ERR_OUT_OF_MEMORY;
    return 0;
}

/* ------------------------------------------------------------------ reader helpers */
static int read_exact(zo_read_fn rd, void *user, uint8_t *buf, size_t n) {
    size_t got = 0;
    while (got < n) { long r = rd(user, buf + got, n - got); if (r <= 0) return -1; got += (size_t)r; }
    return 0;
}
typedef struct { const uint8_t *p; size_t len; } slice_reader;
static long slice_read(void *user, uint8_t *buf, size_t n) {                                     /* impl Read for &[u8] */
    slice_reader *s = (slice_reader *)user;
    size_t k = n < s->len ? n : s->len;
    if (k) memcpy(buf, s->p, k);
    s->p += k; s->len -= k;
    return (long)k;
}

/* ------------------------------------------------------------------ frame header (decoding/frame.rs) */
static int frame_read_header(zo_decoder *d, zo_read_fn rd, void *user, uint8_t *header_size) {   /* read_frame_header :6-85 */
    uint8_t buf[8];
    if (read_exact(rd, user, buf, 4)) return ZO_ERR_MAGIC_NUMBER_READ;
    unsigned bytes_read = 4;
    uint32_t magic = rd32(buf);
    if (magic >= 0x184D2A50u && magic <= 0x184D2A5Fu) {
        if (read_exact(rd, user, buf, 4)) return ZO_ERR_FRAME_DESCRIPTOR_READ;
        d->skip_length = rd32(buf);
        return ZO_ERR_SKIP_FRAME;
    }
    if (magic != MAGIC_NUM) return ZO_ERR_BAD_MAGIC_NUMBER;
    if (read_exact(rd, user, buf, 1)) return ZO_ERR_FRAME_DESCRIPTOR_READ;
    uint8_t desc = buf[0]; bytes_read += 1;
    uint8_t window_descriptor = 0; int has_dict = 0; uint32_t dict_id = 0; uint64_t fcs = 0;
    int single_segment = (desc >> 5) & 1;                                                        /* :188-190 */
    if (!single_segment) {
        if (read_exact(rd, user, buf, 1)) return ZO_ERR_WINDOW_DESCRIPTOR_READ;
        window_descriptor = buf[0]; bytes_read += 1;
    }
    static const uint8_t did_len_tab[4] = {0, 1, 2, 4};                                          /* :232-240 */
    unsigned dict_id_len = did_len_tab[desc & 3];
    if (dict_id_len) {
        if (read_exact(rd, user, buf, dict_id_len)) return ZO_ERR_DICTIONARY_ID_READ;
        bytes_read += dict_id_len;
        for (unsigned i = 0; i < dict_id_len; i++) dict_id += (uint32_t)buf[i] << (8 * i);
        if (dict_id != 0) has_dict = 1;
    }
    unsigned fcs_flag = desc >> 6;                                                               /* :213-227 */
    unsigned fcs_len = fcs_flag == 0 ? (single_segment ? 1 : 0) : (fcs_flag == 1 ? 2 : (fcs_flag == 2 ? 4 : 8));
    if (fcs_len) {
        if (read_exact(rd, user, buf, fcs_len)) return ZO_ERR_FRAME_CONTENT_SIZE_READ;
        bytes_read += fcs_len;
        for (unsigned i = 0; i < fcs_len; i++) fcs += (uint64_t)buf[i] << (8 * i);
        if (fcs_len == 2) fcs += 256;
    }
    d->descriptor = desc; d->window_descriptor = window_descriptor; d->has_dict_id = has_dict; d->dict_id = dict_id;
    d->frame_content_size = fcs;
    *header_size = (uint8_t)bytes_read;
    return 0;
}
static int frame_window_size(const zo_decoder *d, uint64_t *out) {                               /* window_size :116-139 */
    if ((d->descriptor >> 5) & 1) { *out = d->frame_content_size; return 0; }
    uint8_t exp = d->window_descriptor >> 3, mantissa = d->window_descriptor & 7;
    uint64_t window_base = 1ULL << (10 + (uint64_t)exp);
    uint64_t window_size = window_base + (window_base / 8) * mantissa;
    if (window_size >= MIN_WINDOW_SIZE) { if (window_size < MAX_WINDOW_SIZE) { *out = window_size; return 0; } return ZO_ERR_WINDOW_TOO_BIG; }
    return ZO_ERR_WINDOW_TOO_SMALL;
}

/* ------------------------------------------------------------------ literals section header (blocks/literals_section.rs) */
typedef struct { uint32_t regenerated_size; int has_compressed_size; uint32_t compressed_size; int num_streams; int ls_type; } literals_section;
static int litsec_parse(literals_section *s, const uint8_t *raw, size_t len, uint8_t *hdr_bytes) { /* parse_from_header :117-223 */
    if (len * 8 < 2) return ZO_ERR_LITSEC_GET_BITS;                 /* br.get_bits(2)? on an empty slice */
    int ls_type = raw[0] & 3; unsigned size_format = (raw[0] >> 2) & 3;
    s->ls_type = ls_type; s->has_compressed_size = 0; s->num_streams = 0; s->compressed_size = 0;
    unsigned need;                                                                               /* header_bytes_needed :66-114 */
    if (ls_type == 0 || ls_type == 1) need = (size_format == 0 || size_format == 2) ? 1 : (size_format == 1 ? 2 : 3);
    else need = (size_format <= 1) ? 3 : (size_format == 2 ? 4 : 5);
    if (len < need) return ZO_ERR_LITSEC_NOT_ENOUGH_BYTES;
    if (ls_type == 0 || ls_type == 1) {
        if (size_format == 0 || size_format == 2) s->regenerated_size = (uint32_t)raw[0] >> 3;
        else if (size_format == 1) s->regenerated_size = ((uint32_t)raw[0] >> 4) + ((uint32_t)raw[1] << 4);
        else s->regenerated_size = ((uint32_t)raw[0] >> 4) + ((uint32_t)raw[1] << 4) + ((uint32_t)raw[2] << 12);
    } else {
        s->num_streams = size_format == 0 ? 1 : 4;
        s->has_compressed_size = 1;
        if (size_format <= 1) {
            s->regenerated_size = ((uint32_t)raw[0] >> 4) + (((uint32_t)raw[1] & 0x3f) << 4);
            s->compressed_size = (uint32_t)(raw[1] >> 6) + ((uint32_t)raw[2] << 2);
        } else if (size_format == 2) {
            s->regenerated_size = ((uint32_t)raw[0] >> 4) + ((uint32_t)raw[1] << 4) + (((uint32_t)raw[2] & 0x3) << 12);
            s->compressed_size = ((uint32_t)raw[2] >> 2) + ((uint32_t)raw[3] << 6);
        } else {
            s->regenerated_size = ((uint32_t)raw[0] >> 4) + ((uint32_t)raw[1] << 4) + (((uint32_t)raw[2] & 0x3F) << 12);
            s->compressed_size = ((uint32_t)raw[2] >> 6) + ((uint32_t)raw[3] << 2) + ((uint32_t)raw[4] << 10);
        }
    }
    *hdr_bytes = (uint8_t)need;
    return 0;
}

/* ------------------------------------------------------------------ literals decode (decoding/literals_section_decoder.rs) */
static int lit_decode_stream(scratch *sc, const uint8_t *stream, size_t len, int check_landing) { /* :94-122 / :128-146 */
    const huf_table *t = &sc->huf;
    brr br; brr_new(&br, stream, len);
    int skipped = brr_skip_padding(&br);
    if (skipped > 8) return ZO_ERR_LIT_EXTRA_PADDING;
    uint64_t state = brr_get_bits(&br, t->max_num_bits);                      /* HuffmanDecoder::init_state huff0_decoder.rs:32-37 */
    long lim = -(long)t->max_num_bits;
    while (brr_bits_remaining(&br) > lim) {
        if (state >= t->decode_len) return ZO_ERR_REFERENCE_WOULD_PANIC;      /* empty table after a failed build */
        uint8_t sym = t->decode[state].symbol;                                /* decode_symbol :25-27 */
        if (bv_push(&sc->literals_buffer, &sym, 1)) return ZO_ERR_OUT_OF_MEMORY;
        uint8_t nb = t->decode[state].num_bits;                               /* next_state :41-53 */
        uint64_t nbits = brr_get_bits(&br, nb);
        state <<= nb; state &= (uint64_t)t->decode_len - 1; state |= nbits;
    }
    if (check_landing && brr_bits_remaining(&br) != lim) return ZO_ERR_LIT_BITSTREAM_READ_MISMATCH;
    return 0;
}
static int lit_decompress(const literals_section *sec, scratch *sc, const uint8_t *source, uint32_t *bytes_read_out) { /* decompress_literals :40-158 */
    if (!sec->has_compressed_size) return ZO_ERR_LIT_MISSING_COMPRESSED_SIZE;
    if (!sec->num_streams) return ZO_ERR_LIT_MISSING_NUM_STREAMS;
    size_t compressed_size = sec->compressed_size;
    uint32_t bytes_read = 0;
    if (sec->ls_type == 2) {
        uint32_t used = 0;
        int e = huf_build_decoder(&sc->huf, source, compressed_size, &used);
        if (e) return e;
        bytes_read += used;
    } else if (sec->ls_type == 3 && sc->huf.max_num_bits == 0) return ZO_ERR_LIT_UNINITIALIZED_HUFFMAN_TABLE;
    const uint8_t *src = source + bytes_read; size_t len = compressed_size - bytes_read;
    if (sec->num_streams == 4) {
        if (len < 6) return ZO_ERR_LIT_MISSING_BYTES_FOR_JUMP_HEADER;
        size_t jump1 = (size_t)src[0] + ((size_t)src[1] << 8);
        size_t jump2 = jump1 + (size_t)src[2] + ((size_t)src[3] << 8);
        size_t jump3 = jump2 + (size_t)src[4] + ((size_t)src[5] << 8);
        bytes_read += 6; src += 6; len -= 6;
        if (len < jump3) return ZO_ERR_LIT_MISSING_BYTES_FOR_LITERALS;
        const uint8_t *st[4] = {src, src + jump1, src + jump2, src + jump3};
        size_t sl[4] = {jump1, jump2 - jump1, jump3 - jump2, len - jump3};
        for (int i = 0; i < 4; i++) { int e = lit_decode_stream(sc, st[i], sl[i], 1); if (e) return e; }
        bytes_read += (uint32_t)len;
    } else {
        int e = lit_decode_stream(sc, src, len, 0); if (e) return e;
        bytes_read += (uint32_t)len;
    }
    if (sc->literals_buffer.len != sec->regenerated_size) return ZO_ERR_LIT_DECODED_LITERAL_COUNT_MISMATCH;
    *bytes_read_out = bytes_read;
    return 0;
}
static int lit_decode(const literals_section *sec, scratch *sc, const uint8_t *source, uint32_t *bytes_read) { /* decode_literals :12-34 */
    if (sec->ls_type == 0) { if (bv_push(&sc->literals_buffer, source, sec->regenerated_size)) return ZO_ERR_OUT_OF_MEMORY; *bytes_read = sec->regenerated_size; return 0; }
    if (sec->ls_type == 1) {
        if (bv_reserve(&sc->literals_buffer, sec->regenerated_size)) return ZO_ERR_OUT_OF_MEMORY;
        memset(sc->literals_buffer.p + sc->literals_buffer.len, source[0], sec->regenerated_size);
        sc->literals_buffer.len += sec->regenerated_size; *bytes_read = 1; return 0;
    }
    return lit_decompress(sec, sc, source, bytes_read);
}

/* ------------------------------------------------------------------ sequences (blocks/sequence_section.rs, decoding/sequence_section_decoder.rs) */
typedef struct { uint32_t num_sequences; int has_modes; uint8_t modes; } sequences_header;
static int seqhdr_parse(sequences_header *h, const uint8_t *src, size_t len, uint8_t *bytes_read) { /* parse_from_header :108-167 */
    h->num_sequences = 0; h->has_modes = 0; h->modes = 0;
    if (len == 0) return ZO_ERR_SEQHDR_NOT_ENOUGH_BYTES;
    uint8_t b0 = src[0];
    if (b0 == 0) { *bytes_read = 1; return 0; }
    if (b0 < 128) {
        if (len < 2) return ZO_ERR_SEQHDR_NOT_ENOUGH_BYTES;
        h->num_sequences = b0; h->has_modes = 1; h->modes = src[1]; *bytes_read = 2; return 0;
    }
    if (b0 < 255) {
        if (len < 2) return ZO_ERR_SEQHDR_NOT_ENOUGH_BYTES;
        h->num_sequences = (((uint32_t)b0 - 128) << 8) + src[1]; *bytes_read = 2;
        if (h->num_sequences != 0) { if (len < 3) return ZO_ERR_SEQHDR_NOT_ENOUGH_BYTES; h->has_modes = 1; h->modes = src[2]; *bytes_read = 3; }
        return 0;
    }
    if (len < 4) return ZO_ERR_SEQHDR_NOT_ENOUGH_BYTES;
    h->num_sequences = (uint32_t)src[1] + ((uint32_t)src[2] << 8) + 0x7F00; h->has_modes = 1; h->modes = src[3]; *bytes_read = 4;
    return 0;
}
static const int32_t LL_DEFAULT[36] = {4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1};  /* :418-421 */
static const int32_t ML_DEFAULT[53] = {1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1}; /* :429-432 */
static const int32_t OF_DEFAULT[29] = {1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1};           /* :440-442 */
static int lookup_ll_code(uint8_t code, uint32_t *value, uint8_t *bits) {                         /* :227-252 */
    static const uint32_t base[20] = {16,18,20,22,24,28,32,40,48,64,128,256,512,1024,2048,4096,8192,16384,32768,65536};
    static const uint8_t nb[20] = {1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16};
    if (code <= 15) { *value = code; *bits = 0; return 0; }
    if (code > 35) return ZO_ERR_REFERENCE_WOULD_PANIC;                                           /* unreachable! :250 */
    *value = base[code - 16]; *bits = nb[code - 16]; return 0;
}
static int lookup_ml_code(uint8_t code, uint32_t *value, uint8_t *bits) {                         /* :258-284 */
    static const uint32_t base[21] = {35,37,39,41,43,47,51,59,67,83,99,131,259,515,1027,2051,4099,8195,16387,32771,65539};
    static const uint8_t nb[21] = {1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16};
    if (code <= 31) { *value = (uint32_t)code + 3; *bits = 0; return 0; }
    if (code > 52) return ZO_ERR_REFERENCE_WOULD_PANIC;                                           /* unreachable! :282 */
    *value = base[code - 32]; *bits = nb[code - 32]; return 0;
}
/* one of the three arms of maybe_update_fse_tables :305-407 */
static int update_one_table(int mode, fse_table *t, int *rle, const uint8_t *src, size_t len, uint8_t max_log, uint8_t max_code,
                            const int32_t *def, size_t ndef, uint8_t def_log, int missing_byte_err, size_t *bytes) {
    *bytes = 0;
    switch (mode) {
    case 2: { int e = fse_build_decoder(t, src, len, max_log, bytes); if (e) return e; *rle = -1; return 0; }
    case 1:
        if (len == 0) return missing_byte_err;
        *bytes = 1;
        if (src[0] > max_code) return ZO_ERR_SEQ_MISSING_BYTE_FOR_RLE_ML_TABLE;                  /* sic: :321, :356, :391 */
        *rle = src[0]; return 0;
    case 0: { int e = fse_build_from_probabilities(t, def_log, def, ndef); if (e) return e; *rle = -1; return 0; }
    default: return 0;                                                                            /* Repeat: nothing to do */
    }
}
static int maybe_update_fse_tables(const sequences_header *h, const uint8_t *src, size_t len, scratch *sc, size_t *bytes_read) { /* :294-410 */
    if (!h->has_modes) return ZO_ERR_SEQ_MISSING_COMPRESSION_MODE;
    size_t used = 0, b; int e;
    if ((e = update_one_table(h->modes >> 6, &sc->literal_lengths, &sc->ll_rle, src, len, 9, MAX_LITERAL_LENGTH_CODE, LL_DEFAULT, 36, 6, ZO_ERR_SEQ_MISSING_BYTE_FOR_RLE_LL_TABLE, &b))) return e;
    used += b;
    if ((e = update_one_table((h->modes >> 4) & 3, &sc->offsets, &sc->of_rle, src + used, len - used, 8, MAX_OFFSET_CODE, OF_DEFAULT, 29, 5, ZO_ERR_SEQ_MISSING_BYTE_FOR_RLE_OF_TABLE, &b))) return e;
    used += b;
    if ((e = update_one_table((h->modes >> 2) & 3, &sc->match_lengths, &sc->ml_rle, src + used, len - used, 9, MAX_MATCH_LENGTH_CODE, ML_DEFAULT, 53, 6, ZO_ERR_SEQ_MISSING_BYTE_FOR_RLE_ML_TABLE, &b))) return e;
    used += b;
    *bytes_read = used;
    return 0;
}
/* decode_sequences :14-47 with both loops (:49-152 with RLE, :154-221 without) folded: an RLE'd component
 * substitutes its constant code and skips that decoder's init/update, exactly as the _with_rle variant does. */
static int decode_sequences(const sequences_header *h, const uint8_t *source, size_t len, scratch *sc) {
    size_t bytes_read = 0;
    int e = maybe_update_fse_tables(h, source, len, sc, &bytes_read);
    if (e) return e;
    /* fse build_decoder can report more bytes than the slice holds only via GetBitsError, so bytes_read <= len */
    brr br; brr_new(&br, source + bytes_read, len - bytes_read);
    int skipped = brr_skip_padding(&br);
    if (skipped > 8) return ZO_ERR_SEQ_EXTRA_PADDING;
    fse_decoder ll, ml, of; fsed_new(&ll, &sc->literal_lengths); fsed_new(&ml, &sc->match_lengths); fsed_new(&of, &sc->offsets);
    if (sc->ll_rle < 0 && (e = fsed_init_state(&ll, &br))) return e;
    if (sc->of_rle < 0 && (e = fsed_init_state(&of, &br))) return e;
    if (sc->ml_rle < 0 && (e = fsed_init_state(&ml, &br))) return e;
    sc->nseq = 0;
    if (sc->seq_cap < h->num_sequences) {
        sequence *np = (sequence *)realloc(sc->sequences, sizeof(sequence) * h->num_sequences);
        if (!np) return ZO_ERR_OUT_OF_MEMORY;
        sc->sequences = np; sc->seq_cap = h->num_sequences;
    }
    for (uint32_t i = 0; i < h->num_sequences; i++) {
        uint8_t ll_code = sc->ll_rle >= 0 ? (uint8_t)sc->ll_rle : ll.state.symbol;
        uint8_t ml_code = sc->ml_rle >= 0 ? (uint8_t)sc->ml_rle : ml.state.symbol;
        uint8_t of_code = sc->of_rle >= 0 ? (uint8_t)sc->of_rle : of.state.symbol;
        uint32_t ll_value, ml_value; uint8_t ll_bits, ml_bits;
        if ((e = lookup_ll_code(ll_code, &ll_value, &ll_bits))) return e;
        if ((e = lookup_ml_code(ml_code, &ml_value, &ml_bits))) return e;
        if (of_code > MAX_OFFSET_CODE) return ZO_ERR_SEQ_UNSUPPORTED_OFFSET;
        uint64_t obits, ml_add, ll_add;
        brr_get_bits_triple(&br, of_code, ml_bits, ll_bits, &obits, &ml_add, &ll_add);
        uint32_t offset = (uint32_t)obits + (1u << of_code);
        if (offset == 0) return ZO_ERR_SEQ_ZERO_OFFSET;
        sc->sequences[sc->nseq].ll = ll_value + (uint32_t)ll_add;
        sc->sequences[sc->nseq].ml = ml_value + (uint32_t)ml_add;
        sc->sequences[sc->nseq].of = offset;
        sc->nseq++;
        if (sc->nseq < h->num_sequences) {
            if (sc->ll_rle < 0 && fsed_update_state(&ll, &br)) return ZO_ERR_REFERENCE_WOULD_PANIC;
            if (sc->ml_rle < 0 && fsed_update_state(&ml, &br)) return ZO_ERR_REFERENCE_WOULD_PANIC;
            if (sc->of_rle < 0 && fsed_update_state(&of, &br)) return ZO_ERR_REFERENCE_WOULD_PANIC;
        }
        if (brr_bits_remaining(&br) < 0) return ZO_ERR_SEQ_NOT_ENOUGH_BYTES_FOR_NUM_SEQUENCES;
    }
    if (brr_bits_remaining(&br) > 0) return ZO_ERR_SEQ_EXTRA_BITS;
    return 0;
}

/* ------------------------------------------------------------------ sequence execution (decoding/sequence_execution.rs) */
static uint32_t do_offset_history(uint32_t offset_value, uint32_t lit_len, uint32_t scratch_[3]) { /* :59-118 */
    uint32_t actual;
    if (lit_len > 0) {
        if (offset_value >= 1 && offset_value <= 3) actual = scratch_[offset_value - 1]; else actual = offset_value - 3;
    } else {
        if (offset_value == 1 || offset_value == 2) actual = scratch_[offset_value];
        else if (offset_value == 3) actual = scratch_[0] ? scratch_[0] - 1 : 0;                    /* saturating_sub */
        else actual = offset_value - 3;
    }
    if (lit_len > 0) {
        if (offset_value == 1) { /* nothing */ }
        else if (offset_value == 2) { scratch_[1] = scratch_[0]; scratch_[0] = actual; }
        else { scratch_[2] = scratch_[1]; scratch_[1] = scratch_[0]; scratch_[0] = actual; }
    } else {
        if (offset_value == 1) { scratch_[1] = scratch_[0]; scratch_[0] = actual; }
        else { scratch_[2] = scratch_[1]; scratch_[1] = scratch_[0]; scratch_[0] = actual; }
    }
    return actual;
}
uint32_t zo_kat_do_offset_history(uint32_t offset_value, uint32_t lit_len, uint32_t hist[3]) { return do_offset_history(offset_value, lit_len, hist); }

static int trace_push_seq(zo_decoder *d, const sequence *s, uint32_t actual) {
    if (d->ntseq == d->tseq_cap) {
        size_t nc = d->tseq_cap ? d->tseq_cap * 2 : 4096;
        zo_seq_trace *np = (zo_seq_trace *)realloc(d->tseq, nc * sizeof *np);
        if (!np) return ZO_ERR_OUT_OF_MEMORY;
        d->tseq = np; d->tseq_cap = nc;
    }
    d->tseq[d->ntseq].ll = s->ll; d->tseq[d->ntseq].ml = s->ml; d->tseq[d->ntseq].of = s->of; d->tseq[d->ntseq].actual_offset = actual;
    d->ntseq++;
    return 0;
}
static int execute_sequences(zo_decoder *d) {                                                     /* :5-54 */
    scratch *sc = &d->sc;
    size_t literals_copy_counter = 0;
    size_t old_buffer_size = db_len(&sc->buffer);
    uint64_t seq_sum = 0;
    for (size_t idx = 0; idx < sc->nseq; idx++) {
        sequence seq = sc->sequences[idx];
        if (seq.ll > 0) {
            size_t high = literals_copy_counter + seq.ll;
            if (high > sc->literals_buffer.len) return ZO_ERR_EXEC_NOT_ENOUGH_BYTES_FOR_SEQUENCE;
            int e = db_push(&sc->buffer, sc->literals_buffer.p + literals_copy_counter, seq.ll); if (e) return e;
            literals_copy_counter += seq.ll;
        }
        uint32_t actual = do_offset_history(seq.of, seq.ll, sc->offset_hist);
        if (d->trace_on) { int e = trace_push_seq(d, &seq, actual); if (e) return e; }
        if (actual == 0) return ZO_ERR_EXEC_ZERO_OFFSET;
        if (seq.ml > 0) { int e = db_repeat(&sc->buffer, actual, seq.ml); if (e) return e; }
        seq_sum += seq.ml; seq_sum += seq.ll;
        if (seq_sum > 0x7fffffffULL) return ZO_ERR_BLOCK_OUTPUT_LIMIT;   /* u32 seq_sum would wrap -> assert :47 panics */
    }
    if (literals_copy_counter < sc->literals_buffer.len) {
        size_t rest = sc->literals_buffer.len - literals_copy_counter;
        int e = db_push(&sc->buffer, sc->literals_buffer.p + literals_copy_counter, rest); if (e) return e;
        seq_sum += rest;
    }
    if (seq_sum != db_len(&sc->buffer) - old_buffer_size) return ZO_ERR_REFERENCE_WOULD_PANIC;    /* assert :47-52 */
    return 0;
}

/* ------------------------------------------------------------------ block decoder (decoding/block_decoder.rs) */
typedef struct { int last_block; int block_type; uint32_t decompressed_size, content_size; } block_header;
static int read_block_header(zo_read_fn rd, void *user, block_header *h) {                        /* :201-247 */
    uint8_t b[3];
    if (read_exact(rd, user, b, 3)) return ZO_ERR_BLOCK_HEADER_READ;
    int t = (b[0] >> 1) & 3;                                                                      /* :259-268 */
    if (t == 3) return ZO_ERR_FOUND_RESERVED_BLOCK;
    uint32_t size = (uint32_t)(b[0] >> 3) | ((uint32_t)b[1] << 5) | ((uint32_t)b[2] << 13);      /* :279-283 */
    if (size > MAX_BLOCK_SIZE) return ZO_ERR_BLOCK_SIZE_TOO_LARGE;                                /* :270-277 */
    h->block_type = t;
    h->decompressed_size = (t == 0 || t == 1) ? size : 0;
    h->content_size = (t == 1) ? 1 : size;
    h->last_block = b[0] & 1;
    return 0;
}
static int trace_begin_block(zo_decoder *d, int block_type) {
    if (!d->trace_on) return 0;
    if (d->ntb == d->tb_cap) {
        size_t nc = d->tb_cap ? d->tb_cap * 2 : 256;
        zo_block_trace *np = (zo_block_trace *)realloc(d->tb, nc * sizeof *np);
        if (!np) return ZO_ERR_OUT_OF_MEMORY;
        d->tb = np; d->tb_cap = nc;
    }
    zo_block_trace *t = &d->tb[d->ntb++];
    memset(t, 0, sizeof *t);
    t->block_type = (uint32_t)block_type; t->lit_offset = d->tlits.len; t->seq_offset = d->ntseq; t->out_offset = d->trace_out_pos;
    return 0;
}
static void trace_end_block(zo_decoder *d, size_t out_before) {
    if (!d->trace_on) return;
    zo_block_trace *t = &d->tb[d->ntb - 1];
    t->out_size = db_len(&d->sc.buffer) - out_before;
    d->trace_out_pos += t->out_size;
    memcpy(t->offset_hist_after, d->sc.offset_hist, sizeof t->offset_hist_after);
}
static int decompress_block(zo_decoder *d, const block_header *h, zo_read_fn rd, void *user) {    /* :97-197 */
    scratch *sc = &d->sc;
    sc->block_content_buffer.len = 0;
    if (bv_reserve(&sc->block_content_buffer, h->content_size)) return ZO_ERR_OUT_OF_MEMORY;
    sc->block_content_buffer.len = h->content_size;
    d->last_stage = ZO_STAGE_BLOCK_BODY;
    if (read_exact(rd, user, sc->block_content_buffer.p, h->content_size)) return ZO_ERR_BLOCK_CONTENT_READ;
    const uint8_t *raw = sc->block_content_buffer.p; size_t raw_len = h->content_size;
    literals_section section; uint8_t lit_hdr = 0;
    int e = litsec_parse(&section, raw, raw_len, &lit_hdr);
    if (e) return e;
    raw += lit_hdr; raw_len -= lit_hdr;
    size_t upper = section.has_compressed_size ? section.compressed_size : (section.ls_type == 1 ? 1 : section.regenerated_size);
    if (raw_len < upper) return ZO_ERR_MALFORMED_SECTION_HEADER;
    sc->literals_buffer.len = 0;
    uint32_t bytes_used = 0;
    d->last_stage = ZO_STAGE_LITERALS;
    if ((e = lit_decode(&section, sc, raw, &bytes_used))) return e;
    if (section.regenerated_size != sc->literals_buffer.len) return ZO_ERR_REFERENCE_WOULD_PANIC; /* assert :146 */
    if (bytes_used != upper) return ZO_ERR_REFERENCE_WOULD_PANIC;                                  /* assert :152 */
    raw += upper; raw_len -= upper;
    d->last_stage = ZO_STAGE_BLOCK_BODY;
    sequences_header sh; uint8_t seq_hdr = 0;
    if ((e = seqhdr_parse(&sh, raw, raw_len, &seq_hdr))) return e;
    raw += seq_hdr; raw_len -= seq_hdr;
    if (d->trace_on) {
        zo_block_trace *t = &d->tb[d->ntb - 1];
        t->literals_type = (uint32_t)section.ls_type; t->num_streams = (uint32_t)section.num_streams;
        t->regenerated_size = section.regenerated_size; t->num_sequences = sh.num_sequences; t->huf_max_bits = sc->huf.max_num_bits;
        if (bv_push(&d->tlits, sc->literals_buffer.p, sc->literals_buffer.len)) return ZO_ERR_OUT_OF_MEMORY;
    }
    if (sh.num_sequences != 0) {
        d->last_stage = ZO_STAGE_SEQUENCES;
        if ((e = decode_sequences(&sh, raw, raw_len, sc))) return e;
        d->last_stage = ZO_STAGE_EXECUTE;
        if ((e = execute_sequences(d))) return e;
    } else {
        if (raw_len != 0) { d->last_stage = ZO_STAGE_SEQUENCES; return ZO_ERR_SEQ_EXTRA_BITS; }    /* :185-191 */
        if ((e = db_push(&sc->buffer, sc->literals_buffer.p, sc->literals_buffer.len))) return e;
        sc->nseq = 0;
    }
    return 0;
}
static int decode_block_content(zo_decoder *d, const block_header *h, zo_read_fn rd, void *user, uint64_t *bytes_read) { /* :39-95 */
    scratch *sc = &d->sc;
    size_t out_before = db_len(&sc->buffer);
    int e = trace_begin_block(d, h->block_type); if (e) return e;
    d->last_stage = ZO_STAGE_BLOCK_BODY;
    if (h->block_type == 1) {
        uint8_t b;
        if (read_exact(rd, user, &b, 1)) return ZO_ERR_BLOCK_BODY_READ;
        if (bv_reserve(&sc->buffer.buf, h->decompressed_size)) return ZO_ERR_OUT_OF_MEMORY;       /* extend_and_fill :62-64 */
        memset(sc->buffer.buf.p + sc->buffer.buf.len, b, h->decompressed_size); sc->buffer.buf.len += h->decompressed_size;
        *bytes_read = 1;
    } else if (h->block_type == 0) {
        if (bv_reserve(&sc->buffer.buf, h->decompressed_size)) return ZO_ERR_OUT_OF_MEMORY;       /* extend_from_reader :66-72 */
        if (read_exact(rd, user, sc->buffer.buf.p + sc->buffer.buf.len, h->decompressed_size)) return ZO_ERR_BLOCK_BODY_READ;
        sc->buffer.buf.len += h->decompressed_size;
        *bytes_read = h->decompressed_size;
    } else {
        if ((e = decompress_block(d, h, rd, user))) return e;
        *bytes_read = h->content_size;
    }
    trace_end_block(d, out_before);
    return 0;
}

/* ------------------------------------------------------------------ dictionary (decoding/dictionary.rs) */
static void dict_free(dictionary *x) { if (x) { bv_free(&x->content); free(x); } }
static int dict_decode(const uint8_t *raw, size_t len, dictionary **out) {                        /* decode_dict :45-126 */
    if (len < 8) return ZO_ERR_DICT_NOT_ENOUGH_BYTES;
    dictionary *x = (dictionary *)calloc(1, sizeof *x);
    if (!x) return ZO_ERR_OUT_OF_MEMORY;
    fse_new(&x->of, MAX_OFFSET_CODE); fse_new(&x->ll, MAX_LITERAL_LENGTH_CODE); fse_new(&x->ml, MAX_MATCH_LENGTH_CODE);
    x->of_rle = x->ml_rle = x->ll_rle = -1; huf_new(&x->huf);
    x->offset_hist[0] = 2; x->offset_hist[1] = 4; x->offset_hist[2] = 8;
    static const uint8_t magic[4] = {0x37, 0xA4, 0x30, 0xEC};
    int e = 0;
    if (memcmp(raw, magic, 4)) { e = ZO_ERR_DICT_BAD_MAGIC_NUM; goto fail; }
    x->id = rd32(raw + 4);
    const uint8_t *t = raw + 8; size_t tl = len - 8;
    uint32_t huf_size = 0; size_t n;
    if ((e = huf_build_decoder(&x->huf, t, tl, &huf_size))) goto fail;
    if (tl < huf_size) { e = ZO_ERR_DICT_NOT_ENOUGH_BYTES; goto fail; }
    t += huf_size; tl -= huf_size;
    if ((e = fse_build_decoder(&x->of, t, tl, 8, &n))) goto fail;
    if (tl < n) { e = ZO_ERR_DICT_NOT_ENOUGH_BYTES; goto fail; }
    t += n; tl -= n;
    if ((e = fse_build_decoder(&x->ml, t, tl, 9, &n))) goto fail;
    if (tl < n) { e = ZO_ERR_DICT_NOT_ENOUGH_BYTES; goto fail; }
    t += n; tl -= n;
    if ((e = fse_build_decoder(&x->ll, t, tl, 9, &n))) goto fail;
    if (tl < n) { e = ZO_ERR_DICT_NOT_ENOUGH_BYTES; goto fail; }
    t += n; tl -= n;
    if (tl < 12) { e = ZO_ERR_DICT_NOT_ENOUGH_BYTES; goto fail; }
    x->offset_hist[0] = rd32(t); x->offset_hist[1] = rd32(t + 4); x->offset_hist[2] = rd32(t + 8);
    if (bv_push(&x->content, t + 12, tl - 12)) { e = ZO_ERR_OUT_OF_MEMORY; goto fail; }
    *out = x;
    return 0;
fail:
    dict_free(x);
    return e;
}
int zo_kat_decode_dict(const uint8_t *raw, size_t len, uint32_t *id, uint32_t offs[3], size_t *content_len) {
    dictionary *x = NULL; int e = dict_decode(raw, len, &x);
    if (e) return e;
    *id = x->id; memcpy(offs, x->offset_hist, 12); *content_len = x->content.len;
    dict_free(x); return 0;
}
static int dict_insert(zo_decoder *d, dictionary *x) {                                            /* add_dict frame_decoder.rs:224-227 (BTreeMap insert replaces) */
    for (size_t i = 0; i < d->ndicts; i++) if (d->dicts[i]->id == x->id) { dict_free(d->dicts[i]); d->dicts[i] = x; return 0; }
    dictionary **np = (dictionary **)realloc(d->dicts, sizeof(*np) * (d->ndicts + 1));
    if (!np) return ZO_ERR_OUT_OF_MEMORY;
    d->dicts = np; d->dicts[d->ndicts++] = x; return 0;
}
static dictionary *dict_find(zo_decoder *d, uint32_t id) { for (size_t i = 0; i < d->ndicts; i++) if (d->dicts[i]->id == id) return d->dicts[i]; return NULL; }

/* ------------------------------------------------------------------ FrameDecoder (decoding/frame_decoder.rs) */
zo_decoder *zo_new(void) {                                                                        /* :158-164 */
    zo_decoder *d = (zo_decoder *)calloc(1, sizeof *d);
    if (!d) return NULL;
    d->max_window_size = DEFAULT_MAX_WINDOW_SIZE;
    scratch_init(&d->sc, 0);
    return d;
}
void zo_free(zo_decoder *d) {
    if (!d) return;
    bv_free(&d->sc.buffer.buf); bv_free(&d->sc.buffer.dict_content); bv_free(&d->sc.literals_buffer); bv_free(&d->sc.block_content_buffer);
    free(d->sc.sequences);
    for (size_t i = 0; i < d->ndicts; i++) dict_free(d->dicts[i]);
    free(d->dicts); free(d->tb); free(d->tseq); bv_free(&d->tlits);
    free(d);
}
void zo_set_max_window_size(zo_decoder *d, uint64_t m) { d->max_window_size = m < MAX_WINDOW_SIZE ? m : MAX_WINDOW_SIZE; } /* :175-177 */
uint64_t zo_max_window_size(const zo_decoder *d) { return d->max_window_size; }
int zo_last_error_stage(const zo_decoder *d) { return d->last_stage; }

int zo_init(zo_decoder *d, zo_read_fn rd, void *user) {                                           /* reset :200-221, FrameDecoderState::new/reset :103-134 */
    d->last_stage = ZO_STAGE_FRAME_HEADER;
    /* the reference parses into a fresh header first; on failure an existing state keeps its old header but
     * nothing observable depends on that except getters -- we keep the old values by parsing into a copy */
    zo_decoder tmp; memset(&tmp, 0, sizeof tmp);
    uint8_t header_size = 0;
    int e = frame_read_header(&tmp, rd, user, &header_size);
    if (e) { d->skip_length = tmp.skip_length; return e; }
    uint64_t window_size = 0;
    if ((e = frame_window_size(&tmp, &window_size))) return e;
    if (window_size > d->max_window_size) return ZO_ERR_WINDOW_SIZE_TOO_BIG;                      /* check_window_size :137-145 */
    d->descriptor = tmp.descriptor; d->window_descriptor = tmp.window_descriptor; d->has_dict_id = tmp.has_dict_id;
    d->dict_id = tmp.dict_id; d->frame_content_size = tmp.frame_content_size;
    d->frame_finished = 0; d->block_counter = 0;
    scratch_reset(&d->sc, (size_t)window_size);
    d->bytes_read_counter = header_size; d->has_check_sum = 0; d->using_dict = 0;
    d->has_state = 1;
    if (d->has_dict_id) {                                                                          /* :212-219 */
        dictionary *x = dict_find(d, d->dict_id);
        if (!x) return ZO_ERR_DICT_NOT_PROVIDED;
        if ((e = scratch_init_from_dict(&d->sc, x))) return e;
        d->using_dict = 1; d->using_dict_id = d->dict_id;
    }
    d->last_stage = ZO_STAGE_NONE;
    return 0;
}
int zo_add_dict(zo_decoder *d, const uint8_t *raw, size_t len) {
    dictionary *x = NULL; d->last_stage = ZO_STAGE_DICTIONARY;
    int e = dict_decode(raw, len, &x); if (e) return e;
    return dict_insert(d, x);
}
int zo_add_raw_content_dict(zo_decoder *d, uint32_t id, const uint8_t *content, size_t len) {     /* extension, see header */
    dictionary *x = (dictionary *)calloc(1, sizeof *x);
    if (!x) return ZO_ERR_OUT_OF_MEMORY;
    fse_new(&x->of, MAX_OFFSET_CODE); fse_new(&x->ll, MAX_LITERAL_LENGTH_CODE); fse_new(&x->ml, MAX_MATCH_LENGTH_CODE);
    x->of_rle = x->ml_rle = x->ll_rle = -1; huf_new(&x->huf);
    x->id = id; x->offset_hist[0] = 1; x->offset_hist[1] = 4; x->offset_hist[2] = 8;
    if (bv_push(&x->content, content, len)) { dict_free(x); return ZO_ERR_OUT_OF_MEMORY; }
    return dict_insert(d, x);
}
int zo_force_dict(zo_decoder *d, uint32_t dict_id) {                                              /* :229-243 */
    if (!d->has_state) return ZO_ERR_NOT_YET_INITIALIZED;
    dictionary *x = dict_find(d, dict_id);
    if (!x) return ZO_ERR_DICT_NOT_PROVIDED;
    int e = scratch_init_from_dict(&d->sc, x); if (e) return e;
    d->using_dict = 1; d->using_dict_id = dict_id;
    return 0;
}
uint64_t zo_content_size(const zo_decoder *d) { return d->has_state ? d->frame_content_size : 0; }                 /* :246-251 */
int zo_get_checksum_from_data(const zo_decoder *d, uint32_t *out) { if (!d->has_state || !d->has_check_sum) return 0; *out = d->check_sum; return 1; } /* :254-258 */
int zo_get_calculated_checksum(const zo_decoder *d, uint32_t *out) { if (!d->has_state) return 0; *out = (uint32_t)xxh64_digest(&d->sc.buffer.hash); return 1; } /* :262-270 */
uint64_t zo_bytes_read_from_source(const zo_decoder *d) { return d->has_state ? d->bytes_read_counter : 0; }        /* :273-279 */
int zo_is_finished(const zo_decoder *d) {                                                         /* :284-294 */
    if (!d->has_state) return 1;
    if ((d->descriptor >> 2) & 1) return d->frame_finished && d->has_check_sum;
    return d->frame_finished;
}
size_t zo_blocks_decoded(const zo_decoder *d) { return d->has_state ? d->block_counter : 0; }     /* :297-303 */
uint64_t zo_window_size(const zo_decoder *d) { return d->has_state ? d->sc.buffer.window_size : 0; }
int zo_frame_dict_id(const zo_decoder *d, uint32_t *out) { if (!d->has_state || !d->has_dict_id) return 0; *out = d->dict_id; return 1; }

int zo_decode_blocks(zo_decoder *d, zo_read_fn rd, void *user, int strategy, size_t n, int *finished) { /* :309-377 */
    if (!d->has_state) return ZO_ERR_NOT_YET_INITIALIZED;
    size_t buffer_size_before = db_len(&d->sc.buffer), block_counter_before = d->block_counter;
    for (;;) {
        block_header h; int e;
        d->last_stage = ZO_STAGE_BLOCK_HEADER;
        if ((e = read_block_header(rd, user, &h))) return e;
        d->bytes_read_counter += 3;
        uint64_t body = 0;
        if ((e = decode_block_content(d, &h, rd, user, &body))) return e;
        d->bytes_read_counter += body;
        d->block_counter++;
        if (h.last_block) {
            d->frame_finished = 1;
            if ((d->descriptor >> 2) & 1) {
                uint8_t c[4]; d->last_stage = ZO_STAGE_CHECKSUM;
                if (read_exact(rd, user, c, 4)) return ZO_ERR_FAILED_TO_READ_CHECKSUM;
                d->bytes_read_counter += 4; d->check_sum = rd32(c); d->has_check_sum = 1;
            }
            break;
        }
        if (strategy == ZO_STRATEGY_UPTO_BLOCKS) { if (d->block_counter - block_counter_before >= n) break; }
        else if (strategy == ZO_STRATEGY_UPTO_BYTES) { if (db_len(&d->sc.buffer) - buffer_size_before >= n) break; }
    }
    d->last_stage = ZO_STAGE_NONE;
    if (finished) *finished = d->frame_finished;
    return 0;
}
long zo_read(zo_decoder *d, uint8_t *target, size_t len) {                                        /* impl Read :615-627 */
    if (!d->has_state) return 0;
    decode_buffer *b = &d->sc.buffer;
    size_t amount;
    if (d->frame_finished) amount = db_len(b) < len ? db_len(b) : len;                            /* read_all decode_buffer.rs:241-251 */
    else { size_t mx = 0; if (!db_can_drain_to_window_size(b, &mx)) mx = 0; amount = mx < len ? mx : len; } /* read decode_buffer.rs:19-32 */
    if (amount == 0) return 0;
    return db_drain_to(b, amount, NULL, NULL, target);
}
long zo_collect_to_writer(zo_decoder *d, zo_write_fn wr, void *user) {                            /* :393-404 */
    if (!d->has_state) return 0;
    decode_buffer *b = &d->sc.buffer;
    if (zo_is_finished(d)) return db_drain_to(b, db_len(b), wr, user, NULL);                      /* drain_to_writer decode_buffer.rs:236-239 */
    size_t n = 0; if (!db_can_drain_to_window_size(b, &n)) return 0;                              /* :213-218 */
    return db_drain_to(b, n, wr, user, NULL);
}
size_t zo_can_collect(const zo_decoder *d) {                                                      /* :409-424 */
    if (!d->has_state) return 0;
    if (zo_is_finished(d)) return db_len(&d->sc.buffer);
    size_t n = 0; if (db_can_drain_to_window_size(&d->sc.buffer, &n)) return n; return 0;
}
int zo_decode_from_to(zo_decoder *d, const uint8_t *src, size_t src_len, uint8_t *dst, size_t dst_len, size_t *read, size_t *written) { /* :439-529 */
    uint64_t bytes_read_at_start = d->has_state ? d->bytes_read_counter : 0;
    if (!zo_is_finished(d) || !d->has_state) {
        slice_reader mt = {src, src_len};
        if (!d->has_state) { int e = zo_init(d, slice_read, &mt); if (e) return e; }
        if (((d->descriptor >> 2) & 1) && d->frame_finished && !d->has_check_sum) {               /* :465-477 */
            if (mt.len >= 4) { d->bytes_read_counter += 4; d->check_sum = rd32(mt.p); d->has_check_sum = 1; }
            *read = 4; *written = 0; return 0;
        }
        for (;;) {
            if (mt.len < 3) break;
            block_header h; int e;
            d->last_stage = ZO_STAGE_BLOCK_HEADER;
            if ((e = read_block_header(slice_read, &mt, &h))) return e;
            if (mt.len < h.content_size) break;
            d->bytes_read_counter += 3;
            uint64_t body = 0;
            if ((e = decode_block_content(d, &h, slice_read, &mt, &body))) return e;
            d->bytes_read_counter += body; d->block_counter++;
            if (h.last_block) {
                d->frame_finished = 1;
                if ((d->descriptor >> 2) & 1) { if (mt.len >= 4) { d->bytes_read_counter += 4; d->check_sum = rd32(mt.p); d->has_check_sum = 1; } }
                break;
            }
        }
    }
    long r = zo_read(d, dst, dst_len);
    if (r < 0) { d->last_stage = ZO_STAGE_DRAIN; return ZO_ERR_FAILED_TO_DRAIN_DECODEBUFFER; }
    *written = (size_t)r;
    *read = (size_t)(d->bytes_read_counter - bytes_read_at_start);
    d->last_stage = ZO_STAGE_NONE;
    return 0;
}
int zo_decode_all(zo_decoder *d, const uint8_t *input, size_t in_len, uint8_t *output, size_t out_cap, size_t *written) { /* :541-577 */
    slice_reader in = {input, in_len};
    size_t total = 0;
    while (in.len != 0) {
        int e = zo_init(d, slice_read, &in);
        if (e == ZO_ERR_SKIP_FRAME) {
            if ((size_t)d->skip_length > in.len) return ZO_ERR_FAILED_TO_SKIP_FRAME;
            in.p += d->skip_length; in.len -= d->skip_length; continue;
        }
        if (e) return e;
        for (;;) {
            if ((e = zo_decode_blocks(d, slice_read, &in, ZO_STRATEGY_UPTO_BYTES, 1024 * 1024, NULL))) return e;
            long w = zo_read(d, output + total, out_cap - total);
            if (w < 0) return ZO_ERR_FAILED_TO_DRAIN_DECODEBUFFER;
            total += (size_t)w;
            if (zo_can_collect(d) != 0) return ZO_ERR_TARGET_TOO_SMALL;
            if (zo_is_finished(d)) break;
        }
    }
    *written = total;
    return 0;
}

/* ------------------------------------------------------------------ trace accessors */
void zo_trace_enable(zo_decoder *d, int on) { d->trace_on = on; d->ntb = 0; d->ntseq = 0; d->tlits.len = 0; d->trace_out_pos = 0; }
size_t zo_trace_num_blocks(const zo_decoder *d) { return d->ntb; }
const zo_block_trace *zo_trace_blocks(const zo_decoder *d) { return d->tb; }
const uint8_t *zo_trace_literals(const zo_decoder *d, size_t *len) { *len = d->tlits.len; return d->tlits.p; }
const zo_seq_trace *zo_trace_sequences(const zo_decoder *d, size_t *count) { *count = d->ntseq; return d->tseq; }

/* ------------------------------------------------------------------ KAT entry points */
long zo_kat_bitreader_reversed(const uint8_t *src, size_t len, const uint8_t *counts, size_t n, uint64_t *values) {
    brr r; brr_new(&r, src, len);
    for (size_t i = 0; i < n; i++) values[i] = brr_get_bits(&r, counts[i]);
    return brr_bits_remaining(&r);
}
int zo_kat_bitreader_forward(const uint8_t *src, size_t len, const uint8_t *counts, size_t n, uint64_t *values) {
    bitreader b = {0, src, len};
    for (size_t i = 0; i < n; i++) if (br_get_bits(&b, counts[i], &values[i])) return -1;
    return 0;
}
static void export_fse(const fse_table *t, uint32_t *entries3) {
    for (size_t i = 0; i < t->decode_len; i++) { entries3[3 * i] = t->decode[i].base_line; entries3[3 * i + 1] = t->decode[i].num_bits; entries3[3 * i + 2] = t->decode[i].symbol; }
}
int zo_kat_fse_build(const int32_t *probs, size_t nprobs, uint8_t acc_log, uint8_t max_symbol, uint32_t *entries3) {
    fse_table t; fse_new(&t, max_symbol);
    int e = fse_build_from_probabilities(&t, acc_log, probs, nprobs); if (e) return e;
    export_fse(&t, entries3); return 0;
}
long zo_kat_fse_read(const uint8_t *src, size_t len, uint8_t max_log, uint8_t max_symbol, uint8_t *acc_log, uint32_t *entries3, size_t cap) {
    fse_table t; fse_new(&t, max_symbol); size_t used = 0;
    int e = fse_build_decoder(&t, src, len, max_log, &used); if (e) return -(long)e;
    if (t.decode_len > cap) return -(long)ZO_ERR_INVALID_ARGUMENT;
    *acc_log = t.accuracy_log; export_fse(&t, entries3); return (long)used;
}
long zo_kat_huf_build(const uint8_t *src, size_t len, uint8_t *max_bits, uint16_t *entries, size_t cap) {
    huf_table *h = (huf_table *)malloc(sizeof *h); if (!h) return -(long)ZO_ERR_OUT_OF_MEMORY;
    huf_new(h); uint32_t used = 0;
    int e = huf_build_decoder(h, src, len, &used);
    if (e) { free(h); return -(long)e; }
    if (h->decode_len > cap) { free(h); return -(long)ZO_ERR_INVALID_ARGUMENT; }
    *max_bits = h->max_num_bits;
    for (size_t i = 0; i < h->decode_len; i++) entries[i] = (uint16_t)(h->decode[i].symbol | (h->decode[i].num_bits << 8));
    free(h); return (long)used;
}

/* ------------------------------------------------------------------ bulk decode for the CPU baseline */
typedef struct {
    const uint8_t *input; const uint64_t *in_off, *in_sz; size_t nframes; uint8_t *output; const uint64_t *out_off, *out_cap; uint64_t *out_sz;
    const uint8_t *raw_dict; size_t raw_dict_len; int tid, nthreads; int err;
} bulk_job;
static void *bulk_worker(void *arg) {
    bulk_job *j = (bulk_job *)arg;
    zo_decoder *d = zo_new();
    if (!d) { j->err = ZO_ERR_OUT_OF_MEMORY; return NULL; }
    if (j->raw_dict) { int e = zo_add_raw_content_dict(d, 1, j->raw_dict, j->raw_dict_len); if (e) { j->err = e; zo_free(d); return NULL; } }
    size_t lo = j->nframes * (size_t)j->tid / (size_t)j->nthreads, hi = j->nframes * (size_t)(j->tid + 1) / (size_t)j->nthreads;
    for (size_t i = lo; i < hi; i++) {
        /* FrameDecoder::reset + (force_dict) + decode_blocks(All) + read: the loop in tests/decode_corpus.rs:76-100 */
        slice_reader in = {j->input + j->in_off[i], (size_t)j->in_sz[i]};
        int e = zo_init(d, slice_read, &in);
        if (!e && j->raw_dict) e = zo_force_dict(d, 1);
        if (!e) e = zo_decode_blocks(d, slice_read, &in, ZO_STRATEGY_ALL, 0, NULL);
        if (e) { j->err = e; break; }
        size_t got = 0;
        for (;;) {
            long w = zo_read(d, j->output + j->out_off[i] + got, (size_t)j->out_cap[i] - got);
            if (w <= 0) break;
            got += (size_t)w;
        }
        if (zo_can_collect(d) != 0) { j->err = ZO_ERR_TARGET_TOO_SMALL; break; }
        j->out_sz[i] = got;
    }
    zo_free(d);
    return NULL;
}
int zo_bulk_decode(const uint8_t *input, const uint64_t *in_offsets, const uint64_t *in_sizes, size_t nframes, uint8_t *output,
                   const uint64_t *out_offsets, const uint64_t *out_caps, uint64_t *out_sizes, const uint8_t *raw_dict, size_t raw_dict_len, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if ((size_t)nthreads > nframes && nframes > 0) nthreads = (int)nframes;
    bulk_job *jobs = (bulk_job *)calloc((size_t)nthreads, sizeof *jobs);
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof *th);
    if (!jobs || !th) { free(jobs); free(th); return ZO_ERR_OUT_OF_MEMORY; }
    for (int t = 0; t < nthreads; t++) {
        bulk_job j = {input, in_offsets, in_sizes, nframes, output, out_offsets, out_caps, out_sizes, raw_dict, raw_dict_len, t, nthreads, 0};
        jobs[t] = j;
        if (nthreads == 1) bulk_worker(&jobs[t]); else pthread_create(&th[t], NULL, bulk_worker, &jobs[t]);
    }
    int err = 0;
    for (int t = 0; t < nthreads; t++) { if (nthreads > 1) pthread_join(th[t], NULL); if (jobs[t].err && !err) err = jobs[t].err; }
    free(jobs); free(th);
    return err;
}
