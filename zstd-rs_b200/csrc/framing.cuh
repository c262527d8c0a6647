// framing.cuh -- the fixed-size zstd headers, compiled for BOTH device and host.
//
// The host planner parses them on host input (plan_batch, the block-level entry, the frame decoder) and k_walk parses them on
// device-resident input, with this one code.  What they must produce is defined by the reference:
//   read_frame_header        ruzstd/src/decoding/frame.rs:6-85, window_size :116-139
//   read_block_header        ruzstd/src/decoding/block_decoder.rs:201-283
//   LiteralsSection::parse   ruzstd/src/blocks/literals_section.rs:117-223
//   SequencesHeader::parse   ruzstd/src/blocks/sequence_section.rs:108-167
// Table descriptions and bitstreams are parsed by the kernels (tables.cuh, kernels.cu).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/b200zstd.h"
#include "b200z_types.h"

namespace b200z {

B200Z_HD uint32_t rd32le(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

// ---- frame header
constexpr uint32_t ZSTD_MAGIC = 0xFD2FB528u;
B200Z_HD bool skippable_magic(uint32_t magic) { return magic >= 0x184D2A50u && magic <= 0x184D2A5Fu; }

struct FrameHeader {
    uint8_t descriptor = 0, window_descriptor = 0;
    bool has_dict_id = false;
    uint32_t dict_id = 0;
    uint64_t frame_content_size = 0;
    uint8_t header_size = 0;
    B200Z_HD bool single_segment() const { return (descriptor >> 5) & 1; }
    B200Z_HD bool content_checksum() const { return (descriptor >> 2) & 1; }
};

// Bytes of a frame header (magic number included) whose descriptor byte is `desc`: magic, descriptor, window descriptor unless
// single-segment, dictionary id (0, 1, 2 or 4 bytes), frame content size (0 or 1, 2, 4, 8 bytes).
B200Z_HD uint32_t frame_header_length(uint32_t desc) {
    const uint32_t single = (desc >> 5) & 1u, flag = desc >> 6;
    const uint32_t did_len = (1u << (desc & 3u)) >> 1, fcs_len = flag ? 1u << flag : single;
    return 6u - single + did_len + fcs_len;
}

// How far to read before parse_frame_header can decide, given the `have` bytes at p: the magic number, then 4 more bytes of a
// skippable frame or the descriptor byte, then the whole header.  Equal to `have` once nothing more is needed.
B200Z_HD size_t frame_header_want(const uint8_t *p, size_t have) {
    if (have < 4) return 4;
    const uint32_t magic = rd32le(p);
    if (skippable_magic(magic)) return 8;
    if (magic != ZSTD_MAGIC) return 4;
    return have < 5 ? 5 : frame_header_length(p[4]);
}

// Parses a frame header from p[0..len).  Returns 0, B200Z_ERR_SKIP_FRAME (skip_len set, 8 bytes consumed) or the reference's
// ReadFrameHeaderError leaf: each read_exact that would fail maps to the matching *Read error.  `consumed` = bytes taken in every case.
B200Z_HD int parse_frame_header(const uint8_t *p, size_t len, FrameHeader &h, uint32_t &skip_len, size_t &consumed) {
    const size_t want = frame_header_want(p, len);
    consumed = want < len ? want : len;
    if (len < 4) return B200Z_ERR_MAGIC_NUMBER_READ;
    const uint32_t magic = rd32le(p);
    if (skippable_magic(magic)) {
        if (len < 8) return B200Z_ERR_FRAME_DESCRIPTOR_READ;
        skip_len = rd32le(p + 4);
        return B200Z_ERR_SKIP_FRAME;
    }
    if (magic != ZSTD_MAGIC) return B200Z_ERR_BAD_MAGIC_NUMBER;
    if (len < 5) return B200Z_ERR_FRAME_DESCRIPTOR_READ;
    h = FrameHeader();
    h.descriptor = p[4];
    const uint32_t single = h.single_segment(), flag = h.descriptor >> 6;
    const uint32_t did_at = 6u - single, fcs_at = did_at + ((1u << (h.descriptor & 3u)) >> 1);
    if (len < did_at) return B200Z_ERR_WINDOW_DESCRIPTOR_READ;
    if (len < fcs_at) return B200Z_ERR_DICTIONARY_ID_READ;
    if (len < want) return B200Z_ERR_FRAME_CONTENT_SIZE_READ;
    if (!single) h.window_descriptor = p[5];
    for (uint32_t i = did_at; i < fcs_at; i++) h.dict_id += (uint32_t)p[i] << (8 * (i - did_at));
    h.has_dict_id = h.dict_id != 0;
    for (uint32_t i = fcs_at; i < want; i++) h.frame_content_size += (uint64_t)p[i] << (8 * (i - fcs_at));
    if (flag == 1) h.frame_content_size += 256;
    h.header_size = (uint8_t)want;
    return 0;
}

// FrameHeaderError::{WindowTooBig, WindowTooSmall}
B200Z_HD int frame_window_size(const FrameHeader &h, uint64_t &out) {
    if (h.single_segment()) { out = h.frame_content_size; return 0; }
    const uint64_t exp = h.window_descriptor >> 3, mant = h.window_descriptor & 7;
    const uint64_t base = 1ull << (10 + exp);
    const uint64_t w = base + (base / 8) * mant;
    const uint64_t MAXW = (1ull << 41) + 7 * (1ull << 38);
    if (w >= 1024) { if (w < MAXW) { out = w; return 0; } return B200Z_ERR_WINDOW_TOO_BIG; }
    return B200Z_ERR_WINDOW_TOO_SMALL;
}

// ---- block header (3 bytes)
struct BlockHeader {
    bool last = false;
    uint32_t type = 0, decompressed_size = 0, content_size = 0;
};
B200Z_HD int parse_block_header(const uint8_t *b, BlockHeader &h) {
    const uint32_t t = (b[0] >> 1) & 3;
    if (t == 3) return B200Z_ERR_FOUND_RESERVED_BLOCK;
    const uint32_t size = (uint32_t)(b[0] >> 3) | ((uint32_t)b[1] << 5) | ((uint32_t)b[2] << 13);
    if (size > 128u * 1024u) return B200Z_ERR_BLOCK_SIZE_TOO_LARGE;
    h.type = t;
    h.decompressed_size = (t == BT_RAW || t == BT_RLE) ? size : 0;
    h.content_size = t == BT_RLE ? 1 : size;
    h.last = b[0] & 1;
    return 0;
}

// ---- the two section headers of a Compressed block.  Fields stay 0 until the header that holds them has parsed.
struct SectionHeaders {
    uint32_t regen_size;     // literals regenerated size
    uint32_t lit_comp_size;  // literals compressed size (Compressed / Treeless)
    uint32_t nseq;           // number of sequences
    uint32_t seq_off;        // offset of the sequences bitstream (after the 1-4 byte sequences header) inside the block content
    uint32_t status;         // host_status(code, stage, HS_BEFORE_LITERALS / HS_AFTER_LITERALS) of the first header error, 0 = none
    uint8_t lit_type;        // LT_*
    uint8_t nstreams;        // 1 or 4 (Compressed / Treeless), else 0
    uint8_t lit_off;         // length of the literals header = offset of the literals payload; 0 = literals header not parsed
    uint8_t modes;           // compression modes byte
};

// Parses the literals and sequences section headers of the Compressed block content c[0..size), and checks what decompress_block
// checks before the literals stage (block_decoder.rs:120-134) and after it for an empty sequences section (:185-191).
B200Z_HD SectionHeaders parse_section_headers(const uint8_t *c, uint32_t size) {
    SectionHeaders s = {};
    if (size == 0) { s.status = host_status(B200Z_ERR_LITSEC_GET_BITS, B200Z_STAGE_BLOCK_BODY, HS_BEFORE_LITERALS); return s; }
    const uint32_t lt = c[0] & 3, sf = (c[0] >> 2) & 3;
    uint32_t need;
    if (lt == LT_RAW || lt == LT_RLE) need = (sf == 0 || sf == 2) ? 1 : (sf == 1 ? 2 : 3);
    else need = sf <= 1 ? 3 : (sf == 2 ? 4 : 5);
    if (size < need) { s.status = host_status(B200Z_ERR_LITSEC_NOT_ENOUGH_BYTES, B200Z_STAGE_BLOCK_BODY, HS_BEFORE_LITERALS); return s; }
    uint32_t regen = 0, comp = 0;
    if (lt == LT_RAW || lt == LT_RLE) {
        if (sf == 0 || sf == 2) regen = c[0] >> 3;
        else if (sf == 1) regen = (c[0] >> 4) + ((uint32_t)c[1] << 4);
        else regen = (c[0] >> 4) + ((uint32_t)c[1] << 4) + ((uint32_t)c[2] << 12);
    } else {
        s.nstreams = sf == 0 ? 1 : 4;
        if (sf <= 1) { regen = (c[0] >> 4) + (((uint32_t)c[1] & 0x3f) << 4); comp = (c[1] >> 6) + ((uint32_t)c[2] << 2); }
        else if (sf == 2) { regen = (c[0] >> 4) + ((uint32_t)c[1] << 4) + (((uint32_t)c[2] & 3) << 12); comp = (c[2] >> 2) + ((uint32_t)c[3] << 6); }
        else { regen = (c[0] >> 4) + ((uint32_t)c[1] << 4) + (((uint32_t)c[2] & 0x3f) << 12); comp = (c[2] >> 6) + ((uint32_t)c[3] << 2) + ((uint32_t)c[4] << 10); }
    }
    s.lit_type = (uint8_t)lt; s.regen_size = regen; s.lit_comp_size = comp; s.lit_off = (uint8_t)need;
    const uint32_t upper = (lt == LT_COMPRESSED || lt == LT_TREELESS) ? comp : (lt == LT_RLE ? 1 : regen);
    if (size - need < upper) { s.status = host_status(B200Z_ERR_MALFORMED_SECTION_HEADER, B200Z_STAGE_BLOCK_BODY, HS_BEFORE_LITERALS); return s; }
    const uint8_t *q = c + need + upper;
    const uint32_t rem = size - need - upper;
    uint32_t hdr = 0, nseq = 0, modes = 0;
    bool bad = false;
    if (rem == 0) bad = true;
    else if (q[0] == 0) { hdr = 1; }
    else if (q[0] < 128) { if (rem < 2) bad = true; else { nseq = q[0]; modes = q[1]; hdr = 2; } }
    else if (q[0] < 255) {
        if (rem < 2) bad = true;
        else {
            nseq = (((uint32_t)q[0] - 128) << 8) + q[1]; hdr = 2;
            if (nseq != 0) { if (rem < 3) bad = true; else { modes = q[2]; hdr = 3; } }
        }
    } else { if (rem < 4) bad = true; else { nseq = (uint32_t)q[1] + ((uint32_t)q[2] << 8) + 0x7F00; modes = q[3]; hdr = 4; } }
    if (bad) { s.status = host_status(B200Z_ERR_SEQHDR_NOT_ENOUGH_BYTES, B200Z_STAGE_BLOCK_BODY, HS_AFTER_LITERALS); return s; }
    s.nseq = nseq; s.modes = (uint8_t)modes; s.seq_off = need + upper + hdr;
    if (nseq == 0 && rem != hdr) s.status = host_status(B200Z_ERR_SEQ_EXTRA_BITS, B200Z_STAGE_SEQUENCES, HS_AFTER_LITERALS);
    return s;
}

// ---- what k_walk hands the planner for a frame that lives in device memory: the frame header bytes, every block's 3-byte header
// and section headers as parsed above, and the checksum -- instead of copying the compressed input back to the host
struct WalkFrame {
    uint8_t hdr[20];      // the frame's first bytes (magic .. frame header), zero padded
    uint32_t hdr_avail;   // how many of them exist
    uint32_t nblocks;     // block digests of this frame
    uint32_t stop;        // 0 last block seen, 1 block header truncated, 2 reserved type / size too large, 3 content truncated, 4 no walk (frame header)
    uint32_t tail_avail;  // bytes available after the last block (up to 4: the content checksum)
    uint8_t tail[4];
    uint32_t pad;
    uint64_t end_pos;     // frame-relative position after the last walked block
};
struct WalkBlock {
    uint64_t pos;         // frame-relative position of the 3-byte block header
    SectionHeaders sec;   // parse_section_headers of a Compressed block's content, else zero
    uint8_t bh[3];
    uint8_t pad[5];
};

// The header walk of the frame at p[0..len): the planner's parsers along the chain of blocks, run by k_walk on device input and by
// the host on host input.  F gets the frame digest.  fill == 0 only counts the blocks; fill == 1 writes their digests at
// wb[first[idx]].  Anything wrong with the frame header is the planner's to report (stop = 4, no blocks).
B200Z_HD void walk_frame(const uint8_t *p, uint64_t len, WalkFrame &F, WalkBlock *wb, const uint32_t *first, uint32_t idx, int fill) {
    const uint32_t hdr_avail = (uint32_t)(len < 20 ? len : 20);
    for (uint32_t i = 0; i < 20; i++) F.hdr[i] = i < hdr_avail ? p[i] : 0;
    uint32_t nb = 0, stop = 4, tail_avail = 0;
    uint64_t end_pos = 0;
    FrameHeader fh;
    uint32_t skip_len;
    size_t pos;
    if (parse_frame_header(p, len, fh, skip_len, pos) == 0) {
        const uint32_t base = fill ? first[idx] : 0u;
        for (;;) {
            if (len - pos < 3) { stop = 1; break; }
            WalkBlock B = {};
            B.pos = pos; B.bh[0] = p[pos]; B.bh[1] = p[pos + 1]; B.bh[2] = p[pos + 2];
            BlockHeader bh;
            if (parse_block_header(p + pos, bh)) {   // the planner reports FoundReservedBlock / BlockSizeTooLarge from these 3 bytes
                if (fill) wb[base + nb] = B;
                nb++; stop = 2; break;
            }
            pos += 3;
            if (len - pos < bh.content_size) {
                if (fill) wb[base + nb] = B;
                nb++; stop = 3; break;
            }
            if (bh.type == BT_COMPRESSED) B.sec = parse_section_headers(p + pos, bh.content_size);
            if (fill) wb[base + nb] = B;
            nb++;
            pos += bh.content_size;
            if (bh.last) {   // the content checksum may follow
                stop = 0;
                tail_avail = (uint32_t)(len - pos < 4 ? len - pos : 4);
                break;
            }
        }
        end_pos = pos;
    }
    for (uint32_t i = 0; i < 4; i++) F.tail[i] = i < tail_avail ? p[end_pos + i] : 0;
    F.hdr_avail = hdr_avail; F.nblocks = nb; F.stop = stop; F.tail_avail = tail_avail; F.pad = 0; F.end_pos = end_pos;
}

// Where a buffer of concatenated frames goes on after the frame at offset `at` whose walk is F (decode_all, frame_decoder.rs:541-577):
// behind the content checksum, if the descriptor announces one, for a zstd frame whose walk reached its last block; behind the
// skipped bytes for a skippable frame; `at` itself -- the chain ends there -- for anything else.  The caller checks the result
// against the input's length (a skippable frame that runs past it is FailedToSkipFrame).
B200Z_HD uint64_t frame_chain_next(uint64_t at, const WalkFrame &F) {
    if (F.hdr_avail < 4) return at;
    const uint32_t magic = rd32le(F.hdr);
    if (skippable_magic(magic)) return F.hdr_avail < 8 ? at : at + 8 + rd32le(F.hdr + 4);
    if (magic != ZSTD_MAGIC || F.stop != 0) return at;
    return at + F.end_pos + (((F.hdr[4] >> 2) & 1u) ? 4 : 0);
}

}  // namespace b200z
