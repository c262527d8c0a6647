// plan.h -- host-side framing: the part of the reference that stays on the host (SURVEY.md 8(a) row a11).
//   read_frame_header        ruzstd/src/decoding/frame.rs:6-85, window_size :116-139
//   read_block_header        ruzstd/src/decoding/block_decoder.rs:201-283
//   LiteralsSection::parse   ruzstd/src/blocks/literals_section.rs:117-223
//   SequencesHeader::parse   ruzstd/src/blocks/sequence_section.rs:108-167
// The planner walks these fixed-size headers only; table descriptions and bitstreams are parsed on the GPU.
#pragma once
#include <stdint.h>

#include <vector>

#include "../../include/b200zstd.h"
#include "b200z_types.h"

namespace b200z {

struct FrameHeader {
    uint8_t descriptor = 0, window_descriptor = 0;
    bool has_dict_id = false;
    uint32_t dict_id = 0;
    uint64_t frame_content_size = 0;
    uint8_t header_size = 0;
    bool single_segment() const { return (descriptor >> 5) & 1; }
    bool content_checksum() const { return (descriptor >> 2) & 1; }
};

// Parses a frame header from a byte slice.  Returns 0, B200Z_ERR_SKIP_FRAME (skip_len set, 8 bytes consumed) or
// the reference's ReadFrameHeaderError leaf.  `consumed` = bytes taken from the slice in every case.
int parse_frame_header(const uint8_t *p, size_t len, FrameHeader &h, uint32_t &skip_len, size_t &consumed);
int frame_window_size(const FrameHeader &h, uint64_t &out);  // FrameHeaderError::{WindowTooBig,WindowTooSmall}

struct BlockHeader {
    bool last = false;
    uint32_t type = 0, decompressed_size = 0, content_size = 0;
};
int parse_block_header(const uint8_t b[3], BlockHeader &h);

// where a table comes from, resolved to a device pointer once the slot arrays are allocated
struct TabRef {
    enum Kind : uint8_t { NONE = 0, SLOT = 1, PREDEF = 2, CARRY = 3 } kind = NONE;
    uint32_t idx = 0;
};
struct BlockRefs { TabRef huf, ll, of, ml; int32_t build_huf = -1, build_fse = -1; };

// "current tables" of a frame while planning (DecoderScratch.huf / .fse, scratch.rs:15-27)
struct TableCursor {
    TabRef huf, ll, of, ml;
};

// Fills the section-level fields of `d` for a Compressed block whose content is content[0..size).
// Errors the reference raises from header parsing are recorded in d.host_status with their position
// (HS_BEFORE_LITERALS / HS_AFTER_LITERALS) so the device can report the first error in reference order.
void plan_compressed_block(const uint8_t *content, uint32_t size, BlockDesc &d, BlockRefs &r, TableCursor &cur,
                           uint32_t &n_huf_slots, uint32_t &n_fse_slots, uint64_t &lit_bytes, uint64_t &nseq_total);

void plan_compressed_block_view(const uint8_t *lit_hdr, const uint8_t *seq_hdr, uint32_t size, BlockDesc &d, BlockRefs &r, TableCursor &cur,
                                uint32_t &n_huf_slots, uint32_t &n_fse_slots, uint64_t &lit_bytes, uint64_t &nseq_total);

// ---- scheduling decisions of a submission (pure host logic; CPU tests call them through b200z_debug_route_frames / _fse_order)
// Which execution kernel takes a frame.  work[f] = sequences + compressed bytes / 16 of frame f, eligible[f] = the frame may go to
// k_exec_cta (two or more blocks, >= 4096 compressed bytes, no dictionary); the others always take k_exec and only add to the
// load.  Returns the frames of k_exec_cta, largest first (its ticket order).  The cost model and its constants: DESIGN.md 4.1.
void route_exec_frames(const uint64_t *work, const uint8_t *eligible, size_t nframes, uint32_t sms, std::vector<uint32_t> &cta_frames);
// The order in which k_fse takes the blocks (PipelineArgs::fse_order): row by row (block-in-frame index) across the frames that are
// not on k_exec_cta, inside a row by decreasing sequence count, then the blocks of k_exec_cta's frames, frame after frame.  Left
// empty (= descriptor order) when no frame of the warp kernel has two blocks or the frames do not cover the blocks exactly.
void build_fse_order(const uint32_t *first_block, const uint32_t *nblocks, const uint8_t *on_cta, size_t nframes, const uint32_t *nseq,
                     size_t nblocks_total, std::vector<uint32_t> &order);

// XXH64 (seed 0) streaming -- the hash the reference feeds on drain (decode_buffer.rs:42,225,290,301)
struct XXH64State {
    uint64_t v[4], total;
    uint8_t mem[32];
    uint32_t memsize;
    void reset();
    void update(const uint8_t *p, size_t len);
    uint64_t digest() const;
};

}  // namespace b200z
