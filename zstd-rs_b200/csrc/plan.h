// plan.h -- host-side planning of a submission: table slots and scratch offsets of each block from its parsed section headers
// (framing.cuh), the scheduling decisions of a submission, and the streaming XXH64 of the frame decoder.
#pragma once
#include <stdint.h>

#include <vector>

#include "../../include/b200zstd.h"
#include "b200z_types.h"
#include "framing.cuh"

namespace b200z {

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

// Fills the section-level fields of `d` for a Compressed block from its parsed section headers and assigns its table slots and
// scratch offsets.  A header error stays in d.host_status with its position (HS_BEFORE_LITERALS / HS_AFTER_LITERALS) so that the
// device can report the first error in reference order; after HS_AFTER_LITERALS the literals are still decoded.
void plan_compressed_block(const SectionHeaders &sec, BlockDesc &d, BlockRefs &r, TableCursor &cur, uint32_t &n_huf_slots, uint32_t &n_fse_slots,
                           uint64_t &lit_bytes, uint64_t &nseq_total);

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
