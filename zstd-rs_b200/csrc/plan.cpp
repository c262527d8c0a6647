// plan.cpp -- host-side planning of a submission (plan.h).
#include "plan.h"

#include <string.h>

#include <algorithm>
#include <utility>

namespace b200z {

static inline uint64_t rd64le(const uint8_t *p) { return (uint64_t)rd32le(p) | ((uint64_t)rd32le(p + 4) << 32); }

static TabRef one_mode(uint32_t mode, TabRef cur, int32_t slot_idx) {
    TabRef r;
    switch (mode) {
        case MODE_PREDEFINED: r.kind = TabRef::PREDEF; return r;
        case MODE_RLE:
        case MODE_FSE: r.kind = TabRef::SLOT; r.idx = (uint32_t)slot_idx; return r;
        default: return cur;  // Repeat: whatever was last (table or RLE byte), sequence_section_decoder.rs:333-336
    }
}

void plan_compressed_block(const SectionHeaders &sec, BlockDesc &d, BlockRefs &r, TableCursor &cur, uint32_t &n_huf_slots, uint32_t &n_fse_slots,
                           uint64_t &lit_bytes, uint64_t &nseq_total) {
    d.lit_type = sec.lit_type; d.nstreams = sec.nstreams; d.regen_size = sec.regen_size; d.lit_comp_size = sec.lit_comp_size; d.lit_off = sec.lit_off;
    d.nseq = sec.nseq; d.modes = sec.modes; d.seq_off = sec.seq_off; d.host_status = sec.status;
    if (host_status_pos(sec.status) == HS_BEFORE_LITERALS) return;
    const uint32_t lt = sec.lit_type, nseq = sec.nseq, modes = sec.modes;
    if (lt == LT_COMPRESSED) {
        r.build_huf = (int32_t)n_huf_slots++;
        cur.huf.kind = TabRef::SLOT; cur.huf.idx = (uint32_t)r.build_huf;
        r.huf = cur.huf;
    } else if (lt == LT_TREELESS) r.huf = cur.huf;
    if (lt == LT_COMPRESSED || lt == LT_TREELESS) {
        d.lit_buf_off = lit_bytes;
        lit_bytes += ((uint64_t)sec.regen_size + 31) & ~15ull;  // 16-byte aligned, >= 16 bytes of slack for vector stores
    }
    if (nseq == 0) return;   // (also when the sequences header failed)
    uint32_t ml_ = (modes >> 6) & 3, mo = (modes >> 4) & 3, mm = (modes >> 2) & 3;
    bool needs_slot = ml_ == MODE_RLE || ml_ == MODE_FSE || mo == MODE_RLE || mo == MODE_FSE || mm == MODE_RLE || mm == MODE_FSE;
    if (needs_slot) r.build_fse = (int32_t)n_fse_slots++;
    cur.ll = one_mode(ml_, cur.ll, r.build_fse);
    cur.of = one_mode(mo, cur.of, r.build_fse);
    cur.ml = one_mode(mm, cur.ml, r.build_fse);
    r.ll = cur.ll; r.of = cur.of; r.ml = cur.ml;
    d.seq_buf_off = nseq_total;
    nseq_total += (nseq + 3) & ~3ull;   // keeps every block's sequence array 16-byte aligned (3 x u32 x 4)
}

// ---- XXH64 ------------------------------------------------------------------------------------------------
static const uint64_t P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;
static inline uint64_t rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static inline uint64_t rnd(uint64_t acc, uint64_t in) { acc += in * P2; acc = rotl(acc, 31); return acc * P1; }
static inline uint64_t mrg(uint64_t acc, uint64_t v) { v = rnd(0, v); acc ^= v; return acc * P1 + P4; }
void XXH64State::reset() { v[0] = P1 + P2; v[1] = P2; v[2] = 0; v[3] = 0ull - P1; total = 0; memsize = 0; }
void XXH64State::update(const uint8_t *p, size_t len) {
    total += len;
    if (memsize + len < 32) { if (len) memcpy(mem + memsize, p, len); memsize += (uint32_t)len; return; }
    const uint8_t *end = p + len;
    if (memsize) {
        size_t fill = 32 - memsize;
        memcpy(mem + memsize, p, fill);
        for (int i = 0; i < 4; i++) v[i] = rnd(v[i], rd64le(mem + 8 * i));
        p += fill; memsize = 0;
    }
    while (p + 32 <= end) { for (int i = 0; i < 4; i++) v[i] = rnd(v[i], rd64le(p + 8 * i)); p += 32; }
    if (p < end) { memcpy(mem, p, (size_t)(end - p)); memsize = (uint32_t)(end - p); }
}
uint64_t XXH64State::digest() const {
    uint64_t h;
    if (total >= 32) { h = rotl(v[0], 1) + rotl(v[1], 7) + rotl(v[2], 12) + rotl(v[3], 18); for (int i = 0; i < 4; i++) h = mrg(h, v[i]); }
    else h = v[2] + P5;
    h += total;
    const uint8_t *p = mem, *end = mem + memsize;
    while (p + 8 <= end) { h ^= rnd(0, rd64le(p)); h = rotl(h, 27) * P1 + P4; p += 8; }
    if (p + 4 <= end) { h ^= (uint64_t)rd32le(p) * P1; h = rotl(h, 23) * P2 + P3; p += 4; }
    while (p < end) { h ^= (*p) * P5; h = rotl(h, 11) * P1; p++; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

// ---------------------------------------------------------------------------------------------------------------
// Scheduling decisions (plan.h).  k_exec_cta puts a whole CTA on a frame's chain of blocks (~15x faster per frame), k_exec one warp --
// but k_exec keeps ~4,700 frames in flight and needs fewer instructions per byte, so it wins once there are enough frames to fill
// the machine (on 1 MiB Silesia-mix frames of 8 blocks the crossover lies between 1,024 and 2,048 frames).  Model:
//          t_cta  = max(sum w / SMs, largest w) * kCtaMs            (one CTA per frame, a frame at a time)
//          t_warp = largest w * kWarpChainMs + sum w * kWarpMs      (the longest chain, slowed down by everything else in flight)
// The eligible frames are sorted by work; the k largest would go to CTAs and the rest to warps (the two kernels run one after the
// other: each wants whole SMs).  A real split is taken only when the model promises a clear gain over both pure choices: on similar
// frames the time a split saves in k_exec is smaller than what it adds in k_exec_cta.
// ---------------------------------------------------------------------------------------------------------------
void route_exec_frames(const uint64_t *work, const uint8_t *eligible, size_t nframes, uint32_t sms_u, std::vector<uint32_t> &cta_frames) {
    cta_frames.clear();
    std::vector<std::pair<uint64_t, uint32_t>> cand;   // (work, frame)
    uint64_t warp_only_work = 0;
    for (size_t f = 0; f < nframes; f++) {
        if (eligible[f]) cand.emplace_back(work[f], (uint32_t)f);
        else warp_only_work += work[f];
    }
    if (cand.empty()) return;
    constexpr double kCtaMs = 1.06e-5, kWarpChainMs = 5.8e-5, kWarpMs = 1.07e-8;
    const double sms = (double)std::max<uint32_t>(1u, sms_u);
    std::sort(cand.begin(), cand.end(), [](const std::pair<uint64_t, uint32_t> &x, const std::pair<uint64_t, uint32_t> &y) {
        return x.first != y.first ? x.first > y.first : x.second < y.second;
    });
    std::vector<uint64_t> suffix(cand.size() + 1, 0);
    for (size_t i = cand.size(); i-- > 0;) suffix[i] = suffix[i + 1] + cand[i].first;
    size_t best_k = 0;
    double best_t = 0, t_none = 0, t_all = 0;
    uint64_t prefix = 0;
    for (size_t k = 0; k <= cand.size(); k++) {   // the k largest on CTAs
        const double t_cta = k ? std::max((double)prefix / sms, (double)cand[0].first) * kCtaMs : 0.0;
        const double t_warp = (k < cand.size() ? (double)cand[k].first * kWarpChainMs : 0.0) + (double)(suffix[k] + warp_only_work) * kWarpMs;
        if (k == 0) t_none = t_cta + t_warp;
        if (k == cand.size()) t_all = t_cta + t_warp;
        if (k == 0 || t_cta + t_warp < best_t) { best_t = t_cta + t_warp; best_k = k; }
        if (k < cand.size()) prefix += cand[k].first;
    }
    if (best_k != 0 && best_k != cand.size() && best_t > 0.7 * std::min(t_none, t_all)) best_k = t_none <= t_all ? 0 : cand.size();
    for (size_t k = 0; k < best_k; k++) cta_frames.push_back(cand[k].second);
}

// k_exec runs beside k_fse and walks every frame's blocks in order: in descriptor order (frame after frame) the frames at the end of
// the list sit idle until k_fse's last wave and the 16 chains of a k_fse warp are 2 frames x 8 blocks of very different lengths.
// Rows -- block 0 of every frame, then block 1, ... -- sorted by sequence count keep every chain fed and a warp's chains alike
// (a warp takes as long as its longest chain).
void build_fse_order(const uint32_t *first_block, const uint32_t *nblocks, const uint8_t *on_cta, size_t nframes, const uint32_t *nseq,
                     size_t nblocks_total, std::vector<uint32_t> &order) {
    order.clear();
    uint32_t maxb = 0;
    size_t covered = 0;
    bool want = false;
    for (size_t f = 0; f < nframes; f++) {
        covered += nblocks[f];
        if (on_cta[f]) continue;
        maxb = std::max(maxb, nblocks[f]);
        if (nblocks[f] >= 2) want = true;
    }
    if (!want || covered != nblocks_total) return;
    std::vector<uint8_t> seen(nblocks_total, 0);   // the frames must cover every block exactly once
    for (size_t f = 0; f < nframes; f++)
        for (uint32_t k = 0; k < nblocks[f]; k++) {
            const uint64_t b = (uint64_t)first_block[f] + k;
            if (b >= nblocks_total || seen[b]) return;
            seen[b] = 1;
        }
    std::vector<uint32_t> start(maxb + 2, 0);   // start[bi + 1] = blocks with block-in-frame index bi among the warp kernel's frames
    for (size_t f = 0; f < nframes; f++)
        if (!on_cta[f]) for (uint32_t k = 0; k < nblocks[f]; k++) start[k + 1]++;
    for (uint32_t k = 0; k <= maxb; k++) start[k + 1] += start[k];
    uint32_t tail = start[maxb + 1];   // k_exec_cta's frames follow, frame after frame
    order.assign(nblocks_total, 0u);
    for (size_t f = 0; f < nframes; f++)
        for (uint32_t k = 0; k < nblocks[f]; k++) {
            if (on_cta[f]) order[tail++] = first_block[f] + k;
            else order[start[k]++] = first_block[f] + k;
        }
    uint32_t lo = 0;
    for (uint32_t k = 0; k < maxb; k++) {
        const uint32_t hi = start[k];   // (start[k] has advanced to the end of row k)
        std::sort(order.begin() + lo, order.begin() + hi, [&](uint32_t x, uint32_t y) { return nseq[x] != nseq[y] ? nseq[x] > nseq[y] : x < y; });
        lo = hi;
    }
}

}  // namespace b200z
