// exec_cta.cuh -- k_exec_cta: LZ77 execution with the block's output assembled in SHARED MEMORY (included by kernels.cu).
//
// Replaces execute_sequences + do_offset_history (sequence_execution.rs:5-118) and DecodeBuffer::{push, repeat,
// repeat_in_chunks} (decode_buffer.rs:74-141) for the common case; anything else (dictionary reach, invalid offsets,
// blocks larger than the window buffer, error statuses, raw-offset blocks) is left to the warp-per-frame kernel
// k_exec, which resumes the frame at the block where this kernel stopped (`resume[]`).
//
// One persistent CTA per SM takes frames from a ticket counter and walks a frame's blocks in order (the window /
// offset-history chain of frame_decoder.rs:321-374 stays inside one CTA).  Per Compressed block:
//   * the regenerated literals are staged into shared memory by ONE bulk copy (cp.async.bulk + mbarrier, TMA);
//   * the block's output (<= 128 KiB) is assembled in shared memory, so every match source inside the block is a
//     shared-memory read (no DRAM burst per match, which was 6.6 GB per GiB of output in round 1); sources in earlier
//     blocks of the frame come from global memory (L2);
//   * finished pieces leave as bulk stores shared -> global (cp.async.bulk, 16-byte aligned: the window is laid out
//     at (global address & 15) so that shared and global alignment agree), overlapped with the rest of the block.
// Work decomposition: sequences arrive in PREFIX form from k_fse ({out_end, lit_end, offset}), so any thread can place
// any sequence without a scan.  A batch = 1024 sequences, two per thread: the thread resolves the symbolic offsets,
// validates them, and publishes per sequence (a) an 8-byte record {match start, literal delta, offset} into a ring, (b) a bit at the
// sequence's last byte in a block-wide bitmask, (c) for every 64-byte chunk whose first byte it owns, its index.
// Output is then produced in ROWS of 128 bytes, one warp per row, FOUR bytes per lane: owner of the lane's first byte =
// first64[chunk] + popc(mask bits below); a 4-byte word spans at most two sequences (match length >= 3), so two
// records are fetched; each byte selects literal or match source and is read from shared memory; one aligned 32-bit
// store per lane.  Match bytes whose source lies in rows that are being produced at the same time follow the TRUE byte
// dependency, not the row order: every row publishes which of its bytes are still pending (four 32-bit planes per row,
// plane k = ballot of "byte k of the lane's word is pending"); a byte is copied as soon as its source byte's bit is
// clear.  Sources always precede destinations, so the lowest unfinished row can always complete; a row-to-row chain
// (waiting for whole rows instead serialises every block) only forms where the data really chains.
// Overlapping matches use source = start + (k mod offset), the byte-order-preserving form of repeat_in_chunks
// (decode_buffer.rs:113-141).
#pragma once

namespace b200z {

constexpr uint32_t XC_WARPS = 16, XC_THREADS = XC_WARPS * 32;
constexpr uint32_t XC_PER_THREAD = 2;                      // consecutive sequences a thread publishes per batch
constexpr uint32_t XC_BATCH = XC_THREADS * XC_PER_THREAD;  // sequences per batch
constexpr uint32_t XC_RING = 2 * XC_BATCH;                 // record ring, 8-byte entries: the batch being produced + the next one
constexpr uint32_t XC_WIN_MAX = 128u << 10;                // largest block output handled here
constexpr uint32_t XC_ROWS_MAX = XC_WIN_MAX / 128 + 1;     // + 1: the window starts at (global address & 15)
constexpr uint32_t XC_DATA_BYTES = 182u << 10;             // window rows + staged literals
constexpr uint32_t XC_MASK_BYTES = 16448;                  // >= XC_ROWS_MAX * 16, multiple of 64: one bit per window byte
constexpr uint32_t XC_FIRST_BYTES = 8256;                  // >= XC_ROWS_MAX * 8: one u32 per 64 window bytes
constexpr uint32_t XC_PROWS = 256;                         // rows whose pending planes are live at once (a sub-phase)
constexpr uint32_t XC_OFF_MASK = XC_DATA_BYTES;
constexpr uint32_t XC_OFF_FIRST = XC_OFF_MASK + XC_MASK_BYTES;
constexpr uint32_t XC_OFF_RING = XC_OFF_FIRST + XC_FIRST_BYTES;
constexpr uint32_t XC_OFF_PEND = XC_OFF_RING + XC_RING * 8;   // [XC_PROWS][4] u32
constexpr uint32_t XC_OFF_MISC = XC_OFF_PEND + XC_PROWS * 16;
constexpr uint32_t XC_SMEM_BYTES = XC_OFF_MISC + 128;
static_assert(XC_SMEM_BYTES <= 232448, "k_exec_cta: more than 227 KiB of shared memory");
static_assert(XC_MASK_BYTES >= XC_ROWS_MAX * 16 && XC_FIRST_BYTES >= XC_ROWS_MAX * 8, "k_exec_cta tables");
constexpr uint32_t XC_SPIN_LIMIT = 1u << 18;               // bounded waits: a stuck wait turns into a bail-out, never a hang

// Why a frame was handed back to k_exec: bits OR-ed into ticket[2], read by b200z_batch_debug_sched
enum : uint32_t {
    XC_WHY_ERROR = 1u,          // an error status (planner, literals or sequence stage)
    XC_WHY_CAPACITY = 2u,       // the output does not fit
    XC_WHY_SEQ_RECORDS = 4u,    // wide records, or raw offsets that cannot be resolved in place (values >= 2^30)
    XC_WHY_BLOCK_SIZE = 8u,     // block sizes / literal counts it does not take
    XC_WHY_RLE_LITERALS = 16u,  // RLE literals that do not fit beside the window
    XC_WHY_SEQ_CHECK = 32u,     // sequence validation failed (dictionary reach, invalid offsets)
    XC_WHY_TIMEOUT = 64u,       // an internal wait timed out
    XC_WHY_FRAME_STATE = 128u,  // the frame arrived failed or with a dictionary
};

struct XcMisc {               // at XC_OFF_MISC
    unsigned long long mbar;  // literals bulk-copy barrier
    uint32_t ticket;
    uint32_t bail;            // a thread found something this kernel does not handle (or a wait timed out)
    uint32_t ovl[4];          // per batch (mod 4): some match overlaps its own output
    uint32_t end_a[2];        // per batch (mod 2): window position where the batch's last sequence ends
};

// ---- PTX wrappers: mbarrier + bulk async copies (TMA, non-tensor form)
__device__ __forceinline__ void xc_mbar_init(uint32_t a, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "r"(count) : "memory"); }
__device__ __forceinline__ void xc_mbar_expect_tx(uint32_t a, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(a), "r"(bytes) : "memory"); }
__device__ __forceinline__ bool xc_mbar_try_wait(uint32_t a, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(a), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void xc_bulk_g2s(uint32_t sdst, const void *gsrc, uint32_t bytes, uint32_t mbar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(sdst), "l"(gsrc), "r"(bytes), "r"(mbar) : "memory");
}
__device__ __forceinline__ void xc_bulk_s2g(void *gdst, uint32_t ssrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(ssrc), "r"(bytes) : "memory");
}
__device__ __forceinline__ void xc_bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void xc_bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void xc_bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void xc_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void xc_fence_cta() { asm volatile("fence.acq_rel.cta;" ::: "memory"); }
__device__ __forceinline__ uint32_t xc_ld_acquire_shared(uint32_t a) { uint32_t v; asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ uint32_t xc_ldg_cg_u8(const uint8_t *p) { uint32_t v; asm volatile("ld.global.cg.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }

// 8-byte ring record: lo = match start (window position, 18 bits) | literal delta << 18 (low 14 bits),
//                     hi = literal delta >> 14 (4 bits) | offset << 4 (28 bits)
// literal byte at window position a comes from shared-memory offset a + delta; match byte from a - offset.
__device__ __forceinline__ uint2 xc_pack(uint32_t mstart_a, uint32_t lz, uint32_t off) { return make_uint2(mstart_a | (lz << 18), (lz >> 14) | (off << 4)); }
struct XcRec { uint32_t x, lz, noff; };
__device__ __forceinline__ XcRec xc_unpack(uint2 r) {
    XcRec o;
    o.x = r.x & 0x3FFFFu;
    o.lz = __funnelshift_r(r.x, r.y, 18) & 0x3FFFFu;
    o.noff = 0u - (r.y >> 4);
    return o;
}

// Uniform (per block) values every thread holds
struct XcBlk {
    uint32_t S;          // shared-memory byte address of the data area
    uint32_t woff;       // window position of the block's first byte (= its global address & 15)
    uint32_t a_end;      // woff + out_size
    uint32_t nrows;
    uint32_t lit_s;      // shared-memory offset (from S) of literal 0
    uint32_t nseq, ntot; // real sequences; + the trailing-literals pseudo sequence (sentinel record at index ntot)
    uint32_t out_size, regen;
    uint32_t h0, h1, h2; // offset history at the block's start
    uint64_t reach;      // bytes of earlier output of the frame a match may reach back into (produced - drained)
    const uint32_t *seqs;
    uint8_t *gout;       // global address of the block's first output byte
    const uint8_t *lit_gp;  // literals too large to stage beside the window: global address of literal 0 (else null)
};
constexpr uint32_t XC_LITG_BIAS = (1u << 17) + 64u;   // keeps the literal delta of the global-literals mode non-negative (18 bits)

__device__ __forceinline__ uint32_t xc_lds_volatile(uint32_t a) { uint32_t v; asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }

// NR rows of 128 window bytes (rows r0, r0 + XC_WARPS, ...) by one warp, interleaved for instruction-level parallelism;
// branch-free per byte.  `lo_a` = first window position of the current sub-phase: everything below it is final.
// Returns false if a wait timed out.
template <bool FAR, bool LITG, int NR>
__device__ __forceinline__ bool xc_rows(const XcBlk &B, uint32_t r0, uint32_t lo_a, bool has_ovl, uint32_t lane) {
    const uint32_t S = B.S, S_mask = S + XC_OFF_MASK, S_first = S + XC_OFF_FIRST, S_ring = S + XC_OFF_RING, S_pend = S + XC_OFF_PEND;
    // first position of the block in this sub-phase: sources below it are final (earlier sub-phases / phases), or -- below
    // woff -- in earlier blocks of the frame (global memory)
    const int32_t fin_a = (int32_t)max(lo_a, B.woff);
    uint32_t a0[NR], word[NR], pend[NR];
    int32_t src[NR][4];
#pragma unroll
    for (int j = 0; j < NR; j++) {
        const uint32_t r = r0 + (uint32_t)j * XC_WARPS;
        a0[j] = (r << 7) + (lane << 2);
        // ---- who owns my four bytes
        const uint32_t c = a0[j] >> 6;
        const uint2 M = lds64(S_mask + (c << 3));
        const bool hi_half = (a0[j] & 32u) != 0;
        const uint32_t W = hi_half ? M.y : M.x;
        const uint32_t sh = a0[j] & 31u;
        const uint32_t owner0 = lds32(S_first + (c << 2)) + (uint32_t)__popc(W & ((1u << sh) - 1u)) + (hi_half ? (uint32_t)__popc(M.x) : 0u);
        const uint32_t nib = (W >> sh) & 7u;   // sequence ends at my bytes 0..2: the following bytes belong to the next sequence
        const XcRec A = xc_unpack(lds64(S_ring + ((owner0 & (XC_RING - 1u)) << 3)));
        const XcRec Bn = xc_unpack(lds64(S_ring + (((owner0 + 1u) & (XC_RING - 1u)) << 3)));
        word[j] = 0; pend[j] = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const bool useB = k > 0 && (nib & ((1u << k) - 1u)) != 0u;
            const uint32_t x = useB ? Bn.x : A.x, lz = useB ? Bn.lz : A.lz, noff = useB ? Bn.noff : A.noff;
            const uint32_t a = a0[j] + (uint32_t)k;
            const bool mt = a >= x;
            src[j][k] = (int32_t)(a + (mt ? noff : lz));
            if (has_ovl) {   // overlapping match: byte kk comes from kk mod offset (warp-uniform branch, rare)
                const uint32_t kk = a - x, off = 0u - noff;
                if (mt && kk >= off) src[j][k] = (int32_t)(x - off + kk % off);
            }
            // A source produced in this sub-phase: its row's pending plane says whether the byte is there yet (my own row's
            // planes are still all-ones: in-row sources always go through the rounds below).  The plane word is read for every
            // byte (any address inside the plane area is harmless) so that there is no branch.
            const uint32_t sa = (uint32_t)src[j][k];
            const uint32_t pm = xc_lds_volatile(S_pend + (((sa >> 7) & (XC_PROWS - 1u)) << 4) + ((sa & 3u) << 2));
            const bool wait = mt && src[j][k] >= fin_a && ((pm >> ((sa >> 2) & 31u)) & 1u) != 0u;
            const bool far = FAR && mt && src[j][k] < (int32_t)B.woff;
            const bool litg = LITG && !mt;   // literals read from global memory: src = literal index + XC_LITG_BIAS
            uint32_t v = lds8(S + ((wait || far || litg) ? a : sa));   // (a byte that waits / comes from global memory reads itself: harmless)
            if (FAR) { if (far) v = xc_ldg_cg_u8(B.gout + (src[j][k] - (int32_t)B.woff)); }
            if (LITG) { if (litg) v = __ldg(B.lit_gp + min(sa - XC_LITG_BIAS, B.regen - 1u)); }   // (clamp: bytes outside the block in the first / last row)
            word[j] |= v << (8 * k);
            pend[j] |= wait ? (1u << k) : 0u;
        }
    }
    bool anyp = false;
#pragma unroll
    for (int j = 0; j < NR; j++) { sts32(S + a0[j], word[j]); anyp = anyp || pend[j] != 0u; }
    if (__any_sync(0xffffffffu, anyp)) {
        // Bytes whose source was not there yet.  Each round: publish which bytes are still pending (data first, then the
        // planes), then copy every pending byte whose source byte is no longer pending.  The lowest pending byte of the lowest
        // unfinished row never depends on a pending byte, so the loops of all warps terminate.
        uint32_t spins = 0;
        bool publish = true;
        for (;;) {
            __syncwarp();
            uint32_t pm[NR][4], left = 0;
#pragma unroll
            for (int j = 0; j < NR; j++) {
#pragma unroll
                for (int k = 0; k < 4; k++) { pm[j][k] = __ballot_sync(0xffffffffu, (pend[j] >> k) & 1u); left |= pm[j][k]; }
            }
            if (left == 0u) break;
            if (publish) {
                if (lane < 4) {
                    xc_fence_cta();
#pragma unroll
                    for (int j = 0; j < NR; j++) {
                        const uint32_t r = r0 + (uint32_t)j * XC_WARPS;
                        sts32(S_pend + ((r & (XC_PROWS - 1u)) << 4) + (lane << 2), lane == 0 ? pm[j][0] : (lane == 1 ? pm[j][1] : (lane == 2 ? pm[j][2] : pm[j][3])));
                    }
                }
                __syncwarp();
            } else __nanosleep(20);
            bool changed = false;
#pragma unroll
            for (int j = 0; j < NR; j++) {
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const uint32_t sa = (uint32_t)src[j][k];
                    const uint32_t pw = xc_lds_volatile(S_pend + (((sa >> 7) & (XC_PROWS - 1u)) << 4) + ((sa & 3u) << 2));
                    const bool ready = ((pend[j] >> k) & 1u) != 0u && ((pw >> ((sa >> 2) & 31u)) & 1u) == 0u;
                    const uint32_t v = lds8(S + (ready ? sa : a0[j] + (uint32_t)k));
                    const uint32_t m = 0xFFu << (8 * k);
                    word[j] = ready ? ((word[j] & ~m) | (v << (8 * k))) : word[j];
                    pend[j] &= ready ? ~(1u << k) : 0xFFFFFFFFu;
                    changed = changed || ready;
                }
                sts32(S + a0[j], word[j]);
            }
            publish = __any_sync(0xffffffffu, changed);
            if (++spins > XC_SPIN_LIMIT) return false;
        }
    } else __syncwarp();
    // ---- publish: nothing of these rows is pending any more
    if (lane < 4) {
        xc_fence_cta();
#pragma unroll
        for (int j = 0; j < NR; j++) sts32(S_pend + (((r0 + (uint32_t)j * XC_WARPS) & (XC_PROWS - 1u)) << 4) + (lane << 2), 0u);
    }
    return true;
}

// xc_rows for a block's variant (bit 0: FAR, bit 1: LITG); `lo` = first row of the sub-phase
template <int NR>
__device__ __forceinline__ bool xc_rows_of(uint32_t variant, const XcBlk &B, uint32_t r0, uint32_t lo, bool has_ovl, uint32_t lane) {
    switch (variant) {
        case 0: return xc_rows<false, false, NR>(B, r0, lo << 7, has_ovl, lane);
        case 1: return xc_rows<true, false, NR>(B, r0, lo << 7, has_ovl, lane);
        case 2: return xc_rows<false, true, NR>(B, r0, lo << 7, has_ovl, lane);
        default: return xc_rows<true, true, NR>(B, r0, lo << 7, has_ovl, lane);
    }
}

// registers a thread carries from the record loads of a batch to its build step: XC_PER_THREAD consecutive records,
// and (lane 0 only) the record before the warp's first
struct XcLoad { uint32_t out[XC_PER_THREAD], lit[XC_PER_THREAD], of[XC_PER_THREAD], p_out, p_lit; };

__device__ __forceinline__ XcLoad xc_load(const XcBlk &B, uint32_t k, uint32_t tid, uint32_t lane) {
    XcLoad L;
    const uint32_t i0 = k * XC_BATCH + tid * XC_PER_THREAD;
#pragma unroll
    for (uint32_t q = 0; q < XC_PER_THREAD; q++) {
        const uint32_t i = i0 + q;
        L.out[q] = 0; L.lit[q] = 0; L.of[q] = 0;
        // (past the read-only data path: a raw-offset block's records were rewritten by this kernel a moment ago)
        if (i < B.nseq) { const uint32_t *p = B.seqs + (uint64_t)i * 3; L.out[q] = ld_cg_u32(p); L.lit[q] = ld_cg_u32(p + 1); L.of[q] = ld_cg_u32(p + 2); }
        else if (i < B.ntot) { L.out[q] = B.out_size; L.lit[q] = B.regen; }   // trailing literals (sequence_execution.rs:40-44)
    }
    L.p_out = 0; L.p_lit = 0;
    // (no shuffle here: the loads stay in flight while the rows of the previous batch are produced)
    if (lane == 0 && i0 != 0 && i0 <= B.nseq) { const uint32_t *p = B.seqs + (uint64_t)(i0 - 1) * 3; L.p_out = ld_cg_u32(p); L.p_lit = ld_cg_u32(p + 1); }
    return L;
}

// publishes one sequence (record, end bit, chunk owners); validates what the rows rely on
__device__ __forceinline__ void xc_build_one(const XcBlk &B, uint32_t k, uint32_t i, uint32_t cur_out, uint32_t cur_lit, uint32_t of, uint32_t p_out, uint32_t p_lit,
                                             volatile XcMisc *misc) {
    const uint32_t S = B.S, S_mask = S + XC_OFF_MASK, S_first = S + XC_OFF_FIRST, S_ring = S + XC_OFF_RING;
    if (i > B.ntot) return;
    if (i == B.ntot) {
        // sentinel: bytes of the last row beyond the block copy themselves (never a match, literal delta 0)
        const uint2 rec = xc_pack(0x3FFFFu, 0u, 1u);
        sts64(S_ring + ((i & (XC_RING - 1u)) << 3), rec.x, rec.y);
        for (uint32_t c = (B.a_end + 63u) >> 6; c < B.nrows * 2u; c++) sts32(S_first + (c << 2), i);
        misc->end_a[k & 1u] = B.a_end;
        return;
    }
    const bool real = i < B.nseq;
    const uint32_t ll = cur_lit - p_lit, start = p_out, end = cur_out;
    const uint32_t mstart = start + ll;
    const uint32_t ml = end - mstart;
    const uint32_t off = real ? seq_sym_resolve(of, B.h0, B.h1, B.h2) : 1u;
    // everything the rows rely on: positions inside the block, literals inside the literal buffer, offsets inside the
    // frame's earlier output.  (Zero offsets, dictionary reach, offsets beyond the buffer: the warp kernel reports
    // ExecuteSequencesError / DecodeBufferError exactly as the reference does.)
    bool bad = end > B.out_size || end <= start || mstart > end || cur_lit > B.regen || cur_lit < p_lit;
    if (real) bad = bad || off == 0u || off >= (1u << 28) || (uint64_t)off > B.reach + mstart || ml < 3u;
    if (bad) { misc->bail = 1u; return; }
    if (off < ml) misc->ovl[k & 3u] = 1u;
    const uint32_t start_a = B.woff + start, end_a = B.woff + end;
    // literal j of the block sits at shared offset lit_s + j; literal byte at window position a is literal number
    // (a - woff) - (match bytes before this sequence) = a - woff - (mstart - cur_lit)
    const uint32_t lz = (B.lit_gp ? XC_LITG_BIAS : B.lit_s) + cur_lit - B.woff - mstart;
    const uint2 rec = xc_pack(B.woff + mstart, lz, off);
    sts64(S_ring + ((i & (XC_RING - 1u)) << 3), rec.x, rec.y);
    red_or_shared(S_mask + (((end_a - 1u) >> 5) << 2), 1u << ((end_a - 1u) & 31u));
    const uint32_t c_lo = i == 0 ? 0u : (start_a + 63u) >> 6, c_hi = (end_a - 1u) >> 6;
    for (uint32_t c = c_lo; c <= c_hi; c++) sts32(S_first + (c << 2), i);
    if (i + 1 == (k + 1) * XC_BATCH) misc->end_a[k & 1u] = end_a;   // the batch's last sequence (a later batch exists: the sentinel)
}

__device__ __forceinline__ void xc_build(const XcBlk &B, uint32_t k, uint32_t tid, const XcLoad &L, volatile XcMisc *misc) {
    const uint32_t i0 = k * XC_BATCH + tid * XC_PER_THREAD;
    // the record before my first: the last record of the lane below, or (lane 0) loaded by xc_load
    uint32_t p_out = __shfl_up_sync(0xffffffffu, L.out[XC_PER_THREAD - 1], 1), p_lit = __shfl_up_sync(0xffffffffu, L.lit[XC_PER_THREAD - 1], 1);
    if ((tid & 31u) == 0) { p_out = L.p_out; p_lit = L.p_lit; }
#pragma unroll
    for (uint32_t q = 0; q < XC_PER_THREAD; q++) {
        xc_build_one(B, k, i0 + q, L.out[q], L.lit[q], L.of[q], p_out, p_lit, misc);
        p_out = L.out[q]; p_lit = L.lit[q];
    }
}

// all pending planes = "pending": done between phases (everything below the next phase's first row is final and is never looked up)
__device__ __forceinline__ void xc_planes_reset(uint32_t S, uint32_t tid) {
    for (uint32_t j = tid; j < XC_PROWS * 4u / 2u; j += XC_THREADS) sts64(S + XC_OFF_PEND + (j << 3), 0xFFFFFFFFu, 0xFFFFFFFFu);
}

__global__ void __launch_bounds__(XC_THREADS, 1) k_exec_cta(const BlockDesc *__restrict__ descs, const BlockAux *__restrict__ aux,
                                                            const FrameDesc *__restrict__ frames, FrameState *__restrict__ states,
                                                            const uint8_t *__restrict__ input, const uint8_t *__restrict__ lit_scratch,
                                                            const uint32_t *__restrict__ seq_scratch, uint8_t *__restrict__ output, uint64_t output_cap,
                                                            const uint32_t *__restrict__ cta_frames, uint32_t n_cta_frames,
                                                            uint32_t *__restrict__ resume, uint32_t *__restrict__ ticket) {
    extern __shared__ __align__(128) uint8_t xc_smem[];
    const uint32_t S = (uint32_t)__cvta_generic_to_shared(xc_smem);
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    volatile XcMisc *misc = reinterpret_cast<volatile XcMisc *>(xc_smem + XC_OFF_MISC);
    const uint32_t S_mbar = S + XC_OFF_MISC;   // XcMisc::mbar is the first member
    if (tid == 0) {
        xc_mbar_init(S_mbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    uint32_t lit_parity = 0;

    for (;;) {
        if (tid == 0) misc->ticket = atomicAdd(ticket, 1u);
        __syncthreads();
        const uint32_t t = misc->ticket;
        __syncthreads();
        if (t >= n_cta_frames) break;
        const uint32_t f = cta_frames[t];
        const FrameDesc &fd = frames[f];
        const FrameState fs = states[f];
        uint32_t h0 = fs.hist[0], h1 = fs.hist[1], h2 = fs.hist[2];
        uint64_t produced = fs.produced, counter = fs.counter;
        const uint64_t drained = fs.drained;
        const uint64_t cap = frame_out_room(fd, output_cap);
        uint8_t *out = output + fd.out_off;
        uint32_t blocks_done = fs.blocks_done;
        const uint32_t nblocks = fd.nblocks;
        bool bailed = fs.status != 0 || fd.dict != nullptr;
        uint32_t why = bailed ? XC_WHY_FRAME_STATE : 0u;   // debug: why the frame was handed to k_exec (ticket[2] collects the OR, ticket[1] the count)
        bool fresh = true;   // no block of this frame has been stored by this CTA yet
        uint32_t bi = 0;
        for (; bi < nblocks && !bailed; bi++) {
            const uint32_t b = fd.first_block + bi;
            const BlockDesc &d = descs[b];
            const BlockAux &ax = aux[b];
            if (d.host_status || ax.status) { bailed = true; why |= XC_WHY_ERROR; break; }
            if (d.btype != BT_COMPRESSED) {
                const uint32_t n = d.raw_size;
                if (produced + n > cap) { bailed = true; why |= XC_WHY_CAPACITY; break; }
                raw_rle_block(out + produced, d, input, tid, XC_THREADS);
                produced += n;   // extend_from_reader: total_output_counter untouched (decode_buffer.rs:66-72)
                blocks_done++;
                fresh = false;
                __syncthreads();
                continue;
            }
            const uint32_t nseq = d.nseq;
            if (nseq && (ax.seq_status || (ax.flags & AUX_WIDE))) { bailed = true; why |= ax.seq_status ? XC_WHY_ERROR : XC_WHY_SEQ_RECORDS; break; }
            if (nseq && (ax.flags & AUX_RAW_OFFSETS)) {
                // k_fse's exact path left raw offset_values (a sequence with more extra bits than its fast path takes, an offset
                // code >= 30, ...).  do_offset_history (sequence_execution.rs:59-118) is a serial walk: warp 0 runs it over the block's
                // records, 32 at a time, and rewrites them in place as resolved offsets -- after which the block is an ordinary one,
                // for this kernel and (flag cleared, history stored) for k_exec should a later check hand the frame back.
                uint32_t *sq = const_cast<uint32_t *>(seq_scratch) + d.seq_buf_off * 3;
                uint32_t big = (h0 | h1 | h2) >> SEQ_SYM_SHIFT;   // values >= 2^30 cannot be told from symbols afterwards
                for (uint32_t i = tid; i < nseq; i += XC_THREADS) big |= sq[3 * i + 2] >> SEQ_SYM_SHIFT;
                if (__syncthreads_or((int)big)) { bailed = true; why |= XC_WHY_SEQ_RECORDS; break; }
                if (warp == 0) {
                    uint32_t a0 = h0, a1 = h1, a2 = h2, prev_lit = 0;
                    for (uint32_t base = 0; base < nseq; base += 32) {
                        const uint32_t i = base + lane, n = min(32u, nseq - base);
                        const uint32_t of = i < nseq ? sq[3 * i + 2] : 0u, lit = i < nseq ? sq[3 * i + 1] : 0u;
                        uint32_t plit = __shfl_up_sync(0xffffffffu, lit, 1);
                        if (lane == 0) plit = prev_lit;
                        const uint32_t ll = lit - plit;
                        uint32_t mine = 0;
                        for (uint32_t j = 0; j < n; j++) {
                            const uint32_t actual = offset_history_step(__shfl_sync(0xffffffffu, of, j), __shfl_sync(0xffffffffu, ll, j), a0, a1, a2);
                            if (lane == j) mine = actual;
                        }
                        if (i < nseq) sq[3 * i + 2] = mine;
                        prev_lit = __shfl_sync(0xffffffffu, lit, n - 1);
                    }
                    if (lane == 0) {
                        BlockAux *axw = const_cast<BlockAux *>(aux) + b;
                        axw->hist_after[0] = a0; axw->hist_after[1] = a1; axw->hist_after[2] = a2;   // concrete values (< 2^30): resolve to themselves
                        axw->flags = ax.flags & ~AUX_RAW_OFFSETS;
                    }
                }
                __threadfence();
                __syncthreads();
            }
            const uint32_t out_size = ax.out_size, regen = d.regen_size;
            const uint32_t sum_ll = nseq ? ax.sum_ll : 0u;
            if (out_size > XC_WIN_MAX || produced + out_size > cap || sum_ll > regen || regen > out_size) { bailed = true; why |= produced + out_size > cap ? XC_WHY_CAPACITY : XC_WHY_BLOCK_SIZE; break; }
            if (out_size == 0) { blocks_done++; continue; }
            XcBlk B;
            B.S = S;
            B.gout = out + produced;
            B.woff = (uint32_t)((uintptr_t)B.gout & 15u);
            B.a_end = B.woff + out_size;
            const uint32_t wbytes = (B.a_end + 127u) & ~127u;
            B.nrows = wbytes >> 7;
            B.nseq = nseq; B.ntot = nseq + (regen > sum_ll ? 1u : 0u);
            B.out_size = out_size; B.regen = regen;
            B.h0 = h0; B.h1 = h1; B.h2 = h2;
            B.reach = produced - drained;
            B.seqs = seq_scratch + d.seq_buf_off * 3;
            // ---- literals: where they come from, how they are staged
            const uint32_t lt = d.lit_type;
            const uint8_t *lit_g = nullptr;
            uint32_t loff = 0;
            if (lt == LT_RAW) { const uint8_t *p = input + d.src_off + d.lit_off; loff = (uint32_t)((uintptr_t)p & 15u); lit_g = p - loff; }
            else if (lt != LT_RLE) lit_g = lit_scratch + d.lit_buf_off;
            const uint32_t lit_bytes = (loff + regen + 15u) & ~15u;
            // literals that do not fit beside the window are read from global memory byte by byte (a block that is nearly all literals)
            const bool litg = wbytes + lit_bytes > XC_DATA_BYTES;
            if (litg && lt == LT_RLE) { bailed = true; why |= XC_WHY_RLE_LITERALS; break; }
            B.lit_gp = litg ? lit_g + loff : nullptr;
            B.lit_s = wbytes + loff;
            const bool has_far = B.reach != 0;
            // ---- the window and the literal area are free once the previous block's bulk stores have read them; a block
            // that may read earlier output of its frame also needs those stores to be complete in global memory
            if (tid == 0) { if (has_far && !fresh) xc_bulk_wait0(); else xc_bulk_wait_read0(); }
            for (uint32_t j = tid; j < XC_MASK_BYTES / 16; j += XC_THREADS) sts128(S + XC_OFF_MASK + (j << 4), 0u, 0u, 0u, 0u);
            if (tid == 0) { misc->bail = 0; misc->ovl[0] = 0; misc->ovl[1] = 0; misc->ovl[2] = 0; misc->ovl[3] = 0; misc->end_a[0] = 0; misc->end_a[1] = 0; }
            __syncthreads();
            const bool tma_lit = lt != LT_RLE && regen != 0 && !litg;
            if (tma_lit) {
                if (tid == 0) {
                    xc_mbar_expect_tx(S_mbar, lit_bytes);
                    for (uint32_t o = 0; o < lit_bytes; o += 32768u) xc_bulk_g2s(S + wbytes + o, lit_g + o, min(32768u, lit_bytes - o), S_mbar);
                }
            } else if (lt == LT_RLE) {
                const uint32_t v = input[d.src_off + d.lit_off] * 0x01010101u;
                for (uint32_t j = tid; j < lit_bytes / 16; j += XC_THREADS) sts128(S + wbytes + (j << 4), v, v, v, v);
            }
            const uint32_t nbatch = (B.ntot + 1u + XC_BATCH - 1u) / XC_BATCH;
            {
                const XcLoad L0 = xc_load(B, 0, tid, lane);
                xc_build(B, 0, tid, L0, misc);
                xc_planes_reset(S, tid);
            }
            __syncthreads();
            bool blk_bail = misc->bail != 0;
            if (tma_lit) {   // also when bailing out: the copy must have landed before the barrier / the area are used again
                uint32_t spins = 0;
                while (!xc_mbar_try_wait(S_mbar, lit_parity)) { if (++spins > XC_SPIN_LIMIT) { misc->bail = 2u; break; } }
                lit_parity ^= 1u;
            }
            uint32_t row_lo = 0, stored_a = (B.woff + 15u) & ~15u;
            for (uint32_t k = 0; k < nbatch && !blk_bail; k++) {
                const bool last = k + 1 == nbatch;
                XcLoad Ln;
                if (!last) Ln = xc_load(B, k + 1, tid, lane);
                const uint32_t row_hi = last ? B.nrows : (misc->end_a[k & 1u] >> 7);
                const bool has_ovl = (misc->ovl[k & 3u] | misc->ovl[(k + 3u) & 3u]) != 0u;
                if (tid == 0) misc->ovl[(k + 2u) & 3u] = 0u;
                bool ok = true;
                // sub-phases of at most XC_PROWS rows (their pending planes are all-ones when they start, everything below is final)
                for (uint32_t lo = row_lo; lo < row_hi; lo += XC_PROWS) {
                    const uint32_t hi = min(lo + XC_PROWS, row_hi);
                    if (lo != row_lo) { __syncthreads(); xc_planes_reset(S, tid); __syncthreads(); }
                    uint32_t r = lo + warp;
                    const uint32_t variant = (has_far ? 1u : 0u) | (litg ? 2u : 0u);
                    for (; r + XC_WARPS < hi && ok; r += 2 * XC_WARPS) ok = xc_rows_of<2>(variant, B, r, lo, has_ovl, lane);
                    if (r < hi && ok) ok = xc_rows_of<1>(variant, B, r, lo, has_ovl, lane);
                }
                if (!ok && lane == 0) misc->bail = 2u;
                xc_fence_proxy_async();
                __syncthreads();   // the rows of this batch are final; nobody reads the previous batch's records any more
                row_lo = row_hi;
                // ---- rows below row_hi are final: send the aligned part to global memory while the next batch runs
                uint32_t hi_a = min(row_hi << 7, B.a_end) & ~15u;
                if (misc->bail == 0 && hi_a > stored_a) {
                    if (tid == 0) {
                        for (uint32_t o = stored_a; o < hi_a; o += 32768u) xc_bulk_s2g(B.gout + (o - B.woff), S + o, min(32768u, hi_a - o));
                        xc_bulk_commit();
                    }
                    stored_a = hi_a;
                }
                if (!last) {
                    xc_planes_reset(S, tid);
                    xc_build(B, k + 1, tid, Ln, misc);
                    __syncthreads();
                }
                blk_bail = misc->bail != 0;
            }
            if (blk_bail) { bailed = true; why |= misc->bail == 2u ? XC_WHY_TIMEOUT : XC_WHY_SEQ_CHECK; break; }
            // ---- head / tail bytes around the 16-byte aligned part
            {
                const uint32_t head_end = min((B.woff + 15u) & ~15u, B.a_end);
                const uint32_t tail_beg = max((B.woff + 15u) & ~15u, B.a_end & ~15u);
                if (tid < 16) { const uint32_t a = B.woff + tid; if (a < head_end) B.gout[a - B.woff] = (uint8_t)lds8(S + a); }
                else if (tid < 32) { const uint32_t a = tail_beg + (tid - 16u); if (a < B.a_end) B.gout[a - B.woff] = (uint8_t)lds8(S + a); }
            }
            if (nseq) block_hist_after(ax, h0, h1, h2, h0, h1, h2);
            produced += out_size; counter += out_size;
            blocks_done++;
            fresh = false;
            __syncthreads();   // head/tail reads of the window are done before the next block's prologue touches it
        }
        if (tid == 0) {
            FrameState &o = states[f];
            if (fs.status == 0) {
                o.hist[0] = h0; o.hist[1] = h1; o.hist[2] = h2;
                o.produced = produced; o.counter = counter; o.blocks_done = blocks_done;
            }
            // what is left for k_exec: the rest of the frame from block `bi`, or only the frame-level epilogue, or nothing
            resume[f] = bailed ? bi : (fd.host_status ? nblocks : nblocks + 1u);
            if (bailed) { atomicAdd(ticket + 1, 1u); atomicOr(ticket + 2, why); atomicAdd(ticket + 3, nblocks - bi); }
        }
    }
    if (tid == 0) xc_bulk_wait0();
}

}  // namespace b200z
