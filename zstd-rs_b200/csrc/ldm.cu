// ldm.cu -- sm_90a kernels of the compressor's long-distance matches (window_log > 17; DESIGN.md section 4.11; tests/cldm.py
// states the rule line by line).  They run before k_cmatch over spans of at most one block: the blocks of the frames larger than
// one block (batch), or a stream chunk's blocks and the history kept before it.
//
//   k_lanchor  : one CTA per span, LDM_SPAN positions per thread: the gear hash of the LDM_LEN bytes ending at every position; a
//                position is an anchor when its hash passes the mask and no position in the LDM_QUIET before it passes.
//                <false> counts each thread's anchors and the span's, <true> writes them (key, index, input offset, frame) in
//                position order, at the span's prefix offset plus the thread's within the span
//   k_lscan    : one CTA: exclusive prefix sum of a u32 array in place (4,096 at a time, coalesced), its total after it
//   k_lhist / k_lscatter : one stable LSD radix pass (8 bits) of the (key, anchor index) pairs, LDM_TILE pairs per CTA
//   k_lcand    : per sorted pair, the predecessor with the same key -- the nearest earlier anchor with that key -- when it lies
//                in the same frame at an offset in (ENC_WINDOW, 2^window_log]; <true> (B200Z_FLAG_DICT_LONG): without a
//                predecessor in the frame, the dictionary's last anchor with the key (a binary search of its sorted keys)
//   k_lblock   : one warp per span of a block: verify, extend inside the block, trim to the prefix max of earlier ends,
//                coalesce, and write the block's forced matches for k_cmatch<..., true>; <true>: the source is D || X
//   k_ldict    : per sorted pair of a dictionary's anchors, its key and distance from D's end, kept with the dictionary
// The anchors' total stays on the device (scount[nspans]); grids are sized by the capacity and read it.
//
// ULTRA's far stage (compress.h, tests/cultra.py), per group:
//   k_fkey     : one CTA per piece (a 128 KiB block of the group's virtual space): (key8, virtual position) of every keyed position
//                into the pairs, in position order; the piece's unkeyed tail gets no far walk
//   the sort   : k_lhist / k_lscan / k_lscatter as above, four passes: equal keys stay in position order
//   k_fstart   : per sorted pair (position q), the sorted index of the nearest earlier pair with the same key and q - p > ENC_WINDOW,
//                or FAR_NONE: a backward gallop then a binary search inside the key's run
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "compress.h"

namespace b200z {

constexpr uint32_t LS_THREADS = 256, LS_ROUNDS = LDM_TILE / LS_THREADS;
constexpr uint32_t LSCAN_THREADS = 1024;
constexpr uint64_t LDM_KEY_MUL = 0x9E3779B97F4A7C15ull;

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// the exclusive prefix of v over the CTA's 256 threads (and, to all, their total)
__device__ __forceinline__ uint32_t cta_exclusive(uint32_t v, uint32_t *s_warp, uint32_t *total) {
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t inc = v;
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (uint32_t)o) inc += y;
    }
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    uint32_t before = 0, all = 0;
    for (uint32_t k = 0; k < LDM_THREADS / 32; k++) {
        before += k < w ? s_warp[k] : 0u;
        all += s_warp[k];
    }
    *total = all;
    return before + inc - v;
}

// thread t of span sp owns the anchor positions [p0, p1) = [off + t * LDM_SPAN, + LDM_SPAN) of the span.  It hashes from x0, 78
// bytes before p0 (or the span's `lo`), so that the hashes of the LDM_QUIET positions before p0 are complete; a position whose
// LDM_LEN bytes would start before x0 neither passes nor is an anchor.
template <bool FILL>
__global__ void __launch_bounds__(LDM_THREADS, 4)
k_lanchor(const LSpan *__restrict__ spans, const uint8_t *__restrict__ input, uint32_t *__restrict__ tcount, uint32_t *__restrict__ scount,
          uint32_t *__restrict__ keys, uint32_t *__restrict__ vals, uint64_t *__restrict__ apos, uint32_t *__restrict__ aframe) {
    __shared__ uint64_t gear[256];
    __shared__ uint32_t s_warp[LDM_THREADS / 32];
    const uint32_t tid = threadIdx.x, sp = blockIdx.x;
    gear[tid] = splitmix64(tid);
    const LSpan span = spans[sp];
    uint32_t cnt = 0, at = 0, total = 0;
    if (FILL) at = scount[sp] + cta_exclusive(tcount[(size_t)sp * LDM_THREADS + tid], s_warp, &total);
    __syncthreads();
    const uint64_t p0 = span.off + (uint64_t)tid * LDM_SPAN, p1 = min(span.off + span.size, p0 + LDM_SPAN);
    constexpr uint32_t BACK = LDM_LEN - 1 + LDM_QUIET;
    const uint64_t x0 = p0 - span.lo >= BACK ? p0 - BACK : span.lo;
    uint64_t h = 0;
    uint32_t recent = 0;   // pass bits of the positions before x, the latest in bit 0
    uint32_t word = 0;     // the aligned 4 bytes holding input[x] (a word holding an input byte can be read whatever the alignment)
    for (uint64_t x = x0; x < p1; x++) {
        const uintptr_t a = (uintptr_t)(input + x);
        if ((a & 3) == 0 || x == x0) word = __ldg(reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3));
        h = (h << 1) + gear[(word >> (8 * (a & 3))) & 255u];   // from x0 + LDM_LEN - 1 on: the hash of (x - LDM_LEN, x]
        const bool pass = x >= x0 + LDM_LEN - 1 && (h >> LDM_MASK_SHIFT) == 0;
        if (pass && x >= p0 && (recent & ((1u << LDM_QUIET) - 1)) == 0) {
            if (FILL) {
                keys[at] = (uint32_t)((h * LDM_KEY_MUL) >> 32);
                vals[at] = at;
                apos[at] = x;
                aframe[at] = span.frame;
                at++;
            } else {
                cnt++;
            }
        }
        recent = (recent << 1) | (pass ? 1u : 0u);
    }
    if (!FILL) {
        tcount[(size_t)sp * LDM_THREADS + tid] = cnt;
        cta_exclusive(cnt, s_warp, &total);
        if (tid == 0) scount[sp] = total;
    }
}

// exclusive prefix sum of v[0, n) in place, 4 * LSCAN_THREADS at a time (each thread 4 consecutive values); v[n] = the total
__global__ void __launch_bounds__(LSCAN_THREADS) k_lscan(uint32_t *__restrict__ v, uint32_t n) {
    __shared__ uint32_t s_sum[LSCAN_THREADS / 32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    uint32_t carry = 0;
    for (uint32_t base = 0; base < n; base += 4 * LSCAN_THREADS) {
        const uint32_t i0 = base + 4 * tid;
        uint32_t x[4], sum = 0;
        for (int k = 0; k < 4; k++) { x[k] = i0 + k < n ? v[i0 + k] : 0u; sum += x[k]; }
        uint32_t inc = sum;
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= (uint32_t)o) inc += y;
        }
        if (lane == 31) s_sum[w] = inc;
        __syncthreads();
        if (w == 0) {
            const uint32_t y0 = s_sum[lane];
            uint32_t y = y0;
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t z = __shfl_up_sync(0xffffffffu, y, o);
                if (lane >= (uint32_t)o) y += z;
            }
            s_sum[lane] = y - y0;
        }
        __syncthreads();
        uint32_t run = carry + s_sum[w] + inc - sum;
        for (int k = 0; k < 4; k++) {
            if (i0 + k < n) v[i0 + k] = run;
            run += x[k];
        }
        __syncthreads();
        if (tid == LSCAN_THREADS - 1) s_sum[0] = run;   // the running total after this round
        __syncthreads();
        carry = s_sum[0];
        __syncthreads();
    }
    if (tid == 0) v[n] = carry;
}

// digit counts of tile t, digit-major: hist[d * ntiles + t]; *total pairs in all
__global__ void __launch_bounds__(LS_THREADS)
k_lhist(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ total, uint32_t shift, uint32_t *__restrict__ hist) {
    __shared__ uint32_t cnt[256];
    const uint32_t tid = threadIdx.x, t = blockIdx.x, n = *total;
    cnt[tid] = 0;
    __syncthreads();
    const uint32_t lo = t * LDM_TILE, hi = min(n, lo + LDM_TILE);
    for (uint32_t i = lo + tid; i < hi; i += LS_THREADS) atomicAdd(&cnt[(keys[i] >> shift) & 255u], 1u);
    __syncthreads();
    hist[(size_t)tid * gridDim.x + t] = cnt[tid];
}

// stable scatter of tile t: rounds of LS_THREADS pairs in index order; a pair's place is its digit's base for the tile, plus the
// pairs of that digit in earlier rounds and earlier warps of this round, plus its rank among its warp's lanes
__global__ void __launch_bounds__(LS_THREADS)
k_lscatter(const uint32_t *__restrict__ kin, const uint32_t *__restrict__ vin, const uint32_t *__restrict__ total, uint32_t shift,
           const uint32_t *__restrict__ hist, uint32_t *__restrict__ kout, uint32_t *__restrict__ vout) {
    constexpr uint32_t W = LS_THREADS / 32;
    __shared__ uint32_t base[256], wcnt[W][256];
    const uint32_t tid = threadIdx.x, t = blockIdx.x, lane = tid & 31, w = tid >> 5, n = *total;
    if (t * LDM_TILE >= n) return;
    base[tid] = hist[(size_t)tid * gridDim.x + t];
    for (uint32_t r = 0; r < LS_ROUNDS; r++) {
        const uint32_t i = t * LDM_TILE + r * LS_THREADS + tid;
        const bool valid = i < n;
        const uint32_t k = valid ? kin[i] : 0u, d = valid ? (k >> shift) & 255u : 256u;
        for (uint32_t x = 0; x < W; x++) wcnt[x][tid] = 0;
        __syncthreads();
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const uint32_t rank = __popc(peers & ((1u << lane) - 1));
        if (valid && rank == 0) wcnt[w][d] = __popc(peers);
        __syncthreads();
        uint32_t run = base[tid];
        for (uint32_t x = 0; x < W; x++) {
            const uint32_t c = wcnt[x][tid];
            wcnt[x][tid] = run;
            run += c;
        }
        base[tid] = run;
        __syncthreads();
        if (valid) {
            const uint32_t o = wcnt[w][d] + rank;
            kout[o] = k;
            vout[o] = vin[i];
        }
        __syncthreads();
    }
}

template <bool DICT>
__global__ void __launch_bounds__(256)
k_lcand(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals, const uint32_t *__restrict__ total, const uint64_t *__restrict__ apos,
        const uint32_t *__restrict__ aframe, uint64_t reach, uint32_t *__restrict__ cand, LDict ld) {
    const uint32_t k = blockIdx.x * 256 + threadIdx.x;
    if (k >= *total) return;
    const uint32_t i = vals[k];
    uint32_t c = 0;
    bool near = false;   // an earlier anchor of the frame has the key (in range or not)
    if (k > 0 && keys[k - 1] == keys[k]) {
        const uint32_t j = vals[k - 1];   // the stable sort keeps equal keys in anchor order: j < i
        const uint64_t off = apos[i] - apos[j];
        near = aframe[j] == aframe[i];
        if (aframe[j] == aframe[i] && off > ENC_WINDOW && off <= reach) c = (uint32_t)off;
    }
    if constexpr (DICT) {
        if (!near && ld.n) {   // the dictionary's last pair with the key: the first with a larger key, less one
            const uint32_t key = keys[k];
            uint32_t lo = 0, hi = ld.n;
            while (lo < hi) {
                const uint32_t m = lo + (hi - lo) / 2;
                if (ld.keys[m] <= key) lo = m + 1; else hi = m;
            }
            if (lo && ld.keys[lo - 1] == key) {
                const uint64_t off = apos[i] - ld.frames[aframe[i]].src_off + ld.dist[lo - 1];
                if (off > ENC_WINDOW && off <= reach) c = (uint32_t)off;
            }
        }
    }
    cand[i] = c;
}

// byte x (block-relative) of the source `off` back in the virtual stream D || X: in the frame, or before its start (fb: the frame's
// bytes before the block) at D's end.  Byte loads only: nothing before D's first byte or past its end is read
__device__ __forceinline__ uint8_t ldict_src(const uint8_t *src, uint64_t fb, int32_t x, uint32_t off, const LDictSrc &ds) {
    const int64_t q = (int64_t)fb + x - (int64_t)off;   // the source's position in the frame
    return q >= 0 ? __ldg(src + ((int64_t)x - (int64_t)off)) : __ldg(ds.d + (int64_t)ds.len + q);
}

// one warp per span; spans of history (no block) write nothing.  The span's anchors are scount[sp] up to the next span's first
// (scount[nspans]: the total).  Block-relative positions are signed where a 64-byte window may start
// in the previous block.
template <bool DICT>
__global__ void __launch_bounds__(32)
k_lblock(const LSpan *__restrict__ spans, const uint8_t *__restrict__ input, const uint32_t *__restrict__ scount, const uint64_t *__restrict__ apos,
         const uint32_t *__restrict__ cand, LForced *__restrict__ forced, uint32_t *__restrict__ lf_off, uint32_t *__restrict__ lf_cnt, LDictSrc ds) {
    const uint32_t sp = blockIdx.x, lane = threadIdx.x;
    const LSpan span = spans[sp];
    if (span.block == LDM_NO_BLOCK) return;
    const uint8_t *src = input + span.off;
    const int32_t n = (int32_t)span.size;
    const uint64_t fb = span.off - span.lo;   // bytes of the frame (or kept history) before the block
    const uint32_t a0 = scount[sp], a1 = scount[sp + 1];
    uint32_t nk = 0;
    int32_t maxend = 0;
    LForced last{0, 0, 0};
    for (uint32_t i = a0; i < a1; i++) {
        const uint32_t off = cand[i];
        if (!off) continue;
        const int32_t at = (int32_t)(apos[i] - span.off);   // the anchor: the last byte of its window
        // inside the last kept match at the same offset: its extension ends where that one's did, so trimming removes it
        if (nk && off == last.off && at < (int32_t)(last.start + last.len)) continue;
        const uint8_t *ref = src - off;
        const int32_t w0 = at - (int32_t)LDM_LEN + 1;
        bool eq;
        if constexpr (DICT)
            eq = __ldg(src + w0 + lane) == ldict_src(src, fb, w0 + (int32_t)lane, off, ds) &&
                 __ldg(src + w0 + 32 + lane) == ldict_src(src, fb, w0 + 32 + (int32_t)lane, off, ds);
        else
            eq = __ldg(src + w0 + lane) == __ldg(ref + w0 + lane) && __ldg(src + w0 + 32 + lane) == __ldg(ref + w0 + 32 + lane);
        if (!__all_sync(0xffffffffu, eq)) continue;
        int32_t e = at + 1;
        while (true) {
            const int32_t x = e + (int32_t)lane;
            uint32_t sm;
            if constexpr (DICT) sm = __ballot_sync(0xffffffffu, x >= n || __ldg(src + x) != ldict_src(src, fb, x, off, ds));
            else sm = __ballot_sync(0xffffffffu, x >= n || __ldg(src + x) != __ldg(ref + x));
            if (sm) { e += __ffs(sm) - 1; break; }
            e += 32;
        }
        // backward from the window's start, not below the prefix max of earlier ends (the match is trimmed there anyway), the
        // block's start, nor where the source would leave the frame (DICT: D)
        int32_t lo;
        if constexpr (DICT) lo = max(maxend, off > fb + ds.len ? (int32_t)(off - fb - ds.len) : 0);
        else lo = max(maxend, off > fb ? (int32_t)(off - fb) : 0);
        int32_t s = max(w0, lo);
        while (s > lo) {
            const int32_t x = s - 1 - (int32_t)lane;
            uint32_t sm;
            if constexpr (DICT) sm = __ballot_sync(0xffffffffu, x < lo || __ldg(src + x) != ldict_src(src, fb, x, off, ds));
            else sm = __ballot_sync(0xffffffffu, x < lo || __ldg(src + x) != __ldg(ref + x));
            if (sm) { s -= __ffs(sm) - 1; break; }
            s -= 32;
        }
        s = max(s, lo);
        if (e < s + (int32_t)LDM_LEN) continue;
        if (nk && off == last.off && (uint32_t)s == last.start + last.len) {
            last.len = (uint32_t)e - last.start;
        } else {
            if (nk && lane == 0) forced[a0 + nk - 1] = last;
            last = LForced{(uint32_t)s, (uint32_t)(e - s), off};
            nk++;
        }
        maxend = e;
    }
    if (lane == 0) {
        if (nk) forced[a0 + nk - 1] = last;
        lf_off[span.block] = a0;
        lf_cnt[span.block] = nk;
    }
}

__global__ void __launch_bounds__(256)
k_ldict(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals, const uint32_t *__restrict__ total, const uint64_t *__restrict__ apos,
        uint64_t dlen, uint32_t *__restrict__ dkeys, uint32_t *__restrict__ ddist) {
    const uint32_t k = blockIdx.x * 256 + threadIdx.x;
    if (k >= *total) return;
    dkeys[k] = keys[k];
    ddist[k] = (uint32_t)(dlen - apos[vals[k]]);
}

__global__ void __launch_bounds__(256)
k_fkey(const FPiece *__restrict__ pieces, const uint8_t *__restrict__ input, uint32_t npairs, uint32_t *__restrict__ total,
       uint32_t *__restrict__ keys, uint32_t *__restrict__ vals, uint32_t *__restrict__ start) {
    const FPiece pc = pieces[blockIdx.x];
    if (blockIdx.x == 0 && threadIdx.x == 0) *total = npairs;
    const uint32_t keyed = pc.size >= FAR_KEY ? pc.size - (FAR_KEY - 1) : 0u;
    const uint8_t *src = input + pc.off;
    for (uint32_t x = threadIdx.x; x < pc.size; x += 256) {
        if (x < keyed) {
            uint64_t v = 0;
            for (int k = 0; k < 8; k++) v |= (uint64_t)__ldg(src + x + k) << (8 * k);
            keys[pc.pbase + x] = (uint32_t)((v * LDM_KEY_MUL) >> 32);
            vals[pc.pbase + x] = pc.vbase + x;
        } else {
            start[pc.vbase + x] = FAR_NONE;
        }
    }
}

__global__ void __launch_bounds__(256)
k_fstart(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals, uint32_t npairs, uint32_t *__restrict__ start) {
    const uint32_t k = blockIdx.x * 256 + threadIdx.x;
    if (k >= npairs) return;
    const uint32_t key = keys[k], q = vals[k];
    // past(t): pair t is before q's walk -- another (smaller) key, or the same key at q - p > ENC_WINDOW.  It holds for every t below
    // some T and for none in [T, k); the walk starts at T - 1 when that pair has q's key
    auto past = [&](uint32_t t) { return keys[t] != key || q - vals[t] > ENC_WINDOW; };
    uint32_t hi = k, lo = 0;
    uint64_t step = 1;   // [lo, hi): T lies in (lo, hi], past(lo) when lo < hi
    bool found = false;
    while (hi >= step) {
        const uint32_t t = hi - step;
        if (past(t)) { lo = t; found = true; break; }
        hi = t;
        step <<= 1;
    }
    if (!found) {   // every pair from hi on is within the run and near; below hi only pair 0 .. hi - 1 remain
        if (hi == 0 || !past(0)) { start[q] = FAR_NONE; return; }
        lo = 0;
    }
    while (hi - lo > 1) {   // past(lo), !past(hi) (or hi is where the gallop stopped)
        const uint32_t m = lo + (hi - lo) / 2;
        if (past(m)) lo = m; else hi = m;
    }
    start[q] = keys[lo] == key ? lo : FAR_NONE;
}

static uint32_t cdiv_l(uint64_t a, uint32_t b) { return (uint32_t)((a + b - 1) / b); }
static int counted(uint64_t *launched) {
    const int e = (int)cudaGetLastError();
    if (!e) ++*launched;
    return e;
}

int launch_ldm_count(const LdmArgs &a, cudaStream_t s, uint64_t *launched) {
    k_lanchor<false><<<a.nspans, LDM_THREADS, 0, s>>>(a.spans, a.input, a.tcount, a.scount, nullptr, nullptr, nullptr, nullptr);
    if (int e = counted(launched)) return e;
    k_lscan<<<1, LSCAN_THREADS, 0, s>>>(a.scount, a.nspans);
    return counted(launched);
}

// k_lanchor<true> and the four passes of the key sort over a.cap anchors: the sorted pairs end in keys[0] / vals[0]
static int anchors_sorted(const LdmArgs &a, cudaStream_t s, uint64_t *launched) {
    const uint32_t *total = a.scount + a.nspans;
    k_lanchor<true><<<a.nspans, LDM_THREADS, 0, s>>>(a.spans, a.input, a.tcount, a.scount, a.keys[0], a.vals[0], a.apos, a.aframe);
    if (int e = counted(launched)) return e;
    const uint32_t ntiles = cdiv_l(a.cap, LDM_TILE);
    for (uint32_t pass = 0; pass < 4; pass++) {
        const uint32_t in = pass & 1;
        k_lhist<<<ntiles, LS_THREADS, 0, s>>>(a.keys[in], total, 8 * pass, a.hist);
        if (int e = counted(launched)) return e;
        k_lscan<<<1, LSCAN_THREADS, 0, s>>>(a.hist, ntiles * 256);
        if (int e = counted(launched)) return e;
        k_lscatter<<<ntiles, LS_THREADS, 0, s>>>(a.keys[in], a.vals[in], total, 8 * pass, a.hist, a.keys[in ^ 1], a.vals[in ^ 1]);
        if (int e = counted(launched)) return e;
    }
    return 0;
}

int launch_ldm_match(const LdmArgs &a, cudaStream_t s, uint64_t *launched) {
    const uint32_t *total = a.scount + a.nspans;
    if (a.cap) {
        if (int e = anchors_sorted(a, s, launched)) return e;
        if (a.dict_long) k_lcand<true><<<cdiv_l(a.cap, 256), 256, 0, s>>>(a.keys[0], a.vals[0], total, a.apos, a.aframe, 1ull << a.window_log, a.cand, a.ld);
        else k_lcand<false><<<cdiv_l(a.cap, 256), 256, 0, s>>>(a.keys[0], a.vals[0], total, a.apos, a.aframe, 1ull << a.window_log, a.cand, LDict{});
        if (int e = counted(launched)) return e;
    }
    if (a.dict_long) k_lblock<true><<<a.nspans, 32, 0, s>>>(a.spans, a.input, a.scount, a.apos, a.cand, a.forced, a.lf_off, a.lf_cnt, a.ds);
    else k_lblock<false><<<a.nspans, 32, 0, s>>>(a.spans, a.input, a.scount, a.apos, a.cand, a.forced, a.lf_off, a.lf_cnt, LDictSrc{});
    return counted(launched);
}

int launch_ldm_dict(const LdmArgs &a, uint64_t dlen, uint32_t *keys, uint32_t *dist, cudaStream_t s, uint64_t *launched) {
    if (int e = anchors_sorted(a, s, launched)) return e;
    k_ldict<<<cdiv_l(a.cap, 256), 256, 0, s>>>(a.keys[0], a.vals[0], a.scount + a.nspans, a.apos, dlen, keys, dist);
    return counted(launched);
}

int launch_far_stage(const FarArgs &f, cudaStream_t s, uint64_t *launched) {
    k_fkey<<<f.npieces, 256, 0, s>>>(f.pieces, f.input, f.npairs, f.total, f.keys[0], f.vals[0], f.start);
    if (int e = counted(launched)) return e;
    const uint32_t ntiles = std::max(1u, cdiv_l(f.npairs, LDM_TILE));
    for (uint32_t pass = 0; pass < 4; pass++) {
        const uint32_t in = pass & 1;
        k_lhist<<<ntiles, LS_THREADS, 0, s>>>(f.keys[in], f.total, 8 * pass, f.hist);
        if (int e = counted(launched)) return e;
        k_lscan<<<1, LSCAN_THREADS, 0, s>>>(f.hist, ntiles * 256);
        if (int e = counted(launched)) return e;
        k_lscatter<<<ntiles, LS_THREADS, 0, s>>>(f.keys[in], f.vals[in], f.total, 8 * pass, f.hist, f.keys[in ^ 1], f.vals[in ^ 1]);
        if (int e = counted(launched)) return e;
    }
    k_fstart<<<std::max(1u, cdiv_l(f.npairs, 256)), 256, 0, s>>>(f.keys[0], f.vals[0], f.npairs, f.start);
    return counted(launched);
}

}  // namespace b200z
