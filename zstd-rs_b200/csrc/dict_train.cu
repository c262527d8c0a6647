// dict_train.cu -- sm_90a kernels of the raw-content dictionary trainer (b200z_dict_train_raw; DESIGN.md section 4.5).
//
//   k_dtcount : one CTA per 4096 positions: the slot of every position's 16-byte k-mer, and the count of every slot
//   k_dtprev  : one CTA per 2048 positions: the distance back to the nearest earlier position with the same slot
//   k_dtepoch : one launch per epoch, one CTA per 4096 segment starts: every start's score, the best start, and (the CTA
//               that finishes last) the segment's record and the zeroing of its slots' counts
//
// Every kernel uses integer work and atomics only, so the dictionary does not depend on the schedule.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dict_train.h"

namespace b200z {

constexpr uint32_t DC_TILE = 4096, DC_THREADS = 256;
constexpr uint32_t DP_TILE = 2048, DP_THREADS = 256;
constexpr uint32_t DE_TILE = 4096, DE_THREADS = 512, DE_PER = DE_TILE / DE_THREADS;

__device__ __forceinline__ uint32_t dt_slot(const uint8_t *b) {
    uint64_t lo = 0, hi = 0;
#pragma unroll
    for (int j = 7; j >= 0; j--) {
        lo = (lo << 8) | b[j];
        hi = (hi << 8) | b[8 + j];
    }
    const uint64_t m = hi * 0xC2B2AE3D27D4EB4Full;
    const uint64_t x = (lo * 0x9E3779B185EBCA87ull) ^ ((m << 31) | (m >> 33));
    return (uint32_t)((x * 0x9E3779B185EBCA87ull) >> (64 - DT_F));
}

// ------------------------------------------------------------------------------------------------------------
// k_dtcount.  The CTA stages its 4096 positions and the 15 bytes after them, finds the sample holding its first position by
// binary search over the samples' offsets, and walks forward from there: each sample that starts before the tile's end takes
// the slot away from its last 15 positions.  Lanes of a warp that share a slot add their count once (match_any), so a run of
// one k-mer (all-zero input) costs one atomic per warp rather than 32 on one address.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(DC_THREADS)
k_dtcount(const uint8_t *__restrict__ in, uint32_t n, const uint32_t *__restrict__ starts, uint32_t nsamples, uint32_t *__restrict__ slots,
          uint32_t *__restrict__ freq) {
    __shared__ uint8_t s_in[DC_TILE + DT_K];
    __shared__ uint8_t s_ok[DC_TILE];
    __shared__ uint32_t s_k0;
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const uint32_t t0 = blockIdx.x * DC_TILE, tn = min(DC_TILE, n - t0), tend = t0 + tn;
    for (uint32_t i = tid; i < tn + DT_K - 1 && (uint64_t)t0 + i < n; i += DC_THREADS) s_in[i] = __ldg(in + t0 + i);
    for (uint32_t i = tid; i < DC_TILE; i += DC_THREADS) s_ok[i] = 1;
    if (tid == 0) {   // the last sample that starts at or before t0
        uint32_t lo = 0, hi = nsamples - 1;
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1) >> 1;
            if (__ldg(starts + mid) <= t0) lo = mid; else hi = mid - 1;
        }
        s_k0 = lo;
    }
    __syncthreads();
    for (uint32_t k = s_k0 + tid; k < nsamples && __ldg(starts + k) < tend; k += DC_THREADS) {
        const uint32_t a = __ldg(starts + k), b = __ldg(starts + k + 1);
        const uint32_t lo = max(max(a, b >= DT_K - 1 ? b - (DT_K - 1) : 0u), t0), hi = min(b, tend);
        for (uint32_t p = lo; p < hi; p++) s_ok[p - t0] = 0;
    }
    __syncthreads();
    for (uint32_t i = tid; i < DC_TILE; i += DC_THREADS) {   // the same trip count for every lane of the warp
        const uint32_t h = i < tn && s_ok[i] ? dt_slot(s_in + i) : DT_NO_SLOT;
        if (i < tn) slots[t0 + i] = h;
        const uint32_t peers = __match_any_sync(0xffffffffu, h);
        if (h != DT_NO_SLOT && lane == (uint32_t)__ffs(peers) - 1) atomicAdd(freq + h, (uint32_t)__popc(peers));
    }
}

// ------------------------------------------------------------------------------------------------------------
// k_dtprev.  The CTA sorts its 2048 (slot, position) pairs in shared memory (bitonic), so a position's nearest earlier
// same-slot position inside the tile is its predecessor in the sorted order.  For the first position of each slot run, the
// nearest one lies in the halo: the w - 1 positions before the tile.  Each halo position binary-searches its slot in the sorted
// tile and raises that run's latest halo position (atomicMax).  Distances beyond w - 1 are written as 0 (none).
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(DP_THREADS)
k_dtprev(const uint32_t *__restrict__ slots, uint32_t n, uint32_t w, uint16_t *__restrict__ dist) {
    __shared__ unsigned long long key[DP_TILE];
    __shared__ uint32_t near[DP_TILE];   // per sorted entry: 1 + the latest halo position with the entry's slot (0: none)
    const uint32_t tid = threadIdx.x;
    const uint32_t t0 = blockIdx.x * DP_TILE, tn = min(DP_TILE, n - t0);
    for (uint32_t i = tid; i < DP_TILE; i += DP_THREADS) {
        const uint32_t h = i < tn ? __ldg(slots + t0 + i) : DT_NO_SLOT;
        key[i] = ((unsigned long long)h << 32) | i;
        near[i] = 0;
    }
    __syncthreads();
    for (uint32_t k = 2; k <= DP_TILE; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t q = tid; q < DP_TILE / 2; q += DP_THREADS) {
                const uint32_t i = ((q & ~(j - 1)) << 1) | (q & (j - 1)), ixj = i + j;
                const unsigned long long a = key[i], b = key[ixj];
                if ((a > b) == ((i & k) == 0)) { key[i] = b; key[ixj] = a; }
            }
            __syncthreads();
        }
    }
    const uint32_t h0 = t0 > w - 1 ? t0 - (w - 1) : 0;
    for (uint32_t q = h0 + tid; q < t0; q += DP_THREADS) {
        const uint32_t h = __ldg(slots + q);
        if (h == DT_NO_SLOT) continue;
        const unsigned long long want = (unsigned long long)h << 32;
        uint32_t lo = 0, hi = DP_TILE;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (key[mid] < want) lo = mid + 1; else hi = mid;
        }
        if (lo < DP_TILE && (uint32_t)(key[lo] >> 32) == h) atomicMax(near + lo, q + 1);
    }
    __syncthreads();
    for (uint32_t i = tid; i < DP_TILE; i += DP_THREADS) {
        const unsigned long long k = key[i];
        const uint32_t h = (uint32_t)(k >> 32), p = (uint32_t)k;
        if (p >= tn) continue;
        uint32_t d = 0;
        if (h != DT_NO_SLOT) {
            if (i > 0 && (uint32_t)(key[i - 1] >> 32) == h) d = p - (uint32_t)key[i - 1];
            else if (near[i]) d = t0 + p - (near[i] - 1);
        }
        dist[t0 + p] = (uint16_t)(d <= w - 1 ? d : 0);
    }
}

// ------------------------------------------------------------------------------------------------------------
// k_dtepoch.  A position p with a slot adds freq[slot(p)] to every start s of [max(prev(p) + 1, p - we + 1), min(p, e1 - le)]
// (we = le - 15 k-mers per segment): the starts whose window holds p and no earlier position of the same slot.  A prev before e0
// or more than we - 1 back bounds nothing the other two bounds do not, so dist can be applied as it stands.  The CTA scatters
// its tile's contributions into a shared difference array (u64 atomics), scans it, and reduces (score << 32 | ~s): the largest
// score, then the smallest start.  A score is at most the number of positions, below 2^32.  The CTA that finishes last reads
// the epoch's winner, writes its record and zeroes the counts of its slots, so the next epoch's launch sees them gone.
// Positions fit in 32 bits (n < 2^32), but a tile's last start and a loop counter one stride past n - 16 need not: those are
// 64-bit.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(DE_THREADS)
k_dtepoch(const uint32_t *__restrict__ slots, const uint16_t *__restrict__ dist, uint32_t *__restrict__ freq, uint32_t epoch, uint32_t e0,
          uint32_t e1, uint32_t le, unsigned long long *__restrict__ best, uint32_t *__restrict__ done, b200z_dict_segment *__restrict__ seg) {
    __shared__ unsigned long long diff[DE_TILE + 1];
    __shared__ unsigned long long s_warp[DE_THREADS / 32];
    __shared__ bool s_last;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t we = le - (DT_K - 1), smax = e1 - le;
    const uint32_t s0 = e0 + blockIdx.x * DE_TILE, s1 = (uint32_t)min((uint64_t)s0 + DE_TILE - 1, (uint64_t)smax);
    for (uint32_t i = tid; i <= DE_TILE; i += DE_THREADS) diff[i] = 0;
    __syncthreads();
    for (uint64_t pp = (uint64_t)s0 + tid; pp <= (uint64_t)s1 + we - 1; pp += DE_THREADS) {
        const uint32_t p = (uint32_t)pp;
        const uint32_t h = __ldg(slots + p);
        if (h == DT_NO_SLOT) continue;
        const uint32_t f = freq[h];
        if (!f) continue;
        uint32_t lo = max(p >= we - 1 ? p - (we - 1) : 0u, s0);
        const uint32_t d = __ldg(dist + p);
        if (d) lo = max(lo, p - d + 1);
        const uint32_t hi = min(p, s1);
        if (lo > hi) continue;
        atomicAdd(diff + (lo - s0), (unsigned long long)f);
        atomicAdd(diff + (hi - s0 + 1), 0ull - f);
    }
    __syncthreads();
    unsigned long long v[DE_PER], sum = 0;
#pragma unroll
    for (uint32_t j = 0; j < DE_PER; j++) { sum += diff[tid * DE_PER + j]; v[j] = sum; }
    unsigned long long x = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= (uint32_t)o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    unsigned long long off = x - sum;
    for (uint32_t i = 0; i < warp; i++) off += s_warp[i];
    unsigned long long m = 0;
#pragma unroll
    for (uint32_t j = 0; j < DE_PER; j++) {
        const uint64_t s = (uint64_t)s0 + tid * DE_PER + j;
        if (s <= s1) m = max(m, ((off + v[j]) << 32) | (0xffffffffu - (uint32_t)s));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    __syncthreads();
    if (lane == 0) s_warp[warp] = m;
    __syncthreads();
    if (tid == 0) {
        for (uint32_t i = 1; i < DE_THREADS / 32; i++) m = max(m, s_warp[i]);
        atomicMax(best, m);
        __threadfence();
        s_last = atomicAdd(done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    const unsigned long long k = *(volatile unsigned long long *)best;
    const uint32_t s = 0xffffffffu - (uint32_t)k;
    if (tid == 0) {
        b200z_dict_segment r;
        r.src_off = s; r.score = k >> 32; r.epoch = epoch; r.size = le;
        *seg = r;
    }
    for (uint64_t p = (uint64_t)s + tid; p < (uint64_t)s + we; p += DE_THREADS) {
        const uint32_t h = __ldg(slots + p);
        if (h != DT_NO_SLOT) freq[h] = 0;
    }
}

static uint32_t cdiv_u(uint64_t a, uint32_t b) { return (uint32_t)((a + b - 1) / b); }

static int counted(uint64_t *launched) {
    const int e = (int)cudaGetLastError();
    if (!e) ++*launched;
    return e;
}

int launch_dt_count(const uint8_t *in, uint32_t n, const uint32_t *starts, uint32_t nsamples, uint32_t *slots, uint32_t *freq, cudaStream_t s,
                    uint64_t *launched) {
    k_dtcount<<<cdiv_u(n, DC_TILE), DC_THREADS, 0, s>>>(in, n, starts, nsamples, slots, freq);
    return counted(launched);
}

int launch_dt_prev(const uint32_t *slots, uint32_t n, uint32_t w, uint16_t *dist, cudaStream_t s, uint64_t *launched) {
    k_dtprev<<<cdiv_u(n, DP_TILE), DP_THREADS, 0, s>>>(slots, n, w, dist);
    return counted(launched);
}

int launch_dt_epoch(const uint32_t *slots, const uint16_t *dist, uint32_t *freq, uint32_t epoch, uint32_t e0, uint32_t e1, uint32_t le,
                    unsigned long long *best, uint32_t *done, b200z_dict_segment *seg, cudaStream_t s, uint64_t *launched) {
    k_dtepoch<<<cdiv_u((uint64_t)(e1 - le - e0) + 1, DE_TILE), DE_THREADS, 0, s>>>(slots, dist, freq, epoch, e0, e1, le, best, done, seg);
    return counted(launched);
}

}  // namespace b200z
