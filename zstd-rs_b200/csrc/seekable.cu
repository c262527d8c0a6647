// seekable.cu -- sm_90a kernels of seekable archives (EXTENSION: the zstd seekable format; DESIGN.md section 4.10).
//
//   k_cscan        : one CTA per group of frames, after k_cenc and k_cxxh64: places the group's frames back to back behind the
//                    archive so far (a running total kept on the device) by writing each CFrame's dst_off, and writes each frame's
//                    seek-table entry.  k_cassemble<false> then writes the frames exactly as the batch compressor does.
//   k_cseek        : after the last group: the seek table frame behind the last frame
//   k_range_gather : the read plan's copy pieces, one CTA per piece of at most GATHER_CHUNK bytes
#include <cuda_runtime.h>
#include <stdint.h>

#include "compress.h"
#include "encode.cuh"

namespace b200z {

constexpr uint32_t SCAN_THREADS = 1024;
constexpr uint32_t GATHER_THREADS = 256;

__device__ __forceinline__ void put32(uint8_t *p, uint32_t v) {
    p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24);
}

// ------------------------------------------------------------------------------------------------------------
// k_cscan: an inclusive scan over the group's blocks, in chunks of SCAN_THREADS.  A block counts its header and body as
// k_cassemble writes them (3 + size, 3 + 1 for RLE, 3 + csize for Compressed; every block Raw at Uncompressed), a frame's first
// block also the frame header and its last block the checksum.  A frame's packed offset is the running total before its first
// block; its Compressed_Size is the total after its last block less that offset.  Offsets are archive offsets less `origin`
// (the archive offset of the buffer's byte 0).  Entries go to entries[(first_frame + f) * (8 or 12)] in the table's layout.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SCAN_THREADS, 1)
k_cscan(CFrame *__restrict__ frames, const CBlock *__restrict__ blocks, uint32_t nblocks, const CBlockInfo *__restrict__ res,
        const uint64_t *__restrict__ csum, int level, int checksum, uint32_t dict_id, uint64_t *__restrict__ total, uint64_t origin,
        uint8_t *__restrict__ entries, uint64_t first_frame) {
    __shared__ uint64_t s_warp[SCAN_THREADS / 32];
    __shared__ uint64_t s_run;
    const uint32_t tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const uint32_t esz = checksum ? 12u : 8u;
    if (tid == 0) s_run = *total;
    __syncthreads();
    for (uint32_t b0 = 0; b0 < nblocks; b0 += SCAN_THREADS) {
        const uint32_t b = b0 + tid;
        uint64_t v = 0, src_size = 0;
        uint32_t f = 0;
        bool first = false, last = false;
        if (b < nblocks) {
            const CBlock blk = blocks[b];
            f = blk.frame;
            const uint32_t fb = frames[f].first_block, nb = frames[f].nblocks;
            src_size = frames[f].src_size;
            const uint32_t t = level == 0 ? 0u : res[b].type;
            v = 3 + (t == 0 ? blk.size : t == 1 ? 1u : res[b].csize);
            first = b == fb;
            last = b == fb + nb - 1;
            if (first) v += frame_header_size(src_size, dict_id);
            if (last && checksum) v += 4;
        }
        uint64_t x = v;
        for (uint32_t o = 1; o < 32; o <<= 1) {
            const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[w] = x;
        __syncthreads();
        if (w == 0) {
            uint64_t y = s_warp[lane];
            for (uint32_t o = 1; o < 32; o <<= 1) {
                const uint64_t z = __shfl_up_sync(0xffffffffu, y, o);
                if (lane >= o) y += z;
            }
            s_warp[lane] = y;
        }
        __syncthreads();
        const uint64_t incl = s_run + x + (w ? s_warp[w - 1] : 0);
        if (first) frames[f].dst_off = incl - v - origin;
        __syncthreads();   // a frame's offset is written (in this chunk or an earlier one) before its last block reads it
        if (last) {
            uint8_t *e = entries + (first_frame + f) * esz;
            put32(e, (uint32_t)(incl - origin - frames[f].dst_off));
            put32(e + 4, (uint32_t)src_size);
            if (checksum) put32(e + 8, (uint32_t)csum[f]);
        }
        if (tid == SCAN_THREADS - 1) s_run = incl;
        __syncthreads();
    }
    if (tid == 0) *total = s_run;
}

// ------------------------------------------------------------------------------------------------------------
// k_cseek: the seek table frame at archive offset *total (output + *total - origin): the skippable frame's header, the n
// entries k_cscan wrote, the footer.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_cseek(const uint8_t *__restrict__ entries, uint64_t n, int checksum, const uint64_t *__restrict__ total, uint64_t origin,
        uint8_t *__restrict__ output) {
    const uint64_t t = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    const uint32_t esz = checksum ? 12u : 8u;
    uint8_t *dst = output + (*total - origin);
    if (t < n)
        for (uint32_t k = 0; k < esz; k++) dst[8 + t * esz + k] = entries[t * esz + k];
    if (t == 0) {
        put32(dst, SEEK_SKIPPABLE_MAGIC);
        put32(dst + 4, (uint32_t)(n * esz + SEEK_FOOTER));
        uint8_t *ft = dst + 8 + n * esz;
        put32(ft, (uint32_t)n);
        ft[4] = checksum ? 0x80 : 0;
        put32(ft + 5, SEEK_FOOTER_MAGIC);
    }
}

// ------------------------------------------------------------------------------------------------------------
// k_range_gather: one CTA per piece.  Bytes up to the first 16-byte boundary of the destination, then 16-byte stores: from 16-byte
// loads when the source is aligned with the destination, else from aligned 4-byte words of the source joined by funnel shifts
// (the words hold only the piece's source bytes' 4-byte words, so no load leaves its allocation); the tail in bytes.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(GATHER_THREADS)
k_range_gather(const GatherPiece *__restrict__ pieces, uint8_t *__restrict__ base) {
    const GatherPiece p = pieces[blockIdx.x];
    const uint32_t tid = threadIdx.x;
    const uint8_t *src = base + p.src;
    uint8_t *dst = base + p.dst;
    const uint32_t head = min(p.len, (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15));
    for (uint32_t i = tid; i < head; i += GATHER_THREADS) dst[i] = src[i];
    const uint32_t nvec = (p.len - head) / 16;
    uint4 *d4 = reinterpret_cast<uint4 *>(dst + head);
    const uint8_t *s = src + head;
    const uint32_t sh = (uint32_t)((uintptr_t)s & 3) * 8;
    if (((uintptr_t)s & 15) == 0) {
        const uint4 *s4 = reinterpret_cast<const uint4 *>(s);
        for (uint32_t i = tid; i < nvec; i += GATHER_THREADS) d4[i] = s4[i];
    } else if (sh == 0) {
        const uint32_t *w = reinterpret_cast<const uint32_t *>(s);
        for (uint32_t i = tid; i < nvec; i += GATHER_THREADS) d4[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
    } else {
        const uint32_t *w = reinterpret_cast<const uint32_t *>((uintptr_t)s & ~(uintptr_t)3);
        for (uint32_t i = tid; i < nvec; i += GATHER_THREADS) {
            const uint32_t *q = w + 4 * i;
            const uint32_t a0 = q[0], a1 = q[1], a2 = q[2], a3 = q[3], a4 = q[4];
            d4[i] = make_uint4(__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh), __funnelshift_r(a2, a3, sh), __funnelshift_r(a3, a4, sh));
        }
    }
    for (uint32_t i = head + nvec * 16 + tid; i < p.len; i += GATHER_THREADS) dst[i] = src[i];
}

int launch_seek_scan(const CompressArgs &a, uint64_t *total, uint64_t origin, uint8_t *entries, uint64_t first_frame, cudaStream_t s,
                     uint64_t *launched) {
    if (!a.nblocks) return 0;
    k_cscan<<<1, SCAN_THREADS, 0, s>>>(const_cast<CFrame *>(a.frames), a.blocks, a.nblocks, a.res, a.csum, a.level, a.checksum, a.dict_id, total,
                                       origin, entries, first_frame);
    const int e = (int)cudaGetLastError();
    if (!e) ++*launched;
    return e;
}

int launch_seek_table(const uint8_t *entries, uint64_t n, int checksum, const uint64_t *total, uint64_t origin, uint8_t *output, cudaStream_t s,
                      uint64_t *launched) {
    const uint64_t grid = n ? (n + 255) / 256 : 1;
    k_cseek<<<(uint32_t)grid, 256, 0, s>>>(entries, n, checksum, total, origin, output);
    const int e = (int)cudaGetLastError();
    if (!e) ++*launched;
    return e;
}

int launch_range_gather(const GatherPiece *pieces, uint32_t n, uint8_t *base, cudaStream_t s, uint64_t *launched) {
    if (!n) return 0;
    k_range_gather<<<n, GATHER_THREADS, 0, s>>>(pieces, base);
    const int e = (int)cudaGetLastError();
    if (!e) ++*launched;
    return e;
}

}  // namespace b200z
