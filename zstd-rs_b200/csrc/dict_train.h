// dict_train.h -- launch interface between the host library (api.cpp) and the raw-content dictionary trainer's kernels
// (dict_train.cu).  The algorithm is DESIGN.md section 4.5.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200zstd.h"

namespace b200z {

constexpr uint32_t DT_K = 16;            // k-mer length
constexpr uint32_t DT_F = 22;            // log2 of the count table's slots
constexpr uint32_t DT_NO_SLOT = 0xffffffffu;

// slots[p] for every position of in[n] (DT_NO_SLOT where the k-mer leaves p's sample; starts[nsamples + 1] are the samples'
// offsets, starts[nsamples] == n), and freq[1 << DT_F] (zeroed by the caller) += 1 per slot
int launch_dt_count(const uint8_t *in, uint32_t n, const uint32_t *starts, uint32_t nsamples, uint32_t *slots, uint32_t *freq,
                    cudaStream_t s, uint64_t *launched);
// dist[p]: p minus the nearest earlier position with the same slot, when it is at most w - 1 away; else 0
int launch_dt_prev(const uint32_t *slots, uint32_t n, uint32_t w, uint16_t *dist, cudaStream_t s, uint64_t *launched);
// one epoch [e0, e1) with segments of le bytes: scores every start, keeps the best (best[0] and done[0] zeroed by the caller),
// writes *seg and zeroes freq at the chosen segment's slots
int launch_dt_epoch(const uint32_t *slots, const uint16_t *dist, uint32_t *freq, uint32_t epoch, uint32_t e0, uint32_t e1, uint32_t le,
                    unsigned long long *best, uint32_t *done, b200z_dict_segment *seg, cudaStream_t s, uint64_t *launched);

}  // namespace b200z
