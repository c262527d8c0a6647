// kernels.h -- launch interface between the host library (api.cpp / plan.cpp) and kernels.cu
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200z_types.h"
#include "framing.cuh"

namespace b200z {

struct PipelineArgs {
    const BlockDesc *descs;   // [nblocks]  device
    BlockAux *aux;            // [nblocks]  device
    const FrameDesc *frames;  // [nframes]  device
    FrameState *states;       // [nframes]  device, in/out
    const uint8_t *input;     // device, readable up to the next 4-byte boundary past the last frame
    uint8_t *lit_scratch;     // device
    uint32_t *seq_scratch;    // device, 3 x u32 per sequence
    uint8_t *output;          // device
    uint64_t output_cap;
    uint32_t nblocks;
    uint32_t nframes;
    // execution scheduling (one device buffer: ticket counter, resume[nframes], then the frame list of k_exec_cta)
    uint32_t *ticket;             // 16 bytes (ticket + debug counters), followed by resume[]
    uint32_t *resume;             // [nframes] first block the next k_exec launch has to execute, RESUME_SKIP = none.  Starts at 0 for
                                  // the frames of the warp kernel and at RESUME_SKIP for k_exec_cta's frames (which k_exec_cta rewrites)
    const uint32_t *cta_frames;   // [n_cta_frames] frames executed by k_exec_cta
    uint32_t n_cta_frames;
    uint32_t sched_bytes;         // 16 + 4 * nframes
    const uint32_t *sched_init;   // device image of the first sched_bytes, copied over ticket/resume before every pass
    const uint32_t *fse_order;    // [nblocks] or null: the order in which k_fse takes the blocks (null = descriptor order).  Block-major
                                  // across the multi-block frames of the warp kernel, so that k_exec, running beside k_fse, finds the
                                  // next block of EVERY frame ready instead of whole frames one after the other
};

// Every launcher adds the kernels it enqueued to *launched and returns 0 or the cudaError_t of the first failing call.
int init_kernels();  // per-device function attributes (dynamic shared memory); call once per context
int launch_predefined(FseSlot *predef, cudaStream_t s, uint64_t *launched);
constexpr int kNumStages = 5;
extern const char *const kStageNames[kNumStages];
int launch_stage(const PipelineArgs &a, int stage, cudaStream_t s, uint64_t *launched);
int reset_sched(const PipelineArgs &a, cudaStream_t s);      // ticket / resume[] back to their initial image (start of every pass)
int launch_pipeline(const PipelineArgs &a, cudaStream_t s, uint64_t *launched);   // the stages one after the other (streaming decoder)
// device-side header walk for device-resident input (k_walk): fill = 0 counts the blocks of every frame, fill = 1 writes the digests
int launch_walk(const uint8_t *d_input, uint64_t input_len, const uint64_t *d_src_off, const uint64_t *d_src_size, uint32_t nframes, WalkFrame *d_wf,
                const uint32_t *d_first_block, WalkBlock *d_wb, int fill, cudaStream_t s, uint64_t *launched);
// candidate frame starts of a buffer of concatenated frames (k_find_frames): offsets and bytes left from them into d_off / d_size (room for
// cap), the number found into *d_count (zeroed by the caller; it may exceed cap)
int launch_find_frames(const uint8_t *d_input, uint64_t input_len, uint64_t *d_off, uint64_t *d_size, uint32_t cap, unsigned long long *d_count,
                       cudaStream_t s, uint64_t *launched);
// k_place: out_off / out_cap of every frame of a.frames, back to back by decoded size (after k_fse, before execution)
int launch_place(const PipelineArgs &a, cudaStream_t s, uint64_t *launched);
uint32_t num_sms();   // of the current device (132 on H100 SXM)
// on the current device, for a submission of nblocks blocks: out[0] / out[1] the waves k_huf / k_fse take, out[2] / out[3] their
// resident CTAs per SM, k_huf's with the bit-reader ring it takes for nblocks (0 = unknown: init_kernels has not run on this device)
void entropy_waves(uint32_t nblocks, uint32_t out[4]);
int launch_checksum(const PipelineArgs &a, cudaStream_t s, uint64_t *launched);   // optional 5th stage: XXH64 of every frame's plaintext
// the stream decoder (tier 1d): k_place_resume places a submission whose first frame continues behind its carried tail; k_carry hands
// frame `plast` of `prev` to frame 0 of `next` (max_tail: the most bytes it may carry, max(window, 32)); k_xxh64_stream hashes frames
// that may resume from carry_in and stop mid-frame into carry_out
int launch_place_resume(const PipelineArgs &a, cudaStream_t s, uint64_t *launched);
int launch_carry(const PipelineArgs &prev, uint32_t plast, const PipelineArgs &next, const StreamCarry *carry_prev, StreamCarry *carry_next, bool resumed,
                 uint64_t max_tail, cudaStream_t s, uint64_t *launched);
int launch_checksum_stream(const PipelineArgs &a, const StreamCarry *carry_in, StreamCarry *carry_out, bool resumed, bool continues, cudaStream_t s,
                           uint64_t *launched);
struct PipelineStreams { cudaStream_t main, side; cudaEvent_t fork, join; };
int launch_pipeline_overlapped(const PipelineArgs &a, const PipelineStreams &ps, uint64_t *launched);   // the shipped order: k_exec beside k_fse (programmatic dependent launch)
int launch_tables_literals(const PipelineArgs &a, const PipelineStreams &ps, uint64_t *launched);   // k_setup (literals side + k_huf on `side`, sequences side on `main`)
int launch_fse_exec(const PipelineArgs &a, cudaStream_t s, uint64_t *launched);    // k_fse + (beside it) k_exec for the warp kernel's frames
int launch_cta_rest(const PipelineArgs &a, cudaStream_t s, uint64_t *launched);    // k_exec_cta + k_exec for what it handed back

}  // namespace b200z
