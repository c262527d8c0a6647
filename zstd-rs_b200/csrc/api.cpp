// api.cpp -- the C ABI declared in include/b200zstd.h: context, dictionaries, batch entry (tier 1) and the
// FrameDecoder / StreamingDecoder mirrors (tier 2).  Host logic only; all decoding happens in kernels.cu.
// There is no CPU decode path in this library: without a usable CUDA device b200z_ctx_create fails.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <map>
#include <memory>
#include <new>
#include <string>
#include <deque>
#include <vector>

#include "../../include/b200zstd.h"
#include "compress.h"
#include "dict_train.h"
#include "kernels.h"
#include "plan.h"
#include "tables.cuh"

using namespace b200z;

static int ctx_cuda_err(b200z_ctx *c, cudaError_t e, const char *what);   // b200z_ctx::set_cuda_err

// ---------------------------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------------------------
namespace {

struct ErrName { int code; const char *name; };
#define EN(x) {B200Z_##x, #x}
const ErrName kErrNames[] = {
    EN(OK), EN(ERR_MAGIC_NUMBER_READ), EN(ERR_BAD_MAGIC_NUMBER), EN(ERR_FRAME_DESCRIPTOR_READ), EN(ERR_INVALID_FRAME_DESCRIPTOR),
    EN(ERR_WINDOW_DESCRIPTOR_READ), EN(ERR_DICTIONARY_ID_READ), EN(ERR_FRAME_CONTENT_SIZE_READ), EN(ERR_SKIP_FRAME),
    EN(ERR_WINDOW_TOO_BIG), EN(ERR_WINDOW_TOO_SMALL), EN(ERR_WINDOW_SIZE_TOO_BIG), EN(ERR_DICT_NOT_PROVIDED), EN(ERR_NOT_YET_INITIALIZED),
    EN(ERR_FAILED_TO_READ_CHECKSUM), EN(ERR_FAILED_TO_DRAIN_DECODEBUFFER), EN(ERR_FAILED_TO_SKIP_FRAME), EN(ERR_TARGET_TOO_SMALL),
    EN(ERR_BLOCK_HEADER_READ), EN(ERR_FOUND_RESERVED_BLOCK), EN(ERR_BLOCK_SIZE_TOO_LARGE), EN(ERR_DECODER_STATE_IS_FAILED),
    EN(ERR_EXPECTED_HEADER_OF_PREVIOUS_BLOCK), EN(ERR_BLOCK_BODY_READ), EN(ERR_BLOCK_CONTENT_READ), EN(ERR_MALFORMED_SECTION_HEADER),
    EN(ERR_LITSEC_ILLEGAL_TYPE), EN(ERR_LITSEC_GET_BITS), EN(ERR_LITSEC_NOT_ENOUGH_BYTES), EN(ERR_SEQHDR_NOT_ENOUGH_BYTES),
    EN(ERR_LIT_MISSING_COMPRESSED_SIZE), EN(ERR_LIT_MISSING_NUM_STREAMS), EN(ERR_LIT_GET_BITS), EN(ERR_LIT_UNINITIALIZED_HUFFMAN_TABLE),
    EN(ERR_LIT_MISSING_BYTES_FOR_JUMP_HEADER), EN(ERR_LIT_MISSING_BYTES_FOR_LITERALS), EN(ERR_LIT_EXTRA_PADDING),
    EN(ERR_LIT_BITSTREAM_READ_MISMATCH), EN(ERR_LIT_DECODED_LITERAL_COUNT_MISMATCH), EN(ERR_HUF_GET_BITS), EN(ERR_HUF_FSE_DECODER),
    EN(ERR_HUF_SOURCE_IS_EMPTY), EN(ERR_HUF_NOT_ENOUGH_BYTES_FOR_WEIGHTS), EN(ERR_HUF_EXTRA_PADDING), EN(ERR_HUF_TOO_MANY_WEIGHTS),
    EN(ERR_HUF_MISSING_WEIGHTS), EN(ERR_HUF_LEFTOVER_NOT_POWER_OF_2), EN(ERR_HUF_NOT_ENOUGH_BYTES_TO_DECOMPRESS_WEIGHTS),
    EN(ERR_HUF_FSE_TABLE_USED_TOO_MANY_BYTES), EN(ERR_HUF_NOT_ENOUGH_BYTES_IN_SOURCE), EN(ERR_HUF_WEIGHT_BIGGER_THAN_MAX_NUM_BITS),
    EN(ERR_HUF_MAX_BITS_TOO_HIGH), EN(ERR_FSE_ACC_LOG_IS_ZERO), EN(ERR_FSE_ACC_LOG_TOO_BIG), EN(ERR_FSE_GET_BITS),
    EN(ERR_FSE_PROBABILITY_COUNTER_MISMATCH), EN(ERR_FSE_TOO_MANY_SYMBOLS), EN(ERR_FSE_TABLE_IS_UNINITIALIZED), EN(ERR_SEQ_EXTRA_PADDING),
    EN(ERR_SEQ_UNSUPPORTED_OFFSET), EN(ERR_SEQ_ZERO_OFFSET), EN(ERR_SEQ_NOT_ENOUGH_BYTES_FOR_NUM_SEQUENCES), EN(ERR_SEQ_EXTRA_BITS),
    EN(ERR_SEQ_MISSING_COMPRESSION_MODE), EN(ERR_SEQ_MISSING_BYTE_FOR_RLE_LL_TABLE), EN(ERR_SEQ_MISSING_BYTE_FOR_RLE_OF_TABLE),
    EN(ERR_SEQ_MISSING_BYTE_FOR_RLE_ML_TABLE), EN(ERR_EXEC_NOT_ENOUGH_BYTES_FOR_SEQUENCE), EN(ERR_EXEC_ZERO_OFFSET),
    EN(ERR_EXEC_NOT_ENOUGH_BYTES_IN_DICTIONARY), EN(ERR_EXEC_OFFSET_TOO_BIG), EN(ERR_DICT_NOT_ENOUGH_BYTES), EN(ERR_DICT_BAD_MAGIC_NUM),
    EN(ERR_REFERENCE_WOULD_PANIC), EN(ERR_BLOCK_OUTPUT_LIMIT), EN(ERR_INVALID_ARGUMENT), EN(ERR_OUT_OF_MEMORY), EN(ERR_NO_DEVICE), EN(ERR_CUDA),
    EN(ERR_SEEKABLE_TABLE), EN(ERR_SEEKABLE_FRAME_SIZE), EN(ERR_SEEKABLE_IO),
};
#undef EN

// bytes held by every Buf of the process: [0] device, [1] pinned host (b200z_debug_held_bytes)
std::atomic<uint64_t> g_held[2];

// The owners of the library's CUDA resources: each frees what it holds when it is destroyed, so no path, an error path
// included, frees by hand.  Buf is device memory (DevBuf) or pinned host memory (PinnedBuf).
template <bool Pinned> struct Buf {
    void *p = nullptr;
    size_t cap = 0;
    Buf() = default;
    Buf(Buf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    Buf &operator=(Buf &&o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
    ~Buf() { release(); }
    void release() {
        if (p) {
            Pinned ? cudaFreeHost(p) : cudaFree(p);
            g_held[Pinned] -= cap;
        }
        p = nullptr; cap = 0;
    }
    // exactly n bytes in place of what it held; returns CUDA's error, cleared
    cudaError_t alloc(size_t n) {
        release();
        const cudaError_t e = Pinned ? cudaMallocHost(&p, n) : cudaMalloc(&p, n);
        if (e != cudaSuccess) { p = nullptr; cudaGetLastError(); return e; }
        cap = n;
        g_held[Pinned] += n;
        return cudaSuccess;
    }
    // at least n bytes, and at least 1.5 times the old capacity with `grow`; contents are NOT preserved
    int ensure(size_t n, bool grow = true) {
        if (n <= cap) return 0;
        return alloc(grow && cap ? std::max(n, cap + cap / 2) : n) == cudaSuccess ? 0 : B200Z_ERR_OUT_OF_MEMORY;
    }
    template <class T> T *as() const { return (T *)p; }
};
using DevBuf = Buf<false>;
using PinnedBuf = Buf<true>;

// A non-blocking stream and an event.  create() returns 0 or B200Z_ERR_CUDA, with the context's error message set.
struct Stream {
    cudaStream_t s = nullptr;
    Stream() = default;
    Stream(const Stream &) = delete;
    Stream &operator=(const Stream &) = delete;
    ~Stream() { if (s) cudaStreamDestroy(s); }
    int create(b200z_ctx *c, int priority = 0) {   // 0: the default priority
        const cudaError_t e = cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, priority);
        if (e != cudaSuccess) { s = nullptr; return ctx_cuda_err(c, e, "cudaStreamCreateWithPriority"); }
        return 0;
    }
    operator cudaStream_t() const { return s; }
};
struct Event {
    cudaEvent_t e = nullptr;
    Event() = default;
    Event(const Event &) = delete;
    Event &operator=(const Event &) = delete;
    ~Event() { if (e) cudaEventDestroy(e); }
    int create(b200z_ctx *c, unsigned flags = cudaEventDisableTiming) {
        const cudaError_t r = cudaEventCreateWithFlags(&e, flags);
        if (r != cudaSuccess) { e = nullptr; return ctx_cuda_err(c, r, "cudaEventCreateWithFlags"); }
        return 0;
    }
    operator cudaEvent_t() const { return e; }
};

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------------------------
struct PipeResources;
struct CompressResources;
struct DictTrainResources;
struct StreamDecodeResources;

struct b200z_ctx {
    int device = 0;
    Stream stream;
    Stream side;                           // k_huf runs here, beside k_fse
    Event ev_fork, ev_join;
    DevBuf d_predef;                       // FseSlot: the predefined tables
    std::unique_ptr<PipeResources> pipe;         // lazily created by the pipelined one-shot path
    std::unique_ptr<CompressResources> comp;     // lazily created by the first compression
    std::unique_ptr<DictTrainResources> dtrain;  // lazily created by the first dictionary training
    std::unique_ptr<StreamDecodeResources> sdec; // lazily created by the first b200z_decode_all_stream
    std::string err;
    uint64_t launches = 0;
    uint32_t flags = 0;
    ~b200z_ctx();                          // at the end of the file, where the lazily created resources are complete
    int set_cuda_err(cudaError_t e, const char *what) {
        char buf[256];
        snprintf(buf, sizeof buf, "CUDA error in %s: %s", what, cudaGetErrorString(e));
        err = buf;
        cudaGetLastError();
        return B200Z_ERR_CUDA;
    }
    int use() { cudaError_t e = cudaSetDevice(device); return e == cudaSuccess ? 0 : set_cuda_err(e, "cudaSetDevice"); }
};
static int ctx_cuda_err(b200z_ctx *c, cudaError_t e, const char *what) { return c->set_cuda_err(e, what); }

#define CU(ctx, call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return (ctx)->set_cuda_err(_e, #call); } while (0)

extern "C" const char *b200z_error_name(int code) {
    for (const auto &e : kErrNames) if (e.code == code) return e.name;
    return "UNKNOWN";
}
extern "C" int b200z_abi_version(void) { return B200Z_ABI_VERSION; }

extern "C" int b200z_ctx_create(int device, b200z_ctx **out) {
    if (!out) return B200Z_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) { cudaGetLastError(); return B200Z_ERR_NO_DEVICE; }
    std::unique_ptr<b200z_ctx> c(new b200z_ctx());
    c->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return B200Z_ERR_NO_DEVICE; }
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    if (c->stream.create(c.get(), prio_hi)) return B200Z_ERR_NO_DEVICE;
    if (c->side.create(c.get(), prio_lo) || c->ev_fork.create(c.get()) || c->ev_join.create(c.get())) return B200Z_ERR_CUDA;
    if (int e = c->d_predef.ensure(sizeof(FseSlot), false)) return e;
    if (init_kernels() || init_compress_kernels()) { cudaGetLastError(); return B200Z_ERR_CUDA; }
    int e = launch_predefined(c->d_predef.as<FseSlot>(), c->stream, &c->launches);
    if (e || cudaStreamSynchronize(c->stream) != cudaSuccess) { cudaGetLastError(); return B200Z_ERR_CUDA; }
    *out = c.release();
    return 0;
}
extern "C" void b200z_ctx_destroy(b200z_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    delete c;
}
extern "C" const char *b200z_ctx_last_error_message(const b200z_ctx *c) { return c ? c->err.c_str() : ""; }
extern "C" void *b200z_ctx_stream(const b200z_ctx *c) { return c ? (void *)c->stream.s : nullptr; }
extern "C" uint64_t b200z_ctx_kernel_launches(const b200z_ctx *c) { return c ? c->launches : 0; }
extern "C" void b200z_debug_held_bytes(uint64_t *device, uint64_t *pinned) {
    if (device) *device = g_held[0];
    if (pinned) *pinned = g_held[1];
}
extern "C" void b200z_ctx_set_flags(b200z_ctx *c, uint32_t flags) { if (c) c->flags = flags; }
extern "C" uint32_t b200z_ctx_flags(const b200z_ctx *c) { return c ? c->flags : 0; }
extern "C" uint64_t b200z_xxh64(const uint8_t *data, size_t len) { XXH64State s; s.reset(); s.update(data, len); return s.digest(); }

// ---------------------------------------------------------------------------------------------------------------
// dictionaries
// ---------------------------------------------------------------------------------------------------------------
struct b200z_dict {
    b200z_ctx *ctx = nullptr;
    uint32_t id = 0;
    uint32_t hist[3] = {1, 4, 8};
    bool has_tables = false;
    DevBuf d_huf, d_fse;          // HufSlot, FseSlot
    DevBuf d_content;             // content_len bytes
    size_t content_len = 0;
    // Built by the first compression that needs them, and stored only once complete.  The compressor's match table of the
    // content (k_cdict); a formatted dictionary's tables as parsed (Huffman weights; OF / ML / LL normalized counts by ENC_LL /
    // ENC_OF / ENC_ML), and the encoder's view of them (EncDict), built on the host for B200Z_FLAG_DICT_TABLES
    mutable DevBuf d_ctab;
    uint8_t huf_weights[260] = {};
    uint32_t huf_nweights = 0;
    int16_t norm[3][64] = {};
    uint32_t nnorm[3] = {}, log[3] = {};
    mutable DevBuf d_enc;
    // B200Z_FLAG_DICT_LONG: the anchors of the content's last min(len, 2^27) bytes, sorted by key: nlanch keys, then nlanch distances
    // from the content's end (ldm.cu k_ldict), built by the first long-match compression with the flag (lanch_built) and kept
    mutable DevBuf d_lanch;
    mutable uint32_t nlanch = 0;
    mutable bool lanch_built = false;
};

static int dict_upload_content(b200z_dict *d, const uint8_t *content, size_t len) {
    b200z_ctx *c = d->ctx;
    d->content_len = len;
    CU(c, d->d_content.alloc(len + 16));
    if (len) CU(c, cudaMemcpy(d->d_content.p, content, len, cudaMemcpyHostToDevice));
    return 0;
}

// Dictionary::decode_dict (dictionary.rs:45-126).  The table descriptions are parsed and expanded with the same
// code the GPU runs per block (tables.cuh, compiled for the host here) and uploaded once.  The parsed weights and normalized
// counts are kept for the encoder (B200Z_FLAG_DICT_TABLES): each description is read once, then expanded for the decoder.
extern "C" int b200z_dict_create(b200z_ctx *c, const uint8_t *raw, size_t len, b200z_dict **out) {
    if (!c || !out || (!raw && len)) return B200Z_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    if (int e = c->use()) return e;
    if (len < 8) return B200Z_ERR_DICT_NOT_ENOUGH_BYTES;
    static const uint8_t magic[4] = {0x37, 0xA4, 0x30, 0xEC};
    if (memcmp(raw, magic, 4) != 0) return B200Z_ERR_DICT_BAD_MAGIC_NUM;
    std::unique_ptr<b200z_dict> d(new b200z_dict());
    d->ctx = c;
    d->id = rd32le(raw + 4);
    const uint8_t *t = raw + 8;
    size_t tl = len - 8;
    std::unique_ptr<HufSlot> huf(new HufSlot());
    std::unique_ptr<FseSlot> fse(new FseSlot());
    memset(huf.get(), 0, sizeof(HufSlot));
    memset(fse.get(), 0, sizeof(FseSlot));
    uint32_t used = 0, mb = 0;
    // huf_build_decoder's two steps (tables.cuh)
    int e = huf_read_weights(t, (uint32_t)std::min<size_t>(tl, 0x7fffffff), d->huf_weights, d->huf_nweights, used);
    if (e || (e = huf_build_table(d->huf_weights, d->huf_nweights, huf.get(), mb))) return e;
    huf->max_bits = mb;
    if (tl < used) return B200Z_ERR_DICT_NOT_ENOUGH_BYTES;
    t += used; tl -= used;
    struct { FseTab *tab; uint32_t max_log, max_sym, enc; } order[3] = {{&fse->of, 8, 31, ENC_OF}, {&fse->ml, 9, 52, ENC_ML}, {&fse->ll, 9, 35, ENC_LL}};
    for (auto &o : order) {   // OF, ML, LL: fse_build_decoder's steps (tables.cuh)
        int16_t probs[256];
        uint32_t nprobs = 0, acc_log = 0;
        e = fse_read_probabilities(t, (uint32_t)std::min<size_t>(tl, 0x7fffffff), o.max_log, o.max_sym, probs, nprobs, acc_log, used);
        if (e) return e;
        std::vector<uint32_t> wide(FSE_MAX_ENTRIES);
        uint16_t counter[256];
        if ((e = fse_build_table(probs, nprobs, acc_log, o.max_sym, wide.data(), counter))) return e;
        fse_compact(wide.data(), acc_log, o.tab);
        memcpy(d->norm[o.enc], probs, nprobs * sizeof(int16_t));
        d->nnorm[o.enc] = nprobs;
        d->log[o.enc] = acc_log;
        if (tl < used) return B200Z_ERR_DICT_NOT_ENOUGH_BYTES;
        t += used; tl -= used;
    }
    if (tl < 12) return B200Z_ERR_DICT_NOT_ENOUGH_BYTES;
    for (int i = 0; i < 3; i++) d->hist[i] = rd32le(t + 4 * i);
    d->has_tables = true;
    CU(c, d->d_huf.alloc(sizeof(HufSlot)));
    CU(c, d->d_fse.alloc(sizeof(FseSlot)));
    CU(c, cudaMemcpy(d->d_huf.p, huf.get(), sizeof(HufSlot), cudaMemcpyHostToDevice));
    CU(c, cudaMemcpy(d->d_fse.p, fse.get(), sizeof(FseSlot), cudaMemcpyHostToDevice));
    if ((e = dict_upload_content(d.get(), t + 12, tl - 12))) return e;
    *out = d.release();
    return 0;
}
extern "C" int b200z_dict_create_raw_content(b200z_ctx *c, uint32_t id, const uint8_t *content, size_t len, b200z_dict **out) {
    if (!c || !out || (!content && len)) return B200Z_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    if (int e = c->use()) return e;
    std::unique_ptr<b200z_dict> d(new b200z_dict());
    d->ctx = c; d->id = id;
    if (int e = dict_upload_content(d.get(), content, len)) return e;
    *out = d.release();
    return 0;
}
extern "C" uint32_t b200z_dict_id(const b200z_dict *d) { return d ? d->id : 0; }
extern "C" int b200z_dict_offset_history(const b200z_dict *d, uint32_t out[3]) { if (!d) return B200Z_ERR_INVALID_ARGUMENT; memcpy(out, d->hist, 12); return 0; }
extern "C" size_t b200z_dict_content_size(const b200z_dict *d) { return d ? d->content_len : 0; }
extern "C" void b200z_dict_destroy(b200z_dict *d) {
    if (!d) return;
    cudaSetDevice(d->ctx->device);
    delete d;
}

// ---------------------------------------------------------------------------------------------------------------
// A "submission": host-side plan + its device mirror.  Every decoding entry plans one.  A frame starts fresh (add_frame) or resumes
// from a previous submission's state and tables (add_resumed_frame: the stream decoder's first frame, the FrameDecoder mirror's one
// frame).  Below it, the frame-start and block-read rules of the reference, which every entry's planner applies.
// ---------------------------------------------------------------------------------------------------------------
namespace {

// FSE table `which` (0 = LL, 1 = OF, 2 = ML) of a slot
template <class Slot> auto *fse_at(Slot *s, int which) { return which == 0 ? &s->ll : (which == 1 ? &s->of : &s->ml); }

struct CarrySet {
    const HufSlot *huf = nullptr;
    const FseTab *ll = nullptr, *of = nullptr, *ml = nullptr;
    const b200z_dict *dict = nullptr;   // the dictionary these tables belong to (null: tables carried over from a submission)
    const FseTab *fse(int which) const { return which == 0 ? ll : (which == 1 ? of : ml); }
};

CarrySet carry_of_dict(const b200z_dict *d) {
    CarrySet cs;
    cs.dict = d;
    if (d && d->has_tables) {
        const FseSlot *f = d->d_fse.as<FseSlot>();
        cs.huf = d->d_huf.as<HufSlot>(); cs.ll = &f->ll; cs.of = &f->of; cs.ml = &f->ml;
    }
    return cs;
}

struct Submission {
    std::vector<BlockDesc> descs;
    std::vector<BlockRefs> refs;
    std::vector<FrameDesc> frames;
    std::vector<FrameState> states;
    std::vector<CarrySet> carries;   // TabRef::CARRY idx -> device tables (dictionaries / streaming carry)
    uint32_t n_huf = 0, n_fse = 0;
    uint64_t lit_bytes = 0, nseq = 0;
    DevBuf d_descs, d_aux, d_frames, d_states, d_huf, d_fse, d_lit, d_seq, d_sched, d_order;
    std::vector<uint32_t> fse_order;    // PipelineArgs::fse_order (empty: descriptor order)
    std::vector<uint32_t> cta_frames;   // frames executed by k_exec_cta (the rest: k_exec, one warp per frame)
    std::vector<uint32_t> sched_image;  // host copy of the initial ticket / resume[] image (kept alive for the async upload)

    void clear() {
        descs.clear(); refs.clear(); frames.clear(); states.clear(); carries.clear();
        n_huf = n_fse = 0; lit_bytes = 0; nseq = 0;
    }
    // TabRef::CARRY index of a dictionary's tables, added on first use; -1 for no dictionary
    int carry_index(const b200z_dict *dict) {
        if (!dict) return -1;
        for (size_t i = 0; i < carries.size(); i++) if (carries[i].dict == dict) return (int)i;
        carries.push_back(carry_of_dict(dict));
        return (int)carries.size() - 1;
    }
    // Appends a frame whose blocks follow, starting from the dictionary's offset history or {1, 4, 8}.
    // Returns the table cursor of its first block: the dictionary's tables, if any.
    TableCursor add_frame(const b200z_dict *dict, uint64_t out_off, uint64_t out_cap, uint64_t window) {
        static const uint32_t fresh_hist[3] = {1, 4, 8};
        FrameState st;
        memset(&st, 0, sizeof st);
        memcpy(st.hist, dict ? dict->hist : fresh_hist, sizeof st.hist);
        const TableCursor cur = push_frame(dict, window, st, carry_index(dict));
        frames.back().out_off = out_off; frames.back().out_cap = out_cap;
        return cur;
    }
    // Appends a frame that continues from a previous submission, from its state `st` and the tables `cs` its next block starts from;
    // the caller places it.  Returns the table cursor of that block.
    TableCursor add_resumed_frame(const FrameState &st, uint64_t window, const b200z_dict *dict, const CarrySet &cs) {
        carries.push_back(cs);
        return push_frame(dict, window, st, (int)carries.size() - 1);
    }
    // appends a frame's descriptor and state; its first block starts from the tables of carries[ci], if any (scratch.rs:70-78)
    TableCursor push_frame(const b200z_dict *dict, uint64_t window, const FrameState &st, int ci) {
        FrameDesc fd;
        memset(&fd, 0, sizeof fd);
        fd.window_size = window;
        fd.dict = dict ? dict->d_content.as<uint8_t>() : nullptr; fd.dict_len = dict ? dict->content_len : 0;
        fd.first_block = (uint32_t)descs.size();
        frames.push_back(fd); states.push_back(st);
        TableCursor cur;
        if (ci < 0) return cur;
        const CarrySet &cs = carries[ci];
        if (cs.huf) { cur.huf.kind = TabRef::CARRY; cur.huf.idx = (uint32_t)ci; }
        if (cs.ll) { cur.ll.kind = TabRef::CARRY; cur.ll.idx = (uint32_t)ci; }
        if (cs.of) { cur.of.kind = TabRef::CARRY; cur.of.idx = (uint32_t)ci; }
        if (cs.ml) { cur.ml.kind = TabRef::CARRY; cur.ml.idx = (uint32_t)ci; }
        return cur;
    }
    // Appends a block to the last frame and counts it there.  A Compressed block is planned from its section headers, as parsed here
    // from its content or by k_walk (`sec`); `cur` moves on to the tables it leaves current.
    const BlockDesc &add_block(uint64_t src_off, const BlockHeader &bh, uint32_t block_in_frame, const SectionHeaders &sec, TableCursor &cur) {
        BlockDesc d;
        memset(&d, 0, sizeof d);
        BlockRefs r;
        d.src_off = src_off; d.src_size = bh.content_size; d.frame = (uint32_t)frames.size() - 1; d.btype = bh.type; d.raw_size = bh.decompressed_size;
        d.block_in_frame = block_in_frame; d.last = bh.last;
        if (bh.type == BT_COMPRESSED) plan_compressed_block(sec, d, r, cur, n_huf, n_fse, lit_bytes, nseq);
        descs.push_back(d); refs.push_back(r);
        frames.back().nblocks++;
        return descs.back();
    }
    const BlockDesc &add_block(uint64_t src_off, const BlockHeader &bh, uint32_t block_in_frame, const uint8_t *content, TableCursor &cur) {
        const SectionHeaders sec = bh.type == BT_COMPRESSED ? parse_section_headers(content, bh.content_size) : SectionHeaders();
        return add_block(src_off, bh, block_in_frame, sec, cur);
    }
    // The tables a frame's next block starts from after this submission, where its last block left `cur` current: a table built here
    // (SLOT) is copy_carry's copy at `huf_to` / `fse_to`; the predefined tables and those the frame started from (CARRY) stay put.
    CarrySet carry_after(const TableCursor &cur, const HufSlot *huf_to, const FseSlot *fse_to, const FseSlot *predef) const {
        auto fse = [&](const TabRef &t, int which) -> const FseTab * {
            if (t.kind == TabRef::SLOT) return fse_at(fse_to, which);
            if (t.kind == TabRef::PREDEF) return fse_at(predef, which);
            if (t.kind == TabRef::CARRY) return carries[t.idx].fse(which);
            return nullptr;
        };
        CarrySet next;
        next.huf = cur.huf.kind == TabRef::SLOT ? huf_to : (cur.huf.kind == TabRef::CARRY ? carries[cur.huf.idx].huf : nullptr);
        next.ll = fse(cur.ll, 0); next.of = fse(cur.of, 1); next.ml = fse(cur.ml, 2);
        return next;
    }
    // Queues on `stream` the device-to-device copies of the tables built here that `cur` names, to where carry_after put them.
    int copy_carry(b200z_ctx *c, const TableCursor &cur, HufSlot *huf_to, FseSlot *fse_to, cudaStream_t stream) const {
        if (cur.huf.kind == TabRef::SLOT)
            CU(c, cudaMemcpyAsync(huf_to, d_huf.as<HufSlot>() + cur.huf.idx, sizeof(HufSlot), cudaMemcpyDeviceToDevice, stream));
        const TabRef *t[3] = {&cur.ll, &cur.of, &cur.ml};
        for (int k = 0; k < 3; k++)
            if (t[k]->kind == TabRef::SLOT)
                CU(c, cudaMemcpyAsync(fse_at(fse_to, k), fse_at(d_fse.as<FseSlot>() + t[k]->idx, k), sizeof(FseTab), cudaMemcpyDeviceToDevice, stream));
        return 0;
    }
    // Queues on `stream` the copy to host memory of the frame states, or of the aux records of blocks [first, first + n).
    int download_states(b200z_ctx *c, FrameState *to, cudaStream_t stream) const {
        if (!states.empty()) CU(c, cudaMemcpyAsync(to, d_states.p, states.size() * sizeof(FrameState), cudaMemcpyDeviceToHost, stream));
        return 0;
    }
    int download_aux(b200z_ctx *c, BlockAux *to, size_t first, size_t n, cudaStream_t stream) const {
        if (n) CU(c, cudaMemcpyAsync(to, d_aux.as<BlockAux>() + first, n * sizeof(BlockAux), cudaMemcpyDeviceToHost, stream));
        return 0;
    }
    // resolve table references to device pointers and upload descriptors
    int upload(b200z_ctx *c, cudaStream_t stream = nullptr) {
        if (!stream) stream = c->stream;
        int e;
        if ((e = d_descs.ensure(descs.size() * sizeof(BlockDesc)))) return e;
        if ((e = d_aux.ensure(descs.size() * sizeof(BlockAux)))) return e;
        if ((e = d_frames.ensure(frames.size() * sizeof(FrameDesc)))) return e;
        if ((e = d_states.ensure(states.size() * sizeof(FrameState)))) return e;
        if ((e = d_huf.ensure((size_t)n_huf * sizeof(HufSlot)))) return e;
        if ((e = d_fse.ensure((size_t)n_fse * sizeof(FseSlot)))) return e;
        if ((e = d_lit.ensure(lit_bytes + 64))) return e;
        if ((e = d_seq.ensure((nseq + 4) * 12))) return e;
        // which execution kernel takes a frame (route_exec_frames, plan.cpp): single-block frames, tiny frames and frames with a
        // dictionary always stay with the warp kernel (dictionary reach is its exact path); the multi-block frames go to k_exec_cta
        // or k_exec by a cost model on sequences + compressed bytes.  B200Z_EXEC_MODE = warp | cta | auto (default) overrides for
        // tests and measurements.
        cta_frames.clear();
        {
            const char *m = getenv("B200Z_EXEC_MODE");
            const bool force_warp = m && !strcmp(m, "warp"), force_cta = m && !strcmp(m, "cta");
            std::vector<uint64_t> work(frames.size(), 0);
            std::vector<uint8_t> eligible(frames.size(), 0);
            for (size_t f = 0; f < frames.size() && !force_warp; f++) {
                const FrameDesc &fd = frames[f];
                if (fd.nblocks == 0) continue;
                uint64_t src = 0, nseq = 0;
                for (uint32_t k = 0; k < fd.nblocks; k++) { src += descs[fd.first_block + k].src_size; nseq += descs[fd.first_block + k].nseq; }
                work[f] = nseq + src / 16;
                if (fd.dict) continue;
                if (force_cta) cta_frames.push_back((uint32_t)f);
                else eligible[f] = fd.nblocks >= 2 && src >= 4096;
            }
            if (!force_warp && !force_cta) route_exec_frames(work.data(), eligible.data(), frames.size(), num_sms(), cta_frames);
        }
        // the order in which k_fse takes the blocks (build_fse_order, plan.cpp)
        fse_order.clear();
        if (!frames.empty()) {
            std::vector<uint8_t> on_cta(frames.size(), 0);
            for (uint32_t f : cta_frames) on_cta[f] = 1;
            std::vector<uint32_t> fb(frames.size()), nb(frames.size()), nseq(descs.size());
            for (size_t f = 0; f < frames.size(); f++) { fb[f] = frames[f].first_block; nb[f] = frames[f].nblocks; }
            for (size_t i = 0; i < descs.size(); i++) nseq[i] = descs[i].nseq;
            build_fse_order(fb.data(), nb.data(), on_cta.data(), frames.size(), nseq.data(), descs.size(), fse_order);
        }
        if (!fse_order.empty() && (e = d_order.ensure(4 * fse_order.size()))) return e;
        // scheduling buffer: [ticket + 3 counters][resume[nframes]][cta frame list][initial image of the first two parts]
        if ((e = d_sched.ensure(2 * (16 + 4 * frames.size()) + 4 * cta_frames.size() + 32))) return e;
        HufSlot *hs = d_huf.as<HufSlot>();
        FseSlot *fs = d_fse.as<FseSlot>();
        const FseSlot *pd = c->d_predef.as<FseSlot>();
        for (size_t i = 0; i < descs.size(); i++) {
            BlockDesc &d = descs[i];
            const BlockRefs &r = refs[i];
            auto huf = [&](const TabRef &t) -> const HufSlot * {
                if (t.kind == TabRef::SLOT) return hs + t.idx;
                if (t.kind == TabRef::CARRY) return carries[t.idx].huf;
                return nullptr;
            };
            auto fse = [&](const TabRef &t, int which) -> const FseTab * {
                if (t.kind == TabRef::SLOT) return fse_at(fs + t.idx, which);
                if (t.kind == TabRef::PREDEF) return fse_at(pd, which);
                if (t.kind == TabRef::CARRY) return carries[t.idx].fse(which);
                return nullptr;
            };
            d.huf = huf(r.huf);
            d.huf_build = r.build_huf >= 0 ? hs + r.build_huf : nullptr;
            d.ll = fse(r.ll, 0); d.of = fse(r.of, 1); d.ml = fse(r.ml, 2);
            d.fse_build = r.build_fse >= 0 ? fs + r.build_fse : nullptr;
        }
        if (!descs.empty()) CU(c, cudaMemcpyAsync(d_descs.p, descs.data(), descs.size() * sizeof(BlockDesc), cudaMemcpyHostToDevice, stream));
        if (!frames.empty()) CU(c, cudaMemcpyAsync(d_frames.p, frames.data(), frames.size() * sizeof(FrameDesc), cudaMemcpyHostToDevice, stream));
        if (!states.empty()) CU(c, cudaMemcpyAsync(d_states.p, states.data(), states.size() * sizeof(FrameState), cudaMemcpyHostToDevice, stream));
        if (!fse_order.empty()) CU(c, cudaMemcpyAsync(d_order.p, fse_order.data(), 4 * fse_order.size(), cudaMemcpyHostToDevice, stream));
        if (!cta_frames.empty())
            CU(c, cudaMemcpyAsync(d_sched.as<uint8_t>() + 16 + 4 * frames.size(), cta_frames.data(), 4 * cta_frames.size(), cudaMemcpyHostToDevice, stream));
        if (!frames.empty()) {
            sched_image.assign(4 + frames.size(), 0u);
            for (uint32_t f : cta_frames) sched_image[4 + f] = RESUME_SKIP;   // not for the first k_exec launch; k_exec_cta rewrites it
            CU(c, cudaMemcpyAsync(d_sched.as<uint8_t>() + 16 + 4 * (frames.size() + cta_frames.size()), sched_image.data(), 4 * sched_image.size(), cudaMemcpyHostToDevice, stream));
        }
        return 0;
    }
    PipelineArgs args(const uint8_t *d_input, uint8_t *d_output, uint64_t out_cap) const {
        PipelineArgs a;
        a.descs = d_descs.as<BlockDesc>(); a.aux = d_aux.as<BlockAux>(); a.frames = d_frames.as<FrameDesc>(); a.states = d_states.as<FrameState>();
        a.input = d_input; a.lit_scratch = d_lit.as<uint8_t>(); a.seq_scratch = d_seq.as<uint32_t>();
        a.output = d_output; a.output_cap = out_cap; a.nblocks = (uint32_t)descs.size(); a.nframes = (uint32_t)frames.size();
        uint8_t *sp = d_sched.as<uint8_t>();
        a.ticket = (uint32_t *)sp; a.resume = (uint32_t *)(sp + 16); a.cta_frames = (const uint32_t *)(sp + 16 + 4 * frames.size());
        a.n_cta_frames = (uint32_t)cta_frames.size(); a.sched_bytes = (uint32_t)(16 + 4 * frames.size());
        a.sched_init = (const uint32_t *)(sp + 16 + 4 * (frames.size() + cta_frames.size()));
        a.fse_order = fse_order.empty() ? nullptr : d_order.as<uint32_t>();
        return a;
    }
};

// common::MAX_WINDOW_SIZE, the cap of every window limit (FrameDecoder::set_max_window_size, :175-177).  A single-segment frame's
// window is its content size, which frame_window_size does not bound, so the cap decides for such a frame.
constexpr uint64_t MAX_WINDOW_SIZE = (1ull << 41) + 7 * (1ull << 38);
// the window limit of a decoding entry's `max_window`: 0 means the default (frame_decoder.rs:25)
uint64_t window_limit(uint64_t max_window) { return std::min<uint64_t>(max_window ? max_window : B200Z_DEFAULT_MAX_WINDOW_SIZE, MAX_WINDOW_SIZE); }

// The window rule of FrameDecoderState::new / reset (frame_decoder.rs:103-142): `window` from the header, refused when the header
// gives none or when it is above `limit`.  Returns 0 or the error, which the reference raises at B200Z_STAGE_FRAME_HEADER.
int frame_window(const FrameHeader &h, uint64_t limit, uint64_t &window) {
    if (int e = frame_window_size(h, window)) return e;
    return window > limit ? B200Z_ERR_WINDOW_SIZE_TOO_BIG : 0;
}

// The dictionary of a frame on the entries that take a list (FrameDecoder::reset :210-218, then force_dict): the last of `dicts` with
// the header's ID, or `forced` when given.  B200Z_ERR_DICT_NOT_PROVIDED (stage FRAME_HEADER) when none has the ID, forced or not.
int frame_dict(const FrameHeader &h, const b200z_dict *const *dicts, size_t ndicts, const b200z_dict *forced, const b200z_dict *&dict) {
    dict = nullptr;
    if (h.has_dict_id) {
        for (size_t k = 0; k < ndicts; k++) if (dicts[k]->id == h.dict_id) dict = dicts[k];
        if (!dict) return B200Z_ERR_DICT_NOT_PROVIDED;
    }
    if (forced) dict = forced;
    return 0;
}

// The block-read rule of decode_blocks (BlockDecoder::read_block_header, decode_block_content): `hdr` is null when the 3 header bytes
// cannot be read, has_body(n) says whether the n content bytes can.  The status word of a block not read whole, or 0 and `bh`.
template <class HasBody>
uint32_t read_block(const uint8_t *hdr, BlockHeader &bh, HasBody has_body) {
    if (!hdr) return mk_status(B200Z_ERR_BLOCK_HEADER_READ, B200Z_STAGE_BLOCK_HEADER);
    if (int e = parse_block_header(hdr, bh)) return mk_status((uint32_t)e, B200Z_STAGE_BLOCK_HEADER);
    if (!has_body(bh.content_size))
        return mk_status(bh.type == BT_COMPRESSED ? B200Z_ERR_BLOCK_CONTENT_READ : B200Z_ERR_BLOCK_BODY_READ, B200Z_STAGE_BLOCK_BODY);
    return 0;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// tier 1: batch
// ---------------------------------------------------------------------------------------------------------------
struct FramePlanInfo {
    int pre_status = 0, pre_stage = 0;       // failure before any block (frame header / window / dictionary)
    FrameHeader hdr;
    uint64_t window = 0;
    uint64_t bytes_read_full = 0;            // bytes_read_from_source after a fully successful decode
    size_t first_block_end = 0;              // index into block_end_bytes
    bool has_checksum = false;
    uint32_t checksum = 0;
    uint32_t skip_len = 0;
    int32_t sub_frame = -1;                  // index in Submission::frames, -1 if the frame never reaches the GPU
};

struct b200z_batch {
    b200z_ctx *ctx = nullptr;
    Submission sub;
    std::vector<FramePlanInfo> info;
    std::vector<uint64_t> block_end_bytes;   // per planned block: bytes_read_from_source after that block
    DevBuf d_input_own;
    const uint8_t *d_input = nullptr;
    DevBuf d_states_init;
    size_t input_len = 0;
    bool ran = false;
    bool checksummed = false;
    uint64_t run_launches = 0;               // kernels the most recent b200z_batch_run launched
    // decode_all batches (b200z_decode_all_prepare): `info` holds one entry per frame of the chain, in stream order, and k_place
    // places the frames of the submission back to back on every run
    bool decode_all = false;
    std::vector<uint64_t> chain;             // input offset of every frame of the chain
    std::vector<uint8_t> chain_zstd;         // 1 where the chain holds a zstd frame (one b200z_frame_result each)
    uint64_t zstd_frames = 0;
    uint64_t ran_output_cap = 0;             // output_cap of the most recent b200z_batch_run
};

// what k_walk brought back for a batch whose input lives in device memory (the planner then never sees the compressed bytes)
struct WalkHost { std::vector<WalkFrame> wf; std::vector<WalkBlock> wb; std::vector<uint32_t> first; };

static int plan_batch(b200z_batch *b, const uint8_t *in, size_t in_len, const b200z_frame_io *frames, size_t nframes,
                      const b200z_dict *const *dicts, size_t ndicts, const b200z_dict *forced, uint64_t max_window, const WalkHost *walk = nullptr) {
    Submission &s = b->sub;
    s.clear();
    b->info.assign(nframes, FramePlanInfo());
    b->block_end_bytes.clear();
    const uint64_t limit = window_limit(max_window);
    for (size_t i = 0; i < nframes; i++) {
        FramePlanInfo &fi = b->info[i];
        const b200z_frame_io &io = frames[i];
        if (io.src_off > in_len || io.src_size > in_len - io.src_off) { fi.pre_status = B200Z_ERR_INVALID_ARGUMENT; continue; }
        // host input: the frame's bytes; device input: the bytes the header walk picked (frame header here, block digests below)
        const uint8_t *p = walk ? walk->wf[i].hdr : in + io.src_off;
        size_t len = io.src_size, consumed = 0;
        uint32_t wk = walk ? walk->first[i] : 0;   // next block digest of this frame
        const uint32_t wk_end = walk ? wk + walk->wf[i].nblocks : 0;
        int e = parse_frame_header(p, len, fi.hdr, fi.skip_len, consumed);
        if (e) { fi.pre_status = e; fi.pre_stage = B200Z_STAGE_FRAME_HEADER; fi.bytes_read_full = consumed; continue; }
        const b200z_dict *dict = nullptr;
        if ((e = frame_window(fi.hdr, limit, fi.window)) || (e = frame_dict(fi.hdr, dicts, ndicts, forced, dict))) {
            fi.pre_status = e; fi.pre_stage = B200Z_STAGE_FRAME_HEADER;
            continue;
        }

        fi.sub_frame = (int32_t)s.frames.size();
        TableCursor cur = s.add_frame(dict, io.out_off, io.out_cap, fi.window);
        FrameDesc &fd = s.frames.back();
        fi.first_block_end = b->block_end_bytes.size();

        uint64_t pos = consumed, bytes_read = consumed;
        uint32_t bif = 0;
        for (;;) {
            const WalkBlock *wbk = nullptr;
            if (walk && len - pos >= 3) {
                if (wk >= wk_end || walk->wb[wk].pos != pos) return B200Z_ERR_INVALID_ARGUMENT;   // (the walk and the planner follow the same chain)
                wbk = &walk->wb[wk++];
            }
            BlockHeader bh;
            const uint8_t *hdr = len - pos < 3 ? nullptr : (wbk ? wbk->bh : p + pos);
            if (uint32_t w = read_block(hdr, bh, [&](uint32_t n) { return len - pos - 3 >= n; })) { fd.host_status = w; break; }
            pos += 3;
            const BlockDesc &d = wbk ? s.add_block(io.src_off + pos, bh, bif++, wbk->sec, cur)
                                     : s.add_block(io.src_off + pos, bh, bif++, p + pos, cur);
            pos += bh.content_size;
            bytes_read += 3 + bh.content_size;
            b->block_end_bytes.push_back(bytes_read);
            if (d.host_status) break;  // the reference stops here; later blocks are never looked at
            if (bh.last) {
                if (fi.hdr.content_checksum()) {
                    if (len - pos < 4) { fd.host_status = mk_status(B200Z_ERR_FAILED_TO_READ_CHECKSUM, B200Z_STAGE_CHECKSUM); break; }
                    fi.has_checksum = true;
                    if (walk && (walk->wf[i].end_pos != pos || walk->wf[i].tail_avail < 4)) return B200Z_ERR_INVALID_ARGUMENT;
                    fi.checksum = rd32le(walk ? walk->wf[i].tail : p + pos);
                    bytes_read += 4;
                }
                break;
            }
        }
        fi.bytes_read_full = bytes_read;
    }
    return 0;
}

// k_walk twice (count, fill) with a host prefix sum in between; 40 bytes per block and 48 per frame come back.  `counted`: w.wf already
// holds the count pass's frame digests (decode_all's candidate walk), so only the fill pass runs.
static int device_walk(b200z_ctx *c, const uint8_t *d_input, size_t input_len, const b200z_frame_io *frames, size_t nframes, WalkHost &w,
                       bool counted = false) {
    if (!counted) w.wf.assign(nframes, WalkFrame());
    w.first.assign(nframes, 0); w.wb.clear();
    if (!nframes) return 0;
    std::vector<uint64_t> so(2 * nframes);
    for (size_t i = 0; i < nframes; i++) { so[i] = frames[i].src_off; so[nframes + i] = frames[i].src_size; }
    DevBuf d_io, d_wf, d_first, d_wb;
    if (int e = d_io.ensure(so.size() * 8, false)) return e;
    if (int e = d_wf.ensure(nframes * sizeof(WalkFrame), false)) return e;
    if (int e = d_first.ensure(nframes * 4, false)) return e;
    CU(c, cudaMemcpyAsync(d_io.p, so.data(), so.size() * 8, cudaMemcpyHostToDevice, c->stream));
    const uint64_t *d_off = d_io.as<uint64_t>(), *d_sz = d_off + nframes;
    int le = 0;
    if (!counted) {
        le = launch_walk(d_input, input_len, d_off, d_sz, (uint32_t)nframes, d_wf.as<WalkFrame>(), nullptr, nullptr, 0, c->stream, &c->launches);
        if (le) return c->set_cuda_err((cudaError_t)le, "k_walk");
        CU(c, cudaMemcpyAsync(w.wf.data(), d_wf.p, nframes * sizeof(WalkFrame), cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
    }
    uint64_t total = 0;
    for (size_t i = 0; i < nframes; i++) { w.first[i] = (uint32_t)total; total += w.wf[i].nblocks; }
    if (total > 0xFFFFFFF0ull) return B200Z_ERR_INVALID_ARGUMENT;
    if (!total) return 0;
    w.wb.resize(total);
    if (int e = d_wb.ensure(total * sizeof(WalkBlock), false)) return e;
    CU(c, cudaMemcpyAsync(d_first.p, w.first.data(), nframes * 4, cudaMemcpyHostToDevice, c->stream));
    le = launch_walk(d_input, input_len, d_off, d_sz, (uint32_t)nframes, d_wf.as<WalkFrame>(), d_first.as<uint32_t>(), d_wb.as<WalkBlock>(), 1, c->stream, &c->launches);
    if (le) return c->set_cuda_err((cudaError_t)le, "k_walk");
    CU(c, cudaMemcpyAsync(w.wb.data(), d_wb.p, total * sizeof(WalkBlock), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return 0;
}

static int batch_upload(b200z_batch *b, const uint8_t *input, size_t input_len, bool on_device);

extern "C" int b200z_batch_prepare(b200z_ctx *c, const uint8_t *input, size_t input_len, int input_mem, const b200z_frame_io *frames,
                                   size_t nframes, const b200z_dict *const *dicts, size_t ndicts, const b200z_dict *forced,
                                   uint64_t max_window, b200z_batch **out) {
    if (!c || !out || (!input && input_len) || (!frames && nframes) || (!dicts && ndicts)) return B200Z_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    if (int e = c->use()) return e;
    std::unique_ptr<b200z_batch> b(new b200z_batch());
    b->ctx = c; b->input_len = input_len;
    const bool on_device = input_mem == B200Z_MEM_DEVICE;
    WalkHost walk;
    if (on_device) {
        // The input stays on the device: k_walk parses the frame / block / section headers there and brings back what the planner
        // needs of each block (SURVEY.md 8(f).3) -- not the compressed data.
        b->d_input = input;
        if (int e = device_walk(c, input, input_len, frames, nframes, walk)) return e;
    }
    if (int e = plan_batch(b.get(), on_device ? nullptr : input, input_len, frames, nframes, dicts, ndicts, forced, max_window, on_device ? &walk : nullptr))
        return e;
    if (int e = batch_upload(b.get(), input, input_len, on_device)) return e;
    *out = b.release();
    return 0;
}

// the device side of a planned batch: the input (copied in when it lives in host memory), descriptors, tables and frame states
static int batch_upload(b200z_batch *b, const uint8_t *input, size_t input_len, bool on_device) {
    b200z_ctx *c = b->ctx;
    if (!on_device) {
        if (int e = b->d_input_own.ensure(input_len + 16, false)) return e;
        if (input_len) CU(c, cudaMemcpyAsync(b->d_input_own.p, input, input_len, cudaMemcpyHostToDevice, c->stream));
        b->d_input = b->d_input_own.as<uint8_t>();
    }
    if (int e = b->sub.upload(c)) return e;
    if (int e = b->d_states_init.ensure(b->sub.states.size() * sizeof(FrameState), false)) return e;
    if (!b->sub.states.empty())
        CU(c, cudaMemcpyAsync(b->d_states_init.p, b->sub.states.data(), b->sub.states.size() * sizeof(FrameState), cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    return 0;
}

// One decode pass in the shipped overlapped order (launch_pipeline_overlapped), then, if `checksummed` is not null and the context has
// B200Z_FLAG_CHECKSUM, k_xxh64 of every frame; *checksummed says whether it ran.  Adds the kernels launched to *launched.
static int enqueue_pass(b200z_ctx *c, const PipelineArgs &a, const PipelineStreams &ps, bool *checksummed, uint64_t *launched) {
    if (int e = launch_pipeline_overlapped(a, ps, launched)) return c->set_cuda_err((cudaError_t)e, "launch_pipeline");
    if (!checksummed) return 0;
    *checksummed = (c->flags & B200Z_FLAG_CHECKSUM) && a.nframes;
    if (*checksummed)
        if (int e = launch_checksum(a, ps.main, launched)) return c->set_cuda_err((cudaError_t)e, "launch_checksum");
    return 0;
}

// every pass starts from the frame states b200z_batch_prepare planned
static int restore_states(b200z_batch *b) {
    b200z_ctx *c = b->ctx;
    const Submission &s = b->sub;
    if (!s.states.empty())
        CU(c, cudaMemcpyAsync(s.d_states.p, b->d_states_init.p, s.states.size() * sizeof(FrameState), cudaMemcpyDeviceToDevice, c->stream));
    return 0;
}

// A decode_all pass: the frames go back to back by the size they decode to, which is known on the device after k_fse.  So the pass
// runs in two stages, as the frame decoder's submissions do: tables, literals and sequences of every block (k_setup, k_huf, k_fse);
// k_place, which writes every frame's out_off / out_cap; then execution (k_exec_cta, k_exec) and, with B200Z_FLAG_CHECKSUM, k_xxh64.
// There is no host round trip in between; what is given up is k_exec running beside k_fse.
// `resume`: the first frame continues from the stream decoder's previous submission (k_place_resume places it behind its carried tail)
static int enqueue_decode_all_stages(b200z_ctx *c, const PipelineArgs &a, const PipelineStreams &ps, bool resume, uint64_t *launched) {
    PipelineArgs a_dec = a;
    a_dec.nframes = 0;
    if (int e = launch_pipeline_overlapped(a_dec, ps, launched)) return c->set_cuda_err((cudaError_t)e, "launch_pipeline (decode)");
    if (int e = resume ? launch_place_resume(a, ps.main, launched) : launch_place(a, ps.main, launched)) return c->set_cuda_err((cudaError_t)e, "k_place");
    PipelineArgs a_ex = a;
    a_ex.nblocks = 0;
    if (int e = launch_pipeline_overlapped(a_ex, ps, launched)) return c->set_cuda_err((cudaError_t)e, "launch_pipeline (execute)");
    return 0;
}
static int enqueue_decode_all_pass(b200z_ctx *c, const PipelineArgs &a, const PipelineStreams &ps, bool *checksummed, uint64_t *launched) {
    if (int e = enqueue_decode_all_stages(c, a, ps, false, launched)) return e;
    *checksummed = (c->flags & B200Z_FLAG_CHECKSUM) && a.nframes;
    if (*checksummed)
        if (int e = launch_checksum(a, ps.main, launched)) return c->set_cuda_err((cudaError_t)e, "launch_checksum");
    return 0;
}

extern "C" int b200z_batch_run(b200z_batch *b, uint8_t *d_output, size_t output_cap) {
    if (!b) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = b->ctx;
    if (int e = c->use()) return e;
    if (int e = restore_states(b)) return e;
    PipelineArgs a = b->sub.args(b->d_input, d_output, output_cap);
    b->run_launches = 0;
    b->ran_output_cap = output_cap;
    const PipelineStreams ps{c->stream, c->side, c->ev_fork, c->ev_join};
    int e = b->decode_all ? enqueue_decode_all_pass(c, a, ps, &b->checksummed, &b->run_launches)
                          : enqueue_pass(c, a, ps, &b->checksummed, &b->run_launches);
    c->launches += b->run_launches;
    if (e) return e;
    b->ran = true;
    return 0;
}

// Same as b200z_batch_run but with a CUDA event between stages; synchronises and reports per-kernel milliseconds.
extern "C" int b200z_batch_run_profile(b200z_batch *b, uint8_t *d_output, size_t output_cap, float *stage_ms, size_t nstages) {
    if (!b || !stage_ms || b->decode_all) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = b->ctx;
    if (int e = c->use()) return e;
    if (int e = restore_states(b)) return e;
    PipelineArgs a = b->sub.args(b->d_input, d_output, output_cap);
    Event ev[kNumStages + 1];
    for (Event &e : ev) if (e.create(c, cudaEventDefault)) return B200Z_ERR_CUDA;
    if (int e = reset_sched(a, c->stream)) return c->set_cuda_err((cudaError_t)e, "reset_sched");
    CU(c, cudaEventRecord(ev[0], c->stream));
    for (int st = 0; st < kNumStages; st++) {
        int e = launch_stage(a, st, c->stream, &c->launches);
        if (e) return c->set_cuda_err((cudaError_t)e, "launch_stage");
        CU(c, cudaEventRecord(ev[st + 1], c->stream));
    }
    CU(c, cudaStreamSynchronize(c->stream));
    for (int st = 0; st < kNumStages && (size_t)st < nstages; st++) CU(c, cudaEventElapsedTime(&stage_ms[st], ev[st], ev[st + 1]));
    b->ran = true;
    return 0;
}
// One pass as b200z_batch_run launches it, with events on the stream: out_ms[0] = 0, out_ms[1..3] = completion time, relative to
// the start of the pass, of the table builds + k_huf (two streams), of the pair k_fse + k_exec (k_exec runs beside k_fse as its programmatic dependent: an event
// between the two would serialise them) and of k_exec_cta + the k_exec launch that takes what it handed back.
extern "C" int b200z_batch_run_timeline(b200z_batch *b, uint8_t *d_output, size_t output_cap, float *out_ms, size_t n) {
    if (!b || !out_ms || n < 4 || b->decode_all) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = b->ctx;
    if (int e = c->use()) return e;
    if (int e = restore_states(b)) return e;
    PipelineArgs a = b->sub.args(b->d_input, d_output, output_cap);
    if (int e = reset_sched(a, c->stream)) return c->set_cuda_err((cudaError_t)e, "reset_sched");
    Event ev[5];
    for (Event &e : ev) if (e.create(c, cudaEventDefault)) return B200Z_ERR_CUDA;
    CU(c, cudaStreamSynchronize(c->stream));
    CU(c, cudaEventRecord(ev[0], c->stream));
    PipelineStreams ps{c->stream, c->side, c->ev_fork, c->ev_join};
    CU(c, cudaEventRecord(ev[1], c->stream));
    int le = launch_tables_literals(a, ps, &c->launches);
    CU(c, cudaEventRecord(ev[2], c->stream));
    if (!le) le = launch_fse_exec(a, c->stream, &c->launches);
    CU(c, cudaEventRecord(ev[3], c->stream));
    if (!le) le = launch_cta_rest(a, c->stream, &c->launches);
    CU(c, cudaEventRecord(ev[4], c->stream));
    if (le) return c->set_cuda_err((cudaError_t)le, "launch_stage");
    CU(c, cudaStreamSynchronize(c->stream));
    for (int i = 0; i < 4; i++) CU(c, cudaEventElapsedTime(&out_ms[i], ev[0], ev[i + 1]));
    return 0;
}
// host-only views of the scheduling decisions (plan.cpp), for CPU tests: no context, no device
extern "C" int b200z_debug_route_frames(const uint64_t *work, const uint8_t *eligible, size_t nframes, uint32_t sms, uint32_t *cta_frames, size_t *n_cta) {
    if ((!work || !eligible) && nframes) return B200Z_ERR_INVALID_ARGUMENT;
    if (!n_cta) return B200Z_ERR_INVALID_ARGUMENT;
    std::vector<uint32_t> out;
    route_exec_frames(work, eligible, nframes, sms, out);
    if (cta_frames) for (size_t i = 0; i < out.size(); i++) cta_frames[i] = out[i];   // room for nframes entries
    *n_cta = out.size();
    return 0;
}
extern "C" int b200z_debug_fse_order(const uint32_t *first_block, const uint32_t *nblocks, const uint8_t *on_cta, size_t nframes, const uint32_t *nseq,
                                     size_t nblocks_total, uint32_t *order, size_t *n_order) {
    if (!n_order || ((!first_block || !nblocks || !on_cta) && nframes) || (!nseq && nblocks_total)) return B200Z_ERR_INVALID_ARGUMENT;
    std::vector<uint32_t> out;
    build_fse_order(first_block, nblocks, on_cta, nframes, nseq, nblocks_total, out);
    if (order) for (size_t i = 0; i < out.size(); i++) order[i] = out[i];   // room for nblocks_total entries
    *n_order = out.size();
    return 0;
}
extern "C" int b200z_num_stages(void) { return kNumStages; }
extern "C" const char *b200z_stage_kernel_name(int stage) { return stage >= 0 && stage < kNumStages ? kStageNames[stage] : ""; }

static void fill_result(const b200z_batch *b, size_t i, const FrameState *st, b200z_frame_result &r) {
    const FramePlanInfo &fi = b->info[i];
    memset(&r, 0, sizeof r);
    r.content_size = fi.hdr.frame_content_size; r.window_size = fi.window;
    r.has_dict_id = fi.hdr.has_dict_id; r.dict_id = fi.hdr.dict_id;
    if (fi.pre_status) {
        r.status = fi.pre_status; r.stage = fi.pre_stage; r.bytes_read = fi.bytes_read_full;
        if (fi.pre_status == B200Z_ERR_SKIP_FRAME) r.content_size = fi.skip_len;
        return;
    }
    r.out_size = st->produced; r.blocks_decoded = st->blocks_done;
    if (st->status == 0) {
        r.bytes_read = fi.bytes_read_full; r.has_checksum = fi.has_checksum; r.checksum_from_data = fi.checksum;
        if (b->checksummed) { r.has_calculated_checksum = 1; r.calculated_checksum = (uint32_t)st->xxh64; }
        return;
    }
    r.status = (int32_t)status_code(st->status); r.stage = (int32_t)status_stage(st->status); r.error_block = st->error_block;
    // bytes_read_from_source at the point the reference returns the error (frame_decoder.rs:325-341)
    uint32_t j = st->blocks_done;
    uint64_t before = j > 0 ? b->block_end_bytes[fi.first_block_end + j - 1] : fi.hdr.header_size;
    if (r.stage == B200Z_STAGE_BLOCK_HEADER) r.bytes_read = before;
    else if (r.stage == B200Z_STAGE_CHECKSUM) r.bytes_read = before;
    else r.bytes_read = before + 3;
}

extern "C" int b200z_batch_finish(b200z_batch *b, b200z_frame_result *results) {
    if (!b || !results || b->decode_all) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = b->ctx;
    if (int e = c->use()) return e;
    std::vector<FrameState> st(b->sub.states.size());
    if (int e = b->sub.download_states(c, st.data(), c->stream)) return e;
    CU(c, cudaStreamSynchronize(c->stream));
    for (size_t i = 0; i < b->info.size(); i++) {
        int32_t sf = b->info[i].sub_frame;
        fill_result(b, i, sf >= 0 ? &st[sf] : nullptr, results[i]);
    }
    return 0;
}

extern "C" int b200z_batch_info(const b200z_batch *b, uint64_t out[8]) {
    if (!b || !out) return B200Z_ERR_INVALID_ARGUMENT;
    const Submission &s = b->sub;
    uint64_t ncomp = 0, planned = 0;
    for (auto &d : s.descs) { ncomp += d.btype == BT_COMPRESSED; planned += d.src_size + 3; }
    out[0] = b->decode_all ? b->zstd_frames : s.frames.size(); out[1] = s.descs.size(); out[2] = ncomp; out[3] = planned; out[4] = s.lit_bytes; out[5] = s.nseq;
    out[6] = b->run_launches; out[7] = 0;
    return 0;
}

extern "C" int b200z_batch_debug_literals(b200z_batch *b, uint32_t block, uint8_t *host_out, size_t cap, size_t *len) {
    if (!b || block >= b->sub.descs.size() || !len) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = b->ctx;
    const BlockDesc &d = b->sub.descs[block];
    *len = 0;
    if (d.btype != BT_COMPRESSED || (d.lit_type != LT_COMPRESSED && d.lit_type != LT_TREELESS)) return 0;
    if (cap < d.regen_size) return B200Z_ERR_TARGET_TOO_SMALL;
    CU(c, cudaStreamSynchronize(c->stream));
    CU(c, cudaMemcpy(host_out, b->sub.d_lit.as<uint8_t>() + d.lit_buf_off, d.regen_size, cudaMemcpyDeviceToHost));
    *len = d.regen_size;
    return 0;
}
extern "C" int b200z_batch_debug_sequences(b200z_batch *b, uint32_t block, uint32_t *host_out, size_t cap_seqs, size_t *nseq) {
    if (!b || block >= b->sub.descs.size() || !nseq) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = b->ctx;
    const BlockDesc &d = b->sub.descs[block];
    *nseq = 0;
    if (d.btype != BT_COMPRESSED || d.nseq == 0) return 0;
    if (cap_seqs < d.nseq) return B200Z_ERR_TARGET_TOO_SMALL;
    CU(c, cudaStreamSynchronize(c->stream));
    CU(c, cudaMemcpy(host_out, b->sub.d_seq.as<uint32_t>() + d.seq_buf_off * 3, (size_t)d.nseq * 12, cudaMemcpyDeviceToHost));
    // the device holds prefix sums {out_end, lit_end, of}: hand out {ll, ml, of} (of: see b200z_batch_debug_block_flags)
    uint32_t p_out = 0, p_lit = 0;
    for (size_t i = 0; i < d.nseq; i++) {
        uint32_t *r = host_out + 3 * i;
        const uint32_t oe = r[0], le = r[1], ll = le - p_lit, ml = oe - p_out - ll;
        r[0] = ll; r[1] = ml; p_out = oe; p_lit = le;
    }
    *nseq = d.nseq;
    return 0;
}
// the tables a block decodes with, as the planner resolved them into its descriptor (the defining slot for Treeless / Repeat,
// the predefined tables, a dictionary's or the streaming carry's tables), copied raw; a null table is reported absent
extern "C" int b200z_batch_debug_tables(b200z_batch *b, uint32_t block, uint8_t *huf_out, uint8_t *fse_out, uint32_t present[4]) {
    if (!b || block >= b->sub.descs.size() || !huf_out || !fse_out || !present) return B200Z_ERR_INVALID_ARGUMENT;
    static_assert(sizeof(HufSlot) == B200Z_DEBUG_HUF_BYTES && sizeof(FseTab) == B200Z_DEBUG_FSE_BYTES, "b200zstd.h table sizes");
    b200z_ctx *c = b->ctx;
    const BlockDesc &d = b->sub.descs[block];
    CU(c, cudaStreamSynchronize(c->stream));
    present[0] = d.huf != nullptr;
    if (d.huf) CU(c, cudaMemcpy(huf_out, d.huf, sizeof(HufSlot), cudaMemcpyDeviceToHost));
    const FseTab *t[3] = {d.ll, d.of, d.ml};
    for (int k = 0; k < 3; k++) {
        present[1 + k] = t[k] != nullptr;
        if (t[k]) CU(c, cudaMemcpy(fse_out + k * sizeof(FseTab), t[k], sizeof(FseTab), cudaMemcpyDeviceToHost));
    }
    return 0;
}
// flags of a block's sequence stage: bit 0 = `of` values are raw offset_values (otherwise offsets after do_offset_history,
// symbolic where they depend on the history at the block's start: tag << 30 | decrements, tag 1..3 = history slot + 1)
extern "C" int b200z_batch_debug_block_flags(b200z_batch *b, uint32_t block, uint32_t *flags) {
    if (!b || block >= b->sub.descs.size() || !flags) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = b->ctx;
    CU(c, cudaStreamSynchronize(c->stream));
    BlockAux ax;
    CU(c, cudaMemcpy(&ax, b->sub.d_aux.as<BlockAux>() + block, sizeof ax, cudaMemcpyDeviceToHost));
    *flags = ax.flags;
    return 0;
}
// execution scheduling counters of the LAST run: [0] frames given to k_exec_cta, [1] frames it handed back to k_exec,
// [2] OR of the reasons (XC_WHY_* in exec_cta.cuh), [3] blocks left to k_exec
extern "C" int b200z_batch_debug_sched(b200z_batch *b, uint32_t out[4]) {
    if (!b || !out) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = b->ctx;
    out[0] = (uint32_t)b->sub.cta_frames.size(); out[1] = out[2] = out[3] = 0;
    if (!b->sub.d_sched.p) return 0;
    CU(c, cudaStreamSynchronize(c->stream));
    uint32_t h[4];
    CU(c, cudaMemcpy(h, b->sub.d_sched.p, sizeof h, cudaMemcpyDeviceToHost));
    out[1] = h[1]; out[2] = h[2]; out[3] = h[3];
    return 0;
}
// waves of the literal and sequence kernels for this batch's blocks: [0] k_huf, [1] k_fse, [2] / [3] their resident CTAs per SM
extern "C" int b200z_batch_debug_waves(b200z_batch *b, uint32_t out[4]) {
    if (!b || !out) return B200Z_ERR_INVALID_ARGUMENT;
    if (cudaSetDevice(b->ctx->device) != cudaSuccess) { cudaGetLastError(); return B200Z_ERR_CUDA; }
    entropy_waves((uint32_t)b->sub.descs.size(), out);
    return 0;
}
extern "C" void b200z_batch_destroy(b200z_batch *b) {
    if (!b) return;
    cudaSetDevice(b->ctx->device);
    delete b;
}

// ---------------------------------------------------------------------------------------------------------------
// Pipelined one-shot for HOST buffers: the frame list is cut into a few chunks; while chunk i is being decoded,
// chunk i+1 is planned on the host and its input crosses PCIe, and chunk i-1's plaintext is on its way back.
// Three streams (H2D, compute, D2H) + two descriptor/scratch sets; all device buffers live in the context and are
// reused across calls.
// ---------------------------------------------------------------------------------------------------------------
struct PipeResources {
    Stream s_h2d, s_d2h;
    // chunk i's kernels run on stream pair i & 1, so the (latency-bound) kernels of neighbouring chunks overlap
    Stream k_main[2], k_side[2];
    Event k_fork[2], k_join[2];
    std::unique_ptr<b200z_batch> set[2];
    Event ev_h2d[2], ev_k[2], ev_done[2];
    PinnedBuf h_states[2];   // FrameState
    DevBuf d_in[2];
    DevBuf d_out;
};

static int pipe_get(b200z_ctx *c, PipeResources **out) {
    if (!c->pipe) {
        std::unique_ptr<PipeResources> p(new PipeResources());
        if (p->s_h2d.create(c) || p->s_d2h.create(c)) return B200Z_ERR_CUDA;
        int prio_lo = 0, prio_hi = 0;
        cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
        for (int i = 0; i < 2; i++) {
            if (p->k_main[i].create(c, prio_hi) || p->k_side[i].create(c, prio_lo) || p->k_fork[i].create(c) || p->k_join[i].create(c) ||
                p->ev_h2d[i].create(c) || p->ev_k[i].create(c) || p->ev_done[i].create(c))
                return B200Z_ERR_CUDA;
            p->set[i].reset(new b200z_batch());
            p->set[i]->ctx = c;
        }
        c->pipe = std::move(p);
    }
    *out = c->pipe.get();
    return 0;
}

// Host output: copies the byte ranges [lo, hi) of `ranges` from the device output back to `output`, and nothing between them, so the
// caller's bytes outside every frame's slot stay as they were.  Ranges that touch or overlap go back in one copy: frames packed back to
// back cost one copy, as one range over all of them did.  Ranges apart from each other come back one copy each while there are few;
// past that, one copy of their span lands in a host staging buffer and each range is copied out of it (one PCIe transfer, not one
// per frame).  `sync`: the staging path and the caller need the bytes now; without it the direct copies stay queued on `stream`.
static int copy_back_ranges(b200z_ctx *c, cudaStream_t stream, uint8_t *output, const uint8_t *d_out, std::vector<std::pair<uint64_t, uint64_t>> &ranges,
                            bool sync) {
    std::sort(ranges.begin(), ranges.end());
    std::vector<std::pair<uint64_t, uint64_t>> merged;
    for (const auto &r : ranges) {
        if (r.second <= r.first) continue;
        if (!merged.empty() && r.first <= merged.back().second) merged.back().second = std::max(merged.back().second, r.second);
        else merged.push_back(r);
    }
    if (merged.empty()) return 0;
    const size_t kDirect = 16;
    if (merged.size() <= kDirect || !sync) {
        for (const auto &r : merged) CU(c, cudaMemcpyAsync(output + r.first, d_out + r.first, r.second - r.first, cudaMemcpyDeviceToHost, stream));
        if (sync) CU(c, cudaStreamSynchronize(stream));
        return 0;
    }
    const uint64_t lo = merged.front().first, hi = merged.back().second;
    std::vector<uint8_t> staging(hi - lo);
    CU(c, cudaMemcpyAsync(staging.data(), d_out + lo, hi - lo, cudaMemcpyDeviceToHost, stream));
    CU(c, cudaStreamSynchronize(stream));
    for (const auto &r : merged) memcpy(output + r.first, staging.data() + (r.first - lo), r.second - r.first);
    return 0;
}

static int decode_frames_pipelined(b200z_ctx *c, const uint8_t *input, size_t input_len, const b200z_frame_io *frames, size_t nframes,
                                   const b200z_dict *const *dicts, size_t ndicts, const b200z_dict *forced, uint64_t max_window, uint8_t *output,
                                   size_t output_cap, b200z_frame_result *results, size_t nchunks) {
    PipeResources *p = nullptr;
    if (int e = pipe_get(c, &p)) return e;
    if (int e = p->d_out.ensure(output_cap + 64, false)) return e;
    uint8_t *d_out = p->d_out.as<uint8_t>();
    // chunk boundaries: consecutive frames, roughly equal output bytes
    uint64_t total_cap = 0;
    for (size_t i = 0; i < nframes; i++) total_cap += frames[i].out_cap;
    std::vector<size_t> cut(1, 0);
    {
        uint64_t acc = 0, per = total_cap / nchunks + 1;
        for (size_t i = 0; i < nframes; i++) {
            acc += frames[i].out_cap;
            if (acc >= per * cut.size() && i + 1 < nframes && cut.size() < nchunks) cut.push_back(i + 1);
        }
        cut.push_back(nframes);
    }
    struct Pending { size_t f0 = 0, f1 = 0; bool live = false; } pend[2];
    auto retire = [&](int s) -> int {   // results of the chunk that used set s
        if (!pend[s].live) return 0;
        CU(c, cudaEventSynchronize(p->ev_done[s]));
        const b200z_batch *b = p->set[s].get();
        for (size_t i = pend[s].f0; i < pend[s].f1; i++) {
            int32_t sf = b->info[i - pend[s].f0].sub_frame;
            fill_result(b, i - pend[s].f0, sf >= 0 ? p->h_states[s].as<FrameState>() + sf : nullptr, results[i]);
        }
        pend[s].live = false;
        return 0;
    };
    for (size_t ci = 0; ci + 1 < cut.size(); ci++) {
        const int s = (int)(ci & 1);
        const size_t f0 = cut[ci], f1 = cut[ci + 1];
        if (int e = retire(s)) return e;
        b200z_batch *b = p->set[s].get();
        if (int e = plan_batch(b, input, input_len, frames + f0, f1 - f0, dicts, ndicts, forced, max_window)) return e;
        // input byte range and the output slots of this chunk (the frames' sizes are not known before the chunk retires)
        uint64_t ilo = UINT64_MAX, ihi = 0;
        std::vector<std::pair<uint64_t, uint64_t>> slots;
        for (size_t i = f0; i < f1; i++) {
            if (frames[i].src_off > input_len || frames[i].src_size > input_len - frames[i].src_off) continue;
            ilo = std::min<uint64_t>(ilo, frames[i].src_off); ihi = std::max<uint64_t>(ihi, frames[i].src_off + frames[i].src_size);
            if (frames[i].out_cap && frames[i].out_off < output_cap)
                slots.emplace_back(frames[i].out_off, std::min<uint64_t>(frames[i].out_off + std::min<uint64_t>(frames[i].out_cap, output_cap), output_cap));
        }
        if (ihi < ilo) { ilo = ihi = 0; }
        if (int e = p->d_in[s].ensure(ihi - ilo + 32)) return e;
        if (ihi > ilo) CU(c, cudaMemcpyAsync(p->d_in[s].p, input + ilo, ihi - ilo, cudaMemcpyHostToDevice, p->s_h2d));
        if (int e = b->sub.upload(c, p->s_h2d)) return e;
        CU(c, cudaEventRecord(p->ev_h2d[s], p->s_h2d));
        cudaStream_t km = p->k_main[s];
        CU(c, cudaStreamWaitEvent(km, p->ev_h2d[s], 0));
        PipelineArgs a = b->sub.args(p->d_in[s].as<uint8_t>() - ilo, d_out, output_cap);
        if (int e = enqueue_pass(c, a, PipelineStreams{km, p->k_side[s], p->k_fork[s], p->k_join[s]}, &b->checksummed, &c->launches)) return e;
        CU(c, cudaEventRecord(p->ev_k[s], km));
        CU(c, cudaStreamWaitEvent(p->s_d2h, p->ev_k[s], 0));
        if (int e = p->h_states[s].ensure(b->sub.states.size() * sizeof(FrameState))) return e;
        if (int e = b->sub.download_states(c, p->h_states[s].as<FrameState>(), p->s_d2h)) return e;
        if (int e = copy_back_ranges(c, p->s_d2h, output, d_out, slots, false)) return e;
        CU(c, cudaEventRecord(p->ev_done[s], p->s_d2h));
        pend[s].f0 = f0; pend[s].f1 = f1; pend[s].live = true;
    }
    if (int e = retire(0)) return e;
    if (int e = retire(1)) return e;
    return 0;
}

extern "C" int b200z_decode_frames_batch(b200z_ctx *c, const uint8_t *input, size_t input_len, int input_mem, const b200z_frame_io *frames,
                                         size_t nframes, const b200z_dict *const *dicts, size_t ndicts, const b200z_dict *forced,
                                         uint64_t max_window, uint8_t *output, size_t output_cap, int output_mem, b200z_frame_result *results) {
    if (!c || !results || (!output && output_cap)) return B200Z_ERR_INVALID_ARGUMENT;
    if (input_mem != B200Z_MEM_DEVICE && output_mem != B200Z_MEM_DEVICE && nframes >= 64) {
        // host in, host out: overlap planning, PCIe and kernels
        if (int e0 = c->use()) return e0;
        if ((!input && input_len) || (!frames && nframes) || (!dicts && ndicts)) return B200Z_ERR_INVALID_ARGUMENT;
        uint64_t total_cap = 0;
        for (size_t i = 0; i < nframes; i++) total_cap += frames[i].out_cap;
        uint64_t chunk_bytes = 256ull << 20;   // ~4 chunks per GiB: PCIe transfers and kernels of neighbouring chunks overlap
        if (const char *ev = getenv("B200Z_PIPELINE_CHUNK_BYTES")) { uint64_t v = strtoull(ev, nullptr, 10); if (v >= 4096) chunk_bytes = v; }
        size_t nchunks = (size_t)std::min<uint64_t>(16, std::max<uint64_t>(1, total_cap / chunk_bytes));
        return decode_frames_pipelined(c, input, input_len, frames, nframes, dicts, ndicts, forced, max_window, output, output_cap, results, nchunks);
    }
    b200z_batch *b = nullptr;
    int e = b200z_batch_prepare(c, input, input_len, input_mem, frames, nframes, dicts, ndicts, forced, max_window, &b);
    if (e) return e;
    std::unique_ptr<b200z_batch, void (*)(b200z_batch *)> guard(b, b200z_batch_destroy);
    DevBuf d_out;
    uint8_t *dout = output;
    if (output_mem != B200Z_MEM_DEVICE) {
        if ((e = d_out.ensure(output_cap + 16, false))) return e;
        dout = d_out.as<uint8_t>();
    }
    if ((e = b200z_batch_run(b, dout, output_cap))) return e;
    if ((e = b200z_batch_finish(b, results))) return e;
    if (output_mem != B200Z_MEM_DEVICE) {
        // every frame's produced bytes (frames are normally packed back to back by the caller: one copy)
        std::vector<std::pair<uint64_t, uint64_t>> produced;
        for (size_t i = 0; i < nframes; i++)
            if (results[i].out_size && frames[i].out_off < output_cap)
                produced.emplace_back(frames[i].out_off, std::min<uint64_t>(frames[i].out_off + std::min<uint64_t>(results[i].out_size, frames[i].out_cap), output_cap));
        if ((e = copy_back_ranges(c, c->stream, output, dout, produced, true))) return e;
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// tier 1c: decode_all on the batch path (FrameDecoder::decode_all, frame_decoder.rs:541-577) -- find the frames of a buffer of
// concatenated frames, decode them in one submission, place them back to back by decoded size on the device (k_place)
// ---------------------------------------------------------------------------------------------------------------
namespace {

struct Chain {
    std::vector<uint64_t> at;    // input offset of every frame visited, the one where the chain ends included
    std::vector<WalkFrame> wf;   // its header walk (a zeroed digest where no frame starts: it parses as BadMagicNumber / MagicNumberRead)
};

// decode_all's way from one frame to the next, from offset 0 (frame_chain_next, framing.cuh): it ends at the end of the input, at a
// break in the chain, or at a skippable frame that runs past the input.  walk_at(pos) gives the walk of the frame at pos, or null when
// no frame starts there.
template <class WalkAt>
void follow_chain(uint64_t input_len, WalkAt walk_at, Chain &ch) {
    ch.at.clear(); ch.wf.clear();
    for (uint64_t pos = 0; pos < input_len;) {
        WalkFrame none;
        const WalkFrame *F = walk_at(pos);
        if (!F) {
            memset(&none, 0, sizeof none);
            none.hdr_avail = (uint32_t)std::min<uint64_t>(input_len - pos, 20);
            none.stop = 4;
            F = &none;
        }
        ch.at.push_back(pos); ch.wf.push_back(*F);
        const uint64_t next = frame_chain_next(pos, *F);
        if (next == pos || next > input_len) break;
        pos = next;
    }
}

// host input: the same walk as k_walk, on the host
void host_chain(const uint8_t *in, uint64_t input_len, Chain &ch) {
    WalkFrame F;
    follow_chain(input_len, [&](uint64_t pos) -> const WalkFrame * { walk_frame(in + pos, input_len - pos, F, nullptr, nullptr, 0, 0); return &F; }, ch);
}

// device input: the chain through the candidate frame starts (any order) and their walks with the bytes left from each
void chain_from_candidates(uint64_t input_len, const std::vector<uint64_t> &cand, const std::vector<WalkFrame> &cand_wf, Chain &ch) {
    std::vector<uint32_t> order(cand.size());
    for (uint32_t i = 0; i < order.size(); i++) order[i] = i;
    std::sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return cand[x] < cand[y]; });
    std::vector<uint64_t> sorted(cand.size());
    for (size_t i = 0; i < order.size(); i++) sorted[i] = cand[order[i]];
    follow_chain(input_len, [&](uint64_t pos) -> const WalkFrame * {
        auto it = std::lower_bound(sorted.begin(), sorted.end(), pos);
        return it != sorted.end() && *it == pos ? &cand_wf[order[it - sorted.begin()]] : nullptr;
    }, ch);
}

bool is_frame_magic(const uint8_t *p) { const uint32_t m = rd32le(p); return m == ZSTD_MAGIC || skippable_magic(m); }

}  // namespace

// k_find_frames, then k_walk in count mode once per candidate; the candidates' offsets and frame digests come back, not the input
static int device_chain(b200z_ctx *c, const uint8_t *d_input, uint64_t input_len, Chain &ch) {
    std::vector<uint64_t> cand;
    std::vector<WalkFrame> cand_wf;
    uint64_t n = 0;
    if (input_len >= 4) {
        uint64_t cap = 4096 + input_len / 16384;
        DevBuf d_cand, d_count, d_wf;
        for (;;) {
            if (cap > 0xFFFFFFF0ull) return B200Z_ERR_INVALID_ARGUMENT;
            if (int e = d_cand.ensure(2 * cap * 8, false)) return e;
            if (int e = d_count.ensure(8, false)) return e;
            CU(c, cudaMemsetAsync(d_count.p, 0, 8, c->stream));
            uint64_t *d_off = d_cand.as<uint64_t>(), *d_size = d_off + cap;
            if (int le = launch_find_frames(d_input, input_len, d_off, d_size, (uint32_t)cap, d_count.as<unsigned long long>(), c->stream, &c->launches))
                return c->set_cuda_err((cudaError_t)le, "k_find_frames");
            CU(c, cudaMemcpyAsync(&n, d_count.p, 8, cudaMemcpyDeviceToHost, c->stream));
            CU(c, cudaStreamSynchronize(c->stream));
            if (n <= cap) break;
            cap = n;   // more candidates than room (false candidates are ordinary input): grow and scan again
        }
        if (n) {
            uint64_t *d_off = d_cand.as<uint64_t>(), *d_size = d_off + cap;
            if (int e = d_wf.ensure(n * sizeof(WalkFrame), false)) return e;
            if (int le = launch_walk(d_input, input_len, d_off, d_size, (uint32_t)n, d_wf.as<WalkFrame>(), nullptr, nullptr, 0, c->stream, &c->launches))
                return c->set_cuda_err((cudaError_t)le, "k_walk");
            cand.resize(n); cand_wf.resize(n);
            CU(c, cudaMemcpyAsync(cand.data(), d_off, n * 8, cudaMemcpyDeviceToHost, c->stream));
            CU(c, cudaMemcpyAsync(cand_wf.data(), d_wf.p, n * sizeof(WalkFrame), cudaMemcpyDeviceToHost, c->stream));
            CU(c, cudaStreamSynchronize(c->stream));
        }
    }
    chain_from_candidates(input_len, cand, cand_wf, ch);
    return 0;
}

extern "C" int b200z_debug_decode_all_chain(const uint8_t *input, size_t input_len, int by_candidates, uint64_t *at, size_t cap, size_t *n) {
    if (!n || (!input && input_len) || (!at && cap)) return B200Z_ERR_INVALID_ARGUMENT;
    Chain ch;
    if (!by_candidates) host_chain(input, input_len, ch);
    else {
        std::vector<uint64_t> cand;
        std::vector<WalkFrame> cand_wf;
        for (uint64_t p = 0; p + 4 <= input_len; p++) {
            if (!is_frame_magic(input + p)) continue;
            cand.push_back(p);
            cand_wf.emplace_back();
            walk_frame(input + p, input_len - p, cand_wf.back(), nullptr, nullptr, 0, 0);
        }
        std::reverse(cand.begin(), cand.end());   // the device's candidates come in no particular order
        std::reverse(cand_wf.begin(), cand_wf.end());
        chain_from_candidates(input_len, cand, cand_wf, ch);
    }
    for (size_t i = 0; i < ch.at.size() && i < cap; i++) at[i] = ch.at[i];
    *n = ch.at.size();
    return 0;
}

extern "C" int b200z_decode_all_prepare(b200z_ctx *c, const uint8_t *input, size_t input_len, int input_mem, const b200z_dict *const *dicts,
                                        size_t ndicts, const b200z_dict *forced, uint64_t max_window, b200z_batch **out) {
    if (!c || !out || (!input && input_len) || (!dicts && ndicts)) return B200Z_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    if (int e = c->use()) return e;
    std::unique_ptr<b200z_batch> b(new b200z_batch());
    b->ctx = c; b->input_len = input_len; b->decode_all = true;
    const bool on_device = input_mem == B200Z_MEM_DEVICE;
    Chain ch;
    if (on_device) {
        b->d_input = input;
        if (int e = device_chain(c, input, input_len, ch)) return e;
    } else {
        host_chain(input, input_len, ch);
    }
    // every frame of the chain is planned with the rest of the input; the plaintexts are placed by k_place on every run
    std::vector<b200z_frame_io> io(ch.at.size());
    b->chain = ch.at;
    b->chain_zstd.assign(ch.at.size(), 0);
    for (size_t i = 0; i < io.size(); i++) {
        io[i] = b200z_frame_io{ch.at[i], input_len - ch.at[i], 0, 0};
        b->chain_zstd[i] = ch.wf[i].hdr_avail >= 4 && rd32le(ch.wf[i].hdr) == ZSTD_MAGIC;
        b->zstd_frames += b->chain_zstd[i];
    }
    WalkHost walk;
    if (on_device) {
        walk.wf = ch.wf;   // the candidates' count pass: only the fill pass runs again
        if (int e = device_walk(c, input, input_len, io.data(), io.size(), walk, true)) return e;
    }
    if (int e = plan_batch(b.get(), on_device ? nullptr : input, input_len, io.data(), io.size(), dicts, ndicts, forced, max_window, on_device ? &walk : nullptr))
        return e;
    if (int e = batch_upload(b.get(), input, input_len, on_device)) return e;
    *out = b.release();
    return 0;
}

// decode_all's loop over the frame that runs out of output (frame_decoder.rs:556-572): decode_blocks(UptoBytes(1 MiB)), read what the
// output still holds, TargetTooSmall while the decode buffer keeps collectable bytes (the window is kept until the frame is finished).
// size[0..n) are the bytes of the blocks that decode.  fails: the frame's error comes next -- block n fails, or, when
// `last_is_final` (block n - 1 is the frame's last block), the content checksum cannot be read.  Returns true when the reference
// raises TargetTooSmall before that error (or before the end of the frame).
static bool decode_all_runs_out_first(const uint64_t *size, uint32_t n, bool fails, bool last_is_final, uint64_t window, uint64_t room) {
    uint64_t buf = 0;
    uint32_t i = 0;
    for (;;) {
        uint64_t grown = 0;
        bool finished = false;
        for (;;) {
            if (i == n) return false;   // block n fails before anything more is read
            buf += size[i]; grown += size[i]; i++;
            if (i == n && last_is_final) {
                if (fails) return false;   // FailedToReadChecksum, in the same decode_blocks call
                finished = true;
                break;
            }
            if (grown >= (1u << 20)) break;
        }
        const uint64_t drainable = finished ? buf : (buf > window ? buf - window : 0);
        const uint64_t amount = std::min(room, drainable);
        room -= amount; buf -= amount;
        if (finished ? buf : (buf > window ? buf - window : 0)) return true;
        if (finished) return false;
    }
}

extern "C" int b200z_decode_all_finish(b200z_batch *b, b200z_all_result *sum, b200z_frame_result *results) {
    if (!b || !sum || !b->decode_all) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = b->ctx;
    if (int e = c->use()) return e;
    const Submission &s = b->sub;
    std::vector<FrameState> st(s.states.size());
    if (int e = s.download_states(c, st.data(), c->stream)) return e;
    CU(c, cudaStreamSynchronize(c->stream));
    memset(sum, 0, sizeof *sum);
    sum->error_offset = b->input_len;
    sum->error_frame = -1;
    bool failed = false;
    auto fail = [&](uint32_t word, size_t i, int32_t zi) {
        failed = true;
        sum->status = (int32_t)status_code(word); sum->stage = (int32_t)status_stage(word);
        sum->error_offset = b->chain[i]; sum->error_frame = zi;
    };
    int32_t zi = -1;
    for (size_t i = 0; i < b->chain.size(); i++) {
        const FramePlanInfo &fi = b->info[i];
        const FrameState *fs = fi.sub_frame >= 0 ? &st[fi.sub_frame] : nullptr;
        if (b->chain_zstd[i]) { zi++; if (results) fill_result(b, i, fs, results[zi]); }
        if (failed) continue;
        if (fi.pre_status == B200Z_ERR_SKIP_FRAME) {   // `input.get(length..)`: the skipped bytes must be there
            if (b->chain[i] + 8 + fi.skip_len > b->input_len) fail(mk_status(B200Z_ERR_FAILED_TO_SKIP_FRAME, B200Z_STAGE_FRAME_HEADER), i, -1);
            else sum->skippable_frames++;
            continue;
        }
        if (fi.pre_status) { fail(mk_status((uint32_t)fi.pre_status, (uint32_t)fi.pre_stage), i, b->chain_zstd[i] ? zi : -1); continue; }
        if (fs->status == 0) { sum->written += fs->produced; sum->frames++; continue; }
        // The first failing frame.  What the device found first is the reference's error unless the output ran out before it: replay
        // decode_all's loop over the frame's block sizes.  With TargetTooSmall from the device (the frame did not fit), the error that
        // may come before it is the first one stage A or the planner found.
        const FrameDesc &fd = s.frames[fi.sub_frame];
        std::vector<BlockAux> aux(fd.nblocks);
        if (fd.nblocks) {
            if (int e = s.download_aux(c, aux.data(), fd.first_block, fd.nblocks, c->stream)) return e;
            CU(c, cudaStreamSynchronize(c->stream));
        }
        uint32_t word = fs->status, n = fs->blocks_done;
        bool fails = true;
        if (status_code(word) == B200Z_ERR_TARGET_TOO_SMALL) {
            word = fd.host_status; n = fd.nblocks;
            for (uint32_t k = 0; k < fd.nblocks; k++) {
                const BlockAux &x = aux[k];
                if (uint32_t w = block_first_error(s.descs[fd.first_block + k].host_status, x.status, x.seq_status)) { word = w; n = k; break; }
            }
            fails = word != 0;
        }
        std::vector<uint64_t> size(n);
        for (uint32_t k = 0; k < n; k++) size[k] = aux[k].out_size;
        const bool last_is_final = n > 0 && s.descs[fd.first_block + n - 1].last;
        if (decode_all_runs_out_first(size.data(), n, fails, last_is_final, fi.window, b->ran_output_cap - sum->written))
            word = mk_status(B200Z_ERR_TARGET_TOO_SMALL, 0);
        fail(word, i, zi);
    }
    return 0;
}

extern "C" int b200z_decode_all_batch(b200z_ctx *c, const uint8_t *input, size_t input_len, int input_mem, const b200z_dict *const *dicts,
                                      size_t ndicts, const b200z_dict *forced, uint64_t max_window, uint8_t *output, size_t output_cap,
                                      int output_mem, b200z_all_result *summary) {
    if (!c || !summary || (!output && output_cap)) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_batch *b = nullptr;
    int e = b200z_decode_all_prepare(c, input, input_len, input_mem, dicts, ndicts, forced, max_window, &b);
    if (e) return e;
    std::unique_ptr<b200z_batch, void (*)(b200z_batch *)> guard(b, b200z_batch_destroy);
    DevBuf d_out;
    uint8_t *dout = output;
    if (output_mem != B200Z_MEM_DEVICE) {
        if ((e = d_out.ensure(output_cap + 16, false))) return e;
        dout = d_out.as<uint8_t>();
    }
    if ((e = b200z_batch_run(b, dout, output_cap))) return e;
    if ((e = b200z_decode_all_finish(b, summary, nullptr))) return e;
    if (output_mem != B200Z_MEM_DEVICE && summary->written) {
        CU(c, cudaMemcpyAsync(output, dout, summary->written, cudaMemcpyDeviceToHost, c->stream));
        CU(c, cudaStreamSynchronize(c->stream));
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// tier 1d: decode_all from a reader to a writer (b200z_decode_all_stream).  The source is cut at block ends into submissions of
// bounded input and output; each is a decode_all pass (enqueue_decode_all_stages).  A frame that runs past a cut continues in the
// next submission from its state, tables and window tail, carried device to device (k_carry, the table copies below).
// ---------------------------------------------------------------------------------------------------------------
namespace {

constexpr uint64_t SD_BLOCK_ROOM = 18 + 3 + 131072 + 4;   // a frame header, one block and a checksum: a submission always takes one block

// The cut rules' bounds for a chunk of C bytes (DESIGN.md 4.9).  A submission with one block may exceed any of them.
struct SdBounds {
    uint64_t chunk, out, blocks, seqs;
    explicit SdBounds(uint64_t C) : chunk(C), out(4 * C), blocks(std::max<uint64_t>(1, C / 16384)), seqs(C / 4) {}
    uint64_t buffer() const { return chunk + 2 * SD_BLOCK_ROOM; }   // host input per slot: no cut is ever forced by it
    uint64_t out_room() const { return std::max<uint64_t>(out, 131072); }
};

// the source, read into the buffer of the submission being planned: buf[0, have) holds stream bytes from offset `off` on
struct SdSource {
    b200z_read_fn rd = nullptr;
    void *user = nullptr;
    uint8_t *buf = nullptr;
    size_t have = 0, cap = 0, peak = 0;
    uint64_t off = 0;
    bool eof = false;
    std::vector<uint8_t> scratch;
    // buf[0, n) available, unless the source ends first (a read that fails or returns more than asked for ends it, as the frame
    // decoder's reader treats them); n <= cap
    bool fill(size_t n) {
        while (have < n && !eof) {
            const long r = rd(user, buf + have, cap - have);
            if (r <= 0 || (size_t)r > cap - have) { eof = true; break; }
            have += (size_t)r;
        }
        peak = std::max(peak, have);
        return have >= n;
    }
    // drops the n bytes at the front, reading and discarding those past the buffer (a skippable frame is never buffered); false when
    // the source ends first
    bool drop(uint64_t n) {
        if (n <= have) { memmove(buf, buf + n, have - n); have -= (size_t)n; off += n; return true; }
        n -= have; off += have; have = 0;
        scratch.resize(1 << 16);
        while (n) {
            const long r = eof ? 0 : rd(user, scratch.data(), (size_t)std::min<uint64_t>(n, scratch.size()));
            if (r <= 0 || (uint64_t)r > n) { eof = true; return false; }
            n -= (uint64_t)r; off += (uint64_t)r;
        }
        return true;
    }
    // the bytes after a cut at `cut` become the front of `next`, the buffer of the next submission
    void advance(size_t cut, uint8_t *next) {
        if (have > cut) memmove(next, buf + cut, have - cut);
        have -= cut; off += cut; buf = next;
    }
};

struct SdFrame {                  // a frame of a planned submission
    uint64_t at = 0;              // stream offset of its magic number
    int32_t zi = 0;               // its index among the zstd frames
    uint32_t skips_before = 0;    // skippable frames passed between the previous frame and this one
    bool has_checksum = false;    // the checksum it carries was read in this submission
    uint32_t checksum = 0;
};

// the frame that continues past the submission planned last
struct SdCont {
    bool on = false;
    SdFrame frame;
    const b200z_dict *dict = nullptr;
    uint64_t window = 0;
    bool checksum = false;
    uint32_t next_block = 0;
    CarrySet tables;              // what its next block starts from
};

struct SdPlan {
    std::vector<SdFrame> frames;
    bool resumed = false, continues = false, ends = false;   // ends: nothing comes after it (end of the source, or an error)
    size_t cut = 0;               // buffer bytes the submission takes
    uint64_t start = 0, in_bytes = 0, out_bound = 0, nblocks = 0, nseq = 0;
    uint32_t skips_after = 0;
    uint32_t end_word = 0;        // an error the cutter found past the submission's frames (status word), 0 = none
    uint64_t end_at = 0;
    int32_t end_zi = -1;
    uint64_t resume_window = 0;   // window of the resumed frame
    TableCursor cur_end;          // the continuing frame's tables after its last block here (what the next submission copies)
};

struct SdPlanner {
    SdBounds bnd;
    const b200z_dict *const *dicts;
    size_t ndicts;
    const b200z_dict *forced;
    uint64_t max_window;
    const HufSlot *carry_huf = nullptr;     // where the continuing frame's tables are carried (device)
    const FseSlot *carry_fse = nullptr;
    const FseSlot *predef = nullptr;
    SdCont cont;
    int32_t zi = -1;
    uint64_t max_window_seen = 0;
    SdPlanner(uint64_t C, const b200z_dict *const *d, size_t nd, const b200z_dict *f, uint64_t mw)
        : bnd(C), dicts(d), ndicts(nd), forced(f), max_window(window_limit(mw)) {}

    // the most a block adds to the output: a Raw / RLE block's size, min(128 KiB, window) for a Compressed block
    static uint64_t out_of(const BlockHeader &bh, uint64_t window) { return bh.type == BT_COMPRESSED ? std::min<uint64_t>(131072, window) : bh.decompressed_size; }
    static uint64_t seqs_of(const BlockHeader &bh, const uint8_t *content) {
        if (bh.type != BT_COMPRESSED) return 0;
        const SectionHeaders sec = parse_section_headers(content, bh.content_size);
        return ((uint64_t)sec.nseq + 3) & ~3ull;
    }
    bool fits(const SdPlan &p, uint64_t in, uint64_t out, uint64_t seqs) const {
        return p.nblocks == 0 || (p.in_bytes + in <= bnd.chunk && p.out_bound + out <= bnd.out && p.nblocks + 1 <= bnd.blocks && p.nseq + seqs <= bnd.seqs);
    }
    void fail_at(SdPlan &p, uint32_t word, uint64_t at, int32_t z) { p.end_word = word; p.end_at = at; p.end_zi = z; p.ends = true; }

    // Plans the next submission into s / p from the source (its buffer starts with the bytes carried over from the last cut).
    void plan(SdSource &src, Submission &s, SdPlan &p) {
        s.clear();
        p = SdPlan();
        size_t pos = 0;
        bool active = false;   // inside a frame: a block header comes next
        TableCursor cur;
        uint64_t window = 0;
        bool checksum = false;
        uint32_t bif = 0, skips = 0;
        const b200z_dict *fdict = nullptr;
        auto start_frame = [&](const SdFrame &f, const b200z_dict *dict, uint64_t w) {
            p.frames.push_back(f);
            p.frames.back().skips_before = skips;
            skips = 0;
            window = w;
            fdict = dict;
        };
        if (cont.on) {
            // the frame continues from its carried state, tables and tail (k_carry writes its state and placement)
            start_frame(cont.frame, cont.dict, cont.window);
            FrameState st;
            memset(&st, 0, sizeof st);
            cur = s.add_resumed_frame(st, cont.window, cont.dict, cont.tables);
            checksum = cont.checksum; bif = cont.next_block;
            p.resumed = true; p.resume_window = cont.window;
            active = true;
            cont.on = false;
        }
        p.start = src.off;
        for (;;) {
            if (!active) {
                if (!src.fill(pos + 1)) { p.ends = true; break; }   // the end of the source, between frames
                size_t want;
                while ((want = frame_header_want(src.buf + pos, src.have - pos)) > src.have - pos && src.fill(pos + want)) {}
                FrameHeader h;
                uint32_t skip = 0;
                size_t hs = 0;
                const uint64_t at = src.off + pos;
                int e = parse_frame_header(src.buf + pos, src.have - pos, h, skip, hs);
                if (e == B200Z_ERR_SKIP_FRAME) {
                    const uint64_t n = 8ull + skip;
                    if (p.frames.empty()) {   // in front of the submission: dropped, never buffered
                        if (!src.drop(n)) { fail_at(p, mk_status(B200Z_ERR_FAILED_TO_SKIP_FRAME, B200Z_STAGE_FRAME_HEADER), at, -1); break; }
                        p.start = src.off;
                        skips++;
                        continue;
                    }
                    if (p.in_bytes + n > bnd.chunk) break;   // cut in front of it: the next submission drops it
                    if (!src.fill(pos + n)) { fail_at(p, mk_status(B200Z_ERR_FAILED_TO_SKIP_FRAME, B200Z_STAGE_FRAME_HEADER), at, -1); break; }
                    pos += n; p.in_bytes += n;
                    skips++;
                    continue;
                }
                const bool zstd = src.have - pos >= 4 && rd32le(src.buf + pos) == ZSTD_MAGIC;
                if (zstd) zi++;
                const int32_t z = zstd ? zi : -1;
                uint64_t w = 0;
                const b200z_dict *dict = nullptr;
                if (!e) e = frame_window(h, max_window, w);
                if (!e) e = frame_dict(h, dicts, ndicts, forced, dict);
                if (e) { fail_at(p, mk_status((uint32_t)e, B200Z_STAGE_FRAME_HEADER), at, z); break; }
                // the frame header goes with the frame's first block: cut in front of it when that block does not fit
                BlockHeader bh;
                bool have_bh = src.fill(pos + hs + 3), bh_ok = have_bh && !parse_block_header(src.buf + pos + hs, bh);
                if (bh_ok && src.fill(pos + hs + 3 + bh.content_size)) {
                    const uint64_t in = hs + 3 + bh.content_size + (bh.last && h.content_checksum() ? 4 : 0);
                    if (!fits(p, in, out_of(bh, w), seqs_of(bh, src.buf + pos + hs + 3))) { zi--; break; }
                }
                max_window_seen = std::max(max_window_seen, w);
                SdFrame f;
                f.at = at; f.zi = z;
                start_frame(f, dict, w);
                cur = s.add_frame(dict, 0, 0, w);
                checksum = h.content_checksum(); bif = 0;
                pos += hs; p.in_bytes += hs;
                active = true;
            }
            // a block of the active frame
            BlockHeader bh;
            if (uint32_t w = read_block(src.fill(pos + 3) ? src.buf + pos : nullptr, bh, [&](uint32_t n) { return src.fill(pos + 3 + n); })) {
                s.frames.back().host_status = w;
                p.ends = true;
                break;
            }
            const uint64_t in = 3 + bh.content_size + (bh.last && checksum ? 4 : 0), out = out_of(bh, window);
            const uint64_t seqs = seqs_of(bh, src.buf + pos + 3);
            if (!fits(p, in, out, seqs)) break;   // cut at this block end: the frame continues in the next submission
            const BlockDesc &d = s.add_block(pos + 3, bh, bif++, src.buf + pos + 3, cur);
            pos += 3 + bh.content_size;
            p.in_bytes += 3 + bh.content_size; p.out_bound += out; p.nblocks++; p.nseq += seqs;
            if (d.host_status) { p.ends = true; break; }   // the frame fails at this block; nothing after it is looked at
            if (bh.last) {
                active = false;
                if (checksum) {
                    if (!src.fill(pos + 4)) { s.frames.back().host_status = mk_status(B200Z_ERR_FAILED_TO_READ_CHECKSUM, B200Z_STAGE_CHECKSUM); p.ends = true; break; }
                    p.frames.back().has_checksum = true;
                    p.frames.back().checksum = rd32le(src.buf + pos);
                    pos += 4; p.in_bytes += 4;
                }
            }
        }
        p.cut = pos;
        p.skips_after = skips;
        if (active && !p.ends) {   // the active frame continues: its state, tables and tail are carried
            p.continues = true;
            p.cur_end = cur;
            cont.on = true;
            cont.frame = p.frames.back();
            cont.frame.skips_before = 0;
            cont.window = window;
            cont.checksum = checksum;
            cont.next_block = bif;
            cont.dict = fdict;
            // the tables its next block starts from: a table built here is copied to the carry slots after the pass
            cont.tables = s.carry_after(cur, carry_huf, carry_fse, predef);
        }
    }
};

struct SliceReader { const uint8_t *p; size_t len; };
long slice_read(void *user, uint8_t *buf, size_t n) {  // impl Read for &[u8]
    SliceReader *s = (SliceReader *)user;
    const size_t k = std::min(n, s->len);
    if (k) memcpy(buf, s->p, k);
    s->p += k; s->len -= k;
    return (long)k;
}

}  // namespace

struct StreamDecodeResources {
    uint64_t chunk = 0;
    // s_d2h brings back each submission's frame states behind its pass; s_out the plaintext (and a failing frame's block sizes) of a
    // submission whose states are back.  On one stream the plaintext of k - 1 would queue behind the wait for k's pass.
    Stream s_h2d, s_d2h, s_out;
    // ev_read[s]: recorded on the kernel stream once the next submission's k_carry has read slot s (its frame states, placement and
    // tail), so that an upload into slot s waits for it, not only for slot s's own pass
    Event ev_h2d[2], ev_k[2], ev_d2h[2], ev_read[2];
    PinnedBuf h_in[2], h_out, h_states[2];
    DevBuf d_in[2], d_out[2];
    DevBuf d_tab_huf, d_tab_fse;   // the continuing frame's tables built in the previous submission (HufSlot, FseSlot)
    DevBuf d_carry;                // StreamCarry[2]: what flows into the submission of slot s
    Submission sub[2];
    uint64_t window = 0;           // d_out[] holds a tail of max(window, 32) bytes
};

static uint64_t sd_chunk_bytes() {
    uint64_t C = 64ull << 20;
    if (const char *ev = getenv("B200Z_PIPELINE_CHUNK_BYTES")) { const uint64_t v = strtoull(ev, nullptr, 10); if (v) C = v; }
    return C;
}

// every buffer sized for the chunk once, so that the memory held depends on the chunk and the largest window only
static int sd_get(b200z_ctx *c, uint64_t C, StreamDecodeResources **out) {
    if (!c->sdec || c->sdec->chunk != C) {
        c->sdec.reset();
        std::unique_ptr<StreamDecodeResources> r(new StreamDecodeResources());
        r->chunk = C;
        if (r->s_h2d.create(c) || r->s_d2h.create(c) || r->s_out.create(c)) return B200Z_ERR_CUDA;
        for (int i = 0; i < 2; i++)
            if (r->ev_h2d[i].create(c) || r->ev_k[i].create(c) || r->ev_d2h[i].create(c) || r->ev_read[i].create(c)) return B200Z_ERR_CUDA;
        const SdBounds b(C);
        const uint64_t nb = b.blocks, nf = nb + 1, room = b.out_room();
        int e = 0;
        for (int i = 0; i < 2 && !e; i++) {
            Submission &s = r->sub[i];
            if ((e = r->h_in[i].ensure(b.buffer(), false)) || (e = r->h_states[i].ensure(nf * sizeof(FrameState), false)) ||
                (e = r->d_in[i].ensure(b.buffer() + 32, false)) || (e = s.d_descs.ensure(nb * sizeof(BlockDesc), false)) ||
                (e = s.d_aux.ensure(nb * sizeof(BlockAux), false)) || (e = s.d_frames.ensure(nf * sizeof(FrameDesc), false)) ||
                (e = s.d_states.ensure(nf * sizeof(FrameState), false)) || (e = s.d_huf.ensure(nb * sizeof(HufSlot), false)) ||
                (e = s.d_fse.ensure(nb * sizeof(FseSlot), false)) || (e = s.d_lit.ensure(room + 32 * nb + 64, false)) ||
                (e = s.d_seq.ensure((b.seqs + 4 * nb + 4) * 12, false)) || (e = s.d_order.ensure(4 * nb, false)) ||
                (e = s.d_sched.ensure(2 * (16 + 4 * nf) + 4 * nf + 32, false)))
                break;
        }
        if (!e && !(e = r->h_out.ensure(room + 64, false)) && !(e = r->d_tab_huf.ensure(sizeof(HufSlot), false)) && !(e = r->d_tab_fse.ensure(sizeof(FseSlot), false)))
            e = r->d_carry.ensure(2 * sizeof(StreamCarry), false);
        if (e) { c->err = "decode_all_stream: out of memory for chunks of " + std::to_string(C) + " bytes"; return e; }
        c->sdec = std::move(r);
    }
    *out = c->sdec.get();
    return 0;
}

// The stream entries' I/O.  write_all: false on a write <= 0 or one of more than was asked for; *delivered (when given) counts
// the bytes written.  read_chunk: reads up to `cap` bytes, stopping at the first read that returns 0 (*eof; the reference's
// FrameCompressor stops there too); false on a read error (< 0, or more than was asked for).  The frame decoder's read_upto /
// read_exact take a negative read as the end of the source instead, as ruzstd does.
static bool write_all(b200z_write_fn wr, void *wu, const uint8_t *p, size_t n, uint64_t *delivered) {
    while (n) {
        const long w = wr(wu, p, n);
        if (w <= 0 || (size_t)w > n) return false;
        p += w; n -= (size_t)w;
        if (delivered) *delivered += (uint64_t)w;
    }
    return true;
}
static bool read_chunk(b200z_read_fn rd, void *ru, uint8_t *buf, size_t cap, size_t *n, bool *eof) {
    size_t got = 0;
    *eof = false;
    while (got < cap) {
        const long r = rd(ru, buf + got, cap - got);
        if (r < 0 || (size_t)r > cap - got) return false;
        if (r == 0) { *eof = true; break; }
        got += (size_t)r;
    }
    *n = got;
    return true;
}

extern "C" int b200z_decode_all_stream(b200z_ctx *c, b200z_read_fn rd, void *ru, b200z_write_fn wr, void *wu, const b200z_dict *const *dicts, size_t ndicts,
                                       const b200z_dict *forced, uint64_t max_window, b200z_stream_result *result) {
    if (!c || !rd || !wr || !result || (!dicts && ndicts)) return B200Z_ERR_INVALID_ARGUMENT;
    if (int e = c->use()) return e;
    const uint64_t C = sd_chunk_bytes();
    StreamDecodeResources *R = nullptr;
    if (int e = sd_get(c, C, &R)) return e;
    b200z_stream_result res;
    memset(&res, 0, sizeof res);
    res.first_mismatch_frame = -1;
    res.all.error_frame = -1;
    SdPlanner pl(C, dicts, ndicts, forced, max_window);
    pl.carry_huf = R->d_tab_huf.as<HufSlot>(); pl.carry_fse = R->d_tab_fse.as<FseSlot>(); pl.predef = c->d_predef.as<FseSlot>();
    SdSource src;
    src.rd = rd; src.user = ru; src.cap = (size_t)SdBounds(C).buffer();
    src.buf = R->h_in[0].as<uint8_t>();
    SdPlan plan[2];
    const bool hash = (c->flags & B200Z_FLAG_CHECKSUM) != 0;
    const PipelineStreams ps{c->stream, c->side, c->ev_fork, c->ev_join};
    StreamCarry *d_carry = R->d_carry.as<StreamCarry>();
    const uint64_t room = SdBounds(C).out_room();
    uint64_t cont_total = 0;     // plaintext of the continuing frame before the submission being retired
    bool stopped = false;
    auto out_cap_of = [&](const SdPlan &p) { return (p.resumed ? std::max<uint64_t>(p.resume_window, 32) : 0) + p.out_bound; };
    auto enqueue = [&](int s) -> int {
        const SdPlan &p = plan[s];
        Submission &sub = R->sub[s];
        if (p.frames.empty()) return 0;
        // the tail room grows with the largest window seen; only this slot's buffer: the other holds the previous submission's
        // plaintext, not yet written, and the tail k_carry reads
        R->window = std::max(R->window, pl.max_window_seen);
        const uint64_t out_need = std::max<uint64_t>(R->window, 32) + room + 64;
        if (out_need > R->d_out[s].cap) {
            CU(c, cudaEventSynchronize(R->ev_read[s]));   // the previous submission's k_carry may still read the tail there
            if (int e = R->d_out[s].ensure(out_need, false)) return e;
        }
        CU(c, cudaStreamWaitEvent(R->s_h2d, R->ev_k[s], 0));      // the submission two back is done with slot s
        CU(c, cudaStreamWaitEvent(R->s_h2d, R->ev_read[s], 0));   // and the previous one's k_carry has read it
        if (p.cut) CU(c, cudaMemcpyAsync(R->d_in[s].p, R->h_in[s].p, p.cut, cudaMemcpyHostToDevice, R->s_h2d));
        if (int e = sub.upload(c, R->s_h2d)) return e;
        CU(c, cudaEventRecord(R->ev_h2d[s], R->s_h2d));
        CU(c, cudaStreamWaitEvent(c->stream, R->ev_h2d[s], 0));
        PipelineArgs a = sub.args(R->d_in[s].as<uint8_t>(), R->d_out[s].as<uint8_t>(), out_cap_of(p));
        if (p.resumed) {
            const Submission &ps_ = R->sub[s ^ 1];
            PipelineArgs prev = ps_.args(nullptr, R->d_out[s ^ 1].as<uint8_t>(), 0);
            if (int le = launch_carry(prev, (uint32_t)ps_.frames.size() - 1, a, d_carry + (s ^ 1), d_carry + s, plan[s ^ 1].resumed && plan[s ^ 1].frames.size() == 1,
                                      std::max<uint64_t>(p.resume_window, 32), c->stream, &c->launches))
                return c->set_cuda_err((cudaError_t)le, "k_carry");
        }
        CU(c, cudaEventRecord(R->ev_read[s ^ 1], c->stream));
        if (int e = enqueue_decode_all_stages(c, a, ps, p.resumed, &c->launches)) return e;
        if (hash)
            if (int le = launch_checksum_stream(a, d_carry + s, d_carry + (s ^ 1), p.resumed, p.continues, c->stream, &c->launches))
                return c->set_cuda_err((cudaError_t)le, "k_xxh64_stream");
        // the continuing frame's tables built here, for the next submission (the host knows which: no wait)
        if (p.continues)
            if (int e = sub.copy_carry(c, p.cur_end, R->d_tab_huf.as<HufSlot>(), R->d_tab_fse.as<FseSlot>(), c->stream)) return e;
        CU(c, cudaEventRecord(R->ev_k[s], c->stream));
        CU(c, cudaStreamWaitEvent(R->s_d2h, R->ev_k[s], 0));
        if (int e = sub.download_states(c, R->h_states[s].as<FrameState>(), R->s_d2h)) return e;
        CU(c, cudaEventRecord(R->ev_d2h[s], R->s_d2h));
        res.submissions++;
        return 0;
    };
    // the outcome of the submission in slot s, in stream order: its plaintext up to the first failing block goes to the drain
    auto retire = [&](int s) -> int {
        const SdPlan &p = plan[s];
        const Submission &sub = R->sub[s];
        b200z_all_result all = res.all;
        uint64_t ck = res.checksum_frames, mism = res.checksum_mismatches;
        int64_t first_mism = res.first_mismatch_frame;
        uint64_t T0 = 0, len = 0, total = cont_total;
        bool failed = false;
        if (!p.frames.empty()) {
            CU(c, cudaEventSynchronize(R->ev_d2h[s]));
            const FrameState *st = R->h_states[s].as<FrameState>();
            if (p.resumed) T0 = std::min<uint64_t>(cont_total, std::max<uint64_t>(p.resume_window, 32));
            for (size_t f = 0; f < p.frames.size(); f++) {
                const SdFrame &F = p.frames[f];
                all.skippable_frames += F.skips_before;
                const uint64_t before = f == 0 && p.resumed ? cont_total : 0, tail = f == 0 ? T0 : 0;
                if (st[f].status) {
                    // the frame's output before its first failing block (blocks_done counts this submission's blocks)
                    const FrameDesc &fd = sub.frames[f];
                    const uint32_t n = std::min(st[f].blocks_done, fd.nblocks);
                    if (n) {
                        std::vector<BlockAux> aux(n);
                        if (int e = sub.download_aux(c, aux.data(), fd.first_block, n, R->s_out)) return e;
                        CU(c, cudaStreamSynchronize(R->s_out));
                        for (uint32_t k = 0; k < n; k++) len += aux[k].out_size;
                    }
                    uint32_t word = st[f].status;
                    // a block that decodes to more than its bound (RFC 8878 forbids it) ran out of the submission's output room
                    if (status_code(word) == B200Z_ERR_TARGET_TOO_SMALL) word = mk_status(B200Z_ERR_BLOCK_OUTPUT_LIMIT, B200Z_STAGE_EXECUTE);
                    all.status = (int32_t)status_code(word); all.stage = (int32_t)status_stage(word);
                    all.error_offset = F.at; all.error_frame = F.zi;
                    failed = true;
                    break;
                }
                const uint64_t fresh = st[f].produced - tail;
                len += fresh;
                if (f + 1 == p.frames.size() && p.continues) { total = before + fresh; continue; }
                all.frames++; all.written += before + fresh;
                if (hash && F.has_checksum) {
                    ck++;
                    if ((uint32_t)st[f].xxh64 != F.checksum) { mism++; if (first_mism < 0) first_mism = F.zi; }
                }
            }
        }
        if (!failed) {
            all.skippable_frames += p.skips_after;
            if (p.end_word) {
                all.status = (int32_t)status_code(p.end_word); all.stage = (int32_t)status_stage(p.end_word);
                all.error_offset = p.end_at; all.error_frame = p.end_zi;
                failed = true;
            }
        }
        if (len) {
            // the states are back, so this submission's pass is over; the next one keeps running meanwhile
            CU(c, cudaMemcpyAsync(R->h_out.p, R->d_out[s].as<uint8_t>() + T0, len, cudaMemcpyDeviceToHost, R->s_out));
            CU(c, cudaStreamSynchronize(R->s_out));
            if (!write_all(wr, wu, R->h_out.as<uint8_t>(), len, &res.delivered)) {
                res.all.status = B200Z_ERR_FAILED_TO_DRAIN_DECODEBUFFER; res.all.stage = B200Z_STAGE_DRAIN;
                res.all.error_offset = p.frames.front().at; res.all.error_frame = p.frames.front().zi;
                stopped = true;
                return 0;
            }
        }
        res.all = all;
        res.checksum_frames = ck; res.checksum_mismatches = mism; res.first_mismatch_frame = first_mism;
        cont_total = total;
        if (failed) stopped = true;
        return 0;
    };
    int e = 0;
    pl.plan(src, R->sub[0], plan[0]);
    for (int k = 0; !e; k++) {
        const int s = k & 1;
        if ((e = enqueue(s))) break;
        if (k && (e = retire(s ^ 1))) break;
        if (stopped) break;
        if (plan[s].ends) { e = retire(s); break; }
        // the next submission: its buffer (slot s ^ 1) is free once the upload of the submission two back is done
        if (k && cudaEventSynchronize(R->ev_h2d[s ^ 1]) != cudaSuccess) { e = c->set_cuda_err(cudaGetLastError(), "upload"); break; }
        src.advance(plan[s].cut, R->h_in[s ^ 1].as<uint8_t>());
        pl.plan(src, R->sub[s ^ 1], plan[s ^ 1]);
    }
    // leave nothing in flight: the buffers are reused by the next call
    cudaStreamSynchronize(R->s_h2d);
    cudaStreamSynchronize(c->stream);
    cudaStreamSynchronize(R->s_d2h);
    cudaStreamSynchronize(R->s_out);
    // now both slots take the largest window's tail, so that what the context holds does not depend on how many submissions ran
    for (DevBuf &d : R->d_out)
        if (!e) e = d.ensure(std::max<uint64_t>(R->window, 32) + room + 64, false);
    if (!res.all.status) res.all.error_offset = src.off + src.have;
    *result = res;
    return e;
}

// b200z_debug_stream_cut: the planner alone over a byte string, with host buffers (no context, no device)
extern "C" int b200z_debug_stream_cut(const uint8_t *input, size_t input_len, uint64_t chunk, b200z_stream_cut *cuts, size_t cap, size_t *n,
                                      b200z_stream_cut_end *end) {
    if (!n || !end || (!input && input_len) || (!cuts && cap) || !chunk) return B200Z_ERR_INVALID_ARGUMENT;
    SliceReader sr{input, input_len};
    SdPlanner pl(chunk, nullptr, 0, nullptr, 0);
    static const FseSlot *const fake = reinterpret_cast<const FseSlot *>(16);   // table pointers are never dereferenced here
    pl.carry_huf = reinterpret_cast<const HufSlot *>(16); pl.carry_fse = fake; pl.predef = fake;
    SdSource src;
    src.rd = slice_read; src.user = &sr; src.cap = (size_t)pl.bnd.buffer();
    std::vector<uint8_t> buf[2] = {std::vector<uint8_t>(src.cap), std::vector<uint8_t>(src.cap)};
    src.buf = buf[0].data();
    Submission sub;
    SdPlan p;
    size_t k = 0;
    memset(end, 0, sizeof *end);
    end->error_frame = -1;
    for (;; k++) {
        pl.plan(src, sub, p);
        if (!p.frames.empty()) {
            if (k < cap) {
                b200z_stream_cut &o = cuts[k];
                o.start = p.start; o.end = p.start + p.cut; o.in_bytes = p.in_bytes; o.out_bound = p.out_bound; o.nblocks = p.nblocks;
                o.nseq = p.nseq; o.nframes = (uint32_t)p.frames.size(); o.flags = (p.resumed ? 1u : 0u) | (p.continues ? 2u : 0u);
            }
        } else k--;
        end->skippable_frames += p.skips_after;
        for (const SdFrame &f : p.frames) end->skippable_frames += f.skips_before;
        if (p.ends) {
            end->status = (int32_t)status_code(p.end_word); end->stage = (int32_t)status_stage(p.end_word);
            if (!p.end_word && !sub.frames.empty()) {   // a frame that fails on a header the planner read (block header, truncation)
                const uint32_t hs = sub.frames.back().host_status;
                if (hs) { end->status = (int32_t)status_code(hs); end->stage = (int32_t)status_stage(hs); }
                else for (const BlockDesc &d : sub.descs) if (d.host_status) { end->status = (int32_t)status_code(host_status_word(d.host_status)); end->stage = (int32_t)status_stage(host_status_word(d.host_status)); }
                if (end->status) { end->error_offset = p.frames.back().at; end->error_frame = p.frames.back().zi; }
            }
            if (p.end_word) { end->error_offset = p.end_at; end->error_frame = p.end_zi; }
            if (!end->status) end->error_offset = src.off + p.cut;
            k++;
            break;
        }
        src.advance(p.cut, buf[(k + 1) & 1].data());
    }
    end->peak_buffered = src.peak;
    *n = k;
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// tier 1b: block-level batch entry -- replaces the call site of the hot path, BlockDecoder::decompress_block
// (block_decoder.rs:97-197), for a host that keeps the reference's own header parsing.
// ---------------------------------------------------------------------------------------------------------------
extern "C" int b200z_decode_blocks_batch(b200z_ctx *c, const b200z_block_desc *blocks, size_t nblocks, const b200z_block_frame *frames, size_t nframes,
                                         const uint8_t *compressed, size_t compressed_len, int compressed_mem, uint8_t *output, size_t output_cap,
                                         int output_mem, b200z_block_status *status, uint64_t *frame_out_size) {
    if (!c || (!blocks && nblocks) || (!frames && nframes) || (!compressed && compressed_len) || (!output && output_cap)) return B200Z_ERR_INVALID_ARGUMENT;
    if (int e = c->use()) return e;
    std::vector<uint8_t> host_copy;
    const uint8_t *hin = compressed;
    if (compressed_mem == B200Z_MEM_DEVICE) {   // the section headers are walked on the host
        host_copy.resize(compressed_len);
        if (compressed_len) CU(c, cudaMemcpy(host_copy.data(), compressed, compressed_len, cudaMemcpyDeviceToHost));
        hin = host_copy.data();
    }
    Submission s;
    std::vector<int64_t> sub_of(nblocks, -1);      // caller's block index -> descriptor index in the submission
    for (size_t f = 0; f < nframes; f++) {
        const b200z_block_frame &bf = frames[f];
        if ((uint64_t)bf.first_block + bf.num_blocks > nblocks) return B200Z_ERR_INVALID_ARGUMENT;
        TableCursor cur = s.add_frame(bf.dict, bf.out_off, bf.out_cap, bf.window_size);
        for (uint32_t k = 0; k < bf.num_blocks; k++) {
            const b200z_block_desc &bd = blocks[bf.first_block + k];
            if (bd.block_type > BT_COMPRESSED || bd.src_off > compressed_len || bd.content_size > compressed_len - bd.src_off) return B200Z_ERR_INVALID_ARGUMENT;
            if (bd.block_type != BT_COMPRESSED && (bd.block_type == BT_RAW ? bd.content_size != bd.decompressed_size : bd.content_size != 1))
                return B200Z_ERR_INVALID_ARGUMENT;
            BlockHeader bh;
            bh.last = bd.last_block; bh.type = bd.block_type; bh.decompressed_size = bd.decompressed_size; bh.content_size = bd.content_size;
            sub_of[bf.first_block + k] = (int64_t)s.descs.size();
            SectionHeaders sec = {};
            if (bh.type == BT_COMPRESSED) {
                // the descriptor says what the caller's parsers found: it must be what the content says, as far as its headers parse
                sec = parse_section_headers(hin + bd.src_off, bh.content_size);
                if (sec.lit_off != 0 && (sec.lit_type != bd.literals_type || sec.regen_size != bd.regenerated_size)) return B200Z_ERR_INVALID_ARGUMENT;
                if (!sec.status && (sec.nseq != bd.num_sequences || (sec.nseq && sec.modes != bd.modes))) return B200Z_ERR_INVALID_ARGUMENT;
            }
            const BlockDesc &d = s.add_block(bd.src_off, bh, k, sec, cur);
            if (d.host_status) break;   // decompress_block would have returned here: later blocks of the frame are never reached
        }
    }
    DevBuf d_in_own, d_out_own;
    const uint8_t *d_in = compressed;
    if (compressed_mem != B200Z_MEM_DEVICE) {
        if (int e = d_in_own.ensure(compressed_len + 16, false)) return e;
        if (compressed_len) CU(c, cudaMemcpyAsync(d_in_own.p, compressed, compressed_len, cudaMemcpyHostToDevice, c->stream));
        d_in = d_in_own.as<uint8_t>();
    }
    uint8_t *d_out = output;
    if (output_mem != B200Z_MEM_DEVICE) {
        if (int e = d_out_own.ensure(output_cap + 16, false)) return e;
        d_out = d_out_own.as<uint8_t>();
    }
    if (int e = s.upload(c)) return e;
    if (int e = enqueue_pass(c, s.args(d_in, d_out, output_cap), PipelineStreams{c->stream, c->side, c->ev_fork, c->ev_join}, nullptr, &c->launches))
        return e;
    std::vector<FrameState> st(s.states.size());
    std::vector<BlockAux> aux(s.descs.size());
    if (int e = s.download_states(c, st.data(), c->stream)) return e;
    if (int e = s.download_aux(c, aux.data(), 0, aux.size(), c->stream)) return e;
    CU(c, cudaStreamSynchronize(c->stream));
    // host output: each frame's produced bytes come back (copy_back_ranges), so the caller's bytes between two frames' slots stay as they were
    std::vector<std::pair<uint64_t, uint64_t>> copy_back;
    for (size_t f = 0; f < nframes; f++) {
        const b200z_block_frame &bf = frames[f];
        const FrameState &fs = st[f];
        if (frame_out_size) frame_out_size[f] = fs.produced;
        const uint64_t end = std::min<uint64_t>(bf.out_off + std::min<uint64_t>(fs.produced, bf.out_cap), output_cap);
        if (end > bf.out_off) copy_back.emplace_back(bf.out_off, end);
        if (!status) continue;
        for (uint32_t k = 0; k < bf.num_blocks; k++) {
            b200z_block_status &o = status[bf.first_block + k];
            memset(&o, 0, sizeof o);
            const int64_t si = sub_of[bf.first_block + k];
            const bool failed_here = fs.status && k == fs.error_block;
            if (si < 0 || (fs.status && k > fs.error_block)) { o.status = B200Z_BLOCK_NOT_REACHED; continue; }
            if (failed_here) { o.status = (int32_t)status_code(fs.status); o.stage = (int32_t)status_stage(fs.status); continue; }
            const BlockDesc &d = s.descs[(size_t)si];
            o.out_size = d.btype == BT_COMPRESSED ? aux[(size_t)si].out_size : d.raw_size;
        }
    }
    if (output_mem != B200Z_MEM_DEVICE)
        if (int e = copy_back_ranges(c, c->stream, output, d_out, copy_back, true)) return e;
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// tier 2: FrameDecoder mirror (decoding/frame_decoder.rs)
// ---------------------------------------------------------------------------------------------------------------
struct b200z_frame_decoder {
    b200z_ctx *ctx = nullptr;
    uint64_t max_window = B200Z_DEFAULT_MAX_WINDOW_SIZE;
    std::map<uint32_t, std::shared_ptr<b200z_dict>> dicts;   // FrameDecoder.dicts (BTreeMap<u32, Dictionary>)
    // FrameDecoderState (frame_decoder.rs:86-94)
    bool has_state = false;
    FrameHeader hdr;
    uint64_t window = 0;
    bool frame_finished = false;
    size_t block_counter = 0;
    uint64_t bytes_read_counter = 0;
    bool has_check_sum = false;
    uint32_t check_sum = 0;
    // the dictionary the frame started with, kept until the next reset even when add_dict replaces it (the reference copies it
    // into the frame's scratch, DecoderScratch::init_from_dict)
    std::shared_ptr<const b200z_dict> using_dict;
    uint32_t skip_len = 0;
    int last_stage = 0;
    std::string err;
    // decode buffer on the device: frame bytes [base, produced) live at d_out[0 .. produced-base); the host has
    // drained everything below `drained` (DecodeBuffer::len() == produced - drained, decode_buffer.rs:58)
    DevBuf d_out;
    uint64_t base = 0, produced = 0, drained = 0;
    FrameState state;                                  // host mirror of the device-side frame state
    XXH64State hash;                                   // decode_buffer.rs:16, fed on drain
    // "current tables" (DecoderScratch.huf/.fse): which kinds exist + persistent device copies
    DevBuf d_carry_huf, d_carry_fse;                   // HufSlot, FseSlot
    CarrySet carry;                                    // what the next submission starts from
    Submission sub;
    DevBuf d_input;
    std::vector<uint8_t> staging;                      // bytes of the blocks of the current submission
};

static int fd_fail(b200z_frame_decoder *d, int code, int stage) {
    d->last_stage = stage;
    char buf[160];
    snprintf(buf, sizeof buf, "%s (stage %d)", b200z_error_name(code), stage);
    d->err = buf;
    return code;
}

extern "C" int b200z_frame_decoder_new(b200z_ctx *c, b200z_frame_decoder **out) {
    if (!c || !out) return B200Z_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    if (int e = c->use()) return e;
    std::unique_ptr<b200z_frame_decoder> d(new b200z_frame_decoder());
    d->ctx = c;
    memset(&d->state, 0, sizeof d->state);
    d->hash.reset();
    CU(c, d->d_carry_huf.alloc(sizeof(HufSlot)));
    CU(c, d->d_carry_fse.alloc(sizeof(FseSlot)));
    *out = d.release();
    return 0;
}
extern "C" void b200z_frame_decoder_free(b200z_frame_decoder *d) {
    if (!d) return;
    cudaSetDevice(d->ctx->device);
    delete d;
}
extern "C" void b200z_frame_decoder_set_max_window_size(b200z_frame_decoder *d, uint64_t n) {
    d->max_window = std::min<uint64_t>(n, MAX_WINDOW_SIZE);
}
extern "C" uint64_t b200z_frame_decoder_max_window_size(const b200z_frame_decoder *d) { return d->max_window; }
extern "C" uint32_t b200z_frame_decoder_skip_frame_length(const b200z_frame_decoder *d) { return d->skip_len; }
extern "C" int b200z_frame_decoder_last_stage(const b200z_frame_decoder *d) { return d->last_stage; }
extern "C" const char *b200z_frame_decoder_last_error_message(const b200z_frame_decoder *d) { return d->err.c_str(); }

static size_t read_upto(b200z_read_fn rd, void *user, uint8_t *buf, size_t n) {   // stops at the end of the source; returns the bytes read
    size_t got = 0;
    while (got < n) { long r = rd(user, buf + got, n - got); if (r <= 0) break; got += (size_t)r; }
    return got;
}
static bool read_exact(b200z_read_fn rd, void *user, uint8_t *buf, size_t n) { return read_upto(rd, user, buf, n) == n; }

static void fd_apply_dict(b200z_frame_decoder *d, std::shared_ptr<const b200z_dict> dict) {  // DecoderScratch::init_from_dict, scratch.rs:70-78
    d->carry = carry_of_dict(dict.get());
    d->state.hist[0] = dict->hist[0]; d->state.hist[1] = dict->hist[1]; d->state.hist[2] = dict->hist[2];
    d->using_dict = std::move(dict);
}

// reset (frame_decoder.rs:200-221): read the header through the callback as read_frame_header does -- the magic number, then the
// descriptor byte (or a skippable frame's length), then the rest of the header -- and never a byte past it
extern "C" int b200z_frame_decoder_reset(b200z_frame_decoder *d, b200z_read_fn rd, void *user) {
    if (!d || !rd) return B200Z_ERR_INVALID_ARGUMENT;
    uint8_t buf[32];
    size_t have = 0;
    for (size_t want; (want = frame_header_want(buf, have)) > have;) {
        have += read_upto(rd, user, buf + have, want - have);
        if (have < want) break;   // parse_frame_header names the field that could not be read
    }
    FrameHeader h; uint32_t skip = 0; size_t consumed = 0;
    int e = parse_frame_header(buf, have, h, skip, consumed);
    if (e == B200Z_ERR_SKIP_FRAME) d->skip_len = skip;
    if (e) return fd_fail(d, e, B200Z_STAGE_FRAME_HEADER);
    uint64_t window = 0;
    if ((e = frame_window(h, d->max_window, window))) return fd_fail(d, e, B200Z_STAGE_FRAME_HEADER);
    // FrameDecoderState::new / reset (:103-134)
    d->hdr = h; d->window = window; d->frame_finished = false; d->block_counter = 0;
    d->bytes_read_counter = h.header_size; d->has_check_sum = false; d->using_dict = nullptr;
    d->base = d->produced = d->drained = 0;
    memset(&d->state, 0, sizeof d->state);
    d->state.hist[0] = 1; d->state.hist[1] = 4; d->state.hist[2] = 8;
    d->hash.reset();
    d->carry = CarrySet();
    d->has_state = true;
    if (h.has_dict_id) {
        auto it = d->dicts.find(h.dict_id);
        if (it == d->dicts.end()) return fd_fail(d, B200Z_ERR_DICT_NOT_PROVIDED, B200Z_STAGE_FRAME_HEADER);
        fd_apply_dict(d, it->second);
    }
    d->last_stage = 0;
    return 0;
}
extern "C" int b200z_frame_decoder_init(b200z_frame_decoder *d, b200z_read_fn rd, void *user) { return b200z_frame_decoder_reset(d, rd, user); }

// add_dict / add_raw_content_dict: `x` (created with error e) replaces a dictionary of the same ID for the frames that start
// after this call; the frame in progress keeps the one it started with
static int fd_add_dict(b200z_frame_decoder *d, int e, b200z_dict *x) {
    if (e) return fd_fail(d, e, B200Z_STAGE_DICTIONARY);
    d->dicts[x->id] = std::shared_ptr<b200z_dict>(x, b200z_dict_destroy);
    return 0;
}
extern "C" int b200z_frame_decoder_add_dict(b200z_frame_decoder *d, const uint8_t *raw, size_t len) {
    if (!d) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_dict *x = nullptr;
    const int e = b200z_dict_create(d->ctx, raw, len, &x);
    return fd_add_dict(d, e, x);
}
extern "C" int b200z_frame_decoder_add_raw_content_dict(b200z_frame_decoder *d, uint32_t id, const uint8_t *content, size_t len) {
    if (!d) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_dict *x = nullptr;
    const int e = b200z_dict_create_raw_content(d->ctx, id, content, len, &x);
    return fd_add_dict(d, e, x);
}
extern "C" int b200z_frame_decoder_force_dict(b200z_frame_decoder *d, uint32_t dict_id) {  // :229-243
    if (!d) return B200Z_ERR_INVALID_ARGUMENT;
    if (!d->has_state) return fd_fail(d, B200Z_ERR_NOT_YET_INITIALIZED, 0);
    auto it = d->dicts.find(dict_id);
    if (it == d->dicts.end()) return fd_fail(d, B200Z_ERR_DICT_NOT_PROVIDED, 0);
    fd_apply_dict(d, it->second);
    return 0;
}

static size_t fd_buffer_len(const b200z_frame_decoder *d) { return (size_t)(d->produced - d->drained); }
static bool fd_finished(const b200z_frame_decoder *d) {  // is_finished :284-294
    if (!d->has_state) return true;
    if (d->hdr.content_checksum()) return d->frame_finished && d->has_check_sum;
    return d->frame_finished;
}
static size_t fd_can_drain_to_window(const b200z_frame_decoder *d) {  // decode_buffer.rs:182-188
    size_t n = fd_buffer_len(d);
    return n > d->window ? (size_t)(n - d->window) : 0;
}

// make room for `extra` more bytes behind `produced`, dropping drained bytes when that frees enough
static int fd_reserve_out(b200z_frame_decoder *d, uint64_t extra) {
    b200z_ctx *c = d->ctx;
    uint64_t live = d->produced - d->drained;
    uint64_t need = (d->produced - d->base) + extra + 64;
    if (need <= d->d_out.cap) return 0;
    uint64_t want = std::max<uint64_t>(live + extra + 64, (uint64_t)d->d_out.cap + d->d_out.cap / 2);
    want = std::max<uint64_t>(want, 1u << 20);
    DevBuf grown;
    if (int e = grown.ensure(want, false)) return e;
    if (live) {
        cudaError_t ce = cudaMemcpyAsync(grown.p, d->d_out.as<uint8_t>() + (d->drained - d->base), live, cudaMemcpyDeviceToDevice, c->stream);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(c->stream);
        if (ce != cudaSuccess) return c->set_cuda_err(ce, "grow output");
    }
    d->d_out = std::move(grown);
    d->base = d->drained;
    return 0;
}

// Decode the blocks gathered in d->sub (its one frame, opened by fd_decode_blocks_impl) / d->staging on the GPU; updates
// produced/state/carry tables.  Returns 0 or the error of the first failing block; *done_blocks counts the blocks before it.
static int fd_submit(b200z_frame_decoder *d, const TableCursor &cur, uint32_t *done_blocks) {
    b200z_ctx *c = d->ctx;
    Submission &s = d->sub;
    if (int e = c->use()) return e;
    int e;
    if ((e = d->d_input.ensure(d->staging.size() + 16))) return e;
    CU(c, cudaMemcpyAsync(d->d_input.p, d->staging.data(), d->staging.size(), cudaMemcpyHostToDevice, c->stream));
    if ((e = s.upload(c))) return e;
    // stage A: tables + literals + sequences; sizes come back so the output can grow before execution
    PipelineArgs a = s.args(d->d_input.as<uint8_t>(), nullptr, 0);
    PipelineArgs a_dec = a; a_dec.nframes = 0;
    int le = launch_pipeline(a_dec, c->stream, &c->launches);
    if (le) return c->set_cuda_err((cudaError_t)le, "launch decode");
    std::vector<BlockAux> aux(s.descs.size());
    if ((e = s.download_aux(c, aux.data(), 0, aux.size(), c->stream))) return e;
    CU(c, cudaStreamSynchronize(c->stream));
    uint64_t extra = 0;
    for (size_t i = 0; i < aux.size(); i++) {   // blocks after the first failing one are never executed (nor looked at by the reference)
        if (block_first_error(s.descs[i].host_status, aux[i].status, aux[i].seq_status)) break;
        extra += aux[i].out_size;
    }
    if ((e = fd_reserve_out(d, extra))) return e;
    // stage B: execution into the persistent window buffer (frame byte 0 sits at d_out - base)
    s.frames[0].out_cap = d->base + d->d_out.cap;
    CU(c, cudaMemcpyAsync(s.d_frames.p, s.frames.data(), sizeof(FrameDesc), cudaMemcpyHostToDevice, c->stream));
    PipelineArgs a_ex = a; a_ex.nblocks = 0;
    a_ex.output = d->d_out.as<uint8_t>() - d->base; a_ex.output_cap = d->base + d->d_out.cap;
    le = launch_pipeline(a_ex, c->stream, &c->launches);
    if (le) return c->set_cuda_err((cudaError_t)le, "launch exec");
    // carry the current tables over to the next submission (device-to-device, tables never visit the host)
    HufSlot *huf_to = d->d_carry_huf.as<HufSlot>();
    FseSlot *fse_to = d->d_carry_fse.as<FseSlot>();
    if ((e = s.copy_carry(c, cur, huf_to, fse_to, c->stream))) return e;
    const CarrySet next = s.carry_after(cur, huf_to, fse_to, c->d_predef.as<FseSlot>());
    FrameState st;
    if ((e = s.download_states(c, &st, c->stream))) return e;
    CU(c, cudaStreamSynchronize(c->stream));
    d->carry = next;
    d->state = st;
    d->produced = st.produced;
    *done_blocks = st.blocks_done;
    if (st.status) { d->last_stage = (int)status_stage(st.status); return (int)status_code(st.status); }
    return 0;
}

// decode_blocks (frame_decoder.rs:309-377).  `slice` != null selects decode_from_to's trailer rule (:505-516):
// the checksum is taken only if its 4 bytes are present, otherwise left for the next call.
static int fd_decode_blocks_impl(b200z_frame_decoder *d, b200z_read_fn rd, void *user, int strategy, size_t n, int *finished, SliceReader *slice) {
    if (!d || !rd) return B200Z_ERR_INVALID_ARGUMENT;
    if (!d->has_state) return fd_fail(d, B200Z_ERR_NOT_YET_INITIALIZED, 0);
    if (d->state.status) return fd_fail(d, (int)status_code(d->state.status), (int)status_stage(d->state.status));
    const size_t buffer_size_before = fd_buffer_len(d);
    const size_t block_counter_before = d->block_counter;
    bool stop = false;
    while (!stop) {
        // gather blocks for one GPU submission.  All / UptoBlocks know where to stop from the headers alone;
        // UptoBytes must see each block's decoded size, so it submits block by block.
        Submission &s = d->sub;
        s.clear();
        d->staging.clear();
        // the frame, resumed from the state and tables the last submission left (placement: fd_submit, once the output is sized)
        d->state.produced = d->produced; d->state.drained = d->drained; d->state.blocks_done = 0; d->state.status = 0;
        TableCursor cur = s.add_resumed_frame(d->state, d->window, d->using_dict.get(), d->carry);
        std::vector<uint64_t> bytes_after;  // bytes_read_counter after each gathered block
        uint32_t pending = 0;               // status word of the block that could not be read
        bool saw_last = false;
        uint64_t brc = d->bytes_read_counter;
        size_t gathered_target = strategy == B200Z_STRATEGY_UPTO_BYTES ? 1 : (strategy == B200Z_STRATEGY_UPTO_BLOCKS ? std::max<size_t>(n, 1) - (d->block_counter - block_counter_before) : SIZE_MAX);
        if (strategy == B200Z_STRATEGY_ALL) gathered_target = 4096;  // bound the staging buffer; loop continues
        while (s.descs.size() < gathered_target) {
            uint8_t hb[3];
            BlockHeader bh;
            const size_t off = d->staging.size();
            auto read_body = [&](uint32_t len) {
                d->staging.resize(off + len);
                if (read_exact(rd, user, d->staging.data() + off, len)) return true;
                d->staging.resize(off);
                return false;
            };
            if ((pending = read_block(read_exact(rd, user, hb, 3) ? hb : nullptr, bh, read_body))) break;
            const BlockDesc &bd = s.add_block(off, bh, (uint32_t)(d->block_counter + s.descs.size()), d->staging.data() + off, cur);
            brc += 3 + bh.content_size;
            bytes_after.push_back(brc);
            if (bd.host_status) break;
            if (bh.last) { saw_last = true; break; }
        }
        uint32_t done = 0;
        int e = 0;
        if (!s.descs.empty()) e = fd_submit(d, cur, &done);
        // counters exactly as the reference leaves them (:325-343)
        if (done > 0) d->bytes_read_counter = bytes_after[done - 1];
        d->block_counter += done;
        if (e) {
            if (d->last_stage >= B200Z_STAGE_BLOCK_BODY && d->last_stage <= B200Z_STAGE_EXECUTE) d->bytes_read_counter += 3;
            return fd_fail(d, e, d->last_stage);
        }
        if (pending) {
            if (status_stage(pending) == B200Z_STAGE_BLOCK_BODY) d->bytes_read_counter += 3;
            d->state.status = pending;
            return fd_fail(d, (int)status_code(pending), (int)status_stage(pending));
        }
        if (saw_last) {
            d->frame_finished = true;
            if (d->hdr.content_checksum() && !(slice && slice->len < 4)) {
                uint8_t cs[4];
                if (!read_exact(rd, user, cs, 4)) return fd_fail(d, B200Z_ERR_FAILED_TO_READ_CHECKSUM, B200Z_STAGE_CHECKSUM);
                d->bytes_read_counter += 4;
                d->check_sum = rd32le(cs);
                d->has_check_sum = true;
            }
            break;
        }
        if (strategy == B200Z_STRATEGY_UPTO_BLOCKS) stop = d->block_counter - block_counter_before >= n;
        else if (strategy == B200Z_STRATEGY_UPTO_BYTES) stop = fd_buffer_len(d) - buffer_size_before >= n;
    }
    d->last_stage = 0;
    if (finished) *finished = d->frame_finished ? 1 : 0;
    return 0;
}

extern "C" int b200z_frame_decoder_decode_blocks(b200z_frame_decoder *d, b200z_read_fn rd, void *user, int strategy, size_t n, int *finished) {
    return fd_decode_blocks_impl(d, rd, user, strategy, n, finished, nullptr);
}

// drain `amount` bytes from the front of the device buffer into host memory / a writer; feeds the hash
static long fd_drain(b200z_frame_decoder *d, size_t amount, uint8_t *target, b200z_write_fn wr, void *user) {
    if (amount == 0) return 0;
    b200z_ctx *c = d->ctx;
    if (c->use()) return -1;
    std::vector<uint8_t> tmp;
    uint8_t *dst = target;
    if (!dst) { tmp.resize(amount); dst = tmp.data(); }
    if (cudaMemcpyAsync(dst, d->d_out.as<uint8_t>() + (d->drained - d->base), amount, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
        cudaStreamSynchronize(c->stream) != cudaSuccess) { cudaGetLastError(); return -1; }
    size_t written = amount;
    bool failed = false;
    if (!target) {  // write_all_bytes (decode_buffer.rs:318-328)
        written = 0;
        while (written < amount) {
            long w = wr(user, dst + written, amount - written);
            if (w == 0) break;
            if (w < 0) { failed = true; break; }
            written += (size_t)w;
        }
    }
    d->hash.update(dst, written);
    d->drained += written;
    return failed ? -1 : (long)written;
}

extern "C" long b200z_frame_decoder_read(b200z_frame_decoder *d, uint8_t *buf, size_t len) {  // impl Read :615-627
    if (!d || !d->has_state) return 0;
    size_t amount = d->frame_finished ? std::min(len, fd_buffer_len(d)) : std::min(len, fd_can_drain_to_window(d));
    return fd_drain(d, amount, buf, nullptr, nullptr);
}
extern "C" long b200z_frame_decoder_collect_to_writer(b200z_frame_decoder *d, b200z_write_fn wr, void *user) {  // :393-404
    if (!d || !d->has_state || !wr) return 0;
    size_t amount = fd_finished(d) ? fd_buffer_len(d) : fd_can_drain_to_window(d);
    return fd_drain(d, amount, nullptr, wr, user);
}
extern "C" size_t b200z_frame_decoder_can_collect(const b200z_frame_decoder *d) {  // :409-424
    if (!d || !d->has_state) return 0;
    return fd_finished(d) ? fd_buffer_len(d) : fd_can_drain_to_window(d);
}
extern "C" int b200z_frame_decoder_is_finished(const b200z_frame_decoder *d) { return d ? fd_finished(d) : 1; }
extern "C" size_t b200z_frame_decoder_blocks_decoded(const b200z_frame_decoder *d) { return d && d->has_state ? d->block_counter : 0; }
extern "C" uint64_t b200z_frame_decoder_bytes_read_from_source(const b200z_frame_decoder *d) { return d && d->has_state ? d->bytes_read_counter : 0; }
extern "C" uint64_t b200z_frame_decoder_content_size(const b200z_frame_decoder *d) { return d && d->has_state ? d->hdr.frame_content_size : 0; }
extern "C" int b200z_frame_decoder_get_checksum_from_data(const b200z_frame_decoder *d, uint32_t *out) {
    if (!d || !d->has_state || !d->has_check_sum) return 0;
    *out = d->check_sum; return 1;
}
extern "C" int b200z_frame_decoder_get_calculated_checksum(const b200z_frame_decoder *d, uint32_t *out) {
    if (!d || !d->has_state) return 0;
    *out = (uint32_t)d->hash.digest(); return 1;
}

// decode_from_to (frame_decoder.rs:439-529): decodes as many WHOLE blocks as `src` holds
extern "C" int b200z_frame_decoder_decode_from_to(b200z_frame_decoder *d, const uint8_t *src, size_t src_len, uint8_t *dst, size_t dst_len,
                                                  size_t *read, size_t *written) {
    if (!d || !read || !written) return B200Z_ERR_INVALID_ARGUMENT;
    uint64_t at_start = d->has_state ? d->bytes_read_counter : 0;
    if (!fd_finished(d) || !d->has_state) {
        SliceReader mt{src, src_len};
        if (!d->has_state) { int e = b200z_frame_decoder_init(d, slice_read, &mt); if (e) return e; }
        if (d->hdr.content_checksum() && d->frame_finished && !d->has_check_sum) {  // :465-477
            if (mt.len >= 4) {
                d->bytes_read_counter += 4;
                d->check_sum = rd32le(mt.p);
                d->has_check_sum = true;
            }
            *read = 4; *written = 0;
            return 0;
        }
        // the reference loops block by block while a whole block is present (:479-518); count them from the
        // headers, then decode exactly those in one submission
        size_t k = 0;
        int hdr_err = 0;
        {
            SliceReader probe = mt;
            while (probe.len >= 3) {
                BlockHeader bh;
                int e = parse_block_header(probe.p, bh);
                if (e) { hdr_err = e; break; }
                if (probe.len - 3 < bh.content_size) break;
                probe.p += 3 + bh.content_size; probe.len -= 3 + bh.content_size;
                k++;
                if (bh.last) break;
            }
        }
        if (k > 0) {
            int e = fd_decode_blocks_impl(d, slice_read, &mt, B200Z_STRATEGY_UPTO_BLOCKS, k, nullptr, &mt);
            if (e) return e;
        }
        if (hdr_err && !d->frame_finished) return fd_fail(d, hdr_err, B200Z_STAGE_BLOCK_HEADER);
    }
    long r = b200z_frame_decoder_read(d, dst, dst_len);
    if (r < 0) return fd_fail(d, B200Z_ERR_FAILED_TO_DRAIN_DECODEBUFFER, B200Z_STAGE_DRAIN);
    *written = (size_t)r;
    *read = (size_t)(d->bytes_read_counter - at_start);
    return 0;
}

// decode_all (frame_decoder.rs:541-577)
extern "C" int b200z_frame_decoder_decode_all(b200z_frame_decoder *d, const uint8_t *input, size_t input_len, uint8_t *output, size_t output_cap, size_t *written) {
    if (!d || !written) return B200Z_ERR_INVALID_ARGUMENT;
    SliceReader in{input, input_len};
    size_t total = 0;
    while (in.len != 0) {
        int e = b200z_frame_decoder_init(d, slice_read, &in);
        if (e == B200Z_ERR_SKIP_FRAME) {
            if ((size_t)d->skip_len > in.len) return fd_fail(d, B200Z_ERR_FAILED_TO_SKIP_FRAME, 0);
            in.p += d->skip_len; in.len -= d->skip_len;
            continue;
        }
        if (e) return e;
        for (;;) {
            if ((e = b200z_frame_decoder_decode_blocks(d, slice_read, &in, B200Z_STRATEGY_UPTO_BYTES, 1024 * 1024, nullptr))) return e;
            long w = b200z_frame_decoder_read(d, output + total, output_cap - total);
            if (w < 0) return fd_fail(d, B200Z_ERR_FAILED_TO_DRAIN_DECODEBUFFER, B200Z_STAGE_DRAIN);
            total += (size_t)w;
            if (b200z_frame_decoder_can_collect(d) != 0) return fd_fail(d, B200Z_ERR_TARGET_TOO_SMALL, 0);
            if (fd_finished(d)) break;
        }
    }
    *written = total;
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// StreamingDecoder mirror (decoding/streaming_decoder.rs)
// ---------------------------------------------------------------------------------------------------------------
struct b200z_streaming_decoder {
    b200z_frame_decoder *dec = nullptr;
    bool owns = false;
    b200z_read_fn rd = nullptr;
    void *user = nullptr;
};

static int sd_make(b200z_frame_decoder *dec, bool owns, b200z_read_fn rd, void *user, b200z_streaming_decoder **out) {
    int e = b200z_frame_decoder_init(dec, rd, user);
    if (e) { if (owns) b200z_frame_decoder_free(dec); return e; }
    b200z_streaming_decoder *s = new b200z_streaming_decoder();
    s->dec = dec; s->owns = owns; s->rd = rd; s->user = user;
    *out = s;
    return 0;
}
extern "C" int b200z_streaming_decoder_new(b200z_ctx *c, b200z_read_fn rd, void *user, b200z_streaming_decoder **out) {
    if (!c || !rd || !out) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_frame_decoder *dec = nullptr;
    int e = b200z_frame_decoder_new(c, &dec);
    if (e) return e;
    return sd_make(dec, true, rd, user, out);
}
extern "C" int b200z_streaming_decoder_new_with_decoder(b200z_read_fn rd, void *user, b200z_frame_decoder *dec, b200z_streaming_decoder **out) {
    if (!dec || !rd || !out) return B200Z_ERR_INVALID_ARGUMENT;
    return sd_make(dec, false, rd, user, out);
}
extern "C" int b200z_streaming_decoder_new_with_max_window_size(b200z_ctx *c, b200z_read_fn rd, void *user, uint64_t mw, b200z_streaming_decoder **out) {
    if (!c || !rd || !out) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_frame_decoder *dec = nullptr;
    int e = b200z_frame_decoder_new(c, &dec);
    if (e) return e;
    b200z_frame_decoder_set_max_window_size(dec, mw);
    return sd_make(dec, true, rd, user, out);
}
extern "C" long b200z_streaming_decoder_read(b200z_streaming_decoder *s, uint8_t *buf, size_t len, int *error) {  // :118-155
    if (error) *error = 0;
    if (!s) return -1;
    b200z_frame_decoder *d = s->dec;
    if (fd_finished(d) && b200z_frame_decoder_can_collect(d) == 0) return 0;
    while (b200z_frame_decoder_can_collect(d) < len && !fd_finished(d)) {
        size_t need = len - b200z_frame_decoder_can_collect(d);
        int e = b200z_frame_decoder_decode_blocks(d, s->rd, s->user, B200Z_STRATEGY_UPTO_BYTES, need, nullptr);
        if (e) { if (error) *error = e; return -1; }
    }
    return b200z_frame_decoder_read(d, buf, len);
}
extern "C" b200z_frame_decoder *b200z_streaming_decoder_frame_decoder(b200z_streaming_decoder *s) { return s ? s->dec : nullptr; }
extern "C" b200z_frame_decoder *b200z_streaming_decoder_into_frame_decoder(b200z_streaming_decoder *s) {
    if (!s) return nullptr;
    b200z_frame_decoder *d = s->dec;
    delete s;
    return d;
}
extern "C" void b200z_streaming_decoder_free(b200z_streaming_decoder *s) {
    if (!s) return;
    if (s->owns) b200z_frame_decoder_free(s->dec);
    delete s;
}

// ---------------------------------------------------------------------------------------------------------------
// batch compressor (encoding::compress / compress_to_vec / FrameCompressor::compress at Uncompressed and Fastest):
// host checks and the block plan, then k_cmatch -> k_cenc -> k_cxxh64 -> k_cassemble on the ctx stream
// ---------------------------------------------------------------------------------------------------------------
extern "C" size_t b200z_compress_bound(size_t n) {
    const size_t blocks = std::max<size_t>(1, (n + ENC_BLOCK - 1) / ENC_BLOCK);
    return n + 14 + 3 * blocks + 4;
}
// the ID a frame compressed against `d` carries: a formatted dictionary's own, none for raw content (libzstd's convention: it
// rejects a frame whose ID does not match a raw-content dictionary; the decoder selects one with forced_dict)
static uint32_t compress_dict_id(const b200z_dict *d) { return d && d->has_tables ? d->id : 0; }
extern "C" size_t b200z_compress_bound_dict(size_t n, const b200z_dict *d) { return b200z_compress_bound(n) + dict_id_field_size(compress_dict_id(d)); }
extern "C" int b200z_compress_num_stages(void) { return kCompressStages; }
extern "C" const char *b200z_compress_stage_name(int stage) { return stage >= 0 && stage < kCompressStages ? kCompressStageNames[stage] : ""; }

// k_cmatch / k_cenc staging for nblocks blocks (CompressArgs), and at OPT k_copt's chain slots
struct CompressStaging {
    DevBuf lit_stage, seq_stage, lits, seqs, info, res;
    DevBuf opt_prev;   // OPT and ULTRA: opt_ctas() slots of OPT_SPAN words, allocated by the first such submission and kept
    int ensure(uint64_t nblocks, bool grow, int level = B200Z_LEVEL_FASTEST) {
        int e = 0;
        if ((e = lit_stage.ensure(nblocks * ENC_BLOCK, grow)) || (e = seq_stage.ensure(nblocks * CBLOCK_SEQS * sizeof(SeqRec), grow)) ||
            (e = lits.ensure(nblocks * ENC_BLOCK, grow)) || (e = seqs.ensure(nblocks * CBLOCK_SEQS * sizeof(SeqRec), grow)) ||
            (e = info.ensure(nblocks * sizeof(CBlockInfo), grow)) || (e = res.ensure(nblocks * sizeof(CBlockInfo), grow)))
            return e;
        if ((level == B200Z_LEVEL_OPT || level == B200Z_LEVEL_ULTRA) && (e = opt_prev.ensure((uint64_t)opt_ctas() * OPT_SPAN * sizeof(int32_t)))) return e;
        return 0;
    }
    void bind(CompressArgs &a) const {
        a.lit_stage = lit_stage.as<uint8_t>(); a.seq_stage = seq_stage.as<SeqRec>(); a.lits = lits.as<uint8_t>(); a.seqs = seqs.as<SeqRec>();
        a.enc = a.lit_stage; a.info = info.as<CBlockInfo>(); a.res = res.as<CBlockInfo>(); a.opt_prev = opt_prev.as<int32_t>();
    }
};

// The two slots of a host-to-host pipeline around the ctx stream (the stream compressor, the seekable stream writer): slot s serves
// chunk or group k with k & 1 == s; uploads go on s_h2d, downloads on s_d2h.  A slot's buffers are reused only after the event of
// the last work that read them: ev_k (kernels: d_in, d_desc), ev_h2d (upload: h_in, h_desc), ev_d2h (download: d_out, h_out).
struct PipeSlots {
    Stream s_h2d, s_d2h;
    Event ev_h2d[2], ev_k[2], ev_d2h[2];
    PinnedBuf h_in[2], h_out[2], h_desc[2];
    DevBuf d_in[2], d_out[2], d_desc[2];
    int create(b200z_ctx *c) {   // the streams and events, once
        if (!s_h2d && s_h2d.create(c)) return B200Z_ERR_CUDA;
        if (!s_d2h && s_d2h.create(c)) return B200Z_ERR_CUDA;
        for (int i = 0; i < 2; i++)
            for (Event *e : {&ev_h2d[i], &ev_k[i], &ev_d2h[i]})
                if (!*e && e->create(c)) return B200Z_ERR_CUDA;
        return 0;
    }
    int ensure(size_t din, size_t hin, size_t dout, size_t hout, size_t desc) {   // each slot's buffers, at their exact sizes
        int e = 0;
        for (int i = 0; i < 2 && !e; i++)
            if ((e = d_in[i].ensure(din, false)) || (e = d_out[i].ensure(dout, false)) || (e = d_desc[i].ensure(desc, false)) ||
                (e = h_in[i].ensure(hin, false)) || (e = h_out[i].ensure(hout, false)) || (e = h_desc[i].ensure(desc, false)))
                break;
        return e;
    }
    void drain(cudaStream_t ks) {   // leaves nothing in flight on the copy streams and on ks (when given)
        if (s_h2d) cudaStreamSynchronize(s_h2d);
        if (ks) cudaStreamSynchronize(ks);
        if (s_d2h) cudaStreamSynchronize(s_d2h);
    }
    // The source through the slots, once the caller has read chunk 0 into slot 0 (n0 bytes; eof0: the source ended there).  For
    // chunk k in slot s: enqueue(k, s, n) queues a non-empty chunk's upload, kernels and download; read(s ^ 1, n, eof) reads chunk
    // k + 1 once chunk k - 1's upload is done with the other slot; write(k - 1, s ^ 1, n, false) writes chunk k - 1, n being the
    // bytes enqueued in its slot.  At the end of the source write(k, s, n, true) writes chunk k, even an empty one.  Each returns 0
    // or an error code; on an error nothing is left in flight.
    template <class Enqueue, class Read, class Write>
    int run(b200z_ctx *c, size_t n0, bool eof0, Enqueue enqueue, Read read, Write write) {
        size_t n[2] = {n0, 0}, sent[2] = {0, 0};   // the chunk read into h_in[s], and the one whose output is in slot s
        bool eof[2] = {eof0, false};
        int e = 0;
        for (uint64_t k = 0;; k++) {
            const int s = (int)(k & 1);
            sent[s] = n[s];
            if (n[s] && (e = enqueue(k, s, n[s]))) break;
            if (!eof[s]) {   // a chunk shorter than the slot ends the source, so this one is full
                if (k && cudaEventSynchronize(ev_h2d[s ^ 1]) != cudaSuccess) { e = c->set_cuda_err(cudaGetLastError(), "upload"); break; }
                if ((e = read(s ^ 1, n[s ^ 1], eof[s ^ 1]))) break;
            }
            if (k && (e = write(k - 1, s ^ 1, sent[s ^ 1], false))) break;
            if (eof[s]) { e = write(k, s, sent[s], true); break; }
        }
        if (e) drain(c->stream);
        return e;
    }
};

// long-distance matches (window_log > 17): the spans, k_lanchor's counts, the anchors and their sort, the forced matches and
// each block's share of them
struct LdmBufs {
    DevBuf spans, tcount, scount, keys[2], vals[2], hist, pos, frame, cand, forced, off, cnt;
    static size_t tiles(uint32_t cap) { return std::max<size_t>(1, (cap + LDM_TILE - 1) / LDM_TILE); }
    // the buffers for `cap` anchors: 44 bytes each, and 4 per 16 anchors of digit counts
    int ensure(uint32_t cap, bool grow = true) {
        const size_t n = std::max<uint32_t>(cap, 1);
        int e = 0;
        for (int i = 0; i < 2 && !e; i++)
            if ((e = keys[i].ensure(n * 4, grow)) || (e = vals[i].ensure(n * 4, grow))) return e;
        if ((e = hist.ensure((tiles(cap) * 256 + 1) * 4, grow)) || (e = pos.ensure(n * 8, grow)) || (e = frame.ensure(n * 4, grow)) ||
            (e = cand.ensure(n * 4, grow)) || (e = forced.ensure(n * sizeof(LForced), grow)))
            return e;
        return 0;
    }
    void bind(LdmArgs &l) const {
        for (int i = 0; i < 2; i++) { l.keys[i] = keys[i].as<uint32_t>(); l.vals[i] = vals[i].as<uint32_t>(); }
        l.hist = hist.as<uint32_t>(); l.apos = pos.as<uint64_t>(); l.aframe = frame.as<uint32_t>(); l.cand = cand.as<uint32_t>();
        l.forced = forced.as<LForced>(); l.lf_off = off.as<uint32_t>(); l.lf_cnt = cnt.as<uint32_t>();
    }
};

// ULTRA's far stage (compress.h): the largest group's pairs, sort counts and walk starts, and the pieces and per-block FBlocks
struct FarBufs {
    DevBuf pieces, fblk, total, keys[2], vals[2], hist, start;
    // 16 bytes per pair, 4 per virtual position, 4 per 16 pairs of digit counts, and the pieces and blocks
    int ensure(uint64_t npairs, uint64_t nvirt, uint64_t npieces, uint64_t nblocks, bool grow = true) {
        const size_t n = std::max<uint64_t>(npairs, 1);
        int e = 0;
        for (int i = 0; i < 2 && !e; i++)
            if ((e = keys[i].ensure(n * 4, grow)) || (e = vals[i].ensure(n * 4, grow))) return e;
        if ((e = hist.ensure((LdmBufs::tiles((uint32_t)n) * 256 + 1) * 4, grow)) || (e = start.ensure(std::max<uint64_t>(nvirt, 1) * 4, grow)) ||
            (e = total.ensure(4, grow)) || (e = pieces.ensure(std::max<uint64_t>(npieces, 1) * sizeof(FPiece), grow)) ||
            (e = fblk.ensure(std::max<uint64_t>(nblocks, 1) * sizeof(FBlock), grow)))
            return e;
        return 0;
    }
    FarArgs args(const uint8_t *input, const FPiece *d_pieces, uint32_t npieces, uint32_t npairs) const {
        FarArgs f{};
        f.input = input; f.pieces = d_pieces; f.npieces = npieces; f.npairs = npairs; f.total = total.as<uint32_t>();
        for (int i = 0; i < 2; i++) { f.keys[i] = keys[i].as<uint32_t>(); f.vals[i] = vals[i].as<uint32_t>(); }
        f.hist = hist.as<uint32_t>(); f.start = start.as<uint32_t>();
        return f;
    }
    void bind(CompressArgs &a, const FBlock *d_fblk) const {
        a.fblk = d_fblk; a.fkeys = keys[0].as<uint32_t>(); a.fvals = vals[0].as<uint32_t>(); a.fstart = start.as<uint32_t>();
    }
};
// the pieces of one group: adds FPiece{off, vbase, pbase, size} for a 128 KiB block and moves vbase and pbase past it
static void far_piece(std::vector<FPiece> &pc, uint64_t off, uint32_t size, uint64_t &vbase, uint64_t &pbase) {
    pc.push_back(FPiece{off, (uint32_t)vbase, (uint32_t)pbase, size, 0});
    vbase += size;
    pbase += size >= FAR_KEY ? size - (FAR_KEY - 1) : 0;
}
// the group size: B200Z_PIPELINE_CHUNK_BYTES rounded down to whole blocks (64 MiB by default), so that a group's virtual positions
// (its bytes and at most 2^27 before them) fit in 32 bits
static uint64_t far_group_bytes() {
    uint64_t C = 64ull << 20;
    if (const char *ev = getenv("B200Z_PIPELINE_CHUNK_BYTES")) C = strtoull(ev, nullptr, 10);
    return std::min<uint64_t>(1ull << 31, std::max<uint64_t>(ENC_BLOCK, C / ENC_BLOCK * ENC_BLOCK));
}

struct CompressResources {
    DevBuf frames, blocks, csum, results, input, output;
    CompressStaging stage;
    DevBuf dcontent, dtab, dcounts;   // b200z_dict_finalize: the content's tail, its match table and the statistics
    DevBuf seek_entries, seek_total;  // b200z_compress_seekable(_stream): the table's entries and the running archive size
    PipeSlots seek_pipe;              // b200z_compress_seekable_stream: d_desc is a group's size word, CFrames and CBlocks
    DevBuf rd_stage, rd_pieces;       // b200z_seekable_read_ranges: host output's slots and the scratch, the copy pieces
    PinnedBuf rd_host;                // b200z_seekable_read_ranges: the touched frames of a host archive, host output's slots
    LdmBufs ldm;                      // b200z_compress_frames_batch_long
    FarBufs far;                      // b200z_compress_frames_batch_long at ULTRA
    std::deque<Event> far_ev;         // profiled ULTRA submissions: around each group's k_copt
    Event ev[kCompressStages + 1];
    float stage_ms[kCompressStages] = {};
    bool profiled = false;
    // A submission of whole frames (the batch entry, the seekable writers): the staging, csum and results for `frames` frames in
    // `blocks` blocks; Uncompressed takes the blocks' results only, not the match and entropy staging
    int ensure_submission(uint64_t frames, uint64_t blocks, int level) {
        int e = 0;
        if ((e = level != B200Z_LEVEL_UNCOMPRESSED ? stage.ensure(blocks, true, level) : stage.res.ensure(blocks * sizeof(CBlockInfo))) ||
            (e = csum.ensure(frames * 8)) || (e = results.ensure(frames * sizeof(b200z_compress_result))))
            return e;
        return 0;
    }
    int bind_submission(b200z_ctx *c, const b200z_dict *dict, int level, bool checksum, CompressArgs &a);
};
// the context's, created by its first compression or dictionary finalization
static int compress_get(b200z_ctx *c, CompressResources **out) {
    if (!c->comp) {
        std::unique_ptr<CompressResources> r(new CompressResources());
        for (Event &e : r->ev) if (e.create(c, cudaEventDefault)) return B200Z_ERR_CUDA;
        c->comp = std::move(r);
    }
    *out = c->comp.get();
    return 0;
}
extern "C" int b200z_compress_last_profile(const b200z_ctx *c, float *stage_ms, size_t n) {
    if (!c || !stage_ms || !c->comp || !c->comp->profiled) return B200Z_ERR_INVALID_ARGUMENT;
    for (size_t i = 0; i < n && i < (size_t)kCompressStages; i++) stage_ms[i] = c->comp->stage_ms[i];
    return 0;
}

// A submission's CompressArgs but for its frames, blocks, input, output and counts: the dictionary's part (dict_id, the match table,
// the encoder's tables), the staging, csum, results, level and checksum.  The match table is built once and kept with the dictionary
// (not one of the timed stages); offsets stay within the 128 KiB window, so the kernels see the content's last ENC_WINDOW bytes
// only.  The encoder's view of a formatted dictionary's tables is built on the host once and kept with the dictionary (no launch).
int CompressResources::bind_submission(b200z_ctx *c, const b200z_dict *dict, int level, bool checksum, CompressArgs &a) {
    const bool fast = level != B200Z_LEVEL_UNCOMPRESSED;
    const bool match_dict = fast && dict && dict->content_len >= ENC_MIN_MATCH;
    const uint32_t dict_tail = dict ? (uint32_t)std::min<size_t>(dict->content_len, ENC_WINDOW) : 0;
    const uint8_t *dict_at = dict ? dict->d_content.as<uint8_t>() + (dict->content_len - dict_tail) : nullptr;
    if (match_dict && !dict->d_ctab.p) {
        DevBuf tab;
        CU(c, tab.alloc(sizeof(uint32_t) << CD_LOG));
        if (int le = launch_dict_table(dict_at, dict_tail, tab.as<uint32_t>(), c->stream, &c->launches)) return c->set_cuda_err((cudaError_t)le, "k_cdict");
        dict->d_ctab = std::move(tab);
    }
    const bool use_tables = fast && dict && dict->has_tables && (c->flags & B200Z_FLAG_DICT_TABLES);
    if (use_tables && !dict->d_enc.p) {
        std::unique_ptr<EncDict> ed(new EncDict());
        const int16_t *probs[3] = {dict->norm[0], dict->norm[1], dict->norm[2]};
        enc_dict_build(dict->huf_weights, dict->huf_nweights, probs, dict->nnorm, dict->log, *ed);
        DevBuf enc;
        CU(c, enc.alloc(sizeof(EncDict)));
        CU(c, cudaMemcpy(enc.p, ed.get(), sizeof(EncDict), cudaMemcpyHostToDevice));
        dict->d_enc = std::move(enc);
    }
    a.etab = use_tables ? dict->d_enc.as<EncDict>() : nullptr;
    a.dict_id = compress_dict_id(dict);
    if (match_dict) { a.dict = dict_at; a.dtab = dict->d_ctab.as<uint32_t>(); a.dict_len = dict_tail; }
    stage.bind(a);
    a.csum = csum.as<uint64_t>(); a.results = results.as<b200z_compress_result>();
    a.level = level; a.checksum = checksum ? 1 : 0;
    return 0;
}

// The level, window and dictionary rule of every compressing entry, checked before any launch, read or write
static int compress_check(b200z_ctx *c, int level, int window_log, const b200z_dict *dict) {
    if (level >= 2 && level <= 4) {   // Default / Better / Best: unimplemented!() in the reference
        if (c) c->err = "compression levels Default, Better and Best are unimplemented!() in the reference";
        return B200Z_ERR_REFERENCE_WOULD_PANIC;
    }
    if (!c || (level != B200Z_LEVEL_UNCOMPRESSED && level != B200Z_LEVEL_FASTEST && level != B200Z_LEVEL_LAZY && level != B200Z_LEVEL_OPT &&
               level != B200Z_LEVEL_ULTRA))
        return B200Z_ERR_INVALID_ARGUMENT;
    if (window_log < B200Z_WINDOW_LOG_MIN || window_log > B200Z_WINDOW_LOG_MAX || (level == B200Z_LEVEL_UNCOMPRESSED && window_log != B200Z_WINDOW_LOG_MIN)) {
        c->err = "window_log outside [17, 27], or above 17 at level Uncompressed";
        return B200Z_ERR_INVALID_ARGUMENT;
    }
    if (dict && dict->ctx != c) { c->err = "dictionary created on another context"; return B200Z_ERR_INVALID_ARGUMENT; }
    return 0;
}

// One frame's plan: its input [src_off, src_off + size) cut into 128 KiB CBlocks from hb[first_block] on (an empty frame is one empty
// block), each reaching back to the frame's start or ENC_WINDOW bytes; `before` is the frame's input in front of src_off (a stream
// chunk's k * C)
static CFrame plan_frame(uint64_t src_off, uint64_t size, uint64_t dst_off, uint64_t before, uint32_t frame, uint32_t first_block, CBlock *hb) {
    uint32_t b = first_block;
    uint64_t pos = 0;
    do {
        const uint32_t bs = (uint32_t)std::min<uint64_t>(ENC_BLOCK, size - pos);
        hb[b++] = CBlock{src_off + pos, bs, (uint32_t)std::min<uint64_t>(before + pos, ENC_WINDOW), frame, 0};
        pos += bs;
    } while (pos < size);
    return CFrame{src_off, size, dst_off, first_block, b - first_block};
}

extern "C" int b200z_compress_frames_batch(b200z_ctx *c, const uint8_t *input, size_t input_len, int input_mem, const b200z_compress_io *frames,
                                           size_t nframes, int level, int checksum, uint8_t *output, size_t output_cap, int output_mem,
                                           b200z_compress_result *results) {
    return b200z_compress_frames_batch_dict(c, input, input_len, input_mem, frames, nframes, level, checksum, nullptr, output, output_cap,
                                            output_mem, results);
}

extern "C" int b200z_compress_frames_batch_dict(b200z_ctx *c, const uint8_t *input, size_t input_len, int input_mem, const b200z_compress_io *frames,
                                                size_t nframes, int level, int checksum, const b200z_dict *dict, uint8_t *output,
                                                size_t output_cap, int output_mem, b200z_compress_result *results) {
    return b200z_compress_frames_batch_long(c, input, input_len, input_mem, frames, nframes, level, checksum, dict, B200Z_WINDOW_LOG_MIN, output,
                                            output_cap, output_mem, results);
}

// The long-distance match stage (ldm.cu) before k_cmatch, over the spans `sp` (LSpan.block indexes the submission's nblocks): anchors
// counted; with cap == 0 their total is read back to size the buffers (batch), else the buffers hold cap anchors (stream: the
// density bound).  Then anchors, sort, candidates and the blocks' forced matches into a.lforced / lf_*.
static int compress_ldm(b200z_ctx *c, LdmBufs &r, CompressArgs &a, const LSpan *d_spans, uint32_t nspans, uint32_t nblocks, uint32_t window_log,
                        uint32_t cap, cudaStream_t s, const b200z_dict *ldict = nullptr) {
    int e = 0;
    if ((e = r.tcount.ensure((size_t)nspans * LDM_THREADS * sizeof(uint32_t))) || (e = r.scount.ensure((nspans + 1) * sizeof(uint32_t))) ||
        (e = r.off.ensure(nblocks * sizeof(uint32_t))) ||
        (e = r.cnt.ensure(nblocks * sizeof(uint32_t))))
        return e;
    CU(c, cudaMemsetAsync(r.cnt.p, 0, nblocks * sizeof(uint32_t), s));
    LdmArgs l{};
    l.input = a.input; l.spans = d_spans; l.nspans = nspans; l.window_log = window_log; l.tcount = r.tcount.as<uint32_t>();
    l.scount = r.scount.as<uint32_t>();
    if (ldict) {   // B200Z_FLAG_DICT_LONG: candidates and sources in the dictionary too
        l.dict_long = true;
        l.ld = LDict{ldict->d_lanch.as<uint32_t>(), ldict->d_lanch.as<uint32_t>() + ldict->nlanch, ldict->nlanch, a.frames};
        l.ds = LDictSrc{ldict->d_content.as<uint8_t>(), ldict->content_len};
    }
    if (int le = launch_ldm_count(l, s, &c->launches)) return c->set_cuda_err((cudaError_t)le, "k_lanchor");
    l.cap = cap;
    if (!cap) {
        CU(c, cudaMemcpyAsync(&l.cap, l.scount + nspans, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        CU(c, cudaStreamSynchronize(s));
    }
    if ((e = r.ensure(l.cap))) return e;
    r.bind(l);
    if (int le = launch_ldm_match(l, s, &c->launches)) return c->set_cuda_err((cudaError_t)le, "k_lblock");
    a.lforced = l.forced; a.lf_off = l.lf_off; a.lf_cnt = l.lf_cnt;
    return 0;
}

// B200Z_FLAG_DICT_LONG: the dictionary's anchors, by its first use with the flag.  k_lanchor counts them over spans of at most one
// block of the content's last min(len, 2^27) bytes; their total is read back; then k_lanchor fills them, the key sort orders them
// (the scratch is the context's long-match buffers) and k_ldict keeps (key, distance from the end) with the dictionary: 8 bytes per
// anchor, LDM_DICT_LAUNCHES kernels (2 when there is none)
static int dict_long_anchors(b200z_ctx *c, LdmBufs &r, const b200z_dict *d, cudaStream_t s) {
    if (d->lanch_built) return 0;
    const uint64_t len = d->content_len, lo = len - std::min<uint64_t>(len, LDM_DICT_REACH);
    std::vector<LSpan> sp;
    for (uint64_t o = lo; o < len; o += ENC_BLOCK) sp.push_back(LSpan{o, lo, (uint32_t)std::min<uint64_t>(ENC_BLOCK, len - o), 0, LDM_NO_BLOCK, 0});
    if (!sp.empty()) {
        const uint32_t ns = (uint32_t)sp.size();
        int e = 0;
        if ((e = r.spans.ensure(ns * sizeof(LSpan))) || (e = r.tcount.ensure((size_t)ns * LDM_THREADS * sizeof(uint32_t))) ||
            (e = r.scount.ensure((ns + 1) * sizeof(uint32_t))))
            return e;
        CU(c, cudaMemcpyAsync(r.spans.p, sp.data(), ns * sizeof(LSpan), cudaMemcpyHostToDevice, s));
        LdmArgs l{};
        l.input = d->d_content.as<uint8_t>(); l.spans = r.spans.as<LSpan>(); l.nspans = ns; l.window_log = B200Z_WINDOW_LOG_MAX;
        l.tcount = r.tcount.as<uint32_t>(); l.scount = r.scount.as<uint32_t>();
        if (int le = launch_ldm_count(l, s, &c->launches)) return c->set_cuda_err((cudaError_t)le, "k_lanchor");
        CU(c, cudaMemcpyAsync(&l.cap, l.scount + ns, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        CU(c, cudaStreamSynchronize(s));
        if (l.cap) {
            if ((e = r.ensure(l.cap))) return e;
            r.bind(l);
            DevBuf keep;
            CU(c, keep.alloc((size_t)l.cap * 2 * sizeof(uint32_t)));
            if (int le = launch_ldm_dict(l, len, keep.as<uint32_t>(), keep.as<uint32_t>() + l.cap, s, &c->launches))
                return c->set_cuda_err((cudaError_t)le, "k_ldict");
            d->d_lanch = std::move(keep);
            d->nlanch = l.cap;
        }
    }
    d->lanch_built = true;
    return 0;
}

// ULTRA's groups over a submission's blocks hb[nblocks] (frames hf): consecutive blocks of at most C bytes in all.  A group's
// pieces are, for each frame of it whose window Wf is beyond 131072, the frame's blocks in the Wf bytes before its first block in the
// group, then its blocks in the group, numbered on in one virtual space; fb[b] is block b's FBlock.  Returns whether any block has
// a far walk (else ULTRA is OPT and no far stage runs).
struct FarGroup { uint32_t b0, b1, p0, p1; uint64_t npairs, nvirt; };
static bool far_plan(const CFrame *hf, const CBlock *hb, uint32_t nblocks, uint32_t window_log, uint64_t C, std::vector<FarGroup> &groups,
                     std::vector<FPiece> &pieces, std::vector<FBlock> &fb) {
    bool any = false;
    fb.resize(nblocks);
    for (uint32_t b = 0; b < nblocks;) {
        FarGroup g{b, b, (uint32_t)pieces.size(), 0, 0, 0};
        uint64_t bytes = 0, vbase = 0, pbase = 0;
        while (b < nblocks && (b == g.b0 || bytes + hb[b].size <= C)) {
            const CFrame &f = hf[hb[b].frame];
            const uint64_t wf = 1ull << frame_window_log(f.src_size, window_log), pos = hb[b].src_off - f.src_off;
            if (wf > ENC_WINDOW) {
                if (b == g.b0 || hb[b - 1].frame != hb[b].frame)   // the frame's first block in the group: its history first
                    for (uint32_t j = b - (uint32_t)(std::min(pos, wf) / ENC_BLOCK); j < b; j++) far_piece(pieces, hb[j].src_off, hb[j].size, vbase, pbase);
                fb[b] = FBlock{(uint32_t)vbase, (uint32_t)std::min(pos, wf), (uint32_t)wf, 0};
                far_piece(pieces, hb[b].src_off, hb[b].size, vbase, pbase);
                any = true;
            } else {
                fb[b] = FBlock{FAR_NONE, hb[b].back, ENC_WINDOW, 0};
            }
            bytes += hb[b].size;
            b++;
        }
        g.b1 = b; g.p1 = (uint32_t)pieces.size(); g.npairs = pbase; g.nvirt = vbase;
        groups.push_back(g);
    }
    return any;
}

extern "C" int b200z_compress_frames_batch_long(b200z_ctx *c, const uint8_t *input, size_t input_len, int input_mem, const b200z_compress_io *frames,
                                                size_t nframes, int level, int checksum, const b200z_dict *dict, int window_log, uint8_t *output,
                                                size_t output_cap, int output_mem, b200z_compress_result *results) {
    // ---- everything is checked before any device work
    if (int e = compress_check(c, level, window_log, dict)) return e;
    if ((nframes && (!frames || !results)) || (input_mem != B200Z_MEM_HOST && input_mem != B200Z_MEM_DEVICE) ||
        (output_mem != B200Z_MEM_HOST && output_mem != B200Z_MEM_DEVICE) || (input_len && !input) || (output_cap && !output) || nframes > 0xffffffffu) {
        c->err = "invalid argument";
        return B200Z_ERR_INVALID_ARGUMENT;
    }
    std::vector<std::pair<uint64_t, uint64_t>> dst;
    uint64_t nblocks = 0;
    for (size_t i = 0; i < nframes; i++) {
        const b200z_compress_io &f = frames[i];
        if (f.src_off > input_len || f.src_size > input_len - f.src_off || f.dst_off > output_cap || f.dst_cap > output_cap - f.dst_off ||
            f.dst_cap < b200z_compress_bound_dict(f.src_size, dict)) {
            c->err = "frame " + std::to_string(i) + ": range outside input/output or dst_cap < b200z_compress_bound_dict(src_size, dict)";
            return B200Z_ERR_INVALID_ARGUMENT;
        }
        dst.push_back({f.dst_off, f.dst_cap});
        nblocks += std::max<uint64_t>(1, (f.src_size + ENC_BLOCK - 1) / ENC_BLOCK);
    }
    std::sort(dst.begin(), dst.end());
    for (size_t i = 1; i < dst.size(); i++)
        if (dst[i - 1].first + dst[i - 1].second > dst[i].first) { c->err = "overlapping destination ranges"; return B200Z_ERR_INVALID_ARGUMENT; }
    if (nblocks > 0xffffffffu) return B200Z_ERR_INVALID_ARGUMENT;
    if (!nframes) return 0;
    if (int e = c->use()) return e;
    // ---- plan: frames -> 128 KiB blocks
    std::vector<CFrame> hf(nframes);
    std::vector<CBlock> hb(nblocks);
    for (size_t i = 0, b = 0; i < nframes; i++) {
        hf[i] = plan_frame(frames[i].src_off, frames[i].src_size, frames[i].dst_off, 0, (uint32_t)i, (uint32_t)b, hb.data());
        b += hf[i].nblocks;
    }
    CompressResources *rp = nullptr;
    if (int e = compress_get(c, &rp)) return e;
    CompressResources &r = *rp;
    const bool fast = level != B200Z_LEVEL_UNCOMPRESSED;   // Fastest, LAZY or OPT: the blocks are parsed and encoded
    int e = 0;
    if ((e = r.frames.ensure(nframes * sizeof(CFrame))) || (e = r.blocks.ensure(nblocks * sizeof(CBlock))) ||
        (e = r.ensure_submission(nframes, nblocks, level)))
        return e;
    const uint8_t *d_in = input;
    uint8_t *d_out = output;
    cudaStream_t s = c->stream;
    if (input_mem == B200Z_MEM_HOST) {
        if ((e = r.input.ensure(input_len + 16))) return e;
        CU(c, cudaMemcpyAsync(r.input.p, input, input_len, cudaMemcpyHostToDevice, s));
        d_in = r.input.as<uint8_t>();
    }
    if (output_mem == B200Z_MEM_HOST) {
        if ((e = r.output.ensure(output_cap + 16))) return e;
        d_out = r.output.as<uint8_t>();
    }
    CU(c, cudaMemcpyAsync(r.frames.p, hf.data(), nframes * sizeof(CFrame), cudaMemcpyHostToDevice, s));
    CU(c, cudaMemcpyAsync(r.blocks.p, hb.data(), nblocks * sizeof(CBlock), cudaMemcpyHostToDevice, s));
    CompressArgs a{};
    if ((e = r.bind_submission(c, dict, level, checksum != 0, a))) return e;
    a.frames = r.frames.as<CFrame>(); a.blocks = r.blocks.as<CBlock>(); a.input = d_in; a.output = d_out;
    a.nframes = (uint32_t)nframes; a.nblocks = (uint32_t)nblocks;
    a.window_log = (uint32_t)window_log;
    // B200Z_FLAG_DICT_LONG: long matches reach into the dictionary's content, and every frame's window covers it
    const bool dlong = fast && dict && window_log > B200Z_WINDOW_LOG_MIN && (c->flags & B200Z_FLAG_DICT_LONG);
    if (dlong) {
        if ((e = dict_long_anchors(c, r.ldm, dict, s))) return e;
        a.ldict = dict->d_content.as<uint8_t>(); a.ldict_len = dict->content_len;
    }
    if (fast && window_log > B200Z_WINDOW_LOG_MIN) {   // the blocks of the frames larger than one block (with the dictionary's reach: all)
        std::vector<LSpan> sp;
        for (uint32_t b = 0; b < (uint32_t)nblocks; b++)
            if (dlong || hf[hb[b].frame].src_size > ENC_BLOCK) sp.push_back(LSpan{hb[b].src_off, hf[hb[b].frame].src_off, hb[b].size, hb[b].frame, b, 0});
        if (!sp.empty()) {
            if ((e = r.ldm.spans.ensure(sp.size() * sizeof(LSpan)))) return e;
            CU(c, cudaMemcpyAsync(r.ldm.spans.p, sp.data(), sp.size() * sizeof(LSpan), cudaMemcpyHostToDevice, s));
            if ((e = compress_ldm(c, r.ldm, a, r.ldm.spans.as<LSpan>(), (uint32_t)sp.size(), (uint32_t)nblocks, (uint32_t)window_log, 0, s,
                                  dlong ? dict : nullptr)))
                return e;
        }
    }
    // ULTRA: the groups of whole blocks, each with the pieces of its far frames (their history, then their blocks in the group)
    std::vector<FarGroup> groups;
    std::vector<FPiece> pieces;
    std::vector<FBlock> fb;
    if (level == B200Z_LEVEL_ULTRA && window_log > B200Z_WINDOW_LOG_MIN &&
        far_plan(hf.data(), hb.data(), (uint32_t)nblocks, (uint32_t)window_log, far_group_bytes(), groups, pieces, fb)) {
        uint64_t mp = 0, mv = 0;
        for (const FarGroup &g : groups) { mp = std::max(mp, g.npairs); mv = std::max(mv, g.nvirt); }
        if ((e = r.far.ensure(mp, mv, pieces.size(), nblocks))) return e;
        CU(c, cudaMemcpyAsync(r.far.pieces.p, pieces.data(), pieces.size() * sizeof(FPiece), cudaMemcpyHostToDevice, s));
        CU(c, cudaMemcpyAsync(r.far.fblk.p, fb.data(), fb.size() * sizeof(FBlock), cudaMemcpyHostToDevice, s));
    } else {
        groups.clear();
    }
    const bool prof = (c->flags & B200Z_FLAG_PROFILE) != 0;
    if (prof) {
        CU(c, cudaEventRecord(r.ev[0], s));
        while (r.far_ev.size() < 2 * groups.size()) {
            r.far_ev.emplace_back();
            if (r.far_ev.back().create(c, cudaEventDefault)) { r.far_ev.pop_back(); return B200Z_ERR_CUDA; }
        }
    }
    for (int st = 0; st < kCompressStages; st++) {
        if (st == 0 && !groups.empty()) {   // per group: its far stage, then k_copt over its blocks
            for (size_t g = 0; g < groups.size(); g++) {
                const FarGroup &G = groups[g];
                if (G.p1 > G.p0) {
                    const FarArgs fa = r.far.args(d_in, r.far.pieces.as<FPiece>() + G.p0, G.p1 - G.p0, (uint32_t)G.npairs);
                    if (int le = launch_far_stage(fa, s, &c->launches)) return c->set_cuda_err((cudaError_t)le, "k_fkey / k_fstart");
                }
                CompressArgs ga = a;
                const size_t b0 = G.b0;
                ga.blocks = a.blocks + b0; ga.nblocks = G.b1 - G.b0;
                ga.lit_stage = a.lit_stage + b0 * ENC_BLOCK; ga.seq_stage = a.seq_stage + b0 * CBLOCK_SEQS;
                ga.lits = a.lits + b0 * ENC_BLOCK; ga.seqs = a.seqs + b0 * CBLOCK_SEQS; ga.info = a.info + b0;
                ga.lf_off = a.lf_off + b0; ga.lf_cnt = a.lf_cnt + b0;
                r.far.bind(ga, r.far.fblk.as<FBlock>() + b0);
                if (prof) CU(c, cudaEventRecord(r.far_ev[2 * g], s));
                if (int le = launch_compress_stage(ga, 0, s, &c->launches)) return c->set_cuda_err((cudaError_t)le, kCompressStageNames[0]);
                if (prof) CU(c, cudaEventRecord(r.far_ev[2 * g + 1], s));
            }
        } else if (int le = launch_compress_stage(a, st, s, &c->launches)) {
            return c->set_cuda_err((cudaError_t)le, kCompressStageNames[st]);
        }
        if (prof) CU(c, cudaEventRecord(r.ev[st + 1], s));
    }
    CU(c, cudaMemcpyAsync(results, r.results.p, nframes * sizeof(b200z_compress_result), cudaMemcpyDeviceToHost, s));
    CU(c, cudaStreamSynchronize(s));
    if (output_mem == B200Z_MEM_HOST)
        for (size_t i = 0; i < nframes; i++)
            CU(c, cudaMemcpy(output + frames[i].dst_off, d_out + frames[i].dst_off, results[i].dst_size, cudaMemcpyDeviceToHost));
    r.profiled = prof;
    if (prof) {
        for (int st = 0; st < kCompressStages; st++) CU(c, cudaEventElapsedTime(&r.stage_ms[st], r.ev[st], r.ev[st + 1]));
        if (!groups.empty()) {   // stage 0 is the groups' k_copt, not their far stages
            r.stage_ms[0] = 0;
            for (size_t g = 0; g < groups.size(); g++) {
                float ms = 0;
                CU(c, cudaEventElapsedTime(&ms, r.far_ev[2 * g], r.far_ev[2 * g + 1]));
                r.stage_ms[0] += ms;
            }
        }
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// seekable archives (EXTENSION: zstd's seekable format, DESIGN.md section 4.10).  Writing: the batch compressor's kernels per group of
// whole frames, with k_cscan packing each group's frames behind the archive so far, and k_cseek writing the table.  Reading: the table
// is parsed on the host, the ranges become a plan (frames to decode, in place or into scratch, and copy pieces), the frames go through
// the batch decoder's planner and pass, and k_range_gather copies the pieces.
// ---------------------------------------------------------------------------------------------------------------
static uint64_t seek_table_size(uint64_t nframes, bool checksum) { return SEEK_TABLE_FIXED + nframes * (checksum ? 12 : 8); }

extern "C" size_t b200z_seekable_bound(size_t n, size_t frame_size, int checksum, const b200z_dict *dict) {
    if (!frame_size || frame_size > B200Z_SEEKABLE_MAX_FRAME_SIZE) return 0;
    const uint64_t full = n / frame_size, rest = n % frame_size;
    return full * b200z_compress_bound_dict(frame_size, dict) + (rest ? b200z_compress_bound_dict(rest, dict) : 0) +
           seek_table_size(full + (rest ? 1 : 0), checksum != 0);
}

static uint64_t seek_frame_blocks(uint64_t frame_size) { return std::max<uint64_t>(1, (frame_size + ENC_BLOCK - 1) / ENC_BLOCK); }   // of a full frame

// What a group of `bytes` source bytes from a frame boundary holds: frames, blocks, input bytes and its frames' bounds
namespace {
struct SeekGroupSize { uint64_t frames, blocks, in, out; };
}  // namespace
static SeekGroupSize seek_group_size(uint64_t bytes, uint64_t frame_size, const b200z_dict *dict) {
    const uint64_t full = bytes / frame_size, rest = bytes % frame_size;
    return SeekGroupSize{full + (rest ? 1 : 0), full * seek_frame_blocks(frame_size) + (rest ? (rest + ENC_BLOCK - 1) / ENC_BLOCK : 0), bytes,
                         full * b200z_compress_bound_dict(frame_size, dict) + (rest ? b200z_compress_bound_dict(rest, dict) : 0)};
}

// The plan of frames [f0, f1) of a source cut every frame_size bytes and ending at `end`: input offsets less `base`, CBlock.frame
// counted from f0.  Returns the blocks written to hb.
static uint32_t seek_group_plan(uint64_t f0, uint64_t f1, uint64_t frame_size, uint64_t end, uint64_t base, CFrame *hf, CBlock *hb) {
    uint32_t nb = 0;
    for (uint64_t f = f0; f < f1; f++) {
        hf[f - f0] = plan_frame(f * frame_size - base, std::min<uint64_t>(frame_size, end - f * frame_size), 0, 0, (uint32_t)(f - f0), nb, hb);
        nb += hf[f - f0].nblocks;
    }
    return nb;
}

// A group's kernels on stream s, once a's frames, blocks, input and output are set: the compressor's stages, with k_cscan before
// k_cassemble packing the frames behind *total (less origin) and writing their table entries from frame first_frame on
static int seek_group_run(b200z_ctx *c, const CompressArgs &a, uint64_t *total, uint64_t origin, uint8_t *entries, uint64_t first_frame,
                          cudaStream_t s) {
    for (int st = 0; st < kCompressStages; st++) {
        if (st == 3)
            if (int le = launch_seek_scan(a, total, origin, entries, first_frame, s, &c->launches)) return c->set_cuda_err((cudaError_t)le, "k_cscan");
        if (int le = launch_compress_stage(a, st, s, &c->launches)) return c->set_cuda_err((cudaError_t)le, kCompressStageNames[st]);
    }
    return 0;
}

extern "C" int b200z_compress_seekable(b200z_ctx *c, const uint8_t *input, size_t input_len, int input_mem, size_t frame_size, int level,
                                       int checksum, const b200z_dict *dict, uint8_t *output, size_t output_cap, int output_mem, size_t *written) {
    // ---- everything is checked before any device work
    if (int e = compress_check(c, level, B200Z_WINDOW_LOG_MIN, dict)) return e;
    if ((input_mem != B200Z_MEM_HOST && input_mem != B200Z_MEM_DEVICE) || (output_mem != B200Z_MEM_HOST && output_mem != B200Z_MEM_DEVICE) ||
        (input_len && !input) || !output || !written) {
        c->err = "invalid argument";
        return B200Z_ERR_INVALID_ARGUMENT;
    }
    if (!frame_size || frame_size > B200Z_SEEKABLE_MAX_FRAME_SIZE) { c->err = "frame_size must lie in [1, 2^30]"; return B200Z_ERR_INVALID_ARGUMENT; }
    const uint64_t nframes = (input_len + frame_size - 1) / frame_size;
    if (nframes > 0xffffffffull) { c->err = "more than 2^32 - 1 frames"; return B200Z_ERR_INVALID_ARGUMENT; }
    if (output_cap < b200z_seekable_bound(input_len, frame_size, checksum, dict)) {
        c->err = "output_cap < b200z_seekable_bound(input_len, frame_size, checksum, dict)";
        return B200Z_ERR_INVALID_ARGUMENT;
    }
    *written = 0;
    if (int e = c->use()) return e;
    CompressResources *rp = nullptr;
    if (int e = compress_get(c, &rp)) return e;
    CompressResources &r = *rp;
    const bool sum = checksum != 0;
    const uint64_t per_group = std::max<uint64_t>(1, B200Z_SEEKABLE_GROUP_BLOCKS / seek_frame_blocks(frame_size));   // frames per group
    // what the largest group holds -- frames, blocks, input bytes and its frames' bounds -- from the frames the input really has:
    // every group but the last is full, so the first and the last group are the candidates
    SeekGroupSize g{1, 1, 0, 0};
    for (uint64_t f0 : {uint64_t(0), nframes ? (nframes - 1) / per_group * per_group : uint64_t(0)}) {
        const uint64_t f1 = std::min(nframes, f0 + per_group);
        const SeekGroupSize x = seek_group_size(std::min<uint64_t>(f1 * frame_size, input_len) - std::min<uint64_t>(f0 * frame_size, input_len),
                                                frame_size, dict);
        g = SeekGroupSize{std::max(g.frames, x.frames), std::max(g.blocks, x.blocks), std::max(g.in, x.in), std::max(g.out, x.out)};
    }
    const uint64_t gframes = g.frames, gblocks = g.blocks, gin = g.in, gout = g.out;
    const uint64_t table = seek_table_size(nframes, sum);
    int e = 0;
    if ((e = r.frames.ensure(gframes * sizeof(CFrame))) || (e = r.blocks.ensure(gblocks * sizeof(CBlock))) ||
        (e = r.ensure_submission(gframes, gblocks, level)) || (e = r.seek_entries.ensure(std::max<uint64_t>(table, 16))) ||
        (e = r.seek_total.ensure(8)))
        return e;
    if (input_mem == B200Z_MEM_HOST && (e = r.input.ensure(gin + 16))) return e;
    if (output_mem == B200Z_MEM_HOST && (e = r.output.ensure(std::max(gout, table) + 16))) return e;
    cudaStream_t s = c->stream;
    CompressArgs a{};
    if ((e = r.bind_submission(c, dict, level, sum, a))) return e;
    a.frames = r.frames.as<CFrame>(); a.blocks = r.blocks.as<CBlock>();
    uint64_t *d_total = r.seek_total.as<uint64_t>();
    CU(c, cudaMemsetAsync(d_total, 0, 8, s));
    uint64_t origin = 0;        // archive offset of d_out's byte 0 (host output: the group's first byte)
    std::vector<CFrame> hf(gframes);
    std::vector<CBlock> hb(gblocks);
    for (uint64_t f0 = 0; f0 < nframes; f0 += per_group) {
        const uint64_t f1 = std::min(nframes, f0 + per_group);
        const uint64_t in0 = f0 * frame_size, in1 = std::min<uint64_t>(f1 * frame_size, input_len);
        const uint64_t base = input_mem == B200Z_MEM_HOST ? in0 : 0;   // host input: the group is uploaded to r.input's byte 0
        a.nframes = (uint32_t)(f1 - f0);
        a.nblocks = seek_group_plan(f0, f1, frame_size, input_len, base, hf.data(), hb.data());
        a.input = input;
        if (input_mem == B200Z_MEM_HOST) {
            CU(c, cudaMemcpyAsync(r.input.p, input + in0, in1 - in0, cudaMemcpyHostToDevice, s));
            a.input = r.input.as<uint8_t>();
        }
        a.output = output_mem == B200Z_MEM_HOST ? r.output.as<uint8_t>() : output;
        CU(c, cudaMemcpyAsync(r.frames.p, hf.data(), a.nframes * sizeof(CFrame), cudaMemcpyHostToDevice, s));
        CU(c, cudaMemcpyAsync(r.blocks.p, hb.data(), a.nblocks * sizeof(CBlock), cudaMemcpyHostToDevice, s));
        if (int e2 = seek_group_run(c, a, d_total, origin, r.seek_entries.as<uint8_t>(), f0, s)) return e2;
        if (output_mem == B200Z_MEM_HOST) {   // the group's frames, d_out[0, total - origin), to the archive at origin
            uint64_t total = 0;
            CU(c, cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, s));
            CU(c, cudaStreamSynchronize(s));
            CU(c, cudaMemcpy(output + origin, r.output.p, total - origin, cudaMemcpyDeviceToHost));
            origin = total;
        }
    }
    if (int le = launch_seek_table(r.seek_entries.as<uint8_t>(), nframes, a.checksum, d_total, origin,
                                   output_mem == B200Z_MEM_HOST ? r.output.as<uint8_t>() : output, s, &c->launches))
        return c->set_cuda_err((cudaError_t)le, "k_cseek");
    uint64_t total = 0;
    CU(c, cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, s));
    CU(c, cudaStreamSynchronize(s));
    if (output_mem == B200Z_MEM_HOST) CU(c, cudaMemcpy(output + total, r.output.p, table, cudaMemcpyDeviceToHost));
    *written = total + table;
    return 0;
}

// ---- the seekable stream writer: groups of whole frames read from a source, two slots (PipeSlots), the table at the end
static int seek_io(b200z_ctx *c, const std::string &what) {
    c->err = what;
    return B200Z_ERR_SEEKABLE_IO;
}

// Group k (slot s = k & 1) is read into h_in[s], uploaded with its plan, compressed and packed from d_out[s]'s byte 0 behind the
// slot's own running-size word (the first 8 bytes of d_desc[s], uploaded as 0), and downloaded with that word; k_cscan writes the
// entries at their global frame index.  While group k uploads and compresses, the host reads group k + 1 and writes group k - 1.
static int seek_stream(b200z_ctx *c, b200z_read_fn rd, void *ru, b200z_write_fn wr, void *wu, uint64_t fs, int level, bool sum,
                       const b200z_dict *dict, b200z_seekable_stream_result &res) {
    if (int e = c->use()) return e;
    CompressResources *rp = nullptr;
    if (int e = compress_get(c, &rp)) return e;
    CompressResources &r = *rp;
    PipeSlots &P = r.seek_pipe;
    if (P.create(c)) return B200Z_ERR_CUDA;
    const uint64_t C = sd_chunk_bytes(), esz = sum ? 12 : 8;
    const uint64_t G = std::max<uint64_t>(1, std::min<uint64_t>(C / fs, B200Z_SEEKABLE_GROUP_BLOCKS / seek_frame_blocks(fs))) * fs;
    cudaStream_t ks = c->stream;
    const auto oom = [&](int e) { c->err = "seekable stream: out of memory for groups of " + std::to_string(G) + " bytes"; return e; };
    int e = 0;
    if ((e = P.ensure(0, G, 0, 0, 0))) return oom(e);   // the rest is sized by the first group, once it is read
    // the entries so far, doubled when full: the old buffer is copied on the kernel stream and kept until the call ends, since
    // freeing it earlier (cudaFree) would wait for the whole device in the middle of the pipeline
    std::vector<DevBuf> retired;
    const auto grow_entries = [&](uint64_t need) -> int {
        if (need <= r.seek_entries.cap) return 0;
        DevBuf nb;
        if (nb.alloc(std::max<uint64_t>(need, 2 * r.seek_entries.cap)) != cudaSuccess) return oom(B200Z_ERR_OUT_OF_MEMORY);
        if (res.frames) CU(c, cudaMemcpyAsync(nb.p, r.seek_entries.p, res.frames * esz, cudaMemcpyDeviceToDevice, ks));
        std::swap(nb, r.seek_entries);
        retired.push_back(std::move(nb));
        return 0;
    };
    const auto read_group = [&](int s, size_t &n, bool &eof) -> int {
        if (!read_chunk(rd, ru, P.h_in[s].as<uint8_t>(), G, &n, &eof))
            return seek_io(c, "seekable stream: read_cb failed at source offset " + std::to_string(res.read) + " (archive offset " +
                                  std::to_string(res.written) + ")");
        res.read += n;
        return 0;
    };
    size_t n0 = 0;
    bool eof0 = false;
    if ((e = read_group(0, n0, eof0)) || (e = grow_entries(16))) return e;
    // every buffer sized by the first group, the largest one the source has (every group but the last is full)
    const SeekGroupSize g = seek_group_size(n0, fs, dict);
    const uint64_t desc = 8 + g.frames * sizeof(CFrame) + g.blocks * sizeof(CBlock);
    if (n0 && ((e = P.ensure(g.in + 16, G, g.out + 16, g.out + 16, desc)) || (e = r.ensure_submission(g.frames, g.blocks, level)))) return oom(e);
    CompressArgs a{};
    if ((e = r.bind_submission(c, dict, level, sum, a))) return e;
    const auto enqueue = [&](uint64_t k, int s, size_t n) -> int {
        const uint64_t nf = (n + fs - 1) / fs;
        if (res.frames + nf > 0xffffffffull) { c->err = "seekable stream: more than 2^32 - 1 frames"; return B200Z_ERR_INVALID_ARGUMENT; }
        if (int ge = grow_entries((res.frames + nf) * esz)) return ge;
        uint8_t *hd = P.h_desc[s].as<uint8_t>(), *dd = P.d_desc[s].as<uint8_t>();
        memset(hd, 0, 8);
        CFrame *hf = reinterpret_cast<CFrame *>(hd + 8);
        const uint32_t nb = seek_group_plan(0, nf, fs, n, 0, hf, reinterpret_cast<CBlock *>(hf + nf));
        CU(c, cudaStreamWaitEvent(P.s_h2d, P.ev_k[s], 0));   // group k - 2's kernels are done with d_in[s] and d_desc[s]
        CU(c, cudaMemcpyAsync(P.d_in[s].p, P.h_in[s].p, n, cudaMemcpyHostToDevice, P.s_h2d));
        CU(c, cudaMemcpyAsync(dd, hd, 8 + nf * sizeof(CFrame) + nb * sizeof(CBlock), cudaMemcpyHostToDevice, P.s_h2d));
        CU(c, cudaEventRecord(P.ev_h2d[s], P.s_h2d));
        CU(c, cudaStreamWaitEvent(ks, P.ev_h2d[s], 0));
        a.frames = reinterpret_cast<const CFrame *>(dd + 8); a.blocks = reinterpret_cast<const CBlock *>(a.frames + nf);
        a.input = P.d_in[s].as<uint8_t>(); a.output = P.d_out[s].as<uint8_t>();
        a.nframes = (uint32_t)nf; a.nblocks = nb;
        if (int ke = seek_group_run(c, a, reinterpret_cast<uint64_t *>(dd), 0, r.seek_entries.as<uint8_t>(), res.frames, ks)) return ke;
        CU(c, cudaEventRecord(P.ev_k[s], ks));
        // the packed size, then the frames: the download takes their bounds, so that no host wait stands between the two
        CU(c, cudaStreamWaitEvent(P.s_d2h, P.ev_k[s], 0));
        CU(c, cudaMemcpyAsync(hd, dd, 8, cudaMemcpyDeviceToHost, P.s_d2h));
        CU(c, cudaMemcpyAsync(P.h_out[s].p, a.output, seek_group_size(n, fs, dict).out, cudaMemcpyDeviceToHost, P.s_d2h));
        CU(c, cudaEventRecord(P.ev_d2h[s], P.s_d2h));
        res.frames += nf;
        res.groups++;
        return 0;
    };
    const auto write_group = [&](uint64_t k, int s, size_t n, bool final) -> int {
        if (!n) return 0;   // the source ended on a group boundary
        CU(c, cudaEventSynchronize(P.ev_d2h[s]));
        uint64_t packed = 0;
        memcpy(&packed, P.h_desc[s].p, 8);
        if (!write_all(wr, wu, P.h_out[s].as<uint8_t>(), packed, &res.written))
            return seek_io(c, "seekable stream: write_cb failed at archive offset " + std::to_string(res.written));
        return 0;
    };
    if ((e = P.run(c, n0, eof0, enqueue, read_group, write_group))) return e;
    // the table: k_cseek behind a zeroed word into r.output, downloaded and written
    const uint64_t table = seek_table_size(res.frames, sum);
    if ((e = r.output.ensure(table + 16)) || (e = r.seek_total.ensure(8))) return oom(e);
    CU(c, cudaMemsetAsync(r.seek_total.p, 0, 8, ks));
    if (int le = launch_seek_table(r.seek_entries.as<uint8_t>(), res.frames, a.checksum, r.seek_total.as<uint64_t>(), 0, r.output.as<uint8_t>(), ks,
                                   &c->launches))
        return c->set_cuda_err((cudaError_t)le, "k_cseek");
    std::vector<uint8_t> tab(table);
    CU(c, cudaMemcpyAsync(tab.data(), r.output.p, table, cudaMemcpyDeviceToHost, ks));
    CU(c, cudaStreamSynchronize(ks));
    if (!write_all(wr, wu, tab.data(), table, &res.written))
        return seek_io(c, "seekable stream: write_cb failed at archive offset " + std::to_string(res.written));
    return 0;
}

extern "C" int b200z_compress_seekable_stream(b200z_ctx *c, b200z_read_fn rd, void *ru, b200z_write_fn wr, void *wu, size_t frame_size, int level,
                                              int checksum, const b200z_dict *dict, b200z_seekable_stream_result *result) {
    // ---- everything is checked before any read, write or launch
    if (int e = compress_check(c, level, B200Z_WINDOW_LOG_MIN, dict)) return e;
    if (!rd || !wr) { c->err = "invalid argument"; return B200Z_ERR_INVALID_ARGUMENT; }
    if (!frame_size || frame_size > B200Z_SEEKABLE_MAX_FRAME_SIZE) { c->err = "frame_size must lie in [1, 2^30]"; return B200Z_ERR_INVALID_ARGUMENT; }
    b200z_seekable_stream_result res{};
    const int e = seek_stream(c, rd, ru, wr, wu, frame_size, level, checksum != 0, dict, res);
    if (result) *result = res;
    return e;
}

// The table of an archive, parsed and checked: the footer (the archive's last 9 bytes) first, then the table frame in front of it
namespace {
struct SeekTable {
    uint64_t n = 0, len = 0;          // frames, archive bytes
    bool checksum = false;
    std::vector<uint64_t> coff, doff;   // n + 1 prefix sums of Compressed_Size / Decompressed_Size
    std::vector<uint32_t> csum;
};
}  // namespace

static int seek_fail(std::string *why, const char *rule) {
    if (why) *why = std::string("seek table: ") + rule;
    return B200Z_ERR_SEEKABLE_TABLE;
}
// the footer: n, the checksum flag, and the size of the table frame (checked to lie inside the archive)
static int seek_footer(const uint8_t *ft, uint64_t len, SeekTable &t, uint64_t *table_bytes, std::string *why) {
    if (len < SEEK_TABLE_FIXED) return seek_fail(why, "the archive is shorter than a seek table (17 bytes)");
    if (rd32le(ft + 5) != SEEK_FOOTER_MAGIC) return seek_fail(why, "Seekable_Magic_Number is not 0x8F92EAB1");
    if (ft[4] & 0x7c) return seek_fail(why, "Seek_Table_Descriptor's reserved bits (6-2) are not 0");
    t.len = len; t.n = rd32le(ft); t.checksum = (ft[4] & 0x80) != 0;
    *table_bytes = seek_table_size(t.n, t.checksum);
    if (*table_bytes > len) return seek_fail(why, "Number_Of_Frames gives a table larger than the archive");
    return 0;
}
// the table frame (table_bytes of it, the footer included): its header and the entries, whose Compressed_Size must add up to its offset
// the table frame's 8-byte header, against the footer's Number_Of_Frames and flag (Frame_Size is a u32, so this bounds the table)
static int seek_table_header(const uint8_t *p, const SeekTable &t, std::string *why) {
    if (rd32le(p) != SEEK_SKIPPABLE_MAGIC) return seek_fail(why, "the table frame's Skippable_Magic_Number is not 0x184D2A5E");
    if (rd32le(p + 4) != t.n * (t.checksum ? 12 : 8) + SEEK_FOOTER) return seek_fail(why, "Frame_Size is not Number_Of_Frames * (8 or 12) + 9");
    return 0;
}
static int seek_entries(const uint8_t *p, SeekTable &t, std::string *why) {
    const uint64_t esz = t.checksum ? 12 : 8, tb = seek_table_size(t.n, t.checksum);
    if (int e = seek_table_header(p, t, why)) return e;
    t.coff.assign(t.n + 1, 0); t.doff.assign(t.n + 1, 0); t.csum.assign(t.checksum ? t.n : 0, 0);
    for (uint64_t i = 0; i < t.n; i++) {
        const uint8_t *e = p + 8 + i * esz;
        t.coff[i + 1] = t.coff[i] + rd32le(e);
        t.doff[i + 1] = t.doff[i] + rd32le(e + 4);
        if (t.checksum) t.csum[i] = rd32le(e + 8);
    }
    if (t.coff[t.n] != t.len - tb) return seek_fail(why, "the frames' Compressed_Size do not add up to the table frame's offset");
    return 0;
}
static int seek_parse_host(const uint8_t *archive, uint64_t len, SeekTable &t, std::string *why) {
    uint64_t tb = 0;
    if (int e = seek_footer(len >= SEEK_FOOTER ? archive + len - SEEK_FOOTER : archive, len, t, &tb, why)) return e;
    return seek_entries(archive + len - tb, t, why);
}

// The read plan.  Every range is checked first (content and output reach, overlapping output slots); then the frames a range wholly
// contains are decoded in place for the first such range, the other touched frames into scratch, and each range's remaining bytes
// become copy pieces.  `touched[r]`: the frames range r touches, ascending.
namespace {
struct SeekPlan {
    std::vector<b200z_seek_plan_frame> frames;
    std::vector<b200z_seek_plan_piece> pieces;
    std::vector<std::vector<uint64_t>> touched;
    uint64_t scratch = 0;
};
}  // namespace

static int seek_plan(const SeekTable &t, const b200z_range *ranges, size_t n, uint64_t output_cap, SeekPlan &p, std::string *why) {
    const uint64_t content = t.doff[t.n];
    std::vector<std::pair<uint64_t, uint64_t>> slots;
    for (size_t r = 0; r < n; r++) {
        const b200z_range &g = ranges[r];
        if (g.offset > content || g.length > content - g.offset || g.out_off > output_cap || g.length > output_cap - g.out_off) {
            if (why) *why = "range " + std::to_string(r) + " reaches past the content size or the output";
            return B200Z_ERR_INVALID_ARGUMENT;
        }
        if (g.length) slots.push_back({g.out_off, g.length});
    }
    std::sort(slots.begin(), slots.end());
    for (size_t i = 1; i < slots.size(); i++)
        if (slots[i - 1].first + slots[i - 1].second > slots[i].first) {
            if (why) *why = "ranges overlap in the output";
            return B200Z_ERR_INVALID_ARGUMENT;
        }
    p.frames.clear(); p.pieces.clear(); p.scratch = 0;
    p.touched.assign(n, {});
    std::map<uint64_t, int64_t> in_place;   // touched frame -> the range it is decoded in place for, or -1
    for (size_t r = 0; r < n; r++) {
        const uint64_t lo = ranges[r].offset, hi = lo + ranges[r].length;
        if (lo == hi) continue;
        // the first frame holding byte lo: the last one starting at or before it (frames of 0 bytes start where the next one does)
        uint64_t f = (uint64_t)(std::upper_bound(t.doff.begin(), t.doff.end(), lo) - t.doff.begin()) - 1;
        for (; f < t.n && t.doff[f] < hi; f++) {
            if (t.doff[f + 1] == t.doff[f]) continue;
            p.touched[r].push_back(f);
            const bool whole = t.doff[f] >= lo && t.doff[f + 1] <= hi;
            auto it = in_place.find(f);
            if (it == in_place.end()) in_place[f] = whole ? (int64_t)r : -1;
            else if (whole && it->second < 0) it->second = (int64_t)r;
        }
    }
    std::map<uint64_t, uint64_t> at;   // frame -> where its plaintext starts (output or scratch)
    for (const auto &kv : in_place) {
        const uint64_t f = kv.first;
        uint64_t dst;
        if (kv.second >= 0) {
            const b200z_range &g = ranges[kv.second];
            dst = g.out_off + (t.doff[f] - g.offset);
        } else {
            dst = p.scratch;
            p.scratch = (p.scratch + (t.doff[f + 1] - t.doff[f]) + 15) & ~15ull;
        }
        at[f] = dst;
        p.frames.push_back(b200z_seek_plan_frame{f, dst, kv.second});
    }
    for (size_t r = 0; r < n; r++) {
        const b200z_range &g = ranges[r];
        for (uint64_t f : p.touched[r]) {
            const int64_t owner = in_place[f];
            if (owner == (int64_t)r) continue;
            const uint64_t lo = std::max(g.offset, t.doff[f]), hi = std::min(g.offset + g.length, t.doff[f + 1]);
            p.pieces.push_back(b200z_seek_plan_piece{g.out_off + (lo - g.offset), at[f] + (lo - t.doff[f]), hi - lo, owner < 0 ? 1u : 0u, (uint32_t)r});
        }
    }
    return 0;
}

extern "C" int b200z_debug_seekable_plan(const uint8_t *archive, size_t len, const b200z_range *ranges, size_t n, b200z_seek_plan_frame *frames,
                                         size_t frames_cap, size_t *nframes, b200z_seek_plan_piece *pieces, size_t pieces_cap, size_t *npieces,
                                         uint64_t *scratch_bytes) {
    if ((!archive && len) || (!ranges && n) || !nframes || !npieces || !scratch_bytes) return B200Z_ERR_INVALID_ARGUMENT;
    SeekTable t;
    if (int e = seek_parse_host(archive, len, t, nullptr)) return e;
    SeekPlan p;
    if (int e = seek_plan(t, ranges, n, UINT64_MAX, p, nullptr)) return e;
    *nframes = p.frames.size(); *npieces = p.pieces.size(); *scratch_bytes = p.scratch;
    if (p.frames.size() > frames_cap || p.pieces.size() > pieces_cap) return B200Z_ERR_INVALID_ARGUMENT;
    if (!p.frames.empty()) memcpy(frames, p.frames.data(), p.frames.size() * sizeof(b200z_seek_plan_frame));
    if (!p.pieces.empty()) memcpy(pieces, p.pieces.data(), p.pieces.size() * sizeof(b200z_seek_plan_piece));
    return 0;
}

struct b200z_seekable {
    b200z_ctx *ctx = nullptr;
    const uint8_t *archive = nullptr;   // borrowed; null behind read_at
    int mem = B200Z_MEM_HOST;           // a host archive, or one behind read_at
    b200z_read_at_fn read_at = nullptr;
    void *user = nullptr;
    SeekTable t;
};

// an archive that is not in host memory: only the footer, then the table frame, are fetched to the host, by fetch(offset, buf, len).
// The table frame's header is fetched and checked first, so that a corrupt Number_Of_Frames fails before a table of its size is
// allocated or read; a table that still does not fit in host memory is B200Z_ERR_OUT_OF_MEMORY.
template <class Fetch>
static int seek_parse_fetched(uint64_t len, Fetch fetch, SeekTable &t, std::string *why) {
    uint8_t ft[SEEK_FOOTER] = {}, hd[8] = {};
    if (len >= SEEK_FOOTER)
        if (int e = fetch(len - SEEK_FOOTER, ft, (uint64_t)SEEK_FOOTER)) return e;
    uint64_t tb = 0;
    if (int e = seek_footer(ft, len, t, &tb, why)) return e;
    if (int e = fetch(len - tb, hd, (uint64_t)sizeof hd)) return e;
    if (int e = seek_table_header(hd, t, why)) return e;
    try {
        std::vector<uint8_t> tab(tb);
        if (int e = fetch(len - tb, tab.data(), tb)) return e;
        return seek_entries(tab.data(), t, why);
    } catch (const std::bad_alloc &) {
        if (why) *why = "seek table: " + std::to_string(t.n) + " frames do not fit in host memory";
        return B200Z_ERR_OUT_OF_MEMORY;
    }
}

// len bytes at archive offset `at` through read_at, partial reads retried until one returns 0
static int seek_read_at(const b200z_seekable *s, uint64_t at, uint8_t *buf, uint64_t len) {
    for (uint64_t got = 0; got < len;) {
        const long r = s->read_at(s->user, at + got, buf + got, len - got);
        if (r < 0 || (uint64_t)r > len - got) return seek_io(s->ctx, "read_at failed at archive offset " + std::to_string(at + got));
        if (r == 0)
            return seek_io(s->ctx, "read_at came up short at archive offset " + std::to_string(at + got) + ": " + std::to_string(got) + " of " +
                                       std::to_string(len) + " bytes from offset " + std::to_string(at));
        got += (uint64_t)r;
    }
    return 0;
}

extern "C" int b200z_seekable_open(b200z_ctx *c, const uint8_t *archive, size_t len, int mem, b200z_seekable **out) {
    if (!c || !out || (!archive && len) || (mem != B200Z_MEM_HOST && mem != B200Z_MEM_DEVICE)) return B200Z_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    std::unique_ptr<b200z_seekable> s(new b200z_seekable());
    s->ctx = c; s->archive = archive; s->mem = mem;
    if (mem == B200Z_MEM_HOST) {
        if (int e = seek_parse_host(archive, len, s->t, &c->err)) return e;
    } else {
        if (int e = c->use()) return e;
        const auto fetch = [&](uint64_t at, uint8_t *buf, uint64_t n) -> int {
            CU(c, cudaMemcpy(buf, archive + at, n, cudaMemcpyDeviceToHost));
            return 0;
        };
        if (int e = seek_parse_fetched(len, fetch, s->t, &c->err)) return e;
    }
    *out = s.release();
    return 0;
}
extern "C" int b200z_seekable_open_source(b200z_ctx *c, b200z_read_at_fn read_at, void *user, uint64_t len, b200z_seekable **out) {
    if (!c || !out || !read_at) return B200Z_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    std::unique_ptr<b200z_seekable> s(new b200z_seekable());
    s->ctx = c; s->read_at = read_at; s->user = user;
    const auto fetch = [&](uint64_t at, uint8_t *buf, uint64_t n) { return seek_read_at(s.get(), at, buf, n); };
    if (int e = seek_parse_fetched(len, fetch, s->t, &c->err)) return e;
    *out = s.release();
    return 0;
}
extern "C" uint64_t b200z_seekable_num_frames(const b200z_seekable *s) { return s ? s->t.n : 0; }
extern "C" uint64_t b200z_seekable_content_size(const b200z_seekable *s) { return s ? s->t.doff[s->t.n] : 0; }
extern "C" int b200z_seekable_frame(const b200z_seekable *s, uint64_t i, b200z_seek_frame *out) {
    if (!s || !out || i >= s->t.n) return B200Z_ERR_INVALID_ARGUMENT;
    const SeekTable &t = s->t;
    *out = b200z_seek_frame{t.coff[i], t.coff[i + 1] - t.coff[i], t.doff[i], t.doff[i + 1] - t.doff[i], t.checksum ? 1u : 0u, t.checksum ? t.csum[i] : 0u};
    return 0;
}
extern "C" void b200z_seekable_close(b200z_seekable *s) { delete s; }

extern "C" int b200z_seekable_read_ranges(b200z_seekable *s, const b200z_range *ranges, size_t n, const b200z_dict *const *dicts, size_t ndicts,
                                          const b200z_dict *forced_dict, uint64_t max_window_size, uint8_t *output, size_t output_cap, int output_mem,
                                          b200z_range_result *results) {
    if (!s || (!ranges && n) || (n && !results) || (!dicts && ndicts) || (output_cap && !output) ||
        (output_mem != B200Z_MEM_HOST && output_mem != B200Z_MEM_DEVICE))
        return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = s->ctx;
    const SeekTable &t = s->t;
    SeekPlan p;
    if (int e = seek_plan(t, ranges, n, output_cap, p, &c->err)) return e;
    for (size_t r = 0; r < n; r++) results[r] = b200z_range_result{0, 0, -1, (uint64_t)p.touched[r].size(), 0};
    if (p.frames.empty()) return 0;
    if (int e = c->use()) return e;
    CompressResources *rp = nullptr;
    if (int e = compress_get(c, &rp)) return e;
    CompressResources &res = *rp;
    cudaStream_t st = c->stream;
    // Host output: the slots are staged on the device packed in call order, so the plan runs on ranges whose out_off is the packed
    // one; the scratch follows them.  Device output: the scratch is a buffer of its own.
    const bool host_out = output_mem == B200Z_MEM_HOST;
    std::vector<b200z_range> packed;
    uint64_t staged = 0;
    if (host_out) {
        packed.assign(ranges, ranges + n);
        for (b200z_range &g : packed) { g.out_off = staged; staged += g.length; }
        staged = (staged + 15) & ~15ull;
        if (int e = seek_plan(t, packed.data(), n, UINT64_MAX, p, &c->err)) return e;
    }
    if (int e = res.rd_stage.ensure(staged + p.scratch + 16)) return e;
    uint8_t *scratch = res.rd_stage.as<uint8_t>() + staged;
    uint8_t *out_dev = host_out ? res.rd_stage.as<uint8_t>() : output;
    // The batch writes every frame at base + out_off.  Slots and scratch may be two allocations: base is the lower of the two and
    // out_off a distance in the one (unified) device address space; each frame writes only [out_off, out_off + its size).
    const uint64_t out_end = host_out ? staged : output_cap;
    uint8_t *base = std::min(out_dev, scratch);
    const uint64_t o_out = (uint64_t)(out_dev - base), o_scr = (uint64_t)(scratch - base);
    const uint64_t span = std::max(o_out + out_end, o_scr + p.scratch + 16);
    // the touched frames as b200z_frame_io: host archives gather their bytes, device archives are read where they lie
    std::vector<b200z_frame_io> io(p.frames.size());
    uint64_t gathered = 0;
    for (size_t i = 0; i < p.frames.size(); i++) {
        const uint64_t f = p.frames[i].frame, cs = t.coff[f + 1] - t.coff[f], ds = t.doff[f + 1] - t.doff[f];
        io[i].src_off = s->mem == B200Z_MEM_HOST ? gathered : t.coff[f];
        io[i].src_size = cs;
        io[i].out_off = (p.frames[i].range >= 0 ? o_out : o_scr) + p.frames[i].dst_off;
        io[i].out_cap = ds;
        gathered += cs;
    }
    const uint8_t *src = s->archive;
    size_t src_len = t.len;
    // the pinned buffer holds a host archive's gathered frames, then host output's staged slots: sized for both uses it has
    const bool host_arch = s->mem == B200Z_MEM_HOST;
    if (host_arch || host_out)
        if (int e = res.rd_host.ensure(std::max<uint64_t>(host_arch ? gathered : 0, staged) + 16)) return e;
    if (host_arch) {
        uint8_t *h = res.rd_host.as<uint8_t>();
        if (s->read_at) {   // one read_at per run of touched frames adjacent in the archive: they are adjacent in h too
            for (size_t i = 0, j; i < p.frames.size(); i = j) {
                const uint64_t at = t.coff[p.frames[i].frame];
                uint64_t len = io[i].src_size;
                for (j = i + 1; j < p.frames.size() && t.coff[p.frames[j].frame] == at + len; j++) len += io[j].src_size;
                if (int e = seek_read_at(s, at, h + io[i].src_off, len)) return e;
            }
        } else {
            for (size_t i = 0; i < p.frames.size(); i++) memcpy(h + io[i].src_off, s->archive + t.coff[p.frames[i].frame], io[i].src_size);
        }
        src = h; src_len = gathered;
    }
    b200z_batch *bp = nullptr;
    if (int e = b200z_batch_prepare(c, src, src_len, s->mem, io.data(), io.size(), dicts, ndicts, forced_dict, max_window_size, &bp)) return e;
    std::unique_ptr<b200z_batch, void (*)(b200z_batch *)> b(bp, b200z_batch_destroy);
    if (int e = b200z_batch_run(b.get(), base, span)) return e;
    // the copy pieces, cut to GATHER_CHUNK bytes each
    std::vector<GatherPiece> gp;
    for (const b200z_seek_plan_piece &q : p.pieces) {
        const uint64_t so = (q.from_scratch ? o_scr : o_out) + q.src_off, d = o_out + q.dst_off;
        for (uint64_t k = 0; k < q.len; k += GATHER_CHUNK)
            gp.push_back(GatherPiece{so + k, d + k, (uint32_t)std::min<uint64_t>(GATHER_CHUNK, q.len - k), 0});
    }
    if (!gp.empty()) {
        if (int e = res.rd_pieces.ensure(gp.size() * sizeof(GatherPiece))) return e;
        CU(c, cudaMemcpyAsync(res.rd_pieces.p, gp.data(), gp.size() * sizeof(GatherPiece), cudaMemcpyHostToDevice, st));
        if (int le = launch_range_gather(res.rd_pieces.as<GatherPiece>(), (uint32_t)gp.size(), base, st, &c->launches))
            return c->set_cuda_err((cudaError_t)le, "k_range_gather");
    }
    std::vector<b200z_frame_result> fr(io.size());
    if (int e = b200z_batch_finish(b.get(), fr.data())) return e;   // synchronises (and keeps `gp` alive until the copy is done)
    if (host_out) {
        uint8_t *h = res.rd_host.as<uint8_t>();
        CU(c, cudaMemcpy(h, res.rd_stage.p, staged, cudaMemcpyDeviceToHost));
        for (size_t r = 0; r < n; r++) memcpy(output + ranges[r].out_off, h + packed[r].out_off, ranges[r].length);
    }
    // per range: the first failing frame in content order, and the checksum comparisons
    std::map<uint64_t, size_t> idx;
    for (size_t i = 0; i < p.frames.size(); i++) idx[p.frames[i].frame] = i;
    const bool sums = (c->flags & B200Z_FLAG_CHECKSUM) != 0;
    for (size_t r = 0; r < n; r++) {
        b200z_range_result &rr = results[r];
        for (uint64_t f : p.touched[r]) {
            const b200z_frame_result &x = fr[idx[f]];
            const uint64_t ds = t.doff[f + 1] - t.doff[f];
            if (rr.status == 0 && (x.status || x.out_size != ds)) {
                const bool size = x.status == 0 || x.status == B200Z_ERR_TARGET_TOO_SMALL;   // out_cap is the entry's size
                rr.status = size ? B200Z_ERR_SEEKABLE_FRAME_SIZE : x.status;
                rr.stage = size ? B200Z_STAGE_NONE : x.stage;
                rr.error_frame = (int64_t)f;
            }
            if (sums && x.status == 0 && x.has_calculated_checksum &&
                ((t.checksum && x.calculated_checksum != t.csum[f]) || (x.has_checksum && x.calculated_checksum != x.checksum_from_data)))
                rr.checksum_mismatches++;
        }
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// stream compressor (FrameCompressor, frame_compressor.rs:75-276): the source is read into chunks of whole 128 KiB blocks and
// the frame is written chunk by chunk.  Uncompressed frames the blocks on the host.  Fastest (or LAZY) runs k_cmatch -> k_cenc ->
// k_cassemble<true> on each chunk on the ctx stream, uploads on one copy stream and downloads on another, while the calling
// thread reads and hashes the next chunk and writes the previous one (the pattern of decode_frames_pipelined).
// ---------------------------------------------------------------------------------------------------------------
namespace {
constexpr size_t FC_HEADER = 6;       // magic, FHD, Window_Descriptor
constexpr size_t FC_HDR_ROOM = 16;    // in front of a chunk's blocks in its output buffer: the first chunk's header goes there
constexpr size_t FC_TRAILER = 3 + 4;  // after them in the last chunk: the empty last block and the checksum
}  // namespace

struct b200z_frame_compressor {
    b200z_ctx *ctx = nullptr;
    int device = 0;
    int level = B200Z_LEVEL_FASTEST;
    bool checksum = true;
    uint32_t window_log = B200Z_WINDOW_LOG_MIN;
    uint64_t chunk = 64ull << 20;   // bytes per chunk, a multiple of ENC_BLOCK
    std::vector<uint8_t> raw;       // Uncompressed: one chunk's part of the frame
    // Fastest, allocated by its first compress (b200z_frame_compressor_free synchronises the copy streams before any of these is
    // released).  desc: the chunk's CFrame, its CBlocks, its long-match spans, then its b200z_compress_result; d_in: the last
    // `hist` bytes before the chunk (ENC_WINDOW, or 2^window_log + LDM_MARGIN with long matches), then the chunk
    PipeSlots p;
    CompressStaging stage;                    // shared: the kernels run in order on one stream
    LdmBufs ldm;                              // shared, sized for the density bound of the spans
    FarBufs far;                              // ULTRA, shared: sized for a chunk and the 2^window_log bytes before it
    std::vector<FPiece> far_pieces;           // ULTRA: the chunk's pieces and blocks, uploaded on the kernel stream
    std::vector<FBlock> far_blocks;
    uint64_t hist = 0;                        // what the buffers were prepared for (0: not yet)
    uint32_t chunk_blocks() const { return (uint32_t)(chunk / ENC_BLOCK); }
    uint64_t hist_for(uint32_t wl) const { return wl > B200Z_WINDOW_LOG_MIN ? (1ull << wl) + LDM_MARGIN : ENC_WINDOW; }
    uint32_t max_spans() const { return (uint32_t)((hist + ENC_BLOCK - 1) / ENC_BLOCK) + chunk_blocks(); }
    size_t chunk_bound() const { return chunk + 3ull * chunk_blocks(); }   // the chunk's blocks, packed, at most
    size_t span_off() const { return sizeof(CFrame) + (size_t)chunk_blocks() * sizeof(CBlock); }
    size_t res_off() const { return span_off() + (hist > ENC_WINDOW ? (size_t)max_spans() * sizeof(LSpan) : 0); }
    size_t desc_bytes() const { return res_off() + sizeof(b200z_compress_result); }
};

static int fc_valid_level(int level) {   // Uncompressed .. Best, LAZY, OPT, ULTRA
    return (level >= 0 && level <= 4) || level == B200Z_LEVEL_LAZY || level == B200Z_LEVEL_OPT || level == B200Z_LEVEL_ULTRA;
}
static int fc_panic(b200z_ctx *c, const char *what) { c->err = what; return B200Z_ERR_REFERENCE_WOULD_PANIC; }

extern "C" int b200z_frame_compressor_new(b200z_ctx *c, int level, int checksum, b200z_frame_compressor **out) {
    if (!out) return B200Z_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    if (!c || !fc_valid_level(level)) return B200Z_ERR_INVALID_ARGUMENT;
    std::unique_ptr<b200z_frame_compressor> fc(new b200z_frame_compressor());
    fc->ctx = c;
    fc->device = c->device;
    fc->level = level;
    fc->checksum = checksum != 0;
    if (const char *ev = getenv("B200Z_PIPELINE_CHUNK_BYTES"))
        fc->chunk = std::max<uint64_t>(ENC_BLOCK, strtoull(ev, nullptr, 10) / ENC_BLOCK * ENC_BLOCK);
    *out = fc.release();
    return 0;
}
extern "C" void b200z_frame_compressor_free(b200z_frame_compressor *fc) {
    if (!fc) return;
    if (fc->hist) {
        cudaSetDevice(fc->device);
        fc->p.drain(nullptr);
    }
    delete fc;
}
extern "C" int b200z_frame_compressor_set_compression_level(b200z_frame_compressor *fc, int level) {
    if (!fc || !fc_valid_level(level)) return B200Z_ERR_INVALID_ARGUMENT;
    fc->level = level;
    return 0;
}
extern "C" int b200z_frame_compressor_compression_level(const b200z_frame_compressor *fc) { return fc ? fc->level : B200Z_LEVEL_FASTEST; }
extern "C" int b200z_frame_compressor_set_window_log(b200z_frame_compressor *fc, int window_log) {
    if (!fc || window_log < B200Z_WINDOW_LOG_MIN || window_log > B200Z_WINDOW_LOG_MAX) return B200Z_ERR_INVALID_ARGUMENT;
    fc->window_log = (uint32_t)window_log;
    return 0;
}
extern "C" int b200z_frame_compressor_window_log(const b200z_frame_compressor *fc) { return fc ? (int)fc->window_log : B200Z_WINDOW_LOG_MIN; }

static void fc_le(uint8_t *p, uint64_t v, int n) { for (int i = 0; i < n; i++) p[i] = (uint8_t)(v >> (8 * i)); }
// the frame header (frame_compressor.rs:144-151): no Frame_Content_Size, Single_Segment 0, a 2^window_log window (128 KiB by default)
static void fc_header(uint8_t *dst, bool checksum, uint32_t window_log) {
    fc_le(dst, 0xFD2FB528u, 4);
    dst[4] = checksum ? 0x04 : 0x00;
    dst[5] = (uint8_t)((window_log - 10) << 3);
}
// the end of the frame after its last chunk: the empty last Raw block when the source ended on a block boundary (the reference's
// uncompressed_data.is_empty() branch, :175-186), then the checksum (:215-223).  Returns the bytes written at dst.
static size_t fc_trailer(uint8_t *dst, bool empty_block, bool checksum, const XXH64State &h, b200z_compress_result &r) {
    size_t len = 0;
    if (empty_block) { fc_le(dst, 1, 3); len = 3; r.blocks++; r.raw_blocks++; }
    if (checksum) {
        r.has_checksum = 1;
        r.checksum = (uint32_t)h.digest();
        fc_le(dst + len, r.checksum, 4);
        len += 4;
    }
    return len;
}

// Uncompressed: Raw blocks read straight into place behind their headers, one chunk of them per write
static int fc_compress_raw(b200z_frame_compressor *fc, b200z_read_fn rd, void *ru, b200z_write_fn wr, void *wu, XXH64State &h,
                           b200z_compress_result &r) {
    b200z_ctx *c = fc->ctx;
    const uint32_t nb = fc->chunk_blocks();
    fc->raw.resize(FC_HDR_ROOM + (size_t)nb * (3 + ENC_BLOCK) + FC_TRAILER);
    uint8_t *const body = fc->raw.data() + FC_HDR_ROOM;
    for (uint64_t k = 0;; k++) {
        size_t len = 0, n = 0;
        bool eof = false;
        for (uint32_t i = 0; i < nb && !eof; i++) {
            if (!read_chunk(rd, ru, body + len + 3, ENC_BLOCK, &n, &eof)) return fc_panic(c, "FrameCompressor::compress: the source's read failed");
            if (n == 0) break;   // the source ended on a block boundary: the trailer's empty block is the last
            h.update(body + len + 3, n);
            fc_le(body + len, (eof ? 1u : 0u) | ((uint32_t)n << 3), 3);
            len += 3 + n;
            r.blocks++;
            r.raw_blocks++;
        }
        uint8_t *start = body;
        if (k == 0) { start -= FC_HEADER; fc_header(start, fc->checksum, B200Z_WINDOW_LOG_MIN); }
        if (eof) len += fc_trailer(body + len, n == 0, fc->checksum, h, r);
        const size_t w = (size_t)(body + len - start);
        if (!write_all(wr, wu, start, w, nullptr)) return fc_panic(c, "FrameCompressor::compress: the drain's write failed");
        r.dst_size += w;
        if (eof) return 0;
    }
}

// the buffers for the compressor's window_log: kept while a later compress needs no more history
static int fc_prepare(b200z_frame_compressor *fc) {
    if (fc->hist >= fc->hist_for(fc->window_log)) return 0;
    b200z_ctx *c = fc->ctx;
    fc->hist = fc->hist_for(fc->window_log);
    const size_t C = fc->chunk, nb = fc->chunk_blocks(), bound = fc->chunk_bound();
    if (fc->p.create(c)) return B200Z_ERR_CUDA;
    int e = fc->p.ensure(fc->hist + C + 16, C, bound + 16, FC_HDR_ROOM + bound + FC_TRAILER, fc->desc_bytes());
    if (!e) e = fc->stage.ensure(nb, false);
    if (!e && fc->hist > ENC_WINDOW) {
        const uint32_t ns = fc->max_spans();
        if (!(e = fc->ldm.ensure(ns * LDM_SPAN_CAP, false)) && !(e = fc->ldm.tcount.ensure((size_t)ns * LDM_THREADS * 4, false)) &&
            !(e = fc->ldm.scount.ensure((ns + 1) * 4, false)) &&
            !(e = fc->ldm.off.ensure(nb * 4, false)))
            e = fc->ldm.cnt.ensure(nb * 4, false);
    }
    if (e) {
        fc->hist = 0;
        c->err = "FrameCompressor: out of memory for chunks of " + std::to_string(C) + " bytes";
        return e;
    }
    return 0;
}

// Fastest: chunk k (slot s = k & 1) is read into h_in[s] and hashed, uploaded behind the previous chunk's last `hist` bytes
// (for matches that reach back), compressed, downloaded to h_out[s] with its result and written (PipeSlots::run).
static int fc_compress_fast(b200z_frame_compressor *fc, b200z_read_fn rd, void *ru, b200z_write_fn wr, void *wu, XXH64State &h,
                            b200z_compress_result &r) {
    b200z_ctx *c = fc->ctx;
    if (int e = fc_prepare(fc)) return e;
    if (int e = fc->stage.ensure(fc->chunk_blocks(), false, fc->level)) return e;   // OPT's chain slots, whenever the level became OPT
    const uint64_t C = fc->chunk, H = fc->hist_for(fc->window_log), Wf = 1ull << fc->window_log;
    const bool ultra = fc->level == B200Z_LEVEL_ULTRA && fc->window_log > B200Z_WINDOW_LOG_MIN;
    if (ultra) {   // a chunk and the Wf bytes before it, whenever the level became ULTRA
        const uint64_t v = Wf + C;
        if (int e = fc->far.ensure(v, v, Wf / ENC_BLOCK + fc->chunk_blocks(), fc->chunk_blocks(), false)) {
            c->err = "FrameCompressor: out of memory for ULTRA's far stage";
            return e;
        }
    }
    cudaStream_t ks = c->stream;
    auto enqueue = [&](uint64_t k, int s, size_t n) -> int {
        CFrame *hf = fc->p.h_desc[s].as<CFrame>();
        CBlock *hb = reinterpret_cast<CBlock *>(hf + 1);
        *hf = plan_frame(H, n, 0, k * C, 0, 0, hb);
        const uint32_t m = hf->nblocks;
        // long matches: the kept history (from the frame's start while it is shorter than H) and the chunk's blocks, as spans of at
        // most one block in position order; none until the frame has more than one block
        const uint64_t vlo = k * C >= H ? 0 : H - k * C;
        LSpan *hs = reinterpret_cast<LSpan *>(fc->p.h_desc[s].as<uint8_t>() + fc->span_off());
        uint32_t ns = 0;
        if (H > ENC_WINDOW && k * C + n > ENC_BLOCK) {
            for (uint64_t o = vlo; o < H; o += ENC_BLOCK) hs[ns++] = LSpan{o, vlo, (uint32_t)std::min<uint64_t>(ENC_BLOCK, H - o), 0, LDM_NO_BLOCK, 0};
            for (uint32_t i = 0; i < m; i++) hs[ns++] = LSpan{hb[i].src_off, vlo, hb[i].size, 0, i, 0};
        }
        uint8_t *din = fc->p.d_in[s].as<uint8_t>();
        CU(c, cudaStreamWaitEvent(fc->p.s_h2d, fc->p.ev_k[s], 0));   // chunk k - 2's kernels are done with d_in[s] and d_desc[s]
        if (k) CU(c, cudaMemcpyAsync(din, fc->p.d_in[s ^ 1].as<uint8_t>() + C, H, cudaMemcpyDeviceToDevice, fc->p.s_h2d));
        CU(c, cudaMemcpyAsync(din + H, fc->p.h_in[s].p, n, cudaMemcpyHostToDevice, fc->p.s_h2d));
        CU(c, cudaMemcpyAsync(fc->p.d_desc[s].p, hf, sizeof(CFrame) + m * sizeof(CBlock), cudaMemcpyHostToDevice, fc->p.s_h2d));
        if (ns) CU(c, cudaMemcpyAsync(fc->p.d_desc[s].as<uint8_t>() + fc->span_off(), hs, ns * sizeof(LSpan), cudaMemcpyHostToDevice, fc->p.s_h2d));
        CU(c, cudaEventRecord(fc->p.ev_h2d[s], fc->p.s_h2d));
        CU(c, cudaStreamWaitEvent(ks, fc->p.ev_h2d[s], 0));
        CompressArgs a{};
        a.frames = fc->p.d_desc[s].as<CFrame>();
        a.blocks = reinterpret_cast<const CBlock *>(a.frames + 1);
        a.results = reinterpret_cast<b200z_compress_result *>(fc->p.d_desc[s].as<uint8_t>() + fc->res_off());
        a.input = din; a.output = fc->p.d_out[s].as<uint8_t>();
        fc->stage.bind(a);
        a.nframes = 1; a.nblocks = m; a.level = fc->level;   // Fastest, LAZY or OPT
        if (ns)
            if (int le = compress_ldm(c, fc->ldm, a, reinterpret_cast<const LSpan *>(fc->p.d_desc[s].as<uint8_t>() + fc->span_off()), ns, m,
                                      fc->window_log, ns * LDM_SPAN_CAP, ks))
                return le;
        if (ultra && ns) {   // ULTRA's far stage over the last min(k * C, Wf) bytes of the frame and the chunk: one group
            std::vector<FPiece> &pc = fc->far_pieces;
            std::vector<FBlock> &fb = fc->far_blocks;
            pc.clear(); fb.clear();
            const uint64_t hl = std::min(k * C, Wf);
            uint64_t vbase = 0, pbase = 0;
            for (uint64_t o = H - hl; o < H; o += ENC_BLOCK) far_piece(pc, o, ENC_BLOCK, vbase, pbase);
            for (uint32_t i = 0; i < m; i++) {
                fb.push_back(FBlock{(uint32_t)vbase, (uint32_t)std::min(k * C + (uint64_t)i * ENC_BLOCK, Wf), (uint32_t)Wf, 0});
                far_piece(pc, hb[i].src_off, hb[i].size, vbase, pbase);
            }
            CU(c, cudaMemcpyAsync(fc->far.pieces.p, pc.data(), pc.size() * sizeof(FPiece), cudaMemcpyHostToDevice, ks));
            CU(c, cudaMemcpyAsync(fc->far.fblk.p, fb.data(), fb.size() * sizeof(FBlock), cudaMemcpyHostToDevice, ks));
            if (int le = launch_far_stage(fc->far.args(din, fc->far.pieces.as<FPiece>(), (uint32_t)pc.size(), (uint32_t)pbase), ks, &c->launches))
                return c->set_cuda_err((cudaError_t)le, "k_fkey / k_fstart");
            fc->far.bind(a, fc->far.fblk.as<FBlock>());
        }
        if (int le = launch_compress_chunk(a, ks, &c->launches)) return c->set_cuda_err((cudaError_t)le, "k_cmatch / k_cenc / k_cassemble<true>");
        CU(c, cudaEventRecord(fc->p.ev_k[s], ks));
        CU(c, cudaStreamWaitEvent(fc->p.s_d2h, fc->p.ev_k[s], 0));
        CU(c, cudaMemcpyAsync(fc->p.h_desc[s].as<uint8_t>() + fc->res_off(), a.results, sizeof(b200z_compress_result), cudaMemcpyDeviceToHost, fc->p.s_d2h));
        CU(c, cudaMemcpyAsync(fc->p.h_out[s].as<uint8_t>() + FC_HDR_ROOM, a.output, n + 3ull * m, cudaMemcpyDeviceToHost, fc->p.s_d2h));
        CU(c, cudaEventRecord(fc->p.ev_d2h[s], fc->p.s_d2h));
        return 0;
    };
    auto read = [&](int s, size_t &n, bool &eof) -> int {
        if (!read_chunk(rd, ru, fc->p.h_in[s].as<uint8_t>(), C, &n, &eof)) return fc_panic(c, "FrameCompressor::compress: the source's read failed");
        h.update(fc->p.h_in[s].as<uint8_t>(), n);
        return 0;
    };
    auto write = [&](uint64_t k, int s, size_t n, bool final) -> int {
        uint8_t *const body = fc->p.h_out[s].as<uint8_t>() + FC_HDR_ROOM;
        size_t len = 0;
        if (n) {
            CU(c, cudaEventSynchronize(fc->p.ev_d2h[s]));
            const b200z_compress_result &cr = *reinterpret_cast<const b200z_compress_result *>(fc->p.h_desc[s].as<uint8_t>() + fc->res_off());
            len = cr.dst_size;
            r.blocks += cr.blocks; r.raw_blocks += cr.raw_blocks; r.rle_blocks += cr.rle_blocks;
        }
        uint8_t *start = body;
        if (k == 0) { start -= FC_HEADER; fc_header(start, fc->checksum, fc->window_log); }
        if (final) len += fc_trailer(body + len, n % ENC_BLOCK == 0, fc->checksum, h, r);
        const size_t w = (size_t)(body + len - start);
        if (!write_all(wr, wu, start, w, nullptr)) return fc_panic(c, "FrameCompressor::compress: the drain's write failed");
        r.dst_size += w;
        return 0;
    };
    size_t n0 = 0;
    bool eof0 = false;
    if (int e = read(0, n0, eof0)) return e;
    return fc->p.run(c, n0, eof0, enqueue, read, write);
}

extern "C" int b200z_frame_compressor_compress(b200z_frame_compressor *fc, b200z_read_fn rd, void *ru, b200z_write_fn wr, void *wu,
                                               b200z_compress_result *result) {
    if (!fc || !rd || !wr) return B200Z_ERR_INVALID_ARGUMENT;
    b200z_ctx *c = fc->ctx;
    if (int e = compress_check(c, fc->level, (int)fc->window_log, nullptr)) return e;
    b200z_compress_result r{};
    XXH64State h;
    h.reset();
    int e = 0;
    if (fc->level == B200Z_LEVEL_UNCOMPRESSED) e = fc_compress_raw(fc, rd, ru, wr, wu, h, r);
    else if (!(e = c->use())) e = fc_compress_fast(fc, rd, ru, wr, wu, h, r);
    r.status = e;
    if (result) *result = r;
    return e;
}

// ---------------------------------------------------------------------------------------------------------------
// raw-content dictionary trainer (EXTENSION in place of ruzstd::dictionary, DESIGN.md section 4.5): host checks and the epoch
// plan, then k_dtcount -> k_dtprev -> one k_dtepoch per epoch on the ctx stream; the chosen segments' bytes are then gathered
// into the host dictionary by ascending score
// ---------------------------------------------------------------------------------------------------------------
struct DictTrainResources {
    DevBuf input, starts, slots, dist, freq, best, done, segs;
};

b200z_ctx::~b200z_ctx() = default;

struct DtEpoch { uint32_t e0, e1, le; };

// compute_epoch_info (cover.rs:117-132) with the collection's n bytes in place of its k-mer count; the last epoch runs to n
static std::vector<DtEpoch> dt_epochs(uint64_t n, uint64_t dict_size, uint64_t seg) {
    const uint64_t L = std::min(seg, n);
    uint64_t E = std::max<uint64_t>(1, dict_size / L), es = n / E;
    if (es < 10000) {
        es = std::min<uint64_t>(10000, n);
        E = n / es;
    }
    std::vector<DtEpoch> out(E);
    for (uint64_t e = 0; e < E; e++) {
        const uint64_t e0 = e * es, e1 = e + 1 == E ? n : e0 + es;
        out[e] = DtEpoch{(uint32_t)e0, (uint32_t)e1, (uint32_t)std::min(L, e1 - e0)};
    }
    return out;
}

extern "C" int b200z_dict_train_raw(b200z_ctx *c, const uint8_t *samples, size_t samples_len, int samples_mem, const size_t *sample_sizes,
                                    size_t nsamples, size_t dict_size, size_t segment_size, uint8_t *dict, size_t dict_cap, size_t *dict_len,
                                    b200z_dict_segment *segments, size_t segments_cap, size_t *nsegments) {
    // ---- everything is checked before any device work
    if (!c) return B200Z_ERR_INVALID_ARGUMENT;
    auto reject = [c](const char *why) { c->err = why; return B200Z_ERR_INVALID_ARGUMENT; };
    const size_t seg = segment_size ? segment_size : 2048;
    if ((samples_len && !samples) || (samples_mem != B200Z_MEM_HOST && samples_mem != B200Z_MEM_DEVICE) || !dict_len) return reject("invalid argument");
    if (seg < DT_K || seg > 65536) return reject("segment_size outside [16, 65536]");
    if (samples_len >= (1ull << 32)) return reject("samples_len >= 2^32");
    std::vector<uint32_t> starts;
    if (sample_sizes) {
        if (nsamples >= (1ull << 32)) return reject("more than 2^32 - 1 samples");
        uint64_t sum = 0;
        for (size_t i = 0; i < nsamples; i++) {
            if (sample_sizes[i] > samples_len - sum) return reject("sample sizes do not sum to samples_len");
            starts.push_back((uint32_t)sum);
            sum += sample_sizes[i];
        }
        if (sum != samples_len) return reject("sample sizes do not sum to samples_len");
    } else {
        starts.push_back(0);
    }
    starts.push_back((uint32_t)samples_len);
    const uint64_t n = samples_len;
    std::vector<DtEpoch> ep;
    uint64_t total = 0, need = n;
    if (n >= DT_K) {
        if (dict_size) ep = dt_epochs(n, dict_size, seg);
        for (const DtEpoch &x : ep) total += x.le;
        need = std::min<uint64_t>(dict_size, total);
    }
    if (dict_cap < need || (need && !dict)) return reject("dict_cap is smaller than the dictionary");
    if (segments && segments_cap < ep.size()) return reject("segments_cap is smaller than the number of epochs");
    *dict_len = 0;
    if (nsegments) *nsegments = 0;
    if (n < DT_K) {   // the reference's rule: a source this short is its own dictionary
        if (n && samples_mem == B200Z_MEM_DEVICE) {
            if (int e = c->use()) return e;
            CU(c, cudaMemcpy(dict, samples, n, cudaMemcpyDeviceToHost));
        } else if (n) {
            memcpy(dict, samples, n);
        }
        *dict_len = n;
        return 0;
    }
    if (ep.empty()) return 0;
    if (int e = c->use()) return e;
    // ---- device passes
    if (!c->dtrain) c->dtrain.reset(new DictTrainResources());
    DictTrainResources &r = *c->dtrain;
    const uint32_t E = (uint32_t)ep.size(), ns = (uint32_t)(starts.size() - 1);
    int e = 0;
    if ((e = r.starts.ensure(starts.size() * 4)) || (e = r.slots.ensure(n * 4)) || (e = r.dist.ensure(n * 2)) ||
        (e = r.freq.ensure(sizeof(uint32_t) << DT_F)) || (e = r.best.ensure((size_t)E * 8)) || (e = r.done.ensure((size_t)E * 4)) ||
        (e = r.segs.ensure((size_t)E * sizeof(b200z_dict_segment))))
        return e;
    cudaStream_t s = c->stream;
    const uint8_t *d_in = samples;
    if (samples_mem == B200Z_MEM_HOST) {
        if ((e = r.input.ensure(n + 16))) return e;
        CU(c, cudaMemcpyAsync(r.input.p, samples, n, cudaMemcpyHostToDevice, s));
        d_in = r.input.as<uint8_t>();
    }
    CU(c, cudaMemcpyAsync(r.starts.p, starts.data(), starts.size() * 4, cudaMemcpyHostToDevice, s));
    CU(c, cudaMemsetAsync(r.freq.p, 0, sizeof(uint32_t) << DT_F, s));
    CU(c, cudaMemsetAsync(r.best.p, 0, (size_t)E * 8, s));
    CU(c, cudaMemsetAsync(r.done.p, 0, (size_t)E * 4, s));
    uint32_t *slots = r.slots.as<uint32_t>(), *freq = r.freq.as<uint32_t>();
    uint16_t *dist = r.dist.as<uint16_t>();
    if (int le = launch_dt_count(d_in, (uint32_t)n, r.starts.as<uint32_t>(), ns, slots, freq, s, &c->launches)) return c->set_cuda_err((cudaError_t)le, "k_dtcount");
    const uint32_t w = (uint32_t)std::min<uint64_t>(seg, n) - (DT_K - 1);
    if (int le = launch_dt_prev(slots, (uint32_t)n, w, dist, s, &c->launches)) return c->set_cuda_err((cudaError_t)le, "k_dtprev");
    for (uint32_t i = 0; i < E; i++)
        if (int le = launch_dt_epoch(slots, dist, freq, i, ep[i].e0, ep[i].e1, ep[i].le, r.best.as<unsigned long long>() + i, r.done.as<uint32_t>() + i,
                                     r.segs.as<b200z_dict_segment>() + i, s, &c->launches))
            return c->set_cuda_err((cudaError_t)le, "k_dtepoch");
    std::vector<b200z_dict_segment> hs(E);
    CU(c, cudaMemcpyAsync(hs.data(), r.segs.p, (size_t)E * sizeof(b200z_dict_segment), cudaMemcpyDeviceToHost, s));
    CU(c, cudaStreamSynchronize(s));
    // ---- the dictionary: segments by ascending score (ties by epoch), the highest score last, nearest the data; the last `need`
    // bytes of their concatenation
    std::vector<uint32_t> order(E);
    for (uint32_t i = 0; i < E; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return hs[a].score < hs[b].score; });
    uint64_t skip = total - need, at = 0;
    for (uint32_t i : order) {
        const b200z_dict_segment &g = hs[i];
        const uint64_t drop = std::min<uint64_t>(skip, g.size), len = g.size - drop;
        skip -= drop;
        if (!len) continue;
        if (samples_mem == B200Z_MEM_HOST) memcpy(dict + at, samples + g.src_off + drop, len);
        else CU(c, cudaMemcpyAsync(dict + at, samples + g.src_off + drop, len, cudaMemcpyDeviceToHost, s));
        at += len;
    }
    if (samples_mem == B200Z_MEM_DEVICE) CU(c, cudaStreamSynchronize(s));
    *dict_len = at;
    if (segments) memcpy(segments, hs.data(), (size_t)E * sizeof(b200z_dict_segment));
    if (nsegments) *nsegments = E;
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// dictionary finalizer (EXTENSION, ZDICT_finalizeDictionary's counterpart, DESIGN.md section 4.6): host checks, then k_cdict on the
// content's tail and, per submission of at most DS_BLOCKS samples, k_cmatch<true> -> k_dstats on the compressor's staging; the
// counts come back and dict_from_counts (dict_format.cpp) writes the dictionary
// ---------------------------------------------------------------------------------------------------------------
extern "C" int b200z_debug_dict_from_counts(const uint64_t counts[377], const uint8_t *content, size_t content_len, uint32_t dict_id,
                                            uint8_t *dict, size_t dict_cap, size_t *dict_len) {
    return dict_from_counts(counts, content, content_len, dict_id, dict, dict_cap, dict_len);
}

extern "C" int b200z_dict_finalize(b200z_ctx *c, const uint8_t *content, size_t content_len, const uint8_t *samples, size_t samples_len,
                                   int samples_mem, const size_t *sample_sizes, size_t nsamples, uint32_t dict_id, uint8_t *dict,
                                   size_t dict_cap, size_t *dict_len) {
    // ---- everything is checked before any device work
    if (!c) return B200Z_ERR_INVALID_ARGUMENT;
    auto reject = [c](const char *why) { c->err = why; return B200Z_ERR_INVALID_ARGUMENT; };
    if (!content || (samples_len && !samples) || (nsamples && !sample_sizes) || (samples_mem != B200Z_MEM_HOST && samples_mem != B200Z_MEM_DEVICE) ||
        !dict || !dict_len)
        return reject("invalid argument");
    if (dict_check_args(content_len, dict_id, dict_cap))
        return reject("content_len outside [8, 2^31), dict_id >= 2^31 or dict_cap < B200Z_DICT_HEADER_MAX + 8");
    if (nsamples > 0xffffffffu) return reject("more than 2^32 - 1 samples");
    std::vector<CBlock> hb(nsamples);
    uint64_t sum = 0;
    for (size_t i = 0; i < nsamples; i++) {
        if (sample_sizes[i] > samples_len - sum) return reject("sample sizes do not sum to samples_len");
        hb[i] = CBlock{sum, (uint32_t)std::min<size_t>(sample_sizes[i], ENC_BLOCK), 0, (uint32_t)i, 0};
        sum += sample_sizes[i];
    }
    if (sum != samples_len) return reject("sample sizes do not sum to samples_len");
    std::vector<uint64_t> counts(DS_BINS, 0);
    if (nsamples) {
        if (int e = c->use()) return e;
        CompressResources *rp = nullptr;
        if (int e = compress_get(c, &rp)) return e;
        CompressResources &r = *rp;
        const uint64_t per = std::min<uint64_t>(nsamples, DS_BLOCKS);
        const uint32_t tail = (uint32_t)std::min<size_t>(content_len, ENC_WINDOW);   // all a match can reach
        int e = 0;
        if ((e = r.blocks.ensure(nsamples * sizeof(CBlock))) || (e = r.stage.ensure(per, true)) || (e = r.dcontent.ensure(tail + 16)) ||
            (e = r.dtab.ensure(sizeof(uint32_t) << CD_LOG)) || (e = r.dcounts.ensure(DS_BINS * 8)))
            return e;
        cudaStream_t s = c->stream;
        const uint8_t *d_in = samples;
        if (samples_mem == B200Z_MEM_HOST) {
            if ((e = r.input.ensure(samples_len + 16))) return e;
            CU(c, cudaMemcpyAsync(r.input.p, samples, samples_len, cudaMemcpyHostToDevice, s));
            d_in = r.input.as<uint8_t>();
        }
        CU(c, cudaMemcpyAsync(r.dcontent.p, content + (content_len - tail), tail, cudaMemcpyHostToDevice, s));
        CU(c, cudaMemcpyAsync(r.blocks.p, hb.data(), nsamples * sizeof(CBlock), cudaMemcpyHostToDevice, s));
        CU(c, cudaMemsetAsync(r.dcounts.p, 0, DS_BINS * 8, s));
        if (int le = launch_dict_table(r.dcontent.as<uint8_t>(), tail, r.dtab.as<uint32_t>(), s, &c->launches))
            return c->set_cuda_err((cudaError_t)le, "k_cdict");
        CompressArgs a{};
        a.input = d_in;
        r.stage.bind(a);
        a.dict = r.dcontent.as<uint8_t>(); a.dtab = r.dtab.as<uint32_t>(); a.dict_len = tail;
        for (uint64_t b0 = 0; b0 < nsamples; b0 += per) {
            a.blocks = r.blocks.as<CBlock>() + b0;
            a.nblocks = (uint32_t)std::min<uint64_t>(per, nsamples - b0);
            if (int le = launch_dict_stats(a, r.dcounts.as<unsigned long long>(), s, &c->launches)) return c->set_cuda_err((cudaError_t)le, "k_dstats");
        }
        CU(c, cudaMemcpyAsync(counts.data(), r.dcounts.p, DS_BINS * 8, cudaMemcpyDeviceToHost, s));
        CU(c, cudaStreamSynchronize(s));
    }
    return dict_from_counts(counts.data(), content, content_len, dict_id, dict, dict_cap, dict_len);
}
