// capi.cu -- C ABI of libbmb200 (see include/bmb200.h).  Host-side orchestration only: arena
// allocation, H2D/D2H, launches.  There is deliberately NO CPU compute path: without an sm_90
// device bmb200_init fails with BMB200_ERR_NODEVICE.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "agg_kernel.cuh"
#include "aux_kernels.cuh"
#include "runlist_kernel.cuh"
#include "scan_kernel.cuh"
#include "rank_kernel.cuh"
#include "shift_kernel.cuh"
#include "binop_kernel.cuh"
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include "blob_kernel.cuh"
#include "blob_entropy.cuh"
#include "host_pack.hpp"
#include "comm.hpp"
#include <sched.h>
#include <fstream>

using namespace bmb200;

// Slots of the context's grow-only scratch (pool_dev / pool_host), one per buffer and role.  Entry points that do the same job share
// a slot: bmb200_result_fetch and bmb200_result_fetch_view compact through the same buffers, rank and select batches stage through
// the same ones.
enum DevSlot {
    kDevCompactOff,                   // compaction of a result: per-column offsets
    kDevCompactBits,                  //   compacted bit-blocks
    kDevCompactGaps,                  //   compacted GAP words
    kDevRsIn,                         // bmb200_rank_batch / bmb200_select_batch: positions or ranks in
    kDevRsOut,                        //   ranks or positions out
    kDevRsFound,                      //   select's found flags
    kDevSlabMirror,                   // bmb200_set_upload_slabs: the device mirror of the slabs (freed by bmb200_ctx_trim)
    kDevSlabSrc,                      //   where each block sits in the mirror (freed by bmb200_ctx_trim)
    kDevRankDense,                    // bmb200_rank_compress: the dense scatter target
    kDevBlobStage,                    // bmb200_set_upload_blobs: the BLOB bytes
    kDevBlobOff, kDevBlobSize,        //   per-vector offset and size inside the staged bytes
    kDevBlobToks, kDevBlobNToks,      //   pass 1: token table, tokens per segment
    kDevBlobStatus, kDevBlobFull,     //   status words, FULL-block flags
    kDevBlobScratch,                  //   per-warp decode scratch
    kDevBlobSegs, kDevBlobSegCap,     //   pass 1: segments, their token capacities and processing order
    kDevBlobRecs, kDevBlobERecs,      //   decode records: explicit-length tokens, entropy-coded tokens
    kDevBlobDur,                      //   pass 2: clocks per work item (BMB200_TRACE)
    kDevSlots
};
enum HostSlot {
    kHostCompactOff,                  // bmb200_result_fetch: staging of the per-column offsets
    kHostExchange,                    // bmb200_exchange_fetch: the gathered rows
    kHostViewMeta,                    // bmb200_result_fetch_view: kind | nruns | totals | offsets
    kHostViewBits0, kHostViewGaps0,   //   its two block buffers, used in turn (see there)
    kHostViewBits1, kHostViewGaps1,
    kHostSlabSrc,                     // bmb200_set_upload_slabs: staging of the block sources
    kHostBlobStage,                   // bmb200_set_upload_blobs: the BLOB bytes, gathered for one DMA
    kHostSlots
};

struct bmb200_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    uint64_t launches = 0;
    std::string last_err;
    int sm_count = 0, cc_major = 0, cc_minor = 0;
    size_t hbm_bytes = 0;
    uint32_t* d_work = nullptr;             // work counter for the persistent kernel
    uint32_t* d_group = nullptr;            // group member ids, then the 2*n_groups+1 offsets
    size_t group_cap = 0;
    uint32_t* h_group = nullptr;            // pinned staging for the group ids
    std::vector<uint32_t> last_group;       // ids currently resident in d_group (skip the re-upload when unchanged)
    int agg_ctas_per_sm = kCtasPerSm;
    bmb200_set* host_set = nullptr;         // device arena kept between bmb200_aggregate_host calls (cudaMalloc/cudaFree
    bmb200_result* host_res = nullptr;      //   of a multi-GB arena costs tens of ms per call otherwise)
    int gap_mode = 0;                       // 0 = stream sorted GAP lists through the smem ring, 1 = always gather
    bool attr_set = false, merge_attr_set = false;
    size_t agg_dyn[4] = {};                 // dynamic shared memory per agg_kernel<OP> (set_agg_attrs)
    size_t pipe_dyn = 0;                    // ... of agg_pipe_kernel
    int agg_pipeline = 1;                   // 1 = whole-set AND-SUB takes agg_pipe_kernel, 0 = always agg_kernel
    int run_lists = 1;                      // run-list companion of agg_pipe_kernel: 0 never, 1 from a set's second qualifying call, 2 from its first
    int host_threads = 0;                   // host threads of bmb200_set_upload_vectors (0 = hardware concurrency, at most 64)
    uint8_t* h_ring[kStageSlots] = {};      // pinned staging ring of bmb200_set_upload_vectors (grow-only)
    size_t h_ring_cap = 0;
    cudaEvent_t ring_ev[kStageSlots] = {};
    void* d_pool[kDevSlots] = {};           // grow-only device scratch by DevSlot (no cudaMalloc per call once warm)
    size_t d_pool_cap[kDevSlots] = {};
    std::vector<std::pair<uint64_t, uint64_t>> mirror_sig;   // slab list (base, bytes) whose copies into kDevSlabMirror were queued last
    bool mirror_live = false;               // ... by bmb200_host_slabs_prefetch, not yet consumed by an upload
    void* h_pool[kHostSlots] = {};          // grow-only pinned scratch by HostSlot
    size_t h_pool_cap[kHostSlots] = {};
    cudaEvent_t fetch_ev[8] = {};           // one per D2H chunk of bmb200_result_fetch_view_async
    unsigned fetch_flip = 0;                // bmb200_result_fetch_view alternates between two pinned block buffers (see there)
    CommState comm;                         // multi-GPU exchange (bmb200_comm_*), unused on one GPU
    // ONE recycled device arena: bmb200_set_free parks the arrays of the last freed set here and the next set_alloc that fits takes
    // them, so that a cold upload per call (no residency) does not pay cudaMalloc + cudaFree of a multi-GB arena (25 - 230 ms) each time;
    // released by bmb200_ctx_trim / bmb200_destroy
    struct Arena { void *desc = nullptr, *bb = nullptr, *gb = nullptr, *bp = nullptr, *gp = nullptr; size_t cap_desc = 0, cap_base = 0, cap_bit = 0, cap_gap = 0; bool full = false; } arena;
};

struct bmb200_set {
    bmb200_ctx* ctx = nullptr;
    SetView v{};
    bool owns = false;
    uint64_t n_bit_blocks = 0, n_gap_units = 0;
    int flat_gaps = -1;                     // every GAP block in BMB200_DESC_GAP_FLAT form: 1 yes, 0 no, -1 not checked yet (flat_gap_set)
    uint64_t gap_pool_bytes = 0;            // readable bytes of gap_pool (with the allocation slack when owned)
    std::vector<uint32_t> gap_vecs;         // bit v: vector v holds a GAP block in some column; empty until gap_vectors() asks
    // run-list companion of the GAP blocks (runlist_kernel.cuh), always owned by the set and freed with it
    int rl_state = 0;                       // 0 not built, 1 built, -1 cannot be built (device memory): calls run without it
    uint32_t rl_calls = 0;                  // qualifying calls seen while not built
    uint64_t *rl_sgl_base = nullptr, *rl_lr_base = nullptr, *rl_sgl_mid = nullptr, *rl_lr_mid = nullptr;
    uint16_t* rl_sgl = nullptr;
    uint32_t* rl_lr = nullptr;
    uint32_t* rl_listed = nullptr;          // bit i: bit-block i of bit_pool is listed in part B
    uint64_t rl_sgl_units = 0, rl_lr_units = 0;        // part A
    uint64_t rl_b_sgl_units = 0, rl_b_lr_units = 0, rl_listed_blocks = 0;   // part B
    std::vector<uint32_t> listed_vecs;      // bit v: vector v holds a listed bit-block in some column (set with the companion)
    size_t cap_desc = 0, cap_base = 0, cap_bit = 0, cap_gap = 0;   // capacities when the arrays came from set_alloc (elements / blocks / units); 0 = not recyclable
};

struct bmb200_result {
    bmb200_ctx* ctx = nullptr;
    uint32_t n_cols = 0;                    // total columns = n_groups * cols_per_group
    uint32_t n_groups = 1, cols_per_group = 0;
    uint32_t* or_blocks = nullptr;          // [cols_per_group][2048] union of all groups (BMB200_F_OR_TARGET)
    bool has_or = false;                    // the last launch into this result filled or_blocks (a recycled result keeps the buffer)
    bool has_blocks = false, compress = false, gaps_ready = false;
    uint32_t* blocks = nullptr;
    uint32_t* popcnt = nullptr;
    uint64_t* digest = nullptr;
    uint32_t* nruns = nullptr;
    uint8_t*  kind = nullptr;
    uint16_t* gaps = nullptr;
    unsigned long long* total = nullptr;
    // single-group results keep TWO (popcnt[n_cols] | total) buffers back to back and alternate between them while a communicator
    // is attached: bmb200_exchange_popcounts then sends straight out of the buffer the kernel wrote (no staging copy) while the
    // next aggregation already fills the other one
    uint32_t* popcnt_base = nullptr;
    uint32_t xstride = 0, xflip = 0;
    bool total_inline = false;
    uint32_t fetch_chunk_cols = 0, fetch_chunks = 0;   // bmb200_result_fetch_view_async: columns per D2H chunk, chunks in flight
};

struct bmb200_rs {
    bmb200_ctx* ctx = nullptr;
    const bmb200_set* set = nullptr;
    uint32_t vec = 0, nsb = 0, n_blocks = 0;
    uint32_t* bcount = nullptr;
    uint64_t* sub_count = nullptr;
    uint32_t* row_cum = nullptr;
    uint64_t* sb_tot = nullptr;
    uint64_t* sb_cum = nullptr;
    uint32_t* fine = nullptr;               // device-private fine index (aux_kernels.cuh): [n_blocks][128]
    uint32_t* fine_piv = nullptr;           // [n_blocks][8]
    uint32_t* row_piv = nullptr;            // [nsb][16]
};

namespace {

constexpr size_t kSlack = 512;   // readable bytes past the end of each pool (GAP first-load over-read)

#define CU(call)                                                                        \
    do {                                                                                \
        cudaError_t _e = (call);                                                        \
        if (_e != cudaSuccess) {                                                        \
            if (ctx) { ctx->last_err = std::string(#call) + ": " + cudaGetErrorString(_e); } \
            return BMB200_ERR_CUDA;                                                     \
        }                                                                               \
    } while (0)

// BMB200_TRACE=1: phase timings of the host-side entry points on stderr (wall clock; each mark synchronizes the stream first,
// so the time of a phase is attributed to it -- tracing changes the overlap, never the results)
struct PhaseTrace {
    bool on; const char* fn; cudaStream_t st; std::chrono::steady_clock::time_point t0, t_prev;
    PhaseTrace(const char* f, cudaStream_t s) : on(getenv("BMB200_TRACE") != nullptr), fn(f), st(s) { if (on) t0 = t_prev = std::chrono::steady_clock::now(); }
    void mark(const char* what)
    {
        if (!on) return;
        cudaStreamSynchronize(st);
        const auto t = std::chrono::steady_clock::now();
        fprintf(stderr, "[bmb200] %s: %-28s %9.3f ms  (total %9.3f ms)\n", fn, what,
                std::chrono::duration<double, std::milli>(t - t_prev).count(), std::chrono::duration<double, std::milli>(t - t0).count());
        t_prev = t;
    }
};

int after_launch(bmb200_ctx* ctx)
{
    ctx->launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { ctx->last_err = std::string("kernel launch: ") + cudaGetErrorString(e); return BMB200_ERR_CUDA; }
    return BMB200_OK;
}

template <typename T>
int dev_alloc(bmb200_ctx* ctx, T** p, size_t n, size_t slack_bytes = 0)
{
    *p = nullptr;
    cudaError_t e = cudaMalloc((void**)p, n * sizeof(T) + slack_bytes + 16);
    if (e != cudaSuccess) {
        ctx->last_err = std::string("cudaMalloc: ") + cudaGetErrorString(e);
        return e == cudaErrorMemoryAllocation ? BMB200_ERR_BADALLOC : BMB200_ERR_CUDA;
    }
    return BMB200_OK;
}

void free_set_arrays(bmb200_set* s)
{
    if (!s || !s->owns) return;
    cudaFree((void*)s->v.desc); cudaFree((void*)s->v.bit_base); cudaFree((void*)s->v.gap_base);
    cudaFree((void*)s->v.bit_pool); cudaFree((void*)s->v.gap_pool);
}

void free_run_lists(bmb200_set* s)
{
    cudaFree(s->rl_sgl_base); cudaFree(s->rl_lr_base); cudaFree(s->rl_sgl_mid); cudaFree(s->rl_lr_mid);
    cudaFree(s->rl_sgl); cudaFree(s->rl_lr); cudaFree(s->rl_listed);
    s->rl_sgl_base = s->rl_lr_base = s->rl_sgl_mid = s->rl_lr_mid = nullptr; s->rl_sgl = nullptr; s->rl_lr = nullptr; s->rl_listed = nullptr;
    s->rl_sgl_units = s->rl_lr_units = s->rl_b_sgl_units = s->rl_b_lr_units = s->rl_listed_blocks = 0;
    s->listed_vecs.clear();
}

void free_result_arrays(bmb200_result* r)
{
    if (!r) return;
    cudaFree(r->blocks); cudaFree(r->popcnt_base ? r->popcnt_base : r->popcnt); cudaFree(r->digest); cudaFree(r->nruns);
    cudaFree(r->kind); cudaFree(r->gaps); if (!r->total_inline) cudaFree(r->total); cudaFree(r->or_blocks);
}

// grow-only scratch owned by the context: the hot entry points never call cudaMalloc / cudaMallocHost once warm.
// The caller has synchronized (or is ordered on) the context stream before it reuses a slot.
int pool_dev(bmb200_ctx* ctx, DevSlot slot, size_t bytes, void** out)
{
    if (bytes > ctx->d_pool_cap[slot]) {
        if (ctx->d_pool[slot]) { cudaStreamSynchronize(ctx->stream); cudaFree(ctx->d_pool[slot]); ctx->d_pool[slot] = nullptr; ctx->d_pool_cap[slot] = 0; }
        const size_t cap = bytes + (bytes > (1ull << 30) ? 0 : bytes / 4) + 256;     // multi-GB buffers (the slab mirror) are sized exactly
        cudaError_t e = cudaMalloc(&ctx->d_pool[slot], cap);
        if (e != cudaSuccess) { ctx->last_err = std::string("cudaMalloc(pool): ") + cudaGetErrorString(e); return e == cudaErrorMemoryAllocation ? BMB200_ERR_BADALLOC : BMB200_ERR_CUDA; }
        ctx->d_pool_cap[slot] = cap;
    }
    *out = ctx->d_pool[slot];
    return BMB200_OK;
}
int pool_host(bmb200_ctx* ctx, HostSlot slot, size_t bytes, void** out)
{
    if (bytes > ctx->h_pool_cap[slot]) {
        if (ctx->h_pool[slot]) { cudaStreamSynchronize(ctx->stream); cudaFreeHost(ctx->h_pool[slot]); ctx->h_pool[slot] = nullptr; ctx->h_pool_cap[slot] = 0; }
        const size_t cap = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMallocHost(&ctx->h_pool[slot], cap);
        if (e != cudaSuccess) { ctx->last_err = std::string("cudaMallocHost(pool): ") + cudaGetErrorString(e); return BMB200_ERR_BADALLOC; }
        ctx->h_pool_cap[slot] = cap;
    }
    *out = ctx->h_pool[slot];
    return BMB200_OK;
}

void comm_release(bmb200_ctx* ctx)
{
    CommState& c = ctx->comm;
    if (c.side) cudaStreamSynchronize(c.side);
    for (int k = 0; k < CommState::kSlots; ++k) {
        if (c.ready[k]) cudaEventDestroy(c.ready[k]);
        if (c.done[k]) cudaEventDestroy(c.done[k]);
        cudaFree(c.stage[k]); cudaFree(c.gathered[k]);
    }
    if (c.comm && nccl_api().CommDestroy) nccl_api().CommDestroy(c.comm);
    if (c.side) cudaStreamDestroy(c.side);
    c = CommState();
}

}  // namespace

extern "C" {

const char* bmb200_error_msg(int code)
{
    switch (code) {
    case BMB200_OK: return "ok";
    case BMB200_ERR_BADALLOC: return "allocation failed";
    case BMB200_ERR_BADARG: return "bad argument";
    case BMB200_ERR_RANGE: return "index out of range";
    case BMB200_ERR_RS_IDX_MISSING: return "rank-select index missing";
    case BMB200_ERR_CUDA: return "CUDA runtime error (see bmb200_last_error)";
    case BMB200_ERR_NODEVICE: return "no sm_90 (H100) device available; libbmb200 has no CPU fallback";
    case BMB200_ERR_UNSUPPORTED: return "serialized BLOB uses a block encoding the device decoder does not cover";
    default: return "unknown error";
    }
}

int bmb200_init(int device, bmb200_ctx** out)
{
    if (!out) return BMB200_ERR_BADARG;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { cudaGetLastError(); return BMB200_ERR_NODEVICE; }
    if (device < 0 || device >= n) return BMB200_ERR_BADARG;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return BMB200_ERR_NODEVICE;
    if (prop.major != 9 || prop.minor != 0) return BMB200_ERR_NODEVICE;     // kernels are built for sm_90a only
    bmb200_ctx* ctx = new (std::nothrow) bmb200_ctx();
    if (!ctx) return BMB200_ERR_BADALLOC;
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    ctx->cc_major = prop.major; ctx->cc_minor = prop.minor;
    ctx->hbm_bytes = prop.totalGlobalMem;
    if (cudaSetDevice(device) != cudaSuccess ||
        cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaMalloc((void**)&ctx->d_work, 64) != cudaSuccess) {
        delete ctx; return BMB200_ERR_CUDA;
    }
    ctx->own_stream = true;
    // environment overrides go through the same checks as bmb200_ctx_set_tuning (out-of-range values are ignored)
    const char* e = getenv("BMB200_AGG_CTAS_PER_SM");
    if (e) bmb200_ctx_set_tuning(ctx, BMB200_TUNE_CTAS_PER_SM, atoi(e));
    e = getenv("BMB200_GAP_MODE");
    if (e) bmb200_ctx_set_tuning(ctx, BMB200_TUNE_GAP_MODE, atoi(e));
    e = getenv("BMB200_HOST_THREADS");
    if (e) bmb200_ctx_set_tuning(ctx, BMB200_TUNE_HOST_THREADS, atoi(e));
    *out = ctx;
    return BMB200_OK;
}

int bmb200_destroy(bmb200_ctx* ctx)
{
    if (!ctx) return BMB200_ERR_BADARG;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->host_res) bmb200_result_free(ctx->host_res);
    if (ctx->host_set) bmb200_set_free(ctx->host_set);
    bmb200_ctx_trim(ctx);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    cudaFree(ctx->d_work); cudaFree(ctx->d_group);
    if (ctx->h_group) cudaFreeHost(ctx->h_group);
    for (void* q : ctx->d_pool) if (q) cudaFree(q);
    for (void* q : ctx->h_pool) if (q) cudaFreeHost(q);
    for (uint32_t k = 0; k < kStageSlots; ++k) { if (ctx->h_ring[k]) cudaFreeHost(ctx->h_ring[k]); if (ctx->ring_ev[k]) cudaEventDestroy(ctx->ring_ev[k]); }
    for (cudaEvent_t ev : ctx->fetch_ev) if (ev) cudaEventDestroy(ev);
    comm_release(ctx);
    delete ctx;
    return BMB200_OK;
}

int bmb200_last_error(const bmb200_ctx* ctx, char* buf, size_t buflen)
{
    if (!ctx || !buf || !buflen) return BMB200_ERR_BADARG;
    snprintf(buf, buflen, "%s", ctx->last_err.c_str());
    return BMB200_OK;
}

int bmb200_ctx_set_stream(bmb200_ctx* ctx, void* cuda_stream)
{
    if (!ctx) return BMB200_ERR_BADARG;
    cudaSetDevice(ctx->device);
    if (ctx->own_stream) { cudaStreamSynchronize(ctx->stream); cudaStreamDestroy(ctx->stream); }
    ctx->stream = (cudaStream_t)cuda_stream;
    ctx->own_stream = false;
    return BMB200_OK;
}

int bmb200_ctx_get_stream(const bmb200_ctx* ctx, void** cuda_stream)
{
    if (!ctx || !cuda_stream) return BMB200_ERR_BADARG;
    *cuda_stream = (void*)ctx->stream;
    return BMB200_OK;
}

int bmb200_ctx_sync(bmb200_ctx* ctx)
{
    if (!ctx) return BMB200_ERR_BADARG;
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    return BMB200_OK;
}

int bmb200_ctx_launch_count(const bmb200_ctx* ctx, uint64_t* out)
{
    if (!ctx || !out) return BMB200_ERR_BADARG;
    *out = ctx->launches;
    return BMB200_OK;
}

int bmb200_device_info(const bmb200_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor, uint64_t* hbm_bytes)
{
    if (!ctx) return BMB200_ERR_BADARG;
    if (sm_count) *sm_count = ctx->sm_count;
    if (cc_major) *cc_major = ctx->cc_major;
    if (cc_minor) *cc_minor = ctx->cc_minor;
    if (hbm_bytes) *hbm_bytes = ctx->hbm_bytes;
    return BMB200_OK;
}

int bmb200_ctx_set_tuning(bmb200_ctx* ctx, int key, int value)
{
    if (!ctx) return BMB200_ERR_BADARG;
    if (key == BMB200_TUNE_GAP_MODE && (value == 0 || value == 1)) { ctx->gap_mode = value; return BMB200_OK; }
    if (key == BMB200_TUNE_CTAS_PER_SM && value >= 1 && value <= kCtasPerSm) { ctx->agg_ctas_per_sm = value; return BMB200_OK; }
    if (key == BMB200_TUNE_HOST_THREADS && value >= 0 && value <= 64) { ctx->host_threads = value; return BMB200_OK; }
    if (key == BMB200_TUNE_AGG_PIPELINE && (value == 0 || value == 1)) { ctx->agg_pipeline = value; return BMB200_OK; }
    if (key == BMB200_TUNE_RUN_LISTS && value >= 0 && value <= 2) { ctx->run_lists = value; return BMB200_OK; }
    return BMB200_ERR_BADARG;
}

/* ------------------------------------------------------------------ sets */

static int set_alloc(bmb200_ctx* ctx, uint32_t n_vec, uint32_t n_blocks, uint64_t n_bit, uint64_t n_gap_units,
                     bmb200_set** out)
{
    bmb200_set* s = new (std::nothrow) bmb200_set();
    if (!s) return BMB200_ERR_BADALLOC;
    s->ctx = ctx; s->owns = true;
    s->v.n_vec = n_vec; s->v.n_blocks = n_blocks;
    s->n_bit_blocks = n_bit; s->n_gap_units = n_gap_units;
    s->gap_pool_bytes = n_gap_units * 16ull + kSlack;
    int rc;
    uint32_t* desc = nullptr; uint64_t *bb = nullptr, *gb = nullptr; uint32_t* bp = nullptr; uint16_t* gp = nullptr;
    s->cap_desc = (size_t)n_vec * n_blocks; s->cap_base = (size_t)n_blocks + 1; s->cap_bit = n_bit; s->cap_gap = n_gap_units;
    if (ctx->arena.full && ctx->arena.cap_desc >= s->cap_desc && ctx->arena.cap_base >= s->cap_base && ctx->arena.cap_bit >= n_bit && ctx->arena.cap_gap >= n_gap_units) {
        auto& a = ctx->arena;                 // recycle the parked arena (the stream was synchronized when it was parked)
        s->v.desc = (uint32_t*)a.desc; s->v.bit_base = (uint64_t*)a.bb; s->v.gap_base = (uint64_t*)a.gb; s->v.bit_pool = (uint32_t*)a.bp; s->v.gap_pool = (uint16_t*)a.gp;
        s->cap_desc = a.cap_desc; s->cap_base = a.cap_base; s->cap_bit = a.cap_bit; s->cap_gap = a.cap_gap;
        a = bmb200_ctx::Arena();
        cudaMemsetAsync((char*)s->v.gap_pool + (size_t)n_gap_units * kGapUnit * 2, 0, kSlack, ctx->stream);
        *out = s;
        return BMB200_OK;
    }
    if ((rc = dev_alloc(ctx, &desc, (size_t)n_vec * n_blocks)) ||
        (rc = dev_alloc(ctx, &bb, (size_t)n_blocks + 1)) ||
        (rc = dev_alloc(ctx, &gb, (size_t)n_blocks + 1)) ||
        (rc = dev_alloc(ctx, &bp, (size_t)n_bit * kBlockWords, kSlack)) ||
        (rc = dev_alloc(ctx, &gp, (size_t)n_gap_units * kGapUnit, kSlack))) {
        cudaFree(desc); cudaFree(bb); cudaFree(gb); cudaFree(bp); cudaFree(gp);
        delete s; return rc;
    }
    s->v.desc = desc; s->v.bit_base = bb; s->v.gap_base = gb; s->v.bit_pool = bp; s->v.gap_pool = gp;
    // the slack past the GAP pool is read (never interpreted) by the first pair-word load of a GAP block
    cudaMemsetAsync((char*)gp + (size_t)n_gap_units * kGapUnit * 2, 0, kSlack, ctx->stream);
    *out = s;
    return BMB200_OK;
}

// H2D of one packed set into an arena from set_alloc that holds it (bmb200_set_upload, and bmb200_aggregate_host, which reuses its
// arena across calls: the slack behind the GAP pool is zeroed again at the new end)
static int set_copy_in(bmb200_ctx* ctx, bmb200_set* s, const bmb200_packed_set* h, uint64_t n_bit, uint64_t n_gap)
{
    cudaStream_t st = ctx->stream;
    s->v.n_vec = h->n_vec; s->v.n_blocks = h->n_blocks; s->n_bit_blocks = n_bit; s->n_gap_units = n_gap;
    s->gap_pool_bytes = n_gap * 16ull + kSlack;
    CU(cudaMemcpyAsync((void*)s->v.desc, h->desc, (size_t)h->n_vec * h->n_blocks * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync((void*)s->v.bit_base, h->bit_base, ((size_t)h->n_blocks + 1) * 8, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync((void*)s->v.gap_base, h->gap_base, ((size_t)h->n_blocks + 1) * 8, cudaMemcpyHostToDevice, st));
    if (n_bit) CU(cudaMemcpyAsync((void*)s->v.bit_pool, h->bit_pool, (size_t)n_bit * BMB200_BLOCK_BYTES, cudaMemcpyHostToDevice, st));
    if (n_gap) CU(cudaMemcpyAsync((void*)s->v.gap_pool, h->gap_pool, (size_t)n_gap * kGapUnit * 2, cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync((char*)s->v.gap_pool + (size_t)n_gap * kGapUnit * 2, 0, kSlack, st));
    return BMB200_OK;
}

int bmb200_set_upload(bmb200_ctx* ctx, const bmb200_packed_set* h, bmb200_set** out)
{
    if (!ctx || !h || !out || !h->n_vec || !h->n_blocks || !h->desc || !h->bit_base || !h->gap_base)
        return BMB200_ERR_BADARG;
    CU(cudaSetDevice(ctx->device));
    const uint64_t n_bit = h->bit_base[h->n_blocks], n_gap = h->gap_base[h->n_blocks];
    if ((n_bit && !h->bit_pool) || (n_gap && !h->gap_pool)) return BMB200_ERR_BADARG;
    bmb200_set* s = nullptr;
    int rc = set_alloc(ctx, h->n_vec, h->n_blocks, n_bit, n_gap, &s);
    if (rc) return rc;
    if ((rc = set_copy_in(ctx, s, h, n_bit, n_gap))) { free_set_arrays(s); delete s; return rc; }
    *out = s;
    return BMB200_OK;
}

int bmb200_set_upload_vectors(bmb200_ctx* ctx, uint32_t n_vec, uint32_t n_blocks,
                              const bmb200_vec_blocks* vecs, bmb200_set** out)
{
    if (!ctx || !vecs || !out || !n_vec || !n_blocks) return BMB200_ERR_BADARG;
    for (uint32_t v = 0; v < n_vec; ++v)
        if (vecs[v].n_blocks > n_blocks || (vecs[v].n_blocks && (!vecs[v].kind || !vecs[v].ptr))) return BMB200_ERR_BADARG;
    // the block manager stays on the host: its blocks are gathered into the packed column-major layout by a team of host threads
    // (host_pack.hpp) and streamed through a ring of pinned slots -- packing of chunk c+1 overlaps the DMA of chunk c
    PhaseTrace tr("set_upload_vectors", ctx->stream);
    PackLayout L;
    std::vector<PackChunk> chunks;
    try {
        pack_layout(n_vec, n_blocks, vecs, (unsigned)ctx->host_threads, L);
        if (L.rc) return L.rc;
    } catch (...) { return BMB200_ERR_BADALLOC; }
    tr.mark("layout (descriptors, prefix sums)");
    const uint64_t n_bit = L.bb[n_blocks], n_gap = L.gb[n_blocks];
    const uint64_t total = n_bit * (uint64_t)BMB200_BLOCK_BYTES + n_gap * 16ull;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    bmb200_set* s = nullptr;
    int rc = set_alloc(ctx, n_vec, n_blocks, n_bit, n_gap, &s);
    if (rc) return rc;
    auto fail = [&](int code, cudaError_t e) {
        cudaStreamSynchronize(st);
        if (e != cudaSuccess) { ctx->last_err = std::string("set_upload_vectors: ") + cudaGetErrorString(e); code = BMB200_ERR_CUDA; }
        free_set_arrays(s); delete s;
        return code;
    };
    cudaError_t e = cudaMemcpyAsync((void*)s->v.desc, L.desc.data(), L.desc.size() * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync((void*)s->v.bit_base, L.bb.data(), L.bb.size() * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync((void*)s->v.gap_base, L.gb.data(), L.gb.size() * 8, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return fail(BMB200_ERR_CUDA, e);
    if (total) {
        // slot size: 64 MB (PCIe runs at link speed from ~16 MB copies on), never less than the largest column, small sets get small slots
        uint64_t slot_bytes;
        try {
            const uint64_t maxcol = pack_max_column_bytes(L, n_blocks);
            slot_bytes = std::min<uint64_t>(64ull << 20, (total + kStageSlots - 1) / kStageSlots);
            slot_bytes = std::max<uint64_t>(std::max<uint64_t>(slot_bytes, maxcol), 1ull << 16);
            slot_bytes = (slot_bytes + 4095ull) & ~4095ull;
            pack_chunks(L, n_blocks, slot_bytes, chunks);
        } catch (...) { return fail(BMB200_ERR_BADALLOC, cudaSuccess); }
        if (slot_bytes > ctx->h_ring_cap) {
            cudaStreamSynchronize(st);
            for (uint32_t k = 0; k < kStageSlots; ++k) { if (ctx->h_ring[k]) cudaFreeHost(ctx->h_ring[k]); ctx->h_ring[k] = nullptr; }
            ctx->h_ring_cap = 0;
            for (uint32_t k = 0; k < kStageSlots; ++k) {
                e = cudaMallocHost((void**)&ctx->h_ring[k], slot_bytes);
                if (e != cudaSuccess) return fail(BMB200_ERR_BADALLOC, cudaSuccess);
                if (!ctx->ring_ev[k] && (e = cudaEventCreateWithFlags(&ctx->ring_ev[k], cudaEventDisableTiming)) != cudaSuccess) return fail(BMB200_ERR_CUDA, e);
            }
            ctx->h_ring_cap = slot_bytes;
        }
        tr.mark("device arena + staging ring");
        cudaStreamSynchronize(st);                  // a previous upload may still be reading the ring
        try {
            PackPipeline pipe(n_vec, n_blocks, vecs, &L, &chunks, ctx->h_ring);
            pipe.start((unsigned)ctx->host_threads);
            const uint32_t nch = (uint32_t)chunks.size();
            double t_pack = 0, t_dma = 0, t_issue = 0;
            auto now = []() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
            for (uint32_t c = 0; c < nch && e == cudaSuccess; ++c) {
                const double w0 = tr.on ? now() : 0;
                pipe.wait_chunk(c);
                if (tr.on) t_pack += now() - w0;
                const PackChunk& ch = chunks[c];
                uint8_t* base = ctx->h_ring[c % kStageSlots];
                const double w2 = tr.on ? now() : 0;
                if (ch.bit_bytes) e = cudaMemcpyAsync((uint8_t*)s->v.bit_pool + L.bb[ch.c0] * (uint64_t)BMB200_BLOCK_BYTES, base, ch.bit_bytes, cudaMemcpyHostToDevice, st);
                if (e == cudaSuccess && ch.gap_bytes) e = cudaMemcpyAsync((uint8_t*)s->v.gap_pool + L.gb[ch.c0] * 16ull, base + ch.bit_bytes, ch.gap_bytes, cudaMemcpyHostToDevice, st);
                if (e == cudaSuccess) e = cudaEventRecord(ctx->ring_ev[c % kStageSlots], st);
                if (tr.on) t_issue += now() - w2;
                // the copy of chunk c is queued behind the one of chunk c-1: once c-1 has landed its slot goes back to the packers
                if (e == cudaSuccess && c >= 1) { const double w1 = tr.on ? now() : 0; e = cudaEventSynchronize(ctx->ring_ev[(c - 1) % kStageSlots]);
                                                  if (tr.on) t_dma += now() - w1; pipe.release_through(c); }
            }
            pipe.join();
            if (tr.on) fprintf(stderr, "[bmb200] set_upload_vectors: %u chunks of <= %.0f MB, issuing thread waited %.1f ms for the packers and %.1f ms for the DMA, spent %.1f ms inside cudaMemcpyAsync / cudaEventRecord\n",
                               nch, slot_bytes / 1048576.0, t_pack, t_dma, t_issue);
        } catch (...) { return fail(BMB200_ERR_BADALLOC, cudaSuccess); }
        if (e != cudaSuccess) return fail(BMB200_ERR_CUDA, e);
    }
    e = cudaStreamSynchronize(st);                  // L.desc / the ring are host memory of this call
    if (e != cudaSuccess) return fail(BMB200_ERR_CUDA, e);
    tr.mark("pack + H2D (pipelined)");
    *out = s;
    return BMB200_OK;
}

int bmb200_host_slab_alloc(uint64_t bytes, void** out)
{
    if (!out || !bytes) return BMB200_ERR_BADARG;
    void* p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocPortable);
    if (e != cudaSuccess) { cudaGetLastError(); return e == cudaErrorMemoryAllocation ? BMB200_ERR_BADALLOC : BMB200_ERR_CUDA; }
    *out = p;
    return BMB200_OK;
}
int bmb200_host_slab_free(void* slab)
{
    if (!slab) return BMB200_ERR_BADARG;
    return cudaFreeHost(slab) == cudaSuccess ? BMB200_OK : BMB200_ERR_CUDA;
}

// the device mirror of a slab list: slabs back to back (256-byte aligned), sorted by host address for the pointer -> slab search;
// issue = queue the H2D copies now.  ctx->mirror_sig remembers what is in flight so that a prefetch is not repeated.
static int mirror_begin(bmb200_ctx* ctx, const bmb200_host_slab* slabs, uint32_t n_slabs, SlabMap& M, uint8_t** mirror_out, uint64_t* bytes_out)
{
    uint64_t mirror_bytes = 0;
    std::vector<std::pair<uint64_t, uint64_t>> sig;
    try {
        std::vector<uint32_t> order;
        for (uint32_t k = 0; k < n_slabs; ++k) if (slabs[k].base && slabs[k].bytes) order.push_back(k);
        std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return (uintptr_t)slabs[a].base < (uintptr_t)slabs[b].base; });
        for (uint32_t k : order) {
            M.base.push_back((uint64_t)(uintptr_t)slabs[k].base); M.end.push_back(M.base.back() + slabs[k].bytes);
            M.dev_off.push_back(mirror_bytes);
            mirror_bytes += (slabs[k].bytes + 255ull) & ~255ull;
            sig.emplace_back(M.base.back(), slabs[k].bytes);
        }
    } catch (...) { return BMB200_ERR_BADALLOC; }
    *bytes_out = mirror_bytes; *mirror_out = nullptr;
    if (M.base.empty() || mirror_bytes > (128ull << 30)) return BMB200_OK;         // caller falls back to host packing
    CU(cudaSetDevice(ctx->device));
    uint8_t* mirror = nullptr;
    int rc = pool_dev(ctx, kDevSlabMirror, mirror_bytes + mirror_bytes / 16 + 64, (void**)&mirror);      // headroom: a heap that grew by a slab does not force a re-allocation
    if (rc) return rc;
    *mirror_out = mirror;
    if (ctx->mirror_live && ctx->mirror_sig == sig) { ctx->mirror_live = false; return BMB200_OK; }      // prefetched by bmb200_host_slabs_prefetch
    cudaError_t e = cudaSuccess;
    for (size_t k = 0; k < M.base.size() && e == cudaSuccess; ++k)
        e = cudaMemcpyAsync(mirror + M.dev_off[k], (const void*)(uintptr_t)M.base[k], M.end[k] - M.base[k], cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) { cudaStreamSynchronize(ctx->stream); ctx->last_err = std::string("slab mirror: ") + cudaGetErrorString(e); return BMB200_ERR_CUDA; }
    ctx->mirror_sig.swap(sig);
    return BMB200_OK;
}

int bmb200_host_slabs_prefetch(bmb200_ctx* ctx, const bmb200_host_slab* slabs, uint32_t n_slabs)
{
    if (!ctx || (n_slabs && !slabs)) return BMB200_ERR_BADARG;
    SlabMap M; uint8_t* mirror = nullptr; uint64_t bytes = 0;
    ctx->mirror_live = false;
    int rc = mirror_begin(ctx, slabs, n_slabs, M, &mirror, &bytes);
    if (!rc && mirror) ctx->mirror_live = true;
    return rc;
}

int bmb200_set_upload_slabs(bmb200_ctx* ctx, uint32_t n_vec, uint32_t n_blocks, const bmb200_vec_blocks* vecs,
                            const bmb200_host_slab* slabs, uint32_t n_slabs, bmb200_set** out)
{
    if (!ctx || !vecs || !out || !n_vec || !n_blocks || (n_slabs && !slabs)) return BMB200_ERR_BADARG;
    for (uint32_t v = 0; v < n_vec; ++v)
        if (vecs[v].n_blocks > n_blocks || (vecs[v].n_blocks && (!vecs[v].kind || !vecs[v].ptr))) return BMB200_ERR_BADARG;
    PhaseTrace tr("set_upload_slabs", ctx->stream);
    // 1. the slabs start crossing PCIe now (unless a prefetch already started them); everything the host has to do happens underneath
    SlabMap M;
    uint64_t mirror_bytes = 0;
    uint8_t* mirror = nullptr;
    int rc = mirror_begin(ctx, slabs, n_slabs, M, &mirror, &mirror_bytes);
    ctx->mirror_live = false;
    if (rc) return rc;
    if (!mirror) return bmb200_set_upload_vectors(ctx, n_vec, n_blocks, vecs, out);
    cudaStream_t st = ctx->stream;
    cudaError_t e = cudaSuccess;
    if (tr.on) fprintf(stderr, "[bmb200] set_upload_slabs: %zu slabs, %.1f MB queued for DMA\n", M.base.size(), mirror_bytes / 1048576.0);
    // 2. layout (descriptors, prefix sums) + where every block sits in the mirror
    PackLayout L;
    uint32_t* h_src = nullptr;
    bool inside = false;
    try {
        pack_layout(n_vec, n_blocks, vecs, (unsigned)ctx->host_threads, L);
        if (!L.rc && !(rc = pool_host(ctx, kHostSlabSrc, (size_t)n_vec * n_blocks * 4, (void**)&h_src)))
            inside = pack_sources(n_vec, n_blocks, vecs, L, M, (unsigned)ctx->host_threads, h_src);
    } catch (...) { rc = BMB200_ERR_BADALLOC; }
    if (L.rc || rc || !inside) {
        cudaStreamSynchronize(st);                                  // the DMAs read caller memory: let them finish, then take the other road
        if (L.rc) return L.rc;
        if (rc) return rc;
        return bmb200_set_upload_vectors(ctx, n_vec, n_blocks, vecs, out);
    }
    const uint64_t n_bit = L.bb[n_blocks], n_gap = L.gb[n_blocks];
    bmb200_set* s = nullptr;
    if ((rc = set_alloc(ctx, n_vec, n_blocks, n_bit, n_gap, &s))) { cudaStreamSynchronize(st); return rc; }
    uint32_t* d_src = nullptr;
    if ((rc = pool_dev(ctx, kDevSlabSrc, (size_t)n_vec * n_blocks * 4, (void**)&d_src))) { cudaStreamSynchronize(st); free_set_arrays(s); delete s; return rc; }
    e = cudaMemcpyAsync(d_src, h_src, (size_t)n_vec * n_blocks * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync((void*)s->v.desc, L.desc.data(), L.desc.size() * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync((void*)s->v.bit_base, L.bb.data(), L.bb.size() * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync((void*)s->v.gap_base, L.gb.data(), L.gb.size() * 8, cudaMemcpyHostToDevice, st);
    tr.mark("tree layout + source table under the DMA, then their H2D");
    // 3. mirror -> column-major arena
    if (e == cudaSuccess) {
        uint32_t grid = (uint32_t)ctx->sm_count * 8u; if (grid > n_blocks) grid = n_blocks;
        slab_gather_kernel<<<grid, 256, 0, st>>>(s->v, mirror, d_src);
        rc = after_launch(ctx);
        e = cudaStreamSynchronize(st);                              // L / h_src are host memory of this call
    }
    if (e != cudaSuccess || rc) {
        cudaStreamSynchronize(st);
        if (e != cudaSuccess) { ctx->last_err = std::string("set_upload_slabs: ") + cudaGetErrorString(e); rc = BMB200_ERR_CUDA; }
        free_set_arrays(s); delete s;
        return rc;
    }
    tr.mark("gather kernel (mirror -> arena)");
    *out = s;
    return BMB200_OK;
}

/* ---- deserialize-to-device: host side = token walk only (type + payload extent of every block), no decoding ---- */
namespace {

struct ByteRd {
    const uint8_t* b; uint64_t n, p = 0; bool bad = false;
    uint32_t u8()  { if (p + 1 > n) { bad = true; return 0; } return b[p++]; }
    uint32_t u16() { uint32_t a = u8(); return a | (u8() << 8); }
    uint32_t u32() { uint32_t a = u16(); return a | (u16() << 16); }
    void skip(uint64_t k) { if (p + k > n) bad = true; else p += k; }
};

// walks one serialized bvector (src/bmserial.h:5578-6090 token loop); appends one BlobTok per BIT / GAP block, marks FULL blocks
int walk_blob(const uint8_t* blob, uint64_t size, uint32_t n_blocks, std::vector<BlobTok>& toks, std::vector<uint8_t>& full)
{
    ByteRd r{blob, size};
    const uint32_t hf = r.u8();
    if (!(hf & (1u << 3))) r.u8();                                 // byte order
    if (hf & ((1u << 2) | (1u << 6))) return BMB200_ERR_UNSUPPORTED;               // id list / XOR compression
    if (!(hf & (1u << 4))) r.skip(8);                              // GAP levels
    if (hf & (1u << 1)) { r.u32(); if (hf & (1u << 5)) r.u32(); }  // size (64-bit in a BM64ADDR stream)
    uint64_t nb = 0;
    auto ones = [&](uint64_t cnt) { for (uint64_t c = nb; c < nb + cnt && c < n_blocks; ++c) full[c] = 1; nb += cnt; };
    while (!r.bad) {
        const uint32_t bt = r.u8();
        if (r.bad) return BMB200_ERR_BADARG;
        if (bt & 0x80u) { nb += bt & 0x7fu; continue; }
        BlobTok t{}; t.nb = (uint32_t)nb; t.off = r.p; bool blk = true;
        switch (bt) {
        case 0: case 9: return BMB200_OK;                          // set_block_end / set_block_azero
        case 1: blk = false; break;
        case 3: nb += r.u8(); continue;
        case 5: nb += r.u16(); continue;
        case 7: nb += r.u32(); continue;
        case 25: { uint64_t c = r.u32(); c |= (uint64_t)r.u32() << 32; nb += c; continue; }       // set_block_64zero (BM64ADDR streams)
        case 10: ones(nb < n_blocks ? n_blocks - nb : 0); return BMB200_OK;
        case 2: ones(1); continue;
        case 4: ones(r.u8()); continue;
        case 6: ones(r.u16()); continue;
        case 8: ones(r.u32()); continue;
        case 26: { uint64_t c = r.u32(); c |= (uint64_t)r.u32() << 32; ones(c); continue; }       // set_block_64one
        case 11: t.type = DB_BIT; t.kind = BMB200_BLK_BIT; r.skip(BMB200_BLOCK_BYTES); break;
        case 17: { const uint32_t head = r.u16(), tail = r.u16(); if (tail >= BMB200_BLOCK_WORDS || head > tail) return BMB200_ERR_BADARG;
                   t.type = DB_BIT_INTERVAL; t.kind = BMB200_BLK_BIT; r.skip(4ull * (tail - head + 1)); break; }
        case 22: { uint32_t rt = r.u8(), j = 0;
                   while (j < BMB200_BLOCK_WORDS && !r.bad) { const uint32_t len = r.u16(); if (rt) r.skip(4ull * len); j += len; rt ^= 1u; }
                   if (j != BMB200_BLOCK_WORDS) return BMB200_ERR_BADARG;
                   t.type = DB_BIT_0RUNS; t.kind = BMB200_BLK_BIT; break; }
        case 34: { uint64_t d0 = r.u32(); d0 |= (uint64_t)r.u32() << 32; t.type = DB_BIT_DIGEST0; t.kind = BMB200_BLK_BIT;
                   r.skip(128ull * (uint64_t)__builtin_popcountll(d0)); break; }
        case 16: case 30: { const uint32_t n = r.u16(); t.type = bt == 16 ? DB_ARRBIT : DB_ARRBIT_INV; t.kind = BMB200_BLK_BIT; r.skip(2ull * n); break; }
        case 14: case 15: { const uint32_t hdr = r.u16(), len = hdr >> 3; if (len < 1 || len > BMB200_GAP_MAX_WORDS - 5) return BMB200_ERR_UNSUPPORTED;
                   t.type = DB_GAP16; t.kind = BMB200_BLK_GAP; t.first = hdr & 1u; t.gap_words = len + 1; r.skip(2ull * (len - 1)); break; }
        case 19: { const uint32_t pos = r.u16(); t.type = DB_ARRGAP; t.kind = BMB200_BLK_GAP; t.aux = 1; t.off = r.p - 2;
                   t.first = pos == 0; t.gap_words = 4; break; }
        case 18: case 24: { const uint32_t n = r.u16(); if (!n || n > 2048u) return BMB200_ERR_UNSUPPORTED;
                   const uint64_t a0 = r.p; r.skip(2ull * n); if (r.bad) return BMB200_ERR_BADARG;
                   const uint32_t first_pos = blob[a0] | ((uint32_t)blob[a0 + 1] << 8);
                   t.type = bt == 18 ? DB_ARRGAP : DB_ARRGAP_INV; t.kind = BMB200_BLK_GAP; t.aux = n; t.off = a0;
                   t.first = (first_pos == 0) ^ (bt == 24); t.gap_words = arrgap_measure(blob + a0, n);
                   if (!t.gap_words) return BMB200_ERR_BADARG; break; }
        case 67: {   // set_block_gap_egamma_v3: bit stream of 32-bit words, LSB first: gamma(len-1), start bit, use_gamma bit, values
                   const uint64_t w0 = r.p; uint64_t acc = 0; uint32_t have = 0, used = 0, zeros = 0;
                   auto need = [&](uint32_t nbits) { while (have < nbits && !r.bad) { acc |= (uint64_t)r.u32() << have; have += 32; } };
                   for (;;) { need(1); if (r.bad || (acc & 1ull)) break; acc >>= 1; --have; ++used; if (++zeros > 31) break; }
                   if (r.bad || zeros > 31) return BMB200_ERR_BADARG;
                   acc >>= 1; --have; ++used;
                   uint32_t v = 0; if (zeros) { need(zeros); v = (uint32_t)(acc & ((1ull << zeros) - 1)); acc >>= zeros; have -= zeros; used += zeros; }
                   const uint32_t len = (v | (1u << zeros)) + 1u;
                   need(2); const uint32_t start = acc & 1u, use_gamma = (acc >> 1) & 1u; used += 2;
                   if (use_gamma || len > BMB200_GAP_MAX_WORDS - 5) return BMB200_ERR_UNSUPPORTED;
                   const uint64_t total_bits = (uint64_t)used + 16ull * (len - 1);
                   r.p = w0; r.skip(4ull * ((total_bits + 31) / 32));
                   t.type = DB_GAP_V3; t.kind = BMB200_BLK_GAP; t.off = w0; t.aux = used | (len << 8); t.first = start; t.gap_words = len + 1; break; }
        default: return BMB200_ERR_UNSUPPORTED;
        }
        if (r.bad) return BMB200_ERR_BADARG;
        if (blk && nb < n_blocks) toks.push_back(t);
        ++nb;
    }
    return BMB200_ERR_BADARG;       // ran off the end without an end token
}
}  // namespace

int bmb200_set_upload_blobs(bmb200_ctx* ctx, uint32_t n_vec, uint32_t n_blocks, const bmb200_blob* blobs, bmb200_set** out)
{
    if (!ctx || !blobs || !out || !n_vec || !n_blocks) return BMB200_ERR_BADARG;
    for (uint32_t v = 0; v < n_vec; ++v) if (!blobs[v].data || blobs[v].size < 2) return BMB200_ERR_BADARG;
    std::vector<std::vector<BlobTok>> toks(n_vec);
    std::vector<uint8_t> full;
    std::vector<uint32_t> desc; std::vector<uint64_t> bb, gb, stg_off(n_vec), blob_size(n_vec);
    std::vector<BlobRec> recs, erecs;           // explicit-length tokens (blob_decode_kernel) / entropy-coded tokens (blob_entropy_kernel)
    bool device_walk = false;                   // some BLOB holds entropy-coded tokens: its stream can only be walked by decoding it
    PhaseTrace tr("set_upload_blobs", ctx->stream);
    uint64_t stg_bytes = 0;
    try {
        full.assign((size_t)n_vec * n_blocks, 0);
        std::vector<uint8_t> fv(n_blocks);
        for (uint32_t v = 0; v < n_vec; ++v) {
            stg_off[v] = stg_bytes; blob_size[v] = blobs[v].size; stg_bytes += (blobs[v].size + 15ull) & ~15ull;
            if (device_walk) continue;
            std::fill(fv.begin(), fv.end(), 0);
            int rc = walk_blob((const uint8_t*)blobs[v].data, blobs[v].size, n_blocks, toks[v], fv);
            if (rc == BMB200_ERR_UNSUPPORTED) { device_walk = true; continue; }
            if (rc) return rc;
            for (uint32_t nb = 0; nb < n_blocks; ++nb) full[(size_t)nb * n_vec + v] = fv[nb];
        }
    } catch (...) { return BMB200_ERR_BADALLOC; }
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    tr.mark(device_walk ? "host walk (gave up: entropy)" : "host token walk");
    // ---- the compressed bytes are all that crosses PCIe (plus descriptors and the token table): gathered into one pinned
    // buffer so the copy is a single DMA at link speed instead of one pageable copy per vector
    uint8_t* d_stg = nullptr; BlobRec *d_recs = nullptr, *d_erecs = nullptr;
    uint64_t *d_boff = nullptr, *d_bsize = nullptr; BlobTok* d_toks = nullptr; uint32_t* d_ntoks = nullptr; int* d_status = nullptr;
    uint8_t *d_full = nullptr, *d_scratch = nullptr, *h_stg = nullptr;
    bmb200_set* s = nullptr;
    // temporaries live in the context's grow-only pools (the kDevBlob* slots and kHostBlobStage); the stream is synchronized before
    // this function returns, so the next call may reuse them
    auto fail = [&](int rc, cudaError_t e) {
        cudaStreamSynchronize(st);
        if (e != cudaSuccess && (!rc || rc == BMB200_ERR_CUDA)) { ctx->last_err = std::string("set_upload_blobs: ") + cudaGetErrorString(e); rc = BMB200_ERR_CUDA; }
        if (s) { free_set_arrays(s); delete s; }
        return rc;
    };
    int rc = pool_dev(ctx, kDevBlobStage, stg_bytes + 64, (void**)&d_stg);
    if (!rc) rc = pool_host(ctx, kHostBlobStage, stg_bytes, (void**)&h_stg);
    if (rc) return fail(rc, cudaSuccess);
    cudaError_t e = cudaMemsetAsync(d_stg + stg_bytes, 0, 64, st);
    if (e == cudaSuccess) {
        cudaStreamSynchronize(st);                     // a previous call may still be reading the staging buffer
        for (uint32_t v = 0; v < n_vec; ++v) memcpy(h_stg + stg_off[v], blobs[v].data, blobs[v].size);
        e = cudaMemcpyAsync(d_stg, h_stg, stg_bytes, cudaMemcpyHostToDevice, st);
    }
    if (e != cudaSuccess) return fail(BMB200_ERR_CUDA, e);
    tr.mark("stage + H2D of BLOB bytes");
    const uint32_t ent_grid_max = (uint32_t)ctx->sm_count * 8u;       // warps that decode at the same time (one scratch slot each)
    uint32_t n_status = 0;                                             // d_status[n_status] = status word of pass 2
    EntSeg* d_segs = nullptr; uint32_t* d_segcap = nullptr;
    if (device_walk) {
        // ---- pass 1 on the device: one warp per segment (a whole vector, or one bookmark interval of it) walks -- and, for
        // entropy-coded tokens, decodes -- its piece of the token stream
        std::vector<EntSeg> segs; std::vector<uint32_t> seg_cap;
        uint64_t tok_total = 0;
        try {
            for (uint32_t v = 0; v < n_vec; ++v) {
                const size_t first = segs.size();
                rc = ent_find_segments((const uint8_t*)blobs[v].data, blobs[v].size, v, stg_off[v], segs);
                if (rc) return fail(rc, cudaSuccess);
                for (size_t k = first; k < segs.size(); ++k) {            // token slots: one per block the segment can reach (+ super-block records)
                    const uint64_t lo = std::min<uint64_t>(segs[k].nb0, n_blocks);
                    const uint64_t hi = (k + 1 < segs.size()) ? std::min<uint64_t>(std::max<uint64_t>(segs[k + 1].nb0, segs[k].nb0), n_blocks) : n_blocks;
                    const uint64_t cap = (hi - lo) + (hi - lo) / 256u + 2u;
                    segs[k].tok_base = (uint32_t)tok_total; seg_cap.push_back((uint32_t)cap); tok_total += cap;
                    if (tok_total > 0xfffffff0ull) return fail(BMB200_ERR_RANGE, cudaSuccess);
                }
            }
        } catch (...) { return fail(BMB200_ERR_BADALLOC, cudaSuccess); }
        const uint32_t n_segs = (uint32_t)segs.size();
        const uint32_t grid = std::min(n_segs, ent_grid_max);
        if ((rc = pool_dev(ctx, kDevBlobOff, 8ull * n_vec, (void**)&d_boff)) ||
            (rc = pool_dev(ctx, kDevBlobSize, 8ull * n_vec, (void**)&d_bsize)) ||
            (rc = pool_dev(ctx, kDevBlobToks, sizeof(BlobTok) * (size_t)tok_total, (void**)&d_toks)) ||
            (rc = pool_dev(ctx, kDevBlobNToks, 4ull * n_segs, (void**)&d_ntoks)) ||
            (rc = pool_dev(ctx, kDevBlobStatus, 4ull * (n_segs + 3), (void**)&d_status)) ||
            (rc = pool_dev(ctx, kDevBlobFull, (size_t)n_vec * n_blocks, (void**)&d_full)) ||
            (rc = pool_dev(ctx, kDevBlobScratch, (size_t)ent_grid_max * kEntScratchBytes, (void**)&d_scratch)) ||
            (rc = pool_dev(ctx, kDevBlobSegs, sizeof(EntSeg) * (size_t)n_segs, (void**)&d_segs)) ||
            (rc = pool_dev(ctx, kDevBlobSegCap, 8ull * n_segs, (void**)&d_segcap)))           // capacities, then the processing order
            return fail(rc, cudaSuccess);
        e = cudaMemcpyAsync(d_boff, stg_off.data(), 8ull * n_vec, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_bsize, blob_size.data(), 8ull * n_vec, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_segs, segs.data(), sizeof(EntSeg) * (size_t)n_segs, cudaMemcpyHostToDevice, st);
        std::vector<uint32_t> order(n_segs);                              // longest stream first (the launch ends with its slowest warp)
        for (uint32_t k = 0; k < n_segs; ++k) order[k] = k;
        auto seg_len = [&](uint32_t k) { return (segs[k].bounded ? segs[k].end : segs[k].blob_size) - segs[k].start; };
        std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return seg_len(a) > seg_len(b); });
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_segcap, seg_cap.data(), 4ull * n_segs, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_segcap + n_segs, order.data(), 4ull * n_segs, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_full, 0, (size_t)n_vec * n_blocks, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_status, 0, 4ull * (n_segs + 3), st);
        if (e != cudaSuccess) return fail(BMB200_ERR_CUDA, e);
        tr.mark("walk buffers");
        blob_walk_kernel<<<grid, kEntThreads, 0, st>>>(d_stg, d_segs, d_segcap, d_segcap + n_segs, (uint32_t*)d_status + n_segs + 1, n_segs, n_vec, n_blocks, d_toks,
                                                       d_ntoks, d_status, d_full, d_scratch);
        if ((rc = after_launch(ctx))) return fail(rc, cudaGetLastError());
        tr.mark("blob_walk_kernel");
        std::vector<uint32_t> ntoks; std::vector<int> status; std::vector<BlobTok> all;
        try { ntoks.resize(n_segs); status.resize(n_segs); all.resize(tok_total); } catch (...) { return fail(BMB200_ERR_BADALLOC, cudaSuccess); }
        e = cudaMemcpyAsync(ntoks.data(), d_ntoks, 4ull * n_segs, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(status.data(), d_status, 4ull * n_segs, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(full.data(), d_full, (size_t)n_vec * n_blocks, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess && tok_total) e = cudaMemcpyAsync(all.data(), d_toks, sizeof(BlobTok) * (size_t)tok_total, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return fail(BMB200_ERR_CUDA, e);
        for (uint32_t k = 0; k < n_segs; ++k) if (status[k]) return fail(status[k], cudaSuccess);
        try {
            for (uint32_t v = 0; v < n_vec; ++v) toks[v].clear();
            for (uint32_t k = 0; k < n_segs; ++k) {                       // segments are in stream order per vector: concatenate
                if (ntoks[k] > seg_cap[k]) return fail(BMB200_ERR_RANGE, cudaSuccess);
                std::vector<BlobTok>& tv = toks[segs[k].vec];
                tv.insert(tv.end(), all.begin() + segs[k].tok_base, all.begin() + segs[k].tok_base + ntoks[k]);
            }
        } catch (...) { return fail(BMB200_ERR_BADALLOC, cudaSuccess); }
        n_status = n_segs;
    }
    tr.mark("token table D2H");
    // ---- arena layout: per column in vector order; the tokens of one vector are already in block order
    try {
        desc.assign((size_t)n_vec * n_blocks, 0u); bb.assign((size_t)n_blocks + 1, 0); gb.assign((size_t)n_blocks + 1, 0);
        std::vector<size_t> cur(n_vec, 0);
        for (uint32_t nb = 0; nb < n_blocks; ++nb) {
            uint64_t nbit = 0, ngap = 0;
            for (uint32_t v = 0; v < n_vec; ++v) {
                uint32_t d = full[(size_t)nb * n_vec + v] ? BMB200_BLK_FULL : BMB200_BLK_NULL;
                // a super-block token precedes its member blocks: one rec for the whole token, no slot of its own
                while (cur[v] < toks[v].size() && toks[v][cur[v]].type == (kTokEntropy | 68u) && toks[v][cur[v]].nb <= nb) {
                    const BlobTok& t = toks[v][cur[v]++];
                    BlobRec r{}; r.src = stg_off[v] + t.off; r.type = t.type; r.aux = v; r.dst = t.aux;
                    size_t k = cur[v]; while (k < toks[v].size() && toks[v][k].off == t.off) ++k;      // its member blocks share its offset
                    const uint64_t nxt = k < toks[v].size() ? toks[v][k].off : blob_size[v];
                    r.aux2 = (uint32_t)std::min<uint64_t>(nxt > t.off ? nxt - t.off : 0, 0x3fffffffu) << 2;
                    erecs.push_back(r);
                }
                if (cur[v] < toks[v].size() && toks[v][cur[v]].nb == nb) {
                    const BlobTok& t = toks[v][cur[v]++];
                    const bool entropy = (t.type & kTokEntropy) != 0, member = (t.type == kTokSbMember);
                    BlobRec r{}; r.src = stg_off[v] + t.off; r.type = t.type; r.aux = entropy ? v : t.aux; r.kind = t.kind;
                    if (t.kind == BMB200_BLK_BIT) { d = BMB200_BLK_BIT | ((uint32_t)nbit << 2); r.dst = bb[nb] + nbit; ++nbit; }
                    else if (t.kind == BMB200_BLK_GAP) {
                        if (t.gap_words < 2u || t.gap_words > BMB200_GAP_MAX_WORDS) return fail(BMB200_ERR_BADARG, cudaSuccess);
                        const uint32_t pad = t.first ? 0u : 1u;
                        const uint64_t units = (t.gap_words + pad + kGapUnit - 1) / kGapUnit;
                        if (ngap + units > (uint64_t)BMB200_DESC_REL_MASK) return fail(BMB200_ERR_RANGE, cudaSuccess);
                        d = BMB200_BLK_GAP | ((uint32_t)ngap << 2) | (pad ? BMB200_DESC_GAP_PAD : 0u) | BMB200_DESC_GAP_FLAT;
                        r.dst = gb[nb] + ngap; r.aux2 = pad | (t.first << 1) | (entropy ? 0u : t.gap_words << 8); ngap += units;
                    } else return fail(BMB200_ERR_BADARG, cudaSuccess);
                    if (entropy) {      // payload length (to the next record of the vector, or the end of the BLOB): the work estimate pass 2 is sorted by
                        const uint64_t nxt = cur[v] < toks[v].size() ? toks[v][cur[v]].off : blob_size[v];
                        r.aux2 |= (uint32_t)std::min<uint64_t>(nxt > t.off ? nxt - t.off : 0, 0x3fffffffu) << 2;
                    }
                    if (!member) (entropy ? erecs : recs).push_back(r);
                }
                desc[(size_t)nb * n_vec + v] = d;
            }
            bb[nb + 1] = bb[nb] + nbit; gb[nb + 1] = gb[nb] + ngap;
        }
        // every record must have found its column: block indexes that go backwards (a bookmark chain that lies) are a format error
        for (uint32_t v = 0; v < n_vec; ++v) if (cur[v] != toks[v].size()) return fail(BMB200_ERR_BADARG, cudaSuccess);
    } catch (...) { return fail(BMB200_ERR_BADALLOC, cudaSuccess); }
    const uint64_t n_bit = bb[n_blocks], n_gap = gb[n_blocks];
    std::stable_sort(erecs.begin(), erecs.end(), [](const BlobRec& a, const BlobRec& b) { return (a.aux2 >> 2) > (b.aux2 >> 2); });
    tr.mark("arena layout (host)");
    rc = set_alloc(ctx, n_vec, n_blocks, n_bit, n_gap, &s);
    if (rc) { s = nullptr; return fail(rc, cudaSuccess); }
    if ((!recs.empty() && (rc = pool_dev(ctx, kDevBlobRecs, recs.size() * sizeof(BlobRec), (void**)&d_recs))) ||
        (!erecs.empty() && (rc = pool_dev(ctx, kDevBlobERecs, erecs.size() * sizeof(BlobRec), (void**)&d_erecs))))
        return fail(rc, cudaSuccess);
    if (!recs.empty()) e = cudaMemcpyAsync(d_recs, recs.data(), recs.size() * sizeof(BlobRec), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && !erecs.empty()) e = cudaMemcpyAsync(d_erecs, erecs.data(), erecs.size() * sizeof(BlobRec), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync((void*)s->v.desc, desc.data(), desc.size() * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync((void*)s->v.bit_base, bb.data(), bb.size() * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync((void*)s->v.gap_base, gb.data(), gb.size() * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && n_gap) e = cudaMemsetAsync((void*)s->v.gap_pool, 0, n_gap * 16ull, st);   // fill + holes of the FLAT form
    if (e != cudaSuccess) return fail(BMB200_ERR_CUDA, e);
    tr.mark("set alloc + tables H2D");
    if (!recs.empty()) {
        uint32_t grid = (uint32_t)std::min<size_t>(recs.size(), (size_t)ctx->sm_count * 16u);
        blob_decode_kernel<<<grid, kBlobThreads, 0, st>>>(d_stg, d_recs, (uint32_t)recs.size(), (uint32_t*)s->v.bit_pool, (uint16_t*)s->v.gap_pool);
        if ((rc = after_launch(ctx))) return fail(rc, cudaGetLastError());
        tr.mark("blob_decode_kernel");
    }
    int ent_status = 0;
    if (!erecs.empty()) {
        // ---- pass 2: every entropy-coded token of every vector in parallel (their offsets are known now), one warp per token
        uint32_t grid = (uint32_t)std::min<size_t>(erecs.size(), (size_t)ent_grid_max);
        SetView sv{n_vec, n_blocks, s->v.desc, s->v.bit_base, s->v.gap_base, s->v.bit_pool, s->v.gap_pool};
        unsigned long long* d_dur = nullptr;
        if (tr.on && (rc = pool_dev(ctx, kDevBlobDur, 8ull * erecs.size(), (void**)&d_dur))) return fail(rc, cudaSuccess);
        blob_entropy_kernel<<<grid, kEntThreads, 0, st>>>(d_stg, d_boff, d_bsize, d_erecs, (uint32_t)erecs.size(), (uint32_t*)d_status + n_status + 2, sv, (uint32_t*)s->v.bit_pool,
                                                          (uint16_t*)s->v.gap_pool, d_status + n_status, d_scratch, d_dur);
        if ((rc = after_launch(ctx))) return fail(rc, cudaGetLastError());
        if (tr.on) {                                   // the five slowest work items of pass 2
            std::vector<unsigned long long> dur(erecs.size());
            if (cudaMemcpyAsync(dur.data(), d_dur, 8ull * erecs.size(), cudaMemcpyDeviceToHost, st) == cudaSuccess && cudaStreamSynchronize(st) == cudaSuccess) {
                std::vector<uint32_t> idx(erecs.size()); for (uint32_t k = 0; k < idx.size(); ++k) idx[k] = k;
                std::partial_sort(idx.begin(), idx.begin() + std::min<size_t>(5, idx.size()), idx.end(), [&](uint32_t a, uint32_t b) { return dur[a] > dur[b]; });
                unsigned long long sum = 0; for (auto d : dur) sum += d;
                fprintf(stderr, "[bmb200] set_upload_blobs: pass 2: %zu items, %.1f Mclk in total\n", erecs.size(), sum / 1e6);
                for (size_t k = 0; k < std::min<size_t>(5, idx.size()); ++k)
                    fprintf(stderr, "[bmb200]   item %u: token %u, vector %u, payload %u B, kind %u, %.2f Mclk\n", idx[k], erecs[idx[k]].type & 0xffu, erecs[idx[k]].aux,
                            erecs[idx[k]].aux2 >> 2, erecs[idx[k]].kind, dur[idx[k]] / 1e6);
            }
        }
        e = cudaMemcpyAsync(&ent_status, d_status + n_status, 4, cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) return fail(BMB200_ERR_CUDA, e);
    }
    e = cudaStreamSynchronize(st);      // recs / desc staging vectors go out of scope
    if (e != cudaSuccess) return fail(BMB200_ERR_CUDA, e);
    if (ent_status) return fail(ent_status, cudaSuccess);
    tr.mark("blob_entropy_kernel + sync");
    *out = s;
    return BMB200_OK;
}

int bmb200_set_adopt_device(bmb200_ctx* ctx, const bmb200_packed_set* d, bmb200_set** out)
{
    if (!ctx || !d || !out || !d->n_vec || !d->n_blocks || !d->desc || !d->bit_base || !d->gap_base) return BMB200_ERR_BADARG;
    CU(cudaSetDevice(ctx->device));
    bmb200_set* s = new (std::nothrow) bmb200_set();
    if (!s) return BMB200_ERR_BADALLOC;
    s->ctx = ctx; s->owns = false;
    s->v.n_vec = d->n_vec; s->v.n_blocks = d->n_blocks;
    s->v.desc = d->desc; s->v.bit_base = d->bit_base; s->v.gap_base = d->gap_base;
    s->v.bit_pool = d->bit_pool; s->v.gap_pool = d->gap_pool;
    uint64_t tails[2] = {0, 0};
    cudaError_t e1 = cudaMemcpyAsync(&tails[0], d->bit_base + d->n_blocks, 8, cudaMemcpyDeviceToHost, ctx->stream);
    cudaError_t e2 = cudaMemcpyAsync(&tails[1], d->gap_base + d->n_blocks, 8, cudaMemcpyDeviceToHost, ctx->stream);
    cudaError_t e3 = cudaStreamSynchronize(ctx->stream);
    if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess) { delete s; ctx->last_err = "adopt: cannot read bases"; return BMB200_ERR_CUDA; }
    s->n_bit_blocks = tails[0]; s->n_gap_units = tails[1];
    s->gap_pool_bytes = tails[1] * 16ull;      // no slack known for adopted memory
    *out = s;
    return BMB200_OK;
}

int bmb200_set_info(const bmb200_set* s, uint32_t* n_vec, uint32_t* n_blocks, uint64_t* n_bit_blocks, uint64_t* n_gap_units)
{
    if (!s) return BMB200_ERR_BADARG;
    if (n_vec) *n_vec = s->v.n_vec;
    if (n_blocks) *n_blocks = s->v.n_blocks;
    if (n_bit_blocks) *n_bit_blocks = s->n_bit_blocks;
    if (n_gap_units) *n_gap_units = s->n_gap_units;
    return BMB200_OK;
}

static int set_col_bases(const bmb200_set* s, uint32_t nb_from, uint32_t nb_to, uint64_t b[2], uint64_t g[2])
{
    bmb200_ctx* ctx = s->ctx;
    CU(cudaSetDevice(ctx->device));
    CU(cudaMemcpyAsync(&b[0], s->v.bit_base + nb_from, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(&b[1], s->v.bit_base + nb_to, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(&g[0], s->v.gap_base + nb_from, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(&g[1], s->v.gap_base + nb_to, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return BMB200_OK;
}

int bmb200_set_column_sizes(const bmb200_set* s, uint32_t nb_from, uint32_t nb_to, uint64_t* n_bit_blocks, uint64_t* n_gap_units)
{
    if (!s) return BMB200_ERR_BADARG;
    if (nb_from > nb_to || nb_to > s->v.n_blocks) return BMB200_ERR_RANGE;
    uint64_t b[2], g[2];
    int rc = set_col_bases(s, nb_from, nb_to, b, g);
    if (rc) return rc;
    if (n_bit_blocks) *n_bit_blocks = b[1] - b[0];
    if (n_gap_units) *n_gap_units = g[1] - g[0];
    return BMB200_OK;
}

int bmb200_set_download(const bmb200_set* s, uint32_t nb_from, uint32_t nb_to,
                        uint32_t* desc, uint64_t* bit_base, uint64_t* gap_base, uint32_t* bit_pool, uint16_t* gap_pool)
{
    if (!s || !desc || !bit_base || !gap_base) return BMB200_ERR_BADARG;
    if (nb_from > nb_to || nb_to > s->v.n_blocks) return BMB200_ERR_RANGE;
    bmb200_ctx* ctx = s->ctx;
    uint64_t b[2], g[2];
    int rc = set_col_bases(s, nb_from, nb_to, b, g);
    if (rc) return rc;
    const uint32_t nc = nb_to - nb_from;
    if ((b[1] > b[0] && !bit_pool) || (g[1] > g[0] && !gap_pool)) return BMB200_ERR_BADARG;
    CU(cudaMemcpyAsync(desc, s->v.desc + (size_t)nb_from * s->v.n_vec, (size_t)nc * s->v.n_vec * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(bit_base, s->v.bit_base + nb_from, ((size_t)nc + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(gap_base, s->v.gap_base + nb_from, ((size_t)nc + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (b[1] > b[0])
        CU(cudaMemcpyAsync(bit_pool, s->v.bit_pool + b[0] * (size_t)kBlockWords, (size_t)(b[1] - b[0]) * BMB200_BLOCK_BYTES, cudaMemcpyDeviceToHost, ctx->stream));
    if (g[1] > g[0])
        CU(cudaMemcpyAsync(gap_pool, s->v.gap_pool + g[0] * (size_t)kGapUnit, (size_t)(g[1] - g[0]) * kGapUnit * 2, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    for (uint32_t i = 0; i <= nc; ++i) { bit_base[i] -= b[0]; gap_base[i] -= g[0]; }
    return BMB200_OK;
}

int bmb200_set_device_ptrs(const bmb200_set* s, bmb200_packed_set* out)
{
    if (!s || !out) return BMB200_ERR_BADARG;
    out->n_vec = s->v.n_vec; out->n_blocks = s->v.n_blocks;
    out->desc = s->v.desc; out->bit_base = s->v.bit_base; out->gap_base = s->v.gap_base;
    out->bit_pool = s->v.bit_pool; out->gap_pool = s->v.gap_pool;
    return BMB200_OK;
}

int bmb200_set_free(bmb200_set* s)
{
    if (!s) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = s->ctx;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    free_run_lists(s);                                       // derived data: never parked
    if (s->owns && s->cap_desc && !ctx->arena.full) {       // park the arrays for the next upload instead of cudaFree
        auto& a = ctx->arena;
        a.desc = (void*)s->v.desc; a.bb = (void*)s->v.bit_base; a.gb = (void*)s->v.gap_base; a.bp = (void*)s->v.bit_pool; a.gp = (void*)s->v.gap_pool;
        a.cap_desc = s->cap_desc; a.cap_base = s->cap_base; a.cap_bit = s->cap_bit; a.cap_gap = s->cap_gap; a.full = true;
    } else free_set_arrays(s);
    delete s;
    return BMB200_OK;
}

int bmb200_ctx_trim(bmb200_ctx* ctx)
{
    if (!ctx) return BMB200_ERR_BADARG;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    auto& a = ctx->arena;
    if (a.full) { cudaFree(a.desc); cudaFree(a.bb); cudaFree(a.gb); cudaFree(a.bp); cudaFree(a.gp); a = bmb200_ctx::Arena(); }
    for (DevSlot slot : {kDevSlabMirror, kDevSlabSrc})
        if (ctx->d_pool[slot]) { cudaFree(ctx->d_pool[slot]); ctx->d_pool[slot] = nullptr; ctx->d_pool_cap[slot] = 0; }
    return BMB200_OK;
}

int bmb200_synth_set(bmb200_ctx* ctx, uint32_t n_vec, uint32_t n_blocks,
                     const double* density, const uint64_t* seed, int optimize, bmb200_set** out)
{
    if (!ctx || !out || !density || !seed || !n_vec || !n_blocks) return BMB200_ERR_BADARG;
    if ((uint64_t)n_vec * n_blocks > 0x7fffffffull) return BMB200_ERR_RANGE;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    std::vector<uint32_t> thr(n_vec);
    for (uint32_t v = 0; v < n_vec; ++v) {
        double t = density[v] * 65536.0 + 0.5;
        thr[v] = t <= 0 ? 0u : t >= 65536.0 ? 65536u : (uint32_t)t;
    }
    const size_t items = (size_t)n_vec * n_blocks;
    uint64_t* d_seed = nullptr; uint32_t* d_thr = nullptr; uint8_t* d_kind = nullptr; uint16_t* d_glen = nullptr;
    uint64_t *d_cb = nullptr, *d_cg = nullptr;
    uint32_t* desc = nullptr; uint64_t *bb = nullptr, *gb = nullptr;
    int rc = BMB200_OK;
    auto cleanup_tmp = [&]() { cudaFree(d_seed); cudaFree(d_thr); cudaFree(d_kind); cudaFree(d_glen); cudaFree(d_cb); cudaFree(d_cg); };
    if ((rc = dev_alloc(ctx, &d_seed, n_vec)) || (rc = dev_alloc(ctx, &d_thr, n_vec)) ||
        (rc = dev_alloc(ctx, &d_kind, items)) || (rc = dev_alloc(ctx, &d_glen, items)) ||
        (rc = dev_alloc(ctx, &d_cb, n_blocks)) || (rc = dev_alloc(ctx, &d_cg, n_blocks)) ||
        (rc = dev_alloc(ctx, &desc, items)) || (rc = dev_alloc(ctx, &bb, (size_t)n_blocks + 1)) ||
        (rc = dev_alloc(ctx, &gb, (size_t)n_blocks + 1))) {
        cleanup_tmp(); cudaFree(desc); cudaFree(bb); cudaFree(gb); return rc;
    }
    cudaError_t e = cudaMemcpyAsync(d_seed, seed, n_vec * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_thr, thr.data(), n_vec * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        synth_classify_kernel<<<(unsigned)items, kPostThreads, 0, st>>>(n_vec, n_blocks, d_seed, d_thr, optimize, d_kind, d_glen);
        rc = after_launch(ctx);
        if (!rc) { synth_layout_kernel<<<n_blocks, 256, 0, st>>>(n_vec, 1u, d_kind, d_glen, desc, d_cb, d_cg); rc = after_launch(ctx); }
        if (!rc) { scan_u64_kernel<<<1, 1024, 0, st>>>(d_cb, n_blocks, bb); rc = after_launch(ctx); }
        if (!rc) { scan_u64_kernel<<<1, 1024, 0, st>>>(d_cg, n_blocks, gb); rc = after_launch(ctx); }
    }
    if (rc) { cleanup_tmp(); cudaFree(desc); cudaFree(bb); cudaFree(gb); return rc; }
    uint64_t tails[2] = {0, 0};
    if (e == cudaSuccess) e = cudaMemcpyAsync(&tails[0], bb + n_blocks, 8, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&tails[1], gb + n_blocks, 8, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { ctx->last_err = std::string("synth: ") + cudaGetErrorString(e); cleanup_tmp(); cudaFree(desc); cudaFree(bb); cudaFree(gb); return BMB200_ERR_CUDA; }
    uint32_t* bp = nullptr; uint16_t* gp = nullptr;
    if ((rc = dev_alloc(ctx, &bp, (size_t)tails[0] * kBlockWords, kSlack)) ||
        (rc = dev_alloc(ctx, &gp, (size_t)tails[1] * kGapUnit, kSlack))) {
        cleanup_tmp(); cudaFree(desc); cudaFree(bb); cudaFree(gb); cudaFree(bp); cudaFree(gp); return rc;
    }
    cudaMemsetAsync((char*)gp + (size_t)tails[1] * kGapUnit * 2, 0, kSlack, st);
    synth_write_kernel<<<(unsigned)items, kPostThreads, 0, st>>>(n_vec, n_blocks, d_seed, d_thr, desc, bb, gb, bp, gp);
    rc = after_launch(ctx);
    e = cudaStreamSynchronize(st);
    cleanup_tmp();
    if (rc || e != cudaSuccess) {
        if (e != cudaSuccess) ctx->last_err = std::string("synth write: ") + cudaGetErrorString(e);
        cudaFree(desc); cudaFree(bb); cudaFree(gb); cudaFree(bp); cudaFree(gp); return BMB200_ERR_CUDA;
    }
    bmb200_set* s = new (std::nothrow) bmb200_set();
    if (!s) { cudaFree(desc); cudaFree(bb); cudaFree(gb); cudaFree(bp); cudaFree(gp); return BMB200_ERR_BADALLOC; }
    s->ctx = ctx; s->owns = true;
    s->v.n_vec = n_vec; s->v.n_blocks = n_blocks;
    s->v.desc = desc; s->v.bit_base = bb; s->v.gap_base = gb; s->v.bit_pool = bp; s->v.gap_pool = gp;
    s->n_bit_blocks = tails[0]; s->n_gap_units = tails[1];
    s->gap_pool_bytes = tails[1] * 16ull + kSlack;
    *out = s;
    return BMB200_OK;
}

/* ------------------------------------------------------------------ aggregation */

static int result_alloc(bmb200_ctx* ctx, uint32_t n_cols, uint32_t n_groups, bool blocks, bool gaps, bool or_target, bmb200_result** out)
{
    bmb200_result* r = new (std::nothrow) bmb200_result();
    if (!r) return BMB200_ERR_BADALLOC;
    r->ctx = ctx; r->n_cols = n_cols; r->n_groups = n_groups; r->cols_per_group = n_cols / n_groups;
    int rc;
    if (n_groups == 1) {
        const uint32_t n_even = (n_cols + 1u) & ~1u;                     // the 64-bit total sits 8-byte aligned behind the popcounts
        r->xstride = n_even + 2u;
        if ((rc = dev_alloc(ctx, &r->popcnt_base, (size_t)r->xstride * CommState::kSlots))) { delete r; return rc; }
        cudaMemsetAsync(r->popcnt_base, 0, (size_t)r->xstride * CommState::kSlots * 4, ctx->stream);
        r->popcnt = r->popcnt_base; r->total = reinterpret_cast<unsigned long long*>(r->popcnt_base + n_even); r->total_inline = true;
    }
    if ((!r->total_inline && ((rc = dev_alloc(ctx, &r->popcnt, n_cols)) || (rc = dev_alloc(ctx, &r->total, n_groups)))) ||
        (rc = dev_alloc(ctx, &r->digest, n_cols)) ||
        (rc = dev_alloc(ctx, &r->nruns, n_cols)) || (rc = dev_alloc(ctx, &r->kind, n_cols)) ||
        (or_target && (rc = dev_alloc(ctx, &r->or_blocks, (size_t)(n_cols / n_groups) * kBlockWords))) ||
        (blocks && (rc = dev_alloc(ctx, &r->blocks, (size_t)n_cols * kBlockWords))) ||
        (gaps && (rc = dev_alloc(ctx, &r->gaps, (size_t)n_cols * kGapMax)))) {
        free_result_arrays(r); delete r; return rc;
    }
    r->has_blocks = blocks;
    *out = r;
    return BMB200_OK;
}

// dynamic shared memory per aggregation kernel: depends on its static size (the live mask is 8 KB aligned in the shared window)
extern "C++" {
template <typename KFn>
static cudaError_t agg_attr_one(KFn fn, size_t reserved, size_t* dyn_out, size_t ring_bytes = kAggRingSmem)
{
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, fn);
    if (e != cudaSuccess) return e;
    *dyn_out = agg_dyn_smem(fa.sharedSizeBytes, reserved, ring_bytes);
    return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*dyn_out);
}
}
// agg_kernel<op> by op (BMB200_OP_OR .. BMB200_OP_XOR); ctx->agg_dyn is indexed the same way
static void (*const kAggKernels[4])(const AggParams) = {
    agg_kernel<BMB200_OP_OR>, agg_kernel<BMB200_OP_AND>, agg_kernel<BMB200_OP_AND_SUB>, agg_kernel<BMB200_OP_XOR>};

static void set_agg_attrs(bmb200_ctx* ctx, cudaError_t* e)
{
    if (ctx->attr_set) return;
    int reserved = 1024;
    if (cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, ctx->device) != cudaSuccess) { cudaGetLastError(); reserved = 1024; }
    *e = cudaSuccess;
    for (int op = 0; op < 4 && *e == cudaSuccess; ++op) *e = agg_attr_one(kAggKernels[op], (size_t)reserved, &ctx->agg_dyn[op]);
    if (*e == cudaSuccess) *e = agg_attr_one(agg_pipe_kernel, (size_t)reserved, &ctx->pipe_dyn, kPipeRingSmem);
    if (*e == cudaSuccess) ctx->attr_set = true;
}

// agg_kernel<op> on `grid` CTAs with the dynamic shared memory set_agg_attrs sized for it
static void launch_agg_kernel(bmb200_ctx* ctx, int op, uint32_t grid, AggParams& p)
{
    p.dyn_bytes = (uint32_t)ctx->agg_dyn[op];
    kAggKernels[op]<<<grid, kAggThreads, ctx->agg_dyn[op], ctx->stream>>>(p);
}

// The AggParams of a launch that writes result r from set `set`; the caller adds its groups and whatever else differs
static AggParams agg_params(const bmb200_ctx* ctx, const bmb200_set* set, const bmb200_result* r, uint32_t nb_from, uint32_t cols,
                            bool compress, bool store)
{
    AggParams p{};
    p.set = set->v; p.nb_from = nb_from; p.n_cols = cols;
    p.compress = compress ? 1u : 0u; p.store_blocks = store ? 1u : 0u;
    p.blocks = r->blocks; p.popcnt = r->popcnt; p.digest = r->digest; p.nruns = r->nruns; p.kind = r->kind; p.gaps = r->gaps;
    p.total = r->total; p.work_counter = ctx->d_work;
    p.gap_mode = (uint32_t)ctx->gap_mode; p.gap_pool_bytes = set->gap_pool_bytes;
    return p;
}

// Stages the words a[0..na) b[0..nb) into ctx->d_group through the pinned buffer h_group (grown to at least max(1024, n) words) and
// queues their upload.  With `reuse` the words are an aggregate member list: when they equal the list already resident (last_group)
// nothing is uploaded and the stream is not synchronised, otherwise they are recorded as the resident list.  Without it the buffer
// no longer holds member ids.
static int stage_group(bmb200_ctx* ctx, const uint32_t* a, size_t na, const uint32_t* b, size_t nb, bool reuse)
{
    const size_t n = na + nb;
    if (n > ctx->group_cap) {
        cudaStreamSynchronize(ctx->stream);
        cudaFree(ctx->d_group); if (ctx->h_group) cudaFreeHost(ctx->h_group);
        ctx->d_group = nullptr; ctx->h_group = nullptr; ctx->group_cap = 0; ctx->last_group.clear();
        const size_t cap = n < 1024 ? 1024 : n;
        if (cudaMalloc((void**)&ctx->d_group, cap * 4) != cudaSuccess || cudaMallocHost((void**)&ctx->h_group, cap * 4) != cudaSuccess) {
            ctx->last_err = "group buffer allocation"; return BMB200_ERR_BADALLOC;
        }
        ctx->group_cap = cap;
    }
    if (reuse && ctx->last_group.size() == n &&
        (!na || memcmp(ctx->last_group.data(), a, na * 4) == 0) && (!nb || memcmp(ctx->last_group.data() + na, b, nb * 4) == 0))
        return BMB200_OK;
    ctx->last_group.clear();
    cudaError_t e = cudaStreamSynchronize(ctx->stream);     // the staging buffer may still feed a previous launch
    if (e == cudaSuccess) {
        if (na) memcpy(ctx->h_group, a, na * 4);
        if (nb) memcpy(ctx->h_group + na, b, nb * 4);
        e = cudaMemcpyAsync(ctx->d_group, ctx->h_group, n * 4, cudaMemcpyHostToDevice, ctx->stream);
    }
    if (e != cudaSuccess) { ctx->last_err = std::string("group upload: ") + cudaGetErrorString(e); return BMB200_ERR_CUDA; }
    if (reuse) { try { ctx->last_group.assign(ctx->h_group, ctx->h_group + n); } catch (...) { ctx->last_group.clear(); } }
    return BMB200_OK;
}

// agg_pipe_kernel's inputs: one AND-SUB group whose group0 + group1 are every vector of the set exactly once, a set small enough
// for its per-vector role table, and an AND group small enough that its GAP blocks of a column fit the kernel's list
static bool whole_set(const bmb200_batch_args* a, uint32_t n_vec)
{
    if (a->n_groups != 1 || a->op != BMB200_OP_AND_SUB || n_vec == 0 || n_vec > kPipeMaxVec || a->offsets[0] != 0) return false;
    if (a->offsets[1] > kPipeMaxAndGap) return false;
    const uint32_t n = a->offsets[2];
    if (n != n_vec) return false;
    std::vector<bool> seen(n_vec, false);
    for (uint32_t k = 0; k < n; ++k) {
        if (seen[a->members[k]]) return false;
        seen[a->members[k]] = true;
    }
    return true;
}

// Are all GAP blocks of the set in the FLAT form?  Checked once per set on the device (one pass over the descriptors, then a wait
// for the answer) and remembered: a set's descriptors do not change after it is built.
static bool flat_gap_set(bmb200_ctx* ctx, const bmb200_set* set)
{
    bmb200_set* s = const_cast<bmb200_set*>(set);
    if (s->flat_gaps < 0) {
        uint32_t bad = 1u;
        const size_t n = (size_t)set->v.n_vec * set->v.n_blocks;
        const uint32_t grid = (uint32_t)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 8);
        if (cudaMemsetAsync(ctx->d_work + 1, 0, 4, ctx->stream) != cudaSuccess) return false;
        if (grid) desc_flat_check_kernel<<<grid, 256, 0, ctx->stream>>>(set->v.desc, n, ctx->d_work + 1);
        if (cudaMemcpyAsync(&bad, ctx->d_work + 1, 4, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
            cudaStreamSynchronize(ctx->stream) != cudaSuccess) { cudaGetLastError(); return false; }
        s->flat_gaps = bad ? 0 : 1;
    }
    return s->flat_gaps == 1;
}

// Which vectors hold a GAP block in some column: one pass over the descriptors and a wait for the answer, once per set.  Empty on failure.
static const std::vector<uint32_t>& gap_vectors(bmb200_ctx* ctx, const bmb200_set* set)
{
    bmb200_set* s = const_cast<bmb200_set*>(set);
    if (s->gap_vecs.empty()) {
        const uint32_t M = set->v.n_vec, words = (M + 31u) / 32u;
        std::vector<uint32_t> h(words, 0u);
        uint32_t* d = nullptr;
        const dim3 grid((M + 255u) / 256u, std::min(set->v.n_blocks, 256u));
        bool ok = cudaMalloc((void**)&d, words * 4u) == cudaSuccess && cudaMemsetAsync(d, 0, words * 4u, ctx->stream) == cudaSuccess;
        if (ok) { gap_vectors_kernel<<<grid, 256, 0, ctx->stream>>>(set->v.desc, M, set->v.n_blocks, d); ok = cudaGetLastError() == cudaSuccess; }
        ok = ok && cudaMemcpyAsync(h.data(), d, words * 4u, cudaMemcpyDeviceToHost, ctx->stream) == cudaSuccess &&
             cudaStreamSynchronize(ctx->stream) == cudaSuccess;
        cudaFree(d);
        if (ok) s->gap_vecs.swap(h); else cudaGetLastError();
    }
    return s->gap_vecs;
}

// Builds the run-list companion (runlist_kernel.cuh): count pass (which also lists the sparse bit-blocks), scans, one wait to size
// the pools, write pass, then which vectors hold a listed block.  On any failure, or when parts A + B would leave less than
// kRunListMargin of device memory free, the set is marked as having none (rl_state = -1).
constexpr size_t kRunListMargin = size_t(1) << 30;
static bool build_run_lists(bmb200_ctx* ctx, bmb200_set* s)
{
    const uint32_t nb = s->v.n_blocks, M = s->v.n_vec, vwords = (M + 31u) / 32u;
    const size_t lwords = (size_t)(s->n_bit_blocks + 31u) / 32u + 2u;   // + the word the kernel's funnel shift reads past a column
    cudaStream_t st = ctx->stream;
    uint2* wcnt = nullptr; uint64_t *su = nullptr, *lu = nullptr; unsigned long long* tot = nullptr; uint32_t* lv = nullptr;
    uint64_t h_tot[5] = {0, 0, 0, 0, 0};
    std::vector<uint32_t> h_lv(vwords, 0u);
    bool ok = cudaMalloc((void**)&wcnt, (size_t)nb * 2 * kRlWarps * sizeof(uint2)) == cudaSuccess &&
              cudaMalloc((void**)&su, (size_t)nb * 8) == cudaSuccess && cudaMalloc((void**)&lu, (size_t)nb * 8) == cudaSuccess &&
              cudaMalloc((void**)&tot, sizeof(h_tot)) == cudaSuccess && cudaMalloc((void**)&lv, vwords * 4u) == cudaSuccess &&
              cudaMalloc((void**)&s->rl_sgl_base, ((size_t)nb + 1) * 8) == cudaSuccess &&
              cudaMalloc((void**)&s->rl_lr_base, ((size_t)nb + 1) * 8) == cudaSuccess &&
              cudaMalloc((void**)&s->rl_sgl_mid, (size_t)nb * 8) == cudaSuccess && cudaMalloc((void**)&s->rl_lr_mid, (size_t)nb * 8) == cudaSuccess &&
              cudaMalloc((void**)&s->rl_listed, lwords * 4u) == cudaSuccess &&
              cudaMemsetAsync(s->rl_listed, 0, lwords * 4u, st) == cudaSuccess && cudaMemsetAsync(tot, 0, sizeof(h_tot), st) == cudaSuccess &&
              cudaMemsetAsync(lv, 0, vwords * 4u, st) == cudaSuccess;
    if (ok) {
        rl_count_kernel<<<nb, kRlThreads, 0, st>>>(s->v, wcnt, su, lu, s->rl_listed, tot);
        scan_u64_kernel<<<1, 1024, 0, st>>>(su, nb, s->rl_sgl_base);
        scan_u64_kernel<<<1, 1024, 0, st>>>(lu, nb, s->rl_lr_base);
        ok = cudaGetLastError() == cudaSuccess && cudaMemcpyAsync(h_tot, tot, sizeof(h_tot), cudaMemcpyDeviceToHost, st) == cudaSuccess &&
             cudaStreamSynchronize(st) == cudaSuccess;
    }
    const uint64_t sgl_units = h_tot[0] + h_tot[2], lr_units = h_tot[1] + h_tot[3];
    size_t free_b = 0, total_b = 0;
    ok = ok && cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && free_b >= (sgl_units + lr_units) * 16u + kRunListMargin &&
         cudaMalloc((void**)&s->rl_sgl, std::max<uint64_t>(sgl_units, 1u) * 16u) == cudaSuccess &&
         cudaMalloc((void**)&s->rl_lr, std::max<uint64_t>(lr_units, 1u) * 16u) == cudaSuccess;
    if (ok) {
        rl_write_kernel<<<nb, kRlThreads, 0, st>>>(s->v, wcnt, s->rl_sgl_base, s->rl_lr_base, s->rl_listed, s->rl_sgl, s->rl_lr,
                                                   s->rl_sgl_mid, s->rl_lr_mid);
        const dim3 grid((M + 255u) / 256u, std::min(nb, 256u));
        if (h_tot[4]) listed_vectors_kernel<<<grid, 256, 0, st>>>(s->v.desc, s->v.bit_base, s->rl_listed, M, nb, lv);
        ok = cudaGetLastError() == cudaSuccess && cudaMemcpyAsync(h_lv.data(), lv, vwords * 4u, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
             cudaStreamSynchronize(st) == cudaSuccess;
    }
    cudaFree(wcnt); cudaFree(su); cudaFree(lu); cudaFree(tot); cudaFree(lv);
    if (!ok) { cudaGetLastError(); free_run_lists(s); s->rl_state = -1; return false; }
    s->rl_sgl_units = h_tot[0]; s->rl_lr_units = h_tot[1];
    s->rl_b_sgl_units = h_tot[2]; s->rl_b_lr_units = h_tot[3]; s->rl_listed_blocks = h_tot[4];
    s->listed_vecs.swap(h_lv); s->rl_state = 1;
    return true;
}

// agg_pipe_kernel streams the run-list companion in place of the GAP segments when no AND-group member holds a GAP block anywhere
// in the set (then every GAP block is a 1-run source): part A, plus part B in place of the listed bit-blocks when no AND-group
// member holds a listed block either.  Builds it when due (ctx->run_lists); false = the call runs without it.
static bool use_run_lists(bmb200_ctx* ctx, const bmb200_set* set, const bmb200_batch_args* a, RunLists* rl)
{
    bmb200_set* s = const_cast<bmb200_set*>(set);
    if (!ctx->run_lists || s->rl_state < 0) return false;
    const std::vector<uint32_t>& gv = gap_vectors(ctx, set);
    if (gv.empty()) return false;
    for (uint32_t k = a->offsets[0]; k < a->offsets[1]; ++k)
        if ((gv[a->members[k] >> 5] >> (a->members[k] & 31u)) & 1u) return false;
    if (s->rl_state == 0 && (++s->rl_calls < (ctx->run_lists == 1 ? 2u : 1u) || !build_run_lists(ctx, s))) return false;
    bool part_b = s->rl_listed_blocks != 0;
    for (uint32_t k = a->offsets[0]; part_b && k < a->offsets[1]; ++k)
        if ((s->listed_vecs[a->members[k] >> 5] >> (a->members[k] & 31u)) & 1u) part_b = false;
    *rl = RunLists{s->rl_sgl_base, s->rl_lr_base, s->rl_sgl_mid, s->rl_lr_mid, s->rl_sgl, s->rl_lr, part_b ? s->rl_listed : nullptr};
    return true;
}

int bmb200_set_run_lists(const bmb200_set* s, uint64_t* sgl_bytes, uint64_t* lr_bytes)
{
    if (!s || !sgl_bytes || !lr_bytes) return BMB200_ERR_BADARG;
    *sgl_bytes = s->rl_sgl_units * 16u; *lr_bytes = s->rl_lr_units * 16u;
    return BMB200_OK;
}

int bmb200_set_bit_run_lists(const bmb200_set* s, uint64_t* sgl_bytes, uint64_t* lr_bytes, uint64_t* listed_blocks)
{
    if (!s || !sgl_bytes || !lr_bytes || !listed_blocks) return BMB200_ERR_BADARG;
    *sgl_bytes = s->rl_b_sgl_units * 16u; *lr_bytes = s->rl_b_lr_units * 16u; *listed_blocks = s->rl_listed_blocks;
    return BMB200_OK;
}

int bmb200_aggregate_batch(bmb200_ctx* ctx, const bmb200_set* set, const bmb200_batch_args* a, bmb200_result** inout)
{
    if (!ctx || !set || !a || !inout || set->ctx != ctx || !a->n_groups || !a->offsets) return BMB200_ERR_BADARG;
    if (a->op < BMB200_OP_OR || a->op > BMB200_OP_SHIFT_R_AND) return BMB200_ERR_BADARG;
    const uint32_t nb_to = a->nb_to ? a->nb_to : set->v.n_blocks;
    if (a->nb_from >= nb_to || nb_to > set->v.n_blocks) return BMB200_ERR_RANGE;
    const uint32_t ng = a->n_groups;
    const size_t nmem = a->offsets[2 * (size_t)ng];
    for (uint32_t k = 0; k < 2 * ng; ++k) if (a->offsets[k] > a->offsets[k + 1]) return BMB200_ERR_BADARG;
    if (nmem && !a->members) return BMB200_ERR_BADARG;
    for (size_t k = 0; k < nmem; ++k) if (a->members[k] >= set->v.n_vec) return BMB200_ERR_RANGE;
    if (a->op == BMB200_OP_SHIFT_R_AND)
        for (uint32_t g = 0; g < ng; ++g) if (a->offsets[2 * g + 1] - a->offsets[2 * g] > 65536u) return BMB200_ERR_RANGE;
    const uint64_t tot_cols = (uint64_t)(nb_to - a->nb_from) * ng;
    if (tot_cols > 0x7fffffffull) return BMB200_ERR_RANGE;
    CU(cudaSetDevice(ctx->device));
    const uint32_t cols = nb_to - a->nb_from, n_cols = (uint32_t)tot_cols;
    const bool store = !(a->flags & BMB200_F_COUNT_ONLY);
    const bool compress = (a->flags & BMB200_F_OPT_COMPRESS) != 0;
    const bool or_target = (a->flags & BMB200_F_OR_TARGET) != 0;

    bmb200_result* r = *inout;
    if (r && (r->ctx != ctx || r->n_cols != n_cols || r->n_groups != ng || (store && !r->blocks) ||
              (store && compress && !r->gaps) || (or_target && !r->or_blocks))) {
        bmb200_result_free(r); r = nullptr; *inout = nullptr;
    }
    if (!r) {
        int rc = result_alloc(ctx, n_cols, ng, store, store && compress, or_target, &r);
        if (rc) return rc;
    }
    auto bail = [&](int rc) { if (!*inout) bmb200_result_free(r); return rc; };   // a freshly allocated result must not leak
    r->has_blocks = store; r->compress = compress; r->gaps_ready = false; r->has_or = or_target;
    if (r->total_inline && ctx->comm.comm) {
        r->xflip = (r->xflip + 1u) % (uint32_t)CommState::kSlots;
        r->popcnt = r->popcnt_base + (size_t)r->xflip * r->xstride;
        r->total = reinterpret_cast<unsigned long long*>(r->popcnt + (r->xstride - 2u));
        for (int k = 0; k < CommState::kSlots; ++k)          // an all-gather that still sends out of this buffer (kSlots steps back) goes first
            if (ctx->comm.pending[k] && ctx->comm.sendbuf[k] == r->popcnt) cudaStreamWaitEvent(ctx->stream, ctx->comm.done[k], 0);
    }

    // member ids + offsets -> device (pinned staging keeps the copy asynchronous; skipped when unchanged)
    int rc = stage_group(ctx, a->members, nmem, a->offsets, 2 * (size_t)ng + 1, true);
    if (rc) return bail(rc);
    cudaError_t ce = cudaMemsetAsync(ctx->d_work, 0, 4, ctx->stream);
    if (ce == cudaSuccess) ce = cudaMemsetAsync(r->total, 0, 8 * (size_t)ng, ctx->stream);
    if (ce == cudaSuccess && or_target) ce = cudaMemsetAsync(r->or_blocks, 0, (size_t)cols * BMB200_BLOCK_BYTES, ctx->stream);
    if (ce != cudaSuccess) { ctx->last_err = std::string("aggregate: ") + cudaGetErrorString(ce); return bail(BMB200_ERR_CUDA); }

    AggParams p = agg_params(ctx, set, r, a->nb_from, cols, compress, store);
    p.group = ctx->d_group; p.goff = ctx->d_group + nmem; p.n_groups = ng;
    p.or_blocks = or_target ? r->or_blocks : nullptr;
    set_agg_attrs(ctx, &ce);
    if (ce != cudaSuccess) { ctx->last_err = std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(ce); return bail(BMB200_ERR_CUDA); }
    const uint32_t sms = (uint32_t)ctx->sm_count;
    uint32_t grid = sms * (uint32_t)ctx->agg_ctas_per_sm;
    if (grid > n_cols) grid = n_cols;
    RunLists rl{};
    if (ctx->agg_pipeline && ctx->gap_mode == 0 && set->n_gap_units && whole_set(a, set->v.n_vec) &&
        (use_run_lists(ctx, set, a, &rl) || flat_gap_set(ctx, set))) {
        // one AND-SUB group naming every vector once: a producer warp streams whole columns (agg_pipe_kernel), one CTA per SM,
        // with the GAP segments or the run-list companion behind the bit-blocks.
        // OR stays on agg_kernel: its whole-set workloads measured at par or slower through the ring (DESIGN §3.1a)
        p.dyn_bytes = (uint32_t)ctx->pipe_dyn;
        const uint32_t pgrid = sms < n_cols ? sms : n_cols;
        agg_pipe_kernel<<<pgrid, kPipeThreads, ctx->pipe_dyn, ctx->stream>>>(p, rl);
    } else if (a->op == BMB200_OP_SHIFT_R_AND) {
        shift_and_kernel<<<grid, kAggThreads, 0, ctx->stream>>>(p);
    } else {
        launch_agg_kernel(ctx, a->op, grid, p);
    }
    if ((rc = after_launch(ctx))) return bail(rc);
    *inout = r;
    if (store && compress) r->gaps_ready = true;      // bit -> GAP conversion is fused into the kernel epilogue
    return BMB200_OK;
}

int bmb200_aggregate(bmb200_ctx* ctx, const bmb200_set* set, const bmb200_agg_args* a, bmb200_result** inout)
{
    if (!a) return BMB200_ERR_BADARG;
    const uint32_t n1 = (a->op == BMB200_OP_AND_SUB) ? a->n1 : 0u;
    if ((a->n0 && !a->group0) || (n1 && !a->group1)) return BMB200_ERR_BADARG;
    std::vector<uint32_t> mem;
    try { mem.reserve((size_t)a->n0 + n1); mem.insert(mem.end(), a->group0, a->group0 + a->n0); if (n1) mem.insert(mem.end(), a->group1, a->group1 + n1); }
    catch (...) { return BMB200_ERR_BADALLOC; }
    const uint32_t off[3] = {0u, a->n0, a->n0 + n1};
    bmb200_batch_args b{a->op, a->flags & ~BMB200_F_OR_TARGET, 1u, mem.data(), off, a->nb_from, a->nb_to};
    return bmb200_aggregate_batch(ctx, set, &b, inout);
}

int bmb200_binop(bmb200_ctx* ctx, const bmb200_set* set, int op, uint32_t va, uint32_t vb, uint32_t flags,
                 uint32_t nb_from, uint32_t nb_to, bmb200_result** inout)
{
    if (!ctx || !set || !inout || set->ctx != ctx) return BMB200_ERR_BADARG;
    if (op != BMB200_OP_OR && op != BMB200_OP_AND && op != BMB200_OP_XOR && op != BMB200_OP_SUB) return BMB200_ERR_BADARG;
    if (flags & (BMB200_F_COUNT_ONLY | BMB200_F_OR_TARGET)) return BMB200_ERR_BADARG;
    if (va >= set->v.n_vec || vb >= set->v.n_vec) return BMB200_ERR_RANGE;
    if (!nb_to) nb_to = set->v.n_blocks;
    if (nb_from >= nb_to || nb_to > set->v.n_blocks) return BMB200_ERR_RANGE;
    CU(cudaSetDevice(ctx->device));
    const uint32_t cols = nb_to - nb_from;
    const bool compress = (flags & BMB200_F_OPT_COMPRESS) != 0;
    bmb200_result* r = *inout;
    if (r && (r->ctx != ctx || r->n_cols != cols || r->n_groups != 1u || !r->blocks || !r->gaps || r->or_blocks)) { bmb200_result_free(r); r = nullptr; *inout = nullptr; }
    if (!r) { int rc = result_alloc(ctx, cols, 1u, true, true, false, &r); if (rc) return rc; }
    r->has_blocks = true; r->compress = true; r->gaps_ready = true;      // GAP-kind results exist in every opt mode (GAP x GAP merges, cloned GAP blocks)
    auto bail = [&](int rc) { if (!*inout) bmb200_result_free(r); return rc; };
    // the two member ids (a, b) -> device, through the pinned group staging buffer like every aggregate
    const uint32_t mem[2] = {va, vb};
    const uint32_t off[3] = {0u, op == BMB200_OP_SUB ? 1u : 2u, 2u};
    int rc = stage_group(ctx, mem, 2, off, 3, false);
    if (rc) return bail(rc);
    cudaError_t e = cudaMemsetAsync(ctx->d_work, 0, 4, ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(r->total, 0, 8, ctx->stream);
    if (e == cudaSuccess) set_agg_attrs(ctx, &e);
    if (e == cudaSuccess && !ctx->merge_attr_set) { e = cudaFuncSetAttribute(gap_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMergeSmem); ctx->merge_attr_set = (e == cudaSuccess); }
    if (e != cudaSuccess) { ctx->last_err = std::string("binop: ") + cudaGetErrorString(e); return bail(BMB200_ERR_CUDA); }
    const uint32_t bop = op == BMB200_OP_OR ? BINOP_OR : op == BMB200_OP_AND ? BINOP_AND : op == BMB200_OP_XOR ? BINOP_XOR : BINOP_SUB;
    // 1) GAP x GAP columns: merged as run lists (never expanded)
    MergeParams mp{};
    mp.set = set->v; mp.va = va; mp.vb = vb; mp.op = bop; mp.nb_from = nb_from; mp.n_cols = cols;
    mp.kind = r->kind; mp.popcnt = r->popcnt; mp.digest = r->digest; mp.nruns = r->nruns; mp.gaps = r->gaps; mp.total = r->total;
    uint32_t mgrid = (cols + kMergeWarps - 1) / kMergeWarps; const uint32_t mmax = (uint32_t)ctx->sm_count * 8u; if (mgrid > mmax) mgrid = mmax;
    gap_merge_kernel<<<mgrid, kMergeWarps * 32, kMergeSmem, ctx->stream>>>(mp);
    if ((rc = after_launch(ctx))) return bail(rc);
    // 2) every other pairing (and merged blocks that outgrew the GAP format) through the block kernel, kinds by binop_rule
    AggParams p = agg_params(ctx, set, r, nb_from, cols, compress, true);
    p.group = ctx->d_group; p.goff = ctx->d_group + 2; p.n_groups = 1; p.binary = 1u + bop;
    uint32_t grid = (uint32_t)(ctx->sm_count * ctx->agg_ctas_per_sm); if (grid > cols) grid = cols;
    launch_agg_kernel(ctx, op == BMB200_OP_SUB ? BMB200_OP_AND_SUB : op, grid, p);
    if ((rc = after_launch(ctx))) return bail(rc);
    *inout = r;
    return BMB200_OK;
}

int bmb200_scan(bmb200_ctx* ctx, const bmb200_set* set, const bmb200_scan_args* a, bmb200_result** inout)
{
    if (!ctx || !set || !a || !inout || set->ctx != ctx || !a->values || !a->n_values) return BMB200_ERR_BADARG;
    if (a->pred < BMB200_SCAN_EQ || a->pred > BMB200_SCAN_RANGE || !a->n_planes || a->n_planes > 64u) return BMB200_ERR_BADARG;
    if ((uint64_t)a->plane0 + a->n_planes > set->v.n_vec) return BMB200_ERR_RANGE;
    if (a->universe != 0xffffffffu && a->universe >= set->v.n_vec) return BMB200_ERR_RANGE;
    const uint32_t nb_to = a->nb_to ? a->nb_to : set->v.n_blocks;
    if (a->nb_from >= nb_to || nb_to > set->v.n_blocks) return BMB200_ERR_RANGE;
    const uint32_t cols = nb_to - a->nb_from, nv = a->n_values;
    const uint64_t tot_cols = (uint64_t)cols * nv;
    if (tot_cols > 0x7fffffffull) return BMB200_ERR_RANGE;
    CU(cudaSetDevice(ctx->device));
    const uint32_t n_cols = (uint32_t)tot_cols;
    const bool store = !(a->flags & BMB200_F_COUNT_ONLY);
    const bool compress = (a->flags & BMB200_F_OPT_COMPRESS) != 0;

    bmb200_result* r = *inout;
    if (r && (r->ctx != ctx || r->n_cols != n_cols || r->n_groups != nv || (store && !r->blocks) ||
              (store && compress && !r->gaps) || r->or_blocks)) {
        bmb200_result_free(r); r = nullptr; *inout = nullptr;
    }
    if (!r) {
        int rc = result_alloc(ctx, n_cols, nv, store, store && compress, false, &r);
        if (rc) return rc;
    }
    auto bail = [&](int rc) { if (!*inout) bmb200_result_free(r); return rc; };   // a freshly allocated result must not leak
    r->has_blocks = store; r->compress = compress; r->gaps_ready = false;

    // search values -> device through the (pinned) group staging buffer, 2 words per value
    const size_t nvals = (size_t)nv * (a->pred == BMB200_SCAN_RANGE ? 2 : 1);
    int rc = stage_group(ctx, reinterpret_cast<const uint32_t*>(a->values), 2 * nvals, nullptr, 0, false);
    if (rc) return bail(rc);
    cudaError_t e = cudaMemsetAsync(ctx->d_work, 0, 4, ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(r->total, 0, 8 * (size_t)nv, ctx->stream);
    if (e != cudaSuccess) { ctx->last_err = std::string("scan: ") + cudaGetErrorString(e); return bail(BMB200_ERR_CUDA); }

    ScanParams sp{};
    sp.out = agg_params(ctx, set, r, a->nb_from, cols, compress, store);
    sp.out.n_groups = nv;
    sp.plane0 = a->plane0; sp.n_planes = a->n_planes; sp.universe = a->universe; sp.pred = (uint32_t)a->pred;
    sp.values = reinterpret_cast<const uint64_t*>(ctx->d_group);
    // values per pass: find_eq keeps one state per value (4 values share a pass), the inequalities two (2 values), RANGE four (2 values);
    // single searches use the narrow kernels
    const int mode = a->pred == BMB200_SCAN_EQ ? 0 : a->pred == BMB200_SCAN_RANGE ? 2 : 1;
    const uint32_t vg = nv == 1 ? 1u : (mode == 0 && nv >= 4 ? 4u : 2u);
    const uint64_t items = (uint64_t)cols * ((nv + vg - 1) / vg);
    uint32_t grid = (uint32_t)(ctx->sm_count * ctx->agg_ctas_per_sm);
    if (grid > items) grid = (uint32_t)items;
    #define BMB200_SCAN_LAUNCH(VG, MODE) scan_kernel<VG, MODE><<<grid, kAggThreads, 0, ctx->stream>>>(sp)
    if (mode == 0)      { if (vg == 4) BMB200_SCAN_LAUNCH(4, 0); else if (vg == 2) BMB200_SCAN_LAUNCH(2, 0); else BMB200_SCAN_LAUNCH(1, 0); }
    else if (mode == 1) { if (vg == 2) BMB200_SCAN_LAUNCH(2, 1); else BMB200_SCAN_LAUNCH(1, 1); }
    else                { if (vg == 2) BMB200_SCAN_LAUNCH(2, 2); else BMB200_SCAN_LAUNCH(1, 2); }
    #undef BMB200_SCAN_LAUNCH
    if ((rc = after_launch(ctx))) return bail(rc);
    *inout = r;
    if (store && compress) r->gaps_ready = true;
    return BMB200_OK;
}

int bmb200_result_group_totals(bmb200_result* r, uint64_t* totals, uint32_t n_groups)
{
    if (!r || !totals || n_groups != r->n_groups) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = r->ctx;
    CU(cudaSetDevice(ctx->device));
    CU(cudaMemcpyAsync(totals, r->total, 8 * (size_t)n_groups, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return BMB200_OK;
}

int bmb200_result_or_target(bmb200_result* r, bmb200_result** out)
{
    if (!r || !out || !r->or_blocks || !r->has_or) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = r->ctx;
    CU(cudaSetDevice(ctx->device));
    bmb200_result* o = nullptr;
    int rc = result_alloc(ctx, r->cols_per_group, 1u, true, r->compress, false, &o);
    if (rc) return rc;
    o->has_blocks = true; o->compress = r->compress; o->gaps_ready = r->compress;
    if (cudaMemsetAsync(o->total, 0, 8, ctx->stream) != cudaSuccess) { ctx->last_err = "result_or_target: memset"; bmb200_result_free(o); return BMB200_ERR_CUDA; }
    AggParams p{};
    p.n_groups = 1; p.n_cols = r->cols_per_group; p.compress = r->compress ? 1u : 0u; p.store_blocks = 1u;
    p.blocks = o->blocks; p.popcnt = o->popcnt; p.digest = o->digest; p.nruns = o->nruns; p.kind = o->kind; p.gaps = o->gaps;
    p.total = o->total; p.or_blocks = nullptr;
    uint32_t grid = (uint32_t)(ctx->sm_count * ctx->agg_ctas_per_sm); if (grid > p.n_cols) grid = p.n_cols;
    finalize_blocks_kernel<<<grid, kAggThreads, 0, ctx->stream>>>(p, r->or_blocks);
    rc = after_launch(ctx);
    if (rc) { bmb200_result_free(o); return rc; }
    *out = o;
    return BMB200_OK;
}

int bmb200_result_optimize(bmb200_result* r)
{
    if (!r) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = r->ctx;
    if (!r->compress || !r->has_blocks) return BMB200_ERR_BADARG;
    if (r->gaps_ready) return BMB200_OK;
    CU(cudaSetDevice(ctx->device));
    uint32_t grid = (uint32_t)ctx->sm_count * 8u; if (grid > r->n_cols) grid = r->n_cols;
    result_to_gap_kernel<<<grid, kPostThreads, 0, ctx->stream>>>(r->blocks, r->kind, r->gaps, r->n_cols);
    int rc = after_launch(ctx);
    if (!rc) r->gaps_ready = true;
    return rc;
}

int bmb200_result_total(bmb200_result* r, uint64_t* total, int* any)
{
    if (!r) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = r->ctx;
    CU(cudaSetDevice(ctx->device));
    std::vector<unsigned long long> tv(r->n_groups, 0ull);
    CU(cudaMemcpyAsync(tv.data(), r->total, 8 * (size_t)r->n_groups, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    unsigned long long t = 0; for (auto x : tv) t += x;
    if (total) *total = t;
    if (any) *any = t ? 1 : 0;
    return BMB200_OK;
}

int bmb200_result_fetch_meta(bmb200_result* r, const bmb200_result_meta* m)
{
    if (!r || !m) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = r->ctx;
    CU(cudaSetDevice(ctx->device));
    if (m->kind)   CU(cudaMemcpyAsync(m->kind, r->kind, r->n_cols, cudaMemcpyDeviceToHost, ctx->stream));
    if (m->popcnt) CU(cudaMemcpyAsync(m->popcnt, r->popcnt, (size_t)r->n_cols * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (m->digest) CU(cudaMemcpyAsync(m->digest, r->digest, (size_t)r->n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (m->nruns)  CU(cudaMemcpyAsync(m->nruns, r->nruns, (size_t)r->n_cols * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return BMB200_OK;
}

int bmb200_result_fetch_column(bmb200_result* r, uint32_t col, uint8_t* kind_out, uint32_t* bits, uint16_t* gaps)
{
    if (!r || !kind_out || col >= r->n_cols || !r->has_blocks) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = r->ctx;
    CU(cudaSetDevice(ctx->device));
    if (r->compress && !r->gaps_ready) { int rc0 = bmb200_result_optimize(r); if (rc0) return rc0; }
    uint8_t kd = 0;
    CU(cudaMemcpyAsync(&kd, r->kind + col, 1, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    *kind_out = kd;
    if (kd == BMB200_BLK_BIT) {
        if (!bits) return BMB200_ERR_BADARG;
        CU(cudaMemcpyAsync(bits, r->blocks + (size_t)col * kBlockWords, BMB200_BLOCK_BYTES, cudaMemcpyDeviceToHost, ctx->stream));
    } else if (kd == BMB200_BLK_GAP) {
        if (!gaps || !r->gaps) return BMB200_ERR_BADARG;
        CU(cudaMemcpyAsync(gaps, r->gaps + (size_t)col * kGapMax, (size_t)BMB200_GAP_MAX_WORDS * 2, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU(cudaStreamSynchronize(ctx->stream));
    return BMB200_OK;
}

// host-side layout of the compacted result: offsets per column from kinds and run counts
static int result_layout(bmb200_result* r, std::vector<uint8_t>& kind, std::vector<uint64_t>& off, uint64_t* n_bit, uint64_t* n_gap_words)
{
    bmb200_ctx* ctx = r->ctx;
    std::vector<uint32_t> nruns;
    try { kind.resize(r->n_cols); off.assign(r->n_cols, 0); nruns.resize(r->n_cols); } catch (...) { return BMB200_ERR_BADALLOC; }
    CU(cudaSetDevice(ctx->device));
    CU(cudaMemcpyAsync(kind.data(), r->kind, r->n_cols, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(nruns.data(), r->nruns, (size_t)r->n_cols * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    uint64_t nb = 0, ng = 0;
    for (uint32_t c = 0; c < r->n_cols; ++c) {
        if (kind[c] == BMB200_BLK_BIT) off[c] = nb++;
        else if (kind[c] == BMB200_BLK_GAP) { off[c] = ng; ng += ((uint64_t)nruns[c] + 1 + kGapUnit - 1) / kGapUnit * kGapUnit; }
    }
    *n_bit = nb; *n_gap_words = ng;
    return BMB200_OK;
}

int bmb200_result_sizes(bmb200_result* r, uint64_t* n_bit_blocks, uint64_t* n_gap_words)
{
    if (!r || !r->has_blocks) return BMB200_ERR_BADARG;
    std::vector<uint8_t> kind; std::vector<uint64_t> off; uint64_t nb, ng;
    int rc = result_layout(r, kind, off, &nb, &ng);
    if (rc) return rc;
    if (n_bit_blocks) *n_bit_blocks = nb;
    if (n_gap_words) *n_gap_words = ng;
    return BMB200_OK;
}

int bmb200_result_fetch(bmb200_result* r, uint8_t* kind_out, uint64_t* off_out, uint32_t* bits, uint16_t* gaps)
{
    if (!r || !r->has_blocks || !kind_out || !off_out) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = r->ctx;
    if (r->compress && !r->gaps_ready) { int rc = bmb200_result_optimize(r); if (rc) return rc; }
    std::vector<uint8_t> kind; std::vector<uint64_t> off; uint64_t nb, ng;
    int rc = result_layout(r, kind, off, &nb, &ng);
    if (rc) return rc;
    if ((nb && !bits) || (ng && !gaps)) return BMB200_ERR_BADARG;
    memcpy(kind_out, kind.data(), r->n_cols);
    memcpy(off_out, off.data(), (size_t)r->n_cols * 8);
    if (!nb && !ng) return BMB200_OK;
    // compaction scratch and the offsets' staging come from the context's grow-only pools (no allocation once warm)
    uint64_t* d_off = nullptr; uint32_t* d_bits = nullptr; uint16_t* d_gaps = nullptr; uint64_t* h_off = nullptr;
    if ((rc = pool_dev(ctx, kDevCompactOff, (size_t)r->n_cols * 8, (void**)&d_off)) ||
        (rc = pool_dev(ctx, kDevCompactBits, (size_t)nb * BMB200_BLOCK_BYTES + 16, (void**)&d_bits)) ||
        (rc = pool_dev(ctx, kDevCompactGaps, (size_t)ng * 2 + 16, (void**)&d_gaps)) ||
        (rc = pool_host(ctx, kHostCompactOff, (size_t)r->n_cols * 8, (void**)&h_off))) return rc;
    memcpy(h_off, off.data(), (size_t)r->n_cols * 8);
    CU(cudaMemcpyAsync(d_off, h_off, (size_t)r->n_cols * 8, cudaMemcpyHostToDevice, ctx->stream));
    uint32_t grid = (uint32_t)ctx->sm_count * 8u; if (grid > r->n_cols) grid = r->n_cols;
    result_compact_kernel<<<grid, 256, 0, ctx->stream>>>(r->blocks, r->gaps, r->kind, d_off, d_bits, d_gaps, r->n_cols);
    if ((rc = after_launch(ctx))) return rc;
    if (nb) CU(cudaMemcpyAsync(bits, d_bits, (size_t)nb * BMB200_BLOCK_BYTES, cudaMemcpyDeviceToHost, ctx->stream));
    if (ng) CU(cudaMemcpyAsync(gaps, d_gaps, (size_t)ng * 2, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return BMB200_OK;
}

static int fetch_view_impl(bmb200_result* r, const uint8_t** kind_out, const uint64_t** off_out, const uint32_t** bits_out,
                           const uint16_t** gaps_out, uint64_t* n_bit_blocks, uint64_t* n_gap_words, uint64_t* total_out, bool async)
{
    if (!r || !r->has_blocks || !kind_out || !off_out || !bits_out || !gaps_out) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = r->ctx;
    if (r->compress && !r->gaps_ready) { int rc0 = bmb200_result_optimize(r); if (rc0) return rc0; }
    CU(cudaSetDevice(ctx->device));
    // one pinned block of the context: kind | nruns | totals | off ; two stream synchronisations per call, no allocation once warm
    const size_t n = r->n_cols, o_nr = (n + 7) & ~(size_t)7, o_tot = o_nr + n * 4 + ((n & 1) ? 4 : 0), o_off = o_tot + 8 * (size_t)r->n_groups;
    uint8_t* h = nullptr;
    int rc = pool_host(ctx, kHostViewMeta, o_off + n * 8, (void**)&h);
    if (rc) return rc;
    uint8_t* kind = h; uint32_t* nruns = (uint32_t*)(h + o_nr); uint64_t* tot = (uint64_t*)(h + o_tot); uint64_t* off = (uint64_t*)(h + o_off);
    CU(cudaMemcpyAsync(kind, r->kind, n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(nruns, r->nruns, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(tot, r->total, 8 * (size_t)r->n_groups, cudaMemcpyDeviceToHost, ctx->stream));
    static const bool trace = getenv("BMB200_TRACE") != nullptr;
    auto now = []() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double w0 = trace ? now() : 0;
    CU(cudaStreamSynchronize(ctx->stream));
    const double w1 = trace ? now() : 0;
    uint64_t nb = 0, ng = 0;
    for (size_t c = 0; c < n; ++c) {
        off[c] = 0;
        if (kind[c] == BMB200_BLK_BIT) off[c] = nb++;
        else if (kind[c] == BMB200_BLK_GAP) { off[c] = ng; ng += ((uint64_t)nruns[c] + 1 + kGapUnit - 1) / kGapUnit * kGapUnit; }
    }
    uint32_t* hb = nullptr; uint16_t* hg = nullptr;
    if (nb || ng) {
        uint64_t* d_off = nullptr; uint32_t* d_bits = nullptr; uint16_t* d_gaps = nullptr;
        if ((rc = pool_dev(ctx, kDevCompactOff, n * 8, (void**)&d_off)) ||
            (rc = pool_dev(ctx, kDevCompactBits, (size_t)nb * BMB200_BLOCK_BYTES + 16, (void**)&d_bits)) ||
            (rc = pool_dev(ctx, kDevCompactGaps, (size_t)ng * 2 + 16, (void**)&d_gaps))) return rc;
        // two pinned buffers, used in turn: the caller's threads have just READ the previous call's blocks, which parks those lines in
        // their private L2 caches, and a DMA write into lines cached by many cores has to snoop every one of them, which makes
        // it several times slower than a write into cold lines)
        const bool flip = (ctx->fetch_flip ^= 1u) != 0;
        if ((rc = pool_host(ctx, flip ? kHostViewBits1 : kHostViewBits0, (size_t)nb * BMB200_BLOCK_BYTES + 16, (void**)&hb)) ||
            (rc = pool_host(ctx, flip ? kHostViewGaps1 : kHostViewGaps0, (size_t)ng * 2 + 16, (void**)&hg))) return rc;
        CU(cudaMemcpyAsync(d_off, off, n * 8, cudaMemcpyHostToDevice, ctx->stream));
        uint32_t grid = (uint32_t)ctx->sm_count * 8u; if (grid > r->n_cols) grid = r->n_cols;
        result_compact_kernel<<<grid, 256, 0, ctx->stream>>>(r->blocks, r->gaps, r->kind, d_off, d_bits, d_gaps, r->n_cols);
        if ((rc = after_launch(ctx))) return rc;
        r->fetch_chunks = 0;
        if (!async) {
            if (nb) CU(cudaMemcpyAsync(hb, d_bits, (size_t)nb * BMB200_BLOCK_BYTES, cudaMemcpyDeviceToHost, ctx->stream));
            if (ng) CU(cudaMemcpyAsync(hg, d_gaps, (size_t)ng * 2, cudaMemcpyDeviceToHost, ctx->stream));
            CU(cudaStreamSynchronize(ctx->stream));
        } else {
            // the blocks come back in up to 8 column chunks, each followed by an event: the caller starts on the first columns
            // while the later ones are still crossing PCIe (bmb200_result_fetch_wait)
            const uint32_t nch = n >= 2048 ? 8u : 1u, cc = (uint32_t)((n + nch - 1) / nch);
            uint64_t b0 = 0, g0 = 0;
            for (uint32_t c = 0; c < nch; ++c) {
                const size_t c1 = std::min<size_t>(n, (size_t)(c + 1) * cc);
                uint64_t b1 = b0, g1 = g0;                                        // first block / GAP word past this chunk
                for (size_t k = (size_t)c * cc; k < c1; ++k) {
                    if (kind[k] == BMB200_BLK_BIT) b1 = off[k] + 1;
                    else if (kind[k] == BMB200_BLK_GAP) g1 = off[k] + ((uint64_t)nruns[k] + 1 + kGapUnit - 1) / kGapUnit * kGapUnit;
                }
                if (b1 > b0) CU(cudaMemcpyAsync(hb + b0 * kBlockWords, d_bits + b0 * kBlockWords, (size_t)(b1 - b0) * BMB200_BLOCK_BYTES, cudaMemcpyDeviceToHost, ctx->stream));
                if (g1 > g0) CU(cudaMemcpyAsync(hg + g0, d_gaps + g0, (size_t)(g1 - g0) * 2, cudaMemcpyDeviceToHost, ctx->stream));
                if (!ctx->fetch_ev[c]) CU(cudaEventCreateWithFlags(&ctx->fetch_ev[c], cudaEventDisableTiming));
                CU(cudaEventRecord(ctx->fetch_ev[c], ctx->stream));
                b0 = b1; g0 = g1;
            }
            r->fetch_chunk_cols = cc; r->fetch_chunks = nch;
        }
    } else r->fetch_chunks = 0;
    if (trace) fprintf(stderr, "[bmb200] result_fetch_view: waited %.3f ms for the kernel + column kinds, %.3f ms for compaction + D2H of %.1f MB\n",
                       w1 - w0, now() - w1, (nb * (double)BMB200_BLOCK_BYTES + ng * 2.0) / 1048576.0);
    *kind_out = kind; *off_out = off; *bits_out = hb; *gaps_out = hg;
    if (n_bit_blocks) *n_bit_blocks = nb;
    if (n_gap_words) *n_gap_words = ng;
    if (total_out) { uint64_t t = 0; for (uint32_t g = 0; g < r->n_groups; ++g) t += tot[g]; *total_out = t; }
    return BMB200_OK;
}

int bmb200_result_fetch_view(bmb200_result* r, const uint8_t** kind_out, const uint64_t** off_out, const uint32_t** bits_out,
                             const uint16_t** gaps_out, uint64_t* n_bit_blocks, uint64_t* n_gap_words, uint64_t* total_out)
{
    return fetch_view_impl(r, kind_out, off_out, bits_out, gaps_out, n_bit_blocks, n_gap_words, total_out, false);
}

int bmb200_result_fetch_view_async(bmb200_result* r, const uint8_t** kind_out, const uint64_t** off_out, const uint32_t** bits_out,
                                   const uint16_t** gaps_out, uint64_t* n_bit_blocks, uint64_t* n_gap_words, uint64_t* total_out)
{
    return fetch_view_impl(r, kind_out, off_out, bits_out, gaps_out, n_bit_blocks, n_gap_words, total_out, true);
}

int bmb200_result_fetch_wait(bmb200_result* r, uint32_t col)
{
    if (!r) return BMB200_ERR_BADARG;
    if (!r->fetch_chunks) return BMB200_OK;                       // nothing in flight (empty result or the synchronous call)
    uint32_t c = r->fetch_chunk_cols ? col / r->fetch_chunk_cols : 0u;
    if (c >= r->fetch_chunks) c = r->fetch_chunks - 1;
    return cudaEventSynchronize(r->ctx->fetch_ev[c]) == cudaSuccess ? BMB200_OK : BMB200_ERR_CUDA;
}

int bmb200_result_device_ptrs(const bmb200_result* r, void** blocks, void** popcnt, void** digest, void** flag, uint32_t* n_cols)
{
    if (!r) return BMB200_ERR_BADARG;
    if (blocks) *blocks = r->blocks;
    if (popcnt) *popcnt = r->popcnt;
    if (digest) *digest = r->digest;
    if (flag) *flag = r->kind;
    if (n_cols) *n_cols = r->n_cols;
    return BMB200_OK;
}

int bmb200_result_free(bmb200_result* r)
{
    if (!r) return BMB200_ERR_BADARG;
    cudaSetDevice(r->ctx->device);
    cudaStreamSynchronize(r->ctx->stream);
    free_result_arrays(r);
    delete r;
    return BMB200_OK;
}

int bmb200_aggregate_host(bmb200_ctx* ctx, const bmb200_packed_set* host, const bmb200_agg_args* args,
                          const bmb200_result_meta* meta_out, uint64_t* total_out)
{
    if (!ctx || !host || !args || !host->n_vec || !host->n_blocks || !host->desc || !host->bit_base || !host->gap_base)
        return BMB200_ERR_BADARG;
    CU(cudaSetDevice(ctx->device));
    const uint64_t n_bit = host->bit_base[host->n_blocks], n_gap = host->gap_base[host->n_blocks];
    if ((n_bit && !host->bit_pool) || (n_gap && !host->gap_pool)) return BMB200_ERR_BADARG;
    const size_t need_desc = (size_t)host->n_vec * host->n_blocks, need_base = (size_t)host->n_blocks + 1;
    // the device arena and the result buffers persist in the context: every call still copies ALL inputs H2D
    const bmb200_set* hs = ctx->host_set;
    if (!hs || need_desc > hs->cap_desc || need_base > hs->cap_base || n_bit > hs->cap_bit || n_gap > hs->cap_gap) {
        if (ctx->host_set) { bmb200_set_free(ctx->host_set); ctx->host_set = nullptr; }
        int rc = set_alloc(ctx, host->n_vec, host->n_blocks, n_bit, n_gap, &ctx->host_set);
        if (rc) return rc;
    }
    int rc = set_copy_in(ctx, ctx->host_set, host, n_bit, n_gap);
    if (!rc) rc = bmb200_aggregate(ctx, ctx->host_set, args, &ctx->host_res);
    if (!rc && meta_out) rc = bmb200_result_fetch_meta(ctx->host_res, meta_out);
    if (!rc && total_out) rc = bmb200_result_total(ctx->host_res, total_out, nullptr);
    return rc;
}

/* ------------------------------------------------------------------ multi-GPU: block-range shards + one exchange */

int bmb200_shard_range(uint32_t n_blocks, int nranks, int rank, uint32_t* nb_from, uint32_t* nb_to)
{
    if (nranks < 1 || rank < 0 || rank >= nranks || !nb_from || !nb_to) return BMB200_ERR_BADARG;
    // whole 256-block superblocks per rank, so rs_index rows never straddle shards (SURVEY 8e)
    const uint64_t nsb = ((uint64_t)n_blocks + BMB200_SUPERBLOCK - 1) / BMB200_SUPERBLOCK;
    const uint64_t lo = nsb * (uint64_t)rank / (uint64_t)nranks * BMB200_SUPERBLOCK, hi = nsb * ((uint64_t)rank + 1) / (uint64_t)nranks * BMB200_SUPERBLOCK;
    *nb_from = (uint32_t)std::min<uint64_t>(lo, n_blocks); *nb_to = (uint32_t)std::min<uint64_t>(hi, n_blocks);
    return BMB200_OK;
}

int bmb200_comm_unique_id(void* id)
{
    if (!id) return BMB200_ERR_BADARG;
    NcclApi& api = nccl_api();
    if (!api.load()) return BMB200_ERR_UNSUPPORTED;
    NcclApi::UniqueId u;
    if (api.GetUniqueId(&u) != 0) return BMB200_ERR_CUDA;
    memcpy(id, &u, BMB200_COMM_ID_BYTES);
    return BMB200_OK;
}

int bmb200_comm_init(bmb200_ctx* ctx, int nranks, int rank, const void* id)
{
    if (!ctx || !id || nranks < 1 || rank < 0 || rank >= nranks) return BMB200_ERR_BADARG;
    NcclApi& api = nccl_api();
    if (!api.load()) { ctx->last_err = api.err; return BMB200_ERR_UNSUPPORTED; }
    CU(cudaSetDevice(ctx->device));
    comm_release(ctx);
    CommState& c = ctx->comm;
    NcclApi::UniqueId u; memcpy(&u, id, BMB200_COMM_ID_BYTES);
    const int nrc = api.CommInitRank(&c.comm, nranks, u, rank);
    if (nrc != 0) { ctx->last_err = std::string("ncclCommInitRank: ") + api.GetErrorString(nrc); c.comm = nullptr; return BMB200_ERR_CUDA; }
    c.nranks = nranks; c.rank = rank;
    cudaError_t e = cudaStreamCreateWithFlags(&c.side, cudaStreamNonBlocking);
    for (int k = 0; k < CommState::kSlots && e == cudaSuccess; ++k) {
        e = cudaEventCreateWithFlags(&c.ready[k], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c.done[k], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) { ctx->last_err = std::string("comm_init: ") + cudaGetErrorString(e); comm_release(ctx); return BMB200_ERR_CUDA; }
    return BMB200_OK;
}

int bmb200_comm_info(const bmb200_ctx* ctx, int* nranks, int* rank)
{
    if (!ctx) return BMB200_ERR_BADARG;
    if (nranks) *nranks = ctx->comm.comm ? ctx->comm.nranks : 1;
    if (rank) *rank = ctx->comm.comm ? ctx->comm.rank : 0;
    return BMB200_OK;
}

int bmb200_comm_destroy(bmb200_ctx* ctx)
{
    if (!ctx) return BMB200_ERR_BADARG;
    cudaSetDevice(ctx->device);
    comm_release(ctx);
    return BMB200_OK;
}

int bmb200_exchange_popcounts(bmb200_result* r, uint32_t cols_per_rank)
{
    if (!r || r->n_groups != 1 || (cols_per_rank && cols_per_rank < r->n_cols)) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = r->ctx;
    CommState& c = ctx->comm;
    if (!c.comm) return BMB200_ERR_BADARG;
    CU(cudaSetDevice(ctx->device));
    const size_t n = cols_per_rank ? cols_per_rank : r->n_cols, words = n + 2;
    if (n > c.cap_cols) {
        CU(cudaStreamSynchronize(c.side));
        for (int k = 0; k < CommState::kSlots; ++k) { cudaFree(c.stage[k]); cudaFree(c.gathered[k]); c.stage[k] = c.gathered[k] = nullptr; c.pending[k] = false; }
        c.cap_cols = 0;
        for (int k = 0; k < CommState::kSlots; ++k) {
            CU(cudaMalloc((void**)&c.stage[k], words * 4));
            CU(cudaMalloc((void**)&c.gathered[k], words * 4 * (size_t)c.nranks));
        }
        c.cap_cols = n;
    }
    const int k = (int)(c.seq % (uint64_t)CommState::kSlots);
    // slot k was last used by the exchange kSlots steps back: nothing below may overtake that all-gather
    if (c.pending[k]) CU(cudaStreamWaitEvent(ctx->stream, c.done[k], 0));
    const uint32_t* send = c.stage[k];
    if (r->total_inline && n == r->n_cols && !(n & 1u))
        send = r->popcnt;                                      // (popcnt | total) as the kernel wrote them: no staging copy
    else {
        if (n > r->n_cols) CU(cudaMemsetAsync(c.stage[k] + r->n_cols, 0, (n - r->n_cols) * 4, ctx->stream));     // ragged shards: zero padding
        CU(cudaMemcpyAsync(c.stage[k], r->popcnt, (size_t)r->n_cols * 4, cudaMemcpyDeviceToDevice, ctx->stream));
        CU(cudaMemcpyAsync(c.stage[k] + n, r->total, 8, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    c.sendbuf[k] = send;
    CU(cudaEventRecord(c.ready[k], ctx->stream));
    CU(cudaStreamWaitEvent(c.side, c.ready[k], 0));
    const int nrc = nccl_api().AllGather(send, c.gathered[k], words, kNcclUint32, c.comm, c.side);
    if (nrc != 0) { ctx->last_err = std::string("ncclAllGather: ") + nccl_api().GetErrorString(nrc); return BMB200_ERR_CUDA; }
    CU(cudaEventRecord(c.done[k], c.side));
    c.pending[k] = true; c.cols[k] = (uint32_t)n; c.seq++;
    return BMB200_OK;
}

int bmb200_exchange_mode(const bmb200_ctx* ctx, int* mode)
{
    if (!ctx || !mode) return BMB200_ERR_BADARG;
    *mode = (!ctx->comm.comm || !ctx->comm.seq) ? 0 : 1;
    return BMB200_OK;
}

int bmb200_exchange_fence(bmb200_ctx* ctx)
{
    if (!ctx || !ctx->comm.comm) return BMB200_ERR_BADARG;
    CU(cudaSetDevice(ctx->device));
    CommState& c = ctx->comm;
    for (int k = 0; k < CommState::kSlots; ++k) if (c.pending[k]) CU(cudaStreamWaitEvent(ctx->stream, c.done[k], 0));
    return BMB200_OK;
}

int bmb200_exchange_fetch(bmb200_ctx* ctx, uint64_t* global_total, uint64_t* rank_totals, uint32_t* popcnt, const uint32_t** d_gathered, uint32_t* stride)
{
    if (!ctx || !ctx->comm.comm || !ctx->comm.seq) return BMB200_ERR_BADARG;
    CommState& c = ctx->comm;
    CU(cudaSetDevice(ctx->device));
    const int k = (int)((c.seq - 1) % (uint64_t)CommState::kSlots);
    const size_t n = c.cols[k], words = n + 2;
    CU(cudaEventSynchronize(c.done[k]));
    const uint32_t* rows = c.gathered[k];
    if (d_gathered) *d_gathered = rows;
    if (stride) *stride = (uint32_t)words;
    if (global_total || rank_totals || popcnt) {
        uint32_t* h = nullptr;
        int rc = pool_host(ctx, kHostExchange, words * 4 * (size_t)c.nranks, (void**)&h);
        if (rc) return rc;
        CU(cudaMemcpyAsync(h, rows, words * 4 * (size_t)c.nranks, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        uint64_t tot = 0;
        for (int q = 0; q < c.nranks; ++q) {
            uint64_t t; memcpy(&t, h + (size_t)q * words + n, 8);
            if (rank_totals) rank_totals[q] = t;
            tot += t;
            if (popcnt) memcpy(popcnt + (size_t)q * n, h + (size_t)q * words, n * 4);
        }
        if (global_total) *global_total = tot;
    }
    return BMB200_OK;
}

int bmb200_ctx_bind_host_numa(bmb200_ctx* ctx, int* node_out)
{
    if (!ctx) return BMB200_ERR_BADARG;
    if (node_out) *node_out = -1;
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, ctx->device) != cudaSuccess) { cudaGetLastError(); return BMB200_OK; }
    for (char* q = bus; *q; ++q) if (*q >= 'A' && *q <= 'Z') *q = (char)(*q - 'A' + 'a');
    int node = -1;
    { std::ifstream f(std::string("/sys/bus/pci/devices/") + bus + "/numa_node"); if (!(f >> node)) node = -1; }
    if (node < 0) return BMB200_OK;                       // single-node box or no topology information: nothing to do
    std::string list;
    { std::ifstream f("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist"); std::getline(f, list); }
    cpu_set_t cs; CPU_ZERO(&cs); int ncpu = 0;
    for (size_t i = 0; i < list.size();) {               // "0-31,64-95"
        size_t j = i; long a = 0, b; while (j < list.size() && isdigit((unsigned char)list[j])) a = a * 10 + (list[j++] - '0');
        b = a;
        if (j < list.size() && list[j] == '-') { ++j; b = 0; while (j < list.size() && isdigit((unsigned char)list[j])) b = b * 10 + (list[j++] - '0'); }
        for (long c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET((int)c, &cs); ++ncpu; }
        while (j < list.size() && !isdigit((unsigned char)list[j])) ++j;
        if (j == i) break;
        i = j;
    }
    if (ncpu && sched_setaffinity(0, sizeof cs, &cs) == 0 && node_out) *node_out = node;
    return BMB200_OK;
}

/* ------------------------------------------------------------------ rank / select */

static RsView rs_view(const bmb200_rs* rs)
{
    RsView v{};
    v.set = rs->set->v; v.vec = rs->vec; v.nsb = rs->nsb;
    v.bcount = rs->bcount; v.sub_count = rs->sub_count; v.row_cum = rs->row_cum; v.sb_cum = rs->sb_cum;
    v.fine = rs->fine; v.fine_piv = rs->fine_piv; v.row_piv = rs->row_piv;
    return v;
}

int bmb200_rs_build(bmb200_ctx* ctx, const bmb200_set* set, uint32_t vec, bmb200_rs** out)
{
    if (!ctx || !set || !out || set->ctx != ctx) return BMB200_ERR_BADARG;
    if (vec >= set->v.n_vec) return BMB200_ERR_RANGE;
    CU(cudaSetDevice(ctx->device));
    bmb200_rs* rs = new (std::nothrow) bmb200_rs();
    if (!rs) return BMB200_ERR_BADALLOC;
    rs->ctx = ctx; rs->set = set; rs->vec = vec; rs->n_blocks = set->v.n_blocks;
    rs->nsb = (set->v.n_blocks + 255u) / 256u;
    int rc;
    if ((rc = dev_alloc(ctx, &rs->bcount, rs->n_blocks)) || (rc = dev_alloc(ctx, &rs->sub_count, rs->n_blocks)) ||
        (rc = dev_alloc(ctx, &rs->row_cum, (size_t)rs->nsb * 256u)) || (rc = dev_alloc(ctx, &rs->sb_tot, rs->nsb)) ||
        (rc = dev_alloc(ctx, &rs->sb_cum, (size_t)rs->nsb + 1)) ||
        (rc = dev_alloc(ctx, &rs->fine, (size_t)rs->n_blocks * kRsWin)) || (rc = dev_alloc(ctx, &rs->fine_piv, (size_t)rs->n_blocks * kRsPiv)) ||
        (rc = dev_alloc(ctx, &rs->row_piv, (size_t)rs->nsb * kRsRowPiv))) { bmb200_rs_free(rs); return rc; }
    rc = bmb200_rs_rebuild(rs);
    if (rc) { bmb200_rs_free(rs); return rc; }
    *out = rs;
    return BMB200_OK;
}

int bmb200_rs_rebuild(bmb200_rs* rs)
{
    if (!rs) return BMB200_ERR_RS_IDX_MISSING;
    bmb200_ctx* ctx = rs->ctx;
    CU(cudaSetDevice(ctx->device));
    int rc;
    uint32_t grid = (rs->n_blocks + 7u) / 8u;
    const uint32_t maxg = (uint32_t)ctx->sm_count * 16u; if (grid > maxg) grid = maxg;
    rs_block_kernel<<<grid, 256, 0, ctx->stream>>>(rs->set->v, rs->vec, rs->bcount, rs->sub_count, rs->fine, rs->fine_piv);
    if ((rc = after_launch(ctx))) return rc;
    rs_scan_rows_kernel<<<rs->nsb, 256, 0, ctx->stream>>>(rs->bcount, rs->n_blocks, rs->row_cum, rs->sb_tot, rs->row_piv);
    if ((rc = after_launch(ctx))) return rc;
    rs_scan_sb_kernel<<<1, 1024, 0, ctx->stream>>>(rs->sb_tot, rs->nsb, rs->sb_cum);
    return after_launch(ctx);
}

int bmb200_rs_export(bmb200_rs* rs, uint32_t* bcount, uint64_t* sub_count, uint64_t* sb_count)
{
    if (!rs) return BMB200_ERR_RS_IDX_MISSING;
    bmb200_ctx* ctx = rs->ctx;
    CU(cudaSetDevice(ctx->device));
    if (bcount)    CU(cudaMemcpyAsync(bcount, rs->bcount, (size_t)rs->n_blocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (sub_count) CU(cudaMemcpyAsync(sub_count, rs->sub_count, (size_t)rs->n_blocks * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (sb_count)  CU(cudaMemcpyAsync(sb_count, rs->sb_cum, ((size_t)rs->nsb + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return BMB200_OK;
}

int bmb200_rs_total(bmb200_rs* rs, uint64_t* total)
{
    if (!rs) return BMB200_ERR_RS_IDX_MISSING;
    if (!total) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = rs->ctx;
    CU(cudaSetDevice(ctx->device));
    CU(cudaMemcpyAsync(total, rs->sb_cum + rs->nsb, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return BMB200_OK;
}

int bmb200_rank_batch_dev(bmb200_rs* rs, const uint64_t* d_pos, uint64_t n, uint64_t* d_out)
{
    if (!rs) return BMB200_ERR_RS_IDX_MISSING;
    if (!n) return BMB200_OK;
    if (!d_pos || !d_out) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = rs->ctx;
    CU(cudaSetDevice(ctx->device));
    uint64_t g = (n + 255) / 256; const uint64_t maxg = (uint64_t)ctx->sm_count * 32; if (g > maxg) g = maxg;
    rs_rank_kernel<<<(unsigned)g, 256, 0, ctx->stream>>>(rs_view(rs), d_pos, n, d_out);
    return after_launch(ctx);
}

int bmb200_select_batch_dev(bmb200_rs* rs, const uint64_t* d_rank, uint64_t n, uint64_t* d_pos, uint8_t* d_found)
{
    if (!rs) return BMB200_ERR_RS_IDX_MISSING;
    if (!n) return BMB200_OK;
    if (!d_rank || !d_pos || !d_found) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = rs->ctx;
    CU(cudaSetDevice(ctx->device));
    uint64_t g = (n + 255) / 256; const uint64_t maxg = (uint64_t)ctx->sm_count * 32; if (g > maxg) g = maxg;
    rs_select_kernel<<<(unsigned)g, 256, 0, ctx->stream>>>(rs_view(rs), d_rank, n, d_pos, d_found);
    return after_launch(ctx);
}

int bmb200_rank_batch(bmb200_rs* rs, const uint64_t* pos, uint64_t n, uint64_t* out)
{
    if (!rs) return BMB200_ERR_RS_IDX_MISSING;
    if (!n) return BMB200_OK;
    if (!pos || !out) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = rs->ctx;
    CU(cudaSetDevice(ctx->device));
    uint64_t *d_in = nullptr, *d_out = nullptr;       // context pools: no cudaMalloc / cudaFree per call
    int rc;
    if ((rc = pool_dev(ctx, kDevRsIn, n * 8, (void**)&d_in)) || (rc = pool_dev(ctx, kDevRsOut, n * 8, (void**)&d_out))) return rc;
    CU(cudaMemcpyAsync(d_in, pos, n * 8, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = bmb200_rank_batch_dev(rs, d_in, n, d_out))) return rc;
    CU(cudaMemcpyAsync(out, d_out, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return BMB200_OK;
}

int bmb200_select_batch(bmb200_rs* rs, const uint64_t* rank, uint64_t n, uint64_t* pos, uint8_t* found)
{
    if (!rs) return BMB200_ERR_RS_IDX_MISSING;
    if (!n) return BMB200_OK;
    if (!rank || !pos || !found) return BMB200_ERR_BADARG;
    bmb200_ctx* ctx = rs->ctx;
    CU(cudaSetDevice(ctx->device));
    uint64_t *d_in = nullptr, *d_pos = nullptr; uint8_t* d_f = nullptr;
    int rc;
    if ((rc = pool_dev(ctx, kDevRsIn, n * 8, (void**)&d_in)) || (rc = pool_dev(ctx, kDevRsOut, n * 8, (void**)&d_pos)) ||
        (rc = pool_dev(ctx, kDevRsFound, n, (void**)&d_f))) return rc;
    CU(cudaMemcpyAsync(d_in, rank, n * 8, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = bmb200_select_batch_dev(rs, d_in, n, d_pos, d_f))) return rc;
    CU(cudaMemcpyAsync(pos, d_pos, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(found, d_f, n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return BMB200_OK;
}

int bmb200_rs_free(bmb200_rs* rs)
{
    if (!rs) return BMB200_ERR_BADARG;
    cudaSetDevice(rs->ctx->device);
    cudaStreamSynchronize(rs->ctx->stream);
    cudaFree(rs->bcount); cudaFree(rs->sub_count); cudaFree(rs->row_cum); cudaFree(rs->sb_tot); cudaFree(rs->sb_cum);
    cudaFree(rs->fine); cudaFree(rs->fine_piv); cudaFree(rs->row_piv);
    delete rs;
    return BMB200_OK;
}

/* ------------------------------------------------------------------ rank compression (rank_kernel.cuh) */

// *inout recycled when it has the shape asked for, else freed and replaced (as bmb200_scan does)
static int rank_result(bmb200_ctx* ctx, uint32_t n_cols, uint32_t n_groups, bool compress, bmb200_result** inout, bmb200_result** out)
{
    bmb200_result* r = *inout;
    if (r && (r->ctx != ctx || r->n_cols != n_cols || r->n_groups != n_groups || !r->blocks || (compress && !r->gaps) || r->or_blocks)) {
        bmb200_result_free(r); r = nullptr; *inout = nullptr;
    }
    if (!r) { int rc = result_alloc(ctx, n_cols, n_groups, true, compress, false, &r); if (rc) return rc; }
    r->has_blocks = true; r->compress = compress; r->gaps_ready = compress;      // the epilogue writes the GAP form in compress mode
    *out = r;
    return BMB200_OK;
}

int bmb200_rank_decompress(bmb200_ctx* ctx, const bmb200_rs* idx, const bmb200_result* src, uint32_t flags, bmb200_result** inout)
{
    if (!ctx || !idx || !src || !inout || idx->ctx != ctx || src->ctx != ctx || *inout == src) return BMB200_ERR_BADARG;
    if (flags & ~BMB200_F_OPT_COMPRESS) return BMB200_ERR_BADARG;
    // the source's columns are read by their kind: BIT ones need the stored blocks, GAP ones the GAP form
    if (!src->has_blocks || !src->blocks || !src->n_groups || src->n_cols != src->n_groups * src->cols_per_group ||
        (src->compress && (!src->gaps || !src->gaps_ready))) return BMB200_ERR_BADARG;
    const uint64_t tot_cols = (uint64_t)src->n_groups * idx->n_blocks;
    if (tot_cols > 0x7fffffffull) return BMB200_ERR_RANGE;
    CU(cudaSetDevice(ctx->device));
    const bool compress = (flags & BMB200_F_OPT_COMPRESS) != 0;
    bmb200_result* r = nullptr;
    int rc = rank_result(ctx, (uint32_t)tot_cols, src->n_groups, compress, inout, &r);
    if (rc) return rc;
    auto bail = [&](int e) { if (!*inout) bmb200_result_free(r); return e; };
    if (cudaMemsetAsync(r->total, 0, 8 * (size_t)r->n_groups, ctx->stream) != cudaSuccess) { ctx->last_err = "rank_decompress: memset"; return bail(BMB200_ERR_CUDA); }
    AggParams p{};
    p.n_groups = r->n_groups; p.n_cols = r->n_cols; p.compress = compress ? 1u : 0u; p.store_blocks = 1u;
    p.blocks = r->blocks; p.popcnt = r->popcnt; p.digest = r->digest; p.nruns = r->nruns; p.kind = r->kind; p.gaps = r->gaps;
    p.total = r->total;
    RankSrc s{src->kind, src->blocks, src->gaps, src->cols_per_group};
    uint32_t grid = (uint32_t)(ctx->sm_count * kCtasPerSm); if (grid > p.n_cols) grid = p.n_cols;
    rank_decompress_kernel<<<grid, kAggThreads, 0, ctx->stream>>>(p, rs_view(idx), s);
    if ((rc = after_launch(ctx))) return bail(rc);
    *inout = r;
    return BMB200_OK;
}

int bmb200_rank_compress(bmb200_ctx* ctx, const bmb200_rs* idx, uint32_t src_vec, uint32_t flags, bmb200_result** inout)
{
    if (!ctx || !idx || !inout || idx->ctx != ctx) return BMB200_ERR_BADARG;
    if (flags & ~BMB200_F_OPT_COMPRESS) return BMB200_ERR_BADARG;
    if (src_vec >= idx->set->v.n_vec) return BMB200_ERR_RANGE;
    CU(cudaSetDevice(ctx->device));
    uint64_t total = 0;                                   // count(NN) sizes the target
    CU(cudaMemcpyAsync(&total, idx->sb_cum + idx->nsb, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    const uint64_t cols64 = total ? (total + 65535u) >> 16 : 1u;
    if (cols64 > 0x7fffffffull) return BMB200_ERR_RANGE;
    const uint32_t cols = (uint32_t)cols64;
    const bool compress = (flags & BMB200_F_OPT_COMPRESS) != 0;
    uint32_t* dense = nullptr;
    int rc = pool_dev(ctx, kDevRankDense, (size_t)cols * BMB200_BLOCK_BYTES, (void**)&dense);
    if (rc) return rc;
    bmb200_result* r = nullptr;
    if ((rc = rank_result(ctx, cols, 1u, compress, inout, &r))) return rc;
    auto bail = [&](int e) { if (!*inout) bmb200_result_free(r); return e; };
    cudaError_t e = cudaMemsetAsync(dense, 0, (size_t)cols * BMB200_BLOCK_BYTES, ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(r->total, 0, 8, ctx->stream);
    if (e != cudaSuccess) { ctx->last_err = std::string("rank_compress: ") + cudaGetErrorString(e); return bail(BMB200_ERR_CUDA); }
    uint32_t grid = (uint32_t)(ctx->sm_count * kCtasPerSm); if (grid > idx->n_blocks) grid = idx->n_blocks;
    rank_compress_scatter_kernel<<<grid, kAggThreads, 0, ctx->stream>>>(rs_view(idx), src_vec, dense);
    if ((rc = after_launch(ctx))) return bail(rc);
    AggParams p{};
    p.n_groups = 1; p.n_cols = cols; p.compress = compress ? 1u : 0u; p.store_blocks = 1u;
    p.blocks = r->blocks; p.popcnt = r->popcnt; p.digest = r->digest; p.nruns = r->nruns; p.kind = r->kind; p.gaps = r->gaps;
    p.total = r->total;
    grid = (uint32_t)(ctx->sm_count * kCtasPerSm); if (grid > cols) grid = cols;
    finalize_blocks_kernel<<<grid, kAggThreads, 0, ctx->stream>>>(p, dense);
    if ((rc = after_launch(ctx))) return bail(rc);
    *inout = r;
    return BMB200_OK;
}

}  // extern "C"
