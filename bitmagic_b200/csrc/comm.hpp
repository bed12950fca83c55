// comm.hpp -- the one exchange step of a block-range sharded aggregation (SURVEY 8e): every rank owns a contiguous range of
// block columns of every vector, aggregates it locally, and the ranks exchange the per-column popcounts (4 B per column) and
// their cardinalities with ONE ncclAllGather over NVLink / NVSwitch.  There is no data-path collective: result blocks never move.
//
// NCCL is bound at run time (dlopen of libnccl.so.2 -- the copy torch already mapped when the caller is a torch process, the
// system one otherwise), so libbmb200.so itself carries no NCCL dependency and single-GPU users never load it.  The few ABI
// constants below are NCCL 2.x's (nccl.h: ncclUniqueId = 128 bytes, ncclUint8 = 1, ncclUint32 = 3, ncclUint64 = 5, ncclSum = 0).
#pragma once
#include <dlfcn.h>
#include <cstdint>
#include <cstring>
#include <string>

#include <cuda_runtime.h>

namespace bmb200 {

struct NcclApi {
    typedef struct { char internal[128]; } UniqueId;
    typedef void* Comm;
    int  (*GetUniqueId)(UniqueId*) = nullptr;
    int  (*CommInitRank)(Comm*, int, UniqueId, int) = nullptr;
    int  (*CommDestroy)(Comm) = nullptr;
    int  (*AllGather)(const void*, void*, size_t, int, Comm, cudaStream_t) = nullptr;
    int  (*AllReduce)(const void*, void*, size_t, int, int, Comm, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    int  (*GetVersion)(int*) = nullptr;
    void* handle = nullptr;
    std::string err;

    bool load()
    {
        if (handle) return true;
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* n : names) { handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (handle) break; }
        if (!handle) { err = std::string("dlopen(libnccl.so.2): ") + (dlerror() ? dlerror() : "not found"); return false; }
        auto sym = [&](const char* s) { void* p = dlsym(handle, s); if (!p) err = std::string("dlsym ") + s; return p; };
        GetUniqueId   = (decltype(GetUniqueId))sym("ncclGetUniqueId");
        CommInitRank  = (decltype(CommInitRank))sym("ncclCommInitRank");
        CommDestroy   = (decltype(CommDestroy))sym("ncclCommDestroy");
        AllGather     = (decltype(AllGather))sym("ncclAllGather");
        AllReduce     = (decltype(AllReduce))sym("ncclAllReduce");
        GetErrorString = (decltype(GetErrorString))sym("ncclGetErrorString");
        GetVersion    = (decltype(GetVersion))sym("ncclGetVersion");
        if (!GetUniqueId || !CommInitRank || !CommDestroy || !AllGather || !AllReduce || !GetErrorString) { dlclose(handle); handle = nullptr; return false; }
        return true;
    }
};

constexpr int kNcclUint8 = 1, kNcclUint32 = 3, kNcclUint64 = 5, kNcclSum = 0;

inline NcclApi& nccl_api() { static NcclApi api; return api; }

// per-context communicator + the exchange ring
struct CommState {
    NcclApi::Comm comm = nullptr;
    int nranks = 0, rank = -1;
    cudaStream_t side = nullptr;             // the exchange runs here, so that step i's all-gather overlaps step i+1's kernel
    static constexpr int kSlots = 3;         // all-gathers in flight: an all-gather only finds SMs in the gap between two aggregation
                                             // kernels, so the kernel of step i must not wait for the all-gather of step i-2 (it runs in
                                             // the gap right before it) -- with three slots it waits for step i-3's, done one gap earlier
    cudaEvent_t ready[kSlots] = {}, done[kSlots] = {};
    uint32_t* stage[kSlots] = {}; // [cap_cols + 2] u32: this rank's per-column popcounts, then its cardinality (u64)
    uint32_t* gathered[kSlots] = {};   // [nranks][cap_cols + 2]
    size_t cap_cols = 0;                     // columns the buffers were sized for
    uint32_t cols[kSlots] = {};               // columns of the exchange in flight in each slot
    uint64_t seq = 0;                        // exchanges issued
    bool pending[kSlots] = {};
    const uint32_t* sendbuf[kSlots] = {};   // what the all-gather of each slot reads (a staging buffer or the result's own popcount buffer)
};

}  // namespace bmb200
