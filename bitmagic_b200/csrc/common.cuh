// common.cuh -- shared device helpers for libbmb200 (sm_90a only).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/bmb200.h"

namespace bmb200 {

constexpr uint32_t kBlockWords = BMB200_BLOCK_WORDS;   // 2048 u32 = 8 KB = 65536 bits
constexpr uint32_t kGapMax     = BMB200_GAP_MAX_WORDS;
constexpr uint32_t kGapUnit    = BMB200_GAP_UNIT_WORDS; // u16 words per 16-byte arena unit

// rank-select borders, src/bmconst.h:120-124
constexpr uint32_t kRs3B0   = 21824u;
constexpr uint32_t kRs3B1   = 43648u;
constexpr uint32_t kRs3B0_1 = 32736u;
constexpr uint32_t kRs3B1_1 = 54560u;

// Device view of a packed column-major set (see bmb200_packed_set in include/bmb200.h).
struct SetView {
    uint32_t        n_vec;
    uint32_t        n_blocks;
    const uint32_t* desc;
    const uint64_t* bit_base;
    const uint64_t* gap_base;
    const uint32_t* bit_pool;
    const uint16_t* gap_pool;
};

// A GAP descriptor d addresses its block inside the column's GAP segment gseg (gap_pool + gap_base[nb] * kGapUnit): `unit` is
// the 16-byte arena unit the block is stored in, `pad` the u16 words before the block's header inside that unit.
struct GapAddr {
    const uint16_t* unit;
    uint32_t        pad;
};
__device__ __forceinline__ GapAddr gap_block_addr(const uint16_t* gseg, uint32_t d)
{
    const uint32_t rel = d >> 2;
    return {gseg + (size_t)(rel & BMB200_DESC_REL_MASK) * kGapUnit, rel >> 29};
}
// the GAP block of descriptor d: its header word, then its run ends
__device__ __forceinline__ const uint16_t* gap_block_ptr(const uint16_t* gseg, uint32_t d)
{
    const GapAddr a = gap_block_addr(gseg, d);
    return a.unit + a.pad;
}

// streaming 128-bit load: read-only path, do not allocate in L1 (each bit-block is read once)
__device__ __forceinline__ uint4 ld_stream_v4(const uint4* p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream_v4(uint4* p, const uint4& v)
{
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint32_t ld_nc_u32(const uint32_t* p)
{
    uint32_t r;
    asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ void red_or_shared(uint32_t* p, uint32_t v)
{
    asm volatile("red.shared.or.b32 [%0], %1;" :: "r"((uint32_t)__cvta_generic_to_shared(p)), "r"(v) : "memory");
}
__device__ __forceinline__ void red_xor_shared(uint32_t* p, uint32_t v)
{
    asm volatile("red.shared.xor.b32 [%0], %1;" :: "r"((uint32_t)__cvta_generic_to_shared(p)), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t warp_sum(uint32_t v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ uint32_t popc4(const uint4& v)
{
    return __popc(v.x) + __popc(v.y) + __popc(v.z) + __popc(v.w);
}
// mask of bits [lo, hi] inside one 32-bit word
__device__ __forceinline__ uint32_t bit_range_mask(uint32_t lo, uint32_t hi)
{
    return (0xffffffffu << lo) & (0xffffffffu >> (31u - hi));
}

}  // namespace bmb200
