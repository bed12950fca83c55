// microbench_read.cu -- streaming 128-bit reads over a 13 GiB buffer (about the source bytes of one C3 step): the practical
// HBM read ceiling of the card it runs on, to quote the aggregation kernel against beside the data-sheet bandwidth.
// Every byte is read exactly once per pass, coalesced, no reuse; the best of a few (CTAs per SM, loads in flight) shapes is the ceiling.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/_bin/microbench_read scripts/microbench_read.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
template <int U>   // U independent 16-byte loads in flight per thread
__global__ void stream_read(const uint4* __restrict__ buf, uint64_t n, uint32_t* out)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    uint32_t acc = 0;
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    for (; i + (U - 1) * stride < n; i += U * stride) {
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
            asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(v[u].x), "=r"(v[u].y), "=r"(v[u].z), "=r"(v[u].w) : "l"(buf + i + u * stride));
#pragma unroll
        for (int u = 0; u < U; ++u) acc ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
    }
    for (; i < n; i += stride) { const uint4 v = buf[i]; acc ^= v.x ^ v.y ^ v.z ^ v.w; }
    if (acc == 0x9e3779b9u) out[0] = acc;     // keeps the loads alive
}
template <int U>
static float run(const uint4* buf, uint64_t n, uint32_t* out, uint32_t blocks, uint32_t threads)
{
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    float best = 1e30f;
    for (int rep = 0; rep < 4; ++rep) {       // rep 0 is the warm-up
        cudaEventRecord(a);
        stream_read<U><<<blocks, threads>>>(buf, n, out);
        cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b);
        if (rep && ms < best) best = ms;
    }
    cudaEventDestroy(a); cudaEventDestroy(b);
    return best;
}
int main()
{
    const uint64_t bytes = 13ull << 30, n = bytes / 16;
    uint4* buf; uint32_t* out;
    if (cudaMalloc(&buf, bytes) != cudaSuccess || cudaMalloc(&out, 4) != cudaSuccess) { printf("{\"error\": \"allocation\"}\n"); return 1; }
    cudaMemset(buf, 1, bytes);
    cudaDeviceSynchronize();
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    double best_gbs = 0;
    for (int per_sm = 1; per_sm <= 4; per_sm *= 2) {
        for (int u = 4; u <= 16; u *= 2) {
            const uint32_t threads = 512, blocks = (uint32_t)(sms * per_sm);
            const float ms = u == 4 ? run<4>(buf, n, out, blocks, threads) : u == 8 ? run<8>(buf, n, out, blocks, threads) : run<16>(buf, n, out, blocks, threads);
            const double gbs = bytes / (ms * 1e-3) / 1e9;
            if (gbs > best_gbs) best_gbs = gbs;
            printf("{\"ctas_per_sm\": %d, \"threads\": %u, \"loads_in_flight\": %d, \"bytes\": %llu, \"ms\": %.3f, \"GBps\": %.1f}\n",
                   per_sm, threads, u, (unsigned long long)bytes, ms, gbs);
        }
    }
    printf("{\"device\": \"%s\", \"read_ceiling_GBps\": %.1f}\n", prop.name, best_gbs);
    cudaFree(buf); cudaFree(out);
    return 0;
}
