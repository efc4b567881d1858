// Microbenchmark: cost of warp-level digit matching / histogram primitives on sm_90a.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o rank_primitives rank_primitives.cu && ./rank_primitives
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ unsigned lanemask_lt() { unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }
__device__ __forceinline__ uint32_t lcg(uint32_t &s) { s = s * 1664525u + 1013904223u; return s >> 8; }

__device__ __forceinline__ unsigned peers_ballot8(uint32_t d)
{
    unsigned peers = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < 8; b++) {
        const bool bit = (d >> b) & 1u;
        const unsigned bal = __ballot_sync(0xffffffffu, bit);
        peers &= bit ? bal : ~bal;
    }
    return peers;
}

template <int MODE>
__global__ void bench(uint32_t *out, int iters, uint32_t distinct_mask, long long *cycles)
{
    __shared__ uint32_t hist[8][256];
    const unsigned tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < 8 * 256; i += blockDim.x) (&hist[0][0])[i] = 0;
    __syncthreads();
    uint32_t seed = (blockIdx.x * blockDim.x + tid) * 2654435761u + 12345u;
    uint32_t acc = 0;
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
        const uint32_t d = lcg(seed) & distinct_mask;          // distinct_mask 0xff: ~28 distinct per warp; 0x01: 2 distinct
        if (MODE == 0) {            // MATCH.ANY
            acc += __match_any_sync(0xffffffffu, d);
        } else if (MODE == 1) {     // 8 ballots
            acc += peers_ballot8(d);
        } else if (MODE == 2) {     // smem atomicAdd, one per lane (spread addresses)
            atomicAdd(&hist[warp][d], 1u);
        } else if (MODE == 3) {     // ballot peers + leader plain RMW (rank-style, returns old)
            const unsigned peers = peers_ballot8(d);
            const int leader = __ffs(peers) - 1;
            uint32_t old = 0;
            if ((int)lane == leader) { old = hist[warp][d]; hist[warp][d] = old + __popc(peers); }
            __syncwarp();
            old = __shfl_sync(0xffffffffu, old, leader);
            acc += old + __popc(peers & lanemask_lt());
        } else if (MODE == 4) {     // MATCH.ANY + leader atomicAdd (the r01a ranking)
            const unsigned peers = __match_any_sync(0xffffffffu, d);
            const int leader = __ffs(peers) - 1;
            uint32_t old = 0;
            if ((int)lane == leader) old = atomicAdd(&hist[warp][d], (uint32_t)__popc(peers));
            old = __shfl_sync(0xffffffffu, old, leader);
            acc += old + __popc(peers & lanemask_lt());
        } else if (MODE == 5) {     // smem atomicAdd with return value (rank via atomics only; not stable, for cost only)
            acc += atomicAdd(&hist[warp][d], 1u);
        }
    }
    const long long t1 = clock64();
    out[blockIdx.x * blockDim.x + tid] = acc + hist[warp][lane];
    if (tid == 0) atomicAdd((unsigned long long *)cycles, (unsigned long long)(t1 - t0));
}

template <int MODE>
void run(const char *name, uint32_t mask, uint32_t *out, long long *cyc, int blocks, int threads, int sms)
{
    const int iters = 2000;
    cudaMemset(cyc, 0, 8);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    bench<MODE><<<blocks, threads>>>(out, 10, mask, cyc);
    cudaMemset(cyc, 0, 8);
    cudaEventRecord(e0);
    bench<MODE><<<blocks, threads>>>(out, iters, mask, cyc);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    long long c; cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    const double warp_ops = (double)blocks * (threads / 32) * iters;
    printf("%-44s mask %02x  blocks/SM %d x %d thr: %7.2f cycles/op/CTA-clock  %8.2f Gwarp-op/s  (%.3f ms)\n", name, mask,
           blocks / sms, threads, (double)c / blocks / iters, warp_ops / (ms * 1e6), ms);
}

int main()
{
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    const int sms = prop.multiProcessorCount;          // one full wave per occupancy level, whatever the chip
    uint32_t *out; long long *cyc;
    cudaMalloc(&out, (size_t)sms * 8 * 256 * 4); cudaMalloc(&cyc, 8);
    for (int occ : {1, 4, 8}) {
        const int blocks = sms * occ, threads = 256;
        for (uint32_t mask : {0xffu, 0x0fu, 0x01u}) {
            run<0>("MATCH.ANY", mask, out, cyc, blocks, threads, sms);
            run<1>("8x BALLOT peers", mask, out, cyc, blocks, threads, sms);
            run<2>("smem atomicAdd (no return)", mask, out, cyc, blocks, threads, sms);
            run<5>("smem atomicAdd (return)", mask, out, cyc, blocks, threads, sms);
            run<3>("ballot peers + leader RMW + shfl (rank)", mask, out, cyc, blocks, threads, sms);
            run<4>("MATCH.ANY + leader atomicAdd + shfl (rank)", mask, out, cyc, blocks, threads, sms);
        }
    }
    return 0;
}
