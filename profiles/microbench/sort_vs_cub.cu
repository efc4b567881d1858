// sort_vs_cub.cu -- same-box yard-stick for the onesweep (SURVEY.md 8(d)(ii), VERDICT r01 item 2):
// this repo's radix-sort passes (web-splat_b200/csrc/radix_sort.cu, linked as an object file) against
// cub::DeviceRadixSort::SortPairs on the two shapes of a cfg3 frame:
//   (a) depth sort : V = 5.9 M (u32 key = bit pattern of a positive f32 depth, u32 slot), 32 key bits, 4 passes
//   (b) tile sort  : P = 21 M  (u32 tile id < 8160 in short consecutive runs, u32 slot), 13 key bits, 2 passes
// Both sorts are stable LSD radix sorts, so the outputs must be bit-identical: checked here.
//
// build (done by profiles/microbench/build.sh):
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I web-splat_b200/csrc -I include \
//        profiles/microbench/sort_vs_cub.cu web-splat_b200/build/radix_sort.o -o profiles/microbench/sort_vs_cub
// run:  WS_SORT_VARIANT=2 ./sort_vs_cub   (1 = the round-1 pass)
#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "ws_kernels.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(2); } } while (0)

static uint64_t rng_state = 0x9e3779b97f4a7c15ull;
static inline uint32_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return (uint32_t)(rng_state >> 16); }

struct Result { double ours_min, ours_med, ours_passes_min, cub_min, cub_med; bool same; };

static Result run_shape(const char *name, const std::vector<uint32_t> &keys, int key_bits, int sm_count, int reps)
{
    using namespace ws;
    const uint32_t n = (uint32_t)keys.size();
    const int passes = (key_bits + 7) / 8;
    std::vector<uint32_t> vals(n);
    for (uint32_t i = 0; i < n; i++) vals[i] = i;
    uint32_t *d_k0, *d_v0, *kb[2], *vb[2], *ck[2], *cv[2];
    CK(cudaMalloc(&d_k0, (size_t)n * 4)); CK(cudaMalloc(&d_v0, (size_t)n * 4));
    for (int i = 0; i < 2; i++) { CK(cudaMalloc(&kb[i], (size_t)n * 4 + 65536)); CK(cudaMalloc(&vb[i], (size_t)n * 4 + 65536)); CK(cudaMalloc(&ck[i], (size_t)n * 4)); CK(cudaMalloc(&cv[i], (size_t)n * 4)); }
    CK(cudaMemcpy(d_k0, keys.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_v0, vals.data(), (size_t)n * 4, cudaMemcpyHostToDevice));

    const size_t sparts = ((size_t)n + SORT_PART - 1) / SORT_PART, gparts = (sparts + SORT_LB_GROUP - 1) / SORT_LB_GROUP;
    const size_t scratch_words = 8 + 4 * 256 + (size_t)passes * (sparts + gparts) * 256;
    uint32_t *scratch; CK(cudaMalloc(&scratch, scratch_words * 4));
    const int grid = sm_count * sort_pass_blocks_per_sm();

    size_t cub_bytes = 0;
    cub::DoubleBuffer<uint32_t> dbk(ck[0], ck[1]), dbv(cv[0], cv[1]);
    CK(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, dbk, dbv, (int)n, 0, key_bits));
    void *cub_tmp; CK(cudaMalloc(&cub_tmp, cub_bytes));

    cudaEvent_t e0, e1, e2; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); CK(cudaEventCreate(&e2));
    std::vector<float> t_ours, t_passes, t_cub;
    int out_ours = 0;
    for (int r = 0; r < reps + 3; r++) {
        // ---- ours: scratch clear + digit histograms + passes (the frame fuses the histograms into the producers)
        CK(cudaMemcpyAsync(kb[0], d_k0, (size_t)n * 4, cudaMemcpyDeviceToDevice)); CK(cudaMemcpyAsync(vb[0], d_v0, (size_t)n * 4, cudaMemcpyDeviceToDevice));
        CK(cudaEventRecord(e0));
        CK(cudaMemsetAsync(scratch, 0, scratch_words * 4));
        CK(cudaMemcpyAsync(scratch, &n, 4, cudaMemcpyHostToDevice));
        uint32_t *n_ptr = scratch, *tickets = scratch + 4, *hist = scratch + 8, *status = scratch + 8 + 4 * 256, *gstatus = status + (size_t)passes * sparts * 256;
        CK(launch_sort_histogram(kb[0], n_ptr, n, hist, passes, sm_count * 4, 0));
        CK(cudaEventRecord(e1));
        int src = 0;
        for (int p = 0; p < passes; p++) {
            SortPassArgs a;
            a.keys_in = kb[src]; a.vals_in = vb[src]; a.keys_out = kb[src ^ 1]; a.vals_out = vb[src ^ 1];
            a.n_ptr = n_ptr; a.n_cap = n; a.status = status + (size_t)p * sparts * 256; a.gstatus = gstatus + (size_t)p * gparts * 256;
            a.ticket = tickets + p; a.hist = hist + p * 256; a.shift = 8u * (uint32_t)p; a.err = nullptr; a.ranges = nullptr;
            CK(launch_sort_pass(a, grid, 0));
            src ^= 1;
        }
        out_ours = src;
        CK(cudaEventRecord(e2));
        CK(cudaEventSynchronize(e2));
        float a_ms, b_ms; CK(cudaEventElapsedTime(&a_ms, e0, e2)); CK(cudaEventElapsedTime(&b_ms, e1, e2));
        if (r >= 3) { t_ours.push_back(a_ms); t_passes.push_back(b_ms); }
        // ---- CUB
        CK(cudaMemcpyAsync(ck[0], d_k0, (size_t)n * 4, cudaMemcpyDeviceToDevice)); CK(cudaMemcpyAsync(cv[0], d_v0, (size_t)n * 4, cudaMemcpyDeviceToDevice));
        dbk = cub::DoubleBuffer<uint32_t>(ck[0], ck[1]); dbv = cub::DoubleBuffer<uint32_t>(cv[0], cv[1]);
        CK(cudaEventRecord(e0));
        CK(cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, dbk, dbv, (int)n, 0, key_bits));
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float c_ms; CK(cudaEventElapsedTime(&c_ms, e0, e1));
        if (r >= 3) t_cub.push_back(c_ms);
    }
    std::vector<uint32_t> ok(n), ov(n), xk(n), xv(n);
    CK(cudaMemcpy(ok.data(), kb[out_ours], (size_t)n * 4, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(ov.data(), vb[out_ours], (size_t)n * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(xk.data(), dbk.Current(), (size_t)n * 4, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(xv.data(), dbv.Current(), (size_t)n * 4, cudaMemcpyDeviceToHost));
    Result R;
    R.same = (memcmp(ok.data(), xk.data(), (size_t)n * 4) == 0) && (memcmp(ov.data(), xv.data(), (size_t)n * 4) == 0);
    auto mn = [](std::vector<float> &v) { return (double)*std::min_element(v.begin(), v.end()); };
    auto md = [](std::vector<float> &v) { std::sort(v.begin(), v.end()); return (double)v[v.size() / 2]; };
    R.ours_min = mn(t_ours); R.ours_med = md(t_ours); R.ours_passes_min = mn(t_passes); R.cub_min = mn(t_cub); R.cub_med = md(t_cub);
    const double bytes = (double)n * 16.0 * passes;
    printf("{\"shape\": \"%s\", \"n\": %u, \"key_bits\": %d, \"passes\": %d, \"variant\": \"%s\", "
           "\"ours_ms_min\": %.4f, \"ours_ms_median\": %.4f, \"ours_passes_only_ms_min\": %.4f, \"ours_ms_per_pass\": %.4f, "
           "\"cub_ms_min\": %.4f, \"cub_ms_median\": %.4f, \"speedup_vs_cub\": %.3f, \"ours_pass_GBs\": %.1f, \"identical_to_cub\": %s}\n",
           name, n, key_bits, passes, getenv("WS_SORT_VARIANT") ? getenv("WS_SORT_VARIANT") : "default",
           R.ours_min, R.ours_med, R.ours_passes_min, R.ours_passes_min / passes, R.cub_min, R.cub_med, R.cub_min / R.ours_min,
           bytes / (R.ours_passes_min * 1e-3) / 1e9, R.same ? "true" : "false");
    fflush(stdout);
    cudaFree(d_k0); cudaFree(d_v0); cudaFree(scratch); cudaFree(cub_tmp);
    for (int i = 0; i < 2; i++) { cudaFree(kb[i]); cudaFree(vb[i]); cudaFree(ck[i]); cudaFree(cv[i]); }
    return R;
}

int main(int argc, char **argv)
{
    int reps = argc > 1 ? atoi(argv[1]) : 20;
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    bool all_same = true;
    {   // (a) depth keys: zfar - clip.z of a cube seen from 3 units away: positive floats in ~[0.4, 6.3]
        const uint32_t n = 5926921u;
        std::vector<uint32_t> k(n);
        for (uint32_t i = 0; i < n; i++) { float f = 0.4f + 5.9f * (float)(rnd() & 0xffffff) / 16777216.f; memcpy(&k[i], &f, 4); }
        all_same &= run_shape("depth_V5.9M_32bit", k, 32, prop.multiProcessorCount, reps).same;
    }
    {   // (b) tile ids as bin_expand emits them: per splat a w x h rectangle of tiles, row-major, consecutive in x
        const uint32_t target = 20980000u, tx = 120, ty = 68;
        std::vector<uint32_t> k; k.reserve(target + 64);
        while (k.size() < target) {
            const uint32_t w = 1 + rnd() % 3, h = 1 + rnd() % 2, x0 = rnd() % (tx - w + 1), y0 = rnd() % (ty - h + 1);
            for (uint32_t y = 0; y < h; y++) for (uint32_t x = 0; x < w; x++) k.push_back((y0 + y) * tx + x0 + x);
        }
        k.resize(target);
        all_same &= run_shape("tile_P21M_13bit", k, 13, prop.multiProcessorCount, reps).same;
        // near-slab size of a split frame
        k.resize(10500000u);
        all_same &= run_shape("tile_P10.5M_13bit", k, 13, prop.multiProcessorCount, reps).same;
    }
    {   // ragged size + 24-bit keys (compressed layout): identity top pass
        const uint32_t n = 1000003u;
        std::vector<uint32_t> k(n);
        for (uint32_t i = 0; i < n; i++) k[i] = rnd() & 0xffffffu;
        all_same &= run_shape("ragged_1000003_32bit_of_24", k, 32, prop.multiProcessorCount, reps).same;
    }
    return all_same ? 0 : 1;
}
