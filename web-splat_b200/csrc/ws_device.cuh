// ws_device.cuh -- shared device-side definitions for the sm_90a splat render path.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace ws {

// ---- uniforms: byte-identical to the reference's uniform buffers -------------
struct CameraUniform {      // renderer.rs:290-306 / preprocess.wgsl:26-34, 272 B
    float view[16];         // column-major m[c*4+r]
    float view_inv[16];
    float proj[16];         // VIEWPORT_Y_FLIP * proj
    float proj_inv[16];
    float viewport[2];
    float focal[2];
};
struct RenderSettings {     // renderer.rs:604-619 / preprocess.wgsl:77-87, 80 B
    float clip_min[4];
    float clip_max[4];
    float gaussian_scaling;
    uint32_t max_sh_deg;
    uint32_t mip_splatting;
    float kernel_size;
    float walltime;
    float scene_extend;
    uint32_t _pad[2];
    float center[4];
};
struct Quant { int32_t zero_point; float scale; uint32_t _pad[2]; };
struct Quant4 { Quant color_dc, color_rest, opacity, scaling_factor; };

struct FrameUniforms {      // one device-resident block per renderer, rewritten per frame
    CameraUniform cam;
    RenderSettings rs;
    Quant4 quant;
    uint32_t width, height, tiles_x, tiles_y;
    uint32_t num_points, file_sh_deg, pair_capacity, _pad0;
    // per-frame constants of stage 1 that the shaders recompute per invocation (preprocess.wgsl:270-271, :263-264, :199);
    // divided once on the host in IEEE f32 -- the same bits a per-thread IEEE division gives
    float inv_viewport[2];      // 1 / viewport
    float znear, zfar;          // -proj[3][2] / proj[2][2],  -proj[3][2] / (proj[2][2] - 1)
    float inv_scene_extend;     // 1 / scene_extend
    float _padf[3];
};

// ---- per-frame device counters (zeroed by one memset per frame) ---------------
struct FrameCounters {
    uint32_t num_visible;       // V
    uint32_t num_pairs;         // P (pairs needed, may exceed capacity)
    uint32_t pair_overflow;     // 1 if P > capacity
    uint32_t error_flags;       // bit 0: a look-back spin exceeded SPIN_LIMIT (never expected)
    uint32_t ticket[12];        // dynamic partition tickets: [2..5] depth passes, [6..8] tile passes
    uint32_t num_local_visible; // sharded mode: survivors of the local shard (num_visible then counts the received ones)
    uint32_t scatter_done;      // sharded mode: CTAs of the exchange kernel that have finished (last one signals the peers)
    uint32_t composite_done;    // sharded mode: CTAs of the band compositor that have finished
    uint32_t num_pairs_near;    // occlusion split: pairs of the near slab (num_pairs then counts the far slab's)
    // occlusion split on one GPU (binning.cu: split_*): the slabs are cut by depth-key VALUE, not by sorted position
    uint32_t key_max;           // largest depth key of the visible splats (stage 1 count kernel)
    uint32_t key_min_inv;       // ~smallest depth key (atomicMax of ~key: the per-frame memset is the identity)
    uint32_t split_cut;         // near list = visible splats with key >= split_cut
    uint32_t num_near;          // length of the near list
    uint32_t num_far;           // far splats that survive the cull against the saturated tiles
    uint32_t cut_done;          // CTAs of the cut histogram that have finished (the last one picks the cut)
    uint32_t ticket_far[4];     // depth passes over the far survivors
    // exact pair totals (bin_scan_kernel): P can pass 2^32 (screen-filling splats at 16 K viewports), where the 32-bit
    // num_pairs / num_pairs_near above saturate at 0xffffffff -- those stay 32-bit, the tile-sort passes read them as n_ptr
    uint64_t num_pairs64;       // P of the only slab, or of the far slab of a split frame
    uint64_t num_pairs_near64;  // occlusion split: P of the near slab
};

constexpr int TILE = 16;                    // 16x16 pixel tiles
constexpr float CUTOFF = 2.3539888583335364f;               // gaussian.wgsl:2
constexpr float TWO_CUTOFF = 4.707977716667073f;            // discard threshold, gaussian.wgsl:62
constexpr float FOOTPRINT_R = 2.1697876f;                   // sqrt(2*CUTOFF)
constexpr float RECT_PAD = 0.05f;                           // px, conservative pad of the tile rect

// ---- decoupled look-back status words: [31:30] flag, [29:0] value -------------
constexpr uint32_t LB_FLAG_SHIFT = 30;
constexpr uint32_t LB_VALUE_MASK = 0x3fffffffu;
constexpr uint32_t LB_INVALID = 0u;
constexpr uint32_t LB_AGGREGATE = 1u << LB_FLAG_SHIFT;
constexpr uint32_t LB_PREFIX = 2u << LB_FLAG_SHIFT;
constexpr uint32_t SPIN_LIMIT = 1u << 26;    // watchdog: a stuck look-back flags an error instead of hanging the GPU

__device__ __forceinline__ uint32_t ld_relaxed(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(uint32_t *p, uint32_t v)
{
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Warp-parallel decoupled look-back over a chain of single-word statuses.
// Called by one full warp.  status[part] must already hold this partition's
// AGGREGATE (or nothing yet: the caller publishes).  Returns the exclusive prefix
// (sum of all partitions < part).  Each status word carries its own flag, so
// relaxed accesses suffice (no separate payload to order against).
__device__ __forceinline__ uint32_t lookback_warp(const uint32_t *status, uint32_t part, uint32_t *err)
{
    uint32_t spins = 0;
    const unsigned lane = threadIdx.x & 31u;
    uint32_t excl = 0;
    int64_t base = (int64_t)part - 1;          // window covers [base-31, base]
    while (base >= 0) {
        int64_t p = base - (int64_t)lane;
        uint32_t s;
        // spin until every lane's predecessor in the window (up to the first PREFIX) is valid
        for (;;) {
            s = (p >= 0) ? ld_relaxed(status + p) : LB_PREFIX;   // before partition 0: prefix 0
            unsigned pref = __ballot_sync(0xffffffffu, (s >> LB_FLAG_SHIFT) == 2u);
            unsigned inval = __ballot_sync(0xffffffffu, (s >> LB_FLAG_SHIFT) == 0u);
            unsigned upto = pref ? ((pref & (0u - pref)) << 1) - 1u : 0xffffffffu;   // lanes <= first prefix lane
            if ((inval & upto) == 0u) {
                uint32_t v = ((1u << lane) & upto) ? (s & LB_VALUE_MASK) : 0u;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                excl += v;
                if (pref) return excl;
                break;
            }
            if (++spins > SPIN_LIMIT) {
                if (lane == 0 && err) atomicOr(err, 1u);
                return excl;
            }
        }
        base -= 32;
    }
    return excl;
}

// ---- mbarrier + 1-D bulk async copy (TMA engine, UBLKCP) ----------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// global -> shared bulk copy; bytes multiple of 16, both addresses 16-B aligned
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---- cross-GPU signalling through peer-mapped memory (NVLink): release/acquire at system scope ----
__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v)
{
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// spin until *flag has reached `epoch` (epochs only grow; wrap-safe signed difference)
__device__ __forceinline__ bool wait_epoch(const uint32_t *flag, uint32_t epoch, uint32_t *err)
{
    for (uint32_t spins = 0; (int32_t)(ld_acquire_sys(flag) - epoch) < 0; ++spins) {
        if (spins > (SPIN_LIMIT << 2)) { if (err) atomicOr(err, 4u); return false; }   // ~1 s: a peer never arrived
        __nanosleep(64);
    }
    return true;
}

// Exclusive scan of counts[0..n) into bases[0..n) by ONE CTA of 1024 threads; returns the total (64-bit) to every thread.
// 16 K-element tiles, sixteen adjacent elements per thread (four 128-bit loads in flight before the first use): every
// element is read once, scanned in registers + shuffles, written once; three barriers per tile.  cfg3's 23.4 K partition
// counts are two tiles (4 K tiles would take six dependent trips).  The running total is kept in
// 64 bits: pair counts can exceed 2^32 (screen-filling splats); bases saturate at 0xffffffff, which every consumer
// treats as "beyond capacity", so an overflow is reported instead of wrapping into a silently wrong frame.
// counts / bases must be 16-byte aligned (they are 256-byte aligned slices of the scratch allocation).
// ACC = uint64_t where the total can exceed 2^32 (pair counts), uint32_t where it cannot (survivor counts <= N).
template <typename ACC>
__device__ __forceinline__ ACC block_exclusive_scan_1024(const uint32_t *__restrict__ counts, uint32_t *__restrict__ bases, uint32_t n)
{
    constexpr int E = 16;
    __shared__ ACC s_w[32];
    __shared__ ACC s_tot, s_carry;
    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024u * E) {
        const uint32_t i0 = base + tid * E;
        uint32_t c[E];
        if (i0 + E <= n) {
            const uint4 *p4 = reinterpret_cast<const uint4 *>(counts + i0);
#pragma unroll
            for (int q = 0; q < E / 4; q++) { const uint4 v = p4[q]; c[4 * q] = v.x; c[4 * q + 1] = v.y; c[4 * q + 2] = v.z; c[4 * q + 3] = v.w; }
        } else {
#pragma unroll
            for (int k = 0; k < E; k++) c[k] = (i0 + k < n) ? counts[i0 + k] : 0u;
        }
        ACC sum = 0;
#pragma unroll
        for (int k = 0; k < E; k++) sum += c[k];
        ACC incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const ACC t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((int)lane >= o) incl += t;
        }
        if (lane == 31) s_w[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const ACC v = s_w[lane];
            ACC vi = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const ACC t = __shfl_up_sync(0xffffffffu, vi, o);
                if ((int)lane >= o) vi += t;
            }
            s_w[lane] = vi - v;                                   // exclusive offset of each warp
            if (lane == 31) s_tot = vi;
        }
        __syncthreads();
        ACC run = s_carry + s_w[warp] + incl - sum;
        if (i0 + E <= n) {
            uint32_t o[E];
#pragma unroll
            for (int k = 0; k < E; k++) { o[k] = (sizeof(ACC) > 4 && (uint64_t)run > 0xffffffffull) ? 0xffffffffu : (uint32_t)run; run += c[k]; }
            uint4 *p4 = reinterpret_cast<uint4 *>(bases + i0);
#pragma unroll
            for (int q = 0; q < E / 4; q++) p4[q] = make_uint4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
        } else {
#pragma unroll
            for (int k = 0; k < E; k++) {
                if (i0 + k < n) bases[i0 + k] = (sizeof(ACC) > 4 && (uint64_t)run > 0xffffffffull) ? 0xffffffffu : (uint32_t)run;
                run += c[k];
            }
        }
        __syncthreads();                                           // everyone has read s_carry / s_w
        if (tid == 0) s_carry += s_tot;
        __syncthreads();
    }
    return s_carry;
}

// Per-rank mailbox other ranks write into (sharded frame without host-side collectives).
// Double buffered by frame parity: a fast rank can be at most one frame ahead of a slow one.
struct ShardMailbox {
    uint32_t matrix[2][64];     // [parity][src * world + dst]: splats of rank src that touch band dst
    uint32_t flag_rows[8];      // epoch of the last count row received from each source rank
    uint32_t flag_xchg[8];      // epoch whose exchange stores from each source rank have landed
    uint32_t flag_band[8];      // epoch whose band pixels from each rank have landed (read on the root)
    uint32_t _pad[104];
};

__device__ __forceinline__ unsigned lanemask_lt()
{
    unsigned m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

}  // namespace ws
