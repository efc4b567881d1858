// radix_sort.cu -- stage 2: onesweep LSD radix sort of (u32 key, u32 value) pairs on sm_90a.
//
// Replaces the reference's Fuchsia-derived WGSL sort (radix_sort.wgsl:48-512, driven by
// gpu_rs.rs:764-863): same contract -- stable, ascending, 8-bit digits, result back in the
// input buffers after an even number of passes -- but one kernel per digit pass:
//   * persistent CTAs take 4096-pair partitions from an atomic ticket (forward progress
//     for the decoupled look-back does not depend on the hardware's CTA scheduling order,
//     which radix_sort.wgsl:365-387 silently relies on);
//   * ranking: each lane ORs its lane bit into a per-warp, per-digit peer mask in shared memory
//     (atomicOr without return), reads the mask back and the lowest peer bumps the warp's
//     private digit counter with a plain read-modify-write.  MATCH.ANY on random 8-bit digits
//     costs more the more distinct values a warp holds, and an 8-ballot emulation is also slower
//     than shared atomics without return (profiles/microbench/rank_primitives.cu compares the
//     three); the reference emulates match with a per-key shared-memory loop (radix_sort.wgsl:283-302);
//   * decoupled look-back, one thread per digit bin, on single 32-bit status words
//     (2-bit flag | 30-bit count: relaxed accesses suffice), TWO levels deep: partitions are
//     grouped by 16 and the last partition of a group publishes the group's aggregate /
//     inclusive prefix.  A persistent grid starts W partitions at once, none of which has a
//     prefix yet; a flat look-back then reads W^2/2 status rows (100 MB of L2 traffic for
//     W=444), the two-level one 15 + W/16 rows per partition;
//   * keys/values are reordered in shared memory and leave as per-bin contiguous runs;
//   * the last tile-id pass also emits the per-tile [begin,end) ranges (atomicMin on run
//     boundaries), which removes a separate sweep over the sorted pair list.
// The digit histograms are produced by the kernels that generate the keys (preprocess /
// binning), so a pass reads each pair exactly once: 16 B of traffic per pair per pass.
#include "ws_device.cuh"
#include "ws_kernels.h"

#include <stdlib.h>

namespace ws {

namespace {

constexpr int WARPS = SORT_THREADS / 32;
#ifndef WS_RANK_WAYS
#define WS_RANK_WAYS 1                         // items ranked per step; 1, 2 and 4 are built (WS_RANK_WAYS env). 1 was fastest on the cfg3 tile pass -- the pass is bound by shared-memory wavefronts (bank conflicts on random digits), not by the dependent chain
#endif
struct LbState { uint32_t excl; bool done; };

// Walk one level of status words from row p down to row lo (nearest predecessor first).
// `col` already points at this thread's bin column.  Up to LB_WIDTH relaxed loads are issued per
// step (they are independent), then consumed in order; an unpublished word restarts the step at
// that row.  Rows below lo end the level; when `below_is_prefix` they count as "inclusive prefix 0".
// LB_WIDTH: with 4 loads per step a large share of the pass's instructions and stalls sat in this loop:
// the walk over up to 15 + W/16 rows -- a persistent grid starts W partitions at once (W = 396 on
// 132 SMs), none with a prefix -- cost ~8 dependent L2 round trips per partition; 16 loads per step make it ~3.
#ifndef WS_LB_WIDTH
#define WS_LB_WIDTH 16
#endif
constexpr int LB_WIDTH = WS_LB_WIDTH;

__device__ __forceinline__ void lookback_level(const uint32_t *col, int p, int lo, bool below_is_prefix,
                                               LbState &st, uint32_t *err)
{
    uint32_t spins = 0;
    while (!st.done) {
        if (p < lo) { if (below_is_prefix) st.done = true; return; }
        const int n = p - lo;                                  // extra rows available beyond p
        uint32_t s[LB_WIDTH];
#pragma unroll
        for (int k = 0; k < LB_WIDTH; k++) s[k] = (n >= k) ? ld_relaxed(col + (size_t)(p - k) * 256u) : 0u;
        if ((s[0] >> LB_FLAG_SHIFT) == 0u) {                   // nearest one not published yet: poll again
            if (++spins > SPIN_LIMIT) { if (err) atomicOr(err, 1u); st.done = true; }
            continue;
        }
#pragma unroll
        for (int k = 0; k < LB_WIDTH; k++) {
            if (n < k || (s[k] >> LB_FLAG_SHIFT) == 0u) break;          // beyond the level / not published: next step starts here
            st.excl += s[k] & LB_VALUE_MASK; --p;
            if ((s[k] >> LB_FLAG_SHIFT) == 2u) { st.done = true; return; }
        }
    }
}

#ifndef WS_SORT_CTAS
// resident CTAs per SM the pass is compiled for (A/B knob).  On sm_90a, 3 caps the pass at 80 registers and it spills;
// 2 (122 registers, no spill) sorts 15-20 % faster on H100 (profiles/microbench: sort_vs_cub vs sort_vs_cub_c3, every shape), 4 is slower still
#define WS_SORT_CTAS 2
#endif
template <bool EMIT_RANGES, int RANK_WAYS>
__global__ void __launch_bounds__(SORT_THREADS, WS_SORT_CTAS)   // 16 items per thread
onesweep_pass_kernel(SortPassArgs a)
{
    __shared__ __align__(16) uint32_t s_keys[SORT_PART];      // during ranking s_keys / s_vals double as the peer masks
    __shared__ __align__(16) uint32_t s_vals[SORT_PART];
    __shared__ uint32_t s_whist[WARPS][256];
    __shared__ uint32_t s_binstart[256];      // first local position of each bin in the partition
    __shared__ uint32_t s_gbase[256];         // global position of local position 0, per bin
    __shared__ uint32_t s_scan[WARPS];
    __shared__ uint32_t s_part;

    static_assert(SORT_ITEMS % RANK_WAYS == 0 && WARPS * RANK_WAYS * 256 <= 2 * SORT_PART, "peer masks must fit in s_keys + s_vals");
    static_assert((WARPS * RANK_WAYS * 256) % (4 * SORT_THREADS) == 0, "mask area is cleared with one uint4 per thread and step");
    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    uint32_t n = *a.n_ptr;
    if (n > a.n_cap) n = a.n_cap;
    const uint32_t nparts = (n + SORT_PART - 1u) / SORT_PART;
    const uint32_t shift = a.shift;

    // exclusive scan of the global digit histogram: thread tid owns bin tid
    uint32_t g_excl;
    {
        const uint32_t c = a.hist[tid];
        uint32_t incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((int)lane >= o) incl += t;
        }
        if (lane == 31) s_scan[warp] = incl;
        // a pass whose digit is the same for every key (one bin holds all n keys: the top byte of the compressed layout's
        // 24-bit depth key) is the identity permutation: stream the pairs through, no ranking, no look-back
        const int ident = __syncthreads_or((n > 0u && c == n) ? 1 : 0);
        uint32_t woff = 0;
#pragma unroll
        for (int w = 0; w < WARPS; w++) if (w < (int)warp) woff += s_scan[w];
        g_excl = woff + incl - c;
        __syncthreads();
        if (ident) {
            for (uint32_t i = blockIdx.x * SORT_THREADS + tid; i < n; i += gridDim.x * SORT_THREADS) {
                const uint32_t kk = a.keys_in[i];
                if (a.keys_out) a.keys_out[i] = kk;
                a.vals_out[i] = a.vals_in[i];
                if (EMIT_RANGES) {
                    const bool first = (i == 0u) || (a.keys_in[i - 1u] != kk);
                    const bool last = (i == n - 1u) || (a.keys_in[i + 1u] != kk);
                    if (first) atomicMin(&a.ranges[kk].x, i);
                    if (last) atomicMin(&a.ranges[kk].y, ~(i + 1u));
                }
            }
            return;
        }
    }

    for (;;) {
        if (tid == 0) s_part = atomicAdd(a.ticket, 1u);
        __syncthreads();
        const uint32_t part = s_part;
        if (part >= nparts) break;
        const uint32_t base = part * SORT_PART;
        const uint32_t nvalid = (n - base < (uint32_t)SORT_PART) ? (n - base) : (uint32_t)SORT_PART;
        const bool full = nvalid == (uint32_t)SORT_PART;

        // ---- load keys, warp-striped: warp w owns [base + w*512, +512), item i of lane l = i*32 + l
        uint32_t key[SORT_ITEMS];
        const uint32_t wbase = warp * (32u * SORT_ITEMS);
        if (full) {
#pragma unroll
            for (int i = 0; i < SORT_ITEMS; i++) key[i] = a.keys_in[base + wbase + i * 32u + lane];
        } else {
#pragma unroll
            for (int i = 0; i < SORT_ITEMS; i++) {
                const uint32_t li = wbase + i * 32u + lane;
                key[i] = (li < nvalid) ? a.keys_in[base + li] : 0xffffffffu;   // pads rank last (radix_sort.wgsl:79)
            }
        }
        // peer masks: RANK_WAYS x 256 words per warp, carved out of s_keys / s_vals (free until the reorder)
#pragma unroll
        for (int i = 0; i < WARPS; i++) s_whist[i][tid] = 0u;
        {
            uint4 *zk = reinterpret_cast<uint4 *>(s_keys), *zv = reinterpret_cast<uint4 *>(s_vals);
            const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int i = 0; i < (WARPS * RANK_WAYS * 256) / (4 * SORT_THREADS); i++) {
                const unsigned w = i * SORT_THREADS + tid;              // uint4 index over the mask area
                if (w < SORT_PART / 4u) zk[w] = z4; else zv[w - SORT_PART / 4u] = z4;
            }
        }
        __syncthreads();

        // ---- rank inside the warp.  Each lane ORs its lane bit into the peer mask of its digit (atomicOr without
        //      return), reads the mask back, and the lowest peer advances the warp's digit counter.  RANK_WAYS items
        //      are ranked per step with independent shared-memory chains: item j's rank adds the peer counts of the
        //      items before it in the step for its own digit (their masks are complete after the same warp barrier).
        uint32_t rank2[SORT_ITEMS / 2];       // two 16-bit ranks per register (a rank is < 512)
        {
            uint32_t *wh = s_whist[warp];
            const unsigned mw = warp * (RANK_WAYS * 256u);
            uint32_t *wm = (mw < (unsigned)SORT_PART) ? (s_keys + mw) : (s_vals + (mw - SORT_PART));
            const uint32_t lanebit = 1u << lane, lower = lanebit - 1u;
#pragma unroll
            for (int i0 = 0; i0 < SORT_ITEMS; i0 += RANK_WAYS) {
                uint32_t d[RANK_WAYS], peers[RANK_WAYS], rk[RANK_WAYS];
#pragma unroll
                for (int j = 0; j < RANK_WAYS; j++) {
                    d[j] = (key[i0 + j] >> shift) & 255u;
                    atomicOr(&wm[j * 256 + d[j]], lanebit);
                }
                __syncwarp();
#pragma unroll
                for (int j = 0; j < RANK_WAYS; j++) {
                    peers[j] = wm[j * 256 + d[j]];
                    rk[j] = wh[d[j]] + (uint32_t)__popc(peers[j] & lower);      // counter: same value for all peers
#pragma unroll
                    for (int e = 0; e < j; e++) rk[j] += (uint32_t)__popc(wm[e * 256 + d[j]]);
                }
                __syncwarp();
#pragma unroll
                for (int j = 0; j < RANK_WAYS; j++) {
                    if ((peers[j] & lower) == 0u) {                              // lowest peer: advance the counter, clear the mask
                        atomicAdd(&wh[d[j]], (uint32_t)__popc(peers[j]));
                        wm[j * 256 + d[j]] = 0u;
                    }
                    const int i = i0 + j;
                    if (i & 1) rank2[i >> 1] |= rk[j] << 16; else rank2[i >> 1] = rk[j];
                }
                __syncwarp();
            }
        }
        __syncthreads();

        // ---- per bin (thread tid = bin): scan over warps, publish the partition's aggregate
        uint32_t total = 0;
#pragma unroll
        for (int w = 0; w < WARPS; w++) {
            const uint32_t c = s_whist[w][tid];
            s_whist[w][tid] = total;
            total += c;
        }
        uint32_t *st = a.status + (size_t)part * 256u + tid;
        st_relaxed(st, (part == 0u ? LB_PREFIX : LB_AGGREGATE) | total);

        // values are needed only for the reorder: issue their loads now
#if WS_SORT_CTAS >= 4
        constexpr int VAL_NOW = SORT_ITEMS / 2;        // 64-register build: the second half is loaded inside the reorder
#else
        constexpr int VAL_NOW = SORT_ITEMS;
#endif
        uint32_t val[SORT_ITEMS];
        if (full) {
#pragma unroll
            for (int i = 0; i < VAL_NOW; i++) val[i] = a.vals_in[base + wbase + i * 32u + lane];
        } else {
#pragma unroll
            for (int i = 0; i < VAL_NOW; i++) {
                const uint32_t li = wbase + i * 32u + lane;
                val[i] = (li < nvalid) ? a.vals_in[base + li] : 0u;
            }
        }

        // block exclusive scan of `total` over bins -> first local position of each bin
        uint32_t binstart;
        {
            uint32_t incl = total;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
                if ((int)lane >= o) incl += t;
            }
            if (lane == 31) s_scan[warp] = incl;
            __syncthreads();                                   // also: every warp is done with the peer masks in s_keys
            uint32_t woff = 0;
#pragma unroll
            for (int w = 0; w < WARPS; w++) if (w < (int)warp) woff += s_scan[w];
            binstart = woff + incl - total;
        }
        s_binstart[tid] = binstart;
        __syncthreads();

        // ---- reorder in shared memory (needs only block-local information); meanwhile the
        //      predecessors get time to publish, which shortens the look-back below
#if WS_SORT_CTAS >= 4
#pragma unroll
        for (int i = VAL_NOW; i < SORT_ITEMS; i++) {
            const uint32_t li = wbase + i * 32u + lane;
            val[i] = (li < nvalid) ? a.vals_in[base + li] : 0u;
        }
#endif
#pragma unroll
        for (int i = 0; i < SORT_ITEMS; i++) {
            const uint32_t d = (key[i] >> shift) & 255u;
            const uint32_t pos = s_binstart[d] + s_whist[warp][d] + ((rank2[i >> 1] >> ((i & 1) * 16)) & 0xffffu);
            s_keys[pos] = key[i];
            s_vals[pos] = val[i];
        }

        // ---- two-level decoupled look-back
        LbState lb; lb.excl = 0; lb.done = (part == 0u);
        {
            const uint32_t grp = part / SORT_LB_GROUP;
            const bool leader = (part % SORT_LB_GROUP) == SORT_LB_GROUP - 1u;
            lookback_level(a.status + tid, (int)part - 1, (int)(grp * SORT_LB_GROUP), grp == 0u, lb, a.err);   // inside the group
            uint32_t *gst = a.gstatus + (size_t)grp * 256u + tid;
            if (leader) st_relaxed(gst, (lb.done ? LB_PREFIX : LB_AGGREGATE) | ((lb.excl + total) & LB_VALUE_MASK));
            if (!lb.done) {
                lookback_level(a.gstatus + tid, (int)grp - 1, 0, true, lb, a.err);                            // over earlier groups
                if (leader) st_relaxed(gst, LB_PREFIX | ((lb.excl + total) & LB_VALUE_MASK));
            }
            if (part > 0u) st_relaxed(st, LB_PREFIX | ((lb.excl + total) & LB_VALUE_MASK));
        }
        s_gbase[tid] = g_excl + lb.excl - binstart;            // wraps mod 2^32 by design
        __syncthreads();

        // ---- write out: consecutive threads write consecutive addresses within a bin run
#pragma unroll
        for (int k = 0; k < SORT_ITEMS; k++) {
            const uint32_t i = tid + k * SORT_THREADS;
            if (i < nvalid) {
                const uint32_t kk = s_keys[i];
                const uint32_t g = s_gbase[(kk >> shift) & 255u] + i;
                if (a.keys_out) a.keys_out[g] = kk;           // NULL on the last tile pass: nothing downstream reads the sorted tile ids
                a.vals_out[g] = s_vals[i];
                if (EMIT_RANGES) {
                    // The output of the last pass is fully sorted, so equal keys are contiguous in
                    // global memory.  Inside a bin run local neighbours are global neighbours; at
                    // run boundaries the global neighbour is unknown, hence min/max via atomics.
                    const bool first = (i == 0u) || (s_keys[i - 1u] != kk);
                    const bool last = (i == nvalid - 1u) || (s_keys[i + 1u] != kk);
                    if (first) atomicMin(&a.ranges[kk].x, g);
                    if (last) atomicMin(&a.ranges[kk].y, ~(g + 1u));
                }
            }
        }
        __syncthreads();
    }
}


// ---------------------------------------------------------------------------------------------------------------
// V2 of the pass (WS_SORT_VARIANT=2; NOT the default): what profiling named on V1 (short and long scoreboard stalls,
// many shared-memory wavefront cycles per warp-item on random digits) is attacked three ways:
//   * TMA staging: the NEXT partition's keys and values (2 x 16 KB) are fetched by cp.async.bulk (UBLKCP) into a
//     staging buffer while the current partition is in its look-back and write-out; the ticket of the next partition
//     is taken at the top of the iteration, so neither the ticket round trip nor the two global-load latencies sit
//     on the per-partition critical path any more.  Values never pass through registers (80 -> ~56 registers);
//   * ranking on packed {peer mask, running count} 64-bit words: one atomicOr, one LDS.64 and one STS.64 by the
//     lowest peer per item (V1: atomicOr + two LDS + atomicAdd + STS);
//   * the reorder reads ONE table entry (bin start + warp prefix, merged after the per-bin scan) and writes ONE
//     64-bit {key, value} word; the write-out reads it back with one LDS.64.
// Also: a pass whose digit is the same for every key (one histogram bin holds all n keys -- the top byte of the
// compressed layout's 24-bit key) degenerates to a plain copy, and the last tile pass may skip the key store
// (keys_out == NULL: the compositor only needs the values and the tile ranges).
// RESULT: no faster than V1 on its own -- neither the load latency nor the shared-memory wavefronts were the bound; the
// look-back walk was (see lookback_level) -- and with two frames in flight the frame rate fell to a fraction: 3 CTAs x
// 75 KB take nearly all of an SM's 228 KB of shared memory, so no kernel of the other frame can ever share an SM with a
// sort pass.  V1 (41 KB static) stays the default; V2 is kept as the TMA-staged alternative.
struct SortSmemV2 {
    uint32_t stage_k[SORT_PART];              // TMA destination: next partition's keys ...
    uint32_t stage_v[SORT_PART];              // ... and values
    uint2 kv[SORT_PART];                      // reorder buffer; its first 16 KB hold the {mask, count} words while ranking
    uint32_t tbl[WARPS][256];                 // first local position of (warp, bin) in the partition
    uint32_t gbase[256];
    uint32_t scan[WARPS];
    uint32_t part;
    uint64_t bar;
};

template <bool EMIT_RANGES>
__global__ void __launch_bounds__(SORT_THREADS, 3)
onesweep_pass_v2_kernel(SortPassArgs a)
{
    extern __shared__ __align__(128) uint8_t smem_raw[];
    SortSmemV2 &S = *reinterpret_cast<SortSmemV2 *>(smem_raw);
    static_assert(WARPS * 256 * sizeof(uint2) <= sizeof(S.kv), "rank words must fit in the reorder buffer");

    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    uint32_t n = *a.n_ptr;
    if (n > a.n_cap) n = a.n_cap;
    const uint32_t nparts = (n + SORT_PART - 1u) / SORT_PART;
    const uint32_t shift = a.shift;
    const bool use_tma = ((reinterpret_cast<uintptr_t>(a.keys_in) | reinterpret_cast<uintptr_t>(a.vals_in)) & 15u) == 0u;

    // exclusive scan of the global digit histogram (thread tid owns bin tid) + "every key has the same digit"
    uint32_t g_excl;
    {
        const uint32_t c = a.hist[tid];
        uint32_t incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((int)lane >= o) incl += t;
        }
        if (lane == 31) S.scan[warp] = incl;
        if (tid == 0) { mbar_init(&S.bar, 1); fence_mbar_init(); }
        const int ident = __syncthreads_or((n > 0u && c == n) ? 1 : 0);
        uint32_t woff = 0;
#pragma unroll
        for (int w = 0; w < WARPS; w++) if (w < (int)warp) woff += S.scan[w];
        g_excl = woff + incl - c;
        if (ident) {
            // identity permutation: stream the pairs through (grid-stride, no ranking, no look-back)
            for (uint32_t i = blockIdx.x * SORT_THREADS + tid; i < n; i += gridDim.x * SORT_THREADS) {
                const uint32_t kk = a.keys_in[i];
                if (a.keys_out) a.keys_out[i] = kk;
                a.vals_out[i] = a.vals_in[i];
                if (EMIT_RANGES) {
                    const bool first = (i == 0u) || (a.keys_in[i - 1u] != kk);
                    const bool last = (i == n - 1u) || (a.keys_in[i + 1u] != kk);
                    if (first) atomicMin(&a.ranges[kk].x, i);
                    if (last) atomicMin(&a.ranges[kk].y, ~(i + 1u));
                }
            }
            return;
        }
    }

    auto issue = [&](uint32_t part) {                 // thread 0: stage a FULL partition through the TMA engine
        fence_proxy_async();                          // earlier generic-proxy reads of the stage happen-before the async writes
        mbar_arrive_expect_tx(&S.bar, 2u * SORT_PART * 4u);
        bulk_g2s(S.stage_k, a.keys_in + (size_t)part * SORT_PART, SORT_PART * 4u, &S.bar);
        bulk_g2s(S.stage_v, a.vals_in + (size_t)part * SORT_PART, SORT_PART * 4u, &S.bar);
    };
    auto is_full = [&](uint32_t part) { return part < nparts && (n - part * SORT_PART) >= (uint32_t)SORT_PART; };

    if (tid == 0) {
        const uint32_t p0 = atomicAdd(a.ticket, 1u);
        S.part = p0;
        if (use_tma && is_full(p0)) issue(p0);
    }
    __syncthreads();
    uint32_t phase = 0;

    for (;;) {
        const uint32_t part = S.part;
        if (part >= nparts) break;
        const uint32_t base = part * SORT_PART;
        const uint32_t nvalid = (n - base < (uint32_t)SORT_PART) ? (n - base) : (uint32_t)SORT_PART;
        const bool full = nvalid == (uint32_t)SORT_PART;
        uint32_t next_ticket = 0;
        if (tid == 0) next_ticket = atomicAdd(a.ticket, 1u);          // consumed after the reorder: the round trip is hidden

        const uint32_t wbase = warp * (32u * SORT_ITEMS);
        if (use_tma && full) {
            mbar_wait(&S.bar, phase); phase ^= 1u;
        } else {                                                       // ragged tail (or unaligned caller buffers): plain loads
#pragma unroll
            for (int i = 0; i < SORT_ITEMS; i++) {
                const uint32_t li = wbase + i * 32u + lane;
                S.stage_k[li] = (li < nvalid) ? a.keys_in[base + li] : 0xffffffffu;   // pads rank last (radix_sort.wgsl:79)
                S.stage_v[li] = (li < nvalid) ? a.vals_in[base + li] : 0u;
            }
            __syncwarp();                                              // each warp reads back only what it wrote
        }
        // keys, warp-striped: warp w owns [w*512, +512), item i of lane l = i*32 + l
        uint32_t key[SORT_ITEMS];
#pragma unroll
        for (int i = 0; i < SORT_ITEMS; i++) key[i] = S.stage_k[wbase + i * 32u + lane];
        {   // clear the {mask, count} words: 16 KB = 4 x uint4 per thread
            uint4 *z = reinterpret_cast<uint4 *>(S.kv);
            const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int i = 0; i < (WARPS * 256 * 8) / (16 * SORT_THREADS); i++) z[i * SORT_THREADS + tid] = z4;
        }
        __syncthreads();

        // ---- rank inside the warp on packed words {x: peer mask of the current round, y: keys of this digit seen so far}
        uint32_t rank2[SORT_ITEMS / 2];
        {
            uint2 *wt = S.kv + warp * 256u;
            const uint32_t lanebit = 1u << lane, lower = lanebit - 1u;
#pragma unroll
            for (int i = 0; i < SORT_ITEMS; i++) {
                const uint32_t d = (key[i] >> shift) & 255u;
                atomicOr(&wt[d].x, lanebit);
                __syncwarp();
                const uint2 mc = wt[d];
                const uint32_t rk = mc.y + (uint32_t)__popc(mc.x & lower);
                __syncwarp();                                          // every peer has read the word
                if ((mc.x & lower) == 0u) wt[d] = make_uint2(0u, mc.y + (uint32_t)__popc(mc.x));   // lowest peer: advance, clear
                __syncwarp();
                if (i & 1) rank2[i >> 1] |= rk << 16; else rank2[i >> 1] = rk;
            }
        }
        __syncthreads();

        // ---- per bin (thread tid = bin): totals over the warps, publish the partition's aggregate
        uint32_t cw[WARPS];
        uint32_t total = 0;
#pragma unroll
        for (int w = 0; w < WARPS; w++) { cw[w] = S.kv[w * 256u + tid].y; total += cw[w]; }
        uint32_t *st = a.status + (size_t)part * 256u + tid;
        st_relaxed(st, (part == 0u ? LB_PREFIX : LB_AGGREGATE) | total);
        uint32_t binstart;
        {
            uint32_t incl = total;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
                if ((int)lane >= o) incl += t;
            }
            if (lane == 31) S.scan[warp] = incl;
            __syncthreads();                                           // also: every thread has read its rank words out of S.kv
            uint32_t woff = 0;
#pragma unroll
            for (int w = 0; w < WARPS; w++) if (w < (int)warp) woff += S.scan[w];
            binstart = woff + incl - total;
        }
        {
            uint32_t run = binstart;
#pragma unroll
            for (int w = 0; w < WARPS; w++) { S.tbl[w][tid] = run; run += cw[w]; }
        }
        __syncthreads();

        // ---- reorder in shared memory: one table read, one 64-bit {key, value} store per item
#pragma unroll
        for (int i = 0; i < SORT_ITEMS; i++) {
            const uint32_t d = (key[i] >> shift) & 255u;
            const uint32_t pos = S.tbl[warp][d] + ((rank2[i >> 1] >> ((i & 1) * 16)) & 0xffffu);
            S.kv[pos] = make_uint2(key[i], S.stage_v[wbase + i * 32u + lane]);
        }
        __syncthreads();                                               // the stage is free again
        if (tid == 0) {
            S.part = next_ticket;
            if (use_tma && is_full(next_ticket)) issue(next_ticket);   // in flight during the look-back and the write-out
        }

        // ---- two-level decoupled look-back
        LbState lb; lb.excl = 0; lb.done = (part == 0u);
        {
            const uint32_t grp = part / SORT_LB_GROUP;
            const bool leader = (part % SORT_LB_GROUP) == SORT_LB_GROUP - 1u;
            lookback_level(a.status + tid, (int)part - 1, (int)(grp * SORT_LB_GROUP), grp == 0u, lb, a.err);
            uint32_t *gst = a.gstatus + (size_t)grp * 256u + tid;
            if (leader) st_relaxed(gst, (lb.done ? LB_PREFIX : LB_AGGREGATE) | ((lb.excl + total) & LB_VALUE_MASK));
            if (!lb.done) {
                lookback_level(a.gstatus + tid, (int)grp - 1, 0, true, lb, a.err);
                if (leader) st_relaxed(gst, LB_PREFIX | ((lb.excl + total) & LB_VALUE_MASK));
            }
            if (part > 0u) st_relaxed(st, LB_PREFIX | ((lb.excl + total) & LB_VALUE_MASK));
        }
        S.gbase[tid] = g_excl + lb.excl - binstart;                    // wraps mod 2^32 by design
        __syncthreads();

        // ---- write out: consecutive threads write consecutive addresses within a bin run
#pragma unroll
        for (int k = 0; k < SORT_ITEMS; k++) {
            const uint32_t i = tid + k * SORT_THREADS;
            if (i < nvalid) {
                const uint2 p = S.kv[i];
                const uint32_t kk = p.x;
                const uint32_t g = S.gbase[(kk >> shift) & 255u] + i;
                if (a.keys_out) a.keys_out[g] = kk;
                a.vals_out[g] = p.y;
                if (EMIT_RANGES) {                                     // see V1: run boundaries via atomicMin
                    const bool first = (i == 0u) || (S.kv[i - 1u].x != kk);
                    const bool last = (i == nvalid - 1u) || (S.kv[i + 1u].x != kk);
                    if (first) atomicMin(&a.ranges[kk].x, g);
                    if (last) atomicMin(&a.ranges[kk].y, ~(g + 1u));
                }
            }
        }
        __syncthreads();                                               // S.kv is free; S.part (next partition) is visible
    }
}

// Standalone digit histograms (only for the public ws_sort_pairs_u32 entry point; the frame
// path gets its histograms from preprocess / binning).
__global__ void __launch_bounds__(256)
sort_histogram_kernel(const uint32_t *__restrict__ keys, const uint32_t *n_ptr, uint32_t n_cap,
                      uint32_t *hist, int passes)
{
    __shared__ uint32_t s_hist[4 * 256];
    const unsigned tid = threadIdx.x;
    for (unsigned i = tid; i < 4u * 256u; i += 256u) s_hist[i] = 0u;
    __syncthreads();
    uint32_t n = *n_ptr;
    if (n > n_cap) n = n_cap;
    for (uint32_t i = blockIdx.x * 256u + tid; i < n; i += gridDim.x * 256u) {
        const uint32_t k = keys[i];
        for (int d = 0; d < passes; d++) atomicAdd(&s_hist[d * 256 + ((k >> (8 * d)) & 255u)], 1u);   // shared atomics without return
    }
    __syncthreads();
    for (unsigned i = tid; i < (unsigned)passes * 256u; i += 256u) {
        const uint32_t c = s_hist[i];
        if (c) atomicAdd(hist + i, c);
    }
}

}  // namespace

static int rank_ways()
{
    static int ways = [] {
        const char *e = getenv("WS_RANK_WAYS");              // tuning knob for A/B runs; the default is what ships
        const int w = e ? atoi(e) : WS_RANK_WAYS;
        return (w == 1 || w == 2 || w == 4) ? w : WS_RANK_WAYS;
    }();
    return ways;
}

static int sort_variant()
{
    static int v = [] {
        const char *e = getenv("WS_SORT_VARIANT");           // 1 = register-staged pass (default), 2 = the TMA-staged pass (alternative, see above)
        const int w = e ? atoi(e) : 1;
        return (w == 2) ? 2 : 1;
    }();
    return v;
}

constexpr size_t SORT_V2_SMEM = sizeof(SortSmemV2) + 128;    // + slack for the 128-B alignment of the TMA destination

// the opt-in above 48 KB of dynamic shared memory is per device (several contexts may live in one process)
static cudaError_t sort_v2_prepare()
{
    static bool done[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64 && done[dev]) return cudaSuccess;
    e = cudaFuncSetAttribute(onesweep_pass_v2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SORT_V2_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(onesweep_pass_v2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SORT_V2_SMEM);
    if (e == cudaSuccess && dev >= 0 && dev < 64) done[dev] = true;
    return e;
}

cudaError_t launch_sort_pass(const SortPassArgs &a, int grid, cudaStream_t stream)
{
    if (sort_variant() == 2) {
        cudaError_t e = sort_v2_prepare();
        if (e != cudaSuccess) return e;
        if (a.ranges) onesweep_pass_v2_kernel<true><<<grid, SORT_THREADS, SORT_V2_SMEM, stream>>>(a);
        else onesweep_pass_v2_kernel<false><<<grid, SORT_THREADS, SORT_V2_SMEM, stream>>>(a);
        return cudaGetLastError();
    }
    const int w = rank_ways();
#define WS_LAUNCH(R, W) onesweep_pass_kernel<R, W><<<grid, SORT_THREADS, 0, stream>>>(a)
    if (a.ranges) { if (w == 4) WS_LAUNCH(true, 4); else if (w == 2) WS_LAUNCH(true, 2); else WS_LAUNCH(true, 1); }
    else          { if (w == 4) WS_LAUNCH(false, 4); else if (w == 2) WS_LAUNCH(false, 2); else WS_LAUNCH(false, 1); }
#undef WS_LAUNCH
    return cudaGetLastError();
}

bool sort_pass_can_skip_keys() { return true; }

int sort_pass_blocks_per_sm()
{
    int best = 1 << 30;
    auto probe = [&](auto kernel, size_t smem) {
        int nb = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, SORT_THREADS, smem);
        if (nb < best) best = nb;
    };
    if (sort_variant() == 2) {
        if (sort_v2_prepare() != cudaSuccess) return 1;
        probe(onesweep_pass_v2_kernel<false>, SORT_V2_SMEM); probe(onesweep_pass_v2_kernel<true>, SORT_V2_SMEM);
    } else {
        const int w = rank_ways();
        if (w == 4) { probe(onesweep_pass_kernel<false, 4>, 0); probe(onesweep_pass_kernel<true, 4>, 0); }
        else if (w == 2) { probe(onesweep_pass_kernel<false, 2>, 0); probe(onesweep_pass_kernel<true, 2>, 0); }
        else { probe(onesweep_pass_kernel<false, 1>, 0); probe(onesweep_pass_kernel<true, 1>, 0); }
    }
    return best > 0 && best < (1 << 30) ? best : 1;
}

cudaError_t launch_sort_histogram(const uint32_t *keys, const uint32_t *n_ptr, uint32_t n_cap,
                                  uint32_t *hist, int passes, int grid, cudaStream_t stream)
{
    sort_histogram_kernel<<<grid, 256, 0, stream>>>(keys, n_ptr, n_cap, hist, passes);
    return cudaGetLastError();
}

}  // namespace ws
