// binning.cu -- tile binning between the depth sort and the tile sort (new design; the
// reference has no tiles: it draws every splat as one instanced quad, gaussian.wgsl:30-57).
//
// The logical sort key of the tile-binned renderer is 64-bit (tile | depth).  An LSD radix
// sort of that key is "sort by the depth digits, then stably by the tile digits"; the depth
// is a per-SPLAT property, so its four digit passes run on the V visible splats BEFORE they
// are expanded into P >= V (tile, splat) pairs.  This kernel does the expansion: it walks
// the splats in depth order, turns each tile rectangle into its (tile id, slot) pairs at
// offsets given by a scan of the per-partition pair counts, and counts the tile-id digits
// for the onesweep passes that follow.  The result after those passes is bit-identical
// to sorting P 64-bit (tile|depth) keys with (tile, depth, slot) order, at ~1/3 of the traffic.
//
// Three launches, none with an inter-CTA dependency (a single-pass chained scan was tried
// first: at ~900 pairs per partition every partition paid serialised ticket / gather /
// look-back round trips and the kernel ran far below the HBM roofline):
//   COUNT   pairs per 1024-splat partition (slot load + rectangle gather, 4 per thread in flight);
//   SCAN    one CTA: exclusive scan of the partition totals, P, overflow flag;
//   EXPAND  load-balanced over PAIRS, not splats: every splat with at least one tile drops a
//           marker (its index) at the block-local offset of its first pair, a prefix-max over
//           the positions (warp shuffles, 8 positions per thread) tells every output position
//           which splat owns it, and the thread derives (tile x, tile y) from the position with
//           one multiply-high (magic reciprocal of the rectangle width).  Threads emit
//           consecutive pairs straight to global memory, perfectly coalesced, however uneven
//           the rectangles are (a screen-filling splat simply owns many consecutive positions).
//           (A rewrite -- owner thread walks its rectangle, the block walks the large ones,
//           pairs staged in shared memory -- is kept as bin_expand_kernel / WS_BIN_EXPAND=2: it
//           executes a quarter of the instructions and is slower.)
// The digit histogram uses plain shared-memory atomicAdd (no return value): its rate does not
// depend on the address spread, and a MATCH.ANY-aggregated update is far slower
// (profiles/microbench/rank_primitives.cu).
#include "ws_device.cuh"
#include "ws_kernels.h"

#include <stdlib.h>

namespace ws {

namespace {

constexpr int BIN_THREADS = 256;
constexpr int BIN_WARPS = BIN_THREADS / 32;
constexpr int BIN_SPT = 4;                            // splats per thread
constexpr int BIN_PART = BIN_THREADS * BIN_SPT;       // 1024 splats per partition
constexpr int BIN_NDIG = 3;

struct SplatRects { uint32_t slot[BIN_SPT], xy[BIN_SPT], w[BIN_SPT], h[BIN_SPT], cnt[BIN_SPT]; };

// the range of depth-sorted positions this launch expands (ascending key = far -> near, so the near slab is the upper one);
// the split point is a multiple of 4 so that the 16-byte slot loads stay aligned
__device__ __forceinline__ void slab_bounds(const BinningArgs &a, uint32_t V, uint32_t &lo, uint32_t &hi)
{
    // the nearest near_pct % of the depth-sorted splats form the near slab (0 = the default, a quarter: a sweep over
    // 15-65 % at cfg3 and cfg4 peaked at 20-25 % on the previous target GPU; not re-swept on H100) -- a smaller near slab sorts fewer pairs that the far slab's cull would
    // have dropped; below ~20 % too few tiles are saturated when the far slab is binned.
    const uint32_t near = a.near_pct ? (uint32_t)(((uint64_t)V * a.near_pct) / 100u) : (V >> 2);
    const uint32_t split = (V - near) & ~3u;
    lo = (a.slab == 1u) ? split : 0u;
    hi = (a.slab == 2u) ? split : V;
}

// slots + rectangles of the BIN_SPT consecutive depth-sorted splats of one thread (positions first .. first+3, below V).
// keep4: one byte per splat, 0 = emits no pair (far slab, decided by the count kernel); 0x01010101 when there is no filter.
__device__ __forceinline__ void load_rects(const BinningArgs &a, uint32_t first, uint32_t V, SplatRects &r, uint32_t keep4 = 0x01010101u)
{
    if (first + BIN_SPT <= V) {
        const uint4 s4 = *reinterpret_cast<const uint4 *>(a.sorted_slots + first);
        r.slot[0] = s4.x; r.slot[1] = s4.y; r.slot[2] = s4.z; r.slot[3] = s4.w;
    } else {
#pragma unroll
        for (int j = 0; j < BIN_SPT; j++) r.slot[j] = (first + j < V) ? a.sorted_slots[first + j] : 0xffffffffu;
    }
    uint2 rc[BIN_SPT];
#pragma unroll
    for (int j = 0; j < BIN_SPT; j++)
        rc[j] = (r.slot[j] != 0xffffffffu && ((keep4 >> (8 * j)) & 0xffu)) ? __ldg(a.rects + r.slot[j]) : make_uint2(0u, 0u);
#pragma unroll
    for (int j = 0; j < BIN_SPT; j++) {
        r.xy[j] = rc[j].x;
        r.w[j] = rc[j].y & 0xffffu;
        r.h[j] = rc[j].y >> 16;
        r.cnt[j] = r.w[j] * r.h[j];
    }
}

// far slab: a splat all of whose tiles were saturated by the near slab cannot change a pixel.  Only small rectangles are
// tested (they are almost all of them); a pair emitted for a saturated tile is harmless, the compositor skips that tile.
// Returns the keep bytes for load_rects (the expand kernel does not repeat the test, nor fetch the dropped rectangles).
// `done` is the per-tile byte map (global memory, or its copy in shared memory); `bits`, when not NULL, is the same map as
// one BIT per tile in shared memory: a row of up to 16 tiles is then one funnel-shifted compare instead of a byte per tile.
__device__ __forceinline__ uint32_t drop_saturated(uint32_t tiles_x, SplatRects &r, const uint8_t *done, const uint32_t *bits)
{
    uint32_t keep4 = 0u;
#pragma unroll
    for (int j = 0; j < BIN_SPT; j++) {
        if (r.cnt[j] > 0u && r.cnt[j] <= 16u) {
            const uint32_t x0 = r.xy[j] & 0xffffu, y0 = r.xy[j] >> 16;
            bool all = true;
            if (bits) {
                const uint32_t mask = (1u << r.w[j]) - 1u;             // w <= 16
                uint32_t b0 = y0 * tiles_x + x0;
                for (uint32_t yy = 0; yy < r.h[j]; yy++, b0 += tiles_x) {
                    const uint32_t w0 = b0 >> 5;
                    const uint32_t row = __funnelshift_r(bits[w0], bits[w0 + 1u], b0 & 31u);   // bit i = tile b0 + i
                    all = all && ((row & mask) == mask);
                }
            } else {
                for (uint32_t yy = 0; yy < r.h[j]; yy++)
                    for (uint32_t xx = 0; xx < r.w[j]; xx++) all = all && (done[(y0 + yy) * tiles_x + x0 + xx] != 0);
            }
            if (all) r.cnt[j] = 0u;
        }
        if (r.cnt[j] > 0u) keep4 |= 1u << (8 * j);
    }
    return keep4;
}

// The saturation test reads the "saturated" flag of every tile of every small rectangle: random byte gathers from
// global memory would stall on long scoreboard for most of the far half of the frame.  The whole map is
// 8160 tiles at 1080p, 32 400 at 4K: each CTA packs it into ONE BIT per tile in shared memory (1-4 KB), and a rectangle
// row becomes two shared-memory words and a funnel shift.  Called by the whole CTA; ends with a barrier.
__device__ __forceinline__ void pack_done_bits(const uint8_t *tile_done, uint32_t T, uint32_t *s_bits)
{
    const uint32_t nwords = (T + 31u) / 32u;
    for (uint32_t w = threadIdx.x; w <= nwords; w += blockDim.x) {     // one word past the end stays 0: the funnel shift reads w0 + 1
        uint32_t v = 0u;
        if (w < nwords) {
            const uint4 *src = reinterpret_cast<const uint4 *>(tile_done + (size_t)w * 32u);   // 32 flag bytes (allocation padded)
            const uint4 q0 = src[0], q1 = src[1];
            const uint32_t b[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
            for (int k = 0; k < 8; k++) {                              // byte i of the 32 -> bit i (flags are 0 / 1)
                v |= ((b[k] & 0x1u) | ((b[k] >> 7) & 0x2u) | ((b[k] >> 14) & 0x4u) | ((b[k] >> 21) & 0x8u)) << (4 * k);
            }
            const uint32_t valid = T - w * 32u;                         // tiles beyond T (padding bytes) never count as done... nor matter
            if (valid < 32u) v &= (1u << valid) - 1u;
        }
        s_bits[w] = v;
    }
    __syncthreads();
}

// bytes of dynamic shared memory for the bit map (0: too many tiles, the test reads the byte map from global memory).
// One bit per tile + one spare word; up to 16384 x 16384 pixels = 1 Mi tiles = 128 KB would not fit the default 48 KB:
// above 256 Ki tiles the kernels read the byte map from global memory.
static size_t done_bits_bytes(uint32_t num_tiles)
{
    return (num_tiles && num_tiles <= 262144u) ? (((size_t)num_tiles + 31u) / 32u + 1u) * 4u : 0u;
}

// ---- (1) COUNT ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(BIN_THREADS)
bin_count_kernel(BinningArgs a)
{
    __shared__ uint32_t s_red[BIN_WARPS];
    extern __shared__ __align__(16) uint8_t s_done[];   // far slab: the per-tile "saturated" map, one bit per tile (when it fits)
    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const uint32_t V = *a.list_len;
    uint32_t lo, hi;
    slab_bounds(a, V, lo, hi);
    const uint32_t nparts = (hi - lo + BIN_PART - 1u) / BIN_PART;
    const uint8_t *done = a.tile_done;
    const uint32_t *bits = nullptr;
    if (a.tile_done && a.done_in_smem) {
        pack_done_bits(a.tile_done, a.uniforms->tiles_x * a.uniforms->tiles_y, reinterpret_cast<uint32_t *>(s_done));
        bits = reinterpret_cast<const uint32_t *>(s_done);
    }
    for (uint32_t part = blockIdx.x; part < nparts; part += gridDim.x) {
        SplatRects r;
        load_rects(a, lo + part * BIN_PART + tid * BIN_SPT, hi, r);
        if (a.tile_done) a.keep4[part * BIN_THREADS + tid] = drop_saturated(a.uniforms->tiles_x, r, done, bits);
        uint32_t c = r.cnt[0] + r.cnt[1] + r.cnt[2] + r.cnt[3];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) s_red[warp] = c;
        __syncthreads();
        if (tid == 0) {
            uint32_t t = 0;
#pragma unroll
            for (int k = 0; k < BIN_WARPS; k++) t += s_red[k];
            a.part_counts[part] = t;
        }
        __syncthreads();
    }
}

// ---- (2) SCAN: exclusive scan of up to 2^20 partition totals by one CTA --------------------------
__global__ void __launch_bounds__(1024)
bin_scan_kernel(BinningArgs a)
{
    const uint32_t V = *a.list_len;
    uint32_t lo, hi;
    slab_bounds(a, V, lo, hi);
    const uint32_t nparts = (hi - lo + BIN_PART - 1u) / BIN_PART;
    const uint64_t total_out = block_exclusive_scan_1024<uint64_t>(a.part_counts, a.part_bases, nparts);
    if (threadIdx.x == 0) {
        const uint64_t P = (nparts > 0u) ? total_out : 0ull;           // 64-bit: screen-filling splats can push P past 2^32
        *a.num_pairs_out = P > 0xffffffffull ? 0xffffffffu : (uint32_t)P;
        *a.num_pairs64_out = P;
        if (P > (uint64_t)a.pair_cap) a.counters->pair_overflow = 1u;  // zeroed per frame; either slab may set it
    }
}

// ---- (3'') EXPAND, rewrite (WS_BIN_EXPAND=2; NOT the default: slower, see launch_binning) --------------------------------
// Profiling the default kernel (~140 lane-instructions per emitted pair, the marker / prefix-max machinery executed
// for every output position) showed the general
// load-balancing scheme costing 3x what the data needs: a splat touches 3.5 tiles on average, so the owner thread
// simply walks its own rectangle.  Only rectangles above EXP_SMALL tiles (close-ups, gaussian_scaling > 1) are expanded
// cooperatively by the whole block, one 256-wide stride per rectangle.  Pairs are staged in shared memory at their
// block-local output position (scan of the per-splat counts), so the stores to global memory stay perfectly
// coalesced and the output order -- splat (depth order), then row-major tile -- is exactly that of the default kernel.
constexpr int EXP_CAP = 4096;                         // staged pairs per chunk (2 x 16 KB)
constexpr uint32_t EXP_SMALL = 32;                    // rectangles up to this many tiles are walked by their owner thread
constexpr int EXP_BIG = 512;                          // cooperative list entries per partition (beyond: owner thread walks)

__global__ void __launch_bounds__(BIN_THREADS, 4)
bin_expand_kernel(BinningArgs a)
{
    __shared__ uint32_t s_tile[EXP_CAP];
    __shared__ uint32_t s_slot[EXP_CAP];
    __shared__ uint4 s_big[EXP_BIG];                  // {first pair (block-local), x0 | y0<<16, slot, w | h<<16}
    __shared__ uint32_t s_hist[BIN_NDIG][256];
    __shared__ uint32_t s_scan[BIN_WARPS];
    __shared__ uint32_t s_nbig;

    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const uint32_t V = *a.list_len;
    uint32_t lo, hi;
    slab_bounds(a, V, lo, hi);
    const uint32_t nparts = (hi - lo + BIN_PART - 1u) / BIN_PART;
    const uint32_t tiles_x = a.uniforms->tiles_x;
    const uint32_t cap = a.pair_cap;
    const uint32_t ntiles = tiles_x * a.uniforms->tiles_y;
    const int ndig = (ntiles > 65536u) ? 3 : ((ntiles > 256u) ? 2 : 1);

    for (unsigned i = tid; i < (unsigned)(BIN_NDIG * 256); i += BIN_THREADS) (&s_hist[0][0])[i] = 0u;
    if (tid == 0) s_nbig = 0u;
    __syncthreads();

    for (uint32_t part = blockIdx.x; part < nparts; part += gridDim.x) {
        SplatRects r;
        load_rects(a, lo + part * BIN_PART + tid * BIN_SPT, hi, r, a.tile_done ? a.keep4[part * BIN_THREADS + tid] : 0x01010101u);
        const uint32_t base = __ldg(a.part_bases + part);
        if (base >= cap) continue;                        // beyond the pair capacity (overflow is already flagged): nothing of this partition is stored
        const uint32_t mine = r.cnt[0] + r.cnt[1] + r.cnt[2] + r.cnt[3];
        // block scan of the per-thread totals -> block-local position of every splat's first pair
        uint32_t incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((int)lane >= o) incl += t;
        }
        if (lane == 31) s_scan[warp] = incl;
        __syncthreads();
        uint32_t woff = 0, total = 0;
#pragma unroll
        for (int k = 0; k < BIN_WARPS; k++) {
            const uint32_t c = s_scan[k];
            if (k < (int)warp) woff += c;
            total += c;
        }
        uint32_t excl[BIN_SPT];
        excl[0] = incl + woff - mine;
#pragma unroll
        for (int j = 1; j < BIN_SPT; j++) excl[j] = excl[j - 1] + r.cnt[j - 1];
        // large rectangles go to the cooperative list (any order: every pair's position is fixed by excl)
        bool own[BIN_SPT];
#pragma unroll
        for (int j = 0; j < BIN_SPT; j++) {
            own[j] = r.cnt[j] > 0u;
            if (r.cnt[j] > EXP_SMALL) {
                const uint32_t e = atomicAdd(&s_nbig, 1u);
                if (e < (uint32_t)EXP_BIG) { s_big[e] = make_uint4(excl[j], r.xy[j], r.slot[j], r.w[j] | (r.h[j] << 16)); own[j] = false; }
            }
        }
        __syncthreads();
        const uint32_t nbig = s_nbig < (uint32_t)EXP_BIG ? s_nbig : (uint32_t)EXP_BIG;

        for (uint32_t c0 = 0; c0 < total; c0 += EXP_CAP) {
            const uint32_t m = (total - c0 < (uint32_t)EXP_CAP) ? total - c0 : (uint32_t)EXP_CAP;
            // 1. owner threads walk their (small) rectangles, row-major
#pragma unroll
            for (int j = 0; j < BIN_SPT; j++) {
                if (own[j] && excl[j] < c0 + m && excl[j] + r.cnt[j] > c0) {
                    const uint32_t x0 = r.xy[j] & 0xffffu, y0 = r.xy[j] >> 16;
                    uint32_t o = excl[j] - c0;                               // may wrap below 0 for a rectangle continuing from the previous chunk: tested per pair
                    uint32_t row = y0 * tiles_x + x0;
                    for (uint32_t yy = 0; yy < r.h[j]; yy++, row += tiles_x)
                        for (uint32_t xx = 0; xx < r.w[j]; xx++, o++)
                            if (o < m) { s_tile[o] = row + xx; s_slot[o] = r.slot[j]; }
                }
            }
            // 2. the block walks the large rectangles together
            for (uint32_t b = 0; b < nbig; b++) {
                const uint4 inf = s_big[b];
                const uint32_t w = inf.w & 0xffffu, cnt = w * (inf.w >> 16);
                if (inf.x >= c0 + m || inf.x + cnt <= c0) continue;          // block-uniform
                const uint32_t q0 = (inf.x < c0) ? c0 - inf.x : 0u;          // first pair of the rectangle inside this chunk
                const uint32_t q1 = (inf.x + cnt > c0 + m) ? c0 + m - inf.x : cnt;
                const uint32_t origin = (inf.y >> 16) * tiles_x + (inf.y & 0xffffu);
                for (uint32_t q = q0 + tid; q < q1; q += BIN_THREADS) {
                    const uint32_t ty = q / w, tx = q - ty * w;
                    const uint32_t o = inf.x + q - c0;
                    s_tile[o] = origin + ty * tiles_x + tx; s_slot[o] = inf.z;
                }
            }
            __syncthreads();
            // 3. coalesced copy-out + tile-id digit histograms
            for (uint32_t i = tid; i < m; i += BIN_THREADS) {
                const uint64_t g = (uint64_t)base + c0 + i;
                if (g < cap) {
                    const uint32_t tile = s_tile[i];
                    a.pair_tiles[g] = tile;
                    a.pair_slots[g] = s_slot[i];
                    for (int d = 0; d < ndig; d++) atomicAdd(&s_hist[d][(tile >> (8 * d)) & 255u], 1u);
                }
            }
            __syncthreads();
        }
        if (tid == 0) s_nbig = 0u;
        __syncthreads();
    }

    for (unsigned i = tid; i < (unsigned)(ndig * 256); i += BIN_THREADS) {
        const uint32_t c = s_hist[i >> 8][i & 255u];
        if (c) atomicAdd(a.hist + i, c);
    }
}

constexpr int BIN_ROUNDS = 8;                         // (v1) output positions per thread and chunk
constexpr int BIN_CAP = BIN_THREADS * BIN_ROUNDS;     // (v1) 2048 pairs per chunk
// ---- (3) EXPAND (default): load-balanced over PAIRS with markers + prefix-max -----------------------------------------
// (5 resident CTAs per SM: the binning grid is sized by this kernel's occupancy; at 4 the register allocation may grow
// past 48 and the persistent grid of both binning kernels shrinks by a fifth)
__global__ void __launch_bounds__(BIN_THREADS, 5)
bin_expand_v1_kernel(BinningArgs a)
{
    __shared__ uint32_t s_owner[BIN_CAP];             // marker = owner index + 1 at the owner's first position
    __shared__ uint4 s_info[BIN_PART];                // per splat: {first pair (block-local), x0 | y0<<16, slot, width}
    __shared__ uint32_t s_magic[BIN_PART];            // ceil(2^32 / width)
    __shared__ uint32_t s_hist[BIN_NDIG][256];
    __shared__ uint32_t s_scan[BIN_WARPS];
    __shared__ uint32_t s_wcarry[BIN_WARPS];

    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const uint32_t V = *a.list_len;
    uint32_t lo, hi;
    slab_bounds(a, V, lo, hi);
    const uint32_t nparts = (hi - lo + BIN_PART - 1u) / BIN_PART;
    const uint32_t tiles_x = a.uniforms->tiles_x;
    const uint32_t cap = a.pair_cap;
    const uint32_t ntiles = tiles_x * a.uniforms->tiles_y;
    const int ndig = (ntiles > 65536u) ? 3 : ((ntiles > 256u) ? 2 : 1);

    for (unsigned i = tid; i < (unsigned)(BIN_NDIG * 256); i += BIN_THREADS) (&s_hist[0][0])[i] = 0u;
    __syncthreads();

    for (uint32_t part = blockIdx.x; part < nparts; part += gridDim.x) {
        SplatRects r;
        load_rects(a, lo + part * BIN_PART + tid * BIN_SPT, hi, r, a.tile_done ? a.keep4[part * BIN_THREADS + tid] : 0x01010101u);
        const uint32_t base = __ldg(a.part_bases + part);
        if (base >= cap) continue;                        // beyond the pair capacity (overflow is already flagged): nothing of this partition is stored
        const uint32_t mine = r.cnt[0] + r.cnt[1] + r.cnt[2] + r.cnt[3];
        // block scan of the per-thread totals
        uint32_t incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((int)lane >= o) incl += t;
        }
        if (lane == 31) s_scan[warp] = incl;
        __syncthreads();
        uint32_t woff = 0, total = 0;
#pragma unroll
        for (int k = 0; k < BIN_WARPS; k++) {
            const uint32_t c = s_scan[k];
            if (k < (int)warp) woff += c;
            total += c;
        }
        uint32_t excl[BIN_SPT];
        excl[0] = incl + woff - mine;
#pragma unroll
        for (int j = 1; j < BIN_SPT; j++) excl[j] = excl[j - 1] + r.cnt[j - 1];
#pragma unroll
        for (int j = 0; j < BIN_SPT; j++) {
            s_info[tid * BIN_SPT + j] = make_uint4(excl[j], r.xy[j], r.slot[j], r.w[j]);
            s_magic[tid * BIN_SPT + j] = (r.w[j] > 1u) ? __float2uint_ru(__fdiv_ru(4294967296.f, (float)r.w[j])) : 0u;
            // m >= 2^32/w with m*w - 2^32 <= w + 512: floor(t/w) == umulhi(t, m) for every t < 2^20, w <= 1024 (viewport <= 16384)
        }

        // (a chunk that starts at or past the capacity stores nothing: stop there -- an overflowing partition of
        // screen-filling splats would otherwise walk up to 2^30 positions for nothing)
        for (uint32_t c0 = 0; c0 < total && (uint64_t)base + c0 < cap; c0 += BIN_CAP) {
            const uint32_t m = (total - c0 < (uint32_t)BIN_CAP) ? total - c0 : (uint32_t)BIN_CAP;
            const uint32_t rounds = (m + BIN_THREADS - 1u) / BIN_THREADS;       // 32-position rounds per warp
            const uint32_t span = rounds * 32u;                                 // consecutive positions owned by a warp
            // 1. clear, 2. markers
            for (uint32_t q = tid; q < m; q += BIN_THREADS) s_owner[q] = 0u;
            __syncthreads();
#pragma unroll
            for (int j = 0; j < BIN_SPT; j++) {
                if (r.cnt[j] > 0u) {
                    if (excl[j] >= c0 && excl[j] < c0 + m) s_owner[excl[j] - c0] = tid * BIN_SPT + j + 1u;
                    else if (excl[j] < c0 && excl[j] + r.cnt[j] > c0) s_owner[0] = tid * BIN_SPT + j + 1u;   // continues from the previous chunk
                }
            }
            __syncthreads();
            // 3. prefix-max of the markers over this warp's span
            uint32_t own[BIN_ROUNDS];
            uint32_t carry = 0;
#pragma unroll
            for (int k = 0; k < BIN_ROUNDS; k++) {
                own[k] = 0u;
                if ((uint32_t)k < rounds) {
                    const uint32_t q = warp * span + (uint32_t)k * 32u + lane;
                    uint32_t v = (q < m) ? s_owner[q] : 0u;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
                        if ((int)lane >= o) v = v > t ? v : t;
                    }
                    v = v > carry ? v : carry;
                    carry = __shfl_sync(0xffffffffu, v, 31);
                    own[k] = v;
                }
            }
            if (lane == 0) s_wcarry[warp] = carry;
            __syncthreads();
            uint32_t prev = 0;
#pragma unroll
            for (int k = 0; k < BIN_WARPS; k++) if (k < (int)warp) { const uint32_t c = s_wcarry[k]; prev = prev > c ? prev : c; }
            // 4. emit: position -> (tile, slot), coalesced, plus the tile-id digit histogram
#pragma unroll
            for (int k = 0; k < BIN_ROUNDS; k++) {
                if ((uint32_t)k < rounds) {
                    const uint32_t q = warp * span + (uint32_t)k * 32u + lane;
                    const uint64_t g = (uint64_t)base + c0 + q;
                    if (q < m && g < cap) {
                        const uint32_t o = (own[k] > prev ? own[k] : prev) - 1u;
                        const uint4 inf = s_info[o];
                        const uint32_t t = c0 + q - inf.x;
                        const uint32_t ty = (inf.w > 1u) ? __umulhi(t, s_magic[o]) : t;
                        const uint32_t tx = t - ty * inf.w;
                        const uint32_t tile = ((inf.y >> 16) + ty) * tiles_x + (inf.y & 0xffffu) + tx;
                        a.pair_tiles[g] = tile;
                        a.pair_slots[g] = inf.z;
                        for (int d = 0; d < ndig; d++) atomicAdd(&s_hist[d][(tile >> (8 * d)) & 255u], 1u);
                    }
                }
            }
            __syncthreads();
        }
        __syncthreads();
    }

    for (unsigned i = tid; i < (unsigned)(ndig * 256); i += BIN_THREADS) {
        const uint32_t c = s_hist[i >> 8][i & 255u];
        if (c) atomicAdd(a.hist + i, c);
    }
}

// ---- occlusion split on one GPU ------------------------------------------------------------------------------------
// The near slab does not need a global depth order to be chosen: a key VALUE does as well as a position (the image is
// the same wherever the cut is, DESIGN.md section 4), and the far slab's cull is a per-splat test against the saturated
// tiles.  So: pick the cut from a histogram of the keys, compact the near list (key >= cut) and depth-sort only it;
// after its composite, cull the far splats in slot order and depth-sort only the survivors.  Equal keys fall on the
// same side of the cut, and both lists are compacted in slot order, so the stable sort of each list is the order the
// full sort gives them.
static_assert(SPLIT_CUT_BINS == BIN_THREADS * 8, "the cut is picked by one CTA, eight bins per thread");

// the BIN_SPT consecutive keys first .. first+3 (0 beyond V)
__device__ __forceinline__ void load_keys4(const uint32_t *keys, uint32_t first, uint32_t V, uint32_t k[BIN_SPT])
{
    if (first + BIN_SPT <= V) {
        const uint4 q = *reinterpret_cast<const uint4 *>(keys + first);
        k[0] = q.x; k[1] = q.y; k[2] = q.z; k[3] = q.w;
    } else {
#pragma unroll
        for (int j = 0; j < BIN_SPT; j++) k[j] = (first + j < V) ? keys[first + j] : 0u;
    }
}

// inclusive scan of one value per thread over the CTA (BIN_THREADS threads); s_w: BIN_WARPS words
__device__ __forceinline__ uint32_t block_inclusive_scan(uint32_t v, uint32_t *s_w)
{
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
        if ((int)lane >= o) v += t;
    }
    if (lane == 31) s_w[warp] = v;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BIN_WARPS; k++) if (k < (int)warp) v += s_w[k];
    return v;
}

// Histogram of (key - kmin) >> s over the V keys, s the smallest shift that leaves at most SPLIT_CUT_BINS bins; the last
// CTA to finish walks it from the nearest bin down and sets the cut at the boundary of the bin where the count reaches
// the near slab's share (at least one splat when V > 0).  A cut at a bin boundary never separates equal keys.
__global__ void __launch_bounds__(BIN_THREADS)
split_cut_kernel(SplitArgs a)
{
    __shared__ uint32_t s_hist[SPLIT_CUT_BINS];
    __shared__ uint32_t s_w[BIN_WARPS];
    __shared__ bool s_last;
    const unsigned tid = threadIdx.x;
    const uint32_t V = a.counters->num_visible;
    const uint32_t kmin = ~a.counters->key_min_inv, span = a.counters->key_max - kmin;
    uint32_t s = 0;
    while ((span >> s) >= (uint32_t)SPLIT_CUT_BINS) s++;
    for (unsigned i = tid; i < (unsigned)SPLIT_CUT_BINS; i += BIN_THREADS) s_hist[i] = 0u;
    __syncthreads();
    // a small grid (every CTA flushes up to 2048 bins into global memory at the end) with CUT_UNROLL 16-B loads per
    // thread in flight, so that the sweep still keeps enough bytes in flight to stream the keys at DRAM rate
    constexpr uint32_t CUT_UNROLL = 4, STEP = BIN_THREADS * BIN_SPT;
    for (uint32_t first0 = blockIdx.x * STEP * CUT_UNROLL + tid * BIN_SPT; first0 < V; first0 += gridDim.x * STEP * CUT_UNROLL) {
        uint32_t k[CUT_UNROLL][BIN_SPT];
#pragma unroll
        for (uint32_t u = 0; u < CUT_UNROLL; u++) load_keys4(a.keys, first0 + u * STEP, V, k[u]);
#pragma unroll
        for (uint32_t u = 0; u < CUT_UNROLL; u++)
#pragma unroll
            for (int j = 0; j < BIN_SPT; j++) if (first0 + u * STEP + j < V) atomicAdd(&s_hist[(k[u][j] - kmin) >> s], 1u);
    }
    __syncthreads();
    for (unsigned i = tid; i < (unsigned)SPLIT_CUT_BINS; i += BIN_THREADS) {
        const uint32_t c = s_hist[i];
        if (c) atomicAdd(a.cut_hist + i, c);
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(&a.counters->cut_done, 1u) == gridDim.x - 1u;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    uint32_t target = a.near_pct ? (uint32_t)(((uint64_t)V * a.near_pct) / 100u) : (V >> 2);
    if (target == 0u) target = V ? 1u : 0u;
    const int top = SPLIT_CUT_BINS - 1 - 8 * (int)tid;                 // thread 0 owns the nearest 8 bins
    uint32_t c8[8], sum = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) { c8[k] = __ldcg(a.cut_hist + top - k); sum += c8[k]; }
    const uint32_t incl = block_inclusive_scan(sum, s_w);
    const uint32_t excl = incl - sum;
    if (target > 0u && excl < target && target <= incl) {               // exactly one thread: the counts sum to V >= target
        uint32_t acc = excl;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            acc += c8[k];
            if (acc >= target) { a.counters->split_cut = kmin + ((uint32_t)(top - k) << s); break; }
        }
    }
}

// COUNT: which splats of every 1024-splat partition (slot order) enter the list.  Near: key >= cut.  Far: key < cut, a
// non-empty rectangle, and not all of its tiles saturated (drop_saturated, the rule of the position-split far slab).
// The decisions leave as one ballot word per (warp, splat of the thread): 32 words per partition.
__global__ void __launch_bounds__(BIN_THREADS)
split_count_kernel(SplitArgs a)
{
    __shared__ uint32_t s_red[BIN_WARPS];
    extern __shared__ __align__(16) uint8_t s_done[];   // far: the per-tile "saturated" map, one bit per tile (when it fits)
    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const uint32_t V = a.counters->num_visible;
    const uint32_t nparts = (V + BIN_PART - 1u) / BIN_PART;
    const uint32_t cut = a.counters->split_cut;
    const uint32_t tiles_x = a.uniforms->tiles_x;
    const uint32_t *bits = nullptr;
    if (a.far && a.done_in_smem) {
        pack_done_bits(a.tile_done, tiles_x * a.uniforms->tiles_y, reinterpret_cast<uint32_t *>(s_done));
        bits = reinterpret_cast<const uint32_t *>(s_done);
    }
    for (uint32_t part = blockIdx.x; part < nparts; part += gridDim.x) {
        const uint32_t first = part * BIN_PART + tid * BIN_SPT;
        uint32_t k[BIN_SPT];
        load_keys4(a.keys, first, V, k);
        uint32_t keep = 0u;                                             // bit j: splat first + j enters the list
        if (!a.far) {
#pragma unroll
            for (int j = 0; j < BIN_SPT; j++) if (first + j < V && k[j] >= cut) keep |= 1u << j;
        } else {
            bool cand[BIN_SPT], any = false;
#pragma unroll
            for (int j = 0; j < BIN_SPT; j++) { cand[j] = first + j < V && k[j] < cut; any = any || cand[j]; }
            uint2 rc[BIN_SPT];
#pragma unroll
            for (int j = 0; j < BIN_SPT; j++) rc[j] = make_uint2(0u, 0u);
            if (any) {
                if (first + BIN_SPT <= V) {
                    const uint4 *p = reinterpret_cast<const uint4 *>(a.rects + first);   // 32-B aligned: first % 4 == 0
                    const uint4 q0 = p[0], q1 = p[1];
                    rc[0] = make_uint2(q0.x, q0.y); rc[1] = make_uint2(q0.z, q0.w); rc[2] = make_uint2(q1.x, q1.y); rc[3] = make_uint2(q1.z, q1.w);
                } else {
#pragma unroll
                    for (int j = 0; j < BIN_SPT; j++) if (cand[j]) rc[j] = a.rects[first + j];
                }
            }
            SplatRects r;
#pragma unroll
            for (int j = 0; j < BIN_SPT; j++) {
                r.slot[j] = first + j;
                r.xy[j] = rc[j].x;
                r.w[j] = rc[j].y & 0xffffu;
                r.h[j] = rc[j].y >> 16;
                r.cnt[j] = cand[j] ? r.w[j] * r.h[j] : 0u;
            }
            const uint32_t keep4 = drop_saturated(tiles_x, r, a.tile_done, bits);
#pragma unroll
            for (int j = 0; j < BIN_SPT; j++) keep |= ((keep4 >> (8 * j)) & 1u) << j;
        }
        uint32_t b[BIN_SPT], c = 0;
#pragma unroll
        for (int j = 0; j < BIN_SPT; j++) { b[j] = __ballot_sync(0xffffffffu, (keep >> j) & 1u); c += (uint32_t)__popc(b[j]); }
        if (lane == 0) {
            *reinterpret_cast<uint4 *>(a.keep_bits + (size_t)part * (BIN_WARPS * BIN_SPT) + warp * BIN_SPT) = make_uint4(b[0], b[1], b[2], b[3]);
            s_red[warp] = c;
        }
        __syncthreads();
        if (tid == 0) {
            uint32_t t = 0;
#pragma unroll
            for (int w = 0; w < BIN_WARPS; w++) t += s_red[w];
            a.part_counts[part] = t;
        }
        __syncthreads();
    }
}

// SCAN (one CTA): partition bases and the list length
__global__ void __launch_bounds__(1024)
split_scan_kernel(SplitArgs a)
{
    const uint32_t V = a.counters->num_visible;
    const uint32_t nparts = (V + BIN_PART - 1u) / BIN_PART;
    const uint32_t total = block_exclusive_scan_1024<uint32_t>(a.part_counts, a.part_bases, nparts);   // <= V
    if (threadIdx.x == 0) *a.count_out = nparts ? total : 0u;
}

// SCATTER: the kept (key, slot) pairs at their slot-order position in the list + the list's four depth-digit histograms.
// A splat's rank inside its warp counts the kept splats of the lower lanes (all four of each) and its own earlier ones.
__global__ void __launch_bounds__(BIN_THREADS)
split_scatter_kernel(SplitArgs a)
{
    __shared__ uint32_t s_hist[4][256];
    __shared__ uint32_t s_wcnt[BIN_WARPS];
    const unsigned tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    for (unsigned i = tid; i < 4u * 256u; i += BIN_THREADS) (&s_hist[0][0])[i] = 0u;
    __syncthreads();
    const uint32_t V = a.counters->num_visible;
    const uint32_t nparts = (V + BIN_PART - 1u) / BIN_PART;
    const uint32_t lt = lanemask_lt();
    for (uint32_t part = blockIdx.x; part < nparts; part += gridDim.x) {
        const uint4 wb = *reinterpret_cast<const uint4 *>(a.keep_bits + (size_t)part * (BIN_WARPS * BIN_SPT) + warp * BIN_SPT);
        const uint32_t b[BIN_SPT] = {wb.x, wb.y, wb.z, wb.w};
        uint32_t before = 0, total = 0, mine = 0;
#pragma unroll
        for (int j = 0; j < BIN_SPT; j++) {
            before += (uint32_t)__popc(b[j] & lt);
            total += (uint32_t)__popc(b[j]);
            mine |= ((b[j] >> lane) & 1u) << j;
        }
        if (lane == 0) s_wcnt[warp] = total;
        __syncthreads();
        uint32_t pos = __ldg(a.part_bases + part) + before;
#pragma unroll
        for (int w = 0; w < BIN_WARPS; w++) if (w < (int)warp) pos += s_wcnt[w];
        if (mine) {
            const uint32_t first = part * BIN_PART + tid * BIN_SPT;
            uint32_t k[BIN_SPT];
            load_keys4(a.keys, first, V, k);
#pragma unroll
            for (int j = 0; j < BIN_SPT; j++) {
                if ((mine >> j) & 1u) {
                    a.keys_out[pos] = k[j];
                    a.vals_out[pos] = first + j;                        // stage 1 compacts in slot order: position == slot
#pragma unroll
                    for (int d = 0; d < 4; d++) atomicAdd(&s_hist[d][(k[j] >> (8 * d)) & 255u], 1u);
                    pos++;
                }
            }
        }
        __syncthreads();                                                // s_wcnt is rewritten by the next partition
    }
    for (unsigned i = tid; i < 4u * 256u; i += BIN_THREADS) {
        const uint32_t c = (&s_hist[0][0])[i];
        if (c) atomicAdd(a.hist + i, c);
    }
}

}  // namespace

cudaError_t launch_split_cut(const SplitArgs &a, int grid, cudaStream_t stream)
{
    split_cut_kernel<<<grid, BIN_THREADS, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_split_compact(const SplitArgs &a, int grid_count, int grid_scatter, cudaStream_t stream)
{
    SplitArgs ac = a;
    const size_t done_bytes = a.far ? done_bits_bytes(a.num_tiles_hint) : 0u;
    ac.done_in_smem = done_bytes ? 1u : 0u;
    split_count_kernel<<<grid_count, BIN_THREADS, done_bytes, stream>>>(ac);
    split_scan_kernel<<<1, 1024, 0, stream>>>(ac);
    split_scatter_kernel<<<grid_scatter, BIN_THREADS, 0, stream>>>(ac);
    return cudaGetLastError();
}

cudaError_t launch_binning(const BinningArgs &a, int grid_count, int grid_expand, cudaStream_t stream)
{
    // far slab: the tile_done map travels in dynamic shared memory when it fits under the 48 KB default limit
    BinningArgs ac = a;
    const size_t done_bytes = a.tile_done ? done_bits_bytes(a.num_tiles_hint) : 0u;
    ac.done_in_smem = done_bytes ? 1u : 0u;
    bin_count_kernel<<<grid_count, BIN_THREADS, done_bytes, stream>>>(ac);
    bin_scan_kernel<<<1, 1024, 0, stream>>>(a);
    // default: the markers + prefix-max kernel.  The rewrite executes a quarter of the instructions but is slower at cfg3
    // and cfg4: its owner-thread loops serialise on the longest rectangle of each warp and its scattered staging stores conflict.
    static const int variant = [] { const char *e = getenv("WS_BIN_EXPAND"); return (e && atoi(e) == 2) ? 2 : 1; }();
    if (variant == 1) bin_expand_v1_kernel<<<grid_expand, BIN_THREADS, 0, stream>>>(a);
    else bin_expand_kernel<<<grid_expand, BIN_THREADS, 0, stream>>>(a);
    return cudaGetLastError();
}

int binning_blocks_per_sm()
{
    int nb = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, bin_expand_v1_kernel, BIN_THREADS, 0);
    return nb > 0 ? nb : 1;
}

}  // namespace ws
