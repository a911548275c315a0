// dgr_binning.cuh — tile binning (A3 of SURVEY.md §8a) without a global sort.
//
// The reference op sorts ALL (tile, depth) keys with one device-wide 64-bit radix sort (6 passes over N_inst pairs)
// and reads the instance count back to the host.  Here:
//   1. the preprocess kernel histograms the instances of each block of Gaussians per tile in shared memory and adds the
//      block's counts to the per-tile totals: one global atomic per touched (block, tile), not per instance, and what the
//      atomic returns is where the block's run starts inside the tile (kept in a [blocks x tiles] run matrix);
//   2. emit_instances_kernel scans the per-tile totals itself for the range starts, adds its row of the run matrix and
//      appends (depth bits << 32 | Gaussian id) keys there with shared-memory cursors — the order inside a tile is
//      arbitrary at this point.  One extra block of the same launch publishes what everybody else needs: per-tile [start, end) ranges
//      (clipped to the buffer capacity), the instance count (device + pinned host memory, no host round trip), the
//      heaviest-first issue order and the big-tile list;
//   3. (there is no separate scan kernel);
//   4. tile_sort_gather_kernel sorts each tile's segment by (depth, id) in shared memory (keys are unique, so the result
//      is deterministic and identical to the reference's stable (tile, depth) order) and, in the same pass, gathers the
//      48-byte records into depth-sorted, per-tile contiguous order for the bulk-TMA staging of the render kernels.
#pragma once
#include "dgr_common.cuh"

namespace dgr {

// binning scratch: [keys u64 x cap][ids u32 x cap][rec_sorted 48 x cap]
struct BinningLayout {
    size_t off_keys, off_ids, off_rec, total;
    __host__ explicit BinningLayout(uint64_t cap) {
        size_t c = cap > 0 ? (size_t)cap : 1;
        size_t o = 0;
        off_keys = o; o = align_up(o + c * 8, 256);
        off_ids = o;  o = align_up(o + c * 4, 256);
        off_rec = o;  o = align_up(o + c * sizeof(Rec), 256);
        total = o;
    }
};

__device__ __forceinline__ void cmpex(unsigned long long *a, int i, int l) {
    const unsigned long long x = a[i], y = a[l];
    if (x > y) { a[i] = y; a[l] = x; }
}

// Ascending-only bitonic network for arbitrary n (comparators whose upper index is >= n are skipped: they would
// compare against a virtual +inf that never moves).  All index arithmetic is shift/mask.
__device__ __forceinline__ void bitonic_sort_cta(unsigned long long *a, int n) {
    int lg = 0;
    while ((1 << lg) < n) lg++;
    const int half = (1 << lg) >> 1;
    for (int lk = 1; lk <= lg; lk++) {
        const int k = 1 << lk, hk = k >> 1;
        for (int t = threadIdx.x; t < half; t += blockDim.x) {
            const int blk = t >> (lk - 1), off = t & (hk - 1);
            const int i = (blk << lk) + off, l = (blk << lk) + (k - 1 - off);
            if (l < n) cmpex(a, i, l);
        }
        __syncthreads();
        for (int j = k >> 2; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < half; t += blockDim.x) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), l = i + j;
                if (l < n) cmpex(a, i, l);
            }
            __syncthreads();
        }
    }
}

// Sort-kernel populations: tiles with n <= kSortSmallCap are sorted by the grid-wide kernel (one CTA per tile);
// larger ones are appended to a compact list that a small persistent grid walks.
constexpr int kSortSmallCap = 4096;
constexpr int kOrderBins = 128;          // log-scale population classes for the heaviest-first issue order

struct TileWork {                        // lives in image scratch (256 bytes, zeroed by the forward's memset)
    unsigned n_big;                      // number of entries of big_list (written by the metadata block)
    unsigned n_nonempty;                 // tiles with at least one instance = the leading entries of tile_order
    unsigned long long fwd_next;         // work counter of the persistent forward render kernel (zeroed by the metadata block)
    unsigned cost_bpt;                   // backward items per tile the forward grouped its measured costs for (0: none)
    unsigned lazy;                       // 1: the forward staged its records by id (no sorted record copy exists): the backward follows
    unsigned pad[2];
    unsigned cls_count[kCostClasses];    // backward work items per measured-cost class (filled by the forward render kernel)
};
static_assert(sizeof(TileWork) <= 256, "TileWork");

__device__ __forceinline__ int order_bin(unsigned count) {
    // descending population class: 0 = heaviest.  class = 4 * floor(log2(count)) + next two mantissa bits
    if (count == 0) return kOrderBins - 1;
    const int lg = 31 - __clz(count);
    const int frac = lg >= 2 ? (int)((count >> (lg - 2)) & 3u) : (int)((count << (2 - lg)) & 3u);
    const int cls = lg * 4 + frac;                      // 0 .. 127
    return max(0, kOrderBins - 2 - cls);
}

// Tile metadata for the kernels that follow (one CTA of NT threads): exclusive scan of the per-tile instance counts ->
// ranges (clipped to `cap`), total -> header (+ the caller's pinned host memory); the heaviest-first issue order of the
// persistent render kernels (counting sort on log-scale population classes) with the empty tiles at its tail; the list of
// tiles too big for the per-tile sort CTA.  Every thread owns kScanTPT consecutive tiles in registers per pass.
constexpr int kScanTPT = 8;

template <int NT>
__device__ __forceinline__ void
tile_meta_cta(int tiles, const unsigned *__restrict__ tile_count, unsigned long long cap, uint2 *__restrict__ ranges,
              GeomHeader *__restrict__ hdr, unsigned *__restrict__ tile_order, uint2 *__restrict__ order_ranges,
              TileWork *__restrict__ work, unsigned *__restrict__ big_list, volatile unsigned long long *counts_host,
              unsigned long long ticket) {
    constexpr int NW = NT / 32;
    __shared__ unsigned long long s_warp[32];
    __shared__ unsigned long long s_carry, s_total;
    __shared__ unsigned s_bin[kOrderBins], s_nbig, s_nne;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { s_carry = 0; s_nbig = 0; s_nne = 0; }
    for (int i = tid; i < kOrderBins; i += NT) s_bin[i] = 0;
    __syncthreads();
    const int span = NT * kScanTPT;
    for (int base = 0; base < tiles; base += span) {
        unsigned cnt[kScanTPT];
        unsigned long long sum = 0;
        const int t0 = base + tid * kScanTPT;
#pragma unroll
        for (int j = 0; j < kScanTPT; j++) { cnt[j] = (t0 + j < tiles) ? __ldcg(tile_count + t0 + j) : 0u; sum += cnt[j]; }
        unsigned long long inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long n = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += n; }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            const unsigned long long w = lane < NW ? s_warp[lane] : 0ull;
            unsigned long long winc = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned long long n = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += n; }
            s_warp[lane] = winc - w;
            if (lane == 31) s_total = winc;
        }
        __syncthreads();
        unsigned long long run = s_carry + s_warp[warp] + (inc - sum);
#pragma unroll
        for (int j = 0; j < kScanTPT; j++) {
            unsigned pop = 0u;
            int bin = -1;                                                     // -1: no tile here
            if (t0 + j < tiles) {
                const unsigned long long s = run < cap ? run : cap;
                const unsigned long long e = (run + cnt[j]) < cap ? (run + cnt[j]) : cap;
                ranges[t0 + j] = make_uint2((unsigned)s, (unsigned)e);
                pop = (unsigned)(e - s);                                      // clipped population
                bin = order_bin(pop);
                if (pop > (unsigned)kSortSmallCap) big_list[atomicAdd(&s_nbig, 1u)] = (unsigned)(t0 + j);
            }
            // Neighbouring tiles fall into the same population class (and most tiles of a centred object are empty): one
            // shared-memory atomic per (warp, class) — one per tile serialised ~1500 atomics on the "empty" class.
            const unsigned same = __match_any_sync(0xffffffffu, bin);
            if (bin >= 0 && lane == __ffs(same) - 1) atomicAdd(&s_bin[bin], (unsigned)__popc(same));
            const unsigned nz = __ballot_sync(0xffffffffu, pop > 0u);
            if (lane == 0 && nz) atomicAdd(&s_nne, (unsigned)__popc(nz));
            run += cnt[j];
        }
        __syncthreads();
        if (tid == 0) s_carry += s_total;
        __syncthreads();
    }
    if (tid == 0) {
        hdr->n_inst = s_carry; hdr->n_big = s_nbig; work->n_big = s_nbig; work->n_nonempty = s_nne; work->fwd_next = 0ull;
        // The host wants the instance count early (is the caller's capacity guess large enough?).  With a ticket the counts
        // go straight into the caller's pinned, device-mapped host memory: no copy or event between the kernels, the forward
        // chains with programmatic dependent launches while the host polls the ticket.
        if (counts_host && ticket) {
            counts_host[0] = s_carry; counts_host[1] = s_nbig;
            __threadfence_system();
            counts_host[2] = ticket;
        }
    }
    // counting sort of the tiles by population class (heaviest first)
    if (warp == 0) {
        unsigned run = 0;
        for (int b0 = 0; b0 < kOrderBins; b0 += 32) {
            const unsigned v = s_bin[b0 + lane];
            unsigned inc = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned n = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += n; }
            s_bin[b0 + lane] = run + inc - v;
            run += __shfl_sync(0xffffffffu, inc, 31);
        }
    }
    __syncthreads();
    // Plain descending order: the render kernels are persistent and pull work items from this list through an atomic
    // counter (longest processing time first); the empty tiles form its tail (class kOrderBins - 1).
    for (int t0 = 0; t0 < tiles; t0 += NT) {
        const int t = t0 + tid;
        int bin = -1;
        uint2 r = make_uint2(0u, 0u);
        if (t < tiles) { r = ranges[t]; bin = order_bin(r.y - r.x); }
        const unsigned same = __match_any_sync(0xffffffffu, bin);             // warp-aggregated slot reservation per class
        const int leader = __ffs(same) - 1;
        unsigned base = 0;
        if (bin >= 0 && lane == leader) base = atomicAdd(&s_bin[bin], (unsigned)__popc(same));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (bin >= 0) {
            const unsigned pos = base + __popc(same & ((1u << lane) - 1u));
            tile_order[pos] = (unsigned)t;
            order_ranges[pos] = r;                                            // what the sort kernel reads: no second indirection
        }
    }
}

// Instance emission, first half: this block's write cursor of every tile = start of the tile's range (exclusive scan of the
// per-tile totals) + where the preprocess kernel's reservation put this block inside the tile (its run-matrix row).
__device__ __forceinline__ void emit_block_cursors(int tiles, const unsigned *__restrict__ tile_count, unsigned long long cap,
                                                   const unsigned *__restrict__ run_matrix, unsigned *s_off, unsigned long long *s_part) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // range starts: exclusive scan of the per-tile totals.  Warp w owns the contiguous tile range [w R, (w + 1) R); its lanes
    // read 32 consecutive tiles at a time (coalesced, several loads in flight): pass 1 sums the range, pass 2 (after the
    // warp bases are known) scans it and adds the block's run-matrix row.
    constexpr int NW = kPreThreads / 32;
    const int R = ((tiles + NW - 1) / NW + 31) / 32 * 32;
    const int w_lo = min(tiles, warp * R), w_hi = min(tiles, w_lo + R);
    unsigned long long sum = 0;
#pragma unroll 4
    for (int t = w_lo + lane; t < w_hi; t += 32) sum += __ldcg(tile_count + t);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) s_part[warp] = sum;
    __syncthreads();
    unsigned long long run = 0;
    for (int w = 0; w < warp; w++) run += s_part[w];
    const unsigned *row = run_matrix + (size_t)blockIdx.x * tiles;
    // (the totals and run-matrix entries of kE 32-tile pieces are requested before the first of them is scanned: the scans form
    //  a dependent chain through `run`, and one L2 round trip per piece would otherwise sit in front of every link of it)
    constexpr int kE = 4;
    for (int t0 = w_lo; t0 < w_hi; t0 += 32 * kE) {
        unsigned cj[kE], rj[kE];
#pragma unroll
        for (int j = 0; j < kE; j++) {
            const int t = t0 + 32 * j + lane;
            cj[j] = t < w_hi ? __ldcg(tile_count + t) : 0u;
            rj[j] = t < w_hi ? __ldcg(row + t) : 0u;
        }
#pragma unroll
        for (int j = 0; j < kE; j++) {
            if (t0 + 32 * j < w_hi) {                                     // warp-uniform
                const int t = t0 + 32 * j + lane;
                const unsigned c = cj[j];
                unsigned inc = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const unsigned n = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += n; }
                const unsigned long long start = run + (inc - c);
                if (t < w_hi) s_off[t] = (unsigned)(start < cap ? start : cap) + rj[j];
                run += __shfl_sync(0xffffffffu, inc, 31);
            }
        }
    }
    __syncthreads();
}

// Instance emission, second half: one Gaussian's `cnt` instances (the tiles of its packed pixel AABB ax / ay, offset by tile0)
// at the block's tile cursors: ONE shared-memory atomic and one 8-byte store per instance.  Positions at or beyond the
// capacity are dropped.
__device__ __forceinline__ void emit_keys(unsigned long long key, unsigned ax, unsigned ay, int gx, int tile0, int cnt, unsigned *s_off,
                                          unsigned long long *__restrict__ keys, unsigned cap32) {
    const int tx0 = (int)(ax & 0xffffu) >> 4, tw = ((int)(ax >> 16) >> 4) - tx0 + 1;
    const int ty0 = (int)(ay & 0xffffu) >> 4;
    int x = 0, t = tile0 + ty0 * gx + tx0;
#pragma unroll 4
    for (int i = 0; i < cnt; i++) {
        const unsigned pos = atomicAdd(&s_off[t], 1u);
        if (pos < cap32) keys[pos] = key;                             // beyond the instance capacity: dropped
        x++; t++;
        if (x == tw) { x = 0; t += gx - tw; }
    }
}

// Instance emission, same block <-> Gaussian mapping as the preprocess kernel; grid = nblocks + 1.
//   blocks 0 .. nblocks-1:  the block scans the per-tile totals itself for the range starts (every thread owns a run of
//     consecutive tiles; the totals are 4 B x tiles, L2-resident), adds its row of the run matrix (where the preprocess
//     kernel's reservation put this block inside each tile) and appends the keys at that position + (shared-memory atomic
//     rank): ONE shared-memory atomic and one 8-byte store per instance.  Positions at or beyond the capacity are dropped.
//   block nblocks:  the tile metadata the later kernels and the host need (tile_meta_cta).  There is no separate scan kernel.
__global__ void __launch_bounds__(kPreThreads)
emit_instances_kernel(int P, int gx, int tiles, int gpb_iters, int nblocks, const Rec *__restrict__ rec, const unsigned *__restrict__ touched,
                      const unsigned *__restrict__ tile_count, unsigned long long cap, const unsigned *__restrict__ run_matrix,
                      unsigned long long *__restrict__ keys, uint2 *__restrict__ ranges, GeomHeader *__restrict__ hdr,
                      unsigned *__restrict__ tile_order, uint2 *__restrict__ order_ranges, TileWork *__restrict__ work,
                      unsigned *__restrict__ big_list, volatile unsigned long long *counts_host, unsigned long long ticket) {
    extern __shared__ unsigned s_off[];
    __shared__ unsigned long long s_part[kPreThreads / 32];
    pdl_trigger();
    pdl_wait();                          // records, touched counts, per-tile totals and run matrix of the preprocess kernel
    if ((int)blockIdx.x == nblocks) {
        tile_meta_cta<kPreThreads>(tiles, tile_count, cap, ranges, hdr, tile_order, order_ranges, work, big_list, counts_host, ticket);
        return;
    }
    emit_block_cursors(tiles, tile_count, cap, run_matrix, s_off, s_part);
    const unsigned cap32 = (unsigned)cap;
    for (int it = 0; it < gpb_iters; it++) {
        const int g = (int)((blockIdx.x * gpb_iters + it) * kPreThreads + threadIdx.x);
        if (g >= P) continue;
        const int cnt = (int)(__ldg(touched + g) & 0x1fffffffu);                  // = tw * th (same AABB as the histogram)
        if (cnt == 0) continue;
        const float4 q1 = __ldg(&rec[g].q1);
        const unsigned long long key = ((unsigned long long)__float_as_uint(q1.z) << 32) | (unsigned)g;
        emit_keys(key, __float_as_uint(q1.w), __float_as_uint(__ldg(&rec[g].q2.w)), gx, 0, cnt, s_off, keys, cap32);
    }
}

// Batched emission (dgr_views_*): the same block <-> Gaussian mapping as preprocess_views_fwd_kernel; each Gaussian appends the
// instances of all its views: key = depth bits << 32 | record r = v P + g, in the tiles tile_off[v] + local tile (ViewTable).  The
// metadata block covers all tiles of the batch.
__global__ void __launch_bounds__(kPreThreads)
emit_views_kernel(int P, int V, const __grid_constant__ ViewTable vt, int gpb_iters, int nblocks, const Rec *__restrict__ rec, const unsigned *__restrict__ touched,
                  const unsigned *__restrict__ tile_count, unsigned long long cap, const unsigned *__restrict__ run_matrix,
                  unsigned long long *__restrict__ keys, uint2 *__restrict__ ranges, GeomHeader *__restrict__ hdr,
                  unsigned *__restrict__ tile_order, uint2 *__restrict__ order_ranges, TileWork *__restrict__ work,
                  unsigned *__restrict__ big_list, volatile unsigned long long *counts_host, unsigned long long ticket) {
    extern __shared__ unsigned s_off[];
    __shared__ unsigned long long s_part[kPreThreads / 32];
    pdl_trigger();
    pdl_wait();
    const int tiles = vt.tile_off[V];
    if ((int)blockIdx.x == nblocks) {
        tile_meta_cta<kPreThreads>(tiles, tile_count, cap, ranges, hdr, tile_order, order_ranges, work, big_list, counts_host, ticket);
        return;
    }
    emit_block_cursors(tiles, tile_count, cap, run_matrix, s_off, s_part);
    const unsigned cap32 = (unsigned)cap;
    for (int it = 0; it < gpb_iters; it++) {
        const int g = (int)((blockIdx.x * gpb_iters + it) * kPreThreads + threadIdx.x);
        if (g >= P) continue;
        for (int v = 0; v < V; v++) {
            const unsigned r = (unsigned)v * (unsigned)P + (unsigned)g;
            const int cnt = (int)(__ldg(touched + r) & 0x1fffffffu);
            if (cnt == 0) continue;
            const float4 q1 = __ldg(&rec[r].q1);
            const unsigned long long key = ((unsigned long long)__float_as_uint(q1.z) << 32) | r;
            emit_keys(key, __float_as_uint(q1.w), __float_as_uint(__ldg(&rec[r].q2.w)), vt.gx[v], vt.tile_off[v], cnt, s_off, keys, cap32);
        }
    }
}

// ----------------------------------------------------------------------------------------------------------------
// Per-tile sort by (depth, Gaussian id) + record gather: bucket + rank.
//
// A comparison network costs O(n log^2 n) dependent shared-memory round trips and ~20 block barriers; a multi-pass
// radix sort needs ordered (stable) ranking.  Neither is necessary: the keys are unique, so an element's final
// position is simply (start of its bucket) + (number of smaller keys in its bucket).  Each tile
//   1. loads its 64-bit keys and finds its own [min, max] depth,
//   2. drops every key into one of NB equal-width depth buckets (monotone in depth) with shared-memory integer
//      atomics — the order inside a bucket is arbitrary,
//   3. ranks every key inside its bucket by brute-force counting with the FULL (depth, id) key,
//   4. writes the Gaussian id and gathers the 48-byte record straight to the sorted position.
// Four block barriers, no serial phases, ~60 instructions per key for any reasonable depth distribution; a degenerate
// one (many equal depths, e.g. a planar cloud seen head-on) only makes step 3 longer — it stays exact: the result is
// the (depth, id) order, i.e. the reference's stable (tile, depth) order.
// ----------------------------------------------------------------------------------------------------------------
template <int THREADS, int CAP, int NBK>
struct SortSmem {
    static constexpr size_t off_b = 0;                                       // u64 [CAP]  keys grouped by bucket
    static constexpr size_t off_start = off_b + (size_t)CAP * 8;             // u32 [NBK + 1] bucket starts
    static constexpr size_t off_cur = off_start + (NBK + 32) * 4;            // u32 [NBK]     scatter cursors
    static constexpr size_t off_misc = off_cur + NBK * 4;                    // u32 [64]
    static constexpr size_t bytes = off_misc + 64 * 4;
};

// The keys of a tile live in REGISTERS between the phases (CAP / THREADS per thread, one coalesced global read); shared
// memory holds only the bucket-grouped copy the ranking needs — half the footprint of a two-copy layout, so more tiles are
// in flight per SM.
template <int THREADS, int CAP, int NBK>
__device__ __forceinline__ void sort_gather_tile(const uint2 r, unsigned long long *__restrict__ keys, const Rec *__restrict__ rec,
                                                 unsigned *__restrict__ ids_sorted, Rec *__restrict__ rec_sorted, unsigned char *smem,
                                                 const bool gather) {
    using SM = SortSmem<THREADS, CAP, NBK>;
    constexpr int KPT = (CAP + THREADS - 1) / THREADS;
    const int n = (int)(r.y - r.x);
    const int tid = threadIdx.x, lane = tid & 31;
    unsigned long long *gk = keys + r.x;
    if (n > CAP) {                                     // beyond the shared-memory capacity: in-place network in global memory
        __syncthreads();
        bitonic_sort_cta(gk, n);
        for (int i = tid; i < n; i += THREADS) {
            const unsigned gid = (unsigned)(gk[i] & 0xffffffffull);
            ids_sorted[r.x + i] = gid;
            if (gather) {
                const Rec *src = rec + gid;
                Rec v; v.q0 = __ldg(&src->q0); v.q1 = __ldg(&src->q1); v.q2 = __ldg(&src->q2);
                rec_sorted[r.x + i] = v;
            }
        }
        __syncthreads();
        return;
    }
    unsigned long long *B = reinterpret_cast<unsigned long long *>(smem + SM::off_b);
    unsigned *start = reinterpret_cast<unsigned *>(smem + SM::off_start);
    unsigned *cur = reinterpret_cast<unsigned *>(smem + SM::off_cur);
    unsigned *misc = reinterpret_cast<unsigned *>(smem + SM::off_misc);     // [0] min bits, [1] max bits, [2..] warp sums
    // bucket count: a power of two near n/2 (about two keys per bucket for a uniform spread)
    int nb = 64;
    while (nb < NBK && nb * 2 <= n) nb <<= 1;
    if (tid == 0) { misc[0] = 0xffffffffu; misc[1] = 0u; }
    for (int i = tid; i < nb; i += THREADS) cur[i] = 0u;
    unsigned long long k[KPT];
    unsigned lo = 0xffffffffu, hi = 0u;
    const int kslots = (n + THREADS - 1) / THREADS;                           // slots in use (block-uniform): the loops below stop there
#pragma unroll
    for (int j = 0; j < KPT; j++) {
        k[j] = ~0ull;
        if (j < kslots) {
            const int i = tid + j * THREADS;
            if (i < n) { k[j] = __ldcs(gk + i); const unsigned d = (unsigned)(k[j] >> 32); lo = min(lo, d); hi = max(hi, d); }   // read once, streaming
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    __syncthreads();                                   // misc / cur initialised (and the previous tile of this CTA is done with smem)
    if (lane == 0) { atomicMin(&misc[0], lo); atomicMax(&misc[1], hi); }
    __syncthreads();
    const float dmin = __uint_as_float(misc[0]), dmax = __uint_as_float(misc[1]);
    const float scale = (dmax > dmin) ? (float)nb / (dmax - dmin) : 0.f;
    // histogram (cur[] = bucket populations)
#pragma unroll
    for (int j = 0; j < KPT; j++) {
        if (j < kslots) {
            const int i = tid + j * THREADS;
            const float d = __uint_as_float((unsigned)(k[j] >> 32));
            const int bkt = min(nb - 1, (int)((d - dmin) * scale));           // monotone in d
            if (i < n) atomicAdd(&cur[bkt], 1u);
        }
    }
    __syncthreads();
    // exclusive scan of the nb populations -> start[], cur[] = running cursors
    {
        constexpr int PER = (NBK + THREADS - 1) / THREADS;
        unsigned v[PER], sum = 0;
#pragma unroll
        for (int j = 0; j < PER; j++) { const int b = tid * PER + j; v[j] = (b < nb) ? cur[b] : 0u; sum += v[j]; }
        unsigned inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (lane == 31) misc[2 + (tid >> 5)] = inc;
        __syncthreads();
        if (tid < 32) {                                // exclusive scan of the (at most 32) warp totals
            const unsigned w = tid < THREADS / 32 ? misc[2 + tid] : 0u;
            unsigned wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += t; }
            misc[2 + tid] = wi - w;
        }
        __syncthreads();
        unsigned run = misc[2 + (tid >> 5)] + inc - sum;
#pragma unroll
        for (int j = 0; j < PER; j++) { const int b = tid * PER + j; if (b < nb) { start[b] = run; cur[b] = run; } run += v[j]; }
        if (tid == 0) start[nb] = (unsigned)n;
    }
    __syncthreads();
    // scatter into buckets (arbitrary order inside a bucket)
#pragma unroll
    for (int j = 0; j < KPT; j++) {
        if (j < kslots) {
            const int i = tid + j * THREADS;
            const float d = __uint_as_float((unsigned)(k[j] >> 32));
            const int bkt = min(nb - 1, (int)((d - dmin) * scale));
            if (i < n) B[atomicAdd(&cur[bkt], 1u)] = k[j];
        }
    }
    __syncthreads();
    // rank inside the bucket with the full key, write the id to the final position; then the warp moves the records of its
    // (up to) 32 keys together: 96 16-byte pieces, piece c = part c % 3 of key c / 3.  So one 128-bit load or store touches
    // about 11 records, not the 32 scattered ones of a lane per record, and the stores, whose positions are a near-permutation
    // of a contiguous range, coalesce.
    const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
    for (int i0 = tid - lane; i0 < n; i0 += THREADS) {                     // warp-uniform: the shuffles need every lane
        const int i = i0 + lane;
        unsigned gid = 0u;
        int pos = -1;                                                        // -1: no key for this lane
        if (i < n) {
            const unsigned long long kk = B[i];
            const float d = __uint_as_float((unsigned)(kk >> 32));
            const int bk = min(nb - 1, (int)((d - dmin) * scale));
            const int s = (int)start[bk], e = (int)start[bk + 1];
            int rank = 0;
            for (int j = s; j < e; j++) rank += (B[j] < kk) ? 1 : 0;
            gid = (unsigned)(kk & 0xffffffffull);
            pos = s + rank;
            ids_sorted[(size_t)r.x + pos] = gid;
        }
        if (gather) {
#pragma unroll
            for (int m = 0; m < 3; m++) {
                const int c = m * 32 + lane, k = c / 3, part = c - 3 * k;
                const unsigned g = __shfl_sync(0xffffffffu, gid, k);
                const int p = __shfl_sync(0xffffffffu, pos, k);
                if (p >= 0) {
                    const float4 v = ldg_f4_hint(reinterpret_cast<const float4 *>(rec + g) + part, pol_keep);
                    stg_f4_hint(reinterpret_cast<float4 *>(rec_sorted + r.x + p) + part, v, pol_stream);
                }
            }
        }
    }
}

constexpr int kSortSmallThreads = 512, kSortSmallBuckets = 1024;
constexpr int kSortBigThreads = 1024, kSortBigCap = 12288, kSortBigBuckets = 2048;     // 96 KB of keys + 16 KB of bucket tables

// Persistent grid over the NON-EMPTY tiles in issue order (heaviest first, dealt round-robin to the CTAs): CTA c sorts entries
// c, c + G, c + 2G ... of the ordered range list the emit kernel's metadata block wrote; the next entry's range is already
// in flight while a tile is being sorted.  Tiles beyond kSortSmallCap are left to the big-tile kernel.
template <int NBK>
__global__ void __launch_bounds__(kSortSmallThreads, 4)
tile_sort_gather_kernel(const TileWork *__restrict__ work, const uint2 *__restrict__ order_ranges, unsigned long long *__restrict__ keys,
                        const Rec *__restrict__ rec, unsigned *__restrict__ ids_sorted, Rec *__restrict__ rec_sorted, int gather) {
    extern __shared__ __align__(16) unsigned char s_sort[];
    pdl_trigger();
    pdl_wait();
    const unsigned n_tiles = __ldcg(&work->n_nonempty);
    // the look-ahead range travels through shared memory: held in registers across the sort it spills on sm_90 (32-register cap)
    __shared__ uint2 s_range[2];
    unsigned i = blockIdx.x;
    if (threadIdx.x == 0) s_range[0] = i < n_tiles ? __ldcg(order_ranges + i) : make_uint2(0u, 0u);
    __syncthreads();
    for (int b = 0; i < n_tiles; b ^= 1) {
        const unsigned inext = i + gridDim.x;
        if (threadIdx.x == 0) s_range[b ^ 1] = inext < n_tiles ? __ldcg(order_ranges + inext) : make_uint2(0u, 0u);
        const uint2 r = s_range[b];
        const int n = (int)(r.y - r.x);
        if (n > 0 && n <= kSortSmallCap)
            sort_gather_tile<kSortSmallThreads, kSortSmallCap, NBK>(r, keys, rec, ids_sorted, rec_sorted, s_sort, gather != 0);
        __syncthreads();                               // every thread has read s_range[b] before thread 0 refills it
        i = inext;
    }
}

// small persistent grid walking the list of big tiles
__global__ void __launch_bounds__(kSortBigThreads)
tile_sort_gather_big_kernel(const TileWork *__restrict__ work, const unsigned *__restrict__ big_list, const uint2 *__restrict__ ranges,
                            unsigned long long *__restrict__ keys, const Rec *__restrict__ rec, unsigned *__restrict__ ids_sorted,
                            Rec *__restrict__ rec_sorted, int gather) {
    extern __shared__ __align__(16) unsigned char s_sort[];
    pdl_trigger();
    pdl_wait();
    const unsigned nb = work->n_big;
    for (unsigned i = blockIdx.x; i < nb; i += gridDim.x)
        sort_gather_tile<kSortBigThreads, kSortBigCap, kSortBigBuckets>(ranges[big_list[i]], keys, rec, ids_sorted, rec_sorted, s_sort, gather != 0);
}

}  // namespace dgr
