// dgr_render.cuh — per-tile front-to-back compositing (A4) and its reverse-traversal backward (A5).
//
// Design (not the reference's one-thread-per-pixel CTA with a cooperative fetch and a block barrier per batch):
//   * the unit of work is ONE WARP x ONE SUB-TILE (32*PPL pixels of a 16x16 tile).  A persistent grid (as many CTAs as
//     fit on the SMs) of independent warps pulls (tile, sub-tile) items, heaviest tile first, from an atomic counter in
//     global memory: no CTA-level coupling, no block barrier, no idle warps waiting for a slower sibling, and the SMs stay
//     evenly loaded although tile populations differ by orders of magnitude;
//   * a tile's depth-sorted 48-byte records are one contiguous block.  Each warp streams it through its OWN shared-memory
//     ring with 1-D bulk TMA (cp.async.bulk -> UBLKCP, completion on an mbarrier carrying the transaction bytes):
//     chunks of 32 records, kRing chunks in flight, re-armed by lane 0 as soon as the warp has left a chunk;
//   * for every chunk each LANE tests ONE record (opacity-aware pixel AABB + exact alpha >= 1/255 ellipse test against the
//     sub-tile), the ballot gives the records that can touch the sub-tile at all, and only those are evaluated (broadcast
//     reads from shared memory).  This skips most of the (pixel, Gaussian) pairs the reference evaluates and discards;
//   * backward: the only sequential quantities of the reverse traversal are two scalars per (pixel, Gaussian):
//     u = o G dL/dalpha and w = alpha T.  Step 1 (lane = pixel) walks the list backwards and parks (u, w) of the hitting
//     records in a shared-memory matrix; step 2 (lane = record x pixel-quarter) turns 8 parked records at a time into
//     their 10 moments with plain FMAs — no 13-shuffle butterfly per (warp, record) — and issues one red.global.add per
//     moment.  The reference issues ~10 atomics per (pixel, Gaussian) pair.
// Results follow the reference's rules exactly: power > 0 skip, alpha = min(0.99, o G), alpha < 1/255 skip,
// stop at T (1 - alpha) < 1e-4, colour + T*bg, un-normalised depth, alpha = sum alpha T.
#pragma once
#include "dgr_common.cuh"

namespace dgr {

constexpr int kChunk = 32;        // records per bulk copy: one per lane for the cull test (1.5 KB)
constexpr int kRing = 3;          // chunks in flight per warp
constexpr int kRenderWarps = 4;   // independent warps per CTA
constexpr int kRenderThreads = kRenderWarps * 32;

// power * log2(e) for pixel offset (dx, dy); identical instruction sequence in forward and backward so both make
// the same skip decisions.   q0.z = -0.5 A log2e, q0.w = -B log2e, q1.x = -0.5 C log2e
__device__ __forceinline__ float eval_power2(const float4 &q0, const float4 &q1, float dx, float dy) {
    const float t = __fmaf_rn(q0.z, dx, __fmul_rn(q0.w, dy));
    return __fmaf_rn(dx, t, __fmul_rn(__fmul_rn(q1.x, dy), dy));
}

// Lane-level cull of one staged record against a warp's sub-tile [wx0,wx1] x [wy0,wy1]: the opacity-aware pixel AABB
// (which carries the reference's 3-sigma tile-rect clip) AND the exact "can the alpha >= 1/255 ellipse reach it" test.
__device__ __forceinline__ bool record_hits_subtile(const Rec &r, int wx0, int wx1, int wy0, int wy1) {
    const float4 q1 = r.q1;
    const unsigned ax = __float_as_uint(q1.w), ay = __float_as_uint(r.q2.w);
    const int gx0 = (int)(ax & 0xffffu), gx1 = (int)(ax >> 16), gy0 = (int)(ay & 0xffffu), gy1 = (int)(ay >> 16);
    const int x0 = max(gx0, wx0), x1 = min(gx1, wx1), y0 = max(gy0, wy0), y1 = min(gy1, wy1);
    if (x0 > x1 || y0 > y1) return false;
    const float4 q0 = r.q0;
    return ellipse_hits_rect(q0.x, q0.y, q0.z, q0.w, q1.x, alpha_threshold_power2(q1.y), (float)x0, (float)x1, (float)y0, (float)y1);
}

// Sub-tile geometry of one warp for PPL pixels per lane: 8x4 (PPL 1), 8x8 (PPL 2), 16x8 (PPL 4) pixels.
template <int PPL>
struct SubTile {
    static constexpr int kPerTile = 8 / PPL;               // sub-tiles (= work items) per 16x16 tile
    static constexpr int kW = (PPL == 4) ? 16 : 8;         // region width
    static constexpr int kH = (PPL == 1) ? 4 : 8;          // region height
    __device__ static __forceinline__ int x0(int tx, int sub) { return tx * kTile + ((PPL == 4) ? 0 : (sub & 1) * 8); }
    __device__ static __forceinline__ int y0(int ty, int sub) { return ty * kTile + ((PPL == 4) ? sub * 8 : (sub >> 1) * kH); }
    __device__ static __forceinline__ int px(int wx0, int lane, int p) { return wx0 + (lane & 7) + ((PPL == 4 && (p & 1)) ? 8 : 0); }
    __device__ static __forceinline__ int py(int wy0, int lane, int p) { return wy0 + (lane >> 3) + ((PPL == 4) ? (p >> 1) * 4 : p * 4); }
};

// One warp's private bulk-TMA ring.  The mbarrier phase of every stage is tracked in a register bit mask: the ring lives
// across work items, and every chunk that was issued is also waited for (see drain()), so issue and wait counts agree.
struct __align__(128) WarpRing {
    Rec rec[kRing][kChunk];
    uint64_t full[kRing];
    uint64_t pad_[16 - kRing];
};
static_assert(sizeof(WarpRing) % 128 == 0, "WarpRing");

struct RingState {
    unsigned phase;        // bit s = parity the next wait on stage s expects
    int issued, waited;    // chunks of the current work item
};

__device__ __forceinline__ void ring_init(WarpRing &rg, RingState &rs, int lane) {
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < kRing; i++) mbar_init(&rg.full[i], 1);
        mbar_fence_init();
    }
    rs.phase = 0; rs.issued = 0; rs.waited = 0;
    __syncwarp();
}
// lane 0 only: start the copy of `cnt` records from `src` into the stage of sequence number `seq`
__device__ __forceinline__ void ring_issue(WarpRing &rg, int seq, const Rec *src, int cnt) {
    const int st = seq % kRing;
    const uint32_t bytes = (uint32_t)cnt * (uint32_t)sizeof(Rec);
    mbar_expect_tx(&rg.full[st], bytes);
    tma_bulk_g2s(&rg.rec[st][0], src, bytes, &rg.full[st]);
}
// warp-wide: start the copy of list chunk `chunk` (records [chunk*32, chunk*32 + cnt) of the tile's depth-sorted list) into the
// stage of sequence number `seq`.  lazy = false: the records were gathered into sorted order by the sort kernel — one
// contiguous bulk copy (lane 0).  lazy = true: only the sorted Gaussian ids exist; every lane copies ITS record (48 bytes,
// one cp.async.bulk each, all completing on the stage's mbarrier) straight from the per-Gaussian record array — the sort
// kernel then moves 12 instead of 108 bytes per instance and records beyond the end of the walked lists are never touched.
// (tools/tma_gather_probe.cu: 78 ns against 21 ns per 32-record chunk per SM, so the gather pays off where most of every
// list is never walked or where the sort kernel is the long pole: a compile-time variant, chosen per call by the host.)
template <bool LAZY>
__device__ __forceinline__ void ring_fill(WarpRing &rg, int seq, const Rec *src_sorted, const Rec *rec, unsigned my_id, int chunk, int cnt,
                                          int lane) {
    if (!LAZY) {
        if (lane == 0) ring_issue(rg, seq, src_sorted + (size_t)chunk * kChunk, cnt);
    } else {
        const int st = seq % kRing;
        if (lane == 0) mbar_expect_tx(&rg.full[st], (uint32_t)cnt * (uint32_t)sizeof(Rec));
        __syncwarp();
        if (lane < cnt) tma_bulk_g2s(&rg.rec[st][lane], rec + my_id, (uint32_t)sizeof(Rec), &rg.full[st]);
    }
}

// all lanes: wait for the chunk of sequence number `seq`, returns its stage
__device__ __forceinline__ int ring_wait(WarpRing &rg, RingState &rs, int seq) {
    const int st = seq % kRing;
    mbar_wait(&rg.full[st], (rs.phase >> st) & 1u);
    rs.phase ^= 1u << st;
    return st;
}

// Work queue of the persistent render kernels: the (tile, sub-tile) items in issue order (heaviest tile first), ONE 64-bit
// counter holding how many items have been handed out from the heavy end (low word) and from the light end (high word).
// Half of the warps of every SM sub-partition take from the heavy end, the other half from the light end, until the two
// meet: the heavy items are then in flight a few at a time per sub-partition and get re-dealt as warps free up, instead of
// all starting at once and fixing every sub-partition's load for the whole kernel.  (two_ended = 0: everybody takes from
// the heavy end.)  An atomicAdd returns both words as they were, so every item is handed out exactly once.
// `zero` receives bit 63 of the counter — always 0 (it would take 2^31 light-end takes), but only known once the atomic has
// returned: adding it to an address makes that access wait for THIS request instead of being scheduled in front of it.
__device__ __forceinline__ unsigned queue_take(unsigned long long *ctr, bool light, unsigned n, unsigned &zero) {
    const unsigned long long old = atomicAdd(ctr, light ? (1ull << 32) : 1ull);
    const unsigned h = (unsigned)old, l = (unsigned)(old >> 32);
    zero = l >> 31;
    if ((unsigned long long)h + l >= n) return 0xffffffffu;
    return light ? n - 1u - l : h;
}
__device__ __forceinline__ unsigned queue_take(unsigned long long *ctr, bool light, unsigned n) {
    unsigned z;
    return queue_take(ctr, light, n, z);
}

// Measured-cost ordering of the backward.  How long a sub-tile's list really is (early termination!) is only known after
// the forward has walked it, and the tile population the forward orders its own work by is a poor predictor of it.  So the
// forward records what every backward work item cost it (records tested + records that hit; two forward items feed one
// backward item when the backward uses larger sub-tiles) and appends the item to the list of its log-scale cost class; the
// backward hands the items out class by class, heaviest first — a longest-processing-time-first order by MEASURED cost,
// which deals the heavy items evenly over the SMs and leaves only light ones for the tail.
__device__ __forceinline__ int cost_class(unsigned c) {             // 0 = lightest ... kCostClasses-1 = heaviest
    const int lg = 31 - __clz(c | 1u);
    const int half = lg >= 1 ? (int)((c >> (lg - 1)) & 1u) : 0;
    return min(kCostClasses - 1, 2 * lg + half);
}

struct CostOrder {                       // image scratch pieces (all may be NULL: no measured-cost ordering)
    unsigned *cost_acc;                  // [tiles * 8]  sum of (cost << 2 | 1) of the forward items of a backward item
    unsigned *cls_count;                 // [kCostClasses]
    unsigned *cls_items;                 // [kCostClasses][tiles * 8]  ordered-tile index * 8 + backward sub-tile
    unsigned *cost_bpt;                  // TileWork::cost_bpt
    int tiles;
    int bwd_ppl;                         // sub-tile shape the backward will use (1 or 2)
};

// ----------------------------------------------------------------------------------------------------------------
// Forward.
// ----------------------------------------------------------------------------------------------------------------
// U = hits evaluated together: the alpha of a (pixel, record) pair does not depend on the compositing state, so the long
// part of the dependent chain (shared-memory read -> quadratic form -> ex2) of U hitting records is in flight at once and
// only the short T / colour update runs in sequence.  Same per-pixel operation order for every U: bit-identical images.
// One-pixel-per-lane variants are held to 64 registers (8 CTAs per SM): measured 4-5 us per step at 100k / 800^2 against the
// 72 registers ptxas picks on its own (A/B in profiles/r2_ab_variants.log).
//
// VIEWS: a batch of V views (dgr_views_forward_render, dgr_views_mixed_forward_render), each with its own image size (ViewTable
// vt; H, W, gx unused).  A work item's global tile gives its view (view_of_tile: once per item) and local tile; every view has its
// own background (bg [V,3]) and its own blocks of the flat images at pix_off[v]; the records are those of the batch.
//
// CONTRIB (DGR_RASTER_CONTRIB, render_*_fwd_contrib_kernel only): for every record the warp composites, the weights w = alpha T of
// its composited pixels are reduced over the warp right after the record (a shuffle butterfly for the sum, redux.sync on the float
// bits for the max: both a fixed order, so the item's partial is a pure function of the inputs), parked in the lane of the
// record's chunk slot, and after the chunk that lane adds the partial to the record's 64-bit fixed-point sum (integer atomics:
// the total does not depend on the order the items arrive in) and raises its max (atomicMax on the bits of a non-negative float).
struct ContribOut {
    unsigned long long *sum_fx;          // [records] sum of w, fixed point (kContribScale)
    unsigned *max_bits;                  // [records] bits of max w (float, >= 0)
};
constexpr float kContribScale = 274877906944.f;                  // 2^38
constexpr float kContribUnscale = 1.f / 274877906944.f;

template <int PPL, int U, bool LAZY, bool VIEWS, bool CONTRIB = false>
__device__ __forceinline__ void
render_fwd_body(int H, int W, int gx, const unsigned *__restrict__ tile_order, const uint2 *__restrict__ order_ranges,
                  const unsigned *__restrict__ n_tiles_nonempty, unsigned n_items, unsigned long long *__restrict__ work_next,
                  int two_ended, int sms, CostOrder co, unsigned *__restrict__ lazy_note,
                  const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ ids_sorted,
                  const float *__restrict__ bg, float *__restrict__ out_color,
                  float *__restrict__ out_depth, float *__restrict__ out_alpha, unsigned *__restrict__ n_contrib,
                  float *__restrict__ final_T, const ViewTable *vt, ContribOut cw = ContribOut{nullptr, nullptr}) {
    using ST = SubTile<PPL>;
    __shared__ WarpRing rings[kRenderWarps];
    const int lane = threadIdx.x & 31;
    WarpRing &rg = rings[threadIdx.x >> 5];
    RingState rs;
    pdl_trigger();
    ring_init(rg, rs, lane);
    const float b0 = VIEWS ? 0.f : __ldg(bg), b1 = VIEWS ? 0.f : __ldg(bg + 1), b2 = VIEWS ? 0.f : __ldg(bg + 2);    // VIEWS: per item
    const size_t HW = (size_t)H * W;
    pdl_wait();                          // sorted records, ranges, order, work counter

    // Work items = (tile, sub-tile) in issue order (heaviest tile first).  The non-empty tiles come first and are handed out
    // through the atomic counter.  The empty tiles at the tail of the order only need the background written: they are dealt
    // statically, no atomics.
    const unsigned n_queue = __ldcg(n_tiles_nonempty) * (unsigned)ST::kPerTile;
    const unsigned warp_global = blockIdx.x * kRenderWarps + (threadIdx.x >> 5), warps_total = gridDim.x * kRenderWarps;
    const bool costing = co.cost_acc != nullptr && PPL <= co.bwd_ppl;                 // forward sub-tiles nest in the backward's
    if (costing && blockIdx.x == 0 && threadIdx.x == 0) *co.cost_bpt = (unsigned)(8 / co.bwd_ppl);
    constexpr bool lazy = LAZY;
    if (blockIdx.x == 0 && threadIdx.x == 0) *lazy_note = LAZY ? 1u : 0u;             // (for the record; the host hands its choice to the backward)
    const bool light = two_ended && (((blockIdx.x / (unsigned)sms) + (threadIdx.x >> 5)) & 1u);
    bool queue_phase = true;
    unsigned item = 0, empty_next = n_queue + warp_global;
    // cost filing of the previous item (lane 0): the list position comes from an atomic whose round trip is as long as the queue's,
    // so it is only looked at here, after the NEXT item has been requested (the two round trips overlap instead of adding up)
    bool pend = false;
    unsigned pend_pos = 0, pend_base = 0, pend_val = 0;
    for (;;) {
        // (the item is taken when the warp is ready for it, not earlier: reserving the next item ahead of time would
        //  hand out the whole queue at the start and leave nothing to balance with — measured 58 -> 72 us)
        unsigned fetched = 0, zero = 0;
        if (queue_phase && lane == 0) fetched = queue_take(work_next, light, n_queue, zero);
        if (pend) { co.cls_items[(size_t)pend_base + pend_pos + zero] = pend_val; pend = false; }
        if (queue_phase) {
            item = __shfl_sync(0xffffffffu, fetched, 0);
            if (item >= n_queue) queue_phase = false;
        }
        if (!queue_phase) {
            item = empty_next; empty_next += warps_total;
            if (item >= n_items) break;
        }
        const unsigned ot = item / ST::kPerTile;
        const int tile = (int)__ldcg(tile_order + ot), sub = (int)(item % ST::kPerTile);
        const uint2 range = __ldcg(order_ranges + ot);
        int v = 0, lt = tile, iW = W, iH = H, igx = gx;          // VIEWS: the item's view and its size
        if constexpr (VIEWS) { v = view_of_tile(*vt, tile); lt = tile - vt->tile_off[v]; iW = vt->W[v]; iH = vt->H[v]; igx = vt->gx[v]; }
        const int tx = lt % igx, ty = lt / igx;
        const int n = (int)(range.y - range.x);
        const int nchunks = (n + kChunk - 1) / kChunk;
        const Rec *src = rec_sorted + range.x;
        const int wx0 = ST::x0(tx, sub), wy0 = ST::y0(ty, sub);
        const int wx1 = wx0 + ST::kW - 1, wy1 = wy0 + ST::kH - 1;

        const unsigned *ids = ids_sorted + range.x;
        rs.issued = 0; rs.waited = 0;
        unsigned nid = 0;                                       // lazy: this lane's Gaussian id in the next chunk to be issued
        {
            unsigned id0[kRing];
#pragma unroll
            for (int k = 0; k < kRing; k++) id0[k] = (lazy && k * kChunk + lane < n) ? __ldg(ids + k * kChunk + lane) : 0u;
            if (lazy && kRing * kChunk + lane < n) nid = __ldg(ids + kRing * kChunk + lane);
#pragma unroll
            for (int k = 0; k < kRing; k++)
                if (k < nchunks) ring_fill<LAZY>(rg, k, src, rec, id0[k], k, min(kChunk, n - k * kChunk), lane);
        }
        rs.issued = min(kRing, nchunks);

        float fx[PPL], fy[PPL], T[PPL], C0[PPL], C1[PPL], C2[PPL], D[PPL];
        unsigned last[PPL];
        bool done[PPL], inside[PPL];
        bool all_done = true;
#pragma unroll
        for (int p = 0; p < PPL; p++) {
            const int x = ST::px(wx0, lane, p), y = ST::py(wy0, lane, p);
            inside[p] = (x < iW) && (y < iH);
            fx[p] = (float)x; fy[p] = (float)y;
            T[p] = 1.f; C0[p] = 0.f; C1[p] = 0.f; C2[p] = 0.f; D[p] = 0.f; last[p] = 0; done[p] = !inside[p];
            all_done = all_done && done[p];
        }
        bool warp_done = __all_sync(0xffffffffu, all_done);
        unsigned cost = 0;
        for (int c = 0; c < nchunks && !warp_done; c++) {
            const int s = ring_wait(rg, rs, c);
            rs.waited = c + 1;
            const int cnt = min(kChunk, n - c * kChunk);
            bool hit = false;
            if (lane < cnt) hit = record_hits_subtile(rg.rec[s][lane], wx0, wx1, wy0, wy1);
            unsigned mask = __ballot_sync(0xffffffffu, hit);
            cost += 2u + 4u * (unsigned)__popc(mask);
            unsigned cid = 0, cmax = 0;                          // CONTRIB: this lane's record of the chunk, its partial
            float csum = 0.f;
            if constexpr (CONTRIB) { if (hit) cid = __ldg(ids + c * kChunk + lane); }
            while (mask) {
                int js[U];
                int nh = 0;
#pragma unroll
                for (int u = 0; u < U; u++) {
                    js[u] = 0;
                    if (mask) { js[u] = __ffs(mask) - 1; mask &= mask - 1; nh = u + 1; }
                }
                float av[U][PPL], dep[U], cr[U], cg[U], cb[U];
                bool pre[U][PPL];
#pragma unroll
                for (int u = 0; u < U; u++) {
                    if (u < nh) {
                        const Rec *r = &rg.rec[s][js[u]];
                        const float4 q0 = r->q0, q1 = r->q1, q2 = r->q2;
                        dep[u] = q1.z; cr[u] = q2.x; cg[u] = q2.y; cb[u] = q2.z;
#pragma unroll
                        for (int p = 0; p < PPL; p++) {
                            const float dx = q0.x - fx[p], dy = q0.y - fy[p];
                            const float p2 = eval_power2(q0, q1, dx, dy);
                            const float ag = __fmul_rn(q1.y, ex2_approx(p2));
                            av[u][p] = fminf(DGR_ALPHA_MAX, ag);
                            pre[u][p] = (p2 <= 0.f) & (av[u][p] >= DGR_ALPHA_MIN);
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < U; u++) {
                    if (u < nh) {
                        float lsum = 0.f, lmax = 0.f;           // CONTRIB: this lane's pixels
#pragma unroll
                        for (int p = 0; p < PPL; p++) {
                            const float a = av[u][p];
                            bool ok = (!done[p]) & pre[u][p];
                            const float test_T = __fmul_rn(T[p], 1.f - a);
                            if (ok && test_T < DGR_T_STOP) { done[p] = true; ok = false; }
                            if (ok) {
                                const float w = __fmul_rn(a, T[p]);
                                C0[p] = __fmaf_rn(cr[u], w, C0[p]); C1[p] = __fmaf_rn(cg[u], w, C1[p]); C2[p] = __fmaf_rn(cb[u], w, C2[p]);
                                D[p] = __fmaf_rn(dep[u], w, D[p]);
                                T[p] = test_T;
                                last[p] = (unsigned)(c * kChunk + js[u] + 1);
                                if constexpr (CONTRIB) { lsum = __fadd_rn(lsum, w); lmax = fmaxf(lmax, w); }
                            }
                        }
                        if constexpr (CONTRIB) {
                            // w > 0 wherever the record is composited (alpha >= 1/255, T >= 1e-4): max 0 = not composited here
                            if (__any_sync(0xffffffffu, lmax > 0.f)) {
#pragma unroll
                                for (int o = 16; o > 0; o >>= 1) lsum = __fadd_rn(lsum, __shfl_xor_sync(0xffffffffu, lsum, o));
                                const unsigned m = __reduce_max_sync(0xffffffffu, __float_as_uint(lmax));
                                if (lane == js[u]) { csum = lsum; cmax = m; }
                            }
                        }
                    }
                }
            }
            if constexpr (CONTRIB) {
                if (cmax) {
                    atomicAdd(cw.sum_fx + cid, __float2ull_rn(__fmul_rn(csum, kContribScale)));
                    atomicMax(cw.max_bits + cid, cmax);
                }
            }
            all_done = true;
#pragma unroll
            for (int p = 0; p < PPL; p++) all_done = all_done && done[p];
            warp_done = __all_sync(0xffffffffu, all_done);      // (also orders every lane's reads of stage s before its re-use)
            if (!warp_done && rs.issued < nchunks) {
                ring_fill<LAZY>(rg, rs.issued, src, rec, nid, rs.issued, min(kChunk, n - rs.issued * kChunk), lane);
                rs.issued++;
                if (lazy && rs.issued * kChunk + lane < n) nid = __ldg(ids + rs.issued * kChunk + lane);
            }
        }
        // never move on (or leave) with a bulk copy in flight into this warp's ring
        for (int c = rs.waited; c < rs.issued; c++) ring_wait(rg, rs, c);

        if constexpr (VIEWS) {              // view v's background and its [3, H_v, W_v] / [H_v, W_v] blocks at pixel pix_off[v]
            const float vb0 = __ldg(bg + 3 * v), vb1 = __ldg(bg + 3 * v + 1), vb2 = __ldg(bg + 3 * v + 2);
            const size_t vb = (size_t)vt->pix_off[v], vhw = (size_t)iH * iW;
            float *oc = out_color + 3 * vb, *od = out_depth + vb, *oa = out_alpha + vb, *fT = final_T + vb;
            unsigned *nc = n_contrib + vb;
#pragma unroll
            for (int p = 0; p < PPL; p++) {
                if (inside[p]) {
                    const size_t pix = (size_t)ST::py(wy0, lane, p) * iW + ST::px(wx0, lane, p);
                    oc[pix] = C0[p] + T[p] * vb0;
                    oc[vhw + pix] = C1[p] + T[p] * vb1;
                    oc[2 * vhw + pix] = C2[p] + T[p] * vb2;
                    od[pix] = D[p];
                    oa[pix] = 1.f - T[p];
                    nc[pix] = last[p];
                    fT[pix] = T[p];
                }
            }
        } else {
#pragma unroll
        for (int p = 0; p < PPL; p++) {
            if (inside[p]) {
                const size_t pix = (size_t)ST::py(wy0, lane, p) * W + ST::px(wx0, lane, p);
                out_color[pix] = C0[p] + T[p] * b0;
                out_color[HW + pix] = C1[p] + T[p] * b1;
                out_color[2 * HW + pix] = C2[p] + T[p] * b2;
                out_depth[pix] = D[p];
                out_alpha[pix] = 1.f - T[p];
                n_contrib[pix] = last[p];
                final_T[pix] = T[p];
            }
        }
        }
        if (costing && n > 0) {
            // this forward item's share of its backward item's cost; whoever completes the backward item files it under its class
            bool contrib = false;
#pragma unroll
            for (int p = 0; p < PPL; p++) contrib = contrib || (last[p] > 0u);
            contrib = __any_sync(0xffffffffu, contrib);
            if (lane == 0) {
                const int parts = co.bwd_ppl / PPL;                                       // forward items per backward item
                const int bsub = co.bwd_ppl == 1 ? ((wy0 & 15) >> 2) * 2 + ((wx0 & 15) >> 3)
                                                 : ((wy0 & 15) >> 3) * 2 + ((wx0 & 15) >> 3);
                const unsigned mine = contrib ? cost + 1u : 0u;
                unsigned total = mine;
                bool complete = true;
                if (parts > 1) {                  // several forward items feed one backward item: the last one to arrive files it
                    const unsigned old = atomicAdd(co.cost_acc + (size_t)tile * 8 + bsub, (mine << 2) | 1u);
                    complete = (int)(old & 3u) + 1 == parts;
                    total = (old >> 2) + mine;
                }
                if (complete && total > 0u) {
                    const int cls = cost_class(total);
                    pend_pos = atomicAdd(co.cls_count + cls, 1u);                        // (looked at after the next item was requested)
                    pend_base = (unsigned)cls * (unsigned)co.tiles * 8u; pend_val = ot * 8u + (unsigned)bsub; pend = true;
                }
            }
        }
        __syncwarp();
    }
}

template <int PPL, int U, bool LAZY>
__global__ void __launch_bounds__(kRenderThreads, PPL == 1 ? 8 : 1)
render_fwd_kernel(int H, int W, int gx, const unsigned *__restrict__ tile_order, const uint2 *__restrict__ order_ranges,
                  const unsigned *__restrict__ n_tiles_nonempty, unsigned n_items, unsigned long long *__restrict__ work_next,
                  int two_ended, int sms, CostOrder co, unsigned *__restrict__ lazy_note,
                  const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ ids_sorted,
                  const float *__restrict__ bg, float *__restrict__ out_color,
                  float *__restrict__ out_depth, float *__restrict__ out_alpha, unsigned *__restrict__ n_contrib,
                  float *__restrict__ final_T) {
    render_fwd_body<PPL, U, LAZY, false>(H, W, gx, tile_order, order_ranges, n_tiles_nonempty, n_items, work_next, two_ended, sms, co, lazy_note, rec_sorted, rec, ids_sorted, bg, out_color, out_depth, out_alpha, n_contrib, final_T, nullptr);
}

// the batched forward: the default sub-tile shape <1,1> only (8 CTAs per SM, as render_fwd_kernel<1,1>)
template <bool LAZY>
__global__ void __launch_bounds__(kRenderThreads, 8)
render_views_fwd_kernel(const __grid_constant__ ViewTable vt, const unsigned *__restrict__ tile_order, const uint2 *__restrict__ order_ranges,
                  const unsigned *__restrict__ n_tiles_nonempty, unsigned n_items, unsigned long long *__restrict__ work_next,
                  int two_ended, int sms, CostOrder co, unsigned *__restrict__ lazy_note,
                  const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ ids_sorted,
                  const float *__restrict__ bg, float *__restrict__ out_color,
                  float *__restrict__ out_depth, float *__restrict__ out_alpha, unsigned *__restrict__ n_contrib,
                  float *__restrict__ final_T) {
    render_fwd_body<1, 1, LAZY, true>(0, 0, 0, tile_order, order_ranges, n_tiles_nonempty, n_items, work_next, two_ended, sms, co, lazy_note, rec_sorted, rec, ids_sorted, bg, out_color, out_depth, out_alpha, n_contrib, final_T, &vt);
}

// DGR_RASTER_CONTRIB: the default shape <1,1> with the blending-weight statistics (single view and batched).  Separate kernels,
// so every instantiation above stays as it was.
template <bool LAZY>
__global__ void __launch_bounds__(kRenderThreads, 8)
render_fwd_contrib_kernel(int H, int W, int gx, const unsigned *__restrict__ tile_order, const uint2 *__restrict__ order_ranges,
                  const unsigned *__restrict__ n_tiles_nonempty, unsigned n_items, unsigned long long *__restrict__ work_next,
                  int two_ended, int sms, CostOrder co, unsigned *__restrict__ lazy_note,
                  const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ ids_sorted,
                  const float *__restrict__ bg, float *__restrict__ out_color,
                  float *__restrict__ out_depth, float *__restrict__ out_alpha, unsigned *__restrict__ n_contrib,
                  float *__restrict__ final_T, ContribOut cw) {
    render_fwd_body<1, 1, LAZY, false, true>(H, W, gx, tile_order, order_ranges, n_tiles_nonempty, n_items, work_next, two_ended, sms, co, lazy_note, rec_sorted, rec, ids_sorted, bg, out_color, out_depth, out_alpha, n_contrib, final_T, nullptr, cw);
}

template <bool LAZY>
__global__ void __launch_bounds__(kRenderThreads, 8)
render_views_fwd_contrib_kernel(const __grid_constant__ ViewTable vt, const unsigned *__restrict__ tile_order, const uint2 *__restrict__ order_ranges,
                  const unsigned *__restrict__ n_tiles_nonempty, unsigned n_items, unsigned long long *__restrict__ work_next,
                  int two_ended, int sms, CostOrder co, unsigned *__restrict__ lazy_note,
                  const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ ids_sorted,
                  const float *__restrict__ bg, float *__restrict__ out_color,
                  float *__restrict__ out_depth, float *__restrict__ out_alpha, unsigned *__restrict__ n_contrib,
                  float *__restrict__ final_T, ContribOut cw) {
    render_fwd_body<1, 1, LAZY, true, true>(0, 0, 0, tile_order, order_ranges, n_tiles_nonempty, n_items, work_next, two_ended, sms, co, lazy_note, rec_sorted, rec, ids_sorted, bg, out_color, out_depth, out_alpha, n_contrib, final_T, &vt, cw);
}

// the fixed-point sums -> float32 (one thread per record); the max was raised in place
constexpr int kContribFinalizeThreads = 256;
__global__ void __launch_bounds__(kContribFinalizeThreads)
contrib_finalize_kernel(long long n, const unsigned long long *__restrict__ sum_fx, float *__restrict__ weight_sum) {
    const long long i = (long long)blockIdx.x * kContribFinalizeThreads + threadIdx.x;
    if (i < n) weight_sum[i] = __fmul_rn(__ull2float_rn(__ldg(sum_fx + i)), kContribUnscale);
}

// ----------------------------------------------------------------------------------------------------------------
// Backward.
// ----------------------------------------------------------------------------------------------------------------
constexpr int kBatch = 8;                                   // parked records per step-2 pass

template <int PPL>
struct BwdSmem {
    static constexpr int kPix = 32 * PPL;
    static constexpr int kRow = 2 * kPix + 4;               // floats per parked record: (u, w) per pixel; +4: conflict-free LDS.128 by record
    WarpRing ring;
    float uw[kBatch][kRow];
    float4 g[kPix];                                         // per pixel: dL/dC rgb, dL/dD
};

// U = hitting records whose alpha / skip decisions (all independent of the traversal state) are evaluated together before
// the short sequential T / R updates: shortens the dependent chain of a warp that walks a long list.
// ROWSUM = the step-2 accumulation uses that the 8 pixels a lane covers per pass lie on ONE pixel row: dy is constant over them, so
// only sum u, sum u dx, sum u dx^2 run per pixel and the three dy moments follow from them per row (5 instead of 8 floating-point
// instructions per (record, pixel) on the u side).  ROWSUM = false keeps the per-pixel form (A/B: dgr_set_tuning bit 26).
// VIEWS: the batched backward (dgr_views_backward), tiles and images numbered as in render_fwd_body; the moments go to the
// records of the batch (the ids the sort wrote are record numbers v P + g).
// ABS (DGR_RASTER_ABS_GRAD, per-row step 2 only): step 2 also sums |u (A dx + B dy)| and |u (B dx + C dy)| over the pixels, the
// per-pixel terms of the pixel-space mean gradient before they can cancel, into moment slots 10 and 11 (absgrad_stats_kernel
// turns them into the AbsGS statistic).  The conic is parked with the record, its -1/2 log2 e scaling undone once per record.
template <int PPL, int U, bool LAZY, bool ROWSUM, bool VIEWS, bool ABS = false>
__device__ __forceinline__ void
render_bwd_body(int H, int W, int gx, const unsigned *__restrict__ tile_order, const unsigned *__restrict__ n_tiles_nonempty,
                  unsigned long long *__restrict__ work_next, int two_ended, int sms, CostOrder co, const uint2 *__restrict__ order_ranges,
                  const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ lazy_note,
                  const unsigned *__restrict__ ids_sorted, const float *__restrict__ bg,
                  const float *__restrict__ final_T, const unsigned *__restrict__ n_contrib,
                  const float *__restrict__ gC, const float *__restrict__ gD, const float *__restrict__ gA,
                  float *__restrict__ grad_rec, const ViewTable *vt) {
    static_assert(!ABS || ROWSUM, "the absolute moments exist in the per-row step 2 only");
    using ST = SubTile<PPL>;
    using SM = BwdSmem<PPL>;
    constexpr int kPix = SM::kPix;
    constexpr int kQ = 32 / kBatch;                          // pixel groups per record in step 2 (4)
    constexpr int kPixPerLane = kPix / kQ;                   // 8 (PPL 1) or 16 (PPL 2)
    extern __shared__ __align__(128) unsigned char smem_raw[];
    SM &sm = reinterpret_cast<SM *>(smem_raw)[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    WarpRing &rg = sm.ring;
    RingState rs;
    pdl_trigger();                       // the per-Gaussian backward may take the SM resources this grid's tail frees
    ring_init(rg, rs, lane);
    // work list: the measured-cost classes of the forward (heaviest class first) when it grouped its costs for this sub-tile
    // shape, else every sub-tile of the non-empty tiles in population order
    constexpr bool lazy = LAZY;                                      // the host launches the variant its forward used
    (void)lazy_note;
    const bool by_cost = co.cost_acc != nullptr && __ldcg(co.cost_bpt) == (unsigned)ST::kPerTile;
    unsigned cum_end = 0;                                            // lane L: items in classes kCostClasses-1 .. kCostClasses-1-L
    if (by_cost) {
        cum_end = __ldcg(co.cls_count + (kCostClasses - 1 - lane));
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, cum_end, o); if (lane >= o) cum_end += t; }
    }
    const unsigned n_items = by_cost ? __shfl_sync(0xffffffffu, cum_end, 31) : __ldcg(n_tiles_nonempty) * (unsigned)ST::kPerTile;
    float b0 = 0.f, b1 = 0.f, b2 = 0.f;
    if (!VIEWS) { b0 = __ldg(bg); b1 = __ldg(bg + 1); b2 = __ldg(bg + 2); }
    const size_t HW = (size_t)H * W;
    const int my_r = lane & (kBatch - 1), my_q = lane / kBatch;      // step 2: parked record, pixel group

    const bool light = two_ended && (((blockIdx.x / (unsigned)sms) + (threadIdx.x >> 5)) & 1u);
    for (;;) {
        unsigned fetched = 0;                                        // taken when the warp is ready for it (see the forward)
        if (lane == 0) fetched = queue_take(work_next, light, n_items);
        unsigned item = __shfl_sync(0xffffffffu, fetched, 0);
        if (item >= n_items) break;
        if (by_cost) {                                               // rank in the heaviest-first order -> (class, position) -> item
            const unsigned before = __ballot_sync(0xffffffffu, cum_end <= item);
            const int k = __popc(before);                            // classes completely in front of this rank
            const unsigned base = k ? __shfl_sync(0xffffffffu, cum_end, k - 1) : 0u;
            item = __ldcg(co.cls_items + (size_t)(kCostClasses - 1 - k) * co.tiles * 8 + (item - base));
        }
        const unsigned ot = by_cost ? item / 8u : item / ST::kPerTile;
        const int tile = (int)__ldcg(tile_order + ot), sub = (int)(by_cost ? item % 8u : item % ST::kPerTile);
        const uint2 range = __ldcg(order_ranges + ot);
        int v = 0, lt = tile, iW = W, iH = H, igx = gx;          // VIEWS: the item's view and its size
        if constexpr (VIEWS) { v = view_of_tile(*vt, tile); lt = tile - vt->tile_off[v]; iW = vt->W[v]; iH = vt->H[v]; igx = vt->gx[v]; }
        const int tx = lt % igx, ty = lt / igx;
        const int wx0 = ST::x0(tx, sub), wy0 = ST::y0(ty, sub);
        const int wx1 = wx0 + ST::kW - 1, wy1 = wy0 + ST::kH - 1;
        const float *vfT = final_T, *vgC = gC, *vgD = gD, *vgA = gA;
        const unsigned *vnc = n_contrib;
        size_t iHW = HW;
        if constexpr (VIEWS) {
            b0 = __ldg(bg + 3 * v); b1 = __ldg(bg + 3 * v + 1); b2 = __ldg(bg + 3 * v + 2);
            const size_t vb = (size_t)vt->pix_off[v];
            iHW = (size_t)iH * iW;
            vfT += vb; vnc += vb;
            if (gC) vgC += 3 * vb;
            if (gD) vgD += vb;
            if (gA) vgA += vb;
        }

        float fx[PPL], fy[PPL], gc0[PPL], gc1[PPL], gc2[PPL], gd[PPL], ga[PPL], T[PPL], R[PPL];
        unsigned last[PPL];
        unsigned lmax = 0;
#pragma unroll
        for (int p = 0; p < PPL; p++) {
            const int x = ST::px(wx0, lane, p), y = ST::py(wy0, lane, p);
            fx[p] = (float)x; fy[p] = (float)y;
            gc0[p] = 0.f; gc1[p] = 0.f; gc2[p] = 0.f; gd[p] = 0.f; ga[p] = 0.f; T[p] = 1.f; last[p] = 0;
            if ((x < iW) && (y < iH)) {
                const size_t pix = (size_t)y * iW + x;
                last[p] = __ldcg(vnc + pix);
                T[p] = __ldcg(vfT + pix);
                if (gC) { gc0[p] = __ldg(vgC + pix); gc1[p] = __ldg(vgC + iHW + pix); gc2[p] = __ldg(vgC + 2 * iHW + pix); }
                if (gD) gd[p] = __ldg(vgD + pix);
                if (gA) ga[p] = __ldg(vgA + pix);
            }
            // R = T_final * (bg . gC) + sum over Gaussians behind the current one of w * s
            R[p] = T[p] * (b0 * gc0[p] + b1 * gc1[p] + b2 * gc2[p]);
            lmax = max(lmax, last[p]);
            sm.g[p * 32 + lane] = make_float4(gc0[p], gc1[p], gc2[p], gd[p]);
        }
        unsigned wlast = lmax;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) wlast = max(wlast, __shfl_xor_sync(0xffffffffu, wlast, o));
        if (wlast == 0) { __syncwarp(); continue; }
        const int n = (int)wlast;                              // records [0, n) of the tile's list reach this sub-tile
        const int nchunks = (n + kChunk - 1) / kChunk;
        const Rec *src = rec_sorted + range.x;
        const unsigned *ids = ids_sorted + range.x;
        // sequence number k handles chunk nchunks-1-k (back to front)
        rs.issued = 0; rs.waited = 0;
        unsigned nid = 0;                                       // lazy: this lane's Gaussian id in the next chunk to be issued
        {
            unsigned id0[kRing];
#pragma unroll
            for (int k = 0; k < kRing; k++) { const int c = nchunks - 1 - k; id0[k] = (lazy && c >= 0 && c * kChunk + lane < n) ? __ldg(ids + c * kChunk + lane) : 0u; }
            if (lazy && nchunks > kRing) nid = __ldg(ids + (size_t)(nchunks - 1 - kRing) * kChunk + lane);
#pragma unroll
            for (int k = 0; k < kRing; k++) {
                const int c = nchunks - 1 - k;
                if (c >= 0) ring_fill<LAZY>(rg, k, src, rec, id0[k], c, min(kChunk, n - c * kChunk), lane);
            }
        }
        rs.issued = min(kRing, nchunks);

        // parked-record bookkeeping: lane L < kBatch owns slot L (centre relative to the sub-tile origin, Gaussian id)
        int nslots = 0;
        float cap_cx = 0.f, cap_cy = 0.f;
        unsigned cap_id = 0;
        float cap_ca = 0.f, cap_cb = 0.f, cap_cc = 0.f;          // ABS: the record's conic (A, B, C)

        // step 2: the kBatch parked records -> 10 moments each.  Lane (my_r, my_q) covers pixel group my_q of record my_r.
        auto flush = [&]() {
            __syncwarp();
            const float ccx = __shfl_sync(0xffffffffu, cap_cx, my_r), ccy = __shfl_sync(0xffffffffu, cap_cy, my_r);
            float v0 = 0.f, v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f, v5 = 0.f, v6 = 0.f, v7 = 0.f, v8 = 0.f, v9 = 0.f;
            float v10 = 0.f, v11 = 0.f, ca = 0.f, cb = 0.f, cc = 0.f;
            if constexpr (ABS) {
                ca = __shfl_sync(0xffffffffu, cap_ca, my_r); cb = __shfl_sync(0xffffffffu, cap_cb, my_r); cc = __shfl_sync(0xffffffffu, cap_cc, my_r);
            }
            const float *row = &sm.uw[my_r][0];
            if (ROWSUM) {
                static_assert(kPixPerLane % 8 == 0, "a lane's pixels come in rows of 8");
#pragma unroll
                for (int g8 = 0; g8 < kPixPerLane / 8; g8++) {
                    const int kb = my_q * kPixPerLane + 8 * g8;               // first pixel of this row of 8 (p * 32 + lane of step 1)
                    const int pl = kb & 31, pp = kb >> 5;
                    const float dxb = ccx - (float)((PPL == 4 && (pp & 1)) ? 8 : 0);
                    const float dy = ccy - (float)((pl >> 3) + ((PPL == 4) ? (pp >> 1) * 4 : pp * 4));
                    float s0 = 0.f, s1 = 0.f, s3 = 0.f;
                    const float bdy = ABS ? cb * dy : 0.f, cdy = ABS ? cc * dy : 0.f;   // ABS: the row's dy terms of A dx + B dy, B dx + C dy
#pragma unroll
                    for (int i = 0; i < 8; i += 2) {
                        const float4 t = *reinterpret_cast<const float4 *>(row + 2 * (kb + i));   // (u, w) of pixels kb + i, kb + i + 1
#pragma unroll
                        for (int e = 0; e < 2; e++) {
                            const float u = e ? t.z : t.x, w = e ? t.w : t.y;
                            const float dx = dxb - (float)(i + e);
                            const float4 g = sm.g[kb + i + e];
                            const float udx = u * dx;
                            s0 += u; s1 += udx; s3 = __fmaf_rn(udx, dx, s3);
                            v6 = __fmaf_rn(w, g.x, v6); v7 = __fmaf_rn(w, g.y, v7); v8 = __fmaf_rn(w, g.z, v8); v9 = __fmaf_rn(w, g.w, v9);
                            if constexpr (ABS) {
                                const float au = fabsf(u);
                                v10 = __fmaf_rn(au, fabsf(__fmaf_rn(ca, dx, bdy)), v10);
                                v11 = __fmaf_rn(au, fabsf(__fmaf_rn(cb, dx, cdy)), v11);
                            }
                        }
                    }
                    if (g8 == 0) { v0 = s0; v1 = s1; v3 = s3; v2 = dy * s0; v4 = dy * s1; v5 = (dy * dy) * s0; }
                    else {
                        v0 += s0; v1 += s1; v3 += s3;
                        v2 = __fmaf_rn(dy, s0, v2); v4 = __fmaf_rn(dy, s1, v4); v5 = __fmaf_rn(dy * dy, s0, v5);
                    }
                }
            } else {
#pragma unroll
            for (int i = 0; i < kPixPerLane; i += 2) {
                const int k = my_q * kPixPerLane + i;                     // pixel index of the sub-tile (p * 32 + lane of step 1)
                const float4 t = *reinterpret_cast<const float4 *>(row + 2 * k);     // (u, w) of pixels k, k + 1
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int kk = k + e;
                    const float u = e ? t.z : t.x, w = e ? t.w : t.y;
                    const int pl = kk & 31, pp = kk >> 5;
                    const float dx = ccx - (float)((pl & 7) + ((PPL == 4 && (pp & 1)) ? 8 : 0));
                    const float dy = ccy - (float)((pl >> 3) + ((PPL == 4) ? (pp >> 1) * 4 : pp * 4));
                    const float4 g = sm.g[kk];
                    const float udx = u * dx, udy = u * dy;
                    v0 += u; v1 += udx; v2 += udy;
                    v3 = __fmaf_rn(udx, dx, v3); v4 = __fmaf_rn(udx, dy, v4); v5 = __fmaf_rn(udy, dy, v5);
                    v6 = __fmaf_rn(w, g.x, v6); v7 = __fmaf_rn(w, g.y, v7); v8 = __fmaf_rn(w, g.z, v8); v9 = __fmaf_rn(w, g.w, v9);
                }
            }
            }
#pragma unroll
            for (int o = kBatch; o < 32; o <<= 1) {
                v0 += __shfl_xor_sync(0xffffffffu, v0, o); v1 += __shfl_xor_sync(0xffffffffu, v1, o);
                v2 += __shfl_xor_sync(0xffffffffu, v2, o); v3 += __shfl_xor_sync(0xffffffffu, v3, o);
                v4 += __shfl_xor_sync(0xffffffffu, v4, o); v5 += __shfl_xor_sync(0xffffffffu, v5, o);
                v6 += __shfl_xor_sync(0xffffffffu, v6, o); v7 += __shfl_xor_sync(0xffffffffu, v7, o);
                v8 += __shfl_xor_sync(0xffffffffu, v8, o); v9 += __shfl_xor_sync(0xffffffffu, v9, o);
                if constexpr (ABS) { v10 += __shfl_xor_sync(0xffffffffu, v10, o); v11 += __shfl_xor_sync(0xffffffffu, v11, o); }
            }
            // vector reductions (the row is 16-byte aligned, GeomLayout): L2 absorbs about as many reductions per second whatever
            // their width, so 4 per record take 2.5x less time than 10 scalar ones (tools/red_probe.py).  The single-view by-id
            // variant keeps the scalar form: under the 80-register cap the vector operands' register pairs and quads cost it 8 more
            // bytes of stack (16 -> 24).
            if (lane < nslots) {
                float *dst = grad_rec + (size_t)cap_id * kGradRecFloats;
                if constexpr (LAZY && !VIEWS && !ABS) {
                    red_add_f32(dst, v0); red_add_f32(dst + 1, v1); red_add_f32(dst + 2, v2); red_add_f32(dst + 3, v3);
                    red_add_f32(dst + 4, v4); red_add_f32(dst + 5, v5); red_add_f32(dst + 6, v6); red_add_f32(dst + 7, v7);
                    red_add_f32(dst + 8, v8); red_add_f32(dst + 9, v9);
                } else {
                    red_add_v4_f32(dst, v0, v1, v2, v3);
                    if constexpr (ABS) { red_add_v4_f32(dst + 4, v4, v5, v6, v7); red_add_v2_f32(dst + 10, v10, v11); }
                    else { red_add_v2_f32(dst + 4, v4, v5); red_add_v2_f32(dst + 6, v6, v7); }
                    red_add_v2_f32(dst + 8, v8, v9);
                }
            }
            nslots = 0;
            __syncwarp();
        };

        for (int k = 0; k < nchunks; k++) {
            const int c = nchunks - 1 - k;
            const int cnt = min(kChunk, n - c * kChunk);
            unsigned my_id = 0;
            if (lane < cnt) my_id = __ldg(ids + (size_t)c * kChunk + lane);
            const int s = ring_wait(rg, rs, k);
            rs.waited = k + 1;
            bool hit = false;
            if (lane < cnt) hit = record_hits_subtile(rg.rec[s][lane], wx0, wx1, wy0, wy1);
            unsigned mask = __ballot_sync(0xffffffffu, hit);
            while (mask) {
                int js[U];
                int nh = 0;
#pragma unroll
                for (int u = 0; u < U; u++) {
                    js[u] = 0;
                    if (mask) { js[u] = bfind_u32(mask); mask &= ~(1u << js[u]); nh = u + 1; }      // last record of the chunk first
                }
                float agv[U][PPL], av[U][PPL], rcx[U], rcy[U], dep[U], cr[U], cg[U], cb[U], rqa[U], rqb[U], rqc[U];
                bool okv[U][PPL], any_ok[U];
#pragma unroll
                for (int u = 0; u < U; u++) {
                    any_ok[u] = false;
                    if (u < nh) {
                        const Rec *r = &rg.rec[s][js[u]];
                        const float4 q0 = r->q0, q1 = r->q1, q2 = r->q2;
                        const unsigned gidx = (unsigned)(c * kChunk + js[u]);
                        rcx[u] = q0.x - (float)wx0; rcy[u] = q0.y - (float)wy0; dep[u] = q1.z; cr[u] = q2.x; cg[u] = q2.y; cb[u] = q2.z;
                        if constexpr (ABS) { rqa[u] = q0.z; rqb[u] = q0.w; rqc[u] = q1.x; }
                        bool mine = false;
#pragma unroll
                        for (int p = 0; p < PPL; p++) {
                            const float dx = q0.x - fx[p], dy = q0.y - fy[p];
                            const float p2 = eval_power2(q0, q1, dx, dy);
                            agv[u][p] = __fmul_rn(q1.y, ex2_approx(p2));
                            av[u][p] = fminf(DGR_ALPHA_MAX, agv[u][p]);
                            okv[u][p] = (gidx < last[p]) & (p2 <= 0.f) & (av[u][p] >= DGR_ALPHA_MIN);
                            mine = mine || okv[u][p];
                        }
                        any_ok[u] = __any_sync(0xffffffffu, mine);
                    }
                }
#pragma unroll
                for (int u = 0; u < U; u++) {
                    if (u < nh && any_ok[u]) {
                        float *row = &sm.uw[nslots][0];
#pragma unroll
                        for (int p = 0; p < PPL; p++) {
                            float uu = 0.f, w = 0.f;
                            if (okv[u][p]) {
                                const float ir = rcp_approx(1.f - av[u][p]);
                                T[p] = T[p] * ir;
                                const float sdot = __fmaf_rn(cr[u], gc0[p], __fmaf_rn(cg[u], gc1[p], __fmaf_rn(cb[u], gc2[p], __fmaf_rn(dep[u], gd[p], ga[p]))));
                                const float dL_da = T[p] * sdot - R[p] * ir;
                                w = av[u][p] * T[p];
                                R[p] = __fmaf_rn(w, sdot, R[p]);
                                uu = agv[u][p] * dL_da;
                            }
                            *reinterpret_cast<float2 *>(row + 2 * (p * 32 + lane)) = make_float2(uu, w);
                        }
                        const unsigned id_j = __shfl_sync(0xffffffffu, my_id, js[u]);
                        if (lane == nslots) {
                            cap_cx = rcx[u]; cap_cy = rcy[u]; cap_id = id_j;
                            if constexpr (ABS) { cap_ca = rqa[u] * (-2.f / kLog2e); cap_cb = rqb[u] * (-1.f / kLog2e); cap_cc = rqc[u] * (-2.f / kLog2e); }
                        }
                        nslots++;
                        if (nslots == kBatch) flush();
                    }
                }
            }
            __syncwarp();                                       // every lane has left stage s
            if (rs.issued < nchunks) {
                const int c2 = nchunks - 1 - rs.issued;
                ring_fill<LAZY>(rg, rs.issued, src, rec, nid, c2, min(kChunk, n - c2 * kChunk), lane);
                rs.issued++;
                if (lazy && rs.issued < nchunks) nid = __ldg(ids + (size_t)(nchunks - 1 - rs.issued) * kChunk + lane);
            }
        }
        if (nslots > 0) flush();
        __syncwarp();
    }
}

template <int PPL, int U, bool LAZY, bool ROWSUM = true>
__global__ void __launch_bounds__(kRenderThreads)
render_bwd_kernel(int H, int W, int gx, const unsigned *__restrict__ tile_order, const unsigned *__restrict__ n_tiles_nonempty,
                  unsigned long long *__restrict__ work_next, int two_ended, int sms, CostOrder co, const uint2 *__restrict__ order_ranges,
                  const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ lazy_note,
                  const unsigned *__restrict__ ids_sorted, const float *__restrict__ bg,
                  const float *__restrict__ final_T, const unsigned *__restrict__ n_contrib,
                  const float *__restrict__ gC, const float *__restrict__ gD, const float *__restrict__ gA,
                  float *__restrict__ grad_rec) {
    render_bwd_body<PPL, U, LAZY, ROWSUM, false>(H, W, gx, tile_order, n_tiles_nonempty, work_next, two_ended, sms, co, order_ranges, rec_sorted, rec, lazy_note, ids_sorted, bg, final_T, n_contrib, gC, gD, gA, grad_rec, nullptr);
}

// the batched backward: the default sub-tile shape <1,2> with the per-row step 2 only
template <bool LAZY>
__global__ void __launch_bounds__(kRenderThreads)
render_views_bwd_kernel(const __grid_constant__ ViewTable vt, const unsigned *__restrict__ tile_order, const unsigned *__restrict__ n_tiles_nonempty,
                  unsigned long long *__restrict__ work_next, int two_ended, int sms, CostOrder co, const uint2 *__restrict__ order_ranges,
                  const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ lazy_note,
                  const unsigned *__restrict__ ids_sorted, const float *__restrict__ bg,
                  const float *__restrict__ final_T, const unsigned *__restrict__ n_contrib,
                  const float *__restrict__ gC, const float *__restrict__ gD, const float *__restrict__ gA,
                  float *__restrict__ grad_rec) {
    render_bwd_body<1, 2, LAZY, true, true>(0, 0, 0, tile_order, n_tiles_nonempty, work_next, two_ended, sms, co, order_ranges, rec_sorted, rec, lazy_note, ids_sorted, bg, final_T, n_contrib, gC, gD, gA, grad_rec, &vt);
}

// DGR_RASTER_ABS_GRAD: the default shape <1,2> with the per-row step 2 that also leaves the absolute moments in slots 10 and 11
// (single view and batched).  Separate kernels, so every instantiation above stays as it was.
template <bool LAZY>
__global__ void __launch_bounds__(kRenderThreads)
render_bwd_abs_kernel(int H, int W, int gx, const unsigned *__restrict__ tile_order, const unsigned *__restrict__ n_tiles_nonempty,
                  unsigned long long *__restrict__ work_next, int two_ended, int sms, CostOrder co, const uint2 *__restrict__ order_ranges,
                  const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ lazy_note,
                  const unsigned *__restrict__ ids_sorted, const float *__restrict__ bg,
                  const float *__restrict__ final_T, const unsigned *__restrict__ n_contrib,
                  const float *__restrict__ gC, const float *__restrict__ gD, const float *__restrict__ gA,
                  float *__restrict__ grad_rec) {
    render_bwd_body<1, 2, LAZY, true, false, true>(H, W, gx, tile_order, n_tiles_nonempty, work_next, two_ended, sms, co, order_ranges, rec_sorted, rec, lazy_note, ids_sorted, bg, final_T, n_contrib, gC, gD, gA, grad_rec, nullptr);
}

template <bool LAZY>
__global__ void __launch_bounds__(kRenderThreads)
render_views_bwd_abs_kernel(const __grid_constant__ ViewTable vt, const unsigned *__restrict__ tile_order, const unsigned *__restrict__ n_tiles_nonempty,
                  unsigned long long *__restrict__ work_next, int two_ended, int sms, CostOrder co, const uint2 *__restrict__ order_ranges,
                  const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ lazy_note,
                  const unsigned *__restrict__ ids_sorted, const float *__restrict__ bg,
                  const float *__restrict__ final_T, const unsigned *__restrict__ n_contrib,
                  const float *__restrict__ gC, const float *__restrict__ gD, const float *__restrict__ gA,
                  float *__restrict__ grad_rec) {
    render_bwd_body<1, 2, LAZY, true, true, true>(0, 0, 0, tile_order, n_tiles_nonempty, work_next, two_ended, sms, co, order_ranges, rec_sorted, rec, lazy_note, ids_sorted, bg, final_T, n_contrib, gC, gD, gA, grad_rec, &vt);
}

}  // namespace dgr
