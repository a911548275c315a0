// dgr_det.cuh — the deterministic backward render (dgr_backward_det, dgr_views_backward_det, dgr_views_mixed_backward_det).
//
// The default backward (render_bwd_body) sends every (sub-tile, Gaussian) partial of the 10 moments to the Gaussian's row with
// red.global.add.f32, so the order of the float additions depends on which warp reaches which work item first.  Here every sum has
// a fixed order, and nothing is added with an atomic:
//   * render_bwd_det: one CTA = one non-empty tile = 8 warps, one 8x4 sub-tile each.  The CTA streams the tile's records back to front
//     through ONE shared bulk-TMA ring; the 8 warps walk the chunks in step.  Each warp runs the default kernel's step 1 (T, R,
//     dL/dalpha -> u, w per pixel, in list order) and step 2 (the moments of up to 8 parked records, per-row form) for its sub-tile
//     and leaves, per record of the chunk, its 10 moments in shared memory (zero if it did not hit the record).  After a CTA barrier
//     the 8 warps' values are added in warp order 0..7 and stored with plain stores into the record's instance slot;
//   * det_moments_gather: one thread per record sums its instance slots in slot order and stores the record's grad_rec row.
// Instance slots: record r's instances are the tiles of the rectangle of its packed pixel AABB (for_each_touched_tile, the rule of
// emit_keys), touched[r] & 0x1fffffff of them.  Instance (r, tile t) is slot goff[r] + k with k = t's row-major rank in that
// rectangle and goff the exclusive scan of the masked counts (det_counts_kernel + the knn_scan_* kernels).  Slots no sub-tile walks
// (records behind the last contributor of every pixel of the tile) keep the zeros of the backward's memset.
// Which CTA takes which tile, in which order, how many CTAs run, and how the records are staged change no result: every gradient is a
// function of the forward's scratch and the upstream gradients only.
#pragma once
#include "dgr_render.cuh"

namespace dgr {

constexpr int kDetWarps = 8;                          // the 8 sub-tiles of 8x4 pixels of a 16x16 tile
constexpr int kDetThreads = kDetWarps * 32;
constexpr unsigned kTouchedMask = 0x1fffffffu;        // tiles touched; the top 3 bits of `touched` are SH clamp flags

struct __align__(128) DetSmem {
    WarpRing ring;                                    // the CTA's ring of tile records (one ring, all 8 warps read it)
    float4 mom[2][kDetWarps][kChunk][3];              // [chunk parity][warp][record of the chunk]: 10 moments, 2 zero floats
    unsigned slot[2][kChunk];                         // [chunk parity][record of the chunk]: its instance slot
    float uw[kDetWarps][kBatch][BwdSmem<1>::kRow];    // step 1 -> step 2 of each warp: (u, w) per pixel of the parked records
    float4 g[kDetWarps][32];                          // per warp and pixel: dL/dC rgb, dL/dD
    unsigned wlast[kDetWarps];                        // per warp: the largest n_contrib of its sub-tile
    unsigned item;                                    // the tile the CTA works on (position in the tile order)
};

// the instance scratch of the deterministic backward: [moments 48 B x instances][goff u32 x records][scan block sums u32]
struct DetLayout {
    size_t off_mom, off_goff, off_sums, total, nblk;
    __host__ __device__ DetLayout(unsigned long long instances, long long records) {
        const size_t R = records > 0 ? (size_t)records : 1;
        nblk = (R + 4095) / 4096;                     // knn_scan_*: 4096 values per block
        size_t o = 0;
        off_mom = o;  o = align_up(o + (size_t)instances * kGradRecFloats * 4, 256);
        off_goff = o; o = align_up(o + R * 4, 256);
        off_sums = o; o = align_up(o + (nblk + 1) * 4, 256);
        total = o;
    }
};

// masked tiles-touched counts of the records, scanned in place (exclusive) into goff by the knn_scan_* kernels
__global__ void __launch_bounds__(256) det_counts_kernel(long long R, const unsigned *__restrict__ touched, unsigned *__restrict__ counts) {
    const long long r = (long long)blockIdx.x * 256 + threadIdx.x;
    if (r < R) counts[r] = __ldg(touched + r) & kTouchedMask;
}

// ABS (DGR_RASTER_ABS_GRAD): step 2 also leaves the absolute moments of render_bwd_body<.., ABS> in floats 10 and 11 of each row.
template <bool LAZY, bool VIEWS, bool ABS = false>
__device__ __forceinline__ void
render_bwd_det_body(int H, int W, int gx, const unsigned *__restrict__ tile_order, const uint2 *__restrict__ order_ranges,
                    const unsigned *__restrict__ n_tiles_nonempty, unsigned long long *__restrict__ work_next,
                    const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ ids_sorted,
                    const unsigned *__restrict__ goff, unsigned long long n_slots, const float *__restrict__ bg,
                    const float *__restrict__ final_T, const unsigned *__restrict__ n_contrib,
                    const float *__restrict__ gC, const float *__restrict__ gD, const float *__restrict__ gA,
                    float *__restrict__ det_mom, const ViewTable *vt) {
    using ST = SubTile<1>;
    constexpr int U = 2;                                             // hits evaluated together (the default backward's batching)
    constexpr int kPixPerLane = 32 / (32 / kBatch);                  // step 2: one row of 8 pixels per lane
    extern __shared__ __align__(128) unsigned char smem_raw[];
    DetSmem &sm = *reinterpret_cast<DetSmem *>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpRing &rg = sm.ring;
    RingState rs;
    pdl_trigger();                       // the gather kernel may become resident as this grid's tail frees the SMs
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < kRing; i++) mbar_init(&rg.full[i], 1);
        mbar_fence_init();
    }
    rs.phase = 0; rs.issued = 0; rs.waited = 0;
    for (int i = threadIdx.x; i < 2 * kDetWarps * kChunk * 3; i += kDetThreads) (&sm.mom[0][0][0][0])[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    pdl_wait();                          // goff (the scan right before this kernel)

    const unsigned n_tiles = __ldcg(n_tiles_nonempty);
    float b0 = 0.f, b1 = 0.f, b2 = 0.f;
    if (!VIEWS) { b0 = __ldg(bg); b1 = __ldg(bg + 1); b2 = __ldg(bg + 2); }
    const int my_r = lane & (kBatch - 1), my_q = lane / kBatch;      // step 2: parked record, pixel row
    for (;;) {
        if (threadIdx.x == 0) sm.item = (unsigned)atomicAdd(work_next, 1ull);
        __syncthreads();
        const unsigned ot = sm.item;
        if (ot >= n_tiles) break;
        const int tile = (int)__ldcg(tile_order + ot);
        const uint2 range = __ldcg(order_ranges + ot);
        int v = 0, lt = tile, iW = W, iH = H, igx = gx;              // VIEWS: the tile's view and its size
        if constexpr (VIEWS) { v = view_of_tile(*vt, tile); lt = tile - vt->tile_off[v]; iW = vt->W[v]; iH = vt->H[v]; igx = vt->gx[v]; }
        const int tx = lt % igx, ty = lt / igx;
        const int wx0 = ST::x0(tx, warp), wy0 = ST::y0(ty, warp);
        const int wx1 = wx0 + ST::kW - 1, wy1 = wy0 + ST::kH - 1;
        const float *vfT = final_T, *vgC = gC, *vgD = gD, *vgA = gA;
        const unsigned *vnc = n_contrib;
        size_t iHW = (size_t)H * W;
        if constexpr (VIEWS) {
            b0 = __ldg(bg + 3 * v); b1 = __ldg(bg + 3 * v + 1); b2 = __ldg(bg + 3 * v + 2);
            const size_t vb = (size_t)vt->pix_off[v];
            iHW = (size_t)iH * iW;
            vfT += vb; vnc += vb;
            if (gC) vgC += 3 * vb;
            if (gD) vgD += vb;
            if (gA) vgA += vb;
        }
        // step 1 state: lane = pixel of the warp's sub-tile
        const int px = ST::px(wx0, lane, 0), py = ST::py(wy0, lane, 0);
        const float fx = (float)px, fy = (float)py;
        float gc0 = 0.f, gc1 = 0.f, gc2 = 0.f, gd = 0.f, ga = 0.f, T = 1.f;
        unsigned last = 0;
        if (px < iW && py < iH) {
            const size_t pix = (size_t)py * iW + px;
            last = __ldcg(vnc + pix);
            T = __ldcg(vfT + pix);
            if (gC) { gc0 = __ldg(vgC + pix); gc1 = __ldg(vgC + iHW + pix); gc2 = __ldg(vgC + 2 * iHW + pix); }
            if (gD) gd = __ldg(vgD + pix);
            if (gA) ga = __ldg(vgA + pix);
        }
        float R = T * (b0 * gc0 + b1 * gc1 + b2 * gc2);
        sm.g[warp][lane] = make_float4(gc0, gc1, gc2, gd);
        unsigned wl = last;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) wl = max(wl, __shfl_xor_sync(0xffffffffu, wl, o));
        if (lane == 0) sm.wlast[warp] = wl;
        __syncthreads();
        unsigned nt = 0;
#pragma unroll
        for (int w = 0; w < kDetWarps; w++) nt = max(nt, sm.wlast[w]);
        if (nt == 0) continue;
        const int n = (int)nt;                                       // records [0, n) of the tile's list reach some pixel of the tile
        const int nchunks = (n + kChunk - 1) / kChunk;
        const Rec *src = rec_sorted + range.x;
        const unsigned *ids = ids_sorted + range.x;
        // sequence number k handles chunk nchunks-1-k (back to front); warp 0 issues, everybody waits
        if (warp == 0) {
#pragma unroll
            for (int k = 0; k < kRing; k++) {
                const int c = nchunks - 1 - k;
                if (c >= 0) {
                    const int cnt = min(kChunk, n - c * kChunk);
                    const unsigned id = (LAZY && lane < cnt) ? __ldg(ids + c * kChunk + lane) : 0u;
                    ring_fill<LAZY>(rg, k, src, rec, id, c, cnt, lane);
                }
            }
        }
        rs.issued = min(kRing, nchunks);

        int nslots = 0, cap_j = 0;                                   // parked records: lane L < kBatch owns slot L
        float cap_cx = 0.f, cap_cy = 0.f;
        float cap_ca = 0.f, cap_cb = 0.f, cap_cc = 0.f;              // ABS: the record's conic (A, B, C)
        auto flush = [&](int buf) {                                  // step 2 of the default kernel (per-row form), to shared memory
            __syncwarp();
            const float ccx = __shfl_sync(0xffffffffu, cap_cx, my_r), ccy = __shfl_sync(0xffffffffu, cap_cy, my_r);
            const float *row = &sm.uw[warp][my_r][0];
            const int kb = my_q * kPixPerLane;
            const float dy = ccy - (float)my_q;
            float s0 = 0.f, s1 = 0.f, s3 = 0.f, v6 = 0.f, v7 = 0.f, v8 = 0.f, v9 = 0.f;
            float v10 = 0.f, v11 = 0.f, ca = 0.f, cb = 0.f, bdy = 0.f, cdy = 0.f;
            if constexpr (ABS) {
                ca = __shfl_sync(0xffffffffu, cap_ca, my_r); cb = __shfl_sync(0xffffffffu, cap_cb, my_r);
                const float cc = __shfl_sync(0xffffffffu, cap_cc, my_r);
                bdy = cb * dy; cdy = cc * dy;
            }
#pragma unroll
            for (int i = 0; i < 8; i += 2) {
                const float4 t = *reinterpret_cast<const float4 *>(row + 2 * (kb + i));
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const float u = e ? t.z : t.x, w = e ? t.w : t.y;
                    const float dx = ccx - (float)(i + e);
                    const float4 g = sm.g[warp][kb + i + e];
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
            float v0 = s0, v1 = s1, v3 = s3, v2 = dy * s0, v4 = dy * s1, v5 = (dy * dy) * s0;
#pragma unroll
            for (int o = kBatch; o < 32; o <<= 1) {
                v0 += __shfl_xor_sync(0xffffffffu, v0, o); v1 += __shfl_xor_sync(0xffffffffu, v1, o);
                v2 += __shfl_xor_sync(0xffffffffu, v2, o); v3 += __shfl_xor_sync(0xffffffffu, v3, o);
                v4 += __shfl_xor_sync(0xffffffffu, v4, o); v5 += __shfl_xor_sync(0xffffffffu, v5, o);
                v6 += __shfl_xor_sync(0xffffffffu, v6, o); v7 += __shfl_xor_sync(0xffffffffu, v7, o);
                v8 += __shfl_xor_sync(0xffffffffu, v8, o); v9 += __shfl_xor_sync(0xffffffffu, v9, o);
                if constexpr (ABS) { v10 += __shfl_xor_sync(0xffffffffu, v10, o); v11 += __shfl_xor_sync(0xffffffffu, v11, o); }
            }
            if (lane < nslots) {
                float4 *dst = sm.mom[buf][warp][cap_j];
                dst[0] = make_float4(v0, v1, v2, v3); dst[1] = make_float4(v4, v5, v6, v7); dst[2] = make_float4(v8, v9, v10, v11);
            }
            nslots = 0;
            __syncwarp();
        };

        for (int k = 0; k < nchunks; k++) {
            const int c = nchunks - 1 - k;
            const int cnt = min(kChunk, n - c * kChunk);
            const int buf = k & 1;
            unsigned my_id = 0;
            if (lane < cnt) my_id = __ldg(ids + (size_t)c * kChunk + lane);
            const int s = ring_wait(rg, rs, k);
            bool hit = false;
            if (lane < cnt && wl > 0) hit = record_hits_subtile(rg.rec[s][lane], wx0, wx1, wy0, wy1);
            unsigned mask = __ballot_sync(0xffffffffu, hit);
            while (mask) {
                int js[U];
                int nh = 0;
#pragma unroll
                for (int u = 0; u < U; u++) {
                    js[u] = 0;
                    if (mask) { js[u] = bfind_u32(mask); mask &= ~(1u << js[u]); nh = u + 1; }      // last record of the chunk first
                }
                float agv[U], av[U], rcx[U], rcy[U], dep[U], cr[U], cg[U], cb[U], rqa[U], rqb[U], rqc[U];
                bool okv[U], any_ok[U];
#pragma unroll
                for (int u = 0; u < U; u++) {
                    any_ok[u] = false; okv[u] = false;
                    if (u < nh) {
                        const Rec *r = &rg.rec[s][js[u]];
                        const float4 q0 = r->q0, q1 = r->q1, q2 = r->q2;
                        const unsigned gidx = (unsigned)(c * kChunk + js[u]);
                        rcx[u] = q0.x - (float)wx0; rcy[u] = q0.y - (float)wy0; dep[u] = q1.z; cr[u] = q2.x; cg[u] = q2.y; cb[u] = q2.z;
                        if constexpr (ABS) { rqa[u] = q0.z; rqb[u] = q0.w; rqc[u] = q1.x; }
                        const float dx = q0.x - fx, dy = q0.y - fy;
                        const float p2 = eval_power2(q0, q1, dx, dy);
                        agv[u] = __fmul_rn(q1.y, ex2_approx(p2));
                        av[u] = fminf(DGR_ALPHA_MAX, agv[u]);
                        okv[u] = (gidx < last) & (p2 <= 0.f) & (av[u] >= DGR_ALPHA_MIN);
                        any_ok[u] = __any_sync(0xffffffffu, okv[u]);
                    }
                }
#pragma unroll
                for (int u = 0; u < U; u++) {
                    if (u < nh && any_ok[u]) {
                        float uu = 0.f, w = 0.f;
                        if (okv[u]) {
                            const float ir = rcp_approx(1.f - av[u]);
                            T = T * ir;
                            const float sdot = __fmaf_rn(cr[u], gc0, __fmaf_rn(cg[u], gc1, __fmaf_rn(cb[u], gc2, __fmaf_rn(dep[u], gd, ga))));
                            const float dL_da = T * sdot - R * ir;
                            w = av[u] * T;
                            R = __fmaf_rn(w, sdot, R);
                            uu = agv[u] * dL_da;
                        }
                        *reinterpret_cast<float2 *>(&sm.uw[warp][nslots][2 * lane]) = make_float2(uu, w);
                        if (lane == nslots) {
                            cap_cx = rcx[u]; cap_cy = rcy[u]; cap_j = js[u];
                            if constexpr (ABS) { cap_ca = rqa[u] * (-2.f / kLog2e); cap_cb = rqb[u] * (-1.f / kLog2e); cap_cc = rqc[u] * (-2.f / kLog2e); }
                        }
                        nslots++;
                        if (nslots == kBatch) flush(buf);
                    }
                }
            }
            if (nslots > 0) flush(buf);                              // every moment of this chunk is in shared memory
            if (warp == 0 && lane < cnt) {                           // instance slot of record `lane` of the chunk in this tile
                const Rec &r = rg.rec[s][lane];
                const unsigned ax = __float_as_uint(r.q1.w), ay = __float_as_uint(r.q2.w);
                const int tx0 = (int)(ax & 0xffffu) >> 4, tw = ((int)(ax >> 16) >> 4) - tx0 + 1, ty0 = (int)(ay & 0xffffu) >> 4;
                sm.slot[buf][lane] = __ldg(goff + my_id) + (unsigned)((ty - ty0) * tw + (tx - tx0));
            }
            __syncthreads();                                         // every warp has left stage s and written its moments
            if (warp == 0 && rs.issued < nchunks) {
                const int c2 = nchunks - 1 - rs.issued;
                const int cnt2 = min(kChunk, n - c2 * kChunk);
                const unsigned id = (LAZY && lane < cnt2) ? __ldg(ids + (size_t)c2 * kChunk + lane) : 0u;
                ring_fill<LAZY>(rg, rs.issued, src, rec, id, c2, cnt2, lane);
            }
            if (rs.issued < nchunks) rs.issued++;
            if ((int)threadIdx.x < 3 * cnt) {                        // the 8 warps' moments in warp order, one float4 per thread
                const int j = threadIdx.x / 3, q = threadIdx.x % 3;
                float4 a = sm.mom[buf][0][j][q];
                sm.mom[buf][0][j][q] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int w = 1; w < kDetWarps; w++) {
                    const float4 b = sm.mom[buf][w][j][q];
                    sm.mom[buf][w][j][q] = make_float4(0.f, 0.f, 0.f, 0.f);
                    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
                }
                const unsigned long long slot = sm.slot[buf][j];
                if (slot < n_slots) reinterpret_cast<float4 *>(det_mom + slot * kGradRecFloats)[q] = a;
            }
        }
    }
}

template <bool LAZY>
__global__ void __launch_bounds__(kDetThreads)
render_bwd_det_kernel(int H, int W, int gx, const unsigned *__restrict__ tile_order, const uint2 *__restrict__ order_ranges,
                      const unsigned *__restrict__ n_tiles_nonempty, unsigned long long *__restrict__ work_next,
                      const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ ids_sorted,
                      const unsigned *__restrict__ goff, unsigned long long n_slots, const float *__restrict__ bg,
                      const float *__restrict__ final_T, const unsigned *__restrict__ n_contrib,
                      const float *__restrict__ gC, const float *__restrict__ gD, const float *__restrict__ gA, float *__restrict__ det_mom) {
    render_bwd_det_body<LAZY, false>(H, W, gx, tile_order, order_ranges, n_tiles_nonempty, work_next, rec_sorted, rec, ids_sorted, goff,
                                     n_slots, bg, final_T, n_contrib, gC, gD, gA, det_mom, nullptr);
}

template <bool LAZY>
__global__ void __launch_bounds__(kDetThreads)
render_views_bwd_det_kernel(const __grid_constant__ ViewTable vt, const unsigned *__restrict__ tile_order, const uint2 *__restrict__ order_ranges,
                            const unsigned *__restrict__ n_tiles_nonempty, unsigned long long *__restrict__ work_next,
                            const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ ids_sorted,
                            const unsigned *__restrict__ goff, unsigned long long n_slots, const float *__restrict__ bg,
                            const float *__restrict__ final_T, const unsigned *__restrict__ n_contrib,
                            const float *__restrict__ gC, const float *__restrict__ gD, const float *__restrict__ gA, float *__restrict__ det_mom) {
    render_bwd_det_body<LAZY, true>(0, 0, 0, tile_order, order_ranges, n_tiles_nonempty, work_next, rec_sorted, rec, ids_sorted, goff,
                                    n_slots, bg, final_T, n_contrib, gC, gD, gA, det_mom, &vt);
}

// DGR_RASTER_ABS_GRAD: the same two kernels with the absolute moments (separate kernels: the ones above stay as they were)
template <bool LAZY>
__global__ void __launch_bounds__(kDetThreads)
render_bwd_det_abs_kernel(int H, int W, int gx, const unsigned *__restrict__ tile_order, const uint2 *__restrict__ order_ranges,
                          const unsigned *__restrict__ n_tiles_nonempty, unsigned long long *__restrict__ work_next,
                          const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ ids_sorted,
                          const unsigned *__restrict__ goff, unsigned long long n_slots, const float *__restrict__ bg,
                          const float *__restrict__ final_T, const unsigned *__restrict__ n_contrib,
                          const float *__restrict__ gC, const float *__restrict__ gD, const float *__restrict__ gA, float *__restrict__ det_mom) {
    render_bwd_det_body<LAZY, false, true>(H, W, gx, tile_order, order_ranges, n_tiles_nonempty, work_next, rec_sorted, rec, ids_sorted, goff,
                                           n_slots, bg, final_T, n_contrib, gC, gD, gA, det_mom, nullptr);
}

template <bool LAZY>
__global__ void __launch_bounds__(kDetThreads)
render_views_bwd_det_abs_kernel(const __grid_constant__ ViewTable vt, const unsigned *__restrict__ tile_order, const uint2 *__restrict__ order_ranges,
                                const unsigned *__restrict__ n_tiles_nonempty, unsigned long long *__restrict__ work_next,
                                const Rec *__restrict__ rec_sorted, const Rec *__restrict__ rec, const unsigned *__restrict__ ids_sorted,
                                const unsigned *__restrict__ goff, unsigned long long n_slots, const float *__restrict__ bg,
                                const float *__restrict__ final_T, const unsigned *__restrict__ n_contrib,
                                const float *__restrict__ gC, const float *__restrict__ gD, const float *__restrict__ gA, float *__restrict__ det_mom) {
    render_bwd_det_body<LAZY, true, true>(0, 0, 0, tile_order, order_ranges, n_tiles_nonempty, work_next, rec_sorted, rec, ids_sorted, goff,
                                          n_slots, bg, final_T, n_contrib, gC, gD, gA, det_mom, &vt);
}

// One thread per record: the moments of its instance slots, summed in slot order (the row-major order of its tiles) -> grad_rec.
// Records that touch no tile keep the zero row of the backward's memset.  A record whose slots run past n_slots (the caller passed
// fewer instances than the forward binned) gets a NaN row: its gradients come out visibly wrong instead of silently short.
// ABS: also the absolute moments (floats 10 and 11).
template <bool ABS>
__device__ __forceinline__ void
det_moments_gather_body(long long R, const unsigned *__restrict__ touched, const unsigned *__restrict__ goff,
                        const float *__restrict__ det_mom, unsigned long long n_slots, float *__restrict__ grad_rec) {
    pdl_trigger();
    pdl_wait();                          // the instance moments of render_bwd_det
    const long long r = (long long)blockIdx.x * 256 + threadIdx.x;
    if (r >= R) return;
    const unsigned t = __ldg(touched + r) & kTouchedMask;
    if (t == 0) return;
    const unsigned long long o = __ldg(goff + r);
    float4 *dst = reinterpret_cast<float4 *>(grad_rec + (size_t)r * kGradRecFloats);
    if (o + t > n_slots) {
        const float nan = __int_as_float(0x7fffffff);
        dst[0] = make_float4(nan, nan, nan, nan); dst[1] = dst[0]; dst[2] = make_float4(nan, nan, ABS ? nan : 0.f, ABS ? nan : 0.f);
        return;
    }
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a, c = a;
    for (unsigned k = 0; k < t; k++) {
        const float4 *m = reinterpret_cast<const float4 *>(det_mom + (o + k) * kGradRecFloats);
        const float4 x = __ldcg(m), y = __ldcg(m + 1), z = __ldcg(m + 2);
        a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w;
        b.x += y.x; b.y += y.y; b.z += y.z; b.w += y.w;
        c.x += z.x; c.y += z.y;
        if constexpr (ABS) { c.z += z.z; c.w += z.w; }
    }
    dst[0] = a; dst[1] = b; dst[2] = c;
}

__global__ void __launch_bounds__(256)
det_moments_gather_kernel(long long R, const unsigned *__restrict__ touched, const unsigned *__restrict__ goff,
                          const float *__restrict__ det_mom, unsigned long long n_slots, float *__restrict__ grad_rec) {
    det_moments_gather_body<false>(R, touched, goff, det_mom, n_slots, grad_rec);
}

__global__ void __launch_bounds__(256)
det_moments_gather_abs_kernel(long long R, const unsigned *__restrict__ touched, const unsigned *__restrict__ goff,
                              const float *__restrict__ det_mom, unsigned long long n_slots, float *__restrict__ grad_rec) {
    det_moments_gather_body<true>(R, touched, goff, det_mom, n_slots, grad_rec);
}

}  // namespace dgr
