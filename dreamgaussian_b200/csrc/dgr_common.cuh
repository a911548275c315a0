// dgr_common.cuh — shared definitions of the sm_90a rasterizer kernels: scratch layouts, PTX wrappers
// (mbarrier + 1-D bulk TMA), small math helpers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/dgr_constants.h"

namespace dgr {

constexpr int kTile = DGR_TILE;            // 16 x 16 pixel tiles
constexpr int kTileThreads = 256;          // one thread per pixel
constexpr int kPreThreads = 256;           // per-Gaussian kernels
constexpr float kLog2e = 1.4426950408889634f;

// ---------------------------------------------------------------------------------------------------------
// Per-Gaussian record produced by the forward preprocess and consumed (through the depth-sorted, per-tile
// contiguous copy) by both render kernels.  48 bytes = 3 x float4 so a tile's instance range is one contiguous,
// 16-byte aligned block that a single cp.async.bulk (TMA) moves into shared memory.
//   q0 = { mean_px.x, mean_px.y, -0.5 conicA log2e, -conicB log2e }
//   q1 = { -0.5 conicC log2e, opacity, depth (view z), aabb_x = x0 | x1 << 16 }
//   q2 = { r, g, b, aabb_y = y0 | y1 << 16 }
// The conic is stored as the coefficients of power*log2(e), so power2 = dx (q0.z dx + q0.w dy) + q1.x dy^2 is
// 5 instructions and alpha = o * ex2(power2) needs no extra multiply.  aabb = inclusive pixel
// bounds of { pixels whose 16x16 tile is in the 3-sigma tile rect } ∩ { bounding box of alpha >= 1/255 },
// i.e. a conservative superset of the pixels this Gaussian can contribute to under the reference's rules.
// ---------------------------------------------------------------------------------------------------------
struct __align__(16) Rec { float4 q0, q1, q2; };
static_assert(sizeof(Rec) == 48, "Rec must be 48 bytes");

// Per-Gaussian reduction target of the backward render: 12 floats (3 x float4)
//   0 m0 = sum u            1 m1 = sum u dx        2 m2 = sum u dy
//   3 m3 = sum u dx^2       4 m4 = sum u dx dy     5 m5 = sum u dy^2
//   6..8 sum w * dL/dC[rgb] 9 sum w * dL/dD        10, 11 unused
// with u = o * G * dL/dalpha, w = alpha * T, d = mean_px - pixel.
constexpr int kGradRecFloats = 12;
static_assert(kGradRecFloats * 4 % 16 == 0, "moment rows stay 16-byte aligned for the vector reductions of the backward render");

struct GeomHeader {
    unsigned long long n_inst;     // total tile instances of this frame (written by the tile scan)
    unsigned long long n_big;      // tiles whose population exceeds the per-tile sort CTA (need the big-tile sorter)
    unsigned int pad[12];
};
static_assert(sizeof(GeomHeader) == 64, "GeomHeader");

__host__ __device__ inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Gaussians per block of the preprocess / emit kernels = kPreThreads * iters.  Every block keeps a per-tile histogram in
// shared memory, reserves its run of every touched tile with one global atomic and leaves the run starts in one row of a
// [blocks x tiles] matrix: a few thousand Gaussians per block keep that traffic small for big clouds while small clouds
// still spread over all SMs (about 4 blocks per SM at least).
__host__ __device__ inline int choose_gpb_iters(int P, int tiles) {
    long long k = (long long)(P > 0 ? P : 1) / ((long long)kPreThreads * 600);
    if (k < 1) k = 1;
    if (k > 16) k = 16;
    // ... and the run matrix stays below 64 MB
    const long long blocks1 = ((long long)(P > 0 ? P : 1) + kPreThreads - 1) / kPreThreads;
    const long long bytes = blocks1 * (long long)(tiles > 0 ? tiles : 1) * 4;
    const long long k2 = (bytes + (64ll << 20) - 1) / (64ll << 20);
    if (k2 > k) k = k2;
    if (k > 64) k = 64;
    return (int)k;
}

// geom scratch: [header 256][rec 48 x P][touched u32 x P][backward work counter 256][moments 48 x P (backward)]
//               [run matrix u32 x blocks x tiles: where block b's instances start inside tile t's range]
//               (the backward zeroes counter + moments with ONE memset)
// A batch of V views of one cloud (dgr_views_*) keeps V x P records (record r = v P + g) and V x tiles-per-view tiles
// (global tile v T + local tile); the blocks still cover the P Gaussians, so the run matrix is blocks x V T.
// Views of different sizes (dgr_views_mixed_*): the tiles are the batch's total, sum over v of tiles_v (GeomLayout::batch).
struct GeomLayout {
    size_t off_rec, off_touched, off_bwdwork, off_gradrec, off_runs, total;
    int tiles, iters, nblocks;
    __host__ __device__ GeomLayout(int P, int H, int W, int V = 1) {
        int t = ((W + kTile - 1) / kTile) * ((H + kTile - 1) / kTile);
        if (t < 1) t = 1;
        init(P, t * V, V);
    }
    __host__ __device__ static GeomLayout batch(int P, int tiles_total, int V) { GeomLayout L; L.init(P, tiles_total, V); return L; }
  private:
    __host__ __device__ GeomLayout() {}
    __host__ __device__ void init(int P, int tiles_total, int V) {
        size_t Pn = P > 0 ? (size_t)P : 1;
        const size_t Rn = Pn * (size_t)V;
        tiles = tiles_total;
        iters = choose_gpb_iters(P, tiles);
        nblocks = (int)((Pn + (size_t)kPreThreads * iters - 1) / ((size_t)kPreThreads * iters));
        size_t o = 256;
        off_rec = o;     o = align_up(o + Rn * sizeof(Rec), 256);
        off_touched = o; o = align_up(o + Rn * 4, 256);
        off_bwdwork = o; o += 256;
        off_gradrec = o; o = align_up(o + Rn * kGradRecFloats * 4, 256);
        off_runs = o;    o = align_up(o + (size_t)nblocks * tiles * 4, 256);
        total = o;
    }
};

constexpr int kCostClasses = 32;         // log-scale classes of the measured forward cost of a backward work item

// image scratch: [work 256][tile_count u32 x tiles][ranges uint2 x tiles][tile_order u32 x tiles]
//                [big_list u32 x tiles][n_contrib u32 x HW][final_T f32 x HW]
//                ... [cost accumulators u32 x 8 tiles] ... [cost-class item lists u32 x 32 x 8 tiles]
// (work, tile_count and the cost accumulators are adjacent: the forward zeroes them with ONE memset before the preprocess kernel)
// V views (dgr_views_*): every per-tile array covers V x tiles-per-view tiles and n_contrib / final_T are [V, H, W].
// Views of different sizes (ImageLayout::batch): the per-tile arrays cover the batch's total tiles and the pixel state its total
// pixels, view v's [H_v, W_v] block after those of views 0 .. v-1 (gx, gy are then 0).
struct ImageLayout {
    size_t off_ranges, off_oranges, off_count, off_cost, off_order, off_biglist, off_work, off_ncontrib, off_finalT, off_clsitems, total;
    int gx, gy;
    __host__ __device__ ImageLayout(int H, int W, int V = 1) {
        gx = (W + kTile - 1) / kTile; gy = (H + kTile - 1) / kTile;
        size_t tiles = (size_t)gx * gy; if (tiles < 1) tiles = 1;
        size_t hw = (size_t)H * W; if (hw < 1) hw = 1;
        init(tiles * (size_t)V, hw * (size_t)V);
    }
    __host__ __device__ static ImageLayout batch(size_t tiles_total, size_t pixels_total) {
        ImageLayout L; L.gx = 0; L.gy = 0; L.init(tiles_total, pixels_total); return L;
    }
  private:
    __host__ __device__ ImageLayout() {}
    __host__ __device__ void init(size_t tiles, size_t hw) {
        size_t o = 0;
        off_work = o;     o = align_up(o + 256, 256);
        off_count = o;    o = align_up(o + tiles * 4, 256);
        off_cost = o;     o = align_up(o + tiles * 8 * 4, 256);    // measured cost of every backward work item (zeroed with the totals)
        off_ranges = o;   o = align_up(o + tiles * 8, 256);
        off_oranges = o;  o = align_up(o + tiles * 8, 256);      // the ranges again, in issue order (sort kernel)
        off_order = o;    o = align_up(o + tiles * 4, 256);
        off_biglist = o;  o = align_up(o + tiles * 4, 256);
        off_ncontrib = o; o = align_up(o + hw * 4, 256);
        off_finalT = o;   o = align_up(o + hw * 4, 256);
        off_clsitems = o; o = align_up(o + (size_t)kCostClasses * tiles * 8 * 4, 256);   // backward work items grouped by measured cost class
        total = o;
    }
};

// Image sizes of the views of a batch (dgr_views_*, dgr_views_mixed_*), handed to the five batched kernels BY VALUE as a kernel
// parameter (1.3 KB, read through the constant bank; no upload).  View v has H[v] x W[v] pixels and gx[v] tile columns; its tiles
// are the global tiles tile_off[v] .. tile_off[v + 1] - 1 (row-major within the view) and its pixel state / images start at
// pixel pix_off[v] (colour: float 3 pix_off[v], then [3, H_v, W_v]).  tile_off[V .. kMaxViews] = the batch's total tiles, so
// view_of_tile needs no bound.  Same-size batches are the uniform table: tile_off[v] = v T, pix_off[v] = v H W.
constexpr int kMaxViews = 64;
struct ViewTable {
    int tile_off[kMaxViews + 1];
    int pix_off[kMaxViews];
    int H[kMaxViews], W[kMaxViews], gx[kMaxViews];
};

// the view a global tile belongs to: binary search over tile_off (6 steps for 64 views)
__device__ __forceinline__ int view_of_tile(const ViewTable &vt, int tile) {
    int v = 0;
#pragma unroll
    for (int s = kMaxViews / 2; s > 0; s >>= 1)
        if (vt.tile_off[v + s] <= tile) v += s;
    return v;
}

// ------------------------------------------------ PTX wrappers ------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Multi-GPU (view-sharded, SURVEY.md §8e): the per-Gaussian backward can write the gradient rows of Gaussians OWNED by another
// rank straight into that rank's staging area over NVLink (dgr_backward.cuh, dgr_collective.cuh).  delta[o] = distance in
// floats from a local gradient address to the same element of this rank's slot at owner o (0 for o = this rank); Gaussian g
// belongs to owner g / per (per is a multiple of the kernel's block size, so a block has one owner).  per = 0: off.
constexpr int kMaxPeers = 16;
struct PeerPush { long long delta[kMaxPeers]; int per; };

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// 1-D bulk TMA: global -> shared, completion signalled on an mbarrier (SASS: UBLKCP).  16-byte aligned, size % 16 == 0.
__device__ __forceinline__ void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// Programmatic dependent launch (PDL): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start
// while its predecessor in the stream is still running; pdl_wait() blocks until the predecessor grid has completed and its
// memory is visible, pdl_trigger() lets the successor's CTAs become resident as soon as SM resources free up (they then sit in
// pdl_wait()).  Both are no-ops for kernels launched the ordinary way.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ float ex2_approx(float x) {
    float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
}
// index of the most significant set bit (x != 0): one FLO instead of the FLO + two integer ops of 31 - __clz(x)
__device__ __forceinline__ int bfind_u32(unsigned x) { int r; asm("bfind.u32 %0, %1;" : "=r"(r) : "r"(x)); return r; }
__device__ __forceinline__ void red_add_f32(float *addr, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
// sm_90 vector reductions: one L2 operation adds 2 / 4 consecutive floats (SASS: REDG.E.ADD.F32x2 / F32x4).  Each float
// receives exactly the addition the scalar form would make; addr must be 8 / 16-byte aligned.
__device__ __forceinline__ void red_add_v2_f32(float *addr, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void red_add_v4_f32(float *addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ float4 ldg_f4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }
// L2 residency control for the record gather of the per-tile sort: the per-Gaussian record array (48 B x P) is re-read N/P
// times at random and should stay in L2, the sorted copy (48 B x N) is written once and read once by the render kernels.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p;
}
__device__ __forceinline__ float4 ldg_f4_hint(const float4 *p, uint64_t pol) {
    float4 v;
    asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void stg_f4_hint(float4 *p, const float4 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ float lg2_approx(float x) {
    float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y;
}

// power*log2(e) below which a Gaussian of opacity o cannot reach alpha = 1/255 (minus a safety margin of 1% in alpha)
__device__ __forceinline__ float alpha_threshold_power2(float opacity) { return -7.9943534f - lg2_approx(opacity) - 0.015f; }

// Conservative exact test: can ANY point of the pixel rectangle [x0,x1] x [y0,y1] reach power2 >= thr2 for the Gaussian
// with centre (cx, cy) and power2(dx, dy) = nA dx^2 + nB dx dy + nC dy^2 (nA, nC < 0, negative definite)?
// The maximiser of a concave quadratic over a box is the centre if it lies inside, otherwise it lies on one of the (at most
// two) edges facing the centre, where it is the clamped 1-D maximiser.
__device__ __forceinline__ bool ellipse_hits_rect(float cx, float cy, float nA, float nB, float nC, float thr2,
                                                  float x0, float x1, float y0, float y1) {
    const float xe = fminf(fmaxf(cx, x0), x1), ye = fminf(fmaxf(cy, y0), y1);
    const float dxe = cx - xe, dye = cy - ye;
    if (dxe == 0.f && dye == 0.f) return true;
    float best = -3.0e38f;
    if (dxe != 0.f) {
        float dy = -0.5f * nB * dxe * rcp_approx(nC);
        dy = fminf(fmaxf(dy, cy - y1), cy - y0);
        best = nA * dxe * dxe + nB * dxe * dy + nC * dy * dy;
    }
    if (dye != 0.f) {
        float dx = -0.5f * nB * dye * rcp_approx(nA);
        dx = fminf(fmaxf(dx, cx - x1), cx - x0);
        best = fmaxf(best, nA * dx * dx + nB * dx * dye + nC * dye * dye);
    }
    return best >= thr2;
}

// The tiles a Gaussian is binned into: those of its opacity-aware pixel AABB (which already carries the reference's
// 3-sigma tile-rect clip).  Used — with the SAME packed record values — by the preprocess histogram and by the emit kernel,
// so both make identical decisions.  (The exact ellipse test is applied later, per warp sub-tile, in the render kernels:
// it costs more in these two latency-bound per-Gaussian loops than the ~8% of instances it removes.)
template <class F>
__device__ __forceinline__ void for_each_touched_tile(unsigned ax, unsigned ay, int gx, F f) {
    const int bx0 = (int)(ax & 0xffffu), bx1 = (int)(ax >> 16), by0 = (int)(ay & 0xffffu), by1 = (int)(ay >> 16);
    if (bx0 > bx1 || by0 > by1) return;
    for (int ty = by0 >> 4; ty <= (by1 >> 4); ty++)
        for (int tx = bx0 >> 4; tx <= (bx1 >> 4); tx++) f(ty * gx + tx);
}

}  // namespace dgr
