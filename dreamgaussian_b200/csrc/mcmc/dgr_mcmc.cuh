// dgr_mcmc.cuh — opt-in MCMC densification ("3D Gaussian Splatting as Markov Chain Monte Carlo", Kheradmand et al., NeurIPS 2024;
// gsplat's MCMCStrategy): dead Gaussians are moved onto live ones, the cloud grows by 5 % per refinement up to a cap, and
// near-transparent Gaussians get position noise every step.  Random draws come in as device tensors, so every kernel here is a
// pure function of its inputs that a float64 restatement on the host can reproduce.
//
//   mcmc_relocation_kernel      the relocation formula alone (gsplat's `relocation` op), float64 inside
//   mcmc_scan_local_kernel      per block: sampling weights, their block-local inclusive float64 prefix, the dead rows' local rank
//   mcmc_scan_blocks_kernel     one CTA: exclusive scan of the block totals
//   mcmc_scan_add_kernel        block offsets added: C_i = inclusive float64 prefix of the weights, dead_rank_i
//   mcmc_relocate_pick_kernel   dead row j-th in index order: smallest i with C_i > u_j C_last; integer-atomic pick counts
//   mcmc_relocate_write_kernel  ONE pass copying rows [0, P) of the six tensors and both Adam moments (dead rows: their source's)
//   mcmc_relocate_update_kernel the formula on the sources' and their copies' opacity and scaling (float64 inside)
//   mcmc_grow_pick_kernel       the same search over the output's opacities for each of the n_add draws
//   mcmc_grow_update_kernel     picked rows get the formula, their moments are zeroed
//   mcmc_append_kernel          row P + j = copy of picked row j, zero moments
//   mcmc_noise_kernel           xyz += scale g(o) R diag(s^2) R^T z, in place (every step)
// The scan is fixed-order (shuffles, then warps, then blocks), so the prefix sums, and with them the picks, are bit-reproducible;
// the only atomics are integer adds.  No host read-back: n_add is the caller's, u_relocate is sized P.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../../include/dgr_constants.h"

namespace dgr {

constexpr int kMcmcThreads = 256;
constexpr int kMcmcTensors = 6;           // xyz, f_dc, f_rest, opacity, scaling, rotation (DgrDensifyTensors order)

struct McmcTensors {
    const float *in[kMcmcTensors], *m_in[kMcmcTensors], *v_in[kMcmcTensors];
    float *out[kMcmcTensors], *m_out[kMcmcTensors], *v_out[kMcmcTensors];
    int width[kMcmcTensors];              // floats per row
};

__device__ __forceinline__ void mcmc_copy_row(float *dst, const float *src, int w) {
    for (int k = 0; k < w; k++) dst[k] = src[k];
}
__device__ __forceinline__ void mcmc_zero_row(float *dst, int w) {
    for (int k = 0; k < w; k++) dst[k] = 0.f;
}

// Relocated opacity o' = 1 - (1 - o)^(1/n) as -expm1(log1p(-o) / n) (no cancellation at small o or large n) and the scale factor
// o / D, D = sum_{m=1..n} C(n,m) (-1)^(m-1) o'^m / sqrt(m) (the hockey-stick form of the published double sum), both in float64:
// the sum alternates in sign and loses up to 7e-4 of its value in float32 at o = 1 - 2^-23, n = 51.  o = 0 has D = 0: factor 1.
__host__ __device__ __forceinline__ void mcmc_relocate(double o, int n, double &o_new, double &factor) {
    o_new = -expm1(log1p(-o) / (double)n);
    double c = 1.0, p = 1.0, D = 0.0;
    for (int m = 1; m <= n; m++) {
        c = c * (double)(n - m + 1) / (double)m;
        p *= o_new;
        const double t = c * p / sqrt((double)m);
        D += (m & 1) ? t : -t;
    }
    factor = D > 0.0 ? o / D : 1.0;
}

// o = sigmoid(raw) evaluated in float64 and rounded once: the weights a float64 host restatement computes alike
__device__ __forceinline__ float mcmc_opacity(float raw) { return (float)(1.0 / (1.0 + exp(-(double)raw))); }

__device__ __forceinline__ int mcmc_copies(int picked) { return min(1 + picked, DGR_MCMC_N_MAX); }

// Updated raw opacity and scaling of a row picked `picked` times: logit(clamp(o')) and scaling + log(o / D)
__device__ __forceinline__ void mcmc_update_row(float op_raw, const float *sc_raw, int picked, float min_opacity, float &op_out, float *sc_out) {
    double o_new, factor;
    const double o = (double)mcmc_opacity(op_raw);
    mcmc_relocate(o, mcmc_copies(picked), o_new, factor);
    const double oc = fmin(fmax(o_new, (double)min_opacity), DGR_MCMC_OPACITY_MAX);
    op_out = (float)log(oc / (1.0 - oc));
    const double ls = log(factor);
#pragma unroll
    for (int k = 0; k < 3; k++) sc_out[k] = (float)((double)sc_raw[k] + ls);
}

__global__ void __launch_bounds__(kMcmcThreads)
mcmc_relocation_kernel(int n, const float *__restrict__ opacity, const float *__restrict__ scale, const int *__restrict__ ratio,
                       float *__restrict__ new_opacity, float *__restrict__ new_scale) {
    const int i = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (i >= n) return;
    const int r = min(max(ratio[i], 1), DGR_MCMC_N_MAX);
    double o_new, factor;
    mcmc_relocate((double)opacity[i], r, o_new, factor);
    new_opacity[i] = (float)o_new;
#pragma unroll
    for (int k = 0; k < 3; k++) new_scale[3 * i + k] = (float)((double)scale[3 * i + k] * factor);
}

// scratch of dgr_mcmc_refine: [C f64 x P][dead_rank i32 x P][src_of i32 x P][picks i32 x P][grow_picks i32 x P][grow_src i32 x n_add]
// [block totals f64 x nblk][block dead counts i32 x nblk][block offsets f64 x nblk][block dead offsets i32 x nblk][n_dead i32]
struct McmcLayout {
    size_t off_C, off_rank, off_src, off_picks, off_gpicks, off_gsrc, off_bsum, off_bdead, off_boff, off_bdoff, off_ndead, total;
    int nblk;
    __host__ McmcLayout(int P, int n_add) {
        const size_t Pn = P > 0 ? (size_t)P : 1, An = n_add > 0 ? (size_t)n_add : 1;
        nblk = (int)((Pn + kMcmcThreads - 1) / kMcmcThreads);
        auto up = [](size_t o) { return (o + 255) / 256 * 256; };
        size_t o = 0;
        off_C = o;      o = up(o + 8 * Pn);
        off_rank = o;   o = up(o + 4 * Pn);
        off_src = o;    o = up(o + 4 * Pn);
        off_picks = o;  o = up(o + 4 * Pn);
        off_gpicks = o; o = up(o + 4 * Pn);
        off_gsrc = o;   o = up(o + 4 * An);
        off_bsum = o;   o = up(o + 8 * (size_t)nblk);
        off_bdead = o;  o = up(o + 4 * (size_t)nblk);
        off_boff = o;   o = up(o + 8 * (size_t)nblk);
        off_bdoff = o;  o = up(o + 4 * (size_t)nblk);
        off_ndead = o;  o = up(o + 4);
        total = o;
    }
};

// inclusive scan of (w, d) over the CTA in thread order; fixed order, so the same inputs give the same bits
__device__ __forceinline__ void mcmc_block_scan(double &w, int &d) {
    __shared__ double s_w[kMcmcThreads / 32];
    __shared__ int s_d[kMcmcThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double nw = __shfl_up_sync(0xffffffffu, w, o);
        const int nd = __shfl_up_sync(0xffffffffu, d, o);
        if (lane >= o) { w += nw; d += nd; }
    }
    if (lane == 31) { s_w[warp] = w; s_d[warp] = d; }
    __syncthreads();
    if (warp == 0) {
        double x = lane < kMcmcThreads / 32 ? s_w[lane] : 0.0;
        int y = lane < kMcmcThreads / 32 ? s_d[lane] : 0;
#pragma unroll
        for (int o = 1; o < kMcmcThreads / 32; o <<= 1) {
            const double nx = __shfl_up_sync(0xffffffffu, x, o);
            const int ny = __shfl_up_sync(0xffffffffu, y, o);
            if (lane >= o) { x += nx; y += ny; }
        }
        const double xe = __shfl_up_sync(0xffffffffu, x, 1);        // exclusive by shifting, not by subtracting (exact)
        const int ye = __shfl_up_sync(0xffffffffu, y, 1);
        if (lane < kMcmcThreads / 32) { s_w[lane] = lane ? xe : 0.0; s_d[lane] = lane ? ye : 0; }
    }
    __syncthreads();
    if (warp > 0) { w += s_w[warp]; d += s_d[warp]; }
}

// grow = 0 (relocation): weight o for live rows (o > min_opacity), 0 and a dead flag for the rest.  grow = 1: weight o for every row.
__global__ void __launch_bounds__(kMcmcThreads)
mcmc_scan_local_kernel(int P, const float *__restrict__ opacity_raw, float min_opacity, int grow, double *__restrict__ C,
                       int *__restrict__ dead_rank, double *__restrict__ bsum, int *__restrict__ bdead) {
    const int i = blockIdx.x * kMcmcThreads + threadIdx.x;
    double w = 0.0;
    int d = 0;
    if (i < P) {
        const float o = mcmc_opacity(opacity_raw[i]);
        const bool dead = !grow && o <= min_opacity;
        w = dead ? 0.0 : (double)o;
        d = dead ? 1 : 0;
    }
    const int d_own = d;
    mcmc_block_scan(w, d);
    if (i < P) { C[i] = w; dead_rank[i] = d - d_own; }
    if (threadIdx.x == kMcmcThreads - 1) { bsum[blockIdx.x] = w; bdead[blockIdx.x] = d; }
}

// one CTA: exclusive scan over the blocks (the pattern of densify_offsets_kernel), n_dead = the dead rows in all
__global__ void __launch_bounds__(kMcmcThreads)
mcmc_scan_blocks_kernel(int nblk, const double *__restrict__ bsum, const int *__restrict__ bdead, double *__restrict__ boff,
                        int *__restrict__ bdoff, int *__restrict__ n_dead) {
    __shared__ double s_carry_w;
    __shared__ int s_carry_d;
    if (threadIdx.x == 0) { s_carry_w = 0.0; s_carry_d = 0; }
    __syncthreads();
    for (int base = 0; base < nblk; base += kMcmcThreads) {
        const int b = base + threadIdx.x;
        const double v = b < nblk ? bsum[b] : 0.0;
        const int vd = b < nblk ? bdead[b] : 0;
        double w = v;
        int d = vd;
        mcmc_block_scan(w, d);
        // exclusive = the previous thread's inclusive value
        __shared__ double s_inc[kMcmcThreads];
        __shared__ int s_incd[kMcmcThreads];
        s_inc[threadIdx.x] = w; s_incd[threadIdx.x] = d;
        __syncthreads();
        const double cw = s_carry_w;
        const int cd = s_carry_d;
        if (b < nblk) {
            boff[b] = threadIdx.x ? cw + s_inc[threadIdx.x - 1] : cw;
            bdoff[b] = threadIdx.x ? cd + s_incd[threadIdx.x - 1] : cd;
        }
        __syncthreads();
        if (threadIdx.x == 0) { s_carry_w = cw + s_inc[kMcmcThreads - 1]; s_carry_d = cd + s_incd[kMcmcThreads - 1]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) *n_dead = s_carry_d;
}

__global__ void __launch_bounds__(kMcmcThreads)
mcmc_scan_add_kernel(int P, const double *__restrict__ boff, const int *__restrict__ bdoff, double *__restrict__ C, int *__restrict__ dead_rank) {
    const int i = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (i >= P) return;
    C[i] = boff[blockIdx.x] + C[i];
    dead_rank[i] += bdoff[blockIdx.x];
}

// smallest i with C[i] > t, or P when none
__device__ __forceinline__ int mcmc_search(const double *__restrict__ C, int P, double t) {
    int lo = 0, hi = P;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (C[mid] > t) hi = mid; else lo = mid + 1;
    }
    return lo;
}

// one thread per row: a dead row picks its source; src_of = -1 for every other row.  When no row is alive (C_last = 0) nothing moves.
__global__ void __launch_bounds__(kMcmcThreads)
mcmc_relocate_pick_kernel(int P, const float *__restrict__ opacity_raw, float min_opacity, const double *__restrict__ C,
                          const int *__restrict__ dead_rank, const int *__restrict__ n_dead, const float *__restrict__ u,
                          int *__restrict__ src_of, int *__restrict__ picks, int *__restrict__ n_relocated) {
    const int i = blockIdx.x * kMcmcThreads + threadIdx.x;
    const double total = C[P - 1];
    if (i == 0 && n_relocated) *n_relocated = total > 0.0 ? *n_dead : 0;
    if (i >= P) return;
    int s = -1;
    if (total > 0.0 && mcmc_opacity(opacity_raw[i]) <= min_opacity) {
        s = mcmc_search(C, P, (double)u[dead_rank[i]] * total);
        if (s >= P) {                                   // rounding left no C_i above the draw: the last live row
            s = P - 1;
            while (s > 0 && !(mcmc_opacity(opacity_raw[s]) > min_opacity)) s--;
        }
        atomicAdd(&picks[s], 1);
    }
    src_of[i] = s;
}

// Row i takes row r = (dead ? its source : i) in all six tensors.  A source (picks > 0) gets zero moments; a relocated dead row keeps
// its own (the published code leaves them alone).  The formula is the next kernel's: with its float64 calls in this one, the copy
// loops' live values spilled.
__global__ void __launch_bounds__(kMcmcThreads)
mcmc_relocate_write_kernel(int P, McmcTensors T, const int *__restrict__ src_of, const int *__restrict__ picks) {
    const int i = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (i >= P) return;
    const int s = src_of[i];
    const int r = s >= 0 ? s : i;
    const bool zero_m = s < 0 && picks[i] > 0;
#pragma unroll
    for (int t = 0; t < kMcmcTensors; t++) {
        const int w = T.width[t];
        mcmc_copy_row(T.out[t] + (size_t)i * w, T.in[t] + (size_t)r * w, w);
        if (zero_m) {
            mcmc_zero_row(T.m_out[t] + (size_t)i * w, w);
            mcmc_zero_row(T.v_out[t] + (size_t)i * w, w);
        } else {
            mcmc_copy_row(T.m_out[t] + (size_t)i * w, T.m_in[t] + (size_t)i * w, w);
            mcmc_copy_row(T.v_out[t] + (size_t)i * w, T.v_in[t] + (size_t)i * w, w);
        }
    }
}

// the formula for every output row whose row r was picked: the source itself and each dead row that copied it
__global__ void __launch_bounds__(kMcmcThreads)
mcmc_relocate_update_kernel(int P, const float *__restrict__ op_in, const float *__restrict__ sc_in, const int *__restrict__ src_of,
                            const int *__restrict__ picks, float min_opacity, float *__restrict__ op_out, float *__restrict__ sc_out) {
    const int i = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (i >= P) return;
    const int s = src_of[i];
    const int r = s >= 0 ? s : i;
    const int pr = picks[r];
    if (pr == 0) return;
    float op, sc[3];
    mcmc_update_row(op_in[r], sc_in + (size_t)r * 3, pr, min_opacity, op, sc);
    op_out[i] = op;
    sc_out[3 * (size_t)i] = sc[0]; sc_out[3 * (size_t)i + 1] = sc[1]; sc_out[3 * (size_t)i + 2] = sc[2];
}

// one thread per added row: the row it copies (every row eligible; the last row when rounding leaves no C_i above the draw)
__global__ void __launch_bounds__(kMcmcThreads)
mcmc_grow_pick_kernel(int P, int n_add, const double *__restrict__ C, const float *__restrict__ u, int *__restrict__ grow_src,
                      int *__restrict__ grow_picks) {
    const int j = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (j >= n_add) return;
    const int s = min(mcmc_search(C, P, (double)u[j] * C[P - 1]), P - 1);
    grow_src[j] = s;
    atomicAdd(&grow_picks[s], 1);
}

__global__ void __launch_bounds__(kMcmcThreads)
mcmc_grow_update_kernel(int P, McmcTensors T, const int *__restrict__ grow_picks, float min_opacity) {
    const int i = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (i >= P) return;
    const int pr = grow_picks[i];
    if (pr == 0) return;
    float op, sc[3];
    float *srow = T.out[4] + (size_t)i * 3;
    mcmc_update_row(T.out[3][i], srow, pr, min_opacity, op, sc);
    T.out[3][i] = op;
    srow[0] = sc[0]; srow[1] = sc[1]; srow[2] = sc[2];
#pragma unroll
    for (int t = 0; t < kMcmcTensors; t++) {
        const int w = T.width[t];
        mcmc_zero_row(T.m_out[t] + (size_t)i * w, w);
        mcmc_zero_row(T.v_out[t] + (size_t)i * w, w);
    }
}

__global__ void __launch_bounds__(kMcmcThreads)
mcmc_append_kernel(int P, int n_add, McmcTensors T, const int *__restrict__ grow_src) {
    const int j = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (j >= n_add) return;
    const size_t d = (size_t)P + j, s = (size_t)grow_src[j];
#pragma unroll
    for (int t = 0; t < kMcmcTensors; t++) {
        const int w = T.width[t];
        mcmc_copy_row(T.out[t] + d * w, T.out[t] + s * w, w);
        mcmc_zero_row(T.m_out[t] + d * w, w);
        mcmc_zero_row(T.v_out[t] + d * w, w);
    }
}

// xyz += scale * g(o) * R diag(s^2) R^T z, g(o) = 1 / (1 + exp(-k ((1 - o) - x0))): about 0.5 at o = 0.005, below 1e-20 above 0.5
__global__ void __launch_bounds__(kMcmcThreads)
mcmc_noise_kernel(int P, float *__restrict__ xyz, const float *__restrict__ opacity_raw, const float *__restrict__ scaling_raw,
                  const float *__restrict__ rotation_raw, const float *__restrict__ z, float scale) {
    const int i = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (i >= P) return;
    const float o = 1.f / (1.f + expf(-opacity_raw[i]));
    const float g = 1.f / (1.f + expf(-DGR_MCMC_NOISE_K * ((1.f - o) - DGR_MCMC_NOISE_X0)));
    const float *q = rotation_raw + 4 * (size_t)i;
    const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const float r = q[0] / qn, x = q[1] / qn, y = q[2] / qn, zq = q[3] / qn;
    const float R00 = 1.f - 2.f * (y * y + zq * zq), R01 = 2.f * (x * y - r * zq), R02 = 2.f * (x * zq + r * y);
    const float R10 = 2.f * (x * y + r * zq), R11 = 1.f - 2.f * (x * x + zq * zq), R12 = 2.f * (y * zq - r * x);
    const float R20 = 2.f * (x * zq - r * y), R21 = 2.f * (y * zq + r * x), R22 = 1.f - 2.f * (x * x + y * y);
    const size_t b = 3 * (size_t)i;
    const float s0 = expf(scaling_raw[b]), s1 = expf(scaling_raw[b + 1]), s2 = expf(scaling_raw[b + 2]);
    const float z0 = z[b], z1 = z[b + 1], z2 = z[b + 2];
    const float f = scale * g;
    const float a0 = (R00 * z0 + R10 * z1 + R20 * z2) * s0 * s0 * f;         // diag(s^2) R^T z, times scale g
    const float a1 = (R01 * z0 + R11 * z1 + R21 * z2) * s1 * s1 * f;
    const float a2 = (R02 * z0 + R12 * z1 + R22 * z2) * s2 * s2 * f;
    xyz[b] += R00 * a0 + R01 * a1 + R02 * a2;
    xyz[b + 1] += R10 * a0 + R11 * a1 + R12 * a2;
    xyz[b + 2] += R20 * a0 + R21 * a1 + R22 * a2;
}

}  // namespace dgr
