// dgr_densify.cuh — SURVEY.md §8 row f2: the reference's densification as stream compaction.
//
// /root/reference/gs_renderer.py:586-609 `densify_and_prune` = densify_and_clone (:582-600 -> densification_postfix :515-552)
// + densify_and_split (:555-580, which appends 2 children per selected point and then prunes the selected originals)
// + prune_points (:509-513) with the opacity / world-size mask (:601-607).  In the reference that is ~30 boolean-mask
// indexing and torch.cat calls over the six parameter tensors and both Adam moments (optimizer-state surgery :464-552).
// All of it is a pure function of per-point decisions, so the final point order is known up front:
//     [ originals that are neither split nor pruned ] ++ [ surviving clones ] ++ [ first children ] ++ [ second children ]
// (boolean-mask indexing and torch.cat keep the relative order; a clone copies its original's opacity and scaling, so it
// survives the final prune exactly when its original does; children carry log(s / 1.6) as scaling).
//   densify_classify_kernel   per-point class bits + per-block counts of the four output streams
//   densify_offsets_kernel    one CTA: block offsets of the four streams, totals (copied to the host: the new point count)
//   densify_apply_kernel      block-level ranks -> destination rows; copies / creates the rows of the six tensors and both
//                             Adam moments (zero for new points) in ONE pass; split children are sampled and rotated here.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dgr {

constexpr int kDensifyThreads = 256;
constexpr int kDensifyTensors = 6;          // xyz, f_dc, f_rest, opacity, scaling, rotation  (the order of GROUPS in stage1.py)

struct DensifyParams {
    float grad_threshold;      // max_grad
    float dense_extent;        // percent_dense * scene_extent: clone below or at, split above
    float min_opacity;
    float max_world;           // 0.1 * extent, used when use_world != 0 (the reference's `if max_screen_size:`)
    int use_world;
};

struct DensifyTensors {
    const float *in[kDensifyTensors], *m_in[kDensifyTensors], *v_in[kDensifyTensors];
    float *out[kDensifyTensors], *m_out[kDensifyTensors], *v_out[kDensifyTensors];
    int width[kDensifyTensors];     // floats per point
};

enum : unsigned { kKeep = 1u, kClone = 2u, kSplit = 4u, kChild = 8u };

// scratch: [class u8 x P (padded to 256)][block counts u32 x nblk x 4][block offsets u32 x nblk x 4][totals u32 x 4]
struct DensifyLayout {
    size_t off_class, off_counts, off_offsets, off_totals, total;
    int nblk;
    __host__ explicit DensifyLayout(int P) {
        const size_t Pn = P > 0 ? (size_t)P : 1;
        nblk = (int)((Pn + kDensifyThreads - 1) / kDensifyThreads);
        size_t o = 0;
        off_class = o;   o = (o + Pn + 255) / 256 * 256;
        off_counts = o;  o += (size_t)nblk * 16;
        off_offsets = o; o += (size_t)nblk * 16;
        off_totals = o;  o += 256;
        total = o;
    }
};

// ABS (dgr_densify_plan_ex): AbsGS's rule (Ye et al., 2024) — clone by the default statistic as above, split by the absolute one,
// accum_abs / denom >= abs_threshold (NaN -> 0 likewise).
template <bool ABS = false>
__device__ __forceinline__ unsigned densify_class(int i, const float *accum, const float *denom, const float *opacity_raw,
                                                  const float *scaling_raw, const DensifyParams &prm, const float *accum_abs = nullptr,
                                                  float abs_threshold = 0.f) {
    float g = accum[i] / denom[i];                         // grads = xyz_gradient_accum / denom; grads[isnan] = 0 (:593-594)
    if (g != g) g = 0.f;
    const float s0 = expf(scaling_raw[3 * i]), s1 = expf(scaling_raw[3 * i + 1]), s2 = expf(scaling_raw[3 * i + 2]);
    const float smax = fmaxf(s0, fmaxf(s1, s2));
    const bool clone = (fabsf(g) >= prm.grad_threshold) && (smax <= prm.dense_extent);           // :583-585
    bool split = (g >= prm.grad_threshold) && (smax > prm.dense_extent);                         // :558-562
    if constexpr (ABS) {
        float ga = accum_abs[i] / denom[i];
        if (ga != ga) ga = 0.f;
        split = (ga >= abs_threshold) && (smax > prm.dense_extent);
    }
    const float o = 1.f / (1.f + expf(-opacity_raw[i]));
    const bool low = o < prm.min_opacity;                                                        // :601
    const bool prune_self = low || (prm.use_world && smax > prm.max_world);                      // :602-605 (max_radii2D was just zeroed: never)
    // children: scaling = log(s / (0.8 * 2)) (:569); what the final prune reads back is exp of that
    const float c0 = expf(logf(s0 / 1.6f)), c1 = expf(logf(s1 / 1.6f)), c2 = expf(logf(s2 / 1.6f));
    const bool prune_child = low || (prm.use_world && fmaxf(c0, fmaxf(c1, c2)) > prm.max_world);
    unsigned c = 0;
    if (!split && !prune_self) c |= kKeep;
    if (clone && !prune_self) c |= kClone;
    if (split) c |= kSplit;
    if (split && !prune_child) c |= kChild;
    return c;
}

__global__ void __launch_bounds__(kDensifyThreads)
densify_classify_kernel(int P, const float *__restrict__ accum, const float *__restrict__ denom, const float *__restrict__ opacity_raw,
                        const float *__restrict__ scaling_raw, DensifyParams prm, unsigned char *__restrict__ cls,
                        unsigned *__restrict__ block_counts) {
    __shared__ unsigned s_cnt[4];
    if (threadIdx.x < 4) s_cnt[threadIdx.x] = 0u;
    __syncthreads();
    const int i = blockIdx.x * kDensifyThreads + threadIdx.x;
    unsigned c = 0;
    if (i < P) { c = densify_class(i, accum, denom, opacity_raw, scaling_raw, prm); cls[i] = (unsigned char)c; }
#pragma unroll
    for (int b = 0; b < 4; b++) {
        const unsigned m = __ballot_sync(0xffffffffu, (c >> b) & 1u);
        if ((threadIdx.x & 31) == 0 && m) atomicAdd(&s_cnt[b], (unsigned)__popc(m));
    }
    __syncthreads();
    if (threadIdx.x < 4) block_counts[blockIdx.x * 4 + threadIdx.x] = s_cnt[threadIdx.x];
}

__global__ void __launch_bounds__(kDensifyThreads)
densify_classify_abs_kernel(int P, const float *__restrict__ accum, const float *__restrict__ accum_abs, const float *__restrict__ denom,
                            const float *__restrict__ opacity_raw, const float *__restrict__ scaling_raw, DensifyParams prm,
                            float abs_threshold, unsigned char *__restrict__ cls, unsigned *__restrict__ block_counts) {
    __shared__ unsigned s_cnt[4];
    if (threadIdx.x < 4) s_cnt[threadIdx.x] = 0u;
    __syncthreads();
    const int i = blockIdx.x * kDensifyThreads + threadIdx.x;
    unsigned c = 0;
    if (i < P) { c = densify_class<true>(i, accum, denom, opacity_raw, scaling_raw, prm, accum_abs, abs_threshold); cls[i] = (unsigned char)c; }
#pragma unroll
    for (int b = 0; b < 4; b++) {
        const unsigned m = __ballot_sync(0xffffffffu, (c >> b) & 1u);
        if ((threadIdx.x & 31) == 0 && m) atomicAdd(&s_cnt[b], (unsigned)__popc(m));
    }
    __syncthreads();
    if (threadIdx.x < 4) block_counts[blockIdx.x * 4 + threadIdx.x] = s_cnt[threadIdx.x];
}

// one CTA of 1024 threads: exclusive scan over the blocks of each of the four streams
__global__ void __launch_bounds__(1024)
densify_offsets_kernel(int nblk, const unsigned *__restrict__ block_counts, unsigned *__restrict__ block_offsets, unsigned *__restrict__ totals) {
    __shared__ unsigned s_warp[4][32];
    __shared__ unsigned s_carry[4], s_tot[4];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 4) s_carry[tid] = 0u;
    __syncthreads();
    for (int base = 0; base < nblk; base += 1024) {
        const int b = base + tid;
        unsigned v[4], inc[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            v[k] = b < nblk ? block_counts[b * 4 + k] : 0u;
            inc[k] = v[k];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned n = __shfl_up_sync(0xffffffffu, inc[k], o); if (lane >= o) inc[k] += n; }
            if (lane == 31) s_warp[k][warp] = inc[k];
        }
        __syncthreads();
        if (warp == 0) {
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const unsigned w = s_warp[k][lane];
                unsigned winc = w;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const unsigned n = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += n; }
                s_warp[k][lane] = winc - w;
                if (lane == 31) s_tot[k] = winc;
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (b < nblk) block_offsets[b * 4 + k] = s_carry[k] + s_warp[k][warp] + inc[k] - v[k];
        __syncthreads();
        if (tid < 4) s_carry[tid] += s_tot[tid];
        __syncthreads();
    }
    if (tid < 4) totals[tid] = s_carry[tid];
}

__device__ __forceinline__ void copy_row(float *dst, const float *src, int w) {
    for (int k = 0; k < w; k++) dst[k] = src[k];
}
__device__ __forceinline__ void zero_row(float *dst, int w) {
    for (int k = 0; k < w; k++) dst[k] = 0.f;
}

__global__ void __launch_bounds__(kDensifyThreads)
densify_apply_kernel(int P, const unsigned char *__restrict__ cls, const unsigned *__restrict__ block_offsets,
                     const unsigned *__restrict__ totals, DensifyTensors T, const float *__restrict__ noise) {
    __shared__ unsigned s_warp[4][kDensifyThreads / 32];
    const int i = blockIdx.x * kDensifyThreads + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned c = i < P ? cls[i] : 0u;
    unsigned rank[4];
#pragma unroll
    for (int b = 0; b < 4; b++) {
        const unsigned m = __ballot_sync(0xffffffffu, (c >> b) & 1u);
        rank[b] = (unsigned)__popc(m & ((1u << lane) - 1u));
        if (lane == 0) s_warp[b][warp] = (unsigned)__popc(m);
    }
    __syncthreads();
#pragma unroll
    for (int b = 0; b < 4; b++) {
        unsigned off = block_offsets[blockIdx.x * 4 + b];
        for (int w = 0; w < warp; w++) off += s_warp[b][w];
        rank[b] += off;
    }
    if (i >= P) return;
    const unsigned nK = totals[0], nC = totals[1], nS = totals[2], nH = totals[3];
    if (c & kKeep) {
        const size_t d = rank[0];
#pragma unroll
        for (int t = 0; t < kDensifyTensors; t++) {
            const int w = T.width[t];
            copy_row(T.out[t] + d * w, T.in[t] + (size_t)i * w, w);
            copy_row(T.m_out[t] + d * w, T.m_in[t] + (size_t)i * w, w);
            copy_row(T.v_out[t] + d * w, T.v_in[t] + (size_t)i * w, w);
        }
    }
    if (c & kClone) {
        const size_t d = (size_t)nK + rank[1];
#pragma unroll
        for (int t = 0; t < kDensifyTensors; t++) {
            const int w = T.width[t];
            copy_row(T.out[t] + d * w, T.in[t] + (size_t)i * w, w);
            zero_row(T.m_out[t] + d * w, w);
            zero_row(T.v_out[t] + d * w, w);
        }
    }
    if (c & kChild) {
        // stds = exp(scaling), samples = N(0, stds), xyz' = R(q / |q|) samples + xyz, scaling' = log(stds / 1.6)   (:563-570)
        const float *sc = T.in[4] + (size_t)i * 3, *q = T.in[5] + (size_t)i * 4, *x = T.in[0] + (size_t)i * 3;
        const float s0 = expf(sc[0]), s1 = expf(sc[1]), s2 = expf(sc[2]);
        const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        const float r = q[0] / qn, qx = q[1] / qn, qy = q[2] / qn, qz = q[3] / qn;
        const float R[9] = { 1.f - 2.f * (qy * qy + qz * qz), 2.f * (qx * qy - r * qz), 2.f * (qx * qz + r * qy),
                             2.f * (qx * qy + r * qz), 1.f - 2.f * (qx * qx + qz * qz), 2.f * (qy * qz - r * qx),
                             2.f * (qx * qz - r * qy), 2.f * (qy * qz + r * qx), 1.f - 2.f * (qx * qx + qy * qy) };
        for (int child = 0; child < 2; child++) {
            const size_t d = (size_t)nK + nC + (size_t)child * nH + rank[3];
            // the reference draws one normal per row of stds = scaling[selected].repeat(2, 1): row = child * n_selected + rank
            const float *z = noise + ((size_t)child * nS + rank[2]) * 3;
            const float a0 = z[0] * s0, a1 = z[1] * s1, a2 = z[2] * s2;
            float *ox = T.out[0] + d * 3;
            ox[0] = R[0] * a0 + R[1] * a1 + R[2] * a2 + x[0];
            ox[1] = R[3] * a0 + R[4] * a1 + R[5] * a2 + x[1];
            ox[2] = R[6] * a0 + R[7] * a1 + R[8] * a2 + x[2];
            float *os = T.out[4] + d * 3;
            os[0] = logf(s0 / 1.6f); os[1] = logf(s1 / 1.6f); os[2] = logf(s2 / 1.6f);
#pragma unroll
            for (int t = 0; t < kDensifyTensors; t++) {
                const int w = T.width[t];
                if (t != 0 && t != 4) copy_row(T.out[t] + d * w, T.in[t] + (size_t)i * w, w);
                zero_row(T.m_out[t] + d * w, w);
                zero_row(T.v_out[t] + d * w, w);
            }
        }
    }
}

}  // namespace dgr
