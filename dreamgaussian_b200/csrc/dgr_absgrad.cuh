// dgr_absgrad.cuh — the absolute-gradient densification statistic (DGR_RASTER_ABS_GRAD; AbsGS, Ye et al., 2024).
//
// xyz_gradient_accum sums, per render, |dL/dmeans2D[:2]|: the norm of a sum over the pixels a Gaussian covers.  Where those pixels pull
// its centre in opposite directions the sum cancels, and a large Gaussian over detail never reaches the split threshold.  The
// statistic here sums the absolute values of the per-pixel terms first:
//     a_x = sum_p |u_p (A dx + B dy)| W/2,   a_y = sum_p |u_p (B dx + C dy)| H/2,   accum_abs += sqrt(a_x^2 + a_y^2)
// (u_p = o G dL/dalpha of the backward render, (dx, dy) = mean - pixel, (A, B, C) the conic).  The per-pixel sums exist only inside
// the backward render: its ABS variants (render_bwd_body / render_bwd_det_body) leave sum |u (A dx + B dy)| and sum |u (B dx + C dy)|
// in moment slots 10 and 11 of each record.  This kernel runs after the per-Gaussian backward, one thread per Gaussian, and adds the
// term of every view whose bit is set in stats_views, in view order, for the views where the Gaussian has radius > 0 — the views
// and the order preprocess_bwd uses for the other three statistics, which it keeps updating unchanged.
#pragma once
#include "dgr_common.cuh"

namespace dgr {

constexpr int kAbsStatsThreads = 256;

__global__ void __launch_bounds__(kAbsStatsThreads)
absgrad_stats_kernel(int P, int V, const __grid_constant__ ViewTable vt, unsigned long long stats_views, const int *__restrict__ radii,
                     const float *__restrict__ grad_rec, float *__restrict__ accum_abs) {
    const int g = blockIdx.x * kAbsStatsThreads + threadIdx.x;
    if (g >= P) return;
    float acc = accum_abs[g];
#pragma unroll
    for (int v = 0; v < kMaxViews; v++) {          // unrolled: vt is indexed with constants only (a run-time index puts it in local memory)
        if (v >= V) break;
        if (!((stats_views >> v) & 1ull)) continue;
        const size_t rid = (size_t)v * P + g;
        if (__ldg(radii + rid) <= 0) continue;
        const float2 m = __ldg(reinterpret_cast<const float2 *>(grad_rec + rid * kGradRecFloats + 10));
        const float ax = m.x * 0.5f * (float)vt.W[v], ay = m.y * 0.5f * (float)vt.H[v];
        acc += sqrtf(ax * ax + ay * ay);
    }
    accum_abs[g] = acc;
}

}  // namespace dgr
