// dgr_camgrad.cuh — camera gradients (DGR_RASTER_CAMERA_GRADS, include/dgr_b200.h): dL/dviewmatrix, dL/dprojmatrix and dL/dcampos
// of one render, per view.  Launched after the per-Gaussian backward of the same call; it reads the op's inputs, radii, the
// clamp bits in `touched` and each record's 12 moments in grad_rec (after the deterministic render: the moments det_moments_gather
// wrote), so one kernel serves all six backward entry points.
//
// Why a kernel of its own instead of a constexpr switch in dgr_backward_body.cuh: the per-Gaussian backward kernels stay
// instruction-identical (the 80-register preprocess_bwd, which already spills, gets no new live state) and their 44 + 16
// instantiations are not doubled.  The price is that camera_bwd_kernel restates the moments -> (dt, dT) chain of
// backward_camera (dgr_backward.cuh) below; keep the two in step.
//
// Per visible record (radius > 0), with t = [p,1] V (view space), ph = [p,1] PM, T = J Rwv (rows T0, T1):
//   dL/dt        = the J-path terms (dtx, dty, dtz) + (0, 0, dL/ddepth)
//   dL/dV[i][j] += p_i dL/dt_j + sum_r dT[r][i] J[r][j]   (i, j < 3);  dL/dV[3][j] += dL/dt_j;  column 3: 0 (never read)
//   dL/dPM[i][k] += [p,1]_i dL/dph_k, dL/dph = (gndx pw, gndy pw, 0, -(ph.x gndx + ph.y gndy) pw^2);  column 2: 0
//   dL/dcampos  -= the SH view-direction term of dL/dmeans3D (0 with colors_precomp and at degree 0)
// Constants as in the per-Gaussian backward: cull decisions, radius, tile rect, low-pass, eigenvalue floor, the clamped
// tx'/ty' inside J; min(0.99, .) is straight-through.  AA: the opacity-compensation gradient enters (ga, gb, gc) through
// aa_conic_grads and reaches V through T and t.
//
// Reduction without float atomics: each CTA reduces its 27 partials in a fixed order (warp butterfly, then the warps in order)
// into one row per (CTA, view) of the caller's scratch; camera_reduce_kernel adds each view's rows in CTA order.  Bit-reproducible
// whenever the moments are (the deterministic backward).
#pragma once
#include "dgr_backward.cuh"

namespace dgr {

constexpr int kCamPartials = 27;        // 12 V (rows 0-3, columns 0-2), 12 PM (rows 0-3, columns 0, 1, 3), 3 campos
constexpr int kCamReduceThreads = 256;

__host__ __device__ inline size_t camera_grad_rows(int V, int P) {
    return (size_t)(V > 0 ? V : 1) * (((size_t)(P > 0 ? P : 0) + kPreThreads - 1) / kPreThreads);
}
__host__ __device__ inline size_t camera_grad_scratch_bytes(int V, int P) {
    return align_up(camera_grad_rows(V, P) * kCamPartials * 4, 256) + 256;
}

// grid (ceil(P / 256), V): blockIdx.y = the view.  Single view: V = 1, tanfov = NULL (tan0 holds tanfovx, tanfovy).
// Batched: viewmatrix / projmatrix [V,16], campos [V,3], tanfov [V,2]; record r = v P + g.
template <int DEG, bool HAS_SH, bool HAS_COV, bool RAW, bool AA>
__global__ void __launch_bounds__(kPreThreads) camera_bwd_kernel(
    int P, int M, const __grid_constant__ ViewTable vt, float2 tan0, const float *__restrict__ tanfov, float scale_modifier,
    const float *__restrict__ viewmatrix, const float *__restrict__ projmatrix, const float *__restrict__ campos,
    const float *__restrict__ means3D, const float *__restrict__ shs, const float *__restrict__ shs_rest,
    const float *__restrict__ scales, const float *__restrict__ rotations, const float *__restrict__ cov3D_precomp,
    const int *__restrict__ radii, const unsigned *__restrict__ touched, const float *__restrict__ grad_rec,
    float *__restrict__ rows) {
    __shared__ FrameConsts fc;
    __shared__ float s_part[kPreThreads / 32][kCamPartials];
    const int v = blockIdx.y;
    load_frame(fc, viewmatrix + 16 * (size_t)v, projmatrix + 16 * (size_t)v, HAS_SH ? campos + 3 * (size_t)v : nullptr);
    __syncthreads();
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    const size_t rid = (size_t)v * P + g;
    float acc[kCamPartials];
#pragma unroll
    for (int k = 0; k < kCamPartials; k++) acc[k] = 0.f;
    if (g < P && radii[rid] > 0) {
        const float3 p = make_float3(__ldg(means3D + 3 * (size_t)g), __ldg(means3D + 3 * (size_t)g + 1), __ldg(means3D + 3 * (size_t)g + 2));
        float S6[6];
        if (HAS_COV) {
#pragma unroll
            for (int i = 0; i < 6; i++) S6[i] = __ldg(cov3D_precomp + 6 * (size_t)g + i);
        } else {
            const float3 s_in = make_float3(__ldg(scales + 3 * (size_t)g), __ldg(scales + 3 * (size_t)g + 1), __ldg(scales + 3 * (size_t)g + 2));
            cov3d_from_inputs<RAW>(s_in, ldg_f4(rotations + 4 * (size_t)g), scale_modifier, S6);
        }
        const float2 tf = tanfov ? make_float2(__ldg(tanfov + 2 * v), __ldg(tanfov + 2 * v + 1)) : tan0;
        const int H = vt.H[v], W = vt.W[v];
        const float fx = (float)W / (2.f * tf.x), fy = (float)H / (2.f * tf.y);
        Geo geo;
        project_geo(fc, p, S6, fx, fy, DGR_FOV_CLAMP * tf.x, DGR_FOV_CLAMP * tf.y, geo);
        const float a = geo.cxx, b = geo.cxy, c = geo.cyy;
        const float det = a * c - b * b, di = 1.f / det;
        const float cA = c * di, cB = -b * di, cC = a * di;
        const float4 m0 = ldg_f4(grad_rec + rid * kGradRecFloats);
        const float4 m1 = ldg_f4(grad_rec + rid * kGradRecFloats + 4);
        const float4 m2 = ldg_f4(grad_rec + rid * kGradRecFloats + 8);
        // moments: m0 = {u, u dx, u dy, u dx^2}, m1 = {u dx dy, u dy^2, wr, wg}, m2 = {wb, wd, -, -}
        const float gpx = -(cA * m0.y + cB * m0.z), gpy = -(cC * m0.z + cB * m0.y);
        const float gA = -0.5f * m0.w, gB = -m1.x, gC = -0.5f * m1.y;
        const float g_depth = m2.y;
        const float gndx = gpx * 0.5f * (float)W, gndy = gpy * 0.5f * (float)H;

        // projection: dL/dph, then dL/dPM[i][k] = [p,1]_i dL/dph_k (k = 0, 1, 3)
        {
            const float dph[3] = { gndx * geo.pw, gndy * geo.pw, -(geo.ndcx * gndx + geo.ndcy * gndy) * geo.pw };
            const float ph1[4] = { p.x, p.y, p.z, 1.f };
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int k = 0; k < 3; k++) acc[12 + 3 * i + k] = ph1[i] * dph[k];
        }
        // SH view direction: dir = (p - campos) / |p - campos|, so dL/dcampos = -(its term of dL/dmeans3D)
        if (HAS_SH && DEG > 0) {
            float dx = p.x - fc.cam[0], dy = p.y - fc.cam[1], dz = p.z - fc.cam[2];
            const float il = 1.f / sqrtf(dx * dx + dy * dy + dz * dz);
            dx *= il; dy *= il; dz *= il;
            const unsigned flags = __ldg(touched + rid) >> 29;           // SH channels the forward clamped at 0
            float gr[3];
            const float g_rgb[3] = { m1.z, m1.w, m2.x };
#pragma unroll
            for (int ch = 0; ch < 3; ch++) gr[ch] = ((flags >> ch) & 1u) ? 0.f : g_rgb[ch];
            const float *row = RAW ? shs_rest + (size_t)g * (M - 1) * 3 : shs + (size_t)g * M * 3;
            float ddx = 0.f, ddy = 0.f, ddz = 0.f;
            constexpr int NB = (DEG + 1) * (DEG + 1);
#pragma unroll
            for (int k = 1; k < NB; k++) {                                // d basis_0 = 0
                const int off = RAW ? 3 * (k - 1) : 3 * k;
                const float dotc = __ldg(row + off) * gr[0] + __ldg(row + off + 1) * gr[1] + __ldg(row + off + 2) * gr[2];
                float bx, by, bz;
                sh_dbasis(k, dx, dy, dz, bx, by, bz);
                ddx += bx * dotc; ddy += by * dotc; ddz += bz * dotc;
            }
            const float dot = dx * ddx + dy * ddy + dz * ddz;
            acc[24] = -(ddx - dx * dot) * il; acc[25] = -(ddy - dy * dot) * il; acc[26] = -(ddz - dz * dot) * il;
        }

        // conic -> cov2D -> T = J Rwv -> (dT, dL/dt): the chain of backward_camera
        const float d2 = di * di;
        float ga = d2 * (-c * c * gA + b * c * gB - b * b * gC);
        float gc = d2 * (-b * b * gA + a * b * gB - a * a * gC);
        float gb = d2 * (2.f * b * c * gA - (det + 2.f * b * b) * gB + 2.f * a * b * gC);
        if (AA) aa_conic_grads(geo, S6, det, m0.x, ga, gb, gc);
        const float G00 = ga, G01 = 0.5f * gb, G11 = gc;
        const float *T0 = geo.T0, *T1 = geo.T1;
        const float Sg[9] = { S6[0], S6[1], S6[2], S6[1], S6[3], S6[4], S6[2], S6[4], S6[5] };
        float dT0[3], dT1[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float ts0 = T0[0] * Sg[k] + T0[1] * Sg[3 + k] + T0[2] * Sg[6 + k];
            const float ts1 = T1[0] * Sg[k] + T1[1] * Sg[3 + k] + T1[2] * Sg[6 + k];
            dT0[k] = 2.f * (G00 * ts0 + G01 * ts1); dT1[k] = 2.f * (G01 * ts0 + G11 * ts1);
        }
        float dJ00 = 0.f, dJ02 = 0.f, dJ11 = 0.f, dJ12 = 0.f;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            dJ00 += dT0[k] * fc.V[4 * k]; dJ02 += dT0[k] * fc.V[4 * k + 2];
            dJ11 += dT1[k] * fc.V[4 * k + 1]; dJ12 += dT1[k] * fc.V[4 * k + 2];
        }
        const float tz = geo.t[2];
        const float tz2 = 1.f / (tz * tz), tz3 = tz2 / tz;
        const float dt[3] = { geo.clx ? 0.f : -fx * tz2 * dJ02, geo.cly ? 0.f : -fy * tz2 * dJ12,
                              -fx * tz2 * dJ00 - fy * tz2 * dJ11 + 2.f * fx * geo.tx * tz3 * dJ02 + 2.f * fy * geo.ty * tz3 * dJ12 + g_depth };
        // J as project_geo forms it: rows (J00, 0, J02), (0, J11, J12)
        const float J00 = fx / tz, J02 = -(fx * geo.tx) / (tz * tz), J11 = fy / tz, J12 = -(fy * geo.ty) / (tz * tz);
        const float J0[3] = { J00, 0.f, J02 }, J1[3] = { 0.f, J11, J12 };
        const float pv[3] = { p.x, p.y, p.z };
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) acc[3 * i + j] = pv[i] * dt[j] + dT0[i] * J0[j] + dT1[i] * J1[j];
#pragma unroll
        for (int j = 0; j < 3; j++) acc[9 + j] = dt[j];
    }
    // fixed-order CTA reduction: butterfly within the warp (every lane ends with the same sum), then the warps in order
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kCamPartials; k++) {
        float x = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if (lane == 0) s_part[warp][k] = x;
    }
    __syncthreads();
    if (threadIdx.x < kCamPartials) {
        float x = 0.f;
#pragma unroll
        for (int w = 0; w < kPreThreads / 32; w++) x += s_part[w][threadIdx.x];
        rows[((size_t)v * gridDim.x + blockIdx.x) * kCamPartials + threadIdx.x] = x;
    }
}

// grid V, kCamReduceThreads threads: warp w adds rows w, w + 8, w + 16, ... of its view in order, then the 8 warp sums are added in
// warp order.  Writes (never accumulates) every entry of the view's outputs, the columns the forward never reads as 0; any output
// may be NULL.  nblk = 0 (an empty cloud): zeros.
__global__ void __launch_bounds__(kCamReduceThreads) camera_reduce_kernel(int nblk, const float *__restrict__ rows, float *__restrict__ dV,
                                                                          float *__restrict__ dPM, float *__restrict__ dcam) {
    __shared__ float s_part[kCamReduceThreads / 32][32];
    const int v = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int kWarps = kCamReduceThreads / 32;
    float x = 0.f;
    if (lane < kCamPartials) {
        const float *r = rows + (size_t)v * nblk * kCamPartials + lane;
#pragma unroll 8
        for (int b = warp; b < nblk; b += kWarps) x += __ldg(r + (size_t)b * kCamPartials);
    }
    s_part[warp][lane] = x;
    __syncthreads();
    if (warp != 0) return;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; w++) s += s_part[w][lane];
    if (lane < 12) {
        if (dV) dV[16 * (size_t)v + 4 * (lane / 3) + lane % 3] = s;
    } else if (lane < 24) {
        const int i = (lane - 12) / 3, k = (lane - 12) % 3;
        if (dPM) dPM[16 * (size_t)v + 4 * i + (k == 2 ? 3 : k)] = s;
    } else if (lane < kCamPartials) {
        if (dcam) dcam[3 * (size_t)v + lane - 24] = s;
    } else if (lane < kCamPartials + 4) {
        const int i = lane - kCamPartials;
        if (dV) dV[16 * (size_t)v + 4 * i + 3] = 0.f;
        if (dPM) dPM[16 * (size_t)v + 4 * i + 2] = 0.f;
    }
}

}  // namespace dgr
