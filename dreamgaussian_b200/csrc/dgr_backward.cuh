// dgr_backward.cuh — per-Gaussian backward (A6 of SURVEY.md §8a): takes the 10 moments the backward render
// reduced per Gaussian and applies the exact chain rule of the forward preprocess back to
// means3D / means2D / shs (or colors) / opacities / scales / rotations (or cov3D).
// Streaming, HBM-bound: re-reads 44 + 12 M bytes + 48 bytes of moments, writes 56 + 12 M bytes per Gaussian.
// Cull decisions, radius, tile rect, low-pass and eigenvalue floor are constants; the tx/tz, ty/tz clamp masks
// the gradient through the clamped ratio; SH channels clamped at 0 get no colour gradient.
#pragma once
#include "dgr_preprocess.cuh"

namespace dgr {

// d basis_k / d(x, y, z) for one coefficient index (k is a compile-time constant after unrolling)
__device__ __forceinline__ void sh_dbasis(int k, float x, float y, float z, float &dx, float &dy, float &dz) {
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    dx = 0.f; dy = 0.f; dz = 0.f;
    switch (k) {
        case 1: dy = -DGR_SH_C1; break;
        case 2: dz = DGR_SH_C1; break;
        case 3: dx = -DGR_SH_C1; break;
        case 4: dx = DGR_SH_C2_0 * y; dy = DGR_SH_C2_0 * x; break;
        case 5: dy = DGR_SH_C2_1 * z; dz = DGR_SH_C2_1 * y; break;
        case 6: dx = DGR_SH_C2_2 * -2.f * x; dy = DGR_SH_C2_2 * -2.f * y; dz = DGR_SH_C2_2 * 4.f * z; break;
        case 7: dx = DGR_SH_C2_3 * z; dz = DGR_SH_C2_3 * x; break;
        case 8: dx = DGR_SH_C2_4 * 2.f * x; dy = DGR_SH_C2_4 * -2.f * y; break;
        case 9: dx = DGR_SH_C3_0 * 6.f * xy; dy = DGR_SH_C3_0 * (3.f * xx - 3.f * yy); break;
        case 10: dx = DGR_SH_C3_1 * yz; dy = DGR_SH_C3_1 * xz; dz = DGR_SH_C3_1 * xy; break;
        case 11: dx = DGR_SH_C3_2 * -2.f * xy; dy = DGR_SH_C3_2 * (4.f * zz - xx - 3.f * yy); dz = DGR_SH_C3_2 * 8.f * yz; break;
        case 12: dx = DGR_SH_C3_3 * -6.f * xz; dy = DGR_SH_C3_3 * -6.f * yz; dz = DGR_SH_C3_3 * (6.f * zz - 3.f * xx - 3.f * yy); break;
        case 13: dx = DGR_SH_C3_4 * (4.f * zz - 3.f * xx - yy); dy = DGR_SH_C3_4 * -2.f * xy; dz = DGR_SH_C3_4 * 8.f * xz; break;
        case 14: dx = DGR_SH_C3_5 * 2.f * xz; dy = DGR_SH_C3_5 * -2.f * yz; dz = DGR_SH_C3_5 * (xx - yy); break;
        case 15: dx = DGR_SH_C3_6 * (3.f * xx - 3.f * yy); dy = DGR_SH_C3_6 * -6.f * xy; break;
        default: break;
    }
}

// ---- output stage ---------------------------------------------------------------------------------------------------------------
// Every gradient segment is [P, K] row-major, so the 32 rows of a warp are ONE contiguous run of 32 K floats.  Each lane drops its
// K values into the warp's shared-memory image of that run and the warp writes the run back with 16-byte stores on consecutive
// addresses (one store instruction for a [32, 3] block instead of three strided ones; full 32-byte sectors, which is what matters
// when the destination is another GPU's memory behind NVLink).
//   acc:        add to what the LOCAL buffer holds (several views -> one gradient);
//   delta != 0: the result goes to the same element of this rank's slot in the owner rank's staging area (PeerPush) instead of
//               back to the local buffer.
constexpr int kOut3D = 0, kOut2D = 96, kOutOp = 192, kOutScale = 224, kOutRot = 320, kOutCov = 448, kOutCol = 640;    // float offsets per warp
constexpr int kShStrideVec = 28, kShStrideScalar = 25;
constexpr int kStageFloats = 32 * kShStrideVec;               // per warp: >= kOutCol + 32 * 3

__device__ __forceinline__ void warp_flush(float *seg, int K, long long delta, int row_base, int nrows, bool acc, const float *ws) {
    if (!seg) return;
    const int lane = threadIdx.x & 31;
    float *loc = seg + (size_t)row_base * K;
    float *dst = loc + delta;
    const int n = nrows * K;
    int done = 0;
    if ((((size_t)loc | (size_t)dst) & 15) == 0) {
        const int n4 = n >> 2;
        for (int i = lane; i < n4; i += 32) {
            float4 x = reinterpret_cast<const float4 *>(ws)[i];
            if (acc) { const float4 o = reinterpret_cast<const float4 *>(loc)[i]; x.x += o.x; x.y += o.y; x.z += o.z; x.w += o.w; }
            reinterpret_cast<float4 *>(dst)[i] = x;
        }
        done = n4 << 2;
    }
    for (int i = done + lane; i < n; i += 32) {
        float x = ws[i];
        if (acc) x += loc[i];
        dst[i] = x;
    }
}

// SH gradient rows of one warp's 32 Gaussians.  Each lane owns one row (3M floats, of which the first 3*NB are bs[k]*gr[ch] and the
// rest zero).  The rows go through shared memory in chunks of 24 floats; a chunk leaves as 16-byte stores, 96 contiguous bytes
// per row, when the row length is a multiple of 4 floats (row stride 28 words: conflict-free 16-byte accesses), else as 4-byte
// stores with consecutive lanes on consecutive addresses (row stride 25 words).
// FIRST = 1: the destination rows are GaussianModel._features_rest ([P, M-1, 3], coefficients 1 .. M-1).
template <int DEG, int FIRST = 0>
__device__ __forceinline__ void store_sh_grads(float *__restrict__ dL_dshs, int P, int M, const float (&bs)[16],
                                               const float (&gr)[3], bool acc, float *stage /* [kStageFloats] of this warp */,
                                               long long delta = 0) {
    constexpr int NB = (DEG + 1) * (DEG + 1) - FIRST;
    const int lane = threadIdx.x & 31;
    const int row_base = (int)(blockIdx.x * blockDim.x) + (int)(threadIdx.x & ~31u);
    const int nrows = min(32, P - row_base);
    if (nrows <= 0) return;
    const int rowlen = 3 * (M - FIRST);
    const bool vec = (rowlen & 3) == 0 && ((((size_t)dL_dshs) | ((size_t)(dL_dshs + delta))) & 15) == 0;
#pragma unroll
    for (int c = 0; c < 2; c++) {
        if (24 * c < rowlen) {
            const int cw = min(24, rowlen - 24 * c);
            if (vec) {
#pragma unroll
                for (int j4 = 0; j4 < 6; j4++) {
                    float v[4];
#pragma unroll
                    for (int e = 0; e < 4; e++) {
                        const int f = 24 * c + 4 * j4 + e;            // compile-time
                        v[e] = (f / 3 < NB) ? bs[(f / 3 + FIRST) < 16 ? (f / 3 + FIRST) : 0] * gr[f % 3] : 0.f;
                    }
                    if (4 * j4 < cw) reinterpret_cast<float4 *>(stage + lane * kShStrideVec)[j4] = make_float4(v[0], v[1], v[2], v[3]);
                }
                __syncwarp();
                const int q = cw >> 2, total = nrows * q;
                for (int i = lane; i < total; i += 32) {
                    const int row = i / q, c4 = i - row * q;
                    float4 x = *reinterpret_cast<const float4 *>(stage + row * kShStrideVec + 4 * c4);
                    float *loc = dL_dshs + (size_t)(row_base + row) * rowlen + 24 * c + 4 * c4;
                    if (acc) { const float4 o = *reinterpret_cast<const float4 *>(loc); x.x += o.x; x.y += o.y; x.z += o.z; x.w += o.w; }
                    *reinterpret_cast<float4 *>(loc + delta) = x;
                }
            } else {
#pragma unroll
                for (int j = 0; j < 24; j++) {
                    const int f = 24 * c + j;                 // compile-time
                    const float v = (f / 3 < NB) ? bs[(f / 3 + FIRST) < 16 ? (f / 3 + FIRST) : 0] * gr[f % 3] : 0.f;
                    if (f < rowlen) stage[lane * kShStrideScalar + j] = v;
                }
                __syncwarp();
                const unsigned inv = (65536u + (unsigned)cw - 1u) / (unsigned)cw;      // exact idx / cw for idx < 32 * 24
                for (int it = 0; it < cw; it++) {
                    const int idx = it * 32 + lane;
                    const int row = (int)(((unsigned)idx * inv) >> 16), col = idx - row * cw;
                    if (row < nrows) {
                        float *dst = dL_dshs + (size_t)(row_base + row) * rowlen + 24 * c + col;
                        const float v = stage[row * kShStrideScalar + col];
                        dst[delta] = acc ? (*dst + v) : v;
                    }
                }
            }
            __syncwarp();
        }
    }
}

// Anti-aliased mode: the record's opacity is o_eff = o comp, comp = sqrt(max(floor, ratio)), ratio = det0 / det (aa_cov), so the
// moment u = sum dL/dalpha alpha gives dL/do = u / o (unchanged) and dL/dcomp = u / comp.  Where the floor is not active,
// dL/dratio = 0.5 u / ratio and d ratio / dx = (d det0 / dx - ratio d det / dx) / det for x = a, b, c: added to the gradients of the
// low-passed cov2D (ga, gb, gc), from where the conic's chain rule carries them on.  Floored: comp is a constant.
__device__ __forceinline__ void aa_conic_grads(const Geo &g, const float (&S6)[6], float det, float u, float &ga, float &gb, float &gc) {
    const AaCov k = aa_cov(g, S6, det);
    const float ratio = k.ratio;
    if (!(ratio > DGR_AA_RATIO_FLOOR)) return;
    const float s = 0.5f * u / (ratio * det);
    ga += s * (k.c0 - ratio * g.cyy);
    gc += s * (k.a0 - ratio * g.cxx);
    gb += s * (-2.f * g.cxy * (1.f - ratio));
}

// ---- pieces shared by the single-view and the batched (dgr_views_backward) per-Gaussian backward ------------------------------
// The camera-dependent chain rule for one Gaussian that camera rendered (radius > 0): from the moments the backward render reduced
// (fetched by `moments` once the geometry is known) to means2D (NDC units, gndx / gndy), means3D (dmean, SH direction term
// included), the activated opacity (g_op), the colour (g_rgb) and Sigma (dS, full 3x3).  With SH: bs = the basis values of this
// view direction and gr = the colour gradient with the channels the forward clamped (clamp_bits) zeroed, so d L / d sh[k][ch] =
// bs[k] gr[ch].  sh_at(i) = float i of the Gaussian's SH row as the kernels hold it (raw parameters: _features_rest).
// AA: the forward scaled the opacity by aa_comp (dgr_preprocess.cuh); g_op stays the gradient of the uncompensated opacity and
// aa_conic_grads adds the path through comp.
template <int DEG, bool HAS_SH, bool RAW, bool AA = false, class Moments, class ShAt>
__device__ __forceinline__ void backward_camera(const FrameConsts &fc, int H, int W, float tanfovx, float tanfovy, const float3 p,
                                                const float (&S6)[6], float o, unsigned clamp_bits, Moments moments, ShAt sh_at,
                                                float &gndx, float &gndy, float (&dmean)[3], float &g_op, float (&g_rgb)[3],
                                                float (&dS)[9], float (&bs)[16], float (&gr)[3]) {
    const float fx = (float)W / (2.f * tanfovx), fy = (float)H / (2.f * tanfovy);
    Geo geo;
    project_geo(fc, p, S6, fx, fy, DGR_FOV_CLAMP * tanfovx, DGR_FOV_CLAMP * tanfovy, geo);
    const float a = geo.cxx, b = geo.cxy, c = geo.cyy;
    const float det = a * c - b * b, di = 1.f / det;
    const float cA = c * di, cB = -b * di, cC = a * di;
    float4 m0, m1, m2;
    moments(m0, m1, m2);
    // moments: m0 = {u, u dx, u dy, u dx^2}, m1 = {u dx dy, u dy^2, wr, wg}, m2 = {wb, wd, -, -}

    // pixel-space mean gradient and conic gradient from the moments
    const float gpx = -(cA * m0.y + cB * m0.z), gpy = -(cC * m0.z + cB * m0.y);
    const float gA = -0.5f * m0.w, gB = -m1.x, gC = -0.5f * m1.y;
    g_op = (o != 0.f) ? m0.x / o : 0.f;
    g_rgb[0] = m1.z; g_rgb[1] = m1.w; g_rgb[2] = m2.x;
    const float g_depth = m2.y;

    dmean[0] = 0.f; dmean[1] = 0.f; dmean[2] = 0.f;
    // (1) mean_px through the full projection; reported means2D grad is in NDC units
    gndx = gpx * 0.5f * (float)W; gndy = gpy * 0.5f * (float)H;
    {
        const float *PM = fc.PM;
        const float mul1 = geo.ndcx * geo.pw, mul2 = geo.ndcy * geo.pw;     // ph.x * pw^2, ph.y * pw^2
#pragma unroll
        for (int k = 0; k < 3; k++)
            dmean[k] += (PM[4 * k] * geo.pw - PM[4 * k + 3] * mul1) * gndx + (PM[4 * k + 1] * geo.pw - PM[4 * k + 3] * mul2) * gndy;
    }
    // (4) depth = t.z
#pragma unroll
    for (int k = 0; k < 3; k++) dmean[k] += fc.V[4 * k + 2] * g_depth;
    // (3) colour
    if (HAS_SH) {
        float dx = p.x - fc.cam[0], dy = p.y - fc.cam[1], dz = p.z - fc.cam[2];
        const float il = 1.f / sqrtf(dx * dx + dy * dy + dz * dz);
        dx *= il; dy *= il; dz *= il;
        sh_basis<DEG>(dx, dy, dz, bs);
#pragma unroll
        for (int ch = 0; ch < 3; ch++) gr[ch] = ((clamp_bits >> ch) & 1u) ? 0.f : g_rgb[ch];
        float ddx = 0.f, ddy = 0.f, ddz = 0.f;
        constexpr int NB = (DEG + 1) * (DEG + 1);
#pragma unroll
        for (int k = 1; k < NB; k++) {                                // d basis_0 = 0
            const int off = RAW ? 3 * (k - 1) : 3 * k;
            const float dotc = sh_at(off) * gr[0] + sh_at(off + 1) * gr[1] + sh_at(off + 2) * gr[2];
            float bx, by, bz;
            sh_dbasis(k, dx, dy, dz, bx, by, bz);
            ddx += bx * dotc; ddy += by * dotc; ddz += bz * dotc;
        }
        const float dot = dx * ddx + dy * ddy + dz * ddz;
        dmean[0] += (ddx - dx * dot) * il; dmean[1] += (ddy - dy * dot) * il; dmean[2] += (ddz - dz * dot) * il;
    }

    // (2) conic -> cov2D -> (Sigma, T = J Rwv)
    const float d2 = di * di;
    float ga = d2 * (-c * c * gA + b * c * gB - b * b * gC);
    float gc = d2 * (-b * b * gA + a * b * gB - a * a * gC);
    float gb = d2 * (2.f * b * c * gA - (det + 2.f * b * b) * gB + 2.f * a * b * gC);
    if (AA) aa_conic_grads(geo, S6, det, m0.x, ga, gb, gc);
    const float G00 = ga, G01 = 0.5f * gb, G11 = gc;
    const float *T0 = geo.T0, *T1 = geo.T1;
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
        for (int l = 0; l < 3; l++)
            dS[3 * k + l] = T0[k] * (G00 * T0[l] + G01 * T1[l]) + T1[k] * (G01 * T0[l] + G11 * T1[l]);
    const float Sg[9] = { S6[0], S6[1], S6[2], S6[1], S6[3], S6[4], S6[2], S6[4], S6[5] };
    float TS0[3], TS1[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        TS0[k] = T0[0] * Sg[k] + T0[1] * Sg[3 + k] + T0[2] * Sg[6 + k];
        TS1[k] = T1[0] * Sg[k] + T1[1] * Sg[3 + k] + T1[2] * Sg[6 + k];
    }
    float dT0[3], dT1[3];
#pragma unroll
    for (int k = 0; k < 3; k++) { dT0[k] = 2.f * (G00 * TS0[k] + G01 * TS1[k]); dT1[k] = 2.f * (G01 * TS0[k] + G11 * TS1[k]); }
    float dJ00 = 0.f, dJ02 = 0.f, dJ11 = 0.f, dJ12 = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        dJ00 += dT0[k] * fc.V[4 * k]; dJ02 += dT0[k] * fc.V[4 * k + 2];
        dJ11 += dT1[k] * fc.V[4 * k + 1]; dJ12 += dT1[k] * fc.V[4 * k + 2];
    }
    const float tz = geo.t[2];
    const float tz2 = 1.f / (tz * tz), tz3 = tz2 / tz;
    const float dtx = geo.clx ? 0.f : -fx * tz2 * dJ02;
    const float dty = geo.cly ? 0.f : -fy * tz2 * dJ12;
    const float dtz = -fx * tz2 * dJ00 - fy * tz2 * dJ11 + 2.f * fx * geo.tx * tz3 * dJ02 + 2.f * fy * geo.ty * tz3 * dJ12;
#pragma unroll
    for (int k = 0; k < 3; k++) dmean[k] += fc.V[4 * k] * dtx + fc.V[4 * k + 1] * dty + fc.V[4 * k + 2] * dtz;
}

// d L / d Sigma -> scale and rotation gradients (raw parameters: with respect to _scaling and _rotation).  s = the scale the
// forward used (activated, times scale_modifier), R / q its rotation, inv_qnorm = 1 / |_rotation| (raw parameters).  Linear in dS.
template <bool RAW>
__device__ __forceinline__ void backward_scale_rot(const float (&dS)[9], const float (&R)[9], const float3 s, const float4 q, float inv_qnorm,
                                                   float scale_modifier, float (&dsc)[3], float (&dq)[4]) {
    // Sigma = Mx Mx^T, Mx = R diag(s):  dL/dMx = 2 dS Mx
    float Mx[9];
#pragma unroll
    for (int i = 0; i < 3; i++) { Mx[3 * i] = R[3 * i] * s.x; Mx[3 * i + 1] = R[3 * i + 1] * s.y; Mx[3 * i + 2] = R[3 * i + 2] * s.z; }
    float dM[9];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int k = 0; k < 3; k++)
            dM[3 * i + k] = 2.f * (dS[3 * i] * Mx[k] + dS[3 * i + 1] * Mx[3 + k] + dS[3 * i + 2] * Mx[6 + k]);
    const float sv[3] = { s.x, s.y, s.z };
    float dR[9];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float v = 0.f;
#pragma unroll
        for (int i = 0; i < 3; i++) { v += dM[3 * i + k] * R[3 * i + k]; dR[3 * i + k] = dM[3 * i + k] * sv[k]; }
        dsc[k] = RAW ? v * sv[k] : v * scale_modifier;                                   // exp' = exp
    }
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    dq[0] = 2.f * (-z * dR[1] + y * dR[2] + z * dR[3] - x * dR[5] - y * dR[6] + x * dR[7]);
    dq[1] = 2.f * (y * dR[1] + z * dR[2] + y * dR[3] - 2.f * x * dR[4] - r * dR[5] + z * dR[6] + r * dR[7] - 2.f * x * dR[8]);
    dq[2] = 2.f * (-2.f * y * dR[0] + x * dR[1] + r * dR[2] + x * dR[3] + z * dR[5] - r * dR[6] + z * dR[7] - 2.f * y * dR[8]);
    dq[3] = 2.f * (-2.f * z * dR[0] - r * dR[1] + x * dR[2] + r * dR[3] - 2.f * z * dR[4] + y * dR[5] + x * dR[6] + y * dR[7]);
    if (RAW) {          // q = raw / |raw|:  d raw = (dq - q (q . dq)) / |raw|
        const float qd = r * dq[0] + x * dq[1] + y * dq[2] + z * dq[3];
        dq[0] = (dq[0] - r * qd) * inv_qnorm; dq[1] = (dq[1] - x * qd) * inv_qnorm;
        dq[2] = (dq[2] - y * qd) * inv_qnorm; dq[3] = (dq[3] - z * qd) * inv_qnorm;
    }
}

// STAGE: the warp's inputs arrive by bulk TMA in its slice of dynamic shared memory (see dgr_preprocess.cuh, "Input staging");
// once every lane has its values in registers the same slice becomes the warp's output image (warp_flush), so the staged
// variant needs 8 x 32 x (44 + 12 M) bytes per CTA (59 KB at degree 3: three CTAs per SM, as before) and no static stage.
// Parameters of the single-view per-Gaussian backward kernels (preprocess_bwd_kernel, and preprocess_bwd_aa_kernel of the
// anti-aliased mode); both compile the body in dgr_backward_body.cuh.
#define DGR_PRE_BWD_PARAMS                                                                                                    \
    int P, int M, int H, int W, float tanfovx, float tanfovy, float scale_modifier, const float *__restrict__ viewmatrix,      \
        const float *__restrict__ projmatrix, const float *__restrict__ campos, const float *__restrict__ means3D,             \
        const float *__restrict__ shs, const float *__restrict__ shs_rest, const float *__restrict__ opacities,                \
        const float *__restrict__ scales, const float *__restrict__ rotations, const float *__restrict__ cov3D_precomp,        \
        const int *__restrict__ radii, const unsigned *__restrict__ touched, const float *__restrict__ grad_rec,               \
        float *__restrict__ dL_dmeans3D, float *__restrict__ dL_dmeans2D, float *__restrict__ dL_dshs,                         \
        float *__restrict__ dL_dcolors, float *__restrict__ dL_dopacities, float *__restrict__ dL_dscales,                     \
        float *__restrict__ dL_drotations, float *__restrict__ dL_dcov3D, float *__restrict__ dL_dshs_rest,                    \
        float *__restrict__ xyz_gradient_accum, float *__restrict__ denom, float *__restrict__ max_radii2D, int accumulate,    \
        PeerPush push, int warp_smem_floats

template <int DEG, bool HAS_SH, bool HAS_COV, bool RAW, bool STAGE = false>
__global__ void __launch_bounds__(kPreThreads, 3) preprocess_bwd_kernel(DGR_PRE_BWD_PARAMS) {
    constexpr bool AA = false;
#include "dgr_backward_body.cuh"
}
template <int DEG, bool HAS_SH, bool HAS_COV, bool RAW, bool STAGE = false>
__global__ void __launch_bounds__(kPreThreads, 3) preprocess_bwd_aa_kernel(DGR_PRE_BWD_PARAMS) {
    constexpr bool AA = true;
#include "dgr_backward_body.cuh"
}

// ----------------------------------------------------------------------------------------------------------------
// Batched backward (dgr_views_backward): a thread reads its Gaussian's inputs ONCE, then applies every view's chain rule to that
// view's moments (record v P + g) and sums in registers; the sums are written (or added) once.  The scale / rotation and opacity
// gradients are linear in d Sigma and d L / d opacity, so only those two are summed over the views and the rest of their chain
// rule runs once.  means2D is per view: [V, P, 3].  SH + scale / rotation inputs only (plain or raw parameters).  View v's chain
// rule uses its own image size (ViewTable).  Densification statistics: for every view whose bit is set in stats_views, in
// ascending view order, a Gaussian that view rendered gets the single-view rule of preprocess_bwd_kernel with that view's means2D
// gradient and radius (exactly what one single-view backward per selected view, in view order, leaves behind).
// ----------------------------------------------------------------------------------------------------------------
// Parameters of the batched per-Gaussian backward kernels; both compile the body in dgr_backward_views_body.cuh.
#define DGR_VIEWS_BWD_PARAMS                                                                                                  \
    int P, int M, int V, const __grid_constant__ ViewTable vt, float scale_modifier, const float *__restrict__ tanfov,          \
        const float *__restrict__ viewmatrix, const float *__restrict__ projmatrix, const float *__restrict__ campos,          \
        const float *__restrict__ means3D, const float *__restrict__ shs, const float *__restrict__ shs_rest,                  \
        const float *__restrict__ opacities, const float *__restrict__ scales, const float *__restrict__ rotations,            \
        const int *__restrict__ radii, const unsigned *__restrict__ touched, const float *__restrict__ grad_rec,               \
        float *__restrict__ dL_dmeans3D, float *__restrict__ dL_dmeans2D, float *__restrict__ dL_dshs,                         \
        float *__restrict__ dL_dopacities, float *__restrict__ dL_dscales, float *__restrict__ dL_drotations,                  \
        float *__restrict__ dL_dshs_rest, float *__restrict__ xyz_gradient_accum, float *__restrict__ denom,                   \
        float *__restrict__ max_radii2D, unsigned long long stats_views, int accumulate

template <int DEG, bool RAW>
__global__ void __launch_bounds__(kPreThreads, 3) preprocess_views_bwd_kernel(DGR_VIEWS_BWD_PARAMS) {
    constexpr bool AA = false;
#include "dgr_backward_views_body.cuh"
}
template <int DEG, bool RAW>
__global__ void __launch_bounds__(kPreThreads, 3) preprocess_views_bwd_aa_kernel(DGR_VIEWS_BWD_PARAMS) {
    constexpr bool AA = true;
#include "dgr_backward_views_body.cuh"
}

}  // namespace dgr
