// dgr_preprocess.cuh — per-Gaussian forward kernel (A2 of SURVEY.md §8a): frustum cull, cov3D, EWA cov2D, conic,
// radius, pixel mean, SH -> RGB, opacity-aware pixel AABB, and — fused — a per-block tile histogram (shared-memory
// atomics, published with one global atomic per touched tile) that replaces the reference's per-Gaussian prefix sum +
// host read-back.
// Streaming, HBM-bound: reads 44 + 12 M bytes, writes 56 bytes per Gaussian.
//
// Reference behaviour restated (not copied): the `preprocessCUDA` step of the op called at
// /root/reference/gs_renderer.py:800-809; maths anchors: gs_renderer.py:85-132 (R, cov3D), sh_utils.py:57-100 (SH).
#pragma once
#include "dgr_common.cuh"

namespace dgr {

struct FrameConsts {            // staged in shared memory once per block
    float V[16], PM[16], cam[3], pad;
};

__device__ __forceinline__ void load_frame(FrameConsts &fc, const float *V, const float *PM, const float *cam) {
    int t = threadIdx.x;
    if (t < 16) fc.V[t] = __ldg(V + t);
    else if (t < 32) fc.PM[t - 16] = __ldg(PM + t - 16);
    else if (t < 35 && cam) fc.cam[t - 32] = __ldg(cam + t - 32);
}

__device__ __forceinline__ void quat_to_R(const float4 q, float (&R)[9]) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - r * z); R[2] = 2.f * (x * z + r * y);
    R[3] = 2.f * (x * y + r * z); R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - r * x);
    R[6] = 2.f * (x * z - r * y); R[7] = 2.f * (y * z + r * x); R[8] = 1.f - 2.f * (x * x + y * y);
}

// Sigma = (R S)(R S)^T packed xx,xy,xz,yy,yz,zz
__device__ __forceinline__ void cov3d_from_scale_rot(const float3 s, const float (&R)[9], float (&S6)[6]) {
    float M[9];
#pragma unroll
    for (int i = 0; i < 3; i++) { M[3 * i] = R[3 * i] * s.x; M[3 * i + 1] = R[3 * i + 1] * s.y; M[3 * i + 2] = R[3 * i + 2] * s.z; }
    S6[0] = M[0] * M[0] + M[1] * M[1] + M[2] * M[2];
    S6[1] = M[0] * M[3] + M[1] * M[4] + M[2] * M[5];
    S6[2] = M[0] * M[6] + M[1] * M[7] + M[2] * M[8];
    S6[3] = M[3] * M[3] + M[4] * M[4] + M[5] * M[5];
    S6[4] = M[3] * M[6] + M[4] * M[7] + M[5] * M[8];
    S6[5] = M[6] * M[6] + M[7] * M[7] + M[8] * M[8];
}

// SH basis values for a unit direction (sh_utils.py:74-100), b[0..(DEG+1)^2)
template <int DEG>
__device__ __forceinline__ void sh_basis(float x, float y, float z, float (&b)[16]) {
    b[0] = DGR_SH_C0;
    if (DEG > 0) {
        b[1] = -DGR_SH_C1 * y; b[2] = DGR_SH_C1 * z; b[3] = -DGR_SH_C1 * x;
        if (DEG > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            b[4] = DGR_SH_C2_0 * xy; b[5] = DGR_SH_C2_1 * yz; b[6] = DGR_SH_C2_2 * (2.f * zz - xx - yy);
            b[7] = DGR_SH_C2_3 * xz; b[8] = DGR_SH_C2_4 * (xx - yy);
            if (DEG > 2) {
                b[9] = DGR_SH_C3_0 * y * (3.f * xx - yy);
                b[10] = DGR_SH_C3_1 * xy * z;
                b[11] = DGR_SH_C3_2 * y * (4.f * zz - xx - yy);
                b[12] = DGR_SH_C3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy);
                b[13] = DGR_SH_C3_4 * x * (4.f * zz - xx - yy);
                b[14] = DGR_SH_C3_5 * z * (xx - yy);
                b[15] = DGR_SH_C3_6 * x * (xx - 3.f * yy);
            }
        }
    }
}

// Streams one Gaussian's SH row ([M][3] layout) in chunks of 8 coefficients (6 x 128-bit loads in flight when the row is
// 16-byte aligned, i.e. M % 4 == 0: the deg-1 and deg-3 tensors; scalar loads otherwise) and hands every coefficient to f.
// Keeping only one chunk live (instead of all 48 floats) is what keeps the per-Gaussian kernels below 64 registers.
// FIRST = 1 streams coefficients 1 .. NB-1 from a row that starts at coefficient 1 (GaussianModel._features_rest).
template <int DEG, int FIRST = 0, class F>
__device__ __forceinline__ void for_each_sh_coeff(const float *row, bool vec, F f) {
    constexpr int NB = (DEG + 1) * (DEG + 1) - FIRST;
#pragma unroll
    for (int k0 = 0; k0 < NB; k0 += 8) {
        constexpr int dummy = 0; (void)dummy;
        const int n = (NB - k0) < 8 ? (NB - k0) : 8;        // compile-time after unrolling
        float c[24];
        if (vec) {
#pragma unroll
            for (int i = 0; i < 6; i++) {
                if (4 * i < 3 * n) {
                    const float4 v = ldg_f4(row + 3 * k0 + 4 * i);
                    c[4 * i] = v.x; c[4 * i + 1] = v.y; c[4 * i + 2] = v.z; c[4 * i + 3] = v.w;
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < 24; i++) if (i < 3 * n) c[i] = __ldg(row + 3 * k0 + i);
        }
#pragma unroll
        for (int j = 0; j < 8; j++) if (j < n) f(k0 + j + FIRST, c[3 * j], c[3 * j + 1], c[3 * j + 2]);
    }
}

// One Gaussian's whole SH row ([M][3] layout, coefficients FIRST .. NB-1) into registers: 128-bit loads when the row is
// 16-byte aligned (M % 4 == 0: the deg-1 and deg-3 tensors), scalar loads otherwise.  Used at the very top of the
// per-Gaussian kernels, together with every other input of the Gaussian, so that ONE memory round trip feeds the thread
// (these kernels run 2-3 CTAs per SM at 100k Gaussians: latency, not registers, is what limits them).
template <int DEG, int FIRST = 0>
__device__ __forceinline__ void load_sh_row(const float *row, bool vec, float (&c)[48]) {
    constexpr int N = 3 * ((DEG + 1) * (DEG + 1) - FIRST);
    if (vec) {
#pragma unroll
        for (int i = 0; i < (N + 3) / 4; i++) {
            const float4 v = ldg_f4(row + 4 * i);
            c[4 * i] = v.x;
            if (4 * i + 1 < 48) c[4 * i + 1] = v.y;
            if (4 * i + 2 < 48) c[4 * i + 2] = v.z;
            if (4 * i + 3 < 48) c[4 * i + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < N; i++) c[i] = __ldg(row + i);
    }
}

// ----------------------------------------------------------------------------------------------------------------
// Input staging of the per-Gaussian kernels (bulk TMA).  A thread of these kernels needs 44 + 12 M bytes of ITS Gaussian:
// read per thread, a warp-wide 128-bit load of the SH rows touches 32 different 128-byte lines (row stride 12 M bytes), so the
// 12 loads of a degree-3 row cost 12 x 32 L1 wavefronts per warp and the kernel is bound by the load/store unit long before
// HBM.  But the 32 Gaussians of a warp are ONE contiguous run in each input array: lane 0 fetches the warp's five runs with
// five cp.async.bulk copies (completion on the warp's own mbarrier, no CTA-level coupling) and every lane then picks its
// values out of shared memory.  Layout of a warp's staging area, in floats (every piece starts 16-byte aligned):
//   [0, 96) means3D | [96, 192) scales | [192, 320) rotations | [320, 352) opacities | [352, 352 + 96 M) SH rows
//   (raw parameters: [352, 448) _features_dc, [448, 448 + 96 (M - 1)) _features_rest)
// Used for full warps (32 valid Gaussians) when every base pointer is 16-byte aligned; a partial warp at the end of the cloud
// and unaligned inputs take the per-thread loads.
// ----------------------------------------------------------------------------------------------------------------
constexpr int kStgMean = 0, kStgScale = 96, kStgRot = 192, kStgOp = 320, kStgSh = 352;
__host__ __device__ inline int stage_warp_floats(int M) { return 32 * (11 + 3 * M); }

// lane 0 of a warp: start the copies of the 32 Gaussians [g0, g0 + 32) into the warp's staging area
template <bool RAW>
__device__ __forceinline__ void stage_issue(float *ws, uint64_t *bar, int g0, int M, const float *means3D, const float *scales,
                                            const float *rotations, const float *opacities, const float *shs, const float *shs_rest) {
    const uint32_t sh_bytes = RAW ? 384u : 384u * (uint32_t)M, rest_bytes = (RAW && M > 1) ? 384u * (uint32_t)(M - 1) : 0u;
    mbar_expect_tx(bar, 384u + 384u + 512u + 128u + sh_bytes + rest_bytes);
    tma_bulk_g2s(ws + kStgMean, means3D + 3 * (size_t)g0, 384u, bar);
    tma_bulk_g2s(ws + kStgScale, scales + 3 * (size_t)g0, 384u, bar);
    tma_bulk_g2s(ws + kStgRot, rotations + 4 * (size_t)g0, 512u, bar);
    tma_bulk_g2s(ws + kStgOp, opacities + (size_t)g0, 128u, bar);
    if (RAW) {
        tma_bulk_g2s(ws + kStgSh, shs + 3 * (size_t)g0, 384u, bar);                                   // _features_dc [P, 1, 3]
        if (rest_bytes) tma_bulk_g2s(ws + kStgSh + 96, shs_rest + (size_t)g0 * (M - 1) * 3, rest_bytes, bar);
    } else {
        tma_bulk_g2s(ws + kStgSh, shs + (size_t)g0 * M * 3, sh_bytes, bar);
    }
}

// A staged SH row (coefficients FIRST .. NB-1 of lane's Gaussian) into registers; same register image as load_sh_row.
template <int DEG, int FIRST = 0>
__device__ __forceinline__ void lds_sh_row(const float *row, bool vec, float (&c)[48]) {
    constexpr int N = 3 * ((DEG + 1) * (DEG + 1) - FIRST);
    if (vec) {
#pragma unroll
        for (int i = 0; i < (N + 3) / 4; i++) {
            const float4 v = *reinterpret_cast<const float4 *>(row + 4 * i);
            c[4 * i] = v.x;
            if (4 * i + 1 < 48) c[4 * i + 1] = v.y;
            if (4 * i + 2 < 48) c[4 * i + 2] = v.z;
            if (4 * i + 3 < 48) c[4 * i + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < N; i++) c[i] = row[i];
    }
}

// GaussianModel activations (gs_renderer.py:127-138, :196-216), applied in registers when the caller passes the raw
// parameters (DgrGaussians.activations): scaling = exp, opacity = sigmoid, rotation = F.normalize (eps 1e-12).
__device__ __forceinline__ float act_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float4 act_normalize(float4 q, float &inv_norm) {
    inv_norm = 1.f / fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);
    return make_float4(q.x * inv_norm, q.y * inv_norm, q.z * inv_norm, q.w * inv_norm);
}

// Geometry shared by forward and backward: everything up to cov2D for one Gaussian.
struct Geo {
    float t[3];          // view-space position
    float tx, ty;        // clamped*tz (used in J only)
    bool clx, cly;       // tx/tz, ty/tz were clamped
    float T0[3], T1[3];  // rows of T = J * Rwv
    float cxx, cxy, cyy; // cov2D incl. low-pass
    float ndcx, ndcy, pw;
};

__device__ __forceinline__ void project_geo(const FrameConsts &fc, const float3 p, const float (&S6)[6],
                                            float fx, float fy, float limx, float limy, Geo &g) {
    const float *V = fc.V, *PM = fc.PM;
#pragma unroll
    for (int i = 0; i < 3; i++) g.t[i] = p.x * V[i] + p.y * V[4 + i] + p.z * V[8 + i] + V[12 + i];
    float ph[4];
#pragma unroll
    for (int i = 0; i < 4; i++) ph[i] = p.x * PM[i] + p.y * PM[4 + i] + p.z * PM[8 + i] + PM[12 + i];
    g.pw = 1.f / (ph[3] + DGR_W_EPS);
    g.ndcx = ph[0] * g.pw; g.ndcy = ph[1] * g.pw;
    const float tz = g.t[2];
    const float txtz = g.t[0] / tz, tytz = g.t[1] / tz;
    g.clx = (txtz < -limx) || (txtz > limx);
    g.cly = (tytz < -limy) || (tytz > limy);
    g.tx = fminf(limx, fmaxf(-limx, txtz)) * tz;
    g.ty = fminf(limy, fmaxf(-limy, tytz)) * tz;
    const float J00 = fx / tz, J02 = -(fx * g.tx) / (tz * tz), J11 = fy / tz, J12 = -(fy * g.ty) / (tz * tz);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        g.T0[k] = J00 * V[4 * k] + J02 * V[4 * k + 2];
        g.T1[k] = J11 * V[4 * k + 1] + J12 * V[4 * k + 2];
    }
    const float Sg[9] = { S6[0], S6[1], S6[2], S6[1], S6[3], S6[4], S6[2], S6[4], S6[5] };
    float ST0[3], ST1[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        ST0[k] = Sg[3 * k] * g.T0[0] + Sg[3 * k + 1] * g.T0[1] + Sg[3 * k + 2] * g.T0[2];
        ST1[k] = Sg[3 * k] * g.T1[0] + Sg[3 * k + 1] * g.T1[1] + Sg[3 * k + 2] * g.T1[2];
    }
    g.cxx = g.T0[0] * ST0[0] + g.T0[1] * ST0[1] + g.T0[2] * ST0[2] + DGR_COV2D_LOWPASS;
    g.cxy = g.T0[0] * ST1[0] + g.T0[1] * ST1[1] + g.T0[2] * ST1[2];
    g.cyy = g.T1[0] * ST1[0] + g.T1[1] * ST1[1] + g.T1[2] * ST1[2] + DGR_COV2D_LOWPASS;
}

// Anti-aliased mode (the 2D Mip filter of Mip-Splatting): the low-pass dilation keeps its conic, radius and tile rect, and the
// opacity is scaled by comp = sqrt(max(DGR_AA_RATIO_FLOOR, det0 / det)) so that a Gaussian keeps its integrated weight at every
// resolution.  det = the determinant of cov2D with the low-pass, det0 = without it, formed from the diagonal BEFORE the low-pass
// (a0, c0 recomputed here from T and Sigma: subtracting 0.3 again would cost a sub-pixel Gaussian most of its float32 digits, and
// keeping them in Geo would change the default kernels).
struct AaCov { float a0, c0, ratio; };
__device__ __forceinline__ AaCov aa_cov(const Geo &g, const float (&S6)[6], float det) {
    const float Sg[9] = { S6[0], S6[1], S6[2], S6[1], S6[3], S6[4], S6[2], S6[4], S6[5] };
    AaCov r;
    r.a0 = 0.f; r.c0 = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        r.a0 += g.T0[k] * (Sg[3 * k] * g.T0[0] + Sg[3 * k + 1] * g.T0[1] + Sg[3 * k + 2] * g.T0[2]);
        r.c0 += g.T1[k] * (Sg[3 * k] * g.T1[0] + Sg[3 * k + 1] * g.T1[1] + Sg[3 * k + 2] * g.T1[2]);
    }
    r.ratio = (r.a0 * r.c0 - g.cxy * g.cxy) / det;
    return r;
}
__device__ __forceinline__ float aa_comp(const Geo &g, const float (&S6)[6], float det) {
    return sqrtf(fmaxf(DGR_AA_RATIO_FLOOR, aa_cov(g, S6, det).ratio));
}

// ---- pieces shared by the single-view and the batched (dgr_views_*) per-Gaussian kernels --------------------------------
// One Gaussian's inputs out of its warp's staging area (lane = the Gaussian's slot in the warp's run of 32).
template <int DEG, bool RAW>
__device__ __forceinline__ void lds_gaussian(const float *ws, int lane, int M, float3 &p, float3 &s_in, float4 &q_in, float &o_in,
                                             float &dc0, float &dc1, float &dc2, float (&shc)[48]) {
    p = make_float3(ws[kStgMean + 3 * lane], ws[kStgMean + 3 * lane + 1], ws[kStgMean + 3 * lane + 2]);
    s_in = make_float3(ws[kStgScale + 3 * lane], ws[kStgScale + 3 * lane + 1], ws[kStgScale + 3 * lane + 2]);
    q_in = *reinterpret_cast<const float4 *>(ws + kStgRot + 4 * lane);
    o_in = ws[kStgOp + lane];
    if (RAW) {
        dc0 = ws[kStgSh + 3 * lane]; dc1 = ws[kStgSh + 3 * lane + 1]; dc2 = ws[kStgSh + 3 * lane + 2];
        if (DEG > 0) lds_sh_row<DEG, 1>(ws + kStgSh + 96 + lane * (M - 1) * 3, ((M - 1) & 3) == 0, shc);
    } else lds_sh_row<DEG>(ws + kStgSh + lane * M * 3, (M & 3) == 0, shc);
}

// One Gaussian's inputs with per-thread global loads.
template <int DEG, bool HAS_SH, bool HAS_COV, bool RAW>
__device__ __forceinline__ void ldg_gaussian(int g, int M, const float *__restrict__ means3D, const float *__restrict__ shs,
                                             const float *__restrict__ shs_rest, const float *__restrict__ colors_precomp,
                                             const float *__restrict__ opacities, const float *__restrict__ scales,
                                             const float *__restrict__ rotations, const float *__restrict__ cov3D_precomp,
                                             float3 &p, float (&S6)[6], float3 &s_in, float4 &q_in, float &o_in, float &dc0, float &dc1,
                                             float &dc2, float (&shc)[48], float &pc0, float &pc1, float &pc2) {
    p = make_float3(__ldg(means3D + 3 * (size_t)g), __ldg(means3D + 3 * (size_t)g + 1), __ldg(means3D + 3 * (size_t)g + 2));
    if (HAS_COV) {
#pragma unroll
        for (int i = 0; i < 6; i++) S6[i] = __ldg(cov3D_precomp + 6 * (size_t)g + i);
    } else {
        s_in = make_float3(__ldg(scales + 3 * (size_t)g), __ldg(scales + 3 * (size_t)g + 1), __ldg(scales + 3 * (size_t)g + 2));
        q_in = ldg_f4(rotations + 4 * (size_t)g);
    }
    o_in = __ldg(opacities + g);
    if (HAS_SH) {
        if (RAW) {          // _features_dc [P,1,3] + _features_rest [P,M-1,3]: no torch.cat copy
            dc0 = __ldg(shs + 3 * (size_t)g); dc1 = __ldg(shs + 3 * (size_t)g + 1); dc2 = __ldg(shs + 3 * (size_t)g + 2);
            if (DEG > 0) load_sh_row<DEG, 1>(shs_rest + (size_t)g * (M - 1) * 3, ((M - 1) & 3) == 0, shc);
        } else load_sh_row<DEG>(shs + (size_t)g * M * 3, (M & 3) == 0, shc);
    } else {
        pc0 = __ldg(colors_precomp + 3 * (size_t)g); pc1 = __ldg(colors_precomp + 3 * (size_t)g + 1); pc2 = __ldg(colors_precomp + 3 * (size_t)g + 2);
    }
}

// The scale (activated, times scale_modifier), rotation and R the forward uses for (scale, rotation) inputs; raw parameters:
// exp and normalize first, inv_qnorm = 1 / |_rotation| (else 1).
template <bool RAW>
__device__ __forceinline__ void activate_scale_rot(float3 s_in, float4 q_in, float scale_modifier, float3 &s, float4 &q, float &inv_qnorm,
                                                   float (&R)[9]) {
    s = s_in;
    if (RAW) s = make_float3(expf(s.x), expf(s.y), expf(s.z));
    s = make_float3(scale_modifier * s.x, scale_modifier * s.y, scale_modifier * s.z);
    q = q_in;
    inv_qnorm = 1.f;
    if (RAW) q = act_normalize(q, inv_qnorm);
    quat_to_R(q, R);
}

// Sigma from (scale, rotation) inputs (raw parameters: activations first); does not depend on the camera.
template <bool RAW>
__device__ __forceinline__ void cov3d_from_inputs(float3 s_in, float4 q_in, float scale_modifier, float (&S6)[6]) {
    float3 s; float4 q; float inv, R[9];
    activate_scale_rot<RAW>(s_in, q_in, scale_modifier, s, q, inv, R);
    cov3d_from_scale_rot(s, R, S6);
}

// The camera-dependent part of the per-Gaussian forward for a Gaussian in front of the near plane: EWA cov2D, conic, radius,
// pixel mean, SH -> RGB, opacity-aware pixel AABB, packed into the record.  Returns false (outputs untouched) when the Gaussian
// is culled; otherwise the tiles it touches are those of for_each_touched_tile(r.q1.w, r.q2.w, ...).  AA: the record carries the
// compensated opacity (aa_comp) and the opacity-aware pixel AABB is that of the compensated opacity.
template <int DEG, bool HAS_SH, bool RAW, bool AA = false>
__device__ __forceinline__ bool project_gaussian(const FrameConsts &fc, int H, int W, float tanfovx, float tanfovy, const float3 p,
                                                 const float (&S6)[6], float o_in, const float (&shc)[48], float dc0, float dc1, float dc2,
                                                 float pc0, float pc1, float pc2, Rec &r, int &radius_out, unsigned &clamp_flags) {
    const float fx = (float)W / (2.f * tanfovx), fy = (float)H / (2.f * tanfovy);
    Geo geo;
    project_geo(fc, p, S6, fx, fy, DGR_FOV_CLAMP * tanfovx, DGR_FOV_CLAMP * tanfovy, geo);
    const float det = geo.cxx * geo.cyy - geo.cxy * geo.cxy;
    const float mid = 0.5f * (geo.cxx + geo.cyy);
    const float lam = mid + sqrtf(fmaxf(DGR_EIG_FLOOR, mid * mid - det));
    const float rad_f = ceilf(DGR_RADIUS_SIGMAS * sqrtf(lam));
    const float mx = ((geo.ndcx + 1.f) * (float)W - 1.f) * 0.5f;
    const float my = ((geo.ndcy + 1.f) * (float)H - 1.f) * 0.5f;
    // det == 0 is the reference's cull; NaN / non-finite states (undefined upstream) are culled too.
    const bool finite_ok = (det > 0.f) && (fabsf(mx) < 1e9f) && (fabsf(my) < 1e9f) && (rad_f < 1e9f);
    if (!finite_ok) return false;
    const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    // 3-sigma tile rect, truncation toward zero then clamp (reference rule)
    const int rminx = min(gx, max(0, (int)((mx - rad_f) / kTile)));
    const int rminy = min(gy, max(0, (int)((my - rad_f) / kTile)));
    const int rmaxx = min(gx, max(0, (int)((mx + rad_f + (kTile - 1)) / kTile)));
    const int rmaxy = min(gy, max(0, (int)((my + rad_f + (kTile - 1)) / kTile)));
    if (!(rmaxx > rminx && rmaxy > rminy)) return false;
    radius_out = (int)rad_f;
    float o = RAW ? act_sigmoid(o_in) : o_in;
    if (AA) o *= aa_comp(geo, S6, det);
    // colour
    float cr, cg, cb;
    if (HAS_SH) {
        float dx = p.x - fc.cam[0], dy = p.y - fc.cam[1], dz = p.z - fc.cam[2];
        const float il = 1.f / sqrtf(dx * dx + dy * dy + dz * dz);
        dx *= il; dy *= il; dz *= il;
        float b[16]; sh_basis<DEG>(dx, dy, dz, b);
        constexpr int NB = (DEG + 1) * (DEG + 1);
        if (RAW) {
            cr = b[0] * dc0; cg = b[0] * dc1; cb = b[0] * dc2;
#pragma unroll
            for (int k = 1; k < NB; k++) { cr += b[k] * shc[3 * (k - 1)]; cg += b[k] * shc[3 * (k - 1) + 1]; cb += b[k] * shc[3 * (k - 1) + 2]; }
        } else {
            cr = 0.f; cg = 0.f; cb = 0.f;
#pragma unroll
            for (int k = 0; k < NB; k++) { cr += b[k] * shc[3 * k]; cg += b[k] * shc[3 * k + 1]; cb += b[k] * shc[3 * k + 2]; }
        }
        cr += DGR_SH_OFFSET; cg += DGR_SH_OFFSET; cb += DGR_SH_OFFSET;
        // channels clamped at 0 get no colour gradient: remembered in the top bits of `touched`
        clamp_flags = (cr < 0.f ? 1u : 0u) | (cg < 0.f ? 2u : 0u) | (cb < 0.f ? 4u : 0u);
        cr = fmaxf(cr, 0.f); cg = fmaxf(cg, 0.f); cb = fmaxf(cb, 0.f);
    } else {
        cr = pc0; cg = pc1; cb = pc2;
    }
    const float di = 1.f / det;
    const float cA = geo.cyy * di, cB = -geo.cxy * di, cC = geo.cxx * di;
    // opacity-aware pixel AABB: alpha >= 1/255  <=>  d^T conic d <= 2 ln(255 o)
    int bx0 = 1, bx1 = 0, by0 = 1, by1 = 0;
    const float o255 = o * 255.f;
    if (o255 > 1.f) {
        const float tau = 2.f * logf(o255);
        const float ex = sqrtf(tau * geo.cxx) * 1.0005f + 0.02f;
        const float ey = sqrtf(tau * geo.cyy) * 1.0005f + 0.02f;
        const float lim = 1e9f;
        bx0 = max(rminx * kTile, (int)ceilf(fmaxf(mx - ex, -lim)));
        by0 = max(rminy * kTile, (int)ceilf(fmaxf(my - ey, -lim)));
        bx1 = min(min(rmaxx * kTile, W) - 1, (int)floorf(fminf(mx + ex, lim)));
        by1 = min(min(rmaxy * kTile, H) - 1, (int)floorf(fminf(my + ey, lim)));
    }
    if (!(bx0 <= bx1 && by0 <= by1)) { bx0 = 1; bx1 = 0; by0 = 1; by1 = 0; }
    // conic stored as the coefficients of power*log2(e): -0.5 A log2e, -B log2e, -0.5 C log2e
    r.q0 = make_float4(mx, my, cA * (-0.5f * kLog2e), cB * (-kLog2e));
    r.q1 = make_float4(cC * (-0.5f * kLog2e), o, geo.t[2], __uint_as_float((unsigned)bx0 | ((unsigned)bx1 << 16)));
    r.q2 = make_float4(cr, cg, cb, __uint_as_float((unsigned)by0 | ((unsigned)by1 << 16)));
    return true;
}

// End of a per-Gaussian forward block: add the block's tile histogram (shared memory) to the per-tile totals with ONE global
// atomic per touched tile and keep what each atomic returned (where the block's run starts inside the tile) in the block's row
// of the run matrix.
__device__ __forceinline__ void publish_block_histogram(const unsigned *s_hist, int tiles, unsigned *__restrict__ tile_count,
                                                        unsigned *__restrict__ run_matrix) {
    unsigned *row = run_matrix + (size_t)blockIdx.x * tiles;
    constexpr int kB = 12;                               // atomics in flight per thread (800 x 800: all 2500 tiles in ONE round trip)
    for (int t0 = threadIdx.x; t0 < tiles; t0 += kPreThreads * kB) {
        unsigned c[kB], got[kB];
#pragma unroll
        for (int j = 0; j < kB; j++) { const int t = t0 + j * kPreThreads; c[j] = t < tiles ? s_hist[t] : 0u; }
#pragma unroll
        for (int j = 0; j < kB; j++) got[j] = c[j] ? atomicAdd(tile_count + t0 + j * kPreThreads, c[j]) : 0u;
#pragma unroll
        for (int j = 0; j < kB; j++) { const int t = t0 + j * kPreThreads; if (t < tiles) row[t] = got[j]; }
    }
}

// Parameters of the single-view per-Gaussian forward kernels (preprocess_fwd_kernel, and preprocess_fwd_aa_kernel of the
// anti-aliased mode); both compile the body in dgr_preprocess_fwd_body.cuh.
#define DGR_PRE_FWD_PARAMS                                                                                                    \
    int P, int M, int H, int W, float tanfovx, float tanfovy, float scale_modifier, const float *__restrict__ viewmatrix,      \
        const float *__restrict__ projmatrix, const float *__restrict__ campos, const float *__restrict__ means3D,             \
        const float *__restrict__ shs, const float *__restrict__ shs_rest, const float *__restrict__ colors_precomp,           \
        const float *__restrict__ opacities, const float *__restrict__ scales, const float *__restrict__ rotations,            \
        const float *__restrict__ cov3D_precomp, int *__restrict__ radii, Rec *__restrict__ rec, unsigned *__restrict__ touched_out, \
        unsigned *__restrict__ tile_count, unsigned *__restrict__ run_matrix, int tiles, int gpb_iters, int stage_off

template <int DEG, bool HAS_SH, bool HAS_COV, bool RAW, bool STAGE = false>
__global__ void __launch_bounds__(kPreThreads, 3) preprocess_fwd_kernel(DGR_PRE_FWD_PARAMS) {
    constexpr bool AA = false;
#include "dgr_preprocess_fwd_body.cuh"
}
template <int DEG, bool HAS_SH, bool HAS_COV, bool RAW, bool STAGE = false>
__global__ void __launch_bounds__(kPreThreads, 3) preprocess_fwd_aa_kernel(DGR_PRE_FWD_PARAMS) {
    constexpr bool AA = true;
#include "dgr_preprocess_fwd_body.cuh"
}

// ----------------------------------------------------------------------------------------------------------------
// Batched forward (dgr_views_forward_preprocess, dgr_views_mixed_forward_preprocess): ONE cloud, V cameras, each with its own
// image size (ViewTable).  A thread reads its Gaussian's inputs once (bulk-TMA staging or per-thread loads, as above) and then runs
// the camera-dependent part for every camera; the cameras sit in shared memory.  Record r = v P + g, global tile tile_off[v] +
// local tile; the block's histogram spans all tiles of the batch and its run-matrix row is published once.
// ----------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ void load_frames(FrameConsts *fcs, float2 *tan, int V, const float *__restrict__ tanfov,
                                            const float *__restrict__ viewmatrix, const float *__restrict__ projmatrix,
                                            const float *__restrict__ campos) {
    for (int i = threadIdx.x; i < V * 36; i += blockDim.x) {
        const int v = i / 36, k = i - v * 36;
        float x = 0.f;
        if (k < 16) x = __ldg(viewmatrix + 16 * v + k);
        else if (k < 32) x = __ldg(projmatrix + 16 * v + k - 16);
        else if (k < 35) x = __ldg(campos + 3 * v + k - 32);
        reinterpret_cast<float *>(&fcs[v])[k] = x;
    }
    for (int v = threadIdx.x; v < V; v += blockDim.x) tan[v] = make_float2(__ldg(tanfov + 2 * v), __ldg(tanfov + 2 * v + 1));
}

// Parameters of the batched per-Gaussian forward kernels; both compile the body in dgr_preprocess_views_fwd_body.cuh.
#define DGR_VIEWS_FWD_PARAMS                                                                                                  \
    int P, int M, int V, const __grid_constant__ ViewTable vt, float scale_modifier, const float *__restrict__ tanfov,          \
        const float *__restrict__ viewmatrix, const float *__restrict__ projmatrix, const float *__restrict__ campos,          \
        const float *__restrict__ means3D, const float *__restrict__ shs, const float *__restrict__ shs_rest,                  \
        const float *__restrict__ opacities, const float *__restrict__ scales, const float *__restrict__ rotations,            \
        int *__restrict__ radii, Rec *__restrict__ rec, unsigned *__restrict__ touched_out, unsigned *__restrict__ tile_count, \
        unsigned *__restrict__ run_matrix, int gpb_iters, int stage_off

template <int DEG, bool RAW, bool STAGE>
__global__ void __launch_bounds__(kPreThreads, 3) preprocess_views_fwd_kernel(DGR_VIEWS_FWD_PARAMS) {
    constexpr bool AA = false;
#include "dgr_preprocess_views_fwd_body.cuh"
}
template <int DEG, bool RAW, bool STAGE>
__global__ void __launch_bounds__(kPreThreads, 3) preprocess_views_fwd_aa_kernel(DGR_VIEWS_FWD_PARAMS) {
    constexpr bool AA = true;
#include "dgr_preprocess_views_fwd_body.cuh"
}

__global__ void mark_visible_kernel(int P, const float *__restrict__ means3D, const float *__restrict__ V, unsigned char *present) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= P) return;
    const float tz = __ldg(means3D + 3 * (size_t)g) * __ldg(V + 2) + __ldg(means3D + 3 * (size_t)g + 1) * __ldg(V + 6) +
                     __ldg(means3D + 3 * (size_t)g + 2) * __ldg(V + 10) + __ldg(V + 14);
    present[g] = tz > DGR_NEAR_CULL_Z ? 1 : 0;
}

}  // namespace dgr
