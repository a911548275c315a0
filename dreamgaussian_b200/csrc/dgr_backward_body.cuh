// dgr_backward_body.cuh: the body of preprocess_bwd_kernel / preprocess_bwd_aa_kernel (dgr_backward.cuh).
// Each of those kernels includes it with `constexpr bool AA` defined (false: the default mode, true: the anti-aliased
// mode, DGR_RASTER_ANTIALIAS).  The body is included as text so that the default kernels compile instruction for
// instruction as before the anti-aliased variants existed: a shared __forceinline__ function changed their schedule.
// Not a header: no include guard, no includes of its own.
    __shared__ FrameConsts fc;
    __shared__ __align__(16) float s_stage[STAGE ? 4 : (kPreThreads / 32) * kStageFloats];
    __shared__ uint64_t s_stage_bar[kPreThreads / 32];
    extern __shared__ __align__(128) float s_dyn[];              // STAGE: 8 warps x warp_smem_floats (>= kStageFloats)
    static_assert(!STAGE || (HAS_SH && !HAS_COV), "input staging: SH + scale / rotation inputs only");
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    bool staged = false;                                         // warp-uniform: all 32 Gaussians of this warp exist and are staged
    if (STAGE) {
        const int g0 = (int)(blockIdx.x * blockDim.x + (threadIdx.x & ~31u));
        uint64_t *wbar = &s_stage_bar[threadIdx.x >> 5];
        staged = g0 + 32 <= P;
        if ((threadIdx.x & 31) == 0) {
            mbar_init(wbar, 1); mbar_fence_init();
            if (staged) stage_issue<RAW>(s_dyn + (threadIdx.x >> 5) * warp_smem_floats, wbar, g0, M, means3D, scales, rotations, opacities, shs, shs_rest);
        }
        __syncwarp();
    }
    load_frame(fc, viewmatrix, projmatrix, HAS_SH ? campos : nullptr);
    __syncthreads();
    const bool acc = accumulate != 0;
    const bool in_range = g < P;
    // gradient rows of Gaussians another rank owns go to that rank's staging slot (what the local buffer has accumulated over
    // this rank's earlier views of the iteration + this view); every row is written then, culled Gaussians included
    const long long delta = push.per > 0 ? push.delta[(blockIdx.x * blockDim.x) / (unsigned)push.per] : 0;
    const bool pushing = delta != 0;
    float *ws = STAGE ? s_dyn + (threadIdx.x >> 5) * warp_smem_floats
                      : s_stage + (threadIdx.x >> 5) * kStageFloats;   // this warp's output image (see warp_flush)
    const int lane = threadIdx.x & 31;
    // every input of this Gaussian is requested up front (one memory round trip; none of it depends on the backward render)
    int radius_in = 0;
    unsigned touched_in = 0;
    float3 p = make_float3(0.f, 0.f, 0.f), s_in = make_float3(0.f, 0.f, 0.f);
    float4 q_in = make_float4(1.f, 0.f, 0.f, 0.f);
    float o_in = 0.f, S6[6], shc[48];
    if (in_range) {
        radius_in = radii[g];
        touched_in = __ldg(touched + g);
    }
    if (staged) {
        mbar_wait(&s_stage_bar[threadIdx.x >> 5], 0u);
        p = make_float3(ws[kStgMean + 3 * lane], ws[kStgMean + 3 * lane + 1], ws[kStgMean + 3 * lane + 2]);
        s_in = make_float3(ws[kStgScale + 3 * lane], ws[kStgScale + 3 * lane + 1], ws[kStgScale + 3 * lane + 2]);
        q_in = *reinterpret_cast<const float4 *>(ws + kStgRot + 4 * lane);
        o_in = ws[kStgOp + lane];
        if (RAW) { if (DEG > 0) lds_sh_row<DEG, 1>(ws + kStgSh + 96 + lane * (M - 1) * 3, ((M - 1) & 3) == 0, shc); }
        else lds_sh_row<DEG>(ws + kStgSh + lane * M * 3, (M & 3) == 0, shc);
    }
    if (STAGE) __syncwarp();             // every lane has its inputs in registers: from here on the slice is the warp's output image
    if (in_range && !staged) {
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
            if (RAW) { if (DEG > 0) load_sh_row<DEG, 1>(shs_rest + (size_t)g * (M - 1) * 3, ((M - 1) & 3) == 0, shc); }       // d basis_0 = 0
            else load_sh_row<DEG>(shs + (size_t)g * M * 3, (M & 3) == 0, shc);
        }
    }
    const bool visible = in_range && radius_in > 0;
    float bs[16];
    float gr[3] = { 0.f, 0.f, 0.f };
#pragma unroll
    for (int k = 0; k < 16; k++) bs[k] = 0.f;

    if (!visible) {                                                 // culled (or past the end): a zero row in every segment
#pragma unroll
        for (int k = 0; k < 3; k++) { ws[kOut3D + 3 * lane + k] = 0.f; ws[kOut2D + 3 * lane + k] = 0.f; ws[kOutScale + 3 * lane + k] = 0.f; }
        ws[kOutOp + lane] = 0.f;
        *reinterpret_cast<float4 *>(ws + kOutRot + 4 * lane) = make_float4(0.f, 0.f, 0.f, 0.f);
        if (HAS_COV) { for (int k = 0; k < 6; k++) ws[kOutCov + 6 * lane + k] = 0.f; }
        if (!HAS_SH) { for (int k = 0; k < 3; k++) ws[kOutCol + 3 * lane + k] = 0.f; }
    }
    if (visible) {
        float R[9];
        float3 s = make_float3(0.f, 0.f, 0.f);
        float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
        float inv_qnorm = 1.f;
        if (!HAS_COV) {
            s = s_in;
            if (RAW) s = make_float3(expf(s.x), expf(s.y), expf(s.z));
            s = make_float3(scale_modifier * s.x, scale_modifier * s.y, scale_modifier * s.z);
            q = q_in;
            if (RAW) q = act_normalize(q, inv_qnorm);
            quat_to_R(q, R);
            cov3d_from_scale_rot(s, R, S6);
        }
        const float fx = (float)W / (2.f * tanfovx), fy = (float)H / (2.f * tanfovy);
        Geo geo;
        project_geo(fc, p, S6, fx, fy, DGR_FOV_CLAMP * tanfovx, DGR_FOV_CLAMP * tanfovy, geo);
        const float a = geo.cxx, b = geo.cxy, c = geo.cyy;
        const float det = a * c - b * b, di = 1.f / det;
        const float cA = c * di, cB = -b * di, cC = a * di;
        const float o = RAW ? act_sigmoid(o_in) : o_in;

        // Everything above reads only the op's inputs: under a programmatic dependent launch it overlaps the tail of the
        // backward render kernel.  The moments that kernel accumulates are complete after this point.
        pdl_wait();
        const float4 m0 = ldg_f4(grad_rec + (size_t)g * kGradRecFloats);
        const float4 m1 = ldg_f4(grad_rec + (size_t)g * kGradRecFloats + 4);
        const float4 m2 = ldg_f4(grad_rec + (size_t)g * kGradRecFloats + 8);
        // moments: m0 = {u, u dx, u dy, u dx^2}, m1 = {u dx dy, u dy^2, wr, wg}, m2 = {wb, wd, -, -}

        // pixel-space mean gradient and conic gradient from the moments
        const float gpx = -(cA * m0.y + cB * m0.z), gpy = -(cC * m0.z + cB * m0.y);
        const float gA = -0.5f * m0.w, gB = -m1.x, gC = -0.5f * m1.y;
        const float g_op = (o != 0.f) ? m0.x / o : 0.f;
        const float g_rgb[3] = { m1.z, m1.w, m2.x };
        const float g_depth = m2.y;

        float dmean[3] = { 0.f, 0.f, 0.f };
        // (1) mean_px through the full projection; reported means2D grad is in NDC units
        const float gndx = gpx * 0.5f * (float)W, gndy = gpy * 0.5f * (float)H;
        ws[kOut2D + 3 * lane] = gndx; ws[kOut2D + 3 * lane + 1] = gndy; ws[kOut2D + 3 * lane + 2] = 0.f;
        // densification bookkeeping of the training loop (gs_renderer.py:625-627, main.py:279-281), for visible Gaussians:
        // xyz_gradient_accum += |d L / d means2D[:, :2]| of THIS render, denom += 1, max_radii2D = max(max_radii2D, radii)
        if (xyz_gradient_accum) xyz_gradient_accum[g] += sqrtf(gndx * gndx + gndy * gndy);
        if (denom) denom[g] += 1.f;
        if (max_radii2D) max_radii2D[g] = fmaxf(max_radii2D[g], (float)radius_in);
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
            const unsigned flags = touched_in >> 29;                     // SH channels the forward clamped at 0
#pragma unroll
            for (int ch = 0; ch < 3; ch++) gr[ch] = ((flags >> ch) & 1u) ? 0.f : g_rgb[ch];
            float ddx = 0.f, ddy = 0.f, ddz = 0.f;
            constexpr int NB = (DEG + 1) * (DEG + 1);
#pragma unroll
            for (int k = 1; k < NB; k++) {                                // d basis_0 = 0
                const int off = RAW ? 3 * (k - 1) : 3 * k;
                const float dotc = shc[off] * gr[0] + shc[off + 1] * gr[1] + shc[off + 2] * gr[2];
                float bx, by, bz;
                sh_dbasis(k, dx, dy, dz, bx, by, bz);
                ddx += bx * dotc; ddy += by * dotc; ddz += bz * dotc;
            }
            const float dot = dx * ddx + dy * ddy + dz * ddz;
            dmean[0] += (ddx - dx * dot) * il; dmean[1] += (ddy - dy * dot) * il; dmean[2] += (ddz - dz * dot) * il;
        } else {
#pragma unroll
            for (int ch = 0; ch < 3; ch++) ws[kOutCol + 3 * lane + ch] = g_rgb[ch];
        }
        ws[kOutOp + lane] = RAW ? g_op * o * (1.f - o) : g_op;                                              // sigmoid'

        // (2) conic -> cov2D -> (Sigma, T = J Rwv)
        const float d2 = di * di;
        float ga = d2 * (-c * c * gA + b * c * gB - b * b * gC);
        float gc = d2 * (-b * b * gA + a * b * gB - a * a * gC);
        float gb = d2 * (2.f * b * c * gA - (det + 2.f * b * b) * gB + 2.f * a * b * gC);
        if (AA) aa_conic_grads(geo, S6, det, m0.x, ga, gb, gc);
        const float G00 = ga, G01 = 0.5f * gb, G11 = gc;
        const float *T0 = geo.T0, *T1 = geo.T1;
        float dS[9];
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
#pragma unroll
        for (int k = 0; k < 3; k++) ws[kOut3D + 3 * lane + k] = dmean[k];
        if (HAS_COV) {
            float *out = ws + kOutCov + 6 * lane;
            out[0] = dS[0]; out[1] = 2.f * dS[1]; out[2] = 2.f * dS[2]; out[3] = dS[4]; out[4] = 2.f * dS[5]; out[5] = dS[8];
        } else {
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
                ws[kOutScale + 3 * lane + k] = RAW ? v * sv[k] : v * scale_modifier;                                   // exp' = exp
            }
            {
                const float r = q.x, x = q.y, y = q.z, z = q.w;
                float dq[4];
                dq[0] = 2.f * (-z * dR[1] + y * dR[2] + z * dR[3] - x * dR[5] - y * dR[6] + x * dR[7]);
                dq[1] = 2.f * (y * dR[1] + z * dR[2] + y * dR[3] - 2.f * x * dR[4] - r * dR[5] + z * dR[6] + r * dR[7] - 2.f * x * dR[8]);
                dq[2] = 2.f * (-2.f * y * dR[0] + x * dR[1] + r * dR[2] + x * dR[3] + z * dR[5] - r * dR[6] + z * dR[7] - 2.f * y * dR[8]);
                dq[3] = 2.f * (-2.f * z * dR[0] - r * dR[1] + x * dR[2] + r * dR[3] - 2.f * z * dR[4] + y * dR[5] + x * dR[6] + y * dR[7]);
                if (RAW) {          // q = raw / |raw|:  d raw = (dq - q (q . dq)) / |raw|
                    const float qd = r * dq[0] + x * dq[1] + y * dq[2] + z * dq[3];
                    dq[0] = (dq[0] - r * qd) * inv_qnorm; dq[1] = (dq[1] - x * qd) * inv_qnorm;
                    dq[2] = (dq[2] - y * qd) * inv_qnorm; dq[3] = (dq[3] - z * qd) * inv_qnorm;
                }
                *reinterpret_cast<float4 *>(ws + kOutRot + 4 * lane) = make_float4(dq[0], dq[1], dq[2], dq[3]);
            }
        }
    }
    // ---- the warp's rows leave together (see warp_flush); rows past the end of the arrays are not written
    __syncwarp();
    {
        const int row_base = (int)(blockIdx.x * blockDim.x) + (int)(threadIdx.x & ~31u);
        const int nrows = min(32, P - row_base);
        if (nrows > 0) {
            warp_flush(dL_dmeans3D, 3, delta, row_base, nrows, acc, ws + kOut3D);
            warp_flush(dL_dmeans2D, 3, delta, row_base, nrows, acc, ws + kOut2D);
            warp_flush(dL_dopacities, 1, delta, row_base, nrows, acc, ws + kOutOp);
            if (!HAS_COV) {
                warp_flush(dL_dscales, 3, delta, row_base, nrows, acc, ws + kOutScale);
                warp_flush(dL_drotations, 4, delta, row_base, nrows, acc, ws + kOutRot);
            } else warp_flush(dL_dcov3D, 6, delta, row_base, nrows, acc, ws + kOutCov);
            if (!HAS_SH) warp_flush(dL_dcolors, 3, delta, row_base, nrows, acc, ws + kOutCol);
        }
        __syncwarp();
        if (HAS_SH && RAW) {
            if (dL_dshs && nrows > 0) {           // _features_dc gradient [P,1,3] (zero for culled Gaussians: bs = gr = 0)
#pragma unroll
                for (int ch = 0; ch < 3; ch++) ws[3 * lane + ch] = bs[0] * gr[ch];
                __syncwarp();
                warp_flush(dL_dshs, 3, delta, row_base, nrows, acc, ws);
                __syncwarp();
            }
            if (dL_dshs_rest && M > 1) store_sh_grads<DEG, 1>(dL_dshs_rest, P, M, bs, gr, acc, ws, delta);
        } else if (HAS_SH && dL_dshs) store_sh_grads<DEG>(dL_dshs, P, M, bs, gr, acc, ws, delta);
    }
    if (pushing) __threadfence_system();          // the rows are in the owner's memory when this grid completes
