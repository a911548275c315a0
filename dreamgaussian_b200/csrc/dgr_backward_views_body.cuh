// dgr_backward_views_body.cuh: the body of preprocess_views_bwd_kernel / preprocess_views_bwd_aa_kernel (dgr_backward.cuh).
// Each of those kernels includes it with `constexpr bool AA` defined (false: the default mode, true: the anti-aliased
// mode, DGR_RASTER_ANTIALIAS).  The body is included as text so that the default kernels compile instruction for
// instruction as before the anti-aliased variants existed: a shared __forceinline__ function changed their schedule.
// Not a header: no include guard, no includes of its own.
    __shared__ FrameConsts s_fc[kMaxViews];
    __shared__ float2 s_tan[kMaxViews];
    __shared__ __align__(16) float s_stage[(kPreThreads / 32) * kStageFloats];
    constexpr int NB = (DEG + 1) * (DEG + 1);
    load_frames(s_fc, s_tan, V, tanfov, viewmatrix, projmatrix, campos);
    __syncthreads();
    const int g = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
    const bool acc = accumulate != 0;
    float *ws = s_stage + (threadIdx.x >> 5) * kStageFloats;
    float3 p = make_float3(0.f, 0.f, 0.f), s_in = make_float3(0.f, 0.f, 0.f);
    float4 q_in = make_float4(1.f, 0.f, 0.f, 0.f);
    float o_in = 0.f;
    if (g < P) {
        p = make_float3(__ldg(means3D + 3 * (size_t)g), __ldg(means3D + 3 * (size_t)g + 1), __ldg(means3D + 3 * (size_t)g + 2));
        s_in = make_float3(__ldg(scales + 3 * (size_t)g), __ldg(scales + 3 * (size_t)g + 1), __ldg(scales + 3 * (size_t)g + 2));
        q_in = ldg_f4(rotations + 4 * (size_t)g);
        o_in = __ldg(opacities + g);
    }
    // the SH row is re-read per view (L1) instead of being held in registers next to the gradient sums
    const float *shrow = RAW ? shs_rest + (size_t)g * (M - 1) * 3 : shs + (size_t)g * M * 3;
    float R[9], S6[6], inv_qnorm;
    float3 s;
    float4 q;
    activate_scale_rot<RAW>(s_in, q_in, scale_modifier, s, q, inv_qnorm, R);
    cov3d_from_scale_rot(s, R, S6);
    const float o = RAW ? act_sigmoid(o_in) : o_in;

    float sum_mean[3] = { 0.f, 0.f, 0.f }, sum_dS[9], sum_op = 0.f, sum_sh[3 * NB];
#pragma unroll
    for (int k = 0; k < 9; k++) sum_dS[k] = 0.f;
#pragma unroll
    for (int k = 0; k < 3 * NB; k++) sum_sh[k] = 0.f;
    pdl_wait();                          // the moments of the batched backward render
    for (int v = 0; v < V && g < P; v++) {
        const size_t rid = (size_t)v * P + g;
        float gndx = 0.f, gndy = 0.f;
        const int radius_v = radii[rid];
        if (radius_v > 0) {
            const float2 tf = s_tan[v];
            float dmean[3], g_op, g_rgb[3], dS[9], bs[16], gr[3];
            backward_camera<DEG, true, RAW, AA>(s_fc[v], vt.H[v], vt.W[v], tf.x, tf.y, p, S6, o, __ldg(touched + rid) >> 29,
                [&](float4 &m0, float4 &m1, float4 &m2) {
                    m0 = ldg_f4(grad_rec + rid * kGradRecFloats);
                    m1 = ldg_f4(grad_rec + rid * kGradRecFloats + 4);
                    m2 = ldg_f4(grad_rec + rid * kGradRecFloats + 8);
                },
                [&](int i) { return __ldg(shrow + i); }, gndx, gndy, dmean, g_op, g_rgb, dS, bs, gr);
#pragma unroll
            for (int k = 0; k < 3; k++) sum_mean[k] += dmean[k];
#pragma unroll
            for (int k = 0; k < 9; k++) sum_dS[k] += dS[k];
            sum_op += g_op;
#pragma unroll
            for (int k = 0; k < NB; k++)
#pragma unroll
                for (int ch = 0; ch < 3; ch++) sum_sh[3 * k + ch] = __fmaf_rn(bs[k], gr[ch], sum_sh[3 * k + ch]);
            if ((stats_views >> v) & 1ull) {
                if (xyz_gradient_accum) xyz_gradient_accum[g] += sqrtf(gndx * gndx + gndy * gndy);
                if (denom) denom[g] += 1.f;
                if (max_radii2D) max_radii2D[g] = fmaxf(max_radii2D[g], (float)radius_v);
            }
        }
        if (dL_dmeans2D) {
            float *m2d = dL_dmeans2D + rid * 3;
            if (acc) { gndx += m2d[0]; gndy += m2d[1]; }
            m2d[0] = gndx; m2d[1] = gndy; m2d[2] = acc ? m2d[2] : 0.f;
        }
    }
    float dsc[3] = { 0.f, 0.f, 0.f }, dq[4] = { 0.f, 0.f, 0.f, 0.f };
    backward_scale_rot<RAW>(sum_dS, R, s, q, inv_qnorm, scale_modifier, dsc, dq);
#pragma unroll
    for (int k = 0; k < 3; k++) { ws[kOut3D + 3 * lane + k] = sum_mean[k]; ws[kOutScale + 3 * lane + k] = dsc[k]; }
    ws[kOutOp + lane] = RAW ? sum_op * o * (1.f - o) : sum_op;
    *reinterpret_cast<float4 *>(ws + kOutRot + 4 * lane) = make_float4(dq[0], dq[1], dq[2], dq[3]);
    __syncwarp();
    const int row_base = (int)(blockIdx.x * blockDim.x) + (int)(threadIdx.x & ~31u);
    const int nrows = min(32, P - row_base);
    if (nrows > 0) {
        warp_flush(dL_dmeans3D, 3, 0, row_base, nrows, acc, ws + kOut3D);
        warp_flush(dL_dopacities, 1, 0, row_base, nrows, acc, ws + kOutOp);
        warp_flush(dL_dscales, 3, 0, row_base, nrows, acc, ws + kOutScale);
        warp_flush(dL_drotations, 4, 0, row_base, nrows, acc, ws + kOutRot);
    }
    if (g >= P) return;
    // SH rows: coefficients 0 .. NB-1 from the sums, the rest of the row (M > NB) zero
    auto put = [&](float *dst, float v) { *dst = acc ? *dst + v : v; };
    if (RAW) {
        if (dL_dshs) {
#pragma unroll
            for (int ch = 0; ch < 3; ch++) put(dL_dshs + 3 * (size_t)g + ch, sum_sh[ch]);
        }
        if (dL_dshs_rest && M > 1) {
            float *row = dL_dshs_rest + (size_t)g * (M - 1) * 3;
#pragma unroll
            for (int k = 3; k < 3 * NB; k++) put(row + k - 3, sum_sh[k]);
            for (int k = 3 * NB; k < 3 * M; k++) put(row + k - 3, 0.f);
        }
    } else if (dL_dshs) {
        float *row = dL_dshs + (size_t)g * M * 3;
#pragma unroll
        for (int k = 0; k < 3 * NB; k++) put(row + k, sum_sh[k]);
        for (int k = 3 * NB; k < 3 * M; k++) put(row + k, 0.f);
    }
