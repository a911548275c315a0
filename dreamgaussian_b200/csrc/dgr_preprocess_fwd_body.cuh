// dgr_preprocess_fwd_body.cuh: the body of preprocess_fwd_kernel / preprocess_fwd_aa_kernel (dgr_preprocess.cuh).
// Each of those kernels includes it with `constexpr bool AA` defined (false: the default mode, true: the anti-aliased
// mode, DGR_RASTER_ANTIALIAS).  The body is included as text so that the default kernels compile instruction for
// instruction as before the anti-aliased variants existed: a shared __forceinline__ function changed their schedule.
// Not a header: no include guard, no includes of its own.
    // Per-block tile histogram in shared memory (native integer smem atomics); at the end every touched tile's count is
    // added to the per-tile totals with ONE global atomic per (block, tile) — not one per instance — and what the atomic
    // returns (where this block's run starts inside the tile's range) goes into the block's row of the run matrix.
    extern __shared__ __align__(128) unsigned s_hist[];
    __shared__ FrameConsts fc;
    __shared__ uint64_t s_stage_bar[kPreThreads / 32];
    static_assert(!STAGE || (HAS_SH && !HAS_COV), "input staging: SH + scale / rotation inputs only");
    pdl_trigger();                       // the tile scan may become resident now (it waits for this grid's completion)
    // STAGE: this warp's inputs of the first block iteration are on their way before anything else happens
    const int lane = threadIdx.x & 31;
    float *wstage = STAGE ? reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(s_hist) + stage_off) + (threadIdx.x >> 5) * stage_warp_floats(M)
                          : nullptr;
    uint64_t *wbar = &s_stage_bar[threadIdx.x >> 5];
    unsigned stage_phase = 0;
    bool stage_inflight = false;         // warp-uniform: the copies of the NEXT block iteration have been started
    if (STAGE) {
        if (lane == 0) { mbar_init(wbar, 1); mbar_fence_init(); }
        __syncwarp();
        const int g0 = (int)(blockIdx.x * gpb_iters * kPreThreads + (threadIdx.x & ~31u));
        stage_inflight = g0 + 32 <= P;
        if (stage_inflight && lane == 0) stage_issue<RAW>(wstage, wbar, g0, M, means3D, scales, rotations, opacities, shs, shs_rest);
    }
    load_frame(fc, viewmatrix, projmatrix, HAS_SH ? campos : nullptr);
    for (int t = threadIdx.x; t < tiles; t += kPreThreads) s_hist[t] = 0u;
    __syncthreads();
    for (int it = 0; it < gpb_iters; it++) {
    const int g = (int)((blockIdx.x * gpb_iters + it) * kPreThreads + threadIdx.x);
    unsigned touched = 0, clamp_flags = 0;
    // every input of this Gaussian is requested before anything is computed (one memory round trip)
    float3 p = make_float3(0.f, 0.f, 0.f);
    float S6[6];
    float3 s_in = make_float3(0.f, 0.f, 0.f);
    float4 q_in = make_float4(1.f, 0.f, 0.f, 0.f);
    float o_in = 0.f;
    float shc[48], dc0 = 0.f, dc1 = 0.f, dc2 = 0.f, pc0 = 0.f, pc1 = 0.f, pc2 = 0.f;
    const bool staged = STAGE && stage_inflight;                      // warp-uniform: all 32 Gaussians of this warp exist and are staged
    if (staged) {
        mbar_wait(wbar, stage_phase); stage_phase ^= 1u;
        p = make_float3(wstage[kStgMean + 3 * lane], wstage[kStgMean + 3 * lane + 1], wstage[kStgMean + 3 * lane + 2]);
        s_in = make_float3(wstage[kStgScale + 3 * lane], wstage[kStgScale + 3 * lane + 1], wstage[kStgScale + 3 * lane + 2]);
        q_in = *reinterpret_cast<const float4 *>(wstage + kStgRot + 4 * lane);
        o_in = wstage[kStgOp + lane];
        if (RAW) {
            dc0 = wstage[kStgSh + 3 * lane]; dc1 = wstage[kStgSh + 3 * lane + 1]; dc2 = wstage[kStgSh + 3 * lane + 2];
            if (DEG > 0) lds_sh_row<DEG, 1>(wstage + kStgSh + 96 + lane * (M - 1) * 3, ((M - 1) & 3) == 0, shc);
        } else lds_sh_row<DEG>(wstage + kStgSh + lane * M * 3, (M & 3) == 0, shc);
    }
    if (STAGE) {
        __syncwarp();                    // every lane has its values in registers: the staging area is free for the next block iteration
        stage_inflight = false;
        if (it + 1 < gpb_iters) {
            const int g0 = (int)((blockIdx.x * gpb_iters + it + 1) * kPreThreads + (threadIdx.x & ~31u));
            stage_inflight = g0 + 32 <= P;
            if (stage_inflight && lane == 0) stage_issue<RAW>(wstage, wbar, g0, M, means3D, scales, rotations, opacities, shs, shs_rest);
        }
    }
    if (g < P) {
        int radius_out = 0;
        Rec r;
        r.q0 = make_float4(0.f, 0.f, 0.f, 0.f); r.q1 = r.q0; r.q2 = r.q0;
        if (!staged) {
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
        const float tzc = p.x * fc.V[2] + p.y * fc.V[6] + p.z * fc.V[10] + fc.V[14];
        if (tzc > DGR_NEAR_CULL_Z) {
            if (!HAS_COV) {
                float3 s = s_in;
                if (RAW) s = make_float3(expf(s.x), expf(s.y), expf(s.z));
                s = make_float3(scale_modifier * s.x, scale_modifier * s.y, scale_modifier * s.z);
                float4 q = q_in;
                if (RAW) { float inv; q = act_normalize(q, inv); }
                float R[9]; quat_to_R(q, R);
                cov3d_from_scale_rot(s, R, S6);
            }
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
            if (finite_ok) {
                const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
                // 3-sigma tile rect, truncation toward zero then clamp (reference rule)
                const int rminx = min(gx, max(0, (int)((mx - rad_f) / kTile)));
                const int rminy = min(gy, max(0, (int)((my - rad_f) / kTile)));
                const int rmaxx = min(gx, max(0, (int)((mx + rad_f + (kTile - 1)) / kTile)));
                const int rmaxy = min(gy, max(0, (int)((my + rad_f + (kTile - 1)) / kTile)));
                if (rmaxx > rminx && rmaxy > rminy) {
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
                    // per-tile instance histogram of this block
                    for_each_touched_tile(__float_as_uint(r.q1.w), __float_as_uint(r.q2.w), gx,
                                          [&](int t) { atomicAdd(&s_hist[t], 1u); touched++; });
                }
            }
        }
        radii[g] = radius_out;
        rec[g] = r;
        touched_out[g] = touched | (clamp_flags << 29);     // tiles touched (29 bits) | SH clamp flags (3 bits)
    }
    }
    __syncthreads();
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
