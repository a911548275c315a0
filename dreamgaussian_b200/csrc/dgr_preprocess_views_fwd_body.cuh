// dgr_preprocess_views_fwd_body.cuh: the body of preprocess_views_fwd_kernel / preprocess_views_fwd_aa_kernel (dgr_preprocess.cuh).
// Each of those kernels includes it with `constexpr bool AA` defined (false: the default mode, true: the anti-aliased
// mode, DGR_RASTER_ANTIALIAS).  The body is included as text so that the default kernels compile instruction for
// instruction as before the anti-aliased variants existed: a shared __forceinline__ function changed their schedule.
// Not a header: no include guard, no includes of its own.
    extern __shared__ __align__(128) unsigned s_hist[];                 // [tiles of the batch] histogram | STAGE: 8 warp staging areas
    __shared__ FrameConsts s_fc[kMaxViews];
    __shared__ float2 s_tan[kMaxViews];
    __shared__ uint64_t s_stage_bar[kPreThreads / 32];
    pdl_trigger();
    const int lane = threadIdx.x & 31, tiles = vt.tile_off[V];
    float *wstage = STAGE ? reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(s_hist) + stage_off) + (threadIdx.x >> 5) * stage_warp_floats(M)
                          : nullptr;
    uint64_t *wbar = &s_stage_bar[threadIdx.x >> 5];
    unsigned stage_phase = 0;
    bool stage_inflight = false;
    if (STAGE) {
        if (lane == 0) { mbar_init(wbar, 1); mbar_fence_init(); }
        __syncwarp();
        const int g0 = (int)(blockIdx.x * gpb_iters * kPreThreads + (threadIdx.x & ~31u));
        stage_inflight = g0 + 32 <= P;
        if (stage_inflight && lane == 0) stage_issue<RAW>(wstage, wbar, g0, M, means3D, scales, rotations, opacities, shs, shs_rest);
    }
    load_frames(s_fc, s_tan, V, tanfov, viewmatrix, projmatrix, campos);
    for (int t = threadIdx.x; t < tiles; t += kPreThreads) s_hist[t] = 0u;
    __syncthreads();
    for (int it = 0; it < gpb_iters; it++) {
        const int g = (int)((blockIdx.x * gpb_iters + it) * kPreThreads + threadIdx.x);
        float3 p = make_float3(0.f, 0.f, 0.f), s_in = make_float3(0.f, 0.f, 0.f);
        float4 q_in = make_float4(1.f, 0.f, 0.f, 0.f);
        float S6[6], shc[48], o_in = 0.f, dc0 = 0.f, dc1 = 0.f, dc2 = 0.f, unused = 0.f;
        const bool staged = STAGE && stage_inflight;
        if (staged) {
            mbar_wait(wbar, stage_phase); stage_phase ^= 1u;
            lds_gaussian<DEG, RAW>(wstage, lane, M, p, s_in, q_in, o_in, dc0, dc1, dc2, shc);
        }
        if (STAGE) {
            __syncwarp();
            stage_inflight = false;
            if (it + 1 < gpb_iters) {
                const int g0 = (int)((blockIdx.x * gpb_iters + it + 1) * kPreThreads + (threadIdx.x & ~31u));
                stage_inflight = g0 + 32 <= P;
                if (stage_inflight && lane == 0) stage_issue<RAW>(wstage, wbar, g0, M, means3D, scales, rotations, opacities, shs, shs_rest);
            }
        }
        if (g >= P) continue;
        if (!staged)
            ldg_gaussian<DEG, true, false, RAW>(g, M, means3D, shs, shs_rest, nullptr, opacities, scales, rotations, nullptr, p, S6, s_in, q_in,
                                                o_in, dc0, dc1, dc2, shc, unused, unused, unused);
        cov3d_from_inputs<RAW>(s_in, q_in, scale_modifier, S6);
        for (int v = 0; v < V; v++) {
            const FrameConsts &fc = s_fc[v];
            unsigned touched = 0, clamp_flags = 0;
            int radius_out = 0;
            Rec r;
            r.q0 = make_float4(0.f, 0.f, 0.f, 0.f); r.q1 = r.q0; r.q2 = r.q0;
            const float tzc = p.x * fc.V[2] + p.y * fc.V[6] + p.z * fc.V[10] + fc.V[14];
            if (tzc > DGR_NEAR_CULL_Z) {
                const float2 tf = s_tan[v];
                if (project_gaussian<DEG, true, RAW, AA>(fc, vt.H[v], vt.W[v], tf.x, tf.y, p, S6, o_in, shc, dc0, dc1, dc2, 0.f, 0.f, 0.f, r,
                                                         radius_out, clamp_flags)) {
                    unsigned *vh = s_hist + vt.tile_off[v];
                    for_each_touched_tile(__float_as_uint(r.q1.w), __float_as_uint(r.q2.w), vt.gx[v], [&](int t) { atomicAdd(&vh[t], 1u); touched++; });
                }
            }
            const size_t rid = (size_t)v * P + g;
            radii[rid] = radius_out;
            rec[rid] = r;
            touched_out[rid] = touched | (clamp_flags << 29);
        }
    }
    __syncthreads();
    publish_block_histogram(s_hist, tiles, tile_count, run_matrix);
