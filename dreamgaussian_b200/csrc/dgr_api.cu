// dgr_api.cu — C ABI of libdgr_b200.so (see include/dgr_b200.h).  Host-side glue only: argument checks, scratch
// layout, kernel launches on the caller's stream.  No torch, no library kernels (no CUB/cuBLAS), no CPU fallback:
// without a CUDA device every compute entry point fails with an error string.
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <atomic>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/dgr_b200.h"
#include "dgr_absgrad.cuh"
#include "dgr_backward.cuh"
#include "dgr_binning.cuh"
#include "dgr_camgrad.cuh"
#include "dgr_collective.cuh"
#include "dgr_densify.cuh"
#include "dgr_det.cuh"
#include "dgr_knn.cuh"
#include "dgr_fields.cuh"
#include "dgr_optim.cuh"
#include "dgr_common.cuh"
#include "dgr_preprocess.cuh"
#include "dgr_render.cuh"

using namespace dgr;

namespace {
thread_local std::string g_err;
thread_local uint64_t g_launches = 0;

// NVTX range around every C-ABI entry point (SURVEY.md §5: tracing): header-only NVTX v3, a no-op unless a tool is attached
struct NvtxRange {
    explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

int fail(int code, const char *what, const char *detail = nullptr) {
    g_err = what;
    if (detail) { g_err += ": "; g_err += detail; }
    return code;
}

// optional per-kernel CUDA-event timing (bench.py's live roofline): events bracket every launch on its stream
struct ProfRec { const char *name; cudaEvent_t a, b; };
thread_local bool g_prof_on = false;
thread_local std::vector<ProfRec> g_prof;
inline void prof_begin(const char *name, cudaStream_t st) {
    if (!g_prof_on) return;
    ProfRec r; r.name = name;
    cudaEventCreate(&r.a); cudaEventCreate(&r.b);
    cudaEventRecord(r.a, st);
    g_prof.push_back(r);
}
inline void prof_end(cudaStream_t st) {
    if (!g_prof_on) return;
    cudaEventRecord(g_prof.back().b, st);
}

#define DGR_CUDA(call)                                                                         \
    do {                                                                                       \
        cudaError_t e_ = (call);                                                               \
        if (e_ != cudaSuccess) return fail((int)e_, #call, cudaGetErrorString(e_));            \
    } while (0)
// launch a kernel (the statement in __VA_ARGS__), count it, time it when profiling, check it
#define DGR_KERNEL(name, st, dbg, ...)                                                         \
    do {                                                                                       \
        prof_begin(name, st);                                                                  \
        __VA_ARGS__;                                                                           \
        prof_end(st);                                                                          \
        g_launches++;                                                                          \
        cudaError_t e_ = cudaGetLastError();                                                   \
        if (e_ != cudaSuccess) return fail((int)e_, name, cudaGetErrorString(e_));             \
        if (dbg) { e_ = cudaStreamSynchronize(st);                                             \
            if (e_ != cudaSuccess) return fail((int)e_, name, cudaGetErrorString(e_)); }       \
    } while (0)

// Kernel launch with the programmatic-dependent-launch attribute: the kernel may become resident while its predecessor in
// the stream (which must be a kernel, not a copy / memset / event) is still running; it calls pdl_wait() before it touches
// anything the predecessor produces.  g_pdl = 0 (DGR_PDL=0 or dgr_set_tuning bit 3) launches the same kernels the ordinary way.
std::atomic<int> g_pdl{-1};
bool pdl_enabled() {
    int v = g_pdl.load();
    if (v < 0) { const char *e = getenv("DGR_PDL"); v = (e && e[0] == '0') ? 0 : 1; g_pdl = v; }
    return v != 0;
}
template <class... KArgs, class... Args>
void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args &&...args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    const bool on = pdl && pdl_enabled();
    cfg.attrs = on ? attr : nullptr; cfg.numAttrs = on ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);       // errors surface through cudaGetLastError in DGR_KERNEL
}

int check_settings(const DgrSettings *s) {
    if (!s) return fail(-1, "settings is NULL");
    if (s->image_height <= 0 || s->image_width <= 0) return fail(-1, "image size must be positive");
    if (s->image_height > 65535 || s->image_width > 65535) return fail(-1, "image size above 65535 not supported");
    if (s->sh_degree < 0 || s->sh_degree > 3) return fail(-1, "sh_degree must be 0..3");
    if (!s->bg || !s->viewmatrix || !s->projmatrix) return fail(-1, "bg / viewmatrix / projmatrix must not be NULL");
    return 0;
}
int check_gaussians(const DgrSettings *s, const DgrGaussians *g) {
    if (!g) return fail(-1, "gaussians is NULL");
    if (g->P < 0) return fail(-1, "P < 0");
    if (g->P == 0) return 0;                       // empty cloud: empty tensors have NULL data pointers
    if ((g->shs == nullptr) == (g->colors_precomp == nullptr))
        return fail(-2, "Please provide excatly one of either SHs or precomputed colors!");
    if (((g->scales == nullptr || g->rotations == nullptr) && g->cov3D_precomp == nullptr) ||
        ((g->scales != nullptr || g->rotations != nullptr) && g->cov3D_precomp != nullptr))
        return fail(-2, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    if (g->P > 0 && (!g->means3D || !g->opacities)) return fail(-1, "means3D / opacities must not be NULL");
    if (g->activations) {
        if (!g->shs || g->cov3D_precomp || !g->scales || !g->rotations)
            return fail(-2, "activations: raw parameters need features_dc (shs), scaling and rotation; no cov3D_precomp");
        if (g->M > 1 && !g->shs_rest) return fail(-2, "activations: shs_rest (_features_rest) is NULL but M > 1");
    }
    if (g->shs) {
        if (!s->campos) return fail(-1, "campos must not be NULL with SHs");
        const int nb = (s->sh_degree + 1) * (s->sh_degree + 1);
        if (g->M < nb) return fail(-1, "shs has fewer coefficients than sh_degree needs");
        if (g->M > 16) return fail(-1, "shs with more than 16 coefficients per channel not supported");
    }
    return 0;
}

constexpr size_t kMaxTileSmem = 200 * 1024;      // tile-histogram rows live in shared memory: up to 51200 tiles

// tuning knobs of dgr_set_tuning bits 24-26 (atomics, like the ones further down)
std::atomic<int> g_stage_fwd{1}, g_stage_bwd{1};   // per-Gaussian kernels: inputs staged through shared memory by bulk TMA (dgr_preprocess.cuh)
std::atomic<int> g_rowsum{1};                  // backward render, step 2: per-row form of the dy moments (dgr_render.cuh, ROWSUM)

// Can the per-Gaussian kernels stage their inputs with bulk TMA (dgr_preprocess.cuh)?  SH + scale / rotation inputs, every base
// pointer 16-byte aligned (cp.async.bulk), P at least one full warp.
inline bool stage_inputs_ok(const DgrGaussians *g, bool raw) {
    if (!g->shs || g->cov3D_precomp || !g->scales || !g->rotations || g->P < 32) return false;
    uintptr_t bits = (uintptr_t)g->means3D | (uintptr_t)g->scales | (uintptr_t)g->rotations | (uintptr_t)g->opacities | (uintptr_t)g->shs;
    if (raw && g->M > 1) bits |= (uintptr_t)g->shs_rest;
    return (bits & 15u) == 0;
}
constexpr size_t kMaxKernelSmem = 227 * 1024;

// Dynamic shared memory of a per-Gaussian forward kernel: the tile histogram, then, when its inputs are staged by bulk TMA,
// 8 warps x 32 x (44 + 12 M) bytes from stage_off.  Staged when the kernel has a staged variant (stageable: SH + scale /
// rotation inputs), the knob allows it, the inputs qualify and it fits next to the kernel's static shared memory.
struct PreFwdSmem { size_t bytes, stage_off; bool staged; };
PreFwdSmem pre_fwd_smem(const DgrGaussians *g, bool stageable, bool raw, int tiles, size_t static_smem) {
    const size_t hist = (size_t)tiles * 4, stage_off = align_up(hist, 128);
    const size_t staged_bytes = stage_off + (size_t)(kPreThreads / 32) * stage_warp_floats(g->M) * 4;
    const bool staged = stageable && g_stage_fwd.load() && stage_inputs_ok(g, raw) && staged_bytes + static_smem + 1024 <= kMaxKernelSmem;
    return { staged ? staged_bytes : hist, staged ? stage_off : 0, staged };
}


// ---- rasterization options (DgrRasterOptions) ----------------------------------------------------------------------------------
// The forward's flags live in one byte of the image scratch's work block, past TileWork: the forward's memset zeroes it (flags 0
// costs nothing) and an anti-aliased forward sets it; a backward with debug set compares it with its own flags.
constexpr size_t kFlagsByte = 255;
static_assert(sizeof(TileWork) <= kFlagsByte, "the flags byte must lie past TileWork (clear_costs_for_rerun zeroes up to its end)");
static_assert(DGR_RASTER_ANTIALIAS < 256u, "the known flags must fit the flags byte");

int raster_flags(const DgrRasterOptions *opt, uint32_t *flags) {
    *flags = opt ? opt->flags : 0u;
    if (*flags & DGR_RASTER_CAMERA_GRADS) return fail(-1, "DgrRasterOptions: DGR_RASTER_CAMERA_GRADS is backward-only (a forward call refuses it)");
    if (*flags & DGR_RASTER_ABS_GRAD) return fail(-1, "DgrRasterOptions: DGR_RASTER_ABS_GRAD is backward-only (a forward call refuses it)");
    if (*flags & DGR_RASTER_CONTRIB) return fail(-1, "DgrRasterOptions: DGR_RASTER_CONTRIB belongs to the stage-2 render calls (a preprocess call refuses it)");
    if (*flags & ~DGR_RASTER_ANTIALIAS) return fail(-1, "DgrRasterOptions: unknown flag bits");
    return 0;
}
// The stage-2 render calls' options: DGR_RASTER_CONTRIB only (*cb: the statistics' outputs, NULL without the bit), checked
// against `records` (P, or V P).
int raster_flags_render(const DgrRasterOptions *opt, int64_t records, const DgrContrib **cb) {
    const uint32_t flags = opt ? opt->flags : 0u;
    *cb = nullptr;
    if (flags & ~DGR_RASTER_CONTRIB) return fail(-1, "DgrRasterOptions: a stage-2 render call accepts DGR_RASTER_CONTRIB only");
    if (!(flags & DGR_RASTER_CONTRIB)) return 0;
    const DgrContrib *c = opt->contrib;
    if (!c) return fail(-1, "DgrRasterOptions: DGR_RASTER_CONTRIB with contrib == NULL");
    if (!c->weight_sum || !c->weight_max) return fail(-1, "contribution statistics: weight_sum / weight_max is NULL");
    if (!c->scratch) return fail(-1, "contribution statistics: scratch is NULL");
    if (c->scratch_bytes < dgr_contrib_scratch_bytes(records))
        return fail(-1, "contribution statistics: scratch is smaller than dgr_contrib_scratch_bytes(records)");
    *cb = c;
    return 0;
}
// DGR_RASTER_CONTRIB, before the render of every stage-2 run: outputs and scratch zeroed, so the run's values are its own
int contrib_clear(const DgrContrib *cb, int64_t records, cudaStream_t st) {
    if (!cb || records == 0) return 0;
    DGR_CUDA(cudaMemsetAsync(cb->weight_max, 0, (size_t)records * 4, st));
    DGR_CUDA(cudaMemsetAsync(cb->scratch, 0, (size_t)records * 8, st));
    return 0;
}
// ... and after it: the fixed-point sums -> weight_sum
int contrib_finalize(const DgrContrib *cb, int64_t records, int debug, cudaStream_t st) {
    if (!cb || records == 0) return 0;
    DGR_KERNEL("contrib_finalize", st, debug,
               launch_k(contrib_finalize_kernel, dim3((unsigned)((records + kContribFinalizeThreads - 1) / kContribFinalizeThreads)),
                        dim3(kContribFinalizeThreads), 0, st, false, (long long)records,
                        (const unsigned long long *)cb->scratch, cb->weight_sum));
    return 0;
}
ContribOut contrib_out(const DgrContrib *cb) {
    return ContribOut{reinterpret_cast<unsigned long long *>(cb->scratch), reinterpret_cast<unsigned *>(cb->weight_max)};
}
// The backward calls' options: the recorded / compared flags (DGR_RASTER_ANTIALIAS), with DGR_RASTER_CAMERA_GRADS the camera
// outputs (*cam; NULL without the bit) and with DGR_RASTER_ABS_GRAD the absolute-gradient statistic (*abs_accum; NULL without it).
int raster_flags_bwd(const DgrRasterOptions *opt, uint32_t *flags, const DgrCameraGrads **cam, float **abs_accum) {
    *flags = opt ? opt->flags : 0u;
    *cam = nullptr;
    *abs_accum = nullptr;
    if (*flags & DGR_RASTER_CONTRIB) return fail(-1, "DgrRasterOptions: DGR_RASTER_CONTRIB belongs to the stage-2 render calls (a backward call refuses it)");
    if (*flags & ~(DGR_RASTER_ANTIALIAS | DGR_RASTER_CAMERA_GRADS | DGR_RASTER_ABS_GRAD)) return fail(-1, "DgrRasterOptions: unknown flag bits");
    if (*flags & DGR_RASTER_CAMERA_GRADS) {
        if (!opt->camera) return fail(-1, "DgrRasterOptions: DGR_RASTER_CAMERA_GRADS with camera == NULL");
        *cam = opt->camera;
    }
    if (*flags & DGR_RASTER_ABS_GRAD) {
        if (!opt->xyz_gradient_accum_abs) return fail(-1, "DgrRasterOptions: DGR_RASTER_ABS_GRAD with xyz_gradient_accum_abs == NULL");
        *abs_accum = opt->xyz_gradient_accum_abs;
    }
    *flags &= DGR_RASTER_ANTIALIAS;
    return 0;
}
// DGR_RASTER_ABS_GRAD after the per-Gaussian backward: the statistic of the views in stats_views from moment slots 10 and 11
int absgrad_stats(int P, int V, const ViewTable &vt, uint64_t stats_views, const int *radii, const float *grad_rec, float *abs_accum,
                  int debug, cudaStream_t st) {
    DGR_KERNEL("absgrad_stats", st, debug, launch_k(absgrad_stats_kernel, dim3((unsigned)((P + kAbsStatsThreads - 1) / kAbsStatsThreads)),
                                                    dim3(kAbsStatsThreads), 0, st, false, P, V, vt, (unsigned long long)stats_views, radii,
                                                    grad_rec, abs_accum));
    return 0;
}
int check_camera(const DgrCameraGrads *cam, int V, int P) {
    if (!cam) return 0;
    if (!cam->scratch) return fail(-1, "camera gradients: scratch is NULL");
    if (cam->scratch_bytes < camera_grad_scratch_bytes(V, P))
        return fail(-1, "camera gradients: scratch is smaller than dgr_camera_grad_scratch_bytes(V, P)");
    return 0;
}
int record_flags(char *image, const ImageLayout &IL, uint32_t flags, cudaStream_t st) {
    if (flags) DGR_CUDA(cudaMemsetAsync(image + IL.off_work + kFlagsByte, (int)flags, 1, st));
    return 0;
}
int check_forward_flags(const void *image, const ImageLayout &IL, uint32_t flags, int debug, cudaStream_t st) {
    if (!debug) return 0;
    unsigned char fwd = 0;
    DGR_CUDA(cudaMemcpyAsync(&fwd, (const char *)image + IL.off_work + kFlagsByte, 1, cudaMemcpyDeviceToHost, st));
    DGR_CUDA(cudaStreamSynchronize(st));
    if (fwd != flags) return fail(-1, "backward: DgrRasterOptions.flags differ from those of the forward (antialiasing)");
    return 0;
}

template <int DEG, bool HAS_SH, bool HAS_COV, bool RAW>
void launch_pre_fwd(const DgrSettings *s, const DgrGaussians *g, int *radii, char *geom, const GeomLayout &L, unsigned *tile_count,
                    bool aa, cudaStream_t st) {
    const PreFwdSmem sm = pre_fwd_smem(g, HAS_SH && !HAS_COV, RAW, L.tiles, 0);
    auto launch = [&](auto kernel) {
        if (sm.bytes > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm.bytes);
        launch_k(kernel, dim3(L.nblocks), dim3(kPreThreads), sm.bytes, st, false,
            g->P, g->M, s->image_height, s->image_width, s->tanfovx, s->tanfovy, s->scale_modifier, s->viewmatrix, s->projmatrix,
            s->campos, g->means3D, g->shs, g->shs_rest, g->colors_precomp, g->opacities, g->scales, g->rotations, g->cov3D_precomp, radii,
            reinterpret_cast<Rec *>(geom + L.off_rec), reinterpret_cast<unsigned *>(geom + L.off_touched),
            tile_count, reinterpret_cast<unsigned *>(geom + L.off_runs), L.tiles, L.iters, (int)sm.stage_off);
    };
    if constexpr (HAS_SH && !HAS_COV) {
        if (sm.staged) {
            if (aa) launch(preprocess_fwd_aa_kernel<DEG, HAS_SH, HAS_COV, RAW, true>);
            else launch(preprocess_fwd_kernel<DEG, HAS_SH, HAS_COV, RAW, true>);
            return;
        }
    }
    if (aa) launch(preprocess_fwd_aa_kernel<DEG, HAS_SH, HAS_COV, RAW, false>);
    else launch(preprocess_fwd_kernel<DEG, HAS_SH, HAS_COV, RAW, false>);
}

template <int DEG, bool HAS_SH, bool HAS_COV, bool RAW>
void launch_pre_bwd(const DgrSettings *s, const DgrGaussians *g, const int *radii, const unsigned *touched, const float *grad_rec,
                    const DgrGaussianGrads *o, bool aa, cudaStream_t st) {
    const int nb = (g->P + kPreThreads - 1) / kPreThreads;
    PeerPush push;
    memset(&push, 0, sizeof(push));
    if (o->push) {
        push.per = (int)o->push->gaussians_per_owner;
        for (int w = 0; w < o->push->world && w < kMaxPeers; w++) push.delta[w] = o->push->delta_floats[w];
    }
    auto launch = [&](auto kernel, size_t smem, int wfl) {
        if (smem > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        launch_k(kernel, dim3(nb), dim3(kPreThreads), smem, st, true,
            g->P, g->M, s->image_height, s->image_width, s->tanfovx, s->tanfovy, s->scale_modifier, s->viewmatrix, s->projmatrix,
            s->campos, g->means3D, g->shs, g->shs_rest, g->opacities, g->scales, g->rotations, g->cov3D_precomp, radii, touched, grad_rec,
            o->dL_dmeans3D, o->dL_dmeans2D, o->dL_dshs, o->dL_dcolors_precomp, o->dL_dopacities, o->dL_dscales, o->dL_drotations,
            o->dL_dcov3D_precomp, o->dL_dshs_rest, o->xyz_gradient_accum, o->denom, o->max_radii2D, o->accumulate, push, wfl);
    };
    if constexpr (HAS_SH && !HAS_COV) {
        // inputs staged by bulk TMA; the same per-warp slice of dynamic shared memory is the warp's output image afterwards
        const int wfl = max(stage_warp_floats(g->M), kStageFloats);
        const size_t smem = (size_t)(kPreThreads / 32) * wfl * 4;
        if (g_stage_bwd.load() && stage_inputs_ok(g, RAW) && smem + 1024 <= kMaxKernelSmem) {
            if (aa) launch(preprocess_bwd_aa_kernel<DEG, HAS_SH, HAS_COV, RAW, true>, smem, wfl);
            else launch(preprocess_bwd_kernel<DEG, HAS_SH, HAS_COV, RAW, true>, smem, wfl);
            return;
        }
    }
    if (aa) launch(preprocess_bwd_aa_kernel<DEG, HAS_SH, HAS_COV, RAW, false>, 0, 0);
    else launch(preprocess_bwd_kernel<DEG, HAS_SH, HAS_COV, RAW, false>, 0, 0);
}

// camera gradients (dgr_camgrad.cuh): one CTA row per (256 Gaussians, view) into the caller's scratch
template <int DEG, bool HAS_SH, bool HAS_COV, bool RAW>
void launch_camera_bwd(int V, const ViewTable &vt, float2 tan0, const float *tanfov, float scale_modifier, const float *viewmatrix,
                       const float *projmatrix, const float *campos, const DgrGaussians *g, const int *radii, const unsigned *touched,
                       const float *grad_rec, float *rows, bool aa, cudaStream_t st) {
    const dim3 grid((unsigned)((g->P + kPreThreads - 1) / kPreThreads), (unsigned)V);
    launch_k(aa ? camera_bwd_kernel<DEG, HAS_SH, HAS_COV, RAW, true> : camera_bwd_kernel<DEG, HAS_SH, HAS_COV, RAW, false>, grid,
             dim3(kPreThreads), 0, st, false, g->P, g->M, vt, tan0, tanfov, scale_modifier, viewmatrix, projmatrix, campos, g->means3D,
             g->shs, g->shs_rest, g->scales, g->rotations, g->cov3D_precomp, radii, touched, grad_rec, rows);
}

// The compile-time configuration of the per-Gaussian kernels, handed to a generic lambda as integral constants.
template <int N> using IntC = std::integral_constant<int, N>;
// fn(DEG) for a checked SH degree 0..3
template <class Fn>
void with_sh_degree(int sh_degree, Fn &&fn) {
    switch (sh_degree) {
        case 0: fn(IntC<0>{}); break;
        case 1: fn(IntC<1>{}); break;
        case 2: fn(IntC<2>{}); break;
        default: fn(IntC<3>{}); break;
    }
}
// fn(DEG, HAS_SH, HAS_COV, RAW) of a checked call's inputs
template <class Fn>
void dispatch_gaussians(int sh_degree, const DgrGaussians *g, Fn &&fn) {
    using T = std::true_type;
    using F = std::false_type;
    if (g->activations) with_sh_degree(sh_degree, [&](auto deg) { fn(deg, T{}, F{}, T{}); });   // raw parameters: SH + scale/rotation only
    else if (!g->shs) { if (g->cov3D_precomp) fn(IntC<0>{}, F{}, T{}, F{}); else fn(IntC<0>{}, F{}, F{}, F{}); }
    else if (g->cov3D_precomp) with_sh_degree(sh_degree, [&](auto deg) { fn(deg, T{}, T{}, F{}); });
    else with_sh_degree(sh_degree, [&](auto deg) { fn(deg, T{}, F{}, F{}); });
}
// fn(DEG, RAW) of the batched call (SH + scale / rotation inputs only)
template <class Fn>
void dispatch_views(int sh_degree, bool raw, Fn &&fn) {
    if (raw) with_sh_degree(sh_degree, [&](auto deg) { fn(deg, std::true_type{}); });
    else with_sh_degree(sh_degree, [&](auto deg) { fn(deg, std::false_type{}); });
}

// The two camera-gradient kernels after the per-Gaussian backward of a checked call (S = DgrSettings or DgrViews).  tanfov = NULL:
// single view, tan0 = (tanfovx, tanfovy).  An empty cloud launches only the reduction, which writes zeros.
template <class S>
int camera_grads(const S *s, const DgrGaussians *g, const DgrCameraGrads *cam, int V, const ViewTable &vt, float2 tan0, const float *tanfov,
                 const int *radii, const unsigned *touched, const float *grad_rec, bool aa, cudaStream_t st) {
    float *rows = reinterpret_cast<float *>(cam->scratch);
    const int nblk = (g->P + kPreThreads - 1) / kPreThreads;
    if (g->P > 0)
        DGR_KERNEL("camera_bwd", st, s->debug, dispatch_gaussians(s->sh_degree, g, [&](auto deg, auto sh, auto cov, auto raw) {
            launch_camera_bwd<deg, sh, cov, raw>(V, vt, tan0, tanfov, s->scale_modifier, s->viewmatrix, s->projmatrix, s->campos, g, radii,
                                                 touched, grad_rec, rows, aa, st);
        }));
    DGR_KERNEL("camera_reduce", st, s->debug, launch_k(camera_reduce_kernel, dim3((unsigned)V), dim3(kCamReduceThreads), 0, st, false, nblk,
                                                      (const float *)rows, cam->dL_dviewmatrix, cam->dL_dprojmatrix, cam->dL_dcampos));
    return 0;
}

__global__ void debug_geom_kernel(int P, const Rec *rec, const unsigned *touched, float *mean_px, float *depth, float *conic,
                                  float *rgb, int *aabb, unsigned *tiles_touched) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= P) return;
    const Rec r = rec[g];
    if (mean_px) { mean_px[2 * g] = r.q0.x; mean_px[2 * g + 1] = r.q0.y; }
    if (depth) depth[g] = r.q1.z;
    if (conic) { conic[3 * g] = r.q0.z * (-2.f / kLog2e); conic[3 * g + 1] = r.q0.w * (-1.f / kLog2e); conic[3 * g + 2] = r.q1.x * (-2.f / kLog2e); }
    if (rgb) { rgb[3 * g] = r.q2.x; rgb[3 * g + 1] = r.q2.y; rgb[3 * g + 2] = r.q2.z; }
    if (aabb) {
        const unsigned ax = __float_as_uint(r.q1.w), ay = __float_as_uint(r.q2.w);
        aabb[4 * g] = (int)(ax & 0xffffu); aabb[4 * g + 1] = (int)(ay & 0xffffu); aabb[4 * g + 2] = (int)(ax >> 16); aabb[4 * g + 3] = (int)(ay >> 16);
    }
    if (tiles_touched) tiles_touched[g] = touched[g] & 0x1fffffffu;
}

// tuning knobs (dgr_set_tuning): pixels per lane of the render kernels, heaviest-first tile order on/off.  Atomics: any host
// thread may change them while another launches (each launch reads every knob once).
std::atomic<int> g_ppl_fwd{1}, g_ppl_bwd{1}, g_u_fwd{0}, g_u_bwd{0};      // u = 0: the default batching of that sub-tile shape
std::atomic<int> g_two_ended{0};       // work queue of the render kernels consumed from both ends (dgr_render.cuh)
std::atomic<int> g_cost_order{1};      // backward work ordered by the cost the forward measured (dgr_render.cuh)
std::atomic<int> g_lazy{0};            // record staging of the render kernels: 0 = by id when the sorted copy would exceed 2x L2, 1 = always sorted copy, 2 = always by id
std::atomic<int> g_cta_fwd{0}, g_cta_bwd{0};   // persistent CTAs per SM of the render kernels (0 = as many as fit)

using SmS = SortSmem<kSortSmallThreads, kSortSmallCap, kSortSmallBuckets>;
using SmB = SortSmem<kSortBigThreads, kSortBigCap, kSortBigBuckets>;

// Per-DEVICE launch state: cudaFuncSetAttribute (dynamic shared memory above 48 KB) and the occupancy-derived persistent
// grids are properties of a (function, device) pair, so they are kept per device ordinal and set up once under a mutex.
struct DevInfo {
    bool ready = false;
    int sms = 132;                    // H100 SXM until the device is queried
    size_t l2_bytes = 50u << 20;
    int big_grid = 132;               // big-tile sorter: one CTA per SM
    std::map<const void *, int> grids;   // persistent (occupancy x SMs) grid of every render kernel instantiation used so far
};
constexpr int kMaxDevices = 64;
DevInfo g_dev[kMaxDevices];
std::mutex g_dev_mu;

DevInfo *dev_info() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) { fail(-1, "cudaGetDevice failed or device ordinal above 63"); return nullptr; }
    std::lock_guard<std::mutex> lock(g_dev_mu);
    DevInfo &d = g_dev[dev];
    if (d.ready) return &d;
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) d.sms = n;
    d.big_grid = d.sms;
    int l2 = 0;
    if (cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev) == cudaSuccess && l2 > 0) d.l2_bytes = (size_t)l2;
    cudaError_t e = cudaFuncSetAttribute(emit_instances_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxTileSmem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(emit_views_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxTileSmem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tile_sort_gather_kernel<kSortSmallBuckets>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SmS::bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tile_sort_gather_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SmB::bytes);
    if (e != cudaSuccess) { fail((int)e, "cudaFuncSetAttribute", cudaGetErrorString(e)); return nullptr; }
    d.ready = true;
    return &d;
}

// persistent grid of a render kernel on the current device: (CTAs that fit on one SM) x SMs, computed once per (device, kernel)
template <class K>
int persistent_grid(DevInfo *d, K kernel, int threads, size_t smem) {
    std::lock_guard<std::mutex> lock(g_dev_mu);
    const void *key = reinterpret_cast<const void *>(kernel);
    auto it = d->grids.find(key);
    if (it != d->grids.end()) return it->second;
    if (smem > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    const int g = per_sm * d->sms;
    d->grids[key] = g;
    return g;
}

// Launch of a persistent render kernel: its persistent grid, at most max_ctas CTAs (its work items over the warps of a CTA, or the
// tiles of the deterministic backward) and, when the knob cta is set, at most that many CTAs per SM.
template <class K, class... Args>
int launch_persistent(DevInfo *dv, K kernel, const char *name, int threads, size_t smem, int max_ctas, const std::atomic<int> &cta, bool pdl,
                      int debug, cudaStream_t st, const Args &...args) {
    int grid = min(persistent_grid(dv, kernel, threads, smem), max_ctas);
    if (cta.load() > 0) grid = min(grid, cta.load() * dv->sms);
    DGR_KERNEL(name, st, debug, launch_k(kernel, dim3((unsigned)grid), dim3(threads), smem, st, pdl, args...));
    return 0;
}
// work items of a render kernel with ppl pixels per lane: its warps' sub-tiles of every 16x16 tile
constexpr int sub_tiles(int ppl) { return ppl == 4 ? SubTile<4>::kPerTile : ppl == 2 ? SubTile<2>::kPerTile : SubTile<1>::kPerTile; }

// ---- launch steps shared by the single-view and the batched (dgr_views_*) entry points ---------------------------------------
// A forward re-run with corrected capacity guesses repeats everything from instance emission on: the per-tile totals and run
// matrix are still valid, what the first, clipped render pass filed as backward costs is not.
int clear_costs_for_rerun(char *image, const ImageLayout &IL, int tiles, cudaStream_t st) {
    DGR_CUDA(cudaMemsetAsync(image + IL.off_cost, 0, (size_t)tiles * 8 * 4, st));
    DGR_CUDA(cudaMemsetAsync(image + IL.off_work + offsetof(TileWork, cost_bpt), 0, sizeof(TileWork) - offsetof(TileWork, cost_bpt), st));
    return 0;
}

// Without a ticket: { n_instances, n_big_tiles } to the host and the count-ready event, between the emit kernel and the sort
// (this also ends the chain of programmatic dependent launches there).
int copy_counts(const char *geom, uint64_t *counts_host, uint64_t ticket, void *count_ready_event, cudaStream_t st) {
    if (ticket) return 0;
    if (counts_host) DGR_CUDA(cudaMemcpyAsync(counts_host, geom, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    if (count_ready_event) DGR_CUDA(cudaEventRecord((cudaEvent_t)count_ready_event, st));
    return 0;
}

// Record staging of the render kernels.  A sorted copy of the records (written by the sort kernel, read with one contiguous
// bulk-TMA copy per 32 records) is the fast path while that copy lives in L2; once it is several times the L2 size the
// sort kernel's gather + write becomes the long pole and staging by id wins although a chunk then takes 32 small bulk
// copies (tools/tma_gather_probe.cu times both).  The threshold follows the device's L2 size (50 MB on an H100).
// Decided once per forward: its backward must stage its records the same way (the sorted copy is not written when staging
// by id), whatever the knobs say by then — the caller hands counts_host[3] to the backward.  Returns true for staging by id.
bool stage_records_by_id(uint64_t capacity, const DevInfo *dv, uint64_t *counts_host) {
    const int lz = g_lazy.load();
    const bool lazy = lz == 2 || (lz == 0 && (size_t)capacity * sizeof(Rec) > 2 * dv->l2_bytes);
    if (counts_host) counts_host[3] = lazy ? DGR_STAGING_BY_ID : DGR_STAGING_SORTED;
    return lazy;
}

// The per-tile sorts of the instance keys (+ the record gather unless lazy): the small-tile sorter over every tile, then the
// big-tile sorter when the emit kernel found big tiles.
int launch_tile_sorts(DevInfo *dv, const char *image, const ImageLayout &IL, int tiles, bool big_tiles, bool lazy,
                      unsigned long long *keys, const Rec *rec, unsigned *ids, Rec *recs, int debug, cudaStream_t st) {
    const TileWork *work = reinterpret_cast<const TileWork *>(image + IL.off_work);
    const uint2 *oranges = reinterpret_cast<const uint2 *>(image + IL.off_oranges);
    const int sort_grid = min(tiles, persistent_grid(dv, tile_sort_gather_kernel<kSortSmallBuckets>, kSortSmallThreads, SmS::bytes));
    DGR_KERNEL("tile_sort_gather", st, debug,
               launch_k(tile_sort_gather_kernel<kSortSmallBuckets>, dim3(sort_grid), dim3(kSortSmallThreads), SmS::bytes, st, true, work,
                        oranges, keys, rec, ids, recs, lazy ? 0 : 1));
    if (big_tiles)
        DGR_KERNEL("tile_sort_gather_big", st, debug,
                   launch_k(tile_sort_gather_big_kernel, dim3(dv->big_grid), dim3(kSortBigThreads), SmB::bytes, st, true, work,
                            reinterpret_cast<const unsigned *>(image + IL.off_biglist), reinterpret_cast<const uint2 *>(image + IL.off_ranges),
                            keys, rec, ids, recs, lazy ? 0 : 1));
    return 0;
}

// Work order of the render kernels by the cost the forward measured (dgr_render.cuh), or none when that knob is off.  bwd_ppl =
// the sub-tile shape of the backward the costs are grouped for.  (The backward only reads what the forward wrote.)
CostOrder cost_order(const char *image, const ImageLayout &IL, int tiles, int bwd_ppl) {
    CostOrder co{};
    if (g_cost_order.load()) {
        char *im = const_cast<char *>(image);
        TileWork *work = reinterpret_cast<TileWork *>(im + IL.off_work);
        co.cost_acc = reinterpret_cast<unsigned *>(im + IL.off_cost); co.cls_count = work->cls_count;
        co.cls_items = reinterpret_cast<unsigned *>(im + IL.off_clsitems); co.cost_bpt = &work->cost_bpt;
        co.tiles = tiles; co.bwd_ppl = bwd_ppl;
    }
    return co;
}

// ---- the deterministic backward (dgr_*_backward_det, dgr_det.cuh) --------------------------------------------------------------
struct DetArgs { void *scratch; uint64_t bytes; uint64_t instances; };

// the refusals of the deterministic calls on top of their counterparts' (before any device work)
int check_det(const DetArgs &d, const DgrGaussianGrads *gout, uint64_t capacity, long long records) {
    if (gout->push) return fail(-2, "deterministic backward: DgrPeerPush is not supported");
    if (d.instances > capacity) return fail(-1, "deterministic backward: instances above capacity_instances (pass the last stage-2 run's count)");
    if (!d.scratch) return fail(-1, "deterministic backward: det_scratch is NULL");
    if (d.bytes < DetLayout(d.instances, records).total)
        return fail(-1, "deterministic backward: det_scratch is smaller than dgr_det_scratch_bytes(instances, records)");
    return 0;
}

// Everything between the backward's memset and its per-Gaussian kernel: masked counts -> exclusive scan (goff) -> render_bwd_det ->
// det_moments_gather, which leaves grad_rec as the default render kernel would, summed in a fixed order.  head: the render kernel's
// leading arguments, (H, W, gx) of a single view or (vt) of a batch.
template <class... Head>
int det_render(DevInfo *dv, const DetArgs &d, long long R, int tiles, const char *image, const ImageLayout &IL, char *geom,
               const GeomLayout &GL, const char *binning, const BinningLayout &BL, bool lazy, const float *bg, const DgrImageGrads *gin,
               float *grad_rec, bool abs, int debug, cudaStream_t st, const Head &...head) {
    constexpr bool views = sizeof...(Head) == 1;
    if (debug) {                                     // debug: the caller's instance count against the forward's own (a host sync)
        unsigned long long n_fwd = 0;
        DGR_CUDA(cudaMemcpyAsync(&n_fwd, geom + offsetof(GeomHeader, n_inst), sizeof(n_fwd), cudaMemcpyDeviceToHost, st));
        DGR_CUDA(cudaStreamSynchronize(st));
        if (n_fwd != d.instances)
            return fail(-1, "deterministic backward: instances differs from the forward's instance count (pass the last stage-2 run's count)");
    }
    const DetLayout DL(d.instances, R);
    char *det = (char *)d.scratch;
    float *mom = reinterpret_cast<float *>(det + DL.off_mom);
    unsigned *goff = reinterpret_cast<unsigned *>(det + DL.off_goff), *sums = reinterpret_cast<unsigned *>(det + DL.off_sums);
    const unsigned *touched = reinterpret_cast<const unsigned *>(geom + GL.off_touched);
    if (d.instances > 0) {
        prof_begin("det_memset", st);
        const cudaError_t e = cudaMemsetAsync(mom, 0, (size_t)d.instances * kGradRecFloats * 4, st);
        prof_end(st);
        if (e != cudaSuccess) return fail((int)e, "det_memset", cudaGetErrorString(e));
    }
    const unsigned nb = (unsigned)((R + 255) / 256);
    DGR_KERNEL("det_counts", st, debug, launch_k(det_counts_kernel, dim3(nb), dim3(256), 0, st, false, R, touched, goff));
    DGR_KERNEL("det_scan_sums", st, debug, launch_k(knn_scan_sums_kernel, dim3((unsigned)DL.nblk), dim3(1024), 0, st, false,
                                                     (const unsigned *)goff, (size_t)R, sums));
    DGR_KERNEL("det_scan_top", st, debug, launch_k(knn_scan_top_kernel, dim3(1), dim3(1024), 0, st, false, sums, DL.nblk));
    DGR_KERNEL("det_scan_apply", st, debug, launch_k(knn_scan_apply_kernel, dim3((unsigned)DL.nblk), dim3(1024), 0, st, false,
                                                      goff, (size_t)R, (const unsigned *)sums));
    const TileWork *work = reinterpret_cast<const TileWork *>(image + IL.off_work);
    unsigned long long *bwd_next = reinterpret_cast<unsigned long long *>(geom + GL.off_bwdwork);
    const unsigned *order = reinterpret_cast<const unsigned *>(image + IL.off_order);
    const uint2 *oranges = reinterpret_cast<const uint2 *>(image + IL.off_oranges);
    const Rec *recs = reinterpret_cast<const Rec *>(binning + BL.off_rec), *rec = reinterpret_cast<const Rec *>(geom + GL.off_rec);
    const unsigned *ids = reinterpret_cast<const unsigned *>(binning + BL.off_ids);
    const float *fT = reinterpret_cast<const float *>(image + IL.off_finalT);
    const unsigned *nc = reinterpret_cast<const unsigned *>(image + IL.off_ncontrib);
    const unsigned long long n_slots = d.instances;
    const size_t smem = sizeof(DetSmem);
    auto launch = [&](auto kernel, const char *name) {
        return launch_persistent(dv, kernel, name, kDetThreads, smem, tiles, g_cta_bwd, true, debug, st, head..., order, oranges,
                                 &work->n_nonempty, bwd_next, recs, rec, ids, (const unsigned *)goff, n_slots, bg, fT, nc, gin->dL_dcolor,
                                 gin->dL_ddepth, gin->dL_dalpha, mom);
    };
    int e = 0;
    if (d.instances == 0) {}                         // nothing binned: no instance row to fill (the gather flags any touched record)
    else if constexpr (views) {
        if (abs) e = launch(lazy ? render_views_bwd_det_abs_kernel<true> : render_views_bwd_det_abs_kernel<false>, "render_views_bwd_det_abs");
        else e = launch(lazy ? render_views_bwd_det_kernel<true> : render_views_bwd_det_kernel<false>, "render_views_bwd_det");
    } else {
        if (abs) e = launch(lazy ? render_bwd_det_abs_kernel<true> : render_bwd_det_abs_kernel<false>, "render_bwd_det_abs");
        else e = launch(lazy ? render_bwd_det_kernel<true> : render_bwd_det_kernel<false>, "render_bwd_det");
    }
    if (e) return e;
    if (abs)
        DGR_KERNEL("det_moments_gather_abs", st, debug, launch_k(det_moments_gather_abs_kernel, dim3(nb), dim3(256), 0, st, true, R, touched,
                                                                 (const unsigned *)goff, (const float *)mom, n_slots, grad_rec));
    else
        DGR_KERNEL("det_moments_gather", st, debug, launch_k(det_moments_gather_kernel, dim3(nb), dim3(256), 0, st, true, R, touched,
                                                             (const unsigned *)goff, (const float *)mom, n_slots, grad_rec));
    return 0;
}

// ---- the stages shared by the single-view and the batched entry points after their checks -----------------------------------
// head: the leading arguments of the render kernels, (H, W, gx) of a single view or (vt) of a batch; the rest of each render
// kernel family's argument list is written once, below.

// Stage 2 of a forward (instance emission -> per-tile sorts -> render) of P Gaussians and `records` records.  emit(launch) launches
// the emit kernel as launch(kernel, name, its leading arguments); pick(fwd, lazy) launches the render kernel the knobs select as
// fwd(kernel, name, ppl[, ContribOut]).  cost_ppl: the backward sub-tile shape the render files its costs for.
template <class S, class Emit, class Pick, class... Head>
int forward_stage2(const S *s, int P, int64_t records, char *geom, const GeomLayout &GL, char *image, const ImageLayout &IL, char *binning,
                   uint64_t capacity, int32_t flags, uint64_t *counts_host, uint64_t ticket, void *count_ready_event, const DgrImages *out,
                   const DgrContrib *cb, int cost_ppl, cudaStream_t st, Emit &&emit, Pick &&pick, const Head &...head) {
    const BinningLayout BL(capacity);
    const int tiles = GL.tiles;
    const Rec *rec = reinterpret_cast<const Rec *>(geom + GL.off_rec);
    unsigned long long *keys = binning ? reinterpret_cast<unsigned long long *>(binning + BL.off_keys) : nullptr;
    unsigned *ids = binning ? reinterpret_cast<unsigned *>(binning + BL.off_ids) : nullptr;
    Rec *recs = binning ? reinterpret_cast<Rec *>(binning + BL.off_rec) : nullptr;
    unsigned *tile_order = reinterpret_cast<unsigned *>(image + IL.off_order);
    uint2 *oranges = reinterpret_cast<uint2 *>(image + IL.off_oranges);
    TileWork *work = reinterpret_cast<TileWork *>(image + IL.off_work);
    DevInfo *dv = dev_info();
    if (!dv) return -1;
    if (flags & DGR_FLAG_RERUN)
        if (int e = clear_costs_for_rerun(image, IL, tiles, st)) return e;
    if (int e = contrib_clear(cb, records, st)) return e;
    // instance emission; its extra block publishes ranges / order / counts (capacity 0: only that block has work to do)
    const int nb = (P > 0 && capacity > 0) ? GL.nblocks : 0;
    auto launch_emit = [&](auto kernel, const char *name, const auto &...emit_head) -> int {
        DGR_KERNEL(name, st, s->debug,
                   launch_k(kernel, dim3(nb + 1), dim3(kPreThreads), (size_t)tiles * 4, st, !(flags & DGR_FLAG_RERUN), emit_head..., GL.iters, nb,
                            rec, reinterpret_cast<const unsigned *>(geom + GL.off_touched), reinterpret_cast<const unsigned *>(image + IL.off_count),
                            (unsigned long long)capacity, reinterpret_cast<const unsigned *>(geom + GL.off_runs), keys,
                            reinterpret_cast<uint2 *>(image + IL.off_ranges), reinterpret_cast<GeomHeader *>(geom), tile_order, oranges, work,
                            reinterpret_cast<unsigned *>(image + IL.off_biglist), (volatile unsigned long long *)(ticket ? counts_host : nullptr),
                            (unsigned long long)ticket));
        return 0;
    };
    if (int e = emit(launch_emit)) return e;
    if (int e = copy_counts(geom, counts_host, ticket, count_ready_event, st)) return e;
    const bool lazy = stage_records_by_id(capacity, dv, counts_host);
    if (P > 0 && capacity > 0)
        if (int e = launch_tile_sorts(dv, image, IL, tiles, flags & DGR_FLAG_BIG_TILES, lazy, keys, rec, ids, recs, s->debug, st)) return e;
    // persistent forward render: every (tile, sub-tile) is a work item, handed out heaviest tile first
    const CostOrder co = cost_order(image, IL, tiles, cost_ppl);
    auto fwd = [&](auto kernel, const char *name, int ppl, const auto &...contrib) {
        const int items = tiles * sub_tiles(ppl);
        return launch_persistent(dv, kernel, name, kRenderThreads, 0, (items + kRenderWarps - 1) / kRenderWarps, g_cta_fwd, true, s->debug, st,
                                 head..., tile_order, oranges, &work->n_nonempty, (unsigned)items, &work->fwd_next, g_two_ended.load(), dv->sms,
                                 co, &work->lazy, recs, rec, ids, s->bg, out->color, out->depth, out->alpha,
                                 reinterpret_cast<unsigned *>(image + IL.off_ncontrib), reinterpret_cast<float *>(image + IL.off_finalT), contrib...);
    };
    if (int e = pick(fwd, lazy)) return e;
    return contrib_finalize(cb, records, s->debug, st);
}

// A backward of P Gaussians in V views (view table vt, tangents tan0 or tanfov as camera_grads takes them) from its memset on: the
// render (the deterministic one with det), the per-Gaussian backward, the AbsGS statistic of stats_views and the camera gradients.
// pick(bwd, lazy) launches the render kernel the knobs select as bwd(kernel, name, ppl); pre_bwd(touched, grad_rec, aa) launches
// the per-Gaussian backward.
template <class S, class Pick, class PreBwd, class... Head>
int backward_stages(const S *s, const DgrGaussians *g, int V, const ViewTable &vt, float2 tan0, const float *tanfov, uint64_t stats_views,
                    char *geom, const GeomLayout &GL, const char *image, const ImageLayout &IL, const char *binning, uint64_t capacity,
                    int32_t staging, const int32_t *radii, const DgrImageGrads *gin, const DetArgs *det, uint32_t flags,
                    const DgrCameraGrads *cam, float *abs_accum, cudaStream_t st, Pick &&pick, PreBwd &&pre_bwd, const Head &...head) {
    const long long records = (long long)g->P * V;
    const int tiles = GL.tiles;
    float *grad_rec = reinterpret_cast<float *>(geom + GL.off_gradrec);
    // the backward render adds each moment row with 16-byte vector reductions
    if (((uintptr_t)grad_rec & 15u) != 0) return fail(-1, "geometry scratch must be 16-byte aligned");
    // one memset: the work counter of the persistent backward render kernel + the per-Gaussian moment accumulators
    DGR_CUDA(cudaMemsetAsync(geom + GL.off_bwdwork, 0, (GL.off_gradrec - GL.off_bwdwork) + (size_t)records * kGradRecFloats * 4, st));
    if (binning && capacity > 0) {
        DevInfo *dv = dev_info();
        if (!dv) return -1;
        const BinningLayout BL(capacity);
        // the record staging the forward chose (dgr_forward_render): only then does the sorted copy exist
        const bool lazy = staging == DGR_STAGING_BY_ID;
        if (det) {
            if (int e = det_render(dv, *det, records, tiles, image, IL, geom, GL, binning, BL, lazy, s->bg, gin, grad_rec, abs_accum != nullptr,
                                   s->debug, st, head...)) return e;
        } else {
            const TileWork *work = reinterpret_cast<const TileWork *>(image + IL.off_work);
            // ppl 1 or 2: the backward's 8x4 or 8x8 sub-tiles; the work order is the one the forward grouped its costs in for that
            // shape (the kernel checks it)
            auto bwd = [&](auto kernel, const char *name, int ppl) {
                const size_t smem = (ppl == 1 ? sizeof(BwdSmem<1>) : sizeof(BwdSmem<2>)) * kRenderWarps;
                const int items = tiles * sub_tiles(ppl);
                return launch_persistent(dv, kernel, name, kRenderThreads, smem, (items + kRenderWarps - 1) / kRenderWarps, g_cta_bwd, false,
                                         s->debug, st, head..., reinterpret_cast<const unsigned *>(image + IL.off_order), &work->n_nonempty,
                                         reinterpret_cast<unsigned long long *>(geom + GL.off_bwdwork), g_two_ended.load(), dv->sms,
                                         cost_order(image, IL, tiles, ppl), reinterpret_cast<const uint2 *>(image + IL.off_oranges),
                                         reinterpret_cast<const Rec *>(binning + BL.off_rec), reinterpret_cast<const Rec *>(geom + GL.off_rec),
                                         &work->lazy, reinterpret_cast<const unsigned *>(binning + BL.off_ids), s->bg,
                                         reinterpret_cast<const float *>(image + IL.off_finalT),
                                         reinterpret_cast<const unsigned *>(image + IL.off_ncontrib), gin->dL_dcolor, gin->dL_ddepth,
                                         gin->dL_dalpha, grad_rec);
            };
            if (int e = pick(bwd, lazy)) return e;
        }
    }
    const unsigned *touched = reinterpret_cast<const unsigned *>(geom + GL.off_touched);
    const bool aa = flags & DGR_RASTER_ANTIALIAS;
    if (int e = pre_bwd(touched, grad_rec, aa)) return e;
    if (abs_accum)
        if (int e = absgrad_stats(g->P, V, vt, stats_views, radii, grad_rec, abs_accum, s->debug, st)) return e;
    if (cam) return camera_grads(s, g, cam, V, vt, tan0, tanfov, radii, touched, grad_rec, aa, st);
    return 0;
}
}  // namespace

extern "C" {

int dgr_abi_version(void) { return DGR_ABI_VERSION; }
const char *dgr_last_error(void) { return g_err.c_str(); }
uint64_t dgr_launch_count(void) { return g_launches; }
void dgr_reset_launch_count(void) { g_launches = 0; }

void dgr_profile_enable(int on) {
    for (auto &r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    g_prof.clear();
    g_prof_on = on != 0;
}
int dgr_profile_collect(char *names, size_t names_bytes, float *ms, int max) {
    int n = 0; size_t off = 0;
    if (names && names_bytes) names[0] = 0;
    for (auto &r : g_prof) {
        if (n >= max) break;
        if (cudaEventSynchronize(r.b) != cudaSuccess) break;
        float t = 0.f; cudaEventElapsedTime(&t, r.a, r.b);
        ms[n] = t;
        size_t L = strlen(r.name);
        if (names && off + L + 2 < names_bytes) { memcpy(names + off, r.name, L); off += L; names[off++] = '\n'; names[off] = 0; }
        n++;
    }
    for (auto &r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    g_prof.clear();
    return n;
}

int dgr_set_tuning(int ppl_fwd, int ppl_bwd, int tile_order) {
    if ((ppl_fwd != 1 && ppl_fwd != 2 && ppl_fwd != 4) || (ppl_bwd != 1 && ppl_bwd != 2 && ppl_bwd != 4)) return fail(-1, "ppl must be 1, 2 or 4");
    g_ppl_fwd = ppl_fwd; g_ppl_bwd = ppl_bwd == 4 ? 2 : ppl_bwd;          // the backward has 8x4 and 8x8 sub-tiles
    g_pdl = (tile_order & 8) ? 0 : 1;                   // bit 3: programmatic dependent launches OFF (A/B switch)
    g_u_fwd = (tile_order >> 4) & 7;                    // bits 4-6 / 8-10: hits evaluated together by the forward / backward
    g_u_bwd = (tile_order >> 8) & 7;                    // render kernels (1, 2 or 4; 0 = default of the sub-tile shape)
    g_cta_fwd = (tile_order >> 12) & 15;                // bits 12-15 / 16-19: persistent CTAs per SM of the forward / backward
    g_cta_bwd = (tile_order >> 16) & 15;                // render kernels (0 = as many as fit)
    g_two_ended = (tile_order >> 20) & 1;               // bit 20: work queue consumed from both ends (experiment; measured slower)
    g_cost_order = (tile_order >> 21) & 1 ? 0 : 1;      // bit 21: backward work in tile-population order instead of measured cost
    g_lazy = (tile_order >> 22) & 3;                    // bits 22-23: record staging 0 = auto, 1 = always the sorted copy, 2 = always by id
    g_stage_fwd = (tile_order >> 24) & 1 ? 0 : 1;       // bit 24 / 25: per-Gaussian forward / backward kernel reads its inputs with
    g_stage_bwd = (tile_order >> 25) & 1 ? 0 : 1;       // per-thread global loads instead of bulk-TMA staging (A/B switch)
    g_rowsum = (tile_order >> 26) & 1 ? 0 : 1;          // bit 26: backward render step 2 in the per-pixel form (A/B switch; <1,2> non-lazy only)
    return 0;
}

void *dgr_event_create(void) {
    cudaEvent_t e = nullptr;
    if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) { fail(-1, "cudaEventCreate failed"); return nullptr; }
    return (void *)e;
}
int dgr_event_synchronize(void *ev) { DGR_CUDA(cudaEventSynchronize((cudaEvent_t)ev)); return 0; }
void dgr_event_destroy(void *ev) { if (ev) cudaEventDestroy((cudaEvent_t)ev); }

size_t dgr_geom_bytes(int32_t P, int32_t H, int32_t W) { return GeomLayout(P, H, W).total; }
size_t dgr_image_bytes(int32_t H, int32_t W) { return ImageLayout(H, W).total; }
size_t dgr_binning_bytes(uint64_t cap, int32_t H, int32_t W) { (void)H; (void)W; return BinningLayout(cap).total; }

static int forward_preprocess(const DgrSettings *s, const DgrGaussians *g, void *geom_v, void *image_v, int32_t *radii, uint32_t flags,
                              void *stream) {
    if (int e = check_settings(s)) return e;
    if (int e = check_gaussians(s, g)) return e;
    cudaStream_t st = (cudaStream_t)stream;
    char *geom = (char *)geom_v, *image = (char *)image_v;
    if (!geom || !image) return fail(-1, "geom / image scratch is NULL");
    GeomLayout L(g->P, s->image_height, s->image_width);
    ImageLayout IL(s->image_height, s->image_width);
    if ((size_t)L.tiles * 4 > kMaxTileSmem) return fail(-3, "image has more than 51200 tiles (16x16): not supported");
    // one memset: the work block + the per-tile instance totals the preprocess kernel adds into + the backward cost accumulators
    DGR_CUDA(cudaMemsetAsync(image + IL.off_work, 0, (IL.off_cost - IL.off_work) + (size_t)L.tiles * 8 * 4, st));
    if (int e = record_flags(image, IL, flags, st)) return e;
    const bool aa = flags & DGR_RASTER_ANTIALIAS;
    if (g->P > 0) {
        if (!radii) return fail(-1, "radii is NULL");
        DGR_KERNEL("preprocess_fwd", st, s->debug, dispatch_gaussians(s->sh_degree, g, [&](auto deg, auto sh, auto cov, auto raw) {
            launch_pre_fwd<deg, sh, cov, raw>(s, g, radii, geom, L, reinterpret_cast<unsigned *>(image + IL.off_count), aa, st);
        }));
    }
    return 0;
}

int dgr_forward_preprocess(const DgrSettings *s, const DgrGaussians *g, void *geom_v, void *image_v, int32_t *radii, void *stream) {
    NvtxRange nvtx_("dgr_forward_preprocess");
    return forward_preprocess(s, g, geom_v, image_v, radii, 0u, stream);
}

int dgr_forward_preprocess_ex(const DgrSettings *s, const DgrGaussians *g, void *geom_v, void *image_v, int32_t *radii,
                              const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_forward_preprocess_ex");
    uint32_t flags = 0;
    if (int e = raster_flags(opt, &flags)) return e;
    return forward_preprocess(s, g, geom_v, image_v, radii, flags, stream);
}

static int forward_render(const DgrSettings *s, const DgrGaussians *g, void *geom_v, void *binning_v, uint64_t capacity,
                          void *image_v, const DgrImages *out, int32_t flags, uint64_t *counts_host, uint64_t ticket,
                          void *count_ready_event, const DgrRasterOptions *opt, void *stream) {
    if (int e = check_settings(s)) return e;
    if (!g || !geom_v || !image_v || !out) return fail(-1, "NULL argument");
    const DgrContrib *cb = nullptr;
    if (int e = raster_flags_render(opt, g->P, &cb)) return e;
    if (!out->color || !out->depth || !out->alpha) return fail(-1, "output images must not be NULL");
    if (capacity > 0 && !binning_v) return fail(-1, "binning scratch is NULL");
    if (capacity >= 0xffffffffull) return fail(-3, "capacity above 2^32-1 tile instances not supported");
    cudaStream_t st = (cudaStream_t)stream;
    char *geom = (char *)geom_v, *binning = (char *)binning_v, *image = (char *)image_v;
    const int H = s->image_height, W = s->image_width;
    GeomLayout GL(g->P, H, W);
    ImageLayout IL(H, W);
    const int tiles = IL.gx * IL.gy;
    if ((size_t)tiles * 4 > kMaxTileSmem) return fail(-3, "image has more than 51200 tiles (16x16): not supported");
    return forward_stage2(s, g->P, g->P, geom, GL, image, IL, binning, capacity, flags, counts_host, ticket, count_ready_event, out, cb,
                          g_ppl_bwd.load(), st,
                          [&](auto emit) { return emit(emit_instances_kernel, "emit_instances", g->P, IL.gx, tiles); },
                          [&](auto fwd, bool lazy) {
                              // DGR_RASTER_CONTRIB: the default shape's statistics variant, whatever the knobs
                              if (cb) return fwd(lazy ? render_fwd_contrib_kernel<true> : render_fwd_contrib_kernel<false>, "render_fwd_contrib", 1,
                                                 contrib_out(cb));
                              const int ppl = g_ppl_fwd.load(), uf = g_u_fwd.load();
                              if (ppl == 4) return fwd(lazy ? render_fwd_kernel<4, 1, true> : render_fwd_kernel<4, 1, false>, "render_fwd", 4);
                              if (ppl == 2) return fwd(lazy ? render_fwd_kernel<2, 2, true> : render_fwd_kernel<2, 2, false>, "render_fwd", 2);
                              if (uf == 4) return fwd(lazy ? render_fwd_kernel<1, 4, true> : render_fwd_kernel<1, 4, false>, "render_fwd", 1);
                              // default <1,1>: 58 registers, 8 CTAs per SM, no spill
                              return fwd(lazy ? render_fwd_kernel<1, 1, true> : render_fwd_kernel<1, 1, false>, "render_fwd", 1);
                          },
                          H, W, IL.gx);
}

int dgr_forward_render(const DgrSettings *s, const DgrGaussians *g, void *geom_v, void *binning_v, uint64_t capacity,
                       void *image_v, const DgrImages *out, int32_t flags, uint64_t *counts_host, uint64_t ticket,
                       void *count_ready_event, void *stream) {
    NvtxRange nvtx_("dgr_forward_render");
    return forward_render(s, g, geom_v, binning_v, capacity, image_v, out, flags, counts_host, ticket, count_ready_event, nullptr, stream);
}

int dgr_forward_render_ex(const DgrSettings *s, const DgrGaussians *g, void *geom_v, void *binning_v, uint64_t capacity,
                          void *image_v, const DgrImages *out, int32_t flags, uint64_t *counts_host, uint64_t ticket,
                          void *count_ready_event, const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_forward_render_ex");
    return forward_render(s, g, geom_v, binning_v, capacity, image_v, out, flags, counts_host, ticket, count_ready_event, opt, stream);
}

size_t dgr_contrib_scratch_bytes(int64_t records) { return records > 0 ? align_up((size_t)records * 8, 256) : 0; }

static int check_push(const DgrPeerPush *p, int64_t P) {
    if (!p) return 0;
    if (p->world < 1 || p->world > kMaxPeers || p->rank < 0 || p->rank >= p->world) return fail(-1, "push: bad world / rank");
    if (p->gaussians_per_owner <= 0 || p->gaussians_per_owner % kPreThreads != 0) return fail(-1, "push: gaussians_per_owner must be a positive multiple of 256");
    if (p->gaussians_per_owner * p->world < P) return fail(-1, "push: gaussians_per_owner * world < P");
    if (p->delta_floats[p->rank] != 0) return fail(-1, "push: delta_floats[rank] must be 0");
    return 0;
}

static int flat_segs(int32_t n_seg, const int64_t *seg_off, const int32_t *seg_stride, FlatSegs *out) {
    if (n_seg < 1 || n_seg > 8 || !seg_off || !seg_stride) return fail(-1, "1..8 flat segments expected");
    out->n = n_seg;
    for (int k = 0; k < n_seg; k++) {
        if (seg_off[k] < 0 || seg_stride[k] < 1) return fail(-1, "bad flat segment");
        out->off[k] = seg_off[k]; out->stride[k] = seg_stride[k];
    }
    return 0;
}

// dgr_backward, dgr_backward_ex (det = NULL) and dgr_backward_det, dgr_backward_det_ex (opt = NULL: no options)
static int backward_single(const DgrSettings *s, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity,
                           int32_t staging, const void *image_v, const int32_t *radii, const DgrImageGrads *gin,
                           const DgrGaussianGrads *gout, const DetArgs *det, const DgrRasterOptions *opt, void *stream) {
    uint32_t flags = 0;
    const DgrCameraGrads *cam = nullptr;
    float *abs_accum = nullptr;
    if (int e = raster_flags_bwd(opt, &flags, &cam, &abs_accum)) return e;
    if (int e = check_settings(s)) return e;
    if (int e = check_gaussians(s, g)) return e;
    if (int e = check_camera(cam, 1, g->P)) return e;
    if (!geom_v || !image_v || !gin || !gout) return fail(-1, "NULL argument");
    if (staging != DGR_STAGING_SORTED && staging != DGR_STAGING_BY_ID)
        return fail(-1, "staging must be DGR_STAGING_SORTED or DGR_STAGING_BY_ID (counts_host[3] of the forward)");
    if (det)
        if (int e = check_det(*det, gout, capacity, g->P)) return e;
    cudaStream_t st = (cudaStream_t)stream;
    ViewTable vt1;                                   // one view of H x W: the view table of the statistics and camera kernels
    memset(&vt1, 0, sizeof(vt1)); vt1.H[0] = s->image_height; vt1.W[0] = s->image_width;
    const float2 tan0 = make_float2(s->tanfovx, s->tanfovy);
    if (g->P == 0) return cam ? camera_grads(s, g, cam, 1, vt1, tan0, nullptr, radii, nullptr, nullptr, false, st) : 0;
    if (!radii) return fail(-1, "radii is NULL");
    if (int e = check_push(gout->push, g->P)) return e;
    char *geom = (char *)geom_v;
    const char *binning = (const char *)binning_v, *image = (const char *)image_v;
    const int H = s->image_height, W = s->image_width;
    GeomLayout GL(g->P, H, W);
    ImageLayout IL(H, W);
    if (int e = check_forward_flags(image, IL, flags, s->debug, st)) return e;
    return backward_stages(
        s, g, 1, vt1, tan0, nullptr, 1u, geom, GL, image, IL, binning, capacity, staging, radii, gin, det, flags, cam, abs_accum, st,
        [&](auto bwd, bool lazy) {
            // DGR_RASTER_ABS_GRAD: the default shape's ABS variant, whatever the knobs
            if (abs_accum) return bwd(lazy ? render_bwd_abs_kernel<true> : render_bwd_abs_kernel<false>, "render_bwd_abs", 1);
            const int ppl = g_ppl_bwd.load(), ub = g_u_bwd.load();
            // A/B: the default shape with the per-pixel step 2
            if (ppl == 1 && ub != 1 && !lazy && !g_rowsum.load()) return bwd(render_bwd_kernel<1, 2, false, false>, "render_bwd", 1);
            if (ppl == 1) {                              // default <1,2> (in-pipeline sweep, profiles/r2_sweep.txt)
                if (ub == 1) return bwd(lazy ? render_bwd_kernel<1, 1, true> : render_bwd_kernel<1, 1, false>, "render_bwd", 1);
                return bwd(lazy ? render_bwd_kernel<1, 2, true> : render_bwd_kernel<1, 2, false>, "render_bwd", 1);
            }
            if (ub == 2) return bwd(lazy ? render_bwd_kernel<2, 2, true> : render_bwd_kernel<2, 2, false>, "render_bwd", 2);
            return bwd(lazy ? render_bwd_kernel<2, 1, true> : render_bwd_kernel<2, 1, false>, "render_bwd", 2);
        },
        [&](const unsigned *touched, const float *grad_rec, bool aa) -> int {
            DGR_KERNEL("preprocess_bwd", st, s->debug, dispatch_gaussians(s->sh_degree, g, [&](auto deg, auto sh, auto cov, auto raw) {
                launch_pre_bwd<deg, sh, cov, raw>(s, g, radii, touched, grad_rec, gout, aa, st);
            }));
            return 0;
        },
        H, W, IL.gx);
}

int dgr_backward(const DgrSettings *s, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity,
                 int32_t staging, const void *image_v, const int32_t *radii, const float *out_alpha, const DgrImageGrads *gin,
                 const DgrGaussianGrads *gout, void *stream) {
    NvtxRange nvtx_("dgr_backward");
    (void)out_alpha;
    return backward_single(s, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, nullptr, nullptr, stream);
}

int dgr_backward_ex(const DgrSettings *s, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity,
                    int32_t staging, const void *image_v, const int32_t *radii, const float *out_alpha, const DgrImageGrads *gin,
                    const DgrGaussianGrads *gout, const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_backward_ex");
    (void)out_alpha;
    return backward_single(s, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, nullptr, opt, stream);
}

size_t dgr_det_scratch_bytes(uint64_t instances, int64_t records) { return DetLayout(instances, records).total; }
size_t dgr_camera_grad_scratch_bytes(int32_t V, int32_t P) { return camera_grad_scratch_bytes(V, P); }

int dgr_backward_det(const DgrSettings *s, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity,
                     int32_t staging, const void *image_v, const int32_t *radii, const float *out_alpha, const DgrImageGrads *gin,
                     const DgrGaussianGrads *gout, void *det_scratch, uint64_t det_scratch_bytes, uint64_t instances, void *stream) {
    NvtxRange nvtx_("dgr_backward_det");
    (void)out_alpha;
    const DetArgs det{det_scratch, det_scratch_bytes, instances};
    return backward_single(s, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, &det, nullptr, stream);
}

int dgr_backward_det_ex(const DgrSettings *s, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity,
                        int32_t staging, const void *image_v, const int32_t *radii, const float *out_alpha, const DgrImageGrads *gin,
                        const DgrGaussianGrads *gout, void *det_scratch, uint64_t det_scratch_bytes, uint64_t instances,
                        const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_backward_det_ex");
    (void)out_alpha;
    const DetArgs det{det_scratch, det_scratch_bytes, instances};
    return backward_single(s, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, &det, opt, stream);
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------------
// Batched cameras (include/dgr_b200.h, DgrViews): one cloud, V views, same-size (dgr_views_*) or each with its own image size
// (dgr_views_mixed_*).  Same pipeline as the single-view call on a global tile space (view v's tiles start at tile_off[v]) and
// V x P records (record v P + g).  Both entry families run the same five kernels; a same-size batch is the uniform ViewTable.
// ---------------------------------------------------------------------------------------------------------------------------
namespace {
int check_views(const DgrViews *s) {
    if (!s) return fail(-1, "views settings is NULL");
    if (s->V < 1 || s->V > DGR_VIEWS_MAX) return fail(-3, "views: V must be 1..64");
    if (s->image_height <= 0 || s->image_width <= 0) return fail(-1, "image size must be positive");
    if (s->image_height > 65535 || s->image_width > 65535) return fail(-1, "image size above 65535 not supported");
    if (s->sh_degree < 0 || s->sh_degree > 3) return fail(-1, "sh_degree must be 0..3");
    const size_t tiles = (size_t)((s->image_width + kTile - 1) / kTile) * (size_t)((s->image_height + kTile - 1) / kTile) * (size_t)s->V;
    if (tiles * 4 > kMaxTileSmem) return fail(-3, "views: V x tiles per view above 51200 (16x16 tiles) not supported");
    if (!s->tanfov || !s->bg || !s->viewmatrix || !s->projmatrix || !s->campos)
        return fail(-1, "views: tanfov / bg / viewmatrix / projmatrix / campos must not be NULL");
    return 0;
}
// the mixed-size call: image_hw [V,2] (height, width) replaces DgrViews.image_height / image_width
int check_views_mixed_sizes(const DgrViews *s, const int32_t *image_hw) {
    if (!s) return fail(-1, "views settings is NULL");
    if (s->V < 1 || s->V > DGR_VIEWS_MAX) return fail(-3, "views: V must be 1..64");
    if (!image_hw) return fail(-1, "views mixed: image_hw is NULL");
    size_t tiles = 0;
    for (int v = 0; v < s->V; v++) {
        const int h = image_hw[2 * v], w = image_hw[2 * v + 1];
        if (h <= 0 || w <= 0) return fail(-1, "views mixed: every image size must be positive");
        if (h > 65535 || w > 65535) return fail(-1, "views mixed: image size above 65535 not supported");
        tiles += (size_t)((w + kTile - 1) / kTile) * (size_t)((h + kTile - 1) / kTile);
    }
    if (tiles * 4 > kMaxTileSmem) return fail(-3, "views mixed: more than 51200 tiles (16x16) in the batch not supported");
    return 0;
}
int check_views_mixed(const DgrViews *s, const int32_t *image_hw) {
    if (int e = check_views_mixed_sizes(s, image_hw)) return e;
    if (s->sh_degree < 0 || s->sh_degree > 3) return fail(-1, "sh_degree must be 0..3");
    if (!s->tanfov || !s->bg || !s->viewmatrix || !s->projmatrix || !s->campos)
        return fail(-1, "views: tanfov / bg / viewmatrix / projmatrix / campos must not be NULL");
    return 0;
}
int check_views_gaussians(const DgrViews *s, const DgrGaussians *g) {
    if (!g) return fail(-1, "gaussians is NULL");
    if (g->P < 0) return fail(-1, "P < 0");
    if ((long long)s->V * (long long)g->P > DGR_VIEWS_MAX_RECORDS) return fail(-3, "views: V x P above 2^31 - 1 records not supported");
    if (g->P == 0) return 0;
    if (g->colors_precomp || g->cov3D_precomp)
        return fail(-2, "views: precomputed colours / cov3D are not supported by the batched call (SH + scale / rotation only)");
    if (!g->shs || !g->scales || !g->rotations || !g->means3D || !g->opacities)
        return fail(-1, "views: means3D / shs / opacities / scales / rotations must not be NULL");
    if (g->activations && g->M > 1 && !g->shs_rest) return fail(-2, "activations: shs_rest (_features_rest) is NULL but M > 1");
    const int nb = (s->sh_degree + 1) * (s->sh_degree + 1);
    if (g->M < nb) return fail(-1, "shs has fewer coefficients than sh_degree needs");
    if (g->M > 16) return fail(-1, "shs with more than 16 coefficients per channel not supported");
    return 0;
}
// the backward's output checks shared by both entry families (the same-size call refuses the statistics before this)
int check_views_grads(const DgrGaussianGrads *gout) {
    if (gout->push) return fail(-2, "views: DgrPeerPush is not supported by the batched call");
    if (gout->dL_dcolors_precomp || gout->dL_dcov3D_precomp)
        return fail(-2, "views: precomputed colours / cov3D are not supported by the batched call (SH + scale / rotation only)");
    return 0;
}

// The views' sizes as the kernels see them (ViewTable) and the batch totals.  hw = V (height, width) pairs, or ONE pair for every
// view (hw_stride 0: the same-size call).  The sizes have been checked.
struct ViewsBatch {
    ViewTable vt;
    int V, tiles;
    size_t pixels;
};
ViewsBatch views_batch(int V, const int32_t *hw, int hw_stride) {
    ViewsBatch b;
    memset(&b, 0, sizeof(b));
    b.V = V;
    int tiles = 0, pix = 0;
    for (int v = 0; v < V; v++) {
        const int h = hw[v * hw_stride], w = hw[v * hw_stride + 1];
        b.vt.H[v] = h; b.vt.W[v] = w; b.vt.gx[v] = (w + kTile - 1) / kTile;
        b.vt.tile_off[v] = tiles; b.vt.pix_off[v] = pix;
        tiles += b.vt.gx[v] * ((h + kTile - 1) / kTile);
        pix += h * w;                                   // <= 51200 tiles x 256 pixels: fits
    }
    for (int v = V; v <= kMaxViews; v++) b.vt.tile_off[v] = tiles;
    b.tiles = tiles; b.pixels = (size_t)pix;
    return b;
}
ViewsBatch views_batch_uniform(const DgrViews *s) {
    const int32_t hw[2] = { s->image_height, s->image_width };
    return views_batch(s->V, hw, 0);
}

constexpr size_t kViewsFwdStaticSmem = (size_t)kMaxViews * (sizeof(FrameConsts) + sizeof(float2)) + (kPreThreads / 32) * 8;

template <int DEG, bool RAW>
void launch_views_pre_fwd(const DgrViews *s, const ViewsBatch &b, const DgrGaussians *g, int *radii, char *geom, const GeomLayout &L,
                          unsigned *tile_count, bool aa, cudaStream_t st) {
    const PreFwdSmem sm = pre_fwd_smem(g, true, RAW, L.tiles, kViewsFwdStaticSmem);
    auto launch = [&](auto kernel) {
        if (sm.bytes + kViewsFwdStaticSmem > 48 * 1024)          // the cameras' static shared memory counts against the 48 KB
            cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm.bytes);
        launch_k(kernel, dim3(L.nblocks), dim3(kPreThreads), sm.bytes, st, false, g->P, g->M, s->V, b.vt,
                 s->scale_modifier, s->tanfov, s->viewmatrix, s->projmatrix, s->campos, g->means3D, g->shs, g->shs_rest, g->opacities,
                 g->scales, g->rotations, radii, reinterpret_cast<Rec *>(geom + L.off_rec), reinterpret_cast<unsigned *>(geom + L.off_touched),
                 tile_count, reinterpret_cast<unsigned *>(geom + L.off_runs), L.iters, (int)sm.stage_off);
    };
    if (aa) {
        if (sm.staged) launch(preprocess_views_fwd_aa_kernel<DEG, RAW, true>);
        else launch(preprocess_views_fwd_aa_kernel<DEG, RAW, false>);
    } else {
        if (sm.staged) launch(preprocess_views_fwd_kernel<DEG, RAW, true>);
        else launch(preprocess_views_fwd_kernel<DEG, RAW, false>);
    }
}

template <int DEG, bool RAW>
void launch_views_pre_bwd(const DgrViews *s, const ViewsBatch &b, const DgrGaussians *g, const int *radii, const unsigned *touched,
                          const float *grad_rec, const DgrGaussianGrads *o, uint64_t stats_views, bool aa, cudaStream_t st) {
    launch_k(aa ? preprocess_views_bwd_aa_kernel<DEG, RAW> : preprocess_views_bwd_kernel<DEG, RAW>, dim3((g->P + kPreThreads - 1) / kPreThreads),
             dim3(kPreThreads), 0, st, true,
             g->P, g->M, s->V, b.vt, s->scale_modifier, s->tanfov, s->viewmatrix, s->projmatrix, s->campos,
             g->means3D, g->shs, g->shs_rest, g->opacities, g->scales, g->rotations, radii, touched, grad_rec, o->dL_dmeans3D,
             o->dL_dmeans2D, o->dL_dshs, o->dL_dopacities, o->dL_dscales, o->dL_drotations, o->dL_dshs_rest, o->xyz_gradient_accum,
             o->denom, o->max_radii2D, (unsigned long long)stats_views, o->accumulate);
}

// The three stages of a checked batch (s, g and the sizes in b).
int views_preprocess(const DgrViews *s, const ViewsBatch &b, const DgrGaussians *g, void *geom_v, void *image_v, int32_t *radii, uint32_t flags,
                     void *stream) {
    char *geom = (char *)geom_v, *image = (char *)image_v;
    if (!geom || !image) return fail(-1, "geom / image scratch is NULL");
    if (g->P > 0 && !radii) return fail(-1, "radii is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    const GeomLayout L = GeomLayout::batch(g->P, b.tiles, s->V);
    const ImageLayout IL = ImageLayout::batch((size_t)b.tiles, b.pixels);
    DGR_CUDA(cudaMemsetAsync(image + IL.off_work, 0, (IL.off_cost - IL.off_work) + (size_t)L.tiles * 8 * 4, st));
    if (int e = record_flags(image, IL, flags, st)) return e;
    const bool aa = flags & DGR_RASTER_ANTIALIAS;
    if (g->P > 0)
        DGR_KERNEL("preprocess_views_fwd", st, s->debug,
                   dispatch_views(s->sh_degree, g->activations, [&](auto deg, auto raw) {
                       launch_views_pre_fwd<deg, raw>(s, b, g, radii, geom, L, reinterpret_cast<unsigned *>(image + IL.off_count), aa, st);
                   }));
    return 0;
}

int views_render(const DgrViews *s, const ViewsBatch &b, const DgrGaussians *g, void *geom_v, void *binning_v, uint64_t capacity,
                 void *image_v, const DgrImages *out, int32_t flags, uint64_t *counts_host, uint64_t ticket, void *count_ready_event,
                 const DgrRasterOptions *opt, void *stream) {
    if (!geom_v || !image_v || !out) return fail(-1, "NULL argument");
    const int64_t records = (int64_t)g->P * s->V;
    const DgrContrib *cb = nullptr;
    if (int e = raster_flags_render(opt, records, &cb)) return e;
    if (!out->color || !out->depth || !out->alpha) return fail(-1, "output images must not be NULL");
    if (capacity > 0 && !binning_v) return fail(-1, "binning scratch is NULL");
    if (capacity >= 0xffffffffull) return fail(-3, "capacity above 2^32-1 tile instances not supported");
    cudaStream_t st = (cudaStream_t)stream;
    char *geom = (char *)geom_v, *binning = (char *)binning_v, *image = (char *)image_v;
    const GeomLayout GL = GeomLayout::batch(g->P, b.tiles, s->V);
    const ImageLayout IL = ImageLayout::batch((size_t)b.tiles, b.pixels);
    return forward_stage2(s, g->P, records, geom, GL, image, IL, binning, capacity, flags, counts_host, ticket, count_ready_event, out, cb,
                          1, st,                 // the batched backward's 8x4 sub-tiles
                          [&](auto emit) { return emit(emit_views_kernel, "emit_views", g->P, s->V, b.vt); },
                          [&](auto fwd, bool lazy) {
                              if (cb) return fwd(lazy ? render_views_fwd_contrib_kernel<true> : render_views_fwd_contrib_kernel<false>,
                                                 "render_views_fwd_contrib", 1, contrib_out(cb));
                              return fwd(lazy ? render_views_fwd_kernel<true> : render_views_fwd_kernel<false>, "render_views_fwd", 1);
                          },
                          b.vt);
}

int views_backward(const DgrViews *s, const ViewsBatch &b, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity,
                   int32_t staging, const void *image_v, const int32_t *radii, const DgrImageGrads *gin, const DgrGaussianGrads *gout, uint64_t stats_views,
                   const DetArgs *det, uint32_t flags, const DgrCameraGrads *cam, float *abs_accum, void *stream) {
    if (det)
        if (int e = check_det(*det, gout, capacity, (long long)g->P * s->V)) return e;
    if (int e = check_camera(cam, s->V, g->P)) return e;
    cudaStream_t st = (cudaStream_t)stream;
    if (g->P == 0) return cam ? camera_grads(s, g, cam, s->V, b.vt, make_float2(0.f, 0.f), s->tanfov, radii, nullptr, nullptr, false, st) : 0;
    if (!radii) return fail(-1, "radii is NULL");
    char *geom = (char *)geom_v;
    const char *binning = (const char *)binning_v, *image = (const char *)image_v;
    const GeomLayout GL = GeomLayout::batch(g->P, b.tiles, s->V);
    const ImageLayout IL = ImageLayout::batch((size_t)b.tiles, b.pixels);
    if (int e = check_forward_flags(image, IL, flags, s->debug, st)) return e;
    return backward_stages(
        s, g, s->V, b.vt, make_float2(0.f, 0.f), s->tanfov, stats_views, geom, GL, image, IL, binning, capacity, staging, radii, gin, det, flags,
        cam, abs_accum, st,
        [&](auto bwd, bool lazy) {
            // DGR_RASTER_ABS_GRAD: the ABS variant of the same kernel
            if (abs_accum) return bwd(lazy ? render_views_bwd_abs_kernel<true> : render_views_bwd_abs_kernel<false>, "render_views_bwd_abs", 1);
            return bwd(lazy ? render_views_bwd_kernel<true> : render_views_bwd_kernel<false>, "render_views_bwd", 1);
        },
        [&](const unsigned *touched, const float *grad_rec, bool aa) -> int {
            DGR_KERNEL("preprocess_views_bwd", st, s->debug, dispatch_views(s->sh_degree, g->activations, [&](auto deg, auto raw) {
                launch_views_pre_bwd<deg, raw>(s, b, g, radii, touched, grad_rec, gout, stats_views, aa, st);
            }));
            return 0;
        },
        b.vt);
}
}  // namespace

extern "C" {

size_t dgr_views_geom_bytes(int32_t V, int32_t P, int32_t H, int32_t W) { return GeomLayout(P, H, W, V > 0 ? V : 1).total; }
size_t dgr_views_image_bytes(int32_t V, int32_t H, int32_t W) { return ImageLayout(H, W, V > 0 ? V : 1).total; }
size_t dgr_views_binning_bytes(uint64_t cap, int32_t V, int32_t H, int32_t W) { (void)V; (void)H; (void)W; return BinningLayout(cap).total; }

int dgr_views_forward_preprocess(const DgrViews *s, const DgrGaussians *g, void *geom_v, void *image_v, int32_t *radii, void *stream) {
    NvtxRange nvtx_("dgr_views_forward_preprocess");
    if (int e = check_views(s)) return e;
    if (int e = check_views_gaussians(s, g)) return e;
    return views_preprocess(s, views_batch_uniform(s), g, geom_v, image_v, radii, 0u, stream);
}

int dgr_views_forward_preprocess_ex(const DgrViews *s, const DgrGaussians *g, void *geom_v, void *image_v, int32_t *radii,
                                    const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_views_forward_preprocess_ex");
    uint32_t flags = 0;
    if (int e = raster_flags(opt, &flags)) return e;
    if (int e = check_views(s)) return e;
    if (int e = check_views_gaussians(s, g)) return e;
    return views_preprocess(s, views_batch_uniform(s), g, geom_v, image_v, radii, flags, stream);
}

int dgr_views_forward_render(const DgrViews *s, const DgrGaussians *g, void *geom_v, void *binning_v, uint64_t capacity,
                             void *image_v, const DgrImages *out, int32_t flags, uint64_t *counts_host, uint64_t ticket,
                             void *count_ready_event, void *stream) {
    NvtxRange nvtx_("dgr_views_forward_render");
    if (int e = check_views(s)) return e;
    if (int e = check_views_gaussians(s, g)) return e;
    return views_render(s, views_batch_uniform(s), g, geom_v, binning_v, capacity, image_v, out, flags, counts_host, ticket,
                        count_ready_event, nullptr, stream);
}

int dgr_views_forward_render_ex(const DgrViews *s, const DgrGaussians *g, void *geom_v, void *binning_v, uint64_t capacity,
                                void *image_v, const DgrImages *out, int32_t flags, uint64_t *counts_host, uint64_t ticket,
                                void *count_ready_event, const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_views_forward_render_ex");
    if (int e = check_views(s)) return e;
    if (int e = check_views_gaussians(s, g)) return e;
    return views_render(s, views_batch_uniform(s), g, geom_v, binning_v, capacity, image_v, out, flags, counts_host, ticket,
                        count_ready_event, opt, stream);
}

// dgr_views_backward* (det = NULL: not deterministic, opt = NULL: no options)
static int views_backward_same(const DgrViews *s, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity, int32_t staging,
                               const void *image_v, const int32_t *radii, const DgrImageGrads *gin, const DgrGaussianGrads *gout,
                               const DetArgs *det, const DgrRasterOptions *opt, void *stream) {
    uint32_t flags = 0;
    const DgrCameraGrads *cam = nullptr;
    float *abs_accum = nullptr;
    if (int e = raster_flags_bwd(opt, &flags, &cam, &abs_accum)) return e;
    if (int e = check_views(s)) return e;
    if (int e = check_views_gaussians(s, g)) return e;
    if (!geom_v || !image_v || !gin || !gout) return fail(-1, "NULL argument");
    if (staging != DGR_STAGING_SORTED && staging != DGR_STAGING_BY_ID)
        return fail(-1, "staging must be DGR_STAGING_SORTED or DGR_STAGING_BY_ID (counts_host[3] of the forward)");
    if (gout->xyz_gradient_accum || gout->denom || gout->max_radii2D)
        return fail(-2, "views: the fused densification statistics are not supported by the batched call");
    if (abs_accum)
        return fail(-2, "views: DGR_RASTER_ABS_GRAD is not supported by the same-size batched call (it has no densification statistics)");
    if (int e = check_views_grads(gout)) return e;
    return views_backward(s, views_batch_uniform(s), g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, 0, det, flags,
                          cam, nullptr, stream);
}

int dgr_views_backward(const DgrViews *s, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity, int32_t staging,
                       const void *image_v, const int32_t *radii, const DgrImageGrads *gin, const DgrGaussianGrads *gout, void *stream) {
    NvtxRange nvtx_("dgr_views_backward");
    return views_backward_same(s, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, nullptr, nullptr, stream);
}

int dgr_views_backward_ex(const DgrViews *s, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity, int32_t staging,
                          const void *image_v, const int32_t *radii, const DgrImageGrads *gin, const DgrGaussianGrads *gout,
                          const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_views_backward_ex");
    return views_backward_same(s, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, nullptr, opt, stream);
}

int dgr_views_backward_det(const DgrViews *s, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity, int32_t staging,
                           const void *image_v, const int32_t *radii, const DgrImageGrads *gin, const DgrGaussianGrads *gout,
                           void *det_scratch, uint64_t det_scratch_bytes, uint64_t instances, void *stream) {
    NvtxRange nvtx_("dgr_views_backward_det");
    const DetArgs det{det_scratch, det_scratch_bytes, instances};
    return views_backward_same(s, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, &det, nullptr, stream);
}

int dgr_views_backward_det_ex(const DgrViews *s, const DgrGaussians *g, void *geom_v, const void *binning_v, uint64_t capacity, int32_t staging,
                              const void *image_v, const int32_t *radii, const DgrImageGrads *gin, const DgrGaussianGrads *gout,
                              void *det_scratch, uint64_t det_scratch_bytes, uint64_t instances, const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_views_backward_det_ex");
    const DetArgs det{det_scratch, det_scratch_bytes, instances};
    return views_backward_same(s, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, &det, opt, stream);
}

// ---- views of different sizes: image_hw = [V,2] (height, width) on the host ------------------------------------------------------
size_t dgr_views_mixed_geom_bytes(int32_t V, int32_t P, const int32_t *image_hw) {
    DgrViews s{};
    s.V = V;
    if (check_views_mixed_sizes(&s, image_hw)) return 0;
    return GeomLayout::batch(P, views_batch(V, image_hw, 2).tiles, V).total;
}
size_t dgr_views_mixed_image_bytes(int32_t V, const int32_t *image_hw) {
    DgrViews s{};
    s.V = V;
    if (check_views_mixed_sizes(&s, image_hw)) return 0;
    const ViewsBatch b = views_batch(V, image_hw, 2);
    return ImageLayout::batch((size_t)b.tiles, b.pixels).total;
}

int dgr_views_mixed_forward_preprocess(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom_v, void *image_v,
                                       int32_t *radii, void *stream) {
    NvtxRange nvtx_("dgr_views_mixed_forward_preprocess");
    if (int e = check_views_mixed(s, image_hw)) return e;
    if (int e = check_views_gaussians(s, g)) return e;
    return views_preprocess(s, views_batch(s->V, image_hw, 2), g, geom_v, image_v, radii, 0u, stream);
}

int dgr_views_mixed_forward_preprocess_ex(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom_v, void *image_v,
                                          int32_t *radii, const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_views_mixed_forward_preprocess_ex");
    uint32_t flags = 0;
    if (int e = raster_flags(opt, &flags)) return e;
    if (int e = check_views_mixed(s, image_hw)) return e;
    if (int e = check_views_gaussians(s, g)) return e;
    return views_preprocess(s, views_batch(s->V, image_hw, 2), g, geom_v, image_v, radii, flags, stream);
}

int dgr_views_mixed_forward_render(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom_v, void *binning_v,
                                   uint64_t capacity, void *image_v, const DgrImages *out, int32_t flags, uint64_t *counts_host,
                                   uint64_t ticket, void *count_ready_event, void *stream) {
    NvtxRange nvtx_("dgr_views_mixed_forward_render");
    if (int e = check_views_mixed(s, image_hw)) return e;
    if (int e = check_views_gaussians(s, g)) return e;
    return views_render(s, views_batch(s->V, image_hw, 2), g, geom_v, binning_v, capacity, image_v, out, flags, counts_host, ticket,
                        count_ready_event, nullptr, stream);
}

int dgr_views_mixed_forward_render_ex(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom_v, void *binning_v,
                                      uint64_t capacity, void *image_v, const DgrImages *out, int32_t flags, uint64_t *counts_host,
                                      uint64_t ticket, void *count_ready_event, const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_views_mixed_forward_render_ex");
    if (int e = check_views_mixed(s, image_hw)) return e;
    if (int e = check_views_gaussians(s, g)) return e;
    return views_render(s, views_batch(s->V, image_hw, 2), g, geom_v, binning_v, capacity, image_v, out, flags, counts_host, ticket,
                        count_ready_event, opt, stream);
}

// dgr_views_mixed_backward* (det = NULL: not deterministic, opt = NULL: no options)
static int views_backward_mixed(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom_v, const void *binning_v,
                                uint64_t capacity, int32_t staging, const void *image_v, const int32_t *radii, const DgrImageGrads *gin,
                                const DgrGaussianGrads *gout, uint64_t stats_views, const DetArgs *det, const DgrRasterOptions *opt,
                                void *stream) {
    uint32_t flags = 0;
    const DgrCameraGrads *cam = nullptr;
    float *abs_accum = nullptr;
    if (int e = raster_flags_bwd(opt, &flags, &cam, &abs_accum)) return e;
    if (int e = check_views_mixed(s, image_hw)) return e;
    if (int e = check_views_gaussians(s, g)) return e;
    if (!geom_v || !image_v || !gin || !gout) return fail(-1, "NULL argument");
    if (staging != DGR_STAGING_SORTED && staging != DGR_STAGING_BY_ID)
        return fail(-1, "staging must be DGR_STAGING_SORTED or DGR_STAGING_BY_ID (counts_host[3] of the forward)");
    if (s->V < 64 && (stats_views >> s->V) != 0) return fail(-1, "views mixed: stats_views has a bit at or above V");
    if (abs_accum && !stats_views) return fail(-1, "views mixed: DGR_RASTER_ABS_GRAD with stats_views == 0 (no view to take the statistic from)");
    const bool any_stat = gout->xyz_gradient_accum || gout->denom || gout->max_radii2D || abs_accum;
    if (stats_views && !any_stat)
        return fail(-1, "views mixed: stats_views is non-zero but no densification statistic buffer is set");
    if (!stats_views && any_stat)
        return fail(-1, "views mixed: a densification statistic buffer is set but stats_views is 0");
    if (int e = check_views_grads(gout)) return e;
    return views_backward(s, views_batch(s->V, image_hw, 2), g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout,
                          stats_views, det, flags, cam, abs_accum, stream);
}

int dgr_views_mixed_backward(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom_v, const void *binning_v,
                             uint64_t capacity, int32_t staging, const void *image_v, const int32_t *radii, const DgrImageGrads *gin,
                             const DgrGaussianGrads *gout, uint64_t stats_views, void *stream) {
    NvtxRange nvtx_("dgr_views_mixed_backward");
    return views_backward_mixed(s, image_hw, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, stats_views, nullptr, nullptr,
                                stream);
}

int dgr_views_mixed_backward_ex(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom_v, const void *binning_v,
                                uint64_t capacity, int32_t staging, const void *image_v, const int32_t *radii, const DgrImageGrads *gin,
                                const DgrGaussianGrads *gout, uint64_t stats_views, const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_views_mixed_backward_ex");
    return views_backward_mixed(s, image_hw, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, stats_views, nullptr, opt,
                                stream);
}

int dgr_views_mixed_backward_det(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom_v, const void *binning_v,
                                 uint64_t capacity, int32_t staging, const void *image_v, const int32_t *radii, const DgrImageGrads *gin,
                                 const DgrGaussianGrads *gout, uint64_t stats_views, void *det_scratch, uint64_t det_scratch_bytes,
                                 uint64_t instances, void *stream) {
    NvtxRange nvtx_("dgr_views_mixed_backward_det");
    const DetArgs det{det_scratch, det_scratch_bytes, instances};
    return views_backward_mixed(s, image_hw, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, stats_views, &det, nullptr,
                                stream);
}

int dgr_views_mixed_backward_det_ex(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom_v, const void *binning_v,
                                    uint64_t capacity, int32_t staging, const void *image_v, const int32_t *radii, const DgrImageGrads *gin,
                                    const DgrGaussianGrads *gout, uint64_t stats_views, void *det_scratch, uint64_t det_scratch_bytes,
                                    uint64_t instances, const DgrRasterOptions *opt, void *stream) {
    NvtxRange nvtx_("dgr_views_mixed_backward_det_ex");
    const DetArgs det{det_scratch, det_scratch_bytes, instances};
    return views_backward_mixed(s, image_hw, g, geom_v, binning_v, capacity, staging, image_v, radii, gin, gout, stats_views, &det, opt,
                                stream);
}

}  // extern "C"

extern "C" {

#include "dgr_collective_api.cuh"      // dgr_peer_*: the multi-GPU entry points (not part of the single-GPU step)

size_t dgr_knn_scratch_bytes(int32_t P) { return KnnLayout(P).total; }

int dgr_dist_cuda2(int32_t P, const float *points, float *mean_dists, void *scratch_v, void *stream) {
    NvtxRange nvtx_("dgr_dist_cuda2");
    if (P < 0) return fail(-1, "P < 0");
    if (P == 0) return 0;
    if (!points || !mean_dists || !scratch_v) return fail(-1, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    char *scratch = (char *)scratch_v;
    KnnLayout L(P);
    KnnGrid *grid = reinterpret_cast<KnnGrid *>(scratch + L.off_grid);
    unsigned *cell_start = reinterpret_cast<unsigned *>(scratch + L.off_start);
    unsigned *cell_fill = reinterpret_cast<unsigned *>(scratch + L.off_fill);
    unsigned *sums = reinterpret_cast<unsigned *>(scratch + L.off_sums);
    unsigned *cid = reinterpret_cast<unsigned *>(scratch + L.off_cid);
    float4 *sorted = reinterpret_cast<float4 *>(scratch + L.off_sorted);
    DGR_CUDA(cudaMemsetAsync(grid, 0, sizeof(KnnGrid), st));
    DGR_CUDA(cudaMemsetAsync(grid, 0xff, 3 * sizeof(unsigned), st));                      // lo[] = +inf in the ordered encoding
    DGR_CUDA(cudaMemsetAsync(cell_start, 0, (L.cap + 1) * 4, st));
    DGR_CUDA(cudaMemsetAsync(cell_fill, 0, L.cap * 4, st));
    const int nb = (P + 255) / 256;
    const int nb_bbox = nb < 4 * (dev_info() ? dev_info()->sms : 132) ? nb : 4 * (dev_info() ? dev_info()->sms : 132);
    const size_t n_scan = L.cap + 1;
    DGR_KERNEL("knn_bbox", st, 0, knn_bbox_kernel<<<nb_bbox, 256, 0, st>>>(P, points, grid));
    DGR_KERNEL("knn_grid", st, 0, knn_grid_kernel<<<1, 1, 0, st>>>(P, (unsigned)L.cap, grid));
    DGR_KERNEL("knn_count", st, 0, knn_count_kernel<<<nb, 256, 0, st>>>(P, points, grid, cell_start, cid));
    DGR_KERNEL("knn_scan_sums", st, 0, knn_scan_sums_kernel<<<(unsigned)L.nblk, 1024, 0, st>>>(cell_start, n_scan, sums));
    DGR_KERNEL("knn_scan_top", st, 0, knn_scan_top_kernel<<<1, 1024, 0, st>>>(sums, L.nblk));
    DGR_KERNEL("knn_scan_apply", st, 0, knn_scan_apply_kernel<<<(unsigned)L.nblk, 1024, 0, st>>>(cell_start, n_scan, sums));
    DGR_KERNEL("knn_scatter", st, 0, knn_scatter_kernel<<<nb, 256, 0, st>>>(P, points, cid, cell_start, cell_fill, sorted));
    DGR_KERNEL("knn_query", st, 0, knn_query_kernel<<<(P + 127) / 128, 128, 0, st>>>(P, grid, cell_start, sorted, mean_dists));
    return 0;
}

size_t dgr_fields_scratch_bytes(int32_t P, int32_t num_blocks) { return FieldsLayout(P, num_blocks > 0 ? num_blocks : 1).total; }

int dgr_extract_fields(int32_t P, const float *xyz, const float *opacity_raw, const float *scaling_raw, const float *rotation_raw,
                       int32_t resolution, int32_t num_blocks, float relax_ratio, float *occ, float *center_scale, void *scratch_v,
                       void *stream) {
    NvtxRange nvtx_("dgr_extract_fields");
    if (P < 0 || resolution < 2 || num_blocks < 1) return fail(-1, "bad P / resolution / num_blocks");
    if (resolution % num_blocks != 0) return fail(-2, "resolution must be a multiple of num_blocks");
    if (num_blocks > 64) return fail(-3, "num_blocks above 64 not supported");
    const int split = resolution / num_blocks;
    const int V = split * split * split;
    if (V > 16 * kFieldThreads) return fail(-3, "more than 4096 voxels per block not supported");
    if (!occ || !scratch_v || (P > 0 && (!xyz || !opacity_raw || !scaling_raw || !rotation_raw))) return fail(-1, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    char *scratch = (char *)scratch_v;
    FieldsLayout L(P, num_blocks);
    FieldsHeader *hdr = reinterpret_cast<FieldsHeader *>(scratch + L.off_hdr);
    unsigned *cell_start = reinterpret_cast<unsigned *>(scratch + L.off_start);
    unsigned *cell_fill = reinterpret_cast<unsigned *>(scratch + L.off_fill);
    unsigned *cid = reinterpret_cast<unsigned *>(scratch + L.off_cid);
    FieldRec *rec = reinterpret_cast<FieldRec *>(scratch + L.off_rec), *sorted = reinterpret_cast<FieldRec *>(scratch + L.off_sorted);
    DGR_CUDA(cudaMemsetAsync(hdr, 0, sizeof(FieldsHeader), st));
    DGR_CUDA(cudaMemsetAsync(hdr, 0xff, 3 * sizeof(unsigned), st));
    DGR_CUDA(cudaMemsetAsync(cell_start, 0, (L.cells + 1) * 4, st));
    DGR_CUDA(cudaMemsetAsync(cell_fill, 0, L.cells * 4, st));
    const int nbk = P > 0 ? (P + 255) / 256 : 1;
    if (P > 0) {
        const int nb_bbox = nbk < 4 * (dev_info() ? dev_info()->sms : 132) ? nbk : 4 * (dev_info() ? dev_info()->sms : 132);
        DGR_KERNEL("fields_bbox", st, 0, fields_bbox_kernel<<<nb_bbox, 256, 0, st>>>(P, xyz, opacity_raw, hdr));
    }
    DGR_KERNEL("fields_prep", st, 0, fields_prep_kernel<<<nbk, 256, 0, st>>>(P, xyz, opacity_raw, scaling_raw, rotation_raw, hdr, num_blocks,
                                                                              rec, cid, cell_start, center_scale));
    DGR_KERNEL("fields_scan", st, 0, fields_scan_kernel<<<1, 1024, 0, st>>>(cell_start, (int)(L.cells + 1)));
    if (P > 0)
        DGR_KERNEL("fields_scatter", st, 0, fields_scatter_kernel<<<nbk, 256, 0, st>>>(P, cid, cell_start, cell_fill, rec, sorted));
    // reference: vmin -= block_size * relax_ratio with python floats (gs_renderer.py:222,264-265) -> one float32 operand
    const float grow = (float)((2.0 / (double)num_blocks) * (double)relax_ratio);
    const unsigned grid = (unsigned)L.cells;
    const int vpt = (V + kFieldThreads - 1) / kFieldThreads;
#define DGR_FIELDS(VPT_) DGR_KERNEL("fields_eval", st, 0, fields_eval_kernel<VPT_><<<grid, kFieldThreads, 0, st>>>(resolution, num_blocks, split, grow, cell_start, sorted, occ))
    if (vpt <= 1) DGR_FIELDS(1); else if (vpt <= 2) DGR_FIELDS(2); else if (vpt <= 4) DGR_FIELDS(4); else if (vpt <= 8) DGR_FIELDS(8); else DGR_FIELDS(16);
#undef DGR_FIELDS
    return 0;
}

int dgr_adam_step(const DgrAdamGroup *groups, int32_t n_groups, double beta1, double beta2, double eps, void *stream) {
    NvtxRange nvtx_("dgr_adam_step");
    if (!groups || n_groups < 1 || n_groups > kAdamMaxGroups) return fail(-1, "dgr_adam_step: 1..8 groups");
    AdamGroups G;
    G.n_groups = n_groups;
    unsigned long long run = 0;
    for (int k = 0; k < n_groups; k++) {
        const DgrAdamGroup &g = groups[k];
        if (g.n > 0 && (!g.param || !g.grad || !g.exp_avg || !g.exp_avg_sq)) return fail(-1, "dgr_adam_step: NULL tensor in a non-empty group");
        G.param[k] = g.param; G.grad[k] = g.grad; G.m[k] = g.exp_avg; G.v[k] = g.exp_avg_sq; G.n[k] = g.n;
        if (g.step < 1) return fail(-1, "dgr_adam_step: a tensor's step counts from 1");
        const double bc1 = 1.0 - pow(beta1, (double)g.step), bc2 = 1.0 - pow(beta2, (double)g.step);
        G.step_size[k] = (float)((double)g.lr / bc1);
        G.inv_sqrt_bc2[k] = (float)(1.0 / sqrt(bc2));
        G.start[k] = run; run += (g.n + 3) / 4;
    }
    for (int k = n_groups; k <= kAdamMaxGroups; k++) G.start[k] = run;
    G.start[n_groups] = run;
    if (run == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long blocks = (run + 255) / 256;
    const unsigned long long cap = (unsigned long long)(dev_info() ? dev_info()->sms : 132) * 16;
    if (blocks > cap) blocks = cap;
    DGR_KERNEL("adam_multi", st, 0, adam_multi_kernel<<<(unsigned)blocks, 256, 0, st>>>(G, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps));
    return 0;
}

size_t dgr_densify_scratch_bytes(int32_t P) { return DensifyLayout(P).total; }

int dgr_densify_plan(int32_t P, const float *xyz_gradient_accum, const float *denom, const float *opacity_raw, const float *scaling_raw,
                     float grad_threshold, float dense_extent, float min_opacity, float max_world, int32_t use_world,
                     void *scratch_v, uint32_t *counts_host, void *stream) {
    NvtxRange nvtx_("dgr_densify_plan");
    if (P < 0) return fail(-1, "P < 0");
    if (!scratch_v || (P > 0 && (!xyz_gradient_accum || !denom || !opacity_raw || !scaling_raw))) return fail(-1, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    char *scratch = (char *)scratch_v;
    DensifyLayout L(P);
    unsigned *counts = reinterpret_cast<unsigned *>(scratch + L.off_counts), *offsets = reinterpret_cast<unsigned *>(scratch + L.off_offsets);
    unsigned *totals = reinterpret_cast<unsigned *>(scratch + L.off_totals);
    DensifyParams prm{grad_threshold, dense_extent, min_opacity, max_world, use_world};
    if (P > 0)
        DGR_KERNEL("densify_classify", st, 0,
                   densify_classify_kernel<<<L.nblk, kDensifyThreads, 0, st>>>(P, xyz_gradient_accum, denom, opacity_raw, scaling_raw, prm,
                                                                                reinterpret_cast<unsigned char *>(scratch + L.off_class), counts));
    else
        DGR_CUDA(cudaMemsetAsync(counts, 0, 16, st));
    DGR_KERNEL("densify_offsets", st, 0, densify_offsets_kernel<<<1, 1024, 0, st>>>(P > 0 ? L.nblk : 1, counts, offsets, totals));
    if (counts_host) DGR_CUDA(cudaMemcpyAsync(counts_host, totals, 4 * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    return 0;
}

int dgr_densify_plan_ex(int32_t P, const float *xyz_gradient_accum, const float *xyz_gradient_accum_abs, const float *denom,
                        const float *opacity_raw, const float *scaling_raw, float grad_threshold, float abs_grad_threshold,
                        float dense_extent, float min_opacity, float max_world, int32_t use_world, void *scratch_v,
                        uint32_t *counts_host, void *stream) {
    NvtxRange nvtx_("dgr_densify_plan_ex");
    if (P < 0) return fail(-1, "P < 0");
    if (!scratch_v || (P > 0 && (!xyz_gradient_accum || !xyz_gradient_accum_abs || !denom || !opacity_raw || !scaling_raw)))
        return fail(-1, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    char *scratch = (char *)scratch_v;
    DensifyLayout L(P);
    unsigned *counts = reinterpret_cast<unsigned *>(scratch + L.off_counts), *offsets = reinterpret_cast<unsigned *>(scratch + L.off_offsets);
    unsigned *totals = reinterpret_cast<unsigned *>(scratch + L.off_totals);
    DensifyParams prm{grad_threshold, dense_extent, min_opacity, max_world, use_world};
    if (P > 0)
        DGR_KERNEL("densify_classify_abs", st, 0,
                   densify_classify_abs_kernel<<<L.nblk, kDensifyThreads, 0, st>>>(P, xyz_gradient_accum, xyz_gradient_accum_abs, denom, opacity_raw,
                                                                                    scaling_raw, prm, abs_grad_threshold,
                                                                                    reinterpret_cast<unsigned char *>(scratch + L.off_class), counts));
    else
        DGR_CUDA(cudaMemsetAsync(counts, 0, 16, st));
    DGR_KERNEL("densify_offsets", st, 0, densify_offsets_kernel<<<1, 1024, 0, st>>>(P > 0 ? L.nblk : 1, counts, offsets, totals));
    if (counts_host) DGR_CUDA(cudaMemcpyAsync(counts_host, totals, 4 * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    return 0;
}

int dgr_densify_apply(int32_t P, const DgrDensifyTensors *t, const float *noise, const void *scratch_v, void *stream) {
    NvtxRange nvtx_("dgr_densify_apply");
    if (P < 0 || !t || !scratch_v) return fail(-1, "bad argument");
    if (P == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const char *scratch = (const char *)scratch_v;
    DensifyLayout L(P);
    DensifyTensors T;
    for (int k = 0; k < kDensifyTensors; k++) {
        T.in[k] = t->in[k]; T.m_in[k] = t->exp_avg_in[k]; T.v_in[k] = t->exp_avg_sq_in[k];
        T.out[k] = t->out[k]; T.m_out[k] = t->exp_avg_out[k]; T.v_out[k] = t->exp_avg_sq_out[k];
        T.width[k] = t->width[k];
        if (t->width[k] < 0) return fail(-1, "negative row width");
        if (t->width[k] > 0 && (!T.in[k] || !T.m_in[k] || !T.v_in[k])) return fail(-1, "NULL input tensor");
    }
    if (T.width[0] != 3 || T.width[3] != 1 || T.width[4] != 3 || T.width[5] != 4) return fail(-1, "row widths must be xyz 3, opacity 1, scaling 3, rotation 4");
    DGR_KERNEL("densify_apply", st, 0,
               densify_apply_kernel<<<L.nblk, kDensifyThreads, 0, st>>>(P, reinterpret_cast<const unsigned char *>(scratch + L.off_class),
                                                                        reinterpret_cast<const unsigned *>(scratch + L.off_offsets),
                                                                        reinterpret_cast<const unsigned *>(scratch + L.off_totals), T, noise));
    return 0;
}

int dgr_mark_visible(int32_t P, const float *means3D, const float *viewmatrix, const float *projmatrix,
                     uint8_t *present, void *stream) {
    NvtxRange nvtx_("dgr_mark_visible");
    (void)projmatrix;
    if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !present))) return fail(-1, "bad argument");
    if (P == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    DGR_KERNEL("mark_visible", st, 0, mark_visible_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, means3D, viewmatrix, present));
    return 0;
}

int dgr_debug_geom(int32_t P, int32_t H, int32_t W, const void *geom_v, float *mean_px, float *depth, float *conic, float *rgb,
                   int32_t *aabb, uint32_t *tiles_touched, void *stream) {
    if (P <= 0) return 0;
    if (!geom_v) return fail(-1, "geom is NULL");
    const char *geom = (const char *)geom_v;
    GeomLayout L(P, H, W);
    cudaStream_t st = (cudaStream_t)stream;
    DGR_KERNEL("debug_geom", st, 0,
               debug_geom_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, reinterpret_cast<const Rec *>(geom + L.off_rec),
                                                                reinterpret_cast<const unsigned *>(geom + L.off_touched), mean_px,
                                                                depth, conic, rgb, aabb, tiles_touched));
    return 0;
}

}  // extern "C"
