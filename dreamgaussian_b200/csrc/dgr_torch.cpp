// dgr_torch.cpp — compiled host layer over the C ABI (include/dgr_b200.h) for PyTorch callers.
//
// The ctypes path (dreamgaussian_b200/rasterizer.py) costs ~0.25 ms of Python per forward+backward — as much as the GPU
// work at 100k Gaussians (tools/host_overhead.py).  This module does the same calls from C++: tensor checks, scratch
// allocation through the caching allocator, the speculative-capacity protocol of dgr_forward_render (count event, re-run
// on a low guess) and the backward, ~20 µs of host time each.  It adds NO arithmetic: every kernel still lives in
// libdgr_b200.so, which this module links.  Mirrors rasterize_gaussians / rasterize_gaussians_backward of the reference
// package's ext.cpp [EXT] (called from /root/reference/gs_renderer.py:800-809 through GaussianRasterizer).
#include <torch/extension.h>
#include <cstdint>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime.h>

#include <mutex>
#include <unordered_map>
#include <vector>

#include "../../include/dgr_b200.h"

namespace {

using torch::Tensor;
using OptTensor = c10::optional<Tensor>;

const float *fptr(const OptTensor &t) { return (t.has_value() && t->defined() && t->numel() > 0) ? t->data_ptr<float>() : nullptr; }
float *fptr_mut(const OptTensor &t) { return (t.has_value() && t->defined() && t->numel() > 0) ? t->data_ptr<float>() : nullptr; }

Tensor dev_f32(const Tensor &t, const char *name) {
    TORCH_CHECK(t.is_cuda(), name, " is on ", t.device(), ": this rasterizer has no CPU path (it runs as sm_90a CUDA kernels in libdgr_b200.so)");
    Tensor r = t.scalar_type() == torch::kFloat32 ? t : t.to(torch::kFloat32);
    r = r.contiguous();
    // the kernels read rotations / SH rows with 128-bit loads and stage inputs with bulk TMA: a view that starts off a 16-byte
    // boundary gets its own (aligned) allocation
    if (r.numel() > 0 && (reinterpret_cast<uintptr_t>(r.data_ptr()) & 15u) != 0) r = r.clone(at::MemoryFormat::Contiguous);
    return r;
}
OptTensor opt_f32(const OptTensor &t, const char *name) {
    if (!t.has_value() || !t->defined() || (t->numel() == 0 && t->dim() <= 1)) return c10::nullopt;
    return dev_f32(*t, name);
}
void check(int rc) { TORCH_CHECK(rc == 0, "libdgr_b200: ", dgr_last_error()); }

struct State {                       // what one forward leaves behind for its backward (keeps every tensor alive)
    DgrSettings s;
    DgrGaussians g;
    Tensor bg, view, proj, campos;
    Tensor means3D, opac;
    OptTensor sh, colors, scales, rots, cov3D, sh_rest;
    Tensor geom, binning, image, radii;      // NOT the differentiable outputs: State -> output -> grad_fn -> ctx -> State would be an
                                             // uncollectable cycle through C++ reference counts (radii is non-differentiable: no grad_fn)
    int64_t capacity = 0, n_inst = 0;
    int32_t staging = DGR_STAGING_SORTED;    // record staging the last stage-2 run chose (counts_host[3]): the backward's too
    int device = 0;
    DgrRasterOptions opt{0u};                // the forward's options: its backward takes the same
    Tensor weight_sum, weight_max;           // contrib: the blending-weight statistics of the last stage-2 run, [P]
};

// DGR_RASTER_CONTRIB for the stage-2 render calls: the outputs [records] (shape `shape`) and their scratch, and the options that
// carry them; without contrib, NULL options (the counterpart's call).
struct ContribOut {
    DgrContrib c{};
    DgrRasterOptions opt{0u, nullptr, nullptr, nullptr};
    Tensor weight_sum, weight_max, scratch;
    ContribOut(bool contrib, at::IntArrayRef shape, const torch::TensorOptions &f32) {
        if (!contrib) return;
        weight_sum = torch::empty(shape, f32); weight_max = torch::empty(shape, f32);
        const int64_t records = weight_sum.numel();
        scratch = torch::empty({std::max<int64_t>((int64_t)dgr_contrib_scratch_bytes(records), 1)}, f32.dtype(torch::kUInt8));
        c = DgrContrib{records ? weight_sum.data_ptr<float>() : nullptr, records ? weight_max.data_ptr<float>() : nullptr, scratch.data_ptr(),
                       (uint64_t)scratch.numel()};
        opt.flags = DGR_RASTER_CONTRIB;
        opt.contrib = &c;
    }
    const DgrRasterOptions *options() const { return opt.flags ? &opt : nullptr; }
};

// scratch of the deterministic backward (dgr_*_backward_det), taken when torch.use_deterministic_algorithms(True) is in effect
// (warn_only included) at the time the backward runs
Tensor det_scratch(int64_t instances, int64_t records, const torch::TensorOptions &like) {
    return torch::empty({(int64_t)dgr_det_scratch_bytes((uint64_t)instances, records)}, like.dtype(torch::kUInt8));
}

struct Hint { int64_t cap; bool big; };
std::mutex g_mu;
std::unordered_map<uint64_t, Hint> g_hints;
uint64_t hint_key(int dev, int64_t P, int H, int W) { return ((uint64_t)dev << 58) ^ ((uint64_t)P << 28) ^ ((uint64_t)H << 14) ^ (uint64_t)W; }

struct SyncObjs { Tensor counts; void *event = nullptr; uint64_t ticket = 0; };
SyncObjs &sync_objs(int dev) {
    thread_local std::unordered_map<int, SyncObjs> per_dev;
    SyncObjs &o = per_dev[dev];
    if (!o.event) {
        o.counts = torch::zeros({4}, torch::dtype(torch::kInt64)).pin_memory();
        o.event = dgr_event_create();
        TORCH_CHECK(o.event, "libdgr_b200: could not create a CUDA event");
    }
    return o;
}

std::tuple<Tensor, Tensor, Tensor, Tensor, std::shared_ptr<State>>
forward(int64_t H, int64_t W, double tanfovx, double tanfovy, double scale_modifier, int64_t sh_degree, bool prefiltered, bool debug,
        const Tensor &bg, const Tensor &view, const Tensor &proj, const Tensor &campos, const Tensor &means3D, const OptTensor &sh,
        const OptTensor &colors, const Tensor &opac, const OptTensor &scales, const OptTensor &rots, const OptTensor &cov3D,
        const OptTensor &sh_rest, bool activations, bool antialiasing, bool contrib) {
    auto st = std::make_shared<State>();
    st->opt.flags = antialiasing ? DGR_RASTER_ANTIALIAS : 0u;
    st->means3D = dev_f32(means3D, "means3D");
    const c10::cuda::CUDAGuard guard(st->means3D.device());
    st->device = st->means3D.get_device();
    st->opac = dev_f32(opac, "opacities");
    st->bg = dev_f32(bg, "bg"); st->view = dev_f32(view, "viewmatrix"); st->proj = dev_f32(proj, "projmatrix"); st->campos = dev_f32(campos, "campos");
    TORCH_CHECK_VALUE(st->bg.numel() == 3 && st->view.numel() == 16 && st->proj.numel() == 16 && st->campos.numel() == 3,
                "bg/campos must have 3 elements, viewmatrix/projmatrix 16");
    st->sh = opt_f32(sh, "shs"); st->colors = opt_f32(colors, "colors_precomp"); st->scales = opt_f32(scales, "scales");
    st->rots = opt_f32(rots, "rotations"); st->cov3D = opt_f32(cov3D, "cov3D_precomp");
    st->sh_rest = activations ? opt_f32(sh_rest, "features_rest") : c10::nullopt;
    if (st->sh_rest.has_value() && st->sh_rest->numel() == 0) st->sh_rest = c10::nullopt;
    TORCH_CHECK_VALUE(st->means3D.dim() == 2 && st->means3D.size(1) == 3, "means3D must have dimensions (num_points, 3)");
    const int64_t P = st->means3D.size(0);
    int64_t M = 0;
    if (st->sh.has_value()) {
        TORCH_CHECK_VALUE(st->sh->dim() == 3 && st->sh->size(0) == P && st->sh->size(2) == 3, "shs must have dimensions (num_points, num_coeffs, 3)");
        M = st->sh->size(1);
    }
    if (activations) {
        TORCH_CHECK_VALUE(st->sh.has_value() && st->sh->size(1) == 1, "features_dc must have dimensions (num_points, 1, 3)");
        if (st->sh_rest.has_value()) {
            TORCH_CHECK_VALUE(st->sh_rest->dim() == 3 && st->sh_rest->size(0) == P && st->sh_rest->size(2) == 3, "features_rest must have dimensions (num_points, num_coeffs - 1, 3)");
            M = 1 + st->sh_rest->size(1);
        }
    }
    TORCH_CHECK_VALUE(!st->colors.has_value() || st->colors->numel() == P * 3, "colors_precomp must have dimensions (num_points, 3)");
    TORCH_CHECK_VALUE(!st->scales.has_value() || st->scales->numel() == P * 3, "scales must have dimensions (num_points, 3)");
    TORCH_CHECK_VALUE(!st->rots.has_value() || st->rots->numel() == P * 4, "rotations must have dimensions (num_points, 4)");
    TORCH_CHECK_VALUE(!st->cov3D.has_value() || st->cov3D->numel() == P * 6, "cov3D_precomp must have dimensions (num_points, 6)");
    TORCH_CHECK_VALUE(st->opac.numel() == P, "opacities must have dimensions (num_points, 1)");

    st->s = DgrSettings{(int32_t)H, (int32_t)W, (float)tanfovx, (float)tanfovy, (float)scale_modifier, (int32_t)sh_degree,
                        prefiltered ? 1 : 0, debug ? 1 : 0, st->bg.data_ptr<float>(), st->view.data_ptr<float>(), st->proj.data_ptr<float>(),
                        st->campos.data_ptr<float>()};
    st->g = DgrGaussians{(int32_t)P, (int32_t)M, st->means3D.numel() ? st->means3D.data_ptr<float>() : nullptr, fptr(st->sh), fptr(st->colors),
                         st->opac.numel() ? st->opac.data_ptr<float>() : nullptr, fptr(st->scales), fptr(st->rots), fptr(st->cov3D),
                         fptr(st->sh_rest), activations ? 1 : 0};
    const auto f32 = st->means3D.options();
    const auto u8 = f32.dtype(torch::kUInt8);
    Tensor img = torch::empty({5, H, W}, f32);               // color (3) | depth (1) | alpha (1): one allocation
    Tensor color = img.narrow(0, 0, 3), depth = img.narrow(0, 3, 1), alpha = img.narrow(0, 4, 1);
    st->radii = torch::empty({P}, f32.dtype(torch::kInt32));
    st->geom = torch::empty({(int64_t)dgr_geom_bytes((int32_t)P, (int32_t)H, (int32_t)W)}, u8);
    st->image = torch::empty({(int64_t)dgr_image_bytes((int32_t)H, (int32_t)W)}, u8);
    void *stream = c10::cuda::getCurrentCUDAStream(st->device).stream();
    check(dgr_forward_preprocess_ex(&st->s, &st->g, st->geom.data_ptr(), st->image.data_ptr(), st->radii.data_ptr<int32_t>(), &st->opt,
                                    stream));
    DgrImages out{color.data_ptr<float>(), depth.data_ptr<float>(), alpha.data_ptr<float>(), st->radii.data_ptr<int32_t>()};
    Hint hint{std::max<int64_t>(65536, 16 * P), true};
    const uint64_t key = hint_key(st->device, P, (int)H, (int)W);
    { std::lock_guard<std::mutex> lk(g_mu); auto it = g_hints.find(key); if (it != g_hints.end()) hint = it->second; }
    SyncObjs &so = sync_objs(st->device);
    int64_t cap = hint.cap, n_inst = 0, n_big = 0;
    bool big = hint.big;
    int rerun = 0;
    const ContribOut co(contrib, {P}, f32);                  // every stage-2 run rewrites it: the last run's values are kept
    while (true) {
        st->binning = torch::empty({(int64_t)dgr_binning_bytes((uint64_t)cap, (int32_t)H, (int32_t)W)}, u8);
        // ticket protocol: the scan kernel writes the counts and then the ticket into the pinned buffer; nothing but kernels
        // goes into the stream (programmatic dependent launches chain the whole forward) and the host polls the ticket
        const uint64_t ticket = ++so.ticket;
        volatile uint64_t *cnt = reinterpret_cast<volatile uint64_t *>(so.counts.data_ptr<int64_t>());
        if (contrib)
            check(dgr_forward_render_ex(&st->s, &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)cap, st->image.data_ptr(), &out,
                                        (big ? DGR_FLAG_BIG_TILES : 0) | rerun, reinterpret_cast<uint64_t *>(so.counts.data_ptr<int64_t>()), ticket,
                                        nullptr, co.options(), stream));
        else
            check(dgr_forward_render(&st->s, &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)cap, st->image.data_ptr(), &out,
                                     (big ? DGR_FLAG_BIG_TILES : 0) | rerun, reinterpret_cast<uint64_t *>(so.counts.data_ptr<int64_t>()), ticket, nullptr, stream));
        {
            pybind11::gil_scoped_release nogil;              // the wait for the early instance count
            uint64_t spins = 0;
            while (cnt[2] != ticket) {
                if ((++spins & 0xfffff) == 0) {              // every ~1M polls: has the stream failed or finished without the ticket?
                    const cudaError_t q = cudaStreamQuery((cudaStream_t)stream);
                    if (q != cudaErrorNotReady && cnt[2] != ticket) {
                        TORCH_CHECK(q == cudaSuccess, "libdgr_b200: forward failed on the device: ", cudaGetErrorString(q));
                        TORCH_CHECK(false, "libdgr_b200: the instance count never arrived (is the count buffer device-mapped?)");
                    }
                }
            }
        }
        n_inst = so.counts.data_ptr<int64_t>()[0]; n_big = so.counts.data_ptr<int64_t>()[1];
        if (n_inst <= cap && (big || n_big == 0)) break;
        cap = std::max<int64_t>(cap, (int64_t)(n_inst * 1.25) + 4096);      // a guess was wrong: redo stage 2 (rare)
        big = big || n_big > 0;
        rerun = DGR_FLAG_RERUN;
    }
    { std::lock_guard<std::mutex> lk(g_mu); g_hints[key] = Hint{std::max<int64_t>((int64_t)(n_inst * 1.25) + 4096, 65536), n_big > 0}; }
    st->capacity = cap; st->n_inst = n_inst; st->staging = (int32_t)so.counts.data_ptr<int64_t>()[3];
    st->weight_sum = co.weight_sum; st->weight_max = co.weight_max;
    return {color, st->radii, depth, alpha, st};
}

// Camera gradients (DGR_RASTER_CAMERA_GRADS): appends dL/dviewmatrix, dL/dprojmatrix ([V,16] each, [16] for V = 0: single view)
// and dL/dcampos ([V,3] / [3]) to g and returns the options of the backward call; without camera, the forward's options unchanged.
// absgrad (xyz_gradient_accum_abs [P]): DGR_RASTER_ABS_GRAD with it.
struct CameraOut { DgrCameraGrads cg{}; DgrRasterOptions opt{0u, nullptr, nullptr}; Tensor scratch; };
void camera_out(bool camera, int64_t V, int64_t P, const DgrRasterOptions &fwd, const torch::TensorOptions &f32, std::vector<Tensor> &g,
                CameraOut &c, const OptTensor &absgrad) {
    c.opt = fwd;
    if (float *a = fptr_mut(absgrad)) {
        TORCH_CHECK_VALUE(absgrad->is_cuda() && absgrad->scalar_type() == torch::kFloat32 && absgrad->is_contiguous() && absgrad->numel() == P,
                          "xyz_gradient_accum_abs must be a contiguous float32 CUDA tensor of num_points elements");
        c.opt.flags |= DGR_RASTER_ABS_GRAD;
        c.opt.xyz_gradient_accum_abs = a;
    }
    if (!camera) return;
    const std::vector<int64_t> s16 = V ? std::vector<int64_t>{V, 16} : std::vector<int64_t>{16};
    const std::vector<int64_t> s3 = V ? std::vector<int64_t>{V, 3} : std::vector<int64_t>{3};
    g.push_back(torch::empty(s16, f32)); g.push_back(torch::empty(s16, f32)); g.push_back(torch::empty(s3, f32));
    c.scratch = torch::empty({(int64_t)dgr_camera_grad_scratch_bytes((int32_t)std::max<int64_t>(V, 1), (int32_t)P)}, f32.dtype(torch::kUInt8));
    const size_t n = g.size();
    c.cg = DgrCameraGrads{g[n - 3].data_ptr<float>(), g[n - 2].data_ptr<float>(), g[n - 1].data_ptr<float>(), c.scratch.data_ptr(),
                          (uint64_t)c.scratch.numel()};
    c.opt.flags |= DGR_RASTER_CAMERA_GRADS;
    c.opt.camera = &c.cg;
}

// grads: (means3D, means2D, shs | features_dc, colors, opacities, scales, rotations, cov3D, features_rest); undefined where not applicable;
// camera: + (dL/dviewmatrix [16], dL/dprojmatrix [16], dL/dcampos [3])
std::vector<Tensor> backward(const std::shared_ptr<State> &st, const OptTensor &gC, const OptTensor &gD, const OptTensor &gA, bool accumulate,
                             const std::vector<OptTensor> &out, const OptTensor &xyz_gradient_accum, const OptTensor &denom,
                             const OptTensor &max_radii2D, int64_t push_addr, bool camera, const OptTensor &absgrad) {
    const c10::cuda::CUDAGuard guard(st->means3D.device());
    const int64_t P = st->g.P, M = st->g.M;
    const auto f32 = st->means3D.options();
    OptTensor c = gC.has_value() && gC->defined() ? OptTensor(dev_f32(*gC, "grad_color")) : c10::nullopt;
    OptTensor d = gD.has_value() && gD->defined() ? OptTensor(dev_f32(*gD, "grad_depth")) : c10::nullopt;
    OptTensor a = gA.has_value() && gA->defined() ? OptTensor(dev_f32(*gA, "grad_alpha")) : c10::nullopt;
    std::vector<Tensor> g(9);
    auto pick = [&](size_t i, bool wanted, c10::IntArrayRef shape) {
        if (i < out.size() && out[i].has_value() && out[i]->defined()) g[i] = *out[i];
        else if (wanted) g[i] = torch::empty(shape, f32);
    };
    const bool act = st->g.activations != 0;
    pick(0, true, {P, 3}); pick(1, true, {P, 3});
    pick(2, st->sh.has_value(), {P, act ? 1 : M, 3});
    pick(3, st->colors.has_value(), {P, 3});
    pick(4, true, {P, 1});
    pick(5, st->scales.has_value(), {P, 3}); pick(6, st->rots.has_value(), {P, 4}); pick(7, st->cov3D.has_value(), {P, 6});
    pick(8, act && st->sh_rest.has_value(), {P, M - 1, 3});
    auto gp = [&](size_t i) -> float * { return g[i].defined() && g[i].numel() > 0 ? g[i].data_ptr<float>() : nullptr; };
    DgrImageGrads gin{fptr(c), fptr(d), fptr(a)};
    DgrGaussianGrads gout{gp(0), gp(1), gp(2), gp(3), gp(4), gp(5), gp(6), gp(7), accumulate ? 1 : 0, gp(8),
                          fptr_mut(xyz_gradient_accum), fptr_mut(denom), fptr_mut(max_radii2D),
                          reinterpret_cast<const DgrPeerPush *>(push_addr)};      // host struct kept alive by the caller (0 = none)
    CameraOut cam;
    camera_out(camera, 0, P, st->opt, f32, g, cam, absgrad);
    void *stream = c10::cuda::getCurrentCUDAStream(st->device).stream();
    if (at::globalContext().deterministicAlgorithms()) {
        Tensor det = det_scratch(st->n_inst, P, f32);
        check(dgr_backward_det_ex(&st->s, &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)st->capacity, st->staging,
                                  st->image.data_ptr(), st->radii.data_ptr<int32_t>(), nullptr, &gin, &gout, det.data_ptr(),
                                  (uint64_t)det.numel(), (uint64_t)st->n_inst, &cam.opt, stream));
        return g;
    }
    check(dgr_backward_ex(&st->s, &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)st->capacity, st->staging, st->image.data_ptr(),
                          st->radii.data_ptr<int32_t>(), nullptr, &gin, &gout, &cam.opt, stream));
    return g;
}

// ---- batched cameras (DgrViews, dgr_views_*): one cloud, V same-size views per call; dgr_views_mixed_*: a size per view ------
struct ViewsState {
    DgrViews s;
    std::vector<int32_t> hw;         // mixed sizes: [V,2] (height, width) on the host; empty for the same-size call
    DgrGaussians g;
    Tensor tanfov, bg, view, proj, campos;
    Tensor means3D, opac;
    OptTensor sh, scales, rots, sh_rest;
    Tensor geom, binning, image, radii;
    int64_t capacity = 0, n_inst = 0;
    int32_t staging = DGR_STAGING_SORTED;
    int device = 0;
    DgrRasterOptions opt{0u};
    Tensor weight_sum, weight_max;   // contrib: [V,P]
};

std::unordered_map<uint64_t, Hint> g_views_hints;       // keyed by (device, P, H, W, V), apart from the single-view hints
uint64_t views_hint_key(int dev, int64_t P, int H, int W, int V) {
    uint64_t h = 1469598103934665603ull;
    for (uint64_t x : {(uint64_t)dev, (uint64_t)P, (uint64_t)H, (uint64_t)W, (uint64_t)V}) { h ^= x; h *= 1099511628211ull; }
    return h;
}

std::unordered_map<uint64_t, Hint> g_views_mixed_hints; // keyed by (device, P, the views' sizes), apart from the other hints
uint64_t views_mixed_hint_key(int dev, int64_t P, const std::vector<int32_t> &hw) {
    uint64_t h = 1469598103934665603ull;
    auto mix = [&](uint64_t x) { h ^= x; h *= 1099511628211ull; };
    mix((uint64_t)dev); mix((uint64_t)P); mix((uint64_t)hw.size());
    for (int32_t x : hw) mix((uint64_t)(uint32_t)x);
    return h;
}

// instance capacity the binning buffer may be sized for: the 32-bit positions of the kernels, and half the free device memory
int64_t views_capacity_ceiling(int64_t V, int64_t H, int64_t W) {
    size_t free_b = 0, total_b = 0;
    int64_t ceil = 0xfffffffell;
    if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) {
        const int64_t per = (int64_t)dgr_views_binning_bytes(1 << 20, (int32_t)V, (int32_t)H, (int32_t)W) >> 20;   // bytes per instance
        ceil = std::min<int64_t>(ceil, std::max<int64_t>(65536, (int64_t)(free_b / 2) / std::max<int64_t>(per, 1)));
    }
    return ceil;
}

// hw: empty = the same-size call at H x W; else the [V,2] sizes of the mixed call (H, W unused), flat outputs
std::tuple<Tensor, Tensor, Tensor, Tensor, std::shared_ptr<ViewsState>>
views_forward_impl(int64_t H, int64_t W, const std::vector<int32_t> &hw, double scale_modifier, int64_t sh_degree, bool debug,
                   const Tensor &tanfov, const Tensor &bg, const Tensor &view, const Tensor &proj, const Tensor &campos, const Tensor &means3D,
                   const Tensor &sh, const Tensor &opac, const Tensor &scales, const Tensor &rots, const OptTensor &sh_rest, bool activations,
                   bool antialiasing, bool contrib) {
    auto st = std::make_shared<ViewsState>();
    st->hw = hw;
    st->opt.flags = antialiasing ? DGR_RASTER_ANTIALIAS : 0u;
    const bool mixed = !hw.empty();
    st->means3D = dev_f32(means3D, "means3D");
    const c10::cuda::CUDAGuard guard(st->means3D.device());
    st->device = st->means3D.get_device();
    st->opac = dev_f32(opac, "opacities");
    st->tanfov = dev_f32(tanfov, "tanfov"); st->bg = dev_f32(bg, "bg"); st->view = dev_f32(view, "viewmatrix");
    st->proj = dev_f32(proj, "projmatrix"); st->campos = dev_f32(campos, "campos");
    const int64_t V = st->bg.size(0);
    TORCH_CHECK_VALUE(!mixed || (int64_t)hw.size() == 2 * V, "image_hw must have dimensions (num_views, 2)");
    TORCH_CHECK_VALUE(st->tanfov.numel() == 2 * V && st->bg.numel() == 3 * V && st->view.numel() == 16 * V && st->proj.numel() == 16 * V &&
                      st->campos.numel() == 3 * V, "per-view tanfov [V,2], bg / campos [V,3], viewmatrix / projmatrix [V,16] expected");
    st->sh = dev_f32(sh, "shs"); st->scales = dev_f32(scales, "scales"); st->rots = dev_f32(rots, "rotations");
    st->sh_rest = activations ? opt_f32(sh_rest, "features_rest") : c10::nullopt;
    if (st->sh_rest.has_value() && st->sh_rest->numel() == 0) st->sh_rest = c10::nullopt;
    TORCH_CHECK_VALUE(st->means3D.dim() == 2 && st->means3D.size(1) == 3, "means3D must have dimensions (num_points, 3)");
    const int64_t P = st->means3D.size(0);
    TORCH_CHECK_VALUE(st->sh->dim() == 3 && st->sh->size(0) == P && st->sh->size(2) == 3, "shs must have dimensions (num_points, num_coeffs, 3)");
    int64_t M = st->sh->size(1);
    if (activations) {
        TORCH_CHECK_VALUE(M == 1, "features_dc must have dimensions (num_points, 1, 3)");
        if (st->sh_rest.has_value()) {
            TORCH_CHECK_VALUE(st->sh_rest->dim() == 3 && st->sh_rest->size(0) == P && st->sh_rest->size(2) == 3, "features_rest must have dimensions (num_points, num_coeffs - 1, 3)");
            M = 1 + st->sh_rest->size(1);
        }
    }
    TORCH_CHECK_VALUE(st->scales->numel() == P * 3, "scales must have dimensions (num_points, 3)");
    TORCH_CHECK_VALUE(st->rots->numel() == P * 4, "rotations must have dimensions (num_points, 4)");
    TORCH_CHECK_VALUE(st->opac.numel() == P, "opacities must have dimensions (num_points, 1)");
    st->s = DgrViews{(int32_t)V, (int32_t)H, (int32_t)W, (float)scale_modifier, (int32_t)sh_degree, debug ? 1 : 0, st->tanfov.data_ptr<float>(),
                     st->bg.data_ptr<float>(), st->view.data_ptr<float>(), st->proj.data_ptr<float>(), st->campos.data_ptr<float>()};
    st->g = DgrGaussians{(int32_t)P, (int32_t)M, st->means3D.numel() ? st->means3D.data_ptr<float>() : nullptr, fptr(st->sh), nullptr,
                         st->opac.numel() ? st->opac.data_ptr<float>() : nullptr, fptr(st->scales), fptr(st->rots), nullptr,
                         fptr(st->sh_rest), activations ? 1 : 0};
    const auto f32 = st->means3D.options();
    const auto u8 = f32.dtype(torch::kUInt8);
    Tensor color, depth, alpha;
    const int32_t *ihw = mixed ? hw.data() : nullptr;
    if (mixed) {                     // flat: view v's blocks at pixel pix_off[v] (include/dgr_b200.h)
        int64_t pix = 0;
        for (int64_t v = 0; v < V; v++) pix += (int64_t)hw[2 * v] * hw[2 * v + 1];
        color = torch::empty({3 * pix}, f32); depth = torch::empty({pix}, f32); alpha = torch::empty({pix}, f32);
    } else {
        color = torch::empty({V, 3, H, W}, f32); depth = torch::empty({V, 1, H, W}, f32); alpha = torch::empty({V, 1, H, W}, f32);
    }
    st->radii = torch::empty({V, P}, f32.dtype(torch::kInt32));
    void *stream = c10::cuda::getCurrentCUDAStream(st->device).stream();
    if (mixed) {
        const size_t gb = dgr_views_mixed_geom_bytes((int32_t)V, (int32_t)P, ihw), ib = dgr_views_mixed_image_bytes((int32_t)V, ihw);
        st->geom = torch::empty({(int64_t)std::max<size_t>(gb, 1)}, u8);
        st->image = torch::empty({(int64_t)std::max<size_t>(ib, 1)}, u8);
        check(dgr_views_mixed_forward_preprocess_ex(&st->s, ihw, &st->g, st->geom.data_ptr(), st->image.data_ptr(),
                                                    st->radii.data_ptr<int32_t>(), &st->opt, stream));
    } else {
        st->geom = torch::empty({(int64_t)dgr_views_geom_bytes((int32_t)V, (int32_t)P, (int32_t)H, (int32_t)W)}, u8);
        st->image = torch::empty({(int64_t)dgr_views_image_bytes((int32_t)V, (int32_t)H, (int32_t)W)}, u8);
        check(dgr_views_forward_preprocess_ex(&st->s, &st->g, st->geom.data_ptr(), st->image.data_ptr(), st->radii.data_ptr<int32_t>(), &st->opt,
                                              stream));
    }
    DgrImages out{color.data_ptr<float>(), depth.data_ptr<float>(), alpha.data_ptr<float>(), st->radii.data_ptr<int32_t>()};
    const int64_t ceiling = views_capacity_ceiling(V, H, W);
    Hint hint{std::min<int64_t>(std::max<int64_t>(65536, 16 * P * V), ceiling), true};
    auto &hints = mixed ? g_views_mixed_hints : g_views_hints;
    const uint64_t key = mixed ? views_mixed_hint_key(st->device, P, hw) : views_hint_key(st->device, P, (int)H, (int)W, (int)V);
    { std::lock_guard<std::mutex> lk(g_mu); auto it = hints.find(key); if (it != hints.end()) hint = it->second; }
    SyncObjs &so = sync_objs(st->device);
    int64_t cap = hint.cap, n_inst = 0, n_big = 0;
    bool big = hint.big;
    int rerun = 0;
    const ContribOut co(contrib, {V, P}, f32);
    while (true) {
        st->binning = torch::empty({(int64_t)dgr_views_binning_bytes((uint64_t)cap, (int32_t)V, (int32_t)H, (int32_t)W)}, u8);
        const uint64_t ticket = ++so.ticket;
        volatile uint64_t *cnt = reinterpret_cast<volatile uint64_t *>(so.counts.data_ptr<int64_t>());
        uint64_t *counts = reinterpret_cast<uint64_t *>(so.counts.data_ptr<int64_t>());
        if (mixed && contrib)
            check(dgr_views_mixed_forward_render_ex(&st->s, ihw, &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)cap,
                                                    st->image.data_ptr(), &out, (big ? DGR_FLAG_BIG_TILES : 0) | rerun, counts, ticket, nullptr,
                                                    co.options(), stream));
        else if (mixed)
            check(dgr_views_mixed_forward_render(&st->s, ihw, &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)cap, st->image.data_ptr(),
                                                 &out, (big ? DGR_FLAG_BIG_TILES : 0) | rerun, counts, ticket, nullptr, stream));
        else if (contrib)
            check(dgr_views_forward_render_ex(&st->s, &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)cap, st->image.data_ptr(),
                                              &out, (big ? DGR_FLAG_BIG_TILES : 0) | rerun, counts, ticket, nullptr, co.options(), stream));
        else
            check(dgr_views_forward_render(&st->s, &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)cap, st->image.data_ptr(), &out,
                                           (big ? DGR_FLAG_BIG_TILES : 0) | rerun, counts, ticket, nullptr, stream));
        {
            pybind11::gil_scoped_release nogil;
            uint64_t spins = 0;
            while (cnt[2] != ticket) {
                if ((++spins & 0xfffff) == 0) {
                    const cudaError_t q = cudaStreamQuery((cudaStream_t)stream);
                    if (q != cudaErrorNotReady && cnt[2] != ticket) {
                        TORCH_CHECK(q == cudaSuccess, "libdgr_b200: forward failed on the device: ", cudaGetErrorString(q));
                        TORCH_CHECK(false, "libdgr_b200: the instance count never arrived (is the count buffer device-mapped?)");
                    }
                }
            }
        }
        n_inst = so.counts.data_ptr<int64_t>()[0]; n_big = so.counts.data_ptr<int64_t>()[1];
        if (n_inst <= cap && (big || n_big == 0)) break;
        TORCH_CHECK(n_inst < 0xffffffffll, "libdgr_b200: the batch has ", n_inst, " tile instances, above the 2^32-1 the kernels address");
        cap = std::min<int64_t>(std::max<int64_t>(cap, (int64_t)(n_inst * 1.25) + 4096), 0xfffffffell);
        big = big || n_big > 0;
        rerun = DGR_FLAG_RERUN;
    }
    { std::lock_guard<std::mutex> lk(g_mu);
      hints[key] = Hint{std::min<int64_t>(std::max<int64_t>((int64_t)(n_inst * 1.25) + 4096, 65536), 0xfffffffell), n_big > 0}; }
    st->capacity = cap; st->n_inst = n_inst; st->staging = (int32_t)so.counts.data_ptr<int64_t>()[3];
    st->weight_sum = co.weight_sum; st->weight_max = co.weight_max;
    return {color, st->radii, depth, alpha, st};
}

std::tuple<Tensor, Tensor, Tensor, Tensor, std::shared_ptr<ViewsState>>
views_forward(int64_t H, int64_t W, double scale_modifier, int64_t sh_degree, bool debug, const Tensor &tanfov, const Tensor &bg,
              const Tensor &view, const Tensor &proj, const Tensor &campos, const Tensor &means3D, const Tensor &sh, const Tensor &opac,
              const Tensor &scales, const Tensor &rots, const OptTensor &sh_rest, bool activations, bool antialiasing, bool contrib) {
    return views_forward_impl(H, W, {}, scale_modifier, sh_degree, debug, tanfov, bg, view, proj, campos, means3D, sh, opac, scales, rots,
                              sh_rest, activations, antialiasing, contrib);
}

// views of different sizes: image_hw = [V,2] (height, width); color [sum 3 H_v W_v], depth / alpha [sum H_v W_v] (flat)
std::tuple<Tensor, Tensor, Tensor, Tensor, std::shared_ptr<ViewsState>>
views_mixed_forward(const std::vector<int32_t> &image_hw, double scale_modifier, int64_t sh_degree, bool debug, const Tensor &tanfov,
                    const Tensor &bg, const Tensor &view, const Tensor &proj, const Tensor &campos, const Tensor &means3D, const Tensor &sh,
                    const Tensor &opac, const Tensor &scales, const Tensor &rots, const OptTensor &sh_rest, bool activations,
                    bool antialiasing, bool contrib) {
    TORCH_CHECK_VALUE(!image_hw.empty() && image_hw.size() % 2 == 0, "image_hw must have dimensions (num_views, 2)");
    int64_t H = 0, W = 0;                                    // the capacity ceiling's bytes per instance do not depend on the size
    for (size_t i = 0; i < image_hw.size(); i += 2) { H = std::max<int64_t>(H, image_hw[i]); W = std::max<int64_t>(W, image_hw[i + 1]); }
    return views_forward_impl(H, W, image_hw, scale_modifier, sh_degree, debug, tanfov, bg, view, proj, campos, means3D, sh, opac, scales,
                              rots, sh_rest, activations, antialiasing, contrib);
}

// grads: (means3D, means2D [V,P,3], shs | features_dc, opacities, scales, rotations, features_rest); the per-Gaussian ones summed over views.
// Mixed sizes only: the densification statistics of the views in stats_views.  camera: + each view's (dL/dviewmatrix [V,16],
// dL/dprojmatrix [V,16], dL/dcampos [V,3]).
std::vector<Tensor> views_backward_impl(const std::shared_ptr<ViewsState> &st, const OptTensor &gC, const OptTensor &gD, const OptTensor &gA,
                                        bool accumulate, const std::vector<OptTensor> &out, const OptTensor &xyz_gradient_accum,
                                        const OptTensor &denom, const OptTensor &max_radii2D, uint64_t stats_views, bool camera,
                                        const OptTensor &absgrad) {
    const c10::cuda::CUDAGuard guard(st->means3D.device());
    const int64_t P = st->g.P, M = st->g.M, V = st->s.V;
    const auto f32 = st->means3D.options();
    OptTensor c = gC.has_value() && gC->defined() ? OptTensor(dev_f32(*gC, "grad_color")) : c10::nullopt;
    OptTensor d = gD.has_value() && gD->defined() ? OptTensor(dev_f32(*gD, "grad_depth")) : c10::nullopt;
    OptTensor a = gA.has_value() && gA->defined() ? OptTensor(dev_f32(*gA, "grad_alpha")) : c10::nullopt;
    std::vector<Tensor> g(7);
    auto pick = [&](size_t i, bool wanted, c10::IntArrayRef shape) {
        if (i < out.size() && out[i].has_value() && out[i]->defined()) g[i] = *out[i];
        else if (wanted) g[i] = torch::empty(shape, f32);
    };
    const bool act = st->g.activations != 0;
    pick(0, true, {P, 3}); pick(1, true, {V, P, 3}); pick(2, true, {P, act ? 1 : M, 3}); pick(3, true, {P, 1});
    pick(4, true, {P, 3}); pick(5, true, {P, 4}); pick(6, act && st->sh_rest.has_value(), {P, M - 1, 3});
    auto gp = [&](size_t i) -> float * { return g[i].defined() && g[i].numel() > 0 ? g[i].data_ptr<float>() : nullptr; };
    DgrImageGrads gin{fptr(c), fptr(d), fptr(a)};
    DgrGaussianGrads gout{gp(0), gp(1), gp(2), nullptr, gp(3), gp(4), gp(5), nullptr, accumulate ? 1 : 0, gp(6),
                          fptr_mut(xyz_gradient_accum), fptr_mut(denom), fptr_mut(max_radii2D), nullptr};
    CameraOut cam;
    camera_out(camera, V, P, st->opt, f32, g, cam, absgrad);
    void *stream = c10::cuda::getCurrentCUDAStream(st->device).stream();
    if (at::globalContext().deterministicAlgorithms()) {
        Tensor det = det_scratch(st->n_inst, P * V, f32);
        const uint64_t n = (uint64_t)st->n_inst, bytes = (uint64_t)det.numel();
        if (!st->hw.empty())
            check(dgr_views_mixed_backward_det_ex(&st->s, st->hw.data(), &st->g, st->geom.data_ptr(), st->binning.data_ptr(),
                                                  (uint64_t)st->capacity, st->staging, st->image.data_ptr(), st->radii.data_ptr<int32_t>(), &gin,
                                                  &gout, stats_views, det.data_ptr(), bytes, n, &cam.opt, stream));
        else
            check(dgr_views_backward_det_ex(&st->s, &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)st->capacity, st->staging,
                                            st->image.data_ptr(), st->radii.data_ptr<int32_t>(), &gin, &gout, det.data_ptr(), bytes, n, &cam.opt,
                                            stream));
        return g;
    }
    if (!st->hw.empty())
        check(dgr_views_mixed_backward_ex(&st->s, st->hw.data(), &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)st->capacity,
                                          st->staging, st->image.data_ptr(), st->radii.data_ptr<int32_t>(), &gin, &gout, stats_views, &cam.opt,
                                          stream));
    else
        check(dgr_views_backward_ex(&st->s, &st->g, st->geom.data_ptr(), st->binning.data_ptr(), (uint64_t)st->capacity, st->staging,
                                    st->image.data_ptr(), st->radii.data_ptr<int32_t>(), &gin, &gout, &cam.opt, stream));
    return g;
}

std::vector<Tensor> views_backward(const std::shared_ptr<ViewsState> &st, const OptTensor &gC, const OptTensor &gD, const OptTensor &gA,
                                   bool accumulate, const std::vector<OptTensor> &out, bool camera) {
    return views_backward_impl(st, gC, gD, gA, accumulate, out, c10::nullopt, c10::nullopt, c10::nullopt, 0, camera, c10::nullopt);
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    pybind11::class_<State, std::shared_ptr<State>>(m, "State")
        .def_readonly("capacity", &State::capacity)
        .def_readonly("num_rendered", &State::n_inst)
        .def_property_readonly("weight_sum", [](const State &s) { return s.weight_sum; })
        .def_property_readonly("weight_max", [](const State &s) { return s.weight_max; });
    namespace py = pybind11;
    m.def("forward", &forward, "both forward stages through the C ABI (no arithmetic here)", py::arg("H"), py::arg("W"), py::arg("tanfovx"),
          py::arg("tanfovy"), py::arg("scale_modifier"), py::arg("sh_degree"), py::arg("prefiltered"), py::arg("debug"), py::arg("bg"),
          py::arg("view"), py::arg("proj"), py::arg("campos"), py::arg("means3D"), py::arg("sh"), py::arg("colors"), py::arg("opac"),
          py::arg("scales"), py::arg("rots"), py::arg("cov3D"), py::arg("sh_rest"), py::arg("activations"), py::arg("antialiasing") = false,
          py::arg("contrib") = false);
    m.def("backward", &backward, "backward through the C ABI", pybind11::arg("state"), pybind11::arg("grad_color"), pybind11::arg("grad_depth"),
          pybind11::arg("grad_alpha"), pybind11::arg("accumulate"), pybind11::arg("out"), pybind11::arg("xyz_gradient_accum"),
          pybind11::arg("denom"), pybind11::arg("max_radii2D"), pybind11::arg("push_addr") = 0, pybind11::arg("camera") = false,
          pybind11::arg("absgrad") = pybind11::none());
    pybind11::class_<ViewsState, std::shared_ptr<ViewsState>>(m, "ViewsState")
        .def_readonly("capacity", &ViewsState::capacity)
        .def_readonly("num_rendered", &ViewsState::n_inst)
        .def_property_readonly("weight_sum", [](const ViewsState &s) { return s.weight_sum; })
        .def_property_readonly("weight_max", [](const ViewsState &s) { return s.weight_max; });
    m.def("views_forward", &views_forward, "both forward stages of the batched-camera call through the C ABI", py::arg("H"), py::arg("W"),
          py::arg("scale_modifier"), py::arg("sh_degree"), py::arg("debug"), py::arg("tanfov"), py::arg("bg"), py::arg("view"), py::arg("proj"), py::arg("campos"), py::arg("means3D"),
          py::arg("sh"), py::arg("opac"), py::arg("scales"), py::arg("rots"), py::arg("sh_rest"), py::arg("activations"), py::arg("antialiasing") = false,
          py::arg("contrib") = false);
    m.def("views_backward", &views_backward, "backward of the batched-camera call through the C ABI", pybind11::arg("state"),
          pybind11::arg("grad_color"), pybind11::arg("grad_depth"), pybind11::arg("grad_alpha"), pybind11::arg("accumulate"), pybind11::arg("out"),
          pybind11::arg("camera") = false);
    m.def("views_mixed_forward", &views_mixed_forward, "both forward stages of the batched call with a size per view through the C ABI",
          py::arg("image_hw"), py::arg("scale_modifier"), py::arg("sh_degree"), py::arg("debug"), py::arg("tanfov"), py::arg("bg"), py::arg("view"), py::arg("proj"), py::arg("campos"), py::arg("means3D"),
          py::arg("sh"), py::arg("opac"), py::arg("scales"), py::arg("rots"), py::arg("sh_rest"), py::arg("activations"), py::arg("antialiasing") = false,
          py::arg("contrib") = false);
    m.def("views_mixed_backward", &views_backward_impl, "backward of the batched call with a size per view through the C ABI",
          pybind11::arg("state"), pybind11::arg("grad_color"), pybind11::arg("grad_depth"), pybind11::arg("grad_alpha"), pybind11::arg("accumulate"),
          pybind11::arg("out"), pybind11::arg("xyz_gradient_accum"), pybind11::arg("denom"), pybind11::arg("max_radii2D"),
          pybind11::arg("stats_views"), pybind11::arg("camera") = false, pybind11::arg("absgrad") = pybind11::none());
    m.def("set_views_mixed_hint", [](int dev, int64_t P, const std::vector<int32_t> &hw, int64_t cap, bool big) {
        std::lock_guard<std::mutex> lk(g_mu); g_views_mixed_hints[views_mixed_hint_key(dev, P, hw)] = Hint{cap, big}; });
    m.def("get_views_mixed_hint", [](int dev, int64_t P, const std::vector<int32_t> &hw) -> pybind11::object {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_views_mixed_hints.find(views_mixed_hint_key(dev, P, hw));
        if (it == g_views_mixed_hints.end()) return pybind11::none();
        return pybind11::make_tuple(it->second.cap, it->second.big); });
    m.def("set_views_hint", [](int dev, int64_t P, int H, int W, int V, int64_t cap, bool big) {
        std::lock_guard<std::mutex> lk(g_mu); g_views_hints[views_hint_key(dev, P, H, W, V)] = Hint{cap, big}; });
    m.def("get_views_hint", [](int dev, int64_t P, int H, int W, int V) -> pybind11::object {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_views_hints.find(views_hint_key(dev, P, H, W, V));
        if (it == g_views_hints.end()) return pybind11::none();
        return pybind11::make_tuple(it->second.cap, it->second.big); });
    m.def("abi_version", []() { return dgr_abi_version(); });
    m.def("set_hint", [](int dev, int64_t P, int H, int W, int64_t cap, bool big) {
        std::lock_guard<std::mutex> lk(g_mu); g_hints[hint_key(dev, P, H, W)] = Hint{cap, big}; });
    m.def("get_hint", [](int dev, int64_t P, int H, int W) -> pybind11::object {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_hints.find(hint_key(dev, P, H, W));
        if (it == g_hints.end()) return pybind11::none();
        return pybind11::make_tuple(it->second.cap, it->second.big); });
}
