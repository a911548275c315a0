/*
 * dgr_b200.h — C ABI of the B200-native differentiable Gaussian-splat rasterizer (libdgr_b200.so).
 *
 * This is the drop-in boundary for the ONE native call DreamGaussian makes on its hot path:
 *   GaussianRasterizer(raster_settings)(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
 *   cov3D_precomp) -> (color, radii, depth, alpha)          /root/reference/gs_renderer.py:745-809
 * The reference binds that through the pybind module `diff_gaussian_rasterization._C` of an un-vendored package
 * (readme.md:30-32): `rasterize_gaussians`, `rasterize_gaussians_backward`, `mark_visible`  [EXT, SURVEY.md §8b].
 * The entry points below are what those three bindings would call; everything is plain pointers and sizes, no
 * torch types.  All pointers are DEVICE pointers unless named *_host.  All work is enqueued on `stream`
 * (a cudaStream_t passed as void*); nothing here synchronises the device unless stated.
 *
 * Return value: 0 on success, otherwise a cudaError_t / negative dgr error code; dgr_last_error() has the text.
 */
#ifndef DGR_B200_H
#define DGR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DGR_ABI_VERSION 5

/* == GaussianRasterizationSettings, the 12-field NamedTuple built at gs_renderer.py:745-758 == */
typedef struct DgrSettings {
    int32_t image_height;
    int32_t image_width;
    float   tanfovx;
    float   tanfovy;
    float   scale_modifier;
    int32_t sh_degree;       /* active degree, 0..3 */
    int32_t prefiltered;     /* accepted, unused (always False in the reference, gs_renderer.py:756) */
    int32_t debug;           /* !=0: synchronise and check after every kernel */
    const float *bg;         /* [3]   */
    const float *viewmatrix; /* [4,4] row-major, p_view = [p,1] @ V   (gs_renderer.py:656-662) */
    const float *projmatrix; /* [4,4] row-major, full projection      (gs_renderer.py:663-670) */
    const float *campos;     /* [3]   as given by the caller (= -c2w[:3,3], gs_renderer.py:671) */
} DgrSettings;

/* == the per-Gaussian inputs of GaussianRasterizer.forward (gs_renderer.py:800-809); float32, contiguous ==
 * Alignment: `rotations`, and `shs` / `shs_rest` when their rows are a multiple of 16 bytes (M % 4 == 0, (M - 1) % 4 == 0), are read
 * with 128-bit loads and must be 16-byte aligned — what every device allocation is; the two host layers of this repository
 * re-allocate a view that is not (rasterizer.py::_dev_f32, dgr_torch.cpp::dev_f32).  When ALL of means3D / scales / rotations /
 * opacities / shs (/ shs_rest) are 16-byte aligned the per-Gaussian kernels stage them with bulk TMA (see dgr_set_tuning). */
typedef struct DgrGaussians {
    int32_t P;                   /* number of Gaussians */
    int32_t M;                   /* SH coefficients per channel in `shs` (= shs.shape[1]); 0 if shs == NULL */
    const float *means3D;        /* [P,3]   */
    const float *shs;            /* [P,M,3] or NULL (then colors_precomp) */
    const float *colors_precomp; /* [P,3]   or NULL */
    const float *opacities;      /* [P,1]   */
    const float *scales;         /* [P,3]   or NULL (then cov3D_precomp) */
    const float *rotations;      /* [P,4]   (w,x,y,z), consumed un-normalised */
    const float *cov3D_precomp;  /* [P,6]   xx,xy,xz,yy,yz,zz or NULL */
    /* SURVEY.md §8 row f1 — GaussianModel's RAW parameters with the activations fused into the kernels
     * (gs_renderer.py:196-216): when activations != 0, `opacities` is _opacity (sigmoid applied here), `scales` is _scaling
     * (exp), `rotations` is _rotation (F.normalize, eps 1e-12), `shs` is _features_dc [P,1,3] and `shs_rest` is
     * _features_rest [P,M-1,3] (NULL when M == 1) — no torch.cat copy; M stays the TOTAL coefficient count.  Requires
     * shs != NULL and cov3D_precomp == NULL.  The gradients come back with respect to the raw tensors. */
    const float *shs_rest;
    int32_t activations;
} DgrGaussians;

/* == outputs of the forward (gs_renderer.py:800) == */
typedef struct DgrImages {
    float   *color;  /* [3,H,W] */
    float   *depth;  /* [1,H,W] sum depth*alpha*T (not normalised) */
    float   *alpha;  /* [1,H,W] sum alpha*T */
    int32_t *radii;  /* [P]     0 = not rendered */
} DgrImages;

/* == upstream gradients into the backward; any pointer may be NULL (= zeros) == */
typedef struct DgrImageGrads {
    const float *dL_dcolor; /* [3,H,W] */
    const float *dL_ddepth; /* [1,H,W] */
    const float *dL_dalpha; /* [1,H,W] */
} DgrImageGrads;

/* Multi-GPU, view-sharded (SURVEY.md §8e): lets the per-Gaussian backward deliver gradient rows straight to the rank that OWNS
 * them.  Gaussian g belongs to rank g / gaussians_per_owner (a positive multiple of 256 with gaussians_per_owner * world >= P).
 * All the gradient pointers of the call must then lie in ONE local flat buffer, and delta_floats[o] is the distance, in
 * floats, from any address in that buffer to the same element of THIS rank's slot in rank o's staging area (peer-mapped
 * symmetric memory); delta_floats[rank] = 0.  With it the backward writes, for every Gaussian of another owner,
 * (accumulate ? what the local buffer holds : 0) + this view's gradient to the owner instead of to the local buffer — the
 * reduce-scatter half of the all-reduce rides on the kernel; dgr_peer_reduce_staged() finishes the sum. */
typedef struct DgrPeerPush {
    int32_t world, rank;
    int64_t gaussians_per_owner;
    int64_t delta_floats[16];
} DgrPeerPush;

/* == gradients w.r.t. the inputs; any pointer may be NULL (= not wanted) == */
typedef struct DgrGaussianGrads {
    float *dL_dmeans3D;        /* [P,3]   */
    float *dL_dmeans2D;        /* [P,3]   NDC units, z = 0 (gs_renderer.py:626 reads [:, :2]) */
    float *dL_dshs;            /* [P,M,3] */
    float *dL_dcolors_precomp; /* [P,3]   */
    float *dL_dopacities;      /* [P,1]   */
    float *dL_dscales;         /* [P,3]   */
    float *dL_drotations;      /* [P,4]   */
    float *dL_dcov3D_precomp;  /* [P,6]   */
    int32_t accumulate;        /* 0: overwrite; 1: add into the buffers (several views -> one flat gradient) */
    float *dL_dshs_rest;       /* [P,M-1,3] with DgrGaussians.activations (then dL_dshs is [P,1,3]); else unused */
    /* Densification bookkeeping fused into the per-Gaussian backward (gs_renderer.py:625-627, main.py:279-281); each may
     * be NULL.  For every Gaussian with radii > 0 in this render: xyz_gradient_accum += |dL/dmeans2D[:, :2]| (this
     * render's gradient), denom += 1, max_radii2D = max(max_radii2D, radii).  All float32 [P] (the reference's [P,1]). */
    float *xyz_gradient_accum;
    float *denom;
    float *max_radii2D;
    const DgrPeerPush *push;   /* NULL: everything goes to the local buffers */
} DgrGaussianGrads;

/* Scratch sizes.  The caller owns the three scratch buffers (upstream: geomBuffer / binningBuffer / imgBuffer),
 * must keep them alive and untouched between a forward and its backward, and aligns them to 256 bytes. */
size_t dgr_geom_bytes(int32_t P, int32_t image_height, int32_t image_width);
size_t dgr_image_bytes(int32_t image_height, int32_t image_width);
size_t dgr_binning_bytes(uint64_t capacity_instances, int32_t image_height, int32_t image_width);

/* Forward, stage 1: per-Gaussian preprocess (cull, EWA cov2D, conic, radius, SH->RGB, opacity-aware pixel AABB)
 * fused with the per-tile instance histogram (kept in `image` scratch).  Writes radii. */
int dgr_forward_preprocess(const DgrSettings *s, const DgrGaussians *g, void *geom, void *image, int32_t *radii,
                           void *stream);

/* Forward, stage 2: tile ranges (device-side scans), instance emission, per-tile depth sort + record gather, and the
 * per-tile front-to-back compositing.  Nothing here waits for the host.  Two things are guessed by the caller:
 *   - `capacity_instances`, the instance capacity `binning` was sized for;
 *   - DGR_FLAG_BIG_TILES in `flags`: whether to also launch the sorter for tiles with more than 4096 instances.
 * The truth is written to geom scratch and, if counts_host != NULL (pinned host memory, 4 x uint64), made available to
 * the host right after the scan: counts_host[0] = instance count, counts_host[1] = number of big tiles.  Two protocols:
 *   ticket == 0: an asynchronous copy, then count_ready_event (from dgr_event_create, may be NULL) is recorded — the caller
 *                keeps enqueuing work and checks the guesses once that event has fired;
 *   ticket != 0: the scan kernel stores the two counts and then counts_host[2] = ticket straight into the caller's memory
 *                (which must therefore be device-mapped pinned memory — under unified addressing every cudaHostAlloc /
 *                torch pin_memory buffer is); the caller polls counts_host[2] for the ticket value it chose for THIS call.
 *                No copy or event sits between the kernels then, so the whole forward chains with programmatic dependent
 *                launches (each kernel's prologue overlaps its predecessor's tail); count_ready_event is ignored.  If counts_host[0] > capacity_instances, or counts_host[1] > 0 without
 * DGR_FLAG_BIG_TILES, the call produced a memory-safe but wrong image: re-run stage 2 with corrected guesses and
 * DGR_FLAG_RERUN set.
 * counts_host[3] is written by the host before the call returns (either protocol): the record staging this call chose for
 * its render kernels (DGR_STAGING_SORTED or DGR_STAGING_BY_ID, see dgr_set_tuning bits 22-23).  The sorted record copy only
 * exists in `binning` when it says DGR_STAGING_SORTED; the backward of this call must be given that value. */
#define DGR_FLAG_BIG_TILES 1
#define DGR_FLAG_RERUN 2      /* set when stage 2 is repeated for the same stage 1 (corrected guesses) */
#define DGR_STAGING_SORTED 0  /* the sort kernel wrote a depth-sorted copy of the records; the render kernels stream it */
#define DGR_STAGING_BY_ID 1   /* only the sorted Gaussian ids exist; the render kernels fetch every record by id */
int dgr_forward_render(const DgrSettings *s, const DgrGaussians *g, void *geom, void *binning,
                       uint64_t capacity_instances, void *image, const DgrImages *out, int32_t flags,
                       uint64_t *counts_host, uint64_t ticket, void *count_ready_event, void *stream);

/* Tuning knobs (process-wide atomics; results do not depend on them beyond the summation order of the gradient atomics):
 * pixels per lane of the forward / backward render kernels (1, 2 or 4; the backward has 1 and 2) and a bit field:
 *   bit 3        programmatic dependent launches OFF (the environment variable DGR_PDL=0 does the same)
 *   bits 4-6     hits the forward evaluates together (1, 2, 4; 0 = default)      bits 8-10   the same for the backward
 *   bits 12-15   persistent CTAs per SM of the forward render kernel (0 = as many as fit)     bits 16-19   backward
 *   bit 20       render work queue consumed from both ends (experiment, measured slower)
 *   bit 21       backward work in tile-population order instead of the cost the forward measured
 *   bits 22-23   record staging of the render kernels: 0 = automatic (by Gaussian id when the sorted copy would exceed twice
 *                the L2 size), 1 = always the sorted copy, 2 = always by id
 *   bit 24 / 25  the per-Gaussian forward / backward kernel reads its inputs with per-thread global loads instead of staging
 *                each warp's 32 contiguous Gaussians through shared memory with bulk TMA (A/B switch; the staged path needs
 *                SH + scale / rotation inputs and 16-byte aligned base pointers and is otherwise not taken anyway)
 *   bit 26       step 2 of the backward render kernel in its per-pixel form (A/B switch; default sub-tile shape only)
 * the other bits are accepted and ignored.  The knobs may change between a forward and its backward: each call reads them when
 * it launches, and the backward stages its records the way its forward did (counts_host[3] -> dgr_backward's `staging`). */
int dgr_set_tuning(int ppl_fwd, int ppl_bwd, int tile_order);

/* Thin cudaEvent wrappers so a host without the CUDA runtime headers (ctypes, cgo ...) can use the protocol above. */
void *dgr_event_create(void);
int dgr_event_synchronize(void *event);
void dgr_event_destroy(void *event);

/* Backward of both stages.  geom / binning / image are the scratch buffers of the matching forward
 * (`capacity_instances` = the value stage 2 ran with, `staging` = the counts_host[3] that call left: DGR_STAGING_SORTED or
 * DGR_STAGING_BY_ID; when stage 2 was re-run, those of the last run); geom is also used as scratch for the per-Gaussian
 * reduction.  `out_alpha` is the alpha image the forward produced (accepted for signature parity with the
 * reference binding; the final transmittance is kept in `image` at full precision instead of 1 - alpha). */
int dgr_backward(const DgrSettings *s, const DgrGaussians *g, void *geom, const void *binning,
                 uint64_t capacity_instances, int32_t staging, const void *image, const int32_t *radii, const float *out_alpha,
                 const DgrImageGrads *gin, const DgrGaussianGrads *gout, void *stream);

/* == Batched cameras: ONE cloud rendered from V cameras of the same image size in one forward / backward ==
 * Every view has its own camera and background; image size, SH degree and scale modifier are shared.  All arrays are DEVICE
 * arrays.  Outputs: DgrImages.color [V,3,H,W], depth / alpha [V,1,H,W], radii [V,P] int32; view v is what dgr_forward_* returns
 * for camera v (up to the rounding of fused multiply-adds, which ptxas chooses per kernel).  The backward SUMS the gradients of
 * means3D / shs / opacities / scales / rotations over the views (written, or added with DgrGaussianGrads.accumulate) and writes
 * dL_dmeans2D per view, [V,P,3].
 * Supported inputs: SH + scale / rotation, plain or raw (DgrGaussians.activations).  Refused before any device work:
 * colors_precomp / cov3D_precomp, the densification statistics (xyz_gradient_accum / denom / max_radii2D) and DgrPeerPush.
 * Limits, checked before any device work: 1 <= V <= DGR_VIEWS_MAX; V x tiles per view <= 51200 (the shared-memory tile
 * histogram of the single-view call, now spanning the batch); V x P <= DGR_VIEWS_MAX_RECORDS (record r = v P + g is the 32-bit
 * id the sort keys carry); every image-size limit of the single-view call.
 * Scratch: geom holds V x P records and moments (dgr_views_geom_bytes), image V x tiles per-tile arrays and [V,H,W] pixel state.
 * Kernel shapes: the batched render kernels are the default sub-tile shapes only (forward 8x4 pixels per warp, one hit at a time;
 * backward 8x4 with two hits together and the per-row step 2): dgr_set_tuning's pixels-per-lane, hits-together and bit 26 do not
 * apply to them.  The scheduling knobs (cost order, two-ended queue, CTAs per SM, PDL), record staging (bits 22-23), input
 * staging of the forward (bit 24) do. */
#define DGR_VIEWS_MAX 64
#define DGR_VIEWS_MAX_RECORDS 2147483647ll
typedef struct DgrViews {
    int32_t V;
    int32_t image_height;
    int32_t image_width;
    float   scale_modifier;
    int32_t sh_degree;       /* active degree, 0..3 */
    int32_t debug;           /* !=0: synchronise and check after every kernel */
    const float *tanfov;     /* [V,2]   tanfovx, tanfovy */
    const float *bg;         /* [V,3]   */
    const float *viewmatrix; /* [V,4,4] row-major, as DgrSettings.viewmatrix */
    const float *projmatrix; /* [V,4,4] */
    const float *campos;     /* [V,3]   */
} DgrViews;

size_t dgr_views_geom_bytes(int32_t V, int32_t P, int32_t image_height, int32_t image_width);
size_t dgr_views_image_bytes(int32_t V, int32_t image_height, int32_t image_width);
size_t dgr_views_binning_bytes(uint64_t capacity_instances, int32_t V, int32_t image_height, int32_t image_width);
/* As dgr_forward_preprocess / dgr_forward_render / dgr_backward, for the batch (same capacity, DGR_FLAG_BIG_TILES, ticket and
 * counts_host[0..3] protocol; `staging` = the counts_host[3] the batched forward left).  radii: [V,P]. */
int dgr_views_forward_preprocess(const DgrViews *s, const DgrGaussians *g, void *geom, void *image, int32_t *radii, void *stream);
int dgr_views_forward_render(const DgrViews *s, const DgrGaussians *g, void *geom, void *binning, uint64_t capacity_instances,
                             void *image, const DgrImages *out, int32_t flags, uint64_t *counts_host, uint64_t ticket,
                             void *count_ready_event, void *stream);
int dgr_views_backward(const DgrViews *s, const DgrGaussians *g, void *geom, const void *binning, uint64_t capacity_instances,
                       int32_t staging, const void *image, const int32_t *radii, const DgrImageGrads *gin,
                       const DgrGaussianGrads *gout, void *stream);

/* == Batched cameras of DIFFERENT image sizes: the batched call above with a size per view ==
 * image_hw: HOST array [V,2] of (height, width); DgrViews.image_height / image_width are ignored.  Everything else of DgrViews
 * and of the same-size call holds (cameras, shared SH degree and scale modifier, inputs, protocol, kernels).  Outputs are FLAT:
 * with pix_off[v] = sum over u < v of H_u W_u, view v's colour is the contiguous [3,H_v,W_v] block at float 3 pix_off[v] of
 * DgrImages.color, and its depth / alpha the [H_v,W_v] blocks at float pix_off[v] of depth / alpha (the image gradients of the
 * backward use the same layout); radii [V,P] and dL_dmeans2D [V,P,3] as above.  A batch whose sizes are all equal computes what
 * the same-size call computes, bit for bit, with the same scratch sizes.
 * Densification statistics: the backward updates DgrGaussianGrads.xyz_gradient_accum / denom / max_radii2D (float [P], any may
 * be NULL) for the views whose bit is set in stats_views (bit v = view v), in ascending view order, each with the single-view
 * rule (dgr_backward) for that view's means2D gradient and radii: what one single-view backward per selected view would leave.
 * Refused before any device work: image_hw NULL, a size <= 0 or > 65535, more than 51200 tiles (16x16) in the batch, V outside
 * 1..DGR_VIEWS_MAX, V x P > DGR_VIEWS_MAX_RECORDS, a stats_views bit at or above V, stats_views != 0 with no statistic buffer or
 * a statistic buffer with stats_views == 0, colors_precomp / cov3D_precomp, and DgrPeerPush.
 * Scratch: dgr_views_mixed_geom_bytes / dgr_views_mixed_image_bytes (0 for sizes the calls refuse); binning as
 * dgr_views_binning_bytes. */
size_t dgr_views_mixed_geom_bytes(int32_t V, int32_t P, const int32_t *image_hw);
size_t dgr_views_mixed_image_bytes(int32_t V, const int32_t *image_hw);
int dgr_views_mixed_forward_preprocess(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom, void *image,
                                       int32_t *radii, void *stream);
int dgr_views_mixed_forward_render(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom, void *binning,
                                   uint64_t capacity_instances, void *image, const DgrImages *out, int32_t flags, uint64_t *counts_host,
                                   uint64_t ticket, void *count_ready_event, void *stream);
int dgr_views_mixed_backward(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom, const void *binning,
                             uint64_t capacity_instances, int32_t staging, const void *image, const int32_t *radii,
                             const DgrImageGrads *gin, const DgrGaussianGrads *gout, uint64_t stats_views, void *stream);

/* == Deterministic backward: bit-reproducible gradients ==
 * dgr_backward_det / dgr_views_backward_det / dgr_views_mixed_backward_det take the arguments of their counterparts plus
 *   det_scratch        device scratch of at least dgr_det_scratch_bytes(instances, records) bytes (records = P, or V x P for the
 *                      batched calls); its contents need not be initialised;
 *   instances          the tile-instance count of the forward's LAST stage-2 run (counts_host[0]), at most capacity_instances.
 * They compute what the counterpart computes, up to the order of the float additions that gather a Gaussian's gradient from the
 * tiles it touches: here every such sum has a fixed order (within a tile: the 8x4-pixel sub-tiles in a fixed order; over the tiles:
 * row-major within the Gaussian's tile rectangle) and no float atomic is used.  Guarantee: for the same inputs, forward scratch and
 * upstream gradients on the same GPU model and library build, every output — the gradients, the per-view means2D gradients and
 * the densification statistics — is bit-identical from call to call, whatever dgr_set_tuning's knobs (work order, CTAs per SM, PDL,
 * pixels per lane, hits together), the record staging and the caller's thread or stream.  Not covered: a different library build or
 * GPU model (ptxas chooses the fused multiply-adds), DgrGaussianGrads.accumulate onto non-deterministic values, and any
 * cross-rank reduction of the multi-GPU path.
 * Refused before any device work, each with its own dgr_last_error text: det_scratch NULL or smaller than dgr_det_scratch_bytes,
 * instances > capacity_instances, DgrPeerPush, and everything the counterpart refuses.  With debug set (DgrSettings / DgrViews),
 * `instances` is also compared with the forward's own count (one host synchronisation) and a mismatch is refused; without it, a
 * count below the forward's leaves a NaN gradient row for every Gaussian whose tiles it does not cover.
 * Cost: the counterpart's backward render kernel is replaced by render_bwd_det (one CTA per tile, a barrier per 32-record chunk)
 * followed by det_moments_gather, and a scratch memset, a count kernel and three scan kernels run first; a whole forward+backward
 * step measured 1.2-1.6x the default one (DESIGN.md §4 has the per-kernel times). */
size_t dgr_det_scratch_bytes(uint64_t instances, int64_t records);
int dgr_backward_det(const DgrSettings *s, const DgrGaussians *g, void *geom, const void *binning,
                     uint64_t capacity_instances, int32_t staging, const void *image, const int32_t *radii, const float *out_alpha,
                     const DgrImageGrads *gin, const DgrGaussianGrads *gout, void *det_scratch, uint64_t det_scratch_bytes,
                     uint64_t instances, void *stream);
int dgr_views_backward_det(const DgrViews *s, const DgrGaussians *g, void *geom, const void *binning, uint64_t capacity_instances,
                           int32_t staging, const void *image, const int32_t *radii, const DgrImageGrads *gin,
                           const DgrGaussianGrads *gout, void *det_scratch, uint64_t det_scratch_bytes, uint64_t instances,
                           void *stream);
int dgr_views_mixed_backward_det(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom, const void *binning,
                                 uint64_t capacity_instances, int32_t staging, const void *image, const int32_t *radii,
                                 const DgrImageGrads *gin, const DgrGaussianGrads *gout, uint64_t stats_views, void *det_scratch,
                                 uint64_t det_scratch_bytes, uint64_t instances, void *stream);

/* == Rasterization options: anti-aliased rendering (the 2D Mip filter with opacity compensation) ==
 * The *_ex calls take the arguments of their counterparts plus `opt` (NULL = flags 0); with flags 0 they compute exactly what the
 * counterpart computes.  DGR_RASTER_ANTIALIAS: per Gaussian and view, with (a0, b, c0) the 2D covariance in pixels before the
 * low-pass and (a, b, c) = (a0 + 0.3, b, c0 + 0.3) after it, the opacity o (raw parameters: sigmoid first) is replaced by
 *   o_eff = o sqrt(max(DGR_AA_RATIO_FLOOR, (a0 c0 - b^2) / (a c - b^2)))          (Mip-Splatting, Yu et al., CVPR 2024)
 * so a Gaussian smaller than a pixel keeps its integrated weight instead of being dilated and brightened at a low resolution:
 * its image changes little across resolutions and scale_modifier.  Radii, the tile rectangle and the conic are those of the
 * default mode; alpha = min(0.99, o_eff G) with the other compositing rules unchanged; the opacity-aware pixel box follows o_eff,
 * so there are at most as many tile instances as in the default mode.  Gradients are the exact chain rule, with the factor
 * differentiated through the determinant ratio into the 2D covariance (no gradient where the floor is active).
 * Limit: a0 c0 - b^2 is formed in float32 from the covariance entries (as upstream diff-gaussian-rasterization forms it); its
 * relative error is about 3e-8 r^2 for a footprint of aspect ratio r, so needles beyond ~100:1 get a compensation with a float32
 * error of 1e-4 or more, and for a needle far thinner than a pixel and hundreds of pixels long it is rounding noise.
 * The forward's flags are recorded in its `image` scratch; its backward must be given the same flags.  With debug set
 * (DgrSettings / DgrViews) the backward compares them (one host synchronisation) and refuses a mismatch; without debug a mismatch
 * is not detected and gives wrong gradients.  Refused before any device work: unknown flag bits, and everything the counterpart
 * refuses.  Each call accepts everything its counterpart accepts (DgrPeerPush included where the counterpart takes it); the
 * stage-2 render calls need no variant.
 * Cost: only the per-Gaussian forward and backward kernels differ (their *_aa_kernel variants: a few dozen FLOPs and a square
 * root per Gaussian and view); the binning, sort and render kernels are those of the default mode (DESIGN.md §4 has the times). */
#define DGR_RASTER_ANTIALIAS 1u
/* == Camera gradients (DGR_RASTER_CAMERA_GRADS, backward *_ex calls only) ==
 * The backward also returns dL/dviewmatrix [16] (the layout of DgrSettings.viewmatrix: row-major, p_view = [p,1] V),
 * dL/dprojmatrix [16] and dL/dcampos [3] of the render; for dgr_views_* and dgr_views_mixed_* [V,16], [V,16] and [V,3], each view's
 * own.  They are the exact chain rule of the forward as the per-Gaussian backward differentiates it: the cull decisions, radius,
 * tile rectangle, opacity-aware box, the 0.3 low-pass, the eigenvalue floor and the clamped tx'/ty' inside J are constants, and
 * min(0.99, .) is straight-through.  Column 3 of dL/dviewmatrix and column 2 of dL/dprojmatrix are 0 (the forward never reads
 * them); dL/dcampos is 0 with colors_precomp and at sh_degree 0.  With DGR_RASTER_ANTIALIAS the opacity-compensation gradient
 * is included.  tanfovx / tanfovy and bg get no gradient.
 * Any of the three output pointers may be NULL; the others are always written, never accumulated, whatever
 * DgrGaussianGrads.accumulate says.  scratch: device memory of at least dgr_camera_grad_scratch_bytes(V, P) bytes (V = 1 for
 * the single-view calls).  No float atomics: each CTA of the extra kernel (camera_bwd) reduces its partials in a fixed order and
 * camera_reduce adds the CTAs' rows in order, so the gradients are bit-reproducible whenever the moments are (the *_det calls).
 * Refused before any device work: the bit with camera == NULL, scratch that is NULL or too small, and the bit on a forward *_ex
 * call.  The flags a forward records, and the debug comparison of a backward's flags with them, cover DGR_RASTER_ANTIALIAS only.
 * Without the bit a call launches exactly the kernels it launched before the bit existed; `camera` is read only with it, so a
 * caller's DgrRasterOptions that ends after `flags` stays valid.  Bit 2u stays unknown (refused), so a flags-only struct can
 * never be read past its end.  Cost: two kernels after the per-Gaussian backward (DESIGN.md §4). */
#define DGR_RASTER_CAMERA_GRADS 4u
typedef struct DgrCameraGrads {
    float *dL_dviewmatrix;   /* [16] or [V,16], or NULL */
    float *dL_dprojmatrix;   /* [16] or [V,16], or NULL */
    float *dL_dcampos;       /* [3] or [V,3], or NULL */
    void *scratch;           /* device, >= dgr_camera_grad_scratch_bytes(V, P) */
    uint64_t scratch_bytes;
} DgrCameraGrads;
size_t dgr_camera_grad_scratch_bytes(int32_t V, int32_t P);
/* == Absolute-gradient densification statistic (DGR_RASTER_ABS_GRAD, backward *_ex calls only; AbsGS, Ye et al., 2024) ==
 * xyz_gradient_accum adds |dL/dmeans2D[:2]| per render: the norm of a SUM over the pixels a Gaussian covers, which cancels where
 * those pixels pull its centre in opposite directions.  With the bit, the backward also adds, for every Gaussian with radius > 0
 * in the render (dgr_views_mixed_backward*: in each view whose bit is set in stats_views, in view order),
 *   xyz_gradient_accum_abs[g] += sqrt(a_x^2 + a_y^2),   a_x = sum_p |u_p (A dx + B dy)| W/2,   a_y = sum_p |u_p (B dx + C dy)| H/2
 * over the pixels p where the backward render evaluates g (its gradient's pixels and skip rules), u_p = o G_p dL/dalpha_p (o_eff
 * with DGR_RASTER_ANTIALIAS; min(0.99, .) straight-through), (dx, dy) = mean - pixel, (A, B, C) the conic: NDC units like
 * dL/dmeans2D, and >= the xyz_gradient_accum term of the same render (triangle inequality; equal for a one-pixel Gaussian).
 * xyz_gradient_accum_abs: device float32 [P], read only with the bit.  Gradients and the three other statistics are those of the
 * call without the bit, up to the order of float additions (the backward render runs its ABS variant of the default sub-tile
 * shape whatever dgr_set_tuning says); the *_det calls keep their bit-reproducibility for the new statistic too.  Accepted by
 * dgr_backward_ex, dgr_backward_det_ex, dgr_views_mixed_backward_ex and dgr_views_mixed_backward_det_ex, combined with
 * DGR_RASTER_ANTIALIAS and DGR_RASTER_CAMERA_GRADS as wanted.  Refused before any device work, each with its own dgr_last_error
 * text: the bit on a forward call, the bit with xyz_gradient_accum_abs == NULL, the bit on dgr_views_backward_ex /
 * dgr_views_backward_det_ex (the same-size batch has no statistics), and the bit on a mixed call with stats_views == 0.
 * Bits 2u and 8u stay unknown (refused), so a DgrRasterOptions that ends after `flags` or after `camera` is never read past its
 * end; a caller that sets this bit passes the whole struct.
 * Cost: the ABS render variant (about 4 more floating-point instructions per record and pixel in step 2) and one kernel of one
 * thread per Gaussian after the per-Gaussian backward (absgrad_stats); DESIGN.md §4 has the times.  Densify with
 * dgr_densify_plan_ex. */
#define DGR_RASTER_ABS_GRAD 16u
/* == Per-Gaussian blending-weight statistics (DGR_RASTER_CONTRIB, stage-2 render *_ex calls only) ==
 * For one render of view v and record r (r = g for the single-view call, r = v P + g for the batched calls), over exactly the
 * pixels p where the forward composites the record (power <= 0, alpha >= 1/255, before the T < 1e-4 stop), with the blending
 * weight w_p = alpha_p T_p, alpha_p = min(0.99, o G_p) (o = o_eff with DGR_RASTER_ANTIALIAS, the opacity the record carries):
 *   weight_sum[r] = sum_p w_p          weight_max[r] = max_p w_p
 * Both are 0 for a record with radius 0 and for one that is never composited (hidden behind others, or behind the T stop).
 * In exact arithmetic sum_r weight_sum[r] over a view's records equals the sum of that view's alpha image.
 * Outputs: device float32 [records]; DgrContrib.scratch: device memory of at least dgr_contrib_scratch_bytes(records) bytes.
 * Each call zeroes its outputs and scratch before its render and writes them completely, so a stage-2 re-run (DGR_FLAG_RERUN)
 * leaves the last run's values; nothing is accumulated here (a caller adds renders up after the run it keeps).
 * Deterministic by construction: each render warp reduces its (tile, sub-tile) item's weights of a record in a fixed order, the
 * item partials are added as 64-bit fixed point with scale 2^38 (integer atomics, so the order the items arrive in does not
 * matter) and the max is an atomicMax on the bits of a non-negative float.  Bound: an image has at most 51200 tiles of 256 pixels
 * and w <= 0.99, so a record's sum is below 2^24 and its fixed-point total below 2^62; a partial is rounded to the nearest 2^-38
 * (absolute), and the total to float32 once.  The outputs are bit-identical from call to call, whatever dgr_set_tuning's knobs
 * and the record staging, and a view of a batched call gives what the single-view call of that camera gives.
 * With the bit, the forward render runs its default sub-tile shape (<1,1>: 8x4 pixels per warp, one hit at a time) as the
 * render_*_fwd_contrib kernels, whatever the pixels-per-lane and hits-together knobs say, followed by contrib_finalize (one
 * thread per record); images, depth, alpha, radii and the forward state a backward reads are those of the call without the bit.
 * Accepted by dgr_forward_render_ex, dgr_views_forward_render_ex and dgr_views_mixed_forward_render_ex (flags NULL / 0: exactly
 * the counterpart's call).  Refused before any device work, each with its own dgr_last_error text: any other bit on those calls,
 * the bit on a preprocess or backward *_ex call, contrib == NULL, a NULL output or scratch, and a scratch below
 * dgr_contrib_scratch_bytes.  Bits 2u and 8u stay unknown (refused), and `contrib` is read only with the bit, so a
 * DgrRasterOptions that ends before it is never read past its end. */
#define DGR_RASTER_CONTRIB 32u
typedef struct DgrContrib {
    float *weight_sum;       /* [records] */
    float *weight_max;       /* [records] */
    void *scratch;           /* device, >= dgr_contrib_scratch_bytes(records) */
    uint64_t scratch_bytes;
} DgrContrib;
size_t dgr_contrib_scratch_bytes(int64_t records);
typedef struct DgrRasterOptions {
    uint32_t flags;          /* DGR_RASTER_* bits */
    const DgrCameraGrads *camera;   /* read only when flags has DGR_RASTER_CAMERA_GRADS */
    float *xyz_gradient_accum_abs;  /* [P], read only when flags has DGR_RASTER_ABS_GRAD */
    const DgrContrib *contrib;      /* read only when flags has DGR_RASTER_CONTRIB */
} DgrRasterOptions;
int dgr_forward_render_ex(const DgrSettings *s, const DgrGaussians *g, void *geom, void *binning,
                          uint64_t capacity_instances, void *image, const DgrImages *out, int32_t flags,
                          uint64_t *counts_host, uint64_t ticket, void *count_ready_event, const DgrRasterOptions *opt, void *stream);
int dgr_views_forward_render_ex(const DgrViews *s, const DgrGaussians *g, void *geom, void *binning, uint64_t capacity_instances,
                                void *image, const DgrImages *out, int32_t flags, uint64_t *counts_host, uint64_t ticket,
                                void *count_ready_event, const DgrRasterOptions *opt, void *stream);
int dgr_views_mixed_forward_render_ex(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom, void *binning,
                                      uint64_t capacity_instances, void *image, const DgrImages *out, int32_t flags,
                                      uint64_t *counts_host, uint64_t ticket, void *count_ready_event, const DgrRasterOptions *opt,
                                      void *stream);
int dgr_forward_preprocess_ex(const DgrSettings *s, const DgrGaussians *g, void *geom, void *image, int32_t *radii,
                              const DgrRasterOptions *opt, void *stream);
int dgr_views_forward_preprocess_ex(const DgrViews *s, const DgrGaussians *g, void *geom, void *image, int32_t *radii,
                                    const DgrRasterOptions *opt, void *stream);
int dgr_views_mixed_forward_preprocess_ex(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom, void *image,
                                          int32_t *radii, const DgrRasterOptions *opt, void *stream);
int dgr_backward_ex(const DgrSettings *s, const DgrGaussians *g, void *geom, const void *binning, uint64_t capacity_instances,
                    int32_t staging, const void *image, const int32_t *radii, const float *out_alpha, const DgrImageGrads *gin,
                    const DgrGaussianGrads *gout, const DgrRasterOptions *opt, void *stream);
int dgr_views_backward_ex(const DgrViews *s, const DgrGaussians *g, void *geom, const void *binning, uint64_t capacity_instances,
                          int32_t staging, const void *image, const int32_t *radii, const DgrImageGrads *gin,
                          const DgrGaussianGrads *gout, const DgrRasterOptions *opt, void *stream);
int dgr_views_mixed_backward_ex(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom, const void *binning,
                                uint64_t capacity_instances, int32_t staging, const void *image, const int32_t *radii,
                                const DgrImageGrads *gin, const DgrGaussianGrads *gout, uint64_t stats_views,
                                const DgrRasterOptions *opt, void *stream);
int dgr_backward_det_ex(const DgrSettings *s, const DgrGaussians *g, void *geom, const void *binning, uint64_t capacity_instances,
                        int32_t staging, const void *image, const int32_t *radii, const float *out_alpha, const DgrImageGrads *gin,
                        const DgrGaussianGrads *gout, void *det_scratch, uint64_t det_scratch_bytes, uint64_t instances,
                        const DgrRasterOptions *opt, void *stream);
int dgr_views_backward_det_ex(const DgrViews *s, const DgrGaussians *g, void *geom, const void *binning, uint64_t capacity_instances,
                              int32_t staging, const void *image, const int32_t *radii, const DgrImageGrads *gin,
                              const DgrGaussianGrads *gout, void *det_scratch, uint64_t det_scratch_bytes, uint64_t instances,
                              const DgrRasterOptions *opt, void *stream);
int dgr_views_mixed_backward_det_ex(const DgrViews *s, const int32_t *image_hw, const DgrGaussians *g, void *geom, const void *binning,
                                    uint64_t capacity_instances, int32_t staging, const void *image, const int32_t *radii,
                                    const DgrImageGrads *gin, const DgrGaussianGrads *gout, uint64_t stats_views, void *det_scratch,
                                    uint64_t det_scratch_bytes, uint64_t instances, const DgrRasterOptions *opt, void *stream);

/* Multi-GPU (view-sharded data parallelism, SURVEY.md §8e): all-reduce(sum) of the flat float32 gradient buffer over
 * NVLink with this library's own kernel.  The buffer lives in symmetric memory: peer_ptrs[w] (HOST array of `world` device
 * addresses) is rank w's copy mapped into this process; multicast_ptr, if non-zero, is the NVSwitch multicast address of
 * the same buffer (then multimem.ld_reduce / multimem.st are used and peer_ptrs may be NULL).  n_floats % 4 == 0.
 * peer_flag_ptrs (HOST array of `world` device addresses, or NULL): rank w's flag area of dgr_peer_flag_bytes() bytes in
 * the same symmetric allocation, zero-initialised once; with it the kernel carries its own two cross-rank barriers and
 * `epoch` must be 1, 2, 3, ... over successive calls (the same value on every rank).  With NULL the caller synchronises the
 * ranks (device-side barrier) before and after the call. */
size_t dgr_peer_flag_bytes(void);
int dgr_peer_allreduce(const uint64_t *peer_ptrs, int32_t world, int32_t rank, uint64_t n_floats, uint64_t multicast_ptr,
                       const uint64_t *peer_flag_ptrs, uint32_t epoch, void *stream);

/* The all-reduce split in two, its first half fused into the backward (DgrPeerPush): every rank has pushed the rows it does not own;
 * this call makes rank `push->rank` add the `world` staged copies of ITS rows (stage_ptr: local address of its staging area,
 * slot s at stage_ptr + s * padded_floats floats; its own contribution is read from its flat buffer peer_ptrs[rank]) in rank order
 * and publish the sums to every rank's flat buffer (multicast_ptr != 0: multimem.st; else stores to peer_ptrs[w]).  The flat buffer is
 * n_seg (<= 8) segments [P, seg_stride[k]] starting at float seg_off[k].  peer_flag_ptrs / epoch as for dgr_peer_allreduce (NULL: the
 * caller synchronises the ranks before and after).  dgr_peer_push_flat does the push for a rank that has no backward to ride on
 * (no view this iteration): it copies the rows of other owners from `local` (its flat buffer) to their owners. */
int dgr_peer_reduce_staged(const uint64_t *peer_ptrs, const DgrPeerPush *push, int64_t P, int32_t n_seg, const int64_t *seg_off,
                           const int32_t *seg_stride, uint64_t stage_ptr, uint64_t padded_floats, uint64_t multicast_ptr,
                           const uint64_t *peer_flag_ptrs, uint32_t epoch, void *stream);
int dgr_peer_push_flat(const float *local, const DgrPeerPush *push, int64_t P, int32_t n_seg, const int64_t *seg_off,
                       const int32_t *seg_stride, void *stream);

/* SURVEY.md §8 row f3 — replaces simple_knn._C.distCUDA2 (/root/reference/simple-knn/spatial.cu:15-26 -> SimpleKNN::knn,
 * simple_knn.cu:185-221; caller gs_renderer.py:341): mean_dists[i] = mean of the squared distances from point i to its 3
 * nearest OTHER points (exact; a point set smaller than 4 yields the reference's FLT_MAX arithmetic).  points [P,3] float32.
 * scratch: dgr_knn_scratch_bytes(P) bytes of device memory.  Stream-ordered, no host synchronisation, no library sort. */
size_t dgr_knn_scratch_bytes(int32_t P);
int dgr_dist_cuda2(int32_t P, const float *points, float *mean_dists, void *scratch, void *stream);

/* SURVEY.md §8 row f4 — GaussianModel.extract_fields (/root/reference/gs_renderer.py:218-294; gaussian_3d_coeff :64-83):
 * occ[resolution^3] (x-major, z fastest) = per-voxel sum of opacity * exp(-1/2 d^T Sigma^-1 d) over the Gaussians with
 * sigmoid(opacity) > 0.005 whose normalised centre lies strictly inside the voxel's block's bounding box grown by
 * relax_ratio * 2/num_blocks.  Inputs are the RAW model tensors (_xyz [P,3], _opacity [P,1], _scaling [P,3], _rotation
 * [P,4]); center_scale (device, 4 floats, may be NULL) receives the model's `center` and `scale` (:237-238).
 * resolution % num_blocks == 0, num_blocks <= 64, (resolution/num_blocks)^3 <= 4096.  Stream-ordered, no host read-back. */
size_t dgr_fields_scratch_bytes(int32_t P, int32_t num_blocks);
int dgr_extract_fields(int32_t P, const float *xyz, const float *opacity_raw, const float *scaling_raw, const float *rotation_raw,
                       int32_t resolution, int32_t num_blocks, float relax_ratio, float *occ, float *center_scale, void *scratch,
                       void *stream);

/* SURVEY.md §8 row f2 — the optimiser step of the stage-1 loop: torch.optim.Adam(lr per group, eps) over the model's six
 * parameter tensors (/root/reference/gs_renderer.py:361-370, stepped at main.py:274-276) as ONE launch.  bias correction 1 - beta^step per tensor; no weight decay, no amsgrad.  betas / eps are doubles because torch derives 1 - beta and
 * the bias corrections in double before rounding to float32.  Updates param / exp_avg / exp_avg_sq in place. */
typedef struct DgrAdamGroup {
    float *param;
    const float *grad;
    float *exp_avg;
    float *exp_avg_sq;
    uint64_t n;       /* elements */
    float lr;
    int32_t step;     /* this tensor's own step count after the update, from 1 (torch keeps state['step'] per tensor: a tensor
                       * whose .grad was None in some iteration lags behind) */
} DgrAdamGroup;
int dgr_adam_step(const DgrAdamGroup *groups, int32_t n_groups, double beta1, double beta2, double eps, void *stream);

/* SURVEY.md §8 row f2 — the reference's densify_and_prune (/root/reference/gs_renderer.py:586-609 = densify_and_clone
 * :582-600 + densify_and_split :555-580 + prune_points :509-513, with the optimizer-state surgery of :464-552) as stream
 * compaction.  Two calls with ONE host read-back between them (the new point count sizes the output tensors):
 *   dgr_densify_plan   classifies every point (grad = xyz_gradient_accum / denom, NaN -> 0; clone if |grad| >= grad_threshold
 *                      and max(exp(scaling)) <= dense_extent; split if grad >= grad_threshold and max > dense_extent; pruned
 *                      if sigmoid(opacity) < min_opacity or — when use_world != 0, the reference's `if max_screen_size:` —
 *                      max(exp(scaling)) > max_world; max_radii2D never matters: densification_postfix has zeroed it, :551)
 *                      and copies counts_host[4] = { kept originals, surviving clones, points selected for the split,
 *                      surviving children per copy } (pinned host memory) — new point count = [0] + [1] + 2 * [3].
 *   dgr_densify_apply  writes the new tensors in the reference's order (kept originals, clones, first children, second
 *                      children): the six parameter tensors and both Adam moments (zero for new points).  A child's position is
 *                      xyz + R(q/|q|) (noise[child * counts[2] + rank] * exp(scaling)), its scaling log(exp(scaling) / 1.6);
 *                      noise = standard normals [2 * counts[2], 3] (device), rank = the point's rank among the selected.
 * Tensor order in DgrDensifyTensors: xyz, f_dc, f_rest, opacity, scaling, rotation; width = floats per point (f_rest may be 0). */
typedef struct DgrDensifyTensors {
    const float *in[6], *exp_avg_in[6], *exp_avg_sq_in[6];
    float *out[6], *exp_avg_out[6], *exp_avg_sq_out[6];
    int32_t width[6];
} DgrDensifyTensors;
size_t dgr_densify_scratch_bytes(int32_t P);
int dgr_densify_plan(int32_t P, const float *xyz_gradient_accum, const float *denom, const float *opacity_raw, const float *scaling_raw,
                     float grad_threshold, float dense_extent, float min_opacity, float max_world, int32_t use_world,
                     void *scratch, uint32_t *counts_host, void *stream);
int dgr_densify_apply(int32_t P, const DgrDensifyTensors *t, const float *noise, const void *scratch, void *stream);
/* dgr_densify_plan with AbsGS's rule (DGR_RASTER_ABS_GRAD): clone as dgr_densify_plan (grad >= grad_threshold and small), split
 * when xyz_gradient_accum_abs / denom (NaN -> 0) >= abs_grad_threshold and max(exp(scaling)) > dense_extent; the prune rules, the
 * counts and dgr_densify_apply are unchanged.  xyz_gradient_accum_abs must not be NULL when P > 0. */
int dgr_densify_plan_ex(int32_t P, const float *xyz_gradient_accum, const float *xyz_gradient_accum_abs, const float *denom,
                        const float *opacity_raw, const float *scaling_raw, float grad_threshold, float abs_grad_threshold,
                        float dense_extent, float min_opacity, float max_world, int32_t use_world, void *scratch,
                        uint32_t *counts_host, void *stream);

/* GaussianRasterizer.markVisible: present[i] = 1 if Gaussian i passes the near-plane test. */
int dgr_mark_visible(int32_t P, const float *means3D, const float *viewmatrix, const float *projmatrix,
                     uint8_t *present, void *stream);

/* Introspection for tests: copies per-Gaussian forward state out of geom scratch (any pointer may be NULL):
 * mean_px [P,2], depth [P], conic [P,3] (natural units), rgb [P,3], opacity-aware pixel AABB [P,4] int32. */
int dgr_debug_geom(int32_t P, int32_t image_height, int32_t image_width, const void *geom, float *mean_px, float *depth, float *conic, float *rgb,
                   int32_t *aabb, uint32_t *tiles_touched, void *stream);

/* How many kernels of THIS library were launched by the calling thread since the last reset (for bench.py). */
uint64_t dgr_launch_count(void);
void dgr_reset_launch_count(void);

/* Per-kernel CUDA-event timing (tracing hook): when enabled, every kernel this thread launches is bracketed by
 * events on its stream; dgr_profile_collect waits for them and returns (name, ms) pairs, names '\n'-joined. */
void dgr_profile_enable(int on);
int dgr_profile_collect(char *names, size_t names_bytes, float *ms, int max);

int dgr_abi_version(void);
const char *dgr_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* DGR_B200_H */
