/*
 * b200gs.h -- C ABI of the H100-native (sm_90a) differentiable 3D-Gaussian-splatting rasteriser.
 *
 * This is the drop-in boundary for HumanGaussian's hot path.  The reference binds the rasteriser as
 * the Python package `diff_gaussian_rasterization` (an un-vendored torch C++/CUDA extension):
 *     gaussiansplatting/gaussian_renderer/__init__.py:14        import of GaussianRasterizationSettings, GaussianRasterizer
 *     gaussiansplatting/gaussian_renderer/__init__.py:36-51     settings -> GaussianRasterizer(raster_settings=...)
 *     gaussiansplatting/gaussian_renderer/__init__.py:86-94     rasterizer(means3D=, means2D=, shs=, colors_precomp=, opacities=, scales=, rotations=, cov3D_precomp=)
 *     gs_renderer.py:10-13, 951-966, 1006-1015                  same surface, animation path
 * Upstream's extension exposes rasterize_gaussians / rasterize_gaussians_backward / mark_visible to
 * Python; the three entry points below replace exactly those, with plain pointers and sizes
 * (no torch types), plus a view-batched form (n_views > 1) for the SDS view loop
 * (threestudio/systems/GaussianDreamer.py:244-248) and the animation frame loop (animation.py:1002-1013).
 *
 * Conventions
 *   - every `const float*` / `float*` / `int32_t*` / `void*` buffer is DEVICE memory on the current CUDA device
 *     unless the parameter comment says "host";
 *   - all kernels are enqueued on `stream` (a cudaStream_t passed as void*); functions return after enqueueing,
 *     except b200gs_forward which reads the instance count back once per call (upstream blocks on it in the middle of
 *     every view's forward).  For batches of up to 4 M (view, Gaussian) pairs every kernel of the forward is enqueued
 *     FIRST (sized for instance_capacity, the count read on the device) and the host then waits on an event recorded
 *     right after the scan -- the GPU never idles behind the host; larger batches wait once in place.
 *     b200gs_backward_deterministic also waits once, for its partial count;
 *   - return value 0 = success, negative = b200gs_status; nothing throws across the ABI; process state is limited to an
 *     error string, a launch counter, the optional stage profiler and one pinned count word + event per (thread, device);
 *   - matrices are the reference's row-vector-convention 4x4 tensors read as 16 contiguous floats
 *     (world_view_transform / full_proj_transform, gaussiansplatting/scene/cameras.py:50-52).
 */
#ifndef B200GS_H
#define B200GS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200GS_ABI_VERSION 5
#define B200GS_MAX_VIEWS 64 /* per call; callers chunk larger batches */

typedef enum b200gs_status {
    B200GS_OK = 0,
    B200GS_E_ARGS = -1,         /* inconsistent arguments (both/neither of shs|colors_precomp, scales+rotations|cov3D_precomp, ...) */
    B200GS_E_BIN_TOO_SMALL = -2, /* binning buffer cannot hold the instances; *num_rendered holds the count needed: grow and call again */
    B200GS_E_BUFFER = -3,        /* a state buffer is smaller than b200gs_*_bytes() asks for */
    B200GS_E_CUDA = -4,          /* a CUDA call failed; see b200gs_last_cuda_error() */
    B200GS_E_RANGE = -5,         /* sizes outside supported range (sh_degree > 3, n_views > B200GS_MAX_VIEWS, P*V >= 2^32, > 65535 tiles per axis) */
    B200GS_E_INSTANCES = -6,     /* the batch has more than B200GS_MAX_INSTANCES (Gaussian, tile) instances; *num_rendered holds the exact
                                    64-bit count; nothing was emitted: render fewer views per call (the host mirror halves the batch) */
    B200GS_E_UNSUPPORTED = -7    /* this build of the library does not implement the call (the classic comparator's deterministic backward) */
} b200gs_status;
#define B200GS_MAX_INSTANCES 0x7fffffffLL

/* Mirrors GaussianRasterizationSettings (12 fields; built at gaussian_renderer/__init__.py:36-49) plus sizes.
 * tanfovx/tanfovy are per view (host arrays) because every camera of an SDS batch has its own fovy
 * (threestudio/data/uncond.py:421-426). */
typedef struct b200gs_params {
    int32_t abi_version;    /* = B200GS_ABI_VERSION */
    int32_t P;              /* number of Gaussians */
    int32_t n_views;        /* V >= 1 cameras rendered by this call */
    int32_t sh_degree;      /* active degree 0..3 (ignored when colors_precomp is given) */
    int32_t sh_coeffs;      /* M = second dimension of shs [P,M,3]; M >= (sh_degree+1)^2 */
    int32_t image_height;
    int32_t image_width;
    int32_t prefiltered;    /* accepted for surface parity; unused (as upstream) */
    int32_t debug;          /* accepted for surface parity; unused */
    float scale_modifier;
    const float *tanfovx;   /* host, [V] */
    const float *tanfovy;   /* host, [V] */
    int32_t means3D_per_view; /* 0: means3D is [P,3], shared by all views (SDS batch).  1: means3D is [V,P,3] -- every
                               * view has its own positions, everything else shared: the animation frame batch
                               * (animation.py:383-403 moves only xyz between frames).  dL_dmeans3D then is [V,P,3]. */
    int32_t raw_params;       /* 0: opacities / scales / rotations are post-activation values, as upstream's rasteriser takes them.
                               * 1: they are GaussianModel's RAW parameters (_opacity logits, _scaling logs, un-normalised _rotation);
                               * the getters' sigmoid / exp / F.normalize (scene/gaussian_model.py:95-118) are applied inside the
                               * preprocess kernel and their Jacobians inside the backward kernel, so dL_dopacity / dL_dscales /
                               * dL_drots are gradients w.r.t. the raw tensors (SURVEY.md 8f-1).  cov3D_precomp is unaffected. */
} b200gs_params;

/* ---- buffer sizing (bytes).  The caller owns three opaque state buffers, exactly as upstream's
 *      geomBuffer / binningBuffer / imgBuffer tensors are owned by the autograd ctx. -------------------------- */
size_t b200gs_geom_bytes(int32_t P, int32_t n_views);
size_t b200gs_image_bytes(int32_t image_height, int32_t image_width, int32_t n_views);
size_t b200gs_binning_bytes(int64_t instance_capacity, int32_t image_height, int32_t image_width, int32_t P, int32_t n_views);
size_t b200gs_backward_scratch_bytes(int32_t P, int32_t n_views);

/*
 * Forward: preprocess (cull, project, 3D->2D covariance, SH) -> tile binning (scan, key emit, depth sort,
 * tile ranges) -> front-to-back alpha blend.  Replaces rasterize_gaussians.
 *   means3D [P,3] (or [V,P,3], see means3D_per_view); exactly one of shs [P,M,3] | colors_precomp [P,3]; opacities [P] (post-sigmoid);
 *   exactly one of (scales [P,3] post-exp AND rotations [P,4] (w,x,y,z)) | cov3D_precomp [P,6];
 *   bg [3]; viewmatrix [V,16]; projmatrix [V,16]; campos [V,3].
 * Outputs: out_color [V,3,H,W]; out_depth [V,1,H,W]; out_alpha [V,1,H,W]; radii [V,P] int32.
 * instance_capacity = the capacity binning_buf was sized for with b200gs_binning_bytes().
 * num_rendered (host, int64[1]) receives the EXACT (64-bit) number of (Gaussian,tile) instances over all views;
 * if it exceeds instance_capacity the call returns B200GS_E_BIN_TOO_SMALL (grow, call again: the outputs of the failed
 * call are unspecified but every access stayed inside the buffers); above B200GS_MAX_INSTANCES it returns
 * B200GS_E_INSTANCES (render fewer views per call).
 */
int b200gs_forward(const b200gs_params *prm,
                   const float *means3D, const float *shs, const float *colors_precomp, const float *opacities,
                   const float *scales, const float *rotations, const float *cov3D_precomp,
                   const float *bg, const float *viewmatrix, const float *projmatrix, const float *campos,
                   float *out_color, float *out_depth, float *out_alpha, int32_t *radii,
                   void *geom_buf, size_t geom_bytes,
                   void *binning_buf, size_t binning_bytes, int64_t instance_capacity,
                   void *image_buf, size_t image_bytes,
                   int64_t *num_rendered, void *stream);

/*
 * Backward: back-to-front blend replay with per-Gaussian gradient accumulation -> conic/cov2D backward ->
 * projection / depth / SH / cov3D backward.  Replaces rasterize_gaussians_backward.  Uses the three state
 * buffers written by the matching b200gs_forward call (same prm, same inputs).
 *   dL_dcolor [V,3,H,W]; dL_ddepth [V,1,H,W]; dL_dalpha [V,1,H,W]  (any may be NULL = zero).
 * Gradient outputs (overwritten, not accumulated).  Parameter gradients are summed over the V views:
 *   dL_dmeans3D [P,3] (per-view means: [V,P,3], not summed); dL_dmeans2D [V,P,3] (xy in NDC units, z = 0: the densification signal,
 *   GaussianDreamer.py:385-391); dL_dsh [P,M,3] | dL_dcolors [P,3]; dL_dopacity [P];
 *   dL_dscales [P,3] + dL_drots [P,4] | dL_dcov3D [P,6].
 */
int b200gs_backward(const b200gs_params *prm,
                    const float *means3D, const float *shs, const float *colors_precomp, const float *opacities,
                    const float *scales, const float *rotations, const float *cov3D_precomp,
                    const float *bg, const float *viewmatrix, const float *projmatrix, const float *campos,
                    const int32_t *radii,
                    const void *geom_buf, const void *binning_buf, int64_t instance_capacity,
                    const void *image_buf, int64_t num_rendered,
                    const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                    float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors, float *dL_dopacity,
                    float *dL_dscales, float *dL_drots, float *dL_dcov3D,
                    void *scratch, size_t scratch_bytes, void *stream);

/*
 * Deterministic backward: the same arguments, outputs and gradients as b200gs_backward, bit-reproducible from the forward
 * state.  b200gs_backward adds each (tile, 8x4 patch) partial sum of the backward blend into its Gaussian's record with float
 * atomics, in an order that depends on scheduling; this call stores every partial into its own slot of det_buf and then adds
 * each (view, Gaussian)'s partials in a fixed order: its tiles in emission order (its screen rect row-major), within a tile its
 * patches ascending, sequential fp32 adds.  Two calls on the same forward state write identical bytes.
 *   det_buf: b200gs_deterministic_bytes(num_rendered, partial_capacity, P, n_views) bytes, 16-byte aligned.  Its first
 *     num_rendered bytes hold, after the call, the patch mask of every sorted instance (bit p: the instance has a partial for
 *     patch p of its tile).  num_rendered must be the matching forward's count.
 *   partial_capacity: partials det_buf was sized for; *n_partials (host, int64[1]) receives the exact number H the call
 *     needs.  If H > partial_capacity the call returns B200GS_E_BIN_TOO_SMALL before any gradient is written (grow, call
 *     again; every access stayed inside the buffers); H >= 2^32 returns B200GS_E_RANGE.
 * Unlike b200gs_backward this call waits on the host once: for H, read back after the plan pre-pass and before the blend.
 * The classic comparator build returns B200GS_E_UNSUPPORTED.
 */
size_t b200gs_deterministic_bytes(int64_t num_rendered, int64_t partial_capacity, int32_t P, int32_t n_views);
int b200gs_backward_deterministic(const b200gs_params *prm,
                                  const float *means3D, const float *shs, const float *colors_precomp, const float *opacities,
                                  const float *scales, const float *rotations, const float *cov3D_precomp,
                                  const float *bg, const float *viewmatrix, const float *projmatrix, const float *campos,
                                  const int32_t *radii,
                                  const void *geom_buf, const void *binning_buf, int64_t instance_capacity,
                                  const void *image_buf, int64_t num_rendered,
                                  const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                                  float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors, float *dL_dopacity,
                                  float *dL_dscales, float *dL_drots, float *dL_dcov3D,
                                  void *scratch, size_t scratch_bytes,
                                  void *det_buf, size_t det_bytes, int64_t partial_capacity, int64_t *n_partials, void *stream);

/* ---- render options ---------------------------------------------------------------------------------------------------
 * The *_opts entry points take the argument list of their plain counterpart with `opts` after `prm`.  opts == NULL means the
 * defaults, which is exactly what b200gs_forward / b200gs_backward / b200gs_backward_deterministic do.  A backward call MUST
 * get the same options as the forward call whose state buffers it reads.
 *   struct_bytes: sizeof(b200gs_render_opts) of the caller's header.  8 (a header before filter3d_var) reads antialiasing
 *     only; 16 (a header that ends with filter3d_var) reads both; >= sizeof(b200gs_render_opts) reads every field; any other
 *     value is B200GS_E_ARGS.
 *   antialiasing: 0 = off.  Non-zero = the screen-space mip filter: the covariance keeps its +0.3 px^2 dilation and the
 *     opacity is multiplied by rho = sqrt(det(S) / det(S + 0.3 I)), S the projected 2D covariance, floored at rho = 0.005,
 *     so that a Gaussian's integrated footprint does not depend on the pixel scale it is drawn at.  The backward then needs
 *     opacities (as for raw_params); dL_dopacity is w.r.t. the opacity before the filter.
 *   filter3d_var: NULL = off.  Otherwise [P] device fp32 variances v >= 0 (finite; world length^2, e.g. from
 *     b200gs_sampling_rate): the 3D smoothing filter.  Per Gaussian, before scale_modifier, the activated scales become
 *     s'_i = sqrt(s_i^2 + v) and the opacity o * sqrt(prod_i s_i^2 / (s_i^2 + v)), so that its integrated 3D weight is kept;
 *     the backward's dL_dscales / dL_dopacity are w.r.t. the unfiltered parameters, and v gets no gradient.  With
 *     cov3D_precomp it is B200GS_E_ARGS; the backward needs opacities.  Only shape is checked, not the values (no sync).
 * The other fields are NULL when their feature is off; each feature below says which fields turn it on.  A build of the
 * library without a feature returns B200GS_E_UNSUPPORTED for a call that turns it on, before any other argument check: the
 * classic comparator has none of the four, nor the deterministic backward.  Contribution scores together with normals or
 * geometry are B200GS_E_ARGS.
 *
 * Normal maps: each Gaussian's shortest-axis normal blended like its colour.  On in a forward iff gauss_normals is set; on
 * in a backward iff gauss_normals and dL_dnormal are both set (dL_dnormal without gauss_normals is B200GS_E_ARGS).
 * For view v and Gaussian g (DESIGN.md section 2):
 *   axis    k = argmin of the activated scales s (after exp for raw parameters; before scale_modifier and the 3D filter,
 *           which leave the argmin unchanged in exact arithmetic); on a tie the lowest index wins.
 *   normal  n = column k of R(q), q the rotation as the covariance uses it (after the in-kernel normalise for raw), formed
 *           with the covariance's own float operations; not renormalised.
 *   flip    d = n . (campos_v - mean_{v,g}) as fmul, fma, fma over components 0, 1, 2 of fsub(campos, mean); if d < 0, n
 *           becomes -n (it faces the camera).  mean is the per-view position with means3D_per_view.  A NaN d keeps the sign.
 *   image   out_normal[v,c,p] = sum over the blends of pixel p of w n_c, accumulated as N_c = fma(n_c, w, N_c) with the
 *           colour's w = alpha * T and order.  No background term: [V,3,H,W], world space, unnormalised, 0 where nothing
 *           blends.
 *   grads   dL/dN enters dL/dalpha as cg += n . dL/dN.  Wn = sum w dL/dN per (view, Gaussian) is dL/dn; times the flip sign,
 *           through d(column k of R)/dq (and the normalise Jacobian for raw), it is ADDED to dL_drots.  Scales, means and
 *           campos get no gradient through n (the argmin and the flip are piecewise constant), only the alpha-path terms.
 * Colour, depth, alpha, radii and the state buffers are byte-identical to the call without normals, and the deterministic
 * partial count is unchanged.  cov3D_precomp has no axis: B200GS_E_ARGS.
 *   gauss_normals  [V*P] x 16 B device workspace, 16-byte aligned (else B200GS_E_BUFFER): the forward writes (sign n, sign)
 *                  of every (view, Gaussian); the backward reads it, so it must survive from the forward to its backward
 *                  like the state buffers
 *   out_normal     [V,3,H,W] (forward output; NULL in a forward is B200GS_E_ARGS)
 *   dL_dnormal     [V,3,H,W] (backward input); NULL = zero: the backward is then exactly the call without normals
 *   normal_wn      [V*P] x 16 B device workspace, 16-byte aligned (backward with dL_dnormal; NULL is B200GS_E_ARGS, else
 *                  B200GS_E_BUFFER): the Wn sums
 *   nrm_partials   deterministic backward with dL_dnormal: nrm_partials_bytes >= 16 * partial_capacity bytes, 16-byte
 *                  aligned, one float4 per partial at its slot (det_buf's layout and size do not change; NULL is
 *                  B200GS_E_ARGS, too small or misaligned B200GS_E_BUFFER)
 *
 * Geometry outputs: median depth and depth second moment of the blend.  On in a forward iff median_pos is set; on in a
 * backward iff dL_dmedian or dL_ddepth2 is set, and median_pos is then required.
 * For view v and pixel p, over the blends of p in the colour's order, with the colour's alpha, T (before the blend),
 * w = alpha * T and d the Gaussian's view-space depth (DESIGN.md section 2):
 *   depth2   out_depth2[v,0,p] = M2 = sum w d^2, accumulated as M2 = fma(d * d, w, M2).  No background term; 0 where nothing
 *            blends.  With alpha and depth: the depth distortion sum_{i<j} w_i w_j (d_i - d_j)^2 = A * M2 - M1^2.
 *   median   out_median[v,0,p] = d of the LAST blend whose T is > 0.5 (strict, on the float32 T): the blend at which T
 *            crosses 1/2, or the last blend if T never reaches it.  0 where nothing blends.  median_pos[v,p] = its 1-based
 *            position in the tile's list (0 = none).
 *   grads    dL/dM2 enters dL/dalpha as cg += d^2 dL/dM2, and adds sum_p w 2d dL/dM2 to the Gaussian's depth gradient.
 *            dL/dmedian adds dL/dmedian_p to the depth gradient of p's median Gaussian only (the selection is piecewise
 *            constant: no alpha-path term).  Both reach the means through the existing depth term.
 * Colour, depth, alpha, normals, radii and the state buffers are byte-identical to the call without geometry, and the
 * deterministic partial count is unchanged.  Combines with SH or precomputed colours, raw parameters, cov3D_precomp,
 * antialiasing, the 3D filter, per-view means, normals, absgrad and the deterministic backward.
 *   median_pos     [V,H,W] x u32 device workspace, 4-byte aligned (else B200GS_E_BUFFER): the forward writes it, the
 *                  backward reads it, so it must survive from the forward to its backward like the state buffers
 *   out_median     [V,1,H,W] (forward output; NULL in a forward is B200GS_E_ARGS)
 *   out_depth2     [V,1,H,W] (forward output; NULL in a forward is B200GS_E_ARGS)
 *   dL_dmedian     [V,1,H,W] (backward input); NULL = zero
 *   dL_ddepth2     [V,1,H,W] (backward input); NULL = zero.  With both NULL the backward is exactly the call without geometry.
 *
 * Contribution scores: per-Gaussian blend weights of the forward blend.  On in a forward iff any of weight_sum, weight_max and
 * touches is set, and then all three are required (else B200GS_E_ARGS); a backward does not read them.  The forward computes
 * every output exactly as without them (images, radii, state buffers byte-identical), plus three per-Gaussian accumulators
 * over every pixel of every view:
 *   For pixel p and sorted tile-list entry k of p's tile the blend evaluates power, alpha and test_T = T (1 - alpha).
 *   touch: power <= 0 and alpha >= 1/255 while the pixel is live (its T before the entry is > 0; out-of-image pixels never
 *     are).  A touch either blends or is the single terminating hit at which T would drop below 1e-4 (it ends the pixel
 *     without blending).
 *   blend: a touch that blends, with weight w = fmul(alpha, T), the float the colour sum uses.
 *   weight_sum [P] u64 (device, in/out): += sum over blends of q(w) = round-half-even(w * 2^24) (w <= 0.99, so q < 2^24).
 *     weight_sum * 2^-24 is the sum of weights to within 2^-25 per blend.
 *   weight_max [P] u32 (device, in/out): max(weight_max, bits of w) over blends (w > 0: unsigned order is float order;
 *     0 = never blended).  Read it as a float.
 *   touches [P] u32 (device, in/out): += number of touches.
 * Integer adds and maxima: any camera set, in calls of any size and order, folds to the same bits, and two runs write
 * identical bytes.  PRECONDITION: the total pixel count sum(V*H*W) folded into one set of accumulators stays below 2^32
 * (each pixel adds at most 1 to touches and less than 2^24 to weight_sum, so neither can overflow).
 * Removing every Gaussian with touches == 0 over a camera set, survivors kept in order, leaves those cameras' colour,
 * depth and alpha byte-identical and the survivors' radii unchanged (DESIGN.md section 2).
 * This forward always waits for the instance count before the blend: one that returns B200GS_E_BIN_TOO_SMALL or
 * B200GS_E_INSTANCES has not touched the accumulators.
 *
 * Absolute screen-space gradients for densification.  On in a backward iff dL_dmeans2D_abs is set; a forward does not read
 * them.  Every other output is exactly what the call without them computes.
 *   dL_dmeans2D_abs [V,P,3] (device, overwritten): per (view, Gaussian), the per-pixel terms of dL_dmeans2D summed in
 *     absolute value per component: ( sum_p |g_p.x|, sum_p |g_p.y|, 0 ), NDC units like dL_dmeans2D, where g_p = dL_p /
 *     dmean2D is pixel p's term of the signed gradient.  The signed sum cancels where a Gaussian's pixels pull its centre in
 *     opposite directions; this one does not (the "absgrad" / homodirectional densification statistic).  Zero where
 *     radii == 0.  b200gs_densify_stats accepts it in place of dL_dmeans2D.
 *   abs_partials (deterministic backward only): a caller-owned device array of abs_partials_bytes >= 8 * partial_capacity
 *     bytes, 8-byte aligned (else B200GS_E_BUFFER; NULL is B200GS_E_ARGS): one float2 per partial, at the partial's slot.
 *     It is separate from det_buf, whose layout and size (b200gs_deterministic_bytes) do not change.  The absolute sums are
 *     then bit-reproducible like every other output. */
typedef struct b200gs_render_opts {
    int32_t struct_bytes;      /* sizeof(b200gs_render_opts) */
    int32_t antialiasing;      /* 0 | 1 */
    const float *filter3d_var; /* [P] or NULL */
    /* normal maps */
    float *gauss_normals;
    float *out_normal;
    const float *dL_dnormal;
    float *normal_wn;
    void *nrm_partials;
    size_t nrm_partials_bytes;
    /* geometry outputs */
    uint32_t *median_pos;
    float *out_median;
    float *out_depth2;
    const float *dL_dmedian;
    const float *dL_ddepth2;
    /* contribution scores (forward) */
    uint64_t *weight_sum;
    uint32_t *weight_max;
    uint32_t *touches;
    /* absolute screen-space gradients (backward) */
    float *dL_dmeans2D_abs;
    void *abs_partials;
    size_t abs_partials_bytes;
} b200gs_render_opts;
int b200gs_forward_opts(const b200gs_params *prm, const b200gs_render_opts *opts,
                        const float *means3D, const float *shs, const float *colors_precomp, const float *opacities,
                        const float *scales, const float *rotations, const float *cov3D_precomp,
                        const float *bg, const float *viewmatrix, const float *projmatrix, const float *campos,
                        float *out_color, float *out_depth, float *out_alpha, int32_t *radii,
                        void *geom_buf, size_t geom_bytes,
                        void *binning_buf, size_t binning_bytes, int64_t instance_capacity,
                        void *image_buf, size_t image_bytes,
                        int64_t *num_rendered, void *stream);
int b200gs_backward_opts(const b200gs_params *prm, const b200gs_render_opts *opts,
                         const float *means3D, const float *shs, const float *colors_precomp, const float *opacities,
                         const float *scales, const float *rotations, const float *cov3D_precomp,
                         const float *bg, const float *viewmatrix, const float *projmatrix, const float *campos,
                         const int32_t *radii,
                         const void *geom_buf, const void *binning_buf, int64_t instance_capacity,
                         const void *image_buf, int64_t num_rendered,
                         const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                         float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors, float *dL_dopacity,
                         float *dL_dscales, float *dL_drots, float *dL_dcov3D,
                         void *scratch, size_t scratch_bytes, void *stream);
int b200gs_backward_deterministic_opts(const b200gs_params *prm, const b200gs_render_opts *opts,
                                       const float *means3D, const float *shs, const float *colors_precomp, const float *opacities,
                                       const float *scales, const float *rotations, const float *cov3D_precomp,
                                       const float *bg, const float *viewmatrix, const float *projmatrix, const float *campos,
                                       const int32_t *radii,
                                       const void *geom_buf, const void *binning_buf, int64_t instance_capacity,
                                       const void *image_buf, int64_t num_rendered,
                                       const float *dL_dcolor, const float *dL_ddepth, const float *dL_dalpha,
                                       float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors, float *dL_dopacity,
                                       float *dL_dscales, float *dL_drots, float *dL_dcov3D,
                                       void *scratch, size_t scratch_bytes,
                                       void *det_buf, size_t det_bytes, int64_t partial_capacity, int64_t *n_partials, void *stream);

/* ---- 3D smoothing filter: per-Gaussian maximal sampling rate over a camera set (Mip-Splatting's 3D filter) ------------
 * For each of the n_views cameras (viewmatrix [n_views,16] device, tanfovx / tanfovy host [n_views], shared H x W), with
 * (tx, ty, tz) the preprocess's view-space position and fx = W / (2 tanfovx), fy = H / (2 tanfovy): Gaussian k is in view
 * iff tz > 0.2, |tx / tz * fx| <= 0.65 W and |ty / tz * fy| <= 0.65 H (the image plus a 15 % margin per side; a NaN
 * position is out).  Then max_rate[k] = max(max_rate[k], max(fx, fy) / tz) (in/out, device [P]).  The fold is a max, so
 * any camera set passed in chunks of at most B200GS_MAX_VIEWS, in any order, gives the same bits.  The filter variance is
 * then c / max_rate^2 (DESIGN.md section 2; humangaussian_b200.filter3d).  n_views > B200GS_MAX_VIEWS: B200GS_E_RANGE. */
int b200gs_sampling_rate(int32_t P, int32_t n_views, const float *means3D, const float *viewmatrix, const float *tanfovx,
                         const float *tanfovy, int32_t image_height, int32_t image_width, float *max_rate, void *stream);

/* Frustum test only (upstream markVisible): present[i] = 1 if p_view.z > 0.2 for view 0.  positions [P,3]. */
int b200gs_mark_visible(int32_t P, const float *positions, const float *viewmatrix, const float *projmatrix,
                        uint8_t *present, void *stream);

/* ---- animation frame path (reference animation.py) --------------------------------------------------------------
 * Re-attachment of the Gaussians to a re-posed body mesh, for n_frames poses at once (animation.py:383-403 does one
 * frame per call in numpy): xyz_out[f,i] = u*v0 + v*v1 + w*v2 + dist[i] * unit_normal(face), face = faces[mapping_face[i]].
 *   vertices [n_frames, n_verts, 3]; faces [n_faces,3] int32; mapping_face [P] int32; mapping_uvw [P,3]; mapping_dist [P];
 *   xyz_out [n_frames, P, 3] -- feed it to b200gs_forward with means3D_per_view = 1.
 *   A mapping_face outside [0, n_faces) or a face index outside [0, n_verts) is never dereferenced: that Gaussian's
 *   positions become NaN (it is culled by the preprocess), where the reference's numpy indexing raises. */
int b200gs_reattach(int32_t P, int32_t n_frames, int32_t n_verts, int32_t n_faces, const float *vertices, const int32_t *faces,
                    const int32_t *mapping_face, const float *mapping_uvw, const float *mapping_dist, float *xyz_out, void *stream);
/* clamp(color,0,1) (gs_renderer.py:1017) then CHW float -> HWC uint8 by truncation of x*255 (animation.py:1011).
 *   color [n_frames,3,H,W] -> out [n_frames,H,W,3] uint8 */
int b200gs_pack_frames_u8(const float *color, uint8_t *out, int32_t image_height, int32_t image_width, int32_t n_frames, void *stream);

/* ---- scene initialisation helper (reference: simple_knn._C.distCUDA2, gaussiansplatting/submodules/simple-knn/
 * simple_knn.cu:63-221 via spatial.cu:15-26; callers scene/gaussian_model.py:134, gs_renderer.py:386-389) ----------
 * mean_dist2[i] = mean of the squared distances from points[i] to its 3 nearest other points (exact kNN).
 *   points [P,3]; mean_dist2 [P]; scratch of b200gs_knn_scratch_bytes(P) bytes; P >= 4. */
size_t b200gs_knn_scratch_bytes(int32_t P);
int b200gs_dist2_knn3(int32_t P, const float *points, float *mean_dist2, void *scratch, size_t scratch_bytes, void *stream);

/* ---- densification / pruning on the device (reference gaussiansplatting/scene/gaussian_model.py:268-437, driven from
 * threestudio/systems/GaussianDreamer.py:378-408) ----------------------------------------------------------------------
 * Parameters are the RAW (pre-activation) optimiser tensors, one array per group as the reference holds them.
 *
 * b200gs_densify_stats: one optimiser step's bookkeeping for a V-view batch (GaussianDreamer.py:385-391 +
 *   add_densification_stats, gaussian_model.py:433-437): g = sum_v dL_dmeans2D[v] ; r = max_v radii[v] ; where r > 0:
 *   max_radii2D = max(max_radii2D, r), xyz_gradient_accum += |g.xy|, denom += 1.
 *     dL_dmeans2D [V,P,3] (what b200gs_backward wrote), radii [V,P] int32; accum, denom, max_radii2D [P] (in/out).
 *   update_mask [P] uint8 or NULL: ANDed with r > 0 -- the reference's visibility_filter can exclude points before this
 *   bookkeeping (disable_hand_densification / hand_radius, GaussianDreamer.py:288-297). */
int b200gs_densify_stats(int32_t P, int32_t n_views, const float *dL_dmeans2D, const int32_t *radii, const uint8_t *update_mask,
                         float *xyz_gradient_accum, float *denom, float *max_radii2D, void *stream);

typedef struct b200gs_densify_cfg {
    int32_t mode;            /* 0 = densify_and_prune (gaussian_model.py:402-415), 1 = prune_only (:423-430) */
    int32_t n_split;         /* children per split Gaussian; the reference uses N = 2 */
    int32_t use_screen;      /* mode 0: the reference's `if max_screen_size:` (None / 0 -> 0) */
    float max_grad;          /* mode 0 */
    float min_opacity;
    float percent_dense_x_extent; /* mode 0: clone at or below, split above */
    float max_screen_size;   /* mode 0 with use_screen (compared with the statistics AFTER their reset, as the reference does) */
    float big_ws_thresh;     /* mode 0 with use_screen: 0.1 * extent;  mode 1: size_thresh */
} b200gs_densify_cfg;

/* Plans the surgery.  plan [4,P] int32 (device): rows = destination of the surviving original, of its clone, of its first
 * split child (child c lands S_kept*c rows further), and the parent's row in the noise block; -1 = none.
 * counts [5] int32 (device): n_keep, n_clone, S_sel (split parents), S_kept (split parents whose children survive),
 * P_new = n_keep + n_clone + n_split*S_kept.  Output row order is the reference's: surviving unsplit originals, clones,
 * children copy 0, children copy 1.  scratch: b200gs_densify_scratch_bytes(P). */
size_t b200gs_densify_scratch_bytes(int32_t P);
int b200gs_densify_plan(int32_t P, const b200gs_densify_cfg *cfg, const float *xyz_gradient_accum, const float *denom,
                        const float *opacity_raw, const float *scaling_raw, int32_t *plan, int32_t *counts,
                        void *scratch, size_t scratch_bytes, void *stream);

/* Plans a prune by mask in the same plan [4,P] / counts [5] layout, for b200gs_densify_move with n_split = 0: Gaussian i
 * survives iff remove[i] == 0 (remove [P] uint8, device), survivors keep their order, nothing is cloned or split
 * (counts = n_keep, 0, 0, 0, n_keep).  scratch: b200gs_densify_scratch_bytes(P).  P >= 1. */
int b200gs_prune_plan(int32_t P, const uint8_t *remove, int32_t *plan, int32_t *counts, void *scratch, size_t scratch_bytes,
                      void *stream);

/* Moves one [P,row_floats] array to its planned [P_new,row_floats] place.  role: */
enum { B200GS_ROLE_COPY = 0,    /* new rows repeat the parent row (f_dc, f_rest, opacity, rotation; statistics in mode 1) */
       B200GS_ROLE_XYZ = 1,     /* children: R(rotation) (noise * exp(scaling)) + xyz  (gaussian_model.py:369-373) */
       B200GS_ROLE_SCALING = 2, /* children: log(exp(scaling) / (0.8 n_split))          (gaussian_model.py:374) */
       B200GS_ROLE_MOMENT = 3 };/* Adam exp_avg / exp_avg_sq: new rows are zero         (gaussian_model.py:317-341) */
/*   counts_host [5]: the plan's counts, read back by the caller (it needs P_new to allocate dst anyway);
 *   rotation_raw [P,4], scaling_raw [P,3], noise [n_split*S_sel,3] standard-normal draws: only read for B200GS_ROLE_XYZ. */
int b200gs_densify_move(int32_t role, int32_t P, int32_t row_floats, const int32_t *plan, const int32_t *counts_host,
                        int32_t n_split, const float *src, float *dst, const float *rotation_raw, const float *scaling_raw,
                        const float *noise, void *stream);

/* ---- MCMC densification (3DGS-MCMC, Kheradmand et al., NeurIPS 2024): relocation of dead Gaussians, growth to a budget
 * and position noise, in place of the gradient-threshold rule above.  Parameters are the RAW optimiser arrays
 * (opacity logits [P], log-scales [P,3], un-normalised quaternions [P,4]); any row stride-exact fp32 array works, so the
 * packed buffer's field views and separate tensors both do.  sigma(x) = 1/(1+expf(-x)) in float32.
 *
 * b200gs_mcmc_noise: the per-step exploration term, one thread per Gaussian, one launch, no host sync:
 *   xyz_i += noise_scale * sigma(-k (sigma(opacity_i) - t)) * Sigma_i eta_i,   Sigma_i = R(q^_i) diag(exp(2 scaling_i)) R(q^_i)^T
 *   q^ = q / max(||q||, 1e-12) and R as the preprocess forms them; eta [P,3] standard-normal draws (an input);
 *   noise_scale = lambda_noise * lr_xyz (the lr of the step just taken).  Only xyz [P,3] is written. */
int b200gs_mcmc_noise(int32_t P, float *xyz, const float *scaling_raw, const float *rotation_raw, const float *opacity_raw,
                      const float *eta, float noise_scale, float k, float t, void *stream);

/* b200gs_mcmc_ratio: for every row s with c = counts[s] > 0 (s was drawn c times as a source; counts [P] int32, device),
 * the raw opacity and log-scales that all n = min(c+1, 51) members of s (s and its copies) take, in float64, rounded once:
 *   o = sigma(opacity_s);  o' = clamp(1 - (1-o)^(1/n), 0.005, 1 - 2^-23);
 *   D = sum_{k=0}^{n-1} C(n,k+1) (-1)^k o'^(k+1) / sqrt(k+1);
 *   new_opacity[s] = log(o' / (1-o')),  new_scaling[s,j] = log(exp(scaling_s,j) o / D).
 * new_opacity [P], new_scaling [P,3]: rows with counts == 0 are not written. */
int b200gs_mcmc_ratio(int32_t P, const int32_t *counts, const float *opacity_raw, const float *scaling_raw, float *new_opacity,
                      float *new_scaling, void *stream);

/* b200gs_mcmc_move: gathers one [P,row_floats] array into [P_new,row_floats]: dst[i] = src[map[i]] (map [P_new] int32 in
 * [0,P), device).  Row i is reset iff counts[map[i]] > 0; there the role decides:  */
enum { B200GS_MCMC_ROLE_COPY = 0,    /* always the source row (xyz, rotation, SH) */
       B200GS_MCMC_ROLE_OPACITY = 1, /* new_opacity[map[i]] (row_floats 1) */
       B200GS_MCMC_ROLE_SCALING = 2, /* new_scaling[map[i]] (row_floats 3) */
       B200GS_MCMC_ROLE_MOMENT = 3 };/* zero (Adam exp_avg / exp_avg_sq) */
/* Relocation: map = identity except map[dead_j] = sample_j; growth: map = identity ++ samples.  dst must not alias src. */
int b200gs_mcmc_move(int32_t role, int32_t P, int32_t P_new, int32_t row_floats, const int32_t *map, const int32_t *counts,
                     const float *src, float *dst, const float *new_opacity, const float *new_scaling, void *stream);

/* ---- Adam over the packed parameter buffer (the reference's optimiser, gaussian_model.py:156-165) ------------------
 * One step of torch.optim.Adam (amsgrad=False, weight_decay=0, maximize=False) over the flat fp32 buffer
 * [xyz 3P | scaling 3P | rotation 4P | opacity P | sh 3*sh_coeffs*P] that the packed forward reads and the packed backward
 * writes the gradient of, with the reference's six parameter groups: xyz, scaling, rotation and opacity are one field each;
 * inside the sh field [P,sh_coeffs,3] coefficient 0 is f_dc and coefficients 1.. are f_rest.  exp_avg / exp_avg_sq have the
 * same layout.  Floats outside the five fields (alignment padding) are written as zero in params and both moments.
 * The scalars are what torch computes on the host for step t, in double, rounded to float:
 *   step_size[g] = -(lr_g / (1 - beta1^t)),  bias_correction2_sqrt = (1 - beta2^t)^0.5. */
typedef struct b200gs_adam_cfg {
    int64_t off_xyz, off_scaling, off_rotation, off_opacity, off_sh; /* field offsets in floats: ascending, multiples of 4 */
    int32_t P;
    int32_t sh_coeffs;           /* K >= 1 */
    int64_t total;               /* floats in each buffer; a multiple of 4 */
    float step_size[6];          /* by group: xyz, f_dc, f_rest, opacity, scaling, rotation */
    float bias_correction2_sqrt;
    float one_minus_beta1;
    float beta2;
    float one_minus_beta2;
    float eps;
} b200gs_adam_cfg;
/* params, exp_avg, exp_avg_sq updated in place; grads read.  All four 16-byte aligned, `total` floats each. */
int b200gs_adam_packed(const b200gs_adam_cfg *cfg, float *params, const float *grads, float *exp_avg, float *exp_avg_sq,
                       void *stream);

/* ---- mesh export (the reference's GaussianModel.extract_fields / extract_mesh, gs_renderer.py:241-361) -------------
 * b200gs_density_field: field [res,res,res] (device, x-major: field[(x*res + y)*res + z]) of
 *   sum over Gaussians g of block(x,y,z) of opacities[g] * exp(power),  power = -0.5 (d^T Sigma^-1 d) (0 where power > 0),
 *   d = (samples[x], samples[y], samples[z]) - means[g], Sigma^-1 the closed-form inverse of cov6 [a,b,c,d,e,f] =
 *   [xx,xy,xz,yy,yz,zz] with 1e-24 added to the determinant, every product and sum in the reference's order, rounded once.
 *   Blocks are chunks of split = res / num_blocks samples per axis (the last may be short; there may be more than
 *   num_blocks).  Gaussian g belongs to a block iff, on all three axes, min(chunk samples) - relax < mean < max(chunk
 *   samples) + relax in float32.  The sum runs in a fixed order: the same bits on every call.
 *     means [P,3], cov6 [P,6], opacities [P], samples [res] (device); relax = (2 / num_blocks) * relax_ratio as a float;
 *     scratch of b200gs_density_field_scratch_bytes(P, res, num_blocks).  P = 0 zeroes the field.
 *   B200GS_E_ARGS: P < 0, res < 1 or num_blocks < 1; B200GS_E_RANGE: res / num_blocks < 1, or the blocks or the field's
 *   CTAs (one per block and 512 voxels) outgrow 32-bit indices. */
size_t b200gs_density_field_scratch_bytes(int32_t P, int32_t resolution, int32_t num_blocks);
int b200gs_density_field(int32_t P, const float *means, const float *cov6, const float *opacities, int32_t resolution,
                         int32_t num_blocks, const float *samples, float relax, float *field, void *scratch, size_t scratch_bytes,
                         void *stream);
/* b200gs_field_query: the field of b200gs_density_field (same Gaussians, resolution, num_blocks, samples, relax) at
 * n_points arbitrary points q [n,3] of the same normalised frame, with its gradient and an SH colour.
 *   Members: per axis h(q_a) = the largest chunk c with c == 0 or samples[c*split] <= q_a; the members of q are the
 *   Gaussians the field counts for block (h(qx), h(qy), h(qz)) -- at a grid sample, exactly its voxel's members.
 *   Weights w_g = opacities[g] * exp(p_g(q)), p_g in the field's float32 operations and order, with its cut-offs (p > 0
 *   and p <= -104 add nothing).  Sums run over the members in the field's order, so every run writes the same bits and
 *   a point's result does not depend on the other points.
 *     density [n]   D = sum w_g; at a grid sample the same bits as the field's voxel.
 *     normals [n,3] n = -G / |G| with G = sum w_g (-Sigma_g^-1 (q - mean_g)) (Sigma^-1 the field's inverse): outward,
 *                   toward lower density, as marching cubes winds its triangles; 0 where |G| = 0.  The world mapping
 *                   is a uniform scale and a translation, so n is also the world normal.
 *     colors [n,3]  max(SH(S / D, -n) + 0.5, 0) per channel, S = sum w_g sh_g over the first (sh_degree+1)^2
 *                   coefficients of shs [P,sh_coeffs,3], SH the render preprocess's basis; the DC term alone where n = 0
 *                   (pass sh_degree 0 for a view-independent colour).  The SH of the opacity-weighted mean
 *                   coefficients, not the mean of clamped per-Gaussian colours: the two differ only where one
 *                   Gaussian's colour would clamp at 0.
 *   Where D == 0 every output is 0; a non-finite point does not fault, but its outputs may be non-finite.  Any output
 *   may be NULL to skip it; shs may be NULL when colors is.  scratch of b200gs_field_query_scratch_bytes(P, n_points,
 *   res, num_blocks, sh_degree); n_points = 0 does nothing; P = 0 zeroes the outputs.
 *   B200GS_E_ARGS: as b200gs_density_field, and n_points < 0, sh_degree outside 0..3, colors without shs, or
 *   sh_coeffs < (sh_degree+1)^2 with shs; B200GS_E_RANGE as b200gs_density_field. */
size_t b200gs_field_query_scratch_bytes(int32_t P, int32_t n_points, int32_t resolution, int32_t num_blocks, int32_t sh_degree);
int b200gs_field_query(int32_t P, const float *means, const float *cov6, const float *opacities, const float *shs, int32_t sh_coeffs,
                       int32_t sh_degree, int32_t resolution, int32_t num_blocks, const float *samples, float relax, int32_t n_points,
                       const float *points, float *density, float *normals, float *colors, void *scratch, size_t scratch_bytes,
                       void *stream);
/* Marching cubes over volume [X,Y,Z] (device, z fastest) at `iso`: a corner is inside iff its value > iso; one vertex per
 * grid edge whose ends differ, at p0 + t along the edge, t = (iso - v0) / (v1 - v0), in index coordinates; triangles wound
 * with normals toward lower values.  Vertices are numbered in order of (grid point at the edge's low end, axis), triangles
 * in order of (cell, table row); the table is generated by humangaussian_b200/mc_table.py.
 *   b200gs_marching_cubes_count classifies and scans: counts [2] uint64 (device) = vertices, triangles.  The caller reads
 *   them (the one host wait of an extraction) to size vertices [n_vertices,3] float and faces [n_triangles,3] int32, then
 *   b200gs_marching_cubes_emit writes them from the same scratch (either output may be NULL to skip it).
 *   X, Y, Z >= 2 and 3*X*Y*Z <= INT32_MAX (vertex ids are int32), else B200GS_E_RANGE. */
size_t b200gs_marching_cubes_scratch_bytes(int32_t X, int32_t Y, int32_t Z);
int b200gs_marching_cubes_count(int32_t X, int32_t Y, int32_t Z, const float *volume, float iso, void *scratch, size_t scratch_bytes,
                                uint64_t *counts, void *stream);
int b200gs_marching_cubes_emit(int32_t X, int32_t Y, int32_t Z, const float *volume, float iso, const void *scratch,
                               size_t scratch_bytes, float *vertices, int32_t *faces, void *stream);

/* ---- introspection of the state buffers, for parity tests (tile/sort indices must match bit-for-bit) ------- */
typedef struct b200gs_state_view {
    const void *geom_records;     /* [V*P] x 48 B: px,py,hx,hy | conicA,conicB,conicC,opacity | r,g,b,depth */
    const uint32_t *tiles_touched;/* [V*P] */
    const uint32_t *offsets;      /* [V*P] inclusive scan of tiles_touched taken in depth order (see depth_order) */
    const uint8_t *clamped;       /* [V*P] bit c set = channel c clamped at 0 */
    const uint32_t *sorted_tile_keys; /* [num_rendered] view*tiles + tile of each sorted instance; the reference's 64-bit key
                                         of instance j is (sorted_tile_keys[j] << 32) | bits(depth of record point_list[j]) */
    const uint32_t *depth_order;  /* [V*P] record indices (view*P + i) sorted by (depth bits, record index), all views mixed */
    const uint32_t *point_list;   /* [num_rendered] Gaussian index of each sorted instance */
    const uint32_t *ranges;       /* [V*tiles][2] */
    const float *final_T;         /* [V,H,W] */
    const uint32_t *n_contrib;    /* [V,H,W] */
    const uint32_t *contributor_masks; /* [contributor_mask_words] written by the forward blend: word
                                          ((range.x >> 5) + vt + c) * 8 + patch, for tile vt = view*tiles + tile, is chunk c
                                          (list positions [32c, 32c+32)) of that tile and patch = ((py % 16) / 4) * 2 +
                                          (px % 16) / 8; bit l = entry 32c+l was blended by a pixel of the patch.  Defined
                                          for c <= (max n_contrib over the patch - 1) / 32; later words are unspecified */
    int64_t contributor_mask_words;
} b200gs_state_view;
int b200gs_describe_state(const b200gs_params *prm, const void *geom_buf, const void *binning_buf,
                          int64_t instance_capacity, const void *image_buf, b200gs_state_view *out);

/* The stable radix sort of the binning stage, exposed for tests: sorts n (u32 key, u32 value) pairs over the low
 * `nbits` key bits; buffers a/b ping-pong, *result_in_b tells which holds the result. */
int b200gs_test_sort_pairs(uint32_t *keys_a, uint32_t *keys_b, uint32_t *vals_a, uint32_t *vals_b, int64_t n, int32_t nbits,
                           void *scratch, size_t scratch_bytes, int32_t *result_in_b, void *stream);
size_t b200gs_test_sort_scratch_bytes(int64_t n);

/* The deterministic exp used by the blend kernels, evaluated on the device for n floats (parity pin vs oracle). */
int b200gs_test_exp(const float *x, float *y, int64_t n, void *stream);

/* ---- pose maps (humangaussian_b200/pose.py) ----------------------------------------------------------------------
 * The reference's skeleton images for n_views mvp matrices, in two launches on `stream` with no host wait:
 * b200gs_pose_keypoints projects the keypoints and rasterises every shape of every view into scratch, b200gs_pose_draw
 * writes the images from it.  style 0 is HumanSD (17 keypoints, 16 limbs, line thickness 10 * height / 512, so height
 * >= 103), style 1 OpenPose (18 keypoints, 17 limbs).
 *   points     device [n_keypoints, 4] float32, 16-byte aligned (the reference's Skeleton.points3D)
 *   mvp        device [n_views, 4, 4] float32 row-major;  occlusion: device [n_views] uint8 (0 / 1)
 *   limbs      HOST [limbs][2] int32 keypoint pairs in draw order (16 or 17 limbs)
 *   kp         device [n_views, n_keypoints, 2] float32 out, 8-byte aligned: (x, y) pixel coordinates before truncation
 *   colors     HOST [shapes][3] uint8 in draw order: HumanSD one per limb; OpenPose the 18 keypoint circles, then the
 *              17 limbs
 *   out        device [n_views, height, width, 3] float32, 16-byte aligned
 * scratch: b200gs_pose_scratch_bytes(style, n_views, height, width) bytes, 16-byte aligned, kept between the two
 * calls.  Returns B200GS_E_ARGS for a bad style, count, limb index or NULL pointer, B200GS_E_RANGE for sizes outside
 * 1..16384 (or a HumanSD height below 103), B200GS_E_BUFFER for a small or misaligned buffer. */
size_t b200gs_pose_scratch_bytes(int32_t style, int32_t n_views, int32_t height, int32_t width);
int b200gs_pose_keypoints(int32_t style, int32_t n_views, int32_t n_keypoints, int32_t height, int32_t width, const float *points,
                          const float *mvp, const uint8_t *occlusion, const int32_t *limbs, float *kp, void *scratch,
                          size_t scratch_bytes, void *stream);
int b200gs_pose_draw(int32_t style, int32_t n_views, int32_t height, int32_t width, const uint8_t *colors, const void *scratch,
                     size_t scratch_bytes, float *out, void *stream);

/* ---- mesh rendering (humangaussian_b200/meshrender.py; DESIGN.md section 2 is the specification) ------------------
 * Forward-only triangle rasterisation in nvdiffrast's instance mode (one topology, a batch of clip-space vertex sets),
 * attribute interpolation, and the reference's vertex normals and normal image (animation.py:558-601).  Every call
 * enqueues on `stream`; the results are the same bytes on every run.  n_views / n_frames must be 1..B200GS_MAX_VIEWS,
 * height and width 1..16384, n_faces 0..2^24 - 1 (triangle + 1 must be exact in float32), else B200GS_E_RANGE.  A NULL
 * pointer is B200GS_E_ARGS; a buffer smaller than its *_bytes query, or a pos / rast / scratch / pairs / incidence
 * pointer that is not 16-byte aligned (other arrays: 4-byte), is B200GS_E_BUFFER.
 *   pos    device [n_views, n_verts, 4] float32 clip coordinates (X, Y, Z, W)
 *   tri    device [n_faces, 3] int32; a triangle with an index outside [0, n_verts), a non-finite coordinate, or W <= 0
 *          at all three vertices is not drawn (and never dereferenced)
 *   rast   device [n_views, height, width, 4] float32: (u, v, z/w, triangle + 1) of the nearest covering triangle, all 0
 *          where none covers the pixel centre.  Row 0 is clip y = -1.  A triangle covers no pixel outside its pixel
 *          rectangle (its projected bounding box widened by one pixel, where every W > 0), so one whose edge functions
 *          are rounding noise (point-sized) draws at most there.
 * b200gs_mesh_raster_count sets up every (view, triangle), bins them into 16 x 16-pixel tiles and writes the exact number
 * of (tile, triangle) pairs to count (device, uint64[1]).  The caller reads it (the one host wait of a rasterisation) to
 * size pairs (>= 4 * count bytes) and calls b200gs_mesh_raster_emit with the same arguments and scratch, which fills the
 * tile lists and writes rast.  With a pairs buffer smaller than that the output is unspecified, but every access stays
 * inside the buffers. */
size_t b200gs_mesh_raster_scratch_bytes(int32_t n_views, int32_t n_faces, int32_t height, int32_t width);
int b200gs_mesh_raster_count(int32_t n_views, int32_t n_verts, int32_t n_faces, int32_t height, int32_t width, const float *pos,
                             const int32_t *tri, void *scratch, size_t scratch_bytes, uint64_t *count, void *stream);
int b200gs_mesh_raster_emit(int32_t n_views, int32_t n_verts, int32_t n_faces, int32_t height, int32_t width, void *scratch,
                            size_t scratch_bytes, int32_t *pairs, size_t pairs_bytes, float *rast, void *stream);
/* out [n_views, height, width, channels] = a0 u + a1 v + a2 ((1 - u) - v) of the rasterised triangle's vertex attributes,
 * 0 where rast.w is not a triangle id in 1..n_faces (or the triangle has an index outside [0, n_verts)).
 *   attr device [n_views, n_verts, channels] (attr_per_view = 1) or [n_verts, channels] shared by every view (0); channels >= 1 */
int b200gs_mesh_interpolate(int32_t n_views, int32_t height, int32_t width, int32_t n_verts, int32_t n_faces, int32_t channels,
                            const float *attr, int32_t attr_per_view, const float *rast, const int32_t *tri, float *out, void *stream);
/* The per-vertex face lists of one topology, built once for any number of frames: for every vertex its faces where it
 * is corner 0 in ascending face order, then corner 1, then corner 2.  A face with an index outside [0, n_verts) is in no
 * list.  incidence: b200gs_mesh_incidence_bytes(n_verts, n_faces) bytes, 16-byte aligned, kept for the normals calls. */
size_t b200gs_mesh_incidence_bytes(int32_t n_verts, int32_t n_faces);
int b200gs_mesh_incidence(int32_t n_verts, int32_t n_faces, const int32_t *faces, void *incidence, size_t incidence_bytes, void *stream);
/* normals [n_frames, n_verts, 3] of vertices [n_frames, n_verts, 3]: the sum of the unnormalised face normals
 * cross(v1 - v0, v2 - v0) in the incidence order, (0, 0, 1) where its dot is not > 1e-20, then safe_normalize.  faces
 * and incidence must be the ones b200gs_mesh_incidence was given and wrote. */
int b200gs_mesh_vertex_normals(int32_t n_frames, int32_t n_verts, int32_t n_faces, const float *vertices, const int32_t *faces,
                               const void *incidence, size_t incidence_bytes, float *normals, void *stream);
/* The reference's normal image: out [n_views, height, width, 3] = (safe_normalize(interpolated normals) + 1) / 2 where rast
 * holds a triangle (as b200gs_mesh_interpolate decides), 1.0 elsewhere.  normals as attr above with channels = 3. */
int b200gs_mesh_normal_image(int32_t n_views, int32_t height, int32_t width, int32_t n_verts, int32_t n_faces, const float *normals,
                             int32_t normals_per_view, const float *rast, const int32_t *tri, float *out, void *stream);

/* ---- mesh cleanup and decimation (humangaussian_b200/mesh.py clean_mesh / decimate_mesh; DESIGN.md section 2) ------
 * Both take a mesh vertices [n_verts,3] float32, faces [n_faces,3] int32 (device, 4-byte aligned) and write the result
 * to out_vertices / out_faces, which hold at least n_verts and n_faces rows; counts (HOST int64 [2]) receives the output's
 * vertex and face counts and rounds (HOST) the number of rounds.  Surviving vertices and faces keep their relative order.
 * Unlike the other calls these wait on the host: after a check that every face index lies in [0, n_verts) (a face
 * outside is B200GS_E_ARGS, and nothing reads through it), once per round, and once for the counts.  scratch: the
 * *_scratch_bytes query, 16-byte aligned.  n_verts < 2^31 - 1 and n_faces < 2^24, else B200GS_E_RANGE.
 * b200gs_mesh_clean: drops faces that repeat an index or an earlier face's vertex set, then every connected component
 *   (faces sharing a vertex) with fewer than min_faces faces or a bounding-box diagonal below min_diameter times the
 *   whole mesh's, then unreferenced vertices.  Vertex bytes are unchanged.  rounds: labelling rounds.
 * b200gs_mesh_decimate: quadric edge collapse in parallel rounds to at most `target` faces (target >= 4, else
 *   B200GS_E_ARGS); it stops early, above target, when a round finds no valid collapse.  Boundary and non-manifold
 *   vertices stay.  rounds: rounds that collapsed at least one edge. */
size_t b200gs_mesh_clean_scratch_bytes(int32_t n_verts, int32_t n_faces);
int b200gs_mesh_clean(int32_t n_verts, int32_t n_faces, const float *vertices, const int32_t *faces, int32_t min_faces, double min_diameter,
                      void *scratch, size_t scratch_bytes, float *out_vertices, int32_t *out_faces, int64_t *counts, int32_t *rounds,
                      void *stream);
size_t b200gs_mesh_decimate_scratch_bytes(int32_t n_verts, int32_t n_faces);
int b200gs_mesh_decimate(int32_t n_verts, int32_t n_faces, const float *vertices, const int32_t *faces, int32_t target, void *scratch,
                         size_t scratch_bytes, float *out_vertices, int32_t *out_faces, int64_t *counts, int32_t *rounds, void *stream);

/* ---- per-stage device timing (CUDA events recorded on the launch stream around each stage) -----------------
 * enable, run any number of forward/backward calls, then read: accumulated milliseconds and call counts per stage
 * since the last read.  b200gs_profile_read synchronises on the recorded events. */
enum { B200GS_STAGE_PREPROCESS = 0, B200GS_STAGE_SCAN = 1, B200GS_STAGE_BINNING = 2, B200GS_STAGE_BLEND_FWD = 3,
       B200GS_STAGE_BLEND_BWD = 4, B200GS_STAGE_PREPROCESS_BWD = 5, B200GS_STAGE_COUNT = 6 };
void b200gs_profile_enable(int on);
int b200gs_profile_read(double *ms_per_stage /* host [B200GS_STAGE_COUNT] */, int64_t *calls_per_stage /* host */, int32_t n_stages);

const char *b200gs_last_cuda_error(void);
int b200gs_abi_version(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
int64_t b200gs_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200GS_H */
