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

#define B200GS_ABI_VERSION 4
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
