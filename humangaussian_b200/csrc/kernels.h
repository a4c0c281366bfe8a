// kernels.h -- argument blocks and launchers shared by the translation units of libb200gs.
#pragma once
#include "common.cuh"

struct PreArgs {
    int vec16;               // rotations and shs are 16-byte aligned: 128-bit loads allowed
    int raw;                 // scales / rotations / opacities are the RAW parameters: exp / normalize / sigmoid applied here
    int P, deg, M, H, W, grid_x, grid_y;
    size_t means_view_stride; // 0: means shared by all views; 3*P: per-view positions
    float mod;
    const float *means, *shs, *colors_pre, *opac, *scales, *rots, *cov_pre;
    const float *view, *proj, *campos; // [V,16] [V,16] [V,3]
    float tanfovx[GS_MAX_VIEWS], tanfovy[GS_MAX_VIEWS];
    // outputs
    int32_t *radii;          // [V,P]
    GeomRec *recs;           // [V*P]
    uint32_t *tiles_touched; // [V*P]
    uint2 *rects;            // [V*P]
    uint8_t *clamped;        // [V*P]
    uint32_t *dkeys;         // [V*P] depth bits (input of the depth pre-sort; the view rides in the tile key)
    uint32_t *order_in;      // [V*P] = vp
};

struct PreBwdArgs {
    int vec16;               // dL_drots is 16-byte aligned: 128-bit store allowed
    int raw;                 // as PreArgs: gradients are then w.r.t. the raw parameters (activation Jacobians applied)
    int P, V, deg, M, H, W;
    size_t means_view_stride; // as PreArgs; when non-zero dL_dmeans3D is [V,P,3] (per view, not summed)
    float mod;
    const float *means, *shs, *colors_pre, *scales, *rots, *cov_pre, *opac;
    const float *view, *proj, *campos;
    float tanfovx[GS_MAX_VIEWS], tanfovy[GS_MAX_VIEWS];
    const int32_t *radii;
    const uint8_t *clamped;
    const void *sgrad;       // [V*P] ScreenGrad (48 B of floats), see `moments`
    const GeomRec *recs;     // [V*P] forward records (conic, opacity) -- used when sgrad holds moments
    int moments;             // 0: classic float (dx,dy,dA,dBh,dC,dO,dr,dg,db,dd); 1: float moments (S0,Sx,Sy,Sxx,Sxy,Syy,cr,cg,cb,cd)
    float *dL_dmeans3D, *dL_dmeans2D, *dL_dsh, *dL_dcolors, *dL_dopacity, *dL_dscales, *dL_drots, *dL_dcov3D;
    const float *f3d_var;    // [P] 3D filter variances, read by the F3D instantiations (last: the others' layout stays)
};

struct BlendArgs {
    int H, W, grid_x, grid_y, V, P;
    const uint32_t *tile_order; // [V*tiles] (view*tiles + tile) sorted by descending list length: longest first
    const uint2 *ranges;        // [V*tiles]
    const uint32_t *point_list; // [D] index into recs (= v*P + gaussian)
    const GeomRec *recs;        // [V*P]
    const float *bg;            // [3]
    float *final_T;             // [V,H,W]
    uint32_t *n_contrib;        // [V,H,W]
    float *out_color, *out_depth, *out_alpha;
    uint32_t *cmask;            // contributor masks, one word per (32-entry chunk, patch): see BinLayout::cmask
};

struct BlendBwdArgs {
    int H, W, grid_x, grid_y, V, P;
    const uint32_t *tile_order;
    const uint2 *ranges;
    const uint32_t *point_list;
    const GeomRec *recs;
    const float *bg;
    const float *final_T;
    const uint32_t *n_contrib;
    const float *dL_dcolor, *dL_ddepth, *dL_dalpha; // may be null
    const uint32_t *cmask;                          // the forward's contributor masks
    void *sgrad;                                    // [V*P] accumulators (format: blend_sgrad_is_moments()), zeroed by the caller
};

// aa: the antialiasing filter (record opacity op * rho; DESIGN.md section 2).  f3d / f3d_var (NULL = off): the 3D smoothing
// filter (scales widened by the [P] variances, opacity compensated; DESIGN.md section 2)
void launch_preprocess_fwd(const PreArgs &a, int V, bool aa, const float *f3d_var, cudaStream_t st);
void launch_preprocess_bwd(const PreBwdArgs &a, bool aa, bool f3d, cudaStream_t st);
// per-Gaussian maximal sampling rate over n_views <= GS_MAX_VIEWS cameras, folded into max_rate by max (filter3d.cu)
struct RateArgs {
    int P, nviews, H, W;
    const float *means, *view; // [P,3], [nviews,16]
    float tanfovx[GS_MAX_VIEWS], tanfovy[GS_MAX_VIEWS];
    float *max_rate;           // [P] in/out
};
void launch_sampling_rate(const RateArgs &a, cudaStream_t st);
void launch_mark_visible(int P, const float *pos, const float *V, uint8_t *present, cudaStream_t st);

// binning: depth pre-sort of the V*P Gaussians, scan in depth order, tile-key emission, stable tile sort, ranges
struct BinLayout {
    size_t keys_in, keys_out, vals_in, vals_out, ranges; // per-instance tile keys (u32) / record indices (u32), tile ranges
    size_t dkeys_in, dkeys_out, order_in, order;         // per-Gaussian depth keys (u32) and the depth order (u32)
    size_t tile_order, tile_order_cnt;                   // launch order of the tiles (longest list first) + 32 bucket counters
    size_t total_slot;                                   // u64: exact instance count of the batch (written by the tile scan)
    // u32 contributor masks written by the forward blend and read by the backward blend: word
    // ((range.x >> 5) + vt + c) * 8 + patch belongs to chunk c (list positions [32c, 32c+32) of tile vt) and patch 0..7;
    // bit l = entry 32c+l contributed to at least one pixel of the patch.  Tiles' ranges are laid out in vt order, so
    // (range.x >> 5) + c <= (range.y >> 5) keeps the tiles' words apart; range.y <= capacity bounds the index.
    size_t cmask;
    size_t temp, total;
    size_t temp_bytes;
};
BinLayout binning_layout(int64_t capacity, int ntiles_total, int64_t n_vp);
int launch_depth_order(const uint32_t *tiles_touched, uint32_t *offsets_sorted, int64_t n_vp, int V, char *bin_base,
                       const BinLayout &L, const uint32_t **order_sorted, const uint64_t **total_dev, cudaStream_t st, int *n_launches);
#define B200GS_MAX_INSTANCES_I64 ((int64_t)0x7fffffff) // (Gaussian, tile) instances per call: 32-bit indices with headroom
int launch_binning(const uint32_t *order_sorted, const uint2 *rects, const uint32_t *offsets_sorted, int P, int V, int grid_x, int grid_y,
                   int64_t D, const uint64_t *D_dev, char *bin_base, const BinLayout &L, cudaStream_t st, int *n_launches);
int launch_test_sort32(uint32_t *ka, uint32_t *kb, uint32_t *va, uint32_t *vb, int64_t n, int nbits, char *scratch, size_t scratch_bytes,
                       int *result_in_b, cudaStream_t st);
size_t test_sort32_scratch_bytes(int64_t n);

// the optional features of the blend a build implements (blend_caps): all in blend.cu; the classic comparator has none.  The
// host checks them before any launch.
enum { BLEND_CAP_CONTRIB = 1, BLEND_CAP_NORMALS = 2, BLEND_CAP_GEOMETRY = 4, BLEND_CAP_ABSGRAD = 8,
       BLEND_CAP_DETERMINISTIC = 16 };
int blend_caps();
// contribution scores (DESIGN.md section 2): per Gaussian [P], in/out, folded over every pixel of every view of the launch
struct ContribOut {
    uint64_t *weight_sum; // sum of q(w) = rn(w * 2^24) over the blends
    uint32_t *weight_max; // max of the bits of w over the blends
    uint32_t *touches;    // blends plus terminating hits
};
int blend_sgrad_is_moments(); // which ScreenGrad format the linked blend_bwd writes

// ---- deterministic backward (deterministic.cu; B1's deterministic instantiation in blend.cu) ------------------------------
// Every (sorted instance j, patch p) that B1 flushes gets its own partial slot; the reduce adds a Gaussian's partials in
// emission order (the tiles of its rect row-major), patches ascending, so the sums depend on the forward state only.
#define DET_PARTIAL_FLOATS 10 // S0, Sx, Sy, Sxx, Sxy, Syy, W0..W3: 40 bytes
struct DetFlush {
    const uint8_t *pm;    // [D] bit p: B1 flushes a partial for (j, patch p)
    const uint32_t *base; // [D] inclusive scan of popc(pm) (exact: the total is checked to fit 32 bits)
    float *partials;      // [H][DET_PARTIAL_FLOATS]
    float2 *abs_partials; // [H] (Ax, Ay) of each partial: written by the absgrad instantiation only
};
// det_buf carving; pm first (b200gs.h documents that the buffer starts with it)
struct DetLayout {
    size_t pm, base, jpos, start, scan_temp, total_slot, partials, total;
    __host__ DetLayout(int64_t D, int64_t partial_capacity, int64_t n_vp);
};
struct DetPlanArgs {
    int H, W, grid_x, grid_y;
    int64_t D;
    const uint32_t *tile_order; // [V*tiles]: the plan kernel runs one CTA per (view, tile), longest list first
    const uint2 *ranges;
    const uint32_t *point_list, *cmask, *n_contrib;
    const uint2 *rects;         // [V*P] tile rect of each record (preprocess)
    const uint32_t *order, *offsets, *tiles_touched; // depth order, inclusive scan of tiles_touched in it, tiles_touched
    uint32_t *start;            // [V*P] emission start of each record
    uint8_t *pm;
    uint32_t *base, *jpos;      // [D], [D]: jpos[emission index] = sorted position
};
// inclusive scan of popc(pm[j]) over n instances (the binning stage's look-back scan, binning.cu): incl[j] keeps the low 32
// bits, *total the exact sum; temp (popc_scan_temp_bytes) is zeroed by the call
size_t popc_scan_temp_bytes(int64_t n);
int launch_popc_scan(const uint8_t *pm, uint32_t *incl, int64_t n, char *temp, uint64_t *total, cudaStream_t st);
// start scatter, plan, scan of popc(pm) -> base and the exact 64-bit partial count at *total_dev
int launch_det_plan(const DetPlanArgs &a, int64_t n_vp, int n_tiles_all, const DetLayout &L, char *det_base, cudaStream_t st,
                    int *n_launches);
// abs_partials (NULL: none): their (Ax, Ay) are added in the same order into ScreenGrad's padding, which is zero without them.
// nrm_partials (NULL: none): their normal sums are added in the same order and written to wn[vp]
void launch_det_reduce(const DetPlanArgs &a, int64_t n_vp, const float *partials, const float2 *abs_partials, void *sgrad,
                       const float4 *nrm_partials, float4 *wn, cudaStream_t st);
// absolute screen-space gradients (DESIGN.md section 2): B1 writes Ax, Ay into ScreenGrad's padding, and this pass writes
// dL_dmeans2D_abs [V,P,3] from them
void launch_absgrad_out(int64_t n_vp, int H, int W, const int32_t *radii, const GeomRec *recs, const void *sgrad, float *out,
                        cudaStream_t st);
void launch_test_exp(const float *x, float *y, int64_t n, cudaStream_t st);

// ---- normal maps (DESIGN.md section 2; normals.cu, and the NRM instantiations of the blend kernels) -----------------------
struct NormalArgs {
    int P, V, raw;
    size_t means_view_stride;                       // as PreArgs
    const float *means, *scales, *rots, *campos;    // [P,3] or [V,P,3], [P,3], [P,4], [V,3]
};
// gauss_normals [V*P]: (sign n, sign) of every (view, Gaussian), n the axis of its smallest activated scale
void launch_normal_prep(const NormalArgs &a, float4 *gauss_normals, cudaStream_t st);
// dL_drots[i] += dL/dq of sum over the views with radii > 0 of sign * wn[v*P + i]
void launch_normal_bwd(const NormalArgs &a, const int32_t *radii, const float4 *gauss_normals, const float4 *wn, float *dL_drots,
                       cudaStream_t st);
struct NrmBwd {
    const float4 *gauss_normals; // [V*P]
    const float *dL_dnormal;     // [V,3,H,W]
    float4 *wn;                  // [V*P] atomic mode: sum w * dL/dN of every (view, Gaussian), zeroed by the caller
    float4 *partials;            // [H] deterministic mode: each partial's three sums, at its slot
};
// ---- geometry outputs (DESIGN.md section 2; the GEO instantiations of the blend kernels) ---------------------------------
struct GeoFwd {
    float *out_median;    // [V,1,H,W] depth of the last blend with T > 0.5 before it (0: none)
    float *out_depth2;    // [V,1,H,W] M2 = sum w d^2
    uint32_t *median_pos; // [V,H,W] 1-based list position of that blend (0: none); read by the backward
};
struct GeoBwd {
    const float *dL_dmedian;      // [V,1,H,W] or NULL (zero)
    const float *dL_ddepth2;      // [V,1,H,W] or NULL (zero)
    const uint32_t *median_pos;   // [V,H,W] the forward's
};

// F6.  Each feature is off when NULL: co the contribution scores (never with the other two); gauss_normals the normal image
// out_normal [V,3,H,W] = sum w * n; g the geometry outputs.  A build without a feature (blend_caps) ignores its argument.
void launch_blend_fwd(const BlendArgs &a, const ContribOut *co, const float4 *gauss_normals, float *out_normal, const GeoFwd *g,
                      cudaStream_t st);
// B1: atomic (det NULL) or deterministic, with or without the absolute sums (Ax, Ay in ScreenGrad's padding), the normal term
// (n) and the geometry gradients folded into W3 (g); NULL = off.  The deterministic reduce does not depend on geometry.
void launch_blend_bwd(const BlendBwdArgs &a, const DetFlush *det, bool absgrad, const NrmBwd *n, const GeoBwd *g, cudaStream_t st);

// animation frame path (anim.cu)
void launch_reattach(int P, int n_frames, int n_verts, int n_faces, const float *vertices, const int32_t *faces, const int32_t *map_face,
                     const float *map_uvw, const float *map_dist, float *xyz, cudaStream_t st);
void launch_pack_u8(const float *color, uint8_t *out, int H, int W, int n_frames, cudaStream_t st);

// 3-nearest-neighbour mean squared distance (knn.cu)
size_t knn_scratch_bytes(int P);
int launch_knn3(int P, const float *pts, float *mean_d2, char *scratch, size_t scratch_bytes, cudaStream_t st, int *n_launches);

// densify / prune (densify.cu)
struct DensifyCfg {
    int mode;            // 0 = densify_and_prune, 1 = prune_only, 2 = prune by mask (keep = !remove[i])
    int n_split;         // children per split parent (reference: 2)
    int use_screen;      // reference's `if max_screen_size:` branch
    float max_grad, min_opacity;
    float dense_thresh;  // percent_dense * extent
    float max_screen_size;
    float big_ws_thresh; // 0.1 * extent (mode 0) or size_thresh (mode 1)
    const uint8_t *remove; // [P], mode 2
};
size_t densify_scratch_bytes(int P);
void launch_densify_stats(int P, int V, const float *grads, const int32_t *radii, const uint8_t *update_mask, float *accum, float *denom,
                          float *max_radii2D, cudaStream_t st);
void launch_densify_plan(const DensifyCfg &c, int P, const float *accum, const float *denom, const float *opacity, const float *scaling,
                         int *plan, int *counts, char *scratch, cudaStream_t st);
void launch_densify_move(int role, int P, int rf, const int *plan, const float *src, float *dst, int n_split, int S_sel, int S_kept,
                         const float *rotation, const float *scaling, const float *noise, cudaStream_t st);

// MCMC densification (mcmc.cu; DESIGN.md section 2).  Raw parameters; counts [P] = times each row was drawn as a source.
// xyz [P,3] += the opacity-gated position noise of the eta [P,3] draws
void launch_mcmc_noise(int P, float *xyz, const float *scaling, const float *rotation, const float *opacity, const float *eta,
                       float noise_scale, float k, float t, cudaStream_t st);
// rows with counts > 0: new_opacity [P] / new_scaling [P,3] = the split ratio's raw values (other rows are not written)
void launch_mcmc_ratio(int P, const int *counts, const float *opacity, const float *scaling, float *new_opacity, float *new_scaling,
                       cudaStream_t st);
// dst[i] = src[map[i]] for i < P_new (role B200GS_MCMC_ROLE_*: reset rows take the ratio's values or zero moments)
void launch_mcmc_move(int role, int P_new, int rf, const int *map, const int *counts, const float *src, float *dst,
                      const float *new_opacity, const float *new_scaling, cudaStream_t st);

// Adam over the packed buffer (optim.cu).  Groups in the reference's order (gaussian_model.py:156-163).
enum { ADAM_GROUP_XYZ = 0, ADAM_GROUP_F_DC = 1, ADAM_GROUP_F_REST = 2, ADAM_GROUP_OPACITY = 3, ADAM_GROUP_SCALING = 4,
       ADAM_GROUP_ROTATION = 5 };
struct AdamArgs {
    int64_t off[5];      // field offsets (floats) in buffer order xyz, scaling, rotation, opacity, sh; ascending, multiples of 4
    int64_t numel[5];    // 3P, 3P, 4P, P, 3*sh_coeffs*P
    int field_group[5];  // group of each field (the sh field's is chosen per element: f_dc or f_rest)
    int sh_coeffs;
    int lerp_small;      // |1-beta1| < 0.5: the branch ATen's lerp() takes
    float step_size[6];  // -(lr_g / bias_correction1), by group
    float bias_correction2_sqrt, one_minus_beta1, beta2, one_minus_beta2, eps;
};
void launch_adam_packed(const AdamArgs &a, int64_t total, float *params, const float *grads, float *exp_avg, float *exp_avg_sq,
                        cudaStream_t st);

// mesh export (mesh.cu): density field over blocks of `split` samples per axis, and marching cubes.  Nonzero return:
// scratch too small (-1) or a failed launch setup (-2).
size_t density_field_scratch_bytes(int P, int res, int split);
int launch_density_field(int P, const float *means, const float *cov6, const float *opac, int res, int split, const float *samples,
                         float relax, float *field, char *scratch, size_t scratch_bytes, cudaStream_t st, int *n_launches);
// field query at n_points points of the field's frame (sh_degree 0-3; colours only when both shs and colors are given)
size_t field_query_scratch_bytes(int P, int n_points, int res, int split, int sh_degree);
int launch_field_query(int P, const float *means, const float *cov6, const float *opac, const float *shs, int sh_coeffs, int sh_degree,
                       int res, int split, const float *samples, float relax, int n_points, const float *points, float *density,
                       float *normals, float *colors, char *scratch, size_t scratch_bytes, cudaStream_t st, int *n_launches);
size_t marching_cubes_scratch_bytes(int X, int Y, int Z);
int launch_marching_cubes_count(int X, int Y, int Z, const float *vol, float iso, char *scratch, size_t scratch_bytes, uint64_t *counts,
                                cudaStream_t st, int *n_launches);
int launch_marching_cubes_emit(int X, int Y, int Z, const float *vol, float iso, const char *scratch, size_t scratch_bytes, float *verts,
                               int32_t *faces, cudaStream_t st, int *n_launches);

// pose maps (pose.cu): style 0 HumanSD (17 keypoints, 16 limbs), 1 OpenPose (18 keypoints, 18 circles + 17 limbs)
struct PoseArgs {
    int style, V, H, W;
    const float *points;       // [K,4]
    const float *mvp;          // [V,4,4] row-major
    const uint8_t *occlusion;  // [V]
    float *kp;                 // [V,K,2] out
    int2 *hulls;               // scratch [V][S][H][4]: each shape's disjoint runs [lo, hi] per row (empty: lo > hi)
    int2 *polys;               // scratch [V][17][361]: OpenPose ellipse polygons
    float *out;                // [V,H,W,3]
    int8_t limbs[17][2];       // keypoint pairs in draw order
    uint8_t colors[35][3];     // per shape in draw order (OpenPose: the 18 circles, then the 17 limbs)
};
int pose_shapes(int style);
int pose_limbs(int style);
int pose_keypoints(int style);
size_t pose_scratch_bytes(int style, int V, int H);
void pose_layout(PoseArgs &a, char *scratch);
void launch_pose_setup(const PoseArgs &a, cudaStream_t st);
void launch_pose_draw(const PoseArgs &a, cudaStream_t st);

// mesh rendering (meshraster.cu).  Rasterisation: count (setup, per-tile counts, scan; the exact pair total lands at *count)
// then emit from the same scratch.  Nonzero return: a failed memset.
size_t mesh_raster_scratch_bytes(int V, int Nf, int H, int W);
int launch_mesh_raster_count(int V, int Nv, int Nf, int H, int W, const float *pos, const int *tri, char *scratch, uint64_t *count,
                             cudaStream_t st, int *n_launches);
int launch_mesh_raster_emit(int V, int Nf, int H, int W, char *scratch, int *pairs, uint64_t cap, float *rast, cudaStream_t st,
                            int *n_launches);
void launch_mesh_interpolate(int V, int H, int W, int Nv, int Nf, int C, const float *attr, int per_view, const float *rast, const int *tri,
                             float *out, cudaStream_t st);
void launch_mesh_normal_image(int V, int H, int W, int Nv, int Nf, const float *vn, int per_view, const float *rast, const int *tri,
                              float *out, cudaStream_t st);
// per-vertex incidence lists in (corner, face) order; the vertex normals read the buffer the incidence call wrote
size_t mesh_incidence_bytes(int Nv, int Nf);
int launch_mesh_incidence(int Nv, int Nf, const int *faces, char *buf, size_t bytes, cudaStream_t st, int *n_launches);
void launch_mesh_vertex_normals(int F, int Nv, int Nf, const float *verts, const int *faces, const char *incidence, float *out,
                                cudaStream_t st);
// the start [Nv + 1] and list arrays inside an incidence buffer of (Nv, Nf)
void mesh_incidence_lists(int Nv, int Nf, const char *buf, const uint32_t **start, const uint32_t **list);

// mesh cleanup and decimation (meshclean.cu).  Both wait on the host (clean: once per labelling round and once for the
// counts; decimate: once for the index check, once per round and once for the counts).  counts = vertices, faces.
// Nonzero return: -1 a CUDA call failed, -2 a face index outside [0, Nv), -3 (decimate) an internal face-count mismatch
size_t mesh_clean_scratch_bytes(int Nv, int Nf);
int launch_mesh_clean(int Nv, int Nf, const float *verts, const int *faces, int min_faces, double min_diameter, char *scratch,
                      float *out_verts, int *out_faces, int64_t *counts, int *rounds, cudaStream_t st, int *n_launches);
size_t mesh_decimate_scratch_bytes(int Nv, int Nf);
int launch_mesh_decimate(int Nv, int Nf, const float *verts, const int *faces, int target, char *scratch, float *out_verts,
                         int *out_faces, int64_t *counts, int *rounds, cudaStream_t st, int *n_launches);
