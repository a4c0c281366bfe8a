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

void launch_preprocess_fwd(const PreArgs &a, int V, cudaStream_t st);
void launch_preprocess_bwd(const PreBwdArgs &a, cudaStream_t st);
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

void launch_blend_fwd(const BlendArgs &a, cudaStream_t st);
void launch_blend_bwd(const BlendBwdArgs &a, cudaStream_t st);
int blend_sgrad_is_moments(); // which ScreenGrad format the linked blend_bwd writes

// ---- deterministic backward (deterministic.cu; B1's deterministic instantiation in blend.cu) ------------------------------
// Every (sorted instance j, patch p) that B1 flushes gets its own partial slot; the reduce adds a Gaussian's partials in
// emission order (the tiles of its rect row-major), patches ascending, so the sums depend on the forward state only.
#define DET_PARTIAL_FLOATS 10 // S0, Sx, Sy, Sxx, Sxy, Syy, W0..W3: 40 bytes
struct DetFlush {
    const uint8_t *pm;    // [D] bit p: B1 flushes a partial for (j, patch p)
    const uint32_t *base; // [D] inclusive scan of popc(pm) (exact: the total is checked to fit 32 bits)
    float *partials;      // [H][DET_PARTIAL_FLOATS]
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
int blend_bwd_has_deterministic(); // 0 in the classic comparator
void launch_blend_bwd_det(const BlendBwdArgs &a, const DetFlush &det, cudaStream_t st);
// start scatter, plan, scan of popc(pm) -> base and the exact 64-bit partial count at *total_dev
int launch_det_plan(const DetPlanArgs &a, int64_t n_vp, int n_tiles_all, const DetLayout &L, char *det_base, cudaStream_t st,
                    int *n_launches);
void launch_det_reduce(const DetPlanArgs &a, int64_t n_vp, const float *partials, void *sgrad, cudaStream_t st);
void launch_test_exp(const float *x, float *y, int64_t n, cudaStream_t st);

// animation frame path (anim.cu)
void launch_reattach(int P, int n_frames, int n_verts, int n_faces, const float *vertices, const int32_t *faces, const int32_t *map_face,
                     const float *map_uvw, const float *map_dist, float *xyz, cudaStream_t st);
void launch_pack_u8(const float *color, uint8_t *out, int H, int W, int n_frames, cudaStream_t st);

// 3-nearest-neighbour mean squared distance (knn.cu)
size_t knn_scratch_bytes(int P);
int launch_knn3(int P, const float *pts, float *mean_d2, char *scratch, size_t scratch_bytes, cudaStream_t st, int *n_launches);

// densify / prune (densify.cu)
struct DensifyCfg {
    int mode;            // 0 = densify_and_prune, 1 = prune_only
    int n_split;         // children per split parent (reference: 2)
    int use_screen;      // reference's `if max_screen_size:` branch
    float max_grad, min_opacity;
    float dense_thresh;  // percent_dense * extent
    float max_screen_size;
    float big_ws_thresh; // 0.1 * extent (mode 0) or size_thresh (mode 1)
};
size_t densify_scratch_bytes(int P);
void launch_densify_stats(int P, int V, const float *grads, const int32_t *radii, const uint8_t *update_mask, float *accum, float *denom,
                          float *max_radii2D, cudaStream_t st);
void launch_densify_plan(const DensifyCfg &c, int P, const float *accum, const float *denom, const float *opacity, const float *scaling,
                         int *plan, int *counts, char *scratch, cudaStream_t st);
void launch_densify_move(int role, int P, int rf, const int *plan, const float *src, float *dst, int n_split, int S_sel, int S_kept,
                         const float *rotation, const float *scaling, const float *noise, cudaStream_t st);

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
