// api.cu -- the C-ABI of libb200gs (include/b200gs.h): argument validation, state-buffer carving,
// kernel sequencing.  No torch types, no global state except an error string and a launch counter.
#include <atomic>
#include <cstdio>
#include <cstring>

#include "../../include/b200gs.h"
#include "common.cuh"
#include "kernels.h"

static thread_local char g_err[256] = "";
static std::atomic<int64_t> g_launches{0};

// ---- optional per-stage CUDA-event timing (bench.py's roofline numbers; events sit on the launch stream) ----
#include <mutex>
#include <vector>
struct StageSpan { int stage; cudaEvent_t e0, e1; };
static std::mutex g_prof_mu;
static bool g_prof_on = false;
static std::vector<StageSpan> g_spans;
static std::vector<cudaEvent_t> g_event_pool;
static cudaEvent_t prof_event()
{
    if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
}
struct StageTimer {
    bool on; StageSpan sp; cudaStream_t st;
    StageTimer(int stage, cudaStream_t s) : on(g_prof_on), st(s)
    {
        if (!on) return;
        std::lock_guard<std::mutex> lk(g_prof_mu);
        sp.stage = stage; sp.e0 = prof_event(); sp.e1 = prof_event();
        cudaEventRecord(sp.e0, st);
    }
    ~StageTimer()
    {
        if (!on) return;
        cudaEventRecord(sp.e1, st);
        std::lock_guard<std::mutex> lk(g_prof_mu);
        g_spans.push_back(sp);
    }
};

#define B200GS_DEFERRED_MAX_NVP ((int64_t)4 << 20) // (view, Gaussian) pairs up to which the forward does not wait for its instance count
// one pinned 8-byte word + event per (host thread, device): where the forward's instance count lands without a host wait
struct HostSlot { unsigned long long *total; cudaEvent_t ev; };
static HostSlot *host_slot()
{
    static thread_local HostSlot slots[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    HostSlot &s = slots[dev];
    if (!s.total) {
        if (cudaHostAlloc((void **)&s.total, 8, cudaHostAllocDefault) != cudaSuccess) { s.total = nullptr; return nullptr; }
        if (cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming) != cudaSuccess) { cudaFreeHost(s.total); s.total = nullptr; return nullptr; }
    }
    return &s;
}

static int cuda_fail(cudaError_t e, const char *where)
{
    snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
    return B200GS_E_CUDA;
}
#define CK(call, where)                                  \
    do {                                                 \
        cudaError_t e__ = (call);                        \
        if (e__ != cudaSuccess) return cuda_fail(e__, where); \
    } while (0)

extern "C" {

const char *b200gs_last_cuda_error(void) { return g_err; }
int b200gs_abi_version(void) { return B200GS_ABI_VERSION; }
int64_t b200gs_launch_count(void) { return g_launches.load(); }

size_t b200gs_geom_bytes(int32_t P, int32_t V) { return GeomLayout(P, V).total; }
size_t b200gs_image_bytes(int32_t H, int32_t W, int32_t V) { return ImageLayout(H, W, V).total; }
size_t b200gs_binning_bytes(int64_t cap, int32_t H, int32_t W, int32_t P, int32_t V)
{
    const int gx = (W + GS_TILE - 1) / GS_TILE, gy = (H + GS_TILE - 1) / GS_TILE;
    return binning_layout(cap, gx * gy * V, (int64_t)P * V).total;
}
size_t b200gs_backward_scratch_bytes(int32_t P, int32_t V) { return gs_align((size_t)P * V * sizeof(ScreenGrad)); }

static int check_common(const b200gs_params *p, const float *shs, const float *colors, const float *scales,
                        const float *rots, const float *cov)
{
    if (!p || p->abi_version != B200GS_ABI_VERSION) return B200GS_E_ARGS;
    if (p->P < 0 || p->n_views < 1 || p->image_height < 1 || p->image_width < 1 || !p->tanfovx || !p->tanfovy) return B200GS_E_ARGS;
    if ((shs == nullptr) == (colors == nullptr)) return B200GS_E_ARGS;
    if (((scales == nullptr) || (rots == nullptr)) == (cov == nullptr)) return B200GS_E_ARGS;
    if ((scales == nullptr) != (rots == nullptr)) return B200GS_E_ARGS;
    if (p->n_views > B200GS_MAX_VIEWS) return B200GS_E_RANGE;
    if (shs && (p->sh_degree < 0 || p->sh_degree > 3 || p->sh_coeffs < (p->sh_degree + 1) * (p->sh_degree + 1))) return B200GS_E_RANGE;
    if ((int64_t)p->P * p->n_views >= ((int64_t)1 << 32)) return B200GS_E_RANGE;
    if ((p->image_width + GS_TILE - 1) / GS_TILE > 65535 || (p->image_height + GS_TILE - 1) / GS_TILE > 65535) return B200GS_E_RANGE;
    return B200GS_OK;
}

int b200gs_forward(const b200gs_params *prm, const float *means3D, const float *shs, const float *colors_precomp,
                   const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp,
                   const float *bg, const float *viewmatrix, const float *projmatrix, const float *campos,
                   float *out_color, float *out_depth, float *out_alpha, int32_t *radii, void *geom_buf, size_t geom_bytes,
                   void *binning_buf, size_t binning_bytes, int64_t instance_capacity, void *image_buf, size_t image_bytes,
                   int64_t *num_rendered, void *stream)
{
    int rc = check_common(prm, shs, colors_precomp, scales, rotations, cov3D_precomp);
    if (rc) return rc;
    if (!means3D || !opacities || !bg || !viewmatrix || !projmatrix || !campos || !out_color || !out_depth || !out_alpha ||
        !radii || !geom_buf || !binning_buf || !image_buf || !num_rendered)
        return B200GS_E_ARGS;
    cudaStream_t st = (cudaStream_t)stream;
    const int P = prm->P, V = prm->n_views, H = prm->image_height, W = prm->image_width;
    const int gx = (W + GS_TILE - 1) / GS_TILE, gy = (H + GS_TILE - 1) / GS_TILE;
    const GeomLayout GL(P, V);
    const ImageLayout IL(H, W, V);
    const BinLayout BL = binning_layout(instance_capacity, gx * gy * V, (int64_t)P * V);
    if (geom_bytes < GL.total || image_bytes < IL.total || binning_bytes < BL.total) return B200GS_E_BUFFER;
    if ((((uintptr_t)geom_buf) | ((uintptr_t)binning_buf) | ((uintptr_t)image_buf)) & 15) return B200GS_E_BUFFER; // records are 128-bit accessed
    char *gb = (char *)geom_buf, *bb = (char *)binning_buf, *ib = (char *)image_buf;
    const size_t HW = (size_t)H * W;
    *num_rendered = 0;
    HostSlot *pending = nullptr;

    if (P == 0) { // empty scene: background only
        CK(cudaMemsetAsync(bb + BL.ranges, 0, (size_t)gx * gy * V * 8, st), "memset ranges");
        int nl0 = 0;
        if (launch_binning(nullptr, nullptr, nullptr, 0, V, gx, gy, 0, nullptr, bb, BL, st, &nl0)) return cuda_fail(cudaGetLastError(), "binning");
    } else {
        PreArgs a;
        a.P = P; a.deg = shs ? prm->sh_degree : 0; a.M = prm->sh_coeffs; a.H = H; a.W = W; a.grid_x = gx; a.grid_y = gy;
        a.vec16 = ((((uintptr_t)rotations) | ((uintptr_t)shs)) & 15) == 0; // any 4-byte-aligned float pointer is accepted
        a.raw = prm->raw_params != 0;
        a.mod = prm->scale_modifier;
        a.means_view_stride = prm->means3D_per_view ? (size_t)3 * P : 0;
        a.means = means3D; a.shs = shs; a.colors_pre = colors_precomp; a.opac = opacities; a.scales = scales;
        a.rots = rotations; a.cov_pre = cov3D_precomp; a.view = viewmatrix; a.proj = projmatrix; a.campos = campos;
        for (int v = 0; v < V; v++) { a.tanfovx[v] = prm->tanfovx[v]; a.tanfovy[v] = prm->tanfovy[v]; }
        a.radii = radii; a.recs = (GeomRec *)(gb + GL.recs); a.tiles_touched = (uint32_t *)(gb + GL.tiles_touched);
        a.rects = (uint2 *)(gb + GL.rects); a.clamped = (uint8_t *)(gb + GL.clamped);
        a.dkeys = (uint32_t *)(bb + BL.dkeys_in); a.order_in = (uint32_t *)(bb + BL.order_in);
        { StageTimer t(B200GS_STAGE_PREPROCESS, st); launch_preprocess_fwd(a, V, st); }
        g_launches += 1;
        uint32_t *offsets = (uint32_t *)(gb + GL.offsets); // inclusive scan of tiles_touched in DEPTH order
        const int64_t n_vp = (int64_t)P * V;
        const uint32_t *order_sorted = nullptr;
        const uint64_t *total_dev = nullptr;
        int nl = 0;
        {
            StageTimer t(B200GS_STAGE_SCAN, st);
            if (launch_depth_order(a.tiles_touched, offsets, n_vp, V, bb, BL, &order_sorted, &total_dev, st, &nl)) return cuda_fail(cudaGetLastError(), "depth order");
        }
        // The EXACT 64-bit instance count travels to a pinned host word (nothing reads the possibly wrapped 32-bit offsets
        // before it has been checked).
        HostSlot *hs = host_slot();
        if (!hs) return cuda_fail(cudaGetLastError(), "pinned count slot");
        CK(cudaMemcpyAsync(hs->total, total_dev, 8, cudaMemcpyDeviceToHost, st), "D2H num_rendered");
        int64_t cap = instance_capacity < B200GS_MAX_INSTANCES ? instance_capacity : (int64_t)B200GS_MAX_INSTANCES;
        if (cap < 1) cap = 1; // the layout always has room for one instance
        if (n_vp <= B200GS_DEFERRED_MAX_NVP) {
            // Small batches (the per-view drop-in pattern, the 8-view SDS batch): the host does NOT wait here.  Emit / tile
            // sort / ranges / blend are enqueued sized for the caller's capacity and read the count on the device, so the GPU
            // never idles behind a host round trip (upstream blocks on this read-back in the middle of every forward).  The
            // count is checked after the last launch, when the copy has long completed: a batch that did not fit produced
            // clamped, in-bounds garbage and the call reports it (B200GS_E_BIN_TOO_SMALL / _E_INSTANCES) before anything is used.
            CK(cudaEventRecord(hs->ev, st), "event after count copy");
            pending = hs;
            StageTimer t(B200GS_STAGE_BINNING, st);
            const int brc = launch_binning(order_sorted, a.rects, offsets, P, V, gx, gy, cap, total_dev, bb, BL, st, &nl);
            if (brc == -3) return B200GS_E_RANGE;
            if (brc) return cuda_fail(cudaGetLastError(), "binning");
        } else {
            // Large batches: one wait per tens of milliseconds of work costs nothing, and launches sized for the exact count
            // do no work for the unused capacity.
            CK(cudaStreamSynchronize(st), "sync after scan");
            const uint64_t total = *hs->total;
            *num_rendered = (int64_t)total;
            if (total > (uint64_t)B200GS_MAX_INSTANCES) return B200GS_E_INSTANCES;
            if ((int64_t)total > instance_capacity) return B200GS_E_BIN_TOO_SMALL;
            StageTimer t(B200GS_STAGE_BINNING, st);
            const int brc = launch_binning(order_sorted, a.rects, offsets, P, V, gx, gy, (int64_t)total, nullptr, bb, BL, st, &nl);
            if (brc == -3) return B200GS_E_RANGE;
            if (brc) return cuda_fail(cudaGetLastError(), "binning");
        }
        g_launches += nl; // radix count/scan/scatter passes, tile scan, emit, ranges, tile order: all ours
    }
    BlendArgs b;
    b.H = H; b.W = W; b.grid_x = gx; b.grid_y = gy; b.V = V; b.P = P;
    b.ranges = (const uint2 *)(bb + BL.ranges); b.point_list = (const uint32_t *)(bb + BL.vals_out);
    b.tile_order = (const uint32_t *)(bb + BL.tile_order);
    b.recs = (const GeomRec *)(gb + GL.recs); b.bg = bg;
    b.final_T = (float *)(ib + IL.final_T); b.n_contrib = (uint32_t *)(ib + IL.n_contrib);
    b.out_color = out_color; b.out_depth = out_depth; b.out_alpha = out_alpha;
    b.cmask = (uint32_t *)(bb + BL.cmask);
    (void)HW;
    {
        StageTimer t(B200GS_STAGE_BLEND_FWD, st);
        launch_blend_fwd(b, st);
        g_launches += 1;
    }
    CK(cudaGetLastError(), "forward launch");
    if (pending) { // everything is enqueued; now look at the instance count (copied right after the scan)
        CK(cudaEventSynchronize(pending->ev), "wait for the instance count");
        const uint64_t total = *pending->total;
        *num_rendered = (int64_t)total;
        if (total > (uint64_t)B200GS_MAX_INSTANCES) return B200GS_E_INSTANCES;
        if ((int64_t)total > instance_capacity) return B200GS_E_BIN_TOO_SMALL;
    }
    return B200GS_OK;
}

size_t b200gs_deterministic_bytes(int64_t num_rendered, int64_t partial_capacity, int32_t P, int32_t V)
{
    return DetLayout(num_rendered, partial_capacity, (int64_t)(P > 0 ? P : 0) * (V > 0 ? V : 0)).total;
}

// b200gs_backward (det == false) and b200gs_backward_deterministic (det == true)
static int backward_impl(const b200gs_params *prm, const float *means3D, const float *shs, const float *colors_precomp,
                         const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp,
                         const float *bg, const float *viewmatrix, const float *projmatrix, const float *campos,
                         const int32_t *radii, const void *geom_buf, const void *binning_buf, int64_t instance_capacity,
                         const void *image_buf, int64_t num_rendered, const float *dL_dcolor, const float *dL_ddepth,
                         const float *dL_dalpha, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors,
                         float *dL_dopacity, float *dL_dscales, float *dL_drots, float *dL_dcov3D, void *scratch,
                         size_t scratch_bytes, void *stream, bool det, void *det_buf, size_t det_bytes, int64_t partial_capacity,
                         int64_t *n_partials)
{
    if (det) {
        if (!blend_bwd_has_deterministic()) return B200GS_E_UNSUPPORTED;
        if (!n_partials || !det_buf || partial_capacity < 0) return B200GS_E_ARGS;
        *n_partials = 0;
        if (num_rendered < 0 || num_rendered > instance_capacity || num_rendered > B200GS_MAX_INSTANCES) return B200GS_E_ARGS;
        if (((uintptr_t)det_buf) & 15) return B200GS_E_BUFFER;
    }
    int rc = check_common(prm, shs, colors_precomp, scales, rotations, cov3D_precomp);
    if (rc) return rc;
    if (prm->raw_params && !opacities) return B200GS_E_ARGS;
    if (!means3D || !bg || !viewmatrix || !projmatrix || !campos || !radii || !geom_buf || !binning_buf || !image_buf ||
        !dL_dmeans3D || !dL_dmeans2D || !dL_dopacity || !scratch)
        return B200GS_E_ARGS;
    if (shs ? !dL_dsh : !dL_dcolors) return B200GS_E_ARGS;
    if (scales ? (!dL_dscales || !dL_drots) : !dL_dcov3D) return B200GS_E_ARGS;
    cudaStream_t st = (cudaStream_t)stream;
    const int P = prm->P, V = prm->n_views, H = prm->image_height, W = prm->image_width;
    if (P == 0) return B200GS_OK;
    const int gx = (W + GS_TILE - 1) / GS_TILE, gy = (H + GS_TILE - 1) / GS_TILE;
    const GeomLayout GL(P, V);
    const ImageLayout IL(H, W, V);
    const BinLayout BL = binning_layout(instance_capacity, gx * gy * V, (int64_t)P * V);
    if (scratch_bytes < b200gs_backward_scratch_bytes(P, V)) return B200GS_E_BUFFER;
    if ((((uintptr_t)geom_buf) | ((uintptr_t)binning_buf) | ((uintptr_t)image_buf) | ((uintptr_t)scratch)) & 15) return B200GS_E_BUFFER;
    const char *gb = (const char *)geom_buf, *bb = (const char *)binning_buf, *ib = (const char *)image_buf;
    const int64_t n_vp = (int64_t)P * V;
    const DetLayout DL(num_rendered, partial_capacity, n_vp);
    if (det && det_bytes < DL.total) return B200GS_E_BUFFER;

    if (!det) CK(cudaMemsetAsync(scratch, 0, (size_t)P * V * sizeof(ScreenGrad), st), "memset scratch");
    BlendBwdArgs b;
    b.H = H; b.W = W; b.grid_x = gx; b.grid_y = gy; b.V = V; b.P = P;
    b.ranges = (const uint2 *)(bb + BL.ranges); b.point_list = (const uint32_t *)(bb + BL.vals_out);
    b.tile_order = (const uint32_t *)(bb + BL.tile_order);
    b.recs = (const GeomRec *)(gb + GL.recs); b.bg = bg;
    b.final_T = (const float *)(ib + IL.final_T); b.n_contrib = (const uint32_t *)(ib + IL.n_contrib);
    b.dL_dcolor = dL_dcolor; b.dL_ddepth = dL_ddepth; b.dL_dalpha = dL_dalpha;
    b.cmask = (const uint32_t *)(bb + BL.cmask);
    b.sgrad = scratch;
    if (!det) {
        StageTimer t(B200GS_STAGE_BLEND_BWD, st);
        launch_blend_bwd(b, st);
    } else {
        // pre-pass -> (the one host wait: the partial count) -> B1 with per-partial stores -> fixed-order reduce.  The wait
        // sits after the scan so that a call whose partials do not fit returns before B1 runs; every access of the pre-pass
        // stays inside buffers sized by num_rendered and P*V alone.
        StageTimer t(B200GS_STAGE_BLEND_BWD, st);
        char *db = (char *)det_buf;
        DetPlanArgs pa;
        pa.H = H; pa.W = W; pa.grid_x = gx; pa.grid_y = gy; pa.D = num_rendered;
        pa.tile_order = b.tile_order; pa.ranges = b.ranges; pa.point_list = b.point_list; pa.cmask = b.cmask; pa.n_contrib = b.n_contrib;
        pa.rects = (const uint2 *)(gb + GL.rects);
        pa.order = (const uint32_t *)(bb + BL.order_in); // the depth order (four ping-pong passes end where they began)
        pa.offsets = (const uint32_t *)(gb + GL.offsets); pa.tiles_touched = (const uint32_t *)(gb + GL.tiles_touched);
        pa.start = (uint32_t *)(db + DL.start); pa.pm = (uint8_t *)(db + DL.pm); pa.base = (uint32_t *)(db + DL.base);
        pa.jpos = (uint32_t *)(db + DL.jpos);
        uint64_t H_partials = 0;
        if (num_rendered > 0) {
            int nl = 0;
            if (launch_det_plan(pa, n_vp, gx * gy * V, DL, db, st, &nl)) return cuda_fail(cudaGetLastError(), "deterministic plan");
            g_launches += nl;
            HostSlot *hs = host_slot();
            if (!hs) return cuda_fail(cudaGetLastError(), "pinned count slot");
            CK(cudaMemcpyAsync(hs->total, db + DL.total_slot, 8, cudaMemcpyDeviceToHost, st), "D2H partial count");
            CK(cudaEventRecord(hs->ev, st), "event after partial count");
            CK(cudaEventSynchronize(hs->ev), "wait for the partial count");
            H_partials = *hs->total;
        }
        *n_partials = (int64_t)H_partials;
        if (H_partials > 0xffffffffull) return B200GS_E_RANGE; // 32-bit slots; 160 GB of partials would not fit a device anyway
        if ((int64_t)H_partials > partial_capacity) return B200GS_E_BIN_TOO_SMALL;
        float *partials = (float *)(db + DL.partials);
        if (H_partials > 0) launch_blend_bwd_det(b, DetFlush{pa.pm, pa.base, partials}, st);
        launch_det_reduce(pa, n_vp, partials, scratch, st);
        g_launches += (H_partials > 0) + 1;
    }

    PreBwdArgs a;
    a.P = P; a.V = V; a.deg = shs ? prm->sh_degree : 0; a.M = prm->sh_coeffs; a.H = H; a.W = W; a.mod = prm->scale_modifier;
    a.vec16 = (((uintptr_t)dL_drots) & 15) == 0;
    a.raw = prm->raw_params != 0; a.opac = opacities;
    a.means_view_stride = prm->means3D_per_view ? (size_t)3 * P : 0;
    a.means = means3D; a.shs = shs; a.colors_pre = colors_precomp; a.scales = scales; a.rots = rotations; a.cov_pre = cov3D_precomp;
    a.view = viewmatrix; a.proj = projmatrix; a.campos = campos;
    for (int v = 0; v < V; v++) { a.tanfovx[v] = prm->tanfovx[v]; a.tanfovy[v] = prm->tanfovy[v]; }
    a.radii = radii; a.clamped = (const uint8_t *)(gb + GL.clamped); a.sgrad = scratch;
    a.recs = (const GeomRec *)(gb + GL.recs); a.moments = blend_sgrad_is_moments();
    a.dL_dmeans3D = dL_dmeans3D; a.dL_dmeans2D = dL_dmeans2D; a.dL_dsh = dL_dsh; a.dL_dcolors = dL_dcolors;
    a.dL_dopacity = dL_dopacity; a.dL_dscales = dL_dscales; a.dL_drots = dL_drots; a.dL_dcov3D = dL_dcov3D;
    { StageTimer t(B200GS_STAGE_PREPROCESS_BWD, st); launch_preprocess_bwd(a, st); }
    g_launches += det ? 1 : 2; // (the deterministic blend stage counted its own launches)
    CK(cudaGetLastError(), "backward launch");
    return B200GS_OK;
}

int b200gs_backward(const b200gs_params *prm, const float *means3D, const float *shs, const float *colors_precomp,
                    const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp,
                    const float *bg, const float *viewmatrix, const float *projmatrix, const float *campos,
                    const int32_t *radii, const void *geom_buf, const void *binning_buf, int64_t instance_capacity,
                    const void *image_buf, int64_t num_rendered, const float *dL_dcolor, const float *dL_ddepth,
                    const float *dL_dalpha, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors,
                    float *dL_dopacity, float *dL_dscales, float *dL_drots, float *dL_dcov3D, void *scratch,
                    size_t scratch_bytes, void *stream)
{
    return backward_impl(prm, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, bg, viewmatrix, projmatrix,
                         campos, radii, geom_buf, binning_buf, instance_capacity, image_buf, num_rendered, dL_dcolor, dL_ddepth,
                         dL_dalpha, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drots, dL_dcov3D,
                         scratch, scratch_bytes, stream, false, nullptr, 0, 0, nullptr);
}

int b200gs_backward_deterministic(const b200gs_params *prm, const float *means3D, const float *shs, const float *colors_precomp,
                                  const float *opacities, const float *scales, const float *rotations, const float *cov3D_precomp,
                                  const float *bg, const float *viewmatrix, const float *projmatrix, const float *campos,
                                  const int32_t *radii, const void *geom_buf, const void *binning_buf, int64_t instance_capacity,
                                  const void *image_buf, int64_t num_rendered, const float *dL_dcolor, const float *dL_ddepth,
                                  const float *dL_dalpha, float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors,
                                  float *dL_dopacity, float *dL_dscales, float *dL_drots, float *dL_dcov3D, void *scratch,
                                  size_t scratch_bytes, void *det_buf, size_t det_bytes, int64_t partial_capacity,
                                  int64_t *n_partials, void *stream)
{
    return backward_impl(prm, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, bg, viewmatrix, projmatrix,
                         campos, radii, geom_buf, binning_buf, instance_capacity, image_buf, num_rendered, dL_dcolor, dL_ddepth,
                         dL_dalpha, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drots, dL_dcov3D,
                         scratch, scratch_bytes, stream, true, det_buf, det_bytes, partial_capacity, n_partials);
}

int b200gs_mark_visible(int32_t P, const float *positions, const float *viewmatrix, const float *projmatrix,
                        uint8_t *present, void *stream)
{
    (void)projmatrix;
    if (P < 0 || !positions || !viewmatrix || !present) return B200GS_E_ARGS;
    if (P == 0) return B200GS_OK;
    launch_mark_visible(P, positions, viewmatrix, present, (cudaStream_t)stream);
    g_launches += 1;
    CK(cudaGetLastError(), "mark_visible launch");
    return B200GS_OK;
}

int b200gs_describe_state(const b200gs_params *prm, const void *geom_buf, const void *binning_buf, int64_t instance_capacity,
                          const void *image_buf, b200gs_state_view *out)
{
    if (!prm || !out || !geom_buf || !binning_buf || !image_buf) return B200GS_E_ARGS;
    const int P = prm->P, V = prm->n_views, H = prm->image_height, W = prm->image_width;
    const int gx = (W + GS_TILE - 1) / GS_TILE, gy = (H + GS_TILE - 1) / GS_TILE;
    const GeomLayout GL(P, V);
    const ImageLayout IL(H, W, V);
    const BinLayout BL = binning_layout(instance_capacity, gx * gy * V, (int64_t)P * V);
    const char *gb = (const char *)geom_buf, *bb = (const char *)binning_buf, *ib = (const char *)image_buf;
    out->geom_records = gb + GL.recs;
    out->tiles_touched = (const uint32_t *)(gb + GL.tiles_touched);
    out->offsets = (const uint32_t *)(gb + GL.offsets);
    out->clamped = (const uint8_t *)(gb + GL.clamped);
    out->sorted_tile_keys = (const uint32_t *)(bb + BL.keys_out);
    // the depth sort takes 32 / 8 = 4 ping-pong passes starting from order_in: an even count ends where it began
    out->depth_order = (const uint32_t *)(bb + BL.order_in);
    out->point_list = (const uint32_t *)(bb + BL.vals_out);
    out->ranges = (const uint32_t *)(bb + BL.ranges);
    out->final_T = (const float *)(ib + IL.final_T);
    out->n_contrib = (const uint32_t *)(ib + IL.n_contrib);
    out->contributor_masks = (const uint32_t *)(bb + BL.cmask);
    const int64_t cap = instance_capacity > 0 ? instance_capacity : 1;
    out->contributor_mask_words = ((cap >> 5) + (int64_t)gx * gy * V + 1) * 8; // BinLayout::cmask's extent
    return B200GS_OK;
}

void b200gs_profile_enable(int on)
{
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof_on = on != 0;
}

int b200gs_profile_read(double *ms_per_stage, int64_t *calls_per_stage, int32_t n_stages)
{
    if (!ms_per_stage || !calls_per_stage || n_stages < B200GS_STAGE_COUNT) return B200GS_E_ARGS;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (int i = 0; i < n_stages; i++) { ms_per_stage[i] = 0.0; calls_per_stage[i] = 0; }
    for (auto &sp : g_spans) {
        float ms = 0.f;
        cudaError_t e = cudaEventSynchronize(sp.e1);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, sp.e0, sp.e1);
        if (e == cudaSuccess) { ms_per_stage[sp.stage] += ms; calls_per_stage[sp.stage] += 1; }
        g_event_pool.push_back(sp.e0); g_event_pool.push_back(sp.e1);
    }
    g_spans.clear();
    return B200GS_OK;
}

size_t b200gs_knn_scratch_bytes(int32_t P) { return knn_scratch_bytes(P); }

int b200gs_dist2_knn3(int32_t P, const float *points, float *mean_dist2, void *scratch, size_t scratch_bytes, void *stream)
{
    if (P < 0 || !points || !mean_dist2 || !scratch) return B200GS_E_ARGS;
    if (P < 4) return B200GS_E_RANGE; // needs 3 neighbours besides the point itself
    int nl = 0;
    const int rc = launch_knn3(P, points, mean_dist2, (char *)scratch, scratch_bytes, (cudaStream_t)stream, &nl);
    if (rc == -1) return B200GS_E_BUFFER;
    if (rc) return B200GS_E_RANGE;
    g_launches += nl;
    CK(cudaGetLastError(), "knn launch");
    return B200GS_OK;
}

int b200gs_reattach(int32_t P, int32_t n_frames, int32_t n_verts, int32_t n_faces, const float *vertices, const int32_t *faces,
                    const int32_t *mapping_face, const float *mapping_uvw, const float *mapping_dist, float *xyz_out, void *stream)
{
    if (P < 0 || n_frames < 1 || n_verts < 1 || n_faces < 1 || !vertices || !faces || !mapping_face || !mapping_uvw || !mapping_dist || !xyz_out)
        return B200GS_E_ARGS;
    if (n_frames > 65535) return B200GS_E_RANGE;
    if (P == 0) return B200GS_OK;
    launch_reattach(P, n_frames, n_verts, n_faces, vertices, faces, mapping_face, mapping_uvw, mapping_dist, xyz_out, (cudaStream_t)stream);
    g_launches += 1;
    CK(cudaGetLastError(), "reattach launch");
    return B200GS_OK;
}

int b200gs_pack_frames_u8(const float *color, uint8_t *out, int32_t image_height, int32_t image_width, int32_t n_frames, void *stream)
{
    if (!color || !out || image_height < 1 || image_width < 1 || n_frames < 1) return B200GS_E_ARGS;
    if (n_frames > 65535) return B200GS_E_RANGE;
    launch_pack_u8(color, out, image_height, image_width, n_frames, (cudaStream_t)stream);
    g_launches += 1;
    CK(cudaGetLastError(), "pack launch");
    return B200GS_OK;
}

int b200gs_densify_stats(int32_t P, int32_t n_views, const float *dL_dmeans2D, const int32_t *radii, const uint8_t *update_mask,
                         float *xyz_gradient_accum, float *denom, float *max_radii2D, void *stream)
{
    if (P < 0 || n_views < 1 || !dL_dmeans2D || !radii || !xyz_gradient_accum || !denom || !max_radii2D) return B200GS_E_ARGS;
    if (P == 0) return B200GS_OK;
    launch_densify_stats(P, n_views, dL_dmeans2D, radii, update_mask, xyz_gradient_accum, denom, max_radii2D, (cudaStream_t)stream);
    g_launches += 1;
    CK(cudaGetLastError(), "densify_stats launch");
    return B200GS_OK;
}

size_t b200gs_densify_scratch_bytes(int32_t P) { return densify_scratch_bytes(P < 0 ? 0 : P); }

int b200gs_densify_plan(int32_t P, const b200gs_densify_cfg *cfg, const float *xyz_gradient_accum, const float *denom,
                        const float *opacity_raw, const float *scaling_raw, int32_t *plan, int32_t *counts, void *scratch,
                        size_t scratch_bytes, void *stream)
{
    if (P < 1 || !cfg || !opacity_raw || !scaling_raw || !plan || !counts || !scratch) return B200GS_E_ARGS;
    if (cfg->mode != 0 && cfg->mode != 1) return B200GS_E_ARGS;
    if (cfg->mode == 0 && (!xyz_gradient_accum || !denom || cfg->n_split < 1)) return B200GS_E_ARGS;
    if (cfg->n_split > 16 || (int64_t)P * (1 + (cfg->mode == 0 ? 1 + cfg->n_split : 0)) > 0x7fffffffLL) return B200GS_E_RANGE;
    if (scratch_bytes < densify_scratch_bytes(P)) return B200GS_E_BUFFER;
    DensifyCfg c;
    c.mode = cfg->mode; c.n_split = cfg->mode == 0 ? cfg->n_split : 0; c.use_screen = cfg->use_screen;
    c.max_grad = cfg->max_grad; c.min_opacity = cfg->min_opacity; c.dense_thresh = cfg->percent_dense_x_extent;
    c.max_screen_size = cfg->max_screen_size; c.big_ws_thresh = cfg->big_ws_thresh;
    launch_densify_plan(c, P, xyz_gradient_accum, denom, opacity_raw, scaling_raw, plan, counts, (char *)scratch, (cudaStream_t)stream);
    g_launches += 3;
    CK(cudaGetLastError(), "densify_plan launch");
    return B200GS_OK;
}

int b200gs_densify_move(int32_t role, int32_t P, int32_t row_floats, const int32_t *plan, const int32_t *counts_host, int32_t n_split,
                        const float *src, float *dst, const float *rotation_raw, const float *scaling_raw, const float *noise, void *stream)
{
    if (P < 1 || row_floats < 1 || role < 0 || role > 3 || !plan || !counts_host || !src || n_split < 0) return B200GS_E_ARGS;
    const int S_sel = counts_host[2], S_kept = counts_host[3];
    const int64_t P_new = (int64_t)counts_host[0] + counts_host[1] + (int64_t)n_split * S_kept;
    if (counts_host[0] < 0 || counts_host[1] < 0 || S_sel < 0 || S_kept < 0 || S_kept > S_sel || counts_host[4] != P_new) return B200GS_E_ARGS;
    if (P_new > 0 && !dst) return B200GS_E_ARGS;
    if (role == B200GS_ROLE_XYZ && (row_floats != 3 || (S_kept > 0 && (!rotation_raw || !scaling_raw || !noise)))) return B200GS_E_ARGS;
    if (P_new == 0) return B200GS_OK;
    launch_densify_move(role, P, row_floats, plan, src, dst, n_split, S_sel, S_kept, rotation_raw, scaling_raw, noise, (cudaStream_t)stream);
    g_launches += 1;
    CK(cudaGetLastError(), "densify_move launch");
    return B200GS_OK;
}

int b200gs_adam_packed(const b200gs_adam_cfg *cfg, float *params, const float *grads, float *exp_avg, float *exp_avg_sq,
                       void *stream)
{
    if (!cfg || !params || !grads || !exp_avg || !exp_avg_sq || cfg->P < 0) return B200GS_E_ARGS;
    for (const void *p : {(const void *)params, (const void *)grads, (const void *)exp_avg, (const void *)exp_avg_sq})
        if ((uintptr_t)p % 16) return B200GS_E_ARGS;
    if (cfg->sh_coeffs < 1 || cfg->total < 0 || cfg->total % 4) return B200GS_E_RANGE;
    AdamArgs a;
    const int64_t P = cfg->P;
    const int64_t off[5] = {cfg->off_xyz, cfg->off_scaling, cfg->off_rotation, cfg->off_opacity, cfg->off_sh};
    const int64_t numel[5] = {3 * P, 3 * P, 4 * P, P, 3 * (int64_t)cfg->sh_coeffs * P};
    const int group[5] = {ADAM_GROUP_XYZ, ADAM_GROUP_SCALING, ADAM_GROUP_ROTATION, ADAM_GROUP_OPACITY, ADAM_GROUP_F_REST};
    int64_t end = 0;
    for (int f = 0; f < 5; f++) {
        if (off[f] < end || off[f] % 4) return B200GS_E_RANGE; // fields in buffer order, disjoint, 16-byte aligned
        end = off[f] + numel[f];
        a.off[f] = off[f]; a.numel[f] = numel[f]; a.field_group[f] = group[f];
    }
    if (end > cfg->total) return B200GS_E_RANGE;
    a.sh_coeffs = cfg->sh_coeffs;
    a.lerp_small = fabsf(cfg->one_minus_beta1) < 0.5f;
    for (int g = 0; g < 6; g++) a.step_size[g] = cfg->step_size[g];
    a.bias_correction2_sqrt = cfg->bias_correction2_sqrt; a.one_minus_beta1 = cfg->one_minus_beta1; a.beta2 = cfg->beta2;
    a.one_minus_beta2 = cfg->one_minus_beta2; a.eps = cfg->eps;
    if (cfg->total == 0) return B200GS_OK;
    launch_adam_packed(a, cfg->total, params, grads, exp_avg, exp_avg_sq, (cudaStream_t)stream);
    g_launches += 1;
    CK(cudaGetLastError(), "adam_packed launch");
    return B200GS_OK;
}

int b200gs_test_sort_pairs(uint32_t *keys_a, uint32_t *keys_b, uint32_t *vals_a, uint32_t *vals_b, int64_t n, int32_t nbits,
                           void *scratch, size_t scratch_bytes, int32_t *result_in_b, void *stream)
{
    if (n < 1 || nbits < 1 || nbits > 32 || !keys_a || !keys_b || !vals_a || !vals_b || !scratch || !result_in_b) return B200GS_E_ARGS;
    if (scratch_bytes < test_sort32_scratch_bytes(n)) return B200GS_E_BUFFER;
    int in_b = 0;
    if (launch_test_sort32(keys_a, keys_b, vals_a, vals_b, n, nbits, (char *)scratch, scratch_bytes, &in_b, (cudaStream_t)stream))
        return B200GS_E_RANGE;
    *result_in_b = in_b;
    CK(cudaGetLastError(), "test_sort launch");
    return B200GS_OK;
}
size_t b200gs_test_sort_scratch_bytes(int64_t n) { return test_sort32_scratch_bytes(n); }

int b200gs_test_exp(const float *x, float *y, int64_t n, void *stream)
{
    if (n < 0 || !x || !y) return B200GS_E_ARGS;
    if (n == 0) return B200GS_OK;
    launch_test_exp(x, y, n, (cudaStream_t)stream);
    g_launches += 1;
    CK(cudaGetLastError(), "test_exp launch");
    return B200GS_OK;
}

} // extern "C"
