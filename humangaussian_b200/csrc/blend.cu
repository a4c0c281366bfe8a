// blend.cu -- F6 forward alpha blend and B1 backward blend (SURVEY.md Appendix A.4 / A.5).
//
// PATCH-PARALLEL: every warp owns one 8x4 pixel patch of a 16x16 tile and walks the tile's instance list ON ITS
// OWN -- no CTA-wide barrier anywhere in the loops.  (The first version staged 256 instances per CTA between
// __syncthreads; ncu showed 35 % of warp-time parked on that barrier because the eight patches of a tile see very
// different numbers of Gaussians.)  CTAs are 64 threads = two independent warps (a 16x4 strip), so the block
// scheduler balances patches dynamically and a finished warp frees its slot almost immediately.
//   * Forward, chunks of 32 list entries: lane l loads entry l's id and the first 16 bytes of its 48-byte GeomRec
//     (px, py, hx, hy), tests the Gaussian's conservative alpha-support box against the warp's patch, and the
//     warp ballots.  Hits load the rest of the record and are compacted, in order, into a per-warp shared-memory
//     slab; the next chunk's id/box loads are already in flight while the hits are blended.
//     Measured on the bench workload (300 k subsample of sample.ply, counter build of round 2): 2.15 of 8 patches
//     survive the box test per instance, 83 % of those visits have a contributing lane, 13.6 of 32 lanes contribute.
//     The hits' list position and record index ride in the two slab words the support box occupied.
//   * The forward records, per (chunk, patch), which entries contributed to at least one pixel of the patch (the
//     contributor mask, BinLayout::cmask).  The backward walks those masks instead of repeating the cull: it loads ids
//     and records of contributing entries only, and every entry it stages has a contributing lane.  Forward and backward
//     evaluate power, gs_exp and alpha with the same bit-exact expressions, so the (pixel, entry) pairs the backward
//     replays (pos < n_contrib) are exactly those the forward blended.
//   * Tile lists are exactly the reference's (tile/sort indices bit-identical); culling only skips pairs whose
//     alpha is provably < 1/255, so images are unchanged.  Forward arithmetic follows the pinned order of
//     common.cuh: images are bit-identical to the CPU oracle.
//   * Backward: per-pixel terms are expressed as ten sums per Gaussian -- six moments of q = G*dL/dalpha
//     (1, dx, dy, dx^2, dx*dy, dy^2) and four colour/depth weights.  The hit loop parks each pixel's (q, w) in shared
//     memory; every BWD_PARK hits a transposed pass (lane = hit, walking pixels) forms the ten sums in registers and
//     writes them with three vector REDs (v4 + v4 + v2) into the Gaussian's 48-byte ScreenGrad record.  Upstream:
//     ~10 atomics per PIXEL.
//   * Both hit loops are branch-free: the per-pixel decisions (skip, done, blend / contribute) are predicates and the
//     updates are predicated or selected, because a warp that diverges issues both sides.  What ptxas makes of them
//     (CUDA 12.9, sm_90a, -O3; static SASS counts): forward 56 registers, 3 KB smem, no spills; 81 instructions per
//     unrolled pair of hits (40.5 per hit, loop control and two constant moves included; 49 per hit with branches),
//     no BSSY/BSYNC/BRA inside the pair, about 96 per 32-entry chunk of bookkeeping.  Backward 64 registers, 13.1 KB smem,
//     no spills; 107 per unrolled pair of hits (53.5 per hit; about 65 with a branch around the contributing-lane block
//     and separate slot / hit counters), plus the flush.
//   * Two kernel templates: blend_fwd_kernel<CONTRIB, NRM, GEO> (five instantiations: contribution scores never come with
//     normals or geometry) and blend_bwd_kernel<DET, ABS, NRM, GEO> (all sixteen).  A feature flag adds its code under an
//     `if` on the flag, its per-warp shared arrays, and its kernel arguments as members of FwdFeatures / BwdFeatures; with
//     every flag off the code is the default kernel's, so a feature does not change the default kernels' SASS.  The
//     launchers map the option bits to an instantiation in one place each.
//   * Deterministic mode (torch.use_deterministic_algorithms): DET selects a flush that stores each (instance, patch)
//     partial into its own slot instead of the REDs; deterministic.cu plans the slots and adds each Gaussian's partials in
//     a fixed order.
//   * Absolute screen-space gradients (densification statistic, DESIGN.md section 2): with ABS the flush also sums
//     |q (A dx + B dy)| and |q (B dx + C dy)| into ScreenGrad's padding (or a float2 per partial); absgrad_out_kernel scales
//     them to dL_dmeans2D_abs.
//   * Contribution scores (DESIGN.md section 2): with CONTRIB the forward also folds each hit into its Gaussian's
//     weight_sum / weight_max / touches (warp reductions, then three atomics from lane 0).
//   * Normal maps (DESIGN.md section 2): with NRM each hit's normal (normals.cu's gauss_normals) is staged next to its slab
//     record, the forward keeps three more sums per pixel, the backward adds n . dL/dN to cg and the flush sums
//     Wn = sum w dL/dN.
//   * The compile-time switches below are the A/B experiments DESIGN.md section 5 lists: the
//     product is BWD_T_DIV=1 and BWD_PARK=16, everything else 0.
#include "common.cuh"
#include "kernels.h"
#include <type_traits>

#define FULL 0xffffffffu
#ifndef WARPS_PER_CTA
#define WARPS_PER_CTA 2 // independent patches per CTA (1, 2, 4 or 8); H100 (400 W) bench step: 1 and 2 within noise, 4 is 26 % slower
#endif
#ifndef BWD_MIN_BLOCKS
#define BWD_MIN_BLOCKS 16 // caps the backward kernel at 64 registers (32 warps/SM), no spills.  H100 80GB HBM3, 700 W, bench step
                          // with the park buffer: 12 blocks (80 registers) bwd 14.3 ms against 13.1 ms at 16.  Before it (400 W):
                          // 12 within noise, 20 blocks 2.5 % slower
#endif
#define CTAS_PER_TILE (8 / WARPS_PER_CTA)
#ifndef FWD_MIN_BLOCKS
#define FWD_MIN_BLOCKS 18 // caps the default forward kernel at 56 registers (36 warps/SM), no spills; left to itself ptxas takes 60
#endif
#ifndef FWD_FEATURE_MIN_BLOCKS
// the forward kernels with a feature: at the default's cap of 56 registers the contribution variant spills 8 bytes in the hit
// loop; 16 blocks (64 registers, 32 warps/SM, the backward's occupancy) removes the spill (DESIGN.md section 5 lists the
// registers of every instantiation at this bound)
#define FWD_FEATURE_MIN_BLOCKS 16
#endif
#ifndef BWD_PARK
#define BWD_PARK 16 // backward: hits parked per flush (8 or 16); 32 / BWD_PARK lanes share a hit in the flush pass.  H100 80GB
                    // HBM3, 700 W, bench step, bwd: 16 -> 13.1 ms (13.1 KB smem per CTA), 8 -> 14.0 ms (8.7 KB; 15.2-15.5 ms
                    // at 12 blocks)
#endif
#if BWD_PARK != 8 && BWD_PARK != 16
#error "BWD_PARK must be 8 or 16"
#endif
#ifndef BWD_T_DIV
#define BWD_T_DIV 1 // transmittance recovery T <- T/(1-alpha): 0 = MUFU reciprocal, 1 = + one Newton step, 2 = IEEE division.
                    // On the 17 k-deep tiles of the real scene the raw reciprocal's bias compounds over the replay and moves the
                    // worst position-gradient rows out of tolerance; one Newton step (two FMAs) removes the bias.
#endif

// does the support box [px-hx,px+hx] x [py-hy,py+hy] reach the patch [x0,x0+7] x [y0,y0+3] ?  (x1 = x0 + 7, y1 = y0 + 3.)
// The five comparisons have no side effects, so they are and-ed without short-circuit: one predicate chain, no branch.
__device__ __forceinline__ bool box_hits_patch(const float4 g0, float x0, float y0, float x1, float y1)
{
    return (g0.z >= 0.0f) & (g0.x + g0.z >= x0) & (g0.x - g0.z <= x1) & (g0.y + g0.w >= y0) & (g0.y - g0.w <= y1);
}

// power with the conic pre-scaled at staging time (A' = -A/2, B' = -B, C' = -C/2: exact operations, so the
// result is bit-identical to gs_power(A,B,C,dx,dy))
__device__ __forceinline__ float power_prescaled(float Ap, float Bp, float Cp, float dx, float dy)
{
    const float u = ffma(Bp, dy, fmul(Ap, dx));
    const float w = fmul(fmul(Cp, dy), dy);
    return ffma(dx, u, w);
}

// per-warp slab of the (at most 32) hits of the current chunk
// (forward: px,py,list position (bits),the entry's bit in its chunk (bits) -- a pixel that blends the hit ORs that bit into
//  its contributor mask with one instruction; backward: px,py,list position (bits),record index (bits))
struct __align__(16) WarpSlab {
    float4 rec[32 * 3]; // px,py,list position,entry bit or record index | A',B',C',o | r,g,b,depth
};

// ------------------------------------------------------------------------------------------------
// F6
// ------------------------------------------------------------------------------------------------
// A forward pixel's running state.  A live pixel has T >= 1e-4.  A finished pixel keeps its last transmittance with the
// sign bit set (an out-of-image pixel starts at 0): it keeps failing the T test and never accumulates, exactly like
// upstream's `done` flag, and |T| is the transmittance to report.
struct FwdPixel {
    float T, C0, C1, C2, Dd, Aa;
    uint32_t last, used; // 1-based list position of the last blended entry; entries of the chunk this pixel blended
};

// The forward's feature arguments: one member per enabled feature, none for a disabled one (an empty base takes no space), so
// an instantiation's parameters keep the layout (args, contribution outputs, normals, geometry outputs) of the features it has.
// Code that reads a member sits under `if constexpr` on its flag.
template <bool> struct FwdContribArg {};
template <> struct FwdContribArg<true> { ContribOut co; };
template <bool> struct FwdNrmArg {};
template <> struct FwdNrmArg<true> { const float4 *gauss_normals; float *out_normal; }; // [V*P] (normals.cu), [V,3,H,W]
template <bool> struct FwdGeoArg {};
template <> struct FwdGeoArg<true> { GeoFwd geo; };
template <bool CONTRIB, bool NRM, bool GEO> struct FwdFeatures : FwdContribArg<CONTRIB>, FwdNrmArg<NRM>, FwdGeoArg<GEO> {};

// One slab hit s (three words) blended into pixel (fpx, fpy): the operation sequence of DESIGN.md section 2.  The three
// outcomes -- skip (power > 0 or alpha < 1/255), done (T would fall below 1e-4) and blend -- are predicates, not branches:
// 13.6 of 32 lanes blend per visit, so a branch would diverge and the warp would issue both sides anyway.  A lane that does
// not blend keeps C0..C2, Dd, Aa, last and used bit for bit and T up to its sign: its updates are predicated off, never
// scaled by a zero weight (c * 0 is not an exact no-op for every colour a caller may pass).
// Contribution scores (DESIGN.md section 2): one slab hit's warp-wide share of its Gaussian's three accumulators.  A touch is a
// hit on a live pixel (it blends, or it is the terminating hit); a blend adds q(w) = rn(w * 2^24) and competes with the bits
// of w for the maximum (w > 0, so unsigned order is float order).  32 lanes * q < 2^29 fits the u32 lane sum.  The ballot
// is warp-uniform, so the whole warp skips a hit no pixel touched; lane 0 then issues the three reductions.
__device__ __forceinline__ void contrib_hit(bool touch, bool blend, float w, uint32_t gid, const ContribOut &co)
{
    const uint32_t b = __ballot_sync(FULL, touch);
    if (b == 0u) return;
    const uint32_t mx = __reduce_max_sync(FULL, blend ? __float_as_uint(w) : 0u);
    const uint32_t sm = __reduce_add_sync(FULL, blend ? __float2uint_rn(fmul(w, 16777216.0f)) : 0u);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(co.touches + gid, (uint32_t)__popc(b));
        if (mx != 0u) {
            atomicMax(co.weight_max + gid, mx);
            atomicAdd(reinterpret_cast<unsigned long long *>(co.weight_sum) + gid, (unsigned long long)sm);
        }
    }
}

// Geometry outputs of a forward pixel (DESIGN.md section 2): the depth second moment, and the depth and 1-based list position
// of the median entry (0 = none).
struct GeoPixel {
    float M2, med;
    uint32_t mpos;
};

// CONTRIB: the contribution variant also folds the hit into the scores of Gaussian gid (contrib_hit); the pixel's update is
// the same code.
// NRM (normal maps, DESIGN.md section 2): the hit's normal n (its slab word ns) is accumulated as N_c = fma(n_c, w, N_c) under
// the colour's predicate.
// GEO (geometry outputs, DESIGN.md section 2): M2 = fma(d*d, w, M2) under the colour's predicate, and a blend whose transmittance
// before blending is > 0.5 becomes the median (the last such blend wins).
template <bool CONTRIB, bool NRM, bool GEO>
__device__ __forceinline__ void fwd_blend_hit(const float4 *s, float fpx, float fpy, FwdPixel &p, uint32_t gid, const float4 *ns,
                                              float *N, GeoPixel &gp, const FwdFeatures<CONTRIB, NRM, GEO> &f)
{
    const float4 g0 = s[0], q1 = s[1], q2 = s[2];
    const float dx = fsub(g0.x, fpx), dy = fsub(g0.y, fpy);
    const float power = power_prescaled(q1.x, q1.y, q1.z, dx, dy);
    const float alpha = fminf(GS_ALPHA_MAX, fmul(q1.w, gs_exp(power)));
    const float test_T = fmul(p.T, fsub(1.0f, alpha)); // <= 0 once the pixel is done
    const bool hit = !(power > 0.0f) & !(alpha < GS_ALPHA_MIN);
    const bool blend = hit & !(test_T < GS_T_MIN);
    const float w = fmul(alpha, p.T);
    const bool live = p.T > 0.0f; // (read before the update)
    if (blend) {
        p.C0 = ffma(q2.x, w, p.C0); p.C1 = ffma(q2.y, w, p.C1); p.C2 = ffma(q2.z, w, p.C2);
        p.Dd = ffma(q2.w, w, p.Dd);
        p.Aa = fadd(p.Aa, w);
        p.last = __float_as_uint(g0.z);
        p.used |= __float_as_uint(g0.w);
    }
    if (NRM) {
        const float4 n = *ns;
        if (blend) { N[0] = ffma(n.x, w, N[0]); N[1] = ffma(n.y, w, N[1]); N[2] = ffma(n.z, w, N[2]); }
    }
    if (GEO) { // (p.T is still the transmittance before this hit; a finished pixel's is <= 0)
        if (blend) gp.M2 = ffma(fmul(q2.w, q2.w), w, gp.M2);
        if (blend & (p.T > 0.5f)) { gp.med = q2.w; gp.mpos = __float_as_uint(g0.z); }
    }
    p.T = blend ? test_T : (hit ? -fabsf(p.T) : p.T);
    if constexpr (CONTRIB) contrib_hit(hit & live, blend, w, gid, f.co);
}

// Blends the cnt hits staged in slab s, in order, two per iteration.  gids: the hits' Gaussian indices (CONTRIB only).
// NRM: ns holds the hits' normals, N the pixel's three normal sums.  GEO: gp is the pixel's geometry state.
template <bool CONTRIB, bool NRM, bool GEO>
__device__ __forceinline__ void fwd_blend_slab(const float4 *s, int cnt, float fpx, float fpy, FwdPixel &p, const uint32_t *gids,
                                               const float4 *ns, float *N, GeoPixel &gp, const FwdFeatures<CONTRIB, NRM, GEO> &f)
{
    const float4 *const end2 = s + 3 * (cnt & ~1);
#pragma unroll 1
    for (; s != end2; s += 6) {
        fwd_blend_hit(s, fpx, fpy, p, CONTRIB ? gids[0] : 0u, ns, N, gp, f);
        fwd_blend_hit(s + 3, fpx, fpy, p, CONTRIB ? gids[1] : 0u, NRM ? ns + 1 : ns, N, gp, f);
        if (CONTRIB) gids += 2;
        if (NRM) ns += 2;
    }
    if (cnt & 1) fwd_blend_hit(s, fpx, fpy, p, CONTRIB ? gids[0] : 0u, ns, N, gp, f);
}

// Writes the pixel's outputs (out-of-image pixels write nothing).
__device__ __forceinline__ void fwd_store_pixel(const BlendArgs &a, int v, int px, int py, const FwdPixel &p)
{
    const float T_out = fabsf(p.T);
    const size_t HW = (size_t)a.H * a.W;
    const size_t pix = (size_t)py * a.W + px;
    a.final_T[v * HW + pix] = T_out;
    a.n_contrib[v * HW + pix] = p.last;
    float *oc = a.out_color + (size_t)v * 3 * HW;
    oc[pix] = ffma(T_out, a.bg[0], p.C0);
    oc[HW + pix] = ffma(T_out, a.bg[1], p.C1);
    oc[2 * HW + pix] = ffma(T_out, a.bg[2], p.C2);
    a.out_depth[v * HW + pix] = p.Dd;
    a.out_alpha[v * HW + pix] = p.Aa;
}

// The body of the F6 kernel.  CONTRIB (contribution scores, DESIGN.md section 2): compaction also writes each hit's Gaussian
// index (record index - v*P) into the warp's 32-word gid_slabs row, and every hit is folded into f.co; everything else is the
// same code.
// NRM (normal maps, DESIGN.md section 2): hit lanes also gather gauss_normals[record index] into the warp's 32-entry nrm_slabs
// row, the pixel keeps three normal sums, and the pixel writes them to out_normal [V,3,H,W].
// GEO (geometry outputs, DESIGN.md section 2): the pixel keeps M2 and the median (GeoPixel) and writes them to geo's images and
// median_pos.
// A feature's shared arrays are declared in every instantiation; one that never touches them allocates no shared memory for
// them.
template <bool CONTRIB, bool NRM, bool GEO>
__device__ __forceinline__ void blend_fwd_body(const BlendArgs &a, const FwdFeatures<CONTRIB, NRM, GEO> &f)
{
    __shared__ uint32_t gid_slabs[WARPS_PER_CTA][32]; // CONTRIB
    __shared__ float4 nrm_slabs[WARPS_PER_CTA][32];   // NRM
    __shared__ WarpSlab slabs[WARPS_PER_CTA];

    const int ntiles = a.grid_x * a.grid_y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // CTAs are dispatched in blockIdx order; tile_order lists (view, tile) pairs longest list first, so the heavy
    // tiles of a launch start first and the short ones fill in behind them (LPT schedule)
    const uint32_t vt = a.tile_order[blockIdx.x / CTAS_PER_TILE];
    const int v = (int)(vt / (uint32_t)ntiles), tile = (int)(vt % (uint32_t)ntiles);
    const int patch = (blockIdx.x % CTAS_PER_TILE) * WARPS_PER_CTA + warp; // 0..7: bit0 = x half, bits 1-2 = row band
    const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
    const int x0 = tile_x * GS_TILE + (patch & 1) * 8, y0 = tile_y * GS_TILE + (patch >> 1) * 4;
    const int px = x0 + (lane & 7), py = y0 + (lane >> 3);
    const bool inside = px < a.W && py < a.H;
    const float fpx = (float)px, fpy = (float)py, fx0 = (float)x0, fy0 = (float)y0, fx1 = fx0 + 7.0f, fy1 = fy0 + 3.0f;
    float4 *const slab = slabs[warp].rec;

    const uint2 range = a.ranges[(size_t)v * ntiles + tile];
    const int n_total = (int)(range.y - range.x);
    const float4 *recs4 = reinterpret_cast<const float4 *>(a.recs);
    const uint32_t *plist = a.point_list + range.x;
    const uint32_t lt = (1u << lane) - 1u, bit = 1u << lane;
    // contributor mask of chunk c (list positions [32c, 32c+32)) of this patch: cmask[8c]
    uint32_t *const cmask = a.cmask + ((size_t)(range.x >> 5) + vt) * 8 + patch;

    FwdPixel p = {inside ? 1.0f : 0.0f, 0.f, 0.f, 0.f, 0.f, 0.f, 0u, 0u};
    float N[3] = {0.f, 0.f, 0.f};
    GeoPixel gp = {0.f, 0.f, 0u};

    // software pipeline, two deep: while chunk c is blended the support boxes of chunk c+1 and the ids of chunk c+2
    // are in flight (the id -> record address dependency never sits on the critical path)
    uint32_t id_c = 0, id_n = 0;
    float4 g0_c = make_float4(0.f, 0.f, -1.f, -1.f);
    if (lane < n_total) id_c = __ldg(plist + lane);
    if (32 + lane < n_total) id_n = __ldg(plist + 32 + lane);
    if (lane < n_total) g0_c = __ldg(recs4 + 3 * (size_t)id_c);
    uint32_t *cm = cmask;
    for (int base = 0; base < n_total; base += 32, cm += 8) {
        // Chunks after this exit get no mask word.  The backward reads chunks up to (max n_contrib of the patch - 1) / 32
        // only, and that position was blended by a pixel of the patch before every pixel was done, so those were written.
        if (__all_sync(FULL, !(p.T > 0.0f))) break;
        const bool hit = box_hits_patch(g0_c, fx0, fy0, fx1, fy1);
        const uint32_t b = __ballot_sync(FULL, hit);
        float4 g1, g2, gn;
        if (hit) {
            g1 = __ldg(recs4 + 3 * (size_t)id_c + 1);
            g2 = __ldg(recs4 + 3 * (size_t)id_c + 2);
            if constexpr (NRM) gn = __ldg(f.gauss_normals + id_c);
        }
        const float4 g0_h = g0_c;
        const uint32_t id_h = id_c;
        id_c = id_n;
        g0_c = make_float4(0.f, 0.f, -1.f, -1.f);
        if (base + 32 + lane < n_total) g0_c = __ldg(recs4 + 3 * (size_t)id_c);
        if (base + 64 + lane < n_total) id_n = __ldg(plist + base + 64 + lane);
        uint32_t m = 0u;
        if (b != 0u) {
            if (hit) {
                float4 *const s = slab + 3 * __popc(b & lt);
                s[0] = make_float4(g0_h.x, g0_h.y, __uint_as_float((uint32_t)(base + lane + 1)), __uint_as_float(bit));
                s[1] = make_float4(fmul(-0.5f, g1.x), -g1.y, fmul(-0.5f, g1.z), g1.w);
                s[2] = g2;
                if (CONTRIB) gid_slabs[warp][__popc(b & lt)] = id_h - (uint32_t)v * (uint32_t)a.P;
                if constexpr (NRM) nrm_slabs[warp][__popc(b & lt)] = gn;
            }
            __syncwarp();
            p.used = 0u;
            fwd_blend_slab(slab, __popc(b), fpx, fpy, p, gid_slabs[warp], nrm_slabs[warp], N, gp, f);
            m = __reduce_or_sync(FULL, p.used);
            __syncwarp();
        }
        if (lane == 0) *cm = m;
    }
    if (inside) {
        fwd_store_pixel(a, v, px, py, p);
        if constexpr (NRM) {
            const size_t HW = (size_t)a.H * a.W, pix = (size_t)py * a.W + px;
            float *on = f.out_normal + (size_t)v * 3 * HW + pix;
            on[0] = N[0]; on[HW] = N[1]; on[2 * HW] = N[2];
        }
        if constexpr (GEO) {
            const size_t i = (size_t)v * a.H * a.W + (size_t)py * a.W + px;
            f.geo.out_median[i] = gp.med;
            f.geo.out_depth2[i] = gp.M2;
            f.geo.median_pos[i] = gp.mpos;
        }
    }
}

// F6.  The body stays a function of its own, inlined here: the compiler then optimises it before it reaches the kernel, which
// keeps ptxas's register assignment of the feature instantiations as DESIGN.md section 5 lists them (written as the kernel
// itself, the NRM and GEO instantiations come out with some registers renamed).
template <bool CONTRIB, bool NRM, bool GEO>
__global__ void __launch_bounds__(32 * WARPS_PER_CTA, CONTRIB || NRM || GEO ? FWD_FEATURE_MIN_BLOCKS : FWD_MIN_BLOCKS)
    blend_fwd_kernel(BlendArgs a, FwdFeatures<CONTRIB, NRM, GEO> f)
{
    blend_fwd_body(a, f);
}

int blend_caps()
{
    return BLEND_CAP_CONTRIB | BLEND_CAP_NORMALS | BLEND_CAP_GEOMETRY | BLEND_CAP_ABSGRAD | BLEND_CAP_DETERMINISTIC;
}

// Calls k(std::true_type{}) or k(std::false_type{}) as f is set: the launchers turn each option bit into a template argument
// with it, so the instantiation an option set selects is spelled in one place.
template <class K> static void with_flag(bool f, K &&k)
{
    if (f) k(std::true_type{});
    else k(std::false_type{});
}

void launch_blend_fwd(const BlendArgs &a, const ContribOut *co, const float4 *gauss_normals, float *out_normal, const GeoFwd *g,
                      cudaStream_t st)
{
    const unsigned grid = (unsigned)(a.grid_x * a.grid_y * CTAS_PER_TILE * a.V);
    auto launch = [&](auto C, auto N, auto G) {
        FwdFeatures<C, N, G> f;
        if constexpr (C) f.co = *co;
        if constexpr (N) { f.gauss_normals = gauss_normals; f.out_normal = out_normal; }
        if constexpr (G) f.geo = *g;
        blend_fwd_kernel<C, N, G><<<grid, 32 * WARPS_PER_CTA, 0, st>>>(a, f);
    };
    // contribution scores never come with normals or geometry (read_opts refuses the combination)
    if (co) launch(std::true_type{}, std::false_type{}, std::false_type{});
    else with_flag(gauss_normals, [&](auto N) { with_flag(g, [&](auto G) { launch(std::false_type{}, N, G); }); });
}

// ------------------------------------------------------------------------------------------------
// B1
// ------------------------------------------------------------------------------------------------
// The hit loop parks every pixel's (q, w) of a hit here instead of reducing across lanes once per hit.  A flush then sums
// BWD_PARK parked hits at once with a lane per (hit, block of BWD_PARK pixels), so no value crosses a lane until the
// (32 / BWD_PARK)-lane exchange that ends the flush.
#define PARK_LANES (32 / BWD_PARK) // lanes that share one parked hit in the flush
struct __align__(16) WarpPark {
    float2 qw[BWD_PARK][33];     // (q, w) of park slot s at pixel p.  Rows are padded to 33 so that both the lane-per-pixel
                                 // STS.64 of the hit loop and the lane-per-slot LDS.64 of the flush are free of bank conflicts
    float4 pix[32 + PARK_LANES]; // (gC0, gC1, gC2, gD) of pixel p at pix[p + p / BWD_PARK]: the PARK_LANES pixels one flush
                                 // step reads lie in distinct banks
    float4 hit[BWD_PARK];        // slot s: the hit's slab word 0 (px, py, list position, record index)
};
// vector atomic adds without a return value (sm_90): a 16-byte (or 8-byte) aligned run of floats in one L2 request
__device__ __forceinline__ void red_add_v4(float *p, float a, float b, float c, float d)
{
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void red_add_v2(float *p, float a, float b)
{
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// The backward's feature arguments, laid out as FwdFeatures: the deterministic flush's slots, normals, geometry gradients.
// ABS has no argument of its own.
template <bool> struct BwdDetArg {};
template <> struct BwdDetArg<true> { DetFlush det; };
template <bool> struct BwdNrmArg {};
template <> struct BwdNrmArg<true> { NrmBwd nrm; };
template <bool> struct BwdGeoArg {};
template <> struct BwdGeoArg<true> { GeoBwd geo; };
template <bool DET, bool NRM, bool GEO> struct BwdFeatures : BwdDetArg<DET>, BwdNrmArg<NRM>, BwdGeoArg<GEO> {};

// Sums the first n park slots into ScreenGrad.  Lane l takes slot h = l % BWD_PARK over the pixels
// [BWD_PARK*part, BWD_PARK*part + BWD_PARK), part = l / BWD_PARK: BWD_PARK / 8 rows of the 8x4 patch.  Within a row dy is
// constant, so the row accumulates sum q, sum q*dx, sum q*dx^2 and folds dy in once per row; dx and dy are the hit loop's
// expressions.  The parts' sums meet in a (32 / BWD_PARK)-lane exchange, and the lanes of slot h write its record with a
// v4 + v4 + v2 of vector REDs.
// DET (the deterministic backward, DESIGN.md section 5): the ten sums are this (instance, patch)'s partial; they are stored
// with plain stores into its own 40-byte slot of det.partials, slot = base[j] - popc(pm[j] >> patch) (base is the inclusive
// scan of popc(pm)), and det_reduce_kernel adds each Gaussian's partials in a fixed order.
// The tile's range.x and the warp's patch are re-derived here from the kernel parameters (two cached loads per flush), not
// kept live across the hit loop: at the 64-register cap that costs the default kernel nothing and keeps this one from spilling.
// ABS (absolute screen-space gradients, DESIGN.md section 2): the flush also forms Ax = sum |q (A dx + B dy)| and
// Ay = sum |q (B dx + C dy)| over the slot's pixels, with the record's conic (word 1, still in L1 from the hit loop's staging
// load); B dy and C dy are folded once per row.  They go to ScreenGrad's padding (the third RED becomes a v4), or in
// deterministic mode to the partial's own float2 of det.abs_partials.  The ten sums are formed exactly as without ABS.
// NRM (normal maps, DESIGN.md section 2): the flush also sums Wn = sum w * dL/dN over the slot's pixels, dL/dN from the
// warp's second pixel table npix (laid out as pk.pix).  Atomic mode adds (Wn, 0) to nrm.wn[record] with one more v4 RED;
// deterministic mode stores it to nrm.partials[slot].  Everything else is formed exactly as without NRM.
// GEO (geometry outputs, DESIGN.md section 2): the flush also sums Wm = sum w * dL/dM2 and Md = the dL/dmedian of the slot's
// median pixels (the hit loop's ballot gmed[h], bit p = pixel p), both from the warp's pixel table gpix (laid out as pk.pix),
// and each part adds 2d * Wm + Md to its W3 before the exchange, d the record's depth (word 11, an L1 hit as the conic is).
// The depth gradient then reaches the mean through B2's existing depth term; everything else is formed exactly as without GEO.
template <bool ABS, bool DET, bool NRM, bool GEO>
__device__ __forceinline__ void park_flush(const WarpPark &pk, int n, int lane, float fx0, float fy_part, float *sgrad,
                                           const BlendBwdArgs &a, const BwdFeatures<DET, NRM, GEO> &f, const float4 *npix,
                                           const float2 *gpix, const uint32_t *gmed)
{
    __syncwarp();
    const int h = lane % BWD_PARK, part = lane / BWD_PARK;
    const float4 s = pk.hit[h];
    float4 conic = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ABS && h < n) conic = __ldg(reinterpret_cast<const float4 *>(a.recs) + 3 * (size_t)__float_as_uint(s.w) + 1);
    uint32_t mb = 0u;
    float Wm = 0.f, Md = 0.f;
    if (GEO) mb = gmed[h];
    float dxk[8];
#pragma unroll
    for (int k = 0; k < 8; k++) dxk[k] = fsub(s.x, fadd(fx0, (float)k));
    float S0 = 0.f, Sx = 0.f, Sy = 0.f, Sxx = 0.f, Sxy = 0.f, Syy = 0.f, W0 = 0.f, W1 = 0.f, W2 = 0.f, W3 = 0.f;
    float Ax = 0.f, Ay = 0.f, N0 = 0.f, N1 = 0.f, N2 = 0.f;
#pragma unroll
    for (int r = 0; r < BWD_PARK / 8; r++) {
        const int p0 = BWD_PARK * part + 8 * r; // first pixel of the row
        float Bdy = 0.f, Cdy = 0.f;
        if (ABS) {
            const float dy = fsub(s.y, fadd(fy_part, (float)r));
            Bdy = conic.y * dy;
            Cdy = conic.z * dy;
        }
        float R0 = 0.f, Rx = 0.f, Rxx = 0.f;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const float2 v = pk.qw[h][p0 + k];
            const float4 g = pk.pix[p0 + k + part];
            const float qx = v.x * dxk[k];
            R0 += v.x;
            Rx += qx;
            Rxx = fmaf(qx, dxk[k], Rxx);
            W0 = fmaf(v.y, g.x, W0); W1 = fmaf(v.y, g.y, W1); W2 = fmaf(v.y, g.z, W2); W3 = fmaf(v.y, g.w, W3);
            if (ABS) {
                Ax += fabsf(v.x * fmaf(conic.x, dxk[k], Bdy));
                Ay += fabsf(v.x * fmaf(conic.y, dxk[k], Cdy));
            }
            if (NRM) {
                const float4 gn = npix[p0 + k + part];
                N0 = fmaf(v.y, gn.x, N0); N1 = fmaf(v.y, gn.y, N1); N2 = fmaf(v.y, gn.z, N2);
            }
            if (GEO) {
                const float2 gg = gpix[p0 + k + part];
                Wm = fmaf(v.y, gg.x, Wm);
                if ((mb >> (p0 + k)) & 1u) Md += gg.y;
            }
        }
        const float dy = fsub(s.y, fadd(fy_part, (float)r));
        const float qy = R0 * dy;
        S0 += R0; Sx += Rx; Sxx += Rxx; Sy += qy;
        Sxy = fmaf(Rx, dy, Sxy);
        Syy = fmaf(qy, dy, Syy);
    }
    if (GEO && h < n) {
        const float d = __ldg(reinterpret_cast<const float *>(a.recs) + 12 * (size_t)__float_as_uint(s.w) + 11);
        W3 += fmaf(d + d, Wm, Md);
    }
#pragma unroll
    for (int o = BWD_PARK; o < 32; o <<= 1) {
        S0 += __shfl_xor_sync(FULL, S0, o); Sx += __shfl_xor_sync(FULL, Sx, o); Sy += __shfl_xor_sync(FULL, Sy, o);
        Sxx += __shfl_xor_sync(FULL, Sxx, o); Sxy += __shfl_xor_sync(FULL, Sxy, o); Syy += __shfl_xor_sync(FULL, Syy, o);
        W0 += __shfl_xor_sync(FULL, W0, o); W1 += __shfl_xor_sync(FULL, W1, o); W2 += __shfl_xor_sync(FULL, W2, o);
        W3 += __shfl_xor_sync(FULL, W3, o);
        if (ABS) { Ax += __shfl_xor_sync(FULL, Ax, o); Ay += __shfl_xor_sync(FULL, Ay, o); }
        if (NRM) { N0 += __shfl_xor_sync(FULL, N0, o); N1 += __shfl_xor_sync(FULL, N1, o); N2 += __shfl_xor_sync(FULL, N2, o); }
    }
    if constexpr (DET) {
        if (h < n) {
            // partial as S0, Sx | Sy, Sxx | Sxy, Syy | w.gC0, w.gC1 | w.gC2, w.gD: 40 bytes, 8-byte aligned
            const uint32_t range_x = __ldg(&a.ranges[__ldg(a.tile_order + blockIdx.x / CTAS_PER_TILE)].x);
            const int patch = (blockIdx.x % CTAS_PER_TILE) * WARPS_PER_CTA + (threadIdx.x >> 5);
            const uint32_t j = range_x + __float_as_uint(s.z);
            const uint32_t slot = __ldg(f.det.base + j) - (uint32_t)__popc((uint32_t)__ldg(f.det.pm + j) >> patch);
            float2 *rec = reinterpret_cast<float2 *>(f.det.partials + (size_t)slot * DET_PARTIAL_FLOATS);
            if (part == 0) { rec[0] = make_float2(S0, Sx); rec[1] = make_float2(Sy, Sxx); }
            if (part == 1) { rec[2] = make_float2(Sxy, Syy); rec[3] = make_float2(W0, W1); }
            if (part == (PARK_LANES > 2 ? 2 : 0)) {
                rec[4] = make_float2(W2, W3);
                if (ABS) f.det.abs_partials[slot] = make_float2(Ax, Ay);
            }
            if constexpr (NRM) {
                if (part == 1) f.nrm.partials[slot] = make_float4(N0, N1, N2, 0.f);
            }
        }
    } else if (h < n) {
        // ScreenGrad as moments: S0, Sx, Sy, Sxx | Sxy, Syy, w.gC0, w.gC1 | w.gC2, w.gD (| Ax, Ay in the padding with ABS)
        float *rec = sgrad + (size_t)__float_as_uint(s.w) * (sizeof(ScreenGrad) / sizeof(float));
        if (part < 2) {
            const bool hi = part == 1;
            red_add_v4(rec + (hi ? 4 : 0), hi ? Sxy : S0, hi ? Syy : Sx, hi ? W0 : Sy, hi ? W1 : Sxx);
        }
        if (part == (PARK_LANES > 2 ? 2 : 0)) {
            if (ABS) red_add_v4(rec + 8, W2, W3, Ax, Ay);
            else red_add_v2(rec + 8, W2, W3);
        }
        if constexpr (NRM) {
            if (part == 1) red_add_v4(reinterpret_cast<float *>(f.nrm.wn + __float_as_uint(s.w)), N0, N1, N2, 0.f);
        }
    }
    __syncwarp();
}

// B1: DET selects the flush (vector REDs into ScreenGrad, or stores of per-(instance, patch) partials
// into their slots of f.det), ABS adds the absolute sums to it; everything else is the same code.
// NRM (normal maps): contributing lanes also stage gauss_normals[record] in the warp's nslab row, the pixel's dL/dN goes to
// the second pixel table npix, cg gains n . dL/dN, and the flush sums Wn (park_flush).
// GEO (geometry outputs): the pixel's (dL/dM2, dL/dmedian) go to the pixel table gpix, cg gains d^2 * dL/dM2, every parked hit
// ballots the lanes whose median it is into gmed[slot], and the flush folds both depth terms into W3 (park_flush).
// A feature's shared arrays are declared in every instantiation; one that never touches them allocates no shared memory for
// them.
template <bool DET, bool ABS, bool NRM, bool GEO>
__global__ void __launch_bounds__(32 * WARPS_PER_CTA, BWD_MIN_BLOCKS) blend_bwd_kernel(BlendBwdArgs a, BwdFeatures<DET, NRM, GEO> f)
{
    __shared__ float2 gpix[WARPS_PER_CTA][32 + PARK_LANES]; // GEO
    __shared__ uint32_t gmed[WARPS_PER_CTA][BWD_PARK];      // GEO
    __shared__ float4 nslab[WARPS_PER_CTA][32];             // NRM
    __shared__ float4 npix[WARPS_PER_CTA][32 + PARK_LANES]; // NRM
    __shared__ WarpSlab slabs[WARPS_PER_CTA];
    __shared__ WarpPark parks[WARPS_PER_CTA];

    const int ntiles = a.grid_x * a.grid_y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // CTAs are dispatched in blockIdx order; tile_order lists (view, tile) pairs longest list first, so the heavy
    // tiles of a launch start first and the short ones fill in behind them (LPT schedule)
    const uint32_t vt = a.tile_order[blockIdx.x / CTAS_PER_TILE];
    const int v = (int)(vt / (uint32_t)ntiles), tile = (int)(vt % (uint32_t)ntiles);
    const int patch = (blockIdx.x % CTAS_PER_TILE) * WARPS_PER_CTA + warp; // 0..7: bit0 = x half, bits 1-2 = row band
    const int tile_x = tile % a.grid_x, tile_y = tile / a.grid_x;
    const int x0 = tile_x * GS_TILE + (patch & 1) * 8, y0 = tile_y * GS_TILE + (patch >> 1) * 4;
    const int px = x0 + (lane & 7), py = y0 + (lane >> 3);
    const bool inside = px < a.W && py < a.H;
    const float fpx = (float)px, fpy = (float)py;
    WarpSlab &sl = slabs[warp];
    WarpPark &pk = parks[warp];
    const uint2 range = a.ranges[(size_t)v * ntiles + tile];
    const float4 *recs4 = reinterpret_cast<const float4 *>(a.recs);
    const uint32_t *plist = a.point_list + range.x;
    const uint32_t *const cmask = a.cmask + ((size_t)(range.x >> 5) + vt) * 8 + patch; // the forward's word of chunk c: cmask[8c]
    const size_t HW = (size_t)a.H * a.W;
    const size_t pix = (size_t)py * a.W + px;
    const uint32_t lt = (1u << lane) - 1u;

    float T_final = 1.f, gC0 = 0.f, gC1 = 0.f, gC2 = 0.f, gD = 0.f, gA = 0.f;
    float4 gN = make_float4(0.f, 0.f, 0.f, 0.f);
    float gM2 = 0.f, gMed = 0.f;
    uint32_t mpos = 0u; // 1-based list position of the pixel's median entry (0: none)
    int last = 0;
    if (inside) {
        T_final = a.final_T[v * HW + pix];
        last = (int)a.n_contrib[v * HW + pix];
        if (a.dL_dcolor) {
            const float *g = a.dL_dcolor + (size_t)v * 3 * HW;
            gC0 = g[pix]; gC1 = g[HW + pix]; gC2 = g[2 * HW + pix];
        }
        if (a.dL_ddepth) gD = a.dL_ddepth[v * HW + pix];
        if (a.dL_dalpha) gA = a.dL_dalpha[v * HW + pix];
        if constexpr (NRM) {
            const float *g = f.nrm.dL_dnormal + (size_t)v * 3 * HW;
            gN = make_float4(g[pix], g[HW + pix], g[2 * HW + pix], 0.f);
        }
        if constexpr (GEO) {
            if (f.geo.dL_ddepth2) gM2 = f.geo.dL_ddepth2[v * HW + pix];
            if (f.geo.dL_dmedian) gMed = f.geo.dL_dmedian[v * HW + pix];
            mpos = f.geo.median_pos[v * HW + pix];
        }
    }
    int wmax = last; // list positions at or beyond the patch's largest n_contrib cannot contribute here
    wmax = max(wmax, __shfl_xor_sync(FULL, wmax, 16));
    wmax = max(wmax, __shfl_xor_sync(FULL, wmax, 8));
    wmax = max(wmax, __shfl_xor_sync(FULL, wmax, 4));
    wmax = max(wmax, __shfl_xor_sync(FULL, wmax, 2));
    wmax = max(wmax, __shfl_xor_sync(FULL, wmax, 1));
    if (wmax == 0) return;

    const float bg_dot = a.bg[0] * gC0 + a.bg[1] * gC1 + a.bg[2] * gC2;
    pk.pix[lane + lane / BWD_PARK] = make_float4(gC0, gC1, gC2, gD); // read by the flushes, after their __syncwarp
    if (NRM) npix[warp][lane + lane / BWD_PARK] = gN;
    if (GEO) gpix[warp][lane + lane / BWD_PARK] = make_float2(gM2, gMed);
    int np = 0;                                                      // park slots in use (warp-uniform)
    const float fx0 = (float)x0, fy_part = (float)(y0 + (lane / BWD_PARK) * (BWD_PARK / 8)); // the flush lane's first row
    float *const sgrad = reinterpret_cast<float *>(a.sgrad);
    // Per-pixel state of the back-to-front replay.  Upstream keeps five "accumulated colour behind" recurrences
    // (r,g,b,depth,alpha), each rec = last_alpha*last_c + (1-last_alpha)*rec, and forms sum_ch (c_ch - rec_ch)*g_ch.
    // The recurrences are linear with identical coefficients, so their dot product with the pixel's fixed upstream
    // gradient g = (gC, gD, gA) obeys the SAME (convex, numerically stable) recurrence as ONE scalar:
    //   cg_j = c_j.gC + depth_j*gD + gA ;   rg <- last_alpha*last_cg + (1-last_alpha)*rg ;
    //   dL/dalpha_j = T_j*(cg_j - rg) - T_final*(bg.gC)/(1-alpha_j)
    float T = T_final;
    const float Kbg = T_final * bg_dot;
    float rg = 0.f, last_cg = 0.f, last_alpha = 0.f;

    // Back to front over the forward's chunk grid, from the chunk that holds position wmax-1 (the forward wrote every
    // chunk up to it).  Lane l <-> entry 31-l of a chunk, so slots fill in descending list position.  Pipeline: the mask
    // word of chunk c-2 and the ids of chunk c-1 are in flight while chunk c is blended; a zero chunk costs no id or
    // record load.
    int c = (wmax - 1) >> 5;
    uint32_t mr_c = __brev(__ldg(cmask + 8 * (size_t)c)); // bit l: entry 31-l of chunk c contributes to the patch
    uint32_t m_n = c >= 1 ? __ldg(cmask + 8 * (size_t)(c - 1)) : 0u;
    uint32_t id_c = 0;
    if ((mr_c >> lane) & 1u) id_c = __ldg(plist + (32 * c + 31 - lane));
    for (; c >= 0; c--) {
        const uint32_t mr = mr_c, id_h = id_c;
        mr_c = __brev(m_n);
        m_n = c >= 2 ? __ldg(cmask + 8 * (size_t)(c - 2)) : 0u;
        if ((mr_c >> lane) & 1u) id_c = __ldg(plist + (32 * (c - 1) + 31 - lane));
        if (mr == 0u) continue;
        if ((mr >> lane) & 1u) {
            const float4 *rec = recs4 + 3 * (size_t)id_h;
            const float4 g0 = __ldg(rec), g1 = __ldg(rec + 1), g2 = __ldg(rec + 2);
            const int s = __popc(mr & lt);
            sl.rec[3 * s] = make_float4(g0.x, g0.y, __uint_as_float((uint32_t)(32 * c + 31 - lane)), __uint_as_float(id_h));
            sl.rec[3 * s + 1] = make_float4(fmul(-0.5f, g1.x), -g1.y, fmul(-0.5f, g1.z), g1.w);
            sl.rec[3 * s + 2] = g2;
            if constexpr (NRM) nslab[warp][s] = __ldg(f.nrm.gauss_normals + id_h);
        }
        __syncwarp();
        // The chunk's hits in runs that end at the next flush: one counter (np, the park slot) per hit, and the slab, park
        // and slot-table addresses advance as running pointers.
        const float4 *s = sl.rec;
        const float4 *ns = nslab[warp];
        for (int left = __popc(mr); left > 0;) {
            const int run = min(left, BWD_PARK - np);
            left -= run;
            float2 *pq = &pk.qw[np][lane];
            for (const int stop = np + run; np < stop; np++, s += 3, pq += 33) {
                const float4 g0 = s[0], q1 = s[1], q2 = s[2];
                const int pos = (int)__float_as_uint(g0.z); // 0-based position in the tile list
                const float dx = fsub(g0.x, fpx), dy = fsub(g0.y, fpy);
                const float power = power_prescaled(q1.x, q1.y, q1.z, dx, dy);
                const float G = gs_exp(power);
                const float alpha = fminf(GS_ALPHA_MAX, fmul(q1.w, G));
                const bool contrib = (pos < last) & !(power > 0.0f) & !(alpha < GS_ALPHA_MIN);
                // (every entry the contributor mask staged has a contributing lane: no vote.)  The pixel's update is
                // computed on every lane and selected: a lane that does not contribute keeps T, rg, last_cg and last_alpha
                // and parks (0, 0).
                float cg = fmaf(q2.x, gC0, fmaf(q2.y, gC1, fmaf(q2.z, gC2, fmaf(q2.w, gD, gA))));
                if (NRM) { // cg += n . dL/dN, components 2, 1, 0 (the normal image has no background term)
                    const float4 n = *ns++;
                    cg = fmaf(n.x, gN.x, fmaf(n.y, gN.y, fmaf(n.z, gN.z, cg)));
                }
                if (GEO) cg = fmaf(fmul(q2.w, q2.w), gM2, cg); // cg += d^2 dL/dM2 (no background term either)
                const float one_m_a = 1.0f - alpha;
                float inv; // 1/(1-alpha), 1-alpha in [0.01, 1) where the lane contributes
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"(one_m_a));
#if BWD_T_DIV == 2
                const float Tc = __fdiv_rn(T, one_m_a); // the oracle's operation, bit for bit
#elif BWD_T_DIV == 1
                inv = fmaf(fmaf(-one_m_a, inv, 1.0f), inv, inv); // one Newton step: removes the MUFU reciprocal's bias, which a
                const float Tc = T * inv;                         // list thousands of contributors deep would otherwise compound
#else
                const float Tc = T * inv;
#endif
                const float rgc = fmaf(last_alpha, last_cg - rg, rg);
                const float dL_dalpha = fmaf(Tc, cg - rgc, -(Kbg * inv));
                T = contrib ? Tc : T;
                rg = contrib ? rgc : rg;
                last_cg = contrib ? cg : last_cg;
                last_alpha = contrib ? alpha : last_alpha;
                // park (q, w); the flush forms the six moments of q over the patch (1, dx, dy, dx^2, dx*dy, dy^2; the conic /
                // mean combination is linear and happens once per Gaussian in B2) and the four weights of w
                *pq = contrib ? make_float2(G * dL_dalpha, alpha * Tc) : make_float2(0.f, 0.f);
                if (lane == 0) pk.hit[np] = g0;
                if (GEO) { // the lanes whose median this hit is (pos is 0-based, mpos 1-based)
                    const uint32_t mb = __ballot_sync(FULL, contrib & ((uint32_t)pos + 1u == mpos));
                    if (lane == 0) gmed[warp][np] = mb;
                }
            }
            if (np == BWD_PARK) {
                park_flush<ABS>(pk, np, lane, fx0, fy_part, sgrad, a, f, npix[warp], gpix[warp], gmed[warp]);
                np = 0;
            }
        }
        __syncwarp();
    }
    if (np > 0)
        park_flush<ABS>(pk, np, lane, fx0, fy_part, sgrad, a, f, npix[warp], gpix[warp], gmed[warp]);
}

void launch_blend_bwd(const BlendBwdArgs &a, const DetFlush *det, bool absgrad, const NrmBwd *n, const GeoBwd *g, cudaStream_t st)
{
    const unsigned grid = (unsigned)(a.grid_x * a.grid_y * CTAS_PER_TILE * a.V);
    with_flag(det, [&](auto D) { with_flag(absgrad, [&](auto A) { with_flag(n, [&](auto N) { with_flag(g, [&](auto G) {
        BwdFeatures<D, N, G> f;
        if constexpr (D) f.det = *det;
        if constexpr (N) f.nrm = *n;
        if constexpr (G) f.geo = *g;
        blend_bwd_kernel<D, A, N, G><<<grid, 32 * WARPS_PER_CTA, 0, st>>>(a, f);
    }); }); }); });
}

// dL_dmeans2D_abs of every (view, Gaussian): the padding sums (Ax, Ay) times o * W/2 and o * H/2, o the record's opacity --
// the factors B2 applies to the signed moments (preprocess.cu), both positive.  Zero where radii == 0.
__global__ void __launch_bounds__(256) absgrad_out_kernel(int64_t n_vp, int H, int W, const int32_t *__restrict__ radii,
                                                          const GeomRec *__restrict__ recs, const ScreenGrad *__restrict__ sgrad,
                                                          float *__restrict__ out)
{
    const int64_t vp = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (vp >= n_vp) return;
    float gx = 0.f, gy = 0.f;
    if (radii[vp] > 0) {
        const float o = recs[vp].o;
        const float2 s = *reinterpret_cast<const float2 *>(&sgrad[vp].pad0);
        gx = o * s.x * (0.5f * (float)W);
        gy = o * s.y * (0.5f * (float)H);
    }
    out[3 * vp] = gx; out[3 * vp + 1] = gy; out[3 * vp + 2] = 0.f;
}
void launch_absgrad_out(int64_t n_vp, int H, int W, const int32_t *radii, const GeomRec *recs, const void *sgrad, float *out,
                        cudaStream_t st)
{
    absgrad_out_kernel<<<(unsigned)((n_vp + 255) / 256), 256, 0, st>>>(n_vp, H, W, radii, recs, (const ScreenGrad *)sgrad, out);
}

// ScreenGrad holds moments of q = G*dL/dalpha here: S0, Sx, Sy, Sxx, Sxy, Syy = sum q*{1, dx, dy, dx^2, dx*dy, dy^2};
// then colour(3) and depth weights.
int blend_sgrad_is_moments() { return 1; }

__global__ void test_exp_kernel(const float *x, float *y, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = gs_exp(x[i]);
}
void launch_test_exp(const float *x, float *y, int64_t n, cudaStream_t st)
{
    test_exp_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, y, n);
}
