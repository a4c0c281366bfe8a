// preprocess.cu -- F1 (per-Gaussian forward: cull, project, 3D->2D covariance, SH -> colour) and
// B2+B3 (per-Gaussian backward: conic -> cov2D -> cov3D/mean, projection, depth, SH, scale/rotation).
// Restates SURVEY.md Appendix A.2 / A.6 / A.7; the in-tree Python statements of the same math are
//   SH basis      gaussiansplatting/utils/sh_utils.py:57-112
//   covariance    gaussiansplatting/utils/general_utils.py:64-110, scene/gaussian_model.py:27-31
//   projection    gaussiansplatting/utils/graphics_utils.py:22-30
// One thread per Gaussian; grid.y = view.  HBM-bound streaming kernels: inputs are read with
// 128-bit loads where alignment allows, outputs are written as three 16-B words per record.
#include "common.cuh"
#include "kernels.h"
#include "sh.cuh"

__device__ __forceinline__ void build_cov3d(const float *s3, float mod, const float *q, float *c6)
{
    float R[3][3];
    gs_rotmat(q, R);
    const float s[3] = {fmul(mod, s3[0]), fmul(mod, s3[1]), fmul(mod, s3[2])};
    float L[3][3];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int k = 0; k < 3; k++) L[i][k] = fmul(R[i][k], s[k]);
    c6[0] = gs_dot3(L[0][0], L[0][1], L[0][2], L[0][0], L[0][1], L[0][2]);
    c6[1] = gs_dot3(L[0][0], L[0][1], L[0][2], L[1][0], L[1][1], L[1][2]);
    c6[2] = gs_dot3(L[0][0], L[0][1], L[0][2], L[2][0], L[2][1], L[2][2]);
    c6[3] = gs_dot3(L[1][0], L[1][1], L[1][2], L[1][0], L[1][1], L[1][2]);
    c6[4] = gs_dot3(L[1][0], L[1][1], L[1][2], L[2][0], L[2][1], L[2][2]);
    c6[5] = gs_dot3(L[2][0], L[2][1], L[2][2], L[2][0], L[2][1], L[2][2]);
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(hi, max(lo, v)); }

// F1's screen-space covariance of a Gaussian (3D covariance S) in view V (A.2 step 3), in its pinned operations: ca0, cb, cc0
// before the 0.3 px^2 dilation.  The preprocess backward re-runs it for antialiasing, so that its rho is F1's bit for bit.
__device__ __forceinline__ void gs_cov2d(const float *V, const float S[3][3], float tx, float ty, float tz, float fx, float fy,
                                         float tanx, float tany, float &ca0, float &cb, float &cc0)
{
    const float limx = fmul(1.3f, tanx), limy = fmul(1.3f, tany);
    const float txtz = fdiv(tx, tz), tytz = fdiv(ty, tz);
    const float cx = fmul(fminf(limx, fmaxf(-limx, txtz)), tz);
    const float cy = fmul(fminf(limy, fmaxf(-limy, tytz)), tz);
    const float J00 = fdiv(fx, tz), J11 = fdiv(fy, tz);
    const float tz2 = fmul(tz, tz);
    const float J02 = fdiv(-fmul(fx, cx), tz2), J12 = fdiv(-fmul(fy, cy), tz2);
    float M0[3], M1[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        M0[k] = ffma(J02, V[4 * k + 2], fmul(J00, V[4 * k + 0]));
        M1[k] = ffma(J12, V[4 * k + 2], fmul(J11, V[4 * k + 1]));
    }
    float N0[3], N1[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        N0[k] = gs_dot3(M0[0], M0[1], M0[2], S[0][k], S[1][k], S[2][k]);
        N1[k] = gs_dot3(M1[0], M1[1], M1[2], S[0][k], S[1][k], S[2][k]);
    }
    ca0 = gs_dot3(N0[0], N0[1], N0[2], M0[0], M0[1], M0[2]);
    cb = gs_dot3(N0[0], N0[1], N0[2], M1[0], M1[1], M1[2]);
    cc0 = gs_dot3(N1[0], N1[1], N1[2], M1[0], M1[1], M1[2]);
}

// antialiasing's det0 / det of F1's covariance (its floor: rho = sqrt(max(2.5e-5, ratio)))
__device__ __forceinline__ float gs_aa_ratio(float ca0, float cb, float cc0)
{
    const float det = ffma(fadd(ca0, GS_DILATE), fadd(cc0, GS_DILATE), -fmul(cb, cb));
    return fdiv(ffma(ca0, cc0, -fmul(cb, cb)), det);
}

// The 3D smoothing filter (DESIGN.md section 2) on one Gaussian's activated scales s (before scale_modifier) and variance
// v: t_i = s_i^2 + v, s'_i = sqrt(t_i), r_i = s_i^2 / t_i (1 where t_i = 0); returns coef = sqrt(r_0 r_1 r_2), the factor
// that keeps o * sqrt(det Sigma) when the opacity becomes o' = o * coef.  IEEE float32, no contraction.
__device__ __forceinline__ float gs_filter3d(float *s, float v, float *t, float *r)
{
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float s2 = fmul(s[k], s[k]);
        t[k] = fadd(s2, v);
        r[k] = t[k] > 0.0f ? fdiv(s2, t[k]) : 1.0f;
        s[k] = fsqrt(t[k]);
    }
    return fsqrt(fmul(fmul(r[0], r[1]), r[2]));
}

// torch.sigmoid as torch's CUDA kernels evaluate it in float32 (F.normalize: gs_normalize4, common.cuh)
__device__ __forceinline__ float gs_sigmoid(float x) { return fdiv(1.0f, fadd(1.0f, expf(-x))); }

// ------------------------------------------------------------------------------------------------
// F1.  One thread per Gaussian; the thread loads its attributes ONCE (128-bit loads for the SH block when the
// row pitch allows), builds the 3D covariance once, then loops over the V views of the batch writing one
// 48-byte record per view.  Per step this reads P*(44+12K) bytes instead of V times that.
// DEG = -1: colours are given (colors_precomp), no SH.
// AA: the antialiasing filter (DESIGN.md section 2): the record's opacity is op * rho, rho = sqrt(det0 / det), det0 the
// determinant of the 2D covariance before the +0.3 px^2 dilation; the support box is bounded with that opacity too.
// F3D: the 3D smoothing filter, once per Gaussian before the view loop: the activated scales become s' (gs_filter3d) and the
// opacity o * coef; everything after (scale_modifier, the covariance, AA's rho, the support box) sees s' and o * coef.
// ------------------------------------------------------------------------------------------------
#ifndef PFWD_MIN_BLOCKS
#define PFWD_MIN_BLOCKS 3 // 80 registers; H100 (400 W): 2 / 4 blocks make this kernel 33 % / 26 % slower
#endif
template <int DEG, bool AA, bool F3D>
__global__ void __launch_bounds__(256, PFWD_MIN_BLOCKS) preprocess_fwd_kernel(PreArgs a, int nviews, const float *f3d_var)
{
    constexpr int NB = DEG < 0 ? 1 : (DEG + 1) * (DEG + 1);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;

    float px = __ldg(a.means + 3 * (size_t)i), py = __ldg(a.means + 3 * (size_t)i + 1), pz = __ldg(a.means + 3 * (size_t)i + 2);
    float op = __ldg(a.opac + i);
    // raw parameters (SURVEY.md 8f-1): the activations of GaussianModel's getters (gaussian_model.py:95-118) happen here,
    // with the same float operations torch's CUDA kernels use (expf; 1/(1+expf(-x)); x / max(||x||, 1e-12))
    if (a.raw) op = gs_sigmoid(op);
    float c6[6];
    if (a.cov_pre) {
#pragma unroll
        for (int k = 0; k < 6; k++) c6[k] = __ldg(a.cov_pre + 6 * (size_t)i + k);
    } else {
        float s3[3] = {__ldg(a.scales + 3 * (size_t)i), __ldg(a.scales + 3 * (size_t)i + 1),
                       __ldg(a.scales + 3 * (size_t)i + 2)};
        float q[4];
        if (a.vec16) {
            const float4 q4 = __ldg(reinterpret_cast<const float4 *>(a.rots) + i);
            q[0] = q4.x; q[1] = q4.y; q[2] = q4.z; q[3] = q4.w;
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) q[k] = __ldg(a.rots + 4 * (size_t)i + k);
        }
        if (a.raw) {
            s3[0] = expf(s3[0]); s3[1] = expf(s3[1]); s3[2] = expf(s3[2]);
            gs_normalize4(q);
        }
        if (F3D) {
            float t[3], r[3];
            op = fmul(op, gs_filter3d(s3, __ldg(f3d_var + i), t, r));
        }
        build_cov3d(s3, a.mod, q, c6);
    }
    float shc[3 * NB]; // SH coefficients [k][channel], or the precomputed colour
    if (DEG < 0) {
        shc[0] = __ldg(a.colors_pre + 3 * (size_t)i);
        shc[1] = __ldg(a.colors_pre + 3 * (size_t)i + 1);
        shc[2] = __ldg(a.colors_pre + 3 * (size_t)i + 2);
    } else {
        const float *sh = a.shs + (size_t)i * a.M * 3;
        if ((3 * NB) % 4 == 0 && (a.M & 3) == 0 && a.vec16) { // 16-byte aligned rows: 128-bit loads
            const float4 *sh4 = reinterpret_cast<const float4 *>(sh);
#pragma unroll
            for (int k = 0; k < (3 * NB) / 4; k++) {
                const float4 t = __ldg(sh4 + k);
                shc[4 * k] = t.x; shc[4 * k + 1] = t.y; shc[4 * k + 2] = t.z; shc[4 * k + 3] = t.w;
            }
        } else {
#pragma unroll
            for (int k = 0; k < 3 * NB; k++) shc[k] = __ldg(sh + k);
        }
    }
    const float S[3][3] = {{c6[0], c6[1], c6[2]}, {c6[1], c6[3], c6[4]}, {c6[2], c6[4], c6[5]}};

    for (int v = 0; v < nviews; v++) {
        const size_t vp = (size_t)v * a.P + i;
        const float *V = a.view + 16 * v, *PV = a.proj + 16 * v;
        if (a.means_view_stride && v > 0) { // animation frame batch: this view has its own positions
            const float *m = a.means + (size_t)v * a.means_view_stride + 3 * (size_t)i;
            px = __ldg(m); py = __ldg(m + 1); pz = __ldg(m + 2);
        }
        int radius = 0;
        uint32_t tiles = 0;
        uint2 rect_pack = make_uint2(0, 0);
        uint8_t clamped = 0;
        GeomRec rec;
        rec.px = rec.py = 0.f; rec.hx = rec.hy = -1.f; rec.A = rec.B = rec.C = rec.o = 0.f;
        rec.r = rec.g = rec.b = rec.depth = 0.f;

        const float tx = gs_affine(V[0], V[4], V[8], V[12], px, py, pz);
        const float ty = gs_affine(V[1], V[5], V[9], V[13], px, py, pz);
        const float tz = gs_affine(V[2], V[6], V[10], V[14], px, py, pz);
        do {
            if (!(tz > GS_NEAR_Z)) break; // near-plane cull (A.2 step 1); written so that a NaN position is culled too
            const float hx = gs_affine(PV[0], PV[4], PV[8], PV[12], px, py, pz);
            const float hy = gs_affine(PV[1], PV[5], PV[9], PV[13], px, py, pz);
            const float hw = gs_affine(PV[3], PV[7], PV[11], PV[15], px, py, pz);
            const float pw = fdiv(1.0f, fadd(hw, 0.0000001f));
            const float ndcx = fmul(hx, pw), ndcy = fmul(hy, pw);

            const float tanx = a.tanfovx[v], tany = a.tanfovy[v];
            float ca0, cb, cc0;
            gs_cov2d(V, S, tx, ty, tz, gs_focal(a.W, tanx), gs_focal(a.H, tany), tanx, tany, ca0, cb, cc0);
            const float ca = fadd(ca0, GS_DILATE);
            const float cc = fadd(cc0, GS_DILATE);
            const float det = ffma(ca, cc, -fmul(cb, cb));
            if (det == 0.0f) break;
            const float det_inv = fdiv(1.0f, det);
            const float conA = fmul(cc, det_inv), conB = fmul(-cb, det_inv), conC = fmul(ca, det_inv);
            const float mid = fmul(0.5f, fadd(ca, cc));
            const float sq = fsqrt(fmaxf(0.1f, ffma(mid, mid, -det)));
            const float lam = fmaxf(fadd(mid, sq), fsub(mid, sq));
            const int rad = (int)ceilf(fmul(3.0f, fsqrt(lam)));
            const float pxs = fmul(ffma(fadd(ndcx, 1.0f), (float)a.W, -1.0f), 0.5f);
            const float pys = fmul(ffma(fadd(ndcy, 1.0f), (float)a.H, -1.0f), 0.5f);
            const float fr = (float)rad;
            const int gx = a.grid_x, gy = a.grid_y;
            const int x0 = clampi((int)fdiv(fsub(pxs, fr), 16.0f), 0, gx);
            const int y0 = clampi((int)fdiv(fsub(pys, fr), 16.0f), 0, gy);
            const int x1 = clampi((int)fdiv(fsub(fadd(fadd(pxs, fr), 16.0f), 1.0f), 16.0f), 0, gx);
            const int y1 = clampi((int)fdiv(fsub(fadd(fadd(pys, fr), 16.0f), 1.0f), 16.0f), 0, gy);
            const int area = (x1 - x0) * (y1 - y0);
            if (area == 0) break;

            float rgb[3];
            if (DEG >= 0) {
                float dx = fsub(px, a.campos[3 * v]), dy = fsub(py, a.campos[3 * v + 1]), dz = fsub(pz, a.campos[3 * v + 2]);
                const float len = fsqrt(gs_dot3(dx, dy, dz, dx, dy, dz));
                dx = fdiv(dx, len); dy = fdiv(dy, len); dz = fdiv(dz, len);
                float bs[16];
                sh_basis(DEG, dx, dy, dz, bs);
                float acc[3] = {fmul(bs[0], shc[0]), fmul(bs[0], shc[1]), fmul(bs[0], shc[2])};
#pragma unroll
                for (int k = 1; k < NB; k++) {
                    acc[0] = ffma(bs[k], shc[3 * k], acc[0]);
                    acc[1] = ffma(bs[k], shc[3 * k + 1], acc[1]);
                    acc[2] = ffma(bs[k], shc[3 * k + 2], acc[2]);
                }
#pragma unroll
                for (int ch = 0; ch < 3; ch++) {
                    const float rr = fadd(acc[ch], 0.5f);
                    if (rr < 0.0f) clamped |= (1u << ch);
                    rgb[ch] = fmaxf(rr, 0.0f);
                }
            } else {
                rgb[0] = shc[0]; rgb[1] = shc[1]; rgb[2] = shc[2];
            }
            float oe = op; // the record's opacity
            if (AA) {
                // floor rho >= 0.005: a degenerate footprint (det0 <= 0) lands on it
                oe = fmul(op, fsqrt(fmaxf(2.5e-5f, gs_aa_ratio(ca0, cb, cc0))));
            }
            radius = rad;
            tiles = (uint32_t)area;
            rect_pack = make_uint2((uint32_t)x0 | ((uint32_t)y0 << 16), (uint32_t)x1 | ((uint32_t)y1 << 16));
            rec.px = pxs; rec.py = pys;
            rec.A = conA; rec.B = conB; rec.C = conC; rec.o = oe;
            rec.r = rgb[0]; rec.g = rgb[1]; rec.b = rgb[2]; rec.depth = tz;
            // Conservative half extents of {alpha >= 1/255}: power >= -tau, tau = ln(255*o).  Product-only
            // acceleration data (never changes a result: a pixel outside [px+-hx] x [py+-hy] has
            // alpha < 1/255 with margin far above the float error of gs_power/gs_exp; see DESIGN.md).
            {
                const float k255 = 255.0f * oe;
                const float aniso = (ca * cc) * det_inv; // 1/(1-rho^2): amplifies rounding error of power
                if (!(k255 > 1.0f)) {
                    rec.hx = rec.hy = -1.0f; // can never reach 1/255
                } else if (!(aniso < 1.0e4f)) {
                    rec.hx = rec.hy = 3.0e38f; // too ill-conditioned to bound safely: never cull
                } else {
                    const float tau = __logf(k255) * (1.0f + 4.0e-6f * aniso) + 0.02f;
                    rec.hx = sqrtf(2.0f * tau * ca) * 1.0005f + 0.02f;
                    rec.hy = sqrtf(2.0f * tau * cc) * 1.0005f + 0.02f;
                }
            }
        } while (0);

        a.radii[vp] = radius;
        a.dkeys[vp] = __float_as_uint(rec.depth); // culled: depth 0 sorts first, emits nothing
        a.order_in[vp] = (uint32_t)vp;
        a.tiles_touched[vp] = tiles;
        a.rects[vp] = rect_pack;
        a.clamped[vp] = clamped;
        float4 *dst = reinterpret_cast<float4 *>(a.recs + vp);
        dst[0] = make_float4(rec.px, rec.py, rec.hx, rec.hy);
        dst[1] = make_float4(rec.A, rec.B, rec.C, rec.o);
        dst[2] = make_float4(rec.r, rec.g, rec.b, rec.depth);
    }
}

template <bool AA, bool F3D>
static void launch_preprocess_fwd_t(const PreArgs &a, int V, const float *f3d_var, cudaStream_t st)
{
    const dim3 grid((a.P + 255) / 256);
    if (!a.shs) preprocess_fwd_kernel<-1, AA, F3D><<<grid, 256, 0, st>>>(a, V, f3d_var);
    else if (a.deg == 0) preprocess_fwd_kernel<0, AA, F3D><<<grid, 256, 0, st>>>(a, V, f3d_var);
    else if (a.deg == 1) preprocess_fwd_kernel<1, AA, F3D><<<grid, 256, 0, st>>>(a, V, f3d_var);
    else if (a.deg == 2) preprocess_fwd_kernel<2, AA, F3D><<<grid, 256, 0, st>>>(a, V, f3d_var);
    else preprocess_fwd_kernel<3, AA, F3D><<<grid, 256, 0, st>>>(a, V, f3d_var);
}
void launch_preprocess_fwd(const PreArgs &a, int V, bool aa, const float *f3d_var, cudaStream_t st)
{
    if (f3d_var) {
        if (aa) launch_preprocess_fwd_t<true, true>(a, V, f3d_var, st);
        else launch_preprocess_fwd_t<false, true>(a, V, f3d_var, st);
    } else {
        if (aa) launch_preprocess_fwd_t<true, false>(a, V, f3d_var, st);
        else launch_preprocess_fwd_t<false, false>(a, V, f3d_var, st);
    }
}

__global__ void mark_visible_kernel(int P, const float *pos, const float *V, uint8_t *present)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float tz = gs_affine(V[2], V[6], V[10], V[14], pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]);
    present[i] = tz > GS_NEAR_Z;
}
void launch_mark_visible(int P, const float *pos, const float *V, uint8_t *present, cudaStream_t st)
{
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, pos, V, present);
}

// ------------------------------------------------------------------------------------------------
// B2 + B3: one thread per Gaussian, loops over the views of the batch and SUMS parameter gradients
// (deterministic: no atomics at the parameter level).  Plain float arithmetic (tolerance-compared).
// AA: the forward's record opacity was op * rho (F1): dL/dop = rho * S0, and dL/drho = op * S0 joins the cov2D gradient.
// F3D: the view loop yields the gradients w.r.t. the filtered s' and o' = o * coef; after it, once per Gaussian,
//   dL/do = coef * g_o',  dL/ds_i = g_s'_i * s_i / s'_i + o * g_o' * sqrt(r_j r_k) * v / (t_i s'_i)
// (the second factor is dcoef/ds_i in a form without cancellation, finite at s_i = 0).  The filter's quantities are
// recomputed there from the inputs rather than held across the loop; with AA, coef stays live for the per-view o'.
// ------------------------------------------------------------------------------------------------
#ifndef PBWD_MIN_BLOCKS
#define PBWD_MIN_BLOCKS 4 // 128 registers; 5 / 6 blocks (96 / 80 registers) spill the 48 SH accumulators
#endif
template <int DEG, bool AA, bool F3D>
__global__ void __launch_bounds__(128, PBWD_MIN_BLOCKS) preprocess_bwd_kernel(PreBwdArgs a)
{
    constexpr int nb = DEG < 0 ? 1 : (DEG + 1) * (DEG + 1);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    float px = a.means[3 * (size_t)i], py = a.means[3 * (size_t)i + 1], pz = a.means[3 * (size_t)i + 2];

    float c6[6];
    float R[3][3], s[3] = {0, 0, 0}, q[4] = {0, 0, 0, 0}, qnorm = 1.0f;
    bool qproj = true; // F.normalize's Jacobian projects (||q|| >= 1e-12)
    float coef = 1.0f; // F3D: o' = o * coef
    if (a.cov_pre) {
        for (int k = 0; k < 6; k++) c6[k] = a.cov_pre[6 * (size_t)i + k];
    } else {
        float s3[3] = {a.scales[3 * (size_t)i], a.scales[3 * (size_t)i + 1], a.scales[3 * (size_t)i + 2]};
        for (int k = 0; k < 4; k++) q[k] = a.rots[4 * (size_t)i + k];
        if (a.raw) { // the same activations F1 applied
            s3[0] = expf(s3[0]); s3[1] = expf(s3[1]); s3[2] = expf(s3[2]);
            float qlen;
            qnorm = gs_normalize4(q, &qlen);
            qproj = qlen >= 1e-12f;
        }
        if (F3D) { // the same filter F1 applied: s3 becomes s'
            float t[3], r[3];
            coef = gs_filter3d(s3, a.f3d_var[i], t, r);
        }
        build_cov3d(s3, a.mod, q, c6);
        const float r = q[0], x = q[1], y = q[2], z = q[3];
        R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - r * z); R[0][2] = 2.f * (x * z + r * y);
        R[1][0] = 2.f * (x * y + r * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - r * x);
        R[2][0] = 2.f * (x * z - r * y); R[2][1] = 2.f * (y * z + r * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
        for (int k = 0; k < 3; k++) s[k] = a.mod * s3[k];
    }
    const float S[3][3] = {{c6[0], c6[1], c6[2]}, {c6[1], c6[3], c6[4]}, {c6[2], c6[4], c6[5]}};

    float dmean[3] = {0, 0, 0}, dcov[6] = {0, 0, 0, 0, 0, 0}, dop = 0.f, dcol[3] = {0, 0, 0};
    float dsh[3 * nb]; // SH gradient accumulators, in registers
#pragma unroll
    for (int k = 0; k < 3 * nb; k++) dsh[k] = 0.f;
    const float *shp = DEG >= 0 ? a.shs + (size_t)i * a.M * 3 : nullptr; // coefficients: re-read per view (12 x 16 B, L1-resident)
    const bool sh16 = DEG >= 0 && (3 * nb) % 4 == 0 && (a.M & 3) == 0 && ((((uintptr_t)a.shs) & 15) == 0);

    // Software pipeline over the views: the kernel is latency-bound (one dependent gather per view), so the radius of view
    // v+2 and the 64 bytes of per-view state of view v+1 are requested before view v is reduced.
    const float4 *sg4 = reinterpret_cast<const float4 *>(a.sgrad);
    const float4 *rc4 = reinterpret_cast<const float4 *>(a.recs);
    // the ten accumulated sums of one (view, Gaussian): 3 x 16 B of floats
    auto load_sums = [&](size_t rec, float4 &o0, float4 &o1, float4 &o2) {
        o0 = __ldg(sg4 + 3 * rec); o1 = __ldg(sg4 + 3 * rec + 1); o2 = __ldg(sg4 + 3 * rec + 2);
    };
    int rad_n = a.radii[i], rad_nn = a.V > 1 ? a.radii[(size_t)a.P + i] : 0;
    float4 n0 = make_float4(0, 0, 0, 0), n1 = n0, n2 = n0, nr = n0;
    uint8_t ncl = 0;
    if (rad_n > 0) {
        load_sums((size_t)i, n0, n1, n2);
        nr = __ldg(rc4 + 3 * (size_t)i + 1);
        ncl = a.clamped[i];
    }

    for (int v = 0; v < a.V; v++) {
        const size_t vp = (size_t)v * a.P + i;
        float *m2d = a.dL_dmeans2D + 3 * vp;
        const int rad = rad_n;
        const float4 g0 = n0, g1 = n1, g2 = n2, r1 = nr;
        const uint8_t cl = ncl;
        rad_n = rad_nn;
        rad_nn = v + 2 < a.V ? a.radii[vp + 2 * (size_t)a.P] : 0;
        if (rad_n > 0) {
            const size_t vn = vp + (size_t)a.P;
            load_sums(vn, n0, n1, n2);
            nr = __ldg(rc4 + 3 * vn + 1);
            ncl = a.clamped[vn];
        }
        if (a.means_view_stride) { // per-view positions: per-view (not summed) position gradients
            if (v > 0) {
                float *o = a.dL_dmeans3D + 3 * ((size_t)(v - 1) * a.P + i);
                o[0] = dmean[0]; o[1] = dmean[1]; o[2] = dmean[2];
                dmean[0] = dmean[1] = dmean[2] = 0.f;
                const float *m = a.means + (size_t)v * a.means_view_stride + 3 * (size_t)i;
                px = m[0]; py = m[1]; pz = m[2];
            }
        }
        if (!(rad > 0)) {
            m2d[0] = 0.f; m2d[1] = 0.f; m2d[2] = 0.f;
            continue;
        }
        float gdx, gdy, dA, dBh, dC, gO;
        if (a.moments) {
            // moments of q = G*dL/dalpha over the Gaussian's pixels -> screen-space gradients (A.5); r1 = conic A,B,C and opacity
            const float S0 = g0.x, Sx = g0.y, Sy = g0.z, Sxx = g0.w, Sxy = g1.x, Syy = g1.y;
            gO = S0;
            gdx = -r1.w * (r1.x * Sx + r1.y * Sy) * (0.5f * (float)a.W);
            gdy = -r1.w * (r1.z * Sy + r1.y * Sx) * (0.5f * (float)a.H);
            dA = -0.5f * r1.w * Sxx; dBh = -0.5f * r1.w * Sxy; dC = -0.5f * r1.w * Syy;
        } else {
            gdx = g0.x; gdy = g0.y; dA = g0.z; dBh = g0.w; dC = g1.x; gO = g1.y;
        }
        const float gcol[3] = {g1.z, g1.w, g2.x};
        const float gdepth = g2.y;
        m2d[0] = gdx; m2d[1] = gdy; m2d[2] = 0.f;
        if (!AA) dop += gO;

        const float *V = a.view + 16 * v, *PV = a.proj + 16 * v;
        const float tx = gs_affine(V[0], V[4], V[8], V[12], px, py, pz);
        const float ty = gs_affine(V[1], V[5], V[9], V[13], px, py, pz);
        const float tz = gs_affine(V[2], V[6], V[10], V[14], px, py, pz);
        const float tanx = a.tanfovx[v], tany = a.tanfovy[v];
        const float fx = (float)a.W / (2.0f * tanx), fy = (float)a.H / (2.0f * tany);
        const float limx = 1.3f * tanx, limy = 1.3f * tany;
        const float txtz = tx / tz, tytz = ty / tz;
        const float cx = fminf(limx, fmaxf(-limx, txtz)) * tz;
        const float cy = fminf(limy, fmaxf(-limy, tytz)) * tz;
        const float xmul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
        const float ymul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
        const float itz = 1.f / tz, itz2 = itz * itz, itz3 = itz2 * itz;
        const float J00 = fx * itz, J11 = fy * itz, J02 = -(fx * cx) * itz2, J12 = -(fy * cy) * itz2;
        float M0[3], M1[3], Wm[3][3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            Wm[0][k] = V[4 * k]; Wm[1][k] = V[4 * k + 1]; Wm[2][k] = V[4 * k + 2];
            M0[k] = J00 * Wm[0][k] + J02 * Wm[2][k];
            M1[k] = J11 * Wm[1][k] + J12 * Wm[2][k];
        }
        float N0[3], N1[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            N0[k] = M0[0] * S[0][k] + M0[1] * S[1][k] + M0[2] * S[2][k];
            N1[k] = M1[0] * S[0][k] + M1[1] * S[1][k] + M1[2] * S[2][k];
        }
        const float ca0 = N0[0] * M0[0] + N0[1] * M0[1] + N0[2] * M0[2];
        const float ca = ca0 + GS_DILATE;
        const float cb = N0[0] * M1[0] + N0[1] * M1[1] + N0[2] * M1[2];
        const float cc0 = N1[0] * M1[0] + N1[1] * M1[1] + N1[2] * M1[2];
        const float cc = cc0 + GS_DILATE;
        const float denom = ca * cc - cb * cb;
        const float d2inv = 1.0f / (denom * denom + 0.0000001f);
        float ra = 0.f, rb = 0.f, rc = 0.f; // AA: dL/drho * drho/d(a, b, c)
        if (AA) {
            // rho = sqrt(det0 / det), det = det0 + d (ca0 + cc0 + d), d = 0.3: the derivatives in a cancellation-free form
            //   drho/da = d (cc0 cc + b^2) / (2 rho det^2),  drho/dc = d (ca0 ca + b^2) / (2 rho det^2),
            //   drho/db = -d b (ca + cc0) / (rho det^2);  zero where the floor holds
            // rho and its floor's branch are F1's, recomputed in F1's operations: det0 is a cancellation for a needle, so a
            // ratio of this view's own rounding can land on the other side of 2.5e-5, and its rho can be off by more than itself
            float fa0, fb, fc0;
            gs_cov2d(V, S, tx, ty, tz, gs_focal(a.W, tanx), gs_focal(a.H, tany), tanx, tany, fa0, fb, fc0);
            const float ratio = gs_aa_ratio(fa0, fb, fc0);
            const float rho = fsqrt(fmaxf(2.5e-5f, ratio));
            dop += rho * gO;
            if (ratio > 2.5e-5f) {
                // the opacity before the filter (after the sigmoid for raw parameters), re-read per view (an L1 hit) rather
                // than kept live across the view loop
                const float opr = __ldg(a.opac + i);
                float op = a.raw ? gs_sigmoid(opr) : opr;
                if (F3D) op *= coef; // the opacity rho multiplied in F1 is o'
                const float k = GS_DILATE * op * gO / (rho * denom * denom);
                ra = 0.5f * k * (cc0 * cc + cb * cb);
                rc = 0.5f * k * (ca0 * ca + cb * cb);
                rb = -k * cb * (ca + cc0);
            }
        }
        if (d2inv != 0.f) {
            // (denom - a*c) == -b*b and (denom + 2*b*b) == a*c + b*b, written without the cancellation
            float da = d2inv * (-cc * cc * dA + 2.f * cb * cc * dBh - cb * cb * dC);
            float dc = d2inv * (-ca * ca * dC + 2.f * ca * cb * dBh - cb * cb * dA);
            float db = d2inv * 2.f * (cb * cc * dA - (ca * cc + cb * cb) * dBh + ca * cb * dC);
            if (AA) { da += ra; db += rb; dc += rc; }
            dcov[0] += M0[0] * M0[0] * da + M0[0] * M1[0] * db + M1[0] * M1[0] * dc;
            dcov[3] += M0[1] * M0[1] * da + M0[1] * M1[1] * db + M1[1] * M1[1] * dc;
            dcov[5] += M0[2] * M0[2] * da + M0[2] * M1[2] * db + M1[2] * M1[2] * dc;
            dcov[1] += 2.f * M0[0] * M0[1] * da + (M0[0] * M1[1] + M0[1] * M1[0]) * db + 2.f * M1[0] * M1[1] * dc;
            dcov[2] += 2.f * M0[0] * M0[2] * da + (M0[0] * M1[2] + M0[2] * M1[0]) * db + 2.f * M1[0] * M1[2] * dc;
            dcov[4] += 2.f * M0[2] * M0[1] * da + (M0[1] * M1[2] + M0[2] * M1[1]) * db + 2.f * M1[1] * M1[2] * dc;
            float dM0[3], dM1[3];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                dM0[k] = 2.f * da * N0[k] + db * N1[k];
                dM1[k] = db * N0[k] + 2.f * dc * N1[k];
            }
            const float dJ00 = Wm[0][0] * dM0[0] + Wm[0][1] * dM0[1] + Wm[0][2] * dM0[2];
            const float dJ02 = Wm[2][0] * dM0[0] + Wm[2][1] * dM0[1] + Wm[2][2] * dM0[2];
            const float dJ11 = Wm[1][0] * dM1[0] + Wm[1][1] * dM1[1] + Wm[1][2] * dM1[2];
            const float dJ12 = Wm[2][0] * dM1[0] + Wm[2][1] * dM1[1] + Wm[2][2] * dM1[2];
            const float dtx = xmul * -fx * itz2 * dJ02;
            const float dty = ymul * -fy * itz2 * dJ12;
            const float dtz = -fx * itz2 * dJ00 - fy * itz2 * dJ11 + (2.f * fx * cx) * itz3 * dJ02 + (2.f * fy * cy) * itz3 * dJ12;
#pragma unroll
            for (int k = 0; k < 3; k++) dmean[k] += Wm[0][k] * dtx + Wm[1][k] * dty + Wm[2][k] * dtz;
        }
        // projection of the 2D mean (x,y only) and the fork's depth term
        const float hw = gs_affine(PV[3], PV[7], PV[11], PV[15], px, py, pz);
        const float m_w = 1.0f / (hw + 0.0000001f);
        const float mul1 = (PV[0] * px + PV[4] * py + PV[8] * pz + PV[12]) * m_w * m_w;
        const float mul2 = (PV[1] * px + PV[5] * py + PV[9] * pz + PV[13]) * m_w * m_w;
        const float mul3 = V[2] * px + V[6] * py + V[10] * pz + V[14];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            dmean[k] += (PV[4 * k] * m_w - PV[4 * k + 3] * mul1) * gdx + (PV[4 * k + 1] * m_w - PV[4 * k + 3] * mul2) * gdy;
            dmean[k] += (V[4 * k + 2] - V[4 * k + 3] * mul3) * gdepth;
        }
        if (DEG >= 0) {
            const float ddx0 = px - a.campos[3 * v], ddy0 = py - a.campos[3 * v + 1], ddz0 = pz - a.campos[3 * v + 2];
            const float len = sqrtf(ddx0 * ddx0 + ddy0 * ddy0 + ddz0 * ddz0);
            const float x = ddx0 / len, y = ddy0 / len, z = ddz0 / len;
            float bs[16];
            sh_basis(DEG, x, y, z, bs);
            const float dRGB[3] = {(cl & 1) ? 0.f : gcol[0], (cl & 2) ? 0.f : gcol[1], (cl & 4) ? 0.f : gcol[2]};
            float sk[16];
#pragma unroll
            for (int k = 0; k < nb; k++) {
                dsh[3 * k] += bs[k] * dRGB[0];
                dsh[3 * k + 1] += bs[k] * dRGB[1];
                dsh[3 * k + 2] += bs[k] * dRGB[2];
            }
            if (DEG > 0) { // sk[k] = sh_k . dRGB, for the view-direction derivative: four coefficients (3 x 16 B) at a time
                if (sh16) {
#pragma unroll
                    for (int kk = 0; kk < nb / 4; kk++) {
                        const float4 t0 = __ldg(reinterpret_cast<const float4 *>(shp) + 3 * kk);
                        const float4 t1 = __ldg(reinterpret_cast<const float4 *>(shp) + 3 * kk + 1);
                        const float4 t2 = __ldg(reinterpret_cast<const float4 *>(shp) + 3 * kk + 2);
                        sk[4 * kk] = t0.x * dRGB[0] + t0.y * dRGB[1] + t0.z * dRGB[2];
                        sk[4 * kk + 1] = t0.w * dRGB[0] + t1.x * dRGB[1] + t1.y * dRGB[2];
                        sk[4 * kk + 2] = t1.z * dRGB[0] + t1.w * dRGB[1] + t2.x * dRGB[2];
                        sk[4 * kk + 3] = t2.y * dRGB[0] + t2.z * dRGB[1] + t2.w * dRGB[2];
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < nb; k++)
                        sk[k] = __ldg(shp + 3 * k) * dRGB[0] + __ldg(shp + 3 * k + 1) * dRGB[1] + __ldg(shp + 3 * k + 2) * dRGB[2];
                }
            }
            if (DEG > 0) {
                float ddx = -SH_C1 * sk[3], ddy = -SH_C1 * sk[1], ddz = SH_C1 * sk[2];
                if (DEG > 1) {
                    const float xx = x * x, yy = y * y, zz = z * z;
                    ddx += c_SH_C2[0] * y * sk[4] + c_SH_C2[2] * -2.f * x * sk[6] + c_SH_C2[3] * z * sk[7] + c_SH_C2[4] * 2.f * x * sk[8];
                    ddy += c_SH_C2[0] * x * sk[4] + c_SH_C2[1] * z * sk[5] + c_SH_C2[2] * -2.f * y * sk[6] + c_SH_C2[4] * -2.f * y * sk[8];
                    ddz += c_SH_C2[1] * y * sk[5] + c_SH_C2[2] * 4.f * z * sk[6] + c_SH_C2[3] * x * sk[7];
                    if (DEG > 2) {
                        ddx += c_SH_C3[0] * sk[9] * 6.f * x * y + c_SH_C3[1] * sk[10] * y * z + c_SH_C3[2] * sk[11] * -2.f * x * y +
                               c_SH_C3[3] * sk[12] * -6.f * x * z + c_SH_C3[4] * sk[13] * (4.f * zz - 3.f * xx - yy) +
                               c_SH_C3[5] * sk[14] * 2.f * x * z + c_SH_C3[6] * sk[15] * 3.f * (xx - yy);
                        ddy += c_SH_C3[0] * sk[9] * 3.f * (xx - yy) + c_SH_C3[1] * sk[10] * x * z +
                               c_SH_C3[2] * sk[11] * (4.f * zz - xx - 3.f * yy) + c_SH_C3[3] * sk[12] * -6.f * y * z +
                               c_SH_C3[4] * sk[13] * -2.f * x * y + c_SH_C3[5] * sk[14] * -2.f * y * z + c_SH_C3[6] * sk[15] * -6.f * x * y;
                        ddz += c_SH_C3[1] * sk[10] * x * y + c_SH_C3[2] * sk[11] * 8.f * y * z +
                               c_SH_C3[3] * sk[12] * 3.f * (2.f * zz - xx - yy) + c_SH_C3[4] * sk[13] * 8.f * x * z +
                               c_SH_C3[5] * sk[14] * (xx - yy);
                    }
                }
                const float dot = x * ddx + y * ddy + z * ddz;
                dmean[0] += (ddx - x * dot) / len;
                dmean[1] += (ddy - y * dot) / len;
                dmean[2] += (ddz - z * dot) / len;
            }
        } else {
            dcol[0] += gcol[0]; dcol[1] += gcol[1]; dcol[2] += gcol[2];
        }
    }

    {
        float *o = a.dL_dmeans3D + 3 * ((a.means_view_stride ? (size_t)(a.V - 1) * a.P : 0) + (size_t)i);
        o[0] = dmean[0]; o[1] = dmean[1]; o[2] = dmean[2];
    }
    // F3D: dL/ds_i = f3s[i] * dL/ds'_i + f3q[i]; so = the activated scales before the filter (the exp Jacobian's factor)
    float f3s[3] = {1.f, 1.f, 1.f}, f3q[3] = {0.f, 0.f, 0.f}, so[3] = {0.f, 0.f, 0.f};
    if (F3D && !a.cov_pre) {
        const float v = a.f3d_var[i];
        float t[3], r[3], sp[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            so[k] = a.scales[3 * (size_t)i + k];
            if (a.raw) so[k] = expf(so[k]);
            sp[k] = so[k];
        }
        const float cf = gs_filter3d(sp, v, t, r);
        const float opa = a.raw ? gs_sigmoid(a.opac[i]) : a.opac[i];
        const float og = opa * dop; // o * g_o'
        dop *= cf;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            f3s[k] = t[k] > 0.f ? so[k] / sp[k] : 1.f;
            if (v > 0.f) f3q[k] = og * sqrtf(r[(k + 1) % 3] * r[(k + 2) % 3]) * v / (t[k] * sp[k]);
        }
    }
    if (a.raw) { // d sigmoid(x)/dx = o (1 - o)
        const float o = gs_sigmoid(a.opac[i]);
        dop *= o * (1.0f - o);
    }
    a.dL_dopacity[i] = dop;
    if (DEG >= 0) {
        float *o = a.dL_dsh + (size_t)i * a.M * 3;
#pragma unroll
        for (int k = 0; k < 3 * nb; k++) o[k] = dsh[k];
        for (int k = 3 * nb; k < 3 * a.M; k++) o[k] = 0.f;
    } else {
        a.dL_dcolors[3 * (size_t)i] = dcol[0]; a.dL_dcolors[3 * (size_t)i + 1] = dcol[1]; a.dL_dcolors[3 * (size_t)i + 2] = dcol[2];
    }
    if (a.cov_pre) {
        for (int k = 0; k < 6; k++) a.dL_dcov3D[6 * (size_t)i + k] = dcov[k];
    } else {
        const float dS[3][3] = {{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]},
                                {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]},
                                {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}};
        float L[3][3], dLm[3][3], dR[3][3];
#pragma unroll
        for (int r2 = 0; r2 < 3; r2++)
#pragma unroll
            for (int k = 0; k < 3; k++) L[r2][k] = R[r2][k] * s[k];
#pragma unroll
        for (int r2 = 0; r2 < 3; r2++)
#pragma unroll
            for (int k = 0; k < 3; k++) dLm[r2][k] = 2.f * (dS[r2][0] * L[0][k] + dS[r2][1] * L[1][k] + dS[r2][2] * L[2][k]);
#pragma unroll
        for (int k = 0; k < 3; k++) {
            if (F3D) { // through the filter (f3s = 1, f3q = 0 where v = 0), then exp's Jacobian so[k]
                float g = f3s[k] * (a.mod * (R[0][k] * dLm[0][k] + R[1][k] * dLm[1][k] + R[2][k] * dLm[2][k]));
                if (f3q[k] != 0.f) g += f3q[k];
                a.dL_dscales[3 * (size_t)i + k] = a.raw ? g * so[k] : g;
            } else {
                // raw: d exp(x)/dx = exp(x) = s[k] / mod
                a.dL_dscales[3 * (size_t)i + k] = (a.raw ? s[k] : a.mod) * (R[0][k] * dLm[0][k] + R[1][k] * dLm[1][k] + R[2][k] * dLm[2][k]);
            }
#pragma unroll
            for (int r2 = 0; r2 < 3; r2++) dR[r2][k] = dLm[r2][k] * s[k];
        }
        const float r = q[0], x = q[1], y = q[2], z = q[3];
        float4 dq;
        dq.x = 2.f * z * (dR[1][0] - dR[0][1]) + 2.f * y * (dR[0][2] - dR[2][0]) + 2.f * x * (dR[2][1] - dR[1][2]);
        dq.y = 2.f * y * (dR[0][1] + dR[1][0]) + 2.f * z * (dR[0][2] + dR[2][0]) + 2.f * r * (dR[2][1] - dR[1][2]) - 4.f * x * (dR[1][1] + dR[2][2]);
        dq.z = 2.f * x * (dR[0][1] + dR[1][0]) + 2.f * r * (dR[0][2] - dR[2][0]) + 2.f * z * (dR[1][2] + dR[2][1]) - 4.f * y * (dR[0][0] + dR[2][2]);
        dq.w = 2.f * r * (dR[1][0] - dR[0][1]) + 2.f * x * (dR[0][2] + dR[2][0]) + 2.f * y * (dR[1][2] + dR[2][1]) - 4.f * z * (dR[0][0] + dR[1][1]);
        if (a.raw) { // Jacobian of x / max(||x||, eps): (dq - q_hat (q_hat . dq)) / ||x||, dq / eps below eps (F.normalize's autograd)
            const float dot = qproj ? r * dq.x + x * dq.y + y * dq.z + z * dq.w : 0.f;
            const float inv = 1.0f / qnorm;
            dq.x = (dq.x - r * dot) * inv; dq.y = (dq.y - x * dot) * inv; dq.z = (dq.z - y * dot) * inv; dq.w = (dq.w - z * dot) * inv;
        }
        if (a.vec16) reinterpret_cast<float4 *>(a.dL_drots)[i] = dq;
        else {
            float *o = a.dL_drots + 4 * (size_t)i;
            o[0] = dq.x; o[1] = dq.y; o[2] = dq.z; o[3] = dq.w;
        }
    }
}

template <bool AA, bool F3D>
static void launch_preprocess_bwd_t(const PreBwdArgs &a, cudaStream_t st)
{
    const int grid = (a.P + 127) / 128;
    if (!a.shs) preprocess_bwd_kernel<-1, AA, F3D><<<grid, 128, 0, st>>>(a);
    else if (a.deg == 0) preprocess_bwd_kernel<0, AA, F3D><<<grid, 128, 0, st>>>(a);
    else if (a.deg == 1) preprocess_bwd_kernel<1, AA, F3D><<<grid, 128, 0, st>>>(a);
    else if (a.deg == 2) preprocess_bwd_kernel<2, AA, F3D><<<grid, 128, 0, st>>>(a);
    else preprocess_bwd_kernel<3, AA, F3D><<<grid, 128, 0, st>>>(a);
}
void launch_preprocess_bwd(const PreBwdArgs &a, bool aa, bool f3d, cudaStream_t st)
{
    if (f3d) {
        if (aa) launch_preprocess_bwd_t<true, true>(a, st);
        else launch_preprocess_bwd_t<false, true>(a, st);
    } else {
        if (aa) launch_preprocess_bwd_t<true, false>(a, st);
        else launch_preprocess_bwd_t<false, false>(a, st);
    }
}
