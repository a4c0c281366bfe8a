/*
 * gs_oracle.c -- CPU ORACLE for the differentiable 3D-Gaussian-splatting rasteriser.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load it.  The product path
 * (humangaussian_b200/) never links, imports or calls anything in oracle/.
 *
 * PARITY UNPINNED: the algorithm restated here lives in a third-party package that is NOT
 * vendored in the HumanGaussian tree (diff_gaussian_rasterization, ashawkey fork, un-pinned
 * `git clone`, reference README.md:30-32,72-74; call sites
 * gaussiansplatting/gaussian_renderer/__init__.py:14,36-51,86-94 and gs_renderer.py:10-13,
 * 951-966,1006-1015).  The reference ships no tests and no golden vectors for it.  What this
 * file restates is the published 3DGS tile rasteriser (Kerbl et al. 2023) plus the fork's
 * depth/alpha outputs, as specified in SURVEY.md Appendix A.  The in-tree Python math that
 * overlaps (SH basis: gaussiansplatting/utils/sh_utils.py:57-112; covariance packing:
 * utils/general_utils.py:64-110; projection: utils/graphics_utils.py:22-30,73-93) IS pinned,
 * by golden vectors generated from the reference's own code (tests/golden/make_golden.py).
 *
 * NUMERICAL CONTRACT.  Everything that decides an index or a branch (depth bits, radius,
 * tile rectangle, power/alpha/T tests) is written with an explicit float operation order:
 * plain `a*b`, `a+b` are single IEEE-754 binary32 roundings (compile with
 * -ffp-contract=off), `fmaf` is a fused multiply-add, sqrtf and `/` are correctly rounded,
 * and exp() is the fixed polynomial gs_exp() below.  The CUDA kernels use the same sequence
 * (compiled with -fmad=false and explicit fmaf), so the forward pass is comparable
 * BIT-FOR-BIT; the backward pass sums in a different order and is compared to tolerance.
 *
 * Build:  gcc -O2 -fPIC -shared -fopenmp -ffp-contract=off -mfma -mavx2 gs_oracle.c -lm
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define TILE 16
#define NEAR_Z 0.2f
#define DILATE 0.3f
#define ALPHA_MAX 0.99f
#define ALPHA_MIN (1.0f / 255.0f)
#define T_MIN 0.0001f

/* SH constants: gaussiansplatting/utils/sh_utils.py:26-43 (rounded to binary32) */
static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                               0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                               -0.5900435899266435f};

/* ---- deterministic exp: range-reduced degree-5 polynomial, |rel err| < 2e-7 for x in [-87,0] ---- */
static inline float gs_exp(float x)
{
    x = fmaxf(x, -87.0f);
    float t = fmaf(x, 0x1.715476p+0f, 12582912.0f); /* x*log2(e) + 1.5*2^23 : rounds to integer */
    float n = t - 12582912.0f;
    float r = fmaf(n, -0x1.62e430p-1f, x);          /* x - n*ln2 */
    float p = 0x1.0fa834p-7f;
    p = fmaf(p, r, 0x1.573a54p-5f);
    p = fmaf(p, r, 0x1.555a6ap-3f);
    p = fmaf(p, r, 0x1.fffdc6p-2f);
    p = fmaf(p, r, 0x1.fffff6p-1f);
    p = fmaf(p, r, 1.0f);
    uint32_t ti, pi;
    memcpy(&ti, &t, 4);
    memcpy(&pi, &p, 4);
    pi += ti << 23; /* add n to the exponent field */
    memcpy(&p, &pi, 4);
    return p;
}

/* C float->int cast with CUDA's saturating semantics (cvt.rzi.s32.f32) */
static inline int f2i(float v)
{
    if (v != v) return 0;
    if (v >= 2147483648.0f) return 2147483647;
    if (v <= -2147483648.0f) return (-2147483647 - 1);
    return (int)v;
}
static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* m0*x + m1*y + m2*z + m3 as  mul, fma, fma, add */
static inline float affine(float m0, float m1, float m2, float m3, float x, float y, float z)
{
    float a = m0 * x;
    a = fmaf(m1, y, a);
    a = fmaf(m2, z, a);
    return a + m3;
}
static inline float dot3(float a0, float a1, float a2, float b0, float b1, float b2)
{
    float a = a0 * b0;
    a = fmaf(a1, b1, a);
    return fmaf(a2, b2, a);
}

typedef struct gso_ctx {
    /* problem */
    int P, deg, M, H, W, gx, gy, ntiles;
    float tanfovx, tanfovy, mod;
    const float *means, *shs, *colors_pre, *opac, *scales, *rots, *cov_pre, *bg, *view, *proj, *campos;
    /* per-Gaussian state */
    float *xy, *depth, *conic_o, *rgb, *cov3d;
    int *radii;
    uint32_t *tiles_touched, *offsets;
    int *rect; /* [P][4] xmin ymin xmax ymax */
    uint8_t *clamped;
    /* binning */
    int64_t D;
    uint64_t *keys, *keys_tmp;
    uint32_t *vals, *vals_tmp;
    uint32_t *ranges; /* [ntiles][2] */
    /* image state */
    float *final_T;
    uint32_t *n_contrib;
    uint8_t *contrib_patches; /* [D]: bit p = some in-image pixel of 8x4 patch p of the entry's tile blended it */
    int capP, capD, capPix, capTiles;
    int threads;
} gso_ctx;

gso_ctx *gso_create(void)
{
    gso_ctx *c = (gso_ctx *)calloc(1, sizeof(gso_ctx));
    c->threads = 0;
    return c;
}
void gso_set_threads(gso_ctx *c, int n) { c->threads = n; }
static void free_all(gso_ctx *c)
{
    free(c->xy); free(c->depth); free(c->conic_o); free(c->rgb); free(c->cov3d); free(c->radii);
    free(c->tiles_touched); free(c->offsets); free(c->rect); free(c->clamped);
    free(c->keys); free(c->keys_tmp); free(c->vals); free(c->vals_tmp); free(c->ranges);
    free(c->final_T); free(c->n_contrib); free(c->contrib_patches);
}
void gso_destroy(gso_ctx *c)
{
    if (!c) return;
    free_all(c);
    free(c);
}

/* ------------------------------------------------------------------------------------------
 * F1  preprocess one Gaussian  (SURVEY.md Appendix A.2)
 * ---------------------------------------------------------------------------------------- */
static void build_cov3d(const float *s3, float mod, const float *q, float *c6)
{
    /* rotation as in gaussiansplatting/utils/general_utils.py:78-99, WITHOUT normalising q
       (the Python side normalises: gaussian_model.py:41,99-101); packing as :64-73 */
    float r = q[0], x = q[1], y = q[2], z = q[3];
    float R[3][3];
    R[0][0] = fmaf(-2.0f, fmaf(z, z, y * y), 1.0f);
    R[0][1] = 2.0f * fmaf(x, y, -(r * z));
    R[0][2] = 2.0f * fmaf(x, z, r * y);
    R[1][0] = 2.0f * fmaf(x, y, r * z);
    R[1][1] = fmaf(-2.0f, fmaf(z, z, x * x), 1.0f);
    R[1][2] = 2.0f * fmaf(y, z, -(r * x));
    R[2][0] = 2.0f * fmaf(x, z, -(r * y));
    R[2][1] = 2.0f * fmaf(y, z, r * x);
    R[2][2] = fmaf(-2.0f, fmaf(y, y, x * x), 1.0f);
    float s[3] = {mod * s3[0], mod * s3[1], mod * s3[2]};
    float L[3][3];
    for (int i = 0; i < 3; i++)
        for (int k = 0; k < 3; k++) L[i][k] = R[i][k] * s[k];
    c6[0] = dot3(L[0][0], L[0][1], L[0][2], L[0][0], L[0][1], L[0][2]);
    c6[1] = dot3(L[0][0], L[0][1], L[0][2], L[1][0], L[1][1], L[1][2]);
    c6[2] = dot3(L[0][0], L[0][1], L[0][2], L[2][0], L[2][1], L[2][2]);
    c6[3] = dot3(L[1][0], L[1][1], L[1][2], L[1][0], L[1][1], L[1][2]);
    c6[4] = dot3(L[1][0], L[1][1], L[1][2], L[2][0], L[2][1], L[2][2]);
    c6[5] = dot3(L[2][0], L[2][1], L[2][2], L[2][0], L[2][1], L[2][2]);
}

/* the 16 real-SH basis values of sh_utils.py:74-100 (signs folded in), for unit dir (x,y,z) */
static void sh_basis(int deg, float x, float y, float z, float *b)
{
    b[0] = SH_C0;
    if (deg > 0) {
        b[1] = -SH_C1 * y;
        b[2] = SH_C1 * z;
        b[3] = -SH_C1 * x;
        if (deg > 1) {
            float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            b[4] = SH_C2[0] * xy;
            b[5] = SH_C2[1] * yz;
            b[6] = SH_C2[2] * ((2.0f * zz - xx) - yy);
            b[7] = SH_C2[3] * xz;
            b[8] = SH_C2[4] * (xx - yy);
            if (deg > 2) {
                b[9] = (SH_C3[0] * y) * fmaf(3.0f, xx, -yy);
                b[10] = (SH_C3[1] * xy) * z;
                b[11] = (SH_C3[2] * y) * ((4.0f * zz - xx) - yy);
                b[12] = (SH_C3[3] * z) * ((2.0f * zz - 3.0f * xx) - 3.0f * yy);
                b[13] = (SH_C3[4] * x) * ((4.0f * zz - xx) - yy);
                b[14] = (SH_C3[5] * z) * (xx - yy);
                b[15] = (SH_C3[6] * x) * fmaf(-3.0f, yy, xx);
            }
        }
    }
}

static void preprocess_one(gso_ctx *c, int i)
{
    const float *V = c->view, *PV = c->proj;
    c->radii[i] = 0;
    c->tiles_touched[i] = 0;
    const float px = c->means[3 * i], py = c->means[3 * i + 1], pz = c->means[3 * i + 2];
    /* view space; V is the 16 floats of world_view_transform read column-major (A.1) */
    float tx = affine(V[0], V[4], V[8], V[12], px, py, pz);
    float ty = affine(V[1], V[5], V[9], V[13], px, py, pz);
    float tz = affine(V[2], V[6], V[10], V[14], px, py, pz);
    if (tz <= NEAR_Z) return;
    float hx = affine(PV[0], PV[4], PV[8], PV[12], px, py, pz);
    float hy = affine(PV[1], PV[5], PV[9], PV[13], px, py, pz);
    float hw = affine(PV[3], PV[7], PV[11], PV[15], px, py, pz);
    float pw = 1.0f / (hw + 0.0000001f);
    float ndcx = hx * pw, ndcy = hy * pw;

    float *c6 = c->cov3d + 6 * i;
    if (c->cov_pre) memcpy(c6, c->cov_pre + 6 * i, 24);
    else build_cov3d(c->scales + 3 * i, c->mod, c->rots + 4 * i, c6);

    /* EWA projection */
    float fx = (float)c->W / (2.0f * c->tanfovx), fy = (float)c->H / (2.0f * c->tanfovy);
    float limx = 1.3f * c->tanfovx, limy = 1.3f * c->tanfovy;
    float txtz = tx / tz, tytz = ty / tz;
    float cx = fminf(limx, fmaxf(-limx, txtz)) * tz;
    float cy = fminf(limy, fmaxf(-limy, tytz)) * tz;
    float J00 = fx / tz, J11 = fy / tz;
    float tz2 = tz * tz;
    float J02 = -(fx * cx) / tz2, J12 = -(fy * cy) / tz2;
    float M0[3], M1[3];
    for (int k = 0; k < 3; k++) { /* W3[r][k] = V[4k+r] */
        M0[k] = fmaf(J02, V[4 * k + 2], J00 * V[4 * k + 0]);
        M1[k] = fmaf(J12, V[4 * k + 2], J11 * V[4 * k + 1]);
    }
    float S[3][3] = {{c6[0], c6[1], c6[2]}, {c6[1], c6[3], c6[4]}, {c6[2], c6[4], c6[5]}};
    float N0[3], N1[3];
    for (int k = 0; k < 3; k++) {
        N0[k] = dot3(M0[0], M0[1], M0[2], S[0][k], S[1][k], S[2][k]);
        N1[k] = dot3(M1[0], M1[1], M1[2], S[0][k], S[1][k], S[2][k]);
    }
    float a = dot3(N0[0], N0[1], N0[2], M0[0], M0[1], M0[2]) + DILATE;
    float b = dot3(N0[0], N0[1], N0[2], M1[0], M1[1], M1[2]);
    float cc = dot3(N1[0], N1[1], N1[2], M1[0], M1[1], M1[2]) + DILATE;
    float det = fmaf(a, cc, -(b * b));
    if (det == 0.0f) return;
    float det_inv = 1.0f / det;
    float conA = cc * det_inv, conB = -b * det_inv, conC = a * det_inv;
    float mid = 0.5f * (a + cc);
    float sq = sqrtf(fmaxf(0.1f, fmaf(mid, mid, -det)));
    float lam = fmaxf(mid + sq, mid - sq);
    int radius = f2i(ceilf(3.0f * sqrtf(lam)));
    float pxs = fmaf(ndcx + 1.0f, (float)c->W, -1.0f) * 0.5f;
    float pys = fmaf(ndcy + 1.0f, (float)c->H, -1.0f) * 0.5f;
    float fr = (float)radius;
    int x0 = imin(c->gx, imax(0, f2i((pxs - fr) / 16.0f)));
    int y0 = imin(c->gy, imax(0, f2i((pys - fr) / 16.0f)));
    int x1 = imin(c->gx, imax(0, f2i((((pxs + fr) + 16.0f) - 1.0f) / 16.0f)));
    int y1 = imin(c->gy, imax(0, f2i((((pys + fr) + 16.0f) - 1.0f) / 16.0f)));
    if ((x1 - x0) * (y1 - y0) == 0) return;

    /* colour */
    float *rgb = c->rgb + 3 * i;
    if (c->shs) {
        float dx = px - c->campos[0], dy = py - c->campos[1], dz = pz - c->campos[2];
        float len = sqrtf(dot3(dx, dy, dz, dx, dy, dz));
        dx = dx / len; dy = dy / len; dz = dz / len;
        float bs[16];
        sh_basis(c->deg, dx, dy, dz, bs);
        int nb = (c->deg + 1) * (c->deg + 1);
        const float *sh = c->shs + (size_t)i * c->M * 3;
        for (int ch = 0; ch < 3; ch++) {
            float r = bs[0] * sh[ch];
            for (int k = 1; k < nb; k++) r = fmaf(bs[k], sh[3 * k + ch], r);
            r = r + 0.5f;
            c->clamped[3 * i + ch] = (r < 0.0f);
            rgb[ch] = fmaxf(r, 0.0f);
        }
    } else {
        rgb[0] = c->colors_pre[3 * i]; rgb[1] = c->colors_pre[3 * i + 1]; rgb[2] = c->colors_pre[3 * i + 2];
        c->clamped[3 * i] = c->clamped[3 * i + 1] = c->clamped[3 * i + 2] = 0;
    }
    c->depth[i] = tz;
    c->radii[i] = radius;
    c->xy[2 * i] = pxs; c->xy[2 * i + 1] = pys;
    c->conic_o[4 * i] = conA; c->conic_o[4 * i + 1] = conB; c->conic_o[4 * i + 2] = conC;
    c->conic_o[4 * i + 3] = c->opac[i];
    c->rect[4 * i] = x0; c->rect[4 * i + 1] = y0; c->rect[4 * i + 2] = x1; c->rect[4 * i + 3] = y1;
    c->tiles_touched[i] = (uint32_t)((x1 - x0) * (y1 - y0));
}

/* stable LSD radix sort of (u64 key, u32 value), 8-bit digits over `nbits` low bits (A.3).
 * Parallel counting sort per pass: every thread histograms a contiguous chunk, a serial prefix over (digit, thread)
 * gives each chunk its destination of every digit, the chunks scatter in input order -- the result is the serial
 * stable sort's, for any thread count.  Buffers ping-pong; one copy at the end if the result sits in the temporaries. */
static void radix_sort(uint64_t *k, uint64_t *kt, uint32_t *v, uint32_t *vt, int64_t n, int nbits)
{
#ifdef _OPENMP
    int nt = omp_get_max_threads();
#else
    int nt = 1;
#endif
    if (nt > 256) nt = 256;
    if ((int64_t)nt > n / 4096 + 1) nt = (int)(n / 4096 + 1); /* small inputs: fewer chunks */
    int64_t *cnt = (int64_t *)malloc(sizeof(int64_t) * 256 * (size_t)nt);
    uint64_t *ki = k, *ko = kt;
    uint32_t *vi = v, *vo = vt;
    for (int shift = 0; shift < nbits; shift += 8) {
        /* a loop over the nt CHUNKS (not over thread ids): every chunk is processed whatever team size the runtime grants */
#pragma omp parallel for num_threads(nt) schedule(static, 1)
        for (int t = 0; t < nt; t++) {
            const int64_t lo = n * t / nt, hi = n * (t + 1) / nt;
            int64_t *h = cnt + 256 * (size_t)t;
            memset(h, 0, sizeof(int64_t) * 256);
            for (int64_t i = lo; i < hi; i++) h[(ki[i] >> shift) & 255]++;
        }
        int64_t run = 0;
        for (int d = 0; d < 256; d++)
            for (int t = 0; t < nt; t++) {
                const int64_t c0 = cnt[256 * (size_t)t + d];
                cnt[256 * (size_t)t + d] = run;
                run += c0;
            }
#pragma omp parallel for num_threads(nt) schedule(static, 1)
        for (int t = 0; t < nt; t++) {
            const int64_t lo = n * t / nt, hi = n * (t + 1) / nt;
            int64_t *h = cnt + 256 * (size_t)t;
            for (int64_t i = lo; i < hi; i++) {
                const int64_t dst = h[(ki[i] >> shift) & 255]++;
                ko[dst] = ki[i];
                vo[dst] = vi[i];
            }
        }
        uint64_t *tk = ki; ki = ko; ko = tk;
        uint32_t *tv = vi; vi = vo; vo = tv;
    }
    if (ki != k) {
        memcpy(k, ki, (size_t)n * sizeof(uint64_t));
        memcpy(v, vi, (size_t)n * sizeof(uint32_t));
    }
    free(cnt);
}

static inline float eval_power(float A, float B, float C, float dx, float dy)
{
    /* -0.5*(A dx^2 + C dy^2) - B dx dy  evaluated as  dx*(-A/2*dx - B*dy) + (-C/2*dy)*dy */
    float u = fmaf(-B, dy, (-0.5f * A) * dx);
    float w = ((-0.5f * C) * dy) * dy;
    return fmaf(dx, u, w);
}

/* ------------------------------------------------------------------------------------------
 * forward
 * ---------------------------------------------------------------------------------------- */
#define REALLOC(ptr, type, n) ptr = (type *)realloc(ptr, sizeof(type) * (size_t)((n) > 0 ? (n) : 1))

int gso_forward(gso_ctx *c, int P, int deg, int M, int H, int W, float tanfovx, float tanfovy,
                float scale_modifier, const float *means3D, const float *shs,
                const float *colors_precomp, const float *opacities, const float *scales,
                const float *rotations, const float *cov3D_precomp, const float *bg,
                const float *viewmatrix, const float *projmatrix, const float *campos,
                float *out_color, float *out_depth, float *out_alpha, int *radii_out)
{
    if ((shs == NULL) == (colors_precomp == NULL)) return -1;
    if (((scales == NULL) || (rotations == NULL)) == (cov3D_precomp == NULL)) return -2;
    if (deg < 0 || deg > 3 || (shs && M < (deg + 1) * (deg + 1))) return -3;
#ifdef _OPENMP
    if (c->threads > 0) omp_set_num_threads(c->threads);
#endif
    c->P = P; c->deg = deg; c->M = M; c->H = H; c->W = W;
    c->gx = (W + TILE - 1) / TILE; c->gy = (H + TILE - 1) / TILE; c->ntiles = c->gx * c->gy;
    c->tanfovx = tanfovx; c->tanfovy = tanfovy; c->mod = scale_modifier;
    c->means = means3D; c->shs = shs; c->colors_pre = colors_precomp; c->opac = opacities;
    c->scales = scales; c->rots = rotations; c->cov_pre = cov3D_precomp; c->bg = bg;
    c->view = viewmatrix; c->proj = projmatrix; c->campos = campos;
    REALLOC(c->xy, float, 2 * P); REALLOC(c->depth, float, P); REALLOC(c->conic_o, float, 4 * P);
    REALLOC(c->rgb, float, 3 * P); REALLOC(c->cov3d, float, 6 * P); REALLOC(c->radii, int, P);
    REALLOC(c->tiles_touched, uint32_t, P); REALLOC(c->offsets, uint32_t, P);
    REALLOC(c->rect, int, 4 * P); REALLOC(c->clamped, uint8_t, 3 * P);
    memset(c->xy, 0, sizeof(float) * 2 * P); memset(c->depth, 0, sizeof(float) * P);
    memset(c->conic_o, 0, sizeof(float) * 4 * P); memset(c->rgb, 0, sizeof(float) * 3 * P);
    memset(c->clamped, 0, 3 * P); memset(c->rect, 0, sizeof(int) * 4 * P);
    memset(c->cov3d, 0, sizeof(float) * 6 * P);

#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; i++) preprocess_one(c, i);

    /* F2 inclusive scan */
    int64_t D = 0;
    for (int i = 0; i < P; i++) { D += c->tiles_touched[i]; c->offsets[i] = (uint32_t)D; }
    c->D = D;
    REALLOC(c->keys, uint64_t, D); REALLOC(c->keys_tmp, uint64_t, D);
    REALLOC(c->vals, uint32_t, D); REALLOC(c->vals_tmp, uint32_t, D);
    REALLOC(c->ranges, uint32_t, 2 * c->ntiles);
    REALLOC(c->contrib_patches, uint8_t, D);
    memset(c->contrib_patches, 0, (size_t)D);
    /* F3 duplicate with keys: row-major over the tile rectangle */
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; i++) {
        if (c->radii[i] <= 0) continue;
        int64_t off = (i == 0) ? 0 : c->offsets[i - 1];
        uint32_t dbits;
        memcpy(&dbits, &c->depth[i], 4);
        for (int y = c->rect[4 * i + 1]; y < c->rect[4 * i + 3]; y++)
            for (int x = c->rect[4 * i]; x < c->rect[4 * i + 2]; x++) {
                uint64_t key = (uint64_t)(y * c->gx + x);
                c->keys[off] = (key << 32) | dbits;
                c->vals[off] = (uint32_t)i;
                off++;
            }
    }
    /* F4 stable sort on the low 32+msb(ntiles) bits */
    int bit = 0;
    while ((1 << bit) < c->ntiles) bit++; /* enough bits to hold every tile id */
    radix_sort(c->keys, c->keys_tmp, c->vals, c->vals_tmp, D, 32 + bit);
    /* F5 tile ranges */
    memset(c->ranges, 0, sizeof(uint32_t) * 2 * c->ntiles);
    for (int64_t j = 0; j < D; j++) {
        uint32_t t = (uint32_t)(c->keys[j] >> 32);
        if (j == 0 || t != (uint32_t)(c->keys[j - 1] >> 32)) c->ranges[2 * t] = (uint32_t)j;
        if (j == D - 1 || t != (uint32_t)(c->keys[j + 1] >> 32)) c->ranges[2 * t + 1] = (uint32_t)(j + 1);
    }
    /* F6 blend */
    REALLOC(c->final_T, float, H * W); REALLOC(c->n_contrib, uint32_t, H * W);
#pragma omp parallel for schedule(dynamic, 1)
    for (int t = 0; t < c->ntiles; t++) {
        int tx0 = (t % c->gx) * TILE, ty0 = (t / c->gx) * TILE;
        uint32_t r0 = c->ranges[2 * t], r1 = c->ranges[2 * t + 1];
        int n = (int)(r1 - r0);
        float *loc = (float *)malloc(sizeof(float) * 10 * (n > 0 ? n : 1));
        for (int j = 0; j < n; j++) {
            uint32_t g = c->vals[r0 + j];
            float *l = loc + 10 * j;
            l[0] = c->xy[2 * g]; l[1] = c->xy[2 * g + 1];
            l[2] = c->conic_o[4 * g]; l[3] = c->conic_o[4 * g + 1]; l[4] = c->conic_o[4 * g + 2];
            l[5] = c->conic_o[4 * g + 3];
            l[6] = c->rgb[3 * g]; l[7] = c->rgb[3 * g + 1]; l[8] = c->rgb[3 * g + 2];
            l[9] = c->depth[g];
        }
        for (int py = ty0; py < ty0 + TILE && py < H; py++)
            for (int px = tx0; px < tx0 + TILE && px < W; px++) {
                float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, Dd = 0.f, Aa = 0.f;
                uint32_t contributor = 0, last = 0;
                float fx = (float)px, fy = (float)py;
                /* the CUDA blend's patch numbering: bit 0 = x half of the tile, bits 1-2 = band of four rows */
                const uint8_t pbit = (uint8_t)(1u << (((py % TILE) / 4) * 2 + (px % TILE) / 8));
                uint8_t *cp = c->contrib_patches + r0;
                for (int j = 0; j < n; j++) {
                    const float *l = loc + 10 * j;
                    contributor++;
                    float dx = l[0] - fx, dy = l[1] - fy;
                    float power = eval_power(l[2], l[3], l[4], dx, dy);
                    if (power > 0.0f) continue;
                    float alpha = fminf(ALPHA_MAX, l[5] * gs_exp(power));
                    if (alpha < ALPHA_MIN) continue;
                    float test_T = T * (1.0f - alpha);
                    if (test_T < T_MIN) break;
                    float w = alpha * T;
                    C0 = fmaf(l[6], w, C0); C1 = fmaf(l[7], w, C1); C2 = fmaf(l[8], w, C2);
                    Dd = fmaf(l[9], w, Dd);
                    Aa = Aa + w;
                    T = test_T;
                    last = contributor;
                    cp[j] |= pbit;
                }
                size_t pix = (size_t)py * W + px;
                c->final_T[pix] = T;
                c->n_contrib[pix] = last;
                out_color[pix] = fmaf(T, bg[0], C0);
                out_color[(size_t)H * W + pix] = fmaf(T, bg[1], C1);
                out_color[2 * (size_t)H * W + pix] = fmaf(T, bg[2], C2);
                out_depth[pix] = Dd;
                out_alpha[pix] = Aa;
            }
        free(loc);
    }
    if (radii_out) memcpy(radii_out, c->radii, sizeof(int) * P);
    return 0;
}

/* state accessors (valid until the next gso_forward on this ctx) */
int64_t gso_num_rendered(gso_ctx *c) { return c->D; }
const uint64_t *gso_keys(gso_ctx *c) { return c->keys; }
const uint32_t *gso_point_list(gso_ctx *c) { return c->vals; }
const uint32_t *gso_ranges(gso_ctx *c) { return c->ranges; }
const float *gso_xy(gso_ctx *c) { return c->xy; }
const float *gso_depths(gso_ctx *c) { return c->depth; }
const float *gso_conic_opacity(gso_ctx *c) { return c->conic_o; }
const float *gso_rgb(gso_ctx *c) { return c->rgb; }
const float *gso_cov3d(gso_ctx *c) { return c->cov3d; }
const uint32_t *gso_tiles_touched(gso_ctx *c) { return c->tiles_touched; }
const int *gso_rect(gso_ctx *c) { return c->rect; }
const uint8_t *gso_clamped(gso_ctx *c) { return c->clamped; }
const float *gso_final_T(gso_ctx *c) { return c->final_T; }
const uint32_t *gso_n_contrib(gso_ctx *c) { return c->n_contrib; }
const uint8_t *gso_contrib_patches(gso_ctx *c) { return c->contrib_patches; }

/* ------------------------------------------------------------------------------------------
 * backward  (SURVEY.md Appendix A.5-A.7).  Uses the state of the last gso_forward.
 * Upstream accumulates the per-pixel terms with float atomics in an unspecified order (A.9); the
 * oracle resolves that freedom by summing the float32 TERMS exactly enough to be order-free: each
 * per-pixel term is computed in float32 exactly as specified, but the per-(tile,Gaussian) partial
 * sums and their reduction to per-Gaussian sums are carried in double and rounded to float32 once.
 * Partials are formed in parallel, then reduced sequentially in sorted-list order: deterministic
 * for any thread count.
 *
 * Optional export (sums_out / err_out non-NULL, each [P][10]): the per-Gaussian sums in the CUDA backward blend's
 * moments format, in double, for checking that intermediate directly:
 *   S0, Sx, Sy, Sxx, Sxy, Syy = sum q*{1, dx, dy, dx^2, dx*dy, dy^2},  q = G*dL/dalpha (the float32 product used for o[5]),
 *   dx = px_gauss - px, dy = py_gauss - py;   W0..W3 = sum w*{gC0, gC1, gC2, gD},  w = alpha*T (float32).
 * and an error scale per component: the sum over the terms of |term magnitude| * (r + err_const + N_g), where r is the
 * replay depth (transmittance recoveries T <- T/(1-alpha) done for the pixel so far, this one included) and N_g the
 * number of (tile, patch) pairs the Gaussian contributes to (contrib_patches bits of its entries: how many partial sums
 * the CUDA flush writes into its record).  The magnitude of a q moment is
 *   |phi_k(dx,dy)| * G * (T*(|cg|_abs + |rg|_abs) + T_final*|bg.gC|_abs/(1-alpha)),
 * |.|_abs being the same expression on absolute values (cg = c.gC + depth*gD + gA, rg its back-to-front recurrence);
 * that of W_k is |w*g_k|.  tests/test_gpu_parity.py derives err_const and the bound's factor.
 * screen_out (optional, [P][10]): the double per-Gaussian sums o[0..9] below, before their rounding to float32.
 * ---------------------------------------------------------------------------------------- */
int gso_backward(gso_ctx *c, const float *dL_dcolor, const float *dL_ddepth_img, const float *dL_dalpha_img,
                 float *dL_dmeans3D, float *dL_dmeans2D, float *dL_dsh, float *dL_dcolors,
                 float *dL_dopacity, float *dL_dscales, float *dL_drots, float *dL_dcov3D,
                 double err_const, double *sums_out, double *err_out, double *screen_out)
{
    const int P = c->P, H = c->H, W = c->W;
    const int64_t D = c->D;
    const float *bg = c->bg;
    /* every tile owns the slice [r0, r1) of `part`: it zeroes it itself (parallel first touch; a calloc of D*80 bytes
     * followed by a serial reduction made the backward 0.7 s serial per 1024^2 view of 300 k Gaussians) */
    double *part = (double *)malloc((size_t)(D > 0 ? D : 1) * 10 * sizeof(double));
    /* moments export: per instance 10 sums + 10 error scales, laid out and reduced like `part` */
    const int want_sums = sums_out != NULL && err_out != NULL;
    double *sp = want_sums ? (double *)malloc((size_t)(D > 0 ? D : 1) * 20 * sizeof(double)) : NULL;
    double *ng = NULL; /* N_g: (tile, patch) pairs Gaussian g contributes to */
    if (want_sums) {
        ng = (double *)calloc((size_t)(P > 0 ? P : 1), sizeof(double));
        for (int64_t j = 0; j < D; j++) ng[c->vals[j]] += (double)__builtin_popcount(c->contrib_patches[j]);
    }
#pragma omp parallel for schedule(dynamic, 1)
    for (int t = 0; t < c->ntiles; t++) {
        int tx0 = (t % c->gx) * TILE, ty0 = (t / c->gx) * TILE;
        uint32_t r0 = c->ranges[2 * t], r1 = c->ranges[2 * t + 1];
        int n = (int)(r1 - r0);
        if (n == 0) continue;
        memset(part + (size_t)r0 * 10, 0, sizeof(double) * 10 * (size_t)n);
        if (sp) memset(sp + (size_t)r0 * 20, 0, sizeof(double) * 20 * (size_t)n);
        float *loc = (float *)malloc(sizeof(float) * 10 * n);
        for (int j = 0; j < n; j++) {
            uint32_t g = c->vals[r0 + j];
            float *l = loc + 10 * j;
            l[0] = c->xy[2 * g]; l[1] = c->xy[2 * g + 1];
            l[2] = c->conic_o[4 * g]; l[3] = c->conic_o[4 * g + 1]; l[4] = c->conic_o[4 * g + 2];
            l[5] = c->conic_o[4 * g + 3];
            l[6] = c->rgb[3 * g]; l[7] = c->rgb[3 * g + 1]; l[8] = c->rgb[3 * g + 2];
            l[9] = c->depth[g];
        }
        const float ddelx_dx = 0.5f * (float)W, ddely_dy = 0.5f * (float)H;
        for (int py = ty0; py < ty0 + TILE && py < H; py++)
            for (int px = tx0; px < tx0 + TILE && px < W; px++) {
                size_t pix = (size_t)py * W + px;
                const float T_final = c->final_T[pix];
                float T = T_final;
                int last = (int)c->n_contrib[pix];
                float gC[3] = {dL_dcolor[pix], dL_dcolor[(size_t)H * W + pix], dL_dcolor[2 * (size_t)H * W + pix]};
                float gD = dL_ddepth_img[pix], gA = dL_dalpha_img[pix];
                float bg_dot = bg[0] * gC[0] + bg[1] * gC[1] + bg[2] * gC[2];
                float last_alpha = 0.f, last_c[3] = {0, 0, 0}, last_d = 0.f;
                float acc_c[3] = {0, 0, 0}, acc_d = 0.f, acc_a = 0.f;
                float fx = (float)px, fy = (float)py;
                /* moments export: |cg| recurrence on absolute values, replay depth */
                const double bgg_abs = fabs((double)bg[0] * gC[0]) + fabs((double)bg[1] * gC[1]) + fabs((double)bg[2] * gC[2]);
                double rg_abs = 0.0, last_cg_abs = 0.0;
                int depth = 0;
                for (int j = last - 1; j >= 0; j--) {
                    const float *l = loc + 10 * j;
                    float dx = l[0] - fx, dy = l[1] - fy;
                    float power = eval_power(l[2], l[3], l[4], dx, dy);
                    if (power > 0.0f) continue;
                    float G = gs_exp(power);
                    float alpha = fminf(ALPHA_MAX, l[5] * G);
                    if (alpha < ALPHA_MIN) continue;
                    T = T / (1.0f - alpha);
                    float w = alpha * T;
                    double mq = 0.0; /* magnitude of this term's q, without phi_k */
                    if (sp) {
                        const double cg_abs = fabs((double)l[6] * gC[0]) + fabs((double)l[7] * gC[1]) + fabs((double)l[8] * gC[2]) +
                                              fabs((double)l[9] * gD) + fabs((double)gA);
                        rg_abs = (double)last_alpha * last_cg_abs + (1.0 - (double)last_alpha) * rg_abs;
                        last_cg_abs = cg_abs;
                        depth++;
                        mq = (double)G * ((double)T * (cg_abs + rg_abs) + (double)T_final * bgg_abs / (1.0 - (double)alpha));
                    }
                    float dL_dalpha = 0.f;
                    double *o = part + (size_t)(r0 + j) * 10;
                    for (int ch = 0; ch < 3; ch++) {
                        float cc = l[6 + ch];
                        acc_c[ch] = last_alpha * last_c[ch] + (1.f - last_alpha) * acc_c[ch];
                        last_c[ch] = cc;
                        dL_dalpha += (cc - acc_c[ch]) * gC[ch];
                        o[6 + ch] += w * gC[ch];
                    }
                    acc_d = last_alpha * last_d + (1.f - last_alpha) * acc_d;
                    last_d = l[9];
                    dL_dalpha += (l[9] - acc_d) * gD;
                    o[9] += w * gD;
                    acc_a = last_alpha + (1.f - last_alpha) * acc_a;
                    dL_dalpha += (1.f - acc_a) * gA;
                    dL_dalpha *= T;
                    last_alpha = alpha;
                    dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot;
                    /* straight-through the min(0.99,.) clamp, as upstream does */
                    float dL_dG = l[5] * dL_dalpha;
                    float gdx = G * dx, gdy = G * dy;
                    float dG_ddelx = -gdx * l[2] - gdy * l[3];
                    float dG_ddely = -gdy * l[4] - gdx * l[3];
                    o[0] += dL_dG * dG_ddelx * ddelx_dx;
                    o[1] += dL_dG * dG_ddely * ddely_dy;
                    o[2] += -0.5f * gdx * dx * dL_dG;
                    o[3] += -0.5f * gdx * dy * dL_dG; /* HALF of d/dB; doubled in the conic backward */
                    o[4] += -0.5f * gdy * dy * dL_dG;
                    o[5] += G * dL_dalpha;
                    if (sp) {
                        double *s = sp + (size_t)(r0 + j) * 20;
                        const double q = (double)(G * dL_dalpha), ddx = dx, ddy = dy;
                        const double phi[6] = {1.0, ddx, ddy, ddx * ddx, ddx * ddy, ddy * ddy};
                        const double wt = (double)depth + err_const + ng[c->vals[r0 + j]];
                        for (int k = 0; k < 6; k++) {
                            s[k] += q * phi[k];
                            s[10 + k] += fabs(phi[k]) * mq * wt;
                        }
                        const double gk[4] = {gC[0], gC[1], gC[2], gD};
                        for (int k = 0; k < 4; k++) {
                            const double t = (double)w * gk[k];
                            s[6 + k] += t;
                            s[16 + k] += fabs(t) * wt;
                        }
                    }
                }
            }
        free(loc);
    }
    /* deterministic reduction to per-Gaussian screen-space gradients: every thread owns a contiguous range of Gaussian
     * ids, scans the whole sorted list and adds the instances of ITS Gaussians in list order -- the same order of additions
     * per Gaussian as a serial pass, for any thread count */
    double *gs = (double *)malloc((size_t)(P > 0 ? P : 1) * 10 * sizeof(double));
#pragma omp parallel
    {
#ifdef _OPENMP
        const int nt = omp_get_num_threads(), it = omp_get_thread_num();
#else
        const int nt = 1, it = 0;
#endif
        const uint32_t lo = (uint32_t)((uint64_t)P * it / nt), hi = (uint32_t)((uint64_t)P * (it + 1) / nt);
        if (hi > lo) memset(gs + (size_t)lo * 10, 0, sizeof(double) * 10 * (size_t)(hi - lo));
        for (int64_t j = 0; j < D; j++) {
            const uint32_t g = c->vals[j];
            if (g < lo || g >= hi) continue;
            double *d = gs + (size_t)g * 10;
            const double *s = part + (size_t)j * 10;
            for (int k = 0; k < 10; k++) d[k] += s[k];
        }
        if (sp) {
            if (hi > lo) {
                memset(sums_out + (size_t)lo * 10, 0, sizeof(double) * 10 * (size_t)(hi - lo));
                memset(err_out + (size_t)lo * 10, 0, sizeof(double) * 10 * (size_t)(hi - lo));
            }
            for (int64_t j = 0; j < D; j++) {
                const uint32_t g = c->vals[j];
                if (g < lo || g >= hi) continue;
                const double *s = sp + (size_t)j * 20;
                for (int k = 0; k < 10; k++) {
                    sums_out[(size_t)g * 10 + k] += s[k];
                    err_out[(size_t)g * 10 + k] += s[10 + k];
                }
            }
        }
    }
    free(part);
    free(sp);
    free(ng);
    if (screen_out) memcpy(screen_out, gs, sizeof(double) * 10 * (size_t)P);

    const int Mc = c->M;
    const float *V = c->view, *PV = c->proj;
    memset(dL_dmeans3D, 0, sizeof(float) * 3 * P);
    memset(dL_dmeans2D, 0, sizeof(float) * 3 * P);
    memset(dL_dopacity, 0, sizeof(float) * P);
    if (dL_dsh) memset(dL_dsh, 0, sizeof(float) * 3 * (size_t)Mc * P);
    if (dL_dcolors) memset(dL_dcolors, 0, sizeof(float) * 3 * P);
    if (dL_dscales) memset(dL_dscales, 0, sizeof(float) * 3 * P);
    if (dL_drots) memset(dL_drots, 0, sizeof(float) * 4 * P);
    if (dL_dcov3D) memset(dL_dcov3D, 0, sizeof(float) * 6 * P);

#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; i++) {
        if (!(c->radii[i] > 0)) continue;
        float g[10];
        for (int k = 0; k < 10; k++) g[k] = (float)gs[(size_t)i * 10 + k];
        const float px = c->means[3 * i], py = c->means[3 * i + 1], pz = c->means[3 * i + 2];
        dL_dmeans2D[3 * i] = g[0]; dL_dmeans2D[3 * i + 1] = g[1]; dL_dmeans2D[3 * i + 2] = 0.f;
        dL_dopacity[i] = g[5];
        /* ---- B2: conic -> cov2D -> cov3D and mean (A.6) ---- */
        const float *c6 = c->cov3d + 6 * i;
        float tx = affine(V[0], V[4], V[8], V[12], px, py, pz);
        float ty = affine(V[1], V[5], V[9], V[13], px, py, pz);
        float tz = affine(V[2], V[6], V[10], V[14], px, py, pz);
        float fx = (float)W / (2.0f * c->tanfovx), fy = (float)H / (2.0f * c->tanfovy);
        float limx = 1.3f * c->tanfovx, limy = 1.3f * c->tanfovy;
        float txtz = tx / tz, tytz = ty / tz;
        float cx = fminf(limx, fmaxf(-limx, txtz)) * tz;
        float cy = fminf(limy, fmaxf(-limy, tytz)) * tz;
        float xmul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
        float ymul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
        float J00 = fx / tz, J11 = fy / tz, J02 = -(fx * cx) / (tz * tz), J12 = -(fy * cy) / (tz * tz);
        float M0[3], M1[3], Wm[3][3];
        for (int k = 0; k < 3; k++) {
            Wm[0][k] = V[4 * k]; Wm[1][k] = V[4 * k + 1]; Wm[2][k] = V[4 * k + 2];
            M0[k] = J00 * Wm[0][k] + J02 * Wm[2][k];
            M1[k] = J11 * Wm[1][k] + J12 * Wm[2][k];
        }
        float S[3][3] = {{c6[0], c6[1], c6[2]}, {c6[1], c6[3], c6[4]}, {c6[2], c6[4], c6[5]}};
        float N0[3], N1[3];
        for (int k = 0; k < 3; k++) {
            N0[k] = M0[0] * S[0][k] + M0[1] * S[1][k] + M0[2] * S[2][k];
            N1[k] = M1[0] * S[0][k] + M1[1] * S[1][k] + M1[2] * S[2][k];
        }
        float a = N0[0] * M0[0] + N0[1] * M0[1] + N0[2] * M0[2] + DILATE;
        float b = N0[0] * M1[0] + N0[1] * M1[1] + N0[2] * M1[2];
        float cc = N1[0] * M1[0] + N1[1] * M1[1] + N1[2] * M1[2] + DILATE;
        float denom = a * cc - b * b;
        float d2inv = 1.0f / (denom * denom + 0.0000001f);
        float dA = g[2], dBh = g[3], dC = g[4];
        float da = 0, db = 0, dc = 0;
        float dcov[6] = {0, 0, 0, 0, 0, 0};
        float dmean[3] = {0, 0, 0};
        if (d2inv != 0.f) {
            /* (denom - a*c) == -b*b and (denom + 2*b*b) == a*c + b*b, written without the cancellation */
            da = d2inv * (-cc * cc * dA + 2.f * b * cc * dBh - b * b * dC);
            dc = d2inv * (-a * a * dC + 2.f * a * b * dBh - b * b * dA);
            db = d2inv * 2.f * (b * cc * dA - (a * cc + b * b) * dBh + a * b * dC);
            dcov[0] = M0[0] * M0[0] * da + M0[0] * M1[0] * db + M1[0] * M1[0] * dc;
            dcov[3] = M0[1] * M0[1] * da + M0[1] * M1[1] * db + M1[1] * M1[1] * dc;
            dcov[5] = M0[2] * M0[2] * da + M0[2] * M1[2] * db + M1[2] * M1[2] * dc;
            dcov[1] = 2.f * M0[0] * M0[1] * da + (M0[0] * M1[1] + M0[1] * M1[0]) * db + 2.f * M1[0] * M1[1] * dc;
            dcov[2] = 2.f * M0[0] * M0[2] * da + (M0[0] * M1[2] + M0[2] * M1[0]) * db + 2.f * M1[0] * M1[2] * dc;
            dcov[4] = 2.f * M0[2] * M0[1] * da + (M0[1] * M1[2] + M0[2] * M1[1]) * db + 2.f * M1[1] * M1[2] * dc;
            float dM0[3], dM1[3];
            for (int k = 0; k < 3; k++) {
                dM0[k] = 2.f * da * N0[k] + db * N1[k];
                dM1[k] = db * N0[k] + 2.f * dc * N1[k];
            }
            float dJ00 = Wm[0][0] * dM0[0] + Wm[0][1] * dM0[1] + Wm[0][2] * dM0[2];
            float dJ02 = Wm[2][0] * dM0[0] + Wm[2][1] * dM0[1] + Wm[2][2] * dM0[2];
            float dJ11 = Wm[1][0] * dM1[0] + Wm[1][1] * dM1[1] + Wm[1][2] * dM1[2];
            float dJ12 = Wm[2][0] * dM1[0] + Wm[2][1] * dM1[1] + Wm[2][2] * dM1[2];
            float itz = 1.f / tz, itz2 = itz * itz, itz3 = itz2 * itz;
            float dtx = xmul * -fx * itz2 * dJ02;
            float dty = ymul * -fy * itz2 * dJ12;
            float dtz = -fx * itz2 * dJ00 - fy * itz2 * dJ11 + (2.f * fx * cx) * itz3 * dJ02 + (2.f * fy * cy) * itz3 * dJ12;
            for (int k = 0; k < 3; k++) dmean[k] = Wm[0][k] * dtx + Wm[1][k] * dty + Wm[2][k] * dtz;
        }
        /* ---- B3: projection, depth, SH (A.7) ---- */
        float hw = affine(PV[3], PV[7], PV[11], PV[15], px, py, pz);
        float m_w = 1.0f / (hw + 0.0000001f);
        float mul1 = (PV[0] * px + PV[4] * py + PV[8] * pz + PV[12]) * m_w * m_w;
        float mul2 = (PV[1] * px + PV[5] * py + PV[9] * pz + PV[13]) * m_w * m_w;
        for (int k = 0; k < 3; k++) {
            dmean[k] += (PV[4 * k] * m_w - PV[4 * k + 3] * mul1) * g[0] + (PV[4 * k + 1] * m_w - PV[4 * k + 3] * mul2) * g[1];
        }
        /* depth = row 2 of the view transform (fork addition); w-row terms vanish for affine V */
        float mul3 = V[2] * px + V[6] * py + V[10] * pz + V[14];
        for (int k = 0; k < 3; k++) dmean[k] += (V[4 * k + 2] - V[4 * k + 3] * mul3) * g[9];

        if (c->shs) {
            float dx = px - c->campos[0], dy = py - c->campos[1], dz = pz - c->campos[2];
            float len = sqrtf(dx * dx + dy * dy + dz * dz);
            float x = dx / len, y = dy / len, z = dz / len;
            float bs[16];
            sh_basis(c->deg, x, y, z, bs);
            int nb = (c->deg + 1) * (c->deg + 1);
            const float *sh = c->shs + (size_t)i * Mc * 3;
            float dRGB[3];
            for (int ch = 0; ch < 3; ch++) dRGB[ch] = c->clamped[3 * i + ch] ? 0.f : g[6 + ch];
            float *dsh = dL_dsh + (size_t)i * Mc * 3;
            for (int k = 0; k < nb; k++)
                for (int ch = 0; ch < 3; ch++) dsh[3 * k + ch] = bs[k] * dRGB[ch];
            if (c->deg > 0) {
                /* s_k = sum_ch sh[k][ch]*dRGB[ch]; dL/ddir = sum_k d(b_k)/d(dir) * s_k */
                float s[16];
                for (int k = 0; k < nb; k++)
                    s[k] = sh[3 * k] * dRGB[0] + sh[3 * k + 1] * dRGB[1] + sh[3 * k + 2] * dRGB[2];
                float ddx = -SH_C1 * s[3], ddy = -SH_C1 * s[1], ddz = SH_C1 * s[2];
                if (c->deg > 1) {
                    float xx = x * x, yy = y * y, zz = z * z;
                    ddx += SH_C2[0] * y * s[4] + SH_C2[2] * -2.f * x * s[6] + SH_C2[3] * z * s[7] + SH_C2[4] * 2.f * x * s[8];
                    ddy += SH_C2[0] * x * s[4] + SH_C2[1] * z * s[5] + SH_C2[2] * -2.f * y * s[6] + SH_C2[4] * -2.f * y * s[8];
                    ddz += SH_C2[1] * y * s[5] + SH_C2[2] * 4.f * z * s[6] + SH_C2[3] * x * s[7];
                    if (c->deg > 2) {
                        ddx += SH_C3[0] * s[9] * 6.f * x * y + SH_C3[1] * s[10] * y * z + SH_C3[2] * s[11] * -2.f * x * y +
                               SH_C3[3] * s[12] * -6.f * x * z + SH_C3[4] * s[13] * (4.f * zz - 3.f * xx - yy) +
                               SH_C3[5] * s[14] * 2.f * x * z + SH_C3[6] * s[15] * 3.f * (xx - yy);
                        ddy += SH_C3[0] * s[9] * 3.f * (xx - yy) + SH_C3[1] * s[10] * x * z +
                               SH_C3[2] * s[11] * (4.f * zz - xx - 3.f * yy) + SH_C3[3] * s[12] * -6.f * y * z +
                               SH_C3[4] * s[13] * -2.f * x * y + SH_C3[5] * s[14] * -2.f * y * z + SH_C3[6] * s[15] * -6.f * x * y;
                        ddz += SH_C3[1] * s[10] * x * y + SH_C3[2] * s[11] * 8.f * y * z +
                               SH_C3[3] * s[12] * 3.f * (2.f * zz - xx - yy) + SH_C3[4] * s[13] * 8.f * x * z +
                               SH_C3[5] * s[14] * (xx - yy);
                    }
                }
                /* through dir = v/|v| */
                float dot = x * ddx + y * ddy + z * ddz;
                dmean[0] += (ddx - x * dot) / len;
                dmean[1] += (ddy - y * dot) / len;
                dmean[2] += (ddz - z * dot) / len;
            }
        } else if (dL_dcolors) {
            dL_dcolors[3 * i] = g[6]; dL_dcolors[3 * i + 1] = g[7]; dL_dcolors[3 * i + 2] = g[8];
        }
        dL_dmeans3D[3 * i] = dmean[0]; dL_dmeans3D[3 * i + 1] = dmean[1]; dL_dmeans3D[3 * i + 2] = dmean[2];

        if (c->cov_pre) {
            if (dL_dcov3D) memcpy(dL_dcov3D + 6 * i, dcov, 24);
        } else {
            /* ---- cov3D -> scale, rotation (no normalisation Jacobian: Python's F.normalize supplies it) ---- */
            const float *q = c->rots + 4 * i;
            float r = q[0], x = q[1], y = q[2], z = q[3];
            float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                             {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                             {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
            float s[3] = {c->mod * c->scales[3 * i], c->mod * c->scales[3 * i + 1], c->mod * c->scales[3 * i + 2]};
            float dS[3][3] = {{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]},
                              {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]},
                              {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}};
            float L[3][3], dLm[3][3], dR[3][3];
            for (int a2 = 0; a2 < 3; a2++)
                for (int k = 0; k < 3; k++) L[a2][k] = R[a2][k] * s[k];
            for (int a2 = 0; a2 < 3; a2++)
                for (int k = 0; k < 3; k++)
                    dLm[a2][k] = 2.f * (dS[a2][0] * L[0][k] + dS[a2][1] * L[1][k] + dS[a2][2] * L[2][k]);
            for (int k = 0; k < 3; k++) {
                dL_dscales[3 * i + k] = c->mod * (R[0][k] * dLm[0][k] + R[1][k] * dLm[1][k] + R[2][k] * dLm[2][k]);
                for (int a2 = 0; a2 < 3; a2++) dR[a2][k] = dLm[a2][k] * s[k];
            }
            dL_drots[4 * i + 0] = 2.f * z * (dR[1][0] - dR[0][1]) + 2.f * y * (dR[0][2] - dR[2][0]) + 2.f * x * (dR[2][1] - dR[1][2]);
            dL_drots[4 * i + 1] = 2.f * y * (dR[0][1] + dR[1][0]) + 2.f * z * (dR[0][2] + dR[2][0]) + 2.f * r * (dR[2][1] - dR[1][2]) - 4.f * x * (dR[1][1] + dR[2][2]);
            dL_drots[4 * i + 2] = 2.f * x * (dR[0][1] + dR[1][0]) + 2.f * r * (dR[0][2] - dR[2][0]) + 2.f * z * (dR[1][2] + dR[2][1]) - 4.f * y * (dR[0][0] + dR[2][2]);
            dL_drots[4 * i + 3] = 2.f * r * (dR[1][0] - dR[0][1]) + 2.f * x * (dR[0][2] + dR[2][0]) + 2.f * y * (dR[1][2] + dR[2][1]) - 4.f * z * (dR[0][0] + dR[1][1]);
        }
    }
    free(gs);
    return 0;
}

/* the scalar exp, exported so tests can pin it bit-for-bit against the CUDA copy */
float gso_exp(float x) { return gs_exp(x); }
