// common.cuh -- shared device helpers and buffer layouts of the b200gs rasteriser (sm_90a).
//
// NUMERICAL CONTRACT (DESIGN.md "Numerical contract"): everything that decides an index or a branch
// is written with an explicit IEEE-754 binary32 operation order, using the *_rn intrinsics so that the
// result does not depend on nvcc's -fmad setting.  The CPU oracle (oracle/gs_oracle.c) states the same
// sequence independently; tests/ compare the two bit-for-bit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define GS_TILE 16
#define GS_TILE_PIX 256
#define GS_NEAR_Z 0.2f
#define GS_DILATE 0.3f
#define GS_ALPHA_MAX 0.99f
#define GS_ALPHA_MIN (1.0f / 255.0f)
#define GS_T_MIN 0.0001f
#define GS_MAX_VIEWS 64

// ---- pinned-order float arithmetic -------------------------------------------------------------
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float fsqrt(float a) { return __fsqrt_rn(a); }

// deterministic exp for x <= 0: Cody-Waite range reduction + degree-5 polynomial, 8 FMA-pipe ops.
// |relative error| < 2e-7 on [-87, 0].  Bit-identical to gs_exp() in oracle/gs_oracle.c.
__device__ __forceinline__ float gs_exp(float x)
{
    x = fmaxf(x, -87.0f);
    float t = ffma(x, 0x1.715476p+0f, 12582912.0f);
    float n = fsub(t, 12582912.0f);
    float r = ffma(n, -0x1.62e430p-1f, x);
    float p = 0x1.0fa834p-7f;
    p = ffma(p, r, 0x1.573a54p-5f);
    p = ffma(p, r, 0x1.555a6ap-3f);
    p = ffma(p, r, 0x1.fffdc6p-2f);
    p = ffma(p, r, 0x1.fffff6p-1f);
    p = ffma(p, r, 1.0f);
    return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}

// -0.5*(A dx^2 + C dy^2) - B dx dy   evaluated as   dx*(-A/2*dx - B*dy) + (-C/2*dy)*dy
__device__ __forceinline__ float gs_power(float A, float B, float C, float dx, float dy)
{
    float u = ffma(-B, dy, fmul(fmul(-0.5f, A), dx));
    float w = fmul(fmul(fmul(-0.5f, C), dy), dy);
    return ffma(dx, u, w);
}

// m0*x + m1*y + m2*z + m3  as  mul, fma, fma, add
__device__ __forceinline__ float gs_affine(float m0, float m1, float m2, float m3, float x, float y, float z)
{
    float a = fmul(m0, x);
    a = ffma(m1, y, a);
    a = ffma(m2, z, a);
    return fadd(a, m3);
}
__device__ __forceinline__ float gs_dot3(float a0, float a1, float a2, float b0, float b1, float b2)
{
    float a = fmul(a0, b0);
    a = ffma(a1, b1, a);
    return ffma(a2, b2, a);
}

// ---- per-(view,Gaussian) geometry record: 48 B, three 16-B words ----------------------------------
struct __align__(16) GeomRec {
    float px, py;    // pixel-space centre
    float hx, hy;    // conservative half extents of the alpha >= 1/255 support (product-only; <0 = never visible)
    float A, B, C;   // conic (inverse 2D covariance)
    float o;         // opacity
    float r, g, b;   // colour after SH / clamp
    float depth;     // view-space z
};
static_assert(sizeof(GeomRec) == 48, "GeomRec must be 48 bytes");

// per-(view,Gaussian) screen-space gradient accumulator written by the backward blend: 48 B, ten floats + padding.
// blend_sgrad_is_moments() tells which of two formats the linked blend writes (fields below: classic | product):
//   product blend (blend.cu, moments of q = G*dL/dalpha, dx = px_gauss - px, dy = py_gauss - py; w = alpha*T):
//     S0, Sx, Sy, Sxx | Sxy, Syy, W0, W1 | W2, W3  =  sum q*{1, dx, dy, dx^2 | dx*dy, dy^2}, sum w*{gC0, gC1 | gC2, gD}
//   classic comparator (baseline/classic_blend.cu): the screen-space gradients themselves, as named below.
// preprocess_bwd turns the moments into the classic quantities (the conic / mean combination is linear).
struct __align__(16) ScreenGrad {
    float dx, dy;        // dL/dmean2D (NDC-scaled)              | product: S0, Sx
    float dA, dBh, dC;   // dL/dconic (dBh = half of d/dB)        | product: Sy, Sxx, Sxy
    float dO;            // dL/dopacity                           | product: Syy
    float dr, dg, db;    // dL/dcolour                            | product: W0, W1, W2 = sum w*gC
    float dDepth;        // dL/ddepth                             | product: W3 = sum w*gD
    float pad0, pad1;
};
static_assert(sizeof(ScreenGrad) == 48, "ScreenGrad must be 48 bytes");

__host__ __device__ inline size_t gs_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// ---- opaque state buffer layouts (host side computes offsets; all 256-B aligned) ---------------------
struct GeomLayout {
    size_t recs, tiles_touched, offsets, rects, clamped, total;
    __host__ GeomLayout(int P, int V)
    {
        size_t n = (size_t)P * V, o = 0;
        recs = o; o += gs_align(n * sizeof(GeomRec));
        tiles_touched = o; o += gs_align(n * 4);
        offsets = o; o += gs_align(n * 4);
        rects = o; o += gs_align(n * 8);
        clamped = o; o += gs_align(n);
        total = o;
    }
};
struct ImageLayout {
    size_t final_T, n_contrib, total;
    __host__ ImageLayout(int H, int W, int V)
    {
        size_t n = (size_t)H * W * V, o = 0;
        final_T = o; o += gs_align(n * 4);
        n_contrib = o; o += gs_align(n * 4);
        total = o;
    }
};
