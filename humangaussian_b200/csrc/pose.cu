// pose.cu -- pose maps (humangaussian_b200/pose.py): the skeleton images of HumanSD and OpenPose style for a batch of
// views, in two launches.
//
// pose_setup_kernel (one CTA per view): projects the keypoints in a fixed float32 order, applies the occlusion and
// validity rules, and rasterises every shape of the view into up to 4 disjoint runs [lo, hi] per row (scratch
// [V][S][H][4] int2).  One thread owns one shape, so each row has one writer and no atomics are needed.  The rasterisation restates cv2's
// integer drawing rules exactly (tests/pose_reference.py is the specification; DESIGN.md section 2):
//   thick line   segment clipped to the image widened by T; 16.16 rectangle filled by the convex scan converter with
//                its edges drawn as clipped fixed-point lines; discs of radius (T + 1) / 2 on the clipped ends
//   circle       the integer disc dx^2 + dy^2 <= r^2
//   ellipse      ellipse2Poly over a 7-decimal integer-degree sine table, then the convex scan converter at shift 0
//                with 8-connected integer edges
// A cv2 shape is not always one run per row: a thin limb's edge pixels can leave a one-pixel gap.  Four runs per row
// hold every shape seen in the tests (at most two occur); the tests compare the draw with the specification bit for bit.
// pose_draw_kernel: one thread per 4 pixels of a row; each pixel walks the view's shapes in draw order (overwrite for
// HumanSD; for OpenPose circles overwrite, then each limb blends rint(c * 0.4f + colour * 0.6f)) and stores u8 / 255.
// The limb table and the shape colours come from the caller (pose.py holds the style tables) in the argument block.
#include <climits>
#include <cstdint>

#include "common.cuh"
#include "kernels.h"

namespace {

using i64 = long long; // the type of longlong2 components

__device__ __forceinline__ i64 div0(i64 a, i64 b) { return a / b; } // rounds toward zero

constexpr int XY_SHIFT = 16;
constexpr i64 XY_ONE = 1LL << XY_SHIFT;
constexpr i64 HALF = XY_ONE >> 1;
constexpr int HSD_K = 17, HSD_L = 16, OP_K = 18, OP_L = 17;
constexpr int MAX_POLY = 361; // ellipse2Poly(0..360 step 1) before duplicate removal
constexpr float COORD_LIMIT = 1048576.f; // 2^20 px
constexpr int SLOTS = 4;                 // disjoint runs per shape and row (cv2 can leave a one-pixel gap in a thin limb)


struct ShapeRows { // one shape's pixels per row as up to SLOTS disjoint runs [lo, hi] (scratch), clipped to the image
    int2 *rows;
    int W, H;
    __device__ void run(i64 y, i64 x0, i64 x1) const
    {
        if (y < 0 || y >= H) return;
        if (x0 < 0) x0 = 0;
        if (x1 > W - 1) x1 = W - 1;
        if (x0 > x1) return;
        int2 *s = rows + y * SLOTS, keep[SLOTS];
        int n = 0;
        for (int i = 0; i < SLOTS; ++i) { // absorb every run that overlaps or touches [x0, x1]
            const int2 r = s[i];
            if (r.x > r.y) break;
            if (r.y + 1 < x0 || r.x > x1 + 1) keep[n++] = r;
            else { x0 = min(x0, (i64)r.x); x1 = max(x1, (i64)r.y); }
        }
        if (n == SLOTS) { // never seen (at most 2 runs per row on any tested shape): keep the row's hull of the last two
            x0 = min(x0, (i64)keep[SLOTS - 1].x);
            x1 = max(x1, (i64)keep[SLOTS - 1].y);
            --n;
        }
        keep[n++] = make_int2((int)x0, (int)x1);
        for (int i = 0; i < SLOTS; ++i) s[i] = i < n ? keep[i] : make_int2(1, 0);
    }
};


// The part of a segment inside [0, w - 1] x [0, h - 1] (any fixed point), as cv2 keeps it (tests/pose_reference.py,
// clip_line): false when the segment misses.  Ends are slid onto the top / bottom border first, then onto the left /
// right one; the first end moves before the second, whose slide follows the line through the moved first end; each
// slide is trunc(double(border - c) * double(d_other) / double(d_axis)).
__device__ __forceinline__ int side_of(i64 c, i64 lim) { return c < 0 ? -1 : (c > lim ? 1 : 0); }

__device__ bool clip_line(i64 w, i64 h, i64 &x1, i64 &y1, i64 &x2, i64 &y2)
{
    i64 *p[2] = {&x1, &y1}, *q[2] = {&x2, &y2};
    const i64 lim[2] = {w - 1, h - 1};
    for (int a = 1; a >= 0; --a) {
        for (int b = 0; b < 2; ++b) {
            const int sp = side_of(*p[b], lim[b]);
            if (sp != 0 && sp == side_of(*q[b], lim[b])) return false; // both ends beyond one border
        }
        const int o = 1 - a;
        for (int e = 0; e < 2; ++e) {
            i64 **end = e == 0 ? p : q;
            const int s = side_of(*end[a], lim[a]);
            if (s == 0) continue;
            const i64 border = s < 0 ? 0 : lim[a];
            *end[o] += __double2ll_rz(__ddiv_rn(__dmul_rn((double)(border - *end[a]), (double)(*q[o] - *p[o])),
                                                (double)(*q[a] - *p[a])));
            *end[a] = border;
        }
    }
    return true;
}

// pixels of a walk, merged into runs of adjacent pixels before they reach the shape's rows
struct RunBuf {
    const ShapeRows &h;
    i64 y = LLONG_MIN, x0 = 0, x1 = -1;
    __device__ explicit RunBuf(const ShapeRows &hh) : h(hh) {}
    __device__ void px(i64 x, i64 yy)
    {
        if (yy != y || x < x0 - 1 || x > x1 + 1) { flush(); y = yy; x0 = x1 = x; return; } // a new run unless adjacent
        x0 = min(x0, x);
        x1 = max(x1, x);
    }
    __device__ void flush() { if (y != LLONG_MIN) h.run(y, x0, x1); }
};

// a 16.16 polygon edge (cv2's fixed-point line): clipped, walked along the major axis in increasing order
__device__ void line_fixed(const ShapeRows &h, i64 x1, i64 y1, i64 x2, i64 y2)
{
    if (!clip_line((i64)h.W << XY_SHIFT, (i64)h.H << XY_SHIFT, x1, y1, x2, y2)) return;
    RunBuf rb(h);
    const i64 ax = x2 > x1 ? x2 - x1 : x1 - x2, ay = y2 > y1 ? y2 - y1 : y1 - y2;
    if (ax > ay) {
        if (x2 < x1) { i64 t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
        const i64 step = div0((y2 - y1) * XY_ONE, (x2 - x1) | 1), n = (x2 - x1) >> XY_SHIFT;
        const i64 xs = (x1 + HALF) >> XY_SHIFT;
        for (i64 k = 0; k <= n; ++k) rb.px(xs + k, (y1 + HALF + step * k) >> XY_SHIFT);
    } else {
        if (y2 < y1) { i64 t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
        const i64 step = div0((x2 - x1) * XY_ONE, (y2 - y1) | 1), n = (y2 - y1) >> XY_SHIFT;
        const i64 ys = (y1 + HALF) >> XY_SHIFT;
        for (i64 k = 0; k <= n; ++k) rb.px((x1 + HALF + step * k) >> XY_SHIFT, ys + k);
    }
    rb.px((x2 + HALF) >> XY_SHIFT, (y2 + HALF) >> XY_SHIFT);
    rb.flush();
}

// an 8-connected integer edge (fillConvexPoly at shift 0): clipped when an end is outside, walked left to right
__device__ void line_int(const ShapeRows &h, i64 x1, i64 y1, i64 x2, i64 y2)
{
    if (!(x1 >= 0 && x1 < h.W && x2 >= 0 && x2 < h.W && y1 >= 0 && y1 < h.H && y2 >= 0 && y2 < h.H))
        if (!clip_line(h.W, h.H, x1, y1, x2, y2)) return;
    if (x2 < x1) { i64 t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; }
    const i64 dx = x2 - x1, sy = y2 < y1 ? -1 : 1, dy = y2 < y1 ? y1 - y2 : y2 - y1;
    RunBuf rb(h);
    if (dy > dx) {
        for (i64 k = 0; k <= dy; ++k) rb.px(x1 + (2 * dx * k + dy - 1) / (2 * dy), y1 + sy * k);
    } else {
        for (i64 k = 0; k <= dx; ++k) rb.px(x1 + k, y1 + sy * (dx ? (2 * dy * k + dx - 1) / (2 * dx) : 0));
    }
    rb.flush();
}

// One side of the scanline fill (tests/pose_reference.py, _chain): walking from the top vertex in direction `step`,
// the edge that covers a row is the next one ending below the row reached so far (edges that do not are passed over);
// x at a row is the edge's start x plus whole per-row steps, the step being its 16.16 run over its rows plus one half,
// truncated toward zero.
template <class Vert>
struct FillSide {
    const Vert &V;
    int n, step, s;     // s: start vertex of the current edge
    i64 r0, r1, x0, dx; // rows [r0, r1), x at r0, x step (16.16)
    int shift;
    __device__ FillSide(const Vert &v, int n_, int step_, int top, i64 top_row, int shift_)
        : V(v), n(n_), step(step_), s(top), r0(top_row), r1(top_row), x0(0), dx(0), shift(shift_) {}
    __device__ i64 row_of(int i) const { return (V(i).y + ((1LL << shift) >> 1)) >> shift; }
    __device__ i64 x_at(i64 y) // y never decreases between calls
    {
        for (int guard = 0; r1 <= y && guard < n; ++guard) {
            const int j = (s + step) % n;
            const i64 rj = row_of(j);
            if (rj > r1) {
                const i64 L = rj - r1, xs = V(s).x << (XY_SHIFT - shift), xe = V(j).x << (XY_SHIFT - shift);
                r0 = r1;
                r1 = rj;
                x0 = xs;
                dx = ((xe - xs) * 2 + L) / (2 * L); // C division: toward zero
            }
            s = j;
        }
        return x0 + dx * (y - r0);
    }
};

// cv2's fillConvexPoly for a convex polygon of n vertices (`shift` fixed point; V(i) returns vertex i): the outline,
// then one run per row between the two sides, from the top vertex's row to the row above the bottom vertex's.
template <class Vert>
__device__ void fill_convex(const ShapeRows &h, int n, int shift, Vert V)
{
    for (int i = 0; i < n; ++i) {
        const longlong2 a = V(i == 0 ? n - 1 : i - 1), b = V(i);
        if (shift == 0) line_int(h, a.x, a.y, b.x, b.y);
        else line_fixed(h, a.x, a.y, b.x, b.y);
    }
    if (n < 3) return;
    const i64 half = (1LL << shift) >> 1;
    int top = 0;
    i64 top_row = LLONG_MAX, bottom_row = LLONG_MIN, px_min = LLONG_MAX, px_max = LLONG_MIN;
    for (int i = 0; i < n; ++i) {
        const longlong2 p = V(i);
        const i64 r = (p.y + half) >> shift, c = (p.x + half) >> shift;
        if (r < top_row) { top_row = r; top = i; }
        bottom_row = max(bottom_row, r);
        px_min = min(px_min, c);
        px_max = max(px_max, c);
    }
    if (px_max < 0 || bottom_row < 0 || px_min >= h.W || top_row >= h.H) return;
    FillSide<Vert> left(V, n, 1, top, top_row, shift), right(V, n, n - 1, top, top_row, shift);
    const i64 y_end = min(bottom_row, (i64)h.H);
    for (i64 y = max(top_row, (i64)0); y < y_end; ++y) {
        const i64 xl = left.x_at(y), xr = right.x_at(y);
        h.run(y, (min(xl, xr) + HALF) >> XY_SHIFT, (max(xl, xr) + HALF) >> XY_SHIFT);
    }
}

// cv2.circle(img, c, r, colour, -1): the integer disc dx^2 + dy^2 <= r^2
__device__ void circle_filled(const ShapeRows &h, i64 cx, i64 cy, int r)
{
    for (i64 d = -r; d <= r; ++d) {
        if (cy + d < 0 || cy + d >= h.H) continue;
        i64 hw = (i64)sqrt((double)((i64)r * r - d * d)); // exact for r < 2^26, corrected below to the integer root
        while (hw * hw > (i64)r * r - d * d) --hw;
        while ((hw + 1) * (hw + 1) <= (i64)r * r - d * d) ++hw;
        h.run(cy + d, cx - hw, cx + hw);
    }
}

// cv2.line(img, p0, p1, colour, T), LINE_8, T >= 2 (tests/pose_reference.py, thick_line): the segment clipped to the
// image widened by T; unless its ends coincide, the rectangle of half-width ceil(T / 2) around it, its corners the ends
// offset by (rint(dy * f), rint(dx * f)) in 16.16 with f = half-width (16.16) / |d|; a disc of radius (T + 1) / 2 on
// each clipped end.
__device__ void thick_line(const ShapeRows &h, i64 x0, i64 y0, i64 x1, i64 y1, int T)
{
    x0 += T; y0 += T; x1 += T; y1 += T;
    if (!clip_line(h.W + 2 * T, h.H + 2 * T, x0, y0, x1, y1)) return;
    x0 -= T; y0 -= T; x1 -= T; y1 -= T;
    if (x0 != x1 || y0 != y1) {
        const double dx = (double)(x0 - x1), dy = (double)(y1 - y0);
        const double f = __ddiv_rn((double)((i64)((T + 1) / 2) << XY_SHIFT), __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy))));
        const i64 ox = __double2ll_rn(__dmul_rn(dy, f)), oy = __double2ll_rn(__dmul_rn(dx, f));
        const i64 ax = x0 << XY_SHIFT, ay = y0 << XY_SHIFT, bx = x1 << XY_SHIFT, by = y1 << XY_SHIFT;
        const longlong2 q[4] = {{ax + ox, ay + oy}, {ax - ox, ay - oy}, {bx - ox, by - oy}, {bx + ox, by + oy}};
        fill_convex(h, 4, XY_SHIFT, [&](int i) { return q[i]; });
    }
    circle_filled(h, x0, y0, (T + 1) / 2);
    circle_filled(h, x1, y1, (T + 1) / 2);
}

// ellipse2Poly((cx, cy), (a, b), angle, 0, 360, 1) into poly; returns the vertex count
__device__ int ellipse2poly(const float *sin_t, int cx, int cy, int a, int b, int angle, int2 *poly)
{
    while (angle < 0) angle += 360;
    while (angle > 360) angle -= 360;
    const double alpha = sin_t[450 - angle], beta = sin_t[angle];
    int n = 0;
    int2 prev = make_int2(INT32_MIN, INT32_MIN);
    for (int i = 0; i <= 360; ++i) {
        const double x = __dmul_rn((double)a, (double)sin_t[450 - i]), y = __dmul_rn((double)b, (double)sin_t[i]);
        const double px = __dsub_rn(__dadd_rn((double)cx, __dmul_rn(x, alpha)), __dmul_rn(y, beta));
        const double py = __dadd_rn(__dadd_rn((double)cy, __dmul_rn(x, beta)), __dmul_rn(y, alpha));
        const int2 pt = make_int2(__double2int_rn(px), __double2int_rn(py));
        if (pt.x != prev.x || pt.y != prev.y) { poly[n++] = pt; prev = pt; }
    }
    if (n == 1) { poly[0] = poly[1] = make_int2(cx, cy); n = 2; }
    return n;
}

// float32 mean, length and double atan2 in degrees of an OpenPose limb, truncated as the reference truncates them
__device__ void limb_geometry(float xa, float ya, float xb, float yb, int &cx, int &cy, int &half_len, int &angle)
{
    cx = __float2int_rz(__fmul_rn(__fadd_rn(xa, xb), 0.5f));
    cy = __float2int_rz(__fmul_rn(__fadd_rn(ya, yb), 0.5f));
    const float dY = __fsub_rn(ya, yb), dX = __fsub_rn(xa, xb);
    const float len = __fsqrt_rn(__fadd_rn(__fmul_rn(dY, dY), __fmul_rn(dX, dX)));
    half_len = __float2int_rz(__fmul_rn(len, 0.5f));
    double deg;
    if (fabsf(dY) == fabsf(dX) && dX != 0.f) deg = dX > 0.f ? (dY > 0.f ? 45.0 : -45.0) : (dY > 0.f ? 135.0 : -135.0);
    else deg = __dmul_rn(atan2((double)dY, (double)dX), 180.0 / 3.141592653589793);
    angle = (int)deg; // truncation toward zero, as Python's int()
}

__global__ void __launch_bounds__(64) pose_setup_kernel(PoseArgs a)
{
    const int v = blockIdx.x, t = threadIdx.x;
    const bool hsd = a.style == 0;
    const int K = hsd ? HSD_K : OP_K;
    __shared__ float xs[OP_K], ys[OP_K], zs[OP_K];
    __shared__ bool ok[OP_K];
    __shared__ float sin_t[451];
    for (int i = t; i <= 450; i += blockDim.x) { // float32(round(sin(i deg), 7))
        const double s = sin(__dmul_rn((double)i, 3.141592653589793 / 180.0));
        sin_t[i] = (float)__ddiv_rn(rint(__dmul_rn(s, 1e7)), 1e7);
    }
    if (t < K) {
        const float4 p = reinterpret_cast<const float4 *>(a.points)[t];
        const float *m = a.mvp + (size_t)v * 16;
        float c[4];
        for (int r = 0; r < 4; ++r) {
            float acc = __fmul_rn(p.x, m[r * 4 + 0]);
            acc = __fadd_rn(acc, __fmul_rn(p.y, m[r * 4 + 1]));
            acc = __fadd_rn(acc, __fmul_rn(p.z, m[r * 4 + 2]));
            acc = __fadd_rn(acc, __fmul_rn(p.w, m[r * 4 + 3]));
            c[r] = acc;
        }
        const float nx = __fdiv_rn(c[0], c[3]), ny = __fdiv_rn(c[1], c[3]);
        const float x = __fmul_rn(__fdiv_rn(__fadd_rn(nx, 1.f), 2.f), (float)a.H);
        const float y = __fmul_rn(__fdiv_rn(__fadd_rn(ny, 1.f), 2.f), (float)a.W);
        xs[t] = x;
        ys[t] = y;
        zs[t] = __fdiv_rn(c[2], c[3]);
        ok[t] = c[3] > 0.f && fabsf(x) < COORD_LIMIT && fabsf(y) < COORD_LIMIT; // false for NaN too
        reinterpret_cast<float2 *>(a.kp)[(size_t)v * K + t] = make_float2(x, y);
    }
    __syncthreads();
    if (t == 0) { // the reference's visibility and occlusion rules; `ok` becomes "drawable"
        bool m[OP_K];
        for (int i = 0; i < K; ++i) m[i] = true;
        if (!hsd)
            for (int i = 0; i < K; ++i) m[i] = xs[i] >= 0.f && xs[i] < (float)a.H && ys[i] >= 0.f && ys[i] < (float)a.W;
        if (a.occlusion[v]) {
            // HumanSD: 0 nose, 1 / 2 left / right eye, 3 / 4 left / right ear; OpenPose: 0 nose, 14 / 15 right / left
            // eye, 16 / 17 right / left ear.  Both restate the same rule on their own indices.
            const int rear = hsd ? 4 : 16, lear = hsd ? 3 : 17, reye = hsd ? 2 : 14, leye = hsd ? 1 : 15;
            const float z0 = zs[0];
            if (z0 > zs[lear] && z0 < zs[rear]) {
                m[rear] = false;
                if (xs[reye] > xs[leye]) m[reye] = false;
            } else if (z0 < zs[lear] && z0 > zs[rear]) {
                m[lear] = false;
                if (xs[leye] < xs[reye]) m[leye] = false;
            } else if (z0 > zs[lear] && z0 > zs[rear]) {
                m[0] = m[leye] = m[reye] = false;
            }
        }
        // HumanSD: the reference draws a skeleton only when its keypoint array (x, y, and the 0 / 1 confidence after
        // occlusion) sums to > 0, so a NaN coordinate leaves the view blank; the sum is taken in double.
        bool any = true;
        if (hsd) {
            double total = 0.0;
            for (int i = 0; i < K; ++i) total = __dadd_rn(__dadd_rn(__dadd_rn(total, (double)xs[i]), (double)ys[i]), m[i] ? 1.0 : 0.0);
            any = total > 0.0;
        }
        for (int i = 0; i < K; ++i) ok[i] = any && ok[i] && m[i];
    }
    __syncthreads();
    const int S = hsd ? HSD_L : OP_K + OP_L;
    if (t >= S) return;
    const ShapeRows h{a.hulls + ((size_t)v * S + t) * a.H * SLOTS, a.W, a.H};
    for (int i = 0; i < a.H * SLOTS; ++i) h.rows[i] = make_int2(1, 0); // empty
    if (hsd) {
        const int ia = a.limbs[t][0], ib = a.limbs[t][1];
        if (!ok[ia] || !ok[ib]) return;
        const i64 xa = __float2ll_rz(xs[ia]), ya = __float2ll_rz(ys[ia]), xb = __float2ll_rz(xs[ib]), yb = __float2ll_rz(ys[ib]);
        const int T = 10 * a.H / 512;
        thick_line(h, xa, ya, xb, yb, T);
        circle_filled(h, xa, ya, T / 2);
        circle_filled(h, xb, yb, T / 2);
    } else if (t < OP_K) {
        if (ok[t]) circle_filled(h, __float2int_rz(xs[t]), __float2int_rz(ys[t]), 4);
    } else {
        const int l = t - OP_K, ia = a.limbs[l][0], ib = a.limbs[l][1];
        if (!ok[ia] || !ok[ib]) return;
        int cx, cy, hl, ang;
        limb_geometry(xs[ia], ys[ia], xs[ib], ys[ib], cx, cy, hl, ang);
        int2 *poly = a.polys + ((size_t)v * OP_L + l) * MAX_POLY;
        const int n = ellipse2poly(sin_t, cx, cy, hl, 4, ang, poly);
        fill_convex(h, n, 0, [&](int i) { const int2 q = poly[i]; return make_longlong2(q.x, q.y); });
    }
}

__device__ __forceinline__ bool covers(const int2 *slots, int x)
{
    for (int i = 0; i < SLOTS; ++i) {
        const int2 r = slots[i];
        if (r.x > r.y) return false;
        if (x >= r.x && x <= r.y) return true;
    }
    return false;
}

__global__ void __launch_bounds__(128) pose_draw_kernel(PoseArgs a)
{
    const int row = blockIdx.x; // v * H + y
    const int x0 = (blockIdx.y * blockDim.x + threadIdx.x) * 4;
    if (x0 >= a.W) return;
    const int v = row / a.H, y = row - v * a.H;
    const bool hsd = a.style == 0;
    const int S = hsd ? HSD_L : OP_K + OP_L;
    const int2 *hr = a.hulls + ((size_t)v * S * a.H + y) * SLOTS;
    float out[12];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int x = x0 + j;
        int c0 = 0, c1 = 0, c2 = 0;
        const int n_over = hsd ? HSD_L : OP_K; // shapes drawn over what is below; the OpenPose limbs after them blend
        for (int s = 0; s < n_over; ++s) {
            if (covers(hr + (size_t)s * a.H * SLOTS, x)) { c0 = a.colors[s][0]; c1 = a.colors[s][1]; c2 = a.colors[s][2]; }
        }
        for (int s = n_over; s < S; ++s) {
            if (covers(hr + (size_t)s * a.H * SLOTS, x)) { // addWeighted(canvas, 0.4, filled, 0.6, 0) on u8
                c0 = __float2int_rn(__fadd_rn(__fmul_rn((float)c0, 0.4f), __fmul_rn((float)a.colors[s][0], 0.6f)));
                c1 = __float2int_rn(__fadd_rn(__fmul_rn((float)c1, 0.4f), __fmul_rn((float)a.colors[s][1], 0.6f)));
                c2 = __float2int_rn(__fadd_rn(__fmul_rn((float)c2, 0.4f), __fmul_rn((float)a.colors[s][2], 0.6f)));
            }
        }
        out[j * 3 + 0] = __fdiv_rn((float)c0, 255.f);
        out[j * 3 + 1] = __fdiv_rn((float)c1, 255.f);
        out[j * 3 + 2] = __fdiv_rn((float)c2, 255.f);
    }
    float *dst = a.out + ((size_t)row * a.W + x0) * 3;
    if ((a.W & 3) == 0) {
        float4 *d4 = reinterpret_cast<float4 *>(dst);
        d4[0] = make_float4(out[0], out[1], out[2], out[3]);
        d4[1] = make_float4(out[4], out[5], out[6], out[7]);
        d4[2] = make_float4(out[8], out[9], out[10], out[11]);
    } else {
        const int n = min(4, a.W - x0) * 3;
#pragma unroll
        for (int i = 0; i < 12; ++i)
            if (i < n) dst[i] = out[i];
    }
}

} // namespace

int pose_shapes(int style) { return style == 0 ? HSD_L : OP_K + OP_L; }
int pose_limbs(int style) { return style == 0 ? HSD_L : OP_L; }
int pose_keypoints(int style) { return style == 0 ? HSD_K : OP_K; }

size_t pose_scratch_bytes(int style, int V, int H)
{
    const size_t S = pose_shapes(style);
    const size_t hull = (size_t)V * S * H * SLOTS * sizeof(int2);
    const size_t poly = style == 0 ? 0 : (size_t)V * OP_L * MAX_POLY * sizeof(int2);
    return ((hull + 255) & ~(size_t)255) + poly;
}

void pose_layout(PoseArgs &a, char *scratch)
{
    const size_t S = pose_shapes(a.style);
    const size_t hull = (size_t)a.V * S * a.H * SLOTS * sizeof(int2);
    a.hulls = reinterpret_cast<int2 *>(scratch);
    a.polys = a.style == 0 ? nullptr : reinterpret_cast<int2 *>(scratch + ((hull + 255) & ~(size_t)255));
}

void launch_pose_setup(const PoseArgs &a, cudaStream_t st) { pose_setup_kernel<<<a.V, 64, 0, st>>>(a); }

void launch_pose_draw(const PoseArgs &a, cudaStream_t st)
{
    const int threads = 128, per_block = threads * 4;
    pose_draw_kernel<<<dim3((unsigned)a.V * a.H, (a.W + per_block - 1) / per_block), threads, 0, st>>>(a);
}
