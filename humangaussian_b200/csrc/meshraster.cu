// meshraster.cu -- mesh rendering (humangaussian_b200/meshrender.py): triangle rasterisation of a batch of clip-space
// vertex sets into nvdiffrast's visibility buffer, attribute interpolation through it, and the reference's vertex
// normals and normal image (DESIGN.md section 2 is the specification, tests/meshraster_reference.py its restatement).
//
// Rasterisation, count / emit:
//   1. setup (one thread per (view, triangle)): the edge coefficients A, B, C of 2D-homogeneous rasterisation and D,
//      in the specification's float32 order, kept with the sign of D (not folded into A, B, C: a cancelling sum rounds
//      to +0 whatever the signs of its terms, so negated coefficients would flip the sign of a zero u, v or z/w); the
//      triangle's pixel rectangle, part of the specification
//      (the projected vertices' pixel bounding box widened by one pixel, in pinned float32, where every W > 0; the
//      whole image otherwise): no pixel outside it is covered, which also bounds where a point-sized triangle, whose
//      edge functions are rounding noise, can draw; one integer atomicAdd per tile the rectangle touches;
//   2. an exclusive scan of the (view, tile) counts; its exact total is the caller's one host wait;
//   3. emit: scatter every (view, triangle) into its tiles' lists (a slot per entry from a per-tile cursor: the order
//      inside a tile is free, because the result is a minimum over a total order), then one CTA per (view, tile) and
//      one thread per pixel: batches of 256 entries (record and rectangle) are staged in shared memory, and every pixel
//      inside an entry's rectangle tests it and keeps the smallest key
//      (order-preserving bits of z/w) << 32 | triangle with its u, v and z/w in registers.
//   No atomics touch the output: every run writes the same bytes.
// Interpolation, the vertex normals (a per-vertex incidence list in (corner, face) order, built once per topology by
// the binning stage's stable radix sort, then one thread per (frame, vertex)) and the normal image are one thread per
// output element.  Every float operation that reaches an output is an explicit _rn intrinsic (no FMA contraction).
#include "common.cuh"
#include "kernels.h"

namespace {

constexpr int MR_TILE = 16;
constexpr int MR_THREADS = 256;                  // raster CTA: one thread per pixel of a 16 x 16 tile
constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 8; // scan block: 2048 counts
constexpr int SCAN_BLOCK = SCAN_THREADS * SCAN_ITEMS;

struct __align__(16) TriRec { float4 a, b, c, d; }; // A0 A1 A2 B0 | B1 B2 C0 C1 | C2 Z0 Z1 Z2 | W0 W1 W2 sign(D)
static_assert(sizeof(TriRec) == 64, "TriRec must be 64 bytes");

__device__ __forceinline__ bool finite4(float4 p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && isfinite(p.w); }

// pixel centre in NDC: (2i + 1) / n - 1
__device__ __forceinline__ float pix_ndc(int i, int n) { return fsub(fdiv((float)(2 * i + 1), (float)n), 1.0f); }

// the rectangle's pixel range on one axis: [floor(pa) - 1, ceil(pb) + 1] clamped to [0, n - 1], pa and pb the pixel
// coordinates ((s + 1) * (n / 2)) - 1/2 of the NDC extremes [a, b]; false when it is empty
__device__ __forceinline__ bool pixel_span(float a, float b, int n, int &lo, int &hi)
{
    const float h = fmul(0.5f, (float)n);
    const float pa = fsub(fmul(fadd(a, 1.0f), h), 0.5f), pb = fsub(fmul(fadd(b, 1.0f), h), 0.5f);
    const float l = fmaxf(fsub(floorf(pa), 1.0f), 0.0f), r = fminf(fadd(ceilf(pb), 1.0f), (float)(n - 1));
    if (!(l <= r)) return false;
    lo = (int)l;
    hi = (int)r;
    return true;
}

__global__ void __launch_bounds__(256) mr_setup_kernel(int V, int Nv, int Nf, int W, int H, int TX, int TY,
                                                       const float4 *__restrict__ pos, const int *__restrict__ tri,
                                                       TriRec *__restrict__ recs, ushort4 *__restrict__ rects,
                                                       uint32_t *__restrict__ tile_count)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)V * Nf) return;
    const int v = (int)(i / Nf), t = (int)(i - (int64_t)v * Nf);
    ushort4 rect = make_ushort4(1, 0, 0, 0); // pixels [x0, x1] x [y0, y1]; empty: x0 > x1
    const int i0 = tri[3 * t], i1 = tri[3 * t + 1], i2 = tri[3 * t + 2];
    if (i0 >= 0 && i0 < Nv && i1 >= 0 && i1 < Nv && i2 >= 0 && i2 < Nv) {
        const float4 *pv = pos + (size_t)v * Nv;
        const float4 p[3] = {pv[i0], pv[i1], pv[i2]};
        if (finite4(p[0]) && finite4(p[1]) && finite4(p[2]) && !(p[0].w <= 0.0f && p[1].w <= 0.0f && p[2].w <= 0.0f)) {
            float A[3], B[3], C[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float4 pj = p[(k + 1) % 3], pk = p[(k + 2) % 3];
                A[k] = fsub(fmul(pj.y, pk.w), fmul(pj.w, pk.y));
                B[k] = fsub(fmul(pj.w, pk.x), fmul(pj.x, pk.w));
                C[k] = fsub(fmul(pj.x, pk.y), fmul(pj.y, pk.x));
            }
            const float D = fadd(fadd(fmul(p[0].x, A[0]), fmul(p[0].y, B[0])), fmul(p[0].w, C[0]));
            bool ok = D != 0.0f && isfinite(D);
#pragma unroll
            for (int k = 0; k < 3; ++k) ok = ok && isfinite(A[k]) && isfinite(B[k]) && isfinite(C[k]);
            int x0 = 0, x1 = W - 1, y0 = 0, y1 = H - 1;
            if (ok && p[0].w > 0.0f && p[1].w > 0.0f && p[2].w > 0.0f) {
                // every W > 0: the covered pixels lie in the projected triangle; one pixel of margin keeps every pixel
                // centre inside it whatever the rounding of the projection
                float ax = INFINITY, bx = -INFINITY, ay = INFINITY, by = -INFINITY;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const float sx = fdiv(p[k].x, p[k].w), sy = fdiv(p[k].y, p[k].w);
                    ax = fminf(ax, sx); bx = fmaxf(bx, sx); ay = fminf(ay, sy); by = fmaxf(by, sy);
                }
                ok = pixel_span(ax, bx, W, x0, x1) && pixel_span(ay, by, H, y0, y1);
            }
            if (ok) {
                TriRec r;
                r.a = make_float4(A[0], A[1], A[2], B[0]);
                r.b = make_float4(B[1], B[2], C[0], C[1]);
                r.c = make_float4(C[2], p[0].z, p[1].z, p[2].z);
                r.d = make_float4(p[0].w, p[1].w, p[2].w, D < 0.0f ? -1.0f : 1.0f);
                recs[i] = r;
                rect = make_ushort4(x0, y0, x1, y1);
            }
        }
    }
    rects[i] = rect;
    if (rect.x > rect.z) return;
    uint32_t *cnt = tile_count + (size_t)v * TX * TY;
    for (int ty = rect.y / MR_TILE; ty <= rect.w / MR_TILE; ++ty)
        for (int tx = rect.x / MR_TILE; tx <= rect.z / MR_TILE; ++tx) atomicAdd(cnt + ty * TX + tx, 1u);
}

// ---- exclusive scan of n u32 counts into u64 starts: block sums, one CTA over the block sums, block-local scan ----------
__device__ __forceinline__ uint64_t block_exclusive_scan(uint64_t x, uint64_t *total)
{
    __shared__ uint64_t warp_sum[SCAN_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint64_t incl = x;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t y = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += y;
    }
    if (lane == 31) warp_sum[w] = incl;
    __syncthreads();
    uint64_t before = 0, all = 0;
    for (int k = 0; k < SCAN_THREADS / 32; ++k) {
        if (k < w) before += warp_sum[k];
        all += warp_sum[k];
    }
    __syncthreads();
    *total = all;
    return before + incl - x;
}

__global__ void __launch_bounds__(SCAN_THREADS) mr_scan_reduce_kernel(const uint32_t *__restrict__ x, int64_t n,
                                                                      uint64_t *__restrict__ block_sums)
{
    const int64_t base = (int64_t)blockIdx.x * SCAN_BLOCK + (int64_t)threadIdx.x * SCAN_ITEMS;
    uint64_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k)
        if (base + k < n) s += x[base + k];
    uint64_t total;
    block_exclusive_scan(s, &total);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(SCAN_THREADS) mr_scan_blocks_kernel(uint64_t *__restrict__ block_sums, int64_t nb,
                                                                      uint64_t *__restrict__ total_out)
{
    uint64_t carry = 0;
    for (int64_t c = 0; c < nb; c += SCAN_THREADS) {
        const int64_t k = c + threadIdx.x;
        const uint64_t x = k < nb ? block_sums[k] : 0;
        uint64_t total;
        const uint64_t ex = block_exclusive_scan(x, &total);
        if (k < nb) block_sums[k] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) *total_out = carry;
}

__global__ void __launch_bounds__(SCAN_THREADS) mr_scan_down_kernel(const uint32_t *__restrict__ x, int64_t n,
                                                                    const uint64_t *__restrict__ block_off,
                                                                    uint64_t *__restrict__ start)
{
    const int64_t base = (int64_t)blockIdx.x * SCAN_BLOCK + (int64_t)threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS];
    uint64_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        v[k] = base + k < n ? x[base + k] : 0u;
        s += v[k];
    }
    uint64_t total;
    uint64_t run = block_off[blockIdx.x] + block_exclusive_scan(s, &total);
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        if (base + k < n) start[base + k] = run;
        run += v[k];
    }
}

__global__ void __launch_bounds__(256) mr_scatter_kernel(int V, int Nf, int TX, int TY, const ushort4 *__restrict__ rects,
                                                         const uint64_t *__restrict__ start, uint32_t *__restrict__ cursor,
                                                         int *__restrict__ pairs, uint64_t cap)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)V * Nf) return;
    const int v = (int)(i / Nf), t = (int)(i - (int64_t)v * Nf);
    const ushort4 rect = rects[i];
    if (rect.x > rect.z) return;
    const size_t vt0 = (size_t)v * TX * TY;
    for (int ty = rect.y / MR_TILE; ty <= rect.w / MR_TILE; ++ty)
        for (int tx = rect.x / MR_TILE; tx <= rect.z / MR_TILE; ++tx) {
            const size_t vt = vt0 + ty * TX + tx;
            const uint64_t slot = start[vt] + atomicAdd(cursor + vt, 1u);
            if (slot < cap) pairs[slot] = t;
        }
}

__device__ __forceinline__ uint32_t ordered_bits(float f)
{
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__global__ void __launch_bounds__(MR_THREADS) mr_raster_kernel(int Nf, int W, int H, int TX, int TY, const TriRec *__restrict__ recs,
                                                               const ushort4 *__restrict__ rects, const uint64_t *__restrict__ start, const uint32_t *__restrict__ count,
                                                               const int *__restrict__ pairs, uint64_t cap, float4 *__restrict__ rast)
{
    __shared__ float4 s_rec[MR_THREADS][4];
    __shared__ int s_t[MR_THREADS];
    __shared__ ushort4 s_rect[MR_THREADS];
    const int vt = blockIdx.x, v = vt / (TX * TY), tile = vt - v * TX * TY;
    const int x = (tile % TX) * MR_TILE + (threadIdx.x & (MR_TILE - 1)), y = (tile / TX) * MR_TILE + threadIdx.x / MR_TILE;
    const float px = pix_ndc(x, W), py = pix_ndc(y, H);
    const uint64_t beg = start[vt], end = min(beg + count[vt], cap);
    const TriRec *vrecs = recs + (size_t)v * Nf;
    const ushort4 *vrects = rects + (size_t)v * Nf;
    uint64_t best = ~0ull;
    float bu = 0.0f, bv = 0.0f, bz = 0.0f;
    for (uint64_t c = beg; c < end; c += MR_THREADS) {
        const int n = (int)min((uint64_t)MR_THREADS, end - c);
        __syncthreads();
        if (threadIdx.x < n) {
            const int t = pairs[c + threadIdx.x];
            const bool ok = (unsigned)t < (unsigned)Nf;
            s_t[threadIdx.x] = t;
            s_rect[threadIdx.x] = ok ? vrects[t] : make_ushort4(1, 0, 0, 0);
            if (ok) {
                const TriRec r = vrecs[t];
                s_rec[threadIdx.x][0] = r.a; s_rec[threadIdx.x][1] = r.b; s_rec[threadIdx.x][2] = r.c; s_rec[threadIdx.x][3] = r.d;
            }
        }
        __syncthreads();
        for (int k = 0; k < n; ++k) {
            const ushort4 rc = s_rect[k];
            if (x < rc.x || x > rc.z || y < rc.y || y > rc.w) continue; // outside the triangle's pixel rectangle
            const float4 a = s_rec[k][0], b = s_rec[k][1];
            const float e0 = fadd(fadd(fmul(a.x, px), fmul(a.w, py)), b.z);
            const float e1 = fadd(fadd(fmul(a.y, px), fmul(b.x, py)), b.w);
            const float4 cc = s_rec[k][2];
            const float e2 = fadd(fadd(fmul(a.z, px), fmul(b.y, py)), cc.x);
            const float4 d = s_rec[k][3];
            // every e_i has the sign of D or is zero
            if (d.w > 0.0f ? !(e0 >= 0.0f && e1 >= 0.0f && e2 >= 0.0f) : !(e0 <= 0.0f && e1 <= 0.0f && e2 <= 0.0f)) continue;
            const float S = fadd(fadd(e0, e1), e2);
            if (S == 0.0f) continue;
            const float u = fdiv(e0, S), w = fdiv(e1, S), l2 = fdiv(e2, S);
            const float Wp = fadd(fadd(fmul(u, d.x), fmul(w, d.y)), fmul(l2, d.z));
            if (!(Wp > 0.0f)) continue;
            const float zw = fdiv(fadd(fadd(fmul(u, cc.y), fmul(w, cc.z)), fmul(l2, cc.w)), Wp);
            if (!(zw >= -1.0f && zw <= 1.0f)) continue;
            const uint64_t key = ((uint64_t)ordered_bits(zw) << 32) | (uint32_t)s_t[k];
            if (key < best) { best = key; bu = u; bv = w; bz = zw; }
        }
    }
    if (x < W && y < H)
        rast[((size_t)v * H + y) * W + x] = best == ~0ull ? make_float4(0.0f, 0.0f, 0.0f, 0.0f)
                                                         : make_float4(bu, bv, bz, (float)((uint32_t)best + 1u));
}

// triangle of a rasterised pixel, or -1 (rast.w not in 1..Nf, or an index outside [0, Nv))
__device__ __forceinline__ int pixel_triangle(float w, int Nf, int Nv, const int *__restrict__ tri, int &i0, int &i1, int &i2)
{
    if (!(w > 0.0f && w <= (float)Nf)) return -1;
    const int t = (int)w - 1;
    i0 = tri[3 * t]; i1 = tri[3 * t + 1]; i2 = tri[3 * t + 2];
    if (i0 < 0 || i0 >= Nv || i1 < 0 || i1 >= Nv || i2 < 0 || i2 >= Nv) return -1;
    return t;
}

// a0 u + a1 v + a2 ((1 - u) - v), left to right
__device__ __forceinline__ float bary(float a0, float a1, float a2, float u, float v, float b2)
{
    return fadd(fadd(fmul(a0, u), fmul(a1, v)), fmul(a2, b2));
}

__global__ void __launch_bounds__(256) mr_interp_kernel(int V, int HW, int Nv, int Nf, int C, const float *__restrict__ attr,
                                                        int per_view, const float4 *__restrict__ rast, const int *__restrict__ tri,
                                                        float *__restrict__ out)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)V * HW) return;
    const float4 r = rast[i];
    float *o = out + i * C;
    int i0, i1, i2;
    if (pixel_triangle(r.w, Nf, Nv, tri, i0, i1, i2) < 0) {
        for (int c = 0; c < C; ++c) o[c] = 0.0f;
        return;
    }
    const float *a = attr + (per_view ? (size_t)(i / HW) * Nv * C : 0);
    const float *a0 = a + (size_t)i0 * C, *a1 = a + (size_t)i1 * C, *a2 = a + (size_t)i2 * C;
    const float b2 = fsub(fsub(1.0f, r.x), r.y);
    for (int c = 0; c < C; ++c) o[c] = bary(a0[c], a1[c], a2[c], r.x, r.y, b2);
}

// safe_normalize: x / sqrt(max((x0 x0 + x1 x1) + x2 x2, 1e-20)), three divisions (a NaN dot stays NaN, as in torch.clamp)
__device__ __forceinline__ void safe_normalize(float &x, float &y, float &z)
{
    const float d = fadd(fadd(fmul(x, x), fmul(y, y)), fmul(z, z));
    const float l = fsqrt(d < 1e-20f ? 1e-20f : d);
    x = fdiv(x, l); y = fdiv(y, l); z = fdiv(z, l);
}

__global__ void __launch_bounds__(256) mr_normal_image_kernel(int V, int HW, int Nv, int Nf, const float *__restrict__ vn,
                                                              int per_view, const float4 *__restrict__ rast,
                                                              const int *__restrict__ tri, float *__restrict__ out)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)V * HW) return;
    const float4 r = rast[i];
    float *o = out + i * 3;
    int i0, i1, i2;
    if (pixel_triangle(r.w, Nf, Nv, tri, i0, i1, i2) < 0) {
        o[0] = o[1] = o[2] = 1.0f; // background
        return;
    }
    const float *a = vn + (per_view ? (size_t)(i / HW) * Nv * 3 : 0);
    const float *a0 = a + (size_t)i0 * 3, *a1 = a + (size_t)i1 * 3, *a2 = a + (size_t)i2 * 3;
    const float b2 = fsub(fsub(1.0f, r.x), r.y);
    float n[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) n[c] = bary(a0[c], a1[c], a2[c], r.x, r.y, b2);
    safe_normalize(n[0], n[1], n[2]);
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = fdiv(fadd(n[c], 1.0f), 2.0f);
}

// incidence: entry e = corner * Nf + face keyed by its vertex (Nv for a face with an index outside [0, Nv)); the stable
// sort by vertex then leaves each vertex's faces in (corner, face) order
__global__ void __launch_bounds__(256) mr_inc_keys_kernel(int Nv, int Nf, const int *__restrict__ faces, uint32_t *__restrict__ keys,
                                                          uint32_t *__restrict__ vals)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= 3 * (int64_t)Nf) return;
    const int corner = (int)(e / Nf), f = (int)(e - (int64_t)corner * Nf);
    const int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
    const bool ok = i0 >= 0 && i0 < Nv && i1 >= 0 && i1 < Nv && i2 >= 0 && i2 < Nv;
    keys[e] = ok ? (uint32_t)faces[3 * f + corner] : (uint32_t)Nv;
    vals[e] = (uint32_t)f;
}

// list[i] = sorted face for i < n; start[k] = first sorted position with key >= k (a lower-bound search), for k in
// [0, Nv].  Threads run over max(n, Nv + 1).
__global__ void __launch_bounds__(256) mr_inc_finish_kernel(int64_t n, int Nv, const uint32_t *__restrict__ keys,
                                                            const uint32_t *__restrict__ vals, uint32_t *__restrict__ start,
                                                            uint32_t *__restrict__ list)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) list[i] = vals[i];
    if (i > Nv) return;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if ((int64_t)keys[mid] < i) lo = mid + 1; else hi = mid;
    }
    start[i] = (uint32_t)lo;
}

__global__ void __launch_bounds__(256) mr_vertex_normals_kernel(int F, int Nv, const float *__restrict__ verts, const int *__restrict__ faces,
                                                                const uint32_t *__restrict__ start, const uint32_t *__restrict__ list,
                                                                float *__restrict__ out)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)F * Nv) return;
    const int f = (int)(i / Nv), vi = (int)(i - (int64_t)f * Nv);
    const float *P = verts + (size_t)f * Nv * 3;
    float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f;
    for (uint32_t e = start[vi], e1 = start[vi + 1]; e < e1; ++e) {
        const int face = (int)list[e];
        const float *p0 = P + 3 * (size_t)faces[3 * face], *p1 = P + 3 * (size_t)faces[3 * face + 1], *p2 = P + 3 * (size_t)faces[3 * face + 2];
        const float a0 = fsub(p1[0], p0[0]), a1 = fsub(p1[1], p0[1]), a2 = fsub(p1[2], p0[2]);
        const float b0 = fsub(p2[0], p0[0]), b1 = fsub(p2[1], p0[1]), b2 = fsub(p2[2], p0[2]);
        s0 = fadd(s0, fsub(fmul(a1, b2), fmul(a2, b1))); // torch.cross's component formula
        s1 = fadd(s1, fsub(fmul(a2, b0), fmul(a0, b2)));
        s2 = fadd(s2, fsub(fmul(a0, b1), fmul(a1, b0)));
    }
    const float d = fadd(fadd(fmul(s0, s0), fmul(s1, s1)), fmul(s2, s2));
    if (!(d > 1e-20f)) { s0 = 0.0f; s1 = 0.0f; s2 = 1.0f; } // degenerate (or NaN) sums: (0, 0, 1)
    safe_normalize(s0, s1, s2);
    out[3 * i] = s0; out[3 * i + 1] = s1; out[3 * i + 2] = s2;
}

int bits_for_keys(uint64_t n)
{
    int b = 0;
    while (((uint64_t)1 << b) < n) b++;
    return b > 0 ? b : 1;
}

inline unsigned blocks_for(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

struct RasterLayout {
    size_t recs, rects, count, start, cursor, block_sums, total;
    RasterLayout(int V, int Nf, int ntiles)
    {
        const size_t n = (size_t)V * Nf, nt = (size_t)V * ntiles, nb = (nt + SCAN_BLOCK - 1) / SCAN_BLOCK;
        size_t o = 0;
        recs = o; o += gs_align(n * sizeof(TriRec));
        rects = o; o += gs_align(n * sizeof(ushort4));
        count = o; o += gs_align(nt * 4);
        start = o; o += gs_align(nt * 8);
        cursor = o; o += gs_align(nt * 4);
        block_sums = o; o += gs_align(nb * 8);
        total = o;
    }
};

struct IncidenceLayout {
    size_t start, list, ka, kb, va, vb, sort, total;
    IncidenceLayout(int Nv, int Nf)
    {
        const size_t n = 3 * (size_t)Nf;
        size_t o = 0;
        start = o; o += gs_align(((size_t)Nv + 1) * 4);
        list = o; o += gs_align(n * 4);
        ka = o; o += gs_align(n * 4);
        kb = o; o += gs_align(n * 4);
        va = o; o += gs_align(n * 4);
        vb = o; o += gs_align(n * 4);
        sort = o; o += test_sort32_scratch_bytes((int64_t)(n > 0 ? n : 1));
        total = o;
    }
};

} // namespace

size_t mesh_raster_scratch_bytes(int V, int Nf, int H, int W)
{
    return RasterLayout(V, Nf, ((W + MR_TILE - 1) / MR_TILE) * ((H + MR_TILE - 1) / MR_TILE)).total;
}

int launch_mesh_raster_count(int V, int Nv, int Nf, int H, int W, const float *pos, const int *tri, char *scratch, uint64_t *count,
                             cudaStream_t st, int *n_launches)
{
    const int TX = (W + MR_TILE - 1) / MR_TILE, TY = (H + MR_TILE - 1) / MR_TILE;
    const RasterLayout L(V, Nf, TX * TY);
    const int64_t nt = (int64_t)V * TX * TY, nb = (nt + SCAN_BLOCK - 1) / SCAN_BLOCK, n = (int64_t)V * Nf;
    uint32_t *cnt = (uint32_t *)(scratch + L.count);
    uint64_t *sums = (uint64_t *)(scratch + L.block_sums);
    if (cudaMemsetAsync(cnt, 0, (size_t)nt * 4, st) != cudaSuccess) return -1;
    int nl = 0;
    if (n > 0) {
        mr_setup_kernel<<<blocks_for(n, 256), 256, 0, st>>>(V, Nv, Nf, W, H, TX, TY, (const float4 *)pos, tri, (TriRec *)(scratch + L.recs),
                                                              (ushort4 *)(scratch + L.rects), cnt);
        nl++;
    }
    mr_scan_reduce_kernel<<<(unsigned)nb, SCAN_THREADS, 0, st>>>(cnt, nt, sums);
    mr_scan_blocks_kernel<<<1, SCAN_THREADS, 0, st>>>(sums, nb, count);
    mr_scan_down_kernel<<<(unsigned)nb, SCAN_THREADS, 0, st>>>(cnt, nt, sums, (uint64_t *)(scratch + L.start));
    *n_launches = nl + 3;
    return 0;
}

int launch_mesh_raster_emit(int V, int Nf, int H, int W, char *scratch, int *pairs, uint64_t cap, float *rast, cudaStream_t st,
                            int *n_launches)
{
    const int TX = (W + MR_TILE - 1) / MR_TILE, TY = (H + MR_TILE - 1) / MR_TILE;
    const RasterLayout L(V, Nf, TX * TY);
    const int64_t nt = (int64_t)V * TX * TY, n = (int64_t)V * Nf;
    uint32_t *cursor = (uint32_t *)(scratch + L.cursor);
    if (cudaMemsetAsync(cursor, 0, (size_t)nt * 4, st) != cudaSuccess) return -1;
    int nl = 0;
    if (n > 0 && cap > 0) {
        mr_scatter_kernel<<<blocks_for(n, 256), 256, 0, st>>>(V, Nf, TX, TY, (const ushort4 *)(scratch + L.rects),
                                                                (const uint64_t *)(scratch + L.start), cursor, pairs, cap);
        nl++;
    }
    mr_raster_kernel<<<(unsigned)nt, MR_THREADS, 0, st>>>(Nf, W, H, TX, TY, (const TriRec *)(scratch + L.recs),
                                                          (const ushort4 *)(scratch + L.rects), (const uint64_t *)(scratch + L.start), (const uint32_t *)(scratch + L.count),
                                                          pairs, cap, (float4 *)rast);
    *n_launches = nl + 1;
    return 0;
}

void launch_mesh_interpolate(int V, int H, int W, int Nv, int Nf, int C, const float *attr, int per_view, const float *rast, const int *tri,
                             float *out, cudaStream_t st)
{
    const int64_t n = (int64_t)V * H * W;
    mr_interp_kernel<<<blocks_for(n, 256), 256, 0, st>>>(V, H * W, Nv, Nf, C, attr, per_view, (const float4 *)rast, tri, out);
}

void launch_mesh_normal_image(int V, int H, int W, int Nv, int Nf, const float *vn, int per_view, const float *rast, const int *tri,
                              float *out, cudaStream_t st)
{
    const int64_t n = (int64_t)V * H * W;
    mr_normal_image_kernel<<<blocks_for(n, 256), 256, 0, st>>>(V, H * W, Nv, Nf, vn, per_view, (const float4 *)rast, tri, out);
}

size_t mesh_incidence_bytes(int Nv, int Nf) { return IncidenceLayout(Nv, Nf).total; }

void mesh_incidence_lists(int Nv, int Nf, const char *buf, const uint32_t **start, const uint32_t **list)
{
    const IncidenceLayout L(Nv, Nf);
    *start = (const uint32_t *)(buf + L.start);
    *list = (const uint32_t *)(buf + L.list);
}

int launch_mesh_incidence(int Nv, int Nf, const int *faces, char *buf, size_t bytes, cudaStream_t st, int *n_launches)
{
    const IncidenceLayout L(Nv, Nf);
    uint32_t *start = (uint32_t *)(buf + L.start);
    if (Nf == 0) {
        *n_launches = 0;
        return cudaMemsetAsync(start, 0, ((size_t)Nv + 1) * 4, st) != cudaSuccess ? -1 : 0;
    }
    const int64_t n = 3 * (int64_t)Nf;
    uint32_t *ka = (uint32_t *)(buf + L.ka), *kb = (uint32_t *)(buf + L.kb), *va = (uint32_t *)(buf + L.va), *vb = (uint32_t *)(buf + L.vb);
    mr_inc_keys_kernel<<<blocks_for(n, 256), 256, 0, st>>>(Nv, Nf, faces, ka, va);
    const int bits = bits_for_keys((uint64_t)Nv + 1);
    int in_b = 0;
    if (launch_test_sort32(ka, kb, va, vb, n, bits, buf + L.sort, bytes - L.sort, &in_b, st)) return -2;
    mr_inc_finish_kernel<<<blocks_for(n > (int64_t)Nv + 1 ? n : (int64_t)Nv + 1, 256), 256, 0, st>>>(n, Nv, in_b ? kb : ka, in_b ? vb : va, start,
                                                                 (uint32_t *)(buf + L.list));
    *n_launches = 2 + 3 * ((bits + 8) / 9);
    return 0;
}

void launch_mesh_vertex_normals(int F, int Nv, int Nf, const float *verts, const int *faces, const char *incidence, float *out,
                                cudaStream_t st)
{
    const IncidenceLayout L(Nv, Nf);
    const int64_t n = (int64_t)F * Nv;
    mr_vertex_normals_kernel<<<blocks_for(n, 256), 256, 0, st>>>(F, Nv, verts, faces, (const uint32_t *)(incidence + L.start),
                                                                 (const uint32_t *)(incidence + L.list), out);
}
