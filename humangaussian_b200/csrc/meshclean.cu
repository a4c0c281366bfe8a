// meshclean.cu -- mesh cleanup and decimation (humangaussian_b200/mesh.py clean_mesh / decimate_mesh; DESIGN.md section 2
// is the specification, tests/mesh_clean_reference.py and tests/decimate_reference.py its restatements).
//
// Both work on the per-vertex face lists of meshraster.cu (the binning stage's stable radix sort, (corner, face) order)
// and compact with the binning stage's popcount scan, so every output keeps the input's relative order.
//
// Cleanup: one thread per face drops faces that repeat an index or repeat an earlier face's vertex set (searched in the
// list of the face's smallest vertex); components are labelled by min-label hooking with pointer jumping to the fixed
// point where every face's corners share a label, which is then the smallest vertex index of the component whatever
// the schedule; per-component face counts and bounding boxes (order-preserving float bits) use integer atomics, whose
// result does not depend on their order.  Host waits: one per labelling round, and one for the output counts.
//
// Decimation: parallel rounds of quadric edge collapse.  Per round: the face lists of the current faces, a per-vertex
// lock, one thread per half-edge for the candidate (link condition, position, cost, flip test), the per-vertex minimum
// (cost, edge) over incident candidates and then over the closed one-ring, and the selection of every candidate that
// is the minimum of both its ends' one-rings.  One host wait per round reads the selected count; when it would take
// the mesh below the target, the selected collapses are sorted by (cost, edge) with four stable 32-bit radix passes
// and only the cheapest are applied.  Every float64 operation is an explicit _rn intrinsic, so the numpy restatement
// reproduces the bits.
#include "common.cuh"
#include "kernels.h"

namespace {

inline unsigned blocks_for(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }

__device__ __forceinline__ uint32_t ordered_bits(float f)
{
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float unordered(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }

__device__ __forceinline__ bool in_range(int i, int Nv) { return i >= 0 && i < Nv; }
__device__ __forceinline__ bool repeats(int i0, int i1, int i2) { return i0 == i1 || i1 == i2 || i0 == i2; }

__global__ void __launch_bounds__(256) check_faces_kernel(int Nv, int Nf, const int *__restrict__ faces, uint32_t *__restrict__ bad)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 3 * (int64_t)Nf && !in_range(faces[i], Nv)) *bad = 1u;
}

// ---- cleanup ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void sort3(int &a, int &b, int &c)
{
    if (a > b) { const int t = a; a = b; b = t; }
    if (b > c) { const int t = b; b = c; c = t; }
    if (a > b) { const int t = a; a = b; b = t; }
}

__global__ void __launch_bounds__(256) clean_face_kernel(int Nf, const int *__restrict__ faces, const uint32_t *__restrict__ start,
                                                         const uint32_t *__restrict__ list, uint8_t *__restrict__ keep)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf) return;
    int a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
    if (repeats(a, b, c)) { keep[f] = 0; return; }
    sort3(a, b, c);
    bool dup = false;
    for (uint32_t e = start[a], e1 = start[a + 1]; e < e1 && !dup; ++e) {
        const int g = (int)list[e];
        if (g >= f) continue;
        int x = faces[3 * g], y = faces[3 * g + 1], z = faces[3 * g + 2];
        if (repeats(x, y, z)) continue;
        sort3(x, y, z);
        dup = x == a && y == b && z == c;
    }
    keep[f] = !dup;
}

__global__ void __launch_bounds__(256) iota_kernel(int n, int *__restrict__ x)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] = i;
}

// every corner and its label's target take the face's smallest label; labels only decrease and stay in the component
__global__ void __launch_bounds__(256) hook_kernel(int Nf, const int *__restrict__ faces, const uint8_t *__restrict__ keep, int *lab,
                                                   uint32_t *__restrict__ changed)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf || !keep[f]) return;
    const int c[3] = {faces[3 * f], faces[3 * f + 1], faces[3 * f + 2]};
    const int l[3] = {lab[c[0]], lab[c[1]], lab[c[2]]};
    const int m = min(min(l[0], l[1]), l[2]);
    bool ch = false;
#pragma unroll
    for (int k = 0; k < 3; ++k)
        if (l[k] > m) {
            atomicMin(lab + c[k], m);
            atomicMin(lab + l[k], m);
            ch = true;
        }
    if (ch) *changed = 1u;
}

__global__ void __launch_bounds__(256) jump_kernel(int Nv, int *lab)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Nv) return;
    const int l = lab[v], ll = lab[l];
    if (ll < l) lab[v] = ll;
}

__global__ void __launch_bounds__(256) box_init_kernel(int n, uint32_t *__restrict__ box)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 6 * n) box[i] = (i % 6) < 3 ? 0xffffffffu : 0u;
}

__global__ void __launch_bounds__(256) comp_mark_kernel(int Nf, const int *__restrict__ faces, const uint8_t *__restrict__ keep,
                                                        const int *__restrict__ lab, uint32_t *__restrict__ count, uint8_t *__restrict__ used)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf || !keep[f]) return;
    atomicAdd(count + lab[faces[3 * f]], 1u);
    used[faces[3 * f]] = used[faces[3 * f + 1]] = used[faces[3 * f + 2]] = 1;
}

// box [Nv + 1][6]: ordered bits of (min x, y, z, max x, y, z) per label; row Nv is the whole mesh
__global__ void __launch_bounds__(256) comp_box_kernel(int Nv, const float *__restrict__ verts, const uint8_t *__restrict__ used,
                                                       const int *__restrict__ lab, uint32_t *__restrict__ box)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Nv || !used[v]) return;
    uint32_t *r = box + 6 * (size_t)lab[v], *w = box + 6 * (size_t)Nv;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const uint32_t o = ordered_bits(verts[3 * (size_t)v + k]);
        atomicMin(r + k, o); atomicMax(r + 3 + k, o);
        atomicMin(w + k, o); atomicMax(w + 3 + k, o);
    }
}

__device__ __forceinline__ double box_diag(const uint32_t *b)
{
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double d = ds((double)unordered(b[3 + k]), (double)unordered(b[k]));
        s = k == 0 ? dm(d, d) : da(s, dm(d, d));
    }
    return __dsqrt_rn(s);
}

__global__ void __launch_bounds__(256) comp_keep_kernel(int Nv, int Nf, const int *__restrict__ faces, uint8_t *__restrict__ keep,
                                                        const int *__restrict__ lab, const uint32_t *__restrict__ count,
                                                        const uint32_t *__restrict__ box, int min_faces, double min_diameter,
                                                        uint8_t *__restrict__ vkeep)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf || !keep[f]) return;
    const int r = lab[faces[3 * f]];
    const bool ok = count[r] >= (uint32_t)min_faces && !(box_diag(box + 6 * (size_t)r) < dm(min_diameter, box_diag(box + 6 * (size_t)Nv)));
    keep[f] = ok;
    if (ok) vkeep[faces[3 * f]] = vkeep[faces[3 * f + 1]] = vkeep[faces[3 * f + 2]] = 1;
}

// compaction: surviving vertices and faces in order, corners renumbered; incl are the popcount scans of the keep bytes
__global__ void __launch_bounds__(256) emit_verts_kernel(int Nv, const float *__restrict__ verts, const uint8_t *__restrict__ vkeep,
                                                         const uint32_t *__restrict__ vincl, float *__restrict__ out)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Nv || !vkeep[v]) return;
    const size_t o = vincl[v] - 1;
    out[3 * o] = verts[3 * (size_t)v]; out[3 * o + 1] = verts[3 * (size_t)v + 1]; out[3 * o + 2] = verts[3 * (size_t)v + 2];
}

__global__ void __launch_bounds__(256) emit_faces_kernel(int Nf, const int *__restrict__ faces, const uint8_t *__restrict__ keep,
                                                         const uint32_t *__restrict__ fincl, const uint32_t *__restrict__ vincl,
                                                         int *__restrict__ out)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf || (keep && !keep[f])) return;
    const size_t o = keep ? fincl[f] - 1 : (size_t)f; // without keep: every face, in place
#pragma unroll
    for (int k = 0; k < 3; ++k) out[3 * o + k] = (int)vincl[faces[3 * f + k]] - 1;
}

// ---- decimation ------------------------------------------------------------------------------------------------------
// quadric: row-major upper triangle of the symmetric 4x4: 00 01 02 03 11 12 13 22 23 33
struct Q10 { double q[10]; };

__device__ __forceinline__ void cross_d(const double *p0, const double *p1, const double *p2, double *n)
{
    const double e1[3] = {ds(p1[0], p0[0]), ds(p1[1], p0[1]), ds(p1[2], p0[2])};
    const double e2[3] = {ds(p2[0], p0[0]), ds(p2[1], p0[1]), ds(p2[2], p0[2])};
    n[0] = ds(dm(e1[1], e2[2]), dm(e1[2], e2[1]));
    n[1] = ds(dm(e1[2], e2[0]), dm(e1[0], e2[2]));
    n[2] = ds(dm(e1[0], e2[1]), dm(e1[1], e2[0]));
}

__device__ __forceinline__ void load3(const float *P, int v, double *p)
{
    p[0] = (double)P[3 * (size_t)v]; p[1] = (double)P[3 * (size_t)v + 1]; p[2] = (double)P[3 * (size_t)v + 2];
}

__global__ void __launch_bounds__(256) face_quadric_kernel(int Nf, const float *__restrict__ P, const int *__restrict__ faces,
                                                           double *__restrict__ fq)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= Nf) return;
    double p0[3], p1[3], p2[3], n[3];
    load3(P, faces[3 * f], p0); load3(P, faces[3 * f + 1], p1); load3(P, faces[3 * f + 2], p2);
    cross_d(p0, p1, p2, n);
    const double ln = __dsqrt_rn(da(da(dm(n[0], n[0]), dm(n[1], n[1])), dm(n[2], n[2])));
    double *o = fq + 10 * (size_t)f;
    if (!(ln > 0.0)) {
        for (int k = 0; k < 10; ++k) o[k] = 0.0;
        return;
    }
    const double a[4] = {n[0], n[1], n[2], -da(da(dm(n[0], p0[0]), dm(n[1], p0[1])), dm(n[2], p0[2]))};
    const double h = __ddiv_rn(0.5, ln);
    int k = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = i; j < 4; ++j) o[k++] = dm(dm(a[i], a[j]), h);
}

__global__ void __launch_bounds__(256) vertex_quadric_kernel(int Nv, const double *__restrict__ fq, const uint32_t *__restrict__ start,
                                                             const uint32_t *__restrict__ list, double *__restrict__ Q)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Nv) return;
    double s[10] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (uint32_t e = start[v], e1 = start[v + 1]; e < e1; ++e) {
        const double *q = fq + 10 * (size_t)list[e];
        for (int k = 0; k < 10; ++k) s[k] = da(s[k], q[k]);
    }
    for (int k = 0; k < 10; ++k) Q[10 * (size_t)v + k] = s[k];
}

// the corner of v in face g (the first, for a face that repeats v)
__device__ __forceinline__ int corner_of(const int *faces, int g, int v)
{
    return faces[3 * g] == v ? 0 : faces[3 * g + 1] == v ? 1 : 2;
}

// locked: a face around v repeats an index, a directed edge at v occurs other than once each way, or the faces around
// v are more than one fan (the link map next -> prev has more than one cycle)
__global__ void __launch_bounds__(256) lock_kernel(int Nv, const int *__restrict__ faces, const uint32_t *__restrict__ start,
                                                   const uint32_t *__restrict__ list, uint8_t *__restrict__ locked)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Nv) return;
    const uint32_t e0 = start[v], e1 = start[v + 1];
    bool lk = false;
    for (uint32_t e = e0; e < e1 && !lk; ++e) {
        const int g = (int)list[e];
        if (repeats(faces[3 * g], faces[3 * g + 1], faces[3 * g + 2])) lk = true;
    }
    for (uint32_t e = e0; e < e1 && !lk; ++e) {
        const int g = (int)list[e], c = corner_of(faces, g, v);
        const int w2[2] = {faces[3 * g + (c + 1) % 3], faces[3 * g + (c + 2) % 3]};
        for (int j = 0; j < 2 && !lk; ++j) {
            int out = 0, in = 0;
            for (uint32_t x = e0; x < e1; ++x) {
                const int h = (int)list[x], ch = corner_of(faces, h, v);
                out += faces[3 * h + (ch + 1) % 3] == w2[j];
                in += faces[3 * h + (ch + 2) % 3] == w2[j];
            }
            lk = out != 1 || in != 1;
        }
    }
    if (!lk && e1 > e0) {
        const uint32_t deg = e1 - e0;
        const int g0 = (int)list[e0], c0 = corner_of(faces, g0, v);
        const int first = faces[3 * g0 + (c0 + 1) % 3];
        int w = faces[3 * g0 + (c0 + 2) % 3];
        uint32_t steps = 1;
        while (w != first && steps <= deg) {
            for (uint32_t x = e0; x < e1; ++x) {
                const int h = (int)list[x], ch = corner_of(faces, h, v);
                if (faces[3 * h + (ch + 1) % 3] == w) { w = faces[3 * h + (ch + 2) % 3]; break; }
            }
            ++steps;
        }
        lk = !(w == first && steps == deg);
    }
    locked[v] = lk;
}

__device__ __forceinline__ double qcost(const double *q, const double *x)
{
    const double r0 = da(da(da(dm(q[0], x[0]), dm(q[1], x[1])), dm(q[2], x[2])), q[3]);
    const double r1 = da(da(da(dm(q[1], x[0]), dm(q[4], x[1])), dm(q[5], x[2])), q[6]);
    const double r2 = da(da(da(dm(q[2], x[0]), dm(q[5], x[1])), dm(q[7], x[2])), q[8]);
    const double r3 = da(da(da(dm(q[3], x[0]), dm(q[6], x[1])), dm(q[8], x[2])), q[9]);
    const double c = da(da(da(dm(r0, x[0]), dm(r1, x[1])), dm(r2, x[2])), r3);
    return c > 0.0 ? c : 0.0;
}

__device__ __forceinline__ double dsq(const double *a, const double *b)
{
    const double d0 = ds(a[0], b[0]), d1 = ds(a[1], b[1]), d2 = ds(a[2], b[2]);
    return da(da(dm(d0, d0), dm(d1, d1)), dm(d2, d2));
}

__device__ __forceinline__ void round32(const double *x, double *r)
{
    for (int k = 0; k < 3; ++k) r[k] = (double)__double2float_rn(x[k]);
}

// position (float32) and cost of collapsing an edge with quadric q and ends A, B
__device__ double place(const double *q, const double *A, const double *B, float *xo)
{
    if (A[0] == B[0] && A[1] == B[1] && A[2] == B[2]) {
        for (int k = 0; k < 3; ++k) xo[k] = (float)A[k];
        return 0.0;
    }
    double mid[3], mr[3];
    for (int k = 0; k < 3; ++k) mid[k] = dm(da(A[k], B[k]), 0.5);
    round32(mid, mr);
    const double cA = qcost(q, A), cB = qcost(q, B), cM = qcost(q, mr);
    const double *best = A;
    double bc = cA;
    if (cB < bc) { best = B; bc = cB; }
    if (cM < bc) { best = mr; bc = cM; }
    const double c00 = ds(dm(q[4], q[7]), dm(q[5], q[5])), c01 = ds(dm(q[2], q[5]), dm(q[1], q[7]));
    const double c02 = ds(dm(q[1], q[5]), dm(q[2], q[4])), c11 = ds(dm(q[0], q[7]), dm(q[2], q[2]));
    const double c12 = ds(dm(q[1], q[2]), dm(q[0], q[5])), c22 = ds(dm(q[0], q[4]), dm(q[1], q[1]));
    const double det = da(da(dm(q[0], c00), dm(q[1], c01)), dm(q[2], c02));
    const double t = da(da(q[0], q[4]), q[7]);
    const double xopt[3] = {-__ddiv_rn(da(da(dm(c00, q[3]), dm(c01, q[6])), dm(c02, q[8])), det),
                            -__ddiv_rn(da(da(dm(c01, q[3]), dm(c11, q[6])), dm(c12, q[8])), det),
                            -__ddiv_rn(da(da(dm(c02, q[3]), dm(c12, q[6])), dm(c22, q[8])), det)};
    if (det > dm(dm(dm(t, t), t), 1e-10) && dsq(xopt, mid) <= dsq(B, A)) {
        double xr[3];
        round32(xopt, xr);
        for (int k = 0; k < 3; ++k) xo[k] = (float)xr[k];
        return qcost(q, xr);
    }
    for (int k = 0; k < 3; ++k) xo[k] = (float)best[k];
    return bc;
}

struct Key { unsigned long long cost, edge; };
__device__ __forceinline__ bool key_less(Key a, Key b) { return a.cost < b.cost || (a.cost == b.cost && a.edge < b.edge); }
__device__ __forceinline__ Key key_none() { return Key{~0ull, ~0ull}; }

// one thread per half-edge slot s = 3 g + k (a = corner k, b = corner k + 1); the edge's data sit at its a < b slot
__global__ void __launch_bounds__(256) candidate_kernel(int F, const float *__restrict__ P, const double *__restrict__ Q,
                                                        const int *__restrict__ faces, const uint32_t *__restrict__ start,
                                                        const uint32_t *__restrict__ list, const uint8_t *__restrict__ locked,
                                                        uint8_t *__restrict__ valid, double *__restrict__ cost, float *__restrict__ X)
{
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= 3 * (int64_t)F) return;
    const int g = (int)(s / 3), k = (int)(s - 3 * (int64_t)g);
    const int a = faces[3 * g + k], b = faces[3 * g + (k + 1) % 3];
    valid[s] = 0;
    if (a >= b || locked[a] || locked[b]) return;
    const uint32_t a0 = start[a], a1 = start[a + 1], b0 = start[b], b1 = start[b + 1];
    if (a1 - a0 == 3 && b1 - b0 == 3) return; // a tetrahedron
    int common = 0;
    for (uint32_t e = a0; e < a1; ++e) {
        const int h = (int)list[e];
        const int w = faces[3 * h + (corner_of(faces, h, a) + 1) % 3];
        for (uint32_t x = b0; x < b1; ++x) {
            const int h2 = (int)list[x];
            if (faces[3 * h2 + (corner_of(faces, h2, b) + 1) % 3] == w) { ++common; break; }
        }
    }
    if (common != 2) return;
    double q[10];
    for (int i = 0; i < 10; ++i) q[i] = da(Q[10 * (size_t)a + i], Q[10 * (size_t)b + i]);
    double A[3], B[3];
    load3(P, a, A); load3(P, b, B);
    float xf[3];
    const double c = place(q, A, B, xf);
    const double xd[3] = {(double)xf[0], (double)xf[1], (double)xf[2]};
    for (int end = 0; end < 2; ++end) {
        const int v = end ? b : a;
        for (uint32_t e = start[v], e1 = start[v + 1]; e < e1; ++e) {
            const int h = (int)list[e];
            const int i0 = faces[3 * h], i1 = faces[3 * h + 1], i2 = faces[3 * h + 2];
            const bool has_a = i0 == a || i1 == a || i2 == a, has_b = i0 == b || i1 == b || i2 == b;
            if (has_a && has_b) continue; // the edge's own faces
            double p[3][3], no[3], nn[3];
            load3(P, i0, p[0]); load3(P, i1, p[1]); load3(P, i2, p[2]);
            cross_d(p[0], p[1], p[2], no);
            if (no[0] == 0.0 && no[1] == 0.0 && no[2] == 0.0) continue; // zero area: exempt
            const int cv = corner_of(faces, h, v);
            for (int j = 0; j < 3; ++j) p[cv][j] = xd[j];
            cross_d(p[0], p[1], p[2], nn);
            if (da(da(dm(no[0], nn[0]), dm(no[1], nn[1])), dm(no[2], nn[2])) <= 0.0) return;
        }
    }
    valid[s] = 1;
    cost[s] = c;
    X[3 * s] = xf[0]; X[3 * s + 1] = xf[1]; X[3 * s + 2] = xf[2];
}

__device__ __forceinline__ Key slot_key(const int *faces, const double *cost, int64_t s)
{
    const int g = (int)(s / 3), k = (int)(s - 3 * (int64_t)g);
    const uint32_t a = (uint32_t)faces[3 * g + k], b = (uint32_t)faces[3 * g + (k + 1) % 3];
    return Key{(unsigned long long)__double_as_longlong(cost[s]), ((unsigned long long)a << 32) | b};
}

// best1[v]: the smallest valid edge at v (each edge at v is a half-edge of a face around v, starting or ending at v)
__global__ void __launch_bounds__(256) best1_kernel(int Nv, const int *__restrict__ faces, const uint32_t *__restrict__ start,
                                                    const uint32_t *__restrict__ list, const uint8_t *__restrict__ valid,
                                                    const double *__restrict__ cost, Key *__restrict__ best1)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Nv) return;
    Key best = key_none();
    for (uint32_t e = start[v], e1 = start[v + 1]; e < e1; ++e) {
        const int g = (int)list[e], c = corner_of(faces, g, v);
        const int64_t s1 = 3 * (int64_t)g + c, s2 = 3 * (int64_t)g + (c + 2) % 3;
        if (valid[s1]) { const Key kk = slot_key(faces, cost, s1); if (key_less(kk, best)) best = kk; }
        if (valid[s2]) { const Key kk = slot_key(faces, cost, s2); if (key_less(kk, best)) best = kk; }
    }
    best1[v] = best;
}

// best2[v]: the smallest best1 over v and its neighbours (every corner of every face around v)
__global__ void __launch_bounds__(256) best2_kernel(int Nv, const int *__restrict__ faces, const uint32_t *__restrict__ start,
                                                    const uint32_t *__restrict__ list, const Key *__restrict__ best1, Key *__restrict__ best2)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Nv) return;
    Key best = best1[v];
    for (uint32_t e = start[v], e1 = start[v + 1]; e < e1; ++e) {
        const int g = (int)list[e];
        for (int c = 0; c < 3; ++c) {
            const Key kk = best1[faces[3 * g + c]];
            if (key_less(kk, best)) best = kk;
        }
    }
    best2[v] = best;
}

__global__ void __launch_bounds__(256) select_kernel(int F, const int *__restrict__ faces, const uint8_t *__restrict__ valid,
                                                     const double *__restrict__ cost, const Key *__restrict__ best2,
                                                     uint8_t *__restrict__ sel, uint32_t *__restrict__ n_sel)
{
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= 3 * (int64_t)F) return;
    bool on = false;
    if (valid[s]) {
        const Key kk = slot_key(faces, cost, s);
        const Key ka = best2[kk.edge >> 32], kb = best2[kk.edge & 0xffffffffu];
        on = ka.cost == kk.cost && ka.edge == kk.edge && kb.cost == kk.cost && kb.edge == kk.edge;
    }
    sel[s] = on;
    if (on) atomicAdd(n_sel, 1u);
}

__global__ void __launch_bounds__(256) sel_list_kernel(int64_t n, const uint8_t *__restrict__ sel, const uint32_t *__restrict__ incl,
                                                       uint32_t *__restrict__ lst, uint32_t *__restrict__ idx)
{
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n || !sel[s]) return;
    lst[incl[s] - 1] = (uint32_t)s;
    idx[incl[s] - 1] = incl[s] - 1;
}

// word w of the (cost, edge) key of selected collapse lst[idx[i]]: 0 = b, 1 = a, 2 = cost low, 3 = cost high
__global__ void __launch_bounds__(256) key_word_kernel(int64_t n, int w, const int *__restrict__ faces, const double *__restrict__ cost,
                                                       const uint32_t *__restrict__ lst, const uint32_t *__restrict__ idx,
                                                       uint32_t *__restrict__ out)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Key kk = slot_key(faces, cost, lst[idx[i]]);
    const unsigned long long x = w < 2 ? kk.edge : kk.cost;
    out[i] = (w & 1) ? (uint32_t)(x >> 32) : (uint32_t)x;
}

__global__ void __launch_bounds__(256) take_kernel(int64_t k, const uint32_t *__restrict__ lst, const uint32_t *__restrict__ idx,
                                                   uint8_t *__restrict__ sel)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < k) sel[lst[idx[i]]] = 1;
}

__global__ void __launch_bounds__(256) collapse_kernel(int F, const int *__restrict__ faces, const uint8_t *__restrict__ sel,
                                                       const float *__restrict__ X, float *__restrict__ P, double *__restrict__ Q,
                                                       int *__restrict__ remap)
{
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= 3 * (int64_t)F || !sel[s]) return;
    const int g = (int)(s / 3), k = (int)(s - 3 * (int64_t)g);
    const int a = faces[3 * g + k], b = faces[3 * g + (k + 1) % 3];
    for (int j = 0; j < 3; ++j) P[3 * (size_t)a + j] = X[3 * s + j];
    for (int i = 0; i < 10; ++i) Q[10 * (size_t)a + i] = da(Q[10 * (size_t)a + i], Q[10 * (size_t)b + i]);
    remap[b] = a;
}

__global__ void __launch_bounds__(256) rename_kernel(int F, int *__restrict__ faces, const int *__restrict__ remap, uint8_t *__restrict__ keep)
{
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= F) return;
    int c[3];
    for (int k = 0; k < 3; ++k) {
        const int v = faces[3 * g + k], r = remap[v];
        c[k] = r >= 0 ? r : v;
        faces[3 * g + k] = c[k];
    }
    keep[g] = !repeats(c[0], c[1], c[2]);
}

__global__ void __launch_bounds__(256) compact_faces_kernel(int F, const int *__restrict__ faces, const uint8_t *__restrict__ keep,
                                                            const uint32_t *__restrict__ incl, int *__restrict__ out)
{
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= F || !keep[g]) return;
    const size_t o = incl[g] - 1;
    out[3 * o] = faces[3 * g]; out[3 * o + 1] = faces[3 * g + 1]; out[3 * o + 2] = faces[3 * g + 2];
}

__global__ void __launch_bounds__(256) mark_used_kernel(int F, const int *__restrict__ faces, uint8_t *__restrict__ used)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 3 * (int64_t)F) used[faces[i]] = 1;
}

struct CleanLayout {
    size_t inc, keep, lab, count, used, box, vkeep, fincl, vincl, tf, tv, words, total;
    CleanLayout(int Nv, int Nf)
    {
        size_t o = 0;
        inc = o; o += gs_align(mesh_incidence_bytes(Nv, Nf));
        keep = o; o += gs_align((size_t)Nf + 1);
        lab = o; o += gs_align((size_t)Nv * 4 + 4);
        count = o; o += gs_align((size_t)Nv * 4 + 4);
        used = o; o += gs_align((size_t)Nv + 1);
        box = o; o += gs_align(((size_t)Nv + 1) * 24);
        vkeep = o; o += gs_align((size_t)Nv + 1);
        fincl = o; o += gs_align((size_t)Nf * 4 + 4);
        vincl = o; o += gs_align((size_t)Nv * 4 + 4);
        tf = o; o += gs_align(popc_scan_temp_bytes(Nf > 0 ? Nf : 1));
        tv = o; o += gs_align(popc_scan_temp_bytes(Nv > 0 ? Nv : 1));
        words = o; o += 64; // u32 [0] bad index, [1] changed; u64 [2], [3] (bytes 16..31) the two totals
        total = o;
    }
};

struct DecimateLayout {
    size_t P, Q, fa, fb, fq, inc, locked, valid, sel, cost, X, best1, best2, remap, keep, incl, temp, lst, ka, kb, va, vb, sort, words, total;
    DecimateLayout(int Nv, int Nf)
    {
        const size_t n3 = 3 * (size_t)Nf + 1, nmax = n3 > (size_t)Nv + 1 ? n3 : (size_t)Nv + 1;
        size_t o = 0;
        P = o; o += gs_align((size_t)Nv * 12 + 4);
        Q = o; o += gs_align((size_t)Nv * 80 + 8);
        fa = o; o += gs_align(n3 * 4);
        fb = o; o += gs_align(n3 * 4);
        fq = o; o += gs_align((size_t)Nf * 80 + 8);
        inc = o; o += gs_align(mesh_incidence_bytes(Nv, Nf));
        locked = o; o += gs_align((size_t)Nv + 1);
        valid = o; o += gs_align(n3);
        sel = o; o += gs_align(n3);
        cost = o; o += gs_align(n3 * 8);
        X = o; o += gs_align(n3 * 12);
        best1 = o; o += gs_align(((size_t)Nv + 1) * sizeof(Key));
        best2 = o; o += gs_align(((size_t)Nv + 1) * sizeof(Key));
        remap = o; o += gs_align((size_t)Nv * 4 + 4);
        keep = o; o += gs_align(nmax);
        incl = o; o += gs_align(nmax * 4);
        temp = o; o += gs_align(popc_scan_temp_bytes((int64_t)nmax));
        lst = o; o += gs_align(n3 * 4);
        ka = o; o += gs_align(n3 * 4);
        kb = o; o += gs_align(n3 * 4);
        va = o; o += gs_align(n3 * 4);
        vb = o; o += gs_align(n3 * 4);
        sort = o; o += gs_align(test_sort32_scratch_bytes((int64_t)n3));
        words = o; o += 64; // u32 [0] bad index, [1] selected count; u64 [2] (bytes 16..23) a scan total
        total = o;
    }
};

int bits_for(uint64_t n)
{
    int b = 1;
    while (((uint64_t)1 << b) < n) b++;
    return b;
}

int read_words(void *host, const void *dev, size_t bytes, cudaStream_t st)
{
    if (cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) return -1;
    return cudaStreamSynchronize(st) != cudaSuccess ? -1 : 0;
}

} // namespace

size_t mesh_clean_scratch_bytes(int Nv, int Nf) { return CleanLayout(Nv, Nf).total; }
size_t mesh_decimate_scratch_bytes(int Nv, int Nf) { return DecimateLayout(Nv, Nf).total; }

// 0, -1 a CUDA call failed, -2 a face index outside [0, Nv)
int launch_mesh_clean(int Nv, int Nf, const float *verts, const int *faces, int min_faces, double min_diameter, char *scratch,
                      float *out_verts, int *out_faces, int64_t *counts, int *rounds, cudaStream_t st, int *n_launches)
{
    const CleanLayout L(Nv, Nf);
    uint32_t *words = (uint32_t *)(scratch + L.words);
    uint8_t *keep = (uint8_t *)(scratch + L.keep), *used = (uint8_t *)(scratch + L.used), *vkeep = (uint8_t *)(scratch + L.vkeep);
    int *lab = (int *)(scratch + L.lab);
    uint32_t *count = (uint32_t *)(scratch + L.count), *box = (uint32_t *)(scratch + L.box);
    uint32_t *fincl = (uint32_t *)(scratch + L.fincl), *vincl = (uint32_t *)(scratch + L.vincl);
    int nl = 0;
    *rounds = 0;
    counts[0] = counts[1] = 0;
    if (cudaMemsetAsync(words, 0, 64, st) != cudaSuccess) return -1;
    if (Nf == 0) { *n_launches = 0; return 0; }
    check_faces_kernel<<<blocks_for(3 * (int64_t)Nf, 256), 256, 0, st>>>(Nv, Nf, faces, words);
    nl++;
    int inl = 0;
    if (launch_mesh_incidence(Nv, Nf, faces, scratch + L.inc, L.keep - L.inc, st, &inl)) return -1;
    nl += inl;
    const uint32_t *start = nullptr, *list = nullptr;
    mesh_incidence_lists(Nv, Nf, scratch + L.inc, &start, &list);
    uint32_t h[2];
    if (read_words(h, words, 8, st)) return -1; // out-of-range faces are in no list: nothing has read them yet
    if (h[0]) { *n_launches = nl + 1; return -2; }
    clean_face_kernel<<<blocks_for(Nf, 256), 256, 0, st>>>(Nf, faces, start, list, keep);
    iota_kernel<<<blocks_for(Nv, 256), 256, 0, st>>>(Nv, lab);
    nl += 2;
    for (;;) {
        if (cudaMemsetAsync(words + 1, 0, 4, st) != cudaSuccess) return -1;
        hook_kernel<<<blocks_for(Nf, 256), 256, 0, st>>>(Nf, faces, keep, lab, words + 1);
        jump_kernel<<<blocks_for(Nv, 256), 256, 0, st>>>(Nv, lab);
        jump_kernel<<<blocks_for(Nv, 256), 256, 0, st>>>(Nv, lab);
        nl += 3;
        ++*rounds;
        if (read_words(h, words, 8, st)) return -1;
        if (!h[1]) break;
    }
    if (cudaMemsetAsync(count, 0, (size_t)Nv * 4, st) != cudaSuccess || cudaMemsetAsync(used, 0, (size_t)Nv, st) != cudaSuccess ||
        cudaMemsetAsync(vkeep, 0, (size_t)Nv, st) != cudaSuccess)
        return -1;
    box_init_kernel<<<blocks_for(6 * ((int64_t)Nv + 1), 256), 256, 0, st>>>(Nv + 1, box);
    comp_mark_kernel<<<blocks_for(Nf, 256), 256, 0, st>>>(Nf, faces, keep, lab, count, used);
    comp_box_kernel<<<blocks_for(Nv, 256), 256, 0, st>>>(Nv, verts, used, lab, box);
    comp_keep_kernel<<<blocks_for(Nf, 256), 256, 0, st>>>(Nv, Nf, faces, keep, lab, count, box, min_faces, min_diameter, vkeep);
    nl += 4;
    uint64_t *tot = (uint64_t *)(words + 4);
    if (launch_popc_scan(keep, fincl, Nf, scratch + L.tf, tot, st)) return -1;
    if (launch_popc_scan(vkeep, vincl, Nv, scratch + L.tv, tot + 1, st)) return -1;
    nl += 2;
    uint64_t t[2];
    if (read_words(t, tot, 16, st)) return -1;
    counts[0] = (int64_t)t[1];
    counts[1] = (int64_t)t[0];
    emit_verts_kernel<<<blocks_for(Nv, 256), 256, 0, st>>>(Nv, verts, vkeep, vincl, out_verts);
    emit_faces_kernel<<<blocks_for(Nf, 256), 256, 0, st>>>(Nf, faces, keep, fincl, vincl, out_faces);
    *n_launches = nl + 2;
    return 0;
}

// 0, -1 a CUDA call failed, -2 a face index outside [0, Nv), -3 the face count after a round is not the planned one
int launch_mesh_decimate(int Nv, int Nf, const float *verts, const int *faces, int target, char *scratch, float *out_verts,
                         int *out_faces, int64_t *counts, int *rounds, cudaStream_t st, int *n_launches)
{
    const DecimateLayout L(Nv, Nf);
    uint32_t *words = (uint32_t *)(scratch + L.words);
    float *P = (float *)(scratch + L.P), *X = (float *)(scratch + L.X);
    double *Q = (double *)(scratch + L.Q), *fq = (double *)(scratch + L.fq), *cost = (double *)(scratch + L.cost);
    int *fcur = (int *)(scratch + L.fa), *fnext = (int *)(scratch + L.fb), *remap = (int *)(scratch + L.remap);
    uint8_t *locked = (uint8_t *)(scratch + L.locked), *valid = (uint8_t *)(scratch + L.valid), *sel = (uint8_t *)(scratch + L.sel);
    uint8_t *keep = (uint8_t *)(scratch + L.keep);
    uint32_t *incl = (uint32_t *)(scratch + L.incl), *lst = (uint32_t *)(scratch + L.lst);
    Key *best1 = (Key *)(scratch + L.best1), *best2 = (Key *)(scratch + L.best2);
    uint64_t *tot = (uint64_t *)(words + 4);
    char *inc = scratch + L.inc;
    const size_t inc_bytes = L.locked - L.inc;
    int nl = 0, inl = 0;
    *rounds = 0;
    counts[0] = counts[1] = 0;
    if (cudaMemsetAsync(words, 0, 64, st) != cudaSuccess) return -1;
    if (Nf == 0) { *n_launches = 0; return 0; }
    check_faces_kernel<<<blocks_for(3 * (int64_t)Nf, 256), 256, 0, st>>>(Nv, Nf, faces, words);
    nl++;
    uint32_t h[2];
    if (read_words(h, words, 8, st)) return -1;
    if (h[0]) { *n_launches = nl; return -2; }
    if (cudaMemcpyAsync(fcur, faces, (size_t)Nf * 12, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(P, verts, (size_t)Nv * 12, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return -1;
    const uint32_t *start = nullptr, *list = nullptr;
    face_quadric_kernel<<<blocks_for(Nf, 256), 256, 0, st>>>(Nf, P, fcur, fq);
    if (launch_mesh_incidence(Nv, Nf, fcur, inc, inc_bytes, st, &inl)) return -1;
    mesh_incidence_lists(Nv, Nf, inc, &start, &list);
    vertex_quadric_kernel<<<blocks_for(Nv, 256), 256, 0, st>>>(Nv, fq, start, list, Q);
    nl += 2 + inl;
    int F = Nf;
    while (F > target) {
        const int64_t n3 = 3 * (int64_t)F;
        if (launch_mesh_incidence(Nv, F, fcur, inc, inc_bytes, st, &inl)) return -1;
        mesh_incidence_lists(Nv, F, inc, &start, &list);
        if (cudaMemsetAsync(words + 1, 0, 4, st) != cudaSuccess) return -1;
        lock_kernel<<<blocks_for(Nv, 256), 256, 0, st>>>(Nv, fcur, start, list, locked);
        candidate_kernel<<<blocks_for(n3, 256), 256, 0, st>>>(F, P, Q, fcur, start, list, locked, valid, cost, X);
        best1_kernel<<<blocks_for(Nv, 256), 256, 0, st>>>(Nv, fcur, start, list, valid, cost, best1);
        best2_kernel<<<blocks_for(Nv, 256), 256, 0, st>>>(Nv, fcur, start, list, best1, best2);
        select_kernel<<<blocks_for(n3, 256), 256, 0, st>>>(F, fcur, valid, cost, best2, sel, words + 1);
        nl += 5 + inl;
        if (read_words(h, words, 8, st)) return -1; // the round's host wait
        const int64_t S = h[1];
        if (S == 0) break;
        ++*rounds;
        const int64_t k = S < ((int64_t)F - target + 1) / 2 ? S : ((int64_t)F - target + 1) / 2;
        if (k < S) { // keep the k cheapest: stable LSD radix passes over b, a, cost low, cost high
            uint32_t *ka = (uint32_t *)(scratch + L.ka), *kb = (uint32_t *)(scratch + L.kb);
            uint32_t *va = (uint32_t *)(scratch + L.va), *vb = (uint32_t *)(scratch + L.vb);
            if (launch_popc_scan(sel, incl, n3, scratch + L.temp, tot, st)) return -1;
            sel_list_kernel<<<blocks_for(n3, 256), 256, 0, st>>>(n3, sel, incl, lst, va);
            nl += 2;
            const int vbits = bits_for((uint64_t)Nv);
            for (int w = 0; w < 4; ++w) {
                key_word_kernel<<<blocks_for(S, 256), 256, 0, st>>>(S, w, fcur, cost, lst, va, ka);
                int in_b = 0;
                if (launch_test_sort32(ka, kb, va, vb, S, w < 2 ? vbits : 32, scratch + L.sort, L.words - L.sort, &in_b, st)) return -1;
                if (in_b) { uint32_t *t = va; va = vb; vb = t; }
                nl += 1 + 3 * (((w < 2 ? vbits : 32) + 8) / 9);
            }
            if (cudaMemsetAsync(sel, 0, (size_t)n3, st) != cudaSuccess) return -1;
            take_kernel<<<blocks_for(k, 256), 256, 0, st>>>(k, lst, va, sel);
            nl++;
        }
        if (cudaMemsetAsync(remap, 0xff, (size_t)Nv * 4, st) != cudaSuccess) return -1;
        collapse_kernel<<<blocks_for(n3, 256), 256, 0, st>>>(F, fcur, sel, X, P, Q, remap);
        rename_kernel<<<blocks_for(F, 256), 256, 0, st>>>(F, fcur, remap, keep);
        if (launch_popc_scan(keep, incl, F, scratch + L.temp, tot, st)) return -1;
        compact_faces_kernel<<<blocks_for(F, 256), 256, 0, st>>>(F, fcur, keep, incl, fnext);
        nl += 4;
        int *t = fcur; fcur = fnext; fnext = t;
        F -= (int)(2 * k);
    }
    // unreferenced vertices out (the last compaction's total, still in tot[0], checks the face count)
    if (cudaMemsetAsync(keep, 0, (size_t)Nv, st) != cudaSuccess) return -1;
    mark_used_kernel<<<blocks_for(3 * (int64_t)F, 256), 256, 0, st>>>(F, fcur, keep);
    if (launch_popc_scan(keep, incl, Nv, scratch + L.temp, tot + 1, st)) return -1;
    nl += 2;
    uint64_t t[2];
    if (read_words(t, tot, 16, st)) return -1;
    if (*rounds > 0 && t[0] != (uint64_t)F) return -3;
    counts[0] = (int64_t)t[1];
    counts[1] = F;
    emit_verts_kernel<<<blocks_for(Nv, 256), 256, 0, st>>>(Nv, P, keep, incl, out_verts);
    emit_faces_kernel<<<blocks_for(F, 256), 256, 0, st>>>(F, fcur, nullptr, nullptr, incl, out_faces);
    *n_launches = nl + 2;
    return 0;
}
