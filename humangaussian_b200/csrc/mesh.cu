// mesh.cu -- mesh export: the opacity-weighted Gaussian density field on a voxel grid, and marching cubes over it
// (DESIGN.md sections 2 and 5).
//
// Density field (the reference's GaussianModel.extract_fields).  The grid's res samples per axis are split into chunks
// of `split` samples; chunk c's box is [min, max] of its samples widened by `relax` on both sides, and a Gaussian
// counts for every voxel of block (cx, cy, cz) iff its centre lies strictly inside that block's box on all three axes.
// Each voxel gets sum over those Gaussians of opacity * exp(power) (0 where power > 0).
//   1. prep: per Gaussian the closed-form inverse of its covariance (the reference's operation order) and its home
//      chunk per axis, h(x) = #{c >= 1 : sample[c*split] <= x}, monotone in x;
//   2. stable radix sort by home-chunk key (radix.cuh, through launch_test_sort32), gather of the 40 B records into
//      sorted order, and start[key] = first sorted position with that key;
//   3. field: one CTA per (block, group of FIELD_VOX voxels).  Every Gaussian whose centre is inside the widened box
//      has its home chunk in [h(lo), h(hi)] per axis, so the CTA walks those home keys (one contiguous run per
//      (hx, hy)), keeps the exact members, stages them in shared memory and adds them to its voxels in sorted order.
//      No atomics: the field is the same bits on every run.
// Marching cubes: classify every grid point (which of its three forward edges cross the iso value; the case of the cell
// it is the lowest corner of), scan the vertex and triangle counts with the binning stage's look-back scan of byte
// popcounts (launch_popc_scan: a count n is stored as the byte 2^n - 1), and emit.  A
// vertex belongs to the grid point at the low end of its edge; vertices are numbered in (point, axis) order, triangles
// in (cell, table) order.  The triangle table is generated (mc_table.py -> mc_table.h).
#include "common.cuh"
#include "kernels.h"
#include "mc_table.h"

namespace {

constexpr int FIELD_THREADS = 256;
constexpr int FIELD_VPT = 2;                                // voxels per thread
constexpr int FIELD_VOX = FIELD_THREADS * FIELD_VPT;        // voxels per CTA
constexpr int STAGE_CAP = 2 * FIELD_THREADS;                // staged records; a tile of FIELD_THREADS always fits after a flush check

struct MeshRec { float mx, my, mz, ia, ib, ic, id, ie, ifz, o; }; // 40 B: centre, inverse (a,b,c,d,e,f), opacity
static_assert(sizeof(MeshRec) == 40, "MeshRec must be 40 bytes");

__device__ __forceinline__ int home_chunk(const float *__restrict__ samples, int split, int nch, float x)
{
    int lo = 0, hi = nch - 1; // largest c with c == 0 or samples[c*split] <= x
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (samples[(size_t)mid * split] <= x) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(256) field_prep_kernel(int P, const float *__restrict__ means, const float *__restrict__ cov6,
                                                         const float *__restrict__ opac, const float *__restrict__ samples, int split,
                                                         int nch, MeshRec *__restrict__ rec, uint32_t *__restrict__ keys,
                                                         uint32_t *__restrict__ vals)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float a = cov6[6 * i + 0], b = cov6[6 * i + 1], c = cov6[6 * i + 2], d = cov6[6 * i + 3], e = cov6[6 * i + 4],
                f = cov6[6 * i + 5];
    // 1 / (a*d*f + 2*e*c*b - e^2*a - c^2*d - b^2*f + 1e-24), left to right, one rounding per operation
    float det = fmul(fmul(a, d), f);
    det = fadd(det, fmul(fmul(fmul(2.0f, e), c), b));
    det = fsub(det, fmul(fmul(e, e), a));
    det = fsub(det, fmul(fmul(c, c), d));
    det = fsub(det, fmul(fmul(b, b), f));
    det = fadd(det, 1e-24f);
    const float inv_det = fdiv(1.0f, det);
    MeshRec r;
    r.mx = means[3 * i]; r.my = means[3 * i + 1]; r.mz = means[3 * i + 2];
    r.ia = fmul(fsub(fmul(d, f), fmul(e, e)), inv_det);
    r.ib = fmul(fsub(fmul(e, c), fmul(b, f)), inv_det);
    r.ic = fmul(fsub(fmul(e, b), fmul(c, d)), inv_det);
    r.id = fmul(fsub(fmul(a, f), fmul(c, c)), inv_det);
    r.ie = fmul(fsub(fmul(b, c), fmul(e, a)), inv_det);
    r.ifz = fmul(fsub(fmul(a, d), fmul(b, b)), inv_det);
    r.o = opac[i];
    rec[i] = r;
    const uint32_t hx = home_chunk(samples, split, nch, r.mx), hy = home_chunk(samples, split, nch, r.my),
                   hz = home_chunk(samples, split, nch, r.mz);
    keys[i] = (hx * nch + hy) * nch + hz;
    vals[i] = i;
}

// sorted[j] = rec[order[j]]; start[k] = first j with key[j] >= k, for k in [0, nkeys]  (thread j = P writes the tail)
__global__ void __launch_bounds__(256) field_gather_kernel(int P, uint32_t nkeys, const uint32_t *__restrict__ skeys,
                                                           const uint32_t *__restrict__ order, const MeshRec *__restrict__ rec,
                                                           MeshRec *__restrict__ sorted, uint32_t *__restrict__ start)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > P) return;
    const int64_t prev = j == 0 ? -1 : (int64_t)skeys[j - 1];
    const int64_t cur = j == P ? (int64_t)nkeys : (int64_t)skeys[j];
    for (int64_t k = prev + 1; k <= cur; k++) start[k] = (uint32_t)j;
    if (j < P) sorted[j] = rec[order[j]];
}

__global__ void __launch_bounds__(FIELD_THREADS) field_kernel(int res, int split, int nch, int groups, const float *__restrict__ samples,
                                                              float relax, const MeshRec *__restrict__ sorted,
                                                              const uint32_t *__restrict__ start, float *__restrict__ field)
{
    __shared__ float s_rec[10][STAGE_CAP];
    __shared__ float s_lo[3], s_hi[3];
    __shared__ int s_beg[3], s_ext[3], s_h0[3], s_h1[3];
    __shared__ int s_wcount[FIELD_THREADS / 32];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t blk = blockIdx.x / groups;
    const int grp = (int)(blockIdx.x % groups);
    if (tid < 3) {
        const int64_t b = tid == 0 ? blk / ((int64_t)nch * nch) : (tid == 1 ? (blk / nch) % nch : blk % nch);
        const int beg = (int)b * split, end = min(res, beg + split);
        float mn = samples[beg], mx = samples[beg];
        for (int k = beg + 1; k < end; k++) { mn = fminf(mn, samples[k]); mx = fmaxf(mx, samples[k]); }
        const float lo = fsub(mn, relax), hi = fadd(mx, relax);
        s_lo[tid] = lo; s_hi[tid] = hi; s_beg[tid] = beg; s_ext[tid] = end - beg;
        s_h0[tid] = home_chunk(samples, split, nch, lo);
        s_h1[tid] = home_chunk(samples, split, nch, hi);
    }
    __syncthreads();
    const int ex = s_ext[0], ey = s_ext[1], ez = s_ext[2];
    const int nvox = ex * ey * ez;
    if (grp * FIELD_VOX >= nvox) return; // a short edge block: the whole CTA leaves before any further barrier
    const float lox = s_lo[0], loy = s_lo[1], loz = s_lo[2], hix = s_hi[0], hiy = s_hi[1], hiz = s_hi[2];

    float px[FIELD_VPT], py[FIELD_VPT], pz[FIELD_VPT], acc[FIELD_VPT];
    int64_t out[FIELD_VPT];
#pragma unroll
    for (int k = 0; k < FIELD_VPT; k++) {
        const int v = grp * FIELD_VOX + k * FIELD_THREADS + tid;
        const int vv = v < nvox ? v : 0;
        const int iz = vv % ez, iy = (vv / ez) % ey, ix = vv / (ey * ez);
        px[k] = samples[s_beg[0] + ix]; py[k] = samples[s_beg[1] + iy]; pz[k] = samples[s_beg[2] + iz];
        out[k] = v < nvox ? ((int64_t)(s_beg[0] + ix) * res + (s_beg[1] + iy)) * res + (s_beg[2] + iz) : -1;
        acc[k] = 0.0f;
    }

    auto evaluate = [&](int n) {
        for (int r = 0; r < n; r++) {
            const float mx = s_rec[0][r], my = s_rec[1][r], mz = s_rec[2][r];
            const float ia = s_rec[3][r], ib = s_rec[4][r], ic = s_rec[5][r], id = s_rec[6][r], ie = s_rec[7][r], ifz = s_rec[8][r];
            const float o = s_rec[9][r];
#pragma unroll
            for (int k = 0; k < FIELD_VPT; k++) {
                const float x = fsub(px[k], mx), y = fsub(py[k], my), z = fsub(pz[k], mz);
                // -0.5 * (x^2*ia + y^2*id + z^2*if) - x*y*ib - x*z*ic - y*z*ie, left to right
                float s = fadd(fmul(fmul(x, x), ia), fmul(fmul(y, y), id));
                s = fadd(s, fmul(fmul(z, z), ifz));
                float p = fmul(-0.5f, s);
                p = fsub(p, fmul(fmul(x, y), ib));
                p = fsub(p, fmul(fmul(x, z), ic));
                p = fsub(p, fmul(fmul(y, z), ie));
                // p > 0 adds nothing (the reference sets it to -1e10); exp(p) rounds to 0 in float32 below -104 (the smallest
                // subnormal is e^-103.28), so skipping those is exact.  A NaN passes both tests and propagates, as there.
                if (!(p > 0.0f) && !(p <= -104.0f)) acc[k] = fadd(acc[k], fmul(o, expf(p)));
            }
        }
    };

    int staged = 0; // identical in every thread
    const int h0x = s_h0[0], h1x = s_h1[0], h0y = s_h0[1], h1y = s_h1[1], h0z = s_h0[2], h1z = s_h1[2];
    for (int hx = h0x; hx <= h1x; hx++) {
        for (int hy = h0y; hy <= h1y; hy++) {
            const int64_t k0 = ((int64_t)hx * nch + hy) * nch;
            const uint32_t beg = start[k0 + h0z], end = start[k0 + h1z + 1];
            for (uint32_t base = beg; base < end; base += FIELD_THREADS) {
                const uint32_t j = base + tid;
                bool in = false;
                MeshRec r;
                if (j < end) {
                    r = sorted[j];
                    in = r.mx > lox && r.mx < hix && r.my > loy && r.my < hiy && r.mz > loz && r.mz < hiz;
                }
                const uint32_t bal = __ballot_sync(0xffffffffu, in);
                if (lane == 0) s_wcount[warp] = __popc(bal);
                __syncthreads();
                int pos = staged, total = staged;
                for (int w = 0; w < FIELD_THREADS / 32; w++) {
                    const int c = s_wcount[w];
                    if (w < warp) pos += c;
                    total += c;
                }
                if (in) {
                    pos += __popc(bal & ((1u << lane) - 1u));
                    s_rec[0][pos] = r.mx; s_rec[1][pos] = r.my; s_rec[2][pos] = r.mz; s_rec[3][pos] = r.ia; s_rec[4][pos] = r.ib;
                    s_rec[5][pos] = r.ic; s_rec[6][pos] = r.id; s_rec[7][pos] = r.ie; s_rec[8][pos] = r.ifz; s_rec[9][pos] = r.o;
                }
                __syncthreads();
                staged = total;
                if (staged > STAGE_CAP - FIELD_THREADS) {
                    evaluate(staged);
                    staged = 0;
                    __syncthreads();
                }
            }
        }
    }
    if (staged) evaluate(staged);
#pragma unroll
    for (int k = 0; k < FIELD_VPT; k++)
        if (out[k] >= 0) field[out[k]] = acc[k];
}

// ---- marching cubes ----------------------------------------------------------------------------------------------------
__device__ const uint8_t d_edge_corner[12] = MC_EDGE_CORNER_INIT;
__device__ const uint8_t d_edge_axis[12] = MC_EDGE_AXIS_INIT;
__device__ const uint8_t d_tri_count[256] = MC_TRI_COUNT_INIT;
__device__ const int8_t d_tri_edges[256][3 * MC_MAX_TRIS] = MC_TRI_EDGES_INIT;

__global__ void __launch_bounds__(256) mc_classify_kernel(int X, int Y, int Z, const float *__restrict__ vol, float iso,
                                                          uint8_t *__restrict__ emask, uint8_t *__restrict__ cases,
                                                          uint8_t *__restrict__ tmask)
{
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t N = (int64_t)X * Y * Z;
    if (p >= N) return;
    const int z = (int)(p % Z), y = (int)((p / Z) % Y), x = (int)(p / ((int64_t)Y * Z));
    const int64_t sx = (int64_t)Y * Z, sy = Z;
    const bool in0 = vol[p] > iso;
    uint32_t m = 0;
    if (x + 1 < X && (vol[p + sx] > iso) != in0) m |= 1u;
    if (y + 1 < Y && (vol[p + sy] > iso) != in0) m |= 2u;
    if (z + 1 < Z && (vol[p + 1] > iso) != in0) m |= 4u;
    emask[p] = (uint8_t)m;
    uint32_t c = 0;
    if (x + 1 < X && y + 1 < Y && z + 1 < Z) {
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int64_t q = p + (k & 1) * sx + ((k >> 1) & 1) * sy + ((k >> 2) & 1);
            c |= (uint32_t)(vol[q] > iso) << k;
        }
    }
    cases[p] = (uint8_t)c;
    tmask[p] = (uint8_t)((1u << d_tri_count[c]) - 1u); // popc = the cell's triangle count
}

__global__ void __launch_bounds__(256) mc_vertex_kernel(int X, int Y, int Z, const float *__restrict__ vol, float iso,
                                                        const uint8_t *__restrict__ emask, const uint32_t *__restrict__ vincl,
                                                        float *__restrict__ verts)
{
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t N = (int64_t)X * Y * Z;
    if (p >= N) return;
    const uint32_t m = emask[p];
    if (!m) return;
    const int z = (int)(p % Z), y = (int)((p / Z) % Y), x = (int)(p / ((int64_t)Y * Z));
    const int64_t step[3] = {(int64_t)Y * Z, Z, 1};
    const float v0 = vol[p];
    int64_t vid = (int64_t)vincl[p] - __popc(m);
#pragma unroll
    for (int a = 0; a < 3; a++) {
        if (!(m >> a & 1u)) continue;
        const float v1 = vol[p + step[a]];
        const float t = fdiv(fsub(iso, v0), fsub(v1, v0));
        float c[3] = {(float)x, (float)y, (float)z};
        c[a] = fadd(c[a], t);
        verts[3 * vid] = c[0]; verts[3 * vid + 1] = c[1]; verts[3 * vid + 2] = c[2];
        vid++;
    }
}

__global__ void __launch_bounds__(256) mc_face_kernel(int X, int Y, int Z, const uint8_t *__restrict__ emask,
                                                      const uint8_t *__restrict__ cases, const uint32_t *__restrict__ vincl,
                                                      const uint32_t *__restrict__ tincl, int32_t *__restrict__ faces)
{
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t N = (int64_t)X * Y * Z;
    if (p >= N) return;
    const uint32_t c = cases[p];
    const int nt = d_tri_count[c];
    if (!nt) return;
    const int64_t sx = (int64_t)Y * Z, sy = Z;
    const int64_t base = (int64_t)tincl[p] - nt;
    for (int j = 0; j < 3 * nt; j++) {
        const int e = d_tri_edges[c][j];
        const int k = d_edge_corner[e], a = d_edge_axis[e];
        const int64_t q = p + (k & 1) * sx + ((k >> 1) & 1) * sy + ((k >> 2) & 1);
        const uint32_t m = emask[q];
        faces[3 * base + j] = (int32_t)(vincl[q] - __popc(m) + __popc(m & ((1u << a) - 1u)));
    }
}

struct McLayout {
    size_t emask, cases, tmask, vincl, tincl, temp, total;
    McLayout(int64_t N)
    {
        size_t o = 0;
        emask = o; o += gs_align((size_t)N);
        cases = o; o += gs_align((size_t)N);
        tmask = o; o += gs_align((size_t)N);
        vincl = o; o += gs_align((size_t)N * 4);
        tincl = o; o += gs_align((size_t)N * 4);
        temp = o; o += popc_scan_temp_bytes(N);
        total = o;
    }
};

struct FieldLayout {
    size_t rec, sorted, ka, kb, va, vb, start, sort, total;
    FieldLayout(int P, int64_t nkeys)
    {
        const size_t n = (size_t)(P > 0 ? P : 1);
        size_t o = 0;
        rec = o; o += gs_align(n * sizeof(MeshRec));
        sorted = o; o += gs_align(n * sizeof(MeshRec));
        ka = o; o += gs_align(n * 4);
        kb = o; o += gs_align(n * 4);
        va = o; o += gs_align(n * 4);
        vb = o; o += gs_align(n * 4);
        start = o; o += gs_align((size_t)(nkeys + 1) * 4);
        sort = o; o += test_sort32_scratch_bytes((int64_t)n);
        total = o;
    }
};

int bits_for(uint64_t n)
{
    int b = 0;
    while (((uint64_t)1 << b) < n) b++;
    return b > 0 ? b : 1;
}

} // namespace

size_t density_field_scratch_bytes(int P, int res, int split)
{
    const int64_t nch = (res + split - 1) / split;
    return FieldLayout(P, nch * nch * nch).total;
}

int launch_density_field(int P, const float *means, const float *cov6, const float *opac, int res, int split, const float *samples,
                         float relax, float *field, char *scratch, size_t scratch_bytes, cudaStream_t st, int *n_launches)
{
    const int nch = (res + split - 1) / split;
    const int64_t nkeys = (int64_t)nch * nch * nch;
    const FieldLayout L(P, nkeys);
    if (scratch_bytes < L.total) return -1;
    MeshRec *rec = (MeshRec *)(scratch + L.rec), *sorted = (MeshRec *)(scratch + L.sorted);
    uint32_t *ka = (uint32_t *)(scratch + L.ka), *kb = (uint32_t *)(scratch + L.kb), *va = (uint32_t *)(scratch + L.va),
             *vb = (uint32_t *)(scratch + L.vb), *start = (uint32_t *)(scratch + L.start);
    field_prep_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, means, cov6, opac, samples, split, nch, rec, ka, va);
    int in_b = 0;
    if (launch_test_sort32(ka, kb, va, vb, P, bits_for((uint64_t)nkeys), scratch + L.sort, scratch_bytes - L.sort, &in_b, st)) return -2;
    const int nsort = 3 * ((bits_for((uint64_t)nkeys) + 8) / 9);
    field_gather_kernel<<<(P + 1 + 255) / 256, 256, 0, st>>>(P, (uint32_t)nkeys, in_b ? kb : ka, in_b ? vb : va, rec, sorted, start);
    const int64_t vox = (int64_t)split * split * split;
    const int groups = (int)((vox + FIELD_VOX - 1) / FIELD_VOX);
    field_kernel<<<(unsigned)(nkeys * groups), FIELD_THREADS, 0, st>>>(res, split, nch, groups, samples, relax, sorted, start, field);
    *n_launches += 3 + nsort;
    return 0;
}

size_t marching_cubes_scratch_bytes(int X, int Y, int Z) { return McLayout((int64_t)X * Y * Z).total; }

int launch_marching_cubes_count(int X, int Y, int Z, const float *vol, float iso, char *scratch, size_t scratch_bytes, uint64_t *counts,
                                cudaStream_t st, int *n_launches)
{
    const int64_t N = (int64_t)X * Y * Z;
    const McLayout L(N);
    if (scratch_bytes < L.total) return -1;
    uint8_t *emask = (uint8_t *)(scratch + L.emask), *cases = (uint8_t *)(scratch + L.cases), *tmask = (uint8_t *)(scratch + L.tmask);
    const unsigned g = (unsigned)((N + 255) / 256);
    mc_classify_kernel<<<g, 256, 0, st>>>(X, Y, Z, vol, iso, emask, cases, tmask);
    // the scans run one after the other on the stream, so they share one temp area
    if (launch_popc_scan(emask, (uint32_t *)(scratch + L.vincl), N, scratch + L.temp, counts, st)) return -2;
    if (launch_popc_scan(tmask, (uint32_t *)(scratch + L.tincl), N, scratch + L.temp, counts + 1, st)) return -2;
    *n_launches += 3;
    return 0;
}

int launch_marching_cubes_emit(int X, int Y, int Z, const float *vol, float iso, const char *scratch, size_t scratch_bytes, float *verts,
                               int32_t *faces, cudaStream_t st, int *n_launches)
{
    const int64_t N = (int64_t)X * Y * Z;
    const McLayout L(N);
    if (scratch_bytes < L.total) return -1;
    const uint8_t *emask = (const uint8_t *)(scratch + L.emask), *cases = (const uint8_t *)(scratch + L.cases);
    const uint32_t *vincl = (const uint32_t *)(scratch + L.vincl), *tincl = (const uint32_t *)(scratch + L.tincl);
    const unsigned g = (unsigned)((N + 255) / 256);
    if (verts) mc_vertex_kernel<<<g, 256, 0, st>>>(X, Y, Z, vol, iso, emask, vincl, verts);
    if (faces) mc_face_kernel<<<g, 256, 0, st>>>(X, Y, Z, emask, cases, vincl, tincl, faces);
    *n_launches += (verts != nullptr) + (faces != nullptr);
    return 0;
}
