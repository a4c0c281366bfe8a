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
// Field query: the same sum at arbitrary points of the field's frame, with its gradient and the opacity-weighted SH
// coefficients (colour).  The Gaussian side is steps 1-2 above (plus a gather of each Gaussian's first (deg+1)^2 SH
// rows into sorted order); the points are radix-sorted by the key of the block they fall in, and one CTA per
// QUERY_THREADS sorted points walks, block by block, exactly the member ranges field_kernel walks for that block, in the
// same order, so at a grid sample the density is the field's voxel bit for bit.  Results go to the caller's order.
// Marching cubes: classify every grid point (which of its three forward edges cross the iso value; the case of the cell
// it is the lowest corner of), scan the vertex and triangle counts with the binning stage's look-back scan of byte
// popcounts (launch_popc_scan: a count n is stored as the byte 2^n - 1), and emit.  A
// vertex belongs to the grid point at the low end of its edge; vertices are numbered in (point, axis) order, triangles
// in (cell, table) order.  The triangle table is generated (mc_table.py -> mc_table.h).
#include "common.cuh"
#include "kernels.h"
#include "mc_table.h"
#include "sh.cuh"

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

// ---- field query -------------------------------------------------------------------------------------------------------
constexpr int QUERY_THREADS = 32;  // one warp per CTA: a tile spans few blocks, and each block's walk is serial
constexpr int QUERY_CAP = 2 * QUERY_THREADS; // staged members; as STAGE_CAP, a tile always fits after a flush check

__host__ __device__ constexpr int query_coeffs(int deg) { return deg >= 0 ? (deg + 1) * (deg + 1) : 0; }
constexpr size_t query_smem_bytes(int deg) { return (size_t)(10 + 3 * query_coeffs(deg)) * QUERY_CAP * sizeof(float); }

// keys[i] = the key of the block point i falls in (home_chunk per axis, as the field prep keys a Gaussian's centre)
__global__ void __launch_bounds__(256) query_prep_kernel(int n, const float *__restrict__ points, const float *__restrict__ samples,
                                                         int split, int nch, uint32_t *__restrict__ keys, uint32_t *__restrict__ vals)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t hx = home_chunk(samples, split, nch, points[3 * (int64_t)i]),
                   hy = home_chunk(samples, split, nch, points[3 * (int64_t)i + 1]),
                   hz = home_chunk(samples, split, nch, points[3 * (int64_t)i + 2]);
    keys[i] = (hx * nch + hy) * nch + hz;
    vals[i] = i;
}

// sorted_sh[j*k3 + c] = shs[order[j]*stride + c] for c < k3: the first k3 floats of each Gaussian's SH row, in sorted order
__global__ void __launch_bounds__(256) query_gather_sh_kernel(int P, int k3, int stride, const uint32_t *__restrict__ order,
                                                              const float *__restrict__ shs, float *__restrict__ sorted_sh)
{
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)P * k3) return;
    const int64_t j = t / k3;
    const int c = (int)(t - j * k3);
    sorted_sh[t] = shs[(int64_t)order[j] * stride + c];
}

// One CTA per QUERY_THREADS points in key order.  The tile's points fall in one or a few blocks (runs of equal keys); per
// run the CTA stages that block's members as field_kernel does, and the run's threads sum them.  DEG = -1: no colour.
template <int DEG>
__global__ void __launch_bounds__(QUERY_THREADS, 4) field_query_kernel(
    int n, int res, int split, int nch, const float *__restrict__ samples, float relax, const MeshRec *__restrict__ sorted,
    const float *__restrict__ sorted_sh, const uint32_t *__restrict__ start, const uint32_t *__restrict__ pkeys,
    const uint32_t *__restrict__ porder, const float *__restrict__ points, float *__restrict__ density, float *__restrict__ normals,
    float *__restrict__ colors)
{
    constexpr int NC = query_coeffs(DEG), K3 = 3 * NC;
    extern __shared__ float s_dyn[];
    float(*s_rec)[QUERY_CAP] = reinterpret_cast<float(*)[QUERY_CAP]>(s_dyn); // rows 0-9: MeshRec, rows 10..: SH floats
    __shared__ uint32_t s_key[QUERY_THREADS];
    __shared__ float s_lo[3], s_hi[3];
    __shared__ int s_h0[3], s_h1[3];
    __shared__ int s_wcount[QUERY_THREADS / 32];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t first = (int64_t)blockIdx.x * QUERY_THREADS;
    const int tile_n = (int)min((int64_t)QUERY_THREADS, (int64_t)n - first);
    const bool live = tid < tile_n;
    uint32_t key = 0, idx = 0;
    float qx = 0.0f, qy = 0.0f, qz = 0.0f;
    if (live) {
        key = pkeys[first + tid];
        idx = porder[first + tid];
        qx = points[3 * (int64_t)idx]; qy = points[3 * (int64_t)idx + 1]; qz = points[3 * (int64_t)idx + 2];
    }
    s_key[tid] = key;
    float D = 0.0f, gx = 0.0f, gy = 0.0f, gz = 0.0f, S[K3 > 0 ? K3 : 1];
#pragma unroll
    for (int c = 0; c < K3; c++) S[c] = 0.0f;
    __syncthreads();

    for (int seg = 0; seg < tile_n;) {
        const uint32_t cur = s_key[seg];
        const bool mine = live && key == cur;
        if (tid < 3) { // the block's widened box and home-chunk range, as field_kernel computes them
            const uint32_t b = tid == 0 ? cur / ((uint32_t)nch * nch) : (tid == 1 ? (cur / nch) % nch : cur % nch);
            const int beg = (int)b * split, end = min(res, beg + split);
            float mn = samples[beg], mx = samples[beg];
            for (int k = beg + 1; k < end; k++) { mn = fminf(mn, samples[k]); mx = fmaxf(mx, samples[k]); }
            const float lo = fsub(mn, relax), hi = fadd(mx, relax);
            s_lo[tid] = lo; s_hi[tid] = hi;
            s_h0[tid] = home_chunk(samples, split, nch, lo);
            s_h1[tid] = home_chunk(samples, split, nch, hi);
        }
        const int run = __syncthreads_count(mine); // keys are sorted: the run is [seg, seg + run)
        const float lox = s_lo[0], loy = s_lo[1], loz = s_lo[2], hix = s_hi[0], hiy = s_hi[1], hiz = s_hi[2];

        auto evaluate = [&](int cnt) {
            if (!mine) return;
            for (int r = 0; r < cnt; r++) {
                const float mx = s_rec[0][r], my = s_rec[1][r], mz = s_rec[2][r];
                const float ia = s_rec[3][r], ib = s_rec[4][r], ic = s_rec[5][r], id = s_rec[6][r], ie = s_rec[7][r], ifz = s_rec[8][r];
                const float x = fsub(qx, mx), y = fsub(qy, my), z = fsub(qz, mz);
                // the exponent and the cut-offs of field_kernel, operation for operation
                float s = fadd(fmul(fmul(x, x), ia), fmul(fmul(y, y), id));
                s = fadd(s, fmul(fmul(z, z), ifz));
                float p = fmul(-0.5f, s);
                p = fsub(p, fmul(fmul(x, y), ib));
                p = fsub(p, fmul(fmul(x, z), ic));
                p = fsub(p, fmul(fmul(y, z), ie));
                if (!(p > 0.0f) && !(p <= -104.0f)) {
                    const float w = fmul(s_rec[9][r], expf(p));
                    D = fadd(D, w);
                    // w * (-Sigma^-1 d)
                    gx = ffma(-w, ffma(ic, z, ffma(ib, y, fmul(ia, x))), gx);
                    gy = ffma(-w, ffma(ie, z, ffma(id, y, fmul(ib, x))), gy);
                    gz = ffma(-w, ffma(ifz, z, ffma(ie, y, fmul(ic, x))), gz);
#pragma unroll
                    for (int c = 0; c < K3; c++) S[c] = ffma(w, s_rec[10 + c][r], S[c]);
                }
            }
        };

        int staged = 0; // identical in every thread
        const int h0x = s_h0[0], h1x = s_h1[0], h0y = s_h0[1], h1y = s_h1[1], h0z = s_h0[2], h1z = s_h1[2];
        for (int hx = h0x; hx <= h1x; hx++) {
            for (int hy = h0y; hy <= h1y; hy++) {
                const int64_t k0 = ((int64_t)hx * nch + hy) * nch;
                const uint32_t beg = start[k0 + h0z], end = start[k0 + h1z + 1];
                for (uint32_t base = beg; base < end; base += QUERY_THREADS) {
                    const uint32_t g = base + tid;
                    bool in = false;
                    MeshRec r;
                    if (g < end) {
                        r = sorted[g];
                        in = r.mx > lox && r.mx < hix && r.my > loy && r.my < hiy && r.mz > loz && r.mz < hiz;
                    }
                    const uint32_t bal = __ballot_sync(0xffffffffu, in);
                    if (lane == 0) s_wcount[warp] = __popc(bal);
                    __syncthreads();
                    int pos = staged, total = staged;
                    for (int w = 0; w < QUERY_THREADS / 32; w++) {
                        const int c = s_wcount[w];
                        if (w < warp) pos += c;
                        total += c;
                    }
                    if (in) {
                        pos += __popc(bal & ((1u << lane) - 1u));
                        s_rec[0][pos] = r.mx; s_rec[1][pos] = r.my; s_rec[2][pos] = r.mz; s_rec[3][pos] = r.ia; s_rec[4][pos] = r.ib;
                        s_rec[5][pos] = r.ic; s_rec[6][pos] = r.id; s_rec[7][pos] = r.ie; s_rec[8][pos] = r.ifz; s_rec[9][pos] = r.o;
#pragma unroll
                        for (int c = 0; c < K3; c++) s_rec[10 + c][pos] = sorted_sh[(int64_t)g * K3 + c];
                    }
                    __syncthreads();
                    staged = total;
                    if (staged > QUERY_CAP - QUERY_THREADS) {
                        evaluate(staged);
                        staged = 0;
                        __syncthreads();
                    }
                }
            }
        }
        if (staged) evaluate(staged);
        __syncthreads(); // the next run restages s_rec and rewrites the box
        seg += run;
    }
    if (!live) return;

    if (density) density[idx] = D;
    float nx = 0.0f, ny = 0.0f, nz = 0.0f, len = 0.0f;
    if (D != 0.0f) {
        len = norm3df(gx, gy, gz);
        if (len > 0.0f) { nx = -fdiv(gx, len); ny = -fdiv(gy, len); nz = -fdiv(gz, len); }
    }
    if (normals) { normals[3 * (int64_t)idx] = nx; normals[3 * (int64_t)idx + 1] = ny; normals[3 * (int64_t)idx + 2] = nz; }
    if (DEG >= 0 && colors) {
        float rgb[3] = {0.0f, 0.0f, 0.0f};
        if (D != 0.0f) {
            // SH of the mean coefficients S / D, seen along dir = -n (DC alone where n = 0); the preprocess's colour sum
            float bs[16];
            const bool directional = DEG > 0 && len > 0.0f;
            sh_basis(DEG, -nx, -ny, -nz, bs);
            float acc[3];
#pragma unroll
            for (int ch = 0; ch < 3; ch++) acc[ch] = fmul(bs[0], fdiv(S[ch], D));
            if (directional) {
#pragma unroll
                for (int k = 1; k < NC; k++)
#pragma unroll
                    for (int ch = 0; ch < 3; ch++) acc[ch] = ffma(bs[k], fdiv(S[3 * k + ch], D), acc[ch]);
            }
#pragma unroll
            for (int ch = 0; ch < 3; ch++) rgb[ch] = fmaxf(fadd(acc[ch], 0.5f), 0.0f);
        }
        colors[3 * (int64_t)idx] = rgb[0]; colors[3 * (int64_t)idx + 1] = rgb[1]; colors[3 * (int64_t)idx + 2] = rgb[2];
    }
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
    // the Gaussian side (density field and query); the query adds its sorted SH floats and its point keys
    size_t rec, sorted, ka, kb, va, vb, start, sort, sh, pka, pkb, pva, pvb, total;
    FieldLayout(int P, int64_t nkeys, int n_points = 0, int sh_floats = 0)
    {
        const size_t n = (size_t)(P > 0 ? P : 1), m = (size_t)(n_points > 0 ? n_points : 0);
        size_t o = 0;
        rec = o; o += gs_align(n * sizeof(MeshRec));
        sorted = o; o += gs_align(n * sizeof(MeshRec));
        ka = o; o += gs_align(n * 4);
        kb = o; o += gs_align(n * 4);
        va = o; o += gs_align(n * 4);
        vb = o; o += gs_align(n * 4);
        start = o; o += gs_align((size_t)(nkeys + 1) * 4);
        sort = o; o += test_sort32_scratch_bytes((int64_t)(m > n ? m : n));
        sh = o; o += gs_align(n * sh_floats * 4);
        pka = o; o += gs_align(m * 4);
        pkb = o; o += gs_align(m * 4);
        pva = o; o += gs_align(m * 4);
        pvb = o; o += gs_align(m * 4);
        total = o;
    }
};

int bits_for(uint64_t n)
{
    int b = 0;
    while (((uint64_t)1 << b) < n) b++;
    return b > 0 ? b : 1;
}

// Steps 1-2 of the field: prep, sort by home key, gather.  -> the sorted order of the Gaussians (into `rec` index space)
const uint32_t *sort_gaussians(int P, const float *means, const float *cov6, const float *opac, int split, int nch, int64_t nkeys,
                               const float *samples, const FieldLayout &L, char *scratch, size_t scratch_bytes, cudaStream_t st,
                               int *n_launches)
{
    MeshRec *rec = (MeshRec *)(scratch + L.rec), *sorted = (MeshRec *)(scratch + L.sorted);
    uint32_t *ka = (uint32_t *)(scratch + L.ka), *kb = (uint32_t *)(scratch + L.kb), *va = (uint32_t *)(scratch + L.va),
             *vb = (uint32_t *)(scratch + L.vb), *start = (uint32_t *)(scratch + L.start);
    field_prep_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, means, cov6, opac, samples, split, nch, rec, ka, va);
    int in_b = 0;
    if (launch_test_sort32(ka, kb, va, vb, P, bits_for((uint64_t)nkeys), scratch + L.sort, scratch_bytes - L.sort, &in_b, st))
        return nullptr;
    const int nsort = 3 * ((bits_for((uint64_t)nkeys) + 8) / 9);
    field_gather_kernel<<<(P + 1 + 255) / 256, 256, 0, st>>>(P, (uint32_t)nkeys, in_b ? kb : ka, in_b ? vb : va, rec, sorted, start);
    *n_launches += 2 + nsort;
    return in_b ? vb : va;
}

template <int DEG>
void launch_query(int n, int res, int split, int nch, const float *samples, float relax, const char *scratch, const FieldLayout &L,
                  const uint32_t *pkeys, const uint32_t *porder, const float *points, float *density, float *normals, float *colors,
                  cudaStream_t st)
{
    constexpr size_t smem = query_smem_bytes(DEG);
    if (smem > 48 * 1024) cudaFuncSetAttribute(field_query_kernel<DEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    field_query_kernel<DEG><<<(unsigned)(((int64_t)n + QUERY_THREADS - 1) / QUERY_THREADS), QUERY_THREADS, smem, st>>>(
        n, res, split, nch, samples, relax, (const MeshRec *)(scratch + L.sorted), (const float *)(scratch + L.sh),
        (const uint32_t *)(scratch + L.start), pkeys, porder, points, density, normals, colors);
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
    if (!sort_gaussians(P, means, cov6, opac, split, nch, nkeys, samples, L, scratch, scratch_bytes, st, n_launches)) return -2;
    const int64_t vox = (int64_t)split * split * split;
    const int groups = (int)((vox + FIELD_VOX - 1) / FIELD_VOX);
    field_kernel<<<(unsigned)(nkeys * groups), FIELD_THREADS, 0, st>>>(res, split, nch, groups, samples, relax,
                                                                      (const MeshRec *)(scratch + L.sorted),
                                                                      (const uint32_t *)(scratch + L.start), field);
    *n_launches += 1;
    return 0;
}

size_t field_query_scratch_bytes(int P, int n_points, int res, int split, int sh_degree)
{
    const int64_t nch = (res + split - 1) / split;
    return FieldLayout(P, nch * nch * nch, n_points, sh_degree >= 0 ? 3 * query_coeffs(sh_degree) : 0).total;
}

int launch_field_query(int P, const float *means, const float *cov6, const float *opac, const float *shs, int sh_coeffs, int sh_degree,
                       int res, int split, const float *samples, float relax, int n_points, const float *points, float *density,
                       float *normals, float *colors, char *scratch, size_t scratch_bytes, cudaStream_t st, int *n_launches)
{
    const int nch = (res + split - 1) / split;
    const int64_t nkeys = (int64_t)nch * nch * nch;
    const int deg = colors && shs ? sh_degree : -1;
    const int k3 = deg >= 0 ? 3 * query_coeffs(deg) : 0;
    const FieldLayout L(P, nkeys, n_points, k3);
    if (scratch_bytes < L.total) return -1;
    const uint32_t *order = sort_gaussians(P, means, cov6, opac, split, nch, nkeys, samples, L, scratch, scratch_bytes, st, n_launches);
    if (!order) return -2;
    if (k3) {
        query_gather_sh_kernel<<<(unsigned)(((int64_t)P * k3 + 255) / 256), 256, 0, st>>>(P, k3, 3 * sh_coeffs, order, shs,
                                                                                           (float *)(scratch + L.sh));
        *n_launches += 1;
    }
    uint32_t *pka = (uint32_t *)(scratch + L.pka), *pkb = (uint32_t *)(scratch + L.pkb), *pva = (uint32_t *)(scratch + L.pva),
             *pvb = (uint32_t *)(scratch + L.pvb);
    query_prep_kernel<<<(unsigned)(((int64_t)n_points + 255) / 256), 256, 0, st>>>(n_points, points, samples, split, nch, pka, pva);
    int in_b = 0;
    if (launch_test_sort32(pka, pkb, pva, pvb, n_points, bits_for((uint64_t)nkeys), scratch + L.sort, scratch_bytes - L.sort, &in_b, st))
        return -2;
    const uint32_t *pkeys = in_b ? pkb : pka, *porder = in_b ? pvb : pva;
    switch (deg) {
    case -1: launch_query<-1>(n_points, res, split, nch, samples, relax, scratch, L, pkeys, porder, points, density, normals, nullptr, st); break;
    case 0: launch_query<0>(n_points, res, split, nch, samples, relax, scratch, L, pkeys, porder, points, density, normals, colors, st); break;
    case 1: launch_query<1>(n_points, res, split, nch, samples, relax, scratch, L, pkeys, porder, points, density, normals, colors, st); break;
    case 2: launch_query<2>(n_points, res, split, nch, samples, relax, scratch, L, pkeys, porder, points, density, normals, colors, st); break;
    default: launch_query<3>(n_points, res, split, nch, samples, relax, scratch, L, pkeys, porder, points, density, normals, colors, st); break;
    }
    *n_launches += 2 + 3 * ((bits_for((uint64_t)nkeys) + 8) / 9);
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
