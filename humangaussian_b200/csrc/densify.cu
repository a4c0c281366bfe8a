// densify.cu -- the point-set surgery on the other side of backward (SURVEY.md 8f-2; reference
// gaussiansplatting/scene/gaussian_model.py:268-437, driven from threestudio/systems/GaussianDreamer.py:378-408).
//
// The reference runs ~30 small PyTorch ops per call: boolean-mask gathers, torch.cat of every parameter and both
// Adam moments (twice: clone, then split), then two more masked gathers (prune), each with its own implicit host
// sync.  Here the whole densify_and_prune is planned in one pass and every surviving row is moved exactly once:
//
//   stats   one thread per Gaussian folds a V-view batch: sum of the view-space gradients, max radius, then
//           accum += |sum.xy|, denom += 1, max_radii2D = max(...) where visible (GaussianDreamer.py:385-391 +
//           gaussian_model.py:433-437);
//   plan    per Gaussian: clone? split? survive the final opacity / size prune? (for itself and for its children) -- or, for
//           b200gs_prune_plan, survive a caller's removal mask (classify mode 2);
//           three kernels (block counts -> scan of block counts -> block-local ranks) turn the four flag streams
//           into FINAL destination rows, in the reference's output order
//              [surviving unsplit originals | surviving clones | surviving children copy 0 | ... copy N-1];
//   apply   one streaming kernel per array (parameter, Adam moment): row i is read once and written to its 0..1+N
//           destinations; the xyz and scaling arrays compute the split children in flight
//           (xyz' = R(q)(z * exp(s)) + xyz, s' = log(exp(s)/(0.8N))), Adam moments of new rows are zero.
// Everything is HBM-streaming work; nothing here is reshaped for tensor cores.
#include "common.cuh"
#include "kernels.h"

namespace {

constexpr int DB = 256; // threads per block, one Gaussian per thread

struct Flags { bool keep, clone, split_sel, split_kept; };

__device__ __forceinline__ Flags classify(const DensifyCfg &c, int i, const float *__restrict__ accum, const float *__restrict__ denom,
                                           const float *__restrict__ opacity, const float *__restrict__ scaling)
{
    Flags f;
    if (c.mode == 2) { // prune by a caller's mask (b200gs_prune_plan): survivors keep their order, nothing is added
        f.keep = c.remove[i] == 0;
        f.clone = f.split_sel = f.split_kept = false;
        return f;
    }
    const float e0 = expf(scaling[3 * i]), e1 = expf(scaling[3 * i + 1]), e2 = expf(scaling[3 * i + 2]);
    const float smax = fmaxf(e0, fmaxf(e1, e2));
    const bool low_op = gs_sigmoidf(opacity[i]) < c.min_opacity;
    if (c.mode == 1) { // prune_only (gaussian_model.py:423-430)
        f.keep = !(low_op || smax > c.big_ws_thresh);
        f.clone = f.split_sel = f.split_kept = false;
        return f;
    }
    float g = accum[i] / denom[i]; // 0/0 -> nan -> 0 (gaussian_model.py:403-404)
    if (isnan(g)) g = 0.0f;
    const bool want_clone = (fabsf(g) >= c.max_grad) && (smax <= c.dense_thresh);
    const bool want_split = (g >= c.max_grad) && (smax > c.dense_thresh);
    bool prune_self = low_op, prune_child = low_op;
    if (c.use_screen) {
        // max_radii2D was reset to zeros by densification_postfix before this test (gaussian_model.py:358-360,410)
        const bool big_vs = 0.0f > c.max_screen_size;
        const float k = 0.8f * (float)c.n_split;
        const float cmax = fmaxf(expf(logf(e0 / k)), fmaxf(expf(logf(e1 / k)), expf(logf(e2 / k))));
        prune_self = prune_self || big_vs || smax > c.big_ws_thresh;
        prune_child = prune_child || big_vs || cmax > c.big_ws_thresh;
    }
    f.keep = !want_split && !prune_self;
    f.clone = want_clone && !prune_self;
    f.split_sel = want_split;
    f.split_kept = want_split && !prune_child;
    return f;
}

// block-wide exclusive ranks of four flag streams (ballot + per-warp totals); returns block totals in tot[4]
__device__ __forceinline__ void block_ranks(const Flags &f, bool valid, int rank[4], int tot[4])
{
    __shared__ int s_w[4][DB / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t lt = (1u << lane) - 1u;
    const bool fl[4] = {valid && f.keep, valid && f.clone, valid && f.split_sel, valid && f.split_kept};
    uint32_t b[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        b[k] = __ballot_sync(0xffffffffu, fl[k]);
        if (lane == 0) s_w[k][warp] = __popc(b[k]);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; k++) {
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < DB / 32; w++) {
            const int c = s_w[k][w];
            before += (w < warp) ? c : 0;
            total += c;
        }
        rank[k] = before + __popc(b[k] & lt);
        tot[k] = total;
    }
}

__global__ void __launch_bounds__(DB) densify_count_kernel(DensifyCfg c, int P, const float *accum, const float *denom, const float *opacity,
                                                           const float *scaling, int *block_counts /*[4][nblocks]*/)
{
    const int i = blockIdx.x * DB + threadIdx.x;
    Flags f = {false, false, false, false};
    if (i < P) f = classify(c, i, accum, denom, opacity, scaling);
    int rank[4], tot[4];
    block_ranks(f, i < P, rank, tot);
    if (threadIdx.x < 4) block_counts[threadIdx.x * gridDim.x + blockIdx.x] = tot[threadIdx.x];
}

// one block: exclusive scan of the four block-count rows in place, totals to counts[0..3], new P to counts[4]
__global__ void __launch_bounds__(1024) densify_scan_kernel(int nblocks, int n_split, int *block_counts, int *counts)
{
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = 0; k < 4; k++) {
        int *row = block_counts + (size_t)k * nblocks;
        if (threadIdx.x == 0) s_carry = 0;
        __syncthreads();
        for (int base = 0; base < nblocks; base += 1024) {
            const int j = base + threadIdx.x;
            const int v = j < nblocks ? row[j] : 0;
            int x = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, x, d);
                if (lane >= d) x += y;
            }
            if (lane == 31) s_warp[warp] = x;
            __syncthreads();
            if (warp == 0) {
                int w = s_warp[lane];
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const int y = __shfl_up_sync(0xffffffffu, w, d);
                    if (lane >= d) w += y;
                }
                s_warp[lane] = w; // inclusive over warps
            }
            __syncthreads();
            const int incl = x + (warp ? s_warp[warp - 1] : 0) + s_carry;
            if (j < nblocks) row[j] = incl - v;
            __syncthreads();
            if (threadIdx.x == 1023) s_carry = incl;
            __syncthreads();
        }
        if (threadIdx.x == 0) counts[k] = s_carry;
        __syncthreads();
    }
    if (threadIdx.x == 0) counts[4] = counts[0] + counts[1] + n_split * counts[3];
}

__global__ void __launch_bounds__(DB) densify_plan_kernel(DensifyCfg c, int P, const float *accum, const float *denom, const float *opacity,
                                                          const float *scaling, const int *block_offsets, const int *counts,
                                                          int *plan /*[4][P]*/)
{
    const int i = blockIdx.x * DB + threadIdx.x;
    Flags f = {false, false, false, false};
    if (i < P) f = classify(c, i, accum, denom, opacity, scaling);
    int rank[4], tot[4];
    block_ranks(f, i < P, rank, tot);
    if (i >= P) return;
    const int n_keep = counts[0], n_clone = counts[1];
    const int o0 = block_offsets[blockIdx.x], o1 = block_offsets[gridDim.x + blockIdx.x], o2 = block_offsets[2 * gridDim.x + blockIdx.x],
              o3 = block_offsets[3 * gridDim.x + blockIdx.x];
    plan[i] = f.keep ? o0 + rank[0] : -1;
    plan[(size_t)P + i] = f.clone ? n_keep + o1 + rank[1] : -1;
    plan[2 * (size_t)P + i] = f.split_kept ? n_keep + n_clone + o3 + rank[3] : -1;
    plan[3 * (size_t)P + i] = f.split_sel ? o2 + rank[2] : -1; // row of the parent in the reference's noise block
}

__global__ void __launch_bounds__(DB) densify_stats_kernel(int P, int V, const float *__restrict__ grads /*[V,P,3]*/,
                                                           const int32_t *__restrict__ radii /*[V,P]*/, const uint8_t *__restrict__ update_mask /*[P] or null*/,
                                                           float *accum, float *denom, float *max_radii2D)
{
    const int i = blockIdx.x * DB + threadIdx.x;
    if (i >= P) return;
    float gx = 0.0f, gy = 0.0f;
    int rmax = 0;
    for (int v = 0; v < V; v++) {
        const float *g = grads + ((size_t)v * P + i) * 3;
        gx = __fadd_rn(gx, g[0]);
        gy = __fadd_rn(gy, g[1]);
        rmax = max(rmax, radii[(size_t)v * P + i]);
    }
    // visibility_filter = (max radius > 0) [& ~hand_mask when disable_hand_densification is set, GaussianDreamer.py:288-297]
    if (rmax > 0 && (!update_mask || update_mask[i])) {
        max_radii2D[i] = fmaxf(max_radii2D[i], (float)rmax);
        accum[i] = __fadd_rn(accum[i], __fsqrt_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy))));
        denom[i] = __fadd_rn(denom[i], 1.0f);
    }
}

// role: 0 copy (new rows repeat the source row), 1 xyz, 2 scaling, 3 optimizer moment (new rows zero)
template <int ROLE>
__global__ void __launch_bounds__(DB) densify_move_kernel(int P, int rf, const int *__restrict__ plan, const float *__restrict__ src,
                                                          float *__restrict__ dst, int n_split, int S_sel, int S_kept,
                                                          const float *__restrict__ rotation, const float *__restrict__ scaling,
                                                          const float *__restrict__ noise)
{
    const int64_t idx = (int64_t)blockIdx.x * DB + threadIdx.x;
    if (idx >= (int64_t)P * rf) return;
    const int i = (int)(idx / rf), e = (int)(idx - (int64_t)i * rf);
    const float v = src[idx];
    const int d0 = plan[i], d1 = plan[(size_t)P + i], d2 = plan[2 * (size_t)P + i];
    if (d0 >= 0) dst[(size_t)d0 * rf + e] = v;
    if (d1 >= 0) dst[(size_t)d1 * rf + e] = (ROLE == 3) ? 0.0f : v;
    if (d2 >= 0) {
        if (ROLE == 0 || ROLE == 3) {
            for (int c = 0; c < n_split; c++) dst[((size_t)d2 + (size_t)c * S_kept) * rf + e] = (ROLE == 3) ? 0.0f : v;
        } else if (ROLE == 2) {
            const float nv = logf(expf(v) / (0.8f * (float)n_split)); // gaussian_model.py:374
            for (int c = 0; c < n_split; c++) dst[((size_t)d2 + (size_t)c * S_kept) * rf + e] = nv;
        } else {
            // row e of build_rotation(q) (general_utils.py:78-99), applied to z * exp(s) (gaussian_model.py:369-373)
            const float qr = rotation[4 * i], qx = rotation[4 * i + 1], qy = rotation[4 * i + 2], qz = rotation[4 * i + 3];
            const float n = sqrtf(qr * qr + qx * qx + qy * qy + qz * qz);
            const float r = qr / n, x = qx / n, y = qy / n, z = qz / n;
            float R0, R1, R2;
            if (e == 0) { R0 = 1.0f - 2.0f * (y * y + z * z); R1 = 2.0f * (x * y - r * z); R2 = 2.0f * (x * z + r * y); }
            else if (e == 1) { R0 = 2.0f * (x * y + r * z); R1 = 1.0f - 2.0f * (x * x + z * z); R2 = 2.0f * (y * z - r * x); }
            else { R0 = 2.0f * (x * z - r * y); R1 = 2.0f * (y * z + r * x); R2 = 1.0f - 2.0f * (x * x + y * y); }
            const float s0 = expf(scaling[3 * i]), s1 = expf(scaling[3 * i + 1]), s2 = expf(scaling[3 * i + 2]);
            const int nr = plan[3 * (size_t)P + i];
            for (int c = 0; c < n_split; c++) {
                const float *zz = noise + ((size_t)c * S_sel + nr) * 3;
                const float a0 = zz[0] * s0, a1 = zz[1] * s1, a2 = zz[2] * s2;
                dst[((size_t)d2 + (size_t)c * S_kept) * rf + e] = fmaf(R2, a2, fmaf(R1, a1, R0 * a0)) + v;
            }
        }
    }
}

} // namespace

size_t densify_scratch_bytes(int P) { return (size_t)4 * ((P + DB - 1) / DB + 1) * sizeof(int); }

void launch_densify_stats(int P, int V, const float *grads, const int32_t *radii, const uint8_t *update_mask, float *accum, float *denom,
                          float *max_radii2D, cudaStream_t st)
{
    densify_stats_kernel<<<(P + DB - 1) / DB, DB, 0, st>>>(P, V, grads, radii, update_mask, accum, denom, max_radii2D);
}

void launch_densify_plan(const DensifyCfg &c, int P, const float *accum, const float *denom, const float *opacity, const float *scaling,
                         int *plan, int *counts, char *scratch, cudaStream_t st)
{
    const int nb = (P + DB - 1) / DB;
    int *block_counts = reinterpret_cast<int *>(scratch);
    densify_count_kernel<<<nb, DB, 0, st>>>(c, P, accum, denom, opacity, scaling, block_counts);
    densify_scan_kernel<<<1, 1024, 0, st>>>(nb, c.n_split, block_counts, counts);
    densify_plan_kernel<<<nb, DB, 0, st>>>(c, P, accum, denom, opacity, scaling, block_counts, counts, plan);
}

void launch_densify_move(int role, int P, int rf, const int *plan, const float *src, float *dst, int n_split, int S_sel, int S_kept,
                         const float *rotation, const float *scaling, const float *noise, cudaStream_t st)
{
    const int64_t n = (int64_t)P * rf;
    const unsigned grid = (unsigned)((n + DB - 1) / DB);
    switch (role) {
    case 0: densify_move_kernel<0><<<grid, DB, 0, st>>>(P, rf, plan, src, dst, n_split, S_sel, S_kept, rotation, scaling, noise); break;
    case 1: densify_move_kernel<1><<<grid, DB, 0, st>>>(P, rf, plan, src, dst, n_split, S_sel, S_kept, rotation, scaling, noise); break;
    case 2: densify_move_kernel<2><<<grid, DB, 0, st>>>(P, rf, plan, src, dst, n_split, S_sel, S_kept, rotation, scaling, noise); break;
    default: densify_move_kernel<3><<<grid, DB, 0, st>>>(P, rf, plan, src, dst, n_split, S_sel, S_kept, rotation, scaling, noise); break;
    }
}
