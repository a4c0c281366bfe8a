// classic_blend.cu -- COMPARATOR, not product.  The blend kernels of the classic 3DGS tile rasteriser
// structure (SURVEY.md 2.2 rows F6 / B1, "reference-algorithm restatement"): one thread per pixel of a
// 16x16 tile, every thread walks the whole tile list, colours fetched from global memory by Gaussian id,
// and -- in backward -- ten float atomicAdds per contributing (pixel, Gaussian) pair.  The real reference
// (ashawkey/diff-gaussian-rasterization) is not vendored and cannot be installed here (no network), so the
// ">= 5x the reference CUDA rasteriser" target of BASELINE.json is measured against this restatement of its
// structure, recompiled for sm_90a exactly as the reference's setup.py would be (no Hopper-specific features).
// It links against the same preprocess / binning / C-ABI sources as the product (baseline/Makefile), so it is
// called through the identical host path; only the two hot kernels differ.
#include "../humangaussian_b200/csrc/common.cuh"
#include "../humangaussian_b200/csrc/kernels.h"

#define BLOCK_SIZE 256

__global__ void __launch_bounds__(BLOCK_SIZE) classic_fwd(BlendArgs a)
{
    __shared__ uint32_t c_id[BLOCK_SIZE];
    __shared__ float2 c_xy[BLOCK_SIZE];
    __shared__ float4 c_co[BLOCK_SIZE];
    const int ntiles = a.grid_x * a.grid_y;
    const int tile = blockIdx.x, v = blockIdx.y;
    const int px = (tile % a.grid_x) * GS_TILE + threadIdx.x % GS_TILE;
    const int py = (tile / a.grid_x) * GS_TILE + threadIdx.x / GS_TILE;
    const bool inside = px < a.W && py < a.H;
    const float2 pixf = make_float2((float)px, (float)py);
    const uint2 range = a.ranges[(size_t)v * ntiles + tile];
    const int rounds = ((range.y - range.x + BLOCK_SIZE - 1) / BLOCK_SIZE);
    int toDo = range.y - range.x;
    bool done = !inside;
    float T = 1.0f, C[3] = {0, 0, 0}, weight = 0.f, Dd = 0.f;
    uint32_t contributor = 0, last_contributor = 0;
    for (int i = 0; i < rounds; i++, toDo -= BLOCK_SIZE) {
        if (__syncthreads_count(done) == BLOCK_SIZE) break;
        const int progress = i * BLOCK_SIZE + threadIdx.x;
        if (range.x + progress < range.y) {
            const uint32_t id = a.point_list[range.x + progress];
            c_id[threadIdx.x] = id;
            c_xy[threadIdx.x] = make_float2(a.recs[id].px, a.recs[id].py);
            c_co[threadIdx.x] = make_float4(a.recs[id].A, a.recs[id].B, a.recs[id].C, a.recs[id].o);
        }
        __syncthreads();
        for (int j = 0; !done && j < min(BLOCK_SIZE, toDo); j++) {
            contributor++;
            const float2 xy = c_xy[j];
            const float2 d = {xy.x - pixf.x, xy.y - pixf.y};
            const float4 co = c_co[j];
            const float power = -0.5f * (co.x * d.x * d.x + co.z * d.y * d.y) - co.y * d.x * d.y;
            if (power > 0.0f) continue;
            const float alpha = min(0.99f, co.w * expf(power));
            if (alpha < 1.0f / 255.0f) continue;
            const float test_T = T * (1 - alpha);
            if (test_T < 0.0001f) { done = true; continue; }
            const GeomRec *g = a.recs + c_id[j];
            C[0] += g->r * alpha * T; C[1] += g->g * alpha * T; C[2] += g->b * alpha * T;
            weight += alpha * T;
            Dd += g->depth * alpha * T;
            T = test_T;
            last_contributor = contributor;
        }
    }
    if (inside) {
        const size_t HW = (size_t)a.H * a.W, pix = (size_t)py * a.W + px;
        a.final_T[v * HW + pix] = T;
        a.n_contrib[v * HW + pix] = last_contributor;
        for (int ch = 0; ch < 3; ch++) a.out_color[(size_t)v * 3 * HW + ch * HW + pix] = C[ch] + T * a.bg[ch];
        a.out_alpha[v * HW + pix] = weight;
        a.out_depth[v * HW + pix] = Dd;
    }
}

__global__ void __launch_bounds__(BLOCK_SIZE) classic_bwd(BlendBwdArgs a)
{
    __shared__ uint32_t c_id[BLOCK_SIZE];
    __shared__ float2 c_xy[BLOCK_SIZE];
    __shared__ float4 c_co[BLOCK_SIZE];
    __shared__ float c_col[3 * BLOCK_SIZE];
    __shared__ float c_dep[BLOCK_SIZE];
    const int ntiles = a.grid_x * a.grid_y;
    const int tile = blockIdx.x, v = blockIdx.y;
    const int px = (tile % a.grid_x) * GS_TILE + threadIdx.x % GS_TILE;
    const int py = (tile / a.grid_x) * GS_TILE + threadIdx.x / GS_TILE;
    const bool inside = px < a.W && py < a.H;
    const float2 pixf = make_float2((float)px, (float)py);
    const size_t HW = (size_t)a.H * a.W, pix = (size_t)py * a.W + px;
    const uint2 range = a.ranges[(size_t)v * ntiles + tile];
    const int rounds = ((range.y - range.x + BLOCK_SIZE - 1) / BLOCK_SIZE);
    bool done = !inside;
    int toDo = range.y - range.x;
    const float T_final = inside ? a.final_T[v * HW + pix] : 0;
    float T = T_final;
    uint32_t contributor = toDo;
    const int last_contributor = inside ? a.n_contrib[v * HW + pix] : 0;
    float accum_rec[3] = {0, 0, 0}, dL_dpixel[3] = {0, 0, 0}, accum_depth_rec = 0, accum_alpha_rec = 0, dL_ddepth = 0, dL_dalpha_pix = 0;
    if (inside) {
        if (a.dL_dcolor) for (int ch = 0; ch < 3; ch++) dL_dpixel[ch] = a.dL_dcolor[(size_t)v * 3 * HW + ch * HW + pix];
        if (a.dL_ddepth) dL_ddepth = a.dL_ddepth[v * HW + pix];
        if (a.dL_dalpha) dL_dalpha_pix = a.dL_dalpha[v * HW + pix];
    }
    float last_alpha = 0, last_color[3] = {0, 0, 0}, last_depth = 0;
    const float ddelx_dx = 0.5f * a.W, ddely_dy = 0.5f * a.H;
    for (int i = 0; i < rounds; i++, toDo -= BLOCK_SIZE) {
        __syncthreads();
        const int progress = i * BLOCK_SIZE + threadIdx.x;
        if (range.x + progress < range.y) {
            const uint32_t id = a.point_list[range.y - progress - 1];
            c_id[threadIdx.x] = id;
            c_xy[threadIdx.x] = make_float2(a.recs[id].px, a.recs[id].py);
            c_co[threadIdx.x] = make_float4(a.recs[id].A, a.recs[id].B, a.recs[id].C, a.recs[id].o);
            c_col[threadIdx.x] = a.recs[id].r; c_col[BLOCK_SIZE + threadIdx.x] = a.recs[id].g; c_col[2 * BLOCK_SIZE + threadIdx.x] = a.recs[id].b;
            c_dep[threadIdx.x] = a.recs[id].depth;
        }
        __syncthreads();
        for (int j = 0; !done && j < min(BLOCK_SIZE, toDo); j++) {
            contributor--;
            if (contributor >= (uint32_t)last_contributor) continue;
            const float2 xy = c_xy[j];
            const float2 d = {xy.x - pixf.x, xy.y - pixf.y};
            const float4 co = c_co[j];
            const float power = -0.5f * (co.x * d.x * d.x + co.z * d.y * d.y) - co.y * d.x * d.y;
            if (power > 0.0f) continue;
            const float G = expf(power);
            const float alpha = min(0.99f, co.w * G);
            if (alpha < 1.0f / 255.0f) continue;
            T = T / (1.f - alpha);
            const float dchannel_dcolor = alpha * T;
            float dL_dopa = 0.0f;
            const uint32_t gid = c_id[j];
            float *sg = reinterpret_cast<float *>(reinterpret_cast<ScreenGrad *>(a.sgrad) + gid);
            for (int ch = 0; ch < 3; ch++) {
                const float c = c_col[ch * BLOCK_SIZE + j];
                accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch];
                last_color[ch] = c;
                dL_dopa += (c - accum_rec[ch]) * dL_dpixel[ch];
                atomicAdd(sg + 6 + ch, dchannel_dcolor * dL_dpixel[ch]);
            }
            const float c_d = c_dep[j];
            accum_depth_rec = last_alpha * last_depth + (1.f - last_alpha) * accum_depth_rec;
            last_depth = c_d;
            dL_dopa += (c_d - accum_depth_rec) * dL_ddepth;
            atomicAdd(sg + 9, dchannel_dcolor * dL_ddepth);
            accum_alpha_rec = last_alpha + (1.f - last_alpha) * accum_alpha_rec;
            dL_dopa += (1 - accum_alpha_rec) * dL_dalpha_pix;
            dL_dopa *= T;
            last_alpha = alpha;
            float bg_dot_dpixel = 0;
            for (int ch = 0; ch < 3; ch++) bg_dot_dpixel += a.bg[ch] * dL_dpixel[ch];
            dL_dopa += (-T_final / (1.f - alpha)) * bg_dot_dpixel;
            const float dL_dG = co.w * dL_dopa;
            const float gdx = G * d.x, gdy = G * d.y;
            const float dG_ddelx = -gdx * co.x - gdy * co.y, dG_ddely = -gdy * co.z - gdx * co.y;
            atomicAdd(sg + 0, dL_dG * dG_ddelx * ddelx_dx);
            atomicAdd(sg + 1, dL_dG * dG_ddely * ddely_dy);
            atomicAdd(sg + 2, -0.5f * gdx * d.x * dL_dG);
            atomicAdd(sg + 3, -0.5f * gdx * d.y * dL_dG);
            atomicAdd(sg + 4, -0.5f * gdy * d.y * dL_dG);
            atomicAdd(sg + 5, G * dL_dopa);
        }
    }
}

void launch_blend_fwd(const BlendArgs &a, cudaStream_t st)
{
    dim3 grid(a.grid_x * a.grid_y, a.V);
    classic_fwd<<<grid, BLOCK_SIZE, 0, st>>>(a);
}
void launch_blend_bwd(const BlendBwdArgs &a, cudaStream_t st)
{
    dim3 grid(a.grid_x * a.grid_y, a.V);
    classic_bwd<<<grid, BLOCK_SIZE, 0, st>>>(a);
}
int blend_sgrad_is_moments() { return 0; }
// no deterministic backward here: b200gs_backward_deterministic returns B200GS_E_UNSUPPORTED before it would launch this
int blend_bwd_has_deterministic() { return 0; }
void launch_blend_bwd_det(const BlendBwdArgs &, const DetFlush &, cudaStream_t) {}
__global__ void classic_exp_kernel(const float *x, float *y, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = expf(x[i]);
}
void launch_test_exp(const float *x, float *y, int64_t n, cudaStream_t st)
{
    classic_exp_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, y, n);
}
