// mcmc.cu -- MCMC densification (3DGS-MCMC, Kheradmand et al., NeurIPS 2024; DESIGN.md section 2, "MCMC densification")
// on the raw optimiser parameters, the alternative to densify.cu's gradient-threshold rule:
//
//   noise  one thread per Gaussian, every step after the optimiser step: xyz += noise_scale * sigmoid(-k (o - t)) * Sigma eta,
//          Sigma = R(q^) diag(exp(2 s)) R(q^)^T, o = sigmoid(opacity).  The per-step hot path: one launch, no host sync.
//   ratio  one thread per row with c = counts[row] > 0 (row drawn c times as a source): the opacity and scales that n = min(c+1,
//          51) members (the row and its c copies) take so that together they show what the row showed, in float64, rounded once.
//   move   one launch per array: dst[i] = src[map[i]] for the P_new destination rows, where map is the identity except at the
//          relocated rows (relocate) or identity ++ samples (grow).  A row is reset when its source was drawn
//          (counts[map[i]] > 0): its opacity and scales take the ratio's values and its Adam moments are zero.
// Sampling (torch.multinomial) and the counts stay in torch; nothing here reads back to the host.
#include "../../include/b200gs.h"
#include "common.cuh"
#include "kernels.h"

namespace {

constexpr int MB = 256;       // threads per block
constexpr int MCMC_N_MAX = 51; // the split ratio saturates at 51 members

__global__ void __launch_bounds__(MB) mcmc_noise_kernel(int P, float *__restrict__ xyz, const float *__restrict__ scaling,
                                                        const float *__restrict__ rotation, const float *__restrict__ opacity,
                                                        const float *__restrict__ eta, float noise_scale, float k, float t)
{
    const int i = blockIdx.x * MB + threadIdx.x;
    if (i >= P) return;
    float q[4];
#pragma unroll
    for (int c = 0; c < 4; c++) q[c] = rotation[4 * (size_t)i + c];
    gs_normalize4(q); // q^ as F1 forms it for raw parameters
    float R[3][3];
    gs_rotmat(q, R);
    const float o = gs_sigmoidf(opacity[i]);
    // -k (o - t) as one fma: the argument reaches ~100, so a second rounding would cost ~6e-6 of the gate
    const float gate = gs_sigmoidf(ffma(-k, o, fmul(k, t)));
    const float e0 = eta[3 * (size_t)i], e1 = eta[3 * (size_t)i + 1], e2 = eta[3 * (size_t)i + 2];
    // Sigma eta = R (diag(exp(2 s)) (R^T eta))
    float u[3];
#pragma unroll
    for (int j = 0; j < 3; j++) u[j] = (R[0][j] * e0 + R[1][j] * e1 + R[2][j] * e2) * expf(2.0f * scaling[3 * (size_t)i + j]);
    const float f = noise_scale * gate;
#pragma unroll
    for (int r = 0; r < 3; r++) xyz[3 * (size_t)i + r] += f * (R[r][0] * u[0] + R[r][1] * u[1] + R[r][2] * u[2]);
}

__global__ void __launch_bounds__(MB) mcmc_ratio_kernel(int P, const int *__restrict__ counts, const float *__restrict__ opacity,
                                                        const float *__restrict__ scaling, float *__restrict__ new_opacity,
                                                        float *__restrict__ new_scaling)
{
    const int i = blockIdx.x * MB + threadIdx.x;
    if (i >= P) return;
    const int c = counts[i];
    if (c <= 0) return;
    const int n = min(c, MCMC_N_MAX - 1) + 1;
    const double o = (double)gs_sigmoidf(opacity[i]);
    // o' = 1 - (1 - o)^(1/n), written without the cancellation of 1 - pow for small o
    const double op = fmin(fmax(-expm1(log1p(-o) / n), 0.005), 1.0 - 0x1p-23);
    // D = sum_{k<n} C(n, k+1) (-1)^k o'^(k+1) / sqrt(k+1): terms reach ~4e3 D, hence float64 throughout
    double D = 0.0, binom = 1.0, pw = 1.0, sign = 1.0;
    for (int kk = 0; kk < n; kk++) {
        binom = binom * (double)(n - kk) / (double)(kk + 1); // C(n, kk+1)
        pw *= op;
        D += sign * binom * pw / sqrt((double)(kk + 1));
        sign = -sign;
    }
    new_opacity[i] = (float)log(op / (1.0 - op));
    const double f = o / D;
#pragma unroll
    for (int j = 0; j < 3; j++) new_scaling[3 * (size_t)i + j] = (float)log(exp((double)scaling[3 * (size_t)i + j]) * f);
}

template <int ROLE>
__global__ void __launch_bounds__(MB) mcmc_move_kernel(int64_t n, int rf, const int *__restrict__ map, const int *__restrict__ counts,
                                                       const float *__restrict__ src, float *__restrict__ dst,
                                                       const float *__restrict__ new_opacity, const float *__restrict__ new_scaling)
{
    const int64_t idx = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (idx >= n) return;
    const int i = (int)(idx / rf), e = (int)(idx - (int64_t)i * rf);
    const int s = map[i];
    const float v = src[(size_t)s * rf + e];
    if (ROLE == B200GS_MCMC_ROLE_COPY) {
        dst[idx] = v;
        return;
    }
    const bool reset = counts[s] > 0;
    if (ROLE == B200GS_MCMC_ROLE_OPACITY) dst[idx] = reset ? new_opacity[s] : v;
    else if (ROLE == B200GS_MCMC_ROLE_SCALING) dst[idx] = reset ? new_scaling[3 * (size_t)s + e] : v;
    else dst[idx] = reset ? 0.0f : v;
}

} // namespace

void launch_mcmc_noise(int P, float *xyz, const float *scaling, const float *rotation, const float *opacity, const float *eta,
                       float noise_scale, float k, float t, cudaStream_t st)
{
    mcmc_noise_kernel<<<(P + MB - 1) / MB, MB, 0, st>>>(P, xyz, scaling, rotation, opacity, eta, noise_scale, k, t);
}

void launch_mcmc_ratio(int P, const int *counts, const float *opacity, const float *scaling, float *new_opacity, float *new_scaling,
                       cudaStream_t st)
{
    mcmc_ratio_kernel<<<(P + MB - 1) / MB, MB, 0, st>>>(P, counts, opacity, scaling, new_opacity, new_scaling);
}

void launch_mcmc_move(int role, int P_new, int rf, const int *map, const int *counts, const float *src, float *dst,
                      const float *new_opacity, const float *new_scaling, cudaStream_t st)
{
    const int64_t n = (int64_t)P_new * rf;
    const unsigned grid = (unsigned)((n + MB - 1) / MB);
    switch (role) {
    case B200GS_MCMC_ROLE_COPY:
        mcmc_move_kernel<B200GS_MCMC_ROLE_COPY><<<grid, MB, 0, st>>>(n, rf, map, counts, src, dst, new_opacity, new_scaling); break;
    case B200GS_MCMC_ROLE_OPACITY:
        mcmc_move_kernel<B200GS_MCMC_ROLE_OPACITY><<<grid, MB, 0, st>>>(n, rf, map, counts, src, dst, new_opacity, new_scaling); break;
    case B200GS_MCMC_ROLE_SCALING:
        mcmc_move_kernel<B200GS_MCMC_ROLE_SCALING><<<grid, MB, 0, st>>>(n, rf, map, counts, src, dst, new_opacity, new_scaling); break;
    default:
        mcmc_move_kernel<B200GS_MCMC_ROLE_MOMENT><<<grid, MB, 0, st>>>(n, rf, map, counts, src, dst, new_opacity, new_scaling); break;
    }
}
