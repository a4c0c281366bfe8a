// optim.cu -- the Adam step over the packed parameter buffer (the optimiser of gaussian_model.py:156-165, run on the
// flat layout rasterize_views_packed reads and whose gradient its backward writes).
//
// The reference holds six single-tensor groups in torch.optim.Adam(l, lr=0.0, eps=1e-15): xyz, f_dc, f_rest, opacity,
// scaling, rotation, each with its own lr.  In the packed buffer [xyz | scaling | rotation | opacity | sh] the SH field
// [P,K,3] interleaves f_dc (coefficient 0) and f_rest (coefficients 1..K-1) row by row, so the group of an element is
// picked per element from the field offsets; no tensor is unpacked.
//
// One thread per float4 of param / grad / exp_avg / exp_avg_sq: 4 arrays read, 3 written, 28 B per float, HBM-bound,
// no atomics (deterministic: replicas that all-reduced the same gradient stay bit-identical).  Every field starts on a
// 16-byte boundary, so a float4 never holds two fields; it may hold a field's tail and the alignment padding after it,
// and padding floats are written as exact zeros.
//
// The arithmetic is torch's _multi_tensor_adam (torch/optim/adam.py, non-capturable branch, amsgrad=False,
// weight_decay=0) with each foreach op's fp32 rounding stated explicitly; the op bodies follow ATen's functors:
//   _foreach_lerp_(m, g, w)         Lerp.h lerp():  |w| < 0.5 ? m + w*(g-m) : g - (g-m)*(1-w)   (contracted to one fma)
//   _foreach_mul_(v, beta2)         v * beta2
//   _foreach_addcmul_(v, g, g, c)   DeviceAddCmulCdiv.cuh: fma(c, g*g, v)
//   _foreach_sqrt / _foreach_div_(d, bc2_sqrt) / _foreach_add_(d, eps)   IEEE sqrt, IEEE div, add
//   _foreach_addcdiv_(p, m, d, s)   DeviceAddCmulCdiv.cuh: fma(s, m/d, p)
// The scalars (step_size per group = -(lr / (1 - beta1^t)), bias_correction2_sqrt = (1 - beta2^t)^0.5) are computed on
// the host in double and rounded to float, as torch does.
#include "common.cuh"
#include "kernels.h"

namespace {

constexpr int AB = 256; // threads per block, one float4 per thread

__device__ __forceinline__ float adam_elem(const AdamArgs &a, float step_size, float g, float &m, float &v, float p)
{
    const float w = a.one_minus_beta1;
    const float diff = __fsub_rn(g, m);
    m = a.lerp_small ? __fmaf_rn(w, diff, m) : __fmaf_rn(-diff, __fsub_rn(1.0f, w), g);
    v = __fmaf_rn(a.one_minus_beta2, __fmul_rn(g, g), __fmul_rn(v, a.beta2));
    const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), a.bias_correction2_sqrt), a.eps);
    return __fmaf_rn(step_size, __fdiv_rn(m, d), p);
}

__global__ void __launch_bounds__(AB) adam_packed_kernel(AdamArgs a, int64_t n4, float4 *__restrict__ params,
                                                         const float4 *__restrict__ grads, float4 *__restrict__ exp_avg,
                                                         float4 *__restrict__ exp_avg_sq)
{
    const int64_t q = (int64_t)blockIdx.x * AB + threadIdx.x;
    if (q >= n4) return;
    const int64_t e0 = q * 4;
    // field of this float4 (fields ascend in the buffer; a float4 before field 0 or past a field's end is padding)
    const int f = (e0 >= a.off[1]) + (e0 >= a.off[2]) + (e0 >= a.off[3]) + (e0 >= a.off[4]);
    const int64_t rel0 = e0 - a.off[f];
    const int64_t nf = a.numel[f];
    // SH field: column of the first element inside its [K,3] row; coefficient 0 (columns 0..2) is f_dc
    const int row = 3 * a.sh_coeffs;
    int col = 0;
    if (f == 4 && rel0 >= 0) col = (int)(rel0 % row);
    float pv[4], gv[4], mv[4], vv[4];
    const float4 P4 = params[q], G4 = grads[q], M4 = exp_avg[q], V4 = exp_avg_sq[q];
    pv[0] = P4.x; pv[1] = P4.y; pv[2] = P4.z; pv[3] = P4.w;
    gv[0] = G4.x; gv[1] = G4.y; gv[2] = G4.z; gv[3] = G4.w;
    mv[0] = M4.x; mv[1] = M4.y; mv[2] = M4.z; mv[3] = M4.w;
    vv[0] = V4.x; vv[1] = V4.y; vv[2] = V4.z; vv[3] = V4.w;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int64_t rel = rel0 + j;
        if (rel < 0 || rel >= nf) { // alignment padding between fields
            pv[j] = mv[j] = vv[j] = 0.0f;
            continue;
        }
        int grp = a.field_group[f];
        if (f == 4) {
            int c = col + j;
            if (c >= row) c -= row;
            grp = c < 3 ? ADAM_GROUP_F_DC : ADAM_GROUP_F_REST;
        }
        pv[j] = adam_elem(a, a.step_size[grp], gv[j], mv[j], vv[j], pv[j]);
    }
    params[q] = make_float4(pv[0], pv[1], pv[2], pv[3]);
    exp_avg[q] = make_float4(mv[0], mv[1], mv[2], mv[3]);
    exp_avg_sq[q] = make_float4(vv[0], vv[1], vv[2], vv[3]);
}

} // namespace

void launch_adam_packed(const AdamArgs &a, int64_t total, float *params, const float *grads, float *exp_avg, float *exp_avg_sq,
                        cudaStream_t st)
{
    const int64_t n4 = total / 4;
    const unsigned grid = (unsigned)((n4 + AB - 1) / AB);
    adam_packed_kernel<<<grid, AB, 0, st>>>(a, n4, reinterpret_cast<float4 *>(params), reinterpret_cast<const float4 *>(grads),
                                            reinterpret_cast<float4 *>(exp_avg), reinterpret_cast<float4 *>(exp_avg_sq));
}
