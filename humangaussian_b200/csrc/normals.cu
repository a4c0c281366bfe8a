// normals.cu -- per-(view, Gaussian) normals of the normal map (DESIGN.md section 2, "Normal maps") and the chain of their
// gradient to the rotations.  The blend kernels (blend.cu, the NRM instantiations) read gauss_normals; nothing here touches
// the preprocess kernels, whose instantiations are unchanged.
//   normal_prep_kernel  one thread per Gaussian: k = argmin of the activated scales (lowest index on a tie), n = column k of
//                       R(q) (gs_rotmat, the covariance's own sequence), then per view the sign that makes n face the camera;
//                       writes gauss_normals[v*P + i] = (sign n, sign)
//   normal_bwd_kernel   one thread per Gaussian, after the preprocess backward: g = sum over the views with radii > 0, in
//                       view order, of sign * Wn (Wn = dL/dn, the blend's sums of w * dL/dN), then dL/dq of column k of R(q)
//                       (and the normalise Jacobian for raw parameters), ADDED to dL_drots
#include "common.cuh"
#include "kernels.h"

// the rotation and the axis as F1 holds them: q after the in-kernel normalise (raw), k from the activated scales before
// scale_modifier and the 3D filter (both leave the argmin unchanged in exact arithmetic; this pins the float ties).
// Returns max(||q||, 1e-12), the normalise's divisor (1 for post-activation inputs); *qlen gets ||q|| itself.
__device__ __forceinline__ float normal_axis(const NormalArgs &a, int i, float *q, int *k, float *qlen = nullptr)
{
    float s[3];
#pragma unroll
    for (int c = 0; c < 3; c++) s[c] = __ldg(a.scales + 3 * (size_t)i + c);
#pragma unroll
    for (int c = 0; c < 4; c++) q[c] = __ldg(a.rots + 4 * (size_t)i + c);
    float qn = 1.0f;
    if (a.raw) {
        s[0] = expf(s[0]); s[1] = expf(s[1]); s[2] = expf(s[2]);
        qn = gs_normalize4(q, qlen); // torch's F.normalize in float32, as F1 applies it
    }
    // strict comparisons: the lowest index wins a tie
    int kk = 0;
    if (s[1] < s[kk]) kk = 1;
    if (s[2] < s[kk]) kk = 2;
    *k = kk;
    return qn;
}

__global__ void __launch_bounds__(256) normal_prep_kernel(const NormalArgs a, float4 *__restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    float q[4], R[3][3];
    int k;
    normal_axis(a, i, q, &k);
    gs_rotmat(q, R);
    // (selects, not a dynamic index: R stays in registers)
    const float n0 = k == 0 ? R[0][0] : (k == 1 ? R[0][1] : R[0][2]);
    const float n1 = k == 0 ? R[1][0] : (k == 1 ? R[1][1] : R[1][2]);
    const float n2 = k == 0 ? R[2][0] : (k == 1 ? R[2][1] : R[2][2]);
    for (int v = 0; v < a.V; v++) {
        const float *m = a.means + (size_t)v * a.means_view_stride + 3 * (size_t)i;
        const float *cp = a.campos + 3 * v;
        // d = n . (campos - mean): fmul, ffma, ffma over the components 0, 1, 2 (gs_dot3); NaN keeps the sign
        const float d = gs_dot3(n0, n1, n2, fsub(cp[0], __ldg(m)), fsub(cp[1], __ldg(m + 1)), fsub(cp[2], __ldg(m + 2)));
        const float sg = d < 0.0f ? -1.0f : 1.0f;
        out[(size_t)v * a.P + i] = make_float4(sg * n0, sg * n1, sg * n2, sg);
    }
}

// dL/dq of column k of R(q) for the column gradient g (R as gs_rotmat, q = (r, x, y, z))
__device__ __forceinline__ float4 dcol_dq(int k, const float *q, float g0, float g1, float g2)
{
    const float r = q[0], x = q[1], y = q[2], z = q[3];
    if (k == 0) // (1 - 2(y^2 + z^2), 2(xy + rz), 2(xz - ry))
        return make_float4(2.f * (z * g1 - y * g2), 2.f * (y * g1 + z * g2), -4.f * y * g0 + 2.f * (x * g1 - r * g2),
                           -4.f * z * g0 + 2.f * (r * g1 + x * g2));
    if (k == 1) // (2(xy - rz), 1 - 2(x^2 + z^2), 2(yz + rx))
        return make_float4(2.f * (x * g2 - z * g0), 2.f * (y * g0 + r * g2) - 4.f * x * g1, 2.f * (x * g0 + z * g2),
                           2.f * (y * g2 - r * g0) - 4.f * z * g1);
    // (2(xz + ry), 2(yz - rx), 1 - 2(x^2 + y^2))
    return make_float4(2.f * (y * g0 - x * g1), 2.f * (z * g0 - r * g1) - 4.f * x * g2, 2.f * (r * g0 + z * g1) - 4.f * y * g2,
                       2.f * (x * g0 + y * g1));
}

__global__ void __launch_bounds__(256) normal_bwd_kernel(const NormalArgs a, const int32_t *__restrict__ radii,
                                                         const float4 *__restrict__ gauss_normals, const float4 *__restrict__ wn,
                                                         float *__restrict__ dL_drots)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
    bool any = false;
    for (int v = 0; v < a.V; v++) {
        const size_t vp = (size_t)v * a.P + i;
        if (!(radii[vp] > 0)) continue;
        const float sg = gauss_normals[vp].w;
        const float4 w = wn[vp];
        g0 += sg * w.x; g1 += sg * w.y; g2 += sg * w.z;
        any = true;
    }
    if (!any) return;
    float q[4];
    int k;
    float ql = 1.0f;
    const float qn = normal_axis(a, i, q, &k, &ql);
    float4 dq = dcol_dq(k, q, g0, g1, g2);
    if (a.raw) { // F.normalize's Jacobian, as the preprocess backward applies it (no projection below ||q|| = 1e-12)
        const float dot = ql >= 1e-12f ? q[0] * dq.x + q[1] * dq.y + q[2] * dq.z + q[3] * dq.w : 0.f;
        const float inv = 1.0f / qn;
        dq.x = (dq.x - q[0] * dot) * inv; dq.y = (dq.y - q[1] * dot) * inv; dq.z = (dq.z - q[2] * dot) * inv;
        dq.w = (dq.w - q[3] * dot) * inv;
    }
    float *o = dL_drots + 4 * (size_t)i;
    o[0] += dq.x; o[1] += dq.y; o[2] += dq.z; o[3] += dq.w;
}

void launch_normal_prep(const NormalArgs &a, float4 *gauss_normals, cudaStream_t st)
{
    normal_prep_kernel<<<(unsigned)((a.P + 255) / 256), 256, 0, st>>>(a, gauss_normals);
}

void launch_normal_bwd(const NormalArgs &a, const int32_t *radii, const float4 *gauss_normals, const float4 *wn, float *dL_drots,
                       cudaStream_t st)
{
    normal_bwd_kernel<<<(unsigned)((a.P + 255) / 256), 256, 0, st>>>(a, radii, gauss_normals, wn, dL_drots);
}
