// filter3d.cu -- the 3D smoothing filter's per-Gaussian maximal sampling rate (DESIGN.md section 2).
// One thread per Gaussian reads its mean once and loops over the <= 64 cameras of the call; the camera rows are the same
// address for every thread of a warp (a broadcast load), tan(fov/2) rides in the kernel parameters.  F1's view transform
// (gs_affine) and focal lengths (gs_focal) are reused as they are, so "in view" and the depth match what F1 computes.
#include "common.cuh"
#include "kernels.h"

__global__ void __launch_bounds__(256) sampling_rate_kernel(RateArgs a)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    const float px = __ldg(a.means + 3 * (size_t)i), py = __ldg(a.means + 3 * (size_t)i + 1), pz = __ldg(a.means + 3 * (size_t)i + 2);
    const float limx = fmul(0.65f, (float)a.W), limy = fmul(0.65f, (float)a.H); // the image plus a 15 % margin per side
    float rate = a.max_rate[i];
    for (int v = 0; v < a.nviews; v++) {
        const float *V = a.view + 16 * v;
        const float tx = gs_affine(__ldg(V + 0), __ldg(V + 4), __ldg(V + 8), __ldg(V + 12), px, py, pz);
        const float ty = gs_affine(__ldg(V + 1), __ldg(V + 5), __ldg(V + 9), __ldg(V + 13), px, py, pz);
        const float tz = gs_affine(__ldg(V + 2), __ldg(V + 6), __ldg(V + 10), __ldg(V + 14), px, py, pz);
        if (!(tz > GS_NEAR_Z)) continue; // F1's near cull; a NaN position is out
        const float fx = gs_focal(a.W, a.tanfovx[v]), fy = gs_focal(a.H, a.tanfovy[v]);
        if (!(fabsf(fmul(fdiv(tx, tz), fx)) <= limx) || !(fabsf(fmul(fdiv(ty, tz), fy)) <= limy)) continue;
        rate = fmaxf(rate, fdiv(fmaxf(fx, fy), tz));
    }
    a.max_rate[i] = rate;
}

void launch_sampling_rate(const RateArgs &a, cudaStream_t st)
{
    sampling_rate_kernel<<<(a.P + 255) / 256, 256, 0, st>>>(a);
}
