// sh.cuh -- the real spherical-harmonics basis of the colour model (gaussiansplatting/utils/sh_utils.py:57-112), shared by
// the render preprocess (preprocess.cu) and the mesh colour query (mesh.cu) so both evaluate the same constants in the
// same order.  Needs common.cuh.
#pragma once

static __constant__ float c_SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                        -1.0925484305920792f, 0.5462742152960396f};
static __constant__ float c_SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                        0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                        -0.5900435899266435f};
#define SH_C0 0.28209479177387814f
#define SH_C1 0.4886025119029199f

// 16 real-SH basis values, signs folded in (sh_utils.py:74-100)
__device__ __forceinline__ void sh_basis(int deg, float x, float y, float z, float *b)
{
    b[0] = SH_C0;
    if (deg > 0) {
        b[1] = fmul(-SH_C1, y);
        b[2] = fmul(SH_C1, z);
        b[3] = fmul(-SH_C1, x);
        if (deg > 1) {
            const float xx = fmul(x, x), yy = fmul(y, y), zz = fmul(z, z);
            const float xy = fmul(x, y), yz = fmul(y, z), xz = fmul(x, z);
            b[4] = fmul(c_SH_C2[0], xy);
            b[5] = fmul(c_SH_C2[1], yz);
            b[6] = fmul(c_SH_C2[2], fsub(fsub(fmul(2.0f, zz), xx), yy));
            b[7] = fmul(c_SH_C2[3], xz);
            b[8] = fmul(c_SH_C2[4], fsub(xx, yy));
            if (deg > 2) {
                b[9] = fmul(fmul(c_SH_C3[0], y), ffma(3.0f, xx, -yy));
                b[10] = fmul(fmul(c_SH_C3[1], xy), z);
                b[11] = fmul(fmul(c_SH_C3[2], y), fsub(fsub(fmul(4.0f, zz), xx), yy));
                b[12] = fmul(fmul(c_SH_C3[3], z), fsub(fsub(fmul(2.0f, zz), fmul(3.0f, xx)), fmul(3.0f, yy)));
                b[13] = fmul(fmul(c_SH_C3[4], x), fsub(fsub(fmul(4.0f, zz), xx), yy));
                b[14] = fmul(fmul(c_SH_C3[5], z), fsub(xx, yy));
                b[15] = fmul(fmul(c_SH_C3[6], x), ffma(-3.0f, yy, xx));
            }
        }
    }
}
