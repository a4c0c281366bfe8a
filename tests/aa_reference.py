"""Reference of the antialiasing filter (TEST INFRASTRUCTURE ONLY), built on the CPU oracle without changing it.

The filter (DESIGN.md section 2) changes one number per (view, Gaussian): the record's opacity becomes
o_eff = op * rho, rho = sqrt(max(2.5e-5, det0 / det)), where det0 / det are the determinants of the projected 2D
covariance before / after its +0.3 px^2 dilation.  Everything downstream of the record (binning, blend, masks, the
backward blend's sums) consumes o_eff exactly as it consumes an opacity.  So:

  * forward: `preprocess_aa` restates F1's covariance arithmetic in float32 with the same operation order as
    oracle/gs_oracle.c (explicit fused multiply-adds, emulated exactly below) and forms o_eff bit for bit; the oracle then
    renders with o_eff as the opacity.  The result is F1-with-filter bit for bit, which is what the CUDA kernels are
    compared against.
  * backward: the oracle's backward w.r.t. that opacity gives S0 = dL/do_eff and the conic chain unchanged; the filter adds
    dL/dop = rho * S0 and dL/drho = op * S0, which flows into the 2D covariance through the hand-derived
        drho/dx = (ddet0/dx * det - det0 * ddet/dx) / (2 rho det^2)
    and on to the 3D parameters through the hand-derived 2D-covariance chain of B2 (`cov2d_chain`, float64: the same
    standard derivation the oracle's backward states, with dL/d(a, b, c) as its input).
  * `dense_render_aa`: oracle/dense_ref.py's dense float64 formulation with the opacity multiplied by a rho computed from
    a float64 2D covariance (`cov2d`) that torch.autograd differentiates: it shares no code with the two hand-derived steps
    above, so agreement checks both the rho derivative and its chain to the 3D parameters.
"""
from __future__ import annotations

import numpy as np
import torch

RHO2_FLOOR = np.float32(2.5e-5)  # rho >= 0.005
DILATE = 0.3
_f = np.float32


def fma32(a, b, c):
    """float32 fused multiply-add, correctly rounded: the product is exact in float64, TwoSum gives the exact error of the
    float64 sum, round-to-odd on it makes the final rounding to float32 a single correct rounding."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    s = np.asarray(s, np.float64)
    fix = (e != 0) & ((s.view(np.int64) & 1) == 0)
    s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def _affine(m0, m1, m2, m3, x, y, z):
    return fma32(m2, z, fma32(m1, y, m0 * x)) + m3


def _dot3(a0, a1, a2, b0, b1, b2):
    return fma32(a2, b2, fma32(a1, b1, a0 * b0))


def preprocess_aa(inp, cov3d):
    """F1's filter quantities for one view, float32 bit for bit: dict(ca0, cb, cc0, det, ratio = det0/det, rho, o_eff), each
    [P].  inp: the oracle's activated inputs; cov3d [P,6]: F1's 3D covariance (the oracle's state "cov3d").  Only the
    Gaussians the forward keeps (radii > 0) have meaningful values."""
    with np.errstate(all="ignore"):
        V = np.asarray(inp["viewmatrix"], _f).reshape(-1)
        m = np.asarray(inp["means3D"], _f)
        px, py, pz = m[:, 0], m[:, 1], m[:, 2]
        tx = _affine(V[0], V[4], V[8], V[12], px, py, pz)
        ty = _affine(V[1], V[5], V[9], V[13], px, py, pz)
        tz = _affine(V[2], V[6], V[10], V[14], px, py, pz)
        H, W = int(inp["image_height"]), int(inp["image_width"])
        tanx, tany = _f(inp["tanfovx"]), _f(inp["tanfovy"])
        fx, fy = _f(W) / (_f(2) * tanx), _f(H) / (_f(2) * tany)
        limx, limy = _f(1.3) * tanx, _f(1.3) * tany
        cx = np.minimum(limx, np.maximum(-limx, tx / tz)) * tz
        cy = np.minimum(limy, np.maximum(-limy, ty / tz)) * tz
        J00, J11 = fx / tz, fy / tz
        tz2 = tz * tz
        J02, J12 = -(fx * cx) / tz2, -(fy * cy) / tz2
        M0 = [fma32(J02, V[4 * k + 2], J00 * V[4 * k]) for k in range(3)]
        M1 = [fma32(J12, V[4 * k + 2], J11 * V[4 * k + 1]) for k in range(3)]
        c6 = np.asarray(cov3d, _f)
        S = [[c6[:, 0], c6[:, 1], c6[:, 2]], [c6[:, 1], c6[:, 3], c6[:, 4]], [c6[:, 2], c6[:, 4], c6[:, 5]]]
        N0 = [_dot3(M0[0], M0[1], M0[2], S[0][k], S[1][k], S[2][k]) for k in range(3)]
        N1 = [_dot3(M1[0], M1[1], M1[2], S[0][k], S[1][k], S[2][k]) for k in range(3)]
        ca0 = _dot3(*N0, *M0)
        cb = _dot3(*N0, *M1)
        cc0 = _dot3(*N1, *M1)
        ca, cc = ca0 + _f(DILATE), cc0 + _f(DILATE)
        det = fma32(ca, cc, -(cb * cb))
        det0 = fma32(ca0, cc0, -(cb * cb))
        ratio = det0 / det
        rho = np.sqrt(np.maximum(RHO2_FLOOR, ratio))
        o_eff = np.asarray(inp["opacities"], _f).reshape(-1) * rho
    return dict(ca0=ca0, cb=cb, cc0=cc0, det=det, ratio=ratio, rho=rho, o_eff=o_eff)


def cov2d(means3D, viewmatrix, tanfovx, tanfovy, H, W, scales=None, rotations=None, cov3D_precomp=None, scale_modifier=1.0,
          visible=None):
    """Undilated projected 2D covariance (a, b, c) [P] of float64 tensors, differentiable; the EWA projection of
    SURVEY.md A.2 (the clamped tx/tz treated as a constant, as the kernels do).  visible [P] bool masks culled rows."""
    dt = torch.float64
    P = means3D.shape[0]
    Vm = viewmatrix.to(dt).reshape(4, 4)
    pv = torch.cat([means3D, torch.ones(P, 1, dtype=dt)], 1) @ Vm
    if cov3D_precomp is None:
        r, x, y, z = rotations[:, 0], rotations[:, 1], rotations[:, 2], rotations[:, 3]
        R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                         2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                         2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(P, 3, 3)
        L = R * (scale_modifier * scales)[:, None, :]
        S = L @ L.transpose(1, 2)
    else:
        c = cov3D_precomp
        S = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], -1).reshape(P, 3, 3)
    fx, fy = W / (2 * tanfovx), H / (2 * tanfovy)
    tz = pv[:, 2]
    vis = torch.ones(P, dtype=torch.bool) if visible is None else torch.as_tensor(visible)
    tz = torch.where(vis, tz, torch.ones_like(tz))

    def clamp_const(t, lim):
        ratio = t / tz
        clamped = (ratio < -lim) | (ratio > lim)
        return torch.where(clamped, (ratio.clamp(-lim, lim) * tz).detach(), t)

    cx, cy = clamp_const(pv[:, 0], 1.3 * tanfovx), clamp_const(pv[:, 1], 1.3 * tanfovy)
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz, zero, -fx * cx / tz ** 2, zero, fy / tz, -fy * cy / tz ** 2], -1).reshape(P, 2, 3)
    M = J @ Vm[:3, :3].T
    cov = M @ S @ M.transpose(1, 2)
    return cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 1]


def cov2d_chain(inp, cov3d, da, db, dc, visible):
    """Hand-derived chain of a 2D-covariance gradient dL/d(a, b, c) [P] (float64, undilated a, b, c as functions of the
    inputs; the dilation is a constant) to dL/d(means3D, scales, rotations | cov3D_precomp), in float64: the EWA projection
    backward of SURVEY.md A.6 (clamped tx/tz treated as a constant) and the cov3D -> scale / rotation backward of A.7, written
    as in the oracle's B2 (no quaternion normalisation: the caller's activation supplies it).  Rows not visible get zero."""
    V = np.asarray(inp["viewmatrix"], np.float64).reshape(-1)
    m = np.asarray(inp["means3D"], np.float64)
    H, W = int(inp["image_height"]), int(inp["image_width"])
    tanx, tany = float(np.float32(inp["tanfovx"])), float(np.float32(inp["tanfovy"]))
    vis = np.asarray(visible, bool)
    da, db, dc = (np.where(vis, x, 0.0) for x in (da, db, dc))
    Wm = np.array([[V[4 * k + r] for k in range(3)] for r in range(3)])  # Wm[r][k] = V[4k + r]: the w2c rotation
    t = m @ Wm.T + np.array([V[12], V[13], V[14]])
    tx, ty, tz = t[:, 0], t[:, 1], np.where(vis, t[:, 2], 1.0)
    fx, fy = W / (2 * tanx), H / (2 * tany)
    limx, limy = 1.3 * tanx, 1.3 * tany
    txtz, tytz = tx / tz, ty / tz
    cx, cy = np.clip(txtz, -limx, limx) * tz, np.clip(tytz, -limy, limy) * tz
    xmul, ymul = ((txtz >= -limx) & (txtz <= limx)).astype(np.float64), ((tytz >= -limy) & (tytz <= limy)).astype(np.float64)
    J00, J11, J02, J12 = fx / tz, fy / tz, -fx * cx / tz ** 2, -fy * cy / tz ** 2
    M0 = J00[:, None] * Wm[0][None] + J02[:, None] * Wm[2][None]  # [P,3]
    M1 = J11[:, None] * Wm[1][None] + J12[:, None] * Wm[2][None]
    c6 = np.asarray(cov3d, np.float64)
    S = c6[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3)
    N0, N1 = np.einsum("pk,pkj->pj", M0, S), np.einsum("pk,pkj->pj", M1, S)
    # a = M0 S M0^T, b = M0 S M1^T, c = M1 S M1^T:  dL/dS = da M0 M0^T + db (M0 M1^T + M1 M0^T) / 2 + dc M1 M1^T
    dS = (da[:, None, None] * M0[:, :, None] * M0[:, None, :] + 0.5 * db[:, None, None] * (M0[:, :, None] * M1[:, None, :] +
          M1[:, :, None] * M0[:, None, :]) + dc[:, None, None] * M1[:, :, None] * M1[:, None, :])
    dM0 = 2 * da[:, None] * N0 + db[:, None] * N1
    dM1 = db[:, None] * N0 + 2 * dc[:, None] * N1
    dJ00, dJ02 = dM0 @ Wm[0], dM0 @ Wm[2]
    dJ11, dJ12 = dM1 @ Wm[1], dM1 @ Wm[2]
    dtx = xmul * -fx / tz ** 2 * dJ02
    dty = ymul * -fy / tz ** 2 * dJ12
    dtz = -fx / tz ** 2 * dJ00 - fy / tz ** 2 * dJ11 + 2 * fx * cx / tz ** 3 * dJ02 + 2 * fy * cy / tz ** 3 * dJ12
    out = dict(means3D=np.stack([dtx, dty, dtz], 1) @ Wm)
    if inp.get("cov3D_precomp") is not None:  # packed [xx, xy, xz, yy, yz, zz]: off-diagonals appear twice in S
        out["cov3D_precomp"] = np.stack([dS[:, 0, 0], 2 * dS[:, 0, 1], 2 * dS[:, 0, 2], dS[:, 1, 1], 2 * dS[:, 1, 2], dS[:, 2, 2]], 1)
        return out
    q = np.asarray(inp["rotations"], np.float64)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                  2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                  2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    mod = float(inp.get("scale_modifier", 1.0))
    s = mod * np.asarray(inp["scales"], np.float64)
    L = R * s[:, None, :]                     # S = L L^T
    dL = 2 * dS @ L                           # dL/dL
    out["scales"] = mod * np.einsum("prk,prk->pk", R, dL)
    dR = dL * s[:, None, :]
    out["rotations"] = np.stack([
        2 * z * (dR[:, 1, 0] - dR[:, 0, 1]) + 2 * y * (dR[:, 0, 2] - dR[:, 2, 0]) + 2 * x * (dR[:, 2, 1] - dR[:, 1, 2]),
        2 * y * (dR[:, 0, 1] + dR[:, 1, 0]) + 2 * z * (dR[:, 0, 2] + dR[:, 2, 0]) + 2 * r * (dR[:, 2, 1] - dR[:, 1, 2]) - 4 * x * (dR[:, 1, 1] + dR[:, 2, 2]),
        2 * x * (dR[:, 0, 1] + dR[:, 1, 0]) + 2 * r * (dR[:, 0, 2] - dR[:, 2, 0]) + 2 * z * (dR[:, 1, 2] + dR[:, 2, 1]) - 4 * y * (dR[:, 0, 0] + dR[:, 2, 2]),
        2 * r * (dR[:, 1, 0] - dR[:, 0, 1]) + 2 * x * (dR[:, 0, 2] + dR[:, 2, 0]) + 2 * y * (dR[:, 1, 2] + dR[:, 2, 1]) - 4 * z * (dR[:, 0, 0] + dR[:, 1, 1])], 1)
    return out


def rho_of(a, b, c, visible=None):
    """rho (float64 tensor, differentiable) from the undilated 2D covariance"""
    det0 = a * c - b * b
    det = (a + DILATE) * (c + DILATE) - b * b
    if visible is not None:
        det = torch.where(torch.as_tensor(visible), det, torch.ones_like(det))
    return torch.sqrt(torch.clamp_min(det0 / det, float(RHO2_FLOOR)))


class AAOracle:
    """The oracle with the filter on (antialiasing=True) or off: forward() / state() / backward() as oracle.Oracle."""

    def __init__(self, threads: int = 0):
        from oracle.gs_oracle import Oracle
        self.o = Oracle(threads=threads)
        self.f = None

    def forward(self, *, antialiasing=True, **inp):
        self.inp, self.f = inp, None
        if not antialiasing:
            return self.o.forward(**inp)
        _, radii, _, _ = self.o.forward(**inp)  # F1's 3D covariances and the culling of the unfiltered pass
        self.cov3d = self.o.state()["cov3d"]
        f = preprocess_aa(inp, self.cov3d)
        out = self.o.forward(**dict(inp, opacities=f["o_eff"].reshape(np.shape(inp["opacities"]))))
        assert np.array_equal(out[1], radii)  # the filter changes no radius
        self.f = f
        return out

    def state(self):
        return self.o.state()

    def rho_cotangent(self, S0, radii):
        """(da, db, dc) [P] float64: dL/drho * drho/d(a, b, c) for dL/do_eff = S0, zero where the floor holds."""
        f, inp = self.f, self.inp
        op = np.asarray(inp["opacities"], np.float64).reshape(-1)
        a0, b, c0 = (f[k].astype(np.float64) for k in ("ca0", "cb", "cc0"))
        a, c = a0 + DILATE, c0 + DILATE
        with np.errstate(all="ignore"):
            det0, det = a0 * c0 - b * b, a * c - b * b
            rho = np.sqrt(np.maximum(float(RHO2_FLOOR), det0 / det))
            k = op * S0 / (2 * rho * det * det)
            g = [k * (c0 * det - det0 * c), k * (-2 * b * det + det0 * 2 * b), k * (a0 * det - det0 * a)]
        live = (radii > 0) & (f["ratio"] > RHO2_FLOOR)
        return [np.where(live, x, 0.0) for x in g]

    def backward(self, dL_dcolor, dL_ddepth, dL_dalpha, sums_err_const=None):
        g = self.o.backward(dL_dcolor, dL_ddepth, dL_dalpha, sums_err_const=sums_err_const)
        if self.f is None:
            return g
        inp, f = self.inp, self.f
        radii = self.o.state()["tiles_touched"] > 0
        S0 = g["opacities"].reshape(-1).astype(np.float64)
        g["dL_do_eff"] = g["opacities"].copy()
        g["opacities"] = (f["rho"].astype(np.float64) * S0).astype(np.float32).reshape(g["opacities"].shape)
        cot = self.rho_cotangent(S0, radii.astype(np.int32))
        g["rho_cotangent"] = np.stack(cot, 1)
        for k, e in cov2d_chain(inp, self.cov3d, *cot, radii).items():
            g[k] = (g[k].astype(np.float64) + e.reshape(g[k].shape)).astype(np.float32)
        return g


def dense_render_aa(*, opacities, means3D, viewmatrix, tanfovx, tanfovy, H, W, radii, scales=None, rotations=None,
                    cov3D_precomp=None, scale_modifier=1.0, **kw):
    """oracle.dense_ref.dense_render with each visible Gaussian's opacity multiplied by rho (float64, autograd)"""
    from oracle.dense_ref import dense_render
    vis = torch.as_tensor(radii > 0)
    a, b, c = cov2d(means3D, viewmatrix, tanfovx, tanfovy, H, W, scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp,
                    scale_modifier=scale_modifier, visible=vis)
    rho = torch.where(vis, rho_of(a, b, c, vis), torch.ones_like(a))
    op = (opacities.reshape(-1) * rho).reshape(opacities.shape)
    return dense_render(opacities=op, means3D=means3D, viewmatrix=viewmatrix, tanfovx=tanfovx, tanfovy=tanfovy, H=H, W=W, radii=radii,
                        scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp, scale_modifier=scale_modifier, **kw)
