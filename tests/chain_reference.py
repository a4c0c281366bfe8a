"""Float64 chain rule of the per-Gaussian backward, with a running bound on float32 evaluation error (TEST INFRASTRUCTURE).

B2+B3 (preprocess_bwd_kernel, csrc/preprocess.cu) turn each (view, Gaussian) ScreenGrad record of the backward blend into
parameter gradients; normal_bwd_kernel (csrc/normals.cu) adds the normal map's share into dL/drotations.  chain() restates
both in float64, vectorised over Gaussians and looped over views in view order, on the exact float32 inputs the kernels
read: the parameters, the activated values F1 computed (taken as given, never recomputed with a different exp), the
cameras, radii, SH clamp bits, geometry records, ScreenGrad sums and the normal sums.  The rules are the reference's as
they stand (SURVEY.md A.6 / A.7), not autograd of some other forward:

  * the clamped tx/tz * tz of the guard band is a constant (oracle/dense_ref.py), and xmul / ymul zero dtx / dty there;
  * d2inv = 1 / (denom^2 + 1e-7), and a view whose d2inv is 0 adds no covariance or Jacobian term;
  * colour gradients are zeroed per channel where the forward clamped it;
  * antialiasing's rho = sqrt(max(det0 / det, 2.5e-5)) has a zero derivative on the floor;
  * the 3D filter's dL/ds_i = f3s_i dL/ds'_i + f3q_i with f3s = 1 where t_i = 0 and f3q = 0 where the variance is 0;
  * sigmoid, exp and F.normalize Jacobians as torch's autograd defines them; below ||q|| = 1e-12 F.normalize divides by
    the constant 1e-12, so its gradient is g / 1e-12 with no projection.

Branches follow the forward that ran: the guard band from F1's own float32 tx / tz (gs_affine's pinned order, emulated
here bit for bit), the SH clamp from the forward's clamp bits.  Antialiasing's rho and its floor are F1's float32 values
(f1_rho emulates gs_cov2d / gs_aa_ratio bit for bit): B2 recomputes them in F1's operations, because det0 is a
cancellation for a needle and a rho of B2's own rounding could be off by more than itself.

Each quantity is an EB: its float64 value and a bound e on the error a float32 evaluation of the same expression, from
the same float32 inputs, can have:
    e(a +- b) = e_a + e_b + u|a +- b|          e(ab) = |a| e_b + |b| e_a + e_a e_b + u|ab|
    e(a / b) = (e_a + |a / b| e_b) / (|b| - e_b) + u|a / b|
    e(sqrt a) = e_a / (sqrt a + sqrt max(a - e_a, 0)) + u sqrt a          min / max / select: the largest operand e
with u = 2^-24, and 2^-149 more per rounding for results in float32's subnormal range.  An FMA only removes a rounding,
so the bound holds for whatever contraction the compiler picks, and for any association that rounds no more often.
The kernels' plain-float expressions are written here in the kernels' association; where a kernel associates a sum
differently the bound of that sum differs by terms of the same order, which is why a kernel value is required within
K = 2 bounds rather than one: the factor covers a different association of the same terms, not a per-case tolerance.

chain(..., num=EB) is the reference; test_chain_cpu.py runs the same statement with a float32 number type and with
`mutate` switches to show that the check fails on a wrong kernel."""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -149
K = 2.0
f32, f64 = np.float32, np.float64
C = lambda x: float(f32(x))  # a float32 literal of the kernels, as a float64

SH_C0, SH_C1 = C(0.28209479177387814), C(0.4886025119029199)
SH_C2 = [C(x) for x in (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)]
SH_C3 = [C(x) for x in (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
                        1.445305721320277, -0.5900435899266435)]
RHO_FLOOR = C(2.5e-5)
MUTATIONS = ("xmul", "eps7", "dbh2", "clamp", "prefetch", "f3q", "normalize", "sigmoid", "rho_floor")


class EB:
    """float64 value v with the bound e on the error of its float32 evaluation"""
    __slots__ = ("v", "e")
    __array_ufunc__ = None  # numpy operands defer to EB's operators

    def __init__(self, v, e=None):
        self.v = np.asarray(v, f64)
        self.e = np.zeros(self.v.shape) if e is None else e

    @staticmethod
    def w(x):
        return x if isinstance(x, EB) else EB(x)

    @staticmethod
    def rnd(v):
        return U * np.abs(v) + TINY

    def __add__(a, b):
        b = EB.w(b)
        v = a.v + b.v
        return EB(v, a.e + b.e + EB.rnd(v))

    __radd__ = __add__

    def __sub__(a, b):
        b = EB.w(b)
        v = a.v - b.v
        return EB(v, a.e + b.e + EB.rnd(v))

    def __rsub__(a, b):
        return EB.w(b) - a

    def __neg__(a):
        return EB(-a.v, a.e)

    def __mul__(a, b):
        b = EB.w(b)
        v = a.v * b.v
        with np.errstate(invalid="ignore"):
            e = np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e + EB.rnd(v)
        return EB(v, np.where(np.isnan(e), np.inf, e))  # 0 x an unbounded operand: unbounded

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = EB.w(b)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = a.v / b.v
            den = np.abs(b.v) - b.e
            e = np.where(den > 0, (a.e + np.abs(v) * b.e) / np.where(den > 0, den, 1.0), np.inf) + EB.rnd(v)
        return EB(v, e)

    def __rtruediv__(a, b):
        return EB.w(b) / a

    @staticmethod
    def sqrt(a):
        v = np.sqrt(np.maximum(a.v, 0.0))
        lo = np.sqrt(np.maximum(a.v - a.e, 0.0))
        with np.errstate(divide="ignore", invalid="ignore"):
            prop = np.where(v + lo > 0, a.e / np.where(v + lo > 0, v + lo, 1.0), np.sqrt(a.e))
        return EB(v, prop + EB.rnd(v))

    @staticmethod
    def fmax(a, b):
        a, b = EB.w(a), EB.w(b)
        return EB(np.maximum(a.v, b.v), np.maximum(a.e, b.e))

    @staticmethod
    def where(m, a, b):
        a, b = EB.w(a), EB.w(b)
        return EB(np.where(m, a.v, b.v), np.where(m, a.e, b.e))

    @staticmethod
    def inp(x):
        return EB(np.asarray(x, f64))

    def out(self):
        return self.v


# ---- F1's own float32 decisions --------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fmaf(a, b, c) of float32 arrays, correctly rounded (float64 product and sum, with the sum's rounding error carried
    to settle float32 halfway cases)"""
    a, b, c = (np.asarray(x, f32).astype(f64) for x in (a, b, c))
    p = a * b  # exact: 48 significant bits
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)  # s + err == p + c exactly
    r = s.astype(f32)
    d = s - r.astype(f64)
    toward = np.nextafter(r, np.where(d > 0, np.inf, -np.inf).astype(f32))
    half = np.abs(toward.astype(f64) - r.astype(f64)) == 2 * np.abs(d)
    # s on a float32 midpoint: s rounded to even, the exact value lies on err's side of it
    fix = half & (err != 0) & (d != 0)
    alt = np.where(np.sign(err) == np.sign(d), toward, r)
    # s rounded away from err's side: the exact value is nearer r only if err points back to r
    return np.where(fix, alt, r).astype(f32)


def affine32(m, x, y, z):
    """gs_affine: m0 x + m1 y + m2 z + m3 as mul, fma, fma, add"""
    a = (f32(m[0]) * x).astype(f32)
    a = fma32(f32(m[1]), y, a)
    a = fma32(f32(m[2]), z, a)
    return (a + f32(m[3])).astype(f32)


def filter3d32(s, var):
    """gs_filter3d in float32: (s', t, r, coef)"""
    s = np.asarray(s, f32)
    s2 = s * s
    t = s2 + np.asarray(var, f32)[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(t > 0, s2 / t, f32(1)).astype(f32)
    sp = np.sqrt(t)
    coef = np.sqrt(r[:, 0] * r[:, 1] * r[:, 2])
    return sp, t, r, coef.astype(f32)


def guard_band(means_v, view, tanx, tany):
    """F1's clamp side per Gaussian of one view: -1 / 0 / +1 for tx / tz below / inside / above +-1.3 tan(fov x), and the
    same for y"""
    x, y, z = (np.asarray(means_v[:, k], f32) for k in range(3))
    tx = affine32(view[[0, 4, 8, 12]], x, y, z)
    ty = affine32(view[[1, 5, 9, 13]], x, y, z)
    tz = affine32(view[[2, 6, 10, 14]], x, y, z)
    out = []
    for t, tan in ((tx, tanx), (ty, tany)):
        lim = f32(1.3) * f32(tan)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = (t / tz).astype(f32)
        out.append(np.where(q < -lim, -1, np.where(q > lim, 1, 0)))
    return out


def _dot3_32(a, b):
    """gs_dot3: a0 b0, then two FMAs"""
    return fma32(a[2], b[2], fma32(a[1], b[1], (a[0] * b[0]).astype(f32)))


def cov3d32(d):
    """F1's float32 3D covariance [6][P] (build_cov3d, gs_rotmat, gs_filter3d), or cov3D_precomp"""
    if d.get("cov") is not None:
        return [np.asarray(d["cov"][:, k], f32) for k in range(6)]
    q = np.asarray(d["qhat"] if d["raw"] else d["q"], f32)
    r, x, y, z = (q[:, c] for c in range(4))
    m = lambda a, b: (a * b).astype(f32)
    two, one = f32(2), f32(1)
    R = [[fma32(-two, fma32(z, z, m(y, y)), one), m(two, fma32(x, y, -m(r, z))), m(two, fma32(x, z, m(r, y)))],
         [m(two, fma32(x, y, m(r, z))), fma32(-two, fma32(z, z, m(x, x)), one), m(two, fma32(y, z, -m(r, x)))],
         [m(two, fma32(x, z, -m(r, y))), m(two, fma32(y, z, m(r, x))), fma32(-two, fma32(y, y, m(x, x)), one)]]
    s3 = np.asarray(d["s"], f32)
    if d.get("var") is not None:
        s3 = filter3d32(s3, d["var"])[0]
    sm = [m(f32(d["mod"]), s3[:, k]) for k in range(3)]
    L = [[m(R[i][k], sm[k]) for k in range(3)] for i in range(3)]
    return [_dot3_32(L[0], L[0]), _dot3_32(L[0], L[1]), _dot3_32(L[0], L[2]), _dot3_32(L[1], L[1]), _dot3_32(L[1], L[2]),
            _dot3_32(L[2], L[2])]


def f1_rho(d):
    """F1's antialiasing factor per view, bit for bit (gs_cov2d, gs_aa_ratio): rho = sqrt(max(2.5e-5, det0 / det)) [V,P], and
    whether the floor held (not ratio > 2.5e-5) [V,P]"""
    c6 = cov3d32(d)
    S = [[c6[0], c6[1], c6[2]], [c6[1], c6[3], c6[4]], [c6[2], c6[4], c6[5]]]
    m = lambda a, b: (a * b).astype(f32)
    rho, floored = [], []
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for v in range(d["V"]):
            V = np.asarray(d["view"][v], f32)
            x, y, z = (np.asarray(d["means"][v][:, k], f32) for k in range(3))
            tx, ty, tz = (affine32(V[[j, 4 + j, 8 + j, 12 + j]], x, y, z) for j in range(3))
            tanx, tany = f32(d["tanx"][v]), f32(d["tany"][v])
            fx, fy = f32(d["W"]) / m(f32(2), tanx), f32(d["H"]) / m(f32(2), tany)
            limx, limy = m(f32(1.3), tanx), m(f32(1.3), tany)
            cx = m(np.minimum(limx, np.maximum(-limx, (tx / tz).astype(f32))), tz)
            cy = m(np.minimum(limy, np.maximum(-limy, (ty / tz).astype(f32))), tz)
            tz2 = m(tz, tz)
            J00, J11 = (fx / tz).astype(f32), (fy / tz).astype(f32)
            J02, J12 = (-m(fx, cx) / tz2).astype(f32), (-m(fy, cy) / tz2).astype(f32)
            M0 = [fma32(J02, V[4 * k + 2], m(J00, V[4 * k])) for k in range(3)]
            M1 = [fma32(J12, V[4 * k + 2], m(J11, V[4 * k + 1])) for k in range(3)]
            N0 = [_dot3_32(M0, [S[0][k], S[1][k], S[2][k]]) for k in range(3)]
            N1 = [_dot3_32(M1, [S[0][k], S[1][k], S[2][k]]) for k in range(3)]
            ca0, cb, cc0 = _dot3_32(N0, M0), _dot3_32(N0, M1), _dot3_32(N1, M1)
            bb = -m(cb, cb)
            det = fma32((ca0 + f32(0.3)).astype(f32), (cc0 + f32(0.3)).astype(f32), bb)
            ratio = (fma32(ca0, cc0, bb) / det).astype(f32)
            rho.append(np.sqrt(np.maximum(f32(2.5e-5), ratio)))
            floored.append(~(ratio > f32(2.5e-5)))
    return np.stack(rho), np.stack(floored)


def normalize32(q):
    """gs_normalize4 in float32: (q^, max(||q||, 1e-12), ||q||)"""
    q = np.asarray(q, f32)
    n2 = ((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]).astype(f32) + (q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3]).astype(f32)).astype(f32)
    ln = np.sqrt(n2)
    n = np.maximum(ln, f32(1e-12))
    return (q / n[:, None]).astype(f32), n, ln


# ---- the chain ----------------------------------------------------------------------------------------------------------------
def sh_basis(num, deg, x, y, z):
    b = [num.inp(np.full(x.v.shape, SH_C0))]
    if deg > 0:
        b += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b += [SH_C2[0] * xy, SH_C2[1] * yz, SH_C2[2] * ((2.0 * zz - xx) - yy), SH_C2[3] * xz, SH_C2[4] * (xx - yy)]
        if deg > 2:
            b += [(SH_C3[0] * y) * (3.0 * xx - yy), (SH_C3[1] * xy) * z, (SH_C3[2] * y) * ((4.0 * zz - xx) - yy),
                  (SH_C3[3] * z) * ((2.0 * zz - 3.0 * xx) - 3.0 * yy), (SH_C3[4] * x) * ((4.0 * zz - xx) - yy),
                  (SH_C3[5] * z) * (xx - yy), (SH_C3[6] * x) * (xx - 3.0 * yy)]
    return b


def rotmat(q):
    r, x, y, z = q
    return [[1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - r * z), 2.0 * (x * z + r * y)],
            [2.0 * (x * y + r * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - r * x)],
            [2.0 * (x * z - r * y), 2.0 * (y * z + r * x), 1.0 - 2.0 * (x * x + y * y)]]


def dcol_dq(k, q, g0, g1, g2):
    """normals.cu's dcol_dq for the rows whose axis is k (evaluated for all rows; the caller selects)"""
    r, x, y, z = q
    if k == 0:
        return [2.0 * (z * g1 - y * g2), 2.0 * (y * g1 + z * g2), -4.0 * y * g0 + 2.0 * (x * g1 - r * g2),
                -4.0 * z * g0 + 2.0 * (r * g1 + x * g2)]
    if k == 1:
        return [2.0 * (x * g2 - z * g0), 2.0 * (y * g0 + r * g2) - 4.0 * x * g1, 2.0 * (x * g0 + z * g2),
                2.0 * (y * g2 - r * g0) - 4.0 * z * g1]
    return [2.0 * (y * g0 - x * g1), 2.0 * (z * g0 - r * g1) - 4.0 * x * g2, 2.0 * (r * g0 + z * g1) - 4.0 * y * g2,
            2.0 * (x * g0 + y * g1)]


def normalize_jacobian(num, q, dq, qnorm, qlen, mutate):
    """F.normalize's autograd: (dq - q^ (q^ . dq)) / ||q|| at ||q|| >= 1e-12, dq / 1e-12 below"""
    if "normalize" in mutate:
        return dq
    dot = q[0] * dq[0] + q[1] * dq[1] + q[2] * dq[2] + q[3] * dq[3]
    dot = num.where(np.asarray(qlen) >= f32(1e-12), dot, 0.0)
    inv = 1.0 / num.inp(qnorm)
    return [(dq[c] - q[c] * dot) * inv for c in range(4)]


def chain(d, num=EB, mutate=()):
    """d: the call's float32 inputs (see gpu inputs in test_gpu_chain.py):
      P, V, H, W, deg, M, mod, raw, aa, moments;
      means [V,P,3] (per_view: whether the kernel had per-view means), view / proj [V,16] (memory order), campos [V,3],
      tanx / tany [V];
      op [P] (activated), s [P,3] (activated, before the filter), q [P,4] (as read), qhat / qnorm / qlen (normalize32 of q
      for raw parameters), cov [P,6] or None, var [P] (3D filter) or None, shs [P,M,3] or None, colors or None;
      radii [V,P], clamped [V,P], recs [V,P,12], sums [V,P,12];
      normals: None, or dict(sign [V,P], wn [V,P,3], axis [P]).
    Returns {name: num} of the gradients: means3D [P,3] or [V,P,3], means2D [V,P,3], opacities [P], shs [P,M,3] / colors,
    scales, rotations, cov3D."""
    mutate = set(mutate)
    if d["aa"] and "rho" not in d:
        d["rho"], d["floored"] = f1_rho(d)
    P, V, W, H, deg = d["P"], d["V"], d["W"], d["H"], d["deg"]
    nb = 1 if deg < 0 else (deg + 1) ** 2
    I = num.inp
    Z = lambda: I(np.zeros(P))
    cov_pre, var = d.get("cov"), d.get("var")
    f3d = var is not None and cov_pre is None
    raw = d["raw"]
    mod = C(d["mod"])
    coef = I(np.ones(P))
    if cov_pre is not None:
        c6 = [I(cov_pre[:, k]) for k in range(6)]
        Rm = s = q = None
    else:
        q = [I((d["qhat"] if raw else d["q"])[:, c]) for c in range(4)]
        s3 = [I(d["s"][:, k]) for k in range(3)]
        if f3d:
            vv = I(var)
            t = [s3[k] * s3[k] + vv for k in range(3)]
            t32 = filter3d32(d["s"], var)[1]
            r = [num.where(t32[:, k] > 0, (s3[k] * s3[k]) / t[k], 1.0) for k in range(3)]
            s3 = [num.sqrt(t[k]) for k in range(3)]
            coef = num.sqrt((r[0] * r[1]) * r[2])
        Rm = rotmat(q)
        s = [mod * s3[k] for k in range(3)]
        L = [[Rm[i][k] * s[k] for k in range(3)] for i in range(3)]
        dot3 = lambda a, b: a[0] * b[0] + a[1] * b[1] + a[2] * b[2]
        c6 = [dot3(L[0], L[0]), dot3(L[0], L[1]), dot3(L[0], L[2]), dot3(L[1], L[1]), dot3(L[1], L[2]), dot3(L[2], L[2])]
    S = [[c6[0], c6[1], c6[2]], [c6[1], c6[3], c6[4]], [c6[2], c6[4], c6[5]]]
    op = I(d["op"])
    opp = op * coef  # the opacity antialiasing's rho multiplies (o' with the 3D filter)

    dmean = [Z() for _ in range(3)]
    dcov = [Z() for _ in range(6)]
    dop, dcol = Z(), [Z() for _ in range(3)]
    dsh = [[Z() for _ in range(3)] for _ in range(nb)]
    per_view_out = [] if d["per_view"] else None
    m2d = []
    shs = d.get("shs")
    for v in range(V):
        rad = d["radii"][v] > 0
        vis = rad
        sv = v + 1 if "prefetch" in mutate else v
        g = d["sums"][sv] if sv < V else np.zeros_like(d["sums"][0])
        rec = d["recs"][v]
        cl = d["clamped"][v]
        if d["per_view"] and v > 0:
            per_view_out.append(dmean)
            dmean = [Z() for _ in range(3)]
        if not vis.any():
            m2d.append([Z(), Z(), Z()])
            continue
        mv = d["means"][v]
        px, py, pz = (I(mv[:, k]) for k in range(3))
        if d["moments"]:
            S0, Sx, Sy, Sxx, Sxy, Syy = (I(g[:, k]) for k in range(6))
            ro, rA, rB, rC = (I(rec[:, k]) for k in (7, 4, 5, 6))
            gO = S0
            gdx = -ro * (rA * Sx + rB * Sy) * (0.5 * W)
            gdy = -ro * (rC * Sy + rB * Sx) * (0.5 * H)
            dA, dBh, dC = -0.5 * ro * Sxx, -0.5 * ro * Sxy, -0.5 * ro * Syy
        else:
            gdx, gdy, dA, dBh, dC, gO = (I(g[:, k]) for k in range(6))
        gcol = [I(g[:, 6]), I(g[:, 7]), I(g[:, 8])]
        gdepth = I(g[:, 9])
        m2d.append([num.where(rad, gdx, 0.0), num.where(rad, gdy, 0.0), Z()])
        if "dbh2" in mutate:
            dBh = 2.0 * dBh
        contrib_op = Z() if d["aa"] else gO

        Vm, PV = d["view"][v].astype(f64), d["proj"][v].astype(f64)
        tx = Vm[0] * px + Vm[4] * py + Vm[8] * pz + Vm[12]
        ty = Vm[1] * px + Vm[5] * py + Vm[9] * pz + Vm[13]
        tz = Vm[2] * px + Vm[6] * py + Vm[10] * pz + Vm[14]
        tanx, tany = C(d["tanx"][v]), C(d["tany"][v])
        fx = float(W) / (2.0 * num.inp(np.full(P, tanx)))
        fy = float(H) / (2.0 * num.inp(np.full(P, tany)))
        limx, limy = C(f32(1.3) * f32(tanx)), C(f32(1.3) * f32(tany))
        bx, by = guard_band(mv, d["view"][v], tanx, tany)
        cx = num.where(bx == 0, (tx / tz) * tz, (bx * limx) * tz)
        cy = num.where(by == 0, (ty / tz) * tz, (by * limy) * tz)
        xmul = np.ones(P) if "xmul" in mutate else (bx == 0).astype(f64)
        ymul = (by == 0).astype(f64)
        itz = 1.0 / tz
        itz2 = itz * itz
        itz3 = itz2 * itz
        J00, J11 = fx * itz, fy * itz
        J02, J12 = -(fx * cx) * itz2, -(fy * cy) * itz2
        Wm = [[Vm[4 * k + j] for k in range(3)] for j in range(3)]  # Wm[j][k] = V[4k + j]
        M0 = [J00 * Wm[0][k] + J02 * Wm[2][k] for k in range(3)]
        M1 = [J11 * Wm[1][k] + J12 * Wm[2][k] for k in range(3)]
        N0 = [M0[0] * S[0][k] + M0[1] * S[1][k] + M0[2] * S[2][k] for k in range(3)]
        N1 = [M1[0] * S[0][k] + M1[1] * S[1][k] + M1[2] * S[2][k] for k in range(3)]
        ca0 = N0[0] * M0[0] + N0[1] * M0[1] + N0[2] * M0[2]
        ca = ca0 + C(0.3)
        cb = N0[0] * M1[0] + N0[1] * M1[1] + N0[2] * M1[2]
        cc0 = N1[0] * M1[0] + N1[1] * M1[1] + N1[2] * M1[2]
        cc = cc0 + C(0.3)
        denom = ca * cc - cb * cb
        eps = 0.0 if "eps7" in mutate else C(1e-7)
        d2inv = 1.0 / (denom * denom + eps)
        # the float32 square overflows (d2inv == 0): the kernel adds nothing for this view
        live = rad & (np.abs(denom.v) < 1.8e19)
        ra = rb = rc = 0.0
        if d["aa"]:
            ratio = (ca0 * cc0 - cb * cb) / denom
            if "rho_floor" in mutate:
                rho, floored = num.sqrt(ratio), np.zeros(P, bool)
            else:  # F1's rho, an input: B2 recomputes it in F1's operations
                rho, floored = I(d["rho"][v]), d["floored"][v]
            contrib_op = rho * gO
            if "diag" in d and isinstance(ratio, EB):
                d["diag"].append((v, ratio.v, ratio.e, rad))
            k = (C(0.3) * opp * gO) / (rho * denom * denom)
            ra = num.where(floored, 0.0, 0.5 * k * (cc0 * cc + cb * cb))
            rc = num.where(floored, 0.0, 0.5 * k * (ca0 * ca + cb * cb))
            rb = num.where(floored, 0.0, -k * cb * (ca + cc0))
        dop = num.where(rad, dop + contrib_op, dop)
        da = d2inv * ((-cc * cc) * dA + (2.0 * cb * cc) * dBh - (cb * cb) * dC) + ra
        dc = d2inv * ((-ca * ca) * dC + (2.0 * ca * cb) * dBh - (cb * cb) * dA) + rc
        db = d2inv * 2.0 * ((cb * cc) * dA - (ca * cc + cb * cb) * dBh + (ca * cb) * dC) + rb
        upd = [M0[0] * M0[0] * da + M0[0] * M1[0] * db + M1[0] * M1[0] * dc,
               2.0 * M0[0] * M0[1] * da + (M0[0] * M1[1] + M0[1] * M1[0]) * db + 2.0 * M1[0] * M1[1] * dc,
               2.0 * M0[0] * M0[2] * da + (M0[0] * M1[2] + M0[2] * M1[0]) * db + 2.0 * M1[0] * M1[2] * dc,
               M0[1] * M0[1] * da + M0[1] * M1[1] * db + M1[1] * M1[1] * dc,
               2.0 * M0[2] * M0[1] * da + (M0[1] * M1[2] + M0[2] * M1[1]) * db + 2.0 * M1[1] * M1[2] * dc,
               M0[2] * M0[2] * da + M0[2] * M1[2] * db + M1[2] * M1[2] * dc]
        dcov = [num.where(live, dcov[j] + upd[j], dcov[j]) for j in range(6)]
        dM0 = [2.0 * da * N0[k] + db * N1[k] for k in range(3)]
        dM1 = [db * N0[k] + 2.0 * dc * N1[k] for k in range(3)]
        dJ00 = Wm[0][0] * dM0[0] + Wm[0][1] * dM0[1] + Wm[0][2] * dM0[2]
        dJ02 = Wm[2][0] * dM0[0] + Wm[2][1] * dM0[1] + Wm[2][2] * dM0[2]
        dJ11 = Wm[1][0] * dM1[0] + Wm[1][1] * dM1[1] + Wm[1][2] * dM1[2]
        dJ12 = Wm[2][0] * dM1[0] + Wm[2][1] * dM1[1] + Wm[2][2] * dM1[2]
        dtx = xmul * (-fx * itz2 * dJ02)
        dty = ymul * (-fy * itz2 * dJ12)
        dtz = -fx * itz2 * dJ00 - fy * itz2 * dJ11 + (2.0 * fx * cx) * itz3 * dJ02 + (2.0 * fy * cy) * itz3 * dJ12
        dmean = [num.where(live, dmean[k] + (Wm[0][k] * dtx + Wm[1][k] * dty + Wm[2][k] * dtz), dmean[k]) for k in range(3)]
        # the 2D mean's projection and the depth term
        hw = PV[3] * px + PV[7] * py + PV[11] * pz + PV[15]
        m_w = 1.0 / (hw + C(1e-7))
        mul1 = (PV[0] * px + PV[4] * py + PV[8] * pz + PV[12]) * m_w * m_w
        mul2 = (PV[1] * px + PV[5] * py + PV[9] * pz + PV[13]) * m_w * m_w
        mul3 = Vm[2] * px + Vm[6] * py + Vm[10] * pz + Vm[14]
        for k in range(3):
            t = (PV[4 * k] * m_w - PV[4 * k + 3] * mul1) * gdx + (PV[4 * k + 1] * m_w - PV[4 * k + 3] * mul2) * gdy
            t = t + (Vm[4 * k + 2] - Vm[4 * k + 3] * mul3) * gdepth
            dmean[k] = num.where(rad, dmean[k] + t, dmean[k])
        if deg >= 0:
            cp = d["campos"][v].astype(f64)
            dx0, dy0, dz0 = px - cp[0], py - cp[1], pz - cp[2]
            ln = num.sqrt(dx0 * dx0 + dy0 * dy0 + dz0 * dz0)
            x, y, z = dx0 / ln, dy0 / ln, dz0 / ln
            bs = sh_basis(num, deg, x, y, z)
            keep = lambda c: np.ones(P, bool) if "clamp" in mutate else (cl & (1 << c)) == 0
            dRGB = [num.where(keep(c), gcol[c], 0.0) for c in range(3)]
            for kk in range(nb):
                for c in range(3):
                    dsh[kk][c] = num.where(rad, dsh[kk][c] + bs[kk] * dRGB[c], dsh[kk][c])
            if deg > 0:
                sk = [I(shs[:, kk, 0]) * dRGB[0] + I(shs[:, kk, 1]) * dRGB[1] + I(shs[:, kk, 2]) * dRGB[2] for kk in range(nb)]
                ddx, ddy, ddz = -SH_C1 * sk[3], -SH_C1 * sk[1], SH_C1 * sk[2]
                if deg > 1:
                    xx, yy, zz = x * x, y * y, z * z
                    ddx = ddx + SH_C2[0] * y * sk[4] + SH_C2[2] * -2.0 * x * sk[6] + SH_C2[3] * z * sk[7] + SH_C2[4] * 2.0 * x * sk[8]
                    ddy = ddy + SH_C2[0] * x * sk[4] + SH_C2[1] * z * sk[5] + SH_C2[2] * -2.0 * y * sk[6] + SH_C2[4] * -2.0 * y * sk[8]
                    ddz = ddz + SH_C2[1] * y * sk[5] + SH_C2[2] * 4.0 * z * sk[6] + SH_C2[3] * x * sk[7]
                    if deg > 2:
                        ddx = ddx + (SH_C3[0] * sk[9] * 6.0 * x * y + SH_C3[1] * sk[10] * y * z + SH_C3[2] * sk[11] * -2.0 * x * y +
                                     SH_C3[3] * sk[12] * -6.0 * x * z + SH_C3[4] * sk[13] * (4.0 * zz - 3.0 * xx - yy) +
                                     SH_C3[5] * sk[14] * 2.0 * x * z + SH_C3[6] * sk[15] * 3.0 * (xx - yy))
                        ddy = ddy + (SH_C3[0] * sk[9] * 3.0 * (xx - yy) + SH_C3[1] * sk[10] * x * z +
                                     SH_C3[2] * sk[11] * (4.0 * zz - xx - 3.0 * yy) + SH_C3[3] * sk[12] * -6.0 * y * z +
                                     SH_C3[4] * sk[13] * -2.0 * x * y + SH_C3[5] * sk[14] * -2.0 * y * z +
                                     SH_C3[6] * sk[15] * -6.0 * x * y)
                        ddz = ddz + (SH_C3[1] * sk[10] * x * y + SH_C3[2] * sk[11] * 8.0 * y * z +
                                     SH_C3[3] * sk[12] * 3.0 * (2.0 * zz - xx - yy) + SH_C3[4] * sk[13] * 8.0 * x * z +
                                     SH_C3[5] * sk[14] * (xx - yy))
                dot = x * ddx + y * ddy + z * ddz
                for k, (dd, a) in enumerate(((ddx, x), (ddy, y), (ddz, z))):
                    dmean[k] = num.where(rad, dmean[k] + (dd - a * dot) / ln, dmean[k])
        else:
            dcol = [num.where(rad, dcol[c] + gcol[c], dcol[c]) for c in range(3)]

    out = {"means2D": m2d}
    out["means3D"] = per_view_out + [dmean] if d["per_view"] else dmean
    if f3d:
        so = [I(d["s"][:, k]) for k in range(3)]
        vv = I(var)
        sp32, t32, r32, _ = filter3d32(d["s"], var)
        t = [so[k] * so[k] + vv for k in range(3)]
        r = [num.where(t32[:, k] > 0, (so[k] * so[k]) / t[k], 1.0) for k in range(3)]
        sp = [num.sqrt(t[k]) for k in range(3)]
        cf = num.sqrt((r[0] * r[1]) * r[2])
        og = op * dop
        dop = dop * cf
        f3s = [num.where(t32[:, k] > 0, so[k] / sp[k], 1.0) for k in range(3)]
        if "f3q" in mutate:
            f3q = [Z() for _ in range(3)]
        else:
            f3q = [num.where(np.asarray(var) > 0, og * num.sqrt(r[(k + 1) % 3] * r[(k + 2) % 3]) * vv / (t[k] * sp[k]), 0.0)
                   for k in range(3)]
    if raw and "sigmoid" not in mutate:
        dop = dop * (op * (1.0 - op))
    out["opacities"] = dop
    if deg >= 0:
        out["shs"] = dsh
    else:
        out["colors"] = dcol
    if cov_pre is not None:
        out["cov3D"] = dcov
        return out
    dS = [[dcov[0], 0.5 * dcov[1], 0.5 * dcov[2]], [0.5 * dcov[1], dcov[3], 0.5 * dcov[4]], [0.5 * dcov[2], 0.5 * dcov[4], dcov[5]]]
    L = [[Rm[i][k] * s[k] for k in range(3)] for i in range(3)]
    dLm = [[2.0 * (dS[i][0] * L[0][k] + dS[i][1] * L[1][k] + dS[i][2] * L[2][k]) for k in range(3)] for i in range(3)]
    dsc, dR = [], [[None] * 3 for _ in range(3)]
    for k in range(3):
        proj = Rm[0][k] * dLm[0][k] + Rm[1][k] * dLm[1][k] + Rm[2][k] * dLm[2][k]
        if f3d:
            gk = f3s[k] * (mod * proj) + f3q[k]
            dsc.append(gk * so[k] if raw else gk)
        else:
            dsc.append((s[k] if raw else mod) * proj)
        for i in range(3):
            dR[i][k] = dLm[i][k] * s[k]
    out["scales"] = dsc
    r_, x, y, z = q
    dq = [2.0 * z * (dR[1][0] - dR[0][1]) + 2.0 * y * (dR[0][2] - dR[2][0]) + 2.0 * x * (dR[2][1] - dR[1][2]),
          2.0 * y * (dR[0][1] + dR[1][0]) + 2.0 * z * (dR[0][2] + dR[2][0]) + 2.0 * r_ * (dR[2][1] - dR[1][2]) - 4.0 * x * (dR[1][1] + dR[2][2]),
          2.0 * x * (dR[0][1] + dR[1][0]) + 2.0 * r_ * (dR[0][2] - dR[2][0]) + 2.0 * z * (dR[1][2] + dR[2][1]) - 4.0 * y * (dR[0][0] + dR[2][2]),
          2.0 * r_ * (dR[1][0] - dR[0][1]) + 2.0 * x * (dR[0][2] + dR[2][0]) + 2.0 * y * (dR[1][2] + dR[2][1]) - 4.0 * z * (dR[0][0] + dR[1][1])]
    if raw:
        dq = normalize_jacobian(num, q, dq, d["qnorm"], d["qlen"], mutate)
    nrm = d.get("normals")
    if nrm is not None:
        gsum = [Z() for _ in range(3)]
        for v in range(V):
            rad = d["radii"][v] > 0
            sg = I(nrm["sign"][v])
            gsum = [num.where(rad, gsum[c] + sg * I(nrm["wn"][v][:, c]), gsum[c]) for c in range(3)]
        ax = nrm["axis"]
        per_k = [dcol_dq(k, q, *gsum) for k in range(3)]
        dn = [num.where(ax == 0, per_k[0][c], num.where(ax == 1, per_k[1][c], per_k[2][c])) for c in range(4)]
        if raw:
            dn = normalize_jacobian(num, q, dn, d["qnorm"], d["qlen"], mutate)
        seen = (d["radii"] > 0).any(0)
        dq = [num.where(seen, dq[c] + dn[c], dq[c]) for c in range(4)]
    out["rotations"] = dq
    return out


def stack(x):
    """a nested list of numbers (EB or float32 arrays) -> (values [..., P] moved to [P, ...], bounds or None)"""
    if isinstance(x, list):
        parts = [stack(a) for a in x]
        v = np.stack([np.broadcast_to(p[0], parts[0][0].shape) for p in parts], 1)
        e = None if parts[0][1] is None else np.stack([np.broadcast_to(p[1], parts[0][1].shape) for p in parts], 1)
        return v, e
    if isinstance(x, EB):
        return x.v, x.e
    return np.asarray(x.v), None


def arrays(out, num=EB):
    """{name: (value, bound)} with the kernels' shapes: means3D [P,3] or [V,P,3], means2D [V,P,3], opacities [P],
    shs [P,nb,3], scales [P,3], rotations [P,4], colors [P,3], cov3D [P,6]"""
    res = {}
    for k, x in out.items():
        if k in ("means2D",) or (k == "means3D" and isinstance(x[0], list)):
            parts = [stack(a) for a in x]
            res[k] = (np.stack([p[0] for p in parts]), None if parts[0][1] is None else np.stack([p[1] for p in parts]))
        elif k == "opacities":
            res[k] = (x.v if isinstance(x, EB) else np.asarray(x.v), x.e if isinstance(x, EB) else None)
        else:
            res[k] = stack(x)
    return res


def check(got, ref, what=""):
    """every element of got within K * bound of ref, and every reference, bound and kernel value finite (an infinite bound
    would accept anything); returns (worst |got - ref| / (K bound), count of elements)"""
    v, e = ref
    g = np.asarray(got, f64).reshape(v.shape)
    with np.errstate(invalid="ignore"):
        err = np.abs(g - v)
    lim = K * e
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err == 0, 0.0, err / lim)
    bad = ~(err <= lim) | ~np.isfinite(lim) | ~np.isfinite(v) | ~np.isfinite(g)
    if bad.any():
        i = np.unravel_index(int(np.argmax(np.where(bad, np.nan_to_num(ratio, nan=np.inf, posinf=1e300), -1))), v.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} of {v.size} elements over K * bound; worst at {i}: got {g[i]!r} "
                             f"ref {v[i]!r} bound {e[i]!r} ({ratio[i]:.3g} x K * bound)")
    return float(np.nanmax(ratio, initial=0.0)), v.size
