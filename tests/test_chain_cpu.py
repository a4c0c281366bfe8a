"""CPU: the float64 chain rule of tests/chain_reference.py is right, its error bound holds, and the check it backs fails on a
wrong kernel.

  1. against autograd: a float64 torch forward from the parameters to each view's (NDC mean, conic, record opacity,
     colour, depth), with the reference's constants and floors, fed classic screen-space gradients: chain() agrees with
     its gradients to ~1e-12 relative, SH degrees -1..3, raw and activated, antialiasing, the 3D filter, cov3D_precomp,
     per-view means and normals;
  2. the bound holds: chain() run with float32 arithmetic (every operation rounded to float32, with and without FMA
     contraction of a product into the next sum, views accumulated in order) lies within K e of the float64 chain on every
     element of over 10^6 (view, Gaussian) samples, edge scenes included;
  3. the check fails when it should: each of chain_reference.MUTATIONS applied to the float32 run fails it;
  4. how tight the bound is: the median and 99.9th percentile of e / |ref| per gradient, printed (run with -s)."""
import math

import numpy as np
import pytest
import torch

import chain_reference as CH

f32, f64 = np.float32, np.float64


# ---- a float32 number type for chain() ------------------------------------------------------------------------------------
class F32:
    """float32 evaluation: every operation rounded to float32; with `fma`, a product feeding a sum is not rounded first"""
    __slots__ = ("v", "p")
    __array_ufunc__ = None
    fma = False

    def __init__(self, v, p=None):
        self.v = np.asarray(v, f32)
        self.p = p if type(self).fma else None

    @classmethod
    def w(cls, x):
        return x if isinstance(x, F32) else cls(np.asarray(x, f64).astype(f32))

    def _sum(a, b, sign):
        T = type(a)
        b = T.w(b)
        if a.p is not None:
            return T((a.p + sign * b.v.astype(f64)).astype(f32))
        if b.p is not None:
            return T((a.v.astype(f64) + sign * b.p).astype(f32))
        return T(a.v + b.v if sign > 0 else a.v - b.v)

    def __add__(a, b):
        return a._sum(b, 1.0)

    __radd__ = __add__

    def __sub__(a, b):
        return a._sum(b, -1.0)

    def __rsub__(a, b):
        return type(a).w(b) - a

    def __neg__(a):
        return type(a)(-a.v, None if a.p is None else -a.p)

    def __mul__(a, b):
        b = type(a).w(b)
        return type(a)(a.v * b.v, a.v.astype(f64) * b.v.astype(f64))

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = type(a).w(b)
        with np.errstate(divide="ignore", invalid="ignore"):
            return type(a)(a.v / b.v)

    def __rtruediv__(a, b):
        return type(a).w(b) / a

    @classmethod
    def sqrt(cls, a):
        return cls(np.sqrt(np.maximum(a.v, f32(0))))

    @classmethod
    def fmax(cls, a, b):
        a, b = cls.w(a), cls.w(b)
        return cls(np.maximum(a.v, b.v))

    @classmethod
    def where(cls, m, a, b):
        a, b = cls.w(a), cls.w(b)
        return cls(np.where(m, a.v, b.v))

    @classmethod
    def inp(cls, x):
        return cls(np.asarray(x, f32))


class F32Fma(F32):
    fma = True


# ---- scenes ------------------------------------------------------------------------------------------------------------------
def _look_at(eye, H, W, fovy_deg):
    """a camera at `eye` looking at the origin: (view [16], proj [16], campos, tanx, tany) in the kernels' layout"""
    from humangaussian_b200.cameras import getProjectionMatrix
    eye = np.asarray(eye, f64)
    fwd = -eye / np.linalg.norm(eye)
    up = np.array([0.0, 0.0, 1.0])
    right = np.cross(fwd, up)
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    Rw2c = np.stack([right, down, fwd])  # rows: camera axes (x right, y down, z forward)
    W2C = np.eye(4)
    W2C[:3, :3] = Rw2c
    W2C[:3, 3] = -Rw2c @ eye
    tany = math.tan(math.radians(fovy_deg) / 2)
    tanx = tany * W / H
    proj = getProjectionMatrix(0.01, 100.0, 2 * math.atan(tanx), 2 * math.atan(tany)).numpy().astype(f64)
    vm = W2C.T
    pm = (proj @ W2C).T
    return vm.astype(f32).reshape(16), pm.astype(f32).reshape(16), eye.astype(f32), tanx, tany


def scene(P, V, deg, seed, *, raw=False, aa=False, f3d=False, cov=False, per_view=False, normals=False, moments=True,
          edges=False, H=64, W=96, big=False):
    """the inputs chain() takes, without a GPU: random Gaussians around the origin, V cameras on a sphere, radii from the
    near plane and the image, clamp bits and record opacities from a float32 forward, random ScreenGrad sums.  edges adds
    Gaussians beyond the guard band, just above the near plane, needles near antialiasing's floor (both sides), clamped
    channels, zero filter variances and scales, and quaternions of norm 1e-13, 1e-3 and 1e3."""
    rng = np.random.RandomState(seed)
    cams = [_look_at(_sphere(rng) * rng.uniform(2.5, 3.5), H, W, rng.uniform(40, 70)) for _ in range(V)]
    means = rng.uniform(-0.8, 0.8, (P, 3))
    s = np.exp(rng.uniform(np.log(0.01), np.log(0.15), (P, 3))) * (6.0 if big else 1.0)
    q = rng.randn(P, 4)
    op = rng.uniform(0.05, 0.95, P)
    nb = (deg + 1) ** 2 if deg >= 0 else 0
    shs = 0.3 * rng.randn(P, max(nb, 1), 3)
    var = rng.uniform(0, 1, P) * (s.mean(1) ** 2) * 0.5 if f3d else None
    if edges:
        n = P // 8
        vm0, _, _, tx0, ty0 = cams[0]
        inv = np.linalg.inv(vm0.reshape(4, 4).astype(f64))
        z = rng.uniform(1.0, 2.0, n)
        # guard band (x beyond +-1.3 tan in view 0), wide
        pc = np.stack([np.where(rng.rand(n) < 0.5, -1, 1) * rng.uniform(1.35, 1.8, n) * tx0 * z, rng.uniform(-0.3, 0.3, n) * z, z], 1)
        means[:n] = (np.concatenate([pc, np.ones((n, 1))], 1) @ inv)[:, :3]
        s[:n] = 0.3 * z[:, None]
        # just above the near plane in view 0
        pc = np.stack([rng.uniform(-0.02, 0.02, n), rng.uniform(-0.02, 0.02, n), 0.2 + rng.uniform(1e-5, 1e-2, n)], 1)
        means[n:2 * n] = (np.concatenate([pc, np.ones((n, 1))], 1) @ inv)[:, :3]
        s[n:2 * n] = 0.002
        # needles: one long axis, a thin axis across the floor's threshold (some far below it)
        s[2 * n:3 * n] = np.stack([np.full(n, 0.1), np.full(n, 1e-5) * np.exp(rng.uniform(-3, 3, n)), np.full(n, 1e-5)], 1)
        # clamped channels
        shs[3 * n:4 * n, 0] = np.where(rng.rand(n, 3) < 0.5, -3.0, 1.0)
        if f3d:
            var[4 * n:5 * n:2] = 0.0
            s[4 * n:5 * n:3, 0] = 0.0
        q[5 * n:6 * n] *= np.array([1e-13, 1e-3, 1e3])[np.arange(n) % 3, None]
        # sub-pixel footprints: det near the dilation's 0.09, where d2inv's 1e-7 shows
        s[6 * n:7 * n] = 1e-4
    if not raw:
        q /= np.linalg.norm(q, axis=1, keepdims=True)
    d = dict(P=P, V=V, H=H, W=W, deg=deg, M=max(nb, 1), mod=0.9, raw=raw, aa=aa, moments=moments, per_view=per_view)
    mv = np.stack([means] * V)
    if per_view:
        mv = mv + 0.01 * rng.randn(*mv.shape)
    d["means"] = mv.astype(f32)
    d["view"] = np.stack([c[0] for c in cams])
    d["proj"] = np.stack([c[1] for c in cams])
    d["campos"] = np.stack([c[2] for c in cams])
    d["tanx"] = np.array([c[3] for c in cams], f32)
    d["tany"] = np.array([c[4] for c in cams], f32)
    s32, op32 = s.astype(f32), op.astype(f32)
    d.update(op=op32, s=s32, q=q.astype(f32), shs=shs.astype(f32) if deg >= 0 else None,
             colors=None, var=None if var is None else var.astype(f32))
    if raw:
        d["qhat"], d["qnorm"], d["qlen"] = CH.normalize32(d["q"])
    else:
        d["qhat"], d["qnorm"], d["qlen"] = d["q"], np.ones(P, f32), np.ones(P, f32)
    d["op_prime"] = op32 if var is None else (op32 * CH.filter3d32(s32, d["var"])[3]).astype(f32)
    if cov:
        R = _rot(d["qhat"].astype(f64))
        L = R * (s32.astype(f64))[:, None, :]
        Sg = L @ L.transpose(0, 2, 1)
        d["cov"] = Sg[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(f32)
        d["var"] = None
    else:
        d["cov"] = None
    _forward32(d, rng)
    if normals and not cov:
        d["normals"] = dict(sign=np.where(rng.rand(V, P) < 0.5, -1.0, 1.0).astype(f32), wn=rng.randn(V, P, 3).astype(f32),
                            axis=np.argmin(s32, 1))
    return d


def _sphere(rng):
    x = rng.randn(3)
    return x / np.linalg.norm(x)


def _rot(q):
    r, x, y, z = q.T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                     np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                     np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)


def _forward32(d, rng):
    """radii, clamp bits, records and sums of a float32-ish forward: visible where tz > 0.2 and the centre within 1.5x the
    image; the record's conic and opacity from the chain's own float64 quantities rounded to float32"""
    P, V = d["P"], d["V"]
    radii = np.zeros((V, P), np.int32)
    recs = np.zeros((V, P, 12), f32)
    clamped = np.zeros((V, P), np.uint8)
    for v in range(V):
        x, y, z = (d["means"][v][:, k] for k in range(3))
        tz = CH.affine32(d["view"][v][[2, 6, 10, 14]], x, y, z)
        tx = CH.affine32(d["view"][v][[0, 4, 8, 12]], x, y, z)
        ty = CH.affine32(d["view"][v][[1, 5, 9, 13]], x, y, z)
        with np.errstate(divide="ignore", invalid="ignore"):
            inside = (np.abs(tx / tz) < 2.0 * d["tanx"][v]) & (np.abs(ty / tz) < 2.0 * d["tany"][v])
        radii[v] = np.where((tz > 0.2) & inside, 1 + rng.randint(0, 50, P), 0)
        recs[v, :, 4:7] = rng.uniform(0.01, 1.0, (P, 3)) * np.array([1, 0.1, 1])
        if d["deg"] >= 0:
            clamped[v] = rng.randint(0, 8, P) * (rng.rand(P) < 0.3)
    d.update(radii=radii, clamped=clamped, recs=recs)
    sums = rng.randn(V, P, 12).astype(f32)
    sums[..., 10:] = 0
    d["sums"] = sums
    if d["aa"]:  # F1's record opacity o' rho
        d["rho"], d["floored"] = CH.f1_rho(d)
        recs[..., 7] = (d["op_prime"] * d["rho"]).astype(f32)
    else:
        recs[..., 7] = d["op_prime"]


# ---- 1. against autograd ---------------------------------------------------------------------------------------------------
def _autograd(d):
    """the gradients of sum over views of <sums, (ndc x, ndc y, A, 2B, C, o, rgb, depth)> by float64 autograd, the record
    opacity and colour clamps taken from the same branch decisions chain() reads"""
    P, V, deg = d["P"], d["V"], d["deg"]
    T = lambda a: torch.tensor(np.asarray(a, f64), requires_grad=True)
    leaves = {}
    if d["raw"]:
        leaves["opacities"] = T(d["x_op"])
        op = torch.sigmoid(leaves["opacities"])
    else:
        leaves["opacities"] = T(d["op"])
        op = leaves["opacities"]
    cov_pre = d.get("cov")
    coef = torch.ones(P, dtype=torch.float64)
    if cov_pre is None:
        if d["raw"]:
            leaves["scales"], leaves["rotations"] = T(d["x_s"]), T(d["q"])
            s = torch.exp(leaves["scales"])
            q = torch.nn.functional.normalize(leaves["rotations"], dim=1)
        else:
            leaves["scales"], leaves["rotations"] = T(d["s"]), T(d["q"])
            s, q = leaves["scales"], leaves["rotations"]
        if d.get("var") is not None:
            t = s * s + torch.tensor(d["var"].astype(f64))[:, None]
            coef = torch.sqrt(((s * s) / t).prod(1))
            s = torch.sqrt(t)
        r, x, y, z = q.unbind(1)
        R = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                         torch.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                         torch.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)
        L = R * (CH.C(d["mod"]) * s)[:, None, :]
        Sig = L @ L.transpose(1, 2)
    else:
        leaves["cov3D"] = T(cov_pre)
        c = leaves["cov3D"]
        Sig = torch.stack([torch.stack([c[:, 0], c[:, 1], c[:, 2]], -1), torch.stack([c[:, 1], c[:, 3], c[:, 4]], -1),
                           torch.stack([c[:, 2], c[:, 4], c[:, 5]], -1)], 1)
    opp = op * coef
    if deg >= 0:
        leaves["shs"] = T(d["shs"][:, :(deg + 1) ** 2])
    else:
        leaves["colors"] = T(d["colors"])
    leaves["means3D"] = T(d["means"] if d["per_view"] else d["means"][0])
    loss = torch.zeros((), dtype=torch.float64)
    d["rho"], d["floored"] = np.zeros((V, P)), np.zeros((V, P), bool)  # the float64 forward's own, for chain()
    for v in range(V):
        m = leaves["means3D"][v] if d["per_view"] else leaves["means3D"]
        g = torch.tensor(d["sums"][v].astype(f64))
        vis = torch.tensor(d["radii"][v] > 0)
        Vm = torch.tensor(d["view"][v].reshape(4, 4).astype(f64))
        PVm = torch.tensor(d["proj"][v].reshape(4, 4).astype(f64))
        hom = torch.cat([m, torch.ones(P, 1, dtype=torch.float64)], 1)
        tc = hom @ Vm
        tx, ty, tz = tc[:, 0], tc[:, 1], tc[:, 2]
        tanx, tany = CH.C(d["tanx"][v]), CH.C(d["tany"][v])
        fx, fy = d["W"] / (2 * tanx), d["H"] / (2 * tany)
        bx, by = (torch.tensor(b) for b in CH.guard_band(d["means"][v], d["view"][v], tanx, tany))
        limx, limy = CH.C(f32(1.3) * f32(tanx)), CH.C(f32(1.3) * f32(tany))
        cx = torch.where(bx == 0, tx, (bx * limx * tz).detach())
        cy = torch.where(by == 0, ty, (by * limy * tz).detach())
        zero = torch.zeros(P, dtype=torch.float64)
        J = torch.stack([torch.stack([fx / tz, zero, -fx * cx / tz ** 2], -1), torch.stack([zero, fy / tz, -fy * cy / tz ** 2], -1)], 1)
        Tm = J @ Vm[:3, :3].T.expand(P, 3, 3)
        c2 = Tm @ Sig @ Tm.transpose(1, 2)
        a0, b_, c0 = c2[:, 0, 0], c2[:, 0, 1], c2[:, 1, 1]
        a, c = a0 + CH.C(0.3), c0 + CH.C(0.3)
        det = a * c - b_ * b_
        A, B, Cc = c / det, -b_ / det, a / det
        hp = hom @ PVm
        ndcx, ndcy = hp[:, 0] / (hp[:, 3] + CH.C(1e-7)), hp[:, 1] / (hp[:, 3] + CH.C(1e-7))
        orec = opp
        if d["aa"]:
            ratio = (a0 * c0 - b_ * b_) / det
            fl = ~(ratio > CH.RHO_FLOOR)
            rho = torch.sqrt(torch.where(fl, torch.full_like(ratio, CH.RHO_FLOOR), ratio))
            d["rho"][v], d["floored"][v] = rho.detach().numpy(), fl.numpy()
            orec = opp * rho
        if deg >= 0:
            dirs = m - torch.tensor(d["campos"][v].astype(f64))
            dirs = dirs / dirs.norm(dim=1, keepdim=True)
            bs = _basis64(deg, dirs)
            rgb = (bs[:, :, None] * leaves["shs"]).sum(1) + 0.5
            cl = torch.tensor(d["clamped"][v].astype(np.int64))
            keep = torch.stack([(cl >> k) & 1 == 0 for k in range(3)], 1)
            rgb = torch.where(keep, rgb, torch.zeros_like(rgb))
        else:
            rgb = leaves["colors"]
        terms = (g[:, 0] * ndcx + g[:, 1] * ndcy + g[:, 2] * A + 2 * g[:, 3] * B + g[:, 4] * Cc + g[:, 5] * orec +
                 (g[:, 6:9] * rgb).sum(1) + g[:, 9] * tz)
        loss = loss + torch.where(vis, terms, torch.zeros_like(terms)).sum()
        nrm = d.get("normals")
        if nrm is not None:
            col = R[torch.arange(P), :, torch.tensor(nrm["axis"])]
            wn = torch.tensor(nrm["wn"][v].astype(f64)) * torch.tensor(nrm["sign"][v].astype(f64))[:, None]
            loss = loss + torch.where(vis, (wn * col).sum(1), torch.zeros(P, dtype=torch.float64)).sum()
    loss.backward()
    return {k: t.grad.numpy() for k, t in leaves.items()}


def _basis64(deg, dirs):
    x, y, z = dirs.unbind(1)
    C1, C2, C3 = CH.SH_C1, CH.SH_C2, CH.SH_C3
    b = [torch.full_like(x, CH.SH_C0)]
    if deg > 0:
        b += [-C1 * y, C1 * z, -C1 * x]
    if deg > 1:
        xx, yy, zz = x * x, y * y, z * z
        b += [C2[0] * x * y, C2[1] * y * z, C2[2] * (2 * zz - xx - yy), C2[3] * x * z, C2[4] * (xx - yy)]
    if deg > 2:
        b += [C3[0] * y * (3 * xx - yy), C3[1] * x * y * z, C3[2] * y * (4 * zz - xx - yy), C3[3] * z * (2 * zz - 3 * xx - 3 * yy),
              C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy), C3[6] * x * (xx - 3 * yy)]
    return torch.stack(b, 1)


AUTOGRAD = [dict(deg=g, raw=r, aa=a, f3d=f, cov=c, per_view=pv, normals=n)
            for g, r, a, f, c, pv, n in ((-1, 0, 0, 0, 0, 0, 0), (0, 1, 1, 0, 0, 0, 0), (1, 0, 0, 1, 0, 1, 1), (2, 1, 1, 1, 0, 0, 1),
                                        (3, 1, 0, 0, 0, 1, 0), (3, 0, 1, 1, 0, 0, 0), (1, 0, 1, 0, 1, 0, 0), (3, 1, 1, 1, 0, 1, 1))]
# the edge scenes too (guard band, near plane, needles on both sides of the floor, clamped channels, quaternions of norm
# 1e-13, 1e-3 and 1e3): autograd of F.normalize confirms the g / 1e-12 rule below its eps independently of chain()
AUTOGRAD += [dict(deg=3, raw=1, aa=1, f3d=0, cov=0, per_view=0, normals=1, edges=1),
             dict(deg=1, raw=0, aa=1, f3d=0, cov=0, per_view=1, normals=0, edges=1)]


@pytest.mark.parametrize("opts", AUTOGRAD, ids=lambda o: "-".join(f"{k}{v}" for k, v in o.items()))
def test_against_autograd(opts):
    d = scene(200, 3, opts["deg"], seed=11 + opts["deg"], big=True, moments=False,
              **{k: bool(v) for k, v in opts.items() if k != "deg"})
    if d["deg"] < 0:
        d["colors"] = np.random.RandomState(3).rand(d["P"], 3).astype(f32)
    if d["raw"]:  # float64 activations for both sides
        d["x_op"] = np.log(d["op"].astype(f64) / (1 - d["op"]))
        d["x_s"] = np.log(d["s"].astype(f64))
        qn = np.linalg.norm(d["q"].astype(f64), axis=1)
        d["op"], d["s"] = 1 / (1 + np.exp(-d["x_op"])), np.exp(d["x_s"])
        d["qnorm"], d["qlen"] = np.maximum(qn, 1e-12), qn
        d["qhat"] = d["q"] / d["qnorm"][:, None]
    ag = _autograd(d)
    # autograd differentiates 1 / det^2 where the kernels use d2inv = 1 / (det^2 + 1e-7) (A.6): compare without the 1e-7,
    # which test_mutation_fails shows the check resolves
    got = CH.arrays(CH.chain(d, mutate=("eps7",)))
    names = dict(means3D="means3D", opacities="opacities", scales="scales", rotations="rotations", shs="shs", colors="colors",
                 cov3D="cov3D")
    for k, a in ag.items():
        r = got[names[k]][0].reshape(a.shape)
        assert np.abs(a).max() > 0, k
        # per Gaussian row: the edge rows' gradients span twenty orders of magnitude
        rows = lambda x: x.reshape(x.shape[0] * x.shape[1], -1) if x.ndim == 3 and k == "means3D" else x.reshape(x.shape[0], -1)
        ra, rr = rows(a), rows(r)
        err = (np.abs(rr - ra).max(1) / np.maximum(np.abs(ra).max(1), 1e-300)).max()
        assert err < 1e-11, f"{opts} {k}: chain vs autograd {err:.3g} relative"


# ---- 2. and 4. the bound holds, and how tight it is --------------------------------------------------------------------------
BOUND_SCENES = [dict(deg=3, raw=True, aa=True, f3d=True, edges=True, normals=True), dict(deg=1, aa=True, per_view=True, edges=True),
                dict(deg=2, raw=True, cov=True), dict(deg=-1, f3d=True, edges=True, moments=False),
                dict(deg=0, raw=True, normals=True, edges=True, moments=False)]


def _f32_out(d, num, mutate=()):
    return {k: v[0] for k, v in CH.arrays(CH.chain(d, num=num, mutate=mutate)).items()}


def _bound_scene(i, opts):
    d = scene(50_000, 5, opts["deg"], seed=100 + i, **{k: v for k, v in opts.items() if k != "deg"})
    if d["deg"] < 0:
        d["colors"] = np.random.RandomState(4).rand(d["P"], 3).astype(f32)
    return d


def test_bound_holds_and_tightness():
    samples = 0
    tight, unbounded = {}, {}
    for i, opts in enumerate(BOUND_SCENES):
        d = _bound_scene(i, opts)
        samples += int((d["radii"] > 0).sum())
        ref = CH.arrays(CH.chain(d))
        for num in (F32, F32Fma):
            out = _f32_out(d, num)
            for k, r in ref.items():
                CH.check(out[k], r, f"{opts} {num.__name__} {k}")
        for k, (v, e) in ref.items():
            nz = np.abs(v) > 0
            tight.setdefault(k, []).append((e[nz] / np.abs(v[nz])))
            unbounded[k] = unbounded.get(k, 0) + int((~np.isfinite(e)).sum())
    assert samples >= 1_000_000, samples
    print(f"\n{samples} (view, Gaussian) samples; e / |ref|: median, 99.9th percentile")
    for k, parts in tight.items():
        x = np.concatenate(parts)
        x = x[np.isfinite(x)]
        print(f"  {k:10s} {np.median(x):.3g}  {np.percentile(x, 99.9):.3g}   ({unbounded[k]} elements without a finite bound)")


# ---- 3. the check fails when it should ----------------------------------------------------------------------------------------
MUTATION_SCENE = dict(deg=3, raw=True, aa=True, f3d=True, edges=True, normals=True)


@pytest.mark.parametrize("mutation", CH.MUTATIONS)
def test_mutation_fails(mutation):
    opts = {k: v for k, v in MUTATION_SCENE.items() if k != "deg"}
    if mutation == "eps7":  # the filter's own terms dominate a sub-pixel Gaussian's scale gradient
        opts["f3d"] = False
    d = scene(4000, 3, 3, seed=7, **opts)
    ref = CH.arrays(CH.chain(d))
    out = _f32_out(d, F32, (mutation,))
    failed = []
    for k, r in ref.items():
        try:
            CH.check(out[k], r, k)
        except AssertionError as e:
            failed.append(str(e).split(":")[0])
    assert failed, f"mutation {mutation} passes the check"
    print(f"\n{mutation}: fails {failed}")
