"""Reference of the geometry outputs (TEST INFRASTRUCTURE ONLY), beside normal_reference / contribution_reference.

  * images: a replay of the blend on the oracle's state (the loop of contribution_reference.replay, which reproduces n_contrib
    and w bit for bit) that accumulates M2 = fma(d * d, w, M2) and takes as the median the last blend whose T before it is
    > 0.5, with its 1-based list position and its Gaussian;
  * the W3 fold: per Gaussian, the float64 sum of w gD + 2 d w gM2 over its blends plus gMed over the pixels whose median it is,
    and the first-order error bound E of the kernel's float32 sum (DESIGN.md section 2, "Geometry outputs");
  * gradients: oracle/dense_ref.py in float64 autograd, as the sum of the scene's pass under (gC, gD, gA), a pass with
    colors_precomp = (z^2, 0, 0) and bg = 0 under gM2 (z the float64 view-space depth of means3D; dense_ref passes colours
    through unclamped, so its colour image is exactly sum w z^2), and sum_p gMed_p z[g_med(p)] with g_med from the replay."""
from __future__ import annotations

import numpy as np
import torch

from aa_reference import fma32
from contribution_reference import ALPHA_MAX, ALPHA_MIN, T_MIN, _fma, _gs_exp
from util import ROOT  # noqa: F401  (puts the repository root on sys.path)

f32 = np.float32


def replay(st, H, W, depths=None, gD=None, gM2=None, gMed=None, lists=False):
    """One view on the oracle state `st` (or a dict with xy, conic_opacity, point_list, ranges and depths).  Returns a dict of
    median [H,W] f32, depth2 [H,W] f32, median_pos [H,W] u32 (1-based list position, 0 = none), median_gauss [H,W] int64
    (-1 = none).  With gD, gM2, gMed ([H,W] f32): also W3 [P] float64, the fold's float64 sum, and E [P] float64, the
    sum over its terms of |term| (r + 4 + N_g) with r the term's replay depth from the back and N_g the Gaussian's number of
    (instance, patch) partials.  lists=True: also "blends", {(y, x): [(w, d), ...]} in blend order."""
    gx = (W + 15) // 16
    xy, co, pl = st["xy"], st["conic_opacity"], st["point_list"]
    d = np.asarray(st["depths"] if depths is None else depths, f32)
    P = len(xy)
    med = np.zeros((H, W), f32)
    M2 = np.zeros((H, W), f32)
    mpos = np.zeros((H, W), np.uint32)
    mg = np.full((H, W), -1, np.int64)
    fold = gD is not None
    blends = {}
    if fold:
        W3 = np.zeros(P, np.float64)
        terms = []  # (gaussian, |term|, pixel y, pixel x, order of the blend in its pixel) for the bound
        patches = {}  # instance j -> patch bits that blended it
    for t, (r0, r1) in enumerate(st["ranges"]):
        if r1 <= r0:
            continue
        ys, xs = np.mgrid[(t // gx) * 16:(t // gx) * 16 + 16, (t % gx) * 16:(t % gx) * 16 + 16]
        keep = (ys < H) & (xs < W)
        ys, xs = ys[keep], xs[keep]
        fx, fy = xs.astype(f32), ys.astype(f32)
        pbit = (1 << (((ys % 16) // 4) * 2 + (xs % 16) // 8)).astype(np.uint8)
        T = np.ones(len(xs), f32)
        alive = np.ones(len(xs), bool)
        m2 = np.zeros(len(xs), f32)
        nb = np.zeros(len(xs), np.int64)
        for j in range(r0, r1):
            if not alive.any():
                break
            g = pl[j]
            A, B, C, op = co[g]
            dx, dy = (xy[g, 0] - fx).astype(f32), (xy[g, 1] - fy).astype(f32)
            u = _fma(-B, dy, (f32(-0.5) * A * dx).astype(f32))
            w2 = ((f32(-0.5) * C * dy).astype(f32) * dy).astype(f32)
            power = _fma(dx, u, w2)
            alpha = np.minimum(ALPHA_MAX, (op * _gs_exp(np.minimum(power, f32(0)))).astype(f32))
            test_T = (T * (f32(1) - alpha)).astype(f32)
            touch = alive & (power <= 0) & (alpha >= ALPHA_MIN)
            term = touch & (test_T < T_MIN)
            blend = touch & ~term
            if blend.any():
                w = (alpha[blend] * T[blend]).astype(f32)
                m2[blend] = fma32((d[g] * d[g]).astype(f32), w, m2[blend])
                ism = blend & (T > f32(0.5))
                med[ys[ism], xs[ism]] = d[g]
                mpos[ys[ism], xs[ism]] = j - r0 + 1
                mg[ys[ism], xs[ism]] = g
                nb[blend] += 1
                if lists:
                    for y, x, wi in zip(ys[blend], xs[blend], w):
                        blends.setdefault((int(y), int(x)), []).append((wi, d[g]))
                if fold:
                    by, bx = ys[blend], xs[blend]
                    wd = w.astype(np.float64)
                    t3 = wd * gD[by, bx] + 2.0 * float(d[g]) * wd * gM2[by, bx]
                    W3[g] += t3.sum()
                    mag = np.abs(wd * gD[by, bx]) + np.abs(2.0 * float(d[g]) * wd * gM2[by, bx])
                    terms += [(g, m, y, x, k) for m, y, x, k in zip(mag, by, bx, nb[blend])]
                    patches[j] = int(np.bitwise_or.reduce(pbit[blend]))
            alive &= ~term
            T = np.where(blend, test_T, T)
        M2[ys, xs] = m2
    out = dict(median=med, depth2=M2, median_pos=mpos, median_gauss=mg)
    if lists:
        out["blends"] = blends
    if fold:
        nblend = np.zeros((H, W), np.int64)
        for _, _, y, x, k in terms:
            nblend[y, x] = max(nblend[y, x], k)
        Ng = np.zeros(P, np.int64)
        for j, bits in patches.items():
            Ng[pl[j]] += bin(bits).count("1")
        E = np.zeros(P, np.float64)
        for g, m, y, x, k in terms:
            E[g] += m * (nblend[y, x] - k + 1 + 4 + Ng[g])
        ys, xs = np.nonzero(mg >= 0)
        for y, x in zip(ys, xs):
            g = mg[y, x]
            W3[g] += float(gMed[y, x])
            E[g] += abs(float(gMed[y, x])) * (nblend[y, x] + 4 + Ng[g])
        out.update(W3=W3, E=E, N_g=Ng)
    return out


def oracle_state(inp, antialiasing=False, filter_3d=None):
    from contribution_reference import _oracle_state
    o, out, st = _oracle_state(inp, antialiasing, filter_3d)
    return st, np.asarray(out[1]).reshape(-1)


def reference_images(inp, antialiasing=False, filter_3d=None):
    """replay(...) of one view on the oracle's state"""
    st, _ = oracle_state(inp, antialiasing, filter_3d)
    return replay(st, inp["image_height"], inp["image_width"])


def view_depth64(means3D, viewmatrix):
    """float64 view-space z of each mean (row-vector view matrix: z = m . V[:3,2] + V[3,2]), differentiable in means3D"""
    V = torch.as_tensor(np.asarray(viewmatrix, np.float64)).reshape(4, 4).to(means3D)
    return means3D @ V[:3, 2] + V[3, 2]


def reference_grads(inp, gimg, gM2, gMed, antialiasing=False, filter_3d=None, raw=None, gN=None):
    """float64 gradients {name: array} of L = sum gC c + gD d + gA a + sum gM2 M2 + sum gMed median (+ sum gN N with gN) for
    one view, by autograd through oracle/dense_ref.py.  raw: dict of raw opacities / scales / rotations (gradients w.r.t.
    them).  filter_3d: [P] variances applied in float64 (gradients w.r.t. the unfiltered parameters)."""
    from oracle.dense_ref import dense_render
    from aa_reference import dense_render_aa
    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    leaves = {k: t64(inp[k]).requires_grad_(True) for k in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations",
                                                            "cov3D_precomp") if inp.get(k) is not None}
    if raw is not None:
        for k, v in raw.items():
            leaves[k] = t64(v).requires_grad_(True)
        op = torch.sigmoid(leaves["opacities"])
        sc = torch.exp(leaves["scales"])
        q = torch.nn.functional.normalize(leaves["rotations"], dim=1)
    else:
        op, sc, q = leaves["opacities"], leaves.get("scales"), leaves.get("rotations")
    if filter_3d is not None:
        v = t64(filter_3d).reshape(-1, 1)
        t = sc * sc + v
        coef = torch.sqrt(torch.prod(sc * sc / t, 1))
        sc, op = torch.sqrt(t), op * coef.reshape(op.shape)
    st, radii = oracle_state(inp, antialiasing, filter_3d)
    H, W = inp["image_height"], inp["image_width"]
    rp = replay(st, H, W)
    ids = np.nonzero(radii > 0)[0]
    order = ids[np.lexsort((ids, st["depths"][ids]))]
    kw = dict(means3D=leaves["means3D"], means2D=torch.zeros(len(radii), 3, dtype=torch.float64), opacities=op,
              viewmatrix=t64(inp["viewmatrix"]), projmatrix=t64(inp["projmatrix"]), campos=t64(inp["campos"]), H=H, W=W,
              tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], radii=radii, rect=st["rect"], order=order,
              scale_modifier=inp.get("scale_modifier", 1.0))
    if "cov3D_precomp" in leaves:
        kw["cov3D_precomp"] = leaves["cov3D_precomp"]
    else:
        kw.update(scales=sc, rotations=q)
    render = dense_render_aa if antialiasing else dense_render
    gC, gD, gA = (t64(g) for g in gimg)
    if "shs" in leaves:
        c, d, a, _ = render(bg=t64(inp["bg"]), sh_degree=inp.get("sh_degree", 0), shs=leaves["shs"], **kw)
    else:
        c, d, a, _ = render(bg=t64(inp["bg"]), colors_precomp=leaves["colors_precomp"], **kw)
    L = (c * gC).sum() + (d * gD).sum() + (a * gA).sum()
    z = view_depth64(leaves["means3D"], inp["viewmatrix"])
    zc = torch.stack([z * z, torch.zeros_like(z), torch.zeros_like(z)], 1)
    cm, _, _, _ = render(bg=torch.zeros(3, dtype=torch.float64), colors_precomp=zc, **kw)
    L = L + (cm[0] * t64(gM2).reshape(H, W)).sum()
    mg = rp["median_gauss"]
    ys, xs = np.nonzero(mg >= 0)
    L = L + (t64(np.asarray(gMed).reshape(H, W)[ys, xs]) * z[torch.as_tensor(mg[ys, xs])]).sum()
    if gN is not None:
        import normal_reference as NR
        gn32 = NR.gauss_normals(inp["means3D"], inp["campos"], inp["scales"], inp["rotations"])
        n = NR.normals_torch(q, NR.axis(np.asarray(inp["scales"], f32)), gn32[:, 3])
        cn, _, _, _ = render(bg=torch.zeros(3, dtype=torch.float64), colors_precomp=n, **kw)
        L = L + (cn * t64(gN)).sum()
    L.backward()
    return {k: v.grad.numpy() for k, v in leaves.items()}, cm[0].detach().numpy()
