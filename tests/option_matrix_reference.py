"""One float64 reference for every render option at once (TEST INFRASTRUCTURE ONLY), composed from the per-feature
references beside it:

  * images, per view on that view's own means: colour, depth, alpha and radii from the oracle (tests/aa_reference.py and
    tests/filter3d_reference.py wrap it for antialiasing and the 3D filter), the normal image from
    normal_reference.normal_image, and median, depth2 and median_pos from geometry_reference.replay, each on the oracle's
    state;
  * gradients: one float64 autograd loss per view through oracle/dense_ref.py (aa_reference.dense_render_aa with
    antialiasing), the sum of the main pass under (gC, gD, gA), the normal pass under gN (colours n, bg = 0), the z^2 pass
    under gM2 (colours (z^2, 0, 0), bg = 0) and the median term sum_p gMed_p z[g_med(p)].  Raw activations and the 3D filter
    are applied in float64 (as geometry_reference.reference_grads does); the normal's axis and flip come from the activated,
    unfiltered scales and the normalised rotation, taken from the raw arrays themselves for raw parameters.  Gradients of
    shared parameters are summed over the views; means3D keeps one row set per view when the means are per view, and
    means2D always does;
  * means2D_abs: absgrad_reference.absgrad per view with gN and gM2 (the median term is constant in means2D).

The integer decisions (radii, rects, depth order, the median's Gaussian) come from the oracle, as in every dense check."""
from __future__ import annotations

import numpy as np
import torch

import absgrad_reference as AR
import geometry_reference as GR
import normal_reference as NR
from contribution_reference import _oracle_state
from util import ROOT  # noqa: F401  (puts the repository root on sys.path)

f32 = np.float32
PARAMS = ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp")


def view_inputs(inps, means=None):
    """the oracle inputs of each view: inps[v], with means3D = means[v] when the means are per view ([V,P,3])"""
    return [inp if means is None else dict(inp, means3D=np.asarray(means[v], f32)) for v, inp in enumerate(inps)]


def gauss_normals(inp, raw=None):
    """[P,4] float32 (sign n, sign) of one view: from the raw scales and rotations when given, else from inp's"""
    if raw is not None:
        return NR.gauss_normals(inp["means3D"], inp["campos"], raw["scales"], raw["rotations"], raw=True)
    return NR.gauss_normals(inp["means3D"], inp["campos"], inp["scales"], inp["rotations"])


def images(inps, means=None, antialiasing=False, filter_3d=None, raw=None, normals=False, geometry=False):
    """dict of [V,...] float32 images (color, depth, alpha; normal; median, depth2, median_pos) and radii [V,P] int32"""
    out = {}
    for iv in view_inputs(inps, means):
        H, W = iv["image_height"], iv["image_width"]
        _, o, st = _oracle_state(iv, antialiasing, filter_3d)
        im = dict(color=np.asarray(o[0], f32).reshape(3, H, W), radii=np.asarray(o[1]).reshape(-1),
                  depth=np.asarray(o[2], f32).reshape(1, H, W), alpha=np.asarray(o[3], f32).reshape(1, H, W))
        if normals:
            im["normal"] = NR.normal_image(st, H, W, gauss_normals(iv, raw))
        if geometry:
            r = GR.replay(st, H, W)
            im.update(median=r["median"][None], depth2=r["depth2"][None], median_pos=r["median_pos"])
        for k, v in im.items():
            out.setdefault(k, []).append(v)
    return {k: np.stack(v) for k, v in out.items()}


def _activate(leaves, raw):
    if raw is None:
        return leaves["opacities"], leaves.get("scales"), leaves.get("rotations")
    if "scales" not in raw:  # cov3D_precomp: only the opacities are raw
        return torch.sigmoid(leaves["opacities"]), None, None
    return (torch.sigmoid(leaves["opacities"]), torch.exp(leaves["scales"]),
            torch.nn.functional.normalize(leaves["rotations"], dim=1))


def grads(inps, gimgs, gN=None, gM2=None, gMed=None, antialiasing=False, filter_3d=None, raw=None, means=None):
    """float64 gradients {name: array} of sum_v L_v (module docstring).  gimgs: per view (gC [3,H,W], gD [1,H,W], gA [1,H,W]);
    gN [V,3,H,W], gM2 / gMed [V,H,W] or None (a zero gradient).  raw: dict of raw opacities / scales / rotations (the
    gradients are then w.r.t. them).  means: [V,P,3] per-view means, or None for inps[0]["means3D"] shared."""
    from aa_reference import dense_render_aa
    from oracle.dense_ref import dense_render
    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    i0 = inps[0]
    V, P = len(inps), np.asarray(i0["means3D"]).shape[0]
    leaves = {k: t64(i0[k]).requires_grad_(True) for k in PARAMS if i0.get(k) is not None}
    for k, v in (raw or {}).items():
        leaves[k] = t64(v).requires_grad_(True)
    if means is not None:
        leaves["means3D"] = t64(means).requires_grad_(True)
    leaves["means2D"] = torch.zeros(V, P, 3, dtype=torch.float64, requires_grad=True)
    op, sc, q = _activate(leaves, raw)
    if filter_3d is not None:
        v = t64(filter_3d).reshape(-1, 1)
        t = sc * sc + v
        coef = torch.sqrt(torch.prod(sc * sc / t, 1))
        sc, op = torch.sqrt(t), op * coef.reshape(op.shape)
    if gN is not None:  # the axis from the activated, unfiltered scales (float32, as the kernels pick it)
        k_axis = NR.axis(NR.activate(raw["scales"], raw["rotations"], True)[0] if raw is not None else i0["scales"])
    render = dense_render_aa if antialiasing else dense_render
    zero3 = torch.zeros(3, dtype=torch.float64)
    L = 0.0
    for v, iv in enumerate(view_inputs(inps, means)):
        H, W = iv["image_height"], iv["image_width"]
        _, o, st = _oracle_state(iv, antialiasing, filter_3d)
        radii = np.asarray(o[1]).reshape(-1)
        ids = np.nonzero(radii > 0)[0]
        order = ids[np.lexsort((ids, st["depths"][ids]))]
        m3 = leaves["means3D"][v] if means is not None else leaves["means3D"]
        kw = dict(means3D=m3, means2D=leaves["means2D"][v], opacities=op, viewmatrix=t64(iv["viewmatrix"]),
                  projmatrix=t64(iv["projmatrix"]), campos=t64(iv["campos"]), H=H, W=W, tanfovx=iv["tanfovx"],
                  tanfovy=iv["tanfovy"], radii=radii, rect=st["rect"], order=order, scale_modifier=iv.get("scale_modifier", 1.0))
        if "cov3D_precomp" in leaves:
            kw["cov3D_precomp"] = leaves["cov3D_precomp"]
        else:
            kw.update(scales=sc, rotations=q)
        gC, gD, gA = (t64(g) for g in gimgs[v])
        if "shs" in leaves:
            c, d, a, _ = render(bg=t64(iv["bg"]), sh_degree=iv.get("sh_degree", 0), shs=leaves["shs"], **kw)
        else:
            c, d, a, _ = render(bg=t64(iv["bg"]), colors_precomp=leaves["colors_precomp"], **kw)
        L = L + (c * gC).sum() + (d * gD).sum() + (a * gA).sum()
        if gN is not None:
            n = NR.normals_torch(q, k_axis, gauss_normals(iv, raw)[:, 3])
            cn, _, _, _ = render(bg=zero3, colors_precomp=n, **kw)
            L = L + (cn * t64(gN[v])).sum()
        z = GR.view_depth64(m3, iv["viewmatrix"])
        if gM2 is not None:
            zc = torch.stack([z * z, torch.zeros_like(z), torch.zeros_like(z)], 1)
            cm, _, _, _ = render(bg=zero3, colors_precomp=zc, **kw)
            L = L + (cm[0] * t64(gM2[v]).reshape(H, W)).sum()
        if gMed is not None:
            mg = GR.replay(st, H, W)["median_gauss"]
            ys, xs = np.nonzero(mg >= 0)
            L = L + (t64(np.asarray(gMed[v]).reshape(H, W)[ys, xs]) * z[torch.as_tensor(mg[ys, xs])]).sum()
    L.backward()
    return {k: t.grad.numpy() for k, t in leaves.items()}


def means2D_abs(inps, gimgs, gN=None, gM2=None, antialiasing=False, filter_3d=None, means=None):
    """[V,P,3] float64: absgrad_reference.absgrad of each view (on its own means) with its gN and gM2"""
    return np.stack([AR.absgrad(iv, gimgs[v], antialiasing, filter_3d, None if gN is None else gN[v],
                                None if gM2 is None else gM2[v])[0] for v, iv in enumerate(view_inputs(inps, means))])


def reference(inps, gimgs, gN=None, gM2=None, gMed=None, antialiasing=False, filter_3d=None, raw=None, means=None,
              normals=False, geometry=False, absgrad=False):
    """(images, gradients) of one call: images(...) and grads(...), with "means2D_abs" among the gradients when absgrad"""
    im = images(inps, means, antialiasing, filter_3d, raw, normals, geometry)
    g = grads(inps, gimgs, gN, gM2, gMed, antialiasing, filter_3d, raw, means)
    if absgrad:
        g["means2D_abs"] = means2D_abs(inps, gimgs, gN, gM2, antialiasing, filter_3d, means)
    return im, g
