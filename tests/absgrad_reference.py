"""Reference of the absolute screen-space gradient (TEST INFRASTRUCTURE ONLY): sum_p |dL_p / dmeans2D| in float64.

A Gaussian's 2D mean reaches pixel p only through its alpha at p, so the signed gradient dL/dmeans2D = sum_p g_p splits
into per-pixel terms g_p = dL_p / dmeans2D, L_p = sum_c gout_c[p] out_c[p] (colour, depth and alpha channels).  The
reference takes them by forward-mode autograd through oracle/dense_ref.py (whose means2D is the additive NDC offset the
kernels' dL_dmeans2D is w.r.t.), or aa_reference.dense_render_aa with the screen-space filter: one jvp per tangent gives
dL_p / dmeans2D[k, c] for every pixel p at once.  Tangents of Gaussians whose tile rects are disjoint share one jvp -- dense_ref
masks every (pixel, Gaussian) pair outside the rect, so each pixel's tangent then comes from at most one of them.  It shares
no code with the kernels.

The integer decisions (radii, rects, depth order) come from the oracle, as in tests/test_oracle_autograd.py."""
from __future__ import annotations

import numpy as np
import torch

from util import ROOT  # noqa: F401  (puts the repository root on sys.path)


def _state(inp, antialiasing=False):
    from aa_reference import AAOracle
    o = AAOracle(threads=1)
    _, radii, _, _ = o.forward(antialiasing=antialiasing, **inp)
    return o.state(), np.asarray(radii).reshape(-1)


def _rect_colors(rect, ids):
    """greedy colouring of the Gaussians `ids` such that the tile rects of one colour are pairwise disjoint"""
    colors, occ = [], []
    for k in ids:
        x0, y0, x1, y1 = (int(v) for v in rect[k])
        for c, grid in enumerate(occ):
            if not grid[y0:y1, x0:x1].any():
                grid[y0:y1, x0:x1] = True
                colors[c].append(k)
                break
        else:
            grid = np.zeros((int(rect[:, 3].max()) + 1, int(rect[:, 2].max()) + 1), bool)
            grid[y0:y1, x0:x1] = True
            occ.append(grid)
            colors.append([k])
    return colors


def pixel_losses(inp, gimg, antialiasing=False, filter_3d=None, gN=None, gM2=None):
    """(losses, state, radii): losses(m2d) is the [H*W] float64 tensor of L_p for the NDC offsets m2d [P,3], one view of
    `inp` (the oracle's activated inputs).  L_p = gC.c + gD d + gA a at p, plus with gN [3,H,W] the normal pass gN.N (n the
    shortest-scale axis of the unfiltered scales, flipped to face the camera, bg = 0) and with gM2 [H,W] the depth second
    moment gM2 M2 (colours (z^2, 0, 0), bg = 0).  filter_3d: [P] variances; the 3D filter's s', o' are formed as the kernels
    form them (filter3d_reference.filter_params)."""
    from oracle.dense_ref import dense_render
    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    if gN is not None:  # the axis and the flip come from the unfiltered activated parameters
        import normal_reference as NR
        sign = NR.gauss_normals(inp["means3D"], inp["campos"], inp["scales"], inp["rotations"])[:, 3]
        nrm = NR.normals_torch(t64(inp["rotations"]), NR.axis(inp["scales"]), sign)
    if filter_3d is not None:
        from filter3d_reference import filter_params
        sp, op, _ = filter_params(inp["scales"], inp["opacities"], filter_3d)
        inp = dict(inp, scales=sp, opacities=op)
    st, radii = _state(inp, antialiasing)
    H, W = inp["image_height"], inp["image_width"]
    ids = np.nonzero(radii > 0)[0]
    order = ids[np.lexsort((ids, st["depths"][ids]))]
    kw = dict(means3D=t64(inp["means3D"]), opacities=t64(inp["opacities"]), viewmatrix=t64(inp["viewmatrix"]),
              projmatrix=t64(inp["projmatrix"]), campos=t64(inp["campos"]), H=H, W=W, tanfovx=inp["tanfovx"],
              tanfovy=inp["tanfovy"], radii=radii, rect=st["rect"], order=order, scale_modifier=inp.get("scale_modifier", 1.0))
    for k in ("scales", "rotations", "cov3D_precomp"):
        if inp.get(k) is not None:
            kw[k] = t64(inp[k])
    colours = dict(bg=t64(inp["bg"]), sh_degree=inp.get("sh_degree", 0))
    for k in ("shs", "colors_precomp"):
        if inp.get(k) is not None:
            colours[k] = t64(inp[k])
    if antialiasing:
        from aa_reference import dense_render_aa as render
    else:
        render = dense_render
    gC, gD, gA = (t64(g) for g in gimg)
    zero = torch.zeros(3, dtype=torch.float64)
    if gM2 is not None:
        from geometry_reference import view_depth64
        z = view_depth64(kw["means3D"], inp["viewmatrix"])
        z2 = torch.stack([z * z, torch.zeros_like(z), torch.zeros_like(z)], 1)

    def losses(m2d):
        c, d, a, _ = render(means2D=m2d, **colours, **kw)
        Lp = (c * gC).sum(0) + (d * gD)[0] + (a * gA)[0]
        if gN is not None:
            cn, _, _, _ = render(means2D=m2d, bg=zero, colors_precomp=nrm, **kw)
            Lp = Lp + (cn * t64(gN)).sum(0)
        if gM2 is not None:
            cm, _, _, _ = render(means2D=m2d, bg=zero, colors_precomp=z2, **kw)
            Lp = Lp + cm[0] * t64(gM2).reshape(H, W)
        return Lp.reshape(-1)  # L_p, [H*W]

    return losses, st, radii


def per_pixel_jacobian(inp, gimg, antialiasing=False, filter_3d=None, gN=None, gM2=None):
    """dense [P, 2, H*W] float64 array J with J[k, c, p] = dL_p / dmeans2D[k, c] (NDC units), for one view of `inp` (the
    oracle's activated inputs) under the image gradients gimg = (gC [3,H,W], gD [1,H,W], gA [1,H,W]), and with gN / gM2 the
    normal and depth-second-moment terms of L_p (pixel_losses; a median gradient is constant in means2D and adds nothing)."""
    losses, st, radii = pixel_losses(inp, gimg, antialiasing, filter_3d, gN, gM2)
    H, W = inp["image_height"], inp["image_width"]
    P = len(radii)
    ids = np.nonzero(radii > 0)[0]
    J = np.zeros((P, 2, H * W))
    rect = np.asarray(st["rect"]).reshape(P, 4)
    m0 = torch.zeros(P, 3, dtype=torch.float64)
    ys, xs = np.divmod(np.arange(H * W), W)
    for group in _rect_colors(rect, ids):
        for c in range(2):
            tan = torch.zeros(P, 3, dtype=torch.float64)
            tan[group, c] = 1.0
            _, dL = torch.func.jvp(losses, (m0,), (tan,))
            dL = dL.numpy()
            for k in group:  # pixel p of the group's output belongs to the one Gaussian whose rect holds it
                x0, y0, x1, y1 = (int(v) for v in rect[k])
                inr = (xs // 16 >= x0) & (xs // 16 < x1) & (ys // 16 >= y0) & (ys // 16 < y1)
                J[k, c, inr] = dL[inr]
    return J, radii


def absgrad(inp, gimg, antialiasing=False, filter_3d=None, gN=None, gM2=None):
    """(abs [P,3], signed [P,3], radii): sum_p |g_p| and sum_p g_p per component, z = 0 (float64)"""
    J, radii = per_pixel_jacobian(inp, gimg, antialiasing, filter_3d, gN, gM2)
    P = J.shape[0]
    a, s = np.zeros((P, 3)), np.zeros((P, 3))
    a[:, :2] = np.abs(J).sum(2)
    s[:, :2] = J.sum(2)
    return a, s, radii
