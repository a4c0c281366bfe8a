"""Reference of the normal maps (TEST INFRASTRUCTURE ONLY), beside the fixed oracle as aa_reference / contribution_reference.

  * per-Gaussian normals: numpy float32, the kernels' operation order restated with aa_reference.fma32 -- k = argmin of the
    activated scales (lowest index on a tie), n = column k of R(q) in the covariance's fmul / fma sequence, and the flip
    d = n . (campos - mean) as fmul, fma, fma over components 0, 1, 2;
  * the normal image: a replay of the blend on the oracle's state (the loop of contribution_reference.replay, which
    reproduces n_contrib and w bit for bit), accumulating N_c = fma(n_c, w, N_c);
  * gradients: oracle/dense_ref.py in float64 autograd, as the sum of two passes that share alpha and T -- the scene's colours
    under (gC, gD, gA), and colors_precomp = n_v(q) (the flip sign detached) with bg = 0 under gN.  dense_ref passes
    colors_precomp through unclamped, so the second pass's colour image is exactly sum w n."""
from __future__ import annotations

import numpy as np
import torch

from aa_reference import fma32
from contribution_reference import ALPHA_MAX, ALPHA_MIN, T_MIN, _fma, _gs_exp
from util import ROOT  # noqa: F401  (puts the repository root on sys.path)

f32 = np.float32


def activate(scales, rotations, raw=False):
    """(s, q) as F1 holds them: exp of raw scales, F.normalize of raw rotations (float32; the device's expf may differ in the
    last bit, which the GPU tests avoid by comparing against the GPU's own normals for raw parameters)"""
    s, q = np.asarray(scales, f32), np.asarray(rotations, f32)
    if raw:
        s = np.exp(s).astype(f32)
        n2 = ((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]).astype(f32) + (q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3]).astype(f32)).astype(f32)
        q = (q / np.maximum(np.sqrt(n2), f32(1e-12))[:, None]).astype(f32)
    return s, q


def axis(s):
    """argmin of each row of s, the lowest index on a tie"""
    s = np.asarray(s, f32)
    k = np.zeros(len(s), np.int64)
    k = np.where(s[:, 1] < s[np.arange(len(s)), k], 1, k)
    k = np.where(s[:, 2] < s[np.arange(len(s)), k], 2, k)
    return k


def rot_columns(q):
    """R(q) [P,3,3] in gs_rotmat's float32 sequence"""
    q = np.asarray(q, f32)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    m = lambda a, b: (a * b).astype(f32)
    R = np.empty((len(q), 3, 3), f32)
    R[:, 0, 0] = fma32(-2.0, fma32(z, z, m(y, y)), 1.0)
    R[:, 0, 1] = m(2.0, fma32(x, y, -m(r, z)))
    R[:, 0, 2] = m(2.0, fma32(x, z, m(r, y)))
    R[:, 1, 0] = m(2.0, fma32(x, y, m(r, z)))
    R[:, 1, 1] = fma32(-2.0, fma32(z, z, m(x, x)), 1.0)
    R[:, 1, 2] = m(2.0, fma32(y, z, -m(r, x)))
    R[:, 2, 0] = m(2.0, fma32(x, z, -m(r, y)))
    R[:, 2, 1] = m(2.0, fma32(y, z, m(r, x)))
    R[:, 2, 2] = fma32(-2.0, fma32(y, y, m(x, x)), 1.0)
    return R


def gauss_normals(means3D, campos, scales, rotations, raw=False):
    """[P,4] float32 (sign n, sign) of one view, as normal_prep_kernel writes it.  means3D [P,3] (this view's positions)."""
    s, q = activate(scales, rotations, raw)
    k = axis(s)
    n = rot_columns(q)[np.arange(len(q)), :, k]  # column k
    e = (np.asarray(campos, f32).reshape(1, 3) - np.asarray(means3D, f32)).astype(f32)
    with np.errstate(invalid="ignore"):
        d = fma32(n[:, 2], e[:, 2], fma32(n[:, 1], e[:, 1], (n[:, 0] * e[:, 0]).astype(f32)))
    sg = np.where(d < 0, f32(-1), f32(1)).astype(f32)
    return np.concatenate([n * sg[:, None], sg[:, None]], 1).astype(f32)


def normal_image(st, H, W, nrm):
    """[3,H,W] float32: the blend of one view replayed on the oracle state `st` with N_c = fma(n_c, w, N_c), nrm [P,>=3]"""
    gx = (W + 15) // 16
    xy, co, pl = st["xy"], st["conic_opacity"], st["point_list"]
    nrm = np.asarray(nrm, f32)
    out = np.zeros((3, H, W), f32)
    for t, (r0, r1) in enumerate(st["ranges"]):
        if r1 <= r0:
            continue
        ys, xs = np.mgrid[(t // gx) * 16:(t // gx) * 16 + 16, (t % gx) * 16:(t % gx) * 16 + 16]
        keep = (ys < H) & (xs < W)
        ys, xs = ys[keep], xs[keep]
        fx, fy = xs.astype(f32), ys.astype(f32)
        T = np.ones(len(xs), f32)
        alive = np.ones(len(xs), bool)
        N = np.zeros((3, len(xs)), f32)
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
                for c in range(3):
                    N[c, blend] = fma32(nrm[g, c], w, N[c, blend])
            alive &= ~term
            T = np.where(blend, test_T, T)
        out[:, ys, xs] = N
    return out


def oracle_state(inp, antialiasing=False, filter_3d=None):
    """(state, radii) of the oracle for one view; antialiasing and the 3D filter come in through their wrappers"""
    from contribution_reference import _oracle_state
    o, out, st = _oracle_state(inp, antialiasing, filter_3d)
    return st, np.asarray(out[1]).reshape(-1)


def reference_image(inp, antialiasing=False, filter_3d=None, nrm=None):
    """[3,H,W] float32 normal image of one view (nrm: per-Gaussian normals to use in place of gauss_normals(inp))"""
    st, _ = oracle_state(inp, antialiasing, filter_3d)
    if nrm is None:
        nrm = gauss_normals(inp["means3D"], inp["campos"], inp["scales"], inp["rotations"])
    return normal_image(st, inp["image_height"], inp["image_width"], nrm)


def normals_torch(q, k, sign):
    """torch n [P,3] in q's dtype and device: column k of R(q) times the (detached) flip sign; q [P,4] as the covariance uses
    it"""
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    n = R[torch.arange(len(q), device=q.device), :, torch.as_tensor(k, device=q.device)]
    return n * torch.as_tensor(sign, dtype=q.dtype, device=q.device)[:, None]


def reference_grads(inp, gimg, gN, antialiasing=False, filter_3d=None, raw=None):
    """float64 gradients {name: array} of L = sum gC c + gD d + gA a + sum gN N for one view, by autograd through
    oracle/dense_ref.py (two passes sharing alpha and T).  raw: dict of raw opacities / scales / rotations; the gradients are
    then w.r.t. them.  filter_3d: [P] variances, applied in float64 (gradients w.r.t. the unfiltered parameters)."""
    from oracle.dense_ref import dense_render
    from aa_reference import dense_render_aa
    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    leaves = {k: t64(inp[k]).requires_grad_(True) for k in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations")
              if inp.get(k) is not None}
    if raw is not None:
        for k, v in raw.items():
            leaves[k] = t64(v).requires_grad_(True)
        op = torch.sigmoid(leaves["opacities"])
        sc = torch.exp(leaves["scales"])
        q = torch.nn.functional.normalize(leaves["rotations"], dim=1)
    else:
        op, sc, q = leaves["opacities"], leaves["scales"], leaves["rotations"]
    # the integer decisions and the flip come from float32 (the oracle and gauss_normals); the state is the filtered one
    gn32 = gauss_normals(inp["means3D"], inp["campos"], inp["scales"], inp["rotations"])
    k = axis(np.asarray(inp["scales"], f32))
    if filter_3d is not None:
        v = t64(filter_3d).reshape(-1, 1)
        t = sc * sc + v
        coef = torch.sqrt(torch.prod(sc * sc / t, 1))
        sc, op = torch.sqrt(t), op * coef.reshape(op.shape)
    st, radii = oracle_state(inp, antialiasing, filter_3d)
    ids = np.nonzero(radii > 0)[0]
    order = ids[np.lexsort((ids, st["depths"][ids]))]
    H, W = inp["image_height"], inp["image_width"]
    kw = dict(means3D=leaves["means3D"], means2D=torch.zeros(len(radii), 3, dtype=torch.float64), opacities=op,
              viewmatrix=t64(inp["viewmatrix"]), projmatrix=t64(inp["projmatrix"]), campos=t64(inp["campos"]), H=H, W=W,
              tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], radii=radii, rect=st["rect"], order=order, scales=sc, rotations=q,
              scale_modifier=inp.get("scale_modifier", 1.0))
    render = dense_render_aa if antialiasing else dense_render
    gC, gD, gA = (t64(g) for g in gimg)
    if "shs" in leaves:
        c, d, a, _ = render(bg=t64(inp["bg"]), sh_degree=inp.get("sh_degree", 0), shs=leaves["shs"], **kw)
    else:
        c, d, a, _ = render(bg=t64(inp["bg"]), colors_precomp=leaves["colors_precomp"], **kw)
    L = (c * gC).sum() + (d * gD).sum() + (a * gA).sum()
    n = normals_torch(q, k, gn32[:, 3])
    cn, _, _, _ = render(bg=torch.zeros(3, dtype=torch.float64), colors_precomp=n, **kw)
    L = L + (cn * t64(gN)).sum()
    L.backward()
    return {k: v.grad.numpy() for k, v in leaves.items()}, cn.detach().numpy()
