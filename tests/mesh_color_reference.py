"""numpy restatement of the field query (DESIGN.md section 2; mesh.query_field, b200gs_field_query), written from the
definition, not from the CUDA.  Membership, samples and relax come from mesh_reference; the sums are taken in float64.

Each evaluation also returns, per output, the sum of the absolute values of its terms, so a test can bound a float32
result by k * sum|terms|.
"""
from __future__ import annotations

import numpy as np

import mesh_reference as M

f32 = np.float32
SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
SH_C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435]


def sh_basis(deg, d):
    """[n,(deg+1)^2] real SH basis along unit directions d [n,3] (sh_utils.py's order and signs), float64."""
    d = np.asarray(d, np.float64)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    b = [np.full(len(d), SH_C0)]
    if deg > 0:
        b += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b += [SH_C2[0] * xy, SH_C2[1] * yz, SH_C2[2] * (2 * zz - xx - yy), SH_C2[3] * xz, SH_C2[4] * (xx - yy)]
    if deg > 2:
        b += [SH_C3[0] * y * (3 * xx - yy), SH_C3[1] * xy * z, SH_C3[2] * y * (4 * zz - xx - yy),
              SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * zz - xx - yy), SH_C3[5] * z * (xx - yy),
              SH_C3[6] * x * (xx - 3 * yy)]
    return np.stack(b, 1)


def color(mean_sh, deg, dirs, sh_abs=None):
    """max(SH(mean_sh, dirs) + 0.5, 0) [n,3] for mean coefficients mean_sh [n,K,3]; dirs [n,3] unit or 0 (0: DC alone).
    With sh_abs [n,K,3] (the weighted mean of |sh|), also returns sum|terms| per channel."""
    dirs = np.asarray(dirs, np.float64)
    b = sh_basis(deg, dirs)
    b[~np.any(dirs != 0, 1), 1:] = 0.0
    nc = (deg + 1) ** 2
    col = np.maximum(np.einsum("nk,nkc->nc", b, mean_sh[:, :nc]) + 0.5, 0.0)
    if sh_abs is None:
        return col
    return col, np.einsum("nk,nkc->nc", np.abs(b), sh_abs[:, :nc]) + 0.5


def home(lin, split, nch, q):
    """h(q): the largest chunk c with c == 0 or lin[c*split] <= q, per coordinate."""
    starts = lin[np.arange(nch) * split]
    return np.maximum(np.searchsorted(starts, q, side="right") - 1, 0)


class Query:
    """The field query of one Gaussian set: mesh_reference.Field's kept set, frame and blocks, and SH shs [P,K,3] of all
    P Gaussians (None: no colour) evaluated at degree sh_degree."""

    def __init__(self, xyz, opacity, scaling, rotation, resolution, num_blocks=16, relax_ratio=1.5, shs=None, sh_degree=0,
                 raw=True):
        self.F = M.Field(xyz, opacity, scaling, rotation, resolution, num_blocks, relax_ratio, raw)
        op = np.asarray(opacity, f32).reshape(-1)
        keep = (f32(1) / (f32(1) + np.exp(-op)) if raw else op) > f32(0.005)  # mesh_reference.prepare's rule
        self.sh = None if shs is None else np.asarray(shs, np.float64)[keep]
        self.deg = sh_degree

    def eval(self, q):
        """q [n,3] float32 in the field's frame -> dict of D, G [n,3], normal [n,3], mean_sh [n,K,3] (or None), and the
        sums of term magnitudes D_abs = sum w (1 + P), G_abs [n,3] = sum w (1 + P) |Sigma^-1 d| with P the sum of the
        magnitudes of the exponent's terms, sh_abs [n,K,3] = sum w |sh| / D."""
        F = self.F
        q = np.asarray(q, f32)
        n = len(q)
        D = np.zeros(n)
        D_abs = np.zeros(n)
        G = np.zeros((n, 3))
        G_abs = np.zeros((n, 3))
        K = 0 if self.sh is None else self.sh.shape[1]
        S = np.zeros((n, K, 3))
        S_abs = np.zeros((n, K, 3))
        h = np.stack([home(F.lin, F.split, F.nch, q[:, a]) for a in range(3)], 1)
        for b in np.unique(h, axis=0):
            sel = np.nonzero(np.all(h == b, 1))[0]
            idx = M._block_members(F.x, F.lin, F.res, F.split, F.relax, *b)
            if len(idx) == 0:
                continue
            d = q[sel, None, :].astype(np.float64) - F.x[None, idx].astype(np.float64)
            ia, ib, ic, id_, ie, if_ = (F.inv[idx, k].astype(np.float64)[None] for k in range(6))
            dx, dy, dz = d[..., 0], d[..., 1], d[..., 2]
            p = -0.5 * (dx * dx * ia + dy * dy * id_ + dz * dz * if_) - dx * dy * ib - dx * dz * ic - dy * dz * ie
            w = np.where((p > 0) | (p <= -104), 0.0, np.exp(np.minimum(p, 0.0))) * F.op[idx].astype(np.float64)[None]
            # a float32 exponent is off by a few ulp of the sum of its terms' magnitudes (it cancels for thin
            # Gaussians), and w by that much relatively: each weight's term counts (1 + sum|terms of p|) times
            p_abs = 0.5 * (dx * dx * np.abs(ia) + dy * dy * np.abs(id_) + dz * dz * np.abs(if_)) + np.abs(dx * dy * ib) + \
                np.abs(dx * dz * ic) + np.abs(dy * dz * ie)
            Ad = np.stack([ia * dx + ib * dy + ic * dz, ib * dx + id_ * dy + ie * dz, ic * dx + ie * dy + if_ * dz], -1)
            D[sel] = w.sum(1)
            D_abs[sel] = (w * (1 + p_abs)).sum(1)
            G[sel] = -np.einsum("nm,nmc->nc", w, Ad)
            G_abs[sel] = np.einsum("nm,nmc->nc", w * (1 + p_abs), np.abs(Ad))
            if K:
                S[sel] = np.einsum("nm,mkc->nkc", w, self.sh[idx])
                S_abs[sel] = np.einsum("nm,mkc->nkc", w, np.abs(self.sh[idx]))
        norm = np.linalg.norm(G, axis=1)
        with np.errstate(invalid="ignore", divide="ignore"):
            normal = np.where((norm > 0)[:, None], -G / norm[:, None], 0.0)
            mean_sh = np.where(D[:, None, None] > 0, S / D[:, None, None], 0.0) if K else None
            sh_abs = np.where(D[:, None, None] > 0, S_abs / D[:, None, None], 0.0) if K else None
        return dict(D=D, D_abs=D_abs, G=G, G_abs=G_abs, normal=normal, mean_sh=mean_sh, sh_abs=sh_abs)

    def colors(self, r, dirs=None, view_dependent=True):
        """The colour of eval result r along dirs (default -normal), and its sum|terms|; 0 where D == 0."""
        dirs = -r["normal"] if dirs is None else np.asarray(dirs, np.float64)
        col, tabs = color(r["mean_sh"], self.deg if view_dependent else 0, dirs, r["sh_abs"])
        empty = r["D"] == 0
        col[empty] = 0.0
        return col, tabs


def synthetic(P, seed=0, deg=0, spread=0.3, sh=None):
    """Raw (xyz, opacity logits, log-scales, rotations, shs [P,(deg+1)^2,3]) of a seeded blob of P Gaussians; sh [K,3]
    gives every Gaussian the same coefficients."""
    rng = np.random.default_rng(seed)
    K = (deg + 1) ** 2
    xyz = (rng.standard_normal((P, 3)) * spread).astype(f32)
    scaling = np.log(rng.uniform(0.03, 0.12, (P, 3))).astype(f32)
    rotation = rng.standard_normal((P, 4)).astype(f32)
    opacity = (rng.standard_normal((P, 1)) + 1.0).astype(f32)
    shs = (rng.standard_normal((P, K, 3)) * 0.5).astype(f32) if sh is None else np.broadcast_to(np.asarray(sh, f32), (P, K, 3)).copy()
    return xyz, opacity, scaling, rotation, shs


def two_clusters(seed=0, P=1500):
    """Two well-separated blobs with different DC colours: -> raw tensors as `synthetic`, and the two RGB colours."""
    xa, oa, sa, ra, _ = synthetic(P, seed, spread=0.12)
    xb, ob, sb, rb, _ = synthetic(P, seed + 1, spread=0.12)
    xa[:, 0] -= 1.0
    xb[:, 0] += 1.0
    rgb = np.array([[0.9, 0.2, 0.1], [0.1, 0.3, 0.8]], f32)
    dc = ((rgb - 0.5) / SH_C0).astype(f32)
    shs = np.concatenate([np.broadcast_to(dc[0], (P, 1, 3)), np.broadcast_to(dc[1], (P, 1, 3))]).astype(f32)
    cat = lambda a, b: np.concatenate([a, b])
    return (cat(xa, xb), cat(oa, ob), cat(sa, sb), cat(ra, rb), shs), rgb
