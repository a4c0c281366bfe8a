"""numpy restatements for mesh export (DESIGN.md section 2), written from the definition, not from the CUDA:

  * `prepare` / `field` / `field_at`: the density field of extract_fields in float32, one rounding per operation in the
    reference's order (numpy never fuses), summed per voxel over its block's members in ascending Gaussian index;
  * `marching_cubes`: the same marching cubes as csrc/mesh.cu (same table, same vertex and face order), vectorised.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from humangaussian_b200 import mc_table  # noqa: E402

f32 = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_mesh_fields.npz")
SAMPLE_FULL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sample_ply_full.npz")


def golden_inputs(z, tag):
    """Raw (xyz, opacity, scaling, rotation) of golden case `tag`."""
    src = str(z[f"{tag}_inputs_from"]) if f"{tag}_inputs_from" in z.files else tag
    if src == "sample_ply_full.npz":
        d = np.load(SAMPLE_FULL)["data"]
        return d[:, 0:3].copy(), d[:, 6:7].copy(), d[:, 7:10].copy(), d[:, 10:14].copy()
    return tuple(z[f"{src}_{k}"] for k in ("xyz", "opacity", "scaling", "rotation"))


def prepare(xyz, opacity, scaling, rotation, raw=True):
    """-> centres (normalised), cov6 [P,6], opacities, center, scale  of the Gaussians with opacity > 0.005."""
    xyz, opacity, scaling, rotation = (np.asarray(a, f32) for a in (xyz, opacity, scaling, rotation))
    op = (f32(1) / (f32(1) + np.exp(-opacity))).reshape(-1) if raw else opacity.reshape(-1)
    keep = op > f32(0.005)
    x = xyz[keep]
    mn, mx = x.min(0), x.max(0)
    center = (mn + mx) / f32(2)
    scale = 1.8 / float((mx - mn).max())
    x = (x - center) * f32(scale)
    s = (np.exp(scaling[keep]) if raw else scaling[keep]) * f32(scale)
    r = rotation[keep]
    norm = np.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    w, qx, qy, qz = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    one, two = f32(1), f32(2)
    Rm = [[one - two * (qy * qy + qz * qz), two * (qx * qy - w * qz), two * (qx * qz + w * qy)],
          [two * (qx * qy + w * qz), one - two * (qx * qx + qz * qz), two * (qy * qz - w * qx)],
          [two * (qx * qz - w * qy), two * (qy * qz + w * qx), one - two * (qx * qx + qy * qy)]]
    L = [[Rm[i][j] * s[:, j] for j in range(3)] for i in range(3)]
    cv = lambda i, k: L[i][0] * L[k][0] + L[i][1] * L[k][1] + L[i][2] * L[k][2]
    cov6 = np.stack([cv(0, 0), cv(0, 1), cv(0, 2), cv(1, 1), cv(1, 2), cv(2, 2)], 1).astype(f32)
    return x.astype(f32), cov6, op[keep].astype(f32), center, scale


def inverse(cov6):
    a, b, c, d, e, f = (cov6[:, k] for k in range(6))
    det = a * d * f + f32(2) * e * c * b - e * e * a - c * c * d - b * b * f + f32(1e-24)
    inv_det = f32(1) / det
    return np.stack([(d * f - e * e) * inv_det, (e * c - b * f) * inv_det, (e * b - c * d) * inv_det,
                     (a * f - c * c) * inv_det, (b * c - e * a) * inv_det, (a * d - b * b) * inv_det], 1).astype(f32)


def samples(res):
    return torch.linspace(-1, 1, res).numpy()


def _block_members(x, lin, res, split, relax, bx, by, bz):
    lo, hi = [], []
    for b in (bx, by, bz):
        ch = lin[b * split:min(res, (b + 1) * split)]
        lo.append(ch.min() - f32(relax))
        hi.append(ch.max() + f32(relax))
    lo, hi = np.array(lo, f32), np.array(hi, f32)
    return np.nonzero(np.all(x > lo, 1) & np.all(x < hi, 1))[0]


def _eval(pts, x, inv, op):
    """[M] sums over the members (x, inv, op) for points pts [M,3], in member order."""
    d = pts[:, None, :] - x[None]
    dx, dy, dz = d[..., 0], d[..., 1], d[..., 2]
    ia, ib, ic, id_, ie, if_ = (inv[None, :, k] for k in range(6))
    p = f32(-0.5) * (dx * dx * ia + dy * dy * id_ + dz * dz * if_) - dx * dy * ib - dx * dz * ic - dy * dz * ie
    with np.errstate(over="ignore", under="ignore"):
        w = np.where(p > 0, f32(0), np.exp(np.minimum(p, f32(0))))
    return (op[None] * w).astype(np.float64).sum(1).astype(f32)


class Field:
    """The restated field of one Gaussian set: `block(bx, by, bz)` and `at(voxels)` without building the whole grid."""

    def __init__(self, xyz, opacity, scaling, rotation, resolution, num_blocks=16, relax_ratio=1.5, raw=True):
        self.x, cov6, self.op, self.center, self.scale = prepare(xyz, opacity, scaling, rotation, raw)
        self.inv = inverse(cov6)
        self.res, self.split = resolution, resolution // num_blocks
        self.nch = -(-resolution // self.split)
        self.relax = float(f32((2 / num_blocks) * relax_ratio))
        self.lin = samples(resolution)

    def block(self, bx, by, bz):
        s = self.split
        idx = _block_members(self.x, self.lin, self.res, s, self.relax, bx, by, bz)
        xs, ys, zs = (self.lin[b * s:min(self.res, (b + 1) * s)] for b in (bx, by, bz))
        g = np.stack(np.meshgrid(xs, ys, zs, indexing="ij"), -1).reshape(-1, 3)
        if len(idx) == 0:
            return np.zeros((len(xs), len(ys), len(zs)), f32)
        return _eval(g, self.x[idx], self.inv[idx], self.op[idx]).reshape(len(xs), len(ys), len(zs))

    def full(self):
        occ = np.zeros((self.res,) * 3, f32)
        s = self.split
        for bx in range(self.nch):
            for by in range(self.nch):
                for bz in range(self.nch):
                    occ[bx * s:(bx + 1) * s, by * s:(by + 1) * s, bz * s:(bz + 1) * s] = self.block(bx, by, bz)
        return occ

    def at(self, vox):
        """values at voxel indices vox [M,3]"""
        vox = np.asarray(vox)
        out = np.zeros(len(vox), f32)
        blocks = vox // self.split
        for b in np.unique(blocks, axis=0):
            sel = np.all(blocks == b, 1)
            idx = _block_members(self.x, self.lin, self.res, self.split, self.relax, *b)
            if len(idx):
                out[sel] = _eval(self.lin[vox[sel]], self.x[idx], self.inv[idx], self.op[idx])
        return out


# ---- marching cubes ------------------------------------------------------------------------------------------------------
_TABLE = mc_table.build_table()
_COUNT = np.array([len(t) for t in _TABLE], np.int64)
_TRI = np.full((256, 5, 3), -1, np.int64)
for _c, _t in enumerate(_TABLE):
    for _j, _tri in enumerate(_t):
        _TRI[_c, _j] = _tri


def marching_cubes(vol, iso):
    """-> vertices float32 [V,3] (index coordinates), faces int32 [F,3]: the definition of csrc/mesh.cu."""
    vol = np.asarray(vol, f32)
    iso = f32(iso)
    X, Y, Z = vol.shape
    inside = vol > iso
    cross = np.zeros((X, Y, Z, 3), bool)
    cross[:-1, :, :, 0] = inside[:-1] != inside[1:]
    cross[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    cross[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = cross.reshape(-1)
    vid = (np.cumsum(flat) - 1).reshape(X, Y, Z, 3)
    pts = np.nonzero(flat)[0]
    p, a = pts // 3, pts % 3
    x, y, z = p // (Y * Z), (p // Z) % Y, p % Z
    step = np.array([Y * Z, Z, 1])
    v0 = vol.reshape(-1)[p]
    v1 = vol.reshape(-1)[p + step[a]]
    t = (iso - v0) / (v1 - v0)
    verts = np.stack([x, y, z], 1).astype(f32)
    verts[np.arange(len(p)), a] += t
    # cells
    case = np.zeros((X - 1, Y - 1, Z - 1), np.int64)
    for k in range(8):
        dx, dy, dz = k & 1, (k >> 1) & 1, (k >> 2) & 1
        case |= inside[dx:X - 1 + dx, dy:Y - 1 + dy, dz:Z - 1 + dz].astype(np.int64) << k
    cell = np.stack(np.meshgrid(np.arange(X - 1), np.arange(Y - 1), np.arange(Z - 1), indexing="ij"), -1).reshape(-1, 3)
    case = case.reshape(-1)
    nt = _COUNT[case]
    has = nt > 0
    cell, case, nt = cell[has], case[has], nt[has]
    start = np.cumsum(nt) - nt
    faces = np.zeros((int(nt.sum()), 3), np.int64)
    for j in range(5):
        sel = nt > j
        for k in range(3):
            e = _TRI[case[sel], j, k]
            c0 = np.array([mc_table.EDGES[i][0] for i in range(12)])[e]
            ax = np.array([mc_table.EDGES[i][2] for i in range(12)])[e]
            q = cell[sel] + np.stack([c0 & 1, (c0 >> 1) & 1, (c0 >> 2) & 1], 1)
            faces[start[sel] + j, k] = vid[q[:, 0], q[:, 1], q[:, 2], ax]
    return verts, faces.astype(np.int32)


def mesh_stats(verts, faces):
    """(edge -> face count histogram, Euler characteristic V - E + F over used vertices, signed volume)."""
    f = np.asarray(faces, np.int64)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    used = np.unique(f)
    v = np.asarray(verts, np.float64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    vol = np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0
    return np.bincount(cnt), len(used) - len(cnt) + len(f), vol


def sphere(n, r_frac=0.35):
    g = (np.arange(n, dtype=np.float64) - (n - 1) / 2) / (n - 1)
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    return (r_frac - np.sqrt(x * x + y * y + z * z)).astype(f32), r_frac * (n - 1)


def torus(n, R=0.28, r=0.1):
    g = (np.arange(n, dtype=np.float64) - (n - 1) / 2) / (n - 1)
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    q = np.sqrt(x * x + y * y) - R
    return (r - np.sqrt(q * q + z * z)).astype(f32), (R * (n - 1), r * (n - 1))


def pad(vol, value=-1.0):
    out = np.full(tuple(s + 2 for s in vol.shape), f32(value), f32)
    out[1:-1, 1:-1, 1:-1] = vol
    return out
