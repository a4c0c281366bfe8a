"""numpy restatement of mesh cleanup (humangaussian_b200.mesh.clean_mesh, DESIGN.md section 2), written from the
definition, not from the CUDA:

  1. faces that repeat a vertex index are dropped, and so is every face whose vertex set equals an earlier face's;
  2. the remaining faces are grouped into connected components (two faces are connected when they share a vertex);
  3. a component is removed when it has fewer than min_faces faces, or when its vertices' bounding-box diagonal is
     below min_diameter times the diagonal of every vertex the step-1 faces use (float64, sqrt((dx dx + dy dy) + dz dz));
  4. unreferenced vertices are removed; surviving vertices and faces keep their order and their bytes.
"""
from __future__ import annotations

import numpy as np


def face_filter(faces):
    """bool [F]: the faces step 1 keeps."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    ok = (f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])
    idx = np.nonzero(ok)[0]
    if len(idx):
        _, first = np.unique(np.sort(f[idx], 1), axis=0, return_index=True)
        keep = np.zeros(len(idx), bool)
        keep[first] = True  # np.unique returns the first occurrence of every set
        ok[idx[~keep]] = False
    return ok


def vertex_labels(n_verts, faces):
    """int64 [n_verts]: the smallest vertex index of each vertex's component (min-label propagation to its fixed
    point); vertices no face uses label themselves."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    lab = np.arange(n_verts, dtype=np.int64)
    while True:
        m = lab[f].min(1)
        new = lab.copy()
        for k in range(3):
            np.minimum.at(new, f[:, k], m)
        new = new[new]  # pointer jumping; labels only decrease and stay inside the component
        if np.array_equal(new, lab):
            return lab
        lab = new


def _diag(lo, hi):
    d = hi.astype(np.float64) - lo.astype(np.float64)
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def clean_mesh(vertices, faces, min_faces=64, min_diameter=0.2):
    """-> (vertices float32 [V',3], faces int32 [F',3])"""
    v = np.asarray(vertices, np.float32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    f = f[face_filter(f)]
    if len(f):
        lab = vertex_labels(len(v), f)
        flab = lab[f[:, 0]]
        roots, inv, counts = np.unique(flab, return_inverse=True, return_counts=True)
        used = np.unique(f)
        lo = np.full((len(roots), 3), np.inf, np.float32)
        hi = np.full((len(roots), 3), -np.inf, np.float32)
        ridx = np.searchsorted(roots, lab[used])
        np.minimum.at(lo, ridx, v[used])
        np.maximum.at(hi, ridx, v[used])
        whole = _diag(v[used].min(0), v[used].max(0))
        ok = (counts >= min_faces) & ~(_diag(lo, hi) < np.float64(min_diameter) * whole)
        f = f[ok[inv]]
    used = np.zeros(len(v), bool)
    used[f.reshape(-1)] = True
    new_id = np.cumsum(used) - 1
    return v[used].copy(), new_id[f].astype(np.int32).reshape(-1, 3)
