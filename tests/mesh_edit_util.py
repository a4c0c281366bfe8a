"""Shared fixtures and invariant checks of the mesh cleanup / decimation tests (CPU and GPU)."""
from __future__ import annotations

import numpy as np
from scipy.sparse import coo_matrix, csgraph
from scipy.spatial import cKDTree

import mesh_clean_reference as C
import mesh_reference as M


def fixture_meshes():
    """name -> (vertices, faces) of the restated marching cubes: a sphere, a torus and golden case a's body."""
    out = {}
    vol, _ = M.sphere(40)
    out["sphere"] = M.marching_cubes(M.pad(vol), 0.0)
    vol, _ = M.torus(48)
    out["torus"] = M.marching_cubes(M.pad(vol), 0.0)
    out["golden"] = C.clean_mesh(*golden_mesh())
    return out


def golden_mesh():
    z = np.load(M.GOLDEN)
    return M.marching_cubes(z["a_occ"], 1.0)


def face_components(n_verts, faces):
    """scipy's component label of every face (faces connected through shared vertices)."""
    f = np.asarray(faces, np.int64)
    A = coo_matrix((np.ones(2 * len(f)), (np.r_[f[:, 0], f[:, 1]], np.r_[f[:, 1], f[:, 2]])), shape=(n_verts, n_verts))
    _, lab = csgraph.connected_components(A, directed=False)
    return lab[f[:, 0]]


def planted_mesh(seed=0):
    """A sphere with planted defects: small floaters, a repeated-index face, duplicates (same and reversed order), a
    far-away tiny component, unreferenced vertices, and the vertex order shuffled."""
    rng = np.random.default_rng(seed)
    vol, _ = M.sphere(24)
    v, f = M.marching_cubes(M.pad(vol), 0.0)
    parts_v, parts_f = [v], [f]
    n = len(v)
    for k in range(5):  # floaters: small spheres of a few dozen faces
        sv, sf = M.marching_cubes(M.pad(M.sphere(6)[0]), 0.0)
        parts_v.append(sv * np.float32(0.3) + np.float32(30 + 3 * k))
        parts_f.append(sf + n)
        n += len(sv)
    parts_v.append(rng.standard_normal((7, 3)).astype(np.float32) * 5)  # unreferenced
    n += 7
    v = np.concatenate(parts_v)
    f = np.concatenate(parts_f)
    f = np.concatenate([f, f[[3]], f[[10]][:, ::-1], [[f[0, 0], f[0, 0], f[0, 1]]]]).astype(np.int32)
    perm = rng.permutation(len(v))
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(v))
    return np.ascontiguousarray(v[perm]), inv[f].astype(np.int32)


def surface_samples(v, f, n=6):
    v = np.asarray(v, np.float64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return np.concatenate([a + (b - a) * (i / n) + (c - a) * (j / n) for i in range(n + 1) for j in range(n + 1 - i)])


def two_sided_distance(v0, f0, v1, f1):
    """max over vertices of either mesh of the distance to the other mesh's surface, sampled at 28 points per triangle
    (an over-estimate by at most the sample spacing, edge / 6)."""
    t0, t1 = cKDTree(surface_samples(v0, f0)), cKDTree(surface_samples(v1, f1))
    return max(t1.query(np.asarray(v0, np.float64))[0].max(), t0.query(np.asarray(v1, np.float64))[0].max())


def mean_edge(v, f):
    v = np.asarray(v, np.float64)
    return float(np.mean([np.linalg.norm(v[f[:, i]] - v[f[:, (i + 1) % 3]], axis=1).mean() for i in range(3)]))


def check_invariants(v0, f0, v1, f1, target):
    """The decimation invariants: a closed oriented manifold in, the same out (every edge used once in each direction),
    the same number of components with the same Euler characteristics, and F in {target - 1, target}."""
    f1 = np.asarray(f1, np.int64)
    assert len(f1) in (target - 1, target), (len(f1), target)
    assert f1.min() >= 0 and f1.max() < len(v1) and len(np.unique(f1)) == len(v1)  # every vertex used
    he = np.concatenate([f1[:, [0, 1]], f1[:, [1, 2]], f1[:, [2, 0]]])
    key, rkey = he[:, 0] * len(v1) + he[:, 1], he[:, 1] * len(v1) + he[:, 0]
    u, cnt = np.unique(key, return_counts=True)
    assert (cnt == 1).all(), "a directed edge occurs twice"
    assert np.isin(rkey, u).all(), "an edge is not used in both directions"

    def per_component(v, f):
        f = np.asarray(f, np.int64)
        lab = face_components(len(v), f)
        out = []
        for c in np.unique(lab):
            _, chi, _ = M.mesh_stats(v, f[lab == c])
            out.append(chi)
        return sorted(out)

    assert per_component(v0, f0) == per_component(v1, f1)
