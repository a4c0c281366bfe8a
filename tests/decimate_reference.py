"""numpy restatement of quadric edge-collapse decimation (humangaussian_b200.mesh.decimate_mesh, DESIGN.md section 2),
written from the definition, not from the CUDA.  Every float64 operation is one IEEE rounding in the order written
(numpy never fuses), so the CUDA, which pins the same order with _rn intrinsics, gives the same bits.

Quadrics.  A face's plane quadric is n n^T / (2 |n|) of a = (n, -n.p0), n = cross(p1 - p0, p2 - p0): the unit plane's
quadric weighted by the face's area (0 for a face with n = 0).  Ten coefficients, row-major upper triangle of the 4x4.
A vertex starts with the sum over its faces where it is corner 0 in ascending face order, then corner 1, then corner 2,
added left to right from 0.  A collapse of (a, b) gives the survivor a the quadric Qa + Qb.

One round, on the current faces (in order) and float32 positions:
  * a vertex is locked when a face around it repeats an index, when a directed edge at it occurs other than exactly
    once in each direction (boundary or non-manifold), or when the faces around it do not form a single fan;
  * a candidate is an edge a < b (from the face holding a -> b) with neither end locked whose ends share exactly two
    neighbours (the link condition), not both of valence 3 (a tetrahedron);
  * its position x and cost: for pa == pb, x = pa and cost 0.  Else Q = Qa + Qb; with the adjugate C of its 3x3 part A,
    det = q0 C00 + q1 C01 + q2 C02 and t = (q0 + q4) + q7, the optimum -C b / det is used when det > 1e-10 t^3 and it
    lies within |pb - pa| of the midpoint; otherwise the cheapest of pa, pb and the midpoint (the first on a tie).  x is
    stored as float32 and the cost is x^T Q x at the stored point, clamped below at +0;
  * it is valid when no other face around a or b, with a or b moved to x, turns its normal: a face whose normal n_old
    is not zero flips when n_old . n_new <= 0 (zero-area faces are exempt);
  * a valid edge is selected when it is the smallest (cost, a * 2^32 + b) among the valid edges with an end in the closed
    one-ring of a or of b.  Selected edges are then at least two edges apart, so their checks stay true together.  When
    the selected collapses would take the mesh below `target`, only the cheapest ceil((F - target) / 2) are applied;
  * a collapse moves a to x, gives it Qa + Qb, renames b to a in every face and drops the two faces on the edge.
Rounds stop when F <= target or when a round selects nothing.  Finally unreferenced vertices are dropped; vertices and
faces keep their order.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

f64 = np.float64
OPT_DET_REL = 1e-10


def face_quadrics(p, f):
    """[F,10] float64 plane quadrics of faces f over float32 positions p."""
    q = p.astype(f64)
    p0, p1, p2 = q[f[:, 0]], q[f[:, 1]], q[f[:, 2]]
    e1, e2 = p1 - p0, p2 - p0
    nx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    ny = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    nz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    ln = np.sqrt((nx * nx + ny * ny) + nz * nz)
    d = -((nx * p0[:, 0] + ny * p0[:, 1]) + nz * p0[:, 2])
    with np.errstate(divide="ignore"):
        h = np.where(ln > 0, 0.5 / ln, 0.0)
    a = [nx, ny, nz, d]
    out = np.stack([(a[i] * a[j]) * h for i in range(4) for j in range(i, 4)], 1)
    out[ln == 0] = 0.0
    return out


def incidence(n_verts, f):
    """(vertex, face, corner) entries in (vertex, corner, face) order, and start offsets [n_verts + 1]."""
    F = len(f)
    vert = f.T.reshape(-1)                 # entry corner * F + face
    face = np.tile(np.arange(F), 3)
    corner = np.repeat(np.arange(3), F)
    order = np.argsort(vert, kind="stable")
    vert, face, corner = vert[order], face[order], corner[order]
    start = np.searchsorted(vert, np.arange(n_verts + 1))
    return vert, face, corner, start


def vertex_quadrics(p, f):
    fq = face_quadrics(p, f)
    vert, face, _, start = incidence(len(p), f)
    Q = np.zeros((len(p), 10), f64)
    deg = np.diff(start)
    for j in range(int(deg.max()) if len(deg) else 0):
        v = np.nonzero(deg > j)[0]
        Q[v] = Q[v] + fq[face[start[v] + j]]
    return Q


def qcost(Q, x):
    """x^T Q x for x [n,3] float64: r_i = ((Q_i0 x + Q_i1 y) + Q_i2 z) + Q_i3, then ((r0 x + r1 y) + r2 z) + r3."""
    q = [Q[:, k] for k in range(10)]
    X, Y, Z = x[:, 0], x[:, 1], x[:, 2]
    r0 = ((q[0] * X + q[1] * Y) + q[2] * Z) + q[3]
    r1 = ((q[1] * X + q[4] * Y) + q[5] * Z) + q[6]
    r2 = ((q[2] * X + q[5] * Y) + q[7] * Z) + q[8]
    r3 = ((q[3] * X + q[6] * Y) + q[8] * Z) + q[9]
    c = ((r0 * X + r1 * Y) + r2 * Z) + r3
    return np.where(c > 0, c, 0.0)


def _dsq(a, b):
    d = a - b
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def place(Q, pa, pb, rule="quadric"):
    """-> (x float32 [n,3], cost float64 [n]) for edges with quadrics Q [n,10] and float32 ends pa, pb."""
    A, B = pa.astype(f64), pb.astype(f64)
    mid = (A + B) * 0.5
    cands = [A, B, mid]
    costs = [qcost(Q, c.astype(np.float32).astype(f64)) for c in cands]
    best = np.zeros(len(Q), np.int64)
    bc = costs[0].copy()
    for i in (1, 2):
        better = costs[i] < bc
        best[better] = i
        bc[better] = costs[i][better]
    x = np.stack(cands, 0)[best, np.arange(len(Q))]
    if rule == "midpoint":
        x, bc = mid, costs[2]
    else:
        q = [Q[:, k] for k in range(10)]
        c00 = q[4] * q[7] - q[5] * q[5]
        c01 = q[2] * q[5] - q[1] * q[7]
        c02 = q[1] * q[5] - q[2] * q[4]
        c11 = q[0] * q[7] - q[2] * q[2]
        c12 = q[1] * q[2] - q[0] * q[5]
        c22 = q[0] * q[4] - q[1] * q[1]
        det = (q[0] * c00 + q[1] * c01) + q[2] * c02
        t = (q[0] + q[4]) + q[7]
        with np.errstate(divide="ignore", invalid="ignore"):
            xo = np.stack([-(((c00 * q[3] + c01 * q[6]) + c02 * q[8]) / det),
                           -(((c01 * q[3] + c11 * q[6]) + c12 * q[8]) / det),
                           -(((c02 * q[3] + c12 * q[6]) + c22 * q[8]) / det)], 1)
            ok = (det > ((t * t) * t) * OPT_DET_REL) & (_dsq(xo, mid) <= _dsq(B, A))
        xo32 = xo.astype(np.float32)
        co = qcost(Q, xo32.astype(f64))
        x = np.where(ok[:, None], xo, x)
        bc = np.where(ok, co, bc)
    zero = np.all(pa == pb, 1)
    x = np.where(zero[:, None], A, x)
    bc = np.where(zero, 0.0, bc)
    return x.astype(np.float32), bc


def _cross(e1, e2):
    return np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                     e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)


def _normals(p0, p1, p2):
    return _cross(p1 - p0, p2 - p0)


def decimate(vertices, faces, target, *, rule="quadric", link_check=True, flip_check=True):
    """-> (vertices float32 [V',3], faces int32 [F',3], rounds).  rule / link_check / flip_check exist so the tests can
    show that the fixtures see a wrong rule; the definition is their defaults."""
    P = np.asarray(vertices, np.float32).reshape(-1, 3).copy()
    f = np.asarray(faces, np.int64).reshape(-1, 3).copy()
    V = len(P)
    Q = vertex_quadrics(P, f)
    rounds = 0
    while len(f) > target:
        F = len(f)
        vert, face, corner, start = incidence(V, f)
        deg = np.diff(start)
        # directed edges a -> b of every (face, corner)
        ha, hb = f.reshape(-1), np.roll(f, -1, 1).reshape(-1)
        hkey = ha * V + hb
        uk, inv, cnt = np.unique(hkey, return_inverse=True, return_counts=True)
        pos = np.searchsorted(uk, hb * V + ha)
        has_rev = (pos < len(uk)) & (uk[np.minimum(pos, len(uk) - 1)] == hb * V + ha)
        rev_cnt = np.where(has_rev, cnt[np.minimum(pos, len(uk) - 1)], 0)
        bad = (cnt[inv] != 1) | (rev_cnt != 1)
        locked = np.zeros(V, bool)
        locked[ha[bad]] = True
        locked[hb[bad]] = True
        rep = (f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 0] == f[:, 2])
        locked[f[rep].reshape(-1)] = True
        # single fan: the link of v maps f[k+1] -> f[k+2] over its faces; one cycle
        ev, eb, ec = f.reshape(-1), np.roll(f, -1, 1).reshape(-1), np.roll(f, -2, 1).reshape(-1)  # entry 3g + k
        ok_e = ~locked[ev]
        succ = np.arange(3 * F)
        sk = np.searchsorted(uk, ev * V + ec)
        # the entry whose directed edge is v -> c: invert hkey -> half-edge index (unique for unlocked v)
        he_of_key = np.empty(len(uk), np.int64)
        he_of_key[inv] = np.arange(3 * F)
        succ[ok_e] = he_of_key[sk[ok_e]]
        lab = np.arange(3 * F)
        nxt = succ.copy()
        for _ in range(int(np.ceil(np.log2(max(2, int(deg.max()) + 1)))) + 1):
            lab = np.minimum(lab, lab[nxt])
            nxt = nxt[nxt]
        heads = np.zeros(V, np.int64)
        np.add.at(heads, ev[ok_e & (lab == np.arange(3 * F))], 1)
        locked |= heads > 1
        # candidates: canonical half-edges a < b with unlocked ends
        cand = (ha < hb) & ~locked[ha] & ~locked[hb]
        ci = np.nonzero(cand)[0]
        a, b = ha[ci], hb[ci]
        ui, uj = np.r_[ha, hb], np.r_[hb, ha]
        A = sp.csr_matrix((np.ones(len(ui)), (ui, uj)), shape=(V, V))
        A.data[:] = 1.0
        common = np.asarray(A[a].multiply(A[b]).sum(1)).reshape(-1)
        ok = (common == 2) & ~((deg[a] == 3) & (deg[b] == 3)) if link_check else np.ones(len(a), bool)
        Qe = Q[a] + Q[b]
        x, cost = place(Qe, P[a], P[b], rule)
        if flip_check:
            # every (candidate, entry around a or b) pair; faces holding both ends are the edge's own two
            segs = []
            for end in (a, b):
                n = deg[end]
                rid = np.repeat(np.arange(len(end)), n)
                off = np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n)
                segs.append((rid, start[end][rid] + off))
            rid = np.concatenate([s[0] for s in segs])
            e = np.concatenate([s[1] for s in segs])
            g, k = face[e], corner[e]
            fg = f[g]
            both = np.any(fg == a[rid, None], 1) & np.any(fg == b[rid, None], 1)
            q = P.astype(f64)
            p0, p1, p2 = q[fg[:, 0]], q[fg[:, 1]], q[fg[:, 2]]
            n_old = _normals(p0, p1, p2)
            pts = [p0.copy(), p1.copy(), p2.copy()]
            xr = x[rid].astype(f64)
            for c in range(3):
                sel = k == c
                pts[c][sel] = xr[sel]
            n_new = _normals(*pts)
            dot = (n_old[:, 0] * n_new[:, 0] + n_old[:, 1] * n_new[:, 1]) + n_old[:, 2] * n_new[:, 2]
            flip = ~both & np.any(n_old != 0, 1) & (dot <= 0)
            bad_c = np.zeros(len(a), bool)
            bad_c[rid[flip]] = True
            ok &= ~bad_c
        a, b, x, cost, Qe = a[ok], b[ok], x[ok], cost[ok], Qe[ok]
        if len(a) == 0:
            break
        ekey = (a.astype(np.uint64) << np.uint64(32)) | b.astype(np.uint64)
        order = np.lexsort((ekey, cost))
        rank = np.empty(len(a), np.int64)
        rank[order] = np.arange(len(a))
        big = np.iinfo(np.int64).max
        best1 = np.full(V, big)
        np.minimum.at(best1, a, rank)
        np.minimum.at(best1, b, rank)
        best2 = best1.copy()
        np.minimum.at(best2, ha, best1[hb])
        np.minimum.at(best2, hb, best1[ha])
        sel = (best2[a] == rank) & (best2[b] == rank)
        S = int(sel.sum())
        rounds += 1
        if S == 0:
            break
        k_take = min(S, -(-(F - target) // 2))
        if k_take < S:
            thr = np.sort(rank[sel])[k_take - 1]
            sel &= rank <= thr
        a, b = a[sel], b[sel]
        P[a] = x[sel]
        Q[a] = Qe[sel]
        remap = np.arange(V)
        remap[b] = a
        f = remap[f]
        f = f[(f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])]
        assert len(f) == F - 2 * len(a)
    used = np.zeros(V, bool)
    used[f.reshape(-1)] = True
    new_id = np.cumsum(used) - 1
    return P[used].copy(), new_id[f].astype(np.int32).reshape(-1, 3), rounds
