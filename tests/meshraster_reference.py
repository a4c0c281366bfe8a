"""Numpy restatement of the mesh render (humangaussian_b200/meshrender.py, csrc/meshraster.cu; DESIGN.md section 2).

Every float32 operation below is one numpy ufunc on float32 operands, so it is rounded once, left to right, with no FMA
contraction: the CUDA kernels, which spell the same operations with _rn intrinsics, must match it byte for byte.
`rasterize_f64` is the float64 brute force the restatement itself is checked against (tests/test_meshraster_cpu.py).
"""
import os

import numpy as np

F = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_meshraster.npz")
EPS = F(1e-20)


def vertex_transform(vertices, mvp):
    """[x, y, z, 1] @ mvp^T: vertices [Nv, 3] or [V, Nv, 3], mvp [V, 4, 4] -> [V, Nv, 4]; row r is
    ((m_r0 x + m_r1 y) + m_r2 z) + m_r3."""
    v = np.asarray(vertices, F)
    m = np.asarray(mvp, F)
    if v.ndim == 2:
        v = v[None]
    x, y, z = v[..., 0], v[..., 1], v[..., 2]
    rows = [((m[:, r, 0, None] * x + m[:, r, 1, None] * y) + m[:, r, 2, None] * z) + m[:, r, 3, None] for r in range(4)]
    return np.stack(rows, -1).astype(F)


def pixel_ndc(n):
    """(2i + 1) / n - 1 for i in 0..n-1, float32."""
    return (np.arange(1, 2 * n, 2, dtype=F) / F(n) - F(1)).astype(F)


def ordered_bits(z):
    b = np.asarray(z, F).view(np.uint32)
    return np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def triangle_setup(p):
    """Edge coefficients (A, B, C) [3] each and D of clip vertices p [3, 4] (float32), or None when the triangle is not
    drawn at all (non-finite coordinate, or W <= 0 at all three vertices)."""
    p = np.asarray(p, F)
    if not np.isfinite(p).all() or (p[:, 3] <= 0).all():
        return None
    X, Y, W = p[:, 0], p[:, 1], p[:, 3]
    A, B, C = np.zeros(3, F), np.zeros(3, F), np.zeros(3, F)
    with np.errstate(all="ignore"):
        for i in range(3):
            j, k = (i + 1) % 3, (i + 2) % 3
            A[i] = Y[j] * W[k] - W[j] * Y[k]
            B[i] = W[j] * X[k] - X[j] * W[k]
            C[i] = X[j] * Y[k] - Y[j] * X[k]
        D = X[0] * A[0] + Y[0] * B[0] + W[0] * C[0]
    return A, B, C, F(D)


def _span(a, b, n):
    """One axis of the pixel rectangle: [floor(pa) - 1, ceil(pb) + 1] clamped to [0, n - 1], with pa, pb the pixel
    coordinates ((s + 1) * (n / 2)) - 1/2 of the NDC extremes a, b, in float32; None when it is empty."""
    h = F(0.5) * F(n)
    pa, pb = (a + F(1)) * h - F(0.5), (b + F(1)) * h - F(0.5)
    lo, hi = np.maximum(np.floor(pa) - F(1), F(0)), np.minimum(np.ceil(pb) + F(1), F(n - 1))
    return (int(lo), int(hi)) if lo <= hi else None


def pixel_rect(p, H, W):
    """The triangle's pixel rectangle (x0, x1, y0, y1), or None when it is empty.  Where every W > 0 it is the projected
    vertices' bounding box (X / W, Y / W in float32) widened by one pixel: every pixel centre of the exact projected
    triangle lies inside it, and a pixel outside it is not covered whatever its edge functions say (a point-sized
    triangle's edge functions are rounding noise).  Otherwise it is the whole image."""
    if not (p[:, 3] > 0).all():
        return 0, W - 1, 0, H - 1
    with np.errstate(all="ignore"):
        sx, sy = p[:, 0] / p[:, 3], p[:, 1] / p[:, 3]
    x = _span(sx.min(), sx.max(), W)
    y = _span(sy.min(), sy.max(), H)
    return None if x is None or y is None else x + y


def coverage(p, A, B, C, D, px, py):
    """(covered mask, u, v, zw) of one triangle at pixel centres px [w] x py [h] (float32), per the specification."""
    Z, Wc = p[:, 2], p[:, 3]
    with np.errstate(all="ignore"):
        e = [(A[i] * px[None, :] + B[i] * py[:, None]) + C[i] for i in range(3)]
        if D > 0:
            inside = (e[0] >= 0) & (e[1] >= 0) & (e[2] >= 0)
        else:
            inside = (e[0] <= 0) & (e[1] <= 0) & (e[2] <= 0)
        S = (e[0] + e[1]) + e[2]
        u, v, l2 = e[0] / S, e[1] / S, e[2] / S
        Wp = (u * Wc[0] + v * Wc[1]) + l2 * Wc[2]
        zw = ((u * Z[0] + v * Z[1]) + l2 * Z[2]) / Wp
        cov = inside & (S != 0) & (Wp > 0) & (zw >= -1) & (zw <= 1)
    return cov, u, v, zw


def rasterize(pos, tri, H, W, full=False):
    """rast [V, H, W, 4] float32 (u, v, z/w, t + 1) of clip vertices pos [V, Nv, 4] and triangles tri [Nf, 3].
    full=True drops the pixel-rectangle rule and applies the per-pixel coverage rule to every pixel of the image (not the
    specification: the tests use it to show what the rectangle changes)."""
    pos = np.asarray(pos, F)
    tri = np.asarray(tri, np.int64)
    V, Nv = pos.shape[:2]
    PX, PY = pixel_ndc(W), pixel_ndc(H)
    rast = np.zeros((V, H, W, 4), F)
    for v in range(V):
        best = np.full((H, W), np.iinfo(np.uint64).max, np.uint64)
        for t, idx in enumerate(tri):
            if (idx < 0).any() or (idx >= Nv).any():
                continue
            p = pos[v, idx]
            s = triangle_setup(p)
            if s is None:
                continue
            A, B, C, D = s
            if not (np.isfinite(A).all() and np.isfinite(B).all() and np.isfinite(C).all() and np.isfinite(D) and D != 0):
                continue
            rect = (0, W - 1, 0, H - 1) if full else pixel_rect(p, H, W)
            if rect is None:
                continue
            x0, x1, y0, y1 = rect
            cov, u, w, zw = coverage(p, A, B, C, D, PX[x0:x1 + 1], PY[y0:y1 + 1])
            key = (ordered_bits(zw).astype(np.uint64) << np.uint64(32)) | np.uint64(t)
            sub = best[y0:y1 + 1, x0:x1 + 1]
            win = cov & (key < sub)
            sub[win] = key[win]
            r = rast[v, y0:y1 + 1, x0:x1 + 1]
            r[..., 0][win], r[..., 1][win], r[..., 2][win], r[..., 3][win] = u[win], w[win], zw[win], F(t + 1)
    return rast


def _pixel_tri(rast, tri, Nv):
    """Triangle index per pixel (-1 where rast.w is not an id in 1..Nf or the triangle has an index outside [0, Nv))."""
    w = rast[..., 3]
    Nf = tri.shape[0]
    ok = (w > 0) & (w <= Nf)
    t = np.where(ok, w, 1).astype(np.int64) - 1
    idx = tri[t] if Nf else np.zeros(t.shape + (3,), np.int64)
    ok &= ((idx >= 0) & (idx < Nv)).all(-1)
    return np.where(ok, t, -1), np.where(ok[..., None], idx, 0)


def interpolate(attr, rast, tri):
    """[V, H, W, C]: a0 u + a1 v + a2 ((1 - u) - v) where rast holds a triangle, 0 elsewhere.  attr [V, Nv, C] or [Nv, C]."""
    attr = np.asarray(attr, F)
    rast = np.asarray(rast, F)
    tri = np.asarray(tri, np.int64)
    V = rast.shape[0]
    a = np.broadcast_to(attr, (V,) + attr.shape[-2:]) if attr.ndim == 2 else attr
    t, idx = _pixel_tri(rast, tri, a.shape[1])
    vi = np.arange(V)[:, None, None]
    a0, a1, a2 = a[vi, idx[..., 0]], a[vi, idx[..., 1]], a[vi, idx[..., 2]]
    u, v = rast[..., 0:1], rast[..., 1:2]
    b2 = (F(1) - u) - v
    with np.errstate(all="ignore"):
        out = (a0 * u + a1 * v) + a2 * b2
    return np.where((t >= 0)[..., None], out, F(0)).astype(F)


def _dot(x):
    return (x[..., 0] * x[..., 0] + x[..., 1] * x[..., 1]) + x[..., 2] * x[..., 2]


def safe_normalize(x):
    with np.errstate(all="ignore"):
        return (x / np.sqrt(np.maximum(_dot(x), EPS))[..., None]).astype(F)


def face_normals(vertices, faces):
    """cross(v1 - v0, v2 - v0) in torch.cross's component formula, [..., Nf, 3]."""
    v0, v1, v2 = vertices[..., faces[:, 0], :], vertices[..., faces[:, 1], :], vertices[..., faces[:, 2], :]
    a, b = v1 - v0, v2 - v0
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                     a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1).astype(F)


def vertex_normals(vertices, faces):
    """The reference's vertex normals in the fixed order: vertices [Nv, 3] or [F, Nv, 3]."""
    v = np.asarray(vertices, F)
    faces = np.asarray(faces, np.int64)
    single = v.ndim == 2
    if single:
        v = v[None]
    Nv = v.shape[1]
    keep = ((faces >= 0) & (faces < Nv)).all(1)
    f = faces[keep]
    out = np.zeros(v.shape, F)
    with np.errstate(all="ignore"):
        for k in range(v.shape[0]):
            fn = face_normals(v[k], f)
            acc = np.zeros((Nv, 3), F)
            for corner in range(3):  # ufunc.at adds in index order: ascending face index per vertex
                np.add.at(acc, f[:, corner], fn)
            acc = np.where((_dot(acc) > EPS)[:, None], acc, np.array([0, 0, 1], F))
            out[k] = safe_normalize(acc)
    return out[0] if single else out


def normal_image(vn, rast, tri):
    """(safe_normalize(interpolated vn) + 1) / 2 where rast holds a triangle, 1.0 elsewhere: [V, H, W, 3]."""
    rast = np.asarray(rast, F)
    tri = np.asarray(tri, np.int64)
    vn = np.asarray(vn, F)
    t, _ = _pixel_tri(rast, tri, vn.shape[-2])
    n = safe_normalize(interpolate(vn, rast, tri))
    with np.errstate(all="ignore"):
        img = (n + F(1)) / F(2)
    return np.where((t >= 0)[..., None], img, F(1)).astype(F)


def render_mesh_normal(mvp, H, W, vertices, faces):
    pos = vertex_transform(vertices, mvp)
    rast = rasterize(pos, faces, H, W)
    return normal_image(vertex_normals(vertices, faces), rast, faces)


def rasterize_f64(pos, tri, H, W):
    """Float64 brute force over every (pixel, triangle): (winner [V, H, W] int, u, v, zw, clean [V, H, W] bool).  A
    pixel is clean when, for every triangle that is drawn, every |e_i| and |S| is above 1e-4 of its terms' magnitude, Wp
    and zw are 1e-4 away from their limits, and the winner's depth is 1e-4 away from the runner-up's."""
    pos = np.asarray(pos, np.float64)
    tri = np.asarray(tri, np.int64)
    V, Nv = pos.shape[:2]
    px = (2 * np.arange(W) + 1) / W - 1
    py = (2 * np.arange(H) + 1) / H - 1
    PX, PY = np.meshgrid(px, py)
    win = np.full((V, H, W), -1)
    U, Vv, ZW = np.zeros((V, H, W)), np.zeros((V, H, W)), np.zeros((V, H, W))
    clean = np.ones((V, H, W), bool)
    rel = 1e-4
    for v in range(V):
        z1 = np.full((H, W), np.inf)
        z2 = np.full((H, W), np.inf)
        for t, idx in enumerate(tri):
            if (idx < 0).any() or (idx >= Nv).any():
                continue
            p = pos[v, idx]
            if not np.isfinite(p).all() or (p[:, 3] <= 0).all():
                continue
            X, Y, Z, Wc = p.T
            e, mag = [], []
            for i in range(3):
                j, k = (i + 1) % 3, (i + 2) % 3
                A, B, C = Y[j] * Wc[k] - Wc[j] * Y[k], Wc[j] * X[k] - X[j] * Wc[k], X[j] * Y[k] - Y[j] * X[k]
                e.append(A * PX + B * PY + C)
                mag.append(np.abs(A * PX) + np.abs(B * PY) + np.abs(C) + 1e-300)
            D = X[0] * (Y[1] * Wc[2] - Wc[1] * Y[2]) + Y[0] * (Wc[1] * X[2] - X[1] * Wc[2]) + Wc[0] * (X[1] * Y[2] - Y[1] * X[2])
            if D == 0:
                continue
            s = np.sign(D)
            inside = (s * e[0] >= 0) & (s * e[1] >= 0) & (s * e[2] >= 0)
            with np.errstate(all="ignore"):
                S = e[0] + e[1] + e[2]
                u, w = e[0] / S, e[1] / S
                l2 = e[2] / S
                Wp = u * Wc[0] + w * Wc[1] + l2 * Wc[2]
                zw = (u * Z[0] + w * Z[1] + l2 * Z[2]) / Wp
                cov = inside & (S != 0) & (Wp > 0) & (zw >= -1) & (zw <= 1)
                amb = (np.abs(e[0]) < rel * mag[0]) | (np.abs(e[1]) < rel * mag[1]) | (np.abs(e[2]) < rel * mag[2])
                amb |= np.abs(S) < rel * (mag[0] + mag[1] + mag[2])
                amb |= inside & ((np.abs(Wp) < rel * np.abs(Wc).max()) | (np.abs(np.abs(zw) - 1) < rel))
            clean[v] &= ~amb
            zc = np.where(cov, zw, np.inf)
            nearer = zc < z1
            z2 = np.where(nearer, z1, np.minimum(z2, zc))
            z1 = np.where(nearer, zc, z1)
            win[v] = np.where(nearer, t, win[v])
            U[v], Vv[v], ZW[v] = np.where(nearer, u, U[v]), np.where(nearer, w, Vv[v]), np.where(nearer, zw, ZW[v])
        with np.errstate(all="ignore"):
            gap = np.abs(z2 - z1)
        clean[v] &= ~(np.isfinite(z2) & (gap < rel))
    return win, U, Vv, ZW, clean


def load_obj_polygons(path):
    """Vertices [Nv, 3] float32 and the polygons (lists of 0-based indices) of an OBJ file's v / f records."""
    verts, polys = [], []
    with open(path) as fh:
        for line in fh:
            parts = line.split()
            if not parts:
                continue
            if parts[0] == "v":
                verts.append([float(x) for x in parts[1:4]])
            elif parts[0] == "f":
                polys.append([int(p.split("/")[0]) - 1 for p in parts[1:]])
    return np.asarray(verts, F), polys


def fan_triangulate(polys):
    """(p0, p_k, p_k+1) for k = 1..n-2 of every polygon, in file order: [Nf, 3] int32."""
    return np.asarray([(p[0], p[k], p[k + 1]) for p in polys for k in range(1, len(p) - 1)], np.int32)
