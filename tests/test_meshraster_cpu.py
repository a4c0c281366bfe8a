"""CPU: the numpy restatement of the mesh render (tests/meshraster_reference.py) against independent definitions.

  1. rasterisation against a float64 brute force over every (pixel, triangle): the same coverage and winner wherever
     the pixel is clear of every edge, limit and depth tie by a relative 1e-4, and u, v, z/w within float32 tolerance;
  2. the pixel-rectangle rule changes nothing on ordinary triangles, and confines point-sized and corner-cut triangles,
     whose edge functions are rounding noise, to their widened bounding boxes;
  3. a tessellated quad over the whole screen (shared, consistently wound edges, pixel centres on edges) leaves no hole;
  4. the reference viewer's render_mesh_normal, step for step in torch on the CPU with its two nvdiffrast calls served
     by the restatement, against the restatement's normal image: the vertex-normal, safe_normalize and background rules.
"""
import math

import numpy as np
import pytest
import torch

import meshraster_reference as M

F = np.float32


def soup(seed, n, V=2, behind=0.15):
    """n random clip-space triangles per view (independent vertices), some with W <= 0 at one or more corners."""
    rng = np.random.default_rng(seed)
    Nv = 3 * n
    s = rng.uniform(-1.3, 1.3, (V, Nv, 2))
    z = rng.uniform(-1.1, 1.1, (V, Nv))
    w = rng.uniform(0.4, 3.0, (V, Nv))
    w = np.where(rng.random((V, Nv)) < behind, -w * 0.3, w)
    pos = np.stack([s[..., 0] * w, s[..., 1] * w, z * np.abs(w), w], -1).astype(F)
    tri = np.arange(Nv, dtype=np.int32).reshape(n, 3)
    return pos, tri


def corner_cuts(seed, n, V=1, scale=0.02, point=False):
    """n tiny triangles per view, as marching cubes makes them where it cuts a cell corner at t ~ 0: a vertex at a random
    position and two more at t * scale NDC from it, t in [1e-7, 1e-4] (point=True: all three within a few ulps)."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-0.95, 0.95, (V, n, 1, 2))
    t = 10 ** rng.uniform(-7, -4, (V, n, 1, 1)) * scale
    d = rng.normal(size=(V, n, 3, 2))
    d[:, :, 0] = 0
    s = c + (d * 3e-7 * np.abs(c) if point else t * d)
    w = rng.uniform(0.5, 3.0, (V, n, 1, 1)) * np.ones((V, n, 3, 1))
    z = rng.uniform(-0.5, 0.5, (V, n, 1, 1)) * np.ones((V, n, 3, 1))
    pos = np.concatenate([s * w, z * w, w], -1).reshape(V, 3 * n, 4).astype(F)
    return pos, np.arange(3 * n, dtype=np.int32).reshape(n, 3)


def quad_grid(nx, ny, lo=-1.4, hi=1.4, jitter=0.0, seed=0, V=1, exact_px=None):
    """A consistently wound grid of 2 nx ny triangles over [lo, hi]^2 in NDC, W random per vertex (the projection is
    unchanged), interior vertices jittered; exact_px = (H, W) snaps interior vertices to pixel centres."""
    rng = np.random.default_rng(seed)
    gx, gy = np.meshgrid(np.linspace(lo, hi, nx + 1), np.linspace(lo, hi, ny + 1))
    inner = (slice(1, -1), slice(1, -1))
    gx[inner] += rng.uniform(-jitter, jitter, gx[inner].shape)
    gy[inner] += rng.uniform(-jitter, jitter, gy[inner].shape)
    if exact_px is not None:
        H, W = exact_px
        gx[inner] = (2 * np.clip(np.round((gx[inner] + 1) * W / 2 - 0.5), 0, W - 1) + 1) / W - 1
        gy[inner] = (2 * np.clip(np.round((gy[inner] + 1) * H / 2 - 0.5), 0, H - 1) + 1) / H - 1
    sx, sy = gx.ravel(), gy.ravel()
    idx = np.arange((nx + 1) * (ny + 1)).reshape(ny + 1, nx + 1)
    a, b, c, d = idx[:-1, :-1].ravel(), idx[:-1, 1:].ravel(), idx[1:, 1:].ravel(), idx[1:, :-1].ravel()
    tri = np.concatenate([np.stack([a, b, c], 1), np.stack([a, c, d], 1)]).astype(np.int32)
    w = rng.uniform(0.5, 2.0, (V, sx.size)) if exact_px is None else np.ones((V, sx.size))
    pos = np.stack([sx * w, sy * w, 0.25 * w, w], -1).astype(F)
    return pos, tri


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatement_matches_the_float64_brute_force(seed):
    H, W = 37, 53
    pos, tri = soup(seed, 40)
    rast = M.rasterize(pos, tri, H, W)
    win, u, v, zw, clean = M.rasterize_f64(pos, tri, H, W)
    assert clean.mean() > 0.9
    got = rast[..., 3].astype(np.int64) - 1
    assert np.array_equal(got[clean], win[clean])
    cov = clean & (win >= 0)
    assert cov.sum() > 1000
    for a, b in ((rast[..., 0], u), (rast[..., 1], v), (rast[..., 2], zw)):
        assert np.abs(a[cov] - b[cov]).max() < 1e-4


@pytest.mark.parametrize("seed", [3, 4])
def test_bounding_rectangle_changes_nothing(seed):
    """The pixel-rectangle rule removes nothing from ordinary triangles: the same bytes as the per-pixel rule alone."""
    H, W = 40, 33
    pos, tri = soup(seed, 60)
    assert np.array_equal(M.rasterize(pos, tri, H, W), M.rasterize(pos, tri, H, W, full=True))
    pos, tri = quad_grid(5, 4, jitter=0.1, seed=seed, exact_px=(H, W))
    assert np.array_equal(M.rasterize(pos, tri, H, W), M.rasterize(pos, tri, H, W, full=True))


@pytest.mark.parametrize("point", [False, True])
def test_pixel_rectangle_confines_point_sized_triangles(point):
    """Without the rectangle, the per-pixel rule lets a triangle whose edge functions are rounding noise cover pixels far
    from it; with it, every pixel a triangle wins lies in its widened bounding box."""
    H, W = 64, 48
    pos, tri = corner_cuts(6 + point, 300, V=2, point=point)
    rast = M.rasterize(pos, tri, H, W)
    assert (M.rasterize(pos, tri, H, W, full=True)[..., 3] > 0).sum() > 2 * max((rast[..., 3] > 0).sum(), 1)
    for v in range(2):
        for t in np.unique(rast[v, ..., 3]).astype(int):
            if t == 0:
                continue
            x0, x1, y0, y1 = M.pixel_rect(pos[v, tri[t - 1]], H, W)
            assert x1 - x0 <= 3 and y1 - y0 <= 3
            ys, xs = np.nonzero(rast[v, ..., 3] == t)
            assert xs.min() >= x0 and xs.max() <= x1 and ys.min() >= y0 and ys.max() <= y1


@pytest.mark.parametrize("exact", [False, True])
def test_tessellated_quad_over_the_screen_has_no_holes(exact):
    H, W = 29, 41
    pos, tri = quad_grid(7, 5, jitter=0.12, seed=5, exact_px=(H, W) if exact else None)
    rast = M.rasterize(pos, tri, H, W)
    assert (rast[..., 3] > 0).all()
    assert np.allclose(rast[..., 2], 0.25, atol=1e-6)


def _torch_render_mesh_normal(mvp, H, W, vertices, faces, clip=None):
    """animation.py:558-601 (GUI.render_mesh_normal) step for step in torch on the CPU; its dr.rasterize and dr.interpolate
    are served by the restatement.  clip replaces the clip coordinates the rasteriser is given."""
    vertices_clip = torch.matmul(torch.nn.functional.pad(vertices, pad=(0, 1), mode="constant", value=1.0),
                                 torch.transpose(mvp, 0, 1)).float().unsqueeze(0)
    rast = torch.from_numpy(M.rasterize(vertices_clip.numpy() if clip is None else clip, faces.numpy(), H, W))
    i0, i1, i2 = faces[:, 0].long(), faces[:, 1].long(), faces[:, 2].long()
    v0, v1, v2 = vertices[i0, :], vertices[i1, :], vertices[i2, :]
    face_normals = torch.linalg.cross(v1 - v0, v2 - v0, dim=-1)
    vn = torch.zeros_like(vertices)
    for i in (i0, i1, i2):
        vn.scatter_add_(0, i[:, None].repeat(1, 3), face_normals)
    dot = lambda x: torch.sum(x * x, -1, keepdim=True)  # noqa: E731
    safe_normalize = lambda x: x / torch.sqrt(torch.clamp(dot(x), min=1e-20))  # noqa: E731
    vn = torch.where(dot(vn) > 1e-20, vn, torch.tensor([0.0, 0.0, 1.0], dtype=torch.float32))
    vn = safe_normalize(vn)
    normal = torch.from_numpy(M.interpolate(vn.unsqueeze(0).numpy(), rast.numpy(), faces.numpy()))
    normal = safe_normalize(normal)
    img = (normal[0] + 1) / 2
    img = torch.where(rast[..., 3:] > 0, img, torch.tensor(1.0))[0]
    return img.numpy(), vertices_clip[0].numpy(), rast[0].numpy(), vn.numpy()


def human():
    z = np.load(M.GOLDEN)
    v = z["vertices"]
    return np.stack([v[:, 0], -v[:, 2], v[:, 1]], 1).astype(F), z["faces"]  # y-up OBJ -> the cameras' z-up


def mvp_orbit(elev, azim, dist, fovy_deg, H, W, center=(0.0, 0.0, 0.0)):
    from humangaussian_b200.cameras import CameraBatch, orbit_c2w
    cams = CameraBatch(orbit_c2w(elev, azim, dist, center)[None], [math.radians(fovy_deg)], H, W)
    return cams.full_proj_transform.transpose(1, 2)[0].numpy()


@pytest.mark.parametrize("view", [(15.0, 30.0, 2.6), (-10.0, 200.0, 2.2), (5.0, 90.0, 0.9)])
def test_reference_normal_image_body_matches_the_restatement(view):
    H, W = 48, 40
    verts, faces = human()
    mvp = mvp_orbit(*view, 45.0, H, W, center=(0.0, 0.0, -0.1))
    ref, clip, ref_rast, ref_vn = _torch_render_mesh_normal(torch.from_numpy(mvp), H, W, torch.from_numpy(verts), torch.from_numpy(faces))
    pos = M.vertex_transform(verts, mvp[None])
    assert np.abs(pos[0] - clip).max() <= 1e-6 * np.abs(clip).max()
    assert np.abs(M.vertex_normals(verts, faces) - ref_vn).max() < 2e-6
    ours = M.render_mesh_normal(mvp[None], H, W, verts, faces)[0]
    rast = M.rasterize(pos, faces, H, W)[0]
    # the reference's matmul rounds its clip coordinates differently in the last bits: a pixel on an edge may change
    # triangle (and u, v carry that rounding, amplified by the triangle's conditioning)
    assert (rast[..., 3] == ref_rast[..., 3]).mean() > 0.995 and (rast[..., 3] > 0).sum() > 100
    # given the restatement's clip coordinates, the reference's normal rules give the restatement's image
    ref = _torch_render_mesh_normal(torch.from_numpy(mvp), H, W, torch.from_numpy(verts), torch.from_numpy(faces), clip=pos)[0]
    assert np.abs(ours - ref).max() < 2e-6
    assert np.array_equal(ours[rast[..., 3] == 0], np.ones_like(ours[rast[..., 3] == 0]))


def test_vertex_normals_order_and_degenerate_rules():
    """The documented order (corner 0 faces ascending, then corner 1, then corner 2), the (0, 0, 1) rule for a zero sum and
    a NaN one, and a face with an out-of-range index contributing nothing."""
    rng = np.random.default_rng(7)
    v = rng.normal(size=(6, 3)).astype(F)
    faces = np.array([[0, 1, 2], [2, 1, 0], [3, 3, 3], [1, 2, 4], [0, 9, 1]], np.int32)
    got = M.vertex_normals(v, faces)
    fn = M.face_normals(v, faces[:4])
    acc = ((np.zeros(3, F) + fn[1]) + fn[3]) + fn[0]  # vertex 2: corner 0 of face 1, corner 1 of face 3, corner 2 of face 0
    assert np.array_equal(got[2], M.safe_normalize(acc))
    assert np.array_equal(got[3], np.array([0, 0, 1], F)) and np.array_equal(got[5], np.array([0, 0, 1], F))
    v[4] = np.nan
    assert np.array_equal(M.vertex_normals(v, faces)[4], np.array([0, 0, 1], F))
