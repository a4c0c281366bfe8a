"""GPU: mesh rendering (humangaussian_b200.meshrender, csrc/meshraster.cu) against the numpy restatement
(tests/meshraster_reference.py), byte for byte.

  1. rast, interpolation, vertex normals and the normal image on triangle soups with overlaps and equal depths, pixel-
     centre-exact grids with shared edges, degenerate triangles, W <= 0 and near-plane crossings, out-of-range indices and
     NaN vertices, screen-filling triangles, H != W and sizes that are not multiples of 16, the reference's human body from
     orbit, near-head and near-back cameras, and a mesh from mesh.extract_mesh on the sample scene;
  2. batches: a 64-view call equals 64 one-view calls, a 65-view call is chunked, shared and per-view vertices;
  3. two runs write the same bytes;
  4. the argument errors, at the C ABI and in Python;
  5. the convention: a small Gaussian and a triangle fan around the same world point, rendered from the same CameraBatch,
     land on the same pixel.
NaN outputs (from NaN inputs) compare equal whatever their payload bits.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import meshraster_reference as M
from test_meshraster_cpu import corner_cuts, human, quad_grid, soup
from humangaussian_b200 import meshrender as MR
from humangaussian_b200 import rasterizer as R
from humangaussian_b200.cameras import CameraBatch, orbit_c2w

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F = np.float32


def same_bytes(got, want):
    got, want = np.asarray(got, F), np.asarray(want, F)
    if got.shape != want.shape:
        return False
    nan = np.isnan(got)
    return np.array_equal(nan, np.isnan(want)) and np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


def _t(a, dtype=torch.float32):
    return torch.tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def check_case(pos, tri, H, W, channels=(1, 3, 5), seed=0):
    """rast and interpolation (shared and per-view attributes) byte for byte against the restatement; returns rast."""
    rast = MR.rasterize(_t(pos), _t(tri, torch.int32), (H, W)).cpu().numpy()
    want = M.rasterize(pos, tri, H, W)
    assert same_bytes(rast, want), f"rast differs at {np.argwhere(rast != want)[:5]}"
    rng = np.random.default_rng(seed)
    V, Nv = pos.shape[:2]
    for Cn in channels:
        for shape in ((Nv, Cn), (V, Nv, Cn)):
            attr = rng.normal(size=shape).astype(F)
            got = MR.interpolate(_t(attr), _t(rast), _t(tri, torch.int32)).cpu().numpy()
            assert same_bytes(got, M.interpolate(attr, rast, tri)), (Cn, shape)
    return rast


@pytest.mark.parametrize("seed,n,H,W", [(0, 200, 64, 64), (1, 500, 37, 53), (2, 300, 100, 130), (3, 50, 16, 16), (4, 120, 1, 77)])
def test_triangle_soups(seed, n, H, W):
    pos, tri = soup(seed, n, V=3, behind=0.2)
    # equal depths: every fourth triangle is repeated at a higher index
    tri = np.concatenate([tri, tri[::4]]).astype(np.int32)
    rast = check_case(pos, tri, H, W, seed=seed)
    assert (rast[..., 3] > 0).mean() > (0.05 if H > 1 else 0.0)
    assert (rast[..., 3] <= n).all()  # a repeated triangle has its original's depths: the lower index wins every tie


@pytest.mark.parametrize("H,W", [(48, 48), (29, 41), (33, 16)])
def test_pixel_centre_exact_shared_edge_grids(H, W):
    pos, tri = quad_grid(9, 7, jitter=0.15, seed=H, V=2, exact_px=(H, W))
    rast = check_case(pos, tri, H, W)
    assert (rast[..., 3] > 0).all()  # shared edges: no pinholes
    pos, tri = quad_grid(6, 6, jitter=0.1, seed=W, V=2)
    assert (check_case(pos, tri, H, W)[..., 3] > 0).all()


def test_degenerate_behind_and_near_plane_triangles():
    H, W = 40, 56
    P = np.array([
        [-0.5, -0.5, 0.0, 1.0], [0.5, -0.5, 0.0, 1.0], [0.0, 0.6, 0.0, 1.0],      # 0-2 plain
        [-0.9, -0.9, 0.0, 1.0], [0.9, 0.9, 0.0, 1.0], [0.0, 0.0, 0.0, 1.0],       # 3-5 collinear: D = 0
        [0.3, 0.3, 0.5, -1.0], [-0.3, 0.2, 0.1, -0.5], [0.1, -0.4, 0.2, -2.0],    # 6-8 all W < 0
        [-0.8, -0.2, -0.9, 1.0], [0.7, -0.1, 0.5, -0.5], [0.0, 0.9, 0.2, 0.8],    # 9-11 crosses the camera plane
        [-0.6, -0.6, -1.5, 1.0], [0.6, -0.6, 1.5, 1.0], [0.0, 0.7, 0.0, 1.0],     # 12-14 crosses near and far
        [0.2, 0.2, 0.0, 0.0], [0.2, 0.2, 0.0, 0.0], [0.2, 0.2, 0.0, 0.0],         # 15-17 all W = 0
    ], F)[None]
    tri = np.array([[0, 1, 2], [3, 4, 5], [0, 0, 2], [6, 7, 8], [9, 10, 11], [11, 10, 9], [12, 13, 14], [15, 16, 17], [0, 2, 1]],
                   np.int32)
    rast = check_case(P, tri, H, W)
    ids = set(np.unique(rast[..., 3]).astype(int).tolist())
    assert {1, 7} <= ids and not ({2, 3, 4, 8, 9} & ids)
    # near / far: the pixels of triangle 6 where z/w leaves [-1, 1] are dropped
    flat = P.copy()
    flat[..., 2] = 0
    assert 0 < (M.rasterize(P, tri[6:7], H, W)[..., 3] > 0).sum() < (M.rasterize(flat, tri[6:7], H, W)[..., 3] > 0).sum()


@pytest.mark.parametrize("point", [False, True])
def test_point_sized_and_corner_cut_triangles(point):
    """Triangles whose edge functions are rounding noise (marching-cubes corner cuts at t ~ 0, and points within a few
    ulps), over a soup they compete with: the pixel rectangle decides the same pixels on the device as in the
    restatement."""
    H, W = 64, 48
    cut, ctri = corner_cuts(11 + point, 400, V=2, point=point)
    pos, tri = soup(12, 60, V=2)
    both = np.concatenate([cut, pos], 1)
    rast = check_case(both, np.concatenate([ctri, tri + cut.shape[1]]).astype(np.int32), H, W)
    alone = check_case(cut, ctri, H, W, channels=(3,))
    assert (alone[..., 3] > 0).sum() > 0 and (rast[..., 3] > len(ctri)).any()


def test_out_of_range_indices_and_nan_vertices():
    pos, tri = soup(5, 80, V=2)
    pos[0, 7, 1] = np.nan
    pos[1, 20, 3] = np.inf
    pos[1, 30, 0] = -np.inf
    bad = tri.copy()
    bad[3] = [0, -1, 2]
    bad[4] = [0, 1, pos.shape[1]]
    bad[5] = [2 ** 31 - 1, 1, 2]
    check_case(pos, bad.astype(np.int32), 45, 61)
    vn = MR.vertex_normals(_t(pos[0, :, :3]), _t(bad, torch.int32)).cpu().numpy()
    assert same_bytes(vn, M.vertex_normals(pos[0, :, :3], bad))
    # int64 indices beyond int32 (2^32 + 3 would wrap to vertex 3) are out of range too: the face is not drawn
    wide = tri.astype(np.int64)
    wide[6] = [2 ** 32 + 3, 4, 5]
    wide[7] = [-2 ** 33, 1, 2]
    rast = MR.rasterize(_t(pos), _t(wide, torch.int64), (45, 61)).cpu().numpy()
    assert same_bytes(rast, M.rasterize(pos, wide, 45, 61))
    assert same_bytes(MR.vertex_normals(_t(pos[0, :, :3]), _t(wide, torch.int64)).cpu().numpy(), M.vertex_normals(pos[0, :, :3], wide))


def test_single_triangles_covering_the_screen():
    H, W = 70, 90
    big = np.array([[[-50, -50, 0.3, 1], [60, -40, 0.3, 1], [0, 80, 0.3, 1]],
                    [[-3e4, -3e4, 0.1, 1], [3e4, -3e4, 0.1, 1], [0, 3e4, 0.1, 1]]], F)
    for v in range(2):
        rast = check_case(big[v:v + 1], np.array([[0, 1, 2]], np.int32), H, W)
        assert (rast[..., 3] == 1).all()


def human_views(H, W):
    """Orbit, near-head and near-back cameras on the human (z-up, feet near z = -1, head near z = 0.78)."""
    c2w, fov = [], []
    for el, az, d in ((10, 0, 2.8), (30, 70, 2.5), (-20, 160, 3.0), (0, 250, 2.6)):  # orbit
        c2w.append(orbit_c2w(el, az, d, (0.0, 0.0, -0.1))); fov.append(45.0)
    for el, az, d in ((5, 10, 0.45), (20, 300, 0.35)):                               # near the head
        c2w.append(orbit_c2w(el, az, d, (0.0, 0.0, 0.62))); fov.append(60.0)
    for el, az, d in ((0, 180, 0.4), (-10, 200, 0.25)):                              # near the back
        c2w.append(orbit_c2w(el, az, d, (0.0, 0.05, 0.1))); fov.append(70.0)
    return CameraBatch(torch.stack(c2w), [math.radians(f) for f in fov], H, W)


def test_human_from_orbit_near_head_and_near_back_cameras():
    H, W = 96, 80
    verts, faces = human()
    cams = human_views(H, W)
    mvp = MR.camera_mvp(cams).cpu().numpy()
    pos = MR.vertex_transform(_t(verts), _t(mvp)).cpu().numpy()
    assert same_bytes(pos, M.vertex_transform(verts, mvp))
    rast = check_case(pos, faces, H, W, channels=(3,))
    assert (rast[..., 3] > 0).mean(axis=(1, 2)).min() > 0.02
    assert (rast[4:, ..., 3] > 0).mean() > 0.3  # the close-ups are mostly body
    vn = MR.vertex_normals(_t(verts), _t(faces, torch.int32)).cpu().numpy()
    assert same_bytes(vn, M.vertex_normals(verts, faces))
    img = MR.render_mesh_normal(_t(mvp), H, W, _t(verts), _t(faces, torch.int32)).cpu().numpy()
    assert same_bytes(img, M.normal_image(M.vertex_normals(verts, faces), rast, faces))
    # per-view vertices: a different deformation per view
    rng = np.random.default_rng(1)
    frames = (verts[None] + rng.normal(scale=0.01, size=(len(mvp),) + verts.shape)).astype(F)
    img = MR.render_mesh_normal(_t(mvp), H, W, _t(frames), _t(faces, torch.int32)).cpu().numpy()
    assert same_bytes(img, M.render_mesh_normal(mvp, H, W, frames, faces))
    vn = MR.vertex_normals(_t(frames), _t(faces, torch.int32)).cpu().numpy()
    assert same_bytes(vn, M.vertex_normals(frames, faces))


def test_extract_mesh_output_on_the_sample_scene():
    from humangaussian_b200 import mesh as MX
    from humangaussian_b200.scene import sample_ply_scene
    m = MX.extract_mesh(sample_ply_scene().to(DEV), resolution=64)
    verts, faces = m.vertices.cpu().numpy(), m.faces.cpu().numpy()
    assert len(faces) > 1000
    H, W = 64, 48
    ctr = tuple(float(x) for x in (verts.min(0) + verts.max(0)) / 2)
    cams = CameraBatch(torch.stack([orbit_c2w(10, 45, 2.5, ctr), orbit_c2w(-5, 200, 2.0, ctr)]), [math.radians(50)] * 2, H, W)
    mvp = MR.camera_mvp(cams).cpu().numpy()
    rast = check_case(M.vertex_transform(verts, mvp), faces, H, W, channels=(3,))
    assert (rast[..., 3] > 0).mean() > 0.05
    assert same_bytes(MR.vertex_normals(m.vertices, m.faces).cpu().numpy(), M.vertex_normals(verts, faces))
    img = MR.render_mesh_normal(_t(mvp), H, W, m.vertices, m.faces).cpu().numpy()
    assert same_bytes(img, M.render_mesh_normal(mvp, H, W, verts, faces))


def test_batches_of_64_and_65_views_equal_single_view_calls():
    H, W = 48, 40
    verts, faces = human()
    rng = np.random.default_rng(2)
    c2w = torch.stack([orbit_c2w(float(rng.uniform(-30, 30)), float(rng.uniform(-180, 180)), float(rng.uniform(1.0, 3.0)), (0, 0, -0.1))
                       for _ in range(65)])
    mvp = MR.camera_mvp(CameraBatch(c2w, [math.radians(50)] * 65, H, W, device=DEV))
    frames = _t(verts[None] + rng.normal(scale=0.02, size=(65,) + verts.shape).astype(F))
    tri = _t(faces, torch.int32)
    for vin in (_t(verts), frames):
        pos = MR.vertex_transform(vin, mvp)
        r65 = MR.rasterize(pos, tri, (H, W))
        r64 = MR.rasterize(pos[:64], tri, (H, W))
        assert torch.equal(r65[:64].view(torch.int32), r64.view(torch.int32))
        ones = torch.cat([MR.rasterize(pos[v:v + 1], tri, (H, W)) for v in range(65)])
        assert torch.equal(r65.view(torch.int32), ones.view(torch.int32))
        img = MR.render_mesh_normal(mvp, H, W, vin, tri)
        one = torch.cat([MR.render_mesh_normal(mvp[v:v + 1], H, W, vin if vin.dim() == 2 else vin[v:v + 1], tri) for v in range(65)])
        assert torch.equal(img.view(torch.int32), one.view(torch.int32))
        it = MR.interpolate(vin, r65, tri)
        assert torch.equal(it[64:].view(torch.int32), MR.interpolate(vin if vin.dim() == 2 else vin[64:], r65[64:], tri).view(torch.int32))
    vn = MR.vertex_normals(frames, tri)
    assert torch.equal(vn[64].view(torch.int32), MR.vertex_normals(frames[64], tri).view(torch.int32))


def test_two_runs_write_identical_bytes():
    pos, tri = soup(9, 3000, V=4)
    tri = np.concatenate([tri, tri]).astype(np.int32)  # equal depths everywhere: the tie rule decides
    p, t = _t(pos), _t(tri, torch.int32)
    a = MR.rasterize(p, t, (256, 200))
    b = MR.rasterize(p, t, (256, 200))
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert a[..., 3].max().item() <= 3000  # the first copy of each triangle wins its ties


def test_argument_errors_at_the_c_abi():
    L = R.load_library()
    st = R._stream(DEV)
    pos = torch.zeros(2, 5, 4, device=DEV)
    tri = torch.zeros(3, 3, dtype=torch.int32, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
    need = L.b200gs_mesh_raster_scratch_bytes(2, 3, 32, 32)
    scr = torch.zeros(need + 64, dtype=torch.uint8, device=DEV)
    rast = torch.zeros(2, 32, 32, 4, device=DEV)
    ok = lambda *a: L.b200gs_mesh_raster_count(*a, R._ptr(cnt), st)  # noqa: E731
    assert ok(2, 5, 3, 32, 32, R._ptr(pos), R._ptr(tri), R._ptr(scr), need) == R.OK
    assert ok(0, 5, 3, 32, 32, R._ptr(pos), R._ptr(tri), R._ptr(scr), need) == R.E_RANGE
    assert ok(65, 5, 3, 32, 32, R._ptr(pos), R._ptr(tri), R._ptr(scr), need) == R.E_RANGE
    assert ok(2, 5, 3, 0, 32, R._ptr(pos), R._ptr(tri), R._ptr(scr), need) == R.E_RANGE
    assert ok(2, 5, 3, 32, 16385, R._ptr(pos), R._ptr(tri), R._ptr(scr), need) == R.E_RANGE
    assert ok(2, 5, 1 << 24, 32, 32, R._ptr(pos), R._ptr(tri), R._ptr(scr), need) == R.E_RANGE
    assert ok(2, -1, 3, 32, 32, R._ptr(pos), R._ptr(tri), R._ptr(scr), need) == R.E_ARGS
    assert ok(2, 5, 3, 32, 32, None, R._ptr(tri), R._ptr(scr), need) == R.E_ARGS
    assert ok(2, 5, 3, 32, 32, R._ptr(pos), R._ptr(tri), R._ptr(scr), need - 1) == R.E_BUFFER
    assert ok(2, 5, 3, 32, 32, C.c_void_p(pos.data_ptr() + 4), R._ptr(tri), R._ptr(scr), need) == R.E_BUFFER
    assert ok(2, 5, 3, 32, 32, R._ptr(pos), R._ptr(tri), C.c_void_p(scr.data_ptr() + 8), need) == R.E_BUFFER
    assert L.b200gs_mesh_raster_scratch_bytes(65, 3, 32, 32) == 0 and L.b200gs_mesh_raster_scratch_bytes(1, 1 << 24, 32, 32) == 0
    emit = lambda v, sb, pairs, pb, out: L.b200gs_mesh_raster_emit(v, 5, 3, 32, 32, R._ptr(scr), sb, pairs, pb, out, st)  # noqa: E731
    pairs = torch.zeros(64, dtype=torch.int32, device=DEV)
    assert emit(2, need, R._ptr(pairs), 256, R._ptr(rast)) == R.OK
    assert emit(65, need, R._ptr(pairs), 256, R._ptr(rast)) == R.E_RANGE
    assert emit(2, need - 1, R._ptr(pairs), 256, R._ptr(rast)) == R.E_BUFFER
    assert emit(2, need, C.c_void_p(pairs.data_ptr() + 4), 252, R._ptr(rast)) == R.E_BUFFER
    assert emit(2, need, R._ptr(pairs), 256, C.c_void_p(rast.data_ptr() + 4)) == R.E_BUFFER
    assert emit(2, need, None, 256, R._ptr(rast)) == R.E_ARGS
    out = torch.zeros(2, 32, 32, 3, device=DEV)
    vn = torch.zeros(5, 3, device=DEV)
    interp = lambda v, c, a_pv, r: L.b200gs_mesh_interpolate(v, 32, 32, 5, 3, c, R._ptr(vn), a_pv, r, R._ptr(tri), R._ptr(out), st)  # noqa: E731
    assert interp(2, 3, 0, R._ptr(rast)) == R.OK
    assert interp(2, 0, 0, R._ptr(rast)) == R.E_ARGS
    assert interp(2, 3, 2, R._ptr(rast)) == R.E_ARGS
    assert interp(65, 3, 0, R._ptr(rast)) == R.E_RANGE
    assert interp(2, 3, 0, C.c_void_p(rast.data_ptr() + 4)) == R.E_BUFFER
    assert L.b200gs_mesh_normal_image(2, 32, 32, 5, 3, R._ptr(vn), 0, R._ptr(rast), R._ptr(tri), R._ptr(out), st) == R.OK
    assert L.b200gs_mesh_normal_image(65, 32, 32, 5, 3, R._ptr(vn), 0, R._ptr(rast), R._ptr(tri), R._ptr(out), st) == R.E_RANGE
    assert L.b200gs_mesh_normal_image(2, 32, 32, 5, 3, R._ptr(vn), 0, C.c_void_p(rast.data_ptr() + 8), R._ptr(tri), R._ptr(out),
                                      st) == R.E_BUFFER
    ib = L.b200gs_mesh_incidence_bytes(5, 3)
    inc = torch.zeros(ib + 64, dtype=torch.uint8, device=DEV)
    assert L.b200gs_mesh_incidence(5, 3, R._ptr(tri), R._ptr(inc), ib, st) == R.OK
    assert L.b200gs_mesh_incidence(5, 3, R._ptr(tri), R._ptr(inc), ib - 1, st) == R.E_BUFFER
    assert L.b200gs_mesh_incidence(5, 3, R._ptr(tri), C.c_void_p(inc.data_ptr() + 4), ib, st) == R.E_BUFFER
    assert L.b200gs_mesh_incidence(5, 1 << 24, R._ptr(tri), R._ptr(inc), ib, st) == R.E_RANGE
    assert L.b200gs_mesh_incidence(-1, 3, R._ptr(tri), R._ptr(inc), ib, st) == R.E_ARGS
    nrm = lambda f, b: L.b200gs_mesh_vertex_normals(f, 5, 3, R._ptr(vn), R._ptr(tri), R._ptr(inc), b, R._ptr(out), st)  # noqa: E731
    assert nrm(1, ib) == R.OK
    assert nrm(65, ib) == R.E_RANGE and nrm(0, ib) == R.E_RANGE
    assert nrm(1, ib - 1) == R.E_BUFFER
    torch.cuda.synchronize()


def test_argument_errors_in_python():
    pos = torch.zeros(2, 5, 4, device=DEV)
    tri = torch.zeros(3, 3, dtype=torch.int32, device=DEV)
    for bad in (pos.cpu(), pos[..., :3], pos[0], pos.long()):
        with pytest.raises(ValueError):
            MR.rasterize(bad, tri, 32)
    for bad in (tri.cpu(), tri[:, :2], tri.float(), torch.zeros(1 << 24, 3, dtype=torch.int32, device=DEV)):
        with pytest.raises(ValueError):
            MR.rasterize(pos, bad, 32)
    for res in (0, (32,), (32, 16385), 32.0):
        with pytest.raises(ValueError):
            MR.rasterize(pos, tri, res)
    rast = MR.rasterize(pos, tri, (16, 24))
    assert not rast.requires_grad and rast.shape == (2, 16, 24, 4) and not rast.any()
    with pytest.raises(ValueError):
        MR.interpolate(torch.zeros(3, 5, 2, device=DEV), rast, tri)      # 3 views of attributes for 2 of rast
    with pytest.raises(ValueError):
        MR.interpolate(torch.zeros(5, 2, device=DEV), rast.double(), tri)
    mvp = torch.eye(4, device=DEV)[None].repeat(2, 1, 1)
    with pytest.raises(ValueError):
        MR.render_mesh_normal(mvp, 16, 16, torch.zeros(5, 2, device=DEV), tri)
    with pytest.raises(ValueError):
        MR.render_mesh_normal(mvp, 16, 16, torch.zeros(3, 5, 3, device=DEV), tri)
    with pytest.raises(ValueError):
        MR.vertex_transform(torch.zeros(5, 3, device=DEV), torch.eye(4, device=DEV))
    with pytest.raises(ValueError):
        MR.vertex_normals(torch.zeros(5, 3), tri)
    w = torch.zeros(5, 3, device=DEV, requires_grad=True)
    assert not MR.vertex_normals(w, tri).requires_grad and not MR.vertex_transform(w, mvp).requires_grad


def test_mesh_and_gaussian_renders_share_the_pixel_grid():
    """One small isotropic Gaussian and a triangle fan around the same world point, rendered from the same CameraBatch:
    the Gaussian's brightest pixel is covered by the fan."""
    H, W = 61, 83
    rng = np.random.default_rng(3)
    for k in range(4):
        ctr = rng.uniform(-0.3, 0.3, 3)
        cams = CameraBatch(orbit_c2w(float(rng.uniform(-40, 40)), float(rng.uniform(-180, 180)), 2.0, tuple(ctr))[None],
                           [math.radians(50)], H, W, device=DEV)
        p = torch.tensor(ctr + rng.uniform(-0.05, 0.05, 3), dtype=torch.float32)
        img = R.rasterize_views(means3D=p[None].to(DEV), opacities=torch.full((1, 1), 0.9, device=DEV),
                                viewmatrices=cams.world_view_transform, projmatrices=cams.full_proj_transform,
                                camposs=cams.camera_center, tanfovx=cams.tanfovx, tanfovy=cams.tanfovy, image_height=H,
                                image_width=W, bg=torch.zeros(3, device=DEV), sh_degree=0,
                                shs=torch.full((1, 1, 3), 2.0, device=DEV), scales=torch.full((1, 3), 0.004, device=DEV),
                                rotations=torch.tensor([[1.0, 0, 0, 0]], device=DEV))[0]
        g = img[0, 0].cpu().numpy()
        y, x = np.unravel_index(np.argmax(g), g.shape)
        assert g[y, x] > 0
        # a fan of 8 triangles of radius 0.05 (about 1.6 px) around p, in the plane facing the camera
        fwd = (cams.camera_center[0].cpu() - p).numpy()
        fwd /= np.linalg.norm(fwd)
        a = np.cross(fwd, [0.0, 0.0, 1.0]); a /= np.linalg.norm(a)
        b = np.cross(fwd, a)
        ring = [p.numpy() + 0.05 * (math.cos(t) * a + math.sin(t) * b) for t in np.linspace(0, 2 * math.pi, 9)[:-1]]
        verts = torch.tensor(np.array([p.numpy()] + ring), dtype=torch.float32, device=DEV)
        fan = torch.tensor([[0, 1 + i, 1 + (i + 1) % 8] for i in range(8)], dtype=torch.int32, device=DEV)
        rast = MR.rasterize(MR.vertex_transform(verts, MR.camera_mvp(cams)), fan, (H, W))[0].cpu().numpy()
        assert rast[y, x, 3] > 0, (k, y, x)
        cov = np.argwhere(rast[..., 3] > 0)
        assert np.abs(cov.mean(0) - [y, x]).max() < 1.0  # the fan is centred on the Gaussian's pixel
