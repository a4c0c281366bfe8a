"""Mesh rendering on the GPU (csrc/meshraster.cu): the forward surface of threestudio's NVDiffRasterizerContext
(vertex_transform, rasterize in instance mode, interpolate) and the reference viewer's mesh mode, `render_mesh_normal`
(animation.py:558-601), for a whole batch of views, without nvdiffrast.

  * rasterize: rast [V, H, W, 4] = (u, v, z/w, triangle + 1), 0 where no triangle covers the pixel centre; row 0 is clip
    y = -1, so a mesh rendered with camera_mvp(cameras) lines up pixel for pixel with the Gaussian render of the same
    cameras.  Triangles are sampled exactly at pixel centres with inclusive edges, with no clipping: z/w outside
    [-1, 1] is dropped per pixel.  A triangle covers no pixel outside its projected bounding box widened by one pixel
    (where every W > 0), which confines point-sized triangles.  The nearest triangle wins, a depth tie goes to the lower
    index.
  * interpolate: a0 u + a1 v + a2 ((1 - u) - v) of the winner's vertex attributes, 0 on the background.
  * vertex_normals: the reference's sum of face normals per vertex in a fixed order (its faces as corner 0, 1, then 2,
    each in face order), (0, 0, 1) for a degenerate sum, normalised.
  * render_mesh_normal: the reference's normal image, (n + 1) / 2 and 1.0 on the background, [V, H, W, 3].
Every float operation is pinned (DESIGN.md section 2): the outputs are the same bytes on every run, and equal the numpy
restatement in tests/meshraster_reference.py.  Forward only: nothing here has a gradient, and there is no CPU path.
Batches above 64 views are rendered in chunks of 64; each chunk of a rasterisation waits once on the host, for its
(tile, triangle) pair count.
"""
from __future__ import annotations

from typing import Tuple, Union

import torch

from . import rasterizer as R

MAX_VIEWS = 64          # B200GS_MAX_VIEWS: views per C call
MAX_FACES = 1 << 24     # triangle + 1 is exact in float32 below this
MAX_SIZE = 16384


def _err(fn, msg):
    return ValueError(f"b200gs: meshrender.{fn}: {msg}")


def _desc(t):
    return f"{t.dtype} {tuple(t.shape)} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__


def _float_cuda(fn, name, t, dims, dev=None):
    if not isinstance(t, torch.Tensor) or not t.dtype.is_floating_point or t.device.type != "cuda" or t.dim() not in dims or \
            (dev is not None and t.device != dev):
        raise _err(fn, f"{name} must be a floating-point CUDA tensor with {' or '.join(map(str, dims))} dimensions"
                   f"{' on ' + str(dev) if dev is not None else ''} (got {_desc(t)})")
    return t.detach().to(torch.float32).contiguous()


def _faces(fn, tri, dev):
    if not isinstance(tri, torch.Tensor) or tri.dtype.is_floating_point or tri.dtype == torch.bool or tri.dim() != 2 or \
            tri.shape[1] != 3 or tri.device != dev:
        raise _err(fn, f"tri must be an integer [Nf, 3] tensor on {dev} (got {_desc(tri)})")
    if tri.shape[0] >= MAX_FACES:
        raise _err(fn, f"at most {MAX_FACES - 1} triangles are supported (got {tri.shape[0]})")
    tri = tri.detach()
    if tri.dtype not in (torch.int32, torch.int16, torch.int8, torch.uint8):
        # an index outside int32 would wrap in the cast and could name a real vertex: make it -1, which is never drawn
        tri = torch.where((tri < -2 ** 31) | (tri > 2 ** 31 - 1), -1, tri)
    return tri.to(torch.int32).contiguous()


def _resolution(fn, resolution):
    hw = (resolution, resolution) if isinstance(resolution, int) else \
        tuple(resolution) if isinstance(resolution, (tuple, list)) else ()
    if len(hw) != 2 or not all(isinstance(x, int) and not isinstance(x, bool) and 1 <= x <= MAX_SIZE for x in hw):
        raise _err(fn, f"resolution must be an int or an (H, W) pair of ints in 1..{MAX_SIZE} (got {resolution!r})")
    return hw


def _aligned(t):
    return t if t.data_ptr() % 16 == 0 else t.clone()


def camera_mvp(cameras) -> torch.Tensor:
    """The mvp [V, 4, 4] of a CameraBatch (or anything with full_proj_transform [V, 4, 4] in the row-vector convention):
    full_proj_transform transposed, so that a mesh rendered with it lines up with the Gaussian render of the cameras."""
    return cameras.full_proj_transform.transpose(1, 2).contiguous()


@torch.no_grad()
def vertex_transform(vertices: torch.Tensor, mvp: torch.Tensor) -> torch.Tensor:
    """[x, y, z, 1] @ mvp^T per view: vertices [Nv, 3] (shared) or [V, Nv, 3], mvp [V, 4, 4] -> clip coordinates [V, Nv, 4].
    Row r is ((m_r0 x + m_r1 y) + m_r2 z) + m_r3 in float32, one rounding per operation (elementwise, no FMA)."""
    m = _float_cuda("vertex_transform", "mvp", mvp, (3,))
    if m.shape[1:] != (4, 4) or m.shape[0] < 1:
        raise _err("vertex_transform", f"mvp must be [V, 4, 4] with V >= 1 (got {tuple(mvp.shape)})")
    v = _float_cuda("vertex_transform", "vertices", vertices, (2, 3), m.device)
    if v.shape[-1] != 3 or (v.dim() == 3 and v.shape[0] != m.shape[0]):
        raise _err("vertex_transform", f"vertices must be [Nv, 3] or [{m.shape[0]}, Nv, 3] (got {tuple(vertices.shape)})")
    if v.dim() == 2:
        v = v.unsqueeze(0)
    x, y, z = v[..., 0], v[..., 1], v[..., 2]
    rows = [((m[:, r, 0, None] * x + m[:, r, 1, None] * y) + m[:, r, 2, None] * z) + m[:, r, 3, None] for r in range(4)]
    return torch.stack(rows, -1).contiguous()


def _rasterize_chunk(L, pos, tri, H, W, dev, out):
    V, Nv, Nf = pos.shape[0], pos.shape[1], tri.shape[0]
    st = R._stream(dev)
    scratch = torch.empty(L.b200gs_mesh_raster_scratch_bytes(V, Nf, H, W), dtype=torch.uint8, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    R._check(L.b200gs_mesh_raster_count(V, Nv, Nf, H, W, R._ptr(pos), R._ptr(tri), R._ptr(scratch), scratch.numel(), R._ptr(count), st),
             "mesh_raster_count")
    n_pairs = int(count.item())  # the one host wait: the size of the tile lists
    pairs = torch.empty(max(n_pairs, 1), dtype=torch.int32, device=dev)
    R._check(L.b200gs_mesh_raster_emit(V, Nv, Nf, H, W, R._ptr(scratch), scratch.numel(), R._ptr(pairs), 4 * n_pairs, R._ptr(out), st),
             "mesh_raster_emit")


@torch.no_grad()
def rasterize(pos: torch.Tensor, tri: torch.Tensor, resolution: Union[int, Tuple[int, int]]) -> torch.Tensor:
    """nvdiffrast's rasterize in instance mode: pos [V, Nv, 4] clip coordinates, tri [Nf, 3] (int32 or any integer type),
    resolution H or (H, W) -> rast [V, H, W, 4] float32 (u, v, z/w, triangle + 1).  A triangle with an index outside
    [0, Nv), a non-finite coordinate or W <= 0 at all three vertices is not drawn."""
    p = _float_cuda("rasterize", "pos", pos, (3,))
    if p.shape[-1] != 4 or p.shape[0] < 1:
        raise _err("rasterize", f"pos must be [V, Nv, 4] with V >= 1 (got {tuple(pos.shape)})")
    dev = p.device
    t = _faces("rasterize", tri, dev)
    H, W = _resolution("rasterize", resolution)
    L = R.load_library()
    with torch.cuda.device(dev):
        rast = torch.empty(p.shape[0], H, W, 4, dtype=torch.float32, device=dev)
        for v0 in range(0, p.shape[0], MAX_VIEWS):
            _rasterize_chunk(L, _aligned(p[v0:v0 + MAX_VIEWS]), t, H, W, dev, rast[v0:v0 + MAX_VIEWS])
    return rast


def _check_rast(fn, rast):
    if not isinstance(rast, torch.Tensor) or rast.dtype != torch.float32 or rast.device.type != "cuda" or rast.dim() != 4 or \
            rast.shape[-1] != 4 or rast.shape[0] < 1 or not (1 <= rast.shape[1] <= MAX_SIZE and 1 <= rast.shape[2] <= MAX_SIZE):
        raise _err(fn, f"rast must be a float32 CUDA tensor [V, H, W, 4] (got {_desc(rast)})")
    return _aligned(rast.detach().contiguous())


def _per_view_attr(fn, name, attr, V, C_fixed, dev):
    a = _float_cuda(fn, name, attr, (2, 3), dev)
    if (a.dim() == 3 and a.shape[0] != V) or (C_fixed is not None and a.shape[-1] != C_fixed) or a.shape[-1] < 1:
        want = f"[Nv, {C_fixed or 'C'}] or [{V}, Nv, {C_fixed or 'C'}]"
        raise _err(fn, f"{name} must be {want} (got {tuple(attr.shape)})")
    return a


@torch.no_grad()
def interpolate(attr: torch.Tensor, rast: torch.Tensor, tri: torch.Tensor) -> torch.Tensor:
    """nvdiffrast's interpolate (no derivatives): attr [V, Nv, C] or [Nv, C] (shared by every view), rast [V, H, W, 4] from
    rasterize, tri [Nf, 3] -> [V, H, W, C] float32: a0 u + a1 v + a2 ((1 - u) - v) where rast.w > 0, 0 elsewhere."""
    r = _check_rast("interpolate", rast)
    dev = r.device
    V, H, W = r.shape[:3]
    a = _per_view_attr("interpolate", "attr", attr, V, None, dev)
    t = _faces("interpolate", tri, dev)
    Nv, Cn, per_view = a.shape[-2], a.shape[-1], int(a.dim() == 3)
    L = R.load_library()
    with torch.cuda.device(dev):
        out = torch.empty(V, H, W, Cn, dtype=torch.float32, device=dev)
        for v0 in range(0, V, MAX_VIEWS):
            n = min(MAX_VIEWS, V - v0)
            R._check(L.b200gs_mesh_interpolate(n, H, W, Nv, t.shape[0], Cn, R._ptr(a[v0:v0 + n] if per_view else a), per_view,
                                               R._ptr(r[v0:v0 + n]), R._ptr(t), R._ptr(out[v0:v0 + n]), R._stream(dev)),
                     "mesh_interpolate")
    return out


def _incidence(L, Nv, t, dev):
    inc = torch.empty(L.b200gs_mesh_incidence_bytes(Nv, t.shape[0]), dtype=torch.uint8, device=dev)
    R._check(L.b200gs_mesh_incidence(Nv, t.shape[0], R._ptr(t), R._ptr(inc), inc.numel(), R._stream(dev)), "mesh_incidence")
    return inc


def _vertex_normals(L, v, t, dev):
    F, Nv = v.shape[0], v.shape[1]
    inc = _incidence(L, Nv, t, dev)  # once per topology, for every frame
    out = torch.empty(F, Nv, 3, dtype=torch.float32, device=dev)
    for f0 in range(0, F, MAX_VIEWS):
        n = min(MAX_VIEWS, F - f0)
        R._check(L.b200gs_mesh_vertex_normals(n, Nv, t.shape[0], R._ptr(v[f0:f0 + n]), R._ptr(t), R._ptr(inc), inc.numel(),
                                              R._ptr(out[f0:f0 + n]), R._stream(dev)), "mesh_vertex_normals")
    return out


@torch.no_grad()
def vertex_normals(vertices: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """The reference's vertex normals (animation.py:573-590) in a fixed order: vertices [Nv, 3] or [F, Nv, 3] (frames of
    one topology), faces [Nf, 3] -> normals of the same shape.  Each vertex sums cross(v1 - v0, v2 - v0) of its faces
    where it is corner 0 (ascending face index), then corner 1, then corner 2; a sum whose dot is not > 1e-20 becomes
    (0, 0, 1); then x / sqrt(max(dot(x, x), 1e-20)).  A face with an index outside [0, Nv) adds nothing."""
    v = _float_cuda("vertex_normals", "vertices", vertices, (2, 3))
    if v.shape[-1] != 3 or (v.dim() == 3 and v.shape[0] < 1):
        raise _err("vertex_normals", f"vertices must be [Nv, 3] or [F, Nv, 3] (got {tuple(vertices.shape)})")
    dev = v.device
    t = _faces("vertex_normals", faces, dev)
    L = R.load_library()
    with torch.cuda.device(dev):
        out = _vertex_normals(L, v if v.dim() == 3 else v[None], t, dev)
    return out if v.dim() == 3 else out[0]


@torch.no_grad()
def render_mesh_normal(mvp: torch.Tensor, height: int, width: int, vertices: torch.Tensor, faces: torch.Tensor) -> torch.Tensor:
    """The reference viewer's mesh mode (GUI.render_mesh_normal) for V views: mvp [V, 4, 4] (camera_mvp(cameras) for the
    Gaussian cameras), vertices [Nv, 3] shared by every view or [V, Nv, 3] one posed frame per view, faces [Nf, 3] ->
    [V, height, width, 3] float32 HWC: (safe_normalize(interpolated vertex normal) + 1) / 2 on the mesh, 1.0 elsewhere."""
    m = _float_cuda("render_mesh_normal", "mvp", mvp, (3,))
    if m.shape[1:] != (4, 4) or m.shape[0] < 1:
        raise _err("render_mesh_normal", f"mvp must be [V, 4, 4] with V >= 1 (got {tuple(mvp.shape)})")
    dev = m.device
    V = m.shape[0]
    v = _per_view_attr("render_mesh_normal", "vertices", vertices, V, 3, dev)
    t = _faces("render_mesh_normal", faces, dev)
    H, W = _resolution("render_mesh_normal", (height, width))
    pos = vertex_transform(v, m)
    per_view = int(v.dim() == 3)
    L = R.load_library()
    with torch.cuda.device(dev):
        vn = _vertex_normals(L, v if per_view else v[None], t, dev)
        out = torch.empty(V, H, W, 3, dtype=torch.float32, device=dev)
        rast = torch.empty(min(V, MAX_VIEWS), H, W, 4, dtype=torch.float32, device=dev)
        for v0 in range(0, V, MAX_VIEWS):
            n = min(MAX_VIEWS, V - v0)
            _rasterize_chunk(L, pos[v0:v0 + n], t, H, W, dev, rast[:n])
            R._check(L.b200gs_mesh_normal_image(n, H, W, v.shape[-2], t.shape[0], R._ptr(vn[v0:v0 + n] if per_view else vn), per_view,
                                                R._ptr(rast[:n]), R._ptr(t), R._ptr(out[v0:v0 + n]), R._stream(dev)), "mesh_normal_image")
    return out
