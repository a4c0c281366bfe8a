"""Mesh export: the Gaussians' opacity-weighted density field on a voxel grid, and marching cubes over it, on the GPU.

`extract_fields` is the reference's `GaussianModel.extract_fields` (gs_renderer.py:241-331) with the same definition,
quirks included (DESIGN.md section 2):
  * only Gaussians with opacity > 0.005 count; their centres are normalised by center = (min + max) / 2 and
    scale = 1.8 / max(max - min) (a Python float), scales are multiplied by the same scale, and the covariance is
    R(q / |q|) diag(s)^2 R(q / |q|)^T from the rotations as given (normalised again, with no epsilon);
  * the grid samples are torch.linspace(-1, 1, resolution) per axis, field[x, y, z] ('ij' indexing);
  * blocks are chunks of resolution // num_blocks samples per axis; a Gaussian counts for a block iff its centre lies
    strictly inside the block's sample range widened by (2 / num_blocks) * relax_ratio on all three axes.
Those P-sized steps are the reference's own torch ops; the field itself is one CUDA pipeline (csrc/mesh.cu) with a fixed
summation order, so it is the same bits on every run.  `marching_cubes` is a GPU marching cubes with a generated table
(mc_table.py): one welded vertex per crossing grid edge, triangles facing lower density.  `extract_mesh` chains the two
and maps the vertices back to world space as the reference does; by default the output is the raw marching-cubes mesh.
`clean_mesh` (floater removal by connected component) and `decimate_mesh` (quadric edge collapse to a face budget) are
the GPU counterparts of the reference's pymeshlab clean_mesh / decimate_mesh (csrc/meshclean.cu), and extract_mesh runs
them on request.  Isotropic remeshing is not done.  There is no CPU path.

`query_field` evaluates the same field at arbitrary world points (csrc/mesh.cu, b200gs_field_query): the density, the
outward normal -grad / |grad|, and the SH colour of the opacity-weighted mean coefficients seen along -normal.
`extract_colored_mesh` is `extract_mesh` with per-vertex normals and colours from it; `save_obj` and `save_ply_mesh`
write them.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import numpy as np
import torch

from . import rasterizer as R
from .scene import GaussianParams

OPACITY_MIN = 0.005  # the reference's pre-filter


class Fields(NamedTuple):
    occ: torch.Tensor     # float32 [res, res, res] on the device
    center: torch.Tensor  # float32 [3]: the kept centres' bounding-box centre
    scale: float          # 1.8 / the bounding box's longest side


def _f32_cuda(t, name, shape_ok, dev=None):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.device.type != "cuda" or not shape_ok(t) or \
            (dev is not None and t.device != dev):
        desc = f"{tuple(t.shape)} {t.dtype} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
        raise ValueError(f"b200gs: mesh: {name} has the wrong shape, dtype or device ({desc})")
    return t.detach()


def _check_grid(resolution, num_blocks):
    if not isinstance(resolution, (int, np.integer)) or not isinstance(num_blocks, (int, np.integer)) or resolution < 1 or \
            num_blocks < 1:
        raise ValueError(f"b200gs: extract_fields: resolution and num_blocks must be positive integers (got {resolution!r}, "
                         f"{num_blocks!r})")
    resolution, num_blocks = int(resolution), int(num_blocks)
    if resolution % (2 / num_blocks) != 0:  # the reference's `assert resolution % block_size == 0`, as a float modulo
        raise ValueError(f"b200gs: extract_fields: resolution {resolution} is not a multiple of the block size 2 / {num_blocks}")
    if resolution // num_blocks < 1:
        raise ValueError(f"b200gs: extract_fields: {num_blocks} blocks do not fit {resolution} samples per axis")
    return resolution, num_blocks


def _covariance(stds, rotations):
    """build_scaling_rotation + L @ L^T of the reference, element by element: R(q / |q|) with |q| = sqrt of the squares
    summed left to right and no epsilon; L = R diag(s) (the matmul with a diagonal adds exact zeros); cov[i][k] =
    L[i,0] L[k,0] + L[i,1] L[k,1] + L[i,2] L[k,2].  Returns [P,6] = xx, xy, xz, yy, yz, zz."""
    r = rotations
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    Rm = [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
          [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
          [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]
    L = [[Rm[i][j] * stds[:, j] for j in range(3)] for i in range(3)]
    cov = lambda i, k: L[i][0] * L[k][0] + L[i][1] * L[k][1] + L[i][2] * L[k][2]
    return torch.stack([cov(0, 0), cov(0, 1), cov(0, 2), cov(1, 1), cov(1, 2), cov(2, 2)], dim=1).contiguous()


class _Kept(NamedTuple):
    """The Gaussians extract_fields counts, in the field's normalised frame."""
    xyz: torch.Tensor    # [n,3] normalised centres
    cov6: torch.Tensor   # [n,6] normalised covariances
    opac: torch.Tensor   # [n] activated opacities
    keep: torch.Tensor   # bool [P]
    center: torch.Tensor
    scale: float


def _unwrap(fn, means3D, opacities, scales, rotations, raw, shs=None, sh_degree=None):
    """A GaussianParams -> its raw tensors, shs = cat(features_dc, features_rest) and its sh_degree."""
    if isinstance(means3D, GaussianParams):
        if opacities is not None or scales is not None or rotations is not None or shs is not None:
            raise ValueError(f"b200gs: {fn}: pass either a GaussianParams or the tensors")
        g = means3D
        shs = torch.cat([g.features_dc, g.features_rest], 1)
        return g.xyz, g.opacity, g.scaling, g.rotation, True, shs, g.sh_degree if sh_degree is None else sh_degree
    return means3D, opacities, scales, rotations, raw, shs, sh_degree


def _kept(fn, means3D, opacities, scales, rotations, raw, resolution, num_blocks):
    """extract_fields' checks, kept set, bounding-box normalisation and covariances."""
    dev = means3D.device if isinstance(means3D, torch.Tensor) else None
    if dev is None or dev.type != "cuda":
        raise RuntimeError("b200gs: tensors must live on a CUDA device (there is no CPU path)")
    resolution, num_blocks = _check_grid(resolution, num_blocks)
    P = means3D.shape[0] if means3D.dim() == 2 else -1
    means3D = _f32_cuda(means3D, "means3D", lambda t: t.dim() == 2 and t.shape[1] == 3)
    opacities = _f32_cuda(opacities, "opacities", lambda t: tuple(t.shape) in ((P,), (P, 1)), dev).reshape(P)
    scales = _f32_cuda(scales, "scales", lambda t: tuple(t.shape) == (P, 3), dev)
    rotations = _f32_cuda(rotations, "rotations", lambda t: tuple(t.shape) == (P, 4), dev)

    opac = torch.sigmoid(opacities) if raw else opacities
    keep = opac > OPACITY_MIN
    xyz = means3D[keep]
    if xyz.shape[0] == 0:
        raise ValueError(f"b200gs: {fn}: no Gaussian has opacity > {OPACITY_MIN}")
    if not bool(torch.isfinite(xyz).all()):
        raise ValueError(f"b200gs: {fn}: a kept Gaussian has a non-finite position")
    stds = torch.exp(scales[keep]) if raw else scales[keep]
    mn, mx = xyz.amin(0), xyz.amax(0)
    center = (mn + mx) / 2
    extent = (mx - mn).amax().item()
    if extent == 0:
        raise ValueError(f"b200gs: {fn}: the kept Gaussians' centres are a single point")
    scale = 1.8 / extent
    xyz = ((xyz - center) * scale).contiguous()
    cov6 = _covariance(stds * scale, rotations[keep])
    return _Kept(xyz, cov6, opac[keep].contiguous(), keep, center, scale), resolution, num_blocks


@torch.no_grad()
def extract_fields(means3D, opacities=None, scales=None, rotations=None, *, raw=False, resolution=128, num_blocks=16,
                   relax_ratio=1.5) -> Fields:
    """The density field [resolution]^3 of a Gaussian set, on its device.

    means3D [P,3], opacities [P] or [P,1], scales [P,3], rotations [P,4], float32 on one CUDA device.  raw=False: the
    activated values (sigmoid opacities, exp scales); raw=True: the optimiser's raw fields (opacity logits, log-scales),
    activated here as the reference does -- views of the packed buffer (`rasterizer.packed_layout`) work as they are.
    A `scene.GaussianParams` may be passed as means3D alone; it is raw.  Rotations are normalised here either way.
    Raises ValueError for a (resolution, num_blocks) pair the reference's assertion rejects, when no Gaussian has
    opacity > 0.005, when a kept centre is not finite, or when the kept centres are all one point."""
    if isinstance(means3D, GaussianParams):
        if opacities is not None or scales is not None or rotations is not None:
            raise ValueError("b200gs: extract_fields: pass either a GaussianParams or the four tensors")
        means3D, opacities, scales, rotations, raw = means3D.xyz, means3D.opacity, means3D.scaling, means3D.rotation, True
    k, resolution, num_blocks = _kept("extract_fields", means3D, opacities, scales, rotations, raw, resolution, num_blocks)
    return Fields(_density_field(k.xyz, k.cov6, k.opac, resolution, num_blocks, relax_ratio), k.center, k.scale)


def _samples_relax(dev, resolution, num_blocks, relax_ratio):
    samples = torch.linspace(-1, 1, resolution).to(dev)  # built on the CPU, as the reference builds it
    return samples, float(np.float32((2 / num_blocks) * relax_ratio))


def _density_field(xyz, cov6, opac, resolution, num_blocks, relax_ratio):
    """b200gs_density_field on normalised centres [n,3], covariances [n,6] and opacities [n] (all kept)."""
    dev, n = xyz.device, xyz.shape[0]
    samples, relax = _samples_relax(dev, resolution, num_blocks, relax_ratio)
    occ = torch.empty((resolution,) * 3, dtype=torch.float32, device=dev)
    L = R.load_library()
    with torch.cuda.device(dev):
        scratch = torch.empty(L.b200gs_density_field_scratch_bytes(n, resolution, num_blocks), dtype=torch.uint8, device=dev)
        R._check(L.b200gs_density_field(n, R._ptr(xyz), R._ptr(cov6), R._ptr(opac), resolution, num_blocks, R._ptr(samples), relax,
                                        R._ptr(occ), R._ptr(scratch), scratch.numel(), R._stream(dev)), "density_field")
    return occ


@torch.no_grad()
def marching_cubes(volume: torch.Tensor, iso: float):
    """Marching cubes of a float32 [X,Y,Z] CUDA volume at `iso` -> (vertices float32 [V,3] in index coordinates,
    faces int32 [F,3]).  A corner is inside iff value > iso; one vertex per crossing grid edge, shared by every cell around
    it, at t = (iso - v0) / (v1 - v0) along the edge; triangles face lower values.  Vertices come in order of (grid point
    at the edge's low end, axis), faces in order of (cell, table row).  The same surface as `mcubes.marching_cubes`, not
    necessarily the same triangle list.  One host wait, to size the outputs."""
    v = _f32_cuda(volume, "volume", lambda t: t.dim() == 3)
    X, Y, Z = (int(s) for s in v.shape)
    if min(X, Y, Z) < 2:
        raise ValueError(f"b200gs: marching_cubes: every side must have at least 2 samples (got {X}x{Y}x{Z})")
    if 3 * X * Y * Z > 0x7FFFFFFF:
        raise ValueError(f"b200gs: marching_cubes: a {X}x{Y}x{Z} grid has more edges than int32 vertex ids can number "
                         f"(3*X*Y*Z must stay below 2^31)")
    v = v.contiguous()
    dev = v.device
    L = R.load_library()
    with torch.cuda.device(dev):
        scratch = torch.empty(L.b200gs_marching_cubes_scratch_bytes(X, Y, Z), dtype=torch.uint8, device=dev)
        counts = torch.zeros(2, dtype=torch.int64, device=dev)  # uint64 on the device; the counts stay far below 2^63
        st = R._stream(dev)
        R._check(L.b200gs_marching_cubes_count(X, Y, Z, R._ptr(v), float(iso), R._ptr(scratch), scratch.numel(), R._ptr(counts), st),
                 "marching_cubes_count")
        nv, nf = (int(c) for c in counts.cpu())  # the one host wait
        verts = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        faces = torch.empty(nf, 3, dtype=torch.int32, device=dev)
        if nv or nf:
            R._check(L.b200gs_marching_cubes_emit(X, Y, Z, R._ptr(v), float(iso), R._ptr(scratch), scratch.numel(),
                                                  R._ptr(verts) if nv else None, R._ptr(faces) if nf else None, st),
                     "marching_cubes_emit")
    return verts, faces


class Mesh(NamedTuple):
    vertices: torch.Tensor  # float32 [V,3], world space
    faces: torch.Tensor     # int32 [F,3]


def _edit_args(fn, vertices, faces):
    v = _f32_cuda(vertices, "vertices", lambda t: t.dim() == 2 and t.shape[1] == 3)
    if not isinstance(faces, torch.Tensor) or faces.dtype != torch.int32 or faces.device != v.device or faces.dim() != 2 or \
            faces.shape[1] != 3:
        desc = f"{tuple(faces.shape)} {faces.dtype} on {faces.device}" if isinstance(faces, torch.Tensor) else type(faces).__name__
        raise ValueError(f"b200gs: {fn}: faces must be int32 [F,3] on the vertices' device ({desc})")
    Nv, Nf = int(v.shape[0]), int(faces.shape[0])
    if Nv >= 0x7FFFFFFF or Nf >= 1 << 24:
        raise ValueError(f"b200gs: {fn}: {Nv} vertices / {Nf} faces exceed 2^31 - 1 / 2^24")
    return v.contiguous(), faces.detach().contiguous(), Nv, Nf


def _edit(fn, vertices, faces, call, scratch_bytes):
    """Runs b200gs_mesh_clean / _decimate -> (Mesh in the input's frame, rounds)."""
    import ctypes as C
    v, f, Nv, Nf = _edit_args(fn, vertices, faces)
    dev = v.device
    L = R.load_library()
    with torch.cuda.device(dev):
        scratch = torch.empty(max(1, scratch_bytes(L, Nv, Nf)), dtype=torch.uint8, device=dev)
        ov = torch.empty(Nv, 3, dtype=torch.float32, device=dev)
        of = torch.empty(Nf, 3, dtype=torch.int32, device=dev)
        counts, rounds = (C.c_int64 * 2)(), C.c_int32(0)
        rc = call(L, Nv, Nf, R._ptr(v), R._ptr(f), R._ptr(scratch), scratch.numel(), R._ptr(ov), R._ptr(of), counts, C.byref(rounds),
                  R._stream(dev))
    if rc == R.E_ARGS:
        raise ValueError(f"b200gs: {fn}: a face index lies outside [0, {Nv})")
    R._check(rc, fn)
    return Mesh(ov[:counts[0]], of[:counts[1]]), int(rounds.value)


@torch.no_grad()
def clean_mesh(vertices, faces, *, min_faces=64, min_diameter=0.2) -> Mesh:
    """Floater removal (DESIGN.md section 2) on a float32 [V,3] / int32 [F,3] CUDA mesh: drops faces that repeat a
    vertex index and faces whose vertex set repeats an earlier face's, then every connected component (faces sharing a
    vertex) with fewer than min_faces faces or whose bounding-box diagonal is below min_diameter times the whole mesh's,
    then unreferenced vertices.  Surviving vertices and faces keep their order, and vertex bytes are unchanged; every run
    gives the same bytes.  The defaults are recalled from kiui's clean_mesh (min_f=64, min_d=20 %), which the reference
    calls; they have not been checked against its source.  pymeshlab's other cleanup steps are left out: marching cubes
    already welds one vertex per grid edge, its table gives closed 2-manifolds, and remeshing is out of scope.
    Raises ValueError for bad arguments or a face index outside [0, V)."""
    if not isinstance(min_faces, (int, np.integer)) or min_faces < 0 or not np.isfinite(min_diameter) or min_diameter < 0:
        raise ValueError(f"b200gs: clean_mesh: min_faces must be an integer >= 0 and min_diameter finite and >= 0 "
                         f"(got {min_faces!r}, {min_diameter!r})")
    return _edit("clean_mesh", vertices, faces,
                 lambda L, Nv, Nf, *a: L.b200gs_mesh_clean(Nv, Nf, a[0], a[1], int(min_faces), float(min_diameter), *a[2:]),
                 lambda L, Nv, Nf: L.b200gs_mesh_clean_scratch_bytes(Nv, Nf))[0]


def _decimate(vertices, faces, target):
    if not isinstance(target, (int, np.integer)) or target < 4:
        raise ValueError(f"b200gs: decimate_mesh: target must be an integer >= 4 (got {target!r})")
    target = min(int(target), 0x7FFFFFFF)
    return _edit("decimate_mesh", vertices, faces,
                 lambda L, Nv, Nf, *a: L.b200gs_mesh_decimate(Nv, Nf, a[0], a[1], target, *a[2:]),
                 lambda L, Nv, Nf: L.b200gs_mesh_decimate_scratch_bytes(Nv, Nf))


@torch.no_grad()
def decimate_mesh(vertices, faces, target) -> Mesh:
    """Quadric edge collapse (Garland-Heckbert) of a float32 [V,3] / int32 [F,3] CUDA mesh to at most `target` faces, in
    parallel rounds on the GPU (DESIGN.md section 2 is the definition): area-weighted plane quadrics in float64, the
    optimal position where the 3x3 system is well conditioned, else the cheapest of the two ends and the midpoint;
    boundary and non-manifold vertices stay, every collapse keeps the link condition and flips no face.  A closed
    manifold ends at target or target - 1 faces.  When no valid collapse is left above `target`, the mesh at that point
    is returned with a warning.  Vertex attributes are not carried; query the field at the new vertices
    (extract_colored_mesh does).  Surviving faces keep their order; every run gives the same bytes."""
    m, _ = _decimate(vertices, faces, target)
    if m.faces.shape[0] > target:
        import warnings
        warnings.warn(f"b200gs: decimate_mesh: stopped at {m.faces.shape[0]} faces, above the target {target}: no valid collapse "
                      f"is left (boundary, non-manifold or topology-changing edges)", RuntimeWarning, stacklevel=2)
    return m


def _check_edit(clean, min_faces, min_diameter, decimate_target):
    if not isinstance(decimate_target, (int, np.integer)) or (decimate_target != 0 and decimate_target < 4):
        raise ValueError(f"b200gs: extract_mesh: decimate_target must be 0 (off) or an integer >= 4 (got {decimate_target!r})")
    if clean and (not isinstance(min_faces, (int, np.integer)) or min_faces < 0 or not np.isfinite(min_diameter) or min_diameter < 0):
        raise ValueError(f"b200gs: extract_mesh: min_faces must be an integer >= 0 and min_diameter finite and >= 0 "
                         f"(got {min_faces!r}, {min_diameter!r})")


def _mesh(k, resolution, num_blocks, relax_ratio, density_thresh, clean=False, min_faces=64, min_diameter=0.2, decimate_target=0):
    """-> (index-space vertices, faces, world vertices) of extract_mesh from the kept set k; cleanup and decimation run
    on the index-space mesh (grid pitch 1)."""
    occ = _density_field(k.xyz, k.cov6, k.opac, resolution, num_blocks, relax_ratio)
    v, faces = marching_cubes(occ, density_thresh)
    if clean:
        v, faces = clean_mesh(v, faces, min_faces=min_faces, min_diameter=min_diameter)
    if decimate_target:
        v, faces = decimate_mesh(v, faces, decimate_target)
    w = (v.double() / (resolution - 1.0) * 2 - 1) / k.scale + k.center.double()
    return v, faces, w.float()


@torch.no_grad()
def extract_mesh(means3D, opacities=None, scales=None, rotations=None, *, raw=False, density_thresh=1.0, resolution=128,
                 num_blocks=16, relax_ratio=1.5, clean=False, min_faces=64, min_diameter=0.2, decimate_target=0) -> Mesh:
    """The reference's extract_mesh up to its remeshing: extract_fields, marching cubes at density_thresh, and the vertices
    mapped back to world space as v / (resolution - 1) * 2 - 1, then / scale + center (in float64, stored as float32).
    clean=True runs clean_mesh(min_faces, min_diameter) and decimate_target > 0 runs decimate_mesh to that many faces,
    in that order, on the index-space mesh before the world mapping; the defaults give the raw marching-cubes mesh."""
    _check_edit(clean, min_faces, min_diameter, decimate_target)
    if isinstance(means3D, GaussianParams):
        if opacities is not None or scales is not None or rotations is not None:
            raise ValueError("b200gs: extract_fields: pass either a GaussianParams or the four tensors")
        means3D, opacities, scales, rotations, raw = means3D.xyz, means3D.opacity, means3D.scaling, means3D.rotation, True
    k, resolution, num_blocks = _kept("extract_fields", means3D, opacities, scales, rotations, raw, resolution, num_blocks)
    _, faces, w = _mesh(k, resolution, num_blocks, relax_ratio, density_thresh, clean, min_faces, min_diameter, decimate_target)
    return Mesh(w, faces)


# ---- field query: normals and colours ------------------------------------------------------------------------------------
class FieldQuery(NamedTuple):
    density: torch.Tensor            # float32 [n]: the field at each point
    normals: torch.Tensor            # float32 [n,3]: -grad / |grad| (outward, towards lower density); 0 where grad = 0
    colors: Optional[torch.Tensor]   # float32 [n,3] >= 0 (not clamped above), or None without SH


class ColoredMesh(NamedTuple):
    vertices: torch.Tensor          # float32 [V,3], world space (extract_mesh's bytes)
    faces: torch.Tensor             # int32 [F,3] (extract_mesh's bytes)
    normals: torch.Tensor           # float32 [V,3], unit or 0
    colors: Optional[torch.Tensor]  # float32 [V,3], or None without SH


def _check_shs(fn, shs, keep, sh_degree, view_dependent, dev):
    """-> (kept SH rows [n,K,3] contiguous, K, the degree the kernel evaluates), or (None, 0, 0) without SH."""
    if shs is None:
        if sh_degree is not None:
            raise ValueError(f"b200gs: {fn}: sh_degree without shs")
        return None, 0, 0
    P = keep.shape[0]
    shs = _f32_cuda(shs, "shs", lambda t: t.dim() == 3 and t.shape[0] == P and t.shape[1] >= 1 and t.shape[2] == 3, dev)
    K = int(shs.shape[1])
    if sh_degree is None:
        sh_degree = min(3, int(np.sqrt(K)) - 1)
    if not isinstance(sh_degree, (int, np.integer)) or not 0 <= sh_degree <= 3 or (sh_degree + 1) ** 2 > K:
        raise ValueError(f"b200gs: {fn}: sh_degree must be 0..3 with (sh_degree + 1)^2 <= {K} coefficients (got {sh_degree!r})")
    return shs[keep].contiguous(), K, int(sh_degree) if view_dependent else 0


def _query(k, shs, K, deg, q, resolution, num_blocks, relax_ratio) -> FieldQuery:
    """b200gs_field_query at normalised points q [n,3] (contiguous float32) for the kept set k."""
    dev, n, P = q.device, q.shape[0], k.xyz.shape[0]
    if n > 0x7FFFFFFF:
        raise ValueError(f"b200gs: query_field: {n} points do not fit int32 point ids")
    density = torch.empty(n, dtype=torch.float32, device=dev)
    normals = torch.empty(n, 3, dtype=torch.float32, device=dev)
    colors = torch.empty(n, 3, dtype=torch.float32, device=dev) if shs is not None else None
    if n == 0:
        return FieldQuery(density, normals, colors)
    samples, relax = _samples_relax(dev, resolution, num_blocks, relax_ratio)
    L = R.load_library()
    with torch.cuda.device(dev):
        scratch = torch.empty(L.b200gs_field_query_scratch_bytes(P, n, resolution, num_blocks, deg), dtype=torch.uint8, device=dev)
        R._check(L.b200gs_field_query(P, R._ptr(k.xyz), R._ptr(k.cov6), R._ptr(k.opac), R._ptr(shs), K, deg, resolution, num_blocks,
                                      R._ptr(samples), relax, n, R._ptr(q), R._ptr(density), R._ptr(normals), R._ptr(colors),
                                      R._ptr(scratch), scratch.numel(), R._stream(dev)), "field_query")
    return FieldQuery(density, normals, colors)


@torch.no_grad()
def query_field(points, means3D, opacities=None, scales=None, rotations=None, shs=None, *, raw=False, sh_degree=None,
                view_dependent=True, resolution=128, num_blocks=16, relax_ratio=1.5) -> FieldQuery:
    """extract_fields' density at world points [n,3], with the outward normal and an SH colour (DESIGN.md section 2).

    The Gaussians come in any form extract_fields takes (activated tensors, raw=True, views of the packed buffer, or a
    GaussianParams as means3D, whose SH are cat(features_dc, features_rest) at its sh_degree); shs [P,K,3] are the SH
    coefficients of the same Gaussians, sh_degree (default: the largest that K holds, at most 3) the degree evaluated.
    The points are mapped into the field's frame as (p - center) * scale in float32; there each point sees the members of
    the block it falls in, so at a grid sample the density is the field's voxel bit for bit.  colour =
    max(SH(S / D, -normal) + 0.5, 0) with S / D the opacity-weighted mean coefficients; view_dependent=False (or a zero
    normal) keeps the DC term alone.  Where the density is 0 every output is 0.  Use it to colour a mesh that was
    remeshed elsewhere (extract_colored_mesh already colours cleaned and decimated meshes).  Raises ValueError for a non-finite point, and as extract_fields does."""
    means3D, opacities, scales, rotations, raw, shs, sh_degree = _unwrap("query_field", means3D, opacities, scales, rotations, raw, shs,
                                                                         sh_degree)
    k, resolution, num_blocks = _kept("query_field", means3D, opacities, scales, rotations, raw, resolution, num_blocks)
    dev = k.xyz.device
    pts = _f32_cuda(points, "points", lambda t: t.dim() == 2 and t.shape[1] == 3, dev)
    if not bool(torch.isfinite(pts).all()):
        raise ValueError("b200gs: query_field: a point is not finite")
    shs, K, deg = _check_shs("query_field", shs, k.keep, sh_degree, view_dependent, dev)
    q = ((pts - k.center) * k.scale).contiguous()
    return _query(k, shs, K, deg, q, resolution, num_blocks, relax_ratio)


@torch.no_grad()
def extract_colored_mesh(means3D, opacities=None, scales=None, rotations=None, shs=None, *, raw=False, sh_degree=None,
                         view_dependent=True, density_thresh=1.0, resolution=128, num_blocks=16, relax_ratio=1.5, clean=False,
                         min_faces=64, min_diameter=0.2, decimate_target=0) -> ColoredMesh:
    """extract_mesh (the same vertex and face bytes) with per-vertex normals and colours from the field query, evaluated at
    the vertices' normalised positions v / (resolution - 1) * 2 - 1 (float32) -- after cleanup and decimation when they
    are on, so a decimated mesh gets them at its final vertices.  Arguments as extract_mesh and query_field; without SH
    (tensors and shs=None) colors is None."""
    _check_edit(clean, min_faces, min_diameter, decimate_target)
    means3D, opacities, scales, rotations, raw, shs, sh_degree = _unwrap("extract_colored_mesh", means3D, opacities, scales, rotations,
                                                                         raw, shs, sh_degree)
    k, resolution, num_blocks = _kept("extract_colored_mesh", means3D, opacities, scales, rotations, raw, resolution, num_blocks)
    shs, K, deg = _check_shs("extract_colored_mesh", shs, k.keep, sh_degree, view_dependent, k.xyz.device)
    v, faces, w = _mesh(k, resolution, num_blocks, relax_ratio, density_thresh, clean, min_faces, min_diameter, decimate_target)
    q = (v / (resolution - 1) * 2 - 1).contiguous()
    fq = _query(k, shs, K, deg, q, resolution, num_blocks, relax_ratio)
    return ColoredMesh(w, faces, fq.normals, fq.colors)


# ---- files ---------------------------------------------------------------------------------------------------------------
def _np(a, dtype):
    return np.asarray(a.detach().cpu() if isinstance(a, torch.Tensor) else a, dtype=dtype)


def _mesh_arrays(fn, vertices, faces, normals, colors):
    v = _np(vertices, np.float64).reshape(-1, 3)
    f = _np(faces, np.int64).reshape(-1, 3)
    if f.size and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError(f"b200gs: {fn}: a face refers to a vertex that does not exist")
    out = []
    for name, a in (("normals", normals), ("colors", colors)):
        if a is not None:
            a = _np(a, np.float32)
            if a.shape != (len(v), 3):
                raise ValueError(f"b200gs: {fn}: {name} must be [{len(v)}, 3] (got {list(a.shape)})")
        out.append(a)
    return v, f, out[0], out[1]


def save_obj(path, vertices, faces, *, normals=None, colors=None):
    """Wavefront OBJ: `v x y z` lines (`v x y z r g b` with colours, clamped to [0, 1]), `vn x y z` lines with normals,
    then `f a b c` with 1-based indices (`f a//a b//b c//c` with normals)."""
    v, f, n, c = _mesh_arrays("save_obj", vertices, faces, normals, colors)
    with open(path, "w") as fh:
        if len(v):
            if c is None:
                fh.write("\n".join("v %.9g %.9g %.9g" % tuple(r) for r in v) + "\n")
            else:
                vc = np.concatenate([v, np.clip(c, 0, 1).astype(np.float64)], 1)
                fh.write("\n".join("v %.9g %.9g %.9g %.9g %.9g %.9g" % tuple(r) for r in vc) + "\n")
            if n is not None:
                fh.write("\n".join("vn %.9g %.9g %.9g" % tuple(r) for r in n.astype(np.float64)) + "\n")
        if len(f):
            if n is None:
                fh.write("\n".join("f %d %d %d" % tuple(r) for r in f + 1) + "\n")
            else:
                fh.write("\n".join("f %d//%d %d//%d %d//%d" % tuple(r) for r in np.repeat(f + 1, 2, 1)) + "\n")


def save_ply_mesh(path, vertices, faces, normals=None, colors=None):
    """Binary little-endian PLY: vertex properties `x y z` (float), `nx ny nz` (float) with normals, `red green blue`
    (uchar, clamp(c, 0, 1) * 255 truncated, as the frame pack does) with colours; faces as `list uchar int`."""
    v, f, n, c = _mesh_arrays("save_ply_mesh", vertices, faces, normals, colors)
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if n is not None:
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
    if c is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    vert = np.empty(len(v), dtype=np.dtype(fields))
    for i, ax in enumerate("xyz"):
        vert[ax] = v[:, i]
    if n is not None:
        for i, ax in enumerate(("nx", "ny", "nz")):
            vert[ax] = n[:, i]
    if c is not None:
        u8 = (np.clip(c, np.float32(0), np.float32(1)) * np.float32(255)).astype(np.uint8)
        for i, ax in enumerate(("red", "green", "blue")):
            vert[ax] = u8[:, i]
    face = np.empty(len(f), dtype=np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
    face["n"] = 3
    face["i"] = f
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}"]
    head += [f"property {'float' if t == '<f4' else 'uchar'} {name}" for name, t in fields]
    head += [f"element face {len(f)}", "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode("ascii"))
        fh.write(vert.tobytes())
        fh.write(face.tobytes())
