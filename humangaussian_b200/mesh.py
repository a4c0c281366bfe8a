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
and maps the vertices back to world space as the reference does.  The reference's clean_mesh / decimate_mesh
(pymeshlab remeshing) are not part of this module: the output is the raw marching-cubes mesh.  There is no CPU path.
"""
from __future__ import annotations

from typing import NamedTuple

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
        raise ValueError(f"b200gs: extract_fields: no Gaussian has opacity > {OPACITY_MIN}")
    if not bool(torch.isfinite(xyz).all()):
        raise ValueError("b200gs: extract_fields: a kept Gaussian has a non-finite position")
    stds = torch.exp(scales[keep]) if raw else scales[keep]
    mn, mx = xyz.amin(0), xyz.amax(0)
    center = (mn + mx) / 2
    extent = (mx - mn).amax().item()
    if extent == 0:
        raise ValueError("b200gs: extract_fields: the kept Gaussians' centres are a single point")
    scale = 1.8 / extent
    xyz = ((xyz - center) * scale).contiguous()
    cov6 = _covariance(stds * scale, rotations[keep])
    return Fields(_density_field(xyz, cov6, opac[keep].contiguous(), resolution, num_blocks, relax_ratio), center, scale)


def _density_field(xyz, cov6, opac, resolution, num_blocks, relax_ratio):
    """b200gs_density_field on normalised centres [n,3], covariances [n,6] and opacities [n] (all kept)."""
    dev, n = xyz.device, xyz.shape[0]
    samples = torch.linspace(-1, 1, resolution).to(dev)  # built on the CPU, as the reference builds it
    relax = float(np.float32((2 / num_blocks) * relax_ratio))
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


@torch.no_grad()
def extract_mesh(means3D, opacities=None, scales=None, rotations=None, *, raw=False, density_thresh=1.0, resolution=128,
                 num_blocks=16, relax_ratio=1.5) -> Mesh:
    """The reference's extract_mesh up to its remeshing: extract_fields, marching cubes at density_thresh, and the vertices
    mapped back to world space as v / (resolution - 1) * 2 - 1, then / scale + center (in float64, stored as float32)."""
    f = extract_fields(means3D, opacities, scales, rotations, raw=raw, resolution=resolution, num_blocks=num_blocks,
                       relax_ratio=relax_ratio)
    v, faces = marching_cubes(f.occ, density_thresh)
    w = (v.double() / (resolution - 1.0) * 2 - 1) / f.scale + f.center.double()
    return Mesh(w.float(), faces)


def save_obj(path, vertices, faces):
    """Wavefront OBJ: `v x y z` lines, then `f a b c` with 1-based indices."""
    v = np.asarray(vertices.detach().cpu() if isinstance(vertices, torch.Tensor) else vertices, dtype=np.float64).reshape(-1, 3)
    f = np.asarray(faces.detach().cpu() if isinstance(faces, torch.Tensor) else faces, dtype=np.int64).reshape(-1, 3)
    if f.size and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError("b200gs: save_obj: a face refers to a vertex that does not exist")
    with open(path, "w") as fh:
        if len(v):
            fh.write("\n".join("v %.9g %.9g %.9g" % tuple(r) for r in v) + "\n")
        if len(f):
            fh.write("\n".join("f %d %d %d" % tuple(r) for r in f + 1) + "\n")
