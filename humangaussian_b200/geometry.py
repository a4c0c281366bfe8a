"""Geometry regularisers over the rasteriser's geometry outputs (rasterize_views(geometry=True), DESIGN.md section 2).

  * ``depth_distortion(alpha, depth, depth2)`` -- the per-pixel depth distortion sum_{i<j} w_i w_j (d_i - d_j)^2 (Mip-NeRF 360 /
    2DGS), from the alpha, depth and depth second moment images;
  * ``depth_to_normal(depth, viewmatrices, tanfovx, tanfovy)`` -- world-space normals of a depth image by finite differences;
  * ``depth_normal_consistency(normal, depth_normal, alpha)`` -- 1 - cos between the rendered normal and the depth's normal.

Plain torch: these run once per image, not per Gaussian, and autograd carries their gradients to the images.
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn.functional as F


def depth_distortion(alpha: torch.Tensor, depth: torch.Tensor, depth2: torch.Tensor) -> torch.Tensor:
    """A * M2 - M1^2 per pixel, with A = sum w (alpha), M1 = sum w d (depth) and M2 = sum w d^2 (depth2); [...,1,H,W] each.

    This equals sum_{i<j} w_i w_j (d_i - d_j)^2 over the pixel's blends: 0 for a single surface, large for weight spread along
    the ray.  d is the view-space z of each Gaussian, so the value is in world length^2 (not 2DGS's NDC mapping of d).

    Formed in float64 and returned in the inputs' dtype.  It is not clamped, because a clamp would zero the gradient at the
    optimum; rounding in the rendered images can make it slightly negative where it is near 0 (a sum of squares otherwise)."""
    a, m1, m2 = alpha.double(), depth.double(), depth2.double()
    return (a * m2 - m1 * m1).to(depth.dtype)


def _pixel_rays(H: int, W: int, tanfovx: float, tanfovy: float, device, dtype):
    """[H,W] view-space x/z and y/z of each pixel centre: the inverse of the preprocess's NDC-to-pixel map
    p = ((ndc + 1) * S - 1) / 2, i.e. ndc = (2 p + 1) / S - 1, and ndc = x / (z tanfov) for the rasteriser's projection."""
    px = torch.arange(W, device=device, dtype=dtype)
    py = torch.arange(H, device=device, dtype=dtype)
    rx = ((2.0 * px + 1.0) / W - 1.0) * tanfovx
    ry = ((2.0 * py + 1.0) / H - 1.0) * tanfovy
    return rx[None, :].expand(H, W), ry[:, None].expand(H, W)


def depth_to_normal(depth: torch.Tensor, viewmatrices: torch.Tensor, tanfovx: Sequence[float], tanfovy: Sequence[float]) -> torch.Tensor:
    """World-space unit normals [V,3,H,W] of the depth images depth [V,1,H,W] (view-space z, e.g. the median depth).

    Each pixel is unprojected at its centre (the rasteriser's pixel convention) to x = z (2 px + 1 - W) / W tanfovx,
    y = z (2 py + 1 - H) / H tanfovy, and taken to world space with the row-vector view matrix (p_view = [p_world, 1] @ M).
    The normal is the cross product of the central differences along x and along y, normalised and flipped to face the camera
    (as the rendered normal image is).  The one-pixel border, where a central difference does not exist, is 0."""
    V, _, H, W = depth.shape
    dt = depth.dtype
    z = depth[:, 0]
    vm = viewmatrices.reshape(V, 4, 4).to(device=depth.device, dtype=dt)
    pts = []
    for v in range(V):
        rx, ry = _pixel_rays(H, W, float(tanfovx[v]), float(tanfovy[v]), depth.device, dt)
        pv = torch.stack((rx * z[v], ry * z[v], z[v]), -1)  # [H,W,3] view space
        R, t = vm[v, :3, :3], vm[v, 3, :3]
        pts.append((pv - t) @ torch.linalg.inv(R))  # world space
    X = torch.stack(pts)  # [V,H,W,3]
    dx = X[:, 1:-1, 2:] - X[:, 1:-1, :-2]
    dy = X[:, 2:, 1:-1] - X[:, :-2, 1:-1]
    n = F.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    campos = torch.stack([-vm[v, 3, :3] @ torch.linalg.inv(vm[v, :3, :3]) for v in range(V)])  # [V,3]
    to_cam = campos[:, None, None, :] - X[:, 1:-1, 1:-1]
    n = torch.where(((n * to_cam).sum(-1, keepdim=True) < 0), -n, n)
    out = torch.zeros(V, H, W, 3, dtype=dt, device=depth.device)
    out[:, 1:-1, 1:-1] = n
    return out.permute(0, 3, 1, 2)


def depth_normal_consistency(normal: torch.Tensor, depth_normal: torch.Tensor, alpha: torch.Tensor,
                             threshold: float = 0.5) -> torch.Tensor:
    """1 - cos(normal, depth_normal) per pixel [...,1,H,W], inside the silhouette (alpha > threshold) and 0 outside it and
    where either normal is 0 (the depth normal's border, a pixel with no blend).  normal is the rendered normal image
    (rasterize_views(normals=True), unnormalised), depth_normal e.g. depth_to_normal of the median depth."""
    n = F.normalize(normal, dim=-3)
    dn = F.normalize(depth_normal, dim=-3)
    cos = (n * dn).sum(-3, keepdim=True)
    valid = (alpha > threshold) & (normal.abs().sum(-3, keepdim=True) > 0) & (depth_normal.abs().sum(-3, keepdim=True) > 0)
    return torch.where(valid, 1.0 - cos, torch.zeros_like(cos))
