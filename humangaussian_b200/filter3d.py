"""Mip-Splatting's 3D smoothing filter: per-Gaussian variances from a camera set, and baking them into the parameters.

The filter bounds each Gaussian's 3D size from below by what the training cameras could resolve: with nu_k the highest
sampling rate (pixels per world unit) at which any camera of the set sees Gaussian k, the scales become
sqrt(s^2 + c / nu_k^2) and the opacity is scaled so that the integrated 3D weight stays the same (DESIGN.md section 2).
Close-ups and renders at a finer pixel scale than training then show no sub-pixel specks.

  * `compute_filter_3d` gives the [P] variances; pass them as `filter_3d=` to `rasterizer.rasterize_views`,
    `rasterize_views_packed`, `renderer.render`, `render_views` or `animation.render_frames`.  The filtering happens inside
    the preprocess kernels (raw parameters included), gradients stay w.r.t. the unfiltered parameters.
  * `bake_filter_3d` writes the filter into raw parameters (log s', logit o'), for export through `scene.params_to_ply`
    to renderers that do not know the filter.
"""
from __future__ import annotations

import torch

from .rasterizer import MAX_VIEWS, sampling_rate

VARIANCE_SCALE = 0.2  # Mip-Splatting's c


@torch.no_grad()
def compute_filter_3d(xyz: torch.Tensor, viewmatrices: torch.Tensor, tanfovx, tanfovy, image_height: int, image_width: int,
                      variance_scale: float = VARIANCE_SCALE) -> torch.Tensor:
    """Filter variances [P] (float32, world length^2) of the Gaussians at xyz [P,3] for a camera set: viewmatrices [V,4,4]
    (row-vector convention), tanfovx / tanfovy sequences of V floats, one image size.  The cameras are folded in chunks of
    MAX_VIEWS through the sampling-rate kernel (the fold is a max: any order, same bits).  Gaussians no camera sees get the
    smallest positive rate of the set (the widest filter); if no camera sees any Gaussian, every variance is 0."""
    P = xyz.shape[0]
    rate = torch.zeros(P, dtype=torch.float32, device=xyz.device)
    tanx, tany = [float(t) for t in tanfovx], [float(t) for t in tanfovy]
    V = viewmatrices.shape[0]
    if len(tanx) != V or len(tany) != V:
        raise ValueError(f"compute_filter_3d: {V} view matrices but {len(tanx)} / {len(tany)} tan(fov/2) values")
    for i in range(0, V, MAX_VIEWS):
        sampling_rate(xyz, viewmatrices[i:i + MAX_VIEWS], tanx[i:i + MAX_VIEWS], tany[i:i + MAX_VIEWS], image_height, image_width, rate)
    return finalize_filter_3d(rate, variance_scale)


def finalize_filter_3d(max_rate: torch.Tensor, variance_scale: float = VARIANCE_SCALE) -> torch.Tensor:
    """Variances c / nu^2 from folded sampling rates (float32 ops); rate 0 (unseen) takes the smallest positive rate."""
    pos = max_rate > 0
    lo = torch.where(pos, max_rate, torch.full_like(max_rate, float("inf"))).min()
    if not torch.isfinite(lo):  # no Gaussian in view of any camera
        return torch.zeros_like(max_rate)
    nu = torch.where(pos, max_rate, lo)
    return torch.tensor(variance_scale, dtype=torch.float32, device=nu.device) / (nu * nu)


@torch.no_grad()
def bake_filter_3d(scaling_raw: torch.Tensor, opacity_raw: torch.Tensor, var: torch.Tensor):
    """(scaling_raw', opacity_raw'): the raw parameters (log-scales [P,3], opacity logits [P,1]) with the filter applied,
    log(sqrt(exp(s)^2 + v)) and logit(sigmoid(o) * sqrt(prod_i exp(s_i)^2 / (exp(s_i)^2 + v))).  Rendered WITHOUT the
    filter they give what the unbaked parameters give with it, up to the exp / log round trip."""
    if var.shape != (scaling_raw.shape[0],):
        raise ValueError(f"bake_filter_3d: var must be [{scaling_raw.shape[0]}], got {tuple(var.shape)}")
    s = torch.exp(scaling_raw)
    s2 = s * s
    t = s2 + var[:, None]
    r = torch.where(t > 0, s2 / t, torch.ones_like(t))
    coef = torch.sqrt(r.prod(1, keepdim=True))
    o = torch.sigmoid(opacity_raw) * coef.reshape(opacity_raw.shape)
    return torch.log(torch.sqrt(t)), torch.logit(o)
