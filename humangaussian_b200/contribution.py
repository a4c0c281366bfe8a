"""Contribution scores: how much each Gaussian shows in a set of images, from the forward blend's own weights.

For every pixel of every camera the blend gives each Gaussian it reaches a weight w = alpha * T (the share of the pixel's
colour it contributes).  `compute_contribution` folds, per Gaussian, over all pixels of all cameras:

  * weight_sum -- the sum of w (LightGaussian's global significance), exact in fixed point (units of 2^-24);
  * weight_max -- the largest single w (RadSplat's / Taming 3DGS's maximum weight);
  * touches    -- the number of pixels that reached it while still open: those that blended it, plus the one pixel-entry at
                  which a pixel terminated (Mini-Splatting-style counts).

The accumulators are integers on the device, so any camera set, in any order and chunking, gives the same bits.  Removing
every Gaussian with touches == 0 over a camera set (densify.prune_points) leaves those cameras' images byte-identical
(DESIGN.md section 2); a threshold on weight_max or weight_sum prunes further, with a loss.  Colours do not enter the
weights, so no SH is needed.  There is no CPU path.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import torch

from . import rasterizer as R

FIXED_ONE = float(1 << 24)  # weight_sum's unit is 2^-24
MAX_PIXELS = 1 << 32        # per call of compute_contribution: sum of V*H*W (each pixel adds < 2^24 and <= 1 per Gaussian)


class Contribution(NamedTuple):
    weight_sum: torch.Tensor  # float64 [P]: sum of blend weights (the fixed-point sum times 2^-24; exact below 2^29)
    weight_max: torch.Tensor  # float32 [P]: largest blend weight, 0 = never blended
    touches: torch.Tensor     # int64 [P]: pixels that blended it or terminated on it


def _f32_cuda(t, name, shape_ok):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.device.type != "cuda" or not shape_ok(t):
        desc = f"{tuple(t.shape)} {t.dtype} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
        raise ValueError(f"b200gs: compute_contribution: {name} has the wrong shape, dtype or device ({desc})")
    return t.detach().contiguous()


@torch.no_grad()
def compute_contribution(means3D, opacities, scales=None, rotations=None, cov3D_precomp=None, *, viewmatrices, projmatrices,
                         tanfovx, tanfovy, image_height, image_width, scale_modifier=1.0, raw=False, antialiasing=False,
                         filter_3d: Optional[torch.Tensor] = None) -> Contribution:
    """Per-Gaussian contribution scores over any number of cameras (one image size).

    means3D [P,3], or [N,P,3] with one position set per camera (the frames of a motion); opacities [P] or [P,1]; exactly
    one of scales [P,3] + rotations [P,4] | cov3D_precomp [P,6]; viewmatrices / projmatrices [N,4,4]; tanfovx / tanfovy
    sequences of N floats.  raw, antialiasing, filter_3d: as `rasterizer.rasterize_views` -- score with the options the
    images are rendered with.  All float32 on one CUDA device.  For the packed buffer of `optim.PackedAdam`, pass views of
    its fields (`rasterizer.packed_layout`).

    The cameras run through the library in calls of at most 64 views (a call with too many tile instances is halved, as in
    `rasterize_views`), all folding into one set of device accumulators.  The total pixel count N*H*W must stay below 2^32."""
    dev = means3D.device if isinstance(means3D, torch.Tensor) else None
    if dev is None or dev.type != "cuda":
        raise RuntimeError("b200gs: tensors must live on a CUDA device (there is no CPU path)")
    N = viewmatrices.shape[0] if isinstance(viewmatrices, torch.Tensor) else -1
    if N < 1 or tuple(viewmatrices.shape[1:]) != (4, 4) or not isinstance(projmatrices, torch.Tensor) or \
            tuple(projmatrices.shape) != (N, 4, 4) or len(tanfovx) != N or len(tanfovy) != N:
        raise ValueError("b200gs: compute_contribution: viewmatrices / projmatrices must be [N,4,4] with N >= 1 and N tanfovx / tanfovy")
    per_view = means3D.dim() == 3
    P = means3D.shape[-2] if means3D.dim() in (2, 3) else -1
    means3D = _f32_cuda(means3D, "means3D", lambda t: t.shape[-1] == 3 and (t.dim() == 2 or (t.dim() == 3 and t.shape[0] == N)))
    opacities = _f32_cuda(opacities, "opacities", lambda t: t.shape in ((P,), (P, 1)) and t.device == dev)
    if (cov3D_precomp is None) == (scales is None or rotations is None) or (scales is None) != (rotations is None):
        raise ValueError("b200gs: compute_contribution: pass exactly one of scales + rotations | cov3D_precomp")
    if cov3D_precomp is not None:
        cov3D_precomp = _f32_cuda(cov3D_precomp, "cov3D_precomp", lambda t: t.shape == (P, 6) and t.device == dev)
    else:
        scales = _f32_cuda(scales, "scales", lambda t: t.shape == (P, 3) and t.device == dev)
        rotations = _f32_cuda(rotations, "rotations", lambda t: t.shape == (P, 4) and t.device == dev)
    filter_3d = R._check_filter_3d(filter_3d, P, dev, cov3D_precomp)
    H, W = int(image_height), int(image_width)
    if H < 1 or W < 1:
        raise ValueError("b200gs: compute_contribution: image size must be positive")
    if N * H * W >= MAX_PIXELS:
        raise ValueError(f"b200gs: compute_contribution: {N} cameras of {H}x{W} are {N * H * W} pixels; the accumulators "
                         f"allow fewer than 2^32 per call -- score the cameras in several calls and combine")

    acc = (torch.zeros(P, dtype=torch.int64, device=dev), torch.zeros(P, dtype=torch.int32, device=dev),
           torch.zeros(P, dtype=torch.int32, device=dev))
    colors = torch.zeros(P, 3, dtype=torch.float32, device=dev)  # colours do not enter the weights
    bg = torch.zeros(3, dtype=torch.float32, device=dev)
    vm = viewmatrices.detach().to(device=dev, dtype=torch.float32).contiguous()
    pm = projmatrices.detach().to(device=dev, dtype=torch.float32).contiguous()
    campos = torch.zeros(N, 3, dtype=torch.float32, device=dev)  # only SH evaluation reads it
    tx, ty = [float(t) for t in tanfovx], [float(t) for t in tanfovy]

    def score(lo, hi):
        try:
            R._forward_impl(means3D[lo:hi] if per_view else means3D, None, colors, opacities, scales, rotations, cov3D_precomp,
                            bg, vm[lo:hi], pm[lo:hi], campos[lo:hi], tx[lo:hi], ty[lo:hi], H, W, 0, scale_modifier, raw=raw,
                            antialiasing=antialiasing, filter_3d=filter_3d, contrib=acc)
        except R.InstanceLimitError:  # refused before binning (the limit is passed as capacity): nothing was accumulated
            if hi - lo == 1:
                raise
            mid = (lo + hi) // 2
            score(lo, mid)
            score(mid, hi)

    for lo in range(0, N, R.MAX_VIEWS):
        score(lo, min(N, lo + R.MAX_VIEWS))
    wsum, wmax, touches = acc
    return Contribution(wsum.to(torch.float64) / FIXED_ONE, wmax.view(torch.float32).clone(), touches.to(torch.int64) & 0xFFFFFFFF)
