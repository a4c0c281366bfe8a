"""Render wrappers of the hot path, mirroring the reference's two entry points:

  * ``render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, override_color)``
        gaussiansplatting/gaussian_renderer/__init__.py:18-104 -- same keys in the returned dict;
  * ``render_views(cameras, pc, bg_color)`` -- the SDS view loop of
        threestudio/systems/GaussianDreamer.py:244-266 as ONE batched rasteriser call.

``pc`` is anything with GaussianModel's getters (get_xyz, get_opacity, get_scaling, get_rotation,
get_features, active_sh_degree) -- e.g. humangaussian_b200.scene.GaussianParams or the reference's
own GaussianModel.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from .geometry import depth_distortion
from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer, rasterize_views


class PipelineParams:
    """gaussiansplatting/arguments/__init__.py:63-68"""
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False
    antialiasing = False  # the screen-space mip filter (rasterizer.rasterize_views); the name upstream 3DGS gives it


def comp_normal(normal, alpha):
    """threestudio's normal map from the rasteriser's normal image: (F.normalize(N) + 1) / 2 * alpha, channels last.
    normal [...,3,H,W] (rasterize_views(normals=True)), alpha [...,1,H,W]; returns [...,H,W,3] in [0, 1] for alpha in [0, 1].
    A pixel where nothing blended has N = 0, which F.normalize keeps at 0 (so it becomes alpha / 2 = 0 there)."""
    n = F.normalize(normal, dim=-3)
    return ((n + 1.0) * 0.5 * alpha).movedim(-3, -1)


def _raw_tensors(pc):
    """(opacity, scaling, rotation, f_dc, f_rest) raw parameters of the reference's GaussianModel (`_opacity`, ...:
    gaussian_model.py:44-59) or of scene.GaussianParams (`opacity`, ...); None if `pc` exposes neither."""
    for names in (("_opacity", "_scaling", "_rotation", "_features_dc", "_features_rest"),
                  ("opacity", "scaling", "rotation", "features_dc", "features_rest")):
        if all(hasattr(pc, n) for n in names):
            return tuple(getattr(pc, n) for n in names)
    return None


def render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier=1.0, override_color=None, fused_activations=False, filter_3d=None,
           absgrad=False, normals=False, geometry=False):
    """fused_activations=True (optional fast path, SURVEY.md 8f-1): instead of calling the getters (sigmoid / exp /
    F.normalize: three kernels + autograd nodes per view, gaussian_model.py:95-118) the raw parameter tensors go straight
    to the rasteriser, which applies the activations and their Jacobians inside its kernels.  Same dict, same gradients
    (they arrive at the raw tensors directly).  `pipe.antialiasing` (absent = False) turns on the screen-space mip filter.
    filter_3d ([P] variances from filter3d.compute_filter_3d, or None): the 3D smoothing filter; the call then goes through
    rasterize_views (GaussianRasterizer keeps upstream's surface, which has no such input).
    absgrad=True: the dict also holds "viewspace_points_abs" [P,3], whose .grad the backward fills with the absolute
    screen-space gradient (rasterizer.rasterize_views, means2D_abs), the densification statistic that does not cancel; the
    call then goes through rasterize_views as with filter_3d.
    normals=True: the dict also holds "normal_3dgs" [3,H,W], the differentiable normal image (rasterize_views' normals=True),
    through rasterize_views as with filter_3d.
    geometry=True: the dict also holds "median_depth_3dgs" and "depth2_3dgs" [1,H,W] (rasterize_views' geometry=True) and
    "distortion_3dgs" [1,H,W], geometry.depth_distortion of alpha, depth and depth2, all differentiable; through
    rasterize_views as with filter_3d."""
    aa = bool(getattr(pipe, "antialiasing", False))
    xyz = pc.get_xyz
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    extra = {}
    if absgrad:
        extra["viewspace_points_abs"] = torch.zeros_like(xyz, dtype=torch.float32, requires_grad=True, device=xyz.device) + 0
        extra["viewspace_points_abs"].retain_grad()
    settings = GaussianRasterizationSettings(
        image_height=int(viewpoint_camera.image_height), image_width=int(viewpoint_camera.image_width),
        tanfovx=math.tan(viewpoint_camera.FoVx * 0.5), tanfovy=math.tan(viewpoint_camera.FoVy * 0.5),
        bg=bg_color, scale_modifier=scaling_modifier, viewmatrix=viewpoint_camera.world_view_transform,
        projmatrix=viewpoint_camera.full_proj_transform, sh_degree=pc.active_sh_degree,
        campos=viewpoint_camera.camera_center, prefiltered=False, debug=False)
    rasterizer = GaussianRasterizer(raster_settings=settings, antialiasing=aa)
    shs = colors = None
    if override_color is None:
        shs = pc.get_features
    else:
        colors = override_color
    raw = _raw_tensors(pc) if fused_activations else None
    m2d_abs = extra["viewspace_points_abs"][None] if absgrad else None
    if raw is None and (filter_3d is not None or absgrad or normals or geometry):
        outs = rasterize_views(
            means3D=xyz, opacities=pc.get_opacity, viewmatrices=viewpoint_camera.world_view_transform[None],
            projmatrices=viewpoint_camera.full_proj_transform[None], camposs=viewpoint_camera.camera_center[None],
            tanfovx=[settings.tanfovx], tanfovy=[settings.tanfovy], image_height=settings.image_height, image_width=settings.image_width,
            bg=bg_color, sh_degree=pc.active_sh_degree, shs=shs, colors_precomp=colors, scales=pc.get_scaling,
            rotations=pc.get_rotation, means2D=screenspace_points[None], scale_modifier=scaling_modifier, antialiasing=aa,
            filter_3d=filter_3d, means2D_abs=m2d_abs, normals=normals, geometry=geometry)
        image, radii, depth, alpha = outs[0][0], outs[1][0], outs[2][0], outs[3][0]
        if normals:
            extra["normal_3dgs"] = outs[4][0]
        if geometry:
            _geometry_keys(extra, alpha, depth, outs[4 + normals][0], outs[5 + normals][0])
        return {"render": image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0, "radii": radii,
                "depth_3dgs": depth, "alpha_3dgs": alpha, **extra}
    if raw is not None:
        op, sc, rot = raw[0], raw[1], raw[2]
        outs = rasterize_views(
            means3D=xyz, opacities=op, viewmatrices=viewpoint_camera.world_view_transform[None], projmatrices=viewpoint_camera.full_proj_transform[None],
            camposs=viewpoint_camera.camera_center[None], tanfovx=[settings.tanfovx], tanfovy=[settings.tanfovy], image_height=settings.image_height,
            image_width=settings.image_width, bg=bg_color, sh_degree=pc.active_sh_degree, shs=shs, colors_precomp=colors, scales=sc, rotations=rot,
            means2D=screenspace_points[None], scale_modifier=scaling_modifier, raw=True, antialiasing=aa, filter_3d=filter_3d,
            means2D_abs=m2d_abs, normals=normals, geometry=geometry)
        image, radii, depth, alpha = outs[0][0], outs[1][0], outs[2][0], outs[3][0]
        if normals:
            extra["normal_3dgs"] = outs[4][0]
        if geometry:
            _geometry_keys(extra, alpha, depth, outs[4 + normals][0], outs[5 + normals][0])
        return {"render": image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0, "radii": radii,
                "depth_3dgs": depth, "alpha_3dgs": alpha, **extra}
    image, radii, depth, alpha = rasterizer(means3D=xyz, means2D=screenspace_points, shs=shs, colors_precomp=colors,
                                            opacities=pc.get_opacity, scales=pc.get_scaling, rotations=pc.get_rotation,
                                            cov3D_precomp=None)
    return {"render": image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0, "radii": radii,
            "depth_3dgs": depth, "alpha_3dgs": alpha}


def _geometry_keys(extra, alpha, depth, median, depth2):
    extra["median_depth_3dgs"] = median
    extra["depth2_3dgs"] = depth2
    extra["distortion_3dgs"] = depth_distortion(alpha, depth, depth2)


def stack_cameras(cameras, device):
    vm = torch.stack([c.world_view_transform.to(device).float() for c in cameras])
    pm = torch.stack([c.full_proj_transform.to(device).float() for c in cameras])
    cp = torch.stack([c.camera_center.to(device).float() for c in cameras])
    tanx = [math.tan(c.FoVx * 0.5) for c in cameras]
    tany = [math.tan(c.FoVy * 0.5) for c in cameras]
    return vm, pm, cp, tanx, tany


class _StackSinks(torch.autograd.Function):
    """[V,P,3] view-batch gradient sink whose backward hands row v to the v-th per-view sink (a leaf [P,3] tensor), so that
    `sink.grad` is filled exactly as the per-view loop fills `viewspace_point_tensor.grad` (GaussianDreamer.py:249-250,
    385-387).  The sinks alias `base` (all zeros, never written): forward copies nothing."""

    @staticmethod
    def forward(ctx, base, *sinks):
        return base.view_as(base)

    @staticmethod
    def backward(ctx, g):
        return (None, *g.unbind(0))


def render_views(cameras, pc, bg_color, scaling_modifier=1.0, antialiasing=False, filter_3d=None, absgrad=False, normals=False,
                 geometry=False):
    """All cameras share image size.  Returns the dict of `render` with a leading view axis:
    render [V,3,H,W], depth_3dgs/alpha_3dgs [V,1,H,W], radii [V,P], viewspace_points [V,P,3] (its .grad is [V,P,3]),
    plus viewspace_point_list: V leaf tensors [P,3] whose .grad backward fills -- what the reference's
    `self.viewspace_point_list` holds (GaussianDreamer.py:242-250) and on_before_optimizer_step sums (:385-387).
    antialiasing, filter_3d: the screen-space mip filter and the 3D smoothing filter, as `rasterizer.rasterize_views`.
    absgrad=True: also viewspace_points_abs [V,P,3], whose .grad is the absolute screen-space gradient (`rasterize_views`'
    means2D_abs) -- the densification statistic that does not cancel.
    normals=True: also normal_3dgs [V,3,H,W] (rasterize_views' normal image) and comp_normal [V,H,W,3], threestudio's normal
    map of it (`comp_normal`), both differentiable.
    geometry=True: also median_depth_3dgs, depth2_3dgs and distortion_3dgs [V,1,H,W], as `render`'s geometry=True."""
    xyz = pc.get_xyz
    V = len(cameras)
    vm, pm, cp, tanx, tany = stack_cameras(cameras, xyz.device)
    base = torch.zeros(V, xyz.shape[0], 3, dtype=torch.float32, device=xyz.device)
    sinks = [t.requires_grad_(True) for t in base.unbind(0)]
    screenspace_points = _StackSinks.apply(base, *sinks)
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    extra = {}
    if absgrad:
        extra["viewspace_points_abs"] = torch.zeros(V, xyz.shape[0], 3, dtype=torch.float32, device=xyz.device, requires_grad=True)
    outs = rasterize_views(
        means3D=xyz, opacities=pc.get_opacity, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tanx, tanfovy=tany,
        image_height=int(cameras[0].image_height), image_width=int(cameras[0].image_width), bg=bg_color,
        sh_degree=pc.active_sh_degree, shs=pc.get_features, scales=pc.get_scaling, rotations=pc.get_rotation,
        means2D=screenspace_points, scale_modifier=scaling_modifier, antialiasing=antialiasing, filter_3d=filter_3d,
        means2D_abs=extra.get("viewspace_points_abs"), normals=normals, geometry=geometry)
    image, radii, depth, alpha = outs[:4]
    if normals:
        extra["normal_3dgs"] = outs[4]
        extra["comp_normal"] = comp_normal(outs[4], alpha)
    if geometry:
        _geometry_keys(extra, alpha, depth, outs[4 + normals], outs[5 + normals])
    return {"render": image, "viewspace_points": screenspace_points, "viewspace_point_list": sinks, "visibility_filter": radii > 0,
            "radii": radii, "depth_3dgs": depth, "alpha_3dgs": alpha, **extra}
