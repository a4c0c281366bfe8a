"""Animation frame path (reference animation.py), frame-batched and on the GPU.

The reference renders an AMASS sequence one frame at a time: SMPL-X forward on the CPU, numpy re-attachment of every
Gaussian to the re-posed mesh (animation.py:383-403), H2D upload of P*12 bytes, one rasteriser forward, D2H of the
float image, then (x*255).astype(uint8) on the host (animation.py:1002-1013).  Here a block of F frames is one
re-attachment kernel + one batched rasteriser call (per-view positions) + one pack kernel:

    xyz    = reattach(vertices[F,Nv,3], faces, mapping_face, mapping_uvw, mapping_dist)        # [F,P,3]
    frames = render_frames(gaussians, xyz, cameras, bg)                                        # [F,H,W,3] uint8

SMPL-X itself (licensed model files, CPU LBS) stays outside: the caller supplies posed vertices per frame.
"""
from __future__ import annotations

import ctypes as C

import torch

from .rasterizer import MAX_VIEWS, _check, _f32c, _ptr, _stream, load_library, rasterize_views
from .renderer import stack_cameras


def reattach(vertices: torch.Tensor, faces: torch.Tensor, mapping_face: torch.Tensor, mapping_uvw: torch.Tensor,
             mapping_dist: torch.Tensor) -> torch.Tensor:
    """vertices [F,Nv,3] (or [Nv,3]) posed mesh per frame; returns Gaussian centres [F,P,3] (animation.py:383-403)."""
    L = load_library()
    v = _f32c(vertices)
    if v.dim() == 2:
        v = v[None]
    dev = v.device
    if dev.type != "cuda":
        raise RuntimeError("b200gs: tensors must live on a CUDA device (there is no CPU path)")
    F, Nv = v.shape[0], v.shape[1]
    fc = faces.to(device=dev, dtype=torch.int32).contiguous()
    mf = mapping_face.to(device=dev, dtype=torch.int32).contiguous()
    uvw, dist = _f32c(mapping_uvw, dev), _f32c(mapping_dist, dev).reshape(-1)
    P = mf.shape[0]
    out = torch.empty(F, P, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        for f0 in range(0, F, 65535):
            f1 = min(F, f0 + 65535)
            _check(L.b200gs_reattach(P, f1 - f0, Nv, fc.shape[0], _ptr(v[f0:f1]), _ptr(fc), _ptr(mf), _ptr(uvw), _ptr(dist),
                                     _ptr(out[f0:f1]), _stream(dev)), "reattach")
    return out


def pack_frames_u8(color: torch.Tensor) -> torch.Tensor:
    """color [F,3,H,W] float -> [F,H,W,3] uint8 = (clamp(color,0,1)*255).astype(uint8) (gs_renderer.py:1017, animation.py:1011)."""
    L = load_library()
    c = _f32c(color)
    F, _, H, W = c.shape
    out = torch.empty(F, H, W, 3, dtype=torch.uint8, device=c.device)
    with torch.cuda.device(c.device):
        _check(L.b200gs_pack_frames_u8(_ptr(c), _ptr(out), H, W, F, _stream(c.device)), "pack_frames_u8")
    return out


@torch.no_grad()
def render_frames(pc, xyz_frames: torch.Tensor, cameras, bg_color: torch.Tensor, scaling_modifier: float = 1.0,
                  chunk: int = MAX_VIEWS, antialiasing: bool = False, filter_3d: torch.Tensor = None) -> torch.Tensor:
    """Forward-only render of F frames with per-frame Gaussian centres xyz_frames [F,P,3]; everything else (scales,
    rotations, opacities, SH) is shared, exactly what animation.py changes between frames (only `_xyz`, :403).
    Returns uint8 frames [F,H,W,3] (the buffer animation.py appends to its video).  antialiasing: the screen-space mip
    filter (rasterizer.rasterize_views).  filter_3d: the 3D smoothing filter's [P] variances; the filter is per Gaussian, so
    one set (computed in the canonical pose, filter3d.compute_filter_3d) serves every frame."""
    F = xyz_frames.shape[0]
    dev = xyz_frames.device
    vm, pm, cp, tanx, tany = stack_cameras(cameras, dev)
    H, W = int(cameras[0].image_height), int(cameras[0].image_width)
    op, sh, sc, rot = pc.get_opacity, pc.get_features, pc.get_scaling, pc.get_rotation
    outs = []
    for f0 in range(0, F, chunk):
        f1 = min(F, f0 + chunk)
        color = rasterize_views(means3D=xyz_frames[f0:f1], opacities=op, viewmatrices=vm[f0:f1], projmatrices=pm[f0:f1],
                                camposs=cp[f0:f1], tanfovx=tanx[f0:f1], tanfovy=tany[f0:f1], image_height=H, image_width=W,
                                bg=bg_color, sh_degree=pc.active_sh_degree, shs=sh, scales=sc, rotations=rot,
                                scale_modifier=scaling_modifier, antialiasing=antialiasing, filter_3d=filter_3d)[0]
        outs.append(pack_frames_u8(color))
    return torch.cat(outs, 0)
