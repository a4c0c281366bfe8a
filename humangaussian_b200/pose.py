"""Pose maps on the GPU: the skeleton images HumanGaussian conditions its guidance on, for a whole view batch in two
launches (csrc/pose.cu, b200gs_pose_keypoints + b200gs_pose_draw).

`pose_maps` draws what the reference's `Skeleton.humansd_draw` (style "humansd") or `Skeleton.draw` (style "openpose")
draws for each view's mvp matrix (threestudio/utils/poser.py), byte for byte, without leaving the device:
  * keypoints: points3D @ mvp^T in float32 (a fixed summation order), divided by w; xs = (x + 1) / 2 * H and
    ys = (y + 1) / 2 * W (H and W swapped as in the reference), truncated toward zero for drawing;
  * occlusion: the reference's nose / ear depth and eye x-order rules, applied where the view's flag is set;
  * humansd: 16 limbs in table order, each a cv2.line of thickness int(10 * H / 512) plus two filled circles of radius
    thickness // 2, a later limb over an earlier one;
  * openpose: keypoints outside [0, H) x [0, W) are dropped, 18 filled circles of radius 4, then 17 ellipses of
    ellipse2Poly((mX, mY), (length / 2, 4), angle, 0, 360, 1) each blended as addWeighted(canvas, 0.4, filled, 0.6, 0);
  * output float32 u8 / 255, [V, H, W, 3].
The one divergence (DESIGN.md section 2): a keypoint with w <= 0, a non-finite coordinate or |coordinate| >= 2^20 px is
invalid, and nothing that uses it is drawn; the reference crashes or draws garbage there.

The style tables below restate the COCO-17 (HumanSD) and OpenPose-18 conventions the reference draws with; the golden
images pin them.
"""
from __future__ import annotations

import ctypes as C
from typing import Tuple

import torch

from . import rasterizer as R

# HumanSD (COCO-17 keypoints): limb k joins HUMANSD_LIMBS[k] and is coloured with palette entry k ^ 1 (the reference's
# table pairs its colour indices 1, 0, 3, 2, ...).  HUMANSD_COLORS[i] = int(255 * c) of seaborn's 16-colour "hls"
# palette: colorsys.hls_to_rgb((i / 16 + 0.01) % 1, 0.6, 0.65).
HUMANSD_LIMBS = ((0, 1), (0, 2), (1, 3), (2, 4), (3, 5), (4, 6), (5, 7), (6, 8), (7, 9), (8, 10), (5, 11), (6, 12), (11, 13),
                 (12, 14), (13, 15), (14, 16))
HUMANSD_COLOR_INDEX = tuple(k ^ 1 for k in range(16))
HUMANSD_COLORS = ((219, 94, 86), (219, 144, 86), (219, 194, 86), (194, 219, 86), (145, 219, 86), (95, 219, 86),
                  (86, 219, 127), (86, 219, 177), (86, 211, 219), (86, 161, 219), (86, 111, 219), (111, 86, 219),
                  (160, 86, 219), (210, 86, 219), (219, 86, 178), (219, 86, 128))
# OpenPose-18: limb k joins OPENPOSE_LIMBS[k] in OPENPOSE_COLORS[k]; keypoint i's circle is OPENPOSE_COLORS[i].
OPENPOSE_LIMBS = ((0, 1), (1, 2), (2, 3), (3, 4), (1, 5), (5, 6), (6, 7), (1, 8), (8, 9), (9, 10), (1, 11), (11, 12), (12, 13),
                  (0, 14), (14, 16), (0, 15), (15, 17))
OPENPOSE_COLORS = ((255, 0, 0), (255, 85, 0), (255, 170, 0), (255, 255, 0), (170, 255, 0), (85, 255, 0), (0, 255, 0),
                   (0, 255, 85), (0, 255, 170), (0, 255, 255), (0, 170, 255), (0, 85, 255), (0, 0, 255), (85, 0, 255),
                   (170, 0, 255), (255, 0, 255), (255, 0, 170), (255, 0, 85))
STYLES = {"humansd": 0, "openpose": 1}
NUM_KEYPOINTS = {"humansd": 17, "openpose": 18}


def _limbs_and_colors(style):
    if style == "humansd":
        return HUMANSD_LIMBS, [HUMANSD_COLORS[HUMANSD_COLOR_INDEX[k]] for k in range(len(HUMANSD_LIMBS))]
    return OPENPOSE_LIMBS, list(OPENPOSE_COLORS) + [OPENPOSE_COLORS[k] for k in range(len(OPENPOSE_LIMBS))]


@torch.no_grad()
def pose_maps(keypoints, mvp, occlusion, style="humansd", height=512, width=512) -> Tuple[torch.Tensor, torch.Tensor]:
    """The reference's pose images for V views: (pose [V, H, W, 3] float32 in [0, 1], kp [V, K, 2] float32).

    keypoints: [K, 3] or [K, 4] (w = 1 appended to [K, 3]) in the reference's convention (Skeleton.points3D), K = 17 for
    "humansd" and 18 for "openpose"; mvp: [V, 4, 4] (batch['mvp_mtx']); occlusion: [V] bool, the reference's
    enable_occlusion per view.  All on one CUDA device; nothing waits for the device.  kp holds the float pixel
    coordinates the reference returns (xs = (x + 1) / 2 * height, ys = (y + 1) / 2 * width).  "humansd" needs
    height >= 103 (line thickness int(10 * height / 512) >= 2)."""
    if style not in STYLES:
        raise ValueError(f"b200gs: pose_maps: style must be one of {sorted(STYLES)} (got {style!r})")
    K = NUM_KEYPOINTS[style]
    for name, t in (("keypoints", keypoints), ("mvp", mvp), ("occlusion", occlusion)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"b200gs: pose_maps: {name} must be a tensor (got {type(t).__name__})")
        if t.device.type != "cuda":
            raise RuntimeError(f"b200gs: pose_maps: {name} must be on a CUDA device (got {t.device}); there is no CPU path")
    dev = mvp.device
    if keypoints.device != dev or occlusion.device != dev:
        raise ValueError("b200gs: pose_maps: keypoints, mvp and occlusion must be on one device")
    if keypoints.dim() != 2 or keypoints.shape[0] != K or keypoints.shape[1] not in (3, 4) or not keypoints.dtype.is_floating_point:
        raise ValueError(f"b200gs: pose_maps: keypoints must be a float [{K}, 3] or [{K}, 4] tensor for style {style!r} "
                         f"(got {keypoints.dtype} {tuple(keypoints.shape)})")
    if mvp.dim() != 3 or mvp.shape[1:] != (4, 4) or mvp.shape[0] < 1 or not mvp.dtype.is_floating_point:
        raise ValueError(f"b200gs: pose_maps: mvp must be a float [V, 4, 4] tensor with V >= 1 (got {mvp.dtype} {tuple(mvp.shape)})")
    V = mvp.shape[0]
    if occlusion.shape != (V,) or occlusion.dtype != torch.bool:
        raise ValueError(f"b200gs: pose_maps: occlusion must be a [{V}] bool tensor (got {occlusion.dtype} {tuple(occlusion.shape)})")
    if not isinstance(height, int) or not isinstance(width, int) or not (1 <= height <= 16384 and 1 <= width <= 16384):
        raise ValueError(f"b200gs: pose_maps: height and width must be integers in 1..16384 (got {height!r}, {width!r})")
    if style == "humansd" and height < 103:
        raise ValueError(f"b200gs: pose_maps: the humansd style draws lines of thickness int(10 * height / 512), which needs "
                         f"height >= 103 (got {height})")
    pts = keypoints.detach().to(torch.float32)
    if pts.shape[1] == 3:
        pts = torch.cat([pts, torch.ones(K, 1, dtype=torch.float32, device=dev)], 1)
    pts = pts.contiguous()
    if pts.data_ptr() % 16:  # the kernel reads keypoints as float4
        pts = pts.clone()
    m = mvp.detach().to(torch.float32).contiguous()
    occ = occlusion.detach().to(torch.uint8).contiguous()
    limbs, colors = _limbs_and_colors(style)
    limbs_h = (C.c_int32 * (2 * len(limbs)))(*[i for pair in limbs for i in pair])
    colors_h = (C.c_uint8 * (3 * len(colors)))(*[c for rgb in colors for c in rgb])
    s = STYLES[style]
    L = R.load_library()
    with torch.cuda.device(dev):
        kp = torch.empty(V, K, 2, dtype=torch.float32, device=dev)
        pose = torch.empty(V, height, width, 3, dtype=torch.float32, device=dev)
        scratch = torch.empty(L.b200gs_pose_scratch_bytes(s, V, height, width), dtype=torch.uint8, device=dev)
        R._check(L.b200gs_pose_keypoints(s, V, K, height, width, R._ptr(pts), R._ptr(m), R._ptr(occ), limbs_h, R._ptr(kp),
                                         R._ptr(scratch), scratch.numel(), R._stream(dev)), "pose_keypoints")
        R._check(L.b200gs_pose_draw(s, V, height, width, colors_h, R._ptr(scratch), scratch.numel(), R._ptr(pose), R._stream(dev)),
                 "pose_draw")
    return pose, kp
