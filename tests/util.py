"""Shared helpers for the parity tests: seeded small scenes + oracle/dense invocation."""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from humangaussian_b200.cameras import Camera, orbit_c2w  # noqa: E402
from humangaussian_b200.scene import synthetic_body  # noqa: E402


def small_scene(P=200, deg=1, seed=0, H=40, W=56, elev=12.0, azim=35.0, dist=1.6, fovy_deg=55.0, big=True):
    """Activated inputs (numpy float32) + camera for one view of a synthetic body."""
    p = synthetic_body(P, sh_degree=deg, seed=seed)
    if big:  # enlarge so that a few hundred Gaussians cover a tiny image with real overlap
        p.scaling += math.log(6.0)
        p.opacity += 1.5
    cam = Camera(orbit_c2w(elev, azim, dist), math.radians(fovy_deg), H, W)
    with torch.no_grad():
        inp = dict(
            means3D=p.get_xyz.numpy().copy(), opacities=p.get_opacity.numpy().copy(),
            shs=p.get_features.numpy().copy(), scales=p.get_scaling.numpy().copy(),
            rotations=p.get_rotation.numpy().copy(), sh_degree=deg,
            viewmatrix=cam.world_view_transform.numpy().copy(), projmatrix=cam.full_proj_transform.numpy().copy(),
            campos=cam.camera_center.numpy().copy(), bg=np.array([0.1, 0.4, 0.7], np.float32),
            image_height=H, image_width=W, tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5),
            scale_modifier=1.0)
    return inp, cam, p


def screen_scene(px, py, depth, sigma, opacity, color=None, cov2d=None, H=64, W=128, fovy_deg=60.0):
    """Activated inputs (colors_precomp / cov3D_precomp) of Gaussians given in screen space, for scenes that must hit exact
    list and patch positions.  Per Gaussian: pixel centre (px, py), view depth, isotropic screen sigma in pixels (or a
    screen-space 2x2 covariance cov2d [N,2,2], overriding sigma), opacity, colour.  The camera sits at the origin looking
    down +z (identity view matrix); each Gaussian is unprojected through it, with a negligible depth extent.  The rasteriser
    adds 0.3 px^2 to the screen covariance, so with sigma < 0.3 px that dilation sets the footprint: a Gaussian centred in
    an 8x4 patch stays inside it.  Colours default to a fixed pseudo-random draw."""
    from humangaussian_b200.cameras import getProjectionMatrix
    px, py, z = (np.asarray(a, np.float64).reshape(-1) for a in (px, py, depth))
    n = len(px)
    tany = math.tan(math.radians(fovy_deg) / 2)
    tanx = tany * W / H
    f = W / (2 * tanx)  # = H / (2 * tany): square pixels
    x = ((2 * px + 1) / W - 1) * tanx * z
    y = ((2 * py + 1) / H - 1) * tany * z
    if cov2d is None:
        s = np.broadcast_to(np.asarray(sigma, np.float64), (n,))
        cov2d = np.zeros((n, 2, 2))
        cov2d[:, 0, 0] = cov2d[:, 1, 1] = s * s
    k = (z / f) ** 2
    cov = np.stack([cov2d[:, 0, 0] * k, cov2d[:, 0, 1] * k, np.zeros(n), cov2d[:, 1, 1] * k, np.zeros(n), 1e-4 * k], 1)
    if color is None:
        color = np.random.RandomState(n).rand(n, 3) * 0.8 + 0.1
    proj = getProjectionMatrix(0.01, 100.0, 2 * math.atan(tanx), 2 * math.atan(tany)).transpose(0, 1).numpy()
    return dict(means3D=np.stack([x, y, z], 1).astype(np.float32),
                opacities=np.broadcast_to(np.asarray(opacity, np.float32), (n,)).reshape(n, 1).copy(),
                colors_precomp=np.asarray(color, np.float32).reshape(n, 3).copy(), cov3D_precomp=cov.astype(np.float32),
                sh_degree=0, viewmatrix=np.eye(4, dtype=np.float32), projmatrix=proj.astype(np.float32),
                campos=np.zeros(3, np.float32), bg=np.array([0.1, 0.4, 0.7], np.float32), image_height=H, image_width=W,
                tanfovx=tanx, tanfovy=tany, scale_modifier=1.0)


def grad_images(H, W, seed=0):
    rng = np.random.RandomState(seed)
    return (rng.randn(3, H, W).astype(np.float32), rng.randn(1, H, W).astype(np.float32),
            rng.randn(1, H, W).astype(np.float32))


def close(a, b, atol=1e-5, rtol=1e-4):
    """The north-star tolerance: |a-b| <= 1e-5 + 1e-4*|b|.  Returns (ok, worst violation ratio)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    err = np.abs(a - b)
    lim = atol + rtol * np.abs(b)
    return bool((err <= lim).all()), float((err / lim).max()) if err.size else 0.0


def close_rows(a, b, atol=1e-5, rtol=1e-4):
    """Like close(), but the relative term uses each row's largest magnitude: for float32-vs-float64 checks where one
    component of a per-Gaussian gradient vector is a cancellation of terms the size of its neighbours."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    a2, b2 = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
    err = np.abs(a2 - b2)
    lim = atol + rtol * np.abs(b2).max(axis=1, keepdims=True)
    return bool((err <= lim).all()), float((err / lim).max()) if err.size else 0.0


def grads_agree(a, b, atol=1e-5, rtol=1e-4, min_elementwise=0.999, min_rows=1.0, row_cap=1.0):
    """The gradient parity criterion of the GPU tests (DESIGN.md section 2).

    A per-Gaussian gradient is a float32 sum over hundreds of pixels with heavy cancellation (the mean/scale derivatives
    are odd functions over the footprint), accumulated in a different order on the GPU (shuffle tree + float atomics)
    than in the oracle (exact sums).  One component of a Gaussian's gradient vector can therefore be a near-zero
    cancellation of terms the size of its siblings, where *elementwise* relative error is meaningless -- upstream's own
    atomics have the same run-to-run behaviour (SURVEY.md A.9).  So:
      * every Gaussian's gradient VECTOR must satisfy |a-b| <= 1e-5 + 1e-4 * max|row of b|   (all rows, no exceptions);
      * and the plain elementwise |a-b| <= 1e-5 + 1e-4*|b| must hold for at least 99.9 % of the elements.
    Returns (ok, message)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.size == 0:
        return True, "empty"
    a2, b2 = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
    err = np.abs(a2 - b2)
    row_lim = atol + rtol * np.abs(b2).max(axis=1, keepdims=True)
    row_worst = float((err / row_lim).max())
    el_ok = float((err <= atol + rtol * np.abs(b2)).mean())
    rows_ok = float(((err / row_lim).max(axis=1) <= 1.0).mean())
    # parity tests: every row inside the tolerance (min_rows = 1, row_cap = 1).  Property tests that compare two
    # NON-DETERMINISTIC float32 evaluations at full size may allow a 1e-4 fraction of ill-conditioned rows up to row_cap.
    ok = rows_ok >= min_rows and row_worst <= max(row_cap, 1.0) and el_ok >= min_elementwise
    return ok, (f"row-wise worst {row_worst:.2f}x of tolerance, rows inside {100 * rows_ok:.4f}%, "
                f"elementwise pass rate {100 * el_ok:.4f}%")
