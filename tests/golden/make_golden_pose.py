"""Golden pose maps, produced by RUNNING THE REFERENCE'S OWN `Skeleton.humansd_draw` / `Skeleton.draw`
(threestudio/utils/poser.py) with cv2 on the CPU.

    HUMANGAUSSIAN_ROOT=<HumanGaussian checkout> python tests/golden/make_golden_pose.py   ->  tests/golden/ref_pose.npz

poser.py is loaded by file path (threestudio/__init__.py needs pytorch_lightning).  seaborn is stubbed: its
color_palette("hls", n) is seaborn's hls formula, colorsys.hls_to_rgb((i / n + 0.01) % 1, 0.6, 0.65).

Four keypoint sets, each drawn at 512 x 512 for 51 views:
  humansd_default / openpose_default   the Skeleton's built-in keypoints after GaussianDreamer's scale(-10)
  humansd_8head / openpose_2.5head     load_json presets, then scale(-10)
Views (mvp = get_projection_matrix(fovy, 1, 0.1, 1000) @ w2c, threestudio's convention; occlusion flag =
GaussianDreamer's `abs(azimuth) > 120 * pi / 180` with the azimuth in degrees, as the reference computes it):
  32 orbit views from configs/test.yaml's ranges (elevation [-30, 30], distance [1.5, 2], fovy [40, 70] degrees),
  8 near-head close-ups (distance [0.4, 0.6], azimuth [0, 180], centre raised by 0.65),
  8 near-back close-ups (distance [0.6, 0.8], azimuth [-180, 0], centre raised by 0.65),
  one front view (|azimuth| <= 2, occlusion off), one back view (azimuth 180), and one view whose mvp row 0 is minus row 3, so every keypoint lands exactly on x = 0.
A drawn view is redrawn when any keypoint has w <= 0 or |coordinate| >= 2^20 px (where the reference's output is
undefined) or when a truncated quantity (a keypoint coordinate; for OpenPose also a limb's centre, length / 2 or angle)
lies within 1e-4 of an integer, or when a keypoint is so ill-conditioned (w near 0) that the reference's float32
coordinate is 1e-3 px or more from its float64 value, so that any float32 implementation can match these images bit for
bit.  The edge view
is exempt from the latter: its x coordinates are exactly 0.
No reference source is copied into the repository; the reference is not needed to run the tests.
"""
import colorsys
import importlib.util
import math
import os
import sys
import types

import numpy as np
import torch

REF = os.environ["HUMANGAUSSIAN_ROOT"]
HERE = os.path.dirname(os.path.abspath(__file__))
N_ORBIT, N_HEAD, N_BACK = 32, 8, 8
EPS = 1e-4


def _load_poser():
    sns = types.ModuleType("seaborn")

    def color_palette(name, n):
        assert name == "hls"
        return [colorsys.hls_to_rgb((i / n + 0.01) % 1, 0.6, 0.65) for i in range(n)]
    sns.color_palette = color_palette
    sys.modules["seaborn"] = sns
    spec = importlib.util.spec_from_file_location("ref_poser", os.path.join(REF, "threestudio", "utils", "poser.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _mvp(elevation, azimuth, distance, fovy_deg, offset=0.0):
    """threestudio's look-at c2w (uncond.py) and get_mvp_matrix(c2w, get_projection_matrix(fovy, 1, 0.1, 1000))."""
    el, az = torch.tensor(elevation * math.pi / 180), torch.tensor(azimuth * math.pi / 180)
    pos = torch.stack([distance * torch.cos(el) * torch.cos(az), distance * torch.cos(el) * torch.sin(az), distance * torch.sin(el)])
    center = torch.zeros(3)
    pos[2] += offset
    center[2] += offset
    up = torch.tensor([0.0, 0.0, 1.0])
    lookat = torch.nn.functional.normalize(center - pos, dim=-1)
    right = torch.nn.functional.normalize(torch.linalg.cross(lookat, up), dim=-1)
    up = torch.nn.functional.normalize(torch.linalg.cross(right, lookat), dim=-1)
    c2w = torch.eye(4)
    c2w[:3, :3] = torch.stack([right, up, -lookat], dim=-1)
    c2w[:3, 3] = pos
    fovy = torch.tensor(fovy_deg * math.pi / 180)
    far, near = 1000.0, 0.1
    proj = torch.zeros(4, 4)
    proj[0, 0] = 1.0 / torch.tan(fovy / 2.0)
    proj[1, 1] = -1.0 / torch.tan(fovy / 2.0)
    proj[2, 2] = -(far + near) / (far - near)
    proj[2, 3] = -2.0 * far * near / (far - near)
    proj[3, 2] = -1.0
    w2c = torch.zeros(4, 4)
    w2c[:3, :3] = c2w[:3, :3].T
    w2c[:3, 3:] = -c2w[:3, :3].T @ c2w[:3, 3:]
    w2c[3, 3] = 1.0
    return (proj @ w2c).numpy().astype(np.float32)


def _near_int(v):
    v = np.asarray(v, np.float64)
    return bool(np.any(np.abs(v - np.rint(v)) < EPS))


def _truncated(style, kp, poser_lines):
    """Every float the reference truncates for this view."""
    xs, ys = kp[:, 0].astype(np.float32), kp[:, 1].astype(np.float32)
    vals = [xs, ys]
    if style == "openpose":
        for a, b in poser_lines:
            X, Y = xs[[a, b]], ys[[a, b]]
            length = ((Y[0] - Y[1]) ** 2 + (X[0] - X[1]) ** 2) ** 0.5
            vals += [[np.mean(X), np.mean(Y), length / 2, math.degrees(math.atan2(Y[0] - Y[1], X[0] - X[1]))]]
    return np.concatenate([np.ravel(np.asarray(v, np.float64)) for v in vals])


def _usable(points, mvp, H, W):
    p = points @ mvp.T
    if np.any(p[:, 3] <= 0):
        return False
    xy = p[:, :2] / p[:, 3:]
    return bool(np.all(np.isfinite(xy)) and np.all(np.abs((xy + 1) / 2 * max(H, W)) < 2 ** 20))


def make_set(poser, style, preset, seed, H=512, W=512):
    sk = poser.Skeleton(humansd_style=(style == "humansd"))
    if preset:
        sk.load_json(preset)
    sk.scale(-10)
    points = sk.points3D.astype(np.float32)
    rng = np.random.default_rng(seed)
    plans = ([("orbit", i) for i in range(N_ORBIT)] + [("head", i) for i in range(N_HEAD)] + [("back", i) for i in range(N_BACK)] +
             [("front", 0), ("backview", 0), ("edge", 0)])
    mvps, occl, kps, imgs = [], [], [], []
    draw = sk.humansd_draw if style == "humansd" else sk.draw
    for kind, i in plans:
        for _ in range(1000):
            fovy = rng.uniform(40, 70)
            el = rng.uniform(-30, 30)
            if kind == "orbit":
                az = (rng.uniform() + i) / N_ORBIT * 360 - 180
                mvp = _mvp(el, az, rng.uniform(1.5, 2.0), fovy)
            elif kind == "head":
                az = rng.uniform(0, 180)
                mvp = _mvp(el, az, rng.uniform(0.4, 0.6), fovy, 0.65)
            elif kind == "back":
                az = rng.uniform(-180, 0)
                mvp = _mvp(el, az, rng.uniform(0.6, 0.8), fovy, 0.65)
            elif kind == "front":  # |azimuth| <= 2 degrees: the one range where the reference turns occlusion off
                az = rng.uniform(-2, 2)
                mvp = _mvp(el, az, rng.uniform(1.5, 2.0), fovy)
            elif kind == "backview":
                az = 180.0
                mvp = _mvp(el, az, rng.uniform(1.5, 2.0), fovy)
            else:
                az = rng.uniform(-180, 180)
                mvp = _mvp(el, az, rng.uniform(1.5, 2.0), fovy)
                mvp[0] = -mvp[3]
            backview = abs(az) > 120 * np.pi / 180  # GaussianDreamer.forward's expression (azimuth in degrees)
            if not _usable(points, mvp, H, W):
                continue
            img, kp = draw(mvp, H, W, backview)
            kp = np.asarray(kp)[..., :2].reshape(-1, 2) if style == "humansd" else np.asarray(kp)
            t = _truncated(style, kp, sk.lines)
            if kind == "edge":  # x = 0, centre x = 0 and angle +-90 are exact here
                assert np.all(kp[:, 0] == 0)
                t = t[t != np.rint(t)]
            p64 = points.astype(np.float64) @ mvp.astype(np.float64).T
            kp64 = (p64[:, :2] / p64[:, 3:] + 1) / 2 * np.array([H, W])
            if _near_int(t) or np.abs(kp64 - kp).max() >= 1e-3:
                continue
            break
        else:
            raise RuntimeError(f"no usable {kind} view for {style}")
        mvps.append(mvp)
        occl.append(backview)
        kps.append(kp.astype(np.float32))
        imgs.append(np.rint(np.asarray(img) * 255).astype(np.uint8))
        assert np.array_equal(imgs[-1].astype(np.float32) / np.float32(255), np.asarray(img, np.float32))
    return dict(points=points, mvp=np.stack(mvps), occlusion=np.array(occl), kp=np.stack(kps), image=np.stack(imgs))


def main():
    poser = _load_poser()
    out = {}
    for name, style, preset, seed in (("humansd_default", "humansd", None, 1), ("openpose_default", "openpose", None, 2),
                                      ("humansd_8head", "humansd", "8head", 3), ("openpose_2.5head", "openpose", "2.5head", 4)):
        d = make_set(poser, style, preset, seed)
        for k, v in d.items():
            out[f"{name}/{k}"] = v
        print(name, d["image"].shape, "occluded views", int(d["occlusion"].sum()))
    np.savez_compressed(os.path.join(HERE, "ref_pose.npz"), **out)


if __name__ == "__main__":
    main()
