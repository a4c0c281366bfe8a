"""GPU: pose maps (b200gs_pose_keypoints + b200gs_pose_draw; pose.pose_maps) against the reference's images and the
specification (tests/pose_reference.py).

  1. every golden view of both styles, bit for bit, with kp within 1e-3 px of the reference's floats;
  2. 256 seeded views per style (orbit, near-head and near-back cameras of the shipped config, random occlusion flags,
     jittered keypoints) in batches of V = 64, 8 and 1, at 512 x 512, 1024 x 1024 (HumanSD thickness 20), 384 x 640
     (H != W: the reference's xs scale with H, ys with W) and 384 x 509 (a width that is not a multiple of 4): images
     bit-identical to the specification, whose keypoints
     use the GPU's float32 order and so must have the GPU's bits;
  3. bit-identical bytes across runs; exactly two launches and no host sync;
  4. invalid keypoints (w <= 0, non-finite, |coordinate| >= 2^20 px) leave their limbs undrawn and the rest identical;
  5. argument errors, in Python and at the C ABI.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

import pose_reference as PR
from humangaussian_b200 import pose as P
from humangaussian_b200 import rasterizer as R
from util import ROOT

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pose.npz")
SETS = ("humansd_default", "openpose_default", "humansd_8head", "openpose_2.5head")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _u8(pose):
    """The GPU's float32 image as u8, checking that every value is exactly some u8 / 255."""
    p = pose.cpu().numpy()
    u = np.rint(p * 255).astype(np.uint8)
    assert np.array_equal(u.astype(np.float32) / np.float32(255), p)
    return u


def _gpu(points, mvp, occ, style, H, W):
    return P.pose_maps(torch.tensor(points, device=DEV), torch.tensor(mvp, device=DEV), torch.tensor(occ, device=DEV), style, H, W)


@pytest.mark.parametrize("name", SETS)
def test_golden_views_bit_identical(golden, name):
    style = name.split("_")[0]
    pts, mvp, occ, kp, img = (golden[f"{name}/{k}"] for k in ("points", "mvp", "occlusion", "kp", "image"))
    pose, gkp = _gpu(pts, mvp, occ, style, 512, 512)
    u = _u8(pose)
    bad = [v for v in range(len(mvp)) if not np.array_equal(u[v], img[v])]
    assert not bad, f"{name}: views {bad} differ from the reference"
    assert np.abs(gkp.cpu().numpy() - kp).max() < 1e-3


def _mvp(el, az, dist, fovy, offset=0.0):
    """threestudio's look-at camera and get_projection_matrix(fovy, 1, 0.1, 1000) @ w2c, in float64, then float32."""
    el, az, fovy = math.radians(el), math.radians(az), math.radians(fovy)
    pos = np.array([dist * math.cos(el) * math.cos(az), dist * math.cos(el) * math.sin(az), dist * math.sin(el) + offset])
    ctr = np.array([0.0, 0.0, offset])
    look = (ctr - pos) / np.linalg.norm(ctr - pos)
    right = np.cross(look, [0.0, 0.0, 1.0])
    right /= np.linalg.norm(right)
    up = np.cross(right, look)
    Rm = np.stack([right, up, -look], 1)
    w2c = np.eye(4)
    w2c[:3, :3] = Rm.T
    w2c[:3, 3] = -Rm.T @ pos
    t = math.tan(fovy / 2)
    proj = np.zeros((4, 4))
    proj[0, 0], proj[1, 1] = 1 / t, -1 / t
    proj[2, 2], proj[2, 3], proj[3, 2] = -(1000.1) / 999.9, -2 * 1000 * 0.1 / 999.9, -1.0
    return (proj @ w2c).astype(np.float32)


def _random_batch(rng, golden, style, V):
    names = [n for n in SETS if n.startswith(style)]
    pts = golden[f"{names[rng.integers(len(names))]}/points"].copy()
    pts[:, :3] += rng.normal(0, 0.02, (len(pts), 3)).astype(np.float32)
    mvps = []
    for _ in range(V):
        kind = rng.integers(3)
        el, fovy = rng.uniform(-30, 30), rng.uniform(40, 70)
        if kind == 0:
            mvps.append(_mvp(el, rng.uniform(-180, 180), rng.uniform(1.5, 2.0), fovy))
        elif kind == 1:
            mvps.append(_mvp(el, rng.uniform(0, 180), rng.uniform(0.4, 0.6), fovy, 0.65))
        else:
            mvps.append(_mvp(el, rng.uniform(-180, 0), rng.uniform(0.6, 0.8), fovy, 0.65))
    return pts, np.stack(mvps), rng.random(V) < 0.7


@pytest.mark.parametrize("style", ["humansd", "openpose"])
def test_seeded_views_match_the_specification(golden, style):
    rng = np.random.default_rng(11 if style == "humansd" else 12)
    batches = [64, 64, 64] + [8] * 7 + [1] * 8
    sizes = [(512, 512), (1024, 1024), (384, 640), (384, 509)]  # 509: rows end in the draw's scalar-store tail
    n_views = n_near = 0
    for b, V in enumerate(batches):
        H, W = sizes[b % 4]
        pts, mvp, occ = _random_batch(rng, golden, style, V)
        pose, kp = _gpu(pts, mvp, occ, style, H, W)
        u, kp = _u8(pose), kp.cpu().numpy()
        for v in range(V):
            want, wkp = PR.draw(pts, mvp[v], occ[v], style, H, W)
            assert np.array_equal(kp[v].view(np.int32), wkp.view(np.int32)), f"batch {b} view {v}: keypoint bits differ"
            assert np.array_equal(u[v], want), f"batch {b} ({H}x{W}) view {v}: {(u[v] != want).any(-1).sum()} pixels differ"
            f = np.abs(wkp - np.rint(wkp))
            n_near += bool(np.any(f[np.isfinite(f)] < 1e-3))
            n_views += 1
    assert n_views == 256
    print(f"{style}: {n_views} views bit-identical; {n_near} have a keypoint within 1e-3 px of an integer")


@pytest.mark.parametrize("style", ["humansd", "openpose"])
def test_deterministic_two_launches_no_sync(golden, style):
    name = "humansd_default" if style == "humansd" else "openpose_default"
    pts = torch.tensor(golden[f"{name}/points"], device=DEV)
    mvp = torch.tensor(golden[f"{name}/mvp"], device=DEV)
    occ = torch.tensor(golden[f"{name}/occlusion"], device=DEV)
    a, ka = P.pose_maps(pts, mvp, occ, style)
    torch.cuda.synchronize()
    n0 = R.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b, kb = P.pose_maps(pts, mvp, occ, style)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert R.launch_count() - n0 == 2
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)) and torch.equal(ka.view(torch.int32), kb.view(torch.int32))
    p3, _ = P.pose_maps(pts[:, :3].contiguous(), mvp, occ, style)  # [K, 3] keypoints: w = 1 appended
    assert torch.equal(p3, a)


@pytest.mark.parametrize("style", ["humansd", "openpose"])
def test_invalid_keypoints_leave_their_limbs_undrawn(golden, style):
    """Orthographic views (w = the keypoint's own w) make each kind of invalid keypoint exact: w < 0, x = NaN, and
    x = 1e5 w (about 2.6e7 px)."""
    name = "humansd_default" if style == "humansd" else "openpose_default"
    pts0 = golden[f"{name}/points"]
    mvp = np.stack([np.diag([a, -a, a, 1.0]).astype(np.float32) for a in (0.8, 1.0, 1.2)])
    mvp[1, 0, 3] = 0.1
    occ = np.zeros(len(mvp), bool)
    ref = _u8(_gpu(pts0, mvp, occ, style, 512, 512)[0])
    for k, how in ((1, "nan"), (5, "far"), (9, "behind")):
        pts = pts0.copy()
        if how == "nan":
            pts[k, 0] = np.nan
        elif how == "far":
            pts[k, 0] = 1e5 * pts[k, 3]
        else:
            pts[k, 3] = -1.0
        u = _u8(_gpu(pts, mvp, occ, style, 512, 512)[0])
        for v in range(len(mvp)):
            xs, ys, z, valid = PR.keypoints(pts, mvp[v], 512, 512)
            assert not valid[k] and valid[np.arange(len(pts)) != k].all()
            assert np.array_equal(u[v], PR.draw_from_keypoints(xs, ys, z, valid, False, style, 512, 512)), (how, v)
            assert not np.array_equal(u[v], ref[v]), (how, v)  # the limbs at k are gone


def test_humansd_sum_gate(golden):
    """The reference draws a HumanSD skeleton only when its keypoint array sums to > 0.  A NaN coordinate, or one valid
    keypoint about 10^6 px left of the image, leaves the whole view blank, though other limbs lie on the image."""
    pts = golden["humansd_default/points"].copy()
    mvp = np.stack([np.diag([a, -a, a, 1.0]).astype(np.float32) for a in (1.0, 0.9)])
    far, nan = pts.copy(), pts.copy()
    far[16, 0] = -3900.0  # x = (x + 1) / 2 * 512 is about -1.0e6 (inside the 2^20 px limit) for both views
    nan[3, 1] = np.nan
    for p, drawn in ((pts, True), (far, False), (nan, False)):
        u = _u8(_gpu(p, mvp, np.zeros(2, bool), "humansd", 512, 512)[0])
        for v in range(2):
            xs, ys, z, valid = PR.keypoints(p, mvp[v], 512, 512)
            assert valid[16] and np.array_equal(u[v], PR.draw(p, mvp[v], False, "humansd", 512, 512)[0])
            assert u[v].any() == drawn


def test_argument_errors():
    kp = torch.zeros(17, 3, device=DEV)
    mvp = torch.eye(4, device=DEV)[None].repeat(2, 1, 1)
    occ = torch.zeros(2, dtype=torch.bool, device=DEV)
    with pytest.raises(ValueError, match="keypoints"):
        P.pose_maps(kp, mvp, occ, "openpose")  # 17 keypoints for an 18-keypoint style
    with pytest.raises(ValueError, match="occlusion"):
        P.pose_maps(kp, mvp, occ.to(torch.uint8))
    with pytest.raises(ValueError, match="mvp"):
        P.pose_maps(kp, mvp[:, :3], occ)
    with pytest.raises(ValueError, match="103"):
        P.pose_maps(kp, mvp, occ, height=64)
    with pytest.raises(ValueError, match="height"):
        P.pose_maps(kp, mvp, occ, height=0)
    with pytest.raises(RuntimeError, match="CUDA"):
        P.pose_maps(kp.cpu(), mvp, occ)

    L = R.load_library()
    s = torch.cuda.current_stream(DEV).cuda_stream
    pts = torch.zeros(18, 4, device=DEV)
    out_kp = torch.empty(2, 18, 2, device=DEV)
    need = L.b200gs_pose_scratch_bytes(1, 2, 64, 64)
    scratch = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = torch.empty(2, 64, 64, 3, device=DEV)
    limbs = (C.c_int32 * 34)(*[i for pair in P.OPENPOSE_LIMBS for i in pair])
    colors = (C.c_uint8 * 105)()
    o8 = occ.to(torch.uint8)

    def kcall(style=1, V=2, K=18, H=64, W=64, p=pts.data_ptr(), lim=limbs, sc=scratch.data_ptr(), nb=need, k=out_kp.data_ptr()):
        return L.b200gs_pose_keypoints(style, V, K, H, W, p, mvp.data_ptr(), o8.data_ptr(), lim, k, sc, nb, s)

    def dcall(style=1, V=2, H=64, W=64, sc=scratch.data_ptr(), nb=need, o=out.data_ptr()):
        return L.b200gs_pose_draw(style, V, H, W, colors, sc, nb, o, s)
    assert kcall() == R.OK and dcall() == R.OK
    assert kcall(style=2) == R.E_ARGS and dcall(style=-1) == R.E_ARGS
    assert kcall(V=0) == R.E_ARGS and kcall(K=17) == R.E_ARGS and kcall(p=None) == R.E_ARGS and dcall(o=None) == R.E_ARGS
    bad = (C.c_int32 * 34)(*([0] * 33 + [18]))
    assert kcall(lim=bad) == R.E_ARGS
    assert kcall(H=20000) == R.E_RANGE and kcall(style=0, K=17, H=64) == R.E_RANGE
    assert kcall(nb=need - 1) == R.E_BUFFER and dcall(nb=need - 1) == R.E_BUFFER
    assert kcall(p=pts.data_ptr() + 4) == R.E_BUFFER and dcall(o=out.data_ptr() + 4) == R.E_BUFFER
    assert kcall(k=out_kp.data_ptr() + 4) == R.E_BUFFER
    assert L.b200gs_pose_scratch_bytes(3, 2, 64, 64) == 0
    torch.cuda.synchronize()
