"""CPU: the pose-map specification (tests/pose_reference.py) against the reference's own images and, where cv2 is
importable, against cv2's drawing rule by rule.  No GPU."""
import colorsys
import math
import os

import numpy as np
import pytest
import torch

import pose_reference as R
from humangaussian_b200 import pose as P
from util import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pose.npz")
SETS = ("humansd_default", "openpose_default", "humansd_8head", "openpose_2.5head")

try:
    import cv2
except ImportError:  # the restatement is still pinned by the golden images
    cv2 = None
needs_cv2 = pytest.mark.skipif(cv2 is None, reason="cv2 not importable")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _style(name):
    return name.split("_")[0]


def test_palette_is_seaborn_hls():
    """HUMANSD_COLORS = int(255 * c) of seaborn's color_palette("hls", 16): hues i / 16 + 0.01, lightness 0.6,
    saturation 0.65."""
    want = tuple(tuple(int(255 * c) for c in colorsys.hls_to_rgb((i / 16 + 0.01) % 1, 0.6, 0.65)) for i in range(16))
    assert P.HUMANSD_COLORS == want
    assert P.HUMANSD_COLOR_INDEX == (1, 0, 3, 2, 5, 4, 7, 6, 9, 8, 11, 10, 13, 12, 15, 14)


def test_sine_table_is_far_from_its_rounding_boundaries():
    """The GPU builds the 7-decimal sine table from its own double sin(); that gives the same floats as Python's as long
    as no sin(i deg) * 1e7 lies near a half-integer, which holds with a margin far above any last-bit sin error."""
    s = np.array([math.sin(math.radians(i)) * 1e7 for i in range(451)])
    assert np.abs(s - np.floor(s) - 0.5).min() > 1e-3
    assert np.array_equal(R.SIN_TABLE, np.array([np.rint(v) / 1e7 for v in s]).astype(np.float32))


@pytest.mark.parametrize("name", SETS)
def test_restatement_reproduces_every_golden_image(golden, name):
    style = _style(name)
    pts, mvp, occ, kp, img = (golden[f"{name}/{k}"] for k in ("points", "mvp", "occlusion", "kp", "image"))
    assert len(mvp) >= 48 and img.shape[1:] == (512, 512, 3)
    for v in range(len(mvp)):
        mine, mkp = R.draw(pts, mvp[v], occ[v], style, 512, 512)
        assert np.array_equal(mine, img[v]), f"{name} view {v}: {(mine != img[v]).any(-1).sum()} pixels differ"
        assert np.array_equal(np.trunc(mkp), np.trunc(kp[v])), f"{name} view {v}: integer keypoints differ"
        assert np.abs(mkp - kp[v]).max() < 1e-3


@pytest.mark.parametrize("name", SETS)
def test_goldens_are_well_conditioned(golden, name):
    """No truncated quantity of a golden view lies within 1e-4 of an integer (the edge view's exact x = 0, centre x = 0
    and +-90 degree angles aside), so every float32 implementation can match the images bit for bit."""
    style = _style(name)
    kp, occ = golden[f"{name}/kp"], golden[f"{name}/occlusion"]
    assert occ.any() and not occ.all()  # the reference's expression turns occlusion on for all but |azimuth| <= 2.09 deg
    for v in range(len(kp)):
        xs, ys = kp[v, :, 0], kp[v, :, 1]
        vals = [xs, ys]
        if style == "openpose":
            for a, b in P.OPENPOSE_LIMBS:
                X, Y = np.float32([xs[a], xs[b]]), np.float32([ys[a], ys[b]])
                length = ((Y[0] - Y[1]) ** 2 + (X[0] - X[1]) ** 2) ** 0.5
                vals.append([np.mean(X), np.mean(Y), length / 2, math.degrees(math.atan2(Y[0] - Y[1], X[0] - X[1]))])
        t = np.concatenate([np.ravel(np.asarray(x, np.float64)) for x in vals])
        if np.all(xs == 0):
            t = t[t != np.rint(t)]
        assert np.abs(t - np.rint(t)).min() >= 1e-4, f"{name} view {v}"
    assert np.all(kp[-1, :, 0] == 0)  # the edge view


def test_golden_shapes_fit_four_runs_per_row(golden):
    """The GPU stores each shape as up to 4 disjoint runs per row; no HumanSD limb or OpenPose circle / ellipse of the
    goldens needs more (a thin limb's edge pixels can leave a one-pixel gap, so one run is not enough)."""
    for name in SETS:
        style = _style(name)
        pts, mvp, occ = golden[f"{name}/points"], golden[f"{name}/mvp"], golden[f"{name}/occlusion"]
        for v in range(0, len(mvp), 5):
            xs, ys, z, valid = R.keypoints(pts, mvp[v], 512, 512)
            if style == "humansd":
                shapes = [r for _, r in R.humansd_shapes(xs, ys, z, valid, bool(occ[v]), 512, 512)]
            else:
                c, l = R.openpose_shapes(xs, ys, z, valid, bool(occ[v]), 512, 512)
                shapes = [r for _, r in c + l]
            for runs in shapes:
                _assert_few_runs(runs, 512, 512)


def _assert_few_runs(runs, W, H):
    assert R.runs_per_row(runs, W, H).max(initial=0) <= 4


def _cv2_mask(draw, W, H):
    img = np.zeros((H, W), np.uint8)
    draw(img)
    return img > 0


@needs_cv2
def test_thick_lines_and_circles_match_cv2():
    """cv2.line(thickness T, LINE_8) and cv2.circle(-1) on 3 000 seeded segments: degenerate, horizontal, vertical,
    partly and wholly off-image, across corners, and with ends up to 2^20 px away; each at most 4 runs per row."""
    W, H = 160, 120
    rng = np.random.default_rng(7)
    for t in range(3000):
        kind = t % 6
        if kind == 0:
            p = rng.integers(-40, 200, 4)
        elif kind == 1:
            p = rng.integers(-3000, 3000, 4)
        elif kind == 2:
            p = rng.integers(-(1 << 20) + 1, 1 << 20, 4)
        elif kind == 3:  # horizontal / vertical / degenerate
            p = rng.integers(-20, 180, 4)
            p[2 + (t // 6) % 2] = p[(t // 6) % 2]
            if t % 5 == 0:
                p[2:] = p[:2]
        elif kind == 4:  # across a corner
            c = [(0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1)][(t // 6) % 4]
            p = np.array([c[0] - 30, c[1] + 30, c[0] + 30, c[1] - 30]) + rng.integers(-8, 9, 4)
        else:  # wholly off-image
            p = rng.integers(200, 400, 4) * np.array([1, 1, 1, 1]) * rng.choice([-1, 1])
        x0, y0, x1, y1 = map(int, p)
        T = int(rng.choice([2, 3, 4, 5, 10, 11, 20]))
        runs = R.thick_line(x0, y0, x1, y1, T, W, H)
        assert np.array_equal(R.runs_mask(runs, W, H), _cv2_mask(lambda im: cv2.line(im, (x0, y0), (x1, y1), 255, T), W, H)), \
            (x0, y0, x1, y1, T)
        _assert_few_runs(runs, W, H)
        cx, cy, r = x0 % 200 - 20, y0 % 160 - 20, int(rng.integers(0, 12))
        assert np.array_equal(R.runs_mask(R.circle_filled(cx, cy, r, W, H), W, H),
                              _cv2_mask(lambda im: cv2.circle(im, (cx, cy), r, 255, -1), W, H)), (cx, cy, r)


@needs_cv2
def test_fixed_point_edges_and_polygons_match_cv2():
    """fillConvexPoly at shift 16 with two vertices draws only its edge lines, so it pins the fixed-point line by itself;
    at shift 16 with four (thick-line quads) and at shift 0 with ellipse polygons it pins the scan converter."""
    W, H = 160, 120
    rng = np.random.default_rng(8)
    for _ in range(2000):
        p = [int(v) for v in rng.integers(-20 << 16, 180 << 16, 4)]
        want = _cv2_mask(lambda im: cv2.fillConvexPoly(im, np.array([p[:2], p[2:]], np.int32), 255, cv2.LINE_8, 16), W, H)
        assert np.array_equal(R.runs_mask(R.fill_convex([tuple(p[:2]), tuple(p[2:])], 16, W, H), W, H), want), p
    for _ in range(1000):
        c = rng.integers(-30 << 16, 190 << 16, 2)
        d = rng.integers(-60 << 16, 60 << 16, 2)
        e = rng.integers(-(4 << 16), 4 << 16, 2)
        quad = [tuple(int(v) for v in q) for q in (c + e, c - e, c + d - e, c + d + e)]
        want = _cv2_mask(lambda im: cv2.fillConvexPoly(im, np.array(quad, np.int32), 255, cv2.LINE_8, 16), W, H)
        assert np.array_equal(R.runs_mask(R.fill_convex(quad, 16, W, H), W, H), want), quad
    for _ in range(1500):
        cx, cy = (int(v) for v in rng.integers(-60, 220, 2))
        ax, ang = int(rng.integers(0, 200)), int(rng.integers(-180, 181))
        poly = cv2.ellipse2Poly((cx, cy), (ax, 4), ang, 0, 360, 1)
        runs = R.fill_convex([tuple(map(int, q)) for q in poly], 0, W, H)
        assert np.array_equal(R.runs_mask(runs, W, H), _cv2_mask(lambda im: cv2.fillConvexPoly(im, poly, 255), W, H)), (cx, cy, ax, ang)
        _assert_few_runs(runs, W, H)


@needs_cv2
def test_ellipse2poly_matches_cv2_exhaustively():
    """Every (major axis, angle) an OpenPose limb can produce at 512 x 512 (int(length / 2) <= 362, int(angle) in
    [-180, 180]), at the image centre and at a seeded off-centre point."""
    rng = np.random.default_rng(9)
    for a in range(363):
        for cx, cy in ((256, 256), tuple(int(v) for v in rng.integers(-50, 560, 2))):
            for ang in range(-180, 181):
                want = cv2.ellipse2Poly((cx, cy), (a, 4), ang, 0, 360, 1)
                got = R.ellipse2poly(cx, cy, a, 4, ang)
                assert want.tolist() == [list(q) for q in got], (cx, cy, a, ang)


@needs_cv2
def test_add_weighted_matches_cv2_on_every_pair():
    a = np.arange(256, dtype=np.uint8)
    A, B = np.meshgrid(a, a)
    assert np.array_equal(cv2.addWeighted(A, 0.4, B, 0.6, 0), R.add_weighted(A, B))


def test_invalid_keypoints_are_not_drawn():
    """A keypoint behind the camera (w <= 0) or 2^20 px or more away is invalid: its limbs (and OpenPose circle) go."""
    pts = np.concatenate([np.random.default_rng(1).uniform(-0.3, 0.3, (18, 3)), np.ones((18, 1))], 1).astype(np.float32)
    mvp = np.eye(4, dtype=np.float32)
    pts[:, 3] = 1.0
    pts[5, 3] = -1.0  # w < 0
    xs, ys, z, valid = R.keypoints(pts, mvp, 512, 512)
    assert not valid[5] and valid[np.arange(18) != 5].all()
    for style, limbs in (("humansd", P.HUMANSD_LIMBS), ("openpose", P.OPENPOSE_LIMBS)):
        K = P.NUM_KEYPOINTS[style]
        if style == "humansd":
            drawn = [k for k, _ in R.humansd_shapes(xs[:K], ys[:K], z[:K], valid[:K], False, 512, 512)]
        else:
            drawn = [k for k, _ in R.openpose_shapes(xs, ys, z, valid, False, 512, 512)[1]]
        assert drawn == [k for k, (a, b) in enumerate(limbs) if 5 not in (a, b)]


def test_humansd_draws_only_when_the_keypoints_sum_above_zero():
    """The reference's HumanSD drawer skips a skeleton whose keypoint array (x, y, confidence) sums to <= 0 or NaN."""
    pts = np.concatenate([np.random.default_rng(2).uniform(-0.3, 0.3, (17, 3)), np.ones((17, 1))], 1).astype(np.float32)
    mvp = np.diag([1.0, -1.0, 1.0, 1.0]).astype(np.float32)
    assert R.draw(pts, mvp, False, "humansd", 512, 512)[0].any()
    far = pts.copy()
    far[16, 0] = -3900.0  # one valid keypoint about 10^6 px left of the image
    nan = pts.copy()
    nan[2, 1] = np.nan
    for p in (far, nan):
        xs, ys, z, valid = R.keypoints(p, mvp, 512, 512)
        assert not R.humansd_shapes(xs, ys, z, valid, False, 512, 512)
        assert R.openpose_shapes(np.append(xs, 0), np.append(ys, 0), np.append(z, 0), np.append(valid, False), False, 512, 512)[1]


def test_pose_maps_checks_arguments_without_a_gpu():
    """CPU tensors are refused (there is no CPU path), as are a bad style, K, shape or size, before anything is launched."""
    from humangaussian_b200.pose import pose_maps
    kp, mvp, occ = torch.zeros(17, 3), torch.eye(4)[None], torch.zeros(1, dtype=torch.bool)
    with pytest.raises(RuntimeError, match="CUDA device"):
        pose_maps(kp, mvp, occ)
    with pytest.raises(ValueError, match="style"):
        pose_maps(kp, mvp, occ, style="coco")
    with pytest.raises(ValueError, match="tensor"):
        pose_maps(kp.numpy(), mvp, occ)
