"""The specification of pose maps (humangaussian_b200/pose.py): a numpy / integer-Python restatement of what the
reference's `Skeleton.humansd_draw` and `Skeleton.draw` produce with cv2, byte for byte.

cv2's drawing is exact integer arithmetic (with a few double-precision steps).  Each rule below is stated from what cv2
draws, as a closed form per row or per pixel, and pinned against cv2 by tests:
  * clipping: both ends beyond one border drop the segment; otherwise ends are slid along it onto the top / bottom
    border, then onto the left / right one, with truncated double offsets (`clip_line`);
  * thick lines (cv2.line, LINE_8, thickness T >= 2): the segment clipped to the image widened by T, the 16.16
    rectangle of half-width ceil(T / 2) around it filled as a convex polygon, and a disc of radius (T + 1) // 2 on each
    clipped end;
  * filled circles (cv2.circle, thickness -1): the integer disc dx^2 + dy^2 <= r^2;
  * ellipse2Poly(centre, (a, b), angle, 0, 360, 1): a float32 integer-degree sine table, double arithmetic, round half to
    even, consecutive duplicates removed;
  * fillConvexPoly: the outline (fixed-point or 8-connected integer lines, clipped), and per row one run between the
    left and right sides, each side's x stepping from its edge's start vertex by a rounded 16.16 slope, from the top
    vertex's row to the row above the bottom vertex's;
  * addWeighted(a, 0.4, b, 0.6, 0) on u8: rint(a * 0.4f + b * 0.6f).
tests/test_pose_cpu.py pins each rule against cv2 itself (when it is importable) and the whole draw against the
reference's own images (tests/golden/ref_pose.npz).

A shape is returned as a list of row runs (y, x0, x1) inside the image; `runs_per_row` counts how many disjoint runs a
shape has on each row (the GPU stores up to 4 per shape and row).
"""
from __future__ import annotations

import math

import numpy as np

from humangaussian_b200 import pose as P

XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT
COORD_LIMIT = float(1 << 20)  # |keypoint| >= 2^20 px is invalid (pose.py)
SIN_TABLE = np.array([round(math.sin(math.radians(i)), 7) for i in range(451)], dtype=np.float32)


def _trunc_div(a: int, b: int) -> int:
    """a / b rounded toward zero."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def clip_line(w, h, x1, y1, x2, y2):
    """The part of a segment inside [0, w - 1] x [0, h - 1] (any fixed point), as cv2 keeps it: (inside, x1, y1, x2, y2).

    A segment with both ends beyond the same border is dropped.  Otherwise each end beyond the top or bottom border is
    slid along the segment onto that border (the first end, then the second along the line through the moved first
    end), the offset along the other axis being trunc(double(border - y) * double(dx) / double(dy)); if the ends are
    then beyond the same left or right border the segment is dropped, else the ends beyond one are slid onto it the same
    way.  The order and the truncation decide single pixels, and tests/test_pose_cpu.py pins them against cv2."""
    lim = (w - 1, h - 1)
    p, q = [x1, y1], [x2, y2]

    def side(pt, a):
        return -1 if pt[a] < 0 else (1 if pt[a] > lim[a] else 0)
    for a in (1, 0):  # onto the top / bottom border first, then onto the left / right one
        if any(side(p, b) == side(q, b) != 0 for b in (0, 1)):
            return False, x1, y1, x2, y2
        o = 1 - a
        for e in (p, q):
            s = side(e, a)
            if s:
                border = 0 if s < 0 else lim[a]
                e[o] += int(float(border - e[a]) * float(q[o] - p[o]) / float(q[a] - p[a]))
                e[a] = border
    return True, p[0], p[1], q[0], q[1]


def _runs(xs, ys, W, H):
    """Pixels (x, y) -> row runs, keeping those inside the image."""
    xs, ys = np.asarray(xs, np.int64), np.asarray(ys, np.int64)
    keep = (xs >= 0) & (xs < W) & (ys >= 0) & (ys < H)
    return [(int(y), int(x), int(x)) for x, y in zip(xs[keep], ys[keep])]


def line_fixed(p0, p1, W, H):
    """A fixed-point (16.16) polygon edge: clipped to the image first, walked along its major axis in increasing order
    from the rounded start for floor(|major extent|) + 1 pixels, the minor coordinate stepped by a truncated 16.16 slope
    from the unrounded start, plus the rounded end point."""
    ok, x1, y1, x2, y2 = clip_line(W << XY_SHIFT, H << XY_SHIFT, p0[0], p0[1], p1[0], p1[1])
    if not ok:
        return []
    half = XY_ONE >> 1
    if abs(x2 - x1) > abs(y2 - y1):
        if x2 < x1:
            x1, y1, x2, y2 = x2, y2, x1, y1
        step = _trunc_div((y2 - y1) << XY_SHIFT, (x2 - x1) | 1)
        k = np.arange(((x2 - x1) >> XY_SHIFT) + 1, dtype=np.int64)
        xs, ys = ((x1 + half) >> XY_SHIFT) + k, (y1 + half + step * k) >> XY_SHIFT
    else:
        if y2 < y1:
            x1, y1, x2, y2 = x2, y2, x1, y1
        step = _trunc_div((x2 - x1) << XY_SHIFT, (y2 - y1) | 1)
        k = np.arange(((y2 - y1) >> XY_SHIFT) + 1, dtype=np.int64)
        xs, ys = (x1 + half + step * k) >> XY_SHIFT, ((y1 + half) >> XY_SHIFT) + k
    xs = np.append(xs, (x2 + half) >> XY_SHIFT)
    ys = np.append(ys, (y2 + half) >> XY_SHIFT)
    return _runs(xs, ys, W, H)


def line_int(p0, p1, W, H):
    """An 8-connected integer line (a polygon edge of fillConvexPoly at shift 0): clipped to the image when an end lies
    outside it, then walked left to right."""
    x1, y1, x2, y2 = p0[0], p0[1], p1[0], p1[1]
    if not (0 <= x1 < W and 0 <= x2 < W and 0 <= y1 < H and 0 <= y2 < H):
        ok, x1, y1, x2, y2 = clip_line(W, H, x1, y1, x2, y2)
        if not ok:
            return []
    if x2 < x1:
        x1, y1, x2, y2 = x2, y2, x1, y1
    dx, dy = x2 - x1, y2 - y1
    sy = -1 if dy < 0 else 1
    dy = abs(dy)
    if dy > dx:  # walk y, step x
        k = np.arange(dy + 1, dtype=np.int64)
        m = (2 * dx * k + dy - 1) // (2 * dy)  # minor steps after k major steps of the Bresenham walk (err = dy - 2 dx)
        return _runs(x1 + m, y1 + sy * k, W, H)
    k = np.arange(dx + 1, dtype=np.int64)
    m = (2 * dy * k + dx - 1) // (2 * dx) if dx else k * 0
    return _runs(x1 + k, y1 + sy * m, W, H)


def _edge_lines(v, shift, W, H):
    """The outline fillConvexPoly draws: every edge of the closed polygon, as a fixed-point line (shift 16) or an
    8-connected integer line (shift 0)."""
    runs = []
    for i in range(len(v)):
        a, b = v[i - 1], v[i]
        if shift == 0:
            runs += line_int(a, b, W, H)
        else:
            runs += line_fixed((a[0] << (XY_SHIFT - shift), a[1] << (XY_SHIFT - shift)),
                               (b[0] << (XY_SHIFT - shift), b[1] << (XY_SHIFT - shift)), W, H)
    return runs


def _chain(xs, rows, top, step, y_start):
    """One side of the scanline fill: the edges met walking from the top vertex in direction `step`, each as
    (first row, end row, x at its first row in 16.16, x step per row in 16.16).  An edge that does not end below the
    row the walk has reached is passed over (its end becomes the next start).  The x step is the edge's 16.16 run over
    its row count, plus one half, truncated toward zero; x at a row is the start vertex's x plus whole steps, with no
    correction for where the vertex lies inside its first row."""
    n, out = len(rows), []
    s, y = top, y_start
    for _ in range(n):
        j = (s + step) % n
        if rows[j] > y:
            L = rows[j] - y
            out.append((y, rows[j], xs[s], _trunc_div((xs[j] - xs[s]) * 2 + L, 2 * L)))
            y = rows[j]
        s = j
    return out


def fill_convex(v, shift, W, H):
    """fillConvexPoly's pixels for a convex polygon v [(x, y)] in `shift` fixed point: its outline, and one run per row
    between the left and right edges, from the top vertex's row down to the row above the bottom vertex's."""
    runs = _edge_lines(v, shift, W, H)
    n = len(v)
    half = (1 << shift) >> 1
    px = [(x + half) >> shift for x, _ in v]
    rows = [(y + half) >> shift for _, y in v]
    if n < 3 or max(px) < 0 or max(rows) < 0 or min(px) >= W or min(rows) >= H:
        return runs
    top = rows.index(min(rows))
    xs = [x << (XY_SHIFT - shift) for x, _ in v]
    sides = [_chain(xs, rows, top, 1, rows[top]), _chain(xs, rows, top, n - 1, rows[top])]
    ptr = [0, 0]
    H_HALF = XY_ONE >> 1
    for y in range(max(rows[top], 0), min(max(rows), H)):
        x = []
        for k in range(2):
            while sides[k][ptr[k]][1] <= y:
                ptr[k] += 1
            r0, _, x0, dx = sides[k][ptr[k]]
            x.append(x0 + dx * (y - r0))
        lo, hi = (min(x) + H_HALF) >> XY_SHIFT, (max(x) + H_HALF) >> XY_SHIFT
        lo, hi = max(lo, 0), min(hi, W - 1)
        if lo <= hi:
            runs.append((y, lo, hi))
    return runs


def circle_filled(cx, cy, r, W, H):
    """cv2.circle(img, (cx, cy), r, colour, -1): the integer disc, dx^2 + dy^2 <= r^2, clipped."""
    runs = []
    for d in range(-r, r + 1):
        hw = math.isqrt(r * r - d * d)
        y, x0, x1 = cy + d, max(cx - hw, 0), min(cx + hw, W - 1)
        if 0 <= y < H and x0 <= x1:
            runs.append((y, x0, x1))
    return runs


def thick_line(x0, y0, x1, y1, T, W, H):
    """cv2.line(img, (x0, y0), (x1, y1), colour, T) with LINE_8 and T >= 2: the segment is first clipped to the image
    widened by T on every side; then, unless its ends coincide, the rectangle around it of half-width ceil(T / 2) is
    filled, its corners the ends offset by (rint(dy * h / |d|), rint(dx * h / |d|)) in 16.16 (h the half-width in 16.16,
    d = (x0 - x1, y1 - y0), the quotient h / |d| taken first, round half to even); and a disc of radius (T + 1) // 2
    covers each clipped end."""
    ok, x0, y0, x1, y1 = clip_line(W + 2 * T, H + 2 * T, x0 + T, y0 + T, x1 + T, y1 + T)
    if not ok:
        return []
    x0, y0, x1, y1 = x0 - T, y0 - T, x1 - T, y1 - T
    runs = []
    if (x0, y0) != (x1, y1):
        dx, dy = float(x0 - x1), float(y1 - y0)
        f = float(((T + 1) // 2) << XY_SHIFT) / math.sqrt(dx * dx + dy * dy)
        ox, oy = round(dy * f), round(dx * f)  # Python's round is half to even
        a, b = (x0 << XY_SHIFT, y0 << XY_SHIFT), (x1 << XY_SHIFT, y1 << XY_SHIFT)
        quad = [(a[0] + ox, a[1] + oy), (a[0] - ox, a[1] - oy), (b[0] - ox, b[1] - oy), (b[0] + ox, b[1] + oy)]
        runs += fill_convex(quad, XY_SHIFT, W, H)
    rc = (T + 1) // 2
    runs += circle_filled(x0, y0, rc, W, H) + circle_filled(x1, y1, rc, W, H)
    return runs


def ellipse2poly(cx, cy, a, b, angle):
    """cv2.ellipse2Poly((cx, cy), (a, b), angle, 0, 360, 1) for integer arguments: [(x, y)]."""
    while angle < 0:
        angle += 360
    while angle > 360:
        angle -= 360
    alpha, beta = np.float64(SIN_TABLE[450 - angle]), np.float64(SIN_TABLE[angle])
    i = np.arange(361)
    x = np.float64(a) * SIN_TABLE[450 - i].astype(np.float64)
    y = np.float64(b) * SIN_TABLE[i].astype(np.float64)
    px = np.rint((np.float64(cx) + x * alpha) - y * beta).astype(np.int64)
    py = np.rint((np.float64(cy) + x * beta) + y * alpha).astype(np.int64)
    keep = np.ones(361, bool)
    keep[1:] = (px[1:] != px[:-1]) | (py[1:] != py[:-1])
    pts = list(zip(px[keep].tolist(), py[keep].tolist()))
    if len(pts) == 1:
        pts = [(cx, cy), (cx, cy)]
    return pts


def add_weighted(a, b):
    """cv2.addWeighted(a, 0.4, b, 0.6, 0) on u8 arrays."""
    s = a.astype(np.float32) * np.float32(0.4) + b.astype(np.float32) * np.float32(0.6)
    return np.clip(np.rint(s), 0, 255).astype(np.uint8)


def runs_mask(runs, W, H):
    m = np.zeros((H, W), dtype=bool)
    for y, x0, x1 in runs:
        m[y, x0:x1 + 1] = True
    return m


# ---- the draw --------------------------------------------------------------------------------------------------------
def project(points, mvp):
    """points [K,4] float32 @ mvp^T in the GPU's order ((p0 m0 + p1 m1) + p2 m2) + p3 m3, each op rounded to float32;
    returns ndc [K,3] float32 and the validity of w (> 0)."""
    p = np.asarray(points, np.float32)
    m = np.asarray(mvp, np.float32)
    out = np.zeros((len(p), 4), np.float32)
    for r in range(4):
        acc = p[:, 0] * m[r, 0]
        for c in range(1, 4):
            acc = (acc + p[:, c] * m[r, c]).astype(np.float32)
        out[:, r] = acc
    with np.errstate(divide="ignore", invalid="ignore"):
        ndc = out[:, :3] / out[:, 3:]
    return ndc, out[:, 3] > 0


def keypoints(points, mvp, H, W):
    """(xs, ys, z, valid): float32 pixel coordinates as the reference computes them from `project`, the NDC depth, and
    which keypoints are valid (w > 0, finite, |coordinate| < 2^20)."""
    ndc, wpos = project(points, mvp)
    xs = (ndc[:, 0] + np.float32(1)) / np.float32(2) * np.float32(H)
    ys = (ndc[:, 1] + np.float32(1)) / np.float32(2) * np.float32(W)
    with np.errstate(invalid="ignore"):
        valid = wpos & (np.abs(xs) < COORD_LIMIT) & (np.abs(ys) < COORD_LIMIT)
    return xs.astype(np.float32), ys.astype(np.float32), ndc[:, 2], valid


def _occlusion_humansd(z, xs, conf):
    if z[0] > z[3] and z[0] < z[4]:
        conf[4] = False
        if xs[2] > xs[1]:
            conf[2] = False
    elif z[0] < z[3] and z[0] > z[4]:
        conf[3] = False
        if xs[1] < xs[2]:
            conf[1] = False
    elif z[0] > z[3] and z[0] > z[4]:
        conf[0] = conf[1] = conf[2] = False


def _occlusion_openpose(z, xs, mask):
    if z[0] > z[-1] and z[0] < z[-2]:
        mask[-2] = False
        if xs[-4] > xs[-3]:
            mask[-4] = False
    elif z[0] < z[-1] and z[0] > z[-2]:
        mask[-1] = False
        if xs[-3] < xs[-4]:
            mask[-3] = False
    elif z[0] > z[-1] and z[0] > z[-2]:
        mask[0] = mask[-3] = mask[-4] = False


def thickness(H):
    return int(10 * H / 512)


def humansd_shapes(xs, ys, z, valid, occlusion, H, W):
    """[(limb, runs)] in draw order for the HumanSD style.  The reference draws a skeleton only when the sum of its
    keypoint array (every x, y and 0 / 1 confidence after occlusion) is > 0; here the sum is taken in double over the
    float32 values, so a NaN anywhere leaves the view blank as in the reference."""
    conf = np.ones(17, bool)
    if occlusion:
        _occlusion_humansd(z, xs, conf)
    with np.errstate(invalid="ignore", over="ignore"):
        total = np.sum(xs.astype(np.float64)) + np.sum(ys.astype(np.float64)) + float(conf.sum())
    if not total > 0:
        return []
    conf &= valid
    T = thickness(H)
    out = []
    for k, (a, b) in enumerate(P.HUMANSD_LIMBS):
        if conf[a] and conf[b]:
            xa, ya, xb, yb = int(xs[a]), int(ys[a]), int(xs[b]), int(ys[b])
            runs = thick_line(xa, ya, xb, yb, T, W, H)
            runs += circle_filled(xa, ya, T // 2, W, H) + circle_filled(xb, yb, T // 2, W, H)
            out.append((k, runs))
    return out


def openpose_limb_geometry(xa, ya, xb, yb):
    """(centre x, centre y, half length, angle) of an OpenPose limb, as the reference derives them (float32 mean and
    length, double atan2 in degrees), truncated."""
    X = np.array([xa, xb], np.float32)
    Y = np.array([ya, yb], np.float32)
    mX, mY = np.float32(X[0] + X[1]) / np.float32(2), np.float32(Y[0] + Y[1]) / np.float32(2)
    dY, dX = np.float32(Y[0] - Y[1]), np.float32(X[0] - X[1])
    length = np.sqrt(np.float32(dY * dY) + np.float32(dX * dX), dtype=np.float32)
    angle = math.degrees(math.atan2(float(dY), float(dX)))
    return int(mX), int(mY), int(np.float32(length) / np.float32(2)), int(angle)


def openpose_shapes(xs, ys, z, valid, occlusion, H, W):
    """([(keypoint, circle runs)], [(limb, ellipse runs)]) in draw order for the OpenPose style."""
    with np.errstate(invalid="ignore"):
        mask = (xs >= 0) & (xs < H) & (ys >= 0) & (ys < W)
    if occlusion:
        _occlusion_openpose(z, xs, mask)
    mask &= valid
    circles = [(i, circle_filled(int(xs[i]), int(ys[i]), 4, W, H)) for i in range(18) if mask[i]]
    limbs = []
    for k, (a, b) in enumerate(P.OPENPOSE_LIMBS):
        if mask[a] and mask[b]:
            cx, cy, ax, ang = openpose_limb_geometry(xs[a], ys[a], xs[b], ys[b])
            limbs.append((k, fill_convex(ellipse2poly(cx, cy, ax, 4, ang), 0, W, H)))
    return circles, limbs


def draw_from_keypoints(xs, ys, z, valid, occlusion, style, H, W):
    """The u8 [H, W, 3] pose image from float32 keypoints xs, ys, NDC depth z and validity."""
    img = np.zeros((H, W, 3), np.uint8)
    if style == "humansd":
        for k, runs in humansd_shapes(xs, ys, z, valid, occlusion, H, W):
            img[runs_mask(runs, W, H)] = P.HUMANSD_COLORS[P.HUMANSD_COLOR_INDEX[k]]
        return img
    circles, limbs = openpose_shapes(xs, ys, z, valid, occlusion, H, W)
    for i, runs in circles:
        img[runs_mask(runs, W, H)] = P.OPENPOSE_COLORS[i]
    for k, runs in limbs:
        m = runs_mask(runs, W, H)
        img[m] = add_weighted(img[m], np.broadcast_to(np.array(P.OPENPOSE_COLORS[k], np.uint8), img[m].shape))
    return img


def draw(points, mvp, occlusion, style, H, W):
    """(u8 image [H, W, 3], kp float32 [K, 2]) for one view: points [K, 4] (or [K, 3], w = 1 appended), mvp [4, 4]."""
    p = np.asarray(points, np.float32)
    if p.shape[1] == 3:
        p = np.concatenate([p, np.ones((len(p), 1), np.float32)], 1)
    xs, ys, z, valid = keypoints(p, mvp, H, W)
    return draw_from_keypoints(xs, ys, z, valid, bool(occlusion), style, H, W), np.stack([xs, ys], 1)


def runs_per_row(runs, W, H):
    """The number of disjoint pixel runs on each row of a shape (the GPU keeps up to 4 per shape and row)."""
    m = np.pad(runs_mask(runs, W, H).astype(np.int8), ((0, 0), (1, 0)))
    return (np.diff(m, axis=1) == 1).sum(1)
