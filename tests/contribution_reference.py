"""Reference of the contribution scores (TEST INFRASTRUCTURE ONLY): a numpy replay of the blend on the CPU oracle's state.

The replay restates the oracle's blend with the pinned float operation order (the same restatement as
tests/test_oracle_blend_state.py, which it reproduces bit for bit: n_contrib and contrib_patches) and adds, per (pixel,
sorted entry):
  touch = hit (power <= 0, alpha >= 1/255) while the pixel is live (not yet terminated, inside the image);
  blend = a touch whose test_T = T (1 - alpha) stays >= 1e-4; the other touch is the terminating hit;
  w     = float32(alpha * T_before), q(w) = rint(w * 2^24) (round half to even).
Per Gaussian it folds exact Python-integer sums of q and of touches, and the maximum of w's bits, over the view's pixels.
Antialiasing and the 3D filter come through tests/aa_reference.py / tests/filter3d_reference.py (the oracle renders their
filtered opacities / scales bit for bit)."""
from __future__ import annotations

import numpy as np

from util import ROOT  # noqa: F401  (puts the repository root on sys.path)

ALPHA_MIN, ALPHA_MAX, T_MIN = np.float32(1.0 / 255.0), np.float32(0.99), np.float32(1e-4)
f32 = np.float32


def _fma(a, b, c):
    """binary32 fma through double (exact product; one double rounding, then float)"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def _gs_exp(x):
    """gs_exp (gs_oracle.c): range reduction + degree-5 polynomial + exponent add"""
    x = np.maximum(np.asarray(x, f32), f32(-87.0))
    t = _fma(x, f32(float.fromhex("0x1.715476p+0")), f32(12582912.0))
    n = (t - f32(12582912.0)).astype(f32)
    r = _fma(n, f32(-float.fromhex("0x1.62e430p-1")), x)
    p = np.full_like(x, f32(float.fromhex("0x1.0fa834p-7")))
    for cst in ("0x1.573a54p-5", "0x1.555a6ap-3", "0x1.fffdc6p-2", "0x1.fffff6p-1", "0x1p+0"):
        p = _fma(p, r, f32(float.fromhex(cst)))
    return (p.view(np.uint32) + (t.view(np.uint32) << np.uint32(23))).view(f32)


def replay(st, H, W):
    """One view: the oracle state `st` (Oracle.state()) of an H x W image.  Returns a dict of per-Gaussian weight_sum (object
    array of Python ints, units 2^-24), weight_max (u32 bits), touches and blends (int64), and the per-view n_contrib,
    contrib_patches (the oracle's exports, recomputed) and the number of terminated pixels."""
    gx = (W + 15) // 16
    xy, co, pl = st["xy"], st["conic_opacity"], st["point_list"]
    P = len(xy)
    wsum = np.zeros(P, object)
    wsum[:] = 0
    wmax = np.zeros(P, np.uint32)
    touches = np.zeros(P, np.int64)
    blends = np.zeros(P, np.int64)
    patches = np.zeros(st["num_rendered"], np.uint8)
    n_contrib = np.zeros((H, W), np.uint32)
    terminated = 0
    for t, (r0, r1) in enumerate(st["ranges"]):
        if r1 <= r0:
            continue
        ys, xs = np.mgrid[(t // gx) * 16:(t // gx) * 16 + 16, (t % gx) * 16:(t % gx) * 16 + 16]
        keep = (ys < H) & (xs < W)
        ys, xs = ys[keep], xs[keep]
        fx, fy = xs.astype(f32), ys.astype(f32)
        pbit = (1 << (((ys % 16) // 4) * 2 + (xs % 16) // 8)).astype(np.uint8)
        T = np.ones(len(xs), f32)
        alive = np.ones(len(xs), bool)
        for j in range(r0, r1):
            if not alive.any():
                break
            g = pl[j]
            A, B, C, op = co[g]
            dx, dy = (xy[g, 0] - fx).astype(f32), (xy[g, 1] - fy).astype(f32)
            u = _fma(-B, dy, (f32(-0.5) * A * dx).astype(f32))
            w2 = ((f32(-0.5) * C * dy).astype(f32) * dy).astype(f32)
            power = _fma(dx, u, w2)
            alpha = np.minimum(ALPHA_MAX, (op * _gs_exp(np.minimum(power, f32(0)))).astype(f32))
            test_T = (T * (f32(1) - alpha)).astype(f32)
            touch = alive & (power <= 0) & (alpha >= ALPHA_MIN)
            term = touch & (test_T < T_MIN)
            blend = touch & ~term
            if touch.any():
                w = (alpha[blend] * T[blend]).astype(f32)
                touches[g] += int(touch.sum())
                terminated += int(term.sum())
                if blend.any():
                    blends[g] += int(blend.sum())
                    wsum[g] += int(np.rint(w.astype(np.float64) * 2.0 ** 24).astype(np.int64).sum())
                    wmax[g] = max(int(wmax[g]), int(w.view(np.uint32).max()))
                    patches[j] = np.bitwise_or.reduce(pbit[blend])
                    n_contrib[ys[blend], xs[blend]] = j - r0 + 1
            alive &= ~term
            T = np.where(blend, test_T, T)
    return dict(weight_sum=wsum, weight_max=wmax, touches=touches, blends=blends, n_contrib=n_contrib,
                contrib_patches=patches, terminated=terminated)


def _oracle_state(inp, antialiasing=False, filter_3d=None):
    if filter_3d is not None:
        from filter3d_reference import Filter3DOracle
        o = Filter3DOracle(threads=1)
        out = o.forward(filter_3d=filter_3d, antialiasing=antialiasing, **inp)
    else:
        from aa_reference import AAOracle
        o = AAOracle(threads=1)
        out = o.forward(antialiasing=antialiasing, **inp)
    return o, out, o.state()


def contribution(inps, antialiasing=False, filter_3d=None):
    """Folded over the views `inps` (oracle input dicts of one Gaussian set): dict of weight_sum (uint64), weight_max (uint32
    bits), touches and blends (int64) per Gaussian, plus the total terminated pixel count and per-view replays ("views")."""
    P = np.asarray(inps[0]["means3D"]).shape[0]
    acc = dict(weight_sum=np.zeros(P, object), weight_max=np.zeros(P, np.uint32), touches=np.zeros(P, np.int64),
               blends=np.zeros(P, np.int64), terminated=0, views=[])
    acc["weight_sum"][:] = 0
    for inp in inps:
        _, out, st = _oracle_state(inp, antialiasing, filter_3d)
        r = replay(st, inp["image_height"], inp["image_width"])
        r["state"], r["out"] = st, out
        acc["weight_sum"] += r["weight_sum"]
        acc["weight_max"] = np.maximum(acc["weight_max"], r["weight_max"])
        acc["touches"] += r["touches"]
        acc["blends"] += r["blends"]
        acc["terminated"] += r["terminated"]
        acc["views"].append(r)
    acc["weight_sum"] = np.array([int(x) for x in acc["weight_sum"]], np.uint64)
    return acc
