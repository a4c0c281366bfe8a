"""CPU reference of a multi-view step on RAW parameters (TEST INFRASTRUCTURE ONLY): what bench.py's timed step,
rasterize_views_packed(raw=True) over a batch of views, must return.

  * activate(): the raw packed fields turned into the activated inputs the oracle takes, each value the bits F1 computes
    when `device` is the GPU F1 runs on -- scales torch.exp (expf), opacities 1 / (1 + expf(-x)) in float32, quaternions
    normal_reference.activate (gs_normalize4's order).  xyz and SH pass through.
  * iter_views() / views_reference(): Oracle.forward + Oracle.backward (sums_err_const = SUMS_K) once per view, keeping the
    images, radii, num_rendered, the float64 backward-blend sums with their error scales, and the activated-parameter
    gradients of each view.
  * StepSum: the per-view activated gradients summed in float64, then the activation Jacobians applied to the sum in
    float64 in the order B3 applies them (scales x s, opacity x o (1 - o), rotations (I - q^ q^T) / |q|, xyz and SH
    identity), with a per-row tolerance derived from FULL_SIZE's single-view bound:

      A single view v meets FULL_SIZE: each row within tau_v = 1e-5 + 1e-4 * max|o_v| of the oracle's row o_v (none over
      4 tau_v, at most 1e-4 of the rows over tau_v).  B2+B3 add the V per-view terms of a Gaussian in float32, in view
      order, so by the triangle inequality the activated-space sum is within
          T = sum_v tau_v + (V + 8) u sum_v max|o_v|,   u = 2^-24,
      of the float64 sum of the o_v: V u for the float32 additions, 8 u for B3's final multiplications (the rotation
      projection forms dq - q^ (q^ . dq), whose rounding is relative to |dq|, not to the result).  A view in which the
      Gaussian is culled (radius 0, equal on both sides) adds an exact zero on both sides and contributes nothing to T.
      T is then mapped through the Jacobian applied after the sum: x s_k for scales, x o (1 - o) for opacity, x 2 / |q| for
      rotations (1 / |q| is the projection's operator norm in the 2-norm; four components each within T are within 2 T in
      the 2-norm), x 1 for xyz and SH.
    The criterion by analogy with FULL_SIZE: every row within 4 T, at most 1e-4 of the rows over T.
  * bench_args() / bench_scene() / bench_cameras() / bench_shard(): the benchmark's own workload objects, built without a GPU."""
from __future__ import annotations

import math
import sys

import numpy as np
import torch

import normal_reference as NR
from util import ROOT

U = 2.0 ** -24
SUMS_K = 4.0  # test_gpu_parity.SUMS_K: the per-term constant of the oracle's error scale E_k
# packed-buffer field order (rasterizer.packed_layout) and the oracle's name for each
FIELDS = ("xyz", "scales", "rotations", "opacities", "shs")
ORACLE_KEYS = dict(xyz="means3D", scales="scales", rotations="rotations", opacities="opacities", shs="shs")
f32 = np.float32


def activate(raw, device="cpu"):
    """raw: dict of (some of) FIELDS -> float32 arrays ([P,3], [P,3], [P,4], [P,1], [P,K,3]; scales and rotations go
    together).  Returns the oracle's activated inputs for the fields present (means3D, scales, rotations, opacities, shs).
    The exponentials are evaluated by torch on `device`: on the GPU they are F1's expf bit for bit, so the oracle sees the
    kernels' activated values exactly."""
    out = {}
    if "xyz" in raw:
        out["means3D"] = np.asarray(raw["xyz"], f32)
    if "opacities" in raw:
        e = torch.exp(-torch.tensor(np.asarray(raw["opacities"], f32), device=device)).cpu().numpy()
        out["opacities"] = (f32(1) / (f32(1) + e)).astype(f32)
    if "scales" in raw:
        out["scales"] = torch.exp(torch.tensor(np.asarray(raw["scales"], f32), device=device)).cpu().numpy()
        out["rotations"] = NR.activate(raw["scales"], raw["rotations"], raw=True)[1]
    if "shs" in raw:
        out["shs"] = np.asarray(raw["shs"], f32)
    return out


def raw_of_params(p):
    """raw FIELDS of a GaussianParams (float32 numpy), in the packed buffer's order and shapes"""
    with torch.no_grad():
        t = (p.xyz, p.scaling, p.rotation, p.opacity, p.get_features)
        return {k: np.ascontiguousarray(x.detach().cpu().float().numpy()) for k, x in zip(FIELDS, t)}


def cam_inputs(cam):
    """the oracle's camera arguments, from the same tensors renderer.stack_cameras stacks for the kernels"""
    return dict(viewmatrix=cam.world_view_transform.cpu().float().numpy(), projmatrix=cam.full_proj_transform.cpu().float().numpy(),
                campos=cam.camera_center.cpu().float().numpy(), tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5))


def iter_views(act, cams, gws, sh_degree, H, W, bg=None, threads=0):
    """Per view v: the oracle's forward and backward of cams[v] under gws[v] = (gC [3,H,W], gD [1,H,W], gA [1,H,W]).
    Yields dict(color, radii, depth, alpha, num_rendered, rect, depths, sums, sums_err, screen_sums,
    grads = {oracle key: float32 array})."""
    from oracle.gs_oracle import Oracle
    o = Oracle(threads=threads)
    bg = np.zeros(3, f32) if bg is None else np.asarray(bg, f32)
    for v, cam in enumerate(cams):
        color, radii, depth, alpha = o.forward(**act, **cam_inputs(cam), bg=bg, image_height=H, image_width=W, sh_degree=sh_degree)
        st = o.state()
        gC, gD, gA = gws[v]
        g = o.backward(gC, gD, gA, sums_err_const=SUMS_K)
        yield dict(color=color, radii=radii, depth=depth, alpha=alpha, num_rendered=st["num_rendered"], rect=st["rect"],
                   depths=st["depths"], sums=g["sums"], sums_err=g["sums_err"], screen_sums=g["screen_sums"],
                   grads={k: g[k] for k in ORACLE_KEYS.values()})


def views_reference(act, cams, gws, sh_degree, H, W, bg=None, threads=0):
    """iter_views as a list (small scenes; at the benchmark's size the caller consumes the views one at a time)"""
    return list(iter_views(act, cams, gws, sh_degree, H, W, bg, threads))


def jacobian_factors(act, raw):
    """float64 factors of the activation Jacobians: s [P,3], o (1 - o) [P,1], q^ [P,4] and |q| [P,1]"""
    s = act["scales"].astype(np.float64)
    o = act["opacities"].astype(np.float64).reshape(-1, 1)
    q = act["rotations"].astype(np.float64)
    qn = np.maximum(np.linalg.norm(np.asarray(raw["rotations"], np.float64), axis=1, keepdims=True), 1e-12)
    return s, o * (1.0 - o), q, qn


def chain(gsum, act, raw):
    """activated-space gradients (float64, keyed by FIELDS) -> raw-parameter gradients, in B3's order"""
    s, do, q, qn = jacobian_factors(act, raw)
    out = dict(gsum)
    out["scales"] = gsum["scales"] * s
    out["opacities"] = gsum["opacities"].reshape(-1, 1) * do
    g = gsum["rotations"]
    out["rotations"] = (g - q * (q * g).sum(1, keepdims=True)) / qn
    return out


class StepSum:
    """Consumes the views of iter_views: the float64 sum of their activated gradients and the tolerance terms of T."""

    def __init__(self, P):
        self.P, self.V = P, 0
        self.sum = {}
        self.tau = {k: np.zeros(P) for k in FIELDS}   # sum_v tau_v over the views that see the Gaussian
        self.mag = {k: np.zeros(P) for k in FIELDS}   # sum_v max|o_v row|

    def add(self, view):
        vis = view["radii"] > 0
        for k in FIELDS:
            g = view["grads"][ORACLE_KEYS[k]].astype(np.float64).reshape(self.P, -1)
            self.sum[k] = g if k not in self.sum else self.sum[k] + g
            m = np.abs(g).max(1)
            self.tau[k] += np.where(vis, 1e-5 + 1e-4 * m, 0.0)
            self.mag[k] += m
        self.V += 1

    def result(self, act, raw):
        """(reference raw gradients, bounds T per element), both float64 dicts keyed by FIELDS with [P, n] arrays"""
        ref = chain(self.sum, act, raw)
        s, do, _, qn = jacobian_factors(act, raw)
        T = {k: (self.tau[k] + (self.V + 8) * U * self.mag[k])[:, None] for k in FIELDS}
        J = dict(xyz=1.0, scales=s, rotations=2.0 / qn, opacities=do, shs=1.0)
        return ({k: ref[k].reshape(self.P, -1) for k in FIELDS},
                {k: np.broadcast_to(T[k] * J[k], ref[k].reshape(self.P, -1).shape) for k in FIELDS})


def check_step_grads(got, ref, bound, max_frac=1e-4, cap=4.0):
    """got: {field: [P, n]} of one step; every row within cap * bound, at most max_frac of the rows over the bound.
    Returns ({field: (worst ratio, rows over the bound)}, failure message or None)."""
    stats, bad = {}, []
    for k in FIELDS:
        g = np.asarray(got[k], np.float64).reshape(ref[k].shape)
        err = np.abs(g - ref[k])
        b = bound[k]
        ratio = np.where(err == 0, 0.0, err / np.where(b > 0, b, 1e-300)).max(1)
        over = int((ratio > 1.0).sum())
        stats[k] = (float(ratio.max(initial=0.0)), over)
        if ratio.max(initial=0.0) > cap or over > max_frac * len(ratio):
            i = int(np.argmax(ratio))
            bad.append(f"{k}: worst row {i} at {ratio[i]:.3g}x its bound (gpu {g[i]} ref {ref[k][i]}), {over} rows over the bound")
    return stats, ("; ".join(bad) or None)


# ---- the benchmark's workload, without a GPU ------------------------------------------------------------------------------
def _bench():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import bench
    return bench


def bench_args(*extra):
    """bench.py's default workload, as its own argument parser builds it"""
    bench = _bench()
    saved = sys.argv
    sys.argv = ["bench.py", "--gpus", "1", *extra]
    try:
        return bench.parse()
    finally:
        sys.argv = saved


def bench_scene(args):
    """the RAW GaussianParams bench.Harness packs (CPU tensors)"""
    return _bench().load_scene(args)


def bench_cameras(args):
    from humangaussian_b200.cameras import sample_orbit_cameras
    return sample_orbit_cameras(args.views, args.res, args.res, seed=1000, device="cpu")


def bench_shard(args, cams, rank=0, world=1):
    """the views of the batch that rank `rank` renders, in run_b200's order"""
    from humangaussian_b200.dist import shard_views, view_cost_proxy
    return shard_views(args.views, rank, world, "balanced", [view_cost_proxy(c) for c in cams])
