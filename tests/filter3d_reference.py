"""Reference of the 3D smoothing filter (TEST INFRASTRUCTURE ONLY), built on the CPU oracle and tests/aa_reference.py
without changing either.

The filter (DESIGN.md section 2) acts once per Gaussian, before everything the oracle computes: the activated scales s
become s' = sqrt(s^2 + v) and the opacity o becomes o' = o * coef, coef = sqrt(prod_i s_i^2 / (s_i^2 + v)).  So:

  * `sampling_rate` / `finalize`: the per-Gaussian maximal sampling rate in numpy float32 with F1's operation order
    (fused multiply-adds emulated exactly by aa_reference.fma32), and the variance c / nu^2 from it.
  * `filter_params`: s' and o' by the IEEE float32 sequence the kernels use, bit for bit.  The oracle (or AAOracle with
    the screen-space filter on) then renders with them as its post-activation inputs, so `Filter3DOracle`'s forward is
    F1-with-filter bit for bit.
  * `Filter3DOracle.backward`: the oracle's gradients w.r.t. (s', o') chained to (s, o) by the hand-derived float64 rule
        dL/do = coef g_o',   dL/ds_i = g_s'_i s_i / s'_i + o g_o' sqrt(r_j r_k) v / (t_i s'_i)
    (and on to raw parameters through exp and sigmoid when asked).
  * `dense_render_f3d`: oracle/dense_ref.py's dense float64 formulation (or aa_reference.dense_render_aa) fed with s' and
    o' written as torch float64 expressions of (s, o, v) -- o' = o * prod_i s_i / sqrt(s_i^2 + v) -- and differentiated by
    torch.autograd.  It shares no code with the hand-derived chain.
"""
from __future__ import annotations

import numpy as np
import torch

from aa_reference import fma32

_f = np.float32
NEAR_Z = _f(0.2)
MARGIN = _f(0.65)
VARIANCE_SCALE = 0.2  # Mip-Splatting's c


def _affine(m0, m1, m2, m3, x, y, z):
    return fma32(m2, z, fma32(m1, y, m0 * x)) + m3


def sampling_rate(means3D, viewmatrices, tanfovx, tanfovy, H, W, max_rate=None):
    """float32 [P]: max over the cameras that see each Gaussian of max(fx, fy) / tz, folded into max_rate (0 if None).
    viewmatrices [V,4,4] or [V,16] (row-vector convention), tanfovx / tanfovy sequences of V floats."""
    m = np.asarray(means3D, _f)
    px, py, pz = m[:, 0], m[:, 1], m[:, 2]
    rate = np.zeros(len(m), _f) if max_rate is None else np.asarray(max_rate, _f).copy()
    vms = np.asarray(viewmatrices, _f).reshape(-1, 16)
    limx, limy = MARGIN * _f(W), MARGIN * _f(H)
    with np.errstate(all="ignore"):
        for v, Vm in enumerate(vms):
            tx = _affine(Vm[0], Vm[4], Vm[8], Vm[12], px, py, pz)
            ty = _affine(Vm[1], Vm[5], Vm[9], Vm[13], px, py, pz)
            tz = _affine(Vm[2], Vm[6], Vm[10], Vm[14], px, py, pz)
            tanx, tany = _f(tanfovx[v]), _f(tanfovy[v])
            fx, fy = _f(W) / (_f(2) * tanx), _f(H) / (_f(2) * tany)
            inside = (tz > NEAR_Z) & (np.abs((tx / tz) * fx) <= limx) & (np.abs((ty / tz) * fy) <= limy)
            nu = np.maximum(fx, fy) / tz
            rate = np.where(inside, np.maximum(rate, nu), rate).astype(_f)
    return rate


def finalize(rate, variance_scale=VARIANCE_SCALE):
    """float32 [P] variances: unseen Gaussians (rate 0) take the smallest positive rate (the widest filter); no Gaussian
    seen anywhere gives zeros; otherwise c / (nu * nu)."""
    rate = np.asarray(rate, _f)
    pos = rate > 0
    if not pos.any():
        return np.zeros_like(rate)
    nu = np.where(pos, rate, rate[pos].min()).astype(_f)
    return (_f(variance_scale) / (nu * nu)).astype(_f)


def filter_params(scales, opacities, var):
    """(s' [P,3], o' like opacities, dict of t, r, coef): the kernels' IEEE float32 sequence, bit for bit"""
    s = np.asarray(scales, _f)
    v = np.asarray(var, _f).reshape(-1, 1)
    with np.errstate(all="ignore"):
        s2 = s * s
        t = s2 + v
        r = np.where(t > 0, s2 / t, _f(1)).astype(_f)
        sp = np.sqrt(t).astype(_f)
        coef = np.sqrt((r[:, 0] * r[:, 1]) * r[:, 2]).astype(_f)
    o = np.asarray(opacities, _f)
    op = (o.reshape(-1) * coef).astype(_f).reshape(o.shape)
    return sp, op, dict(t=t, r=r, coef=coef)


def chain(g_sp, g_op, scales, opacities, var):
    """Hand-derived float64 chain of dL/d(s', o') to dL/d(s, o); s, o the activated parameters.  Finite at s_i = 0."""
    s = np.asarray(scales, np.float64)
    o = np.asarray(opacities, np.float64).reshape(-1)
    v = np.asarray(var, np.float64).reshape(-1, 1)
    g_sp = np.asarray(g_sp, np.float64).reshape(s.shape)
    g_op = np.asarray(g_op, np.float64).reshape(-1)
    t = s * s + v
    sp = np.sqrt(t)
    with np.errstate(all="ignore"):
        r = np.where(t > 0, s * s / t, 1.0)
        ratio = np.where(t > 0, s / sp, 1.0)
        coef = np.sqrt(r[:, 0] * r[:, 1] * r[:, 2])
        q = np.stack([np.sqrt(r[:, (k + 1) % 3] * r[:, (k + 2) % 3]) for k in range(3)], 1) * v / (t * sp)
    q = np.where(v > 0, q, 0.0)
    ds = g_sp * ratio + (o * g_op)[:, None] * q
    return ds, coef * g_op


class Filter3DOracle:
    """The oracle with the 3D filter (and optionally the screen-space filter) on: forward() / state() / backward().
    Inputs are post-activation; backward() returns gradients w.r.t. them (and, with raw=dict of the raw arrays the
    activations came from, w.r.t. those: exp's and sigmoid's Jacobians in float64)."""

    def __init__(self, threads: int = 0):
        from aa_reference import AAOracle
        self.o = AAOracle(threads=threads)

    def forward(self, *, filter_3d, antialiasing=False, **inp):
        self.inp, self.var = inp, np.asarray(filter_3d, _f)
        sp, op, self.f = filter_params(inp["scales"], inp["opacities"], self.var)
        self.filtered = dict(inp, scales=sp, opacities=op)
        return self.o.forward(antialiasing=antialiasing, **self.filtered)

    def state(self):
        return self.o.state()

    def backward(self, dL_dcolor, dL_ddepth, dL_dalpha, sums_err_const=None, raw=None):
        g = self.o.backward(dL_dcolor, dL_ddepth, dL_dalpha, sums_err_const=sums_err_const)
        g["dL_dsp"], g["dL_dop"] = g["scales"].copy(), g["opacities"].copy()
        ds, do = chain(g["scales"], g["opacities"], self.inp["scales"], self.inp["opacities"], self.var)
        if raw is not None:
            if "scales" in raw:
                ds = ds * np.exp(np.asarray(raw["scales"], np.float64))
            if "opacities" in raw:
                sg = 1.0 / (1.0 + np.exp(-np.asarray(raw["opacities"], np.float64).reshape(-1)))
                do = do * sg * (1.0 - sg)
        g["scales"] = ds.astype(np.float32).reshape(g["scales"].shape)
        g["opacities"] = do.astype(np.float32).reshape(g["opacities"].shape)
        return g


def filtered_tensors(scales, opacities, var):
    """(s', o') as torch float64 expressions of (s, o, v) for autograd: o' = o * prod_i s_i / sqrt(s_i^2 + v)"""
    v = torch.as_tensor(var, dtype=torch.float64).reshape(-1, 1)
    t = scales * scales + v
    sp = torch.sqrt(t)
    op = opacities.reshape(-1) * torch.prod(scales / sp, 1)
    return sp, op.reshape(opacities.shape)


def dense_render_f3d(*, opacities, scales, filter_3d, antialiasing=False, **kw):
    """oracle.dense_ref.dense_render (or aa_reference.dense_render_aa) with the filtered scales and opacities"""
    sp, op = filtered_tensors(scales, opacities, filter_3d)
    if antialiasing:
        from aa_reference import dense_render_aa
        return dense_render_aa(opacities=op, scales=sp, **kw)
    from oracle.dense_ref import dense_render
    kw = {k: v for k, v in kw.items()}
    return dense_render(opacities=op, scales=sp, **kw)
