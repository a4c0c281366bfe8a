"""Densification / pruning on the device (SURVEY.md 8f-2) -- the step on the other side of backward.

Mirrors the reference's `GaussianModel` surgery (gaussiansplatting/scene/gaussian_model.py:268-437) and the
bookkeeping that feeds it (threestudio/systems/GaussianDreamer.py:378-408), with the same names and argument meaning:

    stats = DensifyStats.zeros(P, device)
    add_densification_stats(stats, dL_dmeans2D[V,P,3], radii[V,P])          # after every backward
    params, moments, stats = densify_and_prune(params, moments, stats, max_grad, min_opacity, extent, max_screen_size,
                                               percent_dense)               # every densify_prune_interval steps
    params, moments, stats = prune_only(params, moments, stats, min_opacity, size_thresh)
    params, moments, stats = prune_points(params, moments, stats, remove)  # any rule's bool [P] mask, e.g. contribution
    install_into_optimizer(optimizer, params, moments)                      # what cat_tensors_to_optimizer /
                                                                            # _prune_optimizer do to torch.optim.Adam

`params` is a dict of the RAW optimiser tensors by the reference's group names (xyz, f_dc, f_rest, opacity, scaling,
rotation); `moments` maps the same names to (exp_avg, exp_avg_sq) or is None.  Where the reference runs ~30 PyTorch ops
with a host sync per boolean-mask gather and concatenates every tensor twice, this plans all destinations with one
prefix-sum pass and moves each surviving row once (csrc/densify.cu); one host read-back (the five counts) per call.
`densify_and_prune_packed` / `prune_only_packed` run the same plan on the packed parameter buffer of an
`optim.PackedAdam`, moving every field of it and of its two moment buffers straight into new flat buffers.
There is no CPU path: tensors must live on a CUDA device.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

from .rasterizer import _check, _ptr, _stream, load_library

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
ROLE_COPY, ROLE_XYZ, ROLE_SCALING, ROLE_MOMENT = 0, 1, 2, 3


MODE_PRUNE_MASK = 2  # b200gs_prune_plan (not a b200gs_densify_cfg mode)


class _Cfg(C.Structure):  # == b200gs_densify_cfg
    _fields_ = [("mode", C.c_int32), ("n_split", C.c_int32), ("use_screen", C.c_int32), ("max_grad", C.c_float),
                ("min_opacity", C.c_float), ("percent_dense_x_extent", C.c_float), ("max_screen_size", C.c_float),
                ("big_ws_thresh", C.c_float)]


@dataclass
class DensifyStats:
    """xyz_gradient_accum [P,1], denom [P,1], max_radii2D [P] (gaussian_model.py:151-152, 358-360)."""
    xyz_gradient_accum: torch.Tensor
    denom: torch.Tensor
    max_radii2D: torch.Tensor

    @staticmethod
    def zeros(P: int, device) -> "DensifyStats":
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
        return DensifyStats(z(P, 1), z(P, 1), z(P))


def _need_cuda(t: torch.Tensor):
    if t.device.type != "cuda":
        raise RuntimeError("b200gs: tensors must live on a CUDA device (there is no CPU path)")


def add_densification_stats(stats: DensifyStats, viewspace_grads: torch.Tensor, radii: torch.Tensor,
                            update_mask: Optional[torch.Tensor] = None) -> None:
    """One optimiser step of bookkeeping for a batch of views, in place.
    viewspace_grads [V,P,3] (or [P,3]): the means2D gradients of the step's views; radii [V,P] (or [P]) int32.
    Equals GaussianDreamer.py:385-391: sum the view gradients, visibility = max radius > 0, max_radii2D update,
    then GaussianModel.add_densification_stats (gaussian_model.py:433-437).
    update_mask [P] bool/uint8 (optional) is ANDed with the visibility: the reference removes near-hand points from
    visibility_filter before this bookkeeping when disable_hand_densification is set (GaussianDreamer.py:288-297)."""
    L = load_library()
    g = viewspace_grads.detach()
    if g.dim() == 2:
        g = g[None]
    r = radii if radii.dim() == 2 else radii[None]
    _need_cuda(g)
    g = g.to(torch.float32).contiguous()
    r = r.to(device=g.device, dtype=torch.int32).contiguous()
    V, P = g.shape[0], g.shape[1]
    if r.shape != (V, P) or stats.max_radii2D.shape[0] != P:
        raise ValueError("b200gs: add_densification_stats shape mismatch")
    for t in (stats.xyz_gradient_accum, stats.denom, stats.max_radii2D):
        if not (t.is_contiguous() and t.dtype == torch.float32 and t.device == g.device):
            raise ValueError("b200gs: statistics must be contiguous fp32 tensors on the gradients' device")
    m = None
    if update_mask is not None:
        m = update_mask.to(device=g.device, dtype=torch.uint8).contiguous()
        if m.shape != (P,):
            raise ValueError("b200gs: update_mask must have shape [P]")
    with torch.cuda.device(g.device):
        _check(L.b200gs_densify_stats(P, V, _ptr(g), _ptr(r), _ptr(m), _ptr(stats.xyz_gradient_accum), _ptr(stats.denom),
                                      _ptr(stats.max_radii2D), _stream(g.device)), "densify_stats")


class _Surgery:
    """One planned densify / prune: the plan on the device, its five counts read back once (P_new sizes every
    destination), and the children's noise.  `move` realises the plan for one [P, ...] array into a [P_new, ...]
    destination, which may be a view into a larger buffer (the packed form moves each field into its place in the new
    flat buffer).  Callers run inside `torch.cuda.device(dev)`.  P >= 1."""

    def __init__(self, cfg: _Cfg, stats: DensifyStats, opacity, scaling, rotation, noise, generator, remove=None):
        L = self.L = load_library()
        dev, P = scaling.device, scaling.shape[0]
        self.cfg, self.dev, self.P, self.rotation, self.scaling = cfg, dev, P, rotation, scaling
        self.n_split = cfg.n_split if cfg.mode == 0 else 0
        self.plan = torch.empty(4, P, dtype=torch.int32, device=dev)
        counts = torch.empty(5, dtype=torch.int32, device=dev)
        scratch = torch.empty(L.b200gs_densify_scratch_bytes(P), dtype=torch.uint8, device=dev)
        self.st = _stream(dev)
        if cfg.mode == MODE_PRUNE_MASK:
            _check(L.b200gs_prune_plan(P, _ptr(remove), _ptr(self.plan), _ptr(counts), _ptr(scratch), scratch.numel(), self.st),
                   "prune_plan")
        else:
            _check(L.b200gs_densify_plan(P, C.byref(cfg), _ptr(stats.xyz_gradient_accum), _ptr(stats.denom), _ptr(opacity),
                                         _ptr(scaling), _ptr(self.plan), _ptr(counts), _ptr(scratch), scratch.numel(), self.st),
                   "densify_plan")
        self.counts = counts.cpu()  # the one host sync of the call
        n_keep, n_clone, S_sel, S_kept, P_new = (int(x) for x in self.counts)
        if cfg.mode == MODE_PRUNE_MASK and P_new == 0:
            raise ValueError("b200gs: the prune mask removes every Gaussian")
        self.P_new = P_new
        self.ch = (C.c_int32 * 5)(n_keep, n_clone, S_sel, S_kept, P_new)
        if cfg.mode == 0 and noise is None:
            # torch.normal(mean=0, std=stds) == randn * stds (gaussian_model.py:369-371)
            noise = torch.randn(self.n_split * S_sel, 3, dtype=torch.float32, device=dev, generator=generator)
        if noise is not None:
            noise = noise.to(device=dev, dtype=torch.float32).contiguous()
            if noise.numel() != self.n_split * S_sel * 3:
                raise ValueError(f"b200gs: noise must hold {self.n_split * S_sel} rows of 3 standard-normal draws")
        self.noise = noise

    def move(self, role, src: torch.Tensor, dst: torch.Tensor) -> torch.Tensor:
        rf = src.numel() // self.P
        if rf == 0:  # e.g. f_rest [P,0,3] at SH degree 0
            return dst
        _check(self.L.b200gs_densify_move(role, self.P, rf, _ptr(self.plan), self.ch, self.n_split, _ptr(src), _ptr(dst),
                                          _ptr(self.rotation), _ptr(self.scaling), _ptr(self.noise), self.st), "densify_move")
        return dst

    def new_stats(self, stats: DensifyStats) -> DensifyStats:
        if self.cfg.mode == 0:  # densification_postfix resets all three statistics (gaussian_model.py:358-360)
            return DensifyStats.zeros(self.P_new, self.dev)
        # prune_points gathers them (gaussian_model.py:310-315)
        out = lambda t: self.move(ROLE_COPY, t, torch.empty((self.P_new,) + tuple(t.shape[1:]), dtype=torch.float32, device=self.dev))
        return DensifyStats(out(stats.xyz_gradient_accum), out(stats.denom), out(stats.max_radii2D))


def _run(cfg: _Cfg, params: Dict[str, torch.Tensor], moments, stats: DensifyStats, noise, generator, remove=None):
    xyz = params["xyz"]
    _need_cuda(xyz)
    dev, P = xyz.device, xyz.shape[0]
    src = {k: params[k].detach().to(torch.float32).contiguous() for k in GROUPS}
    if P == 0:
        return ({k: v.clone() for k, v in src.items()}, None if moments is None else {k: (m.clone(), v.clone()) for k, (m, v) in moments.items()},
                DensifyStats.zeros(0, dev), torch.zeros(5, dtype=torch.int32))
    with torch.cuda.device(dev):
        s = _Surgery(cfg, stats, src["opacity"], src["scaling"], src["rotation"], noise, generator, remove)

        def move(role, t):
            return s.move(role, t, torch.empty((s.P_new,) + tuple(t.shape[1:]), dtype=torch.float32, device=dev))
        roles = {"xyz": ROLE_XYZ, "scaling": ROLE_SCALING}
        new_params = {k: move(roles.get(k, ROLE_COPY), src[k]) for k in GROUPS}
        new_moments = None
        if moments is not None:
            new_moments = {k: tuple(move(ROLE_MOMENT, m.detach().to(torch.float32).contiguous()) for m in moments[k]) for k in GROUPS}
        new_stats = s.new_stats(stats)
    return new_params, new_moments, new_stats, s.counts


def densify_and_prune(params, moments, stats: DensifyStats, max_grad: float, min_opacity: float, extent: float,
                      max_screen_size: Optional[float], percent_dense: float = 0.01, N: int = 2,
                      noise: Optional[torch.Tensor] = None, generator: Optional[torch.Generator] = None, return_counts: bool = False):
    """GaussianModel.densify_and_prune (gaussian_model.py:402-415): clone small high-gradient Gaussians, split large ones
    into N children, drop the split parents, then prune by opacity (and, with max_screen_size, by world size).
    `noise` [N*S,3]: optional standard-normal draws for the children (default: torch.randn on the device)."""
    cfg = _Cfg(0, int(N), 1 if max_screen_size else 0, float(max_grad), float(min_opacity), float(percent_dense * extent),
               float(max_screen_size or 0.0), float(0.1 * extent))
    p, m, s, counts = _run(cfg, params, moments, stats, noise, generator)
    return (p, m, s, counts) if return_counts else (p, m, s)


def prune_only(params, moments, stats: DensifyStats, min_opacity: float = 0.005, size_thresh: float = 0.01, return_counts: bool = False):
    """GaussianModel.prune_only (gaussian_model.py:423-430): drop low-opacity or oversized Gaussians; statistics are kept."""
    cfg = _Cfg(1, 0, 0, 0.0, float(min_opacity), 0.0, 0.0, float(size_thresh))
    p, m, s, counts = _run(cfg, params, moments, stats, None, None)
    return (p, m, s, counts) if return_counts else (p, m, s)


# ---- the same surgery on the packed parameter buffer, for optim.PackedAdam -----------------------------------------
def _run_packed(cfg: _Cfg, opt: torch.optim.Optimizer, stats: DensifyStats, noise, generator, remove=None) -> int:
    """Plan once from the flat buffer's opacity / scaling fields, move every field of the parameter buffer and of both
    Adam moment buffers straight into its place in new flat buffers (padding zero), install them into `opt`, and replace
    the three tensors of `stats` in place.  The optimiser's step count is kept."""
    from .rasterizer import packed_layout
    group = opt.param_groups[0]
    old = group["params"][0]
    _need_cuda(old)
    P, K, dev = int(group["P"]), int(group["sh_coeffs"]), old.device
    if P == 0:
        return 0
    fields = packed_layout(P, K)[0]
    views = lambda flat, layout: [flat.narrow(0, o, n).view(shape) for o, n, shape in layout]
    xyz, scaling, rotation, opacity, sh = views(old.detach(), fields)
    state = opt.state.get(old)
    with torch.cuda.device(dev):
        s = _Surgery(cfg, stats, opacity, scaling, rotation, noise, generator, remove)
        new_fields, new_total = packed_layout(s.P_new, K)

        def remap(flat, roles):
            out = torch.zeros(new_total, dtype=torch.float32, device=dev)  # alignment padding stays zero
            for src, dst, role in zip(views(flat, fields), views(out, new_fields), roles):
                s.move(role, src, dst)
            return out
        new_flat = remap(old.detach(), (ROLE_XYZ, ROLE_SCALING, ROLE_COPY, ROLE_COPY, ROLE_COPY))
        new_moments = None
        if state:
            new_moments = tuple(remap(state[k], (ROLE_MOMENT,) * 5) for k in ("exp_avg", "exp_avg_sq"))
        new_stats = s.new_stats(stats)
    install_packed(opt, new_flat, new_moments, s.P_new)
    stats.xyz_gradient_accum, stats.denom, stats.max_radii2D = new_stats.xyz_gradient_accum, new_stats.denom, new_stats.max_radii2D
    return s.P_new


def install_packed(opt: torch.optim.Optimizer, new_flat: torch.Tensor, new_moments, P_new: int) -> None:
    """What _prune_optimizer / cat_tensors_to_optimizer do (gaussian_model.py:284-341), for an `optim.PackedAdam`: `new_flat`
    becomes the parameter leaf, `new_moments` (exp_avg, exp_avg_sq) in the same layout, or None when the optimiser has no
    state yet, its moments, and group["P"] = P_new.  The step count is kept."""
    group = opt.param_groups[0]
    old = group["params"][0]
    state = opt.state.get(old)
    leaf = torch.nn.Parameter(new_flat) if isinstance(old, torch.nn.Parameter) else new_flat.requires_grad_(True)
    group["params"][0] = leaf
    group["P"] = P_new
    opt.state.pop(old, None)
    if new_moments is not None:
        state["exp_avg"], state["exp_avg_sq"] = new_moments
        opt.state[leaf] = state


def densify_and_prune_packed(opt: torch.optim.Optimizer, stats: DensifyStats, max_grad: float, min_opacity: float, extent: float,
                             max_screen_size: Optional[float], percent_dense: float = 0.01, N: int = 2,
                             noise: Optional[torch.Tensor] = None, generator: Optional[torch.Generator] = None) -> int:
    """`densify_and_prune` on the packed buffer of an `optim.PackedAdam`: same plan, same rows, same noise rows, but every
    field of the parameter buffer and of both moment buffers is moved straight into a new flat buffer of the same layout.
    The new buffer becomes the optimiser's parameter (`opt.packed`), `stats` is replaced in place, and the new P is
    returned.  Equal bit for bit to densify_and_prune on the unpacked groups followed by dist.pack."""
    cfg = _Cfg(0, int(N), 1 if max_screen_size else 0, float(max_grad), float(min_opacity), float(percent_dense * extent),
               float(max_screen_size or 0.0), float(0.1 * extent))
    return _run_packed(cfg, opt, stats, noise, generator)


def prune_only_packed(opt: torch.optim.Optimizer, stats: DensifyStats, min_opacity: float = 0.005, size_thresh: float = 0.01) -> int:
    """`prune_only` on the packed buffer of an `optim.PackedAdam` (see densify_and_prune_packed); returns the new P."""
    cfg = _Cfg(1, 0, 0, 0.0, float(min_opacity), 0.0, 0.0, float(size_thresh))
    return _run_packed(cfg, opt, stats, None, None)


def _remove_mask(remove, P: int, dev) -> torch.Tensor:
    if not isinstance(remove, torch.Tensor) or remove.dtype != torch.bool or remove.shape != (P,) or remove.device != dev:
        desc = f"{tuple(remove.shape)} {remove.dtype} on {remove.device}" if isinstance(remove, torch.Tensor) else type(remove).__name__
        raise ValueError(f"b200gs: remove must be a bool [{P}] tensor on {dev}; got {desc}")
    return remove.contiguous().view(torch.uint8)


def prune_points(params, moments, stats: DensifyStats, remove: torch.Tensor, return_counts: bool = False):
    """GaussianModel.prune_points (gaussian_model.py:306-315) by a caller's mask: drop every Gaussian where `remove` (bool [P]
    on the device) is True; survivors keep their order.  Parameters, both Adam moments and the three statistics move
    together, as in `prune_only`.  Any rule can supply the mask: `contribution.compute_contribution(...).touches == 0`
    (lossless for the cameras it was scored over), a weight threshold, or a hand mask.  A mask that removes every Gaussian
    raises ValueError.  Returns (params, moments, stats); the new P is params["xyz"].shape[0]."""
    dev, P = params["xyz"].device, params["xyz"].shape[0]
    _need_cuda(params["xyz"])
    cfg = _Cfg(MODE_PRUNE_MASK, 0, 0, 0.0, 0.0, 0.0, 0.0, 0.0)
    if P == 0:
        raise ValueError("b200gs: nothing to prune (P == 0)")
    p, m, s, counts = _run(cfg, params, moments, stats, None, None, _remove_mask(remove, P, dev))
    return (p, m, s, counts) if return_counts else (p, m, s)


def prune_points_packed(opt: torch.optim.Optimizer, stats: DensifyStats, remove: torch.Tensor) -> int:
    """`prune_points` on the packed buffer of an `optim.PackedAdam` (see densify_and_prune_packed): the parameter buffer,
    both moment buffers and `stats` are replaced; returns the new P."""
    group = opt.param_groups[0]
    P, dev = int(group["P"]), group["params"][0].device
    _need_cuda(group["params"][0])
    if P == 0:
        raise ValueError("b200gs: nothing to prune (P == 0)")
    cfg = _Cfg(MODE_PRUNE_MASK, 0, 0, 0.0, 0.0, 0.0, 0.0, 0.0)
    return _run_packed(cfg, opt, stats, None, None, _remove_mask(remove, P, dev))


def moments_from_optimizer(optimizer: torch.optim.Optimizer) -> Dict[str, Tuple[torch.Tensor, torch.Tensor]]:
    """(exp_avg, exp_avg_sq) per named param group of a reference-style Adam (gaussian_model.py:156-165)."""
    out = {}
    for group in optimizer.param_groups:
        p = group["params"][0]
        st = optimizer.state.get(p)
        if st:
            out[group["name"]] = (st["exp_avg"], st["exp_avg_sq"])
        else:
            out[group["name"]] = (torch.zeros_like(p), torch.zeros_like(p))
    return out


def install_into_optimizer(optimizer: torch.optim.Optimizer, params, moments) -> Dict[str, torch.nn.Parameter]:
    """Swap the resized tensors and Adam moments into the optimiser's single-parameter groups, as
    _prune_optimizer / cat_tensors_to_optimizer do (gaussian_model.py:284-341).  Returns the new nn.Parameters by name."""
    new = {}
    for group in optimizer.param_groups:
        name = group["name"]
        old = group["params"][0]
        st = optimizer.state.pop(old, None)
        par = torch.nn.Parameter(params[name].requires_grad_(True))
        group["params"][0] = par
        if st is not None and moments is not None:
            st["exp_avg"], st["exp_avg_sq"] = moments[name]
            optimizer.state[par] = st
        new[name] = par
    return new
