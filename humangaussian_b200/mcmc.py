"""MCMC densification (3DGS-MCMC, Kheradmand et al., NeurIPS 2024) on the device: the alternative to densify.py's
gradient-threshold rule.  It does not read the SDS gradient and it puts a hard cap on P.

    opt.step(); opt.zero_grad()
    if it % interval == 0:
        relocate_packed(opt)                  # dead Gaussians become copies of live ones; P unchanged
        add_packed(opt, cap_max)              # P -> min(cap_max, floor(1.05 P)); no host sync
    inject_noise_packed(opt)                  # every step, with the xyz lr the step used

Everything works on the optimiser's RAW parameters (opacity logits, log-scales, un-normalised quaternions), as densify.py
does.  A row is dead iff not sigmoid(opacity) > min_opacity (NaN is dead).  Sources are drawn with replacement in proportion
to sigmoid(opacity) over the live rows; a source drawn c times and its c copies all take the split ratio's opacity and
scales (csrc/mcmc.cu, DESIGN.md section 2), and every row written gets zero Adam moments.  The `*_packed` forms work on an
`optim.PackedAdam` and install new flat buffers (densify.install_packed); the dict forms take the reference's six groups
and pair with densify.install_into_optimizer.  There is no CPU path: tensors must live on a CUDA device.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from .densify import GROUPS, install_packed
from .rasterizer import _check, _ptr, _stream, load_library, packed_layout

ROLE_COPY, ROLE_OPACITY, ROLE_SCALING, ROLE_MOMENT = 0, 1, 2, 3  # == B200GS_MCMC_ROLE_*
_DICT_ROLES = {"opacity": ROLE_OPACITY, "scaling": ROLE_SCALING}  # xyz, f_dc, f_rest, rotation: copied
_PACKED_ROLES = (ROLE_COPY, ROLE_SCALING, ROLE_COPY, ROLE_OPACITY, ROLE_COPY)  # xyz, scaling, rotation, opacity, sh


def _need_cuda(t):
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise ValueError("b200gs: MCMC tensors must live on a CUDA device (there is no CPU path)")


def _live(opacity: torch.Tensor, min_opacity: float):
    """sigmoid(opacity) [P] and the live mask.  torch's CUDA sigmoid is 1/(1+expf(-x)) in float32, the kernels' gs_sigmoidf."""
    o = torch.sigmoid(opacity.reshape(-1))
    return o, o > min_opacity


def _draw(o: torch.Tensor, live: torch.Tensor, n: int, generator) -> torch.Tensor:
    """n sources with replacement, P(i) proportional to o_i over the live rows, by inversion of the CDF: one torch.rand
    draw per source from `generator`, then a binary search.  The weights are quantised to q_i = rint(o_i * 2^24) (at most
    2^-25 absolute, 0.00075 % of the smallest live weight) so that the CDF is an exact int64 prefix sum: the draw is
    reproducible by construction, also under use_deterministic_algorithms(True), and it reads nothing back to the host
    (torch.multinomial prefix-sums float weights, and validates the distribution on the host when it draws one sample).
    With no live row every draw is row 0 rather than a device fault (relocate raises ValueError in that state)."""
    q = torch.where(live, torch.round(o.double() * 2.0 ** 24), 0.0).to(torch.int64)
    cdf = torch.cumsum(q, 0)
    total = cdf[-1:]
    u = torch.rand(n, dtype=torch.float64, device=o.device, generator=generator)
    x = torch.minimum((u * total).floor().to(torch.int64), total - 1)
    return torch.searchsorted(cdf, x, right=True)


def _given_samples(samples, n: int, P: int, live: torch.Tensor) -> torch.Tensor:
    if not isinstance(samples, torch.Tensor) or samples.dtype != torch.int64 or tuple(samples.shape) != (n,):
        desc = f"{tuple(samples.shape)} {samples.dtype}" if isinstance(samples, torch.Tensor) else type(samples).__name__
        raise ValueError(f"b200gs: samples must be an int64 [{n}] tensor; got {desc}")
    samples = samples.to(live.device)
    if n and (int(samples.min()) < 0 or int(samples.max()) >= P):
        raise ValueError(f"b200gs: samples must index rows 0..{P - 1}")
    if n and not bool(live[samples].all()):
        raise ValueError("b200gs: samples must point at live rows")
    return samples.contiguous()


class _Plan:
    """The gather map [P_new], the draw counts c [P] (= bincount(samples, minlength=P), without bincount's host read of the
    maximum) and the ratio's new raw opacity / scales of the drawn rows; `move` gathers one [P, ...] array into a [P_new, ...]
    destination, which may be a view into a larger buffer.  Callers run inside `torch.cuda.device(dev)`."""

    def __init__(self, P: int, mapping: torch.Tensor, samples: torch.Tensor, opacity: torch.Tensor, scaling: torch.Tensor):
        L = self.L = load_library()
        dev = opacity.device
        self.P, self.P_new, self.st = P, mapping.numel(), _stream(dev)
        self.map = mapping.to(torch.int32).contiguous()
        self.counts = torch.zeros(P, dtype=torch.int32, device=dev).index_add_(
            0, samples, torch.ones(samples.numel(), dtype=torch.int32, device=dev))
        self.new_opacity = torch.empty(P, dtype=torch.float32, device=dev)  # rows with c == 0 are never written or read
        self.new_scaling = torch.empty(P, 3, dtype=torch.float32, device=dev)
        _check(L.b200gs_mcmc_ratio(P, _ptr(self.counts), _ptr(opacity), _ptr(scaling), _ptr(self.new_opacity),
                                   _ptr(self.new_scaling), self.st), "mcmc_ratio")

    def move(self, role: int, src: torch.Tensor, dst: torch.Tensor) -> torch.Tensor:
        rf = src.numel() // self.P
        if rf == 0:  # f_rest [P,0,3] at SH degree 0
            return dst
        _check(self.L.b200gs_mcmc_move(role, self.P, self.P_new, rf, _ptr(self.map), _ptr(self.counts), _ptr(src), _ptr(dst),
                                       _ptr(self.new_opacity), _ptr(self.new_scaling), self.st), "mcmc_move")
        return dst


def _relocation(opacity: torch.Tensor, min_opacity: float, generator, samples):
    """(d, map, samples): the j-th dead row in ascending order becomes a copy of sample j.  One host read, of d."""
    P = opacity.shape[0]
    o, live = _live(opacity, min_opacity)
    dead = torch.nonzero(~live).view(-1)
    d = dead.numel()
    if d == 0:
        return 0, None, None
    if d == P:
        raise ValueError(f"b200gs: no live Gaussian to relocate onto (every sigmoid(opacity) <= {min_opacity})")
    samples = _draw(o, live, d, generator) if samples is None else _given_samples(samples, d, P, live)
    mapping = torch.arange(P, dtype=torch.int64, device=opacity.device).index_copy_(0, dead, samples)
    return d, mapping, samples


def _growth(opacity: torch.Tensor, P: int, cap_max: int, growth: float, min_opacity: float, generator, samples):
    """(P_new, map, samples): copy j is appended as row P + j.  P_new comes from the host: no host read."""
    P_new = min(int(cap_max), int(math.floor(growth * P)))
    if P_new <= P:
        return P, None, None
    o, live = _live(opacity, min_opacity)
    n = P_new - P
    samples = _draw(o, live, n, generator) if samples is None else _given_samples(samples, n, P, live)
    mapping = torch.cat((torch.arange(P, dtype=torch.int64, device=opacity.device), samples))
    return P_new, mapping, samples


# ---- packed forms, on an optim.PackedAdam --------------------------------------------------------------------------
def _packed_fields(opt):
    group = opt.param_groups[0]
    old = group["params"][0]
    _need_cuda(old)
    P, K = int(group["P"]), int(group["sh_coeffs"])
    fields = packed_layout(P, K)[0]
    return old, P, K, fields, [old.detach().narrow(0, o, n).view(shape) for o, n, shape in fields]


def _move_packed(opt, old, P: int, K: int, fields, views, mapping, samples) -> None:
    """Gather the parameter buffer and both moment buffers into new flat buffers (padding zero) and install them."""
    _, scaling, _, opacity, _ = views
    state = opt.state.get(old)
    split = lambda flat, layout: [flat.narrow(0, o, n).view(shape) for o, n, shape in layout]
    with torch.cuda.device(old.device):
        plan = _Plan(P, mapping, samples, opacity, scaling)
        new_fields, new_total = packed_layout(plan.P_new, K)

        def remap(flat, roles):
            out = torch.zeros(new_total, dtype=torch.float32, device=old.device)  # alignment padding stays zero
            for src, dst, role in zip(split(flat, fields), split(out, new_fields), roles):
                plan.move(role, src, dst)
            return out
        new_flat = remap(old.detach(), _PACKED_ROLES)
        new_moments = tuple(remap(state[k], (ROLE_MOMENT,) * 5) for k in ("exp_avg", "exp_avg_sq")) if state else None
    install_packed(opt, new_flat, new_moments, plan.P_new)


def relocate_packed(opt: torch.optim.Optimizer, min_opacity: float = 0.005, generator: Optional[torch.Generator] = None,
                    samples: Optional[torch.Tensor] = None) -> int:
    """Move every dead Gaussian of an `optim.PackedAdam` onto a live one and return their number d.  The j-th dead row (in
    ascending order) becomes a copy of source j: xyz, rotation and SH bit for bit; every source and copy takes the split
    ratio's opacity and scales and zero Adam moments; every other row is byte-identical.  P and the step count are kept.
    `samples` (int64 [d], live rows) replaces the draw.  d == 0 changes nothing; no live row raises ValueError."""
    old, P, K, fields, views = _packed_fields(opt)
    with torch.cuda.device(old.device):
        d, mapping, samples = _relocation(views[3], min_opacity, generator, samples)
    if d:
        _move_packed(opt, old, P, K, fields, views, mapping, samples)
    return d


def add_packed(opt: torch.optim.Optimizer, cap_max: int, growth: float = 1.05, generator: Optional[torch.Generator] = None,
               samples: Optional[torch.Tensor] = None, min_opacity: float = 0.005) -> int:
    """Grow an `optim.PackedAdam` to P_new = min(cap_max, floor(growth * P)) and return P_new: P_new - P sources drawn over the
    live rows, copy j appended as row P + j; sources and copies take the split ratio's opacity and scales and zero Adam
    moments.  P_new <= P is a no-op.  `samples` (int64 [P_new - P], live rows) replaces the draw."""
    old, P, K, fields, views = _packed_fields(opt)
    with torch.cuda.device(old.device):
        P_new, mapping, samples = _growth(views[3], P, cap_max, growth, min_opacity, generator, samples)
    if P_new > P:
        _move_packed(opt, old, P, K, fields, views, mapping, samples)
    return P_new


# ---- position noise ------------------------------------------------------------------------------------------------
def _noise(xyz, scaling, rotation, opacity, noise_scale: float, k: float, t: float, eta, generator) -> None:
    P, dev = xyz.shape[0], xyz.device
    if eta is None:
        eta = torch.randn(P, 3, dtype=torch.float32, device=dev, generator=generator)
    elif not isinstance(eta, torch.Tensor) or eta.dtype != torch.float32 or tuple(eta.shape) != (P, 3):
        desc = f"{tuple(eta.shape)} {eta.dtype}" if isinstance(eta, torch.Tensor) else type(eta).__name__
        raise ValueError(f"b200gs: eta must be a float32 [{P}, 3] tensor; got {desc}")
    _need_cuda(eta)
    eta = eta.to(dev).contiguous()
    with torch.cuda.device(dev):
        _check(load_library().b200gs_mcmc_noise(P, _ptr(xyz), _ptr(scaling), _ptr(rotation), _ptr(opacity), _ptr(eta),
                                                float(noise_scale), float(k), float(t), _stream(dev)), "mcmc_noise")


def inject_noise_packed(opt: torch.optim.Optimizer, noise_lr: float = 5e5, k: float = 100.0, t: float = 0.005,
                        eta: Optional[torch.Tensor] = None, generator: Optional[torch.Generator] = None) -> None:
    """xyz += noise_lr * lr_xyz * sigmoid(-k (sigmoid(opacity) - t)) * Sigma eta in place, in one launch without a host sync,
    with lr_xyz = the optimiser's current xyz lr (the one its last step used) and Sigma = R diag(exp(2 scaling)) R^T.
    eta [P,3] float32: standard-normal draws (default torch.randn with `generator`).  Only the xyz field is written."""
    old, P, K, fields, views = _packed_fields(opt)
    xyz, scaling, rotation, opacity, _ = views
    _noise(xyz, scaling, rotation, opacity, noise_lr * opt.param_groups[0]["lrs"]["xyz"], k, t, eta, generator)


# ---- dict forms: the reference's six raw groups, for densify.install_into_optimizer ----------------------------------
def _dict_src(params: Dict[str, torch.Tensor]):
    _need_cuda(params["xyz"])
    return {g: params[g].detach().to(torch.float32).contiguous() for g in GROUPS}


def _move_dict(src, moments, mapping, samples):
    P, dev = src["xyz"].shape[0], src["xyz"].device
    with torch.cuda.device(dev):
        plan = _Plan(P, mapping, samples, src["opacity"], src["scaling"])
        out = lambda role, t: plan.move(role, t, torch.empty((plan.P_new,) + tuple(t.shape[1:]), dtype=torch.float32, device=dev))
        new_params = {g: out(_DICT_ROLES.get(g, ROLE_COPY), src[g]) for g in GROUPS}
        new_moments = None
        if moments is not None:
            new_moments = {g: tuple(out(ROLE_MOMENT, m.detach().to(torch.float32).contiguous()) for m in moments[g]) for g in GROUPS}
    return new_params, new_moments


def relocate(params: Dict[str, torch.Tensor], moments, min_opacity: float = 0.005, generator: Optional[torch.Generator] = None,
             samples: Optional[torch.Tensor] = None, return_count: bool = False):
    """`relocate_packed` on the groups xyz, f_dc, f_rest, opacity, scaling, rotation (raw) and their (exp_avg, exp_avg_sq)
    moments (or None).  Returns (params, moments) -- the inputs themselves when no row is dead -- and d with return_count."""
    src = _dict_src(params)
    with torch.cuda.device(src["xyz"].device):
        d, mapping, samples = _relocation(src["opacity"], min_opacity, generator, samples)
    p, m = _move_dict(src, moments, mapping, samples) if d else (src, moments)
    return (p, m, d) if return_count else (p, m)


def add(params: Dict[str, torch.Tensor], moments, cap_max: int, growth: float = 1.05, generator: Optional[torch.Generator] = None,
        samples: Optional[torch.Tensor] = None, min_opacity: float = 0.005):
    """`add_packed` on the six raw groups and their moments (or None): returns (params, moments) with
    min(cap_max, floor(growth * P)) rows (the inputs themselves when that is not more than P)."""
    src = _dict_src(params)
    P = src["xyz"].shape[0]
    with torch.cuda.device(src["xyz"].device):
        P_new, mapping, samples = _growth(src["opacity"], P, cap_max, growth, min_opacity, generator, samples)
    return _move_dict(src, moments, mapping, samples) if P_new > P else (src, moments)


def inject_noise(params: Dict[str, torch.Tensor], lr_xyz: float, noise_lr: float = 5e5, k: float = 100.0, t: float = 0.005,
                 eta: Optional[torch.Tensor] = None, generator: Optional[torch.Generator] = None) -> None:
    """`inject_noise_packed` on the six raw groups: params["xyz"] (contiguous float32 on the device) is updated in place."""
    xyz = params["xyz"]
    _need_cuda(xyz)
    if xyz.dtype != torch.float32 or not xyz.is_contiguous() or xyz.dim() != 2 or xyz.shape[1] != 3:
        raise ValueError("b200gs: params['xyz'] must be a contiguous float32 [P, 3] tensor (it is updated in place)")
    src = {g: params[g].detach().to(device=xyz.device, dtype=torch.float32).contiguous() for g in ("scaling", "rotation", "opacity")}
    _noise(xyz.detach(), src["scaling"], src["rotation"], src["opacity"], noise_lr * lr_xyz, k, t, eta, generator)
