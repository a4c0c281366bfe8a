"""The optimiser step on the packed parameter buffer -- the reference's Adam with its six parameter groups.

The reference trains with torch.optim.Adam(l, lr=0.0, eps=1e-15) over six single-tensor groups xyz, f_dc, f_rest,
opacity, scaling, rotation (gaussiansplatting/scene/gaussian_model.py:156-165) and decays the xyz lr every step
(get_expon_lr_func, utils/general_utils.py:29-62; update_learning_rate, gaussian_model.py:171-176).  The fastest path
of this rasteriser trains ONE flat buffer of raw parameters instead (rasterize_views_packed(raw=True); its backward
writes packed.grad in the same layout), where f_dc and f_rest interleave inside the SH field.  PackedAdam takes the
reference's step on that buffer in one kernel launch (csrc/optim.cu), with each element's lr chosen by its group:

    opt = PackedAdam(packed, P, K, lrs=dict(xyz=..., f_dc=..., f_rest=..., opacity=..., scaling=..., rotation=...),
                     xyz_scheduler=expon_lr_func(lr_init, lr_final, lr_delay_mult=0.01, max_steps=30000))
    opt.update_learning_rate(it)
    color, radii, depth, alpha = rasterize_views_packed(opt.packed, opt.P, K, ..., raw=True)
    loss.backward(); opt.step(); opt.zero_grad()
    densify_and_prune_packed(opt, stats, ...)      # densify.py: new flat buffer, moments and P installed into `opt`

Being a torch.optim.Optimizer, it works with zero_grad, state_dict / load_state_dict and torch.amp.GradScaler (which
unscales packed.grad through param_groups and skips the step on the host when it finds inf / nan).
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Dict, Optional

import numpy as np
import torch

from .rasterizer import _check, _ptr, _stream, load_library, packed_layout, packed_numel

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")  # the reference's group order == step_size order


class _AdamCfg(C.Structure):  # == b200gs_adam_cfg
    _fields_ = [("off_xyz", C.c_int64), ("off_scaling", C.c_int64), ("off_rotation", C.c_int64), ("off_opacity", C.c_int64),
                ("off_sh", C.c_int64), ("P", C.c_int32), ("sh_coeffs", C.c_int32), ("total", C.c_int64),
                ("step_size", C.c_float * 6), ("bias_correction2_sqrt", C.c_float), ("one_minus_beta1", C.c_float),
                ("beta2", C.c_float), ("one_minus_beta2", C.c_float), ("eps", C.c_float)]


def expon_lr_func(lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1000000) -> Callable[[int], float]:
    """get_expon_lr_func (general_utils.py:29-62): log-linear decay from lr_init (step 0) to lr_final (max_steps), eased in
    over lr_delay_steps by a reverse cosine from lr_init * lr_delay_mult; 0 for step < 0 or when both rates are 0."""

    def helper(step):
        if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
            return 0.0
        if lr_delay_steps > 0:
            delay_rate = lr_delay_mult + (1 - lr_delay_mult) * np.sin(0.5 * np.pi * np.clip(step / lr_delay_steps, 0, 1))
        else:
            delay_rate = 1.0
        t = np.clip(step / max_steps, 0, 1)
        return delay_rate * np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t)

    return helper


def adam_cfg(P: int, sh_coeffs: int, lrs: Dict[str, float], betas, eps: float, step: float) -> _AdamCfg:
    """The kernel's arguments for step t = `step` (already incremented): torch's host scalars of _multi_tensor_adam
    (torch/optim/adam.py, non-capturable branch) in double, rounded to float by the ctypes fields."""
    beta1, beta2 = betas
    bias_correction1 = 1 - beta1 ** step
    bias_correction2 = 1 - beta2 ** step
    fields, total = packed_layout(P, sh_coeffs)
    cfg = _AdamCfg(*(o for o, _, _ in fields), P, sh_coeffs, total)
    for g, name in enumerate(GROUPS):
        cfg.step_size[g] = (lrs[name] / bias_correction1) * -1
    cfg.bias_correction2_sqrt = bias_correction2 ** 0.5
    cfg.one_minus_beta1, cfg.beta2, cfg.one_minus_beta2, cfg.eps = 1 - beta1, beta2, 1 - beta2, eps
    return cfg


class PackedAdam(torch.optim.Optimizer):
    """torch.optim.Adam(amsgrad=False, weight_decay=0) with the reference's six groups, over the packed buffer.

    One param group holds the flat leaf tensor, the six lrs by the reference's names (group["lrs"]), betas, eps, and the
    buffer's P and sh_coeffs (so that state_dict / load_state_dict carry the layout).  The state holds exp_avg and
    exp_avg_sq as flat buffers of the same layout and `step` (a CPU float tensor, as torch's Adam keeps it)."""

    def __init__(self, packed: torch.Tensor, P: int, sh_coeffs: int, lrs: Dict[str, float], betas=(0.9, 0.999), eps: float = 1e-15,
                 xyz_scheduler: Optional[Callable[[int], float]] = None):
        if set(lrs) != set(GROUPS):
            raise ValueError(f"PackedAdam: lrs must name exactly the groups {GROUPS}")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0 or not eps >= 0.0:
            raise ValueError("PackedAdam: invalid betas / eps")
        if packed.dim() != 1 or packed.dtype != torch.float32 or not packed.is_contiguous() or packed.numel() != packed_numel(P, sh_coeffs):
            raise ValueError(f"PackedAdam: the buffer must be contiguous fp32 with {packed_numel(P, sh_coeffs)} elements")
        group = dict(params=[packed], lrs={k: float(lrs[k]) for k in GROUPS}, P=int(P), sh_coeffs=int(sh_coeffs))
        super().__init__([group], dict(betas=(float(betas[0]), float(betas[1])), eps=float(eps)))
        self.xyz_scheduler = xyz_scheduler

    @property
    def packed(self) -> torch.Tensor:
        """The current flat parameter leaf (densify / prune replace it)."""
        return self.param_groups[0]["params"][0]

    @property
    def P(self) -> int:
        return int(self.param_groups[0]["P"])

    @property
    def sh_coeffs(self) -> int:
        return int(self.param_groups[0]["sh_coeffs"])

    def update_learning_rate(self, iteration: int) -> float:
        """GaussianModel.update_learning_rate (gaussian_model.py:171-176): only xyz is scheduled."""
        if self.xyz_scheduler is None:
            raise RuntimeError("PackedAdam: no xyz_scheduler was given")
        lr = self.xyz_scheduler(iteration)
        group = self.param_groups[0]
        group["lrs"] = {**group["lrs"], "xyz": lr}  # a new dict: a state_dict taken earlier shares the old one
        return lr

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        group = self.param_groups[0]
        p = group["params"][0]
        if p.grad is None:
            return loss
        g = p.grad
        if p.device.type != "cuda":
            raise RuntimeError("b200gs: tensors must live on a CUDA device (there is no CPU path)")
        if g.is_sparse or g.dtype != torch.float32 or not g.is_contiguous() or g.shape != p.shape:
            raise ValueError("PackedAdam: the gradient must be a dense contiguous fp32 buffer of the parameter's layout")
        state = self.state[p]
        if not state:
            state["step"] = torch.tensor(0.0)
            state["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        state["step"] += 1
        cfg = adam_cfg(group["P"], group["sh_coeffs"], group["lrs"], group["betas"], group["eps"], state["step"].item())
        L = load_library()
        with torch.cuda.device(p.device):
            _check(L.b200gs_adam_packed(C.byref(cfg), _ptr(p), _ptr(g), _ptr(state["exp_avg"]), _ptr(state["exp_avg_sq"]),
                                        _stream(p.device)), "adam_packed")
        return loss
