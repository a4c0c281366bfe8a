"""CPU: the host side of PackedAdam -- the xyz lr schedule against the reference's own values, the ctypes mirror of
b200gs_adam_cfg against the header, and the kernel's scalars against torch's Adam expressions."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from util import ROOT

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_lr.npz"))
REF_LRS = dict(xyz=0.00005, f_dc=0.0125, f_rest=0.0125 / 20.0, opacity=0.01, scaling=0.005, rotation=0.001)


@pytest.mark.parametrize("case", ["default", "delayed"])
def test_expon_lr_func_equals_the_reference(case):
    from humangaussian_b200.optim import expon_lr_func
    lr_init, lr_final, delay_steps, delay_mult, max_steps = GOLD[case + "_args"]
    f = expon_lr_func(lr_init=float(lr_init), lr_final=float(lr_final), lr_delay_steps=int(delay_steps), lr_delay_mult=float(delay_mult),
                      max_steps=int(max_steps))
    got = np.array([float(f(int(s))) for s in GOLD["steps"]])
    np.testing.assert_array_equal(got, GOLD[case + "_lr"])


def test_update_learning_rate_schedules_only_xyz():
    from humangaussian_b200.optim import PackedAdam, expon_lr_func
    from humangaussian_b200.rasterizer import packed_numel
    f = expon_lr_func(0.00016, 0.0000016, lr_delay_mult=0.01, max_steps=30000)
    opt = PackedAdam(torch.zeros(packed_numel(5, 4), requires_grad=True), 5, 4, REF_LRS, xyz_scheduler=f)
    sd = opt.state_dict()
    assert opt.update_learning_rate(1234) == f(1234)
    lrs = opt.param_groups[0]["lrs"]
    assert lrs["xyz"] == f(1234) and all(lrs[k] == REF_LRS[k] for k in REF_LRS if k != "xyz")
    assert sd["param_groups"][0]["lrs"]["xyz"] == REF_LRS["xyz"]  # an earlier snapshot is not changed


def test_adam_cfg_struct_matches_the_header_layout(tmp_path):
    """sizeof / offsetof of b200gs_adam_cfg as gcc sees include/b200gs.h equal the ctypes mirror."""
    from humangaussian_b200.optim import _AdamCfg
    names = [f[0] for f in _AdamCfg._fields_]
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200gs.h"', 'int main(void){',
            'printf("sizeof %zu\\n", sizeof(b200gs_adam_cfg));']
    body += [f'printf("{n} %zu\\n", offsetof(b200gs_adam_cfg, {n}));' for n in names]
    body.append("return 0;}")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(body))
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got["sizeof"]) == C.sizeof(_AdamCfg)
    for n in names:
        assert int(got[n]) == getattr(_AdamCfg, n).offset, n


@pytest.mark.parametrize("step", [1, 2, 3, 10, 1000, 30000])
@pytest.mark.parametrize("betas,eps", [((0.9, 0.999), 1e-15), ((0.8, 0.99), 1e-8)])
def test_host_scalars_equal_torch_expressions(step, betas, eps):
    """The floats handed to the kernel are torch's own host expressions (torch/optim/adam.py, _multi_tensor_adam,
    non-capturable branch), evaluated in double and rounded to float as a foreach scalar argument is."""
    from humangaussian_b200.optim import GROUPS, adam_cfg
    from humangaussian_b200.rasterizer import packed_layout
    beta1, beta2 = betas
    st = torch.tensor(float(step))
    cfg = adam_cfg(7, 16, REF_LRS, betas, eps, st.item())
    bias_correction1 = 1 - beta1 ** st.item()
    bias_correction2 = 1 - beta2 ** st.item()
    f32 = lambda x: np.float32(x).tobytes()
    for g, name in enumerate(GROUPS):
        assert f32(cfg.step_size[g]) == f32((REF_LRS[name] / bias_correction1) * -1), name
    assert f32(cfg.bias_correction2_sqrt) == f32(bias_correction2 ** 0.5)
    assert f32(cfg.one_minus_beta1) == f32(1 - beta1) and f32(cfg.beta2) == f32(beta2)
    assert f32(cfg.one_minus_beta2) == f32(1 - beta2) and f32(cfg.eps) == f32(eps)
    fields, total = packed_layout(7, 16)
    assert [cfg.off_xyz, cfg.off_scaling, cfg.off_rotation, cfg.off_opacity, cfg.off_sh] == [o for o, _, _ in fields]
    assert (cfg.P, cfg.sh_coeffs, cfg.total) == (7, 16, total)


def test_packed_adam_validates_its_arguments():
    from humangaussian_b200.optim import PackedAdam
    from humangaussian_b200.rasterizer import packed_numel
    flat = torch.zeros(packed_numel(5, 4), requires_grad=True)
    with pytest.raises(ValueError):
        PackedAdam(flat, 6, 4, REF_LRS)                              # wrong layout size
    with pytest.raises(ValueError):
        PackedAdam(flat, 5, 4, {k: v for k, v in REF_LRS.items() if k != "f_rest"})
    opt = PackedAdam(flat, 5, 4, REF_LRS)
    flat.grad = torch.zeros_like(flat)
    with pytest.raises(RuntimeError, match="CUDA device"):           # no CPU path
        opt.step()
    assert opt.P == 5 and opt.sh_coeffs == 4 and opt.packed is flat


def test_library_rejects_bad_adam_arguments():
    """Argument validation of b200gs_adam_packed runs before any launch, so it is checked here without a GPU."""
    from humangaussian_b200 import rasterizer as R
    from humangaussian_b200.optim import adam_cfg
    L = R.load_library()
    buf = (C.c_float * 64)()
    addr = (C.addressof(buf) + 15) & ~15
    p = C.c_void_p(addr)

    def call(cfg, ptrs=(p, p, p, p)):
        return L.b200gs_adam_packed(C.byref(cfg), *ptrs, None)
    good = adam_cfg(1, 2, REF_LRS, (0.9, 0.999), 1e-15, 1.0)
    assert call(good, (None, p, p, p)) == R.E_ARGS
    assert call(good, (C.c_void_p(addr + 4), p, p, p)) == R.E_ARGS  # not 16-byte aligned
    bad = adam_cfg(1, 2, REF_LRS, (0.9, 0.999), 1e-15, 1.0); bad.sh_coeffs = 0
    assert call(bad) == R.E_RANGE
    bad = adam_cfg(1, 2, REF_LRS, (0.9, 0.999), 1e-15, 1.0); bad.off_rotation += 2
    assert call(bad) == R.E_RANGE                                   # not a multiple of 4
    bad = adam_cfg(1, 2, REF_LRS, (0.9, 0.999), 1e-15, 1.0); bad.total -= 4
    assert call(bad) == R.E_RANGE                                   # sh field runs past the buffer
    bad = adam_cfg(1, 2, REF_LRS, (0.9, 0.999), 1e-15, 1.0); bad.off_scaling = 0
    assert call(bad) == R.E_RANGE                                   # overlaps xyz
