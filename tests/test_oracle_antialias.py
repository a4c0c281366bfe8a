"""CPU: the antialiasing filter's reference (tests/aa_reference.py) against torch.autograd over the dense float64
formulation, its scale consistency, its floor, and the C ABI of the render options."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from util import ROOT, close, close_rows, grad_images, screen_scene, small_scene


def _run(inp, seed, raw=None):
    """AA oracle forward + backward against dense float64 autograd with the filter.  raw (optional dict of raw opacity /
    scale / rotation arrays): the activations run in front of both sides (float32 torch for the oracle's inputs, float64
    autograd for the reference) and the oracle's gradients are chained through their Jacobians, as the kernels do."""
    from aa_reference import AAOracle, dense_render_aa
    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    acts = {"opacities": torch.sigmoid, "scales": torch.exp, "rotations": torch.nn.functional.normalize}
    if raw is not None:
        inp = dict(inp, **{k: acts[k](torch.tensor(v)).numpy() for k, v in raw.items()})
    o = AAOracle(threads=1)
    col, radii, dep, alp = o.forward(**inp)
    st = o.state()
    H, W = inp["image_height"], inp["image_width"]
    gC, gD, gA = grad_images(H, W, seed)
    g = o.backward(gC, gD, gA)
    names = [k for k in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp") if inp.get(k) is not None]
    leaves = {k: t64(raw[k] if raw is not None and k in raw else inp[k]).requires_grad_(True) for k in names}
    ten = {k: (acts[k](v) if raw is not None and k in raw else v) for k, v in leaves.items()}
    if raw is not None:  # chain the oracle's activated-input gradients through the activations (float64)
        for k in raw:
            v = t64(raw[k]).requires_grad_(True)
            g[k] = torch.autograd.grad(acts[k](v), v, t64(g[k]).reshape(v.shape))[0].numpy()
    m2d = torch.zeros(len(radii), 3, dtype=torch.float64, requires_grad=True)
    ids = np.nonzero(radii > 0)[0]
    order = ids[np.lexsort((ids, st["depths"][ids]))]
    c, d, a, _ = dense_render_aa(means3D=ten["means3D"], means2D=m2d, opacities=ten["opacities"], viewmatrix=t64(inp["viewmatrix"]),
                                 projmatrix=t64(inp["projmatrix"]), campos=t64(inp["campos"]), bg=t64(inp["bg"]), H=H, W=W,
                                 tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], radii=radii, rect=st["rect"], order=order,
                                 sh_degree=inp.get("sh_degree", 0), shs=ten.get("shs"), colors_precomp=ten.get("colors_precomp"),
                                 scales=ten.get("scales"), rotations=ten.get("rotations"), cov3D_precomp=ten.get("cov3D_precomp"))
    for got, ref in ((col, c), (dep, d), (alp, a)):
        ok, worst = close(got, ref.detach().numpy())
        assert ok, f"filtered forward differs from dense float64 reference ({worst:.2f}x tolerance)"
    ((c * t64(gC)).sum() + (d * t64(gD)).sum() + (a * t64(gA)).sum()).backward()
    ref = dict(means2D=m2d.grad, **{k: leaves[k].grad for k in names})
    for k, r in ref.items():
        # the criterion of test_oracle_autograd.py
        cmp = close_rows if k == "cov3D_precomp" else close
        ok, worst = cmp(g[k], r.numpy().reshape(g[k].shape), atol=1e-4, rtol=1e-3)
        assert ok, f"dL/d{k}: AA oracle vs autograd {worst:.2f}x over (1e-4 abs, 1e-3 rel)"
    return o, g


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_aa_backward_vs_autograd(deg):
    inp, _, _ = small_scene(P=300, deg=deg, seed=deg)
    o, g = _run(inp, deg)
    assert (o.f["rho"][g["opacities"].reshape(-1) != 0] < 0.999).all()  # the filter is active on every Gaussian that renders
    assert np.abs(g["rho_cotangent"]).max() > 0


def test_aa_backward_opaque_layers():
    inp, _, _ = small_scene(P=500, deg=1, seed=9, H=32, W=32, dist=1.3)
    inp["opacities"] = np.clip(inp["opacities"] * 8, 0, 0.99999).astype(np.float32)
    inp["scales"] = (inp["scales"] * 2.0).astype(np.float32)
    inp["shs"][:, 0, :] -= 1.2
    o, _ = _run(inp, 1)
    assert (o.state()["final_T"] < 1e-3).any()


def test_aa_backward_precomputed_inputs():
    from oracle.gs_oracle import Oracle
    inp, _, _ = small_scene(P=250, deg=0, seed=3)
    o = Oracle(threads=1)
    o.forward(**inp)
    st = o.state()
    inp2 = {k: v for k, v in inp.items() if k not in ("shs", "scales", "rotations")}
    inp2["colors_precomp"] = (np.abs(st["rgb"]) + 0.1).astype(np.float32)
    inp2["cov3D_precomp"] = st["cov3d"].copy()
    inp2["sh_degree"] = 0
    _run(inp2, 2)


def test_aa_backward_guard_band_clamp():
    inp, _, _ = small_scene(P=300, deg=0, seed=4, H=48, W=48, fovy_deg=25.0, dist=1.1)
    inp["scales"] = (inp["scales"] * 3).astype(np.float32)
    _run(inp, 3)


def test_aa_backward_raw_parameters():
    """Raw parameters (opacity logits, log-scales, un-normalised quaternions): the filter's opacity gradient then passes
    through the sigmoid's Jacobian, as in the kernels."""
    _, _, p = small_scene(P=300, deg=2, seed=8)
    inp, _, _ = small_scene(P=300, deg=2, seed=8)
    rng = np.random.RandomState(0)
    raw = dict(opacities=p.opacity.detach().numpy().copy(), scales=p.scaling.detach().numpy().copy(),
               rotations=(p.rotation.detach().numpy() * (0.5 + rng.rand(300, 1))).astype(np.float32))
    _run(inp, 4, raw=raw)


def _sub_pixel_scene(H, W, n=120, seed=0):
    rng = np.random.RandomState(seed)
    px, py = rng.uniform(2, W - 3, n), rng.uniform(2, H - 3, n)
    sigma = np.exp(rng.uniform(np.log(0.15), np.log(2.0), n))  # sub-pixel to 2 px at W x H
    return screen_scene(px, py, rng.uniform(2.0, 4.0, n), sigma, rng.uniform(0.3, 0.9, n).astype(np.float32), H=H, W=W)


def test_scale_consistency_box_filtered():
    """The same cameras at W x H and at 4W x 4H: with this repository's pixel centres ((ndc + 1) * W - 1) / 2, the high-res
    pixels 4i..4i+3 average to exactly the low-res coordinate i, so a 4x4 box average of the large render should match the
    small one.  The filter must bring it closer, in colour and in alpha (DESIGN.md section 6 records both errors)."""
    from aa_reference import AAOracle
    H, W = 24, 32
    lo = _sub_pixel_scene(H, W)
    hi = dict(lo, image_height=4 * H, image_width=4 * W)
    err = {}
    for aa in (False, True):
        c0, _, _, a0 = AAOracle().forward(antialiasing=aa, **lo)
        c1, _, _, a1 = AAOracle().forward(antialiasing=aa, **hi)
        box = lambda x: x.reshape(x.shape[0], H, 4, W, 4).mean(axis=(2, 4))
        err[aa] = (float(np.abs(box(c1) - c0).mean()), float(np.abs(box(a1) - a0).mean()))
    print(f"mean |box4(4x render) - render|: colour {err[False][0]:.5f} -> {err[True][0]:.5f}, "
          f"alpha {err[False][1]:.5f} -> {err[True][1]:.5f} (filter off -> on)")
    assert err[True][0] < err[False][0] and err[True][1] < err[False][1]


def floor_scenes(H=25, W=33):
    """Two scenes whose every rendered Gaussian has rho on its floor (0.005): flat Gaussians seen edge-on, and a precomputed
    covariance with det0 < 0 < det.  Opacity 0.99, so that the floored opacity (0.00495) still blends where the footprint's
    centre falls on a pixel centre (odd image sizes put the optical axis on one) and the floor's gradient path runs."""
    base = _sub_pixel_scene(H, W, n=24, seed=3)
    base["opacities"] = np.full_like(base["opacities"], 0.99)
    # (1) edge-on disks: identity view, a disk in the x-z plane (zero y axis) on the optical axis, so its depth extent
    # projects to nothing and its footprint is a segment; and lines (rank 1 in 3D)
    inp = {k: v[:6] if isinstance(v, np.ndarray) and v.ndim and v.shape[0] == 24 else v for k, v in base.items() if k != "cov3D_precomp"}
    inp["scales"] = np.tile(np.array([[0.02, 0.0, 0.015]], np.float32), (6, 1))
    inp["scales"][3:] = [0.0, 0.02, 0.0]
    inp["rotations"] = np.tile(np.array([[1, 0, 0, 0]], np.float32), (6, 1))
    inp["means3D"] = inp["means3D"].copy()
    inp["means3D"][:, :2] = 0.0
    inp["means3D"][:, 2] = np.linspace(2.0, 3.0, 6)
    # (2) det0 < 0 < det from a precomputed covariance (slightly indefinite in the screen plane)
    inp2 = dict(base)
    inp2["cov3D_precomp"] = base["cov3D_precomp"].copy()
    inp2["cov3D_precomp"][:, 0] *= -0.01
    return [("edge-on", inp), ("det0 <= 0", inp2)]


def test_rho_floor_is_finite_and_flat():
    """rho reaches its floor (0.005) for a flat Gaussian (one zero scale axis) seen edge-on and for a precomputed covariance
    whose 2D determinant det0 is <= 0: outputs stay finite and the rho-gradient is zero there."""
    from aa_reference import AAOracle, RHO2_FLOOR
    for case, x in floor_scenes():
        o = AAOracle(threads=1)
        out = o.forward(**x)
        vis = out[1] > 0
        assert vis.any(), case
        floor = o.f["ratio"][vis] <= RHO2_FLOOR
        assert floor.all(), f"{case}: ratios {o.f['ratio'][vis]}"
        assert np.all(o.f["rho"][vis] == np.sqrt(RHO2_FLOOR)), case
        for img in out:
            assert np.isfinite(img).all(), case
        g = o.backward(*grad_images(x["image_height"], x["image_width"], 0))
        assert np.abs(g["dL_do_eff"]).max() > 0, f"{case}: no floored Gaussian blends"
        assert np.all(g["rho_cotangent"][vis] == 0.0), case
        for k, v in g.items():
            if isinstance(v, np.ndarray):
                assert np.isfinite(v).all(), (case, k)


# ---- C ABI of the render options ---------------------------------------------------------------------------------------
LIB = os.path.join(ROOT, "humangaussian_b200", "libb200gs.so")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        import __graft_entry__ as g
        g.build()
    from humangaussian_b200 import rasterizer
    rasterizer.load_library()
    return rasterizer._lib


def test_render_opts_layout_matches_the_header(tmp_path):
    from humangaussian_b200.rasterizer import _RenderOpts
    src = tmp_path / "opts.c"
    fields = [f[0] for f in _RenderOpts._fields_]
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200gs.h"', 'int main(void){',
            'printf("size %zu\\n", sizeof(b200gs_render_opts));']
    body += [f'printf("{f} %zu\\n", offsetof(b200gs_render_opts, {f}));' for f in fields]
    body.append("return 0;}")
    src.write_text("\n".join(body))
    exe = tmp_path / "opts"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(_RenderOpts)
    for f in fields:
        assert int(got[f]) == getattr(_RenderOpts, f).offset, f


def test_render_opts_abi5_struct_bytes_is_checked(lib):
    """Too small a struct_bytes is an argument error on every *_opts entry; NULL and a full struct are accepted.  An empty
    scene (P = 0) returns from the backward before any device work, so this runs without a GPU."""
    from humangaussian_b200 import rasterizer as R
    prm, _, _ = R._make_params(0, 1, 0, 1, 16, 16, 1.0, [1.0], [1.0])
    fake = C.c_void_p(256)  # never dereferenced: every call below returns before touching a buffer
    n = C.c_int64(0)
    # means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, bg, viewmatrix, projmatrix, campos, radii
    inputs = [fake, fake, None, fake, fake, fake, None, fake, fake, fake, fake, fake]

    def bwd(opts, det=False, ins=inputs):
        args = [C.byref(prm), opts] + ins + [fake, fake, 1 << 16, fake, 0] + [fake] * 11 + [fake, 1 << 20]
        if det:
            return lib.b200gs_backward_deterministic_opts(*args, fake, 1 << 20, 1 << 16, C.byref(n), None)
        return lib.b200gs_backward_opts(*args, None)

    def fwd(opts):
        return lib.b200gs_forward_opts(C.byref(prm), opts, *inputs[:11], fake, fake, fake, fake, fake, 1, fake, 1, 1, fake, 1,
                                       C.byref(n), None)

    for small in (0, 4, C.sizeof(R._RenderOpts) - 1):
        o = R._RenderOpts(small, 1)
        assert bwd(C.byref(o)) == R.E_ARGS and fwd(C.byref(o)) == R.E_ARGS, small
        assert bwd(C.byref(o), det=True) == R.E_ARGS, small
    larger = R._RenderOpts(C.sizeof(R._RenderOpts) + 64, 1)  # a newer header's struct: the fields this library knows are read
    for o in (None, C.byref(R._render_opts(True)), C.byref(R._render_opts(False)), C.byref(larger)):
        assert bwd(o) == R.OK
    # the filtered backward needs the opacities it multiplies (as raw parameters do)
    no_op = list(inputs)
    no_op[3] = None
    assert bwd(C.byref(R._render_opts(True)), ins=no_op) == R.E_ARGS
    assert bwd(None, ins=no_op) == R.OK
