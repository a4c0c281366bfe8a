"""CPU: the 3D smoothing filter's reference (tests/filter3d_reference.py) -- its hand-derived chain against torch.autograd over
the dense float64 formulation, the weight invariant, the sampling rate's edge cases, the filter's lower bound on the
projected footprint, and the C ABI of the render options with the filter pointer."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from filter3d_reference import (VARIANCE_SCALE, Filter3DOracle, chain, dense_render_f3d, filter_params, filtered_tensors, finalize,
                                sampling_rate)
from util import ROOT, close, grad_images, small_scene

CASES = ("v=0", "v>>s^2", "v<<s^2", "s=0", "s=1e-7")


def filter_case(inp, case, seed=0):
    """(inputs, variances [P]) for one of CASES; the degenerate cases zero / shrink one scale axis of a third of the
    Gaussians and use a variance of the scene's median s^2"""
    s = np.asarray(inp["scales"], np.float32).copy()
    P = len(s)
    med = float(np.median(s * s))
    rng = np.random.RandomState(seed)
    if case == "v=0":
        var = np.zeros(P, np.float32)
    elif case == "v>>s^2":  # coef < 0.1 everywhere: near-opaque Gaussians, so that the filtered ones still blend
        var = (5.0 * (s * s).max(1) * rng.uniform(1, 2, P)).astype(np.float32)
        inp = dict(inp, opacities=np.full_like(inp["opacities"], 0.995))
    elif case == "v<<s^2":
        var = (1e-4 * (s * s).min(1) * rng.uniform(1, 2, P)).astype(np.float32)
    else:
        idx = np.arange(0, P, 3)
        s[idx, rng.randint(0, 3, len(idx))] = 0.0 if case == "s=0" else 1e-7
        var = (med * rng.uniform(0.5, 2, P)).astype(np.float32)
    return dict(inp, scales=s), var


def _run(inp, var, seed, aa=False, raw=None):
    """Filter3DOracle forward + backward against dense float64 autograd.  raw (optional dict of raw opacity / scale
    arrays): the activations run in front of both sides, and the reference chains through their Jacobians."""
    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    acts = {"opacities": torch.sigmoid, "scales": torch.exp}
    if raw is not None:
        inp = dict(inp, **{k: acts[k](torch.tensor(v)).numpy() for k, v in raw.items()})
    o = Filter3DOracle(threads=1)
    col, radii, dep, alp = o.forward(filter_3d=var, antialiasing=aa, **inp)
    st = o.state()
    H, W = inp["image_height"], inp["image_width"]
    gC, gD, gA = grad_images(H, W, seed)
    g = o.backward(gC, gD, gA, raw=raw)
    for k, v in g.items():
        if isinstance(v, np.ndarray):
            assert np.isfinite(v).all(), k
    names = ("means3D", "opacities", "shs", "scales", "rotations")
    leaves = {k: t64(raw[k] if raw is not None and k in raw else inp[k]).requires_grad_(True) for k in names}
    ten = {k: (acts[k](v) if raw is not None and k in raw else v) for k, v in leaves.items()}
    m2d = torch.zeros(len(radii), 3, dtype=torch.float64, requires_grad=True)
    ids = np.nonzero(radii > 0)[0]
    order = ids[np.lexsort((ids, st["depths"][ids]))]
    c, d, a, _ = dense_render_f3d(means3D=ten["means3D"], means2D=m2d, opacities=ten["opacities"], scales=ten["scales"], filter_3d=var,
                                  antialiasing=aa, viewmatrix=t64(inp["viewmatrix"]), projmatrix=t64(inp["projmatrix"]),
                                  campos=t64(inp["campos"]), bg=t64(inp["bg"]), H=H, W=W, tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"],
                                  radii=radii, rect=st["rect"], order=order, sh_degree=inp["sh_degree"], shs=ten["shs"],
                                  rotations=ten["rotations"])
    for got, ref in ((col, c), (dep, d), (alp, a)):
        ok, worst = close(got, ref.detach().numpy())
        assert ok, f"filtered forward differs from dense float64 reference ({worst:.2f}x tolerance)"
    ((c * t64(gC)).sum() + (d * t64(gD)).sum() + (a * t64(gA)).sum()).backward()
    ref = dict(means2D=m2d.grad, **{k: leaves[k].grad for k in names})
    for k, r in ref.items():
        assert torch.isfinite(r).all(), k
        ok, worst = close(g[k], r.numpy().reshape(g[k].shape), atol=1e-4, rtol=1e-3)
        assert ok, f"dL/d{k}: 3D-filter reference vs autograd {worst:.2f}x over (1e-4 abs, 1e-3 rel)"
    return o, g


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("case", CASES)
def test_chain_vs_autograd(case, aa):
    inp, _, _ = small_scene(P=300, deg=1, seed=3)
    inp, var = filter_case(inp, case)
    o, g = _run(inp, var, 1, aa=aa)
    if case == "v=0":  # no filter: s' = s and o' = o exactly
        assert np.array_equal(o.filtered["scales"], inp["scales"]) and np.array_equal(o.filtered["opacities"], inp["opacities"])
    else:
        assert (o.f["coef"] < 1).mean() > 0.9
    assert np.abs(g["scales"]).max() > 0


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("case", ["v>>s^2", "v<<s^2", "s=1e-7"])
def test_chain_vs_autograd_raw(case, aa):
    """raw log-scales and opacity logits: the reference chains exp's and sigmoid's Jacobians after the filter's"""
    inp, _, p = small_scene(P=300, deg=2, seed=8)
    inp, var = filter_case(inp, case, seed=1)
    with np.errstate(divide="ignore"):
        raw = dict(opacities=p.opacity.detach().numpy().copy(), scales=np.log(inp["scales"]).astype(np.float32))
    _run(inp, var, 4, aa=aa, raw=raw)


def test_weight_invariant_float64():
    """o' sqrt(det Sigma') = o sqrt(det Sigma): the filter keeps each Gaussian's integrated 3D weight (rotation drops out)"""
    rng = np.random.RandomState(0)
    s = torch.tensor(np.exp(rng.uniform(-9, 0, (2000, 3))), dtype=torch.float64)
    o = torch.tensor(rng.uniform(0.01, 1, 2000), dtype=torch.float64)
    v = torch.tensor(np.exp(rng.uniform(-12, 0, 2000)), dtype=torch.float64)
    sp, op = filtered_tensors(s, o, v)
    lhs, rhs = op * sp.prod(1), o * s.prod(1)
    assert torch.allclose(lhs, rhs, rtol=1e-12, atol=0)
    # the hand chain's coef (a product of per-axis ratios: dL/do for g_o' = 1) is the same number
    _, do = chain(np.zeros((2000, 3)), np.ones(2000), s.numpy(), o.numpy(), v.numpy())
    assert np.allclose(do, (op / o).numpy(), rtol=1e-12)


def test_filter_params_is_the_ieee_sequence():
    """s' = sqrt(fl(s*s) + v) exactly, and with v = 0 the filter is the identity for scales >= 1e-6"""
    rng = np.random.RandomState(1)
    s = np.exp(rng.uniform(np.log(1e-6), 0, (5000, 3))).astype(np.float32)
    o = rng.uniform(0.01, 1, (5000, 1)).astype(np.float32)
    sp, op, f = filter_params(s, o, np.zeros(5000, np.float32))
    assert np.array_equal(sp, s) and np.array_equal(op, o) and np.all(f["coef"] == 1)
    v = rng.uniform(0, 1e-3, 5000).astype(np.float32)
    sp, op, f = filter_params(s, o, v)
    assert np.array_equal(sp, np.sqrt(np.float32(s * s) + v[:, None]))
    assert (sp >= s).all() and (op <= o).all()


# ---- sampling rate ------------------------------------------------------------------------------------------------------
def axis_camera(W=100, H=80, tanx=0.5, tany=0.5):
    """identity view matrix (camera at the origin looking down +z): tx, ty, tz = x, y, z exactly"""
    return np.eye(4, dtype=np.float32)[None], [tanx], [tany], H, W


def margin_points(W=100, H=80, tanx=0.5, tany=0.5):
    """(means [N,3], expected in-view [N]): points exactly on the +-0.65 W / +-0.65 H margins (in), the next float outward
    (out), tz = 0.2 exactly (out), NaN (out) and the optical axis (in)"""
    fx, fy = np.float32(W) / (np.float32(2) * np.float32(tanx)), np.float32(H) / (np.float32(2) * np.float32(tany))
    limx, limy = np.float32(0.65) * np.float32(W), np.float32(0.65) * np.float32(H)
    pts, want = [], []
    for z in (np.float32(1.0), np.float32(2.5)):
        for lim, f, axis in ((limx, fx, 0), (limy, fy, 1)):
            # the largest float whose projection is still <= lim, and the next one
            x = np.float32(lim / f * z)
            while np.abs(np.float32(np.float32(x / z) * f)) > lim:
                x = np.nextafter(x, np.float32(0))
            while np.abs(np.float32(np.float32(np.nextafter(x, np.float32(np.inf)) / z) * f)) <= lim:
                x = np.nextafter(x, np.float32(np.inf))
            for sign in (1, -1):
                for xx, ok in ((x, True), (np.nextafter(x, np.float32(np.inf)), False)):
                    p = [0.0, 0.0, z]
                    p[axis] = sign * xx
                    pts.append(p)
                    want.append(ok)
    pts += [[0, 0, 0.2], [0, 0, np.nextafter(np.float32(0.2), np.float32(1))], [np.nan] * 3, [0, 0, np.nan], [0, 0, 3.0]]
    want += [False, True, False, False, True]
    return np.asarray(pts, np.float32), np.asarray(want)


def test_sampling_rate_margins_near_plane_and_nan():
    vm, tx, ty, H, W = axis_camera()
    m, want = margin_points()
    rate = sampling_rate(m, vm, tx, ty, H, W)
    assert np.array_equal(rate > 0, want), np.nonzero((rate > 0) != want)
    f = np.float32(W) / (np.float32(2) * np.float32(0.5))
    assert np.array_equal(rate[want], (np.maximum(f, np.float32(H) / np.float32(1.0)) / m[want, 2]).astype(np.float32))


def test_sampling_rate_fold_and_finalize():
    vm, tx, ty, H, W = axis_camera()
    m = np.array([[0, 0, 1], [0, 0, 2], [50, 0, 1], [0, 0, -1]], np.float32)  # the last two are never in view
    rate = sampling_rate(m, vm, tx, ty, H, W)
    assert rate[0] == 100 and rate[1] == 50 and rate[2] == 0 and rate[3] == 0
    # fold order does not matter: a second camera further away changes nothing, and max is commutative
    vm2 = vm.copy()
    vm2[0, 3, 2] = 1.0  # tz = z + 1
    both = sampling_rate(m, np.concatenate([vm, vm2]), tx * 2, ty * 2, H, W)
    assert np.array_equal(both, sampling_rate(m, np.concatenate([vm2, vm]), tx * 2, ty * 2, H, W))
    assert np.array_equal(both, sampling_rate(m, vm2, tx, ty, H, W, max_rate=rate))
    var = finalize(rate)
    assert var.dtype == np.float32
    assert var[0] == np.float32(VARIANCE_SCALE) / np.float32(100 * 100)
    assert var[2] == var[3] == var[1] == np.float32(VARIANCE_SCALE) / np.float32(50 * 50)  # unseen: the widest filter
    assert np.array_equal(finalize(np.zeros(5, np.float32)), np.zeros(5, np.float32))


def test_filter_bounds_the_footprint_at_the_densest_camera():
    """Square pixels, Gaussians on the optical axis: at the camera that attains nu, the smaller eigenvalue of the projected
    covariance before the +0.3 px^2 dilation is >= c px^2 (float32 tolerance), however small the Gaussian"""
    from aa_reference import preprocess_aa
    from oracle.gs_oracle import Oracle
    from util import screen_scene
    n, H, W = 40, 64, 128
    rng = np.random.RandomState(2)
    base = screen_scene(np.full(n, (W - 1) / 2), np.full(n, (H - 1) / 2), rng.uniform(1.0, 6.0, n), 1.0, 0.8, H=H, W=W)
    base = {k: v for k, v in base.items() if k != "cov3D_precomp"}
    base["means3D"][:, :2] = 0.0
    base["scales"] = np.exp(rng.uniform(np.log(1e-6), np.log(1e-2), (n, 3))).astype(np.float32)
    q = rng.randn(n, 4)
    base["rotations"] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    rate = sampling_rate(base["means3D"], base["viewmatrix"][None], [base["tanfovx"]], [base["tanfovy"]], H, W)
    assert (rate > 0).all()
    var = finalize(rate)
    sp, op, _ = filter_params(base["scales"], base["opacities"], var)
    inp = dict(base, scales=sp, opacities=op)
    o = Oracle(threads=1)
    o.forward(**inp)
    f = preprocess_aa(inp, o.state()["cov3d"])
    a, b, c = (f[k].astype(np.float64) for k in ("ca0", "cb", "cc0"))
    lam = 0.5 * (a + c) - np.sqrt(0.25 * (a - c) ** 2 + b * b)
    assert (lam >= VARIANCE_SCALE * (1 - 1e-4)).all(), lam.min()
    assert (lam < VARIANCE_SCALE * 1.5).any()  # the tiny Gaussians sit right at the bound


# ---- C ABI of the render options with the filter pointer ------------------------------------------------------------------
LIB = os.path.join(ROOT, "humangaussian_b200", "libb200gs.so")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        import __graft_entry__ as g
        g.build()
    from humangaussian_b200 import rasterizer
    rasterizer.load_library()
    return rasterizer._lib


def test_render_opts_keeps_the_filter_pointer_at_offset_8():
    from humangaussian_b200.rasterizer import _RenderOpts
    assert C.sizeof(_RenderOpts) == 152 and _RenderOpts.filter3d_var.offset == 8


def test_render_opts_abi5_struct_bytes_rule(lib):
    """struct_bytes 8 (a header before the filter pointer), 16 (a header that ends with it) and >= sizeof are accepted; 0, 4,
    9..15 (a cut pointer) and the sizes between 16 and sizeof (a cut feature block) are argument errors.  The filter with cov3D_precomp is an argument error; the filtered backward needs opacities.  P = 0:
    every call returns before any device work, so this runs without a GPU."""
    from humangaussian_b200 import rasterizer as R
    prm, _, _ = R._make_params(0, 1, 0, 1, 16, 16, 1.0, [1.0], [1.0])
    fake = C.c_void_p(256)  # never dereferenced
    n = C.c_int64(0)
    inputs = [fake, fake, None, fake, fake, fake, None, fake, fake, fake, fake, fake]

    def bwd(opts, det=False, ins=inputs):
        args = [C.byref(prm), opts] + ins + [fake, fake, 1 << 16, fake, 0] + [fake] * 11 + [fake, 1 << 20]
        if det:
            return lib.b200gs_backward_deterministic_opts(*args, fake, 1 << 20, 1 << 16, C.byref(n), None)
        return lib.b200gs_backward_opts(*args, None)

    def fwd(opts, ins=inputs):
        return lib.b200gs_forward_opts(C.byref(prm), opts, *ins[:11], fake, fake, fake, fake, fake, 1, fake, 1, 1, fake, 1,
                                       C.byref(n), None)

    full = C.sizeof(R._RenderOpts)
    for nbytes in (0, 4, *range(9, 16), 17, 24, 64, full - 8, full - 1):
        o = R._RenderOpts(nbytes, 1, 256)
        assert fwd(C.byref(o)) == R.E_ARGS and bwd(C.byref(o)) == R.E_ARGS and bwd(C.byref(o), det=True) == R.E_ARGS, nbytes
    for nbytes in (8, 16, full, full + 64):
        for ptr in (None, 256):
            assert bwd(C.byref(R._RenderOpts(nbytes, 1, ptr))) == R.OK, (nbytes, ptr)
    # cov3D_precomp + filter: an argument error from the forward and the backward; an old 8-byte header never reads the pointer
    cov = list(inputs)
    cov[4] = cov[5] = None
    cov[6] = fake
    with_f = C.byref(R._RenderOpts(16, 0, 256))
    assert fwd(with_f, ins=cov) == R.E_ARGS and bwd(with_f, ins=cov) == R.E_ARGS
    assert bwd(C.byref(R._RenderOpts(8, 0, 256)), ins=cov) == R.OK
    assert bwd(C.byref(R._RenderOpts(16, 0, None)), ins=cov) == R.OK
    no_op = list(inputs)
    no_op[3] = None
    assert bwd(with_f, ins=no_op) == R.E_ARGS


def test_sampling_rate_abi_arguments(lib):
    """b200gs_sampling_rate: more than 64 cameras is a range error, P = 0 is a no-op, missing arguments are errors"""
    from humangaussian_b200 import rasterizer as R
    fake = C.c_void_p(256)
    t = (C.c_float * 65)(*([0.5] * 65))
    assert lib.b200gs_sampling_rate(10, 65, fake, fake, t, t, 16, 16, fake, None) == R.E_RANGE
    assert lib.b200gs_sampling_rate(0, 64, None, None, t, t, 16, 16, None, None) == R.OK
    assert lib.b200gs_sampling_rate(10, 0, fake, fake, t, t, 16, 16, fake, None) == R.E_ARGS
    assert lib.b200gs_sampling_rate(10, 1, fake, fake, None, t, 16, 16, fake, None) == R.E_ARGS
    assert lib.b200gs_sampling_rate(-1, 1, fake, fake, t, t, 16, 16, fake, None) == R.E_ARGS


def test_host_argument_checks_without_gpu():
    """filter_3d's shape / dtype / device and cov3D_precomp are checked on the host before any library call"""
    from humangaussian_b200.rasterizer import _check_filter_3d
    dev = torch.device("cpu")
    ok = torch.zeros(5)
    assert _check_filter_3d(None, 5, dev) is None
    assert _check_filter_3d(ok, 5, dev) is not None
    for bad in (torch.zeros(4), torch.zeros(5, dtype=torch.float64), torch.zeros(5, 1), np.zeros(5, np.float32)):
        with pytest.raises(ValueError):
            _check_filter_3d(bad, 5, dev)
    with pytest.raises(ValueError):
        _check_filter_3d(ok, 5, torch.device("cuda", 0))
    with pytest.raises(ValueError):
        _check_filter_3d(ok, 5, dev, cov3D_precomp=torch.zeros(5, 6))
