"""CPU: the absolute screen-space gradient's float64 reference (tests/absgrad_reference.py) against per-pixel reverse-mode
autograd and central finite differences, its bounds, and the absgrad C ABI on P = 0 calls (no device work)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import absgrad_reference as AR
from util import ROOT, close, grad_images, small_scene


def _tiny(seed=5, deg=1):
    inp, _, _ = small_scene(P=14, deg=deg, seed=seed, H=20, W=36)
    return inp, grad_images(20, 36, seed)


def _dense_losses(inp, gimg):
    """L(m2d) -> per-pixel losses [H*W] through oracle/dense_ref.py (float64), with the oracle's integer decisions"""
    from oracle.dense_ref import dense_render
    st, radii = AR._state(inp)
    ids = np.nonzero(radii > 0)[0]
    order = ids[np.lexsort((ids, st["depths"][ids]))]
    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    H, W = inp["image_height"], inp["image_width"]
    kw = dict(means3D=t64(inp["means3D"]), opacities=t64(inp["opacities"]), viewmatrix=t64(inp["viewmatrix"]),
              projmatrix=t64(inp["projmatrix"]), campos=t64(inp["campos"]), bg=t64(inp["bg"]), H=H, W=W, tanfovx=inp["tanfovx"],
              tanfovy=inp["tanfovy"], radii=radii, rect=st["rect"], order=order, sh_degree=inp["sh_degree"], shs=t64(inp["shs"]),
              scales=t64(inp["scales"]), rotations=t64(inp["rotations"]))
    gC, gD, gA = (t64(g) for g in gimg)

    def losses(m2d):
        c, d, a, _ = dense_render(means2D=m2d, **kw)
        return ((c * gC).sum(0) + (d * gD)[0] + (a * gA)[0]).reshape(-1)
    return losses, radii


def test_reference_equals_per_pixel_reverse_mode_and_finite_differences():
    inp, gimg = _tiny()
    J, radii = AR.per_pixel_jacobian(inp, gimg)
    assert (radii > 0).sum() >= 10
    losses, _ = _dense_losses(inp, gimg)
    P, N = J.shape[0], J.shape[2]
    m0 = torch.zeros(P, 3, dtype=torch.float64, requires_grad=True)
    Lv = losses(m0)
    brute = np.zeros_like(J)
    for p in range(N):  # brute force: one reverse pass per pixel
        (g,) = torch.autograd.grad(Lv[p], m0, retain_graph=True)
        brute[:, :, p] = g[:, :2].numpy()
    assert np.abs(J - brute).max() <= 1e-12 * max(1.0, np.abs(brute).max())
    # central differences of every pixel's loss, per (Gaussian, component)
    h = 1e-7
    with torch.no_grad():
        for k in np.nonzero(radii > 0)[0][:6]:
            for c in range(2):
                e = torch.zeros(P, 3, dtype=torch.float64)
                e[k, c] = h
                fd = ((losses(e) - losses(-e)) / (2 * h)).numpy()
                assert np.abs(fd - J[k, c]).max() <= 1e-5 * max(1.0, np.abs(J[k, c]).max()), (k, c)


@pytest.mark.parametrize("deg", [0, 3])
def test_reference_bounds_and_signed_sum(deg):
    """sum |g_p| >= |sum g_p|, strictly somewhere; sum_p g_p is dense_ref's own reverse-mode dL/dmeans2D, and the float32
    oracle's within the float32-vs-float64 tolerance of tests/test_oracle_autograd.py"""
    from oracle.gs_oracle import Oracle
    inp, _, _ = small_scene(P=40, deg=deg, seed=deg + 2, H=24, W=40)
    gimg = grad_images(24, 40, deg)
    a, s, radii = AR.absgrad(inp, gimg)
    assert (a >= np.abs(s) - 1e-12).all() and (a[radii > 0, :2] > np.abs(s[radii > 0, :2]) * 1.01).mean() > 0.5
    assert (a[radii == 0] == 0).all() and (a[:, 2] == 0).all()
    losses, _ = _dense_losses(inp, gimg)
    m0 = torch.zeros(len(radii), 3, dtype=torch.float64, requires_grad=True)
    losses(m0).sum().backward()
    assert np.allclose(s[:, :2], m0.grad[:, :2].numpy(), rtol=1e-10, atol=1e-12)
    o = Oracle(threads=1)
    o.forward(**inp)
    ok, worst = close(o.backward(*gimg)["means2D"], s, atol=1e-4, rtol=1e-3)
    assert ok, worst


# ---- C ABI -------------------------------------------------------------------------------------------------------------
def _lib(path):
    if not os.path.exists(path):
        import __graft_entry__ as g
        g.build()
    return C.CDLL(path)


def _abs_call(L, det, m2d_abs=True, abs_partials=True, abs_bytes=8 * 16, **fields):
    """one P = 0 call of b200gs_backward_opts / b200gs_backward_deterministic_opts with the absolute gradients in the options
    (and any other option fields given): every device pointer is a host dummy (nothing is dereferenced for P = 0)"""
    from humangaussian_b200 import rasterizer as R
    prm, _tx, _ty = R._make_params(0, 1, 0, 1, 8, 8, 1.0, [1.0], [1.0])
    buf = (C.c_float * 64)()
    d = C.cast(buf, C.c_void_p)
    n = C.c_int64(-1)
    o = R._RenderOpts(C.sizeof(R._RenderOpts), 0, None)
    o.dL_dmeans2D_abs = d if m2d_abs else None
    if det:
        o.abs_partials, o.abs_partials_bytes = (d if abs_partials else None), abs_bytes
    for k, v in fields.items():
        setattr(o, k, v)
    grads = [d] * 8  # dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors (NULL below), dL_dopacity, dL_dscales, dL_drots, dL_dcov3D
    grads[3], grads[7] = None, None
    common = [C.byref(prm), C.byref(o), d, d, None, d, d, d, None, d, d, d, d, d, d, d, C.c_int64(1), d, C.c_int64(0), None, None,
              None, *grads, d, C.c_size_t(256)]
    if not det:
        return L.b200gs_backward_opts(*common, None)
    return L.b200gs_backward_deterministic_opts(*common, d, C.c_size_t(256), C.c_int64(16), C.byref(n), None)


def _fwd_call(L, **fields):
    """one P = 0 b200gs_forward_opts call with the given option fields, for argument errors found before any device work"""
    from humangaussian_b200 import rasterizer as R
    prm, _tx, _ty = R._make_params(0, 1, 0, 1, 8, 8, 1.0, [1.0], [1.0])
    buf = (C.c_float * 64)()
    d = C.cast(buf, C.c_void_p)
    n = C.c_int64(-1)
    o = R._RenderOpts(C.sizeof(R._RenderOpts), 0, None)
    for k, v in fields.items():
        setattr(o, k, v)
    ins = [d, d, None, d, d, d, None, d, d, d, d]  # means3D .. campos, as in _abs_call
    return L.b200gs_forward_opts(C.byref(prm), C.byref(o), *ins, d, d, d, d, d, C.c_size_t(1 << 20), d, C.c_size_t(1 << 20),
                                 C.c_int64(1 << 16), d, C.c_size_t(1 << 20), C.byref(n), None)


def test_abi_absgrad_options_on_empty_scenes():
    from humangaussian_b200 import rasterizer as R
    L = _lib(os.path.join(ROOT, "humangaussian_b200", "libb200gs.so"))
    for det in (False, True):
        assert _abs_call(L, det) == R.OK
        assert _abs_call(L, det, m2d_abs=False) == R.OK  # no dL_dmeans2D_abs: the call without absolute gradients
    assert _abs_call(L, True, abs_partials=False) == R.E_ARGS
    assert _abs_call(L, True, abs_bytes=8 * 16 - 1) == R.E_BUFFER  # 8 bytes per partial of partial_capacity = 16
    assert _abs_call(L, True, m2d_abs=False, abs_partials=False) == R.OK  # abs_partials is read with dL_dmeans2D_abs only


def test_abi_option_combinations_on_empty_scenes():
    """The rules of b200gs_render_opts that the C layer checks before any device work: contribution scores with normals or
    geometry, dL_dnormal without gauss_normals, and a geometry gradient without median_pos are argument errors."""
    from humangaussian_b200 import rasterizer as R
    L = _lib(os.path.join(ROOT, "humangaussian_b200", "libb200gs.so"))
    ws = (C.c_uint64 * 4)()
    aligned = (C.c_float * 64)()  # 16-byte aligned host memory stands in for the device workspaces
    p = C.cast(aligned, C.c_void_p)
    contrib = dict(weight_sum=C.cast(ws, C.c_void_p), weight_max=p, touches=p)
    assert _fwd_call(L, **contrib, gauss_normals=p, out_normal=p) == R.E_ARGS
    assert _fwd_call(L, **contrib, median_pos=p, out_median=p, out_depth2=p) == R.E_ARGS
    assert _fwd_call(L, weight_sum=C.cast(ws, C.c_void_p)) == R.E_ARGS  # an accumulator without the other two
    for det in (False, True):
        assert _abs_call(L, det, dL_dnormal=p) == R.E_ARGS
        assert _abs_call(L, det, dL_dnormal=p, gauss_normals=p, normal_wn=p, nrm_partials=p, nrm_partials_bytes=1 << 20) == R.OK
        for grad in ("dL_dmedian", "dL_ddepth2"):
            assert _abs_call(L, det, **{grad: p}) == R.E_ARGS
            assert _abs_call(L, det, **{grad: p}, median_pos=p) == R.OK


def test_abi_classic_comparator_rejects_absgrad_options():
    from humangaussian_b200 import rasterizer as R
    L = _lib(os.path.join(ROOT, "baseline", "libb200gs_classic.so"))
    for det in (False, True):
        assert _abs_call(L, det) == R.E_UNSUPPORTED
