"""CPU: the composed option-matrix reference (tests/option_matrix_reference.py) and the case table of
tests/test_gpu_option_matrix.py, without a GPU.

  1. with one feature on, the composed reference is the per-feature reference: normal_reference.reference_grads,
     geometry_reference.reference_grads and absgrad_reference.absgrad, to 1e-12 relative;
  2. the extended per-pixel Jacobian (normal and depth-second-moment terms on) sums over the pixels to the signed means2D
     gradient of reverse mode, and a central finite difference of the per-pixel losses gives its means2D_abs;
  3. the case table covers every pair of axis values, every backward variant at least twice and at least once with three
     views and per-view means, and no illegal combination."""
import itertools

import numpy as np
import torch

import absgrad_reference as AR
import geometry_reference as GR
import normal_reference as NR
import option_matrix_reference as OR
from test_gpu_option_matrix import CASES, FWD_VARIANTS, Case, forward_variants, legal
from util import grad_images, small_scene


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _scene(deg=1, seed=3, P=30, H=16, W=24):
    inp, _, p = small_scene(P=P, deg=deg, seed=seed, H=H, W=W)
    return inp, p


def _raw(p, inp):
    raw = dict(opacities=p.opacity.detach().numpy().copy(), scales=p.scaling.detach().numpy().copy(),
               rotations=(p.rotation.detach().numpy() * 1.3).astype(np.float32))
    s, q = NR.activate(raw["scales"], raw["rotations"], raw=True)
    return raw, dict(inp, scales=s, rotations=q)


# ---- 1. one feature on: the per-feature references --------------------------------------------------------------------------
def test_reduces_to_normal_reference():
    inp, p = _scene()
    gimg = grad_images(16, 24, 1)
    gN = np.random.RandomState(2).randn(3, 16, 24).astype(np.float32)
    for raw, iv, opts in ((None, inp, {}), (*_raw(p, inp), dict(antialiasing=True)),
                          (None, inp, dict(filter_3d=np.full(30, 1e-3, np.float32)))):
        ref, _ = NR.reference_grads(iv, gimg, gN, raw=raw, **opts)
        g = OR.grads([iv], [gimg], gN=gN[None], raw=raw, **opts)
        for k, r in ref.items():
            assert _rel(g[k], r) < 1e-12, (k, opts, raw is None)


def test_reduces_to_geometry_reference():
    inp, p = _scene(deg=2, seed=4)
    gimg = grad_images(16, 24, 3)
    rng = np.random.RandomState(4)
    gM2, gMed = rng.randn(16, 24).astype(np.float32), rng.randn(16, 24).astype(np.float32)
    for raw, iv, opts in ((None, inp, {}), (*_raw(p, inp), {}),
                          (None, dict(inp, scale_modifier=0.7), dict(antialiasing=True, filter_3d=np.full(30, 1e-3, np.float32)))):
        ref, _ = GR.reference_grads(iv, gimg, gM2, gMed, raw=raw, **opts)
        g = OR.grads([iv], [gimg], gM2=gM2[None], gMed=gMed[None], raw=raw, **opts)
        for k, r in ref.items():
            assert _rel(g[k], r) < 1e-12, (k, opts, raw is None)
        im = OR.images([iv], geometry=True, **opts)
        r = GR.reference_images(iv, **opts)
        for k in ("median", "depth2", "median_pos"):
            assert np.array_equal(im[k][0].reshape(r[k].shape), r[k]), k


def test_reduces_to_absgrad_reference_and_three_views():
    inp, _ = _scene(deg=0, seed=5)
    from humangaussian_b200.cameras import sample_orbit_cameras
    import math
    inps = [dict(inp, viewmatrix=c.world_view_transform.numpy(), projmatrix=c.full_proj_transform.numpy(),
                 campos=c.camera_center.numpy(), tanfovx=math.tan(c.FoVx * 0.5), tanfovy=math.tan(c.FoVy * 0.5))
            for c in sample_orbit_cameras(3, 16, 24, seed=5)]
    rng = np.random.RandomState(6)
    means = np.stack([inp["means3D"] + (0.02 * rng.randn(30, 3)).astype(np.float32) for _ in range(3)])
    gimgs = [grad_images(16, 24, 20 + v) for v in range(3)]
    a = OR.means2D_abs(inps, gimgs, means=means)
    for v in range(3):
        r, s, _ = AR.absgrad(dict(inps[v], means3D=means[v]), gimgs[v])
        assert _rel(a[v], r) < 1e-12
    # per-view means: each view's gradients are that view's own, and shared parameters sum over the views
    g = OR.grads(inps, gimgs, means=means)
    for v in range(3):
        gv = OR.grads([inps[v]], [gimgs[v]], means=means[v:v + 1])
        assert _rel(g["means3D"][v], gv["means3D"][0]) < 1e-12 and _rel(g["means2D"][v], gv["means2D"][0]) < 1e-12
    parts = [OR.grads([dict(inps[v], means3D=means[v])], [gimgs[v]]) for v in range(3)]
    for k in ("opacities", "shs", "scales", "rotations"):
        assert _rel(g[k], sum(p_[k] for p_ in parts)) < 1e-12, k


# ---- 2. the extended Jacobian -----------------------------------------------------------------------------------------------
def test_jacobian_sums_to_the_signed_gradient():
    inp, _ = _scene(deg=3, seed=6, P=40)
    inp["scale_modifier"] = 0.7
    H, W = 16, 24
    gimg = grad_images(H, W, 7)
    rng = np.random.RandomState(7)
    gN, gM2, gMed = rng.randn(3, H, W), rng.randn(H, W), rng.randn(H, W)
    opts = dict(antialiasing=True)  # (no 3D filter: the Jacobian forms it in float32, as the kernels do, the gradients in float64)
    J, radii = AR.per_pixel_jacobian(inp, gimg, gN=gN, gM2=gM2, **opts)
    g = OR.grads([inp], [gimg], gN=gN[None], gM2=gM2[None], gMed=gMed[None], **opts)
    assert (radii > 0).sum() > 20
    assert _rel(J.sum(2), g["means2D"][0][:, :2]) < 1e-10
    # and the normal and z^2 terms matter: without them the sums differ
    J0, _ = AR.per_pixel_jacobian(inp, gimg, **opts)
    assert _rel(J0.sum(2), g["means2D"][0][:, :2]) > 1e-3


def test_finite_difference_matches_means2D_abs():
    """6 Gaussians on 16 x 16, opacities below the 0.99 clamp (whose straight-through gradient a difference cannot see)"""
    inp, _ = _scene(deg=1, seed=8, P=6, H=16, W=16)
    inp["opacities"] = np.minimum(inp["opacities"], 0.8).astype(np.float32)
    rng = np.random.RandomState(9)
    gimg = grad_images(16, 16, 9)
    gN, gM2 = rng.randn(3, 16, 16), rng.randn(16, 16)
    a, s, radii = AR.absgrad(inp, gimg, gN=gN, gM2=gM2)
    assert (radii > 0).sum() >= 4
    losses, _, _ = AR.pixel_losses(inp, gimg, gN=gN, gM2=gM2)
    h = 1e-7
    fd = np.zeros((6, 3))
    fs = np.zeros((6, 3))
    with torch.no_grad():
        for k in range(6):
            for c in range(2):
                e = torch.zeros(6, 3, dtype=torch.float64)
                e[k, c] = h
                d = ((losses(e) - losses(-e)) / (2 * h)).numpy()
                fd[k, c], fs[k, c] = np.abs(d).sum(), d.sum()
    assert np.abs(a).max() > 1e-2
    assert _rel(fd, a) < 1e-5 and _rel(fs, s) < 1e-5


# ---- 3. the case table ------------------------------------------------------------------------------------------------------
AXES = dict(det=(0, 1), abs=(0, 1), nrm=(0, 1), geo=(0, 1), colour=("sh0", "sh1", "sh3", "pre"), params=("act", "raw"),
            cov=("sr", "cov"), aa=(0, 1), f3d=(0, 1), V=(1, 3), means=("shared", "per_view"), mod=(1.0, 0.7),
            scene=("small", "dense", "flush", "edge"))


def test_case_table_covers_every_pair():
    assert set(Case._fields) == set(AXES) and 30 <= len(CASES) <= 60
    assert all(legal(c) for c in CASES), [c for c in CASES if not legal(c)]
    for c in CASES:
        assert all(getattr(c, k) in v for k, v in AXES.items()), c
    pairs = lambda rows: {(a, getattr(c, a), b, getattr(c, b)) for c in rows for a, b in itertools.combinations(Case._fields, 2)}
    every_legal = [c for c in itertools.starmap(Case, itertools.product(*(AXES[k] for k in Case._fields))) if legal(c)]
    missing = pairs(every_legal) - pairs(CASES)
    assert not missing, f"no case has {sorted(missing, key=str)[:5]}"


def test_case_table_variants_and_exclusions():
    for v in itertools.product((0, 1), repeat=4):
        rows = [c for c in CASES if (c.det, c.abs, c.nrm, c.geo) == v]
        assert len(rows) >= 2, v
        assert any(c.V == 3 and c.means == "per_view" for c in rows), v
    # illegal pairs: normals or the 3D filter with cov3D_precomp
    assert not any(c.cov == "cov" and (c.nrm or c.f3d) for c in CASES)
    assert not legal(CASES[0]._replace(cov="cov", nrm=1)) and not legal(CASES[0]._replace(cov="cov", f3d=1, nrm=0))
    # the forward matrix: contribution never with normals or geometry, normals never with cov3D_precomp, all five kernels run
    seen = set()
    for c in CASES:
        for v in forward_variants(c):
            n, g, ctb = FWD_VARIANTS[v]
            assert not (ctb and (n or g)) and not (n and c.cov == "cov")
            seen.add(v)
    assert seen == set(FWD_VARIANTS)
