"""GPU: the absolute screen-space gradient (means2D_abs=) against its float64 reference (tests/absgrad_reference.py), and its
properties, in the atomic and the deterministic backward.

  1. grads_agree with the reference at the float32-vs-float64 tolerance of the other autograd checks (1e-4 abs, 1e-3 rel):
     degrees 0-3, dense-opaque, a 3-view batch, raw parameters, antialiasing, the 3D filter, cov3D_precomp, and screen-space
     scenes whose patches stage 1, 15, 16, 17, 31, 32, 33 and 64 hits, and partial patches at the image edge;
  2. abs >= |signed|, equality for one-signed per-pixel terms, zero where radii == 0, z = 0;
  3. every other output and gradient unchanged (byte for byte in deterministic mode), deterministic reruns byte-identical,
     2x the image gradient gives exactly 2x, its negation identical bytes; atomic and deterministic agree;
  4. the same properties on the full-size scene (300 k, degree 3, 1024^2, 8 views), where no float64 reference exists;
  5. a 20-step packed training loop densifying on the absolute statistic, reproducible under deterministic algorithms."""
import contextlib
import math

import numpy as np
import pytest
import torch

import absgrad_reference as AR
from util import grad_images, grads_agree, screen_scene, small_scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REF_TOL = dict(atol=1e-4, rtol=1e-3)
KEYS = ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp")


@contextlib.contextmanager
def deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _views(inps):
    """stack per-view camera fields of single-view inputs into rasterize_views' keywords"""
    g = lambda k: torch.stack([torch.as_tensor(np.asarray(i[k], np.float32)) for i in inps]).to(DEV)
    i0 = inps[0]
    return dict(viewmatrices=g("viewmatrix").reshape(-1, 4, 4), projmatrices=g("projmatrix").reshape(-1, 4, 4),
                camposs=g("campos").reshape(-1, 3), tanfovx=[i["tanfovx"] for i in inps], tanfovy=[i["tanfovy"] for i in inps],
                image_height=i0["image_height"], image_width=i0["image_width"], bg=torch.tensor(i0["bg"], device=DEV),
                sh_degree=i0.get("sh_degree", 0), scale_modifier=i0.get("scale_modifier", 1.0))


def _run(inps, gimgs, absgrad=True, det=False, raw=None, scale=1.0, **opts):
    """rasterize_views over the views `inps` (one Gaussian set) with image gradients gimgs * scale; returns a dict of numpy
    arrays: images, radii, every parameter gradient, means2D's and (absgrad) means2D_abs's .grad.  raw: dict of raw
    opacities / scales / rotations to pass instead (raw=True)."""
    from humangaussian_b200.rasterizer import rasterize_views
    i0 = inps[0]
    t = {k: torch.tensor(i0[k], device=DEV, requires_grad=True) for k in KEYS if i0.get(k) is not None}
    if raw is not None:
        for k, v in raw.items():
            t[k] = torch.tensor(v, device=DEV, requires_grad=True)
    V, P = len(inps), i0["means3D"].shape[0]
    m2d = torch.zeros(V, P, 3, device=DEV, requires_grad=True)
    m2a = torch.zeros(V, P, 3, device=DEV, requires_grad=True) if absgrad else None
    with deterministic(det):
        c, r, d, a = rasterize_views(means2D=m2d, means2D_abs=m2a, raw=raw is not None, **{k: t[k] for k in t}, **_views(inps), **opts)
        gC, gD, gA = (torch.tensor(np.stack([g[j] for g in gimgs]), device=DEV) * scale for j in range(3))
        torch.autograd.backward([c, d, a], [gC, gD, gA])
    out = dict(color=c, depth=d, alpha=a, radii=r, means2D=m2d.grad, **{k: v.grad for k, v in t.items()})
    if absgrad:
        out["means2D_abs"] = m2a.grad
    return {k: v.detach().cpu().numpy() for k, v in out.items()}


def _reference(inps, gimgs, **kw):
    return np.stack([AR.absgrad(i, g, **kw)[0] for i, g in zip(inps, gimgs)])


def _check(inps, gimgs, ref_kw=None, raw=None, **opts):
    ref = _reference(inps, gimgs, **(ref_kw or {}))
    for det in (False, True):
        g = _run(inps, gimgs, det=det, raw=raw, **opts)
        ok, msg = grads_agree(g["means2D_abs"].reshape(-1, 3), ref.reshape(-1, 3), **REF_TOL)
        assert ok, f"deterministic={det}: means2D_abs vs float64 reference: {msg}"
        _properties(g)
    return g


def _properties(g):
    a, s, radii = g["means2D_abs"], g["means2D"], g["radii"]
    assert np.isfinite(a).all()
    assert (a[..., :2] >= np.abs(s[..., :2]) * (1 - 1e-4) - 1e-6).all(), "abs < |signed|"
    assert (a[radii == 0] == 0).all() and (a[..., 2] == 0).all()


# ---- 1. against the float64 reference ------------------------------------------------------------------------------------
def _small(deg, seed=None, P=60, H=32, W=48, **kw):
    inp, _, p = small_scene(P=P, deg=deg, seed=deg if seed is None else seed, H=H, W=W, **kw)
    return inp, p


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_small_scenes(deg):
    inp, _ = _small(deg)
    _check([inp], [grad_images(32, 48, deg)])


def test_dense_opaque_scene():
    inp, _ = _small(1, seed=9, P=80, H=32, W=32, dist=1.3)
    inp["opacities"] = np.clip(inp["opacities"] * 8, 0, 0.99999).astype(np.float32)
    inp["scales"] = (inp["scales"] * 2.0).astype(np.float32)
    _check([inp], [grad_images(32, 32, 1)])


def test_three_view_batch():
    from humangaussian_b200.cameras import sample_orbit_cameras
    inp, _ = _small(2, P=50)
    inps = []
    for cam in sample_orbit_cameras(3, 32, 48, seed=5):
        inps.append(dict(inp, viewmatrix=cam.world_view_transform.cpu().numpy(), projmatrix=cam.full_proj_transform.cpu().numpy(),
                         campos=cam.camera_center.cpu().numpy(), tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5)))
    _check(inps, [grad_images(32, 48, 10 + v) for v in range(3)])


def test_raw_parameters():
    inp, p = _small(1, seed=7)
    raw = dict(opacities=p.opacity.detach().numpy().copy(), scales=p.scaling.detach().numpy().copy(),
               rotations=p.rotation.detach().numpy().copy())
    _check([inp], [grad_images(32, 48, 7)], raw=raw)


def test_antialiasing():
    inp, _ = _small(1, seed=11)
    _check([inp], [grad_images(32, 48, 11)], ref_kw=dict(antialiasing=True), antialiasing=True)


def test_filter_3d():
    from test_gpu_filter3d import _var_for
    inp, _ = _small(3, seed=12)
    var = _var_for(inp, seed=12)
    _check([inp], [grad_images(32, 48, 12)], ref_kw=dict(filter_3d=var), filter_3d=torch.tensor(var, device=DEV))


def test_cov3D_precomp():
    from oracle.gs_oracle import Oracle
    inp, _ = _small(0, seed=3)
    o = Oracle(threads=1)
    o.forward(**inp)
    st = o.state()
    inp2 = {k: v for k, v in inp.items() if k not in ("shs", "scales", "rotations")}
    inp2["colors_precomp"] = (np.abs(st["rgb"]) + 0.1).astype(np.float32)
    inp2["cov3D_precomp"] = st["cov3d"].copy()
    _check([inp2], [grad_images(32, 48, 3)])


def _stack(x, y, n, z0, opacity=0.05):
    return dict(px=np.full(n, x), py=np.full(n, y), depth=z0 + 1e-3 * np.arange(n), opacity=np.full(n, opacity))


def _cat(parts):
    return {k: np.concatenate([p[k] for p in parts]) for k in ("px", "py", "depth", "opacity")}


def test_flush_boundaries():
    """stacks of 1, 15, 16, 17, 31, 32, 33 and 64 hits, each in patch 0 of its own tile (n mod 16 = 0, 1, 15 and the chunk
    edges); sigma 0.6 px so that every hit covers several pixels of its patch"""
    counts = (1, 15, 16, 17, 31, 32, 33, 64)
    parts = [_stack(16 * i + 3.5, 1.5, n, 1.0 + i) for i, n in enumerate(counts)]
    g = _cat(parts)
    inp = screen_scene(g["px"], g["py"], g["depth"], 0.6, g["opacity"], H=16, W=128)
    _check([inp], [grad_images(16, 128, 41)])


def test_partial_edge_patches():
    """stacks in the partial patches of a 123x61 image: cols 120-122 and row 60"""
    parts = [_stack(121.0, 9.5, 17, 1.0), _stack(121.0, 60.45, 15, 2.0), _stack(51.5, 60.45, 33, 3.0), _stack(3.5, 60.45, 1, 4.0)]
    g = _cat(parts)
    inp = screen_scene(g["px"], g["py"], g["depth"], 0.6, g["opacity"], H=61, W=123)
    _check([inp], [grad_images(61, 123, 42)])


# ---- 2./3. properties ----------------------------------------------------------------------------------------------------
def test_one_signed_terms_give_equality():
    """Axis-aligned, disjoint Gaussians centred off the left edge (every pixel has dx < 0) or off the top edge (dy < 0), on a
    black background, with non-negative colour and alpha weights: dL/dalpha > 0 at every pixel, so each Gaussian's per-pixel
    x terms (left) or y terms (top) share one sign and abs = |signed| for that component."""
    py_left = np.array([8.0, 24.0, 40.0, 56.0])
    px_top = np.array([24.0, 56.0, 88.0])
    px = np.concatenate([np.full(4, -2.5), px_top])
    py = np.concatenate([py_left, np.full(3, -2.5)])
    inp = screen_scene(px, py, 1.0 + 0.01 * np.arange(7), 3.0, 0.5, H=64, W=112)
    inp["bg"] = np.zeros(3, np.float32)
    H, W = 64, 112
    gimg = (np.ones((3, H, W), np.float32), np.zeros((1, H, W), np.float32), np.ones((1, H, W), np.float32))
    for det in (False, True):
        g = _run([inp], [gimg], det=det)
        a, s = g["means2D_abs"][0], g["means2D"][0]
        assert (g["radii"][0] > 0).all()
        for rows, c in ((slice(0, 4), 0), (slice(4, 7), 1)):
            assert (np.abs(s[rows, c]) > 1e-3).all()
            assert np.allclose(a[rows, c], np.abs(s[rows, c]), rtol=1e-4, atol=1e-6), (c, a[rows, c], s[rows, c])
        _properties(g)


def _byte_checks(inps, gimgs, full=False):
    """outputs unchanged by absgrad; deterministic reruns, 2x and -1x image gradients; atomic vs deterministic"""
    crit = dict(min_rows=1.0 - 1e-4, row_cap=4.0) if full else {}
    on = _run(inps, gimgs, det=True)
    off = _run(inps, gimgs, det=True, absgrad=False)
    for k in off:
        assert off[k].tobytes() == on[k].tobytes(), f"deterministic {k} changes with absgrad on"
    again = _run(inps, gimgs, det=True)
    assert all(again[k].tobytes() == on[k].tobytes() for k in on), "deterministic reruns differ"
    two = _run(inps, gimgs, det=True, scale=2.0)
    assert two["means2D_abs"].tobytes() == (2 * on["means2D_abs"]).tobytes()
    neg = _run(inps, gimgs, det=True, scale=-1.0)
    assert neg["means2D_abs"].tobytes() == on["means2D_abs"].tobytes()
    at_on = _run(inps, gimgs)
    at_off = _run(inps, gimgs, absgrad=False)
    for k in ("color", "depth", "alpha", "radii"):
        assert at_on[k].tobytes() == at_off[k].tobytes() == on[k].tobytes(), k
    for k in at_off:
        if k not in ("color", "depth", "alpha", "radii"):
            a_ = at_on[k].reshape(-1, 3) if k == "means2D" else at_on[k].reshape(at_on[k].shape[0], -1)
            b_ = at_off[k].reshape(a_.shape)
            ok, msg = grads_agree(a_, b_, **crit)
            assert ok, f"atomic {k} with absgrad on vs off: {msg}"
    ok, msg = grads_agree(at_on["means2D_abs"].reshape(-1, 3), on["means2D_abs"].reshape(-1, 3), **crit)
    assert ok, f"atomic vs deterministic means2D_abs: {msg}"
    _properties(on)
    _properties(at_on)


def test_outputs_unchanged_and_deterministic_bytes():
    from humangaussian_b200.cameras import sample_orbit_cameras
    inp, _ = _small(3, P=600, H=72, W=104)
    inps = []
    for cam in sample_orbit_cameras(3, 72, 104, seed=6):
        inps.append(dict(inp, viewmatrix=cam.world_view_transform.cpu().numpy(), projmatrix=cam.full_proj_transform.cpu().numpy(),
                         campos=cam.camera_center.cpu().numpy(), tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5)))
    _byte_checks(inps, [grad_images(72, 104, 20 + v) for v in range(3)])


def test_full_size_300k_deg3_1024_8_views():
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.scene import sample_ply_scene
    p = sample_ply_scene(300000, 3)
    with torch.no_grad():
        base = dict(means3D=p.get_xyz.cpu().numpy().copy(), opacities=p.get_opacity.cpu().numpy().copy(),
                    shs=p.get_features.cpu().numpy().copy(), scales=p.get_scaling.cpu().numpy().copy(),
                    rotations=p.get_rotation.cpu().numpy().copy(), sh_degree=3, bg=np.array([0.1, 0.4, 0.7], np.float32),
                    image_height=1024, image_width=1024, scale_modifier=1.0)
    inps = [dict(base, viewmatrix=c.world_view_transform.cpu().numpy(), projmatrix=c.full_proj_transform.cpu().numpy(),
                 campos=c.camera_center.cpu().numpy(), tanfovx=math.tan(c.FoVx * 0.5), tanfovy=math.tan(c.FoVy * 0.5))
            for c in sample_orbit_cameras(64, 1024, 1024, seed=1000)[:8]]
    _byte_checks(inps, [grad_images(1024, 1024, 30 + v) for v in range(8)], full=True)


# ---- 5. training ---------------------------------------------------------------------------------------------------------
def _train(seed):
    """20 packed raw steps with PackedAdam; the densify after step 10 plans on the absolute statistic"""
    from humangaussian_b200 import dist as D
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.densify import DensifyStats, add_densification_stats, densify_and_prune_packed
    from humangaussian_b200.optim import PackedAdam, expon_lr_func
    from humangaussian_b200.rasterizer import rasterize_views_packed
    from humangaussian_b200.renderer import stack_cameras
    _, _, sc = small_scene(P=3001, deg=3, seed=seed)
    K, H = 16, 64
    raw = dict(xyz=sc.xyz, scaling=sc.scaling, rotation=sc.rotation, opacity=sc.opacity,
               features=torch.cat((sc.features_dc, sc.features_rest), 1))
    flat = D.pack({k: v.detach().float().to(DEV).contiguous() for k, v in raw.items()}).requires_grad_(True)
    lrs = dict(xyz=0.00016, f_dc=0.0125, f_rest=0.0125 / 20.0, opacity=0.01, scaling=0.005, rotation=0.001)
    sched = expon_lr_func(lr_init=0.00016, lr_final=0.0000016, lr_delay_mult=0.01, max_steps=30000)
    opt = PackedAdam(flat, 3001, K, lrs, xyz_scheduler=sched)
    vm, pm, cp, tx, ty = stack_cameras(sample_orbit_cameras(4, H, H, seed=3), DEV)
    bg = torch.tensor([0.8, 0.5, 0.2], device=DEV)
    stats = DensifyStats.zeros(opt.P, DEV)
    for it in range(20):
        opt.update_learning_rate(it)
        m2d = torch.zeros(4, opt.P, 3, device=DEV, requires_grad=True)
        m2a = torch.zeros(4, opt.P, 3, device=DEV, requires_grad=True)
        color, radii, _, _ = rasterize_views_packed(opt.packed, opt.P, K, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx,
                                                    tanfovy=ty, image_height=H, image_width=H, bg=bg, sh_degree=3, means2D=m2d,
                                                    means2D_abs=m2a, raw=True)
        loss = (color - bg.view(1, 3, 1, 1)).square().mean()
        loss.backward()
        assert math.isfinite(loss.item()) and torch.isfinite(opt.packed.grad).all() and torch.isfinite(m2a.grad).all()
        assert (m2a.grad[..., :2] >= m2d.grad[..., :2].abs() * (1 - 1e-4) - 1e-6).all()
        add_densification_stats(stats, m2a.grad, radii)
        opt.step()
        opt.zero_grad()
        if it == 9:
            thr = float(torch.quantile((stats.xyz_gradient_accum / stats.denom.clamp_min(1)).flatten(), 0.8))
            densify_and_prune_packed(opt, stats, thr, 0.005, 1.0, None, generator=torch.Generator(device=DEV).manual_seed(7))
    st = opt.state[opt.packed]
    assert torch.isfinite(opt.packed).all()
    return dict(P=opt.P, packed=opt.packed.detach().clone(), exp_avg=st["exp_avg"].clone(), exp_avg_sq=st["exp_avg_sq"].clone(),
                accum=stats.xyz_gradient_accum.clone(), denom=stats.denom.clone(), max_radii2D=stats.max_radii2D.clone())


def test_training_loop_densifies_on_absgrad_and_reproduces():
    a = _train(4)
    assert a["P"] != 3001
    with deterministic():
        b, c = _train(4), _train(4)
    assert b["P"] == c["P"] != 3001
    for k in b:
        if k != "P":
            assert b[k].cpu().numpy().tobytes() == c[k].cpu().numpy().tobytes(), f"training loop: {k} differs between runs"
