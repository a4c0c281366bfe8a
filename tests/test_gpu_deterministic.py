"""GPU: the deterministic backward (torch.use_deterministic_algorithms(True)).

Under the flag the backward blend stores every (instance, patch) partial sum into its own slot and a reduce adds each
(view, Gaussian)'s partials in a fixed order (its tiles in emission order, patches ascending), so the gradients depend on
the forward state alone.  Checked here, with the flag on (fixture `deterministic`, warn_only=True, restored afterwards):
  1. two forward + backward runs are byte-identical in every parameter gradient, dL/dmeans2D and the [V,P,12] ScreenGrad
     records, also when the first call goes through the partial-capacity retry or the binning buffer has another capacity;
  2. the per-instance patch masks equal the oracle's contrib_patches, and the partial count is their popcount sum;
  3. the records hold the per-Gaussian sums bound of tests/test_gpu_parity.py (unchanged: the reduce's sequential sum over
     N_g partials is inside its N_g - 1 term);
  4. gradients meet grads_agree against the oracle, and agree with the default (atomic) backward;
  5. rasterize_views(raw=True) and rasterize_views_packed(raw=True) give bit-identical gradients;
  6. a 20-step packed training loop with a densify in the middle is bit-identical from run to run."""
import numpy as np
import pytest
import torch

from test_gpu_parity import (DEV, _check_backward, _check_sums, _gpu_blend_state, _gpu_inputs, _oracle, _settings)
from util import grad_images, grads_agree, screen_scene, small_scene

pytestmark = pytest.mark.gpu

KEYS = ("means3D", "opacities", "shs", "scales", "rotations")
FULL_SIZE = dict(min_rows=1.0 - 1e-4, row_cap=4.0, min_elementwise=0.999)  # test_gpu_fullsize.py's form


@pytest.fixture(autouse=True)
def deterministic():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _keys(inp):
    return [k for k in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp") if inp.get(k) is not None]


def _grads(inp, gimg):
    """parameter gradients and dL/dmeans2D of one GaussianRasterizer forward + backward"""
    from humangaussian_b200.rasterizer import GaussianRasterizer
    t = _gpu_inputs(inp, _keys(inp))
    P = inp["means3D"].shape[0]
    m2d = torch.zeros(P, 3, device=DEV, requires_grad=True)
    c, _, d, a = GaussianRasterizer(_settings(inp))(means3D=t["means3D"], means2D=m2d, shs=t.get("shs"), opacities=t["opacities"],
                                                   colors_precomp=t.get("colors_precomp"), scales=t.get("scales"),
                                                   rotations=t.get("rotations"), cov3D_precomp=t.get("cov3D_precomp"))
    gC, gD, gA = (torch.tensor(g, device=DEV) for g in gimg)
    ((c * gC).sum() + (d * gD).sum() + (a * gA).sum()).backward()
    out = {k: t[k].grad.detach().clone() for k in t}
    out["means2D"] = m2d.grad.detach().clone()
    return out


def _same(a, b, what):
    for k in a:
        x, y = (np.ascontiguousarray(v.cpu().numpy() if torch.is_tensor(v) else v) for v in (a[k], b[k]))
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), f"{what}: {k} differs between two runs"


def _check_scene(inp, seed, criterion=None, oracle_grads=True):
    """items 1-4 on one single-view scene (oracle_grads=False: the parameter gradients are compared with the default
    backward's only, as the screen-space scenes' suite does)"""
    o_out, o_st, gimg, o_grads = _oracle(inp, seed)
    st1, sums1 = _gpu_blend_state(inp, gimg)
    st2, sums2 = _gpu_blend_state(inp, gimg)
    assert sums1.tobytes() == sums2.tobytes(), "ScreenGrad records differ between two runs"
    pm = st1["patch_masks"]
    assert np.array_equal(pm, o_st["contrib_patches"].astype(np.uint8)), "patch masks differ from the oracle's contrib_patches"
    assert st1["n_partials"] == int(np.unpackbits(pm).sum()) and st1["n_partials"] > 0
    _check_sums(sums1[0], o_grads)
    _same(_grads(inp, gimg), _grads(inp, gimg), "gradients")
    if oracle_grads:
        _check_backward(inp, o_out, gimg, o_grads, keys=_keys(inp), criterion=criterion)
    # against the default backward: the same quantities up to float summation order
    det = _grads(inp, gimg)
    torch.use_deterministic_algorithms(False)
    atomic = _grads(inp, gimg)
    torch.use_deterministic_algorithms(True, warn_only=True)
    for k in det:
        ok, msg = grads_agree(det[k].cpu().numpy(), atomic[k].cpu().numpy(), **(criterion or {}))
        assert ok, f"deterministic vs default dL/d{k}: {msg}"
    return o_st


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_small_scenes(deg):
    inp, _, _ = small_scene(P=600, deg=deg, seed=deg, H=72, W=104)
    _check_scene(inp, deg)


def test_dense_opaque_scene():
    inp, _, _ = small_scene(P=4000, deg=1, seed=5, H=64, W=64, dist=1.2)
    inp["opacities"] = np.clip(inp["opacities"] * 6, 0, 0.9999).astype(np.float32)
    inp["scales"] = (inp["scales"] * 2.5).astype(np.float32)
    o_st = _check_scene(inp, 2)
    assert (o_st["final_T"] < 1e-3).mean() > 0.05


def _boundary_scenes():
    """The screen-space scenes of tests/test_gpu_blend_boundaries.py: 1..97 staged hits per patch and zero chunks, wmax 32 / 33 /
    64, partial patches at the image edge, and needles on both sides of the never-cull threshold."""
    from test_gpu_blend_boundaries import COUNTS, SIG, _cat, _needle_cov, _patch_origin, _stack, _stacks_scene
    g, _ = _stacks_scene()
    yield "stacks", screen_scene(g["px"], g["py"], g["depth"], SIG, g["opacity"], H=64, W=128), 31
    parts = [_stack(*np.add(_patch_origin(i, 0, 0), (3.5, 1.5)), n, 1.0 + i) for i, n in enumerate((31, 32, 63))]
    parts.append(_stack(24.0, 8.0, 2, 10.0, opacity=0.999))
    g = _cat(parts)
    yield "early_termination", screen_scene(g["px"], g["py"], g["depth"], np.where(g["opacity"] > 0.5, 2000.0, SIG), g["opacity"],
                                            H=16, W=48), 32
    spots = [(7, 0, 3), (7, 1, 3), (7, 2, 5), (7, 3, 7)] + [(tx, 3, 6) for tx in range(7)] + [(0, 3, 7)]
    parts = []
    for i, (n, (tx, ty, p)) in enumerate(zip(COUNTS, spots)):
        x0, y0 = _patch_origin(tx, ty, p)
        parts.append(_stack(121.0 if x0 == 120 else x0 + 3.5, 60.45 if y0 == 60 else y0 + 1.5, n, 1.0 + i))
    g = _cat(parts)
    yield "partial_patches", screen_scene(g["px"], g["py"], g["depth"], SIG, g["opacity"], H=61, W=123), 33
    op = (1.0 / 255.0) * (1 + 1e-3)
    cov = np.zeros((4, 2, 2))
    cov[0], cov[1] = _needle_cov(0.99e4), _needle_cov(1.01e4)
    cov[2, 0, 0] = cov[2, 1, 1] = cov[3, 0, 0] = cov[3, 1, 1] = SIG * SIG
    yield "needles", screen_scene(np.array([40.0, 90.0, 20.5, 100.5]), np.array([30.0, 33.0, 9.5, 53.5]), np.array([2.0, 3.0, 1.0, 1.5]),
                                  SIG, np.array([op, op, 0.05, 0.05]), cov2d=cov, H=64, W=128), 34


def test_boundary_scenes():
    for name, inp, seed in _boundary_scenes():
        try:
            _check_scene(inp, seed, oracle_grads=False)
        except AssertionError as e:
            raise AssertionError(f"{name}: {e}") from e


def _batch_kw(inp, V, H, W, seed):
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import stack_cameras
    vm, pm, cp, tanx, tany = stack_cameras(sample_orbit_cameras(V, H, W, seed=seed), "cpu")
    return vm, pm, cp, [float(t) for t in tanx], [float(t) for t in tany]


def test_three_view_batch_masks_sums_and_retries():
    """V = 3 cameras in one call: per view, patch masks and sums against that camera's oracle; byte-identical across runs,
    across a first call forced through the partial-capacity retry, and across another binning capacity."""
    from humangaussian_b200 import rasterizer as R
    V, H, W, P = 3, 72, 104, 1500
    inp, _, _ = small_scene(P=P, deg=1, seed=6, H=H, W=W)
    vm, pm, cp, tanx, tany = _batch_kw(inp, V, H, W, 4)
    views = [_oracle(dict(inp, viewmatrix=vm[v].numpy(), projmatrix=pm[v].numpy(), campos=cp[v].numpy(), tanfovx=tanx[v],
                          tanfovy=tany[v]), 40 + v) for v in range(V)]
    kw = {k: (torch.tensor(x, device=DEV) if isinstance(x, np.ndarray) else x) for k, x in inp.items()}
    kw.update(viewmatrix=vm.to(DEV), projmatrix=pm.to(DEV), campos=cp.to(DEV), tanfovx=tanx, tanfovy=tany)
    gimg = [torch.tensor(np.stack([views[v][2][k] for v in range(V)]), device=DEV) for k in range(3)]

    def run():
        *_, st, sums = R.forward_backward_with_state(*gimg, **kw)
        return st, sums.cpu().numpy()

    st, sums = run()
    pmask, ranges = st["patch_masks"].cpu().numpy(), st["ranges"].cpu().numpy()
    ntiles = ((W + 15) // 16) * ((H + 15) // 16)
    for v, (_, o_st, _, o_grads) in enumerate(views):
        off = int(ranges[v * ntiles:(v + 1) * ntiles, 0][ranges[v * ntiles:(v + 1) * ntiles, 1] > 0].min())
        seg = pmask[off:off + int(o_st["num_rendered"])]
        assert np.array_equal(seg, o_st["contrib_patches"].astype(np.uint8)), f"view {v}: patch masks differ from the oracle"
        _check_sums(sums[v], o_grads, what=f"view {v}: ")
    assert st["n_partials"] == int(np.unpackbits(pmask).sum())
    key = (torch.device(DEV).index or 0, P, V, H, W)
    _, sums2 = run()
    assert sums.tobytes() == sums2.tobytes()
    R._partial_hint[key] = 1  # the first call cannot fit: B200GS_E_BIN_TOO_SMALL, then a retry with the reported count
    _, sums3 = run()
    assert sums.tobytes() == sums3.tobytes() and R._partial_hint[key] > st["n_partials"]
    R._cap_hint[key] = st["num_rendered"] + 333  # another instance capacity: other mask and plan offsets, same result
    st4, sums4 = run()
    assert st4["num_rendered"] == st["num_rendered"] and sums.tobytes() == sums4.tobytes()


def _views_grads(inp, V, H, W, seed, per_view_means=False):
    from humangaussian_b200.rasterizer import rasterize_views
    vm, pm, cp, tanx, tany = _batch_kw(inp, V, H, W, seed)
    t = _gpu_inputs(inp, KEYS)
    m3 = t["means3D"]
    if per_view_means:
        off = torch.linspace(-0.02, 0.02, V, device=DEV).view(V, 1, 1)
        m3 = torch.tensor(inp["means3D"], device=DEV).unsqueeze(0).repeat(V, 1, 1).add(off).requires_grad_(True)
        t["means3D"] = m3
    P = inp["means3D"].shape[0]
    m2d = torch.zeros(V, P, 3, device=DEV, requires_grad=True)
    c, _, d, a = rasterize_views(means3D=m3, opacities=t["opacities"], viewmatrices=vm.to(DEV), projmatrices=pm.to(DEV),
                                 camposs=cp.to(DEV), tanfovx=tanx, tanfovy=tany, image_height=H, image_width=W,
                                 bg=torch.tensor(inp["bg"], device=DEV), sh_degree=inp["sh_degree"], shs=t["shs"], scales=t["scales"],
                                 rotations=t["rotations"], means2D=m2d)
    g = torch.Generator(device=DEV).manual_seed(seed)
    torch.autograd.backward([c, d, a], [torch.randn(x.shape, device=DEV, generator=g) for x in (c, d, a)])
    out = {k: t[k].grad.detach().clone() for k in t}
    out["means2D"] = m2d.grad.detach().clone()
    return out


def test_per_view_means_batch():
    inp, _, _ = small_scene(P=2000, deg=2, seed=8, H=64, W=80)
    a, b = _views_grads(inp, 4, 64, 80, 9, per_view_means=True), _views_grads(inp, 4, 64, 80, 9, per_view_means=True)
    assert a["means3D"].shape == (4, 2000, 3)
    _same(a, b, "per-view means")


def test_entry_points_raw_views_and_packed():
    """With the flag on, the packed and per-tensor raw entry points give bit-identical gradients."""
    from humangaussian_b200 import dist as D
    from humangaussian_b200.rasterizer import rasterize_views, rasterize_views_packed
    _, _, sc = small_scene(P=3001, deg=3, seed=4)
    K, H = 16, 64
    raw = dict(xyz=sc.xyz, scaling=sc.scaling, rotation=sc.rotation, opacity=sc.opacity,
               features=torch.cat((sc.features_dc, sc.features_rest), 1))
    raw = {k: v.detach().float().to(DEV).contiguous() for k, v in raw.items()}
    P = raw["xyz"].shape[0]
    vm, pm, cp, tx, ty = _batch_kw(None, 4, H, H, 3)
    cams = dict(viewmatrices=vm.to(DEV), projmatrices=pm.to(DEV), camposs=cp.to(DEV), tanfovx=tx, tanfovy=ty, image_height=H,
                image_width=H, bg=torch.tensor([0.8, 0.5, 0.2], device=DEV), sh_degree=3, raw=True)
    g = torch.Generator(device=DEV).manual_seed(11)
    gw = [torch.randn(4, c, H, H, device=DEV, generator=g) for c in (3, 1, 1)]
    flat = D.pack(raw).requires_grad_(True)
    m2d_p = torch.zeros(4, P, 3, device=DEV, requires_grad=True)
    c, _, d, a = rasterize_views_packed(flat, P, K, means2D=m2d_p, **cams)
    torch.autograd.backward([c, d, a], gw)
    t = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    m2d_v = torch.zeros(4, P, 3, device=DEV, requires_grad=True)
    c2, _, d2, a2 = rasterize_views(means3D=t["xyz"], opacities=t["opacity"], scales=t["scaling"], rotations=t["rotation"],
                                    shs=t["features"], means2D=m2d_v, **cams)
    torch.autograd.backward([c2, d2, a2], gw)
    assert torch.equal(c, c2) and torch.equal(d, d2) and torch.equal(a, a2)
    got = D.unpack(flat.grad, P, K)
    for k in raw:
        assert torch.equal(got[k], t[k].grad), f"packed and per-tensor dL/d{k} differ"
    assert torch.equal(m2d_p.grad, m2d_v.grad)


def _train(seed):
    """20 packed steps (raw=True) with a densify after step 10, as tests/test_gpu_optim.py's loop"""
    from humangaussian_b200 import dist as D
    from humangaussian_b200.densify import DensifyStats, add_densification_stats, densify_and_prune_packed
    from humangaussian_b200.optim import PackedAdam, expon_lr_func
    from humangaussian_b200.rasterizer import rasterize_views_packed
    from humangaussian_b200.renderer import stack_cameras
    from humangaussian_b200.cameras import sample_orbit_cameras
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
        color, radii, _, _ = rasterize_views_packed(opt.packed, opt.P, K, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx,
                                                    tanfovy=ty, image_height=H, image_width=H, bg=bg, sh_degree=3, means2D=m2d, raw=True)
        (color - bg.view(1, 3, 1, 1)).square().mean().backward()
        add_densification_stats(stats, m2d.grad, radii)
        opt.step()
        opt.zero_grad()
        if it == 9:
            thr = float(torch.quantile((stats.xyz_gradient_accum / stats.denom.clamp_min(1)).flatten(), 0.8))
            densify_and_prune_packed(opt, stats, thr, 0.005, 1.0, None, generator=torch.Generator(device=DEV).manual_seed(7))
    st = opt.state[opt.packed]
    return dict(P=opt.P, packed=opt.packed.detach().clone(), exp_avg=st["exp_avg"].clone(), exp_avg_sq=st["exp_avg_sq"].clone(),
                accum=stats.xyz_gradient_accum.clone(), denom=stats.denom.clone(), max_radii2D=stats.max_radii2D.clone())


def test_training_loop_reproducible():
    a, b = _train(4), _train(4)
    assert a["P"] == b["P"] and a["P"] != 3001
    _same({k: v for k, v in a.items() if k != "P"}, {k: v for k, v in b.items() if k != "P"}, "training loop")


def test_classic_comparator_reports_unsupported():
    import os
    from humangaussian_b200 import rasterizer as R
    lib = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "baseline", "libb200gs_classic.so")
    inp, _, _ = small_scene(P=300, deg=0, seed=1, H=40, W=56)
    with R.use_library(lib):
        with pytest.raises(RuntimeError, match="not supported"):
            _grads(inp, grad_images(40, 56, 1))


def test_full_size_300k_four_views():
    """The bench's scene at full size: 4 cameras of its 64 at 1024^2, byte-identical twice; view 0 against the oracle with
    test_gpu_fullsize.py's full-size criterion and the sums bound."""
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.scene import sample_ply_scene
    from test_gpu_fullsize import _inputs
    p = sample_ply_scene(300000, 3)
    cams = sample_orbit_cameras(64, 1024, 1024, seed=1000)
    inp = _inputs(p, cams[0], 1024, 1024, 3)
    o_out, o_st, gimg, o_grads = _oracle(inp, 22)
    st1, sums1 = _gpu_blend_state(inp, gimg)
    assert np.array_equal(st1["patch_masks"], o_st["contrib_patches"].astype(np.uint8))
    _check_sums(sums1[0], o_grads)
    _check_backward(inp, o_out, gimg, o_grads, keys=_keys(inp), criterion=FULL_SIZE)
    from humangaussian_b200.rasterizer import rasterize_views
    from humangaussian_b200.renderer import stack_cameras
    vm, pm, cp, tx, ty = stack_cameras([cams[i] for i in (0, 16, 32, 48)], DEV)

    def run():
        t = _gpu_inputs(inp, KEYS)
        m2d = torch.zeros(4, 300000, 3, device=DEV, requires_grad=True)
        c, _, d, a = rasterize_views(means3D=t["means3D"], opacities=t["opacities"], viewmatrices=vm, projmatrices=pm, camposs=cp,
                                     tanfovx=tx, tanfovy=ty, image_height=1024, image_width=1024, bg=torch.zeros(3, device=DEV),
                                     sh_degree=3, shs=t["shs"], scales=t["scales"], rotations=t["rotations"], means2D=m2d)
        g = torch.Generator(device=DEV).manual_seed(5)
        torch.autograd.backward([c, d, a], [torch.randn(x.shape, device=DEV, generator=g) for x in (c, d, a)])
        out = {k: t[k].grad.detach().clone() for k in t}
        out["means2D"] = m2d.grad.detach().clone()
        return out

    _same(run(), run(), "full size, 4 views")
