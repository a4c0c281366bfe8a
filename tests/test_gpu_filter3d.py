"""GPU: the 3D smoothing filter (filter_3d=) against its reference (tests/filter3d_reference.py: s' and o' formed bit for
bit, the oracle -- or the antialiasing reference -- rendering with them, and the hand-derived chain back to (s, o)).

  1. b200gs_sampling_rate bit-identical to the reference: 1, 7 and 64 cameras, 130 cameras folded in three calls in two
     orders, and the margin / near-plane / NaN cases;
  2. forward state, images, radii and contributor masks bit-identical to the reference, AA off and on: small, dense-opaque,
     512^2, 3-view, per-view means and full-size scenes;
  3. gradients: grads_agree against the reference chain (post-activation and raw, AA off and on), against dense float64
     autograd, and the backward blend's sums bound;
  4. raw parameters: packed == per-tensor bit for bit, images within the raw-activation tolerance;
  5. all-zero variances == no filter, bit for bit; deterministic reruns; degenerate scales; argument errors;
  6. bake_filter_3d (also through the PLY codec) and a 20-step packed training loop with a densify."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from filter3d_reference import Filter3DOracle, dense_render_f3d, filter_params, finalize, sampling_rate
from test_gpu_parity import DEV, SUMS_K, _check_forward_state, _check_masks, _check_sums, _gpu_blend_state, _gpu_inputs
from test_oracle_filter3d import axis_camera, filter_case, margin_points
from util import close, grad_images, grads_agree, small_scene

pytestmark = pytest.mark.gpu

KEYS = ("means3D", "opacities", "shs", "scales", "rotations")
FULL_SIZE = dict(min_rows=1.0 - 1e-4, row_cap=4.0, min_elementwise=0.999)


def _orbit(V, H, W, seed):
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import stack_cameras
    return stack_cameras(sample_orbit_cameras(V, H, W, seed=seed), "cpu")


def _var_for(inp, n_cams=16, seed=0):
    """the helper's variances for the scene under an orbit camera set (float32 numpy)"""
    from humangaussian_b200.filter3d import compute_filter_3d
    H, W = inp["image_height"], inp["image_width"]
    vm, _, _, tanx, tany = _orbit(n_cams, H, W, seed)
    var = compute_filter_3d(torch.tensor(inp["means3D"], device=DEV), vm.to(DEV), tanx, tany, H, W).cpu().numpy()
    assert np.array_equal(var, finalize(sampling_rate(inp["means3D"], vm.numpy(), tanx, tany, H, W)))
    return var


# ---- 1. sampling rate ---------------------------------------------------------------------------------------------------
def _gpu_rate(means, vm, tanx, tany, H, W, rate=None):
    from humangaussian_b200.rasterizer import sampling_rate as gpu_rate
    r = torch.zeros(len(means), device=DEV) if rate is None else rate
    return gpu_rate(torch.tensor(means, device=DEV), torch.as_tensor(vm).to(DEV), tanx, tany, H, W, r)


@pytest.mark.parametrize("V", [1, 7, 64])
def test_sampling_rate_bit_identical(V):
    inp, _, _ = small_scene(P=20000, deg=0, seed=V, H=300, W=420)
    vm, _, _, tanx, tany = _orbit(V, 300, 420, V)
    got = _gpu_rate(inp["means3D"], vm, tanx, tany, 300, 420).cpu().numpy()
    want = sampling_rate(inp["means3D"], vm.numpy(), tanx, tany, 300, 420)
    assert (want > 0).mean() > 0.5
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_sampling_rate_130_cameras_any_order():
    inp, _, _ = small_scene(P=20000, deg=0, seed=1, H=256, W=256)
    vm, _, _, tanx, tany = _orbit(130, 256, 256, 3)
    want = sampling_rate(inp["means3D"], vm.numpy(), tanx, tany, 256, 256)
    outs = []
    for order in (np.arange(130), np.random.RandomState(0).permutation(130)):
        r = torch.zeros(len(inp["means3D"]), device=DEV)
        for sl in (slice(0, 64), slice(64, 128), slice(128, 130)):
            idx = order[sl]
            _gpu_rate(inp["means3D"], vm[idx], [tanx[i] for i in idx], [tany[i] for i in idx], 256, 256, r)
        outs.append(r.cpu().numpy())
    assert outs[0].tobytes() == outs[1].tobytes() == want.tobytes()
    from humangaussian_b200.filter3d import compute_filter_3d
    var = compute_filter_3d(torch.tensor(inp["means3D"], device=DEV), vm.to(DEV), tanx, tany, 256, 256).cpu().numpy()
    assert var.tobytes() == finalize(want).tobytes()


def test_sampling_rate_edge_cases():
    vm, tx, ty, H, W = axis_camera()
    m, want = margin_points()
    got = _gpu_rate(m, vm, tx, ty, H, W).cpu().numpy()
    assert np.array_equal(got > 0, want)
    assert got.tobytes() == sampling_rate(m, vm, tx, ty, H, W).tobytes()
    from humangaussian_b200.filter3d import compute_filter_3d
    away = torch.tensor([[0.0, 0.0, -1.0], [0.0, 0.0, -2.0]], device=DEV)  # behind the camera: nothing in view
    assert torch.equal(compute_filter_3d(away, torch.tensor(vm, device=DEV), tx, ty, H, W), torch.zeros(2, device=DEV))


# ---- 2./3. forward and gradients against the reference --------------------------------------------------------------------
def _f3d_oracle(inp, var, seed, aa):
    o = Filter3DOracle()
    out = o.forward(filter_3d=var, antialiasing=aa, **inp)
    gimg = grad_images(inp["image_height"], inp["image_width"], seed)
    return out, o.state(), gimg, o.backward(*gimg, sums_err_const=SUMS_K)


def _gpu_grads(inp, var, gimg, aa, keys=KEYS):
    from humangaussian_b200.rasterizer import rasterize_views
    t = _gpu_inputs(inp, keys)
    V = 1
    m2d = torch.zeros(V, inp["means3D"].shape[0], 3, device=DEV, requires_grad=True)
    g = lambda k: torch.tensor(inp[k], device=DEV)
    c, _, d, a = rasterize_views(means3D=t["means3D"], opacities=t["opacities"], shs=t["shs"], scales=t["scales"], rotations=t["rotations"],
                                 viewmatrices=g("viewmatrix").reshape(1, 4, 4), projmatrices=g("projmatrix").reshape(1, 4, 4),
                                 camposs=g("campos").reshape(1, 3), tanfovx=[inp["tanfovx"]], tanfovy=[inp["tanfovy"]],
                                 image_height=inp["image_height"], image_width=inp["image_width"], bg=g("bg"), sh_degree=inp["sh_degree"],
                                 means2D=m2d, scale_modifier=inp.get("scale_modifier", 1.0), antialiasing=aa,
                                 filter_3d=torch.tensor(var, device=DEV))
    gC, gD, gA = (torch.tensor(x, device=DEV)[None] for x in gimg)
    ((c * gC).sum() + (d * gD).sum() + (a * gA).sum()).backward()
    out = {k: t[k].grad.detach().cpu().numpy() for k in t}
    out["means2D"] = m2d.grad[0].detach().cpu().numpy()
    return out


def _check_scene(inp, var, seed, aa, criterion=None):
    o_out, o_st, gimg, o_grads = _f3d_oracle(inp, var, seed, aa)
    _check_forward_state(dict(inp, antialiasing=aa, filter_3d=var), o_out, o_st)
    g = _gpu_grads(inp, var, gimg, aa)
    for k in g:
        ok, msg = grads_agree(g[k].reshape(o_grads[k].shape), o_grads[k], **(criterion or {}))
        assert ok, f"3D filter (AA {aa}) dL/d{k}: {msg}"
    _, sums = _gpu_blend_state(dict(inp, antialiasing=aa, filter_3d=var), gimg)
    _check_sums(sums[0], o_grads)
    return o_st


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("deg", [0, 3])
def test_small_scenes(deg, aa):
    inp, _, _ = small_scene(P=600, deg=deg, seed=deg, H=72, W=104)
    var = _var_for(inp, seed=deg)
    _, _, f = filter_params(inp["scales"], inp["opacities"], var)
    assert (f["coef"] < 1).mean() > 0.9  # the filter is on
    _check_scene(inp, var, deg, aa)


@pytest.mark.parametrize("aa", [False, True])
def test_dense_opaque_scene(aa):
    inp, _, _ = small_scene(P=4000, deg=1, seed=5, H=64, W=64, dist=1.2)
    inp["opacities"] = np.clip(inp["opacities"] * 6, 0, 0.9999).astype(np.float32)
    inp["scales"] = (inp["scales"] * 2.5).astype(np.float32)
    o_st = _check_scene(inp, _var_for(inp, seed=1), 2, aa)
    assert (o_st["final_T"] < 1e-3).mean() > 0.05


@pytest.mark.parametrize("aa", [False, True])
def test_medium_scene_512(aa):
    inp, _, _ = small_scene(P=60000, deg=0, seed=11, H=512, W=512, big=False, dist=2.0, fovy_deg=70.0, elev=15.0, azim=0.0)
    o_st = _check_scene(inp, _var_for(inp, n_cams=64, seed=2), 5, aa)
    assert o_st["num_rendered"] > 50000


@pytest.mark.parametrize("aa", [False, True])
def test_degenerate_scales(aa):
    """a zero and a 1e-7 scale axis: finite gradients that meet the reference"""
    for case in ("s=0", "s=1e-7"):
        inp, _, _ = small_scene(P=600, deg=1, seed=7, H=72, W=104)
        inp, var = filter_case(inp, case)
        _check_scene(inp, var, 3, aa)


@pytest.mark.parametrize("aa", [False, True])
def test_three_view_batch(aa):
    from humangaussian_b200.rasterizer import forward_backward_with_state
    V, H, W = 3, 72, 104
    inp, _, _ = small_scene(P=1500, deg=1, seed=6, H=H, W=W)
    var = _var_for(inp, seed=6)
    vm, pm, cp, tanx, tany = _orbit(V, H, W, 4)
    views = [_f3d_oracle(dict(inp, viewmatrix=vm[v].numpy(), projmatrix=pm[v].numpy(), campos=cp[v].numpy(), tanfovx=float(tanx[v]),
                              tanfovy=float(tany[v])), var, 40 + v, aa) for v in range(V)]
    kw = {k: (torch.tensor(x, device=DEV) if isinstance(x, np.ndarray) else x) for k, x in inp.items()}
    kw.update(viewmatrix=vm.to(DEV), projmatrix=pm.to(DEV), campos=cp.to(DEV), tanfovx=[float(t) for t in tanx],
              tanfovy=[float(t) for t in tany], antialiasing=aa, filter_3d=torch.tensor(var, device=DEV))
    gimg = [torch.tensor(np.stack([views[v][2][k] for v in range(V)]), device=DEV) for k in range(3)]
    color, radii, depth, alpha, st, sums = forward_backward_with_state(*gimg, **kw)
    masks, ranges, nc = (st[k].cpu().numpy() for k in ("contributor_masks", "ranges", "n_contrib"))
    f = lambda x: np.ascontiguousarray(x).view(np.uint32)
    for v, (o_out, o_st, _, o_grads) in enumerate(views):
        for got, want in zip((color[v], radii[v], depth[v], alpha[v]), o_out):
            assert np.array_equal(f(got.cpu().numpy()), f(want)), f"view {v}"
        checked, _ = _check_masks(masks, ranges, nc[v], o_st, H, W, v=v)
        assert checked > 100
        _check_sums(sums[v].cpu().numpy(), o_grads, what=f"view {v}: ")


def test_per_view_means():
    """[V,P,3] means: each view equals a single-view call with that view's positions and the same (canonical) variances"""
    from humangaussian_b200.rasterizer import rasterize_views
    P, H, W, V = 1500, 72, 104, 3
    inp, _, _ = small_scene(P=P, deg=1, seed=21, H=H, W=W)
    var = torch.tensor(_var_for(inp), device=DEV)
    vm, pm, cp, tanx, tany = (x.to(DEV) if torch.is_tensor(x) else x for x in _orbit(V, H, W, 2))
    t = {k: torch.tensor(inp[k], device=DEV) for k in ("opacities", "shs", "scales", "rotations")}
    xyz_v = (torch.tensor(inp["means3D"], device=DEV)[None] + 0.01 * torch.randn(V, P, 3, device=DEV,
                                                                                generator=torch.Generator(device=DEV).manual_seed(3)))
    kw = dict(image_height=H, image_width=W, bg=torch.tensor(inp["bg"], device=DEV), sh_degree=1, filter_3d=var, **t)
    for aa in (False, True):
        with torch.no_grad():
            outs = rasterize_views(means3D=xyz_v.contiguous(), viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tanx, tanfovy=tany,
                                   antialiasing=aa, **kw)
            for v in range(V):
                one = rasterize_views(means3D=xyz_v[v].contiguous(), viewmatrices=vm[v:v + 1], projmatrices=pm[v:v + 1],
                                      camposs=cp[v:v + 1], tanfovx=tanx[v:v + 1], tanfovy=tany[v:v + 1], antialiasing=aa, **kw)
                for x, y in zip(outs, one):
                    assert torch.equal(x[v], y[0]), f"per-view means, view {v}"


@pytest.mark.parametrize("aa", [False, True])
def test_full_size_300k_deg3_1024(aa):
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.scene import sample_ply_scene
    from test_gpu_fullsize import _inputs
    p = sample_ply_scene(300000, 3)
    cam = sample_orbit_cameras(64, 1024, 1024, seed=1000)[0]
    inp = _inputs(p, cam, 1024, 1024, 3)
    o_st = _check_scene(inp, _var_for(inp, n_cams=64, seed=1000), 22, aa, criterion=FULL_SIZE)
    assert o_st["num_rendered"] > 400000


def test_cuda_backward_vs_float64_autograd():
    for aa in (False, True):
        for deg, seed, kw in ((3, 1, {}), (1, 9, dict(H=32, W=32, dist=1.3)), (2, 4, dict(H=48, W=48, fovy_deg=25.0, dist=1.1))):
            inp, _, _ = small_scene(P=400, deg=deg, seed=seed, **kw)
            H, W = inp["image_height"], inp["image_width"]
            var = _var_for(inp, seed=seed)
            o = Filter3DOracle(threads=1)
            _, radii, _, _ = o.forward(filter_3d=var, antialiasing=aa, **inp)
            st = o.state()
            gimg = grad_images(H, W, seed)
            t64 = lambda a: torch.tensor(a, dtype=torch.float64)
            ten = {k: t64(inp[k]).requires_grad_(True) for k in KEYS}
            m2d = torch.zeros(len(radii), 3, dtype=torch.float64, requires_grad=True)
            ids = np.nonzero(radii > 0)[0]
            order = ids[np.lexsort((ids, st["depths"][ids]))]
            c, d, a, _ = dense_render_f3d(means3D=ten["means3D"], means2D=m2d, opacities=ten["opacities"], scales=ten["scales"],
                                          filter_3d=var, antialiasing=aa, viewmatrix=t64(inp["viewmatrix"]),
                                          projmatrix=t64(inp["projmatrix"]), campos=t64(inp["campos"]), bg=t64(inp["bg"]), H=H, W=W,
                                          tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], radii=radii, rect=st["rect"], order=order,
                                          sh_degree=deg, shs=ten["shs"], rotations=ten["rotations"])
            ((c * t64(gimg[0])).sum() + (d * t64(gimg[1])).sum() + (a * t64(gimg[2])).sum()).backward()
            g = _gpu_grads(inp, var, gimg, aa)
            ref = dict(means2D=m2d.grad.numpy(), **{k: ten[k].grad.numpy() for k in KEYS})
            for k, r in ref.items():
                ok, msg = grads_agree(g[k].reshape(r.shape), r, atol=1e-4, rtol=1e-3)
                assert ok, f"deg {deg} AA {aa}: dL/d{k} CUDA vs float64 autograd: {msg}"


# ---- 4. raw parameters ------------------------------------------------------------------------------------------------------
def _body(P, deg, seed):
    from humangaussian_b200.scene import synthetic_body
    p = synthetic_body(P, sh_degree=deg, seed=seed)
    p.scaling += math.log(6.0)
    p.opacity += 1.5
    return p.to(DEV)


@pytest.mark.parametrize("aa", [False, True])
def test_raw_and_packed(aa):
    from humangaussian_b200.filter3d import compute_filter_3d
    from humangaussian_b200.rasterizer import packed_layout, rasterize_views, rasterize_views_packed
    P, H, W, V, deg = 1500, 72, 104, 3, 3
    K = (deg + 1) ** 2
    p = _body(P, deg, 21)
    vm, pm, cp, tanx, tany = (x.to(DEV) if torch.is_tensor(x) else x for x in _orbit(V, H, W, 2))
    var = compute_filter_3d(p.xyz, vm, tanx, tany, H, W)
    bg = torch.tensor([0.1, 0.4, 0.7], device=DEV)
    rng = np.random.RandomState(1)
    gw = [torch.tensor(rng.randn(V, c, H, W).astype(np.float32), device=DEV) for c in (3, 1, 1)]
    kw = dict(viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tanx, tanfovy=tany, image_height=H, image_width=W, bg=bg,
              sh_degree=deg, antialiasing=aa, filter_3d=var)
    loss = lambda c, d, a: (c * gw[0]).sum() + (d * gw[1]).sum() + (a * gw[2]).sum()
    names = ("xyz", "scaling", "rotation", "opacity", "features_dc", "features_rest")
    # post-activation inputs with the reference's filtered parameters and no filter: the raw path must agree within tolerance
    with torch.no_grad():
        sp, op, _ = filter_params(torch.exp(p.scaling).cpu().numpy(), torch.sigmoid(p.opacity).cpu().numpy(), var.cpu().numpy())
        ref = rasterize_views(means3D=p.xyz, opacities=torch.tensor(op, device=DEV), shs=torch.cat((p.features_dc, p.features_rest), 1),
                              scales=torch.tensor(sp, device=DEV), rotations=torch.nn.functional.normalize(p.rotation),
                              **dict(kw, filter_3d=None))
    raw = {k: getattr(p, k).clone().requires_grad_(True) for k in names}
    out1 = rasterize_views(means3D=raw["xyz"], opacities=raw["opacity"], shs=torch.cat((raw["features_dc"], raw["features_rest"]), 1),
                           scales=raw["scaling"], rotations=raw["rotation"], raw=True, **kw)
    loss(out1[0], out1[2], out1[3]).backward()
    for x, y in zip(ref, out1):
        ok, worst = close(y.detach().float().cpu().numpy(), x.detach().float().cpu().numpy())
        assert ok, worst
    # autograd through torch activations with the filter in the kernels: same gradients within grads_agree
    raw0 = {k: getattr(p, k).clone().requires_grad_(True) for k in names}
    out0 = rasterize_views(means3D=raw0["xyz"], opacities=torch.sigmoid(raw0["opacity"]),
                           shs=torch.cat((raw0["features_dc"], raw0["features_rest"]), 1), scales=torch.exp(raw0["scaling"]),
                           rotations=torch.nn.functional.normalize(raw0["rotation"]), **kw)
    loss(out0[0], out0[2], out0[3]).backward()
    for k in names:
        ok, msg = grads_agree(raw[k].grad.cpu().numpy(), raw0[k].grad.cpu().numpy())
        assert ok, f"raw 3D-filter dL/d{k}: {msg}"
    fields, n = packed_layout(P, K)
    flat = torch.zeros(n, device=DEV)
    with torch.no_grad():
        for (o, m, _), t in zip(fields, (p.xyz, p.scaling, p.rotation, p.opacity, torch.cat((p.features_dc, p.features_rest), 1))):
            flat.narrow(0, o, m).copy_(t.reshape(-1))
    flat.requires_grad_(True)
    out2 = rasterize_views_packed(flat, P, K, raw=True, **kw)
    loss(out2[0], out2[2], out2[3]).backward()
    for x, y in zip(out1, out2):
        assert torch.equal(x, y)
    grads = [raw["xyz"].grad, raw["scaling"].grad, raw["rotation"].grad, raw["opacity"].grad,
             torch.cat((raw["features_dc"].grad, raw["features_rest"].grad), 1)]
    for (o, m, shape), g in zip(fields, grads):
        got = flat.grad.narrow(0, o, m).view(shape)
        ok, msg = grads_agree(got.cpu().numpy().reshape(P, -1), g.cpu().numpy().reshape(P, -1))
        assert ok, f"packed raw 3D-filter gradient field at {o}: {msg}"


# ---- 5. identity, determinism, errors ---------------------------------------------------------------------------------------
def _all_grads(p, kw, raw, det=False):
    from humangaussian_b200.rasterizer import rasterize_views
    names = ("xyz", "scaling", "rotation", "opacity", "features_dc", "features_rest")
    t = {k: getattr(p, k).clone().requires_grad_(True) for k in names}
    acts = (t["opacity"], t["scaling"], t["rotation"]) if raw else (torch.sigmoid(t["opacity"]), torch.exp(t["scaling"]),
                                                                     torch.nn.functional.normalize(t["rotation"]))
    out = rasterize_views(means3D=t["xyz"], opacities=acts[0], scales=acts[1], rotations=acts[2],
                          shs=torch.cat((t["features_dc"], t["features_rest"]), 1), raw=raw, **kw)
    rng = np.random.RandomState(0)
    loss = sum((o * torch.tensor(rng.randn(*o.shape).astype(np.float32), device=DEV)).sum() for o in (out[0], out[2], out[3]))
    loss.backward()
    return [x.detach().cpu().numpy() for x in out] + [t[k].grad.cpu().numpy() for k in names]


@pytest.mark.parametrize("raw", [False, True])
def test_zero_variances_equal_no_filter(raw):
    """v = 0: s' = sqrt(fl(s*s)) = s for the scene's scales (>= 1e-6), coef = 1; forward and gradients bit-identical to
    filter_3d=None under the deterministic backward"""
    P, H, W, V = 1500, 72, 104, 2
    p = _body(P, 2, 4)
    with torch.no_grad():
        p.scaling.clamp_(min=math.log(1e-6))
    vm, pm, cp, tanx, tany = (x.to(DEV) if torch.is_tensor(x) else x for x in _orbit(V, H, W, 9))
    kw = dict(viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tanx, tanfovy=tany, image_height=H, image_width=W,
              bg=torch.tensor([0.1, 0.4, 0.7], device=DEV), sh_degree=2)
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        for aa in (False, True):
            a = _all_grads(p, dict(kw, antialiasing=aa), raw)
            b = _all_grads(p, dict(kw, antialiasing=aa, filter_3d=torch.zeros(P, device=DEV)), raw)
            for i, (x, y) in enumerate(zip(a, b)):
                assert x.tobytes() == y.tobytes(), (aa, i)
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def test_deterministic_reruns_are_identical():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        inp, _, _ = small_scene(P=2000, deg=2, seed=12, H=96, W=128)
        var = _var_for(inp, seed=12)
        gimg = grad_images(96, 128, 1)
        for aa in (False, True):
            st1, s1 = _gpu_blend_state(dict(inp, antialiasing=aa, filter_3d=var), gimg)
            st2, s2 = _gpu_blend_state(dict(inp, antialiasing=aa, filter_3d=var), gimg)
            assert s1.tobytes() == s2.tobytes() and np.array_equal(st1["patch_masks"], st2["patch_masks"])
            g1, g2 = _gpu_grads(inp, var, gimg, aa), _gpu_grads(inp, var, gimg, aa)
            for k in g1:
                assert g1[k].tobytes() == g2[k].tobytes(), k
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def test_argument_errors():
    from humangaussian_b200 import rasterizer as R
    from humangaussian_b200.rasterizer import rasterize_views, rasterize_views_packed
    inp, _, _ = small_scene(P=300, deg=0, seed=2)
    P = 300
    g = lambda k: torch.tensor(inp[k], device=DEV)
    cams = dict(viewmatrices=g("viewmatrix").reshape(1, 4, 4), projmatrices=g("projmatrix").reshape(1, 4, 4),
                camposs=g("campos").reshape(1, 3), tanfovx=[inp["tanfovx"]], tanfovy=[inp["tanfovy"]], image_height=inp["image_height"],
                image_width=inp["image_width"], bg=g("bg"))
    base = dict(means3D=g("means3D"), opacities=g("opacities"), shs=g("shs"), **cams)
    ok = torch.zeros(P, device=DEV)
    for bad in (torch.zeros(P - 1, device=DEV), torch.zeros(P, device=DEV, dtype=torch.float64), torch.zeros(P), torch.zeros(P, 1, device=DEV)):
        with pytest.raises(ValueError):
            rasterize_views(scales=g("scales"), rotations=g("rotations"), filter_3d=bad, **base)
        with pytest.raises(ValueError):
            rasterize_views_packed(torch.zeros(R.packed_numel(P, 1), device=DEV), P, 1, filter_3d=bad, **cams)
    cov = torch.zeros(P, 6, device=DEV)
    with pytest.raises(ValueError):
        rasterize_views(cov3D_precomp=cov, filter_3d=ok, **base)
    # the ABI rejects the same combination on its own: B200GS_E_ARGS from the forward
    L = R.load_library()
    prm, _, _ = R._make_params(P, 1, 0, 1, inp["image_height"], inp["image_width"], 1.0, [inp["tanfovx"]], [inp["tanfovy"]])
    opts = R._render_opts(False, ok)
    n = C.c_int64(0)
    dummy = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    d = R._ptr(dummy)
    rc = L.b200gs_forward_opts(C.byref(prm), C.byref(opts), R._ptr(g("means3D")), R._ptr(g("shs")), None, R._ptr(g("opacities")), None,
                               None, R._ptr(cov), R._ptr(g("bg")), R._ptr(g("viewmatrix")), R._ptr(g("projmatrix")), R._ptr(g("campos")),
                               d, d, d, d, d, 1 << 20, d, 1 << 20, 1, d, 1 << 20, C.byref(n), None)
    assert rc == R.E_ARGS


# ---- 6. baking, and training with the filter --------------------------------------------------------------------------------
def test_bake_filter_3d_and_ply_round_trip(tmp_path):
    from humangaussian_b200.filter3d import bake_filter_3d, compute_filter_3d
    from humangaussian_b200.rasterizer import rasterize_views
    from humangaussian_b200 import scene as S
    P, H, W, V, deg = 3000, 96, 128, 3, 1
    p = _body(P, deg, 8)
    vm, pm, cp, tanx, tany = (x.to(DEV) if torch.is_tensor(x) else x for x in _orbit(V, H, W, 6))
    var = compute_filter_3d(p.xyz, vm, tanx, tany, H, W)
    kw = dict(viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tanx, tanfovy=tany, image_height=H, image_width=W,
              bg=torch.tensor([0.2, 0.1, 0.3], device=DEV), sh_degree=deg, raw=True)
    shs = torch.cat((p.features_dc, p.features_rest), 1)
    with torch.no_grad():
        want = rasterize_views(means3D=p.xyz, opacities=p.opacity, scales=p.scaling, rotations=p.rotation, shs=shs, filter_3d=var, **kw)
        sc, op = bake_filter_3d(p.scaling, p.opacity, var)
        got = rasterize_views(means3D=p.xyz, opacities=op, scales=sc, rotations=p.rotation, shs=shs, **kw)
        plain = rasterize_views(means3D=p.xyz, opacities=p.opacity, scales=p.scaling, rotations=p.rotation, shs=shs, **kw)
    assert not torch.equal(want[0], plain[0])
    for x, y in zip(want, got):
        ok, worst = close(y.float().cpu().numpy(), x.float().cpu().numpy())
        assert ok, worst
    q = S.GaussianParams(p.xyz, p.features_dc, p.features_rest, sc, p.rotation, op, sh_degree=deg).to("cpu")
    path = str(tmp_path / "baked.ply")
    S.params_to_ply(path, q)
    r = S.params_from_ply(path, sh_degree=deg).to(DEV)
    with torch.no_grad():
        got2 = rasterize_views(means3D=r.xyz, opacities=r.opacity, scales=r.scaling, rotations=r.rotation,
                               shs=torch.cat((r.features_dc, r.features_rest), 1), **kw)
    for x, y in zip(want, got2):
        ok, worst = close(y.float().cpu().numpy(), x.float().cpu().numpy())
        assert ok, worst


def test_packed_training_loop_with_densify():
    """20 packed raw steps with PackedAdam (tests/test_gpu_deterministic.py's loop) with the filter on: a densify after step
    10 changes P, and the filter, recomputed from a fixed camera set whenever P changed, follows it"""
    from humangaussian_b200 import dist as D
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.densify import DensifyStats, add_densification_stats, densify_and_prune_packed
    from humangaussian_b200.filter3d import compute_filter_3d
    from humangaussian_b200.optim import PackedAdam, expon_lr_func
    from humangaussian_b200.rasterizer import packed_layout, rasterize_views_packed
    from humangaussian_b200.renderer import stack_cameras
    _, _, sc = small_scene(P=3001, deg=3, seed=4)
    K, H = 16, 64
    raw = dict(xyz=sc.xyz, scaling=sc.scaling, rotation=sc.rotation, opacity=sc.opacity,
               features=torch.cat((sc.features_dc, sc.features_rest), 1))
    flat = D.pack({k: v.detach().float().to(DEV).contiguous() for k, v in raw.items()}).requires_grad_(True)
    lrs = dict(xyz=0.00016, f_dc=0.0125, f_rest=0.0125 / 20.0, opacity=0.01, scaling=0.005, rotation=0.001)
    sched = expon_lr_func(lr_init=0.00016, lr_final=0.0000016, lr_delay_mult=0.01, max_steps=30000)
    opt = PackedAdam(flat, 3001, K, lrs, xyz_scheduler=sched)
    vm, pm, cp, tx, ty = stack_cameras(sample_orbit_cameras(4, H, H, seed=3), DEV)
    fvm, _, _, ftx, fty = stack_cameras(sample_orbit_cameras(256, H, H, seed=11), DEV)  # the filter's fixed camera set
    bg = torch.tensor([0.8, 0.5, 0.2], device=DEV)
    stats = DensifyStats.zeros(opt.P, DEV)
    var, seen = None, []
    for it in range(20):
        if var is None or var.shape[0] != opt.P:
            off, n, _ = packed_layout(opt.P, K)[0][0]
            var = compute_filter_3d(opt.packed.detach().narrow(0, off, n).view(opt.P, 3), fvm, ftx, fty, H, H)
        opt.update_learning_rate(it)
        m2d = torch.zeros(4, opt.P, 3, device=DEV, requires_grad=True)
        color, radii, _, _ = rasterize_views_packed(opt.packed, opt.P, K, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx,
                                                    tanfovy=ty, image_height=H, image_width=H, bg=bg, sh_degree=3, means2D=m2d, raw=True,
                                                    filter_3d=var)
        loss = (color - bg.view(1, 3, 1, 1)).square().mean()
        loss.backward()
        assert math.isfinite(loss.item()) and torch.isfinite(opt.packed.grad).all()
        add_densification_stats(stats, m2d.grad, radii)
        opt.step()
        opt.zero_grad()
        seen.append((opt.P, var.shape[0]))
        if it == 9:
            thr = float(torch.quantile((stats.xyz_gradient_accum / stats.denom.clamp_min(1)).flatten(), 0.8))
            densify_and_prune_packed(opt, stats, thr, 0.005, 1.0, None, generator=torch.Generator(device=DEV).manual_seed(7))
            with pytest.raises(ValueError):  # a stale filter is rejected by its length
                rasterize_views_packed(opt.packed, opt.P, K, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx, tanfovy=ty,
                                       image_height=H, image_width=H, bg=bg, sh_degree=3, raw=True, filter_3d=var)
    assert opt.P != 3001 and all(p == v for p, v in seen) and len({p for p, _ in seen}) == 2
    assert torch.isfinite(opt.packed).all()
