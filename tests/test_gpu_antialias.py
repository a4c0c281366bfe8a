"""GPU: the antialiasing filter (antialiasing=True) against its reference (tests/aa_reference.py: the CPU oracle with the
filter's opacity o_eff = op * rho formed bit for bit, and the hand-derived rho chain in the backward).

  1. forward state, images, depth, alpha, radii and contributor masks bit-identical to the reference: small, dense-opaque,
     precomputed-input, 512^2, 3-view batched and full-size scenes;
  2. gradients by grads_agree (test_gpu_fullsize.py's form at full size), and the backward blend's sums bound of
     tests/test_gpu_parity.py unchanged (K = 4, C = 10);
  3. the CUDA backward against torch.autograd over the dense float64 formulation with the filter;
  4. raw parameters, the packed entry and per-view means;
  5. byte-identical reruns under torch.use_deterministic_algorithms(True);
  6. with the filter off, the *_opts entry points (NULL options, and options with antialiasing = 0) equal the plain ones;
  7. render(pipe.antialiasing), render_views, GaussianRasterizer with a 13-field settings tuple and render_frames agree with
     rasterize_views(antialiasing=True)."""
import collections
import math

import numpy as np
import pytest
import torch

from aa_reference import AAOracle, dense_render_aa
from test_gpu_parity import (DEV, SUMS_K, _check_forward_state, _check_masks, _check_sums, _gpu_blend_state, _gpu_inputs,
                             _settings)
from util import close, grad_images, grads_agree, small_scene

pytestmark = pytest.mark.gpu

KEYS = ("means3D", "opacities", "shs", "scales", "rotations")
FULL_SIZE = dict(min_rows=1.0 - 1e-4, row_cap=4.0, min_elementwise=0.999)  # test_gpu_fullsize.py's form


def _aa_oracle(inp, seed):
    o = AAOracle()
    out = o.forward(**inp)
    st = o.state()
    gimg = grad_images(inp["image_height"], inp["image_width"], seed)
    return out, st, gimg, o.backward(*gimg, sums_err_const=SUMS_K)


def _gpu_grads(inp, gimg, keys):
    from humangaussian_b200.rasterizer import GaussianRasterizer
    t = _gpu_inputs(inp, keys)
    m2d = torch.zeros(inp["means3D"].shape[0], 3, device=DEV, requires_grad=True)
    c, _, d, a = GaussianRasterizer(_settings(inp), antialiasing=True)(
        means3D=t["means3D"], means2D=m2d, shs=t.get("shs"), colors_precomp=t.get("colors_precomp"), opacities=t["opacities"],
        scales=t.get("scales"), rotations=t.get("rotations"), cov3D_precomp=t.get("cov3D_precomp"))
    gC, gD, gA = (torch.tensor(g, device=DEV) for g in gimg)
    ((c * gC).sum() + (d * gD).sum() + (a * gA).sum()).backward()
    out = {k: t[k].grad.detach().cpu().numpy() for k in t}
    out["means2D"] = m2d.grad.detach().cpu().numpy()
    return out


def _check_scene(inp, seed, keys=KEYS, criterion=None):
    o_out, o_st, gimg, o_grads = _aa_oracle(inp, seed)
    vis = o_out[1] > 0
    co, op = o_st["conic_opacity"][vis, 3], np.asarray(inp["opacities"]).reshape(-1)[vis]
    assert (co <= op).all() and (co < op).mean() > 0.5  # the filter is on
    _check_forward_state(dict(inp, antialiasing=True), o_out, o_st)
    g = _gpu_grads(inp, gimg, keys)
    for k in g:
        crit = dict(criterion or {})
        if k == "cov3D_precomp":
            # row-wise only, as tests/test_oracle_autograd.py compares covariance gradients: the reference forms the rho
            # chain in float64, the kernel in float32, whose det = a*c - b^2 of an elongated footprint carries the
            # cancellation; single covariance entries that are near-zero sums of such terms then miss elementwise
            crit["min_elementwise"] = 0.0
        ok, msg = grads_agree(g[k].reshape(o_grads[k].shape), o_grads[k], **crit)
        if k == "cov3D_precomp":
            print(f"AA dL/dcov3D_precomp: {msg}")
        assert ok, f"AA dL/d{k}: {msg}"
    _, sums = _gpu_blend_state(dict(inp, antialiasing=True), gimg)
    _check_sums(sums[0], o_grads)
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


def test_precomputed_cov_and_colors():
    from oracle.gs_oracle import Oracle
    inp, _, _ = small_scene(P=500, deg=0, seed=7, H=48, W=80)
    o = Oracle()
    o.forward(**inp)
    st = o.state()
    inp2 = {k: v for k, v in inp.items() if k not in ("shs", "scales", "rotations")}
    inp2["colors_precomp"] = np.abs(st["rgb"]).astype(np.float32) + 0.05
    inp2["cov3D_precomp"] = st["cov3d"].copy()
    inp2["sh_degree"] = 0
    _check_scene(inp2, 3, keys=("means3D", "opacities", "colors_precomp", "cov3D_precomp"))


def test_rho_floor_scenes():
    """Every rendered Gaussian on rho's floor (tests/test_oracle_antialias.py: edge-on flat Gaussians, det0 < 0), blending:
    F1's floor and B2's zero rho-gradient there, against the reference."""
    from test_oracle_antialias import floor_scenes
    keys = {"edge-on": ("means3D", "opacities", "colors_precomp", "scales", "rotations"),
            "det0 <= 0": ("means3D", "opacities", "colors_precomp", "cov3D_precomp")}
    for case, inp in floor_scenes():
        o_st = _check_scene(inp, 6, keys=keys[case])
        assert o_st["num_rendered"] > 0, case


def test_medium_scene_512():
    inp, _, _ = small_scene(P=60000, deg=0, seed=11, H=512, W=512, big=False, dist=2.0, fovy_deg=70.0, elev=15.0, azim=0.0)
    o_st = _check_scene(inp, 5)
    assert o_st["num_rendered"] > 50000


def test_three_view_batch():
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.rasterizer import forward_backward_with_state
    from humangaussian_b200.renderer import stack_cameras
    V, H, W = 3, 72, 104
    inp, _, _ = small_scene(P=1500, deg=1, seed=6, H=H, W=W)
    vm, pm, cp, tanx, tany = stack_cameras(sample_orbit_cameras(V, H, W, seed=4), "cpu")
    views = [_aa_oracle(dict(inp, viewmatrix=vm[v].numpy(), projmatrix=pm[v].numpy(), campos=cp[v].numpy(), tanfovx=float(tanx[v]),
                              tanfovy=float(tany[v])), 40 + v) for v in range(V)]
    kw = {k: (torch.tensor(x, device=DEV) if isinstance(x, np.ndarray) else x) for k, x in inp.items()}
    kw.update(viewmatrix=vm.to(DEV), projmatrix=pm.to(DEV), campos=cp.to(DEV), tanfovx=[float(t) for t in tanx],
              tanfovy=[float(t) for t in tany], antialiasing=True)
    gimg = [torch.tensor(np.stack([views[v][2][k] for v in range(V)]), device=DEV) for k in range(3)]
    color, radii, depth, alpha, st, sums = forward_backward_with_state(*gimg, **kw)
    masks, ranges, nc = (st[k].cpu().numpy() for k in ("contributor_masks", "ranges", "n_contrib"))
    f = lambda x: np.ascontiguousarray(x).view(np.uint32)
    for v, (o_out, o_st, _, o_grads) in enumerate(views):
        for got, want in zip((color[v], radii[v], depth[v], alpha[v]), o_out):
            assert np.array_equal(f(got.cpu().numpy()), f(want)), f"view {v}"
        assert np.array_equal(nc[v].view(np.uint32), o_st["n_contrib"])
        checked, _ = _check_masks(masks, ranges, nc[v], o_st, H, W, v=v)
        assert checked > 100
        _check_sums(sums[v].cpu().numpy(), o_grads, what=f"view {v}: ")


def test_full_size_300k_deg3_1024():
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.scene import sample_ply_scene
    from test_gpu_fullsize import _inputs
    p = sample_ply_scene(300000, 3)
    cam = sample_orbit_cameras(64, 1024, 1024, seed=1000)[0]
    o_st = _check_scene(_inputs(p, cam, 1024, 1024, 3), 22, criterion=FULL_SIZE)
    assert o_st["num_rendered"] > 400000


def test_cuda_backward_vs_float64_autograd():
    """The filtered CUDA backward against torch.autograd over dense float64 with the filter (as test_gpu_fullsize.py does
    without it); integer decisions from the oracle."""
    for deg, seed, kw in ((3, 1, {}), (1, 9, dict(H=32, W=32, dist=1.3)), (2, 4, dict(H=48, W=48, fovy_deg=25.0, dist=1.1))):
        inp, _, _ = small_scene(P=400, deg=deg, seed=seed, **kw)
        H, W = inp["image_height"], inp["image_width"]
        o = AAOracle(threads=1)
        _, radii, _, _ = o.forward(**inp)
        st = o.state()
        gimg = grad_images(H, W, seed)
        t64 = lambda a: torch.tensor(a, dtype=torch.float64)
        ten = {k: t64(inp[k]).requires_grad_(True) for k in KEYS}
        m2d = torch.zeros(len(radii), 3, dtype=torch.float64, requires_grad=True)
        ids = np.nonzero(radii > 0)[0]
        order = ids[np.lexsort((ids, st["depths"][ids]))]
        c, d, a, _ = dense_render_aa(means3D=ten["means3D"], means2D=m2d, opacities=ten["opacities"], viewmatrix=t64(inp["viewmatrix"]),
                                     projmatrix=t64(inp["projmatrix"]), campos=t64(inp["campos"]), bg=t64(inp["bg"]), H=H, W=W,
                                     tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], radii=radii, rect=st["rect"], order=order,
                                     sh_degree=deg, shs=ten["shs"], scales=ten["scales"], rotations=ten["rotations"])
        ((c * t64(gimg[0])).sum() + (d * t64(gimg[1])).sum() + (a * t64(gimg[2])).sum()).backward()
        g = _gpu_grads(inp, gimg, KEYS)
        ref = dict(means2D=m2d.grad.numpy(), **{k: ten[k].grad.numpy() for k in KEYS})
        for k, r in ref.items():
            ok, msg = grads_agree(g[k].reshape(r.shape), r, atol=1e-4, rtol=1e-3)
            assert ok, f"deg {deg}: AA dL/d{k} CUDA vs float64 autograd: {msg}"


def _body(P, deg, seed):
    from humangaussian_b200.scene import synthetic_body
    p = synthetic_body(P, sh_degree=deg, seed=seed)
    p.scaling += math.log(6.0)
    p.opacity += 1.5
    return p.to(DEV)


def test_raw_packed_and_per_view_means():
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.rasterizer import packed_layout, rasterize_views, rasterize_views_packed
    from humangaussian_b200.renderer import stack_cameras
    P, H, W, V, deg = 1500, 72, 104, 3, 3
    K = (deg + 1) ** 2
    p = _body(P, deg, 21)
    vm, pm, cp, tanx, tany = stack_cameras(sample_orbit_cameras(V, H, W, seed=2, device=DEV), DEV)
    bg = torch.tensor([0.1, 0.4, 0.7], device=DEV)
    rng = np.random.RandomState(1)
    gw = [torch.tensor(rng.randn(V, c, H, W).astype(np.float32), device=DEV) for c in (3, 1, 1)]
    kw = dict(viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tanx, tanfovy=tany, image_height=H, image_width=W, bg=bg,
              sh_degree=deg, antialiasing=True)
    loss = lambda c, d, a: (c * gw[0]).sum() + (d * gw[1]).sum() + (a * gw[2]).sum()
    names = ("xyz", "scaling", "rotation", "opacity", "features_dc", "features_rest")
    raw = {k: getattr(p, k).clone().requires_grad_(True) for k in names}
    out0 = rasterize_views(means3D=raw["xyz"], opacities=torch.sigmoid(raw["opacity"]), shs=torch.cat((raw["features_dc"], raw["features_rest"]), 1),
                           scales=torch.exp(raw["scaling"]), rotations=torch.nn.functional.normalize(raw["rotation"]), **kw)
    loss(out0[0], out0[2], out0[3]).backward()
    raw2 = {k: getattr(p, k).clone().requires_grad_(True) for k in names}
    out1 = rasterize_views(means3D=raw2["xyz"], opacities=raw2["opacity"], shs=torch.cat((raw2["features_dc"], raw2["features_rest"]), 1),
                           scales=raw2["scaling"], rotations=raw2["rotation"], raw=True, **kw)
    loss(out1[0], out1[2], out1[3]).backward()
    assert torch.equal(out0[1], out1[1])
    for x, y in zip(out0, out1):
        ok, worst = close(y.detach().float().cpu().numpy(), x.detach().float().cpu().numpy())
        assert ok, worst
    for k in names:
        ok, msg = grads_agree(raw2[k].grad.cpu().numpy(), raw[k].grad.cpu().numpy())
        assert ok, f"raw AA dL/d{k}: {msg}"
    # packed raw == per-tensor raw, bit for bit
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
    ref = [raw2["xyz"].grad, raw2["scaling"].grad, raw2["rotation"].grad, raw2["opacity"].grad,
           torch.cat((raw2["features_dc"].grad, raw2["features_rest"].grad), 1)]
    for (o, m, shape), g in zip(fields, ref):
        ok, msg = grads_agree(flat.grad.narrow(0, o, m).view(shape).cpu().numpy().reshape(P, -1), g.cpu().numpy().reshape(P, -1))
        assert ok, f"packed raw AA gradient field at {o}: {msg}"
    # per-view means [V,P,3]: each view equals a single-view call with that view's positions
    xyz_v = (p.xyz[None] + 0.01 * torch.randn(V, P, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))).contiguous()
    common = dict(opacities=torch.sigmoid(p.opacity), shs=torch.cat((p.features_dc, p.features_rest), 1), scales=torch.exp(p.scaling),
                  rotations=torch.nn.functional.normalize(p.rotation))
    with torch.no_grad():
        outs = rasterize_views(means3D=xyz_v, **common, **kw)
        for v in range(V):
            one = rasterize_views(means3D=xyz_v[v], **common, **dict(kw, viewmatrices=vm[v:v + 1], projmatrices=pm[v:v + 1],
                                                                      camposs=cp[v:v + 1], tanfovx=tanx[v:v + 1], tanfovy=tany[v:v + 1]))
            for x, y in zip(outs, one):
                assert torch.equal(x[v], y[0]), f"per-view means, view {v}"


def test_deterministic_backward_reruns_are_identical():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        inp, _, _ = small_scene(P=2000, deg=2, seed=12, H=96, W=128)
        gimg = grad_images(96, 128, 1)
        st1, s1 = _gpu_blend_state(dict(inp, antialiasing=True), gimg)
        st2, s2 = _gpu_blend_state(dict(inp, antialiasing=True), gimg)
        assert s1.tobytes() == s2.tobytes() and np.array_equal(st1["patch_masks"], st2["patch_masks"])
        g1, g2 = _gpu_grads(inp, gimg, KEYS), _gpu_grads(inp, gimg, KEYS)
        for k in g1:
            assert g1[k].tobytes() == g2[k].tobytes(), k
        _, _, _, o_grads = _aa_oracle(inp, 1)
        for k in g1:
            ok, msg = grads_agree(g1[k].reshape(o_grads[k].shape), o_grads[k])
            assert ok, f"deterministic AA dL/d{k}: {msg}"
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


@pytest.mark.parametrize("det", [False, True])
def test_opts_entry_points_with_the_filter_off_equal_the_plain_ones(monkeypatch, det):
    """b200gs_*_opts with NULL options, and with antialiasing = 0, write the bytes b200gs_forward / _backward write: the
    outputs always, the backward's records and gradients under the deterministic backward (the default one adds with float
    atomics in a scheduling-dependent order, so there the gradients meet grads_agree)."""
    import ctypes as C
    from humangaussian_b200 import rasterizer as R
    L = R.load_library()
    inp, _, _ = small_scene(P=1500, deg=3, seed=13, H=72, W=104)
    gimg = grad_images(72, 104, 2)

    def run():
        _, sums = _gpu_blend_state(inp, gimg)
        return sums, _gpu_grads_plain(inp, gimg)

    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(det, warn_only=True)
    try:
        ref = run()
        for opts in (None, C.byref(R._render_opts(False))):
            with monkeypatch.context() as m:
                m.setattr(L, "b200gs_forward", lambda prm, *a, o=opts: L.b200gs_forward_opts(prm, o, *a))
                m.setattr(L, "b200gs_backward", lambda prm, *a, o=opts: L.b200gs_backward_opts(prm, o, *a))
                m.setattr(L, "b200gs_backward_deterministic", lambda prm, *a, o=opts: L.b200gs_backward_deterministic_opts(prm, o, *a))
                got = run()
            assert not det or got[0].tobytes() == ref[0].tobytes()
            for k in ref[1]:
                if det or k in ("color", "depth", "alpha", "radii"):
                    assert got[1][k].tobytes() == ref[1][k].tobytes(), k
                else:
                    ok, msg = grads_agree(got[1][k], ref[1][k])
                    assert ok, f"{k}: {msg}"
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _gpu_grads_plain(inp, gimg):
    from humangaussian_b200.rasterizer import GaussianRasterizer
    t = _gpu_inputs(inp, KEYS)
    m2d = torch.zeros(inp["means3D"].shape[0], 3, device=DEV, requires_grad=True)
    c, r, d, a = GaussianRasterizer(_settings(inp))(means3D=t["means3D"], means2D=m2d, shs=t["shs"], opacities=t["opacities"],
                                                   scales=t["scales"], rotations=t["rotations"])
    gC, gD, gA = (torch.tensor(g, device=DEV) for g in gimg)
    ((c * gC).sum() + (d * gD).sum() + (a * gA).sum()).backward()
    out = {k: t[k].grad.cpu().numpy() for k in t}
    out.update(means2D=m2d.grad.cpu().numpy(), color=c.detach().cpu().numpy(), depth=d.detach().cpu().numpy(),
               alpha=a.detach().cpu().numpy(), radii=r.cpu().numpy())
    return out


def test_wrappers_agree_with_rasterize_views():
    from humangaussian_b200.animation import pack_frames_u8, render_frames
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer, rasterize_views
    from humangaussian_b200.renderer import PipelineParams, render, render_views, stack_cameras
    from humangaussian_b200.scene import synthetic_body
    H, W, V = 96, 128, 3
    p = synthetic_body(3000, sh_degree=1, seed=2)
    p.scaling += math.log(3.0)
    p = p.to(DEV)
    cams = sample_orbit_cameras(V, H, W, seed=5, device=DEV)
    vm, pm, cp, tanx, tany = stack_cameras(cams, DEV)
    bg = torch.tensor([0.2, 0.1, 0.3], device=DEV)
    with torch.no_grad():
        common = dict(opacities=p.get_opacity, shs=p.get_features, scales=p.get_scaling, rotations=p.get_rotation, sh_degree=1,
                      image_height=H, image_width=W, bg=bg, antialiasing=True)
        ref = rasterize_views(means3D=p.get_xyz, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tanx, tanfovy=tany, **common)
        off = rasterize_views(means3D=p.get_xyz, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tanx, tanfovy=tany,
                              **dict(common, antialiasing=False))
        assert not torch.equal(ref[0], off[0])
        pipe = PipelineParams()
        pipe.antialiasing = True
        s13 = collections.namedtuple("Settings13", list(GaussianRasterizationSettings._fields) + ["antialiasing"])
        for v, cam in enumerate(cams):
            out = render(cam, p, pipe, bg)
            assert torch.equal(out["render"], ref[0][v]) and torch.equal(out["radii"], ref[1][v])
            assert torch.equal(out["depth_3dgs"], ref[2][v]) and torch.equal(out["alpha_3dgs"], ref[3][v])
            s = GaussianRasterizationSettings(H, W, tanx[v], tany[v], bg, 1.0, vm[v], pm[v], 1, cp[v], False, False)
            c, r, d, a = GaussianRasterizer(s13(*s, True))(means3D=p.get_xyz, means2D=torch.zeros_like(p.get_xyz), shs=p.get_features,
                                                           opacities=p.get_opacity, scales=p.get_scaling, rotations=p.get_rotation)
            assert torch.equal(c, ref[0][v]) and torch.equal(r, ref[1][v])
            c, _, _, _ = GaussianRasterizer(s)(means3D=p.get_xyz, means2D=torch.zeros_like(p.get_xyz), shs=p.get_features,
                                               opacities=p.get_opacity, scales=p.get_scaling, rotations=p.get_rotation)
            assert torch.equal(c, off[0][v])  # the 12-field settings keep the filter off
            out = render(cam, p, pipe, bg, fused_activations=True)
            ok, worst = close(out["render"].cpu().numpy(), ref[0][v].cpu().numpy())
            assert ok, worst
        pkg = render_views(cams, p, bg, antialiasing=True)
        for got, want in zip((pkg["render"], pkg["radii"], pkg["depth_3dgs"], pkg["alpha_3dgs"]), ref):
            assert torch.equal(got, want)
        xyz_f = (p.get_xyz[None] + 0.02 * torch.randn(V, 3000, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(0)))
        frames = render_frames(p, xyz_f.contiguous(), cams, bg, antialiasing=True)
        col = rasterize_views(means3D=xyz_f.contiguous(), viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tanx, tanfovy=tany,
                              **common)[0]
        assert torch.equal(frames, pack_frames_u8(col))
