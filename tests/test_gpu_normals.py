"""GPU: the normal maps (rasterize_views(normals=True)) against tests/normal_reference.py, and their properties.

  1. normal images bit for bit against the replay on the oracle's state: degrees 0-3, dense-opaque, 512^2, a 3-view batch,
     per-view means, antialiasing, the 3D filter, screen-space scenes whose patches stage 1, 15, 16, 17, 31, 32, 33 and 64
     hits and partial patches at the image edge; raw parameters against the replay on the GPU forward's own records and
     normals (the device's activations need not equal the host's bit for bit);
  2. colour, depth, alpha, radii and the forward state byte-identical to normals off;
  3. gradients against the float64 two-pass reference (grads_agree at 1e-4 abs / 1e-3 rel), atomic and deterministic:
     degrees 0-3, raw, antialiasing, the 3D filter, the staging / flush boundary scenes, and a 3-view batch with shared and
     with per-view means against the per-view references summed (each view flips its normals its own way);
  4. a zero normal gradient leaves every gradient torch.equal to normals off (deterministic); deterministic reruns are
     byte-identical; with absgrad, means2D_abs matches absgrad alone when gN = 0;
  5. full size (300 k, degree 3, 1024^2, 8 views): the normal image torch.equal to the two-pass workaround's colour image
     (colors_precomp = n_v, bg = 0, one call per view), and the gradients against the plain backward plus the workaround's
     gradients chained through n(q) by torch, at the full-size criterion of test_gpu_fullsize.py;
  6. cov3D_precomp raises ValueError; the packed entry and render_views carry the fifth output; a packed training loop with a
     normal loss runs through a densify."""
import contextlib
import math

import numpy as np
import pytest
import torch

import normal_reference as NR
from util import grad_images, grads_agree, screen_scene, small_scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REF_TOL = dict(atol=1e-4, rtol=1e-3)
KEYS = ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations")


@contextlib.contextmanager
def deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _views(inps):
    g = lambda k: torch.stack([torch.as_tensor(np.asarray(i[k], np.float32)) for i in inps]).to(DEV)
    i0 = inps[0]
    return dict(viewmatrices=g("viewmatrix").reshape(-1, 4, 4), projmatrices=g("projmatrix").reshape(-1, 4, 4),
                camposs=g("campos").reshape(-1, 3), tanfovx=[i["tanfovx"] for i in inps], tanfovy=[i["tanfovy"] for i in inps],
                image_height=i0["image_height"], image_width=i0["image_width"], bg=torch.tensor(i0["bg"], device=DEV),
                sh_degree=i0.get("sh_degree", 0), scale_modifier=i0.get("scale_modifier", 1.0))


def _run(inps, gimgs=None, gN=None, normals=True, det=False, raw=None, means=None, absgrad=False, **opts):
    """rasterize_views over the views `inps`; with gimgs, the backward of sum gC c + gD d + gA a (+ sum gN N).  Returns numpy
    outputs and gradients.  raw: dict of raw opacities / scales / rotations; means: [V,P,3] per-view positions."""
    from humangaussian_b200.rasterizer import rasterize_views
    i0 = inps[0]
    t = {k: torch.tensor(i0[k], device=DEV, requires_grad=True) for k in KEYS if i0.get(k) is not None}
    if raw is not None:
        for k, v in raw.items():
            t[k] = torch.tensor(v, device=DEV, requires_grad=True)
    if means is not None:
        t["means3D"] = torch.tensor(means, device=DEV, requires_grad=True)
    V, P = len(inps), i0["means3D"].shape[0]
    m2d = torch.zeros(V, P, 3, device=DEV, requires_grad=True)
    m2a = torch.zeros(V, P, 3, device=DEV, requires_grad=True) if absgrad else None
    with deterministic(det):
        outs = rasterize_views(means2D=m2d, means2D_abs=m2a, raw=raw is not None, normals=normals, **t, **_views(inps), **opts)
        res = dict(color=outs[0], radii=outs[1], depth=outs[2], alpha=outs[3])
        if normals:
            res["normal"] = outs[4]
        if gimgs is not None:
            gs = [torch.tensor(np.stack([g[j] for g in gimgs]), device=DEV) for j in range(3)]
            ts, gt = [outs[0], outs[2], outs[3]], gs
            if normals and gN is not None:
                ts, gt = ts + [outs[4]], gs + [torch.as_tensor(np.asarray(gN, np.float32), device=DEV)]
            torch.autograd.backward(ts, gt)
            res.update(means2D=m2d.grad, **{k: v.grad for k, v in t.items()})
            if absgrad:
                res["means2D_abs"] = m2a.grad
    return {k: v.detach().cpu().numpy() for k, v in res.items()}


def _small(deg, seed=None, P=60, H=32, W=48, **kw):
    inp, _, p = small_scene(P=P, deg=deg, seed=deg if seed is None else seed, H=H, W=W, **kw)
    return inp, p


def _orbit(inp, V, seed=5):
    from humangaussian_b200.cameras import sample_orbit_cameras
    H, W = inp["image_height"], inp["image_width"]
    return [dict(inp, viewmatrix=c.world_view_transform.cpu().numpy(), projmatrix=c.full_proj_transform.cpu().numpy(),
                 campos=c.camera_center.cpu().numpy(), tanfovx=math.tan(c.FoVx * 0.5), tanfovy=math.tan(c.FoVy * 0.5))
            for c in sample_orbit_cameras(V, H, W, seed=seed)]


def _check_images(inps, raw=None, means=None, gauss=None, **opts):
    """every view's normal image bit for bit against the replay; the other outputs byte-identical to normals off"""
    on = _run(inps, raw=raw, means=means, **opts)
    off = _run(inps, normals=False, raw=raw, means=means, **opts)
    for k in ("color", "depth", "alpha", "radii"):
        assert on[k].tobytes() == off[k].tobytes(), f"{k} changed with normals on"
    aa, f3d = opts.get("antialiasing", False), opts.get("filter_3d")
    for v, inp in enumerate(inps):
        iv = inp if means is None else dict(inp, means3D=means[v])
        nrm = None if gauss is None else gauss[v]
        ref = NR.reference_image(iv, antialiasing=aa, filter_3d=None if f3d is None else f3d.cpu().numpy(), nrm=nrm)
        assert np.array_equal(on["normal"][v], ref), f"view {v}: {int((on['normal'][v] != ref).sum())} normal values differ"
    assert np.abs(on["normal"]).max() > 0.05
    return on


# ---- 1, 2. images ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_images_small(deg):
    inp, _ = _small(deg)
    _check_images([inp])


def test_images_dense_opaque():
    inp, _ = _small(1, seed=9, P=80, H=32, W=32, dist=1.3)
    inp["opacities"] = np.clip(inp["opacities"] * 8, 0, 0.99999).astype(np.float32)
    inp["scales"] = (inp["scales"] * 2.0).astype(np.float32)
    _check_images([inp])


def test_images_512():
    inp, _ = _small(3, seed=11, P=400, H=512, W=512, big=False)
    _check_images([inp])


def test_images_three_views_and_per_view_means():
    inp, _ = _small(2, P=50)
    inps = _orbit(inp, 3)
    _check_images(inps)
    rng = np.random.RandomState(3)
    means = np.stack([inp["means3D"] + (0.02 * rng.randn(*inp["means3D"].shape)).astype(np.float32) for _ in range(3)])
    _check_images(inps, means=means)


def test_images_antialiasing_and_filter3d():
    inp, _ = _small(1, seed=7)
    _check_images([inp], antialiasing=True)
    f3d = torch.full((inp["means3D"].shape[0],), 1e-3, device=DEV)
    _check_images([inp], filter_3d=f3d)


def test_images_raw_against_device_normals():
    from humangaussian_b200.rasterizer import forward_with_state
    inp, p = _small(2, seed=12)
    raw = dict(opacities=p.opacity.detach().numpy().copy(), scales=p.scaling.detach().numpy().copy(),
               rotations=(p.rotation.detach().numpy() * 1.7).astype(np.float32))
    kw = dict(means3D=torch.tensor(inp["means3D"], device=DEV), shs=torch.tensor(inp["shs"], device=DEV), sh_degree=2,
              bg=torch.tensor(inp["bg"], device=DEV), viewmatrix=torch.tensor(inp["viewmatrix"], device=DEV),
              projmatrix=torch.tensor(inp["projmatrix"], device=DEV), campos=torch.tensor(inp["campos"], device=DEV),
              tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], image_height=32, image_width=48, raw=True, normals=True,
              **{k: torch.tensor(v, device=DEV) for k, v in raw.items()})
    _, _, _, _, normal, state, _ = forward_with_state(**kw)
    gn = state["gauss_normals"].cpu().numpy()
    ref_n = NR.gauss_normals(inp["means3D"], inp["campos"], raw["scales"], raw["rotations"], raw=True)
    assert np.array_equal(gn[:, 3], ref_n[:, 3]) and np.abs(gn - ref_n).max() < 1e-6
    # the replay on the GPU forward's own records (centre, conic, opacity), sorted lists and normals: bit for bit
    recs = state["recs"].cpu().numpy()
    st = dict(xy=recs[:, :2], conic_opacity=recs[:, 4:8], point_list=state["point_list"].cpu().numpy(),
              ranges=state["ranges"].cpu().numpy())
    ref = NR.normal_image(st, 32, 48, gn)
    assert np.abs(ref).max() > 0.05
    assert np.array_equal(normal[0].cpu().numpy(), ref), f"{int((normal[0].cpu().numpy() != ref).sum())} values differ"
    # and through rasterize_views: the same image, the other outputs byte-identical to normals off
    on, off = _run([inp], raw=raw), _run([inp], normals=False, raw=raw)
    assert np.array_equal(on["normal"][0], ref)
    for k in ("color", "depth", "alpha", "radii"):
        assert on[k].tobytes() == off[k].tobytes(), k


def test_forward_state_unchanged():
    from humangaussian_b200.rasterizer import forward_with_state
    inp, _ = _small(3, seed=2, P=120)
    kw = {k: (torch.tensor(v, device=DEV) if isinstance(v, np.ndarray) else v) for k, v in inp.items()}
    a = forward_with_state(**kw)
    b = forward_with_state(normals=True, **kw)
    for k in ("recs", "point_list", "ranges", "n_contrib", "final_T", "sorted_keys"):
        assert torch.equal(a[4][k], b[5][k]), k
    assert a[4]["num_rendered"] == b[5]["num_rendered"]


# ---- 3. gradients -----------------------------------------------------------------------------------------------------
def _gN(H, W, seed):
    return np.random.RandomState(100 + seed).randn(3, H, W).astype(np.float32)


def _check_grads(inp, seed, raw=None, aa=False, f3d=None):
    H, W = inp["image_height"], inp["image_width"]
    gimg, gN = grad_images(H, W, seed), _gN(H, W, seed)
    ref, _ = NR.reference_grads(inp, gimg, gN, antialiasing=aa, filter_3d=f3d, raw=raw)
    opts = dict(antialiasing=aa, filter_3d=None if f3d is None else torch.tensor(f3d, device=DEV))
    for det in (False, True):
        g = _run([inp], [gimg], gN[None], det=det, raw=raw, **opts)
        for k, r in ref.items():
            ok, msg = grads_agree(g[k].reshape(r.shape[0], -1), r.reshape(r.shape[0], -1), **REF_TOL)
            assert ok, f"deterministic={det} {k}: {msg}"


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_grads_small(deg):
    inp, _ = _small(deg)
    _check_grads(inp, deg)


def test_grads_raw():
    inp, p = _small(1, seed=13)
    raw = dict(opacities=p.opacity.detach().numpy().copy(), scales=p.scaling.detach().numpy().copy(),
               rotations=(p.rotation.detach().numpy() * 1.3).astype(np.float32))
    _check_grads(inp, 5, raw=raw)


def test_grads_antialiasing_and_filter3d():
    inp, _ = _small(2, seed=14)
    _check_grads(inp, 6, aa=True)
    _check_grads(inp, 7, f3d=np.full(inp["means3D"].shape[0], 1e-3, np.float32))


# ---- 4. zero gradient, determinism, absgrad ----------------------------------------------------------------------------
def test_zero_normal_gradient_is_normals_off():
    inp, _ = _small(3, seed=15, P=100)
    gimg = grad_images(32, 48, 3)
    off = _run([inp], [gimg], normals=False, det=True)
    for gN in (None, np.zeros((1, 3, 32, 48), np.float32)):
        on = _run([inp], [gimg], gN, det=True)
        for k in off:
            if k != "normal":
                assert torch.equal(torch.as_tensor(on[k]), torch.as_tensor(off[k])), k


def test_deterministic_reruns_and_absgrad():
    inps = _orbit(_small(2, seed=16, P=80)[0], 2)
    gimgs = [grad_images(32, 48, v) for v in range(2)]
    gN = np.stack([_gN(32, 48, v) for v in range(2)])
    a = _run(inps, gimgs, gN, det=True, absgrad=True)
    b = _run(inps, gimgs, gN, det=True, absgrad=True)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    plain = _run(inps, gimgs, normals=False, det=True, absgrad=True)
    zero = _run(inps, gimgs, np.zeros_like(gN), det=True, absgrad=True)
    assert np.array_equal(zero["means2D_abs"], plain["means2D_abs"])
    # atomic and deterministic agree
    c = _run(inps, gimgs, gN, det=False, absgrad=True)
    for k in ("rotations", "opacities", "means3D"):
        ok, msg = grads_agree(c[k].reshape(len(c[k]), -1), a[k].reshape(len(a[k]), -1), atol=1e-5, rtol=1e-4)
        assert ok, f"{k}: {msg}"


# ---- 5. restrictions and the other entry points -----------------------------------------------------------------------
def test_cov3d_precomp_raises():
    from humangaussian_b200.rasterizer import rasterize_views
    inp, _ = _small(0)
    t = {k: torch.tensor(inp[k], device=DEV) for k in ("means3D", "opacities", "shs")}
    with pytest.raises(ValueError):
        rasterize_views(cov3D_precomp=torch.zeros(inp["means3D"].shape[0], 6, device=DEV), normals=True, **t, **_views([inp]))


def test_packed_matches_unpacked_and_trains():
    from humangaussian_b200.rasterizer import packed_layout, rasterize_views_packed
    inp, p = _small(3, seed=17, P=64)
    P, K = 64, 16
    layout, total = packed_layout(P, K)
    flat = torch.zeros(total, device=DEV)
    raw = dict(opacities=p.opacity.detach().numpy().copy(), scales=p.scaling.detach().numpy().copy(),
               rotations=p.rotation.detach().numpy().copy())
    for (o, n, shape), v in zip(layout, (inp["means3D"], raw["scales"], raw["rotations"], raw["opacities"], inp["shs"])):
        flat[o:o + n] = torch.tensor(np.asarray(v, np.float32).reshape(-1), device=DEV)
    flat.requires_grad_(True)
    gimg, gN = grad_images(32, 48, 9), _gN(32, 48, 9)
    with deterministic(True):
        outs = rasterize_views_packed(flat, P, K, raw=True, normals=True, **_views([inp]))
        gs = [torch.tensor(g[None], device=DEV) for g in gimg]
        torch.autograd.backward([outs[0], outs[2], outs[3], outs[4]], [gs[0], gs[1], gs[2], torch.tensor(gN[None], device=DEV)])
    ref = _run([inp], [gimg], gN[None], det=True, raw=raw)
    assert np.array_equal(outs[4].detach().cpu().numpy(), ref["normal"])
    o, n, _ = layout[2]
    assert np.array_equal(flat.grad[o:o + n].cpu().numpy().reshape(P, 4), ref["rotations"])
    # a few steps of a normal-consistency loss move the normals toward a target
    target = torch.tensor([0.0, 0.0, -1.0], device=DEV).view(1, 3, 1, 1)
    opt = torch.optim.Adam([flat], lr=1e-2)
    losses = []
    for _ in range(15):
        opt.zero_grad()
        c, r, d, a, nm = rasterize_views_packed(flat, P, K, raw=True, normals=True, **_views([inp]))
        loss = ((nm - target * a) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert np.isfinite(losses).all() and losses[-1] < losses[0]


def test_render_views_comp_normal():
    from humangaussian_b200.renderer import comp_normal, render_views
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.scene import synthetic_body
    pc = synthetic_body(500, sh_degree=1, seed=1).to(DEV)
    pc.rotation.requires_grad_(True)
    cams = sample_orbit_cameras(2, 32, 48, seed=3)
    out = render_views(cams, pc, torch.zeros(3, device=DEV), normals=True)
    assert out["normal_3dgs"].shape == (2, 3, 32, 48) and out["comp_normal"].shape == (2, 32, 48, 3)
    cn = out["comp_normal"]
    assert torch.equal(cn, comp_normal(out["normal_3dgs"], out["alpha_3dgs"]))
    assert float(cn.min()) >= 0 and float(cn.max()) <= 1.0 + 1e-6
    cn.sum().backward()
    assert pc.rotation.grad is not None and float(pc.rotation.grad.abs().sum()) > 0


# ---- staging and flush boundaries -----------------------------------------------------------------------------------------
def _screen_rs(g, sigma, H, W, seed):
    """screen_scene's Gaussians with scales and rotations in place of its diagonal covariance: per Gaussian the scales
    (1, 0.7, 0.85) * (sigma px at its depth) in a random order and a random rotation, so the screen footprint stays within
    sigma while the normals point every way"""
    inp = screen_scene(g["px"], g["py"], g["depth"], sigma, g["opacity"], H=H, W=W)
    s = np.sqrt(inp.pop("cov3D_precomp")[:, 0].astype(np.float64))
    rng = np.random.RandomState(seed)
    n = len(s)
    fac = np.stack([rng.permutation([1.0, 0.7, 0.85]) for _ in range(n)])
    q = rng.randn(n, 4)
    inp["scales"] = (s[:, None] * fac).astype(np.float32)
    inp["rotations"] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    return inp


def _stack(x, y, n, z0, opacity=0.05):
    return dict(px=np.full(n, x), py=np.full(n, y), depth=z0 + 1e-3 * np.arange(n), opacity=np.full(n, opacity))


def _cat(parts):
    return {k: np.concatenate([p[k] for p in parts]) for k in ("px", "py", "depth", "opacity")}


def test_flush_boundaries():
    """stacks of 1, 15, 16, 17, 31, 32, 33 and 64 hits, each in patch 0 of its own tile: the backward's 16-slot flushes end
    at n mod 16 = 0, 1, 15, the forward's 32-entry chunks at 31, 32, 33; sigma 0.6 px so every hit covers several pixels"""
    counts = (1, 15, 16, 17, 31, 32, 33, 64)
    inp = _screen_rs(_cat([_stack(16 * i + 3.5, 1.5, n, 1.0 + i) for i, n in enumerate(counts)]), 0.6, 16, 128, seed=1)
    _check_images([inp])
    _check_grads(inp, 41)


def test_partial_edge_patches():
    """stacks in the partial patches of a 123x61 image: cols 120-122 and row 60"""
    parts = [_stack(121.0, 9.5, 17, 1.0), _stack(121.0, 60.45, 15, 2.0), _stack(51.5, 60.45, 33, 3.0), _stack(3.5, 60.45, 1, 4.0)]
    inp = _screen_rs(_cat(parts), 0.6, 61, 123, seed=2)
    _check_images([inp])
    _check_grads(inp, 42)


# ---- multi-view gradients ---------------------------------------------------------------------------------------------
def _check_grads_views(inps, seed, means=None):
    """a V-view batch against the float64 reference of each view, summed over the views (per-view means: stacked)"""
    H, W = inps[0]["image_height"], inps[0]["image_width"]
    gimgs = [grad_images(H, W, seed + v) for v in range(len(inps))]
    gNs = np.stack([_gN(H, W, seed + v) for v in range(len(inps))])
    refs = [NR.reference_grads(inp if means is None else dict(inp, means3D=means[v]), gimgs[v], gNs[v])[0]
            for v, inp in enumerate(inps)]
    ref = {k: np.sum([r[k] for r in refs], 0) for k in refs[0]}
    if means is not None:
        ref["means3D"] = np.stack([r["means3D"] for r in refs])
    for det in (False, True):
        g = _run(inps, gimgs, gNs, det=det, means=means)
        for k, r in ref.items():
            rows = r.shape[0] if r.ndim < 3 or k != "means3D" else r.shape[0] * r.shape[1]
            ok, msg = grads_agree(g[k].reshape(rows, -1), r.reshape(rows, -1), **REF_TOL)
            assert ok, f"deterministic={det} {k}: {msg}"


def test_grads_three_views_and_per_view_means():
    inp, _ = _small(2, seed=18, P=50)
    inps = _orbit(inp, 3, seed=6)
    flips = np.stack([NR.gauss_normals(i["means3D"], i["campos"], i["scales"], i["rotations"])[:, 3] for i in inps])
    assert (flips != flips[:1]).any(), "the views should flip some normals differently"
    _check_grads_views(inps, 50)
    rng = np.random.RandomState(4)
    means = np.stack([inp["means3D"] + (0.02 * rng.randn(*inp["means3D"].shape)).astype(np.float32) for _ in range(3)])
    _check_grads_views(inps, 60, means=means)


# ---- full size --------------------------------------------------------------------------------------------------------
FULL_SIZE = dict(min_rows=1.0 - 1e-4, row_cap=4.0, min_elementwise=0.999)  # test_gpu_fullsize.py's full-size row criterion


def test_full_size_against_the_two_pass_workaround():
    from humangaussian_b200 import rasterizer as R
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import stack_cameras
    from humangaussian_b200.scene import sample_ply_scene
    p = sample_ply_scene(300000, 3)
    with torch.no_grad():
        base = {k: v.detach().float().to(DEV).contiguous() for k, v in dict(
            means3D=p.get_xyz, opacities=p.get_opacity, shs=p.get_features, scales=p.get_scaling, rotations=p.get_rotation).items()}
    P, V, H = base["means3D"].shape[0], 8, 1024
    vm, pm, cp, tx, ty = stack_cameras(sample_orbit_cameras(64, H, H, seed=1000)[:V], DEV)
    cam = lambda s: dict(viewmatrices=vm[s], projmatrices=pm[s], camposs=cp[s], tanfovx=tx[s], tanfovy=ty[s], image_height=H,
                         image_width=H)
    bg, zero = torch.tensor([0.1, 0.4, 0.7], device=DEV), torch.zeros(3, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(0)
    gC, gD, gA, gN = (torch.randn(V, c, H, H, device=DEV, generator=gen) for c in (3, 1, 1, 3))
    # the GPU's own normals: the workaround's colours are these bits (F1 passes colors_precomp through unchanged)
    st = R.forward_with_state(viewmatrix=vm, projmatrix=pm, campos=cp, tanfovx=tx, tanfovy=ty, image_height=H, image_width=H,
                              bg=bg, sh_degree=3, normals=True, **base)[5]
    gauss = st["gauss_normals"].reshape(V, P, 4)
    leaves = lambda: {k: v.clone().requires_grad_(True) for k, v in base.items()}
    with deterministic():
        t = leaves()
        # start the partial-capacity hint low, so this call goes through the deterministic retry with pooled normal partials
        R._partial_hint[(DEV.index or 0, P, V, H, H)] = 1 << 16
        c, r, d, a, nm = R.rasterize_views(bg=bg, sh_degree=3, normals=True, **t, **cam(slice(0, V)))
        torch.autograd.backward([c, d, a, nm], [gC, gD, gA, gN])
        assert R.last_num_partials() > 1 << 16
        u = leaves()
        c2, r2, d2, a2 = R.rasterize_views(bg=bg, sh_degree=3, **u, **cam(slice(0, V)))
        for x, y in ((c, c2), (r, r2), (d, d2), (a, a2)):
            assert torch.equal(x, y)
        torch.autograd.backward([c2, d2, a2], [gC, gD, gA])
        k = base["scales"].argmin(1)  # the first index of the minimum, as the kernels take it
        for v in range(V):
            n_t = NR.normals_torch(u["rotations"], k, gauss[v, :, 3])
            n_v = gauss[v, :, :3] + (n_t - n_t.detach())  # the GPU's values, the torch expression's gradient
            img = R.rasterize_views(means3D=u["means3D"], opacities=u["opacities"], colors_precomp=n_v, scales=u["scales"],
                                    rotations=u["rotations"], bg=zero, **cam(slice(v, v + 1)))[0]
            assert torch.equal(img[0], nm[v].detach()), f"view {v}: normal image differs from the workaround's"
            torch.autograd.backward([img], [gN[v:v + 1]])
    for key in ("means3D", "opacities", "shs", "scales", "rotations"):
        ok, msg = grads_agree(t[key].grad.cpu().numpy().reshape(P, -1), u[key].grad.cpu().numpy().reshape(P, -1), **FULL_SIZE)
        assert ok, f"{key}: {msg}"


# ---- training through a densify ---------------------------------------------------------------------------------------
def test_packed_training_loop_with_normal_loss_densifies():
    """20 packed raw steps with PackedAdam and a normal loss; a densify after step 10 changes P, and the loop keeps rendering
    normals at the new size (gauss_normals, normal_wn and the pooled buffers sized from it)"""
    from humangaussian_b200 import dist as D
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.densify import DensifyStats, add_densification_stats, densify_and_prune_packed
    from humangaussian_b200.optim import PackedAdam, expon_lr_func
    from humangaussian_b200.rasterizer import rasterize_views_packed
    from humangaussian_b200.renderer import comp_normal, stack_cameras
    _, _, sc = small_scene(P=3001, deg=3, seed=4)
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
    sizes = []
    for it in range(20):
        opt.update_learning_rate(it)
        m2d = torch.zeros(4, opt.P, 3, device=DEV, requires_grad=True)
        color, radii, _, alpha, normal = rasterize_views_packed(
            opt.packed, opt.P, K, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx, tanfovy=ty, image_height=H,
            image_width=H, bg=bg, sh_degree=3, means2D=m2d, raw=True, normals=True)
        cn = comp_normal(normal, alpha)
        n = torch.nn.functional.normalize(normal, dim=1)
        smooth = (n[..., 1:, :] - n[..., :-1, :]).abs().mean() + (n[..., :, 1:] - n[..., :, :-1]).abs().mean()
        loss = (color - bg.view(1, 3, 1, 1)).square().mean() + 0.1 * smooth
        loss.backward()
        assert math.isfinite(loss.item()) and torch.isfinite(opt.packed.grad).all() and torch.isfinite(cn).all()
        sizes.append(opt.P)
        add_densification_stats(stats, m2d.grad, radii)
        opt.step()
        opt.zero_grad()
        if it == 9:
            thr = float(torch.quantile((stats.xyz_gradient_accum / stats.denom.clamp_min(1)).flatten(), 0.8))
            densify_and_prune_packed(opt, stats, thr, 0.005, 1.0, None, generator=torch.Generator(device=DEV).manual_seed(7))
    assert sizes[0] == 3001 and sizes[-1] != 3001, sizes
    assert torch.isfinite(opt.packed).all()

