"""GPU: the geometry outputs (rasterize_views(geometry=True)) against tests/geometry_reference.py, and their properties.

  1. median and depth2 images bit for bit against the replay on the oracle's state: degrees 0-3, dense-opaque, 512^2, a
     3-view batch, per-view means, antialiasing + the 3D filter, cov3D_precomp, one full-size 300 k / 1024^2 view; raw
     parameters against the replay on the GPU forward's own records;
  2. colour, depth, alpha, normals, radii and the forward state byte-identical to geometry off;
  3. gradients against the float64 reference (grads_agree at 1e-4 abs / 1e-3 rel), atomic and deterministic, with random
     gC, gD, gA, gM2, gMed: small scenes, raw, antialiasing + the 3D filter, with normals on, a 3-view batch, and screen-space
     scenes whose median hits straddle the 16-hit flushes and whose patches are cut by the image edge;
  4. the W3 fold against the reference's float64 sum under |gpu - ref| <= 10 u E (E from geometry_reference.replay; the
     bound of DESIGN.md section 2, "Geometry outputs", fixed before the first GPU run);
  5. zero geometry gradients give gradients torch.equal to geometry off; deterministic reruns with absgrad and normals on are
     byte-identical;
  6. the packed entry equals the unpacked one; render / render_views return the geometry keys; a short packed training
     loop with a distortion + depth-normal consistency term lowers the mean distortion inside the silhouette."""
import contextlib
import math

import numpy as np
import pytest
import torch

import geometry_reference as GR
from util import grad_images, grads_agree, screen_scene, small_scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REF_TOL = dict(atol=1e-4, rtol=1e-3)
KEYS = ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp")
U = 2.0 ** -24


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


def _run(inps, gimgs=None, gM2=None, gMed=None, gN=None, geometry=True, normals=False, det=False, raw=None, means=None,
         absgrad=False, **opts):
    """rasterize_views over the views `inps`; with gimgs, the backward of sum gC c + gD d + gA a (+ gM2 M2 + gMed median + gN N
    where given).  Returns numpy outputs and gradients."""
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
        outs = rasterize_views(means2D=m2d, means2D_abs=m2a, raw=raw is not None, normals=normals, geometry=geometry, **t,
                               **_views(inps), **opts)
        res = dict(color=outs[0], radii=outs[1], depth=outs[2], alpha=outs[3])
        if normals:
            res["normal"] = outs[4]
        if geometry:
            res["median"], res["depth2"] = outs[4 + normals], outs[5 + normals]
        if gimgs is not None:
            gs = [torch.tensor(np.stack([g[j] for g in gimgs]), device=DEV) for j in range(3)]
            ts, gt = [outs[0], outs[2], outs[3]], gs
            for key, gx in (("normal", gN), ("median", gMed), ("depth2", gM2)):
                if gx is not None and key in res:
                    ts, gt = ts + [res[key]], gt + [torch.as_tensor(np.asarray(gx, np.float32), device=DEV)]
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


def _check_images(inps, means=None, normals=False, **opts):
    """every view's median and depth2 bit for bit against the replay; the other outputs byte-identical to geometry off"""
    on = _run(inps, means=means, normals=normals, **opts)
    off = _run(inps, means=means, normals=normals, geometry=False, **opts)
    for k in ("color", "depth", "alpha", "radii") + (("normal",) if normals else ()):
        assert on[k].tobytes() == off[k].tobytes(), f"{k} changed with geometry on"
    aa, f3d = opts.get("antialiasing", False), opts.get("filter_3d")
    for v, inp in enumerate(inps):
        iv = inp if means is None else dict(inp, means3D=means[v])
        ref = GR.reference_images(iv, antialiasing=aa, filter_3d=None if f3d is None else f3d.cpu().numpy())
        for k in ("median", "depth2"):
            assert np.array_equal(on[k][v, 0], ref[k]), f"view {v}: {int((on[k][v, 0] != ref[k]).sum())} {k} values differ"
    assert on["depth2"].max() > 0 and (on["median"] > 0).any()
    return on


# ---- 1, 2. images --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_images_small(deg):
    inp, _ = _small(deg)
    _check_images([inp])


def test_images_dense_opaque():
    inp, _ = _small(1, seed=9, P=80, H=32, W=32, dist=1.3)
    inp["opacities"] = np.clip(inp["opacities"] * 8, 0, 0.99999).astype(np.float32)
    inp["scales"] = (inp["scales"] * 2.0).astype(np.float32)
    _check_images([inp], normals=True)


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


def test_images_antialiasing_filter3d_and_cov3d_precomp():
    inp, _ = _small(1, seed=7)
    f3d = torch.full((inp["means3D"].shape[0],), 1e-3, device=DEV)
    _check_images([inp], antialiasing=True, filter_3d=f3d)
    sc = screen_scene(np.arange(20) * 5.3 + 3, (np.arange(20) % 5) * 6.1 + 4, 1.0 + 0.1 * np.arange(20), 2.5,
                      0.4 + 0.02 * np.arange(20), H=40, W=112)
    _check_images([sc])


def test_images_raw_against_device_records():
    from humangaussian_b200.rasterizer import forward_with_state
    inp, p = _small(2, seed=12)
    raw = dict(opacities=p.opacity.detach().numpy().copy(), scales=p.scaling.detach().numpy().copy(),
               rotations=(p.rotation.detach().numpy() * 1.7).astype(np.float32))
    kw = dict(means3D=torch.tensor(inp["means3D"], device=DEV), shs=torch.tensor(inp["shs"], device=DEV), sh_degree=2,
              bg=torch.tensor(inp["bg"], device=DEV), viewmatrix=torch.tensor(inp["viewmatrix"], device=DEV),
              projmatrix=torch.tensor(inp["projmatrix"], device=DEV), campos=torch.tensor(inp["campos"], device=DEV),
              tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], image_height=32, image_width=48, raw=True, geometry=True,
              **{k: torch.tensor(v, device=DEV) for k, v in raw.items()})
    _, _, _, _, median, depth2, state, _ = forward_with_state(**kw)
    recs = state["recs"].cpu().numpy()
    st = dict(xy=recs[:, :2], conic_opacity=recs[:, 4:8], point_list=state["point_list"].cpu().numpy(),
              ranges=state["ranges"].cpu().numpy(), depths=recs[:, 11])
    ref = GR.replay(st, 32, 48)
    assert ref["depth2"].max() > 0
    assert np.array_equal(median[0, 0].cpu().numpy(), ref["median"])
    assert np.array_equal(depth2[0, 0].cpu().numpy(), ref["depth2"])
    assert np.array_equal(state["median_pos"][0].cpu().numpy().astype(np.uint32), ref["median_pos"])


def test_forward_state_unchanged():
    from humangaussian_b200.rasterizer import forward_with_state
    inp, _ = _small(3, seed=2, P=120)
    kw = {k: (torch.tensor(v, device=DEV) if isinstance(v, np.ndarray) else v) for k, v in inp.items()}
    a = forward_with_state(**kw)
    b = forward_with_state(geometry=True, normals=True, **kw)
    for k in ("recs", "point_list", "ranges", "n_contrib", "final_T", "sorted_keys"):
        assert torch.equal(a[4][k], b[-2][k]), k
    assert a[4]["num_rendered"] == b[-2]["num_rendered"]


def test_images_full_size_view():
    """300 k Gaussians, degree 3, one 1024^2 view (too large for the numpy replay): depth2 torch.equal to the two-pass
    workaround's colour channel 0 (colors_precomp = (d*d, 0, 0) from the records' own depths, bg = 0: the same fma chain),
    every median equal to the record depth at its list position, and the other outputs byte-identical to geometry off"""
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.rasterizer import forward_with_state
    from humangaussian_b200.scene import synthetic_body
    pc = synthetic_body(300_000, sh_degree=3, seed=0)
    c = sample_orbit_cameras(1, 1024, 1024, seed=0)[0]
    kw = dict(means3D=pc.get_xyz, opacities=pc.get_opacity, shs=pc.get_features, scales=pc.get_scaling,
              rotations=pc.get_rotation, viewmatrix=c.world_view_transform, projmatrix=c.full_proj_transform,
              campos=c.camera_center, tanfovx=math.tan(c.FoVx * 0.5), tanfovy=math.tan(c.FoVy * 0.5), image_height=1024,
              image_width=1024, sh_degree=3, bg=torch.ones(3))
    kw = {k: (v.detach().float().to(DEV).contiguous() if torch.is_tensor(v) else v) for k, v in kw.items()}
    on = forward_with_state(geometry=True, **kw)
    off = forward_with_state(**kw)
    for i in range(4):
        assert torch.equal(on[i], off[i]), i
    median, depth2, state = on[4][0, 0], on[5][0, 0], on[6]
    d = state["recs"][:, 11].contiguous()
    two = forward_with_state(**dict(kw, shs=None, sh_degree=0, bg=torch.zeros(3, device=DEV),
                                    colors_precomp=torch.stack([d * d, torch.zeros_like(d), torch.zeros_like(d)], 1)))
    assert torch.equal(depth2, two[0][0, 0]) and float(depth2.max()) > 0
    pos = state["median_pos"][0].long()
    ys, xs = torch.nonzero(pos > 0, as_tuple=True)
    assert len(ys) > 100_000
    tile = (ys // 16) * 64 + xs // 16
    j = state["ranges"][tile, 0].long() + pos[ys, xs] - 1
    g = state["point_list"][j].long()
    assert torch.equal(median[ys, xs], d[g])
    assert torch.all(median[pos == 0] == 0)


# ---- 3, 4. gradients and the W3 fold ---------------------------------------------------------------------------------------
def _ggeo(H, W, seed):
    rng = np.random.RandomState(200 + seed)
    return rng.randn(1, H, W).astype(np.float32), rng.randn(1, H, W).astype(np.float32)


def _check_grads(inp, seed, raw=None, aa=False, f3d=None, normals=False, dets=(False, True)):
    H, W = inp["image_height"], inp["image_width"]
    gimg = grad_images(H, W, seed)
    gM2, gMed = _ggeo(H, W, seed)
    gN = np.random.RandomState(300 + seed).randn(3, H, W).astype(np.float32) if normals else None
    ref, _ = GR.reference_grads(inp, gimg, gM2[0], gMed[0], antialiasing=aa, filter_3d=f3d, raw=raw, gN=gN)
    opts = dict(antialiasing=aa, filter_3d=None if f3d is None else torch.tensor(f3d, device=DEV))
    for det in dets:
        g = _run([inp], [gimg], gM2[None], gMed[None], None if gN is None else gN[None], det=det, raw=raw, normals=normals,
                 **opts)
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


def test_grads_antialiasing_filter3d_and_normals():
    inp, _ = _small(2, seed=14)
    _check_grads(inp, 6, aa=True, f3d=np.full(inp["means3D"].shape[0], 1e-3, np.float32))
    _check_grads(inp, 7, normals=True)


def test_grads_three_views():
    inp, _ = _small(2, P=50, seed=21)
    inps = _orbit(inp, 3)
    H, W = 32, 48
    gimgs = [grad_images(H, W, 30 + v) for v in range(3)]
    geo = [_ggeo(H, W, 30 + v) for v in range(3)]
    refs = [GR.reference_grads(iv, gimgs[v], geo[v][0][0], geo[v][1][0])[0] for v, iv in enumerate(inps)]
    for det in (False, True):
        g = _run(inps, gimgs, np.stack([x[0] for x in geo]), np.stack([x[1] for x in geo]), det=det)
        for k in refs[0]:
            r = sum(rf[k] for rf in refs)
            ok, msg = grads_agree(g[k].reshape(r.shape[0], -1), r.reshape(r.shape[0], -1), **REF_TOL)
            assert ok, f"deterministic={det} {k}: {msg}"


def _check_fold(inp, seed, det):
    """W3 of every (view, Gaussian) against the float64 fold, |gpu - ref| <= 10 u E"""
    from humangaussian_b200.rasterizer import forward_backward_with_state
    H, W = inp["image_height"], inp["image_width"]
    gimg = grad_images(H, W, seed)
    gM2, gMed = _ggeo(H, W, seed)
    kw = {k: (torch.tensor(v, device=DEV) if isinstance(v, np.ndarray) else v) for k, v in inp.items()}
    with deterministic(det):
        *_, sums = forward_backward_with_state(*[torch.tensor(g[None], device=DEV) for g in gimg],
                                               g_median=torch.tensor(gMed[None], device=DEV),
                                               g_depth2=torch.tensor(gM2[None], device=DEV), geometry=True, **kw)
    st, _ = GR.oracle_state(inp)
    r = GR.replay(st, H, W, gD=gimg[1][0].astype(np.float64), gM2=gM2[0].astype(np.float64), gMed=gMed[0].astype(np.float64))
    w3 = sums[0, :, 9].cpu().numpy().astype(np.float64)
    err = np.abs(w3 - r["W3"])
    bound = 10 * U * r["E"]
    assert (r["median_gauss"] >= 0).sum() > 50 and np.abs(r["W3"]).max() > 0.1
    worst = int(np.argmax(err / np.maximum(bound, 1e-30)))
    assert np.all(err <= bound), f"W3 row {worst}: |gpu - ref| = {err[worst]:.3e} > bound {bound[worst]:.3e}"
    return float((err / np.maximum(bound, 1e-30)).max())


@pytest.mark.parametrize("det", [False, True])
def test_w3_fold_bound(det):
    inp, _ = _small(3, seed=22, P=200)
    _check_fold(inp, 8, det)
    inp, _ = _small(1, seed=9, P=80, H=32, W=32, dist=1.3)
    inp["opacities"] = np.clip(inp["opacities"] * 8, 0, 0.99999).astype(np.float32)
    _check_fold(inp, 9, det)


# ---- flush boundaries and partial patches ----------------------------------------------------------------------------------
def _stack(x, y, n, z0, opacity, sigma_jitter=0.0):
    return dict(px=np.full(n, x) + sigma_jitter * np.sin(np.arange(n)), py=np.full(n, y), depth=z0 + 1e-2 * np.arange(n),
                opacity=np.full(n, opacity))


def _cat(parts):
    return {k: np.concatenate([p[k] for p in parts]) for k in ("px", "py", "depth", "opacity")}


def test_flush_boundaries():
    """stacks of 17, 33, 64 and 16 hits, each in patch 0 of its own tile, with per-hit opacities that put T = 1/2 near hit 16,
    32 and 60: within one patch the medians land on both sides of the backward's 16-slot flushes (15-17, 31-33) and in the
    last flush of a 64-hit run; sigma 8 px so every hit covers the patch with slightly different alphas per pixel"""
    parts = [_stack(32 * 0 + 3.5, 1.5, 17, 1.0, 0.047, 1.0), _stack(32 * 1 + 3.5, 1.5, 33, 2.0, 0.0225, 1.0),
             _stack(32 * 2 + 3.5, 1.5, 64, 3.0, 0.0118, 1.0), _stack(32 * 3 + 3.5, 1.5, 16, 4.0, 0.05, 1.0)]
    g = _cat(parts)
    inp = screen_scene(g["px"], g["py"], g["depth"], 8.0, g["opacity"], H=16, W=128)
    _check_images([inp])
    pos = GR.reference_images(inp)["median_pos"][:4]
    p0, p1, p2 = (set(pos[:, 32 * i:32 * i + 8].ravel().tolist()) for i in range(3))
    assert min(p0) <= 16 < max(p0) and min(p1) <= 32 < max(p1) and min(p2) > 48, (p0, p1, p2)
    _check_grads(inp, 10)


def test_partial_edge_patches():
    """600 Gaussians over a 123x61 image, whose last column band (120-122) and last row (60) are partial patches.  The
    screen scene's flat covariances become scales and rotations (as test_gpu_normals' stacks do): the gradient of a
    near-degenerate cov3D_precomp entry is a cancellation where elementwise error means nothing"""
    rng = np.random.RandomState(4)
    n = 600
    inp = screen_scene(rng.uniform(-2, 125, n), rng.uniform(-2, 63, n), rng.uniform(1, 3, n), rng.uniform(0.5, 3, n),
                       rng.uniform(0.1, 0.9, n), H=61, W=123)
    s = np.sqrt(inp.pop("cov3D_precomp")[:, 0].astype(np.float64))
    q = rng.randn(n, 4)
    inp["scales"] = (s[:, None] * np.stack([rng.permutation([1.0, 0.7, 0.85]) for _ in range(n)])).astype(np.float32)
    inp["rotations"] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    on = _check_images([inp])
    assert (on["median"][0, 0, 60] > 0).any() and (on["median"][0, 0, :, 120:] > 0).any()
    _check_grads(inp, 11)


# ---- 5. zero gradients and determinism -------------------------------------------------------------------------------------
def test_zero_geometry_gradients_are_geometry_off():
    inp, _ = _small(3, seed=15, P=100)
    gimg = grad_images(32, 48, 3)
    off = _run([inp], [gimg], geometry=False, det=True)
    z = np.zeros((1, 1, 32, 48), np.float32)
    for gM2, gMed in ((None, None), (z, z), (z, None), (None, z)):
        on = _run([inp], [gimg], gM2, gMed, det=True)
        for k in off:
            if k in ("median", "depth2"):
                continue
            assert torch.equal(torch.tensor(on[k]), torch.tensor(off[k])), k


def test_deterministic_reruns_with_absgrad_and_normals():
    inp, _ = _small(2, seed=16, P=150)
    gimg = grad_images(32, 48, 4)
    gM2, gMed = _ggeo(32, 48, 4)
    gN = np.random.RandomState(5).randn(1, 3, 32, 48).astype(np.float32)
    a = _run([inp], [gimg], gM2[None], gMed[None], gN, normals=True, absgrad=True, det=True)
    b = _run([inp], [gimg], gM2[None], gMed[None], gN, normals=True, absgrad=True, det=True)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    # and absgrad's statistic is what it is without geometry gradients when they are zero (atomic: within rounding)
    c = _run([inp], [gimg], None, None, gN, normals=True, absgrad=True, det=True, geometry=False)
    z = _run([inp], [gimg], np.zeros_like(gM2[None]), np.zeros_like(gMed[None]), gN, normals=True, absgrad=True, det=True)
    assert z["means2D_abs"].tobytes() == c["means2D_abs"].tobytes()


# ---- 6. entry points and the training loop ---------------------------------------------------------------------------------
def test_packed_matches_unpacked():
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
    gimg = grad_images(32, 48, 9)
    gM2, gMed = _ggeo(32, 48, 9)
    with deterministic(True):
        outs = rasterize_views_packed(flat, P, K, raw=True, geometry=True, **_views([inp]))
        gs = [torch.tensor(g[None], device=DEV) for g in gimg]
        torch.autograd.backward([outs[0], outs[2], outs[3], outs[4], outs[5]],
                                gs + [torch.tensor(gMed[None], device=DEV), torch.tensor(gM2[None], device=DEV)])
    ref = _run([inp], [gimg], gM2[None], gMed[None], det=True, raw=raw)
    assert np.array_equal(outs[4].detach().cpu().numpy(), ref["median"])
    assert np.array_equal(outs[5].detach().cpu().numpy(), ref["depth2"])
    for i, k in ((0, "means3D"), (3, "opacities")):
        o, n, _ = layout[i]
        assert np.array_equal(flat.grad[o:o + n].cpu().numpy().reshape(ref[k].shape), ref[k]), k


def test_render_and_render_views_keys():
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.geometry import depth_distortion
    from humangaussian_b200.renderer import PipelineParams, render, render_views
    from humangaussian_b200.scene import synthetic_body
    pc = synthetic_body(500, sh_degree=1, seed=1).to(DEV)
    pc.xyz.requires_grad_(True)
    cams = sample_orbit_cameras(2, 32, 48, seed=3)
    out = render_views(cams, pc, torch.zeros(3, device=DEV), geometry=True, normals=True)
    for k in ("median_depth_3dgs", "depth2_3dgs", "distortion_3dgs"):
        assert out[k].shape == (2, 1, 32, 48), k
    assert torch.equal(out["distortion_3dgs"], depth_distortion(out["alpha_3dgs"], out["depth_3dgs"], out["depth2_3dgs"]))
    (out["distortion_3dgs"].sum() + out["median_depth_3dgs"].sum()).backward()
    assert float(pc.xyz.grad.abs().sum()) > 0
    one = render(cams[0], pc, PipelineParams(), torch.zeros(3, device=DEV), geometry=True)
    assert torch.equal(one["median_depth_3dgs"], out["median_depth_3dgs"][0].detach())
    assert torch.equal(one["depth2_3dgs"], out["depth2_3dgs"][0].detach())


def test_packed_training_loop_lowers_distortion():
    """a short packed raw loop on a synthetic scene: image loss, with and without lam * distortion + lam' * consistency.
    With the terms, the mean distortion inside the silhouette ends lower than without them, and the image loss still falls."""
    from humangaussian_b200 import dist as D
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.geometry import depth_distortion, depth_normal_consistency, depth_to_normal
    from humangaussian_b200.optim import PackedAdam, expon_lr_func
    from humangaussian_b200.rasterizer import rasterize_views_packed
    from humangaussian_b200.renderer import stack_cameras
    _, _, sc = small_scene(P=3000, deg=1, seed=4)
    K, H = 4, 64
    raw = dict(xyz=sc.xyz, scaling=sc.scaling, rotation=sc.rotation, opacity=sc.opacity,
               features=torch.cat((sc.features_dc, sc.features_rest), 1))
    vm, pm, cp, tx, ty = stack_cameras(sample_orbit_cameras(4, H, H, seed=3), DEV)
    bg = torch.tensor([0.8, 0.5, 0.2], device=DEV)
    view = dict(viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx, tanfovy=ty, image_height=H, image_width=H, bg=bg,
                sh_degree=1, raw=True)
    with torch.no_grad():
        flat0 = D.pack({k: v.detach().float().to(DEV).contiguous() for k, v in raw.items()})
        target = rasterize_views_packed(flat0, 3000, K, **view)[0].clone()
        noisy = flat0.clone()
        noisy[:3 * 3000] += 0.02 * torch.randn(3 * 3000, device=DEV, generator=torch.Generator(DEV).manual_seed(0))

    def loop(lam, lam_n):
        flat = noisy.clone().requires_grad_(True)
        lrs = dict(xyz=0.0005, f_dc=0.0125, f_rest=0.0125 / 20.0, opacity=0.02, scaling=0.005, rotation=0.001)
        opt = PackedAdam(flat, 3000, K, lrs, xyz_scheduler=expon_lr_func(lr_init=0.0005, lr_final=0.00005, max_steps=100))
        img, dist = [], []
        for it in range(40):
            c, _, d, a, nrm, med, d2 = rasterize_views_packed(opt.packed, opt.P, K, normals=True, geometry=True, **view)
            Ld = depth_distortion(a, d, d2)
            inside = a.detach() > 0.5
            loss = (c - target).abs().mean()
            img.append(loss.item())
            dist.append(float(Ld.detach()[inside].mean()))
            if lam > 0:
                dn = depth_to_normal(med, vm, tx, ty)
                loss = loss + lam * Ld[inside].mean() + lam_n * depth_normal_consistency(nrm, dn, a).mean()
            loss.backward()
            opt.step()
            opt.zero_grad()
        return img, dist

    img0, dist0 = loop(0.0, 0.0)
    img1, dist1 = loop(50.0, 0.05)
    assert np.isfinite(img1).all() and np.isfinite(dist1).all()
    assert img1[-1] < img1[0], (img1[0], img1[-1])
    assert dist1[-1] < dist0[-1], (dist0[-1], dist1[-1])
