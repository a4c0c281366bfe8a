"""GPU: the render options combined, every blend kernel variant against one composed float64 reference
(tests/option_matrix_reference.py).

The backward blend has one kernel per combination of DET (the deterministic backward), ABS (the absolute screen-space
gradient), NRM (normal maps) and GEO (the geometry outputs), 16 in all; the forward blend has five (plain, contribution,
normals, geometry, normals + geometry).  The feature files test each feature with the others mostly off; this file walks
the combinations.

  1. CASES, a fixed table that covers every pair of axis values (test_option_matrix_cpu.py checks the covering rule): the
     variant, the colours (SH degree 0, 1, 3 or colors_precomp), activated or raw parameters, scales + rotations or
     cov3D_precomp, antialiasing, the 3D filter, 1 or 3 views, shared or per-view means, scale_modifier 1 or 0.7, and four
     scenes (small random, dense opaque, flush-boundary stacks, partial edge patches).  Per case: every gradient including
     means2D and means2D_abs with grads_agree at 1e-4 abs / 1e-3 rel, and every image bit for bit against the oracle and
     the replays;
  2. the forward matrix: switching one feature on leaves every other output, the radii and the forward state
     byte-identical, and the contribution accumulators equal the replay's;
  3. the deterministic backward: ABS changes no other gradient's bytes, NRM / GEO with absent gradients change no bytes
     and with zero gradients no values, reruns are byte-identical, the atomic twin agrees;
  4. the retries with the options on: the deterministic partial-capacity retry and the forward's instance-capacity retry
     give the bytes of a call that needed none;
  5. one larger case: 128 x 128, 3 views, per-view means, raw, SH degree 3, every option, atomic and deterministic."""
import contextlib
import math
from collections import namedtuple

import numpy as np
import pytest
import torch

import bench_step_reference as BS
import contribution_reference as CR
import option_matrix_reference as OR
from util import grad_images, grads_agree, screen_scene, small_scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REF_TOL = dict(atol=1e-4, rtol=1e-3)
STATE_KEYS = ("recs", "point_list", "ranges", "n_contrib", "final_T")

Case = namedtuple("Case", "det abs nrm geo colour params cov aa f3d V means mod scene")
# Generated once by a greedy all-pairs search over the axes below, with two rules on top: each of the 16 backward variants
# appears at least twice, and at least once with 3 views and per-view means.  Illegal rows (normals or the 3D filter with
# cov3D_precomp; per-view means with one view) never appear, and absgrad on the flush-boundary stacks has one view (its
# float64 Jacobian takes one forward-mode pass per overlapping Gaussian).
CASES = tuple(Case(*c) for c in (
    # det abs nrm geo  colour params cov  aa f3d V  means       mod  scene
    (0, 0, 0, 0, "sh1", "act", "cov", 1, 0, 3, "per_view", 0.7, "dense"),
    (0, 0, 0, 1, "sh0", "act", "sr", 1, 0, 3, "per_view", 1.0, "small"),
    (0, 0, 1, 0, "sh1", "act", "sr", 1, 1, 3, "per_view", 1.0, "dense"),
    (0, 0, 1, 1, "sh0", "raw", "sr", 0, 0, 3, "per_view", 1.0, "edge"),
    (0, 1, 0, 0, "sh0", "act", "sr", 1, 1, 3, "per_view", 0.7, "dense"),
    (0, 1, 0, 1, "sh1", "act", "sr", 0, 0, 3, "per_view", 1.0, "dense"),
    (0, 1, 1, 0, "sh0", "act", "sr", 0, 1, 3, "per_view", 0.7, "dense"),
    (0, 1, 1, 1, "sh0", "act", "sr", 1, 1, 3, "per_view", 0.7, "small"),
    (1, 0, 0, 0, "sh3", "raw", "sr", 0, 0, 3, "per_view", 0.7, "small"),
    (1, 0, 0, 1, "sh3", "raw", "sr", 0, 1, 3, "per_view", 1.0, "small"),
    (1, 0, 1, 0, "pre", "act", "sr", 1, 0, 3, "per_view", 0.7, "small"),
    (1, 0, 1, 1, "sh1", "raw", "sr", 1, 0, 3, "per_view", 1.0, "small"),
    (1, 1, 0, 0, "sh0", "raw", "cov", 1, 0, 3, "per_view", 0.7, "small"),
    (1, 1, 0, 1, "sh1", "act", "sr", 1, 1, 3, "per_view", 1.0, "dense"),
    (1, 1, 1, 0, "sh1", "raw", "sr", 0, 1, 3, "per_view", 1.0, "small"),
    (1, 1, 1, 1, "sh1", "raw", "sr", 0, 0, 3, "per_view", 0.7, "small"),
    (0, 0, 0, 0, "pre", "raw", "cov", 0, 0, 1, "shared", 1.0, "flush"),
    (0, 0, 0, 1, "sh3", "act", "sr", 1, 1, 1, "shared", 0.7, "edge"),
    (0, 0, 1, 0, "sh3", "act", "sr", 1, 1, 3, "shared", 0.7, "flush"),
    (0, 0, 1, 1, "pre", "raw", "sr", 1, 1, 1, "shared", 0.7, "dense"),
    (0, 1, 0, 0, "sh1", "act", "cov", 0, 0, 1, "shared", 0.7, "edge"),
    (0, 1, 0, 1, "sh0", "act", "cov", 1, 0, 1, "shared", 1.0, "flush"),
    (0, 1, 1, 0, "sh3", "raw", "sr", 1, 1, 1, "shared", 0.7, "small"),
    (0, 1, 1, 1, "pre", "act", "sr", 1, 0, 1, "shared", 0.7, "edge"),
    (1, 0, 0, 0, "sh1", "raw", "sr", 1, 0, 1, "shared", 1.0, "flush"),
    (1, 0, 0, 1, "sh3", "act", "cov", 0, 0, 3, "per_view", 0.7, "dense"),
    (1, 0, 1, 0, "sh0", "raw", "sr", 0, 0, 3, "per_view", 0.7, "flush"),
    (1, 0, 1, 1, "sh0", "raw", "sr", 1, 0, 3, "per_view", 0.7, "edge"),
    (1, 1, 0, 0, "sh1", "act", "sr", 0, 1, 1, "shared", 1.0, "small"),
    (1, 1, 0, 1, "sh0", "act", "sr", 1, 1, 3, "per_view", 1.0, "edge"),
    (1, 1, 1, 0, "sh1", "act", "sr", 0, 1, 1, "shared", 0.7, "edge"),
    (1, 1, 1, 1, "pre", "raw", "sr", 1, 1, 3, "per_view", 0.7, "small"),
))
# the forward blend's kernels: (normals, geometry, contribution)
FWD_VARIANTS = dict(plain=(0, 0, 0), contrib=(0, 0, 1), nrm=(1, 0, 0), geo=(0, 1, 0), nrm_geo=(1, 1, 0))


def legal(case):
    """the combinations the library accepts (rasterizer._forward_impl / _check_filter_3d), and per-view means need views"""
    return not (case.cov == "cov" and (case.nrm or case.f3d)) and not (case.means == "per_view" and case.V == 1)


def forward_variants(case):
    """the forward kernels a case's options allow: no normals with cov3D_precomp, contribution never with normals or geometry"""
    return [k for k, (n, g, c) in FWD_VARIANTS.items() if not (n and case.cov == "cov") and not (c and (n or g))]


@contextlib.contextmanager
def deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


# ---- scenes -----------------------------------------------------------------------------------------------------------------
def _screen_to_scales(inp, rng, depth_axis=0.0):
    """a screen scene's axis-aligned covariances as scales and random-axis-order rotations (normals need scales).  The depth
    axis is at least `depth_axis` times the screen scale: the flush stacks' low opacities would vanish under the 3D filter,
    which scales a flat Gaussian's opacity by its thin axis over the filter's width."""
    c = inp.pop("cov3D_precomp").astype(np.float64)
    n = len(c)
    s = np.sqrt(np.stack([c[:, 0], c[:, 3], np.maximum(c[:, 5], depth_axis ** 2 * c[:, 0])], 1))
    inp["scales"] = (s * np.stack([rng.permutation([1.0, 0.93, 0.86]) for _ in range(n)])).astype(np.float32)
    q = np.zeros((n, 4))
    q[:, 0] = 1.0
    q += 0.05 * rng.randn(n, 4)
    inp["rotations"] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    return inp


def _stack(x, y, n, z0, opacity):
    return dict(px=np.full(n, x) + np.sin(np.arange(n)), py=np.full(n, y), depth=z0 + 1e-2 * np.arange(n),
                opacity=np.full(n, opacity))


def _scene(name):
    """activated inputs with SH degree 3 colours and scales + rotations; `cams` says how further views are made"""
    rng = np.random.RandomState(dict(small=1, dense=2, flush=3, edge=4)[name])
    if name in ("small", "dense"):
        if name == "small":
            inp, _, _ = small_scene(P=60, deg=3, seed=1, H=32, W=48)
        else:
            inp, _, _ = small_scene(P=80, deg=3, seed=9, H=32, W=32, dist=1.3)
            inp["opacities"] = np.clip(inp["opacities"] * 8, 0, 0.9999).astype(np.float32)
            inp["scales"] = (inp["scales"] * 2.0).astype(np.float32)
        return inp, "orbit"
    if name == "flush":  # stacks of 17, 33, 64 and 16 hits in patch 0 of their tiles, T = 1/2 near hits 16, 32 and 60
        parts = [_stack(3.5, 1.5, 17, 1.0, 0.047), _stack(35.5, 1.5, 33, 2.0, 0.0225), _stack(67.5, 1.5, 64, 3.0, 0.0118),
                 _stack(99.5, 1.5, 16, 4.0, 0.05)]
        g = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
        inp = screen_scene(g["px"], g["py"], g["depth"], 8.0, g["opacity"], H=16, W=128)
    else:  # partial patches: columns 120-122 and row 60 of a 123 x 61 image
        n = 200
        px = np.concatenate([rng.uniform(-2, 125, 120), rng.uniform(112, 125, 40), rng.uniform(-2, 125, 40)])
        py = np.concatenate([rng.uniform(-2, 63, 120), rng.uniform(-2, 63, 40), rng.uniform(52, 63, 40)])
        inp = screen_scene(px, py, rng.uniform(1, 3, n), rng.uniform(0.5, 3, n), rng.uniform(0.1, 0.9, n), H=61, W=123)
    inp = _screen_to_scales(inp, rng, 0.3 if name == "flush" else 0.0)
    P = len(inp["means3D"])
    shs = 0.3 * rng.randn(P, 16, 3)
    shs[:, 0] = (inp.pop("colors_precomp") - 0.5) / 0.28209479177387814
    inp.update(shs=shs.astype(np.float32), sh_degree=3)
    return inp, "shift"


def _views(inp, cams, V):
    if V == 1:
        return [inp]
    if cams == "orbit":
        from humangaussian_b200.cameras import sample_orbit_cameras
        H, W = inp["image_height"], inp["image_width"]
        return [dict(inp, viewmatrix=c.world_view_transform.cpu().numpy(), projmatrix=c.full_proj_transform.cpu().numpy(),
                     campos=c.camera_center.cpu().numpy(), tanfovx=math.tan(c.FoVx * 0.5), tanfovy=math.tan(c.FoVy * 0.5))
                for c in sample_orbit_cameras(V, H, W, seed=5)]
    out = []  # the screen scenes' camera sits at the origin (identity view matrix): shift it a little per view
    for v in range(V):
        t = np.array([0.03 * v, -0.02 * v, 0.0], np.float32)
        vm = np.eye(4, dtype=np.float32)
        vm[3, :3] = -t
        out.append(dict(inp, viewmatrix=vm, projmatrix=(vm.astype(np.float64) @ inp["projmatrix"]).astype(np.float32), campos=t))
    return out


def _raw_of(inp):
    """raw parameters whose activations are inp's up to rounding, and inp re-activated from them as the kernels activate
    (bench_step_reference.activate on the device), so the oracle sees the kernels' activated values bit for bit"""
    o = np.asarray(inp["opacities"], np.float64)
    raw = dict(opacities=np.log(o / (1 - o)).astype(np.float32))
    if inp.get("scales") is not None:
        raw.update(scales=np.log(inp["scales"].astype(np.float64)).astype(np.float32),
                   rotations=(inp["rotations"] * 1.3).astype(np.float32))
    return raw, dict(inp, **BS.activate(raw, DEV))


def setup(case, scene=None):
    """(views, raw, means, filter variances) of a case: activated oracle inputs per view (shared means in each), the raw
    arrays or None, per-view means [V,P,3] or None, and the 3D filter's [P] variances or None.  scene: (inputs, camera
    rule) in place of _scene(case.scene)."""
    inp, cams = _scene(case.scene) if scene is None else scene
    deg = dict(sh0=0, sh1=1, sh3=3).get(case.colour)
    if deg is None:
        inp["colors_precomp"] = (np.random.RandomState(7).rand(len(inp["means3D"]), 3) * 0.8 + 0.1).astype(np.float32)
        del inp["shs"]
        inp["sh_degree"] = 0
    else:
        inp["shs"] = np.ascontiguousarray(inp["shs"][:, :(deg + 1) ** 2])
        inp["sh_degree"] = deg
    if case.cov == "cov":
        from oracle.gs_oracle import Oracle
        o = Oracle(threads=1)
        o.forward(**dict(inp, scale_modifier=1.0))
        inp["cov3D_precomp"] = o.state()["cov3d"].astype(np.float32).copy()
        del inp["scales"], inp["rotations"]
    inp["scale_modifier"] = case.mod
    raw = None
    if case.params == "raw":
        raw, inp = _raw_of(inp)
    inps = _views(inp, cams, case.V)
    means = None
    if case.means == "per_view":
        rng = np.random.RandomState(11)
        step = 0.02 if cams == "orbit" else 0.004
        means = np.stack([inp["means3D"] + (step * rng.randn(*inp["means3D"].shape)).astype(np.float32) for _ in inps])
    var = None
    if case.f3d:
        import filter3d_reference as FR
        i0 = inps[0]
        rate = FR.sampling_rate(i0["means3D"], [i["viewmatrix"] for i in inps], [i["tanfovx"] for i in inps],
                                [i["tanfovy"] for i in inps], i0["image_height"], i0["image_width"])
        var = FR.finalize(rate)
    return inps, raw, means, var


def out_grads(case, inps, seed=0):
    """(gimgs, gN [V,3,H,W] | None, gM2 [V,H,W] | None, gMed [V,H,W] | None) of a case"""
    H, W = inps[0]["image_height"], inps[0]["image_width"]
    V = len(inps)
    rng = np.random.RandomState(100 + seed)
    gimgs = [grad_images(H, W, 10 * seed + v) for v in range(V)]
    gN = rng.randn(V, 3, H, W).astype(np.float32) if case.nrm else None
    gM2, gMed = (rng.randn(V, H, W).astype(np.float32) for _ in range(2)) if case.geo else (None, None)
    return gimgs, gN, gM2, gMed


# ---- the harness ------------------------------------------------------------------------------------------------------------
def _run(inps, gimgs=None, gN=None, gM2=None, gMed=None, *, det=False, raw=None, means=None, normals=False, geometry=False,
         absgrad=False, antialiasing=False, filter_3d=None):
    """rasterize_views over the views `inps` with every option; with gimgs, the backward of sum gC c + gD d + gA a (+ gN N
    + gM2 M2 + gMed median where given).  Returns numpy images, radii and gradients (means2D and means2D_abs included)."""
    from humangaussian_b200.rasterizer import rasterize_views
    i0 = inps[0]
    t = {k: torch.tensor(i0[k], device=DEV, requires_grad=True) for k in OR.PARAMS if i0.get(k) is not None}
    for k, v in (raw or {}).items():
        t[k] = torch.tensor(v, device=DEV, requires_grad=True)
    if means is not None:
        t["means3D"] = torch.tensor(means, device=DEV, requires_grad=True)
    V, P = len(inps), i0["means3D"].shape[0]
    m2d = torch.zeros(V, P, 3, device=DEV, requires_grad=True)
    m2a = torch.zeros(V, P, 3, device=DEV, requires_grad=True) if absgrad else None
    g = lambda k: torch.stack([torch.as_tensor(np.asarray(i[k], np.float32)) for i in inps]).to(DEV)
    cams = dict(viewmatrices=g("viewmatrix").reshape(-1, 4, 4), projmatrices=g("projmatrix").reshape(-1, 4, 4),
                camposs=g("campos").reshape(-1, 3), tanfovx=[i["tanfovx"] for i in inps], tanfovy=[i["tanfovy"] for i in inps],
                image_height=i0["image_height"], image_width=i0["image_width"], bg=torch.tensor(i0["bg"], device=DEV),
                sh_degree=i0.get("sh_degree", 0), scale_modifier=i0.get("scale_modifier", 1.0))
    f3d = None if filter_3d is None else torch.tensor(filter_3d, device=DEV)
    with deterministic(det):
        outs = rasterize_views(means2D=m2d, means2D_abs=m2a, raw=raw is not None, normals=normals, geometry=geometry,
                               antialiasing=antialiasing, filter_3d=f3d, **t, **cams)
        res = dict(color=outs[0], radii=outs[1], depth=outs[2], alpha=outs[3])
        if normals:
            res["normal"] = outs[4]
        if geometry:
            res["median"], res["depth2"] = outs[4 + normals], outs[5 + normals]
        if gimgs is not None:
            ts = [outs[0], outs[2], outs[3]]
            gt = [torch.tensor(np.stack([x[j] for x in gimgs]), device=DEV) for j in range(3)]
            for key, gx in (("normal", gN), ("median", gMed), ("depth2", gM2)):
                if gx is not None and key in res:
                    ts.append(res[key])
                    gt.append(torch.as_tensor(np.asarray(gx, np.float32), device=DEV).reshape(res[key].shape))
            torch.autograd.backward(ts, gt)
            res.update(means2D=m2d.grad, **{k: v.grad for k, v in t.items()})
            if absgrad:
                res["means2D_abs"] = m2a.grad
    return {k: v.detach().cpu().numpy() for k, v in res.items()}


def _rows(k, a):
    """per-(view,) Gaussian rows: grads_agree's row criterion is per Gaussian vector"""
    a = np.asarray(a)
    return a.reshape(-1, 3) if k in ("means2D", "means2D_abs") or (k == "means3D" and a.ndim == 3) else a.reshape(a.shape[0], -1)


def _worst(a, b, atol, rtol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float((np.abs(a - b) / (atol + rtol * np.abs(b).max(axis=1, keepdims=True))).max()) if a.size else 0.0


def check_against_reference(case, inps, raw, means, var, dets=None, seed=0):
    """every image bit for bit and every gradient within REF_TOL, for the case's variant (or each det in `dets`); returns the
    worst row-wise margin over the gradients (1.0 = at the tolerance)"""
    gimgs, gN, gM2, gMed = out_grads(case, inps, seed)
    opts = dict(antialiasing=bool(case.aa), filter_3d=var)
    im, ref = OR.reference(inps, gimgs, gN, gM2, gMed, raw=raw, means=means, normals=bool(case.nrm),
                           geometry=bool(case.geo), absgrad=bool(case.abs), **opts)
    assert im["alpha"].max() > 0.02
    worst = 0.0
    for det in (bool(case.det),) if dets is None else dets:
        g = _run(inps, gimgs, gN, gM2, gMed, det=det, raw=raw, means=means, normals=bool(case.nrm), geometry=bool(case.geo),
                 absgrad=bool(case.abs), **opts)
        for k, r in im.items():
            if k == "median_pos":
                continue
            got = g[k].reshape(r.shape)
            assert got.tobytes() == r.astype(got.dtype).tobytes(), f"{case} det={det}: {int((got != r).sum())} {k} values differ"
        for k, r in ref.items():
            # every means2D row must hold; its elementwise rate is over two components per row, each a sum over the
            # footprint that cancels to near zero for a Gaussian centred on a pixel, so 0.2 % of them may miss alone
            crit = dict(min_elementwise=0.998) if k == "means2D" else {}
            ok, msg = grads_agree(_rows(k, g[k]), _rows(k, r), **REF_TOL, **crit)
            assert ok, f"{case} det={det} {k}: {msg}"
            worst = max(worst, _worst(_rows(k, g[k]), _rows(k, r), **REF_TOL))
        if case.abs:
            assert np.abs(ref["means2D_abs"]).max() > 0 and (g["means2D_abs"][..., 2] == 0).all()
    return worst


# ---- 1. the backward matrix -------------------------------------------------------------------------------------------------
def _id(c):
    return (f"{'det' if c.det else 'atomic'}{'-abs' if c.abs else ''}{'-nrm' if c.nrm else ''}{'-geo' if c.geo else ''}-{c.colour}-"
            f"{c.params}-{c.cov}{'-aa' if c.aa else ''}{'-f3d' if c.f3d else ''}-V{c.V}-{c.means}-m{c.mod}-{c.scene}")


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_backward_matrix(case):
    inps, raw, means, var = setup(case)
    worst = check_against_reference(case, inps, raw, means, var)
    print(f"\nworst grads_agree margin {worst:.3f} ({_id(case)})")


# ---- 2. the forward matrix --------------------------------------------------------------------------------------------------
def _forward(inps, variant, raw=None, means=None, antialiasing=False, filter_3d=None):
    from humangaussian_b200.rasterizer import forward_with_state
    n, g, c = FWD_VARIANTS[variant]
    i0 = inps[0]
    P = i0["means3D"].shape[0]
    t = lambda a: torch.tensor(np.asarray(a, np.float32), device=DEV)
    kw = {k: t(i0[k]) for k in OR.PARAMS if i0.get(k) is not None}
    kw.update({k: t(v) for k, v in (raw or {}).items()})
    if means is not None:
        kw["means3D"] = t(means)
    acc = (torch.zeros(P, dtype=torch.int64, device=DEV), torch.zeros(P, dtype=torch.int32, device=DEV),
           torch.zeros(P, dtype=torch.int32, device=DEV)) if c else None
    outs = forward_with_state(viewmatrix=t(np.stack([i["viewmatrix"] for i in inps])).reshape(-1, 4, 4),
                              projmatrix=t(np.stack([i["projmatrix"] for i in inps])).reshape(-1, 4, 4),
                              campos=t(np.stack([i["campos"] for i in inps])).reshape(-1, 3),
                              tanfovx=[i["tanfovx"] for i in inps], tanfovy=[i["tanfovy"] for i in inps],
                              image_height=i0["image_height"], image_width=i0["image_width"], bg=t(i0["bg"]),
                              sh_degree=i0.get("sh_degree", 0), scale_modifier=i0.get("scale_modifier", 1.0), raw=raw is not None,
                              antialiasing=antialiasing, filter_3d=None if filter_3d is None else t(filter_3d), normals=bool(n),
                              geometry=bool(g), contrib=acc, **kw)
    res = dict(zip(("color", "radii", "depth", "alpha"), outs[:4]))
    extra = list(outs[4:-2])
    if n:
        res["normal"] = extra.pop(0)
    if g:
        res["median"], res["depth2"] = extra
        res["median_pos"] = outs[-2]["median_pos"]
    res.update({k: outs[-2][k] for k in STATE_KEYS})
    if c:
        res.update(weight_sum=acc[0], weight_max=acc[1], touches=acc[2])
    return {k: v.cpu().numpy() for k, v in res.items()}


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_forward_matrix(case):
    inps, raw, means, var = setup(case)
    opts = dict(raw=raw, means=means, antialiasing=bool(case.aa), filter_3d=var)
    runs = {v: _forward(inps, v, **opts) for v in forward_variants(case)}
    plain = runs["plain"]
    for v, r in runs.items():
        for k, x in r.items():
            # every output of the variant that another variant also has is byte-identical to it
            for w, s in runs.items():
                if k in s and w != v:
                    assert x.tobytes() == s[k].tobytes(), f"{_id(case)}: {k} differs between the {v} and {w} forwards"
        assert all(k in r for k in plain)
    if "contrib" in runs:
        acc = CR.contribution(OR.view_inputs(inps, means), bool(case.aa), var)
        got = runs["contrib"]
        assert np.array_equal(got["weight_sum"].view(np.uint64), acc["weight_sum"])
        assert np.array_equal(got["weight_max"].view(np.uint32), acc["weight_max"])
        assert np.array_equal(got["touches"].astype(np.int64), acc["touches"])
        assert acc["weight_sum"].max() > 0


# ---- 3. independence in the deterministic backward --------------------------------------------------------------------------
INDEP = Case(1, 0, 0, 0, "sh3", "act", "sr", 1, 1, 3, "per_view", 0.7, "small")


@pytest.mark.parametrize("variant", [(a, n, g) for a in (0, 1) for n in (0, 1) for g in (0, 1)],
                         ids=lambda v: "det" + "".join(f"-{k}" for k, on in zip(("abs", "nrm", "geo"), v) if on) or "det")
def test_deterministic_independence(variant):
    a, n, g = variant
    case = INDEP._replace(abs=a, nrm=n, geo=g)
    inps, raw, means, var = setup(case)
    gimgs, gN, gM2, gMed = out_grads(case, inps, 3)
    kw = dict(raw=raw, means=means, antialiasing=True, filter_3d=var, normals=bool(n), geometry=bool(g))
    on = _run(inps, gimgs, gN, gM2, gMed, det=True, absgrad=bool(a), **kw)
    again = _run(inps, gimgs, gN, gM2, gMed, det=True, absgrad=bool(a), **kw)
    assert all(on[k].tobytes() == again[k].tobytes() for k in on), "deterministic reruns differ"
    # ABS on changes no other output or gradient
    other = _run(inps, gimgs, gN, gM2, gMed, det=True, absgrad=not a, **kw)
    for k in set(on) & set(other) - {"means2D_abs"}:
        assert on[k].tobytes() == other[k].tobytes(), f"{k} changes with absgrad {'off' if a else 'on'}"
    # NRM / GEO with zero or absent gradients: the bytes of the variant without them
    for feat in [f for f, on_ in (("nrm", n), ("geo", g)) if on_]:
        # the variant without `feat`, and `feat` on with zero and with absent gradients
        keep = dict(gN=gN, gM2=gM2, gMed=gMed)
        off = dict(keep, **(dict(gN=None) if feat == "nrm" else dict(gM2=None, gMed=None)))
        zeros = {k: (np.zeros_like(v) if v is not None and off[k] is None else v) for k, v in keep.items()}
        base = _run(inps, gimgs, **off, det=True, absgrad=bool(a), **dict(kw, **{dict(nrm="normals", geo="geometry")[feat]: False}))
        z = _run(inps, gimgs, **off, det=True, absgrad=bool(a), **kw)
        for k in base:
            assert z[k].tobytes() == base[k].tobytes(), f"{k} changes with the {feat} gradient absent"
        # a zero gradient runs the feature's kernel: the same values, where a term n * 0 may leave -0 for +0
        z = _run(inps, gimgs, **zeros, det=True, absgrad=bool(a), **kw)
        for k in base:
            assert np.array_equal(z[k], base[k]), f"{k} changes with a zero {feat} gradient"
    # the atomic twin agrees
    at = _run(inps, gimgs, gN, gM2, gMed, det=False, absgrad=bool(a), **kw)
    for k in on:
        if k in ("color", "depth", "alpha", "radii", "normal", "median", "depth2"):
            assert at[k].tobytes() == on[k].tobytes(), k
        else:
            ok, msg = grads_agree(_rows(k, at[k]), _rows(k, on[k]))
            assert ok, f"atomic vs deterministic {k}: {msg}"


# ---- 4. the retries with the options on -------------------------------------------------------------------------------------
RETRY = Case(1, 1, 1, 1, "sh3", "act", "sr", 1, 1, 3, "per_view", 1.0, "small")


def test_deterministic_retry_with_every_option(monkeypatch):
    import humangaussian_b200.rasterizer as R
    monkeypatch.setattr(R, "_partial_hint", {})
    inps, raw, means, var = setup(RETRY)
    gimgs, gN, gM2, gMed = out_grads(RETRY, inps, 4)
    kw = dict(det=True, raw=raw, means=means, normals=True, geometry=True, absgrad=True, antialiasing=True, filter_3d=var)
    one = _run(inps, gimgs, gN, gM2, gMed, **kw)
    P, H, W = inps[0]["means3D"].shape[0], inps[0]["image_height"], inps[0]["image_width"]
    key = (DEV.index or 0, P, 3, H, W)
    assert R.last_num_partials() > 1
    R._partial_hint[key] = 1  # the first call cannot fit: B200GS_E_BIN_TOO_SMALL, then a retry with the reported count
    two = _run(inps, gimgs, gN, gM2, gMed, **kw)
    assert R._partial_hint[key] > R.last_num_partials()
    three = _run(inps, gimgs, gN, gM2, gMed, **kw)  # on the grown hint, with the pooled buffers of the retry
    for k in one:
        assert one[k].tobytes() == two[k].tobytes() == three[k].tobytes(), k


def test_forward_retry_with_every_option(monkeypatch):
    import humangaussian_b200.rasterizer as R
    monkeypatch.setattr(R, "_cap_hint", {})
    inps, raw, means, var = setup(RETRY)
    kw = dict(raw=raw, means=means, normals=True, geometry=True, antialiasing=True, filter_3d=var)
    one = _run(inps, **kw)
    n = R.last_num_rendered()
    P, H, W = inps[0]["means3D"].shape[0], inps[0]["image_height"], inps[0]["image_width"]
    key = (DEV.index or 0, P, 3, H, W)
    R._cap_hint[key] = n // 2  # below the count: B200GS_E_BIN_TOO_SMALL, then a retry with the reported count
    two = _run(inps, **kw)
    assert R._cap_hint[key] > n
    for k in one:
        assert one[k].tobytes() == two[k].tobytes(), k


# ---- 5. one larger case -----------------------------------------------------------------------------------------------------
def test_larger_case_every_option():
    """128 x 128, 3 views, per-view means, raw parameters, SH degree 3, antialiasing + the 3D filter + normals + geometry +
    absgrad, atomic and deterministic"""
    case = Case(1, 1, 1, 1, "sh3", "raw", "sr", 1, 1, 3, "per_view", 1.0, "small")
    inp, _, _ = small_scene(P=100, deg=3, seed=31, H=128, W=128, big=False)
    inps, raw, means, var = setup(case, (inp, "orbit"))
    worst = check_against_reference(case, inps, raw, means, var, dets=(False, True), seed=5)
    print(f"\nworst grads_agree margin {worst:.3f} (128x128, every option)")
