"""GPU: contribution scores (b200gs_forward_contrib_opts, contribution.compute_contribution) and pruning by mask.

  1. weight_sum, weight_max and touches bit-exact against the numpy replay of tests/contribution_reference.py: degrees 0 and
     3, dense-opaque, stacks of 1..64 hits in a patch, partial edge patches, a 3-view batch, per-view means, antialiasing,
     the 3D filter and cov3D_precomp;
  2. the variant's images, radii and forward state (final_T, n_contrib, contributor masks) byte-identical to the plain
     forward's; weight_max > 0 iff a contributor-mask bit of the Gaussian is set (raw parameters included);
  3. fold invariance over 130 cameras (one call, explicit 64 + 64 + 2 ABI chunks, one view at a time in reverse) and
     identical bytes from two runs;
  4. lossless prune: removing touches == 0 leaves the scoring cameras' colour, depth and alpha byte-identical and the
     survivors' radii unchanged, and in deterministic mode their gradients too; at full size (300 k, 512^2, 8 views) as well;
  5. prune_points / prune_points_packed bit-exact against boolean indexing, their edge cases, and training after a packed
     prune; argument errors and the classic comparator's B200GS_E_UNSUPPORTED."""
import contextlib
import math
import os

import numpy as np
import pytest
import torch

import contribution_reference as CR
from util import grad_images, screen_scene, small_scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GEOM = ("means3D", "opacities", "scales", "rotations", "cov3D_precomp")


def _cams(inps):
    g = lambda k: torch.stack([torch.as_tensor(np.asarray(i[k], np.float32)) for i in inps]).to(DEV)
    return dict(viewmatrices=g("viewmatrix").reshape(-1, 4, 4), projmatrices=g("projmatrix").reshape(-1, 4, 4),
                tanfovx=[i["tanfovx"] for i in inps], tanfovy=[i["tanfovy"] for i in inps],
                image_height=inps[0]["image_height"], image_width=inps[0]["image_width"])


def _score(inps, per_view=False, **kw):
    from humangaussian_b200.contribution import compute_contribution
    i0 = inps[0]
    t = {k: torch.tensor(np.asarray(i0[k], np.float32), device=DEV) for k in GEOM if i0.get(k) is not None}
    if per_view:
        t["means3D"] = torch.stack([torch.tensor(i["means3D"], device=DEV) for i in inps])
    if "filter_3d" in kw and kw["filter_3d"] is not None:
        kw["filter_3d"] = torch.tensor(kw["filter_3d"], device=DEV)
    return compute_contribution(**t, **_cams(inps), **kw)


def _check_exact(inps, per_view=False, antialiasing=False, filter_3d=None):
    ref = CR.contribution(inps, antialiasing=antialiasing, filter_3d=filter_3d)
    got = _score(inps, per_view=per_view, antialiasing=antialiasing, filter_3d=filter_3d)
    ws = (got.weight_sum.cpu().numpy() * 2.0 ** 24).astype(np.uint64)
    assert np.array_equal(ws, ref["weight_sum"]), "weight_sum differs from the replay"
    assert np.array_equal(got.weight_max.cpu().numpy().view(np.uint32), ref["weight_max"]), "weight_max differs"
    assert np.array_equal(got.touches.cpu().numpy(), ref["touches"]), "touches differ"
    assert (ref["blends"] > 0).sum() > 0
    return got, ref


def _small(deg, seed=None, P=120, H=32, W=48, **kw):
    inp, _, p = small_scene(P=P, deg=deg, seed=deg if seed is None else seed, H=H, W=W, **kw)
    return inp, p


def _orbit_inps(inp, n, H, W, seed):
    from humangaussian_b200.cameras import sample_orbit_cameras
    out = []
    for cam in sample_orbit_cameras(n, H, W, seed=seed):
        out.append(dict(inp, viewmatrix=cam.world_view_transform.cpu().numpy(), projmatrix=cam.full_proj_transform.cpu().numpy(),
                        campos=cam.camera_center.cpu().numpy(), tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5),
                        image_height=H, image_width=W))
    return out


def _dense(seed=9):
    inp, p = _small(1, seed=seed, P=300, H=32, W=32, dist=1.3)
    inp["opacities"] = np.clip(inp["opacities"] * 8, 0, 0.99999).astype(np.float32)
    inp["scales"] = (inp["scales"] * 2.0).astype(np.float32)
    return inp


def _stack(x, y, n, z0, opacity=0.05):
    return dict(px=np.full(n, x), py=np.full(n, y), depth=z0 + 1e-3 * np.arange(n), opacity=np.full(n, opacity))


def _cat(parts):
    return {k: np.concatenate([p[k] for p in parts]) for k in ("px", "py", "depth", "opacity")}


# ---- 1. bit-exact against the replay ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 3])
def test_small_scenes(deg):
    _check_exact([_small(deg)[0]])


def test_dense_opaque_scene():
    _, ref = _check_exact([_dense()])
    assert ref["terminated"] > 50


def test_stacks_of_hits():
    counts = (1, 15, 16, 17, 31, 32, 33, 64)
    g = _cat([_stack(16 * i + 3.5, 1.5, n, 1.0 + i, opacity=0.3) for i, n in enumerate(counts)])
    _check_exact([screen_scene(g["px"], g["py"], g["depth"], 0.6, g["opacity"], H=16, W=128)])


def test_partial_edge_patches():
    parts = [_stack(121.0, 9.5, 17, 1.0), _stack(121.0, 60.45, 15, 2.0), _stack(51.5, 60.45, 33, 3.0), _stack(3.5, 60.45, 1, 4.0)]
    g = _cat(parts)
    _check_exact([screen_scene(g["px"], g["py"], g["depth"], 0.6, g["opacity"], H=61, W=123)])


def test_three_view_batch():
    _check_exact(_orbit_inps(_small(2, P=100)[0], 3, 32, 48, seed=5))


def test_per_view_means():
    inp, _ = _small(1, seed=4)
    rng = np.random.RandomState(4)
    inps = [dict(inp, means3D=(inp["means3D"] + 0.02 * rng.randn(*inp["means3D"].shape)).astype(np.float32)) for _ in range(3)]
    _check_exact(inps, per_view=True)


def test_antialiasing():
    _check_exact([_small(1, seed=11)[0]], antialiasing=True)


def test_filter_3d():
    from test_gpu_filter3d import _var_for
    inp, _ = _small(3, seed=12)
    _check_exact([inp], filter_3d=_var_for(inp, seed=12))


def test_cov3D_precomp():
    from oracle.gs_oracle import Oracle
    inp, _ = _small(0, seed=3)
    o = Oracle(threads=1)
    o.forward(**inp)
    inp2 = {k: v for k, v in inp.items() if k not in ("shs", "scales", "rotations")}
    inp2["colors_precomp"] = np.full((len(inp["means3D"]), 3), 0.5, np.float32)
    inp2["cov3D_precomp"] = o.state()["cov3d"].copy()
    _check_exact([inp2])


def test_sample_ply_100k_512_bit_exact():
    """one 512^2 view of the seed-0 100 k subsample of sample.ply: tile lists thousands of entries deep, many 32-entry chunks,
    heavy atomic traffic; the replay reproduces the oracle's n_contrib and contributor patches (about 15 s of numpy)"""
    from humangaussian_b200.cameras import Camera, orbit_c2w
    from humangaussian_b200.scene import sample_ply_scene
    from test_gpu_fullsize import _inputs
    inp = _inputs(sample_ply_scene(100000, 0), Camera(orbit_c2w(15.0, 0.0, 2.0), math.radians(70.0), 512, 512), 512, 512, 0)
    _, ref = _check_exact([inp])
    v = ref["views"][0]
    assert np.array_equal(v["n_contrib"], v["state"]["n_contrib"])
    assert np.array_equal(v["contrib_patches"], v["state"]["contrib_patches"])
    lens = v["state"]["ranges"][:, 1] - v["state"]["ranges"][:, 0]
    assert lens.max() > 1000 and (ref["blends"] > 0).sum() > 20000


def test_full_size_300k_1024_eight_views_against_the_oracle_backward():
    """300 k Gaussians (seed-0 subsample of sample.ply), 1024^2, 8 views, colours precomputed.  With dL/dcolor = 1 on channel 0
    and 0 elsewhere, the oracle backward's dL/dcolors[g, 0] is sum_p w'_pg, summed in double and rounded to float32, where w'
    is alpha * T' with T' recovered from final_T by divisions T' <- T' / (1 - alpha).  Bound, fixed before the first run:
    the forward's T_k and the recovered T'_k differ by one multiplication and one division rounding per later blend of the
    pixel, so |w' - w| <= w (2 m + 1) u (1.01), m < N = the largest n_contrib of the views, u = 2^-24; weight_sum's
    quantisation adds at most 2^-25 per blend (<= touches); the oracle's float32 result adds u |result|:
        |weight_sum_g - oracle_g| <= weight_sum_g (2 N + 2) u 1.01 + touches_g 2^-25 + u |oracle_g|.
    Global identity on the GPU: sum_g weight_sum = sum over pixels of the alpha images up to
    sum_p max(n_contrib_p - 1, 0) u + (sum_g touches) 2^-25 (float32 accumulation of each alpha, plus the quantisation)."""
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.rasterizer import forward_with_state
    from humangaussian_b200.scene import sample_ply_scene
    from oracle.gs_oracle import Oracle
    from test_gpu_fullsize import _inputs
    u = 2.0 ** -24
    p = sample_ply_scene(300000, 3)
    cams = sample_orbit_cameras(8, 1024, 1024, seed=1000)
    inps = []
    for cam in cams:
        i = _inputs(p, cam, 1024, 1024, 3)
        i.pop("shs")
        i["colors_precomp"] = np.random.RandomState(5).rand(300000, 3).astype(np.float32)
        i["sh_degree"] = 0
        inps.append(i)
    P = 300000
    acc = _acc(P)
    t = {k: torch.tensor(np.asarray(inps[0][k], np.float32), device=DEV) for k in ("means3D", "opacities", "colors_precomp", "scales",
                                                                                   "rotations", "bg")}
    c = _cams(inps)
    t.update(viewmatrix=c["viewmatrices"], projmatrix=c["projmatrices"],
             campos=torch.stack([torch.tensor(i["campos"]) for i in inps]).to(DEV), tanfovx=c["tanfovx"], tanfovy=c["tanfovy"],
             image_height=1024, image_width=1024)
    _, _, _, alpha, s, _ = forward_with_state(contrib=acc, **t)
    ws = acc[0].cpu().numpy().astype(np.float64) * u
    touches = acc[2].cpu().numpy().view(np.uint32).astype(np.float64)
    ncon = s["n_contrib"].cpu().numpy().astype(np.float64)
    # the global identity
    bound = float(np.maximum(ncon - 1, 0).sum()) * u + touches.sum() * u / 2
    a_sum = float(alpha.double().sum())
    assert abs(ws.sum() - a_sum) <= bound, (ws.sum(), a_sum, bound)
    # against the oracle backward, view by view
    oracle = np.zeros(P, np.float64)
    for i in inps:
        o = Oracle()
        o.forward(**i)
        g = o.backward(np.stack([np.ones((1024, 1024), np.float32), np.zeros((1024, 1024), np.float32),
                                 np.zeros((1024, 1024), np.float32)]), np.zeros((1, 1024, 1024), np.float32),
                       np.zeros((1, 1024, 1024), np.float32))
        oracle += g["colors_precomp"][:, 0].astype(np.float64)
    N = float(ncon.max())
    lim = ws * (2 * N + 2) * u * 1.01 + touches * u / 2 + u * np.abs(oracle) * len(inps)
    err = np.abs(ws - oracle)
    print(f"300k / 1024^2 / 8 views: N = {N:.0f}, worst |err| / bound = {float((err / np.maximum(lim, 1e-300)).max()):.3g}, "
          f"median relative error of the blended = {float(np.median(err[ws > 0] / ws[ws > 0])):.3g}")
    assert (err <= lim).all(), f"{int((err > lim).sum())} Gaussians outside the bound"
    assert (ws > 0).sum() > 100000


# ---- 2. the variant leaves the forward unchanged ---------------------------------------------------------------------------
def _state(inp, contrib=None, **kw):
    from humangaussian_b200.rasterizer import forward_with_state
    t = {k: torch.tensor(np.asarray(v), device=DEV) if isinstance(v, np.ndarray) else v for k, v in inp.items()}
    c, r, d, a, st, _ = forward_with_state(contrib=contrib, **t, **kw)
    out = dict(color=c, radii=r, depth=d, alpha=a, final_T=st["final_T"], n_contrib=st["n_contrib"], point_list=st["point_list"],
               ranges=st["ranges"])
    # contributor masks: only the words up to each patch's last contributing chunk are defined; compare them via the ranges
    out["cmask"] = st["contributor_masks"]
    return {k: v.cpu().numpy() for k, v in out.items()}


def _acc(P):
    return (torch.zeros(P, dtype=torch.int64, device=DEV), torch.zeros(P, dtype=torch.int32, device=DEV),
            torch.zeros(P, dtype=torch.int32, device=DEV))


def _mask_words(s, P, H, W):
    """the defined contributor-mask words (each patch's chunks up to its largest n_contrib) as {(tile, patch, chunk): word},
    and per Gaussian whether any of those bits belongs to one of its instances"""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    seen = np.zeros(P, bool)
    words = {}
    pl, cm = s["point_list"].view(np.uint32), s["cmask"].view(np.uint32)
    ncon = s["n_contrib"].reshape(-1, H, W)
    for vt, (r0, r1) in enumerate(s["ranges"].view(np.uint32)):
        v, t = divmod(vt, gx * gy)
        ty, tx = divmod(t, gx)
        for patch in range(8):
            y0, x0 = ty * 16 + (patch >> 1) * 4, tx * 16 + (patch & 1) * 8
            nmax = int(ncon[v, y0:y0 + 4, x0:x0 + 8].max()) if y0 < H and x0 < W else 0
            for c in range((nmax + 31) // 32):
                word = int(cm[((r0 >> 5) + vt + c) * 8 + patch])
                words[(vt, patch, c)] = word
                for l in range(32):
                    if word >> l & 1:
                        seen[pl[r0 + 32 * c + l] - v * P] = True
    return words, seen


@pytest.mark.parametrize("scene", ["small", "dense", "aa"])
def test_variant_state_byte_identical_and_consistent(scene):
    inp = _dense() if scene == "dense" else _small(2, seed=6)[0]
    kw = dict(antialiasing=scene == "aa")
    P, H, W = len(inp["means3D"]), inp["image_height"], inp["image_width"]
    plain = _state(inp, **kw)
    acc = _acc(P)
    var = _state(inp, contrib=acc, **kw)
    for k in plain:
        if k != "cmask":
            assert plain[k].tobytes() == var[k].tobytes(), f"{k} differs with the contribution scores on"
    words_p, seen_p = _mask_words(plain, P, H, W)
    words_v, seen_v = _mask_words(var, P, H, W)
    assert words_p == words_v, "a defined contributor-mask word differs with the contribution scores on"
    assert len(words_v) > 20 and np.array_equal(seen_p, seen_v)
    wmax = acc[1].cpu().numpy().view(np.uint32)
    assert np.array_equal(wmax > 0, seen_v), "weight_max > 0 must mean a contributor-mask bit"
    touches = acc[2].cpu().numpy().view(np.uint32)
    assert (touches[wmax > 0] >= 1).all()


def _replay_gpu_state(s, H, W):
    """the replay on the GPU's own forward state of one view (records px, py | A, B, C, o), in the oracle state's format"""
    recs = s["recs"].cpu().numpy()
    st = dict(xy=recs[:, 0:2].copy(), conic_opacity=recs[:, 4:8].copy(), point_list=s["point_list"].cpu().numpy().view(np.uint32),
              ranges=s["ranges"].cpu().numpy().view(np.uint32), num_rendered=s["num_rendered"])
    return CR.replay(st, H, W)


def test_raw_parameters_bit_exact():
    """raw=True: the activations run inside F1 with the device's exp / sigmoid / normalize, whose bits need not be the host's,
    so the oracle (fed host-activated values) is not the reference here.  The replay runs on the GPU forward's own records
    instead: it reproduces that forward's n_contrib, and the three scores bit for bit."""
    from humangaussian_b200.contribution import compute_contribution
    from humangaussian_b200.rasterizer import forward_with_state
    inp, p = _small(1, seed=7)
    H, W = inp["image_height"], inp["image_width"]
    raw = dict(opacities=p.opacity.detach().to(DEV).reshape(-1), scales=p.scaling.detach().to(DEV), rotations=p.rotation.detach().to(DEV))
    got = compute_contribution(means3D=torch.tensor(inp["means3D"], device=DEV), raw=True, **raw, **_cams([inp]))
    t = {k: torch.tensor(np.asarray(v), device=DEV) if isinstance(v, np.ndarray) else v for k, v in inp.items()}
    t.update(raw)
    *_, s, _ = forward_with_state(raw=True, **t)
    ref = _replay_gpu_state(s, H, W)
    assert np.array_equal(ref["n_contrib"], s["n_contrib"].cpu().numpy().reshape(H, W).view(np.uint32))
    ws = (got.weight_sum.cpu().numpy() * 2.0 ** 24).astype(np.uint64)
    assert np.array_equal(ws, np.array([int(x) for x in ref["weight_sum"]], np.uint64))
    assert np.array_equal(got.weight_max.cpu().numpy().view(np.uint32), ref["weight_max"])
    assert np.array_equal(got.touches.cpu().numpy(), ref["touches"])
    assert (ref["blends"] > 0).sum() > 20


def test_view_halving_does_not_double_count(monkeypatch):
    """compute_contribution halves a chunk that has too many instances.  The contribution forward passes the instance limit
    as its capacity, so a refused call stops before its blend: with the limit lowered below a 4-view chunk (4 -> 2 -> 1 views
    per call), the scores equal the unsplit call's bit for bit."""
    from humangaussian_b200 import rasterizer as R
    inp, _ = _small(1, seed=21, P=300)
    inps = [inp] * 4  # equal instance counts per view, so the single views fit under total // 3
    full = _score(inps)
    total = R.last_num_rendered()
    monkeypatch.setattr(R, "MAX_INSTANCES", total // 3)
    split = _score(inps)
    for a, b in zip(full, split):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    assert R.last_num_rendered() == total // 4
    single = _score([inp])
    assert torch.equal(full.touches, 4 * single.touches)


# ---- 3. fold invariance ----------------------------------------------------------------------------------------------------
def test_fold_invariance_130_cameras():
    from humangaussian_b200 import rasterizer as R
    from humangaussian_b200.contribution import compute_contribution
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import stack_cameras
    inp, _ = _small(1, seed=8, P=400)
    H, W = 40, 56
    cams = sample_orbit_cameras(130, H, W, seed=8)
    vm, pm, cp, tx, ty = stack_cameras(cams, DEV)
    g = {k: torch.tensor(inp[k], device=DEV) for k in ("means3D", "opacities", "scales", "rotations")}
    kw = dict(tanfovx=tx, tanfovy=ty, image_height=H, image_width=W)
    one = compute_contribution(**g, viewmatrices=vm, projmatrices=pm, **kw)
    again = compute_contribution(**g, viewmatrices=vm, projmatrices=pm, **kw)
    bytes_of = lambda c: b"".join(t.cpu().numpy().tobytes() for t in c)
    assert bytes_of(one) == bytes_of(again)
    P = len(inp["means3D"])
    colors, bg = torch.zeros(P, 3, device=DEV), torch.zeros(3, device=DEV)

    def explicit(chunks):
        acc = _acc(P)
        for lo, hi in chunks:
            R._forward_impl(g["means3D"], None, colors, g["opacities"], g["scales"], g["rotations"], None, bg, vm[lo:hi], pm[lo:hi],
                            cp[lo:hi], tx[lo:hi], ty[lo:hi], H, W, 0, 1.0, contrib=acc)
        return acc
    a = explicit([(0, 64), (64, 128), (128, 130)])
    b = explicit([(i, i + 1) for i in reversed(range(130))])
    assert a[0].cpu().numpy().tobytes() == b[0].cpu().numpy().tobytes() == (one.weight_sum * 2.0 ** 24).to(torch.int64).cpu().numpy().tobytes()
    assert a[1].cpu().numpy().tobytes() == b[1].cpu().numpy().tobytes() == one.weight_max.cpu().numpy().tobytes()
    assert a[2].cpu().numpy().tobytes() == b[2].cpu().numpy().tobytes() == one.touches.to(torch.int32).cpu().numpy().tobytes()
    assert (one.touches > 0).sum() > 100


# ---- 4. lossless prune -----------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _render(g, cams, keep=None, grads=False, **kw):
    from humangaussian_b200.rasterizer import rasterize_views
    t = {}
    for k, v in g.items():
        if k == "means3D" and v.dim() == 3:
            t[k] = v if keep is None else v[:, keep]
        else:
            t[k] = v if keep is None else v[keep]
        t[k] = t[k].clone().requires_grad_(grads)
    f3d = kw.pop("filter_3d", None)
    if f3d is not None and keep is not None:
        f3d = f3d[keep]
    with _deterministic(grads):
        c, r, d, a = rasterize_views(**t, **cams, filter_3d=f3d, **kw)
        out = dict(color=c, radii=r, depth=d, alpha=a)
        if grads:
            gC, gD, gA = (torch.tensor(np.stack([grad_images(c.shape[-2], c.shape[-1], 5 + v)[j] for v in range(c.shape[0])]), device=DEV)
                          for j in range(3))
            torch.autograd.backward([c, d, a], [gC, gD, gA])
            for k in t:
                out["d_" + k] = t[k].grad
    return {k: v.detach().cpu().numpy() for k, v in out.items()}


def _lossless(g, cams, grads=True, **kw):
    from humangaussian_b200.contribution import compute_contribution
    sc = compute_contribution(**{k: v for k, v in g.items() if k != "shs"}, **{k: cams[k] for k in ("viewmatrices", "projmatrices",
                              "tanfovx", "tanfovy", "image_height", "image_width")}, **{k: v for k, v in kw.items()})
    keep = (sc.touches > 0)
    assert 0 < int(keep.sum()) < keep.numel(), "scene must have both touched and untouched Gaussians"
    full = _render(g, cams, grads=grads, **dict(kw))
    pruned = _render(g, cams, keep=keep, grads=grads, **dict(kw))
    for k in ("color", "depth", "alpha"):
        assert full[k].tobytes() == pruned[k].tobytes(), f"{k} changed after removing untouched Gaussians"
    kn = keep.cpu().numpy()
    assert np.array_equal(full["radii"][:, kn], pruned["radii"])
    if grads:
        for k in full:
            if k.startswith("d_"):
                a = full[k][:, kn] if (k == "d_means3D" and full[k].ndim == 3) else full[k][kn]
                assert a.tobytes() == pruned[k].tobytes(), f"deterministic {k} of the survivors changed"
    return keep


def _gpu_geom(inp, keys=("means3D", "opacities", "shs", "scales", "rotations")):
    return {k: torch.tensor(np.asarray(inp[k], np.float32), device=DEV) for k in keys}


def _render_cams(inps, deg):
    c = _cams(inps)
    g = lambda k: torch.stack([torch.as_tensor(np.asarray(i[k], np.float32)) for i in inps]).to(DEV)
    return dict(c, camposs=g("campos").reshape(-1, 3), bg=torch.tensor(inps[0]["bg"], device=DEV), sh_degree=deg)


def _opaque(deg, seed, P=300):
    """a dense, nearly opaque body: from any one camera many of its Gaussians sit behind the surface"""
    inp, _ = _small(deg, seed=seed, P=P, H=32, W=48, dist=1.3)
    inp["opacities"] = np.clip(inp["opacities"] * 8, 0, 0.99999).astype(np.float32)
    inp["scales"] = (inp["scales"] * 2.0).astype(np.float32)
    return inp


@pytest.mark.parametrize("n_cams", [1, 2])
def test_lossless_prune_small_scenes(n_cams):
    inp = _opaque(1, seed=13 + n_cams)
    _lossless(_gpu_geom(inp), _render_cams(_orbit_inps(inp, n_cams, 32, 48, seed=13), 1))


def test_lossless_prune_aa_and_filter_3d():
    from test_gpu_filter3d import _var_for
    inp = _opaque(2, seed=15, P=600)
    var = torch.tensor(_var_for(inp, seed=15), device=DEV)
    _lossless(_gpu_geom(inp), _render_cams(_orbit_inps(inp, 1, 32, 48, seed=15), 2), antialiasing=True, filter_3d=var)


def test_lossless_prune_per_view_means():
    inp = _opaque(1, seed=16)
    rng = np.random.RandomState(16)
    g = _gpu_geom(inp)
    g["means3D"] = torch.stack([g["means3D"] + 0.01 * torch.tensor(rng.randn(300, 3), dtype=torch.float32, device=DEV)
                                for _ in range(2)])
    _lossless(g, _render_cams([inp] * 2, 1))


def test_lossless_prune_300k_512_eight_views():
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import stack_cameras
    from humangaussian_b200.scene import sample_ply_scene
    p = sample_ply_scene(300000, 0)
    with torch.no_grad():
        g = dict(means3D=p.get_xyz.to(DEV).contiguous(), opacities=p.get_opacity.to(DEV).contiguous(),
                 shs=p.get_features.to(DEV).contiguous(), scales=p.get_scaling.to(DEV).contiguous(),
                 rotations=p.get_rotation.to(DEV).contiguous())
    vm, pm, cp, tx, ty = stack_cameras(sample_orbit_cameras(8, 512, 512, seed=77), DEV)
    cams = dict(viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx, tanfovy=ty, image_height=512, image_width=512,
                bg=torch.zeros(3, device=DEV), sh_degree=0)
    keep = _lossless(g, cams, grads=False)
    print(f"300k / 512^2 / 8 views: {int((~keep).sum())} of 300000 untouched")


# ---- 5. prune by mask ------------------------------------------------------------------------------------------------------
def _random_groups(P, K, seed):
    from test_gpu_densify import random_state, to_device
    st = random_state(P, K, seed)
    return to_device(st)


@pytest.mark.parametrize("P,mode", [(1000, "random"), (257, "none"), (300, "all_but_one"), (65_537, "random")])
def test_prune_points_matches_boolean_indexing(P, mode):
    from humangaussian_b200.densify import prune_points
    params, moments, stats = _random_groups(P, 4, P)
    rng = np.random.RandomState(P)
    rm = {"random": rng.rand(P) < 0.4, "none": np.zeros(P, bool), "all_but_one": np.arange(P) != P // 3}[mode]
    remove = torch.tensor(rm, device=DEV)
    keep = ~remove
    p2, m2, s2 = prune_points(params, moments, stats, remove)
    for k in params:
        assert p2[k].cpu().numpy().tobytes() == params[k][keep].cpu().numpy().tobytes(), k
        for a, b in zip(m2[k], moments[k]):
            assert a.cpu().numpy().tobytes() == b[keep].cpu().numpy().tobytes(), k
    for k in ("xyz_gradient_accum", "denom", "max_radii2D"):
        assert getattr(s2, k).cpu().numpy().tobytes() == getattr(stats, k)[keep].cpu().numpy().tobytes(), k


def test_prune_points_refuses_removing_everything_and_bad_masks():
    from humangaussian_b200.densify import prune_points
    params, moments, stats = _random_groups(100, 1, 1)
    with pytest.raises(ValueError, match="every Gaussian"):
        prune_points(params, moments, stats, torch.ones(100, dtype=torch.bool, device=DEV))
    with pytest.raises(ValueError):
        prune_points(params, moments, stats, torch.ones(100, dtype=torch.uint8, device=DEV))
    with pytest.raises(ValueError):
        prune_points(params, moments, stats, torch.ones(99, dtype=torch.bool, device=DEV))


def test_prune_points_packed_then_keep_training():
    from humangaussian_b200 import dist
    from humangaussian_b200.densify import DensifyStats, prune_points_packed
    from humangaussian_b200.optim import PackedAdam
    from humangaussian_b200.rasterizer import packed_layout, rasterize_views_packed
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import stack_cameras
    from humangaussian_b200.scene import synthetic_body
    P, K = 3001, 4  # SH degree 1
    p = synthetic_body(P, sh_degree=1, seed=3)
    raw = dict(xyz=p.xyz, scaling=p.scaling, rotation=p.rotation, opacity=p.opacity,
               features=torch.cat((p.features_dc, p.features_rest), 1))
    flat = dist.pack({k: v.to(DEV) for k, v in raw.items()})
    lrs = dict(xyz=1e-4, f_dc=1e-3, f_rest=1e-4, opacity=1e-2, scaling=1e-3, rotation=1e-3)
    opt = PackedAdam(flat.requires_grad_(True), P, K, lrs)
    vm, pm, cp, tx, ty = stack_cameras(sample_orbit_cameras(2, 64, 64, seed=3), DEV)
    kw = dict(viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx, tanfovy=ty, image_height=64, image_width=64,
              bg=torch.zeros(3, device=DEV), sh_degree=1, raw=True)
    c, *_ = rasterize_views_packed(opt.packed, P, K, **kw)
    c.square().mean().backward()
    opt.step()
    opt.zero_grad()
    stats = DensifyStats.zeros(P, DEV)
    stats.denom += torch.arange(P, device=DEV, dtype=torch.float32)[:, None]
    old = opt.packed.detach().clone()
    m_old = {k: opt.state[opt.packed][k].clone() for k in ("exp_avg", "exp_avg_sq")}
    remove = torch.tensor(np.random.RandomState(3).rand(P) < 0.3, device=DEV)
    keep = ~remove
    P2 = prune_points_packed(opt, stats, remove)
    assert P2 == int(keep.sum()) and opt.P == P2
    for (o, n, shape), (o2, n2, shape2) in zip(packed_layout(P, K)[0], packed_layout(P2, K)[0]):
        want = old[o:o + n].view(shape)[keep]
        assert opt.packed.detach()[o2:o2 + n2].view(shape2).cpu().numpy().tobytes() == want.cpu().numpy().tobytes()
        for k in m_old:
            assert opt.state[opt.packed][k][o2:o2 + n2].view(shape2).cpu().numpy().tobytes() == \
                m_old[k][o:o + n].view(shape)[keep].cpu().numpy().tobytes()
    assert stats.denom.cpu().numpy().tobytes() == torch.arange(P, dtype=torch.float32)[keep.cpu()][:, None].numpy().tobytes()
    c, *_ = rasterize_views_packed(opt.packed, P2, K, **kw)
    c.square().mean().backward()
    opt.step()
    assert torch.isfinite(opt.packed).all()


def test_argument_errors():
    from humangaussian_b200.contribution import compute_contribution
    inp, _ = _small(0, seed=1, P=50)
    g = {k: torch.tensor(inp[k], device=DEV) for k in ("means3D", "opacities", "scales", "rotations")}
    cams = _cams([inp])
    with pytest.raises(ValueError):
        compute_contribution(**dict(g, means3D=g["means3D"].double()), **cams)
    with pytest.raises(ValueError):
        compute_contribution(**dict(g, opacities=g["opacities"][:10]), **cams)
    with pytest.raises(ValueError):
        compute_contribution(g["means3D"], g["opacities"], g["scales"], None, **cams)
    with pytest.raises(ValueError):
        compute_contribution(g["means3D"], g["opacities"], cov3D_precomp=torch.zeros(50, 6, device=DEV),
                             filter_3d=torch.zeros(50, device=DEV), **cams)
    big = dict(cams, image_height=65536, image_width=65536)
    with pytest.raises(ValueError, match="2\\^32"):
        compute_contribution(**g, **big)
    with pytest.raises(ValueError):
        compute_contribution(**g, **dict(cams, tanfovx=[]))


def test_classic_comparator_reports_unsupported():
    from humangaussian_b200 import rasterizer as R
    lib = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "baseline", "libb200gs_classic.so")
    inp, _ = _small(0, seed=1, P=50)
    with R.use_library(lib):
        with pytest.raises(RuntimeError, match="not supported"):
            _score([inp])
