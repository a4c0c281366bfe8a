"""GPU parity tests proper: the CUDA path (through the C-ABI) against the CPU oracle on the same seeded inputs.

Bar (BASELINE.json north_star): bit-exact on tile / sort indices; 1e-5 abs / 1e-4 rel on RGB, depth, alpha and
all gradients.  Because both sides follow the same pinned float operation order the forward pass is in fact
compared BIT-FOR-BIT (images included); the backward (different summation order) uses the 1e-5 / 1e-4 tolerance in the
form util.grads_agree states: per-Gaussian gradient vectors row-wise with no exceptions, elementwise for >= 99.9 %.
The backward blend's own intermediates are checked directly as well (below _oracle): the forward's contributor masks bit
for bit, and its per-Gaussian sums against float64 sums within a derived error bound, with no exceptions."""
import math

import numpy as np
import pytest
import torch

from util import close, grad_images, grads_agree, small_scene

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _gpu_inputs(inp, keys=("means3D", "opacities", "shs", "scales", "rotations"), extra=None):
    t = {k: torch.tensor(inp[k], device=DEV, requires_grad=True) for k in keys if inp.get(k) is not None}
    if extra:
        for k, v in extra.items():
            t[k] = torch.tensor(v, device=DEV, requires_grad=True)
    return t


def _settings(inp):
    from humangaussian_b200.rasterizer import GaussianRasterizationSettings
    g = lambda k: torch.tensor(inp[k], device=DEV)
    return GaussianRasterizationSettings(
        image_height=inp["image_height"], image_width=inp["image_width"], tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"],
        bg=g("bg"), scale_modifier=inp.get("scale_modifier", 1.0), viewmatrix=g("viewmatrix"), projmatrix=g("projmatrix"),
        sh_degree=inp.get("sh_degree", 0), campos=g("campos"), prefiltered=False, debug=False)


def _oracle(inp, seed=0, threads=0):
    from oracle.gs_oracle import Oracle
    o = Oracle(threads=threads)
    out = o.forward(**inp)
    st = o.state()
    gimg = grad_images(inp["image_height"], inp["image_width"], seed)
    grads = o.backward(*gimg, sums_err_const=SUMS_K)
    return out, st, gimg, grads


# ---- the backward blend's intermediates -------------------------------------------------------------------------------
#
# Contributor masks.  The forward writes one u32 per (32-entry chunk, patch); the backward walks only their set bits.  They
# are integer state of a bit-exact forward, so every word the backward reads -- chunks c <= (wmax - 1) >> 5, wmax = the
# largest n_contrib over the patch's pixels -- must equal the word packed from the oracle's per-entry contrib_patches.
#
# Sums.  The backward blend leaves, per (view, Gaussian), ten float32 sums in the ScreenGrad record: six moments of
# q = G*dL/dalpha (1, dx, dy, dx^2, dx*dy, dy^2) and W0..W3 = sum w*(gC, gD), w = alpha*T.  The oracle exports the same
# sums in float64 and an error scale per component, E_k = sum over terms of m * (r + K + N_g), where m is the term's
# magnitude (gs_oracle.c: |phi_k| * G * (T*(|cg|_abs + |rg|_abs) + T_final*|bg.gC|_abs/(1-alpha)) for a q moment, |w*g_k|
# for W_k), r its replay depth (transmittance recoveries done for the pixel so far, this one included) and N_g the number of
# (tile, patch) partial sums the kernel adds into the Gaussian's record.  The check is |gpu - ref| <= C * u * E_k for every
# (Gaussian, component), u = 2^-24, no exceptions.  Both sides compute G, alpha, dx, dy, the colours and the upstream
# gradients bit-identically; the error model counts, in units of u * m and to first order (r*u <= 2e-3 even for the
# 17 k-deep tiles), the three ways they differ:
#   transmittance chain -- the oracle divides (IEEE, 1 rounding per recovery), the kernel multiplies by a Newton-refined
#     reciprocal (<= 1 for the reciprocal + 1 for the product): 3r between the two.
#   the cg - rg cancellation -- the kernel folds the five colour/depth/alpha recurrences into one scalar (fma form, <= 3 per
#     step), the oracle keeps five (<= 4 per step, relative to their absolute sum): 7r; forming cg, the difference and the
#     background term 1/(1-alpha) * T_final * bg.gC: kernel 4 + 1 + 6 + 2, oracle 6 + 7 + 1: 27.
#   summation order -- the oracle sums in float64 (negligible); the kernel forms phi_k * q in float32 (<= 2), sums a row of
#     8 pixels, two rows and the two half-warps (<= 9; W_k: 16 fmas + 1 = 17), then adds the Gaussian's N_g partial sums with
#     float atomics in any order (<= N_g - 1, relative to the sum of |partials|).
# q moments: 10r + 27 + 2 + 9 + N_g - 1 = 10r + 37 + N_g;  W_k: 3r + 2 (w = alpha*T on both sides) + 17 + N_g - 1.
# Both are <= 10 * (r + 4 + N_g): K = 4, C = 10.
SUMS_K = 4.0
SUMS_C = 10.0
U = 2.0 ** -24
SUM_NAMES = ("S0", "Sx", "Sy", "Sxx", "Sxy", "Syy", "W0", "W1", "W2", "W3")


def _patch_wmax(n_contrib, H, W):
    """[tiles, 8]: largest n_contrib over the in-image pixels of each 8x4 patch (patch = band * 2 + x half)"""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    nc = np.zeros((gy * 16, gx * 16), np.int64)
    nc[:H, :W] = n_contrib
    return nc.reshape(gy, 4, 4, gx, 2, 8).max(axis=(2, 5)).transpose(0, 2, 1, 3).reshape(gx * gy, 8)


def _packed_masks(contrib_patches, r0, r1, nch):
    """[nch, 8] u32: the contributor-mask words of one tile packed from the oracle's per-entry patch bits"""
    bits = np.zeros(nch * 32, np.uint8)
    seg = contrib_patches[r0:min(r1, r0 + nch * 32)]
    bits[:len(seg)] = seg
    b = (bits[:, None] >> np.arange(8, dtype=np.uint8)) & 1
    return (b.reshape(nch, 32, 8).astype(np.uint64) << np.arange(32, dtype=np.uint64)[None, :, None]).sum(1).astype(np.uint32)


def _check_masks(masks, ranges, n_contrib, o_st, H, W, v=0):
    """Contributor masks of view v (GPU words, GPU ranges of the batch, GPU n_contrib [H,W] of the view) against the
    oracle's state of that view, bit for bit.  Returns (words compared, per-tile [8] wmax) for coverage assertions."""
    masks = np.ascontiguousarray(masks).view(np.uint32)
    ntiles = ((W + 15) // 16) * ((H + 15) // 16)
    wmax = _patch_wmax(n_contrib, H, W)
    checked = 0
    for t in np.nonzero(wmax.max(1) > 0)[0]:
        vt = v * ntiles + int(t)
        nch = (int(wmax[t].max()) + 31) >> 5
        r0, r1 = (int(x) for x in o_st["ranges"][t])
        want = _packed_masks(o_st["contrib_patches"], r0, r1, nch)
        base = ((int(ranges[vt, 0]) >> 5) + vt) * 8
        got = masks[base + 8 * np.arange(nch)[:, None] + np.arange(8)[None, :]]
        read = np.arange(nch)[:, None] <= (wmax[t][None, :] - 1) >> 5  # the words the backward reads
        bad = read & (got != want)
        if bad.any():
            c, p = np.argwhere(bad)[0]
            raise AssertionError(f"view {v} tile {t}: {int(bad.sum())} contributor-mask words differ; first: chunk {c} patch {p} "
                                 f"gpu {got[c, p]:#010x} oracle {want[c, p]:#010x} (wmax {wmax[t][p]})")
        checked += int(read.sum())
    return checked, wmax


def _check_sums(gpu_sums, o_grads, what=""):
    """gpu_sums [P,12] (one view's ScreenGrad records) against the oracle's float64 sums and error scales: no exceptions."""
    ref, E = o_grads["sums"], o_grads["sums_err"]
    err = np.abs(gpu_sums[:, :10].astype(np.float64) - ref)
    lim = SUMS_C * U * E
    bad = err > lim
    if bad.any():
        ratio = err / np.maximum(lim, 1e-300)
        worst = np.unravel_index(np.argmax(np.where(bad, ratio, 0)), bad.shape)
        per = {SUM_NAMES[k]: int(bad[:, k].sum()) for k in range(10) if bad[:, k].any()}
        raise AssertionError(f"{what}backward-blend sums outside C*u*E in {int(bad.any(1).sum())} Gaussians {per}; worst: Gaussian "
                             f"{worst[0]} {SUM_NAMES[worst[1]]} gpu {gpu_sums[worst[0], worst[1]]:.9g} ref {ref[worst]:.9g} "
                             f"|diff| {err[worst]:.3g} = {ratio[worst]:.3g}x the bound")
    assert np.abs(gpu_sums[:, 10:]).max(initial=0.0) == 0.0, "ScreenGrad padding written"


def _gpu_blend_state(inp, gimg):
    """One forward + backward through the library: (state dict as numpy, sums [V,P,12])."""
    from humangaussian_b200.rasterizer import forward_backward_with_state
    kw = {k: (torch.tensor(v, device=DEV) if isinstance(v, np.ndarray) else v) for k, v in inp.items()}
    gC, gD, gA = (torch.tensor(g, device=DEV) for g in gimg)
    *_, st, sums = forward_backward_with_state(gC, gD, gA, **kw)
    return {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in st.items()}, sums.cpu().numpy()


def _check_backward_sums(inp, gimg, o_grads):
    """The backward blend's sums of a single-view call against the oracle's (beside _check_backward, same inputs)."""
    _, sums = _gpu_blend_state(inp, gimg)
    _check_sums(sums[0], o_grads)


def test_exp_bit_exact():
    from humangaussian_b200.rasterizer import device_exp
    from oracle.gs_oracle import gs_exp
    rng = np.random.RandomState(0)
    x = np.concatenate([-rng.rand(20000) * 20, -rng.rand(2000) * 100, np.array([0.0, -1e-8, -87.0, -88.0, -1e4, -5.541263545])]).astype(np.float32)
    y = device_exp(torch.tensor(x, device=DEV)).cpu().numpy()
    assert np.array_equal(y.view(np.uint32), gs_exp(x).view(np.uint32))
    m = x > -10  # the range that can reach alpha >= 1/255; beyond it the single-step reduction error grows with |x|
    assert np.max(np.abs(y[m] / np.exp(x[m].astype(np.float64)) - 1)) < 2.5e-7
    m = x > -80
    assert np.max(np.abs(y[m] / np.exp(x[m].astype(np.float64)) - 1)) < 2e-6


def _check_forward_state(inp, o_out, o_st):
    from humangaussian_b200.rasterizer import forward_with_state
    kw = {k: (torch.tensor(v, device=DEV) if isinstance(v, np.ndarray) else v) for k, v in inp.items()}
    color, radii, depth, alpha, st, _ = forward_with_state(**kw)
    col, rad, dep, alp = o_out
    P = len(rad)
    assert np.array_equal(radii[0].cpu().numpy(), rad)
    assert np.array_equal(st["tiles_touched"].cpu().numpy().view(np.uint32), o_st["tiles_touched"])
    assert st["num_rendered"] == o_st["num_rendered"]
    assert np.array_equal(st["sorted_keys"].cpu().numpy().view(np.uint64), o_st["keys"]), "sorted (tile|depth) keys differ"
    assert np.array_equal(st["point_list"].cpu().numpy().view(np.uint32), o_st["point_list"]), "sort order differs"
    assert np.array_equal(st["ranges"].cpu().numpy().view(np.uint32), o_st["ranges"])
    recs = st["recs"].cpu().numpy()
    vis = rad > 0
    f = lambda a: np.ascontiguousarray(a).view(np.uint32)
    assert np.array_equal(f(recs[vis][:, 0:2]), f(o_st["xy"][vis])), "pixel centres not bit-identical"
    assert np.array_equal(f(recs[vis][:, 4:8]), f(o_st["conic_opacity"][vis])), "conic/opacity not bit-identical"
    assert np.array_equal(f(recs[vis][:, 8:11]), f(o_st["rgb"][vis])), "SH colours not bit-identical"
    assert np.array_equal(f(recs[vis][:, 11]), f(o_st["depths"][vis])), "depths not bit-identical"
    assert np.array_equal(st["clamped"].cpu().numpy()[vis], (o_st["clamped"][vis] * np.array([1, 2, 4], np.uint8)).sum(1).astype(np.uint8))
    assert np.array_equal(st["n_contrib"][0].cpu().numpy().view(np.uint32), o_st["n_contrib"])
    assert np.array_equal(f(st["final_T"][0].cpu().numpy()), f(o_st["final_T"]))
    assert np.array_equal(f(color[0].cpu().numpy()), f(col)), "RGB not bit-identical"
    assert np.array_equal(f(depth[0].cpu().numpy()), f(dep)), "depth image not bit-identical"
    assert np.array_equal(f(alpha[0].cpu().numpy()), f(alp)), "alpha image not bit-identical"
    _check_masks(st["contributor_masks"].cpu().numpy(), st["ranges"].cpu().numpy(), st["n_contrib"][0].cpu().numpy(), o_st,
                 inp["image_height"], inp["image_width"])


def _check_backward(inp, o_out, gimg, o_grads, keys=("means3D", "opacities", "shs", "scales", "rotations"), extra=None, criterion=None):
    criterion = criterion or {}
    from humangaussian_b200.rasterizer import GaussianRasterizer
    t = _gpu_inputs(inp, keys, extra)
    P = inp["means3D"].shape[0]
    m2d = torch.zeros(P, 3, device=DEV, requires_grad=True)
    r = GaussianRasterizer(_settings(inp))
    c, rad, d, a = r(means3D=t["means3D"], means2D=m2d, shs=t.get("shs"), colors_precomp=t.get("colors_precomp"),
                     opacities=t["opacities"], scales=t.get("scales"), rotations=t.get("rotations"), cov3D_precomp=t.get("cov3D_precomp"))
    gC, gD, gA = (torch.tensor(g, device=DEV) for g in gimg)
    ((c * gC).sum() + (d * gD).sum() + (a * gA).sum()).backward()
    names = {"means3D": "means3D", "opacities": "opacities", "shs": "shs", "scales": "scales", "rotations": "rotations",
             "colors_precomp": "colors_precomp", "cov3D_precomp": "cov3D_precomp"}
    for k in t:
        ok, msg = grads_agree(t[k].grad.cpu().numpy().reshape(o_grads[names[k]].shape), o_grads[names[k]], **criterion)
        assert ok, f"dL/d{k}: {msg}"
    ok, msg = grads_agree(m2d.grad.cpu().numpy(), o_grads["means2D"], **criterion)
    assert ok, f"dL/dmeans2D: {msg}"


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("seed", [0, 1])
def test_small_scene_fwd_bwd(deg, seed):
    inp, _, _ = small_scene(P=600, deg=deg, seed=seed, H=72, W=104)  # partial edge tiles on both axes
    o_out, o_st, gimg, o_grads = _oracle(inp, seed)
    _check_forward_state(inp, o_out, o_st)
    _check_backward(inp, o_out, gimg, o_grads)
    _check_backward_sums(inp, gimg, o_grads)


def test_dense_opaque_scene_terminates():
    """High opacity, many layers: exercises the T < 1e-4 stop, the 0.99 clamp and n_contrib < list length."""
    inp, _, p = small_scene(P=4000, deg=1, seed=5, H=64, W=64, dist=1.2)
    inp["opacities"] = np.clip(inp["opacities"] * 6, 0, 0.9999).astype(np.float32)
    inp["scales"] = (inp["scales"] * 2.5).astype(np.float32)
    o_out, o_st, gimg, o_grads = _oracle(inp, 2)
    assert (o_st["final_T"] < 1e-3).mean() > 0.05, "scene is not opaque enough to test early termination"
    _check_forward_state(inp, o_out, o_st)
    _check_backward(inp, o_out, gimg, o_grads)
    _check_backward_sums(inp, gimg, o_grads)


def test_precomputed_cov_and_colors():
    inp, _, _ = small_scene(P=500, deg=0, seed=7, H=48, W=80)
    from oracle.gs_oracle import Oracle
    o = Oracle()
    o.forward(**inp)
    st = o.state()
    inp2 = dict(inp)
    inp2.pop("shs"); inp2.pop("scales"); inp2.pop("rotations")
    inp2["colors_precomp"] = np.abs(st["rgb"]).astype(np.float32) + 0.05
    inp2["cov3D_precomp"] = st["cov3d"].copy()
    inp2["sh_degree"] = 0
    o_out, o_st, gimg, o_grads = _oracle(inp2, 3)
    _check_forward_state(inp2, o_out, o_st)
    _check_backward(inp2, o_out, gimg, o_grads, keys=("means3D", "opacities", "colors_precomp", "cov3D_precomp"))
    _check_backward_sums(inp2, gimg, o_grads)


def test_behind_camera_and_empty():
    from humangaussian_b200.rasterizer import GaussianRasterizer
    inp, _, _ = small_scene(P=300, deg=0, seed=1, H=32, W=32)
    inp["means3D"] = (inp["means3D"] + np.array([50.0, 0, 0], np.float32)).astype(np.float32)  # behind the camera: all culled
    o_out, o_st, gimg, o_grads = _oracle(inp, 0)
    assert o_st["num_rendered"] == 0
    _check_forward_state(inp, o_out, o_st)
    _check_backward(inp, o_out, gimg, o_grads)
    _check_backward_sums(inp, gimg, o_grads)
    # P == 0
    s = _settings(inp)
    z = lambda *shape: torch.zeros(*shape, device=DEV, requires_grad=True)
    c, rad, d, a = GaussianRasterizer(s)(means3D=z(0, 3), means2D=z(0, 3), shs=z(0, 1, 3), colors_precomp=None, opacities=z(0, 1),
                                          scales=z(0, 3), rotations=z(0, 4), cov3D_precomp=None)
    assert rad.numel() == 0
    assert torch.equal(c, torch.tensor(inp["bg"], device=DEV)[:, None, None].expand(3, 32, 32))
    assert float(d.abs().max()) == 0 and float(a.abs().max()) == 0


def test_argument_errors_match_reference_wrapper():
    from humangaussian_b200.rasterizer import GaussianRasterizer
    inp, _, _ = small_scene(P=10, deg=0, seed=1, H=16, W=16)
    t = _gpu_inputs(inp)
    r = GaussianRasterizer(_settings(inp))
    m2d = torch.zeros(10, 3, device=DEV)
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        r(means3D=t["means3D"], means2D=m2d, shs=None, colors_precomp=None, opacities=t["opacities"], scales=t["scales"], rotations=t["rotations"])
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(means3D=t["means3D"], means2D=m2d, shs=t["shs"], opacities=t["opacities"], scales=None, rotations=None, cov3D_precomp=None)


def test_batched_views_equal_per_view_loop():
    """rasterize_views (V cameras, one call) == V single-view calls: outputs bit-identical, parameter grads = sum."""
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.rasterizer import GaussianRasterizer, GaussianRasterizationSettings, rasterize_views
    from humangaussian_b200.renderer import stack_cameras
    inp, _, _ = small_scene(P=3000, deg=2, seed=4, H=80, W=96)
    cams = sample_orbit_cameras(5, 80, 96, seed=1, device=DEV)
    vm, pm, cp, tanx, tany = stack_cameras(cams, DEV)
    bg = torch.tensor(inp["bg"], device=DEV)
    keys = ("means3D", "opacities", "shs", "scales", "rotations")
    ta, tb = _gpu_inputs(inp, keys), _gpu_inputs(inp, keys)
    V, P = 5, 3000
    m2d_b = torch.zeros(V, P, 3, device=DEV, requires_grad=True)
    cb, rb, db, ab = rasterize_views(means3D=tb["means3D"], opacities=tb["opacities"], viewmatrices=vm, projmatrices=pm, camposs=cp,
                                     tanfovx=tanx, tanfovy=tany, image_height=80, image_width=96, bg=bg, sh_degree=2,
                                     shs=tb["shs"], scales=tb["scales"], rotations=tb["rotations"], means2D=m2d_b)
    rng = np.random.RandomState(0)
    gw = [torch.tensor(rng.randn(V, c, 80, 96).astype(np.float32), device=DEV) for c in (3, 1, 1)]
    ((cb * gw[0]).sum() + (db * gw[1]).sum() + (ab * gw[2]).sum()).backward()
    loss = 0
    m2ds = []
    for v in range(V):
        s = GaussianRasterizationSettings(80, 96, tanx[v], tany[v], bg, 1.0, vm[v], pm[v], 2, cp[v], False, False)
        m2d = torch.zeros(P, 3, device=DEV, requires_grad=True)
        m2ds.append(m2d)
        c, r, d, a = GaussianRasterizer(s)(means3D=ta["means3D"], means2D=m2d, shs=ta["shs"], opacities=ta["opacities"],
                                            scales=ta["scales"], rotations=ta["rotations"])
        assert torch.equal(c, cb[v]) and torch.equal(d, db[v]) and torch.equal(a, ab[v]) and torch.equal(r, rb[v])
        loss = loss + (c * gw[0][v]).sum() + (d * gw[1][v]).sum() + (a * gw[2][v]).sum()
    loss.backward()
    for k in keys:
        ok, worst = close(tb[k].grad.cpu().numpy(), ta[k].grad.cpu().numpy())
        assert ok, f"batched dL/d{k} differs from the per-view sum ({worst:.2f}x tolerance)"
    for v in range(V):
        ok, worst = close(m2d_b.grad[v].cpu().numpy(), m2ds[v].grad.cpu().numpy())
        assert ok


def test_batched_views_masks_and_sums_per_camera():
    """V = 3 cameras in one call: each view's contributor masks (inside the batch's shared mask region, tile vt = v*tiles +
    tile) and ScreenGrad records (record v*P + g) against that camera's own oracle run."""
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.rasterizer import forward_backward_with_state
    from humangaussian_b200.renderer import stack_cameras
    V, H, W = 3, 72, 104
    inp, _, _ = small_scene(P=1500, deg=1, seed=6, H=H, W=W)
    cams = sample_orbit_cameras(V, H, W, seed=4)
    vm, pm, cp, tanx, tany = stack_cameras(cams, "cpu")
    views = []
    for v in range(V):
        iv = dict(inp, viewmatrix=vm[v].numpy(), projmatrix=pm[v].numpy(), campos=cp[v].numpy(), tanfovx=float(tanx[v]),
                  tanfovy=float(tany[v]))
        views.append(_oracle(iv, 40 + v))
    kw = {k: (torch.tensor(x, device=DEV) if isinstance(x, np.ndarray) else x) for k, x in inp.items()}
    kw.update(viewmatrix=vm.to(DEV), projmatrix=pm.to(DEV), campos=cp.to(DEV), tanfovx=[float(t) for t in tanx],
              tanfovy=[float(t) for t in tany])
    gimg = [torch.tensor(np.stack([views[v][2][k] for v in range(V)]), device=DEV) for k in range(3)]
    *_, st, sums = forward_backward_with_state(*gimg, **kw)
    masks, ranges, nc = (st[k].cpu().numpy() for k in ("contributor_masks", "ranges", "n_contrib"))
    sums = sums.cpu().numpy()
    for v, (o_out, o_st, _, o_grads) in enumerate(views):
        assert np.array_equal(nc[v].view(np.uint32), o_st["n_contrib"])
        checked, _ = _check_masks(masks, ranges, nc[v], o_st, H, W, v=v)
        assert checked > 100
        _check_sums(sums[v], o_grads, what=f"view {v}: ")
        assert np.abs(o_grads["sums"]).max() > 0


def test_medium_scene_512():
    """BASELINE config 2 shape: 512x512, forward+backward, tens of thousands of Gaussians (synthetic body)."""
    inp, _, _ = small_scene(P=60000, deg=0, seed=11, H=512, W=512, big=False, dist=2.0, fovy_deg=70.0, elev=15.0, azim=0.0)
    o_out, o_st, gimg, o_grads = _oracle(inp, 5)
    assert o_st["num_rendered"] > 50000
    _check_forward_state(inp, o_out, o_st)
    _check_backward(inp, o_out, gimg, o_grads)
    _check_backward_sums(inp, gimg, o_grads)


def test_render_wrapper_dict_and_densification_signal():
    """render() mirror returns the reference's keys; viewspace_points.grad carries the means2D gradient
    (consumed at threestudio/systems/GaussianDreamer.py:385-391)."""
    from humangaussian_b200.cameras import Camera, orbit_c2w
    from humangaussian_b200.renderer import PipelineParams, render
    from humangaussian_b200.scene import synthetic_body
    p = synthetic_body(5000, sh_degree=0, seed=2).to(DEV)
    for t in (p.xyz, p.features_dc, p.features_rest, p.scaling, p.rotation, p.opacity):
        t.requires_grad_(True)
    cam = Camera(orbit_c2w(10, 30, 1.8), math.radians(60), 128, 128, device=DEV)
    with torch.autocast("cuda", dtype=torch.float16):  # the trainer runs under 16-mixed (configs/test.yaml:104)
        out = render(cam, p, PipelineParams(), torch.zeros(3, device=DEV))
    assert set(out) == {"render", "viewspace_points", "visibility_filter", "radii", "depth_3dgs", "alpha_3dgs"}
    assert out["render"].shape == (3, 128, 128) and out["render"].dtype == torch.float32
    assert out["radii"].dtype == torch.int32 and out["visibility_filter"].dtype == torch.bool
    (out["render"].sum() + out["depth_3dgs"].sum()).backward()
    g = out["viewspace_points"].grad
    assert g is not None and g.shape == (5000, 3) and float(g[:, 2].abs().max()) == 0 and float(g[:, :2].abs().max()) > 0
    assert p.xyz.grad is not None and torch.isfinite(p.xyz.grad).all() and p.scaling.grad.abs().max() > 0


def test_mark_visible():
    from humangaussian_b200.rasterizer import GaussianRasterizer
    inp, _, _ = small_scene(P=1000, deg=0, seed=1, H=32, W=32)
    r = GaussianRasterizer(_settings(inp))
    vis = r.markVisible(torch.tensor(inp["means3D"], device=DEV)).cpu().numpy()
    V = inp["viewmatrix"].reshape(-1)
    m = inp["means3D"]
    z = (V[2] * m[:, 0] + V[6] * m[:, 1]) + V[10] * m[:, 2] + V[14]
    assert (vis == (z > 0.2)).mean() > 0.999


def test_real_scene_512_config2():
    """BASELINE config 2 in miniature: the reference's own scene (a seed-0 8k subsample of content/sample.ply: real
    anisotropy / opacity statistics; fixture tests/golden/sample_ply_8k.npz), eval-orbit camera, 512x512, fwd+bwd."""
    import os
    from humangaussian_b200.cameras import Camera, orbit_c2w
    from util import ROOT
    c = np.load(os.path.join(ROOT, "tests", "golden", "sample_ply_8k.npz"))
    xyz = np.stack([c["x"], c["y"], c["z"]], 1)
    sc = (np.exp(np.stack([c["scale_0"], c["scale_1"], c["scale_2"]], 1)) * 4.0).astype(np.float32)
    q = np.stack([c["rot_0"], c["rot_1"], c["rot_2"], c["rot_3"]], 1)
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    op = (1 / (1 + np.exp(-c["opacity"]))).astype(np.float32)
    sh = np.stack([c["f_dc_0"], c["f_dc_1"], c["f_dc_2"]], 1)[:, None, :].astype(np.float32)
    cam = Camera(orbit_c2w(15.0, 0.0, 2.0), math.radians(70), 512, 512)
    inp = dict(means3D=xyz.astype(np.float32), opacities=op, shs=sh, scales=sc, rotations=q, sh_degree=0,
               viewmatrix=cam.world_view_transform.numpy(), projmatrix=cam.full_proj_transform.numpy(), campos=cam.camera_center.numpy(),
               bg=np.zeros(3, np.float32), image_height=512, image_width=512, tanfovx=math.tan(cam.FoVx / 2), tanfovy=math.tan(cam.FoVy / 2),
               scale_modifier=1.0)
    o_out, o_st, gimg, o_grads = _oracle(inp, 9)
    assert o_st["num_rendered"] > 20000 and (o_out[1] > 0).all()
    _check_forward_state(inp, o_out, o_st)
    _check_backward(inp, o_out, gimg, o_grads)
    _check_backward_sums(inp, gimg, o_grads)


def test_render_views_feeds_reference_optimizer_hook():
    """INTEGRATION.md section 3: render_views' `viewspace_point_list` must let the reference's on_before_optimizer_step
    (threestudio/systems/GaussianDreamer.py:385-391) run unchanged, and give what the per-view loop (:244-256) gives."""
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import PipelineParams, render, render_views
    from humangaussian_b200.scene import synthetic_body
    H = W = 96
    cams = sample_orbit_cameras(4, H, W, seed=3, device=DEV)
    bg = torch.zeros(3, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(0)
    wts = torch.randn(4, 3, H, W, device=DEV, generator=g)

    def fresh():
        p = synthetic_body(3000, sh_degree=1, seed=2)
        p.scaling += math.log(5.0)
        p = p.to(DEV)
        for t in (p.xyz, p.features_dc, p.features_rest, p.scaling, p.rotation, p.opacity):
            t.requires_grad_(True)
        return p

    # the reference's loop (:244-256) ...
    pa = fresh()
    vlist, radii, loss = [], None, 0
    for i, cam in enumerate(cams):
        pkg = render(cam, pa, PipelineParams(), bg)
        vlist.append(pkg["viewspace_points"])
        radii = pkg["radii"] if radii is None else torch.max(pkg["radii"], radii)
        loss = loss + (pkg["render"] * wts[i]).sum() + pkg["depth_3dgs"].sum()
    loss.backward()
    # ... and its hook body (:385-387), verbatim
    grad_ref = torch.zeros_like(vlist[0])
    for idx in range(len(vlist)):
        grad_ref = grad_ref + vlist[idx].grad
    # the batched wiring
    pb = fresh()
    pkg = render_views(cams, pb, bg)
    viewspace_point_list = pkg["viewspace_point_list"]
    ((pkg["render"] * wts).sum() + pkg["depth_3dgs"].sum()).backward()
    viewspace_point_tensor_grad = torch.zeros_like(viewspace_point_list[0])
    for idx in range(len(viewspace_point_list)):
        viewspace_point_tensor_grad = viewspace_point_tensor_grad + viewspace_point_list[idx].grad
    assert viewspace_point_tensor_grad.shape == (3000, 3)
    # two float32 evaluations with atomics in different orders: the gradient criterion (row-wise strict), not bit equality
    ok, msg = grads_agree(viewspace_point_tensor_grad.cpu().numpy(), grad_ref.cpu().numpy())
    assert ok, msg
    assert torch.equal(pkg["radii"].max(0).values, radii)
    ok, msg = grads_agree(pkg["viewspace_points"].grad.sum(0).cpu().numpy(), viewspace_point_tensor_grad.cpu().numpy())
    assert ok, msg
    ok, msg = grads_agree(pb.xyz.grad.cpu().numpy(), pa.xyz.grad.cpu().numpy())
    assert ok, msg


@pytest.mark.parametrize("deg", [0, 3])
def test_fused_raw_activations_match_torch_activations_and_autograd(deg):
    """SURVEY.md 8f-1: raw=True applies exp / F.normalize / sigmoid (gaussian_model.py:95-118) inside F1 and their Jacobians
    (incl. normalize's, which the reference gets from autograd) inside B3.  Against torch activations + autograd through
    the classic entry: images to the north-star tolerance, gradients w.r.t. the RAW tensors by the gradient criterion."""
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.rasterizer import packed_layout, rasterize_views, rasterize_views_packed
    from humangaussian_b200.renderer import stack_cameras
    from humangaussian_b200.scene import synthetic_body
    P, H, W, V = 1500, 72, 104, 3
    K = (deg + 1) ** 2
    p = synthetic_body(P, sh_degree=deg, seed=21)
    p.scaling += math.log(6.0)
    p.opacity += 1.5
    p = p.to(DEV)
    cams = sample_orbit_cameras(V, H, W, seed=2, device=DEV)
    vm, pm, cp, tanx, tany = stack_cameras(cams, DEV)
    bg = torch.tensor([0.1, 0.4, 0.7], device=DEV)
    rng = np.random.RandomState(1)
    gw = [torch.tensor(rng.randn(V, c, H, W).astype(np.float32), device=DEV) for c in (3, 1, 1)]
    kw = dict(viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tanx, tanfovy=tany, image_height=H, image_width=W, bg=bg, sh_degree=deg)
    # reference chain: torch activations (the getters) + autograd
    raw = {k: getattr(p, k).clone().requires_grad_(True) for k in ("xyz", "scaling", "rotation", "opacity", "features_dc", "features_rest")}
    sh = torch.cat((raw["features_dc"], raw["features_rest"]), dim=1)
    c0, r0, d0, a0 = rasterize_views(means3D=raw["xyz"], opacities=torch.sigmoid(raw["opacity"]), shs=sh, scales=torch.exp(raw["scaling"]),
                                     rotations=torch.nn.functional.normalize(raw["rotation"]), **kw)
    ((c0 * gw[0]).sum() + (d0 * gw[1]).sum() + (a0 * gw[2]).sum()).backward()
    # fused: raw tensors straight in (unpacked entry) ...
    raw2 = {k: getattr(p, k).clone().requires_grad_(True) for k in raw}
    sh2 = torch.cat((raw2["features_dc"], raw2["features_rest"]), dim=1)
    c1, r1, d1, a1 = rasterize_views(means3D=raw2["xyz"], opacities=raw2["opacity"], shs=sh2, scales=raw2["scaling"], rotations=raw2["rotation"],
                                     raw=True, **kw)
    ((c1 * gw[0]).sum() + (d1 * gw[1]).sum() + (a1 * gw[2]).sum()).backward()
    assert torch.equal(r0, r1)
    for x, y in ((c0, c1), (d0, d1), (a0, a1)):
        ok, worst = close(y.detach().cpu().numpy(), x.detach().cpu().numpy())
        assert ok, f"fused-activation image differs ({worst:.2f}x tolerance)"
    for k in raw:
        ok, msg = grads_agree(raw2[k].grad.cpu().numpy(), raw[k].grad.cpu().numpy())
        assert ok, f"raw dL/d{k}: {msg}"
    # ... and through the packed entry: flat.grad IS the raw-parameter gradient
    fields, n = packed_layout(P, K)
    flat = torch.zeros(n, device=DEV)
    with torch.no_grad():
        for (o, m, _), t in zip(fields, (p.xyz, p.scaling, p.rotation, p.opacity, torch.cat((p.features_dc, p.features_rest), 1))):
            flat.narrow(0, o, m).copy_(t.reshape(-1))
    flat.requires_grad_(True)
    c2, r2, d2, a2 = rasterize_views_packed(flat, P, K, raw=True, **kw)
    ((c2 * gw[0]).sum() + (d2 * gw[1]).sum() + (a2 * gw[2]).sum()).backward()
    assert torch.equal(c2, c1) and torch.equal(d2, d1) and torch.equal(a2, a1)
    ref = [raw["xyz"].grad, raw["scaling"].grad, raw["rotation"].grad, raw["opacity"].grad,
           torch.cat((raw["features_dc"].grad, raw["features_rest"].grad), 1)]
    for (o, m, shape), g in zip(fields, ref):
        ok, msg = grads_agree(flat.grad.narrow(0, o, m).view(shape).cpu().numpy().reshape(P, -1), g.cpu().numpy().reshape(P, -1))
        assert ok, f"packed raw gradient field at {o}: {msg}"


def test_render_fused_activation_option_matches_the_getter_path():
    """renderer.render(fused_activations=True): raw tensors into the kernels instead of the getters' torch kernels; same
    dict, images to tolerance, gradients at the raw tensors by the gradient criterion (incl. the means2D sink)."""
    from humangaussian_b200.cameras import Camera, orbit_c2w
    from humangaussian_b200.renderer import PipelineParams, render
    from humangaussian_b200.scene import synthetic_body
    cam = Camera(orbit_c2w(10, 30, 1.8), math.radians(60), 96, 128, device=DEV)
    outs = []
    for fused in (False, True):
        p = synthetic_body(4000, sh_degree=2, seed=5)
        p.scaling += math.log(5.0)
        p = p.to(DEV)
        leaves = (p.xyz, p.features_dc, p.features_rest, p.scaling, p.rotation, p.opacity)
        for t in leaves:
            t.requires_grad_(True)
        out = render(cam, p, PipelineParams(), torch.tensor([0.2, 0.1, 0.3], device=DEV), fused_activations=fused)
        (out["render"].square().sum() + out["depth_3dgs"].sum() + out["alpha_3dgs"].sum()).backward()
        outs.append((out, [t.grad for t in leaves]))
    (a, ga), (b, gb) = outs
    assert set(a) == set(b) and torch.equal(a["radii"], b["radii"])
    for k in ("render", "depth_3dgs", "alpha_3dgs"):
        ok, worst = close(b[k].detach().cpu().numpy(), a[k].detach().cpu().numpy())
        assert ok, (k, worst)
    for x, y in zip(ga, gb):
        ok, msg = grads_agree(y.cpu().numpy().reshape(4000, -1), x.cpu().numpy().reshape(4000, -1))
        assert ok, msg
    ok, msg = grads_agree(b["viewspace_points"].grad.cpu().numpy(), a["viewspace_points"].grad.cpu().numpy())
    assert ok, msg
