"""PackedAdam (csrc/optim.cu) against the reference's optimiser -- torch.optim.Adam(l, lr=0.0, eps=1e-15) over six
single-tensor groups (gaussian_model.py:156-165) -- and the packed densify / prune against the reference's outputs.

Per-step bound, u = 2^-24 (one fp32 rounding).  Each foreach op of torch's Adam stores an fp32 result, and the kernel
states the same ops with explicit roundings; where the two may still differ (e.g. an fma contracted on one side only),
each op differs by at most one rounding of its result:
    m = lerp(m0, g, 1-b1)           two roundings of terms bounded by |m0|+|g|        ->  |dm| <= 2u (|m0| + |g|)
    v = v0*b2 + (1-b2)*g*g          three roundings of terms bounded by v0+g^2        ->  |dv| <= 3u (v0 + g^2)
    U = s * m / (sqrt(v)/c + eps)   relative: 2u (m) + 1.5u (v through sqrt) + u (sqrt) + u (/c) + u (+eps) + u (m/d)
                                    = 7.5u <= 8u of |U|, and the final p + U rounds once -> |dp| <= u|p| + 8u|U|
with U torch's update (p_torch - p0) and p torch's new parameter.  The bound was written before the first GPU run.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
DEV = "cuda:0"
REF_LRS = dict(xyz=0.00005, f_dc=0.0125, f_rest=0.0125 / 20.0, opacity=0.01, scaling=0.005, rotation=0.001)  # arguments/__init__.py:73-80
GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def pack_groups(t):
    """six reference tensors -> the flat layout (dist.pack: SH = cat(f_dc, f_rest))"""
    from humangaussian_b200 import dist as D
    return D.pack(dict(xyz=t["xyz"], scaling=t["scaling"], rotation=t["rotation"], opacity=t["opacity"],
                       features=torch.cat((t["f_dc"], t["f_rest"]), 1)))


def unpack_groups(flat, P, K):
    from humangaussian_b200 import dist as D
    v = D.unpack(flat, P, K)
    return dict(xyz=v["xyz"], f_dc=v["features"][:, :1], f_rest=v["features"][:, 1:], opacity=v["opacity"], scaling=v["scaling"],
                rotation=v["rotation"])


def random_groups(P, K, gen, scale=1.0):
    f = lambda *s: torch.randn(*s, device=DEV, generator=gen) * scale
    return dict(xyz=f(P, 3) * 0.4, f_dc=f(P, 1, 3), f_rest=f(P, K - 1, 3) * 0.1, opacity=f(P, 1) - 1.0, scaling=f(P, 3) - 4.0,
                rotation=f(P, 4))


def random_grads(P, K, gen):
    g = {k: v * 1e-3 for k, v in random_groups(P, K, gen).items()}
    for k in g:  # a few exact zeros and a spread of magnitudes
        mask = torch.rand(g[k].shape, device=DEV, generator=gen)
        g[k] = torch.where(mask < 0.05, torch.zeros_like(g[k]), g[k] * torch.exp(4 * (mask - 0.5)))
    return g


class Pair:
    """The reference's six-tensor Adam and a PackedAdam on the same values, moments and step count."""

    def __init__(self, P, K, step0, seed, lrs=REF_LRS, scheduler=None):
        from humangaussian_b200.optim import PackedAdam
        gen = torch.Generator(device=DEV).manual_seed(seed)
        self.P, self.K = P, K
        vals = random_groups(P, K, gen)
        m0 = {k: torch.randn(v.shape, device=DEV, generator=gen) * 1e-3 for k, v in vals.items()}
        v0 = {k: torch.rand(v.shape, device=DEV, generator=gen) * 1e-6 for k, v in vals.items()}
        self.ref = {k: torch.nn.Parameter(vals[k].clone()) for k in GROUPS}
        self.ref_opt = torch.optim.Adam([{"params": [self.ref[k]], "lr": lrs[k], "name": k} for k in GROUPS], lr=0.0, eps=1e-15)
        self.packed = pack_groups(vals).requires_grad_(True)
        self.opt = PackedAdam(self.packed, P, K, lrs, xyz_scheduler=scheduler)
        for k in GROUPS:  # non-trivial moments, also before step 1
            self.ref_opt.state[self.ref[k]] = {"step": torch.tensor(float(step0)), "exp_avg": m0[k].clone(), "exp_avg_sq": v0[k].clone()}
        self.opt.state[self.packed] = {"step": torch.tensor(float(step0)), "exp_avg": pack_groups(m0), "exp_avg_sq": pack_groups(v0)}

    def step(self, grads):
        for k in GROUPS:
            self.ref[k].grad = grads[k].clone()
        self.opt.packed.grad = pack_groups(grads)
        self.ref_opt.step()
        self.opt.step()

    def packed_groups(self, what):
        st = self.opt.state[self.opt.packed]
        flat = {"p": self.opt.packed.detach(), "m": st["exp_avg"], "v": st["exp_avg_sq"]}[what]
        return unpack_groups(flat, self.opt.P, self.K)

    def ref_groups(self, what):
        if what == "p":
            return {k: self.ref[k].detach() for k in GROUPS}
        return {k: self.ref_opt.state[self.ref[k]]["exp_avg" if what == "m" else "exp_avg_sq"] for k in GROUPS}


def padding_mask(P, K):
    from humangaussian_b200.rasterizer import packed_layout
    fields, total = packed_layout(P, K)
    pad = torch.ones(total, dtype=torch.bool, device=DEV)
    for o, n, _ in fields:
        pad[o:o + n] = False
    return pad


@pytest.mark.parametrize("step", [1, 2, 1000])
@pytest.mark.parametrize("K", [1, 16])
@pytest.mark.parametrize("P", [1, 5, 4099, 300_000])
def test_single_step_matches_torch_adam(P, K, step):
    pair = Pair(P, K, step - 1, seed=P + 7 * K + step)
    gen = torch.Generator(device=DEV).manual_seed(11 * P + K)
    g = random_grads(P, K, gen)
    p0 = {k: v.detach().clone().double() for k, v in pair.ref.items()}
    m0 = {k: v.clone().double() for k, v in pair.ref_groups("m").items()}
    v0 = {k: v.clone().double() for k, v in pair.ref_groups("v").items()}
    pair.step(g)
    assert float(pair.opt.state[pair.opt.packed]["step"]) == step
    rp, rm, rv = (pair.ref_groups(w) for w in "pmv")
    qp, qm, qv = (pair.packed_groups(w) for w in "pmv")
    bit_identical = True
    for k in GROUPS:
        gd = g[k].double()
        dm = (qm[k].double() - rm[k].double()).abs()
        dv = (qv[k].double() - rv[k].double()).abs()
        dp = (qp[k].double() - rp[k].double()).abs()
        Uk = rp[k].double() - p0[k]
        assert bool((dm <= 2 * U32 * (m0[k].abs() + gd.abs())).all()), (k, float(dm.max()))
        assert bool((dv <= 3 * U32 * (v0[k] + gd * gd)).all()), (k, float(dv.max()))
        assert bool((dp <= U32 * rp[k].double().abs() + 8 * U32 * Uk.abs()).all()), (k, float(dp.max()))
        bit_identical &= all(torch.equal(a, b) for a, b in ((qp[k], rp[k]), (qm[k], rm[k]), (qv[k], rv[k])))
    pad = padding_mask(P, K)
    st = pair.opt.state[pair.opt.packed]
    for t in (pair.opt.packed.detach(), st["exp_avg"], st["exp_avg_sq"]):
        assert int(torch.count_nonzero(t[pad])) == 0
    print(f"P={P} K={K} step={step}: bit-identical to torch.optim.Adam (foreach): {bit_identical}")


def test_trajectory_follows_torch_adam_with_the_xyz_schedule():
    from humangaussian_b200.optim import expon_lr_func
    P, K, T = 4099, 16, 200
    sched = expon_lr_func(lr_init=0.00016, lr_final=0.0000016, lr_delay_steps=50, lr_delay_mult=0.01, max_steps=300)
    pair = Pair(P, K, 0, seed=3, scheduler=sched)
    gen = torch.Generator(device=DEV).manual_seed(5)
    worst = {k: torch.zeros_like(v, dtype=torch.float64) for k, v in pair.ref.items()}  # max over steps of the per-step bound
    for it in range(T):
        lr = pair.opt.update_learning_rate(it)
        for grp in pair.ref_opt.param_groups:  # GaussianModel.update_learning_rate
            if grp["name"] == "xyz":
                grp["lr"] = sched(it)
        assert pair.opt.param_groups[0]["lrs"]["xyz"] == lr == sched(it)
        before = {k: v.detach().double().clone() for k, v in pair.ref.items()}
        pair.step(random_grads(P, K, gen))
        for k in GROUPS:
            p = pair.ref[k].detach().double()
            worst[k] = torch.maximum(worst[k], U32 * p.abs() + 8 * U32 * (p - before[k]).abs())
    qp = pair.packed_groups("p")
    for k in GROUPS:
        dp = (qp[k].double() - pair.ref[k].detach().double()).abs()
        assert bool((dp <= 200 * worst[k]).all()), (k, float(dp.max()))
    pad = padding_mask(P, K)
    st = pair.opt.state[pair.opt.packed]
    for t in (pair.opt.packed.detach(), st["exp_avg"], st["exp_avg_sq"]):
        assert int(torch.count_nonzero(t[pad])) == 0


def test_two_runs_from_identical_state_are_bit_identical():
    runs = []
    for _ in range(2):
        pair = Pair(300_001, 16, 10, seed=42)
        gen = torch.Generator(device=DEV).manual_seed(9)
        for _ in range(5):
            g = random_grads(300_001, 16, gen)
            pair.opt.packed.grad = pack_groups(g)
            pair.opt.step()
        st = pair.opt.state[pair.opt.packed]
        runs.append((pair.opt.packed.detach().clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_grad_scaler_unscales_and_skips_inf_steps():
    P, K = 4099, 16
    a, b = Pair(P, K, 3, seed=1), Pair(P, K, 3, seed=1)
    g = random_grads(P, K, torch.Generator(device=DEV).manual_seed(2))
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12)
    scaler.scale(torch.ones((), device=DEV))  # what scaler.scale(loss) does first: the scale tensor lives on the device
    a.opt.packed.grad = pack_groups(g) * scaler.get_scale()   # what backward of scaler.scale(loss) produces
    scaler.step(a.opt)
    scaler.update()
    b.opt.packed.grad = pack_groups(g)
    b.opt.step()
    sa, sb = a.opt.state[a.opt.packed], b.opt.state[b.opt.packed]
    assert torch.equal(a.opt.packed, b.opt.packed) and torch.equal(sa["exp_avg"], sb["exp_avg"]) and torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"])
    assert float(sa["step"]) == 4
    # an inf in the scaled gradient: the step is skipped on the host, nothing moves
    before = (a.opt.packed.detach().clone(), sa["exp_avg"].clone(), sa["exp_avg_sq"].clone())
    grad = pack_groups(g) * scaler.get_scale()
    grad[17] = float("inf")
    a.opt.packed.grad = grad
    scale_before = scaler.get_scale()
    scaler.step(a.opt)
    scaler.update()
    assert torch.equal(a.opt.packed.detach(), before[0]) and torch.equal(sa["exp_avg"], before[1]) and torch.equal(sa["exp_avg_sq"], before[2])
    assert float(sa["step"]) == 4 and scaler.get_scale() < scale_before


def test_state_dict_round_trip():
    from humangaussian_b200.optim import PackedAdam
    pair = Pair(257, 4, 0, seed=8)
    pair.step(random_grads(257, 4, torch.Generator(device=DEV).manual_seed(1)))
    sd = pair.opt.state_dict()
    fresh = PackedAdam(pair.opt.packed, 257, 4, {k: 0.0 for k in GROUPS})
    fresh.load_state_dict(sd)
    st0, st1 = pair.opt.state[pair.opt.packed], fresh.state[fresh.packed]
    assert fresh.param_groups[0]["lrs"] == REF_LRS and float(st1["step"]) == 1
    assert torch.equal(st0["exp_avg"], st1["exp_avg"]) and torch.equal(st0["exp_avg_sq"], st1["exp_avg_sq"])


# ---- densify / prune in the flat layout ----------------------------------------------------------------------------
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_densify.npz"))
RTOL, ATOL = 2e-6, 1e-7  # as test_gpu_densify.py


def golden_packed(tag):
    """a PackedAdam holding a golden state (params, both moments; the golden states took two Adam steps) + its stats"""
    from humangaussian_b200.densify import DensifyStats
    from humangaussian_b200.optim import PackedAdam
    t = lambda k: torch.from_numpy(np.ascontiguousarray(GOLD[f"{tag}_in_{k}"])).to(DEV)
    params = {g: t(g) for g in GROUPS}
    P, K = params["xyz"].shape[0], 1 + params["f_rest"].shape[1]
    opt = PackedAdam(pack_groups(params).requires_grad_(True), P, K, REF_LRS)
    opt.state[opt.packed] = {"step": torch.tensor(2.0), "exp_avg": pack_groups({g: t("m_" + g) for g in GROUPS}),
                             "exp_avg_sq": pack_groups({g: t("v_" + g) for g in GROUPS})}
    stats = DensifyStats(t("accum"), t("denom"), t("max_radii2D"))
    moments = {g: (t("m_" + g), t("v_" + g)) for g in GROUPS}
    return opt, stats, params, moments


def check_against(opt, stats, want, rtol, atol, exact=False):
    P, K = opt.P, opt.sh_coeffs
    st = opt.state[opt.packed]
    got = dict(unpack_groups(opt.packed.detach(), P, K))
    for pre, flat in (("m_", st["exp_avg"]), ("v_", st["exp_avg_sq"])):
        got.update({pre + k: v for k, v in unpack_groups(flat, P, K).items()})
    got.update(accum=stats.xyz_gradient_accum, denom=stats.denom, max_radii2D=stats.max_radii2D)
    for k, w in want.items():
        g = got[k].cpu().numpy()
        assert g.shape == w.shape, (k, g.shape, w.shape)
        if exact:
            np.testing.assert_array_equal(g, w, err_msg=k)
        else:
            np.testing.assert_allclose(g, w, rtol=rtol, atol=atol, err_msg=k)
    pad = padding_mask(P, K)
    for t in (opt.packed.detach(), st["exp_avg"], st["exp_avg_sq"]):
        assert int(torch.count_nonzero(t[pad])) == 0


def golden_out(tag):
    keys = [pre + g for g in GROUPS for pre in ("", "m_", "v_")] + ["accum", "denom", "max_radii2D"]
    return {k: GOLD[f"{tag}_out_{k}"] for k in keys}


@pytest.mark.parametrize("tag", ["dp_noscreen", "dp_screen", "dp_deg0"])
def test_densify_and_prune_packed_matches_reference_and_the_group_form(tag):
    from humangaussian_b200.densify import DensifyStats, densify_and_prune, densify_and_prune_packed
    max_grad, min_opacity, extent, screen, pd = GOLD[tag + "_args"]
    noise = torch.from_numpy(GOLD[tag + "_noise"])
    opt, stats, params, moments = golden_packed(tag)
    ref_stats = DensifyStats(stats.xyz_gradient_accum, stats.denom, stats.max_radii2D)
    old_leaf = opt.packed
    P_new = densify_and_prune_packed(opt, stats, max_grad, min_opacity, extent, None if screen < 0 else screen, pd, noise=noise)
    want = golden_out(tag)
    assert P_new == opt.P == want["xyz"].shape[0] and opt.packed is not old_leaf and opt.packed.requires_grad
    assert float(opt.state[opt.packed]["step"]) == 2 and old_leaf not in opt.state
    check_against(opt, stats, want, RTOL, ATOL)
    # bit for bit the per-group surgery followed by dist.pack
    p, m, s = densify_and_prune(params, moments, ref_stats, max_grad, min_opacity, extent, None if screen < 0 else screen, pd, noise=noise)
    st = opt.state[opt.packed]
    assert torch.equal(opt.packed.detach(), pack_groups(p))
    assert torch.equal(st["exp_avg"], pack_groups({g: m[g][0] for g in GROUPS}))
    assert torch.equal(st["exp_avg_sq"], pack_groups({g: m[g][1] for g in GROUPS}))
    assert torch.equal(stats.denom, s.denom) and torch.equal(stats.xyz_gradient_accum, s.xyz_gradient_accum)


def test_prune_only_packed_matches_reference_and_the_group_form():
    from humangaussian_b200.densify import DensifyStats, prune_only, prune_only_packed
    min_opacity, size_thresh = GOLD["po_args"]
    opt, stats, params, moments = golden_packed("po")
    ref_stats = DensifyStats(stats.xyz_gradient_accum, stats.denom, stats.max_radii2D)
    P_new = prune_only_packed(opt, stats, min_opacity, size_thresh)
    want = golden_out("po")
    assert P_new == want["xyz"].shape[0]
    check_against(opt, stats, want, 0, 0, exact=True)
    p, m, s = prune_only(params, moments, ref_stats, min_opacity, size_thresh)
    st = opt.state[opt.packed]
    assert torch.equal(opt.packed.detach(), pack_groups(p))
    assert torch.equal(st["exp_avg"], pack_groups({g: m[g][0] for g in GROUPS}))
    assert torch.equal(st["exp_avg_sq"], pack_groups({g: m[g][1] for g in GROUPS}))
    assert torch.equal(stats.max_radii2D, s.max_radii2D)


# ---- end to end ----------------------------------------------------------------------------------------------------
def test_training_loop_on_the_flat_buffer():
    """20 steps of rasterize_views_packed(raw=True) -> loss -> backward -> add_densification_stats -> PackedAdam.step, with
    one densify after step 10; a reference-style six-tensor Adam is fed the same gradients (and densified with the same
    plan inputs and noise) and the parameters must stay within check 2's bound."""
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.densify import (DensifyStats, add_densification_stats, densify_and_prune, densify_and_prune_packed,
                                            install_into_optimizer, moments_from_optimizer)
    from humangaussian_b200.optim import PackedAdam, expon_lr_func
    from humangaussian_b200.rasterizer import rasterize_views_packed
    from humangaussian_b200.renderer import stack_cameras
    from util import small_scene
    _, _, sc = small_scene(P=3001, deg=3, seed=4)
    K, H = 16, 64
    vals = dict(xyz=sc.xyz, f_dc=sc.features_dc, f_rest=sc.features_rest, opacity=sc.opacity, scaling=sc.scaling, rotation=sc.rotation)
    vals = {k: v.detach().float().to(DEV).contiguous() for k, v in vals.items()}
    lrs = dict(REF_LRS, xyz=0.00016)
    sched = expon_lr_func(lr_init=0.00016, lr_final=0.0000016, lr_delay_mult=0.01, max_steps=30000)
    opt = PackedAdam(pack_groups(vals).requires_grad_(True), vals["xyz"].shape[0], K, lrs, xyz_scheduler=sched)
    ref = {k: torch.nn.Parameter(v.clone()) for k, v in vals.items()}
    ref_opt = torch.optim.Adam([{"params": [ref[k]], "lr": lrs[k], "name": k} for k in GROUPS], lr=0.0, eps=1e-15)
    vm, pm, cp, tx, ty = stack_cameras(sample_orbit_cameras(4, H, H, seed=3), DEV)
    bg = torch.tensor([0.8, 0.5, 0.2], device=DEV)
    target = bg.view(1, 3, 1, 1)  # a plain backdrop: the loss is the Gaussians' coverage and colour error
    stats = DensifyStats.zeros(opt.P, DEV)
    losses, umax = [], {k: 0.0 for k in GROUPS}
    for it in range(20):
        opt.update_learning_rate(it)
        ref_opt.param_groups[0]["lr"] = sched(it)
        m2d = torch.zeros(4, opt.P, 3, device=DEV, requires_grad=True)
        color, radii, _, _ = rasterize_views_packed(opt.packed, opt.P, K, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx,
                                                    tanfovy=ty, image_height=H, image_width=H, bg=bg, sh_degree=3, means2D=m2d, raw=True)
        loss = (color - target).square().mean()
        loss.backward()
        losses.append(float(loss.detach()))
        add_densification_stats(stats, m2d.grad, radii)
        grads = unpack_groups(opt.packed.grad, opt.P, K)
        before = {k: v.detach().double().clone() for k, v in ref.items()}
        for k in GROUPS:
            ref[k].grad = grads[k].clone()
        ref_opt.step()
        opt.step()
        opt.zero_grad()
        for k in GROUPS:
            umax[k] = max(umax[k], float((ref[k].detach().double() - before[k]).abs().max()))
        if it == 9:
            thr = float(torch.quantile((stats.xyz_gradient_accum / stats.denom.clamp_min(1)).flatten(), 0.8))
            ref_stats = DensifyStats(stats.xyz_gradient_accum, stats.denom, stats.max_radii2D)
            P_new = densify_and_prune_packed(opt, stats, thr, 0.005, 1.0, None, generator=torch.Generator(device=DEV).manual_seed(7))
            p, m, _ = densify_and_prune({k: ref[k].data for k in GROUPS}, moments_from_optimizer(ref_opt), ref_stats, thr, 0.005, 1.0,
                                        None, generator=torch.Generator(device=DEV).manual_seed(7))
            ref = install_into_optimizer(ref_opt, p, m)
            assert P_new == ref["xyz"].shape[0] and P_new != 3001
    assert losses[-1] < losses[0], losses
    got = unpack_groups(opt.packed.detach(), opt.P, K)
    for k in GROUPS:
        p = ref[k].detach().double()
        dp = (got[k].double() - p).abs()
        assert bool((dp <= 200 * (U32 * p.abs() + 8 * U32 * umax[k])).all()), (k, float(dp.max()))
    assert float(opt.state[opt.packed]["step"]) == 20
