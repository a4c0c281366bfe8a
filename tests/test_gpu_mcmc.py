"""GPU: MCMC densification (humangaussian_b200/mcmc.py, csrc/mcmc.cu) against the float64 reference
(tests/mcmc_reference.py): the split ratio to 1 float32 ulp, relocation and growth with given samples row by row, the
position noise, the dict forms against the packed ones, and a packed training loop with all three."""
import copy
import math
import warnings

import numpy as np
import pytest
import torch

import mcmc_reference as M
from util import small_scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LRS = dict(xyz=0.00016, f_dc=0.0125, f_rest=0.0125 / 20.0, opacity=0.05, scaling=0.005, rotation=0.001)


def _ulps(got32, want64):
    """float32 ulp distance between the kernel's values and the float64 reference rounded to float32"""
    a = np.asarray(got32, np.float32).view(np.int32).astype(np.int64)
    b = np.asarray(want64, np.float64).astype(np.float32).view(np.int32).astype(np.int64)
    a = np.where(a < 0, np.int64(-2 ** 31) - a, a)  # sign-magnitude -> monotone integers
    b = np.where(b < 0, np.int64(-2 ** 31) - b, b)
    return np.abs(a - b)


def _scene(P, K=16, seed=0, dead=0.15):
    """raw packed fields of a seeded scene; a `dead` share of rows gets opacity logit -8 (sigmoid 3e-4), row 1 a NaN"""
    _, _, sc = small_scene(P=P, deg=int(math.isqrt(K)) - 1, seed=seed)
    g = torch.Generator().manual_seed(seed)
    op = sc.opacity.detach().float().clone()
    op[torch.rand(P, generator=g) < dead] = -8.0
    op[1] = float("nan")
    return dict(xyz=sc.xyz.detach().float(), scaling=sc.scaling.detach().float(), rotation=sc.rotation.detach().float() * 1.7,
                opacity=op, features=torch.cat((sc.features_dc, sc.features_rest), 1).detach().float())


def _optimizer(raw, K=16, steps=1):
    """PackedAdam over the packed scene, with `steps` steps of a random gradient so that the moments are non-zero"""
    from humangaussian_b200 import dist as D
    from humangaussian_b200.optim import PackedAdam
    flat = D.pack({k: v.to(DEV).contiguous() for k, v in raw.items()}).requires_grad_(True)
    opt = PackedAdam(flat, raw["xyz"].shape[0], K, LRS)
    g = torch.Generator(device=DEV).manual_seed(9)
    for _ in range(steps):
        opt.packed.grad = torch.randn(opt.packed.shape, device=DEV, generator=g) * 1e-3
        opt.step()
    opt.zero_grad()
    return opt


def _fields(flat, P, K):
    from humangaussian_b200 import dist as D
    return D.unpack(flat.detach(), P, K)


def _padding(flat, P, K):
    from humangaussian_b200.rasterizer import packed_layout
    fields, total = packed_layout(P, K)
    mask = torch.ones(total, dtype=torch.bool, device=flat.device)
    for o, n, _ in fields:
        mask[o:o + n] = False
    return flat.detach()[mask]


def _snapshot(opt):
    st = opt.state[opt.packed]
    return opt.P, opt.packed.detach().clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone(), float(st["step"])


def _check_surgery(before, after, K, mapping, counts):
    """row i of the result is source row mapping[i]; rows whose source was drawn (counts > 0) take the ratio's opacity and
    scales (1 ulp) and zero moments; xyz, rotation, SH of every row and every field of other rows are byte-exact copies"""
    P0, flat0, m0, v0, step0 = before
    P1, flat1, m1, v1, step1 = after
    assert P1 == len(mapping) and step1 == step0
    mapping = np.asarray(mapping)
    reset = counts[mapping] > 0
    f0, f1 = _fields(flat0, P0, K), _fields(flat1, P1, K)
    for k in ("xyz", "rotation", "features"):
        assert np.array_equal(f1[k].cpu().numpy().view(np.int32), f0[k].cpu().numpy()[mapping].view(np.int32)), k
    for k in ("opacity", "scaling"):
        a, b = f1[k].cpu().numpy(), f0[k].cpu().numpy()[mapping]
        assert np.array_equal(a[~reset].view(np.int32), b[~reset].view(np.int32)), k
    o32 = torch.sigmoid(f0["opacity"].reshape(-1)).cpu().numpy()
    src = mapping[reset]
    logit, scale = M.new_raw(o32[src], f0["scaling"].cpu().numpy()[src], counts[src])
    assert _ulps(f1["opacity"].cpu().numpy()[reset, 0], logit).max() <= 1
    assert _ulps(f1["scaling"].cpu().numpy()[reset], scale).max() <= 1
    for mom0, mom1 in ((m0, m1), (v0, v1)):
        g0, g1 = _fields(mom0, P0, K), _fields(mom1, P1, K)
        for k in g1:
            a, b = g1[k].cpu().numpy(), g0[k].cpu().numpy()[mapping]
            assert np.array_equal(a[reset].view(np.int32), np.zeros_like(a[reset]).view(np.int32)), k
            assert np.array_equal(a[~reset].view(np.int32), b[~reset].view(np.int32)), k
        assert (_padding(mom1, P1, K) == 0).all()
    assert (_padding(flat1, P1, K) == 0).all()


def test_ratio_within_one_ulp_of_float64():
    from humangaussian_b200 import mcmc
    o_grid = [0.0051, 0.006, 0.01, 0.05, 0.1, 0.3, 0.5, 0.7, 0.9, 0.99, 0.999, 0.99999]
    logits = [math.log(o / (1 - o)) for o in o_grid] + [16.0, 20.0]  # sigmoid32: 1 - 2^-23 and 1
    cs = list(range(1, 51)) + [60, 1000]                             # n = 2..51, then saturated
    lg = torch.tensor([l for l in logits for _ in cs], dtype=torch.float32, device=DEV)
    c = np.array([c for _ in logits for c in cs], np.int64)
    P = lg.numel()
    scaling = (torch.rand(P, 3, generator=torch.Generator().manual_seed(0)) * 6.0 - 6.0).to(DEV)
    o32 = torch.sigmoid(lg).cpu().numpy()
    assert np.float32(1.0 - 2.0 ** -23) in o32 and np.float32(1.0) in o32
    samples = torch.repeat_interleave(torch.arange(P, device=DEV), torch.from_numpy(c).to(DEV))
    with torch.cuda.device(DEV):
        plan = mcmc._Plan(P, torch.arange(P, device=DEV), samples, lg, scaling)
    assert np.array_equal(plan.counts.cpu().numpy(), c)
    logit, scale = M.new_raw(o32, scaling.cpu().numpy(), c)
    assert _ulps(plan.new_opacity.cpu().numpy(), logit).max() <= 1
    assert _ulps(plan.new_scaling.cpu().numpy(), scale).max() <= 1


@pytest.mark.parametrize("P,K", [(3001, 16), (1000, 1)])
def test_relocate_with_given_samples(P, K):
    from humangaussian_b200.mcmc import relocate_packed
    opt = _optimizer(_scene(P, K, seed=P), K)
    before = _snapshot(opt)
    o = torch.sigmoid(_fields(before[1], P, K)["opacity"].reshape(-1))
    live = (o > 0.005).cpu().numpy()
    dead = np.flatnonzero(~live)
    assert 1 in dead and len(dead) > 50
    rng = np.random.default_rng(P)
    samples = rng.choice(np.flatnonzero(live), len(dead))
    samples[:30] = samples[0]  # one source drawn 30 times (n = 31)
    d = relocate_packed(opt, samples=torch.from_numpy(samples).to(DEV))
    assert d == len(dead) and opt.P == P
    mapping = np.arange(P)
    mapping[dead] = samples
    _check_surgery(before, _snapshot(opt), K, mapping, np.bincount(samples, minlength=P))


def test_relocate_without_dead_rows_is_a_no_op():
    from humangaussian_b200 import rasterizer as R
    from humangaussian_b200.mcmc import relocate_packed
    raw = _scene(1001, dead=0.0)
    raw["opacity"][1] = 0.0
    raw["opacity"].clamp_(min=-3.0)
    opt = _optimizer(raw)
    leaf, before = opt.packed, _snapshot(opt)
    n = R.launch_count()
    assert relocate_packed(opt, generator=torch.Generator(device=DEV).manual_seed(1)) == 0
    assert R.launch_count() == n and opt.packed is leaf
    after = _snapshot(opt)
    for a, b in zip(before[1:4], after[1:4]):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def test_relocate_errors():
    from humangaussian_b200.mcmc import relocate_packed
    raw = _scene(400)
    opt = _optimizer(raw)
    d = int((~(torch.sigmoid(raw["opacity"].reshape(-1)) > 0.005)).sum())
    with pytest.raises(ValueError, match="int64"):
        relocate_packed(opt, samples=torch.zeros(d + 1, dtype=torch.int64, device=DEV))
    with pytest.raises(ValueError, match="live"):
        relocate_packed(opt, samples=torch.ones(d, dtype=torch.int64, device=DEV))  # row 1 is NaN: dead
    with pytest.raises(ValueError, match="index rows"):
        relocate_packed(opt, samples=torch.full((d,), 400, dtype=torch.int64, device=DEV))
    raw["opacity"][:] = -9.0
    with pytest.raises(ValueError, match="no live"):
        relocate_packed(_optimizer(raw))


@pytest.mark.parametrize("P,cap", [(1001, 10 ** 6), (1001, 1020), (998, 1046)])
def test_grow_with_given_samples(P, cap):
    from humangaussian_b200.mcmc import add_packed
    from humangaussian_b200.optim import PackedAdam
    K = 16
    opt = _optimizer(_scene(P, K, seed=7), K, steps=3)
    before = _snapshot(opt)
    P_new = min(cap, math.floor(1.05 * P))
    live = (torch.sigmoid(_fields(before[1], P, K)["opacity"].reshape(-1)) > 0.005).cpu().numpy()
    samples = np.random.default_rng(3).choice(np.flatnonzero(live), P_new - P)
    assert add_packed(opt, cap, samples=torch.from_numpy(samples).to(DEV)) == P_new == opt.P
    _check_surgery(before, _snapshot(opt), K, np.concatenate([np.arange(P), samples]), np.bincount(samples, minlength=P))
    # state_dict round trip: a fresh optimiser on the grown buffer loads the layout, the step count and both moments
    twin = PackedAdam(torch.zeros_like(opt.packed).requires_grad_(True), P_new, K, LRS)
    twin.load_state_dict(copy.deepcopy(opt.state_dict()))
    assert twin.P == P_new and twin.sh_coeffs == K and float(twin.state[twin.packed]["step"]) == before[4]
    for k in ("exp_avg", "exp_avg_sq"):
        a, b = opt.state[opt.packed][k], twin.state[twin.packed][k]
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), k


def test_grow_to_budget_and_no_op():
    from humangaussian_b200.mcmc import add_packed
    opt = _optimizer(_scene(1001))
    leaf = opt.packed
    assert add_packed(opt, 1001) == 1001 and add_packed(opt, 500) == 1001 and opt.packed is leaf
    g = torch.Generator(device=DEV).manual_seed(4)
    xyz0 = _fields(opt.packed, 1001, 16)["xyz"].clone()
    live = torch.sigmoid(_fields(opt.packed, 1001, 16)["opacity"].reshape(-1)) > 0.005
    sizes = []
    while opt.P < 1200:
        sizes.append(add_packed(opt, 1200, generator=g))
    assert sizes == [1051, 1103, 1158, 1200]
    # the drawn sources are live rows: every appended row's xyz is a live row's (xyz is copied bit for bit)
    xyz = _fields(opt.packed, 1200, 16)["xyz"]
    src = (xyz[1001:1051, None, :] == xyz0[None]).all(-1)
    assert (src.sum(1) >= 1).all() and live[src.float().argmax(1)].all()


def _noise_scene(P, seed=5):
    raw = _scene(P, seed=seed, dead=0.3)
    raw["opacity"][1] = -3.0
    raw["opacity"] = raw["opacity"] + torch.rand(P, 1, generator=torch.Generator().manual_seed(seed)) * 4.0 - 2.0
    return raw


def test_noise_matches_reference():
    from humangaussian_b200 import dist as D
    from humangaussian_b200.mcmc import inject_noise, inject_noise_packed
    P, K = 20001, 16
    raw = _noise_scene(P)
    eta = torch.randn(P, 3, generator=torch.Generator().manual_seed(1)).to(DEV)
    lr, scale = 1.6e-4, 5e5 * 1.6e-4
    o32 = torch.sigmoid(raw["opacity"].to(DEV).reshape(-1)).cpu().numpy()
    ref = M.noise_delta(raw["scaling"].numpy(), raw["rotation"].numpy(), o32, eta.cpu().numpy(), scale)
    # the row's largest possible step, scale * lambda_max(Sigma) * ||eta||, ungated and gated
    ungated = scale * np.exp(2.0 * raw["scaling"].numpy().astype(np.float64).max(1)) * np.linalg.norm(eta.cpu().numpy(), axis=1)
    bound = M.gate(o32) * ungated
    # tolerance: 1e-5 of the gated step, and 1e-29 of the ungated one, below which float32 cannot hold the gate
    # (sigmoid(opacity) > ~0.7 puts it under 1e-30, denormal or zero)
    tol = 1e-5 * bound + 1e-29 * ungated
    # from xyz = 0 the result is the step itself
    params = dict(xyz=torch.zeros(P, 3, device=DEV), scaling=raw["scaling"].to(DEV), rotation=raw["rotation"].to(DEV),
                  opacity=raw["opacity"].to(DEV))
    inject_noise(params, lr, eta=eta)
    err = np.abs(params["xyz"].cpu().numpy().astype(np.float64) - ref).max(1)
    assert (err <= tol).all(), float((err / tol).max())
    assert (np.abs(ref).max(1) > 1e-3 * bound).mean() > 0.5 and (bound > 1e-4 * ungated).mean() > 0.3  # not vacuous
    # the packed form on the real positions: xyz + step, rounded once; every other float untouched
    opt = _optimizer(raw, K, steps=0)  # lrs["xyz"] == lr; no step, so the fields are the reference's inputs
    flat0 = opt.packed.detach().clone()
    inject_noise_packed(opt, eta=eta)
    f0, f1 = _fields(flat0, P, K), _fields(opt.packed, P, K)
    want = f0["xyz"].cpu().numpy().astype(np.float64) + ref
    err = np.abs(f1["xyz"].cpu().numpy() - want).max(1)
    assert (err <= tol + 2.0 ** -24 * np.abs(want).max(1)).all()
    mask = torch.ones_like(flat0, dtype=torch.bool)
    mask[:3 * P] = False
    assert flat0[mask].cpu().numpy().tobytes() == opt.packed.detach()[mask].cpu().numpy().tobytes()
    # eta = 0 leaves the buffer byte-identical
    flat1 = opt.packed.detach().clone()
    inject_noise_packed(opt, eta=torch.zeros(P, 3, device=DEV))
    assert flat1.cpu().numpy().tobytes() == opt.packed.detach().cpu().numpy().tobytes()
    # the default draw is torch.randn with the caller's generator
    flat2 = opt.packed.detach().clone()
    inject_noise_packed(opt, generator=torch.Generator(device=DEV).manual_seed(3))
    inject_noise_packed(opt, eta=-torch.randn(P, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3)))
    assert torch.allclose(opt.packed.detach(), flat2, rtol=0, atol=1e-6)
    assert D.unpack(opt.packed.detach(), P, K)["xyz"].shape == (P, 3)


def test_noise_errors():
    from humangaussian_b200.mcmc import inject_noise_packed
    opt = _optimizer(_scene(100))
    for bad in (torch.zeros(100, 2, device=DEV), torch.zeros(100, 3, device=DEV, dtype=torch.float64), torch.zeros(100, 3)):
        with pytest.raises(ValueError):
            inject_noise_packed(opt, eta=bad)


def _dicts(opt, K):
    f = _fields(opt.packed, opt.P, K)
    st = opt.state[opt.packed]
    split = lambda d: dict(xyz=d["xyz"], f_dc=d["features"][:, :1], f_rest=d["features"][:, 1:], opacity=d["opacity"],
                           scaling=d["scaling"], rotation=d["rotation"])
    params = {k: v.clone() for k, v in split(f).items()}
    m, v = split(_fields(st["exp_avg"], opt.P, K)), split(_fields(st["exp_avg_sq"], opt.P, K))
    return params, {k: (m[k].clone(), v[k].clone()) for k in params}


def _pack(params):
    from humangaussian_b200 import dist as D
    return D.pack(dict(xyz=params["xyz"], scaling=params["scaling"], rotation=params["rotation"], opacity=params["opacity"],
                       features=torch.cat((params["f_dc"], params["f_rest"]), 1)))


def test_dict_forms_equal_packed_forms():
    from humangaussian_b200 import mcmc
    K = 16
    opt = _optimizer(_scene(2001, K, seed=11), K, steps=2)
    params, moments = _dicts(opt, K)
    seed = lambda s: torch.Generator(device=DEV).manual_seed(s)
    d = mcmc.relocate_packed(opt, generator=seed(1))
    params, moments, d2 = mcmc.relocate(params, moments, generator=seed(1), return_count=True)
    P_new = mcmc.add_packed(opt, 2090, generator=seed(2))
    params, moments = mcmc.add(params, moments, 2090, generator=seed(2))
    mcmc.inject_noise_packed(opt, generator=seed(3))
    mcmc.inject_noise(params, LRS["xyz"], generator=seed(3))
    assert d == d2 > 0 and P_new == 2090 == params["xyz"].shape[0]
    st = opt.state[opt.packed]
    for got, want in ((_pack(params), opt.packed), (_pack({k: m for k, (m, _) in moments.items()}), st["exp_avg"]),
                      (_pack({k: v for k, (_, v) in moments.items()}), st["exp_avg_sq"])):
        assert got.cpu().numpy().tobytes() == want.detach().cpu().numpy().tobytes()


def test_strict_deterministic_mode_admits_every_call():
    """relocate, add and noise run under use_deterministic_algorithms(True) without warn_only, and repeat bit for bit"""
    from humangaussian_b200 import mcmc
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        out = []
        for _ in range(2):
            opt = _optimizer(_scene(1500, seed=2))
            g = torch.Generator(device=DEV).manual_seed(5)
            with warnings.catch_warnings():
                warnings.simplefilter("error")
                mcmc.relocate_packed(opt, generator=g)
                mcmc.add_packed(opt, 10 ** 6, generator=g)
                mcmc.inject_noise_packed(opt, generator=g)
            out.append(_snapshot(opt))
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    assert out[0][0] == out[1][0]
    for a, b in zip(out[0][1:4], out[1][1:4]):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def train_mcmc(seed=4, steps=220, cap_max=2400, interval=50, lam_o=0.01, lam_s=0.01):
    """A packed training loop fitting 8 target views of a seeded scene from a perturbed start: Adam, then every `interval`
    steps relocate and add, noise every step, and the opacity / scale regulariser.  Returns per-step losses and the final
    state."""
    from humangaussian_b200 import dist as D
    from humangaussian_b200 import mcmc
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.optim import PackedAdam, expon_lr_func
    from humangaussian_b200.rasterizer import rasterize_views_packed
    from humangaussian_b200.renderer import stack_cameras
    K, H = 16, 64
    vm, pm, cp, tx, ty = stack_cameras(sample_orbit_cameras(8, H, H, seed=3), DEV)
    bg = torch.tensor([0.8, 0.5, 0.2], device=DEV)
    render = lambda flat, P: rasterize_views_packed(flat, P, K, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx,
                                                    tanfovy=ty, image_height=H, image_width=H, bg=bg, sh_degree=3, raw=True)[0]
    with torch.no_grad():
        tgt = _scene(3000, seed=100, dead=0.0)
        tgt["opacity"][1] = 2.0
        target = render(D.pack({k: v.to(DEV).contiguous() for k, v in tgt.items()}), 3000)
    raw = _scene(2000, seed=seed, dead=0.2)
    raw["xyz"] = raw["xyz"] + 0.05 * torch.randn(raw["xyz"].shape, generator=torch.Generator().manual_seed(seed))
    raw["opacity"][raw["opacity"] < -7] = -20.0  # dead from the start: relocation has rows to move
    raw["opacity"][1] = -20.0
    flat = D.pack({k: v.to(DEV).contiguous() for k, v in raw.items()}).requires_grad_(True)
    opt = PackedAdam(flat, 2000, K, LRS, xyz_scheduler=expon_lr_func(1.6e-4, 1.6e-6, lr_delay_mult=0.01, max_steps=30000))
    g = torch.Generator(device=DEV).manual_seed(seed)
    losses, sizes, moved = [], [], []
    for it in range(steps):
        opt.update_learning_rate(it)
        f = D.unpack(opt.packed, opt.P, K)
        loss = (render(opt.packed, opt.P) - target).abs().mean()
        reg = lam_o * torch.sigmoid(f["opacity"]).mean() + lam_s * torch.exp(f["scaling"]).mean()
        (loss + reg).backward()
        opt.step()
        opt.zero_grad()
        if it and it % interval == 0:
            moved.append(mcmc.relocate_packed(opt, generator=g))
            mcmc.add_packed(opt, cap_max, generator=g)
        mcmc.inject_noise_packed(opt, generator=g)
        losses.append(float(loss.detach()))
        sizes.append(opt.P)
    st = opt.state[opt.packed]
    return dict(losses=losses, sizes=sizes, moved=moved, packed=opt.packed.detach().clone(), exp_avg=st["exp_avg"].clone(),
                exp_avg_sq=st["exp_avg_sq"].clone())


def test_training_loop():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        a, b = train_mcmc(), train_mcmc()
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    assert max(a["sizes"]) <= 2400 and a["sizes"][-1] == 2400
    assert a["moved"][0] > 0
    for k in ("packed", "exp_avg", "exp_avg_sq"):
        assert torch.isfinite(a[k]).all(), k
    first, last = np.mean(a["losses"][:5]), np.mean(a["losses"][-5:])
    assert last < 0.8 * first, (first, last)
    assert a["losses"] == b["losses"] and a["sizes"] == b["sizes"] and a["moved"] == b["moved"]
    for k in ("packed", "exp_avg", "exp_avg_sq"):
        assert a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k
