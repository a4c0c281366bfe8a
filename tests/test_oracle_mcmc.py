"""CPU tests of the MCMC densification definition (DESIGN.md section 2): the float64 reference (tests/mcmc_reference.py)
against the identities the split ratio is built on, the paper's double sum, the pinned covariance, and the host-side
draw of humangaussian_b200/mcmc.py."""
import math

import numpy as np
import pytest
import torch
from scipy import integrate

import mcmc_reference as M

O_GRID = [0.005, 0.01, 0.05, 0.2, 0.5, 0.9, 0.99, 1.0 - 2.0 ** -23]
N_GRID = [1, 2, 3, 5, 10, 25, 51]


def _coverage(o_or_op, s, n):
    """integral over x of 1 - (1 - a g(x/s))^n, g(x) = exp(-x^2/2) (n = 1: a g(x/s) itself)"""
    f = lambda x: -math.expm1(n * math.log1p(-o_or_op * math.exp(-0.5 * (x / s) ** 2)))
    return 2.0 * integrate.quad(f, 0.0, np.inf, epsabs=0.0, epsrel=1e-13, limit=500)[0]


@pytest.mark.parametrize("o", O_GRID)
def test_split_preserves_opacity_and_footprint(o):
    """without the clamp: 1 - (1 - o')^n = o, and n members of scale s' = s o / D cover what the row covered"""
    s = 1.0
    for n in N_GRID:
        op = M.split_opacity(o, n, clamp=False)
        assert abs(-math.expm1(n * math.log1p(-op)) - o) <= 1e-12 * o
        s_new = s * o / M.D_one_sum(op, n)
        want = o * s * math.sqrt(2.0 * math.pi)
        assert abs(_coverage(op, s_new, n) - want) <= 1e-8 * want, (o, n)


def test_one_sum_equals_double_sum():
    """the hockey-stick collapse; both float64 sums cancel (worst here 6e-13 relative, at o = 1 - 2^-23, n = 40)"""
    for o in O_GRID:
        for n in range(1, M.N_MAX + 1):
            op = M.split_opacity(o, n)
            a, b = M.D_one_sum(op, n), M.D_double_sum(op, n)
            assert abs(a - b) <= 1e-12 * abs(b), (o, n, a, b)


def test_one_member_is_the_identity():
    """n = 1 gives the row its own opacity and scales (inside the clamp range)"""
    o32 = M.sigmoid32(np.linspace(-5.0, 12.0, 64, dtype=np.float32))
    s = np.random.default_rng(0).normal(-4.0, 1.0, (64, 3)).astype(np.float32)
    logit, scale = M.new_raw(o32, s, np.zeros(64, np.int64))
    o = o32.astype(np.float64)
    np.testing.assert_allclose(logit, np.log(o / (1.0 - o)), rtol=0, atol=1e-9)
    np.testing.assert_allclose(scale, s.astype(np.float64), rtol=0, atol=1e-12)


def test_clamp_ends():
    # o = 1 (float32 sigmoid of a large logit) and o = 1 - 2^-23 both stay finite: o' = 1 - 2^-23 for n = 1
    for o in (1.0, 1.0 - 2.0 ** -23):
        assert M.split_opacity(o, 1) == M.O_MAX
        logit, scale = M.new_raw(np.float32([o]), np.zeros((1, 3), np.float32), [0])
        assert np.isfinite(logit).all() and np.isfinite(scale).all()
        assert abs(logit[0] - math.log(M.O_MAX / (1.0 - M.O_MAX))) < 1e-9
    # a row just above the dead threshold, drawn 50 times: 1 - (1-o)^(1/51) < 0.005 clamps to 0.005
    assert M.split_opacity(0.006, 51, clamp=False) < M.O_MIN
    assert M.split_opacity(0.006, 51) == M.O_MIN
    assert M.members(10 ** 6) == M.N_MAX and M.members(50) == M.N_MAX and M.members(49) == 50


def test_float32_sum_is_not_enough():
    """the alternating sum's terms reach thousands of times D: in float32 it is off by far more than an ulp"""
    worst, term_ratio = 0.0, 0.0
    for o in np.linspace(0.01, 1.0 - 2.0 ** -23, 200):
        for n in (20, 30, 40, 51):
            op = M.split_opacity(o, n)
            d64 = M.D_one_sum(op, n)
            worst = max(worst, abs(float(M.D_one_sum_f32(op, n)) - d64) / d64)
            term_ratio = max(term_ratio, max(math.comb(n, k + 1) * op ** (k + 1) / math.sqrt(k + 1) for k in range(n)) / d64)
    assert worst > 1e-4, worst          # ~1700 float32 ulps
    assert term_ratio > 1e3, term_ratio


def test_noise_covariance_matches_pinned_cov3d():
    """Sigma = R diag(exp(2 s)) R^T equals the oracle's cov3D (pinned against the reference's build_scaling_rotation in
    test_oracle_golden.py), and the noise step is noise_scale * gate * Sigma eta with that Sigma"""
    from test_oracle_golden import _oracle_preprocess
    rng = np.random.default_rng(1)
    P = 256
    s = rng.uniform(-5.0, -1.0, (P, 3)).astype(np.float32)
    q = rng.normal(size=(P, 4)).astype(np.float32) * rng.uniform(0.2, 3.0, (P, 1)).astype(np.float32)
    qn = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    st = _oracle_preprocess(np.tile(np.array([0, 0, 5.0], np.float32), (P, 1)), np.zeros((P, 1, 3), np.float32), 0,
                            np.exp(s).astype(np.float32), qn)
    c = st["cov3d"].astype(np.float64)
    pinned = np.stack([np.stack([c[:, 0], c[:, 1], c[:, 2]], -1), np.stack([c[:, 1], c[:, 3], c[:, 4]], -1),
                       np.stack([c[:, 2], c[:, 4], c[:, 5]], -1)], 1)
    S = M.covariance(s, q)
    scale = np.abs(S).max(axis=(1, 2), keepdims=True)
    assert (np.abs(S - pinned) / scale).max() < 1e-6
    o32 = M.sigmoid32(rng.uniform(-8.0, 3.0, P))
    eta = rng.normal(size=(P, 3))
    got = M.noise_delta(s, q, o32, eta, 80.0)
    want = M.noise_delta(s, q, o32, eta, 80.0, cov=pinned)
    row = np.abs(want).max(1, keepdims=True) + 80.0 * M.gate(o32)[:, None] * scale[:, 0] * np.abs(eta).max(1, keepdims=True)
    assert (np.abs(got - want) / row).max() < 1e-6
    # the gate: 0.5 at the dead threshold, ~0.011 at o = 0.05, below 1e-4 from o = 0.1
    g = M.gate(np.float32([0.005, 0.05, 0.1, 1.0]))
    assert abs(g[0] - 0.5) < 1e-5 and abs(g[1] - 0.011) < 1e-3 and g[2] < 1e-4 and g[3] < 1e-40


def test_draw_follows_the_live_weights():
    """the device draw's host logic on CPU tensors: dead rows are never drawn, frequencies follow sigmoid(opacity)"""
    from humangaussian_b200 import mcmc
    g = torch.Generator().manual_seed(0)
    logits = torch.tensor([-8.0, 0.0, 2.0, float("nan"), -1.0, -6.0, 4.0, -5.4], dtype=torch.float32)
    o, live = mcmc._live(logits, 0.005)
    assert live.tolist() == [False, True, True, False, True, False, True, False]  # NaN is dead; sigmoid(-5.4) < 0.005
    n = 400_000
    s = mcmc._draw(o, live, n, g)
    assert s.dtype == torch.int64 and s.shape == (n,)
    freq = torch.bincount(s, minlength=8).double() / n
    w = torch.where(live, o, torch.zeros_like(o)).double()
    p = w / w.sum()
    assert freq[~live].sum() == 0
    assert (freq - p).abs().max() < 5 * math.sqrt(0.25 / n)


def test_given_samples_are_checked():
    from humangaussian_b200 import mcmc
    live = torch.tensor([True, False, True])
    ok = torch.tensor([0, 2, 2])
    assert torch.equal(mcmc._given_samples(ok, 3, 3, live), ok)
    for bad in (ok.int(), ok[:2], ok.float(), [0, 2, 2]):
        with pytest.raises(ValueError, match="int64"):
            mcmc._given_samples(bad, 3, 3, live)
    with pytest.raises(ValueError, match="index rows"):
        mcmc._given_samples(torch.tensor([0, 3, 2]), 3, 3, live)
    with pytest.raises(ValueError, match="live"):
        mcmc._given_samples(torch.tensor([0, 1, 2]), 3, 3, live)


def test_cpu_tensors_are_refused():
    from humangaussian_b200 import mcmc
    from humangaussian_b200.densify import GROUPS
    params = {k: torch.zeros(4, 3) for k in GROUPS}
    for call in (lambda: mcmc.relocate(params, None), lambda: mcmc.add(params, None, 8), lambda: mcmc.inject_noise(params, 1e-4)):
        with pytest.raises(ValueError, match="CUDA"):
            call()
