"""Float64 numpy reference of MCMC densification (DESIGN.md section 2, "MCMC densification"; humangaussian_b200/mcmc.py,
csrc/mcmc.cu): the split ratio in its one-sum and double-sum forms, the raw values a drawn row takes, and the position
noise.  Structurally independent of the kernels: binomials from math.comb, the covariance as a matrix product."""
from __future__ import annotations

import math

import numpy as np

N_MAX = 51                      # the ratio saturates at 51 members
O_MIN, O_MAX = 0.005, 1.0 - 2.0 ** -23


def sigmoid32(x):
    """1/(1+expf(-x)) in float32 (numpy's float32 exp may differ from the device's expf in the last bit)."""
    x = np.asarray(x, np.float32)
    return (np.float32(1.0) / (np.float32(1.0) + np.exp(-x))).astype(np.float32)


def members(c):
    return np.minimum(np.asarray(c, np.int64) + 1, N_MAX)


def split_opacity(o, n, clamp=True):
    """o' = 1 - (1 - o)^(1/n), clamped to [0.005, 1 - 2^-23]."""
    with np.errstate(divide="ignore"):  # o = 1: log1p(-1) = -inf, o' = 1 before the clamp
        op = -np.expm1(np.log1p(-np.asarray(o, np.float64)) / n)
    return np.clip(op, O_MIN, O_MAX) if clamp else op


def D_one_sum(op, n: int):
    """sum_{k=0}^{n-1} C(n, k+1) (-1)^k o'^(k+1) / sqrt(k+1)"""
    op = np.asarray(op, np.float64)
    return sum(math.comb(n, k + 1) * (-1.0) ** k * op ** (k + 1) / math.sqrt(k + 1) for k in range(n))


def D_double_sum(op, n: int):
    """the paper's form: sum_{i=1}^{n} sum_{k<i} C(i-1, k) (-1)^k o'^(k+1) / sqrt(k+1)"""
    op = np.asarray(op, np.float64)
    return sum(math.comb(i - 1, k) * (-1.0) ** k * op ** (k + 1) / math.sqrt(k + 1) for i in range(1, n + 1) for k in range(i))


def D_one_sum_f32(op, n: int):
    """the same alternating sum evaluated in float32 (what a float32 kernel would get)"""
    op = np.float32(op)
    acc = np.float32(0.0)
    for k in range(n):
        acc = np.float32(acc + np.float32(math.comb(n, k + 1)) * np.float32((-1.0) ** k) * op ** np.float32(k + 1)
                         / np.float32(math.sqrt(k + 1)))
    return acc


def new_raw(o32, scaling32, c):
    """float64 new opacity logit [R] and log-scales [R,3] of rows drawn c >= 1 times; o32 = the float32 sigmoid of the
    row's opacity logit, scaling32 [R,3] its log-scales."""
    o = np.asarray(o32, np.float32).astype(np.float64)
    n = members(c)
    op = np.array([split_opacity(oi, ni) for oi, ni in zip(o, n)])
    D = np.array([D_one_sum(opi, int(ni)) for opi, ni in zip(op, n)])
    logit = np.log(op / (1.0 - op))
    scale = np.log(np.exp(np.asarray(scaling32, np.float32).astype(np.float64)) * (o / D)[:, None])
    return logit, scale


def rotmat(q):
    """R(q / max(||q||, 1e-12)) [P,3,3] in float64, the reference's build_rotation"""
    q = np.asarray(q, np.float64)
    q = q / np.maximum(np.linalg.norm(q, axis=1, keepdims=True), 1e-12)
    r, x, y, z = q.T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                     np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                     np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)


def covariance(scaling, rotation):
    """Sigma = R diag(exp(2 s)) R^T [P,3,3] in float64, from raw log-scales and quaternions"""
    R = rotmat(rotation)
    return R @ (np.exp(2.0 * np.asarray(scaling, np.float64))[:, :, None] * R.transpose(0, 2, 1))


def gate(o32, k=100.0, t=0.005):
    """sigmoid(-k (o - t)) in float64 of the float32 opacity o"""
    o = np.asarray(o32, np.float32).astype(np.float64)
    return 1.0 / (1.0 + np.exp(k * (o - t)))


def noise_delta(scaling, rotation, o32, eta, noise_scale, k=100.0, t=0.005, cov=None):
    """the position step [P,3] in float64: noise_scale * gate * Sigma eta (cov: a [P,3,3] Sigma to use instead)"""
    S = covariance(scaling, rotation) if cov is None else cov
    return noise_scale * gate(o32, k, t)[:, None] * np.einsum("pij,pj->pi", S, np.asarray(eta, np.float64))
