"""CPU: the oracle's exports of the two intermediates the CUDA backward blend is built on (DESIGN.md section 3).

  * contrib_patches: per sorted instance, which 8x4 patches of its tile blended it.  Checked against a brute-force numpy
    replay of the blend that shares nothing with gs_oracle.c but the pinned float operation order.
  * the moments export of gso_backward (sums in the kernel's ScreenGrad format, with error scales): checked against the
    oracle's own per-Gaussian screen-space sums through the linear map the CUDA preprocess backward applies."""
import numpy as np

from util import grad_images, small_scene

ALPHA_MIN, ALPHA_MAX, T_MIN = np.float32(1.0 / 255.0), np.float32(0.99), np.float32(1e-4)
U = 2.0 ** -24
f32 = np.float32


def _fma(a, b, c):
    """binary32 fma: the product of two floats is exact in double; the one rounding of the sum is done in double and then to
    float (a double rounding, which can differ from a fused rounding only on an exact float midpoint)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def _gs_exp(x):
    """numpy restatement of gs_exp (gs_oracle.c): range reduction + degree-5 polynomial + exponent add."""
    x = np.maximum(np.asarray(x, f32), f32(-87.0))
    t = _fma(x, f32(float.fromhex("0x1.715476p+0")), f32(12582912.0))
    n = (t - f32(12582912.0)).astype(f32)
    r = _fma(n, f32(-float.fromhex("0x1.62e430p-1")), x)
    p = np.full_like(x, f32(float.fromhex("0x1.0fa834p-7")))
    for cst in ("0x1.573a54p-5", "0x1.555a6ap-3", "0x1.fffdc6p-2", "0x1.fffff6p-1", "0x1p+0"):
        p = _fma(p, r, f32(float.fromhex(cst)))
    return (p.view(np.uint32) + (t.view(np.uint32) << np.uint32(23))).view(f32)


def _scene():
    inp, _, _ = small_scene(P=300, deg=1, seed=2, H=37, W=50)  # partial tiles and partial patches on both axes
    from oracle.gs_oracle import Oracle
    o = Oracle(threads=2)
    o.forward(**inp)
    return inp, o, o.state()


def test_contrib_patches_match_a_numpy_replay():
    inp, o, st = _scene()
    H, W = inp["image_height"], inp["image_width"]
    gx = (W + 15) // 16
    xy, co, pl = st["xy"], st["conic_opacity"], st["point_list"]
    want = np.zeros(st["num_rendered"], np.uint8)
    n_contrib = np.zeros((H, W), np.uint32)
    powers = []
    for t, (r0, r1) in enumerate(st["ranges"]):
        ys, xs = np.mgrid[(t // gx) * 16:(t // gx) * 16 + 16, (t % gx) * 16:(t % gx) * 16 + 16]
        keep = (ys < H) & (xs < W)
        ys, xs = ys[keep], xs[keep]
        fx, fy = xs.astype(f32), ys.astype(f32)
        pbit = (1 << (((ys % 16) // 4) * 2 + (xs % 16) // 8)).astype(np.uint8)
        T = np.ones(len(xs), f32)
        alive = np.ones(len(xs), bool)
        for j in range(r0, r1):
            g = pl[j]
            A, B, C, op = co[g]
            dx, dy = (xy[g, 0] - fx).astype(f32), (xy[g, 1] - fy).astype(f32)
            u = _fma(-B, dy, (f32(-0.5) * A * dx).astype(f32))
            w = ((f32(-0.5) * C * dy).astype(f32) * dy).astype(f32)
            power = _fma(dx, u, w)
            powers.append(power[power <= 0])
            alpha = np.minimum(ALPHA_MAX, (op * _gs_exp(np.minimum(power, f32(0)))).astype(f32))
            test_T = (T * (f32(1) - alpha)).astype(f32)
            cand = alive & (power <= 0) & (alpha >= ALPHA_MIN)
            alive &= ~(cand & (test_T < T_MIN))            # the terminating entry is not blended
            blend = cand & alive
            T = np.where(blend, test_T, T)
            want[j] = np.bitwise_or.reduce(pbit[blend]) if blend.any() else 0
            n_contrib[ys[blend], xs[blend]] = j - r0 + 1
    # the replay's exp is the oracle's, bit for bit, on every power it evaluated
    from oracle.gs_oracle import gs_exp
    pw = np.concatenate(powers)
    sample = pw[np.random.RandomState(0).choice(len(pw), min(len(pw), 4000), replace=False)]
    assert np.array_equal(_gs_exp(sample).view(np.uint32), gs_exp(sample).view(np.uint32))
    assert np.array_equal(n_contrib, st["n_contrib"]), "replay does not reproduce the oracle's n_contrib"
    assert (want != 0).sum() > 200 and len(np.unique(want)) > 20, "scene too thin to exercise the patch bits"
    assert np.array_equal(st["contrib_patches"], want)


def test_moment_sums_map_onto_the_oracle_screen_sums():
    """The preprocess backward's map from moments to screen-space gradients, applied to the export, gives the oracle's own
    double sums o[0..9].  S0 is o[5] term for term (the same float32 q, the same double additions): equal exactly.  The other
    components agree to the float32 rounding of the oracle's per-term products (o[k] multiplies G, dx, conic and opacity in
    float32 before adding in double): a few u per term, bounded with the error scale, which is >= the sum of |term|."""
    inp, o, st = _scene()
    H, W = inp["image_height"], inp["image_width"]
    g = o.backward(*grad_images(H, W, 4), sums_err_const=1.0)
    S, E, ref = g["sums"], g["sums_err"], g["screen_sums"]
    A, B, C, op = (st["conic_opacity"][:, k].astype(np.float64) for k in range(4))
    vis = g["sums_err"][:, 0] > 0
    assert vis.sum() > 150
    assert np.array_equal(S[:, 0], ref[:, 5])
    assert np.array_equal(np.float32(S[:, 0]), g["opacities"][:, 0])
    assert (np.abs(S) <= E).all(), "an error scale is smaller than its sum's magnitude"
    mapped = np.stack([-op * (A * S[:, 1] + B * S[:, 2]) * (0.5 * W), -op * (C * S[:, 2] + B * S[:, 1]) * (0.5 * H),
                       -0.5 * op * S[:, 3], -0.5 * op * S[:, 4], -0.5 * op * S[:, 5], S[:, 0],
                       S[:, 6], S[:, 7], S[:, 8], S[:, 9]], 1)
    scale = np.stack([op * (np.abs(A) * E[:, 1] + np.abs(B) * E[:, 2]) * (0.5 * W),
                      op * (np.abs(C) * E[:, 2] + np.abs(B) * E[:, 1]) * (0.5 * H),
                      0.5 * op * E[:, 3], 0.5 * op * E[:, 4], 0.5 * op * E[:, 5], E[:, 0], E[:, 6], E[:, 7], E[:, 8], E[:, 9]], 1)
    err = np.abs(mapped - ref)
    assert (err <= 8 * U * scale + 1e-300).all(), f"worst {float((err / (8 * U * scale + 1e-300)).max()):.2f}x"
    # and the map is not vacuous: every component is populated
    assert (np.abs(ref[vis]).max(0) > 0).all()
