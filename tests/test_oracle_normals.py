"""CPU: the normal-map reference (tests/normal_reference.py) against float64 autograd and oracle/dense_ref.py.

  1. d(column k of R(q))/dq as normal_bwd_kernel chains it (restated below), post-activation and raw, against autograd;
  2. the replayed normal image against dense_ref's colour image with colors_precomp = n and bg = 0;
  3. edge cases: the flip toward the camera, argmin ties (the lowest index wins), a Gaussian seen exactly edge-on (d = 0)."""
import numpy as np
import pytest
import torch

import normal_reference as NR
from util import small_scene


def dcol_dq(k, q, g):
    """normals.cu's dcol_dq: dL/dq of column k of R(q) for the column gradient g (float64 restatement)"""
    r, x, y, z = q
    g0, g1, g2 = g
    if k == 0:
        return np.array([2 * (z * g1 - y * g2), 2 * (y * g1 + z * g2), -4 * y * g0 + 2 * (x * g1 - r * g2), -4 * z * g0 + 2 * (r * g1 + x * g2)])
    if k == 1:
        return np.array([2 * (x * g2 - z * g0), 2 * (y * g0 + r * g2) - 4 * x * g1, 2 * (x * g0 + z * g2), 2 * (y * g2 - r * g0) - 4 * z * g1])
    return np.array([2 * (y * g0 - x * g1), 2 * (z * g0 - r * g1) - 4 * x * g2, 2 * (r * g0 + z * g1) - 4 * y * g2, 2 * (x * g0 + y * g1)])


@pytest.mark.parametrize("raw", [False, True])
@pytest.mark.parametrize("k", [0, 1, 2])
def test_hand_chain_matches_autograd(k, raw):
    rng = np.random.RandomState(k + 3 * raw)
    for _ in range(20):
        q0 = rng.randn(4) * (2.0 if raw else 1.0)
        if not raw:
            q0 /= np.linalg.norm(q0)
        g = rng.randn(3)
        qt = torch.tensor(q0, requires_grad=True)
        q = torch.nn.functional.normalize(qt, dim=0) if raw else qt
        n = NR.normals_torch(q[None], np.array([k]), np.array([1.0]))[0]
        (n * torch.tensor(g)).sum().backward()
        qn = q.detach().numpy()
        dq = dcol_dq(k, qn, g)
        if raw:  # F.normalize's Jacobian, as the kernel applies it
            dq = (dq - qn * (qn @ dq)) / np.linalg.norm(q0)
        np.testing.assert_allclose(dq, qt.grad.numpy(), rtol=1e-12, atol=1e-12)


def test_rotation_columns_are_the_covariance_axes():
    _, q = NR.activate(np.ones((50, 3)), np.random.RandomState(1).randn(50, 4), raw=True)
    R = NR.rot_columns(q).astype(np.float64)
    np.testing.assert_allclose(R @ R.transpose(0, 2, 1), np.broadcast_to(np.eye(3), (50, 3, 3)), atol=2e-6)


@pytest.mark.parametrize("deg", [0, 3])
def test_replayed_image_matches_dense_ref(deg):
    from oracle.dense_ref import dense_render
    inp, _, _ = small_scene(P=80, deg=deg, seed=4 + deg, H=32, W=48)
    nrm = NR.gauss_normals(inp["means3D"], inp["campos"], inp["scales"], inp["rotations"])
    img = NR.reference_image(inp, nrm=nrm)
    st, radii = NR.oracle_state(inp)
    ids = np.nonzero(radii > 0)[0]
    order = ids[np.lexsort((ids, st["depths"][ids]))]
    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    c, _, _, _ = dense_render(means3D=t64(inp["means3D"]), means2D=torch.zeros(len(radii), 3, dtype=torch.float64),
                              opacities=t64(inp["opacities"]), viewmatrix=t64(inp["viewmatrix"]), projmatrix=t64(inp["projmatrix"]),
                              campos=t64(inp["campos"]), bg=torch.zeros(3, dtype=torch.float64), H=32, W=48,
                              tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], radii=radii, rect=st["rect"], order=order,
                              colors_precomp=t64(nrm[:, :3]), scales=t64(inp["scales"]), rotations=t64(inp["rotations"]))
    assert np.abs(img).max() > 0.1
    np.testing.assert_allclose(img, c.numpy(), atol=2e-5, rtol=1e-4)


def test_flip_faces_the_camera():
    inp, _, _ = small_scene(P=200, deg=0, seed=2)
    g = NR.gauss_normals(inp["means3D"], inp["campos"], inp["scales"], inp["rotations"])
    e = inp["campos"].reshape(1, 3) - inp["means3D"]
    assert ((g[:, :3] * e).sum(1) >= 0).all()
    assert set(np.unique(g[:, 3])) <= {-1.0, 1.0} and (g[:, 3] == -1).any() and (g[:, 3] == 1).any()
    # the faced normal is the axis column itself or its negation, never anything else
    k = NR.axis(inp["scales"])
    R = NR.rot_columns(inp["rotations"])
    col = R[np.arange(200), :, k]
    np.testing.assert_array_equal(g[:, :3], col * g[:, 3:4])
    # turning the Gaussian by pi about another of its own axes, q -> q (x) (0, e_j) with j != k, negates column k; the faced
    # normal stays the same
    q = np.asarray(inp["rotations"], np.float64)
    j = (k + 1) % 3
    e = np.zeros((200, 4)); e[np.arange(200), 1 + j] = 1.0
    r0, v0 = q[:, :1], q[:, 1:]
    r1, v1 = e[:, :1], e[:, 1:]
    q2 = np.concatenate([r0 * r1 - (v0 * v1).sum(1, keepdims=True), r0 * v1 + r1 * v0 + np.cross(v0, v1)], 1).astype(np.float32)
    col2 = NR.rot_columns(q2)[np.arange(200), :, k]
    assert np.abs(col2 + col).max() < 1e-5
    g2 = NR.gauss_normals(inp["means3D"], inp["campos"], inp["scales"], q2)
    np.testing.assert_allclose(g2[:, :3], g[:, :3], atol=1e-5)


def test_argmin_ties_take_the_lowest_index():
    s = np.array([[1, 1, 1], [2, 1, 1], [1, 2, 1], [3, 2, 2], [0.5, 0.5, 0.7], [np.nan, 1, 2]], np.float32)
    # (strict comparisons: a NaN in front is never displaced, as in the kernel)
    np.testing.assert_array_equal(NR.axis(s), [0, 1, 0, 1, 0, 0])


def test_edge_on_keeps_the_sign():
    # a Gaussian whose axis is perpendicular to the view ray: d = 0 exactly, no flip; a NaN position keeps the sign too
    q = np.array([[1, 0, 0, 0], [1, 0, 0, 0]], np.float32)  # identity: the columns are the coordinate axes
    s = np.array([[0.1, 1, 1], [0.1, 1, 1]], np.float32)      # axis 0 = +x
    means = np.array([[0, 0, 5], [np.nan, 0, 0]], np.float32)
    g = NR.gauss_normals(means, np.zeros(3, np.float32), s, q)
    np.testing.assert_array_equal(g, [[1, 0, 0, 1], [1, 0, 0, 1]])
    g2 = NR.gauss_normals(np.array([[3, 0, 0]], np.float32), np.zeros(3, np.float32), s[:1], q[:1])
    np.testing.assert_array_equal(g2, [[-1, 0, 0, -1]])
