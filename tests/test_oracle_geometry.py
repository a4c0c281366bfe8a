"""CPU: the geometry-output reference (tests/geometry_reference.py) and humangaussian_b200/geometry.py.

  1. the replayed M2 against dense_ref's float64 colour image with colors_precomp = (z^2, 0, 0), bg = 0; the median against a
     float64 restatement of the rule over each pixel's blends;
  2. depth_distortion = A M2 - M1^2 against the pairwise sum sum_{i<j} w_i w_j (d_i - d_j)^2;
  3. the median rule's edges: T exactly 0.5 (an alpha = 0.5 Gaussian at its centre pixel), a pixel that never reaches
     alpha = 1/2, an empty pixel;
  4. depth_to_normal on an analytic plane; depth_normal_consistency's mask."""
import math

import numpy as np
import pytest
import torch

import geometry_reference as GR
from util import screen_scene, small_scene

from humangaussian_b200 import geometry as G


@pytest.mark.parametrize("deg", [0, 3])
def test_replay_matches_float64(deg):
    from oracle.dense_ref import dense_render
    inp, _, _ = small_scene(P=80, deg=deg, seed=4 + deg, H=32, W=48)
    st, radii = GR.oracle_state(inp)
    r = GR.replay(st, 32, 48, lists=True)
    ids = np.nonzero(radii > 0)[0]
    order = ids[np.lexsort((ids, st["depths"][ids]))]
    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    z = GR.view_depth64(t64(inp["means3D"]), inp["viewmatrix"])
    # the oracle's record depth is the float32 view-space z
    assert np.abs(st["depths"][ids] - z.numpy()[ids]).max() <= 1e-6 * np.abs(z.numpy()[ids]).max()
    zc = torch.stack([z * z, torch.zeros_like(z), torch.zeros_like(z)], 1)
    c, _, _, _ = dense_render(means3D=t64(inp["means3D"]), means2D=torch.zeros(len(radii), 3, dtype=torch.float64),
                              opacities=t64(inp["opacities"]), viewmatrix=t64(inp["viewmatrix"]), projmatrix=t64(inp["projmatrix"]),
                              campos=t64(inp["campos"]), bg=torch.zeros(3, dtype=torch.float64), H=32, W=48,
                              tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], radii=radii, rect=st["rect"], order=order,
                              colors_precomp=zc, scales=t64(inp["scales"]), rotations=t64(inp["rotations"]))
    m2 = c[0].numpy()
    assert r["depth2"].max() > 0.1 and (r["median_pos"] > 0).mean() > 0.15
    np.testing.assert_allclose(r["depth2"], m2, rtol=1e-4, atol=1e-5 * m2.max())
    # the median rule restated in float64 over each pixel's blends (T_before = prod (1 - alpha) of the earlier blends)
    checked = 0
    for (y, x), bl in r["blends"].items():
        T, med = 1.0, 0.0
        for w, d in bl:
            if T > 0.5 and abs(T - 0.5) > 1e-5:
                med = float(d)
            elif abs(T - 0.5) <= 1e-5:
                med = None
                break
            T -= float(w)
        if med is None:
            continue
        checked += 1
        assert r["median"][y, x] == np.float32(med), (y, x)
    assert checked > 200
    empty = r["median_pos"] == 0
    assert np.all(r["median"][empty] == 0) and np.all(r["depth2"][empty] == 0)


def test_distortion_is_the_pairwise_sum():
    inp, _, _ = small_scene(P=80, deg=1, seed=6, H=32, W=48)
    st, _ = GR.oracle_state(inp)
    r = GR.replay(st, 32, 48, lists=True)
    A = np.zeros((1, 32, 48))
    M1 = np.zeros((1, 32, 48))
    pair = np.zeros((1, 32, 48))
    for (y, x), bl in r["blends"].items():
        w = np.array([b[0] for b in bl], np.float64)
        d = np.array([b[1] for b in bl], np.float64)
        A[0, y, x], M1[0, y, x] = w.sum(), (w * d).sum()
        pair[0, y, x] = sum(w[i] * w[j] * (d[i] - d[j]) ** 2 for i in range(len(w)) for j in range(i + 1, len(w)))
    M2 = np.zeros((1, 32, 48))
    for (y, x), bl in r["blends"].items():
        M2[0, y, x] = sum(float(w) * float(d) ** 2 for w, d in bl)
    dist = G.depth_distortion(torch.tensor(A), torch.tensor(M1), torch.tensor(M2)).numpy()
    assert pair.max() > 1e-3
    np.testing.assert_allclose(dist, pair, rtol=1e-9, atol=1e-12 * M2.max())
    # float32 inputs: formed in float64, returned in float32, unclamped
    d32 = G.depth_distortion(torch.tensor(A, dtype=torch.float32), torch.tensor(M1, dtype=torch.float32),
                             torch.tensor(M2, dtype=torch.float32))
    assert d32.dtype == torch.float32


def _edge_scene():
    # pixel (12, 6): an alpha = 0.5 Gaussian at its centre over a second one behind (T lands exactly on 0.5);
    # pixel (44, 6): two Gaussians of opacity 0.2 (T never reaches 0.5); pixel (100, 40): nothing
    px = [12, 12, 44, 44]
    py = [6, 6, 6, 6]
    depth = [2.0, 3.0, 2.5, 4.0]
    op = [0.5, 0.7, 0.2, 0.2]
    return screen_scene(px, py, depth, 0.2, op, H=64, W=128)


def test_median_rule_edges():
    inp = _edge_scene()
    r = GR.reference_images(inp)
    st, _ = GR.oracle_state(inp)
    d = st["depths"]
    # T before the first is 1 and before the second exactly 0.5: the strict > keeps the first
    assert r["median_pos"][6, 12] == 1 and r["median"][6, 12] == d[0]
    # T stays above 0.5: the median is the last blend
    assert r["median_pos"][6, 44] == 2 and r["median"][6, 44] == d[3]
    # nothing blends
    assert r["median_pos"][40, 100] == 0 and r["median"][40, 100] == 0 and r["depth2"][40, 100] == 0
    # alpha is exactly 0.5 at the centre: 0.5 * gs_exp(0)
    assert st["conic_opacity"][0, 3] == np.float32(0.5)


def test_depth_to_normal_plane():
    H, W = 40, 56
    tanx, tany = 0.5, 0.5 * H / W
    # camera at the origin looking down +z (identity view matrix); plane n . p = c with n = (0.3, -0.2, -1) normalised
    n = np.array([0.3, -0.2, -1.0])
    n /= np.linalg.norm(n)
    c = -3.0
    px, py = np.meshgrid(np.arange(W), np.arange(H))
    rx = ((2 * px + 1) / W - 1) * tanx
    ry = ((2 * py + 1) / H - 1) * tany
    z = c / (n[0] * rx + n[1] * ry + n[2])
    out = G.depth_to_normal(torch.tensor(z[None, None]), torch.eye(4, dtype=torch.float64)[None], [tanx], [tany])
    inner = out[0, :, 1:-1, 1:-1].reshape(3, -1).T.numpy()
    # faces the camera: n . (0 - p) > 0, i.e. the normal whose z is negative here
    np.testing.assert_allclose(inner, np.broadcast_to(n, inner.shape), atol=1e-9)
    assert torch.all(out[0, :, 0] == 0) and torch.all(out[0, :, :, -1] == 0)
    # a translated camera: world = view - t for an identity rotation (row-vector p_view = p_world @ R + t)
    vm = torch.eye(4, dtype=torch.float64)
    vm[3, :3] = torch.tensor([0.5, -1.0, 2.0])
    out2 = G.depth_to_normal(torch.tensor(z[None, None]), vm[None], [tanx], [tany])
    np.testing.assert_allclose(out2.numpy(), out.numpy(), atol=1e-9)


def test_consistency_mask():
    normal = torch.zeros(1, 3, 4, 4)
    normal[:, 2] = 1.0
    dn = torch.zeros(1, 3, 4, 4)
    dn[:, 2, 1:3, 1:3] = 1.0
    dn[:, 0, 1, 1] = 1.0  # 45 degrees at (1, 1)
    alpha = torch.ones(1, 1, 4, 4)
    alpha[..., 2, 2] = 0.2
    L = G.depth_normal_consistency(normal, dn, alpha)
    assert L[0, 0, 1, 2] == 0 and L[0, 0, 2, 2] == 0 and L[0, 0, 0, 0] == 0
    assert abs(float(L[0, 0, 1, 1]) - (1 - math.cos(math.pi / 4))) < 1e-6
