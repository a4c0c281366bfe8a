"""CPU: the multi-view raw-parameter step reference (tests/bench_step_reference.py) that test_gpu_bench_step.py holds
bench.py's timed step to, checked without a GPU.

  1. On a small scene (2 000 Gaussians, SH degree 3, raw parameters with un-normalised quaternions, 4 views at 64^2) the
     float64 sum of the oracle's per-view gradients, chained through the activation Jacobians, equals float64 autograd of the
     same raw-parameter loss through oracle/dense_ref.py within test_oracle_autograd.py's 1e-4 abs / 1e-3 rel.
  2. The three Jacobians equal torch.autograd.functional.jacobian of exp, sigmoid and F.normalize in float64.
  3. The benchmark's scene, cameras and view order come out of the same calls bench.Harness and run_b200 make."""
import math

import numpy as np
import pytest
import torch

import bench_step_reference as BS
from util import close, grad_images


def _small_step():
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.scene import synthetic_body
    p = synthetic_body(2000, sh_degree=3, seed=12)
    p.scaling += math.log(4.0)  # real overlap at 64^2
    p.opacity += 1.0
    raw = BS.raw_of_params(p)
    n = np.linalg.norm(raw["rotations"].astype(np.float64), axis=1)
    assert n.min() < 0.9 and n.max() > 1.1, "the quaternions should be far from unit length"
    cams = sample_orbit_cameras(4, 64, 64, seed=3)
    gws = [grad_images(64, 64, 70 + v) for v in range(4)]
    return raw, cams, gws


def test_summed_chained_reference_matches_float64_autograd_of_the_raw_loss():
    from oracle.dense_ref import dense_render
    raw, cams, gws = _small_step()
    act = BS.activate(raw)
    views = BS.views_reference(act, cams, gws, sh_degree=3, H=64, W=64, threads=1)
    acc = BS.StepSum(len(act["means3D"]))
    for v in views:
        acc.add(v)
    assert all((v["radii"] > 0).sum() > 500 and v["num_rendered"] > 2000 for v in views), [v["num_rendered"] for v in views]
    ref, bound = acc.result(act, raw)

    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    leaves = {k: t64(raw[k]).requires_grad_(True) for k in BS.FIELDS}
    P = len(act["means3D"])
    for i, (v, cam) in enumerate(zip(views, cams)):
        ci = BS.cam_inputs(cam)
        ids = np.nonzero(v["radii"] > 0)[0]
        order = ids[np.lexsort((ids, v["depths"][ids]))]
        c, d, a, _ = dense_render(
            means3D=leaves["xyz"], means2D=torch.zeros(P, 3, dtype=torch.float64), opacities=torch.sigmoid(leaves["opacities"]),
            viewmatrix=t64(ci["viewmatrix"]), projmatrix=t64(ci["projmatrix"]), campos=t64(ci["campos"]),
            bg=torch.zeros(3, dtype=torch.float64), H=64, W=64, tanfovx=ci["tanfovx"], tanfovy=ci["tanfovy"], radii=v["radii"],
            rect=v["rect"], order=order, sh_degree=3, shs=leaves["shs"], scales=torch.exp(leaves["scales"]),
            rotations=torch.nn.functional.normalize(leaves["rotations"]))
        gC, gD, gA = (t64(x) for x in gws[i])
        for got, want in ((v["color"], c), (v["depth"], d), (v["alpha"], a)):
            ok, worst = close(got, want.detach().numpy())
            assert ok, f"oracle image vs float64 dense image: {worst:.2f}x tolerance"
        ((c * gC).sum() + (d * gD).sum() + (a * gA).sum()).backward()  # one graph per view: autograd sums the views
    for k in BS.FIELDS:
        want = leaves[k].grad.numpy().reshape(P, -1)
        assert np.abs(want).max() > 0
        ok, worst = close(ref[k], want, atol=1e-4, rtol=1e-3)
        assert ok, f"raw dL/d{k}: summed and chained reference vs float64 autograd {worst:.2f}x over (1e-4 abs, 1e-3 rel)"
        assert bound[k].shape == ref[k].shape and (bound[k] >= 0).all()
    # a Gaussian no view sees has a zero bound: its raw gradient must be exactly zero
    unseen = ~np.any([v["radii"] > 0 for v in views], axis=0)
    assert all(float(bound[k][unseen].max(initial=0.0)) == 0.0 for k in BS.FIELDS)


@pytest.mark.parametrize("field", ["scales", "opacities", "rotations"])
def test_activation_jacobians_match_autograd(field):
    rng = np.random.RandomState(dict(scales=0, opacities=1, rotations=2)[field])
    n, width = 16, dict(scales=3, opacities=1, rotations=4)[field]
    f = dict(scales=torch.exp, opacities=torch.sigmoid, rotations=lambda x: x / x.norm())[field]
    rows = rng.randn(n, width) * (2.0 if field != "rotations" else 1.0)
    if field == "rotations":
        rows *= rng.uniform(0.2, 3.0, (n, 1))  # far from unit length
    g = rng.randn(n, width)
    raw = dict(scales=np.zeros((n, 3)), rotations=np.tile([1.0, 0, 0, 0], (n, 1)), opacities=np.zeros((n, 1)))
    raw[field] = rows
    act = dict(scales=np.exp(raw["scales"]), opacities=1.0 / (1.0 + np.exp(-raw["opacities"])),
               rotations=raw["rotations"] / np.linalg.norm(raw["rotations"], axis=1, keepdims=True))
    zero = dict(xyz=np.zeros((n, 3)), shs=np.zeros((n, 3)), scales=np.zeros((n, 3)), rotations=np.zeros((n, 4)), opacities=np.zeros((n, 1)))
    got = BS.chain(dict(zero, **{field: g}), act, raw)[field]
    for i in range(n):
        J = torch.autograd.functional.jacobian(f, torch.tensor(rows[i], dtype=torch.float64)).numpy().reshape(width, width)
        want = J.T @ g[i]
        assert np.allclose(got[i], want, rtol=1e-12, atol=1e-14), (field, i, got[i], want)


def test_bench_scene_cameras_and_view_order_are_the_harness_objects(monkeypatch):
    """bench.Harness built on the host (its pinned staging buffer as a plain one) holds the reference's scene in its packed
    buffer and the reference's cameras; run_b200's balanced shard of one rank is the identity order."""
    import bench
    args = BS.bench_args()
    assert (args.gaussians, args.views, args.res, args.sh_degree, args.scene) == (300000, 64, 1024, 3, "sample")
    zeros = torch.zeros

    def host_zeros(*a, pin_memory=False, **k):
        return zeros(*a, **k)
    monkeypatch.setattr(torch, "zeros", host_zeros)
    h = bench.Harness(args, torch.device("cpu"), 0, 1)
    monkeypatch.setattr(torch, "zeros", zeros)
    p = BS.bench_scene(args)
    raw = BS.raw_of_params(p)
    assert (h.P, h.K, h.HW, h.deg) == (p.P, 16, 1024, 3) == (300000, 16, 1024, 3)
    for (o, n, shape), k in zip(h.fields, BS.FIELDS):
        assert np.array_equal(h.host_flat.narrow(0, o, n).view(shape).numpy(), raw[k]), k
        assert np.array_equal(h.flat.detach().narrow(0, o, n).view(shape).numpy(), raw[k]), k
    cams = BS.bench_cameras(args)
    assert len(cams) == len(h.all_cams) == 64
    for a, b in zip(cams, h.all_cams):
        for k in ("world_view_transform", "full_proj_transform", "camera_center"):
            assert torch.equal(getattr(a, k), getattr(b, k)), k
        assert (a.FoVx, a.FoVy, a.image_width, a.image_height) == (b.FoVx, b.FoVy, b.image_width, b.image_height)
    assert BS.bench_shard(args, h.all_cams) == list(range(64))
    # the 8-view operating point is the first eight of the same cameras
    assert all(torch.equal(a.world_view_transform, b.world_view_transform) for a, b in zip(cams[:8], h.all_cams[:8]))
