"""GPU parity at BASELINE sizes: ONE view each of BASELINE.md 2.3's configs 2, 3 and 4 through the same bit-exact
forward-state check and gradient criterion as the small scenes (tests/test_gpu_parity.py), against the CPU oracle
(~1-2 s per view on the box), plus a CUDA-vs-float64-autograd backward check against oracle/dense_ref.py -- code the
CUDA backward shares no text with.

  config 2: the full content/sample.ply (531 327 Gaussians, SH deg 0), 512x512, eval-orbit camera
            (threestudio/data/uncond.py:526-608: elevation 15, azimuth 0, distance 2.0, fovy 70)
  config 3: 100 k Gaussians initialised as create_from_pcd does (gaussian_model.py:124-147) on a 100 k subsample of
            sample.ply's positions, SH deg 3 (f_rest ~ N(0, 0.1^2)), 1024x1024
  config 4: the seed-0 300 k subsample of sample.ply, SH deg 3, 1024x1024, cameras 0 and 37 of the bench's 64
The scene comes from tests/golden/sample_ply_full.npz (the reference's own file, repacked)."""
import math

import numpy as np
import pytest
import torch

from test_gpu_parity import DEV, _check_backward, _check_backward_sums, _check_forward_state, _oracle
from util import grad_images, grads_agree

pytestmark = pytest.mark.gpu


def _inputs(p, cam, H, W, deg):
    with torch.no_grad():
        return dict(means3D=p.get_xyz.cpu().numpy().copy(), opacities=p.get_opacity.cpu().numpy().copy(),
                    shs=p.get_features.cpu().numpy().copy(), scales=p.get_scaling.cpu().numpy().copy(),
                    rotations=p.get_rotation.cpu().numpy().copy(), sh_degree=deg,
                    viewmatrix=cam.world_view_transform.cpu().numpy().copy(), projmatrix=cam.full_proj_transform.cpu().numpy().copy(),
                    campos=cam.camera_center.cpu().numpy().copy(), bg=np.zeros(3, np.float32), image_height=H, image_width=W,
                    tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5), scale_modifier=1.0)


# Gradient criterion at full size.  Forward state and images: bit-exact, no exceptions (as everywhere).  Backward: of the
# 100 k - 531 k per-Gaussian gradient rows, at most a 1e-4 fraction may leave the row-wise 1e-5 / 1e-4 tolerance, and none by
# more than 4x.  The rows that leave it (tests/gpu_diag_fullsize.py lists them) are small, low-opacity
# Gaussians deep inside 5-45 k-long tile lists whose gradient is a near-zero sum of mixed-sign pixel terms; two correct float32
# evaluation orders (the oracle's and the kernels') differ there by more than 1e-4 of the row.  Double accumulators and a
# bit-identical transmittance chain were both tried and do not move these rows (DESIGN.md); the small scenes keep the strict form.
FULL_SIZE = dict(min_rows=1.0 - 1e-4, row_cap=4.0, min_elementwise=0.999)


def _full_check(inp, seed, min_instances):
    o_out, o_st, gimg, o_grads = _oracle(inp, seed)
    assert o_st["num_rendered"] >= min_instances, o_st["num_rendered"]
    _check_forward_state(inp, o_out, o_st)  # includes the contributor masks, bit for bit
    _check_backward(inp, o_out, gimg, o_grads, criterion=FULL_SIZE)
    _check_backward_sums(inp, gimg, o_grads)  # the backward blend's sums: the derived bound, no exceptions
    return o_st


def test_config2_full_sample_ply_512():
    from humangaussian_b200.cameras import Camera, orbit_c2w
    from humangaussian_b200.scene import sample_ply_scene
    p = sample_ply_scene()
    assert p.P == 531327
    cam = Camera(orbit_c2w(15.0, 0.0, 2.0), math.radians(70.0), 512, 512)
    st = _full_check(_inputs(p, cam, 512, 512, 0), 21, 900000)
    lens = st["ranges"][:, 1] - st["ranges"][:, 0]
    assert lens.max() > 5000, "expected the deep tiles of the real scene"


@pytest.mark.parametrize("view", [0, 37])
def test_config4_300k_deg3_1024(view):
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.scene import sample_ply_scene
    p = sample_ply_scene(300000, 3)
    cam = sample_orbit_cameras(64, 1024, 1024, seed=1000)[view]  # the bench's camera set (rank 0)
    st = _full_check(_inputs(p, cam, 1024, 1024, 3), 22 + view, 500000)
    assert st["n_contrib"].max() > 2000, "deep early-terminated tiles expected"


def test_config3_100k_pcd_init_deg3_1024():
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.scene import params_from_pcd, sample_ply_scene, with_sh_degree
    src = sample_ply_scene(100000, 0)
    p = params_from_pcd(src.xyz, torch.full((100000, 3), 0.5), sh_degree=0, device=DEV)  # scales from this repo's distCUDA2
    p = with_sh_degree(p.to("cpu"), 3, seed=0)
    cam = sample_orbit_cameras(64, 1024, 1024, seed=1000)[5]
    _full_check(_inputs(p, cam, 1024, 1024, 3), 23, 200000)


def test_cuda_backward_vs_float64_autograd():
    """The CUDA backward against torch.autograd over the dense float64 formulation (oracle/dense_ref.py): no shared
    source with csrc/.  Integer decisions (radii, rects, order) come from the oracle, as in tests/test_oracle_autograd.py.
    Criterion: the north-star tolerance in the row-wise form (float32 sums vs float64)."""
    from oracle.dense_ref import dense_render
    from humangaussian_b200.rasterizer import GaussianRasterizer
    from test_gpu_parity import _gpu_inputs, _settings
    from util import small_scene
    from oracle.gs_oracle import Oracle
    for deg, seed, kw in ((3, 1, {}), (1, 9, dict(H=32, W=32, dist=1.3, opaque=True)), (2, 4, dict(H=48, W=48, fovy_deg=25.0, dist=1.1))):
        opaque = kw.pop("opaque", False)
        inp, _, _ = small_scene(P=400, deg=deg, seed=seed, **kw)
        if opaque:
            inp["opacities"] = np.clip(inp["opacities"] * 8, 0, 0.99999).astype(np.float32)
            inp["shs"][:, 0, :] -= 1.2
        H, W = inp["image_height"], inp["image_width"]
        o = Oracle(threads=1)
        col, radii, dep, alp = o.forward(**inp)
        st = o.state()
        gC, gD, gA = grad_images(H, W, seed)
        t64 = lambda a: torch.tensor(a, dtype=torch.float64)
        names = ("means3D", "opacities", "shs", "scales", "rotations")
        ten = {k: t64(inp[k]).requires_grad_(True) for k in names}
        m2d = torch.zeros(len(radii), 3, dtype=torch.float64, requires_grad=True)
        ids = np.nonzero(radii > 0)[0]
        order = ids[np.lexsort((ids, st["depths"][ids]))]
        c, d, a, _ = dense_render(means3D=ten["means3D"], means2D=m2d, opacities=ten["opacities"], viewmatrix=t64(inp["viewmatrix"]),
                                  projmatrix=t64(inp["projmatrix"]), campos=t64(inp["campos"]), bg=t64(inp["bg"]), H=H, W=W,
                                  tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], radii=radii, rect=st["rect"], order=order,
                                  sh_degree=deg, shs=ten["shs"], scales=ten["scales"], rotations=ten["rotations"])
        ((c * t64(gC)).sum() + (d * t64(gD)).sum() + (a * t64(gA)).sum()).backward()
        # CUDA side
        t = _gpu_inputs(inp)
        m2g = torch.zeros(len(radii), 3, device=DEV, requires_grad=True)
        cc, rr, dd, aa = GaussianRasterizer(_settings(inp))(means3D=t["means3D"], means2D=m2g, shs=t["shs"], opacities=t["opacities"],
                                                            scales=t["scales"], rotations=t["rotations"])
        assert np.abs(cc.detach().cpu().numpy() - c.detach().numpy()).max() < 2e-4  # float32 image vs float64 image
        g = lambda x: torch.tensor(x, device=DEV)
        ((cc * g(gC)).sum() + (dd * g(gD)).sum() + (aa * g(gA)).sum()).backward()
        for k in names:
            ref = ten[k].grad.numpy()
            # float32 kernels vs float64 autograd: 10x the north-star tolerance, as tests/test_oracle_autograd.py uses for
            # the float32 oracle (float32 rounding of the forward state enters the float32 side only)
            ok, msg = grads_agree(t[k].grad.cpu().numpy().reshape(ref.shape), ref, atol=1e-4, rtol=1e-3)
            assert ok, f"deg {deg}: dL/d{k} CUDA vs float64 autograd: {msg}"
        ok, msg = grads_agree(m2g.grad.cpu().numpy(), m2d.grad.numpy(), atol=1e-4, rtol=1e-3)
        assert ok, f"deg {deg}: dL/dmeans2D CUDA vs float64 autograd: {msg}"


def test_config5_animation_frames_full_sample_ply_1024():
    """BASELINE config 5 at its real size: content/sample.ply through the animation convention (gs_renderer.py:576-581;
    531 327 Gaussians), per-frame positions through the frame-batched entry, 1024x1024, MiniCam orbit (animation.py:993-1004:
    azimuth = frame index, fovy 50, radius 2): every uint8 frame equals the oracle's forward image after
    clamp(0,1) (gs_renderer.py:1017) and (x*255).astype(uint8) (animation.py:1011)."""
    from humangaussian_b200.animation import render_frames
    from humangaussian_b200.cameras import MiniCamC2W, orbit_c2w
    from humangaussian_b200.scene import sample_ply_scene
    from oracle.gs_oracle import Oracle
    p = sample_ply_scene(convention="animation")
    H = W = 1024
    fovy = math.radians(50.0)
    yup = np.eye(4, dtype=np.float32)[[0, 2, 1, 3]]
    frames_ids = (0, 77)
    cams = [MiniCamC2W(yup @ orbit_c2w(0.0, float(i), 2.0).numpy(), W, H, fovy, fovy, 0.01, 100.0, device=DEV) for i in frames_ids]
    g = torch.Generator().manual_seed(0)
    xyz = torch.stack([p.xyz, p.xyz + 0.002 * torch.randn(p.P, 3, generator=g)]).to(DEV)   # frame 1: displaced positions
    # the activations are evaluated ONCE (host libm and the device's expf differ in the last bit) and the same values feed both
    # sides: `pc` is anything with GaussianModel's getters
    import types
    with torch.no_grad():
        act = dict(get_opacity=p.get_opacity, get_features=p.get_features.contiguous(), get_scaling=p.get_scaling, get_rotation=p.get_rotation)
    pc = types.SimpleNamespace(active_sh_degree=0, **{k: v.to(DEV) for k, v in act.items()})
    frames = render_frames(pc, xyz, cams, torch.zeros(3, device=DEV)).cpu().numpy()
    assert frames.shape == (2, H, W, 3) and frames.dtype == np.uint8
    base = dict(opacities=act["get_opacity"].numpy(), shs=act["get_features"].numpy(), scales=act["get_scaling"].numpy(),
                rotations=act["get_rotation"].numpy(), sh_degree=0, bg=np.zeros(3, np.float32), image_height=H, image_width=W,
                tanfovx=math.tan(fovy * 0.5), tanfovy=math.tan(fovy * 0.5))
    for f, cam in enumerate(cams):
        o = Oracle()
        col, rad, dep, alp = o.forward(means3D=xyz[f].cpu().numpy(), viewmatrix=cam.world_view_transform.cpu().numpy(),
                                       projmatrix=cam.full_proj_transform.cpu().numpy(), campos=cam.camera_center.cpu().numpy(), **base)
        assert o.state()["num_rendered"] > 1000000
        want = (np.clip(col, 0.0, 1.0).transpose(1, 2, 0) * np.float32(255.0)).astype(np.uint8)
        assert np.array_equal(frames[f], want), f"frame {f}: {(frames[f] != want).sum()} bytes differ"
