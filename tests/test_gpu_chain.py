"""GPU: the per-Gaussian backward (B2+B3 and the normal chain) against its float64 chain rule, element by element.

Each case runs one forward and backward (rasterizer.forward_backward_with_state) and reads back the kernels' own inputs of
that call -- radii, clamp bits, geometry records, ScreenGrad sums, normal sums -- with the gradients it returned.
tests/chain_reference.py restates the chain on exactly those float32 inputs in float64, with a running bound e on the
error of float32 evaluation; every element of every gradient (means3D, per view with per-view means; scales; rotations;
opacities; SH or colours; cov3D_precomp; means2D of every view) must lie within K e of it.  No exceptions, no per-case
constants: the blend's float32 noise is out of the comparison, so what is left is the chain's own rounding.

Exact values: a Gaussian culled in every view gets exactly 0 in every parameter gradient, means2D rows of culled views are
0, and SH entries beyond the active degree are 0.

The table walks the 20 instantiations of preprocess_bwd_kernel (DEG -1..3 x AA x F3D) in the product library (moments
format), DEG -1..3 plain and with AA + F3D in the classic comparator (classic format), the deterministic backward,
raw and activated parameters, cov3D_precomp, scale_modifier 0.7, a stored degree above the active one, misaligned SH and
rotations (the scalar SH path), normals, P in {1, 127, 128, 129, 4099}, V in {1, 2, 3, 5}, per-view means, scenes built
to hit one branch each, with a coverage count that must be non-zero, and the benchmark's own step (BENCH: the raw 64-view,
300 k-Gaussian step, which drives the view prefetch across 64 views; about 19 M (view, Gaussian) records)."""
import contextlib
import math
import os

import numpy as np
import pytest
import torch

import chain_reference as CH
from util import ROOT, grad_images, small_scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
CLASSIC = os.path.join(ROOT, "baseline", "libb200gs_classic.so")
f32 = np.float32

DEFAULT = dict(lib="prod", det=False, deg=3, aa=False, f3d=False, raw=False, cov=False, mod=1.0, P=129, V=2, per_view=False,
               M=None, misalign=False, normals=False, scene="body", H=48, W=64)


def case(**kw):
    c = dict(DEFAULT, **kw)
    assert set(c) == set(DEFAULT)
    return c


CASES = (
    # the 20 instantiations, product library (moments), atomic backward
    [case(deg=g, aa=a, f3d=f, raw=bool((g + a + f) % 2)) for g in (-1, 0, 1, 2, 3) for a in (0, 1) for f in (0, 1)]
    # the classic comparator (classic format), plain and AA + F3D
    + [case(lib="classic", deg=g, aa=a, f3d=a, raw=bool(g % 2)) for g in (-1, 0, 1, 2, 3) for a in (0, 1)]
    # the deterministic backward (the product library's; the classic comparator has none)
    + [case(det=True, deg=3, aa=1, f3d=1, raw=True, V=3), case(det=True, deg=-1, cov=True, V=3)]
    # paths
    + [case(cov=True, deg=0), case(cov=True, deg=-1, aa=1, mod=0.7), case(mod=0.7, raw=True, aa=1, f3d=1),
       case(deg=1, M=16, raw=True), case(deg=3, misalign=True, raw=True), case(deg=1, misalign=True, aa=1),
       case(normals=True, raw=True, V=3), case(normals=True, aa=1, f3d=1, deg=1, per_view=True, V=3)]
    # shapes
    + [case(P=p, V=v, raw=True, aa=int(p % 2)) for p, v in ((1, 1), (127, 2), (128, 3), (4099, 5), (129, 1))]
    + [case(P=300, V=3, per_view=True, raw=True), case(P=300, V=3, per_view=True, deg=-1, f3d=1)]
    # scenes built to hit one branch each
    + [case(scene="guard", deg=1, raw=True), case(scene="guard", deg=0, aa=1, lib="classic"),
       case(scene="clamp", deg=1), case(scene="clamp", deg=3, raw=True),
       case(scene="subsets", V=3, raw=True, deg=1), case(scene="subsets", V=3, normals=True, aa=1),
       case(scene="closeup", V=2, raw=True, H=128, W=128), case(scene="near", raw=True, deg=2),
       case(scene="needles", aa=1, deg=0, V=1), case(scene="needles", aa=1, raw=True, deg=1, V=2),
       case(scene="f3d_zero", f3d=1, deg=1), case(scene="f3d_zero", f3d=1, aa=1, deg=0),
       case(scene="quat", raw=True, deg=1), case(scene="quat", raw=True, normals=True, deg=0)]
)


def case_id(c):
    d = {k: v for k, v in c.items() if v != DEFAULT[k]}
    return "-".join(f"{k}{'' if v is True else v}" for k, v in d.items()) or "default"


# ---- scenes -----------------------------------------------------------------------------------------------------------------
def _orbit_views(V, H, W, seed=5, **kw):
    from humangaussian_b200.cameras import sample_orbit_cameras
    return [dict(viewmatrix=c.world_view_transform.numpy().astype(f32), projmatrix=c.full_proj_transform.numpy().astype(f32),
                 campos=c.camera_center.numpy().astype(f32), tanfovx=math.tan(c.FoVx * 0.5), tanfovy=math.tan(c.FoVy * 0.5))
            for c in sample_orbit_cameras(V, H, W, seed=seed, **kw)]


def _shift_views(V, H, W, shifts, fovy_deg=60.0):
    """cameras at `shifts[v]` looking down +z (identity rotation)"""
    from humangaussian_b200.cameras import getProjectionMatrix
    tany = math.tan(math.radians(fovy_deg) / 2)
    tanx = tany * W / H
    proj = getProjectionMatrix(0.01, 100.0, 2 * math.atan(tanx), 2 * math.atan(tany)).transpose(0, 1).numpy().astype(np.float64)
    out = []
    for v in range(V):
        t = np.asarray(shifts[v], np.float64)
        vm = np.eye(4)
        vm[3, :3] = -t
        out.append(dict(viewmatrix=vm.astype(f32), projmatrix=(vm @ proj).astype(f32), campos=t.astype(f32), tanfovx=tanx,
                        tanfovy=tany))
    return out


def _unit_quats(rng, n, spread=1.0):
    q = rng.randn(n, 4) * spread
    q[:, 0] += 1.0
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def _to_world(cam, pc):
    """camera-space points of a view -> world (the view matrix is stored transposed: p_cam = [p, 1] @ vm)"""
    inv = np.linalg.inv(cam["viewmatrix"].astype(np.float64))
    return (np.concatenate([pc, np.ones((len(pc), 1))], 1) @ inv)[:, :3]


def make_scene(c):
    """activated parameters (float32 numpy) and the views of case c; SH stored for degree 3 unless c says otherwise"""
    P, V, H, W = c["P"], c["V"], c["H"], c["W"]
    rng = np.random.RandomState(1000 + P + 7 * V)
    scene = c["scene"]
    if scene in ("body", "closeup", "near", "quat", "f3d_zero", "clamp"):
        inp, _, _ = small_scene(P=P, deg=3, seed=P % 17, H=H, W=W, big=P < 1000)
        p = dict(means3D=inp["means3D"], scales=inp["scales"], rotations=inp["rotations"], opacities=inp["opacities"].reshape(P),
                 shs=inp["shs"])
        views = _orbit_views(V, H, W, seed=5 + P)
        if scene == "closeup":  # footprints of 10^6 px^2 and more: large Gaussians a short way from the camera
            views = _orbit_views(V, H, W, seed=9, distance_range=(0.3, 0.35))
            p["scales"] = (p["scales"] * 8).astype(f32)
        if scene == "near":  # view depth just above the near plane (0.2) in view 0
            cam = views[0]
            pc = np.stack([rng.uniform(-0.05, 0.05, P), rng.uniform(-0.05, 0.05, P), 0.2 + rng.uniform(1e-6, 2e-2, P)], 1)
            p["means3D"] = _to_world(cam, pc).astype(f32)
            p["scales"] = np.full((P, 3), 0.004, f32) * rng.uniform(0.5, 2, (P, 3)).astype(f32)
        if scene == "clamp":  # each channel clamped on its own in a quarter of the Gaussians (from the DC term)
            sh = p["shs"].copy()
            sh[:, 1:] *= 0.05
            sh[:, 0] = 1.0
            ch = np.arange(P) % 4
            sh[np.nonzero(ch < 3)[0], 0, ch[ch < 3]] = -3.0
            p["shs"] = sh.astype(f32)
        if scene == "f3d_zero":  # activated scales of exactly 0 (one axis) and some zero filter variances (set in run_case)
            s = p["scales"].copy()
            s[::3, 0] = 0.0
            s[1::5, 2] = 0.0
            p["scales"] = s
        if scene == "quat":  # raw quaternions of norm 1e-13, 1e-3, 1e3 (and 1)
            q = _unit_quats(rng, P, 0.4) * np.array([1e-13, 1e-3, 1e3, 1.0])[np.arange(P) % 4, None]
            p["rotations"] = q.astype(f32)
    elif scene == "guard":  # centres beyond +-1.3 tan(fov) in x (half) and in y (half), wide enough to reach the image
        views = _orbit_views(V, H, W, seed=21)
        cam = views[0]
        z = rng.uniform(1.0, 2.0, P)
        side = np.where(rng.rand(P) < 0.5, -1.0, 1.0)
        on_x = np.arange(P) % 2 == 0
        ax = np.where(on_x, side * rng.uniform(1.35, 1.8, P) * cam["tanfovx"], rng.uniform(-0.5, 0.5, P) * cam["tanfovx"])
        ay = np.where(~on_x, side * rng.uniform(1.35, 1.8, P) * cam["tanfovy"], rng.uniform(-0.5, 0.5, P) * cam["tanfovy"])
        pc = np.stack([ax * z, ay * z, z], 1)
        p = dict(means3D=_to_world(cam, pc).astype(f32), scales=(rng.uniform(0.2, 0.5, (P, 3)) * z[:, None]).astype(f32),
                 rotations=_unit_quats(rng, P).astype(f32), opacities=rng.uniform(0.2, 0.9, P).astype(f32),
                 shs=(0.3 * rng.randn(P, 16, 3)).astype(f32))
    elif scene == "subsets":  # three shifted cameras: every visibility subset of the three views occurs
        views = _shift_views(V, H, W, [(0, 0, 0), (1.2, 0, 0), (0.6, 0.9, 0)])
        P = c["P"]
        pm = np.stack([rng.uniform(-3.5, 4.5, P), rng.uniform(-3.0, 3.8, P), rng.uniform(3, 5, P)], 1)
        p = dict(means3D=pm.astype(f32), scales=rng.uniform(0.02, 0.12, (P, 3)).astype(f32),
                 rotations=_unit_quats(rng, P).astype(f32), opacities=rng.uniform(0.2, 0.9, P).astype(f32),
                 shs=(0.3 * rng.randn(P, 16, 3)).astype(f32))
    elif scene == "needles":  # screen-space needles whose det0 / det is near antialiasing's floor 2.5e-5
        views = _orbit_views(V, H, W, seed=33)
        cam = views[0]
        z = rng.uniform(1.5, 2.5, P)
        pc = np.stack([rng.uniform(-0.5, 0.5, P) * cam["tanfovx"] * z, rng.uniform(-0.5, 0.5, P) * cam["tanfovy"] * z, z], 1)
        fx = W / (2 * cam["tanfovx"])
        # long axis ~ 6 px, thin axis sigma with (f sigma / z)^2 / 0.3 around 2.5e-5, at 45 degrees in the image plane
        thin = np.sqrt(0.3 * 2.5e-5 * rng.uniform(0.7, 1.4, P)) * z / fx
        s = np.stack([6.0 * z / fx, thin, thin], 1)
        ang = np.pi / 4 + rng.uniform(-0.05, 0.05, P)
        qc = np.stack([np.cos(ang / 2), np.zeros(P), np.zeros(P), np.sin(ang / 2)], 1)  # about the view axis
        # camera-space rotation -> world: R_world = R_c2w R_cam
        c2w = np.linalg.inv(cam["viewmatrix"].astype(np.float64)).T[:3, :3]
        from scipy.spatial.transform import Rotation
        Rw = Rotation.from_matrix(c2w) * Rotation.from_quat(np.stack([qc[:, 1], qc[:, 2], qc[:, 3], qc[:, 0]], 1))
        xyzw = Rw.as_quat()
        p = dict(means3D=_to_world(cam, pc).astype(f32), scales=s.astype(f32),
                 rotations=np.stack([xyzw[:, 3], xyzw[:, 0], xyzw[:, 1], xyzw[:, 2]], 1).astype(f32),
                 opacities=rng.uniform(0.3, 0.9, P).astype(f32), shs=(0.3 * rng.randn(P, 16, 3)).astype(f32))
    elif scene == "bench":  # the benchmark's step: its raw scene and cameras (bench_step_reference)
        import bench_step_reference as BS
        args = BS.bench_args()
        assert (V, H, W) == (args.views, args.res, args.res)
        raw = BS.raw_of_params(BS.bench_scene(args))
        views = [BS.cam_inputs(cm) for cm in BS.bench_cameras(args)]
        p = dict(means3D=raw["xyz"], shs=raw["shs"],
                 raw=dict(opacities=raw["opacities"], scales=raw["scales"], rotations=raw["rotations"]))
    else:
        raise ValueError(scene)
    return p, views


# ---- one call ---------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _mode(c):
    import humangaussian_b200.rasterizer as R
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(bool(c["det"]))
    try:
        if c["lib"] == "classic":
            with R.use_library(CLASSIC):
                yield
        else:
            yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _device_activate(raw_op, raw_s):
    """F1's activations bit for bit: torch's exp on the device (expf) and 1 / (1 + expf(-x)) in float32"""
    e = torch.exp(-torch.tensor(raw_op, device=DEV)).cpu().numpy()
    op = (f32(1) / (f32(1) + e)).astype(f32)
    s = None if raw_s is None else torch.exp(torch.tensor(raw_s, device=DEV)).cpu().numpy()
    return op, s


def _misaligned(a):
    """a contiguous device copy of `a` whose data pointer is 4 bytes past a 16-byte boundary"""
    flat = torch.zeros(a.size + 4, dtype=torch.float32, device=DEV)
    flat[1:1 + a.size] = torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).to(DEV)
    t = flat[1:1 + a.size].view(*a.shape)
    assert t.data_ptr() % 16 == 4
    return t


def run_case(c):
    """(reference inputs d for chain_reference.chain, the kernels' gradients {name: numpy}, radii [V,P])"""
    import normal_reference as NR
    from humangaussian_b200.rasterizer import forward_backward_with_state
    p, views = make_scene(c)
    P, V, H, W, deg = len(p["means3D"]), c["V"], c["H"], c["W"], c["deg"]
    rng = np.random.RandomState(77 + P + V)
    nb = (deg + 1) ** 2 if deg >= 0 else 0
    M = c["M"] or nb
    means = np.stack([p["means3D"]] * V)
    if c["per_view"]:
        means = (means + 0.01 * rng.randn(*means.shape)).astype(f32)
    raw = c["raw"]
    par = {}
    if "raw" in p:  # the scene's own raw parameters
        raw_op, raw_s, q_in = p["raw"]["opacities"].reshape(P), p["raw"]["scales"], p["raw"]["rotations"]
    else:
        s_act, q_in, op = p["scales"].astype(f32), p["rotations"].astype(f32), p["opacities"].astype(f32)
    if raw:
        if "raw" not in p:
            raw_op = np.log(op.astype(np.float64) / (1 - op)).astype(f32)
            with np.errstate(divide="ignore"):
                raw_s = np.log(s_act.astype(np.float64)).astype(f32)
            if c["scene"] != "quat":
                q_in = (q_in * 1.3).astype(f32)
        op, s_act = _device_activate(raw_op, raw_s)
        par.update(opacities=raw_op.reshape(P, 1), scales=raw_s, rotations=q_in)
        qhat, qnorm, qlen = CH.normalize32(q_in)
    else:
        par.update(opacities=op.reshape(P, 1), scales=s_act, rotations=q_in)
        qhat, qnorm, qlen = q_in, np.ones(P, f32), np.ones(P, f32)
    cov = None
    if c["cov"]:
        from scipy.spatial.transform import Rotation
        R = Rotation.from_quat(np.stack([qhat[:, 1], qhat[:, 2], qhat[:, 3], qhat[:, 0]], 1)).as_matrix()
        S = R * s_act.astype(np.float64)[:, None, :]
        Sig = S @ S.transpose(0, 2, 1)
        cov = Sig[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(f32)
        del par["scales"], par["rotations"]
    var = None
    if c["f3d"]:
        var = (0.3 * rng.uniform(0, 1, P) * s_act.astype(np.float64).mean(1) ** 2).astype(f32)
        if c["scene"] == "f3d_zero":
            var[::2] = 0.0
    shs = colors = None
    if deg >= 0:
        shs = np.ascontiguousarray(p["shs"][:, :M]).astype(f32)
    else:
        colors = rng.uniform(0.1, 0.9, (P, 3)).astype(f32)
    if V * H * W > 1 << 24:  # the benchmark's shape: the image gradients drawn on the device
        gen = torch.Generator(device=DEV).manual_seed(P)
        gimgs = [torch.randn(V, ch, H, W, device=DEV, generator=gen) for ch in (3, 1, 1)]
    else:
        gimgs = [np.stack([grad_images(H, W, 3 * v + P)[j] for v in range(V)]) for j in range(3)]
    gN = rng.randn(V, 3, H, W).astype(f32) if c["normals"] else None

    T = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    kw = {k: T(v) for k, v in par.items()}
    if c["misalign"]:
        kw["rotations"] = _misaligned(par["rotations"])
    kw.update(means3D=T(means if c["per_view"] else p["means3D"]), cov3D_precomp=T(cov), colors_precomp=T(colors),
              shs=_misaligned(shs) if c["misalign"] and shs is not None else T(shs))
    st = lambda k: np.stack([np.asarray(v[k], f32) for v in views])
    vm, pm, cp = st("viewmatrix").reshape(V, 16), st("projmatrix").reshape(V, 16), st("campos").reshape(V, 3)
    tanx, tany = [v["tanfovx"] for v in views], [v["tanfovy"] for v in views]
    with _mode(c):
        outs = forward_backward_with_state(
            *(g if torch.is_tensor(g) else T(g) for g in gimgs),
            g_normal=T(gN), viewmatrix=T(vm).reshape(V, 4, 4), projmatrix=T(pm).reshape(V, 4, 4), campos=T(cp),
            tanfovx=tanx, tanfovy=tany, image_height=H, image_width=W, bg=T(np.array([0.1, 0.4, 0.7], f32)),
            sh_degree=max(deg, 0), scale_modifier=c["mod"], raw=raw, antialiasing=bool(c["aa"]), filter_3d=T(var),
            normals=c["normals"], **kw)
    state, sums = outs[-2], outs[-1]
    radii = outs[1].cpu().numpy().reshape(V, P)
    dm3, dm2, dsh, dcol, dop, dsc, drot, dcov = (None if g is None else g.cpu().numpy() for g in state["grads"])
    op_prime = op if var is None else (op * CH.filter3d32(s_act, var)[3]).astype(f32)
    d = dict(P=P, V=V, H=H, W=W, deg=deg, M=M, mod=c["mod"], raw=raw, aa=bool(c["aa"]), moments=c["lib"] == "prod",
             means=means, per_view=c["per_view"], view=vm, proj=pm, campos=cp, tanx=np.array(tanx, f32), tany=np.array(tany, f32),
             op=op, op_prime=op_prime, s=s_act, q=q_in, qhat=qhat, qnorm=qnorm, qlen=qlen, cov=cov, var=var, shs=shs,
             radii=radii, clamped=state["clamped"].cpu().numpy().reshape(V, P), recs=state["recs"].cpu().numpy().reshape(V, P, 12),
             sums=sums.cpu().numpy(), diag=[])
    if c["normals"]:
        d["normals"] = dict(sign=state["gauss_normals"].cpu().numpy().reshape(V, P, 4)[..., 3],
                            wn=state["normal_wn"].cpu().numpy()[..., :3], axis=NR.axis(s_act))
    got = dict(means3D=dm3, means2D=dm2, opacities=dop.reshape(P))
    if deg >= 0:
        got["shs"] = dsh
    else:
        got["colors"] = dcol
    if cov is not None:
        got["cov3D"] = dcov
    else:
        got.update(scales=dsc, rotations=drot)
    return d, got


def coverage(c, d):
    """the count of (view, Gaussian) pairs that take the branch the case's scene is built for"""
    vis = d["radii"] > 0
    scene = c["scene"]
    if scene == "guard":
        bx, by = CH.guard_band(d["means"][0], d["view"][0], d["tanx"][0], d["tany"][0])
        return dict(xmul0=int((vis[0] & (bx != 0)).sum()), ymul0=int((vis[0] & (by != 0)).sum()))
    if scene == "clamp":
        return {f"clamp{b}": int((vis & (d["clamped"] == b)).sum()) for b in (1, 2, 4)}
    if scene == "subsets":
        pat = (vis * np.array([1, 2, 4])[:, None]).sum(0)
        return {f"subset{k}": int((pat == k).sum()) for k in range(8)}
    if scene == "closeup":
        return dict(footprint_1e6=int((vis & ((2.0 * d["radii"]) ** 2 >= 1e6)).sum()))
    if scene == "near":
        tz = CH.affine32(d["view"][0][[2, 6, 10, 14]], *(d["means"][0][:, k] for k in range(3)))
        return dict(near=int((vis[0] & (tz < 0.21)).sum()))
    if scene == "needles":
        n = 0
        for v, r, e, rad in d["diag"]:
            n += int((rad & (np.abs(r - CH.RHO_FLOOR) <= e)).sum())
        floored = int((vis & d["floored"]).sum())
        return dict(ratio_within_rounding=n, floored=floored, unfloored=int(vis.sum()) - floored)
    if scene == "f3d_zero":
        seen = vis.any(0)
        return dict(var0=int((seen & (d["var"] == 0)).sum()), scale0=int((seen & (d["s"] == 0).any(1)).sum()))
    if scene == "quat":
        n = np.linalg.norm(d["q"].astype(np.float64), axis=1)
        seen = vis.any(0)
        return {f"qnorm{x:g}": int((seen & (np.abs(np.log10(n) - np.log10(x)) < 0.5)).sum()) for x in (1e-13, 1e-3, 1e3)}
    return {}


# the benchmark's step: raw parameters, 64 views of 300 k Gaussians at its resolution, the reference one view at a time
BENCH = case(scene="bench", raw=True, deg=3, P=300000, V=64, H=1024, W=1024)


@pytest.mark.parametrize("c", CASES + [BENCH], ids=case_id)
def test_chain(c):
    d, got = run_case(c)
    ref = CH.arrays(CH.chain(d))
    name = case_id(c)
    P, V = d["P"], d["V"]
    vis = d["radii"] > 0
    assert vis.any(), f"{name}: nothing visible"
    worst = {}
    for k, r in ref.items():
        g = got[k]
        if k == "shs":
            nb = r[0].shape[1]
            assert (g[:, nb:] == 0).all(), f"{name}: SH gradients beyond the active degree are not 0"
            g = g[:, :nb]
        worst[k] = CH.check(g, r, f"{name} {k}")[0]
    # exact zeros: culled in every view -> every parameter gradient row; a culled view -> its means2D row
    gone = ~vis.any(0)
    for k, g in got.items():
        if k == "means2D":
            assert (g[~vis] == 0).all(), f"{name}: means2D rows of culled views are not 0"
        elif g.ndim == 3 and k == "means3D":
            assert (g[:, gone] == 0).all(), f"{name}: {k} of Gaussians culled in every view is not 0"
        else:
            assert (g.reshape(P, -1)[gone] == 0).all(), f"{name}: {k} of Gaussians culled in every view is not 0"
    cov = coverage(c, d)
    for k, n in cov.items():
        assert n > 0, f"{name}: the scene no longer covers {k}"
    print(f"\n{name}: worst |gpu - ref| / (K e) " + ", ".join(f"{k} {w:.3g}" for k, w in worst.items()) +
          (f"; coverage {cov}" if cov else "") + f"; culled everywhere {int(gone.sum())}")
