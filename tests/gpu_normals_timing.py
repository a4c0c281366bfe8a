"""Timing of the normal maps (rasterize_views_packed(normals=True)) against the default and the two-pass workaround.  Not a
test.

    python tests/gpu_normals_timing.py [out.json]

Workloads: the bench's (300 k Gaussians of sample.ply, SH degree 3, 1024^2, its 64 cameras) and the 8-view SDS batch (the
first 8 of them); one step = forward + backward with random image gradients (and a random normal gradient).  Arms:
  plain       rasterize_views_packed(raw=True), colour / depth / alpha;
  normals     the same call with normals=True and a normal gradient;
  workaround  the plain call plus, per view, a second rasterize_views pass with colors_precomp = that view's camera-facing
              normals (a torch expression of the raw rotations and scales) and bg = 0 -- the only way to a differentiable
              normal map without normals=True.
Alternated in 5 windows of 3 steps after warm-up, CUDA events, median and spread; per-stage CUDA-event times of one step of
plain and normals.  The card's name, power limit and clocks are read before and after."""
import json
import statistics
import sys

import torch

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
from gpu_antialias_timing import card, events_ms  # noqa: E402
from humangaussian_b200 import dist as D  # noqa: E402
from humangaussian_b200 import rasterizer as R  # noqa: E402


def facing_normals(xyz, scaling, rotation, campos):
    """[V,P,3] world-space normals of the shortest axis, flipped toward each camera (torch; differentiable in the rotation)"""
    q = torch.nn.functional.normalize(rotation, dim=1)
    r, x, y, z = q.unbind(1)
    Rm = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                      2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                      2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    k = scaling.detach().argmin(1)
    n = Rm[torch.arange(len(q), device=q.device), :, k]
    sg = torch.where(((campos[:, None, :] - xyz.detach()[None]) * n.detach()[None]).sum(-1) < 0, -1.0, 1.0)
    return n[None] * sg[..., None]


def workload(V, flat, P, K, cams, g):
    vm, pm, cp, tx, ty = cams
    gw = [torch.randn(V, c, 1024, 1024, device="cuda", generator=g) for c in (3, 1, 1, 3)]
    bg, zero = torch.zeros(3, device="cuda"), torch.zeros(3, device="cuda")
    kw = lambda s: dict(viewmatrices=vm[s], projmatrices=pm[s], camposs=cp[s], tanfovx=tx[s], tanfovy=ty[s], image_height=1024,
                        image_width=1024)

    def step(arm):
        flat.grad = None
        if arm == "workaround":
            c, r, d, a = R.rasterize_views_packed(flat, P, K, bg=bg, sh_degree=3, raw=True, **kw(slice(0, V)))
            xyz, sc, rot, op, _ = R._split_packed(flat, P, K)
            n = facing_normals(xyz, sc, rot, cp[:V])
            imgs = [R.rasterize_views(means3D=xyz, opacities=op, colors_precomp=n[v], scales=sc, rotations=rot, raw=True, bg=zero,
                                      **kw(slice(v, v + 1)))[0] for v in range(V)]
            torch.autograd.backward([c, d, a, torch.cat(imgs, 0)], gw)
            return
        outs = R.rasterize_views_packed(flat, P, K, bg=bg, sh_degree=3, raw=True, normals=arm == "normals", **kw(slice(0, V)))
        torch.autograd.backward([outs[0], outs[2], outs[3]] + ([outs[4]] if arm == "normals" else []), gw[:len(outs) - 1])
    return step


def measure(step, n=3, windows=5):
    arms = ("plain", "normals", "workaround")
    for arm in arms:
        for _ in range(2):
            step(arm)
    torch.cuda.synchronize()
    t = {arm: [] for arm in arms}
    for _ in range(windows):
        for arm in arms:
            t[arm].append(events_ms(lambda: step(arm), n))
    stages = {}
    for arm in arms[:2]:
        torch.cuda.synchronize()
        R.profile_read()
        R.profile_enable(True)
        step(arm)
        torch.cuda.synchronize()
        R.profile_enable(False)
        stages[arm] = {k: round(v[0], 3) for k, v in R.profile_read().items()}
    med = {a: statistics.median(v) for a, v in t.items()}
    return dict(ms=med, spread_ms={a: [round(min(v), 3), round(max(v), 3)] for a, v in t.items()},
                normals_over_plain=med["normals"] / med["plain"], workaround_over_normals=med["workaround"] / med["normals"],
                stage_ms_one_step=stages)


def main():
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import stack_cameras
    from humangaussian_b200.scene import sample_ply_scene
    before = card()
    P, deg = 300_000, 3
    K = (deg + 1) ** 2
    sc = sample_ply_scene(P, deg, seed=0)
    raw = dict(xyz=sc.xyz, scaling=sc.scaling, rotation=sc.rotation, opacity=sc.opacity,
               features=torch.cat((sc.features_dc, sc.features_rest), 1))
    flat = D.pack({k: v.detach().float().cuda().contiguous() for k, v in raw.items()}).requires_grad_(True)
    cams = stack_cameras(sample_orbit_cameras(64, 1024, 1024, seed=1000, device="cpu"), "cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card_before": before, "P": P, "sh_degree": deg, "resolution": 1024}
    for V in (8, 64):
        res[f"views{V}"] = measure(workload(V, flat, P, K, cams, g))
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
