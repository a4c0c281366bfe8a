"""Timing of the geometry outputs (rasterize_views_packed(geometry=True)) against the default and the two-pass workaround for
M2.  Not a test.

    python tests/gpu_geometry_timing.py [out.json]

Workloads: the bench's (300 k Gaussians of sample.ply, SH degree 3, 1024^2, its 64 cameras) and the 8-view SDS batch (the
first 8 of them); one step = forward + backward with random image gradients (and random median / depth2 gradients).  Arms:
  plain       rasterize_views_packed(raw=True), colour / depth / alpha;
  geometry    the same call with geometry=True and gradients on both new images;
  workaround  the plain call plus, per view, a second rasterize_views pass with colors_precomp = (z^2, 0, 0) (z the view-space
              depth of each mean, a torch expression) and bg = 0 -- the way to a differentiable M2 without geometry=True
              (the median has no workaround).  Each second pass runs its backward at once, so 64 of them fit in memory.
Alternated in 5 windows of 3 steps after warm-up, CUDA events, median and spread; per-stage CUDA-event times of one step of
plain and geometry.  The card's name, power limit and clocks are read before and after."""
import gc
import json
import statistics
import sys

import torch

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
from gpu_antialias_timing import card, events_ms  # noqa: E402
from humangaussian_b200 import dist as D  # noqa: E402
from humangaussian_b200 import rasterizer as R  # noqa: E402

ARMS = ("plain", "geometry", "workaround")


def workload(V, flat, P, K, cams, g):
    vm, pm, cp, tx, ty = cams
    gw = [torch.randn(V, c, 1024, 1024, device="cuda", generator=g) for c in (3, 1, 1, 1, 1)]
    bg, zero = torch.zeros(3, device="cuda"), torch.zeros(3, device="cuda")
    kw = lambda s: dict(viewmatrices=vm[s], projmatrices=pm[s], camposs=cp[s], tanfovx=tx[s], tanfovy=ty[s], image_height=1024,
                        image_width=1024)

    def step(arm):
        flat.grad = None
        if arm == "workaround":
            c, r, d, a = R.rasterize_views_packed(flat, P, K, bg=bg, sh_degree=3, raw=True, **kw(slice(0, V)))
            torch.autograd.backward([c, d, a], gw[:3])
            for v in range(V):
                xyz, sc, rot, op, _ = R._split_packed(flat, P, K)
                z = xyz @ vm[v, :3, 2] + vm[v, 3, 2]
                col = torch.stack([z * z, torch.zeros_like(z), torch.zeros_like(z)], 1)
                img = R.rasterize_views(means3D=xyz, opacities=op, colors_precomp=col, scales=sc, rotations=rot, raw=True,
                                        bg=zero, **kw(slice(v, v + 1)))[0][:, :1]
                img.backward(gw[3][v:v + 1])
            return
        geo = arm == "geometry"
        outs = R.rasterize_views_packed(flat, P, K, bg=bg, sh_degree=3, raw=True, geometry=geo, **kw(slice(0, V)))
        torch.autograd.backward([outs[0], outs[2], outs[3]] + ([outs[4], outs[5]] if geo else []), gw[:len(outs) - 1])
    return step


def fresh():
    """drop the parked state buffers of the other arms (outside the timed region): 64 per-view and one 64-view set do not
    fit beside each other"""
    gc.collect()
    R.release_cached_buffers()
    torch.cuda.empty_cache()


def measure(step, n=3, windows=5):
    for arm in ARMS:
        for _ in range(2):
            step(arm)
    torch.cuda.synchronize()
    t = {arm: [] for arm in ARMS}
    for _ in range(windows):
        for arm in ARMS:
            fresh()
            t[arm].append(events_ms(lambda: step(arm), n))
    stages = {}
    for arm in ARMS[:2]:
        torch.cuda.synchronize()
        R.profile_read()
        R.profile_enable(True)
        step(arm)
        torch.cuda.synchronize()
        R.profile_enable(False)
        stages[arm] = {k: round(v[0], 3) for k, v in R.profile_read().items()}
    med = {a: statistics.median(v) for a, v in t.items()}
    return dict(ms=med, spread_ms={a: [round(min(v), 3), round(max(v), 3)] for a, v in t.items()},
                geometry_over_plain=med["geometry"] / med["plain"], workaround_over_geometry=med["workaround"] / med["geometry"],
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
        fresh()
        try:
            res[f"views{V}"] = measure(workload(V, flat, P, K, cams, g))
        except torch.OutOfMemoryError as e:
            res[f"views{V}"] = {"error": str(e).split(".")[0]}
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
