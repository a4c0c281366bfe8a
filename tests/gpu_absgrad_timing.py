"""Timing of the absolute screen-space gradient (rasterize_views_packed(means2D_abs=...)) against the default.  Not a test.

    python tests/gpu_absgrad_timing.py [out.json]

Workloads: the bench's (300 k Gaussians of sample.ply, SH degree 3, 1024^2, its 64 cameras) and the 8-view SDS batch (the
first 8 of them); one step = rasterize_views_packed(raw=True) forward + backward, as bench.py times it, in the atomic and in
the deterministic backward (torch.use_deterministic_algorithms).  Arms (absgrad off, on) alternated in 5 windows of 5 steps
after warm-up, CUDA events, median and spread (min..max of the windows).  Reported alongside: the library's per-stage
CUDA-event times of one step (blend_bwd holds B1, the deterministic pre-pass and reduce, and absgrad's output pass).  The
card's name, power limit and clocks are read before and after.
"""
import json
import statistics
import sys

import torch

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
from gpu_antialias_timing import card, events_ms  # noqa: E402
from humangaussian_b200 import dist as D  # noqa: E402
from humangaussian_b200 import rasterizer as R  # noqa: E402


def workload(V, flat, P, K, cams, g):
    vm, pm, cp, tx, ty = cams
    gw = [torch.randn(V, c, 1024, 1024, device="cuda", generator=g) for c in (3, 1, 1)]
    bg = torch.zeros(3, device="cuda")
    m2a = torch.zeros(V, P, 3, device="cuda", requires_grad=True)

    def step(on):
        flat.grad = None
        m2a.grad = None
        c, r, d, a = R.rasterize_views_packed(flat, P, K, viewmatrices=vm[:V], projmatrices=pm[:V], camposs=cp[:V], tanfovx=tx[:V],
                                              tanfovy=ty[:V], image_height=1024, image_width=1024, bg=bg, sh_degree=3, raw=True,
                                              means2D_abs=m2a if on else None)
        torch.autograd.backward([c, d, a], gw)
    return step


def measure(step, det, n=5, windows=5):
    arms = (False, True)
    torch.use_deterministic_algorithms(det)
    try:
        for on in arms:
            for _ in range(2):
                step(on)
        torch.cuda.synchronize()
        t = {on: [] for on in arms}
        for _ in range(windows):
            for on in arms:
                t[on].append(events_ms(lambda: step(on), n))
        stages = {}
        for on in arms:
            torch.cuda.synchronize()
            R.profile_read()
            R.profile_enable(True)
            step(on)
            torch.cuda.synchronize()
            R.profile_enable(False)
            stages[on] = {k: round(v[0], 3) for k, v in R.profile_read().items()}
    finally:
        torch.use_deterministic_algorithms(False)
    name = {False: "off", True: "absgrad"}
    return dict(ms={name[a]: statistics.median(v) for a, v in t.items()},
                spread_ms={name[a]: [round(min(v), 3), round(max(v), 3)] for a, v in t.items()},
                windows_ms={name[a]: [round(x, 3) for x in v] for a, v in t.items()},
                absgrad_over_off=statistics.median(t[True]) / statistics.median(t[False]),
                stage_ms_one_step={name[a]: s for a, s in stages.items()})


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
    for V in (64, 8):
        step = workload(V, flat, P, K, cams, g)
        for det in (False, True):
            res[f"views{V}_{'deterministic' if det else 'atomic'}"] = measure(step, det)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
