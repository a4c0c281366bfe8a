"""Timing of the antialiasing filter (rasterize_views_packed(antialiasing=True)) against the default.  Not a test.

    python tests/gpu_antialias_timing.py [out.json]

Workloads: the bench's (300 k Gaussians of sample.ply, SH degree 3, 1024^2, its 64 cameras) and the 8-view SDS batch (the
first 8 of them); one step = rasterize_views_packed(raw=True) forward + backward, as bench.py times it.  Arms (filter off,
on) alternated in 5 windows of 5 steps after warm-up, CUDA events, median and spread (min..max of the windows).  Reported
alongside: the instance count D of each arm (the filter lowers the record opacities, so the support boxes shrink), and the
library's per-stage CUDA-event times of one step.  The card's name, power limit and clocks are read before and after.
"""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from humangaussian_b200 import dist as D  # noqa: E402
from humangaussian_b200 import rasterizer as R  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def events_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def workload(V, flat, P, K, cams, g):
    vm, pm, cp, tx, ty = cams
    gw = [torch.randn(V, c, 1024, 1024, device="cuda", generator=g) for c in (3, 1, 1)]
    bg = torch.zeros(3, device="cuda")

    def step(aa):
        flat.grad = None
        c, r, d, a = R.rasterize_views_packed(flat, P, K, viewmatrices=vm[:V], projmatrices=pm[:V], camposs=cp[:V], tanfovx=tx[:V],
                                              tanfovy=ty[:V], image_height=1024, image_width=1024, bg=bg, sh_degree=3, raw=True,
                                              antialiasing=aa)
        torch.autograd.backward([c, d, a], gw)
    return step


def measure(step, n=5, windows=5):
    arms = (False, True)
    for aa in arms:
        for _ in range(2):
            step(aa)
    torch.cuda.synchronize()
    t = {aa: [] for aa in arms}
    for _ in range(windows):
        for aa in arms:
            t[aa].append(events_ms(lambda: step(aa), n))
    stages, inst = {}, {}
    for aa in arms:
        torch.cuda.synchronize()
        R.profile_read()
        R.profile_enable(True)
        step(aa)
        torch.cuda.synchronize()
        R.profile_enable(False)
        stages[aa] = {k: round(v[0], 3) for k, v in R.profile_read().items()}
        inst[aa] = R.last_num_rendered()
    name = {False: "off", True: "aa"}
    return dict(ms={name[a]: statistics.median(v) for a, v in t.items()},
                spread_ms={name[a]: [round(min(v), 3), round(max(v), 3)] for a, v in t.items()},
                windows_ms={name[a]: [round(x, 3) for x in v] for a, v in t.items()},
                aa_over_off=statistics.median(t[True]) / statistics.median(t[False]),
                stage_ms_one_step={name[a]: s for a, s in stages.items()}, instances={name[a]: d for a, d in inst.items()})


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
        res[f"views{V}"] = measure(workload(V, flat, P, K, cams, g))
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
