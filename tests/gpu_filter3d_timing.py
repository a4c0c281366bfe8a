"""Timing of the 3D smoothing filter (rasterize_views_packed(filter_3d=...)) against the default.  Not a test.

    python tests/gpu_filter3d_timing.py [out.json]

Workloads: the bench's (300 k Gaussians of sample.ply, SH degree 3, 1024^2, its 64 cameras) and the 8-view SDS batch (the
first 8 of them); one step = rasterize_views_packed(raw=True) forward + backward, as bench.py times it.  The variances come
from compute_filter_3d over 256 orbit cameras of the training distribution at 1024^2.  Arms (filter off, filter on,
antialiasing + filter) alternated in 5 windows of 5 steps after warm-up, CUDA events, median and spread (min..max of the
windows).  Reported alongside: the instance count D of each arm (the filter widens small Gaussians, so radii and D can
grow), the library's per-stage CUDA-event times of one step, and the time of compute_filter_3d itself (300 k x 256
cameras).  The card's name, power limit and clocks are read before and after.
"""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from humangaussian_b200 import dist as D  # noqa: E402
from humangaussian_b200 import rasterizer as R  # noqa: E402

ARMS = ("off", "f3d", "aa+f3d")


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


def workload(V, flat, P, K, cams, var, g):
    vm, pm, cp, tx, ty = cams
    gw = [torch.randn(V, c, 1024, 1024, device="cuda", generator=g) for c in (3, 1, 1)]
    bg = torch.zeros(3, device="cuda")

    def step(arm):
        flat.grad = None
        c, r, d, a = R.rasterize_views_packed(flat, P, K, viewmatrices=vm[:V], projmatrices=pm[:V], camposs=cp[:V], tanfovx=tx[:V],
                                              tanfovy=ty[:V], image_height=1024, image_width=1024, bg=bg, sh_degree=3, raw=True,
                                              antialiasing=arm == "aa+f3d", filter_3d=None if arm == "off" else var)
        torch.autograd.backward([c, d, a], gw)
    return step


def measure(step, n=5, windows=5):
    for arm in ARMS:
        for _ in range(2):
            step(arm)
    torch.cuda.synchronize()
    t = {arm: [] for arm in ARMS}
    for _ in range(windows):
        for arm in ARMS:
            t[arm].append(events_ms(lambda: step(arm), n))
    stages, inst = {}, {}
    for arm in ARMS:
        torch.cuda.synchronize()
        R.profile_read()
        R.profile_enable(True)
        step(arm)
        torch.cuda.synchronize()
        R.profile_enable(False)
        stages[arm] = {k: round(v[0], 3) for k, v in R.profile_read().items()}
        inst[arm] = R.last_num_rendered()
    med = {a: statistics.median(v) for a, v in t.items()}
    return dict(ms=med, spread_ms={a: [round(min(v), 3), round(max(v), 3)] for a, v in t.items()},
                windows_ms={a: [round(x, 3) for x in v] for a, v in t.items()},
                over_off={a: med[a] / med["off"] for a in ARMS}, stage_ms_one_step=stages, instances=inst)


def main():
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.filter3d import compute_filter_3d
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
    fvm, _, _, ftx, fty = stack_cameras(sample_orbit_cameras(256, 1024, 1024, seed=7, device="cpu"), "cuda")
    xyz = sc.xyz.detach().float().cuda().contiguous()
    f = lambda: compute_filter_3d(xyz, fvm, ftx, fty, 1024, 1024)
    var = f()
    torch.cuda.synchronize()
    f_ms = sorted(events_ms(f, 5) for _ in range(5))
    s = torch.exp(sc.scaling.detach().float().cuda())
    ratio = (var[:, None] / (s * s)).max(1).values  # v / s_min^2: how much the filter widens the smallest axis
    res = {"card_before": before, "P": P, "sh_degree": deg, "resolution": 1024,
           "compute_filter_3d_ms_256_cameras": dict(median=f_ms[2], spread=[f_ms[0], f_ms[-1]]),
           "v_over_smin2_quantiles": {q: float(torch.quantile(ratio[:100000], q)) for q in (0.1, 0.5, 0.9)}}
    g = torch.Generator(device="cuda").manual_seed(0)
    for V in (64, 8):
        res[f"views{V}"] = measure(workload(V, flat, P, K, cams, var, g))
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
