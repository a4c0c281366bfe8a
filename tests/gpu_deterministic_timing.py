"""Timing of the deterministic backward against the default (atomic) one.  Not a test.

    python tests/gpu_deterministic_timing.py [out.json]

Workloads: the bench's (300 k Gaussians of sample.ply, SH degree 3, 1024^2, its 64 cameras) and the 8-view SDS batch (the
first 8 of them); one step = rasterize_views_packed(raw=True) forward + backward, as bench.py times it.  Arms, alternated in
5 windows of 5 steps after warm-up, CUDA events, median and spread (min..max of the windows) reported:
  * atomic:        torch.use_deterministic_algorithms(False), the default backward;
  * deterministic: the flag on, torch.utils.deterministic.fill_uninitialized_memory OFF -- torch's NaN fill of the
                   torch.empty outputs is not in this arm's time;
  * deterministic_fill: the flag on with fill_uninitialized_memory at its default (on): what a user gets by default.
Reported alongside: the measured partial count H and partial bytes (40 B each), the instance count D, the library's
per-stage CUDA-event times (blend_bwd holds the pre-pass, B1 and the reduce in deterministic mode), and, from a separate
torch.profiler run, the deterministic backward's split into pre-pass / B1 / reduce kernels.  The card's name, power limit
and clocks are read in the same run, before and after.
"""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from humangaussian_b200 import dist as D  # noqa: E402
from humangaussian_b200 import rasterizer as R  # noqa: E402

PREPASS = ("det_start_kernel", "det_plan_kernel", "PopcLoad")
B1 = ("blend_bwd_kernel<true, false, false, false>",)
REDUCE = ("det_reduce_kernel",)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def set_mode(mode):
    torch.use_deterministic_algorithms(mode != "atomic", warn_only=True)
    torch.utils.deterministic.fill_uninitialized_memory = mode != "deterministic"


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

    def step():
        flat.grad = None
        c, r, d, a = R.rasterize_views_packed(flat, P, K, viewmatrices=vm[:V], projmatrices=pm[:V], camposs=cp[:V], tanfovx=tx[:V],
                                              tanfovy=ty[:V], image_height=1024, image_width=1024, bg=bg, sh_degree=3, raw=True)
        torch.autograd.backward([c, d, a], gw)
    return step


def measure(step, arms=("atomic", "deterministic", "deterministic_fill"), n=5, windows=5):
    for m in arms:  # warm-up (and the deterministic arm's first-call sizing)
        set_mode(m)
        for _ in range(2):
            step()
    torch.cuda.synchronize()
    t = {m: [] for m in arms}
    for _ in range(windows):
        for m in arms:
            set_mode(m)
            t[m].append(events_ms(step, n))
    stages = {}
    for m in ("atomic", "deterministic"):
        set_mode(m)
        torch.cuda.synchronize()
        R.profile_read()
        R.profile_enable(True)
        step()
        torch.cuda.synchronize()
        R.profile_enable(False)
        stages[m] = {k: round(v[0], 3) for k, v in R.profile_read().items()}
    set_mode("deterministic")
    step()
    torch.cuda.synchronize()
    H, Dn = R.last_num_partials(), R.last_num_rendered()
    split = profile_split(step)
    set_mode("atomic")
    return dict(ms={m: statistics.median(v) for m, v in t.items()},
                spread_ms={m: [round(min(v), 3), round(max(v), 3)] for m, v in t.items()},
                windows_ms={m: [round(x, 3) for x in v] for m, v in t.items()},
                deterministic_over_atomic=statistics.median(t["deterministic"]) / statistics.median(t["atomic"]),
                stage_ms_one_step=stages, instances=Dn, partials=H, partials_per_instance=H / max(Dn, 1),
                partial_GB=H * 40 / 1e9, det_split_ms=split)


def profile_split(step):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    out = {"prepass": 0.0, "b1": 0.0, "reduce": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = getattr(e, "cuda_time_total", 0.0)
        for k, names in (("prepass", PREPASS), ("b1", B1), ("reduce", REDUCE)):
            if any(n in e.key for n in names):
                out[k] += us / 1e3
    return {k: round(v, 3) for k, v in out.items()}


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
    res = {"card_before": before, "P": P, "sh_degree": deg, "resolution": 1024,
           "fill_uninitialized_memory": "off in 'deterministic', on (torch's default) in 'deterministic_fill'"}
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
