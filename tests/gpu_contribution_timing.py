"""Timing of the contribution scores on the GPU (run as a script, not collected by pytest).

  1. plain vs contribution forward (rasterizer._forward_impl with and without the accumulators) on the bench scene (seed-0
     300 k subsample of sample.ply, SH degree 3, 1024^2) at 8 and 64 views, alternated over windows: medians, spread and
     the forward blend kernels' device time alone (torch.profiler, a separate pass);
  2. compute_contribution for the full 531 k file over 256 orbit cameras at 1024^2;
  3. the fraction of that file with touches == 0; after removing them, the same 256 cameras render byte-identical, timed
     before and after;
  4. one lossy threshold on weight_max and its PSNR against the unpruned render on 16 held-out cameras.
Writes the results as JSON to <dir>/contribution_timing.json, <dir> = argv[1] (default gpu_out)."""
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from humangaussian_b200 import rasterizer as R  # noqa: E402
from humangaussian_b200.cameras import sample_orbit_cameras  # noqa: E402
from humangaussian_b200.contribution import compute_contribution  # noqa: E402
from humangaussian_b200.renderer import stack_cameras  # noqa: E402
from humangaussian_b200.scene import sample_ply_scene  # noqa: E402

DEV = torch.device("cuda:0")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def tensors(p):
    with torch.no_grad():
        return dict(means3D=p.get_xyz.to(DEV).contiguous(), opacities=p.get_opacity.to(DEV).contiguous(),
                    shs=p.get_features.to(DEV).contiguous(), scales=p.get_scaling.to(DEV).contiguous(),
                    rotations=p.get_rotation.to(DEV).contiguous())


def fwd(g, cams, deg, contrib=None):
    vm, pm, cp, tx, ty, H, W = cams
    return R._forward_impl(g["means3D"], g["shs"], None, g["opacities"], g["scales"], g["rotations"], None, torch.zeros(3, device=DEV),
                           vm, pm, cp, tx, ty, H, W, deg, 1.0, contrib=contrib)


def time_windows(fns, reps, windows):
    """alternate the callables over `windows` windows of `reps` calls each; ms per call per window"""
    out = {k: [] for k in fns}
    for _ in range(windows):
        for k, f in fns.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(reps):
                f()
            torch.cuda.synchronize()
            out[k].append((time.perf_counter() - t0) * 1e3 / reps)
    return out


def kernel_ms(fns, reps):
    """device time per call of the forward blend kernels alone, from torch.profiler's CUDA activity records (a separate
    pass after the timed windows): {variant: {kernel name: ms per call}}"""
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for k, f in fns.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                f()
            torch.cuda.synchronize()
        tot = {}
        for e in prof.key_averages():
            if "blend_fwd" in e.key and e.self_device_time_total > 0:
                tot[e.key] = e.self_device_time_total / 1e3 / reps
        out[k] = tot
    return out


def main(out_dir):
    res = dict(gpu=gpu_info(), torch=torch.__version__)
    p = sample_ply_scene(300000, 3)
    g = tensors(p)
    P = g["means3D"].shape[0]
    acc = (torch.zeros(P, dtype=torch.int64, device=DEV), torch.zeros(P, dtype=torch.int32, device=DEV),
           torch.zeros(P, dtype=torch.int32, device=DEV))
    for V in (8, 64):
        vm, pm, cp, tx, ty = stack_cameras(sample_orbit_cameras(V, 1024, 1024, seed=1000), DEV)
        cams = (vm, pm, cp, tx, ty, 1024, 1024)
        fns = dict(plain=lambda: fwd(g, cams, 3), contrib=lambda: fwd(g, cams, 3, acc))
        for f in fns.values():  # warm-up (pool, capacity hints)
            f(); f()
        reps = 20 if V == 8 else 4
        w = time_windows(fns, reps, 7)
        res[f"fwd_{V}v"] = {k: dict(median_ms=statistics.median(v), min_ms=min(v), max_ms=max(v)) for k, v in w.items()}
        res[f"fwd_{V}v"]["blend_kernel_ms"] = kernel_ms(fns, reps)
        res[f"fwd_{V}v"]["ratio_median"] = statistics.median(w["contrib"]) / statistics.median(w["plain"])
        print(V, json.dumps(res[f"fwd_{V}v"]), flush=True)
    del g, acc

    full = sample_ply_scene()
    g = tensors(full)
    P = g["means3D"].shape[0]
    cams = sample_orbit_cameras(256 + 16, 1024, 1024, seed=2024)
    vm, pm, cp, tx, ty = stack_cameras(cams[:256], DEV)
    geo = {k: g[k] for k in ("means3D", "opacities", "scales", "rotations")}
    kw = dict(viewmatrices=vm, projmatrices=pm, tanfovx=tx, tanfovy=ty, image_height=1024, image_width=1024)
    compute_contribution(**geo, **kw)  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sc = compute_contribution(**geo, **kw)
    torch.cuda.synchronize()
    res["compute_contribution_531k_256cams_1024_ms"] = (time.perf_counter() - t0) * 1e3
    untouched = sc.touches == 0
    res["untouched_fraction"] = float(untouched.float().mean())
    keep = ~untouched
    gk = {k: v[keep] for k, v in g.items()}

    def render(gg, lo, hi, vm_, pm_, cp_, tx_, ty_):
        with torch.no_grad():
            return R.rasterize_views(**gg, viewmatrices=vm_[lo:hi], projmatrices=pm_[lo:hi], camposs=cp_[lo:hi], tanfovx=tx_[lo:hi],
                                     tanfovy=ty_[lo:hi], image_height=1024, image_width=1024, bg=torch.zeros(3, device=DEV), sh_degree=0)

    same = True
    for lo in range(0, 256, 32):
        a, b = render(g, lo, lo + 32, vm, pm, cp, tx, ty), render(gk, lo, lo + 32, vm, pm, cp, tx, ty)
        same &= all(torch.equal(x, y) for x, y in ((a[0], b[0]), (a[2], b[2]), (a[3], b[3])))
    res["pruned_renders_byte_identical"] = bool(same)
    w = time_windows(dict(full=lambda: render(g, 0, 32, vm, pm, cp, tx, ty), pruned=lambda: render(gk, 0, 32, vm, pm, cp, tx, ty)), 3, 5)
    res["render_32v_1024"] = {k: dict(median_ms=statistics.median(v), frames_per_s=32e3 / statistics.median(v)) for k, v in w.items()}

    thr = 0.01
    lossy = keep & (sc.weight_max >= thr)
    gl = {k: v[lossy] for k, v in g.items()}
    hvm, hpm, hcp, htx, hty = stack_cameras(cams[256:], DEV)
    a = render(g, 0, 16, hvm, hpm, hcp, htx, hty)[0].clamp(0, 1)
    b = render(gl, 0, 16, hvm, hpm, hcp, htx, hty)[0].clamp(0, 1)
    mse = ((a - b) ** 2).flatten(1).mean(1)
    res["lossy_weight_max_threshold"] = thr
    res["lossy_kept_fraction"] = float(lossy.float().mean())
    res["lossy_heldout_psnr_db_median"] = float(statistics.median((10 * torch.log10(1.0 / mse.clamp_min(1e-12))).tolist()))
    print(json.dumps(res, indent=1), flush=True)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "contribution_timing.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "gpu_out")
