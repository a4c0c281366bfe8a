"""Timing of mesh export (humangaussian_b200.mesh) on the GPU.  Not a test.

    python tests/gpu_mesh_timing.py [out.json]

Scenes: the full sample.ply (531 327 Gaussians) and the bench's seed-0 300 k subsample.  For each, at 128^3, 256^3 and
512^3 (16 blocks, relax 1.5, the reference's defaults besides the resolution):
  field      b200gs_density_field alone (prep, sort, gather, field kernel) on the prepared Gaussians;
  extract    extract_fields end to end (the torch prep of the P-sized inputs included);
  mc         marching_cubes of that field at iso 1 (classify, two scans, the one host wait, emit).
CUDA events after a warm-up call, the median of 5 repeats.  The work is counted from shapes: voxel-candidate pairs =
sum over blocks of (voxels in the block) x (Gaussians whose centre is inside its widened box), each one exponent and 26
float32 operations (3 subtractions, 15 multiplications, 5 additions / subtractions, the opacity product and the sum);
the share of the FP32 peak is 26 x pairs / time over SMs x 128 lanes x the SM clock read in the same call (one op per
lane per cycle; FMA-counted peaks are twice that, and this kernel has no FMA to count).  The reference algorithm,
restated in torch on the same GPU (per-block loop, [M, L, 3] / [M, L, 6] temporaries, batches of 1024 Gaussians), is
timed at 128^3 and 256^3; an out-of-memory error is reported, not raised.  The card's name, power limit and clocks are
read before and after.
"""
import json
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from humangaussian_b200 import mesh as MX  # noqa: E402
from humangaussian_b200.scene import sample_ply_scene  # noqa: E402

OPS_PER_PAIR = 26


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def sm_clock_mhz():
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return float(q[0]) if q else float("nan")


def timed(fn, n=5):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out), min(out), max(out)


def prepared(p):
    """the kept, normalised Gaussians as extract_fields hands them to the library"""
    op = torch.sigmoid(p.opacity).reshape(-1)
    keep = op > MX.OPACITY_MIN
    xyz = p.xyz[keep]
    mn, mx = xyz.amin(0), xyz.amax(0)
    center, scale = (mn + mx) / 2, 1.8 / (mx - mn).amax().item()
    xyz = ((xyz - center) * scale).contiguous()
    return xyz, MX._covariance(torch.exp(p.scaling[keep]) * scale, p.rotation[keep]), op[keep].contiguous()


def pair_count(xyz, res, num_blocks=16, relax_ratio=1.5):
    """sum over blocks of voxels x members, from per-axis chunk intervals (membership is a box of blocks per Gaussian)"""
    split = res // num_blocks
    lin = torch.linspace(-1, 1, res)
    starts = list(range(0, res, split))
    relax = np.float32((2 / num_blocks) * relax_ratio)
    lo = torch.tensor([lin[s:s + split].min().item() for s in starts]) - torch.tensor(relax)
    hi = torch.tensor([lin[s:s + split].max().item() for s in starts]) + torch.tensor(relax)
    ext = torch.tensor([min(split, res - s) for s in starts], dtype=torch.float64)
    x = xyz.cpu()
    tot = torch.ones(x.shape[0], dtype=torch.float64)
    for a in range(3):
        m = (x[:, a:a + 1] > lo[None]) & (x[:, a:a + 1] < hi[None])
        tot *= (m.double() * ext[None]).sum(1)
    return float(tot.sum())


def reference_algorithm(xyz, cov6, opac, res, num_blocks=16, relax_ratio=1.5):
    """the reference's extract_fields loop, restated in torch on the device (its algorithm and temporaries)"""
    dev = xyz.device
    block_size = 2 / num_blocks
    split = res // num_blocks
    occ = torch.zeros((res,) * 3, dtype=torch.float32, device=dev)
    X = torch.linspace(-1, 1, res).split(split)
    a, b, c, d, e, f = cov6.unbind(1)
    for xi, xs in enumerate(X):
        for yi, ys in enumerate(X):
            for zi, zs in enumerate(X):
                pts = torch.stack(torch.meshgrid(xs, ys, zs, indexing="ij"), -1).reshape(-1, 3).to(dev)
                vmin, vmax = pts.amin(0) - block_size * relax_ratio, pts.amax(0) + block_size * relax_ratio
                m = (xyz < vmax).all(-1) & (xyz > vmin).all(-1)
                if not m.any():
                    continue
                gx, gc, go = xyz[m], cov6[m], opac[m].view(1, -1)
                d3 = pts.unsqueeze(1).repeat(1, gx.shape[0], 1) - gx.unsqueeze(0)
                c6 = gc.unsqueeze(0).repeat(pts.shape[0], 1, 1)
                val = 0
                for s in range(0, gx.shape[0], 1024):
                    q, k = d3[:, s:s + 1024].reshape(-1, 3), c6[:, s:s + 1024].reshape(-1, 6)
                    A, B, C, D, E, F = k.unbind(1)
                    inv_det = 1 / (A * D * F + 2 * E * C * B - E ** 2 * A - C ** 2 * D - B ** 2 * F + 1e-24)
                    x, y, z = q.unbind(1)
                    pw = (-0.5 * (x ** 2 * (D * F - E ** 2) * inv_det + y ** 2 * (A * F - C ** 2) * inv_det + z ** 2 * (A * D - B ** 2) * inv_det)
                          - x * y * (E * C - B * F) * inv_det - x * z * (E * B - C * D) * inv_det - y * z * (B * C - E * A) * inv_det)
                    pw[pw > 0] = -1e10
                    val = val + (go[:, s:s + 1024] * torch.exp(pw).reshape(pts.shape[0], -1)).sum(-1)
                occ[xi * split:xi * split + len(xs), yi * split:yi * split + len(ys), zi * split:zi * split + len(zs)] = \
                    val.reshape(len(xs), len(ys), len(zs))
    return occ


def main():
    assert torch.cuda.is_available(), "needs a GPU"
    out = {"card_before": card(), "rows": []}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    clock = sm_clock_mhz()
    scenes = {"full_531k": sample_ply_scene().to("cuda"), "bench_300k": sample_ply_scene(n=300000).to("cuda")}
    for name, p in scenes.items():
        xyz, cov6, opac = prepared(p)
        for res in (128, 256, 512):
            pairs = pair_count(xyz, res)
            t_field = timed(lambda: MX._density_field(xyz, cov6, opac, res, 16, 1.5))
            t_ext = timed(lambda: MX.extract_fields(p, resolution=res))
            occ = MX.extract_fields(p, resolution=res).occ
            t_mc = timed(lambda: MX.marching_cubes(occ, 1.0))
            v, f = MX.marching_cubes(occ, 1.0)
            peak = sms * 128 * clock * 1e6
            row = dict(scene=name, P_kept=int(xyz.shape[0]), res=res, pairs=pairs, field_ms=t_field, extract_ms=t_ext, mc_ms=t_mc,
                       vertices=len(v), faces=len(f), field_max=float(occ.max()),
                       exp_per_s=pairs / (t_field[0] * 1e-3), fp32_share=OPS_PER_PAIR * pairs / (t_field[0] * 1e-3) / peak)
            print(json.dumps(row), flush=True)
            out["rows"].append(row)
            del occ
            torch.cuda.empty_cache()
        for res in (128, 256):
            try:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ref = reference_algorithm(xyz, cov6, opac, res)
                torch.cuda.synchronize()
                dt = (time.perf_counter() - t0) * 1e3
                mine = MX._density_field(xyz, cov6, opac, res, 16, 1.5)
                diff = float((mine - ref).abs().max())
                row = dict(scene=name, res=res, reference_algorithm_ms=dt, max_abs_diff=diff)
                del ref, mine
            except torch.cuda.OutOfMemoryError as e:
                row = dict(scene=name, res=res, reference_algorithm="out of memory: " + str(e).splitlines()[0])
            torch.cuda.empty_cache()
            print(json.dumps(row), flush=True)
            out["rows"].append(row)
    out["card_after"] = card()
    out["sm_count"], out["sm_clock_max_mhz"] = sms, clock
    print(json.dumps({k: out[k] for k in ("card_before", "card_after", "sm_count", "sm_clock_max_mhz")}))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
