"""Timing of the field query (humangaussian_b200.mesh.query_field, b200gs_field_query) on the GPU.  Not a test.

    python tests/gpu_mesh_color_timing.py [out.json]

Scene: the full sample.ply (531 327 Gaussians) at 128^3 (16 blocks, relax 1.5).  The points are all vertices of its
marching-cubes mesh at iso 1, in the field's frame.  Timed, next to the density field of the same Gaussians:
  field        b200gs_density_field alone (prep, sort, gather, field kernel);
  query_none   b200gs_field_query, density and normals only;
  query_deg0   the same with colours from the scene's degree-0 SH;
  query_deg3   the same with seeded synthetic degree-3 SH (N(0, 0.1^2) rest coefficients);
  colored_mesh extract_colored_mesh end to end (torch prep, field, marching cubes with its host wait, query).
CUDA events after a warm-up call, the median of 7 repeats.  The card's name, power limit and clocks are read in the same
call.
"""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from humangaussian_b200 import mesh as MX  # noqa: E402
from humangaussian_b200.scene import sample_ply_scene  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn, n=7):
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


def main():
    dev = torch.device("cuda:0")
    res = {"card_before": card()}
    p = sample_ply_scene(sh_degree=3, seed=0).to(dev)
    k = MX._kept("timing", p.xyz, p.opacity, p.scaling, p.rotation, True, 128, 16)[0]
    occ = MX._density_field(k.xyz, k.cov6, k.opac, 128, 16, 1.5)
    v, f = MX.marching_cubes(occ, 1.0)
    q = (v / 127 * 2 - 1).contiguous()
    sh3 = torch.cat([p.features_dc, p.features_rest], 1)[k.keep].contiguous()
    sh0 = p.features_dc[k.keep].contiguous()
    res.update(P=int(p.P), kept=int(k.xyz.shape[0]), vertices=int(len(v)), faces=int(len(f)), resolution=128)
    runs = {
        "field": lambda: MX._density_field(k.xyz, k.cov6, k.opac, 128, 16, 1.5),
        "query_none": lambda: MX._query(k, None, 0, 0, q, 128, 16, 1.5),
        "query_deg0": lambda: MX._query(k, sh0, 1, 0, q, 128, 16, 1.5),
        "query_deg3": lambda: MX._query(k, sh3, 16, 3, q, 128, 16, 1.5),
        "colored_mesh": lambda: MX.extract_colored_mesh(p, resolution=128),
    }
    for name, fn in runs.items():
        med, lo, hi = timed(fn)
        res[name + "_ms"] = {"median": round(med, 3), "min": round(lo, 3), "max": round(hi, 3)}
        print(f"{name:13s} median {med:8.3f} ms  (min {lo:.3f}, max {hi:.3f})", flush=True)
    res["card_after"] = card()
    print(json.dumps(res))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
