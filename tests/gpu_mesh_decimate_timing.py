"""Timing of mesh cleanup and decimation (humangaussian_b200.mesh.clean_mesh / decimate_mesh) on the GPU.  Not a test.

    python tests/gpu_mesh_decimate_timing.py [out.json]

The full sample.ply at 256^3 and 512^3 (iso 1, 16 blocks, relax 1.5): marching cubes, then clean_mesh at the defaults
and decimate_mesh of the cleaned mesh to 1e5 faces.  Host clock around calls that end in a device synchronise, after a
warm-up call, the median of 3 repeats.  Host waits: clean has 1 + (labelling rounds) + 1, decimate 1 + (rounds + 1 when
a round selects nothing) + 1.  For scale only, the numpy restatements' host time on the same meshes (one run, this
machine's CPU; they are not an optimised implementation).  The card's name and power limit are read in the same run.
"""
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, ".")
sys.path.insert(0, os.path.join(".", "tests"))
import decimate_reference as D  # noqa: E402
import mesh_clean_reference as C  # noqa: E402
from humangaussian_b200 import mesh as MX  # noqa: E402
from humangaussian_b200.scene import sample_ply_scene  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts), out


def main():
    dev = torch.device("cuda:0")
    p = sample_ply_scene().to(dev)
    rows = {"card": card()}
    for res in (256, 512):
        k, r, nb = MX._kept("t", p.xyz, p.opacity, p.scaling, p.rotation, True, res, 16)
        v, f, _ = MX._mesh(k, r, nb, 1.5, 1.0)
        L = MX.R.load_library()
        t_clean, (cv, cf) = timed(lambda: MX.clean_mesh(v, f))
        _, crounds = MX._edit("clean_mesh", v, f,
                              lambda L, Nv, Nf, *a: L.b200gs_mesh_clean(Nv, Nf, a[0], a[1], 64, 0.2, *a[2:]),
                              lambda L, Nv, Nf: L.b200gs_mesh_clean_scratch_bytes(Nv, Nf))
        t_dec, (dm, drounds) = timed(lambda: MX._decimate(cv, cf, 100_000))
        row = dict(faces_in=int(f.shape[0]), faces_clean=int(cf.shape[0]), faces_out=int(dm.faces.shape[0]),
                   clean_ms=t_clean * 1e3, clean_label_rounds=crounds, clean_host_waits=crounds + 2,
                   decimate_ms=t_dec * 1e3, decimate_rounds=drounds, decimate_host_waits_at_most=drounds + 3)
        if res == 256:
            vn, fn_ = v.cpu().numpy(), f.cpu().numpy()
            t = time.perf_counter()
            cvn, cfn = C.clean_mesh(vn, fn_)
            row["numpy_clean_host_ms"] = (time.perf_counter() - t) * 1e3
            t = time.perf_counter()
            D.decimate(cvn, cfn, 100_000)
            row["numpy_decimate_host_ms"] = (time.perf_counter() - t) * 1e3
        rows[f"{res}^3"] = row
        print(res, row, flush=True)
    rows["card_after"] = card()
    print(json.dumps(rows))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
