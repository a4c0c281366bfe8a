"""Timing of the mesh render (humangaussian_b200.meshrender, csrc/meshraster.cu) on the GPU.

    python tests/gpu_meshraster_timing.py [--out results.json]

CUDA-event time per call (mean of 10 calls after 2 warm-up calls, the whole measurement repeated --repeats times and
reported as min / median / max) of `rasterize`, of the emit call alone on the first 64 views (tile scatter and the raster
kernel, no host wait), and of the whole `render_mesh_normal` (vertex transform, incidence, vertex normals,
rasterisation with its one host wait per 64 views, normal image), for:
  * the reference's human body (1 629 vertices, 3 226 triangles) at 1024^2 from 8 and 64 orbit cameras;
  * 136 deformed frames of it at 800^2, the viewer's default size, one frame per view (per-view vertices, 3 chunks);
  * the extract_mesh output of the full sample scene at 128^3, 8 orbit views at 1024^2.
The card's name and power limit are read in the same run, and the (tile, triangle) pair count of each rasterisation is
reported with it.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from humangaussian_b200 import mesh as MX  # noqa: E402
from humangaussian_b200 import meshrender as MR  # noqa: E402
from humangaussian_b200 import rasterizer as R  # noqa: E402
from humangaussian_b200.cameras import CameraBatch, orbit_c2w  # noqa: E402
from humangaussian_b200.scene import sample_ply_scene  # noqa: E402
from test_meshraster_cpu import human  # noqa: E402

DEV = torch.device("cuda:0")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def cams(V, H, W, center, seed=0):
    rng = np.random.default_rng(seed)
    c2w = torch.stack([orbit_c2w(float(rng.uniform(-30, 30)), float(rng.uniform(-180, 180)), float(rng.uniform(1.5, 3.0)), center)
                       for _ in range(V)])
    return MR.camera_mvp(CameraBatch(c2w, [math.radians(float(rng.uniform(40, 70))) for _ in range(V)], H, W, device=DEV))


def ms_per_call(fn, reps=10, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def emit_timer(pos, faces, H, W):
    """The emit call on the first 64 views, after one count: tile scatter and raster kernel, no host wait."""
    L = R.load_library()
    p, t = pos[:64].contiguous(), faces.to(torch.int32).contiguous()
    V, Nv, Nf = p.shape[0], p.shape[1], t.shape[0]
    st = R._stream(DEV)
    scratch = torch.empty(L.b200gs_mesh_raster_scratch_bytes(V, Nf, H, W), dtype=torch.uint8, device=DEV)
    count = torch.zeros(1, dtype=torch.int64, device=DEV)
    R._check(L.b200gs_mesh_raster_count(V, Nv, Nf, H, W, R._ptr(p), R._ptr(t), R._ptr(scratch), scratch.numel(), R._ptr(count), st), "count")
    n = int(count.item())
    pairs = torch.empty(max(n, 1), dtype=torch.int32, device=DEV)
    out = torch.empty(V, H, W, 4, device=DEV)
    return n, lambda: R._check(L.b200gs_mesh_raster_emit(V, Nv, Nf, H, W, R._ptr(scratch), scratch.numel(), R._ptr(pairs), 4 * n,
                                                         R._ptr(out), st), "emit")


def spread(fn, repeats):
    t = sorted(ms_per_call(fn) for _ in range(repeats))
    return dict(min=round(t[0], 3), median=round(t[len(t) // 2], 3), max=round(t[-1], 3))


def case(name, verts, faces, mvp, H, W, repeats):
    pos = MR.vertex_transform(verts, mvp)
    rast = MR.rasterize(pos, faces, (H, W))
    pairs, emit = emit_timer(pos, faces, H, W)
    r = dict(case=name, views=int(mvp.shape[0]), H=H, W=W, vertices=int(verts.shape[-2]), faces=int(faces.shape[0]),
             covered=round(float((rast[..., 3] > 0).float().mean()), 4), pairs_first_64_views=pairs,
             rasterize_ms=spread(lambda: MR.rasterize(pos, faces, (H, W)), repeats),
             emit_first_64_views_ms=spread(emit, repeats),
             render_mesh_normal_ms=spread(lambda: MR.render_mesh_normal(mvp, H, W, verts, faces), repeats))
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the timing needs a GPU"
    v, f = human()
    verts, faces = torch.tensor(v, device=DEV), torch.tensor(f, device=DEV)
    rows = []
    for V in (8, 64):
        rows.append(case("human", verts, faces, cams(V, 1024, 1024, (0.0, 0.0, -0.1)), 1024, 1024, args.repeats))
    rng = np.random.default_rng(5)
    frames = verts[None] + torch.tensor(rng.normal(scale=0.01, size=(136,) + v.shape), dtype=torch.float32, device=DEV)
    rows.append(case("human, 136 deformed frames", frames, faces, cams(136, 800, 800, (0.0, 0.0, -0.1), seed=1), 800, 800,
                     args.repeats))
    m = MX.extract_mesh(sample_ply_scene().to(DEV), resolution=128)
    ctr = tuple(float(x) for x in (m.vertices.min(0).values + m.vertices.max(0).values) / 2)
    rows.append(case("extract_mesh, full sample scene, 128^3", m.vertices, m.faces, cams(8, 1024, 1024, ctr, seed=2), 1024, 1024,
                     args.repeats))
    res = dict(card=card(), results=rows)
    print("card:", res["card"])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
