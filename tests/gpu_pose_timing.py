"""Timing of the pose-map kernels (b200gs_pose_keypoints + b200gs_pose_draw) on the GPU.

    python tests/gpu_pose_timing.py [--out results.json]

For V in {8, 64} views at 512^2 and 1024^2, in both styles, on seeded shipped-config cameras (orbit, near-head and
near-back close-ups) with the golden skeletons, jittered: CUDA-event time of the two launches per call (mean of 50 calls after 5
warm-up calls, buffers allocated once), and the output bytes V * H * W * 12 over that time.  The card's name and power
limit are read in the same run.  For comparison, the reference's own poser.py drawing one 512^2 view with cv2 took
1.43 ms (HumanSD) and 6.1 ms (OpenPose) on an 8-vCPU x86 host, before its device sync and 3 MB upload; that is a
host-CPU figure, not a GPU measurement.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from humangaussian_b200 import pose as P  # noqa: E402
from humangaussian_b200 import rasterizer as R  # noqa: E402
from test_gpu_pose import _random_batch  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_pose.npz")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def time_case(L, golden, style, V, H, W, reps=50, warm=5):
    rng = np.random.default_rng(V * 7 + H)
    pts, mvp, occ = _random_batch(rng, golden, style, V)
    dev = torch.device("cuda:0")
    pts = torch.tensor(pts, device=dev).contiguous()
    mvp = torch.tensor(mvp, device=dev).contiguous()
    occ = torch.tensor(occ, device=dev).to(torch.uint8)
    s = P.STYLES[style]
    K = P.NUM_KEYPOINTS[style]
    limbs, colors = P._limbs_and_colors(style)
    limbs_h = (C.c_int32 * (2 * len(limbs)))(*[i for pair in limbs for i in pair])
    colors_h = (C.c_uint8 * (3 * len(colors)))(*[c for rgb in colors for c in rgb])
    kp = torch.empty(V, K, 2, device=dev)
    out = torch.empty(V, H, W, 3, device=dev)
    scratch = torch.empty(L.b200gs_pose_scratch_bytes(s, V, H, W), dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream

    def call():
        R._check(L.b200gs_pose_keypoints(s, V, K, H, W, pts.data_ptr(), mvp.data_ptr(), occ.data_ptr(), limbs_h, kp.data_ptr(),
                                         scratch.data_ptr(), scratch.numel(), st), "pose_keypoints")
        R._check(L.b200gs_pose_draw(s, V, H, W, colors_h, scratch.data_ptr(), scratch.numel(), out.data_ptr(), st), "pose_draw")
    for _ in range(warm):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    # the setup kernel alone, for the split
    e0.record()
    for _ in range(reps):
        R._check(L.b200gs_pose_keypoints(s, V, K, H, W, pts.data_ptr(), mvp.data_ptr(), occ.data_ptr(), limbs_h, kp.data_ptr(),
                                         scratch.data_ptr(), scratch.numel(), st), "pose_keypoints")
    e1.record()
    torch.cuda.synchronize()
    setup_ms = e0.elapsed_time(e1) / reps
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    nbytes = V * H * W * 12
    return dict(style=style, V=V, H=H, W=W, ms=round(ms, 4), setup_ms=round(setup_ms, 4), out_bytes=nbytes,
                out_GBps=round(nbytes / (ms * 1e-3) / 1e9, 1), scratch_bytes=scratch.numel())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the timing needs a GPU"
    golden = np.load(GOLDEN)
    L = R.load_library()
    rows = []
    for style in ("humansd", "openpose"):
        for V in (8, 64):
            for H in (512, 1024):
                r = time_case(L, golden, style, V, H, H)
                rows.append(r)
                print(json.dumps(r), flush=True)
    res = dict(card=card(), results=rows)
    print("card:", res["card"])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
