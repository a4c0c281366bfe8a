"""Timing of the optimiser step on the packed buffer (PackedAdam, csrc/optim.cu) at the bench workload.  Not a test.

    python tests/gpu_train_step_timing.py [P] [sh_degree]

Prints one JSON line:
  * adam_ms: one Adam step over P Gaussians at the given degree for PackedAdam (one launch over the flat buffer), the
    reference's torch.optim.Adam over six tensors (foreach, its default on CUDA) and torch's fused=True Adam over six
    tensors; CUDA events over 200 steps per window after warm-up, arms alternated, 5 windows each, median reported;
  * packed_GBps / packed_fraction_of_3.35TBps: algorithmic bytes (28 B per float: param, grad, exp_avg, exp_avg_sq read,
    three written) over PackedAdam's time;
  * step_ms: the 64-view 1024^2 packed training step (rasterize_views_packed(raw=True) forward + backward) with and
    without PackedAdam.step, alternated the same way;
  * bit_identical_to_foreach: whether one PackedAdam step from identical state equals the reference's Adam bit for bit;
  * the card's name, power limit and SM clock, read in the same run.
"""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from humangaussian_b200 import dist as D  # noqa: E402
from humangaussian_b200.optim import PackedAdam  # noqa: E402
from humangaussian_b200.rasterizer import packed_numel, rasterize_views_packed  # noqa: E402

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
LRS = dict(xyz=0.00005, f_dc=0.0125, f_rest=0.0125 / 20.0, opacity=0.01, scaling=0.005, rotation=0.001)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
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


def alternate(arms, n, windows=5):
    for fn in arms.values():  # warm-up
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    t = {k: [] for k in arms}
    for _ in range(windows):
        for k, fn in arms.items():
            t[k].append(events_ms(fn, n))
    return {k: statistics.median(v) for k, v in t.items()}, {k: [round(x, 4) for x in v] for k, v in t.items()}


def pack(t):
    return D.pack(dict(xyz=t["xyz"], scaling=t["scaling"], rotation=t["rotation"], opacity=t["opacity"],
                       features=torch.cat((t["f_dc"], t["f_rest"]), 1)))


def main():
    P = int(sys.argv[1]) if len(sys.argv) > 1 else 300_000
    deg = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    K, dev = (deg + 1) ** 2, "cuda:0"
    g = torch.Generator(device=dev).manual_seed(0)
    f = lambda *s: torch.randn(*s, device=dev, generator=g)
    shapes = dict(xyz=(P, 3), f_dc=(P, 1, 3), f_rest=(P, K - 1, 3), opacity=(P, 1), scaling=(P, 3), rotation=(P, 4))
    vals = {k: f(*s) for k, s in shapes.items()}
    grads = {k: f(*s) * 1e-3 for k, s in shapes.items()}

    def six(**kw):
        ps = {k: torch.nn.Parameter(v.clone()) for k, v in vals.items()}
        for k in GROUPS:
            ps[k].grad = grads[k].clone()
        return ps, torch.optim.Adam([{"params": [ps[k]], "lr": LRS[k], "name": k} for k in GROUPS], lr=0.0, eps=1e-15, **kw)

    flat = pack(vals).requires_grad_(True)
    flat.grad = pack(grads)
    opt = PackedAdam(flat, P, K, LRS)
    ref_ps, ref = six()
    _, fused = six(fused=True)
    # bit-identity of one step from identical (fresh) state
    opt.step()
    ref.step()
    st = opt.state[flat]
    same = torch.equal(flat.detach(), pack({k: ref_ps[k].detach() for k in GROUPS})) and \
        torch.equal(st["exp_avg"], pack({k: ref.state[ref_ps[k]]["exp_avg"] for k in GROUPS})) and \
        torch.equal(st["exp_avg_sq"], pack({k: ref.state[ref_ps[k]]["exp_avg_sq"] for k in GROUPS}))
    adam, adam_windows = alternate({"packed": opt.step, "torch_foreach_six_tensors": ref.step, "torch_fused_six_tensors": fused.step}, 200)
    n_float = packed_numel(P, K)
    gbps = 28 * n_float / (adam["packed"] * 1e-3) / 1e9

    # the 64-view training step of bench.py's workload (same scene, cameras and resolution)
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import stack_cameras
    from humangaussian_b200.scene import sample_ply_scene
    sc = sample_ply_scene(P, deg, seed=0)
    scene = dict(xyz=sc.xyz, f_dc=sc.features_dc, f_rest=sc.features_rest, opacity=sc.opacity, scaling=sc.scaling, rotation=sc.rotation)
    sflat = pack({k: v.detach().float().to(dev) for k, v in scene.items()}).requires_grad_(True)
    sopt = PackedAdam(sflat, P, K, LRS)
    HW = 1024
    vm, pm, cp, tx, ty = stack_cameras(sample_orbit_cameras(64, HW, HW, seed=1000, device="cpu"), dev)
    gw = [torch.randn(64, c, HW, HW, device=dev, generator=g) for c in (3, 1, 1)]
    bg = torch.zeros(3, device=dev)

    def fwd_bwd():
        sflat.grad = None
        c, r, d, a = rasterize_views_packed(sflat, P, K, viewmatrices=vm, projmatrices=pm, camposs=cp, tanfovx=tx, tanfovy=ty,
                                            image_height=HW, image_width=HW, bg=bg, sh_degree=deg, raw=True)
        torch.autograd.backward([c, d, a], gw)

    def train_step():
        fwd_bwd()
        # a tiny lr keeps the scene (and so the step's work) essentially fixed over the timed windows
        sopt.step()

    sopt.param_groups[0]["lrs"] = {k: 1e-12 for k in GROUPS}
    step, step_windows = alternate({"fwd_bwd": fwd_bwd, "fwd_bwd_adam": train_step}, 10)
    print(json.dumps({
        "card": card(), "P": P, "sh_degree": deg, "floats_per_buffer": n_float, "MB_per_buffer": 4 * n_float / 1e6,
        "adam_ms": adam, "adam_windows_ms": adam_windows,
        "packed_vs_foreach": adam["torch_foreach_six_tensors"] / adam["packed"], "packed_vs_fused": adam["torch_fused_six_tensors"] / adam["packed"],
        "packed_GBps": gbps, "packed_fraction_of_3.35TBps": gbps / 3350.0,
        "step_ms": step, "step_windows_ms": step_windows, "adam_share_of_step": (step["fwd_bwd_adam"] - step["fwd_bwd"]) / step["fwd_bwd_adam"],
        "bit_identical_to_foreach": bool(same), "card_after": card()}))


if __name__ == "__main__":
    main()
