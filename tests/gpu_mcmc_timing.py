"""Timing of MCMC densification on the GPU (DESIGN.md section 6): the noise kernel against the same formula composed in
torch at 300 k, and relocate / add on an optim.PackedAdam at 300 k (synthetic body) and 531 k (content/sample.ply, all of
it), plus the loss ratio of tests/test_gpu_mcmc.py's training loop.  Not a test.
    python tests/gpu_mcmc_timing.py [out.json]
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from humangaussian_b200 import dist as D  # noqa: E402
from humangaussian_b200 import mcmc  # noqa: E402
from humangaussian_b200.optim import PackedAdam  # noqa: E402
from humangaussian_b200.scene import sample_ply_scene, synthetic_body  # noqa: E402

DEV = torch.device("cuda:0")
LRS = dict(xyz=0.00016, f_dc=0.0125, f_rest=0.0125 / 20.0, opacity=0.05, scaling=0.005, rotation=0.001)


def events(fn, n):
    """mean milliseconds per call over n calls after 3 warm-up calls, by CUDA events"""
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def torch_noise(xyz, scaling, rotation, opacity, eta, scale, k=100.0, t=0.005):
    """the noise step composed of torch ops (as an MCMC trainer writes it without a kernel)"""
    q = torch.nn.functional.normalize(rotation)
    r, x, y, z = q.unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    S = R @ torch.diag_embed(torch.exp(2 * scaling)) @ R.transpose(1, 2)
    gate = torch.sigmoid(-k * (torch.sigmoid(opacity) - t))
    xyz += scale * gate * torch.bmm(S, eta.unsqueeze(-1)).squeeze(-1)


def optimizer(p, dead=0.05):
    K = p.features_rest.shape[1] + 1
    op = p.opacity.clone()
    op[torch.rand(op.shape, generator=torch.Generator().manual_seed(0)) < dead] = -8.0
    raw = dict(xyz=p.xyz, scaling=p.scaling, rotation=p.rotation, opacity=op, features=torch.cat((p.features_dc, p.features_rest), 1))
    flat = D.pack({k: v.float().to(DEV).contiguous() for k, v in raw.items()}).requires_grad_(True)
    opt = PackedAdam(flat, p.xyz.shape[0], K, LRS)
    opt.packed.grad = torch.full_like(opt.packed, 1e-4)
    opt.step()
    opt.zero_grad()
    return opt


def surgery(name, p, out):
    P = p.xyz.shape[0]
    base = optimizer(p)
    g = torch.Generator(device=DEV).manual_seed(1)
    n_dead = int((~(torch.sigmoid(D.unpack(base.packed.detach(), P, base.sh_coeffs)["opacity"]) > 0.005)).sum())

    def fresh():
        o = PackedAdam(base.packed.detach().clone().requires_grad_(True), P, base.sh_coeffs, LRS)
        o.load_state_dict(base.state_dict())
        return o

    def timed(fn, n=10):
        """per call on a fresh copy, only one copy alive at a time (as in training, where the old buffers are freed), so
        the caching allocator serves the new buffers; the call includes relocate's host read of d"""
        total = 0.0
        for i in range(n + 3):
            o = fresh()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(o)
            e1.record()
            torch.cuda.synchronize()
            total += e0.elapsed_time(e1) if i >= 3 else 0.0
            del o
        return total / n
    rel = timed(lambda o: mcmc.relocate_packed(o, generator=g))
    add = timed(lambda o: mcmc.add_packed(o, 10 ** 9, generator=g))
    K = base.sh_coeffs
    floats = base.packed.numel()
    out[name] = dict(P=P, K=K, dead=n_dead, relocate_ms=rel, add_ms=add, P_after_add=int(1.05 * P),
                     relocate_algorithmic_MB=floats * 4 * 3 * 2 / 1e6,  # three flat buffers read and written
                     add_algorithmic_MB=(floats + floats * 1.05) * 4 * 3 / 1e6)


def main():
    out = {}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    out["gpu"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    # noise at 300 k
    P = 300_000
    g = torch.Generator(device=DEV).manual_seed(0)
    f = lambda *s: torch.randn(*s, device=DEV, generator=g)
    xyz, scaling, rotation, opacity, eta = f(P, 3) * 0.4, f(P, 3) * 0.9 - 5.0, f(P, 4), f(P, 1) * 3 - 2.0, f(P, 3)
    params = dict(xyz=xyz.clone(), scaling=scaling, rotation=rotation, opacity=opacity)
    ours = events(lambda: mcmc.inject_noise(params, 1.6e-4, eta=eta), 200)
    x2 = xyz.clone()
    comp = events(lambda: torch_noise(x2, scaling, rotation, opacity, eta, 80.0), 200)
    ref = xyz.clone()
    torch_noise(ref, scaling, rotation, opacity, eta, 80.0)
    mine = dict(xyz=xyz.clone(), scaling=scaling, rotation=rotation, opacity=opacity)
    mcmc.inject_noise(mine, 1.6e-4, eta=eta)
    out["noise_300k"] = dict(kernel_ms=ours, torch_composed_ms=comp, speedup=comp / ours, algorithmic_MB=P * 68 / 1e6,
                             kernel_GBps=P * 68 / 1e9 / (ours / 1e3),
                             max_abs_diff_vs_torch=float((mine["xyz"] - ref).abs().max()))
    surgery("synthetic_300k", synthetic_body(300_000, sh_degree=3, seed=0), out)
    surgery("sample_ply_531k", sample_ply_scene(None, 3), out)
    from test_gpu_mcmc import train_mcmc
    r = train_mcmc()
    out["training_loop"] = dict(first5=sum(r["losses"][:5]) / 5, last5=sum(r["losses"][-5:]) / 5, sizes=r["sizes"][::50] + r["sizes"][-1:],
                                moved=r["moved"])
    out["training_loop"]["loss_ratio"] = out["training_loop"]["last5"] / out["training_loop"]["first5"]
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
