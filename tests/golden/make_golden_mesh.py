"""Golden density fields for mesh export, produced by RUNNING THE REFERENCE'S OWN `GaussianModel.extract_fields`
(gs_renderer.py:241-331) on the CPU.

    HUMANGAUSSIAN_ROOT=<HumanGaussian checkout> python tests/golden/make_golden_mesh.py   ->  tests/golden/ref_mesh_fields.npz

The reference hard-codes device="cuda" and imports modules this path does not use; it is run here unmodified by
patching torch.zeros to ignore the device keyword and stubbing `plyfile`, `kiui` (lo, sh, mesh, mesh_utils),
`diff_gaussian_rasterization` and `simple_knn`.  Case (a), the full scene at 64^3, takes a few minutes.

Cases (raw GaussianModel fields in, occ / center / scale out):
  a  content/sample.ply (tests/golden/sample_ply_full.npz; its inputs are not repeated here), 64^3, 16 blocks
  b  the 8k subsample (tests/golden/sample_ply_8k.npz), 40^3, 16 blocks: split 2 gives 20 chunks per axis
  c  the 8k subsample, 33^3, 8 blocks: the last chunk has one sample
  d  a seeded synthetic scene of 3000 Gaussians with sigma comparable to a block, 32^3, 8 blocks, relax_ratio 0.5,
     so that which Gaussians count for which block shows in the field
No reference source is copied into the repository; the reference is not needed to run the tests.
"""
import os
import sys
import time
import types

import numpy as np
import torch

REF = os.environ["HUMANGAUSSIAN_ROOT"]
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def _patch():
    orig = torch.zeros

    def zeros(*a, **k):
        k.pop("device", None)
        return orig(*a, **k)
    torch.zeros = zeros
    stubs = {
        "plyfile": dict(PlyData=object, PlyElement=object),
        "diff_gaussian_rasterization": dict(GaussianRasterizationSettings=object, GaussianRasterizer=object),
        "simple_knn": {}, "simple_knn._C": dict(distCUDA2=None),
        "kiui": dict(lo=lambda *a, **k: None), "kiui.sh": dict(eval_sh=None, SH2RGB=None, RGB2SH=None),
        "kiui.mesh": dict(Mesh=object), "kiui.mesh_utils": dict(decimate_mesh=None, clean_mesh=None),
    }
    for name, attrs in stubs.items():
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m


def sample_8k():
    c = np.load(os.path.join(HERE, "sample_ply_8k.npz"))
    st = lambda *ks: np.stack([c[k] for k in ks], 1).astype(np.float32)
    return (st("x", "y", "z"), st("opacity"), st("scale_0", "scale_1", "scale_2"), st("rot_0", "rot_1", "rot_2", "rot_3"))


def sample_full():
    d = np.load(os.path.join(HERE, "sample_ply_full.npz"))["data"]
    return d[:, 0:3].copy(), d[:, 6:7].copy(), d[:, 7:10].copy(), d[:, 10:14].copy()


def synthetic(P=3000, seed=5):
    g = np.random.default_rng(seed)
    xyz = g.uniform(-1.0, 1.0, (P, 3)).astype(np.float32)
    opacity = (g.standard_normal((P, 1)) * 1.5).astype(np.float32)
    scaling = (np.log(0.1) + 0.4 * g.standard_normal((P, 3))).astype(np.float32)
    rotation = g.standard_normal((P, 4)).astype(np.float32)
    return xyz, opacity, scaling, rotation


def run(GaussianModel, inputs, res, nb, rr):
    m = GaussianModel(0)
    m._xyz, m._opacity, m._scaling, m._rotation = (torch.tensor(a) for a in inputs)
    t = time.time()
    occ = m.extract_fields(resolution=res, num_blocks=nb, relax_ratio=rr)
    print(f"  {res}^3 / {nb} blocks, relax {rr}: {time.time() - t:.1f} s, max {occ.max().item():.4f}")
    return occ.numpy(), m.center.numpy(), np.float64(m.scale)


def main():
    _patch()
    from gs_renderer import GaussianModel
    torch.set_num_threads(os.cpu_count())
    out = {}
    s8k, syn = sample_8k(), synthetic()
    for tag, inputs, res, nb, rr, keep in (("b", s8k, 40, 16, 1.5, True), ("c", s8k, 33, 8, 1.5, False),
                                           ("d", syn, 32, 8, 0.5, True), ("a", sample_full(), 64, 16, 1.5, False)):
        print(tag)
        occ, center, scale = run(GaussianModel, inputs, res, nb, rr)
        out[f"{tag}_occ"], out[f"{tag}_center"], out[f"{tag}_scale"] = occ, center, scale
        out[f"{tag}_args"] = np.array([res, nb, rr], np.float64)
        if keep:
            for k, v in zip(("xyz", "opacity", "scaling", "rotation"), inputs):
                out[f"{tag}_{k}"] = v
    out["c_inputs_from"] = np.array("b")
    out["a_inputs_from"] = np.array("sample_ply_full.npz")
    np.savez_compressed(os.path.join(HERE, "ref_mesh_fields.npz"), **out)
    print("wrote ref_mesh_fields.npz", os.path.getsize(os.path.join(HERE, "ref_mesh_fields.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()
