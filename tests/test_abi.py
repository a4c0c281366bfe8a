"""CPU: the C-ABI shared library loads and exports every symbol include/b200gs.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

from util import ROOT

LIB = os.path.join(ROOT, "humangaussian_b200", "libb200gs.so")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        import __graft_entry__ as g
        g.build()
    return ctypes.CDLL(LIB)


def test_every_declared_symbol_is_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "b200gs.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(b200gs_[a-z_0-9]+)\s*\(", hdr))
    assert {"b200gs_forward", "b200gs_backward", "b200gs_mark_visible"} <= declared
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/b200gs.h but not exported"
    from humangaussian_b200 import rasterizer
    assert set(rasterizer.EXPORTS) == declared


def test_abi_version_4_and_size_queries_are_sane(lib):
    """ABI 4: b200gs_state_view ends with the contributor-mask region.  The library, the header and the ctypes mirror agree."""
    sz, i32, i64 = ctypes.c_size_t, ctypes.c_int32, ctypes.c_int64
    lib.b200gs_geom_bytes.restype = sz; lib.b200gs_geom_bytes.argtypes = [i32, i32]
    lib.b200gs_image_bytes.restype = sz; lib.b200gs_image_bytes.argtypes = [i32, i32, i32]
    lib.b200gs_binning_bytes.restype = sz; lib.b200gs_binning_bytes.argtypes = [i64, i32, i32, i32, i32]
    lib.b200gs_backward_scratch_bytes.restype = sz; lib.b200gs_backward_scratch_bytes.argtypes = [i32, i32]
    from humangaussian_b200 import rasterizer
    hdr = open(os.path.join(ROOT, "include", "b200gs.h")).read()
    assert re.search(r"#define B200GS_ABI_VERSION 4\b", hdr)
    assert lib.b200gs_abi_version() == 4 and rasterizer.ABI_VERSION == 4
    assert [f[0] for f in rasterizer._StateView._fields_][-2:] == ["contributor_masks", "contributor_mask_words"]
    assert lib.b200gs_geom_bytes(1000, 1) >= 1000 * (48 + 4 + 4 + 8 + 1)
    assert lib.b200gs_geom_bytes(1000, 4) >= 4 * 1000 * 65
    assert lib.b200gs_image_bytes(64, 64, 2) >= 2 * 64 * 64 * 8
    a, b = lib.b200gs_binning_bytes(1000, 64, 64, 100, 1), lib.b200gs_binning_bytes(100000, 64, 64, 100, 1)
    assert b > a >= 1000 * 16 + 100 * 16  # 16 B per instance + 16 B per Gaussian (depth pre-sort: 4 B keys + indices, ping-pong)
    assert lib.b200gs_backward_scratch_bytes(1000, 2) >= 2000 * 48


def test_product_never_imports_the_oracle():
    """The oracle is test infrastructure: nothing under humangaussian_b200/ or diff_gaussian_rasterization/ may touch it."""
    for pkg in ("humangaussian_b200", "diff_gaussian_rasterization"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, pkg)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h")):
                    src = open(os.path.join(dirpath, f)).read()
                    assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f"{f} imports oracle/"
                    assert "libgs_oracle" not in src and "gso_" not in src, f"{f} links the oracle"


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from humangaussian_b200 import rasterizer
    monkeypatch.setattr(rasterizer, "_lib", None)
    monkeypatch.setattr(rasterizer, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(RuntimeError, match="no CPU/PyTorch fallback"):
        rasterizer.load_library()


def test_cpu_tensors_are_rejected():
    import torch
    from humangaussian_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    s = GaussianRasterizationSettings(16, 16, 1.0, 1.0, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)
    z = torch.zeros
    with pytest.raises(RuntimeError, match="CUDA device"):
        GaussianRasterizer(s)(means3D=z(4, 3), means2D=z(4, 3), shs=z(4, 1, 3), opacities=z(4, 1), scales=z(4, 3), rotations=z(4, 4))


def test_ctypes_structs_match_the_header_layout(tmp_path):
    """sizeof / offsetof of every struct that crosses the ABI, as gcc sees include/b200gs.h, equal the ctypes mirrors."""
    import ctypes as C
    import subprocess
    from humangaussian_b200 import densify, rasterizer
    src = tmp_path / "layout.c"
    fields = {"b200gs_params": [f[0] for f in rasterizer._Params._fields_],
              "b200gs_densify_cfg": [f[0] for f in densify._Cfg._fields_],
              "b200gs_state_view": [f[0] for f in rasterizer._StateView._fields_]}
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200gs.h"', 'int main(void){']
    for s, fs in fields.items():
        body.append(f'printf("{s} %zu\\n", sizeof({s}));')
        for f in fs:
            body.append(f'printf("{s}.{f} %zu\\n", offsetof({s}, {f}));')
    body.append("return 0;}")
    src.write_text("\n".join(body))
    exe = tmp_path / "layout"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    mirrors = {"b200gs_params": rasterizer._Params, "b200gs_densify_cfg": densify._Cfg, "b200gs_state_view": rasterizer._StateView}
    for s, cls in mirrors.items():
        assert int(got[s]) == C.sizeof(cls), s
        for f in fields[s]:
            assert int(got[f"{s}.{f}"]) == getattr(cls, f).offset, f"{s}.{f}"


def test_packed_layout_is_dist_pack_layout():
    """rasterize_views_packed reads the buffer dist.pack writes: same field order, same views (pure torch, CPU)."""
    import torch
    from humangaussian_b200 import dist as D
    from humangaussian_b200 import rasterizer as R
    P, K = 7, 4
    g = torch.Generator().manual_seed(0)
    t = {k: torch.randn(*shape, generator=g) for k, shape in D.field_shapes(P, K).items()}
    flat = D.pack(t)
    assert flat.numel() == R.packed_numel(P, K)
    for got, want in zip(R._split_packed(flat, P, K), (t[k] for k in D.FIELDS)):
        assert torch.equal(got, want) and got.data_ptr() >= flat.data_ptr()
    with __import__("pytest").raises((RuntimeError, ValueError)):
        R.rasterize_views_packed(flat, P, K, viewmatrices=torch.eye(4)[None], projmatrices=torch.eye(4)[None], camposs=torch.zeros(1, 3),
                                 tanfovx=[1.0], tanfovy=[1.0], image_height=8, image_width=8, bg=torch.zeros(3))  # CPU tensors: no fallback


def test_packed_layout_fields_are_16_byte_aligned_for_any_P():
    import torch
    from humangaussian_b200 import dist as D
    from humangaussian_b200 import rasterizer as R
    for P in (1, 2, 3, 5, 531327, 300000):
        for K in (1, 4, 16):
            fields, total = R.packed_layout(P, K)
            assert all(o % 4 == 0 for o, _, _ in fields) and total % 4 == 0
            assert total >= P * (11 + 3 * K) and total - P * (11 + 3 * K) < 5 * 4
            if P % 4 == 0:
                assert total == P * (11 + 3 * K)  # back to back: nothing changes for the bench configuration
    P, K = 5, 4
    g = torch.Generator().manual_seed(1)
    t = {k: torch.randn(*shape, generator=g) for k, shape in D.field_shapes(P, K).items()}
    back = D.unpack(D.pack(t), P, K)
    assert all(torch.equal(back[k], t[k]) for k in t)


def test_state_pool_parks_and_reuses_buffer_sets():
    """Host logic of the state-buffer pool (no GPU): sets return when their owner is collected, are handed out again for the
    same key, and parking is bounded."""
    import gc
    import torch
    from humangaussian_b200 import rasterizer as R
    pool = R._StatePool(max_bytes=3000)
    mk = lambda n: dict(geom=torch.empty(n, dtype=torch.uint8), image=torch.empty(n, dtype=torch.uint8))
    assert pool.take("k") is None
    a = mk(500)
    pool.give("k", a)
    assert pool.parked == 1000 and pool.take("other") is None
    assert pool.take("k") is a and pool.parked == 0 and pool.take("k") is None
    pool.give("k", a)
    pool.give("k", mk(500))
    pool.give("k", mk(600))            # 1000 + 1000 + 1200 > 3000: dropped, not parked
    assert pool.parked == 2000 and len(pool.free["k"]) == 2
    pool.clear()
    assert pool.parked == 0 and pool.take("k") is None
    # the autograd state object hands its set back when it dies (weakref.finalize, as _forward_impl wires it)
    import weakref
    st = R._Ctx()
    bufs = mk(100)
    weakref.finalize(st, pool.give, "ctx", bufs)
    assert pool.take("ctx") is None
    del st
    gc.collect()
    assert pool.take("ctx") is bufs
    e = R.InstanceLimitError(1 << 32)
    assert e.count == 1 << 32 and "4294967296" in str(e) and isinstance(e, RuntimeError)


def test_view_batch_sink_hands_each_view_its_gradient_row():
    """renderer._StackSinks (pure autograd, no GPU): the [V,P,3] batch sink aliases V leaf tensors; backward fills each
    leaf's .grad with its row, which is what the reference's hook sums (GaussianDreamer.py:385-387)."""
    import torch
    from humangaussian_b200.renderer import _StackSinks
    V, P = 4, 6
    base = torch.zeros(V, P, 3)
    sinks = [t.requires_grad_(True) for t in base.unbind(0)]
    m = _StackSinks.apply(base, *sinks)
    m.retain_grad()
    assert m.shape == (V, P, 3) and m.data_ptr() == base.data_ptr()      # forward copies nothing
    w = torch.arange(V * P * 3, dtype=torch.float32).reshape(V, P, 3)
    (m * w).sum().backward()
    for v in range(V):
        assert sinks[v].is_leaf and torch.equal(sinks[v].grad, w[v])
    assert torch.equal(m.grad, w)
    # the hook body of the reference, verbatim
    viewspace_point_tensor_grad = torch.zeros_like(sinks[0])
    for idx in range(len(sinks)):
        viewspace_point_tensor_grad = viewspace_point_tensor_grad + sinks[idx].grad
    assert torch.equal(viewspace_point_tensor_grad, w.sum(0))
