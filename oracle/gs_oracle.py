"""ctypes binding of the CPU oracle (oracle/gs_oracle.c).

TEST INFRASTRUCTURE ONLY -- importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs; never from humangaussian_b200/.

PARITY UNPINNED for the rasteriser kernel semantics (see gs_oracle.c header): the algorithm is
the un-vendored diff_gaussian_rasterization package, restated from SURVEY.md Appendix A.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libgs_oracle.so")
_lib = None

_F = C.POINTER(C.c_float)
_I = C.POINTER(C.c_int)


def build(force: bool = False) -> str:
    """Compile the oracle with the committed Makefile (gcc only; no reference sources involved)."""
    src = os.path.join(_HERE, "gs_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = C.CDLL(_LIB_PATH)
        L.gso_create.restype = C.c_void_p
        L.gso_destroy.argtypes = [C.c_void_p]
        L.gso_set_threads.argtypes = [C.c_void_p, C.c_int]
        L.gso_forward.restype = C.c_int
        L.gso_forward.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_float] * 3 + [C.c_void_p] * 15
        L.gso_backward.restype = C.c_int
        L.gso_backward.argtypes = [C.c_void_p] * 12 + [C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
        L.gso_num_rendered.restype = C.c_int64
        L.gso_num_rendered.argtypes = [C.c_void_p]
        for name in ("keys", "point_list", "ranges", "xy", "depths", "conic_opacity", "rgb", "cov3d",
                     "tiles_touched", "rect", "clamped", "final_T", "n_contrib", "contrib_patches"):
            fn = getattr(L, "gso_" + name)
            fn.restype = C.c_void_p
            fn.argtypes = [C.c_void_p]
        L.gso_exp.restype = C.c_float
        L.gso_exp.argtypes = [C.c_float]
        _lib = L
    return _lib


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _view(addr, dtype, count):
    if count == 0 or not addr:
        return np.zeros(0, dtype=dtype)
    buf = (C.c_char * (count * np.dtype(dtype).itemsize)).from_address(addr)
    return np.frombuffer(buf, dtype=dtype, count=count).copy()


def gs_exp(x):
    """The oracle's deterministic exp, elementwise over an array (slow; for pinning tests)."""
    L = lib()
    x = np.asarray(x, dtype=np.float32)
    return np.array([L.gso_exp(float(v)) for v in x.ravel()], dtype=np.float32).reshape(x.shape)


class Oracle:
    """One rasterisation context.  forward() then (optionally) backward() on the same view."""

    def __init__(self, threads: int = 0):
        self.L = lib()
        self.h = C.c_void_p(self.L.gso_create())
        self.L.gso_set_threads(self.h, int(threads))
        self._keep = None

    def __del__(self):
        try:
            self.L.gso_destroy(self.h)
        except Exception:
            pass

    def forward(self, *, means3D, opacities, viewmatrix, projmatrix, campos, bg, image_height, image_width,
                tanfovx, tanfovy, sh_degree=0, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, scale_modifier=1.0):
        """Arguments mirror GaussianRasterizationSettings + GaussianRasterizer.forward
        (call sites gaussiansplatting/gaussian_renderer/__init__.py:36-49,86-94).
        viewmatrix/projmatrix are the row-vector-convention 4x4 tensors of scene/cameras.py:50-52."""
        means3D = _f32(means3D)
        P = means3D.shape[0]
        shs = _f32(shs)
        M = 0 if shs is None else shs.shape[1]
        a = dict(means=means3D, shs=shs, colors=_f32(colors_precomp), opac=_f32(opacities).reshape(-1),
                 scales=_f32(scales), rots=_f32(rotations), cov=_f32(cov3D_precomp), bg=_f32(bg),
                 view=_f32(viewmatrix).reshape(-1), proj=_f32(projmatrix).reshape(-1), campos=_f32(campos))
        H, W = int(image_height), int(image_width)
        color = np.zeros((3, H, W), np.float32)
        depth = np.zeros((1, H, W), np.float32)
        alpha = np.zeros((1, H, W), np.float32)
        radii = np.zeros(P, np.int32)
        rc = self.L.gso_forward(self.h, P, int(sh_degree), M, H, W, float(tanfovx), float(tanfovy),
                                float(scale_modifier), _ptr(a["means"]), _ptr(a["shs"]), _ptr(a["colors"]),
                                _ptr(a["opac"]), _ptr(a["scales"]), _ptr(a["rots"]), _ptr(a["cov"]), _ptr(a["bg"]),
                                _ptr(a["view"]), _ptr(a["proj"]), _ptr(a["campos"]), _ptr(color), _ptr(depth),
                                _ptr(alpha), _ptr(radii))
        if rc != 0:
            raise ValueError(f"gso_forward failed with code {rc} (bad argument combination)")
        self._keep = a
        self.P, self.M, self.H, self.W = P, M, H, W
        self.ntiles = ((W + 15) // 16) * ((H + 15) // 16)
        return color, radii, depth, alpha

    def state(self):
        """Intermediate buffers of the last forward (copies)."""
        L, h, P = self.L, self.h, self.P
        D = int(L.gso_num_rendered(h))
        return dict(
            num_rendered=D,
            keys=_view(L.gso_keys(h), np.uint64, D),
            point_list=_view(L.gso_point_list(h), np.uint32, D),
            ranges=_view(L.gso_ranges(h), np.uint32, 2 * self.ntiles).reshape(-1, 2),
            xy=_view(L.gso_xy(h), np.float32, 2 * P).reshape(-1, 2),
            depths=_view(L.gso_depths(h), np.float32, P),
            conic_opacity=_view(L.gso_conic_opacity(h), np.float32, 4 * P).reshape(-1, 4),
            rgb=_view(L.gso_rgb(h), np.float32, 3 * P).reshape(-1, 3),
            cov3d=_view(L.gso_cov3d(h), np.float32, 6 * P).reshape(-1, 6),
            tiles_touched=_view(L.gso_tiles_touched(h), np.uint32, P),
            rect=_view(L.gso_rect(h), np.int32, 4 * P).reshape(-1, 4),
            clamped=_view(L.gso_clamped(h), np.uint8, 3 * P).reshape(-1, 3),
            final_T=_view(L.gso_final_T(h), np.float32, self.H * self.W).reshape(self.H, self.W),
            n_contrib=_view(L.gso_n_contrib(h), np.uint32, self.H * self.W).reshape(self.H, self.W),
            # per sorted instance: bit p = an in-image pixel of patch p = ((py % 16) // 4) * 2 + (px % 16) // 8 blended it
            contrib_patches=_view(L.gso_contrib_patches(h), np.uint8, D),
        )

    def backward(self, dL_dcolor, dL_ddepth, dL_dalpha, sums_err_const=None):
        """Gradients in the order GaussianRasterizer.backward returns them (SURVEY.md A.8).

        sums_err_const (optional float): also return out["sums"] [P,10], the float64 per-Gaussian sums in the CUDA backward
        blend's moments format (S0, Sx, Sy, Sxx, Sxy, Syy, W0..W3), and out["sums_err"] [P,10], their error scales with
        this constant in the per-term weight (gs_oracle.c, gso_backward); and out["screen_sums"] [P,10], the float64 sums the
        oracle's own screen-space gradients are rounded from (dL/dmean2D x/y, dL/dA, dL/dB / 2, dL/dC, dL/dopacity, colour, depth)."""
        P, M = self.P, self.M
        a = self._keep
        gc, gd, ga = _f32(dL_dcolor), _f32(dL_ddepth), _f32(dL_dalpha)
        out = dict(means3D=np.zeros((P, 3), np.float32), means2D=np.zeros((P, 3), np.float32),
                   opacities=np.zeros((P, 1), np.float32))
        out["shs"] = np.zeros((P, M, 3), np.float32) if a["shs"] is not None else None
        out["colors_precomp"] = np.zeros((P, 3), np.float32) if a["colors"] is not None else None
        out["scales"] = np.zeros((P, 3), np.float32) if a["scales"] is not None else None
        out["rotations"] = np.zeros((P, 4), np.float32) if a["rots"] is not None else None
        out["cov3D_precomp"] = np.zeros((P, 6), np.float32) if a["cov"] is not None else None
        if sums_err_const is not None:
            out["sums"], out["sums_err"] = np.zeros((P, 10), np.float64), np.zeros((P, 10), np.float64)
            out["screen_sums"] = np.zeros((P, 10), np.float64)
        rc = self.L.gso_backward(self.h, _ptr(gc), _ptr(gd), _ptr(ga), _ptr(out["means3D"]), _ptr(out["means2D"]),
                                 _ptr(out["shs"]), _ptr(out["colors_precomp"]), _ptr(out["opacities"]),
                                 _ptr(out["scales"]), _ptr(out["rotations"]), _ptr(out["cov3D_precomp"]),
                                 float(sums_err_const or 0.0), _ptr(out.get("sums")), _ptr(out.get("sums_err")),
                                 _ptr(out.get("screen_sums")))
        if rc != 0:
            raise RuntimeError(f"gso_backward failed with code {rc}")
        return out
