"""Host side of the drop-in boundary: the `diff_gaussian_rasterization` surface over the C-ABI.

Mirrors the un-vendored package HumanGaussian imports (same names, argument meaning, error behaviour):
  * ``GaussianRasterizationSettings`` -- 12-field NamedTuple built at
    gaussiansplatting/gaussian_renderer/__init__.py:36-49 and gs_renderer.py:951-964;
  * ``GaussianRasterizer(raster_settings=...)`` -- nn.Module called with keywords
    (gaussian_renderer/__init__.py:86-94, gs_renderer.py:1006-1015) returning
    ``(color[3,H,W], radii[P] int32, depth[1,H,W], alpha[1,H,W])``, differentiable w.r.t.
    means3D, means2D (gradient sink), shs | colors_precomp, opacities, scales+rotations | cov3D_precomp.
Plus the view-batched entry ``rasterize_views`` (one call for the V cameras of an SDS batch,
threestudio/systems/GaussianDreamer.py:244-248).

Everything numerical happens in libb200gs.so (hand-written sm_90a CUDA behind include/b200gs.h),
reached through ctypes with raw device pointers.  There is NO CPU or PyTorch fallback: if the
library is missing or the tensors are not on a CUDA device this module raises.
"""
from __future__ import annotations

import ctypes as C
import os
import weakref
from typing import NamedTuple, Optional

import torch
from torch import nn

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200GS_LIB selects another build of the SAME C-ABI (only used to time baseline/libb200gs_classic.so, the
# classic-structure comparator, through the identical host path).  It is not a fallback: the default is the product.
LIB_PATH = os.environ.get("B200GS_LIB") or os.path.join(_HERE, "libb200gs.so")
ABI_VERSION = 5
MAX_VIEWS = 64
MAX_INSTANCES = 0x7FFFFFFF  # (Gaussian, tile) instances per call (B200GS_MAX_INSTANCES); larger batches are split by views

OK, E_ARGS, E_BIN_TOO_SMALL, E_BUFFER, E_CUDA, E_RANGE, E_INSTANCES, E_UNSUPPORTED = 0, -1, -2, -3, -4, -5, -6, -7


class InstanceLimitError(RuntimeError):
    """The view batch has more (Gaussian, tile) instances than one call supports (B200GS_E_INSTANCES).  `rasterize_views`
    catches it and renders the batch in two halves; a single view that exceeds the limit propagates it."""

    def __init__(self, count):
        super().__init__(f"b200gs: {count} (Gaussian, tile) instances in one call exceed the supported {MAX_INSTANCES}; "
                         "render fewer views per call")
        self.count = count


class _Params(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("P", C.c_int32), ("n_views", C.c_int32), ("sh_degree", C.c_int32),
                ("sh_coeffs", C.c_int32), ("image_height", C.c_int32), ("image_width", C.c_int32),
                ("prefiltered", C.c_int32), ("debug", C.c_int32), ("scale_modifier", C.c_float),
                ("tanfovx", C.POINTER(C.c_float)), ("tanfovy", C.POINTER(C.c_float)), ("means3D_per_view", C.c_int32),
                ("raw_params", C.c_int32)]


class _RenderOpts(C.Structure):
    """b200gs_render_opts (include/b200gs.h): options of the *_opts entry points; a NULL buffer turns its feature off"""
    _fields_ = ([("struct_bytes", C.c_int32), ("antialiasing", C.c_int32), ("filter3d_var", C.c_void_p)] +
                [(n, C.c_void_p) for n in ("gauss_normals", "out_normal", "dL_dnormal", "normal_wn", "nrm_partials")] +
                [("nrm_partials_bytes", C.c_size_t)] +
                [(n, C.c_void_p) for n in ("median_pos", "out_median", "out_depth2", "dL_dmedian", "dL_ddepth2", "weight_sum",
                                           "weight_max", "touches", "dL_dmeans2D_abs", "abs_partials")] +
                [("abs_partials_bytes", C.c_size_t)])


def _render_opts(antialiasing: bool, filter_3d: Optional[torch.Tensor] = None, **buffers):
    """b200gs_render_opts: the two filters, and feature buffers by field name (tensors, None = absent).  A *_partials
    buffer (uint8) also sets its *_bytes field."""
    o = _RenderOpts(C.sizeof(_RenderOpts), int(bool(antialiasing)), None if filter_3d is None else filter_3d.data_ptr())
    for name, t in buffers.items():
        if t is not None:
            setattr(o, name, _ptr(t))
            if name.endswith("_partials"):
                setattr(o, name + "_bytes", t.numel())
    return o


def _opts_or_plain(plain, with_opts, antialiasing, filter_3d, **buffers):
    """The entry point to call and its options: the plain one when every option is off (b200gs_forward and friends equal
    their *_opts form with NULL options), else the *_opts form with `opts` bound after `prm`."""
    if not antialiasing and filter_3d is None and all(t is None for t in buffers.values()):
        return plain
    opts = _render_opts(antialiasing, filter_3d, **buffers)
    return lambda prm, *a: with_opts(prm, C.byref(opts), *a)


def _check_filter_3d(filter_3d, P, device, cov3D_precomp=None):
    """The 3D smoothing filter's variances: a [P] fp32 tensor on the Gaussians' device, or None.  The values are the
    caller's contract (finite, >= 0; filter3d.compute_filter_3d meets it); checking them would cost a host sync."""
    if filter_3d is None:
        return None
    if cov3D_precomp is not None:
        raise ValueError("b200gs: the 3D filter widens scales; it cannot be used with cov3D_precomp")
    if not isinstance(filter_3d, torch.Tensor) or filter_3d.dtype != torch.float32 or filter_3d.device != device or \
            filter_3d.dim() != 1 or filter_3d.shape[0] != P:
        raise ValueError(f"b200gs: filter_3d must be a [{P}] float32 tensor on {device} (recompute it after densify / prune); got "
                         f"{tuple(filter_3d.shape) if isinstance(filter_3d, torch.Tensor) else type(filter_3d).__name__}"
                         f"{'' if not isinstance(filter_3d, torch.Tensor) else f' {filter_3d.dtype} on {filter_3d.device}'}")
    return filter_3d.detach().contiguous()


class _StateView(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("geom_records", "tiles_touched", "offsets", "clamped", "sorted_tile_keys",
                                          "depth_order", "point_list", "ranges", "final_T", "n_contrib",
                                          "contributor_masks")] + [("contributor_mask_words", C.c_int64)]


_lib = None
EXPORTS = ["b200gs_forward", "b200gs_backward", "b200gs_mark_visible", "b200gs_describe_state", "b200gs_test_exp",
           "b200gs_geom_bytes", "b200gs_image_bytes", "b200gs_binning_bytes", "b200gs_backward_scratch_bytes",
           "b200gs_last_cuda_error", "b200gs_abi_version", "b200gs_launch_count", "b200gs_profile_enable", "b200gs_profile_read",
           "b200gs_test_sort_pairs", "b200gs_test_sort_scratch_bytes", "b200gs_reattach", "b200gs_pack_frames_u8",
           "b200gs_knn_scratch_bytes", "b200gs_dist2_knn3", "b200gs_densify_stats", "b200gs_densify_scratch_bytes",
           "b200gs_densify_plan", "b200gs_densify_move", "b200gs_adam_packed", "b200gs_deterministic_bytes",
           "b200gs_backward_deterministic", "b200gs_forward_opts", "b200gs_backward_opts",
           "b200gs_backward_deterministic_opts", "b200gs_sampling_rate", "b200gs_prune_plan", "b200gs_mcmc_noise",
           "b200gs_mcmc_ratio", "b200gs_mcmc_move", "b200gs_density_field_scratch_bytes", "b200gs_density_field",
           "b200gs_field_query_scratch_bytes", "b200gs_field_query",
           "b200gs_marching_cubes_scratch_bytes", "b200gs_marching_cubes_count", "b200gs_marching_cubes_emit",
           "b200gs_pose_scratch_bytes", "b200gs_pose_keypoints", "b200gs_pose_draw",
           "b200gs_mesh_raster_scratch_bytes", "b200gs_mesh_raster_count", "b200gs_mesh_raster_emit", "b200gs_mesh_interpolate",
           "b200gs_mesh_incidence_bytes", "b200gs_mesh_incidence", "b200gs_mesh_vertex_normals", "b200gs_mesh_normal_image",
           "b200gs_mesh_clean_scratch_bytes", "b200gs_mesh_clean", "b200gs_mesh_decimate_scratch_bytes", "b200gs_mesh_decimate"]
STAGES = ["preprocess_fwd", "scan", "binning", "blend_fwd", "blend_bwd", "preprocess_bwd"]


def load_library():
    """dlopen libb200gs.so and declare signatures.  Raises (never falls back) if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"b200gs: {LIB_PATH} not built -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a).  There is no CPU/PyTorch fallback for the rasteriser.")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t
    L.b200gs_abi_version.restype = C.c_int
    if L.b200gs_abi_version() != ABI_VERSION:
        raise RuntimeError("b200gs: ABI version mismatch between rasterizer.py and libb200gs.so")
    L.b200gs_geom_bytes.restype = sz; L.b200gs_geom_bytes.argtypes = [i32, i32]
    L.b200gs_image_bytes.restype = sz; L.b200gs_image_bytes.argtypes = [i32, i32, i32]
    L.b200gs_binning_bytes.restype = sz; L.b200gs_binning_bytes.argtypes = [i64, i32, i32, i32, i32]
    L.b200gs_backward_scratch_bytes.restype = sz; L.b200gs_backward_scratch_bytes.argtypes = [i32, i32]
    L.b200gs_forward.restype = C.c_int
    L.b200gs_forward.argtypes = [C.POINTER(_Params)] + [vp] * 15 + [vp, sz, vp, sz, i64, vp, sz, C.POINTER(i64), vp]
    L.b200gs_backward.restype = C.c_int
    L.b200gs_backward.argtypes = [C.POINTER(_Params)] + [vp] * 12 + [vp, vp, i64, vp, i64] + [vp] * 11 + [vp, sz, vp]
    L.b200gs_deterministic_bytes.restype = sz; L.b200gs_deterministic_bytes.argtypes = [i64, i64, i32, i32]
    L.b200gs_backward_deterministic.restype = C.c_int
    L.b200gs_backward_deterministic.argtypes = ([C.POINTER(_Params)] + [vp] * 12 + [vp, vp, i64, vp, i64] + [vp] * 11 + [vp, sz] +
                                                [vp, sz, i64, C.POINTER(i64), vp])
    # the *_opts forms: the same argument lists with the options pointer after prm
    L.b200gs_forward_opts.restype = C.c_int
    L.b200gs_forward_opts.argtypes = [L.b200gs_forward.argtypes[0], vp] + L.b200gs_forward.argtypes[1:]
    L.b200gs_backward_opts.restype = C.c_int
    L.b200gs_backward_opts.argtypes = [L.b200gs_backward.argtypes[0], vp] + L.b200gs_backward.argtypes[1:]
    L.b200gs_backward_deterministic_opts.restype = C.c_int
    L.b200gs_backward_deterministic_opts.argtypes = ([L.b200gs_backward_deterministic.argtypes[0], vp] +
                                                     L.b200gs_backward_deterministic.argtypes[1:])
    L.b200gs_sampling_rate.restype = C.c_int
    L.b200gs_sampling_rate.argtypes = [i32, i32, vp, vp, C.POINTER(C.c_float), C.POINTER(C.c_float), i32, i32, vp, vp]
    L.b200gs_mark_visible.restype = C.c_int
    L.b200gs_mark_visible.argtypes = [i32, vp, vp, vp, vp, vp]
    L.b200gs_describe_state.restype = C.c_int
    L.b200gs_describe_state.argtypes = [C.POINTER(_Params), vp, vp, i64, vp, C.POINTER(_StateView)]
    L.b200gs_test_exp.restype = C.c_int
    L.b200gs_test_exp.argtypes = [vp, vp, i64, vp]
    L.b200gs_test_sort_pairs.restype = C.c_int
    L.b200gs_test_sort_pairs.argtypes = [vp, vp, vp, vp, i64, i32, vp, sz, C.POINTER(i32), vp]
    L.b200gs_test_sort_scratch_bytes.restype = sz; L.b200gs_test_sort_scratch_bytes.argtypes = [i64]
    L.b200gs_reattach.restype = C.c_int
    L.b200gs_reattach.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp]
    L.b200gs_pack_frames_u8.restype = C.c_int
    L.b200gs_pack_frames_u8.argtypes = [vp, vp, i32, i32, i32, vp]
    L.b200gs_knn_scratch_bytes.restype = sz; L.b200gs_knn_scratch_bytes.argtypes = [i32]
    L.b200gs_dist2_knn3.restype = C.c_int
    L.b200gs_dist2_knn3.argtypes = [i32, vp, vp, vp, sz, vp]
    L.b200gs_densify_stats.restype = C.c_int
    L.b200gs_densify_stats.argtypes = [i32, i32, vp, vp, vp, vp, vp, vp, vp]
    L.b200gs_densify_scratch_bytes.restype = sz; L.b200gs_densify_scratch_bytes.argtypes = [i32]
    L.b200gs_densify_plan.restype = C.c_int
    L.b200gs_densify_plan.argtypes = [i32, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.b200gs_prune_plan.restype = C.c_int
    L.b200gs_prune_plan.argtypes = [i32, vp, vp, vp, vp, sz, vp]
    L.b200gs_densify_move.restype = C.c_int
    L.b200gs_densify_move.argtypes = [i32, i32, i32, vp, C.POINTER(i32), i32, vp, vp, vp, vp, vp, vp]
    L.b200gs_mcmc_noise.restype = C.c_int
    L.b200gs_mcmc_noise.argtypes = [i32, vp, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float, vp]
    L.b200gs_mcmc_ratio.restype = C.c_int
    L.b200gs_mcmc_ratio.argtypes = [i32, vp, vp, vp, vp, vp, vp]
    L.b200gs_mcmc_move.restype = C.c_int
    L.b200gs_mcmc_move.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp]
    L.b200gs_adam_packed.restype = C.c_int
    L.b200gs_adam_packed.argtypes = [vp, vp, vp, vp, vp, vp]
    L.b200gs_density_field_scratch_bytes.restype = sz; L.b200gs_density_field_scratch_bytes.argtypes = [i32, i32, i32]
    L.b200gs_density_field.restype = C.c_int
    L.b200gs_density_field.argtypes = [i32, vp, vp, vp, i32, i32, vp, C.c_float, vp, vp, sz, vp]
    L.b200gs_field_query_scratch_bytes.restype = sz; L.b200gs_field_query_scratch_bytes.argtypes = [i32, i32, i32, i32, i32]
    L.b200gs_field_query.restype = C.c_int
    L.b200gs_field_query.argtypes = [i32, vp, vp, vp, vp, i32, i32, i32, i32, vp, C.c_float, i32, vp, vp, vp, vp, vp, sz, vp]
    L.b200gs_pose_scratch_bytes.restype = sz; L.b200gs_pose_scratch_bytes.argtypes = [i32, i32, i32, i32]
    L.b200gs_pose_keypoints.restype = C.c_int
    L.b200gs_pose_keypoints.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, sz, vp]
    L.b200gs_pose_draw.restype = C.c_int
    L.b200gs_pose_draw.argtypes = [i32, i32, i32, i32, vp, vp, sz, vp, vp]
    L.b200gs_marching_cubes_scratch_bytes.restype = sz; L.b200gs_marching_cubes_scratch_bytes.argtypes = [i32, i32, i32]
    L.b200gs_marching_cubes_count.restype = C.c_int
    L.b200gs_marching_cubes_count.argtypes = [i32, i32, i32, vp, C.c_float, vp, sz, vp, vp]
    L.b200gs_marching_cubes_emit.restype = C.c_int
    L.b200gs_marching_cubes_emit.argtypes = [i32, i32, i32, vp, C.c_float, vp, sz, vp, vp, vp]
    L.b200gs_mesh_raster_scratch_bytes.restype = sz; L.b200gs_mesh_raster_scratch_bytes.argtypes = [i32, i32, i32, i32]
    L.b200gs_mesh_raster_count.restype = C.c_int
    L.b200gs_mesh_raster_count.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, sz, vp, vp]
    L.b200gs_mesh_raster_emit.restype = C.c_int
    L.b200gs_mesh_raster_emit.argtypes = [i32, i32, i32, i32, i32, vp, sz, vp, sz, vp, vp]
    L.b200gs_mesh_interpolate.restype = C.c_int
    L.b200gs_mesh_interpolate.argtypes = [i32, i32, i32, i32, i32, i32, vp, i32, vp, vp, vp, vp]
    L.b200gs_mesh_incidence_bytes.restype = sz; L.b200gs_mesh_incidence_bytes.argtypes = [i32, i32]
    L.b200gs_mesh_incidence.restype = C.c_int
    L.b200gs_mesh_incidence.argtypes = [i32, i32, vp, vp, sz, vp]
    L.b200gs_mesh_vertex_normals.restype = C.c_int
    L.b200gs_mesh_vertex_normals.argtypes = [i32, i32, i32, vp, vp, vp, sz, vp, vp]
    L.b200gs_mesh_normal_image.restype = C.c_int
    L.b200gs_mesh_normal_image.argtypes = [i32, i32, i32, i32, i32, vp, i32, vp, vp, vp, vp]
    L.b200gs_mesh_clean_scratch_bytes.restype = sz; L.b200gs_mesh_clean_scratch_bytes.argtypes = [i32, i32]
    L.b200gs_mesh_clean.restype = C.c_int
    L.b200gs_mesh_clean.argtypes = [i32, i32, vp, vp, i32, C.c_double, vp, sz, vp, vp, C.POINTER(i64), C.POINTER(i32), vp]
    L.b200gs_mesh_decimate_scratch_bytes.restype = sz; L.b200gs_mesh_decimate_scratch_bytes.argtypes = [i32, i32]
    L.b200gs_mesh_decimate.restype = C.c_int
    L.b200gs_mesh_decimate.argtypes = [i32, i32, vp, vp, i32, vp, sz, vp, vp, C.POINTER(i64), C.POINTER(i32), vp]
    L.b200gs_last_cuda_error.restype = C.c_char_p
    L.b200gs_launch_count.restype = i64
    L.b200gs_profile_enable.restype = None; L.b200gs_profile_enable.argtypes = [C.c_int]
    L.b200gs_profile_read.restype = C.c_int
    L.b200gs_profile_read.argtypes = [C.POINTER(C.c_double), C.POINTER(i64), i32]
    _lib = L
    return L


class use_library:
    """Context manager: run the SAME host path against another build of the C-ABI (bench.py times
    baseline/libb200gs_classic.so, the classic-structure CUDA comparator, next to the product in one process).
    Not a fallback mechanism: outside the `with` block the product library is back."""

    def __init__(self, path):
        self.path = path

    def __enter__(self):
        global _lib, LIB_PATH
        self.saved = (_lib, LIB_PATH)
        _lib, LIB_PATH = None, self.path
        _pool.clear()
        _det_pool.clear()
        return load_library()

    def __exit__(self, *exc):
        global _lib, LIB_PATH
        _lib, LIB_PATH = self.saved
        _pool.clear()
        _det_pool.clear()
        return False


def launch_count() -> int:
    return int(load_library().b200gs_launch_count())


def profile_enable(on: bool):
    load_library().b200gs_profile_enable(int(bool(on)))


def profile_read():
    """{stage: (total_ms, calls)} accumulated since the last read (CUDA events on the launch stream)."""
    n = len(STAGES)
    ms, calls = (C.c_double * n)(), (C.c_int64 * n)()
    _check(load_library().b200gs_profile_read(ms, calls, n), "profile_read")
    return {STAGES[i]: (float(ms[i]), int(calls[i])) for i in range(n)}


def _check(rc, what):
    if rc == OK:
        return
    L = load_library()
    msg = {E_ARGS: "inconsistent arguments", E_BUFFER: "state buffer too small", E_RANGE: "size outside supported range",
           E_INSTANCES: "too many (Gaussian, tile) instances in one call",
           E_UNSUPPORTED: "not supported by this build of the library", E_BIN_TOO_SMALL: "buffer too small after retries",
           E_CUDA: "CUDA error: " + (L.b200gs_last_cuda_error() or b"").decode()}.get(rc, f"status {rc}")
    raise RuntimeError(f"b200gs {what} failed: {msg}")


_dummy: dict = {}


def _ptr(t: Optional[torch.Tensor]):
    """Raw device pointer.  A zero-element tensor (P == 0) has a null data_ptr; the ABI treats NULL as "argument
    absent", so hand it a small valid dummy allocation instead."""
    if t is None:
        return None
    if t.numel() == 0:
        key = (t.device.type, t.device.index)
        if key not in _dummy:
            _dummy[key] = torch.zeros(64, dtype=torch.float32, device=t.device)
        return C.c_void_p(_dummy[key].data_ptr())
    return C.c_void_p(t.data_ptr())


def _f32c(t: Optional[torch.Tensor], device=None):
    if t is None:
        return None
    if device is not None and t.device != device:
        t = t.to(device)
    return t.detach().to(torch.float32).contiguous()


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


# instance-capacity hint per (device, P, V, H, W): the largest count seen so far (+25 %), so that after the first few
# cameras a call neither retries nor re-sizes its binning buffer
_cap_hint: dict = {}


_last_num_rendered = 0


def last_num_rendered() -> int:
    """Instance count D of the most recent forward call in this process (workload statistic for bench.py)."""
    return _last_num_rendered


_last_num_partials = 0


def last_num_partials() -> int:
    """Partial count H of the most recent deterministic backward call in this process (workload statistic)."""
    return _last_num_partials


class _StatePool:
    """Free lists of the opaque state buffers (geom | image | binning | backward scratch), keyed by (device, stream, sizes).
    A forward checks a set out, its autograd ctx holds it until the graph is freed, then the set returns here instead of
    going back to the allocator: the per-view calling pattern (GaussianDreamer.py:244-248) re-uses the same few sets every
    step.  Bounded: at most `max_bytes` are parked; anything beyond is simply dropped (freed by torch)."""

    def __init__(self, max_bytes=24 << 30):
        self.free: dict = {}
        self.parked = 0
        self.max_bytes = max_bytes

    def take(self, key):
        lst = self.free.get(key)
        if lst:
            bufs = lst.pop()
            self.parked -= sum(b.numel() for b in bufs.values())
            return bufs
        return None

    def give(self, key, bufs):
        n = sum(b.numel() for b in bufs.values())
        if self.parked + n > self.max_bytes:
            return
        self.free.setdefault(key, []).append(bufs)
        self.parked += n

    def clear(self):
        self.free.clear()
        self.parked = 0


_pool = _StatePool()
# the deterministic backward's work buffer (plan + partials), checked out for the duration of one backward call
_det_pool = _StatePool()
# partial-capacity hint of the deterministic backward per (device, P, V, H, W): the largest partial count seen (+25 %)
_partial_hint: dict = {}


def release_cached_buffers():
    """Drop the parked state buffers (e.g. after densification changed P)."""
    _pool.clear()
    _det_pool.clear()


class _Ctx:
    """What one forward keeps for its backward (upstream keeps geomBuffer/binningBuffer/imgBuffer the same way)."""
    __slots__ = ("prm", "tanx", "tany", "geom", "binning", "image", "scratch", "capacity", "num_rendered", "radii", "V", "P", "H",
                 "W", "M", "aa", "f3d", "gauss_normals", "normal", "normal_wn", "median", "depth2", "median_pos", "__weakref__")


def _make_params(P, V, deg, M, H, W, mod, tanx, tany, prefiltered=False, debug=False, per_view_means=False, raw=False):
    tx = (C.c_float * V)(*[float(t) for t in tanx])
    ty = (C.c_float * V)(*[float(t) for t in tany])
    prm = _Params(ABI_VERSION, P, V, int(deg), int(M), int(H), int(W), int(bool(prefiltered)), int(bool(debug)), float(mod),
                  C.cast(tx, C.POINTER(C.c_float)), C.cast(ty, C.POINTER(C.c_float)), int(bool(per_view_means)), int(bool(raw)))
    return prm, tx, ty


def _forward_impl(means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, bg, viewmatrix, projmatrix,
                  campos, tanfovx, tanfovy, H, W, sh_degree, scale_modifier, prefiltered=False, debug=False, raw=False,
                  antialiasing=False, filter_3d=None, contrib=None, normals=False, geometry=False):
    """All tensors float32 contiguous on one CUDA device.  viewmatrix/projmatrix [V,4,4], campos [V,3].
    raw: opacities / scales / rotations are GaussianModel's raw parameters (activations fused into the kernels).
    antialiasing: the screen-space mip filter; filter_3d: the 3D smoothing filter's [P] variances (b200gs_render_opts).
    The state remembers both for the backward.
    contrib: None, or the contribution accumulators (weight_sum, weight_max, touches), [P] int64 / int32 / int32 device tensors
    read as u64 / u32 / u32: the forward then folds this call's views into them.
    normals=True: the state holds the normal image `normal` [V,3,H,W] and the per-(view, Gaussian) normals `gauss_normals`
    [V,P,4] its backward reads.
    geometry=True: the state holds the images `median` and `depth2` [V,1,H,W] and the median positions `median_pos` [V,H,W]
    int32 its backward reads.
    Every option travels in b200gs_render_opts; with all of them off the plain b200gs_forward runs."""
    L = load_library()
    dev = means3D.device
    if dev.type != "cuda":
        raise RuntimeError("b200gs: tensors must live on a CUDA device (there is no CPU path)")
    V = viewmatrix.shape[0]
    per_view_means = means3D.dim() == 3  # [V,P,3]: animation frame batch
    if per_view_means and means3D.shape[0] != V:
        raise ValueError(f"per-view means3D has {means3D.shape[0]} views, cameras have {V}")
    P = means3D.shape[-2]
    if (shs is None) == (colors_precomp is None):
        raise Exception("Please provide excatly one of either SHs or precomputed colors!")
    if ((scales is None or rotations is None) and cov3D_precomp is None) or \
            ((scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
    M = 0 if shs is None else shs.shape[1]
    if normals and cov3D_precomp is not None:
        raise ValueError("b200gs: normals take each Gaussian's shortest scale axis; a precomputed covariance has none")
    if normals and contrib is not None:
        raise ValueError("b200gs: the contribution forward does not render normals")
    if geometry and contrib is not None:
        raise ValueError("b200gs: the contribution forward does not render the geometry outputs")
    filter_3d = _check_filter_3d(filter_3d, P, dev, cov3D_precomp)
    prm, tx, ty = _make_params(P, V, sh_degree, M, H, W, scale_modifier, tanfovx, tanfovy, prefiltered, debug, per_view_means, raw)
    u8 = dict(dtype=torch.uint8, device=dev)
    color = torch.empty(V, 3, H, W, dtype=torch.float32, device=dev)
    depth = torch.empty(V, 1, H, W, dtype=torch.float32, device=dev)
    alpha = torch.empty(V, 1, H, W, dtype=torch.float32, device=dev)
    radii = torch.empty(V, P, dtype=torch.int32, device=dev)
    key = (dev.index, P, V, H, W)
    cap = _cap_hint.get(key, max(1 << 16, 4 * P * V))
    n_out = C.c_int64(0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    gauss_normals = normal = median = depth2 = median_pos = None
    if normals:
        gauss_normals = torch.empty(V, P, 4, dtype=torch.float32, device=dev)
        normal = torch.empty(V, 3, H, W, dtype=torch.float32, device=dev)
    if geometry:
        median = torch.empty(V, 1, H, W, dtype=torch.float32, device=dev)
        depth2 = torch.empty(V, 1, H, W, dtype=torch.float32, device=dev)
        median_pos = torch.empty(V, H, W, dtype=torch.int32, device=dev)
    weight_sum, weight_max, touches = contrib if contrib is not None else (None, None, None)
    fwd = _opts_or_plain(L.b200gs_forward, L.b200gs_forward_opts, antialiasing, filter_3d, gauss_normals=gauss_normals,
                         out_normal=normal, median_pos=median_pos, out_median=median, out_depth2=depth2, weight_sum=weight_sum,
                         weight_max=weight_max, touches=touches)
    with torch.cuda.device(dev):
        for _ in range(3):
            pkey = (key, stream, cap)
            bufs = _pool.take(pkey)
            if bufs is None:
                bufs = dict(geom=torch.empty(L.b200gs_geom_bytes(P, V), **u8), image=torch.empty(L.b200gs_image_bytes(H, W, V), **u8),
                            binning=torch.empty(L.b200gs_binning_bytes(cap, H, W, P, V), **u8),
                            scratch=torch.empty(max(L.b200gs_backward_scratch_bytes(P, V), 16), **u8))
            geom, image, binning = bufs["geom"], bufs["image"], bufs["binning"]
            # The contribution forward folds into accumulators, so MAX_INSTANCES (which tests can lower) must stop a call before
            # its blend: it is passed as the capacity, and the library then refuses the call before binning.
            call_cap = min(cap, MAX_INSTANCES) if contrib is not None else cap
            rc = fwd(C.byref(prm), _ptr(means3D), _ptr(shs), _ptr(colors_precomp), _ptr(opacities), _ptr(scales),
                                  _ptr(rotations), _ptr(cov3D_precomp), _ptr(bg), _ptr(viewmatrix), _ptr(projmatrix),
                                  _ptr(campos), _ptr(color), _ptr(depth), _ptr(alpha), _ptr(radii), _ptr(geom), geom.numel(),
                                  _ptr(binning), binning.numel(), call_cap, _ptr(image), image.numel(), C.byref(n_out),
                                  C.c_void_p(stream))
            if n_out.value > MAX_INSTANCES and (rc == OK or (contrib is not None and rc == E_BIN_TOO_SMALL)):
                rc = E_INSTANCES  # (the library applies the same limit; this one can be lowered in tests)
            if rc != E_BIN_TOO_SMALL:
                break
            cap = int(n_out.value * 1.25) + 1024
        if rc == E_INSTANCES:
            raise InstanceLimitError(int(n_out.value))
        _check(rc, "forward")
    _cap_hint[key] = max(int(n_out.value * 1.25) + 1024, 1 << 16, _cap_hint.get(key, 0))
    global _last_num_rendered
    _last_num_rendered = int(n_out.value)
    st = _Ctx()
    st.prm, st.tanx, st.tany = prm, tx, ty
    st.geom, st.binning, st.image, st.scratch, st.capacity, st.num_rendered = geom, binning, image, bufs["scratch"], call_cap, \
        int(n_out.value)
    st.radii, st.V, st.P, st.H, st.W, st.M = radii, V, P, H, W, M
    st.aa, st.f3d = antialiasing, filter_3d  # the backward gets the same options (st keeps the variances alive)
    st.gauss_normals, st.normal, st.normal_wn = gauss_normals, normal, None
    st.median, st.depth2, st.median_pos = median, depth2, median_pos
    weakref.finalize(st, _pool.give, pkey, bufs)  # when the autograd graph drops the state, the buffers are parked for re-use
    return color, radii, depth, alpha, st


def _backward_deterministic(L, st: _Ctx, dev, args, det_state=None, **buffers):
    """b200gs_backward_deterministic with the work buffer from _det_pool, sized by the partial-capacity hint; a call whose
    partials do not fit is repeated with room for the count it reported (at most two retries).  buffers: the backward's
    option buffers (_backward_impl).  With dL_dmeans2D_abs the float2-per-partial array abs_partials, with dL_dnormal the
    float4-per-partial array nrm_partials, are pooled beside the work buffer; geometry needs no buffer of its own."""
    absgrad, nrm = buffers.get("dL_dmeans2D_abs") is not None, buffers.get("dL_dnormal") is not None
    P, V, H, W = st.P, st.V, st.H, st.W
    key = (dev.index, P, V, H, W)
    pcap = _partial_hint.get(key, max(1 << 16, 2 * st.num_rendered))
    n_out = C.c_int64(0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    for _ in range(3):
        # sized for the forward's instance capacity (>= its count), so the pool key stays the same from call to call
        pkey = (dev.index, stream, st.capacity, pcap, P, V, absgrad, nrm)
        bufs = _det_pool.take(pkey)
        if bufs is None:
            bufs = dict(det=torch.empty(L.b200gs_deterministic_bytes(st.capacity, pcap, P, V), dtype=torch.uint8, device=dev))
            if absgrad:
                bufs["abs"] = torch.empty(max(8 * pcap, 16), dtype=torch.uint8, device=dev)
            if nrm:
                bufs["nrm"] = torch.empty(max(16 * pcap, 16), dtype=torch.uint8, device=dev)
        det = bufs["det"]
        bwd = _opts_or_plain(L.b200gs_backward_deterministic, L.b200gs_backward_deterministic_opts, st.aa, st.f3d, **buffers,
                             abs_partials=bufs.get("abs"), nrm_partials=bufs.get("nrm"))
        rc = bwd(*args, _ptr(det), det.numel(), pcap, C.byref(n_out), C.c_void_p(stream))
        if rc == OK and det_state is not None:
            det_state["patch_masks"] = det[:st.num_rendered].clone()
            det_state["n_partials"] = int(n_out.value)
        _det_pool.give(pkey, bufs)  # stream-ordered: the next call on this stream runs after this one's kernels
        if rc != E_BIN_TOO_SMALL:
            break
        pcap = int(n_out.value * 1.25) + 1024
    if rc == OK:
        _partial_hint[key] = max(int(n_out.value * 1.25) + 1024, 1 << 16, _partial_hint.get(key, 0))
        global _last_num_partials
        _last_num_partials = int(n_out.value)
    return rc


def _backward_impl(st: _Ctx, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, bg, viewmatrix,
                   projmatrix, campos, g_color, g_depth, g_alpha, out=None, det_state=None, absgrad=False, g_normal=None,
                   g_median=None, g_depth2=None):
    """`out` (optional): dict of preallocated contiguous fp32 gradient buffers by name (means3D, sh, opacity, scales,
    rotations) -- the packed entry points them into one flat buffer so that B3 writes the all-reduce payload in place.

    absgrad=True: a ninth value is returned: dL_dmeans2D_abs [V,P,3], the per-pixel terms of dL_dmeans2D summed in absolute
    value (include/b200gs.h).  Every other gradient is what absgrad=False gives.

    g_normal [V,3,H,W] (a forward with normals=True): dL/dN reaches the opacities, means and colours through the blend
    weights and the rotations through the normals; st.normal_wn then holds the [V,P,4] sums Wn.  None: the call without
    normals.

    g_median, g_depth2 [V,1,H,W] (a forward with geometry=True; None = zero): dL/dM2 reaches the opacities, means and colours
    through the blend weights and the means through the depth; dL/dmedian reaches the means of each pixel's median Gaussian
    through its depth.  With both None the call is the one without geometry.

    Every option travels in b200gs_render_opts; with all of them off the plain b200gs_backward[_deterministic] runs.

    Under torch.use_deterministic_algorithms(True) the backward is the library's deterministic one: the same gradients up
    to float rounding, bit-identical from run to run (one host wait per call, for its partial count).  `det_state`
    (optional dict) then receives the per-instance patch masks ("patch_masks", uint8 [num_rendered]) and the partial count
    ("n_partials")."""
    L = load_library()
    dev = means3D.device
    P, V, M = st.P, st.V, st.M
    f = dict(dtype=torch.float32, device=dev)
    out = out or {}
    d_means3D = out.get("means3D") if "means3D" in out else torch.empty(means3D.shape, **f)  # [P,3], or [V,P,3] per-view
    d_means2D = torch.empty(V, P, 3, **f)
    d_op = out.get("opacity") if "opacity" in out else torch.empty(P, 1, **f)
    d_sh = (out.get("sh") if "sh" in out else torch.empty(P, M, 3, **f)) if shs is not None else None
    d_col = torch.empty(P, 3, **f) if colors_precomp is not None else None
    d_sc = (out.get("scales") if "scales" in out else torch.empty(P, 3, **f)) if scales is not None else None
    d_rot = (out.get("rotations") if "rotations" in out else torch.empty(P, 4, **f)) if rotations is not None else None
    d_cov = torch.empty(P, 6, **f) if cov3D_precomp is not None else None
    d_abs = torch.empty(V, P, 3, **f) if absgrad else None
    grads = (d_means3D, d_means2D, d_sh, d_col, d_op, d_sc, d_rot, d_cov) + ((d_abs,) if absgrad else ())
    if P == 0:
        return grads
    scratch = st.scratch
    args = (C.byref(st.prm), _ptr(means3D), _ptr(shs), _ptr(colors_precomp), _ptr(opacities), _ptr(scales), _ptr(rotations),
            _ptr(cov3D_precomp), _ptr(bg), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), _ptr(st.radii), _ptr(st.geom),
            _ptr(st.binning), st.capacity, _ptr(st.image), st.num_rendered, _ptr(g_color), _ptr(g_depth), _ptr(g_alpha),
            _ptr(d_means3D), _ptr(d_means2D), _ptr(d_sh), _ptr(d_col), _ptr(d_op), _ptr(d_sc), _ptr(d_rot), _ptr(d_cov),
            _ptr(scratch), scratch.numel())
    # the option buffers: the forward's filters and workspaces (from st) with the gradients that turn a feature on
    buffers = dict(dL_dmeans2D_abs=d_abs)
    if g_normal is not None and st.gauss_normals is not None:
        st.normal_wn = torch.empty(V, P, 4, **f)
        buffers.update(gauss_normals=st.gauss_normals, dL_dnormal=g_normal, normal_wn=st.normal_wn)
    if (g_median is not None or g_depth2 is not None) and st.median_pos is not None:
        buffers.update(median_pos=st.median_pos, dL_dmedian=g_median, dL_ddepth2=g_depth2)
    with torch.cuda.device(dev):
        if torch.are_deterministic_algorithms_enabled():
            rc = _backward_deterministic(L, st, dev, args, det_state, **buffers)
        else:
            rc = _opts_or_plain(L.b200gs_backward, L.b200gs_backward_opts, st.aa, st.f3d, **buffers)(*args, _stream(dev))
    _check(rc, "backward")
    return grads


def _save(ctx, tensors):
    """save_for_backward with None holes: autograd's version counters then catch an in-place update of a parameter
    between forward and backward (the saved tensors are the caller's own storage whenever it already was contiguous fp32)."""
    ctx.none_mask = [t is None for t in tensors]
    ctx.save_for_backward(*[t for t in tensors if t is not None])


def _saved(ctx):
    it = iter(ctx.saved_tensors)
    return [None if m else next(it) for m in ctx.none_mask]


class _RasterizeViews(torch.autograd.Function):
    """V >= 1 views of one Gaussian set.  means2D is [V,P,3] (or [P,3] when V == 1 and squeeze=True)."""

    @staticmethod
    def forward(ctx, means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, cams, squeeze,
                means2D_abs=None, normals=False, geometry=False):
        bg, viewmatrix, projmatrix, campos, tanx, tany, H, W, deg, mod, prefiltered, debug = cams[:12]
        raw = bool(cams[12]) if len(cams) > 12 else False
        aa = bool(cams[13]) if len(cams) > 13 else False
        f3d = cams[14] if len(cams) > 14 else None
        dev = means3D.device
        args = [_f32c(t, dev) for t in (means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp)]
        camt = [_f32c(t, dev) for t in (bg, viewmatrix, projmatrix, campos)]
        color, radii, depth, alpha, st = _forward_impl(*args, *camt, tanx, tany, H, W, deg, mod, prefiltered, debug, raw, aa, f3d,
                                                       normals=normals, geometry=geometry)
        ctx.st, ctx.squeeze, ctx.absgrad, ctx.normals = st, squeeze, means2D_abs is not None, normals
        _save(ctx, args + camt)
        ctx.in_shapes = [None if t is None else t.shape for t in (means3D, means2D, shs, colors_precomp, opacities, scales,
                                                                  rotations, cov3D_precomp)]
        ctx.mark_non_differentiable(radii)
        if squeeze:
            return color[0], radii[0], depth[0], alpha[0]
        if normals or geometry:
            # an output the loss does not use gets None, not zeros: a normal or geometry image returned but not in the loss then
            # runs the plain backward kernels (the C ABI's NULL gradients), and an unused image is skipped like a zero one
            ctx.set_materialize_grads(False)
            return (color, radii, depth, alpha) + ((st.normal,) if normals else ()) + ((st.median, st.depth2) if geometry else ())
        return color, radii, depth, alpha

    @staticmethod
    def backward(ctx, g_color, g_radii, g_depth, g_alpha, *g_extra):
        st = ctx.st  # kept until the graph is freed: a second backward (retain_graph=True) recomputes from the same state
        means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, bg, viewmatrix, projmatrix, campos = _saved(ctx)
        dev = means3D.device
        g = [None if t is None else _f32c(t, dev) for t in (g_color, g_depth, g_alpha)]
        g_normal, g_median, g_depth2 = _extra_grads(g_extra, ctx.normals, dev)
        d_means3D, d_means2D, d_sh, d_col, d_op, d_sc, d_rot, d_cov, *d_abs = _backward_impl(
            st, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, bg, viewmatrix, projmatrix, campos, *g,
            absgrad=ctx.absgrad, g_normal=g_normal, g_median=g_median, g_depth2=g_depth2)
        if ctx.squeeze:
            d_means2D = d_means2D[0]
        # gradients take the shape the caller passed (e.g. opacities [P] or [P,1])
        grads = [g if (g is None or shp is None) else g.reshape(shp)
                 for g, shp in zip((d_means3D, d_means2D, d_sh, d_col, d_op, d_sc, d_rot, d_cov), ctx.in_shapes)]
        return (*grads, None, None, d_abs[0] if d_abs else None, None, None)


def _extra_grads(g_extra, normals, dev):
    """(g_normal, g_median, g_depth2) from the gradients of the outputs after alpha: the normal image if `normals`, then the
    median and depth2 images if there are more (None where absent or unused)."""
    g_extra = list(g_extra)
    g_normal = g_extra.pop(0) if normals else None
    g_median, g_depth2 = (g_extra + [None, None])[:2]
    return tuple(None if t is None else _f32c(t, dev) for t in (g_normal, g_median, g_depth2))


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


def _cams_from_settings(s: GaussianRasterizationSettings, antialiasing=False):
    return (s.bg, s.viewmatrix.reshape(1, 4, 4), s.projmatrix.reshape(1, 4, 4), s.campos.reshape(1, 3), [s.tanfovx], [s.tanfovy],
            int(s.image_height), int(s.image_width), int(s.sh_degree), float(s.scale_modifier), s.prefiltered, s.debug, False,
            bool(antialiasing))


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
                        antialiasing=False):
    return _RasterizeViews.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                 _cams_from_settings(raster_settings, antialiasing), True)


class GaussianRasterizer(nn.Module):
    """antialiasing: the screen-space mip filter (DESIGN.md section 2).  None takes `raster_settings.antialiasing` when the
    settings tuple has that field (upstream's 13-field settings do), else off."""

    def __init__(self, raster_settings, antialiasing=None):
        super().__init__()
        self.raster_settings = raster_settings
        self.antialiasing = bool(getattr(raster_settings, "antialiasing", False) if antialiasing is None else antialiasing)

    def markVisible(self, positions):
        L = load_library()
        s = self.raster_settings
        with torch.no_grad():
            pos = _f32c(positions)
            present = torch.empty(pos.shape[0], dtype=torch.uint8, device=pos.device)
            with torch.cuda.device(pos.device):
                rc = L.b200gs_mark_visible(pos.shape[0], _ptr(pos), _ptr(_f32c(s.viewmatrix, pos.device)),
                                           _ptr(_f32c(s.projmatrix, pos.device)), _ptr(present), _stream(pos.device))
            _check(rc, "mark_visible")
        return present.bool()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                   self.raster_settings, self.antialiasing)


def rasterize_views(*, means3D, opacities, viewmatrices, projmatrices, camposs, tanfovx, tanfovy, image_height, image_width,
                    bg, sh_degree=0, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None,
                    means2D=None, scale_modifier=1.0, raw=False, antialiasing=False, filter_3d=None, means2D_abs=None,
                    normals=False, geometry=False):
    """Render V cameras of one Gaussian set in ONE call (one preprocess/sort/blend launch set, one host sync).

    normals=True: a fifth output, the normal image [V,3,H,W] = sum over each pixel's blends of w * n, n the world-space axis of
    the Gaussian's smallest scale flipped to face the camera (unnormalised, no background, 0 where nothing blends; DESIGN.md
    section 2).  It is differentiable: its gradient reaches the opacities, means and colours through the blend weights and
    the rotations through n.  Every other output is unchanged.  Not with cov3D_precomp (ValueError).  comp_normal() turns it
    into threestudio's normal map.

    geometry=True: two more outputs after the normal image (or after alpha without normals): `median_depth` [V,1,H,W], the
    view-space depth of the last blend whose transmittance before it is > 0.5, and `depth2` [V,1,H,W] = sum w * d^2, the depth
    second moment (no background; both 0 where nothing blends; DESIGN.md section 2).  Both are differentiable: depth2 through
    the blend weights and the depths, the median through its Gaussian's depth only.  Every other output is unchanged.
    geometry.depth_distortion(alpha, depth, depth2) forms the depth distortion from them.

    means2D_abs: None, or a [V,P,3] fp32 gradient sink like means2D (zeros, requires_grad): the backward then fills its
    .grad with the absolute screen-space gradient -- per (view, Gaussian) the per-pixel terms of means2D's gradient summed
    in absolute value per component (x, y; z = 0), which does not cancel where a Gaussian's pixels pull it in opposite
    directions (DESIGN.md section 2).  Feed it to densify.add_densification_stats in place of means2D.grad.  Every other
    output and gradient is unchanged.

    filter_3d: [P] fp32 variances of the 3D smoothing filter (`filter3d.compute_filter_3d`), or None: each Gaussian's
    activated scales become sqrt(s^2 + v) and its opacity is scaled to keep its integrated 3D weight, inside the kernels
    (DESIGN.md section 2).  Gradients stay w.r.t. the unfiltered parameters; v gets none.  Not with cov3D_precomp.

    antialiasing=True: the screen-space mip filter -- each Gaussian's opacity is scaled by sqrt(det(S) / det(S + 0.3 I)) of
    its projected covariance S, so its footprint keeps its integrated weight at any pixel scale (DESIGN.md section 2).

    raw=True: `opacities`, `scales`, `rotations` are GaussianModel's RAW parameters (`_opacity`, `_scaling`, `_rotation`,
    gaussian_model.py:44-59); sigmoid / exp / F.normalize run inside the preprocess kernel and their Jacobians inside the
    backward kernel, so the returned gradients are w.r.t. the raw tensors and no activation kernels / autograd nodes exist.

    viewmatrices/projmatrices [V,4,4], camposs [V,3], tanfovx/tanfovy sequences of V floats.  means3D is [P,3]
    (shared: the SDS view batch) or [V,P,3] (per-view positions: the animation frame batch).  means2D, if given,
    is a [V,P,3] gradient sink.  Returns color [V,3,H,W], radii [V,P], depth [V,1,H,W], alpha [V,1,H,W].
    Parameter gradients are summed over views, exactly what V separate rasterizer calls would accumulate."""
    V = viewmatrices.shape[0]
    if V > MAX_VIEWS:
        outs = [rasterize_views(means3D=means3D if means3D.dim() == 2 else means3D[i:i + MAX_VIEWS], opacities=opacities,
                                viewmatrices=viewmatrices[i:i + MAX_VIEWS],
                                projmatrices=projmatrices[i:i + MAX_VIEWS], camposs=camposs[i:i + MAX_VIEWS],
                                tanfovx=tanfovx[i:i + MAX_VIEWS], tanfovy=tanfovy[i:i + MAX_VIEWS], image_height=image_height,
                                image_width=image_width, bg=bg, sh_degree=sh_degree, shs=shs, colors_precomp=colors_precomp,
                                scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp,
                                means2D=None if means2D is None else means2D[i:i + MAX_VIEWS], scale_modifier=scale_modifier, raw=raw,
                                antialiasing=antialiasing, filter_3d=filter_3d,
                                means2D_abs=None if means2D_abs is None else means2D_abs[i:i + MAX_VIEWS], normals=normals,
                                geometry=geometry)
                for i in range(0, V, MAX_VIEWS)]
        return tuple(torch.cat([o[k] for o in outs], 0) for k in range(4 + bool(normals) + 2 * bool(geometry)))
    _check_filter_3d(filter_3d, means3D.shape[-2], means3D.device, cov3D_precomp)
    if means2D is None:
        means2D = torch.zeros(V, means3D.shape[-2], 3, dtype=torch.float32, device=means3D.device)
    cams = (bg, viewmatrices, projmatrices, camposs, list(tanfovx), list(tanfovy), int(image_height), int(image_width),
            int(sh_degree), float(scale_modifier), False, False, bool(raw), bool(antialiasing), filter_3d)
    try:
        return _RasterizeViews.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, cams, False,
                                     means2D_abs, bool(normals), bool(geometry))
    except InstanceLimitError:
        if V == 1:
            raise
    # more (Gaussian, tile) instances than one call supports: render the two halves of the view batch and concatenate
    h = V // 2
    outs = [rasterize_views(means3D=means3D if means3D.dim() == 2 else means3D[sl], opacities=opacities, viewmatrices=viewmatrices[sl],
                            projmatrices=projmatrices[sl], camposs=camposs[sl], tanfovx=list(tanfovx)[sl], tanfovy=list(tanfovy)[sl],
                            image_height=image_height, image_width=image_width, bg=bg, sh_degree=sh_degree, shs=shs,
                            colors_precomp=colors_precomp, scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp,
                            means2D=means2D[sl], scale_modifier=scale_modifier, raw=raw, antialiasing=antialiasing,
                            filter_3d=filter_3d, means2D_abs=None if means2D_abs is None else means2D_abs[sl], normals=normals,
                            geometry=geometry)
            for sl in (slice(0, h), slice(h, V))]
    return tuple(torch.cat([o[k] for o in outs], 0) for k in range(4 + bool(normals) + 2 * bool(geometry)))


# ---- packed entry: one flat SoA parameter buffer in, one flat gradient buffer out ---------------------------------
PACKED_FIELDS = ("xyz", "scales", "rotations", "opacities", "shs")  # == dist.FIELDS order


def packed_layout(P: int, sh_coeffs: int):
    """[(offset, numel, shape)] of xyz, scales, rotations, opacities, shs in the flat buffer, and its total length (floats).
    Every field starts on a 16-byte boundary (offsets rounded up to 4 floats), so the kernels' 128-bit loads/stores of
    rotations and SH rows stay legal for any P; for P % 4 == 0 the fields are simply back to back."""
    out, o = [], 0
    for n, shape in ((3 * P, (P, 3)), (3 * P, (P, 3)), (4 * P, (P, 4)), (P, (P, 1)), (3 * sh_coeffs * P, (P, sh_coeffs, 3))):
        out.append((o, n, shape))
        o = (o + n + 3) & ~3
    return out, o


def packed_numel(P: int, sh_coeffs: int) -> int:
    return packed_layout(P, sh_coeffs)[1]


def _split_packed(flat: torch.Tensor, P: int, M: int):
    """contiguous views [P,3] [P,3] [P,4] [P,1] [P,M,3] into the flat buffer (no copies)"""
    return [flat.narrow(0, o, n).view(shape) for o, n, shape in packed_layout(P, M)[0]]


class _RasterizePacked(torch.autograd.Function):
    @staticmethod
    def forward(ctx, packed, means2D, P, M, cams, means2D_abs=None, normals=False, geometry=False):
        bg, viewmatrix, projmatrix, campos, tanx, tany, H, W, deg, mod, raw, aa, f3d = cams
        dev = packed.device
        xyz, sc, rot, op, sh = _split_packed(packed.detach(), P, M)
        camt = [_f32c(t, dev) for t in (bg, viewmatrix, projmatrix, campos)]
        color, radii, depth, alpha, st = _forward_impl(xyz, sh, None, op, sc, rot, None, *camt, tanx, tany, H, W, deg, mod, raw=raw,
                                                       antialiasing=aa, filter_3d=f3d, normals=normals, geometry=geometry)
        ctx.st, ctx.P, ctx.M, ctx.absgrad, ctx.normals = st, P, M, means2D_abs is not None, normals
        ctx.save_for_backward(packed, *camt)
        ctx.mark_non_differentiable(radii)
        if normals or geometry:
            ctx.set_materialize_grads(False)  # as _RasterizeViews: an unused normal or geometry image costs no backward term
            return (color, radii, depth, alpha) + ((st.normal,) if normals else ()) + ((st.median, st.depth2) if geometry else ())
        return color, radii, depth, alpha

    @staticmethod
    def backward(ctx, g_color, g_radii, g_depth, g_alpha, *g_extra):
        packed, bg, viewmatrix, projmatrix, campos = ctx.saved_tensors
        packed = packed.detach()
        P, M, dev = ctx.P, ctx.M, packed.device
        xyz, sc, rot, op, sh = _split_packed(packed, P, M)
        d_packed = torch.empty_like(packed) if P % 4 == 0 else torch.zeros_like(packed)  # alignment padding carries zero gradient
        d_xyz, d_sc, d_rot, d_op, d_sh = _split_packed(d_packed, P, M)
        g = [None if t is None else _f32c(t, dev) for t in (g_color, g_depth, g_alpha)]
        g_normal, g_median, g_depth2 = _extra_grads(g_extra, ctx.normals, dev)
        _, d_means2D, *rest = _backward_impl(ctx.st, xyz, sh, None, op, sc, rot, None, bg, viewmatrix, projmatrix, campos, *g,
                                             out=dict(means3D=d_xyz, sh=d_sh, opacity=d_op, scales=d_sc, rotations=d_rot),
                                             absgrad=ctx.absgrad, g_normal=g_normal, g_median=g_median, g_depth2=g_depth2)
        return d_packed, d_means2D, None, None, None, rest[6] if ctx.absgrad else None, None, None


def rasterize_views_packed(packed: torch.Tensor, P: int, sh_coeffs: int, *, viewmatrices, projmatrices, camposs, tanfovx, tanfovy,
                           image_height, image_width, bg, sh_degree=0, means2D=None, scale_modifier=1.0, raw=False, antialiasing=False,
                           filter_3d=None, means2D_abs=None, normals=False, geometry=False):
    """`rasterize_views` over ONE flat fp32 buffer [xyz 3P | scales 3P | rotations 4P | opacities P | shs 3*K*P], each
    field starting on a 16-byte boundary (`packed_layout`; what `dist.pack` produces, broadcast once per parameter
    version).  raw=False: post-activation values, as the rasteriser's classic inputs.  raw=True: the buffer holds the
    optimiser's RAW parameters (log-scales, un-normalised quaternions, opacity logits; SH = cat(f_dc, f_rest)); the
    activations of gaussian_model.py:95-118 and their Jacobians run inside the kernels, so `packed.grad` is the gradient
    of the raw parameters and a training step needs no activation kernels, no pack copy and no autograd nodes besides
    this one.  antialiasing, filter_3d, means2D_abs, normals, geometry: as `rasterize_views`.  The backward
    kernels write the parameter gradients straight into one buffer of the same layout, which becomes `packed.grad`
    as is: no per-tensor gradient accumulation, and on several GPUs that buffer is the all-reduce payload in place.
    V <= MAX_VIEWS.  Returns color [V,3,H,W], radii [V,P], depth [V,1,H,W], alpha [V,1,H,W]."""
    if packed.dim() != 1 or packed.numel() != packed_numel(P, sh_coeffs) or packed.dtype != torch.float32 or not packed.is_contiguous():
        raise ValueError(f"b200gs: packed buffer must be contiguous fp32 with {packed_numel(P, sh_coeffs)} elements")
    if packed.device.type != "cuda":
        raise RuntimeError("b200gs: tensors must live on a CUDA device (there is no CPU path)")
    V = viewmatrices.shape[0]
    if V > MAX_VIEWS:
        raise ValueError(f"b200gs: at most {MAX_VIEWS} views per packed call")
    _check_filter_3d(filter_3d, P, packed.device)
    if means2D is None:
        means2D = torch.zeros(V, P, 3, dtype=torch.float32, device=packed.device)
    cams = (bg, viewmatrices, projmatrices, camposs, list(tanfovx), list(tanfovy), int(image_height), int(image_width),
            int(sh_degree), float(scale_modifier), bool(raw), bool(antialiasing), filter_3d)
    try:
        return _RasterizePacked.apply(packed, means2D, int(P), int(sh_coeffs), cams, means2D_abs, bool(normals), bool(geometry))
    except InstanceLimitError:
        if V == 1:
            raise
    h = V // 2  # too many instances for one call: two half batches; autograd sums the two packed gradients
    outs = [rasterize_views_packed(packed, P, sh_coeffs, viewmatrices=viewmatrices[sl], projmatrices=projmatrices[sl], camposs=camposs[sl],
                                   tanfovx=list(tanfovx)[sl], tanfovy=list(tanfovy)[sl], image_height=image_height,
                                   image_width=image_width, bg=bg, sh_degree=sh_degree, means2D=means2D[sl],
                                   scale_modifier=scale_modifier, raw=raw, antialiasing=antialiasing, filter_3d=filter_3d,
                                   means2D_abs=None if means2D_abs is None else means2D_abs[sl], normals=normals,
                                   geometry=geometry)
            for sl in (slice(0, h), slice(h, V))]
    return tuple(torch.cat([o[k] for o in outs], 0) for k in range(4 + bool(normals) + 2 * bool(geometry)))


# ---- test / debugging access to the forward state (tile and sort indices) -----------------------------------
def forward_with_state(**kw):
    """Non-differentiable forward returning outputs + a dict of the intermediate buffers as torch tensors.
    contrib=(weight_sum, weight_max, touches): the contribution forward, folding into those accumulators (_forward_impl).
    normals=True: the normals forward; the normal image [V,3,H,W] is then a fifth output after alpha, and the state also holds
    "gauss_normals" [V*P,4] (sign * n, sign) of every (view, Gaussian)."""
    L = load_library()
    dev = kw["means3D"].device
    t = lambda k: _f32c(kw.get(k), dev)
    vm, pm, cp = kw["viewmatrix"], kw["projmatrix"], kw["campos"]
    V = 1 if vm.dim() == 2 else vm.shape[0]
    tanx, tany = kw["tanfovx"], kw["tanfovy"]
    if not isinstance(tanx, (list, tuple)):
        tanx, tany = [tanx], [tany]
    color, radii, depth, alpha, st = _forward_impl(
        t("means3D"), t("shs"), t("colors_precomp"), t("opacities"), t("scales"), t("rotations"), t("cov3D_precomp"),
        _f32c(kw["bg"], dev), _f32c(vm, dev).reshape(V, 4, 4), _f32c(pm, dev).reshape(V, 4, 4), _f32c(cp, dev).reshape(V, 3),
        tanx, tany, int(kw["image_height"]), int(kw["image_width"]), int(kw.get("sh_degree", 0)),
        float(kw.get("scale_modifier", 1.0)), raw=bool(kw.get("raw", False)), antialiasing=bool(kw.get("antialiasing", False)),
        filter_3d=kw.get("filter_3d"), contrib=kw.get("contrib"), normals=bool(kw.get("normals", False)),
        geometry=bool(kw.get("geometry", False)))
    sv = _StateView()
    _check(L.b200gs_describe_state(C.byref(st.prm), _ptr(st.geom), _ptr(st.binning), st.capacity, _ptr(st.image), C.byref(sv)),
           "describe_state")
    P, H, W, D = st.P, st.H, st.W, st.num_rendered
    ntiles = ((W + 15) // 16) * ((H + 15) // 16)

    def view(buf, addr, dtype, count):
        off = addr - buf.data_ptr()
        nbytes = count * torch.empty((), dtype=dtype).element_size()
        return buf[off:off + nbytes].view(dtype).clone()

    state = dict(
        num_rendered=D,
        recs=view(st.geom, sv.geom_records, torch.float32, V * P * 12).reshape(V * P, 12),
        tiles_touched=view(st.geom, sv.tiles_touched, torch.int32, V * P),
        offsets=view(st.geom, sv.offsets, torch.int32, V * P),
        clamped=view(st.geom, sv.clamped, torch.uint8, V * P),
        sorted_tile_keys=view(st.binning, sv.sorted_tile_keys, torch.int32, D),
        depth_order=view(st.binning, sv.depth_order, torch.int32, V * P),
        point_list=view(st.binning, sv.point_list, torch.int32, D),
        ranges=view(st.binning, sv.ranges, torch.int32, V * ntiles * 2).reshape(V * ntiles, 2),
        final_T=view(st.image, sv.final_T, torch.float32, V * H * W).reshape(V, H, W),
        n_contrib=view(st.image, sv.n_contrib, torch.int32, V * H * W).reshape(V, H, W),
        # the forward blend's contributor masks (int32 words; layout in include/b200gs.h, b200gs_state_view)
        contributor_masks=view(st.binning, sv.contributor_masks, torch.int32, sv.contributor_mask_words),
    )
    # the reference's 64-bit sort key of every instance: (view*tiles + tile) << 32 | depth bits of its Gaussian
    dbits = state["recs"][:, 11].contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    pl = state["point_list"].to(torch.int64) & 0xFFFFFFFF
    state["sorted_keys"] = ((state["sorted_tile_keys"].to(torch.int64) & 0xFFFFFFFF) << 32) | dbits[pl]
    extra = ()
    if st.normal is not None:
        state["gauss_normals"] = st.gauss_normals.reshape(V * P, 4).clone()
        extra += (st.normal,)
    if st.median is not None:
        state["median_pos"] = st.median_pos.clone()
        extra += (st.median, st.depth2)
    return (color, radii, depth, alpha) + extra + (state, st)


def forward_backward_with_state(g_color, g_depth, g_alpha, g_normal=None, g_median=None, g_depth2=None, **kw):
    """forward_with_state(**kw), then the backward of that same call for the image gradients g_color [V,3,H,W],
    g_depth [V,1,H,W], g_alpha [V,1,H,W].  Returns (color, radii, depth, alpha, state, sums): `sums` [V,P,12] float32 is
    the backward blend's ScreenGrad record of every (view, Gaussian) -- record v*P + g, in the format
    blend_sgrad_is_moments() names (csrc/common.cuh) -- copied out before the state buffers can be re-used.  Under
    torch.use_deterministic_algorithms(True) the deterministic backward runs, and `state` also holds its "patch_masks"
    (uint8 per sorted instance, bit p = a partial for patch p of the instance's tile) and "n_partials".
    normals=True: the normal image is a fifth output after alpha, and g_normal [V,3,H,W] (None: no normal gradient) its
    gradient; with g_normal, `state` also holds "normal_wn" [V,P,4], the sums Wn = sum w * dL/dN (DESIGN.md section 2).
    geometry=True: the median and depth2 images follow (after the normal image, if any), and g_median / g_depth2 [V,1,H,W]
    (None: zero) are their gradients; `state` holds "median_pos".  `state["grads"]` is the gradient tuple of that backward
    (d_means3D, d_means2D, d_sh, d_colors, d_opacity, d_scales, d_rotations, d_cov3D; None where the input was absent)."""
    outs = forward_with_state(**kw)
    images = outs[:-2]
    state, st = outs[-2:]
    dev = kw["means3D"].device
    V, P = st.V, st.P
    t = lambda k: _f32c(kw.get(k), dev)
    g = [_f32c(x, dev).reshape(V, c, st.H, st.W) for x, c in ((g_color, 3), (g_depth, 1), (g_alpha, 1))]
    det_state = {}
    grads = _backward_impl(st, t("means3D"), t("shs"), t("colors_precomp"), t("opacities"), t("scales"), t("rotations"),
                   t("cov3D_precomp"), _f32c(kw["bg"], dev), t("viewmatrix").reshape(V, 4, 4), t("projmatrix").reshape(V, 4, 4),
                   t("campos").reshape(V, 3), *g, det_state=det_state,
                   g_normal=None if g_normal is None else _f32c(g_normal, dev).reshape(V, 3, st.H, st.W),
                   g_median=None if g_median is None else _f32c(g_median, dev).reshape(V, 1, st.H, st.W),
                   g_depth2=None if g_depth2 is None else _f32c(g_depth2, dev).reshape(V, 1, st.H, st.W))
    state.update(det_state)
    state["grads"] = grads
    if st.normal_wn is not None:
        state["normal_wn"] = st.normal_wn.clone()
    nbytes = V * P * 48
    sums = st.scratch[:nbytes].view(torch.float32).reshape(V, P, 12).clone()
    return tuple(images) + (state, sums)


def sampling_rate(means3D: torch.Tensor, viewmatrices: torch.Tensor, tanfovx, tanfovy, image_height: int, image_width: int,
                  max_rate: torch.Tensor) -> torch.Tensor:
    """b200gs_sampling_rate: fold up to MAX_VIEWS cameras into max_rate [P] (in place, by max) and return it.
    means3D [P,3]; viewmatrices [V,4,4]; tanfovx / tanfovy sequences of V floats."""
    L = load_library()
    dev = means3D.device
    if dev.type != "cuda":
        raise RuntimeError("b200gs: tensors must live on a CUDA device (there is no CPU path)")
    V = viewmatrices.shape[0]
    if V > MAX_VIEWS:
        raise ValueError(f"b200gs: at most {MAX_VIEWS} cameras per sampling_rate call")
    if max_rate.dtype != torch.float32 or max_rate.device != dev or not max_rate.is_contiguous() or max_rate.shape != (means3D.shape[0],):
        raise ValueError("b200gs: max_rate must be a contiguous [P] float32 tensor on the means' device")
    pts, vm = _f32c(means3D), _f32c(viewmatrices, dev)
    tx = (C.c_float * V)(*[float(t) for t in tanfovx])
    ty = (C.c_float * V)(*[float(t) for t in tanfovy])
    with torch.cuda.device(dev):
        _check(L.b200gs_sampling_rate(pts.shape[0], V, _ptr(pts), _ptr(vm), tx, ty, int(image_height), int(image_width),
                                      _ptr(max_rate), _stream(dev)), "sampling_rate")
    return max_rate


def device_sort_pairs(keys: torch.Tensor, vals: torch.Tensor, nbits: int):
    """The binning stage's stable radix sort (int32 tensors reinterpreted as u32), exposed for tests."""
    L = load_library()
    ka, va = keys.contiguous().clone(), vals.contiguous().clone()
    kb, vb = torch.empty_like(ka), torch.empty_like(va)
    n = ka.numel()
    scratch = torch.empty(L.b200gs_test_sort_scratch_bytes(n), dtype=torch.uint8, device=ka.device)
    in_b = C.c_int32(0)
    with torch.cuda.device(ka.device):
        _check(L.b200gs_test_sort_pairs(_ptr(ka), _ptr(kb), _ptr(va), _ptr(vb), n, int(nbits), _ptr(scratch), scratch.numel(),
                                        C.byref(in_b), _stream(ka.device)), "test_sort_pairs")
    return (kb, vb) if in_b.value else (ka, va)


def distCUDA2(points: torch.Tensor) -> torch.Tensor:
    """Mean squared distance to the 3 nearest neighbours, per point (the reference's simple_knn._C.distCUDA2)."""
    L = load_library()
    pts = _f32c(points)
    if pts.device.type != "cuda":
        raise RuntimeError("b200gs: tensors must live on a CUDA device (there is no CPU path)")
    P = pts.shape[0]
    out = torch.empty(P, dtype=torch.float32, device=pts.device)
    scratch = torch.empty(L.b200gs_knn_scratch_bytes(P), dtype=torch.uint8, device=pts.device)
    with torch.cuda.device(pts.device):
        _check(L.b200gs_dist2_knn3(P, _ptr(pts), _ptr(out), _ptr(scratch), scratch.numel(), _stream(pts.device)), "dist2_knn3")
    return out


def device_exp(x: torch.Tensor) -> torch.Tensor:
    """gs_exp evaluated by the CUDA library (pinned bit-for-bit against the oracle in tests)."""
    L = load_library()
    x = _f32c(x)
    y = torch.empty_like(x)
    with torch.cuda.device(x.device):
        _check(L.b200gs_test_exp(_ptr(x), _ptr(y), x.numel(), _stream(x.device)), "test_exp")
    return y
