"""GPU: every binning intermediate of the forward against the numpy reference (tests/binning_reference.py), bit for bit.

tiles_touched, the depth order, the offsets in depth order, the instance count, the sorted tile keys, point_list and the
ranges are compared as uint32 at the shapes where radix sorts and scans go wrong: one, two and three tile-sort passes, the
benchmark's 64-view step, both sides of the deferred / exact-count threshold, record counts at the CTA edges, depth ties,
culled prefixes, long emission runs, short range tails and capacities just below the instance count.  Every case also
asserts its own precondition (key bits, record counts, ties), so it cannot silently stop covering its edge.
test_oracle_binning.py pins the reference to the oracle's 64-bit sort."""
import ctypes as C

import numpy as np
import pytest
import torch

from binning_reference import BinningReference, bits_for
from util import screen_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DEFERRED_MAX_NVP = 4 << 20  # api.cu: up to this many (view, Gaussian) pairs the forward does not wait for its instance count
TILE_SORT_BITS = 9          # binning.cu: digit width of the tile sort


@pytest.fixture(autouse=True)
def _free_states():
    yield
    from humangaussian_b200.rasterizer import release_cached_buffers
    release_cached_buffers()
    torch.cuda.empty_cache()


def _np32(t):
    return np.ascontiguousarray(t.cpu().numpy() if torch.is_tensor(t) else t).view(np.uint32)


def _eq(got, want, what):
    got = _np32(got)
    if got.shape == want.shape and np.array_equal(got, want):
        return
    if got.shape != want.shape:
        raise AssertionError(f"{what}: shape {got.shape}, reference {want.shape}")
    i = np.argwhere(got != want)[0]
    raise AssertionError(f"{what}: {int((got != want).sum())} entries differ; first at {tuple(int(x) for x in i)}: "
                         f"{got[tuple(i)]} vs reference {want[tuple(i)]}")


def check_binning(st, radii, H, W):
    """forward_with_state's binning intermediates against the reference, view by view.  Returns the reference."""
    V = radii.shape[0]
    recs = st["recs"]
    px, py, depth = (recs[:, k].contiguous().cpu().numpy() for k in (0, 1, 11))
    ref = BinningReference(radii.reshape(-1).cpu().numpy(), px, py, depth, H, W, V)
    _eq(st["tiles_touched"], ref.tiles_touched, "tiles_touched")
    assert st["num_rendered"] == ref.num_rendered, f"num_rendered {st['num_rendered']}, reference {ref.num_rendered}"
    _eq(st["depth_order"], ref.depth_order, "depth order")
    _eq(st["offsets"], ref.offsets, "offsets in depth order")
    nt = ref.ntiles
    for v in range(V):
        want = ref.view(v)
        a, b = int(ref.view_start[v]), int(ref.view_start[v + 1])
        _eq(st["sorted_tile_keys"][a:b], want["sorted_tile_keys"], f"view {v}: sorted tile keys")
        _eq(st["point_list"][a:b], want["point_list"], f"view {v}: point_list")
        _eq(st["ranges"][v * nt:(v + 1) * nt], want["ranges"], f"view {v}: ranges")
    return ref


def _forward(kw):
    from humangaussian_b200.rasterizer import forward_with_state
    color, radii, depth, alpha, st, _ = forward_with_state(**kw)
    ref = check_binning(st, radii, kw["image_height"], kw["image_width"])
    return st, ref, radii


def _body(P, V, H, W, seed=0, cam_seed=1000):
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import stack_cameras
    from humangaussian_b200.scene import synthetic_body
    p = synthetic_body(P, sh_degree=0, seed=seed).to(DEV)
    vm, pm, cp, tanx, tany = stack_cameras(sample_orbit_cameras(V, H, W, seed=cam_seed, device=DEV), DEV)
    with torch.no_grad():
        kw = dict(means3D=p.get_xyz, opacities=p.get_opacity, shs=p.get_features.contiguous(), scales=p.get_scaling,
                  rotations=p.get_rotation)
    return dict(kw, viewmatrix=vm, projmatrix=pm, campos=cp, tanfovx=tanx, tanfovy=tany, image_height=H, image_width=W,
                sh_degree=0, bg=torch.zeros(3, device=DEV))


def _screen(px, py, depth, sigma, opacity=0.5, H=64, W=128, V=1):
    """util.screen_scene on the device, seen by V identical cameras"""
    inp = screen_scene(px, py, depth, sigma, opacity, H=H, W=W)
    kw = {k: (torch.tensor(v, device=DEV) if isinstance(v, np.ndarray) else v) for k, v in inp.items()}
    kw["viewmatrix"] = kw["viewmatrix"].expand(V, 4, 4).contiguous()
    kw["projmatrix"] = kw["projmatrix"].expand(V, 4, 4).contiguous()
    kw["campos"] = kw["campos"].expand(V, 3).contiguous()
    kw["tanfovx"], kw["tanfovy"] = [inp["tanfovx"]] * V, [inp["tanfovy"]] * V
    return kw


def _random_screen(n, H, W, seed, V=1):
    """n Gaussians with centres inside the image, random depths, sigma 0.2 .. 20 px"""
    rng = np.random.RandomState(seed)
    return _screen(rng.uniform(0, W, n), rng.uniform(0, H, n), rng.uniform(1, 10, n),
                   np.exp(rng.uniform(np.log(0.2), np.log(20), n)), 0.6, H=H, W=W, V=V)


# ---- 1. tile-sort pass counts ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,H,W,nbits", [(2, 128, 128, 7), (64, 1024, 1024, 18), (64, 1040, 1024, 19), (17, 2048, 2048, 19)])
def test_tile_sort_pass_counts(V, H, W, nbits):
    """V*ntiles = 128 (one pass), exactly 2^18 (two full 9-bit passes), 266 240 and 278 528 (19 bits: passes of 9, 9 and 1)"""
    kw = _body(20_000, V, H, W)
    st, ref, _ = _forward(kw)
    assert bits_for(V * ref.ntiles) == nbits
    keys = st["sorted_tile_keys"]
    assert ref.num_rendered > 0 and int(keys[-1]) >= 1 << (nbits - 1), "the top key bit must vary"
    if nbits == 18:
        assert V * ref.ntiles == 1 << 18


# ---- 2. the benchmark's step ----------------------------------------------------------------------------------------
def test_bench_step_binning():
    """bench.py's single-GPU step at its defaults, as one call: sample scene, 300 k Gaussians, SH degree 3, RAW parameters,
    64 seed-1000 orbit cameras at 1024^2.  V*P = 19.2 M takes the exact-count path; tile keys span exactly 18 bits."""
    from humangaussian_b200.cameras import sample_orbit_cameras
    from humangaussian_b200.renderer import stack_cameras
    from humangaussian_b200.scene import sample_ply_scene
    P, V, HW = 300_000, 64, 1024
    p = sample_ply_scene(P, 3, seed=0)
    vm, pm, cp, tanx, tany = stack_cameras(sample_orbit_cameras(V, HW, HW, seed=1000), DEV)
    t = lambda x: x.detach().to(DEV, torch.float32).contiguous()
    kw = dict(means3D=t(p.xyz), scales=t(p.scaling), rotations=t(p.rotation), opacities=t(p.opacity), shs=t(p.get_features),
              viewmatrix=vm, projmatrix=pm, campos=cp, tanfovx=tanx, tanfovy=tany, image_height=HW, image_width=HW, sh_degree=3,
              bg=torch.zeros(3, device=DEV), raw=True)
    st, ref, radii = _forward(kw)
    assert V * P > DEFERRED_MAX_NVP and bits_for(V * ref.ntiles) == 18
    assert ref.num_rendered > 10_000_000 and bool((radii > 0).any(1).all())


# ---- 3. deferred / exact-count threshold ----------------------------------------------------------------------------
@pytest.mark.parametrize("P", [65_536, 65_537])
def test_deferred_and_exact_count_threshold(P):
    """64 x 65 536 = 4 * 2^20 pairs: the last batch size whose binning is sized for the capacity and reads the count on the
    device; one more Gaussian per view and the forward waits for the exact count instead."""
    V = 64
    kw = _body(P, V, 72, 88, seed=2, cam_seed=7)
    _, ref, _ = _forward(kw)
    assert (V * P <= DEFERRED_MAX_NVP) == (P == 65_536) and ref.num_rendered > 0


# ---- 4. record counts at the CTA edges ------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 2, 31, 32, 33, 255, 257, 2047, 2048, 2049, 3071, 3072, 3073, 6145])
def test_record_counts_at_cta_edges(P):
    """depth-sort tile 3072, scan tile 2048, emission warp 32, block 256: one view of P records"""
    kw = _random_screen(P, 96, 160, seed=P)
    _, ref, radii = _forward(kw)
    assert radii.numel() == P and ref.num_rendered > 0


def test_three_views_of_1024():
    kw = _body(1024, 3, 200, 136, seed=5, cam_seed=11)
    _, ref, radii = _forward(kw)
    assert radii.shape == (3, 1024) and bool((radii > 0).any(1).all())


# ---- 5. depth ties --------------------------------------------------------------------------------------------------
def test_one_depth_over_identical_views():
    """all records at one depth in V identical views: the order falls back to the record index v*P + i everywhere"""
    n, V = 700, 5
    rng = np.random.RandomState(1)
    kw = _screen(rng.uniform(0, 256, n), rng.uniform(0, 96, n), np.full(n, 3.0), rng.uniform(0.3, 25, n), 0.4, H=96, W=256, V=V)
    st, ref, radii = _forward(kw)
    assert bool((radii > 0).all()) and len(np.unique(ref.depth_keys)) == 1
    assert np.array_equal(_np32(st["depth_order"]), np.arange(V * n, dtype=np.uint32))
    assert int(ref.tiles_touched.max()) > 1


def test_two_depths_interleaved_by_index():
    n, V = 900, 3
    rng = np.random.RandomState(2)
    depth = np.where(np.arange(n) % 2 == 0, 2.0, 4.0)
    kw = _screen(rng.uniform(0, 200, n), rng.uniform(0, 120, n), depth, rng.uniform(0.3, 15, n), 0.4, H=120, W=200, V=V)
    _, ref, radii = _forward(kw)
    assert bool((radii > 0).all()) and len(np.unique(ref.depth_keys)) == 2


# ---- 6. culled prefix ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_culled", [33, 45, 257])
def test_culled_prefix(n_culled):
    """zero-tile records sort first, so the visible records start mid-warp (33, 45) or mid-block (257) in emission"""
    n_vis, H, W = 400, 96, 128
    n = n_vis + n_culled
    rng = np.random.RandomState(n_culled)
    px, py = rng.uniform(0, W, n), rng.uniform(0, H, n)
    depth, sigma = rng.uniform(1, 10, n), rng.uniform(0.3, 10, n)
    culled = rng.permutation(n)[:n_culled]
    depth[culled[::2]] = -1.0    # behind the camera
    px[culled[1::2]] = -500.0    # off screen: an empty rect
    sigma[culled[1::2]] = 1.0
    kw = _screen(px, py, depth, sigma, 0.5, H=H, W=W)
    st, ref, radii = _forward(kw)
    assert int((radii == 0).sum()) == n_culled
    assert not ref.tiles_touched[ref.depth_order[:n_culled]].any() and ref.tiles_touched[ref.depth_order[n_culled:]].all()


# ---- 7. long emission runs ------------------------------------------------------------------------------------------
def test_screen_fillers_mixed_with_single_tile_gaussians():
    """screen-filling records (256 tiles each) between one-tile ones: warps loop over many 32-instance rounds, and the runs
    of the following records start mid-round"""
    n, H, W, V = 260, 256, 256, 2
    rng = np.random.RandomState(7)
    filler = rng.rand(n) < 0.15
    px = np.where(filler, W / 2, rng.randint(0, 16, n) * 16 + 7.5)
    py = np.where(filler, H / 2, rng.randint(0, 16, n) * 16 + 7.5)
    kw = _screen(px, py, rng.uniform(1, 10, n), np.where(filler, 400.0, 0.2), 0.05, H=H, W=W, V=V)
    _, ref, _ = _forward(kw)
    tt = ref.tiles_touched.reshape(V, n)[0]
    assert (tt[filler] == ref.ntiles).all() and (tt[~filler] == 1).all() and filler.sum() > 20


# ---- 8. ranges tail ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 7])
def test_short_lists_ranges_tail(D):
    """D single-tile Gaussians (sigma 0.2 px at tile centres): the ranges kernel's four-key groups end at every D % 4"""
    H, W = 64, 128
    rng = np.random.RandomState(D)
    tiles = rng.choice(32, D, replace=True)
    kw = _screen(tiles % 8 * 16 + 7.5, tiles // 8 * 16 + 7.5, rng.uniform(1, 10, D), 0.2, 0.7, H=H, W=W)
    st, ref, _ = _forward(kw)
    assert ref.num_rendered == D and (ref.tiles_touched == 1).all()


def test_first_and_last_tiles_only():
    H, W = 72, 136  # 9 x 5 tiles, partial on both axes
    last = (W + 15) // 16 * ((H + 15) // 16) - 1
    gx = (W + 15) // 16
    tiles = np.array([0, last, 0, last, last, 0, last])
    kw = _screen(tiles % gx * 16 + 4.5, tiles // gx * 16 + 3.5, np.arange(7) * 0.5 + 1, 0.2, 0.7, H=H, W=W)
    st, ref, _ = _forward(kw)
    r = _np32(st["ranges"])
    occupied = np.nonzero(r[:, 1] > r[:, 0])[0]
    assert occupied.tolist() == [0, last] and ref.num_rendered == 7


# ---- 9. a three-pass batch equals its single-view calls -------------------------------------------------------------
def _read_mask_words(masks, ranges, n_contrib, H, W, v):
    """the contributor-mask words the backward reads for view v (test_gpu_parity._check_masks), in (tile, patch, chunk)
    order: tile t's words start at ((range.x >> 5) + vt) * 8, vt = v * ntiles + t"""
    from test_gpu_parity import _patch_wmax
    nt = ((W + 15) // 16) * ((H + 15) // 16)
    wmax = _patch_wmax(n_contrib, H, W)
    nread = np.where(wmax > 0, ((wmax - 1) >> 5) + 1, 0)
    t, p = np.nonzero(nread)
    cnt = nread[t, p]
    tt, pp = np.repeat(t, cnt), np.repeat(p, cnt)
    chunk = np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    vt = v * nt + tt
    return masks[((ranges[vt, 0].astype(np.int64) >> 5) + vt) * 8 + chunk * 8 + pp]


@pytest.fixture
def deterministic():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def test_three_pass_batch_equals_single_view_calls(deterministic):
    """64 x 1040x1024 in one call (19 key bits, three tile-sort passes) against 64 single-view calls (13 bits, two passes):
    images, radii, final_T, n_contrib, the contributor-mask words the backward reads and the deterministic backward's
    per-(view, Gaussian) ScreenGrad records, byte for byte; views 0 and 63 also against the oracle."""
    from humangaussian_b200.rasterizer import forward_backward_with_state
    from oracle.gs_oracle import Oracle
    from test_gpu_parity import _check_masks
    V, H, W, P = 64, 1040, 1024, 20_000
    kw = _body(P, V, H, W)
    g = torch.Generator(device=DEV).manual_seed(0)
    gimg = [torch.randn(V, c, H, W, device=DEV, generator=g) for c in (3, 1, 1)]
    color, radii, depth, alpha, st, sums = forward_backward_with_state(*gimg, **kw)
    ref = check_binning(st, radii, H, W)
    nt = ref.ntiles
    assert bits_for(V * nt) == 19 and bits_for(nt) == 13
    assert st["n_partials"] > 0, "the deterministic backward did not run"
    masks, ranges = _np32(st["contributor_masks"]), _np32(st["ranges"])
    n_contrib, final_T = st["n_contrib"], st["final_T"]
    pl = _np32(st["point_list"])
    per_view = lambda v: dict(kw, viewmatrix=kw["viewmatrix"][v:v + 1], projmatrix=kw["projmatrix"][v:v + 1],
                              campos=kw["campos"][v:v + 1], tanfovx=kw["tanfovx"][v:v + 1], tanfovy=kw["tanfovy"][v:v + 1])
    same = lambda a, b: torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))
    n_words = 0
    for v in range(V):
        c1, r1, d1, a1, s1, sums1 = forward_backward_with_state(*(x[v:v + 1] for x in gimg), **per_view(v))
        assert same(c1[0], color[v]) and same(d1[0], depth[v]) and same(a1[0], alpha[v]), f"view {v}: images differ"
        assert torch.equal(r1[0], radii[v]), f"view {v}: radii differ"
        assert same(s1["final_T"][0], final_T[v]) and torch.equal(s1["n_contrib"][0], n_contrib[v]), f"view {v}: final_T / n_contrib"
        nc = n_contrib[v].cpu().numpy()
        want = _read_mask_words(_np32(s1["contributor_masks"]), _np32(s1["ranges"]), nc, H, W, 0)
        got = _read_mask_words(masks, ranges, nc, H, W, v)
        assert np.array_equal(got, want), f"view {v}: {int((got != want).sum())} contributor-mask words differ"
        n_words += got.size
        assert same(sums1[0], sums[v]), f"view {v}: deterministic ScreenGrad records differ from the single-view call's"
        del c1, r1, d1, a1, s1, sums1
    assert n_words > V * nt
    o = Oracle()
    for v in (0, V - 1):
        inp = {k: (x.detach().cpu().numpy() if torch.is_tensor(x) else x) for k, x in per_view(v).items()}
        inp.update(viewmatrix=inp["viewmatrix"][0], projmatrix=inp["projmatrix"][0], campos=inp["campos"][0],
                   tanfovx=inp["tanfovx"][0], tanfovy=inp["tanfovy"][0])
        o_col, o_rad, o_dep, o_alp = o.forward(**inp)
        o_st = o.state()
        f = lambda a: np.ascontiguousarray(a).view(np.uint32)
        assert np.array_equal(radii[v].cpu().numpy(), o_rad)
        assert np.array_equal(f(color[v].cpu().numpy()), f(o_col)) and np.array_equal(f(depth[v].cpu().numpy()), f(o_dep))
        assert np.array_equal(f(alpha[v].cpu().numpy()), f(o_alp))
        assert np.array_equal(_np32(n_contrib[v]), o_st["n_contrib"]) and np.array_equal(f(final_T[v].cpu().numpy()), f(o_st["final_T"]))
        a, b = int(ref.view_start[v]), int(ref.view_start[v + 1])
        assert b - a == o_st["num_rendered"]
        assert np.array_equal(pl[a:b] - np.uint32(v * P), o_st["point_list"])
        r = ranges[v * nt:(v + 1) * nt].astype(np.int64)
        assert np.array_equal(np.where(r[:, 1:] > r[:, :1], r - a, 0), o_st["ranges"].astype(np.int64))
        _check_masks(masks, ranges, n_contrib[v].cpu().numpy(), o_st, H, W, v=v)


# ---- 10. capacity truncation ----------------------------------------------------------------------------------------
TAIL = 4096


def _call_forward(kw, cap):
    """b200gs_forward with capacity `cap` and no retry.  The geom, binning and image buffers each carry a 4 KiB patterned tail
    past the size passed, which must be unchanged after the call.  Returns (rc, num_rendered, state or None)."""
    from humangaussian_b200 import rasterizer as R
    L = R.load_library()
    vm, pm, cp = kw["viewmatrix"], kw["projmatrix"], kw["campos"]
    V, P, H, W = vm.shape[0], kw["means3D"].shape[0], kw["image_height"], kw["image_width"]
    prm, tx, ty = R._make_params(P, V, 0, 0, H, W, 1.0, kw["tanfovx"], kw["tanfovy"])
    sizes = dict(geom=L.b200gs_geom_bytes(P, V), binning=L.b200gs_binning_bytes(cap, H, W, P, V), image=L.b200gs_image_bytes(H, W, V))
    pattern = (torch.arange(TAIL, device=DEV) * 37 + 11).to(torch.uint8)
    bufs = {k: torch.zeros(n + TAIL, dtype=torch.uint8, device=DEV) for k, n in sizes.items()}
    for k, b in bufs.items():
        b[sizes[k]:] = pattern
    color = torch.empty(V, 3, H, W, device=DEV)
    depth, alpha = torch.empty(V, 1, H, W, device=DEV), torch.empty(V, 1, H, W, device=DEV)
    radii = torch.empty(V, P, dtype=torch.int32, device=DEV)
    n_out = C.c_int64(-1)
    p = R._ptr
    rc = L.b200gs_forward(C.byref(prm), p(kw["means3D"]), None, p(kw["colors_precomp"]), p(kw["opacities"]), None, None,
                          p(kw["cov3D_precomp"]), p(kw["bg"]), p(vm), p(pm), p(cp), p(color), p(depth), p(alpha), p(radii),
                          p(bufs["geom"]), sizes["geom"], p(bufs["binning"]), sizes["binning"], cap, p(bufs["image"]),
                          sizes["image"], C.byref(n_out), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    for k, b in bufs.items():
        assert torch.equal(b[sizes[k]:], pattern), f"capacity {cap}: the {k} buffer was written past its size"
    if rc != R.OK:
        return rc, n_out.value, None
    sv = R._StateView()
    R._check(L.b200gs_describe_state(C.byref(prm), p(bufs["geom"]), p(bufs["binning"]), cap, p(bufs["image"]), C.byref(sv)),
             "describe_state")
    nt = ((W + 15) // 16) * ((H + 15) // 16)

    def view(buf, addr, count, dtype=torch.int32):
        off = addr - buf.data_ptr()
        return buf[off:off + 4 * count].view(dtype)

    g, bb = bufs["geom"], bufs["binning"]
    D = n_out.value
    st = dict(num_rendered=D, recs=view(g, sv.geom_records, V * P * 12, torch.float32).reshape(V * P, 12),
              tiles_touched=view(g, sv.tiles_touched, V * P), offsets=view(g, sv.offsets, V * P),
              depth_order=view(bb, sv.depth_order, V * P), sorted_tile_keys=view(bb, sv.sorted_tile_keys, D),
              point_list=view(bb, sv.point_list, D), ranges=view(bb, sv.ranges, V * nt * 2).reshape(V * nt, 2))
    return rc, D, (st, radii)


def test_capacity_below_the_instance_count_deferred_path():
    """a deferred-path call whose capacity is short reports B200GS_E_BIN_TOO_SMALL with the exact count and writes nothing
    past its buffers; with capacity D exactly the state equals the reference"""
    from humangaussian_b200 import rasterizer as R
    n, V, H, W = 500, 3, 96, 160
    kw = _random_screen(n, H, W, seed=11, V=V)
    _, ref, _ = _forward(kw)
    D = ref.num_rendered
    assert V * n <= DEFERRED_MAX_NVP and D > 64
    for cap in (1, D - 33, D - 1):
        rc, d, _ = _call_forward(kw, cap)
        assert rc == R.E_BIN_TOO_SMALL and d == D, f"capacity {cap}: rc {rc}, num_rendered {d}"
    rc, d, (st, radii) = _call_forward(kw, D)
    assert rc == R.OK and d == D
    check_binning(st, radii, H, W)


def test_capacity_below_the_instance_count_exact_path():
    from humangaussian_b200 import rasterizer as R
    n, V, H, W = 65_537, 64, 32, 48
    rng = np.random.RandomState(12)
    kw = _screen(rng.uniform(0, W, n), rng.uniform(0, H, n), rng.uniform(1, 10, n), rng.uniform(0.2, 3, n), 0.5, H=H, W=W, V=V)
    _, ref, _ = _forward(kw)
    D = ref.num_rendered
    assert V * n > DEFERRED_MAX_NVP and D > V * n
    for cap in (1, D - 1):
        rc, d, _ = _call_forward(kw, cap)
        assert rc == R.E_BIN_TOO_SMALL and d == D, f"capacity {cap}: rc {rc}, num_rendered {d}"
