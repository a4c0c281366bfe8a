"""CPU: the numpy binning reference (tests/binning_reference.py) against the oracle's single 64-bit sort.

From the oracle's pixel centres, radii and depths alone, the reference must reproduce the oracle's rects, tiles_touched,
instance count, (tile | depth) keys, point_list and ranges bit for bit.  That makes it the oracle's sort, so the GPU tests
(test_gpu_binning.py) can check every binning intermediate against it at sizes the oracle cannot reach."""
import numpy as np
import pytest

from binning_reference import BinningReference
from util import screen_scene, small_scene


def _check(inp):
    from oracle.gs_oracle import Oracle
    o = Oracle(threads=4)
    _, radii, _, _ = o.forward(**inp)
    st = o.state()
    H, W = inp["image_height"], inp["image_width"]
    ref = BinningReference(radii, st["xy"][:, 0], st["xy"][:, 1], st["depths"], H, W)
    vis = radii > 0
    assert np.array_equal(ref.rect[vis], st["rect"][vis])
    assert np.array_equal(ref.tiles_touched, st["tiles_touched"])
    assert ref.num_rendered == st["num_rendered"]
    got = ref.view(0)
    assert np.array_equal(got["sorted_tile_keys"], (st["keys"] >> np.uint64(32)).astype(np.uint32))
    assert np.array_equal(got["point_list"], st["point_list"])
    assert np.array_equal(got["ranges"], st["ranges"])
    keys64 = (got["sorted_tile_keys"].astype(np.uint64) << np.uint64(32)) | ref.depth_keys[got["point_list"]].astype(np.uint64)
    assert np.array_equal(keys64, st["keys"])
    return ref, radii


@pytest.mark.parametrize("P,H,W,seed,D", [(600, 72, 104, 0, 1495), (4000, 64, 64, 3, 10390), (400, 17, 33, 3, 835),
                                          (60_000, 512, 512, 0, 1_358_430)])
def test_reference_is_the_oracle_sort_on_body_scenes(P, H, W, seed, D):
    """partial tiles on both axes, sub-tile images, and a 512^2 scene whose tile lists reach thousands of entries"""
    inp, _, _ = small_scene(P=P, deg=0, seed=seed, H=H, W=W)
    ref, _ = _check(inp)
    assert ref.num_rendered == D


def test_screen_fillers_mixed_with_single_tile_gaussians():
    H, W = 80, 112
    rng = np.random.RandomState(3)
    n = 90
    big = np.arange(n) % 3 == 0
    sigma = np.where(big, 60.0, 0.2)
    px = np.where(big, W / 2, (rng.randint(0, 7, n) * 16 + 7.5))
    py = np.where(big, H / 2, (rng.randint(0, 5, n) * 16 + 7.5))
    inp = screen_scene(px, py, rng.uniform(1, 5, n), sigma, 0.5, H=H, W=W)
    ref, _ = _check(inp)
    assert (ref.tiles_touched == ref.ntiles).sum() == big.sum() and (ref.tiles_touched == 1).sum() == n - big.sum()


def test_equal_depths_keep_index_order():
    H, W = 64, 96
    rng = np.random.RandomState(4)
    n = 300
    inp = screen_scene(rng.uniform(0, W, n), rng.uniform(0, H, n), np.full(n, 2.0), rng.uniform(0.3, 12, n), 0.6, H=H, W=W)
    ref, radii = _check(inp)
    assert (radii > 0).all() and len(np.unique(ref.depth_keys)) == 1
    assert np.array_equal(ref.depth_order, np.arange(n))


def test_every_gaussian_culled():
    H, W = 48, 64
    n = 50
    inp = screen_scene(np.linspace(0, W, n), np.linspace(0, H, n), np.full(n, -2.0), 3.0, 0.8, H=H, W=W)
    ref, radii = _check(inp)
    assert not radii.any() and ref.num_rendered == 0
    assert not ref.view(0)["ranges"].any()
