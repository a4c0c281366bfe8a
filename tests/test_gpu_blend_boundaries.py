"""GPU: the backward blend's contributor masks and sums on screen-space scenes built to hit its boundaries.

The backward blend stages only entries whose contributor-mask bit is set, parks each hit's per-pixel (q, w), and turns every
16 parked hits (and the rest at the end) into the ten per-Gaussian sums.  Random scenes reach the edges of that machinery only
by chance, so these scenes place Gaussians by pixel (tests/util.py, screen_scene) to reach them on purpose:
  * flush and chunk counts: a patch that stages n in {1, 15, 16, 17, 31, 32, 33, 48, 63, 64, 65, 97} hits (n = 0, 1, 15 mod 16;
    largest n_contrib on and next to a chunk edge);
  * zero chunks: runs of entries of a neighbouring patch, interleaved in depth with the target patch's, that pass the target
    patch's support-box test without contributing to it;
  * early termination on a chunk edge: wmax = 32, 33 and 64;
  * partial patches at the right and bottom edges of a 123x61 image;
  * the cull edge: needles just under and just over the 1e4 anisotropy above which the kernels never cull a Gaussian, at
    opacity (1/255)(1 + 1e-3), so that alpha sits on the 1/255 threshold.
Every scene asserts, from the oracle's state, that it still exercises its case; then the masks must match the oracle bit for
bit and the sums must hold the bound of tests/test_gpu_parity.py."""
import math

import numpy as np
import pytest

from test_gpu_parity import _check_backward_sums, _check_forward_state, _gpu_blend_state, _oracle, _packed_masks, _patch_wmax
from util import screen_scene

pytestmark = pytest.mark.gpu

COUNTS = (1, 15, 16, 17, 31, 32, 33, 48, 63, 64, 65, 97)
SIG = 0.2  # screen sigma (px): the 0.3 px^2 dilation dominates the footprint


def _patch_origin(tile_x, tile_y, patch):
    return tile_x * 16 + (patch & 1) * 8, tile_y * 16 + (patch >> 1) * 4


def _stack(x, y, n, z0, opacity=0.05):
    """n Gaussians centred at pixel-space (x, y), depths z0, z0 + 1e-3, ... (list order = stack order)"""
    return dict(px=np.full(n, x), py=np.full(n, y), depth=z0 + 1e-3 * np.arange(n), opacity=np.full(n, opacity))


def _cat(parts):
    return {k: np.concatenate([p[k] for p in parts]) for k in ("px", "py", "depth", "opacity")}


def _staged(o_st, H, W):
    """[tiles, 8] number of entries each patch's backward stages (contributor-mask bits set in the words it reads)"""
    wmax = _patch_wmax(o_st["n_contrib"], H, W)
    cnt = np.zeros_like(wmax)
    for t, (r0, r1) in enumerate(o_st["ranges"]):
        for p in range(8):
            if wmax[t, p] > 0:
                cnt[t, p] = int(((o_st["contrib_patches"][r0:r0 + wmax[t, p]] >> p) & 1).sum())
    return cnt, wmax


def _run(inp, seed):
    o_out, o_st, gimg, o_grads = _oracle(inp, seed)
    _check_forward_state(inp, o_out, o_st)  # forward state bit-exact, contributor masks included
    _check_backward_sums(inp, gimg, o_grads)
    return o_st, o_grads


def _stacks_scene():
    """Tiles 0..11 of a 128x64 image: a stack of n in COUNTS in patch 0.  Tile 12: the zero-chunk case."""
    parts = []
    for i, n in enumerate(COUNTS):
        x0, y0 = _patch_origin(i % 8, i // 8, 0)
        parts.append(_stack(x0 + 3.5, y0 + 1.5, n, 1.0 + i))
    # tile (4, 1): target patch 0 gets 5 + 5 + 5 entries, separated by runs of 70 entries of patch 1 placed where their
    # support box still reaches patch 0 (|dx| to column 7 just above the true support of alpha >= 1/255, below the box's
    # conservative half width) but alpha < 1/255 on all of patch 0's pixels
    x0, y0 = _patch_origin(4, 1, 0)
    ca = SIG * SIG + 0.3
    tau = math.log(255 * 0.05)
    sup = math.sqrt(2 * tau * ca - 0.25)                          # rows at dy = 0.5 from the centre
    box = math.sqrt(2 * (tau + 0.02) * ca) * 1.0005 + 0.02
    xr = x0 + 7 + 0.5 * (sup + box)
    z = 20.0
    for k in range(3):
        parts.append(_stack(x0 + 3.5, y0 + 1.5, 5, z))
        z += 1.0
        if k < 2:
            parts.append(_stack(xr, y0 + 1.5, 70, z))
            z += 1.0
    return _cat(parts), (12, xr)


def test_flush_and_chunk_counts_and_zero_chunks():
    g, (zt, xr) = _stacks_scene()
    inp = screen_scene(g["px"], g["py"], g["depth"], SIG, g["opacity"], H=64, W=128)
    o_st, _ = _run(inp, 31)
    cnt, wmax = _staged(o_st, 64, 128)
    # coverage: every stack's patch stages exactly n hits, and nothing else stages there
    assert [int(cnt[i, 0]) for i in range(len(COUNTS))] == list(COUNTS), cnt[:12, 0]
    assert {n % 16 for n in COUNTS} >= {0, 1, 15} and {32, 33, 64, 65} <= set(wmax[:12, 0].tolist())
    assert o_st["final_T"].min() > 1e-3, "stacks must not terminate"
    # coverage of the zero-chunk tile: target patch 0 of tile 12 reads chunks 0..4; 1 and 3 are zero, 2 and 4 are not, and every
    # entry of chunk 1 passes patch 0's support-box test (the GPU's own hx, hy) without contributing
    r0, r1 = (int(v) for v in o_st["ranges"][zt])
    words = _packed_masks(o_st["contrib_patches"], r0, r1, 5)[:, 0]
    assert wmax[zt, 0] == 155 and list(words != 0) == [True, False, True, False, True], words
    st, _ = _gpu_blend_state(inp, _grad(inp))
    recs = st["recs"]
    ids = o_st["point_list"][r0 + 32:r0 + 64]
    px_, py_, hx, hy = (recs[ids, k] for k in range(4))
    x0, y0 = _patch_origin(4, 1, 0)
    hit = (hx >= 0) & (px_ + hx >= x0) & (px_ - hx <= x0 + 7) & (py_ + hy >= y0) & (py_ - hy <= y0 + 3)
    assert hit.all(), "the runs no longer reach the target patch's support box"


def _grad(inp):
    from util import grad_images
    return grad_images(inp["image_height"], inp["image_width"], 31)


def test_early_termination_on_chunk_edges():
    """Tiles 0..2 of a 48x16 image hold 31, 32 and 63 faint entries in patch 0; two image-wide opaque Gaussians behind them
    stop every pixel at the second one, so every patch's wmax is 32, 33 or 64."""
    parts = []
    for i, n in enumerate((31, 32, 63)):
        x0, y0 = _patch_origin(i, 0, 0)
        parts.append(_stack(x0 + 3.5, y0 + 1.5, n, 1.0 + i))
    parts.append(_stack(24.0, 8.0, 2, 10.0, opacity=0.999))
    g = _cat(parts)
    sig = np.where(g["opacity"] > 0.5, 2000.0, SIG)
    inp = screen_scene(g["px"], g["py"], g["depth"], sig, g["opacity"], H=16, W=48)
    o_st, _ = _run(inp, 32)
    _, wmax = _staged(o_st, 16, 48)
    assert [sorted(set(wmax[t].tolist())) for t in range(3)] == [[32], [33], [64]], wmax
    assert (o_st["final_T"] < 0.011).all()  # every pixel stopped at the second opaque entry


def test_partial_patches_at_the_image_edge():
    """The stacks in the edge patches of a 123x61 image: cols 120-122 (3 of 8) and row 60 (1 of 4)."""
    W, H = 123, 61
    spots = [(7, 0, 3), (7, 1, 3), (7, 2, 5), (7, 3, 7)] + [(tx, 3, 6) for tx in range(7)] + [(0, 3, 7)]
    parts = []
    for i, (n, (tx, ty, p)) in enumerate(zip(COUNTS, spots)):
        x0, y0 = _patch_origin(tx, ty, p)
        x = 121.0 if x0 == 120 else x0 + 3.5
        y = 60.45 if y0 == 60 else y0 + 1.5  # row 59 (dy 1.45) is outside the alpha support: only row 60 sees it
        parts.append(_stack(x, y, n, 1.0 + i))
    g = _cat(parts)
    inp = screen_scene(g["px"], g["py"], g["depth"], SIG, g["opacity"], H=H, W=W)
    o_st, _ = _run(inp, 33)
    cnt, _ = _staged(o_st, H, W)
    gx = 8
    got = [int(cnt[ty * gx + tx, p]) for (tx, ty, p) in spots]
    assert got == list(COUNTS), got


def _needle_cov(aniso):
    """screen covariance of a 45-degree needle whose dilated 2D covariance has (ca*cc)/det = aniso"""
    L2 = 1.0
    for _ in range(200):  # aniso = (L2/2 + 0.3)^2 / (0.3 L2 + 0.09), increasing in L2: bisect on a log scale
        L2 *= 2.0
        if (L2 / 2 + 0.3) ** 2 / (0.3 * L2 + 0.09) > aniso:
            break
    lo, hi = L2 / 2, L2
    for _ in range(100):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if (mid / 2 + 0.3) ** 2 / (0.3 * mid + 0.09) < aniso else (lo, mid)
    return np.array([[lo / 2, lo / 2], [lo / 2, lo / 2]])


def test_cull_edge_needles():
    """Two needles through pixel centres, anisotropy 0.99e4 (support box computed) and 1.01e4 (never culled), at opacity
    (1/255)(1 + 1e-3): only pixels within ~0.02 px of the centre line reach alpha >= 1/255, a decision both sides must take
    identically; plus faint stacks in patches the never-culled needle stages without contributing."""
    op = (1.0 / 255.0) * (1 + 1e-3)
    px = np.array([40.0, 90.0, 20.5, 100.5])
    py = np.array([30.0, 33.0, 9.5, 53.5])
    depth = np.array([2.0, 3.0, 1.0, 1.5])
    opac = np.array([op, op, 0.05, 0.05])
    cov = np.zeros((4, 2, 2))
    cov[0], cov[1] = _needle_cov(0.99e4), _needle_cov(1.01e4)
    cov[2, 0, 0] = cov[2, 1, 1] = cov[3, 0, 0] = cov[3, 1, 1] = SIG * SIG
    inp = screen_scene(px, py, depth, SIG, opac, cov2d=cov, H=64, W=128)
    o_st, _ = _run(inp, 34)
    st, _ = _gpu_blend_state(inp, _grad(inp))
    hx = st["recs"][:2, 2]
    assert hx[0] < 1e3 and hx[1] > 1e37, f"needles no longer straddle the never-cull threshold: hx = {hx}"
    # both needles contribute at a few pixels on their centre line and nowhere else
    cp, pl = o_st["contrib_patches"], o_st["point_list"]
    for g in (0, 1):
        assert 0 < int(np.count_nonzero(cp[pl == g])) < 8
