"""CPU: the contribution-score reference (tests/contribution_reference.py) against the oracle and against float64 autograd.

  1. The replay reproduces the oracle's n_contrib and contrib_patches bit for bit, so its (pixel, entry) decisions are the
     oracle's, and hence the kernels' (the GPU forward state is bit-identical to the oracle's).
  2. With colours precomputed and L = sum over pixels of colour channel 0, dL/dcolors[g, 0] = sum_p w_pg exactly.  The
     replay's weight_sum * 2^-24 matches that gradient of oracle/dense_ref.py (float64, torch.autograd; no code shared with
     the replay) at the float32-vs-float64 tolerance of the other autograd checks (1e-4 abs, 1e-3 rel).
  3. Global identity: sum_g weight_sum * 2^-24 equals the sum over pixels of the oracle's alpha image up to
       sum_p (n_p - 1) 2^-24   (each alpha is a float32 sequential sum of n_p weights, every partial sum <= 1, so each add
                                 rounds by at most 2^-25 ... 2^-24 of a value <= 1; n_p = blends at pixel p)
     + n 2^-25                  (one quantisation of at most 2^-25 per blend, n blends in total),
     a bound fixed before the test was first run.
  4. touches - blends = the number of pixels that terminated."""
import numpy as np
import pytest
import torch

import contribution_reference as CR
from util import grads_agree, small_scene

U = 2.0 ** -24


def _colors_inp(inp, seed=0):
    """the same scene with precomputed colours in place of SH (colours do not enter the weights)"""
    out = {k: v for k, v in inp.items() if k not in ("shs",)}
    out["colors_precomp"] = np.random.RandomState(seed).rand(len(inp["means3D"]), 3).astype(np.float32)
    out["sh_degree"] = 0
    return out


def _dense_weight_sums(inp, st, radii, antialiasing=False):
    from oracle.dense_ref import dense_render
    t64 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)
    ids = np.nonzero(radii > 0)[0]
    order = ids[np.lexsort((ids, st["depths"][ids]))]
    col = t64(inp["colors_precomp"]).requires_grad_(True)
    H, W = inp["image_height"], inp["image_width"]
    kw = dict(means3D=t64(inp["means3D"]), means2D=torch.zeros(len(radii), 3, dtype=torch.float64),
              opacities=t64(inp["opacities"]), viewmatrix=t64(inp["viewmatrix"]), projmatrix=t64(inp["projmatrix"]),
              campos=t64(inp["campos"]), bg=t64(inp["bg"]), H=H, W=W, tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"],
              radii=radii, rect=st["rect"], order=order, colors_precomp=col, scales=t64(inp["scales"]),
              rotations=t64(inp["rotations"]))
    if antialiasing:
        from aa_reference import dense_render_aa
        c = dense_render_aa(**kw)[0]
    else:
        c = dense_render(**kw)[0]
    c[0].sum().backward()
    return col.grad[:, 0].numpy()


def _check(inp, antialiasing=False):
    ref = CR.contribution([inp], antialiasing=antialiasing)
    v = ref["views"][0]
    st, out = v["state"], v["out"]
    radii = np.asarray(out[1]).reshape(-1)
    # 1. the replay's decisions are the oracle's
    assert np.array_equal(v["n_contrib"], st["n_contrib"])
    assert np.array_equal(v["contrib_patches"], st["contrib_patches"])
    # 2. against float64 autograd
    ws = ref["weight_sum"].astype(np.float64) * U
    dense = _dense_weight_sums(inp, st, radii, antialiasing)
    ok, msg = grads_agree(ws[:, None], dense[:, None], atol=1e-4, rtol=1e-3)
    assert ok, f"weight_sum vs float64 autograd: {msg}"
    # 3. the global alpha identity, with the bound stated in the module docstring
    alpha = np.asarray(out[3], np.float64)
    n_blends = int(ref["blends"].sum())
    # a pixel blends at most n_contrib (its last blended list position) entries
    bound = float(np.maximum(v["n_contrib"].astype(np.float64) - 1, 0).sum()) * U + n_blends * U / 2
    assert abs(ws.sum() - alpha.sum()) <= bound, (ws.sum(), alpha.sum(), bound)
    # 4. touches - blends = terminated pixels
    assert int(ref["touches"].sum() - ref["blends"].sum()) == ref["terminated"]
    # consistency: a Gaussian has a maximum iff it blended, and every blend is a touch
    assert np.array_equal(ref["weight_max"] > 0, ref["blends"] > 0)
    assert (ref["touches"] >= ref["blends"]).all()
    assert (ref["blends"] > 0).sum() > 20
    return ref


@pytest.mark.parametrize("deg", [0, 2])
def test_small_scene_against_autograd(deg):
    inp, _, _ = small_scene(P=300, deg=deg, seed=deg, H=37, W=50)
    _check(_colors_inp(inp, deg))


def test_dense_opaque_scene_terminates():
    inp, _, _ = small_scene(P=500, deg=1, seed=9, H=32, W=32, dist=1.3)
    inp["opacities"] = np.clip(inp["opacities"] * 8, 0, 0.99999).astype(np.float32)
    inp["scales"] = (inp["scales"] * 2.0).astype(np.float32)
    ref = _check(_colors_inp(inp, 9))
    assert ref["terminated"] > 100, "scene too thin to exercise the terminating hit"


def test_antialiasing():
    inp, _, _ = small_scene(P=300, deg=1, seed=11, H=37, W=50)
    _check(_colors_inp(inp, 11), antialiasing=True)


def test_blend_state_scene_replay():
    """the scene of tests/test_oracle_blend_state.py (partial tiles and patches on both axes)"""
    inp, _, _ = small_scene(P=300, deg=1, seed=2, H=37, W=50)
    ref = CR.contribution([inp])
    v = ref["views"][0]
    assert np.array_equal(v["n_contrib"], v["state"]["n_contrib"])
    assert np.array_equal(v["contrib_patches"], v["state"]["contrib_patches"])
