"""CPU: the numpy restatements of mesh cleanup (mesh_clean_reference) and decimation (decimate_reference).

  * components of golden case a's marching-cubes mesh equal scipy's; at the defaults exactly the 7 424-face body stays;
  * the planted-defect mesh loses exactly its floaters, duplicate and repeated-index faces and unreferenced vertices;
  * decimation of the sphere, the torus and the golden body at several targets keeps the invariants (mesh_edit_util)
    and stays within each case's distance bound of the input, both ways;
  * the fixtures see a wrong rule: a midpoint-only position breaks the distance bound, a missing link check the
    topology.

The distance bound.  A flat triangle of edge l interpolating a surface of curvature k deviates from it by about
k l^2 / 8, so the bound of each case grows with its mean output edge and the surface's curvature.  Each case states its
bound in grid units: the two-sided distance the quadric rule gives there, rounded up by about 20 %.  Measured (quadric /
midpoint-only): sphere 50 % 0.17 / 0.19, sphere 5 % 0.51 / 0.70, torus 20 % 0.42 / 0.40, torus 10 % 0.64 / 0.62, golden
body 50 % 0.78 / 1.24, golden body 20 % 1.37 / 1.75.  The midpoint rule, which cuts chords inward, breaks three bounds.
"""
import numpy as np
import pytest

import decimate_reference as D
import mesh_clean_reference as C
import mesh_edit_util as U

CASES = [("sphere", 0.5, 0.25), ("sphere", 0.05, 0.6), ("torus", 0.2, 0.55), ("torus", 0.1, 0.8), ("golden", 0.5, 1.0),
         ("golden", 0.2, 1.7)]  # (mesh, share of the faces kept, distance bound in grid units)


@pytest.fixture(scope="module")
def meshes():
    return U.fixture_meshes()


def test_components_of_the_golden_mesh_match_scipy_and_only_the_body_stays():
    v, f = U.golden_mesh()
    ff = np.asarray(f, np.int64)
    lab = C.vertex_labels(len(v), ff)[ff[:, 0]]
    ref = U.face_components(len(v), ff)
    # the same partition: a bijection between the labels
    pairs = np.unique(np.stack([lab, ref], 1), axis=0)
    assert len(pairs) == len(np.unique(lab)) == len(np.unique(ref)) == 65
    cv, cf = C.clean_mesh(v, f)
    assert len(cf) == 7424
    assert len(np.unique(U.face_components(len(cv), cf))) == 1
    used = np.unique(ff[ref == np.bincount(ref).argmax()])
    assert np.array_equal(cv, v[used]) and len(cv) == len(used)


def test_planted_defects_are_removed():
    v, f = U.planted_mesh()
    ok = C.face_filter(f)
    assert ok.sum() == len(f) - 3  # a repeated index, a duplicate, a reversed duplicate
    cv, cf = C.clean_mesh(v, f)
    assert len(np.unique(U.face_components(len(cv), cf))) == 1
    assert len(np.unique(cf)) == len(cv)
    keep_all_v, keep_all_f = C.clean_mesh(v, f, min_faces=0, min_diameter=0.0)
    assert len(keep_all_f) == len(f) - 3 and len(keep_all_v) == len(v) - 7


@pytest.mark.parametrize("name,frac,bound", CASES)
def test_decimation_keeps_the_invariants(meshes, name, frac, bound):
    v, f = meshes[name]
    target = int(len(f) * frac)
    dv, df, rounds = D.decimate(v, f, target)
    U.check_invariants(v, f, dv, df, target)
    assert U.two_sided_distance(v, f, dv, df) < bound
    dv2, df2, _ = D.decimate(v, f, target)
    assert np.array_equal(dv, dv2) and np.array_equal(df, df2)


def test_fixture_detects_a_midpoint_only_rule(meshes):
    broken = 0
    for name, frac, bound in CASES:
        v, f = meshes[name]
        target = int(len(f) * frac)
        dv, df, _ = D.decimate(v, f, target, rule="midpoint")
        broken += U.two_sided_distance(v, f, dv, df) >= bound
    assert broken >= 3


def test_fixture_detects_a_missing_link_check(meshes):
    v, f = meshes["golden"]
    target = int(len(f) * 0.5)
    dv, df, _ = D.decimate(v, f, target, link_check=False)
    with pytest.raises(AssertionError):
        U.check_invariants(v, f, dv, df, target)


def test_tetrahedron_and_open_meshes_stop_early():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)
    dv, df, rounds = D.decimate(v, f, 4)
    assert rounds == 0 and len(df) == 4
    # an open grid: every vertex touches the boundary or is locked by it only at the rim; interior collapses happen
    n = 6
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2)
    gv = np.concatenate([g, np.zeros((len(g), 1))], 1).astype(np.float32)
    quads = [(i * n + j, (i + 1) * n + j, (i + 1) * n + j + 1, i * n + j + 1) for i in range(n - 1) for j in range(n - 1)]
    gf = np.array([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))], np.int32)
    dv, df, rounds = D.decimate(gv, gf, 4)
    assert len(df) > 4 and rounds >= 1
    rim = (g[:, 0] == 0) | (g[:, 0] == n - 1) | (g[:, 1] == 0) | (g[:, 1] == n - 1)
    assert {tuple(r) for r in gv[rim]} <= {tuple(r) for r in dv}  # boundary vertices never move
