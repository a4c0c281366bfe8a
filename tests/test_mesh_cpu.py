"""CPU: mesh export without a device.

  * the numpy restatement of the density field (mesh_reference) against the reference's own extract_fields
    (tests/golden/ref_mesh_fields.npz, tests/golden/make_golden_mesh.py), and the fixture's power to see a wrong
    block-membership rule;
  * the generated marching-cubes table: regeneration reproduces the committed header, and all 256 cases are checked;
  * the CPU marching cubes on analytic closed surfaces: 2-manifold, Euler characteristic, outward orientation, volume;
  * argument checks of humangaussian_b200.mesh that need no device.
"""
import os

import numpy as np
import pytest
import torch

import mesh_reference as M
from humangaussian_b200 import mc_table
from humangaussian_b200 import mesh as MX

TOL_ABS = TOL_REL = 1e-5


@pytest.fixture(scope="module")
def golden():
    return np.load(M.GOLDEN)


def _field(z, tag, relax_shift=0.0):
    res, nb, rr = z[f"{tag}_args"]
    return M.Field(*M.golden_inputs(z, tag), int(res), int(nb), rr + relax_shift)


def _ratio(got, ref):
    return float((np.abs(got - ref) / (TOL_ABS + TOL_REL * np.abs(ref))).max())


@pytest.mark.parametrize("tag", ["b", "c", "d"])
def test_restated_field_matches_the_reference(golden, tag):
    """b: 40^3 / 16 blocks (split 2, 20 chunks); c: 33^3 / 8 (last chunk 1 sample); d: synthetic, relax 0.5."""
    F = _field(golden, tag)
    assert np.array_equal(F.center, golden[f"{tag}_center"]) and F.scale == float(golden[f"{tag}_scale"])
    ref = golden[f"{tag}_occ"]
    assert ref.max() > 0.1
    assert _ratio(F.full(), ref) <= 1.0


def test_restated_field_matches_the_reference_full_scene(golden):
    """a: the full sample.ply at 64^3 / 16 blocks, on a seeded sample of 48 non-empty blocks (the whole grid takes minutes)."""
    F = _field(golden, "a")
    ref = golden["a_occ"]
    assert np.array_equal(F.center, golden["a_center"]) and F.scale == float(golden["a_scale"])
    s = F.split
    nz = np.argwhere(ref.reshape(16, s, 16, s, 16, s).max((1, 3, 5)) > 0)
    pick = nz[np.random.default_rng(0).choice(len(nz), 48, replace=False)]
    assert any(ref[bx * s:(bx + 1) * s, by * s:(by + 1) * s, bz * s:(bz + 1) * s].max() > 1 for bx, by, bz in pick)
    for bx, by, bz in pick:
        got = F.block(bx, by, bz)
        assert _ratio(got, ref[bx * s:(bx + 1) * s, by * s:(by + 1) * s, bz * s:(bz + 1) * s]) <= 1.0, (bx, by, bz)


def test_fixture_detects_a_wrong_membership_rule(golden):
    """Case d with relax_ratio moved by one block either way differs from the reference far beyond the tolerance."""
    ref = golden["d_occ"]
    for shift in (+1.0, -0.5):  # 0.5 -> 1.5 blocks, and 0.5 -> 0 (no widening)
        assert _ratio(_field(golden, "d", shift).full(), ref) > 1e3


def test_triangle_table_regenerates_the_committed_header():
    with open(mc_table.HEADER) as f:
        assert f.read() == mc_table.render_header(mc_table.build_table())


def _corner_pos(k):
    return np.array(mc_table.corner(k))


def test_every_case_uses_only_crossing_edges_and_closes_across_faces():
    """For all 256 cases: each triangle vertex sits on a crossing edge, each crossing edge is used, every triangle edge
    is either an interior diagonal (two triangles, not inside one face) or a boundary segment on a cube face (one
    triangle); and the boundary segments on a face depend only on that face's signs, with opposite direction seen from the
    neighbouring cell -- so the pieces of adjacent cells pair up."""
    table = mc_table.build_table()
    edges = mc_table.EDGES
    face_of = {}  # case -> {(axis, side): set of directed segments in face-local form}
    for case in range(256):
        crossing = {e for e, (c0, c1, _) in enumerate(edges) if ((case >> c0) & 1) != ((case >> c1) & 1)}
        used = {e for t in table[case] for e in t}
        assert used == crossing, case
        directed = [(t[i], t[(i + 1) % 3]) for t in table[case] for i in range(3)]
        und = {}
        for a, b in directed:
            und.setdefault(frozenset((a, b)), []).append((a, b))
        segs = {}
        for key, uses in und.items():
            a, b = tuple(key)
            common = mc_table.edge_faces(a) & mc_table.edge_faces(b)
            if len(uses) == 2:
                assert not common, (case, a, b)  # an interior diagonal
                assert uses[0] == uses[1][::-1], case  # consistent winding
            else:
                assert len(uses) == 1 and len(common) == 1, (case, a, b)
                (fa, fs), = common
                segs.setdefault((fa, fs), set()).add(uses[0])
        face_of[case] = segs
    # a segment in face-local form: the two edges' corner positions with the face axis dropped
    def local(seg, fa):
        out = []
        for e in seg:
            c0, c1, _ = edges[e]
            out.append(tuple(sorted(tuple(np.delete(_corner_pos(c), fa)) for c in (c0, c1))))
        return tuple(out)
    for fa in range(3):
        for ca in range(256):
            for cb in range(256):
                # cell B sits on the +fa side of cell A: A's face (fa, 1) is B's face (fa, 0)
                if any(((ca >> k) & 1) != ((cb >> (k ^ (1 << fa))) & 1) for k in range(8) if (k >> fa) & 1):
                    continue
                sa = {local(s, fa) for s in face_of[ca].get((fa, 1), set())}
                sb = {local(s[::-1], fa) for s in face_of[cb].get((fa, 0), set())}
                assert sa == sb, (fa, ca, cb)


@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_cpu_marching_cubes_closed_surfaces(shape):
    vol, prm = M.sphere(64) if shape == "sphere" else M.torus(64)
    v, f = M.marching_cubes(M.pad(vol), 0.0)
    hist, chi, vol_signed = M.mesh_stats(v, f)
    assert len(hist) == 3 and hist[2] > 0 and hist[:2].sum() == 0  # every edge in exactly two faces
    assert chi == (2 if shape == "sphere" else 0)
    analytic = 4 / 3 * np.pi * prm ** 3 if shape == "sphere" else 2 * np.pi ** 2 * prm[0] * prm[1] ** 2
    assert vol_signed > 0 and abs(vol_signed / analytic - 1) < 0.01


def test_cpu_marching_cubes_noise_is_a_closed_manifold():
    """Seeded noise exercises the ambiguous faces; padded below iso, the surface is closed."""
    vol = M.pad(np.random.default_rng(0).standard_normal((32, 32, 32)).astype(np.float32), -10.0)
    v, f = M.marching_cubes(vol, 0.0)
    hist, _, vol_signed = M.mesh_stats(v, f)
    assert len(hist) == 3 and hist[:2].sum() == 0 and vol_signed > 0
    assert len(np.unique(f)) == len(v)  # every vertex is used


def test_cpu_marching_cubes_vertex_positions_and_empty():
    vol = np.zeros((3, 3, 3), np.float32)
    vol[1, 1, 1] = 4.0
    v, f = M.marching_cubes(vol, 1.0)
    assert len(v) == 6 and len(f) == 8  # an octahedron
    assert np.array_equal(np.abs(v - 1).sum(1), np.full(6, 0.75, np.float32))  # iso 1 is 3/4 of the way from 4 down to 0
    v, f = M.marching_cubes(vol, 4.0)  # nothing is > iso
    assert v.shape == (0, 3) and f.shape == (0, 3)


def test_argument_checks_without_a_device():
    z = torch.zeros
    with pytest.raises(RuntimeError, match="CUDA device"):
        MX.extract_fields(z(4, 3), z(4, 1), z(4, 3), z(4, 4))
    for res, nb in ((128, 3), (10, 16), (0, 16), (128, 0), (64.0, 16)):
        with pytest.raises(ValueError):
            MX._check_grid(res, nb)
    for res, nb in ((128, 16), (40, 16), (33, 8), (512, 16), (7, 2)):
        assert MX._check_grid(res, nb) == (res, nb)
    with pytest.raises(ValueError, match="wrong shape"):
        MX.marching_cubes(z(4, 4, 4), 0.0)  # a CPU volume
    with pytest.raises(ValueError):
        MX.save_obj(os.devnull, np.zeros((3, 3)), np.array([[0, 1, 3]]))


def test_save_obj(tmp_path):
    p = tmp_path / "m.obj"
    MX.save_obj(p, torch.tensor([[0.0, 0, 0], [1, 0, 0], [0, 1, 0]]), torch.tensor([[0, 1, 2]], dtype=torch.int32))
    assert p.read_text().split("\n")[:4] == ["v 0 0 0", "v 1 0 0", "v 0 1 0", "f 1 2 3"]
