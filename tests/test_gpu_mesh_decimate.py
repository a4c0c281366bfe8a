"""GPU: quadric edge-collapse decimation (humangaussian_b200.mesh.decimate_mesh, csrc/meshclean.cu).

  * equal to the numpy restatement (decimate_reference) byte for byte -- the same faces in the same order, the same
    vertex bits and the same round count -- on the sphere, the torus, the golden body and the planted-defect mesh after
    cleanup, at several targets;
  * the full sample.ply scene at 256^3, cleaned and decimated to 1e5 faces: the invariants of the CPU tests
    (mesh_edit_util.check_invariants), two runs give the same bytes, and extract_colored_mesh(clean=True,
    decimate_target=100_000) returns finite unit normals at its vertices;
  * extract_mesh with the defaults is unchanged, and with the options equals clean + decimate + the world mapping;
  * argument errors.
"""
import numpy as np
import pytest
import torch

import decimate_reference as D
import mesh_clean_reference as C
import mesh_edit_util as U
from humangaussian_b200 import mesh as MX
from humangaussian_b200.scene import sample_ply_scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _gpu(v, f):
    return torch.tensor(np.ascontiguousarray(v), dtype=torch.float32, device=DEV), \
        torch.tensor(np.ascontiguousarray(f), dtype=torch.int32, device=DEV)


@pytest.fixture(scope="module")
def meshes():
    m = U.fixture_meshes()
    m["planted"] = C.clean_mesh(*U.planted_mesh(), min_faces=0, min_diameter=0.0)
    return m


@pytest.mark.parametrize("name,frac", [("sphere", 0.5), ("sphere", 0.05), ("torus", 0.2), ("torus", 0.1), ("golden", 0.5),
                                       ("golden", 0.2), ("golden", 0.05), ("planted", 0.3)])
def test_decimate_matches_the_restatement(meshes, name, frac):
    v, f = meshes[name]
    target = max(4, int(len(f) * frac))
    rv, rf, rrounds = D.decimate(v, f, target)
    m, rounds = MX._decimate(*_gpu(v, f), target)
    assert rounds == rrounds
    assert np.array_equal(m.faces.cpu().numpy(), rf)
    assert np.array_equal(m.vertices.cpu().numpy().view(np.uint32), rv.view(np.uint32))


@pytest.fixture(scope="module")
def scene():
    return sample_ply_scene().to(DEV)


def test_full_scene_at_256_decimated_to_1e5(scene):
    k, res, nb = MX._kept("t", scene.xyz, scene.opacity, scene.scaling, scene.rotation, True, 256, 16)
    v, f, _ = MX._mesh(k, res, nb, 1.5, 1.0)
    cv, cf = MX.clean_mesh(v, f)
    a = MX.decimate_mesh(cv, cf, 100_000)
    b = MX.decimate_mesh(cv, cf, 100_000)
    assert torch.equal(a.faces, b.faces) and torch.equal(a.vertices.view(torch.int32), b.vertices.view(torch.int32))
    U.check_invariants(cv.cpu().numpy(), cf.cpu().numpy(), a.vertices.cpu().numpy(), a.faces.cpu().numpy(), 100_000)
    cm = MX.extract_colored_mesh(scene, resolution=256, clean=True, decimate_target=100_000)
    assert cm.faces.shape[0] in (99_999, 100_000) and torch.equal(cm.faces, a.faces)
    n = cm.normals
    assert torch.isfinite(n).all() and torch.allclose(n.norm(dim=1), torch.ones(n.shape[0], device=DEV), atol=1e-5)
    assert cm.colors is not None and torch.isfinite(cm.colors).all()


def test_extract_mesh_options(scene):
    plain = MX.extract_mesh(scene, resolution=64)
    k, res, nb = MX._kept("t", scene.xyz, scene.opacity, scene.scaling, scene.rotation, True, 64, 16)
    v, f, w = MX._mesh(k, res, nb, 1.5, 1.0)
    assert torch.equal(plain.faces, f) and torch.equal(plain.vertices, w)
    opt = MX.extract_mesh(scene, resolution=64, clean=True, decimate_target=3000)
    cv, cf = MX.clean_mesh(v, f)
    dv, df = MX.decimate_mesh(cv, cf, 3000)
    world = ((dv.double() / 63.0 * 2 - 1) / k.scale + k.center.double()).float()
    assert torch.equal(opt.faces, df) and torch.equal(opt.vertices, world)


def test_decimate_argument_errors(meshes):
    v, f = _gpu(*meshes["sphere"])
    for t in (3, 0, -5, 4.5):
        with pytest.raises(ValueError):
            MX.decimate_mesh(v, f, t)
    bad = f.clone()
    bad[7, 2] = v.shape[0] + 3
    with pytest.raises(ValueError, match="outside"):
        MX.decimate_mesh(v, bad, 100)
    with pytest.raises(ValueError):
        MX.decimate_mesh(v.cpu(), f.cpu(), 100)
    with pytest.raises(ValueError):
        MX.decimate_mesh(v, f.long(), 100)
    with pytest.raises(ValueError):
        MX.extract_mesh(torch.zeros(4, 3, device=DEV), torch.ones(4, device=DEV), torch.ones(4, 3, device=DEV),
                        torch.ones(4, 4, device=DEV), decimate_target=2)
    tet_v = torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=torch.float32, device=DEV)
    tet_f = torch.tensor([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], dtype=torch.int32, device=DEV)
    m = MX.decimate_mesh(tet_v, tet_f, 4)
    assert torch.equal(m.faces, tet_f)
    with pytest.warns(RuntimeWarning, match="above the target"):
        MX.decimate_mesh(torch.cat([tet_v, tet_v + 5]), torch.cat([tet_f, tet_f + 4]), 4)
