"""GPU: mesh cleanup (humangaussian_b200.mesh.clean_mesh, csrc/meshclean.cu) equals its numpy restatement
(mesh_clean_reference) byte for byte: the same faces in the same order and the same vertex bits, on golden case a's
marching-cubes mesh at several thresholds and on a mesh with planted floaters, duplicate and repeated-index faces and
unreferenced vertices; two runs give the same bytes; and the argument errors."""
import numpy as np
import pytest
import torch

import mesh_clean_reference as C
import mesh_edit_util as U
from humangaussian_b200 import mesh as MX

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _gpu(v, f):
    return torch.tensor(np.ascontiguousarray(v), dtype=torch.float32, device=DEV), \
        torch.tensor(np.ascontiguousarray(f), dtype=torch.int32, device=DEV)


def _same(m, ref):
    assert np.array_equal(m.faces.cpu().numpy(), ref[1])
    assert np.array_equal(m.vertices.cpu().numpy().view(np.uint32), np.asarray(ref[0], np.float32).view(np.uint32))


@pytest.mark.parametrize("kw", [{}, dict(min_faces=0, min_diameter=0.0), dict(min_faces=10, min_diameter=0.05),
                                dict(min_faces=2000, min_diameter=0.0)])
def test_clean_matches_the_restatement_on_the_golden_mesh(kw):
    v, f = U.golden_mesh()
    m = MX.clean_mesh(*_gpu(v, f), **kw)
    _same(m, C.clean_mesh(v, f, **kw))
    if not kw:
        assert m.faces.shape[0] == 7424


@pytest.mark.parametrize("seed", [0, 1])
def test_clean_matches_the_restatement_on_planted_defects(seed):
    v, f = U.planted_mesh(seed)
    for kw in ({}, dict(min_faces=0, min_diameter=0.0)):
        a = MX.clean_mesh(*_gpu(v, f), **kw)
        _same(a, C.clean_mesh(v, f, **kw))
        b = MX.clean_mesh(*_gpu(v, f), **kw)
        assert torch.equal(a.faces, b.faces) and torch.equal(a.vertices, b.vertices)


def test_clean_edge_cases_and_argument_errors():
    v, f = _gpu(*U.planted_mesh())
    empty = MX.clean_mesh(v, f[:0])
    assert empty.vertices.shape == (0, 3) and empty.faces.shape == (0, 3)
    bad = f.clone()
    bad[5, 1] = v.shape[0]
    with pytest.raises(ValueError, match="outside"):
        MX.clean_mesh(v, bad)
    bad[5, 1] = -1
    with pytest.raises(ValueError, match="outside"):
        MX.clean_mesh(v, bad)
    with pytest.raises(ValueError):
        MX.clean_mesh(v.cpu(), f.cpu())
    with pytest.raises(ValueError):
        MX.clean_mesh(v, f.long())
    with pytest.raises(ValueError):
        MX.clean_mesh(v.double(), f)
    with pytest.raises(ValueError):
        MX.clean_mesh(v, f, min_faces=-1)
