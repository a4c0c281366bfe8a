"""CPU: coloured mesh export without a device.

  * the numpy restatement of the field query (mesh_color_reference) against itself and mesh_reference: G is the
    gradient of D (central differences), D at grid samples is the restated field, a uniform-SH scene has that colour
    everywhere, and a degree-1 scene has SH(sh, -n) along its own normals;
  * save_obj: the same bytes as before without normals or colours, and v / vn / f lines that parse back exactly with them;
  * save_ply_mesh: parsed back by a small numpy reader;
  * argument checks of humangaussian_b200.mesh that need no device.
"""
import numpy as np
import pytest
import torch

import mesh_color_reference as C
import mesh_reference as M
from humangaussian_b200 import mesh as MX
from humangaussian_b200.scene import GaussianParams

f32 = np.float32


def _query(P=400, seed=0, deg=0, res=32, nb=8, sh=None):
    xyz, op, sc, rot, shs = C.synthetic(P, seed, deg, sh=sh)
    return C.Query(xyz, op, sc, rot, res, nb, 1.5, shs, deg)


def _points(Q, n, seed):
    """n seeded float32 points on a 2^-10 lattice inside the kept centres' box (so q +- 2^-12 is exact)."""
    rng = np.random.default_rng(seed)
    lo, hi = Q.F.x.min(0), Q.F.x.max(0)
    return (np.round(rng.uniform(lo, hi, (n, 3)) * 1024) / 1024).astype(f32)


def test_gradient_is_the_central_difference_of_density():
    Q = _query()
    q = _points(Q, 300, 1)
    r = Q.eval(q)
    h = 2.0 ** -12
    hq = np.stack([C.home(Q.F.lin, Q.F.split, Q.F.nch, q[:, a]) for a in range(3)], 1)
    checked = 0
    for a in range(3):
        e = np.zeros(3, f32)
        e[a] = h
        qp, qm = q + e, q - e
        same = np.ones(len(q), bool)
        for qq in (qp, qm):  # membership must not change across the stencil
            same &= np.all(np.stack([C.home(Q.F.lin, Q.F.split, Q.F.nch, qq[:, b]) for b in range(3)], 1) == hq, 1)
        fd = (Q.eval(qp)["D"] - Q.eval(qm)["D"]) / (2 * h)
        err = np.abs(fd - r["G"][:, a])[same]
        assert np.all(err <= 2e-3 * r["G_abs"][same, a] + 1e-9), err.max()
        checked += int(same.sum())
    assert checked > 600 and (r["D"] > 0.1).sum() > 50


@pytest.mark.parametrize("tag", ["b", "d"])
def test_density_at_grid_samples_is_the_restated_field(tag):
    z = np.load(M.GOLDEN)
    res, nb, rr = z[f"{tag}_args"]
    raw = M.golden_inputs(z, tag)
    Q = C.Query(*raw, int(res), int(nb), float(rr))
    rng = np.random.default_rng(2)
    hot = np.argwhere(z[f"{tag}_occ"] > 0.2 * z[f"{tag}_occ"].max())
    vox = np.concatenate([hot[rng.choice(len(hot), 1000)], rng.integers(0, int(res), (1000, 3))])
    want = Q.F.at(vox).astype(np.float64)
    got = Q.eval(Q.F.lin[vox])["D"]
    assert (want > 0.1).sum() > 500
    assert np.all(np.abs(got - want) <= 1e-6 * np.abs(want) + 1e-9)
    # and it is the golden field of the reference itself
    occ = z[f"{tag}_occ"][vox[:, 0], vox[:, 1], vox[:, 2]]
    assert np.all(np.abs(got - occ) <= 1e-5 * np.abs(occ) + 1e-5)


def test_uniform_sh_gives_that_colour_everywhere():
    sh = np.array([[0.3, -0.2, 1.1]], f32)
    Q = _query(deg=0, sh=sh)
    r = Q.eval(_points(Q, 500, 3))
    col, _ = Q.colors(r)
    inside = r["D"] > 0
    want = np.maximum(C.SH_C0 * sh[0].astype(np.float64) + 0.5, 0.0)
    assert inside.sum() > 400
    assert np.allclose(col[inside], want, rtol=0, atol=1e-12) and np.all(col[~inside] == 0)
    # degree 3, view-independent: the DC term alone
    sh3 = np.random.default_rng(4).standard_normal((16, 3)).astype(f32)
    Q3 = _query(deg=3, sh=sh3)
    r3 = Q3.eval(_points(Q3, 200, 5))
    col3, _ = Q3.colors(r3, view_dependent=False)
    ok = r3["D"] > 0
    assert np.allclose(col3[ok], np.maximum(C.SH_C0 * sh3[0].astype(np.float64) + 0.5, 0.0), rtol=0, atol=1e-12)


def test_degree_1_colour_is_sh_along_minus_the_normal():
    sh = np.array([[0.4, 0.1, -0.3], [0.5, -0.6, 0.2], [-0.7, 0.3, 0.9], [0.2, 0.8, -0.4]], f32).astype(np.float64)
    Q = _query(deg=1, sh=sh.astype(f32))
    r = Q.eval(_points(Q, 400, 6))
    col, _ = Q.colors(r)
    ok = np.linalg.norm(r["normal"], axis=1) > 0
    x, y, z = (-r["normal"][ok, k][:, None] for k in range(3))  # dir = -n
    want = C.SH_C0 * sh[0] - C.SH_C1 * y * sh[1] + C.SH_C1 * z * sh[2] - C.SH_C1 * x * sh[3] + 0.5
    assert ok.sum() > 300
    assert np.allclose(col[ok], np.maximum(want, 0.0), rtol=0, atol=1e-12)
    assert np.allclose(np.linalg.norm(r["normal"][ok], axis=1), 1.0)


def _old_save_obj(path, v, f):
    """save_obj as it was before normals and colours: the byte format existing files and readers rely on."""
    v = np.asarray(v, np.float64).reshape(-1, 3)
    f = np.asarray(f, np.int64).reshape(-1, 3)
    with open(path, "w") as fh:
        if len(v):
            fh.write("\n".join("v %.9g %.9g %.9g" % tuple(r) for r in v) + "\n")
        if len(f):
            fh.write("\n".join("f %d %d %d" % tuple(r) for r in f + 1) + "\n")


def _mesh(seed=0, V=50, F=80):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((V, 3)).astype(f32)
    f = rng.integers(0, V, (F, 3)).astype(np.int32)
    n = rng.standard_normal((V, 3)).astype(f32)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    c = rng.uniform(-0.3, 1.3, (V, 3)).astype(f32)
    return v, f, n, c


def test_save_obj_plain_is_unchanged_and_extended_lines_parse_back(tmp_path):
    v, f, n, c = _mesh()
    _old_save_obj(tmp_path / "old.obj", v, f)
    MX.save_obj(tmp_path / "new.obj", torch.tensor(v), torch.tensor(f))
    assert (tmp_path / "new.obj").read_bytes() == (tmp_path / "old.obj").read_bytes()
    MX.save_obj(tmp_path / "e.obj", v, f)
    assert (tmp_path / "e.obj").read_bytes() == (tmp_path / "old.obj").read_bytes()

    MX.save_obj(tmp_path / "c.obj", v, f, normals=n, colors=c)
    lines = (tmp_path / "c.obj").read_text().splitlines()
    vl = np.array([[float(t) for t in ln.split()[1:]] for ln in lines if ln.startswith("v ")], np.float64)
    nl = np.array([[float(t) for t in ln.split()[1:]] for ln in lines if ln.startswith("vn ")], np.float64)
    fl = [ln.split()[1:] for ln in lines if ln.startswith("f ")]
    assert vl.shape == (len(v), 6) and nl.shape == (len(v), 3) and len(fl) == len(f)
    assert np.array_equal(vl[:, :3].astype(f32), v) and np.array_equal(nl.astype(f32), n)
    assert np.array_equal(vl[:, 3:].astype(f32), np.clip(c, 0, 1))
    idx = np.array([[[int(x) for x in t.split("//")] for t in row] for row in fl])
    assert np.array_equal(idx[..., 0], idx[..., 1]) and np.array_equal(idx[..., 0] - 1, f)
    # colours alone: `f a b c`
    MX.save_obj(tmp_path / "co.obj", v, f, colors=c)
    assert any(ln == "f %d %d %d" % tuple(f[0] + 1) for ln in (tmp_path / "co.obj").read_text().splitlines())


def _read_ply(path):
    """A small reader of binary little-endian PLY with float / uchar vertex properties and `list uchar int` faces."""
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").splitlines()
    assert head[0] == "ply" and head[1] == "format binary_little_endian 1.0"
    props, counts, elem = [], {}, None
    for ln in head[2:-1]:
        t = ln.split()
        if t[0] == "element":
            elem = t[1]
            counts[elem] = int(t[2])
        elif t[0] == "property" and elem == "vertex":
            props.append((t[2], {"float": "<f4", "uchar": "u1"}[t[1]]))
        elif t[0] == "property":
            assert t[1:] == ["list", "uchar", "int", "vertex_indices"]
    vdt = np.dtype(props)
    vert = np.frombuffer(data, vdt, counts["vertex"], end)
    fdt = np.dtype([("n", "u1"), ("i", "<i4", (3,))])
    face = np.frombuffer(data, fdt, counts["face"], end + vdt.itemsize * counts["vertex"])
    assert len(data) == end + vdt.itemsize * counts["vertex"] + fdt.itemsize * counts["face"]
    assert np.all(face["n"] == 3)
    return vert, face["i"]


def test_save_ply_mesh_parses_back(tmp_path):
    v, f, n, c = _mesh(1)
    MX.save_ply_mesh(tmp_path / "a.ply", torch.tensor(v), torch.tensor(f), normals=torch.tensor(n), colors=torch.tensor(c))
    vert, faces = _read_ply(tmp_path / "a.ply")
    assert vert.dtype.names == ("x", "y", "z", "nx", "ny", "nz", "red", "green", "blue")
    assert np.array_equal(np.stack([vert["x"], vert["y"], vert["z"]], 1), v)
    assert np.array_equal(np.stack([vert["nx"], vert["ny"], vert["nz"]], 1), n)
    want = (np.clip(c, f32(0), f32(1)) * f32(255)).astype(np.uint8)
    assert np.array_equal(np.stack([vert["red"], vert["green"], vert["blue"]], 1), want)
    assert want.max() == 255 and want.min() == 0
    assert np.array_equal(faces, f)
    MX.save_ply_mesh(tmp_path / "b.ply", v, f)
    vert, faces = _read_ply(tmp_path / "b.ply")
    assert vert.dtype.names == ("x", "y", "z") and np.array_equal(faces, f)


def test_argument_checks_without_a_device(tmp_path):
    v, f, n, c = _mesh(2)
    with pytest.raises(ValueError, match="normals"):
        MX.save_obj(tmp_path / "x.obj", v, f, normals=n[:-1])
    with pytest.raises(ValueError, match="colors"):
        MX.save_ply_mesh(tmp_path / "x.ply", v, f, colors=c[:, :2])
    with pytest.raises(ValueError, match="does not exist"):
        MX.save_ply_mesh(tmp_path / "x.ply", v, f + len(v))
    z = torch.zeros
    with pytest.raises(RuntimeError, match="CUDA device"):
        MX.query_field(z(4, 3), z(4, 3), z(4), z(4, 3), z(4, 4))
    with pytest.raises(RuntimeError, match="CUDA device"):
        MX.extract_colored_mesh(z(4, 3), z(4), z(4, 3), z(4, 4), z(4, 1, 3))
    g = GaussianParams(z(4, 3), z(4, 1, 3), z(4, 0, 3), z(4, 3), z(4, 4), z(4, 1), 0)
    with pytest.raises(ValueError, match="GaussianParams"):
        MX.query_field(z(2, 3), g, z(4))
    with pytest.raises(ValueError, match="GaussianParams"):
        MX.extract_colored_mesh(g, shs=z(4, 1, 3))
