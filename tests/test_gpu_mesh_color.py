"""GPU: the field query (b200gs_field_query; mesh.query_field, mesh.extract_colored_mesh) against the field and the numpy
restatement (mesh_color_reference).

  1. grid-sample invariant: the density at every grid sample of the golden cases, and at a seeded 10^5-voxel subset of
     the full scene at 128^3, has the bits of b200gs_density_field's voxel;
  2. density, normals and colours against the float64 restatement at seeded random points and at marching-cubes
     vertices: golden cases and the full scene at degree 0, and seeded degree-3 SH on the 8 k sample;
  3. bit-identical results across runs and under a permutation of the points;
  4. extract_colored_mesh: extract_mesh's vertex and face bytes, vertex normals that agree with the triangle winding,
     a uniform-SH scene's colour at every vertex, and two differently coloured clusters;
  5. activated tensors, raw=True, a GaussianParams and packed-buffer views give the same bits;
  6. argument errors, in Python and at the C ABI.

Tolerance: |gpu - ref| <= K_TOL * sum|terms| + 1e-7 per output, with sum|terms| from the restatement: for the density
sum w (1 + P), P the sum of the magnitudes of the exponent's terms (a float32 exponent is off by a few ulp of P, which
for a thin Gaussian is far larger than |p|); for the gradient sum w (1 + P) |Sigma^-1 d| per component; for a colour
channel 0.5 + sum |basis_k| * mean |sh_k|.  Normals are compared by the distance of the unit vectors, bounded by
2 * K_TOL * |sum|terms|| / |G|, where |G| is at least 1e-3 of |sum|terms||.  Colours are compared along the GPU's own
normal, so a normal's error is not counted twice, and where D > 1e-6: far from every centre a float32 weight underflows
where the float64 one does not, and a point whose weights all underflow has D = 0 and colour 0.  K_TOL = 1e-5, the value first proposed; the H100 run (H100 80GB HBM3, 700 W) measured
the worst ratio of |gpu - ref| - 1e-7 to K_TOL * sum|terms| at 0.11 (density), 0.06 (normals) and 0.49 (colours).

Face orientation (test 4) was measured on the full scene at 128^3, iso 1: 92.2 % of the faces point the same way as the
mean of their three vertex normals, 93.4 % weighted by area.  Normals from the grid's central differences give 96.6 %,
so the rest is the surface of a 128^3 sampling of a field with finer detail, not the normals; the test asserts 90 % and
92 %.
"""
import numpy as np
import pytest
import torch

import mesh_color_reference as C
import mesh_reference as M
from humangaussian_b200 import mesh as MX
from humangaussian_b200 import rasterizer as R
from humangaussian_b200.scene import sample_ply_scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
K_TOL = 1e-5
f32 = np.float32


@pytest.fixture(scope="module")
def golden():
    return np.load(M.GOLDEN)


def _t(a):
    return torch.tensor(np.ascontiguousarray(a), dtype=torch.float32, device=DEV)


def _args(z, tag):
    res, nb, rr = z[f"{tag}_args"]
    return int(res), int(nb), float(rr)


def _kept(raw, res, nb):
    return MX._kept("test", *(_t(a) for a in raw[:4]), True, res, nb)[0]


def _query_norm(raw, q, res, nb, rr, shs=None, deg=0):
    """b200gs_field_query at normalised points q (torch [n,3]) for raw inputs (numpy)."""
    k = _kept(raw, res, nb)
    sk, K = (None, 0) if shs is None else (_t(shs)[k.keep].contiguous(), shs.shape[1])
    return MX._query(k, sk, K, deg, q.contiguous(), res, nb, rr)


@pytest.mark.parametrize("tag", ["a", "b", "c", "d"])
def test_density_at_every_grid_sample_is_the_field(golden, tag):
    res, nb, rr = _args(golden, tag)
    raw = M.golden_inputs(golden, tag)
    occ = MX.extract_fields(*(_t(a) for a in raw), raw=True, resolution=res, num_blocks=nb, relax_ratio=rr).occ
    lin = torch.linspace(-1, 1, res).to(DEV)
    q = torch.stack(torch.meshgrid(lin, lin, lin, indexing="ij"), -1).reshape(-1, 3)
    got = _query_norm(raw, q, res, nb, rr).density.reshape(res, res, res)
    assert occ.max() > 0.1 and torch.equal(got, occ)


def test_density_at_grid_samples_is_the_field_full_scene():
    p = sample_ply_scene().to(DEV)
    raw = (p.xyz, p.opacity, p.scaling, p.rotation)
    occ = MX.extract_fields(p, resolution=128).occ
    vox = torch.tensor(np.random.default_rng(0).integers(0, 128, (100000, 3)), device=DEV)
    lin = torch.linspace(-1, 1, 128).to(DEV)
    k = MX._kept("test", *raw, True, 128, 16)[0]
    got = MX._query(k, None, 0, 0, lin[vox].contiguous(), 128, 16, 1.5).density
    want = occ[vox[:, 0], vox[:, 1], vox[:, 2]]
    assert (want > 0).sum() > 1000 and torch.equal(got, want)


def _compare(Q, q, fq, what):
    """Ratios (|gpu - ref| - 1e-7) / (K_TOL * sum|terms|) of density, normals and colours; asserts each <= 1."""
    r = Q.eval(q)
    D = fq.density.double().cpu().numpy()
    dr = float(((np.abs(D - r["D"]) - 1e-7) / (K_TOL * r["D_abs"] + 1e-30)).max())
    nrm = fq.normals.double().cpu().numpy()
    Gn, Gabs = np.linalg.norm(r["G"], axis=1), np.linalg.norm(r["G_abs"], axis=1)
    ok = (Gn > 1e-3 * Gabs) & (r["D"] > 1e-6)
    nr = float(((np.linalg.norm(nrm - r["normal"], axis=1) - 1e-6) / (2 * K_TOL * Gabs / np.maximum(Gn, 1e-30)))[ok].max())
    assert np.all(nrm[r["D"] == 0] == 0) and np.allclose(np.linalg.norm(nrm[ok], axis=1), 1.0, atol=1e-6)
    cr = 0.0
    if fq.colors is not None:
        col, tabs = Q.colors(r, dirs=-nrm)
        got = fq.colors.double().cpu().numpy()
        dense = r["D"] > 1e-6  # far from every centre, float32 weights underflow where the float64 ones do not
        cr = float(((np.abs(got - col) - 1e-7) / (K_TOL * tabs))[dense].max())
        assert np.all(got[r["D"] == 0] == 0)
    print(f"{what}: {len(q)} points, {int(ok.sum())} with a well-conditioned normal; worst ratio density {dr:.3f}, "
          f"normals {nr:.3f}, colours {cr:.3f}")
    assert ok.sum() > len(q) // 10
    assert dr <= 1.0 and nr <= 1.0 and cr <= 1.0, (what, dr, nr, cr)


def _points_and_vertices(raw, res, nb, rr, n, seed):
    """Seeded points in the normalised box, and the marching-cubes vertices of the field at iso 0.2 * max (normalised)."""
    k = _kept(raw, res, nb)
    occ = MX._density_field(k.xyz, k.cov6, k.opac, res, nb, rr)
    v, _ = MX.marching_cubes(occ, float(occ.max()) * 0.2)
    rng = np.random.default_rng(seed)
    v = v[torch.tensor(rng.choice(len(v), min(n, len(v)), replace=False), device=DEV)]
    x = k.xyz.cpu().numpy()
    near = x[rng.integers(0, len(x), n - n // 2)] + rng.normal(0, 0.03, (n - n // 2, 3))
    pts = torch.tensor(np.concatenate([rng.uniform(-0.95, 0.95, (n // 2, 3)), near]).astype(f32), device=DEV)
    return pts, (v / (res - 1) * 2 - 1).contiguous()


@pytest.mark.parametrize("tag", ["a", "b", "c", "d"])
def test_query_matches_the_restatement_degree_0(golden, tag):
    res, nb, rr = _args(golden, tag)
    raw = M.golden_inputs(golden, tag)
    shs = np.random.default_rng(7).standard_normal((len(raw[0]), 1, 3)).astype(f32) * 0.5
    Q = C.Query(*raw, res, nb, rr, shs, 0)
    for name, q in zip(("random", "vertices"), _points_and_vertices(raw, res, nb, rr, 3000, 8)):
        _compare(Q, q.cpu().numpy(), _query_norm(raw, q, res, nb, rr, shs, 0), f"{tag} {name}")


def test_query_matches_the_restatement_degree_3_on_the_8k_sample(golden):
    res, nb, rr = _args(golden, "b")
    raw = M.golden_inputs(golden, "b")
    shs = np.random.default_rng(9).standard_normal((len(raw[0]), 16, 3)).astype(f32) * 0.3
    Q = C.Query(*raw, res, nb, rr, shs, 3)
    for name, q in zip(("random", "vertices"), _points_and_vertices(raw, res, nb, rr, 4000, 10)):
        _compare(Q, q.cpu().numpy(), _query_norm(raw, q, res, nb, rr, shs, 3), f"b deg 3 {name}")


def test_query_matches_the_restatement_full_scene():
    p = sample_ply_scene()
    raw = tuple(a.numpy() for a in (p.xyz, p.opacity, p.scaling, p.rotation))
    shs = p.features_dc.numpy()
    Q = C.Query(*raw, 128, 16, 1.5, shs, 0)
    for name, q in zip(("random", "vertices"), _points_and_vertices(raw, 128, 16, 1.5, 2000, 11)):
        _compare(Q, q.cpu().numpy(), _query_norm(raw, q, 128, 16, 1.5, shs, 0), f"full {name}")


def _near(xyz, n, seed):
    """n seeded world points near the Gaussian centres xyz."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    i = torch.randint(0, len(xyz), (n,), generator=g)
    return (xyz.cpu()[i] + torch.randn(n, 3, generator=g) * 0.02).to(DEV).contiguous(), g


def test_bit_identical_across_runs_and_under_permutation():
    p = sample_ply_scene(n=100000, sh_degree=3).to(DEV)
    pts, g = _near(p.xyz, 200000, 12)
    a = MX.query_field(pts, p, resolution=96)
    b = MX.query_field(pts, p, resolution=96)
    perm = torch.randperm(len(pts), generator=g).to(DEV)
    c = MX.query_field(pts[perm], p, resolution=96)
    assert (a.density > 0).sum() > 10000
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x[perm], z)


def test_extract_colored_mesh_full_scene():
    res = 128
    p = sample_ply_scene().to(DEV)
    m = MX.extract_mesh(p, resolution=res)
    cm = MX.extract_colored_mesh(p, resolution=res)
    assert torch.equal(cm.vertices, m.vertices) and torch.equal(cm.faces, m.faces)
    assert cm.normals.shape == cm.vertices.shape and cm.colors.shape == cm.vertices.shape
    v = cm.vertices.double().cpu().numpy()
    f = cm.faces.cpu().numpy().astype(np.int64)
    n = cm.normals.double().cpu().numpy()
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    k = MX._kept("test", p.xyz, p.opacity, p.scaling, p.rotation, True, res, 16)[0]
    vi = (cm.vertices.double() - k.center.double()) * k.scale  # normalised; the boundary is |x| near 1
    border = (vi.abs() > 1 - 2.5 / (res - 1)).any(1).cpu().numpy()
    inner = ~border[f].any(1)
    agree = (np.einsum("ij,ij->i", fn, n[f].mean(1)) > 0)[inner].mean()
    area = np.linalg.norm(fn, axis=1) * 0.5 * (k.scale * (res - 1) / 2) ** 2  # in grid cells^2
    big = inner & (area > 0.05)
    agree_big = (np.einsum("ij,ij->i", fn, n[f].mean(1)) > 0)[big].mean()
    wsum = (np.einsum("ij,ij->i", fn, n[f].mean(1)) > 0)[inner] @ area[inner] / area[inner].sum()
    # the same with normals from the grid: -central differences of the field, interpolated along each vertex's edge
    occ = MX.extract_fields(p, resolution=res).occ.double()
    gg = torch.zeros(res, res, res, 3, dtype=torch.float64, device=DEV)
    for a in range(3):
        gg[..., a] = torch.gradient(occ, dim=a)[0]
    vi_ = ((cm.vertices.double() - k.center.double()) * k.scale + 1) / 2 * (res - 1)
    i0 = vi_.floor().long().clamp(0, res - 2)
    t = vi_ - i0
    gv = torch.zeros_like(vi_)
    for corner in range(8):
        o = torch.tensor([(corner >> 0) & 1, (corner >> 1) & 1, (corner >> 2) & 1], device=DEV)
        wgt = torch.where(o.bool(), t, 1 - t).prod(1)
        ii = i0 + o
        gv += wgt[:, None] * gg[ii[:, 0], ii[:, 1], ii[:, 2]]
    gn = (-gv).cpu().numpy()
    agree_grid = (np.einsum("ij,ij->i", fn, gn[f].mean(1)) > 0)[inner].mean()
    print(f"full scene {res}^3: {len(f)} faces, {int(inner.sum())} away from the boundary; {agree:.5f} agree with the "
          f"mean of their vertex normals; {agree_big:.5f} of {int(big.sum())} faces over 0.05 cell^2; area-weighted {wsum:.5f}; "
          f"with grid-gradient normals {agree_grid:.5f}")
    assert agree >= 0.9 and wsum >= 0.92
    c = cm.colors.cpu().numpy()
    assert np.all(c >= 0) and np.isfinite(c).all()


def test_uniform_sh_colours_every_vertex():
    """Degree 0, and degree 3 seen view-independently: the DC colour within 1e-6.  Degree 3 along -normal: SH of the one
    coefficient set, within K_TOL * sum|terms| (S / D carries the rounding of two float32 sums)."""
    sh = np.random.default_rng(14).standard_normal((16, 3)) * 0.3
    dc = np.maximum(C.SH_C0 * sh[0].astype(f32).astype(np.float64) + 0.5, 0)[None]
    for deg, vd in ((0, True), (3, False), (3, True)):
        xyz, op, sc, rot, shs = C.synthetic(4000, 13, deg, sh=sh[:(deg + 1) ** 2])
        cm = MX.extract_colored_mesh(*(_t(a) for a in (xyz, op, sc, rot, shs)), raw=True, resolution=64, view_dependent=vd,
                                     density_thresh=0.5)
        assert len(cm.faces) > 1000
        got = cm.colors.double().cpu().numpy()
        if deg == 3 and vd:
            mean = np.broadcast_to(shs[0].astype(np.float64), (len(got), 16, 3))
            want, tabs = C.color(mean, 3, -cm.normals.double().cpu().numpy(), np.abs(mean))
            assert np.all(np.abs(got - want) <= K_TOL * tabs + 1e-7)
        else:
            assert np.abs(got - dc).max() <= 1e-6, (deg, vd)


def test_two_clusters_keep_their_colours():
    (xyz, op, sc, rot, shs), rgb = C.two_clusters(15)
    cm = MX.extract_colored_mesh(*(_t(a) for a in (xyz, op, sc, rot, shs)), raw=True, resolution=96, density_thresh=0.5)
    v, c = cm.vertices.cpu().numpy(), cm.colors.cpu().numpy()
    left = v[:, 0] < 0
    assert left.sum() > 500 and (~left).sum() > 500
    assert np.abs(c[left] - rgb[0]).max() <= 1e-5 and np.abs(c[~left] - rgb[1]).max() <= 1e-5


def test_input_forms_give_the_same_bits():
    p = sample_ply_scene(n=8192, sh_degree=3, seed=3).to(DEV)
    shs = torch.cat([p.features_dc, p.features_rest], 1)
    pts, _ = _near(p.xyz, 20000, 16)
    kw = dict(resolution=64, num_blocks=16)
    P = p.P
    fields, total = R.packed_layout(P, 16)
    flat = torch.zeros(total, dtype=torch.float32, device=DEV)
    xv, sv, rv, ov, hv = R._split_packed(flat, P, 16)
    xv.copy_(p.xyz); sv.copy_(p.scaling); rv.copy_(p.rotation); ov.copy_(p.opacity); hv.copy_(shs)
    forms = {
        "activated": MX.query_field(pts, p.xyz, torch.sigmoid(p.opacity), torch.exp(p.scaling), p.rotation, shs, **kw),
        "raw": MX.query_field(pts, p.xyz, p.opacity, p.scaling, p.rotation, shs, raw=True, **kw),
        "params": MX.query_field(pts, p, **kw),
        "packed": MX.query_field(pts, xv, ov, sv, rv, hv, raw=True, **kw),
    }
    ref = forms["raw"]
    assert (ref.density > 0).sum() > 1000
    for name, fq in forms.items():
        for x, y in zip(fq, ref):
            assert torch.equal(x, y), name
    meshes = [MX.extract_colored_mesh(p, density_thresh=0.05, **kw),
              MX.extract_colored_mesh(xv, ov, sv, rv, hv, raw=True, density_thresh=0.05, **kw)]
    assert len(meshes[0].faces) > 100
    for x, y in zip(*meshes):
        assert torch.equal(x, y)


def test_argument_errors():
    xyz, op, sc, rot, shs = (_t(a) for a in C.synthetic(500, 17, 1))
    pts = xyz[:10].clone()
    with pytest.raises(ValueError, match="not finite"):
        bad = pts.clone()
        bad[2, 0] = float("inf")
        MX.query_field(bad, xyz, op, sc, rot, shs, raw=True)
    with pytest.raises(ValueError, match="sh_degree"):
        MX.query_field(pts, xyz, op, sc, rot, shs, raw=True, sh_degree=2)  # 4 coefficients hold degree 1
    with pytest.raises(ValueError, match="sh_degree"):
        MX.query_field(pts, xyz, op, sc, rot, raw=True, sh_degree=1)
    with pytest.raises(ValueError, match="wrong shape"):
        MX.query_field(pts, xyz, op, sc, rot, shs[:-1], raw=True)
    with pytest.raises(ValueError, match="wrong shape"):
        MX.query_field(pts[:, :2], xyz, op, sc, rot, raw=True)
    with pytest.raises(ValueError, match="block size"):
        MX.extract_colored_mesh(xyz, op, sc, rot, shs, raw=True, resolution=128, num_blocks=3)
    fq = MX.query_field(pts[:0], xyz, op, sc, rot, shs, raw=True)
    assert fq.density.shape == (0,) and fq.colors.shape == (0, 3)
    fq = MX.query_field(pts, xyz, op, sc, rot, raw=True)
    assert fq.colors is None and (fq.density > 0).all()
    # the C ABI
    L = R.load_library()
    k = _kept([a.cpu().numpy() for a in (xyz, op, sc, rot)], 32, 8)
    lin = torch.linspace(-1, 1, 32).to(DEV)
    out = torch.zeros(10, 3, device=DEV)
    n = k.xyz.shape[0]
    scratch = torch.empty(L.b200gs_field_query_scratch_bytes(n, 10, 32, 8, 1), dtype=torch.uint8, device=DEV)
    call = lambda shs_p, K, deg, colors, nb=8, P=n, sb=scratch.numel(): L.b200gs_field_query(
        P, R._ptr(k.xyz), R._ptr(k.cov6), R._ptr(k.opac), shs_p, K, deg, 32, nb, R._ptr(lin), 0.1875, 10, R._ptr(pts),
        None, None, colors, R._ptr(scratch), sb, R._stream(DEV))
    sk = shs[k.keep].contiguous()
    assert call(None, 0, 0, R._ptr(out)) == R.E_ARGS            # colours without SH
    assert call(R._ptr(sk), 3, 1, R._ptr(out)) == R.E_ARGS       # 3 < (1+1)^2 coefficients
    assert call(R._ptr(sk), 4, 4, R._ptr(out)) == R.E_ARGS       # degree 4
    assert call(R._ptr(sk), 4, 1, R._ptr(out), nb=0) == R.E_ARGS
    assert call(R._ptr(sk), 4, 1, R._ptr(out), nb=64) == R.E_RANGE  # 32 / 64 < 1 sample per block
    assert call(R._ptr(sk), 4, 1, R._ptr(out), P=-1) == R.E_ARGS
    assert call(R._ptr(sk), 4, 1, R._ptr(out), sb=16) == R.E_BUFFER
    assert call(R._ptr(sk), 4, 1, R._ptr(out)) == R.OK
    torch.cuda.synchronize()
    assert (out > 0).any()
    assert L.b200gs_field_query_scratch_bytes(n, 10, 32, 8, 4) == 0 and L.b200gs_field_query_scratch_bytes(n, -1, 32, 8, 0) == 0
