"""GPU: the step bench.py times, as it runs it, against the CPU oracle -- every view of the 64-view raw packed step, its
backward-blend sums and the summed raw-parameter gradient.

The harness is bench.Harness itself (world size 1, the parser's default workload: 300 k Gaussians of sample.ply, SH degree 3,
the 64 seed-1000 orbit cameras at 1024^2, raw parameters), with the camera set built as run_b200 builds it.  The module
fixture runs the benchmark's sequence once -- warm-up and the steps before the timed region, a backward-blend state call,
the 8-view operating point, the 64-view step again, the per-view render() loops, the end-to-end host-buffer path and the
deterministic backward -- then the oracle over the 64 views and the 8 views (tests/bench_step_reference.py, activations
bit-identical to F1's).  Each test checks one stage:

  1. the 6th step (the harness's 6th call; calls >= 6 are the cached-buffer calls the benchmark times): all 64 views'
     colour, depth, alpha and radii bit for bit against the oracle, and byte-identical to the 1st step's;
  2. its packed gradient field by field against the summed, chained reference within the derived per-row bound T
     (bench_step_reference: every row within 4 T, at most 1e-4 of the rows over T); padding floats exactly zero;
  3. every (view, Gaussian) ScreenGrad record of forward_backward_with_state(raw=True) on the same inputs within
     test_gpu_parity's C u E bound, no exceptions;
  4. the roofline statistics n_vis and D as run_b200 reads them equal the oracle's totals;
  5. after the 8-view camera set (images and gradient against its own oracle run) the 64-view step is byte-identical again;
  6. the per-view render() loops: the fused loop's radii equal and its gradient meets FULL_SIZE against the batched step's;
     the getters' loop (torch activations) has radii equal wherever its activations are F1's bits, and its gradient is an
     expected failure (GETTER_BITS below);
  7. run_e2e's last loss equals, bit for bit, the loss of the resident step's images (its host gradient copy is not exposed
     and stays unchecked);
  8. under torch.use_deterministic_algorithms(True) the step meets the same reference and criterion, byte-identical twice.
Measured margins and the oracle's wall time are printed (run with -s)."""
import contextlib
import time

import numpy as np
import pytest
import torch

import bench_step_reference as BS
from test_gpu_fullsize import FULL_SIZE
from test_gpu_parity import SUMS_C, U, _check_sums
from util import grads_agree

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
IMAGES = ("color", "depth", "alpha")


@contextlib.contextmanager
def _deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


class _HostGrads:
    """the upstream images of a camera set, one view at a time on the host"""

    def __init__(self, gw):
        self.gw = gw

    def __getitem__(self, v):
        return tuple(g[v].cpu().numpy() for g in self.gw)


def _snap(h):
    """copies of what the latest batched step returned (h.last: images, radii, the packed gradient)"""
    return {k: t.detach().clone() for k, t in h.last.items()}


def _bytes(t):
    return t.contiguous().view(torch.int32)


def _same_bytes(a, b, keys=IMAGES):
    return all(torch.equal(_bytes(a[k]), _bytes(b[k])) for k in keys)


def _fields(h, grad):
    """the packed gradient as {field: [P, n] numpy}"""
    return {k: grad.narrow(0, o, n).view(shape).reshape(h.P, -1).cpu().numpy() for (o, n, shape), k in zip(h.fields, BS.FIELDS)}


def _padding(h, grad):
    """the floats of the packed buffer that belong to no field"""
    keep = torch.zeros(h.n_flat, dtype=torch.bool, device=grad.device)
    for o, n, _ in h.fields:
        keep[o:o + n] = True
    return grad[~keep]


def _view_vs_oracle(snap, v, ov):
    """names of the outputs of view v of a step that are not the oracle's bits"""
    bad = [k for k in IMAGES if not np.array_equal(snap[k][v].cpu().numpy().view(np.uint32), ov[k].view(np.uint32))]
    return bad + ([] if np.array_equal(snap["radii"][v].cpu().numpy(), ov["radii"]) else ["radii"])


def _sums_verdict(gpu, ov):
    """(worst |gpu - ref| / (C u E) of one view's ScreenGrad records, _check_sums's message or None)"""
    err = np.abs(gpu[:, :10].astype(np.float64) - ov["sums"])
    lim = SUMS_C * U * ov["sums_err"]
    worst = float(np.where(err == 0, 0.0, err / np.maximum(lim, 1e-300)).max(initial=0.0))
    try:
        _check_sums(gpu, ov)
        return worst, None
    except AssertionError as e:
        return worst, str(e)


def _oracle_pass(raw, act, h, cs, snap, sums=None):
    """the oracle over a camera set: per-view verdicts against the step `snap` (and the ScreenGrad records `sums`), and the
    summed reference with its bounds"""
    acc, views = BS.StepSum(h.P), []
    for v, ov in enumerate(BS.iter_views(act, cs["cams"], _HostGrads(cs["gw"]), h.deg, h.HW, h.HW)):
        acc.add(ov)
        views.append(dict(mismatch=_view_vs_oracle(snap, v, ov), num_rendered=ov["num_rendered"], visible=int((ov["radii"] > 0).sum()),
                          sums=None if sums is None else _sums_verdict(sums[v].cpu().numpy(), ov)))
    ref, bound = acc.result(act, raw)
    return views, ref, bound


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    import bench
    from humangaussian_b200 import rasterizer as R
    torch.cuda.set_device(DEV)
    R.load_library()
    args = BS.bench_args("--dump-outputs", str(tmp_path_factory.mktemp("dump")))  # so that h.last keeps each step's outputs
    h = bench.Harness(args, DEV, 0, 1)
    calls = []
    step = h.step_batched

    def counted(cs, allreduce=True):
        calls.append(cs["V"])
        return step(cs, allreduce)
    h.step_batched = counted
    mine = BS.bench_shard(args, h.all_cams)
    cs = h.camera_set([h.all_cams[i] for i in mine], seed=0)
    r = dict(h=h, cs=cs, calls=calls)

    # 1. the warm-up steps, the two before the timed region, and the first timed step: the harness's 6th call
    for i in range(max(args.warmup, 3) + 2 + 1):
        h.step_batched(cs)
        if i == 0:
            r["step1"] = _snap(h)
    r["step6"], r["step6_call"] = _snap(h), len(calls)
    # 4. the roofline statistics, read as run_b200 reads them after its timed steps
    r["n_vis"], r["D"] = int((h.stats["radii"] > 0).sum()), int(R.last_num_rendered())
    r["loss6"] = float((r["step6"]["color"] * cs["gw"][0]).sum() + (r["step6"]["depth"] * cs["gw"][1]).sum()
                       + (r["step6"]["alpha"] * cs["gw"][2]).sum())
    # 3. every ScreenGrad record of the same inputs and upstream images
    xyz, sc, rot, op, sh = [h.flat.detach().narrow(0, o, n).view(shape) for o, n, shape in h.fields]
    c, radii, d, a, state, sums = R.forward_backward_with_state(*cs["gw"], means3D=xyz, scales=sc, rotations=rot, opacities=op, shs=sh,
                                                            viewmatrix=cs["vm"], projmatrix=cs["pm"], campos=cs["cp"],
                                                            tanfovx=cs["tanx"], tanfovy=cs["tany"], image_height=h.HW,
                                                            image_width=h.HW, sh_degree=h.deg, bg=h.bg, raw=True)
    r["state_call_same"] = _same_bytes(dict(color=c, depth=d, alpha=a, radii=radii), r["step6"], IMAGES + ("radii",))
    r["sums"] = sums
    del c, d, a, radii, state
    # 5. the 8-view operating point (run_b200's views8), then the 64-view step again
    cs8 = h.camera_set(h.all_cams[:8], seed=8)
    for _ in range(3):
        h.step_batched(cs8)
    r["cs8"], r["views8"] = cs8, _snap(h)
    h.step_batched(cs)
    r["again"] = _snap(h)
    # 6. the per-view render() loops over the same cameras
    cs["dev_cams"] = bench._dev_cams(h, cs["cams"])
    for fused in (False, True):
        h.step_per_view(cs, fused=fused)
        r[f"per_view_fused_{fused}"] = (h.flat.grad.clone(), h.stats["radii"].clone())
    # 7. the end-to-end path with host buffers
    r["e2e"] = bench.run_e2e(h, cs, n_steps=2)
    # 8. the deterministic backward
    with _deterministic():
        r["det"] = []
        for _ in range(2):
            h.step_batched(cs)
            r["det"].append(_snap(h))
    torch.cuda.synchronize()

    # the oracle: the 64 views under the step's upstream images, the first 8 under the views8 set's
    raw = {k: h.flat.detach().narrow(0, o, n).view(shape).cpu().numpy() for (o, n, shape), k in zip(h.fields, BS.FIELDS)}
    act = BS.activate(raw, DEV)
    r["act"] = act
    # the activations of the per-view loop's getters (torch.exp / sigmoid / F.normalize on the device), bit for bit against F1's
    with torch.no_grad():
        pc = dict(scales=torch.exp(sc), opacities=torch.sigmoid(op), rotations=torch.nn.functional.normalize(rot))
    r["getter_rows_differ"] = {k: np.any(t.cpu().numpy().reshape(h.P, -1).view(np.uint32) != act[k].reshape(h.P, -1).view(np.uint32), 1)
                               for k, t in pc.items()}
    t0 = time.perf_counter()
    r["views"], r["ref"], r["bound"] = _oracle_pass(raw, act, h, cs, r["step6"], sums)
    r["views8_oracle"], r["ref8"], r["bound8"] = _oracle_pass(raw, act, h, cs8, r["views8"])
    r["oracle_s"] = time.perf_counter() - t0
    print(f"\n[bench step] oracle: {len(r['views']) + len(r['views8_oracle'])} views fwd+bwd in {r['oracle_s']:.1f} s")
    yield r
    h.step_batched = step
    r.clear()
    R.release_cached_buffers()
    torch.cuda.empty_cache()


def _check_grads(h, grad, ref, bound, what):
    stats, msg = BS.check_step_grads(_fields(h, grad), ref, bound)
    print(f"[bench step] {what}: worst |gpu - ref| / T per field (4 = the cap), rows over T: "
          + ", ".join(f"{k} {w:.3g} ({n})" for k, (w, n) in stats.items()))
    assert msg is None, f"{what}: {msg}"
    return stats


def test_sixth_step_images_are_the_oracles_and_the_first_steps(run):
    assert run["step6_call"] == 6 and run["calls"][:6] == [64] * 6, run["calls"]
    views = run["views"]
    assert len(views) == 64
    assert sum(v["num_rendered"] for v in views) > 10_000_000
    assert all(v["visible"] > 0 for v in views), "a view sees no Gaussian"
    bad = {v: m["mismatch"] for v, m in enumerate(views) if m["mismatch"]}
    assert not bad, f"views whose outputs are not the oracle's bits: {bad}"
    assert _same_bytes(run["step1"], run["step6"], IMAGES + ("radii",)), "the 6th step's images differ from the 1st step's"


def test_sixth_step_parameter_gradient_against_the_summed_reference(run):
    h, g = run["h"], run["step6"]["grad_params"]
    pad = _padding(h, g)
    print(f"[bench step] packed buffer: {h.n_flat} floats, {pad.numel()} of them padding")
    assert pad.numel() == 0 or float(pad.abs().max()) == 0.0, "padding between packed fields carries a gradient"
    assert all(float(np.abs(run["ref"][k]).max()) > 0 for k in BS.FIELDS)
    _check_grads(h, g, run["ref"], run["bound"], "64-view step 6 gradient")


def test_backward_blend_sums_of_every_view_and_gaussian(run):
    sums, views, h = run["sums"], run["views"], run["h"]
    assert tuple(sums.shape) == (64, h.P, 12) and sums.shape[0] * sums.shape[1] == 19_200_000
    assert run["state_call_same"], "forward_backward_with_state's images differ from the step's"
    worst = max(v["sums"][0] for v in views)
    print(f"[bench step] ScreenGrad sums: worst |gpu - ref| / (C u E) {worst:.3g} over 64 x {h.P} records")
    bad = {v: m["sums"][1] for v, m in enumerate(views) if m["sums"][1]}
    assert not bad, f"ScreenGrad records outside C u E in {len(bad)} views; first: view {min(bad)}: {bad[min(bad)]}"
    assert float(sums[:, :, :10].abs().max()) > 0


def test_roofline_statistics_are_the_oracles(run):
    views = run["views"]
    assert run["n_vis"] == sum(v["visible"] for v in views)
    assert run["D"] == sum(v["num_rendered"] for v in views)
    assert run["D"] > 10_000_000


def test_eight_view_set_then_the_64_view_step_again(run):
    assert run["calls"][6:10] == [8, 8, 8, 64], run["calls"]
    h, views8 = run["h"], run["views8_oracle"]
    assert len(views8) == 8 and all(v["visible"] > 0 for v in views8)
    bad = {v: m["mismatch"] for v, m in enumerate(views8) if m["mismatch"]}
    assert not bad, f"8-view set: views whose outputs are not the oracle's bits: {bad}"
    _check_grads(h, run["views8"]["grad_params"], run["ref8"], run["bound8"], "8-view step gradient")
    assert _same_bytes(run["again"], run["step6"], IMAGES + ("radii",)), "the 64-view step after the 8-view set differs from step 6"


@pytest.mark.parametrize("fused", [False, True])
def test_per_view_render_loop_radii_are_the_batched_steps(run, fused):
    h = run["h"]
    _, radii = run[f"per_view_fused_{fused}"]
    diff = (radii != run["step6"]["radii"]).any(0).cpu().numpy()
    rows = {k: int(m.sum()) for k, m in run["getter_rows_differ"].items()}
    print(f"[bench step] per-view loop (fused {fused}): {int(diff.sum())} Gaussians with a radius that differs in some view; "
          f"getter activations not F1's bits in {rows} rows")
    if fused:
        assert not diff.any(), "the fused per-view loop's radii differ from the batched step's"
    else:
        # F.normalize's norm is not evaluated in gs_normalize4's order (common.cuh), so the getters' quaternions may differ
        # from F1's in the last bit, and such a Gaussian's radius may round the other way; every other Gaussian's radii equal
        # the batched step's in every view
        same = ~run["getter_rows_differ"]["rotations"] & ~run["getter_rows_differ"]["scales"] & ~run["getter_rows_differ"]["opacities"]
        assert not (diff & same).any(), "per-view radii differ from the batched step's where the activations are F1's bits"
        assert diff.sum() <= 1e-4 * h.P, f"{int(diff.sum())} Gaussians' radii differ"


# The getters' loop renders quaternions that differ from F1's in the last bit (about one in six on this scene), so its images
# are not the batched step's bits: blend decisions at the 1/255 threshold flip, and on an H100 0.04 % of the dL/dxyz rows
# (worst 126x) leave FULL_SIZE, which assumes the same inputs summed in another order.  Strict: it fails as soon as the
# two activations agree and the loop meets the criterion.
GETTER_BITS = pytest.mark.xfail(strict=True, reason="torch's F.normalize and F1's gs_normalize4 differ in the last bit")


@pytest.mark.parametrize("fused", [pytest.param(False, marks=GETTER_BITS), True])
def test_per_view_render_loop_gradient_agrees_with_the_batched_step(run, fused):
    h = run["h"]
    grad, _ = run[f"per_view_fused_{fused}"]
    got, want = _fields(h, grad), _fields(h, run["step6"]["grad_params"])
    for k in BS.FIELDS:
        ok, msg = grads_agree(got[k], want[k], **FULL_SIZE)
        print(f"[bench step] per-view loop (fused {fused}) dL/d{k}: {msg}")
        assert ok, f"per-view loop (fused {fused}) dL/d{k} vs the batched step: {msg}"


def test_end_to_end_loss_is_the_resident_steps(run):
    e = run["e2e"]
    assert e["steps"] == 2 and e["last_loss"] is not None
    assert e["last_loss"] == run["loss6"], (e["last_loss"], run["loss6"])


def test_deterministic_step_against_the_reference_and_itself(run):
    h, (a, b) = run["h"], run["det"]
    assert run["calls"][10:] == [64, 64], run["calls"]
    assert _same_bytes(a, run["step6"], IMAGES + ("radii",)), "the deterministic step's images differ from step 6's"
    assert torch.equal(_bytes(a["grad_params"]), _bytes(b["grad_params"])), "two deterministic steps give different gradients"
    _check_grads(h, a["grad_params"], run["ref"], run["bound"], "deterministic 64-view step gradient")
