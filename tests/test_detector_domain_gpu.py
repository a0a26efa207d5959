"""The detector over its whole input-size range (check_detector_input: multiples of 32 in 128..2176 x 128..3840), op by op
against float64 (tools/op_report.py).  The engine picks every op's kernel and tiling from its map shape, so which code runs
depends on the input size; the sizes checked here come from the range itself, not from a hand-picked list:

- the axis sample op_report.detector_domain_sample() (every value of each axis) must build an engine at every size, and
  each launch of each engine gets a signature (op_report.launch_signature: layer, kernel, tiling and where the map's
  border falls in the kernel's tile);
- a greedy set cover of those signatures and of the plan structures, cheapest sizes first, is checked op by op against
  float64 at batch 3 (a letterboxed real frame, uint8 noise and a near-uniform grey frame): every op within its bound,
  every signature and every plan structure of the sample checked;
- for every kernel whose tile hangs over some sampled map's border, the comparator must reject an error of 8x the bound
  planted in one border-tile element of a host copy of that kernel's output."""
import os
import sys
import time

import pytest

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

BATCH = 3


def _last_pixel_in_border_tile(R, kernel, info, o):
    """Whether the last pixel of the batch's last image lies in a tile that hangs over the border (a partial tile)."""
    return bool(R.edge_tile(kernel, info, o.H, o.W, o.H - 1, o.W - 1, BATCH - 1, BATCH))


@pytest.fixture(scope="module")
def sample(tmp_path_factory):
    """(directory of the retargeted files, {size: signatures of its launches} over the axis sample, the engine failures,
    the kernels whose tiles hang over the border of some sampled launch).  Each retargeted file is deleted once its
    engine is built: all of them would take 10 GB."""
    import op_report as R
    from peppa_pig_face_landmark_b200.core.api.onnx_model_base import ONNXEngine
    sizes = R.detector_domain_sample()
    t0 = time.time()
    d = str(tmp_path_factory.mktemp("det_domain"))
    t_engine = 0.0
    out, refused, ragged = {}, {}, set()
    for hw, path, structure in R.lower_detector_domain(sizes, d, keep=True):
        t1 = time.time()
        try:
            eng = R.EngineOps(ONNXEngine(path, max_batch=BATCH), BATCH)
        except RuntimeError as e:
            refused[hw] = str(e)
            continue
        finally:
            os.remove(path)
        assert R.plan_structure(eng.plan) == structure
        sigs = {("plan", structure)}
        for i, op in enumerate(eng.plan.ops):
            kernel, info = eng.op_kernel(i)
            o = op.outs[0]
            sigs.add(R.launch_signature(op, kernel, info, o.H, o.W, BATCH))
            if _last_pixel_in_border_tile(R, kernel, info, o):
                ragged.add(kernel)
        out[hw] = sigs
        del eng
        t_engine += time.time() - t1
    t = time.time() - t0
    print("\n%d sizes in %.1f s: retarget and lower on %d CPUs alongside engine creation and op kernels (%.1f ms per "
          "size)" % (len(sizes), t, os.cpu_count(), 1e3 * t_engine / len(sizes)))
    assert not os.listdir(d)
    return d, out, refused, ragged


def test_engine_builds_at_every_sampled_size(sample):
    _, out, refused, _ = sample
    sigs = set().union(*out.values())
    n_plans = sum(s[0] == "plan" for s in sigs)
    print("%d sizes built, %d launch signatures, %d plan structures" % (len(out), len(sigs) - n_plans, n_plans))
    assert not refused, "\n".join("%dx%d: %s" % (hw + (e,)) for hw, e in sorted(refused.items()))


def _keep_one_border_op(R, kept):
    """keep= for check_engine: the first op per kernel whose batch ends in a border tile (its tensors are kept for the
    planted-error test; one per kernel over the whole cover keeps host memory small)."""
    def keep(r):
        o = r.op.outs[0]
        if r.kernel in kept or r.op.flags & R.P.FLAG_HM_PART or not _last_pixel_in_border_tile(R, r.kernel, r.info, o):
            return False
        kept.add(r.kernel)
        return True
    return keep


@pytest.fixture(scope="module")
def checked(sample):
    """float64 op check of the detector at every size of the cover of the sample's signatures."""
    import op_report as R
    from peppa_pig_face_landmark_b200.core.api.onnx_model_base import ONNXEngine
    d, out, _, _ = sample
    cover = R.greedy_cover(out)
    print("\ncover: %d sizes" % len(cover))
    results, details, kept = {}, {}, set()
    keep = _keep_one_border_op(R, kept)
    t_all = time.time()
    for hw in cover:
        t0 = time.time()
        _, path, _ = R.retarget_and_lower((hw, d, True))
        try:
            eng = ONNXEngine(path, max_batch=BATCH)
        finally:
            os.remove(path)
        res, detail = R.check_engine(eng, R.detector_inputs(hw, BATCH), keep=keep)
        structure = R.plan_structure(eng.plan)
        del eng
        results[hw] = (structure, res)
        details.update({(hw, i): d for i, d in detail.items()})
        print("  %4dx%-4d %2d ops %3d signatures  worst err/bound %.3f  %.1f s" % (
            hw + (len(res), len(out[hw]), max(r.ratio for r in res), time.time() - t0)))
    print("cover checked in %.1f s" % (time.time() - t_all))
    return results, details


def test_every_signature_is_checked_in_float64_within_its_bound(sample, checked):
    import op_report as R
    _, out, _, _ = sample
    results, _ = checked
    worst, bad, seen = {}, [], set()
    for hw, (structure, res) in results.items():
        seen.add(("plan", structure))
        for r in res:
            o = r.op.outs[0]
            seen.add(R.launch_signature(r.op, r.kernel, r.info, o.H, o.W, BATCH))
            worst[r.cls] = max(worst.get(r.cls, 0.0), r.ratio)
            if not r.ok:
                bad.append("%dx%d %s kernel %s %s worst (n,y,x,c)=%s edge tile=%s ratio %.3e" % (
                    hw + (r.name, R.KERNELS[r.kernel], r.info, r.where, r.edge, r.ratio)))
    print("worst err/bound per kernel class:")
    for k, v in sorted(worst.items()):
        print("  %-18s %.3e" % (k, v))
    assert not bad, "\n".join(bad)
    sampled = set().union(*out.values())
    assert seen == sampled, "%d sampled signatures not checked, %d checked ones not sampled" % (
        len(sampled - seen), len(seen - sampled))


def test_checker_rejects_an_error_planted_in_each_kernels_border_tile(sample, checked):
    """On a host copy of what the kernel wrote: 8x the element's bound added to the last element of the batch (a border
    tile) of one op per kernel must fail the comparison; the unmodified copy passes."""
    import op_report as R
    ragged = sample[3]
    results, details = checked
    planted = {}
    for (hw, i), (got, rows) in sorted(details.items()):
        r = results[hw][1][i]
        o = rows[0][0]
        where = (BATCH - 1, o.H - 1, o.W - 1, o.C - 1)
        assert R.edge_tile(r.kernel, r.info, o.H, o.W, where[1], where[2], where[0], BATCH)
        clean = R._worst([rows[0][:3]], {k: R._to64(x, o.buf) if k == o.buf.idx else x for k, x in got.items()})[0]
        assert clean <= 1
        planted[r.kernel] = R.planted_ratio(r.op, got, rows, 0, where)
        print("%-7s %dx%d op %d %s map %dx%d: planted error reported at %.2f x the bound" % (
            R.KERNELS[r.kernel], hw[0], hw[1], i, r.info, o.H, o.W, planted[r.kernel]))
    assert set(planted) == ragged, (sorted(R.KERNELS[k] for k in planted), sorted(R.KERNELS[k] for k in ragged))
    assert all(v > 1.0 for v in planted.values()), planted
