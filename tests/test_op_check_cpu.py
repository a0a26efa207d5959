"""The op-isolated checker of tools/op_report.py without a GPU: the float32 PlanInterp stands in for the engine on the
detector lowered at 128x128 (batch 3).  Every op of the float32 interpreter must pass its float64 bound, and a one-element
error planted on a host copy of an output must fail; the float64 single-op step must agree with the float32 run."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))


@pytest.fixture(scope="module")
def checked():
    import op_report as R
    from peppa_pig_face_landmark_b200 import lowering
    from peppa_pig_face_landmark_b200.graph_tools import ensure_detector_onnx
    path = ensure_detector_onnx(os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "yolov5n-0.5.onnx"),
                                (128, 128))
    plan = lowering.lower(path, (128, 128))
    rng = np.random.default_rng(0)
    x = R._with_noise(rng.integers(0, 256, (128, 128, 3), dtype=np.uint8), 3)
    res, detail = R.check_ops(R.InterpOps(plan, 3), x, keep=lambda r: True)
    return plan, x, res, detail


def test_float32_interpreter_passes_every_bound(checked):
    import op_report as R
    _, _, res, _ = checked
    assert len(res) > 50
    bad = [str(r) for r in res if not r.ok]
    assert not bad, "\n".join(bad)
    classes = R.worst_per_class(res)
    assert {"tc", "simt", "dw", "xf", "exact", "det_decode"} <= set(classes), classes


@pytest.mark.parametrize("kind", ["tc", "dw", "xf", "exact", "det_decode"])
def test_planted_one_element_error_fails(checked, kind):
    import op_report as R
    _, _, res, detail = checked
    r = [r for r in res if r.cls == kind][-1]
    got, rows = detail[r.index]
    v = rows[0][0]
    ref, B = rows[0][1], rows[0][2]
    where = tuple(s - 1 for s in ref.shape[:3]) + (ref.shape[3] - 1,)
    planted = R.planted_ratio(r.op, got, rows, 0, where)
    if kind == "exact":
        # bit-exact ops have a zero bound: any change is infinitely far; plant one ulp of a non-zero element instead
        g = {k: R._to64(x, v.buf) for k, x in got.items()}
        nz = torch.nonzero(ref != 0)[0].tolist()
        g[v.buf.idx] = g[v.buf.idx].clone()
        g[v.buf.idx][nz[0], nz[1], nz[2], v.c_off + nz[3] * v.c_stride] *= 1 + 2.0 ** -23
        planted = R._worst([(v, ref, B)], g)[0]
    assert planted > 1.0, (kind, r.index, planted)


def test_float64_step_matches_float32_run(checked):
    """PlanInterp.step in float64 over the whole plan stays within float32 noise of run() (same semantics)."""
    from oracle.plan_interp import PlanInterp
    plan, x, _, _ = checked
    outs32 = PlanInterp(plan).run(x)
    interp = PlanInterp(plan)
    bufs = [torch.zeros(x.shape[0], b.H, b.W, b.C, dtype=torch.float64) for b in plan.bufs]
    bufs[plan.input.buf.idx] = torch.from_numpy(x).double() / 255.0
    for op in plan.ops:
        interp.step(op, bufs, torch.float64)
    v = plan.outputs[0]
    out64 = bufs[v.buf.idx].reshape(x.shape[0], v.buf.H, v.C).numpy()
    assert out64.dtype == np.float64
    np.testing.assert_allclose(outs32[0], out64, rtol=1e-4, atol=1e-3)
