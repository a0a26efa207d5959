"""conv_fpw's paired path (conv_fpw_pair in csrc/conv_fpw.cu): the student's two decoder up-sample layers, whose A tile the
transform warps build once for two 64-channel units that two MMA warpgroups multiply side by side.  Bit for bit what
conv_xf (skps_debug_conv_xf) computes, at a small batch and at the benchmark's batch of 256, with images past the batch
untouched; and through the engine, the launches it reports: one work item per pixel tile and pair of units."""
import os
import sys

import numpy as np
import pytest

from test_conv_fpw_gpu import SENTINEL, _call, _ids, _inputs

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
STUDENT = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "kps_student.onnx")
NONE, RELU = 0, 1

# mode, N, batch, H, W, Cx, Cl, Cout, x_split, dw_act, act, with_res, out_split: ops 53 (4 units: two pairs per tile) and
# 57 (2 units: one pair), each with the other output format too; N > batch leaves images past the batch
CASES = []
for batch in (3, 256):
    CASES += [
        (1, batch + 1, batch, 32, 32, 40, 256, 256, True, NONE, RELU, False, True),
        (1, batch + 2, batch, 64, 64, 24, 256, 128, True, NONE, RELU, False, False),
    ]
CASES += [
    (1, 4, 3, 32, 32, 40, 256, 256, True, NONE, NONE, False, False),
    (1, 4, 3, 64, 64, 24, 256, 128, True, NONE, NONE, False, True),
]


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_pair_layers_equal_conv_xf(case):
    from peppa_pig_face_landmark_b200 import runtime as rt
    mode, N, batch, H, W, Cx, Cl, Cout, x_split, dw_act, act, with_res, out_split = case
    lib = rt.load_library()
    d = _inputs(case)
    out = np.full((N, H, W, Cout), SENTINEL, np.float32)
    rt.check(_call(lib.skps_debug_conv_fpw, case, d, out, (batch,)))
    assert np.array_equal(out[batch:], np.full_like(out[batch:], SENTINEL))
    ref = np.full((N, H, W, Cout), np.nan, np.float32)
    rt.check(_call(lib.skps_debug_conv_xf, case, d, ref))
    assert np.array_equal(out[:batch].view(np.uint32), ref[:batch].view(np.uint32)), \
        int((out[:batch] != ref[:batch]).sum())


def test_engine_launches_one_item_per_tile_and_unit_pair():
    """Ops 53 and 57 launch batch x tiles x nsplit / 2 work items, the kernel report stays (128, 64, nsplit, XF_DW), and
    under a cap of 7 SMs some CTA walks an odd number of items, at least 3."""
    import ctypes as C
    import op_report as R
    from peppa_pig_face_landmark_b200 import ONNXEngine, runtime as rt
    lib = rt.load_library()
    B = 5
    eng = ONNXEngine(STUDENT, max_batch=B)
    info = (C.c_int32 * 4)()
    g = (C.c_int32 * 2)()
    try:
        for i, nsplit in ((53, 4), (57, 2)):
            assert lib.skps_engine_op_kernel(eng.handle, i, info) == R.K_FPW
            assert tuple(info) == (128, 64, nsplit, 1), (i, tuple(info))
            o = eng.plan.ops[i].outs[0].buf
            items = B * (o.H // 8) * (o.W // 16) * nsplit // 2
            rt.check(lib.skps_engine_op_grid(eng.handle, i, B, g))
            assert g[1] == items, (i, tuple(g), items)
            rt.check(lib.skps_engine_set_num_sms(eng.handle, 7))
            rt.check(lib.skps_engine_op_grid(eng.handle, i, B, g))
            per = R.units_per_cta(g[0], g[1])
            assert tuple(g) == (7, items) and any(n >= 3 and n % 2 for n in per), (i, tuple(g), per)
            rt.check(lib.skps_engine_set_num_sms(eng.handle, 0))
    finally:
        lib.skps_engine_set_num_sms(eng.handle, 0)
