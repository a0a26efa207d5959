"""The register-accumulator fused kernel (csrc/conv_fpw.cu) through skps_debug_conv_fpw: every student layer shape of the
depthwise -> 1x1 and squeeze-excite -> 1x1 layers, against float64 within the tensor-core bound of tools/op_report.py and
bit for bit against conv_xf (skps_debug_conv_xf) on the same inputs.  Images past the batch must come back as they went
in.  And the engine must route exactly the student's 14 fused layers to it and leave every detector DWPW layer on
conv_xf."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

SENTINEL = 1234.5              # exact in split-fp16, so untouched elements come back bit for bit
NONE, RELU, HSWISH = 0, 1, 2

# mode, N, batch, H, W, Cx, Cl, Cout, x_split, dw_act, act, with_res, out_split
CASES = [
    # squeeze-excite scale ahead of conv_pwl (ops 7, 11/15, 28, 32, 36, 40/44)
    (0, 3, 2, 32, 32, 72, 0, 40, True, NONE, NONE, False, True),
    (0, 3, 3, 32, 32, 120, 0, 40, True, NONE, NONE, True, True),
    (0, 2, 2, 16, 16, 480, 0, 112, True, NONE, NONE, False, False),
    (0, 2, 2, 16, 16, 672, 0, 112, True, NONE, NONE, True, True),
    (0, 2, 1, 16, 16, 672, 0, 160, True, NONE, NONE, False, True),
    (0, 3, 3, 16, 16, 960, 0, 160, True, NONE, RELU, True, False),
    # depthwise 3x3 ahead of conv_pwl (ops 3, 20, 22/24): float32 and split-fp16 x
    (1, 2, 2, 64, 64, 72, 0, 24, False, RELU, NONE, True, True),
    (1, 3, 2, 16, 16, 200, 0, 80, False, HSWISH, NONE, True, True),
    (1, 2, 2, 16, 16, 184, 0, 80, True, HSWISH, RELU, False, False),
    # bilinear x2 -> concat -> depthwise -> 1x1 (ops 53, 57)
    (1, 3, 2, 32, 32, 40, 256, 256, True, NONE, RELU, False, True),
    (1, 2, 2, 64, 64, 24, 256, 128, True, NONE, RELU, False, False),
    # more tiles than SMs: the persistent loop wraps every ring
    (1, 150, 150, 16, 16, 184, 0, 80, False, HSWISH, NONE, True, True),
    (0, 150, 149, 16, 16, 480, 0, 112, True, NONE, NONE, False, True),
]


def _ids(c):
    mode, N, b, H, W, Cx, Cl, Cout, xs, da, act, res, os_ = c
    return "%s b%d of %d %dx%d %d%s->%d%s act%d%s %s" % ("scale" if mode == 0 else "dw", b, N, H, W, Cx,
                                                     "+up%d" % Cl if Cl else "", Cout, " x16" if xs else "", act,
                                                     " res" if res else "", "split" if os_ else "f32")


def _inputs(case, seed=0):
    from peppa_pig_face_landmark_b200 import plan as P
    mode, N, batch, H, W, Cx, Cl, Cout, x_split, dw_act, act, with_res, out_split = case
    rng = np.random.default_rng(seed + Cx * 7 + Cout)
    K = Cx + Cl
    kpad = -(-K // 64) * 64
    d = {}
    d["x"] = (rng.standard_normal((N, H, W, Cx)) * 2).astype(np.float32)
    d["low"] = (rng.standard_normal((N, H // 2, W // 2, Cl)) * 2).astype(np.float32) if Cl else None
    d["gate"] = rng.uniform(0, 1, (N, Cx)).astype(np.float32) if mode == 0 else None
    dw_w = (rng.standard_normal((9, K)) / 3).astype(np.float32)
    dw_b = rng.standard_normal(K).astype(np.float32)
    dww = np.zeros((10, kpad), np.float32)
    dww[:9, :K], dww[9, :K] = dw_w, dw_b
    d["dw_w"], d["dw_b"], d["dww"] = dw_w, dw_b, dww
    d["w"] = (rng.standard_normal((Cout, 1, 1, K)) / np.sqrt(K)).astype(np.float32)
    d["b"] = rng.standard_normal(Cout).astype(np.float32)
    d["res"] = rng.standard_normal((N, H, W, Cout)).astype(np.float32) if with_res else None
    n_tile, n_tiles = P.tc_tiling(Cout)
    assert n_tiles == 1
    hi, lo, out_scale = P.pack_tc_weights(d["w"], n_tile, n_tiles)
    d["hi"], d["lo"], d["out_scale"], d["n_tile"] = np.ascontiguousarray(hi), np.ascontiguousarray(lo), out_scale, n_tile
    d["weff"] = P.pack_upcat_class_weights(dw_w[:, :Cl]) if Cl else None
    return d


def _call(fn, case, d, out, extra=()):
    mode, N, batch, H, W, Cx, Cl, Cout, x_split, dw_act, act, with_res, out_split = case
    ptr = lambda a: a.ctypes.data if a is not None else None
    return fn(mode, ptr(d["x"]), N, H, W, Cx, 1 if x_split else 0, ptr(d["low"]), Cl, ptr(d["gate"]), ptr(d["dww"]), dw_act,
              ptr(d["hi"]), ptr(d["lo"]), ptr(d["b"]), Cout, act, d["n_tile"], d["out_scale"], ptr(d["res"]), 0,
              1 if out_split else 0, ptr(out), ptr(d["weff"]), *extra)


def _reference(case, d):
    """float64 result and its tensor-core error bound for images [0, batch)."""
    import torch
    import torch.nn.functional as F
    import op_report as R
    from oracle.plan_interp import _act
    mode, N, batch, H, W, Cx, Cl, Cout, x_split, dw_act, act, with_res, out_split = case
    x = torch.from_numpy(d["x"][:batch]).double().permute(0, 3, 1, 2)
    if x_split or mode == 0:            # the kernel reads x through split-fp16 planes
        x = torch.from_numpy(_split_round(d["x"][:batch])).double().permute(0, 3, 1, 2)
    if mode == 0:
        a = x * torch.from_numpy(d["gate"][:batch]).double()[:, :, None, None]
    else:
        if Cl:
            low = torch.from_numpy(d["low"][:batch]).double().permute(0, 3, 1, 2)
            up = F.interpolate(low, scale_factor=2, mode="bilinear", align_corners=False)
            x = torch.cat([up, x], 1)
        K = Cx + Cl
        wd = torch.from_numpy(d["dw_w"]).double().T.reshape(K, 1, 3, 3).contiguous()
        a = _act(F.conv2d(x, wd, torch.from_numpy(d["dw_b"]).double(), padding=1, groups=K), dw_act)
    a = a.permute(0, 2, 3, 1).reshape(-1, Cx + Cl)
    wt = torch.from_numpy(d["w"]).double().reshape(Cout, -1)
    bt = torch.from_numpy(d["b"]).double()
    z = a @ wt.T + bt
    mag = a.abs() @ wt.abs().T + bt.abs()
    K = Cx + Cl
    E = R.tc_rel(K) * mag + R.TC_ABS * wt.abs().sum(1)
    y = _act(z, act)
    B = R.LIP[act] * E + R.act_eval(z, y, act)
    if with_res:
        y = y + torch.from_numpy(d["res"][:batch]).double().reshape(-1, Cout)
    # the A operand itself is rounded to split fp16 (2^-22 relative) after the depthwise / scale stage
    B = B + 2.0 ** -21 * (a.abs() @ wt.abs().T)
    if out_split:
        B = B + R.SPLIT_REL * y.abs() + R.SPLIT_ABS
    return y, B


def _split_round(v):
    hi = v.astype(np.float16).astype(np.float32)
    lo = (v - hi).astype(np.float16).astype(np.float32)
    return (hi.astype(np.float64) + lo).astype(np.float64)


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_conv_fpw_matches_fp64_and_conv_xf(case):
    import torch
    import op_report as R
    from peppa_pig_face_landmark_b200 import runtime as rt
    mode, N, batch, H, W, Cx, Cl, Cout, x_split, dw_act, act, with_res, out_split = case
    lib = rt.load_library()
    d = _inputs(case)
    out = np.full((N, H, W, Cout), SENTINEL, np.float32)
    rt.check(_call(lib.skps_debug_conv_fpw, case, d, out, (batch,)))
    y, B = _reference(case, d)
    got = torch.from_numpy(out[:batch].reshape(-1, Cout)).double()
    ratio = float(R.ratio_of(got, y, B).max())
    print(_ids(case), "worst err/bound %.3e" % ratio)
    assert ratio <= 1.0, ratio
    # images past the batch come back as they went in
    assert np.array_equal(out[batch:], np.full_like(out[batch:], SENTINEL))
    # bit for bit what conv_xf computes on the same inputs (it runs all N images)
    ref = np.full((N, H, W, Cout), np.nan, np.float32)
    rt.check(_call(lib.skps_debug_conv_xf, case, d, ref))
    assert np.array_equal(out[:batch].view(np.uint32), ref[:batch].view(np.uint32)), \
        int((out[:batch] != ref[:batch]).sum())


def _fused_ops(plan):
    from peppa_pig_face_landmark_b200 import plan as P
    return [i for i, op in enumerate(plan.ops)
            if op.type == P.OP_DWPW or (op.type == P.OP_CONV and op.flags & P.FLAG_XF)]


def test_engine_routes_the_student_fused_layers_to_conv_fpw():
    import ctypes as C
    import op_report as R
    from peppa_pig_face_landmark_b200 import ONNXEngine, runtime as rt
    lib = rt.load_library()
    info = (C.c_int32 * 4)()
    eng = ONNXEngine(os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "kps_student.onnx"), max_batch=3)
    fused = _fused_ops(eng.plan)
    assert fused == [3, 7, 11, 15, 20, 22, 24, 28, 32, 36, 40, 44, 53, 57], fused
    for i in fused:
        k = lib.skps_engine_op_kernel(eng.handle, i, info)
        assert k == R.K_FPW, (i, k)
        pix, n, units, mode = tuple(info)
        n_tile = eng.plan.ops[i].ints[0]
        assert pix == 128 and n <= 64 and n * (units - 1) < n_tile <= n * units, (i, tuple(info))


def test_engine_keeps_the_detector_dwpw_layers_on_conv_xf():
    import ctypes as C
    import op_report as R
    from peppa_pig_face_landmark_b200 import ONNXEngine, runtime as rt
    lib = rt.load_library()
    info = (C.c_int32 * 4)()
    eng = ONNXEngine(os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "yolov5n-0.5.onnx"), max_batch=2)
    fused = _fused_ops(eng.plan)
    assert len(fused) >= 13, fused
    kinds = [lib.skps_engine_op_kernel(eng.handle, i, info) for i in fused]
    assert all(k == R.K_XF for k in kinds), list(zip(fused, kinds))
