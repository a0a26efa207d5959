"""The pointwise wgmma kernel (csrc/conv_pw.cu) through skps_debug_conv_pw, element by element against float64 within the
tensor-core bound of tools/op_report.py: the student's 1x1 layer shapes, partial last pixel tiles, channel windows of wider
buffers, both output formats and all three activations.  Every element the conv must not write (other channels, images
past the batch) has to come back exactly as it went in.  And the engine must route the student's 1x1 stride-1 layers to
this kernel and leave the dilated ASPP convs on conv_tc."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

SENTINEL = 1234.5              # exact in split-fp16 (hi 1234, lo 0.5), so untouched elements come back bit for bit
NONE, RELU, HSWISH = 0, 1, 2

CASES = [
    # batch, max_batch, H, W, Cin, Cout, act, out_split, (in_ld, in_coff), (out_ld, out_coff)
    # the student's layers (ops 1 ... 52 of the batch-256 plan) at batch 2
    (2, 2, 64, 64, 64, 24, NONE, True, None, None),
    (2, 2, 64, 64, 24, 72, RELU, False, None, None),
    (2, 2, 32, 32, 40, 120, RELU, False, None, None),
    (2, 2, 32, 32, 40, 240, HSWISH, False, None, None),
    (2, 2, 16, 16, 240, 80, NONE, True, None, None),
    (2, 2, 16, 16, 80, 200, HSWISH, False, None, None),
    (2, 2, 16, 16, 80, 184, HSWISH, False, None, None),
    (2, 2, 16, 16, 80, 480, HSWISH, False, None, None),
    (2, 2, 16, 16, 112, 672, HSWISH, False, None, None),
    (2, 2, 16, 16, 160, 960, HSWISH, False, None, None),
    (2, 2, 16, 16, 160, 64, RELU, True, None, (256, 192)),          # into the 256-channel concat
    (2, 2, 16, 16, 256, 256, RELU, False, None, None),
    # partial last tile (720 and 70 pixels), images past the batch left alone
    (3, 5, 12, 20, 80, 48, NONE, False, None, None),
    (3, 5, 12, 20, 40, 200, HSWISH, True, None, None),
    (2, 3, 5, 7, 24, 72, RELU, True, None, None),
    (1, 2, 5, 7, 112, 672, NONE, False, None, None),
    # channel windows of wider buffers on both sides
    (2, 3, 12, 20, 40, 120, HSWISH, False, (64, 16), (136, 8)),
    (2, 2, 16, 16, 80, 184, RELU, True, (96, 8), (200, 16)),
    (3, 4, 5, 7, 160, 960, NONE, True, (176, 16), (1000, 24)),
    # more units than SMs: every CTA walks several units, so both consumer warpgroups take work and every ring wraps
    (150, 150, 16, 16, 80, 184, HSWISH, False, None, None),         # 300 tiles x 2 chunks
    # ... with the partial last tile (188 tiles, the last one 64 pixels) on a CTA's second unit, that is on warpgroup 1
    # on 132 SMs, and channel windows on both sides
    (100, 101, 12, 20, 40, 120, HSWISH, True, (64, 16), (136, 8)),
]


def _ids(c):
    b, mb, H, W, Cin, Cout, act, split, inv, outv = c
    return "b%d of %d %dx%d %d->%d act%d %s%s%s" % (b, mb, H, W, Cin, Cout, act, "split" if split else "f32",
                                                    " in%s" % (inv,) if inv else "", " out%s" % (outv,) if outv else "")


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_conv_pw_matches_fp64_within_the_tc_bound(case):
    import torch
    import op_report as R
    from oracle.plan_interp import _act
    from peppa_pig_face_landmark_b200 import plan as P, runtime as rt
    batch, max_batch, H, W, Cin, Cout, act, split, inv, outv = case
    in_ld, in_coff = inv or (Cin, 0)
    out_ld, out_coff = outv or (Cout, 0)
    lib = rt.load_library()
    rng = np.random.default_rng(Cin * 1000 + Cout)
    x = (rng.standard_normal((max_batch, H, W, in_ld)) * 2).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin)) / np.sqrt(Cin)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    n_tile, n_tiles = P.tc_tiling(Cout)
    hi, lo, out_scale = P.pack_tc_weights(w.reshape(Cout, 1, 1, Cin), n_tile, n_tiles)
    hi, lo = np.ascontiguousarray(hi), np.ascontiguousarray(lo)
    out = np.full((max_batch, H, W, out_ld), SENTINEL, np.float32)
    rt.check(lib.skps_debug_conv_pw(x.ctypes.data, batch, max_batch, H, W, Cin, in_ld, in_coff, hi.ctypes.data,
                                    lo.ctypes.data, b.ctypes.data, Cout, act, n_tile, n_tiles, out_scale, 1 if split else 0,
                                    out_ld, out_coff, out.ctypes.data))
    xs = torch.from_numpy(x[:batch, :, :, in_coff:in_coff + Cin].reshape(-1, Cin)).double()
    wt, bt = torch.from_numpy(w).double(), torch.from_numpy(b).double()
    z = xs @ wt.T + bt
    mag = xs.abs() @ wt.abs().T + bt.abs()
    E = R.tc_rel(Cin) * mag + R.TC_ABS * wt.abs().sum(1)
    y = _act(z, act)
    B = R.LIP[act] * E + R.act_eval(z, y, act)
    if split:
        B = B + R.SPLIT_REL * y.abs() + R.SPLIT_ABS
    got = torch.from_numpy(out[:batch, :, :, out_coff:out_coff + Cout].reshape(-1, Cout)).double()
    ratio = float(R.ratio_of(got, y, B).max())
    print(_ids(case), "worst err/bound %.3e" % ratio)
    assert ratio <= 1.0, ratio
    # nothing outside the conv's window may change: other channels, and every pixel of the images past the batch
    keep = np.ones(out.shape, bool)
    keep[:batch, :, :, out_coff:out_coff + Cout] = False
    assert np.array_equal(out[keep], np.full(int(keep.sum()), SENTINEL, np.float32))


def test_engine_routes_the_student_pointwise_layers_to_conv_pw():
    import ctypes as C
    import bench_pw
    import op_report as R
    from peppa_pig_face_landmark_b200 import ONNXEngine, runtime as rt
    eng = ONNXEngine(os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "kps_student.onnx"), max_batch=3)
    lib = rt.load_library()
    info = (C.c_int32 * 4)()
    kinds = {}
    for i in range(len(eng.plan.ops)):
        kinds[i] = (lib.skps_engine_op_kernel(eng.handle, i, info), tuple(info))
    pw = sorted(i for i, (k, _) in kinds.items() if k == R.K_PW)
    expected = bench_pw.pointwise_ops(eng.plan)
    assert len(expected) == 17, expected
    assert pw == expected, (pw, expected)
    for i in pw:
        nc, chunks = kinds[i][1][:2]
        assert nc in (32, 64, 96, 128) and chunks * nc >= eng.plan.ops[i].outs[0].C, (i, kinds[i])
    assert kinds[46][0] == R.K_TC and kinds[47][0] == R.K_TC, (kinds[46], kinds[47])
