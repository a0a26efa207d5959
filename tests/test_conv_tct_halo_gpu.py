"""The halo-row stages of the transposed convolution kernel (csrc/conv_tct.cu) through skps_debug_conv_tc2, element by
element against float64 within the tensor-core bound of tools/op_report.py.  One activation load feeds the three vertical
taps of a (kx, 32-channel half-chunk), so the cases cover what that load depends on: the row offset of a tap inside the
slot (dilation 1 and 2, maps 64, 32 and 16 pixels wide), channel counts that end in a partial half-chunk or a partial
64-channel chunk (96, 160, 72), a ring of two halo slots instead of three (W = 128), the first and last rows of an image,
whose halo rows are the TMA's out-of-bounds zeros, and more tiles than SMs, where both rings run on across tile boundaries.
Through the engine: the student's decoder conv runs on this kernel and leaves the images past the batch as they were."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

NONE, RELU, HSWISH = 0, 1, 2

CASES = [
    # N, H, W, Cin, Cout, k, dil, act
    (2, 64, 64, 128, 128, 3, 1, RELU),       # the student's decoder conv2: 6-row halo slots, three in the ring
    (2, 32, 32, 96, 128, 3, 2, NONE),        # dilation 2 at 32 x 32: 12-row slots, taps 2 rows apart, 3 half-chunks
    (3, 16, 16, 160, 128, 3, 2, RELU),       # 16-wide map: a tile is a whole image, every halo row of ky = 0 / 2 is padding
    (2, 32, 32, 160, 96, 3, 1, HSWISH),      # 5 half-chunks, Cout < 128
    (3, 8, 128, 72, 104, 3, 1, NONE),        # 4-row slots of 128 pixels: two in the ring; a last half-chunk of 8 channels
    (12, 64, 64, 128, 128, 3, 1, RELU),      # 192 tiles: more than the SMs, the rings wrap across tiles
]


def _ids(c):
    return "b%d %dx%d %d->%d k%d d%d act%d" % c


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_conv_tct_halo_stage_within_the_tensor_core_bound(case):
    import torch
    import torch.nn.functional as F
    import op_report as R
    from oracle.plan_interp import _act
    from peppa_pig_face_landmark_b200 import plan as P, runtime as rt
    N, H, W, Cin, Cout, k, dil, act = case
    lib = rt.load_library()
    rng = np.random.default_rng(Cin * 1000 + Cout + dil)
    x = (rng.standard_normal((N, H, W, Cin)) * 2).astype(np.float32)
    w = (rng.standard_normal((Cout, k, k, Cin)) / np.sqrt(k * k * Cin)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    n_tile, n_tiles = P.tc_tiling(Cout)
    hi, lo, out_scale = P.pack_tc_weights(w, n_tile, n_tiles)
    hi, lo = np.ascontiguousarray(hi), np.ascontiguousarray(lo)
    out = np.empty((N, H, W, Cout), np.float32)
    rt.check(lib.skps_debug_conv_tc2(x.ctypes.data, N, H, W, Cin, hi.ctypes.data, lo.ctypes.data, b.ctypes.data, Cout, k, dil,
                                     act, n_tile, n_tiles, out_scale, None, 1, out.ctypes.data, 1, 0, N))
    xt = torch.from_numpy(x).permute(0, 3, 1, 2).double()
    wt = torch.from_numpy(w).permute(0, 3, 1, 2).contiguous().double()
    bt = torch.from_numpy(b).double()
    pad = dil * (k - 1) // 2

    def nhwc(t):
        return t.permute(0, 2, 3, 1)

    z = nhwc(F.conv2d(xt, wt, bt, padding=pad, dilation=dil))
    mag = nhwc(F.conv2d(xt.abs(), wt.abs(), bt.abs(), padding=pad, dilation=dil))
    wsum = nhwc(F.conv2d(torch.ones_like(xt), wt.abs(), padding=pad, dilation=dil))
    E = R.tc_rel(k * k * Cin) * mag + R.TC_ABS * wsum
    y = _act(z, act)
    B = R.LIP[act] * E + R.act_eval(z, y, act) + R.SPLIT_REL * y.abs() + R.SPLIT_ABS
    ratio = R.ratio_of(torch.from_numpy(out).double(), y, B)
    print(_ids(case), "worst err/bound %.3e, first/last image rows %.3e" % (
        float(ratio.max()), float(torch.maximum(ratio[:, 0].max(), ratio[:, -1].max()))))
    assert float(ratio.max()) <= 1.0, float(ratio.max())


def test_student_decoder_conv_runs_on_conv_tct_and_leaves_images_past_the_batch():
    import ctypes as C
    import torch
    import frames
    import op_report as R
    from peppa_pig_face_landmark_b200 import ONNXEngine, plan as P, runtime as rt
    eng = ONNXEngine(os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "kps_student.onnx"), max_batch=4)
    lib = rt.load_library()
    info = (C.c_int32 * 4)()
    tct = [i for i in range(len(eng.plan.ops)) if lib.skps_engine_op_kernel(eng.handle, i, info) == R.K_TCT]
    dense = [i for i, op in enumerate(eng.plan.ops)
             if op.type == P.OP_CONV and tuple(op.k) == (3, 3) and op.d[0] == 1 and op.ins[0].C == 128 and op.outs[0].C == 128]
    assert tct == dense and len(tct) == 1, (tct, dense)
    assert lib.skps_engine_op_kernel(eng.handle, tct[0], info) == R.K_TCT and info[0] == 4     # 4 rows of 64 pixels
    buf = eng.plan.ops[tct[0]].outs[0].buf.idx
    x4 = torch.from_numpy(frames.noise_crops(4, seed=7)).cuda()
    eng.forward_device(x4)
    torch.cuda.synchronize()
    full = eng.read_buffer(buf, 4)
    x2 = torch.from_numpy(frames.noise_crops(2, seed=8)).cuda()
    eng.forward_device(x2)
    torch.cuda.synchronize()
    rt.check(lib.skps_engine_run_op(eng.handle, tct[0], 2, eng.stream.cuda_stream))
    torch.cuda.synchronize()
    after = eng.read_buffer(buf, 4)
    assert not np.array_equal(after[:2], full[:2])
    assert np.array_equal(after[2:], full[2:])
