"""The fused stem block (op 0 of the student, csrc/stem_block.cu) on its own, as the engine launches it: one CTA per SM
walking 8 x 16 output tiles, each CTA carrying its next tile's prefetched input window and its double-buffered expansion
chunks from tile to tile.  Grids capped at 1, 2, 5 and 7 SMs make every CTA walk one, a few or many tiles, an odd number
included; every stored output must equal the uncapped run bit for bit and pass op_report's float64 comparator.  The
student at 256, 192 and 320 (the input sizes stem_block_supported takes: H % 32 == W % 64 == 0), batches 1, 3 and 133,
crops with saturated borders so that the zero-padding masks of the border tiles matter, and the float32 input mode the
engine's host float32 forward uses, which must store exactly what the uint8 input mode stores for the same pixels."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
STUDENT = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "kps_student.onnx")

CAPS = [1, 2, 5, 7]
CASES = [(256, 1), (256, 3), (256, 133), (192, 3), (320, 3)]


def _bits(a):
    return a if a.dtype == np.uint8 else a.view(np.uint32)


def _crops(size, batch):
    import op_report as R
    import frames
    from oracle.host_ref import resize_linear_u8
    real = frames.crop_variants(1)[0]
    if size != 256:
        real = resize_linear_u8(real, size, size)
    x = R._with_noise(real, batch).copy()
    # saturated borders: stem(255) at the map edge differs most from the zero padding the next conv sees there
    x[-1, :8] = 255
    x[-1, -8:] = 255
    x[-1, :, :8] = 255
    x[-1, :, -8:] = 255
    return np.ascontiguousarray(x)


def _engine(size, batch, tmp_path):
    from peppa_pig_face_landmark_b200 import ONNXEngine, graph_tools
    path = STUDENT
    if size != 256:
        path = graph_tools.retarget_input_size(STUDENT, str(tmp_path / ("s%d.onnx" % size)), size)
    return ONNXEngine(path, max_batch=batch)


@pytest.mark.parametrize("size,batch", CASES, ids=["student@%d-b%d" % c for c in CASES])
def test_stem_block_capped_grids_bit_identical_and_within_bound(size, batch, tmp_path):
    import op_report as R
    from peppa_pig_face_landmark_b200 import plan as P
    from oracle.plan_interp import PlanInterp
    eng = _engine(size, batch, tmp_path)
    ex = R.EngineOps(eng, batch)
    i = [k for k, op in enumerate(eng.plan.ops) if op.type == P.OP_STEM_BLOCK]
    assert i == [0], i
    op = eng.plan.ops[0]
    kernel, info = ex.op_kernel(0)
    assert kernel == R.K_STEM, kernel
    x = _crops(size, batch)
    ex.forward(x)
    ins = {v.buf.idx: ex.read(v.buf.idx) for v in R._views_in(op)}
    stored = sorted({v.buf.idx for v in R._stored(op)})
    tiles = batch * (size // 32) * (size // 64)
    runs = {}
    try:
        for cap in [0] + CAPS:
            ex.set_num_sms(cap)
            ex.run_op(0)
            ctas, units = ex.op_grid(0)
            assert units == tiles and (cap == 0 or ctas == min(tiles, cap)), (cap, ctas, units)
            runs[cap] = {b: ex.read(b) for b in stored}
    finally:
        ex.set_num_sms(0)
    for cap in CAPS:
        for b in stored:
            assert np.array_equal(_bits(runs[cap][b].numpy()), _bits(runs[0][b].numpy())), (cap, b)
    ratio, where, _ = R.evaluate(op, kernel, info, PlanInterp(eng.plan), ins, runs[0], batch)
    print("student@%d batch %d: stem block worst err/bound %.3e at %s" % (size, batch, ratio, where))
    assert ratio <= 1.0, (ratio, where)


@pytest.mark.parametrize("size", [256, 320])
def test_stem_block_float32_input_matches_uint8(size, tmp_path):
    """ONNXEngine.__call__ feeds float32 pixels / 255 (the stem block's in_f32 mode); the uint8 mode divides through a
    table of i / 255 rounded the same way, so both modes store the same bits, under any grid cap."""
    from peppa_pig_face_landmark_b200 import plan as P, runtime as rt
    batch = 3
    eng = _engine(size, batch, tmp_path)
    lib = rt.load_library()
    op = [o for o in eng.plan.ops if o.type == P.OP_STEM_BLOCK][0]
    x = _crops(size, batch)
    x_f32 = np.ascontiguousarray(x.transpose(0, 3, 1, 2).astype(np.float32) / np.float32(255))
    eng.run_u8(x)
    ref = [_bits(eng.read_buffer(v.buf.idx, batch)).copy() for v in op.outs]
    try:
        for cap in [0] + CAPS:
            rt.check(lib.skps_engine_set_num_sms(eng.handle, cap))
            eng(x_f32)
            got = [_bits(eng.read_buffer(v.buf.idx, batch)) for v in op.outs]
            for a, b in zip(got, ref):
                assert np.array_equal(a, b), cap
    finally:
        rt.check(lib.skps_engine_set_num_sms(eng.handle, 0))
