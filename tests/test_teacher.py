"""Teacher (HRNet-w18 + Decoder, model.py:302-345; SURVEY 8a row a12 / benchmark config 4).

The reference ships no teacher weights and timm is absent, so parity for this row is UNPINNED by the reference:
what is pinned is the architecture (parameter count = README's 11.53 "M" = 12 085 570; conv MACs within the
thop figure) and, for the numbers, our CUDA path against the oracle's fp64 execution of the same generated
.onnx file.  Tolerances are wider than the student's 1e-3 px because the synthetic random-weight network
amplifies fp32 ordering noise: the oracle's own fp32 run differs from its fp64 run by ~1.5e-3 px / 4e-4 score
(measured below), so the bar is 1e-2 px / 5e-3 score against fp64 for fp32 execution, and 6e-2 px / 2e-2 score for
the tensor-core path (see TOL_PX_TC).
"""
import os

import numpy as np
import pytest

TOL_PX, TOL_SCORE = 1e-2, 5e-3            # fp32 execution (plan interpreter, CUDA-core kernels) vs the fp64 oracle
# tensor-core path (fp16 hi/lo split, fp32 tensor-core accumulation): each conv is within 1e-5 relative of fp32
# (tests/test_conv_tc_gpu.py, HRNet shapes included); through this random-weight network that per-layer noise is
# amplified to the order of 2.5e-2 px / 7e-3 score, against 9e-5 px for the trained student.
# Where the gap to the fp32 path (2e-3 px) comes from: NOT the operand format - tools/split_error.py executes the same plan
# on the CPU with every tensor-core conv's operands rounded to the stored fp16 hi/lo planes and exact accumulation and lands
# at 1.6e-3 px (fp32 execution: 3.6e-3 px) - but the tensor core's fp32 accumulation: each 16-term product block is added
# into the accumulator with its own rounding, and the three-product scheme makes 3*K/16 adds per output (216 at K = 1152,
# bounded per conv by test_conv_tc_matches_fp32); 100 layers of random weights amplify that to a few 1e-2 px.  The legacy mma.sync kernel is not the cause (its layers on the other kernels: same numbers).
TOL_PX_TC, TOL_SCORE_TC = 6e-2, 2e-2


@pytest.fixture(scope="module")
def teacher_onnx():
    from peppa_pig_face_landmark_b200 import teacher_graph as T
    return T.ensure_teacher_onnx()


def _oracle64(path, crops):
    import torch
    from oracle.onnx_exec import Session
    s = Session(path, dtype=torch.float64)
    xy, sc = [], []
    for c in crops:
        o, k = s.run(c.transpose(2, 0, 1)[None].astype(np.float64) / 255.0)
        xy.append(o.reshape(-1)); sc.append(k.reshape(-1))
    return np.array(xy), np.array(sc)


def test_teacher_graph_matches_readme_parameter_count(tmp_path):
    from peppa_pig_face_landmark_b200 import teacher_graph as T
    r = T.build_teacher_onnx(str(tmp_path / "t.onnx"))
    # README model table: teacher 11.53 "M" params (thop: / 2**20), 5.53 "G" (thop counts BN/elementwise too)
    assert r["params"] == 12085570 and round(r["params"] / 2 ** 20, 2) == 11.53
    assert r["macs"] == 5757497344 and 0.95 < r["macs"] / (5.53 * 2 ** 30) < 1.0


def test_teacher_plan_matches_oracle_graph(teacher_onnx):
    from peppa_pig_face_landmark_b200 import lowering, plan as P, teacher_graph as T
    from oracle.plan_interp import PlanInterp
    plan = lowering.lower(teacher_onnx, (256, 256))
    assert plan.macs == 5757497344                       # zero-padded channels (18->24, 36->40) are not counted
    convs = [o for o in plan.ops if o.type == P.OP_CONV]
    tc = [o for o in convs if o.flags & P.FLAG_TC]
    # everything but the uint8 stem, the ASPP pooling FC (the cSE FCs and the sSE conv are one OP_GAP_SSE + OP_SE_FC pair) and
    # the thin HBM-bound pointwise layers
    # (Cout 24 on >= 32x32 maps: pw_small_kernel) rides the tensor-core kernel
    thin = [o for o in convs if not (o.flags & P.FLAG_TC) and list(o.k) == [1, 1] and o.outs[0].C == 16
            and o.ins[0].C <= 32 and o.outs[0].H * o.outs[0].W >= 1024]
    mma = [o for o in convs if o.flags & P.FLAG_MMA]         # 24->24 @64x64 branch convs (halo-tile mma.sync kernel)
    assert len(mma) == 64 and all(list(o.k) == [3, 3] and o.ins[0].C == 24 for o in mma)
    assert len(convs) - len(tc) - len(mma) - len(thin) == 2 and sum(o.type == P.OP_ADDN for o in plan.ops) == 40
    assert sum(o.type == P.OP_GAP_SSE for o in plan.ops) == 1
    assert not any(o.type == P.OP_RESIZE_NEAREST and o.ins[0].H > 1 for o in plan.ops)   # HRNet upsamples are fused
    crops = T.synthetic_crops(2, 256, 99)
    xy, sc = PlanInterp(plan).run(crops)
    rxy, rsc = _oracle64(teacher_onnx, crops)
    assert np.abs(xy - rxy).max() * 256 < TOL_PX and np.abs(sc - rsc).max() < TOL_SCORE
    words, blob = plan.serialize()
    assert words[3] == len(plan.ops)


def test_channel_padding_leaves_shipped_graphs_alone():
    from peppa_pig_face_landmark_b200 import lowering
    from peppa_pig_face_landmark_b200.onnx_loader import load_onnx
    pre = os.path.join(os.path.dirname(lowering.__file__), "pretrained")
    for f in ("kps_student.onnx", "yolov5n-0.5.onnx"):
        g = load_onnx(os.path.join(pre, f))
        g2 = lowering.pad_channels(g)
        assert all(g2.weights[k].shape == v.shape for k, v in g.weights.items()), f


@pytest.mark.gpu
def test_teacher_cuda_matches_fp64_oracle(teacher_onnx):
    from peppa_pig_face_landmark_b200 import ONNXEngine, teacher_graph as T
    crops = T.synthetic_crops(3, 256, 7)
    eng = ONNXEngine(teacher_onnx, max_batch=4)
    xy, sc = eng.run_u8(crops)
    rxy, rsc = _oracle64(teacher_onnx, crops)
    dpx, dsc = np.abs(xy - rxy).max() * 256, np.abs(sc - rsc).max()
    print("teacher cuda vs fp64 oracle: %.2e px, %.2e score" % (dpx, dsc))
    assert dpx < TOL_PX_TC and dsc < TOL_SCORE_TC
    # batch invariance: a sample alone equals the same sample inside the batch
    xy1, sc1 = eng.run_u8(crops[1:2])
    assert np.abs(xy1[0] - xy[1]).max() * 256 < 1e-4 and np.abs(sc1[0] - sc[1]).max() < 1e-5


@pytest.mark.gpu
def test_teacher_cuda_fp32_fallback_path_agrees(teacher_onnx):
    """The same plan with every conv on the CUDA-core fp32 kernel (use_tc=False): independent of the tensor-core kernels and TMA."""
    from peppa_pig_face_landmark_b200 import ONNXEngine, teacher_graph as T
    crops = T.synthetic_crops(2, 256, 11)
    a = ONNXEngine(teacher_onnx, max_batch=2).run_u8(crops)
    b = ONNXEngine(teacher_onnx, max_batch=2, use_tc=False).run_u8(crops)
    rxy, rsc = _oracle64(teacher_onnx, crops)
    d32 = (np.abs(b[0] - rxy).max() * 256, np.abs(b[1] - rsc).max())
    dtc = (np.abs(a[0] - b[0]).max() * 256, np.abs(a[1] - b[1]).max())
    print("teacher fp32 CUDA-core path vs fp64 oracle: %.2e px %.2e; tensor-core path vs fp32 path: %.2e px %.2e" % (d32 + dtc))
    assert d32[0] < TOL_PX and d32[1] < TOL_SCORE            # graph lowering + every non-tensor-core kernel, tight
    assert dtc[0] < TOL_PX_TC and dtc[1] < TOL_SCORE_TC


def test_retargeted_128_exports_lower_and_match_oracle(tmp_path):
    """README's @128 variants (8f-3): the shipped student export re-targeted to 128 px, and the Teacher built at
    128 px, run through the same lowering; the plan interpreter must agree with the oracle executor."""
    import frames
    from peppa_pig_face_landmark_b200 import graph_tools, lowering, teacher_graph as T
    from oracle.plan_interp import PlanInterp
    from oracle.onnx_exec import Session
    src = os.path.join(os.path.dirname(lowering.__file__), "pretrained", "kps_student.onnx")
    s128 = graph_tools.retarget_input_size(src, str(tmp_path / "s128.onnx"), 128)
    plan = lowering.lower(s128, (128, 128))
    assert abs(plan.macs * 4 / 1482829696 - 1) < 0.01           # quarter of the @256 work (SE/FC layers do not scale)
    crops = frames.crop_variants(2)[:, ::2, ::2].copy()
    xy, sc = PlanInterp(plan).run(crops)
    sess = Session(s128)
    for i in range(2):
        o, k = sess.run(crops[i].transpose(2, 0, 1)[None].astype(np.float32) / np.float32(255))
        assert np.abs(xy[i] - o.reshape(-1)).max() * 128 < 1e-3 and np.abs(sc[i] - k.reshape(-1)).max() < 1e-4
    t128 = str(tmp_path / "t128.onnx")
    r = T.build_teacher_onnx(t128, size=128)
    assert r["params"] == 12085570
    plan = lowering.lower(t128, (128, 128))
    crops = T.synthetic_crops(1, 128, 5)
    xy, sc = PlanInterp(plan).run(crops)
    rxy, rsc = _oracle64(t128, crops)
    assert np.abs(xy - rxy).max() * 128 < TOL_PX and np.abs(sc - rsc).max() < TOL_SCORE


@pytest.mark.parametrize("size", [192, 320])
def test_retargeted_odd_sizes_lower_and_match_oracle(tmp_path, size):
    """Sizes the 128-pixel row-block tiling does not divide (48-/80-wide maps): the lowering still routes the dense convs to the
    tensor-core kernels (ragged tiles) and the plan interpreter agrees with the oracle executor."""
    import frames
    from peppa_pig_face_landmark_b200 import graph_tools, lowering, plan as P
    from oracle.plan_interp import PlanInterp
    from oracle.onnx_exec import Session
    from oracle.host_ref import resize_linear_u8
    src = os.path.join(os.path.dirname(lowering.__file__), "pretrained", "kps_student.onnx")
    path = graph_tools.retarget_input_size(src, str(tmp_path / "s.onnx"), size)
    plan = lowering.lower(path, (size, size))
    convs = [o for o in plan.ops if o.type == P.OP_CONV]
    assert sum(1 for o in convs if o.flags & P.FLAG_TC) >= len(convs) - 6
    crop = resize_linear_u8(frames.crop_variants(1)[0], size, size)[None]
    xy, sc = PlanInterp(plan).run(crop)
    o, k = Session(path).run(crop[0].transpose(2, 0, 1)[None].astype(np.float32) / np.float32(255))
    assert np.abs(xy[0] - o.reshape(-1)).max() * size < 1e-3 and np.abs(sc[0] - k.reshape(-1)).max() < 1e-4


@pytest.mark.gpu
def test_student_128_cuda_matches_oracle(tmp_path):
    import frames
    from peppa_pig_face_landmark_b200 import ONNXEngine, graph_tools, lowering
    from oracle.onnx_exec import Session
    src = os.path.join(os.path.dirname(lowering.__file__), "pretrained", "kps_student.onnx")
    s128 = graph_tools.retarget_input_size(src, str(tmp_path / "s128.onnx"), 128)
    crops = frames.crop_variants(5)[:, ::2, ::2].copy()
    xy, sc = ONNXEngine(s128, max_batch=5).run_u8(crops)          # odd batch: 8x8 maps share tiles between images
    sess = Session(s128)
    for i in range(5):
        o, k = sess.run(crops[i].transpose(2, 0, 1)[None].astype(np.float32) / np.float32(255))
        assert np.abs(xy[i] - o.reshape(-1)).max() * 128 < 1e-3 and np.abs(sc[i] - k.reshape(-1)).max() < 1e-4


@pytest.mark.gpu
def test_student_192_cuda_matches_oracle(tmp_path):
    """A size the 128-pixel row-block tiling does not divide (48-, 24-, 12-wide maps): ragged tensor-core tiles, the fused
    kernels' overhanging tiles and the pixels-on-lanes heat-map epilogue (48 x 48 maps are not whole 256-pixel row blocks)."""
    import frames
    from peppa_pig_face_landmark_b200 import ONNXEngine, graph_tools, lowering
    from oracle.onnx_exec import Session
    from oracle.host_ref import resize_linear_u8
    src = os.path.join(os.path.dirname(lowering.__file__), "pretrained", "kps_student.onnx")
    s192 = graph_tools.retarget_input_size(src, str(tmp_path / "s192.onnx"), 192)
    crops = np.stack([resize_linear_u8(c, 192, 192) for c in frames.crop_variants(3)])
    xy, sc = ONNXEngine(s192, max_batch=3).run_u8(crops)
    sess = Session(s192)
    for i in range(3):
        o, k = sess.run(crops[i].transpose(2, 0, 1)[None].astype(np.float32) / np.float32(255))
        assert np.abs(xy[i] - o.reshape(-1)).max() * 192 < 1e-3 and np.abs(sc[i] - k.reshape(-1)).max() < 1e-4


@pytest.mark.gpu
def test_teacher_128_cuda_matches_fp64_oracle(tmp_path):
    """README's Teacher@128 variant on the GPU (SURVEY 8f-3): 32 x 32 ... 4 x 4 branch maps (multi-image tiles)."""
    from peppa_pig_face_landmark_b200 import ONNXEngine, teacher_graph as T
    t128 = str(tmp_path / "t128.onnx")
    T.build_teacher_onnx(t128, size=128)
    import torch
    from oracle.onnx_exec import Session
    crops = T.synthetic_crops(3, 128, 5)
    xy, sc = ONNXEngine(t128, max_batch=4).run_u8(crops)
    # The random-weight heat maps have near-tied maxima (landmark 35 of crop 0: 3.06885 at (23, 8) vs 3.06864 at (31, 18)); an
    # arg-max flip there is a 44 px jump that even the oracle's own float32 run makes on some hosts.  A landmark whose fp64
    # map has a second peak (outside the 5x5 neighbourhood of the first) within 1e-2 of the maximum - three times the score
    # error this path shows on these weights - is ill-conditioned and left out of the coordinate comparison; its score still
    # has to match.
    s64 = Session(t128, dtype=torch.float64)
    rxy, rsc, tie = [], [], []
    for c in crops:
        outs, kept = s64.run(c.transpose(2, 0, 1)[None].astype(np.float64) / 255.0, keep="all")
        rxy.append(outs[0].reshape(-1)); rsc.append(outs[1].reshape(-1))
        hm = [v for v in kept.values() if hasattr(v, "ndim") and v.ndim == 4 and v.shape[1] == 294][-1][0, :98].numpy()
        t = np.zeros(98, bool)
        for l in range(98):
            h = hm[l].copy()
            y, x = np.unravel_index(int(h.argmax()), h.shape)
            v1 = h[y, x]
            h[max(0, y - 2):y + 3, max(0, x - 2):x + 3] = -np.inf
            t[l] = (v1 - h.max()) < 1e-2
        tie.append(np.repeat(t, 2))
    rxy, rsc, tie = np.array(rxy), np.array(rsc), np.array(tie)
    assert tie.mean() < 0.05
    dpx, dsc = (np.abs(xy - rxy) * ~tie).max() * 128, np.abs(sc - rsc).max()
    print("teacher@128 cuda vs fp64 oracle: %.2e px, %.2e score (%d near-tied landmark coordinates left out)" % (dpx, dsc, int(tie.sum())))
    assert dpx < TOL_PX_TC and dsc < TOL_SCORE_TC
