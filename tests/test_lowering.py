"""CPU checks of the host logic: the ONNX->plan lowering (executed by the torch plan interpreter)
against the oracle graph executor, plan serialisation, and the C-ABI export list."""
import os
import re

import numpy as np
import pytest

import frames

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
PRE = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained")


def test_student_plan_matches_oracle_graph():
    from peppa_pig_face_landmark_b200 import lowering
    from oracle.plan_interp import PlanInterp
    from oracle.onnx_exec import Session
    plan = lowering.lower(os.path.join(PRE, "kps_student.onnx"), (256, 256))
    assert plan.macs == 1482829696            # SURVEY.md 8(d): 1.4828e9 MAC per face
    crops = frames.crop_variants(2)
    xy, sc = PlanInterp(plan).run(crops)
    sess = Session(os.path.join(PRE, "kps_student.onnx"))
    for i in range(2):
        x = crops[i].transpose(2, 0, 1).astype(np.float32)[None] / np.float32(255)
        o, s = sess.run(x)
        assert np.abs(xy[i] - o.reshape(-1)).max() * 256 < 1e-3
        assert np.abs(sc[i] - s.reshape(-1)).max() < 1e-4


def test_detector_plan_matches_oracle_graph():
    from peppa_pig_face_landmark_b200 import lowering, plan as P
    from oracle.plan_interp import PlanInterp
    from oracle.onnx_exec import Session
    from oracle import host_ref as H
    plan = lowering.lower(os.path.join(PRE, "yolov5n-0.5.onnx"), (384, 640))
    assert plan.macs == 441169920
    assert sum(o.type == P.OP_COPY for o in plan.ops) == 13      # only the shuffle pass-through halves move
    x, _ = H.letterbox(frames.load_test1())
    u8 = np.round(x[0].transpose(1, 2, 0) * 255).astype(np.uint8)[None]
    out = PlanInterp(plan).run(u8)[0][0]
    ref = Session(os.path.join(PRE, "yolov5n-0.5.onnx")).run(x)[0].reshape(15120, 16)
    assert np.array_equal(np.where(out[:, 4] > 0.5)[0], np.where(ref[:, 4] > 0.5)[0])
    assert np.abs(out - ref).max() < 5e-3


def test_plan_serialisation_is_header_buffers_and_ops():
    """The int32 words are the header, the buffer table and the op table, and nothing after them."""
    from peppa_pig_face_landmark_b200 import lowering, plan as P
    plan = lowering.lower(os.path.join(PRE, "kps_student.onnx"), (256, 256))
    words, blob = plan.serialize()
    assert words[0] == 0x534B5053 and words[2] == len(plan.bufs) and words[3] == len(plan.ops)
    body = 8 + 4 * len(plan.bufs) + P.OP_WORDS * len(plan.ops)
    assert words.size == body
    assert blob.dtype == np.float32 and all(op.w_off % 4 == 0 for op in plan.ops if op.w_off >= 0)


def test_c_abi_exports_every_declared_symbol():
    """include/skps_b200.h vs the built library vs the ctypes table (no compute calls)."""
    from peppa_pig_face_landmark_b200 import build, runtime
    build.build()
    hdr = open(os.path.join(ROOT, "include", "skps_b200.h")).read()
    declared = set(re.findall(r"SKPS_API [\w\s\*]+?(skps_\w+)\(", hdr))
    assert len(declared) >= 25
    assert declared == set(runtime.SIGNATURES), declared ^ set(runtime.SIGNATURES)
    lib = runtime.load_library()
    for name in declared:
        assert hasattr(lib, name)
    assert lib.skps_version() == 1


def test_product_path_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from peppa_pig_face_landmark_b200 import FaceAna
    with pytest.raises(RuntimeError):
        FaceAna()


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "peppa_pig_face_landmark_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, os.path.join(dp, f)


def test_product_package_reads_no_environment_variables():
    """Plans and kernels are chosen from layer shapes alone, so what a forward pass computes never depends on process
    state.  The one variable read is build.py's NVCC: which compiler builds the library."""
    pkg = os.path.join(ROOT, "peppa_pig_face_landmark_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".h")):
                path = os.path.join(dp, f)
                src = open(path).read()
                if path == os.path.join(pkg, "build.py"):
                    src = src.replace('os.environ.get("NVCC")', "", 1)
                assert "getenv(" not in src and "os.environ" not in src, path


def test_onnx_writer_round_trips_the_shipped_graphs(tmp_path):
    """onnx_writer.save_onnx is the inverse of onnx_loader.load_onnx on everything the shipped files contain
    (0-d tensors, int64 constants, string/int/float/list attributes)."""
    from peppa_pig_face_landmark_b200.onnx_loader import load_onnx
    from peppa_pig_face_landmark_b200.onnx_writer import save_onnx
    from oracle import onnx_lite
    for f in ("kps_student.onnx", "yolov5n-0.5.onnx"):
        g = load_onnx(os.path.join(PRE, f))
        out = str(tmp_path / f)
        save_onnx(out, g.nodes, g.weights, [(g.inputs[0], g.input_shapes[g.inputs[0]])], [(o, [1]) for o in g.outputs])
        g2, g3 = load_onnx(out), onnx_lite.load(out)           # product reader and the oracle's independent reader
        assert len(g.nodes) == len(g2.nodes) == len(g3.nodes) and g2.inputs == g.inputs and g2.outputs == g.outputs
        for a, b, c in zip(g.nodes, g2.nodes, g3.nodes):
            assert (a.op, a.name, a.inputs, a.outputs) == (b.op, b.name, b.inputs, b.outputs) == (c.op, c.name, c.inputs, c.outputs)
            assert a.attrs.keys() == b.attrs.keys()
            for k, va in a.attrs.items():
                if isinstance(va, np.ndarray):
                    assert va.dtype == b.attrs[k].dtype and va.shape == b.attrs[k].shape and np.array_equal(va, b.attrs[k])
                    assert np.array_equal(va, c.attrs[k])
                else:
                    assert va == b.attrs[k] == c.attrs[k]
        assert all(np.array_equal(v, g2.weights[k]) and v.dtype == g2.weights[k].dtype for k, v in g.weights.items())


def test_student_plan_fusions():
    """The fusions the student plan relies on: 8 squeeze-excite chains (GAP + 2 FC -> per-tile sums + one gate op) whose
    scale rides inside the projection conv (FLAG_XF, no OP_SCALE_CH pass), both decoder heads (upsample + concat +
    depthwise + 1x1 as one OP_DWPW), the depthwise -> 1x1 pairs of the blocks without squeeze-excite, the split heat-map
    head."""
    from peppa_pig_face_landmark_b200 import lowering, plan as P
    plan = lowering.lower(os.path.join(PRE, "kps_student.onnx"), (256, 256))
    kinds = [o.type for o in plan.ops]
    # 8 encoder squeeze-excite gates + the decoder's cSE branch (scSE front end fused: OP_GAP_SSE -> OP_SE_FC); the one
    # GlobalAveragePool left is the ASPP pooling branch
    assert kinds.count(P.OP_SE_FC) == 9 and kinds.count(P.OP_GAP) == 1 and kinds.count(P.OP_GAP_SSE) == 1
    assert kinds.count(P.OP_UPCAT_DW) == 0 and kinds.count(P.OP_SCALE_CH) == 0
    fused = [o for o in plan.ops if o.type == P.OP_DWPW]
    assert len(fused) == 6 and sum(1 for o in fused if o.ins[2] is not None) == 2          # 4 encoder pairs + 2 decoder heads
    # the full-resolution head (stem, blocks.0.0, blocks.1.0 expand + stride-2 depthwise) is one op on the uint8 input
    sb = plan.ops[0]
    assert sb.type == P.OP_STEM_BLOCK and sb.ins[0].buf is plan.input.buf and sb.outs[0].C == 64 and sb.outs[0].H == 64
    assert sb.w.size == 27 * 16 + 16 + 144 + 16 + 256 + 16 + 1024 + 64 and sb.extra.shape == (10, 64) and len(sb.sub_ops) == 4
    assert sum(1 for o in plan.ops if o.type == P.OP_STEM_BLOCK) == 1
    for o in fused:
        K = o.ins[0].C + (o.ins[2].C if o.ins[2] is not None else 0)
        assert o.extra.shape == (10, -(-K // 64) * 64) and o.extra_slot == 3 and o.w.shape[1] == o.extra.shape[1]
    scaled = [o for o in plan.ops if o.type == P.OP_CONV and o.flags & P.FLAG_XF]
    assert len(scaled) == 8 and all(o.ins[2] is not None and o.ins[0].buf.dtype == P.DT_SPLIT16 for o in scaled)
    for o in scaled:                     # each gate comes from the squeeze-excite op of the same block
        assert any(se.outs[0].buf is o.ins[2].buf for se in plan.ops if se.type == P.OP_SE_FC)
    for se in (o for o in plan.ops if o.type == P.OP_SE_FC and not any(g.type == P.OP_GAP_SSE and g.outs[0].buf is o.ins[0].buf for g in plan.ops)):
        dw = [o for o in plan.ops if o.type == P.OP_DWCONV and len(o.outs) == 2 and o.outs[1].buf is se.ins[0].buf]
        assert len(dw) == 1 and dw[0].flags & P.FLAG_GAP_PARTIAL
        o = dw[0].outs[0]
        th = P.dw_tile_rows(dw[0].k[0], dw[0].s[0])
        assert se.ins[0].buf.H == -(-o.H // th) * -(-o.W // P.DW_TILE_W) and se.ints[3] == o.H * o.W
    dec = plan.ops[-1]
    hm = plan.ops[-2]
    assert dec.type == P.OP_HM_DECODE and len(dec.ins) == 3 and dec.w.shape == (196, 128) and dec.ints[:2] == [98, 128]
    # the score maps are reduced to per-tile (max, arg-max) rows in the head conv's epilogue: 16 row-block tiles of 256 pixels
    # per face (the transposed head kernel, csrc/conv_hm.cu)
    assert (hm.flags & P.FLAG_HM_PART) and (dec.flags & P.FLAG_HM_PART) and hm.outs[1].buf is dec.ins[2].buf
    assert (hm.outs[1].buf.H, hm.outs[1].buf.W, hm.outs[1].buf.C) == (16, 1, 256)
    # the ASPP tail's BatchNorm+ReLU over the 256-channel concat is folded into the four producers: the only affine op left
    # works on the pooled branch's 64 x 1 x 1 tensor
    aff = [o for o in plan.ops if o.type == P.OP_AFFINE_ACT]
    assert len(aff) == 1 and aff[0].outs[0].H * aff[0].outs[0].W == 1 and aff[0].outs[0].C == 64
    aspp = [o for o in plan.ops if o.type == P.OP_CONV and "/aspp/conv" in o.name]
    assert len(aspp) == 3 and all(o.act == P.ACT_RELU and o.b is not None for o in aspp)
    assert hm.type == P.OP_CONV and hm.outs[0].buf.C == 104 and hm.ins[0].buf is dec.ins[1].buf


def test_upcat_effective_weights_equal_upsample_then_depthwise():
    """plan.upcat_effective_weights: depthwise3x3(bilinear_x2(low)) as a class-dependent 3x3 stencil on the low-res map."""
    import torch
    import torch.nn.functional as F
    from peppa_pig_face_landmark_b200 import plan as P
    rng = np.random.default_rng(0)
    C, Hl, Wl = 8, 5, 7
    low = rng.standard_normal((1, C, Hl, Wl)).astype(np.float32)
    w = rng.standard_normal((9, C)).astype(np.float32)
    b = rng.standard_normal(C).astype(np.float32)
    up = F.interpolate(torch.from_numpy(low), scale_factor=2, mode="bilinear", align_corners=False)
    ref = F.conv2d(up, torch.from_numpy(w.T.reshape(C, 1, 3, 3).copy()), torch.from_numpy(b), padding=1, groups=C).numpy()[0]
    we = P.upcat_effective_weights(w)
    H, W = 2 * Hl, 2 * Wl

    def cls(p, n):
        return 0 if p == 0 else (3 if p == n - 1 else 1 + (p & 1))
    out = np.zeros((C, H, W), np.float32)
    for y in range(H):
        for x in range(W):
            acc = b.astype(np.float64).copy()
            for a in range(3):
                for bb in range(3):
                    acc += we[cls(y, H), cls(x, W), a, bb].astype(np.float64) * \
                        low[0, :, min(max(y // 2 + a - 1, 0), Hl - 1), min(max(x // 2 + bb - 1, 0), Wl - 1)]
            out[:, y, x] = acc
    assert np.abs(out - ref).max() < 5e-6


def test_pad_channels_on_a_synthetic_residual_graph(tmp_path):
    """18-channel tensors between dense convs are zero-padded to 24 without changing the result; tensors that reach a
    depthwise conv or a graph output are left alone."""
    import torch
    from peppa_pig_face_landmark_b200 import lowering
    from peppa_pig_face_landmark_b200.onnx_loader import OnnxNode, load_onnx
    from peppa_pig_face_landmark_b200.onnx_writer import save_onnx
    from oracle.onnx_exec import Session
    rng = np.random.default_rng(1)
    conv = dict(dilations=[1, 1], group=1, kernel_shape=[3, 3], pads=[1, 1, 1, 1], strides=[1, 1])
    W = {"w0": rng.standard_normal((18, 3, 3, 3)).astype(np.float32) * 0.2, "b0": rng.standard_normal(18).astype(np.float32),
         "w1": rng.standard_normal((18, 18, 3, 3)).astype(np.float32) * 0.1,
         "w2": rng.standard_normal((16, 18, 3, 3)).astype(np.float32) * 0.1}
    nodes = [OnnxNode("Conv", "c0", ["input", "w0", "b0"], ["t0"], dict(conv)), OnnxNode("Relu", "r0", ["t0"], ["t1"], {}),
             OnnxNode("Conv", "c1", ["t1", "w1"], ["t2"], dict(conv)), OnnxNode("Add", "a", ["t2", "t1"], ["t3"], {}),
             OnnxNode("Relu", "r1", ["t3"], ["t4"], {}), OnnxNode("Conv", "c2", ["t4", "w2"], ["out"], dict(conv))]
    path = str(tmp_path / "res.onnx")
    save_onnx(path, nodes, W, [("input", [1, 3, 16, 16])], [("out", [1, 16, 16, 16])])
    g = lowering.pad_channels(load_onnx(path))
    assert g.weights["w0"].shape == (24, 3, 3, 3) and g.weights["b0"].shape == (24,)
    assert g.weights["w1"].shape == (24, 24, 3, 3) and g.weights["w2"].shape == (16, 24, 3, 3)
    padded = str(tmp_path / "res_padded.onnx")
    save_onnx(padded, [OnnxNode(n.op, n.name, n.inputs, n.outputs, {k: v for k, v in n.attrs.items() if not k.startswith("_")})
                       for n in g.nodes], g.weights, [("input", [1, 3, 16, 16])], [("out", [1, 16, 16, 16])])
    x = rng.standard_normal((1, 3, 16, 16)).astype(np.float32)
    assert np.abs(Session(path).run(x)[0] - Session(padded).run(x)[0]).max() < 1e-5
