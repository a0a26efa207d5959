"""CPU checks of the detector at other input sizes (graph_tools.retarget_detector_input): the retargeted graph is the
shipped one at 384x640, bad sizes and non-detector graphs are refused, its output is the yolov5-face decode of its own
head convolutions, and the lowered plan agrees with the oracle executor."""
import os

import numpy as np
import pytest
import torch

import frames

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
PRE = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained")
DET = os.path.join(PRE, "yolov5n-0.5.onnx")
SIZES = [(640, 640), (768, 1280), (1152, 1920)]
# yolov5n-0.5-face anchors (w, h) per stride, SURVEY.md 2.2 K4
ANCHORS = {8: [(4, 5), (8, 10), (13, 16)], 16: [(23, 29), (43, 55), (73, 105)], 32: [(146, 217), (231, 300), (335, 433)]}


@pytest.fixture(scope="module")
def retargeted(tmp_path_factory):
    from peppa_pig_face_landmark_b200.graph_tools import retarget_detector_input
    d = tmp_path_factory.mktemp("det")
    return {hw: retarget_detector_input(DET, str(d / ("det_%dx%d.onnx" % hw)), hw) for hw in SIZES}


def test_retarget_to_the_export_size_gives_back_the_shipped_graph(tmp_path):
    from peppa_pig_face_landmark_b200.graph_tools import retarget_detector_input
    from peppa_pig_face_landmark_b200.onnx_loader import load_onnx
    g = load_onnx(DET)
    g2 = load_onnx(retarget_detector_input(DET, str(tmp_path / "d.onnx"), (384, 640)))
    assert g2.inputs == g.inputs and g2.outputs == g.outputs and g2.input_shapes == g.input_shapes
    assert len(g.nodes) == len(g2.nodes)
    for a, b in zip(g.nodes, g2.nodes):
        assert (a.op, a.name, a.inputs, a.outputs) == (b.op, b.name, b.inputs, b.outputs)
        assert a.attrs.keys() == b.attrs.keys()
        for k, va in a.attrs.items():
            vb = b.attrs[k]
            if isinstance(va, np.ndarray):
                assert va.dtype == vb.dtype and va.shape == vb.shape and va.tobytes() == vb.tobytes(), a.name
            else:
                assert va == vb, a.name
    assert g.weights.keys() == g2.weights.keys()
    assert all(v.dtype == g2.weights[k].dtype and v.tobytes() == g2.weights[k].tobytes() for k, v in g.weights.items())


@pytest.mark.parametrize("hw", [(384, 650), (380, 640), (96, 640), (384, 96), (2208, 3840), (384, 3872), (384,), "big"])
def test_retarget_refuses_bad_sizes(tmp_path, hw):
    from peppa_pig_face_landmark_b200.graph_tools import check_detector_input, retarget_detector_input
    with pytest.raises(ValueError):
        check_detector_input(hw)
    with pytest.raises(ValueError):
        retarget_detector_input(DET, str(tmp_path / "d.onnx"), hw)
    assert not os.path.exists(tmp_path / "d.onnx")


def test_retarget_refuses_a_graph_that_is_not_the_detector(tmp_path):
    from peppa_pig_face_landmark_b200.graph_tools import retarget_detector_input
    with pytest.raises(ValueError):
        retarget_detector_input(os.path.join(PRE, "kps_student.onnx"), str(tmp_path / "d.onnx"), (640, 640))


def test_size_range_and_row_counts():
    from peppa_pig_face_landmark_b200.graph_tools import check_detector_input, detector_rows
    assert check_detector_input((128, 128)) == (128, 128)
    assert check_detector_input([2176, 3840]) == (2176, 3840)
    assert [detector_rows(hw) for hw in [(384, 640)] + SIZES] == [15120, 25200, 60480, 136080]


def _decode(heads, hw):
    """yolov5-face Detect (SURVEY.md 2.2 K4) on the three (1, 48, H, W) head conv outputs: per stride s,
    xy = (2 sigmoid(t) - 0.5 + grid) s, wh = (2 sigmoid(t))^2 anchor, obj and cls = sigmoid, 5 landmarks = t anchor + grid s;
    rows ordered stride, anchor, y, x."""
    rows = []
    for (s, anchors), t in zip(sorted(ANCHORS.items()), heads):
        H, W = hw[0] // s, hw[1] // s
        assert t.shape == (1, 48, H, W)
        t = t.reshape(3, 16, H, W).permute(0, 2, 3, 1)                       # (anchor, y, x, 16)
        gy, gx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
        grid = torch.stack((gx, gy), -1)[None]                                 # (1, H, W, 2) as (x, y)
        anc = torch.tensor(anchors, dtype=torch.float32)[:, None, None, :]      # (3, 1, 1, 2) as (w, h)
        sg = torch.sigmoid(t)
        out = torch.empty_like(t)
        out[..., 0:2] = (sg[..., 0:2] * 2 - 0.5 + grid) * s
        out[..., 2:4] = (sg[..., 2:4] * 2) ** 2 * anc
        out[..., 4] = sg[..., 4]
        for k in range(5):
            out[..., 5 + 2 * k:7 + 2 * k] = t[..., 5 + 2 * k:7 + 2 * k] * anc + grid * s
        out[..., 15] = sg[..., 15]
        rows.append(out.reshape(-1, 16))
    return torch.cat(rows).numpy()


@pytest.mark.parametrize("hw", SIZES)
def test_retargeted_graph_output_is_the_yolov5_face_decode(retargeted, hw):
    """The regenerated grid, anchor-grid and reshape constants, checked against the decode restated from its definition."""
    from oracle import host_ref as H
    from oracle.onnx_exec import Session
    from peppa_pig_face_landmark_b200.graph_tools import detector_rows
    heads = ["/model.21/m.%d/Conv_output_0" % i for i in range(3)]
    x, _ = H.letterbox(frames.frame_4k(), *hw)
    (out,), kept = Session(retargeted[hw]).run(x, keep=set(heads))
    out = out.reshape(-1, 16)
    assert out.shape == (detector_rows(hw), 16)
    ref = _decode([kept[h] for h in heads], hw)
    np.testing.assert_allclose(out, ref, rtol=1e-6, atol=1e-5)
    assert (out[:, 4] > 0.5).sum() > 100                  # the 16 faces of the frame are found


@pytest.mark.parametrize("hw", SIZES)
def test_retargeted_plan_matches_oracle_graph(retargeted, hw):
    from oracle import host_ref as H
    from oracle.onnx_exec import Session
    from oracle.plan_interp import PlanInterp
    from peppa_pig_face_landmark_b200 import lowering
    from peppa_pig_face_landmark_b200.graph_tools import detector_rows
    plan = lowering.lower(retargeted[hw], hw)
    assert plan.outputs[0].buf.H == detector_rows(hw)
    x, _ = H.letterbox(frames.frame_4k(), *hw)
    u8 = np.round(x[0].transpose(1, 2, 0) * 255).astype(np.uint8)[None]
    out = PlanInterp(plan).run(u8)[0][0]
    ref = Session(retargeted[hw]).run(x)[0].reshape(-1, 16)
    assert np.array_equal(np.where(out[:, 4] > 0.5)[0], np.where(ref[:, 4] > 0.5)[0])
    assert np.abs(out - ref).max() < 5e-3


def test_default_plan_is_unchanged_by_detector_onnx_for():
    """FaceDetector builds the default (Skps.yml 384x640) engine from the shipped file itself: the same plan as before."""
    from peppa_pig_face_landmark_b200 import lowering
    from peppa_pig_face_landmark_b200.graph_tools import detector_onnx_for
    assert detector_onnx_for(DET, (384, 640)) == DET
    w0, b0 = lowering.lower(DET, (384, 640)).serialize()
    w1, b1 = lowering.lower(detector_onnx_for(DET, [384, 640]), (384, 640)).serialize()
    assert np.array_equal(w0, w1) and np.array_equal(b0, b1)
