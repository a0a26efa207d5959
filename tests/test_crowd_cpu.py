"""Crowd frames for the NMS of any size (csrc/nms.cu), checked without a GPU: the fixtures really pass both old limits (more
than 1024 candidates, more than 256 kept boxes), no row sits close enough to the score threshold for GPU-versus-CPU detector
rounding to flip it, and the new kernels compile for sm_90a without spilling."""
import os
import re

import numpy as np
import pytest

import frames
from test_wgmma_codegen import _ptxas_report

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
DET = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "yolov5n-0.5.onnx")

# name -> (grid of test1.jpg copies, face width in px, detector input) on a 3840x2160 frame
CROWDS = {
    "crowd96_768x1280": ((8, 12), 240, (768, 1280)),
    "crowd192_1152x1920": ((12, 16), 180, (1152, 1920)),
    "crowd384_1152x1920": ((16, 24), 150, (1152, 1920)),
}
# the smallest |obj - 0.5| over all rows of each fixture (CPU oracle); the GPU detector agrees with it to about 1e-5
THRESHOLD_CLEARANCE = 1e-4


def crowd_frame(name):
    grid, face_w, _ = CROWDS[name]
    return frames.multi_face_frame(2160, 3840, grid, face_w)


@pytest.fixture(scope="module")
def oracle_raw(tmp_path_factory):
    """Raw detector rows of every crowd from the oracle executor on the retargeted graph (written under tmp_path)."""
    from oracle import host_ref as H
    from oracle.onnx_exec import Session
    from peppa_pig_face_landmark_b200.graph_tools import retarget_detector_input
    d = tmp_path_factory.mktemp("crowd")
    out, nets = {}, {}
    for name, (_, _, hw) in CROWDS.items():
        if hw not in nets:
            nets[hw] = Session(retarget_detector_input(DET, str(d / ("det_%dx%d.onnx" % hw)), hw))
        x, recover = H.letterbox(crowd_frame(name), *hw)
        out[name] = (np.asarray(nets[hw].run(x)[0]).reshape(-1, 16), recover)
    return out


def test_crowd96_has_more_candidates_than_the_old_limit(oracle_raw):
    raw, _ = oracle_raw["crowd96_768x1280"]
    assert raw.shape == (60480, 16)
    assert (raw[:, 4] > 0.5).sum() > 1024


def test_crowd384_keeps_more_boxes_than_the_old_limit(oracle_raw):
    from oracle import host_ref as H
    raw, recover = oracle_raw["crowd384_1152x1920"]
    kept, idx = H.detect_post(raw, recover)
    assert len(idx) > 256


@pytest.mark.parametrize("name", sorted(CROWDS))
def test_no_row_near_the_score_threshold(oracle_raw, name):
    raw, _ = oracle_raw[name]
    assert np.abs(raw[:, 4] - 0.5).min() > THRESHOLD_CLEARANCE, name


def test_each_nms_and_selection_kernel_does_not_spill():
    # the four NMS kernels of nms.cu and the one selection kernel FaceAna and FaceAnaStreams share, each by name
    found = []
    for src, names in (("nms.cu", ("nms_",)), ("image_ops.cu", ("select_",))):
        out = _ptxas_report(src)
        props = re.findall(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                           r"(\d+) bytes spill loads", out)
        mine = [p for p in props if any(k in p[0] for k in names)]
        assert mine, out
        found += mine
    for k in ("nms_greedy_kernel", "nms_merge_kernel", "nms_chunk_sort_kernel", "nms_compact_kernel",
              "select_frames_kernel"):
        assert any(k in p[0] for p in found), (k, found)
    bad = [p for p in found if p[1:] != ("0", "0", "0")]
    assert not bad, bad
