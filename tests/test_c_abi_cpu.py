"""What Python hands the C API, without a GPU: every function of include/skps_b200.h has as many ctypes argtypes in
runtime.SIGNATURES as the header has parameters (a stale list is not an error to ctypes but a garbled call), and FaceAna
and FaceAnaStreams build the same skps_pipeline_cfg from Skps.yml apart from top_k."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _header_arity():
    """name -> parameter count of every SKPS_API function the header declares."""
    with open(os.path.join(ROOT, "include", "skps_b200.h")) as f:
        hdr = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    out = {}
    for name, params in re.findall(r"SKPS_API\s[\w\s\*]*?(skps_\w+)\s*\(([^)]*)\)", hdr):
        params = params.strip()
        out[name] = 0 if params in ("", "void") else params.count(",") + 1
    return out


def test_signatures_match_header_arity():
    from peppa_pig_face_landmark_b200 import runtime
    arity = _header_arity()
    assert len(arity) >= 25
    assert set(arity) == set(runtime.SIGNATURES), set(arity) ^ set(runtime.SIGNATURES)
    wrong = {name: (n, len(runtime.SIGNATURES[name][1])) for name, n in arity.items()
             if n != len(runtime.SIGNATURES[name][1])}
    assert not wrong, "header parameters vs argtypes: %s" % wrong


def test_frame_staging_entry_points_arity():
    """Host frames are staged only by skps_pipeline_frame_diff / skps_mpipe_submit, and run / commit_frame take no frame."""
    from peppa_pig_face_landmark_b200 import runtime
    arity = _header_arity()
    want = {"skps_pipeline_run": 17, "skps_pipeline_frame_diff": 6, "skps_pipeline_commit_frame": 1,
            "skps_mpipe_submit": 5}
    for name, n in want.items():
        assert arity[name] == n == len(runtime.SIGNATURES[name][1]), name


class _Built(Exception):
    pass


def _cfg_of(monkeypatch, module, make):
    """The PipelineCfg that make() builds through module.pipeline_cfg (construction stops there, before any engine)."""
    seen = []
    real = module.pipeline_cfg

    def spy(*args):
        seen.append(real(*args))
        raise _Built
    monkeypatch.setattr(module, "pipeline_cfg", spy)
    with pytest.raises(_Built):
        make()
    return seen[0]


def test_faceana_and_streams_share_pipeline_cfg(monkeypatch):
    from peppa_pig_face_landmark_b200 import runtime as rt
    from peppa_pig_face_landmark_b200.core.api import face_landmark, facer, streams
    hw = (1080, 1920)
    a = _cfg_of(monkeypatch, facer, lambda: facer.FaceAna(top_k=512, max_frame_hw=hw))
    b = _cfg_of(monkeypatch, streams, lambda: streams.FaceAnaStreams(n_streams=4, top_k=8, max_frame_hw=hw))
    assert (a.top_k, b.top_k) == (512, 8)
    fields = [f for f, _ in rt.PipelineCfg._fields_ if f != "top_k"]
    assert {f: getattr(a, f) for f in fields} == {f: getattr(b, f) for f in fields}
    cfg = facer.get_cfg()['Skps']
    det, trace = cfg['Detect'], cfg['Trace']
    f32 = np.float32
    assert (a.score_thres, a.iou_thres, a.min_face) == (f32(det['score_thrs']), f32(det['iou_thrs']), f32(det['min_face']))
    assert (a.track_iou, a.alpha) == (f32(trace['iou_thres']), f32(trace['smooth_box']))
    assert a.face_scale == f32(1 + 2 * cfg['Keypoints']['base_extend_range'][0])
    assert a.face_scale == face_landmark.face_scale(cfg['Keypoints'])
    assert a.kps_min_face == face_landmark.MIN_FACE == 20
    assert (a.max_h, a.max_w) == hw
