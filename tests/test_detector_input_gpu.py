"""The detector at other input sizes on the GPU (FaceDetector / FaceAna / FaceAnaStreams with det_input): letterbox,
network and kept rows against the oracle run on the retargeted graph, whole-pipeline parity, the small face that only a
larger input finds, and the default 384x640 plan left as it was.  The unmodified reference cannot run these graphs (its
decode reshapes to a fixed 15120 rows), so the oracle executor on the retargeted file is the checker."""
import os

import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames
from test_parity_gpu import KPS_TOL_PX, SCORE_TOL

pytestmark = pytest.mark.gpu

PRE = os.path.join(os.path.dirname(__file__), "..", "peppa_pig_face_landmark_b200", "pretrained")
DET = os.path.join(PRE, "yolov5n-0.5.onnx")
SIZES = [(640, 640), (768, 1280), (1152, 1920)]


def _detector_ref(hw):
    from oracle.faceana_ref import DetectorRef
    from oracle.onnx_exec import Session
    from peppa_pig_face_landmark_b200.graph_tools import ensure_detector_onnx
    ref = DetectorRef(in_hw=hw)
    if hw != (384, 640):
        ref.net = Session(ensure_detector_onnx(DET, hw))
    return ref


def _faceana_ref(hw, top_k=5):
    from oracle.faceana_ref import FaceAnaRef
    ref = FaceAnaRef(top_k=top_k)
    ref.det = _detector_ref(hw)
    return ref


def _detector(hw):
    from peppa_pig_face_landmark_b200 import FaceDetector
    from peppa_pig_face_landmark_b200.core.api.facer import get_cfg
    cfg = get_cfg()['Skps']['Detect']
    cfg['input_shape'] = [hw[0], hw[1], 3]
    return FaceDetector(cfg)


def _close(res, ref, what):
    assert len(res) == len(ref), (what, len(res), len(ref))
    for a, b in zip(res, ref):
        assert np.abs(a["kps"].astype(np.float64) - b["kps"]).max() <= KPS_TOL_PX, what
        assert np.abs(a["scores"] - b["scores"]).max() <= SCORE_TOL, what
        assert np.abs(np.asarray(a["box"], np.float64) - np.asarray(b["box"], np.float64)).max() <= KPS_TOL_PX, what


def small_face_4k():
    """A 3840x2160 frame holding test1.jpg scaled to 140x93: a face of about 53x62 px, which the 384x640 detector input
    shrinks to 9x10 px (below the smallest anchors) and 1152x1920 to 26x31 px."""
    face = frames._resize(frames.load_test1(), 140, 93)
    f = frames._background(2160, 3840)
    f[1000:1093, 1800:1940] = face
    return f


@pytest.fixture(scope="module", params=SIZES, ids=lambda hw: "%dx%d" % hw)
def sized(request):
    hw = request.param
    return hw, _detector(hw), _detector_ref(hw)


@pytest.mark.parametrize("name", ["test1", "canvas640", "hd1080", "uhd4k"])
def test_letterbox_bit_exact(sized, name):
    from oracle import host_ref as H
    hw, det, _ = sized
    img = {"test1": frames.load_test1, "canvas640": frames.canvas_640, "hd1080": frames.frame_1080p,
           "uhd4k": frames.frame_4k}[name]()
    got, rec = det.preprocess(img)
    ref, rec_ref = H.letterbox(img, *hw)
    assert got.shape == (1, 3) + hw
    assert rec == rec_ref
    assert np.array_equal(got, ref)


def test_detector_layerwise_and_outputs(sized):
    import io
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "tools"))
    from layer_report import report
    hw = sized[0]
    buf = io.StringIO()
    worst = report("detector", out=buf, det_input=hw)
    assert worst < 2e-4, buf.getvalue()[-4000:]


def test_onnxengine_rows_and_outputs(sized):
    from oracle import host_ref as H
    from peppa_pig_face_landmark_b200 import ONNXEngine
    from peppa_pig_face_landmark_b200.graph_tools import detector_rows, ensure_detector_onnx
    hw, _, ref = sized
    x, _ = H.letterbox(frames.frame_4k(), *hw)
    out = ONNXEngine(ensure_detector_onnx(DET, hw))(x)[0][0]
    want = np.asarray(ref.net.run(x)[0]).reshape(-1, 16)
    assert out.shape == want.shape == (detector_rows(hw), 16)
    assert np.array_equal(np.where(out[:, 4] > 0.5)[0], np.where(want[:, 4] > 0.5)[0])
    assert (np.abs(out - want) < 5e-3 + 2e-5 * np.abs(want)).all()


def test_detector_kept_rows_match_oracle(sized):
    hw, det, ref = sized
    for name, fr in [("test1", frames.load_test1()), ("canvas640", frames.canvas_640()), ("uhd4k", frames.frame_4k())]:
        boxes = det(fr)
        want, idx = ref(fr, return_indices=True)
        assert np.array_equal(det.last_keep_idx, idx), (hw, name)
        assert boxes.shape == want.shape
        assert (np.abs(boxes - want) < 5e-3 + 2e-5 * np.abs(want)).all(), (hw, name)


@pytest.mark.parametrize("hw", SIZES, ids=lambda hw: "%dx%d" % hw)
@pytest.mark.parametrize("name,top_k", [("canvas640", 5), ("uhd4k", 16)])
def test_faceana_still_frame_and_tracker_path_match_oracle(hw, name, top_k):
    from Skps import FaceAna
    fr = {"canvas640": frames.canvas_640, "uhd4k": frames.frame_4k}[name]()
    facer, ref = FaceAna(top_k=top_k, det_input=hw), _faceana_ref(hw, top_k)
    r0, w0 = facer.run(fr), ref.run(fr)
    want_idx = ref.det(fr, return_indices=True)[1]
    assert np.array_equal(facer.last_det_idx, want_idx), (hw, name)
    assert len(r0) > 0
    _close(r0, w0, (hw, name, 0))
    _close(facer.run(fr), ref.run(fr), (hw, name, 1))         # unchanged frame: tracker path, no detector


@pytest.mark.parametrize("hw", SIZES, ids=lambda hw: "%dx%d" % hw)
def test_faceana_video_matches_oracle(hw):
    from Skps import FaceAna
    facer, ref = FaceAna(det_input=hw), _faceana_ref(hw)
    for t, fr in enumerate(video_frames()):
        _close(facer.run(fr), ref.run(fr), (hw, t))


@pytest.mark.parametrize("hw", [(768, 1280), (1152, 1920)], ids=lambda hw: "%dx%d" % hw)
def test_streams_match_single_stream_faceana(hw):
    """Frames of 1080x1920, 640x640 and 273x410 in one batch, with align and pose on: every stream returns what its own
    FaceAna(det_input=hw) returns."""
    from Skps import FaceAna, FaceAnaStreams
    v = video_frames()
    c, t1 = frames.canvas_640(), frames.load_test1()
    seqs = [v, [c, c, v[4], c, c, c], [t1, t1, t1, v[1], t1, t1]]
    fa = FaceAnaStreams(n_streams=len(seqs), det_input=hw, align=112, pose=True)
    singles = [FaceAna(det_input=hw, align=112, pose=True) for _ in seqs]
    found = 0
    for t in range(6):
        res = fa.run([s[t] for s in seqs])
        for k, s in enumerate(seqs):
            want = singles[k].run(s[t])
            assert len(res[k]) == len(want), (hw, t, k)
            for x, y in zip(res[k], want):
                assert np.abs(np.asarray(x["kps"], np.float64) - np.asarray(y["kps"], np.float64)).max() <= 1e-6
                assert np.abs(np.asarray(x["box"], np.float64) - np.asarray(y["box"], np.float64)).max() <= 1e-6
                assert np.array_equal(x["scores"], y["scores"])
                assert np.abs(x["M"] - y["M"]).max() <= 1e-4
                assert np.abs(x["pose"]["euler"] - y["pose"]["euler"]).max() <= 1e-2
            found += len(want)
    assert found > 10


def test_small_face_in_4k_is_found_only_at_the_larger_input():
    from Skps import FaceAna
    fr = small_face_4k()
    assert len(_detector_ref((384, 640))(fr)) == 0
    assert len(_detector_ref((1152, 1920))(fr)) == 1
    assert FaceAna().run(fr) == [] and _faceana_ref((384, 640)).run(fr) == []
    facer, ref = FaceAna(det_input=(1152, 1920)), _faceana_ref((1152, 1920))
    res, want = facer.run(fr), ref.run(fr)
    assert len(res) == 1
    _close(res, want, "small face")
    x0, y0, x1, y1 = res[0]["box"]
    assert 1790 < x0 < x1 < 1950 and 990 < y0 < y1 < 1100


def test_default_plan_unchanged_and_retarget_only_when_asked():
    from Skps import FaceAna, FaceAnaStreams
    from peppa_pig_face_landmark_b200 import lowering
    words, blob = lowering.lower(DET, (384, 640)).serialize()
    for fa in (FaceAna(), FaceAna(det_input=(384, 640))):
        w, b = fa.face_detector.model.plan.serialize()
        assert np.array_equal(w, words) and np.array_equal(b, blob)
    w, b = FaceAnaStreams(n_streams=2).det.plan.serialize()
    assert np.array_equal(w, words) and np.array_equal(b, blob)
    assert FaceAna(det_input=(640, 640)).face_detector.model.in_hw == (640, 640)
    for bad in [(640, 600), (64, 640), (2304, 640)]:
        with pytest.raises(ValueError):
            FaceAna(det_input=bad)
        with pytest.raises(ValueError):
            FaceAnaStreams(n_streams=2, det_input=bad)


def test_engine_refuses_a_batch_past_32_bit_indexing():
    """At 2176x3840 the stem output has 33.4 M elements per frame, so 65 frames pass 2^31: the engine reports it at
    creation instead of running kernels whose 32-bit thread numbers would not reach the end of the tensor."""
    from peppa_pig_face_landmark_b200 import ONNXEngine
    from peppa_pig_face_landmark_b200.graph_tools import ensure_detector_onnx
    with pytest.raises(RuntimeError, match="2\\^31"):
        ONNXEngine(ensure_detector_onnx(DET, (2176, 3840)), max_batch=65)
