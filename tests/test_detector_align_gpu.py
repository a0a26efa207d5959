"""FaceDetector(align=...): ArcFace chips from the detector's own five landmarks.  Every frame's rows and kept indices are
those of FaceDetector without align; its points are the host restatement (landmark_points) of its returned rows; its
matrices are align_faces' estimator on those points promoted to float64, bit for bit; its chips are cv2.warpAffine under
that matrix, byte for byte; and host frames, CUDA frames in every layout and CUDA frames with out= give the same."""
import numpy as np
import pytest

import frames
from oracle import align_ref as A
from test_align_gpu import cv2_warp
from test_crowd_cpu import crowd_frame
from test_detector_batch_gpu import _cfg
from test_frame_layouts_gpu import OTHER, as_layout
from test_landmark_batch_gpu import LAYOUTS, _cuda

pytestmark = pytest.mark.gpu


def _frames():
    """test1, the 640x640 canvas, 1080p with 4 faces, 4K with 16 faces and a faceless 720p frame: five sizes, one call."""
    return [frames.load_test1(), frames.canvas_640(), frames.frame_1080p(), frames.frame_4k(), frames._background(720, 1280)]


@pytest.fixture(scope="module")
def fs():
    return _frames()


@pytest.fixture(scope="module")
def plain(fs):
    from Skps import FaceDetector
    det = FaceDetector()
    rows = det.run_batch(fs)
    return rows, det.last_keep_idx


def _estimate(frame, points, size):
    """align_faces (core/api/align.py) on the five points placed at the WFLW-98 indices it reads, in float64."""
    from peppa_pig_face_landmark_b200.core.api.align import WFLW98_FIVE, align_faces
    kps = np.zeros((len(points), 98, 2), np.float64)
    kps[:, list(WFLW98_FIVE)] = points.astype(np.float64)
    return align_faces(frame, kps, size)


def _check(fs, res, keep, want, size, max_chips, in_hw=(384, 640), what=""):
    """res: FaceDetector(align=size, max_chips=max_chips).run_batch(fs) and its last_keep_idx; want: (rows, keep) of
    FaceDetector without align."""
    from peppa_pig_face_landmark_b200.core.api.face_detector import landmark_points, letterbox_geometry
    assert len(res) == len(fs) == len(keep)
    for i, (f, (rows, points, chips, M)) in enumerate(zip(fs, res)):
        k = min(len(rows), max_chips)
        assert rows.dtype == np.float32 and np.array_equal(rows, want[0][i]), (what, i)
        assert np.array_equal(keep[i], want[1][i]), (what, i)
        assert points.shape == (k, 5, 2) and points.dtype == np.float32, (what, i, points.shape)
        assert chips.shape == (k, size, size, 3) and chips.dtype == np.uint8, (what, i, chips.shape)
        assert M.shape == (k, 2, 3) and M.dtype == np.float64, (what, i, M.shape)
        if k == 0:
            continue
        scale, _, _, top, left = letterbox_geometry(f.shape[0], f.shape[1], *in_hw)
        assert np.array_equal(points, landmark_points(rows[:k], [scale, left, top])), (what, i)
        ac, aM = _estimate(f, points, size)
        assert np.array_equal(M, aM), (what, i, np.abs(M - aM).max())
        assert np.array_equal(chips, ac), (what, i)
        for j in range(k):
            want_M = A.umeyama(points[j].astype(np.float64), A.template(size))
            assert np.abs(M[j] - want_M).max() <= 1e-9 * np.abs(want_M).max(), (what, i, j)
            assert np.array_equal(chips[j], cv2_warp(f, M[j], size)), (what, i, j, int((chips[j] != cv2_warp(f, M[j], size)).sum()))


def _same(a, b, what):
    assert len(a) == len(b), what
    for i, (x, y) in enumerate(zip(a, b)):
        for u, v in zip(x, y):
            assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v), (what, i)


def _from_out(out, n, max_chips):
    """(rows, points, chips, M) per frame from new_results buffers."""
    cnt = out["count"][:n].cpu().numpy()
    res = []
    for i, c in enumerate(cnt.tolist()):
        k = min(c, max_chips)
        res.append((out["rows"][i, :c].cpu().numpy(), out["points"][i, :k].cpu().numpy(), out["chip"][i, :k].cpu().numpy(),
                    out["M"][i, :k].cpu().numpy()))
    return res


@pytest.mark.parametrize("size", [16, 112, 512])
def test_host_frames_equal_the_host_restatement(fs, plain, size):
    from Skps import FaceDetector
    det = FaceDetector(align=size)
    res = det.run_batch(fs)
    _check(fs, res, det.last_keep_idx, plain, size, 64, what=size)
    assert [len(r[2]) for r in res] == [len(r) for r in plain[0]]
    assert len(plain[0][3]) == 16 and len(plain[0][4]) == 0
    # __call__ still returns the rows
    rows = det(fs[2])
    assert np.array_equal(rows, plain[0][2]) and np.array_equal(det.last_keep_idx, plain[1][2])


@pytest.mark.parametrize("size", [16, 112, 512])
def test_cuda_frames_and_out_equal_host_frames(fs, plain, size):
    from Skps import FaceDetector
    det = FaceDetector(align=size, max_chips=5)
    host = det.run_batch(fs)
    _check(fs, host, det.last_keep_idx, plain, size, 5, what=size)
    assert [len(r[2]) for r in host] == [min(len(r), 5) for r in plain[0]] and len(host[3][2]) == 5
    for kind in sorted(LAYOUTS):
        dev = [LAYOUTS[kind](f) for f in fs]
        _same(det.run_batch(dev), host, (size, kind))
        out = det.new_results(len(fs) + 2)
        det.submit(dev, out=out)
        assert det.collect() is out
        _same(_from_out(out, len(fs), 5), host, (size, kind, "out"))


def test_every_cuda_layout_gives_the_bgr_result(fs, plain):
    from Skps import FaceDetector
    det = FaceDetector(align=112, max_chips=8)
    host = det.run_batch(fs)
    for layout in OTHER:
        for kind in ("packed", "roi"):
            dev = [as_layout(f, layout, kind, seed=i) for i, f in enumerate(fs)]
            _same(det.run_batch(dev, layout=layout), host, (layout, kind))
            out = det.new_results(len(fs))
            det.submit(dev, out=out, layout=layout)
            det.collect()
            _same(_from_out(out, len(fs), 8), host, (layout, kind, "out"))


def test_crowd_beyond_max_chips_and_max_det():
    """det_input 1152x1920: a 384-face crowd keeps more rows than max_chips and than come back with the counts; its first
    max_chips rows get chips."""
    from Skps import FaceDetector
    hw = (1152, 1920)
    fs = [frames.load_test1(), crowd_frame("crowd384_1152x1920"), frames._background(720, 1280),
          crowd_frame("crowd192_1152x1920")]
    ref = FaceDetector(_cfg(hw), max_frames=4)
    want = (ref.run_batch(fs), ref.last_keep_idx)
    assert len(want[0][1]) == 384 and len(want[0][3]) == 192
    det = FaceDetector(_cfg(hw), max_frames=4, align=112, max_chips=100)
    host = det.run_batch(fs)
    _check(fs, host, det.last_keep_idx, want, 112, 100, hw, "crowd host")
    assert [len(r[2]) for r in host] == [min(len(r), 100) for r in want[0]] and len(host[2][2]) == 0
    _same(det.run_batch([_cuda(f) for f in fs]), host, "crowd cuda")
    out = det.new_results(4)
    det.submit([_cuda(f) for f in fs], out=out)
    det.collect()
    _same(_from_out(out, 4, 100), host, "crowd out")
    # every kept row gets a chip once max_chips reaches the count
    big = FaceDetector(_cfg(hw), max_frames=4, align=16, max_chips=1024)
    res = big.run_batch(fs[1:2])
    _check(fs[1:2], res, big.last_keep_idx, ([want[0][1]], [want[1][1]]), 16, 1024, hw, "crowd all")
    assert len(res[0][2]) == 384


def test_two_calls_in_flight_and_more_frames_than_max_frames(fs, plain):
    """max_frames 2: a call of 8 frames runs in four chunks; two calls in flight into out= buffers, a host call between
    them, and a third call reusing the first call's slot while the second is pending."""
    import torch
    from Skps import FaceDetector
    det = FaceDetector(align=112, max_frames=2, max_chips=6)
    order = [3, 0, 4, 2, 1, 3, 2, 0]
    batch = [fs[i] for i in order]
    want = FaceDetector(align=112, max_chips=6).run_batch(fs)
    want_b = [want[i] for i in order]
    _same(det.run_batch(batch), want_b, "chunks host")
    dev = [_cuda(f) for f in batch]
    _same(det.run_batch(dev), want_b, "chunks cuda")
    bufs = [det.new_results(len(batch)) for _ in range(2)]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        det.submit(dev, out=bufs[0])
    det.submit(dev[::-1], out=bufs[1])
    det.collect()
    det.submit(batch[:3])                         # host frames into the first call's slot
    det.collect()
    host = det.collect()
    torch.cuda.synchronize()
    _same(_from_out(bufs[0], len(batch), 6), want_b, "in flight 0")
    _same(_from_out(bufs[1], len(batch), 6), want_b[::-1], "in flight 1")
    _same(host, want_b[:3], "in flight host")
    # two host calls in flight, each warped at its collect()
    det.submit(batch)
    det.submit(batch[::-1])
    _same(det.collect(), want_b, "host 0")
    _same(det.collect(), want_b[::-1], "host 1")


def test_refused_calls_enqueue_nothing(fs):
    from Skps import FaceDetector
    det = FaceDetector(align=16, max_chips=2)
    good = _cuda(fs[0])
    with pytest.raises(ValueError):
        det.submit([fs[0]], out=det.new_results(1))                 # out= takes CUDA frames
    res = det.new_results(1)
    plain_keys = {k: res[k] for k in ("rows", "idx", "count")}
    for bent in (plain_keys, dict(res, chip=res["chip"][:, :1]), dict(res, M=res["M"].float()),
                 dict(res, points=res["points"][:, :, :4])):
        with pytest.raises(ValueError):
            det.submit([good], out=bent)
    assert not det._pending
    assert set(det.new_results(2)) == {"rows", "idx", "count", "points", "M", "chip"}
    assert det.run_batch([]) == []


def test_eye_points_lie_near_the_landmark_nets_pupils():
    """A sanity check, not parity: on test1.jpg the detector's two eye points are ordered left to right and lie near
    landmarks 96 / 97 (the pupils) of the 98-point net."""
    from Skps import FaceAna, FaceDetector
    img = frames.load_test1()
    (rows, points, chips, M), = FaceDetector(align=112).run_batch([img])
    kps = FaceAna().run(img)[0]["kps"]
    assert len(points) == 1
    eyes = points[0, :2].astype(np.float64)
    assert eyes[0, 0] < eyes[1, 0]
    d = np.linalg.norm(eyes - kps[[96, 97]].astype(np.float64), axis=1)
    iod = np.linalg.norm(kps[97] - kps[96])
    print("test1 eye points vs landmarks 96 / 97: %.2f / %.2f px (inter-pupil distance %.2f px)" % (d[0], d[1], iod))
