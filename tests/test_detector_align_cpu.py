"""FaceDetector(align=...) without a GPU: the five landmarks' un-letterbox against the reference's scale_coords on the
oracle's kept rows, the align / max_chips checks, the result buffers with and without align, and the per-frame result
tuples (a frame without faces included)."""
import numpy as np
import pytest

from oracle import host_ref as H


def _kept_rows(g):
    """The oracle's kept detector rows (letterbox coordinates, columns 5..14 untouched) of a golden frame."""
    cand, keep = g["f0_det_cand_idx"], g["f0_det_keep_idx"]
    return np.stack([g["f0_det_cand_rows"][int(np.flatnonzero(cand == k)[0])] for k in keep]).astype(np.float32)


@pytest.mark.parametrize("name", ["test1", "canvas640"])
def test_points_are_scale_coords_of_the_landmark_columns(golden, name):
    from peppa_pig_face_landmark_b200.core.api.face_detector import landmark_points
    g = golden(name)
    rows, recover = _kept_rows(g), [float(v) for v in g["f0_recover"]]
    assert len(rows) >= 1
    got = landmark_points(rows, recover)
    assert got.shape == (len(rows), 5, 2) and got.dtype == np.float32
    for p in range(5):
        # scale_coords (face_detector.py:82-93) on (x, y, x, y) of point p: the arithmetic it applies to the box
        xyxy = np.ascontiguousarray(rows[:, [5 + 2 * p, 6 + 2 * p, 5 + 2 * p, 6 + 2 * p]])
        want = H.scale_coords(xyxy, recover)
        assert np.array_equal(got[:, p, 0], want[:, 0]) and np.array_equal(got[:, p, 1], want[:, 1]), (name, p)
    assert np.array_equal(rows, _kept_rows(g))                          # the rows are not modified
    # the points lie in the frame's pixels, inside the kept box
    box = H.scale_coords(H.xywh2xyxy(rows[:, :4].copy()), recover)
    assert (got[..., 0] > box[:, None, 0]).all() and (got[..., 0] < box[:, None, 2]).all()
    assert (got[..., 1] > box[:, None, 1]).all() and (got[..., 1] < box[:, None, 3]).all()


@pytest.mark.parametrize("kw", [dict(align=15), dict(align=513), dict(align=112.0), dict(align=True), dict(align="112"),
                                dict(align=112, max_chips=0), dict(align=112, max_chips=1025),
                                dict(align=112, max_chips=64.0), dict(align=112, max_chips=True),
                                dict(max_chips=None), dict(max_chips=-1)])
def test_bad_align_or_max_chips_raise_before_anything_is_allocated(kw, monkeypatch):
    from peppa_pig_face_landmark_b200.core.api import face_detector as fd

    def no_engine(*a, **k):
        raise AssertionError("the engine was built before the arguments were checked")
    monkeypatch.setattr(fd, "ONNXEngine", no_engine)
    with pytest.raises(ValueError):
        fd.FaceDetector(**kw)


def test_good_sizes_pass_the_checks():
    from peppa_pig_face_landmark_b200.core.api.align import check_size
    from peppa_pig_face_landmark_b200.core.api.face_detector import check_max_chips
    for v in (1, 64, 1024, np.int32(7)):
        assert check_max_chips(v) == int(v) and type(check_max_chips(v)) is int
    for v in (16, 112, 512):
        assert check_size(v) == v


def test_result_buffers_with_and_without_align():
    from peppa_pig_face_landmark_b200.core.api import face_detector as fd
    R = 15120
    plain = fd.result_fields(3, R)
    assert plain == {"rows": ((3, R, 16), "float32"), "idx": ((3, R), "int32"), "count": ((3,), "int32")}
    assert fd.result_fields(3, R, None, 64) == plain
    al = fd.result_fields(3, R, 112, 64)
    assert {k: al[k] for k in plain} == plain
    assert {k: v for k, v in al.items() if k not in plain} == {
        "points": ((3, 64, 5, 2), "float32"), "M": ((3, 64, 2, 3), "float64"), "chip": ((3, 64, 112, 112, 3), "uint8")}
    # the object's own fields: a detector built without running __init__'s engine
    for align, keys in ((None, set(plain)), (16, set(al))):
        d = object.__new__(fd.FaceDetector)
        d._rows, d.align, d.max_chips = R, align, 8
        f = d._fields(2)
        assert set(f) == keys
        if align:
            assert f["chip"] == ((2, 8, 16, 16, 3), "uint8") and f["M"] == ((2, 8, 2, 3), "float64")
    # 38.5 MB of chips per call slot for 16 frames at the defaults
    shape = fd.result_fields(16, R, 112, 64)["chip"][0]
    assert np.prod(shape) == 16 * 64 * 112 * 112 * 3 == 38535168


def test_result_tuples_of_frames_with_and_without_faces():
    from peppa_pig_face_landmark_b200.core.api.face_detector import align_results
    C, S = 3, 16
    rng = np.random.default_rng(0)
    count = np.array([0, 2, 5, 0], np.int32)
    rows = [rng.normal(size=(int(k), 16)).astype(np.float32) for k in count]
    points = rng.normal(size=(4, C, 5, 2)).astype(np.float32)
    M = rng.normal(size=(4, C, 2, 3))
    chips = rng.integers(0, 256, (2 + 3, S, S, 3), dtype=np.uint8)
    res = align_results(rows, count, points, chips, M, C)
    assert len(res) == 4
    for i, (r, p, c, m) in enumerate(res):
        k = min(int(count[i]), C)
        assert r is rows[i]
        assert p.shape == (k, 5, 2) and p.dtype == np.float32
        assert c.shape == (k, S, S, 3) and c.dtype == np.uint8
        assert m.shape == (k, 2, 3) and m.dtype == np.float64
        assert np.array_equal(p, points[i, :k]) and np.array_equal(m, M[i, :k])
    assert np.array_equal(res[1][2], chips[:2]) and np.array_equal(res[2][2], chips[2:5])
    # copies: the caller may keep them while the buffers are reused
    res[1][1][:] = 0
    assert not np.array_equal(points[1, :2], 0)
