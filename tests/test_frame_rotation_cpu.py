"""Frames stored turned, without a GPU: the rotate= check (device_frames.check_rotate) and the upright size
(device_frames.upright_shape) on shapes and strides of every layout, the refusals of the shared frame check, and the arity
of the *_rotate entry points next to the entries they extend, whose signatures and structs stay as they were."""
import numpy as np
import pytest

from test_c_abi_cpu import _header_arity
from test_frame_layouts_cpu import INTERLEAVED, PLANAR, _view


def _api():
    from peppa_pig_face_landmark_b200.core.api import device_frames
    return device_frames


@pytest.mark.parametrize("rotate, turns", [(0, 0), (90, 1), (180, 2), (270, 3), (np.int64(90), 1), (np.int32(270), 3)])
def test_rotate_values(rotate, turns):
    assert _api().check_rotate(rotate) == turns
    assert _api().check_rotate(rotate, 3) == [turns] * 3


def test_rotate_per_frame():
    cr = _api().check_rotate
    assert cr([0, 90, 180, 270], 4) == [0, 1, 2, 3]
    assert cr((270,), 1) == [3]
    assert cr(np.array([90, 0]), 2) == [1, 0]
    assert cr([], 0) == []
    assert cr([0, 0], 2, cuda=False) == [0, 0]


@pytest.mark.parametrize("rotate", [45, -90, 360, 1, 3, True, False, 90.0, "90", None, b"90", 90 + 0j, np.bool_(True)])
def test_refused_rotate_values(rotate):
    with pytest.raises(ValueError, match=r"rotate: expected one of 0, 90, 180, 270"):
        _api().check_rotate(rotate)
    with pytest.raises(ValueError, match=r"rotate"):
        _api().check_rotate(rotate, 2)
    with pytest.raises(ValueError, match=r"rotate"):
        _api().check_rotate([0, rotate], 2)


@pytest.mark.parametrize("rotate, n", [([0, 90], 3), ([90], 2), ([], 1), ((0, 90, 180), 2)])
def test_refused_rotate_lengths(rotate, n):
    with pytest.raises(ValueError, match=r"one value or one per frame \(%d\)" % n):
        _api().check_rotate(rotate, n)


@pytest.mark.parametrize("rotate", [90, 180, 270, [0, 90]])
def test_host_frames_take_no_turn(rotate):
    from peppa_pig_face_landmark_b200.core.api.staging import check_frames
    with pytest.raises(ValueError, match="host frames are upright"):
        _api().check_rotate(rotate, 2, cuda=False)
    frames = [np.zeros((4, 5, 3), np.uint8)] * 2
    with pytest.raises(ValueError, match="host frames are upright"):
        check_frames(frames, "cuda", "bgr", rotate)
    call = check_frames(frames, "cuda", "bgr", 0)
    assert call.turns == [0, 0] and not call.turned and call.upright == [(4, 5), (4, 5)]
    assert tuple(call.shapes[0]) == (4, 5, 15, 0, 0)


def test_shared_check_refuses_before_anything():
    from peppa_pig_face_landmark_b200.core.api.staging import check_frames
    with pytest.raises(ValueError, match="rotate"):
        check_frames([np.zeros((4, 5, 3), np.uint8)], "cuda", "bgr", [0, 90])
    with pytest.raises(ValueError, match="rotate"):
        check_frames([np.zeros((4, 5, 3), np.uint8)], "cuda", "bgr", True)
    assert check_frames([], "cuda", "bgr", []).turns == []


@pytest.mark.parametrize("rotate", [0, 90, 180, 270])
@pytest.mark.parametrize("layout", list(INTERLEAVED))
@pytest.mark.parametrize("H, W, pad, x0", [(4, 5, 0, 0), (6, 7, 3, 2), (1, 9, 0, 0), (5, 1, 0, 0), (1, 1, 0, 0),
                                           (1080, 1920, 64, 3)])
def test_upright_shape_interleaved(rotate, layout, H, W, pad, x0):
    C = INTERLEAVED[layout]
    shape, strides = _view((H + 2, W + pad + x0, C), (slice(1, 1 + H), slice(x0, x0 + W)))
    want = (W, H) if rotate in (90, 270) else (H, W)
    assert _api().upright_shape(shape, strides, layout, rotate) == want
    assert _api().upright_hw(H, W, rotate // 90) == want


@pytest.mark.parametrize("rotate", [0, 90, 180, 270])
@pytest.mark.parametrize("layout", PLANAR)
def test_upright_shape_planar(rotate, layout):
    H, W = 6, 11
    odd = rotate in (90, 270)
    for shape, strides in [((3, H, W), (H * W, W, 1)),
                           _view((3, H + 4, W + 5), (slice(None), slice(2, 2 + H), slice(3, 3 + W))),
                           ((3, 1, W), (W, 12345, 1)), ((3, H, 1), (H * 7, 7, 5))]:
        h, w = shape[1], shape[2]
        assert _api().upright_shape(shape, strides, layout, rotate) == ((w, h) if odd else (h, w))


def test_upright_shape_refusals():
    with pytest.raises(ValueError, match="rotate"):
        _api().upright_shape((4, 5, 3), (15, 3, 1), "bgr", 45)
    with pytest.raises(ValueError, match="strides"):
        _api().upright_shape((4, 5, 3), (14, 3, 1), "bgr", 90)


def test_rotate_entry_points_arity():
    from peppa_pig_face_landmark_b200 import runtime
    arity = _header_arity()
    want = {"skps_frame_ingest_rotate": 11, "skps_pipeline_frame_diff_device_rotate": 11,
            "skps_mpipe_submit_device_rotate": 12, "skps_letterbox_frames_rotate": 8, "skps_crop_faces_rotate": 11,
            "skps_warp_faces_rotate": 9, "skps_warp_faces_count_rotate": 11}
    for name, n in want.items():
        assert arity[name] == n == len(runtime.SIGNATURES[name][1]), name


def test_existing_entry_points_and_structs_unchanged():
    from peppa_pig_face_landmark_b200 import runtime
    from test_frame_layouts_cpu import _struct_fields
    arity = _header_arity()
    want = {"skps_frame_ingest_layout": 10, "skps_pipeline_frame_diff_device_layout": 10,
            "skps_mpipe_submit_device_layout": 11, "skps_letterbox_frames_layout": 7, "skps_crop_faces_layout": 10,
            "skps_warp_faces_layout": 8, "skps_warp_faces_count": 10, "skps_letterbox_frames": 6, "skps_crop_faces": 9,
            "skps_warp_faces": 7, "skps_frame_ingest": 8, "skps_pipeline_frame_diff_device": 8,
            "skps_mpipe_submit_device": 8, "skps_mpipe_submit_device_streams": 9}
    for name, n in want.items():
        assert arity[name] == n == len(runtime.SIGNATURES[name][1]), name
    assert [n for n, _ in _struct_fields("skps_frame_layout")] == ["layout", "plane_pitch"]
    from peppa_pig_face_landmark_b200.core.api.face_detector import DET_SRC
    from peppa_pig_face_landmark_b200.core.api.face_landmark import FACE_SRC
    assert DET_SRC.itemsize == FACE_SRC.itemsize == 40
