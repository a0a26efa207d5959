"""Frame layouts without a GPU: the pure check device_frames.frame_layout on shapes and strides (in bytes of a uint8
frame), the layout= check of host frames, the skps_frame_layout dtype against include/skps_b200.h, and the arity of the
new entry points next to the ones they extend."""
import os
import re

import numpy as np
import pytest

from test_c_abi_cpu import _header_arity

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
INTERLEAVED = {"bgr": 3, "rgb": 3, "bgra": 4, "rgba": 4}
PLANAR = ["bgr_planar", "rgb_planar"]


def _fl(shape, strides, layout):
    from peppa_pig_face_landmark_b200.core.api.device_frames import frame_layout
    return frame_layout(shape, strides, layout)


def _view(base_shape, index):
    """shape and strides (bytes) of a view of a C-contiguous uint8 buffer, as numpy gives them."""
    strides = tuple(int(np.prod(base_shape[i + 1:])) for i in range(len(base_shape)))
    v = np.lib.stride_tricks.as_strided(np.zeros(1, np.uint8), base_shape, strides)[index]
    return v.shape, v.strides


def test_layout_codes_match_the_header():
    from peppa_pig_face_landmark_b200.core.api.device_frames import LAYOUTS
    with open(os.path.join(ROOT, "include", "skps_b200.h")) as f:
        hdr = f.read()
    codes = {k.lower(): int(v) for k, v in re.findall(r"SKPS_LAYOUT_(\w+)\s*=\s*(\d+)", hdr)}
    assert codes == LAYOUTS
    assert LAYOUTS["bgr"] == 0


@pytest.mark.parametrize("layout", list(INTERLEAVED))
@pytest.mark.parametrize("H, W, pad, x0", [(4, 5, 0, 0), (6, 7, 3, 2), (1, 9, 0, 0), (5, 1, 0, 0), (2160, 3840, 16, 1)])
def test_interleaved_packed_pitched_and_roi(layout, H, W, pad, x0):
    C = INTERLEAVED[layout]
    shape, strides = _view((H + 2, W + pad + x0, C), (slice(1, 1 + H), slice(x0, x0 + W)))
    fl = _fl(shape, strides, layout)
    assert (fl.H, fl.W, fl.pitch, fl.plane) == (H, W, C * (W + pad + x0) if H > 1 else C * W, 0)
    from peppa_pig_face_landmark_b200.core.api.device_frames import LAYOUTS
    assert fl.code == LAYOUTS[layout]


@pytest.mark.parametrize("layout", PLANAR)
def test_planar_views(layout):
    H, W = 6, 11
    # packed (3, H, W)
    fl = _fl((3, H, W), (H * W, W, 1), layout)
    assert (fl.H, fl.W, fl.pitch, fl.plane) == (H, W, W, H * W)
    # an ROI of (3, H', W'): plane pitch H' W', not H * pitch
    shape, strides = _view((3, H + 4, W + 5), (slice(None), slice(2, 2 + H), slice(3, 3 + W)))
    fl = _fl(shape, strides, layout)
    assert (fl.H, fl.W, fl.pitch, fl.plane) == (H, W, W + 5, (H + 4) * (W + 5))
    # image 2 of an (N, 3, H, W) batch, and every other plane of a (5, H, W) buffer
    shape, strides = _view((4, 3, H, W), (2,))
    assert tuple(_fl(shape, strides, layout))[:4] == (H, W, W, H * W)
    shape, strides = _view((5, H, W), (slice(None, None, 2),))
    assert tuple(_fl(shape, strides, layout))[:4] == (H, W, W, 2 * H * W)
    # one row: any row stride; one column: any column stride
    assert tuple(_fl((3, 1, W), (W, 12345, 1), layout))[:4] == (1, W, W, W)
    assert tuple(_fl((3, H, 1), (H * 7, 7, 5), layout))[:4] == (H, 1, 7, H * 7)
    # three planes at the same place (a grey frame broadcast) are planes too
    assert _fl((3, H, W), (0, W, 1), layout).plane == 0


@pytest.mark.parametrize("layout", list(INTERLEAVED))
def test_interleaved_one_row_and_one_column(layout):
    C = INTERLEAVED[layout]
    assert tuple(_fl((1, 7, C), (999, C, 1), layout))[:3] == (1, 7, 7 * C)
    assert tuple(_fl((5, 1, C), (C * 9, 77, 1), layout))[:3] == (5, 1, C * 9)


@pytest.mark.parametrize("shape, strides, layout, words", [
    ((4, 5, 4), (20, 4, 1), "bgr", "(H, W, 3)"),                # wrong channel count
    ((4, 5, 3), (15, 3, 1), "bgra", "(H, W, 4)"),
    ((4, 5, 3), (15, 3, 1), "rgba", "(H, W, 4)"),
    ((4, 3, 5), (15, 5, 1), "bgr_planar", "(3, H, W)"),
    ((3, 4, 5), (20, 5, 1), "rgb", "rgb_planar"),               # a planar tensor passed as interleaved
    ((4, 5, 3), (15, 1, 5), "rgb", "interleaved"),              # stride(2) != 1
    ((3, 4, 5), (20, 5, 2), "rgb_planar", "strides"),
    ((4, 5, 3), (14, 3, 1), "bgr", "strides"),                  # a short row stride
    ((4, 5, 4), (19, 4, 1), "rgba", "strides"),
    ((3, 4, 5), (20, 4, 1), "bgr_planar", "strides"),
    ((3, 4, 5), (1, 15, 3), "rgb_planar", "interleaved layout"),   # t.permute(2, 0, 1) of a packed (4, 5, 3) tensor
    ((3, 4, 5), (-20, 5, 1), "bgr_planar", "strides"),          # planes at a negative distance
    ((4, 5), (5, 1), "bgr", "3-d"),
    ((0, 5, 3), (15, 3, 1), "bgr", "empty"),
    ((3, 2, 0), (0, 0, 1), "rgb_planar", "empty"),
    ((2, 2 ** 30, 3), (3 * 2 ** 30, 3, 1), "rgb", "32 bits"),   # row pitch 3 * 2**30
    ((3, 2, 8), (2 ** 31, 8, 1), "bgr_planar", "32 bits"),      # plane pitch 2**31
])
def test_refused_shapes_and_strides(shape, strides, layout, words):
    with pytest.raises(ValueError, match=re.escape(words)):
        _fl(shape, strides, layout)


@pytest.mark.parametrize("layout", ["BGR", "yuv", "nv12", "", "rgb ", "planar", None, 0, 3, b"bgr", ("bgr",)])
def test_refused_layouts(layout):
    from peppa_pig_face_landmark_b200.core.api.device_frames import check_layout
    with pytest.raises(ValueError, match="layout"):
        _fl((4, 5, 3), (15, 3, 1), layout)
    with pytest.raises(ValueError, match="layout"):
        check_layout(layout)


@pytest.mark.parametrize("layout", ["rgb", "bgra", "rgba", "bgr_planar", "rgb_planar"])
def test_host_frames_take_bgr_only(layout):
    from peppa_pig_face_landmark_b200.core.api.device_frames import check_layout
    from peppa_pig_face_landmark_b200.core.api.staging import check_frames
    assert check_layout("bgr", cuda=False) == 0
    with pytest.raises(ValueError, match="host frames"):
        check_layout(layout, cuda=False)
    with pytest.raises(ValueError, match="host frames"):
        check_frames([np.zeros((4, 5, 3), np.uint8)], "cuda", layout)
    call = check_frames([np.zeros((4, 5, 3), np.uint8)], "cuda")
    assert tuple(call.shapes[0]) == (4, 5, 15, 0, 0)


def _struct_fields(name):
    with open(os.path.join(ROOT, "include", "skps_b200.h")) as f:
        hdr = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), hdr, re.S).group(1)
    fields = []
    for ctype, names in re.findall(r"([\w\s\*]+?)\s+(\w+(?:\s*,\s*\w+)*);", body):
        fields += [(n.strip(), "ptr" if "*" in ctype else ctype.split()[-1]) for n in names.split(",")]
    return fields


def test_frame_layout_matches_the_header_and_zero_is_bgr():
    from peppa_pig_face_landmark_b200.core.api.device_frames import FRAME_LAYOUT
    fields = _struct_fields("skps_frame_layout")
    assert fields == [(n, "int32_t") for n in FRAME_LAYOUT.names]
    assert FRAME_LAYOUT.itemsize == 4 * len(fields) and all(FRAME_LAYOUT[n] == np.dtype("<i4") for n in FRAME_LAYOUT.names)
    z = np.zeros(1, FRAME_LAYOUT)
    assert int(z["layout"][0]) == 0 and int(z["plane_pitch"][0]) == 0      # a zeroed entry is a BGR frame


def test_frame_descriptors_keep_their_layout():
    """The layout travels beside skps_det_src / skps_face_src, which keep their fields and sizes."""
    from peppa_pig_face_landmark_b200.core.api.face_detector import DET_SRC
    from peppa_pig_face_landmark_b200.core.api.face_landmark import FACE_SRC
    assert [n for n, _ in _struct_fields("skps_det_src")] == list(DET_SRC.names) and DET_SRC.itemsize == 40
    assert [n for n, _ in _struct_fields("skps_face_src")] == list(FACE_SRC.names) and FACE_SRC.itemsize == 40


def test_layout_entry_points_arity():
    from peppa_pig_face_landmark_b200 import runtime
    arity = _header_arity()
    want = {"skps_frame_ingest_layout": 10, "skps_pipeline_frame_diff_device_layout": 10,
            "skps_mpipe_submit_device_layout": 11, "skps_letterbox_frames_layout": 7, "skps_crop_faces_layout": 10,
            "skps_warp_faces_layout": 8, "skps_letterbox_frames": 6, "skps_crop_faces": 9, "skps_warp_faces": 7,
            # the entries they extend keep their signatures
            "skps_frame_ingest": 8, "skps_pipeline_frame_diff_device": 8, "skps_mpipe_submit_device": 8,
            "skps_mpipe_submit_device_streams": 9}
    for name, n in want.items():
        assert arity[name] == n == len(runtime.SIGNATURES[name][1]), name
