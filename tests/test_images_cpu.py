"""FaceAnaImages without a GPU: the kernels it adds compile for sm_90a without spilling, and the host-side packing of a
call's faces (first / count per image, the face -> image map, the capacity check of out=) agrees with plain numpy."""
import re

import numpy as np
import pytest

from test_image_ops_codegen import _kernels
from test_wgmma_codegen import _ptxas_report

SPILL = r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"


def _spills(src):
    out = _ptxas_report(src)
    return out, {name: (st, ld) for name, st, ld in re.findall(SPILL, out)}


def test_landmark_boxes_selection_and_pose_kernels_do_not_spill():
    out, sp = _spills("image_ops.cu")
    names = _kernels(out)
    assert "landmark_boxes_kernel" in names and "select_frames_kernel" in names, names
    for kernel in ("landmark_boxes_kernel", "select_frames_kernel"):
        mangled = [m for m in sp if kernel in m]
        assert mangled and all(sp[m] == ("0", "0") for m in mangled), (kernel, {m: sp[m] for m in mangled})
    _, sp = _spills("headpose.cu")
    pose = [m for m in sp if "head_pose" in m]
    assert pose and all(sp[m] == ("0", "0") for m in pose), {m: sp[m] for m in pose}


def _numpy_packing(counts):
    first, face_image, o = [], [], 0
    for i, k in enumerate(counts):
        first.append(o)
        face_image += [i] * k
        o += k
    return np.array(first, np.int32), np.array(face_image, np.int32)


@pytest.mark.parametrize("top_k", [1, 5, 16, 1024])
def test_packing_equals_numpy(top_k):
    from peppa_pig_face_landmark_b200.core.api.images import pack_faces
    rng = np.random.default_rng(top_k)
    for n in (0, 1, 2, 7, 40, 300):
        counts = rng.integers(0, top_k + 1, n)
        counts[rng.random(n) < 0.3] = 0                                 # images without a face
        first, face_image = pack_faces(counts)
        wf, wi = _numpy_packing(counts.tolist())
        assert first.dtype == face_image.dtype == np.int32
        assert np.array_equal(first, wf) and np.array_equal(face_image, wi), (top_k, n)
        assert len(face_image) == counts.sum() <= n * top_k
        for i, k in enumerate(counts.tolist()):                          # image i's rows, and only those
            assert np.all(face_image[first[i]:first[i] + k] == i)
    first, face_image = pack_faces([top_k] * 3)
    assert first.tolist() == [0, top_k, 2 * top_k] and len(face_image) == 3 * top_k
