"""FaceDetector's host-frame upload without a GPU: the rows it sends for a letterbox (letterbox_rows, host_upload_rows)
are every row cv2.resize reads, so overwriting all the others leaves the resized image byte for byte the same; the row
pairs are used exactly when they are fewer rows than the frame; and skps_det_src's layout in Python matches the header."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
INPUTS = [(384, 640), (768, 1280), (1152, 1920)]


def _fd():
    from peppa_pig_face_landmark_b200.core.api import face_detector
    return face_detector


def _sizes(seed, n):
    """n seeded (H, W) from 32x32 to 4000x6000, log-uniform per side, either orientation."""
    rng = np.random.default_rng(seed)
    h = np.exp(rng.uniform(np.log(32), np.log(6000), n)).astype(int)
    w = np.exp(rng.uniform(np.log(32), np.log(6000), n)).astype(int)
    return [(int(min(a, 4000) if i % 2 else a), int(b)) for i, (a, b) in enumerate(zip(h, w))]


@pytest.mark.parametrize("in_hw", INPUTS, ids=lambda hw: "%dx%d" % hw)
def test_rows_not_uploaded_do_not_change_the_resize(in_hw):
    """cv2 is the oracle: resize the frame, then fill every row letterbox_rows does not list with noise and resize again.
    Frames whose letterbox does not fill the input (letterbox_geometry refuses them) are skipped."""
    import cv2
    fd = _fd()
    rng = np.random.default_rng(in_hw[0])
    done = pairs = 0
    for H, W in _sizes(in_hw[1], 120) + [(2160, 3840), (1080, 1920), (3000, 4000), (4000, 3000), (6000, 4000)]:
        try:
            _, rw, rh, _, _ = fd.letterbox_geometry(H, W, *in_hw)
        except ValueError:
            continue
        rows = fd.letterbox_rows(H, rh)
        assert rows.shape == (2 * rh,) and rows.min() >= 0 and rows.max() < H
        frame = np.frombuffer(rng.bytes(H * W * 3), np.uint8).reshape(H, W, 3).copy()
        want = cv2.resize(frame, (rw, rh))
        other = np.ones(H, bool)
        other[rows] = False
        frame[other] = np.frombuffer(rng.bytes(int(other.sum()) * W * 3), np.uint8).reshape(-1, W, 3)
        got = cv2.resize(frame, (rw, rh))
        assert np.array_equal(got, want), (H, W, in_hw)
        done += 1
        pairs += fd.host_upload_rows(H, rh) is not None
    assert done >= 80 and pairs >= 20, (done, pairs)


def test_row_pairs_exactly_when_fewer_rows_than_the_frame():
    fd = _fd()
    seen = set()
    for in_hw in INPUTS:
        for H, W in _sizes(7, 400):
            try:
                _, rw, rh, _, _ = fd.letterbox_geometry(H, W, *in_hw)
            except ValueError:
                continue
            rows = fd.host_upload_rows(H, rh)
            assert (rows is not None) == (2 * rh < H), (H, W, in_hw)
            if rows is not None:
                assert np.array_equal(rows, fd.letterbox_rows(H, rh))
            seen.add(rows is None)
    assert seen == {True, False}


@pytest.mark.parametrize("frame_hw,in_hw,rows,mb", [
    ((2160, 3840), (384, 640), 720, 8.29), ((1080, 1920), (384, 640), 720, 4.15), ((3000, 4000), (384, 640), 768, 9.22),
    ((640, 640), (384, 640), None, None), ((2160, 3840), (1152, 1920), None, None)])
def test_upload_bytes(frame_hw, in_hw, rows, mb):
    """The bytes a host frame sends: the row pairs of a large frame, the whole frame otherwise."""
    fd = _fd()
    H, W = frame_hw
    _, rw, rh, _, _ = fd.letterbox_geometry(H, W, *in_hw)
    got = fd.host_upload_rows(H, rh)
    if rows is None:
        assert got is None
        return
    assert len(got) == rows
    assert round(len(got) * 3 * W / 1e6, 2) == mb
    whole = {(2160, 3840): 24.88, (1080, 1920): 6.22, (3000, 4000): 36.0}[frame_hw]
    assert round(H * 3 * W / 1e6, 2) == whole


def test_det_src_layout_matches_the_header():
    fd = _fd()
    with open(os.path.join(ROOT, "include", "skps_b200.h")) as f:
        hdr = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    body = re.search(r"typedef struct skps_det_src \{(.*?)\} skps_det_src;", hdr, re.S).group(1)
    fields = []
    for ctype, names in re.findall(r"([\w\s\*]+?)\s+(\w+(?:\s*,\s*\w+)*);", body):
        fields += [(n.strip(), "ptr" if "*" in ctype else ctype.split()[-1]) for n in names.split(",")]
    assert [n for n, _ in fields] == list(fd.DET_SRC.names)
    assert all((t == "ptr") == (fd.DET_SRC[n] == np.dtype("<u8")) for n, t in fields)
    assert all(t in ("ptr", "int32_t") for _, t in fields)
    assert fd.DET_SRC.itemsize == 8 + 4 * (len(fields) - 1)
