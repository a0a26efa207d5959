"""Aligned face chips, CPU side: the oracle's restatement of OpenCV's warpAffine arithmetic equals the installed cv2 bit for
bit (so a kernel mismatch on the GPU is a kernel bug, not an OpenCV change), its Umeyama estimate recovers a known
similarity, the five landmark indices sit where the template expects them, and the Python API rejects bad input before it
touches the GPU."""
import math

import numpy as np
import pytest

from oracle import align_ref as A


def random_affine(rng, H, W, size, where, shear):
    """A frame -> chip affine with scale 0.1..3 (chip px per frame px) and any rotation, whose chip centre maps to a frame
    point inside the frame, near an edge (chip partly outside) or far outside it.  shear adds an off-diagonal term."""
    s = rng.uniform(0.1, 3.0)
    th = rng.uniform(-math.pi, math.pi)
    Am = s * np.array([[math.cos(th), -math.sin(th)], [math.sin(th), math.cos(th)]])
    if shear:
        Am = Am @ np.array([[1.0, rng.uniform(-0.6, 0.6)], [rng.uniform(-0.6, 0.6), 1.0]])
    reach = size / np.linalg.svd(Am, compute_uv=False).min()          # frame px the chip spans at most
    if where == "inside":
        c = np.array([rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H])
    elif where == "partial":
        if rng.integers(2):
            c = np.array([rng.choice([0.0, W - 1.0]) + rng.uniform(-0.3, 0.3) * reach, rng.uniform(0, H)])
        else:
            c = np.array([rng.uniform(0, W), rng.choice([0.0, H - 1.0]) + rng.uniform(-0.3, 0.3) * reach])
    else:
        c = np.array([rng.choice([-1.0, 1.0]) * (W + 2 * reach), rng.uniform(-H, 2 * H)])
    t = np.array([size / 2.0, size / 2.0]) - Am @ c
    return np.hstack([Am, t[:, None]])


FRAMES = [(480, 640), (1080, 1920), (481, 1283)]


@pytest.fixture(scope="module")
def noise_frames():
    rng = np.random.default_rng(7)
    return {hw: rng.integers(0, 256, hw + (3,), dtype=np.uint8) for hw in FRAMES}


@pytest.mark.parametrize("hw", FRAMES)
@pytest.mark.parametrize("size", [112, 224])
def test_warp_restatement_equals_cv2(noise_frames, hw, size):
    import cv2
    img = noise_frames[hw]
    rng = np.random.default_rng(hw[1] * 1000 + size)
    n = 0
    for where in ("inside", "partial", "outside"):
        for shear in (False, True):
            for _ in range(3):
                M = random_affine(rng, hw[0], hw[1], size, where, shear)
                ref = cv2.warpAffine(img, M, (size, size), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT,
                                     borderValue=0)
                got = A.warp_affine_u8(img, M, (size, size))
                assert np.array_equal(ref, got), (where, shear, M, int((ref != got).sum()))
                if where == "outside":
                    assert not ref.any()
                n += 1
    assert n == 18          # x 6 parametrisations = 108 matrices


def test_umeyama_recovers_a_known_similarity():
    rng = np.random.default_rng(3)
    for _ in range(50):
        src = rng.uniform(0, 1000, (5, 2))
        c, th = rng.uniform(0.05, 5), rng.uniform(-math.pi, math.pi)
        R = np.array([[math.cos(th), -math.sin(th)], [math.sin(th), math.cos(th)]])
        t = rng.uniform(-500, 500, 2)
        dst = c * src @ R.T + t
        M = A.umeyama(src, dst)
        want = np.hstack([c * R, t[:, None]])
        assert np.abs(M - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


def test_five_point_indices_on_golden_landmarks(golden):
    g = golden("test1")
    for kps in (g["f0_kps_raw"].reshape(98, 2), g["f0_res_kps"][0]):
        le, re, nose, lm, rm = (kps[i] for i in A.WFLW98_FIVE)
        assert le[0] < re[0] and lm[0] < rm[0]                         # left / right as seen in the image
        assert le[0] < nose[0] < re[0]
        assert max(le[1], re[1]) < nose[1] < min(lm[1], rm[1])         # eyes above the nose above the mouth
    M = A.align_matrix(g["f0_res_kps"][0], 112)
    assert np.linalg.det(M[:, :2]) > 0                                # a similarity without reflection


def test_library_constants_match_the_oracle():
    from peppa_pig_face_landmark_b200.core.api import align
    assert np.array_equal(align.ARCFACE_TEMPLATE_112, A.ARCFACE_TEMPLATE_112)
    assert tuple(align.WFLW98_FIVE) == tuple(A.WFLW98_FIVE)


def test_bad_inputs_raise_value_error():
    from peppa_pig_face_landmark_b200.core.api.align import align_faces, warp_affine
    from Skps import FaceAna, FaceAnaStreams
    img = np.zeros((64, 80, 3), np.uint8)
    kps = np.tile(np.arange(196, dtype=np.float64).reshape(1, 98, 2), (2, 1, 1))
    M = np.tile(np.array([[1.0, 0, 0], [0, 1, 0]]), (3, 1, 1))
    bad_calls = [
        lambda: warp_affine(img[..., :2], M, (32, 32)),
        lambda: warp_affine(img.astype(np.float32), M, (32, 32)),
        lambda: warp_affine(img[0], M, (32, 32)),
        lambda: warp_affine(img, M[0], (32, 32)),
        lambda: warp_affine(img, np.zeros((3, 3, 3)), (32, 32)),
        lambda: warp_affine(img, M * np.nan, (32, 32)),
        lambda: warp_affine(img, M, (0, 32)),
        lambda: warp_affine(img, M, 32),
        lambda: align_faces(img.astype(np.int16), kps),
        lambda: align_faces(img, kps[0]),
        lambda: align_faces(img, kps[:, :68]),
        lambda: align_faces(img, np.where(np.arange(98)[None, :, None] == 54, np.inf, kps)),
        lambda: align_faces(img, np.ones((2, 98, 2))),                      # zero spread
        lambda: align_faces(img, kps, size=15),
        lambda: align_faces(img, kps, size=513),
        lambda: align_faces(img, kps, size=112.0),
        lambda: align_faces(img, kps, size=True),
        lambda: FaceAna(align=8),
        lambda: FaceAnaStreams(n_streams=2, align=1024),
    ]
    for i, call in enumerate(bad_calls):
        with pytest.raises(ValueError):
            call()
