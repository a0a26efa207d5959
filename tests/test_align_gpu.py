"""Aligned face chips on the GPU (csrc/align.cu): warp_affine is cv2.warpAffine byte for byte, align_faces' matrices are the
oracle's Umeyama estimate, and FaceAna / FaceAnaStreams with align=size add a 'chip' and an 'M' to every face without
changing anything else they return.  Chips are always compared with cv2.warpAffine under the library's own M: a 1e-13
difference in M may move a rounding and so a pixel."""
import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames
from oracle import align_ref as A
from test_align_oracle import random_affine
from test_streams_gpu import _sequences

pytestmark = pytest.mark.gpu


def cv2_warp(img, M, size):
    import cv2
    return cv2.warpAffine(img, np.asarray(M, np.float64), (size, size), flags=cv2.INTER_LINEAR,
                          borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def check_faces(frame, res, size):
    """Every face: 'chip' == cv2.warpAffine(frame, 'M'), 'M' == the oracle's estimate from the returned 'kps'."""
    for r in res:
        assert r['chip'].shape == (size, size, 3) and r['chip'].dtype == np.uint8
        assert r['M'].shape == (2, 3) and r['M'].dtype == np.float64
        want = A.align_matrix(np.asarray(r['kps'], np.float64), size)
        assert np.abs(r['M'] - want).max() <= 1e-9 * np.abs(want).max()
        assert np.array_equal(r['chip'], cv2_warp(frame, r['M'], size))


@pytest.mark.parametrize("hw", [(480, 640), (1080, 1920), (2160, 3840)])
@pytest.mark.parametrize("size", [112, 224])
def test_warp_affine_equals_cv2(hw, size):
    from peppa_pig_face_landmark_b200.core.api.align import warp_affine
    rng = np.random.default_rng(hw[0] + size)
    img = rng.integers(0, 256, hw + (3,), dtype=np.uint8)
    kinds = [(w, s) for w in ("inside", "partial", "outside") for s in (False, True)]
    for n in (1, 7, 64):
        Ms = np.stack([random_affine(rng, hw[0], hw[1], size, *kinds[i % len(kinds)]) for i in range(n)])
        got = warp_affine(img, Ms, (size, size))
        assert got.shape == (n, size, size, 3)
        for i in range(n):
            ref = cv2_warp(img, Ms[i], size)
            assert np.array_equal(got[i], ref), (n, i, kinds[i % len(kinds)], int((got[i] != ref).sum()))


def test_warp_affine_non_square_output():
    from peppa_pig_face_landmark_b200.core.api.align import warp_affine
    import cv2
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (301, 517, 3), dtype=np.uint8)
    Ms = np.stack([random_affine(rng, 301, 517, 96, "inside", True) for _ in range(4)])
    got = warp_affine(img, Ms, (96, 40))
    for i in range(4):
        assert np.array_equal(got[i], cv2.warpAffine(img, Ms[i], (96, 40)))


@pytest.mark.parametrize("size", [112, 224, 16, 512])
def test_align_faces_matches_oracle_and_cv2(golden, size):
    from peppa_pig_face_landmark_b200.core.api.align import align_faces
    img = frames.frame_4k()
    base = golden("test1")["f0_res_kps"][0].astype(np.float64)
    rng = np.random.default_rng(size)
    kps = []
    for _ in range(24):             # the golden face moved, scaled and turned over the 4K frame (some past its edges)
        th, s = rng.uniform(-np.pi, np.pi), rng.uniform(0.3, 4.0)
        R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
        c = base.mean(0)
        kps.append((base - c) @ R.T * s + rng.uniform([-200, -200], [4040, 2360]) + rng.normal(0, 0.7, base.shape))
    kps = np.stack(kps)
    chips, M = align_faces(img, kps, size)
    assert chips.shape == (24, size, size, 3) and M.shape == (24, 2, 3)
    for i in range(24):
        want = A.align_matrix(kps[i], size)
        assert np.abs(M[i] - want).max() <= 1e-9 * np.abs(want).max()
        assert np.array_equal(chips[i], cv2_warp(img, M[i], size))


def _golden_sequences():
    return {"test1": [frames.load_test1()], "canvas640": [frames.canvas_640()], "video1080": video_frames(),
            "uhd4k_top16": [frames.frame_4k()]}


@pytest.mark.parametrize("size", [112, 224])
@pytest.mark.parametrize("name", ["test1", "canvas640", "video1080", "uhd4k_top16"])
def test_faceana_align_adds_chips_and_changes_nothing_else(name, size):
    from Skps import FaceAna
    top_k = 16 if name == "uhd4k_top16" else None
    plain, aligned = FaceAna(top_k=top_k), FaceAna(top_k=top_k, align=size)
    n_faces = 0
    for fr in _golden_sequences()[name]:
        a, b = plain.run(fr), aligned.run(fr)
        assert len(a) == len(b)
        for x, y in zip(a, b):
            assert set(x) == {'box', 'kps', 'scores'} and set(y) == {'box', 'kps', 'scores', 'chip', 'M'}
            for k in ('box', 'kps', 'scores'):
                assert np.array_equal(x[k], y[k]) and np.asarray(x[k]).dtype == np.asarray(y[k]).dtype
        check_faces(fr, b, size)
        n_faces += len(b)
    assert n_faces > 0


def test_streams_align_matches_cv2_and_unaligned_streams():
    from Skps import FaceAnaStreams
    seqs = _sequences()
    S = len(seqs)
    plain, aligned = FaceAnaStreams(n_streams=S), FaceAnaStreams(n_streams=S, align=112)

    def same_and_checked(batch, a, b):
        for s, (x, y) in enumerate(zip(a, b)):
            assert len(x) == len(y)
            for u, v in zip(x, y):
                for k in ('box', 'kps', 'scores'):
                    assert np.array_equal(u[k], v[k])
            check_faces(batch[s], y, 112)
        return sum(len(y) for y in b)

    # two batches in flight on the aligned object, blocking runs on the plain one
    batches = [[s[t] for s in seqs] for t in range(6)]
    want = [plain.run(b) for b in batches]
    got = []
    aligned.submit(batches[0])
    for t in range(1, 6):
        aligned.submit(batches[t])
        got.append(aligned.collect())
    got.append(aligned.collect())
    n = sum(same_and_checked(batches[t], want[t], got[t]) for t in range(6))
    assert n > 0
    # reset one stream, then a partial batch (streams 0 and 1 only)
    v = video_frames()
    plain.reset(1); aligned.reset(1)
    part = [v[1], v[0]]
    n = same_and_checked(part, plain.run(part), aligned.run(part))
    assert n > 0 and list(aligned.last_ran_detector) == list(plain.last_ran_detector)
