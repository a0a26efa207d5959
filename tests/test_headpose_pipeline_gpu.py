"""Head pose of every face (csrc/headpose.cu): the 98-point get_head_pose of the reference's training tree
(TRAIN/face_landmark/lib/dataset/headpose.py:48-78) against cv2, a face's pose independent of the batch it is solved in,
and FaceAna(pose=True) / FaceAnaStreams(pose=True) adding a 'pose' to every face without changing anything else.
Tolerances as in test_headpose_gpu: Euler 1e-3 degrees, cube corners 1e-2 px, rotation matrix 1e-5, tvec 1e-2."""
import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames
from test_align_gpu import _golden_sequences, check_faces
from test_headpose_gpu import _synthetic_shapes
from test_streams_gpu import _sequences

pytestmark = pytest.mark.gpu


def _reference_pose_98(shape, img_hw):
    """headpose.py:48-78 in behaviour: the same cv2 calls on the 98-point indices."""
    import cv2
    from peppa_pig_face_landmark_b200.core.headpose.pose import POSE_POINTS_98, object_pts, reprojectsrc
    h, w = img_hw
    cam = np.array([w, 0.0, w // 2, 0.0, w, h // 2, 0.0, 0.0, 1.0]).reshape(3, 3).astype(np.float32)
    dist = np.zeros((5, 1), np.float32)
    image_pts = np.float32([shape[i] for i in POSE_POINTS_98])
    _, rvec, tvec = cv2.solvePnP(object_pts, image_pts, cam, dist)
    dst, _ = cv2.projectPoints(reprojectsrc, rvec, tvec, cam, dist)
    rot, _ = cv2.Rodrigues(rvec)
    euler = cv2.decomposeProjectionMatrix(cv2.hconcat((rot, tvec)))[6]
    return dst.reshape(8, 2), euler.reshape(3), rvec.reshape(3), tvec.reshape(3)


def _check_cv2(pose, shape, img_hw, what):
    import cv2
    dst, euler, rvec, tvec = _reference_pose_98(shape, img_hw)
    d = np.abs(pose["euler"] - euler)
    assert np.minimum(d, 360 - d).max() < 1e-3, (what, pose["euler"], euler)
    assert np.abs(pose["reproject"] - dst).max() < 1e-2, what
    assert np.abs(cv2.Rodrigues(pose["rvec"])[0] - cv2.Rodrigues(rvec)[0]).max() < 1e-5, what
    assert np.abs(pose["tvec"] - tvec).max() < 1e-2, what


def _shapes98(n, img_hw, seed):
    """test_headpose_gpu's synthetic faces, their 10 pose points moved to the 98-point indices."""
    from peppa_pig_face_landmark_b200.core.headpose.pose import POSE_POINTS, POSE_POINTS_98
    s68 = _synthetic_shapes(n, img_hw, seed=seed)
    rng = np.random.default_rng(seed + 1)
    s98 = rng.uniform(0, img_hw[1], (n, 98, 2)).astype(np.float32)
    s98[:, POSE_POINTS_98] = s68[:, POSE_POINTS]
    return s98


def _same_pose(a, b, what):
    for k in ("rvec", "tvec", "euler", "reproject"):
        assert a[k].dtype == np.float64 and np.array_equal(a[k], b[k]), (what, k)


def _slice(poses, i):
    return {k: v[i] for k, v in poses.items()}


@pytest.mark.parametrize("img_hw", [(480, 640), (1080, 1920)])
def test_head_poses_98_points_match_opencv(img_hw):
    from Skps.core.headpose.pose import POSE_POINTS_98, head_poses
    shapes = _shapes98(64, img_hw, seed=img_hw[1])
    got = head_poses(shapes, img_hw, points=POSE_POINTS_98)
    for i in range(len(shapes)):
        _check_cv2(_slice(got, i), shapes[i], img_hw, i)


def test_head_poses_do_not_depend_on_the_batch():
    from peppa_pig_face_landmark_b200.core.headpose.pose import POSE_POINTS_98, head_poses
    hw = (1080, 1920)
    shapes = _shapes98(1024, hw, seed=7)
    full = head_poses(shapes, hw, points=POSE_POINTS_98)
    _same_pose(full, head_poses(shapes, hw, points=POSE_POINTS_98), "second call")
    for i in range(len(shapes)):
        _same_pose(_slice(full, i), _slice(head_poses(shapes[i:i + 1], hw, points=POSE_POINTS_98), 0), i)


def test_head_poses_points_argument_is_checked():
    from peppa_pig_face_landmark_b200.core.headpose.pose import POSE_POINTS_98, head_poses
    with pytest.raises(ValueError):
        head_poses(np.zeros((2, 68, 2), np.float32), (480, 640), points=POSE_POINTS_98)
    with pytest.raises(ValueError):
        head_poses(np.zeros((2, 98, 2), np.float32), (480, 640), points=POSE_POINTS_98[:9])


@pytest.mark.parametrize("name", ["test1", "canvas640", "video1080", "uhd4k_top16"])
def test_faceana_pose_adds_pose_and_changes_nothing_else(name):
    from Skps import FaceAna
    from Skps.core.headpose.pose import POSE_POINTS_98, head_poses
    top_k = 16 if name == "uhd4k_top16" else None
    plain, posed = FaceAna(top_k=top_k), FaceAna(top_k=top_k, pose=True)
    n_faces = 0
    for fr in _golden_sequences()[name]:
        a, b = plain.run(fr), posed.run(fr)
        assert len(a) == len(b)
        for x, y in zip(a, b):
            assert set(x) == {'box', 'kps', 'scores'} and set(y) == {'box', 'kps', 'scores', 'pose'}
            for k in ('box', 'kps', 'scores'):
                assert np.array_equal(x[k], y[k]) and np.asarray(x[k]).dtype == np.asarray(y[k]).dtype
            assert set(y['pose']) == {'euler', 'rvec', 'tvec', 'reproject'}
            assert y['pose']['reproject'].shape == (8, 2) and y['pose']['euler'].shape == (3,)
            want = _slice(head_poses(np.asarray(y['kps'])[None], fr.shape[:2], points=POSE_POINTS_98), 0)
            _same_pose(y['pose'], want, name)
            _check_cv2(y['pose'], np.asarray(y['kps']), fr.shape[:2], name)
        n_faces += len(b)
    assert n_faces > 0


@pytest.mark.parametrize("align", [None, 112])
def test_streams_pose_matches_head_poses_and_plain_streams(align):
    from Skps import FaceAnaStreams
    from Skps.core.headpose.pose import POSE_POINTS_98, head_poses
    seqs = _sequences()
    S = len(seqs)
    plain, posed = FaceAnaStreams(n_streams=S), FaceAnaStreams(n_streams=S, pose=True, align=align)
    extra = {'pose'} | ({'chip', 'M'} if align else set())

    def same_and_checked(batch, a, b):
        for s, (x, y) in enumerate(zip(a, b)):
            assert len(x) == len(y)
            for u, v in zip(x, y):
                assert set(v) == set(u) | extra
                for k in ('box', 'kps', 'scores'):
                    assert np.array_equal(u[k], v[k])
                want = _slice(head_poses(v['kps'][None], batch[s].shape[:2], points=POSE_POINTS_98), 0)
                _same_pose(v['pose'], want, s)
            if align:
                check_faces(batch[s], y, align)
        return sum(len(y) for y in b)

    # two batches in flight on the posed object, blocking runs on the plain one; the streams' frames are 1080x1920,
    # 640x640 and 273x410, so each stream's camera is its own
    batches = [[s[t] for s in seqs] for t in range(6)]
    assert len({f.shape for b in batches for f in b}) == 3
    want = [plain.run(b) for b in batches]
    got = []
    posed.submit(batches[0])
    for t in range(1, 6):
        posed.submit(batches[t])
        got.append(posed.collect())
    got.append(posed.collect())
    n = sum(same_and_checked(batches[t], want[t], got[t]) for t in range(6))
    assert n > 0
    # reset one stream, then a partial batch (streams 0 and 1 only)
    v = video_frames()
    plain.reset(1); posed.reset(1)
    part = [v[1], frames.load_test1()]
    n = same_and_checked(part, plain.run(part), posed.run(part))
    assert n > 0 and list(posed.last_ran_detector) == list(plain.last_ran_detector)
