"""The host temporal layer of FaceAna at crowd size, without a GPU: the vectorised GroupTrack.calculate and FaceAna.judge_boxs
return exactly the arrays (values and dtype) of the reference's pair-by-pair loops (oracle.host_ref), and the top_k bounds of
FaceAna (1..1024) and FaceAnaStreams (1..64) are checked before anything is allocated."""
import numpy as np
import pytest

from oracle import host_ref as H

P = 98
IMG = np.broadcast_to(np.zeros(1, np.uint8), (2160, 3840, 3))       # calculate reads only the frame's shape
SIZES = (0, 1, 7, 64, 65, 384, 1024)
# (n_now, n_prev): every size on both sides; the scalar oracle costs about n_now * n_prev pair checks
PAIRS = [(0, 0), (0, 7), (7, 0), (1, 1), (1, 1024), (1024, 1), (7, 64), (64, 7), (64, 65), (65, 64), (65, 384), (384, 384),
         (1024, 7)]


def _trace_cfg():
    from peppa_pig_face_landmark_b200.core.api.facer import get_cfg
    return get_cfg()['Skps']['Trace']


def _faceana_host():
    """A FaceAna with only what judge_boxs reads (no engines, no GPU)."""
    from peppa_pig_face_landmark_b200.core.api.facer import FaceAna
    from peppa_pig_face_landmark_b200.core.smoother.lk import EmaFilter
    cfg = _trace_cfg()
    fa = FaceAna.__new__(FaceAna)
    fa.iou_thres, fa.alpha = cfg['iou_thres'], cfg['smooth_box']
    fa.filter = EmaFilter(fa.alpha)
    return fa


def _rects(rng, n, special=True):
    """n boxes [x0, y0, x1, y1] on a 3840x2160 frame, with duplicates and zero-area boxes mixed in."""
    xy = rng.uniform(0, 3600, (n, 2)) * [1, 0.55]
    wh = rng.uniform(20, 240, (n, 2))
    r = np.concatenate([xy, xy + wh], 1)
    if special and n >= 4:
        r[1] = r[0]                                    # duplicate
        r[2, 2] = r[2, 0]                              # zero width
        r[3, 3] = r[3, 1]                              # zero height
    return r


def _half_pairs(rng, k):
    """k rectangle pairs (now, prev) whose IoU is exactly 0.5 or 1/64 px either side of it (dyadic coordinates)."""
    now, prev = [], []
    for i in range(k):
        x, y, a = float(rng.integers(0, 3000)), float(rng.integers(0, 1800)), float(rng.integers(8, 128))
        d = (0.0, 1 / 64, -1 / 64)[i % 3]
        prev.append([x, y, x + 2 * a, y + a])
        now.append([x, y, x + a + d, y + a])
    return np.array(now), np.array(prev)


def _sets(rng, rects, dtype):
    """Landmark sets whose min/max rectangles are exactly `rects`."""
    n = len(rects)
    r = rects.astype(dtype)
    t = rng.uniform(0, 1, (n, P, 2))
    pts = r[:, None, :2] + t * (r[:, None, 2:] - r[:, None, :2])
    pts[:, 0] = r[:, :2]
    pts[:, 1] = r[:, 2:]
    return np.clip(pts, r[:, None, :2], r[:, None, 2:]).astype(dtype)


def _jitter(rng, rects, px):
    return rects + rng.normal(0, px, rects.shape)


def _landmarks(rng, n_now, prev_rects):
    """Rectangles of n_now faces: jittered copies of some of prev_rects (matches, some at IoU 0.5 exactly), shuffled, plus
    new faces."""
    m = len(prev_rects)
    out = []
    if m:
        take = rng.choice(m, min(n_now // 2, m), replace=False)
        out.append(_jitter(rng, prev_rects[take], 2.0))
    out.append(_rects(rng, n_now - sum(len(o) for o in out)))
    r = np.concatenate(out)[:n_now]
    rng.shuffle(r)
    return r


def _same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype, (what, a.dtype, b.dtype)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.array_equal(a, b, equal_nan=True), what


def _track_pair():
    from peppa_pig_face_landmark_b200.core.smoother.lk import GroupTrack
    cfg = _trace_cfg()
    return GroupTrack(cfg), H.GroupTrackRef(cfg['iou_thres'])


def _set_state(gt, ref, prev, prev_dx):
    gt.previous_landmarks_set, gt.previous_dx = prev.copy(), prev_dx.copy()
    ref.prev, ref.prev_dx = prev.copy(), prev_dx.copy()


def _calc(gt, ref, now, what):
    got = gt.calculate(IMG, now.copy())
    want = ref.calculate(IMG, now.copy())
    _same(got, want, what)
    _same(gt.previous_dx, ref.prev_dx, (what, "dx"))
    _same(gt.previous_landmarks_set, ref.prev, (what, "state"))
    return got


@pytest.mark.parametrize("n_now,n_prev", PAIRS)
@pytest.mark.parametrize("state", ["float32", "float64"])
def test_group_track_matches_scalar_loop(n_now, n_prev, state):
    rng = np.random.default_rng(n_now * 7919 + n_prev * 31 + (state == "float64"))
    gt, ref = _track_pair()
    prev_rects = _rects(rng, n_prev)
    dt = np.dtype(state)
    prev = _sets(rng, prev_rects, dt) if n_prev else np.zeros((0, P, 2), dt)
    if dt == np.float64 and n_prev:
        prev = prev + rng.uniform(-1e-3, 1e-3, prev.shape)            # values a float32 cannot hold
    dx = rng.normal(0, 0.5, prev.shape).astype(dt)
    _set_state(gt, ref, prev, dx)
    now_rects = _landmarks(rng, n_now, prev_rects)
    now = _sets(rng, now_rects, np.float32) if n_now else np.array([])
    _calc(gt, ref, now, (n_now, n_prev, state, 0))
    # two more frames from the smoothed state (float64 once a face matched), then one with no face; at 1024 faces the
    # state then holds 1024 sets, which the scalar oracle takes about a minute per frame to match
    for t in ((1, 2) if n_now <= 384 else ()):
        base = prev_rects
        if ref.prev.ndim == 3 and len(ref.prev):
            base = np.array([H.GroupTrackRef._rect(s) for s in ref.prev], np.float64)
        r = _landmarks(rng, n_now, base)
        now = _sets(rng, r, np.float32) if n_now else np.array([])
        _calc(gt, ref, now, (n_now, n_prev, state, t))
    _calc(gt, ref, np.array([]), (n_now, n_prev, state, "empty"))


@pytest.mark.parametrize("state", ["float32", "float64"])
def test_group_track_iou_at_one_half(state):
    rng = np.random.default_rng(5)
    now_r, prev_r = _half_pairs(rng, 60)
    dt = np.dtype(state)
    prev = _sets(rng, prev_r, dt)
    gt, ref = _track_pair()
    _set_state(gt, ref, prev, np.zeros_like(prev))
    # the sets' rectangles are the pairs: exactly 0.5 does not match, 0.5 + a little does
    from peppa_pig_face_landmark_b200.core.smoother.lk import first_match, rects
    m = first_match(rects(_sets(rng, now_r, np.float32)), rects(prev), 0.5)
    assert (m[0::3] == -1).all() and (m[1::3] >= 0).all() and (m[2::3] == -1).all()
    _calc(gt, ref, _sets(rng, now_r, np.float32), state)


def test_group_track_first_frame_and_reset():
    rng = np.random.default_rng(9)
    gt, ref = _track_pair()
    now = _sets(rng, _rects(rng, 65), np.float32)
    _calc(gt, ref, now, "first")
    _calc(gt, ref, now + np.float32(0.25), "second")
    gt.previous_landmarks_set, ref.prev = None, None
    _calc(gt, ref, now, "after reset")


def _boxes(rng, n, dtype):
    return _rects(rng, n).astype(dtype)


@pytest.mark.parametrize("n_now,n_prev", [(a, b) for a in SIZES for b in SIZES if a * b <= 70000 or a == b == 1024])
def test_judge_boxs_matches_scalar_loop(n_now, n_prev):
    rng = np.random.default_rng(n_now * 131 + n_prev)
    fa = _faceana_host()
    prev = _boxes(rng, n_prev, np.float32)                    # boxes_return: float32 from the pipeline
    for dt in (np.float32, np.float64):                       # tmp_box: the dtype of the smoothed landmarks
        if n_now == 0:
            now = np.array([])
        else:
            k = min(n_now // 2, n_prev)
            r = _rects(rng, n_now)
            if k:
                r[:k] = _jitter(rng, prev[rng.choice(n_prev, k, replace=False)].astype(np.float64), 3.0)
            rng.shuffle(r)
            now = r.astype(dt)
        _same(fa.judge_boxs(prev, now), H.judge_boxs(prev, now, fa.iou_thres, fa.alpha), (n_now, n_prev, dt))


@pytest.mark.parametrize("dt", [np.float32, np.float64])
def test_judge_boxs_iou_at_one_half(dt):
    rng = np.random.default_rng(3)
    now_r, prev_r = _half_pairs(rng, 90)
    fa = _faceana_host()
    now, prev = now_r.astype(dt), prev_r.astype(np.float32)
    now[5] = now[4]                                           # duplicate rows
    got = fa.judge_boxs(prev, now)
    _same(got, H.judge_boxs(prev, now, fa.iou_thres, fa.alpha), dt)
    assert not np.array_equal(got, now)                       # some rows matched
    assert fa.judge_boxs(None, now) is now


def test_faceana_top_k_bounds():
    from peppa_pig_face_landmark_b200.core.api.facer import FaceAna
    from peppa_pig_face_landmark_b200.core.api.streams import FaceAnaStreams
    for k in (0, 1025):
        with pytest.raises(ValueError, match="top_k"):
            FaceAna(top_k=k)
    for k in (0, 65):
        with pytest.raises(ValueError, match="top_k"):
            FaceAnaStreams(n_streams=2, top_k=k)
