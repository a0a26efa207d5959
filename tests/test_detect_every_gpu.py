"""Detection cadence on the GPU (FaceAna(detect_every=N, detect_offset=o), FaceAnaStreams(detect_every=N)): frame i of a
stream runs the detector when it has no previous frame of its size, or when (i + o) % N == 0 and the frame-difference gate
fires; every other frame takes the tracker path.  FaceAna is checked against the oracle with that rule, every stream of
FaceAnaStreams against its own FaceAna(detect_every=N, detect_offset=s % N), the packed detector batch against the number
of keyframes, and N = 1 against the default objects."""
import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames
from test_align_gpu import check_faces
from test_parity_gpu import KPS_TOL_PX, SCORE_TOL
from test_streams_gpu import _same, _sequences

pytestmark = pytest.mark.gpu

JITTERS = [(0, 0), (12, -8), (-12, 8), (8, 12), (-8, -12), (16, 4), (-16, -4), (4, 16), (-4, -16)]


def _jittered_1080p():
    """9 frames of frames.frame_1080p, each with its own jitter: the mean difference of any two is > 5, so the gate fires."""
    return [frames.frame_1080p(jitter=j) for j in JITTERS]


def _gate(prev, cur):
    return np.abs(prev.astype(np.int16) - cur.astype(np.int16)).sum() / prev.shape[0] / prev.shape[1] / 3. > 5


class _Rule:
    """The keyframe rule of one stream, restated: frames counted since construction / reset; forced = no previous frame
    of this size; by_count = (i + offset) % every == 0."""

    def __init__(self, every, offset):
        self.every, self.offset = every, offset
        self.reset()

    def reset(self):
        self.i, self.prev = 0, None

    def step(self, frame):
        """(forced, keyframe, runs the detector) of the stream's next frame."""
        forced = self.prev is None or self.prev.shape != frame.shape
        by_count = (self.i + self.offset) % self.every == 0
        ran = forced or (by_count and _gate(self.prev, frame))
        self.i += 1
        self.prev = frame
        return forced, forced or by_count, ran


# ----------------------------------------------------------------------------- FaceAna against the oracle
def _cadence_ref(every, offset):
    from oracle.faceana_ref import FaceAnaRef

    class CadenceRef(FaceAnaRef):
        """FaceAnaRef whose diff_frames applies the keyframe rule."""

        def reset(self):
            super().reset()
            self.rule = _Rule(every, offset)

        def diff_frames(self, prev, image):
            forced, key, _ = self.rule.step(image)
            self.ran = forced or (key and super().diff_frames(prev, image))
            return self.ran

    return CadenceRef()


@pytest.mark.parametrize("offset", [0, 2])
def test_faceana_detect_every_3_matches_oracle(offset):
    from Skps import FaceAna
    seq = _jittered_1080p()
    for a, b in zip(seq, seq[1:]):
        assert _gate(a, b)
    facer, ref = FaceAna(detect_every=3, detect_offset=offset), _cadence_ref(3, offset)
    ran = []
    for t, fr in enumerate(seq):
        got, want = facer.run(fr), ref.run(fr)
        assert facer.last_ran_detector == ref.ran, t
        ran.append(facer.last_ran_detector)
        assert len(got) == len(want) == 4, (t, len(got), len(want))
        for a, b in zip(got, want):
            assert np.abs(np.asarray(a["kps"], np.float64) - b["kps"]).max() <= KPS_TOL_PX, t
            assert np.abs(np.asarray(a["box"], np.float64) - np.asarray(b["box"], np.float64)).max() <= KPS_TOL_PX, t
            assert np.abs(a["scores"] - b["scores"]).max() <= SCORE_TOL, t
    assert ran == [t == 0 or (t + offset) % 3 == 0 for t in range(9)]


def test_faceana_reset_restarts_the_count():
    from Skps import FaceAna
    seq = _jittered_1080p()
    facer = FaceAna(detect_every=4, detect_offset=1)
    ran = []
    for fr in seq[:5]:
        facer.run(fr)
        ran.append(facer.last_ran_detector)
    facer.reset()
    for fr in seq[5:]:
        facer.run(fr)
        ran.append(facer.last_ran_detector)
    # frame 0 is forced; then (i + 1) % 4 == 0 at i = 3; after reset() frame 0 again, then none of i = 1..3
    assert ran == [True, False, False, True, False, True, False, False, True]


# ----------------------------------------------------------------------------- FaceAnaStreams against per-stream FaceAna
def _stream_clips(T):
    """The test_streams_gpu clips (cycled to T frames) and a jittered 1080p clip.  Clip 3 changes size at its frames 2 and
    3 (273x410 -> 1080x1920 -> 273x410)."""
    clips = [[c[t % len(c)] for t in range(T)] for c in _sequences()]
    j = _jittered_1080p()
    clips.append([j[t % len(j)] for t in range(T)])
    return clips


def _plan(T, S):
    """(streams fed, stream reset before the call or None) of each call: partial batches at calls 4 and 7, reset(1) before
    call 6.  Stream 3 is fed at its frames 2 and 3, where its frame size changes."""
    n = {4: 2, 7: 3}
    return [(n.get(t, S), 1 if t == 6 else None) for t in range(T)]


def _same_at(a, b, what, tol=1e-6):
    """test_streams_gpu._same, naming the call and stream that differ."""
    assert len(a) == len(b), (what, len(a), len(b))
    for i, (x, y) in enumerate(zip(a, b)):
        for k in ("kps", "box"):
            d = np.abs(np.asarray(x[k], np.float64) - np.asarray(y[k], np.float64)).max()
            assert d <= tol, (what, i, k, d)
        assert np.array_equal(x["scores"], y["scores"]), (what, i)


def _check_stream(res_s, want, frame, feats, what):
    _same_at(res_s, want, what)
    if "track_ids" in feats:
        assert [r["id"] for r in res_s] == [r["id"] for r in want]
    if "pose" in feats:
        from Skps.core.headpose.pose import POSE_POINTS_98, head_poses
        for r in res_s:
            p = head_poses(np.asarray(r["kps"])[None], frame.shape[:2], points=POSE_POINTS_98)
            for k in ("rvec", "tvec", "euler", "reproject"):
                assert np.array_equal(r["pose"][k], p[k][0]), k
    if "align" in feats:
        check_faces(frame, res_s, 112)


def _device_results(out, n):
    """Host lists of {'box','kps','scores'} from a new_results() dict (n streams), and ran_detector."""
    cnt = out["n"].cpu().numpy()
    box, kps, sc = out["box"].cpu().numpy(), out["kps"].cpu().numpy(), out["scores"].cpu().numpy()
    res = [[{"box": box[s, i], "kps": kps[s, i], "scores": sc[s, i]} for i in range(int(cnt[s]))] for s in range(n)]
    return res, out["ran_detector"].cpu().numpy()[:n].astype(bool)


@pytest.mark.parametrize("kind", ["host", "cuda"])
@pytest.mark.parametrize("every", [2, 3, 5])
def test_streams_equal_per_stream_faceana(every, kind):
    """Two batches in flight, partial batches, reset(stream), a size change on a non-keyframe; host frames with align, pose
    and track ids on, or CUDA frames with results left on the GPU (out=) on every other call."""
    import torch
    from Skps import FaceAna, FaceAnaStreams
    T = 9
    clips = _stream_clips(T)
    S = len(clips)
    feats = {"align": 112, "pose": True, "track_ids": True} if kind == "host" else {}
    fa = FaceAnaStreams(n_streams=S, detect_every=every, **feats)
    singles = [FaceAna(detect_every=every, detect_offset=s % every, **feats) for s in range(S)]
    rules = [_Rule(every, s % every) for s in range(S)]
    plan = _plan(T, S)
    bufs = [fa.new_results(), fa.new_results()] if kind == "cuda" else None
    pending = []
    forced_seen = set()

    def submit(t):
        n, _ = plan[t]
        batch = [clips[s][t] for s in range(n)]
        if kind == "cuda":
            batch = [torch.from_numpy(f).cuda() for f in batch]
        out = bufs[t % 2] if kind == "cuda" and t % 2 == 0 else None
        fa.submit(batch, out=out)
        pending.append((t, out))

    def collect():
        t, out = pending.pop(0)
        n, _ = plan[t]
        r = fa.collect()
        if out is not None:
            got[t] = _device_results(r, n) + (fa.last_detector_frames,)
        else:
            got[t] = (r, fa.last_ran_detector, fa.last_detector_frames)

    got = {}
    for t in range(T):
        _, reset = plan[t]
        if reset is not None:
            while pending:
                collect()
            fa.reset(reset)
        submit(t)
        if len(pending) == 2:
            collect()
    while pending:
        collect()
    torch.cuda.synchronize()
    # the per-stream FaceAna objects run once FaceAnaStreams is done, in the same order of frames and resets
    for t in range(T):
        n, reset = plan[t]
        if reset is not None:
            singles[reset].reset()
            rules[reset].reset()
        res, ran, m = got[t]
        keys = 0
        for s in range(n):
            want = singles[s].run(clips[s][t])
            forced, key, want_ran = rules[s].step(clips[s][t])
            keys += key
            if forced and not (rules[s].i - 1 + rules[s].offset) % every == 0:
                forced_seen.add((t, s))
            assert bool(ran[s]) == singles[s].last_ran_detector == want_ran, (t, s)
            _check_stream(res[s], want, clips[s][t], feats, (t, s))
        assert m == keys, (t, m, keys)
    # clip 3 changes size at its frames 2 and 3: one of them is not a keyframe by count, and runs the detector all the same
    assert forced_seen & {(2, 3), (3, 3)}


def test_streams_detector_batch_is_the_keyframes():
    """N = 4 > 3 streams, jittered frames (the gate always fires): ran_detector is the rule, the detector batch is the
    number of keyframe streams, and calls 1 and 5 have none."""
    from Skps import FaceAna, FaceAnaStreams
    j = _jittered_1080p()
    S, N, T = 3, 4, 9
    fa = FaceAnaStreams(n_streams=S, detect_every=N)
    singles = [FaceAna(detect_every=N, detect_offset=s % N) for s in range(S)]
    m = []
    for t in range(T):
        batch = [j[(t + 2 * s) % len(j)] for s in range(S)]
        res = fa.run(batch)
        want_ran = [t == 0 or (t + s) % N == 0 for s in range(S)]
        assert list(fa.last_ran_detector) == want_ran, t
        m.append(fa.last_detector_frames)
        for s in range(S):
            _same(res[s], singles[s].run(batch[s]))
        assert sum(len(r) for r in res) == 4 * S
    assert m == [3, 0, 1, 1, 1, 0, 1, 1, 1]


# ----------------------------------------------------------------------------- N = 1 changes nothing
def test_detect_every_1_changes_nothing():
    from Skps import FaceAna, FaceAnaStreams
    seqs = _sequences()
    S = len(seqs)
    a, b = FaceAnaStreams(n_streams=S), FaceAnaStreams(n_streams=S, detect_every=1)
    fa, fb = FaceAna(), FaceAna(detect_every=1, detect_offset=0)
    for t in range(6):
        batch = [s[t] for s in seqs]
        ra, rb = a.run(batch), b.run(batch)
        assert b.last_detector_frames == a.last_detector_frames == S
        assert list(a.last_ran_detector) == list(b.last_ran_detector)
        for x, y in zip(ra, rb):
            _same(x, y, tol=0.0)
        x, y = fa.run(seqs[0][t]), fb.run(seqs[0][t])
        assert fa.last_ran_detector == fb.last_ran_detector
        _same(x, y, tol=0.0)
    part = [video_frames()[0]]
    ra, rb = a.run(part), b.run(part)
    assert b.last_detector_frames == 1
    _same(ra[0], rb[0], tol=0.0)
