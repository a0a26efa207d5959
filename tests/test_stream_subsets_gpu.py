"""FaceAnaStreams calls that feed any subset of the streams, in any order (submit(frames, streams=...)): every stream must
return what its own FaceAna(detect_every=N, detect_offset=s % N) returns when fed only that stream's frames, with the
same resets, so a stream a call leaves out is untouched (no frame counted, no filter step, no id_memory gap, no cadence
step, its previous frame kept).  Results stay in call order.  streams=None and streams=list(range(n)) change nothing, and
a refused map enqueues and counts nothing."""
import numpy as np
import pytest

from test_detect_every_gpu import _Rule, _check_stream, _jittered_1080p, _stream_clips
from test_streams_gpu import _same, _sequences

pytestmark = pytest.mark.gpu

T_CLIP = 16


def _clips():
    """Six streams: the _stream_clips clips (the golden video, re-ordered frames with face-less ones, sub-threshold
    motion, a size change at frames 2 and 3, jittered 1080p) and a second jittered 1080p clip, phase-shifted."""
    clips = _stream_clips(T_CLIP)
    j = _jittered_1080p()
    clips.append([j[(t + 4) % len(j)] for t in range(T_CLIP)])
    return clips


# Streams of each call, before the order is shuffled; None: streams=None with frames for streams 0..4.
#  - single-stream calls 1 and 6; full calls 11 (streams=list(range(6))) and 12
#  - stream 1 is absent from calls 5..8, right after its face-less frame 3: its lost tracks must not age meanwhile
#  - stream 2's frames fall on calls 2, 4, 8, 10 (one slot parity); stream 4's on calls 5, 6, 7 (alternating)
#  - reset(3) before call 7, which does not feed stream 3; stream 5 is fed for the first time at call 8
_MEMBERS = [None, [2], [0, 1, 2, 3], [0, 1, 3, 4], [0, 1, 2], [0, 3, 4], [4], [0, 4], [0, 2, 3, 5], [0, 1, 3, 4, 5],
            [0, 1, 2, 4, 5], list(range(6)), list(range(6))]
_RESETS = {7: 3}
_IN_ORDER = {0, 11}


def _schedule(seed=2024):
    """[(streams or None, stream reset before the call or None)] with every call's order but 0 and 11 shuffled."""
    rng = np.random.default_rng(seed)
    plan = []
    for t, m in enumerate(_MEMBERS):
        if m is not None and t not in _IN_ORDER:
            m = [int(x) for x in rng.permutation(m)]
        plan.append((m, _RESETS.get(t)))
    return plan


def _streams_of(entry):
    return list(range(5)) if entry is None else entry


def test_schedule_covers_the_cases():
    plan = _schedule()
    fed = [_streams_of(m) for m, _ in plan]
    assert any(len(f) == 1 for f in fed) and any(len(f) == 6 for f in fed)
    assert any(m is not None and m != sorted(m) for m, _ in plan)
    calls = {s: [t for t, f in enumerate(fed) if s in f] for s in range(6)}
    assert max(b - a for a, b in zip(calls[1], calls[1][1:])) >= 4          # absent for 3+ calls in a row
    assert calls[2][2:6] == [2, 4, 8, 10] and calls[4][2:5] == [5, 6, 7]
    assert 3 not in fed[7] and plan[7][1] == 3
    assert calls[5][0] >= 8


def _device_results(out, n, feats):
    """Host lists of result dicts (call order) from a new_results() dict, and ran_detector."""
    cnt = out["n"].cpu().numpy()
    h = {k: v.cpu().numpy() for k, v in out.items()}
    res = []
    for i in range(n):
        faces = []
        for j in range(int(cnt[i])):
            r = {"box": h["box"][i, j], "kps": h["kps"][i, j], "scores": h["scores"][i, j]}
            if "id" in h:
                r["id"] = int(h["id"][i, j])
            if "chip" in h:
                r["chip"], r["M"] = h["chip"][i, j], h["M"][i, j]
            if "rvec" in h:
                r["pose"] = {k: h[k][i, j] for k in ("rvec", "tvec", "euler", "reproject")}
            faces.append(r)
        res.append(faces)
    return res, h["ran_detector"][:n].astype(bool)


CASES = {
    "every1-ids": ("host", 1, {"track_ids": True, "id_memory": 2}),
    "every3-ids": ("host", 3, {"track_ids": True, "id_memory": 2}),
    "align-pose": ("host", 1, {"align": 112, "pose": True}),
    "cuda-out": ("cuda", 3, {"track_ids": True, "id_memory": 2}),
    "mixed": ("mixed", 1, {"track_ids": True, "id_memory": 2, "pose": True}),
}


@pytest.mark.parametrize("case", list(CASES))
def test_subset_calls_equal_per_stream_faceana(case):
    """Two calls in flight throughout (but across reset); host frames, CUDA frames with out= on every other call, or host
    calls and CUDA out= calls on one object."""
    import torch
    from Skps import FaceAna, FaceAnaStreams
    kind, every, feats = CASES[case]
    clips = _clips()
    S = len(clips)
    plan = _schedule()
    fa = FaceAnaStreams(n_streams=S, detect_every=every, **feats)
    singles = [FaceAna(detect_every=every, detect_offset=s % every, **feats) for s in range(S)]
    rules = [_Rule(every, s % every) for s in range(S)]
    bufs = fa.new_results() if kind != "host" else None
    taken = [0] * S                     # frames of each stream fed so far: stream s's next frame is clips[s][taken[s]]
    frames_of = {}
    pending, got = [], {}

    def submit(t):
        streams, _ = plan[t]
        order = _streams_of(streams)
        batch = []
        for s in order:
            batch.append(clips[s][taken[s]])
            taken[s] += 1
        frames_of[t] = batch
        cuda = kind == "cuda" or (kind == "mixed" and t % 2 == 1)
        out = None
        if cuda:
            batch = [torch.from_numpy(f).cuda() for f in batch]
            out = bufs if (kind == "mixed" or t % 2 == 0) else None
        fa.submit(batch, out=out, streams=streams)
        pending.append((t, out))

    def collect():
        t, out = pending.pop(0)
        n = len(frames_of[t])
        r = fa.collect()
        got[t] = (_device_results(r, n, feats) if out is not None else (r, fa.last_ran_detector)) \
            + (fa.last_detector_frames,)

    for t in range(len(plan)):
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
    # the per-stream FaceAna objects, each fed only its stream's frames, in order, with the same resets
    for t in range(len(plan)):
        streams, reset = plan[t]
        if reset is not None:
            singles[reset].reset()
            rules[reset].reset()
        res, ran, m = got[t]
        order = _streams_of(streams)
        assert len(res) == len(order) == len(ran), t
        keys = 0
        for i, (s, frame) in enumerate(zip(order, frames_of[t])):
            want = singles[s].run(frame)
            _, key, want_ran = rules[s].step(frame)
            keys += key
            assert bool(ran[i]) == singles[s].last_ran_detector == want_ran, (t, i, s)
            _check_stream(res[i], want, frame, feats, (t, i, s))
        assert m == keys, (t, m, keys)


def test_identity_maps_change_nothing():
    """streams=None and streams=list(range(n)) return exactly what a call without the argument returns."""
    from Skps import FaceAnaStreams
    seqs = _sequences()
    S = len(seqs)
    feats = dict(n_streams=S, detect_every=2, track_ids=True)
    a, b, c = FaceAnaStreams(**feats), FaceAnaStreams(**feats), FaceAnaStreams(**feats)
    calls = [[s[t] for s in seqs] for t in range(6)] + [[seqs[0][1], seqs[1][2]]]
    for t, batch in enumerate(calls):
        ra = a.run(batch)
        rb = b.run(batch, streams=None)
        rc = c.run(batch, streams=list(range(len(batch))))
        assert list(a.last_ran_detector) == list(b.last_ran_detector) == list(c.last_ran_detector), t
        assert a.last_detector_frames == b.last_detector_frames == c.last_detector_frames, t
        for x, y, z in zip(ra, rb, rc):
            _same(x, y, tol=0.0)
            _same(x, z, tol=0.0)
            assert [f["id"] for f in x] == [f["id"] for f in y] == [f["id"] for f in z], t


def test_refused_call_enqueues_nothing():
    """Duplicate ids, an id >= n_streams and a length mismatch raise ValueError, also with a call in flight; the next
    calls return what per-stream FaceAna returns, so the refused ones counted no frame (detect_every=2 would shift)."""
    from Skps import FaceAna, FaceAnaStreams
    j = _jittered_1080p()
    S, N = 3, 2
    fa = FaceAnaStreams(n_streams=S, detect_every=N, track_ids=True)
    singles = [FaceAna(detect_every=N, detect_offset=s % N, track_ids=True) for s in range(S)]
    nxt = [0] * S

    def frames_for(streams):
        out = []
        for s in streams:
            out.append(j[(nxt[s] + 3 * s) % len(j)])
            nxt[s] += 1
        return out

    def check(res, streams, batch):
        for i, s in enumerate(streams):
            want = singles[s].run(batch[i])
            assert fa.last_ran_detector[i] == singles[s].last_ran_detector, (streams, i)
            _same(res[i], want)
            assert [f["id"] for f in res[i]] == [f["id"] for f in want]

    first = [2, 0]
    batch = frames_for(first)
    check(fa.run(batch, streams=first), first, batch)
    for bad, n in (([1, 1], 2), ([0, S], 2), ([0, 1, 2], 2), ([1], 2)):
        with pytest.raises(ValueError):
            fa.run([j[0]] * n, streams=bad)
    inflight = [1, 2]
    b1 = frames_for(inflight)
    fa.submit(b1, streams=inflight)
    with pytest.raises(ValueError):
        fa.submit([j[1], j[2]], streams=[0, 0])
    check(fa.collect(), inflight, b1)
    for streams in ([0, 1, 2], [1], [2, 0, 1]):
        batch = frames_for(streams)
        check(fa.run(batch, streams=streams), streams, batch)
