"""Track ids on the GPU (FaceAna(track_ids=True), FaceAnaStreams(track_ids=True)): turning them on changes nothing else;
FaceAna's ids equal an independent numpy restatement of the rule, whose sources come from facer.py's judge_boxs and
sort_and_filter on the previous call's boxes and the detector's kept rows; lost faces come back with new ids, skipped frames
keep every id, reset() numbers from 0; every stream of FaceAnaStreams gives the ids of its own FaceAna; crowds on both
selection branches."""
import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames
from test_crowd_cpu import crowd_frame

pytestmark = pytest.mark.gpu

IOU, ALPHA, MIN_FACE = 0.5, 0.3, 1600


def _bright(f, d):
    """The frame with every byte raised by d: a mean difference of about d, so the gate runs the detector at d > 5."""
    return np.clip(f.astype(np.int16) + d, 0, 255).astype(np.uint8)


def _equal_results(a, b, what):
    assert len(a) == len(b), (what, len(a), len(b))
    for x, y in zip(a, b):
        for k in ("box", "kps", "scores"):
            assert np.array_equal(np.asarray(x[k]), np.asarray(y[k])), (what, k)
            assert np.asarray(x[k]).dtype == np.asarray(y[k]).dtype, (what, k)


# ----------------------------------------------------------------------------- the restatement
def _sources(prev_boxes, det_rows, top_k):
    """facer.py:56-66 on the host: the source of every face the call returns, in output order.  prev_boxes: the previous
    call's returned boxes as float32 (what FaceAna hands the device); det_rows: the kept detector rows of a detector frame,
    or None on a gate-skipped frame."""
    from oracle import host_ref as H
    prev = np.asarray(prev_boxes, np.float32).reshape(-1, 4)
    if det_rows is None:                                   # facer.py:61: the faces are the track boxes
        judged, src = prev, list(range(len(prev)))
    else:                                                  # judge_boxs: the first track box with IoU > iou_thres
        now = np.asarray(det_rows, np.float32)[:, :4]
        judged, src = now.copy(), [-1] * len(now)
        for i, r in enumerate(now):
            for j, p in enumerate(prev):
                if H.iou_xyxy(r, p) > IOU:
                    judged[i] = ALPHA * r + (1 - ALPHA) * p
                    src[i] = j
                    break
    if len(judged) == 0:
        return []
    area = (judged[:, 2] - judged[:, 0]) * (judged[:, 3] - judged[:, 1])
    keep = np.where(area > MIN_FACE)[0]                    # sort_and_filter, equal areas later index first
    if len(keep) > top_k:
        keep = keep[area[keep].argsort(kind="stable")[-top_k:][::-1]]
    return [src[i] for i in keep]


def _rule(sources, prev_ids, next_id):
    out = []
    for s in sources:
        if s >= 0 and prev_ids[s] not in out:
            out.append(prev_ids[s])
        else:
            out.append(next_id)
            next_id += 1
    return out, next_id


class _Restated:
    """Follows a FaceAna(track_ids=True) call by call and checks its ids against the restatement."""

    def __init__(self, facer):
        self.facer, self.prev, self.ids, self.next_id = facer, np.zeros((0, 4), np.float32), [], 0
        self.paths = set()

    def run(self, frame, what):
        f = self.facer
        f.last_det_rows = None                             # set again only if this call runs the detector
        res = f.run(frame)
        rows = f.last_det_rows
        src = _sources(self.prev, rows, f.top_k)
        want, self.next_id = _rule(src, self.ids, self.next_id)
        assert len(src) == len(res), (what, len(src), len(res))
        assert [r["id"] for r in res] == want, (what, [r["id"] for r in res], want)
        assert all(type(r["id"]) is int for r in res)
        self.paths.add(("det" if rows is not None else "skip", any(s >= 0 for s in src)))
        self.prev = np.asarray([r["box"] for r in res], np.float32).reshape(-1, 4)
        self.ids = want
        return res


# ----------------------------------------------------------------------------- FaceAna
def _clips():
    t1, c, f4 = frames.load_test1(), frames.canvas_640(), frames.frame_4k()
    return {"test1": ([t1, t1, _bright(t1, 8)], 5), "canvas640": ([c, c, _bright(c, 8)], 5),
            "video1080": (video_frames(), 5), "uhd4k_top16": ([f4, f4, frames.frame_4k(jitter=(4, 4)), _bright(f4, 8)], 16)}


@pytest.mark.parametrize("name", ["test1", "canvas640", "video1080", "uhd4k_top16"])
def test_faceana_ids_change_nothing_else(name):
    from Skps import FaceAna
    clip, top_k = _clips()[name]
    on, off = FaceAna(top_k=top_k, track_ids=True), FaceAna(top_k=top_k)
    for t, fr in enumerate(clip):
        a, b = on.run(fr), off.run(fr)
        _equal_results(a, b, (name, t))
        assert all(set(r) == {"box", "kps", "scores", "id"} for r in a)
        assert all(set(r) == {"box", "kps", "scores"} for r in b)


def test_faceana_ids_equal_the_restatement_on_video1080():
    from Skps import FaceAna
    r = _Restated(FaceAna(track_ids=True))
    v = video_frames()
    # the golden clip (detect, unchanged x2, moved, empty x2), then faces again: re-detected where they were last seen
    for t, fr in enumerate(v + [_bright(v[3], 8), v[0], _bright(v[0], 8), v[0]]):
        r.run(fr, t)
    # the clip reaches a detector frame that continues faces, one that starts them, and a skipped frame
    assert {("det", True), ("det", False), ("skip", True)} <= r.paths, r.paths


def _scene():
    """Four faces at 1080p; face 3 (bottom right) is covered for two frames.  The brightness alternates by 8 so that the
    gate runs the detector wherever a frame differs from the one before."""
    full = frames.multi_face_frame(1080, 1920, (2, 2), 440)
    gone = full.copy()
    gone[540:, 960:] = frames._background(1080, 1920)[540:, 960:]
    return [full, full, _bright(gone, 8), gone, _bright(full, 8), _bright(full, 8)]


def _by_place(res):
    """{(row, col) of the face's grid cell: id}."""
    return {(int((r["box"][1] + r["box"][3]) / 2 >= 540), int((r["box"][0] + r["box"][2]) / 2 >= 960)): r["id"] for r in res}


def test_faceana_lost_face_gets_a_new_id_and_the_others_keep_theirs():
    from Skps import FaceAna
    facer = FaceAna(track_ids=True)
    r = _Restated(facer)
    got = [_by_place(r.run(fr, t)) for t, fr in enumerate(_scene())]
    first = got[0]
    assert len(first) == 4 and sorted(first.values()) == [0, 1, 2, 3]
    assert got[1] == first                                     # identical frame: the gate skips the detector
    kept = {k: v for k, v in first.items() if k != (1, 1)}
    assert got[2] == kept and got[3] == kept                   # face (1, 1) is gone, the others keep their ids
    assert got[4] == {**kept, (1, 1): 4}                       # it comes back as a new face
    assert got[5] == got[4]
    assert ("skip", True) in r.paths and ("det", True) in r.paths
    facer.reset()
    again = facer.run(_scene()[0])
    assert _by_place(again) == first                           # numbering starts from 0 again, in the same order


# ----------------------------------------------------------------------------- FaceAnaStreams
def _stream_seqs():
    from test_streams_gpu import _sequences
    return _sequences() + [_scene()]


def test_streams_ids_change_nothing_else():
    """Host and device results of FaceAnaStreams(track_ids=True) against FaceAnaStreams() on the same frames."""
    import torch
    from Skps import FaceAnaStreams
    seqs = _stream_seqs()
    S = len(seqs)
    on, off, dev = (FaceAnaStreams(n_streams=S, track_ids=True), FaceAnaStreams(n_streams=S),
                    FaceAnaStreams(n_streams=S, track_ids=True))
    out = dev.new_results()
    assert out["id"].dtype == torch.int64 and tuple(out["id"].shape) == (S, dev.top_k)
    assert "id" not in off.new_results()
    for t in range(6):
        batch = [s[t] for s in seqs]
        a, b = on.run(batch), off.run(batch)
        dev.submit([torch.from_numpy(f).cuda() for f in batch], out=out)
        d = {k: v.cpu().numpy() for k, v in dev.collect().items()}
        for s in range(S):
            _equal_results(a[s], b[s], (t, s))
            n = int(d["n"][s])
            assert n == len(b[s])
            for i, w in enumerate(b[s]):
                for k in ("box", "kps", "scores"):
                    assert np.array_equal(d[k][s, i], w[k]), (t, s, k)
            assert [int(v) for v in d["id"][s, :n]] == [r["id"] for r in a[s]], (t, s)


def _check_ids(res, singles, frames_of, what):
    for s, fr in frames_of.items():
        want = [r["id"] for r in singles[s].run(fr)]
        got = [r if isinstance(r, int) else r["id"] for r in res[s]]
        assert got == want, (what, s, got, want)


def test_streams_ids_equal_single_stream_faceana_host_frames():
    """Host frames and host results, partial batches and reset(stream)."""
    from Skps import FaceAna, FaceAnaStreams
    seqs = _stream_seqs()
    S = len(seqs)
    fa = FaceAnaStreams(n_streams=S, track_ids=True)
    singles = [FaceAna(track_ids=True) for _ in range(S)]
    for t in range(6):
        n = S if t % 3 != 2 else 2                              # streams 2.. skip every third call
        if t == 4:
            fa.reset(1)
            singles[1].reset()
        res = fa.run([seqs[s][t] for s in range(n)])
        assert len(res) == n
        _check_ids(res, singles, {s: seqs[s][t] for s in range(n)}, t)
    fa.reset()
    for s in singles:
        s.reset()
    _check_ids(fa.run([s[0] for s in seqs]), singles, {s: seqs[s][0] for s in range(S)}, "after reset()")


def test_streams_ids_equal_single_stream_faceana_cuda_frames_two_in_flight():
    """CUDA frames, two batches in flight, device and host results alternating."""
    import torch
    from Skps import FaceAna, FaceAnaStreams
    seqs = _stream_seqs()
    S = len(seqs)
    fa = FaceAnaStreams(n_streams=S, track_ids=True)
    singles = [FaceAna(track_ids=True) for _ in range(S)]
    bufs, pending = [fa.new_results(), fa.new_results()], []
    modes = ["dev", "host", "dev", "dev", "host", "dev"]

    def submit(t):
        batch = [torch.from_numpy(s[t]).cuda() for s in seqs]
        out = bufs[t % 2] if modes[t] == "dev" else None
        fa.submit(batch, out=out)
        pending.append(t)

    def collect():
        t = pending.pop(0)
        r = fa.collect()
        if modes[t] == "dev":
            ids, n = r["id"].cpu().numpy(), r["n"].cpu().numpy()
            r = [[int(v) for v in ids[s, :int(n[s])]] for s in range(S)]
        _check_ids(r, singles, {s: seqs[s][t] for s in range(S)}, (t, modes[t]))

    submit(0)
    for t in range(1, 6):
        submit(t)
        collect()
    collect()


# ----------------------------------------------------------------------------- crowds
@pytest.fixture(scope="module")
def crowd384():
    return crowd_frame("crowd384_1152x1920")


def test_crowd_ids_top_k_512(crowd384):
    """384 faces, every one of them returned: a permutation of 0..383, kept face by face on the unchanged frame."""
    from Skps import FaceAna
    facer = FaceAna(top_k=512, det_input=(1152, 1920), track_ids=True)
    r = _Restated(facer)
    first = r.run(crowd384, "first")
    assert len(first) == 384
    assert sorted(x["id"] for x in first) == list(range(384))
    second = r.run(crowd384, "unchanged")
    assert [x["id"] for x in second] == [x["id"] for x in first]
    r.run(_bright(crowd384, 8), "re-detected")
    assert ("det", True) in r.paths


def test_crowd_ids_radix_select(crowd384):
    """top_k 256 of 384 faces: the selection takes its radix-select branch and orders faces by area, on the first frame and
    on a re-detected one whose detections are judged against 256 track boxes."""
    from Skps import FaceAna
    facer = FaceAna(top_k=256, det_input=(1152, 1920), track_ids=True)
    r = _Restated(facer)
    first = r.run(crowd384, "first")
    assert len(first) == 256 and len(facer.last_det_rows) == 384
    assert sorted(x["id"] for x in first) == list(range(256))
    again = r.run(_bright(crowd384, 8), "re-detected")
    assert len(again) == 256
    assert ("det", True) in r.paths
    assert any(x["id"] < 256 for x in again)
