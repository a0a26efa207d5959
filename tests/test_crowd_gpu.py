"""Crowds on the GPU: the NMS of any size (skps_detect_post_batch, csrc/nms.cu) against the numpy restatement of py_nms on
synthetic rows and on the detector's own output, FaceDetector / FaceAna / FaceAnaStreams on frames of 96 to 384 faces against
the oracle, and skps_detect_post keeping its 1024-candidate contract."""
import numpy as np
import pytest

import frames
from test_crowd_cpu import CROWDS, crowd_frame
from test_detector_input_gpu import _close, _detector, _detector_ref, _faceana_ref

pytestmark = pytest.mark.gpu


def _nms_ranked(raw, recover, iou_thres=0.3, score_thres=0.5):
    """oracle.host_ref.detect_post with the candidate order spelled out: score descending, equal scores by row index
    descending (np.argsort(score)[::-1] of a stable sort; the reference's default sort leaves equal scores unordered)."""
    from oracle import host_ref as H
    out = np.array(raw, dtype=np.float32).reshape(-1, 16)
    out[:, :4] = H.xywh2xyxy(out[:, :4])
    cand = np.where(out[:, 4] > score_thres)[0]
    b = out[cand]
    order = np.argsort(b[:, 4], kind="stable")[::-1]
    keep = []
    while order.shape[0] > 0:
        cur = order[0]
        keep.append(cur)
        rest = order[1:]
        area = (b[cur, 2] - b[cur, 0]) * (b[cur, 3] - b[cur, 1])
        xx1 = np.maximum(b[cur, 0], b[rest, 0])
        yy1 = np.maximum(b[cur, 1], b[rest, 1])
        xx2 = np.minimum(b[cur, 2], b[rest, 2])
        yy2 = np.minimum(b[cur, 3], b[rest, 3])
        inter = np.maximum(0, yy2 - yy1) * np.maximum(0, xx2 - xx1)
        other = (b[rest, 3] - b[rest, 1]) * (b[rest, 2] - b[rest, 0])
        iou = inter / (area + other - inter)
        order = rest[np.where(iou < iou_thres)[0]]
    keep = np.asarray(keep, dtype=np.int64)
    kept = b[keep]
    kept[:, :4] = H.scale_coords(kept[:, :4], recover)
    return kept, cand[keep]


def _post_batch(raws, recovers, capacity=None):
    """skps_detect_post_batch on a stack of raw outputs -> [(kept rows, kept indices)] per frame."""
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    B, rows = len(raws), raws[0].shape[0]
    cap = capacity or rows
    d = torch.from_numpy(np.ascontiguousarray(np.stack(raws), np.float32)).cuda()
    rec = torch.tensor(np.asarray(recovers, np.float64), dtype=torch.float32, device="cuda")
    kept = torch.full((B, cap, 16), -7.0, dtype=torch.float32, device="cuda")
    idx = torch.full((B, cap), -7, dtype=torch.int32, device="cuda")
    cnt = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    nbytes = lib.skps_detect_post_workspace_size(rows, B)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    rt.check(lib.skps_detect_post_batch(d.data_ptr(), rows, B, 0.5, 0.3, rec.data_ptr(), kept.data_ptr(), idx.data_ptr(),
                                        cnt.data_ptr(), cap, ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    out = []
    for b in range(B):
        n = int(cnt[b])
        out.append((kept[b, :n].cpu().numpy(), idx[b, :n].cpu().numpy().astype(np.int64)))
    return out


def _legacy(raw, max_det=256):
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    d = torch.from_numpy(raw).cuda()
    kept = torch.zeros((256, 16), dtype=torch.float32, device="cuda")
    idx = torch.zeros(256, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    rt.check(lib.skps_detect_post(d.data_ptr(), raw.shape[0], 0.5, 0.3, 1.0, 0.0, 0.0, kept.data_ptr(), idx.data_ptr(),
                                  cnt.data_ptr(), max_det, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    n = int(cnt.item())
    return n, kept[:max(n, 0)].cpu().numpy(), idx[:max(n, 0)].cpu().numpy().astype(np.int64), float(kept.abs().max())


def _rows(rng, rows, n_hot, canvas=(640, 384), wh=(40, 90), clusters=None, jitter=9.0, scores=None):
    raw = np.zeros((rows, 16), np.float32)
    raw[:, 4] = rng.uniform(0, 0.45, rows)
    hot = rng.choice(rows, n_hot, replace=False)
    if clusters:
        centers = rng.uniform((50, 50), (canvas[0] - 50, canvas[1] - 50), (clusters, 2))
        raw[hot, 0:2] = centers[np.arange(n_hot) % clusters] + rng.normal(0, jitter, (n_hot, 2))
    else:
        raw[hot, 0:2] = rng.uniform((0, 0), canvas, (n_hot, 2))
    raw[hot, 2:4] = rng.uniform(wh[0], wh[1], (n_hot, 2))
    raw[hot, 4] = rng.uniform(0.5001, 0.99, n_hot) if scores is None else scores
    raw[hot, 5:] = rng.normal(0, 1, (n_hot, 11))
    return raw


def _same_kept_as_oracle(idx, rows, want_idx, want_rows, what):
    """Kept rows of the GPU detector against the CPU oracle's: the same rows, ranked the same way up to boxes whose scores
    are closer than the two networks' rounding (about 1e-6 in obj; a crowd has thousands of candidates), which may swap."""
    assert len(idx) == len(want_idx), what
    assert np.array_equal(np.sort(idx), np.sort(want_idx)), what
    assert np.abs(rows[:, 4] - want_rows[:, 4]).max() < 1e-5, what
    swapped = idx != want_idx
    assert swapped.sum() <= max(2, len(idx) // 20), (what, int(swapped.sum()))


def _assert_same(got, want, what):
    (rows_g, idx_g), (rows_w, idx_w) = got, want
    assert np.array_equal(idx_g, idx_w), (what, len(idx_g), len(idx_w))
    assert np.array_equal(rows_g, rows_w), what


@pytest.mark.parametrize("n_hot", [1024, 1025])
def test_nms_at_the_old_candidate_limit(n_hot):
    raw = _rows(np.random.default_rng(n_hot), 15120, n_hot, clusters=40)
    rec = [0.3333333333333333, 0.0, 12.0]
    want = _nms_ranked(raw, rec)
    _assert_same(_post_batch([raw], [rec])[0], want, n_hot)
    # skps_detect_post keeps its contract: up to 1024 candidates the first 256 kept boxes, past that count = -candidates
    n, kept, idx, _ = _legacy(raw)
    if n_hot <= 1024:
        want1 = _nms_ranked(raw, [1.0, 0.0, 0.0])
        assert n == min(256, len(want1[1])) and np.array_equal(idx, want1[1][:n]) and np.array_equal(kept, want1[0][:n])
    else:
        assert n == -n_hot


def test_legacy_entry_refuses_more_than_1024_and_writes_nothing():
    raw = _rows(np.random.default_rng(11), 60480, 3000)
    n, _, _, peak = _legacy(raw)
    assert n == -3000 and peak == 0.0


def test_nms_5000_candidates_more_than_256_kept():
    raw = _rows(np.random.default_rng(5), 60480, 5000, canvas=(1280, 768), wh=(8, 30))
    rec = [0.5, 3.0, 7.0]
    want = _nms_ranked(raw, rec)
    assert len(want[1]) > 256
    got = _post_batch([raw], [rec])[0]
    _assert_same(got, want, "5000")
    from oracle import host_ref as H
    s = raw[raw[:, 4] > 0.5, 4]
    if len(np.unique(s)) == len(s):                    # no equal scores: the reference's own loop gives the same
        _assert_same(got, H.detect_post(raw.copy(), rec, 0.3, 0.5), "5000 host_ref")


def test_nms_every_row_over_the_threshold():
    rng = np.random.default_rng(6)
    raw = _rows(rng, 60480, 60480, canvas=(1280, 768), wh=(150, 220), clusters=24, jitter=6.0)
    rec = [1.0, 0.0, 0.0]
    want = _nms_ranked(raw, rec)
    _assert_same(_post_batch([raw], [rec])[0], want, "all rows")


def test_nms_equal_scores_rank_by_later_row_first():
    rng = np.random.default_rng(7)
    n_hot = 3000
    raw = _rows(rng, 15120, n_hot, clusters=60, jitter=12.0, scores=rng.choice([0.6, 0.7, 0.8], n_hot).astype(np.float32))
    rec = [1.0, 0.0, 0.0]
    want = _nms_ranked(raw, rec)
    got = _post_batch([raw], [rec])[0]
    _assert_same(got, want, "ties")
    # the tie rule decides: ranking equal scores by the earlier row first keeps other boxes
    flipped = _nms_ranked(raw[::-1].copy(), rec)[1]
    assert not np.array_equal(np.sort(raw.shape[0] - 1 - flipped), np.sort(want[1]))


def test_nms_batched_frames_one_without_candidates():
    rng = np.random.default_rng(8)
    rows = 15120
    raws = [_rows(rng, rows, 600, clusters=12), np.zeros((rows, 16), np.float32), _rows(rng, rows, 2500, canvas=(640, 384),
                                                                                         wh=(10, 40)),
            _rows(rng, rows, 1100, clusters=30)]
    raws[1][:, 4] = rng.uniform(0, 0.5, rows)
    recs = [[0.3333333333333333, 0.0, 12.0], [1.0, 0.0, 0.0], [0.5, 4.0, 0.0], [0.25, 0.0, 32.0]]
    got = _post_batch(raws, recs)
    assert len(got[1][1]) == 0
    for b in range(4):
        _assert_same(got[b], _nms_ranked(raws[b], recs[b]), b)
        _assert_same(_post_batch([raws[b]], [recs[b]])[0], got[b], ("alone", b))
    # a smaller capacity keeps the first boxes in rank order
    small = _post_batch(raws, recs, capacity=7)
    for b in range(4):
        assert np.array_equal(small[b][1], got[b][1][:7])


def _engine_raw(det):
    from peppa_pig_face_landmark_b200 import runtime as rt
    import ctypes as C
    lib = rt.load_library()
    buf = det.model.plan.outputs[0].buf.idx
    h, w, c, t = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    rt.check(lib.skps_engine_buffer_dims(det.model.handle, buf, C.byref(h), C.byref(w), C.byref(c), C.byref(t)))
    assert h.value * w.value * c.value == det._rows * 16
    raw = np.empty((det._rows, 16), np.float32)
    rt.check(lib.skps_engine_read_buffer(det.model.handle, buf, 1, raw.ctypes.data))
    return raw


@pytest.fixture(scope="module")
def detectors():
    return {hw: _detector(hw) for hw in sorted({v[2] for v in CROWDS.values()})}


@pytest.mark.parametrize("name", sorted(CROWDS))
def test_engine_output_through_nms(detectors, name):
    """The detector's own raw output, run through py_nms on the host, keeps exactly the rows the GPU kept: independent of
    GPU-versus-CPU detector rounding."""
    from peppa_pig_face_landmark_b200.core.api.face_detector import letterbox_geometry
    hw = CROWDS[name][2]
    det, fr = detectors[hw], crowd_frame(name)
    boxes = det(fr)
    raw = _engine_raw(det)
    scale, rw, rh, top, left = letterbox_geometry(fr.shape[0], fr.shape[1], *hw)
    kept, idx = _nms_ranked(raw, [scale, left, top])
    assert (raw[:, 4] > 0.5).sum() > 1024
    assert np.array_equal(det.last_keep_idx, idx), name
    assert np.array_equal(boxes, kept), name


@pytest.mark.parametrize("name", sorted(CROWDS))
def test_face_detector_matches_oracle_on_crowds(detectors, name):
    hw = CROWDS[name][2]
    fr = crowd_frame(name)
    boxes = detectors[hw](fr)
    want, idx = _detector_ref(hw)(fr, return_indices=True)
    assert len(idx) == {"crowd96_768x1280": 96, "crowd192_1152x1920": 192, "crowd384_1152x1920": 384}[name]
    _same_kept_as_oracle(detectors[hw].last_keep_idx, boxes, idx, want, name)
    order = np.argsort(detectors[hw].last_keep_idx)
    want = want[np.argsort(idx)]
    assert (np.abs(boxes[order] - want) < 5e-3 + 2e-5 * np.abs(want)).all(), name


@pytest.mark.parametrize("name,top_k", [("crowd96_768x1280", 16), ("crowd192_1152x1920", 16), ("crowd384_1152x1920", 16),
                                        ("crowd384_1152x1920", 64)])
def test_faceana_crowd_matches_oracle(name, top_k):
    from Skps import FaceAna
    hw = CROWDS[name][2]
    fr = crowd_frame(name)
    facer, ref = FaceAna(top_k=top_k, det_input=hw), _faceana_ref(hw, top_k)
    r0, w0 = facer.run(fr), ref.run(fr)
    want_rows, want_idx = ref.det(fr, return_indices=True)
    _same_kept_as_oracle(facer.last_det_idx, facer.last_det_rows, want_idx, want_rows, name)
    assert len(r0) == top_k
    _close(r0, w0, (name, top_k, 0))
    _close(facer.run(fr), ref.run(fr), (name, top_k, 1))          # unchanged frame: tracker path, no detector


def test_streams_run_a_crowd_next_to_ordinary_streams():
    """A 384-face crowd, a 1080p frame, test1 and a faceless frame in one batch: every stream returns what its own FaceAna
    returns, also after one stream is reset."""
    from Skps import FaceAna, FaceAnaStreams
    hw = (1152, 1920)
    crowd = crowd_frame("crowd384_1152x1920")
    hd, t1, empty = frames.frame_1080p(), frames.load_test1(), frames._background(480, 640)
    hd2 = frames.frame_1080p(jitter=(40, 24))
    seqs = [[crowd, crowd, hd, crowd, crowd], [hd, hd, hd2, crowd, hd2], [t1, t1, t1, t1, crowd], [empty, crowd, empty, t1, t1]]
    fa = FaceAnaStreams(n_streams=len(seqs), top_k=16, det_input=hw)
    singles = [FaceAna(top_k=16, det_input=hw) for _ in seqs]
    found = 0
    for t in range(len(seqs[0])):
        if t == 3:
            fa.reset(1)
            singles[1].reset()
        res = fa.run([s[t] for s in seqs])
        for k, s in enumerate(seqs):
            want = singles[k].run(s[t])
            assert len(res[k]) == len(want), (t, k)
            for x, y in zip(res[k], want):
                assert np.abs(np.asarray(x["kps"], np.float64) - np.asarray(y["kps"], np.float64)).max() <= 1e-6, (t, k)
                assert np.abs(np.asarray(x["box"], np.float64) - np.asarray(y["box"], np.float64)).max() <= 1e-6, (t, k)
                assert np.array_equal(x["scores"], y["scores"]), (t, k)
            found += len(want)
    assert found > 100
