"""Landmarks for every face of a crowd on the GPU: skps_select_faces at any top_k up to 1024 against judge_boxs +
sort_and_filter, and FaceAna with top_k past the landmark chunk (64 faces per forward) against the oracle: the 384-face
crowd over a short sequence, the chunk boundary, a faceless frame, aligned chips and head pose for every face."""
import numpy as np
import pytest

import frames
from test_crowd_cpu import crowd_frame
from test_detector_input_gpu import _close, _faceana_ref

pytestmark = pytest.mark.gpu

CHUNK = 64
MIN_FACE = 1600.0
IOU, ALPHA = 0.5, 0.3
# n_det -> number of track boxes it is judged against
N_TRACK = {0: 0, 1: 1, 64: 64, 65: 65, 1000: 1024, 4097: 256, 20000: 16}
TOP_K = (1, 5, 64, 65, 384, 1024)


def _sort_and_filter(boxes, min_face, top_k):
    """oracle.host_ref.sort_and_filter with the order of equal areas spelled out: later index first (argsort of a stable
    sort read backwards; the reference's default sort leaves equal areas unordered)."""
    if len(boxes) < 1:
        return np.zeros((0, 4), np.float32)
    area = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
    keep = area > min_face
    area, boxes = area[keep], boxes[keep]
    if boxes.shape[0] > top_k:
        return boxes[area.argsort(kind="stable")[-top_k:][::-1]]
    return boxes


def _synthetic(n_det, n_track, seed):
    """Detector rows (n_det, 16) on a 3840x2160 frame and track boxes (n_track, 4): about half the rows overlap a track
    box, many share an area with another row, and some have an area of exactly min_face or just above it."""
    rng = np.random.default_rng(seed)
    rows = np.zeros((n_det, 16), np.float32)
    xy = rng.uniform(0, 3600, (n_det, 2)) * [1, 0.55]
    wh = rng.choice([30.0, 40.0, 48.0, 64.0, 80.0, 100.0], (n_det, 2)) + rng.integers(0, 3, (n_det, 2)) * 0.5
    rows[:, 0:2], rows[:, 2:4] = xy, xy + wh
    rows[:, 4] = rng.uniform(0.5, 1.0, n_det)
    if n_det >= 8:
        edge = rng.choice(n_det, n_det // 8, replace=False)
        x = np.float32(6000) + np.arange(len(edge), dtype=np.float32) * 100          # far from every track box
        rows[edge, 0], rows[edge, 1] = x, 10.0
        rows[edge, 2], rows[edge, 3] = x + 40.0, 10.0 + np.where(np.arange(len(edge)) % 2, 40.0, 40.03125)
    track = np.zeros((n_track, 4), np.float32)
    if n_track:
        src = rows[rng.choice(n_det, min(n_track, n_det), replace=False), :4]
        track[:len(src)] = src + rng.normal(0, 4.0, src.shape)
        if n_track > n_det:
            track[n_det:] = _synthetic(n_track - n_det, 0, seed + 1)[0][:, :4]
    return rows, track


def _select(rows, track, top_k):
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    n = len(rows)
    d_rows = torch.from_numpy(np.ascontiguousarray(rows) if n else np.zeros((1, 16), np.float32)).cuda()
    d_cnt = torch.tensor([n], dtype=torch.int32, device="cuda")
    d_track = torch.from_numpy(track).cuda() if len(track) else None
    out = torch.full((top_k, 4), -7.0, dtype=torch.float32, device="cuda")
    cnt = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    rt.check(lib.skps_select_faces(d_rows.data_ptr(), d_cnt.data_ptr(), 16, None if d_track is None else d_track.data_ptr(),
                                   len(track), IOU, ALPHA, float(np.float32(1.0 - ALPHA)), MIN_FACE, top_k,
                                   out.data_ptr(), cnt.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    m = int(cnt.item())
    return m, out[:max(m, 0)].cpu().numpy()


@pytest.mark.parametrize("n_det", sorted(N_TRACK))
def test_select_faces_any_top_k(n_det):
    from oracle import host_ref as H
    rows, track = _synthetic(n_det, N_TRACK[n_det], n_det)
    judged = H.judge_boxs(track if len(track) else None, rows, IOU, ALPHA)
    judged = np.asarray(judged, np.float32).reshape(-1, judged.shape[-1] if len(judged) else 4)[:, :4]
    if n_det > 1024:
        area = (judged[:, 2] - judged[:, 0]) * (judged[:, 3] - judged[:, 1])
        assert len(np.unique(area[area > MIN_FACE])) < (area > MIN_FACE).sum() // 2       # many equal areas
        assert (area == MIN_FACE).any() and (area > MIN_FACE).sum() > 1024
    for top_k in TOP_K:
        want = _sort_and_filter(judged, MIN_FACE, top_k)
        m, got = _select(rows, track, top_k)
        assert m == len(want), (n_det, top_k, m, len(want))
        assert np.array_equal(got, want), (n_det, top_k)


def _close_on_grid(res, ref, what):
    """_close with both lists in grid order (row, then column of the box centre).  Below top_k the faces come in detector
    order, and two faces of the crowd whose scores the GPU and CPU networks round differently may swap there."""
    def order(rs):
        c = np.array([[(r["box"][1] + r["box"][3]) / 2, (r["box"][0] + r["box"][2]) / 2] for r in rs]).reshape(-1, 2)
        return [rs[i] for i in np.lexsort((np.round(c[:, 1] / 40), np.round(c[:, 0] / 40)))]
    _close(order(res), order(ref), what)


@pytest.fixture(scope="module")
def crowd384():
    return crowd_frame("crowd384_1152x1920")


def test_faceana_top_k_512_on_384_faces(crowd384):
    from Skps import FaceAna
    hw = (1152, 1920)
    facer, ref = FaceAna(top_k=512, det_input=hw), _faceana_ref(hw, 512)
    r0, w0 = facer.run(crowd384), ref.run(crowd384)
    assert len(r0) == 384
    _close_on_grid(r0, w0, "first")
    _close_on_grid(facer.run(crowd384), ref.run(crowd384), "unchanged")          # tracker path: GroupTrack at 384 faces
    for t, j in enumerate([(3, 2), (-4, 9)]):                                    # judge_boxs against 384 track boxes
        fr = frames.multi_face_frame(2160, 3840, (16, 24), 150, jitter=j)
        _close_on_grid(facer.run(fr), ref.run(fr), ("jitter", t))


@pytest.mark.parametrize("top_k", [CHUNK, CHUNK + 1])
def test_faceana_chunk_boundary(top_k):
    """96 faces with top_k 64 (one full chunk) and 65 (a full chunk and a last chunk of one face)."""
    from Skps import FaceAna
    hw = (768, 1280)
    fr = crowd_frame("crowd96_768x1280")
    facer, ref = FaceAna(top_k=top_k, det_input=hw), _faceana_ref(hw, top_k)
    r0 = facer.run(fr)
    assert len(r0) == top_k
    _close(r0, ref.run(fr), (top_k, 0))
    _close(facer.run(fr), ref.run(fr), (top_k, 1))


def test_faceana_1024_faceless_and_chunk_memory():
    from Skps import FaceAna
    facer = FaceAna(top_k=1024)
    assert facer.face_landmark.model.max_batch == CHUNK
    empty = frames._background(2160, 3840)
    assert facer.run(empty) == []
    assert facer.run(empty) == []
    assert len(facer.run(frames.load_test1())) == 1


def test_faceana_crowd_chips_and_pose(crowd384):
    from Skps import FaceAna
    facer = FaceAna(top_k=512, det_input=(1152, 1920), align=112, pose=True)
    plain = FaceAna(top_k=512, det_input=(1152, 1920))
    from Skps.core.headpose.pose import POSE_POINTS_98
    from test_headpose_edges_gpu import cost, cv2_solve, is_stationary, not_worse_bound, stationarity
    res, want = facer.run(crowd384), plain.run(crowd384)
    hw = crowd384.shape[:2]
    assert len(res) == 384
    for r, w in zip(res, want):
        assert np.array_equal(r["kps"], w["kps"]) and np.array_equal(r["box"], w["box"])
        assert r["chip"].shape == (112, 112, 3) and r["chip"].dtype == np.uint8 and r["chip"].any()
        assert r["M"].shape == (2, 3) and np.isfinite(r["M"]).all()
        p = r["pose"]
        assert p["euler"].shape == (3,) and np.isfinite(p["euler"]).all() and np.isfinite(p["reproject"]).all()
        # every face's pose is a stationary point of its reprojection error and no worse than cv2.solvePnP's
        img = np.asarray(r["kps"], np.float32)[POSE_POINTS_98]
        assert is_stationary(img, p["rvec"], p["tvec"], hw), stationarity(img, p["rvec"], p["tvec"], hw)
        assert cost(img, p["rvec"], p["tvec"], hw) <= not_worse_bound(img, *cv2_solve(img, hw), hw)
    # every face of the crowd is the same picture, so every chip is nearly the same
    chips = np.stack([r["chip"] for r in res]).astype(np.int16)
    assert np.median(np.abs(chips - chips[0]).mean(axis=(1, 2, 3))) < 20
