"""The device temporal layer of FaceAnaStreams (csrc/temporal.cu, mp_temporal_kernel) on its own, through
skps_debug_mp_temporal: scripted landmark sequences, with the state kept in torch tensors from launch to launch, bit for bit
against FaceAna's host layer as FaceAna.run applies it (GroupTrack.calculate, judge_boxs, assign_track_ids) and, on the
scripted streams, against the scalar loops of oracle.host_ref as well.

The scripts force the branches natural video never reaches: IoUs whose float32 and float64 values fall on either side of
Trace.iou_thres (both for the landmark-set match and for the track-box EMA), IoU exactly at the threshold, a first match that
is not the best one, two faces on one previous set, One-Euro speeds just either side of 0.002, frame size changes, empty
frames, every kind of track-id source, 64 faces per stream, 256 streams per launch and launches that cover only part of the
streams.  A coverage count asserts that the host trace met every forced case.  Last, the frame-difference gate of
FaceAnaStreams and FaceAna at exactly a mean difference of 5."""
import collections
import ctypes as C

import numpy as np
import pytest

import frames
from oracle import host_ref as H

pytestmark = pytest.mark.gpu

P = 98
F32, F64 = np.float32, np.float64
HW0 = (720, 1280)
SIZES = [(720, 1280), (480, 854), (1080, 1920), (361, 643)]
FORCED = ("gt_flip_prev_f32", "gt_flip_prev_f64", "ema_flip_now_f32", "ema_flip_now_f64", "gt_iou_at_thres",
          "ema_iou_at_thres", "dtype_f32_f64_f32", "first_match_not_best", "two_faces_one_prev", "more_prev_than_faces",
          "more_faces_than_prev", "euro_just_below", "euro_just_above", "euro_jump", "detector_after_skip",
          "empty_64_0_64", "size_change_matched", "count0_with_prev", "src_negative", "src_duplicate", "src_past_old",
          "inherit_at_63", "next_id_over_1000")


def _cfg(top_k):
    from peppa_pig_face_landmark_b200.core.api.facer import get_cfg, pipeline_cfg
    return pipeline_cfg(get_cfg()['Skps'], top_k, (2160, 3840))


def _trace_cfg():
    from peppa_pig_face_landmark_b200.core.api.facer import get_cfg
    return get_cfg()['Skps']['Trace']


def _same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    assert np.array_equal(a, b), what


# ----------------------------------------------------------------------------- IoU in three precisions
def _iou_variants(r1, r2):
    """IoU of two rectangles as facer.py / lk.py compute it on numpy scalars of the rows' own dtypes, then with both rows in
    float32 and both in float64."""
    return (H.iou_xyxy(r1, r2), H.iou_xyxy(r1.astype(F32), r2.astype(F32)),
            H.iou_xyxy(r1.astype(F64), r2.astype(F64)))


def _iou64(r1, r2):
    """(n, m) float64 IoU matrix (for choosing which pairs to look at closely)."""
    a, b = r1.astype(F64)[:, None, :], r2.astype(F64)[None, :, :]
    w = np.maximum(0, np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]))
    h = np.maximum(0, np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]))
    inter = w * h
    s = (a[..., 2] - a[..., 0]) * (a[..., 3] - a[..., 1]) + (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])
    with np.errstate(all="ignore"):
        return inter / (s - inter)


def _flipped(r1, r2, thres):
    """The host's decision iou > thres differs from the one in the other precision: float64 when both rows are float32,
    all-float32 otherwise."""
    host, v32, v64 = _iou_variants(r1, r2)
    alt = v64 if (r1.dtype == F32 and r2.dtype == F32) else v32
    return (host > thres) != (alt > thres)


def _flip_partner(fixed, thres, fixed_first, prefer=None):
    """A float32 rectangle q whose IoU with `fixed` lies on different sides of thres in the two precisions of _flipped:
    q spans `fixed` vertically and thres of its width, and its corners are walked over neighbouring float32 values.
    fixed_first: fixed is the first operand (judge_boxs: the landmark rectangle against boxes4), else the second
    (GroupTrack: this frame's rectangle against the previous set's).  prefer: True / False for a flip the host counts as a
    match / no match, if there is one."""
    f = fixed.astype(F64)
    base = np.array([f[0], f[1], f[0] + thres * (f[2] - f[0]), f[3]]).astype(F32)
    found = []
    for d3 in range(-4, 5):
        for d0 in range(-2, 3):
            for d2 in range(-48, 49):
                q = base.copy()
                q[0] = _ulps(q[0], d0)
                q[2] = _ulps(q[2], d2)
                q[3] = _ulps(q[3], d3)
                pair = (fixed, q) if fixed_first else (q, fixed)
                if _flipped(*pair, thres):
                    hit = _iou_variants(*pair)[0] > thres
                    if prefer is None or hit == prefer:
                        return q
                    found.append(q)
    assert found, ("no float32 / float64 flip near", fixed)
    return found[0]


def _ulps(x, k):
    x = F32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, F32(np.inf) if k > 0 else F32(-np.inf))
    return x


# ----------------------------------------------------------------------------- the host layer, one stream
class _Host:
    """One stream of FaceAna.run's host temporal layer after the landmark stage (facer.py: previous_landmarks_set = None
    on detector frames, GroupTrack.calculate, judge_boxs(boxes_return, rects(landmarks)), assign_track_ids), optionally
    checked against the scalar oracle, and counting the forced cases it meets."""

    def __init__(self, oracle=False):
        from peppa_pig_face_landmark_b200.core.api.facer import FaceAna
        from peppa_pig_face_landmark_b200.core.smoother.lk import EmaFilter, GroupTrack
        cfg = _trace_cfg()
        self.thres = cfg['iou_thres']
        self.gt = GroupTrack(cfg)
        self.fa = FaceAna.__new__(FaceAna)
        self.fa.iou_thres, self.fa.alpha = cfg['iou_thres'], cfg['smooth_box']
        self.fa.filter = EmaFilter(self.fa.alpha)
        self.ref = H.GroupTrackRef(cfg['iou_thres']) if oracle else None
        self.landmarks = np.zeros((0, P, 2), F32)
        self.track_box, self.ids, self.next_id = None, [], 0
        self.hits = collections.Counter()
        self.hist = []              # per launch: (flag, hw, n, dtype of the previous set or None)

    def track(self, flag, hw, kps):
        """GroupTrack of one frame; returns tmp_box, the rectangles judge_boxs gets."""
        from peppa_pig_face_landmark_b200.core.smoother.lk import rects
        img = np.broadcast_to(np.zeros(1, np.uint8), (hw[0], hw[1], 3))      # calculate reads only the shape
        if flag:
            self.gt.previous_landmarks_set = None
            if self.ref is not None:
                self.ref.prev = None
        now = kps.copy() if len(kps) else np.array([])
        self._count_track(flag, hw, now)
        got = self.gt.calculate(img, now)
        if self.ref is not None:
            _same(got, self.ref.calculate(img, now.copy()), "GroupTrackRef")
            _same(self.gt.previous_dx, self.ref.prev_dx, "GroupTrackRef dx")
        self.landmarks = got
        prev = self.gt.previous_landmarks_set
        self.hist.append((flag, tuple(hw), len(kps), None if len(prev) == 0 else prev.dtype))
        self._count_history()
        return rects(got) if got.shape[0] else np.array([])

    def judge(self, boxes4, tmp_box, src):
        from peppa_pig_face_landmark_b200.core.smoother.lk import assign_track_ids
        self._count_ema(boxes4, tmp_box)
        self.track_box = self.fa.judge_boxs(boxes4, tmp_box)
        if self.ref is not None:
            _same(self.track_box, H.judge_boxs(boxes4, tmp_box, self.fa.iou_thres, self.fa.alpha), "judge_boxs oracle")
        n_old, old = len(self.ids), list(self.ids)
        if len(boxes4):
            self.ids, self.next_id = assign_track_ids(src, self.ids, self.next_id)
        else:
            self.ids = []
        self._count_ids(src, n_old, old)

    # ---- coverage of the forced cases
    def _pairs(self, r1, r2, match):
        """The (i, j) pairs the reference loop evaluates (j up to i's first match) whose float64 IoU is near the threshold."""
        near = np.abs(_iou64(r1, r2) - self.thres) < 1e-4
        for i, j in zip(*np.nonzero(near)):
            if match[i] < 0 or j <= match[i]:
                yield i, j

    def _count_track(self, flag, hw, now):
        from peppa_pig_face_landmark_b200.core.smoother.lk import first_match, rects
        prev = self.gt.previous_landmarks_set
        n = now.shape[0]
        if self.hist and flag and self.hist[-1][0] == 0 and self.hist[-1][2] > 0:
            self.hits["detector_after_skip"] += 1
        if prev is None or prev.shape[0] == 0:
            return
        if n == 0:
            self.hits["count0_with_prev"] += 1
            return
        m = prev.shape[0]
        self.hits["more_prev_than_faces"] += m > n
        self.hits["more_faces_than_prev"] += n > m
        r1, r2 = rects(now), rects(prev)
        match = first_match(r1, r2, self.thres)
        for i, j in self._pairs(r1, r2, match):
            v = _iou_variants(r1[i], r2[j])[0]
            self.hits["gt_iou_at_thres"] += bool(v == self.thres)
            if _flipped(r1[i], r2[j], self.thres):
                self.hits["gt_flip_prev_f32" if prev.dtype == F32 else "gt_flip_prev_f64"] += 1
        hit = match >= 0
        if not hit.any():
            return
        iou = _iou64(r1, r2)
        for i in np.nonzero(hit)[0]:
            self.hits["first_match_not_best"] += bool(iou[i].max() > iou[i, match[i]] + 1e-6)
        self.hits["two_faces_one_prev"] += int(len(set(match[hit])) < hit.sum())
        if self.hist and tuple(hw) != self.hist[-1][1]:
            self.hits["size_change_matched"] += 1
        # One-Euro: normalised speeds of the matched faces, counted where the face also has a previous delta
        scale = [hw[1], hw[0]]
        j = match[hit]
        speed = np.sqrt(np.sum((now[hit] / scale - prev[j] / scale) ** 2, axis=-1))
        moving = (np.abs(self.gt.previous_dx[j]).reshape(len(j), -1).max(1) > 0)[:, None]
        self.hits["euro_just_below"] += int(((speed >= 0.00198) & (speed < 0.002) & moving).sum())
        self.hits["euro_just_above"] += int(((speed >= 0.002) & (speed <= 0.00202) & moving).sum())
        self.hits["euro_jump"] += int(((speed > 0.05) & moving).sum())

    def _count_history(self):
        ns = [h[2] for h in self.hist[-3:]]
        self.hits["empty_64_0_64"] += ns == [64, 0, 64]
        dts = [h[3] for h in self.hist[-3:]]
        self.hits["dtype_f32_f64_f32"] += dts == [np.dtype(F32), np.dtype(F64), np.dtype(F32)]

    def _count_ema(self, boxes4, tmp_box):
        from peppa_pig_face_landmark_b200.core.smoother.lk import first_match
        if len(tmp_box) == 0 or len(boxes4) == 0:
            return
        match = first_match(tmp_box, boxes4, self.thres)
        for i, j in self._pairs(tmp_box, boxes4, match):
            self.hits["ema_iou_at_thres"] += bool(_iou_variants(tmp_box[i], boxes4[j])[0] == self.thres)
            if _flipped(tmp_box[i], boxes4[j], self.thres):
                self.hits["ema_flip_now_f32" if tmp_box.dtype == F32 else "ema_flip_now_f64"] += 1

    def _count_ids(self, src, n_old, old):
        valid = [int(s) for s in src if 0 <= s < n_old]
        self.hits["src_negative"] += any(s < 0 for s in src)
        self.hits["src_past_old"] += any(s >= n_old for s in src)
        self.hits["src_duplicate"] += len(set(valid)) < len(valid)
        if n_old == 64:
            self.hits["inherit_at_63"] += any(int(s) == 63 and self.ids[i] == old[63] for i, s in enumerate(src))
        self.hits["next_id_over_1000"] += self.next_id > 1000


# ----------------------------------------------------------------------------- the device layer, S streams
class _Device:
    """The state of S streams in torch tensors, started where skps_mpipe_create / skps_mpipe_reset leave it."""

    def __init__(self, S, K):
        import torch
        from peppa_pig_face_landmark_b200 import runtime as rt
        self.torch, self.lib, self.S, self.K = torch, rt.load_library(), S, K
        self.cfg = _cfg(K)
        dev, f64, i32 = "cuda", torch.float64, torch.int32
        z = lambda *shape, dt=f64: torch.zeros(shape, dtype=dt, device=dev)        # noqa: E731
        self.inp = dict(kps_now=z(S, K, P, 2, dt=torch.float32), count=z(S, dt=i32), flag=z(S, dt=i32), hw=z(S, 2, dt=i32),
                        boxes4=z(S, K, 4, dt=torch.float32), src=z(S, K, dt=i32))
        self.state = dict(prev_lm=z(S, 2, K, P, 2), prev_dx=z(S, 2, K, P, 2), n_prev=z(S, dt=i32) - 1,
                          prev_f32=z(S, dt=i32) + 1, state_idx=z(S, dt=i32), track_box=z(S, K, 4),
                          track_f32=z(S, K, 4, dt=torch.float32), n_track=z(S, dt=i32), ids=z(S, K, dt=torch.int64) - 1,
                          next_id=z(S, dt=torch.int64), out_kps=z(S, K, P, 2))

    def launch(self, n, arrays):
        torch = self.torch
        for k, v in arrays.items():
            self.inp[k].copy_(torch.from_numpy(v))
        before = {k: v.clone() for k, v in self.state.items()} if n < self.S else None
        i, s = self.inp, self.state
        from peppa_pig_face_landmark_b200 import runtime as rt
        rt.check(self.lib.skps_debug_mp_temporal(
            C.byref(self.cfg), n, self.K, P, i["kps_now"].data_ptr(), i["count"].data_ptr(), i["flag"].data_ptr(),
            i["hw"].data_ptr(), i["boxes4"].data_ptr(), i["src"].data_ptr(), s["prev_lm"].data_ptr(),
            s["prev_dx"].data_ptr(), s["n_prev"].data_ptr(), s["prev_f32"].data_ptr(), s["state_idx"].data_ptr(),
            s["track_box"].data_ptr(), s["track_f32"].data_ptr(), s["n_track"].data_ptr(), s["ids"].data_ptr(),
            s["next_id"].data_ptr(), s["out_kps"].data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        if before is not None:
            for k, v in self.state.items():          # streams the launch did not cover: every byte as it was
                assert torch.equal(v[n:].view(torch.uint8), before[k][n:].view(torch.uint8)), ("uncovered stream changed", k)
        return {k: v[:n].cpu().numpy() for k, v in self.state.items()}


def _check(st, s, host, what):
    """Stream s of the device state after a launch against its host layer."""
    n = len(host.ids) if len(host.track_box) else 0
    g = host.gt
    prev = g.previous_landmarks_set
    assert st["n_track"][s] == len(host.track_box) == n, (what, st["n_track"][s], len(host.track_box))
    assert st["n_prev"][s] == len(prev), (what, st["n_prev"][s], len(prev))
    assert st["next_id"][s] == host.next_id, (what, st["next_id"][s], host.next_id)
    if n == 0:
        return
    # the dtype of an empty previous set is never read: GroupTrack starts over whenever it has no rows
    assert st["prev_f32"][s] == (prev.dtype == F32), (what, st["prev_f32"][s], prev.dtype)
    _same(st["out_kps"][s, :n], host.landmarks.astype(F64), (what, "kps"))
    _same(st["track_box"][s, :n], host.track_box.astype(F64), (what, "box"))
    _same(st["track_f32"][s, :n], host.track_box.astype(F32), (what, "box f32"))
    _same(st["ids"][s, :n], np.array(host.ids, np.int64), (what, "ids"))
    half = st["state_idx"][s]
    _same(st["prev_lm"][s, half, :n], prev.astype(F64), (what, "previous set"))
    _same(st["prev_dx"][s, half, :n], g.previous_dx.astype(F64), (what, "previous delta"))


def _run(scripts, K, launches, cover=None, oracle=()):
    """Runs len(scripts) streams for `launches` launches; cover(t) is the number of streams launch t covers (default all).
    Every launch is checked stream by stream; returns the host layers."""
    S = len(scripts)
    hosts = [_Host(oracle=s in oracle) for s in range(S)]
    gens = [make(hosts[s], np.random.default_rng(1000 + s), K) for s, make in enumerate(scripts)]
    dev = _Device(S, K)
    for t in range(launches):
        n = S if cover is None else cover(t)
        arrays = dict(kps_now=np.zeros((S, K, P, 2), F32), count=np.zeros(S, np.int32), flag=np.zeros(S, np.int32),
                      hw=np.ones((S, 2), np.int32), boxes4=np.zeros((S, K, 4), F32), src=np.full((S, K), -1, np.int32))
        for s in range(n):
            fr = next(gens[s])
            k = len(fr["kps"])
            assert k <= K
            tmp = hosts[s].track(fr["flag"], fr["hw"], fr["kps"])
            boxes = fr["boxes"](tmp) if callable(fr["boxes"]) else fr["boxes"]
            boxes = np.asarray(boxes, F32).reshape(k, 4)
            src = np.asarray(fr["src"], np.int32).reshape(k)
            hosts[s].judge(boxes, tmp, src)
            arrays["kps_now"][s, :k] = fr["kps"]
            arrays["count"][s], arrays["flag"][s], arrays["hw"][s] = k, fr["flag"], fr["hw"]
            arrays["boxes4"][s, :k], arrays["src"][s, :k] = boxes, src
        st = dev.launch(n, arrays)
        for s in range(n):
            _check(st, s, hosts[s], (t, s))
    return hosts


# ----------------------------------------------------------------------------- building frames
def _sets(rng, rects):
    """float32 landmark sets whose min / max rectangles are exactly the float32 `rects` (points 0 and 1 are the corners)."""
    r = np.asarray(rects, F32).reshape(-1, 4)
    t = rng.uniform(0.05, 0.95, (len(r), P, 2))
    lo, hi = r[:, None, :2].astype(F64), r[:, None, 2:].astype(F64)
    pts = np.clip((lo + t * (hi - lo)).astype(F32), r[:, None, :2], r[:, None, 2:])
    pts[:, 0], pts[:, 1] = r[:, :2], r[:, 2:]
    return pts


def _frame(kps, flag=0, hw=HW0, boxes=None, src=None):
    n = len(kps)
    return dict(flag=flag, hw=hw, kps=np.asarray(kps, F32).reshape(n, P, 2),
                boxes=_boxes_close if boxes is None else boxes, src=np.arange(n) if src is None else src)


def _boxes_close(tmp):
    """boxes4 that each face's own rectangle overlaps by far more than the threshold (the EMA runs)."""
    return np.asarray(tmp, F64).reshape(-1, 4).astype(F32) + F32(0.75) if len(tmp) else np.zeros((0, 4), F32)


def _follow(h, rng, px=0.3):
    """This frame's landmarks: the last result moved by a little noise (every face matches its previous set)."""
    return (h.landmarks.astype(F64) + rng.normal(0, px, h.landmarks.shape)).astype(F32)


def _grid(n, hw=HW0, rows=8):
    """n small non-overlapping face rectangles on a grid of the frame."""
    cols = -(-n // rows)
    ch, cw = hw[0] / rows, hw[1] / cols
    return np.array([[c * cw + 5.25, r * ch + 4.5, (c + 1) * cw - 6.5, (r + 1) * ch - 3.75]
                     for r in range(rows) for c in range(cols)][:n], F32)


def _random(h, rng, K, hw=HW0):
    """Seeded random sequence: faces that stay (small moves, or moves that put the IoU near the threshold), leave and
    arrive, detector frames, frame size changes, boxes4 near the threshold and track-id sources of every kind."""
    while True:
        if rng.random() < 0.05:
            hw = SIZES[rng.integers(len(SIZES))]
        prev = h.landmarks if h.landmarks.ndim == 3 else np.zeros((0, P, 2), F32)
        m = len(prev)
        n = int(rng.integers(0, K + 1)) if rng.random() < 0.25 else int(np.clip(m + rng.integers(-2, 3), 0, K))
        keep = rng.permutation(m)[:n]
        faces, src = [], []
        for j in keep:
            p = prev[j].astype(F64)
            mode = rng.random()
            if mode < 0.5:
                p = p + rng.normal(0, rng.choice([0.05, 0.5, 3.0]), p.shape)
            elif mode < 0.8:                       # shifted by a third of the width: IoU about 1/2
                wdt = p[:, 0].max() - p[:, 0].min()
                p = p + [wdt / 3 * (1 + rng.normal(0, 0.01)), 0]
            else:                                  # a few points jump inside the face
                k = rng.choice(P, 8, replace=False)
                p[k] = p[k].min(0) + rng.uniform(0, 1, (8, 2)) * (p.max(0) - p.min(0))
            faces.append(p.astype(F32))
            u = rng.random()
            src.append(int(j) if u < 0.8 else int(rng.integers(-1, m + 3)))
        while len(faces) < n:
            x, y = rng.uniform(0, hw[1] - 120), rng.uniform(0, hw[0] - 120)
            w = rng.uniform(40, 120)
            faces.append(_sets(rng, [[x, y, x + w, y + w * rng.uniform(0.8, 1.3)]])[0])
            src.append(-1)
        yield dict(flag=int(rng.random() < 0.15), hw=hw, kps=np.array(faces, F32).reshape(len(faces), P, 2),
                   boxes=lambda tmp, r=rng: _boxes_random(tmp, r), src=src)


def _boxes_random(tmp, rng):
    out = []
    for r in np.asarray(tmp, F64).reshape(-1, 4):
        u = rng.random()
        if u < 0.5:
            out.append(r + rng.normal(0, 0.5, 4))
        elif u < 0.8:
            out.append(r + [(r[2] - r[0]) / 3 * (1 + rng.normal(0, 0.01)), 0, (r[2] - r[0]) / 3, 0])
        else:
            out.append(r + 2000)
    return np.array(out, F64).reshape(-1, 4).astype(F32)


# ----------------------------------------------------------------------------- the forced scripts
def _s_ids(h, rng, K):
    """64 faces; sources -1, duplicated, past the old count, and inheritance from track box 63 (the last bit of the mask)."""
    yield _frame(_sets(rng, _grid(64)), flag=1, src=np.full(64, -1))
    src = np.arange(64)
    src[1] = src[2] = 0                 # face 2 asks for the id face 1 took: a new one
    src[3] = -1
    src[4], src[5] = 64, 1000           # past the old track boxes: new ids
    yield _frame(_follow(h, rng), src=src)                      # face 63 inherits from box 63
    src = np.arange(64)
    src[0] = 63                         # box 63's id goes to face 0; face 63 gets a new one
    yield _frame(_follow(h, rng), src=src)
    yield from _random(h, rng, K)


def _s_gt_flip(h, rng, K):
    """One wide face whose rectangle is walked over float32 neighbours until the float32 and float64 IoU with the previous
    set fall on either side of the threshold, against a float32 and a float64 previous set, matching and not."""
    from peppa_pig_face_landmark_b200.core.smoother.lk import rects
    face = np.array([[0.75, 8.5, 1201.3, 700.6]], F32)
    for prefer in (True, False):
        yield _frame(_sets(rng, face), flag=1)                                  # previous set float32
        q = _flip_partner(rects(h.gt.previous_landmarks_set)[0], h.thres, False, prefer)
        yield _frame(_sets(rng, q))
        yield _frame(_sets(rng, face), flag=1)
        yield _frame(_follow(h, rng))                                           # previous set float64
        q = _flip_partner(rects(h.gt.previous_landmarks_set)[0], h.thres, False, prefer)
        yield _frame(_sets(rng, q))
    yield from _random(h, rng, K)


def _flip_boxes(prefer):
    def make(tmp):
        return np.array([_flip_partner(r, _trace_cfg()['iou_thres'], True, prefer) for r in tmp], F32)
    return make


def _s_ema_flip(h, rng, K):
    """boxes4 walked over float32 neighbours until the EMA match of a float32 and of a float64 landmark rectangle differs
    between the precisions."""
    faces = np.array([[0.5, 3.25, 610.3, 700.1], [650.2, 10.7, 1270.9, 690.3]], F32)
    for prefer in (True, False):
        yield _frame(_sets(rng, faces), flag=1, boxes=_flip_boxes(prefer))   # landmarks float32
        yield _frame(_sets(rng, faces), flag=1)
        yield _frame(_follow(h, rng), boxes=_flip_boxes(prefer))             # landmarks float64
    yield from _random(h, rng, K)


def _s_dtypes(h, rng, K):
    """previous sets float32 -> float64 -> float32 twice: through a frame where every face moves away and through a
    detector frame."""
    faces = _grid(6)
    yield _frame(_sets(rng, faces), flag=1)
    yield _frame(_follow(h, rng))
    yield _frame(_follow(h, rng) + F32(300))                                # nothing matches: the rows as they came
    yield _frame(_follow(h, rng))
    yield _frame(_follow(h, rng), flag=1)
    yield from _random(h, rng, K)


def _s_exact(h, rng, K):
    """IoU exactly 1/2 (dyadic rectangles): no match, for the landmark sets and for the EMA."""
    prev = np.array([[64, 32, 64 + 2 * 96, 32 + 96], [512, 256, 512 + 2 * 40, 256 + 40]], F32)
    now = prev.copy()
    now[:, 2] = now[:, 0] + (prev[:, 2] - prev[:, 0]) / 2
    yield _frame(_sets(rng, prev), flag=1)
    yield _frame(_sets(rng, now), boxes=prev)                               # both IoUs exactly 0.5
    yield _frame(_sets(rng, prev), flag=1, boxes=now)
    yield from _random(h, rng, K)


def _s_order(h, rng, K):
    """The first matching previous set is not the best, two faces on one previous set, then fewer and more faces than
    previous sets."""
    a, b = [100, 100, 300, 300], [120, 100, 320, 300]           # IoU(a, b) = 0.8
    prev = np.array([a, b, [800, 100, 1000, 300], [800, 400, 1000, 600]], F32)
    yield _frame(_sets(rng, prev), flag=1)
    yield _frame(_sets(rng, np.array([b, [101, 99, 302, 301]], F32)))   # both match set 0 first; face 0 is set 1 exactly
    more = np.concatenate([_follow(h, rng), _sets(rng, _grid(5)[2:])])
    yield _frame(more)
    yield from _random(h, rng, K)


def _s_euro(h, rng, K):
    """One face whose points move at normalised speeds just under and just over 0.002, and some that jump, after a frame
    that gave every point a previous delta."""
    yield _frame(_sets(rng, [[300.5, 150.25, 700.75, 550.5]]), flag=1)
    yield _frame((h.landmarks.astype(F64) + [3.0, -2.0] + rng.normal(0, 0.5, h.landmarks.shape)).astype(F32))
    for _ in range(3):
        W = HW0[1]
        q = h.gt.previous_landmarks_set[0].astype(F64)
        now = q.copy()
        for p in range(2, P):
            g = p % 4
            sign = 1 if p % 8 < 4 else -1
            if g == 0:
                now[p, 0] += sign * 0.002 * (1 - rng.uniform(0.001, 0.008)) * W
            elif g == 1:
                now[p, 0] += sign * 0.002 * (1 + rng.uniform(0.001, 0.008)) * W
            elif g == 2:
                now[p] = q.min(0) + rng.uniform(0.1, 0.9, 2) * (q.max(0) - q.min(0))   # a jump inside the face
        yield _frame(now.astype(F32)[None])
    yield from _random(h, rng, K)


def _s_empty(h, rng, K):
    """64 faces, none, 64 again (a first frame without the detector), then a detector frame after skipped ones."""
    yield _frame(_sets(rng, _grid(64)), flag=1)
    yield _frame(_follow(h, rng))
    keep = h.landmarks
    yield _frame(np.zeros((0, P, 2), F32))
    yield _frame(keep.astype(F32))
    yield _frame(_follow(h, rng))
    yield _frame(_follow(h, rng), flag=1)
    yield from _random(h, rng, K)


def _s_size(h, rng, K):
    """Matched faces while the frame size changes (the One-Euro normalisation by W and H)."""
    yield _frame(_sets(rng, _grid(3)), flag=1)
    yield _frame(_follow(h, rng, 1.0))
    for hw in ((480, 854), (1080, 1920), (361, 643)):
        yield _frame(_follow(h, rng, 1.0), hw=hw)
    yield from _random(h, rng, K)


def _s_churn(h, rng, K):
    """K faces that keep moving a little, about half of them with a source: next_id grows by about K / 2 a launch."""
    yield _frame(_sets(rng, _grid(K)), flag=1, src=np.full(K, -1))
    while True:
        src = np.where(rng.random(K) < 0.5, -1, rng.integers(-1, K + 4, K))
        yield _frame(_follow(h, rng, 0.5), flag=int(rng.random() < 0.1), src=src, boxes=lambda tmp: _boxes_random(tmp, rng))


def _random_script(h, rng, K):
    yield from _random(h, rng, K)


FORCED_SCRIPTS = [_s_ids, _s_gt_flip, _s_ema_flip, _s_dtypes, _s_exact, _s_order, _s_euro, _s_empty, _s_size]


def test_forced_cases_match_the_host_layer_and_the_oracle():
    """K = 64, 16 streams: the forced scripts then random sequences, every fourth launch covering half the streams, all of
    it also against the scalar oracle; then 300 launches that cover 2 of 16 streams, one of them churning through ids."""
    S, K = 16, 64
    scripts = FORCED_SCRIPTS + [_random_script] * (S - len(FORCED_SCRIPTS))
    hosts = _run(scripts, K, 24, cover=lambda t: S if t % 4 != 3 else S // 2, oracle=range(S))
    hits = sum((h.hits for h in hosts), collections.Counter())
    tail = _run_tail(K, 300)
    hits.update(tail)
    counts = {k: hits[k] for k in FORCED}
    print("forced cases:", counts)
    assert all(counts.values()), "forced cases never met: %s (all counts: %s)" % ([k for k, v in counts.items() if not v],
                                                                                  counts)


def _run_tail(K, launches):
    """A random sequence and one whose ids churn, for many launches (next_id grows), each launch but the first covering
    2 of 16 streams."""
    hosts = _run([_random_script, _s_churn] + [_random_script] * 14, K, launches, cover=lambda t: 2 if t else 16)
    return sum((h.hits for h in hosts), collections.Counter())


@pytest.mark.parametrize("K", [1, 5, 64])
def test_random_sequences_256_streams(K):
    """256 streams in one launch at K = 1, 5 and 64, seeded random sequences with jitter around the thresholds; every
    third launch covers 100 streams and leaves the other 156 as they were."""
    S = 256
    hosts = _run([_random_script] * S, K, 12, cover=lambda t: S if t % 3 != 2 else 100, oracle=range(4))
    assert sum(h.next_id for h in hosts) > 0
    assert max(n for h in hosts for _, _, n, _ in h.hist) == K


def test_debug_entry_refuses_bad_arguments():
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    dev = _Device(2, 4)
    i, s = dev.inp, dev.state
    ptrs = [i[k].data_ptr() for k in ("kps_now", "count", "flag", "hw", "boxes4", "src")] + \
           [s[k].data_ptr() for k in ("prev_lm", "prev_dx", "n_prev", "prev_f32", "state_idx", "track_box", "track_f32",
                                      "n_track", "ids", "next_id", "out_kps")]
    for k in (0, 65):
        assert lib.skps_debug_mp_temporal(C.byref(_cfg(4)), 2, k, P, *ptrs, None) != 0
        assert b"top_k" in lib.skps_last_error()
    for at in range(len(ptrs)):
        bad = list(ptrs)
        bad[at] = None
        assert lib.skps_debug_mp_temporal(C.byref(_cfg(4)), 2, 4, P, *bad, None) != 0
    assert lib.skps_debug_mp_temporal(None, 2, 4, P, *ptrs, None) != 0


# ----------------------------------------------------------------------------- the frame-difference gate
def _gate_frames(h, w):
    """Faceless frames whose byte difference to the frame before sums to 15 H W (mean exactly 5: no detector) or one more
    or one less."""
    f0 = frames._background(h, w).astype(np.int16)
    d = np.full(f0.shape, 5, np.int16)
    f1 = f0 + d                                     # 15 H W
    d2 = d.copy()
    d2.reshape(-1)[-1] += 1
    f2 = f1 + d2                                    # 15 H W + 1, the extra byte last
    d3 = -d
    d3.reshape(-1)[d3.size // 2] += 1
    f3 = f2 + d3                                    # 15 H W - 1
    d4 = d.copy()
    d4.reshape(-1)[0] += 1
    f4 = f3 + d4                                    # 15 H W + 1, the extra byte first
    return [f.astype(np.uint8) for f in (f0, f1, f2, f3, f4)], [True, False, True, False, True]


def test_frame_difference_gate_at_exactly_five():
    """mp_decide_kernel, FaceAna.diff_frames and np.sum(diff) / H / W / 3. > 5 decide alike at odd frame sizes; a mean of
    exactly 5 does not run the detector."""
    from Skps import FaceAna, FaceAnaStreams
    sizes = [(719, 1279), (33, 31)]
    seqs = [_gate_frames(h, w) for h, w in sizes]
    streams = FaceAnaStreams(n_streams=len(sizes))
    singles = [FaceAna() for _ in sizes]
    for t in range(5):
        res = streams.run([fr[t] for fr, _ in seqs])
        assert all(len(r) == 0 for r in res)
        for k, ((fr, want), (h, w)) in enumerate(zip(seqs, sizes)):
            singles[k].last_det_rows = None
            assert singles[k].run(fr[t]) == []
            host = singles[k].last_det_rows is not None
            formula = t == 0 or np.sum(np.abs(fr[t].astype(np.int64) - fr[t - 1])) / h / w / 3. > 5
            assert bool(streams.last_ran_detector[k]) == host == formula == want[t], (t, (h, w))
