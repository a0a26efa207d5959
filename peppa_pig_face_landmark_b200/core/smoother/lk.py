"""Temporal smoothing of landmarks and boxes — host-side numpy, stateful.
Same classes and call signatures as the reference's Skps/core/smoother/lk.py (GroupTrack :6-91,
OneEuroFilter :105-149, EmaFilter :155-162).  The reference matches faces pair by pair in Python; here one
(n_now, n_prev) IoU matrix and one filter call per frame give bit for bit the same arrays, dtypes included."""
import math

import numpy as np


def _alpha(cutoff, t_e=1.0):
    r = 2 * math.pi * cutoff * t_e
    return r / (r + 1)


def _blend(a, x, x_prev):
    return a * x + (1 - a) * x_prev


def _bbox_of(points):
    return [np.min(points[:, 0]), np.min(points[:, 1]), np.max(points[:, 0]), np.max(points[:, 1])]


def rects(sets):
    """[min x, min y, max x, max y] of every landmark set (n, P, 2) -> (n, 4), in the sets' dtype."""
    return np.stack([sets[:, :, 0].min(1), sets[:, :, 1].min(1), sets[:, :, 0].max(1), sets[:, :, 1].max(1)], 1)


def first_match(r1, r2, thres):
    """For every row of r1 (n, 4), the first row of r2 (m, 4) with iou > thres, else -1: what the reference's loop
    `for prev in r2: if iou(now, prev) > thres: break` finds with _iou on numpy scalars."""
    n, m = r1.shape[0], r2.shape[0]
    if n == 0 or m == 0:
        return np.full(n, -1, np.int64)
    hit = iou_hits(r1, r2, thres)
    return np.where(hit.any(1), hit.argmax(1), -1)


def iou_hits(r1, r2, thres):
    """(n, m) bool: _iou(r1[i], r2[j]) > thres on numpy scalars of the rows' own dtypes, for n, m >= 1.

    Python's min / max return one of their operands, each with its own dtype, and numpy then computes in float32 only
    when both operands are float32 (float64 otherwise).  With r1 and r2 of different dtypes that choice is made per
    element, so each intermediate carries a "float32" flag next to its float64 value."""
    f32, f64 = np.float32, np.float64
    a32, b32 = r1.dtype == f32, r2.dtype == f32
    a, b = r1.astype(f64)[:, None, :], r2.astype(f64)[None, :, :]

    def pick(take_b, c):                 # value and float32 flag of `b[c] if take_b else a[c]`
        return np.where(take_b, b[..., c], a[..., c]), np.where(take_b, b32, a32)

    def sub(x, y):
        (xv, x32), (yv, y32) = x, y
        both = x32 & y32
        return np.where(both, (xv.astype(f32) - yv.astype(f32)).astype(f64), xv - yv), both

    with np.errstate(all="ignore"):      # the float32 branch of np.where is also evaluated on float64 values
        w = sub(pick(b[..., 2] < a[..., 2], 2), pick(b[..., 0] > a[..., 0], 0))     # min(r1[2], r2[2]) - max(r1[0], r2[0])
        h = sub(pick(b[..., 3] < a[..., 3], 3), pick(b[..., 1] > a[..., 1], 1))
        both = w[1] & h[1]
        inter = np.where(both, (w[0].astype(f32) * h[0].astype(f32)).astype(f64), w[0] * h[0])
        area1 = (r1[:, 2] - r1[:, 0]) * (r1[:, 3] - r1[:, 1])
        area2 = (r2[:, 2] - r2[:, 0]) * (r2[:, 3] - r2[:, 1])
        s = area1[:, None] + area2[None, :]                       # float32 only when both rects are float32
        inter = inter.astype(s.dtype)
        iou = inter / (s - inter)
        # max(0, w) * max(0, h) is 0 (iou 0 or nan) unless both are positive
        return (w[0] > 0) & (h[0] > 0) & (iou > thres)


def assign_track_ids(sources, prev_ids, next_id):
    """Track ids of one call's faces, in output order.  sources[i] is the index into prev_ids (the ids of the previous
    call's faces) of the track box face i continues, or -1.  A face inherits that id unless an earlier face of the call
    already took it; every other face, including one whose source is past the previous call's faces, gets the next unused
    number, as on the device.  Returns (ids as a list of ints, the new next_id)."""
    ids, taken = [], set()
    for s in sources:
        s = int(s)
        if 0 <= s < len(prev_ids) and prev_ids[s] not in taken:
            ids.append(prev_ids[s])
        else:
            ids.append(next_id)
            next_id += 1
        taken.add(ids[-1])
    return ids, next_id


MAX_ID_MEMORY = 2 ** 31 - 1      # frames: the device keeps each lost track's gap as an int32


class IdMemory:
    """Track ids with a memory of lost tracks (SORT's max_age, applied to ids only).  A track returned by one call and
    carried by no face of the next is lost; its id and its float32 box of the call that last returned it are remembered.
    A face that assign_track_ids would give a fresh number first takes the id of the first remembered track it overlaps
    with iou > iou_thres (both boxes float32, as judge_boxs compares two float32 rows) that has been missing for at most
    `frames` calls in a row; that entry is then forgotten.

    Entries are kept most recently lost first, tracks lost at the same call in the order their faces were returned.  At
    most `capacity` are kept: the oldest go first, and among tracks lost at the same call the last returned.  An entry
    whose gap can no longer qualify is dropped.  frames=0 keeps nothing, and assign() then gives assign_track_ids's ids."""

    def __init__(self, frames, capacity, iou_thres):
        self.frames, self.capacity, self.iou_thres = int(frames), int(capacity), iou_thres
        self.reset()

    def reset(self):
        self.ids = []                                # most recently lost first
        self.boxes = np.zeros((0, 4), np.float32)
        self.gaps = []                               # calls in a row without the track so far

    def assign(self, sources, boxes, prev_ids, prev_boxes, next_id):
        """One call: sources as for assign_track_ids, boxes (n, 4) the float32 boxes of this call's faces (the boxes the
        landmark stage used), prev_ids / prev_boxes (len(prev_ids), 4) the ids and float32 boxes of the previous call's
        faces.  Returns (ids as a list of ints, the new next_id) and remembers the tracks this call loses."""
        n, m = len(sources), len(self.ids)
        hit = None
        if n and m:
            hit = iou_hits(np.asarray(boxes, np.float32).reshape(-1, 4), self.boxes, self.iou_thres)
        ids, taken, used = [], set(), set()
        for i, s in enumerate(sources):
            s = int(s)
            if 0 <= s < len(prev_ids) and prev_ids[s] not in taken:
                ids.append(prev_ids[s])
            else:
                k = next((k for k in range(m) if k not in used and self.gaps[k] <= self.frames and hit[i, k]), None)
                if k is not None:
                    used.add(k)
                    ids.append(self.ids[k])
                else:
                    ids.append(next_id)
                    next_id += 1
            taken.add(ids[-1])
        lost = ([j for j, v in enumerate(prev_ids) if v not in taken] if self.frames else [])[:self.capacity]
        keep = [k for k in range(m) if k not in used and self.gaps[k] < self.frames][:self.capacity - len(lost)]
        prev_boxes = np.asarray(prev_boxes, np.float32).reshape(-1, 4)
        self.ids = [prev_ids[j] for j in lost] + [self.ids[k] for k in keep]
        self.boxes = np.concatenate([prev_boxes[lost], self.boxes[keep]]).reshape(-1, 4)
        self.gaps = [1] * len(lost) + [self.gaps[k] + 1 for k in keep]
        return ids, next_id


def _iou(r1, r2):
    a1 = (r1[2] - r1[0]) * (r1[3] - r1[1])
    a2 = (r2[2] - r2[0]) * (r2[3] - r2[1])
    w = max(0, min(r1[2], r2[2]) - max(r1[0], r2[0]))
    h = max(0, min(r1[3], r2[3]) - max(r1[1], r2[1]))
    inter = w * h
    return inter / (a1 + a2 - inter)


class OneEuroFilter:
    """One-Euro filter with unit time step; the derivative is the per-point displacement norm."""

    def __init__(self, dx0=0.0, min_cutoff=0.15, beta=0.8, d_cutoff=1):
        self.min_cutoff, self.beta, self.d_cutoff = min_cutoff, beta, d_cutoff

    def __call__(self, x, x_prev, dx_prev):
        """x, x_prev, dx_prev: (P, 2) for one face or (n, P, 2) for n faces at once."""
        speed = np.sqrt(np.sum((x - x_prev) ** 2, axis=-1))
        speed_prev = np.sqrt(np.sum(dx_prev ** 2, axis=-1))
        speed_hat = _blend(_alpha(self.d_cutoff), speed, speed_prev)
        a = _alpha(self.min_cutoff + self.beta * np.abs(speed_hat))
        a = np.expand_dims(a, -1)
        a[speed < 0.002] = 0.01            # nearly static points are held almost fixed
        self.dx_prev = speed_hat
        return _blend(a, x, x_prev)


class EmaFilter:
    def __init__(self, alpha):
        self.alpha = alpha

    def __call__(self, p_now, p_previous):
        return _blend(self.alpha, p_now, p_previous)


class GroupTrack:
    """Matches each face's landmark set to last frame's by bounding-box IoU and filters it."""

    def __init__(self, cfg):
        self.old_frame = None
        self.previous_landmarks_set = None
        self.with_landmark = True
        self.thres = cfg['pixel_thres']
        self.iou_thres = cfg['iou_thres']
        self.filter = OneEuroFilter()

    def iou(self, p_set0, p_set1):
        return _iou(_bbox_of(p_set0), _bbox_of(p_set1))

    def smooth(self, now_landmarks, previous_landmarks, previous_df):
        return self.filter(now_landmarks, previous_landmarks, previous_df)

    def calculate(self, img, now_landmarks_set):
        h, w = img.shape[0], img.shape[1]
        scale = [w, h]
        prev = self.previous_landmarks_set
        if prev is None or prev.shape[0] == 0:
            self.previous_landmarks_set = now_landmarks_set
            self.previous_dx = np.zeros_like(now_landmarks_set)
            return now_landmarks_set
        now = now_landmarks_set
        if now.shape[0] == 0:
            result, deltas = np.array([]), np.array([])
        else:
            match = first_match(rects(now), rects(prev), self.iou_thres)
            hit = match >= 0
            if not hit.any():
                result, deltas = now.copy(), np.zeros_like(now)
            else:
                # np.array of float32 and float64 rows is float64: unmatched rows are the landmarks as they came
                j = match[hit]
                f = self.smooth(now[hit] / scale, prev[j] / scale, self.previous_dx[j] / scale) * scale
                result = now.astype(np.float64)
                result[hit] = f
                deltas = np.zeros(now.shape, np.float64)
                deltas[hit] = prev[j] - f
        self.previous_landmarks_set = result
        self.previous_dx = deltas
        return result
