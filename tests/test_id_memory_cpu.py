"""Id memory without a GPU: the host rule FaceAna(track_ids=True, id_memory=m) applies (core/smoother/lk.py IdMemory)
against a restatement written out here on hand-built and random calls, argument checks of FaceAna and FaceAnaStreams, and
the two C exports of FaceAnaStreams' id memory, declared in the header and bound in runtime.py."""
import ctypes as C

import numpy as np
import pytest

from oracle import host_ref as H
from test_c_abi_cpu import _header_arity

IOU = 0.5
F32 = np.float32


class _Restated:
    """The rule as the feature states it, with frame numbers: a track returned at frame a and carried by no face of frame
    a + 1 is remembered as (id, its float32 box of frame a, a).  A face at frame b that would get a fresh number takes the
    id of the first entry, most recently lost first, with b - a - 1 <= m and float32 IoU(face box, entry box) > 0.5.  At
    most cap entries: unqualifiable ones are dropped, then the oldest (the last returned among the same frame)."""

    def __init__(self, m, cap):
        self.m, self.cap = m, cap
        self.reset()

    def reset(self):
        self.frame, self.mem, self.ids, self.boxes, self.next_id = 0, [], [], np.zeros((0, 4), F32), 0

    def call(self, sources, boxes, returned):
        b = self.frame
        out = []
        for i, s in enumerate(sources):
            if 0 <= s < len(self.ids) and self.ids[s] not in out:
                out.append(self.ids[s])
                continue
            entry = None
            for e in self.mem:
                if b - e[2] - 1 <= self.m and H.iou_xyxy(np.asarray(boxes[i], F32), e[1]) > IOU:
                    entry = e
                    break
            if entry is not None:
                self.mem.remove(entry)
                out.append(entry[0])
            else:
                out.append(self.next_id)
                self.next_id += 1
        lost = [(v, self.boxes[j].copy(), b - 1) for j, v in enumerate(self.ids) if v not in out]
        self.mem = [e for e in lost + self.mem if (b + 1) - e[2] - 1 <= self.m][:self.cap]
        self.ids, self.boxes = out, np.asarray(returned, F32).reshape(-1, 4)
        self.frame += 1
        return out

    def contents(self):
        """(ids, boxes, frames missing so far) of the entries, in order."""
        return ([e[0] for e in self.mem], np.array([e[1] for e in self.mem], F32).reshape(-1, 4),
                [self.frame - e[2] - 1 for e in self.mem])


class _Host:
    """IdMemory driven as FaceAna drives it: the previous call's ids and returned boxes go back in."""

    def __init__(self, m, cap):
        from peppa_pig_face_landmark_b200.core.smoother.lk import IdMemory
        self.mem = IdMemory(m, cap, IOU)
        self.ids, self.boxes, self.next_id = [], np.zeros((0, 4), F32), 0

    def call(self, sources, boxes, returned):
        self.ids, self.next_id = self.mem.assign(np.asarray(sources, np.int32), np.asarray(boxes, F32).reshape(-1, 4),
                                                 self.ids, self.boxes, self.next_id)
        self.boxes = np.asarray(returned, F32).reshape(-1, 4)
        return self.ids

    def reset(self):
        self.mem.reset()
        self.ids, self.boxes, self.next_id = [], np.zeros((0, 4), F32), 0


def _pair(m, cap):
    return _Restated(m, cap), _Host(m, cap)


def _both(r, h, sources, boxes, returned=None):
    returned = boxes if returned is None else returned
    want = r.call(list(sources), boxes, returned)
    got = h.call(sources, boxes, returned)
    assert got == want, (got, want)
    assert all(type(i) is int for i in got)
    ids, bx, gaps = r.contents()
    assert h.mem.ids == ids and h.mem.gaps == gaps, ((h.mem.ids, h.mem.gaps), (ids, gaps))
    assert h.mem.boxes.dtype == F32 and np.array_equal(h.mem.boxes, bx)
    assert h.next_id == r.next_id
    return got


BOX = {k: np.array(v, F32) for k, v in dict(a=[100, 100, 200, 200], b=[400, 100, 500, 200], c=[100, 400, 200, 500],
                                              d=[400, 400, 500, 500], e=[700, 100, 800, 200]).items()}


def _boxes(*names, shift=0.0):
    return np.array([BOX[n] + F32(shift) for n in names], F32).reshape(-1, 4)


@pytest.mark.parametrize("m", [1, 2, 5])
def test_a_gap_of_id_memory_frames_revives_the_id_and_one_more_does_not(m):
    for gap, revived in ((m, True), (m + 1, False)):
        r, h = _pair(m, 5)
        assert _both(r, h, [-1, -1], _boxes("b", "a")) == [0, 1]
        for _ in range(gap):
            assert _both(r, h, [0], _boxes("b")) == [0]             # face a missing
        got = _both(r, h, [0, -1], _boxes("b", "a", shift=3.0))
        assert got == ([0, 1] if revived else [0, 2]), (gap, got)


def test_a_source_beats_memory():
    r, h = _pair(3, 5)
    _both(r, h, [-1, -1], _boxes("a", "b"))                         # ids 0, 1
    _both(r, h, [1], _boxes("b"))                                   # a lost: entry 0
    # a face where a was, continuing track 0 (id 1): its source wins over the entry it overlaps
    assert _both(r, h, [0], _boxes("a")) == [1]
    assert h.mem.ids == [0]
    # a second face continuing the same track and overlapping the entry: the source is taken, so it gets the entry
    assert _both(r, h, [0, 0], _boxes("a", "a")) == [1, 0]


def test_memory_order_most_recently_lost_first_then_return_order():
    # the faces are found at e and d, but their returned boxes (what the entries keep) are all at a
    r, h = _pair(5, 8)
    _both(r, h, [-1], _boxes("e"), returned=_boxes("a"))            # id 0
    _both(r, h, [], _boxes())                                       # 0 lost at frame 1
    _both(r, h, [-1, -1], _boxes("e", "d"), returned=_boxes("a", "a"))      # ids 1, 2
    _both(r, h, [], _boxes())                                       # 1 and 2 lost at frame 3, in return order
    assert h.mem.ids == [1, 2, 0] and h.mem.gaps == [1, 1, 3]
    # three faces at a, each overlapping every entry: most recently lost first, then return order
    assert _both(r, h, [-1, -1, -1, -1], _boxes("a", "a", "a", "a")) == [1, 2, 0, 3]
    assert h.mem.ids == []


def test_an_entry_is_given_out_once():
    r, h = _pair(4, 5)
    _both(r, h, [-1], _boxes("a"))
    _both(r, h, [], _boxes())
    assert _both(r, h, [-1, -1], _boxes("a", "a")) == [0, 1]
    assert h.mem.ids == []


def test_eviction_at_top_k_entries():
    r, h = _pair(9, 2)
    _both(r, h, [-1, -1, -1], _boxes("a", "b", "c"))                # 0, 1, 2
    _both(r, h, [], _boxes())                                       # all lost: the last returned (2) goes
    assert h.mem.ids == [0, 1]
    _both(r, h, [-1], _boxes("d"))                                  # 3
    _both(r, h, [], _boxes())                                       # 3 lost: the oldest (1) goes
    assert h.mem.ids == [3, 0]
    assert _both(r, h, [-1, -1, -1], _boxes("b", "a", "d")) == [4, 0, 3]


def test_an_empty_frame_loses_every_track():
    r, h = _pair(2, 5)
    _both(r, h, [-1, -1], _boxes("a", "b"))
    _both(r, h, [], _boxes())
    assert h.mem.ids == [0, 1] and h.mem.gaps == [1, 1]
    _both(r, h, [], _boxes())
    assert h.mem.gaps == [2, 2]
    _both(r, h, [], _boxes())                                       # a gap of 3 > 2 can no longer qualify: dropped
    assert h.mem.ids == []


def test_reset_clears_everything():
    r, h = _pair(3, 5)
    _both(r, h, [-1, -1], _boxes("a", "b"))
    _both(r, h, [], _boxes())
    r.reset()
    h.reset()
    assert h.mem.ids == [] and h.mem.gaps == [] and len(h.mem.boxes) == 0
    assert _both(r, h, [-1], _boxes("b")) == [0]


def _random_call(rng, n_prev, places):
    n = int(rng.integers(0, 7)) if rng.random() < 0.85 else 0
    src = [int(rng.integers(-1, n_prev + 2)) if rng.random() < 0.7 else -1 for _ in range(n)]
    boxes = places[rng.integers(len(places), size=n)].astype(np.float64)
    u = rng.random((n, 1))
    # small moves, moves that put the IoU with the place near 1/2, and far ones
    boxes = boxes + np.where(u < 0.5, rng.normal(0, 2, (n, 4)), np.where(u < 0.8, [[1, 0, 1, 0]] * (boxes[:, 2:3] - boxes[:, 0:1])
                                                                           / 3 * (1 + rng.normal(0, 0.01, (n, 1))), 900))
    boxes = boxes.astype(F32).reshape(n, 4)
    returned = (boxes + rng.normal(0, 1, boxes.shape)).astype(F32)
    return src, boxes, returned


@pytest.mark.parametrize("m,cap", [(1, 5), (2, 1), (3, 3), (7, 64), (30, 16)])
def test_random_scripts_against_the_restatement(m, cap):
    rng = np.random.default_rng(100 * m + cap)
    places = np.array([[x, y, x + w, y + w] for x, y, w in rng.uniform([0, 0, 40], [1800, 1000, 160], (8, 3))], F32)
    revived = 0
    for _ in range(20):
        r, h = _pair(m, cap)
        for t in range(40):
            src, boxes, returned = _random_call(rng, len(r.ids), places)
            before = set(r.ids) | {e[0] for e in r.mem}
            got = _both(r, h, src, boxes, returned)
            revived += sum(1 for i, s in zip(got, src) if i in before and not (0 <= s < len(r.ids)))
            if rng.random() < 0.03:
                r.reset()
                h.reset()
    assert revived > 0


@pytest.mark.parametrize("seed", range(4))
def test_id_memory_0_gives_assign_track_ids_exactly(seed):
    from peppa_pig_face_landmark_b200.core.smoother.lk import IdMemory, assign_track_ids
    rng = np.random.default_rng(seed)
    places = np.array([[x, y, x + 100, y + 100] for x, y in rng.uniform(0, 900, (6, 2))], F32)
    mem = IdMemory(0, 8, IOU)
    ids_a, next_a, ids_b, next_b, prev = [], 0, [], 0, np.zeros((0, 4), F32)
    for t in range(300):
        src, boxes, returned = _random_call(rng, len(ids_a), places)
        ids_a, next_a = mem.assign(np.asarray(src, np.int32), boxes, ids_a, prev, next_a)
        ids_b, next_b = assign_track_ids(np.asarray(src, np.int32), ids_b, next_b)
        assert ids_a == ids_b and next_a == next_b and mem.ids == [] and len(mem.boxes) == 0
        prev = returned


# ----------------------------------------------------------------------------- arguments
BAD = [-1, True, False, np.bool_(True), 1.5, 2.0, "3", None, 2 ** 31, [1]]


@pytest.mark.parametrize("value", BAD)
def test_bad_id_memory_raises(value):
    from peppa_pig_face_landmark_b200.core.api.facer import FaceAna, check_id_memory
    from peppa_pig_face_landmark_b200.core.api.streams import FaceAnaStreams
    with pytest.raises(ValueError):
        check_id_memory(value, True)
    with pytest.raises(ValueError):
        FaceAna(track_ids=True, id_memory=value)
    with pytest.raises(ValueError):
        FaceAnaStreams(n_streams=2, track_ids=True, id_memory=value)


@pytest.mark.parametrize("value", [1, 30, np.int64(5)])
def test_id_memory_needs_track_ids(value):
    from peppa_pig_face_landmark_b200.core.api.facer import FaceAna
    from peppa_pig_face_landmark_b200.core.api.streams import FaceAnaStreams
    with pytest.raises(ValueError, match="track_ids"):
        FaceAna(id_memory=value)
    with pytest.raises(ValueError, match="track_ids"):
        FaceAnaStreams(n_streams=2, id_memory=value)


def test_good_id_memory():
    import inspect
    from peppa_pig_face_landmark_b200.core.api import facer, streams
    from peppa_pig_face_landmark_b200.core.smoother.lk import MAX_ID_MEMORY
    assert MAX_ID_MEMORY == 2 ** 31 - 1
    for v in (0, 1, np.int32(7), np.int64(2 ** 31 - 1)):
        got = facer.check_id_memory(v, True)
        assert got == int(v) and type(got) is int
    assert facer.check_id_memory(0, False) == 0
    for cls in (facer.FaceAna, streams.FaceAnaStreams):
        assert inspect.signature(cls.__init__).parameters["id_memory"].default == 0


def test_exports_declared_bound_and_built():
    from peppa_pig_face_landmark_b200 import build, runtime
    arity = _header_arity()
    assert arity["skps_mpipe_set_id_memory"] == 2
    assert runtime.SIGNATURES["skps_mpipe_set_id_memory"] == (C.c_int, [C.c_void_p, C.c_int])
    # the memory entry: skps_debug_mp_temporal's 22 parameters with id_memory and the four buffers before the stream
    assert arity["skps_debug_mp_temporal"] == 22 and arity["skps_debug_mp_temporal_mem"] == 27
    args = runtime.SIGNATURES["skps_debug_mp_temporal_mem"][1]
    assert args[:21] == runtime.SIGNATURES["skps_debug_mp_temporal"][1][:21]
    assert args[21] is C.c_int and args[22:] == [C.c_void_p] * 5
    build.build()
    lib = runtime.load_library()
    for name in ("skps_mpipe_set_id_memory", "skps_debug_mp_temporal_mem"):
        assert hasattr(lib, name), name
