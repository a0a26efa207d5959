"""Detection cadence without a GPU: the keyframe rule FaceAna applies (DetectCadence) against a numpy restatement on
hand-built sequences (resets, size changes, offsets, more streams than N and fewer, partial batches), argument checks of
FaceAna and FaceAnaStreams, and the two C exports of FaceAnaStreams' cadence, declared in the header and bound in
runtime.py."""
import itertools

import numpy as np
import pytest

from test_c_abi_cpu import _header_arity


def _keyframes_np(sizes, resets, every, offset):
    """Keyframes of one stream's frames: sizes[i] is frame i's size id, resets the frame indices a reset comes before.
    The count restarts at every reset; a frame is forced when it starts a segment or its size differs from the frame
    before it."""
    sizes = np.asarray(sizes)
    n = len(sizes)
    starts = np.zeros(n, bool)
    starts[0] = True
    starts[list(resets)] = True
    seg = np.cumsum(starts) - 1
    idx = np.arange(n) - np.flatnonzero(starts)[seg]
    same = np.r_[False, sizes[1:] == sizes[:-1]] & ~starts
    return ~same | ((idx + offset) % every == 0)


def _cadence_keyframes(sizes, resets, every, offset):
    from peppa_pig_face_landmark_b200.core.api.facer import DetectCadence
    c, prev, out = DetectCadence(every, offset), None, []
    for i, sz in enumerate(sizes):
        if i in resets:
            c.reset()
            prev = None
        out.append(c.step(prev != sz))
        prev = sz
    return np.array(out)


def test_hand_built_sequences():
    # no size change, no reset: forced frame 0, then every N-th by count
    assert list(_keyframes_np([0] * 7, [], 3, 0)) == [1, 0, 0, 1, 0, 0, 1]
    assert list(_keyframes_np([0] * 7, [], 3, 2)) == [1, 1, 0, 0, 1, 0, 0]
    # a size change on a non-keyframe index forces it; the count runs on
    assert list(_keyframes_np([0, 0, 1, 1, 1, 1, 1], [], 4, 0)) == [1, 0, 1, 0, 1, 0, 0]
    # a reset restarts the count and forces the next frame
    assert list(_keyframes_np([0] * 7, [3], 4, 1)) == [1, 0, 0, 1, 0, 0, 1]
    # N = 1: every frame
    assert _keyframes_np([0, 1, 1, 0], [2], 1, 0).all()
    for sizes, resets, every, offset in [([0] * 7, [], 3, 0), ([0] * 7, [], 3, 2), ([0, 0, 1, 1, 1, 1, 1], [], 4, 0),
                                         ([0] * 7, [3], 4, 1), ([0, 1, 1, 0], [2], 1, 0)]:
        assert np.array_equal(_cadence_keyframes(sizes, resets, every, offset),
                              _keyframes_np(sizes, resets, every, offset))


@pytest.mark.parametrize("every", [1, 2, 3, 5, 8])
def test_random_sequences(every):
    rng = np.random.default_rng(every)
    for _ in range(200):
        n = int(rng.integers(1, 40))
        sizes = rng.choice(3, size=n, p=[0.85, 0.1, 0.05])
        resets = set(int(i) for i in np.flatnonzero(rng.random(n) < 0.05))
        for offset in range(every):
            assert np.array_equal(_cadence_keyframes(sizes, resets, every, offset),
                                  _keyframes_np(sizes, resets, every, offset))


def _streams_schedule(calls, every):
    """FaceAnaStreams' keyframes: calls[t] = (streams fed, {stream: size id}); stream s has offset s % every and counts
    only the calls that feed it.  Returns the keyframe flags per call and the detector batch m per call."""
    S = max(n for n, _ in calls)
    per = {s: [] for s in range(S)}
    for t, (n, sizes) in enumerate(calls):
        for s in range(n):
            per[s].append((t, sizes.get(s, 0)))
    key = {}
    for s, fr in per.items():
        k = _keyframes_np([z for _, z in fr], [], every, s % every) if fr else []
        for (t, _), v in zip(fr, k):
            key[t, s] = bool(v)
    flags = [[key[t, s] for s in range(n)] for t, (n, _) in enumerate(calls)]
    return flags, [sum(f) for f in flags]


def test_streams_staggered_schedule():
    every, S = 4, 8
    flags, m = _streams_schedule([(S, {})] * 9, every)
    assert m[0] == S                                    # every stream's first frame is forced
    assert m[1:] == [2] * 8                             # then S / N keyframes per call, staggered
    for t in range(1, 9):
        assert [s for s in range(S) if flags[t][s]] == [s for s in range(S) if (t + s) % every == 0]


def test_streams_more_every_than_streams_has_empty_calls():
    flags, m = _streams_schedule([(3, {})] * 9, 5)
    assert m == [3, 0, 0, 1, 1, 1, 0, 0, 1]
    assert [t for t, v in enumerate(m) if v == 0] == [1, 2, 6, 7]


def test_streams_partial_batches_and_size_changes():
    # stream 2 is left out of calls 2 and 3: its count does not advance there; stream 1 changes size at call 4
    calls = [(3, {}), (3, {}), (2, {}), (2, {}), (3, {1: 1}), (3, {1: 1}), (3, {})]
    flags, m = _streams_schedule(calls, 3)
    # stream 0 offset 0: frames 0..6 -> keys 0, 3, 6; stream 1 offset 1: keys at i = 2, 5 and forced at 4 (size change)
    # and 6 (back to size 0); stream 2 offset 2: fed at calls 0, 1, 4, 5, 6 = its frames 0..4 -> keys 0, 1, 4
    assert [f[0] for f in flags] == [True, False, False, True, False, False, True]
    assert [f[1] for f in flags] == [True, False, True, False, True, True, True]
    assert [f[2] for f in flags if len(f) > 2] == [True, True, False, False, True]
    assert m == [3, 1, 1, 1, 1, 1, 3]


def test_cadence_per_stream_equals_schedule():
    """One DetectCadence per stream, driven call by call, gives the schedule's flags (what FaceAnaStreams computes in C
    and what the per-stream FaceAna objects it is tested against compute)."""
    from peppa_pig_face_landmark_b200.core.api.facer import DetectCadence
    rng = np.random.default_rng(7)
    for every, S in itertools.product([2, 3, 5, 7], [1, 3, 4, 16]):
        calls = [(int(rng.integers(1, S + 1)), {int(s): int(rng.integers(0, 2)) for s in range(S) if rng.random() < 0.1})
                 for _ in range(30)]
        flags, m = _streams_schedule(calls, every)
        cad, prev = [DetectCadence(every, s % every) for s in range(S)], [None] * S
        for t, (n, sizes) in enumerate(calls):
            got = []
            for s in range(n):
                z = sizes.get(s, 0)
                got.append(cad[s].step(prev[s] != z))
                prev[s] = z
            assert got == flags[t] and sum(got) == m[t], (every, S, t)


@pytest.mark.parametrize("every,offset", [(0, 0), (-1, 0), (2.0, 0), (True, 0), ("2", 0), (None, 0), (3, 3), (3, -1),
                                          (1, 1), (2, 0.5), (2, None)])
def test_bad_arguments_raise(every, offset):
    from peppa_pig_face_landmark_b200.core.api.facer import FaceAna, check_detect_every
    from peppa_pig_face_landmark_b200.core.api.streams import FaceAnaStreams
    with pytest.raises(ValueError):
        check_detect_every(every, offset)
    with pytest.raises(ValueError):
        FaceAna(detect_every=every, detect_offset=offset)
    if offset == 0:
        with pytest.raises(ValueError):
            FaceAnaStreams(n_streams=2, detect_every=every)


def test_good_arguments():
    from peppa_pig_face_landmark_b200.core.api.facer import check_detect_every
    assert check_detect_every(1) == (1, 0)
    assert check_detect_every(np.int64(4), np.int32(3)) == (4, 3)
    assert all(type(v) is int for v in check_detect_every(np.int64(4), np.int32(3)))


def test_exports_declared_and_bound():
    import ctypes as C
    from peppa_pig_face_landmark_b200 import runtime
    arity = _header_arity()
    assert arity["skps_mpipe_set_detect_every"] == 2 and arity["skps_mpipe_detector_frames"] == 3
    assert runtime.SIGNATURES["skps_mpipe_set_detect_every"] == (C.c_int, [C.c_void_p, C.c_int])
    assert runtime.SIGNATURES["skps_mpipe_detector_frames"] == (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int32)])
