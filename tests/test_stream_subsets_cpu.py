"""FaceAnaStreams calls that feed a subset of the streams, without a GPU: the check of submit(streams=...) and the arity of
the C entry points that take a call -> stream map next to the ones that do not."""
import numpy as np
import pytest

from test_c_abi_cpu import _header_arity


def test_streams_none_is_the_identity():
    from peppa_pig_face_landmark_b200.core.api.streams import check_streams
    assert check_streams(None, 3, 8) is None


@pytest.mark.parametrize("streams, n, n_streams, want", [
    ([5, 2, 9], 3, 16, [5, 2, 9]),
    ((0,), 1, 1, [0]),
    (range(4), 4, 4, [0, 1, 2, 3]),
    ([3, 2, 1, 0], 4, 4, [3, 2, 1, 0]),
    (np.array([7, 0], np.int64), 2, 8, [7, 0]),
    ([np.int32(1), np.uint8(6)], 2, 7, [1, 6]),
])
def test_accepted_maps(streams, n, n_streams, want):
    from peppa_pig_face_landmark_b200.core.api.streams import check_streams
    got = check_streams(streams, n, n_streams)
    assert got == want
    assert all(type(t) is int for t in got)


@pytest.mark.parametrize("streams, n, n_streams", [
    ([0, 1], 3, 4),                 # fewer ids than frames
    ([0, 1, 2], 2, 4),              # more ids than frames
    ([1, 1], 2, 4),                 # two frames of one stream in one call
    ([2, 0, 2], 3, 4),
    ([4], 1, 4),                    # id == n_streams
    ([-1], 1, 4),
    ([0.0, 1], 2, 4),               # not ints
    (["0"], 1, 4),
    ([None], 1, 4),
    ([True, 0], 2, 4),              # bool is not a stream id
    ([np.bool_(False)], 1, 4),
    ("01", 2, 4),                   # a string is not a sequence of ids
    (3, 1, 4),                      # nor is an int
])
def test_refused_maps(streams, n, n_streams):
    from peppa_pig_face_landmark_b200.core.api.streams import check_streams
    with pytest.raises(ValueError):
        check_streams(streams, n, n_streams)


def test_stream_map_entry_points_arity():
    from peppa_pig_face_landmark_b200 import runtime
    arity = _header_arity()
    want = {"skps_mpipe_submit_streams": 6, "skps_mpipe_submit_device_streams": 9, "skps_mpipe_submit": 5,
            "skps_mpipe_submit_device": 8}
    for name, n in want.items():
        assert arity[name] == n == len(runtime.SIGNATURES[name][1]), name
