"""Track ids without a GPU: the host rule FaceAna applies (core/smoother/lk.py assign_track_ids) on hand-built calls, and
the C exports and struct field FaceAna and FaceAnaStreams read the ids through."""
import os

import numpy as np
import pytest

from peppa_pig_face_landmark_b200.core.smoother.lk import assign_track_ids

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


class _Track:
    """The state FaceAna keeps between calls: the ids of the last call's faces and the next unused id."""

    def __init__(self):
        self.ids, self.next_id = [], 0

    def call(self, sources):
        self.ids, self.next_id = assign_track_ids(sources, self.ids, self.next_id)
        return self.ids


def test_first_call_numbers_faces_in_output_order():
    t = _Track()
    assert t.call([-1, -1, -1]) == [0, 1, 2]
    assert t.next_id == 3


def test_ids_follow_the_face_through_a_reordering():
    t = _Track()
    t.call([-1, -1, -1])                        # ids 0, 1, 2
    assert t.call([2, 0, 1]) == [2, 0, 1]      # output order changed (sort_and_filter by area): ids follow the faces
    assert t.call([1, 2, 0]) == [0, 1, 2]


def test_only_the_first_face_with_a_source_inherits():
    t = _Track()
    t.call([-1, -1])                            # ids 0, 1
    assert t.call([1, 1, 0]) == [1, 2, 0]       # the second face matched track box 1 too: a fresh number
    assert t.next_id == 3
    assert t.call([0, 0, 0]) == [1, 3, 4]


def test_fresh_numbers_are_given_in_output_order_and_never_reused():
    t = _Track()
    t.call([-1, -1, -1, -1])                    # ids 0..3
    assert t.call([-1, 3, -1, 0]) == [4, 3, 5, 0]
    assert t.call([-1]) == [6]                  # ids 1 and 2 were lost; their numbers stay used
    assert t.call([0, -1]) == [6, 7]


def test_an_empty_frame_ends_every_track():
    t = _Track()
    t.call([-1, -1])
    assert t.call([]) == []
    assert t.next_id == 2
    assert t.call([-1, -1, -1]) == [2, 3, 4]    # nothing to continue: all new


def test_numbering_after_reset():
    t = _Track()
    t.call([-1, -1, -1])
    t.call([0, 1, 2])
    t = _Track()                                # FaceAna.reset(): no track, numbering from 0
    assert t.call([-1, -1]) == [0, 1]


def test_a_source_past_the_previous_faces_gets_a_fresh_number():
    t = _Track()
    t.call([-1, -1])                            # ids 0, 1
    assert t.call([2, 1, 5, 0]) == [2, 1, 3, 0]
    assert t.next_id == 4


def test_ids_are_python_ints():
    ids, nxt = assign_track_ids(np.array([-1, 0], np.int32), [7], 8)
    assert ids == [8, 7] and nxt == 9
    assert all(type(i) is int for i in ids)


def test_new_exports_are_in_the_built_library():
    from peppa_pig_face_landmark_b200 import build, runtime
    build.build()
    lib = runtime.load_library()
    for name in ("skps_pipeline_face_sources", "skps_mpipe_track_ids"):
        assert name in runtime.SIGNATURES
        assert hasattr(lib, name), name
    with open(os.path.join(ROOT, "include", "skps_b200.h")) as f:
        hdr = f.read()
    assert "int64_t* ids;" in hdr
    # the ids field is appended: every earlier field keeps its offset
    fields = [f for f, _ in runtime.MpipeOutputs._fields_]
    assert fields[-1] == "ids" and fields[:-1] == ["n_faces", "ran_detector", "boxes", "kps", "scores", "chips", "M", "rvec",
                                                   "tvec", "euler", "reproject"]


@pytest.mark.parametrize("make", ["FaceAna", "FaceAnaStreams"])
def test_track_ids_option_defaults_off(make):
    import inspect
    from peppa_pig_face_landmark_b200.core.api import facer, streams
    cls = {"FaceAna": facer.FaceAna, "FaceAnaStreams": streams.FaceAnaStreams}[make]
    assert inspect.signature(cls.__init__).parameters["track_ids"].default is False
