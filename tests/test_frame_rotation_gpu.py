"""CUDA frames stored turned (rotate=90, 180, 270): every result of every class equals, bit for bit, the result of the same
call on the upright frame materialised as a contiguous tensor, cv2.rotate(stored, code) on a host copy.  Frames are
passed in every layout, packed and as pitched ROI views at odd byte offsets.  The ingest kernel is also checked on its
own against cv2.rotate at the sizes that reach its partial tiles."""
import ctypes as C

import cv2
import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames
from test_device_frames_gpu import _eq, _same
from test_frame_layouts_gpu import CODES, as_layout
from test_streams_gpu import _sequences

pytestmark = pytest.mark.gpu

LAYOUTS = list(CODES)
CV = {90: cv2.ROTATE_90_CLOCKWISE, 180: cv2.ROTATE_180, 270: cv2.ROTATE_90_COUNTERCLOCKWISE}


def stored(upright, rotate):
    """The frame a camera stores when it must be turned `rotate` degrees clockwise to give `upright`."""
    s = np.ascontiguousarray(np.rot90(upright, rotate // 90))
    if rotate:
        assert np.array_equal(cv2.rotate(s, CV[rotate]), upright)
    return s


def turned(upright, rotate, layout="bgr", kind="packed", seed=0):
    return as_layout(stored(upright, rotate), layout, kind, seed=seed)


def _bgr(f):
    return as_layout(f, "bgr")


def test_direction_is_cv2_rotate():
    """rotate=R analyses cv2.rotate(frame, code): torch.rot90(frame, -R // 90, dims=(0, 1)) for (H, W, C) tensors and
    dims=(1, 2) for planar ones."""
    import torch
    f = np.random.default_rng(0).integers(0, 256, size=(5, 7, 3), dtype=np.uint8)
    for r, code in CV.items():
        want = cv2.rotate(f, code)
        assert np.array_equal(torch.rot90(torch.from_numpy(f), -r // 90, dims=(0, 1)).numpy(), want)
        planar = torch.from_numpy(np.ascontiguousarray(f.transpose(2, 0, 1)))
        assert np.array_equal(torch.rot90(planar, -r // 90, dims=(1, 2)).permute(1, 2, 0).numpy(), want)


# ---------------------------------------------------------------------------------------------------- ingest kernel
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("rotate", [90, 180, 270])
@pytest.mark.parametrize("hw", [(1, 1), (1, 37), (37, 1), (37, 1001), (1080, 1920), (2160, 3840)])
@pytest.mark.parametrize("kind", ["packed", "roi"])
def test_ingest_turned_equals_cv2_rotate(layout, rotate, hw, kind):
    """skps_frame_ingest_rotate: the packed frame equals cv2.rotate of the stored BGR frame byte for byte, nothing past it
    is written, and the sum is the integer sum of |upright - prev|."""
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    H, W = hw
    rng = np.random.default_rng(H * 131 + W + rotate)
    f = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)              # as stored
    up = cv2.rotate(f, CV[rotate])
    p = rng.integers(0, 256, size=up.shape, dtype=np.uint8)
    src = as_layout(f, layout, kind, seed=W)
    planar = layout.endswith("_planar")
    pitch = src.stride(1 if planar else 0) if H > 1 else W * (1 if planar else src.shape[2])
    plane = src.stride(0) if planar else 0
    n = H * W * 3
    packed = torch.full((n + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    prev = _bgr(p).reshape(-1)
    got = torch.zeros(1, dtype=torch.int64, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rt.check(lib.skps_frame_ingest_rotate(src.data_ptr(), H, W, pitch, CODES[layout], plane, rotate // 90,
                                          packed.data_ptr(), prev.data_ptr(), got.data_ptr(), s))
    assert np.array_equal(packed[:n].cpu().numpy(), up.reshape(-1))
    assert bool((packed[n:] == 0xAB).all())
    assert int(got.item()) == int(np.abs(up.astype(np.int64) - p.astype(np.int64)).sum())


def test_ingest_refuses_bad_turns():
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    f = torch.zeros((4, 5, 3), dtype=torch.uint8, device="cuda")
    packed = torch.zeros((64,), dtype=torch.uint8, device="cuda")
    sums = torch.zeros(1, dtype=torch.int64, device="cuda")
    for t in (-1, 4, 90):
        assert lib.skps_frame_ingest_rotate(f.data_ptr(), 4, 5, 15, 0, 0, t, packed.data_ptr(), None, sums.data_ptr(), None)
    assert lib.skps_frame_ingest_rotate(f.data_ptr(), 4, 5, 15, 0, 0, 3, packed.data_ptr(), None, sums.data_ptr(), None) == 0


# ---------------------------------------------------------------------------------------------------- batch classes
def _golden():
    return [frames.load_test1(), video_frames()[0], frames.frame_4k()]


def test_detector_align_mixed_rotations_and_layouts():
    """FaceDetector(align=112).run_batch with a rotation per frame, in every layout: rows, kept indices, points, M and
    chips equal the call on the upright frames; out= gives the same with no host synchronisation."""
    import torch
    from Skps import FaceDetector
    fs = _golden() + [frames.multi_face_frame(1920, 1080, (2, 2), 440)]
    fd = FaceDetector(max_frames=2, align=112)
    want = fd.run_batch([_bgr(f) for f in fs])
    want_idx = fd.last_keep_idx
    wbuf = fd.new_results(len(fs))
    fd.submit([_bgr(f) for f in fs], out=wbuf)
    fd.collect()
    for j, layout in enumerate(LAYOUTS):
        rot = [[90, 0, 270, 180], [180, 270, 90, 0], [270, 90, 180, 90]][j % 3]
        kind = ("packed", "roi")[j % 2]
        got = fd.run_batch([turned(f, r, layout, kind) for f, r in zip(fs, rot)], layout=layout, rotate=rot)
        for i in range(len(fs)):
            for a, b in zip(got[i], want[i]):
                _eq(a, b, "%s %s frame %d" % (layout, rot, i))
            _eq(fd.last_keep_idx[i], want_idx[i], "%s idx %d" % (layout, i))
        buf = fd.new_results(len(fs))
        fd.submit([turned(f, r, layout, "roi") for f, r in zip(fs, rot)], out=buf, layout=layout, rotate=rot)
        fd.collect()
        torch.cuda.synchronize()
        for i, k in enumerate(wbuf["count"].tolist()):
            assert int(buf["count"][i]) == k
            c = min(k, fd.max_chips)
            for name in ("rows", "idx"):
                assert torch.equal(buf[name][i, :k], wbuf[name][i, :k]), (layout, name, i)
            for name in ("points", "M", "chip"):
                assert torch.equal(buf[name][i, :c], wbuf[name][i, :c]), (layout, name, i)


def test_landmark_align_turned_frames():
    """FaceLandmark(align=112) with boxes in upright coordinates, host and CUDA boxes, out= too."""
    import torch
    from Skps import FaceDetector, FaceLandmark
    fs = _golden()
    rot = [270, 90, 180]
    boxes = [np.ascontiguousarray(b[:, :4]) for b in FaceDetector().run_batch(fs)]
    fl = FaceLandmark(max_faces=8, align=112)
    want = fl.run_batch([_bgr(f) for f in fs], boxes)
    n = sum(len(b) for b in boxes)
    wbuf = fl.new_results(n)
    fl.submit([_bgr(f) for f in fs], [torch.from_numpy(b).cuda() for b in boxes], out=wbuf)
    fl.collect()
    for layout in ("bgr", "rgb_planar", "bgra"):
        got = fl.run_batch([turned(f, r, layout, "roi") for f, r in zip(fs, rot)], boxes, layout=layout, rotate=rot)
        for i, (g, w) in enumerate(zip(got, want)):
            for a, b in zip(g, w):
                _eq(a, b, "%s frame %d" % (layout, i))
        buf = fl.new_results(n)
        fl.submit([turned(f, r, layout) for f, r in zip(fs, rot)], [torch.from_numpy(b).cuda() for b in boxes], out=buf,
                  layout=layout, rotate=rot)
        fl.collect()
        torch.cuda.synchronize()
        for k in wbuf:
            assert torch.equal(buf[k][:n], wbuf[k][:n]), (layout, k)


def test_images_pose_align_turned_images():
    from Skps import FaceAnaImages
    fs = _golden() + [frames.canvas_640()]
    fi = FaceAnaImages(align=112, pose=True, max_frames=2)
    want = fi.run_batch([_bgr(f) for f in fs])
    assert all(len(w) for w in want)
    for layout, rot in (("bgr", [90, 180, 270, 0]), ("rgb_planar", 270), ("rgba", [180, 90, 0, 270])):
        got = fi.run_batch([turned(f, r, layout, "roi") for f, r in
                            zip(fs, rot if isinstance(rot, list) else [rot] * len(fs))], layout=layout, rotate=rot)
        for i in range(len(fs)):
            _same(got[i], want[i], "%s %s image %d" % (layout, rot, i))


# ---------------------------------------------------------------------------------------------------- FaceAna
def _jittered_1080p(n):
    return [frames.frame_1080p(jitter=((3 * t) % 7, (5 * t) % 9)) if t % 4 != 3 else frames.frame_1080p()
            for t in range(n)]


@pytest.mark.parametrize("rotate", [90, 180, 270])
def test_faceana_turned_sequence(rotate):
    """A jittered 1080p sequence stored turned: every result, gate decision and detector row equals a second FaceAna fed
    the upright frames.  The One-Euro filter normalises by the frame size, so a wrong (H, W) in the host layer fails."""
    from Skps import FaceAna
    kw = dict(align=112, pose=True, track_ids=True, id_memory=2, detect_every=3)
    got_fa, want_fa = FaceAna(**kw), FaceAna(**kw)
    for t, f in enumerate(_jittered_1080p(8)):
        layout, kind = LAYOUTS[t % len(LAYOUTS)], ("roi", "packed")[t % 2]
        got = got_fa.run(turned(f, rotate, layout, kind, seed=t), layout=layout, rotate=rotate)
        want = want_fa.run(_bgr(f))
        _same(got, want, "t %d" % t)
        assert got_fa.last_ran_detector == want_fa.last_ran_detector, t
        if want_fa.last_ran_detector:
            _eq(got_fa.last_det_rows, want_fa.last_det_rows, "t %d rows" % t)


def test_faceana_rotation_changes_mid_sequence():
    from Skps import FaceAna
    kw = dict(align=112, pose=True, track_ids=True, detect_every=2)
    got_fa, want_fa = FaceAna(**kw), FaceAna(**kw)
    clip = _sequences()[0]
    for t, (f, r) in enumerate(zip(clip + clip, [0, 0, 90, 90, 180, 180, 0, 180, 270, 90, 90, 0])):
        got = got_fa.run(turned(f, r, "rgb", "roi", seed=t), layout="rgb", rotate=r)
        want = want_fa.run(_bgr(f))
        _same(got, want, "t %d rotate %d" % (t, r))
        assert got_fa.last_ran_detector == want_fa.last_ran_detector, t


def test_faceana_refuses_before_enqueueing():
    from Skps import FaceAna
    fa = FaceAna()
    f = frames.canvas_640()
    for frame, rot in [(_bgr(f), 45), (_bgr(f), True), (_bgr(f), "90"), (_bgr(f), [90]), (f, 90)]:
        with pytest.raises(ValueError, match="rotate"):
            fa.run(frame, rotate=rot)
    assert fa.previous_image is None
    _same(fa.run(turned(f, 90), rotate=90), FaceAna().run(_bgr(f)), "after refusals")


# ---------------------------------------------------------------------------------------------------- FaceAnaStreams
def _streams_plan_results(fa, plan, seqs, frame_of):
    """Runs `plan` on fa, calls 2k and 2k + 1 in flight together: per call, host results or cloned out= tensors."""
    import torch
    pos = [0, 0, 0, 0]
    bufs = [fa.new_results(), fa.new_results()]
    res = []
    for c0 in range(0, len(plan), 2):
        pending = []
        for j, (streams, rot, layout, dev_out) in enumerate(plan[c0:c0 + 2]):
            fs = [seqs[s][pos[s] % 6] for s in streams]
            for s in streams:
                pos[s] += 1
            frs, kw = frame_of(fs, rot, layout, j, c0)
            fa.submit(frs, out=bufs[j] if dev_out else None, streams=streams, **kw)
            pending.append((len(streams), dev_out))
        for n, dev_out in pending:
            got = fa.collect()
            if dev_out:
                torch.cuda.synchronize()
                got = {k: v[:n].clone() for k, v in got.items()}
            res.append((got, list(fa.last_ran_detector) if not dev_out else None))
    return res


def test_streams_rotations_subsets_switches_out_and_two_in_flight():
    """Streams with different rotations in one call, subsets of the streams, one stream switching 0 -> 90 -> 180, host
    results and out=, two calls in flight: every entry equals an upright twin fed the same pixels on the same schedule.
    The twin runs first, on its own, so that the two objects' work never overlaps on the GPU."""
    import torch
    from Skps import FaceAnaStreams
    seqs = _sequences()
    kw = dict(n_streams=4, align=112, pose=True, track_ids=True, detect_every=2)
    # (streams, rotate per frame, layout, out=); stream 3 switches 0 -> 90 -> 180
    plan = [([0, 1, 2, 3], [90, 270, 180, 0], "bgr", False), ([2, 0], [180, 90], "rgb_planar", True),
            ([3, 1, 0], [90, 270, 90], "bgra", True), ([1, 2, 3, 0], [270, 180, 90, 90], "bgr", False),
            ([0, 3], [90, 180], "rgb", False), ([2, 1, 3], [180, 270, 180], "bgr", True),
            ([3, 2, 1, 0], [180, 0, 270, 90], "rgb_planar", True), ([1, 0, 2], [270, 90, 180], "bgr", False)]
    want = _streams_plan_results(FaceAnaStreams(**kw), plan, seqs, lambda fs, rot, layout, j, c0: ([_bgr(f) for f in fs], {}))
    got = _streams_plan_results(
        FaceAnaStreams(**kw), plan, seqs,
        lambda fs, rot, layout, j, c0: ([turned(f, r, layout, ("roi", "packed")[j], seed=c0 + j) for f, r in zip(fs, rot)],
                                        dict(layout=layout, rotate=rot)))
    for c, ((g, g_ran), (w, w_ran)) in enumerate(zip(got, want)):
        if isinstance(w, dict):
            for k in w:
                assert torch.equal(g[k], w[k]), (c, k)
        else:
            for i in range(len(w)):
                _same(g[i], w[i], "call %d entry %d" % (c, i))
            assert g_ran == w_ran, c


def test_streams_one_rotation_for_the_call():
    from Skps import FaceAnaStreams
    f = frames.multi_face_frame(1920, 1080, (2, 2), 440)
    got =FaceAnaStreams(n_streams=2).run([turned(f, 270), turned(f, 270)], rotate=270)
    want = FaceAnaStreams(n_streams=2).run([_bgr(f), _bgr(f)])
    for g, w in zip(got, want):
        _same(g, w)


def test_batch_classes_and_streams_refuse_before_enqueueing():
    from Skps import FaceAnaImages, FaceAnaStreams, FaceDetector, FaceLandmark
    f = frames.canvas_640()
    cuda, host = [_bgr(f), _bgr(f)], [f, f]
    box = [np.array([[100, 100, 300, 300]], np.float32)] * 2
    bad = [(cuda, 45), (cuda, True), (cuda, [90]), (cuda, [90, 90, 90]), (cuda, [0, 91]), (cuda, 90.0), (host, 90),
           (host, [0, 180])]
    fd, fl, fi, fs = FaceDetector(), FaceLandmark(), FaceAnaImages(), FaceAnaStreams(n_streams=2)
    for frs, rot in bad:
        for call in (lambda: fd.submit(frs, rotate=rot), lambda: fl.submit(frs, box, rotate=rot),
                     lambda: fi.submit(frs, rotate=rot), lambda: fs.submit(frs, rotate=rot)):
            with pytest.raises(ValueError, match="rotate"):
                call()
        assert not fd._pending and not fl._pending and not fi._pending and not fs._pending
    got = fs.run([turned(f, 90), turned(f, 180)], rotate=[90, 180])
    want = FaceAnaStreams(n_streams=2).run(cuda)
    for g, w in zip(got, want):
        _same(g, w, "after refusals")


# ---------------------------------------------------------------------------------------------------- the portrait scene
@pytest.mark.parametrize("rotate", [90, 180, 270])
def test_portrait_scene_stored_turned(rotate):
    """Four upright faces in a portrait frame: stored turned, the detector keeps 0 to 2 of them when the frame is read
    as stored; with rotate= it returns the upright frame's 4, bit for bit."""
    from Skps import FaceAna
    f = frames.multi_face_frame(1920, 1080, (2, 2), 440)
    want = FaceAna().run(_bgr(f))
    assert len(want) == 4
    got = FaceAna().run(turned(f, rotate, "rgb_planar", "roi"), layout="rgb_planar", rotate=rotate)
    _same(got, want, "rotate %d" % rotate)
