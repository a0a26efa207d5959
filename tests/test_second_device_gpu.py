"""The library on a second GPU.  A = cuda:0, B = the last visible device.  Before anything runs on B, one engine of each
kind is created and run on A (the detector at 384x640 and 416x736, and the student), so every per-process first use
(kernel attributes, zero biases, occupancy) happens on A.  Then on B: every engine op is within its float64 bound and
the outputs equal A's bit for bit; every pipeline equals the same pipeline on A bit for bit, with host frames and with
CUDA frames on B, and still meets the reference contracts; the image kernels match their CPU references; no public
call moves the caller's current device; objects on A and B take turns with calls in flight; and a pipeline refuses
engines on two devices.  Calls on B are made with A current unless a test says otherwise."""
import contextlib
import ctypes as C
import os
import sys

import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames
from test_align_gpu import check_faces, cv2_warp
from test_detector_batch_gpu import mixed_frames, portrait
from test_images_gpu import _same as _same_images
from test_streams_gpu import _sequences

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

ENGINES = [("detector", (384, 640)), ("detector", (416, 736)), ("student", None)]


def _tag(which, hw):
    return which if hw is None else "%s@%dx%d" % (which, hw[0], hw[1])


@pytest.fixture(scope="module")
def devs():
    """(A, B), or a skip of the whole module when fewer than two devices are visible."""
    import torch
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs two visible CUDA devices, found %d" % n)
    A, B = torch.device("cuda:0"), torch.device("cuda:%d" % (n - 1))
    print("devices: %d; A = %s (%s), B = %s (%s)" % (n, A, torch.cuda.get_device_name(A), B,
                                                    torch.cuda.get_device_name(B)))
    torch.cuda.set_device(A)
    return A, B


@pytest.fixture(scope="module")
def on_a(devs):
    """Each engine kind created and run on A first: tag -> (input batch, A's outputs)."""
    import op_report as R
    A, _ = devs
    out = {}
    for which, hw in ENGINES:
        eng, x = R.make_engine(which, hw, 3, device=A)
        out[_tag(which, hw)] = (x, eng.run_u8(x))
        del eng
    return out


@contextlib.contextmanager
def _current(dev):
    """Runs the body with `dev` current and checks that the body leaves it current."""
    import torch
    with torch.cuda.device(dev):
        yield
        assert torch.cuda.current_device() == dev.index, "the current device moved to %d" % torch.cuda.current_device()


def _cuda(f, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(f)).to(dev)


def _same_rows(got, keep, want, want_keep, what):
    assert len(got) == len(want), what
    for i, (r, k, wr, wk) in enumerate(zip(got, keep, want, want_keep)):
        assert r.dtype == np.float32 and np.array_equal(r, wr), (what, i)
        assert np.array_equal(k, wk), (what, i)


def _same_faces(a, b, what):
    """Two FaceAna / FaceAnaStreams result lists equal bit for bit, every key (chip, M and pose included)."""
    assert len(a) == len(b), (what, len(a), len(b))
    for j, (x, y) in enumerate(zip(a, b)):
        assert set(x) == set(y), (what, j)
        for k in x:
            if k == "pose":
                for p in x[k]:
                    assert np.array_equal(x[k][p], y[k][p]), (what, j, k, p)
            else:
                assert np.asarray(x[k]).dtype == np.asarray(y[k]).dtype, (what, j, k)
                assert np.array_equal(x[k], y[k]), (what, j, k)


def _golden_boxes(fd):
    """(frames, boxes): test1, canvas640 and uhd4k with FaceAna's selection of the detector's boxes, and a frame with
    no box."""
    from oracle import host_ref as H
    fs = [frames.load_test1(), frames.canvas_640(), frames.frame_4k(), frames.load_test1()]
    rows = fd.run_batch(fs[:3])
    bs = [np.asarray(H.sort_and_filter(r, 1600, k), np.float32)[:, :4] for r, k in zip(rows, (5, 5, 16))]
    assert all(len(b) for b in bs) and len(bs[2]) == 16
    return fs, bs + [np.zeros((0, 4), np.float32)]


# ------------------------------------------------------------------------------------------------ 1. engine ops
@pytest.mark.parametrize("which,hw", ENGINES, ids=[_tag(w, h) for w, h in ENGINES])
def test_every_engine_op_on_b_within_its_bound_and_equal_to_a(devs, on_a, which, hw):
    import op_report as R
    A, B = devs
    x, want = on_a[_tag(which, hw)]
    with _current(A):
        eng, x_b = R.make_engine(which, hw, 3, device=B)
        assert np.array_equal(x_b, x)
        res, _ = R.check_engine(eng, x)
        got = eng.run_u8(x)
    bad = ["%s kernel %s %s worst (n,y,x,c)=%s ratio %.3e" % (r.name, R.KERNELS[r.kernel], r.info, r.where, r.ratio)
           for r in res if not r.ok]
    assert not bad, "\n".join(bad)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and np.array_equal(g, w)


# ------------------------------------------------------------------------------------------------ 2. pipelines
def test_face_detector_on_b_equals_a(devs, golden):
    from Skps import FaceDetector
    A, B = devs
    mixed = mixed_frames()
    with _current(A):
        fa = FaceDetector(device=A)
        want, want_keep = fa.run_batch(mixed), fa.last_keep_idx
        fb = FaceDetector(device=B)
        _same_rows(fb.run_batch(mixed), fb.last_keep_idx, want, want_keep, "host frames")
        _same_rows(fb.run_batch([_cuda(f, B) for f in mixed]), fb.last_keep_idx, want, want_keep, "cuda frames")
        assert any(len(r) == 0 for r in want) and sum(len(r) > 0 for r in want) >= 8
    for name, i in (("test1", 0), ("uhd4k_top16", 8)):              # test_parity_gpu's contract: the oracle's rows
        assert np.array_equal(fb.last_keep_idx[i], golden(name)["f0_det_keep_idx"]), name


def test_face_landmark_on_b_equals_a(devs):
    import torch
    from Skps import FaceDetector, FaceLandmark
    A, B = devs
    with _current(A):
        fs, bs = _golden_boxes(FaceDetector(device=A))
        want = FaceLandmark(device=A).run_batch(fs, bs)
        fl = FaceLandmark(device=B)
        host = fl.run_batch(fs, bs)
        cf = [_cuda(f, B) for f in fs]
        cuda = fl.run_batch(cf, bs)
        out = fl.new_results(sum(len(b) for b in bs))
        fl.submit(cf, [_cuda(b, B) for b in bs], out=out)
        dev = fl.collect()
        torch.cuda.synchronize(B)
    for what, got in (("host", host), ("cuda", cuda), ("out=", dev)):
        assert len(got) == len(want), what
        for i, ((k, s), (wk, ws)) in enumerate(zip(got, want)):
            if torch.is_tensor(k):
                assert k.device == B, what
                k, s = k.cpu().numpy(), s.cpu().numpy()
            assert np.array_equal(k, wk) and np.array_equal(s, ws), (what, i)


def test_face_ana_images_on_b_equals_a(devs):
    from Skps import FaceAnaImages
    A, B = devs
    v = video_frames()
    images = [frames.load_test1(), frames.frame_4k(), frames.canvas_640(), v[0], v[4], portrait()]
    with _current(A):
        want = FaceAnaImages(pose=True, device=A).run_batch(images)
        fi = FaceAnaImages(pose=True, device=B)
        _same_images(fi.run_batch(images), want, "host images")
        _same_images(fi.run_batch([_cuda(f, B) for f in images]), want, "cuda images")
    assert sum(len(r) > 0 for r in want) >= 4 and any(len(r) == 0 for r in want)


def _streams_run(fs, seqs, cuda_dev=None):
    """Every step of the sequences through fs with two batches in flight; host frames, or CUDA frames on cuda_dev."""
    fs.reset()
    steps = [[s[t] if cuda_dev is None else _cuda(s[t], cuda_dev) for s in seqs] for t in range(len(seqs[0]))]
    got = []
    fs.submit(steps[0])
    for st in steps[1:]:
        fs.submit(st)
        got.append(fs.collect())
    got.append(fs.collect())
    return got


def test_face_ana_streams_on_b_equals_a(devs):
    from Skps import FaceAnaStreams
    A, B = devs
    seqs = _sequences()
    with _current(A):
        fa = FaceAnaStreams(n_streams=len(seqs), align=112, pose=True, device=A)
        want = [fa.run([s[t] for s in seqs]) for t in range(6)]
        fb = FaceAnaStreams(n_streams=len(seqs), align=112, pose=True, device=B)
        for kind, dev in (("host", None), ("cuda", B)):
            got = _streams_run(fb, seqs, dev)
            for t in range(6):
                for k in range(len(seqs)):
                    _same_faces(got[t][k], want[t][k], (kind, t, k))
                    check_faces(seqs[k][t], got[t][k], 112)          # 'chip' == cv2.warpAffine(frame, 'M')
    assert sum(len(r) for w in want for r in w) >= 10


def test_face_ana_built_under_device_b_equals_a(devs, golden):
    import torch
    from Skps import FaceAna
    from test_parity_gpu import _check_result
    A, B = devs
    seq = video_frames()
    with _current(A):
        fa = FaceAna(align=112, pose=True)
        want = [fa.run(f) for f in seq]
    with _current(B):
        fb = FaceAna(align=112, pose=True)
    assert fb._device == B and fb.face_detector.device == B and fb.face_landmark.device == B
    g = golden("video1080")
    with _current(A):
        for kind in ("host", "cuda"):
            fb.reset()
            for t, f in enumerate(seq):
                res = fb.run(f if kind == "host" else _cuda(f, B))
                _same_faces(res, want[t], (kind, t))
                check_faces(f, res, 112)
                _check_result(res, g, t, "video1080 on %s" % B)
        torch.cuda.synchronize(B)


# ------------------------------------------------------------------------------------------------ 3. image kernels
def test_image_kernels_on_b_match_their_cpu_references(devs, golden):
    """skps_letterbox_frames and skps_crop_faces on B (B frames, B streams, A current) against host_ref's letterbox and
    crop_face; the align functions on B against cv2.warpAffine."""
    import torch
    from Skps import FaceDetector, FaceLandmark
    from oracle import host_ref as H
    from peppa_pig_face_landmark_b200.core.api.align import align_faces, warp_affine
    from test_align_oracle import random_affine
    A, B = devs
    rng = np.random.default_rng(23)
    imgs = [frames.load_test1(), frames.frame_4k(), rng.integers(0, 256, (723, 1281, 3), dtype=np.uint8),
            rng.integers(0, 256, (2000, 900, 3), dtype=np.uint8)]
    with _current(A):
        fd = FaceDetector(max_frames=len(imgs), device=B)
        for kind in ("host", "cuda"):
            fd.run_batch(imgs if kind == "host" else [_cuda(f, B) for f in imgs])
            u8 = fd.model.read_buffer(fd.model.plan.input.buf.idx, len(imgs))
            for i, img in enumerate(imgs):
                ref, _ = H.letterbox(img)
                assert np.array_equal(u8[i].transpose(2, 0, 1)[None].astype(np.float32) / np.float32(255.0), ref), \
                    (kind, i)
        img = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
        boxes = np.array([[-30.5, -20.25, 120.0, 150.75], [500.2, 300.4, 700.9, 520.1], [100, 100, 130.5, 300.25],
                          [10.1, 200.2, 600.3, 260.4], [300.7, 10.2, 333.3, 45.9], [0, 0, 639, 479],
                          [200.5, 150.5, 420.25, 400.75]], np.float32)
        fl = FaceLandmark(max_faces=len(boxes), device=B)
        for kind in ("host", "cuda"):
            slot = fl._next
            fl.run_batch([img if kind == "host" else _cuda(img, B)], [boxes])
            crops = fl.model.read_buffer(fl.model.plan.input.buf.idx, len(boxes))
            detail = fl._slots[slot]["detail"][:len(boxes)].cpu().numpy()
            for i, b in enumerate(boxes):
                ref, d = H.crop_face(img, b.copy())
                assert list(detail[i]) == [int(v) for v in d], (kind, i)
                assert np.array_equal(crops[i], ref), (kind, i)
    # the align functions take host images and run on the current device
    img = rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8)
    Ms = np.stack([random_affine(rng, 1080, 1920, 112, w, s) for w in ("inside", "partial", "outside")
                   for s in (False, True)])
    base = golden("test1")["f0_res_kps"][0].astype(np.float64)
    kps = np.stack([base * s + o for s, o in ((1.0, 0.0), (2.5, 300.0), (0.5, -20.0))])
    with _current(B):
        got = warp_affine(img, Ms, (112, 112))
        chips, M = align_faces(img, kps, 112)
    for i in range(len(Ms)):
        assert np.array_equal(got[i], cv2_warp(img, Ms[i], 112)), i
    for i in range(len(kps)):
        assert np.array_equal(chips[i], cv2_warp(img, M[i], 112)), i


# ------------------------------------------------------------------------------------------------ 4. current device
def _every_public_call(dev, imgs):
    """Constructs one object of each class on dev and makes every public call on it, checking around each that the
    caller's current device does not move; returns the objects."""
    import torch
    from Skps import FaceAna, FaceAnaImages, FaceAnaStreams, FaceDetector, FaceLandmark
    from peppa_pig_face_landmark_b200 import ONNXEngine
    from peppa_pig_face_landmark_b200.core.api.align import align_faces, warp_affine
    cur = torch.cuda.current_device()

    def call(what, f, *a, **k):
        r = f(*a, **k)
        assert torch.cuda.current_device() == cur, "%s on %s moved the current device %d -> %d" % (
            what, dev, cur, torch.cuda.current_device())
        return r

    cuda = [_cuda(f, dev) for f in imgs]
    fd = call("FaceDetector()", FaceDetector, max_frames=2, device=dev)
    call("FaceDetector.run_batch", fd.run_batch, imgs)
    call("FaceDetector.__call__", fd, imgs[0])
    call("FaceDetector.preprocess", fd.preprocess, imgs[0])
    out = call("FaceDetector.new_results", fd.new_results, len(imgs))
    call("FaceDetector.submit", fd.submit, cuda, out=out)
    call("FaceDetector.submit", fd.submit, imgs)
    call("FaceDetector.collect", fd.collect)
    call("FaceDetector.collect", fd.collect)
    boxes = [r[:, :4] for r in fd.run_batch(imgs)]
    fl = call("FaceLandmark()", FaceLandmark, max_faces=4, device=dev)
    call("FaceLandmark.run_batch", fl.run_batch, imgs, boxes)
    call("FaceLandmark.__call__", fl, imgs[0], boxes[0])
    call("FaceLandmark.crops", fl.crops, imgs[0], boxes[0])
    out = call("FaceLandmark.new_results", fl.new_results, sum(len(b) for b in boxes))
    call("FaceLandmark.submit", fl.submit, cuda, boxes, out=out)
    call("FaceLandmark.submit", fl.submit, imgs, boxes)
    call("FaceLandmark.collect", fl.collect)
    call("FaceLandmark.collect", fl.collect)
    fi = call("FaceAnaImages()", FaceAnaImages, pose=True, max_frames=2, max_faces=8, device=dev)
    call("FaceAnaImages.run_batch", fi.run_batch, imgs)
    out = call("FaceAnaImages.new_results", fi.new_results, len(imgs))
    call("FaceAnaImages.submit", fi.submit, cuda, out=out)
    call("FaceAnaImages.submit", fi.submit, imgs)
    call("FaceAnaImages.collect", fi.collect)
    call("FaceAnaImages.collect", fi.collect)
    fs = call("FaceAnaStreams()", FaceAnaStreams, n_streams=len(imgs), align=112, pose=True, device=dev)
    call("FaceAnaStreams.run", fs.run, imgs)
    out = call("FaceAnaStreams.new_results", fs.new_results)
    call("FaceAnaStreams.submit", fs.submit, cuda, out=out)
    call("FaceAnaStreams.submit", fs.submit, imgs)
    call("FaceAnaStreams.collect", fs.collect)
    call("FaceAnaStreams.collect", fs.collect)
    call("FaceAnaStreams.reset", fs.reset)
    eng = call("ONNXEngine()", ONNXEngine, _detector_path(), device=dev, max_batch=1)
    x = np.zeros((1, 384, 640, 3), np.uint8)
    call("ONNXEngine.run_u8", eng.run_u8, x)
    call("ONNXEngine.__call__", eng, x.transpose(0, 3, 1, 2).astype(np.float32))
    call("ONNXEngine.stream_u8", lambda: list(eng.stream_u8([x, x, x])))
    call("ONNXEngine.forward_device", eng.forward_device, _cuda(x, dev))
    call("ONNXEngine.read_buffer", eng.read_buffer, 0, 1)
    kps = fi.run_batch(imgs[:1])[0][0]["kps"][None].astype(np.float64)
    call("warp_affine", warp_affine, imgs[0], np.eye(2, 3)[None], (64, 32))
    call("align_faces", align_faces, imgs[0], kps)
    torch.cuda.synchronize(dev)
    return fd, fl, fi, fs


def _detector_path():
    from peppa_pig_face_landmark_b200.core.api import face_detector as m
    from peppa_pig_face_landmark_b200.core.api.facer import get_cfg
    root = m.pathlib.Path(m.__file__).resolve().parents[2]
    return str(root / get_cfg()['Skps']['Detect']['model_path'])


def _face_ana_calls(fa, imgs, cur, what):
    import torch
    for f in imgs + [_cuda(imgs[0], fa._device)]:
        fa.run(f)
        assert torch.cuda.current_device() == cur, (what, "run")
    fa.reset()
    assert torch.cuda.current_device() == cur, (what, "reset")


def test_calls_leave_the_current_device_alone(devs):
    from Skps import FaceAna
    A, B = devs
    imgs = [frames.load_test1(), video_frames()[0]]
    with _current(A):                                   # objects on B with A current
        _every_public_call(B, imgs)
    with _current(B):                                   # objects on A under torch.cuda.device(B)
        _every_public_call(A, imgs)
    with _current(B):
        fb = FaceAna(align=112, pose=True, track_ids=True)
    with _current(A):
        fa = FaceAna(align=112, pose=True, track_ids=True)
        _face_ana_calls(fb, imgs, A.index, "FaceAna on B")
    with _current(B):
        _face_ana_calls(fa, imgs, B.index, "FaceAna on A")


# ------------------------------------------------------------------------------------------------ 5. taking turns
def _take_turns(objs, calls, submit):
    """submit(obj, k, i) for call i on every object in turn, collecting an object's oldest call before its third;
    returns each object's results in call order."""
    got = [[] for _ in objs]
    for i in range(len(calls)):
        for k, o in enumerate(objs):
            if len(o._pending) == 2:
                got[k].append(o.collect())
            submit(o, k, i)
    for k, o in enumerate(objs):
        while o._pending:
            got[k].append(o.collect())
    return got


def test_two_devices_take_turns_with_calls_in_flight(devs):
    """Objects of one class on A and B alternate their calls, two in flight on each; every result equals a blocking
    run on the object's own device.  B takes CUDA frames on every other call."""
    from Skps import FaceAnaImages, FaceAnaStreams, FaceDetector, FaceLandmark
    v = video_frames()
    calls = [[frames.load_test1(), v[0]], [frames.frame_4k(), frames.canvas_640()], [v[3], frames.load_test1()],
             [v[4], v[1]]]

    def frames_of(k, i):
        return calls[i] if k == 0 or i % 2 else [_cuda(f, devs[k]) for f in calls[i]]

    with _current(devs[0]):
        for name, make in (("FaceDetector", lambda d: FaceDetector(max_frames=2, device=d)),
                           ("FaceAnaImages", lambda d: FaceAnaImages(pose=True, max_frames=2, max_faces=8, device=d))):
            objs = [make(d) for d in devs]
            want = [[o.run_batch(c) for c in calls] for o in objs]
            got = _take_turns(objs, calls, lambda o, k, i: o.submit(frames_of(k, i)))
            for k in range(2):
                for i, (g, w) in enumerate(zip(got[k], want[k])):
                    if name == "FaceDetector":
                        assert len(g) == len(w) and all(np.array_equal(x, y) for x, y in zip(g, w)), (name, k, i)
                    else:
                        _same_images(g, w, (name, k, i))
        boxes = [[r[:, :4] for r in FaceDetector(device=devs[0]).run_batch(c)] for c in calls]
        fls = [FaceLandmark(max_faces=4, device=d) for d in devs]
        want = [[o.run_batch(c, b) for c, b in zip(calls, boxes)] for o in fls]
        got = _take_turns(fls, calls, lambda o, k, i: o.submit(frames_of(k, i), boxes[i]))
        for k in range(2):
            for i, (g, w) in enumerate(zip(got[k], want[k])):
                for (a, s), (wa, ws) in zip(g, w):
                    assert np.array_equal(a, wa) and np.array_equal(s, ws), ("FaceLandmark", k, i)
        seqs = _sequences()
        steps = [[s[t] for s in seqs] for t in range(6)]
        ref = [FaceAnaStreams(n_streams=len(seqs), align=112, pose=True, device=d) for d in devs]
        want = [[o.run(st) for st in steps] for o in ref]
        fss = [FaceAnaStreams(n_streams=len(seqs), align=112, pose=True, device=d) for d in devs]
        got = _take_turns(fss, steps, lambda o, k, i: o.submit(steps[i]))
        for k in range(2):
            for t in range(6):
                for j in range(len(seqs)):
                    _same_faces(got[k][t][j], want[k][t][j], ("FaceAnaStreams", k, t, j))
                    _same_faces(got[k][t][j], want[0][t][j], ("FaceAnaStreams vs A", k, t, j))


# ------------------------------------------------------------------------------------------------ 6. mismatched engines
def test_pipelines_refuse_engines_on_two_devices(devs):
    import torch
    from Skps import FaceDetector, FaceLandmark
    from peppa_pig_face_landmark_b200 import runtime as rt
    from peppa_pig_face_landmark_b200.core.api.facer import get_cfg, pipeline_cfg
    A, B = devs
    lib = rt.load_library()
    pc = pipeline_cfg(get_cfg()['Skps'], 5, (1080, 1920))
    with _current(A):
        det = {d: FaceDetector(max_frames=2, device=d).model for d in (A, B)}
        kps = {d: FaceLandmark(max_faces=10, device=d).model for d in (A, B)}
        for dd, kd in ((A, B), (B, A)):
            for name, create in (
                    ("skps_pipeline_create", lambda h: lib.skps_pipeline_create(det[dd].handle, kps[kd].handle,
                                                                                C.byref(pc), C.byref(h))),
                    ("skps_mpipe_create", lambda h: lib.skps_mpipe_create(det[dd].handle, kps[kd].handle, C.byref(pc),
                                                                          2, C.byref(h)))):
                h = C.c_void_p()
                assert create(h) != 0 and not h.value, name
                msg = lib.skps_last_error().decode()
                assert "device %d" % dd.index in msg and "device %d" % kd.index in msg, (name, msg)
                assert torch.cuda.current_device() == A.index
        h = C.c_void_p()                                 # engines on one device (B) still make a pipeline there
        rt.check(lib.skps_pipeline_create(det[B].handle, kps[B].handle, C.byref(pc), C.byref(h)))
        lib.skps_pipeline_destroy(h)
