"""FaceLandmark over many frames per call (run_batch, submit / collect, out=) and its crop kernel skps_crop_faces.  The
reference for every comparison is a per-frame restatement of what FaceLandmark.__call__ did before it ran on the batched
path: the whole frame uploaded, then per chunk of max_faces skps_crop_resize, skps_engine_forward and skps_landmark_post.
Every comparison is exact."""
import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames

pytestmark = pytest.mark.gpu

EDGE = np.array([[-30.5, -20.25, 120.0, 150.75], [500.2, 300.4, 700.9, 520.1], [100, 100, 130.5, 300.25],
                 [10.1, 200.2, 600.3, 260.4], [300.7, 10.2, 333.3, 45.9], [0, 0, 639, 479],
                 [200.5, 150.5, 420.25, 400.75],
                 [-400, -300, -100.5, -20], [700, 500, 1000.25, 800], [640.5, 10, 700, 80],     # wholly outside
                 [50, 60, 70, 90], [50, 60, 90, 80.5], [10, 10, 31, 31.5],                     # sides <= 20, and just over
                 [-2000, -1500, 2600.5, 1900]], np.float32)                                   # larger than the frame


def _lib():
    from peppa_pig_face_landmark_b200 import runtime as rt
    return rt, rt.load_library()


def _restated(fl, img, boxes):
    """FaceLandmark(cfg)(img, boxes) as it was computed before the batched path, for k >= 0 boxes."""
    import torch
    rt, lib = _lib()
    K, P, S = fl.max_faces, fl.keypoints_num, fl.input_size[0]
    boxes = np.asarray(boxes, np.float32).reshape(-1, np.shape(boxes)[-1] if np.size(boxes) else 4)
    lms, scs = [np.zeros((0, P, 2), np.float32)], [np.zeros((0, P), np.float32)]
    if not len(boxes):
        return lms[0], scs[0]
    img = np.ascontiguousarray(img)
    h, w = img.shape[:2]
    frame = torch.from_numpy(img).cuda()
    d_boxes = torch.zeros((K, 4), dtype=torch.float32, device="cuda")
    count = torch.zeros((1,), dtype=torch.int32, device="cuda")
    detail = torch.zeros((K, 5), dtype=torch.int32, device="cuda")
    kps = torch.zeros((K, P, 2), dtype=torch.float32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    for i in range(0, len(boxes), K):
        b = boxes[i:i + K]
        n = len(b)
        d_boxes[:n].copy_(torch.from_numpy(np.ascontiguousarray(b[:, :4])))
        count.fill_(n)
        rt.check(lib.skps_crop_resize(frame.data_ptr(), h, w, w * 3, d_boxes.data_ptr(), count.data_ptr(), K,
                                      fl.face_scale, float(fl.min_face), fl.model.input_ptr(), S, detail.data_ptr(), s))
        rt.check(lib.skps_engine_forward(fl.model.handle, fl.model.input_ptr(), K, None, s))
        rt.check(lib.skps_landmark_post(fl.model.output_ptr(0), detail.data_ptr(), count.data_ptr(), K, P, kps.data_ptr(), s))
        torch.cuda.synchronize()
        scores = np.empty((K, P), np.float32)
        rt.check(lib.skps_engine_read_buffer(fl.model.handle, fl.model.plan.outputs[1].buf.idx, K, scores.ctypes.data))
        lms.append(kps[:n].cpu().numpy())
        scs.append(scores[:n].copy())
    return np.concatenate(lms), np.concatenate(scs)


def _same(got, want, what=""):
    assert len(got) == len(want), (what, len(got), len(want))
    for i, ((k, s), (wk, ws)) in enumerate(zip(got, want)):
        k, s = (k.cpu().numpy() if hasattr(k, "cpu") else k), (s.cpu().numpy() if hasattr(s, "cpu") else s)
        assert k.dtype == wk.dtype == np.float32 and s.dtype == ws.dtype == np.float32, (what, i)
        assert k.shape == wk.shape and s.shape == ws.shape, (what, i, k.shape, wk.shape)
        assert np.array_equal(k, wk), (what, i, np.abs(k - wk).max() if k.size else 0)
        assert np.array_equal(s, ws), (what, i)


def _cuda(f):
    import torch
    return torch.from_numpy(np.ascontiguousarray(f)).cuda()


def _pitched(f):
    """f as a view of a wider buffer whose rows are not 16-byte multiples apart."""
    import torch
    H, W = f.shape[:2]
    pad = next(p for p in range(1, 16) if (3 * (W + p)) % 16)
    buf = torch.full((H, W + pad, 3), 201, dtype=torch.uint8, device="cuda")
    buf[:, :W] = _cuda(f)
    return buf[:, :W]


def _roi(f):
    """f as big[y0:y1, x0:x1] of a larger frame, starting at an odd byte offset."""
    import torch
    H, W = f.shape[:2]
    buf = torch.full((H + 3, W + 4, 3), 37, dtype=torch.uint8, device="cuda")
    buf[2:2 + H, 1:1 + W] = _cuda(f)
    v = buf[2:2 + H, 1:1 + W]
    assert v.storage_offset() % 2 == 1
    return v


LAYOUTS = {"packed": _cuda, "pitched": _pitched, "roi": _roi}


@pytest.fixture(scope="module")
def fl():
    from Skps import FaceLandmark
    return FaceLandmark()


@pytest.fixture(scope="module")
def golden_set():
    """(frames, boxes): test1, canvas640 and uhd4k (16 faces) with the oracle detector's boxes, the 1080p clip with its
    first frame's boxes, a 480x640 noise frame with the edge boxes (and 16-column rows), and a frame with no boxes."""
    from oracle import host_ref as H
    from oracle.faceana_ref import DetectorRef
    det = DetectorRef()
    fs, bs = [], []
    for fr, k in ((frames.load_test1(), 5), (frames.canvas_640(), 5), (frames.frame_4k(), 16)):
        fs.append(fr)
        bs.append(np.asarray(H.sort_and_filter(det(fr), 1600, k), np.float32))
    clip = video_frames()
    b0 = np.asarray(H.sort_and_filter(det(clip[0]), 1600, 5), np.float32)
    for fr in clip:
        fs.append(fr)
        bs.append(b0)
    rng = np.random.default_rng(11)
    fs.append(rng.integers(0, 256, (480, 640, 3), dtype=np.uint8))
    rows = np.concatenate([EDGE, rng.uniform(0, 1, (len(EDGE), 12)).astype(np.float32)], 1)
    bs.append(rows)
    fs.append(frames.load_test1())
    bs.append(np.zeros((0, 4), np.float32))
    assert all(len(b) for b in bs[:3]) and len(bs[2]) == 16
    return fs, bs


@pytest.fixture(scope="module")
def want(fl, golden_set):
    return [_restated(fl, f, b) for f, b in zip(*golden_set)]


def test_host_frames_equal_the_restatement(fl, golden_set, want):
    fs, bs = golden_set
    keep = [b.copy() for b in bs]
    _same(fl.run_batch(fs, bs), want, "host")
    assert all(np.array_equal(a, b) for a, b in zip(bs, keep))                 # the caller's boxes are not modified


def test_call_equals_the_restatement(fl, golden_set, want):
    fs, bs = golden_set
    for i, (f, b) in enumerate(zip(fs, bs)):
        if len(b):
            _same([fl(f, b)], [want[i]], "call %d" % i)
            assert fl.last_detail.shape == (len(b), 5)


def test_chunks_smaller_than_a_call():
    """max_faces 4: every call runs in several chunks, with faces of one frame split between chunks."""
    from Skps import FaceLandmark
    small = FaceLandmark(max_faces=4)
    f4k, f1 = frames.frame_4k(), frames.load_test1()
    rng = np.random.default_rng(3)
    b4k = np.array([[x, y, x + 600, y + 400] for y in (140, 680, 1220, 1760) for x in (180, 1140, 2100, 3060)], np.float32)
    b4k += rng.uniform(-3, 3, b4k.shape).astype(np.float32)
    b1 = np.array([[153.4755, 49.7373, 306.6512, 234.0922], [100, 40, 260, 200]], np.float32)
    fs, bs = [f1, f4k, f1, f1], [b1, b4k, np.zeros((0, 4), np.float32), b1[:1]]
    want = [_restated(small, f, b) for f, b in zip(fs, bs)]
    _same(small.run_batch(fs, bs), want, "host chunks")
    _same(small.run_batch([_cuda(f) for f in fs], bs), want, "cuda chunks")
    _same(small.run_batch([_cuda(f) for f in fs], [_cuda(b) for b in bs]), want, "cuda boxes chunks")


@pytest.mark.parametrize("kind", sorted(LAYOUTS))
def test_cuda_frames_equal_the_restatement(fl, golden_set, want, kind):
    fs, bs = golden_set
    dev = [LAYOUTS[kind](f) for f in fs]
    _same(fl.run_batch(dev, bs), want, kind + " host boxes")
    wide = [_cuda(np.concatenate([b, np.full((len(b), 3), 7, np.float32)], 1)) for b in bs]    # (k, >= 4) CUDA boxes
    _same(fl.run_batch(dev, wide), want, kind + " cuda boxes")


def test_device_results_equal_host_results(fl, golden_set, want):
    """Two calls in flight into out= buffers, then a host-result call in between."""
    fs, bs = golden_set
    dev = [_cuda(f) for f in fs]
    n = sum(len(b) for b in bs)
    bufs = [fl.new_results(n), fl.new_results(n + 5)]
    fl.submit(dev, bs, out=bufs[0])
    fl.submit(dev[::-1], [_cuda(b) for b in bs[::-1]], out=bufs[1])
    r0 = fl.collect()
    fl.submit(fs[:3], bs[:3])
    r1 = fl.collect()
    r2 = fl.collect()
    _same(r0, want, "out 0")
    _same(r1, want[::-1], "out 1")
    _same(r2, want[:3], "host between")
    assert r0[0][0].data_ptr() == bufs[0]["kps"].data_ptr()


def test_calls_in_flight_keep_their_staging(fl, golden_set, want):
    """The first call is held back behind a sleeping producer stream, so its crops run late; the third call reuses the
    first call's staging slot while they are pending.  Without the wait for the first call's read, its descriptors and
    boxes would be overwritten by the third call's before its crops run."""
    import torch
    fs, bs = golden_set
    dev = [_cuda(f) for f in fs]
    order = [list(range(len(fs))), list(range(len(fs)))[::-1], [2, 0, 1, 3]]
    n = sum(len(b) for b in bs)
    bufs = [fl.new_results(n) for _ in range(3)]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        fl.submit([dev[i] for i in order[0]], [bs[i] for i in order[0]], out=bufs[0])
    fl.submit([dev[i] for i in order[1]], [bs[i] for i in order[1]], out=bufs[1])
    got = [fl.collect()]
    fl.submit([dev[i] for i in order[2]], [bs[i] for i in order[2]], out=bufs[2])
    got += [fl.collect(), fl.collect()]
    for t in range(3):
        _same(got[t], [want[i] for i in order[t]], "call %d" % t)
    # host frames: the third call's rectangles go into the first call's pinned staging
    fl.submit(fs, bs)
    fl.submit(fs[:3], bs[:3])
    r0 = fl.collect()
    fl.submit(fs[3:], bs[3:])
    _same(r0, want, "host 0")
    _same(fl.collect(), want[:3], "host 1")
    _same(fl.collect(), want[3:], "host 2")


def test_frames_are_read_after_the_producer_stream(fl):
    """Frame and CUDA boxes are written on a side stream behind a sleep and submitted under it: without the wait on the
    producer's stream the crops would read the blank frame."""
    import torch
    f = frames.frame_1080p()
    b = np.array([[x, y, x + 440, y + 293] for y in (123, 663) for x in (260, 1220)], np.float32)
    want = [_restated(fl, f, b)]
    src, bsrc = _cuda(f), _cuda(b)
    frame, boxes = torch.zeros_like(src), torch.zeros_like(bsrc)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        frame.copy_(src)
        boxes.copy_(bsrc)
        got = fl.run_batch([frame], [boxes])
    _same(got, want)
    torch.cuda.synchronize()


def test_producer_may_overwrite_the_frame_once_submit_returns(fl):
    """Right after submit the caller zeroes the frame and the boxes on its stream.  The landmark stream is held back (a
    first call waits on a sleeping side stream), so without the wait for the read the zeroing would land first."""
    import torch
    f0, f1 = frames.frame_1080p(), frames.frame_1080p(jitter=(8, -4))
    b = np.array([[x, y, x + 440, y + 293] for y in (123, 663) for x in (260, 1220)], np.float32)
    want = [[_restated(fl, f0, b)], [_restated(fl, f1, b)]]
    a, c, bb = _cuda(f0), _cuda(f1), _cuda(b)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        fl.submit([a], [b])
    fl.submit([c], [bb])
    c.zero_()
    bb.zero_()
    _same(fl.collect(), want[0], "call 0")
    _same(fl.collect(), want[1], "call 1")


def test_invalid_inputs_raise_before_anything_is_enqueued(fl):
    import torch
    f = frames.load_test1()
    good, b = _cuda(f), np.array([[153.4755, 49.7373, 306.6512, 234.0922]], np.float32)
    planar = _cuda(np.ascontiguousarray(f.transpose(2, 0, 1))).permute(1, 2, 0)
    bad_calls = [
        ([f, f], [b]),                                               # lengths differ
        ([f, good], [b, b]),                                         # host and CUDA frames
        ([f.astype(np.float32)], [b]), ([f[:, :, :2]], [b]), ([f[0]], [b]),
        ([good.float()], [b]), ([planar], [b]), ([good[0]], [b]), ([good, torch.from_numpy(f)], [b, b]),
        ([f], [b[:, :3]]), ([f], [b[0]]), ([f], [np.array([[np.nan, 0, 50, 50]], np.float32)]),
        ([f], [np.array([[0, 0, 3e7, 50]], np.float32)]),
        ([f], [_cuda(b)]),                                           # CUDA boxes with host frames
        ([good, good], [_cuda(b), b]),                               # CUDA and host boxes
        ([good], [_cuda(b).double()]), ([good], [_cuda(b)[:, :3]]), ([good], [torch.from_numpy(b)[None].cuda()]),
    ]
    for i, (fs, bs) in enumerate(bad_calls):
        with pytest.raises(ValueError):
            fl.submit(fs, bs)
        assert not fl._pending, i
    with pytest.raises(ValueError):
        fl.submit([f], [b], out=fl.new_results(1))                   # out= takes CUDA frames
    res = fl.new_results(2)
    for bent in ({"kps": res["kps"]}, {"kps": res["kps"][:0], "scores": res["scores"][:0]},
                 {"kps": res["kps"].double(), "scores": res["scores"]}, {"kps": res["kps"].cpu(), "scores": res["scores"]},
                 {"kps": res["kps"][:, :, :1], "scores": res["scores"]}):
        with pytest.raises(ValueError):
            fl.submit([good, good], [b, b], out=bent)
    with pytest.raises(ValueError):
        fl.submit([good, good, good], [b, b, b], out=res)            # too small
    assert not fl._pending
    fl.submit([good], [b], out=res)
    with pytest.raises(ValueError):
        fl.submit([good], [b], out=res)                              # still in flight
    fl.submit([f], [b])
    with pytest.raises(RuntimeError):
        fl.submit([f], [b])                                          # a third call
    assert len(fl._pending) == 2
    want = [_restated(fl, f, b)]
    _same(fl.collect(), want)
    _same(fl.collect(), want)


def test_crop_faces_equals_crop_resize(fl):
    """skps_crop_faces with whole-frame descriptors and with host-style rectangle descriptors writes the crops and
    details skps_crop_resize writes for the same boxes, face for face."""
    import torch
    from peppa_pig_face_landmark_b200.core.api.face_landmark import FACE_SRC, crop_read_rects
    rt, lib = _lib()
    rng = np.random.default_rng(5)
    imgs = [rng.integers(0, 256, (480, 640, 3), dtype=np.uint8), frames.load_test1(),
            rng.integers(0, 256, (1, 1, 3), dtype=np.uint8), rng.integers(0, 256, (37, 23, 3), dtype=np.uint8)]
    boxes = [EDGE, np.array([[153.4755, 49.7373, 306.6512, 234.0922], [-50, -50, 500, 400]], np.float32),
             np.array([[-30, -30, 10.5, 12], [0, 0, 1, 1], [-0.5, -0.25, 25, 25]], np.float32),
             np.array([[2.5, 3, 30, 40], [-10, 20, 14, 45.5]], np.float32)]
    S, fs, mf = fl.input_size[0], fl.face_scale, float(fl.min_face)
    s = torch.cuda.current_stream().cuda_stream
    want_c, want_d = [], []
    for img, b in zip(imgs, boxes):
        K = len(b)
        fr, d_b = _cuda(img), _cuda(b)
        count = torch.tensor([K], dtype=torch.int32, device="cuda")
        crops = torch.zeros((K, S, S, 3), dtype=torch.uint8, device="cuda")
        det = torch.zeros((K, 5), dtype=torch.int32, device="cuda")
        rt.check(lib.skps_crop_resize(fr.data_ptr(), img.shape[0], img.shape[1], img.shape[1] * 3, d_b.data_ptr(),
                                      count.data_ptr(), K, fs, mf, crops.data_ptr(), S, det.data_ptr(), s))
        want_c.append(crops.cpu().numpy())
        want_d.append(det.cpu().numpy())
    want_c, want_d = np.concatenate(want_c), np.concatenate(want_d)
    n = len(want_d)
    all_boxes = _cuda(np.concatenate(boxes))
    keep = []
    for mode in ("whole", "rect"):
        desc = np.zeros(n, FACE_SRC)
        o = 0
        for img, b in zip(imgs, boxes):
            H, W = img.shape[:2]
            if mode == "whole":
                fr = _pitched(img)
                keep.append(fr)
                d = desc[o:o + len(b)]
                d["base"], d["pitch"], d["H"], d["W"], d["rw"], d["rh"] = fr.data_ptr(), fr.stride(0), H, W, W, H
            else:
                for j, r in enumerate(crop_read_rects(b, H, W, fs)):
                    x0, y0, x1, y1 = (int(v) for v in r)
                    part = _cuda(img[y0:y1, x0:x1]) if x1 > x0 else torch.zeros(1, dtype=torch.uint8, device="cuda")
                    keep.append(part)
                    desc[o + j] = (part.data_ptr(), 3 * (x1 - x0), H, W, x0, y0, x1 - x0, y1 - y0, 0)
            o += len(b)
        d_desc = _cuda(desc.view(np.uint8))
        crops = torch.full((n, S, S, 3), 99, dtype=torch.uint8, device="cuda")
        det = torch.full((n, 5), -9, dtype=torch.int32, device="cuda")
        rt.check(lib.skps_crop_faces(d_desc.data_ptr(), all_boxes.data_ptr(), n, fs, mf, crops.data_ptr(), S,
                                     det.data_ptr(), s))
        assert np.array_equal(det.cpu().numpy(), want_d), mode
        got = crops.cpu().numpy()
        for i in range(n):
            assert np.array_equal(got[i], want_c[i]), (mode, i)
    rt.check(lib.skps_crop_faces(None, None, 0, fs, mf, None, S, None, s))          # no faces: nothing to do
