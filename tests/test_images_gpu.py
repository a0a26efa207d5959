"""FaceAnaImages: FaceAna.run after reset() for many still images per call.  The reference for every comparison is
FaceAna itself, run image by image on a just-reset object, and every comparison with it is bit for bit (np.array_equal
and dtype).  The golden results of the reference project are checked within test_parity_gpu's tolerances.  The FaceAna
reference results are always computed before or after the FaceAnaImages calls, never between a submit and its collect."""
import types

import numpy as np
import pytest

import frames
from test_crowd_cpu import crowd_frame
from test_detector_batch_gpu import mixed_frames
from test_landmark_batch_gpu import LAYOUTS, _cuda
from test_parity_gpu import _check_result, _edge_frames

pytestmark = pytest.mark.gpu

BIG = (4096, 4096)          # FaceAna's max_frame_hw: large enough for every image here


def _lib():
    from peppa_pig_face_landmark_b200 import runtime as rt
    return rt, rt.load_library()


def faceana_results(images, top_k=None, det_input=None, pose=False):
    """FaceAna(...).run(image) on a just-reset FaceAna, image by image."""
    from Skps import FaceAna
    fa = FaceAna(top_k=top_k, det_input=det_input, pose=pose, max_frame_hw=BIG)
    res = []
    for img in images:
        fa.reset()
        res.append(fa.run(img))
    return res


def _same(got, want, what="", pose=None):
    """got equals want bit for bit; pose=False drops want's 'pose' (FaceAna(pose=True) is FaceAna plus 'pose')."""
    assert len(got) == len(want), (what, len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w), (what, i, len(g), len(w))
        for j, (a, b) in enumerate(zip(g, w)):
            keys = set(b) - ({"pose"} if pose is False else set())
            assert set(a) == keys, (what, i, j, set(a), keys)
            for k in ("box", "kps", "scores"):
                assert a[k].dtype == b[k].dtype == np.float32, (what, i, j, k, a[k].dtype, b[k].dtype)
                assert np.array_equal(a[k], b[k]), (what, i, j, k, np.abs(a[k].astype(np.float64) - b[k]).max())
            if "pose" in keys:
                assert set(a["pose"]) == set(b["pose"]), (what, i, j)
                for k, v in b["pose"].items():
                    assert a["pose"][k].dtype == v.dtype == np.float64 and np.array_equal(a["pose"][k], v), (what, i, j, k)


def _from_out(out, n, pose):
    """The per-image result lists held in new_results buffers."""
    first, count = out["first"][:n].cpu().numpy(), out["count"][:n].cpu().numpy()
    host = {k: v.cpu().numpy() for k, v in out.items() if k not in ("first", "count")}
    res = []
    for o, k in zip(first.tolist(), count.tolist()):
        faces = [{"box": host["box"][o + j], "kps": host["kps"][o + j], "scores": host["scores"][o + j]} for j in range(k)]
        if pose:
            for j, r in enumerate(faces):
                r["pose"] = {name: host[name][o + j] for name in ("rvec", "tvec", "euler", "reproject")}
        res.append(faces)
    return res


@pytest.fixture(scope="module")
def images():
    """mixed_frames (twelve frames of eight sizes: a 4000x3000 still, a portrait frame, a faceless frame, a 96-face
    crowd) and test_parity_gpu's edge frames."""
    return mixed_frames() + list(_edge_frames().values())


@pytest.fixture(scope="module")
def want16(images):
    return faceana_results(images, top_k=16, pose=True)


@pytest.fixture(scope="module")
def fi16():
    from Skps import FaceAnaImages
    return FaceAnaImages(top_k=16, pose=True)


# ----------------------------------------------------------------------------- 1. against FaceAna, image by image
@pytest.mark.parametrize("top_k,det_input", [(5, None), (16, None), (5, (768, 1280)), (16, (768, 1280))],
                         ids=["top5", "top16", "top5-768x1280", "top16-768x1280"])
def test_one_mixed_call_equals_faceana_per_image(images, top_k, det_input):
    from Skps import FaceAnaImages
    want = faceana_results(images, top_k, det_input, pose=True)
    assert any(len(w) == 0 for w in want) and sum(len(w) for w in want) > 2 * len(images)
    for pose in (False, True):
        fi = FaceAnaImages(top_k=top_k, det_input=det_input, pose=pose)
        _same(fi.run_batch(images), want, (top_k, det_input, pose), pose=pose)
        del fi


# ----------------------------------------------------------------------------- 2. against the reference's golden results
def test_golden_results(golden):
    from Skps import FaceAnaImages
    imgs = [frames.load_test1(), frames.canvas_640(), frames.frame_4k()]
    for top_k, names in ((5, ["test1", "canvas640", "uhd4k_top5"]), (16, ["test1", "canvas640", "uhd4k_top16"])):
        res = FaceAnaImages(top_k=top_k).run_batch(imgs)
        for r, name in zip(res, names):
            _check_result(r, golden(name), 0, name)


# ----------------------------------------------------------------------------- 3. crowds
@pytest.mark.parametrize("top_k", [1024, 16])
def test_crowd(top_k):
    from Skps import FaceAnaImages
    hw = (1152, 1920)
    crowd = crowd_frame("crowd384_1152x1920")
    imgs = [crowd, crowd.copy()]
    want = faceana_results(imgs[:1], top_k, hw) * 2
    assert len(want[0]) == min(top_k, 384)
    fi = FaceAnaImages(top_k=top_k, det_input=hw)
    _same(fi.run_batch(imgs), want, top_k)
    _same(fi.run_batch([_cuda(f) for f in imgs]), want, (top_k, "cuda"))


# ----------------------------------------------------------------------------- 4. frame forms and out=
@pytest.mark.parametrize("kind", sorted(LAYOUTS))
def test_cuda_images_and_out_equal_host_images(fi16, images, want16, kind):
    dev = [LAYOUTS[kind](f) for f in images]
    _same(fi16.run_batch(dev), want16, kind)
    out = fi16.new_results(len(images) + 2)
    fi16.submit(dev, out=out)
    assert fi16.collect() is out
    _same(_from_out(out, len(images), True), want16, kind + " out")


# ----------------------------------------------------------------------------- 5. chunking
def test_small_chunks_equal_the_defaults(images):
    from Skps import FaceAnaImages
    imgs = images[:9]
    big = FaceAnaImages(top_k=16).run_batch(imgs)
    assert 30 <= sum(len(r) for r in big)
    small = FaceAnaImages(top_k=16, max_frames=3, max_faces=5)
    _same(small.run_batch(imgs), big, "host")
    _same(small.run_batch([_cuda(f) for f in imgs]), big, "cuda")


# ----------------------------------------------------------------------------- 6. calls in flight
def test_two_calls_in_flight_equal_blocking_calls(fi16, images, want16):
    a, b = list(range(0, len(images), 2)), list(range(1, len(images), 2))[::-1]
    fi16.submit([images[i] for i in a])
    fi16.submit([images[i] for i in b])
    ra, rb = fi16.collect(), fi16.collect()
    _same(ra, [want16[i] for i in a], "first")
    _same(rb, [want16[i] for i in b], "second")
    dev = [_cuda(f) for f in images]
    outs = [fi16.new_results(len(a)), fi16.new_results(len(b))]
    fi16.submit([dev[i] for i in a], out=outs[0])
    fi16.submit([dev[i] for i in b])
    assert fi16.collect() is outs[0]
    rb = fi16.collect()
    fi16.submit([dev[i] for i in b], out=outs[1])                     # reuses the first call's slot
    fi16.collect()
    _same(_from_out(outs[0], len(a), True), [want16[i] for i in a], "out 0")
    _same(rb, [want16[i] for i in b], "host 1")
    _same(_from_out(outs[1], len(b), True), [want16[i] for i in b], "out 1")


# ----------------------------------------------------------------------------- 7. ordering on the producer's stream
def test_images_are_read_after_the_producer_stream(fi16):
    """The image is written on a side stream behind a sleep and submitted under it: without the wait on the producer's
    stream the letterbox would read the blank image."""
    import torch
    f = frames.frame_1080p()
    want = faceana_results([f], 16, pose=True)
    src = _cuda(f)
    img = torch.zeros_like(src)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        img.copy_(src)
        got = fi16.run_batch([img])
    _same(got, want)
    assert len(want[0]) == 4
    torch.cuda.synchronize()


def test_producer_may_overwrite_the_images_once_submit_returns(fi16):
    """Right after submit the caller zeroes the image on its stream.  The engines' streams are held back (a first call
    waits on a sleeping side stream), so without the waits for the reads the zeroing would land first."""
    import torch
    f0, f1 = frames.frame_1080p(), frames.frame_1080p(jitter=(8, -4))
    w0, w1 = faceana_results([f0], 16, pose=True), faceana_results([f1], 16, pose=True)
    a, c = _cuda(f0), _cuda(f1)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        fi16.submit([a])
    fi16.submit([c])
    c.zero_()
    _same(fi16.collect(), w0, "call 0")
    _same(fi16.collect(), w1, "call 1")


# ----------------------------------------------------------------------------- 8. bad inputs
def test_invalid_inputs_raise_before_anything_is_enqueued(fi16):
    import torch
    from Skps import FaceAnaImages
    f = frames.load_test1()
    want = faceana_results([f], 16, pose=True)
    good = _cuda(f)
    planar = _cuda(np.ascontiguousarray(f.transpose(2, 0, 1))).permute(1, 2, 0)
    bad_calls = [
        [f, good],                                                   # host and CUDA images
        [f.astype(np.float32)], [f[:, :, :2]], [f[0]], [good.float()], [planar], [good[0]],
        [good, torch.from_numpy(f)],                                 # a CPU tensor among CUDA images
        [np.zeros((1, 4000, 3), np.uint8)], [_cuda(np.zeros((1, 4000, 3), np.uint8))],     # an empty letterbox
    ]
    for i, imgs in enumerate(bad_calls):
        with pytest.raises(ValueError):
            fi16.submit(imgs)
        assert not fi16._pending, i
    with pytest.raises(ValueError):
        fi16.submit([f], out=fi16.new_results(1))                    # out= takes CUDA images
    res = fi16.new_results(2)
    for bent in ({k: v for k, v in res.items() if k != "euler"}, {k: v[:1] for k, v in res.items()},
                 dict(res, box=res["box"].double()), dict(res, kps=res["kps"].cpu()), dict(res, count=res["count"].long())):
        with pytest.raises(ValueError):
            fi16.submit([good, good], out=bent)
    with pytest.raises(ValueError):
        fi16.submit([good, good, good], out=res)                     # too small
    for top_k in (0, 1025):
        with pytest.raises(ValueError):
            FaceAnaImages(top_k=top_k)
    assert not fi16._pending
    _same(fi16.run_batch([f]), want, "after the errors")
    fi16.submit([good], out=res)
    with pytest.raises(ValueError):
        fi16.submit([good], out=res)                                 # still in flight
    fi16.submit([f])
    with pytest.raises(RuntimeError):
        fi16.submit([f])                                             # a third call
    with pytest.raises(RuntimeError):
        fi16.run_batch([f])
    assert len(fi16._pending) == 2
    assert fi16.collect() is res
    _same(_from_out(res, 1, True), want, "out")
    _same(fi16.collect(), want, "host")
    assert fi16.run_batch([]) == []
    _same(fi16.run_batch([f, f]), want * 2, "after")


# ----------------------------------------------------------------------------- 9. the kernels on their own
def _select_per_image(rows, count, cap, top_k, min_face):
    """skps_select_faces on each image alone: (counts, boxes) on the host."""
    import torch
    rt, lib = _lib()
    n = count.shape[0]
    s = torch.cuda.current_stream().cuda_stream
    b = torch.zeros((n, top_k, 4), dtype=torch.float32, device="cuda")
    c = torch.zeros((n,), dtype=torch.int32, device="cuda")
    for i in range(n):
        rt.check(lib.skps_select_faces(rows.data_ptr() + 64 * cap * i, count.data_ptr() + 4 * i, 16, None, 0, 0.5, 0.3, 0.7,
                                       min_face, top_k, b.data_ptr() + 16 * top_k * i, c.data_ptr() + 4 * i, s))
    return c.cpu().numpy(), b.cpu().numpy()


def _select_batch(rows, count, cap, top_k, min_face):
    import torch
    rt, lib = _lib()
    n = count.shape[0]
    b = torch.full((n, top_k, 4), 7.0, dtype=torch.float32, device="cuda")
    c = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    rt.check(lib.skps_select_faces_batch(rows.data_ptr(), count.data_ptr(), cap, n, min_face, top_k, b.data_ptr(),
                                         c.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return c.cpu().numpy(), b.cpu().numpy()


def _same_selection(got, want, what):
    (gc, gb), (wc, wb) = got, want
    assert np.array_equal(gc, wc), (what, gc, wc)
    for i, k in enumerate(wc.tolist()):
        assert np.array_equal(gb[i, :k], wb[i, :k]), (what, i)


def test_select_faces_batch_equals_select_faces(images):
    import torch
    from Skps import FaceDetector
    rt, lib = _lib()
    fd = FaceDetector()
    out = fd.new_results(len(images))
    fd.submit([_cuda(f) for f in images], out=out)
    fd.collect()
    for top_k in (1, 5, 16, 1024):
        _same_selection(_select_batch(out["rows"], out["count"], fd._rows, top_k, 1600.0),
                        _select_per_image(out["rows"], out["count"], fd._rows, top_k, 1600.0), ("nms", top_k))
    # synthetic rows: past the 8192-row shared cache, equal areas, areas equal to min_face, empty images
    rng = np.random.default_rng(5)
    cap, n = 9000, 6
    rows = np.zeros((n, cap, 16), np.float32)
    xy = rng.uniform(0, 3000, (n, cap, 2)).astype(np.float32)
    side = rng.choice(np.array([40, 40, 41, 39, 50, 80, 120], np.float32), (n, cap, 2))
    rows[:, :, 0:2], rows[:, :, 2:4] = xy, xy + side                 # many equal areas, 40 x 40 = min_face exactly
    rows[:, :, 4:] = rng.uniform(0, 1, (n, cap, 12))
    count = np.array([cap, 8193, 8192, 0, 5, 3000], np.int32)
    d_rows, d_count = _cuda(rows), _cuda(count)
    for top_k in (1, 16, 1024):
        for min_face in (1600.0, 0.0):
            _same_selection(_select_batch(d_rows, d_count, cap, top_k, min_face),
                            _select_per_image(d_rows, d_count, cap, top_k, min_face), ("synthetic", top_k, min_face))
    torch.cuda.synchronize()


def _judge_reference(kps, face_image, sel, sel_count):
    """FaceAna.judge_boxs(boxes, rects(kps)) per image: the host code FaceAna.run runs."""
    from peppa_pig_face_landmark_b200.core.api.facer import FaceAna
    from peppa_pig_face_landmark_b200.core.smoother.lk import EmaFilter, rects
    host = types.SimpleNamespace(iou_thres=0.5, filter=EmaFilter(0.3))
    out = np.zeros((len(kps), 4), np.float32)
    for g in range(len(sel)):
        mine = np.flatnonzero(face_image == g)
        if not len(mine):
            continue
        r = FaceAna.judge_boxs(host, sel[g, :sel_count[g]], rects(kps[mine]))
        assert r.dtype == np.float32
        out[mine] = r
    return out


def test_landmark_boxes_equal_judge_boxs():
    import torch
    rt, lib = _lib()
    P, K = 98, 8
    rng = np.random.default_rng(3)
    n_img = 40
    sel = rng.uniform(0, 1000, (n_img, K, 4)).astype(np.float32)
    sel[:, :, 2:] = sel[:, :, :2] + rng.uniform(30, 300, (n_img, K, 2)).astype(np.float32)
    sel_count = rng.integers(0, K + 1, n_img).astype(np.int32)
    sel_count[3] = 0                                                  # an image with no selected box
    kps, face_image = [], []

    def face(g, rect):
        x0, y0, x1, y1 = (np.float32(v) for v in rect)
        p = np.empty((P, 2), np.float32)
        p[:, 0] = rng.uniform(x0, x1, P)
        p[:, 1] = rng.uniform(y0, y1, P)
        p[0], p[1] = (x0, y0), (x1, y1)                               # the rectangle is exactly rect
        kps.append(p)
        face_image.append(g)

    for g in range(n_img):
        for j in range(sel_count[g]):
            b = sel[g, j]
            jit = rng.uniform(-0.3, 0.3, 4).astype(np.float32) * np.tile(b[2:] - b[:2], 2)
            face(g, b + jit)                                          # near its box: IoU on both sides of 0.5
        face(g, np.tile(rng.uniform(0, 1000, 2), 2))                  # a zero-area rectangle
    # several selected boxes match: the first wins
    sel[5, :3] = [[100, 100, 300, 300], [100, 100, 300, 300], [110, 110, 300, 300]]
    sel_count[5] = max(sel_count[5], 3)
    face(5, [105, 105, 300, 300])
    # IoU exactly at the threshold: [0, 0, 2, 2] against [0, 0, 2, 1] is 2 / 4
    sel[6, 0], sel_count[6] = [0, 0, 2, 1], max(sel_count[6], 1)
    face(6, [0, 0, 2, 2])
    face(3, [0, 0, 50, 50])                                           # its image has no selected box
    kps, face_image = np.stack(kps), np.array(face_image, np.int32)
    want = _judge_reference(kps, face_image, sel, sel_count)
    got = torch.full((len(kps), 4), 7.0, dtype=torch.float32, device="cuda")
    d_kps, d_img, d_sel, d_cnt = _cuda(kps), _cuda(face_image), _cuda(sel), _cuda(sel_count)
    rt.check(lib.skps_landmark_boxes(d_kps.data_ptr(), P, d_img.data_ptr(), len(kps), d_sel.data_ptr(), d_cnt.data_ptr(),
                                     K, 0.5, 0.3, 1 - 0.3, got.data_ptr(), torch.cuda.current_stream().cuda_stream))
    got = got.cpu().numpy()
    assert np.array_equal(got, want), np.abs(got - want).max()
    # both branches were taken: some boxes blended, some left at the landmark rectangle
    rect = np.stack([kps[:, :, 0].min(1), kps[:, :, 1].min(1), kps[:, :, 0].max(1), kps[:, :, 1].max(1)], 1)
    same = np.all(want == rect, 1)
    assert 10 < same.sum() < len(kps) - 10, same.sum()
    assert not np.array_equal(want[-3], rect[-3])                                     # the first of the matches
    assert np.array_equal(want[-2], rect[-2]) and np.array_equal(want[-1], rect[-1])     # at the threshold, no box
