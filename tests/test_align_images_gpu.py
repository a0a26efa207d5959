"""Aligned chips in the batched APIs: FaceAnaImages(align=s) against FaceAna(align=s) image by image, FaceLandmark(align=s)
against cv2.warpAffine and align_faces, and skps_warp_faces' per-face sources (whole images, or only the rectangle
chip_read_rects gives) against each other.  Every comparison is bit for bit."""
import numpy as np
import pytest

import frames
from test_align_gpu import cv2_warp
from test_detector_batch_gpu import mixed_frames
from test_images_gpu import BIG, _from_out, _same
from test_landmark_batch_gpu import LAYOUTS, _cuda
from test_parity_gpu import _edge_frames

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def images():
    """test_images_gpu's images: mixed_frames (a 4000x3000 still, a portrait frame, a faceless frame, a 96-face crowd)
    and test_parity_gpu's edge frames, whose faces touch the border so that chips read outside the image."""
    return mixed_frames() + list(_edge_frames().values())


def faceana_align(images, size):
    """FaceAna(align=size, top_k=16, pose=True).run(image) on a just-reset FaceAna, image by image."""
    from Skps import FaceAna
    fa = FaceAna(top_k=16, pose=True, align=size, max_frame_hw=BIG)
    res = []
    for img in images:
        fa.reset()
        res.append(fa.run(img))
    return res


def _same_chips(got, want, what):
    """got equals want bit for bit, 'chip' and 'M' included."""
    _same(got, want, what)
    for i, (g, w) in enumerate(zip(got, want)):
        for j, (a, b) in enumerate(zip(g, w)):
            assert a["chip"].dtype == b["chip"].dtype == np.uint8 and a["M"].dtype == b["M"].dtype == np.float64
            assert np.array_equal(a["M"], b["M"]), (what, i, j)
            assert np.array_equal(a["chip"], b["chip"]), (what, i, j, int((a["chip"] != b["chip"]).sum()))


def _from_out_chips(out, n):
    res = _from_out(out, n, True)
    first = out["first"][:n].cpu().numpy()
    chip, M = out["chip"].cpu().numpy(), out["M"].cpu().numpy()
    for o, faces in zip(first.tolist(), res):
        for j, r in enumerate(faces):
            r["chip"], r["M"] = chip[o + j], M[o + j]
    return res


@pytest.mark.parametrize("size", [16, 112, 512])
def test_faceanaimages_align_equals_faceana(images, size):
    from Skps import FaceAnaImages
    want = faceana_align(images, size)
    assert any(len(w) == 0 for w in want) and sum(len(w) for w in want) > 2 * len(images)
    fi = FaceAnaImages(top_k=16, pose=True, align=size)
    _same_chips(fi.run_batch(images), want, ("host", size))
    kinds = sorted(LAYOUTS) if size == 112 else ["pitched"]
    for kind in kinds:
        dev = [LAYOUTS[kind](f) for f in images]
        _same_chips(fi.run_batch(dev), want, (kind, size))
    out = fi.new_results(len(images) + 1)
    assert out["chip"].shape == (16 * (len(images) + 1), size, size, 3) and out["M"].shape == (16 * (len(images) + 1), 2, 3)
    fi.submit(dev, out=out)
    assert fi.collect() is out
    _same_chips(_from_out_chips(out, len(images)), want, ("out", size))
    # two calls in flight: host, host; then CUDA with out= beside host
    a, b = list(range(0, len(images), 2)), list(range(1, len(images), 2))[::-1]
    fi.submit([images[i] for i in a])
    fi.submit([images[i] for i in b])
    ra, rb = fi.collect(), fi.collect()
    _same_chips(ra, [want[i] for i in a], ("first", size))
    _same_chips(rb, [want[i] for i in b], ("second", size))
    o2 = fi.new_results(len(a))
    fi.submit([dev[i] for i in a], out=o2)
    fi.submit([images[i] for i in b])
    assert fi.collect() is o2
    rb = fi.collect()
    _same_chips(_from_out_chips(o2, len(a)), [want[i] for i in a], ("out in flight", size))
    _same_chips(rb, [want[i] for i in b], ("host in flight", size))


def test_without_chips_results_equal_no_align(images):
    from Skps import FaceAnaImages
    plain = FaceAnaImages(top_k=16, pose=True).run_batch(images)
    got = FaceAnaImages(top_k=16, pose=True, align=112).run_batch(images)
    stripped = [[{k: v for k, v in r.items() if k not in ("chip", "M")} for r in g] for g in got]
    _same(stripped, plain, "stripped")
    for g in got:
        for r in g:
            assert set(r) == {"box", "kps", "scores", "pose", "chip", "M"}


def test_facelandmark_align_equals_cv2_and_align_faces(images):
    import torch
    from Skps import FaceAnaImages, FaceLandmark
    from peppa_pig_face_landmark_b200.core.api.align import align_faces
    boxes = [np.stack([r["box"] for r in g]) if g else np.zeros((0, 4), np.float32)
             for g in FaceAnaImages(top_k=16).run_batch(images)]
    # widen some boxes past the image so that their chips read outside it
    boxes = [np.concatenate([b, b[:1] + np.float32([-0.6, -0.6, 0.6, 0.6]) * np.tile(b[:1, 2:] - b[:1, :2], 2)])
             if len(b) else b for b in boxes]
    plain = FaceLandmark(max_faces=32).run_batch(images, boxes)
    for size in (16, 112, 512):
        fl = FaceLandmark(max_faces=32, align=size)
        host = fl.run_batch(images, boxes)
        dev = fl.run_batch([_cuda(f) for f in images], [_cuda(b) for b in boxes])
        devb = fl.run_batch([LAYOUTS["roi"](f) for f in images], boxes)
        for i, f in enumerate(images):
            kps, scores, chips, M = host[i]
            assert np.array_equal(kps, plain[i][0]) and np.array_equal(scores, plain[i][1])
            assert chips.shape == (len(kps), size, size, 3) and chips.dtype == np.uint8 and M.dtype == np.float64
            for other in (dev[i], devb[i]):
                for a, b in zip(other, host[i]):
                    assert np.array_equal(a, b), (size, i)
            for j in range(len(kps)):
                assert np.array_equal(chips[j], cv2_warp(f, M[j], size)), (size, i, j)
            if len(kps):
                ac, aM = align_faces(f, kps.astype(np.float64), size)
                assert np.array_equal(aM, M) and np.array_equal(ac, chips), (size, i)
        assert fl(images[0], boxes[0])[0].shape == plain[0][0].shape           # __call__ returns (kps, scores)
        # out= with CUDA frames
        n = sum(len(b) for b in boxes)
        out = fl.new_results(n)
        fl.submit([_cuda(f) for f in images], boxes, out=out)
        res = fl.collect()
        for i in range(len(images)):
            for a, b in zip(res[i], host[i]):
                assert np.array_equal(a.cpu().numpy(), b), (size, "out", i)
        with pytest.raises(ValueError):
            fl.submit([_cuda(images[0])], [boxes[0]], out={k: v for k, v in out.items() if k != "chip"})
    torch.cuda.synchronize()


def _sources(rects, H, W, d_img, pitch, d_roi, starts):
    from peppa_pig_face_landmark_b200.core.api.face_landmark import FACE_SRC
    n = len(rects)
    whole = np.zeros(n, FACE_SRC)
    whole["base"], whole["pitch"], whole["H"], whole["W"], whole["rw"], whole["rh"] = d_img, pitch, H, W, W, H
    part = whole.copy()
    rw, rh = rects[:, 2] - rects[:, 0], rects[:, 3] - rects[:, 1]
    part["base"], part["pitch"], part["ox"], part["oy"], part["rw"], part["rh"] = d_roi + starts, 3 * rw, rects[:, 0], \
        rects[:, 1], rw, rh
    return whole, part


def test_warp_faces_rectangles_equal_whole_images():
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    from peppa_pig_face_landmark_b200.core.api.align import chip_read_rects
    from test_align_oracle import random_affine
    lib = rt.load_library()
    rng = np.random.default_rng(21)
    H, W, size = 517, 731, 64
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    kinds = [(w, s) for w in ("inside", "partial", "outside") for s in (False, True)]
    Ms = np.stack([random_affine(rng, H, W, size, *kinds[i % len(kinds)]) for i in range(300)])
    rects = chip_read_rects(Ms, size, H, W)
    nb = (rects[:, 2] - rects[:, 0]) * (rects[:, 3] - rects[:, 1]) * 3
    starts = np.concatenate(([0], np.cumsum(nb)[:-1]))
    roi = np.concatenate([img[y0:y1, x0:x1].reshape(-1) for x0, y0, x1, y1 in rects] + [np.zeros(1, np.uint8)])
    d_img, d_roi, d_M = _cuda(img), _cuda(roi), _cuda(Ms)
    whole, part = _sources(rects, H, W, d_img.data_ptr(), 3 * W, d_roi.data_ptr(), starts)
    s = torch.cuda.current_stream().cuda_stream
    outs = []
    for src in (whole, part):
        d_src = _cuda(src.view(np.uint8))
        o = torch.full((len(Ms), size, size, 3), 7, dtype=torch.uint8, device="cuda")
        rt.check(lib.skps_warp_faces(d_src.data_ptr(), d_M.data_ptr(), len(Ms), size, size, o.data_ptr(), s))
        outs.append(o.cpu().numpy())
    assert np.array_equal(outs[0], outs[1])
    for i in range(0, len(Ms), 7):
        assert np.array_equal(outs[0][i], cv2_warp(img, Ms[i], size)), i
    # a rectangle one column too narrow shows up as wrong bytes, not as a read outside it
    thin = part.copy()
    wide = np.flatnonzero((nb > 0) & (rects[:, 2] - rects[:, 0] > 1))[:20]
    thin["rw"][wide] -= 1
    d_src = _cuda(thin.view(np.uint8))
    o = torch.full((len(Ms), size, size, 3), 7, dtype=torch.uint8, device="cuda")
    rt.check(lib.skps_warp_faces(d_src.data_ptr(), d_M.data_ptr(), len(Ms), size, size, o.data_ptr(), s))
    o = o.cpu().numpy()
    assert any(not np.array_equal(o[i], outs[0][i]) for i in wide)
    # more faces than a grid's y dimension holds: 70000 chips of one 16x16 warp each
    n = 70000
    M1 = np.repeat(Ms[:1], n, 0) + np.arange(n)[:, None, None] * np.float64([[0, 0, 1e-3], [0, 0, 0]])
    src = np.repeat(whole[:1], n)
    d_src, d_M1 = _cuda(src.view(np.uint8)), _cuda(M1)
    o = torch.zeros((n, 16, 16, 3), dtype=torch.uint8, device="cuda")
    rt.check(lib.skps_warp_faces(d_src.data_ptr(), d_M1.data_ptr(), n, 16, 16, o.data_ptr(), s))
    o = o.cpu().numpy()
    for i in (0, 65534, 65535, 65536, n - 1):
        assert np.array_equal(o[i], cv2_warp(img, M1[i], 16)), i
    rt.check(lib.skps_warp_faces(None, None, 0, 16, 16, None, s))                  # no faces: nothing to do
    # the estimate from float32 landmarks is skps_align_faces' on the same landmarks promoted to float64
    kps = (rng.uniform(0, 500, (n, 98, 2))).astype(np.float32)
    Me = torch.zeros((n, 2, 3), dtype=torch.float64, device="cuda")
    rt.check(lib.skps_align_estimate(_cuda(kps).data_ptr(), n, 98, 112, Me.data_ptr(), s))
    from peppa_pig_face_landmark_b200.core.api.align import align_faces
    _, want = align_faces(img, kps[:300].astype(np.float64), 112)
    assert np.array_equal(Me[:300].cpu().numpy(), want)
    torch.cuda.synchronize()


def test_host_call_with_align_uploads_less_than_the_images():
    """On sixteen 4K frames with 16 faces, a host call sends the detector's rows, the crop rectangles and the chip
    rectangles: less than the images.  The selected boxes are the oracle's sort_and_filter of the detector's rows."""
    from Skps import FaceAnaImages
    from oracle.host_ref import sort_and_filter
    from peppa_pig_face_landmark_b200.core.api.align import chip_read_rects
    from peppa_pig_face_landmark_b200.core.api.face_detector import host_upload_rows, letterbox_geometry
    from peppa_pig_face_landmark_b200.core.api.face_landmark import crop_read_rects
    imgs = [frames.frame_4k(jitter=(i % 5, -(i % 3))) for i in range(16)]
    fi = FaceAnaImages(top_k=16, align=112)
    res = fi.run_batch(imgs)
    sent = 0
    for img, faces, rows in zip(imgs, res, fi.detector.run_batch(imgs)):
        H, W = img.shape[:2]
        r = host_upload_rows(H, letterbox_geometry(H, W, *fi.detector.input_size[:2])[2])
        sent += (H if r is None else len(r)) * 3 * W
        assert len(faces) == 16
        rect = chip_read_rects(np.stack([f["M"] for f in faces]), 112, H, W)
        sent += int(((rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1]) * 3).sum())
        boxes = np.asarray(sort_and_filter(rows, fi.min_face, fi.top_k), np.float32).reshape(-1, 16)
        crop = crop_read_rects(boxes, H, W, fi.landmark.face_scale)
        sent += int(((crop[:, 2] - crop[:, 0]) * (crop[:, 3] - crop[:, 1]) * 3).sum())
    whole = sum(f.nbytes for f in imgs)
    assert sent < whole, (sent, whole)
