"""CUDA frames in every pixel layout (layout="rgb", "bgra", "rgba", "bgr_planar", "rgb_planar"): every result of every
class equals, bit for bit, the result of the same call on the same pixels as an interleaved BGR (H, W, 3) tensor.  Each
layout is passed packed and as a pitched ROI view (odd byte offset, row pitch above the packed one, planes not H rows
apart).  The ingest kernel is also checked on its own at the widths and heights that reach each of its paths."""
import ctypes as C

import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames
from test_device_frames_gpu import _eq, _same
from test_streams_gpu import _sequences

pytestmark = pytest.mark.gpu

OTHER = ["rgb", "bgra", "rgba", "bgr_planar", "rgb_planar"]
CODES = {"bgr": 0, "rgb": 1, "bgra": 2, "rgba": 3, "bgr_planar": 4, "rgb_planar": 5}


def _channels(f, layout, rng):
    """f (H, W, 3) BGR as the (H, W, C) interleaved or (3, H, W) planar numpy array of `layout`; the 4th channel is noise."""
    rgb = layout.startswith("rgb")
    c = f[..., ::-1] if rgb else f
    if layout in ("bgra", "rgba"):
        a = rng.integers(0, 256, size=f.shape[:2] + (1,), dtype=np.uint8)
        return np.concatenate([c, a], 2)
    if layout.endswith("_planar"):
        return np.ascontiguousarray(c.transpose(2, 0, 1))
    return np.ascontiguousarray(c)


def as_layout(f, layout, kind="packed", seed=0, y0=2, x0=1):
    """f (H, W, 3) BGR numpy -> a CUDA tensor in `layout`.  kind "packed": a contiguous tensor; "roi": a view of a larger
    buffer filled with other bytes, starting at row y0, column x0 (x0 odd: an odd byte offset), rows 5 pixels longer
    than the frame's, and for planar layouts every other plane of a (5, H + 3, W + 5) buffer, so the plane pitch is
    2 (H + 3) (W + 5) bytes, not H times the row pitch."""
    import torch
    if layout == "bgr" and kind == "packed":
        return torch.from_numpy(np.ascontiguousarray(f)).cuda()
    rng = np.random.default_rng(seed)
    a = torch.from_numpy(_channels(f, layout, rng)).cuda()
    if kind == "packed":
        return a
    H, W = f.shape[:2]
    if layout.endswith("_planar"):
        buf = torch.randint(0, 256, (5, H + 3, W + 5), dtype=torch.uint8, device="cuda")
        v = buf[::2, y0:y0 + H, x0:x0 + W]
    else:
        buf = torch.randint(0, 256, (H + 3, W + 5, a.shape[2]), dtype=torch.uint8, device="cuda")
        v = buf[y0:y0 + H, x0:x0 + W]
    v.copy_(a)
    return v


def _bgr(f):
    return as_layout(f, "bgr")


def _golden_frames():
    return {"test1": frames.load_test1(), "video1080": video_frames()[0], "uhd4k": frames.frame_4k()}


# ---------------------------------------------------------------------------------------------------- ingest kernel
@pytest.mark.parametrize("layout", OTHER)
@pytest.mark.parametrize("hw", [(1, 1), (1, 2), (3, 3), (2, 5), (4, 15), (3, 16), (5, 17), (2, 33), (1, 33), (6, 64),
                                (2160, 3840)])
@pytest.mark.parametrize("kind", ["packed", "roi", "roi5"])
def test_ingest_layout_equals_bgr_ingest(layout, hw, kind):
    """skps_frame_ingest_layout: the packed frame and the sum equal skps_frame_ingest's on the BGR frame, byte for byte,
    and nothing past the packed frame is written.  Widths 1..33 reach the 16-pixel vector units, the ragged tails and
    units that cross a row end; roi / roi5 start at byte offsets that are not 16-byte aligned."""
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    H, W = hw
    rng = np.random.default_rng(H * 131 + W)
    f = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)
    p = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)
    src = as_layout(f, layout, "packed" if kind == "packed" else "roi", seed=W, x0=5 if kind == "roi5" else 1)
    planar = layout.endswith("_planar")
    pitch = src.stride(1 if planar else 0) if H > 1 else W * (1 if planar else src.shape[2])
    plane = src.stride(0) if planar else 0
    n = H * W * 3
    packed = torch.full((n + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    want = torch.empty((n + 64,), dtype=torch.uint8, device="cuda")
    prev = _bgr(p).reshape(-1)
    got, ref = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    bgr = _bgr(f)
    rt.check(lib.skps_frame_ingest(bgr.data_ptr(), H, W, 3 * W, want.data_ptr(), prev.data_ptr(), ref.data_ptr(), s))
    rt.check(lib.skps_frame_ingest_layout(src.data_ptr(), H, W, pitch, CODES[layout], plane, packed.data_ptr(),
                                          prev.data_ptr(), got.data_ptr(), s))
    assert torch.equal(packed[:n], want[:n]) and torch.equal(packed[:n], bgr.reshape(-1))
    assert bool((packed[n:] == 0xAB).all())
    assert int(got.item()) == int(ref.item()) == int(np.abs(f.astype(np.int64) - p.astype(np.int64)).sum())
    packed.fill_(0)
    rt.check(lib.skps_frame_ingest_layout(src.data_ptr(), H, W, pitch, CODES[layout], plane, packed.data_ptr(), None,
                                          got.data_ptr(), s))
    assert torch.equal(packed[:n], want[:n]) and int(got.item()) == 0


def test_ingest_layout_refuses_bad_arguments():
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    f = torch.zeros((4, 5, 4), dtype=torch.uint8, device="cuda")
    packed = torch.zeros((64,), dtype=torch.uint8, device="cuda")
    sums = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.skps_frame_ingest_layout(f.data_ptr(), 4, 5, 20, 6, 0, packed.data_ptr(), None, sums.data_ptr(), None)
    assert lib.skps_frame_ingest_layout(f.data_ptr(), 4, 5, 19, 2, 0, packed.data_ptr(), None, sums.data_ptr(), None)
    assert lib.skps_frame_ingest_layout(f.data_ptr(), 4, 5, 5, 4, -1, packed.data_ptr(), None, sums.data_ptr(), None)
    assert lib.skps_frame_ingest_layout(f.data_ptr(), 4, 5, 20, 2, 0, packed.data_ptr(), None, sums.data_ptr(), None) == 0


# ---------------------------------------------------------------------------------------------------- FaceAna
@pytest.mark.parametrize("name", ["test1", "video1080", "uhd4k"])
def test_faceana_golden_frames_in_every_layout(name):
    """A fresh FaceAna on a golden frame in each layout, packed and as an ROI: the same results, chips, pose, ids and
    kept detector rows as on the BGR frame."""
    from Skps import FaceAna
    f = _golden_frames()[name]
    fa = FaceAna(align=112, pose=True, track_ids=True)
    want = fa.run(_bgr(f))
    want_rows, want_idx = fa.last_det_rows.copy(), fa.last_det_idx.copy()
    assert len(want) > 0
    for layout in OTHER:
        for kind in ("packed", "roi"):
            fa.reset()
            got = fa.run(as_layout(f, layout, kind), layout=layout)
            _same(got, want, "%s %s %s" % (name, layout, kind))
            _eq(fa.last_det_rows, want_rows, "%s %s %s det_rows" % (name, layout, kind))
            _eq(fa.last_det_idx, want_idx, "%s %s %s det_idx" % (name, layout, kind))
            assert fa.last_ran_detector


@pytest.mark.parametrize("detect_every", [1, 3])
def test_faceana_sequence_alternating_layouts(detect_every):
    """The golden clip and the 640 canvas clip, every call in another layout (BGR among them), packed and ROI views in
    turn, with align, pose, track ids and detect_every: every result and gate decision equals FaceAna on BGR frames."""
    from Skps import FaceAna
    seqs = _sequences()
    clip = seqs[0] + seqs[2] + seqs[1]
    order = ["bgr"] + OTHER
    kw = dict(align=112, pose=True, track_ids=True, id_memory=2, detect_every=detect_every)
    got_fa, want_fa = FaceAna(**kw), FaceAna(**kw)
    for t, f in enumerate(clip):
        layout, kind = order[t % len(order)], ("roi", "packed")[t % 2]
        got = got_fa.run(as_layout(f, layout, kind, seed=t), layout=layout)
        want = want_fa.run(_bgr(f))
        _same(got, want, "t %d %s %s" % (t, layout, kind))
        assert got_fa.last_ran_detector == want_fa.last_ran_detector, t


# ---------------------------------------------------------------------------------------------------- FaceAnaStreams
def test_streams_layouts_subsets_out_and_two_in_flight():
    """FaceAnaStreams over the _sequences() clips (golden video, 640 canvas, test1) and a 4K clip, one layout per call
    and a new one on every call: full calls and calls on a subset of the streams in any order, host results and out=
    buffers, two calls in flight.  Every entry equals a BGR twin fed the same pixels on the same schedule."""
    import torch
    from Skps import FaceAnaStreams
    seqs = _sequences()
    k0 = frames.frame_4k()
    seqs[3] = [k0, k0, frames.frame_4k(jitter=(8, 4)), k0, k0, k0]
    kw = dict(n_streams=4, align=112, pose=True, track_ids=True, detect_every=2)
    got_fa, want_fa = FaceAnaStreams(**kw), FaceAnaStreams(**kw)
    # (streams, layout, kind, out=) per call; calls 2k and 2k + 1 are in flight together
    plan = [([0, 1, 2, 3], "rgb_planar", "roi", False), ([2, 0], "bgra", "packed", True),
            ([3, 1, 0], "rgb", "roi", True), ([1, 2, 3, 0], "bgr_planar", "packed", False),
            ([0, 3], "rgba", "roi", False), ([2, 1, 3], "bgr", "roi", True),
            ([3, 2, 1, 0], "rgb_planar", "packed", True), ([1, 0, 2], "bgra", "roi", False)]
    pos = [0, 0, 0, 0]
    gbufs = [got_fa.new_results(), got_fa.new_results()]
    wbufs = [want_fa.new_results(), want_fa.new_results()]
    for c0 in range(0, len(plan), 2):
        pending = []
        for j, (streams, layout, kind, dev_out) in enumerate(plan[c0:c0 + 2]):
            fs = [seqs[s][pos[s] % 6] for s in streams]
            for s in streams:
                pos[s] += 1
            got_fa.submit([as_layout(f, layout, kind, seed=c0 + j) for f in fs], out=gbufs[j] if dev_out else None,
                          streams=streams, layout=layout)
            want_fa.submit([_bgr(f) for f in fs], out=wbufs[j] if dev_out else None, streams=streams)
            pending.append((c0 + j, len(streams), dev_out))
        for c, n, dev_out in pending:
            got, want = got_fa.collect(), want_fa.collect()
            if dev_out:
                torch.cuda.synchronize()
                for k in want:
                    assert torch.equal(got[k][:n], want[k][:n]), (c, k)
            else:
                for i in range(n):
                    _same(got[i], want[i], "call %d entry %d" % (c, i))
                assert list(got_fa.last_ran_detector) == list(want_fa.last_ran_detector), c


def test_streams_refuse_bad_layouts_before_enqueueing():
    from Skps import FaceAnaStreams
    fa = FaceAnaStreams(n_streams=2)
    f = frames.canvas_640()
    for frame, layout in [(as_layout(f, "bgr"), "bgr_planar"), (as_layout(f, "rgb_planar"), "rgb"),
                          (as_layout(f, "bgra"), "rgb"), (as_layout(f, "rgb"), "yuv"), (f, "rgb")]:
        with pytest.raises(ValueError):
            fa.submit([frame], layout=layout)
        assert not fa._pending
    # nothing was counted: the first accepted frame is each stream's first
    got = fa.run([as_layout(f, "rgb_planar")], layout="rgb_planar")
    _same(got[0], FaceAnaStreams(n_streams=1).run([f])[0], "after refusals")


# ---------------------------------------------------------------------------------------------------- batch classes
def test_detector_rows_and_kept_indices_in_every_layout():
    import torch
    from Skps import FaceDetector
    fs = list(_golden_frames().values())
    fd = FaceDetector(max_frames=2)
    want = fd.run_batch([_bgr(f) for f in fs])
    want_idx = fd.last_keep_idx
    wbuf = fd.new_results(len(fs))
    fd.submit([_bgr(f) for f in fs], out=wbuf)
    fd.collect()
    for layout in OTHER:
        for kind in ("packed", "roi"):
            got = fd.run_batch([as_layout(f, layout, kind) for f in fs], layout=layout)
            for i in range(len(fs)):
                _eq(got[i], want[i], "%s %s rows %d" % (layout, kind, i))
                _eq(fd.last_keep_idx[i], want_idx[i], "%s %s idx %d" % (layout, kind, i))
        buf = fd.new_results(len(fs))
        fd.submit([as_layout(f, layout, "roi") for f in fs], out=buf, layout=layout)
        fd.collect()
        torch.cuda.synchronize()
        for i, k in enumerate(wbuf["count"].tolist()):
            assert int(buf["count"][i]) == k
            assert torch.equal(buf["rows"][i, :k], wbuf["rows"][i, :k]) and torch.equal(buf["idx"][i, :k], wbuf["idx"][i, :k])


def test_landmark_align_cuda_boxes_and_out_in_every_layout():
    import torch
    from Skps import FaceDetector, FaceLandmark
    fs = list(_golden_frames().values())
    boxes = [torch.from_numpy(np.ascontiguousarray(b[:, :4])).cuda() for b in FaceDetector().run_batch(fs)]
    fl = FaceLandmark(max_faces=8, align=112)
    n = sum(int(b.shape[0]) for b in boxes)
    want = fl.new_results(n)
    fl.submit([_bgr(f) for f in fs], boxes, out=want)
    fl.collect()
    want_host = fl.run_batch([_bgr(f) for f in fs], [b.cpu().numpy() for b in boxes])
    for layout in OTHER:
        for kind in ("packed", "roi"):
            got = fl.new_results(n)
            fl.submit([as_layout(f, layout, kind) for f in fs], boxes, out=got, layout=layout)
            fl.collect()
            torch.cuda.synchronize()
            for k in want:
                assert torch.equal(got[k][:n], want[k][:n]), (layout, kind, k)
        host = fl.run_batch([as_layout(f, layout, "roi") for f in fs], [b.cpu().numpy() for b in boxes], layout=layout)
        for i, (g, w) in enumerate(zip(host, want_host)):
            for a, b in zip(g, w):
                _eq(a, b, "%s host results frame %d" % (layout, i))


def test_images_align_pose_in_every_layout():
    from Skps import FaceAnaImages
    fs = list(_golden_frames().values())
    fi = FaceAnaImages(align=112, pose=True, max_frames=2)
    want = fi.run_batch([_bgr(f) for f in fs])
    assert all(len(w) for w in want)
    for layout in OTHER:
        for kind in ("packed", "roi"):
            got = fi.run_batch([as_layout(f, layout, kind) for f in fs], layout=layout)
            for i in range(len(fs)):
                _same(got[i], want[i], "%s %s image %d" % (layout, kind, i))
