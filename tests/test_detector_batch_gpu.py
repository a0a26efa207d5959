"""FaceDetector over many frames per call (run_batch, submit / collect, out=) and its letterbox skps_letterbox_frames.  The
reference for every comparison is a per-frame restatement of what FaceDetector.__call__ did before it ran on the batched
path: the whole frame uploaded, skps_letterbox, a batch-1 engine and skps_detect_post_batch.  Every comparison with it is
exact; the kept indices are also checked against the CPU oracle."""
import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames
from test_crowd_cpu import crowd_frame
from test_crowd_gpu import _same_kept_as_oracle
from test_detector_input_gpu import _detector_ref
from test_landmark_batch_gpu import LAYOUTS, _cuda, _roi

pytestmark = pytest.mark.gpu


def _lib():
    from peppa_pig_face_landmark_b200 import runtime as rt
    return rt, rt.load_library()


def _cfg(hw):
    from peppa_pig_face_landmark_b200.core.api.facer import get_cfg
    cfg = get_cfg()['Skps']['Detect']
    cfg['input_shape'] = [hw[0], hw[1], 3]
    return cfg


class Restated:
    """FaceDetector(cfg)(frame) as it was computed before the batched path."""

    def __init__(self, hw):
        import torch
        from peppa_pig_face_landmark_b200 import ONNXEngine
        from peppa_pig_face_landmark_b200.core.api import face_detector as fd
        from peppa_pig_face_landmark_b200.graph_tools import detector_onnx_for
        rt, lib = _lib()
        cfg = _cfg(hw)
        path = fd.pathlib.Path(fd.__file__).resolve().parents[2] / cfg['model_path']
        self.hw, self.cfg, self.lib, self.rt = hw, cfg, lib, rt
        self.eng = ONNXEngine(detector_onnx_for(str(path), hw), max_batch=1)
        self.R = self.eng.out_elems[0] // 16
        self.kept = torch.zeros((self.R, 16), dtype=torch.float32, device="cuda")
        self.idx = torch.zeros((self.R,), dtype=torch.int32, device="cuda")
        self.count = torch.zeros((1,), dtype=torch.int32, device="cuda")
        self.ws_bytes = lib.skps_detect_post_workspace_size(self.R, 1)
        self.ws = torch.empty((self.ws_bytes,), dtype=torch.uint8, device="cuda")

    def __call__(self, image):
        import torch
        from peppa_pig_face_landmark_b200.core.api.face_detector import letterbox_geometry
        rt, lib = self.rt, self.lib
        h, w = image.shape[:2]
        frame = torch.from_numpy(np.ascontiguousarray(image)).cuda()
        scale, rw, rh, top, left = letterbox_geometry(h, w, *self.hw)
        s = torch.cuda.current_stream().cuda_stream
        rt.check(lib.skps_letterbox(frame.data_ptr(), h, w, w * 3, self.eng.input_ptr(), self.hw[0], self.hw[1],
                                    rw, rh, top, left, s))
        rt.check(lib.skps_engine_forward(self.eng.handle, self.eng.input_ptr(), 1, None, s))
        rec = torch.tensor([scale, float(left), float(top)], dtype=torch.float32).cuda()
        rt.check(lib.skps_detect_post_batch(self.eng.output_ptr(0), self.R, 1, self.cfg['score_thrs'],
                                            self.cfg['iou_thrs'], rec.data_ptr(), self.kept.data_ptr(),
                                            self.idx.data_ptr(), self.count.data_ptr(), self.R, self.ws.data_ptr(),
                                            self.ws_bytes, s))
        torch.cuda.synchronize()
        n = int(self.count.item())
        return self.kept[:n].cpu().numpy(), self.idx[:n].cpu().numpy().astype(np.int64)


def _same(got, keep, want, what=""):
    assert len(got) == len(keep) == len(want), (what, len(got), len(want))
    for i, (rows, idx, (wr, wi)) in enumerate(zip(got, keep, want)):
        assert rows.dtype == np.float32 and rows.shape == wr.shape, (what, i, rows.shape, wr.shape)
        assert idx.dtype == np.int64 and np.array_equal(idx, wi), (what, i)
        assert np.array_equal(rows, wr), (what, i)


def _from_out(out, n):
    cnt = out["count"][:n].cpu().numpy()
    rows = [out["rows"][i, :k].cpu().numpy() for i, k in enumerate(cnt)]
    idx = [out["idx"][i, :k].cpu().numpy().astype(np.int64) for i, k in enumerate(cnt)]
    return rows, idx


def still_4000x3000():
    return frames.multi_face_frame(3000, 4000, (2, 3), 560)


def portrait():
    return frames.multi_face_frame(1920, 1080, (3, 1), 420)


def mixed_frames():
    """test1, canvas640, the 1080p clip (one frame without a face), uhd4k_top16, a 4000x3000 still, a portrait frame and
    a 96-face crowd: twelve frames of eight sizes in one call."""
    return ([frames.load_test1(), frames.canvas_640()] + video_frames() +
            [frames.frame_4k(), still_4000x3000(), portrait(), crowd_frame("crowd96_768x1280")])


@pytest.fixture(scope="module")
def mixed():
    return mixed_frames()


@pytest.fixture(scope="module")
def fd():
    from Skps import FaceDetector
    return FaceDetector()


@pytest.fixture(scope="module")
def want(mixed):
    ref = Restated((384, 640))
    return [ref(f) for f in mixed]


@pytest.mark.parametrize("hw", [(384, 640), (768, 1280)], ids=lambda hw: "%dx%d" % hw)
def test_run_batch_equals_the_parent_call(fd, mixed, want, hw):
    from Skps import FaceDetector
    det = fd if hw == (384, 640) else FaceDetector(_cfg(hw))
    w = want if hw == (384, 640) else [Restated(hw)(f) for f in mixed]
    got = det.run_batch(mixed)
    _same(got, det.last_keep_idx, w, hw)
    assert any(len(r) == 0 for r in got) and sum(len(r) > 0 for r in got) >= 8
    for i, f in enumerate(mixed):                                          # __call__, one frame at a time
        rows = det(f)
        _same([rows], [det.last_keep_idx], [w[i]], (hw, "call", i))


def test_kept_indices_equal_the_oracle(fd, mixed, want):
    """The golden frames keep exactly the oracle's rows (test_parity_gpu's rule); the others the same rows up to
    near-equal scores swapping (test_crowd_gpu's rule)."""
    ref = _detector_ref((384, 640))
    for i, f in enumerate(mixed):
        w_rows, w_idx = ref(f, return_indices=True)
        rows, idx = want[i]
        if i < 2 + 6 + 1:                                                  # test1, canvas640, the clip, uhd4k
            assert np.array_equal(idx, w_idx), i
        else:
            _same_kept_as_oracle(idx, rows, w_idx, w_rows, i)


def test_crowd_beyond_max_det():
    """A 384-face crowd keeps more rows than come back with the counts: the rest are fetched for that frame only."""
    from Skps import FaceDetector
    hw = (1152, 1920)
    det, ref = FaceDetector(_cfg(hw), max_frames=4), Restated(hw)
    fs = [frames.load_test1(), crowd_frame("crowd384_1152x1920"), frames.frame_4k(), crowd_frame("crowd192_1152x1920")]
    w = [ref(f) for f in fs]
    assert len(w[1][1]) == 384 > det.MAX_DET
    _same(det.run_batch(fs), det.last_keep_idx, w, "host")
    _same(det.run_batch([_cuda(f) for f in fs]), det.last_keep_idx, w, "cuda")
    out = det.new_results(4)
    det.submit([_roi(f) for f in fs], out=out)
    assert det.collect() is out
    rows, idx = _from_out(out, 4)
    _same(rows, idx, w, "out")


def test_letterbox_frames_equal_letterbox():
    """skps_letterbox_frames writes, frame for frame, the bytes skps_letterbox writes on the whole frame: with every
    frame in row pairs, and with every frame read in place (packed, pitched and odd-offset views), in one launch."""
    import torch
    from peppa_pig_face_landmark_b200.core.api.face_detector import DET_SRC, letterbox_geometry, letterbox_rows
    rt, lib = _lib()
    rng = np.random.default_rng(9)
    imgs = [frames.load_test1(), frames.frame_4k(), still_4000x3000(), portrait()]
    imgs += [rng.integers(0, 256, hw + (3,), dtype=np.uint8) for hw in [(723, 1281), (2000, 900), (37, 23), (1, 1),
                                                                         (1080, 1921), (3001, 4003)]]
    s = torch.cuda.current_stream().cuda_stream
    for hw in [(384, 640), (1152, 1920)]:
        geo, want = [], []
        for img in imgs:
            H, W = img.shape[:2]
            try:
                g = letterbox_geometry(H, W, *hw)
            except ValueError:
                continue
            geo.append((img, g))
            out = torch.full(hw + (3,), 7, dtype=torch.uint8, device="cuda")
            fr = _cuda(img)
            _, rw, rh, top, left = g
            rt.check(lib.skps_letterbox(fr.data_ptr(), H, W, 3 * W, out.data_ptr(), hw[0], hw[1], rw, rh, top, left, s))
            want.append(out.cpu().numpy())
        assert len(geo) >= 7
        for form in ["pairs"] + sorted(LAYOUTS):
            keep = []
            desc = np.zeros(len(geo), DET_SRC)
            for i, (img, (_, rw, rh, top, left)) in enumerate(geo):
                H, W = img.shape[:2]
                if form == "pairs":
                    t = _cuda(img[letterbox_rows(H, rh)])
                    pitch = 3 * W
                else:
                    t = LAYOUTS[form](img)
                    pitch = t.stride(0) if H > 1 else 3 * W
                keep.append(t)
                desc[i] = (t.data_ptr(), pitch, H, W, rw, rh, top, left, int(form == "pairs"))
            d_desc = _cuda(desc.view(np.uint8))
            out = torch.full((len(geo),) + hw + (3,), 7, dtype=torch.uint8, device="cuda")
            rt.check(lib.skps_letterbox_frames(d_desc.data_ptr(), len(geo), out.data_ptr(), hw[0], hw[1], s))
            got = out.cpu().numpy()
            for i in range(len(geo)):
                assert np.array_equal(got[i], want[i]), (hw, form, i)
    rt.check(lib.skps_letterbox_frames(None, 0, None, 384, 640, s))                 # no frames: nothing to do


@pytest.mark.parametrize("kind", sorted(LAYOUTS))
def test_cuda_frames_equal_host_frames(fd, mixed, want, kind):
    dev = [LAYOUTS[kind](f) for f in mixed]
    _same(fd.run_batch(dev), fd.last_keep_idx, want, kind)
    out = fd.new_results(len(mixed) + 3)
    fd.submit(dev, out=out)
    res = fd.collect()
    assert res is out
    rows, idx = _from_out(out, len(mixed))
    _same(rows, idx, want, kind + " out")


def test_chunks_and_position_in_a_batch(mixed, want):
    """max_frames 4: twelve frames run in three chunks.  With max_frames 16, a frame gives the same rows alone and at
    position 7 of a batch of 16."""
    from Skps import FaceDetector
    small = FaceDetector(max_frames=4)
    _same(small.run_batch(mixed), small.last_keep_idx, want, "chunks")
    _same(small.run_batch([_cuda(f) for f in mixed]), small.last_keep_idx, want, "cuda chunks")
    big = FaceDetector(max_frames=16)
    order = [(i * 5) % len(mixed) for i in range(16)]
    for target in (0, 9, 10):
        batch = [mixed[j] for j in order]
        batch[7] = mixed[target]
        got = big.run_batch(batch)
        keep = big.last_keep_idx
        alone = big.run_batch([mixed[target]])
        assert np.array_equal(got[7], alone[0]) and np.array_equal(got[7], want[target][0]), target
    _same(got, keep, [want[10] if k == 7 else want[j] for k, j in enumerate(order)], "16")


def test_calls_in_flight_keep_their_staging(fd, mixed, want):
    """The first call is held back behind a sleeping producer stream; the third call reuses the first call's staging
    slot while it is pending.  Host frames: the third call's rows go into the first call's pinned staging."""
    import torch
    dev = [_cuda(f) for f in mixed]
    n = len(mixed)
    order = [list(range(n)), list(range(n))[::-1], [2, 0, 1, 3]]
    bufs = [fd.new_results(n) for _ in range(3)]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        fd.submit([dev[i] for i in order[0]], out=bufs[0])
    fd.submit([dev[i] for i in order[1]], out=bufs[1])
    fd.collect()
    fd.submit([dev[i] for i in order[2]], out=bufs[2])
    fd.collect()
    fd.collect()
    torch.cuda.synchronize()
    for t in range(3):
        rows, idx = _from_out(bufs[t], len(order[t]))
        _same(rows, idx, [want[i] for i in order[t]], "call %d" % t)
    fd.submit(mixed)
    fd.submit(mixed[:3])
    r0, k0 = fd.collect(), fd.last_keep_idx
    fd.submit(mixed[3:])
    _same(r0, k0, want, "host 0")
    _same(fd.collect(), fd.last_keep_idx, want[:3], "host 1")
    _same(fd.collect(), fd.last_keep_idx, want[3:], "host 2")


def test_frames_are_read_after_the_producer_stream(fd):
    """The frame is written on a side stream behind a sleep and submitted under it: without the wait on the producer's
    stream the letterbox would read the blank frame."""
    import torch
    f = frames.frame_1080p()
    w = [Restated((384, 640))(f)]
    src = _cuda(f)
    frame = torch.zeros_like(src)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        frame.copy_(src)
        got = fd.run_batch([frame])
    _same(got, fd.last_keep_idx, w)
    assert len(w[0][0]) == 4
    torch.cuda.synchronize()


def test_producer_may_overwrite_the_frame_once_submit_returns(fd):
    """Right after submit the caller zeroes the frame on its stream.  The detector stream is held back (a first call
    waits on a sleeping side stream), so without the wait for the read the zeroing would land first."""
    import torch
    f0, f1 = frames.frame_1080p(), frames.frame_1080p(jitter=(8, -4))
    ref = Restated((384, 640))
    w0, w1 = [ref(f0)], [ref(f1)]
    a, c = _cuda(f0), _cuda(f1)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        fd.submit([a])
    fd.submit([c])
    c.zero_()
    _same(fd.collect(), fd.last_keep_idx, w0, "call 0")
    _same(fd.collect(), fd.last_keep_idx, w1, "call 1")


def test_invalid_inputs_raise_before_anything_is_enqueued(fd):
    import torch
    f = frames.load_test1()
    good = _cuda(f)
    planar = _cuda(np.ascontiguousarray(f.transpose(2, 0, 1))).permute(1, 2, 0)
    bad_calls = [
        [f, good],                                                   # host and CUDA frames
        [f.astype(np.float32)], [f[:, :, :2]], [f[0]], [f, f[:, :, :2]],
        [good.float()], [planar], [good[0]], [good, torch.from_numpy(f)],
        [np.zeros((1, 4000, 3), np.uint8)],                          # a letterbox with no rows
        [f, np.zeros((4000, 1, 3), np.uint8)], [_cuda(np.zeros((1, 4000, 3), np.uint8))],
    ]
    for i, fs in enumerate(bad_calls):
        with pytest.raises(ValueError):
            fd.submit(fs)
        assert not fd._pending, i
    with pytest.raises(ValueError):
        fd.submit([f], out=fd.new_results(1))                        # out= takes CUDA frames
    res = fd.new_results(2)
    for bent in ({"rows": res["rows"], "idx": res["idx"]}, {k: v[:0] for k, v in res.items()},
                 dict(res, rows=res["rows"].double()), dict(res, idx=res["idx"].cpu()),
                 dict(res, rows=res["rows"][:, :100]), dict(res, count=res["count"].long())):
        with pytest.raises(ValueError):
            fd.submit([good, good], out=bent)
    with pytest.raises(ValueError):
        fd.submit([good, good, good], out=res)                       # too small
    assert not fd._pending
    fd.submit([good], out=res)
    with pytest.raises(ValueError):
        fd.submit([good], out=res)                                   # still in flight
    fd.submit([f])
    with pytest.raises(RuntimeError):
        fd.submit([f])                                               # a third call
    with pytest.raises(RuntimeError):
        fd.run_batch([f])
    assert len(fd._pending) == 2
    w = [Restated((384, 640))(f)]
    assert fd.collect() is res
    rows, idx = _from_out(res, 1)
    _same(rows, idx, w)
    _same(fd.collect(), fd.last_keep_idx, w)
    assert fd.run_batch([]) == [] and fd.last_keep_idx == []
