"""Frames already in GPU memory (torch.uint8 CUDA tensors of any row pitch) in FaceAna.run and FaceAnaStreams.submit, and
FaceAnaStreams results left on the GPU (submit(out=...)).  The same kernels run on the same bytes as for numpy frames, so
every comparison is exact."""
import ctypes as C

import numpy as np
import pytest

import frames
from golden.make_golden_frames import video_frames
from test_streams_gpu import _sequences

pytestmark = pytest.mark.gpu


def _eq(x, y, what):
    if isinstance(x, dict):
        assert set(x) == set(y), (what, set(x) ^ set(y))
        for k in x:
            _eq(x[k], y[k], "%s.%s" % (what, k))
        return
    x, y = np.asarray(x), np.asarray(y)
    assert x.dtype == y.dtype and x.shape == y.shape, (what, x.dtype, y.dtype, x.shape, y.shape)
    np.testing.assert_array_equal(x, y, err_msg=what)


def _same(a, b, what=""):
    assert len(a) == len(b), (what, len(a), len(b))
    for i, (x, y) in enumerate(zip(a, b)):
        _eq(x, y, "%s face %d" % (what, i))


def _cuda(f):
    import torch
    return torch.from_numpy(np.ascontiguousarray(f)).cuda()


def _pitched(f):
    """f as a view of a wider buffer: rows 3 (W + pad) bytes apart, not a multiple of 16."""
    import torch
    H, W = f.shape[:2]
    pad = next(p for p in range(1, 16) if (3 * (W + p)) % 16)
    buf = torch.full((H, W + pad, 3), 201, dtype=torch.uint8, device="cuda")
    buf[:, :W] = _cuda(f)
    v = buf[:, :W]
    assert v.stride(0) == 3 * (W + pad) and v.stride(0) % 16
    return v


def _roi(f):
    """f as big[y0:y1, x0:x1] of a larger frame: the view starts at an odd byte offset."""
    import torch
    H, W = f.shape[:2]
    buf = torch.full((H + 3, W + 4, 3), 37, dtype=torch.uint8, device="cuda")
    buf[2:2 + H, 1:1 + W] = _cuda(f)
    v = buf[2:2 + H, 1:1 + W]
    assert (v.storage_offset() % 2) == 1 and v.stride(0) == 3 * (W + 4)
    return v


LAYOUTS = {"packed": _cuda, "pitched": _pitched, "roi": _roi}


def test_faceana_cuda_frames_equal_numpy_frames():
    """The golden clip (detect, two static frames the gate skips, a moved frame, two empty frames) as CUDA tensors, with
    chips and pose: every result equals FaceAna on the numpy frames, and so do the kept detector rows."""
    from Skps import FaceAna
    v = video_frames()
    dev, host = FaceAna(align=112, pose=True), FaceAna(align=112, pose=True)
    kinds = ["packed", "roi", "pitched", "packed", "roi", "pitched"]
    for t, (f, kind) in enumerate(zip(v, kinds)):
        got = dev.run(LAYOUTS[kind](f))
        want = host.run(f)
        _same(got, want, "frame %d (%s)" % (t, kind))
        _eq(dev.last_det_idx, host.last_det_idx, "frame %d det_idx" % t)
        _eq(dev.last_det_rows, host.last_det_rows, "frame %d det_rows" % t)


def _four_layouts():
    """_sequences() of test_streams_gpu with its last clip replaced by a 4K one (16 faces, a static frame, a moved one)."""
    seqs = _sequences()
    k0 = frames.frame_4k()
    k1 = k0.copy()
    k1[::11, ::3] = np.clip(k1[::11, ::3].astype(np.int16) - 2, 0, 255).astype(np.uint8)
    k2 = frames.frame_4k(jitter=(8, 4))
    seqs[3] = [k0, k1, k1, k2, k0, k2]
    return seqs, ["packed", "pitched", "roi", "packed"]


def test_streams_cuda_frame_layouts_equal_numpy_frames():
    from Skps import FaceAnaStreams
    seqs, kinds = _four_layouts()
    dev, host = FaceAnaStreams(n_streams=4), FaceAnaStreams(n_streams=4)
    for t in range(6):
        got = dev.run([LAYOUTS[k](s[t]) for s, k in zip(seqs, kinds)])
        want = host.run([s[t] for s in seqs])
        for i in range(4):
            _same(got[i], want[i], "t %d stream %d (%s)" % (t, i, kinds[i]))
        assert list(dev.last_ran_detector) == list(host.last_ran_detector)


@pytest.mark.parametrize("hw", [(5, 1), (7, 13), (33, 101), (2160, 3840)])
@pytest.mark.parametrize("kind", ["packed", "pitched", "roi"])
def test_ingest_gathers_and_diffs_exactly(hw, kind):
    """skps_frame_ingest: the packed frame equals frame.contiguous() byte for byte, nothing past it is written, and the sum
    equals skps_frame_absdiff_sum of the packed copies (and numpy's)."""
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    H, W = hw
    rng = np.random.default_rng(H * 7 + W)
    f = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)
    p = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)
    src = LAYOUTS[kind](f)
    pitch = src.stride(0) if H > 1 else 3 * W
    n = H * W * 3
    packed = torch.full((n + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    prev = _cuda(p).reshape(-1)
    got, ref = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rt.check(lib.skps_frame_ingest(src.data_ptr(), H, W, pitch, packed.data_ptr(), prev.data_ptr(), got.data_ptr(), s))
    want = src.contiguous().reshape(-1)
    rt.check(lib.skps_frame_absdiff_sum(prev.data_ptr(), want.data_ptr(), n, ref.data_ptr(), s))
    assert torch.equal(packed[:n], want)
    assert bool((packed[n:] == 0xAB).all())
    assert int(got.item()) == int(ref.item()) == int(np.abs(f.astype(np.int64) - p.astype(np.int64)).sum())
    # no previous frame: copy only
    packed.fill_(0)
    rt.check(lib.skps_frame_ingest(src.data_ptr(), H, W, pitch, packed.data_ptr(), None, got.data_ptr(), s))
    assert torch.equal(packed[:n], want) and int(got.item()) == 0


def test_frame_is_read_after_the_producer_stream():
    """The frame is written on a side stream behind a sleep and submitted under that stream: without the wait on the
    producer's stream the pipeline would read the stale (blank) bytes and find no face."""
    import torch
    from Skps import FaceAna, FaceAnaStreams
    f = frames.frame_1080p()
    want_streams = FaceAnaStreams(n_streams=1).run([f])
    want_single = FaceAna().run(f)
    assert len(want_single) > 0
    fa_s, fa_1 = FaceAnaStreams(n_streams=1), FaceAna()
    src = _cuda(f)
    for run, want in ((lambda x: fa_s.run([x])[0], want_streams[0]), (fa_1.run, want_single)):
        frame = torch.zeros_like(src)
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(100_000_000)
            frame.copy_(src)
            got = run(frame)
        _same(got, want)
        torch.cuda.synchronize()


def test_producer_may_overwrite_the_frame_once_submit_returns():
    """Right after submit the caller zeroes the frame on its stream.  The pipeline's stream is held back (a first batch
    waits on a sleeping side stream), so without the wait for the read the zeroing would land first."""
    import torch
    from Skps import FaceAnaStreams
    f0, f1 = frames.frame_1080p(), frames.frame_1080p(jitter=(8, -4))
    host = FaceAnaStreams(n_streams=1)
    want = [host.run([f0])[0], host.run([f1])[0]]
    dev = FaceAnaStreams(n_streams=1)
    a, b = _cuda(f0), _cuda(f1)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        dev.submit([a])
    dev.submit([b])
    b.zero_()
    _same(dev.collect()[0], want[0], "batch 0")
    _same(dev.collect()[0], want[1], "batch 1")


def _lists(snap, n, align, pose):
    """A device result dict (copied to the host) in collect()'s list-of-dicts form."""
    res = []
    for s in range(n):
        faces = []
        for i in range(int(snap["n"][s])):
            r = {"box": snap["box"][s, i], "kps": snap["kps"][s, i], "scores": snap["scores"][s, i]}
            if align:
                r["chip"], r["M"] = snap["chip"][s, i], snap["M"][s, i]
            if pose:
                r["pose"] = {k: snap[k][s, i] for k in ("rvec", "tvec", "euler", "reproject")}
            faces.append(r)
        res.append(faces)
    return res


def test_device_results_equal_host_results():
    """Two batches in flight with out= buffers and host-result batches in between: every field, chips and pose included,
    equals what collect() returns on the host for a twin object fed the numpy frames."""
    import torch
    from Skps import FaceAnaStreams
    seqs, kinds = _four_layouts()
    S = len(seqs)
    dev = FaceAnaStreams(n_streams=S, align=112, pose=True)
    host = FaceAnaStreams(n_streams=S, align=112, pose=True)
    want = [host.run([s[t] for s in seqs]) for t in range(6)]
    modes = ["dev", "dev", "host", "dev", "host", "dev"]
    bufs = [dev.new_results(), dev.new_results()]
    free = [0, 1]
    pending, got = [], []

    def submit(t):
        batch = [LAYOUTS[k](s[t]) for s, k in zip(seqs, kinds)]
        if modes[t] == "dev":
            i = free.pop(0)
            dev.submit(batch, out=bufs[i])
            pending.append(i)
        else:
            dev.submit(batch)
            pending.append(None)

    def collect():
        i = pending.pop(0)
        r = dev.collect()
        if i is None:
            got.append(r)
            return
        assert r is bufs[i]
        snap = {k: v.cpu().numpy() for k, v in r.items()}         # on the current stream, which now waits for the batch
        got.append(_lists(snap, S, True, True))
        free.append(i)

    submit(0)
    for t in range(1, 6):
        submit(t)
        collect()
    collect()
    for t in range(6):
        for s in range(S):
            _same(got[t][s], want[t][s], "t %d stream %d (%s results)" % (t, s, modes[t]))


def test_invalid_inputs_raise_before_anything_is_enqueued():
    import torch
    from Skps import FaceAna, FaceAnaStreams
    f = frames.canvas_640()
    good = _cuda(f)
    fa = FaceAnaStreams(n_streams=2)
    one = FaceAna()
    planar = _cuda(np.ascontiguousarray(f.transpose(2, 0, 1))).permute(1, 2, 0)     # CHW storage seen as HWC
    oversize = torch.zeros((2161, 3840, 3), dtype=torch.uint8, device="cuda")
    bad = {"dtype": good.float(), "planar": planar, "oversize": oversize, "rank": good[0], "channels": good[:, :, :2]}
    for name, x in bad.items():
        with pytest.raises(ValueError):
            fa.submit([good, x])
        with pytest.raises(ValueError):
            one.run(x)
        assert not fa._pending, name
    with pytest.raises(ValueError):
        fa.submit([good, torch.from_numpy(f)])                  # a CPU tensor in a CUDA batch
    with pytest.raises(ValueError):
        fa.submit([good, f])                                    # host and CUDA frames mixed
    with pytest.raises(ValueError):
        fa.submit([f, f], out=fa.new_results())                 # device results take CUDA frames
    res = fa.new_results()
    for k, t in [("box", torch.zeros((2, 5, 3), dtype=torch.float64, device="cuda")),
                 ("kps", res["kps"].float()), ("scores", res["scores"].cpu()), ("n", res["n"][:1])]:
        bent = dict(res)
        bent[k] = t
        with pytest.raises(ValueError):
            fa.submit([good, good], out=bent)
    with pytest.raises(ValueError):
        fa.submit([good, good], out={k: v for k, v in res.items() if k != "scores"})
    assert not fa._pending
    fa.submit([good, good], out=res)
    with pytest.raises(ValueError):
        fa.submit([good, good], out=res)                        # still in flight
    assert len(fa._pending) == 1
    r = fa.collect()
    assert r is res
    want = FaceAnaStreams(n_streams=2).run([f, f])
    _same(_lists({k: v.cpu().numpy() for k, v in r.items()}, 2, False, False)[0], want[0])


def test_frame_on_another_device_raises():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    from Skps import FaceAna, FaceAnaStreams
    x = torch.zeros((64, 64, 3), dtype=torch.uint8, device="cuda:1")
    with torch.cuda.device(0):
        fa, one = FaceAnaStreams(n_streams=1, device="cuda:0"), FaceAna()
    with pytest.raises(ValueError):
        fa.submit([x])
    with pytest.raises(ValueError):
        one.run(x)
