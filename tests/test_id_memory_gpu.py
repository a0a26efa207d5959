"""Id memory on the GPU.  The device rule (mp_temporal_kernel through skps_debug_mp_temporal_mem) on scripted and random
sequences of up to 256 streams, ids, memory contents and next ids checked against the restatement of
test_id_memory_cpu after every launch; with the memory off, the launch is skps_debug_mp_temporal's byte for byte.  End to
end, a face covered for 1, 2 or 3 frames gets its id back exactly when the gap is at most id_memory, nothing but 'id'
changes, the ids equal the restatement fed from the detector's kept rows, and every stream of FaceAnaStreams gives the ids
of its own FaceAna."""
import ctypes as C

import numpy as np
import pytest

import frames
import test_temporal_kernel_gpu as T
from test_id_memory_cpu import _Restated
from test_track_ids_gpu import ALPHA, IOU, MIN_FACE, _bright

pytestmark = pytest.mark.gpu

P, F32 = T.P, np.float32


# ----------------------------------------------------------------------------- the kernel
class _MemHost(T._Host):
    """One stream of the host layer whose ids follow the restated memory rule instead of assign_track_ids."""

    def __init__(self, m, K, oracle=False):
        super().__init__(oracle)
        self.rule = _Restated(m, K)

    def judge(self, boxes4, tmp_box, src):
        super().judge(boxes4, tmp_box, src)
        n = len(boxes4)
        returned = np.asarray(self.track_box, np.float64).reshape(-1, 4).astype(F32) if n else np.zeros((0, 4), F32)
        self.ids = self.rule.call([int(s) for s in src][:n], boxes4, returned)
        self.next_id = self.rule.next_id


class _MemDevice(T._Device):
    """The state of S streams plus their id memory, launched through skps_debug_mp_temporal_mem (or, legacy=True, through
    skps_debug_mp_temporal)."""

    def __init__(self, S, K, m, legacy=False, null=False):
        super().__init__(S, K)
        torch = self.torch
        self.m, self.legacy, self.null = m, legacy, null
        z = lambda *shape, dt: torch.zeros(shape, dtype=dt, device="cuda")        # noqa: E731
        self.mem = dict(mem_ids=z(S, K, dt=torch.int64) - 7, mem_box=z(S, K, 4, dt=torch.float32) + 3,
                        mem_gap=z(S, K, dt=torch.int32) - 5, mem_n=z(S, dt=torch.int32))

    def launch(self, n, arrays):
        from peppa_pig_face_landmark_b200 import runtime as rt
        torch = self.torch
        for k, v in arrays.items():
            self.inp[k].copy_(torch.from_numpy(v))
        every = {**self.state, **self.mem}
        before = {k: v.clone() for k, v in every.items()}
        i, s = self.inp, self.state
        head = [C.byref(self.cfg), n, self.K, P, i["kps_now"].data_ptr(), i["count"].data_ptr(), i["flag"].data_ptr(),
                i["hw"].data_ptr(), i["boxes4"].data_ptr(), i["src"].data_ptr()] + \
               [s[k].data_ptr() for k in ("prev_lm", "prev_dx", "n_prev", "prev_f32", "state_idx", "track_box", "track_f32",
                                          "n_track", "ids", "next_id", "out_kps")]
        stream = torch.cuda.current_stream().cuda_stream
        if self.legacy:
            rt.check(self.lib.skps_debug_mp_temporal(*head, stream))
        else:
            mem = [None] * 4 if self.null else [self.mem[k].data_ptr() for k in ("mem_ids", "mem_box", "mem_gap", "mem_n")]
            rt.check(self.lib.skps_debug_mp_temporal_mem(*head, self.m, *mem, stream))
        torch.cuda.synchronize()
        for k, v in every.items():                   # streams the launch did not cover: every byte as it was
            assert torch.equal(v[n:].view(torch.uint8), before[k][n:].view(torch.uint8)), ("uncovered stream changed", k)
        if self.m == 0:                              # memory off: the memory buffers are not touched at all
            for k, v in self.mem.items():
                assert torch.equal(v.view(torch.uint8), before[k].view(torch.uint8)), ("memory written while off", k)
        out = {k: v[:n].cpu().numpy() for k, v in every.items()}
        return out


def _check_memory(st, s, host, what):
    ids, boxes, gaps = host.rule.contents()
    k = int(st["mem_n"][s])
    assert k == len(ids), (what, "entries", k, len(ids))
    assert st["mem_ids"][s, :k].tolist() == ids, (what, "entry ids")
    assert st["mem_gap"][s, :k].tolist() == gaps, (what, "entry gaps")
    T._same(st["mem_box"][s, :k], boxes, (what, "entry boxes"))


def _run_mem(scripts, K, m, launches, cover=None):
    """scripts[s](host, rng, K) per stream; every launch checked stream by stream against the restatement."""
    S = len(scripts)
    hosts = [_MemHost(m, K) for _ in range(S)]
    gens = [make(hosts[s], np.random.default_rng(2000 + s), K) for s, make in enumerate(scripts)]
    dev = _MemDevice(S, K, m)
    revived = fullest = 0
    for t in range(launches):
        n = S if cover is None else cover(t)
        arrays = dict(kps_now=np.zeros((S, K, P, 2), F32), count=np.zeros(S, np.int32), flag=np.zeros(S, np.int32),
                      hw=np.ones((S, 2), np.int32), boxes4=np.zeros((S, K, 4), F32), src=np.full((S, K), -1, np.int32))
        for s in range(n):
            fr = next(gens[s])
            k = len(fr["kps"])
            h = hosts[s]
            tmp = h.track(fr["flag"], fr["hw"], fr["kps"])
            boxes = fr["boxes"](tmp) if callable(fr["boxes"]) else fr["boxes"]
            boxes = np.asarray(boxes, F32).reshape(k, 4)
            src = np.asarray(fr["src"], np.int32).reshape(k)
            remembered = {e[0] for e in h.rule.mem}
            h.judge(boxes, tmp, src)
            revived += sum(1 for i in h.ids if i in remembered)
            fullest = max(fullest, len(h.rule.mem))
            arrays["kps_now"][s, :k] = fr["kps"]
            arrays["count"][s], arrays["flag"][s], arrays["hw"][s] = k, fr["flag"], fr["hw"]
            arrays["boxes4"][s, :k], arrays["src"][s, :k] = boxes, src
        st = dev.launch(n, arrays)
        for s in range(n):
            T._check(st, s, hosts[s], (t, s))
            _check_memory(st, s, hosts[s], (t, s))
    return hosts, revived, fullest


def _blink(h, rng, K, p_away=0.3):
    """Up to K faces on a grid, each missing from a frame with probability p_away (runs of misses of any length): every
    present face continues its previous set when it was there the frame before, else comes back at its place."""
    n = int(rng.integers(1, K + 1))
    base = T._sets(rng, T._grid(n))
    yield T._frame(base, flag=1, src=np.full(n, -1))
    prev_present = list(range(n))
    while True:
        present = [f for f in range(n) if rng.random() >= p_away]
        kps = np.array([base[f] + rng.normal(0, 0.3, base[f].shape) for f in present], F32).reshape(-1, P, 2)
        src = [prev_present.index(f) if f in prev_present and rng.random() < 0.9 else int(rng.integers(-1, 3))
               for f in present]
        yield T._frame(kps, flag=int(rng.random() < 0.3), src=src)
        prev_present = present


def _flip(h, rng, K):
    """A face lost for one frame comes back with a box whose float32 IoU with the remembered one lies either side of the
    threshold by the last float32 steps (_flip_partner: the float32 and float64 decisions differ), then random frames."""
    face = np.array([[0.75, 8.5, 1201.3, 700.6]], F32)
    for prefer in (True, False, True, False):
        yield T._frame(T._sets(rng, face), flag=1, src=[-1])
        yield T._frame(np.zeros((0, P, 2), F32))
        entry = h.rule.mem[0][1]
        q = T._flip_partner(entry, IOU, False, prefer)
        assert (T.H.iou_xyxy(q, entry) > IOU) == prefer
        yield T._frame(T._sets(rng, face), flag=1, boxes=q[None], src=[-1])
        yield T._frame(np.zeros((0, P, 2), F32), flag=1)
    yield from T._random(h, rng, K)


def _blink_script(h, rng, K):
    yield from _blink(h, rng, K)


def _overflow(h, rng, K):
    """K faces, then K others half a cell to the right, K others half a cell down (IoU about 0.3 with the first: no id
    comes back), then the first K again: 2 K tracks were lost, only the K most recent are remembered."""
    g = T._grid(K)
    cw, ch = g[0, 2] - g[0, 0], g[0, 3] - g[0, 1]
    for shift in ([0, 0], [cw / 2, 0], [0, ch / 2], [0, 0]):
        yield T._frame(T._sets(rng, g + np.array(shift * 2, F32)), flag=1, src=np.full(K, -1))
    assert len(h.rule.mem) == K
    yield from _blink(h, rng, K)


def test_kernel_scripted_streams_against_the_restatement():
    """K = 64, 16 streams, id_memory 5: one-ulp IoU flips against remembered boxes, 128 tracks lost within two frames,
    blinking faces, random sequences, every fourth launch covering half the streams."""
    S, K = 16, 64
    scripts = [_flip, _flip, _overflow, _overflow] + [_blink_script] * 8 + [T._random_script, T._s_empty, T._s_ids,
                                                                              T._s_churn]
    hosts, revived, fullest = _run_mem(scripts, K, 5, 24, cover=lambda t: S if t % 4 != 3 else S // 2)
    assert revived > 100, revived
    assert fullest == K


@pytest.mark.parametrize("K", [1, 5, 64])
def test_kernel_256_streams(K):
    """256 streams at K = 1, 5 and 64 with id_memory 3; every third launch covers 100 streams."""
    S = 256
    scripts = [_blink_script if s % 2 == 0 else T._random_script for s in range(S)]
    hosts, revived, fullest = _run_mem(scripts, K, 3, 10, cover=lambda t: S if t % 3 != 2 else 100)
    assert revived > 0
    assert fullest == K or K == 64


@pytest.mark.parametrize("null", [False, True])
def test_kernel_memory_off_is_the_existing_launch(null):
    """id_memory 0 through the new entry (with or without memory buffers) and skps_debug_mp_temporal give the same state,
    byte for byte, launch after launch."""
    S, K = 12, 64
    scripts = [_blink_script] * 6 + [T._random_script] * 6
    hosts = [T._Host() for _ in range(S)]
    gens = [make(hosts[s], np.random.default_rng(3000 + s), K) for s, make in enumerate(scripts)]
    new, old = _MemDevice(S, K, 0, null=null), _MemDevice(S, K, 0, legacy=True)
    for t in range(16):
        n = S if t % 3 else 5
        arrays = dict(kps_now=np.zeros((S, K, P, 2), F32), count=np.zeros(S, np.int32), flag=np.zeros(S, np.int32),
                      hw=np.ones((S, 2), np.int32), boxes4=np.zeros((S, K, 4), F32), src=np.full((S, K), -1, np.int32))
        for s in range(n):
            fr = next(gens[s])
            k = len(fr["kps"])
            tmp = hosts[s].track(fr["flag"], fr["hw"], fr["kps"])
            boxes = fr["boxes"](tmp) if callable(fr["boxes"]) else fr["boxes"]
            boxes = np.asarray(boxes, F32).reshape(k, 4)
            src = np.asarray(fr["src"], np.int32).reshape(k)
            hosts[s].judge(boxes, tmp, src)
            arrays["kps_now"][s, :k] = fr["kps"]
            arrays["count"][s], arrays["flag"][s], arrays["hw"][s] = k, fr["flag"], fr["hw"]
            arrays["boxes4"][s, :k], arrays["src"][s, :k] = boxes, src
        a, b = new.launch(n, arrays), old.launch(n, arrays)
        for key in new.state:
            T._same(a[key], b[key], (t, key))
        for s in range(n):
            T._check(a, s, hosts[s], (t, s))


def test_kernel_entry_refuses_bad_arguments():
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    dev = _MemDevice(2, 4, 1)
    i, s = dev.inp, dev.state
    ptrs = [i[k].data_ptr() for k in ("kps_now", "count", "flag", "hw", "boxes4", "src")] + \
           [s[k].data_ptr() for k in ("prev_lm", "prev_dx", "n_prev", "prev_f32", "state_idx", "track_box", "track_f32",
                                      "n_track", "ids", "next_id", "out_kps")]
    mem = [dev.mem[k].data_ptr() for k in ("mem_ids", "mem_box", "mem_gap", "mem_n")]
    cfg = C.byref(T._cfg(4))
    assert lib.skps_debug_mp_temporal_mem(cfg, 2, 4, P, *ptrs, -1, *mem, None) != 0
    assert b"id_memory" in lib.skps_last_error()
    for at in range(4):
        bad = list(mem)
        bad[at] = None
        assert lib.skps_debug_mp_temporal_mem(cfg, 2, 4, P, *ptrs, 1, *bad, None) != 0
    assert lib.skps_debug_mp_temporal_mem(cfg, 2, 65, P, *ptrs, 1, *mem, None) != 0


# ----------------------------------------------------------------------------- FaceAna end to end
CELL = (slice(540, 1080), slice(960, 1920))      # grid cell (1, 1) at 1080p (2 x 2 faces) and at 4K (4 x 4 faces)


def _gap_scene(gap, big=False, length=7):
    """Faces on a grid; the one in the cell at grid position (1, 1) is covered for `gap` frames from frame 2.  The
    brightness alternates by 8 so that the gate runs the detector wherever a frame differs from the one before."""
    full = frames.frame_4k() if big else frames.multi_face_frame(1080, 1920, (2, 2), 440)
    gone = full.copy()
    gone[CELL] = frames._background(*full.shape[:2])[CELL]
    seq = [full, full] + [_bright(gone, 8) if i % 2 == 0 else gone for i in range(gap)]
    back = full if gap % 2 else _bright(full, 8)
    return (seq + [back] * length)[:length]


def _covered(r):
    cx, cy = (r["box"][0] + r["box"][2]) / 2, (r["box"][1] + r["box"][3]) / 2
    return 960 <= cx < 1920 and 540 <= cy < 1080


def _sources_boxes(prev_boxes, det_rows, top_k):
    """facer.py:56-66 restated: the source and the float32 box of every face the call returns, in output order (the
    boxes the landmark stage gets; a face judged against a track box gets the EMA of the two rows in float32)."""
    from oracle import host_ref as H
    prev = np.asarray(prev_boxes, F32).reshape(-1, 4)
    if det_rows is None:
        judged, src = prev.copy(), list(range(len(prev)))
    else:
        now = np.asarray(det_rows, F32)[:, :4]
        judged, src = now.copy(), [-1] * len(now)
        for i, r in enumerate(now):
            for j, p in enumerate(prev):
                if H.iou_xyxy(r, p) > IOU:
                    judged[i] = ALPHA * r + (1 - ALPHA) * p
                    src[i] = j
                    break
    if len(judged) == 0:
        return [], np.zeros((0, 4), F32)
    area = (judged[:, 2] - judged[:, 0]) * (judged[:, 3] - judged[:, 1])
    keep = np.where(area > MIN_FACE)[0]
    if len(keep) > top_k:
        keep = keep[area[keep].argsort(kind="stable")[-top_k:][::-1]]
    return [src[i] for i in keep], judged[keep]


class _Follow:
    """Follows a FaceAna(track_ids=True, id_memory=m) call by call: its ids against the restated rule, fed with the
    sources and boxes restated from last_det_rows and the previous call's returned boxes."""

    def __init__(self, facer, m):
        self.facer, self.rule = facer, _Restated(m, facer.top_k)

    def run(self, frame, what):
        f = self.facer
        f.last_det_rows = None
        res = f.run(frame)
        src, boxes = _sources_boxes(self.rule.boxes, f.last_det_rows, f.top_k)
        returned = np.asarray([r["box"] for r in res], F32).reshape(-1, 4)
        want = self.rule.call(src, boxes, returned)
        assert len(src) == len(res), (what, len(src), len(res))
        assert [r["id"] for r in res] == want, (what, [r["id"] for r in res], want)
        assert all(type(r["id"]) is int for r in res)
        return res

    def reset(self):
        self.facer.reset()
        self.rule.reset()


def _same_but_id(a, b, what):
    assert len(a) == len(b), (what, len(a), len(b))
    for x, y in zip(a, b):
        assert set(x) == set(y), what
        for k in x:
            if k == "id":
                continue
            if k == "pose":
                for q in x[k]:
                    assert np.array_equal(x[k][q], y[k][q]) and x[k][q].dtype == y[k][q].dtype, (what, k, q)
                continue
            assert np.asarray(x[k]).dtype == np.asarray(y[k]).dtype and np.array_equal(x[k], y[k]), (what, k)


@pytest.mark.parametrize("gap", [1, 2, 3])
def test_faceana_covered_face_gets_its_id_back_within_id_memory(gap):
    from Skps import FaceAna
    clip = _gap_scene(gap)
    runs = {}
    for m in (0, 1, 2, 5):
        follow = _Follow(FaceAna(track_ids=True, id_memory=m, pose=m == 2), m)
        runs[m] = [follow.run(fr, (gap, m, t)) for t, fr in enumerate(clip)]
    base = FaceAna(track_ids=True, pose=True)
    base_res = [base.run(fr) for fr in clip]
    for m, res in runs.items():
        first = {i: r["id"] for i, r in enumerate(res[0])}
        assert len(first) == 4 and sorted(first.values()) == [0, 1, 2, 3]
        covered_id = next(r["id"] for r in res[0] if _covered(r))
        for t, (got, ref) in enumerate(zip(res, base_res if m == 2 else runs[0])):
            _same_but_id(got, ref, (gap, m, t))
            others = sorted(r["id"] for r in got if not _covered(r))
            assert others == sorted(v for v in first.values() if v != covered_id), (gap, m, t, others)
            back = [r["id"] for r in got if _covered(r)]
            if 2 <= t < 2 + gap:
                assert back == [], (gap, m, t)
            else:
                want = covered_id if t < 2 or gap <= m else 4
                assert back == [want], (gap, m, t, back, want)
        n_ids = len({r["id"] for fr in res for r in fr})
        print("covered %d frames, id_memory %d: %d ids" % (gap, m, n_ids))
        assert n_ids == (4 if gap <= m else 5)


def test_faceana_id_memory_detect_every_3():
    from Skps import FaceAna
    for gap in (1, 2, 3):
        clip = _gap_scene(gap, length=9)
        f = _Follow(FaceAna(track_ids=True, id_memory=2, detect_every=3), 2)
        off = FaceAna(track_ids=True, detect_every=3)
        for t, fr in enumerate(clip):
            _same_but_id(f.run(fr, (gap, t)), off.run(fr), (gap, t))


def test_faceana_id_memory_4k_top_k_16():
    from Skps import FaceAna
    clip = _gap_scene(2, big=True)
    f = _Follow(FaceAna(top_k=16, track_ids=True, id_memory=2), 2)
    off = FaceAna(top_k=16, track_ids=True)
    res = []
    for t, fr in enumerate(clip):
        res.append(f.run(fr, t))
        _same_but_id(res[-1], off.run(fr), t)
    assert len(res[0]) == 16 and len(res[2]) == 15
    assert sorted(r["id"] for r in res[-1]) == list(range(16))
    f.reset()
    assert [r["id"] for r in f.run(clip[0], "after reset")] == [r["id"] for r in res[0]]


# ----------------------------------------------------------------------------- FaceAnaStreams
def _stream_seqs():
    from test_streams_gpu import _sequences
    return [_gap_scene(g, length=6) for g in (1, 2, 3)] + _sequences()


def _check_ids(res, singles, frames_of, what):
    """The ids of each stream equal its FaceAna's; host results also agree as test_streams_gpu compares them."""
    from test_streams_gpu import _same
    for s, fr in frames_of.items():
        want = singles[s].run(fr)
        got = [r if isinstance(r, int) else r["id"] for r in res[s]]
        assert got == [r["id"] for r in want], (what, s, got, [r["id"] for r in want])
        if res[s] and not isinstance(res[s][0], int):
            _same(res[s], want)


@pytest.mark.parametrize("m", [1, 2])
def test_streams_equal_single_stream_faceana_host_frames(m):
    """Host frames and host results, partial batches, reset(stream) inside stream 1's memory window, and reset()."""
    from Skps import FaceAna, FaceAnaStreams
    seqs = _stream_seqs()
    S = len(seqs)
    fa = FaceAnaStreams(n_streams=S, track_ids=True, id_memory=m)
    singles = [FaceAna(track_ids=True, id_memory=m) for _ in range(S)]
    for t in range(6):
        n = S if t % 3 != 1 else 2                              # streams 2.. skip frame 1
        if t == 3:
            fa.reset(1)                                         # stream 1's face is covered at its frames 2 and 3
            singles[1].reset()
        res = fa.run([seqs[s][t] for s in range(n)])
        assert len(res) == n
        _check_ids(res, singles, {s: seqs[s][t] for s in range(n)}, t)
    fa.reset()
    for s in singles:
        s.reset()
    _check_ids(fa.run([s[0] for s in seqs]), singles, {s: seqs[s][0] for s in range(S)}, "after reset()")


def test_streams_equal_single_stream_faceana_cuda_frames_two_in_flight():
    """CUDA frames, two batches in flight, device (out=) and host results alternating."""
    import torch
    from Skps import FaceAna, FaceAnaStreams
    seqs = _stream_seqs()
    S = len(seqs)
    fa = FaceAnaStreams(n_streams=S, track_ids=True, id_memory=2)
    singles = [FaceAna(track_ids=True, id_memory=2) for _ in range(S)]
    bufs, pending = [fa.new_results(), fa.new_results()], []
    modes = ["dev", "host", "dev", "dev", "host", "dev"]

    def submit(t):
        batch = [torch.from_numpy(s[t]).cuda() for s in seqs]
        fa.submit(batch, out=bufs[t % 2] if modes[t] == "dev" else None)
        pending.append(t)

    def collect():
        t = pending.pop(0)
        r = fa.collect()
        if modes[t] == "dev":
            ids, n = r["id"].cpu().numpy(), r["n"].cpu().numpy()
            r = [[int(v) for v in ids[s, :int(n[s])]] for s in range(S)]
        _check_ids(r, singles, {s: seqs[s][t] for s in range(S)}, (t, modes[t]))

    submit(0)
    for t in range(1, 6):
        submit(t)
        collect()
    collect()


def test_streams_detect_every_3():
    from Skps import FaceAna, FaceAnaStreams
    seqs = [_gap_scene(g, length=8) for g in (1, 2, 3, 1, 2)]
    S = len(seqs)
    fa = FaceAnaStreams(n_streams=S, track_ids=True, id_memory=2, detect_every=3)
    singles = [FaceAna(track_ids=True, id_memory=2, detect_every=3, detect_offset=s % 3) for s in range(S)]
    for t in range(8):
        _check_ids(fa.run([s[t] for s in seqs]), singles, {s: seqs[s][t] for s in range(S)}, t)
