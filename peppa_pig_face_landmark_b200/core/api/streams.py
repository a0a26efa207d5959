"""FaceAnaStreams — FaceAna.run for many concurrent video streams on one GPU (additive API, SURVEY.md 8b / 8f-1).

The reference serves one stream per FaceAna instance and keeps the temporal state (previous frame, track boxes,
GroupTrack / One-Euro history; facer.py:28-50, lk.py:6-91) in Python.  Here one object owns S streams: each call takes
one frame for each of any subset of the streams and runs ONE detector forward and ONE landmark forward for all of them,
the state lives on the device (csrc/mpipe.cu, csrc/temporal.cu) and two batches can be in flight so that frame uploads
overlap compute.

    fa = FaceAnaStreams(n_streams=16, top_k=4)
    results = fa.run(frames)            # list of S lists of {'box','kps','scores'} - what S FaceAna.run calls return
    # cameras at their own frame rates: frames for streams 5, 2 and 9 only; results[i] is stream [5, 2, 9][i]'s, and the
    # other streams are untouched (no frame counted, no filter step, no id_memory gap)
    results = fa.run([f5, f2, f9], streams=[5, 2, 9])
    # FaceAnaStreams(..., align=112): each dict also has 'chip' (112x112x3 uint8, aligned) and 'M' (2x3 float64)
    # FaceAnaStreams(..., pose=True): each dict also has 'pose' {'euler', 'rvec', 'tvec', 'reproject'} as FaceAna returns it
    # FaceAnaStreams(..., track_ids=True): each dict also has 'id', the track id FaceAna(track_ids=True) gives the face
    # FaceAnaStreams(..., detect_every=4): stream s runs the detector on a quarter of its frames, staggered by s % 4
    # FaceAnaStreams(..., track_ids=True, id_memory=30): a face lost for up to 30 frames gets its old id back
    # or, overlapped:
    fa.submit(frames_t0); fa.submit(frames_t1); r0 = fa.collect(); fa.submit(frames_t2); r1 = fa.collect(); ...
    # frames already on the GPU (torch.uint8 CUDA tensors (H, W, 3), any row pitch), results left on the GPU:
    res = [fa.new_results(), fa.new_results()]
    fa.submit(cuda_frames_t0, out=res[0]); fa.submit(cuda_frames_t1, out=res[1]); r0 = fa.collect(); ...
"""
import ctypes as C
import os
import pathlib

import numpy as np

from ... import runtime as rt
from ...graph_tools import check_detector_input, detector_onnx_for
from .align import check_size
from .device_frames import check_cuda_frame, check_host_frame, check_layout, check_rotate, is_cuda_tensor
from .facer import check_detect_every, check_id_memory, get_cfg, pipeline_cfg
from .onnx_model_base import ONNXEngine


def check_streams(streams, n, n_streams):
    """The streams of a call of n frames as a list of ints, or None for streams 0..n-1 (streams None): a sequence of n
    distinct ints in 0..n_streams-1, one per frame, else ValueError."""
    if streams is None:
        return None
    if isinstance(streams, (str, bytes)) or not hasattr(streams, "__len__"):
        raise ValueError("streams must be a sequence of ints, got %r" % (streams,))
    ids = list(streams)
    if len(ids) != n:
        raise ValueError("streams: %d ids for %d frames" % (len(ids), n))
    for i, t in enumerate(ids):
        if not isinstance(t, (int, np.integer)) or isinstance(t, (bool, np.bool_)):
            raise ValueError("streams[%d] must be an int, got %r" % (i, t))
        if not 0 <= t < n_streams:
            raise ValueError("streams[%d] = %d is outside 0..%d" % (i, t, n_streams - 1))
    ids = [int(t) for t in ids]
    if len(set(ids)) != n:
        # two frames of one stream in one call would depend on each other: the second's previous frame is the first
        dup = sorted({t for t in ids if ids.count(t) > 1})
        raise ValueError("streams: each stream takes at most one frame per call, got %s more than once" % dup)
    return ids


class FaceAnaStreams:
    def __init__(self, n_streams, top_k=None, max_frame_hw=(2160, 3840), device="cuda", align=None, pose=False,
                 det_input=None, track_ids=False, detect_every=1, id_memory=0):
        """align: None, or a chip side in 16..512: every result dict then also carries 'chip' and 'M' as FaceAna(align=...)
        returns them, warped inside the same submit on the device from the smoothed landmarks and the frame in the ring.
        pose: every result dict then also carries 'pose' as FaceAna(pose=True) returns it, solved inside the same submit
        from the smoothed landmarks, with each stream's own frame size for the camera.
        det_input: None (Skps.yml's 384x640) or the detector input size (h, w), as FaceAna(det_input=...) takes it.  The
        detector runs on all n_streams frames at once, so its activations take n_streams times FaceAna's memory (about
        0.35 GB per stream at 1152x1920).
        track_ids: every result dict then also carries 'id', the int FaceAna(track_ids=True) returns for the face: ids
        are numbered per stream from 0, reset(stream) starts that stream again from 0, and the rule that assigns them is
        FaceAna's.  The ids are kept on the device next to the track boxes, whether or not they are returned.
        id_memory: FaceAna(track_ids=True, id_memory=...) for every stream: up to top_k lost tracks per stream (about 28
        bytes each) whose ids a face that reappears where one was lost takes back, kept and matched on the device.  A
        stream's frames are the calls that include it (submit(streams=...)): a call without it does not age its lost
        tracks; reset(stream) forgets them.
        detect_every: the detection cadence of FaceAna(detect_every=N, detect_offset=s % N) for stream s, which it
        returns bit for bit.  A stream counts its frames from construction or reset(stream), advancing only on calls
        that include a frame for it; frame i runs the detector when the stream has no previous frame of its size, or
        when (i + s % N) % N == 0 and the frame-difference gate fires, and otherwise takes the tracker path.  A face that
        enters is found up to N - 1 frames late; one that leaves is followed by its landmark box until the next keyframe.
        The staggered offsets spread the keyframes over the calls: the detector runs on about n_streams / N frames per
        call, packed into one batch, and not at all on a call without keyframes (last_detector_frames).  The detector
        engine keeps one CUDA graph per batch size it meets; with the stagger those are only a few sizes.  The offset is
        keyed to the stream id, not to the frame's position in a call.

        Streams need not be frame-synchronous: a call feeds any subset of them, in any order (submit(streams=...)), and
        costs what its frames cost - the detector batch is its keyframes, the landmark batch len(frames) * top_k faces.
        A stream a call does not feed is untouched: no frame is counted, no filter step runs, no id_memory gap is counted,
        its cadence phase does not move and its previous frame stays."""
        self.detect_every = check_detect_every(detect_every)[0]
        self.id_memory = check_id_memory(id_memory, track_ids)
        self.align = None if align is None else check_size(align)
        self.pose = bool(pose)
        self.track_ids = bool(track_ids)
        cfg = get_cfg()['Skps']
        det_cfg, kps_cfg = cfg['Detect'], cfg['Keypoints']
        self.n_streams = int(n_streams)
        self.top_k = int(top_k if top_k is not None else det_cfg['topk'])
        if not 1 <= self.top_k <= 64:
            # one landmark forward of n_streams * top_k faces per call, sized on the device with no host read-back, so
            # top_k bounds its memory (about 47 MB per face); FaceAna takes up to 1024
            raise ValueError("FaceAnaStreams: top_k %d outside 1..64 (the landmark batch is n_streams * top_k faces; "
                             "FaceAna takes up to 1024)" % self.top_k)
        pc = pipeline_cfg(cfg, self.top_k, max_frame_hw)
        root = pathlib.Path(__file__).resolve().parents[2]
        det_hw = det_cfg['input_shape'][:2] if det_input is None else check_detector_input(det_input)
        self.det = ONNXEngine(detector_onnx_for(os.path.join(root, det_cfg['model_path']), det_hw), device=device,
                              max_batch=self.n_streams)
        self.kps = ONNXEngine(os.path.join(root, kps_cfg['model_path']), device=device,
                              max_batch=self.n_streams * self.top_k)
        self.n_points = int(kps_cfg['num_points'])
        self.device = self.det.device
        self.max_frame_hw = (int(max_frame_hw[0]), int(max_frame_hw[1]))
        self.lib = rt.load_library()
        h = C.c_void_p()
        rt.check(self.lib.skps_mpipe_create(self.det.handle, self.kps.handle, C.byref(pc), self.n_streams, C.byref(h)))
        self._h = h
        if self.detect_every != 1:
            rt.check(self.lib.skps_mpipe_set_detect_every(h, self.detect_every))
        if self.id_memory:
            rt.check(self.lib.skps_mpipe_set_id_memory(h, self.id_memory))
        S, K, P = self.n_streams, self.top_k, self.n_points
        self._out = [dict(n=np.zeros(S, np.int32), box=np.zeros((S, K, 4), np.float64), kps=np.zeros((S, K, P, 2), np.float64),
                          sc=np.zeros((S, K, P), np.float32), det=np.zeros(S, np.int32), ids=np.zeros((S, K), np.int64))
                     for _ in range(2)]
        if self.align is not None:
            rt.check(self.lib.skps_mpipe_set_align(h, self.align))
            for o in self._out:
                o["chips"] = np.zeros((S, K, self.align, self.align, 3), np.uint8)
                o["M"] = np.zeros((S, K, 2, 3), np.float64)
        if self.pose:
            rt.check(self.lib.skps_mpipe_set_pose(h, 1))
            for o in self._out:
                o["pose"] = {k: np.zeros((S, K, 3), np.float64) for k in ("rvec", "tvec", "euler")}
                o["pose"]["reproject"] = np.zeros((S, K, 8, 2), np.float64)
        self._pending = []              # [(slot, n, keep-alive frames, device results or None)]
        self._next = 0
        self.last_ran_detector = None
        self.last_detector_frames = None      # frames the detector ran on in the last collected batch
        self._m = C.c_int32(0)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            self.lib.skps_mpipe_destroy(h)
            self._h = None

    def reset(self, stream=None):
        """FaceAna.reset (facer.py:200-208) for one stream, or for all of them; the stream's frame count starts again
        from 0."""
        while self._pending:
            self.collect()
        rt.check(self.lib.skps_mpipe_reset(self._h, -1 if stream is None else int(stream)))

    def submit(self, frames, out=None, streams=None, layout="bgr", rotate=0):
        """Enqueue one frame for each of some streams.  At most two batches may be pending; results come back from
        collect() in submission order.

        streams: None, frames[i] -> stream i (len(frames) <= n_streams); or a sequence of distinct ints in
        0..n_streams-1, one per frame in any order, frames[i] being the next frame of stream streams[i].  Everything per
        call stays in call order: collect()'s entry i, last_ran_detector[i] and, with out=, row i of every result tensor
        belong to frames[i].  A stream the call does not feed is untouched (its frame count, cadence phase, filters,
        previous frame, track boxes, ids and lost tracks stay as they are).  A length mismatch, a duplicate, an id out of
        range or one that is not an int raises ValueError before anything is enqueued.

        frames: all HxWx3 uint8 BGR numpy arrays, or all torch.uint8 CUDA tensors (H, W, 3) in BGR order on this object's
        device with stride(2) == 1, stride(1) == 3 and any row pitch stride(0) >= 3W (packed tensors, pitched decoder
        surfaces, big[y0:y1, x0:x1] views); a mix raises ValueError.  CUDA frames never cross PCIe: one kernel for the
        batch gathers them into the pipeline's frame ring.  Ordering on torch.cuda.current_stream(): they are read after all
        work already queued on it, and work queued on it after submit() returns runs after they have been read, so a
        decoder may reuse its surfaces at once.

        layout: the pixel layout of all CUDA frames of the call (device_frames.frame_layout): "bgr" (the default),
        "rgb", "bgra", "rgba" (H, W, 4), or "bgr_planar", "rgb_planar" (3, H, W) with any row and plane pitch.  The
        gathering kernel packs them into the ring as BGR, so the results are, bit for bit, those of the same pixels
        passed as interleaved BGR, and the gate, detect_every, track ids and smoothing do not see the layout: calls may
        change it.  Host frames are BGR only.

        rotate: the clockwise angle in degrees (0, 90, 180 or 270) by which CUDA frames, as stored, must be turned to be
        upright (device_frames.check_rotate), one for the call or one per frame, so cameras mounted differently are fed
        in one call.  The gathering kernel puts each frame into the ring upright, and the results are in the upright
        frame's pixels, bit for bit those of the upright frames passed as contiguous tensors.  A stream sees the upright
        frame: a change between 0 and 90 changes its frame size (the next frame runs the detector), one between 0 and
        180 does not.  Host frames take 0.

        out: None (collect() returns host results), or, with CUDA frames, a dict from new_results() not used by a batch
        still in flight: the batch's results are written into it on the GPU and nothing is copied to the host."""
        if len(self._pending) == 2:
            raise RuntimeError("FaceAnaStreams: two batches already in flight; call collect() first")
        n = len(frames)
        if not 0 < n <= self.n_streams:
            raise ValueError("expected 1..%d frames, got %d" % (self.n_streams, n))
        ids = check_streams(streams, n, self.n_streams)
        smap = None if ids is None else np.array(ids, np.int32)
        on_device = [is_cuda_tensor(f) for f in frames]
        check_layout(layout, any(on_device))
        turns = check_rotate(rotate, n, any(on_device))
        if any(on_device):
            if not all(on_device):
                raise ValueError("one batch takes either host frames or CUDA frames, got both (streams %s are CUDA)"
                                 % [i for i, d in enumerate(on_device) if d])
            self._submit_device(frames, out, smap, layout, turns)
            return
        if out is not None:
            raise ValueError("out= keeps results on the GPU and takes CUDA frames; these are host frames")
        keep = [check_host_frame(f) for f in frames]
        ptrs = (C.c_void_p * n)(*[f.ctypes.data for f in keep])
        hw = np.array([[f.shape[0], f.shape[1]] for f in keep], np.int32)
        slot = self._next
        rt.check(self.lib.skps_mpipe_submit_streams(self._h, slot, None if smap is None else smap.ctypes.data, ptrs,
                                                    hw.ctypes.data, n))
        self._pending.append((slot, n, keep, None))
        self._next ^= 1

    def _submit_device(self, frames, out, smap, layout, turns):
        import torch
        n = len(frames)
        shapes = [check_cuda_frame(f, self.device, self.max_frame_hw, layout) for f in frames]
        outs = None
        if out is not None:
            self._check_out(out)
            outs = rt.MpipeOutputs(n_faces=out["n"].data_ptr(), ran_detector=out["ran_detector"].data_ptr(),
                                   boxes=out["box"].data_ptr(), kps=out["kps"].data_ptr(), scores=out["scores"].data_ptr())
            for k, field in (("chip", "chips"), ("M", "M"), ("rvec", "rvec"), ("tvec", "tvec"), ("euler", "euler"),
                             ("reproject", "reproject"), ("id", "ids")):
                if k in out:
                    setattr(outs, field, out[k].data_ptr())
        ptrs = (C.c_void_p * n)(*[f.data_ptr() for f in frames])
        pitches = np.array([f.pitch for f in shapes], np.int32)
        planes = np.array([f.plane for f in shapes], np.int32)
        hw = np.array([[f.H, f.W] for f in shapes], np.int32)
        slot = self._next
        q = np.array(turns, np.int32)                 # as stored: hw, pitches; the ring gets them upright
        rt.check(self.lib.skps_mpipe_submit_device_rotate(self._h, slot, None if smap is None else smap.ctypes.data, ptrs,
                                                          pitches.ctypes.data, hw.ctypes.data, n, shapes[0].code,
                                                          planes.ctypes.data, q.ctypes.data if any(turns) else None,
                                                          None if outs is None else C.byref(outs),
                                                          torch.cuda.current_stream(self.device).cuda_stream))
        self._pending.append((slot, n, list(frames), out))
        self._next ^= 1

    def _result_layout(self):
        import torch
        S, K, P = self.n_streams, self.top_k, self.n_points
        f64 = torch.float64
        r = {"n": ((S,), torch.int32), "ran_detector": ((S,), torch.int32), "box": ((S, K, 4), f64),
             "kps": ((S, K, P, 2), f64), "scores": ((S, K, P), torch.float32)}
        if self.align is not None:
            r["chip"] = ((S, K, self.align, self.align, 3), torch.uint8)
            r["M"] = ((S, K, 2, 3), f64)
        if self.pose:
            r.update(rvec=((S, K, 3), f64), tvec=((S, K, 3), f64), euler=((S, K, 3), f64), reproject=((S, K, 8, 2), f64))
        if self.track_ids:
            r["id"] = ((S, K), torch.int64)
        return r

    def new_results(self):
        """Device result buffers for submit(cuda_frames, out=...): a dict of CUDA tensors on this object's device,
        n (S,) int32 faces per frame; ran_detector (S,) int32, whether the frame used the detector's rows (a keyframe
        whose frame-difference gate fired, or with no previous frame of its size); box (S,K,4) and kps
        (S,K,P,2) float64; scores (S,K,P) float32; with align, chip (S,K,size,size,3) uint8 and M (S,K,2,3) float64; with
        pose, rvec, tvec, euler (S,K,3) and reproject (S,K,8,2) float64; with track_ids, id (S,K) int64.  Row i belongs
        to frames[i] of the submit, in call order whatever its streams=; face rows j >= n[i] of row i, and rows
        i >= len(frames), are unspecified."""
        import torch
        return {k: torch.empty(shape, dtype=dt, device=self.device) for k, (shape, dt) in self._result_layout().items()}

    def _check_out(self, out):
        import torch
        want = self._result_layout()
        if not isinstance(out, dict) or set(out) != set(want):
            raise ValueError("out: expected a dict with keys %s (see new_results())" % sorted(want))
        for k, (shape, dt) in want.items():
            t = out[k]
            if (not isinstance(t, torch.Tensor) or tuple(t.shape) != shape or t.dtype != dt or t.device != self.device
                    or not t.is_contiguous()):
                got = ("%s %s on %s" % (t.dtype, tuple(t.shape), t.device)) if isinstance(t, torch.Tensor) \
                    else type(t).__name__
                raise ValueError("out[%r]: expected a contiguous %s tensor %s on %s, got %s" % (k, dt, shape, self.device,
                                                                                               got))
        busy = {t.data_ptr() for _, _, _, o in self._pending if o is not None for t in o.values()}
        if any(t.data_ptr() in busy for t in out.values()):
            raise ValueError("out: these buffers belong to a batch still in flight; collect() it first")

    def collect(self):
        """Results of the oldest pending batch: a list, entry i for frames[i] of its submit (stream i, or streams[i]),
        of lists of {'box','kps','scores'}; last_ran_detector[i] likewise; for a batch submitted with out=, that dict, with no host synchronisation: torch.cuda.current_stream() is made to wait
        for the batch, so work queued on it afterwards sees the results (last_ran_detector is then None; the gate's
        decisions are out['ran_detector'])."""
        if not self._pending:
            raise RuntimeError("FaceAnaStreams: nothing submitted")
        slot, n, _keep, out = self._pending.pop(0)
        rt.check(self.lib.skps_mpipe_detector_frames(self._h, slot, C.byref(self._m)))
        self.last_detector_frames = int(self._m.value)
        if out is not None:
            import torch
            rt.check(self.lib.skps_mpipe_wait_stream(self._h, slot, torch.cuda.current_stream(self.device).cuda_stream))
            self.last_ran_detector = None
            return out
        o = self._out[slot]
        rt.check(self.lib.skps_mpipe_wait(self._h, slot, o["n"].ctypes.data, o["box"].ctypes.data, o["kps"].ctypes.data,
                                          o["sc"].ctypes.data, o["det"].ctypes.data))
        self.last_ran_detector = o["det"][:n].astype(bool)
        if self.align is not None:
            rt.check(self.lib.skps_mpipe_align_results(self._h, slot, o["chips"].ctypes.data, o["M"].ctypes.data))
        if self.pose:
            q = o["pose"]
            rt.check(self.lib.skps_mpipe_pose_results(self._h, slot, q["rvec"].ctypes.data, q["tvec"].ctypes.data,
                                                      q["euler"].ctypes.data, q["reproject"].ctypes.data))
        if self.track_ids:
            rt.check(self.lib.skps_mpipe_track_ids(self._h, slot, o["ids"].ctypes.data))
        res = []
        for s in range(n):
            k = int(o["n"][s])
            res.append([{'box': o["box"][s, i].copy(), 'kps': o["kps"][s, i].copy(), 'scores': o["sc"][s, i].copy()}
                        for i in range(k)])
            if self.align is not None:
                for i, r in enumerate(res[-1]):
                    r['chip'] = o["chips"][s, i].copy()
                    r['M'] = o["M"][s, i].copy()
            if self.pose:
                for i, r in enumerate(res[-1]):
                    r['pose'] = {k: v[s, i].copy() for k, v in o["pose"].items()}
            if self.track_ids:
                for i, r in enumerate(res[-1]):
                    r['id'] = int(o["ids"][s, i])
        return res

    def run(self, frames, streams=None, layout="bgr", rotate=0):
        """One frame for each of some streams in (submit's streams=, layout= and rotate=), their results out in call
        order (blocking)."""
        self.submit(frames, streams=streams, layout=layout, rotate=rotate)
        return self.collect()
