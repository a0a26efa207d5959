"""FaceLandmark — same surface as the reference's Skps/core/api/face_landmark.py:14-115
(`FaceLandmark(cfg)(img, bboxes) -> ((K,98,2) float32, (K,98) float32)`).  The reference loops
over faces in Python with one batch-1 network call each (:40-48); here all faces are cropped by
one kernel straight into the network's input buffer and run as one batch.  The caller's `bboxes`
array is not modified (the reference mutates the rows in place, :81-90; facer.py:66 copies
first for that reason).

Additive: landmarks for faces the caller already has, from many frames per call (SURVEY.md 8b):

    fl = FaceLandmark(max_faces=256)
    res = fl.run_batch(frames, boxes)      # [(kps (k_i,98,2), scores (k_i,98)) per frame], host frames or CUDA frames
    # overlapped, results left on the GPU (CUDA frames; boxes may be CUDA tensors straight from a GPU detector):
    bufs = [fl.new_results(n), fl.new_results(n)]
    fl.submit(frames_0, boxes_0, out=bufs[0]); fl.submit(frames_1, boxes_1, out=bufs[1]); r0 = fl.collect(); ...
"""
import ctypes as C
import os
import pathlib
import time

import numpy as np

from ... import runtime as rt
from ...logger.logger import logger
from .device_frames import check_cuda_frame, check_host_frame, is_cuda_tensor, is_tensor
from .onnx_model_base import ONNXEngine

MIN_FACE = 20              # face_landmark.py:26,76: boxes with a side of at most this many pixels get no landmarks
MAX_SIDE = 1 << 20         # largest frame side run_batch takes: keeps every crop coordinate in int32
BOX_LIMIT = 2.0 ** 24      # largest |box coordinate| of host boxes: the host and device crop geometry stay exact in int32

# skps_face_src of include/skps_b200.h
FACE_SRC = np.dtype([("base", "<u8"), ("pitch", "<i4"), ("H", "<i4"), ("W", "<i4"), ("ox", "<i4"), ("oy", "<i4"),
                     ("rw", "<i4"), ("rh", "<i4"), ("_pad", "<i4")])
assert FACE_SRC.itemsize == 40


def face_scale(cfg):
    """Crop side over box side, float32(1 + 2 * base_extend_range[0]) (face_landmark.py:83 in float32); cfg: Skps.yml's
    Keypoints section."""
    return float(np.float32(1 + 2 * cfg['base_extend_range'][0]))


def crop_read_rects(boxes, H, W, face_scale, min_face=MIN_FACE):
    """(n, 4) int64 [x0, y0, x1, y1) per box: the rectangle of an H x W frame that the crop of the box (skps_crop_resize,
    skps_crop_faces) can read, widened by one pixel on each side and clipped to the frame; all zero when it reads nothing
    (too small a box, or one wholly outside the frame).  `boxes`: (n, >= 4) float32 with finite coordinates of at most
    BOX_LIMIT.  The geometry is crop_geometry's float32 arithmetic in image_ops.cu: crop column j reads frame column
    x1 - add + j (j < w) or the zero border, and the same for rows."""
    b = np.asarray(boxes, np.float32)[:, :4]
    fs, mf, two = np.float32(face_scale), np.float32(min_face), np.float32(2)
    bw, bh = b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]
    ok = ~((bw <= mf) | (bh <= mf))
    add = np.trunc(np.fmax(bw, bh)).astype(np.int64)
    fa = add.astype(np.float32)
    x0, y0, x1, y1 = b[:, 0] + fa, b[:, 1] + fa, b[:, 2] + fa, b[:, 3] + fa
    cx, cy = np.floor((x0 + x1) / two), np.floor((y0 + y1) / two)
    half = np.floor((fs * bw) / two)
    ix1 = np.maximum(np.trunc(cx - half).astype(np.int64), 0)
    iy1 = np.maximum(np.trunc(cy - half).astype(np.int64), 0)
    ix2 = np.minimum(np.trunc(cx + half).astype(np.int64), W + 2 * add)
    iy2 = np.minimum(np.trunc(cy + half).astype(np.int64), H + 2 * add)
    w, h = np.maximum(ix2 - ix1, 0), np.maximum(iy2 - iy1, 0)
    ok &= (w > 0) & (h > 0)
    c0, r0 = ix1 - add, iy1 - add
    ok &= (c0 < W) & (c0 + w > 0) & (r0 < H) & (r0 + h > 0)          # not wholly outside the frame
    out = np.stack([np.clip(c0 - 1, 0, W), np.clip(r0 - 1, 0, H), np.clip(c0 + w + 1, 0, W), np.clip(r0 + h + 1, 0, H)], 1)
    out[~ok] = 0
    return out


def _grow(t, n, make):
    """t when it holds n elements, else make(max(n, 2 * len(t)))."""
    if t is not None and t.shape[0] >= n:
        return t
    return make(max(n, 0 if t is None else 2 * t.shape[0], 1))


class FaceLandmark:
    def __init__(self, cfg=None, max_faces=16, device="cuda"):
        """cfg: Skps.yml's Keypoints section (None: read it from Skps.yml).  max_faces: faces per network forward; the
        Student@256 plan holds about 47 MB of activations per face of it.  Calls of run_batch / submit take any number
        of faces and run them in chunks of at most max_faces."""
        if cfg is None:
            from .facer import get_cfg
            cfg = get_cfg()['Skps']['Keypoints']
        root_path = pathlib.Path(__file__).resolve().parents[2]
        model_path = os.path.join(root_path, cfg['model_path'])
        self.max_faces = int(max_faces)
        if self.max_faces < 1:
            raise ValueError("max_faces %d < 1" % self.max_faces)
        self.model = ONNXEngine(model_path, device=device, max_batch=self.max_faces)
        self.device = self.model.device
        self.min_face = MIN_FACE
        self.keypoints_num = cfg['num_points']
        self.input_size = cfg['input_shape']
        self.extend = cfg['base_extend_range']
        self.face_scale = face_scale(cfg)
        self.lib = rt.load_library()
        torch = rt.require_cuda()
        K = self.max_faces
        self._boxes = torch.zeros((K, 4), dtype=torch.float32, device=self.device)
        self._count = torch.zeros((1,), dtype=torch.int32, device=self.device)
        self._detail = torch.zeros((K, 5), dtype=torch.int32, device=self.device)
        self.last_detail = None
        self._slots = None            # staging of the batched path, made on first use
        self._pending = []            # [(slot, faces per frame, out or None)]
        self._next = 0

    def crops(self, img, bboxes):
        """The (K,S,S,3) uint8 crops the network sees (face_landmark.py:66-104), for parity tests."""
        torch = rt.require_cuda()
        bboxes = np.asarray(bboxes, dtype=np.float32).reshape(-1, bboxes.shape[-1] if len(bboxes) else 4)
        n = bboxes.shape[0]
        assert n <= self.max_faces
        frame = torch.from_numpy(np.ascontiguousarray(img)).to(self.model.device)
        h, w = img.shape[:2]
        s = self.model.stream
        s.wait_stream(torch.cuda.current_stream(self.model.device))
        with torch.cuda.stream(s):
            self._boxes[:n].copy_(torch.from_numpy(np.ascontiguousarray(bboxes[:, :4])))
            self._count.fill_(n)
        S = self.input_size[0]
        rt.check(self.lib.skps_crop_resize(frame.data_ptr(), h, w, w * 3, self._boxes.data_ptr(),
                                           self._count.data_ptr(), self.max_faces, self.face_scale,
                                           float(self.min_face), self.model.input_ptr(), S,
                                           self._detail.data_ptr(), s.cuda_stream))
        s.synchronize()
        out = np.empty((self.max_faces, S, S, 3), np.uint8)
        rt.check(self.lib.skps_engine_read_buffer(self.model.handle, self.model.plan.input.buf.idx, self.max_faces,
                                                  out.ctypes.data))
        return out[:n], self._detail[:n].cpu().numpy()

    def __call__(self, img, bboxes):
        t0 = time.time()
        if len(bboxes) == 0:
            return np.array([]), np.array([])
        bboxes = np.asarray(bboxes, dtype=np.float32)
        slot = self._next
        (kps, scores), = self.run_batch([img], [bboxes])
        self.last_detail = self._slots[slot]["detail"][:len(kps)].cpu().numpy()
        duration = time.time() - t0
        logger.info('keypoints done, time consume: %.5f and %.5f per face' % (duration, duration / len(bboxes)))
        return kps, scores

    # ------------------------------------------------------------------ batched path
    def run_batch(self, frames, boxes):
        """Landmarks for the faces the caller has, over many frames (blocking): frames[i] with boxes[i] -> the i-th
        (kps (k_i, 98, 2) float32, scores (k_i, 98) float32) of the returned list, bit for bit what
        FaceLandmark(cfg)(frames[i], boxes[i]) returns.  See submit() for what frames and boxes may be."""
        if self._pending:
            raise RuntimeError("FaceLandmark: %d calls in flight; collect() them first" % len(self._pending))
        self.submit(frames, boxes)
        return self.collect()

    def new_results(self, n_faces):
        """Device result buffers for submit(cuda_frames, boxes, out=...) of up to n_faces faces: a dict of CUDA tensors
        on this object's device, kps (n_faces, 98, 2) and scores (n_faces, 98) float32."""
        torch = rt.require_cuda()
        n, P = int(n_faces), self.keypoints_num
        return {"kps": torch.empty((n, P, 2), dtype=torch.float32, device=self.device),
                "scores": torch.empty((n, P), dtype=torch.float32, device=self.device)}

    def submit(self, frames, boxes, out=None):
        """Enqueue landmarks for boxes[i] on frames[i]; at most two calls may be in flight and collect() returns them in
        submission order.  Everything is checked before anything is enqueued.

        frames: all HxWx3 uint8 BGR numpy arrays, or all torch.uint8 CUDA tensors (H, W, 3) on this object's device with
        stride(2) == 1, stride(1) == 3 and any row pitch (FaceAna.run's frames); a mix raises ValueError.  Sizes may
        differ.  Of a host frame only the rectangle each crop reads crosses PCIe; a CUDA frame is read where it is.
        boxes: one (k_i, >= 4) float array per frame (k_i may be 0); columns 0..3 are x1, y1, x2, y2 and nothing else
        is read or modified.  Host boxes are converted to float32 and must be finite with |value| <= 2**24.  With CUDA
        frames, boxes may also be float32 CUDA tensors (all of them), read on the device.
        Ordering on torch.cuda.current_stream(): CUDA frames and boxes are read after the work already queued on it, and
        work queued on it after submit() returns runs after they have been read.
        out: None (collect() returns numpy arrays), or, with CUDA frames, a dict from new_results(n) with n >= the call's
        faces, not used by a call still in flight: the results are written there on the GPU."""
        if len(self._pending) == 2:
            raise RuntimeError("FaceLandmark: two calls already in flight; call collect() first")
        checked = self._check_call(frames, boxes)
        if out is not None:
            if not checked[3]:
                raise ValueError("out= keeps results on the GPU and takes CUDA frames; these are host frames")
            self._check_out(out, sum(checked[5]))
        slot = self._enqueue(checked, out)
        self._pending.append((slot, checked[5], out))

    def _enqueue_to(self, frames, boxes, out):
        """submit() with results left in out (a new_results(n) dict) for host frames as well as CUDA frames, and not
        counted as a call in flight: FaceAnaImages orders its own work after it on the engine's stream.  Returns the
        faces per frame."""
        checked = self._check_call(frames, boxes)
        self._check_out(out, sum(checked[5]))
        self._enqueue(checked, out)
        return checked[5]

    def _check_call(self, frames, boxes):
        """Checks the frames and boxes of a call: (frames, boxes, layout, cuda frames, cuda boxes, faces per frame)."""
        frames, boxes = list(frames), list(boxes)
        if len(frames) != len(boxes):
            raise ValueError("%d frames but %d box arrays" % (len(frames), len(boxes)))
        on_dev = [is_cuda_tensor(f) for f in frames]
        cuda = bool(on_dev) and all(on_dev)
        if any(on_dev) and not cuda:
            raise ValueError("one call takes either host frames or CUDA frames, got both (frames %s are CUDA)"
                             % [i for i, d in enumerate(on_dev) if d])
        if cuda:
            layout = [check_cuda_frame(f, self.device, (MAX_SIDE, MAX_SIDE)) for f in frames]
        else:
            frames = [check_host_frame(f) for f in frames]
            layout = [(f.shape[0], f.shape[1], 3 * f.shape[1]) for f in frames]
        for H, W, _ in layout:
            if not (0 < H <= MAX_SIDE and 0 < W <= MAX_SIDE):
                raise ValueError("frame %dx%d: sides must be in 1..%d" % (H, W, MAX_SIDE))
        box_dev = [is_cuda_tensor(b) for b in boxes]
        cuda_boxes = bool(box_dev) and all(box_dev)
        if any(box_dev) and not cuda_boxes:
            raise ValueError("boxes are either all host arrays or all CUDA tensors (boxes %s are CUDA)"
                             % [i for i, d in enumerate(box_dev) if d])
        if cuda_boxes and not cuda:
            raise ValueError("CUDA boxes take CUDA frames: the host frames' upload is cut to the boxes on the host")
        boxes = [self._check_cuda_boxes(b, i) if cuda_boxes else self._check_host_boxes(b, i) for i, b in enumerate(boxes)]
        counts = [int(b.shape[0]) for b in boxes]
        return frames, boxes, layout, cuda, cuda_boxes, counts

    def _enqueue(self, checked, out):
        """Stages a checked call into the next slot and enqueues crops, network and post-processing (and, without out,
        the copy back) on the engine's stream; returns the slot."""
        torch = rt.require_cuda()
        frames, boxes, layout, cuda, cuda_boxes, counts = checked
        n = sum(counts)
        P = self.keypoints_num
        if self._slots is None:
            self._slots = [self._new_slot() for _ in range(2)]
        slot = self._next
        st = self._slots[slot]
        rects = None if cuda else [crop_read_rects(b, H, W, self.face_scale, self.min_face)
                                   for b, (H, W, _) in zip(boxes, layout)]
        roi_bytes = 0 if cuda else [(r[:, 2] - r[:, 0]) * (r[:, 3] - r[:, 1]) * 3 for r in rects]
        box_off = (n * FACE_SRC.itemsize + 15) // 16 * 16
        roi_off = box_off + (n * 16 + 15) // 16 * 16
        total = roi_off + (0 if cuda else int(sum(int(r.sum()) for r in roi_bytes)))
        sent = box_off if cuda_boxes else total       # bytes of the host staging the call sends
        if (st["host"] is None or st["host"].shape[0] < total or st["kps"] is None or st["kps"].shape[0] < n):
            st["done"].synchronize()                  # the slot's last call has finished with what is replaced
            st["host"] = _grow(st["host"], total, lambda k: torch.empty((k,), dtype=torch.uint8).pin_memory())
            st["dev"] = _grow(st["dev"], total, lambda k: torch.empty((k,), dtype=torch.uint8, device=self.device))
            st["kps"] = _grow(st["kps"], n, lambda k: torch.empty((k, P, 2), dtype=torch.float32, device=self.device))
            st["scores"] = _grow(st["scores"], n, lambda k: torch.empty((k, P), dtype=torch.float32, device=self.device))
            st["detail"] = _grow(st["detail"], n, lambda k: torch.empty((k, 5), dtype=torch.int32, device=self.device))
            st["hkps"] = _grow(st["hkps"], n, lambda k: torch.empty((k, P, 2), dtype=torch.float32).pin_memory())
            st["hscores"] = _grow(st["hscores"], n, lambda k: torch.empty((k, P), dtype=torch.float32).pin_memory())
        st["copied"].synchronize()                    # the slot's last upload has left the pinned staging
        host = st["host"].numpy()
        dev = st["dev"].data_ptr()
        # host staging = [n face descriptors | n boxes | the host frames' rectangles], sent with one copy
        desc = host[:n * FACE_SRC.itemsize].view(FACE_SRC)
        o, at = 0, roi_off
        for i, (f, (H, W, pitch), k) in enumerate(zip(frames, layout, counts)):
            if k == 0:
                continue
            d = desc[o:o + k]
            d["H"], d["W"], d["_pad"] = H, W, 0
            if not cuda_boxes:
                host[box_off + 16 * o:box_off + 16 * (o + k)].view(np.float32).reshape(k, 4)[:] = boxes[i]
            if cuda:
                d["base"], d["pitch"], d["ox"], d["oy"], d["rw"], d["rh"] = f.data_ptr(), pitch, 0, 0, W, H
            else:
                r, nb = rects[i], roi_bytes[i]
                starts = at + np.concatenate(([0], np.cumsum(nb)[:-1]))
                rw, rh = r[:, 2] - r[:, 0], r[:, 3] - r[:, 1]
                d["base"], d["pitch"], d["ox"], d["oy"], d["rw"], d["rh"] = dev + starts, 3 * rw, r[:, 0], r[:, 1], rw, rh
                for j in np.flatnonzero(nb):
                    x0, y0, x1, y1 = (int(v) for v in r[j])
                    host[starts[j]:starts[j] + nb[j]].reshape(y1 - y0, 3 * (x1 - x0))[:] = \
                        f[y0:y1, x0:x1].reshape(y1 - y0, 3 * (x1 - x0))
                at += int(nb.sum())
            o += k

        s, cp = self.model.stream, st["copy"]
        if sent:
            cp.wait_event(st["read"])                 # the slot's last crops have read its device staging
            with torch.cuda.stream(cp):
                st["dev"][:sent].copy_(st["host"][:sent], non_blocking=True)
        st["copied"].record(cp)
        s.wait_stream(torch.cuda.current_stream(self.device))
        s.wait_event(st["copied"])
        if cuda_boxes and n:
            with torch.cuda.stream(s):
                dst = st["dev"][box_off:box_off + 16 * n].view(torch.float32).view(n, 4)
                torch.cat([b[:, :4] for b in boxes if b.shape[0]], out=dst)
        kps = out["kps"] if out is not None else st["kps"]
        scores = out["scores"] if out is not None else st["scores"]
        K, S = self.max_faces, self.input_size[0]
        inp = self.model.input_ptr()
        det = st["detail"].data_ptr()
        for c0 in range(0, n, K):
            m = min(K, n - c0)
            rt.check(self.lib.skps_crop_faces(dev + FACE_SRC.itemsize * c0, dev + box_off + 16 * c0, m, self.face_scale,
                                              float(self.min_face), inp, S, det + 20 * c0, s.cuda_stream))
            if c0 + K >= n:
                st["read"].record(s)
            outs = (C.c_void_p * 2)(None, scores.data_ptr() + 4 * P * c0)
            rt.check(self.lib.skps_engine_forward(self.model.handle, inp, m, outs, s.cuda_stream))
            rt.check(self.lib.skps_landmark_post(self.model.output_ptr(0), det + 20 * c0, st["count"].data_ptr(), m, P,
                                                 kps.data_ptr() + 8 * P * c0, s.cuda_stream))
        if n == 0:
            st["read"].record(s)
        torch.cuda.current_stream(self.device).wait_event(st["read"])
        if out is None and n:
            with torch.cuda.stream(s):
                st["hkps"][:n].copy_(kps[:n], non_blocking=True)
                st["hscores"][:n].copy_(scores[:n], non_blocking=True)
        st["done"].record(s)
        self._next ^= 1
        return slot

    def collect(self):
        """Results of the oldest call in flight: a list with one (kps (k_i, 98, 2), scores (k_i, 98)) pair per frame, as
        float32 numpy arrays; for a call submitted with out=, views of out's rows, with no host synchronisation:
        torch.cuda.current_stream() is made to wait for the call, so work queued on it afterwards sees the results."""
        if not self._pending:
            raise RuntimeError("FaceLandmark: nothing submitted")
        slot, counts, out = self._pending.pop(0)
        st = self._slots[slot]
        if out is not None:
            import torch
            torch.cuda.current_stream(self.device).wait_event(st["done"])
            kps, scores = out["kps"], out["scores"]
        else:
            st["done"].synchronize()
            kps, scores = st["hkps"].numpy(), st["hscores"].numpy()
        res, o = [], 0
        for k in counts:
            if out is None:
                res.append((kps[o:o + k].copy(), scores[o:o + k].copy()))
            else:
                res.append((kps[o:o + k], scores[o:o + k]))
            o += k
        return res

    def _new_slot(self):
        import torch
        ev = {name: torch.cuda.Event() for name in ("copied", "read", "done")}
        return dict(copy=torch.cuda.Stream(device=self.device), host=None, dev=None, kps=None, scores=None, detail=None,
                    hkps=None, hscores=None, count=torch.full((1,), self.max_faces, dtype=torch.int32, device=self.device),
                    **ev)

    @staticmethod
    def _check_host_boxes(b, i):
        b = np.asarray(b, dtype=np.float32)
        if b.size == 0:
            return np.zeros((0, 4), np.float32)
        if b.ndim != 2 or b.shape[1] < 4:
            raise ValueError("boxes[%d]: expected a (k, >= 4) array, got shape %s" % (i, b.shape))
        xy = b[:, :4]
        if not np.isfinite(xy).all() or np.abs(xy).max() > BOX_LIMIT:
            raise ValueError("boxes[%d]: coordinates must be finite with |value| <= 2**24" % i)
        return xy

    def _check_cuda_boxes(self, b, i):
        import torch
        if b.dtype != torch.float32 or b.device != self.device:
            raise ValueError("boxes[%d]: expected float32 on %s, got %s on %s" % (i, self.device, b.dtype, b.device))
        if b.numel() == 0:
            return b.reshape(0, 4)
        if b.dim() != 2 or b.shape[1] < 4:
            raise ValueError("boxes[%d]: expected a (k, >= 4) tensor, got shape %s" % (i, tuple(b.shape)))
        return b

    def _check_out(self, out, n):
        import torch
        P = self.keypoints_num
        if not isinstance(out, dict) or set(out) != {"kps", "scores"}:
            raise ValueError("out: expected a dict with keys ['kps', 'scores'] (see new_results())")
        for k, tail in (("kps", (P, 2)), ("scores", (P,))):
            t = out[k]
            if (not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.device != self.device
                    or not t.is_contiguous() or tuple(t.shape[1:]) != tail or t.shape[0] < n):
                got = ("%s %s on %s" % (t.dtype, tuple(t.shape), t.device)) if is_tensor(t) else type(t).__name__
                raise ValueError("out[%r]: expected a contiguous float32 tensor (>= %d, %s) on %s, got %s"
                                 % (k, n, ", ".join(map(str, tail)), self.device, got))
        busy = {t.data_ptr() for _, _, o in self._pending if o is not None for t in o.values()}
        if any(t.data_ptr() in busy for t in out.values()):
            raise ValueError("out: these buffers belong to a call still in flight; collect() it first")
