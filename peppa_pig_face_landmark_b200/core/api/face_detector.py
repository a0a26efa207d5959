"""FaceDetector — same surface as the reference's Skps/core/api/face_detector.py:11-136
(`FaceDetector(cfg)(image) -> (K,16) float32`), with letterbox, the yolov5-face network,
score filter + greedy NMS and the un-letterbox all executed on the GPU by the kernels behind
include/skps_b200.h.  Host code only computes the letterbox geometry (python floats, exactly
as face_detector.py:51-62) and owns the containers.

Additive: the detector over many frames per call (SURVEY.md 8b):

    fd = FaceDetector(max_frames=16)
    res = fd.run_batch(frames)             # [(k_i, 16) float32 per frame], host frames or CUDA frames of any sizes
    # overlapped, results left on the GPU (CUDA frames):
    bufs = [fd.new_results(n), fd.new_results(n)]
    fd.submit(frames_0, out=bufs[0]); fd.submit(frames_1, out=bufs[1]); r0 = fd.collect(); ...
"""
import os
import pathlib
import time

import numpy as np

from ... import runtime as rt
from ...graph_tools import detector_onnx_for
from ...logger.logger import logger
from .device_frames import check_cuda_frame, check_host_frame, is_cuda_tensor, is_tensor
from .onnx_model_base import ONNXEngine

MAX_SIDE = 1 << 20         # largest frame side submit takes: keeps every row pitch in int32

# skps_det_src of include/skps_b200.h
DET_SRC = np.dtype([("base", "<u8"), ("pitch", "<i4"), ("H", "<i4"), ("W", "<i4"), ("rw", "<i4"), ("rh", "<i4"),
                    ("top", "<i4"), ("left", "<i4"), ("row_pairs", "<i4")])
assert DET_SRC.itemsize == 40


def letterbox_geometry(h, w, in_h, in_w):
    """face_detector.py:51-62."""
    scale = min(in_h / h, in_w / w)
    rw, rh = int(w * scale), int(h * scale)
    dh = (in_h - rh) / 2
    dw = (in_w - rw) / 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    if rh + top + bottom != in_h or rw + left + right != in_w:
        # the reference would feed a wrongly sized tensor to the fixed-size graph and fail in np.reshape
        raise ValueError("letterbox of %dx%d does not fill %dx%d" % (h, w, in_h, in_w))
    return scale, rw, rh, top, left


def letterbox_rows(H, rh):
    """(2 rh,) int64: the frame rows resized row y reads, as the pair [i0, i1] at 2y, 2y + 1 (skps_det_src's row_pairs
    layout).  The vertical tap of linear_tap in image_ops.cu (cv2.resize INTER_LINEAR): float32 source position of
    ((y + 0.5) / (rh / H) - 0.5) in double, its floor and the next row, both clamped to the frame.  Row i1 is listed even
    where its weight is 0: the kernel reads it."""
    y = np.arange(rh, dtype=np.float64)
    f = ((y + 0.5) * (1.0 / (rh / H)) - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    return np.stack([np.clip(s, 0, H - 1), np.clip(s + 1, 0, H - 1)], 1).reshape(-1)


def host_upload_rows(H, rh):
    """The rows of an H-row host frame FaceDetector sends for a letterbox of rh rows: letterbox_rows(H, rh) when that is
    fewer rows than the frame (2 rh < H), else None (the whole frame)."""
    return letterbox_rows(H, rh) if 2 * rh < H else None


def _grow(t, n, make):
    """t when it holds n elements, else make(max(n, 2 * len(t)))."""
    if t is not None and t.shape[0] >= n:
        return t
    return make(max(n, 0 if t is None else 2 * t.shape[0], 1))


def _pad16(n):
    return (n + 15) // 16 * 16


class FaceDetector:
    MAX_DET = 256           # kept rows per frame copied back with the counts (the rest only for frames that keep more)

    def __init__(self, cfg=None, max_frames=16, device="cuda"):
        """cfg: Skps.yml's Detect section (None: read it from Skps.yml).  The engine is built for cfg['input_shape']
        ([h, w, 3]): from the export itself when that is its input size, else from the export retargeted to (h, w)
        (graph_tools.detector_onnx_for; h and w multiples of 32 in 128..2176 x 128..3840), so the letterbox and the
        network always agree on the size.

        max_frames: frames per network forward.  Calls of run_batch / submit take any number of frames and run them in
        chunks of at most max_frames.  Memory: the engine holds about 39 MB of activations per frame of max_frames at
        384x640 and 0.35 GB at 1152x1920, plus an NMS workspace of skps_detect_post_workspace_size(rows, max_frames)
        bytes (rows = 15120 at 384x640).  Each of the two call slots keeps, per frame of its largest call, every
        detector row as a possible kept box (rows x 68 bytes, about 1 MB at 384x640) and, for host frames, the pinned
        staging of the rows it uploads."""
        if cfg is None:
            from .facer import get_cfg
            cfg = get_cfg()['Skps']['Detect']
        root_path = pathlib.Path(__file__).resolve().parents[2]
        model_path = os.path.join(root_path, cfg['model_path'])
        self.max_frames = int(max_frames)
        if self.max_frames < 1:
            raise ValueError("max_frames %d < 1" % self.max_frames)
        self.input_size = cfg['input_shape']
        self.model = ONNXEngine(detector_onnx_for(model_path, self.input_size[:2]), device=device,
                                max_batch=self.max_frames)
        self.device = self.model.device
        self.score_thrs = cfg['score_thrs']
        self.iou_thrs = cfg['iou_thrs']
        self.lib = rt.load_library()
        torch = rt.require_cuda()
        self._rows = self.model.out_elems[0] // 16
        self._ws_bytes = self.lib.skps_detect_post_workspace_size(self._rows, self.max_frames)
        self._ws = torch.empty((self._ws_bytes,), dtype=torch.uint8, device=self.device)
        self.last_keep_idx = None
        self._slots = None            # staging and results of the two call slots, made on first use
        self._pending = []            # [(slot, frames, out or None)]
        self._next = 0

    # ------------------------------------------------------------------ reference contract
    def preprocess(self, image, color=(114, 114, 114)):
        """face_detector.py:45-71: returns ((1,3,H,W) float32 RGB/255, [scale, left, top])."""
        if self._pending:
            raise RuntimeError("FaceDetector: %d calls in flight; collect() them first" % len(self._pending))
        image = check_host_frame(image)
        h, w = image.shape[:2]
        in_h, in_w = self.input_size[0], self.input_size[1]
        scale, rw, rh, top, left = letterbox_geometry(h, w, in_h, in_w)
        st = self._enqueue([image], None, detect=False)
        st["done"].synchronize()
        u8 = np.empty((in_h, in_w, 3), np.uint8)
        rt.check(self.lib.skps_engine_read_buffer(self.model.handle, self.model.plan.input.buf.idx, 1, u8.ctypes.data))
        img = u8.transpose(2, 0, 1).astype(np.float32)
        img /= 255.0
        return np.expand_dims(img, axis=0), [scale, left, top]

    def __call__(self, image):
        t0 = time.time()
        bboxes, = self.run_batch([image])
        self.last_keep_idx = self.last_keep_idx[0]
        logger.info('detect done, time consume: %.5f' % (time.time() - t0))
        return bboxes

    # ------------------------------------------------------------------ batched path
    def run_batch(self, frames):
        """The detector over many frames (blocking): the i-th (k_i, 16) float32 array of the returned list is bit for bit
        what FaceDetector(cfg)(frames[i]) returns; last_keep_idx is then the list of the frames' kept row indices (int64).
        See submit() for what frames may be."""
        if self._pending:
            raise RuntimeError("FaceDetector: %d calls in flight; collect() them first" % len(self._pending))
        self.submit(frames)
        return self.collect()

    def new_results(self, n_frames):
        """Device result buffers for submit(cuda_frames, out=...) of up to n_frames frames: a dict of CUDA tensors on
        this object's device, rows (n, R, 16) float32, idx (n, R) int32 and count (n,) int32, where R is the detector's
        row count (15120 at 384x640): frame i keeps rows[i, :count[i]], the detector rows idx[i, :count[i]]."""
        torch = rt.require_cuda()
        n, R = int(n_frames), self._rows
        return {"rows": torch.empty((n, R, 16), dtype=torch.float32, device=self.device),
                "idx": torch.empty((n, R), dtype=torch.int32, device=self.device),
                "count": torch.empty((n,), dtype=torch.int32, device=self.device)}

    def submit(self, frames, out=None):
        """Enqueue the detector on frames; at most two calls may be in flight and collect() returns them in submission
        order.  Everything is checked before anything is enqueued.

        frames: all HxWx3 uint8 BGR numpy arrays, or all torch.uint8 CUDA tensors (H, W, 3) on this object's device with
        stride(2) == 1, stride(1) == 3 and any row pitch (FaceAna.run's frames); a mix raises ValueError.  Sizes may
        differ, as long as their letterbox fills the input (letterbox_geometry).  A host frame sends only the rows the
        letterbox reads when that is fewer than its rows (host_upload_rows), else the whole frame; a CUDA frame is read
        where it is.
        Ordering on torch.cuda.current_stream(): CUDA frames are read after the work already queued on it, and work
        queued on it after submit() returns runs after they have been read.
        out: None (collect() returns numpy arrays), or, with CUDA frames, a dict from new_results(n) with n >= the call's
        frames, not used by a call still in flight: the kept rows, their indices and counts are written there on the
        GPU."""
        if len(self._pending) == 2:
            raise RuntimeError("FaceDetector: two calls already in flight; call collect() first")
        frames = list(frames)
        if out is not None:
            if not (frames and all(is_cuda_tensor(f) for f in frames)):
                raise ValueError("out= keeps results on the GPU and takes CUDA frames")
            self._check_out(out, len(frames))
        slot = self._next
        self._enqueue(frames, out, detect=True)
        self._pending.append((slot, len(frames), out))

    def collect(self):
        """Results of the oldest call in flight: a list with one (k_i, 16) float32 numpy array per frame, and
        last_keep_idx the list of their kept row indices; for a call submitted with out=, the out dict, with no host
        synchronisation: torch.cuda.current_stream() is made to wait for the call, so work queued on it afterwards sees
        the results."""
        if not self._pending:
            raise RuntimeError("FaceDetector: nothing submitted")
        slot, n, out = self._pending.pop(0)
        st = self._slots[slot]
        if out is not None:
            import torch
            torch.cuda.current_stream(self.device).wait_event(st["done"])
            return out
        st["done"].synchronize()
        M = min(self.MAX_DET, self._rows)
        count = st["hcount"].numpy()[:n]
        hrows, hidx = st["hrows"].numpy(), st["hidx"].numpy()
        res, keep = [], []
        for i, k in enumerate(count.tolist()):
            if k <= M:
                res.append(hrows[i, :k].copy())
                keep.append(hidx[i, :k].astype(np.int64))
            else:
                # a crowd: the first M kept rows came back with the counts, the device holds all of them
                res.append(st["rows"][i, :k].cpu().numpy())
                keep.append(st["idx"][i, :k].cpu().numpy().astype(np.int64))
        self.last_keep_idx = keep
        return res

    # ------------------------------------------------------------------
    def _layout(self, frames):
        """Checks every frame; [(H, W, row pitch, geometry, rows uploaded or None)] and whether they are CUDA frames."""
        on_dev = [is_cuda_tensor(f) for f in frames]
        cuda = bool(on_dev) and all(on_dev)
        if any(on_dev) and not cuda:
            raise ValueError("one call takes either host frames or CUDA frames, got both (frames %s are CUDA)"
                             % [i for i, d in enumerate(on_dev) if d])
        if cuda:
            shapes = [check_cuda_frame(f, self.device, (MAX_SIDE, MAX_SIDE)) for f in frames]
        else:
            frames = [check_host_frame(f) for f in frames]
            shapes = [(f.shape[0], f.shape[1], 3 * f.shape[1]) for f in frames]
        in_h, in_w = self.input_size[0], self.input_size[1]
        layout = []
        for H, W, pitch in shapes:
            if not (0 < H <= MAX_SIDE and 0 < W <= MAX_SIDE):
                raise ValueError("frame %dx%d: sides must be in 1..%d" % (H, W, MAX_SIDE))
            geo = letterbox_geometry(H, W, in_h, in_w)
            if geo[1] < 1 or geo[2] < 1:
                raise ValueError("frame %dx%d: its letterbox at %dx%d is %dx%d, empty" % (H, W, in_h, in_w, geo[2], geo[1]))
            layout.append((H, W, pitch, geo, None if cuda else host_upload_rows(H, geo[2])))
        return frames, layout, cuda

    def _enqueue(self, frames, out, detect, checked=None):
        """Stages the frames into the next slot and enqueues letterbox (and, with detect, network, NMS and the copy back
        of host results) on the engine's stream; returns the slot.  out: None, or result buffers of new_results(n) the
        kept rows go to, for host frames as well as CUDA frames (FaceAnaImages keeps them on the GPU); nothing is then
        copied back.  checked: what _layout(frames) returned, when the caller has checked the frames already."""
        torch = rt.require_cuda()
        frames, layout, cuda = self._layout(frames) if checked is None else checked
        n, R, M = len(frames), self._rows, min(self.MAX_DET, self._rows)
        if self._slots is None:
            self._slots = [self._new_slot() for _ in range(2)]
        slot = self._next
        st = self._slots[slot]
        rec_off = _pad16(n * DET_SRC.itemsize)
        frame_off = rec_off + _pad16(n * 12)
        sizes = [0 if cuda else _pad16((H if rows is None else len(rows)) * pitch) for H, W, pitch, geo, rows in layout]
        total = frame_off + sum(sizes)
        own = detect and out is None                  # results go to the slot's buffers and come back to the host
        if st["host"] is None or st["host"].shape[0] < total:
            st["done"].synchronize()                  # the slot's last call has finished with what is replaced
            st["host"] = _grow(st["host"], total, lambda k: torch.empty((k,), dtype=torch.uint8).pin_memory())
            st["dev"] = _grow(st["dev"], total, lambda k: torch.empty((k,), dtype=torch.uint8, device=self.device))
        if own and (st["rows"] is None or st["rows"].shape[0] < n):
            st["done"].synchronize()
            st["rows"] = _grow(st["rows"], n, lambda k: torch.empty((k, R, 16), dtype=torch.float32, device=self.device))
            st["idx"] = _grow(st["idx"], n, lambda k: torch.empty((k, R), dtype=torch.int32, device=self.device))
            st["count"] = _grow(st["count"], n, lambda k: torch.empty((k,), dtype=torch.int32, device=self.device))
            st["hrows"] = _grow(st["hrows"], n, lambda k: torch.empty((k, M, 16), dtype=torch.float32).pin_memory())
            st["hidx"] = _grow(st["hidx"], n, lambda k: torch.empty((k, M), dtype=torch.int32).pin_memory())
            st["hcount"] = _grow(st["hcount"], n, lambda k: torch.empty((k,), dtype=torch.int32).pin_memory())
        st["copied"].synchronize()                    # the slot's last upload has left the pinned staging
        host = st["host"].numpy()
        dev = st["dev"].data_ptr()
        # host staging = [n frame descriptors | n (scale, left, top) | the host frames' rows], sent with one copy
        desc = host[:n * DET_SRC.itemsize].view(DET_SRC)
        rec = host[rec_off:rec_off + 12 * n].view(np.float32).reshape(n, 3)
        at = frame_off
        for i, (f, (H, W, pitch, (scale, rw, rh, top, left), rows), nb) in enumerate(zip(frames, layout, sizes)):
            rec[i] = (scale, left, top)
            d = desc[i:i + 1]
            d["H"], d["W"], d["rw"], d["rh"], d["top"], d["left"] = H, W, rw, rh, top, left
            d["pitch"], d["row_pairs"] = pitch, int(rows is not None)
            if cuda:
                d["base"] = f.data_ptr()
                continue
            d["base"] = dev + at
            if rows is None:
                host[at:at + H * pitch] = f.reshape(-1)
            else:
                np.take(f.reshape(H, pitch), rows, axis=0, out=host[at:at + len(rows) * pitch].reshape(-1, pitch),
                        mode="clip")
            at += nb

        s, cp = self.model.stream, st["copy"]
        sent = frame_off if cuda else total
        if sent:
            cp.wait_event(st["done"])                 # the slot's last call has read its device staging (NMS reads recover)
            with torch.cuda.stream(cp):
                st["dev"][:sent].copy_(st["host"][:sent], non_blocking=True)
        st["copied"].record(cp)
        s.wait_stream(torch.cuda.current_stream(self.device))
        s.wait_event(st["copied"])
        res = out if out is not None else st
        rows_t, idx_t, count_t = res["rows"], res["idx"], res["count"]
        K = self.max_frames
        in_h, in_w = self.input_size[0], self.input_size[1]
        inp = self.model.input_ptr()
        for c0 in range(0, n, K):
            m = min(K, n - c0)
            rt.check(self.lib.skps_letterbox_frames(dev + DET_SRC.itemsize * c0, m, inp, in_h, in_w, s.cuda_stream))
            if c0 + K >= n:
                st["read"].record(s)
            if not detect:
                continue
            rt.check(self.lib.skps_engine_forward(self.model.handle, inp, m, None, s.cuda_stream))
            rt.check(self.lib.skps_detect_post_batch(self.model.output_ptr(0), R, m, self.score_thrs, self.iou_thrs,
                                                     dev + rec_off + 12 * c0, rows_t.data_ptr() + 64 * R * c0,
                                                     idx_t.data_ptr() + 4 * R * c0, count_t.data_ptr() + 4 * c0, R,
                                                     self._ws.data_ptr(), self._ws_bytes, s.cuda_stream))
        if n == 0:
            st["read"].record(s)
        torch.cuda.current_stream(self.device).wait_event(st["read"])
        if own and n:
            with torch.cuda.stream(s):
                st["hrows"][:n].copy_(rows_t[:n, :M], non_blocking=True)
                st["hidx"][:n].copy_(idx_t[:n, :M], non_blocking=True)
                st["hcount"][:n].copy_(count_t[:n], non_blocking=True)
        st["done"].record(s)
        self._next ^= 1
        return st

    def _new_slot(self):
        import torch
        ev = {name: torch.cuda.Event() for name in ("copied", "read", "done")}
        return dict(copy=torch.cuda.Stream(device=self.device), host=None, dev=None, rows=None, idx=None, count=None,
                    hrows=None, hidx=None, hcount=None, **ev)

    def _check_out(self, out, n):
        import torch
        R = self._rows
        if not isinstance(out, dict) or set(out) != {"rows", "idx", "count"}:
            raise ValueError("out: expected a dict with keys ['count', 'idx', 'rows'] (see new_results())")
        for k, dt, tail in (("rows", torch.float32, (R, 16)), ("idx", torch.int32, (R,)), ("count", torch.int32, ())):
            t = out[k]
            if (not isinstance(t, torch.Tensor) or t.dtype != dt or t.device != self.device or not t.is_contiguous()
                    or t.dim() != 1 + len(tail) or tuple(t.shape[1:]) != tail or t.shape[0] < n):
                got = ("%s %s on %s" % (t.dtype, tuple(t.shape), t.device)) if is_tensor(t) else type(t).__name__
                raise ValueError("out[%r]: expected a contiguous %s tensor (>= %d%s) on %s, got %s"
                                 % (k, dt, n, "".join(", %d" % v for v in tail), self.device, got))
        busy = {t.data_ptr() for _, _, o in self._pending if o is not None for t in o.values()}
        if any(t.data_ptr() in busy for t in out.values()):
            raise ValueError("out: these buffers belong to a call still in flight; collect() it first")
