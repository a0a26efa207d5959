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
    # ArcFace chips from the detector's own five landmarks, for a recognition model without the landmark net:
    fd = FaceDetector(align=112)
    res = fd.run_batch(frames)             # [(rows, points (k_i,5,2), chips (k_i,112,112,3) uint8, M (k_i,2,3)) per frame]
"""
import os
import pathlib
import time

import numpy as np

from ... import runtime as rt
from ...graph_tools import detector_onnx_for
from ...logger.logger import logger
from .align import check_size
from .device_frames import FRAME_LAYOUT, check_host_frame
from .face_landmark import FACE_SRC, HostChips
from .onnx_model_base import ONNXEngine
from .staging import Staging, check_frames, check_out, grow, new_buffers, pad16

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


MAX_CHIPS = 1024            # largest max_chips


def check_max_chips(max_chips):
    """Chips per frame: an int in 1..MAX_CHIPS (ValueError otherwise)."""
    if isinstance(max_chips, (bool, np.bool_)) or not isinstance(max_chips, (int, np.integer)) \
            or not 1 <= max_chips <= MAX_CHIPS:
        raise ValueError("max_chips must be an int in 1..%d, got %r" % (MAX_CHIPS, max_chips))
    return int(max_chips)


def landmark_points(rows, recover):
    """(k, 5, 2) float32: the five landmarks of kept rows (k, 16) float32 (columns 5..14, letterbox coordinates) in frame
    pixels, with the letterbox's recover = [scale, left, top]: what scale_coords (face_detector.py:82-93) does to columns
    0..3, in the same float32 arithmetic, so that the points and the box share one frame.  The host restatement of
    skps_det_align_estimate's points."""
    scale, left, top = recover
    p = np.array(rows, np.float32).reshape(-1, 16)[:, 5:15].reshape(-1, 5, 2)
    p[:, :, 0] -= np.float32(left)
    p[:, :, 1] -= np.float32(top)
    p /= np.float32(scale)
    return p


def result_fields(n_frames, rows, align=None, max_chips=None):
    """{name: (shape, dtype name)} of new_results(n_frames) of FaceDetector(align=align, max_chips=max_chips) with `rows`
    rows."""
    f = {"rows": ((n_frames, rows, 16), "float32"), "idx": ((n_frames, rows), "int32"),
         "count": ((n_frames,), "int32")}
    if align is not None:
        f.update({"points": ((n_frames, max_chips, 5, 2), "float32"), "M": ((n_frames, max_chips, 2, 3), "float64"),
                  "chip": ((n_frames, max_chips, align, align, 3), "uint8")})
    return f


def align_results(rows, count, points, chips, M, max_chips):
    """collect()'s list with align: (rows[i], points[i, :k], chips of frame i, M[i, :k]) per frame i, as copies, with
    k = min(count[i], max_chips).  points (n, max_chips, 5, 2) and M (n, max_chips, 2, 3) hold a slot per chip; chips
    (>= sum k, s, s, 3) holds them packed in frame order."""
    res, o = [], 0
    for i, c in enumerate(count):
        k = min(int(c), max_chips)
        res.append((rows[i], points[i, :k].copy(), chips[o:o + k].copy(), M[i, :k].copy()))
        o += k
    return res


class FaceDetector:
    MAX_DET = 256           # kept rows per frame copied back with the counts (the rest only for frames that keep more)

    def __init__(self, cfg=None, max_frames=16, device="cuda", align=None, max_chips=64):
        """cfg: Skps.yml's Detect section (None: read it from Skps.yml).  The engine is built for cfg['input_shape']
        ([h, w, 3]): from the export itself when that is its input size, else from the export retargeted to (h, w)
        (graph_tools.detector_onnx_for; h and w multiples of 32 in 128..2176 x 128..3840), so the letterbox and the
        network always agree on the size.

        max_frames: frames per network forward.  Calls of run_batch / submit take any number of frames and run them in
        chunks of at most max_frames.  Memory: the engine holds about 39 MB of activations per frame of max_frames at
        384x640 and 0.35 GB at 1152x1920, plus an NMS workspace of skps_detect_post_workspace_size(rows, max_frames)
        bytes (rows = 15120 at 384x640).  Each of the two call slots keeps, per frame of its largest call, every
        detector row as a possible kept box (rows x 68 bytes, about 1 MB at 384x640) and, for host frames, the pinned
        staging of the rows it uploads.

        align: None, or a chip side in 16..512: run_batch / collect then return, per frame, (rows, points, chips, M)
        for the first min(count, max_chips) kept rows, in NMS order (score descending): points (k, 5, 2) float32, the
        row's five landmarks (eyes, nose tip, mouth corners) mapped back to the frame the way scale_coords maps the box
        (landmark_points; the rows themselves keep them in letterbox coordinates, as the reference does); M (k, 2, 3)
        float64, the similarity from the points promoted to float64 to the ArcFace template scaled by align/112, the
        estimator of core/api/align.py:align_faces; chips (k, align, align, 3) uint8 BGR, cv2.warpAffine(frame, M,
        (align, align)) byte for byte.  max_chips: chips per frame, an int in 1..1024.  Each call slot then keeps
        max_chips x align^2 x 3 bytes of chips on the device per frame of its largest call with CUDA frames (38.5 MB
        for a call of 16 frames at the default max_chips and align 112), and the points and matrices (88 bytes per chip
        slot) on the device and pinned.  A bad align or max_chips raises ValueError before anything is allocated."""
        self.align = None if align is None else check_size(align)
        self.max_chips = check_max_chips(max_chips)
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
        self._pending = []            # [(slot, frames, out or None, checked host frames to align or None)]
        self._next = 0
        self.host_chips = None if self.align is None else HostChips(self.device, self.align)

    # ------------------------------------------------------------------ reference contract
    def preprocess(self, image, color=(114, 114, 114)):
        """face_detector.py:45-71: returns ((1,3,H,W) float32 RGB/255, [scale, left, top])."""
        if self._pending:
            raise RuntimeError("FaceDetector: %d calls in flight; collect() them first" % len(self._pending))
        call = check_frames([check_host_frame(image)], self.device)
        layout = self._layout(call)
        scale, _, _, top, left = layout[0][3]
        in_h, in_w = self.input_size[0], self.input_size[1]
        st = self._enqueue(call, layout, None, detect=False)
        st["done"].synchronize()
        u8 = np.empty((in_h, in_w, 3), np.uint8)
        rt.check(self.lib.skps_engine_read_buffer(self.model.handle, self.model.plan.input.buf.idx, 1, u8.ctypes.data))
        img = u8.transpose(2, 0, 1).astype(np.float32)
        img /= 255.0
        return np.expand_dims(img, axis=0), [scale, left, top]

    def __call__(self, image):
        t0 = time.time()
        bboxes, = self.run_batch([image])
        if self.align is not None:
            bboxes = bboxes[0]
        self.last_keep_idx = self.last_keep_idx[0]
        logger.info('detect done, time consume: %.5f' % (time.time() - t0))
        return bboxes

    # ------------------------------------------------------------------ batched path
    def run_batch(self, frames, layout="bgr", rotate=0):
        """The detector over many frames (blocking): the i-th (k_i, 16) float32 array of the returned list is bit for bit
        what FaceDetector(cfg)(frames[i]) returns; last_keep_idx is then the list of the frames' kept row indices (int64).
        With align, the i-th entry is (rows, points, chips, M) (see __init__).  See submit() for what frames, layout and
        rotate may be."""
        if self._pending:
            raise RuntimeError("FaceDetector: %d calls in flight; collect() them first" % len(self._pending))
        self.submit(frames, layout=layout, rotate=rotate)
        return self.collect()

    def new_results(self, n_frames):
        """Device result buffers for submit(cuda_frames, out=...) of up to n_frames frames: a dict of CUDA tensors on
        this object's device, rows (n, R, 16) float32, idx (n, R) int32 and count (n,) int32, where R is the detector's
        row count (15120 at 384x640): frame i keeps rows[i, :count[i]], the detector rows idx[i, :count[i]].  With
        align, also points (n, max_chips, 5, 2) float32, M (n, max_chips, 2, 3) float64 and chip
        (n, max_chips, align, align, 3) uint8: slot j < min(count[i], max_chips) of frame i holds row j's; the other
        slots are unspecified."""
        rt.require_cuda()
        return new_buffers(self._fields(int(n_frames)), self.device)

    def _fields(self, n_frames):
        return result_fields(n_frames, self._rows, self.align, self.max_chips)

    def submit(self, frames, out=None, layout="bgr", rotate=0):
        """Enqueue the detector on frames; at most two calls may be in flight and collect() returns them in submission
        order.  Everything is checked before anything is enqueued.

        frames: all HxWx3 uint8 BGR numpy arrays, or all torch.uint8 CUDA tensors (H, W, 3) on this object's device with
        stride(2) == 1, stride(1) == 3 and any row pitch (FaceAna.run's frames); a mix raises ValueError.  Sizes may
        differ, as long as their letterbox fills the input (letterbox_geometry).  A host frame sends only the rows the
        letterbox reads when that is fewer than its rows (host_upload_rows), else the whole frame; a CUDA frame is read
        where it is.
        layout: the pixel layout of all CUDA frames of the call (device_frames.frame_layout): "bgr" (the default), "rgb",
        "bgra", "rgba" (H, W, 4), "bgr_planar" or "rgb_planar" (3, H, W).  The letterbox reads them in place, and the
        results are, bit for bit, those of the same pixels passed as interleaved BGR.  Host frames are BGR only.
        rotate: the clockwise angle in degrees (0, 90, 180 or 270) by which CUDA frames, as stored, must be turned to be
        upright (device_frames.check_rotate), one for the call or one per frame (each photo has its own EXIF
        orientation).  They are read in place, and every result (rows, kept indices, points, M, chips) is in the
        upright frame's pixels, bit for bit that of the upright frame passed as a contiguous tensor.  Host frames take 0.
        Ordering on torch.cuda.current_stream(): CUDA frames are read after the work already queued on it, and work
        queued on it after submit() returns runs after they have been read.
        out: None (collect() returns numpy arrays), or, with CUDA frames, a dict from new_results(n) with n >= the call's
        frames, not used by a call still in flight: the kept rows, their indices and counts (with align, the points,
        matrices and chips) are written there on the GPU.

        With align, CUDA frames are warped into chips on the GPU right after the NMS, with no host synchronisation, and
        are read until then.  Host frames are warped at collect(): the points and M come back with the rows, and only
        the rectangle of the frame each chip reads (core/api/align.py:chip_read_rects) is uploaded and warped.  That is
        one more upload per call, and the host frames must stay unchanged until collect() returns."""
        if len(self._pending) == 2:
            raise RuntimeError("FaceDetector: two calls already in flight; call collect() first")
        call = check_frames(frames, self.device, layout, rotate)
        geo = self._layout(call)
        n = len(call.frames)
        if out is not None:
            if not call.cuda:
                raise ValueError("out= keeps results on the GPU and takes CUDA frames")
            check_out(out, self._fields(n), self.device, [p[2] for p in self._pending])
        slot = self._next
        self._enqueue(call, geo, out, detect=True)
        self._pending.append((slot, n, out, call if self.align is not None and not call.cuda else None))

    def collect(self):
        """Results of the oldest call in flight: a list with one (k_i, 16) float32 numpy array per frame, and
        last_keep_idx the list of their kept row indices; with align, one (rows, points, chips, M) tuple per frame.  For
        a call submitted with out=, the out dict, with no host synchronisation: torch.cuda.current_stream() is made to
        wait for the call, so work queued on it afterwards sees the results.  A call of host frames with align is warped
        here (see submit())."""
        if not self._pending:
            raise RuntimeError("FaceDetector: nothing submitted")
        slot, n, out, host_call = self._pending.pop(0)
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
        if self.align is None:
            return res
        chips = self._chips(st, host_call, count.tolist())
        return align_results(res, count, st["hpoints"].numpy(), chips, st["hM"].numpy(), self.max_chips)

    def _chips(self, st, host_call, count):
        """The chips of a collected call without out=, packed in frame order, min(count[i], max_chips) for frame i: a
        pinned (n, align, align, 3) uint8 array.  CUDA frames were warped into the slot's chips at submit(); host frames
        are warped here."""
        torch = rt.require_cuda()
        A, ks = self.align, [min(k, self.max_chips) for k in count]
        F = sum(ks)
        make = lambda k: torch.empty((k, A, A, 3), dtype=torch.uint8)
        st["hchip"] = grow(st["hchip"], F, lambda k: make(k).pin_memory())
        if host_call is not None:
            if F:
                st["dchip"] = grow(st["dchip"], F, lambda k: make(k).to(self.device))
                hM = st["hM"].numpy()
                M = np.concatenate([hM[i, :k] for i, k in enumerate(ks)])
                self.host_chips.warp(self.lib, self.model.stream, host_call, ks, M, st["dchip"], st["hchip"])
        else:
            cs = st["stage"].copy                     # idle until this slot's next call: the call is done
            with torch.cuda.stream(cs):
                o = 0
                for i, k in enumerate(ks):
                    if k:
                        st["hchip"][o:o + k].copy_(st["chip"][i, :k], non_blocking=True)
                    o += k
            cs.synchronize()
        return st["hchip"].numpy()

    # ------------------------------------------------------------------
    def _layout(self, call):
        """[(H, W, row pitch, letterbox geometry, rows uploaded or None)] of the frames of a call checked by
        check_frames, H, W and pitch as stored, the geometry that of the upright frame; ValueError for a frame whose
        letterbox is empty."""
        in_h, in_w = self.input_size[0], self.input_size[1]
        layout = []
        for (H, W, pitch, _, _), (Hu, Wu) in zip(call.shapes, call.upright):
            geo = letterbox_geometry(Hu, Wu, in_h, in_w)
            if geo[1] < 1 or geo[2] < 1:
                raise ValueError("frame %dx%d: its letterbox at %dx%d is %dx%d, empty" % (Hu, Wu, in_h, in_w, geo[2], geo[1]))
            layout.append((H, W, pitch, geo, None if call.cuda else host_upload_rows(H, geo[2])))
        return layout

    def _enqueue(self, call, layout, out, detect):
        """Stages a checked call (check_frames, _layout) into the next slot and enqueues letterbox (and, with detect,
        network, NMS and the copy back of host results) on the engine's stream; returns the slot.  out: None, or result
        buffers of new_results(n) the kept rows go to, for host frames as well as CUDA frames (FaceAnaImages keeps them
        on the GPU); nothing is then copied back."""
        torch = rt.require_cuda()
        frames, cuda = call.frames, call.cuda
        n, R, M = len(frames), self._rows, min(self.MAX_DET, self._rows)
        A, C = self.align, self.max_chips
        align = detect and A is not None
        warp_now = align and cuda                     # CUDA frames are warped here, host frames at collect()
        if self._slots is None:
            self._slots = [self._new_slot() for _ in range(2)]
        slot = self._next
        st = self._slots[slot]
        # CUDA frames in a layout other than BGR: one skps_frame_layout per frame after the recoveries; a call holding a
        # turned frame: then the quarter turns of every frame, int32
        lay = cuda and n > 0 and call.shapes[0].code != 0
        turned = cuda and call.turned
        rec_off = pad16(n * DET_SRC.itemsize)
        lay_off = rec_off + pad16(n * 12)
        turn_off = lay_off + (pad16(n * FRAME_LAYOUT.itemsize) if lay else 0)
        face_off = turn_off + (pad16(n * 4) if turned else 0)
        frame_off = face_off + (pad16(n * FACE_SRC.itemsize) if warp_now else 0)
        sizes = [0 if cuda else pad16((H if rows is None else len(rows)) * pitch) for H, W, pitch, geo, rows in layout]
        total = frame_off + sum(sizes)
        own = detect and out is None                  # results go to the slot's buffers and come back to the host
        host, dev = st["stage"].reserve(total, st["done"])
        if own and st["capacity"] < max(n, 1):
            st["done"].synchronize()                  # the slot's last call has finished with what is replaced
            st["capacity"] = k = max(n, 2 * st["capacity"], 1)
            fields = result_fields(k, R, A, C)
            fields.pop("chip", None)                  # warped at submit() for CUDA frames only: below
            st.update(new_buffers(fields, self.device))
            # the first M kept rows of every frame come back with the counts, and with align the points and matrices
            fields = result_fields(k, M, A, C)
            fields.pop("chip", None)
            st.update({"h" + name: t.pin_memory() for name, t in new_buffers(fields, "cpu").items()})
        if own and warp_now and (st["chip"] is None or st["chip"].shape[0] < n):
            st["done"].synchronize()
            st["chip"] = grow(st["chip"], n, lambda k: torch.empty((k, C, A, A, 3), dtype=torch.uint8, device=self.device))
        # host staging = [n frame descriptors | n (scale, left, top) | n layouts | n turns | n face sources | the host
        # frames' rows], sent with one copy
        desc = host[:n * DET_SRC.itemsize].view(DET_SRC)
        rec = host[rec_off:rec_off + 12 * n].view(np.float32).reshape(n, 3)
        if lay:
            fl = host[lay_off:lay_off + n * FRAME_LAYOUT.itemsize].view(FRAME_LAYOUT)
            fl["layout"] = [f.code for f in call.shapes]
            fl["plane_pitch"] = [f.plane for f in call.shapes]
        if turned:
            host[turn_off:turn_off + 4 * n].view(np.int32)[:] = call.turns
        if warp_now:                                  # the chips' sources: the whole frames
            fs = host[face_off:face_off + n * FACE_SRC.itemsize].view(FACE_SRC)
            H, W, pitch = np.array([f[:3] for f in call.shapes], np.int64).reshape(-1, 3).T
            fs["base"] = [f.data_ptr() for f in frames]
            fs["pitch"], fs["H"], fs["W"], fs["rw"], fs["rh"] = pitch, H, W, W, H
            fs["ox"], fs["oy"], fs["_pad"] = 0, 0, 0
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

        s = self.model.stream
        st["stage"].send(frame_off if cuda else total, st["done"])     # NMS reads the recoveries from the staging
        s.wait_stream(torch.cuda.current_stream(self.device))
        s.wait_event(st["stage"].copied)
        res = out if out is not None else st
        rows_t, idx_t, count_t = res["rows"], res["idx"], res["count"]
        K = self.max_frames
        in_h, in_w = self.input_size[0], self.input_size[1]
        inp = self.model.input_ptr()
        for c0 in range(0, n, K):
            m = min(K, n - c0)
            with torch.cuda.device(self.device):      # the kernels launch on the current device
                rt.check(self.lib.skps_letterbox_frames_rotate(dev + DET_SRC.itemsize * c0,
                                                               dev + lay_off + FRAME_LAYOUT.itemsize * c0 if lay else None,
                                                               dev + turn_off + 4 * c0 if turned else None,
                                                               m, inp, in_h, in_w, s.cuda_stream))
            if c0 + K >= n and not warp_now:
                st["read"].record(s)
            if not detect:
                continue
            rt.check(self.lib.skps_engine_forward(self.model.handle, inp, m, None, s.cuda_stream))
            with torch.cuda.device(self.device):
                rt.check(self.lib.skps_detect_post_batch(self.model.output_ptr(0), R, m, self.score_thrs, self.iou_thrs,
                                                         dev + rec_off + 12 * c0, rows_t.data_ptr() + 64 * R * c0,
                                                         idx_t.data_ptr() + 4 * R * c0, count_t.data_ptr() + 4 * c0, R,
                                                         self._ws.data_ptr(), self._ws_bytes, s.cuda_stream))
        if align and n:
            points, mats = res["points"], res["M"]
            with torch.cuda.device(self.device):
                rt.check(self.lib.skps_det_align_estimate(rows_t.data_ptr(), count_t.data_ptr(), R, dev + rec_off, n, C, A,
                                                          points.data_ptr(), mats.data_ptr(), s.cuda_stream))
                if warp_now:
                    rt.check(self.lib.skps_warp_faces_count_rotate(dev + face_off, dev + lay_off if lay else None,
                                                                   dev + turn_off if turned else None, count_t.data_ptr(),
                                                                   n, C, mats.data_ptr(), A, A, res["chip"].data_ptr(),
                                                                   s.cuda_stream))
        if n == 0 or warp_now:
            st["read"].record(s)
        torch.cuda.current_stream(self.device).wait_event(st["read"])
        if own and n:
            with torch.cuda.stream(s):
                st["hrows"][:n].copy_(rows_t[:n, :M], non_blocking=True)
                st["hidx"][:n].copy_(idx_t[:n, :M], non_blocking=True)
                st["hcount"][:n].copy_(count_t[:n], non_blocking=True)
                if align:
                    st["hpoints"][:n].copy_(res["points"][:n], non_blocking=True)
                    st["hM"][:n].copy_(res["M"][:n], non_blocking=True)
        st["done"].record(s)
        self._next ^= 1
        return st

    def _new_slot(self):
        import torch
        return dict(stage=Staging(self.device), capacity=0, rows=None, idx=None, count=None, chip=None, hchip=None,
                    dchip=None, read=torch.cuda.Event(), done=torch.cuda.Event())
