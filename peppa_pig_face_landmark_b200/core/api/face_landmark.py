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
    # aligned chips of the same faces (core/api/align.py), for a detector that feeds its own aligner:
    fl = FaceLandmark(max_faces=256, align=112)
    res = fl.run_batch(frames, boxes)      # [(kps, scores, chips (k_i,112,112,3) uint8, M (k_i,2,3) float64) per frame]
"""
import ctypes as C
import os
import pathlib
import time

import numpy as np

from ... import runtime as rt
from ...logger.logger import logger
from .align import check_size, chip_read_rects
from .device_frames import FRAME_LAYOUT, is_cuda_tensor
from .onnx_model_base import ONNXEngine
from .staging import Staging, check_frames, check_out, grow, new_buffers, pad16

MIN_FACE = 20              # face_landmark.py:26,76: boxes with a side of at most this many pixels get no landmarks
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


def result_fields(n_faces, n_points, align=None):
    """{name: (shape, dtype name)} of new_results(n_faces) of FaceLandmark(align=align) with n_points landmarks."""
    f = {"kps": ((n_faces, n_points, 2), "float32"), "scores": ((n_faces, n_points), "float32")}
    if align is not None:
        f.update({"chip": ((n_faces, align, align, 3), "uint8"), "M": ((n_faces, 2, 3), "float64")})
    return f


def _rect_bytes(rects):
    """Bytes of the BGR pixels of each [x0, y0, x1, y1) rectangle of rects (n, 4)."""
    return (rects[:, 2] - rects[:, 0]) * (rects[:, 3] - rects[:, 1]) * 3


def _gather_rects(frames, rects, image, host, at, dev):
    """Stages the parts of host frames that kernels read through FACE_SRC descriptors: rectangle j, rects[j] of
    frames[image[j]], goes into the pinned staging `host` from byte `at` on, one after the other, and descriptor j at the
    start of `host` points at it in the device copy of the staging at address `dev`."""
    nb = _rect_bytes(rects)
    starts = at + np.cumsum(nb) - nb
    rw, rh = rects[:, 2] - rects[:, 0], rects[:, 3] - rects[:, 1]
    hw = np.array([f.shape[:2] for f in frames], np.int64)[image]
    desc = host[:len(rects) * FACE_SRC.itemsize].view(FACE_SRC)
    desc["H"], desc["W"], desc["_pad"] = hw[:, 0], hw[:, 1], 0
    desc["base"], desc["pitch"] = dev + starts, 3 * rw
    desc["ox"], desc["oy"], desc["rw"], desc["rh"] = rects[:, 0], rects[:, 1], rw, rh
    for j in np.flatnonzero(nb):
        x0, y0, x1, y1 = (int(v) for v in rects[j])
        host[starts[j]:starts[j] + nb[j]].reshape(y1 - y0, 3 * (x1 - x0))[:] = \
            frames[image[j]][y0:y1, x0:x1].reshape(y1 - y0, 3 * (x1 - x0))


class HostChips:
    """The chip stage of host frames, which FaceLandmark, FaceAnaImages and FaceDetector with align run at collect(): of
    each frame only the rectangle each chip reads (core/api/align.py:chip_read_rects) crosses PCIe, through a pinned
    staging on a copy stream, and is warped with skps_warp_faces."""

    def __init__(self, device, size):
        self.device, self.size = device, size
        self._stage = None            # (Staging, done event), made on first use

    def warp(self, lib, stream, call, counts, M, chips, h_chips):
        """(blocking) counts[i] faces of call.frames[i] (a call checked by check_frames), whose matrices M (n, 2, 3)
        float64 are on the host.  Uploads the matrices and the rectangles, warps chips[:n] (a device (>= n, size, size, 3)
        uint8 tensor) on `stream`, where no other kernel runs beside it, and copies them to the pinned h_chips[:n]."""
        torch = rt.require_cuda()
        n, A = len(M), self.size
        rects = np.concatenate([chip_read_rects(M[o:o + k], A, f.H, f.W) for o, k, f
                                in zip(np.cumsum([0] + list(counts[:-1])), counts, call.shapes)])
        m_off = pad16(n * FACE_SRC.itemsize)
        roi_off = m_off + 48 * n
        total = roi_off + int(_rect_bytes(rects).sum())
        if self._stage is None:
            self._stage = (Staging(self.device), torch.cuda.Event())
        cs, done = self._stage
        host, dev = cs.reserve(total, done)
        # host staging = [n face descriptors | n matrices | the frames' rectangles], sent with one copy
        host[m_off:roi_off].view(np.float64)[:] = np.asarray(M, np.float64).reshape(-1)
        _gather_rects(call.frames, rects, np.repeat(np.arange(len(counts)), counts), host, roi_off, dev)
        cs.send(total, done)
        stream.wait_event(cs.copied)
        with torch.cuda.device(self.device):
            rt.check(lib.skps_warp_faces(dev, dev + m_off, n, A, A, chips.data_ptr(), stream.cuda_stream))
        with torch.cuda.stream(stream):
            h_chips[:n].copy_(chips[:n], non_blocking=True)
        done.record(stream)
        done.synchronize()                            # the staging is free again and h_chips holds the chips


class FaceLandmark:
    def __init__(self, cfg=None, max_faces=16, device="cuda", align=None):
        """cfg: Skps.yml's Keypoints section (None: read it from Skps.yml).  max_faces: faces per network forward; the
        Student@256 plan holds about 47 MB of activations per face of it.  Calls of run_batch / submit take any number
        of faces and run them in chunks of at most max_faces.

        align: None, or a chip side in 16..512: run_batch / collect then also return every face's chip (align, align, 3)
        uint8 BGR and M (2, 3) float64, what FaceAna(align=align) computes from its 'kps': M is the similarity from the
        landmarks promoted to float64 to the ArcFace template, the chip cv2.warpAffine(frame, M, (align, align)) bit for
        bit (core/api/align.py).  Each of the two call slots then keeps align^2 x 3 bytes per face of its largest call
        on the device and as much pinned (37.6 kB at 112, 786 kB at 512).  __call__ returns (kps, scores) as before."""
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
        self.align = None if align is None else check_size(align)
        self.lib = rt.load_library()
        torch = rt.require_cuda()
        K = self.max_faces
        self._boxes = torch.zeros((K, 4), dtype=torch.float32, device=self.device)
        self._count = torch.zeros((1,), dtype=torch.int32, device=self.device)
        self._detail = torch.zeros((K, 5), dtype=torch.int32, device=self.device)
        self.last_detail = None
        self._slots = None            # staging of the batched path, made on first use
        self._pending = []            # [(slot, faces per frame, out or None, checked host frames to align or None)]
        self._next = 0
        self.host_chips = None if self.align is None else HostChips(self.device, self.align)

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
        with torch.cuda.device(self.device):          # the kernel launches on the current device
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
        kps, scores = self.run_batch([img], [bboxes])[0][:2]
        self.last_detail = self._slots[slot]["detail"][:len(kps)].cpu().numpy()
        duration = time.time() - t0
        logger.info('keypoints done, time consume: %.5f and %.5f per face' % (duration, duration / len(bboxes)))
        return kps, scores

    # ------------------------------------------------------------------ batched path
    def run_batch(self, frames, boxes, layout="bgr", rotate=0):
        """Landmarks for the faces the caller has, over many frames (blocking): frames[i] with boxes[i] -> the i-th
        (kps (k_i, 98, 2) float32, scores (k_i, 98) float32) of the returned list, bit for bit what
        FaceLandmark(cfg)(frames[i], boxes[i]) returns; with align, (kps, scores, chips (k_i, s, s, 3) uint8,
        M (k_i, 2, 3) float64).  See submit() for what frames, boxes, layout and rotate may be."""
        if self._pending:
            raise RuntimeError("FaceLandmark: %d calls in flight; collect() them first" % len(self._pending))
        self.submit(frames, boxes, layout=layout, rotate=rotate)
        return self.collect()

    def new_results(self, n_faces):
        """Device result buffers for submit(cuda_frames, boxes, out=...) of up to n_faces faces: a dict of CUDA tensors
        on this object's device, kps (n_faces, 98, 2) and scores (n_faces, 98) float32; with align also chip
        (n_faces, s, s, 3) uint8 and M (n_faces, 2, 3) float64."""
        rt.require_cuda()
        return new_buffers(self._fields(int(n_faces)), self.device)

    def _fields(self, n_faces):
        return result_fields(n_faces, self.keypoints_num, self.align)

    def submit(self, frames, boxes, out=None, layout="bgr", rotate=0):
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
        faces, not used by a call still in flight: the results are written there on the GPU.
        layout: the pixel layout of all CUDA frames of the call (device_frames.frame_layout): "bgr" (the default), "rgb",
        "bgra", "rgba" (H, W, 4), "bgr_planar" or "rgb_planar" (3, H, W).  Crops and chips read them in place and come
        out BGR, bit for bit those of the same pixels passed as interleaved BGR.  Host frames are BGR only.
        rotate: the clockwise angle in degrees (0, 90, 180 or 270) by which CUDA frames, as stored, must be turned to be
        upright (device_frames.check_rotate), one for the call or one per frame.  The boxes are in the upright frame's
        pixels, and so are the results, bit for bit those of the upright frame passed as a contiguous tensor; crops and
        chips read the stored frame in place.  Host frames take 0.

        With align, CUDA frames are warped into chips on the GPU right after the landmarks, with no host synchronisation,
        and are read until then.  Host frames are warped at collect(): M comes back with kps and scores, and
        core/api/align.py:chip_read_rects picks the rectangle of the frame each chip reads, which is uploaded and warped.
        That is one more read-back and one more upload per call, and the host frames must stay unchanged until
        collect() returns."""
        if len(self._pending) == 2:
            raise RuntimeError("FaceLandmark: two calls already in flight; call collect() first")
        call = check_frames(frames, self.device, layout, rotate)
        boxes, cuda_boxes = self._check_boxes(call, boxes)
        counts = [int(b.shape[0]) for b in boxes]
        if out is not None:
            if not call.cuda:
                raise ValueError("out= keeps results on the GPU and takes CUDA frames; these are host frames")
            check_out(out, self._fields(sum(counts)), self.device, [p[2] for p in self._pending])
        slot = self._enqueue(call, boxes, cuda_boxes, out)
        align_host = self.align is not None and not call.cuda
        self._pending.append((slot, counts, out, call if align_host else None))

    def _check_boxes(self, call, boxes):
        """Checks the boxes of a call whose frames check_frames has checked: (boxes, whether they are CUDA tensors)."""
        boxes = list(boxes)
        if len(call.frames) != len(boxes):
            raise ValueError("%d frames but %d box arrays" % (len(call.frames), len(boxes)))
        box_dev = [is_cuda_tensor(b) for b in boxes]
        cuda_boxes = bool(box_dev) and all(box_dev)
        if any(box_dev) and not cuda_boxes:
            raise ValueError("boxes are either all host arrays or all CUDA tensors (boxes %s are CUDA)"
                             % [i for i, d in enumerate(box_dev) if d])
        if cuda_boxes and not call.cuda:
            raise ValueError("CUDA boxes take CUDA frames: the host frames' upload is cut to the boxes on the host")
        check = self._check_cuda_boxes if cuda_boxes else self._check_host_boxes
        return [check(b, i) for i, b in enumerate(boxes)], cuda_boxes

    def _enqueue(self, call, boxes, cuda_boxes, out):
        """Stages a call checked by check_frames and _check_boxes into the next slot and enqueues crops, network and
        post-processing (and, without out, the copy back) on the engine's stream; returns the slot.  out: None, or
        result buffers of new_results(n) the results go to, for host frames as well as CUDA frames (FaceAnaImages keeps
        them on the GPU)."""
        torch = rt.require_cuda()
        counts = [int(b.shape[0]) for b in boxes]
        n, P, A = sum(counts), self.keypoints_num, self.align
        if self._slots is None:
            self._slots = [self._new_slot() for _ in range(2)]
        slot = self._next
        st = self._slots[slot]
        warp_now = A is not None and call.cuda     # CUDA frames are warped here, host frames at collect()
        image = np.repeat(np.arange(len(counts)), counts)
        rects = None if call.cuda or n == 0 else np.concatenate(
            [crop_read_rects(b, f.H, f.W, self.face_scale, self.min_face) for b, f in zip(boxes, call.shapes)])
        # CUDA frames in a layout other than BGR: one skps_frame_layout per face after the descriptors; a call holding a
        # turned frame: then the quarter turns of every face's frame, int32
        lay = call.cuda and n > 0 and call.shapes[0].code != 0
        turned = call.cuda and n > 0 and call.turned
        lay_off = pad16(n * FACE_SRC.itemsize)
        turn_off = lay_off + (pad16(n * FRAME_LAYOUT.itemsize) if lay else 0)
        box_off = turn_off + (pad16(n * 4) if turned else 0)
        roi_off = box_off + pad16(n * 16)
        total = roi_off + (0 if rects is None else int(_rect_bytes(rects).sum()))
        sent = box_off if cuda_boxes else total       # bytes of the host staging the call sends
        host, dev = st["stage"].reserve(total, st["done"])
        if st["kps"] is None or st["kps"].shape[0] < n:
            st["done"].synchronize()                  # the slot's last call has finished with what is replaced
            st["kps"] = grow(st["kps"], n, lambda k: torch.empty((k, P, 2), dtype=torch.float32, device=self.device))
            st["scores"] = grow(st["scores"], n, lambda k: torch.empty((k, P), dtype=torch.float32, device=self.device))
            st["detail"] = grow(st["detail"], n, lambda k: torch.empty((k, 5), dtype=torch.int32, device=self.device))
            st["hkps"] = grow(st["hkps"], n, lambda k: torch.empty((k, P, 2), dtype=torch.float32).pin_memory())
            st["hscores"] = grow(st["hscores"], n, lambda k: torch.empty((k, P), dtype=torch.float32).pin_memory())
        if A is not None and out is None and (st["chip"] is None or st["chip"].shape[0] < n):
            st["done"].synchronize()
            st["M"] = grow(st["M"], n, lambda k: torch.empty((k, 2, 3), dtype=torch.float64, device=self.device))
            st["hM"] = grow(st["hM"], n, lambda k: torch.empty((k, 2, 3), dtype=torch.float64).pin_memory())
            st["chip"] = grow(st["chip"], n, lambda k: torch.empty((k, A, A, 3), dtype=torch.uint8, device=self.device))
            st["hchip"] = grow(st["hchip"], n, lambda k: torch.empty((k, A, A, 3), dtype=torch.uint8).pin_memory())
        # host staging = [n face descriptors | n layouts | n turns | n boxes | the host frames' rectangles], sent with one
        # copy
        if n and not cuda_boxes:
            host[box_off:box_off + 16 * n].view(np.float32).reshape(n, 4)[:] = np.concatenate(boxes)
        if call.cuda:                                 # descriptors of the whole frames
            desc = host[:n * FACE_SRC.itemsize].view(FACE_SRC)
            H, W, pitch, plane, code = np.array(call.shapes, np.int64).reshape(-1, 5)[image].T
            desc["base"] = np.array([f.data_ptr() for f in call.frames], np.uint64)[image]
            desc["pitch"], desc["H"], desc["W"], desc["rw"], desc["rh"] = pitch, H, W, W, H
            desc["ox"], desc["oy"], desc["_pad"] = 0, 0, 0
            if lay:
                fl = host[lay_off:lay_off + n * FRAME_LAYOUT.itemsize].view(FRAME_LAYOUT)
                fl["layout"], fl["plane_pitch"] = code, plane
            if turned:
                host[turn_off:turn_off + 4 * n].view(np.int32)[:] = np.array(call.turns, np.int32)[image]
        elif n:
            _gather_rects(call.frames, rects, image, host, roi_off, dev)

        s = self.model.stream
        st["stage"].send(sent, st["read"])            # the slot's last crops have read its device staging
        s.wait_stream(torch.cuda.current_stream(self.device))
        s.wait_event(st["stage"].copied)
        if cuda_boxes and n:
            with torch.cuda.stream(s):
                dst = st["stage"].dev[box_off:box_off + 16 * n].view(torch.float32).view(n, 4)
                torch.cat([b[:, :4] for b in boxes if b.shape[0]], out=dst)
        res = out if out is not None else st
        kps, scores = res["kps"], res["scores"]
        K, S = self.max_faces, self.input_size[0]
        inp = self.model.input_ptr()
        det = st["detail"].data_ptr()
        for c0 in range(0, n, K):
            m = min(K, n - c0)
            with torch.cuda.device(self.device):      # the kernels launch on the current device
                rt.check(self.lib.skps_crop_faces_rotate(dev + FACE_SRC.itemsize * c0,
                                                         dev + lay_off + FRAME_LAYOUT.itemsize * c0 if lay else None,
                                                         dev + turn_off + 4 * c0 if turned else None,
                                                         dev + box_off + 16 * c0, m, self.face_scale, float(self.min_face),
                                                         inp, S, det + 20 * c0, s.cuda_stream))
            if c0 + K >= n and not warp_now:
                st["read"].record(s)
            outs = (C.c_void_p * 2)(None, scores.data_ptr() + 4 * P * c0)
            rt.check(self.lib.skps_engine_forward(self.model.handle, inp, m, outs, s.cuda_stream))
            with torch.cuda.device(self.device):
                rt.check(self.lib.skps_landmark_post(self.model.output_ptr(0), det + 20 * c0, st["count"].data_ptr(), m,
                                                     P, kps.data_ptr() + 8 * P * c0, s.cuda_stream))
        if A is not None and n:
            M, chips = res["M"], res["chip"]
            with torch.cuda.device(self.device):
                rt.check(self.lib.skps_align_estimate(kps.data_ptr(), n, P, A, M.data_ptr(), s.cuda_stream))
                if warp_now:                          # the face descriptors hold the whole CUDA frames
                    rt.check(self.lib.skps_warp_faces_rotate(dev, dev + lay_off if lay else None,
                                                             dev + turn_off if turned else None, M.data_ptr(), n, A, A,
                                                             chips.data_ptr(), s.cuda_stream))
        if n == 0 or warp_now:
            st["read"].record(s)
        torch.cuda.current_stream(self.device).wait_event(st["read"])
        if out is None and n:
            with torch.cuda.stream(s):
                for k in self._fields(0):
                    if k != "chip" or warp_now:       # host frames are warped at collect()
                        st["h" + k][:n].copy_(st[k][:n], non_blocking=True)
        st["done"].record(s)
        self._next ^= 1
        return slot

    def collect(self):
        """Results of the oldest call in flight: a list with one (kps (k_i, 98, 2), scores (k_i, 98)) pair per frame, as
        float32 numpy arrays (with align, (kps, scores, chips, M)); for a call submitted with out=, views of out's rows,
        with no host synchronisation: torch.cuda.current_stream() is made to wait for the call, so work queued on it
        afterwards sees the results.  A call of host frames with align is warped here (see submit())."""
        if not self._pending:
            raise RuntimeError("FaceLandmark: nothing submitted")
        slot, counts, out, host_call = self._pending.pop(0)
        st = self._slots[slot]
        names = list(self._fields(0))
        if out is not None:
            import torch
            torch.cuda.current_stream(self.device).wait_event(st["done"])
            arrays = [out[k] for k in names]
        else:
            st["done"].synchronize()
            n = sum(counts)
            if host_call is not None and n:
                self.host_chips.warp(self.lib, self.model.stream, host_call, counts, st["hM"].numpy()[:n], st["chip"],
                                     st["hchip"])
            arrays = [st["h" + k].numpy() for k in names]
        res, o = [], 0
        for k in counts:
            if out is None:
                res.append(tuple(a[o:o + k].copy() for a in arrays))
            else:
                res.append(tuple(a[o:o + k] for a in arrays))
            o += k
        return res

    def _new_slot(self):
        import torch
        return dict(stage=Staging(self.device), kps=None, scores=None, detail=None, hkps=None, hscores=None, M=None,
                    hM=None, chip=None, hchip=None,
                    count=torch.full((1,), self.max_faces, dtype=torch.int32, device=self.device),
                    read=torch.cuda.Event(), done=torch.cuda.Event())

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
