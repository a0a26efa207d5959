"""FaceAna — same public surface as the reference's Skps/core/api/facer.py:25-208:
`FaceAna(verbose=False)`, `.run(image) -> [{'box','kps','scores'}, ...]`, `.reset()`.

Per frame the GPU does, with no host round trip in between (skps_pipeline_run):
letterbox -> yolov5-face -> NMS -> judge_boxs(track) -> sort_and_filter -> crops -> landmark net
-> de-normalise.  The host keeps what is stateful and tiny: the frame-diff decision, One-Euro
landmark smoothing (GroupTrack) and the EMA of the track boxes (facer.py:71-82)."""
import ctypes as C
import logging
import os
import pathlib

import numpy as np
import yaml

from ... import runtime as rt
from ...graph_tools import check_detector_input
from ...logger.logger import logger
from ..smoother.lk import MAX_ID_MEMORY, EmaFilter, GroupTrack, IdMemory, assign_track_ids, first_match, rects
from .face_detector import FaceDetector, letterbox_geometry
from .face_landmark import MIN_FACE, FaceLandmark, face_scale
from .align import check_size
from .device_frames import PLANAR, check_cuda_frame, check_host_frame, check_layout, check_rotate, is_cuda_tensor


MAX_TOP_K = 1024           # SKPS_MAX_TOP_K of include/skps_b200.h
LANDMARK_CHUNK = 64        # SKPS_LANDMARK_CHUNK: faces per landmark forward in skps_pipeline_run


def check_detect_every(every, offset=0):
    """(every, offset) as ints: every >= 1 and offset in 0..every-1, else ValueError."""
    def is_int(v):
        return isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))
    if not is_int(every) or every < 1:
        raise ValueError("detect_every must be an int >= 1, got %r" % (every,))
    if not is_int(offset) or not 0 <= offset < every:
        raise ValueError("detect_offset must be an int in 0..%d, got %r" % (every - 1, offset))
    return int(every), int(offset)


def check_id_memory(frames, track_ids):
    """id_memory as an int in 0..MAX_ID_MEMORY, and > 0 only with track_ids, else ValueError."""
    if (not isinstance(frames, (int, np.integer)) or isinstance(frames, (bool, np.bool_))
            or not 0 <= frames <= MAX_ID_MEMORY):
        raise ValueError("id_memory must be an int in 0..%d, got %r" % (MAX_ID_MEMORY, frames))
    if frames and not track_ids:
        raise ValueError("id_memory=%d keeps the ids of lost tracks and needs track_ids=True" % frames)
    return int(frames)


class DetectCadence:
    """The detection cadence of one stream: frames are counted from construction or reset(), i = 0, 1, 2, ..., and frame
    i is a keyframe when it is forced (no previous frame of its size) or (i + offset) % every == 0.  FaceAna keeps one;
    skps_mpipe keeps the same count per stream in C, with offset s % every."""

    def __init__(self, every=1, offset=0):
        self.every, self.offset = check_detect_every(every, offset)
        self.frame = 0

    def step(self, forced):
        """Whether the next frame is a keyframe; counts it."""
        key = bool(forced) or (self.frame + self.offset) % self.every == 0
        self.frame += 1
        return key

    def reset(self):
        self.frame = 0


def get_cfg():
    root_path = pathlib.Path(__file__).resolve().parents[2]
    cfg_path = os.path.join(root_path, 'config', 'Skps.yml')
    with open(cfg_path, encoding="UTF-8") as f:
        return yaml.load(f, Loader=yaml.FullLoader)


def pipeline_cfg(cfg, top_k, max_frame_hw):
    """The skps_pipeline_cfg of FaceAna and FaceAnaStreams from Skps.yml's Skps section."""
    det, trace = cfg['Detect'], cfg['Trace']
    return rt.PipelineCfg(score_thres=det['score_thrs'], iou_thres=det['iou_thrs'], min_face=float(det['min_face']),
                          top_k=int(top_k), track_iou=float(trace['iou_thres']), alpha=float(trace['smooth_box']),
                          face_scale=face_scale(cfg['Keypoints']), kps_min_face=float(MIN_FACE),
                          max_h=int(max_frame_hw[0]), max_w=int(max_frame_hw[1]))


class FaceAna():
    def __init__(self, verbose=False, top_k=None, max_frame_hw=(2160, 3840), align=None, pose=False, det_input=None,
                 track_ids=False, detect_every=1, detect_offset=0, id_memory=0):
        """align: None, or a chip side in 16..512: every result dict then also carries 'chip' ((align, align, 3) uint8
        BGR, the face warped to the ArcFace five-point template) and 'M' ((2, 3) float64, the frame -> chip matrix for
        cv2.warpAffine), computed on the GPU from the returned 'kps' and the frame already in HBM (core/api/align.py).
        pose: every result dict then also carries 'pose': {'euler': (3,), 'rvec': (3,), 'tvec': (3,), 'reproject': (8, 2)},
        float64, Euler angles in degrees - head_poses(kps[None], frame.shape[:2], points=POSE_POINTS_98) of the returned
        'kps', solved on the GPU.
        det_input: None (Skps.yml's Detect.input_shape, 384x640), or the detector input size (h, w): multiples of 32 in
        128..2176 x 128..3840.  Every frame is letterboxed to that size, so a larger one finds smaller faces: at 1152x1920
        a 3840x2160 frame is scaled by 1/2 instead of 1/6.  The detector's work and activation memory grow with h*w
        (3.97 GMAC and 0.35 GB at 1152x1920, 0.44 GMAC and 0.04 GB at 384x640).
        top_k: None (Skps.yml's Detect.topk, 5), or 1..1024 faces per frame.  The landmark net runs on the faces found,
        in chunks of at most 64, so its activation memory is that of min(top_k, 64) faces (about 47 MB per face).
        track_ids: every result dict then also carries 'id', an int that follows the face from call to call.  Ids are
        numbered per FaceAna from 0, and reset() starts again from 0.  Each returned face has a source: on a frame that ran
        the detector, the first of the previous call's faces whose box its detection overlaps with IoU > Trace.iou_thres
        (the match judge_boxs smooths the box with), or none; on a frame the difference gate skipped, the previous face
        it is.  In the order of the returned list, a face inherits its source's id unless an earlier face of the same
        call already took it, and every other face gets the next unused number.  With id_memory=0 (the default) a face
        the tracker loses for one frame comes back with a new id.
        id_memory: 0..2**31 - 1 frames (track_ids only).  A track returned at frame a that no face of frame a + 1 carries
        is lost; its id and its float32 box of frame a are remembered, up to top_k of them.  A face that would get the
        next unused number first takes back the id of the first remembered track, most recently lost first, that it
        overlaps with IoU > Trace.iou_thres (its float32 landmark-stage box against the remembered one) and that has been
        missing for at most id_memory frames in a row.  Only 'id' changes: such a face's box, landmarks and smoothing
        start afresh as without the memory.  Frames are counted from construction or reset(), which forgets the lost
        tracks too.
        detect_every, detect_offset: the detection cadence.  Frames are counted from construction or reset(), i = 0, 1,
        2, ...; frame i runs the detector when there is no previous frame of its size (the first frame, a size change),
        or when (i + detect_offset) % detect_every == 0 and the frame-difference gate fires.  Every other frame takes the
        tracker path on the last frame's landmark boxes, One-Euro smoothing included.  So a face that enters the scene is
        found at the next keyframe, up to detect_every - 1 frames late, and a face that leaves is followed by its
        landmark box until the next keyframe.  detect_every=1 (the default) is the reference's behaviour.
        last_ran_detector tells whether the last run() used the detector."""
        self.id_memory = check_id_memory(id_memory, track_ids)
        self._cadence = DetectCadence(detect_every, detect_offset)
        self.detect_every, self.detect_offset = self._cadence.every, self._cadence.offset
        cfg = get_cfg()
        self.top_k = int(top_k if top_k is not None else cfg['Skps']['Detect']['topk'])
        if not 1 <= self.top_k <= MAX_TOP_K:
            raise ValueError("top_k %d outside 1..%d" % (self.top_k, MAX_TOP_K))
        pc = pipeline_cfg(cfg['Skps'], self.top_k, max_frame_hw)
        if det_input is not None:
            det_input = check_detector_input(det_input)
        self.align = None if align is None else check_size(align)
        self.pose = bool(pose)
        self.track_ids = bool(track_ids)
        if verbose:
            logger.setLevel(logging.DEBUG)
        if det_input is not None:
            cfg['Skps']['Detect']['input_shape'] = [det_input[0], det_input[1], 3]
        self.face_detector = FaceDetector(cfg['Skps']['Detect'], max_frames=1)
        self.face_landmark = FaceLandmark(cfg['Skps']['Keypoints'], max_faces=min(self.top_k, LANDMARK_CHUNK))
        self.trace = GroupTrack(cfg['Skps']['Trace'])
        logger.info('model init done!')
        self.track_box = None
        self.previous_image = None
        self.previous_box = None
        self.diff_thres = 5
        self.min_face = cfg['Skps']['Detect']['min_face']
        self.iou_thres = cfg['Skps']['Trace']['iou_thres']
        self.alpha = cfg['Skps']['Trace']['smooth_box']
        self.filter = EmaFilter(self.alpha)

        self.lib = rt.load_library()
        det, kps = self.face_detector, self.face_landmark
        h = C.c_void_p()
        rt.check(self.lib.skps_pipeline_create(det.model.handle, kps.model.handle, C.byref(pc), C.byref(h)))
        self._pipe = h
        self._stream = det.model.stream
        self._device = det.model.device
        self._max_hw = (int(max_frame_hw[0]), int(max_frame_hw[1]))
        K, P = self.top_k, kps.keypoints_num
        self._n = C.c_int32(0)
        self._ndet = C.c_int32(0)
        self._boxes = np.zeros((K, 4), np.float32)
        self._kps = np.zeros((K, P, 2), np.float32)
        self._scores = np.zeros((K, P), np.float32)
        self._det_idx = np.zeros((FaceDetector.MAX_DET,), np.int32)
        self._det_rows = np.zeros((FaceDetector.MAX_DET, 16), np.float32)
        self._have_prev = False
        self._ids, self._next_id = [], 0     # ids of the track boxes (index-aligned with track_box), next unused id
        self._memory = IdMemory(self.id_memory, self.top_k, self.iou_thres) if self.id_memory else None
        self.last_det_idx = None       # kept detector rows of the last detector run (parity checks)
        self.last_ran_detector = None
        self.last_det_rows = None

    def __del__(self):
        h = getattr(self, "_pipe", None)
        if h is not None and h.value:
            self.lib.skps_pipeline_destroy(h)
            self._pipe = None

    # ------------------------------------------------------------------ facer.py:52-85
    def run(self, image, layout="bgr", rotate=0):
        """image: an HxWx3 uint8 BGR numpy array, or a torch.uint8 CUDA tensor (H, W, 3) in BGR order on this object's
        device with stride(2) == 1, stride(1) == 3 and any row pitch stride(0) >= 3W (a packed tensor, a pitched decoder
        surface, big[y0:y1, x0:x1]).  A CUDA frame is copied once on the GPU, never through the host, and the results are
        those of image.cpu().numpy() bit for bit.  Ordering on torch.cuda.current_stream(): the frame is read after all
        work already queued on it, and work queued on it after run() returns runs after the frame has been read, so a
        decoder may overwrite the surface at once.

        layout: the pixel layout of a CUDA frame (device_frames.frame_layout): "bgr" (the default), "rgb", "bgra",
        "rgba" (H, W, 4), or "bgr_planar", "rgb_planar" (3, H, W) with any row and plane pitch.  The frame is packed
        into BGR by the same GPU copy, and the results are, bit for bit, those of the same pixels passed as an
        interleaved BGR frame.  Calls may change layouts from frame to frame.  Host frames are BGR only.

        rotate: the clockwise angle in degrees (0, 90, 180 or 270) by which a CUDA frame, as stored, must be turned to
        be upright (device_frames.check_rotate): a portrait clip NVDEC returns as coded, a ceiling camera.  The same GPU
        copy stages the frame upright, and the results are in the upright frame's pixels, bit for bit those of the
        upright frame passed as a contiguous tensor; the gate, tracking and smoothing see the upright frame, so a change
        between 0 and 90 is a change of frame size.  Host frames take 0."""
        check_layout(layout, is_cuda_tensor(image))
        turns = check_rotate(rotate, cuda=is_cuda_tensor(image))
        image = image if is_cuda_tensor(image) else check_host_frame(image)
        d = self._frame_diff(image, layout, turns)     # checks a CUDA frame, stages the frame on the device as upright BGR
        if layout in PLANAR:
            image = image.permute(1, 2, 0)      # an (H, W, 3) view: from here on only the frame's size is read
        if turns & 1:
            image = image.permute(1, 0, 2)      # a view of the upright frame's size
        forced = self.previous_image is None or d < 0       # no previous frame of this size
        run_det = self._cadence.step(forced) and (forced or d > self.diff_thres)
        self.last_ran_detector = run_det
        H, W = image.shape[:2]
        self.previous_image = image
        det = self.face_detector
        in_h, in_w = det.input_size[0], det.input_size[1]
        scale, rw, rh, top, left = letterbox_geometry(H, W, in_h, in_w)
        track = self.track_box
        n_track = 0 if track is None else int(len(track))
        track32 = None
        if n_track:
            track32 = np.ascontiguousarray(np.asarray(track)[:, :4], dtype=np.float32)
        src = np.zeros((0,), np.int32)
        if not run_det and n_track == 0:
            # facer.py:61 with an empty/None track: nothing to do (the reference would fail on None)
            boxes_return = np.zeros((0, 4), np.float32)
            landmarks, states = np.array([]), np.array([])
            rt.check(self.lib.skps_pipeline_commit_frame(self._pipe))     # the staged frame is the new "previous"
        else:
            rt.check(self.lib.skps_pipeline_run(
                self._pipe, 1 if run_det else 0, rw, rh, top, left, float(scale), rt.ptr(track32), n_track, C.byref(self._n),
                self._boxes.ctypes.data, self._kps.ctypes.data, self._scores.ctypes.data, C.byref(self._ndet),
                self._det_idx.ctypes.data, self._det_rows.ctypes.data, self._stream.cuda_stream))
            n = self._n.value
            boxes_return = self._boxes[:n].copy()
            landmarks = self._kps[:n].copy() if n else np.array([])
            states = self._scores[:n].copy() if n else np.array([])
            if self.track_ids and n:
                src = np.empty((n,), np.int32)
                rt.check(self.lib.skps_pipeline_face_sources(self._pipe, n, src.ctypes.data))
            if run_det:
                nd = self._ndet.value
                idx, rows = self._det_idx, self._det_rows
                if nd > len(idx):
                    # a crowd: skps_pipeline_run returned the first 256 kept rows, the device holds all of them
                    idx, rows = np.empty((nd,), np.int32), np.empty((nd, 16), np.float32)
                    rt.check(self.lib.skps_pipeline_det_results(self._pipe, nd, idx.ctypes.data, rows.ctypes.data))
                self.last_det_idx = idx[:nd].astype(np.int64)
                self.last_det_rows = rows[:nd].copy()
        if run_det:
            self.trace.previous_landmarks_set = None
        ids = []
        if self._memory is not None:          # every call, faceless ones included: they lose every track
            prev = track32 if n_track else np.zeros((0, 4), np.float32)
            ids, self._next_id = self._memory.assign(src, boxes_return, self._ids, prev, self._next_id)
        elif len(src):
            ids, self._next_id = assign_track_ids(src, self._ids, self._next_id)

        landmarks = self.trace.calculate(image, landmarks)

        tmp_box = rects(landmarks) if landmarks.shape[0] else np.array([])
        self.track_box = self.judge_boxs(boxes_return, tmp_box)
        res = self.to_dict(self.track_box, landmarks, states)
        if self.track_ids:
            self._ids = ids
            for r, i in zip(res, ids):
                r['id'] = i
        if self.align is not None and res:
            self._add_chips(res)
        if self.pose and res:
            self._add_pose(res, H, W)
        return res

    def _add_pose(self, res, H, W):
        """'pose' for every face, from its returned 'kps' promoted to float64 (skps_pipeline_pose)."""
        n = len(res)
        kps = np.ascontiguousarray(np.stack([np.asarray(r['kps'], np.float64) for r in res]))
        out = {k: np.empty((n, 3), np.float64) for k in ('rvec', 'tvec', 'euler')}
        out['reproject'] = np.empty((n, 8, 2), np.float64)
        rt.check(self.lib.skps_pipeline_pose(self._pipe, kps.ctypes.data, n, H, W, out['rvec'].ctypes.data,
                                             out['tvec'].ctypes.data, out['euler'].ctypes.data,
                                             out['reproject'].ctypes.data, self._stream.cuda_stream))
        for i, r in enumerate(res):
            r['pose'] = {k: v[i] for k, v in out.items()}

    def _add_chips(self, res):
        """'chip' and 'M' for every face, from its returned 'kps' promoted to float64 (skps_pipeline_align)."""
        n, size = len(res), self.align
        kps = np.ascontiguousarray(np.stack([np.asarray(r['kps'], np.float64) for r in res]))
        chips = np.empty((n, size, size, 3), np.uint8)
        M = np.empty((n, 2, 3), np.float64)
        rt.check(self.lib.skps_pipeline_align(self._pipe, kps.ctypes.data, n, size, chips.ctypes.data, M.ctypes.data,
                                              self._stream.cuda_stream))
        for i, r in enumerate(res):
            r['chip'] = chips[i]
            r['M'] = M[i]

    def to_dict(self, bboxes, kps, states):
        return [{'box': bboxes[i], 'kps': kps[i], 'scores': states[i]} for i in range(len(bboxes))]

    def diff_frames(self, previous_frame, image):
        """facer.py:98-118: mean |prev - cur| > 5 -> run the detector.  The sum is taken on the GPU
        against the previous frame kept in HBM; the frame uploaded here is reused by run()."""
        d = self._frame_diff(image)
        if previous_frame is None or d < 0:
            return True
        return bool(d > self.diff_thres)

    def _frame_diff(self, image, layout="bgr", turns=0):
        """Stages `image` (a CUDA frame in layout `layout`, stored `turns` quarter turns clockwise from upright) on the
        device as upright BGR and returns the mean |prev - cur| against the previous staged frame, or a negative number
        when that frame has another size (or there is none)."""
        d = C.c_double(0.0)
        if is_cuda_tensor(image):
            import torch
            f = check_cuda_frame(image, self._device, self._max_hw, layout)
            if turns:
                rt.check(self.lib.skps_pipeline_frame_diff_device_rotate(
                    self._pipe, image.data_ptr(), f.H, f.W, f.pitch, f.code, f.plane, turns,
                    torch.cuda.current_stream(self._device).cuda_stream, C.byref(d), self._stream.cuda_stream))
            else:
                rt.check(self.lib.skps_pipeline_frame_diff_device_layout(
                    self._pipe, image.data_ptr(), f.H, f.W, f.pitch, f.code, f.plane,
                    torch.cuda.current_stream(self._device).cuda_stream, C.byref(d), self._stream.cuda_stream))
        else:
            rt.check(self.lib.skps_pipeline_frame_diff(self._pipe, image.ctypes.data, *image.shape[:2], C.byref(d),
                                                       self._stream.cuda_stream))
        return d.value

    def sort_and_filter(self, bboxes):
        """facer.py:120-142 (host copy of what skps_select_faces does on the device)."""
        if len(bboxes) < 1:
            return []
        area = (bboxes[:, 2] - bboxes[:, 0]) * (bboxes[:, 3] - bboxes[:, 1])
        keep = area > self.min_face
        area, bboxes = area[keep], bboxes[keep, :]
        if bboxes.shape[0] > self.top_k:
            order = area.argsort()[-self.top_k:][::-1]
            return np.array([bboxes[i] for i in order])
        return np.array(bboxes)

    def judge_boxs(self, previuous_bboxs, now_bboxs):
        """facer.py:144-189."""
        if previuous_bboxs is None:
            return now_bboxs
        if len(now_bboxs) == 0:
            return np.array([])
        now = now_bboxs[:, :4]
        prev = previuous_bboxs[:, :4] if len(previuous_bboxs) else np.zeros((0, 4), now.dtype)
        match = first_match(now, prev, self.iou_thres)
        hit = match >= 0
        if not hit.any():
            return now.copy()
        ema = self.filter(now[hit], prev[match[hit]])
        out = now.astype(np.result_type(now, ema))        # np.array of the rows: float64 if any row is
        out[hit] = ema
        return out

    def smooth(self, now_box, previous_box):
        return self.filter(now_box[:4], previous_box[:4])

    def reset(self):
        """facer.py:200-208."""
        self.track_box = None
        self.previous_image = None
        self.previous_box = None
        self._ids, self._next_id = [], 0
        if self._memory is not None:
            self._memory.reset()
        self._cadence.reset()
        rt.check(self.lib.skps_pipeline_reset(self._pipe))

