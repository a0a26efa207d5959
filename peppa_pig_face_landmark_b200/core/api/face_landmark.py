"""FaceLandmark — same surface as the reference's Skps/core/api/face_landmark.py:14-115
(`FaceLandmark(cfg)(img, bboxes) -> ((K,98,2) float32, (K,98) float32)`).  The reference loops
over faces in Python with one batch-1 network call each (:40-48); here all faces are cropped by
one kernel straight into the network's input buffer and run as one batch.  The caller's `bboxes`
array is not modified (the reference mutates the rows in place, :81-90; facer.py:66 copies
first for that reason)."""
import os
import pathlib
import time

import numpy as np

from ... import runtime as rt
from ...logger.logger import logger
from .onnx_model_base import ONNXEngine

MIN_FACE = 20              # face_landmark.py:26,76: boxes with a side of at most this many pixels get no landmarks


def face_scale(cfg):
    """Crop side over box side, float32(1 + 2 * base_extend_range[0]) (face_landmark.py:83 in float32); cfg: Skps.yml's
    Keypoints section."""
    return float(np.float32(1 + 2 * cfg['base_extend_range'][0]))


class FaceLandmark:
    def __init__(self, cfg, max_faces=16):
        root_path = pathlib.Path(__file__).resolve().parents[2]
        model_path = os.path.join(root_path, cfg['model_path'])
        self.max_faces = int(max_faces)
        self.model = ONNXEngine(model_path, max_batch=self.max_faces)
        self.min_face = MIN_FACE
        self.keypoints_num = cfg['num_points']
        self.input_size = cfg['input_shape']
        self.extend = cfg['base_extend_range']
        self.face_scale = face_scale(cfg)
        self.lib = rt.load_library()
        torch = rt.require_cuda()
        dev = self.model.device
        K, P = self.max_faces, self.keypoints_num
        self._boxes = torch.zeros((K, 4), dtype=torch.float32, device=dev)
        self._count = torch.zeros((1,), dtype=torch.int32, device=dev)
        self._detail = torch.zeros((K, 5), dtype=torch.int32, device=dev)
        self._kps = torch.zeros((K, P, 2), dtype=torch.float32, device=dev)
        self.last_detail = None

    def _run_chunk(self, frame, h, w, boxes):
        torch = rt.require_cuda()
        n = boxes.shape[0]
        K, P = self.max_faces, self.keypoints_num
        s = self.model.stream
        with torch.cuda.stream(s):
            self._boxes[:n].copy_(torch.from_numpy(np.ascontiguousarray(boxes[:, :4], dtype=np.float32)))
            self._count.fill_(n)
        rt.check(self.lib.skps_crop_resize(frame.data_ptr(), h, w, w * 3, self._boxes.data_ptr(),
                                           self._count.data_ptr(), K, self.face_scale, float(self.min_face),
                                           self.model.input_ptr(), self.input_size[0], self._detail.data_ptr(),
                                           s.cuda_stream))
        rt.check(self.lib.skps_engine_forward(self.model.handle, self.model.input_ptr(), K, None, s.cuda_stream))
        rt.check(self.lib.skps_landmark_post(self.model.output_ptr(0), self._detail.data_ptr(),
                                             self._count.data_ptr(), K, P, self._kps.data_ptr(), s.cuda_stream))
        s.synchronize()
        scores = np.empty((K, P), np.float32)
        rt.check(self.lib.skps_engine_read_buffer(self.model.handle, self.model.plan.outputs[1].buf.idx, K,
                                                  scores.ctypes.data))
        return self._kps[:n].cpu().numpy(), scores[:n].copy(), self._detail[:n].cpu().numpy()

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
        torch = rt.require_cuda()
        t0 = time.time()
        if len(bboxes) == 0:
            return np.array([]), np.array([])
        bboxes = np.asarray(bboxes, dtype=np.float32)
        img = np.ascontiguousarray(img)
        h, w = img.shape[:2]
        frame = torch.from_numpy(img).to(self.model.device)
        self.model.stream.wait_stream(torch.cuda.current_stream(self.model.device))
        lms, scs, dets = [], [], []
        for i in range(0, bboxes.shape[0], self.max_faces):
            k, sc, dt = self._run_chunk(frame, h, w, bboxes[i:i + self.max_faces])
            lms.append(k); scs.append(sc); dets.append(dt)
        self.last_detail = np.concatenate(dets)
        duration = time.time() - t0
        logger.info('keypoints done, time consume: %.5f and %.5f per face' % (duration, duration / len(bboxes)))
        return np.concatenate(lms), np.concatenate(scs)
