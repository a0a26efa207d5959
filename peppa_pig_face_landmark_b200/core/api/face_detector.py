"""FaceDetector — same surface as the reference's Skps/core/api/face_detector.py:11-136
(`FaceDetector(cfg)(image) -> (K,16) float32`), with letterbox, the yolov5-face network,
score filter + greedy NMS and the un-letterbox all executed on the GPU by the kernels behind
include/skps_b200.h.  Host code only computes the letterbox geometry (python floats, exactly
as face_detector.py:51-62) and owns the containers."""
import ctypes as C
import os
import pathlib
import time

import numpy as np

from ... import runtime as rt
from ...graph_tools import detector_onnx_for
from ...logger.logger import logger
from .device_frames import check_host_frame
from .onnx_model_base import ONNXEngine


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


class FaceDetector:
    MAX_DET = 256           # kept rows skps_pipeline_run returns (FaceAna fetches the rest when there are more)

    def __init__(self, cfg):
        """cfg: Skps.yml's Detect section.  The engine is built for cfg['input_shape'] ([h, w, 3]): from the export itself
        when that is its input size, else from the export retargeted to (h, w) (graph_tools.detector_onnx_for; h and w
        multiples of 32 in 128..2176 x 128..3840), so the letterbox and the network always agree on the size."""
        root_path = pathlib.Path(__file__).resolve().parents[2]
        model_path = os.path.join(root_path, cfg['model_path'])
        self.input_size = cfg['input_shape']
        self.model = ONNXEngine(detector_onnx_for(model_path, self.input_size[:2]), max_batch=1)
        self.score_thrs = cfg['score_thrs']
        self.iou_thrs = cfg['iou_thrs']
        self.lib = rt.load_library()
        torch = rt.require_cuda()
        dev = self.model.device
        self._rows = self.model.out_elems[0] // 16
        # every detector row can be a kept box: output and NMS workspace for all of them, sized once here
        self._kept = torch.zeros((self._rows, 16), dtype=torch.float32, device=dev)
        self._idx = torch.zeros((self._rows,), dtype=torch.int32, device=dev)
        self._count = torch.zeros((1,), dtype=torch.int32, device=dev)
        self._recover = torch.zeros((3,), dtype=torch.float32, device=dev)
        self._ws_bytes = self.lib.skps_detect_post_workspace_size(self._rows, 1)
        self._ws = torch.empty((self._ws_bytes,), dtype=torch.uint8, device=dev)
        self.last_keep_idx = None

    # ------------------------------------------------------------------
    def _upload(self, image):
        torch = rt.require_cuda()
        return torch.from_numpy(check_host_frame(image)).to(self.model.device, non_blocking=False)

    def _letterbox_device(self, frame_dev, h, w):
        in_h, in_w = self.input_size[0], self.input_size[1]
        scale, rw, rh, top, left = letterbox_geometry(h, w, in_h, in_w)
        s = self.model.stream
        rt.check(self.lib.skps_letterbox(frame_dev.data_ptr(), h, w, w * 3, self.model.input_ptr(), in_h, in_w,
                                         rw, rh, top, left, s.cuda_stream))
        return [scale, left, top]

    def preprocess(self, image, color=(114, 114, 114)):
        """face_detector.py:45-71: returns ((1,3,H,W) float32 RGB/255, [scale, left, top])."""
        torch = rt.require_cuda()
        h, w = image.shape[:2]
        frame = self._upload(image)
        s = self.model.stream
        s.wait_stream(torch.cuda.current_stream(self.model.device))
        recover = self._letterbox_device(frame, h, w)
        s.synchronize()
        in_h, in_w = self.input_size[0], self.input_size[1]
        u8 = np.empty((in_h, in_w, 3), np.uint8)
        rt.check(self.lib.skps_engine_read_buffer(self.model.handle, self.model.plan.input.buf.idx, 1, u8.ctypes.data))
        img = u8.transpose(2, 0, 1).astype(np.float32)
        img /= 255.0
        return np.expand_dims(img, axis=0), recover

    def __call__(self, image):
        torch = rt.require_cuda()
        t0 = time.time()
        h, w = image.shape[:2]
        frame = self._upload(image)
        s = self.model.stream
        s.wait_stream(torch.cuda.current_stream(self.model.device))
        scale, left, top = self._letterbox_device(frame, h, w)
        rt.check(self.lib.skps_engine_forward(self.model.handle, self.model.input_ptr(), 1, None, s.cuda_stream))
        with torch.cuda.stream(s):
            self._recover.copy_(torch.tensor([scale, float(left), float(top)], dtype=torch.float32), non_blocking=False)
        rt.check(self.lib.skps_detect_post_batch(self.model.output_ptr(0), self._rows, 1, self.score_thrs, self.iou_thrs,
                                                 self._recover.data_ptr(), self._kept.data_ptr(), self._idx.data_ptr(),
                                                 self._count.data_ptr(), self._rows, self._ws.data_ptr(), self._ws_bytes,
                                                 s.cuda_stream))
        s.synchronize()
        n = int(self._count.item())
        bboxes = self._kept[:n].cpu().numpy()
        self.last_keep_idx = self._idx[:n].cpu().numpy().astype(np.int64)
        logger.info('detect done, time consume: %.5f' % (time.time() - t0))
        return bboxes
