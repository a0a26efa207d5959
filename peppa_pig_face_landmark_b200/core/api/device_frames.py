"""The frames FaceAna.run and FaceAnaStreams.submit accept, checked before anything is enqueued: numpy arrays, and frames
already in GPU memory (a decoder surface, a tensor from NVDEC / DALI / torchvision, an ROI view of either).  Pixels stay
HxWx3 uint8 BGR as the reference's run(image) takes them; only where the frame lives and its row pitch differ between the
two."""
import sys

import numpy as np


def check_host_frame(frame):
    """`frame` as a C-contiguous numpy array; ValueError unless it is an HxWx3 uint8 image."""
    frame = np.ascontiguousarray(frame)
    if frame.dtype != np.uint8 or frame.ndim != 3 or frame.shape[2] != 3:
        raise ValueError("expected an HxWx3 uint8 BGR image, got %s %s" % (frame.dtype, frame.shape))
    return frame


def is_cuda_tensor(x):
    """True for a torch tensor on a CUDA device (torch is not imported for anything else)."""
    torch = sys.modules.get("torch")
    return torch is not None and isinstance(x, torch.Tensor) and x.is_cuda


def is_tensor(x):
    torch = sys.modules.get("torch")
    return torch is not None and isinstance(x, torch.Tensor)


def check_cuda_frame(frame, device, max_hw):
    """(H, W, row pitch in bytes) of `frame`, a torch.uint8 CUDA tensor (H, W, 3) on `device` with interleaved channels:
    stride(2) == 1, stride(1) == 3 and stride(0) >= 3 W, so packed tensors, pitched surfaces and big[y0:y1, x0:x1] views
    all qualify.  ValueError for anything else, or for more pixels than max_hw = (max_h, max_w) allows."""
    if not is_tensor(frame):
        raise ValueError("expected a CUDA tensor, got %s" % type(frame).__name__)
    if not frame.is_cuda:
        raise ValueError("expected a CUDA tensor, got a tensor on %s" % frame.device)
    if str(frame.dtype) != "torch.uint8" or frame.dim() != 3 or frame.shape[2] != 3:
        raise ValueError("expected an HxWx3 uint8 BGR frame, got %s %s" % (frame.dtype, tuple(frame.shape)))
    if frame.device != device:
        raise ValueError("the frame is on %s, the pipeline on %s" % (frame.device, device))
    H, W = int(frame.shape[0]), int(frame.shape[1])
    if H < 1 or W < 1:
        raise ValueError("empty frame %s" % (tuple(frame.shape),))
    sy, sx, sc = frame.stride()
    if sc != 1 or (W > 1 and sx != 3) or (H > 1 and sy < 3 * W):
        raise ValueError("expected interleaved BGR pixels, strides (>= 3W, 3, 1); got strides %s for shape %s "
                         "(a planar or permuted view: pass .contiguous())" % ((sy, sx, sc), tuple(frame.shape)))
    if H * W > max_hw[0] * max_hw[1]:
        raise ValueError("frame %dx%d has more pixels than max_frame_hw %dx%d" % (H, W, max_hw[0], max_hw[1]))
    pitch = sy if H > 1 else 3 * W
    if pitch >= 2 ** 31:
        raise ValueError("row pitch %d does not fit 32 bits" % pitch)
    return H, W, pitch
