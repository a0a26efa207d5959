"""Aligned face chips on the GPU (csrc/align.cu): what a caller does with the 98 landmarks before a recognition, attribute
or expression model.

    chips, M = align_faces(frame, kps)      # kps (n, 98, 2) -> chips (n, 112, 112, 3) uint8 BGR, M (n, 2, 3) float64

M is the least-squares similarity (rotation, uniform scale, translation; no reflection; Umeyama 1991) from the landmarks
WFLW98_FIVE (pupils, nose tip, mouth corners) to ARCFACE_TEMPLATE_112 scaled by size/112, in float64, and every chip is
byte for byte cv2.warpAffine(frame, M, (size, size), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0).
FaceAna(align=size) and FaceAnaStreams(align=size) add the same 'chip' and 'M' to every result without uploading the
frame again.
"""
import numpy as np

from ... import runtime as rt

# ArcFace 112x112 five-point template: left eye, right eye, nose tip, left and right mouth corner (left / right as seen in
# the image).  A public data constant.
ARCFACE_TEMPLATE_112 = np.array([[38.2946, 51.6963], [73.5318, 51.5014], [56.0252, 71.7366],
                                 [41.5493, 92.3655], [70.7299, 92.2041]], np.float64)
# The WFLW-98 landmarks at those five points: left pupil, right pupil, nose tip, left and right mouth corner.
WFLW98_FIVE = (96, 97, 54, 76, 82)
MIN_SIZE, MAX_SIZE = 16, 512
MAX_WARP_SIDE = 4096


def check_size(size):
    """The chip side: an int in 16..512 (ValueError otherwise)."""
    if isinstance(size, (bool, np.bool_)) or not isinstance(size, (int, np.integer)) or not MIN_SIZE <= size <= MAX_SIZE:
        raise ValueError("align size must be an int in %d..%d, got %r" % (MIN_SIZE, MAX_SIZE, size))
    return int(size)


def _frame(image):
    if not isinstance(image, np.ndarray) or image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3 \
            or image.shape[0] < 1 or image.shape[1] < 1:
        raise ValueError("expected an HxWx3 uint8 BGR image, got %s" % (
            "%s %s" % (image.dtype, image.shape) if isinstance(image, np.ndarray) else type(image).__name__))
    return np.ascontiguousarray(image)


def check_kps(kps):
    """(n, P, 2) float64 landmarks with P >= 98, finite, whose five alignment points are not all one point."""
    k = np.asarray(kps, dtype=np.float64)
    if k.ndim != 3 or k.shape[1] < 98 or k.shape[2] != 2:
        raise ValueError("expected landmarks of shape (n, 98, 2), got %s" % (k.shape,))
    if not np.isfinite(k).all():
        raise ValueError("landmarks must be finite")
    five = k[:, list(WFLW98_FIVE)]
    spread = ((five - five.mean(axis=1, keepdims=True)) ** 2).sum(axis=(1, 2))
    if (spread == 0).any():
        raise ValueError("the five alignment points of face %d coincide" % int(np.flatnonzero(spread == 0)[0]))
    return np.ascontiguousarray(k)


def warp_affine(image, M, dsize):
    """cv2.warpAffine(image, M[i], dsize, INTER_LINEAR, BORDER_CONSTANT, 0) for every i, on the GPU.
    image HxWx3 uint8, M (n, 2, 3) (any affine, float64), dsize (w, h) -> (n, h, w, 3) uint8."""
    image = _frame(image)
    M = np.asarray(M, dtype=np.float64)
    if M.ndim != 3 or M.shape[1:] != (2, 3):
        raise ValueError("expected matrices of shape (n, 2, 3), got %s" % (M.shape,))
    if not np.isfinite(M).all():
        raise ValueError("matrices must be finite")
    try:
        w, h = (int(v) for v in dsize)
    except (TypeError, ValueError):
        raise ValueError("dsize must be (width, height), got %r" % (dsize,)) from None
    if not (1 <= w <= MAX_WARP_SIDE and 1 <= h <= MAX_WARP_SIDE):
        raise ValueError("dsize %r outside 1..%d" % (dsize, MAX_WARP_SIDE))
    n = M.shape[0]
    if n == 0:
        return np.zeros((0, h, w, 3), np.uint8)
    torch = rt.require_cuda()
    lib = rt.load_library()
    H, W = image.shape[:2]
    frame = torch.from_numpy(image).cuda()
    m = torch.from_numpy(np.ascontiguousarray(M)).cuda()
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=frame.device)
    with torch.cuda.device(frame.device):
        rt.check(lib.skps_warp_affine(frame.data_ptr(), H, W, W * 3, m.data_ptr(), None, n, h, w, out.data_ptr(),
                                      torch.cuda.current_stream(frame.device).cuda_stream))
    return out.cpu().numpy()


def align_faces(image, kps, size=112):
    """Aligned chips for n faces of one frame: kps (n, 98, 2) -> (chips (n, size, size, 3) uint8 BGR, M (n, 2, 3) float64)."""
    image = _frame(image)
    size = check_size(size)
    k = check_kps(kps)
    n = k.shape[0]
    if n == 0:
        return np.zeros((0, size, size, 3), np.uint8), np.zeros((0, 2, 3), np.float64)
    torch = rt.require_cuda()
    lib = rt.load_library()
    H, W = image.shape[:2]
    frame = torch.from_numpy(image).cuda()
    dk = torch.from_numpy(k).cuda()
    chips = torch.empty((n, size, size, 3), dtype=torch.uint8, device=frame.device)
    M = torch.empty((n, 2, 3), dtype=torch.float64, device=frame.device)
    with torch.cuda.device(frame.device):
        rt.check(lib.skps_align_faces(frame.data_ptr(), H, W, W * 3, dk.data_ptr(), None, n, k.shape[1], size,
                                      chips.data_ptr(), M.data_ptr(), torch.cuda.current_stream(frame.device).cuda_stream))
    return chips.cpu().numpy(), M.cpu().numpy()
