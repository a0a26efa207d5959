"""Aligned face chips on the GPU (csrc/align.cu): what a caller does with the 98 landmarks before a recognition, attribute
or expression model.

    chips, M = align_faces(frame, kps)      # kps (n, 98, 2) -> chips (n, 112, 112, 3) uint8 BGR, M (n, 2, 3) float64

M is the least-squares similarity (rotation, uniform scale, translation; no reflection; Umeyama 1991) from the landmarks
WFLW98_FIVE (pupils, nose tip, mouth corners) to ARCFACE_TEMPLATE_112 scaled by size/112, in float64, and every chip is
byte for byte cv2.warpAffine(frame, M, (size, size), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0).
FaceAna(align=size) and FaceAnaStreams(align=size) add the same 'chip' and 'M' to every result without uploading the
frame again; FaceAnaImages(align=size) and FaceLandmark(align=size) do it for faces of many images per call, uploading
of a host image only the rectangle each chip reads (chip_read_rects).
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


def chip_read_rects(M, size, H, W):
    """(n, 4) int64 [x0, y0, x1, y1) per matrix of M (n, 2, 3): the smallest rectangle of an H x W image that holds every
    pixel inside the image that the size x size warp of M (skps_warp_faces, cv2.warpAffine) reads; all zero when the chip
    reads no pixel of the image, and the whole image when a source coordinate of the warp leaves int32 (cvRound's INT_MIN,
    or the wrap of OpenCV's int arithmetic).  FaceLandmark(align=...) uploads only these rectangles of host frames.

    The inverse map is computed in float64 in the kernel's order of operations (numpy does not fuse, align.cu is built
    with -fmad=false).  Chip pixel (x, y) reads columns sx, sx + 1 with sx = sat_short((X0[y] + adelta[x]) >> 10),
    X0[y] = cvRound((m1 * y + m2) * 1024) + 16, adelta[x] = cvRound(m0 * x * 1024), and rows the same way.  adelta is
    monotone in x, so in each chip row the pixels with a column and a row tap inside the image form one run of x, found by
    binary search, and sx, sy are extreme at the ends of the runs.  O(size log size) per face."""
    M = np.asarray(M, np.float64).reshape(-1, 6)
    n, s = M.shape[0], int(size)
    out = np.zeros((n, 4), np.int64)
    if n == 0:
        return out
    m0, m1, m2, m3, m4, m5 = (M[:, j, None] for j in range(6))
    t = np.arange(s, dtype=np.float64)
    with np.errstate(all="ignore"):
        D = m0 * m4 - m1 * m3
        D = np.where(D != 0.0, 1.0 / np.where(D != 0.0, D, 1.0), 0.0)
        m0, m4, m1, m3 = m4 * D, m0 * D, m1 * -D, m3 * -D
        m2, m5 = -m0 * m2 - m1 * m5, -m3 * m2 - m4 * m5
        # per face: row terms (n, s) and column terms (n, s) in 1/1024 px
        raw = [(m1 * t + m2) * 1024.0, m0 * t * 1024.0, (m4 * t + m5) * 1024.0, m3 * t * 1024.0]
    bad = np.zeros(n, bool)
    for r in raw:
        bad |= ~(np.abs(r) < 2147483647.5).all(1)              # cvRound -> INT_MIN
    X0, ad, Y0, bd = (np.rint(np.where(bad[:, None], 0.0, r)).astype(np.int64) for r in raw)
    X0 += 16
    Y0 += 16
    for r0, d in ((X0, ad), (Y0, bd)):
        bad |= (r0.max(1) > 2**31 - 1)                          # the + 16 wraps
        bad |= (r0.min(1) + d.min(1) < -2**31) | (r0.max(1) + d.max(1) > 2**31 - 1)
    X0, ad, Y0, bd = (np.where(bad[:, None], 0, v) for v in (X0, ad, Y0, bd))

    face = np.arange(n, dtype=np.int64)[:, None]

    def run(r0, d, side):
        """Per face and chip row: the run [a, b] of x whose tap sat_short(v >> 10), v = r0[y] + d[x], is in
        [-1, side - 1] (a column or row tap inside the image); a > b when there is none."""
        lo, hi = -1024, (side * 1024 - 1 if side <= 32767 else 2**40)
        rev = d[:, -1] < d[:, 0]
        asc = np.where(rev[:, None], d[:, ::-1], d)
        key = (asc + face * 2**35).ravel()                      # one sorted array for all faces
        q0 = np.clip(lo - r0, -2**33, 2**33) + face * 2**35
        q1 = np.clip(hi - r0, -2**33, 2**33) + face * 2**35
        ka = np.searchsorted(key, q0, "left") - face * s
        kb = np.searchsorted(key, q1, "right") - face * s - 1
        a = np.where(rev[:, None], s - 1 - kb, ka)
        b = np.where(rev[:, None], s - 1 - ka, kb)
        return a, b

    ax, bx = run(X0, ad, W)
    ay, by = run(Y0, bd, H)
    a, b = np.maximum(ax, ay), np.minimum(bx, by)
    ok = a <= b
    a, b = np.where(ok, a, 0), np.where(ok, b, 0)

    def tap(r0, d, x):
        return np.clip((r0 + np.take_along_axis(d, x, 1)) >> 10, -32768, 32767)

    lo, hi = [], []
    for r0, d in ((X0, ad), (Y0, bd)):
        ends = np.stack([tap(r0, d, a), tap(r0, d, b)])
        lo.append(np.where(ok, ends, 2**40).min(axis=(0, 2)))
        hi.append(np.where(ok, ends, -2**40).max(axis=(0, 2)))
    rect = np.stack([np.maximum(lo[0], 0), np.maximum(lo[1], 0), np.minimum(hi[0] + 2, W), np.minimum(hi[1] + 2, H)], 1)
    reads = ok.any(1)
    out[reads] = rect[reads]
    out[bad] = (0, 0, W, H)
    return out


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
