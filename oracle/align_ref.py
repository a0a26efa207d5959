"""ORACLE for aligned face chips (peppa_pig_face_landmark_b200/core/api/align.py, csrc/align.cu).

Two numpy restatements, float64 throughout:
  * umeyama(src, dst): the least-squares similarity (rotation, uniform scale, translation; no reflection) mapping src onto
    dst, in the SVD form of Umeyama 1991 ("Least-squares estimation of transformation parameters between two point
    patterns", eq. 40-42).  Returns the 2x3 matrix one passes to cv2.warpAffine.
  * warp_affine_u8(img, M, size): cv2.warpAffine(img, M, (w, h), INTER_LINEAR, BORDER_CONSTANT, 0) written out with
    OpenCV's fixed-point arithmetic: the inverse map in double, source coordinates in 1/1024 px rounded to 1/32 px,
    integer bilinear weights summing to 2^15.
cv2 stays the authority: the restatement pins which arithmetic the installed OpenCV uses, so that a change of OpenCV can be
told apart from a kernel bug.
"""
import numpy as np

# ArcFace 112x112 five-point template (left eye, right eye, nose tip, left / right mouth corner; left/right as seen in the
# image) and the WFLW-98 landmarks that correspond to it.
ARCFACE_TEMPLATE_112 = np.array([[38.2946, 51.6963], [73.5318, 51.5014], [56.0252, 71.7366],
                                 [41.5493, 92.3655], [70.7299, 92.2041]], np.float64)
WFLW98_FIVE = (96, 97, 54, 76, 82)

AB_BITS, INTER_BITS = 10, 5
AB_SCALE, INTER_TAB = 1 << AB_BITS, 1 << INTER_BITS
COEF_BITS = 15


def template(size):
    return ARCFACE_TEMPLATE_112 * (size / 112.0)


def umeyama(src, dst):
    src = np.asarray(src, np.float64)
    dst = np.asarray(dst, np.float64)
    n = src.shape[0]
    mu_s, mu_d = src.mean(0), dst.mean(0)
    a, b = src - mu_s, dst - mu_d
    var_s = (a * a).sum() / n
    cov = b.T @ a / n
    U, D, Vt = np.linalg.svd(cov)
    S = np.eye(2)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[1, 1] = -1
    R = U @ S @ Vt
    c = np.trace(np.diag(D) @ S) / var_s
    t = mu_d - c * R @ mu_s
    return np.hstack([c * R, t[:, None]])


def align_matrix(kps98, size=112):
    """M (2,3) float64 for one face's 98 landmarks."""
    pts = np.asarray(kps98, np.float64)[list(WFLW98_FIVE)]
    return umeyama(pts, template(size))


def _cv_round(v):
    """cvRound on x86 (cvtsd2si): round half to even; out of int32 range or NaN -> INT_MIN."""
    v = np.asarray(v, np.float64)
    bad = ~(np.abs(v) < 2147483647.5)
    r = np.rint(np.where(bad, 0.0, v)).astype(np.int64)
    return np.where(bad, np.int64(-2147483648), r)


def _i32(v):
    return np.asarray(v, np.int64).astype(np.int32).astype(np.int64)      # two's-complement wrap of int arithmetic


def warp_affine_u8(img, M, dsize):
    """cv2.warpAffine(img, M, dsize=(w, h), flags=INTER_LINEAR, borderMode=BORDER_CONSTANT, borderValue=0), HxWxC uint8."""
    img = np.asarray(img)
    assert img.dtype == np.uint8 and img.ndim == 3
    H, W, C = img.shape
    w, h = int(dsize[0]), int(dsize[1])
    m = [float(x) for x in np.asarray(M, np.float64).reshape(6)]
    # invertAffineTransform as warpAffine does it (imgwarp.cpp), same order of operations
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = m[4] * D, m[0] * D
    m[0], m[4] = A11, A22
    m[1] *= -D
    m[3] *= -D
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    xs = np.arange(w, dtype=np.float64)
    ys = np.arange(h, dtype=np.float64)
    adelta = _cv_round(m[0] * xs * AB_SCALE)
    bdelta = _cv_round(m[3] * xs * AB_SCALE)
    rd = AB_SCALE // INTER_TAB // 2
    X0 = _i32(_cv_round((m[1] * ys + m[2]) * AB_SCALE) + rd)
    Y0 = _i32(_cv_round((m[4] * ys + m[5]) * AB_SCALE) + rd)
    X = _i32(X0[:, None] + adelta[None, :]) >> (AB_BITS - INTER_BITS)
    Y = _i32(Y0[:, None] + bdelta[None, :]) >> (AB_BITS - INTER_BITS)
    sx = np.clip(X >> INTER_BITS, -32768, 32767)
    sy = np.clip(Y >> INTER_BITS, -32768, 32767)
    fx, fy = X & (INTER_TAB - 1), Y & (INTER_TAB - 1)
    wts = [(INTER_TAB - fx) * (INTER_TAB - fy), fx * (INTER_TAB - fy), (INTER_TAB - fx) * fy, fx * fy]
    acc = np.zeros((h, w, C), np.int64)
    for k, (dx, dy) in enumerate([(0, 0), (1, 0), (0, 1), (1, 1)]):
        tx, ty = sx + dx, sy + dy
        inside = (tx >= 0) & (tx < W) & (ty >= 0) & (ty < H)
        v = img[np.where(inside, ty, 0), np.where(inside, tx, 0)].astype(np.int64)
        v[~inside] = 0
        acc += v * (wts[k] * ((1 << COEF_BITS) // (INTER_TAB * INTER_TAB)))[..., None]
    out = (acc + (1 << (COEF_BITS - 1))) >> COEF_BITS
    return np.clip(out, 0, 255).astype(np.uint8)
