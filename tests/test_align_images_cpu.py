"""core/api/align.py:chip_read_rects, the rectangle of a host image that FaceLandmark(align=...) and
FaceAnaImages(align=...) upload for a chip, against the taps of every chip pixel enumerated with oracle/align_ref.py's
restatement of cv2.warpAffine's fixed-point arithmetic.  No GPU."""
import math

import numpy as np
import pytest

from oracle.align_ref import AB_BITS, AB_SCALE, INTER_BITS, INTER_TAB, _cv_round, _i32


def taps(M, size, H, W):
    """(x0, y0, x1, y1) [x0, x1) x [y0, y1): the tight box of every tap inside the H x W image that the size x size warp
    of M reads, all zero when there is none, and whether every source coordinate stayed in int32 (no wrap, no INT_MIN):
    warp_affine_u8's arithmetic, pixel by pixel."""
    m = [float(x) for x in np.asarray(M, np.float64).reshape(6)]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = m[4] * D, m[0] * D
    m[0], m[4] = A11, A22
    m[1] *= -D
    m[3] *= -D
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    t = np.arange(size, dtype=np.float64)
    with np.errstate(all="ignore"):
        raw = [(m[1] * t + m[2]) * AB_SCALE, m[0] * t * AB_SCALE, (m[4] * t + m[5]) * AB_SCALE, m[3] * t * AB_SCALE]
    exact = all((np.abs(r) < 2147483647.5).all() for r in raw)
    adelta, bdelta = _cv_round(raw[1]), _cv_round(raw[3])
    rd = AB_SCALE // INTER_TAB // 2
    X0, Y0 = _cv_round(raw[0]) + rd, _cv_round(raw[2]) + rd
    vx, vy = X0[:, None] + adelta[None, :], Y0[:, None] + bdelta[None, :]
    exact = exact and all(np.array_equal(_i32(v), v) for v in (X0, Y0, vx, vy))
    X = _i32(_i32(X0)[:, None] + adelta[None, :]) >> (AB_BITS - INTER_BITS)
    Y = _i32(_i32(Y0)[:, None] + bdelta[None, :]) >> (AB_BITS - INTER_BITS)
    sx = np.clip(X >> INTER_BITS, -32768, 32767)
    sy = np.clip(Y >> INTER_BITS, -32768, 32767)
    xs, ys = [], []
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        tx, ty = sx + dx, sy + dy
        inside = (tx >= 0) & (tx < W) & (ty >= 0) & (ty < H)
        xs.append(tx[inside])
        ys.append(ty[inside])
    xs, ys = np.concatenate(xs), np.concatenate(ys)
    if not len(xs):
        return (0, 0, 0, 0), exact
    return (int(xs.min()), int(ys.min()), int(xs.max()) + 1, int(ys.max()) + 1), exact


def similarity(angle_deg, scale, tx, ty):
    c, s = scale * math.cos(math.radians(angle_deg)), scale * math.sin(math.radians(angle_deg))
    return np.array([[c, -s, tx], [s, c, ty]], np.float64)


def _check(Ms, size, H, W):
    from peppa_pig_face_landmark_b200.core.api.align import chip_read_rects
    got = chip_read_rects(np.asarray(Ms), size, H, W)
    assert got.shape == (len(Ms), 4) and got.dtype == np.int64
    kinds = {"inside": 0, "partly": 0, "outside": 0, "fallback": 0}
    for i, M in enumerate(Ms):
        want, exact = taps(M, size, H, W)
        if not exact:
            kinds["fallback"] += 1
            assert tuple(got[i]) == (0, 0, W, H), (i, M, got[i])
            continue
        assert tuple(got[i]) == want, (i, M.tolist(), size, H, W, got[i], want)
        area = (want[2] - want[0]) * (want[3] - want[1])
        edge = want[0] == 0 or want[1] == 0 or want[2] == W or want[3] == H
        kinds["outside" if area == 0 else "partly" if edge else "inside"] += 1
    return kinds


def _chip_matrix(rng, size, H, W, angle, scale):
    """A similarity frame -> chip that takes a face of side ~ size / scale somewhere in or around the image."""
    cx, cy = rng.uniform(-0.3 * W, 1.3 * W), rng.uniform(-0.3 * H, 1.3 * H)
    M = similarity(angle, scale, 0.0, 0.0)
    M[:, 2] = size / 2 - M[:, :2] @ np.array([cx, cy])
    return M


@pytest.mark.parametrize("size", [16, 112, 512])
def test_similarities_equal_the_enumerated_taps(size):
    rng = np.random.default_rng(size)
    H, W = 480, 640
    Ms = []
    for angle in (0.0, 45.0, 90.0, 180.0, -30.0, 135.0):
        for scale in (1 / 50, 1 / 7, 0.5, 1.0, 2.5, 50.0):
            for _ in range(4):
                Ms.append(_chip_matrix(rng, size, H, W, angle + rng.uniform(-1, 1) * (angle not in (0, 90, 180)),
                                       scale))
    for _ in range(40):
        Ms.append(_chip_matrix(rng, size, H, W, rng.uniform(-180, 180), math.exp(rng.uniform(-4, 4))))
    kinds = _check(Ms, size, H, W)
    assert min(kinds["outside"], kinds["partly"], kinds["inside"]) > 0, kinds


def test_shears_and_degenerate_matrices():
    rng = np.random.default_rng(7)
    H, W = 300, 200
    Ms = [rng.uniform(-2, 2, (2, 3)) * [1, 1, 100] + [0, 0, 50] for _ in range(60)]          # shears, reflections
    Ms += [np.zeros((2, 3)), np.array([[1.0, 2.0, 3.0], [2.0, 4.0, 6.0]]),                 # D == 0
           np.array([[0.0, 0.0, 10.0], [0.0, 0.0, -5.0]])]
    Ms += [np.eye(2, 3), np.array([[1.0, 0, -0.5], [0, 1.0, -0.5]]), np.array([[1.0, 0, 1e-9], [0, 1.0, 0]])]
    for dx, dy in ((W - 0.5, 0), (0, H - 0.5), (-W + 0.49, 0), (W + 0.5, H + 0.5)):
        Ms.append(np.array([[1.0, 0, -dx], [0, 1.0, -dy]]))                                # at the image's edges
    _check(Ms, 64, H, W)


def test_int32_fallback_is_the_whole_image():
    H, W = 100, 120
    Ms = [np.array([[1e-7, 0, 0], [0, 1e-7, 0]]),            # an inverse scale of 1e7: cvRound leaves int32
          np.array([[1.0, 0, -2.097e6], [0, 1.0, 0]]),       # X0 near INT_MAX: the sums wrap
          np.array([[1e-5, 0, 0.0], [0, 1.0, 0]])]           # adelta leaves int32 within the chip
    kinds = _check(Ms, 512, H, W)
    assert kinds["fallback"] == len(Ms), kinds


def test_big_images_and_no_matrices():
    from peppa_pig_face_landmark_b200.core.api.align import chip_read_rects
    assert chip_read_rects(np.zeros((0, 2, 3)), 112, 10, 10).shape == (0, 4)
    rng = np.random.default_rng(11)
    H, W = 40000, 50000                                      # sides past sat_short's 32767
    Ms = [_chip_matrix(rng, 112, H, W, rng.uniform(-180, 180), math.exp(rng.uniform(-7, 0))) for _ in range(30)]
    Ms.append(np.array([[1.0, 0, -32760.0], [0, 1.0, -32700.0]]))
    _check(Ms, 112, H, W)
