"""Head pose (csrc/headpose.cu) beyond the frontal faces of test_headpose_gpu: its rotation helpers at the rotations where
they are ill-conditioned, and its solver over the whole pose space, small and far faces included, checked against a
converged float64 solve rather than only against cv2.

Why not only against cv2: cv2.solvePnP stops after 20 Levenberg-Marquardt iterations.  On small noisy faces that is often
not converged (test_stationarity_check_has_teeth shows faces whose Euler angles are far from the converged minimum of the
same problem), so "equal to cv2" is asked only where cv2 itself passes the stationarity test below.  Everywhere the
kernel's solution must be no worse than cv2's, and a stationary point of the reprojection error wherever cv2's is; where
cv2's is not, a few small noisy faces per hundred lie in long flat valleys that the kernel's 100 iterations do not cross
either (at most 2 % of the faces of a frame size).

The stationarity test: at (rvec, tvec) with residuals e (20 pixel coordinates) and Jacobian J = d e / d(rvec, tvec)
(cv2.projectPoints' first six columns, analytic, float64),
    |J^T e| <= |J|_F * (STATIONARY * |e| + eta).
STATIONARY = 1e-6: the kernel differentiates numerically (central differences, h = 1e-6 max(1, |p_j|)), and a residual
of up to 4e3 px evaluated in float64 (2.2e-16 relative) divided by 2h leaves about 1e-7 px per unit parameter in J, so
its own stationary point has |J^T e| / (|J| |e|) down to about 1e-7 of |J|; cv2's converged answers sit at 1e-7 and
below; a rotation off by 1e-4 rad gives 2e-5 or more on the smallest faces (test_stationarity_check_has_teeth).
eta = 1e-12 |J|_F + 1e-14 * max|uv| * sqrt(20): the solver stops on a step below 1e-12, and the residuals themselves carry
float64 rounding of a few ulp of the pixel coordinates - both matter only on noise-free faces, where |e| is only the
float32 rounding of the image points (~1e-4 px)."""
import math

import numpy as np
import pytest

EPS = np.finfo(np.float64).eps
DEG = 180.0 / math.pi
STATIONARY = 1e-6
FRAMES = [(480, 640), (1080, 1920), (2160, 3840), (721, 1281)]     # (h, w); 1281 x 721 has odd cx = W // 2, cy = H // 2


def _obj():
    from peppa_pig_face_landmark_b200.core.headpose.pose import object_pts
    return object_pts


def _camera(hw):
    h, w = hw
    return np.array([[w, 0.0, w // 2], [0.0, w, h // 2], [0.0, 0.0, 1.0]])


def _Rx(a):
    return np.array([[1, 0, 0], [0, math.cos(a), -math.sin(a)], [0, math.sin(a), math.cos(a)]])


def _Ry(a):
    return np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])


def _Rz(a):
    return np.array([[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1]])


def _compose(euler_deg):
    """The rotation an RQDecomp3x3 Euler triple stands for: R = Rz(roll) Ry(yaw) Rx(pitch)."""
    a, b, c = np.radians(euler_deg)
    return _Rz(c) @ _Ry(b) @ _Rx(a)


# ------------------------------------------------------------------------------------------------------------------
# the float64 yardstick: residuals, Jacobian, cost and the stationarity test


def residuals(img, rvec, tvec, hw):
    """-> (e (20,), J (20,6), uv (10,2)): reprojection residuals of the 10 model points and their analytic Jacobian."""
    import cv2
    uv, jac = cv2.projectPoints(_obj().astype(np.float64), np.asarray(rvec, np.float64).reshape(3, 1),
                                np.asarray(tvec, np.float64).reshape(3, 1), _camera(hw), None)
    uv = uv.reshape(10, 2)
    return (uv - np.asarray(img, np.float32).astype(np.float64)).reshape(20), jac[:, :6], uv


def cost(img, rvec, tvec, hw):
    e = residuals(img, rvec, tvec, hw)[0]
    return float(e @ e)


def stationarity(img, rvec, tvec, hw):
    """-> (ratio, bound): |J^T e| / (|J|_F |e|) and the largest value the test accepts for this face."""
    e, J, uv = residuals(img, rvec, tvec, hw)
    nJ, ne = np.linalg.norm(J), np.linalg.norm(e)
    eta = 1e-12 * nJ + 1e-14 * np.abs(uv).max() * math.sqrt(20)
    g = np.linalg.norm(J.T @ e)
    return g / (nJ * ne), (STATIONARY * ne + eta) / ne


def is_stationary(img, rvec, tvec, hw):
    r, bound = stationarity(img, rvec, tvec, hw)
    return bool(r <= bound)


def not_worse_bound(img, rvec, tvec, hw):
    """Largest cost a solution may have to count as no worse than (rvec, tvec): its cost (1 + 1e-9), plus the float64
    rounding of the two evaluations (residuals within 4 ulp of the pixel coordinates: 2 |e| delta + delta^2)."""
    e, _, uv = residuals(img, rvec, tvec, hw)
    delta = 4 * EPS * np.abs(uv).max() * math.sqrt(20)
    c = float(e @ e)
    return c * (1 + 1e-9) + 2 * math.sqrt(c) * delta + delta * delta


def cv2_solve(img, hw):
    import cv2
    ok, rvec, tvec = cv2.solvePnP(_obj(), np.asarray(img, np.float32), _camera(hw).astype(np.float32),
                                  np.zeros((5, 1), np.float32))
    assert ok
    return rvec.reshape(3), tvec.reshape(3)


def cv2_euler(rvec, tvec):
    import cv2
    rot = cv2.Rodrigues(np.asarray(rvec, np.float64).reshape(3, 1))[0]
    return cv2.decomposeProjectionMatrix(cv2.hconcat((rot, np.asarray(tvec, np.float64).reshape(3, 1))))[6].reshape(3)


def synthetic_face(rng, hw, size, noise, R=None):
    """One face of about `size` px (the model's eye-corner span is 13.65 units) at a random place in the frame, with
    yaw within +-80 degrees, pitch +-50 and any roll unless R is given -> (10,2) float32 image points, R, t."""
    h, w = hw
    if R is None:
        R = _Rz(rng.uniform(-math.pi, math.pi)) @ _Ry(math.radians(rng.uniform(-80, 80))) @ \
            _Rx(math.radians(rng.uniform(-50, 50))) @ _Rx(math.pi)
    z = w * 13.65 / size
    m = 0.5 * min(size, w, h)
    u0, v0 = rng.uniform(m, w - m), rng.uniform(m, h - m)
    t = np.array([(u0 - w // 2) * z / w, (v0 - h // 2) * z / w, z])
    X = _obj().astype(np.float64) @ R.T + t
    uv = np.stack([w * X[:, 0] / X[:, 2] + w // 2, w * X[:, 1] / X[:, 2] + h // 2], 1)
    return (uv + rng.normal(0, noise, (10, 2)) if noise else uv).astype(np.float32), R, t


def _angle_diff(a, b):
    d = np.abs(np.asarray(a) - np.asarray(b)) % 360
    return np.minimum(d, 360 - d)


# ------------------------------------------------------------------------------------------------------------------
# the checker itself (no GPU)


def test_stationarity_check_has_teeth():
    """Small faces in a 1920 x 1080 frame (20-45 px, 0.8 px noise): cv2.solvePnP's 20-iteration answers that are more than
    1e-3 degrees away from the converged minimum must fail the test, the converged minimum (solvePnPRefineLM to 2000
    iterations) must pass it, and the converged minimum with the rotation moved by 1e-4 rad must fail it."""
    import cv2
    hw = (1080, 1920)
    rng = np.random.default_rng(20)
    K32, dist = _camera(hw).astype(np.float32), np.zeros((5, 1), np.float32)
    unconverged = wandered = 0
    for i in range(300):
        img = synthetic_face(rng, hw, rng.uniform(20, 45), 0.8)[0]
        rvec, tvec = cv2_solve(img, hw)
        r2, t2 = cv2.solvePnPRefineLM(_obj(), img, K32, dist, rvec.reshape(3, 1).copy(), tvec.reshape(3, 1).copy(),
                                      (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 2000, 1e-300))
        r2, t2 = r2.reshape(3), t2.reshape(3)
        if t2[2] <= 0 or cost(img, r2, t2, hw) > cost(img, rvec, tvec, hw):
            wandered += 1                                  # refined to a point behind the camera: no minimum to compare
            continue
        assert is_stationary(img, r2, t2, hw), (i, stationarity(img, r2, t2, hw))
        if _angle_diff(cv2_euler(rvec, tvec), cv2_euler(r2, t2)).max() > 1e-3:
            unconverged += 1
            assert not is_stationary(img, rvec, tvec, hw), (i, stationarity(img, rvec, tvec, hw))
        for axis in np.eye(3):
            assert not is_stationary(img, r2 + 1e-4 * axis, t2, hw), (i, axis)
    assert unconverged >= 3 and wandered <= 30, (unconverged, wandered)   # the regime really holds unconverged answers


# ------------------------------------------------------------------------------------------------------------------
# the rotation helpers (rodrigues, rodrigues_inv, euler_rq) on their own


def debug_rotation(r, R):
    """The kernel's rodrigues(r), rodrigues_inv(R) and euler_rq(R), run in device code (skps_debug_rotation)."""
    from peppa_pig_face_landmark_b200 import runtime as rt
    rt.require_cuda()
    lib = rt.load_library()
    r = np.ascontiguousarray(r, np.float64).reshape(-1, 3)
    R = np.ascontiguousarray(R, np.float64).reshape(-1, 3, 3)
    n = len(r)
    R_out, r_out, euler = np.zeros((n, 3, 3)), np.zeros((n, 3)), np.zeros((n, 3))
    rt.check(lib.skps_debug_rotation(r.ctypes.data, R.ctypes.data, n, R_out.ctypes.data, r_out.ctypes.data,
                                     euler.ctypes.data))
    return R_out, r_out, euler


def _rotation_cases():
    """-> r (n,3), R (n,3,3) = cv2.Rodrigues(r) (or r = cv2.Rodrigues(R) for the cases given as matrices), axis_pi (n,)
    True for the exact 180-degree rotations about the 26 axes of {-1,0,1}^3."""
    import cv2
    rng = np.random.default_rng(90)
    rs, Rs, axis_pi = [], [], []

    def add_r(r, is_pi=False):
        r = np.asarray(r, np.float64)
        rs.append(r), Rs.append(cv2.Rodrigues(r)[0]), axis_pi.append(is_pi)

    def add_R(R):
        R = np.asarray(R, np.float64)
        rs.append(cv2.Rodrigues(R)[0].reshape(3)), Rs.append(R), axis_pi.append(False)

    q = rng.normal(size=(20000, 4))                        # uniform rotations: normalised Gaussian quaternions
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q *= np.where(q[:, :1] < 0, -1, 1)
    for w, *v in q:
        v = np.array(v)
        add_r(v / np.linalg.norm(v) * 2 * math.acos(min(w, 1.0)))
    axes = [np.array([1.0, 0, 0]), np.array([0, 1.0, 0]), np.array([0, 0, 1.0])] + \
        [a / np.linalg.norm(a) for a in rng.normal(size=(5, 3))]
    for k in range(1, 14):                                 # theta = pi - 10^-k and 10^-k
        for a in axes:
            add_r(a * (math.pi - 10.0 ** -k))
            add_r(a * 10.0 ** -k)
    for a in np.array(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1])).reshape(3, -1).T:
        if a.any():                                        # exactly pi about each axis of {-1,0,1}^3
            add_r(a / np.linalg.norm(a) * math.pi, True)
    for d in [0.0] + [10.0 ** -k for k in range(12, 1, -1)]:   # yaw +-90 degrees - delta (gimbal lock at delta = 0)
        for sgn in (1, -1):
            for pitch, roll in [(0, 0), (20, -30), (-45, 170)]:
                add_R(_Rz(math.radians(roll)) @ _Ry(sgn * (math.pi / 2 - d)) @ _Rx(math.radians(pitch)) @ _Rx(math.pi))
    for roll in (90, 135, 170, 179, 179.9, 180):            # frontal faces rolled far over
        for sgn in (1, -1):
            add_R(_Rz(sgn * math.radians(roll)) @ _Rx(math.pi))
    return np.array(rs), np.array(Rs), np.array(axis_pi)


@pytest.mark.gpu
def test_rotation_helpers_match_opencv():
    """Bounds, from the conditioning of each map (EPS = 2.2e-16, the float64 rounding unit):
    - rodrigues: every entry is c + k_i k_j (1 - c) +- k s, three terms of magnitude <= 1, cos / sin within 2 ulp on the
      GPU: 1e-14.
    - rodrigues_inv: r = theta / (2 s) (R - R^T)v with s = sin(theta); rounding of R (EPS absolute) moves the vector by
      EPS / s relative, so 16 EPS (1 + pi / s).  Where s < 1e-5 the kernel, like OpenCV, rebuilds the axis from the
      diagonal only, sqrt((R_ii + 1) / 2).  Both run that same formula, so they differ only by its rounding, and sqrt
      turns an ulp in the argument of a near-zero component into sqrt(2 EPS): 4 pi sqrt(2 EPS) ~ 2.6e-7.  (How far the
      formula is from the true r, up to pi - theta, is the same for both and not what is compared.)  Near pi, r and -r
      differ by at most 2 (pi - theta) < 2e-5 in rotation, so the sign is not compared there.  Below s = 1e-5 near zero both return 0: |r| <= theta.
    - euler_rq: each angle is acos of a normalised Givens cosine; acos' slope is infinite at +-1, so an ulp there costs
      sqrt(2 ulp) ~ 2e-8 rad; the first Givens pair has norm cos(yaw) and OpenCV's normalisation 1 / sqrt(c^2 + s^2 + EPS)
      moves its angle by up to sqrt(2 EPS) / cos(yaw); the pitch / roll cosines are divided by cos(yaw):
      DEG (8 sqrt(EPS) + sqrt(2 EPS) / cos yaw + 64 EPS / cos^2 yaw),
      asked where |cos yaw| >= 1e-3 and R is not an exact axis-pi rotation.  Where the pitch is 0 or 180 degrees to
      rounding, (p, y, r) and (p + 180, 180 - y, r + 180) are the same rotation and OpenCV 4.13 sometimes picks the other
      one (Ry(pi - 0.1): (180, 5.73, 180) here, (0, 174.27, 0) from cv2), so either is accepted there.  Everywhere, the triple
      must compose back to R within three acos errors, 3 sqrt(8 EPS), plus the Givens normalisation's sqrt(2 EPS) / cos(yaw),
      used down to cos(yaw) = 1e-3 (below that the kernel normalises exactly)."""
    import cv2
    r, R, axis_pi = _rotation_cases()
    R_out, r_out, euler = debug_rotation(r, R)
    for i in range(len(r)):
        assert np.abs(R_out[i] - cv2.Rodrigues(r[i])[0]).max() <= 1e-14, (i, r[i])

        rc = cv2.Rodrigues(R[i])[0].reshape(3)
        th = np.linalg.norm(rc)
        s = 0.5 * np.linalg.norm([R[i, 2, 1] - R[i, 1, 2], R[i, 0, 2] - R[i, 2, 0], R[i, 1, 0] - R[i, 0, 1]])
        if s >= 1e-5:
            d, tol = np.abs(r_out[i] - rc).max(), 16 * EPS * (1 + math.pi / s)
        elif th > 1:
            d = min(np.abs(r_out[i] - rc).max(), np.abs(r_out[i] + rc).max())
            tol = 4 * math.pi * math.sqrt(2 * EPS)
        else:
            d, tol = np.abs(r_out[i]).max(), th + 1e-15
        assert d <= tol, (i, R[i], r_out[i], rc, d, tol)

        cos_yaw = math.hypot(R[i, 2, 1], R[i, 2, 2])
        if cos_yaw >= 1e-3 and not axis_pi[i]:
            want = cv2.RQDecomp3x3(R[i])[0]
            tol = DEG * (8 * math.sqrt(EPS) + math.sqrt(2 * EPS) / cos_yaw + 64 * EPS / cos_yaw ** 2)
            d = _angle_diff(euler[i], want).max()
            if abs(R[i, 2, 1]) <= 1e-12 * abs(R[i, 2, 2]):
                # pitch 0 or 180 to rounding: (p, y, r) and (p + 180, 180 - y, r + 180) are the same rotation
                d = min(d, _angle_diff(euler[i], [want[0] + 180, 180 - want[1], want[2] + 180]).max())
            assert d <= tol, (i, R[i], euler[i], want)
        tol = 3 * math.sqrt(8 * EPS) + math.sqrt(2 * EPS) / max(cos_yaw, 1e-3)
        assert np.abs(_compose(euler[i]) - R[i]).max() <= tol, (i, R[i], euler[i])


# ------------------------------------------------------------------------------------------------------------------
# the solver over the pose space


def solve(points10, hw):
    """The kernel on (n, 10, 2) image points -> dict of rvec, tvec, euler, reproject."""
    from peppa_pig_face_landmark_b200.core.headpose.pose import head_poses
    return head_poses(np.asarray(points10, np.float32), hw, points=list(range(10)))


def _pose_space_faces(hw, seed):
    """-> list of (image points, R, t, noise, size): yaw +-80, pitch +-50, any roll, faces from 15 px up to 1500 px (or
    three quarters of the frame width) at 0, 0.8 and 3 px of noise, and noise-free faces at theta = pi - 10^-k."""
    import cv2
    rng = np.random.default_rng(seed)
    hi = min(1500.0, 0.75 * hw[1])
    faces = []
    for noise in (0.0, 0.8, 3.0):
        for _ in range(160):
            size = math.exp(rng.uniform(math.log(15), math.log(hi)))
            faces.append(synthetic_face(rng, hw, size, noise) + (noise, size))
    for k in range(1, 14):
        for axis in (np.array([1.0, 0, 0]), np.array([1.0, 0.05, -0.03]) / math.sqrt(1 + 0.05 ** 2 + 0.03 ** 2)):
            R = cv2.Rodrigues(axis * (math.pi - 10.0 ** -k))[0]
            size = math.exp(rng.uniform(math.log(30), math.log(hi)))
            faces.append(synthetic_face(rng, hw, size, 0.0, R=R) + (0.0, size))
    return faces


def _band(size):
    return "<50px" if size < 50 else "<200px" if size < 200 else "<600px" if size < 600 else ">=600px"


def check_pose_space(hw, seed):
    """Every check of test_solver_over_the_pose_space on one frame size -> per-regime report
    {(noise, band): [faces, cv2 unconverged, matched cv2, of those matched only by a widened bound, worst stationarity]}."""
    import cv2
    faces = _pose_space_faces(hw, seed)
    got = solve(np.stack([f[0] for f in faces]), hw)
    report, failed, crawling = {}, [], 0
    for i, (img, R_true, t_true, noise, size) in enumerate(faces):
        rvec, tvec = got["rvec"][i], got["tvec"][i]
        what = (hw, i, noise, size)
        assert np.linalg.norm(rvec) <= math.pi * (1 + 4 * EPS), what           # documented range of rvec
        ratio, bound = stationarity(img, rvec, tvec, hw)
        r_cv, t_cv = cv2_solve(img, hw)
        cv2_converged = is_stationary(img, r_cv, t_cv, hw)
        if ratio > bound:
            # where cv2 itself has not converged the face lies in a long flat valley, along which Levenberg-Marquardt
            # crawls (a few small noisy faces per hundred); there the kernel must be no worse than cv2, and is counted
            crawling += 1
            if cv2_converged:
                failed.append(("not stationary", what, ratio))
        if cost(img, rvec, tvec, hw) > not_worse_bound(img, r_cv, t_cv, hw):
            failed.append(("worse than cv2", what, cost(img, rvec, tvec, hw), cost(img, r_cv, t_cv, hw)))
        # the cube corners are projected with the reported rvec (finding: a matrix round trip near pi moved rvec by 2e-5)
        cube, _ = cv2.projectPoints(_cube(), rvec.reshape(3, 1), tvec.reshape(3, 1), _camera(hw), None)
        cube = cube.reshape(8, 2)
        assert np.abs(got["reproject"][i] - cube).max() <= 1e-9 * max(1.0, np.abs(cube).max()), what
        if cv2_converged:
            # each answer lies within its Gauss-Newton step of the minimum; on a flat minimum (the smallest faces) a
            # gradient within the stationarity bound still leaves that step above the tolerances, so it widens them
            steps = [_gauss_newton_step(img, r, t, hw) for r, t in ((rvec, tvec), (r_cv, t_cv))]
            gr = sum(np.linalg.norm(d[:3]) for d in steps)
            gt = sum(np.linalg.norm(d[3:]) for d in steps)
            gc = sum(np.abs(_cube_jacobian(r, t, hw) @ d).max() for d, (r, t) in zip(steps, ((rvec, tvec), (r_cv, t_cv))))
            assert _angle_diff(got["euler"][i], cv2_euler(r_cv, t_cv)).max() < max(1e-3, 4 * DEG * gr), (what, gr)
            want_cube = cv2.projectPoints(_cube(), r_cv.reshape(3, 1), t_cv.reshape(3, 1), _camera(hw), None)[0]
            assert np.abs(got["reproject"][i] - want_cube.reshape(8, 2)).max() < max(1e-2, 4 * gc), (what, gc)
            assert np.abs(cv2.Rodrigues(rvec)[0] - cv2.Rodrigues(r_cv)[0]).max() < max(1e-5, 4 * gr), (what, gr)
            t_tol = 1e-2 * max(1.0, np.linalg.norm(t_cv) / 100)
            assert np.abs(tvec - t_cv).max() < max(t_tol, 4 * gt), (what, gt)
            widened = 4 * DEG * gr > 1e-3 or 4 * gc > 1e-2 or 4 * gr > 1e-5 or 4 * gt > t_tol
        if noise == 0:
            # the generating pose, up to what the float32 rounding of the image points (2^-24 relative) can move:
            # |dp| <= |J^+| |d img|, four times over
            e, J, uv = residuals(img, cv2.Rodrigues(R_true)[0], t_true, hw)
            dimg = math.sqrt(20) * np.abs(uv).max() * 2.0 ** -24
            dp = 4 * dimg / np.linalg.svd(J, compute_uv=False)[-1] + 1e-9
            assert np.abs(cv2.Rodrigues(rvec)[0] - R_true).max() <= dp, (what, dp)
            assert np.abs(tvec - t_true).max() <= dp * max(1.0, np.linalg.norm(t_true)), (what, dp)
        row = report.setdefault((noise, _band(size)), [0, 0, 0, 0, 0.0])
        row[0] += 1
        row[1] += not cv2_converged
        row[2] += cv2_converged
        row[3] += cv2_converged and widened
        row[4] = max(row[4], ratio)
    assert not failed, (len(failed), failed[:10])
    assert crawling <= 0.02 * len(faces), crawling
    return report


def _gauss_newton_step(img, rvec, tvec, hw):
    e, J, _ = residuals(img, rvec, tvec, hw)
    return np.linalg.lstsq(J, -e, rcond=None)[0]


def _cube_jacobian(rvec, tvec, hw):
    import cv2
    return cv2.projectPoints(_cube(), np.asarray(rvec, np.float64).reshape(3, 1), np.asarray(tvec, np.float64).reshape(3, 1),
                             _camera(hw), None)[1][:, :6]


def _cube():
    from peppa_pig_face_landmark_b200.core.headpose.pose import reprojectsrc
    return reprojectsrc.astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("hw", FRAMES)
def test_solver_over_the_pose_space(hw):
    """The kernel's pose of every face is a stationary point of the reprojection error, no worse than cv2.solvePnP's,
    equal to cv2's wherever cv2 is converged (test_headpose_gpu's tolerances, tvec relative to |t| beyond 100), the
    generating pose on noise-free faces, and its cube corners are cv2.projectPoints of its own (rvec, tvec)."""
    report = check_pose_space(hw, seed=hw[1])
    for (noise, band), (n, unconv, matched, widened, worst) in sorted(report.items()):
        print("%dx%d noise %.1f %-7s faces %3d  cv2 unconverged %3d  matched cv2 %3d (by a widened bound %2d)  "
              "worst stationarity %.1e" % (hw[1], hw[0], noise, band, n, unconv, matched, widened, worst))


# ------------------------------------------------------------------------------------------------------------------
# degenerate faces in a launch with ordinary ones


@pytest.mark.gpu
def test_degenerate_faces_do_not_disturb_their_neighbours():
    """All ten points equal, ten collinear points, a face five times the frame and NaN points, interleaved with ordinary
    faces in one launch: the ordinary faces' results are bit-identical to solving them alone, and the degenerate ones
    come back (whatever they hold) without an error."""
    hw = (1080, 1920)
    rng = np.random.default_rng(5)
    ordinary = np.stack([synthetic_face(rng, hw, rng.uniform(30, 600), 0.8)[0] for _ in range(16)])
    line = np.stack([np.linspace(100, 900, 10), np.linspace(200, 700, 10)], 1)
    degenerate = [np.full((10, 2), 500.0), line, synthetic_face(rng, hw, 5 * hw[1], 0.0)[0],
                  np.full((10, 2), np.nan), np.where(np.arange(20).reshape(10, 2) == 7, np.nan, ordinary[0])]
    batch, where = [], []
    for i, face in enumerate(ordinary):
        batch.append(face)
        where.append(len(batch) - 1)
        if i % 3 == 0 and degenerate:
            batch.append(degenerate.pop())
    batch += degenerate
    got = solve(np.stack(batch), hw)
    alone = solve(ordinary, hw)
    for k in ("rvec", "tvec", "euler", "reproject"):
        assert got[k].shape[0] == len(batch)
        assert np.array_equal(got[k][where], alone[k]), k
