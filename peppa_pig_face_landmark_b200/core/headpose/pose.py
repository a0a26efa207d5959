"""Head pose from facial landmarks — same call as the reference's Skps/core/headpose/pose.py:48-77:

    reprojectdst, euler_angle = get_head_pose(shape, img)

`shape` is a 68-point landmark array (the function reads points 17,21,22,26,36,39,42,45,31,35), `img` the frame (only
its size is used: camera matrix [[w,0,w//2],[0,w,h//2],[0,0,1]], no distortion).  The reference calls cv2.solvePnP,
cv2.projectPoints, cv2.Rodrigues and cv2.decomposeProjectionMatrix per face; here the whole batch is solved by one CUDA
kernel (csrc/headpose.cu: DLT start + Levenberg-Marquardt in float64, OpenCV's RQ-based Euler angles).  Additive:
`head_poses(shapes, (h, w))` for many faces at once, returning rotation/translation vectors too, and
`head_poses(shapes98, (h, w), points=POSE_POINTS_98)` for the 98-point landmarks the shipped model returns."""
import numpy as np

from ... import runtime as rt

# pose.py:22-31 and :32-39 (the 3-D model points and the cube that is re-projected for drawing)
object_pts = np.float32([[6.825897, 6.760612, 4.402142],
                         [1.330353, 7.122144, 6.903745],
                         [-1.330353, 7.122144, 6.903745],
                         [-6.825897, 6.760612, 4.402142],
                         [5.311432, 5.485328, 3.987654],
                         [1.789930, 5.393625, 4.413414],
                         [-1.789930, 5.393625, 4.413414],
                         [-5.311432, 5.485328, 3.987654],
                         [2.005628, 1.409845, 6.165652],
                         [-2.005628, 1.409845, 6.165652]])
reprojectsrc = np.float32([[10.0, 10.0, 10.0],
                           [10.0, 10.0, -10.0],
                           [10.0, -10.0, -10.0],
                           [10.0, -10.0, 10.0],
                           [-10.0, 10.0, 10.0],
                           [-10.0, 10.0, -10.0],
                           [-10.0, -10.0, -10.0],
                           [-10.0, -10.0, 10.0]])
line_pairs = [[0, 1], [1, 2], [2, 3], [3, 0],
              [4, 5], [5, 6], [6, 7], [7, 4],
              [0, 4], [1, 5], [2, 6], [3, 7]]
POSE_POINTS = [17, 21, 22, 26, 36, 39, 42, 45, 31, 35]
# The same ten points in the 98-point WFLW convention of the shipped landmark model: the reference's training tree solves
# the head pose on these (TRAIN/face_landmark/lib/dataset/headpose.py:64-65), and its Euler angles are the pose targets the
# network was trained with.  FaceAna(pose=True) and FaceAnaStreams(pose=True) use them.
POSE_POINTS_98 = [33, 37, 42, 46, 60, 64, 68, 72, 55, 59]


def head_poses(shapes, img_hw, points=POSE_POINTS):
    """shapes: (N, P, 2) landmark sets; `points` are the 10 landmarks paired with object_pts (POSE_POINTS for 68-point
    shapes, POSE_POINTS_98 for 98-point ones) -> dict of float64 arrays
    rvec (N,3), tvec (N,3), euler (N,3) in degrees [pitch, yaw, roll as cv2 orders them], reproject (N,8,2)."""
    rt.require_cuda()
    lib = rt.load_library()
    shapes = np.asarray(shapes)
    points = [int(i) for i in points]
    if len(points) != len(object_pts) or min(points) < 0:
        raise ValueError("expected %d non-negative landmark indices, got %s" % (len(object_pts), points))
    if shapes.ndim != 3 or shapes.shape[1] <= max(points) or shapes.shape[2] != 2:
        raise ValueError("expected (N, >%d, 2) landmark sets, got %s" % (max(points), shapes.shape))
    pts = np.ascontiguousarray(shapes[:, points, :], dtype=np.float32)
    n = pts.shape[0]
    h, w = int(img_hw[0]), int(img_hw[1])
    out = {"rvec": np.zeros((n, 3)), "tvec": np.zeros((n, 3)), "euler": np.zeros((n, 3)), "reproject": np.zeros((n, 8, 2))}
    if n:
        rt.check(lib.skps_head_pose(pts.ctypes.data, n, w, h, object_pts.ctypes.data, reprojectsrc.ctypes.data,
                                    out["rvec"].ctypes.data, out["tvec"].ctypes.data, out["euler"].ctypes.data,
                                    out["reproject"].ctypes.data))
    return out


def get_head_pose(shape, img):
    """pose.py:48-77: -> (tuple of 8 (x, y) tuples, (3,1) Euler angles in degrees)."""
    h, w, _ = img.shape
    r = head_poses(np.asarray(shape)[None], (h, w))
    reprojectdst = tuple(map(tuple, r["reproject"][0].astype(np.float32)))
    return reprojectdst, r["euler"][0].reshape(3, 1)
