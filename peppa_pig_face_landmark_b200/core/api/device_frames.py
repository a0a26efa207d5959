"""The frames FaceAna.run and FaceAnaStreams.submit accept, checked before anything is enqueued: numpy arrays, and frames
already in GPU memory (a decoder surface, a tensor from NVDEC / DALI / torchvision, an ROI view of either).  Host frames
are HxWx3 uint8 BGR as the reference's run(image) takes them.  CUDA frames are read where they are, at any row pitch, in
the pixel layout the caller names with layout= (LAYOUTS): interleaved BGR (the default), RGB, BGRA or RGBA, or planar
(3, H, W) BGR or RGB.  Every layout gives, bit for bit, the results of the same pixels passed as interleaved BGR.
CUDA frames stored sideways or upside down (a portrait clip from NVDEC, a photo whose EXIF orientation nvJPEG did not
apply, a ceiling camera) are read in place as the upright frame with rotate= (check_rotate)."""
import collections
import numbers
import sys

import numpy as np

# layout= name -> SKPS_LAYOUT_* code of include/skps_b200.h
LAYOUTS = {"bgr": 0, "rgb": 1, "bgra": 2, "rgba": 3, "bgr_planar": 4, "rgb_planar": 5}
PLANAR = ("bgr_planar", "rgb_planar")
# skps_frame_layout of include/skps_b200.h: a frame's layout code and plane pitch, beside its skps_det_src / skps_face_src
FRAME_LAYOUT = np.dtype([("layout", "<i4"), ("plane_pitch", "<i4")])

FrameLayout = collections.namedtuple("FrameLayout", "H W pitch plane code")
FrameLayout.__doc__ = """Where a CUDA frame's pixels are: its height and width, the bytes from one row to the next (pitch)
and from one plane to the next (plane, 0 for interleaved layouts), and its SKPS_LAYOUT_* code."""


def check_layout(layout, cuda=True):
    """The SKPS_LAYOUT_* code of layout=, one of LAYOUTS.  ValueError for anything else, and for a layout other than "bgr"
    with host frames (cuda False), which are HxWx3 BGR."""
    if not isinstance(layout, str) or layout not in LAYOUTS:
        raise ValueError("layout: expected one of %s, got %r" % (", ".join(repr(k) for k in LAYOUTS), layout))
    if not cuda and layout != "bgr":
        raise ValueError("layout=%r takes CUDA frames; host frames are HxWx3 uint8 BGR (layout='bgr')" % layout)
    return LAYOUTS[layout]


def frame_layout(shape, strides, layout):
    """FrameLayout of a uint8 frame with this shape and these strides (in bytes) in layout `layout`:
      "bgr", "rgb"            (H, W, 3), strides (>= 3W, 3, 1)
      "bgra", "rgba"          (H, W, 4), strides (>= 4W, 4, 1); the 4th channel's values are never used
      "bgr_planar", "rgb_planar"  (3, H, W), strides (any, >= W, 1): planes at any distance
    A stride that never moves (the row stride of a one-row frame, the column stride of a one-column one) may be anything.
    Row and plane pitches must fit 32 bits.  ValueError for anything else: the layout is what the caller says, never
    guessed from the shape (a (3, W, 3) tensor fits two of them)."""
    code = check_layout(layout)
    shape, strides = tuple(int(v) for v in shape), tuple(int(v) for v in strides)
    if len(shape) != 3 or len(strides) != 3:
        raise ValueError("layout=%r: expected a 3-d frame, got shape %s" % (layout, shape))
    if layout in PLANAR:
        (C, H, W), (plane, sy, sx) = shape, strides
        if C != 3:
            raise ValueError("layout=%r: expected a (3, H, W) frame, got shape %s" % (layout, shape))
        if H < 1 or W < 1:
            raise ValueError("empty frame %s" % (shape,))
        if (W > 1 and sx != 1) or (H > 1 and sy < W) or plane < 0:
            raise ValueError("layout=%r: expected planes of rows, strides (any, >= W, 1); got strides %s for shape %s "
                             "(an HxWxC tensor takes an interleaved layout such as layout='rgb')" % (layout, strides, shape))
        pitch = sy if H > 1 else W
    else:
        C = 4 if layout in ("bgra", "rgba") else 3
        (H, W, c), (sy, sx, sc) = shape, strides
        if c != C:
            raise ValueError("layout=%r: expected an (H, W, %d) frame, got shape %s%s"
                             % (layout, C, shape, " (a planar tensor takes layout='rgb_planar' or 'bgr_planar')"
                                if shape[0] == 3 else ""))
        if H < 1 or W < 1:
            raise ValueError("empty frame %s" % (shape,))
        if sc != 1 or (W > 1 and sx != C) or (H > 1 and sy < C * W):
            raise ValueError("layout=%r: expected interleaved pixels, strides (>= %dW, %d, 1); got strides %s for shape %s "
                             "(name the frame's layout with layout=, e.g. 'rgb_planar' for a (3, H, W) tensor)"
                             % (layout, C, C, strides, shape))
        pitch, plane = (sy if H > 1 else C * W), 0
    if pitch >= 2 ** 31:
        raise ValueError("row pitch %d does not fit 32 bits" % pitch)
    if plane >= 2 ** 31:
        raise ValueError("plane pitch %d does not fit 32 bits" % plane)
    return FrameLayout(H, W, pitch, plane, code)


ROTATIONS = (0, 90, 180, 270)


def _turns(rotate):
    if isinstance(rotate, (bool, np.bool_)) or not isinstance(rotate, numbers.Integral) or int(rotate) not in ROTATIONS:
        raise ValueError("rotate: expected one of %s (degrees clockwise), got %r" % (", ".join(map(str, ROTATIONS)), rotate))
    return int(rotate) // 90


def check_rotate(rotate, n=None, cuda=True):
    """Quarter turns clockwise (0..3) of rotate=: the clockwise angle in degrees, one of ROTATIONS, by which a stored
    frame must be turned to be upright.  The frame is analysed as cv2.rotate(frame, code), 90 being ROTATE_90_CLOCKWISE,
    180 ROTATE_180 and 270 ROTATE_90_COUNTERCLOCKWISE; for an (H, W, C) tensor that is
    torch.rot90(frame, -rotate // 90, dims=(0, 1)), for a planar one the same with dims=(1, 2).
    n None: rotate is one int, and so is the result.  n an int: rotate is one int for all n frames or a sequence of n,
    and the result a list of n turns.  ValueError for a value outside ROTATIONS, a bool or a non-int, a sequence of
    another length, and any turn with host frames (cuda False): cv2.imread and VideoCapture give them upright already,
    and the caller can cv2.rotate them."""
    if n is None or isinstance(rotate, (numbers.Number, np.bool_, str, bytes)) or not hasattr(rotate, "__len__"):
        t = _turns(rotate)
        turns = t if n is None else [t] * n
    else:
        if len(rotate) != n:
            raise ValueError("rotate: expected one value or one per frame (%d), got %d values" % (n, len(rotate)))
        turns = [_turns(r) for r in rotate]
    if not cuda and any(turns if n is not None else [turns]):
        raise ValueError("rotate=%r takes CUDA frames; host frames are upright as cv2 decodes them (cv2.rotate them)"
                         % (rotate,))
    return turns


def upright_hw(H, W, turns):
    """(H, W) of the upright frame of an H x W frame stored `turns` quarter turns from upright."""
    return (W, H) if turns & 1 else (H, W)


def upright_shape(shape, strides, layout="bgr", rotate=0):
    """(H, W) of the upright frame a call analyses for a uint8 frame with this shape and these strides (in bytes) in
    layout `layout` (frame_layout) stored turned by rotate= degrees (check_rotate).  ValueError as those two raise it."""
    fl = frame_layout(shape, strides, layout)
    return upright_hw(fl.H, fl.W, check_rotate(rotate))


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


def check_cuda_frame(frame, device, max_hw, layout="bgr"):
    """FrameLayout of `frame`, a torch.uint8 CUDA tensor on `device` in layout `layout` (frame_layout): with the default
    "bgr", (H, W, 3) with stride(2) == 1, stride(1) == 3 and stride(0) >= 3 W, so packed tensors, pitched surfaces and
    big[y0:y1, x0:x1] views all qualify.  ValueError for anything else, or for more pixels than max_hw = (max_h, max_w)
    allows."""
    if not is_tensor(frame):
        raise ValueError("expected a CUDA tensor, got %s" % type(frame).__name__)
    if not frame.is_cuda:
        raise ValueError("expected a CUDA tensor, got a tensor on %s" % frame.device)
    if str(frame.dtype) != "torch.uint8" or frame.dim() != 3:
        raise ValueError("expected a uint8 frame in layout=%r, got %s %s" % (layout, frame.dtype, tuple(frame.shape)))
    if frame.device != device:
        raise ValueError("the frame is on %s, the pipeline on %s" % (frame.device, device))
    fl = frame_layout(frame.shape, frame.stride(), layout)
    if fl.H * fl.W > max_hw[0] * max_hw[1]:
        raise ValueError("frame %dx%d has more pixels than max_frame_hw %dx%d" % (fl.H, fl.W, max_hw[0], max_hw[1]))
    return fl
