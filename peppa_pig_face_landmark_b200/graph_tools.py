"""Re-targets the shipped exports to other input sizes.

Landmark net, to another square input size (`retarget_input_size`):
`tools/convert_to_onnx.py --img_size S` (the reference's TRAIN/face_landmark/tools/convert_to_onnx.py:15-60)
traces the same network at S x S: every convolution is size-agnostic, and the only constants the tracer bakes
in are (a) the ASPP pooling branch's `F.interpolate(x, size=size)` target (model.py:58-61) = S/16 and (b) the
heat-map side S/4 used by postp (model.py:511-554: `idx % W`, `idx // W`, `/ W`, `/ H`).  Patching those
reproduces the graph the exporter would have written for the README's @128 variants from the shipped @256
file (the weights are whatever the source file holds).

Detector (`retarget_detector_input`): yolov5n-0.5-face is fully convolutional; the yolov5-face exporter bakes the
feature-map sizes of its three strides (8, 16, 32) into the ShuffleNetV2 channel-shuffle reshapes, the Detect
tail's `[1,3,16,H,W]` reshapes and the tail's grid / anchor-grid constants.  Rewriting those gives the graph the
exporter writes at another (h, w).
"""
import os

import numpy as np

from .onnx_loader import OnnxNode, load_onnx
from .onnx_writer import save_onnx


def retarget_input_size(src_onnx, dst_onnx, size):
    g = load_onnx(src_onnx)
    shp = g.input_shapes[g.inputs[0]]
    old = int(shp[2])
    if shp[2] != shp[3] or size % 32 or size <= 0:
        raise ValueError("retarget_input_size: square inputs, multiples of 32 (got %s -> %d)" % (shp, size))
    old_hm, new_hm, old_p, new_p = old // 4, size // 4, old // 16, size // 16
    users = {}
    for n in g.nodes:
        for i in n.inputs:
            users.setdefault(i, []).append(n)
    has_argmax = any(n.op == "ArgMax" for n in g.nodes)
    nodes, patched = [], 0
    for n in g.nodes:
        attrs = dict(n.attrs)
        if n.op == "Constant":
            v = np.asarray(attrs["value"])
            us = users.get(n.outputs[0], [])
            if has_argmax and v.size == 1 and float(v.reshape(-1)[0]) == old_hm and us and \
                    all(u.op in ("Mod", "Div") and u.inputs[1] == n.outputs[0] for u in us):
                attrs["value"] = np.full(v.shape, new_hm, v.dtype)               # postp: % W, // W, / W, / H
                patched += 1
            elif v.dtype == np.int64 and v.shape == (2,) and list(v) == [old_p, old_p] and "fm_pool" in n.name:
                attrs["value"] = np.array([new_p, new_p], np.int64)                # ASPP pooling branch target size
                patched += 1
        nodes.append(OnnxNode(n.op, n.name, list(n.inputs), list(n.outputs), attrs))
    if patched != 5:
        raise ValueError("retarget_input_size: expected 5 size constants in a Skps landmark export, found %d" % patched)
    save_onnx(dst_onnx, nodes, g.weights, [(g.inputs[0], [1, 3, size, size])],
              [(o, [1, 196] if o == "output" else [1, 98]) for o in g.outputs])
    return dst_onnx


# Detector input sizes accepted by retarget_detector_input / FaceAna(det_input=...): multiples of 32 (the coarsest
# stride), from 128 up to a 2160 x 3840 frame (FaceAna's default max_frame_hw) rounded up to the next multiple of 32.
DET_INPUT_MIN = (128, 128)
DET_INPUT_MAX = (2176, 3840)
_DET_STRIDES = (8, 16, 32)
# the size-carrying constants of the shipped yolov5n-0.5-face export, by kind
_DET_SIZE_CONSTANTS = dict(shuffle=32, head_reshape=3, zeros=3, grid=3, anchor_grid=18, grid_stride=15)
_HERE = os.path.dirname(os.path.abspath(__file__))


def check_detector_input(hw):
    """(h, w) -> (int h, int w), or ValueError when the detector cannot run at that input size."""
    try:
        h, w = (int(v) for v in hw)
    except (TypeError, ValueError):
        raise ValueError("detector input size must be a pair (h, w), got %r" % (hw,))
    if h % 32 or w % 32:
        raise ValueError("detector input %dx%d: h and w must be multiples of 32" % (h, w))
    if not (DET_INPUT_MIN[0] <= h <= DET_INPUT_MAX[0] and DET_INPUT_MIN[1] <= w <= DET_INPUT_MAX[1]):
        raise ValueError("detector input %dx%d outside %d..%d x %d..%d" % (h, w, DET_INPUT_MIN[0], DET_INPUT_MAX[0],
                                                                          DET_INPUT_MIN[1], DET_INPUT_MAX[1]))
    return h, w


def detector_rows(hw):
    """Rows of the detector output at input size hw: 3 anchors per cell of the stride-8, 16 and 32 maps."""
    h, w = hw
    return sum(3 * (h // s) * (w // s) for s in _DET_STRIDES)


def _grid(h, w):
    gx, gy = np.meshgrid(np.arange(w), np.arange(h))
    return np.broadcast_to(np.stack((gx, gy), -1)[None, None], (1, 3, h, w, 2)).astype(np.float32)


def retarget_detector_input(src_onnx, dst_onnx, hw):
    """Write the shipped yolov5n-0.5-face export `src_onnx` at input size hw = (h, w) to `dst_onnx`.

    Rewritten constants, per stride s in (8, 16, 32) with map size (h/s, w/s):
      - the channel-shuffle reshape targets [1,2,C,H,W] and [1,-1,H,W] of the ShuffleNetV2 units;
      - the Detect tail's [1,3,16,H,W] reshapes, one per head;
      - the tail's (1,3,H,W,16) zero tensor (the exporter's `torch.full_like(x, 0)`);
      - the (1,3,H,W,2) grid (meshgrid of x, y), grid * stride (landmark offsets) and anchor grid (each head's three
        (w, h) anchors broadcast over the map).
    The tail flattens each head with [1,-1,16], so no row count is baked in; the declared output becomes
    (1, detector_rows(hw), 16).  Weights and every other node are copied unchanged, so hw equal to the source's own
    size gives back the source graph.  ValueError for a size check_detector_input refuses, or for a graph whose
    size-carrying constants are not those of the shipped export."""
    h, w = check_detector_input(hw)
    g = load_onnx(src_onnx)
    shp = g.input_shapes[g.inputs[0]]
    if len(shp) != 4 or shp[:2] != [1, 3] or shp[2] % 32 or shp[3] % 32 or len(g.outputs) != 1:
        raise ValueError("retarget_detector_input: %s is not a yolov5-face detector export (input %s)" % (src_onnx, shp))
    old = {(shp[2] // s, shp[3] // s): s for s in _DET_STRIDES}
    users = {}
    for n in g.nodes:
        for i in n.inputs:
            users.setdefault(i, []).append(n)
    count = dict.fromkeys(_DET_SIZE_CONSTANTS, 0)
    nodes = []
    for n in g.nodes:
        attrs = dict(n.attrs)
        if n.op == "Constant":
            v = np.asarray(attrs["value"])
            us = users.get(n.outputs[0], [])
            kind = None
            if v.dtype == np.int64 and v.ndim == 1 and v.size in (4, 5) and tuple(v[-2:]) in old and us and \
                    all(u.op == "Reshape" and u.inputs[1] == n.outputs[0] for u in us):
                s = old[tuple(v[-2:])]
                if v.size == 5 and list(v[:3]) == [1, 3, 16]:
                    kind = "head_reshape"
                elif (v.size == 5 and list(v[:2]) == [1, 2]) or (v.size == 4 and list(v[:2]) == [1, -1]):
                    kind = "shuffle"
                if kind:
                    nv = v.copy()
                    nv[-2:] = (h // s, w // s)
            elif v.dtype == np.float32 and v.ndim == 5 and v.shape[:2] == (1, 3) and v.shape[2:4] in old:
                s = old[v.shape[2:4]]
                H, W = v.shape[2:4]
                nh, nw = h // s, w // s
                if v.shape[4] == 16 and not v.any():
                    kind, nv = "zeros", np.zeros((1, 3, nh, nw, 16), np.float32)
                elif v.shape[4] == 2 and np.ptp(v, axis=(2, 3)).max() == 0 and H * W > 1:
                    kind = "anchor_grid"
                    nv = np.ascontiguousarray(np.broadcast_to(v[:, :, :1, :1, :], (1, 3, nh, nw, 2)))
                elif v.shape[4] == 2 and np.array_equal(v, _grid(H, W)):
                    kind, nv = "grid", _grid(nh, nw)
                elif v.shape[4] == 2 and np.array_equal(v, _grid(H, W) * np.float32(s)):
                    kind, nv = "grid_stride", _grid(nh, nw) * np.float32(s)
            if kind is None and v.ndim >= 1 and v.size > 1 and any(
                    v.shape[i:i + 2] in old for i in range(v.ndim - 1)):
                raise ValueError("retarget_detector_input: constant %s %s carries a map size but is not one the "
                                 "yolov5-face exporter writes" % (n.name, v.shape))
            if kind:
                attrs["value"] = nv.astype(v.dtype)
                count[kind] += 1
        nodes.append(OnnxNode(n.op, n.name, list(n.inputs), list(n.outputs), attrs))
    if count != _DET_SIZE_CONSTANTS:
        raise ValueError("retarget_detector_input: %s has size constants %s, the yolov5n-0.5-face export has %s"
                         % (src_onnx, count, _DET_SIZE_CONSTANTS))
    save_onnx(dst_onnx, nodes, g.weights, [(g.inputs[0], [1, 3, h, w])], [(g.outputs[0], [1, detector_rows((h, w)), 16])])
    return dst_onnx


def ensure_detector_onnx(src_onnx, hw):
    """Path of `src_onnx` retargeted to hw, written once under pretrained/_generated/ (git-ignored) and reused.
    The file is written to a temporary name and moved into place, so concurrent callers never read half a file."""
    h, w = check_detector_input(hw)
    d = os.path.join(_HERE, "pretrained", "_generated")
    os.makedirs(d, exist_ok=True)
    p = os.path.join(d, "%s_%dx%d.onnx" % (os.path.splitext(os.path.basename(src_onnx))[0], h, w))
    if not os.path.exists(p):
        tmp = p + ".tmp%d" % os.getpid()
        retarget_detector_input(src_onnx, tmp, (h, w))
        os.replace(tmp, p)
    return p


def detector_onnx_for(src_onnx, hw):
    """The detector file to build an engine from for input size hw: `src_onnx` itself when hw is its own input size,
    else its retargeted copy (ensure_detector_onnx)."""
    g = load_onnx(src_onnx)
    shp = g.input_shapes[g.inputs[0]]
    if (int(shp[2]), int(shp[3])) == (int(hw[0]), int(hw[1])):
        return src_onnx
    return ensure_detector_onnx(src_onnx, hw)
