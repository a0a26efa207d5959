"""Layer-by-layer parity report (GPU box): runs a network through the CUDA engine and through
the oracle executor on the same input and prints, per plan buffer, the max abs / rel error
against the ONNX tensor of the same name.  Usage: python tools/layer_report.py [student|detector [H W]]
(H W: the detector retargeted to that input size, graph_tools.retarget_detector_input)"""
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def report(which="student", batch=2, out=sys.stdout, det_input=None):
    import frames
    from oracle import host_ref as H
    from oracle.onnx_exec import Session
    from peppa_pig_face_landmark_b200.core.api.onnx_model_base import ONNXEngine
    pre = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained")
    if which == "student":
        path = os.path.join(pre, "kps_student.onnx")
        x_u8 = frames.crop_variants(batch)
    else:
        path = os.path.join(pre, "yolov5n-0.5.onnx")
        hw = (384, 640)
        if det_input is not None:
            from peppa_pig_face_landmark_b200.graph_tools import ensure_detector_onnx
            path, hw = ensure_detector_onnx(path, det_input), tuple(det_input)
        x, _ = H.letterbox(frames.load_test1() if det_input is None else frames.frame_4k(), *hw)
        x_u8 = np.round(x.transpose(0, 2, 3, 1) * 255).astype(np.uint8)
        batch = 1
    eng = ONNXEngine(path, max_batch=batch)
    outs = eng.run_u8(x_u8)
    sess = Session(path)
    worst = 0.0
    rows = []
    written = {}                                      # buffer -> logical channels some op writes (fusions leave tensors unmaterialised)
    read = {}
    from peppa_pig_face_landmark_b200 import plan as P
    for op in eng.plan.ops:
        stored = op.outs[1:] if (op.type == P.OP_CONV and op.flags & P.FLAG_HM_PART) else op.outs     # the heat map itself is not stored
        for v in stored:
            written[v.buf.idx] = max(written.get(v.buf.idx, 0), v.c_off + (v.C - 1) * v.c_stride + 1)
        for v in op.ins:
            if v is not None:
                read[v.buf.idx] = max(read.get(v.buf.idx, 0), v.c_off + (v.C - 1) * v.c_stride + 1)
    for k in written:                                 # a conv may also write the zero padding channels of its buffer
        if k in read:
            written[k] = min(written[k], read[k])
    for n in range(batch):
        xf = x_u8[n].transpose(2, 0, 1).astype(np.float32)[None] / np.float32(255.)
        ref_outs, kept = sess.run(xf, keep="all")
        for b in eng.plan.bufs:
            if b.name not in kept or b.idx == eng.plan.input.buf.idx or b.idx not in written:
                continue
            ref = kept[b.name].numpy()
            if ref.ndim != 4:
                continue
            got = eng.read_buffer(b.idx, batch)[n]
            ref = ref[0].transpose(1, 2, 0)
            nc = min(ref.shape[-1], written[b.idx])  # buffers may be channel-padded; the split heat-map head keeps only the score maps
            got, ref = got[..., :nc], ref[..., :nc]
            if got.shape != ref.shape:
                rows.append((b.idx, b.name, "SHAPE %s vs %s" % (got.shape, ref.shape)))
                continue
            err = float(np.abs(got - ref).max())
            scale = float(np.abs(ref).max()) + 1e-12
            rows.append((b.idx, b.name, "n=%d max_abs=%.3e ref_max=%.3e rel=%.3e" % (n, err, scale, err / scale)))
            worst = max(worst, err / scale)
        for i, (g, r) in enumerate(zip(outs, ref_outs)):
            e = float(np.abs(g[n].reshape(-1) - np.asarray(r).reshape(-1)).max())
            rows.append((-1, "output%d" % i, "n=%d max_abs=%.3e" % (n, e)))
    for r in rows:
        print("%4d %-70s %s" % r, file=out)
    print("worst relative error over buffers: %.3e" % worst, file=out)
    return worst


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "student"
    det_input = (int(sys.argv[2]), int(sys.argv[3])) if len(sys.argv) > 3 else None
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "layer_report_%s.txt" % which), "w") as f:
        report(which, out=f, det_input=det_input)
    print(open(os.path.join(ROOT, "gpurun_out", "layer_report_%s.txt" % which)).read()[-3000:])
