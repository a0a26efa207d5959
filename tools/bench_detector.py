"""Detector (yolov5n-0.5-face @384x640) forward time on one GPU: python tools/bench_detector.py [--det-input H W] [batch ...]
Device-resident letterboxed uint8 canvases -> (N,rows,16) rows (15120 at 384x640); CUDA events on the engine's stream.
--det-input H W times the detector retargeted to that input size (graph_tools.retarget_detector_input).
Prints one JSON line per batch with the share of conv MACs routed to the tensor-core kernels and the roofline fractions
(tensor: 2*MAC / time against the measured bf16 peak; HBM: the plan's per-op tensor bytes / time against the measured copy rate)."""
import json
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


def run(B, n=50, peaks=None, hw=(384, 640)):
    import torch
    from peppa_pig_face_landmark_b200 import ONNXEngine, plan as P
    from peppa_pig_face_landmark_b200.graph_tools import detector_onnx_for
    path = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "yolov5n-0.5.onnx")
    eng = ONNXEngine(detector_onnx_for(path, hw), max_batch=B)
    tc = tot = 0
    for op in eng.plan.ops:
        if op.type == P.OP_CONV:
            o = op.outs[0]
            m = o.C * o.H * o.W * op.ins[0].C * op.k[0] * op.k[1]
            tot += m
            tc += m if op.flags & P.FLAG_TC else 0
    x = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (B, hw[0], hw[1], 3), dtype=np.uint8)).cuda()
    outs = [torch.empty((B, e), dtype=torch.float32, device="cuda") for e in eng.out_elems]
    s = eng.stream
    with torch.cuda.stream(s):
        for _ in range(5):
            eng.forward_device(x, outs, s)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            eng.forward_device(x, outs, s)
        e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    bytes_per_frame = sum(eng.plan.bytes_per_sample(op) for op in eng.plan.ops)
    r = {"workload": "yolov5n-0.5-face %dx%d forward+decode" % tuple(hw), "batch": B, "ms": ms,
         "frames_per_s": B / ms * 1e3, "tc_mac_share": tc / tot, "launches": len(eng.plan.ops),
         "tflops_2mac": 2 * eng.plan.macs * B / ms / 1e9, "gbs_plan_bytes": bytes_per_frame * B / ms / 1e6,
         "plan_bytes_per_frame": bytes_per_frame, "mac_per_frame": int(eng.plan.macs)}
    if peaks:
        r["frac_tensor_peak"] = r["tflops_2mac"] / peaks[0]
        r["frac_hbm_peak"] = r["gbs_plan_bytes"] / peaks[1]
    del eng
    return r


if __name__ == "__main__":
    a = sys.argv[1:]
    hw = (384, 640)
    if "--det-input" in a:
        i = a.index("--det-input")
        hw = (int(a[i + 1]), int(a[i + 2]))
        del a[i:i + 3]
    for B in [int(v) for v in a] or [1, 16]:
        print(json.dumps(run(B, hw=hw)))
