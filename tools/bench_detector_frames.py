"""FaceDetector throughput on one GPU, four ways, alternated in one run:
  (a) engine   the detector engine alone at batch B on device-resident letterboxed canvases (tools/bench_detector.py's run);
  (b) cuda     FaceDetector.submit(cuda_frames, out=...) with two calls in flight;
  (c) host     FaceDetector.submit(host_frames) with two calls in flight, results back on the host;
  (d) call     a loop of single-frame FaceDetector(cfg)(frame).
Workloads: 16 frames of 1080p with 4 faces, of 4K with 16 faces (tests/frames.py) and of 4000x3000 stills, at the
384x640 and 1152x1920 detector inputs.  Prints one JSON line per workload and mode (median frames/s over the rounds, the
spread, and the bytes a host frame uploads), then the card's name and power limit read in the same run.

    python tools/bench_detector_frames.py [--rounds 5] [--iters 20] [--frames 16] [--det-input H W ...]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402


def workloads(n):
    import frames
    still = frames.multi_face_frame(3000, 4000, (2, 3), 560)
    return {"1080p_4faces": [frames.frame_1080p(jitter=(i % 5, -(i % 3))) for i in range(n)],
            "4k_16faces": [frames.frame_4k(jitter=(i % 5, -(i % 3))) for i in range(n)],
            "still_4000x3000": [np.roll(still, i, axis=1) for i in range(n)]}


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def upload_bytes(fs, hw):
    from peppa_pig_face_landmark_b200.core.api.face_detector import host_upload_rows, letterbox_geometry
    out = []
    for f in fs:
        H, W = f.shape[:2]
        rows = host_upload_rows(H, letterbox_geometry(H, W, *hw)[2])
        out.append((H if rows is None else len(rows)) * 3 * W)
    return int(np.mean(out)), int(np.mean([f.nbytes for f in fs]))


def in_flight(det, calls, iters, out=None):
    """iters calls of det.submit with two in flight; seconds from the first submit to the last result."""
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(iters):
        if len(det._pending) == 2:
            det.collect()
        det.submit(calls[i % len(calls)], out=None if out is None else out[i % 2])
    while det._pending:
        det.collect()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def single(det, fs, iters):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(iters):
        for f in fs:
            det(f)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20, help="calls of --frames frames per mode and round")
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--det-input", type=int, nargs="+", default=[384, 640, 1152, 1920])
    a = ap.parse_args()
    import logging
    import torch
    import bench_detector
    from peppa_pig_face_landmark_b200.core.api.face_detector import FaceDetector
    from peppa_pig_face_landmark_b200.core.api.facer import get_cfg
    from peppa_pig_face_landmark_b200.logger.logger import logger
    logger.setLevel(logging.WARNING)
    B = a.frames
    loads = workloads(B)
    hws = [(a.det_input[i], a.det_input[i + 1]) for i in range(0, len(a.det_input), 2)]
    for hw in hws:
        cfg = get_cfg()['Skps']['Detect']
        cfg['input_shape'] = [hw[0], hw[1], 3]
        det = FaceDetector(cfg, max_frames=B)
        call = FaceDetector(cfg, max_frames=1)
        bufs = [det.new_results(B), det.new_results(B)]
        for name, fs in loads.items():
            dev = [torch.from_numpy(f).cuda() for f in fs]
            host_calls, dev_calls = [fs], [dev]
            rates = {m: [] for m in ("engine", "cuda", "host", "call")}
            # warm every mode and shape once
            bench_detector.run(B, n=3, hw=hw)
            in_flight(det, dev_calls, 2, bufs)
            in_flight(det, host_calls, 2)
            single(call, fs[:2], 1)
            n_call = max(1, a.iters // 4)
            for _ in range(a.rounds):
                rates["engine"].append(bench_detector.run(B, n=a.iters, hw=hw)["frames_per_s"])
                rates["cuda"].append(a.iters * B / in_flight(det, dev_calls, a.iters, bufs))
                rates["host"].append(a.iters * B / in_flight(det, host_calls, a.iters))
                rates["call"].append(n_call * B / single(call, fs, n_call))
            up, whole = upload_bytes(fs, hw)
            for m, r in rates.items():
                print(json.dumps({"workload": name, "det_input": "%dx%d" % hw, "mode": m, "frames": B,
                                  "frames_per_s": float(np.median(r)), "min": float(min(r)), "max": float(max(r)),
                                  "host_upload_bytes_per_frame": up if m in ("host", "call") else 0,
                                  "host_frame_bytes": whole}), flush=True)
            del dev
        del det, call, bufs
        torch.cuda.empty_cache()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
