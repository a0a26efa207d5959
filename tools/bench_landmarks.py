"""Throughput of FaceLandmark's batched path against the landmark net alone, in one process:

  (a) engine   faces/s of the net on crops already in HBM at max_faces per forward (what bench.py reports)
  (b) device   FaceLandmark.submit / collect on CUDA 1080p frames (4 faces each), CUDA boxes, results left in out=
  (c) host     FaceLandmark.submit / collect on host 1024x1024 frames with one face each, through the rectangle upload;
               with the bytes uploaded per face beside the whole frame's

  With --align SIZE, (b) and (c) also run on FaceLandmark(align=SIZE), alternated with the runs without it, and the
  host upload per face counts the chip's rectangle (chip_read_rects) as well.

    python tools/bench_landmarks.py [--max-faces 256] [--calls 40] [--warmup 5] [--align SIZE]
Prints one JSON line; the card's name and power limit are part of it."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def timed(step, n, warmup):
    """Seconds per step over n steps after warmup steps; every step ends with the device idle."""
    import torch
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        step()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def pipelined(fl, calls, n, warmup):
    """Seconds per call over n calls with two in flight; calls: (frames, boxes[, out]) tuples, cycled."""
    import torch

    def run(k):
        fl.submit(*calls[0])
        for i in range(1, k):
            fl.submit(*calls[i % len(calls)])
            fl.collect()
        fl.collect()
    run(max(warmup, 2))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(n)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-faces", type=int, default=256)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--align", type=int, default=None, help="chip side: also time FaceLandmark(align=SIZE)")
    args = ap.parse_args()
    import torch
    import frames
    from Skps import FaceLandmark
    from peppa_pig_face_landmark_b200.core.api.face_landmark import crop_read_rects
    K = args.max_faces
    fl = FaceLandmark(max_faces=K)
    eng = fl.model

    # (a) the net alone on resident crops, as bench.py times it
    x = torch.from_numpy(frames.noise_crops(K, seed=100)).cuda()
    outs = [torch.empty((K, e), dtype=torch.float32, device="cuda") for e in eng.out_elems]
    s = eng.stream
    t_a = timed(lambda: eng.forward_device(x, outs, s), args.calls, args.warmup)

    # (b) CUDA 1080p frames, 4 faces each, CUDA boxes, results in out=
    n_frames = K // 4
    base = np.array([[x0, y0, x0 + 440, y0 + 293] for y0 in (123, 663) for x0 in (260, 1220)], np.float32)
    rng = np.random.default_rng(0)
    dev_frames = [torch.from_numpy(frames.frame_1080p(jitter=(int(j), 0))).cuda() for j in rng.integers(-8, 9, 4)]
    dev_boxes = [torch.from_numpy(base + rng.uniform(-2, 2, base.shape).astype(np.float32)).cuda() for _ in range(8)]
    bufs = [fl.new_results(4 * n_frames) for _ in range(2)]
    calls_b = [([dev_frames[(i + j) % 4] for j in range(n_frames)], [dev_boxes[(i + j) % 8] for j in range(n_frames)],
                bufs[i % 2]) for i in range(2)]
    t_b = pipelined(fl, calls_b, args.calls, args.warmup)

    # (c) host 1024x1024 frames, one 300-px face each, through the rectangle upload
    host = [frames.multi_face_frame(1024, 1024, (1, 1), 300, jitter=(int(j), 0)) for j in rng.integers(-20, 21, 4)]
    hb = np.array([[362, 412, 662, 612]], np.float32)
    calls_c = [([host[(i + j) % 4] for j in range(K)], [hb] * K) for i in range(2)]
    t_c = pipelined(fl, calls_c, args.calls, args.warmup)
    r = crop_read_rects(hb, 1024, 1024, fl.face_scale)[0]
    roi = int((r[2] - r[0]) * (r[3] - r[1]) * 3)
    name, limit = card()
    res = {"card": name, "power_limit": limit, "max_faces": K,
           "engine_faces_per_s": K / t_a, "device_faces_per_s": 4 * n_frames / t_b, "host_faces_per_s": K / t_c,
           "device_vs_engine": (4 * n_frames / t_b) / (K / t_a),
           "host_upload_bytes_per_face": roi, "whole_frame_bytes": 1024 * 1024 * 3}
    if args.align is not None:
        from peppa_pig_face_landmark_b200.core.api.align import chip_read_rects
        fl_al = FaceLandmark(max_faces=K, align=args.align)
        bufs_al = [fl_al.new_results(4 * n_frames) for _ in range(2)]
        calls_b_al = [c[:2] + (bufs_al[i],) for i, c in enumerate(calls_b)]
        # alternated: without, with, without, with
        t = {"b": [t_b], "c": [t_c], "b_al": [], "c_al": []}
        for _ in range(2):
            t["b_al"].append(pipelined(fl_al, calls_b_al, args.calls, args.warmup))
            t["c_al"].append(pipelined(fl_al, calls_c, args.calls, args.warmup))
            t["b"].append(pipelined(fl, calls_b, args.calls, args.warmup))
            t["c"].append(pipelined(fl, calls_c, args.calls, args.warmup))
        med = {k: float(np.median(v)) for k, v in t.items()}
        M = fl_al.run_batch([host[0]], [hb])[0][3]
        c = chip_read_rects(M, args.align, 1024, 1024)[0]
        res.update({"align": args.align, "device_faces_per_s": 4 * n_frames / med["b"], "host_faces_per_s": K / med["c"],
                    "device_align_faces_per_s": 4 * n_frames / med["b_al"], "host_align_faces_per_s": K / med["c_al"],
                    "host_align_upload_bytes_per_face": roi + int((c[2] - c[0]) * (c[3] - c[1]) * 3)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
