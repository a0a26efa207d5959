"""FaceAna over still images on one GPU, the modes alternated in one run:
  (a) faceana  FaceAna.run(image) + reset() per image;
  (b) streams  FaceAnaStreams(n) reset() + run(images), on the images that fit its max_frame_hw (the rest are skipped
               and counted);
  (c) host     FaceAnaImages.submit(host images) with two calls in flight, results back on the host;
  (d) cuda     the same with CUDA images;
  (e) out      the same with CUDA images and out= (results left on the GPU);
  (f) engines  the detector engine alone at batch max_frames and the landmark engine alone at batch max_faces, as the
               ceiling: a call's engine time is n images x detector time per frame + its faces x landmark time per face.
With --align SIZE, (c), (d) and (e) also run with FaceAnaImages(align=SIZE), as host_align, cuda_align and out_align,
alternated with the others, and the host upload counts the chip rectangles (chip_read_rects) as well.
Workloads: 16 x 1080p with 4 faces, 16 x 4K with 16 faces (top_k 16), and a photo collection of 16 images of mixed
sizes (4000x3000, 3000x4000, 1920x1080, 1280x720, 640x480) with 0-6 faces each.  Prints one JSON line per workload and
mode: median images/s over the rounds and its spread, faces/s, ms per call, call time over engine time, and for host
images the bytes one call uploads; then the card's name and power limit read in the same run.

    python tools/bench_images.py [--rounds 5] [--iters 10] [--images 16] [--align SIZE]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


def photos(n):
    """n images cycling through five sizes, with 0..6 faces each."""
    import frames
    sizes = [(3000, 4000), (4000, 3000), (1080, 1920), (720, 1280), (480, 640)]
    grids = [(0, 0), (1, 1), (1, 2), (1, 3), (2, 2), (1, 5), (2, 3)]
    out = []
    for i in range(n):
        h, w = sizes[i % len(sizes)]
        rows, cols = grids[i % len(grids)]
        if rows == 0:
            out.append(frames._background(h, w))
            continue
        face_w = int(min(0.7 * w / cols, 0.7 * h / rows * 410 / 273))
        out.append(frames.multi_face_frame(h, w, (rows, cols), face_w))
    return out


def workloads(n):
    import frames
    return {"1080p_4faces": (5, [frames.frame_1080p(jitter=(i % 5, -(i % 3))) for i in range(n)]),
            "4k_16faces": (16, [frames.frame_4k(jitter=(i % 5, -(i % 3))) for i in range(n)]),
            "photos_mixed": (6, photos(n))}


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def upload_bytes(fi, imgs):
    """Bytes one host-image call of FaceAnaImages sends: the detector's rows (host_upload_rows) and descriptors, and the
    crop rectangles of the selected faces (crop_read_rects) with their descriptors and boxes; with align, also the chip
    rectangles (chip_read_rects) with their descriptors."""
    from peppa_pig_face_landmark_b200.core.api.align import chip_read_rects
    from oracle.host_ref import sort_and_filter
    from peppa_pig_face_landmark_b200.core.api.face_detector import DET_SRC, host_upload_rows, letterbox_geometry
    from peppa_pig_face_landmark_b200.core.api.face_landmark import FACE_SRC, crop_read_rects
    fd, fl = fi.detector, fi.landmark
    n, det, kps, chips = len(imgs), (DET_SRC.itemsize + 12) * len(imgs), 0, 0
    res = fi.run_batch(imgs) if fi.align is not None else [[]] * n
    for img, rows, faces in zip(imgs, fd.run_batch(imgs), res):
        H, W = img.shape[:2]
        r = host_upload_rows(H, letterbox_geometry(H, W, *fd.input_size[:2])[2])
        det += (H if r is None else len(r)) * 3 * W
        boxes = np.asarray(sort_and_filter(rows, fi.min_face, fi.top_k), np.float32).reshape(-1, 16)
        rect = crop_read_rects(boxes, H, W, fl.face_scale)
        kps += int(((rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1]) * 3).sum()) + (FACE_SRC.itemsize + 16) * len(rect)
        if faces:
            rect = chip_read_rects(np.stack([r["M"] for r in faces]), fi.align, H, W)
            chips += int(((rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1]) * 3).sum()) + FACE_SRC.itemsize * len(rect)
    out = {"detector": det, "landmarks": kps, "whole_images": int(sum(f.nbytes for f in imgs)), "images": n}
    if fi.align is not None:
        out["chips"] = chips
    return out


def engine_times(fi, iters):
    """ms per frame of the detector engine at batch max_frames, ms per face of the landmark engine at max_faces."""
    import torch
    out = []
    for eng, B in ((fi.detector.model, fi.max_frames), (fi.landmark.model, fi.max_faces)):
        h, w = eng.plan.input.H, eng.plan.input.W
        x = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (B, h, w, 3), dtype=np.uint8)).cuda()
        outs = [torch.empty((B, e), dtype=torch.float32, device="cuda") for e in eng.out_elems]
        s = eng.stream
        with torch.cuda.stream(s):
            for _ in range(3):
                eng.forward_device(x, outs, s)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                eng.forward_device(x, outs, s)
            e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / iters / B)
    return out


def in_flight(fi, calls, iters, outs=None):
    """iters calls with two in flight; seconds from the first submit to the last result."""
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(iters):
        if len(fi._pending) == 2:
            fi.collect()
        fi.submit(calls, out=None if outs is None else outs[i % 2])
    while fi._pending:
        fi.collect()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def per_image(fa, imgs, iters):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        for f in imgs:
            fa.reset()
            fa.run(f)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def streams(fs, imgs, iters):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fs.reset()
        fs.run(imgs)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10, help="calls of --images images per mode and round")
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--align", type=int, default=None, help="chip side: also time FaceAnaImages(align=SIZE)")
    a = ap.parse_args()
    import logging
    import torch
    from Skps import FaceAna, FaceAnaImages, FaceAnaStreams
    from peppa_pig_face_landmark_b200.logger.logger import logger
    logger.setLevel(logging.WARNING)
    B = a.images
    for name, (top_k, imgs) in workloads(B).items():
        fi = FaceAnaImages(top_k=top_k)
        fa = FaceAna(top_k=top_k, max_frame_hw=(4096, 4096))
        fs = FaceAnaStreams(B, top_k=top_k)
        max_px = fs.max_frame_hw[0] * fs.max_frame_hw[1]
        fit = [f for f in imgs if f.shape[0] * f.shape[1] <= max_px]
        dev = [torch.from_numpy(f).cuda() for f in imgs]
        outs = [fi.new_results(B), fi.new_results(B)]
        faces = sum(len(r) for r in fi.run_batch(imgs))
        faces_fit = sum(len(r) for r in fi.run_batch(fit)) if fit else 0
        up = upload_bytes(fi, imgs)
        fis = {"": fi}
        if a.align is not None:
            fis["_align"] = FaceAnaImages(top_k=top_k, align=a.align)
            up_align = upload_bytes(fis["_align"], imgs)
            outs_align = [fis["_align"].new_results(B), fis["_align"].new_results(B)]
        # warm every mode once
        for suffix, f in fis.items():
            o = outs if not suffix else outs_align
            in_flight(f, imgs, 2)
            in_flight(f, dev, 2)
            in_flight(f, dev, 2, o)
        per_image(fa, imgs, 1)
        if fit:
            streams(fs, fit, 1)
        engine_times(fi, 3)
        n_one = max(1, a.iters // 5)
        secs = {m + x: [] for m in ("faceana", "streams", "host", "cuda", "out") for x in fis
                if not x or m in ("host", "cuda", "out")}
        eng = []
        for _ in range(a.rounds):
            secs["faceana"].append(per_image(fa, imgs, n_one) / n_one)
            if fit:
                secs["streams"].append(streams(fs, fit, a.iters) / a.iters)
            for suffix, f in fis.items():
                o = outs if not suffix else outs_align
                secs["host" + suffix].append(in_flight(f, imgs, a.iters) / a.iters)
                secs["cuda" + suffix].append(in_flight(f, dev, a.iters) / a.iters)
                secs["out" + suffix].append(in_flight(f, dev, a.iters, o) / a.iters)
            eng.append(engine_times(fi, a.iters))
        det_ms, kps_ms = (float(np.median([e[i] for e in eng])) for i in range(2))
        engine_ms = B * det_ms + faces * kps_ms
        for m, t in secs.items():
            if not t:
                continue
            n_img, n_face = (len(fit), faces_fit) if m == "streams" else (B, faces)
            ms = 1e3 * float(np.median(t))
            r = {"workload": name, "mode": m, "top_k": top_k, "images": n_img, "faces": n_face, "ms_per_call": ms,
                 "ms_min": 1e3 * min(t), "ms_max": 1e3 * max(t), "images_per_s": n_img / ms * 1e3,
                 "faces_per_s": n_face / ms * 1e3}
            if m == "streams":
                r["skipped_images"] = B - len(fit)
            if m.split("_")[0] in ("host", "cuda", "out"):
                r["call_over_engine_time"] = ms / engine_ms
            if m in ("host", "host_align", "faceana"):
                r["host_upload_bytes_per_call"] = {"host": up, "faceana": up["whole_images"]}.get(m) or up_align
            print(json.dumps(r), flush=True)
        print(json.dumps({"workload": name, "mode": "engines", "detector_ms_per_frame": det_ms,
                          "landmark_ms_per_face": kps_ms, "engine_ms_per_call": engine_ms,
                          "images_per_s": B / engine_ms * 1e3, "faces_per_s": faces / engine_ms * 1e3}), flush=True)
        del fi, fa, fs, dev, outs, fis
        torch.cuda.empty_cache()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
