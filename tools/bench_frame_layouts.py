"""CUDA frames in other pixel layouts than interleaved BGR (layout= of FaceAnaStreams, FaceAnaImages, FaceDetector), in
one process, on the GPU named in the output (name and power limit read in the same run):

1. The ingest kernel alone at 4K (skps_frame_ingest_layout), every layout from a pitched ROI view (odd byte offset, rows
   and planes padded) against a previous frame, CUDA events over --iters launches, the layouts alternated over --rounds
   rounds.  Bytes moved = the source bytes (3 or 4 per pixel, 3 for planar) + the previous frame + the packed frame.
   Before timing, every layout's packed frame and sum are checked to equal the BGR ingest's.
2. FaceAnaStreams, --streams streams, two calls in flight, CUDA frames (tools/bench_streams.py configs), three modes
   alternated over --rounds rounds: "bgr" (BGR (H, W, 3) tensors), "rgb_planar" (planar RGB (3, H, W) tensors passed
   with layout="rgb_planar"), "convert" (the same planar RGB tensors turned into BGR by the caller with
   t.permute(1, 2, 0).flip(-1).contiguous() on the current stream, inside the timed region, and passed as BGR).  The
   three modes' results are checked to be identical before timing.
3. FaceAnaImages.run_batch and FaceDetector.run_batch on --images CUDA images of each config, the same three modes.

    python tools/bench_frame_layouts.py [--streams 16] [--batches 12] [--rounds 5] [--iters 200] [--images 16]
                                        [--configs 1080p_4faces,4k_16faces] [--parts ingest,streams,images]"""
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

from bench_streams import CONFIGS, HBM_PEAK_BPS, gpu_info, make_streams  # noqa: E402

LAYOUTS = {"bgr": 0, "rgb": 1, "bgra": 2, "rgba": 3, "bgr_planar": 4, "rgb_planar": 5}
MODES = ("bgr", "rgb_planar", "convert")


def to_layout(torch, f, layout, roi):
    """BGR numpy frame f as a CUDA tensor in `layout`; roi: a view at row 1, column 1 of a buffer 3 pixels wider and 2
    rows higher (planar: planes of a (3, H + 2, W + 3) buffer)."""
    t = torch.from_numpy(np.ascontiguousarray(f)).cuda()
    if layout.startswith("rgb"):
        t = t.flip(-1)
    if layout in ("bgra", "rgba"):
        t = torch.cat([t, torch.full(t.shape[:2] + (1,), 255, dtype=torch.uint8, device="cuda")], 2)
    planar = layout.endswith("_planar")
    if planar:
        t = t.permute(2, 0, 1)
    t = t.contiguous()
    if not roi:
        return t
    if planar:
        big = torch.zeros((3, t.shape[1] + 2, t.shape[2] + 3), dtype=torch.uint8, device="cuda")
        v = big[:, 1:1 + t.shape[1], 1:1 + t.shape[2]]
    else:
        big = torch.zeros((t.shape[0] + 2, t.shape[1] + 3, t.shape[2]), dtype=torch.uint8, device="cuda")
        v = big[1:1 + t.shape[0], 1:1 + t.shape[1]]
    v.copy_(t)
    return v


def time_ingest(torch, rounds=5, iters=200):
    import frames
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    f = frames.frame_4k()
    H, W = f.shape[:2]
    n = H * W * 3
    prev = torch.from_numpy(frames.frame_4k(jitter=(4, 4))).cuda().reshape(-1)
    packed = torch.empty(n, dtype=torch.uint8, device="cuda")
    acc = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    srcs = {k: to_layout(torch, f, k, roi=True) for k in LAYOUTS}

    def launcher(k):
        src, planar = srcs[k], k.endswith("_planar")
        pitch, plane = (src.stride(1), src.stride(0)) if planar else (src.stride(0), 0)

        def launch():
            rt.check(lib.skps_frame_ingest_layout(src.data_ptr(), H, W, pitch, LAYOUTS[k], plane, packed.data_ptr(),
                                                  prev.data_ptr(), acc.data_ptr(), stream))
        return launch
    launch = {k: launcher(k) for k in LAYOUTS}
    want, sums = torch.from_numpy(f).cuda().reshape(-1), {}
    for k in LAYOUTS:
        launch[k]()
        torch.cuda.synchronize()
        sums[k] = int(acc.item())
        assert torch.equal(packed, want), k
    assert len(set(sums.values())) == 1, sums
    times = {k: [] for k in LAYOUTS}
    order = list(LAYOUTS)
    for r in range(rounds):
        for k in (order if r % 2 == 0 else order[::-1]):
            for _ in range(20):
                launch[k]()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                launch[k]()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(1e3 * e0.elapsed_time(e1) / iters)
    res = {}
    for k in LAYOUTS:
        us = float(np.median(times[k]))
        src_bytes = H * W * (4 if k in ("bgra", "rgba") else 3)
        moved = src_bytes + 2 * n
        res[k] = {"kernel_us": us, "kernel_us_rounds": times[k], "bytes_moved": moved,
                  "moved_TBps": moved / (us * 1e-6) / 1e12, "moved_share_of_hbm_peak": moved / (us * 1e-6) / HBM_PEAK_BPS,
                  "source_strides": list(srcs[k].stride()), "source_offset_bytes": int(srcs[k].storage_offset())}
    bgr = res["bgr"]["moved_TBps"]
    for k in LAYOUTS:
        res[k]["bytes_per_s_vs_bgr"] = res[k]["moved_TBps"] / bgr
    return {"ingest_kernel_4k": res, "identical_packed_frame_and_sum": True,
            "timing": "median over %d alternated rounds of CUDA events around %d back-to-back launches (each includes the "
                      "8-byte memset of the sum)" % (rounds, iters)}


def _planar(torch, f):
    return torch.from_numpy(np.ascontiguousarray(f[..., ::-1].transpose(2, 0, 1))).cuda()


def _bgr_of_planar(t):
    return t.permute(1, 2, 0).flip(-1).contiguous()


def _same(a, b):
    if isinstance(a, dict):
        return set(a) == set(b) and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b))


def run_streams(torch, name, n_streams=16, batches=12, rounds=5, warmup=3, length=6):
    import frames
    from Skps import FaceAnaStreams
    maker, topk = getattr(frames, CONFIGS[name][0]), CONFIGS[name][1]
    seqs = make_streams(torch, frames, maker, n_streams, length=length, pin=False)
    H, W = seqs[0][0].shape[:2]
    bgr, planar = {}, {}
    for s in seqs:
        for f in s:
            if id(f) not in bgr:
                bgr[id(f)] = torch.from_numpy(f).cuda()
                planar[id(f)] = _planar(torch, f)
    fa = FaceAnaStreams(n_streams=n_streams, top_k=topk, max_frame_hw=(H, W))

    def submit(t, mode):
        fs = [seqs[s][t % length] for s in range(n_streams)]
        if mode == "bgr":
            fa.submit([bgr[id(f)] for f in fs])
        elif mode == "rgb_planar":
            fa.submit([planar[id(f)] for f in fs], layout="rgb_planar")
        else:
            fa.submit([_bgr_of_planar(planar[id(f)]) for f in fs])

    def calls(mode, keep=False):
        out = []
        submit(0, mode)
        for t in range(1, batches + 1):
            if t < batches:
                submit(t, mode)
            r = fa.collect()
            if keep:
                out.append(r)
        return out
    for mode in MODES:
        for t in range(warmup):
            submit(t, mode)
            fa.collect()
    ref, same = None, {}
    for mode in MODES:
        fa.reset()
        got = calls(mode, keep=True)
        ref = got if ref is None else ref
        same[mode] = _same(got, ref)
    times = {m: [] for m in MODES}
    for r in range(rounds):
        for mode in (MODES if r % 2 == 0 else MODES[::-1]):
            fa.reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            calls(mode)
            torch.cuda.synchronize()
            times[mode].append(time.perf_counter() - t0)
    del fa
    out = {"part": "FaceAnaStreams", "config": name, "streams": n_streams, "calls": batches, "rounds": rounds,
           "frame_hw": [H, W], "results_identical_to_bgr": same,
           "api": "FaceAnaStreams.submit/collect, CUDA frames, host results, 2 calls in flight; timed from a reset, "
                  "ending in torch.cuda.synchronize()"}
    for mode in MODES:
        ms = 1e3 * float(np.median(times[mode])) / batches
        out[mode] = {"ms_per_call": ms, "frames_per_s": 1e3 * n_streams / ms,
                     "ms_per_call_rounds": [1e3 * v / batches for v in times[mode]]}
    return out


def run_images(torch, name, n_images=16, calls=6, rounds=5):
    import frames
    from Skps import FaceAnaImages, FaceDetector
    maker, topk = getattr(frames, CONFIGS[name][0]), CONFIGS[name][1]
    base = make_streams(torch, frames, maker, 1, length=6, pin=False)[0]
    fs = [base[i % len(base)] for i in range(n_images)]
    H, W = fs[0].shape[:2]
    bgr = [torch.from_numpy(f).cuda() for f in fs]
    planar = [_planar(torch, f) for f in fs]
    objs = {"FaceAnaImages": FaceAnaImages(top_k=topk, max_frames=n_images),
            "FaceDetector": FaceDetector(max_frames=n_images)}

    def call(obj, mode):
        if mode == "bgr":
            return obj.run_batch(bgr)
        if mode == "rgb_planar":
            return obj.run_batch(planar, layout="rgb_planar")
        return obj.run_batch([_bgr_of_planar(t) for t in planar])
    res = []
    for cls, obj in objs.items():
        got = {m: call(obj, m) for m in MODES}
        for m in MODES:
            call(obj, m)
        same = {m: _same(got[m], got["bgr"]) for m in MODES}
        times = {m: [] for m in MODES}
        for r in range(rounds):
            for mode in (MODES if r % 2 == 0 else MODES[::-1]):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(calls):
                    call(obj, mode)
                torch.cuda.synchronize()
                times[mode].append((time.perf_counter() - t0) / calls)
        out = {"part": cls, "config": name, "images_per_call": n_images, "calls": calls, "rounds": rounds,
               "frame_hw": [H, W], "results_identical_to_bgr": same,
               "api": "%s.run_batch on CUDA images (blocking), host results" % cls}
        for mode in MODES:
            ms = 1e3 * float(np.median(times[mode]))
            out[mode] = {"ms_per_call": ms, "images_per_s": 1e3 * n_images / ms,
                         "ms_per_call_rounds": [1e3 * v for v in times[mode]]}
        res.append(out)
    return res


def main():
    import torch
    a = sys.argv[1:]

    def opt(name, default):
        return a[a.index(name) + 1] if name in a else default
    n_streams, batches, rounds = int(opt("--streams", 16)), int(opt("--batches", 12)), int(opt("--rounds", 5))
    iters, n_images = int(opt("--iters", 200)), int(opt("--images", 16))
    names = opt("--configs", ",".join(CONFIGS)).split(",")
    parts = opt("--parts", "ingest,streams,images").split(",")
    print(json.dumps(gpu_info(torch)))
    sys.stdout.flush()
    if "ingest" in parts:
        print(json.dumps(time_ingest(torch, rounds, iters)))
        sys.stdout.flush()
    for name in names:
        if "streams" in parts:
            print(json.dumps(run_streams(torch, name, n_streams, batches, rounds)))
            sys.stdout.flush()
        if "images" in parts:
            for r in run_images(torch, name, n_images, rounds=rounds):
                print(json.dumps(r))
                sys.stdout.flush()


if __name__ == "__main__":
    main()
