"""Frame ingest from GPU memory in FaceAnaStreams (benchmark configs 3 and 5): the same S synthetic video streams fed as
pinned host frames, as CUDA frames with host results, and as CUDA frames with results left on the GPU (submit(out=...)),
two calls in flight, alternating the three modes over --rounds rounds in one process.  Faces jitter every frame so the
frame-difference gate re-runs the detector on every frame.  Before timing, every mode runs the same calls from a reset
state and its results are checked to be identical to the pinned-host mode's.  At 4K the ingest kernel alone
(skps_frame_ingest of a pitched ROI view against the previous frame) is timed with CUDA events and reported as bytes
moved per second.  The GPU name and power limit are read in the same run.

    python tools/bench_device_frames.py [--streams 16] [--batches 12] [--rounds 5] [--configs 1080p_4faces,4k_16faces]"""
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

MODES = ("host_pinned", "cuda_frames_host_results", "cuda_frames_device_results")


def _host_lists(res, n):
    """Device results (a dict of CUDA tensors) in collect()'s list-of-dicts form."""
    snap = {k: v.cpu().numpy() for k, v in res.items()}
    return [[{"box": snap["box"][s, i], "kps": snap["kps"][s, i], "scores": snap["scores"][s, i]}
             for i in range(int(snap["n"][s]))] for s in range(n)]


def _identical(a, b):
    """Two runs' results (calls -> streams -> faces) are equal field by field."""
    if len(a) != len(b):
        return False
    for call_a, call_b in zip(a, b):
        for faces_a, faces_b in zip(call_a, call_b):
            if len(faces_a) != len(faces_b):
                return False
            for p, q in zip(faces_a, faces_b):
                if any(not np.array_equal(np.asarray(p[k]), np.asarray(q[k])) for k in ("box", "kps", "scores")):
                    return False
    return True


def run_config(name, n_streams=16, batches=12, rounds=5, warmup=3, length=6):
    import torch
    import frames
    from Skps import FaceAnaStreams
    maker, topk = getattr(frames, CONFIGS[name][0]), CONFIGS[name][1]
    seqs = make_streams(torch, frames, maker, n_streams, length=length)
    H, W = seqs[0][0].shape[:2]
    on_gpu = {}
    for s in seqs:
        for f in s:
            if id(f) not in on_gpu:
                on_gpu[id(f)] = torch.from_numpy(f).cuda()
    fa = FaceAnaStreams(n_streams=n_streams, top_k=topk, max_frame_hw=(H, W))
    bufs = [fa.new_results(), fa.new_results()]
    L = len(seqs[0])

    def batch(t, mode):
        fs = [seqs[s][t % L] for s in range(n_streams)]
        return fs if mode == "host_pinned" else [on_gpu[id(f)] for f in fs]

    def calls(mode, keep=False):
        """`batches` calls, two in flight; returns every call's results as host lists when keep."""
        out, k = [], 0

        def submit(t):
            nonlocal k
            if mode == "cuda_frames_device_results":
                fa.submit(batch(t, mode), out=bufs[k])
                k ^= 1
            else:
                fa.submit(batch(t, mode))

        def collect():
            r = fa.collect()
            if keep:
                out.append(_host_lists(r, n_streams) if isinstance(r, dict) else r)
        submit(0)
        for t in range(1, batches):
            submit(t)
            collect()
        collect()
        return out

    for mode in MODES:
        for t in range(warmup):
            fa.submit(batch(t, mode))
            fa.collect()
    ref, same = None, {}
    for mode in MODES:
        fa.reset()
        got = calls(mode, keep=True)
        ref = got if ref is None else ref
        same[mode] = _identical(got, ref)
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
    out = {"config": name, "streams_per_gpu": n_streams, "calls": batches, "rounds": rounds, "frame_hw": [H, W],
           "frame_bytes": int(H * W * 3), "results_identical_to_host_pinned": same}
    for mode in MODES:
        ms = 1e3 * float(np.median(times[mode])) / batches
        out[mode] = {"ms_per_call": ms, "frames_per_s": 1e3 * n_streams / ms,
                     "ms_per_call_rounds": [1e3 * v / batches for v in times[mode]]}
    out["api"] = "FaceAnaStreams.submit/collect, 2 calls in flight; timed from a reset, ending in torch.cuda.synchronize()"
    return out


def time_ingest_kernel(torch, iters=200):
    """CUDA-event time of one skps_frame_ingest of a 3840x2160 frame: a view at an odd byte offset of a wider buffer,
    gathered into a packed buffer and diffed against a previous frame (3 x 24.9 MB moved)."""
    import ctypes as C
    import frames
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    f = frames.frame_4k()
    H, W = f.shape[:2]
    n = H * W * 3
    big = torch.zeros((H + 2, W + 3, 3), dtype=torch.uint8, device="cuda")
    big[1:1 + H, 1:1 + W] = torch.from_numpy(f).cuda()
    rows = {"roi": big[1:1 + H, 1:1 + W], "packed": torch.from_numpy(f).cuda()}
    prev = torch.from_numpy(frames.frame_4k(jitter=(4, 4))).cuda().reshape(-1)
    packed = torch.empty(n, dtype=torch.uint8, device="cuda")
    acc = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    res = {}
    for name, src in rows.items():
        def launch():
            rt.check(lib.skps_frame_ingest(src.data_ptr(), H, W, src.stride(0), packed.data_ptr(), prev.data_ptr(),
                                           acc.data_ptr(), stream))
        for _ in range(20):
            launch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            launch()
        e1.record()
        torch.cuda.synchronize()
        assert torch.equal(packed, src.contiguous().reshape(-1))
        us = 1e3 * e0.elapsed_time(e1) / iters
        moved = 3 * n
        res[name] = {"kernel_us": us, "bytes_moved": moved, "moved_GBps": moved / (us * 1e-6) / 1e9,
                     "moved_share_of_hbm_peak": moved / (us * 1e-6) / HBM_PEAK_BPS,
                     "source_pitch": int(src.stride(0)), "source_offset_bytes": int(src.storage_offset())}
    return {"ingest_kernel_4k": res, "timing": "CUDA events around %d back-to-back launches (each includes the 8-byte "
                                               "memset of the sum)" % iters}


def main():
    import torch
    a = sys.argv[1:]

    def opt(name, default):
        return a[a.index(name) + 1] if name in a else default
    n_streams, batches, rounds = int(opt("--streams", 16)), int(opt("--batches", 12)), int(opt("--rounds", 5))
    names = opt("--configs", ",".join(CONFIGS)).split(",")
    print(json.dumps(gpu_info(torch)))
    print(json.dumps(time_ingest_kernel(torch)))
    sys.stdout.flush()
    for name in names:
        print(json.dumps(run_config(name, n_streams, batches, rounds)))
        sys.stdout.flush()


if __name__ == "__main__":
    main()
