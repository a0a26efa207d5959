"""CUDA frames stored turned (rotate= of FaceAnaStreams, FaceDetector, FaceAnaImages), in one process, on the GPU named in
the output (name and power limit read in the same run):

1. The ingest kernel alone on a 4K frame (2160 x 3840 upright) stored as a pitched ROI view (odd byte offset, rows and
   planes padded), every layout x rotate 0 / 90 / 180 / 270 (skps_frame_ingest_rotate; rotate 0 runs the unturned
   kernel), against a previous frame, CUDA events over --iters launches, rotations alternated over --rounds rounds.
   Bytes moved = the source bytes (3 or 4 per pixel) + the previous frame + the packed frame.  Before timing, every
   packed frame is checked to equal the upright frame byte for byte and every sum to agree.
2. FaceAnaStreams, --streams streams of portrait content (1080 x 1920 with 4 faces, 2160 x 3840 with 16 faces, upright
   H x W), two calls in flight, CUDA frames, three modes alternated over --rounds rounds: "rotate" (frames stored turned,
   passed with rotate=90), "caller" (the same stored frames turned by the caller with
   torch.rot90(t, -1, (0, 1)).contiguous() on the current stream, inside the timed region), "upright" (frames already
   upright).  The three modes' results are checked to be identical before timing.
3. FaceDetector.run_batch and FaceAnaImages.run_batch on --images CUDA images of each config, the same three modes.

    python tools/bench_frame_rotation.py [--streams 16] [--batches 12] [--rounds 5] [--iters 200] [--images 16]
                                         [--configs portrait1080_4faces,portrait4k_16faces] [--parts ingest,streams,images]"""
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

from bench_frame_layouts import LAYOUTS, _same, to_layout  # noqa: E402
from bench_streams import HBM_PEAK_BPS, gpu_info  # noqa: E402

# upright H, W, face grid, face width, top_k
CONFIGS = {"portrait1080_4faces": (1920, 1080, (2, 2), 440, 4), "portrait4k_16faces": (3840, 2160, (4, 4), 520, 16)}
MODES = ("rotate", "caller", "upright")
ROTATES = (0, 90, 180, 270)


def _stored(f, rotate):
    """The stored frame that rotate= turns upright into f (numpy)."""
    return np.ascontiguousarray(np.rot90(f, rotate // 90))


def time_ingest(torch, rounds=5, iters=200):
    import frames
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    up = frames.frame_4k()
    H, W = up.shape[:2]
    n = H * W * 3
    prev = torch.from_numpy(frames.frame_4k(jitter=(4, 4))).cuda().reshape(-1)
    packed = torch.empty(n, dtype=torch.uint8, device="cuda")
    acc = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    want = torch.from_numpy(up).cuda().reshape(-1)
    res, sums = {}, set()
    for layout in LAYOUTS:
        srcs = {r: to_layout(torch, _stored(up, r), layout, roi=True) for r in ROTATES}

        def launcher(r):
            src, planar = srcs[r], layout.endswith("_planar")
            hs, ws = (src.shape[1], src.shape[2]) if planar else (src.shape[0], src.shape[1])
            pitch, plane = (src.stride(1), src.stride(0)) if planar else (src.stride(0), 0)

            def launch():
                rt.check(lib.skps_frame_ingest_rotate(src.data_ptr(), hs, ws, pitch, LAYOUTS[layout], plane, r // 90,
                                                      packed.data_ptr(), prev.data_ptr(), acc.data_ptr(), stream))
            return launch
        launch = {r: launcher(r) for r in ROTATES}
        for r in ROTATES:
            packed.zero_()
            launch[r]()
            torch.cuda.synchronize()
            sums.add(int(acc.item()))
            assert torch.equal(packed, want), (layout, r)
        times = {r: [] for r in ROTATES}
        for k in range(rounds):
            for r in (ROTATES if k % 2 == 0 else ROTATES[::-1]):
                for _ in range(20):
                    launch[r]()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    launch[r]()
                e1.record()
                torch.cuda.synchronize()
                times[r].append(1e3 * e0.elapsed_time(e1) / iters)
        moved = H * W * (4 if layout in ("bgra", "rgba") else 3) + 2 * n
        res[layout] = {}
        for r in ROTATES:
            us = float(np.median(times[r]))
            res[layout][r] = {"kernel_us": us, "moved_TBps": moved / (us * 1e-6) / 1e12,
                              "moved_share_of_hbm_peak": moved / (us * 1e-6) / HBM_PEAK_BPS}
        for r in ROTATES:
            res[layout][r]["bytes_per_s_vs_rotate0"] = res[layout][0]["kernel_us"] / res[layout][r]["kernel_us"]
    assert len(sums) == 1, sums
    return {"ingest_kernel_4k_roi": res, "identical_packed_frame_and_sum": True,
            "timing": "median over %d alternated rounds of CUDA events around %d back-to-back launches (each includes the "
                      "8-byte memset of the sum)" % (rounds, iters)}


def make_content(name, n, length=6):
    """`length` distinct upright frames (faces jittered by multiples of 4 px); entry s of the result walks them from s."""
    import frames
    h, w, grid, face_w, _ = CONFIGS[name]
    base = [frames.multi_face_frame(h, w, grid, face_w, jitter=(4 * (t % 3), 4 * (t // 3))) for t in range(length)]
    return [[base[(t + s) % length] for t in range(length)] for s in range(n)]


class Inputs:
    """The three modes' CUDA frames of each upright frame: stored turned (rotate=90), and upright."""

    def __init__(self, torch, seqs):
        self.torch, self.stored, self.up = torch, {}, {}
        for s in seqs:
            for f in s:
                if id(f) not in self.up:
                    self.up[id(f)] = torch.from_numpy(f).cuda()
                    self.stored[id(f)] = torch.from_numpy(_stored(f, 90)).cuda()

    def args(self, fs, mode):
        """(frames, rotate) of the call in `mode`"""
        if mode == "rotate":
            return [self.stored[id(f)] for f in fs], 90
        if mode == "caller":
            return [self.torch.rot90(self.stored[id(f)], -1, (0, 1)).contiguous() for f in fs], 0
        return [self.up[id(f)] for f in fs], 0


def run_streams(torch, name, n_streams=16, batches=12, rounds=5, warmup=3, length=6):
    from Skps import FaceAnaStreams
    seqs = make_content(name, n_streams, length)
    H, W = seqs[0][0].shape[:2]
    inp = Inputs(torch, seqs)
    fa = FaceAnaStreams(n_streams=n_streams, top_k=CONFIGS[name][4], max_frame_hw=(H, W))

    def submit(t, mode):
        fs, rot = inp.args([seqs[s][t % length] for s in range(n_streams)], mode)
        fa.submit(fs, rotate=rot)

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
           "upright_hw": [H, W], "results_identical": same,
           "api": "FaceAnaStreams.submit/collect, CUDA frames, host results, 2 calls in flight; timed from a reset, "
                  "ending in torch.cuda.synchronize()"}
    for mode in MODES:
        ms = 1e3 * float(np.median(times[mode])) / batches
        out[mode] = {"ms_per_call": ms, "frames_per_s": 1e3 * n_streams / ms,
                     "ms_per_call_rounds": [1e3 * v / batches for v in times[mode]]}
    out["rotate_vs_upright_frames_per_s"] = out["upright"]["ms_per_call"] / out["rotate"]["ms_per_call"]
    out["rotate_vs_caller_frames_per_s"] = out["caller"]["ms_per_call"] / out["rotate"]["ms_per_call"]
    return out


def run_images(torch, name, n_images=16, calls=6, rounds=5):
    from Skps import FaceAnaImages, FaceDetector
    base = make_content(name, 1)[0]
    fs = [base[i % len(base)] for i in range(n_images)]
    H, W = fs[0].shape[:2]
    inp = Inputs(torch, [fs])
    objs = {"FaceAnaImages": FaceAnaImages(top_k=CONFIGS[name][4], max_frames=n_images),
            "FaceDetector": FaceDetector(max_frames=n_images)}

    def call(obj, mode):
        frs, rot = inp.args(fs, mode)
        return obj.run_batch(frs, rotate=rot)
    res = []
    for cls, obj in objs.items():
        got = {m: call(obj, m) for m in MODES}
        for m in MODES:
            call(obj, m)
        same = {m: _same(got[m], got["upright"]) for m in MODES}
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
               "upright_hw": [H, W], "results_identical": same,
               "api": "%s.run_batch on CUDA images (blocking), host results" % cls}
        for mode in MODES:
            ms = 1e3 * float(np.median(times[mode]))
            out[mode] = {"ms_per_call": ms, "images_per_s": 1e3 * n_images / ms,
                         "ms_per_call_rounds": [1e3 * v for v in times[mode]]}
        out["rotate_vs_upright_images_per_s"] = out["upright"]["ms_per_call"] / out["rotate"]["ms_per_call"]
        out["rotate_vs_caller_images_per_s"] = out["caller"]["ms_per_call"] / out["rotate"]["ms_per_call"]
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
