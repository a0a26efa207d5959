"""Aligned chips from the detector's own landmarks (FaceDetector(align=112)) against the detector alone and against the
98-point path (FaceAnaImages(align=112)), in one process, on the GPU named in the output (name and power limit read in
the same run).  Per config (tools/bench_streams.py: 1080p with 4 faces, 4K with 16 faces), --images frames per call:

    align_cuda_out   FaceDetector(align=112).submit(CUDA frames, out=...), two calls in flight, results left on the GPU
    plain_cuda_out   FaceDetector().submit(CUDA frames, out=...), the same
    align_host       FaceDetector(align=112).run_batch(host frames): chips warped at collect() from the rectangles
    plain_host       FaceDetector().run_batch(host frames)
    images_align     FaceAnaImages(align=112).run_batch(CUDA frames): detector, landmark net, 98-point chips

The modes are alternated over --rounds rounds of --calls calls each; the median is reported.  Before timing, the chips
of align_cuda_out are checked to equal align_host's.

    python tools/bench_detector_align.py [--images 16] [--calls 8] [--rounds 5] [--configs 1080p_4faces,4k_16faces]"""
import json
import os
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

from bench_streams import CONFIGS, gpu_info, make_streams  # noqa: E402

MODES = ("align_cuda_out", "plain_cuda_out", "align_host", "plain_host", "images_align")
SIZE = 112


def run(torch, name, n_images=16, calls=8, rounds=5):
    import frames
    from Skps import FaceAnaImages, FaceDetector
    maker, topk = getattr(frames, CONFIGS[name][0]), CONFIGS[name][1]
    base = make_streams(torch, frames, maker, 1, length=6, pin=False)[0]
    host = [base[i % len(base)] for i in range(n_images)]
    dev = [torch.from_numpy(f).cuda() for f in host]
    H, W = host[0].shape[:2]
    aligned, plain = FaceDetector(max_frames=n_images, align=SIZE), FaceDetector(max_frames=n_images)
    images = FaceAnaImages(top_k=topk, max_frames=n_images, align=SIZE)
    bufs = {"align_cuda_out": [aligned.new_results(n_images) for _ in range(2)],
            "plain_cuda_out": [plain.new_results(n_images) for _ in range(2)]}

    def pipelined(det, mode):
        for c in range(calls):
            if len(det._pending) == 2:
                det.collect()
            det.submit(dev, out=bufs[mode][c % 2])
        while det._pending:
            det.collect()

    def step(mode):
        if mode == "align_cuda_out":
            pipelined(aligned, mode)
        elif mode == "plain_cuda_out":
            pipelined(plain, mode)
        else:
            obj, frames_ = {"align_host": (aligned, host), "plain_host": (plain, host),
                            "images_align": (images, dev)}[mode]
            for _ in range(calls):
                obj.run_batch(frames_)

    # the chips left on the GPU equal the host frames' chips
    want = aligned.run_batch(host)
    out = aligned.new_results(n_images)
    aligned.submit(dev, out=out)
    aligned.collect()
    count = out["count"].cpu().numpy()
    same = all(np.array_equal(out["chip"][i, :min(int(c), aligned.max_chips)].cpu().numpy(), want[i][2]) and
               np.array_equal(out["M"][i, :min(int(c), aligned.max_chips)].cpu().numpy(), want[i][3])
               for i, c in enumerate(count))
    chips = sum(len(w[2]) for w in want)
    for mode in MODES:
        step(mode)
    torch.cuda.synchronize()
    times = {m: [] for m in MODES}
    for r in range(rounds):
        for mode in (MODES if r % 2 == 0 else MODES[::-1]):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(mode)
            torch.cuda.synchronize()
            times[mode].append((time.perf_counter() - t0) / calls)
    res = {"config": name, "images_per_call": n_images, "calls": calls, "rounds": rounds, "frame_hw": [H, W],
           "chip_size": SIZE, "chips_per_call": chips, "device_chips_equal_host_chips": bool(same)}
    for mode in MODES:
        ms = 1e3 * float(np.median(times[mode]))
        res[mode] = {"ms_per_call": ms, "images_per_s": 1e3 * n_images / ms,
                     "ms_per_call_rounds": [1e3 * v for v in times[mode]]}
    return res


def main():
    import torch
    a = sys.argv[1:]

    def opt(name, default):
        return a[a.index(name) + 1] if name in a else default
    n_images, calls, rounds = int(opt("--images", 16)), int(opt("--calls", 8)), int(opt("--rounds", 5))
    names = opt("--configs", ",".join(CONFIGS)).split(",")
    print(json.dumps(gpu_info(torch)))
    sys.stdout.flush()
    for name in names:
        print(json.dumps(run(torch, name, n_images, calls, rounds)))
        sys.stdout.flush()


if __name__ == "__main__":
    main()
