"""Crowd frames on one GPU: the detector post-processing of any size (csrc/nms.cu) and the whole pipeline on frames of 48 to
384 faces, plus the ordinary-frame benchmarks alternated with an earlier build.

    python tools/bench_crowd.py [--iters 50] [--rounds 3] [--parent DIR] [--out DIR]

1. NMS stage alone (skps_detect_post_batch, CUDA events, median over --iters launches) on the raw detector output of
   3840x2160 crowds of test1.jpg copies: 48 faces at 384x640 (about 576 candidates), 96 at 768x1280 (about 1250), 192 and 384
   at 1152x1920 (about 2200 and 5200), and a synthetic frame with every one of the 60480 rows of 768x1280 over the threshold.
   With --parent, the parent's skps_detect_post (its single-block kernel, at most 1024 candidates) is timed on the same rows
   where it accepts them.
2. Whole pipeline at det_input=(1152, 1920): FaceAna.run and FaceAnaStreams.run (4 streams) per call on the 384-face crowd,
   the detector running on every call.
   FaceAna.run on the 384-face crowd at top_k 16, 64 and 512, split into the frame-difference gate, the device chain
   (detector + selection + landmark chunks; skps_pipeline_run), the landmark forwards alone (CUDA events on the landmark
   engine at the chunk sizes that many faces take) and the host temporal layer (the rest of the call).
3. With --parent DIR (a built checkout of an earlier commit): tools/bench_streams.py at 1080p_4faces and 4k_16faces,
   tools/bench_detector.py and FaceAna.run at the default config on the golden frames, alternating this tree and DIR over
   --rounds rounds, and whether FaceAna / FaceAnaStreams return bit-identical results at the default 384x640 input on the
   golden frames in both trees.
The GPU name and power limit are read in the same run.  Nothing is written outside --out."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _paths(root):
    for p in (os.path.join(root, "tests"), root):
        if p not in sys.path:
            sys.path.insert(0, p)


CROWDS = [("crowd48_384x640", (6, 8), 300, (384, 640)), ("crowd96_768x1280", (8, 12), 240, (768, 1280)),
          ("crowd192_1152x1920", (12, 16), 180, (1152, 1920)), ("crowd384_1152x1920", (16, 24), 150, (1152, 1920))]


def gpu_info(torch):
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except Exception as e:            # the numbers stay valid, only the label is missing
        info["power_limit_and_max_sm_clock"] = "unavailable: %s" % e
    return info


def _events(torch, fn, iters):
    s = torch.cuda.current_stream()
    for _ in range(3):
        fn(s)
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        fn(s)
        b.record(s)
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def time_nms(torch, iters, parent_lib=None):
    import numpy as np
    import frames
    from peppa_pig_face_landmark_b200 import runtime as rt
    from peppa_pig_face_landmark_b200.core.api.face_detector import FaceDetector, letterbox_geometry
    from peppa_pig_face_landmark_b200.core.api.facer import get_cfg
    lib = rt.load_library()
    cases = []
    for name, grid, fw, hw in CROWDS:
        cfg = get_cfg()['Skps']['Detect']
        cfg['input_shape'] = [hw[0], hw[1], 3]
        det = FaceDetector(cfg)
        fr = frames.multi_face_frame(2160, 3840, grid, fw)
        kept = det(fr)
        raw = torch.empty((det._rows, 16), dtype=torch.float32, device="cuda")
        rows = det._rows
        # the engine's output buffer, copied out so that only the post-processing is timed
        tmp = np.empty((rows, 16), np.float32)
        rt.check(lib.skps_engine_read_buffer(det.model.handle, det.model.plan.outputs[0].buf.idx, 1, tmp.ctypes.data))
        raw.copy_(torch.from_numpy(tmp))
        scale, _, _, top, left = letterbox_geometry(2160, 3840, *hw)
        cases.append((name, raw, rows, [scale, float(left), float(top)], len(kept)))
    rng = np.random.default_rng(0)
    rows = 60480
    syn = np.zeros((rows, 16), np.float32)
    centers = rng.uniform((50, 50), (1230, 718), (24, 2))
    syn[:, 0:2] = centers[np.arange(rows) % 24] + rng.normal(0, 6.0, (rows, 2))
    syn[:, 2:4] = rng.uniform(150, 220, (rows, 2))
    syn[:, 4] = rng.uniform(0.5001, 0.99, rows)
    cases.append(("all_rows_768x1280", torch.from_numpy(syn).cuda(), rows, [1.0, 0.0, 0.0], None))
    out = []
    for name, raw, rows, rec, n_kept in cases:
        cand = int((raw[:, 4] > 0.5).sum())
        recd = torch.tensor(rec, dtype=torch.float32, device="cuda")
        keep = torch.empty((rows, 16), dtype=torch.float32, device="cuda")
        idx = torch.empty((rows,), dtype=torch.int32, device="cuda")
        cnt = torch.empty((1,), dtype=torch.int32, device="cuda")
        nb = lib.skps_detect_post_workspace_size(rows, 1)
        ws = torch.empty((nb,), dtype=torch.uint8, device="cuda")

        def run(s):
            rt.check(lib.skps_detect_post_batch(raw.data_ptr(), rows, 1, 0.5, 0.3, recd.data_ptr(), keep.data_ptr(),
                                                idx.data_ptr(), cnt.data_ptr(), rows, ws.data_ptr(), nb, s.cuda_stream))
        r = {"case": name, "rows": rows, "candidates": cand, "ms_nms": round(_events(torch, run, iters), 4)}
        r["kept"] = int(cnt.item())
        if n_kept is not None:
            assert r["kept"] == n_kept
        if parent_lib is not None and cand <= 1024:
            def run_parent(s):
                rt.check(parent_lib.skps_detect_post(raw.data_ptr(), rows, 0.5, 0.3, rec[0], rec[1], rec[2], keep.data_ptr(),
                                                     idx.data_ptr(), cnt.data_ptr(), 256, s.cuda_stream))
            r["ms_parent_detect_post"] = round(_events(torch, run_parent, iters), 4)
        out.append(r)
    return out


def time_pipeline(torch, iters):
    import time
    import frames
    from Skps import FaceAna, FaceAnaStreams
    fr = frames.multi_face_frame(2160, 3840, (16, 24), 150)
    res = {}
    facer = FaceAna(det_input=(1152, 1920))
    fa = FaceAnaStreams(n_streams=4, det_input=(1152, 1920))
    for what, call in (("faceana_ms_per_call", lambda: (facer.reset(), facer.run(fr))),
                       ("streams4_ms_per_call", lambda: (fa.reset(), fa.run([fr] * 4)))):
        for _ in range(3):
            call()
        ts = []
        for _ in range(max(5, iters // 5)):
            torch.cuda.synchronize()
            t = time.perf_counter()
            call()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t) * 1e3)
        ts.sort()
        res[what] = round(ts[len(ts) // 2], 3)
    res.update(case="pipeline_crowd384_1152x1920", faces=len(facer.run(fr)))
    return res


class _TimedLib:
    """The library with host-clock timers around the two synchronous pipeline calls of FaceAna.run."""

    def __init__(self, lib):
        self._lib, self.ms = lib, {}

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if name not in ("skps_pipeline_run", "skps_pipeline_frame_diff"):
            return f

        def timed(*a):
            import time
            t = time.perf_counter()
            rc = f(*a)
            self.ms[name] = self.ms.get(name, 0.0) + (time.perf_counter() - t) * 1e3
            return rc
        return timed


def time_crowd_top_k(torch, iters):
    """FaceAna.run on the 384-face crowd (detector on every call) at several top_k, split by stage."""
    import time
    import frames
    from Skps import FaceAna
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    fr = frames.multi_face_frame(2160, 3840, (16, 24), 150)
    out = []
    for top_k in (16, 64, 512):
        facer = FaceAna(top_k=top_k, det_input=(1152, 1920))
        timed = _TimedLib(facer.lib)
        facer.lib = timed
        for _ in range(3):
            facer.reset()
            n = len(facer.run(fr))
        reps = max(5, iters // 5)
        totals = []
        timed.ms = {}
        for _ in range(reps):
            facer.reset()
            torch.cuda.synchronize()
            t = time.perf_counter()
            facer.run(fr)
            totals.append((time.perf_counter() - t) * 1e3)
        ms = {k: v / reps for k, v in timed.ms.items()}
        # the landmark forwards alone: chunks of 64 and the remainder, on the engine FaceAna built
        eng = facer.face_landmark.model
        chunk = eng.max_batch
        sizes = [chunk] * (n // chunk) + ([n % chunk] if n % chunk else [])

        def fwd(s):
            for b in sizes:
                rt.check(lib.skps_engine_forward(eng.handle, eng.input_ptr(), b, None, s.cuda_stream))
        lm = _events(torch, fwd, max(5, iters // 5))
        totals.sort()
        out.append({"case": "faceana_crowd384_top_k", "top_k": top_k, "faces": n, "landmark_chunks": len(sizes),
                    "ms_per_call_median": round(totals[len(totals) // 2], 3),
                    "ms_per_call_mean": round(sum(totals) / reps, 3),
                    "ms_frame_diff": round(ms.get("skps_pipeline_frame_diff", 0.0), 3),
                    "ms_pipeline_run": round(ms.get("skps_pipeline_run", 0.0), 3),
                    "ms_landmark_forwards": round(lm, 3),
                    "ms_detector_selection_crops": round(ms.get("skps_pipeline_run", 0.0) - lm, 3),
                    "ms_host_temporal_and_rest": round(sum(totals) / reps - sum(ms.values()), 3)})
        del facer
    return out


def time_default(iters):
    """FaceAna.run per call at the default config (top_k 5, 384x640) on the golden frames: test1.jpg with the detector on
    every call, and the golden video sequence (detector or tracker path as the frame difference decides)."""
    import time
    import torch
    import frames
    from golden.make_golden_frames import video_frames
    from Skps import FaceAna
    f = FaceAna()
    t1, v = frames.load_test1(), video_frames()
    res = {}
    for what, call, per in (("faceana_default_test1_ms", lambda: (f.reset(), f.run(t1)), 1),
                            ("faceana_default_video_ms", lambda: [f.run(x) for x in v], len(v))):
        for _ in range(3):
            call()
        ts = []
        for _ in range(max(10, iters)):
            torch.cuda.synchronize()
            t = time.perf_counter()
            call()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t) * 1e3 / per)
        ts.sort()
        res[what] = round(ts[len(ts) // 2], 4)
    return res


def dump_default(path):
    """FaceAna / FaceAnaStreams at the default detector input on the golden frames, every returned array, into one npz."""
    import numpy as np
    import frames
    from golden.make_golden_frames import video_frames
    from Skps import FaceAna, FaceAnaStreams
    out = {}
    for name, fr, k in [("test1", frames.load_test1(), 5), ("canvas640", frames.canvas_640(), 5),
                        ("uhd4k_top5", frames.frame_4k(), 5), ("uhd4k_top16", frames.frame_4k(), 16)]:
        f = FaceAna(top_k=k)
        for t in range(2):
            for i, r in enumerate(f.run(fr)):
                for key in ("box", "kps", "scores"):
                    out["%s_%d_%d_%s" % (name, t, i, key)] = np.asarray(r[key])
        out["%s_det_idx" % name] = f.last_det_idx
    f = FaceAna()
    v = video_frames()
    for t, fr in enumerate(v):
        for i, r in enumerate(f.run(fr)):
            for key in ("box", "kps", "scores"):
                out["video_%d_%d_%s" % (t, i, key)] = np.asarray(r[key])
    fa = FaceAnaStreams(n_streams=3, top_k=16)
    seqs = [v, [frames.frame_4k()] * 6, [frames.load_test1()] * 6]
    for t in range(6):
        for s, res in enumerate(fa.run([q[t] for q in seqs])):
            for i, r in enumerate(res):
                for key in ("box", "kps", "scores"):
                    out["streams_%d_%d_%d_%s" % (t, s, i, key)] = np.asarray(r[key])
    np.savez(path, **out)


def _run_json(cmd, cwd):
    r = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("%s failed in %s:\n%s" % (cmd, cwd, r.stdout[-3000:]))
    return [json.loads(l) for l in r.stdout.splitlines() if l.startswith("{")]


def compare_with_parent(parent, rounds, out_dir):
    import numpy as np
    trees = {"this": ROOT, "parent": os.path.abspath(parent)}
    py = sys.executable
    res = {k: {"streams": [], "detector": [], "default": []} for k in trees}
    for _ in range(rounds):
        for k, root in trees.items():
            res[k]["streams"] += _run_json([py, "tools/bench_streams.py", "--configs", "1080p_4faces,4k_16faces"], root)
            res[k]["detector"] += _run_json([py, "tools/bench_detector.py"], root)
            res[k]["default"] += _run_json([py, os.path.abspath(__file__), "--time-default", "--root", root], root)
    summary = {}
    for k in trees:
        by = {}
        for r in res[k]["default"]:
            for name, v in r.items():
                by.setdefault(name, []).append(v)
        for r in res[k]["streams"]:
            if "config" in r and "ms_per_call" in r:
                by.setdefault(r["config"], []).append(r["ms_per_call"])
        for r in res[k]["detector"]:
            for key in ("ms", "ms_per_batch", "ms_per_forward"):
                if key in r:
                    by.setdefault("detector_b%s_%s" % (r.get("batch", r.get("B", "?")), key), []).append(r[key])
        summary[k] = {name: {"median": float(np.median(v)), "all": v} for name, v in by.items()}
    summary["raw_lines"] = res
    dumps = {}
    for k, root in trees.items():
        path = os.path.join(out_dir, "default_%s.npz" % k)
        subprocess.run([py, os.path.abspath(__file__), "--dump", path, "--root", root], check=True, cwd=root)
        dumps[k] = np.load(path)
    a, b = dumps["this"], dumps["parent"]
    same = sorted(a.files) == sorted(b.files) and all(np.array_equal(a[f], b[f]) for f in a.files)
    summary["default_outputs_bit_identical"] = bool(same)
    summary["default_outputs_arrays"] = len(a.files)
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dump", default=None)
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--time-default", action="store_true")
    args = ap.parse_args()
    _paths(args.root)
    if args.dump:
        dump_default(args.dump)
        return
    if args.time_default:
        print(json.dumps(time_default(args.iters)), flush=True)
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_crowd: no CUDA device")
    print(json.dumps(gpu_info(torch)), flush=True)
    parent_lib = None
    if args.parent:
        parent_lib = C.CDLL(os.path.join(os.path.abspath(args.parent), "peppa_pig_face_landmark_b200", "libskps_b200.so"))
        parent_lib.skps_detect_post.restype = C.c_int
        parent_lib.skps_detect_post.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    for r in time_nms(torch, args.iters, parent_lib):
        print(json.dumps(r), flush=True)
    print(json.dumps(time_pipeline(torch, args.iters)), flush=True)
    for r in time_crowd_top_k(torch, args.iters):
        print(json.dumps(r), flush=True)
    if args.parent:
        out_dir = os.path.abspath(args.out or tempfile.mkdtemp(prefix="bench_crowd_"))
        os.makedirs(out_dir, exist_ok=True)
        print(json.dumps(compare_with_parent(args.parent, args.rounds, out_dir)), flush=True)


if __name__ == "__main__":
    main()
