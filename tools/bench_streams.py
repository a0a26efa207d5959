"""Full-pipeline throughput with FaceAnaStreams (benchmark configs 3 and 5): S concurrent synthetic video streams per GPU,
one frame per stream per call, two calls in flight (frame uploads overlap compute).  Faces jitter every frame so the
frame-difference gate re-runs the detector on every frame (the worst case for the pipeline).  Host (pinned) frames in,
host results out: every H2D / D2H is inside the timed region.

    python tools/bench_streams.py [--streams 16] [--batches 12] [--configs 1080p_4faces,4k_16faces] [--gather]
    python tools/bench_streams.py --align 112 [--rounds 5] [--streams 16] [--batches 12] [--configs ...]
    python tools/bench_streams.py --pose [--parent-headpose OLD_headpose.cu --out DIR] [--rounds 5] [--configs ...]
    python tools/bench_streams.py --det-input H W [--rounds 5] [--streams 16] [--batches 12] [--configs ...]
    python tools/bench_streams.py --track-ids [--id-memory N] [--rounds 5] [--streams 16] [--batches 12] [--configs ...]
    python tools/bench_streams.py --detect-every N [--det-input H W] [--rounds 5] [--streams 16] [--batches 12] [--configs ...]

--align SIZE times every config with and without aligned face chips (FaceAnaStreams(align=SIZE)) in the same process,
alternating the two over --rounds rounds, and reports the median ms_per_call of both.  At 4k_16faces it also times the
alignment kernel alone with CUDA events (skps_align_faces on one 4K frame in HBM, the landmarks of every face of the last
call) and reports the bytes it writes per second.  The GPU name and power limit are read in the same run.

--pose does the same with and without head pose (FaceAnaStreams(pose=True)), then times the pose solver alone
(head_pose_warp_kernel, torch.profiler kernel times) at 16, 256 and 1024 faces.  --parent-headpose compiles an earlier
csrc/headpose.cu into a side library under --out (not part of the package), times its kernel at the same sizes in the same
run and reports the largest difference of its skps_head_pose results from this build's on tests/test_headpose_gpu.py's inputs.

--det-input H W does the same with the detector at Skps.yml's 384x640 and at H x W (FaceAnaStreams(det_input=(H, W))).

--track-ids does the same without and with track ids in the results (FaceAnaStreams(track_ids=True)).  With --id-memory N
it compares FaceAnaStreams(track_ids=True) and FaceAnaStreams(track_ids=True, id_memory=N) instead.

--detect-every N does the same with FaceAnaStreams(detect_every=1) and (detect_every=N), at Skps.yml's detector input or,
with --det-input H W, at H x W, and reports detector_frames_per_call of both (the mean of last_detector_frames).  Every
detector batch size the staggered cadence meets is warmed up first (the detector engine captures one CUDA graph per batch
size).  It then times FaceAna.run per call on stream 0's frames at detect_every 1 and N, alternating over the same rounds.

Under torchrun every rank drives its own S streams on its own GPU (streams shard across GPUs, no collective on the data
path); time = max over ranks.  --gather adds one NCCL all_gather of the packed (box, landmarks, scores) rows per call."""
import json
import os
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

CONFIGS = {"1080p_4faces": ("frame_1080p", 4), "4k_16faces": ("frame_4k", 16)}


def make_streams(torch, frames, maker, n_streams, length=6, seed0=0, pin=True):
    """`length` distinct frames per rank (faces jittered by multiples of 4 px), every stream walks them with its own phase:
    consecutive frames of a stream differ, so the frame-difference gate re-runs the detector, and the set-up cost does not
    grow with the number of streams (a 4K frame takes ~0.3 s to synthesise on a host core)."""
    rng = np.random.default_rng(seed0)
    jit = []
    while len(jit) < length:                      # no two consecutive frames alike (the walk is cyclic)
        j = (int(rng.integers(-2, 3)) * 4, int(rng.integers(-2, 3)) * 4)
        if not jit or (j != jit[-1] and (len(jit) < length - 1 or j != jit[0])):
            jit.append(j)
    base = [maker(jitter=j) for j in jit]
    if pin:
        base = [torch.from_numpy(f).pin_memory().numpy() for f in base]       # what a capture / decoder ring hands over
    return [[base[(t + s) % length] for t in range(length)] for s in range(n_streams)]


def run_config(name, n_streams=16, batches=12, warmup=3, gather=False, dist=None, rank=0, world=1, length=6):
    """Returns a dict with whole-job frames/s and faces/s (all ranks), or None on ranks != 0."""
    import torch
    import frames
    from Skps import FaceAnaStreams
    maker, topk = getattr(frames, CONFIGS[name][0]), CONFIGS[name][1]
    seqs = make_streams(torch, frames, maker, n_streams, length=length, seed0=1000 * rank)
    H, W = seqs[0][0].shape[:2]
    fa = FaceAnaStreams(n_streams=n_streams, top_k=topk, max_frame_hw=(H, W))
    L = len(seqs[0])
    rows = torch.zeros((n_streams * topk, 298), device="cuda") if (gather and dist is not None) else None
    allrows = [torch.zeros_like(rows) for _ in range(world)] if rows is not None else None

    def batch(t):
        return [seqs[s][t % L] for s in range(n_streams)]

    def consume(res):
        n = sum(len(r) for r in res)
        if rows is not None:
            host = np.zeros((n_streams * topk, 298), np.float32)
            for s, faces in enumerate(res):
                for i, r in enumerate(faces):
                    host[s * topk + i, :4] = r["box"]
                    host[s * topk + i, 4:200] = np.asarray(r["kps"], np.float32).reshape(-1)
                    host[s * topk + i, 200:] = r["scores"]
            rows.copy_(torch.from_numpy(host))
            dist.all_gather(allrows, rows)
        return n

    for t in range(warmup):
        fa.run(batch(t))

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    barrier()
    t0 = time.perf_counter()
    faces = 0
    fa.submit(batch(0))
    for t in range(1, batches):
        fa.submit(batch(t))
        faces += consume(fa.collect())
    faces += consume(fa.collect())
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    det_share = float(np.mean(fa.last_ran_detector))
    if dist is not None:
        t = torch.tensor([dt, float(faces)], device="cuda", dtype=torch.float64)
        tmax = t.clone(); dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        tsum = t.clone(); dist.all_reduce(tsum, op=dist.ReduceOp.SUM)
        dt, faces = float(tmax[0]), float(tsum[1])
    del fa
    if rank != 0:
        return None
    frames_total = world * n_streams * batches
    return {"config": name, "n_gpus": world, "streams_per_gpu": n_streams, "calls": batches,
            "frames_per_s": frames_total / dt, "faces_per_s": faces / dt, "faces_per_frame": faces / frames_total,
            "ms_per_call": 1e3 * dt / batches, "h2d_bytes_per_frame": int(H * W * 3),
            "d2h_bytes_per_frame": int(topk * (32 + 98 * 2 * 8 + 98 * 4)), "detector_runs_per_frame": det_share,
            "api": "FaceAnaStreams.submit/collect, pinned host frames, 2 calls in flight, temporal layer on the device",
            "gather_to_rank0": bool(rows is not None)}


def gpu_info(torch):
    """Name and power limit of the current GPU (read-only nvidia-smi query; None where it is not available)."""
    import subprocess
    idx = torch.cuda.current_device()
    info = {"gpu": torch.cuda.get_device_name(idx), "power_limit_w": None, "max_sm_clock_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        pw, clk = [v.strip() for v in out.strip().splitlines()[0].split(",")]
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(pw), float(clk)
    except Exception:
        pass
    return info


HBM_PEAK_BPS = 3.35e12          # H100 SXM data sheet (HBM3)


def time_align_kernel(torch, frame, kps, size, iters=200):
    """CUDA-event time of one skps_align_faces launch (estimate + warp of len(kps) chips from one frame in HBM)."""
    import ctypes as C
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    H, W = frame.shape[:2]
    n = kps.shape[0]
    d_frame = torch.from_numpy(np.ascontiguousarray(frame)).cuda()
    d_kps = torch.from_numpy(np.ascontiguousarray(kps, dtype=np.float64)).cuda()
    chips = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
    M = torch.empty((n, 2, 3), dtype=torch.float64, device="cuda")
    stream = torch.cuda.current_stream()

    def launch():
        rt.check(lib.skps_align_faces(d_frame.data_ptr(), H, W, W * 3, d_kps.data_ptr(), None, n, kps.shape[1], size,
                                      chips.data_ptr(), M.data_ptr(), C.c_void_p(stream.cuda_stream)))
    for _ in range(20):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        launch()
    e1.record()
    torch.cuda.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / iters
    written = n * size * size * 3
    return {"chips": n, "size": size, "kernel_us": us, "bytes_written": written,
            "written_GBps": written / (us * 1e-6) / 1e9, "written_share_of_hbm_peak": written / (us * 1e-6) / HBM_PEAK_BPS,
            "timing": "CUDA events around %d back-to-back launches" % iters}


def run_align_pair(name, size, n_streams=16, batches=12, warmup=3, rounds=5, length=6, feature="align"):
    """The same config with and without alignment (feature="align", chip side `size`), head pose (feature="pose"), track
    ids (feature="track_ids"), the memory of lost track ids (feature="id_memory", `size` frames, both with track ids) or
    the detector at input size `size` = (h, w) (feature="det_input"), alternating; median ms_per_call of each."""
    import torch
    import frames
    from Skps import FaceAnaStreams
    maker, topk = getattr(frames, CONFIGS[name][0]), CONFIGS[name][1]
    seqs = make_streams(torch, frames, maker, n_streams, length=length)
    H, W = seqs[0][0].shape[:2]
    on = {"align": {"align": size}, "pose": {"pose": True}, "det_input": {"det_input": size},
          "track_ids": {"track_ids": True}, "id_memory": {"track_ids": True, "id_memory": size}}[feature]
    off = {"track_ids": True} if feature == "id_memory" else {}
    fas = {"off": FaceAnaStreams(n_streams=n_streams, top_k=topk, max_frame_hw=(H, W), **off),
           "on": FaceAnaStreams(n_streams=n_streams, top_k=topk, max_frame_hw=(H, W), **on)}
    L = len(seqs[0])

    def batch(t):
        return [seqs[s][t % L] for s in range(n_streams)]
    for fa in fas.values():
        for t in range(warmup):
            fa.run(batch(t))
    times = {"off": [], "on": []}
    faces, last = {}, None
    for r in range(rounds):
        for key in (("off", "on") if r % 2 == 0 else ("on", "off")):
            fa = fas[key]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            nf = 0
            fa.submit(batch(0))
            for t in range(1, batches):
                fa.submit(batch(t))
                nf += sum(len(x) for x in fa.collect())
            res = fa.collect()
            nf += sum(len(x) for x in res)
            torch.cuda.synchronize()
            times[key].append(time.perf_counter() - t0)
            faces[key] = nf
            if key == "on":
                last = res
    per_face = 32 + 98 * 2 * 8 + 98 * 4
    if feature == "det_input":
        del fas
        ms = {k: 1e3 * float(np.median(v)) / batches for k, v in times.items()}
        return {"config": name, "streams_per_gpu": n_streams, "calls": batches, "rounds": rounds, "det_input": list(size),
                "ms_per_call_384x640": ms["off"], "ms_per_call_det_input": ms["on"],
                "frames_per_s_384x640": 1e3 * n_streams / ms["off"], "frames_per_s_det_input": 1e3 * n_streams / ms["on"],
                "ms_per_call_384x640_rounds": [1e3 * v / batches for v in times["off"]],
                "ms_per_call_det_input_rounds": [1e3 * v / batches for v in times["on"]],
                "faces_per_frame_384x640": faces["off"] / (n_streams * batches),
                "faces_per_frame_det_input": faces["on"] / (n_streams * batches),
                "api": "FaceAnaStreams.submit/collect, pinned host frames, 2 calls in flight"}
    if feature == "track_ids":
        del fas
        ms = {k: 1e3 * float(np.median(v)) / batches for k, v in times.items()}
        return {"config": name, "streams_per_gpu": n_streams, "calls": batches, "rounds": rounds,
                "ms_per_call": ms["off"], "ms_per_call_track_ids": ms["on"],
                "frames_per_s": 1e3 * n_streams / ms["off"], "frames_per_s_track_ids": 1e3 * n_streams / ms["on"],
                "ms_per_call_rounds": [1e3 * v / batches for v in times["off"]],
                "ms_per_call_track_ids_rounds": [1e3 * v / batches for v in times["on"]],
                "faces_per_frame": faces["on"] / (n_streams * batches),
                "api": "FaceAnaStreams.submit/collect, pinned host frames, 2 calls in flight; ids kept on the device"}
    if feature == "id_memory":
        del fas
        ms = {k: 1e3 * float(np.median(v)) / batches for k, v in times.items()}
        return {"config": name, "streams_per_gpu": n_streams, "calls": batches, "rounds": rounds, "id_memory": size,
                "ms_per_call_id_memory_0": ms["off"], "ms_per_call_id_memory": ms["on"],
                "ms_per_call_id_memory_0_rounds": [1e3 * v / batches for v in times["off"]],
                "ms_per_call_id_memory_rounds": [1e3 * v / batches for v in times["on"]],
                "faces_per_frame": faces["on"] / (n_streams * batches),
                "api": "FaceAnaStreams(track_ids=True).submit/collect, pinned host frames, 2 calls in flight"}
    if feature == "pose":
        del fas
        return {"config": name, "streams_per_gpu": n_streams, "calls": batches, "rounds": rounds,
                "ms_per_call": 1e3 * float(np.median(times["off"])) / batches,
                "ms_per_call_pose": 1e3 * float(np.median(times["on"])) / batches,
                "ms_per_call_rounds": [1e3 * v / batches for v in times["off"]],
                "ms_per_call_pose_rounds": [1e3 * v / batches for v in times["on"]],
                "faces_per_frame": faces["on"] / (n_streams * batches),
                "d2h_bytes_per_frame": int(topk * per_face), "d2h_bytes_per_frame_pose": int(topk * (per_face + 25 * 8)),
                "api": "FaceAnaStreams.submit/collect, pinned host frames, 2 calls in flight; pose: solved in submit"}
    out = {"config": name, "streams_per_gpu": n_streams, "calls": batches, "rounds": rounds, "align_size": size,
           "ms_per_call": 1e3 * float(np.median(times["off"])) / batches,
           "ms_per_call_align": 1e3 * float(np.median(times["on"])) / batches,
           "ms_per_call_rounds": [1e3 * v / batches for v in times["off"]],
           "ms_per_call_align_rounds": [1e3 * v / batches for v in times["on"]],
           "faces_per_frame": faces["on"] / (n_streams * batches),
           "d2h_bytes_per_frame": int(topk * per_face),
           "d2h_bytes_per_frame_align": int(topk * (per_face + size * size * 3 + 6 * 8)),
           "api": "FaceAnaStreams.submit/collect, pinned host frames, 2 calls in flight; align: chips warped in submit"}
    del fas
    if name == "4k_16faces":
        kps = np.stack([f["kps"] for faces_s in last for f in faces_s])
        out["align_kernel"] = time_align_kernel(torch, batch(batches - 1)[0], kps, size)
    return out


def build_parent_headpose(src, out_dir):
    """An earlier csrc/headpose.cu as a library of its own (skps_head_pose only) under out_dir."""
    import shutil
    import subprocess
    from peppa_pig_face_landmark_b200 import build
    os.makedirs(out_dir, exist_ok=True)
    cu = os.path.join(out_dir, "parent_headpose.cu")
    shutil.copyfile(src, cu)
    stub = os.path.join(out_dir, "parent_error_stub.cu")
    with open(stub, "w") as f:       # the error-string helpers live in engine.cu, which the side library leaves out
        f.write("namespace skps { void set_error(const char*, ...) {} const char* get_error() { return \"\"; } }\n")
    lib = os.path.join(out_dir, "libparent_headpose.so")
    subprocess.check_call([build._nvcc()] + build.ARCH + build.COMMON + build.SOURCES["headpose.cu"] +
                          ["-I", build.CSRC, "-shared", "-o", lib, cu, stub])
    return lib


def _bind_head_pose(path):
    import ctypes as C
    lib = C.CDLL(path)
    fn = lib.skps_head_pose
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 6
    return fn


def _head_pose(fn, pts, hw):
    from peppa_pig_face_landmark_b200.core.headpose.pose import object_pts, reprojectsrc
    n = pts.shape[0]
    out = {"rvec": np.zeros((n, 3)), "tvec": np.zeros((n, 3)), "euler": np.zeros((n, 3)), "reproject": np.zeros((n, 8, 2))}
    rc = fn(pts.ctypes.data, n, hw[1], hw[0], object_pts.ctypes.data, reprojectsrc.ctypes.data, out["rvec"].ctypes.data,
            out["tvec"].ctypes.data, out["euler"].ctypes.data, out["reproject"].ctypes.data)
    assert rc == 0, "skps_head_pose failed"
    return out


def time_pose_kernels(torch, parent_lib=None, sizes=(16, 256, 1024), iters=30):
    """Kernel time of the pose solver (and of the parent's, if given) per launch, from torch.profiler kernel records."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from peppa_pig_face_landmark_b200 import runtime as rt
    from peppa_pig_face_landmark_b200.core.headpose.pose import POSE_POINTS
    from test_headpose_gpu import _synthetic_shapes
    impls = {"head_pose_warp_kernel": _bind_head_pose(rt.LIB_PATH)}
    if parent_lib:
        impls["parent_head_pose_kernel"] = _bind_head_pose(parent_lib)
    hw = (1080, 1920)
    out = []
    for n in sizes:
        pts = np.ascontiguousarray(_synthetic_shapes(n, hw, seed=n)[:, POSE_POINTS], np.float32)
        row = {"faces": n}
        for name, fn in impls.items():
            for _ in range(3):
                _head_pose(fn, pts, hw)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(iters):
                    _head_pose(fn, pts, hw)
                torch.cuda.synchronize()
            us = [e.time_range.elapsed_us() for e in prof.events()
                  if e.device_type == DeviceType.CUDA and "head_pose" in e.name]
            assert len(us) == iters, (name, len(us))
            row[name + "_us"] = float(np.median(us))
            row[name + "_name"] = [e.name for e in prof.events() if "head_pose" in e.name][0]
        out.append(row)
    return {"pose_kernel": out, "timing": "torch.profiler CUDA kernel records, median of %d launches" % iters}


def parent_pose_diff(parent_lib):
    """Largest difference of this build's skps_head_pose from the parent's on test_headpose_gpu's inputs."""
    from peppa_pig_face_landmark_b200 import runtime as rt
    from peppa_pig_face_landmark_b200.core.headpose.pose import POSE_POINTS
    from test_headpose_gpu import _synthetic_shapes
    new, old = _bind_head_pose(rt.LIB_PATH), _bind_head_pose(parent_lib)
    d = {k: 0.0 for k in ("rvec", "tvec", "euler", "reproject")}
    for hw in [(480, 640), (1080, 1920)]:
        pts = np.ascontiguousarray(_synthetic_shapes(64, hw, seed=hw[0])[:, POSE_POINTS], np.float32)
        a, b = _head_pose(new, pts, hw), _head_pose(old, pts, hw)
        for k in d:
            d[k] = max(d[k], float(np.abs(a[k] - b[k]).max()))
    return {"max_abs_diff_from_parent": d, "inputs": "test_headpose_gpu._synthetic_shapes(64, hw, seed=hw[0]), 480x640 and 1080x1920"}


def run_detect_every_pair(name, every, det_input=None, n_streams=16, batches=12, rounds=5, length=6, single_calls=60):
    """FaceAnaStreams at detect_every 1 and `every` (alternating rounds, median ms_per_call and the mean detector batch of
    each), then FaceAna.run on stream 0's frames at both settings."""
    import torch
    import frames
    from Skps import FaceAna, FaceAnaStreams
    maker, topk = getattr(frames, CONFIGS[name][0]), CONFIGS[name][1]
    seqs = make_streams(torch, frames, maker, n_streams, length=length)
    H, W = seqs[0][0].shape[:2]
    kw = {} if det_input is None else {"det_input": det_input}
    fas = {1: FaceAnaStreams(n_streams=n_streams, top_k=topk, max_frame_hw=(H, W), detect_every=1, **kw),
           every: FaceAnaStreams(n_streams=n_streams, top_k=topk, max_frame_hw=(H, W), detect_every=every, **kw)}
    L = len(seqs[0])

    def batch(t):
        return [seqs[s][t % L] for s in range(n_streams)]
    for fa in fas.values():
        for t in range(every + 2):         # the first call (all streams) and every staggered batch size after it
            fa.run(batch(t))
    times = {k: [] for k in fas}
    det_frames = {k: [] for k in fas}
    for r in range(rounds):
        for key in (list(fas) if r % 2 == 0 else list(fas)[::-1]):
            fa = fas[key]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fa.submit(batch(0))
            for t in range(1, batches):
                fa.submit(batch(t))
                fa.collect()
                det_frames[key].append(fa.last_detector_frames)
            fa.collect()
            det_frames[key].append(fa.last_detector_frames)
            torch.cuda.synchronize()
            times[key].append(time.perf_counter() - t0)
    del fas
    singles = {k: FaceAna(top_k=topk, max_frame_hw=(H, W), detect_every=k, **kw) for k in (1, every)}
    for f in singles.values():
        for t in range(2 * every):
            f.run(seqs[0][t % L])
    single_times = {k: [] for k in singles}
    ran = {k: 0 for k in singles}
    for r in range(rounds):
        for key in (list(singles) if r % 2 == 0 else list(singles)[::-1]):
            f = singles[key]
            t0 = time.perf_counter()
            for t in range(single_calls):
                f.run(seqs[0][t % L])
                ran[key] += f.last_ran_detector
            single_times[key].append(time.perf_counter() - t0)
    del singles
    ms = {k: 1e3 * float(np.median(v)) / batches for k, v in times.items()}
    ms1 = {k: 1e3 * float(np.median(v)) / single_calls for k, v in single_times.items()}
    return {"config": name, "streams_per_gpu": n_streams, "calls": batches, "rounds": rounds, "detect_every": every,
            "det_input": list(det_input) if det_input is not None else [384, 640],
            "ms_per_call_every_1": ms[1], "ms_per_call_every_n": ms[every],
            "frames_per_s_every_1": 1e3 * n_streams / ms[1], "frames_per_s_every_n": 1e3 * n_streams / ms[every],
            "ms_per_call_every_1_rounds": [1e3 * v / batches for v in times[1]],
            "ms_per_call_every_n_rounds": [1e3 * v / batches for v in times[every]],
            "detector_frames_per_call_every_1": float(np.mean(det_frames[1])),
            "detector_frames_per_call_every_n": float(np.mean(det_frames[every])),
            "faceana_ms_per_run_every_1": ms1[1], "faceana_ms_per_run_every_n": ms1[every],
            "faceana_ms_per_run_every_1_rounds": [1e3 * v / single_calls for v in single_times[1]],
            "faceana_ms_per_run_every_n_rounds": [1e3 * v / single_calls for v in single_times[every]],
            "faceana_detector_share_every_1": ran[1] / (rounds * single_calls),
            "faceana_detector_share_every_n": ran[every] / (rounds * single_calls),
            "api": "FaceAnaStreams.submit/collect, pinned host frames, 2 calls in flight; FaceAna.run on stream 0's "
                   "frames (host results, synchronous)"}


def main():
    import torch
    a = sys.argv[1:]

    def opt(name, default):
        return a[a.index(name) + 1] if name in a else default
    n_streams, batches = int(opt("--streams", 16)), int(opt("--batches", 12))
    names = opt("--configs", ",".join(CONFIGS)).split(",")
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0"))))
    if "--pose" in a:
        rounds = int(opt("--rounds", 5))
        print(json.dumps(gpu_info(torch)))
        parent = None
        if "--parent-headpose" in a:
            parent = build_parent_headpose(opt("--parent-headpose", None), opt("--out", "bench_out"))
            print(json.dumps(parent_pose_diff(parent)))
        print(json.dumps(time_pose_kernels(torch, parent)))
        sys.stdout.flush()
        for name in names:
            print(json.dumps(run_align_pair(name, 0, n_streams, batches, rounds=rounds, feature="pose")))
            sys.stdout.flush()
        return
    if "--detect-every" in a:
        every, rounds = int(opt("--detect-every", 4)), int(opt("--rounds", 5))
        hw = None
        if "--det-input" in a:
            i = a.index("--det-input")
            hw = (int(a[i + 1]), int(a[i + 2]))
        print(json.dumps(gpu_info(torch)))
        for name in names:
            print(json.dumps(run_detect_every_pair(name, every, hw, n_streams, batches, rounds=rounds)))
            sys.stdout.flush()
        return
    if "--det-input" in a:
        i = a.index("--det-input")
        hw, rounds = (int(a[i + 1]), int(a[i + 2])), int(opt("--rounds", 5))
        print(json.dumps(gpu_info(torch)))
        for name in names:
            print(json.dumps(run_align_pair(name, hw, n_streams, batches, rounds=rounds, feature="det_input")))
            sys.stdout.flush()
        return
    if "--track-ids" in a:
        rounds = int(opt("--rounds", 5))
        print(json.dumps(gpu_info(torch)))
        for name in names:
            if "--id-memory" in a:
                r = run_align_pair(name, int(opt("--id-memory", 0)), n_streams, batches, rounds=rounds, feature="id_memory")
            else:
                r = run_align_pair(name, 0, n_streams, batches, rounds=rounds, feature="track_ids")
            print(json.dumps(r))
            sys.stdout.flush()
        return
    if "--align" in a:
        size, rounds = int(opt("--align", 112)), int(opt("--rounds", 5))
        print(json.dumps(gpu_info(torch)))
        for name in names:
            print(json.dumps(run_align_pair(name, size, n_streams, batches, rounds=rounds)))
            sys.stdout.flush()
        return
    for name in names:
        r = run_config(name, n_streams, batches, gather="--gather" in a, dist=dist, rank=rank, world=world)
        if r is not None:
            print(json.dumps(r))
            sys.stdout.flush()
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
