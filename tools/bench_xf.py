"""Per-layer time of the student's fused producer -> 1x1 layers (depthwise -> 1x1, up-sample + concat + depthwise -> 1x1,
squeeze-excite scale -> 1x1) at batch 256:
python tools/bench_xf.py [--batch B] [--reps N] [--json PATH]

Builds Student@256, runs one forward on noise crops, then launches each OP_DWPW and each OP_CONV with FLAG_XF alone
(skps_engine_run_op on the buffers the forward left) and takes the median over N launches of CUDA-event times.  The layers
are picked from the plan's shapes, not from the kernel the engine chose, so the same table comes out of any version of
the engine.  Bytes are the algorithmic ones (plan.bytes_per_sample x B: every input read once, the output written once),
set against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.  FLOP are the three-product fp16 ones the precision
scheme needs (3 x 2 x pixels x K x Cout, K = the 1x1 conv's input channels), set against the data-sheet dense fp16 rate of
989 TFLOP/s.  The depthwise stage's CUDA-core work is not counted."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BPS = 3.35e12
TC_FLOPS = 989e12


def card():
    """Name, power limit and max SM clock of GPU 0, read now."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        import torch
        return torch.cuda.get_device_name(0) + ", power limit not read"


def fused_ops(plan):
    from peppa_pig_face_landmark_b200 import plan as P
    return [i for i, op in enumerate(plan.ops)
            if op.type == P.OP_DWPW or (op.type == P.OP_CONV and op.flags & P.FLAG_XF)]


def gemm_k(op):
    """Input channels of the layer's 1x1 conv: the up-sampled low-res channels (third input of a DWPW op) plus x's."""
    k = op.ins[0].C
    if len(op.ins) > 2 and op.ins[2] is not None and op.ins[2].buf.H * 2 == op.outs[0].buf.H:
        k += op.ins[2].C
    return k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this path")
    args = ap.parse_args()
    import numpy as np
    import torch
    import frames
    from peppa_pig_face_landmark_b200 import ONNXEngine, plan as P, runtime as rt
    B = args.batch
    eng = ONNXEngine(os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "kps_student.onnx"), max_batch=B)
    lib = rt.load_library()
    s = eng.stream
    x = torch.from_numpy(frames.noise_crops(B, seed=100)).cuda()
    outs = [torch.empty((B, e), dtype=torch.float32, device="cuda") for e in eng.out_elems]
    with torch.cuda.stream(s):
        eng.forward_device(x, outs, s)
    torch.cuda.synchronize()
    info = (C.c_int32 * 4)()
    rows = []
    for i in fused_ops(eng.plan):
        op = eng.plan.ops[i]
        ts = []
        with torch.cuda.stream(s):
            for _ in range(3):
                rt.check(lib.skps_engine_run_op(eng.handle, i, B, s.cuda_stream))
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                rt.check(lib.skps_engine_run_op(eng.handle, i, B, s.cuda_stream))
                e1.record()
                ts.append((e0, e1))
        torch.cuda.synchronize()
        us = float(np.median([a.elapsed_time(b) for a, b in ts])) * 1e3
        o = op.outs[0]
        nbytes = eng.plan.bytes_per_sample(op) * B
        k = gemm_k(op)
        flop = 3 * 2 * B * o.buf.H * o.buf.W * k * o.C
        kernel = lib.skps_engine_op_kernel(eng.handle, i, info)
        rows.append({"op": i, "mode": "dw" if op.type == P.OP_DWPW else "scale", "k": k, "cout": o.C,
                     "map": "%dx%d" % (o.buf.H, o.buf.W), "us": us, "bytes": nbytes, "flop": flop,
                     "frac_hbm": nbytes / (us * 1e-6) / HBM_BPS, "frac_tc": flop / (us * 1e-6) / TC_FLOPS,
                     "kernel": kernel, "info": list(info)})
    total = sum(r["us"] for r in rows)
    nb = sum(r["bytes"] for r in rows)
    nf = sum(r["flop"] for r in rows)
    print("card: %s" % card())
    print("%4s %6s %10s %8s %9s %9s %8s %7s %7s %6s" % ("op", "mode", "K->Cout", "map", "us", "MB", "GFLOP", "HBM", "TC",
                                                       "kernel"))
    for r in rows:
        print("%4d %6s %10s %8s %9.1f %9.1f %8.1f %6.1f%% %6.1f%% %6d" % (
            r["op"], r["mode"], "%d->%d" % (r["k"], r["cout"]), r["map"], r["us"], r["bytes"] / 1e6, r["flop"] / 1e9,
            100 * r["frac_hbm"], 100 * r["frac_tc"], r["kernel"]))
    print("%d layers: %.1f us, %.1f MB (%.1f%% of 3.35 TB/s), %.1f GFLOP (%.1f%% of 989 TFLOP/s); HBM bound %.1f us, "
          "tensor bound %.1f us" % (len(rows), total, nb / 1e6, 100 * nb / (total * 1e-6) / HBM_BPS, nf / 1e9,
                                    100 * nf / (total * 1e-6) / TC_FLOPS, nb / HBM_BPS * 1e6, nf / TC_FLOPS * 1e6))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "batch": B, "rows": rows, "total_us": total}, f, indent=1)


if __name__ == "__main__":
    main()
