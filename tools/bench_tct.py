"""Per-layer time of the student's dense k x k and heat-map convolutions at batch 256, against the tensor, HBM and
shared-memory-fill rates:
python tools/bench_tct.py [--batch B] [--reps N] [--json PATH]

Builds Student@256, runs one forward on noise crops, then launches each chosen OP_CONV alone (skps_engine_run_op on the
buffers the forward left) and takes the median over N launches of CUDA-event times.  The layers are picked from the plan's
shapes, not from the kernel the engine chose: every stride-1 tensor-core conv with a 3x3 or larger window (the decoder conv
that conv_tct.cu runs, the ASPP convs of conv_tc.cu) and the heat-map head (conv_hm.cu).

Per layer: ms; algorithmic FLOP/s (2 x MACs) against the three-product ceiling, 989 / 3 TFLOP/s (H100 SXM data sheet, dense
fp16, one third because every K-step is three MMAs); algorithmic HBM bytes (input read once, output written once) against
the data-sheet 3.35 TB/s; and the bytes the kernel's TMA loads bring from L2 into shared memory per launch, computed below
from the staging constants of the kernel the engine reports, with the rate that makes."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_pw import HBM_BPS, card  # noqa: E402

SPLIT_CEILING = 989e12 / 3
K_TC, K_TCT, K_HM = 1, 2, 3
KERNEL_NAMES = {K_TC: "tc", K_TCT: "tct", K_HM: "hm"}


def dense_ops(plan):
    from peppa_pig_face_landmark_b200 import plan as P
    return [i for i, op in enumerate(plan.ops)
            if op.type == P.OP_CONV and op.flags & P.FLAG_TC and not op.flags & P.FLAG_XF and tuple(op.s) == (1, 1)
            and (op.k[0] >= 3 or op.flags & P.FLAG_HM_PART)]


def fill_bytes(kernel, info, op, batch, grid_ctas):
    """Bytes one launch loads into shared memory through TMA, from the staging of csrc/conv_tct.cu, conv_hm.cu and
    conv_tc.cu.  None for any other kernel."""
    from peppa_pig_face_landmark_b200 import plan as P
    cin, cout, H, W = op.ins[0].C, op.outs[0].C, op.outs[0].H, op.outs[0].W
    kh, kw, dil = op.k[0], op.k[1], op.d[0]
    if kernel == K_TCT:
        # per 256-pixel tile and (kx, 32-channel half-chunk): one halo slot of bh + dil (kh - 1) rows x W pixels x 64 B,
        # hi and lo, and kh weight slices of 128 rows x 64 B, hi and lo
        bh, halves = info[0], -(-cin // 32)
        tiles = batch * H * W // 256
        return tiles * kw * halves * (2 * (bh + dil * (kh - 1)) * W * 64 + kh * 2 * 128 * 64)
    if kernel == K_HM:
        # the weights once per CTA; per 256-pixel tile and 64-channel chunk 256 pixel rows x 128 B, hi and lo
        cchunks = -(-cin // 64)
        return grid_ctas * cchunks * 2 * 128 * 128 + (batch * H * W // 256) * cchunks * 2 * 256 * 128
    if kernel == K_TC:
        # per work item (mt pixel tiles of 128 x one weight tile) and (tap, 64-channel chunk): mt activation tiles of
        # 128 pixel rows x 128 B and one weight tile of n_tile rows x 128 B, hi and lo each
        mt = max(1, info[3])
        n_tile, n_tiles = P.tc_tiling(cout)
        items = -(-(batch * H * W // 128) // mt) * n_tiles
        return items * kh * kw * -(-cin // 64) * 2 * 128 * (mt * 128 + n_tile)
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this path")
    args = ap.parse_args()
    import numpy as np
    import torch
    import frames
    from peppa_pig_face_landmark_b200 import ONNXEngine, runtime as rt
    B = args.batch
    eng = ONNXEngine(os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "kps_student.onnx"), max_batch=B)
    lib = rt.load_library()
    s = eng.stream
    x = torch.from_numpy(frames.noise_crops(B, seed=100)).cuda()
    outs = [torch.empty((B, e), dtype=torch.float32, device="cuda") for e in eng.out_elems]
    with torch.cuda.stream(s):
        eng.forward_device(x, outs, s)
    torch.cuda.synchronize()
    info, grid = (C.c_int32 * 4)(), (C.c_int32 * 2)()
    rows = []
    for i in dense_ops(eng.plan):
        op = eng.plan.ops[i]
        ts = []
        with torch.cuda.stream(s):
            for _ in range(5):
                rt.check(lib.skps_engine_run_op(eng.handle, i, B, s.cuda_stream))
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                rt.check(lib.skps_engine_run_op(eng.handle, i, B, s.cuda_stream))
                e1.record()
                ts.append((e0, e1))
        torch.cuda.synchronize()
        sec = float(np.median([a.elapsed_time(b) for a, b in ts])) * 1e-3
        kernel = lib.skps_engine_op_kernel(eng.handle, i, info)
        rt.check(lib.skps_engine_op_grid(eng.handle, i, B, grid))
        flop = 2.0 * op.outs[0].C * op.outs[0].H * op.outs[0].W * op.ins[0].C * op.k[0] * op.k[1] * B
        nbytes = eng.plan.bytes_per_sample(op) * B
        fill = fill_bytes(kernel, list(info), op, B, grid[0])
        rows.append({"op": i, "name": op.name, "k": op.k[0], "dil": op.d[0], "cin": op.ins[0].C, "cout": op.outs[0].C,
                     "map": "%dx%d" % (op.outs[0].H, op.outs[0].W), "kernel": KERNEL_NAMES.get(kernel, str(kernel)),
                     "ms": sec * 1e3, "tflops": flop / sec / 1e12, "frac_split_ceiling": flop / sec / SPLIT_CEILING,
                     "hbm_bytes": nbytes, "frac_hbm": nbytes / sec / HBM_BPS,
                     "fill_bytes": fill, "fill_tbs": fill / sec / 1e12 if fill else None})
    print("card: %s" % card())
    print("%4s %4s %3s %10s %8s %8s %8s %7s %9s %6s %9s %8s" % ("op", "kern", "k/d", "Cin->Cout", "map", "ms", "TFLOP/s",
                                                             "of 330", "HBM MB", "HBM", "fill MB", "fill TB/s"))
    for r in rows:
        print("%4d %4s %3s %10s %8s %8.3f %8.1f %6.1f%% %9.1f %5.1f%% %9s %8s" % (
            r["op"], r["kernel"], "%d/%d" % (r["k"], r["dil"]), "%d->%d" % (r["cin"], r["cout"]), r["map"], r["ms"],
            r["tflops"], 100 * r["frac_split_ceiling"], r["hbm_bytes"] / 1e6, 100 * r["frac_hbm"],
            "%.1f" % (r["fill_bytes"] / 1e6) if r["fill_bytes"] else "-", "%.2f" % r["fill_tbs"] if r["fill_tbs"] else "-"))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "batch": B, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
