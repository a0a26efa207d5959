"""Time of the student's fused stem block (op 0, csrc/stem_block.cu) at batch 256, against the HBM and FP32 bounds:
python tools/bench_stem.py [--batch B] [--reps N] [--json PATH]

Builds Student@256, runs one forward on noise crops, then launches the stem block alone (skps_engine_run_op on the buffers
the forward left) and takes the median and spread over N launches of CUDA-event times.

Bounds: the op's algorithmic HBM bytes (plan.bytes_per_sample: the uint8 crop read once, the E-channel quarter-resolution
output written once) against the data-sheet 3.35 TB/s; and the FP32 FMAs the kernel runs on the CUDA cores per 8 x 16
output tile, counted from its windows (the stem over 19 x 35 half-resolution pixels, the block-0 depthwise and 16->16
pointwise over 17 x 33, the stride-2 depthwise over the 8 x 16 tile), against SMs x 128 FMA/clk at the card's max SM clock.
The 16->E expansion runs on the tensor cores and is left out of the FP32 count."""
import argparse
import ctypes as C
import json
import os
import re
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_pw import HBM_BPS, card  # noqa: E402

TH, TW = 8, 16                                   # output tile (quarter resolution)
EH, EW = 2 * TH + 1, 2 * TW + 1                  # 17 x 33 half-resolution window of the stride-2 depthwise
SH, SW = EH + 2, EW + 2                          # 19 x 35 stem outputs the block-0 depthwise reads


def fp32_fmas_per_tile(E):
    stem = SH * SW * 16 * 27
    dw0 = EH * EW * 16 * 9
    pw0 = EH * EW * 16 * 16
    dw1 = TH * TW * E * 9
    return {"stem": stem, "dw0": dw0, "pw0": pw0, "dw_s2": dw1, "total": stem + dw0 + pw0 + dw1}


def max_sm_clock_hz(card_line):
    m = re.search(r"(\d+)\s*MHz\s*$", card_line)
    return float(m.group(1)) * 1e6 if m else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    args = ap.parse_args()
    import numpy as np
    import torch
    import frames
    from peppa_pig_face_landmark_b200 import ONNXEngine, plan as P, runtime as rt
    B = args.batch
    eng = ONNXEngine(os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "kps_student.onnx"), max_batch=B)
    lib = rt.load_library()
    s = eng.stream
    ops = [i for i, op in enumerate(eng.plan.ops) if op.type == P.OP_STEM_BLOCK]
    if not ops:
        raise SystemExit("the plan has no stem block op")
    i = ops[0]
    op = eng.plan.ops[i]
    x = torch.from_numpy(frames.noise_crops(B, seed=100)).cuda()
    outs = [torch.empty((B, e), dtype=torch.float32, device="cuda") for e in eng.out_elems]
    with torch.cuda.stream(s):
        eng.forward_device(x, outs, s)
    torch.cuda.synchronize()
    ts = []
    with torch.cuda.stream(s):
        for _ in range(10):
            rt.check(lib.skps_engine_run_op(eng.handle, i, B, s.cuda_stream))
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rt.check(lib.skps_engine_run_op(eng.handle, i, B, s.cuda_stream))
            e1.record()
            ts.append((e0, e1))
    torch.cuda.synchronize()
    ms = np.array([a.elapsed_time(b) for a, b in ts])
    grid = (C.c_int32 * 2)()
    rt.check(lib.skps_engine_op_grid(eng.handle, i, B, grid))
    ctas, tiles = grid[0], grid[1]
    E = op.outs[0].C
    fmas = fp32_fmas_per_tile(E)
    line = card()
    clk = max_sm_clock_hz(line)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nbytes = eng.plan.bytes_per_sample(op) * B
    med = float(np.median(ms))
    hbm_ms = nbytes / HBM_BPS * 1e3
    fp32_ms = tiles * fmas["total"] / (sms * 128 * clk) * 1e3 if clk else None
    res = {"card": line, "batch": B, "op": i, "ctas": ctas, "tiles": tiles, "reps": args.reps,
           "ms_median": med, "ms_min": float(ms.min()), "ms_p10": float(np.percentile(ms, 10)),
           "ms_p90": float(np.percentile(ms, 90)), "us_per_tile_per_cta": med * 1e3 * ctas / tiles,
           "hbm_bytes": nbytes, "hbm_bound_ms": hbm_ms, "fp32_fmas_per_tile": fmas,
           "fp32_bound_ms": fp32_ms, "sms": sms, "max_sm_clock_hz": clk}
    print("card: %s" % line)
    print("op %d stem block, batch %d: %d tiles of %dx%d on %d CTAs (%.1f tiles each)" % (
        i, B, tiles, TH, TW, ctas, tiles / ctas))
    print("median %.3f ms over %d launches (min %.3f, p10 %.3f, p90 %.3f); %.2f us per tile per CTA" % (
        med, args.reps, res["ms_min"], res["ms_p10"], res["ms_p90"], res["us_per_tile_per_cta"]))
    print("HBM: %.1f MB algorithmic, bound %.3f ms at 3.35 TB/s (%.1f%% reached)" % (
        nbytes / 1e6, hbm_ms, 100 * hbm_ms / med))
    if fp32_ms:
        print("FP32: %d FMAs per tile (stem %d, dw0 %d, pw0 %d, dw s2 %d), bound %.3f ms at %d SMs x 128 FMA/clk x %.2f GHz"
              " (%.1f%% reached)" % (fmas["total"], fmas["stem"], fmas["dw0"], fmas["pw0"], fmas["dw_s2"], fp32_ms, sms,
                                     clk / 1e9, 100 * fp32_ms / med))
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
