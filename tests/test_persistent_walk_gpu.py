"""The persistent kernels with many work units per CTA.  conv_tc, conv_tct, conv_hm, conv_pw, conv_xf, conv_fpw and the stem
block launch min(units, SMs) CTAs (conv_mma SMs x its CTAs per SM), and each CTA walks units blockIdx.x, + gridDim.x, ...
A CTA's second and later units are where these kernels carry state across work: mbarrier ring phases, conv_pw's
alternating consumer warpgroups, epilogue staging buffers reused behind earlier TMA stores, the stem block's prefetch of
its next tile, conv_mma's double buffer.  At the batches of test_op_isolated_gpu.py most of the student's ops run one
unit per CTA, so its float64 checks never see that state.

skps_engine_set_num_sms caps the grids without touching any kernel.  A unit's K order and arithmetic depend only on its
index, and no conv kernel uses atomics, so every op's output must stay the same bit for bit under any cap: the capped
sweep of the op-isolated plans is checked against the uncapped one, which test_op_isolated_gpu.py checks against float64.
skps_engine_op_grid reports every launch's CTAs and units, so the sweep can show that the caps took effect and reached
several units per CTA in every persistent kernel.  And the student at the benchmark's batch of 256: every intermediate
buffer of three images among 256 must equal a batch-3 run of the same three images."""
import hashlib
import os
import sys
import time

import numpy as np
import pytest

from test_op_isolated_gpu import PLANS, _tag

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
STUDENT = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "kps_student.onnx")

CAPS = [1, 2, 3, 7]            # SMs the capped runs size their grids for (0: the device's count)
_SWEEPS = {}


def _bits(a):
    """The bits of a buffer as read back: uint8 stays, float32 is compared as uint32."""
    return a if a.dtype == np.uint8 else a.view(np.uint32)


def _digest(a):
    return hashlib.blake2b(np.ascontiguousarray(_bits(a)).tobytes(), digest_size=16).digest()


def _walk(ex, x_u8):
    """One forward, then every op re-run in plan order as op_report.check_ops does it.  -> per op: (digest of every
    buffer the op stores, (CTAs, units) of its launch)."""
    import op_report as R
    ex.forward(x_u8)
    out = []
    for i, op in enumerate(ex.plan.ops):
        ex.run_op(i)
        bufs = sorted({v.buf.idx for v in R._stored(op)})
        out.append((tuple(_digest(ex.eng.read_buffer(b, ex.batch)) for b in bufs), ex.op_grid(i)))
    return out


def _sweep(which, hw, batch):
    """{cap: _walk result} over 0 (uncapped) and CAPS on one engine, and each op's (kernel, info)."""
    key = _tag(which, hw)
    if key not in _SWEEPS:
        import op_report as R
        t0 = time.time()
        eng, x = R.make_engine(which, hw, batch)
        ex = R.EngineOps(eng, batch)
        kinds = [ex.op_kernel(i) for i in range(len(eng.plan.ops))]
        runs = {}
        try:
            for cap in [0] + CAPS:
                ex.set_num_sms(cap)
                runs[cap] = _walk(ex, x)
        finally:
            ex.set_num_sms(0)
        _SWEEPS[key] = (eng.plan, kinds, runs)
        del ex, eng
        print("%s: %d ops x %d grids in %.1f s" % (key, len(kinds), len(runs), time.time() - t0))
    return _SWEEPS[key]


@pytest.mark.parametrize("which,hw,batch", PLANS, ids=[_tag(w, h) for w, h, _ in PLANS])
def test_capped_grids_give_bit_identical_ops(which, hw, batch):
    """Every op's stored outputs under grids capped at 1, 2, 3 and 7 SMs equal the uncapped run's bit for bit."""
    import op_report as R
    plan, kinds, runs = _sweep(which, hw, batch)
    bad = []
    for cap in CAPS:
        for i, ((dig, (ctas, units)), (dig0, _)) in enumerate(zip(runs[cap], runs[0])):
            if dig != dig0:
                bad.append("cap %d: op %d %s kernel %s %s, %d units on %d CTAs" % (
                    cap, i, plan.ops[i].name, R.KERNELS[kinds[i][0]], kinds[i][1], units, ctas))
    assert not bad, "\n".join(bad)


def test_grid_query_and_cap_take_effect():
    """skps_engine_op_grid reports a launch for exactly the persistent ops; under a cap of c SMs every one launches
    min(units, c) CTAs (conv_mma: min(units, c x its CTAs per SM)), the units do not change, and cap 0 restores the
    uncapped grids."""
    import op_report as R
    for which, hw, batch in PLANS:
        plan, kinds, runs = _sweep(which, hw, batch)
        mma_per_sm = max([runs[1][i][1][0] for i, (k, _) in enumerate(kinds) if k == R.K_MMA] or [1])
        for i, (k, _) in enumerate(kinds):
            ctas0, units = runs[0][i][1]
            tag = "%s op %d %s" % (_tag(which, hw), i, R.KERNELS[k])
            if k not in R.PERSISTENT:
                assert all(runs[c][i][1] == (0, 0) for c in runs), (tag, [runs[c][i][1] for c in runs])
                continue
            assert 0 < ctas0 <= units, (tag, ctas0, units)
            for cap in CAPS:
                per = mma_per_sm if k == R.K_MMA else 1
                assert runs[cap][i][1] == (min(units, cap * per), units), (tag, cap, runs[cap][i][1], units)


def test_set_num_sms_rejects_counts_outside_the_device():
    import ctypes as C
    import torch
    from peppa_pig_face_landmark_b200 import ONNXEngine, runtime as rt
    lib = rt.load_library()
    eng = ONNXEngine(STUDENT, max_batch=2)
    sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
    assert lib.skps_engine_set_num_sms(eng.handle, -1) != 0
    assert lib.skps_engine_set_num_sms(eng.handle, sms + 1) != 0
    g = (C.c_int32 * 2)()
    rt.check(lib.skps_engine_op_grid(eng.handle, 0, 2, g))          # op 0: the stem block, 2 x 32 tiles
    assert tuple(g) == (64, 64), tuple(g)
    rt.check(lib.skps_engine_set_num_sms(eng.handle, sms))
    rt.check(lib.skps_engine_set_num_sms(eng.handle, 5))
    rt.check(lib.skps_engine_op_grid(eng.handle, 0, 2, g))
    assert tuple(g) == (5, 64), tuple(g)
    rt.check(lib.skps_engine_set_num_sms(eng.handle, 0))
    rt.check(lib.skps_engine_op_grid(eng.handle, 0, 2, g))
    assert tuple(g) == (64, 64), tuple(g)


def test_capped_sweep_walks_several_units_per_cta():
    """Over the capped sweep, every persistent kernel class has an op where some CTA walks at least 3 units, and conv_pw
    one where every CTA walks at least 4 with the last unit on warpgroup 0 on some CTAs and on warpgroup 1 on others
    (op_report.WALK_BRANCHES).  Prints the most units one CTA walks, per class, uncapped and per cap."""
    import op_report as R
    walks, table = [], {}
    for which, hw, batch in PLANS:
        _, kinds, runs = _sweep(which, hw, batch)
        for cap, run in runs.items():
            for i, (_, (ctas, units)) in enumerate(run):
                k = kinds[i][0]
                if k not in R.PERSISTENT:
                    continue
                most = max(R.units_per_cta(ctas, units))
                row = table.setdefault(R.PERSISTENT[k], {})
                row[cap] = max(row.get(cap, 0), most)
                if cap:
                    walks.append(("%s:%d@%d" % (_tag(which, hw), i, cap), k, ctas, units))
    print("most units per CTA   uncapped  " + "  ".join("cap %d" % c for c in CAPS))
    for cls, row in sorted(table.items()):
        print("  %-18s %8d  " % (cls, row[0]) + "  ".join("%5d" % row[c] for c in CAPS))
    cov = R.walk_coverage(walks)
    for b in R.WALK_BRANCHES:
        print("  %-52s %4d launches  e.g. %s" % (b, len(cov[b]), ", ".join(cov[b][:3])))
    missing = [b for b in R.WALK_BRANCHES if not cov[b]]
    assert not missing, missing


def test_student_batch256_every_buffer_matches_batch3():
    """The student at the benchmark's batch, 256 (about 62 pixel tiles per CTA on its 64 x 64 layers): the three
    op_report.crop_inputs images at positions 0, 129 and 255 among noise crops.  After one forward every intermediate
    buffer at those positions must equal, bit for bit, a batch-3 forward of the three images.  Extends
    test_student_batch256_invariance from the final outputs to every layer."""
    import frames
    import op_report as R
    from peppa_pig_face_landmark_b200 import ONNXEngine
    pos = [0, 129, 255]
    three = R.crop_inputs(3)
    x = frames.noise_crops(256, seed=7)
    x[pos] = three
    big = ONNXEngine(STUDENT, max_batch=256)
    big.run_u8(x)
    small = ONNXEngine(STUDENT, max_batch=3)
    small.run_u8(three)
    ex = R.EngineOps(big, 256)
    most = {}
    for i in range(len(big.plan.ops)):
        k, _ = ex.op_kernel(i)
        if k in R.PERSISTENT:
            ctas, units = ex.op_grid(i)
            most[R.PERSISTENT[k]] = max(most.get(R.PERSISTENT[k], 0), max(R.units_per_cta(ctas, units)))
    print("batch 256, most units per CTA: " + ", ".join("%s %d" % kv for kv in sorted(most.items())))
    n = big.lib.skps_engine_num_buffers(big.handle)
    bad = []
    for b in range(n):
        got = big.read_buffer(b, 256)[pos]          # one buffer at a time: a whole one can take a gigabyte on the host
        ref = small.read_buffer(b, 3)
        if not np.array_equal(_bits(got), _bits(ref)):
            diff = (_bits(got) != _bits(ref)).reshape(3, -1).any(1)
            bad.append("buffer %d %s: positions %s differ" % (b, ref.shape[1:], [p for p, d in zip(pos, diff) if d]))
        del got, ref
    assert not bad, "\n".join(bad)
