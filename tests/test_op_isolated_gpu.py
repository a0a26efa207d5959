"""Every engine op against float64 on its own inputs (tools/op_report.py): the detector at its default size and at the
input sizes whose ragged maps reach the edge-tile branches of the tensor-core and TMA kernels, the student and the
Teacher.  Batch 3 (2 for the Teacher): odd, so multi-image tiles get a partial last tile.  The batch is a letterboxed
real frame, uint8 noise and a near-uniform grey frame.  Each op must stay within its element-wise bound, the sweep as
a whole must run every branch in op_report.BRANCHES, and the comparator must reject an error of 8x the bound planted
in one edge-tile element of a host copy of real kernel output."""
import os
import sys
import time

import pytest

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

DET_SIZES = [(384, 640), (128, 128), (416, 736), (480, 864), (160, 3840), (2176, 128), (224, 288)]
PLANS = [("detector", hw, 3) for hw in DET_SIZES] + [("student", None, 3), ("teacher", None, 2)]
_CACHE = {}


def _tag(which, hw):
    return which if hw is None else "%s@%dx%d" % (which, hw[0], hw[1])


def _keep(r):
    """Per-op tensors kept for the planted-error test: ragged conv_tc ops and dw_tma ops."""
    import op_report as R
    from peppa_pig_face_landmark_b200 import plan as P
    if r.kernel == R.K_TC and r.info[2] == 1:
        o = r.op.outs[0]
        return bool(o.W % r.info[0] or o.H % r.info[1]) and not (r.op.flags & P.FLAG_HM_PART)
    return r.kernel == R.K_DW_TMA


def _results(which, hw, batch):
    key = _tag(which, hw)
    if key not in _CACHE:
        import op_report as R
        t0 = time.time()
        eng, x = R.make_engine(which, hw, batch)
        res, detail = R.check_engine(eng, x, keep=_keep if which == "detector" and hw == (416, 736) else None)
        del eng
        _CACHE[key] = (res, detail)
        print("%s: %d ops in %.1f s" % (key, len(res), time.time() - t0))
    return _CACHE[key]


@pytest.mark.parametrize("which,hw,batch", PLANS, ids=[_tag(w, h) for w, h, _ in PLANS])
def test_every_op_within_its_bound(which, hw, batch):
    import op_report as R
    res, _ = _results(which, hw, batch)
    for k, v in sorted(R.worst_per_class(res).items()):
        print("  %-18s worst err/bound %.3e" % (k, v))
    bad = ["%s kernel %s %s worst (n,y,x,c)=%s edge tile=%s ratio %.3e" % (
        r.name, R.KERNELS[r.kernel], r.info, r.where, r.edge, r.ratio) for r in res if not r.ok]
    assert not bad, "\n".join(bad)


def test_sweep_covers_the_edge_tile_branches():
    """The plans above must together execute every branch in op_report.BRANCHES (kernel and tiling as the engine reports
    them, skps_engine_op_kernel): a change to lowering or tiling that moves the sweep off a branch fails here."""
    import op_report as R
    tagged = []
    for which, hw, batch in PLANS:
        tagged += [(_tag(which, hw), r) for r in _results(which, hw, batch)[0]]
    cov = R.coverage(tagged)
    for b in R.BRANCHES:
        print("  %-26s %3d ops  e.g. %s" % (b, len(cov[b]), ", ".join(cov[b][:3])))
    missing = [b for b in R.BRANCHES if not cov[b]]
    assert not missing, missing


def test_checker_rejects_an_error_planted_in_an_edge_tile():
    """On a host copy of what the kernel wrote: 8x the element's bound added to one element of the last (edge) tile of a
    ragged conv_tc op and of a dw_tma op must fail the comparison; the unmodified copy passes."""
    import op_report as R
    res, detail = _results("detector", (416, 736), 3)
    picked = {}
    for r in res:
        if r.index in detail:
            picked.setdefault("tc" if r.kernel == R.K_TC else "dw_tma", []).append(r)
    assert set(picked) == {"tc", "dw_tma"}, picked.keys()
    for kind, rs in picked.items():
        # prefer an op whose last tile hangs over both borders
        r = max(rs, key=lambda r: (R.edge_tile(r.kernel, r.info, r.op.outs[0].H, r.op.outs[0].W,
                                               r.op.outs[0].H - 1, r.op.outs[0].W - 1), r.index))
        got, rows = detail[r.index]
        o = rows[0][0]
        where = (r.batch - 1, o.H - 1, o.W - 1, o.C - 1)           # last image, last pixel, last channel
        assert R.edge_tile(r.kernel, r.info, o.H, o.W, where[1], where[2]), (kind, r.info, o.H, o.W)
        assert R._worst([rows[0][:3]], {k: R._to64(x, o.buf) if k == o.buf.idx else x for k, x in got.items()})[0] <= 1
        planted = R.planted_ratio(r.op, got, rows, 0, where)
        print("%s op %d %s: planted error reported at %.2f x the bound" % (kind, r.index, r.info, planted))
        assert planted > 1.0
