"""The detector's lowering over its input-size range (check_detector_input), without a GPU: every size of the axis sample
op_report.detector_domain_sample() lowers, and the plans it gives have exactly the known structures (op_report.
plan_structure: the sequence of op types and flags).  tests/test_detector_domain_gpu.py checks every structure and kernel
tiling of the same sample against float64 on the GPU; a lowering change that adds a structure fails here first."""
import collections
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

# one representative input size per plan structure, with its op count (the test prints every sampled size of each): most
# of the range lowers to 89 ops; narrow or short inputs, whose stride-32 maps are a few pixels across, to 92 or 99
STRUCTURES = {(384, 640): 89, (384, 256): 92, (224, 640): 92, (128, 128): 99, (128, 160): 99}


def test_every_sampled_size_lowers_to_a_known_plan_structure(tmp_path):
    import op_report as R
    sizes = R.detector_domain_sample()
    lowered = list(R.lower_detector_domain(sizes + sorted(STRUCTURES), str(tmp_path)))
    assert not os.listdir(tmp_path)
    pinned = {hw: st for hw, _, st in lowered if hw in STRUCTURES}
    assert {hw: len(st) for hw, st in pinned.items()} == STRUCTURES
    assert len(set(pinned.values())) == len(STRUCTURES), "two pinned sizes share a plan structure"
    groups = collections.defaultdict(list)
    for hw, _, st in lowered[:len(sizes)]:
        groups[st].append(hw)
    print("%d sizes, %d plan structures" % (len(sizes), len(groups)))
    for hw, st in sorted(pinned.items()):
        print("  %3d ops at %-10s %3d sizes: %s" % (len(st), "%dx%d" % hw, len(groups.get(st, [])),
                                                   " ".join("%dx%d" % s for s in groups.get(st, []))))
    unknown = {len(st): hws[:8] for st, hws in groups.items() if st not in set(pinned.values())}
    assert not unknown, "plan structures no pinned size has (op count: sizes): %s" % unknown
    assert set(groups) == set(pinned.values()), "a pinned structure no longer occurs in the sample"
