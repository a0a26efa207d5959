"""The head-pose solver keeps its scratch in shared memory and registers: every kernel of csrc/headpose.cu compiles for
sm_90a without spilling (the one-thread-per-face solver it replaced spilled 1948 bytes per thread).  No GPU needed."""
import re

from test_wgmma_codegen import _ptxas_report


def test_headpose_kernels_do_not_spill():
    out = _ptxas_report("headpose.cu")
    spills = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", out)
    assert any("head_pose" in name for name, _, _ in spills), out
    bad = [(name, st, ld) for name, st, ld in spills if st != "0" or ld != "0"]
    assert not bad, bad
