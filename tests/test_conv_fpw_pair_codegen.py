"""conv_fpw_pair (csrc/conv_fpw.cu), the paired-unit kernel of the decoder's up-sample layers, as ptxas compiles it for
sm_90a (no GPU needed): one instantiation per activation (none / ReLU) and output format (split fp16 / float32), none
with its wgmma serialised (the C75xx warnings are checked over the whole file by test_conv_fpw_codegen.py).

Its 640 threads leave ptxas 96 registers per thread for every role, setmaxnreg notwithstanding, which is less than the
transform warps and the 64-accumulator MMA warpgroups take without spilling.  The spills are a few loop-invariant values
and epilogue temporaries; this test keeps them from growing."""
import re

from test_conv_fpw_codegen import _ptxas_report

SPILL_STORES_MAX = 192          # bytes per instantiation; 88-184 as committed


def _pair_kernels():
    return re.findall(r"Function properties for (\S*conv_fpw_pair\S*)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads\s*\n[^\n]*Used (\d+) registers", _ptxas_report())


def test_conv_fpw_pair_instantiations():
    kernels = _pair_kernels()
    assert len(kernels) == 4, kernels
    assert not any("conv_fpw_kernel" in k[0] for k in kernels)
    for name, st, ld, regs in kernels:
        assert int(regs) <= 96, (name, regs)
        assert int(st) <= SPILL_STORES_MAX, (name, st, ld)
