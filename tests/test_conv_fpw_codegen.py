"""The register-accumulator fused kernel (conv_fpw.cu) must keep its wgmma asynchronous and everything in registers: ptxas
reports C7520 / C7511 / C7512 when it serialises wgmma, C7507 when it ignores a setmaxnreg, and a stack frame with spill
stores when a role's code does not fit its registers.  Compiles the source as build.py does, for sm_90a, with -Xptxas -v
(no GPU needed), and checks every instantiation."""
import os
import re
import shutil
import subprocess

import pytest

from peppa_pig_face_landmark_b200 import build

_report = []


def _ptxas_report():
    if _report:
        return _report[0]
    nvcc = build._nvcc()
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    src = "conv_fpw.cu"
    cmd = [nvcc] + build.ARCH + build.COMMON + build.SOURCES[src] + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, src),
                                                                     "-o", os.devnull]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    _report.append(r.stdout)
    return r.stdout


def _spills():
    return re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads", _ptxas_report())


def test_conv_fpw_wgmma_not_serialized():
    out = _ptxas_report()
    for code in ("C7520", "C7511", "C7512", "C7507"):
        assert code not in out, out


def test_conv_fpw_instantiations_and_spills():
    kernels = [(name, int(st), int(ld)) for name, st, ld in _spills() if "conv_fpw_kernel" in name]
    # 2 modes x 2 unit widths x activations none / ReLU x split-fp16 / float32 output
    assert len(kernels) == 16, kernels
    scale = [k for k in kernels if "conv_fpw_kernelILi0E" in k[0]]
    dw = [k for k in kernels if "conv_fpw_kernelILi1E" in k[0]]
    assert len(scale) == 8 and len(dw) == 8
    bad = [k for k in kernels if k[1] or k[2]]
    assert not bad, bad
