"""The pointwise wgmma kernel (conv_pw.cu) must keep its wgmma asynchronous and its accumulators in registers: ptxas
reports C7520 when it serialises wgmma, and a stack frame with spill stores when the accumulator does not fit.  Compiles the
source as build.py does, for sm_90a, with -Xptxas -v (no GPU needed), and checks every instantiation."""
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
    src = "conv_pw.cu"
    cmd = [nvcc] + build.ARCH + build.COMMON + build.SOURCES[src] + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, src),
                                                                     "-o", os.devnull]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    _report.append(r.stdout)
    return r.stdout


def test_conv_pw_wgmma_not_serialized():
    out = _ptxas_report()
    assert "C7520" not in out, out


def test_conv_pw_does_not_spill():
    out = _ptxas_report()
    spills = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", out)
    kernels = [name for name, _, _ in spills if "conv_pw_kernel" in name]
    # chunk widths 32, 64, 96, 128 x activations none, ReLU, h-swish x split-fp16 / float32 output
    assert len(kernels) == 24, kernels
    bad = [(name, st, ld) for name, st, ld in spills if st != "0" or ld != "0"]
    assert not bad, bad
