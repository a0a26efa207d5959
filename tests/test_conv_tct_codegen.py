"""The transposed convolution kernel (conv_tct.cu) must keep its wgmma asynchronous, its accumulators in registers and its
shared memory inside what an H100 CTA can have: ptxas reports C7510 / C7511 / C7512 / C7520 when it serialises wgmma and a
stack frame with spill stores when the code does not fit its registers, and the halo and weight rings are sized on the host
against TCT_SMEM_LIMIT, which with the kernel's static shared memory has to stay within 227 KB.  Compiles the source as
build.py does, for sm_90a, with -Xptxas -v (no GPU needed), and checks every instantiation."""
import os
import re
import shutil
import subprocess

import pytest

from peppa_pig_face_landmark_b200 import build

SRC = "conv_tct.cu"
_report = []


def _ptxas_report():
    if _report:
        return _report[0]
    nvcc = build._nvcc()
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    cmd = [nvcc] + build.ARCH + build.COMMON + build.SOURCES[SRC] + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, SRC),
                                                                     "-o", os.devnull]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    _report.append(r.stdout)
    return r.stdout


def _kernels():
    """(name, spill stores, spill loads, static shared memory) of every conv_tct_kernel instantiation."""
    found = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads\s*\n[^\n]*Used \d+ registers[^\n]*?(\d+) bytes smem", _ptxas_report())
    return [(n, int(st), int(ld), int(sm)) for n, st, ld, sm in found if "conv_tct_kernel" in n]


def test_conv_tct_wgmma_not_serialized():
    out = _ptxas_report()
    for code in ("C7510", "C7511", "C7512", "C7520"):
        assert code not in out, out


def test_conv_tct_instantiations_do_not_spill():
    kernels = _kernels()
    assert len(kernels) == 5, kernels                # activations none / ReLU / h-swish / sigmoid / hard-sigmoid
    bad = [k for k in kernels if k[1] or k[2]]
    assert not bad, bad


def test_conv_tct_shared_memory_fits_the_cta():
    with open(os.path.join(build.CSRC, SRC)) as f:
        m = re.search(r"constexpr int TCT_SMEM_LIMIT = 227 \* 1024 - (\d+);", f.read())
    assert m, "TCT_SMEM_LIMIT not found"
    dynamic_limit = 227 * 1024 - int(m.group(1))
    for name, _, _, static in _kernels():
        assert static > 0, name                      # the mbarriers of the two rings
        assert dynamic_limit + static <= 227 * 1024, (name, static)
