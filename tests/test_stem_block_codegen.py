"""What ptxas makes of the fused stem block (csrc/stem_block.cu), compiled as build.py does for sm_90a with -Xptxas -v (no
GPU needed): its wgmma stays asynchronous and is not diagnosed as in-warpgroup dependent, its registers fit the 576-thread
launch at one CTA per SM, its shared memory fits the 227 KB an H100 CTA may opt into, and its spills stay within a small
stated cap (a few per-tile scalars at the register limit the launch bounds impose)."""
import os
import re
import shutil
import subprocess

import pytest

from peppa_pig_face_landmark_b200 import build

THREADS = 576                       # SB_THREADS
SMEM_LIMIT = 227 * 1024             # cudaFuncAttributeMaxDynamicSharedMemorySize on sm_90
SPILL_CAP = 32                      # bytes of spill stores / loads allowed per kernel
_report = []


def _ptxas():
    if _report:
        return _report[0]
    nvcc = build._nvcc()
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    cmd = [nvcc] + build.ARCH + build.COMMON + build.SOURCES["stem_block.cu"] + [
        "-Xptxas", "-v", "-c", os.path.join(build.CSRC, "stem_block.cu"), "-o", os.devnull]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    _report.append(r.stdout)
    return r.stdout


def _kernel_props():
    """[(name, stack, spill stores, spill loads, registers, static smem)] of every stem block kernel."""
    out = _ptxas()
    props = re.findall(r"Function properties for (\S*stem_block_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                       r"stores, (\d+) bytes spill loads\s*\n.*?Used (\d+) registers.*?(\d+) bytes smem", out)
    assert props, out
    return [(n, int(a), int(b), int(c), int(d), int(e)) for n, a, b, c, d, e in props]


def _dynamic_smem():
    """SB_SMEM as the source computes it, evaluated from its constants."""
    src = open(os.path.join(build.CSRC, "stem_block.cu")).read()
    hdr = open(os.path.join(build.CSRC, "stem_block.h")).read()
    env = {"max": max, "min": min}
    exec("SB_MAX_E = %s" % re.search(r"constexpr int SB_MAX_E = (\d+);", hdr).group(1), env)
    for line in re.findall(r"^constexpr int (SB_\w+ = [^;]+(?:, SB_\w+ = [^;]+)*);", src, re.M):
        for part in re.split(r",\s*(?=SB_\w+ =)", line):
            name, expr = part.split("=", 1)
            expr = re.sub(r"\(([^()]*)\)\s*\?\s*([^:]+):\s*(.+)", r"(\2 if \1 else \3)", expr.strip())
            exec("%s = int(%s)" % (name.strip(), expr.replace("/", "//")), env)
    return env["SB_SMEM"]


def test_wgmma_not_serialized_or_dependent():
    out = _ptxas()
    assert "C7520" not in out and "C7507" not in out, out


def test_registers_fit_the_launch():
    for name, _, _, _, regs, _ in _kernel_props():
        # 576 threads = 18 warps, up to 5 on one SM sub-partition of 16 K registers
        assert 5 * 32 * regs <= 16384, (name, regs)


def test_shared_memory_fits():
    dyn = _dynamic_smem()
    for name, _, _, _, _, static in _kernel_props():
        assert dyn + static <= SMEM_LIMIT, (name, dyn, static)


def test_spills_within_cap():
    for name, _, st, ld, _, _ in _kernel_props():
        assert st <= SPILL_CAP and ld <= SPILL_CAP, (name, st, ld)
