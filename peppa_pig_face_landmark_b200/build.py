"""Builds libskps_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache: the library is built once by build()
and loaded from the package directory)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libskps_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
          "-I", os.path.join(HERE, "..", "include")]
# per-file extra flags
SOURCES = {
    "engine.cu": [],
    "pipeline.cu": [],
    "mpipe.cu": [],
    "headpose.cu": [],
    "temporal.cu": ["-fmad=false"],  # float64 arithmetic must round like numpy's (no contraction)
    "conv_simt.cu": [],
    "conv_tc.cu": [],
    "conv_xf.cu": [],
    "conv_hm.cu": [],
    "conv_tct.cu": [],
    "conv_pw.cu": [],
    "conv_fpw.cu": [],
    "stem_block.cu": [],
    "conv_mma.cu": [],
    "dw_tma.cu": [],
    "ops_misc.cu": [],
    "debug_ops.cu": [],
    "image_ops.cu": ["-fmad=false"],     # float32/double expressions must round like numpy's
    "nms.cu": ["-fmad=false"],           # the NMS IoU and scale_coords must round like numpy's
    "align.cu": ["-fmad=false"],         # double source coordinates must round like OpenCV's warpAffine
}


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "skps_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    objs = []
    procs = []
    for src, extra in SOURCES.items():
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc] + ARCH + COMMON + extra + (["-Xptxas", "-v"] if verbose else []) + \
              ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write("---- %s\n%s\n" % (src, out))
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    cmd = [nvcc] + ARCH + ["-shared", "-o", OUT] + objs + ["-lcudart"]
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
