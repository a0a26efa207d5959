"""Per-device state, read from the sources (no GPU): kernel attributes and the current device belong to one device.

- cudaFuncSetAttribute(..., MaxDynamicSharedMemorySize, ...) applies to the current device only, so every launcher
  raises its kernel's limit through common.h's smem_limit, which keeps the limit per device; a launcher with a flag of
  its own would launch on a second device without the opt-in.
- cudaSetDevice is called only by common.h's DeviceGuard, which gives the caller back its current device on every
  return path; and no entry takes its device from cudaGetDevice where its engines name one."""
import os
import re

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
CSRC = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "csrc")


def _sources():
    out = {}
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".h")):
            with open(os.path.join(CSRC, name)) as f:
                src = f.read()
            out[name] = re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", src, flags=re.S))
    return out


def _body(src, head):
    """The text of the definition that starts at `head`, up to its matching closing brace."""
    i = src.index(head)
    j = src.index("{", i)
    depth = 0
    for k in range(j, len(src)):
        depth += {"{": 1, "}": -1}.get(src[k], 0)
        if depth == 0:
            return src[i:k + 1]
    raise AssertionError("unbalanced braces after %r" % head)


def _outside(srcs, head):
    """Every source, with the definition that starts at `head` in common.h cut out."""
    srcs = dict(srcs)
    body = _body(srcs["common.h"], head)
    srcs["common.h"] = srcs["common.h"].replace(body, "")
    return srcs, body


def test_shared_memory_opt_in_only_through_the_per_device_helper():
    srcs, body = _outside(_sources(), "inline int smem_limit(")
    assert re.search(r"cudaFuncSetAttribute\s*\([^;]*MaxDynamicSharedMemorySize", body)
    assert re.search(r"set_bytes\s*\[\s*dev\s*\]", body)
    bad = [name for name, s in srcs.items() if re.search(r"cudaFuncSetAttribute\s*\([^;]*MaxDynamicSharedMemorySize", s)]
    assert not bad, "cudaFuncSetAttribute(MaxDynamicSharedMemorySize) outside smem_limit in %s" % bad
    flags = [name for name, s in srcs.items() if re.search(r"static\s+bool\s+attr_set", s)]
    assert not flags, flags
    users = [name for name, s in srcs.items() if re.search(r"\bsmem_limit\s*\(", s)]
    assert len(users) >= 10, users


def test_zero_bias_is_per_device():
    srcs, body = _outside(_sources(), "inline const float* zero_bias(")
    assert re.search(r"static\s+float\s*\*\s*z\s*\[\s*MAX_DEVICES\s*\]", body)
    others = [name for name, s in srcs.items() if re.search(r"\bzero_bias\s*\(\s*\)\s*\{", s)]
    assert not others, others
    for name in ("conv_tc.cu", "conv_xf.cu", "conv_fpw.cu"):
        assert re.search(r"\bzero_bias\s*\(\s*\)", srcs[name]), name


def test_current_device_set_only_by_the_guard():
    srcs, body = _outside(_sources(), "class DeviceGuard")
    assert "cudaGetDevice" in body and body.count("cudaSetDevice") == 2
    bad = [name for name, s in srcs.items() if "cudaSetDevice" in s]
    assert not bad, "cudaSetDevice outside DeviceGuard in %s" % bad
    for name in ("engine.cu", "pipeline.cu", "mpipe.cu"):
        assert "SKPS_ON_DEVICE" in srcs[name] and "DeviceGuard on(" in srcs[name], name
    for name in ("pipeline.cu", "mpipe.cu"):
        assert not re.search(r"cudaGetDevice\s*\(\s*&\s*p->device", srcs[name]), name
        assert "engine_pair_device(" in srcs[name], name
