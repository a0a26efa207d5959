"""The image ops of csrc/image_ops.cu have one kernel each, shared by FaceAna's single-frame pipeline, FaceAnaStreams'
batches and the public C entries: the single-frame copies are gone, and no kernel spills.  Compiles the source as
build.py does, for sm_90a, with -Xptxas -v (no GPU needed)."""
import re

from test_wgmma_codegen import _ptxas_report

REMOVED = ["letterbox_kernel", "crop_resize_kernel", "select_faces_kernel", "landmark_post_kernel",
           "absdiff_sum_kernel"]


def _kernels(out):
    # "Compiling entry function '_ZN4skps<len><name>...'": the unqualified name of every kernel
    names = []
    for mangled in re.findall(r"Compiling entry function '(\w+)'", out):
        m = re.match(r"_ZN4skps(\d+)", mangled)
        assert m, mangled
        names.append(mangled[m.end():m.end() + int(m.group(1))])
    return names


def test_one_kernel_per_image_op():
    names = _kernels(_ptxas_report("image_ops.cu"))
    assert "crop_faces_kernel" in names, names
    assert not set(REMOVED) & set(names), names
    assert not [n for n in names if n.startswith("mp_")], names


def test_image_ops_kernels_do_not_spill():
    out = _ptxas_report("image_ops.cu")
    spills = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", out)
    assert len(spills) == len(_kernels(out)), out
    bad = [(name, st, ld) for name, st, ld in spills if st != "0" or ld != "0"]
    assert not bad, bad
