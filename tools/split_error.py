"""What does the fp16 hi/lo activation/weight format alone cost?  The plan is executed on the CPU with every tensor-core
conv's operands rounded to the stored format (hi = fp16(v), lo = fp16(v - hi), subnormals included) and accumulated in
fp64, and compared with the fp64 oracle and with plain fp32 execution:  python tools/split_error.py [teacher|student] [n]"""
import os, sys
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
from peppa_pig_face_landmark_b200 import lowering
from oracle.plan_interp import PlanInterp
from oracle.onnx_exec import Session

model = sys.argv[1] if len(sys.argv) > 1 else "teacher"
n = int(sys.argv[2]) if len(sys.argv) > 2 else 2
if model == "teacher":
    from peppa_pig_face_landmark_b200 import teacher_graph as T
    path = T.ensure_teacher_onnx(); crops = T.synthetic_crops(n, 256, 7)
else:
    import frames
    path = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "kps_student.onnx"); crops = frames.crop_variants(n)
s64 = Session(path, dtype=torch.float64)
ref = np.array([s64.run(c.transpose(2, 0, 1)[None].astype(np.float64) / 255.0)[0].reshape(-1) for c in crops])
pl = lowering.lower(path, (256, 256))
for name, kw in (("fp32", {}), ("split16", dict(emulate_split=True)), ("split16, lo x 2^11", dict(emulate_split=True, lo_scale=2048.0))):
    xy = PlanInterp(pl, **kw).run(crops)[0].reshape(n, -1)
    print("%-22s vs fp64 oracle: %.3e px" % (name, np.abs(xy - ref).max() * 256))
