"""Drop-in import path of the reference: `from Skps.core.headpose.pose import get_head_pose` (Skps/core/headpose/pose.py)."""
from peppa_pig_face_landmark_b200.core.headpose.pose import (POSE_POINTS_98, get_head_pose, head_poses,  # noqa: F401
                                                              line_pairs, object_pts, reprojectsrc)
