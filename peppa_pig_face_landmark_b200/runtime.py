"""ctypes binding of libskps_b200.so (include/skps_b200.h).

There is no CPU fallback: if the CUDA library is missing or does not load, importing the
product path raises.  Build it with `python -m peppa_pig_face_landmark_b200.build`
(or `__graft_entry__.build()`).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libskps_b200.so")

c_i32p = C.POINTER(C.c_int32)
c_f32p = C.POINTER(C.c_float)
c_u8p = C.POINTER(C.c_uint8)
c_vp = C.c_void_p


class PipelineCfg(C.Structure):
    _fields_ = [("score_thres", C.c_float), ("iou_thres", C.c_float), ("min_face", C.c_float),
                ("top_k", C.c_int), ("track_iou", C.c_float), ("alpha", C.c_float),
                ("face_scale", C.c_float), ("kps_min_face", C.c_float),
                ("max_h", C.c_int), ("max_w", C.c_int)]


class MpipeOutputs(C.Structure):
    """skps_mpipe_outputs: device addresses of one batch's result buffers."""
    _fields_ = [(name, c_vp) for name in ("n_faces", "ran_detector", "boxes", "kps", "scores", "chips", "M", "rvec", "tvec",
                                          "euler", "reproject", "ids")]


# name -> (restype, argtypes); every symbol include/skps_b200.h declares
SIGNATURES = {
    "skps_last_error": (C.c_char_p, []),
    "skps_version": (C.c_int, []),
    "skps_engine_create": (C.c_int, [c_vp, C.c_size_t, c_vp, C.c_size_t, C.c_int, C.c_int, C.POINTER(c_vp)]),
    "skps_engine_destroy": (None, [c_vp]),
    "skps_engine_input_dims": (C.c_int, [c_vp, c_i32p, c_i32p, c_i32p]),
    "skps_engine_num_outputs": (C.c_int, [c_vp]),
    "skps_engine_output_elems": (C.c_int, [c_vp, C.c_int]),
    "skps_engine_input_ptr": (c_vp, [c_vp]),
    "skps_engine_output_ptr": (c_vp, [c_vp, C.c_int]),
    "skps_engine_forward": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp]),
    "skps_engine_forward_host_f32": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp]),
    "skps_engine_forward_host_u8": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp]),
    "skps_engine_submit_host_u8": (C.c_int, [c_vp, C.c_int, c_vp, C.c_int, c_vp]),
    "skps_engine_wait": (C.c_int, [c_vp, C.c_int]),
    "skps_engine_num_buffers": (C.c_int, [c_vp]),
    "skps_engine_buffer_dims": (C.c_int, [c_vp, C.c_int, c_i32p, c_i32p, c_i32p, c_i32p]),
    "skps_engine_read_buffer": (C.c_int, [c_vp, C.c_int, C.c_int, c_vp]),
    "skps_engine_launches_per_forward": (C.c_int, [c_vp]),
    "skps_engine_launches_for_batch": (C.c_int, [c_vp, C.c_int]),
    "skps_engine_run_op": (C.c_int, [c_vp, C.c_int, C.c_int, c_vp]),
    "skps_engine_op_kernel": (C.c_int, [c_vp, C.c_int, c_i32p]),
    "skps_engine_set_num_sms": (C.c_int, [c_vp, C.c_int]),
    "skps_engine_op_grid": (C.c_int, [c_vp, C.c_int, C.c_int, c_i32p]),
    "skps_debug_conv_tc": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, C.c_int, C.c_int,
                                     C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, c_vp, C.c_int, c_vp]),
    "skps_debug_conv_tc2": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, C.c_int, C.c_int,
                                      C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, c_vp, C.c_int, c_vp, C.c_int,
                                      C.c_int, C.c_int]),
    "skps_debug_conv_pw": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp,
                                     C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, c_vp]),
    "skps_debug_conv_xf": (C.c_int, [C.c_int, c_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, C.c_int, c_vp, c_vp,
                                     C.c_int, c_vp, c_vp, c_vp, C.c_int, C.c_int, C.c_int, C.c_float, c_vp, C.c_int, C.c_int, c_vp, c_vp]),
    "skps_debug_conv_fpw": (C.c_int, [C.c_int, c_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, C.c_int, c_vp, c_vp,
                                      C.c_int, c_vp, c_vp, c_vp, C.c_int, C.c_int, C.c_int, C.c_float, c_vp, C.c_int, C.c_int, c_vp,
                                      c_vp, C.c_int]),
    "skps_debug_conv_hm": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, C.c_int, C.c_int, C.c_float,
                                    c_vp, c_vp]),
    "skps_debug_se_fc": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_vp]),
    "skps_debug_hm_decode": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, C.c_int, c_vp, c_vp, c_vp, c_vp]),
    "skps_debug_conv_mma": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_vp, C.c_int, C.c_float, c_vp,
                                      C.c_int, C.c_int, c_vp]),
    "skps_letterbox": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, c_vp, C.c_int, C.c_int,
                                 C.c_int, C.c_int, C.c_int, C.c_int, c_vp]),
    "skps_letterbox_frames": (C.c_int, [c_vp, C.c_int, c_vp, C.c_int, C.c_int, c_vp]),
    "skps_letterbox_frames_layout": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, C.c_int, C.c_int, c_vp]),
    "skps_letterbox_frames_rotate": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, c_vp, C.c_int, C.c_int, c_vp]),
    "skps_detect_post": (C.c_int, [c_vp, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                   c_vp, c_vp, c_vp, C.c_int, c_vp]),
    "skps_detect_post_workspace_size": (C.c_size_t, [C.c_int, C.c_int]),
    "skps_detect_post_batch": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_float, C.c_float, c_vp, c_vp, c_vp, c_vp, C.c_int,
                                         c_vp, C.c_size_t, c_vp]),
    "skps_select_faces": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, C.c_int, C.c_float, C.c_float, C.c_float,
                                    C.c_float, C.c_int, c_vp, c_vp, c_vp]),
    "skps_select_faces_batch": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.c_float, C.c_int, c_vp, c_vp, c_vp]),
    "skps_landmark_boxes": (C.c_int, [c_vp, C.c_int, c_vp, C.c_int, c_vp, c_vp, C.c_int, C.c_float, C.c_float, C.c_float,
                                      c_vp, c_vp]),
    "skps_crop_resize": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp, C.c_int, C.c_float, C.c_float,
                                   c_vp, C.c_int, c_vp, c_vp]),
    "skps_crop_faces": (C.c_int, [c_vp, c_vp, C.c_int, C.c_float, C.c_float, c_vp, C.c_int, c_vp, c_vp]),
    "skps_crop_faces_layout": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, C.c_float, C.c_float, c_vp, C.c_int, c_vp, c_vp]),
    "skps_crop_faces_rotate": (C.c_int, [c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_float, C.c_float, c_vp, C.c_int, c_vp, c_vp]),
    "skps_landmark_post": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, C.c_int, c_vp, c_vp]),
    "skps_frame_absdiff_sum": (C.c_int, [c_vp, c_vp, C.c_size_t, c_vp, c_vp]),
    "skps_frame_ingest": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp]),
    "skps_frame_ingest_layout": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp]),
    "skps_frame_ingest_rotate": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp,
                                           c_vp]),
    "skps_pipeline_create": (C.c_int, [c_vp, c_vp, C.POINTER(PipelineCfg), C.POINTER(c_vp)]),
    "skps_pipeline_destroy": (None, [c_vp]),
    "skps_pipeline_reset": (C.c_int, [c_vp]),
    "skps_pipeline_run": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, c_vp, C.c_int,
                                    c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "skps_pipeline_det_results": (C.c_int, [c_vp, C.c_int, c_vp, c_vp]),
    "skps_pipeline_face_sources": (C.c_int, [c_vp, C.c_int, c_vp]),
    "skps_crop_rect": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, C.c_int, c_vp]),
    "skps_nme": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_vp]),
    "skps_head_pose": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "skps_debug_rotation": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp]),
    "skps_mpipe_create": (C.c_int, [c_vp, c_vp, C.POINTER(PipelineCfg), C.c_int, C.POINTER(c_vp)]),
    "skps_mpipe_destroy": (None, [c_vp]),
    "skps_mpipe_reset": (C.c_int, [c_vp, C.c_int]),
    "skps_mpipe_dims": (C.c_int, [c_vp, c_i32p, c_i32p, c_i32p]),
    "skps_mpipe_submit": (C.c_int, [c_vp, C.c_int, c_vp, c_vp, C.c_int]),
    "skps_mpipe_wait": (C.c_int, [c_vp, C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "skps_mpipe_submit_device": (C.c_int, [c_vp, C.c_int, c_vp, c_vp, c_vp, C.c_int, C.POINTER(MpipeOutputs), c_vp]),
    "skps_mpipe_submit_streams": (C.c_int, [c_vp, C.c_int, c_vp, c_vp, c_vp, C.c_int]),
    "skps_mpipe_submit_device_streams": (C.c_int, [c_vp, C.c_int, c_vp, c_vp, c_vp, c_vp, C.c_int, C.POINTER(MpipeOutputs),
                                                   c_vp]),
    "skps_mpipe_submit_device_layout": (C.c_int, [c_vp, C.c_int, c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_int, c_vp,
                                                  C.POINTER(MpipeOutputs), c_vp]),
    "skps_mpipe_submit_device_rotate": (C.c_int, [c_vp, C.c_int, c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_int, c_vp, c_vp,
                                                  C.POINTER(MpipeOutputs), c_vp]),
    "skps_mpipe_wait_stream": (C.c_int, [c_vp, C.c_int, c_vp]),
    "skps_mpipe_track_ids": (C.c_int, [c_vp, C.c_int, c_vp]),
    "skps_debug_mp_temporal": (C.c_int, [C.POINTER(PipelineCfg), C.c_int, C.c_int, C.c_int] + [c_vp] * 18),
    "skps_pipeline_commit_frame": (C.c_int, [c_vp]),
    "skps_pipeline_frame_diff": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.POINTER(C.c_double), c_vp]),
    "skps_pipeline_frame_diff_device": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.c_int, c_vp, C.POINTER(C.c_double), c_vp]),
    "skps_pipeline_frame_diff_device_layout": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_vp,
                                                         C.POINTER(C.c_double), c_vp]),
    "skps_pipeline_frame_diff_device_rotate": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                         c_vp, C.POINTER(C.c_double), c_vp]),
    "skps_warp_affine": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp]),
    "skps_align_faces": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp,
                                   c_vp]),
    "skps_warp_faces": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp]),
    "skps_warp_faces_layout": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp]),
    "skps_warp_faces_rotate": (C.c_int, [c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp]),
    "skps_align_estimate": (C.c_int, [c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp]),
    "skps_warp_faces_count": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, C.c_int, c_vp, C.c_int, C.c_int, c_vp, c_vp]),
    "skps_warp_faces_count_rotate": (C.c_int, [c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_int, c_vp, C.c_int, C.c_int, c_vp,
                                               c_vp]),
    "skps_det_align_estimate": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp]),
    "skps_pipeline_align": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, c_vp, c_vp, c_vp]),
    "skps_mpipe_set_align": (C.c_int, [c_vp, C.c_int]),
    "skps_mpipe_align_results": (C.c_int, [c_vp, C.c_int, c_vp, c_vp]),
    "skps_pipeline_pose": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "skps_head_pose_faces": (C.c_int, [c_vp, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "skps_mpipe_set_pose": (C.c_int, [c_vp, C.c_int]),
    "skps_mpipe_pose_results": (C.c_int, [c_vp, C.c_int, c_vp, c_vp, c_vp, c_vp]),
    "skps_mpipe_set_detect_every": (C.c_int, [c_vp, C.c_int]),
    "skps_mpipe_detector_frames": (C.c_int, [c_vp, C.c_int, c_i32p]),
    "skps_mpipe_set_id_memory": (C.c_int, [c_vp, C.c_int]),
    "skps_debug_mp_temporal_mem": (C.c_int, [C.POINTER(PipelineCfg), C.c_int, C.c_int, C.c_int] + [c_vp] * 17 + [C.c_int]
                                   + [c_vp] * 5),
}

_lib = None


def load_library():
    """Load libskps_b200.so and bind every declared symbol (raises if anything is missing)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("skps_b200: %s not found - build the CUDA library first "
                           "(python -m peppa_pig_face_landmark_b200.build); there is no CPU fallback" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)       # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise RuntimeError("skps_b200: " + load_library().skps_last_error().decode(errors="replace"))


def ptr(a):
    """Raw address of a numpy array or torch tensor (containers only)."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("skps_b200: no CUDA device visible; this implementation has no CPU path")
    return torch
