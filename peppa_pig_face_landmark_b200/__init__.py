"""H100-native (sm_90a) implementation of the FaceAna inference path of 610265158/Peppa_Pig_Face_Landmark.

    from peppa_pig_face_landmark_b200 import FaceAna      # or:  from Skps import FaceAna
    facer = FaceAna()
    result = facer.run(image_bgr_uint8)                   # [{'box','kps','scores'}, ...]

Importing the package does not touch CUDA; constructing FaceAna / ONNXEngine loads
libskps_b200.so and fails loudly if it (or a CUDA device) is missing.
"""


def __getattr__(name):
    if name == "FaceAna":
        from .core.api.facer import FaceAna
        return FaceAna
    if name == "FaceAnaImages":
        from .core.api.images import FaceAnaImages
        return FaceAnaImages
    if name == "FaceAnaStreams":
        from .core.api.streams import FaceAnaStreams
        return FaceAnaStreams
    if name == "FaceDetector":
        from .core.api.face_detector import FaceDetector
        return FaceDetector
    if name == "FaceLandmark":
        from .core.api.face_landmark import FaceLandmark
        return FaceLandmark
    if name == "ONNXEngine":
        from .core.api.onnx_model_base import ONNXEngine
        return ONNXEngine
    raise AttributeError(name)


__all__ = ["FaceAna", "FaceAnaImages", "FaceAnaStreams", "FaceDetector", "FaceLandmark", "ONNXEngine"]
