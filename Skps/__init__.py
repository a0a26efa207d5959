"""Drop-in import surface: `from Skps import FaceAna` (reference: Skps/__init__.py:7)."""
from peppa_pig_face_landmark_b200.core.api.facer import FaceAna

from peppa_pig_face_landmark_b200.core.api.streams import FaceAnaStreams   # additive: many streams per GPU
from peppa_pig_face_landmark_b200.core.api.face_landmark import FaceLandmark   # additive: landmarks on the caller's boxes
from peppa_pig_face_landmark_b200.core.api.face_detector import FaceDetector   # additive: the detector over many frames

__all__ = ['FaceAna', 'FaceAnaStreams', 'FaceDetector', 'FaceLandmark']
