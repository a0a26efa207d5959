"""The out= capacity check that FaceDetector, FaceLandmark and FaceAnaImages share (core/api/staging.py), on each class's
result fields, without a GPU."""
import pytest

K, P, R = 16, 98, 15120            # FaceAnaImages' top_k, the landmarks per face, the detector rows at 384x640


def _specs(kind):
    """(fields(n) of the kind's results for a call of n images, frames or faces; the same with another row size; the
    same with other keys, or None)."""
    from peppa_pig_face_landmark_b200.core.api import face_detector, face_landmark, images
    return {
        "images": (lambda n: images.result_fields(n, K, P, False), lambda n: images.result_fields(n, K + 1, P, False),
                   lambda n: images.result_fields(n, K, P, True)),
        "images_pose": (lambda n: images.result_fields(n, K, P, True), lambda n: images.result_fields(n, K + 1, P, True),
                        lambda n: images.result_fields(n, K, P, False)),
        "images_align": (lambda n: images.result_fields(n, K, P, True, 112),
                         lambda n: images.result_fields(n, K, P + 1, True, 112),
                         lambda n: images.result_fields(n, K, P, True)),
        "detector": (lambda n: face_detector.result_fields(n, R), lambda n: face_detector.result_fields(n, R + 1), None),
        "landmark": (lambda n: face_landmark.result_fields(n, P), lambda n: face_landmark.result_fields(n, P + 1),
                     lambda n: face_landmark.result_fields(n, P, 112)),
        "landmark_align": (lambda n: face_landmark.result_fields(n, P, 112),
                           lambda n: face_landmark.result_fields(n, P, 16),
                           lambda n: face_landmark.result_fields(n, P)),
    }[kind]


@pytest.mark.parametrize("kind", ["images", "images_pose", "images_align", "detector", "landmark", "landmark_align"])
def test_out_capacity_check(kind):
    import torch
    from peppa_pig_face_landmark_b200.core.api.staging import check_out, new_buffers
    cpu = torch.device("cpu")
    fields, resized, rekeyed = _specs(kind)
    out = new_buffers(fields(4), cpu)
    if kind.startswith("images"):
        assert out["box"].shape == (64, 4) and out["kps"].shape == (64, P, 2) and out["count"].shape == (4,)
    for n in (0, 1, 4):
        check_out(out, fields(n), cpu, [])
    with pytest.raises(ValueError):
        check_out(out, fields(5), cpu, [])                              # one image, frame or face too many
    with pytest.raises(ValueError):
        check_out(out, resized(4), cpu, [])                             # rows of another size (e.g. a smaller top_k)
    if rekeyed is not None:
        with pytest.raises(ValueError):
            check_out(out, rekeyed(1), cpu, [])                         # optional fields missing or extra
    bent = []
    for k, t in out.items():
        bent += [dict(out, **{k: t.double() if t.dtype != torch.float64 else t.float()}), dict(out, **{k: t.long()}),
                 dict(out, **{k: t.tolist()}), {j: v for j, v in out.items() if j != k}]
        if t.dim() > 1:
            bent += [dict(out, **{k: t[:, :-1]}),                                    # a trailing dimension too small
                     dict(out, **{k: t.transpose(0, 1).contiguous().transpose(0, 1)})]   # not contiguous
    if kind.startswith("images"):
        bent += [dict(out, kps=out["kps"][:, :97]), dict(out, scores=out["scores"].t())]
    for b in bent:
        with pytest.raises(ValueError):
            check_out(b, fields(1), cpu, [])
    with pytest.raises(ValueError):
        check_out(out, fields(1), cpu, busy=[None, {"x": out[next(iter(out))]}])     # a buffer of a call in flight
    check_out(out, fields(1), cpu, busy=[None, new_buffers(fields(1), cpu)])
