"""Direct kernel-vs-oracle unit tests of the small fused kernels that the whole-network tests only cover implicitly:
skps_select_faces (judge_boxs + sort_and_filter, facer.py:120-189), se_fc_kernel (squeeze-excite gate) and
hm_decode_kernel (arg-max + offsets, model.py:511-554; ties -> first index)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _select(lib, rt, torch, det, track, top_k, min_face=1600.0, iou=0.5, alpha=0.3):
    n = det.shape[0]
    d_det = torch.from_numpy(np.ascontiguousarray(det if n else np.zeros((1, det.shape[1])), np.float32)).cuda()   # non-null when empty
    d_cnt = torch.tensor([n], dtype=torch.int32, device="cuda")
    d_trk = torch.from_numpy(np.ascontiguousarray(track, np.float32)).cuda() if track is not None and len(track) else None
    d_box = torch.zeros((top_k, 4), dtype=torch.float32, device="cuda")
    d_out = torch.zeros((1,), dtype=torch.int32, device="cuda")
    rt.check(lib.skps_select_faces(d_det.data_ptr(), d_cnt.data_ptr(), det.shape[1],
                                   d_trk.data_ptr() if d_trk is not None else None, 0 if d_trk is None else d_trk.shape[0],
                                   iou, alpha, float(1.0 - alpha), min_face, top_k, d_box.data_ptr(), d_out.data_ptr(), None))
    torch.cuda.synchronize()
    m = int(d_out.item())
    return d_box[:m].cpu().numpy()


@pytest.mark.parametrize("seed,n,n_track,top_k", [(0, 12, 0, 5), (1, 12, 4, 5), (2, 40, 16, 16), (3, 3, 2, 5), (4, 0, 3, 5)])
def test_select_faces_matches_oracle(seed, n, n_track, top_k):
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    from oracle import host_ref
    lib = rt.load_library()
    rng = np.random.default_rng(seed)
    xy = rng.uniform(0, 1500, (n, 2))
    wh = rng.uniform(10, 300, (n, 2))           # some faces under the 1600 px^2 area floor
    det = np.zeros((n, 16), np.float32)
    det[:, :2], det[:, 2:4] = xy, xy + wh
    det[:, 4:] = rng.uniform(0, 1, (n, 12))
    track = None
    if n_track:
        pick = rng.integers(0, max(n, 1), n_track)
        track = (det[pick, :4] + rng.uniform(-12, 12, (n_track, 4))).astype(np.float32) if n else \
            rng.uniform(0, 500, (n_track, 4)).astype(np.float32)
    got = _select(lib, rt, torch, det, track, top_k)
    want = host_ref.sort_and_filter(host_ref.judge_boxs(track, det) if n else np.zeros((0, 4), np.float32), 1600, top_k)
    want = np.asarray(want, np.float64).reshape(-1, det.shape[1] if (n and track is None) else 4)[:, :4]
    assert got.shape == want.shape, (got.shape, want.shape)
    assert np.abs(got - want).max(initial=0) <= 1e-3          # EMA in float32 on the device, float64 mix on the host


@pytest.mark.parametrize("C_,Cr,tiles,hw", [(72, 24, 8, 1024), (120, 32, 4, 1024), (480, 120, 2, 256), (960, 240, 1, 256)])
def test_se_fc_kernel_matches_fp32(C_, Cr, tiles, hw):
    from peppa_pig_face_landmark_b200 import runtime as rt
    lib = rt.load_library()
    rng = np.random.default_rng(C_)
    N = 9                                        # not a multiple of the 4 samples a CTA handles
    part = rng.standard_normal((N, tiles, C_)).astype(np.float32) * 50
    w1 = (rng.standard_normal((Cr, C_)) / np.sqrt(C_)).astype(np.float32)
    w2 = (rng.standard_normal((C_, Cr)) / np.sqrt(Cr)).astype(np.float32)
    b1, b2 = rng.standard_normal(Cr).astype(np.float32), rng.standard_normal(C_).astype(np.float32)
    w1t, w2t = np.ascontiguousarray(w1.T), np.ascontiguousarray(w2.T)
    gate = np.empty((N, C_), np.float32)
    rt.check(lib.skps_debug_se_fc(part.ctypes.data, N, tiles, C_, w1t.ctypes.data, b1.ctypes.data, w2t.ctypes.data,
                                  b2.ctypes.data, Cr, 1, 5, hw, gate.ctypes.data))
    mean = part.astype(np.float64).sum(1) / hw
    h = np.maximum(mean @ w1.T.astype(np.float64) + b1, 0)
    g = np.clip((h @ w2.T.astype(np.float64) + b2) * np.float32(1 / 6) + 0.5, 0, 1)
    assert np.abs(gate - g).max() < 2e-5


@pytest.mark.parametrize("split", [False, True])
def test_hm_decode_kernel_matches_oracle_and_breaks_ties_by_first_index(split):
    import torch
    from peppa_pig_face_landmark_b200 import runtime as rt
    from oracle.plan_interp import PlanInterp
    lib = rt.load_library()
    rng = np.random.default_rng(5)
    N, H, W, P, K = 3, 64, 64, 98, 128
    ld = 104 if split else 3 * P + 2                 # padded pixel rows, as the engine allocates them
    hm = rng.standard_normal((N, H, W, ld)).astype(np.float32)
    # exact ties: the same maximum at several pixels of some maps -> the first (row-major) index must win
    for n in range(N):
        for c in (0, 17, 97):
            pos = np.sort(rng.choice(H * W, 3, replace=False))
            hm[n].reshape(H * W, ld)[pos, c] = 9.5
    feat = rng.standard_normal((N, H, W, K)).astype(np.float32) if split else None
    w_off = (rng.standard_normal((2 * P, K)) / 16).astype(np.float32) if split else None
    b_off = rng.standard_normal(2 * P).astype(np.float32) if split else None
    xy, sc = np.empty((N, 2 * P), np.float32), np.empty((N, P), np.float32)
    rt.check(lib.skps_debug_hm_decode(hm.ctypes.data, N, H, W, ld, P, feat.ctypes.data if split else None, K,
                                      w_off.ctypes.data if split else None, b_off.ctypes.data if split else None,
                                      xy.ctypes.data, sc.ctypes.data))
    if split:
        rxy, rsc = PlanInterp._hm_decode_split(torch.from_numpy(hm[..., :P]), torch.from_numpy(feat), w_off, b_off, P)
    else:
        rxy, rsc = PlanInterp._hm_decode(torch.from_numpy(hm[..., :3 * P]), P)
    rxy, rsc = rxy.numpy().reshape(N, -1), rsc.numpy()
    assert np.array_equal(sc, rsc)                               # the maxima themselves: exact
    assert np.abs(xy - rxy).max() * W < (1e-4 if split else 1e-6)   # px; the split head re-evaluates two 128-long dot products
