"""Unit tests of the fused producer -> 1x1 conv kernels (csrc/conv_xf.cu) through skps_debug_conv_xf, against
plain PyTorch float32 on the CPU: squeeze-excite scale ahead of conv_pwl (XF_SCALE), depthwise 3x3 ahead of
conv_pw[l] (XF_DW), and the DecoderBlock head bilinear-x2 -> concat -> depthwise -> 1x1 (model.py:133-196).
Shapes are the landmark network's (kps_student.onnx blocks.0-5, decoder/upsampler1-2) plus ragged maps."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _act(y, act):
    import torch
    if act == 1:
        return torch.relu(y)
    if act == 2:
        return y * torch.clamp(y * np.float32(1 / 6) + 0.5, 0, 1)
    return y


def _run(mode, N, H, W, Cx, Cout, Cl=0, x_split=False, dw_act=0, act=0, with_res=False, out_split=True, seed=0,
         x_scale=2.0):
    import torch
    import torch.nn.functional as F
    from peppa_pig_face_landmark_b200 import plan as P, runtime as rt
    lib = rt.load_library()
    rng = np.random.default_rng(seed)
    K = Cx + Cl
    kpad = -(-K // 64) * 64
    x = (rng.standard_normal((N, H, W, Cx)) * x_scale).astype(np.float32)
    low = (rng.standard_normal((N, H // 2, W // 2, Cl)) * x_scale).astype(np.float32) if Cl else None
    gate = rng.uniform(0, 1, (N, Cx)).astype(np.float32) if mode == 0 else None
    dw_w = (rng.standard_normal((9, K)) / 3).astype(np.float32)
    dw_b = rng.standard_normal(K).astype(np.float32)
    dww = np.zeros((10, kpad), np.float32)
    dww[:9, :K], dww[9, :K] = dw_w, dw_b
    w = (rng.standard_normal((Cout, 1, 1, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    res = rng.standard_normal((N, H, W, Cout)).astype(np.float32) if with_res else None
    n_tile, n_tiles = P.tc_tiling(Cout)
    assert n_tiles == 1
    hi, lo, out_scale = P.pack_tc_weights(w, n_tile, n_tiles)
    hi, lo = np.ascontiguousarray(hi), np.ascontiguousarray(lo)
    out = np.full((N, H, W, Cout), np.nan, np.float32)
    weff = P.pack_upcat_class_weights(dw_w[:, :Cl]) if Cl else None
    rt.check(lib.skps_debug_conv_xf(mode, x.ctypes.data, N, H, W, Cx, 1 if x_split else 0,
                                    low.ctypes.data if low is not None else None, Cl,
                                    gate.ctypes.data if gate is not None else None, dww.ctypes.data, dw_act,
                                    hi.ctypes.data, lo.ctypes.data, b.ctypes.data, Cout, act, n_tile, out_scale,
                                    res.ctypes.data if res is not None else None, 0, 1 if out_split else 0,
                                    out.ctypes.data, weff.ctypes.data if weff is not None else None))
    xt = torch.from_numpy(x).permute(0, 3, 1, 2)
    if mode == 0:
        a = xt * torch.from_numpy(gate)[:, :, None, None]
    else:
        if low is not None:
            up = F.interpolate(torch.from_numpy(low).permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False)
            xt = torch.cat([up, xt], 1)
        wd = torch.from_numpy(dw_w).T.reshape(K, 1, 3, 3).contiguous()
        a = _act(F.conv2d(xt, wd, torch.from_numpy(dw_b), padding=1, groups=K), dw_act)
    y = F.conv2d(a, torch.from_numpy(w).permute(0, 3, 1, 2).contiguous(), torch.from_numpy(b))
    y = _act(y, act).permute(0, 2, 3, 1).numpy()
    if res is not None:
        y = y + res
    assert np.isfinite(out).all(), "kernel left outputs unwritten"
    err = np.abs(out - y).max() / (np.abs(y).max() + 1e-9)
    print('conv_xf', (mode, N, H, W, Cx, Cl, Cout, dw_act, act), 'rel err %.3e' % err)
    return err


@pytest.mark.parametrize("cfg", [
    # N, H, W, Cx, Cout, with_res      squeeze-excite scale ahead of conv_pwl
    (3, 32, 32, 72, 40, False),         # blocks.2.0
    (3, 32, 32, 120, 40, True),         # blocks.2.1 / 2.2
    (3, 16, 16, 480, 112, False),       # blocks.4.0
    (2, 16, 16, 672, 160, False),       # blocks.5.0 (N tile 160 -> two halves of 80)
    (3, 16, 16, 960, 160, True),        # blocks.5.1 / 5.2: 15 K chunks
    (150, 16, 16, 64, 16, False),       # more tiles than SMs: the persistent loop wraps the rings
])
def test_xf_scale_matches_fp32(cfg):
    N, H, W, Cx, Cout, with_res = cfg
    err = _run(0, N, H, W, Cx, Cout, with_res=with_res)
    assert err < 1e-5, (cfg, err)


@pytest.mark.parametrize("cfg", [
    # N, H, W, Cx, Cout, dw_act, act, with_res, x_split
    (2, 128, 128, 16, 16, 1, 0, True, False),     # blocks.0.0: dw 3x3 + relu -> pw 16->16 + shortcut
    (2, 64, 64, 72, 24, 1, 0, True, False),       # blocks.1.1
    (3, 16, 16, 200, 80, 2, 0, True, False),      # blocks.3.1 (h-swish)
    (3, 16, 16, 184, 80, 2, 0, True, False),      # blocks.3.2 / 3.3
    (2, 32, 32, 40, 64, 0, 1, False, True),       # float16 hi/lo input planes
    (2, 24, 40, 32, 32, 1, 1, False, False),      # ragged map: edge tiles hang over the border
    (150, 16, 16, 96, 32, 1, 0, False, False),    # more tiles than SMs
])
def test_xf_depthwise_pointwise_matches_fp32(cfg):
    N, H, W, Cx, Cout, dw_act, act, with_res, x_split = cfg
    err = _run(1, N, H, W, Cx, Cout, x_split=x_split, dw_act=dw_act, act=act, with_res=with_res)
    assert err < 1e-5, (cfg, err)


@pytest.mark.parametrize("cfg", [
    # N, H, W, Cskip, Clow, Cout
    (2, 64, 64, 24, 256, 128),          # decoder/upsampler2 head
    (3, 32, 32, 40, 256, 256),          # decoder/upsampler1 head (N = 256: two halves of 128)
    (1, 16, 32, 8, 64, 16),             # smallest legal map, one skip sub-chunk
    (2, 16, 16, 40, 64, 32),            # map one tile wide: first and last columns in the same tile (Student@128)
    (150, 16, 16, 40, 64, 32),          # more tiles than SMs (300): the persistent loop wraps the rings
])
def test_xf_upsample_concat_depthwise_pointwise_matches_fp32(cfg):
    N, H, W, Cs, Cl, Cout = cfg
    err = _run(1, N, H, W, Cs, Cout, Cl=Cl, x_split=True, dw_act=0, act=1)
    assert err < 1e-5, (cfg, err)


def test_xf_scale_small_and_large_magnitudes():
    """Element-relative check away from N(0, 2^2): the hi/lo split keeps ~22 bits for |x| from 1e-3 to 1e+3."""
    for scale in (1e-3, 1e3):
        err = _run(0, 2, 16, 16, 128, 64, x_scale=scale, seed=3)
        assert err < 2e-5, (scale, err)
