"""conv_tc and conv_xf on the ragged output maps re-targeted detector inputs produce: maps whose width neither divides
nor is a multiple of 128, so conv_tc's tc_pick_bw tiles them with bw x (128/bw) boxes whose edge tiles hang over the
right and/or bottom border (the TMA loads zero-fill, the stores clip or are masked).  The tile each shape gets:
    13x23 -> bw 8 (ragged right and bottom)      15x27 -> bw 32 (both)       5x120 -> bw 64, bh 2 (both)
    14x18 -> bw 8 (both)                         136x8 -> bw 8 (bottom only) 20x20 -> bw 32 (right only)
    26x46 -> bw 16 (both)
Batch 3 with 3 or 9 pixel tiles: odd tile counts for the two-tiles-per-weight-load (mt = 2) schedule."""
import pytest

import test_conv_tc_gpu as tc
import test_conv_xf_gpu as xf

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cfg", [
    # N, H, W, Cin, Cout, k, dil, act (+ options): H x W is the input, the output is H/stride x W/stride
    (3, 13, 23, 64, 64, 3, 1, 1),        # bw 8, 3x3
    (3, 13, 23, 96, 40, 1, 1, 0),        # bw 8, 1x1
    (3, 15, 27, 64, 48, 1, 1, 0),        # bw 32
    (3, 15, 27, 72, 64, 3, 1, 2),
    (3, 5, 120, 32, 64, 3, 1, 2),        # bw 64, bh 2
    (3, 5, 120, 64, 24, 1, 1, 1),
    (3, 14, 18, 40, 72, 3, 1, 1),        # bw 8
    (3, 136, 8, 64, 32, 1, 1, 1),        # bw 8, ragged at the bottom only
    (3, 136, 8, 32, 32, 3, 1, 0),
    (3, 20, 20, 96, 96, 3, 1, 0),        # bw 32, ragged at the right only
    (3, 26, 46, 64, 64, 3, 1, 1),        # bw 16
    (3, 26, 46, 48, 64, 1, 1, 0),
    (3, 26, 46, 64, 128, 3, 1, 1, dict(stride=2)),       # stride 2 onto 13x23 (bw 8)
    (3, 30, 54, 48, 96, 3, 1, 1, dict(stride=2)),        # stride 2 onto 15x27 (bw 32)
    (3, 10, 240, 32, 64, 3, 1, 2, dict(stride=2)),       # stride 2 onto 5x120 (bw 64, bh 2)
    (3, 15, 27, 64, 64, 3, 2, 0),        # dilation 2: the halo reaches two pixels past the edge tile
    (3, 13, 23, 64, 64, 3, 2, 1),
    (3, 13, 23, 64, 294, 1, 1, 0),       # two N tiles, ragged Cout
    (2, 5, 120, 160, 960, 1, 1, 2),      # four N tiles
    (3, 15, 27, 64, 64, 3, 1, 1, dict(with_res=True, out_split=True)),
    (3, 13, 23, 40, 40, 3, 1, 1, dict(with_res=True, res_first=True, out_split=True)),
    (3, 20, 20, 64, 32, 1, 1, 0, dict(with_res=True)),
    (1, 20, 20, 64, 64, 3, 1, 1),        # 5 pixel tiles, mt = 2: the last weight load serves one tile
    (3, 13, 23, 64, 64, 3, 1, 1, dict(max_batch=4)),     # 9 tiles (odd) with spare buffer capacity
])
def test_conv_tc_ragged_edge_tiles(cfg):
    err = tc._run(*cfg[:8], **(cfg[8] if len(cfg) > 8 else {}))
    assert err < 1e-5, (cfg, err)


@pytest.mark.parametrize("cfg", [
    # N, H, W, Cx, Cout, dw_act, act, with_res: depthwise 3x3 -> 1x1 (OP_DWPW) on maps whose height is not a multiple of 8
    (3, 13, 23, 64, 64, 1, 0, True),
    (3, 15, 27, 32, 64, 0, 1, False),
    (3, 10, 240, 64, 32, 2, 0, True),
])
def test_xf_depthwise_pointwise_ragged_maps(cfg):
    N, H, W, Cx, Cout, dw_act, act, with_res = cfg
    err = xf._run(1, N, H, W, Cx, Cout, dw_act=dw_act, act=act, with_res=with_res)
    assert err < 1e-5, (cfg, err)
