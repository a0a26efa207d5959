"""K tails of three 16-channel steps (a last 64-channel chunk of 33-48 channels) in the transposed kernels: conv_tct.cu and
conv_hm.cu issue each tail length from its own straight-line case, and the other lengths (4, 2 and 1 steps) are covered by
test_conv_tc_gpu.py."""
import pytest

import test_conv_tc_gpu as base

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cfg", [
    # N, H, W, Cin, Cout, k, dil, act
    (2, 32, 32, 112, 128, 3, 1, 1),      # one chunk of 64 + a tail of 48
    (2, 16, 256, 176, 96, 3, 1, 0),      # two chunks + a tail of 48, one row per tile, Cout < 128
])
def test_conv_tct_three_step_tail(cfg):
    err = base._run(*cfg, out_split=True)
    assert err < 1e-5, (cfg, err)


def test_conv_hm_three_step_tail():
    base.test_conv_hm_transposed_head_matches_fp64_argmax((2, 32, 32, 112, 104))
