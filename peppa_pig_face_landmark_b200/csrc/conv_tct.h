// Host/device structs of the transposed wgmma convolution (conv_tct.cu): channels as M, 256 pixels as N.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_tc.h"

namespace skps {

struct TctK {                    // kernel parameters
    int W, bh, tiles_per_img, m_tiles, img0;    // tile = bh whole rows = 256 pixels
    int taps, kw, dil, pad, cchunks, Cin, Cout, act;
    int x_plane, x_slots;        // bytes of one plane of a halo slot (bh + dil (kh - 1) rows x W pixels x 64 B); slots in the ring
    float out_scale;             // exact power of two undoing the weight pre-scale
    const float* bias;
};

struct TctLayer {
    CUtensorMap x_hi, x_lo, w_hi, w_lo, o_hi, o_lo;
    TctK k;
    int smem_bytes = 0;
};

bool tct_applicable(const TcSetup& s);          // s.H, s.W: the (stride-1) map; split-fp16 contiguous output, no residual
int tct_prepare(TctLayer& L, const TcSetup& s);
Grid tct_grid(const TctLayer& L, int batch, int num_sms, TctK* k = nullptr);   // as tc_grid
int tct_launch(const TctLayer& L, int batch, int num_sms, cudaStream_t stream);

}  // namespace skps
