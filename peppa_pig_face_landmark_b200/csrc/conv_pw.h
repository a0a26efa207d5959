// Host/device structs of the pointwise wgmma convolution (conv_pw.cu): 1x1 stride-1 convs as one GEMM over the flat pixel
// index, C[batch*H*W][Cout] = A[batch*H*W][Cin] * W[Cout][Cin]^T.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_tc.h"

namespace skps {

struct PwK {                     // kernel parameters
    int m_tiles;                 // 128-pixel tiles of the launch (the last one may be partial)
    int n_chunks;                // output-channel chunks of nc channels per pixel tile
    int kblocks, Cin, Cout, stages, out_bufs;
    float out_scale;             // exact power of two undoing the weight pre-scale
    const float* bias;
};

struct PwLayer {                 // prepared once per conv op at engine creation
    CUtensorMap a_hi, a_lo, b_hi, b_lo;
    PwK k;
    int nc = 0;                  // output channels per work unit: 32, 64, 96 or 128
    int act = 0, out_fmt = 0;
    // output view: its tensor maps are encoded per launch, over the launch's batch * H * W rows, so the TMA stores of the
    // last (partial) pixel tile clip at the batch and never touch the rows of images past it
    void* out = nullptr; long long out_plane = 0; int out_ld = 0, out_coff = 0;
    long long hw = 0;            // pixels per image
    int smem_bytes = 0;
};

bool pw_applicable(const TcSetup& s);
int pw_prepare(PwLayer& L, const TcSetup& s);
Grid pw_grid(const PwLayer& L, int batch, int num_sms, PwK* k = nullptr);   // as tc_grid
int pw_launch(const PwLayer& L, int batch, int num_sms, cudaStream_t stream);

}  // namespace skps
