// Host/device structs of the small-channel 3x3 convolution kernel (conv_mma.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.h"

namespace skps {

struct ConvMmaK {
    int H, W, tiles_x, tiles_img, batch, img0;
    const void* w;               // packed fp16 weights [tap][plane hi/lo][Cout][Cin]
    const float* bias;
    float out_scale;             // exact power of two undoing the weight pre-scale
    int act;
    void* out; int out_fmt; long long out_plane; int out_ld, out_coff;
    const void* res; int res_fmt; long long res_plane; int res_ld, res_coff; int res_first;
};

struct ConvMmaLayer {
    CUtensorMap a_hi, a_lo;      // (Cin, W, H, N) fp16 planes of the input view, box (Cin, 18, 10, 1)
    ConvMmaK k;
    int cin, cout;
    int ctas_per_sm = 1;         // resident CTAs of the kernel per SM (occupancy): the grid is num_sms x ctas_per_sm at most
};

bool conv_mma_supported(int cin, int cout, int kh, int kw, int stride, int dil, int pad);
int conv_mma_prepare(ConvMmaLayer& L, const TView& in, const TView& out, const TView& res, int res_first, const void* w_packed,
                     const float* bias, float out_scale, int act, int max_batch);
Grid conv_mma_grid(const ConvMmaLayer& L, int batch, int num_sms);   // as tc_grid
int conv_mma_launch(const ConvMmaLayer& L, int batch, int num_sms, cudaStream_t stream);

}  // namespace skps
