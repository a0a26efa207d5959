// Host/device structs of the transposed heat-map head kernel (conv_hm.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_tc.h"

namespace skps {

struct HmK {                     // kernel parameters
    int bh, tiles_per_img, m_tiles, img0;       // tile = bh whole rows = 256 pixels
    int cchunks, Cin, Cout;
    float out_scale;             // exact power of two undoing the weight pre-scale
    const float* bias;
    float* hm_val; int* hm_idx; int hm_ld;      // [img][tile][hm_ld] each: per-tile maximum and first arg-max (pixel index y*W+x)
};

struct HmLayer {
    CUtensorMap x_hi, x_lo, w_hi, w_lo;
    HmK k;
    int smem_bytes = 0;
};

constexpr int HM_TILE_PIXELS = 256;

bool hm_shape_ok(int H, int W, int Cin, int Cout, int in_ld, int in_coff);
int hm_prepare(HmLayer& L, const TcSetup& s);                 // s.hm_val / hm_idx / hm_ld set, 1x1, linear
Grid hm_grid(const HmLayer& L, int batch, int num_sms, HmK* k = nullptr);   // as tc_grid
int hm_launch(const HmLayer& L, int batch, int num_sms, cudaStream_t stream);

}  // namespace skps
