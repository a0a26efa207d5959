// Fused full-resolution head of the landmark encoder (stem_block.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.h"

namespace skps {

constexpr int SB_MAX_E = 64;

// Dense weights travel in the kernel-parameter (constant) bank; layouts chosen so that unrolled loops index them with
// compile-time constants.
struct StemBlockW {
    float stem_w[27 * 16];     // [(ky*3+kx)*3+ci][co]
    float stem_b[16];
    float dw0_w[9 * 16];       // [tap][c]
    float dw0_b[16];
    float pw0_w[16 * 16];      // [ci][co]
    float pw0_b[16];
    float pw1_w[16 * SB_MAX_E];   // [ci][co]
    float pw1_b[SB_MAX_E];
};

struct StemBlockK {
    const uint8_t* in;         // [N][H][W][3] uint8
    const float* in_f32;       // or [N][H][W][3] float32 already divided by 255 (ONNXEngine.__call__ feeds float32); null = uint8
    int H, W, Hq, Wq;          // input size, output (quarter-resolution) size
    int img0, n_tiles;         // first sample, tiles in this launch
    const float* dw1;          // device: [9][E] stride-2 depthwise weights then [E] bias
    void* out; int out_fmt; long long out_plane; int out_ld, out_coff;
};

bool stem_block_supported(int H, int W, int E, const TView& out);
Grid stem_block_grid(const StemBlockK& k, int num_sms);      // k.n_tiles set
int stem_block_launch(const StemBlockK& k, const StemBlockW& w, int num_sms, cudaStream_t s);

}  // namespace skps
