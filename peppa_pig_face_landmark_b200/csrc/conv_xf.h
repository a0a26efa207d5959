// Fused "producer -> pointwise conv" kernels on wgmma (conv_xf.cu): the A operand of a 1x1 convolution is produced
// inside the kernel by transform warps instead of being read from HBM (xf_producer.h).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "xf_producer.h"

namespace skps {

struct XfK {
    XfProducer a;                                   // the A producer
    int m_tiles;                                    // 16 x 8 pixel tiles of the launch
    int n_tile, nsplit, n_sub;                      // UMMA N per instruction = n_sub = n_tile / nsplit
    int bs, out_bufs;                               // ring depths: B tiles, epilogue staging buffers
    // epilogue (same meaning as TcK)
    int Cout, act;
    float out_scale;
    const float* bias;
    void* out; int out_fmt; long long out_plane; int out_ld, out_coff, out_cstride; int tma_store;
    const void* res; int res_fmt; long long res_plane; int res_ld, res_coff; int res_first;
};

struct XfLayer {
    CUtensorMap src0, src1_hi, src1_lo, b_hi, b_lo, o_hi, o_lo, w_eff;
    XfK k;
    int mode, smem_bytes;
};

int xf_prepare(XfLayer& L, const XfSetup& s);
Grid xf_grid(const XfLayer& L, int batch, int num_sms, XfK* k = nullptr);   // as tc_grid
int xf_launch(const XfLayer& L, int batch, int num_sms, cudaStream_t stream);

}  // namespace skps
