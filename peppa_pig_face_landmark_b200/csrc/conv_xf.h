// Fused "producer -> pointwise conv" kernels on wgmma (conv_xf.cu): the A operand of a 1x1 convolution is produced
// inside the kernel by transform warps instead of being read from HBM.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.h"

namespace skps {

enum { XF_SCALE = 0, XF_DW = 1 };                                   // kernel mode
enum { XS_UP_F32 = 0, XS_DW_F32 = 1, XS_DW_SPLIT = 2 };             // source of one 32-channel sub-chunk (XF_DW)
constexpr int XF_MAX_CHUNKS = 16;                                   // K <= 1024 channels

struct XfK {
    int H, W, tiles_x, tiles_per_img, m_tiles;      // output map, 16 x 8 pixel tiles
    int img0, img_end;
    int n_tile, nsplit, n_sub;                      // UMMA N per instruction = n_sub = n_tile / nsplit
    int cchunks, Cin;                               // K chunks of 64 channels
    int rs, as, bs, out_bufs;                       // ring depths: raw tiles, A tiles, B tiles, epilogue staging buffers
    int dw_act;                                     // activation between the depthwise stage and the pointwise conv
    int Hl, Wl;                                     // low-res map of the up-sampled channels (XS_UP_F32)
    int halves;                                     // transform mapping: 1 = two halves x 2-row patches (layers with up-sampled channels)
    int wcx;                                        // column classes per staged weight block: 3, or 4 when the map is one tile wide
    uint8_t sub_mode[2 * XF_MAX_CHUNKS];            // per 32-channel sub-chunk
    int16_t sub_c[2 * XF_MAX_CHUNKS];               // channel coordinate of the sub-chunk in its source tensor
    uint8_t chunk_subs[XF_MAX_CHUNKS];              // sub-chunks that hold real channels (1 or 2)
    uint8_t chunk_ksteps[XF_MAX_CHUNKS];            // 16-channel MMA steps that hold real channels (1..4)
    const float* dww;                               // [9][Kpad] depthwise weights then [Kpad] bias, zero padded (Kpad = cchunks*64)
    const float* gate; int gate_ld, gate_coff;      // XF_SCALE: squeeze-excite gate (N,1,1,C) float32
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
    bool valid = false;
};

struct XfSetup {
    int mode;                      // XF_SCALE / XF_DW
    int max_batch;
    // XF_SCALE: x = SPLIT16 input of the 1x1 conv, gate = (N,1,1,C) float32
    // XF_DW:    x = depthwise input (F32 or SPLIT16), or the skip tensor when `low` is set; low = F32 low-res tensor (H/2 x W/2)
    TView x, low, gate;
    const float* dww;              // device: [9][Kpad] + [Kpad]
    const float* weff;             // device: [low.C/32][4][4][9][32] row/column-class stencil weights of the up-sampled channels
    int dw_act;
    // pointwise conv
    int Cout, act, n_tile, n_tiles;
    float out_scale;
    const void* w_hi; const void* w_lo;      // [n_tile*n_tiles][Kpad] float16, K order = concat(low channels, x channels)
    const float* bias;
    TView out, res;
    int res_first;
};

bool xf_supported(const XfSetup& s);
int xf_prepare(XfLayer& L, const XfSetup& s);
int xf_launch(const XfLayer& L, int batch, int num_sms, cudaStream_t stream);

}  // namespace skps
