// Fused "producer -> pointwise conv" layers on a wgmma kernel whose accumulators stay in registers (conv_fpw.cu): the
// student's depthwise -> 1x1 and squeeze-excite -> 1x1 layers.  Same layers and setup as conv_xf.cu (XfSetup); the engine
// routes a layer here when fpw_supported() holds and leaves the rest (ragged maps, channel-shuffled outputs) on conv_xf.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_xf.h"

namespace skps {

struct FpwK {
    int H, W, tiles_x, tiles_per_img;               // output map, 16 x 8 pixel tiles (no edge tiles: H % 8 == W % 16 == 0)
    int units;                                      // work units of the launch: batch * tiles_per_img * nsplit
    int nsplit;                                     // work units per tile: ceil(N tile / unit width)
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
    const float* dww;                               // [9][Kpad] depthwise weights then [Kpad] bias, zero padded
    const float* gate; int gate_ld, gate_coff;      // XF_SCALE: squeeze-excite gate (N,1,1,C) float32
    // epilogue: act(fmaf(acc, out_scale, bias) [+ res]) as in conv_xf
    int Cout;
    float out_scale;
    const float* bias;
    const void* res; int res_fmt; long long res_plane; int res_ld, res_coff; int res_first;
};

struct FpwLayer {
    CUtensorMap src0, src1_hi, src1_lo, b_hi, b_lo, o_hi, o_lo, w_eff;
    FpwK k;
    int mode = 0, n = 0, act = 0, out_fmt = 0;      // n: output channels per work unit (the kernel's N)
    int smem_bytes = 0;
    bool valid = false;
};

bool fpw_supported(const XfSetup& s);
int fpw_prepare(FpwLayer& L, const XfSetup& s);
int fpw_launch(const FpwLayer& L, int batch, int num_sms, cudaStream_t stream);

}  // namespace skps
