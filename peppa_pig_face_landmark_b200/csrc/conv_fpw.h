// Fused "producer -> pointwise conv" layers on a wgmma kernel whose accumulators stay in registers (conv_fpw.cu): the
// student's depthwise -> 1x1 and squeeze-excite -> 1x1 layers.  The A producer is conv_xf's (xf_producer.h); the engine
// routes a layer here when fpw_supported() holds and leaves the rest (ragged maps, channel-shuffled outputs) on conv_xf.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "xf_producer.h"

namespace skps {

struct FpwK {
    XfProducer a;                                   // the A producer (no edge tiles: H % 8 == W % 16 == 0)
    int units;                                      // work items of the launch: batch * tiles_per_img * nsplit (/ 2 paired)
    int nsplit;                                     // work units per tile: ceil(N tile / unit width)
    int bs, out_bufs;                               // ring depths: B tiles, epilogue staging buffers
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
    bool pair = false;                              // on conv_fpw_pair: work items of two units sharing each A tile
    int smem_bytes = 0;
};

bool fpw_supported(const XfSetup& s);
int fpw_prepare(FpwLayer& L, const XfSetup& s);
Grid fpw_grid(const FpwLayer& L, int batch, int num_sms, FpwK* k = nullptr);   // as tc_grid
int fpw_launch(const FpwLayer& L, int batch, int num_sms, cudaStream_t stream);

}  // namespace skps
