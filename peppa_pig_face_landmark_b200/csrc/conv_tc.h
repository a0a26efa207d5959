// Host/device structs of the wgmma convolution path (conv_tc.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.h"

namespace skps {

struct TcK {                     // kernel parameters
    int H, W, bw, bh, tiles_per_img, m_tiles, n_tiles, n_tile;
    int img0;                    // first sample of this launch (always 0: a launch covers the whole batch)
    int img_end;                 // img0 + batch: rows of a multi-image tile past it are not stored
    int ipt;                     // images per 128-pixel tile (> 1 when Ho*Wo < 128, e.g. 8x8 maps)
    int stride;                  // conv stride (1 or 2): the A box walks the input with TMA element strides
    int mt;                      // pixel tiles per weight-tile load (1 or 2)
    int tma_store;               // epilogue stages 32-channel chunks in smem and stores them with TMA
    int out_bufs;                // staging buffers per epilogue warp group (1 or 2)
    int taps, kw, dil, pad, cchunks;
    int Cout, Cin, act, stages;
    float out_scale;             // exact power of two undoing the weight pre-scale
    const float* bias;
    void* out; int out_fmt; long long out_plane; int out_ld, out_coff, out_cstride;
    const void* res; int res_fmt; long long res_plane; int res_ld, res_coff;
    int res_first;               // act(acc + bias + res) (ResNet/HRNet blocks) instead of act(acc + bias) + res
    // heat-map head: instead of storing the map, the epilogue reduces every 128-pixel tile to per-channel (max, first arg-max)
    float* hm_val; int* hm_idx; int hm_ld;      // [img][tile][hm_ld] each; null = store the map as usual
};

struct TcLayer {                 // prepared once per conv op at engine creation
    CUtensorMap a_hi, a_lo, b_hi, b_lo, o_hi, o_lo;
    TcK k;
    int smem_bytes;
};

struct TcSetup {
    int H, W, Cin, in_ld, in_coff, max_batch;
    const void* in_base; long long in_plane;      // hi plane base (fp16), lo plane = base + in_plane elements
    int kh, kw, dil, pad, stride;                 // H, W above are INPUT dims; output dims = ceil(H/stride) x ceil(W/stride)
    int Cout, act, n_tile, n_tiles;
    float out_scale;
    const void* w_hi; const void* w_lo;           // device, (n_tiles*n_tile, K_pad) fp16
    const float* bias;
    void* out; int out_fmt; long long out_plane; int out_ld, out_coff, out_cstride;
    const void* res; int res_fmt; long long res_plane; int res_ld, res_coff;
    int res_first;
    float* hm_val; int* hm_idx; int hm_ld;        // per-tile (max, arg-max) partials of the heat-map head, or null
};

bool tc_shape_ok(int Ho, int Wo, int Cin, int in_ld, int in_coff);
int tc_prepare(TcLayer& L, const TcSetup& s);
// The launch at `batch` on num_sms SMs; fills the batch's kernel parameters into *k when k is not null
Grid tc_grid(const TcLayer& L, int batch, int num_sms, TcK* k = nullptr);
int tc_launch(const TcLayer& L, int batch, int num_sms, cudaStream_t stream);

}  // namespace skps
