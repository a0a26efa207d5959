// TMA-staged depthwise convolution (dw_tma.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "common.h"

namespace skps {

struct DwTmaK {
    int C, Ho, Wo, pad, act, img0;
    int chunks, batch;           // channel chunks per image, images in this launch (grid = tiles x chunks x batch)
    float* part; int part_ld, part_coff;   // optional [n][tile][C] per-tile channel sums of the outputs (squeeze-excite GAP)
    int w_ld;                    // channel stride of the weight rows (>= C when this layer is a channel slice)
    const float* w; const float* bias;
    void* out; int out_fmt; long long out_plane; int out_ld, out_coff;
};

struct DwTmaLayer {
    CUtensorMap hi, lo;
    DwTmaK k;
    int k_size, stride, dil, split, chunks, smem_bytes;
};

bool dw_tma_supported(const TView& in, const TView& out, int k, int s, int d, int pad);
int dw_tma_prepare(DwTmaLayer& L, const TView& in, const TView& out, const float* w, const float* bias, int k, int s,
                   int d, int pad, int act, int max_batch, const TView* part = nullptr);
int dw_tile_rows(int k, int s);                  // output rows per tile (8, or 16 for 5x5 stride-1 layers); tiles are 16 columns wide
int dw_tma_launch(const DwTmaLayer& L, int batch, cudaStream_t stream);

// depthwise3x3(concat(bilinear_x2(low), skip)): TMA-staged low-res tiles for the up-sampled channels plus a
// plain TMA depthwise pass over the skip channels (kps_student.onnx nodes 176-178, 193-195)
struct UpcatTmaLayer {
    CUtensorMap low;
    DwTmaK k;            // C = channels taken from `low`
    int Hl, Wl, chunks, smem_bytes;
    DwTmaLayer skip;
};
bool upcat_tma_supported(const TView& low, const TView& skip, const TView& out);
int upcat_tma_prepare(UpcatTmaLayer& L, const TView& low, const TView& skip, const TView& out, const float* w,
                      const float* bias, int act, int max_batch);
int upcat_tma_launch(const UpcatTmaLayer& L, int batch, cudaStream_t stream);

}  // namespace skps
