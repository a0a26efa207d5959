// The full-resolution head of the landmark encoder as ONE kernel (sm_90a; FP32 pipes + one wgmma K-step for the expansion):
//
//   uint8 crop (H x W x 3)  -> conv_stem 3x3 s2 (+/255, h-swish)                        16 ch @ H/2      [kps_student.onnx
//                           -> blocks.0.0: depthwise 3x3 + ReLU -> 1x1 16->16 + shortcut 16 ch @ H/2       /student/encoder/
//                           -> blocks.1.0: 1x1 16->E + ReLU -> depthwise 3x3 s2 + ReLU   E ch @ H/4        conv_stem .. blocks.1.0/conv_dw]
//
// (timm mobilenetv3 stem + DepthwiseSeparable block + the expand/depthwise half of the first InvertedResidual;
// TRAIN/face_landmark/lib/core/base_trainer/model.py:247-262.)  Run as separate launches these four layers move 3.5 GB
// of 16- and 64-channel full-resolution tensors through HBM per 256-face batch;
// fused, a CTA reads a 39 x 71 pixel window of the crop and writes an 8 x 16 tile of the E-channel quarter-resolution
// tensor, everything in between lives in shared memory.  The work is ~1.2 M FMAs per tile on tensors with 3 / 16 input
// channels.  The stem, the block-0 depthwise and its 16->16 pointwise run on the FP32 pipes with every dense weight taken from
// the kernel-parameter (constant) bank (FFMA with a constant operand, each activation read from shared memory once per 16
// outputs); the 16->E expansion - half of the FMAs - is a single wgmma K-step per 64 window pixels; the next tile's input
// window is prefetched into registers.
//
// Per tile, between CTA-wide barriers: S0 input window -> S1 stem -> S2 block-0 depthwise (warp-uniform channel group) ->
// S3 block-0 pointwise into the fp16 hi/lo A operand -> then, per 16-channel chunk ch of the expansion, one interval that
// issues the wgmma of chunk ch, runs the stride-2 depthwise and output store of chunk ch - 1 while it is in flight, and
// writes chunk ch through bias / ReLU / mask into the other of two chunk buffers.  A tile takes 4 + E / 16 + 1 barriers.
#include <cuda_fp16.h>
#include <string.h>

#include "common.h"
#include "stem_block.h"
#include "tc_ptx.h"

namespace skps {

constexpr int SB_THREADS = 576;
constexpr int SB_TH = 8, SB_TW = 16;                       // output tile (quarter resolution)
constexpr int SB_EH = 2 * SB_TH + 1, SB_EW = 2 * SB_TW + 1;   // 17 x 33: half-resolution window the stride-2 depthwise reads
constexpr int SB_SH = SB_EH + 2, SB_SW = SB_EW + 2;        // 19 x 35: stem outputs the 3x3 depthwise of block 0 reads
constexpr int SB_IH = 2 * SB_SH + 1, SB_IW = 2 * SB_SW + 1;   // 39 x 71: input pixels the stem reads
constexpr int SB_PS = 20;                                  // floats per pixel in shared memory (16 + pad: conflict-free float4 rows)
constexpr int SB_NE = SB_EH * SB_EW, SB_NS = SB_SH * SB_SW, SB_NI = SB_IH * SB_IW;
constexpr int SB_A_FLOATS = (SB_NI * 4 > SB_NE * SB_PS) ? SB_NI * 4 : SB_NE * SB_PS;    // input window, later block-0 depthwise output
constexpr int SB_B_FLOATS = SB_NS * SB_PS;                 // stem output, later the even 16-channel chunks of the expanded tensor
// The 16 -> E expansion (half of the block's FMAs) is ONE wgmma K-step.  S3 writes the block-0 output as float16 hi/lo rows
// (64-byte swizzled rows of which only the first 32 bytes = 16 channels are used), nine 64-row MMA blocks cover the 561
// window pixels (warpgroup 0 takes three, warpgroups 1-3 two each), per 16-channel chunk the accumulators live in
// registers and S4 is wgmma -> bias/ReLU/mask -> shared memory.  Same fp16 hi/lo three-product scheme as conv_tc.cu.
constexpr int SB_T_TILES = (SB_NE + 127) / 128;            // 5
constexpr int SB_T_PLANE = SB_T_TILES * 128 * 64;          // one plane of the A operand: 640 rows x 64 B
constexpr int SB_WB_PLANE = SB_MAX_E * 64;                 // one plane of the B operand: E rows x 64 B
constexpr int SB_SMEM = (SB_A_FLOATS + SB_B_FLOATS + 11 * SB_MAX_E + 256) * 4 + 1024 + 2 * SB_T_PLANE + 2 * SB_WB_PLANE;

// 8 floats -> 16 bytes of float16 hi and 16 bytes of float16 lo (v = hi + lo)
__device__ __forceinline__ void split8(const float* v, uint4& hi, uint4& lo) {
    uint32_t* hp = reinterpret_cast<uint32_t*>(&hi);
    uint32_t* lp = reinterpret_cast<uint32_t*>(&lo);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const __half2 h2 = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
        const float2 hf = __half22float2(h2);
        const __half2 l2 = __floats2half2_rn(v[2 * j] - hf.x, v[2 * j + 1] - hf.y);
        hp[j] = *reinterpret_cast<const uint32_t*>(&h2);
        lp[j] = *reinterpret_cast<const uint32_t*>(&l2);
    }
}

__device__ __forceinline__ float hswish_f(float v) { return v * hsigmoid_f(v); }

// block-0 depthwise: 3 consecutive pixels of one window row x channel group G (weights as constant operands).  Strips of
// 3 tile the 33-pixel row exactly, and 8 lanes on consecutive strips of a row read 8 distinct bank quads (pixel stride 20
// floats, strip stride 60 floats = 7 quads mod 8)
constexpr int SB_STRIP = 3;
template <int G>
__device__ __forceinline__ void dw16_strip(const float* __restrict__ s1, float* __restrict__ s2, int row, int x0, const StemBlockW& Wt) {
    float4 acc[SB_STRIP];
#pragma unroll
    for (int q = 0; q < SB_STRIP; ++q) acc[q] = make_float4(Wt.dw0_b[4 * G], Wt.dw0_b[4 * G + 1], Wt.dw0_b[4 * G + 2], Wt.dw0_b[4 * G + 3]);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        float4 in[SB_STRIP + 2];
#pragma unroll
        for (int i = 0; i < SB_STRIP + 2; ++i)
            in[i] = *reinterpret_cast<const float4*>(s1 + ((row + ky) * SB_SW + x0 + i) * SB_PS + 4 * G);
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int t = ky * 3 + kx;
#pragma unroll
            for (int q = 0; q < SB_STRIP; ++q) {
                acc[q].x = fmaf(in[q + kx].x, Wt.dw0_w[t * 16 + 4 * G], acc[q].x);
                acc[q].y = fmaf(in[q + kx].y, Wt.dw0_w[t * 16 + 4 * G + 1], acc[q].y);
                acc[q].z = fmaf(in[q + kx].z, Wt.dw0_w[t * 16 + 4 * G + 2], acc[q].z);
                acc[q].w = fmaf(in[q + kx].w, Wt.dw0_w[t * 16 + 4 * G + 3], acc[q].w);
            }
        }
    }
#pragma unroll
    for (int q = 0; q < SB_STRIP; ++q) {
        float4 v = acc[q];
        v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
        *reinterpret_cast<float4*>(s2 + (row * SB_EW + x0 + q) * SB_PS + 4 * G) = v;
    }
}

// one 16-output slice of a 1x1 conv on a 16-channel pixel: acc[j] = b[j] + sum_ci x[ci] * w[ci][j] (constant operands)
template <int CO, int OFF>
__device__ __forceinline__ void pw16in(const float* __restrict__ x, const float* w, const float* b, float* acc) {
    float in[16];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        const float4 v = *reinterpret_cast<const float4*>(x + 4 * g);
        in[4 * g] = v.x; in[4 * g + 1] = v.y; in[4 * g + 2] = v.z; in[4 * g + 3] = v.w;
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = b[OFF + j];
#pragma unroll
    for (int ci = 0; ci < 16; ++ci)
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[j] = fmaf(in[ci], w[ci * CO + OFF + j], acc[j]);
}

template <int E>
__global__ void __launch_bounds__(SB_THREADS, 1)
stem_block_kernel(const StemBlockK p, const __grid_constant__ StemBlockW Wt) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float s_wmax[SB_THREADS / 32];
    float* sA = sm;                                    // input window (float4 per pixel: b, g, r, 0), later s2, then odd chunks
    float* sB = sA + SB_A_FLOATS;                      // stem output s1, later the even expanded chunks
    float* sW = sB + SB_B_FLOATS;                      // stride-2 depthwise weights [9][E] + bias [E]
    float* sPB = sW + 10 * SB_MAX_E;                   // expansion bias [E]
    float* lut = sPB + SB_MAX_E;                       // i / 255
    // A operand (block-0 output as fp16 hi/lo rows), then the B operand (expand weights), 1024-byte aligned
    const uint32_t sT = (smem_u32(lut + 256) + 1023u) & ~1023u;
    const uint32_t sWB = sT + 2u * SB_T_PLANE;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < 256; i += SB_THREADS) lut[i] = __fdiv_rn((float)i, 255.f);
    for (int i = tid; i < 10 * E; i += SB_THREADS) sW[i] = p.dw1[i];
    for (int i = tid; i < E; i += SB_THREADS) sPB[i] = Wt.pw1_b[i];
    const int tiles_x = p.Wq / SB_TW, tiles_per_img = tiles_x * (p.Hq / SB_TH);
    const int Hh = p.H / 2, Wh = p.W / 2;              // half-resolution map
    // expand weights -> fp16 hi/lo B operand [E rows][16 K], pre-multiplied by an exact power of two (undone after the
    // MMA) so that the lo parts stay in float16's normal range, as plan.pack_tc_weights does for the other layers
    float wm = 0.f;
    for (int i = tid; i < 16 * E; i += SB_THREADS) wm = fmaxf(wm, fabsf(Wt.pw1_w[i]));
#pragma unroll
    for (int o = 16; o; o >>= 1) wm = fmaxf(wm, __shfl_xor_sync(0xffffffffu, wm, o));
    if (lane == 0) s_wmax[warp] = wm;
    __syncthreads();
    wm = 0.f;
#pragma unroll
    for (int i = 0; i < SB_THREADS / 32; ++i) wm = fmaxf(wm, s_wmax[i]);
    const int s_exp = wm > 0.f ? ilogbf(8192.f / wm) : 0;
    const float w_scale = ldexpf(1.f, s_exp);
    const float w_inv = ldexpf(1.f, -s_exp);
    if (tid < 2 * E) {
        const int co = tid >> 1, c = tid & 1;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = Wt.pw1_w[(8 * c + j) * E + co] * w_scale;
        uint4 hi, lo;
        split8(v, hi, lo);
        const uint32_t a = sWB + (uint32_t)co * 64u + (uint32_t)((c ^ ((co >> 1) & 3)) << 4);
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(hi.x), "r"(hi.y), "r"(hi.z), "r"(hi.w) : "memory");
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a + (uint32_t)SB_WB_PLANE), "r"(lo.x), "r"(lo.y), "r"(lo.z), "r"(lo.w) : "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    // uint8 input: the 39 x 71 window of the NEXT tile is fetched into registers (packed b | g << 8 | r << 16 | valid << 24,
    // 5 pixels per thread) while the current tile is in its expansion / depthwise phases, so S0 never waits on HBM
    constexpr int SB_PRE = (SB_NI + SB_THREADS - 1) / SB_THREADS;
    uint32_t pre[SB_PRE];
    auto prefetch = [&](int tl) {
        const int il = tl / tiles_per_img, tt = tl - il * tiles_per_img;
        const int y0 = 4 * ((tt / tiles_x) * SB_TH) - 5, x0 = 4 * ((tt % tiles_x) * SB_TW) - 5;      // = iy0, ix0 of that tile
        const uint8_t* src = p.in + (long long)(il + p.img0) * p.H * p.W * 3;
#pragma unroll
        for (int k = 0; k < SB_PRE; ++k) {
            const int i = tid + k * SB_THREADS;
            const int r = i / SB_IW, c = i - r * SB_IW, y = y0 + r, x = x0 + c;
            uint32_t v = 0;
            if (i < SB_NI && y >= 0 && y < p.H && x >= 0 && x < p.W) {
                const uint8_t* q = src + ((long long)y * p.W + x) * 3;
                v = (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | (1u << 24);
            }
            pre[k] = v;
        }
    };
    if (!p.in_f32 && (int)blockIdx.x < p.n_tiles) prefetch(blockIdx.x);
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const int img_l = tile / tiles_per_img, t = tile - img_l * tiles_per_img, img = img_l + p.img0;
        const int oy0 = (t / tiles_x) * SB_TH, ox0 = (t % tiles_x) * SB_TW;     // quarter-res origin of the tile
        const int ey0 = 2 * oy0 - 1, ex0 = 2 * ox0 - 1;       // half-res origin of the 17 x 33 window
        const int sy0 = ey0 - 1, sx0 = ex0 - 1;               // half-res origin of the 19 x 35 stem window
        const int iy0 = 2 * sy0 - 1, ix0 = 2 * sx0 - 1;       // input origin of the 39 x 71 window
        // ---- S0: input window, /255 (true division, as numpy does), zero outside the crop (the stem's padding)
        if (p.in_f32) {
            for (int i = tid; i < SB_NI; i += SB_THREADS) {
                const int r = i / SB_IW, c = i - r * SB_IW, y = iy0 + r, x = ix0 + c;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (y >= 0 && y < p.H && x >= 0 && x < p.W) {
                    const long long o = (((long long)img * p.H + y) * p.W + x) * 3;
                    v.x = p.in_f32[o]; v.y = p.in_f32[o + 1]; v.z = p.in_f32[o + 2];
                }
                *reinterpret_cast<float4*>(sA + 4 * i) = v;
            }
        } else {
#pragma unroll
            for (int k = 0; k < SB_PRE; ++k) {
                const int i = tid + k * SB_THREADS;
                if (i < SB_NI) {
                    const uint32_t u = pre[k];
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (u >> 24) { v.x = lut[u & 255u]; v.y = lut[(u >> 8) & 255u]; v.z = lut[(u >> 16) & 255u]; }
                    *reinterpret_cast<float4*>(sA + 4 * i) = v;
                }
            }
        }
        __syncthreads();
        // ---- S1: stem 3x3 stride 2 + h-swish over the 19 x 35 window; item = (pixel, 8 output channels)
        for (int it = tid; it < 2 * ((SB_NS + 31) / 32) * 32; it += SB_THREADS) {
            const int hf = (it >> 5) & 1, px = ((it >> 6) << 5) | (it & 31);       // the channel half is warp-uniform
            if (px >= SB_NS) continue;
            const int r = px / SB_SW, c = px - r * SB_SW;
            float acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = 0.f;
            const int y = sy0 + r, x = sx0 + c;
            const bool inside = y >= 0 && y < Hh && x >= 0 && x < Wh;
            if (inside) {
#pragma unroll
                for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx) {
                        const float4 v = *reinterpret_cast<const float4*>(sA + 4 * ((2 * r + ky) * SB_IW + 2 * c + kx));
                        const int tp = (ky * 3 + kx) * 3;
                        if (hf == 0) {
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                acc[j] = fmaf(v.x, Wt.stem_w[(tp + 0) * 16 + j], acc[j]);
                                acc[j] = fmaf(v.y, Wt.stem_w[(tp + 1) * 16 + j], acc[j]);
                                acc[j] = fmaf(v.z, Wt.stem_w[(tp + 2) * 16 + j], acc[j]);
                            }
                        } else {
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                acc[j] = fmaf(v.x, Wt.stem_w[(tp + 0) * 16 + 8 + j], acc[j]);
                                acc[j] = fmaf(v.y, Wt.stem_w[(tp + 1) * 16 + 8 + j], acc[j]);
                                acc[j] = fmaf(v.z, Wt.stem_w[(tp + 2) * 16 + 8 + j], acc[j]);
                            }
                        }
                    }
                if (hf == 0) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[j] = hswish_f(acc[j] + Wt.stem_b[j]);
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[j] = hswish_f(acc[j] + Wt.stem_b[8 + j]);
                }
            }
            // outside the half-resolution map the tensor is the NEXT conv's zero padding, not stem(padding)
            float* o = sB + px * SB_PS + 8 * hf;
            *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
            *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
        }
        __syncthreads();
        // ---- S2: blocks.0.0 depthwise 3x3 + ReLU over the 17 x 33 window; item = (3-pixel strip, 4-channel group)
        {
            constexpr int STRIPS = SB_EW / SB_STRIP, NSTRIP = SB_EH * STRIPS;     // 11 strips per row, 187 in all
            for (int it = tid; it < 4 * ((NSTRIP + 31) / 32) * 32; it += SB_THREADS) {
                const int g = (it >> 5) & 3, sidx = ((it >> 7) << 5) | (it & 31);    // the channel group is warp-uniform
                if (sidx >= NSTRIP) continue;
                const int row = sidx / STRIPS, x0 = (sidx - row * STRIPS) * SB_STRIP;
                switch (g) {
                    case 0: dw16_strip<0>(sB, sA, row, x0, Wt); break;
                    case 1: dw16_strip<1>(sB, sA, row, x0, Wt); break;
                    case 2: dw16_strip<2>(sB, sA, row, x0, Wt); break;
                    default: dw16_strip<3>(sB, sA, row, x0, Wt); break;
                }
            }
        }
        __syncthreads();
        // ---- S3: blocks.0.0 pointwise 16->16 (linear) + shortcut (the stem output at the same pixel) -> s3
        for (int px = tid; px < SB_NE; px += SB_THREADS) {
            const int r = px / SB_EW, c = px - r * SB_EW;
            float acc[16];
            pw16in<16, 0>(sA + px * SB_PS, Wt.pw0_w, Wt.pw0_b, acc);
            const float* res = sB + ((r + 1) * SB_SW + c + 1) * SB_PS;
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                const float4 rv = *reinterpret_cast<const float4*>(res + 4 * g);
                acc[4 * g] += rv.x; acc[4 * g + 1] += rv.y; acc[4 * g + 2] += rv.z; acc[4 * g + 3] += rv.w;
            }
            // row px of the A operand: logical 16-byte chunk c (8 channels) sits at chunk c ^ ((px / 2) % 4) of the 64-byte row
#pragma unroll
            for (int c2 = 0; c2 < 2; ++c2) {
                uint4 hi, lo;
                split8(acc + 8 * c2, hi, lo);
                const uint32_t a = sT + (uint32_t)px * 64u + (uint32_t)((c2 ^ ((px >> 1) & 3)) << 4);
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(hi.x), "r"(hi.y), "r"(hi.z), "r"(hi.w) : "memory");
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a + (uint32_t)SB_T_PLANE), "r"(lo.x), "r"(lo.y), "r"(lo.z), "r"(lo.w) : "memory");
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        // ---- S4/S5 per 16-channel chunk ch of the expanded tensor: 1x1 16->E + ReLU into xb[ch & 1] (S4), then depthwise
        // 3x3 s2 + ReLU from it to the output (S5).  Warpgroups 0-3 run both; one barrier interval holds S4 of chunk ch and
        // S5 of chunk ch - 1, whose shared-memory reads and FMAs cover the wgmma of chunk ch.  sA (block-0 depthwise output)
        // is dead after S3 and holds the odd chunks.
        if (!p.in_f32 && tile + (int)gridDim.x < p.n_tiles) prefetch(tile + gridDim.x);     // in flight during S4 / S5
        const int y_ok0 = max(0, -ey0), y_ok1 = min(SB_EH, Hh - ey0), x_ok0 = max(0, -ex0), x_ok1 = min(SB_EW, Wh - ex0);
        float* const xb[2] = {sB, sA};
        const int wg = warp >> 2, w = warp & 3;
        // warpgroup wg multiplies the 64-row MMA blocks wg and wg + 4 of the window pixels, warpgroup 0 also block 8
        float acc[3][8];
        auto mma_issue = [&](int ch) {
            const uint64_t b_hi = make_smem_desc_sw64(sWB + (uint32_t)(ch * 16 * 64));
            const uint64_t b_lo = make_smem_desc_sw64(sWB + (uint32_t)SB_WB_PLANE + (uint32_t)(ch * 16 * 64));
            auto blk = [&](float* d, int m) {
                const uint32_t ao = sT + (uint32_t)m * 4096u;
                wg_mma3<16>(d, make_smem_desc_sw64(ao), make_smem_desc_sw64(ao + (uint32_t)SB_T_PLANE), b_hi, b_lo, 0u);
            };
            // straight-line issue per warpgroup role (a branch inside the group would serialise the wgmma)
            if (wg == 0) {
                wg_fence();
                blk(acc[0], 0);
                blk(acc[1], 4);
                blk(acc[2], 8);
                wg_commit();
            } else {
                wg_fence();
                blk(acc[0], wg);
                blk(acc[1], wg + 4);
                wg_commit();
            }
        };
        // accumulator fragment of block m: rows 64m + 16w + lane/4 (+8), columns 8i + 2(lane%4) (+1), written as column pairs
        // through bias / ReLU / mask
        auto epilogue = [&](int ch, float* dst) {
#pragma unroll
            for (int t = 0; t < 3; ++t) {
                if (t == 2 && wg) break;
                const int m = t == 2 ? 8 : wg + 4 * t;
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    const int px = 64 * m + 16 * w + (lane >> 2) + 8 * rr;
                    if (px < SB_NE) {
                        const int r = px / SB_EW, c = px - r * SB_EW;
                        const bool inside = r >= y_ok0 && r < y_ok1 && c >= x_ok0 && c < x_ok1;
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const int co = 8 * i + 2 * (lane & 3);
                            const float2 bb = *reinterpret_cast<const float2*>(sPB + ch * 16 + co);
                            float2 v;
                            v.x = inside ? fmaxf(fmaf(acc[t][4 * i + 2 * rr], w_inv, bb.x), 0.f) : 0.f;
                            v.y = inside ? fmaxf(fmaf(acc[t][4 * i + 2 * rr + 1], w_inv, bb.y), 0.f) : 0.f;
                            *reinterpret_cast<float2*>(dst + px * SB_PS + co) = v;
                        }
                    }
                }
            }
        };
        // depthwise 3x3 stride 2: item = (output pixel, 4-channel group), 128 x 4 = 512 items on warpgroups 0-3.  A quarter
        // warp takes 4 consecutive output columns x 2 groups: 8 distinct bank quads of the 20-float pixel rows.
        auto dw_s2 = [&](int ch, const float* src) {
            const int g = (lane & 1) | ((lane >> 2) & 2);
            const int ocol = ((lane >> 1) & 3) | ((lane >> 2) & 4) | ((warp & 1) << 3), orow = warp >> 1;
            const int c0 = ch * 16 + 4 * g;
            float4 a = *reinterpret_cast<const float4*>(sW + 9 * E + c0);
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float4 v = *reinterpret_cast<const float4*>(src + ((2 * orow + ky) * SB_EW + 2 * ocol + kx) * SB_PS + 4 * g);
                    const float4 wv = *reinterpret_cast<const float4*>(sW + (ky * 3 + kx) * E + c0);
                    a.x = fmaf(v.x, wv.x, a.x); a.y = fmaf(v.y, wv.y, a.y);
                    a.z = fmaf(v.z, wv.z, a.z); a.w = fmaf(v.w, wv.w, a.w);
                }
            a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f);
            const long long o = (((long long)img * p.Hq + oy0 + orow) * p.Wq + ox0 + ocol) * p.out_ld + p.out_coff + c0;
            st4(p.out, p.out_fmt, p.out_plane, o, a);
        };
        if (wg < 4) {
            mma_issue(0);
            wg_wait0();
            wg_fence_acc(acc[0]); wg_fence_acc(acc[1]); wg_fence_acc(acc[2]);
            epilogue(0, xb[0]);
        }
        __syncthreads();
#pragma unroll
        for (int ch = 1; ch < E / 16; ++ch) {
            if (wg < 4) {
                mma_issue(ch);
                dw_s2(ch - 1, xb[(ch - 1) & 1]);
                wg_wait0();
                wg_fence_acc(acc[0]); wg_fence_acc(acc[1]); wg_fence_acc(acc[2]);
                epilogue(ch, xb[ch & 1]);
            }
            __syncthreads();
        }
        if (wg < 4) dw_s2(E / 16 - 1, xb[(E / 16 - 1) & 1]);
        __syncthreads();
    }
}

bool stem_block_supported(int H, int W, int E, const TView& out) {
    if (H % 32 || W % 64 || (E != 64)) return false;          // whole 8 x 16 quarter-resolution tiles; E fixed by the template
    return out.base && out.c_stride == 1 && out.C == E && out.H == H / 4 && out.W == W / 4 && !((out.ld | out.c_off) & 3) &&
           (out.fmt == DT_F32 || out.fmt == DT_SPLIT16);
}

Grid stem_block_grid(const StemBlockK& k, int num_sms) { return persistent_grid(k.n_tiles, num_sms); }

int stem_block_launch(const StemBlockK& k, const StemBlockW& w, int num_sms, cudaStream_t s) {
    static int attr_bytes[MAX_DEVICES] = {};
    if (smem_limit((const void*)stem_block_kernel<64>, attr_bytes, SB_SMEM)) return 1;
    const int grid = stem_block_grid(k, num_sms).ctas;
    stem_block_kernel<64><<<grid, SB_THREADS, SB_SMEM, s>>>(k, w);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace skps
