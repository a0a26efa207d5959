// Fused "A-producer -> pointwise convolution" kernels on wgmma (sm_90a).
//
// The landmark network's 1x1 convolutions are HBM-bound when their input is a 4-6x expanded tensor that an elementwise or
// depthwise kernel has just written and the next one reads back.  Here the A operand of the GEMM
//     C[128 pixels][Cout] = A[128 pixels][K] * W[Cout][K]
// never exists in HBM: transform warps build each 128 x 64 fp16 hi/lo tile in shared memory, in the 128-byte-swizzled
// K-major layout wgmma reads, from a raw tile that TMA staged:
//
//   XF_DW     A = act(depthwise3x3(x))                                 (MobileNetV3 blocks without squeeze-excite:
//             or act(depthwise3x3(concat(bilinear_x2(low), skip)))      conv_dw -> conv_pwl; DecoderBlock heads,
//                                                                       model.py:133-196: Resize -> Concat -> dw -> pw)
//   XF_SCALE  A = x * gate[n, c]                                        (squeeze-excite scale ahead of conv_pwl: replaces
//                                                                       the OP_SCALE_CH pass over the expanded tensor)
//
// Warp roles (512 threads): 0 raw-tile TMA producer, 3 weight-tile TMA producer, 4-7 MMA warpgroup + epilogue (registers ->
// bias/act/residual -> swizzled smem -> TMA store), 8-15 transform.  Three mbarrier rings (raw tiles, A tiles, weight tiles)
// decouple the stages; persistent CTAs, one per SM.
// Output tiles are 16 x 8 pixel blocks (halo 1.4x instead of 2x for row-block tiles); ragged maps hang over the border.
// Precision scheme as conv_tc.cu: fp16 hi/lo operands, three MMAs per K-step, fp32 accumulation in registers.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_xf.h"
#include "tc_ptx.h"

namespace skps {

constexpr int XF_THREADS = 512;
constexpr int XF_TW = 16, XF_TH = 8;                 // output tile
constexpr int XF_IW = XF_TW + 2, XF_IH = XF_TH + 2;  // depthwise input window
constexpr int XF_LW = XF_TW / 2 + 2, XF_LH = XF_TH / 2 + 2;   // low-res window of an up-sampled tile
constexpr int XF_RAW_BYTES = XF_IH * XF_IW * 128;    // 23040: 32 float32 channels (or 2 x 32 float16) per pixel
constexpr int XF_UP_BYTES = XF_LH * XF_LW * 128;     // 7680
// + stencil weights of the up-sampled channels: (3 row classes) x (3 or 4 column classes) x 9 taps x 32 float32 channels
constexpr int XF_A_PLANE = 128 * 128;                // 128 rows x 64 fp16
constexpr int XF_A_BYTES = 2 * XF_A_PLANE;
constexpr int XF_RING = 4;
constexpr int XF_XS_BYTES = 16384;                 // accumulator hand-off buffer of the MMA warpgroup (wg_rows32)
constexpr int XF_ACC_CHUNKS = 8;                   // 32-column accumulator chunks per tile (n_tile <= 256)

__device__ __forceinline__ void split_store4(uint32_t addr_hi, const float4 v) {
    const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
    const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
    const __half2 l01 = __floats2half2_rn(v.x - f01.x, v.y - f01.y), l23 = __floats2half2_rn(v.z - f23.x, v.w - f23.y);
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr_hi), "r"(*reinterpret_cast<const uint32_t*>(&h01)),
                 "r"(*reinterpret_cast<const uint32_t*>(&h23)) : "memory");
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr_hi + (uint32_t)XF_A_PLANE),
                 "r"(*reinterpret_cast<const uint32_t*>(&l01)), "r"(*reinterpret_cast<const uint32_t*>(&l23)) : "memory");
}
__device__ __forceinline__ float4 f4_fma(const float4 a, const float4 w, const float4 c) {
    return make_float4(fmaf(a.x, w.x, c.x), fmaf(a.y, w.y, c.y), fmaf(a.z, w.z, c.z), fmaf(a.w, w.w, c.w));
}
__device__ __forceinline__ float4 f4_mix(const float wa, const float4 a, const float wb, const float4 b) {
    return make_float4(fmaf(wb, b.x, wa * a.x), fmaf(wb, b.y, wa * a.y), fmaf(wb, b.z, wa * a.z), fmaf(wb, b.w, wa * a.w));
}

template <int ACT>
__device__ __forceinline__ void act16(float4* acc) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        acc[q].x = act_t<ACT>(acc[q].x); acc[q].y = act_t<ACT>(acc[q].y);
        acc[q].z = act_t<ACT>(acc[q].z); acc[q].w = act_t<ACT>(acc[q].w);
    }
}

template <int MODE, int ACT, bool OUT_SPLIT>
__global__ void __launch_bounds__(XF_THREADS, 1)
conv_xf_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1_hi,
               const __grid_constant__ CUtensorMap tm1_lo, const __grid_constant__ CUtensorMap tmB_hi,
               const __grid_constant__ CUtensorMap tmB_lo, const __grid_constant__ CUtensorMap tmO_hi,
               const __grid_constant__ CUtensorMap tmO_lo, const __grid_constant__ CUtensorMap tmW,
               const __grid_constant__ XfK p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t raw_full[XF_RING], raw_empty[XF_RING], a_raw[XF_RING], a_full[XF_RING], a_empty[XF_RING],
        b_full[XF_RING], b_empty[XF_RING];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    // weight planes hold n_sub rows rounded up to 32: the 32-column MMA chunks read whole planes (rows past n_sub only feed
    // accumulator columns that are never stored)
    const uint32_t b_plane = (uint32_t)((p.n_sub + 31) & ~31) * 128u, b_slot = 2u * b_plane;
    // [A ring][B ring][epilogue staging][raw ring][depthwise weights]
    const uint32_t a_off = base;
    const uint32_t b_off = a_off + (uint32_t)p.as * XF_A_BYTES;
    const uint32_t o_off = b_off + (uint32_t)p.bs * b_slot;
    const uint32_t r_off = o_off + (uint32_t)p.out_bufs * 16384u;
    const uint32_t w_off = r_off + (MODE == XF_DW ? (uint32_t)p.rs * XF_RAW_BYTES : 0u);
    const int Kpad = p.cchunks * 64;
    const uint32_t xs_off = w_off + (MODE == XF_DW ? (uint32_t)(10 * Kpad * 4) : 0u);

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm0) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm1_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_lo) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < XF_RING; ++s) {
            mbar_init(smem_u32(&raw_full[s]), 1);
            mbar_init(smem_u32(&raw_empty[s]), p.halves ? 4 : 8);   // one arrival per warp that consumes the slot
            mbar_init(smem_u32(&a_raw[s]), 1);
            mbar_init(smem_u32(&a_full[s]), 8);
            mbar_init(smem_u32(&a_empty[s]), 4);              // one arrival per MMA warp
            mbar_init(smem_u32(&b_full[s]), 1);
            mbar_init(smem_u32(&b_empty[s]), 4);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (MODE == XF_DW) {
        // depthwise weights + bias of the whole layer stay in shared memory for the life of the (persistent) CTA
        float* dws = reinterpret_cast<float*>(smem_raw + (w_off - smem_u32(smem_raw)));
        for (int i = threadIdx.x; i < 10 * Kpad; i += XF_THREADS) dws[i] = __ldg(p.dww + i);
    }
    __syncthreads();
    const int total_tiles = p.m_tiles;

    if (warp == 0) {
        // ================================================================== raw-tile / A-tile TMA producer
        if (lane == 0) {
            int st = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int img_l = tile / p.tiles_per_img, t = tile - img_l * p.tiles_per_img;
                const int img = img_l + p.img0;
                const int oy0 = (t / p.tiles_x) * XF_TH, ox0 = (t % p.tiles_x) * XF_TW;
                for (int kc = 0; kc < p.cchunks; ++kc) {
                    if (MODE == XF_SCALE) {
                        mbar_wait_g(smem_u32(&a_empty[st]), ph ^ 1u);
                        const uint32_t fb = smem_u32(&a_raw[st]);
                        mbar_expect_tx(fb, XF_A_BYTES);
                        const uint32_t dst = a_off + (uint32_t)st * XF_A_BYTES;
                        tma_load_4d(dst, &tm1_hi, fb, kc * 64, ox0, oy0, img);
                        tma_load_4d(dst + XF_A_PLANE, &tm1_lo, fb, kc * 64, ox0, oy0, img);
                        if (++st == p.as) { st = 0; ph ^= 1u; }
                    } else {
                        const int subs = p.chunk_subs[kc];
                        for (int h = 0; h < subs; ++h) {
                            const int si = kc * 2 + h, sm = p.sub_mode[si], c = p.sub_c[si];
                            mbar_wait_g(smem_u32(&raw_empty[st]), ph ^ 1u);
                            const uint32_t fb = smem_u32(&raw_full[st]);
                            const uint32_t dst = r_off + (uint32_t)st * XF_RAW_BYTES;
                            if (sm == XS_UP_F32) {
                                // low-res window + the 3 x 3 block of row/column-class stencil weights this tile can need
                                // (classes first|even|odd|last: a tile at the top/left border starts at "first", else at "even")
                                // (a map one tile wide holds first AND last columns: 4 column classes, p.wcx = 4)
                                mbar_expect_tx(fb, XF_UP_BYTES + (uint32_t)p.wcx * 3u * 9u * 128u);
                                tma_load_4d(dst, &tm0, fb, c, (ox0 >> 1) - 1, (oy0 >> 1) - 1, img);
                                tma_load_5d(dst + XF_UP_BYTES, &tmW, fb, 0, 0, (p.wcx == 4 || ox0 == 0) ? 0 : 1, oy0 == 0 ? 0 : 1, c >> 5);
                            } else if (sm == XS_DW_F32) {
                                mbar_expect_tx(fb, XF_RAW_BYTES);
                                tma_load_4d(dst, &tm0, fb, c, ox0 - 1, oy0 - 1, img);
                            } else {
                                mbar_expect_tx(fb, XF_RAW_BYTES);
                                tma_load_4d(dst, &tm1_hi, fb, c, ox0 - 1, oy0 - 1, img);
                                tma_load_4d(dst + XF_RAW_BYTES / 2, &tm1_lo, fb, c, ox0 - 1, oy0 - 1, img);
                            }
                            if (++st == p.rs) { st = 0; ph ^= 1u; }
                        }
                    }
                }
            }
        }
    } else if (warp == 3) {
        // ================================================================== weight-tile TMA producer
        if (lane == 0) {
            int st = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                for (int kc = 0; kc < p.cchunks; ++kc) {
                    for (int nh = 0; nh < p.nsplit; ++nh) {
                        mbar_wait_g(smem_u32(&b_empty[st]), ph ^ 1u);
                        const uint32_t fb = smem_u32(&b_full[st]);
                        mbar_expect_tx(fb, 2u * (uint32_t)p.n_sub * 128u);
                        const uint32_t dst = b_off + (uint32_t)st * b_slot;
                        tma_load_2d(dst, &tmB_hi, fb, kc * 64, nh * p.n_sub);
                        tma_load_2d(dst + b_plane, &tmB_lo, fb, kc * 64, nh * p.n_sub);
                        if (++st == p.bs) { st = 0; ph ^= 1u; }
                    }
                }
            }
        }
    } else if (warp >= 8) {
        // ================================================================== transform warps: raw tile -> A tile
        const int tt = threadIdx.x - 256;
        int ast = 0, rst = 0;
        uint32_t aph = 0, rph = 0;
        if (MODE == XF_SCALE) {
            // thread = physical 16-byte slot (tt & 7) of rows (tt >> 3) + 32 i: its logical 8-channel group is the same in
            // every row it touches (128-byte swizzle: logical = physical ^ (row & 7))
            const int r0 = tt >> 3, ps = tt & 7, j = ps ^ (r0 & 7);
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int img = tile / p.tiles_per_img + p.img0;
                const float* grow = p.gate + (long long)img * p.gate_ld + p.gate_coff;
                for (int kc = 0; kc < p.cchunks; ++kc) {
                    const int c = kc * 64 + j * 8;
                    float g[8];
                    if (c < p.Cin) {
                        const float4 g0 = __ldg(reinterpret_cast<const float4*>(grow + c));
                        const float4 g1 = __ldg(reinterpret_cast<const float4*>(grow + c + 4));
                        g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w; g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
                    } else {
#pragma unroll
                        for (int e = 0; e < 8; ++e) g[e] = 0.f;
                    }
                    mbar_wait_g(smem_u32(&a_raw[ast]), aph);
                    const uint32_t sa = a_off + (uint32_t)ast * XF_A_BYTES + (uint32_t)ps * 16u;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const uint32_t ad = sa + (uint32_t)(r0 + 32 * i) * 128u;
                        uint32_t hv[4], lv[4];
                        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(hv[0]), "=r"(hv[1]), "=r"(hv[2]), "=r"(hv[3]) : "r"(ad) : "memory");
                        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(lv[0]), "=r"(lv[1]), "=r"(lv[2]), "=r"(lv[3]) : "r"(ad + (uint32_t)XF_A_PLANE) : "memory");
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hv[e]));
                            const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lv[e]));
                            const float v0 = (hf.x + lf.x) * g[2 * e], v1 = (hf.y + lf.y) * g[2 * e + 1];
                            const __half2 h2 = __floats2half2_rn(v0, v1);
                            const float2 h2f = __half22float2(h2);
                            const __half2 l2 = __floats2half2_rn(v0 - h2f.x, v1 - h2f.y);
                            hv[e] = *reinterpret_cast<const uint32_t*>(&h2);
                            lv[e] = *reinterpret_cast<const uint32_t*>(&l2);
                        }
                        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(ad), "r"(hv[0]), "r"(hv[1]), "r"(hv[2]), "r"(hv[3]) : "memory");
                        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(ad + (uint32_t)XF_A_PLANE), "r"(lv[0]), "r"(lv[1]), "r"(lv[2]), "r"(lv[3]) : "memory");
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    __syncwarp();
                    if (lane == 0) mbar_arrive(smem_u32(&a_full[ast]));
                    if (++ast == p.as) { ast = 0; aph ^= 1u; }
                }
            }
        } else if (!p.halves) {
            // layers without up-sampled channels: all 256 threads work on one 32-channel sub-chunk at a time,
            // thread = 4 consecutive output pixels of one tile row x 4 channels
            const int cl = tt & 7, pg = tt >> 3, prow = pg >> 2, xs = (pg & 3) * 4;
            const float* dws = reinterpret_cast<const float*>(smem_raw + (w_off - smem_u32(smem_raw)));
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int t = tile % p.tiles_per_img;
                const int oy0 = (t / p.tiles_x) * XF_TH, ox0 = (t % p.tiles_x) * XF_TW;
                const int oy = oy0 + prow, ox = ox0 + xs;
                for (int kc = 0; kc < p.cchunks; ++kc) {
                    mbar_wait_g(smem_u32(&a_empty[ast]), aph ^ 1u);
                    const uint32_t sa = a_off + (uint32_t)ast * XF_A_BYTES;
                    const int subs = p.chunk_subs[kc];
                    for (int h = 0; h < subs; ++h) {
                        const int sm = p.sub_mode[kc * 2 + h];
                        const int cw = kc * 64 + h * 32 + cl * 4;
                        const float4 bias4 = *reinterpret_cast<const float4*>(dws + 9 * Kpad + cw);
                        float4 acc[4] = {bias4, bias4, bias4, bias4};
                        mbar_wait_g(smem_u32(&raw_full[rst]), rph);
                        const uint8_t* raw = smem_raw + (r_off + (uint32_t)rst * XF_RAW_BYTES - smem_u32(smem_raw));
                        {
#pragma unroll
                            for (int ky = 0; ky < 3; ++ky) {
                                float4 in[6];
#pragma unroll
                                for (int i = 0; i < 6; ++i) {
                                    const int px = (prow + ky) * XF_IW + xs + i;
                                    if (sm == XS_DW_F32) {
                                        in[i] = *reinterpret_cast<const float4*>(raw + (px * 32 + cl * 4) * 4);
                                    } else {
                                        const uint2 a = *reinterpret_cast<const uint2*>(raw + (px * 32 + cl * 4) * 2);
                                        const uint2 b = *reinterpret_cast<const uint2*>(raw + XF_RAW_BYTES / 2 + (px * 32 + cl * 4) * 2);
                                        const float2 a01 = __half22float2(*reinterpret_cast<const __half2*>(&a.x));
                                        const float2 a23 = __half22float2(*reinterpret_cast<const __half2*>(&a.y));
                                        const float2 b01 = __half22float2(*reinterpret_cast<const __half2*>(&b.x));
                                        const float2 b23 = __half22float2(*reinterpret_cast<const __half2*>(&b.y));
                                        in[i] = make_float4(a01.x + b01.x, a01.y + b01.y, a23.x + b23.x, a23.y + b23.y);
                                    }
                                }
#pragma unroll
                                for (int kx = 0; kx < 3; ++kx) {
                                    const float4 w = *reinterpret_cast<const float4*>(dws + (ky * 3 + kx) * Kpad + cw);
#pragma unroll
                                    for (int q = 0; q < 4; ++q) acc[q] = f4_fma(in[q + kx], w, acc[q]);
                                }
                            }
                        }
                        // the raw tile has been consumed into registers: hand the slot back to the TMA producer
                        __syncwarp();
                        if (lane == 0) mbar_arrive(smem_u32(&raw_empty[rst]));
                        if (++rst == p.rs) { rst = 0; rph ^= 1u; }
                        // activation, fp16 hi/lo split, store into the swizzled K-major A tile
                        const int jc = h * 4 + (cl >> 1);                    // logical 16-byte chunk of the 128-byte row
                        switch (p.dw_act) {               // one branch per sub-chunk, not one per element
                            case ACT_RELU: act16<ACT_RELU>(acc); break;
                            case ACT_HSWISH: act16<ACT_HSWISH>(acc); break;
                            case ACT_SILU: act16<ACT_SILU>(acc); break;
                            default: break;
                        }
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const float4 v = acc[q];
                            const int r = prow * XF_TW + xs + q;
                            split_store4(sa + (uint32_t)r * 128u + (uint32_t)((jc ^ (r & 7)) << 4) + (uint32_t)(cl & 1) * 8u, v);
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    __syncwarp();
                    if (lane == 0) mbar_arrive(smem_u32(&a_full[ast]));
                    if (++ast == p.as) { ast = 0; aph ^= 1u; }
                }
            }
        } else {
            // The 256 transform threads split into two halves, one per 32-channel sub-chunk of the current 64-channel chunk.
            // A thread = 4 channels x a 2-row x 4-pixel patch of the tile: every staged value it loads feeds several outputs
            // (the first version - one row per thread - was shared-memory-bandwidth bound: l1tex 80 %, 12 LDS.128 per output).
            //   depthwise 3x3      rows (2k, 2k+1): 4 window rows x 6 columns + 9 weights           = 33 loads / 8 outputs
            //   up-sampled stencil rows (r, r+2) of equal parity share their class weights:
            //                      4 low-res rows x 4 columns + 2 column classes x 9 taps             = 34 loads / 8 outputs
            const int half = tt >> 7, t7 = tt & 127;
            const int cl = t7 & 7, pg = t7 >> 3, xs = (pg & 3) * 4, rp = pg >> 2;
            const float* dws = reinterpret_cast<const float*>(smem_raw + (w_off - smem_u32(smem_raw)));
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int t = tile % p.tiles_per_img;
                const int oy0 = (t / p.tiles_x) * XF_TH, ox0 = (t % p.tiles_x) * XF_TW;
                const int ox = ox0 + xs;
                for (int kc = 0; kc < p.cchunks; ++kc) {
                    mbar_wait_g(smem_u32(&a_empty[ast]), aph ^ 1u);
                    const uint32_t sa = a_off + (uint32_t)ast * XF_A_BYTES;
                    const int subs = p.chunk_subs[kc];
                    if (half < subs) {
                        // ring slot of this half's sub-chunk: sub 0 sits at rst, sub 1 one slot further
                        int slot = rst + half;
                        uint32_t sph = rph;
                        if (slot >= p.rs) { slot -= p.rs; sph ^= 1u; }
                        const int sm = p.sub_mode[kc * 2 + half];
                        const int cw = kc * 64 + half * 32 + cl * 4;
                        const float4 bias4 = *reinterpret_cast<const float4*>(dws + 9 * Kpad + cw);
                        float4 acc[2][4] = {{bias4, bias4, bias4, bias4}, {bias4, bias4, bias4, bias4}};
                        int r0, r1;                                       // the two tile rows of this thread
                        mbar_wait_g(smem_u32(&raw_full[slot]), sph);
                        const uint8_t* raw = smem_raw + (r_off + (uint32_t)slot * XF_RAW_BYTES - smem_u32(smem_raw));
                        if (sm == XS_UP_F32) {
                            // depthwise3x3(bilinear_x2(low)) == a 3x3 stencil on the LOW-res window whose weights depend only on
                            // the output pixel's row/column class first|even|odd|last (plan.upcat_effective_weights)
                            r0 = (rp >> 1) * 4 + (rp & 1); r1 = r0 + 2;
                            const int y0 = oy0 + r0, y1 = oy0 + r1;
                            const int ly0 = (oy0 >> 1) - 1, lx0 = (ox0 >> 1) - 1, m = y0 >> 1, c2 = ox >> 1;
                            const int cyb = oy0 == 0 ? 0 : 1, cxb = (p.wcx == 4 || ox0 == 0) ? 0 : 1;
                            const int cyA = (y0 == 0 ? 0 : (y0 == p.H - 1 ? 3 : 1 + (y0 & 1))) - cyb;
                            const int cyB = (y1 == 0 ? 0 : (y1 == p.H - 1 ? 3 : 1 + (y1 & 1))) - cyb;
                            const bool same_cy = cyA == cyB;                  // warp-uniform (one row pair per warp)
                            const bool xfirst = ox == 0, xlast = ox + 4 == p.W;
                            const float* wt = reinterpret_cast<const float*>(raw + XF_UP_BYTES) + cl * 4;
                            const int sE = (1 - cxb) * 9 * 32, sO = (2 - cxb) * 9 * 32, sF = 0, sL = (3 - cxb) * 9 * 32;
                            const float* wA = wt + cyA * p.wcx * 9 * 32;
                            const float* wB = wt + cyB * p.wcx * 9 * 32;
                            int lr[4], lc[4];
#pragma unroll
                            for (int u = 0; u < 4; ++u) lr[u] = min(max(m - 1 + u, 0), p.Hl - 1) - ly0;
#pragma unroll
                            for (int u = 0; u < 4; ++u) lc[u] = min(max(c2 - 1 + u, 0), p.Wl - 1) - lx0;
                            float4 wpE[3], wpO[3];                            // previous tap row's weights (row r1 lags one low row)
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                float4 L[4];
#pragma unroll
                                for (int v = 0; v < 4; ++v)
                                    L[v] = *reinterpret_cast<const float4*>(raw + ((lr[u] * XF_LW + lc[v]) * 32 + cl * 4) * 4);
#pragma unroll
                                for (int v = 0; v < 3; ++v) {
                                    float4 wE = wpE[v], wO = wpO[v];          // (u - 1, v) weights of the shared class
                                    if (u > 0) {                              // row r1: this low row is its tap row a = u - 1
                                        const int o = ((u - 1) * 3 + v) * 32;
                                        if (!same_cy) {
                                            wE = *reinterpret_cast<const float4*>(wB + sE + o);
                                            wO = *reinterpret_cast<const float4*>(wB + sO + o);
                                        }
                                        float4 x0 = wE, x3 = wO;
                                        if (xfirst) x0 = *reinterpret_cast<const float4*>(wB + sF + o);
                                        if (xlast) x3 = *reinterpret_cast<const float4*>(wB + sL + o);
                                        acc[1][0] = f4_fma(L[v], x0, acc[1][0]); acc[1][1] = f4_fma(L[v], wO, acc[1][1]);
                                        acc[1][2] = f4_fma(L[1 + v], wE, acc[1][2]); acc[1][3] = f4_fma(L[1 + v], x3, acc[1][3]);
                                    }
                                    if (u < 3) {                              // row r0: this low row is its tap row a = u
                                        const int o = (u * 3 + v) * 32;
                                        wE = *reinterpret_cast<const float4*>(wA + sE + o);
                                        wO = *reinterpret_cast<const float4*>(wA + sO + o);
                                        float4 x0 = wE, x3 = wO;
                                        if (xfirst) x0 = *reinterpret_cast<const float4*>(wA + sF + o);
                                        if (xlast) x3 = *reinterpret_cast<const float4*>(wA + sL + o);
                                        acc[0][0] = f4_fma(L[v], x0, acc[0][0]); acc[0][1] = f4_fma(L[v], wO, acc[0][1]);
                                        acc[0][2] = f4_fma(L[1 + v], wE, acc[0][2]); acc[0][3] = f4_fma(L[1 + v], x3, acc[0][3]);
                                        wpE[v] = wE; wpO[v] = wO;
                                    }
                                }
                            }
                        } else {
                            r0 = 2 * rp; r1 = r0 + 1;
                            float4 wprev[3];
#pragma unroll
                            for (int u = 0; u < 4; ++u) {                     // window row r0 + u: tap row u of r0, u - 1 of r1
                                float4 in[6];
#pragma unroll
                                for (int i = 0; i < 6; ++i) {
                                    const int px = (r0 + u) * XF_IW + xs + i;
                                    if (sm == XS_DW_F32) {
                                        in[i] = *reinterpret_cast<const float4*>(raw + (px * 32 + cl * 4) * 4);
                                    } else {
                                        const uint2 a = *reinterpret_cast<const uint2*>(raw + (px * 32 + cl * 4) * 2);
                                        const uint2 b = *reinterpret_cast<const uint2*>(raw + XF_RAW_BYTES / 2 + (px * 32 + cl * 4) * 2);
                                        const float2 a01 = __half22float2(*reinterpret_cast<const __half2*>(&a.x));
                                        const float2 a23 = __half22float2(*reinterpret_cast<const __half2*>(&a.y));
                                        const float2 b01 = __half22float2(*reinterpret_cast<const __half2*>(&b.x));
                                        const float2 b23 = __half22float2(*reinterpret_cast<const __half2*>(&b.y));
                                        in[i] = make_float4(a01.x + b01.x, a01.y + b01.y, a23.x + b23.x, a23.y + b23.y);
                                    }
                                }
#pragma unroll
                                for (int kx = 0; kx < 3; ++kx) {
                                    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
                                    if (u < 3) {
                                        w = *reinterpret_cast<const float4*>(dws + (u * 3 + kx) * Kpad + cw);
#pragma unroll
                                        for (int q = 0; q < 4; ++q) acc[0][q] = f4_fma(in[q + kx], w, acc[0][q]);
                                    }
                                    if (u > 0) {
                                        const float4 x = wprev[kx];
#pragma unroll
                                        for (int q = 0; q < 4; ++q) acc[1][q] = f4_fma(in[q + kx], x, acc[1][q]);
                                    }
                                    wprev[kx] = w;
                                }
                            }
                        }
                        // the raw tile has been consumed into registers: hand the slot back to the TMA producer
                        __syncwarp();
                        if (lane == 0) mbar_arrive(smem_u32(&raw_empty[slot]));
                        // activation, fp16 hi/lo split, store into the swizzled K-major A tile
                        switch (p.dw_act) {               // one branch per sub-chunk, not one per element
                            case ACT_RELU: act16<ACT_RELU>(acc[0]); act16<ACT_RELU>(acc[1]); break;
                            case ACT_HSWISH: act16<ACT_HSWISH>(acc[0]); act16<ACT_HSWISH>(acc[1]); break;
                            case ACT_SILU: act16<ACT_SILU>(acc[0]); act16<ACT_SILU>(acc[1]); break;
                            default: break;
                        }
                        const int jc = half * 4 + (cl >> 1);                 // logical 16-byte chunk of the 128-byte row
#pragma unroll
                        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                const int r = (rr ? r1 : r0) * XF_TW + xs + q;
                                split_store4(sa + (uint32_t)r * 128u + (uint32_t)((jc ^ (r & 7)) << 4) + (uint32_t)(cl & 1) * 8u, acc[rr][q]);
                            }
                    }
                    rst += subs;
                    if (rst >= p.rs) { rst -= p.rs; rph ^= 1u; }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    __syncwarp();
                    if (lane == 0) mbar_arrive(smem_u32(&a_full[ast]));
                    if (++ast == p.as) { ast = 0; aph ^= 1u; }
                }
            }
        }
    } else if (warp >= 4) {
        // ================================================================== MMA + epilogue (one warpgroup)
        // accumulator chunk (nh, j) = columns nh * n_sub + 32 j .. of weight slot nh; wg_rows32 hands it over as one pixel
        // row (row = 32q + lane) x 32 columns per thread
        const int q = warp & 3;
        const int row = q * 32 + lane;
        float* xs = reinterpret_cast<float*>(smem_raw + (xs_off - smem_u32(smem_raw)));
        const int cps = (p.n_sub + 31) >> 5;                    // chunks per weight slot
        int ast = 0, bst = 0;
        uint32_t aph = 0, bph = 0;
        int store_i = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            float accv[XF_ACC_CHUNKS][32];
            for (int kc = 0; kc < p.cchunks; ++kc) {
                mbar_wait_g(smem_u32(&a_full[ast]), aph);
                const uint32_t sa = a_off + (uint32_t)ast * XF_A_BYTES;
                const uint64_t a_hi = make_smem_desc(sa), a_lo = make_smem_desc(sa + XF_A_PLANE);
                const int ksteps = p.chunk_ksteps[kc];
                for (int nh = 0; nh < p.nsplit; ++nh) {
                    mbar_wait_g(smem_u32(&b_full[bst]), bph);
                    const uint32_t sb = b_off + (uint32_t)bst * b_slot;
                    const uint64_t b_hi = make_smem_desc(sb), b_lo = make_smem_desc(sb + b_plane);
                    wg_fence();
#pragma unroll
                    for (int c = 0; c < XF_ACC_CHUNKS; ++c) {
                        if (c < nh * cps || c >= (nh + 1) * cps) continue;
                        const uint64_t bo = (uint64_t)((c - nh * cps) * 32 * 128 >> 4);
                        for (int k = 0; k < ksteps; ++k) {
                            const uint64_t koff = (uint64_t)(k * 32 >> 4);
                            wg_mma3_128x32(accv[c], a_hi + koff, a_lo + koff, 64u * 128u, b_hi + bo + koff, b_lo + bo + koff,
                                           (kc | k) != 0);
                        }
                    }
                    wg_commit();
                    wg_wait0();
                    if (lane == 0) mbar_arrive(smem_u32(&b_empty[bst]));
                    if (++bst == p.bs) { bst = 0; bph ^= 1u; }
                }
                if (lane == 0) mbar_arrive(smem_u32(&a_empty[ast]));
                if (++ast == p.as) { ast = 0; aph ^= 1u; }
            }
            const int img_l = tile / p.tiles_per_img, t = tile - img_l * p.tiles_per_img, img = img_l + p.img0;
            const int ty0 = (t / p.tiles_x) * XF_TH, tx0 = (t % p.tiles_x) * XF_TW;
            const int y = ty0 + row / XF_TW, x = tx0 + row % XF_TW;
            const bool row_ok = y < p.H && x < p.W;
            const long long pix = row_ok ? ((long long)img * p.H + y) * p.W + x : 0;
#pragma unroll 1
            for (int c = 0; c < p.nsplit * cps; ++c) {
                const int nh = c / cps, c0 = nh * p.n_sub + (c - nh * cps) * 32;
                if (c0 >= p.Cout) break;
                float v[32];
#pragma unroll
                for (int o = 0; o < XF_ACC_CHUNKS; ++o)
                    if (o == c) wg_rows32(accv[o], xs, 2, q, lane, v);
                const int nvalid = min(min(32, (nh + 1) * p.n_sub - c0), p.Cout - c0);
                const long long o_el = pix * p.out_ld + p.out_coff + c0;
                const long long r_el = pix * p.res_ld + p.res_coff + c0;
                if (p.tma_store && (nvalid == 32 || c0 + nvalid == p.Cout)) {
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        float* w = v + 8 * g;
                        if (8 * g < nvalid) {
                            const float4* b4 = reinterpret_cast<const float4*>(p.bias + c0 + 8 * g);
                            epilogue8<ACT>(w, __ldg(b4), __ldg(b4 + 1), p, r_el + 8 * g);
                        }
                    }
                    const uint32_t sbuf = o_off + (uint32_t)(store_i % p.out_bufs) * 16384u;
                    if (q == 0 && lane == 0) {
                        if (p.out_bufs == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                        else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    }
                    ++store_i;
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                    if (OUT_SPLIT) {
                        const uint32_t rh = sbuf + (uint32_t)row * 64u, rl = rh + 8192u;
#pragma unroll
                        for (int g = 0; g < 4; ++g) {
                            uint32_t hp[4], lp[4];
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const float a0 = v[8 * g + 2 * j], a1 = v[8 * g + 2 * j + 1];
                                const __half2 h2 = __floats2half2_rn(a0, a1);
                                const float2 hf = __half22float2(h2);
                                const __half2 l2 = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
                                hp[j] = *reinterpret_cast<const uint32_t*>(&h2);
                                lp[j] = *reinterpret_cast<const uint32_t*>(&l2);
                            }
                            const uint32_t slot = (uint32_t)((g ^ (row >> 1)) & 3) * 16u;          // 64-byte swizzle
                            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(rh + slot), "r"(hp[0]), "r"(hp[1]), "r"(hp[2]), "r"(hp[3]) : "memory");
                            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(rl + slot), "r"(lp[0]), "r"(lp[1]), "r"(lp[2]), "r"(lp[3]) : "memory");
                        }
                    } else {
                        const uint32_t rf = sbuf + (uint32_t)row * 128u;
#pragma unroll
                        for (int g = 0; g < 8; ++g) {
                            const uint32_t slot = (uint32_t)((g ^ row) & 7) * 16u;                 // 128-byte swizzle
                            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(rf + slot), "f"(v[4 * g]), "f"(v[4 * g + 1]), "f"(v[4 * g + 2]), "f"(v[4 * g + 3]) : "memory");
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                    if (q == 0 && lane == 0) {
                        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                     ::"l"(&tmO_hi), "r"(sbuf), "r"(c0), "r"(tx0), "r"(ty0), "r"(img) : "memory");
                        if (OUT_SPLIT)
                            asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                         ::"l"(&tmO_lo), "r"(sbuf + 8192u), "r"(c0), "r"(tx0), "r"(ty0), "r"(img) : "memory");
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    }
                    continue;
                }
                if (p.out_cstride != 1 && (nvalid & 7) == 0) {
                    // Strided destination (the detector's ShuffleNetV2 units write straight into channel-shuffled views,
                    // c_stride 2).  A lane owns a pixel, so a direct store instruction would touch 32 different sectors with
                    // 2-4 bytes each (several times the kernel's own work).  The 32 x 32 block is
                    // transposed through this warp's 4 KB staging slice (XOR-swizzled, conflict-free both ways) and stored
                    // pixel by pixel with lane = channel: 4 sectors per instruction.
                    #pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        float* w = v + 8 * g;
                        if (8 * g < nvalid) {
                            const float4* b4 = reinterpret_cast<const float4*>(p.bias + c0 + 8 * g);
                            epilogue8<ACT>(w, __ldg(b4), __ldg(b4 + 1), p, r_el + 8 * g);
                        }
                    }
                    float* xs = reinterpret_cast<float*>(smem_raw + (o_off - smem_u32(smem_raw))) + (warp - 4) * 1024;
                    __syncwarp();
#pragma unroll
                    for (int j = 0; j < 32; ++j) xs[lane * 32 + (j ^ lane)] = v[j];
                    __syncwarp();
                    const int pix_lo = (int)(pix & 0xffffffffll), pix_hi = (int)(pix >> 32);
#pragma unroll 4
                    for (int i = 0; i < 32; ++i) {
                        const bool ok_i = __shfl_sync(0xffffffffu, (int)row_ok, i) != 0;
                        const long long pix_i = ((long long)__shfl_sync(0xffffffffu, pix_hi, i) << 32) |
                                                (unsigned int)__shfl_sync(0xffffffffu, pix_lo, i);
                        if (ok_i && lane < nvalid)
                            st1(p.out, OUT_SPLIT ? DT_SPLIT16 : DT_F32, p.out_plane,
                                pix_i * p.out_ld + p.out_coff + (long long)(c0 + lane) * p.out_cstride, xs[i * 32 + (lane ^ i)]);
                    }
                    __syncwarp();
                    continue;
                }
                if (!row_ok) continue;
                const bool fast = (nvalid & 7) == 0 && p.out_cstride == 1 && ((p.out_ld | (p.out_coff + c0)) & 7) == 0;
                if (fast) {
                    const int ng = nvalid >> 3;
                    const float4* b4 = reinterpret_cast<const float4*>(p.bias + c0);
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        if (g < ng) {
                            float* w = v + 8 * g;
                            epilogue8<ACT>(w, __ldg(b4 + 2 * g), __ldg(b4 + 2 * g + 1), p, r_el + 8 * g);
                            float8 o8;
#pragma unroll
                            for (int j = 0; j < 8; ++j) o8.v[j] = w[j];
                            st8(p.out, OUT_SPLIT ? DT_SPLIT16 : DT_F32, p.out_plane, o_el + 8 * g, o8);
                        }
                    }
                } else {
#pragma unroll 1
                    for (int j = 0; j < nvalid; ++j) {
                        float f = fmaf(v_at(v, j), p.out_scale, __ldg(p.bias + c0 + j));
                        const float r = p.res ? ld1(p.res, p.res_fmt, p.res_plane, r_el + j) : 0.f;
                        f = p.res_first ? act_t<ACT>(f + r) : act_t<ACT>(f) + r;
                        st1(p.out, OUT_SPLIT ? DT_SPLIT16 : DT_F32, p.out_plane,
                            pix * p.out_ld + p.out_coff + (long long)(c0 + j) * p.out_cstride, f);
                    }
                }
            }
        }
        if (p.tma_store && q == 0 && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

// ------------------------------------------------------------------------------------------ host side
static const float* xf_zero_bias() {
    static float* z = nullptr;
    if (!z) {
        if (cudaMalloc(&z, 1024 * sizeof(float)) != cudaSuccess) return nullptr;
        cudaMemset(z, 0, 1024 * sizeof(float));
    }
    return z;
}

static bool view_ok8(const TView& v) { return v.base && v.c_stride == 1 && !((v.C | v.ld | v.c_off) & 7); }

bool xf_supported(const XfSetup& s) {
    if (s.n_tiles != 1 || s.n_tile > 256 || (s.n_tile & 15) || s.Cout > s.n_tile) return false;
    if (!s.out.base || s.out.H < XF_TH || s.out.W < XF_TW) return false;
    if (s.mode == XF_SCALE) {
        if (!view_ok8(s.x) || s.x.fmt != DT_SPLIT16 || !s.gate.base || s.gate.fmt != DT_F32 || s.gate.c_stride != 1) return false;
        if ((s.gate.ld | s.gate.c_off) & 3) return false;
        return s.x.H == s.out.H && s.x.W == s.out.W && (s.x.C + 63) / 64 <= XF_MAX_CHUNKS;
    }
    if (!view_ok8(s.x) || (s.x.fmt != DT_F32 && s.x.fmt != DT_SPLIT16)) return false;
    if (s.x.H != s.out.H || s.x.W != s.out.W) return false;
    int K = s.x.C;
    if (s.low.base) {
        if (!view_ok8(s.low) || s.low.fmt != DT_F32 || s.x.fmt != DT_SPLIT16 || !s.weff) return false;   // one float32 source map per layer
        if (s.low.C % 64 || s.out.H != 2 * s.low.H || s.out.W != 2 * s.low.W) return false;
        if (s.out.H % XF_TH || s.out.W % XF_TW || s.out.H < 2 * XF_TH) return false;     // no tile holds first AND last rows
        K += s.low.C;
    }
    return (K + 63) / 64 <= XF_MAX_CHUNKS;
}

static int encode4(EncodeTiledFn enc, CUtensorMap* m, const TView& v, int plane, int max_batch, int box_c, int box_w, int box_h,
                   CUtensorMapSwizzle swz) {
    const bool split = v.fmt == DT_SPLIT16;
    const int esz = split ? 2 : 4;
    cuuint64_t dims[4] = {(cuuint64_t)v.C, (cuuint64_t)v.W, (cuuint64_t)v.H, (cuuint64_t)max_batch};
    cuuint64_t strides[3] = {(cuuint64_t)v.ld * esz, (cuuint64_t)v.W * v.ld * esz, (cuuint64_t)v.H * v.W * v.ld * esz};
    cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    char* base = (char*)v.base + (size_t)v.c_off * esz + (plane ? (size_t)v.plane * 2 : 0);
    CUresult r = enc(m, split ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, dims, strides, box,
                     estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    SKPS_CHECK(r == CUDA_SUCCESS, "conv_xf: cuTensorMapEncodeTiled failed: %d", (int)r);
    return 0;
}

int xf_prepare(XfLayer& L, const XfSetup& s) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    SKPS_CHECK(xf_supported(s), "conv_xf: unsupported layer");
    memset(&L.k, 0, sizeof(L.k));
    XfK& k = L.k;
    L.mode = s.mode;
    const TView& out = s.out;
    k.H = out.H; k.W = out.W;
    k.tiles_x = (out.W + XF_TW - 1) / XF_TW;
    k.tiles_per_img = k.tiles_x * ((out.H + XF_TH - 1) / XF_TH);
    const int Cu = s.low.base ? s.low.C : 0;
    k.Cin = Cu + s.x.C;
    k.cchunks = (k.Cin + 63) / 64;
    k.n_tile = s.n_tile;
    k.nsplit = s.n_tile > 128 ? 2 : 1;
    if (k.nsplit == 2 && (s.n_tile % 32)) k.nsplit = 1;          // halves must stay multiples of 16
    k.n_sub = s.n_tile / k.nsplit;
    k.dw_act = s.dw_act;
    k.halves = s.low.base ? 1 : 0;
    k.Hl = s.low.base ? s.low.H : 0; k.Wl = s.low.base ? s.low.W : 0;
    for (int kc = 0; kc < k.cchunks; ++kc) {
        const int valid = k.Cin - kc * 64 < 64 ? k.Cin - kc * 64 : 64;
        k.chunk_subs[kc] = valid <= 32 ? 1 : 2;
        k.chunk_ksteps[kc] = (uint8_t)((valid + 15) / 16);
        for (int h = 0; h < 2; ++h) {
            const int c = kc * 64 + h * 32;
            if (c < Cu) { k.sub_mode[kc * 2 + h] = XS_UP_F32; k.sub_c[kc * 2 + h] = (int16_t)c; }
            else { k.sub_mode[kc * 2 + h] = s.x.fmt == DT_SPLIT16 ? XS_DW_SPLIT : XS_DW_F32; k.sub_c[kc * 2 + h] = (int16_t)(c - Cu); }
        }
    }
    k.dww = s.dww;
    if (s.mode == XF_SCALE) {
        k.gate = (const float*)s.gate.base; k.gate_ld = s.gate.ld; k.gate_coff = s.gate.c_off;
    }
    // tensor maps
    L.src0 = CUtensorMap(); L.src1_hi = CUtensorMap(); L.src1_lo = CUtensorMap();
    if (s.mode == XF_SCALE) {
        if (encode4(enc, &L.src1_hi, s.x, 0, s.max_batch, 64, XF_TW, XF_TH, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
        if (encode4(enc, &L.src1_lo, s.x, 1, s.max_batch, 64, XF_TW, XF_TH, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
        L.src0 = L.src1_hi;
    } else {
        if (s.low.base) {
            if (encode4(enc, &L.src0, s.low, 0, s.max_batch, 32, XF_LW, XF_LH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
        }
        if (s.x.fmt == DT_SPLIT16) {
            if (encode4(enc, &L.src1_hi, s.x, 0, s.max_batch, 32, XF_IW, XF_IH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
            if (encode4(enc, &L.src1_lo, s.x, 1, s.max_batch, 32, XF_IW, XF_IH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
            if (!s.low.base) L.src0 = L.src1_hi;
        } else {
            if (encode4(enc, &L.src0, s.x, 0, s.max_batch, 32, XF_IW, XF_IH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
            L.src1_hi = L.src0; L.src1_lo = L.src0;
        }
    }
    L.w_eff = L.src0;
    if (s.low.base) {
        // [sub][cy 4][cx 4][tap 9][32 ch] float32; a tile takes the 3 x 3 classes it can contain
        cuuint64_t dims[5] = {32, 9, 4, 4, (cuuint64_t)(s.low.C / 32)};
        cuuint64_t strides[4] = {128, 9 * 128, 4 * 9 * 128, 16 * 9 * 128};
        k.wcx = k.tiles_x == 1 ? 4 : 3;
        cuuint32_t box[5] = {32, 9, (cuuint32_t)k.wcx, 3, 1};
        cuuint32_t estr[5] = {1, 1, 1, 1, 1};
        CUresult r = enc(&L.w_eff, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, (void*)s.weff, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "conv_xf: cuTensorMapEncodeTiled(weff) failed: %d", (int)r);
    }
    const int K_pad = k.cchunks * 64;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)K_pad, (cuuint64_t)s.n_tile};
        cuuint64_t strides[1] = {(cuuint64_t)K_pad * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)k.n_sub};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(plane ? &L.b_lo : &L.b_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)(plane ? s.w_lo : s.w_hi), dims,
                         strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "conv_xf: cuTensorMapEncodeTiled(B) failed: %d", (int)r);
    }
    const int oes = out.fmt == DT_SPLIT16 ? 2 : 4;
    k.tma_store = (out.c_stride == 1 && (s.Cout % 8) == 0 && ((size_t)out.ld * oes) % 16 == 0 &&
                   ((size_t)out.c_off * oes) % 16 == 0) ? 1 : 0;
    if (k.tma_store) {
        for (int plane = 0; plane < (out.fmt == DT_SPLIT16 ? 2 : 1); ++plane) {
            cuuint64_t dims[4] = {(cuuint64_t)s.Cout, (cuuint64_t)out.W, (cuuint64_t)out.H, (cuuint64_t)s.max_batch};
            cuuint64_t strides[3] = {(cuuint64_t)out.ld * oes, (cuuint64_t)out.W * out.ld * oes,
                                     (cuuint64_t)out.H * out.W * out.ld * oes};
            cuuint32_t box[4] = {32, XF_TW, XF_TH, 1};
            cuuint32_t estr[4] = {1, 1, 1, 1};
            char* base = (char*)out.base + (size_t)out.c_off * oes + (plane ? (size_t)out.plane * 2 : 0);
            CUresult r = enc(plane ? &L.o_lo : &L.o_hi,
                             out.fmt == DT_SPLIT16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base,
                             dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             out.fmt == DT_SPLIT16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            SKPS_CHECK(r == CUDA_SUCCESS, "conv_xf: cuTensorMapEncodeTiled(out) failed: %d", (int)r);
        }
        if (out.fmt != DT_SPLIT16) L.o_lo = L.o_hi;
    } else {
        L.o_hi = L.b_hi; L.o_lo = L.b_hi;
    }
    // shared-memory budget: minimal rings first, then spend what is left on depth
    const size_t budget = 227 * 1024 - 1024 - 512 - XF_XS_BYTES;
    const size_t b_slot = (size_t)((k.n_sub + 31) & ~31) * 256;
    const size_t w_bytes = s.mode == XF_DW ? (size_t)10 * K_pad * 4 : 0;
    k.as = 2; k.bs = 2; k.rs = s.mode == XF_DW ? 2 : 0; k.out_bufs = 1;
    auto total = [&]() { return (size_t)k.as * XF_A_BYTES + (size_t)k.bs * b_slot + (size_t)k.out_bufs * 16384 +
                                (size_t)k.rs * XF_RAW_BYTES + w_bytes; };
    SKPS_CHECK(total() <= budget, "conv_xf: layer does not fit shared memory (%zu bytes)", total());
    // two halves consume two raw slots at once: a third slot is what lets the TMA producer run ahead
    if (s.mode == XF_DW) { k.rs = 3; if (total() > budget) k.rs = 2; }
    if (k.tma_store) { k.out_bufs = 2; if (total() > budget) k.out_bufs = 1; }     // the store of chunk i drains under chunk i+1
    k.bs = 3; if (total() > budget) k.bs = 2;
    if (s.mode == XF_DW && k.rs == 3) { k.rs = 4; if (total() > budget) k.rs = 3; }
    k.as = 3; if (total() > budget) k.as = 2;
    if (k.bs == 3) { k.bs = 4; if (total() > budget) k.bs = 3; }
    L.smem_bytes = (int)(total() + XF_XS_BYTES + 1024);
    k.Cout = s.Cout; k.act = s.act; k.out_scale = s.out_scale;
    k.bias = s.bias ? s.bias : xf_zero_bias();
    SKPS_CHECK(k.bias, "conv_xf: zero-bias allocation failed");
    k.out = out.base; k.out_fmt = out.fmt; k.out_plane = out.plane; k.out_ld = out.ld; k.out_coff = out.c_off;
    k.out_cstride = out.c_stride;
    k.res = s.res.base; k.res_fmt = s.res.fmt; k.res_plane = s.res.plane; k.res_ld = s.res.ld; k.res_coff = s.res.c_off;
    k.res_first = s.res.base ? s.res_first : 0;
    L.valid = true;
    return 0;
}

template <int MODE, int ACT, bool SPLIT>
static int xf_launch_t(const XfLayer& L, const XfK& k, int grid, cudaStream_t stream) {
    static bool attr_set = false;
    if (!attr_set) {
        SKPS_CUDA(cudaFuncSetAttribute(conv_xf_kernel<MODE, ACT, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       227 * 1024 - 1024));
        attr_set = true;
    }
    conv_xf_kernel<MODE, ACT, SPLIT><<<grid, XF_THREADS, L.smem_bytes, stream>>>(L.src0, L.src1_hi, L.src1_lo, L.b_hi, L.b_lo,
                                                                                  L.o_hi, L.o_lo, L.w_eff, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

template <int MODE>
static int xf_launch_m(const XfLayer& L, const XfK& k, int grid, cudaStream_t stream) {
    const bool sp = k.out_fmt == DT_SPLIT16;
    switch (k.act) {
        case ACT_NONE: return sp ? xf_launch_t<MODE, ACT_NONE, true>(L, k, grid, stream) : xf_launch_t<MODE, ACT_NONE, false>(L, k, grid, stream);
        case ACT_RELU: return sp ? xf_launch_t<MODE, ACT_RELU, true>(L, k, grid, stream) : xf_launch_t<MODE, ACT_RELU, false>(L, k, grid, stream);
        case ACT_HSWISH: return sp ? xf_launch_t<MODE, ACT_HSWISH, true>(L, k, grid, stream) : xf_launch_t<MODE, ACT_HSWISH, false>(L, k, grid, stream);
        case ACT_SILU: return sp ? xf_launch_t<MODE, ACT_SILU, true>(L, k, grid, stream) : xf_launch_t<MODE, ACT_SILU, false>(L, k, grid, stream);
        default: break;
    }
    set_error("conv_xf: activation %d not instantiated", k.act);
    return 1;
}

int xf_launch(const XfLayer& L, int batch, int num_sms, cudaStream_t stream) {
    XfK k = L.k;
    k.m_tiles = batch * k.tiles_per_img;
    k.img_end = batch;
    const int grid = k.m_tiles < num_sms ? k.m_tiles : num_sms;
    return L.mode == XF_SCALE ? xf_launch_m<XF_SCALE>(L, k, grid, stream) : xf_launch_m<XF_DW>(L, k, grid, stream);
}

}  // namespace skps

using namespace skps;

namespace {
__global__ void xf_f32_to_split(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = src[i];
    const __half h = __float2half_rn(v);
    hi[i] = h;
    lo[i] = __float2half_rn(v - __half2float(h));
}
struct DevBuf {
    void* p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    int alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 16) == cudaSuccess ? 0 : 1; }
};
}  // namespace

// Debug/unit-test entry: one fused layer on host data (tests/test_conv_xf_gpu.py).
//   mode 0 (XF_SCALE): out = act(conv1x1(x * gate[n,c]) ...)            x (N,H,W,Cx) float32, gate (N,Cx)
//   mode 1 (XF_DW)   : out = act(conv1x1(dw_act(dw3x3(concat(up2(low), x)))))   low (N,H/2,W/2,Cl) or null
//   x_split: the kernel reads x as fp16 hi/lo planes (else float32; XF_SCALE always splits)
//   dww: [9][Kpad] depthwise weights then [Kpad] bias, Kpad = ceil((Cl+Cx)/64)*64 (XF_DW)
//   w_hi/w_lo: (n_tile, Kpad) float16 as packed by plan.pack_tc_weights; residual (N,H,W,Cout) float32 or null
//   weff: [Cl/32][4][4][9][32] class weights of the up-sampled channels (plan.pack_upcat_class_weights), null without low
extern "C" SKPS_API int skps_debug_conv_xf(int mode, const float* x, int N, int H, int W, int Cx, int x_split,
                                           const float* low, int Cl, const float* gate, const float* dww, int dw_act,
                                           const void* w_hi, const void* w_lo, const float* bias, int Cout, int act,
                                           int n_tile, float out_scale, const float* residual, int res_first,
                                           int out_split, float* out, const float* weff) {
    SKPS_CHECK(x && w_hi && w_lo && out && N > 0, "debug_conv_xf: null argument");
    const int K = Cx + (low ? Cl : 0), Kpad = (K + 63) / 64 * 64;
    const long long nx = (long long)N * H * W * Cx, nl = low ? (long long)N * (H / 2) * (W / 2) * Cl : 0;
    const long long nout = (long long)N * H * W * Cout;
    const bool xs = x_split || mode == XF_SCALE;
    DevBuf dx, dxs, dl, dg, dw, dwh, dwl, db, dr, dout, dwe;
    SKPS_CHECK(!dx.alloc(nx * 4) && !dxs.alloc(nx * 4) && !dl.alloc(nl * 4) && !dg.alloc((size_t)N * Cx * 4) &&
               !dw.alloc((size_t)10 * Kpad * 4) && !dwh.alloc((size_t)n_tile * Kpad * 2) && !dwl.alloc((size_t)n_tile * Kpad * 2) &&
               !db.alloc((size_t)Cout * 4) && !dr.alloc(nout * 4) && !dout.alloc(nout * 4), "debug_conv_xf: cudaMalloc failed");
    SKPS_CUDA(cudaMemcpy(dx.p, x, nx * 4, cudaMemcpyHostToDevice));
    if (xs) {
        xf_f32_to_split<<<(unsigned)((nx + 255) / 256), 256>>>((const float*)dx.p, (__half*)dxs.p, (__half*)dxs.p + nx, nx);
        SKPS_CUDA(cudaGetLastError());
    }
    if (low) SKPS_CUDA(cudaMemcpy(dl.p, low, nl * 4, cudaMemcpyHostToDevice));
    if (low) {
        SKPS_CHECK(weff && Cl % 32 == 0 && !dwe.alloc((size_t)Cl * 144 * 4), "debug_conv_xf: class weights");
        SKPS_CUDA(cudaMemcpy(dwe.p, weff, (size_t)Cl * 144 * 4, cudaMemcpyHostToDevice));
    }
    if (gate) SKPS_CUDA(cudaMemcpy(dg.p, gate, (size_t)N * Cx * 4, cudaMemcpyHostToDevice));
    if (dww) SKPS_CUDA(cudaMemcpy(dw.p, dww, (size_t)10 * Kpad * 4, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(dwh.p, w_hi, (size_t)n_tile * Kpad * 2, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(dwl.p, w_lo, (size_t)n_tile * Kpad * 2, cudaMemcpyHostToDevice));
    if (bias) SKPS_CUDA(cudaMemcpy(db.p, bias, (size_t)Cout * 4, cudaMemcpyHostToDevice));
    if (residual) SKPS_CUDA(cudaMemcpy(dr.p, residual, nout * 4, cudaMemcpyHostToDevice));
    auto view = [&](void* base, int C, int h, int w, int fmt, long long plane) {
        TView t;
        memset(&t, 0, sizeof(t));
        t.base = base; t.ld = C; t.c_off = 0; t.c_stride = 1; t.C = C; t.H = h; t.W = w;
        t.sample = (long long)C * h * w; t.fmt = fmt; t.plane = plane;
        return t;
    };
    XfSetup s;
    memset(&s, 0, sizeof(s));
    s.mode = mode; s.max_batch = N;
    s.x = xs ? view(dxs.p, Cx, H, W, DT_SPLIT16, nx) : view(dx.p, Cx, H, W, DT_F32, 0);
    if (low) s.low = view(dl.p, Cl, H / 2, W / 2, DT_F32, 0);
    if (gate) s.gate = view(dg.p, Cx, 1, 1, DT_F32, 0);
    s.dww = (const float*)dw.p; s.dw_act = dw_act; s.weff = low ? (const float*)dwe.p : nullptr;
    s.Cout = Cout; s.act = act; s.n_tile = n_tile; s.n_tiles = 1; s.out_scale = out_scale;
    s.w_hi = dwh.p; s.w_lo = dwl.p; s.bias = bias ? (const float*)db.p : nullptr;
    s.out = view(dout.p, Cout, H, W, out_split ? DT_SPLIT16 : DT_F32, nout);
    if (residual) s.res = view(dr.p, Cout, H, W, DT_F32, 0);
    s.res_first = res_first;
    XfLayer L;
    if (xf_prepare(L, s)) return 1;
    const int sms = sm_count();
    if (xf_launch(L, N, sms, 0)) return 1;
    SKPS_CUDA(cudaDeviceSynchronize());
    if (out_split) {
        __half* tmp = (__half*)malloc(nout * 4);
        SKPS_CUDA(cudaMemcpy(tmp, dout.p, nout * 4, cudaMemcpyDeviceToHost));
        for (long long i = 0; i < nout; ++i) out[i] = __half2float(tmp[i]) + __half2float(tmp[nout + i]);
        free(tmp);
    } else {
        SKPS_CUDA(cudaMemcpy(out, dout.p, nout * 4, cudaMemcpyDeviceToHost));
    }
    return 0;
}
