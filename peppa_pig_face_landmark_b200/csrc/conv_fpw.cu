// The student's fused "A-producer -> pointwise convolution" layers on wgmma with the accumulators in registers (sm_90a).
//
// Same layers and the same A producers as conv_xf.cu: the A operand of
//     C[128 pixels][N] = A[128 pixels][K] * W[N][K]
// is built in shared memory by transform warps, in the 128-byte-swizzled K-major fp16 hi/lo layout wgmma reads:
//
//   XF_DW     A = dw_act(depthwise3x3(x)), x float32 or split-fp16,
//             or depthwise3x3(concat(bilinear_x2(low), skip)) through the row/column-class stencil weights
//   XF_SCALE  A = x * gate[n, c] on a split-fp16 x
//
// What differs from conv_xf is the MMA side.  conv_xf's MMA warpgroup keeps a 128 x 256 accumulator whatever the layer's
// width and issues m64n32 chunks from loops bounded at run time, so ptxas serialises every wgmma and spills the accumulator.
// Here the unit width N is a template parameter of at most 64 output channels: the MMA warpgroup holds exactly N fp32
// accumulators per thread for its 128 x N unit and issues m64nNk16 wgmma from straight-line code, one K-chunk's group kept
// in flight while the next is issued (as conv_pw.cu).  ptxas sizes wgmma accumulators against the launch's 128 registers per
// thread (512 threads, one CTA per SM), setmaxnreg notwithstanding, so a wider layer runs as nsplit units of 64 channels per pixel tile (N tile 80 or 112 or 128 -> 2 units, 160 -> 3, 256 -> 4).
// Each unit re-stages the tile and recomputes the A producer; the units of one tile are consecutive, so persistent CTAs
// run them side by side and the re-reads hit L2.
//
// Warp roles (512 threads, one persistent CTA per SM):
//   0      TMA producer: per K-chunk the weight tile, then the raw tile(s) (XF_DW) or the A tile (XF_SCALE)
//   1-3    idle after set-up; warps 0-3 drop to 32 registers each (setmaxnreg)
//   4-7    MMA + epilogue warpgroup, raised to 160 registers
//   8-15   transform warps: raw tile -> A tile (conv_xf's code), raised to 160 registers
// The epilogue works straight from the accumulator fragment: fmaf(acc, out_scale, bias), residual, activation, then the
// split-fp16 hi/lo or float32 value into a swizzled 16 KB staging buffer per 32-channel slab, which leaves as one TMA store
// per plane: a 32-channel x 16 x 8 pixel box in the output buffer's channel window.  Images past the batch are never
// touched.  While the MMA warpgroup runs an epilogue, the producer and the transform warps fill the rings for its next unit.
// Precision: the fp16 hi/lo operands, K order, three-product order and epilogue expressions of conv_xf, so the outputs are
// bit-identical to it.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_fpw.h"
#include "tc_ptx.h"

namespace skps {

constexpr int FPW_THREADS = 512;
constexpr int FPW_TW = 16, FPW_TH = 8;                    // output tile
constexpr int FPW_IW = FPW_TW + 2, FPW_IH = FPW_TH + 2;   // depthwise input window
constexpr int FPW_LW = FPW_TW / 2 + 2, FPW_LH = FPW_TH / 2 + 2;   // low-res window of an up-sampled tile
constexpr int FPW_RAW_BYTES = FPW_IH * FPW_IW * 128;      // 23040: 32 float32 channels (or 2 x 32 float16) per pixel
constexpr int FPW_UP_BYTES = FPW_LH * FPW_LW * 128;       // 7680
constexpr int FPW_A_PLANE = 128 * 128;                    // 128 rows x 64 fp16
constexpr int FPW_A_BYTES = 2 * FPW_A_PLANE;
constexpr int FPW_RING = 4;
constexpr int FPW_OUT_BUF = 16384;                        // one 32-channel slab of 128 pixels, hi + lo or float32
// setmaxnreg: warps 0-3 give 4 x 32 x (128 - 32) registers; the transform warps take 8 x 32 x (160 - 128) and the MMA
// warpgroup 4 x 32 x (160 - 128) of them
constexpr int FPW_PRODUCER_REGS = 32, FPW_TRANSFORM_REGS = 160, FPW_MMA_REGS = 160;
static_assert(128 * FPW_PRODUCER_REGS + 256 * FPW_TRANSFORM_REGS + 128 * FPW_MMA_REGS <= 65536, "register file split");

__device__ __forceinline__ void fpw_split_store4(uint32_t addr_hi, const float4 v) {
    const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
    const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
    const __half2 l01 = __floats2half2_rn(v.x - f01.x, v.y - f01.y), l23 = __floats2half2_rn(v.z - f23.x, v.w - f23.y);
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr_hi), "r"(*reinterpret_cast<const uint32_t*>(&h01)),
                 "r"(*reinterpret_cast<const uint32_t*>(&h23)) : "memory");
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr_hi + (uint32_t)FPW_A_PLANE),
                 "r"(*reinterpret_cast<const uint32_t*>(&l01)), "r"(*reinterpret_cast<const uint32_t*>(&l23)) : "memory");
}
__device__ __forceinline__ float4 fpw_f4_fma(const float4 a, const float4 w, const float4 c) {
    return make_float4(fmaf(a.x, w.x, c.x), fmaf(a.y, w.y, c.y), fmaf(a.z, w.z, c.z), fmaf(a.w, w.w, c.w));
}

template <int ACT>
__device__ __forceinline__ void fpw_act16(float4* acc) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        acc[q].x = act_t<ACT>(acc[q].x); acc[q].y = act_t<ACT>(acc[q].y);
        acc[q].z = act_t<ACT>(acc[q].z); acc[q].w = act_t<ACT>(acc[q].w);
    }
}

// two fp32 values of channels i, i + 1 (i even) of a float32 or split-fp16 tensor; same sums as ld1 / ld4
__device__ __forceinline__ float2 fpw_ld2(const void* base, int fmt, long long plane, long long i) {
    if (fmt == DT_SPLIT16) {
        const __half* h = (const __half*)base;
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(h + i));
        const float2 b = __half22float2(*reinterpret_cast<const __half2*>(h + i + plane));
        return make_float2(a.x + b.x, a.y + b.y);
    }
    return *reinterpret_cast<const float2*>((const float*)base + i);
}

// KS K-steps of 16 of the three-product scheme on a 128 x N accumulator held by one warpgroup: acc[0..N/2) = pixel rows
// 0-63, acc[N/2..N) = rows 64-127 (row 64 of the A tile at +8 KB).  Per element the order of conv_xf's wg_mma3_128x32:
// lo*hi, hi*lo, hi*hi for each K-step.
template <int N, int KS>
__device__ __forceinline__ void fpw_mma(float* acc, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                        uint32_t accumulate) {
    constexpr uint64_t A_HALF = 64 * 128 >> 4;
#pragma unroll
    for (int k = 0; k < KS; ++k) {
        const uint64_t koff = (uint64_t)(k * 32 >> 4);     // 16 fp16 = 32 bytes along K
#pragma unroll
        for (int m = 0; m < 2; ++m)
            wg_mma3<N>(acc + (N / 2) * m, a_hi + m * A_HALF + koff, a_lo + m * A_HALF + koff, b_hi + koff, b_lo + koff,
                       k ? 1u : accumulate);
    }
}

template <int MODE, int N, int ACT, bool OUT_SPLIT>
__global__ void __launch_bounds__(FPW_THREADS, 1)
conv_fpw_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1_hi,
                const __grid_constant__ CUtensorMap tm1_lo, const __grid_constant__ CUtensorMap tmB_hi,
                const __grid_constant__ CUtensorMap tmB_lo, const __grid_constant__ CUtensorMap tmO_hi,
                const __grid_constant__ CUtensorMap tmO_lo, const __grid_constant__ CUtensorMap tmW,
                const __grid_constant__ FpwK p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t raw_full[FPW_RING], raw_empty[FPW_RING], a_raw[FPW_RING], a_full[FPW_RING],
        a_empty[FPW_RING], b_full[FPW_RING], b_empty[FPW_RING];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t b_plane = (uint32_t)N * 128u, b_slot = 2u * b_plane;
    // [A ring][B ring][epilogue staging][raw ring][depthwise weights]
    const uint32_t a_off = base;
    const uint32_t b_off = a_off + (uint32_t)p.as * FPW_A_BYTES;
    const uint32_t o_off = b_off + (uint32_t)p.bs * b_slot;
    const uint32_t r_off = o_off + (uint32_t)p.out_bufs * FPW_OUT_BUF;
    const uint32_t w_off = r_off + (MODE == XF_DW ? (uint32_t)p.rs * FPW_RAW_BYTES : 0u);
    const int Kpad = p.cchunks * 64;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm0) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tm1_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_lo) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < FPW_RING; ++s) {
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
        for (int i = threadIdx.x; i < 10 * Kpad; i += FPW_THREADS) dws[i] = __ldg(p.dww + i);
    }
    __syncthreads();
    // Registers: the launch gives every thread 128 (65536 / 512).  The producer warpgroup (warps 0-3) needs few, so it drops
    // to FPW_PRODUCER_REGS and the transform warps and the MMA warpgroup take what it frees.  The unit width stays <= 64:
    // ptxas sizes the wgmma accumulators against the launch's 128 registers whatever setmaxnreg grants, and serialises
    // wider units (C7511 / C7512).
    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(FPW_PRODUCER_REGS));
    if (warp == 0) {
        // ================================================================== TMA producer
        // One thread, K-chunk by K-chunk: the weight tile, then the raw tile(s) or the A tile.  Every ring is consumed in
        // this order, so a wait on one ring's slot only ever depends on loads already issued.
        if (lane == 0) {
            int st = 0, bst = 0;
            uint32_t ph = 0, bph = 0;
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                const int tile = u / p.nsplit, nh = u - tile * p.nsplit;
                const int img = tile / p.tiles_per_img, t = tile - img * p.tiles_per_img;
                const int oy0 = (t / p.tiles_x) * FPW_TH, ox0 = (t % p.tiles_x) * FPW_TW;
                for (int kc = 0; kc < p.cchunks; ++kc) {
                    {
                        mbar_wait_g(smem_u32(&b_empty[bst]), bph ^ 1u);
                        const uint32_t fb = smem_u32(&b_full[bst]);
                        mbar_expect_tx(fb, b_slot);
                        const uint32_t dst = b_off + (uint32_t)bst * b_slot;
                        tma_load_2d(dst, &tmB_hi, fb, kc * 64, nh * N);
                        tma_load_2d(dst + b_plane, &tmB_lo, fb, kc * 64, nh * N);
                        if (++bst == p.bs) { bst = 0; bph ^= 1u; }
                    }
                    if (MODE == XF_SCALE) {
                        mbar_wait_g(smem_u32(&a_empty[st]), ph ^ 1u);
                        const uint32_t fb = smem_u32(&a_raw[st]);
                        mbar_expect_tx(fb, FPW_A_BYTES);
                        const uint32_t dst = a_off + (uint32_t)st * FPW_A_BYTES;
                        tma_load_4d(dst, &tm1_hi, fb, kc * 64, ox0, oy0, img);
                        tma_load_4d(dst + FPW_A_PLANE, &tm1_lo, fb, kc * 64, ox0, oy0, img);
                        if (++st == p.as) { st = 0; ph ^= 1u; }
                    } else {
                        const int subs = p.chunk_subs[kc];
                        for (int h = 0; h < subs; ++h) {
                            const int si = kc * 2 + h, sm = p.sub_mode[si], c = p.sub_c[si];
                            mbar_wait_g(smem_u32(&raw_empty[st]), ph ^ 1u);
                            const uint32_t fb = smem_u32(&raw_full[st]);
                            const uint32_t dst = r_off + (uint32_t)st * FPW_RAW_BYTES;
                            if (sm == XS_UP_F32) {
                                // low-res window + the 3 x 3 block of row/column-class stencil weights this tile can need
                                // (classes first|even|odd|last: a tile at the top/left border starts at "first", else at "even")
                                // (a map one tile wide holds first AND last columns: 4 column classes, p.wcx = 4)
                                mbar_expect_tx(fb, FPW_UP_BYTES + (uint32_t)p.wcx * 3u * 9u * 128u);
                                tma_load_4d(dst, &tm0, fb, c, (ox0 >> 1) - 1, (oy0 >> 1) - 1, img);
                                tma_load_5d(dst + FPW_UP_BYTES, &tmW, fb, 0, 0, (p.wcx == 4 || ox0 == 0) ? 0 : 1, oy0 == 0 ? 0 : 1, c >> 5);
                            } else if (sm == XS_DW_F32) {
                                mbar_expect_tx(fb, FPW_RAW_BYTES);
                                tma_load_4d(dst, &tm0, fb, c, ox0 - 1, oy0 - 1, img);
                            } else {
                                mbar_expect_tx(fb, FPW_RAW_BYTES);
                                tma_load_4d(dst, &tm1_hi, fb, c, ox0 - 1, oy0 - 1, img);
                                tma_load_4d(dst + FPW_RAW_BYTES / 2, &tm1_lo, fb, c, ox0 - 1, oy0 - 1, img);
                            }
                            if (++st == p.rs) { st = 0; ph ^= 1u; }
                        }
                    }
                }
            }
        }
    }
    } else if (warp >= 8) {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(FPW_TRANSFORM_REGS));
        // ================================================================== transform warps: raw tile -> A tile
        const int tt = threadIdx.x - 256;
        int ast = 0, rst = 0;
        uint32_t aph = 0, rph = 0;
        if (MODE == XF_SCALE) {
            // thread = physical 16-byte slot (tt & 7) of rows (tt >> 3) + 32 i: its logical 8-channel group is the same in
            // every row it touches (128-byte swizzle: logical = physical ^ (row & 7))
            const int r0 = tt >> 3, ps = tt & 7, j = ps ^ (r0 & 7);
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                const int tile = u / p.nsplit;
                const int img = tile / p.tiles_per_img;
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
                    const uint32_t sa = a_off + (uint32_t)ast * FPW_A_BYTES + (uint32_t)ps * 16u;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const uint32_t ad = sa + (uint32_t)(r0 + 32 * i) * 128u;
                        uint32_t hv[4], lv[4];
                        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(hv[0]), "=r"(hv[1]), "=r"(hv[2]), "=r"(hv[3]) : "r"(ad) : "memory");
                        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(lv[0]), "=r"(lv[1]), "=r"(lv[2]), "=r"(lv[3]) : "r"(ad + (uint32_t)FPW_A_PLANE) : "memory");
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
                        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(ad + (uint32_t)FPW_A_PLANE), "r"(lv[0]), "r"(lv[1]), "r"(lv[2]), "r"(lv[3]) : "memory");
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
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                for (int kc = 0; kc < p.cchunks; ++kc) {
                    mbar_wait_g(smem_u32(&a_empty[ast]), aph ^ 1u);
                    const uint32_t sa = a_off + (uint32_t)ast * FPW_A_BYTES;
                    const int subs = p.chunk_subs[kc];
                    for (int h = 0; h < subs; ++h) {
                        const int sm = p.sub_mode[kc * 2 + h];
                        const int cw = kc * 64 + h * 32 + cl * 4;
                        const float4 bias4 = *reinterpret_cast<const float4*>(dws + 9 * Kpad + cw);
                        float4 acc[4] = {bias4, bias4, bias4, bias4};
                        mbar_wait_g(smem_u32(&raw_full[rst]), rph);
                        const uint8_t* raw = smem_raw + (r_off + (uint32_t)rst * FPW_RAW_BYTES - smem_u32(smem_raw));
                        {
#pragma unroll
                            for (int ky = 0; ky < 3; ++ky) {
                                float4 in[6];
#pragma unroll
                                for (int i = 0; i < 6; ++i) {
                                    const int px = (prow + ky) * FPW_IW + xs + i;
                                    if (sm == XS_DW_F32) {
                                        in[i] = *reinterpret_cast<const float4*>(raw + (px * 32 + cl * 4) * 4);
                                    } else {
                                        const uint2 a = *reinterpret_cast<const uint2*>(raw + (px * 32 + cl * 4) * 2);
                                        const uint2 b = *reinterpret_cast<const uint2*>(raw + FPW_RAW_BYTES / 2 + (px * 32 + cl * 4) * 2);
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
                                    for (int q = 0; q < 4; ++q) acc[q] = fpw_f4_fma(in[q + kx], w, acc[q]);
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
                            case ACT_RELU: fpw_act16<ACT_RELU>(acc); break;
                            case ACT_HSWISH: fpw_act16<ACT_HSWISH>(acc); break;
                            case ACT_SILU: fpw_act16<ACT_SILU>(acc); break;
                            default: break;
                        }
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const float4 v = acc[q];
                            const int r = prow * FPW_TW + xs + q;
                            fpw_split_store4(sa + (uint32_t)r * 128u + (uint32_t)((jc ^ (r & 7)) << 4) + (uint32_t)(cl & 1) * 8u, v);
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
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                const int tile = u / p.nsplit;
                const int t = tile % p.tiles_per_img;
                const int oy0 = (t / p.tiles_x) * FPW_TH, ox0 = (t % p.tiles_x) * FPW_TW;
                const int ox = ox0 + xs;
                for (int kc = 0; kc < p.cchunks; ++kc) {
                    mbar_wait_g(smem_u32(&a_empty[ast]), aph ^ 1u);
                    const uint32_t sa = a_off + (uint32_t)ast * FPW_A_BYTES;
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
                        const uint8_t* raw = smem_raw + (r_off + (uint32_t)slot * FPW_RAW_BYTES - smem_u32(smem_raw));
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
                            const float* wt = reinterpret_cast<const float*>(raw + FPW_UP_BYTES) + cl * 4;
                            const int sE = (1 - cxb) * 9 * 32, sO = (2 - cxb) * 9 * 32, sF = 0, sL = (3 - cxb) * 9 * 32;
                            const float* wA = wt + cyA * p.wcx * 9 * 32;
                            const float* wB = wt + cyB * p.wcx * 9 * 32;
                            int lr[4], lc[4];
#pragma unroll
                            for (int j = 0; j < 4; ++j) lr[j] = min(max(m - 1 + j, 0), p.Hl - 1) - ly0;
#pragma unroll
                            for (int j = 0; j < 4; ++j) lc[j] = min(max(c2 - 1 + j, 0), p.Wl - 1) - lx0;
                            float4 wpE[3], wpO[3];                            // previous tap row's weights (row r1 lags one low row)
#pragma unroll
                            for (int wr = 0; wr < 4; ++wr) {
                                float4 L[4];
#pragma unroll
                                for (int v = 0; v < 4; ++v)
                                    L[v] = *reinterpret_cast<const float4*>(raw + ((lr[wr] * FPW_LW + lc[v]) * 32 + cl * 4) * 4);
#pragma unroll
                                for (int v = 0; v < 3; ++v) {
                                    float4 wE = wpE[v], wO = wpO[v];          // (wr - 1, v) weights of the shared class
                                    if (wr > 0) {                              // row r1: this low row is its tap row a = wr - 1
                                        const int o = ((wr - 1) * 3 + v) * 32;
                                        if (!same_cy) {
                                            wE = *reinterpret_cast<const float4*>(wB + sE + o);
                                            wO = *reinterpret_cast<const float4*>(wB + sO + o);
                                        }
                                        float4 x0 = wE, x3 = wO;
                                        if (xfirst) x0 = *reinterpret_cast<const float4*>(wB + sF + o);
                                        if (xlast) x3 = *reinterpret_cast<const float4*>(wB + sL + o);
                                        acc[1][0] = fpw_f4_fma(L[v], x0, acc[1][0]); acc[1][1] = fpw_f4_fma(L[v], wO, acc[1][1]);
                                        acc[1][2] = fpw_f4_fma(L[1 + v], wE, acc[1][2]); acc[1][3] = fpw_f4_fma(L[1 + v], x3, acc[1][3]);
                                    }
                                    if (wr < 3) {                              // row r0: this low row is its tap row a = wr
                                        const int o = (wr * 3 + v) * 32;
                                        wE = *reinterpret_cast<const float4*>(wA + sE + o);
                                        wO = *reinterpret_cast<const float4*>(wA + sO + o);
                                        float4 x0 = wE, x3 = wO;
                                        if (xfirst) x0 = *reinterpret_cast<const float4*>(wA + sF + o);
                                        if (xlast) x3 = *reinterpret_cast<const float4*>(wA + sL + o);
                                        acc[0][0] = fpw_f4_fma(L[v], x0, acc[0][0]); acc[0][1] = fpw_f4_fma(L[v], wO, acc[0][1]);
                                        acc[0][2] = fpw_f4_fma(L[1 + v], wE, acc[0][2]); acc[0][3] = fpw_f4_fma(L[1 + v], x3, acc[0][3]);
                                        wpE[v] = wE; wpO[v] = wO;
                                    }
                                }
                            }
                        } else {
                            r0 = 2 * rp; r1 = r0 + 1;
                            float4 wprev[3];
#pragma unroll
                            for (int wr = 0; wr < 4; ++wr) {                     // window row r0 + wr: tap row wr of r0, wr - 1 of r1
                                float4 in[6];
#pragma unroll
                                for (int i = 0; i < 6; ++i) {
                                    const int px = (r0 + wr) * FPW_IW + xs + i;
                                    if (sm == XS_DW_F32) {
                                        in[i] = *reinterpret_cast<const float4*>(raw + (px * 32 + cl * 4) * 4);
                                    } else {
                                        const uint2 a = *reinterpret_cast<const uint2*>(raw + (px * 32 + cl * 4) * 2);
                                        const uint2 b = *reinterpret_cast<const uint2*>(raw + FPW_RAW_BYTES / 2 + (px * 32 + cl * 4) * 2);
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
                                    if (wr < 3) {
                                        w = *reinterpret_cast<const float4*>(dws + (wr * 3 + kx) * Kpad + cw);
#pragma unroll
                                        for (int q = 0; q < 4; ++q) acc[0][q] = fpw_f4_fma(in[q + kx], w, acc[0][q]);
                                    }
                                    if (wr > 0) {
                                        const float4 x = wprev[kx];
#pragma unroll
                                        for (int q = 0; q < 4; ++q) acc[1][q] = fpw_f4_fma(in[q + kx], x, acc[1][q]);
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
                            case ACT_RELU: fpw_act16<ACT_RELU>(acc[0]); fpw_act16<ACT_RELU>(acc[1]); break;
                            case ACT_HSWISH: fpw_act16<ACT_HSWISH>(acc[0]); fpw_act16<ACT_HSWISH>(acc[1]); break;
                            case ACT_SILU: fpw_act16<ACT_SILU>(acc[0]); fpw_act16<ACT_SILU>(acc[1]); break;
                            default: break;
                        }
                        const int jc = half * 4 + (cl >> 1);                 // logical 16-byte chunk of the 128-byte row
#pragma unroll
                        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                const int r = (rr ? r1 : r0) * FPW_TW + xs + q;
                                fpw_split_store4(sa + (uint32_t)r * 128u + (uint32_t)((jc ^ (r & 7)) << 4) + (uint32_t)(cl & 1) * 8u, acc[rr][q]);
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
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(FPW_MMA_REGS));
        // acc[(N/2) m + 4 i + e] = pixel row 64m + 16q + lane/4 + 8(e/2) of the tile (row = 16 y + x), channel
        // 8i + 2(lane%4) + e%2 of the unit
        const int q = warp & 3;
        const bool leader = q == 0 && lane == 0;       // issues and drains the warpgroup's TMA stores
        int ast = 0, bst = 0;
        uint32_t aph = 0, bph = 0;
        int store_i = 0;                               // TMA stores issued so far
        for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
            const int tile = u / p.nsplit, nh = u - tile * p.nsplit;
            float acc[N];
            int prev_a = 0, prev_b = 0;
            for (int kc = 0; kc < p.cchunks; ++kc) {
                mbar_wait_g(smem_u32(&a_full[ast]), aph);
                mbar_wait_g(smem_u32(&b_full[bst]), bph);
                const uint32_t sa = a_off + (uint32_t)ast * FPW_A_BYTES, sb = b_off + (uint32_t)bst * b_slot;
                const uint64_t a_hi = make_smem_desc(sa), a_lo = make_smem_desc(sa + FPW_A_PLANE);
                const uint64_t b_hi = make_smem_desc(sb), b_lo = make_smem_desc(sb + b_plane);
                const uint32_t accumulate = kc != 0;
                wg_fence_acc(acc);
                switch (p.chunk_ksteps[kc]) {          // uniform over the CTA
                    case 4: wg_fence(); fpw_mma<N, 4>(acc, a_hi, a_lo, b_hi, b_lo, accumulate); wg_commit(); break;
                    case 3: wg_fence(); fpw_mma<N, 3>(acc, a_hi, a_lo, b_hi, b_lo, accumulate); wg_commit(); break;
                    case 2: wg_fence(); fpw_mma<N, 2>(acc, a_hi, a_lo, b_hi, b_lo, accumulate); wg_commit(); break;
                    default: wg_fence(); fpw_mma<N, 1>(acc, a_hi, a_lo, b_hi, b_lo, accumulate); wg_commit(); break;
                }
                wg_fence_acc(acc);
                // keep this chunk's group in flight; the previous one has finished reading its A and B slots
                wg_wait<1>();
                wg_fence_acc(acc);
                if (kc > 0 && lane == 0) {
                    mbar_arrive(smem_u32(&a_empty[prev_a]));
                    mbar_arrive(smem_u32(&b_empty[prev_b]));
                }
                prev_a = ast; prev_b = bst;
                if (++ast == p.as) { ast = 0; aph ^= 1u; }
                if (++bst == p.bs) { bst = 0; bph ^= 1u; }
            }
            wg_wait<0>();
            wg_fence_acc(acc);
            if (lane == 0) {
                mbar_arrive(smem_u32(&a_empty[prev_a]));
                mbar_arrive(smem_u32(&b_empty[prev_b]));
            }
            const int img = tile / p.tiles_per_img, t = tile - img * p.tiles_per_img;
            const int ty0 = (t / p.tiles_x) * FPW_TH, tx0 = (t % p.tiles_x) * FPW_TW;
            const long long pix0 = ((long long)img * p.H + ty0) * p.W + tx0;      // pixel index of the tile's row 0
#pragma unroll
            for (int s = 0; s < (N + 31) / 32; ++s) {
                const int co = nh * N + 32 * s;                 // first output channel of the slab
                if (co >= p.Cout) break;                        // uniform: slabs past Cout hold zero-weight columns
                // staging buffer of this slab: the store issued out_bufs slabs ago from it must have finished reading it
                const uint32_t sbuf = o_off + (uint32_t)(store_i % p.out_bufs) * FPW_OUT_BUF;
                if (leader) {
                    if (p.out_bufs == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                    else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                }
                ++store_i;
                asm volatile("bar.sync 1, 128;" ::: "memory");
                float bias[8];                                  // channels co + 8i + 2(lane%4) + j, i < 4, j < 2
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const int c = co + 8 * i + 2 * (lane & 3) + j;
                        bias[2 * i + j] = c < p.Cout ? __ldg(p.bias + c) : 0.f;
                    }
#pragma unroll
                for (int m = 0; m < 2; ++m)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int r = 64 * m + 16 * q + (lane >> 2) + 8 * h;      // pixel row of the tile
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            if (32 * s + 8 * i >= N) continue;                   // columns past the unit (N % 32 == 16)
                            const float* a = acc + (N / 2) * m + 4 * (4 * s + i) + 2 * h;
                            float v0 = fmaf(a[0], p.out_scale, bias[2 * i]);
                            float v1 = fmaf(a[1], p.out_scale, bias[2 * i + 1]);
                            if (p.res && co + 8 * i < p.Cout) {
                                const long long pix = pix0 + (r / FPW_TW) * p.W + r % FPW_TW;
                                const float2 rv = fpw_ld2(p.res, p.res_fmt, p.res_plane,
                                                          pix * p.res_ld + p.res_coff + co + 8 * i + 2 * (lane & 3));
                                if (p.res_first) { v0 = act_t<ACT>(v0 + rv.x); v1 = act_t<ACT>(v1 + rv.y); }
                                else { v0 = act_t<ACT>(v0) + rv.x; v1 = act_t<ACT>(v1) + rv.y; }
                            } else {
                                v0 = act_t<ACT>(v0); v1 = act_t<ACT>(v1);
                            }
                            if (OUT_SPLIT) {
                                // rows of 64 B per plane, [hi 8 KB][lo 8 KB]; 64-byte swizzle: 16-byte chunk ^= (r/2) % 4
                                const __half2 h2 = __floats2half2_rn(v0, v1);
                                const float2 hf = __half22float2(h2);
                                const __half2 l2 = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
                                const uint32_t addr = sbuf + (uint32_t)r * 64u + (uint32_t)((i ^ (r >> 1)) & 3) * 16u +
                                                      (uint32_t)(lane & 3) * 4u;
                                asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(*reinterpret_cast<const uint32_t*>(&h2)) : "memory");
                                asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr + 8192u), "r"(*reinterpret_cast<const uint32_t*>(&l2)) : "memory");
                            } else {
                                // rows of 128 B; 128-byte swizzle: 16-byte chunk ^= r % 8
                                const uint32_t addr = sbuf + (uint32_t)r * 128u +
                                                      (uint32_t)(((2 * i + ((lane & 3) >> 1)) ^ r) & 7) * 16u +
                                                      (uint32_t)(lane & 1) * 8u;
                                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v0), "f"(v1) : "memory");
                            }
                        }
                    }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                asm volatile("bar.sync 1, 128;" ::: "memory");
                if (leader) {
                    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                 ::"l"(&tmO_hi), "r"(sbuf), "r"(co), "r"(tx0), "r"(ty0), "r"(img) : "memory");
                    if (OUT_SPLIT)
                        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                     ::"l"(&tmO_lo), "r"(sbuf + 8192u), "r"(co), "r"(tx0), "r"(ty0), "r"(img) : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

// ------------------------------------------------------------------------------------------ host side
// Output channels per work unit (the kernel's N) for an N tile: the tile itself up to 64 channels, else units of 64.  Every
// unit but the last is then two whole 32-channel slabs, so no unit's TMA store box reaches into the next unit's channels;
// the last unit's columns past the N tile have zero weights and its stores clip at Cout.  The student's layers: XF_DW 32,
// 80 -> 2 x 64, 128 -> 2 x 64, 256 -> 4 x 64; XF_SCALE 48, 112 -> 2 x 64, 160 -> 3 x 64.  0 for a width not instantiated.
static int fpw_unit_width(int mode, int n_tile) {
    const int n = n_tile <= 64 ? n_tile : 64;
    if (mode == XF_DW) return n == 32 || n == 64 ? n : 0;
    return n == 48 || n == 64 ? n : 0;
}

constexpr int FPW_MAX_DEVICES = 64;

// zeros standing in for a missing bias, one allocation per device
static const float* fpw_zero_bias() {
    static float* z[FPW_MAX_DEVICES] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= FPW_MAX_DEVICES) return nullptr;
    if (!z[dev]) {
        if (cudaMalloc(&z[dev], 1024 * sizeof(float)) != cudaSuccess) { z[dev] = nullptr; return nullptr; }
        if (cudaMemset(z[dev], 0, 1024 * sizeof(float)) != cudaSuccess) return nullptr;
    }
    return z[dev];
}

// shared-memory rings of a layer: minimal first, then spend what is left on depth (conv_xf's order, without its 16 KB
// accumulator hand-off buffer)
static size_t fpw_rings(FpwK& k, int mode, int n) {
    const size_t budget = 227 * 1024 - 1024 - 512;
    const size_t b_slot = (size_t)n * 256;
    const size_t w_bytes = mode == XF_DW ? (size_t)10 * k.cchunks * 64 * 4 : 0;
    k.as = 2; k.bs = 2; k.rs = mode == XF_DW ? 2 : 0; k.out_bufs = 1;
    auto total = [&]() { return (size_t)k.as * FPW_A_BYTES + (size_t)k.bs * b_slot + (size_t)k.out_bufs * FPW_OUT_BUF +
                                (size_t)k.rs * FPW_RAW_BYTES + w_bytes; };
    if (total() > budget) return 0;
    if (mode == XF_DW) { k.rs = 3; if (total() > budget) k.rs = 2; }
    k.out_bufs = 2; if (total() > budget) k.out_bufs = 1;         // the store of slab i drains under slab i+1
    k.bs = 3; if (total() > budget) k.bs = 2;
    if (mode == XF_DW && k.rs == 3) { k.rs = 4; if (total() > budget) k.rs = 3; }
    k.as = 3; if (total() > budget) k.as = 2;
    if (k.bs == 3) { k.bs = 4; if (total() > budget) k.bs = 3; }
    return total();
}

// A conv_xf layer this kernel takes: whole 16 x 8 tiles (H % 8 == W % 16 == 0, so a SCALE tile never straddles two
// images and H*W % 128 == 0), a unit-stride 16-byte-aligned output of whole groups of 8 channels (TMA stores into its
// channel window), a unit-stride residual of the output's shape, an instantiated activation and unit width.
bool fpw_supported(const XfSetup& s) {
    if (!xf_supported(s)) return false;
    if (s.act != ACT_NONE && s.act != ACT_RELU) return false;
    if (!fpw_unit_width(s.mode, s.n_tile)) return false;
    const TView& o = s.out;
    if (o.fmt != DT_SPLIT16 && o.fmt != DT_F32) return false;
    const size_t oes = o.fmt == DT_SPLIT16 ? 2 : 4;
    if (o.c_stride != 1 || (s.Cout % 8) || ((size_t)o.ld * oes) % 16 || ((size_t)o.c_off * oes) % 16) return false;
    if (((uintptr_t)o.base % 16) || (o.fmt == DT_SPLIT16 && ((size_t)o.plane * 2) % 16)) return false;
    if (o.H % FPW_TH || o.W % FPW_TW) return false;
    if (s.res.base) {
        if (s.res.c_stride != 1 || (s.res.fmt != DT_SPLIT16 && s.res.fmt != DT_F32)) return false;
        if (s.res.H != o.H || s.res.W != o.W || s.res.C < s.Cout || ((s.res.ld | s.res.c_off) & 1) || (s.res.plane & 1))
            return false;
    }
    FpwK k;
    k.cchunks = ((s.low.base ? s.low.C : 0) + s.x.C + 63) / 64;
    return fpw_rings(k, s.mode, fpw_unit_width(s.mode, s.n_tile)) != 0;
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
    SKPS_CHECK(r == CUDA_SUCCESS, "conv_fpw: cuTensorMapEncodeTiled failed: %d", (int)r);
    return 0;
}

int fpw_prepare(FpwLayer& L, const XfSetup& s) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    SKPS_CHECK(fpw_supported(s), "conv_fpw: unsupported layer");
    memset(&L.k, 0, sizeof(L.k));
    FpwK& k = L.k;
    L.mode = s.mode;
    L.n = fpw_unit_width(s.mode, s.n_tile);
    L.act = s.act;
    L.out_fmt = s.out.fmt;
    const TView& out = s.out;
    k.H = out.H; k.W = out.W;
    k.tiles_x = out.W / FPW_TW;
    k.tiles_per_img = k.tiles_x * (out.H / FPW_TH);
    k.nsplit = (s.n_tile + L.n - 1) / L.n;
    const int Cu = s.low.base ? s.low.C : 0;
    k.Cin = Cu + s.x.C;
    k.cchunks = (k.Cin + 63) / 64;
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
    // input tensor maps: conv_xf's boxes
    L.src0 = CUtensorMap(); L.src1_hi = CUtensorMap(); L.src1_lo = CUtensorMap();
    if (s.mode == XF_SCALE) {
        if (encode4(enc, &L.src1_hi, s.x, 0, s.max_batch, 64, FPW_TW, FPW_TH, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
        if (encode4(enc, &L.src1_lo, s.x, 1, s.max_batch, 64, FPW_TW, FPW_TH, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
        L.src0 = L.src1_hi;
    } else {
        if (s.low.base) {
            if (encode4(enc, &L.src0, s.low, 0, s.max_batch, 32, FPW_LW, FPW_LH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
        }
        if (s.x.fmt == DT_SPLIT16) {
            if (encode4(enc, &L.src1_hi, s.x, 0, s.max_batch, 32, FPW_IW, FPW_IH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
            if (encode4(enc, &L.src1_lo, s.x, 1, s.max_batch, 32, FPW_IW, FPW_IH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
            if (!s.low.base) L.src0 = L.src1_hi;
        } else {
            if (encode4(enc, &L.src0, s.x, 0, s.max_batch, 32, FPW_IW, FPW_IH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
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
        SKPS_CHECK(r == CUDA_SUCCESS, "conv_fpw: cuTensorMapEncodeTiled(weff) failed: %d", (int)r);
    }
    // weights: (K_pad, n_tile) as packed; one box = 64 K x the unit's N rows
    const int K_pad = k.cchunks * 64;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)K_pad, (cuuint64_t)s.n_tile};
        cuuint64_t strides[1] = {(cuuint64_t)K_pad * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)L.n};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(plane ? &L.b_lo : &L.b_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)(plane ? s.w_lo : s.w_hi), dims,
                         strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "conv_fpw: cuTensorMapEncodeTiled(B) failed: %d", (int)r);
    }
    // output: {Cout, W, H, max_batch} per plane of the channel window, box = 32 channels x one 16 x 8 tile in the staging
    // layout the epilogue writes; stores clip at Cout
    const bool split = out.fmt == DT_SPLIT16;
    const int oes = split ? 2 : 4;
    for (int plane = 0; plane < (split ? 2 : 1); ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)s.Cout, (cuuint64_t)out.W, (cuuint64_t)out.H, (cuuint64_t)s.max_batch};
        cuuint64_t strides[3] = {(cuuint64_t)out.ld * oes, (cuuint64_t)out.W * out.ld * oes,
                                 (cuuint64_t)out.H * out.W * out.ld * oes};
        cuuint32_t box[4] = {32, FPW_TW, FPW_TH, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        char* base = (char*)out.base + (size_t)out.c_off * oes + (plane ? (size_t)out.plane * 2 : 0);
        CUresult r = enc(plane ? &L.o_lo : &L.o_hi, split ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                         4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         split ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "conv_fpw: cuTensorMapEncodeTiled(out) failed: %d", (int)r);
    }
    if (!split) L.o_lo = L.o_hi;
    const size_t smem = fpw_rings(k, s.mode, L.n);
    SKPS_CHECK(smem, "conv_fpw: layer does not fit shared memory");
    L.smem_bytes = (int)smem + 1024;
    k.Cout = s.Cout; k.out_scale = s.out_scale;
    k.bias = s.bias ? s.bias : fpw_zero_bias();
    SKPS_CHECK(k.bias, "conv_fpw: zero-bias allocation failed");
    k.res = s.res.base; k.res_fmt = s.res.fmt; k.res_plane = s.res.plane; k.res_ld = s.res.ld; k.res_coff = s.res.c_off;
    k.res_first = s.res.base ? s.res_first : 0;
    L.valid = true;
    return 0;
}

template <int MODE, int N, int ACT, bool SPLIT>
static int fpw_launch_t(const FpwLayer& L, const FpwK& k, int grid, cudaStream_t stream) {
    // the shared-memory attribute is per device: remember what was set on each
    static int attr_bytes[FPW_MAX_DEVICES] = {};
    int dev = 0;
    SKPS_CUDA(cudaGetDevice(&dev));
    SKPS_CHECK(dev >= 0 && dev < FPW_MAX_DEVICES, "conv_fpw: device %d out of range", dev);
    if (L.smem_bytes > attr_bytes[dev]) {
        SKPS_CUDA(cudaFuncSetAttribute(conv_fpw_kernel<MODE, N, ACT, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       L.smem_bytes));
        attr_bytes[dev] = L.smem_bytes;
    }
    conv_fpw_kernel<MODE, N, ACT, SPLIT><<<grid, FPW_THREADS, L.smem_bytes, stream>>>(
        L.src0, L.src1_hi, L.src1_lo, L.b_hi, L.b_lo, L.o_hi, L.o_lo, L.w_eff, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

template <int MODE, int N>
static int fpw_launch_n(const FpwLayer& L, const FpwK& k, int grid, cudaStream_t stream) {
    const bool sp = L.out_fmt == DT_SPLIT16;
    switch (L.act) {
        case ACT_NONE: return sp ? fpw_launch_t<MODE, N, ACT_NONE, true>(L, k, grid, stream) : fpw_launch_t<MODE, N, ACT_NONE, false>(L, k, grid, stream);
        case ACT_RELU: return sp ? fpw_launch_t<MODE, N, ACT_RELU, true>(L, k, grid, stream) : fpw_launch_t<MODE, N, ACT_RELU, false>(L, k, grid, stream);
        default: break;
    }
    set_error("conv_fpw: activation %d not instantiated", L.act);
    return 1;
}

int fpw_launch(const FpwLayer& L, int batch, int num_sms, cudaStream_t stream) {
    SKPS_CHECK(L.valid, "conv_fpw: layer not prepared");
    FpwK k = L.k;
    k.units = batch * k.tiles_per_img * k.nsplit;
    const int grid = k.units < num_sms ? k.units : num_sms;
    if (L.mode == XF_DW) {
        switch (L.n) {
            case 32: return fpw_launch_n<XF_DW, 32>(L, k, grid, stream);
            case 64: return fpw_launch_n<XF_DW, 64>(L, k, grid, stream);
            default: break;
        }
    } else {
        switch (L.n) {
            case 48: return fpw_launch_n<XF_SCALE, 48>(L, k, grid, stream);
            case 64: return fpw_launch_n<XF_SCALE, 64>(L, k, grid, stream);
            default: break;
        }
    }
    set_error("conv_fpw: mode %d width %d not instantiated", L.mode, L.n);
    return 1;
}

}  // namespace skps

using namespace skps;

namespace {
__global__ void fpw_f32_to_split(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, long long n) {
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

// Debug/unit-test entry: one fused layer through conv_fpw on host data (tests/test_conv_fpw_gpu.py).  The arguments of
// skps_debug_conv_xf, then `batch` <= N: the kernel runs images [0, batch) of buffers sized for N, and `out` comes in as
// well as out, so that images past the batch can be checked to come back as they went in (through the split-fp16 planes
// when out_split != 0).  Fails for a layer conv_fpw does not take.
extern "C" SKPS_API int skps_debug_conv_fpw(int mode, const float* x, int N, int H, int W, int Cx, int x_split,
                                            const float* low, int Cl, const float* gate, const float* dww, int dw_act,
                                            const void* w_hi, const void* w_lo, const float* bias, int Cout, int act,
                                            int n_tile, float out_scale, const float* residual, int res_first,
                                            int out_split, float* out, const float* weff, int batch) {
    SKPS_CHECK(x && w_hi && w_lo && out && N > 0 && batch > 0 && batch <= N, "debug_conv_fpw: bad argument");
    const int K = Cx + (low ? Cl : 0), Kpad = (K + 63) / 64 * 64;
    const long long nx = (long long)N * H * W * Cx, nl = low ? (long long)N * (H / 2) * (W / 2) * Cl : 0;
    const long long nout = (long long)N * H * W * Cout;
    const bool xs = x_split || mode == XF_SCALE;
    DevBuf dx, dxs, dl, dg, dw, dwh, dwl, db, dr, dout, dwe;
    SKPS_CHECK(!dx.alloc(nx * 4) && !dxs.alloc(nx * 4) && !dl.alloc(nl * 4) && !dg.alloc((size_t)N * Cx * 4) &&
               !dw.alloc((size_t)10 * Kpad * 4) && !dwh.alloc((size_t)n_tile * Kpad * 2) && !dwl.alloc((size_t)n_tile * Kpad * 2) &&
               !db.alloc((size_t)Cout * 4) && !dr.alloc(nout * 4) && !dout.alloc(nout * 4 * (out_split ? 2 : 1)),
               "debug_conv_fpw: cudaMalloc failed");
    SKPS_CUDA(cudaMemcpy(dx.p, x, nx * 4, cudaMemcpyHostToDevice));
    if (xs) {
        fpw_f32_to_split<<<(unsigned)((nx + 255) / 256), 256>>>((const float*)dx.p, (__half*)dxs.p, (__half*)dxs.p + nx, nx);
        SKPS_CUDA(cudaGetLastError());
    }
    if (low) SKPS_CUDA(cudaMemcpy(dl.p, low, nl * 4, cudaMemcpyHostToDevice));
    if (low) {
        SKPS_CHECK(weff && Cl % 32 == 0 && !dwe.alloc((size_t)Cl * 144 * 4), "debug_conv_fpw: class weights");
        SKPS_CUDA(cudaMemcpy(dwe.p, weff, (size_t)Cl * 144 * 4, cudaMemcpyHostToDevice));
    }
    if (gate) SKPS_CUDA(cudaMemcpy(dg.p, gate, (size_t)N * Cx * 4, cudaMemcpyHostToDevice));
    if (dww) SKPS_CUDA(cudaMemcpy(dw.p, dww, (size_t)10 * Kpad * 4, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(dwh.p, w_hi, (size_t)n_tile * Kpad * 2, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(dwl.p, w_lo, (size_t)n_tile * Kpad * 2, cudaMemcpyHostToDevice));
    if (bias) SKPS_CUDA(cudaMemcpy(db.p, bias, (size_t)Cout * 4, cudaMemcpyHostToDevice));
    if (residual) SKPS_CUDA(cudaMemcpy(dr.p, residual, nout * 4, cudaMemcpyHostToDevice));
    // the output's initial contents: float32, or split into the hi/lo planes
    SKPS_CUDA(cudaMemcpy(dout.p, out, nout * 4, cudaMemcpyHostToDevice));
    void* obase = dout.p;
    if (out_split) {
        obase = (float*)dout.p + nout;
        fpw_f32_to_split<<<(unsigned)((nout + 255) / 256), 256>>>((const float*)dout.p, (__half*)obase, (__half*)obase + nout, nout);
        SKPS_CUDA(cudaGetLastError());
    }
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
    s.out = view(obase, Cout, H, W, out_split ? DT_SPLIT16 : DT_F32, nout);
    if (residual) s.res = view(dr.p, Cout, H, W, DT_F32, 0);
    s.res_first = res_first;
    FpwLayer L;
    if (fpw_prepare(L, s)) return 1;
    if (fpw_launch(L, batch, sm_count(), 0)) return 1;
    SKPS_CUDA(cudaDeviceSynchronize());
    if (out_split) {
        __half* tmp = (__half*)malloc(nout * 4);
        SKPS_CHECK(tmp, "debug_conv_fpw: host allocation failed");
        SKPS_CUDA(cudaMemcpy(tmp, obase, nout * 4, cudaMemcpyDeviceToHost));
        for (long long i = 0; i < nout; ++i) out[i] = __half2float(tmp[i]) + __half2float(tmp[nout + i]);
        free(tmp);
    } else {
        SKPS_CUDA(cudaMemcpy(out, dout.p, nout * 4, cudaMemcpyDeviceToHost));
    }
    return 0;
}
