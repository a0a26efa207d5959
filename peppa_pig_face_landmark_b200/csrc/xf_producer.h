// The A producer of the fused "producer -> pointwise convolution" kernels, conv_xf.cu and conv_fpw.cu.  The A operand of
//     C[128 pixels][N] = A[128 pixels][K] * W[N][K]
// never exists in HBM: transform warps build each 128 x 64 fp16 hi/lo tile in shared memory, in the 128-byte-swizzled
// K-major layout wgmma reads, from a raw tile that TMA staged:
//
//   XF_DW     A = dw_act(depthwise3x3(x))                              (MobileNetV3 blocks without squeeze-excite:
//             or dw_act(depthwise3x3(concat(bilinear_x2(low), skip)))   conv_dw -> conv_pwl; DecoderBlock heads,
//                                                                       model.py:133-196: Resize -> Concat -> dw -> pw)
//   XF_SCALE  A = x * gate[n, c]                                        (squeeze-excite scale ahead of conv_pwl: replaces
//                                                                       the OP_SCALE_CH pass over the expanded tensor)
//
// Both kernels take this side whole: the tile geometry, the CTA's shared-memory layout and mbarrier rings, the A-side TMA
// loads of each K-chunk, the transform warps (warps 8-15) and the host set-up of the A-side tensor maps.  They differ only
// on the MMA side and in how a CTA walks its work, so both multiply the same A tiles in the same K order.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.h"
#include "tc_ptx.h"

namespace skps {

enum { XF_SCALE = 0, XF_DW = 1 };                                   // kernel mode
enum { XS_UP_F32 = 0, XS_DW_F32 = 1, XS_DW_SPLIT = 2 };             // source of one 32-channel sub-chunk (XF_DW)
constexpr int XF_MAX_CHUNKS = 16;                                   // K <= 1024 channels

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
constexpr int XF_OUT_BUF = 16384;                    // epilogue staging: one 32-channel slab of 128 pixels, hi + lo or float32

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

// Parameters of the A producer: the TMA loads of raw or A tiles and the transform warps.
struct XfProducer {
    int H, W, tiles_x, tiles_per_img;               // output map, 16 x 8 pixel tiles
    int cchunks, Cin;                               // K chunks of 64 channels
    int rs, as;                                     // ring depths: raw tiles, A tiles
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
};

// ------------------------------------------------------------------------------------------ host side (conv_xf.cu)
// A layer conv_xf takes; conv_fpw takes a subset of these.
bool xf_supported(const XfSetup& s);
// Fills the producer parameters of a layer and encodes its A-side tensor maps: src0 / src1_hi / src1_lo (the raw or A tile
// sources) and w_eff (the class weights of up-sampled channels).  Maps a mode does not use alias a used one.
int xf_producer_prepare(XfProducer& k, CUtensorMap& src0, CUtensorMap& src1_hi, CUtensorMap& src1_lo, CUtensorMap& w_eff,
                        const XfSetup& s);
// Ring depths of a layer (k.rs, k.as, bs, out_bufs): minimal rings first, then what is left of the shared memory, less
// `reserve` bytes, goes on depth.  b_slot = bytes of one weight-ring slot; two_out_bufs: a second staging buffer is of use.
// Returns the bytes of the rings and the depthwise weights, or 0 when even the minimal rings do not fit.
size_t xf_rings(XfProducer& k, int mode, size_t b_slot, size_t reserve, bool two_out_bufs, int& bs, int& out_bufs);

// ------------------------------------------------------------------------------------------ device side
struct XfBarriers {
    uint64_t raw_full[XF_RING], raw_empty[XF_RING], a_raw[XF_RING], a_full[XF_RING], a_empty[XF_RING], b_full[XF_RING],
        b_empty[XF_RING];
};

// Shared-memory layout, from the 1024-byte aligned start of the dynamic window:
// [A ring][B ring][epilogue staging][raw ring][depthwise weights (XF_DW)]
struct XfSmem {
    uint32_t a_off, b_off, o_off, r_off, w_off;
};

template <int MODE>
__device__ __forceinline__ XfSmem xf_smem(const uint8_t* smem_raw, const XfProducer& p, int bs, uint32_t b_slot, int out_bufs) {
    XfSmem s;
    s.a_off = (smem_u32(smem_raw) + 1023u) & ~1023u;
    s.b_off = s.a_off + (uint32_t)p.as * XF_A_BYTES;
    s.o_off = s.b_off + (uint32_t)bs * b_slot;
    s.r_off = s.o_off + (uint32_t)out_bufs * XF_OUT_BUF;
    s.w_off = s.r_off + (MODE == XF_DW ? (uint32_t)p.rs * XF_RAW_BYTES : 0u);
    return s;
}

// CTA set-up: tensor-map prefetch, mbarrier rings, the layer's depthwise weights.  Ends in __syncthreads.  mma_warps: the
// warps that read each A and B slot and release it (one MMA warpgroup, or two sharing every slot); nthreads: the CTA's.
template <int MODE>
__device__ __forceinline__ void xf_cta_init(const XfProducer& p, XfBarriers& bar, const XfSmem& sm, uint8_t* smem_raw,
                                            const CUtensorMap* tm0, const CUtensorMap* tm1_hi, const CUtensorMap* tmB_hi,
                                            const CUtensorMap* tmB_lo, int mma_warps = 4, int nthreads = XF_THREADS) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(tm0) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(tm1_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(tmB_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(tmB_lo) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < XF_RING; ++s) {
            mbar_init(smem_u32(&bar.raw_full[s]), 1);
            mbar_init(smem_u32(&bar.raw_empty[s]), p.halves ? 4 : 8);   // one arrival per warp that consumes the slot
            mbar_init(smem_u32(&bar.a_raw[s]), 1);
            mbar_init(smem_u32(&bar.a_full[s]), 8);
            mbar_init(smem_u32(&bar.a_empty[s]), mma_warps);      // one arrival per MMA warp
            mbar_init(smem_u32(&bar.b_full[s]), 1);
            mbar_init(smem_u32(&bar.b_empty[s]), mma_warps);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (MODE == XF_DW) {
        // depthwise weights + bias of the whole layer stay in shared memory for the life of the (persistent) CTA
        float* dws = reinterpret_cast<float*>(smem_raw + (sm.w_off - smem_u32(smem_raw)));
        for (int i = threadIdx.x; i < 10 * p.cchunks * 64; i += nthreads) dws[i] = __ldg(p.dww + i);
    }
    __syncthreads();
}

// One thread: the A-side TMA loads of K-chunk kc of the tile at (img, oy0, ox0) - the A tile itself (XF_SCALE) or the raw
// tile of each of its 32-channel sub-chunks (XF_DW).  st / ph: the producer's position in the A ring (XF_SCALE) or the raw
// ring (XF_DW).
template <int MODE>
__device__ __forceinline__ void xf_load_a(const XfProducer& p, XfBarriers& bar, const XfSmem& sm, const CUtensorMap* tm0,
                                          const CUtensorMap* tm1_hi, const CUtensorMap* tm1_lo, const CUtensorMap* tmW,
                                          int kc, int img, int oy0, int ox0, int& st, uint32_t& ph) {
    if (MODE == XF_SCALE) {
        mbar_wait_g(smem_u32(&bar.a_empty[st]), ph ^ 1u);
        const uint32_t fb = smem_u32(&bar.a_raw[st]);
        mbar_expect_tx(fb, XF_A_BYTES);
        const uint32_t dst = sm.a_off + (uint32_t)st * XF_A_BYTES;
        tma_load_4d(dst, tm1_hi, fb, kc * 64, ox0, oy0, img);
        tma_load_4d(dst + XF_A_PLANE, tm1_lo, fb, kc * 64, ox0, oy0, img);
        if (++st == p.as) { st = 0; ph ^= 1u; }
        return;
    }
    const int subs = p.chunk_subs[kc];
    for (int h = 0; h < subs; ++h) {
        const int si = kc * 2 + h, smode = p.sub_mode[si], c = p.sub_c[si];
        mbar_wait_g(smem_u32(&bar.raw_empty[st]), ph ^ 1u);
        const uint32_t fb = smem_u32(&bar.raw_full[st]);
        const uint32_t dst = sm.r_off + (uint32_t)st * XF_RAW_BYTES;
        if (smode == XS_UP_F32) {
            // low-res window + the 3 x 3 block of row/column-class stencil weights this tile can need
            // (classes first|even|odd|last: a tile at the top/left border starts at "first", else at "even")
            // (a map one tile wide holds first AND last columns: 4 column classes, p.wcx = 4)
            mbar_expect_tx(fb, XF_UP_BYTES + (uint32_t)p.wcx * 3u * 9u * 128u);
            tma_load_4d(dst, tm0, fb, c, (ox0 >> 1) - 1, (oy0 >> 1) - 1, img);
            tma_load_5d(dst + XF_UP_BYTES, tmW, fb, 0, 0, (p.wcx == 4 || ox0 == 0) ? 0 : 1, oy0 == 0 ? 0 : 1, c >> 5);
        } else if (smode == XS_DW_F32) {
            mbar_expect_tx(fb, XF_RAW_BYTES);
            tma_load_4d(dst, tm0, fb, c, ox0 - 1, oy0 - 1, img);
        } else {
            mbar_expect_tx(fb, XF_RAW_BYTES);
            tma_load_4d(dst, tm1_hi, fb, c, ox0 - 1, oy0 - 1, img);
            tma_load_4d(dst + XF_RAW_BYTES / 2, tm1_lo, fb, c, ox0 - 1, oy0 - 1, img);
        }
        if (++st == p.rs) { st = 0; ph ^= 1u; }
    }
}

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

template <int ACT>
__device__ __forceinline__ void act16(float4* acc) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        acc[q].x = act_t<ACT>(acc[q].x); acc[q].y = act_t<ACT>(acc[q].y);
        acc[q].z = act_t<ACT>(acc[q].z); acc[q].w = act_t<ACT>(acc[q].w);
    }
}

// The transform warps (8-15): raw tile -> A tile, K-chunk by K-chunk of each work item u = blockIdx.x, + gridDim.x, ...
// below n_work; tile_of(u) is the pixel tile of item u.  Every item takes the cchunks A tiles the producer loads for it.
template <int MODE, class TileOf>
__device__ __forceinline__ void xf_transform(const XfProducer& p, XfBarriers& bar, const XfSmem& sm, uint8_t* smem_raw,
                                             int n_work, TileOf tile_of) {
    const int lane = threadIdx.x & 31;
    const int tt = threadIdx.x - 256;
    const int Kpad = p.cchunks * 64;
    int ast = 0, rst = 0;
    uint32_t aph = 0, rph = 0;
    if (MODE == XF_SCALE) {
        // thread = physical 16-byte slot (tt & 7) of rows (tt >> 3) + 32 i: its logical 8-channel group is the same in
        // every row it touches (128-byte swizzle: logical = physical ^ (row & 7))
        const int r0 = tt >> 3, ps = tt & 7, j = ps ^ (r0 & 7);
        for (int u = blockIdx.x; u < n_work; u += gridDim.x) {
            const int img = tile_of(u) / p.tiles_per_img;
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
                mbar_wait_g(smem_u32(&bar.a_raw[ast]), aph);
                const uint32_t sa = sm.a_off + (uint32_t)ast * XF_A_BYTES + (uint32_t)ps * 16u;
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
                if (lane == 0) mbar_arrive(smem_u32(&bar.a_full[ast]));
                if (++ast == p.as) { ast = 0; aph ^= 1u; }
            }
        }
    } else if (!p.halves) {
        // layers without up-sampled channels: all 256 threads work on one 32-channel sub-chunk at a time,
        // thread = 4 consecutive output pixels of one tile row x 4 channels
        const int cl = tt & 7, pg = tt >> 3, prow = pg >> 2, xs = (pg & 3) * 4;
        const float* dws = reinterpret_cast<const float*>(smem_raw + (sm.w_off - smem_u32(smem_raw)));
        for (int u = blockIdx.x; u < n_work; u += gridDim.x) {
            for (int kc = 0; kc < p.cchunks; ++kc) {
                mbar_wait_g(smem_u32(&bar.a_empty[ast]), aph ^ 1u);
                const uint32_t sa = sm.a_off + (uint32_t)ast * XF_A_BYTES;
                const int subs = p.chunk_subs[kc];
                for (int h = 0; h < subs; ++h) {
                    const int smode = p.sub_mode[kc * 2 + h];
                    const int cw = kc * 64 + h * 32 + cl * 4;
                    const float4 bias4 = *reinterpret_cast<const float4*>(dws + 9 * Kpad + cw);
                    float4 acc[4] = {bias4, bias4, bias4, bias4};
                    mbar_wait_g(smem_u32(&bar.raw_full[rst]), rph);
                    const uint8_t* raw = smem_raw + (sm.r_off + (uint32_t)rst * XF_RAW_BYTES - smem_u32(smem_raw));
                    {
#pragma unroll
                        for (int ky = 0; ky < 3; ++ky) {
                            float4 in[6];
#pragma unroll
                            for (int i = 0; i < 6; ++i) {
                                const int px = (prow + ky) * XF_IW + xs + i;
                                if (smode == XS_DW_F32) {
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
                    if (lane == 0) mbar_arrive(smem_u32(&bar.raw_empty[rst]));
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
                if (lane == 0) mbar_arrive(smem_u32(&bar.a_full[ast]));
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
        const float* dws = reinterpret_cast<const float*>(smem_raw + (sm.w_off - smem_u32(smem_raw)));
        for (int u = blockIdx.x; u < n_work; u += gridDim.x) {
            const int t = tile_of(u) % p.tiles_per_img;
            const int oy0 = (t / p.tiles_x) * XF_TH, ox0 = (t % p.tiles_x) * XF_TW;
            const int ox = ox0 + xs;
            for (int kc = 0; kc < p.cchunks; ++kc) {
                mbar_wait_g(smem_u32(&bar.a_empty[ast]), aph ^ 1u);
                const uint32_t sa = sm.a_off + (uint32_t)ast * XF_A_BYTES;
                const int subs = p.chunk_subs[kc];
                if (half < subs) {
                    // ring slot of this half's sub-chunk: sub 0 sits at rst, sub 1 one slot further
                    int slot = rst + half;
                    uint32_t sph = rph;
                    if (slot >= p.rs) { slot -= p.rs; sph ^= 1u; }
                    const int smode = p.sub_mode[kc * 2 + half];
                    const int cw = kc * 64 + half * 32 + cl * 4;
                    const float4 bias4 = *reinterpret_cast<const float4*>(dws + 9 * Kpad + cw);
                    float4 acc[2][4] = {{bias4, bias4, bias4, bias4}, {bias4, bias4, bias4, bias4}};
                    int r0, r1;                                       // the two tile rows of this thread
                    mbar_wait_g(smem_u32(&bar.raw_full[slot]), sph);
                    const uint8_t* raw = smem_raw + (sm.r_off + (uint32_t)slot * XF_RAW_BYTES - smem_u32(smem_raw));
                    if (smode == XS_UP_F32) {
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
                        for (int j = 0; j < 4; ++j) lr[j] = min(max(m - 1 + j, 0), p.Hl - 1) - ly0;
#pragma unroll
                        for (int j = 0; j < 4; ++j) lc[j] = min(max(c2 - 1 + j, 0), p.Wl - 1) - lx0;
                        float4 wpE[3], wpO[3];                            // previous tap row's weights (row r1 lags one low row)
#pragma unroll
                        for (int wr = 0; wr < 4; ++wr) {
                            float4 L[4];
#pragma unroll
                            for (int v = 0; v < 4; ++v)
                                L[v] = *reinterpret_cast<const float4*>(raw + ((lr[wr] * XF_LW + lc[v]) * 32 + cl * 4) * 4);
#pragma unroll
                            for (int v = 0; v < 3; ++v) {
                                float4 wE = wpE[v], wO = wpO[v];          // (wr - 1, v) weights of the shared class
                                if (wr > 0) {                             // row r1: this low row is its tap row a = wr - 1
                                    const int o = ((wr - 1) * 3 + v) * 32;
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
                                if (wr < 3) {                             // row r0: this low row is its tap row a = wr
                                    const int o = (wr * 3 + v) * 32;
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
                        for (int wr = 0; wr < 4; ++wr) {                  // window row r0 + wr: tap row wr of r0, wr - 1 of r1
                            float4 in[6];
#pragma unroll
                            for (int i = 0; i < 6; ++i) {
                                const int px = (r0 + wr) * XF_IW + xs + i;
                                if (smode == XS_DW_F32) {
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
                                if (wr < 3) {
                                    w = *reinterpret_cast<const float4*>(dws + (wr * 3 + kx) * Kpad + cw);
#pragma unroll
                                    for (int q = 0; q < 4; ++q) acc[0][q] = f4_fma(in[q + kx], w, acc[0][q]);
                                }
                                if (wr > 0) {
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
                    if (lane == 0) mbar_arrive(smem_u32(&bar.raw_empty[slot]));
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
                if (lane == 0) mbar_arrive(smem_u32(&bar.a_full[ast]));
                if (++ast == p.as) { ast = 0; aph ^= 1u; }
            }
        }
    }
}

}  // namespace skps
