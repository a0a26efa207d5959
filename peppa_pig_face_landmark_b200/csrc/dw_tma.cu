// Depthwise convolution with TMA-staged input tiles (sm_90a).
//
// The register-gather depthwise kernel (ops_misc.cu) is latency bound: each thread has only a
// handful of 8-byte loads in flight.  Here one CTA owns an 8x16 output tile x CB channels; a single
// thread issues one 4-D TMA box per float16 plane (or one float32 box) covering the tile plus its
// halo, with the convolution's zero padding coming from TMA out-of-bounds fill, and everything else
// is computed out of shared memory.  Several CTAs per SM keep ~100 KB of loads in flight per SM.
//
// Covers the landmark network's depthwise layers (kps_student.onnx conv_dw nodes; 3x3 and 5x5,
// stride 1/2, dilation 1/2) and the detector's (3x3, stride 1/2).  Same arithmetic order as
// dwconv_kernel: bias first, then taps in (ky,kx) order with fmaf.
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.h"
#include "dw_tma.h"

namespace skps {

__device__ __forceinline__ uint32_t dsmem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

constexpr int TH = 8, TW = 16;          // output tile (TH x RY rows)
constexpr int DW_THREADS = 256;

// Per-tile channel sums of the activated outputs (squeeze-excite: the GlobalAveragePool over this layer's output is
// assembled from these partial sums by se_fc_kernel, so the tensor is not read again).  Every thread of the CTA calls
// this with its float4 of per-channel sums (zeros when it owns no valid pixel/channel); fixed summation order.
template <int CG>
__device__ __forceinline__ void tile_channel_sums(float4 s, float* __restrict__ dst, bool write_ok) {
    __shared__ float4 red[DW_THREADS / 32][CG];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cg = threadIdx.x % CG;
#pragma unroll
    for (int off = 16; off >= CG; off >>= 1) {
        s.x += __shfl_xor_sync(0xffffffffu, s.x, off); s.y += __shfl_xor_sync(0xffffffffu, s.y, off);
        s.z += __shfl_xor_sync(0xffffffffu, s.z, off); s.w += __shfl_xor_sync(0xffffffffu, s.w, off);
    }
    if (lane < CG) red[warp][cg] = s;
    __syncthreads();
    if (threadIdx.x < CG) {
        float4 t = red[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < DW_THREADS / 32; ++w) {
            const float4 v = red[w][threadIdx.x];
            t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
        }
        if (write_ok) *reinterpret_cast<float4*>(dst) = t;
    }
}

// Output rows per thread: the 5x5 stride-1 layers are shared-memory-bandwidth bound (many LDS.128 per FMA, DRAM
// far from busy); a thread that owns rows r and r+D of the same columns re-uses K-1 of the K input rows it loads for the
// first row, so the tile is 16 rows high for them and the loads per output drop 1.75x.
template <int K, int S, int D, bool SPLIT_IN, int RY>
__global__ void __launch_bounds__(DW_THREADS)
dw_tma_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo, const DwTmaK p) {
    constexpr int THT = TH * RY;                           // tile height in output rows
    constexpr int CB = SPLIT_IN ? 64 : 32;                 // channels per CTA: 128-byte pixel rows in smem
    constexpr int CG = CB / 4;                             // 4-channel groups
    constexpr int PGS = DW_THREADS / CG;                   // pixel groups
    constexpr int PX = TH * TW / PGS;                      // consecutive output pixels (along x) per thread and row
    constexpr int IH = (THT - 1) * S + (K - 1) * D + 1, IW = (TW - 1) * S + (K - 1) * D + 1;
    constexpr int SPAN = (PX - 1) * S + (K - 1) * D + 1;
    constexpr int ROW_BYTES = 128;
    constexpr int PLANE_BYTES = IH * IW * ROW_BYTES;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar;

    const int tid = threadIdx.x;
    const int tiles_x = (p.Wo + TW - 1) / TW;
    const int ty = blockIdx.x / tiles_x, tx = blockIdx.x - ty * tiles_x;
    const int chunk = blockIdx.y;
    const int n = blockIdx.z + p.img0;
    const int oy0 = ty * THT, ox0 = tx * TW;
    const uint32_t sbase = (dsmem_u32(smem) + 127u) & ~127u;
    const uint32_t bar_a = dsmem_u32(&bar);

    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a),
                     "r"((uint32_t)(SPLIT_IN ? 2 * PLANE_BYTES : PLANE_BYTES)) : "memory");
        const int cx = ox0 * S - p.pad, cy = oy0 * S - p.pad, cc = chunk * CB;
        asm volatile(
            "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
            ::"r"(sbase), "l"(&tm_hi), "r"(bar_a), "r"(cc), "r"(cx), "r"(cy), "r"(n) : "memory");
        if (SPLIT_IN)
            asm volatile(
                "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                ::"r"(sbase + PLANE_BYTES), "l"(&tm_lo), "r"(bar_a), "r"(cc), "r"(cx), "r"(cy), "r"(n) : "memory");
    }
    // thread -> (4-channel group, row slot, x segment); row slot pr owns output rows row0 + ry*D (ry < RY)
    const int cg = tid % CG, pg = tid / CG;
    constexpr int SEGS = TW / PX;
    const int pr = pg / SEGS, xs = (pg % SEGS) * PX;
    const int row0 = RY == 1 ? pr : (pr / D) * (RY * D) + (pr % D);
    const int c = chunk * CB + cg * 4;
    const bool c_ok = c < p.C;
    // this CTA's slice of the weights ([K*K][CB]) and bias, staged in shared memory while the TMA load is in flight: the
    // tap loop reads them as warp-wide broadcasts instead of one global load per tap (loads that otherwise stall the tap loop)
    __shared__ float4 wsm[K * K + 1][CG];
    for (int i = tid; i < (K * K + 1) * CG; i += DW_THREADS) {
        const int r = i / CG, g = i - r * CG, cc = chunk * CB + g * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (cc < p.C) v = *reinterpret_cast<const float4*>((r < K * K ? p.w + (long long)r * p.w_ld : p.bias) + cc);
        wsm[r][g] = v;
    }
    __syncthreads();        // weights staged; barrier init visible to all waiters
    float4 acc[RY][PX];
    {
        const float4 b = wsm[K * K][cg];
#pragma unroll
        for (int ry = 0; ry < RY; ++ry)
#pragma unroll
            for (int q = 0; q < PX; ++q) acc[ry][q] = b;
    }
    {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "DW_WAIT:\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t"
            "@p bra DW_DONE;\n\t"
            "bra DW_WAIT;\n\t"
            "DW_DONE:\n\t"
            "}\n" ::"r"(bar_a) : "memory");
    }
    const uint8_t* tile = smem + (sbase - dsmem_u32(smem));
    float4 psum = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c_ok) {
        // input row j (= row0*S + j*D) feeds tap ky = j of output row 0 and tap ky = j-1 of output row 1
        float4 wprev[K];
#pragma unroll
        for (int j = 0; j < K + RY - 1; ++j) {
            float4 in[SPAN];
            const int iy = row0 * S + j * D;
#pragma unroll
            for (int i = 0; i < SPAN; ++i) {
                bool used = false;
#pragma unroll
                for (int kx = 0; kx < K; ++kx)
#pragma unroll
                    for (int q = 0; q < PX; ++q) used |= (q * S + kx * D == i);
                if (!used) continue;
                const int off = (iy * IW + xs * S + i) * ROW_BYTES;
                if (SPLIT_IN) {
                    const uint2 a = *reinterpret_cast<const uint2*>(tile + off + cg * 8);
                    const uint2 b = *reinterpret_cast<const uint2*>(tile + PLANE_BYTES + off + cg * 8);
                    const __half2* a2 = reinterpret_cast<const __half2*>(&a);
                    const __half2* b2 = reinterpret_cast<const __half2*>(&b);
                    const float2 a01 = __half22float2(a2[0]), a23 = __half22float2(a2[1]);
                    const float2 b01 = __half22float2(b2[0]), b23 = __half22float2(b2[1]);
                    in[i] = make_float4(a01.x + b01.x, a01.y + b01.y, a23.x + b23.x, a23.y + b23.y);
                } else {
                    in[i] = *reinterpret_cast<const float4*>(tile + off + cg * 16);
                }
            }
#pragma unroll
            for (int kx = 0; kx < K; ++kx) {
                float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
                if (j < K) {
                    w = wsm[j * K + kx][cg];
#pragma unroll
                    for (int q = 0; q < PX; ++q) {
                        const float4 v = in[q * S + kx * D];
                        acc[0][q].x = fmaf(v.x, w.x, acc[0][q].x);
                        acc[0][q].y = fmaf(v.y, w.y, acc[0][q].y);
                        acc[0][q].z = fmaf(v.z, w.z, acc[0][q].z);
                        acc[0][q].w = fmaf(v.w, w.w, acc[0][q].w);
                    }
                }
                if (RY == 2 && j >= 1) {
                    const float4 u = wprev[kx];          // weights of tap row j-1, loaded in the previous iteration
#pragma unroll
                    for (int q = 0; q < PX; ++q) {
                        const float4 v = in[q * S + kx * D];
                        acc[RY - 1][q].x = fmaf(v.x, u.x, acc[RY - 1][q].x);
                        acc[RY - 1][q].y = fmaf(v.y, u.y, acc[RY - 1][q].y);
                        acc[RY - 1][q].z = fmaf(v.z, u.z, acc[RY - 1][q].z);
                        acc[RY - 1][q].w = fmaf(v.w, u.w, acc[RY - 1][q].w);
                    }
                }
                wprev[kx] = w;
            }
        }
#pragma unroll
        for (int ry = 0; ry < RY; ++ry) {
            const int oy = oy0 + row0 + ry * D;
            if (oy < p.Ho) {
#pragma unroll
                for (int q = 0; q < PX; ++q) {
                    const int ox = ox0 + xs + q;
                    if (ox >= p.Wo) break;
                    float4 a = acc[ry][q];
                    a.x = apply_act(a.x, p.act); a.y = apply_act(a.y, p.act);
                    a.z = apply_act(a.z, p.act); a.w = apply_act(a.w, p.act);
                    psum.x += a.x; psum.y += a.y; psum.z += a.z; psum.w += a.w;
                    st4(p.out, p.out_fmt, p.out_plane, (((long long)n * p.Ho + oy) * p.Wo + ox) * p.out_ld + p.out_coff + c, a);
                }
            }
        }
    }
    if (p.part) {
        const int cw = chunk * CB + (tid % CG) * 4;          // channel quad written by thread tid < CG
        tile_channel_sums<CG>(psum, p.part + ((long long)n * gridDim.x + blockIdx.x) * p.part_ld + p.part_coff + cw,
                              cw < p.C);
    }
}

// ------------------------------------------------------------------------------------------
// Up-sampled channels of a DecoderBlock head: out[:, :Cu] = depthwise3x3(bilinear_x2(low)) with the
// 2x interpolation done out of a TMA-staged low-res tile (float32, 32 channels per CTA).
// One thread = a 2x2 block of output pixels x 4 channels (fixed .25/.75 blend weights).
// ------------------------------------------------------------------------------------------
constexpr int LH = TH / 2 + 2, LW = TW / 2 + 2;      // low-res tile incl. halo

__global__ void __launch_bounds__(DW_THREADS)
upcat_tma_kernel(const __grid_constant__ CUtensorMap tm_low, const DwTmaK p, const int Hl, const int Wl) {
    // Phase 0: TMA the low-res tile (6x10 pixels x 32 channels, float32).
    // Phase 1: every up-sampled pixel of the (8+2)x(16+2) high-res window is interpolated exactly once into shared
    //          memory (zero outside the high-res image = the depthwise conv's padding).
    // Phase 2: ordinary register-tiled depthwise 3x3 out of shared memory (4 pixels x 4 channels per thread).
    constexpr int CB = 32, CG = CB / 4;
    constexpr int LOW_BYTES = LH * LW * 128;
    constexpr int UH = TH + 2, UW = TW + 2;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar;
    const int tid = threadIdx.x;
    const int tiles_x = (p.Wo + TW - 1) / TW;
    const int ty = blockIdx.x / tiles_x, tx = blockIdx.x - ty * tiles_x;
    const int chunk = blockIdx.y;
    const int n = blockIdx.z + p.img0;
    const int oy0 = ty * TH, ox0 = tx * TW;
    const int ly0 = oy0 / 2 - 1, lx0 = ox0 / 2 - 1;          // low-res origin of the tile (may be -1)
    const uint32_t sbase = (dsmem_u32(smem) + 127u) & ~127u;
    const uint32_t bar_a = dsmem_u32(&bar);
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"((uint32_t)LOW_BYTES) : "memory");
        asm volatile(
            "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
            ::"r"(sbase), "l"(&tm_low), "r"(bar_a), "r"(chunk * CB), "r"(lx0), "r"(ly0), "r"(n) : "memory");
    }
    const int cg = tid % CG, pg = tid / CG;
    const int c = chunk * CB + cg * 4;
    const bool c_ok = c < p.C;
    __syncthreads();
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "UP_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t"
        "@p bra UP_DONE;\n\t"
        "bra UP_WAIT;\n\t"
        "UP_DONE:\n\t"
        "}\n" ::"r"(bar_a) : "memory");
    const uint8_t* low = smem + (sbase - dsmem_u32(smem));
    float* up = reinterpret_cast<float*>(const_cast<uint8_t*>(low) + LOW_BYTES);      // [UH][UW][32] float32
    // ---- phase 1: bilinear x2 (half_pixel, align_corners=False): source = dst/2 - 0.25, edge-replicated
    for (int item = pg; item < UH * UW; item += DW_THREADS / CG) {
        const int uy = item / UW, ux = item - uy * UW;
        const int ny = oy0 - 1 + uy, nx = ox0 - 1 + ux;                      // high-res coordinates
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ny >= 0 && ny < p.Ho && nx >= 0 && nx < p.Wo) {
            const int y0 = (ny & 1) ? (ny >> 1) : (ny >> 1) - 1, x0 = (nx & 1) ? (nx >> 1) : (nx >> 1) - 1;
            const float ly = (ny & 1) ? 0.25f : 0.75f, lx = (nx & 1) ? 0.25f : 0.75f;
            const float hy = 1.f - ly, hx = 1.f - lx;
            const int ya = min(max(y0, 0), Hl - 1) - ly0, yb = min(max(y0 + 1, 0), Hl - 1) - ly0;
            const int xa = min(max(x0, 0), Wl - 1) - lx0, xb = min(max(x0 + 1, 0), Wl - 1) - lx0;
            const float4 p00 = *reinterpret_cast<const float4*>(low + (ya * LW + xa) * 128 + cg * 16);
            const float4 p01 = *reinterpret_cast<const float4*>(low + (ya * LW + xb) * 128 + cg * 16);
            const float4 p10 = *reinterpret_cast<const float4*>(low + (yb * LW + xa) * 128 + cg * 16);
            const float4 p11 = *reinterpret_cast<const float4*>(low + (yb * LW + xb) * 128 + cg * 16);
            v.x = hy * (hx * p00.x + lx * p01.x) + ly * (hx * p10.x + lx * p11.x);
            v.y = hy * (hx * p00.y + lx * p01.y) + ly * (hx * p10.y + lx * p11.y);
            v.z = hy * (hx * p00.z + lx * p01.z) + ly * (hx * p10.z + lx * p11.z);
            v.w = hy * (hx * p00.w + lx * p01.w) + ly * (hx * p10.w + lx * p11.w);
        }
        *reinterpret_cast<float4*>(up + (item * CB + cg * 4)) = v;
    }
    __syncthreads();
    if (!c_ok) return;
    // ---- phase 2: depthwise 3x3 from the staged window, PX = 4 outputs along x per thread
    constexpr int PX = 4, SEGS = TW / PX;
    const int row = pg / SEGS, xs = (pg % SEGS) * PX;
    const float4 bias = *reinterpret_cast<const float4*>(p.bias + c);
    float4 acc[PX] = {bias, bias, bias, bias};
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        float4 in[PX + 2];
#pragma unroll
        for (int j = 0; j < PX + 2; ++j)
            in[j] = *reinterpret_cast<const float4*>(up + (((row + ky) * UW + xs + j) * CB + cg * 4));
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const float4 w = *reinterpret_cast<const float4*>(p.w + (ky * 3 + kx) * p.w_ld + c);
#pragma unroll
            for (int q = 0; q < PX; ++q) {
                const float4 v = in[q + kx];
                acc[q].x = fmaf(v.x, w.x, acc[q].x); acc[q].y = fmaf(v.y, w.y, acc[q].y);
                acc[q].z = fmaf(v.z, w.z, acc[q].z); acc[q].w = fmaf(v.w, w.w, acc[q].w);
            }
        }
    }
    const int oy = oy0 + row;
    if (oy >= p.Ho) return;
#pragma unroll
    for (int q = 0; q < PX; ++q) {
        const int ox = ox0 + xs + q;
        if (ox >= p.Wo) break;
        float4 a = acc[q];
        a.x = apply_act(a.x, p.act); a.y = apply_act(a.y, p.act); a.z = apply_act(a.z, p.act); a.w = apply_act(a.w, p.act);
        st4(p.out, p.out_fmt, p.out_plane, (((long long)n * p.Ho + oy) * p.Wo + ox) * p.out_ld + p.out_coff + c, a);
    }
}

// ------------------------------------------------------------------------------------------ host side
// Output rows per tile: 16 for the 5x5 stride-1 layers (two output rows per thread), else 8.  plan.dw_tile_rows mirrors
// this (rows of the per-tile channel-sum buffer).
int dw_tile_rows(int k, int s) { return (k == 5 && s == 1) ? 2 * TH : TH; }

static bool variant_ok(int k, int s, int d) {
    return (k == 3 && s == 1 && d == 1) || (k == 3 && s == 2 && d == 1) || (k == 5 && s == 1 && d == 1) ||
           (k == 5 && s == 2 && d == 1) || (k == 5 && s == 1 && d == 2);
}

bool dw_tma_supported(const TView& in, const TView& out, int k, int s, int d, int pad) {
    if (!variant_ok(k, s, d) || pad != d * (k - 1) / 2) return false;
    if (in.fmt != DT_F32 && in.fmt != DT_SPLIT16) return false;
    if (in.c_stride != 1 || out.c_stride != 1 || in.C != out.C) return false;
    if ((in.C | in.ld | in.c_off | out.ld | out.c_off) & 7) return false;
    return true;
}

int dw_tma_prepare(DwTmaLayer& L, const TView& in, const TView& out, const float* w, const float* bias, int k, int s,
                   int d, int pad, int act, int max_batch, const TView* part) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    SKPS_CHECK(dw_tma_supported(in, out, k, s, d, pad), "dw_tma: unsupported layer");
    const bool split = in.fmt == DT_SPLIT16;
    const int CB = split ? 64 : 32, esz = split ? 2 : 4;
    const int tht = dw_tile_rows(k, s);
    const int IH = (tht - 1) * s + (k - 1) * d + 1, IW = (TW - 1) * s + (k - 1) * d + 1;
    for (int plane = 0; plane < (split ? 2 : 1); ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)in.C, (cuuint64_t)in.W, (cuuint64_t)in.H, (cuuint64_t)max_batch};
        cuuint64_t strides[3] = {(cuuint64_t)in.ld * esz, (cuuint64_t)in.W * in.ld * esz, (cuuint64_t)in.H * in.W * in.ld * esz};
        cuuint32_t box[4] = {(cuuint32_t)CB, (cuuint32_t)IW, (cuuint32_t)IH, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        char* base = (char*)in.base + (size_t)in.c_off * esz + (plane ? (size_t)in.plane * 2 : 0);
        CUresult r = enc(plane ? &L.lo : &L.hi, split ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4,
                         base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(dw) failed: %d", (int)r);
    }
    if (!split) L.lo = L.hi;
    DwTmaK& kk = L.k;
    kk.C = in.C; kk.Ho = out.H; kk.Wo = out.W; kk.pad = pad; kk.act = act; kk.img0 = 0;
    kk.w = w; kk.bias = bias; kk.w_ld = in.C;
    kk.out = out.base; kk.out_fmt = out.fmt; kk.out_plane = out.plane; kk.out_ld = out.ld; kk.out_coff = out.c_off;
    kk.part = nullptr; kk.part_ld = 0; kk.part_coff = 0;
    if (part && part->base) {
        const int tiles = ((out.H + tht - 1) / tht) * ((out.W + TW - 1) / TW);
        SKPS_CHECK(part->fmt == DT_F32 && part->c_stride == 1 && part->C == in.C && part->H * part->W == tiles &&
                   ((part->ld | part->c_off) & 3) == 0, "dw_tma: partial-sum view must be float32 [tiles=%d][C]", tiles);
        kk.part = (float*)part->base; kk.part_ld = part->ld; kk.part_coff = part->c_off;
    }
    L.k_size = k; L.stride = s; L.dil = d; L.split = split ? 1 : 0;
    L.chunks = (in.C + CB - 1) / CB;
    L.smem_bytes = IH * IW * 128 * (split ? 2 : 1) + 128;
    return 0;
}

template <int K, int S, int D, bool SPLIT>
static int launch_variant(const DwTmaLayer& L, const DwTmaK& k, dim3 grid, cudaStream_t stream) {
    constexpr int RY = (K == 5 && S == 1) ? 2 : 1;      // dw_tile_rows(K, S) / TH
    static int attr_bytes[MAX_DEVICES] = {};
    if (smem_limit((const void*)dw_tma_kernel<K, S, D, SPLIT, RY>, attr_bytes, 200 * 1024)) return 1;
    dw_tma_kernel<K, S, D, SPLIT, RY><<<grid, DW_THREADS, L.smem_bytes, stream>>>(L.hi, L.lo, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

int dw_tma_launch(const DwTmaLayer& L, int batch, cudaStream_t stream) {
    DwTmaK k = L.k;
    k.chunks = L.chunks;
    k.batch = batch;
    const int tht = dw_tile_rows(L.k_size, L.stride);
    dim3 grid(((k.Ho + tht - 1) / tht) * ((k.Wo + TW - 1) / TW), L.chunks, batch);
#define DW_CASE(K_, S_, D_)                                                                              \
    if (L.k_size == K_ && L.stride == S_ && L.dil == D_)                                                 \
        return L.split ? launch_variant<K_, S_, D_, true>(L, k, grid, stream)                            \
                       : launch_variant<K_, S_, D_, false>(L, k, grid, stream);
    DW_CASE(3, 1, 1) DW_CASE(3, 2, 1) DW_CASE(5, 1, 1) DW_CASE(5, 2, 1) DW_CASE(5, 1, 2)
#undef DW_CASE
    set_error("dw_tma: variant k=%d s=%d d=%d not instantiated", L.k_size, L.stride, L.dil);
    return 1;
}


bool upcat_tma_supported(const TView& low, const TView& skip, const TView& out) {
    if (low.fmt != DT_F32 || low.c_stride != 1 || out.c_stride != 1) return false;
    if ((low.C | low.ld | low.c_off | out.ld | out.c_off) & 7) return false;
    if (out.H != 2 * low.H || out.W != 2 * low.W || (out.H & 1) || (out.W & 1)) return false;
    TView o2 = out;
    o2.c_off += low.C; o2.C = skip.C;
    return dw_tma_supported(skip, o2, 3, 1, 1, 1);
}

int upcat_tma_prepare(UpcatTmaLayer& L, const TView& low, const TView& skip, const TView& out, const float* w,
                      const float* bias, int act, int max_batch) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    SKPS_CHECK(upcat_tma_supported(low, skip, out), "upcat_tma: unsupported layer");
    cuuint64_t dims[4] = {(cuuint64_t)low.C, (cuuint64_t)low.W, (cuuint64_t)low.H, (cuuint64_t)max_batch};
    cuuint64_t strides[3] = {(cuuint64_t)low.ld * 4, (cuuint64_t)low.W * low.ld * 4, (cuuint64_t)low.H * low.W * low.ld * 4};
    cuuint32_t box[4] = {32, (cuuint32_t)LW, (cuuint32_t)LH, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&L.low, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (char*)low.base + (size_t)low.c_off * 4, dims, strides, box,
                     estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(upcat) failed: %d", (int)r);
    const int Ctot = low.C + skip.C;
    DwTmaK& k = L.k;
    k.C = low.C; k.Ho = out.H; k.Wo = out.W; k.pad = 1; k.act = act; k.img0 = 0; k.w_ld = Ctot;
    k.w = w; k.bias = bias;
    k.out = out.base; k.out_fmt = out.fmt; k.out_plane = out.plane; k.out_ld = out.ld; k.out_coff = out.c_off;
    L.Hl = low.H; L.Wl = low.W;
    L.chunks = (low.C + 31) / 32;
    L.smem_bytes = LH * LW * 128 + (TH + 2) * (TW + 2) * 32 * 4 + 128;     // low tile + staged up-sampled window
    // skip channels: an ordinary depthwise layer over the channel slice [Cu, Ctot)
    TView o2 = out;
    o2.c_off += low.C; o2.C = skip.C;
    if (dw_tma_prepare(L.skip, skip, o2, w + low.C, bias + low.C, 3, 1, 1, 1, act, max_batch, nullptr)) return 1;
    L.skip.k.w_ld = Ctot;
    return 0;
}

int upcat_tma_launch(const UpcatTmaLayer& L, int batch, cudaStream_t stream) {
    const DwTmaK& k = L.k;
    dim3 grid(((k.Ho + TH - 1) / TH) * ((k.Wo + TW - 1) / TW), L.chunks, batch);
    upcat_tma_kernel<<<grid, DW_THREADS, L.smem_bytes, stream>>>(L.low, k, L.Hl, L.Wl);
    SKPS_CUDA(cudaGetLastError());
    return dw_tma_launch(L.skip, batch, stream);
}

}  // namespace skps
