// Heat-map head of the landmark networks as a TRANSPOSED wgmma GEMM with the arg-max in the epilogue (sm_90a).
//
//   scores[co][pixel] = bias[co] + sum_ci W[co][ci] * x[pixel][ci]          (kps graph: /student/hm/Conv, 1x1, no activation)
//   postp (TRAIN/.../model.py:511-554) needs, per score map, only the maximum and the first arg-max.
//
// conv_tc.cu computes C[pixel][co] (pixels as accumulator rows); reducing over pixels then needs a warp reduce-scatter of
// every 32-column chunk and the epilogue, not the tensor cores or HBM, bounds the layer.  Here the operands swap roles:
//     D[M = 128 channel rows][N = 256 pixels] = W[128][K] * X[256][K]^T
// so an accumulator row IS a score map and the pixels of the tile are its columns: each epilogue thread scans its columns
// of its rows with a running (max, first index), a quad shuffle and one exchange between the two warpgroups finish the
// row, and one (max, arg-max) pair per tile and channel is written, which OP_HM_DECODE combines (same partial-row format as
// conv_tc's FLAG_HM_PART path, 256-pixel tiles instead of 128).
// The weight matrix (<= 128 x 128, hi/lo) is fetched once per persistent CTA and stays in shared memory; activations
// stream through a 2-stage ring of [256 pixels][64 channels] hi/lo boxes (4-D TMA straight from the NHWC tensor).
// Precision scheme as everywhere: fp16 hi/lo operands, three MMAs per K-step into one fp32 register accumulator.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_hm.h"
#include "tc_ptx.h"

namespace skps {

constexpr int HM_THREADS = 384;          // warp 0 TMA, 4-11 MMA + epilogue
constexpr int HM_M = 128;                // channel rows of the accumulator (Cout <= 128, zero rows above)
constexpr int HM_N = 256;                // pixels per tile
constexpr int HM_W_TILE = HM_M * 128;    // one 64-channel K chunk of the weights, one plane: 128 rows x 128 B
constexpr int HM_X_TILE = HM_N * 128;    // one K chunk of a pixel tile, one plane
constexpr int HM_STAGES = 2;

__global__ void __launch_bounds__(HM_THREADS, 1)
conv_hm_kernel(const __grid_constant__ CUtensorMap tmX_hi, const __grid_constant__ CUtensorMap tmX_lo,
               const __grid_constant__ CUtensorMap tmW_hi, const __grid_constant__ CUtensorMap tmW_lo, const HmK p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t w_bar, full_bar[HM_STAGES], empty_bar[HM_STAGES];
    __shared__ float xch_v[2][HM_M];
    __shared__ int xch_i[2][HM_M];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t w_off = base;                                            // [chunk][plane][128 x 128 B]
    const uint32_t x_off = w_off + (uint32_t)p.cchunks * 2u * HM_W_TILE;    // [stage][plane][256 x 128 B]
    const int tiles = p.m_tiles;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW_lo) : "memory");
    }
    if (warp == 1 && lane == 0) {
        mbar_init(smem_u32(&w_bar), 1);
        for (int s = 0; s < HM_STAGES; ++s) {
            mbar_init(smem_u32(&full_bar[s]), 1);
            mbar_init(smem_u32(&empty_bar[s]), 8);            // one arrival per MMA warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        // ================================================================== TMA producer
        if (lane == 0) {
            // the whole weight matrix once: rows past the packed matrix (Cout rounded up to 16) are zero-filled by TMA
            const uint32_t wb = smem_u32(&w_bar);
            mbar_expect_tx(wb, (uint32_t)p.cchunks * 2u * HM_W_TILE);
            for (int kc = 0; kc < p.cchunks; ++kc) {
                tma_load_2d(w_off + (uint32_t)(kc * 2) * HM_W_TILE, &tmW_hi, wb, kc * 64, 0);
                tma_load_2d(w_off + (uint32_t)(kc * 2 + 1) * HM_W_TILE, &tmW_lo, wb, kc * 64, 0);
            }
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
                const int img_l = tile / p.tiles_per_img, t = tile - img_l * p.tiles_per_img;
                const int y0 = t * p.bh;
                for (int kc = 0; kc < p.cchunks; ++kc) {
                    mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1u);
                    const uint32_t fb = smem_u32(&full_bar[stage]);
                    mbar_expect_tx(fb, 2u * HM_X_TILE);
                    const uint32_t sx = x_off + (uint32_t)stage * 2u * HM_X_TILE;
                    tma_load_4d(sx, &tmX_hi, fb, kc * 64, 0, y0, img_l + p.img0);
                    tma_load_4d(sx + HM_X_TILE, &tmX_lo, fb, kc * 64, 0, y0, img_l + p.img0);
                    if (++stage == HM_STAGES) { stage = 0; phase ^= 1u; }
                }
            }
        }
    } else if (warp >= 4) {
        // ================================================================== MMA + epilogue: rows = score maps, columns = pixels
        // Warpgroup half_id accumulates pixel columns [128 half_id, 128 half_id + 128) of all 128 channel rows.  A thread holds
        // channel rows 64m + 16q + lane/4 + 8h (m, h in {0, 1}) and, per 32-pixel chunk ci, columns 8i + 2(lane%4) + {0, 1}.
        const int q = warp & 3;
        const int half_id = (warp - 4) >> 2;
        float bias[4];
        int ch[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            ch[r] = 64 * (r >> 1) + 16 * q + (lane >> 2) + 8 * (r & 1);
            bias[r] = ch[r] < p.Cout ? __ldg(p.bias + ch[r]) : 0.f;
        }
        mbar_wait(smem_u32(&w_bar), 0);
        int stage = 0;
        uint32_t phase = 0;
        int xb = 0;
        for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
            const int img_l = tile / p.tiles_per_img, t = tile - img_l * p.tiles_per_img;
            float acc[128];                            // acc[64 m + 4 i + e]: rows 64m + 16q + lane/4 + 8(e/2), column 8i + ...
            int prev = 0;
            for (int kc = 0; kc < p.cchunks; ++kc) {
                mbar_wait(smem_u32(&full_bar[stage]), phase);
                const uint32_t sx = x_off + (uint32_t)stage * 2u * HM_X_TILE + (uint32_t)(half_id * 128 * 128);
                const uint64_t w_hi = make_smem_desc(w_off + (uint32_t)(kc * 2) * HM_W_TILE);
                const uint64_t w_lo = make_smem_desc(w_off + (uint32_t)(kc * 2 + 1) * HM_W_TILE);
                const uint64_t x_hi = make_smem_desc(sx), x_lo = make_smem_desc(sx + HM_X_TILE);
                const uint32_t accumulate = kc != 0;
                wg_fence_acc(acc);
                switch (min(4, (p.Cin - kc * 64 + 15) / 16)) {   // 16-channel steps that hold real channels; uniform
                    case 4: wg_fence(); wg_mma3_128x128<4>(acc, w_hi, w_lo, x_hi, x_lo, accumulate); wg_commit(); break;
                    case 3: wg_fence(); wg_mma3_128x128<3>(acc, w_hi, w_lo, x_hi, x_lo, accumulate); wg_commit(); break;
                    case 2: wg_fence(); wg_mma3_128x128<2>(acc, w_hi, w_lo, x_hi, x_lo, accumulate); wg_commit(); break;
                    default: wg_fence(); wg_mma3_128x128<1>(acc, w_hi, w_lo, x_hi, x_lo, accumulate); wg_commit(); break;
                }
                wg_fence_acc(acc);
                wg_wait<1>();                          // the previous chunk's group has finished reading its stage
                wg_fence_acc(acc);
                if (kc > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
                prev = stage;
                if (++stage == HM_STAGES) { stage = 0; phase ^= 1u; }
            }
            wg_wait<0>();
            wg_fence_acc(acc);
            if (lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
            // running (max, first arg-max) per channel row over this thread's columns, in increasing column order
            float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
            int bi[4] = {0x7fffffff, 0x7fffffff, 0x7fffffff, 0x7fffffff};
#pragma unroll
            for (int ci = 0; ci < 4; ++ci)
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
#pragma unroll
                        for (int m = 0; m < 2; ++m) {
                            const int r = 2 * m + (e >> 1);
                            const float sc = fmaf(acc[64 * m + 16 * ci + 4 * i + e], p.out_scale, bias[r]);  // as conv_tc forms it
                            const bool take = sc > best[r];                 // strict: ties keep the earlier pixel
                            best[r] = take ? sc : best[r];
                            bi[r] = take ? half_id * 128 + ci * 32 + 8 * i + 2 * (lane & 3) + (e & 1) : bi[r];
                        }
                    }
            // the four lanes of a quad hold interleaved columns of the same rows: equal maxima keep the smaller index
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int off = 1; off <= 2; off <<= 1) {
                    const float ov = __shfl_xor_sync(0xffffffffu, best[r], off);
                    const int oi = __shfl_xor_sync(0xffffffffu, bi[r], off);
                    if (ov > best[r] || (ov == best[r] && oi < bi[r])) { best[r] = ov; bi[r] = oi; }
                }
            if (half_id == 1 && (lane & 3) == 0) {
#pragma unroll
                for (int r = 0; r < 4; ++r) { xch_v[xb][ch[r]] = best[r]; xch_i[xb][ch[r]] = bi[r]; }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            if (half_id == 0 && (lane & 3) == 0) {
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (ch[r] >= p.Cout) continue;
                    float b = best[r];
                    int id = bi[r];
                    const float ov = xch_v[xb][ch[r]];
                    const int oi = xch_i[xb][ch[r]];
                    if (ov > b) { b = ov; id = oi; }                    // ties: the lower half holds the smaller indices
                    const long long o = ((long long)(img_l + p.img0) * p.tiles_per_img + t) * p.hm_ld + ch[r];
                    p.hm_val[o] = b;
                    p.hm_idx[o] = t * HM_N + id;                        // tiles are whole row blocks: pixel index = y * W + x
                }
            }
            xb ^= 1;
        }
    }
}

// ------------------------------------------------------------------------------------------ host side
bool hm_shape_ok(int H, int W, int Cin, int Cout, int in_ld, int in_coff) {
    if (W < 8 || W > HM_N || HM_N % W || (H * W) % HM_N) return false;      // whole 256-pixel row blocks
    if (Cin % 8 || Cin > 128 || Cout > HM_M || (in_ld % 8) || (in_coff % 8)) return false;
    return true;
}

int hm_prepare(HmLayer& L, const TcSetup& s) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    SKPS_CHECK(s.kh == 1 && s.kw == 1 && (s.stride <= 1) && s.act == ACT_NONE && !s.res && s.hm_val && s.hm_idx,
               "conv_hm: 1x1, linear, partial-maximum output only");
    SKPS_CHECK(hm_shape_ok(s.H, s.W, s.Cin, s.Cout, s.in_ld, s.in_coff), "conv_hm: unsupported shape %dx%d Cin=%d Cout=%d",
               s.H, s.W, s.Cin, s.Cout);
    SKPS_CHECK(s.n_tiles == 1 && s.hm_ld >= s.Cout && s.bias, "conv_hm: one weight tile, a bias, partial rows of >= Cout entries");
    HmK& k = L.k;
    memset(&k, 0, sizeof(k));
    k.bh = HM_N / s.W;
    k.tiles_per_img = s.H / k.bh;
    k.cchunks = (s.Cin + 63) / 64;
    k.Cin = s.Cin; k.Cout = s.Cout; k.out_scale = s.out_scale; k.bias = s.bias;
    k.hm_val = s.hm_val; k.hm_idx = s.hm_idx; k.hm_ld = s.hm_ld;
    L.smem_bytes = k.cchunks * 2 * HM_W_TILE + HM_STAGES * 2 * HM_X_TILE + 1024;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)s.Cin, (cuuint64_t)s.W, (cuuint64_t)s.H, (cuuint64_t)s.max_batch};
        cuuint64_t strides[3] = {(cuuint64_t)s.in_ld * 2, (cuuint64_t)s.W * s.in_ld * 2, (cuuint64_t)s.H * s.W * s.in_ld * 2};
        cuuint32_t box[4] = {64, (cuuint32_t)s.W, (cuuint32_t)k.bh, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        void* base = (void*)((__half*)s.in_base + (plane ? s.in_plane : 0) + s.in_coff);
        CUresult r = enc(plane ? &L.x_lo : &L.x_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(hm X) failed: %d", (int)r);
    }
    const int K_pad = k.cchunks * 64;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)K_pad, (cuuint64_t)s.n_tile};        // rows beyond n_tile: OOB zero fill
        cuuint64_t strides[1] = {(cuuint64_t)K_pad * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)HM_M};
        cuuint32_t estr[2] = {1, 1};
        void* base = (void*)(plane ? s.w_lo : s.w_hi);
        CUresult r = enc(plane ? &L.w_lo : &L.w_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(hm W) failed: %d", (int)r);
    }
    return 0;
}

Grid hm_grid(const HmLayer& L, int batch, int num_sms, HmK* kp) {
    HmK k = L.k;
    k.m_tiles = batch * k.tiles_per_img;
    if (kp) *kp = k;
    return persistent_grid(k.m_tiles, num_sms);
}

int hm_launch(const HmLayer& L, int batch, int num_sms, cudaStream_t stream) {
    static int attr_bytes[MAX_DEVICES] = {};
    if (smem_limit((const void*)conv_hm_kernel, attr_bytes, L.smem_bytes)) return 1;
    HmK k;
    const int grid = hm_grid(L, batch, num_sms, &k).ctas;
    conv_hm_kernel<<<grid, HM_THREADS, L.smem_bytes, stream>>>(L.x_hi, L.x_lo, L.w_hi, L.w_lo, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace skps

using namespace skps;

namespace {
__global__ void hm_f32_to_split(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = src[i];
    const __half h = __float2half_rn(v);
    hi[i] = h;
    lo[i] = __float2half_rn(v - __half2float(h));
}
}  // namespace

// Unit-test entry (tests/test_conv_tc_gpu.py): x (N,H,W,Cin) float32 host, w_hi/w_lo (n_tile, Kpad) float16 as packed by
// plan.pack_tc_weights -> per-tile partial rows val/idx [N][H*W/256][128] (float32 / int32, host).
extern "C" SKPS_API int skps_debug_conv_hm(const float* x, int N, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                                           const float* bias, int Cout, int n_tile, float out_scale, float* val, int* idx) {
    SKPS_CHECK(x && w_hi && w_lo && bias && val && idx && N > 0, "debug_conv_hm: null argument");
    SKPS_CHECK(hm_shape_ok(H, W, Cin, Cout, Cin, 0), "debug_conv_hm: unsupported shape");
    const long long nx = (long long)N * H * W * Cin;
    const int Kpad = (Cin + 63) / 64 * 64, tiles = H * W / HM_N, ld = HM_M;
    float *d_x = nullptr, *d_b = nullptr, *d_val = nullptr;
    int* d_idx = nullptr;
    __half *d_s = nullptr, *d_wh = nullptr, *d_wl = nullptr;
    SKPS_CUDA(cudaMalloc(&d_x, nx * 4));
    SKPS_CUDA(cudaMalloc(&d_s, nx * 4));
    SKPS_CUDA(cudaMalloc(&d_wh, (size_t)n_tile * Kpad * 2));
    SKPS_CUDA(cudaMalloc(&d_wl, (size_t)n_tile * Kpad * 2));
    SKPS_CUDA(cudaMalloc(&d_b, Cout * 4));
    SKPS_CUDA(cudaMalloc(&d_val, (size_t)N * tiles * ld * 4));
    SKPS_CUDA(cudaMalloc(&d_idx, (size_t)N * tiles * ld * 4));
    SKPS_CUDA(cudaMemset(d_val, 0, (size_t)N * tiles * ld * 4));
    SKPS_CUDA(cudaMemset(d_idx, 0, (size_t)N * tiles * ld * 4));
    SKPS_CUDA(cudaMemcpy(d_x, x, nx * 4, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(d_wh, w_hi, (size_t)n_tile * Kpad * 2, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(d_wl, w_lo, (size_t)n_tile * Kpad * 2, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(d_b, bias, Cout * 4, cudaMemcpyHostToDevice));
    hm_f32_to_split<<<(unsigned)((nx + 255) / 256), 256>>>(d_x, d_s, d_s + nx, nx);
    SKPS_CUDA(cudaGetLastError());
    TcSetup s = {};
    s.H = H; s.W = W; s.Cin = Cin; s.in_ld = Cin; s.in_coff = 0; s.max_batch = N;
    s.in_base = d_s; s.in_plane = nx;
    s.kh = s.kw = 1; s.dil = 1; s.pad = 0; s.stride = 1;
    s.Cout = Cout; s.act = ACT_NONE; s.n_tile = n_tile; s.n_tiles = 1; s.out_scale = out_scale;
    s.w_hi = d_wh; s.w_lo = d_wl; s.bias = d_b;
    s.hm_val = d_val; s.hm_idx = d_idx; s.hm_ld = ld;
    HmLayer L;
    int rc = hm_prepare(L, s);
    const int sms = sm_count();
    if (!rc) rc = hm_launch(L, N, sms, 0);
    if (!rc && cudaDeviceSynchronize() != cudaSuccess) { set_error("debug_conv_hm: kernel failed"); rc = 1; }
    if (!rc) {
        cudaMemcpy(val, d_val, (size_t)N * tiles * ld * 4, cudaMemcpyDeviceToHost);
        cudaMemcpy(idx, d_idx, (size_t)N * tiles * ld * 4, cudaMemcpyDeviceToHost);
    }
    cudaFree(d_x); cudaFree(d_s); cudaFree(d_wh); cudaFree(d_wl); cudaFree(d_b); cudaFree(d_val); cudaFree(d_idx);
    return rc;
}
