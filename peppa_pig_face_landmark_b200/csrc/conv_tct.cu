// Dense k x k convolution as a TRANSPOSED wgmma implicit GEMM (sm_90a): output channels as M, pixels as N.
//
//   D[M = 128 channel rows][N = 256 pixels] = sum over taps, ci of  W[co][tap][ci] * X[pixel + tap][ci]
//
// Why: conv_tc.cu computes C[128 pixels][Cout]; with Cout = 128 both operands of every MMA come from shared memory and the
// TMA fill and the epilogue staging compete with the tensor cores for its bandwidth.  With the weights as the 128-row A
// operand and 256 pixels as N, a tile reuses each weight slice for twice the pixels.  Same fp16 hi/lo three-product scheme,
// same 4-D TMA activation boxes (padding / dilation = OOB fill) and K-padded weight matrix as conv_tc.
//
// Tile = 256 pixels = bh whole rows of one image (W | 256).  Stage = one (tap, 64-channel chunk): weights 2 x 16 KB +
// activations 2 x 32 KB; two stages.  Warpgroups 1 and 2 each accumulate 128 channels x 128 pixels (pixel columns [0,128) and
// [128,256)) in registers with m64n128k16 wgmma, one k-block's group kept in flight while the next is issued, and run the
// epilogue on them straight from the accumulator fragment: bias / activation / fp16 hi-lo split, written TRANSPOSED
// (pixel rows of 32 channels) into the warpgroup's 16 KB staging buffer, 32 pixels at a time, which leaves as one TMA store
// per 32-channel quarter and plane, so the NHWC layout of the output is unchanged.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <string.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_tct.h"
#include "tc_ptx.h"

namespace skps {

constexpr int TCT_THREADS = 288;         // warps 0-7 MMA + epilogue (two warpgroups), warp 8 TMA
constexpr int TCT_M = 128, TCT_N = 256;
constexpr int TCT_W_TILE = TCT_M * 128;  // weights of one k-block, one plane: 128 rows x 128 B
constexpr int TCT_X_TILE = TCT_N * 128;  // activations of one k-block, one plane: 256 pixel rows x 128 B
constexpr int TCT_STAGE = 2 * TCT_W_TILE + 2 * TCT_X_TILE;      // 96 KB
constexpr int TCT_STAGES = 2;

template <int ACT>
__global__ void __launch_bounds__(TCT_THREADS, 1)
conv_tct_kernel(const __grid_constant__ CUtensorMap tmX_hi, const __grid_constant__ CUtensorMap tmX_lo,
                const __grid_constant__ CUtensorMap tmW_hi, const __grid_constant__ CUtensorMap tmW_lo,
                const __grid_constant__ CUtensorMap tmO_hi, const __grid_constant__ CUtensorMap tmO_lo, const TctK p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[TCT_STAGES], empty_bar[TCT_STAGES];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t out_off = base + (uint32_t)TCT_STAGES * TCT_STAGE;       // 2 epilogue warpgroups x 16 KB
    const int tiles = p.m_tiles;
    const int kblocks = p.taps * p.cchunks;

    if (warp == 8 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW_lo) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < TCT_STAGES; ++s) {
            mbar_init(smem_u32(&full_bar[s]), 1);
            mbar_init(smem_u32(&empty_bar[s]), 8);            // one arrival per MMA warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        // ================================================================== TMA producer
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
                const int img_l = tile / p.tiles_per_img, t = tile - img_l * p.tiles_per_img;
                const int y0 = t * p.bh;
                for (int kb = 0; kb < kblocks; ++kb) {
                    const int tap = kb / p.cchunks, cc = kb - tap * p.cchunks;
                    const int ky = tap / p.kw, kx = tap - ky * p.kw;
                    mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1u);
                    const uint32_t fb = smem_u32(&full_bar[stage]);
                    mbar_expect_tx(fb, (uint32_t)TCT_STAGE);
                    const uint32_t ss = base + (uint32_t)stage * TCT_STAGE;
                    tma_load_2d(ss, &tmW_hi, fb, kb * 64, 0);
                    tma_load_2d(ss + TCT_W_TILE, &tmW_lo, fb, kb * 64, 0);
                    const int cx = kx * p.dil - p.pad, cy = y0 + ky * p.dil - p.pad;
                    tma_load_4d(ss + 2 * TCT_W_TILE, &tmX_hi, fb, cc * 64, cx, cy, img_l + p.img0);
                    tma_load_4d(ss + 2 * TCT_W_TILE + TCT_X_TILE, &tmX_lo, fb, cc * 64, cx, cy, img_l + p.img0);
                    if (++stage == TCT_STAGES) { stage = 0; phase ^= 1u; }
                }
            }
        }
    } else {
        // ================================================================== MMA + epilogue
        // Warpgroup half_id accumulates all 128 channel rows x pixel columns [128 half_id, 128 half_id + 128): one
        // m64n128 accumulator per 64-row half, acc[64 m + 4 i + e] = channel 64m + 16q + lane/4 + 8(e/2), column
        // 8i + 2(lane%4) + e%2.
        const int q = warp & 3;
        const int half_id = warp >> 2;
        const bool leader = q == 0 && lane == 0;       // issues and drains the warpgroup's TMA stores
        float bias[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int c = 64 * (r >> 1) + 16 * q + (lane >> 2) + 8 * (r & 1);
            bias[r] = c < p.Cout ? __ldg(p.bias + c) : 0.f;
        }
        // the warpgroup's 16 KB staging buffer: per 32-channel quarter [hi: 32 pixel rows x 64 B][lo: same].  Pixel j of a
        // 32-pixel block is row j; channel c of quarter c/32 sits in 16-byte chunk ((c%32)/8) ^ ((j/2)%4) of that row (64-byte
        // swizzle).  A thread's pixels are j = 8i + 2(lane%4) + e%2, so (j/2)%4 = lane%4 and its address for row class r =
        // 2m + e/2 is row_addr[r] + 64 (8i + e%2).
        const uint32_t sbuf = out_off + (uint32_t)half_id * 16384u;
        uint32_t row_addr[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int cq = 16 * (q & 1) + (lane >> 2) + 8 * (r & 1);       // channel within its quarter
            row_addr[r] = sbuf + (uint32_t)(2 * (r >> 1) + (q >> 1)) * 4096u + (uint32_t)(2 * (lane & 3)) * 64u +
                          (uint32_t)((((cq >> 3) ^ (lane & 3)) & 3) << 4) + (uint32_t)(cq & 7) * 2u;
        }
        // 16-channel steps of the last 64-channel chunk that hold real channels (TMA zero-fills the rest)
        const int ks_last = min(4, (p.Cin - (p.cchunks - 1) * 64 + 15) / 16);
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
            const int img_l = tile / p.tiles_per_img, t = tile - img_l * p.tiles_per_img;
            float acc[128];
            int prev = 0;
            for (int kb = 0; kb < kblocks; ++kb) {
                mbar_wait(smem_u32(&full_bar[stage]), phase);
                const uint32_t ss = base + (uint32_t)stage * TCT_STAGE;
                const uint64_t w_hi = make_smem_desc(ss), w_lo = make_smem_desc(ss + TCT_W_TILE);
                const uint32_t xo = ss + 2 * TCT_W_TILE + (uint32_t)(half_id * 128 * 128);
                const uint64_t x_hi = make_smem_desc(xo), x_lo = make_smem_desc(xo + TCT_X_TILE);
                const int ks = kb % p.cchunks == p.cchunks - 1 ? ks_last : 4;
                const uint32_t accumulate = kb != 0;
                wg_fence_acc(acc);
                switch (ks) {                          // uniform over the CTA
                    case 4: wg_fence(); wg_mma3_128x128<4>(acc, w_hi, w_lo, x_hi, x_lo, accumulate); wg_commit(); break;
                    case 3: wg_fence(); wg_mma3_128x128<3>(acc, w_hi, w_lo, x_hi, x_lo, accumulate); wg_commit(); break;
                    case 2: wg_fence(); wg_mma3_128x128<2>(acc, w_hi, w_lo, x_hi, x_lo, accumulate); wg_commit(); break;
                    default: wg_fence(); wg_mma3_128x128<1>(acc, w_hi, w_lo, x_hi, x_lo, accumulate); wg_commit(); break;
                }
                wg_fence_acc(acc);
                // keep this k-block's group in flight; the previous one has finished reading its stage
                wg_wait<1>();
                wg_fence_acc(acc);
                if (kb > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
                prev = stage;
                if (++stage == TCT_STAGES) { stage = 0; phase ^= 1u; }
            }
            wg_wait<0>();
            wg_fence_acc(acc);
            if (lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
#pragma unroll
            for (int ci = 0; ci < 4; ++ci) {
                if (leader) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the buffer's last store has drained
                asm volatile("bar.sync %0, 128;" ::"r"(5 + half_id) : "memory");
                // bias / activation / fp16 hi-lo split straight from the fragment into the staging rows
#pragma unroll
                for (int m = 0; m < 2; ++m)
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float f = act_t<ACT>(fmaf(acc[64 * m + 16 * ci + 4 * i + e], p.out_scale, bias[2 * m + (e >> 1)]));
                            const __half h = __float2half_rn(f);
                            const __half l = __float2half_rn(f - __half2float(h));
                            const uint32_t a = row_addr[2 * m + (e >> 1)] + (uint32_t)(8 * i + (e & 1)) * 64u;
                            asm volatile("st.shared.b16 [%0], %1;" ::"r"(a), "h"(__half_as_ushort(h)) : "memory");
                            asm volatile("st.shared.b16 [%0], %1;" ::"r"(a + 2048u), "h"(__half_as_ushort(l)) : "memory");
                        }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                asm volatile("bar.sync %0, 128;" ::"r"(5 + half_id) : "memory");
                if (leader) {
                    const int col0 = half_id * 128 + ci * 32;              // first pixel of the block inside the tile
                    const int x0 = col0 % p.W, y0 = t * p.bh + col0 / p.W;
                    for (int cq = 0; cq < 4 && cq * 32 < p.Cout; ++cq) {   // quarters past Cout hold zero rows
                        const uint32_t sq = sbuf + (uint32_t)cq * 4096u;
                        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                     ::"l"(&tmO_hi), "r"(sq), "r"(cq * 32), "r"(x0), "r"(y0), "r"(img_l + p.img0) : "memory");
                        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                     ::"l"(&tmO_lo), "r"(sq + 2048u), "r"(cq * 32), "r"(x0), "r"(y0), "r"(img_l + p.img0) : "memory");
                    }
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

// ------------------------------------------------------------------------------------------ host side
// The layers this kernel is for: tensor-bound k x k convs whose Cout fills the 128 accumulator rows (else the rows idle and
// the pixels-as-rows kernel wins), whole 256-pixel row blocks, split-fp16 contiguous output, no residual.
bool tct_applicable(const TcSetup& s) {
    const int stride = s.stride > 0 ? s.stride : 1;
    if (stride != 1 || s.kh != s.kw || s.kh < 3 || s.pad != s.dil * (s.kh - 1) / 2) return false;
    if (s.W < 16 || s.W > TCT_N || TCT_N % s.W || s.H % (TCT_N / s.W)) return false;
    if (s.Cin < 64 || (s.Cin % 8) || (s.in_ld % 8) || (s.in_coff % 8)) return false;
    // Cout from 96: below it the idle accumulator rows cost more than the operand reuse buys
    if (s.Cout < 96 || s.Cout > TCT_M || (s.Cout % 8) || s.n_tiles != 1) return false;
    if (s.res || s.hm_val || s.out_fmt != DT_SPLIT16 || s.out_cstride != 1 || (s.out_ld % 8) || (s.out_coff % 8)) return false;
    // SiLU's correctly rounded division is a subroutine call that does not fit beside the 128 accumulator registers without
    // spilling; conv_tc runs such layers
    if (s.act == ACT_SILU) return false;
    return true;
}

int tct_prepare(TctLayer& L, const TcSetup& s) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    SKPS_CHECK(tct_applicable(s), "conv_tct: layer not applicable");
    TctK& k = L.k;
    memset(&k, 0, sizeof(k));
    k.W = s.W; k.bh = TCT_N / s.W; k.tiles_per_img = s.H / k.bh;
    k.taps = s.kh * s.kw; k.kw = s.kw; k.dil = s.dil; k.pad = s.pad;
    k.cchunks = (s.Cin + 63) / 64; k.Cin = s.Cin; k.Cout = s.Cout; k.act = s.act; k.out_scale = s.out_scale;
    SKPS_CHECK(s.bias, "conv_tct: bias required");
    k.bias = s.bias;
    L.smem_bytes = TCT_STAGES * TCT_STAGE + 8 * 4096 + 1024;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)s.Cin, (cuuint64_t)s.W, (cuuint64_t)s.H, (cuuint64_t)s.max_batch};
        cuuint64_t strides[3] = {(cuuint64_t)s.in_ld * 2, (cuuint64_t)s.W * s.in_ld * 2, (cuuint64_t)s.H * s.W * s.in_ld * 2};
        cuuint32_t box[4] = {64, (cuuint32_t)s.W, (cuuint32_t)k.bh, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        void* base = (void*)((__half*)s.in_base + (plane ? s.in_plane : 0) + s.in_coff);
        CUresult r = enc(plane ? &L.x_lo : &L.x_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(tct X) failed: %d", (int)r);
    }
    const int K_pad = k.taps * k.cchunks * 64;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)K_pad, (cuuint64_t)s.n_tile};        // rows beyond n_tile: OOB zero fill
        cuuint64_t strides[1] = {(cuuint64_t)K_pad * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)TCT_M};
        cuuint32_t estr[2] = {1, 1};
        void* base = (void*)(plane ? s.w_lo : s.w_hi);
        CUresult r = enc(plane ? &L.w_lo : &L.w_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(tct W) failed: %d", (int)r);
    }
    // output: one box per 32-channel quarter and 32-pixel block: 32 channels x 32 consecutive pixels, 64-byte swizzled rows
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)s.Cout, (cuuint64_t)s.W, (cuuint64_t)s.H, (cuuint64_t)s.max_batch};
        cuuint64_t strides[3] = {(cuuint64_t)s.out_ld * 2, (cuuint64_t)s.W * s.out_ld * 2, (cuuint64_t)s.H * s.W * s.out_ld * 2};
        const cuuint32_t obw = (cuuint32_t)(s.W < 32 ? s.W : 32);                // 32 consecutive pixels = 32/obw whole rows
        cuuint32_t box[4] = {32, obw, 32 / obw, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        char* base = (char*)s.out + (size_t)s.out_coff * 2 + (plane ? (size_t)s.out_plane * 2 : 0);
        CUresult r = enc(plane ? &L.o_lo : &L.o_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(tct out) failed: %d", (int)r);
    }
    return 0;
}

template <int ACT>
static int tct_launch_t(const TctLayer& L, const TctK& k, int grid, cudaStream_t stream) {
    static int attr_bytes = 0;
    if (L.smem_bytes > attr_bytes) {
        SKPS_CUDA(cudaFuncSetAttribute(conv_tct_kernel<ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, L.smem_bytes));
        attr_bytes = L.smem_bytes;
    }
    conv_tct_kernel<ACT><<<grid, TCT_THREADS, L.smem_bytes, stream>>>(L.x_hi, L.x_lo, L.w_hi, L.w_lo, L.o_hi, L.o_lo, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

Grid tct_grid(const TctLayer& L, int batch, int num_sms, TctK* kp) {
    TctK k = L.k;
    k.m_tiles = batch * k.tiles_per_img;
    if (kp) *kp = k;
    return persistent_grid(k.m_tiles, num_sms);
}

int tct_launch(const TctLayer& L, int batch, int num_sms, cudaStream_t stream) {
    TctK k;
    const int grid = tct_grid(L, batch, num_sms, &k).ctas;
    switch (k.act) {
        case ACT_NONE: return tct_launch_t<ACT_NONE>(L, k, grid, stream);
        case ACT_RELU: return tct_launch_t<ACT_RELU>(L, k, grid, stream);
        case ACT_HSWISH: return tct_launch_t<ACT_HSWISH>(L, k, grid, stream);
        case ACT_SIGMOID: return tct_launch_t<ACT_SIGMOID>(L, k, grid, stream);
        case ACT_HSIGMOID: return tct_launch_t<ACT_HSIGMOID>(L, k, grid, stream);
        default: break;
    }
    set_error("conv_tct: activation %d not instantiated", k.act);
    return 1;
}

}  // namespace skps
