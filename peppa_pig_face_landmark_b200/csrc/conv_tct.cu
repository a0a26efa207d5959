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
// [128,256)) in registers and run the epilogue on them: a thread owns one output channel and 32 pixels per chunk (wg_rows32);
// bias / activation / fp16 hi-lo split, then the 32 x 32 block is written TRANSPOSED into the
// warp's 4 KB staging slice (one 64-byte pixel row per store instruction, lane = channel) and leaves as one TMA store per
// plane, so the NHWC layout of the output is unchanged.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <string.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_tct.h"
#include "tc_ptx.h"

namespace skps {

constexpr int TCT_THREADS = 384;         // warp 0 TMA, 4-11 MMA + epilogue
constexpr int TCT_M = 128, TCT_N = 256;
constexpr int TCT_W_TILE = TCT_M * 128;  // weights of one k-block, one plane: 128 rows x 128 B
constexpr int TCT_X_TILE = TCT_N * 128;  // activations of one k-block, one plane: 256 pixel rows x 128 B
constexpr int TCT_STAGE = 2 * TCT_W_TILE + 2 * TCT_X_TILE;      // 96 KB
constexpr int TCT_STAGES = 2;

__global__ void __launch_bounds__(TCT_THREADS, 1)
conv_tct_kernel(const __grid_constant__ CUtensorMap tmX_hi, const __grid_constant__ CUtensorMap tmX_lo,
                const __grid_constant__ CUtensorMap tmW_hi, const __grid_constant__ CUtensorMap tmW_lo,
                const __grid_constant__ CUtensorMap tmO_hi, const __grid_constant__ CUtensorMap tmO_lo, const TctK p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[TCT_STAGES], empty_bar[TCT_STAGES];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t out_off = base + (uint32_t)TCT_STAGES * TCT_STAGE;       // 8 epilogue warps x 4 KB
    const int tiles = p.m_tiles;
    const int kblocks = p.taps * p.cchunks;

    if (warp == 0 && lane == 0) {
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

    if (warp == 0) {
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
    } else if (warp >= 4) {
        // ================================================================== MMA + epilogue: lane = output channel, columns = pixels
        const int q = warp & 3;                        // channels 32q .. 32q+31 in the epilogue
        const int half_id = (warp - 4) >> 2;           // pixel columns [0,128) or [128,256)
        const int c = q * 32 + lane;
        const float bias = c < p.Cout ? __ldg(p.bias + c) : 0.f;
        const uint32_t sbuf = out_off + (uint32_t)(warp - 4) * 4096u;       // [hi: 32 pixel rows x 64 B][lo: same]
        const bool q_ok = q * 32 < p.Cout;             // quarters past Cout hold zero rows: nothing to store
        // the warpgroup's four 4 KB staging slices double as its accumulator hand-off buffer (wg_rows32)
        float* xs = reinterpret_cast<float*>(smem_raw + (out_off - smem_u32(smem_raw))) + half_id * 4096;
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
            const int img_l = tile / p.tiles_per_img, t = tile - img_l * p.tiles_per_img;
            float accv[4][32];                         // 32-pixel chunk ci of this warpgroup's 128 columns
            for (int kb = 0; kb < kblocks; ++kb) {
                mbar_wait(smem_u32(&full_bar[stage]), phase);
                const uint32_t ss = base + (uint32_t)stage * TCT_STAGE;
                const uint64_t w_hi = make_smem_desc(ss), w_lo = make_smem_desc(ss + TCT_W_TILE);
                const uint32_t xo = ss + 2 * TCT_W_TILE + (uint32_t)(half_id * 128 * 128);
                const int cc = kb % p.cchunks;
                const int ksteps = min(4, (p.Cin - cc * 64 + 15) / 16);
                wg_fence();
#pragma unroll
                for (int ci = 0; ci < 4; ++ci) {
                    const uint64_t x_hi = make_smem_desc(xo + (uint32_t)(ci * 32 * 128));
                    const uint64_t x_lo = make_smem_desc(xo + (uint32_t)(ci * 32 * 128) + TCT_X_TILE);
                    for (int k = 0; k < ksteps; ++k) {
                        const uint64_t koff = (uint64_t)(k * 32 >> 4);
                        wg_mma3_128x32(accv[ci], w_hi + koff, w_lo + koff, 64u * 128u, x_hi + koff, x_lo + koff, (kb | k) != 0);
                    }
                }
                wg_commit();
                wg_wait0();
                if (lane == 0) mbar_arrive(smem_u32(&empty_bar[stage]));
                if (++stage == TCT_STAGES) { stage = 0; phase ^= 1u; }
            }
#pragma unroll
            for (int ci = 0; ci < 4; ++ci) {
                float v[32];
                if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");      // the slice's previous store has drained
                asm volatile("bar.sync %0, 128;" ::"r"(5 + half_id) : "memory");   // ... in all four slices wg_rows32 writes
                wg_rows32(accv[ci], xs, 5 + half_id, q, lane, v);
                if (!q_ok) continue;
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const float f = apply_act(fmaf(v[j], p.out_scale, bias), p.act);
                    const __half h = __float2half_rn(f);
                    const __half l = __float2half_rn(f - __half2float(h));
                    // pixel row j of the block: 64 bytes = 32 channels; the 32 lanes fill one row per store instruction
                    asm volatile("st.shared.b16 [%0], %1;" ::"r"(sbuf + (uint32_t)(j * 64 + lane * 2)), "h"(__half_as_ushort(h)) : "memory");
                    asm volatile("st.shared.b16 [%0], %1;" ::"r"(sbuf + 2048u + (uint32_t)(j * 64 + lane * 2)), "h"(__half_as_ushort(l)) : "memory");
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if (lane == 0) {
                    const int col0 = half_id * 128 + ci * 32;              // first pixel of the block inside the tile
                    const int x0 = col0 % p.W, y0 = t * p.bh + col0 / p.W;
                    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                 ::"l"(&tmO_hi), "r"(sbuf), "r"(q * 32), "r"(x0), "r"(y0), "r"(img_l + p.img0) : "memory");
                    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                 ::"l"(&tmO_lo), "r"(sbuf + 2048u), "r"(q * 32), "r"(x0), "r"(y0), "r"(img_l + p.img0) : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
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
    // output: one box per epilogue warp and 32-pixel block: 32 channels x 32 consecutive pixels of a row, plain 64-byte rows
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)s.Cout, (cuuint64_t)s.W, (cuuint64_t)s.H, (cuuint64_t)s.max_batch};
        cuuint64_t strides[3] = {(cuuint64_t)s.out_ld * 2, (cuuint64_t)s.W * s.out_ld * 2, (cuuint64_t)s.H * s.W * s.out_ld * 2};
        const cuuint32_t obw = (cuuint32_t)(s.W < 32 ? s.W : 32);                // 32 consecutive pixels = 32/obw whole rows
        cuuint32_t box[4] = {32, obw, 32 / obw, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        char* base = (char*)s.out + (size_t)s.out_coff * 2 + (plane ? (size_t)s.out_plane * 2 : 0);
        CUresult r = enc(plane ? &L.o_lo : &L.o_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(tct out) failed: %d", (int)r);
    }
    L.valid = true;
    return 0;
}

int tct_launch(const TctLayer& L, int batch, int num_sms, cudaStream_t stream) {
    static int attr_bytes = 0;
    if (L.smem_bytes > attr_bytes) {
        SKPS_CUDA(cudaFuncSetAttribute(conv_tct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L.smem_bytes));
        attr_bytes = L.smem_bytes;
    }
    TctK k = L.k;
    k.m_tiles = batch * k.tiles_per_img;
    const int grid = k.m_tiles < num_sms ? k.m_tiles : num_sms;
    conv_tct_kernel<<<grid, TCT_THREADS, L.smem_bytes, stream>>>(L.x_hi, L.x_lo, L.w_hi, L.w_lo, L.o_hi, L.o_lo, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace skps
