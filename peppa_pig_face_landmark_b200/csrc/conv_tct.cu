// Dense k x k convolution as a TRANSPOSED wgmma implicit GEMM (sm_90a): output channels as M, pixels as N.
//
//   D[M = 128 channel rows][N = 256 pixels] = sum over taps, ci of  W[co][tap][ci] * X[pixel + tap][ci]
//
// Why: conv_tc.cu computes C[128 pixels][Cout]; with Cout = 128 both operands of every MMA come from shared memory and the
// TMA fill and the epilogue staging compete with the tensor cores for its bandwidth.  With the weights as the 128-row A
// operand and 256 pixels as N, a tile reuses each weight slice for twice the pixels.  Same fp16 hi/lo three-product scheme,
// same 4-D TMA activation boxes (padding / dilation = OOB fill) and K-padded weight matrix as conv_tc.
//
// Tile = 256 pixels = bh whole rows of one image (W | 256).  K runs in the order (kx, 32-channel half-chunk, ky, 16-channel
// step), and the kh vertical taps of one (kx, half-chunk) read ONE activation load:
//   halo slot   = the bh + dil (kh - 1) input rows y0 - pad ... y0 + bh - 1 + pad at column shift kx dil - pad, W pixels x 64 B
//                 each (64-byte swizzle), hi and lo plane, one 4-D TMA box per plane (padding = OOB fill).  Tap ky's B operand
//                 is the slot from row ky dil on: a byte offset of ky dil W 64, a whole number of 512-byte swizzle atoms for
//                 every admitted W, and a warpgroup's 128 pixels are contiguous in it because whole rows are.
//   weight slot = the 128 x 32 slice of the packed matrix for one (tap, half-chunk), hi and lo: 16 KB.
// The two have their own mbarrier rings: three weight slots, and as many halo slots (at most three, at least two) as fit
// beside them and the epilogue staging; the MMA warps free a weight slot per tap and the halo slot after the last ky.  A
// tile so fetches each input row once per column shift kx, not once per tap.  Layers whose halo slot does not fit twice run
// on conv_tc.
// Warpgroups 1 and 2 each accumulate 128 channels x 128 pixels (pixel columns [0,128) and [128,256)) in registers with
// m64n128k16 wgmma, one tap's group kept in flight while the next is issued, and run the
// epilogue on them straight from the accumulator fragment: bias / activation / fp16 hi-lo split, written TRANSPOSED
// (pixel rows of 32 channels) into the warpgroup's 16 KB staging buffer, 32 pixels at a time, which leaves as one TMA store
// per 32-channel quarter and plane, so the NHWC layout of the output is unchanged.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <string.h>

#include <algorithm>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_tct.h"
#include "tc_ptx.h"

namespace skps {

constexpr int TCT_THREADS = 288;         // warps 0-7 MMA + epilogue (two warpgroups), warp 8 TMA
constexpr int TCT_M = 128, TCT_N = 256;
constexpr int TCT_KC = 32;               // channels per slot: one 64-byte swizzled row, two K-steps of 16
constexpr int TCT_W_PLANE = TCT_M * 2 * TCT_KC;      // weights of one (tap, half-chunk), one plane: 128 rows x 64 B
constexpr int TCT_W_SLOT = 2 * TCT_W_PLANE;          // 16 KB
constexpr int TCT_W_SLOTS = 3;
constexpr int TCT_MAX_X_SLOTS = 3;
constexpr int TCT_OUT_BYTES = 2 * 16384;             // epilogue staging of the two warpgroups
constexpr int TCT_SMEM_LIMIT = 227 * 1024 - 256;     // dynamic shared memory a CTA may ask for beside the barriers

template <int ACT>
__global__ void __launch_bounds__(TCT_THREADS, 1)
conv_tct_kernel(const __grid_constant__ CUtensorMap tmX_hi, const __grid_constant__ CUtensorMap tmX_lo,
                const __grid_constant__ CUtensorMap tmW_hi, const __grid_constant__ CUtensorMap tmW_lo,
                const __grid_constant__ CUtensorMap tmO_hi, const __grid_constant__ CUtensorMap tmO_lo, const TctK p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_w[TCT_W_SLOTS], empty_w[TCT_W_SLOTS], full_x[TCT_MAX_X_SLOTS],
        empty_x[TCT_MAX_X_SLOTS];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;            // the weight ring
    const uint32_t x_base = base + (uint32_t)TCT_W_SLOTS * TCT_W_SLOT;      // the halo ring
    const uint32_t x_slot = 2u * (uint32_t)p.x_plane;
    const uint32_t out_off = x_base + (uint32_t)p.x_slots * x_slot;         // 2 epilogue warpgroups x 16 KB
    const int tiles = p.m_tiles;
    const int kh = p.taps / p.kw;
    const int halves = (p.Cin + TCT_KC - 1) / TCT_KC;
    const int groups = p.kw * halves;                  // (kx, half-chunk) pairs of a tile, kx outer

    if (warp == 8 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW_lo) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < TCT_W_SLOTS; ++s) {
            mbar_init(smem_u32(&full_w[s]), 1);
            mbar_init(smem_u32(&empty_w[s]), 8);              // one arrival per MMA warp
        }
        for (int s = 0; s < p.x_slots; ++s) {
            mbar_init(smem_u32(&full_x[s]), 1);
            mbar_init(smem_u32(&empty_x[s]), 8);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        // ================================================================== TMA producer
        // The CTA's groups are numbered across its tiles, so the rings run ahead over tile boundaries.  Halo slot n + 1 is
        // requested after the first weight slice of group n: the MMA warps free a halo slot when the first tap of the next
        // group has been issued, so with two halo slots that slice must already be on its way.
        if (lane == 0 && (int)blockIdx.x < tiles) {
            const int total = ((tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x) * groups;
            int xs = 0, ws = 0;
            uint32_t xphase = 0, wphase = 0;
            auto load_halo = [&](int n) {
                const int i = n / groups, g = n - i * groups;
                const int kx = g / halves, hc = g - kx * halves;
                const int tile = (int)blockIdx.x + i * (int)gridDim.x;
                const int img_l = tile / p.tiles_per_img, t = tile - img_l * p.tiles_per_img;
                mbar_wait(smem_u32(&empty_x[xs]), xphase ^ 1u);
                const uint32_t fb = smem_u32(&full_x[xs]);
                mbar_expect_tx(fb, x_slot);
                const uint32_t sx = x_base + (uint32_t)xs * x_slot;
                const int cx = kx * p.dil - p.pad, cy = t * p.bh - p.pad;
                tma_load_4d(sx, &tmX_hi, fb, hc * TCT_KC, cx, cy, img_l + p.img0);
                tma_load_4d(sx + (uint32_t)p.x_plane, &tmX_lo, fb, hc * TCT_KC, cx, cy, img_l + p.img0);
                if (++xs == p.x_slots) { xs = 0; xphase ^= 1u; }
            };
            load_halo(0);
            for (int n = 0, g = 0; n < total; ++n) {
                const int kx = g / halves, hc = g - kx * halves;
                for (int ky = 0; ky < kh; ++ky) {
                    mbar_wait(smem_u32(&empty_w[ws]), wphase ^ 1u);
                    const uint32_t fb = smem_u32(&full_w[ws]);
                    mbar_expect_tx(fb, (uint32_t)TCT_W_SLOT);
                    const uint32_t sw = base + (uint32_t)ws * TCT_W_SLOT;
                    const int col = (ky * p.kw + kx) * p.cchunks * 64 + hc * TCT_KC;
                    tma_load_2d(sw, &tmW_hi, fb, col, 0);
                    tma_load_2d(sw + TCT_W_PLANE, &tmW_lo, fb, col, 0);
                    if (++ws == TCT_W_SLOTS) { ws = 0; wphase ^= 1u; }
                    if (ky == 0 && n + 1 < total) load_halo(n + 1);
                }
                if (++g == groups) g = 0;
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
        // 16-channel steps of the last half-chunk that hold real channels (TMA zero-fills the rest)
        const int ks_last = (p.Cin - (halves - 1) * TCT_KC + 15) / 16;
        const uint32_t tap_step = (uint32_t)(p.dil * p.W * 2 * TCT_KC);     // bytes between the rows of taps ky and ky + 1
        int xs = 0, ws = 0;
        uint32_t xphase = 0, wphase = 0;
        for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
            const int img_l = tile / p.tiles_per_img, t = tile - img_l * p.tiles_per_img;
            float acc[128];
            int prev_w = -1, prev_x = -1;          // slots the group in flight reads; prev_x only behind a group's last tap
            for (int g = 0, hc = 0; g < groups; ++g) {
                mbar_wait(smem_u32(&full_x[xs]), xphase);
                // the warpgroup's 128 pixels of tap ky: whole rows, ky dil rows below the slot's first
                const uint32_t xo = x_base + (uint32_t)xs * x_slot + (uint32_t)(half_id * 128 * 2 * TCT_KC);
                const bool two = hc != halves - 1 || ks_last == 2;
                for (int ky = 0; ky < kh; ++ky) {
                    mbar_wait(smem_u32(&full_w[ws]), wphase);
                    const uint32_t sw = base + (uint32_t)ws * TCT_W_SLOT;
                    const uint64_t w_hi = make_smem_desc_sw64(sw), w_lo = make_smem_desc_sw64(sw + TCT_W_PLANE);
                    const uint32_t xk = xo + (uint32_t)ky * tap_step;
                    const uint64_t x_hi = make_smem_desc_sw64(xk), x_lo = make_smem_desc_sw64(xk + (uint32_t)p.x_plane);
                    const uint32_t accumulate = (g | ky) != 0;
                    wg_fence_acc(acc);
                    if (two) {                         // uniform over the CTA
                        wg_fence(); wg_mma3_128x128<2, 64>(acc, w_hi, w_lo, x_hi, x_lo, accumulate); wg_commit();
                    } else {
                        wg_fence(); wg_mma3_128x128<1, 64>(acc, w_hi, w_lo, x_hi, x_lo, accumulate); wg_commit();
                    }
                    wg_fence_acc(acc);
                    // keep this tap's group in flight; the previous one has finished reading its slots
                    wg_wait<1>();
                    wg_fence_acc(acc);
                    if (lane == 0) {
                        if (prev_w >= 0) mbar_arrive(smem_u32(&empty_w[prev_w]));
                        if (prev_x >= 0) mbar_arrive(smem_u32(&empty_x[prev_x]));
                    }
                    prev_w = ws;
                    prev_x = ky == kh - 1 ? xs : -1;
                    if (++ws == TCT_W_SLOTS) { ws = 0; wphase ^= 1u; }
                }
                if (++xs == p.x_slots) { xs = 0; xphase ^= 1u; }
                if (++hc == halves) hc = 0;
            }
            wg_wait<0>();
            wg_fence_acc(acc);
            if (lane == 0) {
                mbar_arrive(smem_u32(&empty_w[prev_w]));
                mbar_arrive(smem_u32(&empty_x[prev_x]));
            }
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
// Bytes of one plane of a halo slot: the tile's rows and the dil (k - 1) rows around them, W pixels of 32 channels each.
static int tct_x_plane(const TcSetup& s) { return (TCT_N / s.W + s.dil * (s.kh - 1)) * s.W * 2 * TCT_KC; }
// Halo slots that fit beside the weight ring and the epilogue staging.
static int tct_x_slots(const TcSetup& s) {
    const int room = TCT_SMEM_LIMIT - 1024 - TCT_W_SLOTS * TCT_W_SLOT - TCT_OUT_BYTES;
    return std::min(TCT_MAX_X_SLOTS, room / (2 * tct_x_plane(s)));
}

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
    // the halo ring needs two slots to overlap a fill with the MMAs; wider halos (5x5 on 256-wide maps) run on conv_tc
    return tct_x_slots(s) >= 2;
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
    k.x_plane = tct_x_plane(s); k.x_slots = tct_x_slots(s);
    L.smem_bytes = 1024 + TCT_W_SLOTS * TCT_W_SLOT + k.x_slots * 2 * k.x_plane + TCT_OUT_BYTES;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)s.Cin, (cuuint64_t)s.W, (cuuint64_t)s.H, (cuuint64_t)s.max_batch};
        cuuint64_t strides[3] = {(cuuint64_t)s.in_ld * 2, (cuuint64_t)s.W * s.in_ld * 2, (cuuint64_t)s.H * s.W * s.in_ld * 2};
        cuuint32_t box[4] = {TCT_KC, (cuuint32_t)s.W, (cuuint32_t)(k.bh + s.dil * (s.kh - 1)), 1};   // one halo slot plane
        cuuint32_t estr[4] = {1, 1, 1, 1};
        void* base = (void*)((__half*)s.in_base + (plane ? s.in_plane : 0) + s.in_coff);
        CUresult r = enc(plane ? &L.x_lo : &L.x_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(tct X) failed: %d", (int)r);
    }
    const int K_pad = k.taps * k.cchunks * 64;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)K_pad, (cuuint64_t)s.n_tile};        // rows beyond n_tile: OOB zero fill
        cuuint64_t strides[1] = {(cuuint64_t)K_pad * 2};
        cuuint32_t box[2] = {TCT_KC, (cuuint32_t)TCT_M};
        cuuint32_t estr[2] = {1, 1};
        void* base = (void*)(plane ? s.w_lo : s.w_hi);
        CUresult r = enc(plane ? &L.w_lo : &L.w_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B,
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
    static int attr_bytes[MAX_DEVICES] = {};
    if (smem_limit((const void*)conv_tct_kernel<ACT>, attr_bytes, L.smem_bytes)) return 1;
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
