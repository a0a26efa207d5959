// Pointwise (1x1, stride 1) convolution as one wgmma GEMM over the flat NHWC pixel index (sm_90a):
//
//   C[M = batch*H*W pixels][Cout] = A[M][Cin] * W[Cout][Cin]^T
//
// A 1x1 stride-1 conv needs none of conv_tc's geometry (taps, dilation, stride 2, ragged bw x bh edge tiles, multi-image
// tiles): a 128-pixel tile simply runs across image boundaries and only the last tile of the launch is partial.  Same fp16
// hi/lo three-product scheme and the same packed, K-padded weight matrix as conv_tc (plan.pack_tc_weights).
//
// * Work unit = 128 pixels x one chunk of NC output channels (NC in {32, 64, 96, 128}, picked per layer from Cout); the
//   units of one pixel tile are consecutive, so persistent CTAs run them side by side and the A re-reads hit L2.
// * A: 2-D TMA box of 64 channels x 128 pixels over {Cin, max_batch*H*W} (channels past Cin and rows past the buffer are
//   zero-filled); B: box of 64 x NC over the weight rows (rows past the packed matrix are zero-filled).  128-byte swizzle.
// * Warp 8 is the TMA producer; warpgroups 0 and 1 take alternate units of the CTA, so one warpgroup's epilogue overlaps
//   the other's MMAs and the producer's loads.  A warpgroup accumulates its 128 x NC unit in registers with m64nNCk16
//   wgmma issued from straight-line code, one k-block's group kept in flight while the next is issued.
// * Epilogue straight from the accumulator fragment: fmaf(acc, out_scale, bias), activation, then the split-fp16 hi/lo or
//   float32 value into a swizzled 16 KB staging buffer per 32-channel slab, which leaves as one TMA store per plane.  The
//   output tensor map spans {Cout, batch*H*W}, so stores clip at Cout and at the batch.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_pw.h"
#include "tc_ptx.h"

namespace skps {

constexpr int PW_THREADS = 288;          // warps 0-7 MMA + epilogue (two warpgroups), warp 8 TMA
constexpr int PW_BM = 128;               // pixels per unit
constexpr int PW_BK = 64;                // channels per k-block (one 128-byte swizzle atom of fp16)
constexpr int PW_A_TILE = PW_BM * 128;   // one plane of one k-block: 128 pixel rows x 128 B
constexpr int PW_OUT_BUF = 16384;        // one 32-channel slab of 128 pixels: hi + lo planes of 64-B rows, or 128-B float rows
constexpr int PW_MAX_STAGES = 4;
constexpr int PW_SMEM = 227 * 1024;      // dynamic shared memory per block on sm_90

__host__ __device__ constexpr int pw_stage_bytes(int nc) { return 2 * PW_A_TILE + 2 * nc * 128; }

// KS K-steps of 16 of the three-product scheme on a 128 x N accumulator held by one warpgroup: acc[0..N/2) = pixel rows
// 0-63, acc[N/2..N) = rows 64-127 (row 64 of the A tile at +8 KB).  Same order per element as conv_tc: lo*hi, hi*lo, hi*hi.
template <int N, int KS>
__device__ __forceinline__ void pw_mma(float* acc, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
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

template <int NC, int ACT, bool OUT_SPLIT>
__global__ void __launch_bounds__(PW_THREADS, 1)
conv_pw_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
               const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
               const __grid_constant__ CUtensorMap tmO_hi, const __grid_constant__ CUtensorMap tmO_lo, const PwK p) {
    constexpr uint32_t B_TILE = NC * 128;
    constexpr uint32_t STAGE = (uint32_t)pw_stage_bytes(NC);
    extern __shared__ uint8_t smem_raw[];
    // a stage is filled for one warpgroup at a time, so each warpgroup has its own full barriers: their phases then count
    // only that warpgroup's fills, in the order it consumes them
    __shared__ __align__(8) uint64_t full_bar[2][PW_MAX_STAGES], empty_bar[PW_MAX_STAGES];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t out_base = base + (uint32_t)p.stages * STAGE;       // 2 warpgroups x out_bufs x 16 KB
    const int units = p.m_tiles * p.n_chunks;

    if (warp == 8 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_lo) : "memory");
    }
    if (warp == 0 && lane == 0) {
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(smem_u32(&full_bar[0][s]), 1);
            mbar_init(smem_u32(&full_bar[1][s]), 1);
            mbar_init(smem_u32(&empty_bar[s]), 4);            // one arrival per warp of the consuming warpgroup
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        // ================================================================== TMA producer
        if (lane == 0) {
            int it = 0;                                        // stage fills so far
            int local = 0;                                     // units of this CTA so far: unit `local` is warpgroup local % 2's
            for (int u = blockIdx.x; u < units; u += gridDim.x, ++local) {
                const int mt = u / p.n_chunks, ch = u - mt * p.n_chunks;
                for (int kb = 0; kb < p.kblocks; ++kb, ++it) {
                    const int stage = it % p.stages;
                    mbar_wait(smem_u32(&empty_bar[stage]), (uint32_t)((it / p.stages) & 1) ^ 1u);
                    const uint32_t fb = smem_u32(&full_bar[local & 1][stage]);
                    mbar_expect_tx(fb, STAGE);
                    const uint32_t ss = base + (uint32_t)stage * STAGE;
                    tma_load_2d(ss, &tmA_hi, fb, kb * PW_BK, mt * PW_BM);
                    tma_load_2d(ss + PW_A_TILE, &tmA_lo, fb, kb * PW_BK, mt * PW_BM);
                    tma_load_2d(ss + 2 * PW_A_TILE, &tmB_hi, fb, kb * PW_BK, ch * NC);
                    tma_load_2d(ss + 2 * PW_A_TILE + B_TILE, &tmB_lo, fb, kb * PW_BK, ch * NC);
                }
            }
        }
    } else {
        // ================================================================== MMA + epilogue
        // Warpgroup wg accumulates its units' 128 pixels x NC channels: acc[(NC/2) m + 4 i + e] = pixel 64m + 16q + lane/4 +
        // 8(e/2), channel 8i + 2(lane%4) + e%2 of the chunk.
        const int q = warp & 3;
        const int wg = warp >> 2;
        const bool leader = q == 0 && lane == 0;       // issues and drains the warpgroup's TMA stores
        // 16-channel steps of the last k-block that hold real channels (TMA zero-fills the rest), as in conv_tc
        const int ks_last = min(4, (p.Cin - (p.kblocks - 1) * PW_BK + 15) / 16);
        uint32_t full_phase = 0;                       // bit s: parity of this warpgroup's next fill of stage s
        int store_i = 0;                               // TMA stores issued by this warpgroup so far
        int local = 0;
        for (int u = blockIdx.x; u < units; u += gridDim.x, ++local) {
            if ((local & 1) != wg) continue;
            const int mt = u / p.n_chunks, ch = u - mt * p.n_chunks;
            float acc[NC];
            int prev = 0;
            for (int kb = 0; kb < p.kblocks; ++kb) {
                const int stage = (local * p.kblocks + kb) % p.stages;
                mbar_wait(smem_u32(&full_bar[wg][stage]), (full_phase >> stage) & 1u);
                full_phase ^= 1u << stage;
                const uint32_t ss = base + (uint32_t)stage * STAGE;
                const uint64_t a_hi = make_smem_desc(ss), a_lo = make_smem_desc(ss + PW_A_TILE);
                const uint64_t b_hi = make_smem_desc(ss + 2 * PW_A_TILE), b_lo = make_smem_desc(ss + 2 * PW_A_TILE + B_TILE);
                const int ks = kb == p.kblocks - 1 ? ks_last : 4;
                const uint32_t accumulate = kb != 0;
                wg_fence_acc(acc);
                switch (ks) {                          // uniform over the CTA
                    case 4: wg_fence(); pw_mma<NC, 4>(acc, a_hi, a_lo, b_hi, b_lo, accumulate); wg_commit(); break;
                    case 3: wg_fence(); pw_mma<NC, 3>(acc, a_hi, a_lo, b_hi, b_lo, accumulate); wg_commit(); break;
                    case 2: wg_fence(); pw_mma<NC, 2>(acc, a_hi, a_lo, b_hi, b_lo, accumulate); wg_commit(); break;
                    default: wg_fence(); pw_mma<NC, 1>(acc, a_hi, a_lo, b_hi, b_lo, accumulate); wg_commit(); break;
                }
                wg_fence_acc(acc);
                // keep this k-block's group in flight; the previous one has finished reading its stage
                wg_wait<1>();
                wg_fence_acc(acc);
                if (kb > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
                prev = stage;
            }
            wg_wait<0>();
            wg_fence_acc(acc);
            if (lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
#pragma unroll
            for (int s = 0; s < NC / 32; ++s) {
                const int co = ch * NC + 32 * s;                // first channel of the slab
                if (co >= p.Cout) break;                        // uniform: slabs past Cout hold zero-weight columns
                // staging buffer of this slab: the store issued out_bufs slabs ago from it must have finished reading it
                const uint32_t sbuf = out_base + (uint32_t)(wg * p.out_bufs + store_i % p.out_bufs) * PW_OUT_BUF;
                if (leader) {
                    if (p.out_bufs == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                    else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                }
                ++store_i;
                asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
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
                        const int r = 64 * m + 16 * q + (lane >> 2) + 8 * h;      // pixel row of the unit
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const float* a = acc + (NC / 2) * m + 4 * (4 * s + i) + 2 * h;
                            const float v0 = act_t<ACT>(fmaf(a[0], p.out_scale, bias[2 * i]));
                            const float v1 = act_t<ACT>(fmaf(a[1], p.out_scale, bias[2 * i + 1]));
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
                asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
                if (leader) {
                    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                                 ::"l"(&tmO_hi), "r"(sbuf), "r"(co), "r"(mt * PW_BM) : "memory");
                    if (OUT_SPLIT)
                        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                                     ::"l"(&tmO_lo), "r"(sbuf + 8192u), "r"(co), "r"(mt * PW_BM) : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

// ------------------------------------------------------------------------------------------ host side
// 1x1 stride-1 layers without residual or heat-map partials whose activation the epilogue instantiates, with a unit-stride
// 16-byte aligned output of whole groups of 8 channels.  SiLU stays on conv_tc: its correctly rounded division spills beside
// the accumulators.
bool pw_applicable(const TcSetup& s) {
    const int stride = s.stride > 0 ? s.stride : 1;
    if (s.kh != 1 || s.kw != 1 || stride != 1 || s.pad != 0) return false;
    if (s.res || s.hm_val || !s.bias) return false;
    if (s.act != ACT_NONE && s.act != ACT_RELU && s.act != ACT_HSWISH) return false;
    if (s.Cin < 1 || (s.Cin % 8) || (s.in_ld % 8) || (s.in_coff % 8)) return false;
    if (s.out_fmt != DT_SPLIT16 && s.out_fmt != DT_F32) return false;
    const int oes = s.out_fmt == DT_SPLIT16 ? 2 : 4;
    if (s.out_cstride != 1 || (s.Cout % 8) || ((size_t)s.out_ld * oes) % 16 || ((size_t)s.out_coff * oes) % 16) return false;
    if (((uintptr_t)s.out % 16) || (s.out_fmt == DT_SPLIT16 && ((size_t)s.out_plane * 2) % 16)) return false;
    return true;
}

// chunk width: the fewest chunks (each re-reads the pixel tile), then the narrowest width that still covers Cout
static int pw_pick_nc(int Cout) {
    const int chunks = (Cout + 127) / 128;
    for (int nc = 32; nc < 128; nc += 32)
        if (chunks * nc >= Cout) return nc;
    return 128;
}

int pw_prepare(PwLayer& L, const TcSetup& s) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    SKPS_CHECK(pw_applicable(s), "conv_pw: layer not applicable");
    PwK& k = L.k;
    memset(&k, 0, sizeof(k));
    L.nc = pw_pick_nc(s.Cout);
    k.n_chunks = (s.Cout + L.nc - 1) / L.nc;
    k.kblocks = (s.Cin + PW_BK - 1) / PW_BK;
    k.Cin = s.Cin; k.Cout = s.Cout; k.out_scale = s.out_scale; k.bias = s.bias;
    // two staging buffers per warpgroup (the store of the previous slab overlaps the next one) while that leaves three
    // pipeline stages, else one
    const int budget = PW_SMEM - 2048;                     // alignment pad and static shared memory
    const int stage = pw_stage_bytes(L.nc);
    k.out_bufs = (budget - 4 * PW_OUT_BUF) / stage >= 3 ? 2 : 1;
    k.stages = (budget - 2 * k.out_bufs * PW_OUT_BUF) / stage;
    if (k.stages > PW_MAX_STAGES) k.stages = PW_MAX_STAGES;
    SKPS_CHECK(k.stages >= 2, "conv_pw: stages do not fit in shared memory");
    L.smem_bytes = k.stages * stage + 2 * k.out_bufs * PW_OUT_BUF + 1024;
    L.act = s.act; L.out_fmt = s.out_fmt;
    L.out = s.out; L.out_plane = s.out_plane; L.out_ld = s.out_ld; L.out_coff = s.out_coff;
    L.hw = (long long)s.H * s.W;
    // activations: {Cin, max_batch*H*W} fp16, rows of in_ld channels from channel in_coff
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)s.Cin, (cuuint64_t)(L.hw * s.max_batch)};
        cuuint64_t strides[1] = {(cuuint64_t)s.in_ld * 2};
        cuuint32_t box[2] = {PW_BK, PW_BM};
        cuuint32_t estr[2] = {1, 1};
        void* base = (void*)((__half*)s.in_base + (plane ? s.in_plane : 0) + s.in_coff);
        CUresult r = enc(plane ? &L.a_lo : &L.a_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(pw A) failed: %d", (int)r);
    }
    // weights: (K_pad, n_tiles*n_tile) as packed; rows past it (the last chunk's tail) are zero-filled
    const int K_pad = k.kblocks * PW_BK;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)K_pad, (cuuint64_t)s.n_tile * s.n_tiles};
        cuuint64_t strides[1] = {(cuuint64_t)K_pad * 2};
        cuuint32_t box[2] = {PW_BK, (cuuint32_t)L.nc};
        cuuint32_t estr[2] = {1, 1};
        void* base = (void*)(plane ? s.w_lo : s.w_hi);
        CUresult r = enc(plane ? &L.b_lo : &L.b_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(pw B) failed: %d", (int)r);
    }
    return 0;
}

template <int NC, int ACT, bool SPLIT>
static int pw_launch_t(const PwLayer& L, const PwK& k, const CUtensorMap& o_hi, const CUtensorMap& o_lo, int grid,
                       cudaStream_t stream) {
    static int attr_bytes[MAX_DEVICES] = {};
    if (smem_limit((const void*)conv_pw_kernel<NC, ACT, SPLIT>, attr_bytes, L.smem_bytes)) return 1;
    conv_pw_kernel<NC, ACT, SPLIT><<<grid, PW_THREADS, L.smem_bytes, stream>>>(L.a_hi, L.a_lo, L.b_hi, L.b_lo, o_hi, o_lo, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

template <int NC, bool SPLIT>
static int pw_launch_act(const PwLayer& L, const PwK& k, const CUtensorMap& o_hi, const CUtensorMap& o_lo, int grid,
                         cudaStream_t stream) {
    switch (L.act) {
        case ACT_NONE: return pw_launch_t<NC, ACT_NONE, SPLIT>(L, k, o_hi, o_lo, grid, stream);
        case ACT_RELU: return pw_launch_t<NC, ACT_RELU, SPLIT>(L, k, o_hi, o_lo, grid, stream);
        case ACT_HSWISH: return pw_launch_t<NC, ACT_HSWISH, SPLIT>(L, k, o_hi, o_lo, grid, stream);
        default: break;
    }
    set_error("conv_pw: activation %d not instantiated", L.act);
    return 1;
}

template <bool SPLIT>
static int pw_launch_nc(const PwLayer& L, const PwK& k, const CUtensorMap& o_hi, const CUtensorMap& o_lo, int grid,
                        cudaStream_t stream) {
    switch (L.nc) {
        case 32: return pw_launch_act<32, SPLIT>(L, k, o_hi, o_lo, grid, stream);
        case 64: return pw_launch_act<64, SPLIT>(L, k, o_hi, o_lo, grid, stream);
        case 96: return pw_launch_act<96, SPLIT>(L, k, o_hi, o_lo, grid, stream);
        case 128: return pw_launch_act<128, SPLIT>(L, k, o_hi, o_lo, grid, stream);
        default: break;
    }
    set_error("conv_pw: chunk width %d not instantiated", L.nc);
    return 1;
}

Grid pw_grid(const PwLayer& L, int batch, int num_sms, PwK* kp) {
    PwK k = L.k;
    k.m_tiles = (int)((L.hw * batch + PW_BM - 1) / PW_BM);
    if (kp) *kp = k;
    return persistent_grid((long long)k.m_tiles * k.n_chunks, num_sms);
}

int pw_launch(const PwLayer& L, int batch, int num_sms, cudaStream_t stream) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    const long long rows = L.hw * batch;
    PwK k;
    const int grid = pw_grid(L, batch, num_sms, &k).ctas;
    // output: {Cout, batch*H*W} per plane, one box = 32 channels x 128 pixels in the staging layout the epilogue writes
    const bool split = L.out_fmt == DT_SPLIT16;
    const int oes = split ? 2 : 4;
    CUtensorMap o[2];
    for (int plane = 0; plane < (split ? 2 : 1); ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)k.Cout, (cuuint64_t)rows};
        cuuint64_t strides[1] = {(cuuint64_t)L.out_ld * oes};
        cuuint32_t box[2] = {32, PW_BM};
        cuuint32_t estr[2] = {1, 1};
        char* base = (char*)L.out + (size_t)L.out_coff * oes + (plane ? (size_t)L.out_plane * 2 : 0);
        CUresult r = enc(&o[plane], split ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims,
                         strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         split ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(pw out) failed: %d", (int)r);
    }
    if (!split) o[1] = o[0];
    return split ? pw_launch_nc<true>(L, k, o[0], o[1], grid, stream) : pw_launch_nc<false>(L, k, o[0], o[1], grid, stream);
}

// float32 -> hi/lo float16 planes (the debug entry's input)
__global__ void pw_f32_to_split(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = src[i];
    const __half h = __float2half_rn(v);
    hi[i] = h;
    lo[i] = __float2half_rn(v - __half2float(h));
}

}  // namespace skps

using namespace skps;

// Debug/unit-test entry: one 1x1 conv through conv_pw on host buffers of max_batch images, run for the first `batch`.
//   x   [host] float32 (max_batch, H, W, in_ld); the conv reads channels [in_coff, in_coff + Cin)
//   w_hi/w_lo [host] float16 (n_tiles*n_tile, K_pad) as packed by plan.pack_tc_weights
//   out [host] float32 (max_batch, H, W, out_ld), in and out: channels [out_coff, out_coff + Cout) of the first batch*H*W
//       pixels are overwritten, everything else must come back as it went in
extern "C" SKPS_API int skps_debug_conv_pw(const float* x, int batch, int max_batch, int H, int W, int Cin, int in_ld,
                                           int in_coff, const void* w_hi, const void* w_lo, const float* bias, int Cout,
                                           int act, int n_tile, int n_tiles, float out_scale, int out_split, int out_ld,
                                           int out_coff, float* out) {
    SKPS_CHECK(x && w_hi && w_lo && bias && out, "debug_conv_pw: null argument");
    SKPS_CHECK(batch >= 1 && max_batch >= batch && in_coff + Cin <= in_ld && out_coff + Cout <= out_ld,
               "debug_conv_pw: bad shape");
    const long long nin = (long long)max_batch * H * W * in_ld, nout = (long long)max_batch * H * W * out_ld;
    const size_t wbytes = (size_t)n_tiles * n_tile * ((Cin + PW_BK - 1) / PW_BK) * PW_BK * 2;
    float *d_x = nullptr, *d_bias = nullptr, *d_out = nullptr;
    __half *d_in = nullptr, *d_wh = nullptr, *d_wl = nullptr, *d_osplit = nullptr;
    SKPS_CUDA(cudaMalloc(&d_x, nin * 4));
    SKPS_CUDA(cudaMalloc(&d_in, nin * 4));
    SKPS_CUDA(cudaMalloc(&d_wh, wbytes));
    SKPS_CUDA(cudaMalloc(&d_wl, wbytes));
    SKPS_CUDA(cudaMalloc(&d_bias, Cout * 4));
    SKPS_CUDA(cudaMalloc(&d_out, nout * 4));
    SKPS_CUDA(cudaMemcpy(d_x, x, nin * 4, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(d_wh, w_hi, wbytes, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(d_wl, w_lo, wbytes, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(d_bias, bias, Cout * 4, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(d_out, out, nout * 4, cudaMemcpyHostToDevice));
    pw_f32_to_split<<<(unsigned)((nin + 255) / 256), 256>>>(d_x, d_in, d_in + nin, nin);
    SKPS_CUDA(cudaGetLastError());
    if (out_split) {
        SKPS_CUDA(cudaMalloc(&d_osplit, nout * 4));
        pw_f32_to_split<<<(unsigned)((nout + 255) / 256), 256>>>(d_out, d_osplit, d_osplit + nout, nout);
        SKPS_CUDA(cudaGetLastError());
    }
    TcSetup s = {};
    s.H = H; s.W = W; s.Cin = Cin; s.in_ld = in_ld; s.in_coff = in_coff; s.max_batch = max_batch;
    s.in_base = d_in; s.in_plane = nin;
    s.kh = s.kw = 1; s.dil = 1; s.pad = 0; s.stride = 1;
    s.Cout = Cout; s.act = act; s.n_tile = n_tile; s.n_tiles = n_tiles; s.out_scale = out_scale;
    s.w_hi = d_wh; s.w_lo = d_wl; s.bias = d_bias;
    s.out = out_split ? (void*)d_osplit : (void*)d_out; s.out_fmt = out_split ? DT_SPLIT16 : DT_F32;
    s.out_plane = nout; s.out_ld = out_ld; s.out_coff = out_coff; s.out_cstride = 1;
    PwLayer L;
    if (pw_prepare(L, s)) return 1;
    if (pw_launch(L, batch, sm_count(), 0)) return 1;
    SKPS_CUDA(cudaDeviceSynchronize());
    if (out_split) {
        __half* tmp = (__half*)malloc(nout * 4);
        SKPS_CHECK(tmp, "debug_conv_pw: host allocation failed");
        SKPS_CUDA(cudaMemcpy(tmp, d_osplit, nout * 4, cudaMemcpyDeviceToHost));
        for (long long i = 0; i < nout; ++i) out[i] = __half2float(tmp[i]) + __half2float(tmp[nout + i]);
        free(tmp);
    } else {
        SKPS_CUDA(cudaMemcpy(out, d_out, nout * 4, cudaMemcpyDeviceToHost));
    }
    cudaFree(d_x); cudaFree(d_in); cudaFree(d_wh); cudaFree(d_wl); cudaFree(d_bias); cudaFree(d_out);
    if (d_osplit) cudaFree(d_osplit);
    return 0;
}
