// 3x3 convolution for small channel counts (24 / 40: HRNet-w18's 18- and 36-channel branches after
// channel padding) on the warp-level tensor-core path (mma.sync m16n8k16 / m16n8k8, fp16 hi/lo operands,
// fp32 accumulate: the same three-product scheme as conv_tc.cu).
//
// Why not the wgmma kernel (conv_tc.cu): it fetches one TMA box per filter tap, i.e. every input pixel row is
// pulled from L2 nine times, and with 48-byte pixel rows each fetch costs a full sector group, so L2->SM traffic is
// several times the real input and the tensor cores mostly wait.  Here the (8+2) x (16+2) halo tile of the input is fetched
// ONCE per output tile (one TMA box per float16 plane, conv padding = TMA out-of-bounds zero fill), all
// nine taps read it from shared memory through ldmatrix with per-row addresses (implicit im2col), and
// the whole weight set (9 x Cout x Cin, hi and lo) stays resident in shared memory of a persistent CTA.
//
// Replaces the Conv(+Relu | +Add,+Relu) node groups of timm's BasicBlock in the Teacher export
// (model.py:302-345 TeacherNet -> hrnet_w18 branches).
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_mma.h"

namespace skps {

constexpr int MT_H = 8, MT_W = 16;                                   // output tile (pixels)
constexpr int HALO_H = MT_H + 2, HALO_W = MT_W + 2, HALO_PX = HALO_H * HALO_W;
constexpr int MMA_THREADS = 128;                                     // 4 warps; warp w owns output rows 2w, 2w+1

__device__ __forceinline__ uint32_t msmem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t* r) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t* r) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}
// D(16x8, fp32) += A(16x16, fp16, row) * B(16x8, fp16, col)
__device__ __forceinline__ void mma_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// D(16x8) += A(16x8) * B(8x8)
__device__ __forceinline__ void mma_1688(float* c, const uint32_t* a, uint32_t b0) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(b0));
}

template <int CIN, int COUT>
struct MmaCfg {
    static constexpr int PITCH = CIN * 2;                             // bytes per pixel row and per weight row
    static constexpr int PLANE = HALO_PX * PITCH;                     // halo bytes per float16 plane
    static constexpr int PLANE_AL = (PLANE + 127) & ~127;
    static constexpr int BUF = 2 * PLANE_AL;                          // hi + lo
    static constexpr int WPLANE = COUT * PITCH;                       // weights per (tap, plane): [Cout][Cin]
    static constexpr int WBYTES = 9 * 2 * WPLANE;
    static constexpr int SMEM = 2 * BUF + WBYTES + 128;
};

template <int CIN, int COUT>
__global__ void __launch_bounds__(MMA_THREADS)
conv_mma_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo, const ConvMmaK p) {
    using Cfg = MmaCfg<CIN, COUT>;
    constexpr int PITCH = Cfg::PITCH, PLANE = Cfg::PLANE, PLANE_AL = Cfg::PLANE_AL, BUF = Cfg::BUF, WPLANE = Cfg::WPLANE;
    constexpr int NT = COUT / 8, KS16 = CIN / 16;
    constexpr bool K8 = (CIN % 16) == 8;
    static_assert(CIN % 8 == 0 && COUT % 8 == 0, "channel counts must be multiples of 8");
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar[2];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t sbase = (msmem_u32(smem) + 127u) & ~127u;
    const uint32_t wsm = sbase + 2u * BUF;
    // the whole weight set, once per (persistent) CTA
    {
        uint8_t* wdst = smem + (sbase - msmem_u32(smem)) + 2 * BUF;
        for (int i = tid; i < Cfg::WBYTES / 16; i += MMA_THREADS)
            reinterpret_cast<uint4*>(wdst)[i] = __ldg(reinterpret_cast<const uint4*>(p.w) + i);
    }
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(msmem_u32(&bar[0])));
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(msmem_u32(&bar[1])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int total = p.tiles_img * p.batch;
    auto issue = [&](int t, int b) {
        const int n = t / p.tiles_img + p.img0, sp = t % p.tiles_img;
        const int ty = sp / p.tiles_x, tx = sp - ty * p.tiles_x;
        const uint32_t bar_a = msmem_u32(&bar[b]), dst = sbase + (uint32_t)b * BUF;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"((uint32_t)(2 * PLANE)) : "memory");
        const int cx = tx * MT_W - 1, cy = ty * MT_H - 1;
        asm volatile(
            "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
            ::"r"(dst), "l"(&tm_hi), "r"(bar_a), "r"(0), "r"(cx), "r"(cy), "r"(n) : "memory");
        asm volatile(
            "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
            ::"r"(dst + (uint32_t)PLANE_AL), "l"(&tm_lo), "r"(bar_a), "r"(0), "r"(cx), "r"(cy), "r"(n) : "memory");
    };
    // ldmatrix row addresses: lane l supplies row (l % 8) of matrix (l / 8)
    //   A x4: m0 = pixels 0-7 / k 0-7, m1 = pixels 8-15 / k 0-7, m2 = pixels 0-7 / k 8-15, m3 = pixels 8-15 / k 8-15
    //   B x4: m0 = hi k 0-7, m1 = hi k 8-15, m2 = lo k 0-7, m3 = lo k 8-15 (rows = output channels)
    const uint32_t a_px_off = (uint32_t)((lane & 7) + 8 * ((lane >> 3) & 1)) * PITCH;
    const uint32_t a_lane_off = a_px_off + (uint32_t)(lane >> 4) * 16u;
    const uint32_t b_lane_off = (uint32_t)(lane & 7) * PITCH + (uint32_t)((lane >> 3) & 1) * 16u + (uint32_t)(lane >> 4) * WPLANE;
    const uint32_t b8_lane_off = (uint32_t)(lane & 7) * PITCH + (uint32_t)((lane >> 3) & 1) * WPLANE;   // x2: m0 = hi, m1 = lo
    const int g = lane >> 2, tq = lane & 3;

    int t = blockIdx.x;
    if (tid == 0 && t < total) issue(t, 0);
    for (int k = 0; t < total; ++k, t += gridDim.x) {
        const int b = k & 1;
        if (tid == 0 && t + (int)gridDim.x < total) issue(t + gridDim.x, b ^ 1);
        {
            const uint32_t bar_a = msmem_u32(&bar[b]), parity = (uint32_t)(k >> 1) & 1u;
            asm volatile(
                "{\n\t"
                ".reg .pred p;\n\t"
                "MMA_WAIT:\n\t"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                "@p bra MMA_DONE;\n\t"
                "bra MMA_WAIT;\n\t"
                "MMA_DONE:\n\t"
                "}\n" ::"r"(bar_a), "r"(parity) : "memory");
        }
        const uint32_t tile = sbase + (uint32_t)b * BUF;
        float acc[2][NT][4];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < NT; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[h][j][e] = 0.f;
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int ky = tap / 3, kx = tap - 3 * ky;
            const uint32_t wtap = wsm + (uint32_t)tap * 2u * WPLANE;
            uint32_t arow[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) arow[h] = tile + (uint32_t)((2 * warp + h + ky) * HALO_W + kx) * PITCH;
#pragma unroll
            for (int ks = 0; ks < KS16; ++ks) {
                uint32_t ah[2][4], al[2][4];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    ldsm_x4(arow[h] + a_lane_off + ks * 32, ah[h]);
                    ldsm_x4(arow[h] + PLANE_AL + a_lane_off + ks * 32, al[h]);
                }
                // per accumulator the three products are added in the order lo*hi, hi*lo, hi*hi (small terms first); the passes
                // are issued across all 2*NT accumulators so that consecutive MMAs are independent
                uint32_t bw[NT][4];
#pragma unroll
                for (int j = 0; j < NT; ++j) ldsm_x4(wtap + (uint32_t)(j * 8) * PITCH + ks * 32 + b_lane_off, bw[j]);
#pragma unroll
                for (int j = 0; j < NT; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h) mma_16816(acc[h][j], al[h], bw[j][0], bw[j][1]);
#pragma unroll
                for (int j = 0; j < NT; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h) mma_16816(acc[h][j], ah[h], bw[j][2], bw[j][3]);
#pragma unroll
                for (int j = 0; j < NT; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h) mma_16816(acc[h][j], ah[h], bw[j][0], bw[j][1]);
            }
            if (K8) {
                uint32_t ah[2][2], al[2][2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    ldsm_x2(arow[h] + a_px_off + KS16 * 32, ah[h]);
                    ldsm_x2(arow[h] + PLANE_AL + a_px_off + KS16 * 32, al[h]);
                }
                uint32_t bw[NT][2];
#pragma unroll
                for (int j = 0; j < NT; ++j) ldsm_x2(wtap + (uint32_t)(j * 8) * PITCH + KS16 * 32 + b8_lane_off, bw[j]);
#pragma unroll
                for (int j = 0; j < NT; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h) mma_1688(acc[h][j], al[h], bw[j][0]);
#pragma unroll
                for (int j = 0; j < NT; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h) mma_1688(acc[h][j], ah[h], bw[j][1]);
#pragma unroll
                for (int j = 0; j < NT; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h) mma_1688(acc[h][j], ah[h], bw[j][0]);
            }
        }
        // ---- epilogue: the accumulator fragments (2 channels of 2 pixels per register pair) go through shared memory so that
        // one thread finishes one pixel x all COUT channels with 16-byte residual loads and stores
        __syncthreads();                                   // all warps are done with this buffer's halo tile: reuse it as staging
        {
            float* stage = reinterpret_cast<float*>(smem + (sbase - msmem_u32(smem)) + (size_t)b * BUF);     // [128 px][COUT + 4]
            constexpr int SP = COUT + 4;                   // row pitch in floats (bank spread for the fragment writes)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int half = 0; half < 2; ++half)
#pragma unroll
                    for (int j = 0; j < NT; ++j)
                        *reinterpret_cast<float2*>(stage + ((2 * warp + h) * MT_W + g + 8 * half) * SP + 8 * j + 2 * tq) =
                            make_float2(acc[h][j][2 * half], acc[h][j][2 * half + 1]);
            __syncthreads();
            const int n = t / p.tiles_img + p.img0, sp = t % p.tiles_img;
            const int ty = sp / p.tiles_x, tx = sp - ty * p.tiles_x;
            const int y = ty * MT_H + tid / MT_W, x = tx * MT_W + tid % MT_W;          // thread -> pixel of the tile
            if (y < p.H && x < p.W) {
                const long long pix = ((long long)n * p.H + y) * p.W + x;
                const float* srow = stage + tid * SP;
#pragma unroll
                for (int c8 = 0; c8 < COUT; c8 += 8) {
                    float8 v, r;
                    const float4 s0 = *reinterpret_cast<const float4*>(srow + c8), s1 = *reinterpret_cast<const float4*>(srow + c8 + 4);
                    const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + c8));
                    const float4 b1 = __ldg(reinterpret_cast<const float4*>(p.bias + c8 + 4));
                    v.v[0] = fmaf(s0.x, p.out_scale, b0.x); v.v[1] = fmaf(s0.y, p.out_scale, b0.y);
                    v.v[2] = fmaf(s0.z, p.out_scale, b0.z); v.v[3] = fmaf(s0.w, p.out_scale, b0.w);
                    v.v[4] = fmaf(s1.x, p.out_scale, b1.x); v.v[5] = fmaf(s1.y, p.out_scale, b1.y);
                    v.v[6] = fmaf(s1.z, p.out_scale, b1.z); v.v[7] = fmaf(s1.w, p.out_scale, b1.w);
                    if (p.res) r = ld8(p.res, p.res_fmt, p.res_plane, pix * p.res_ld + p.res_coff + c8);
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                        const float rr = p.res ? r.v[e] : 0.f;
                        v.v[e] = p.res_first ? apply_act(v.v[e] + rr, p.act) : apply_act(v.v[e], p.act) + rr;
                    }
                    st8(p.out, p.out_fmt, p.out_plane, pix * p.out_ld + p.out_coff + c8, v);
                }
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // staging writes (generic proxy) before the next TMA refill
        __syncthreads();          // every warp is done with buffer b before the next iteration refills it
    }
}

// ------------------------------------------------------------------------------------------ host side
// Shared-memory limit of the instantiation and its resident CTAs per SM, on the current device
template <int CIN, int COUT>
static int mma_setup_t(int* ctas_per_sm) {
    static int attr_bytes[MAX_DEVICES] = {};
    static int ctas[MAX_DEVICES] = {};
    constexpr int smem = MmaCfg<CIN, COUT>::SMEM;
    if (smem_limit((const void*)conv_mma_kernel<CIN, COUT>, attr_bytes, smem)) return 1;
    int dev = 0;
    SKPS_CUDA(cudaGetDevice(&dev));
    if (!ctas[dev]) {
        int n = 0;
        SKPS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, conv_mma_kernel<CIN, COUT>, MMA_THREADS, smem));
        ctas[dev] = n < 1 ? 1 : n;
    }
    *ctas_per_sm = ctas[dev];
    return 0;
}

bool conv_mma_supported(int cin, int cout, int kh, int kw, int stride, int dil, int pad) {
    return kh == 3 && kw == 3 && stride == 1 && dil == 1 && pad == 1 && cin == cout && (cin == 24 || cin == 40);
}

int conv_mma_prepare(ConvMmaLayer& L, const TView& in, const TView& out, const TView& res, int res_first, const void* w_packed,
                     const float* bias, float out_scale, int act, int max_batch) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    SKPS_CHECK(conv_mma_supported(in.C, out.C, 3, 3, 1, 1, 1), "conv_mma: unsupported channels %d -> %d", in.C, out.C);
    SKPS_CHECK(in.fmt == DT_SPLIT16 && in.c_stride == 1 && ((in.ld | in.c_off) & 7) == 0, "conv_mma: input view");
    SKPS_CHECK(out.c_stride == 1 && ((out.ld | out.c_off) & 7) == 0 && in.H == out.H && in.W == out.W &&
               (out.fmt == DT_SPLIT16 || out.fmt == DT_F32) && bias, "conv_mma: output view / bias");
    SKPS_CHECK(!res.base || (res.c_stride == 1 && ((res.ld | res.c_off) & 7) == 0 && res.C == out.C), "conv_mma: residual view");
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)in.C, (cuuint64_t)in.W, (cuuint64_t)in.H, (cuuint64_t)max_batch};
        cuuint64_t strides[3] = {(cuuint64_t)in.ld * 2, (cuuint64_t)in.W * in.ld * 2, (cuuint64_t)in.H * in.W * in.ld * 2};
        cuuint32_t box[4] = {(cuuint32_t)in.C, (cuuint32_t)HALO_W, (cuuint32_t)HALO_H, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        void* base = (void*)((__half*)in.base + (plane ? in.plane : 0) + in.c_off);
        CUresult r = enc(plane ? &L.a_lo : &L.a_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(conv_mma) failed: %d", (int)r);
    }
    ConvMmaK& k = L.k;
    k.H = in.H; k.W = in.W;
    k.tiles_x = (in.W + MT_W - 1) / MT_W;
    k.tiles_img = k.tiles_x * ((in.H + MT_H - 1) / MT_H);
    k.batch = 0; k.img0 = 0;
    k.w = w_packed; k.bias = bias; k.out_scale = out_scale; k.act = act;
    k.out = out.base; k.out_fmt = out.fmt; k.out_plane = out.plane; k.out_ld = out.ld; k.out_coff = out.c_off;
    k.res = res.base; k.res_fmt = res.fmt; k.res_plane = res.plane; k.res_ld = res.ld; k.res_coff = res.c_off;
    k.res_first = res.base ? res_first : 0;
    L.cin = in.C; L.cout = out.C;
    if ((in.C == 24 ? mma_setup_t<24, 24>(&L.ctas_per_sm) : mma_setup_t<40, 40>(&L.ctas_per_sm))) return 1;
    return 0;
}

template <int CIN, int COUT>
static int mma_launch_t(const ConvMmaLayer& L, const ConvMmaK& k, int grid, cudaStream_t stream) {
    conv_mma_kernel<CIN, COUT><<<grid, MMA_THREADS, MmaCfg<CIN, COUT>::SMEM, stream>>>(L.a_hi, L.a_lo, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

Grid conv_mma_grid(const ConvMmaLayer& L, int batch, int num_sms) {
    return persistent_grid((long long)L.k.tiles_img * batch, (long long)num_sms * L.ctas_per_sm);
}

int conv_mma_launch(const ConvMmaLayer& L, int batch, int num_sms, cudaStream_t stream) {
    ConvMmaK k = L.k;
    k.batch = batch;
    const int grid = conv_mma_grid(L, batch, num_sms).ctas;
    if (L.cin == 24) return mma_launch_t<24, 24>(L, k, grid, stream);
    if (L.cin == 40) return mma_launch_t<40, 40>(L, k, grid, stream);
    set_error("conv_mma: %d channels not instantiated", L.cin);
    return 1;
}

static __global__ void mma_f32_to_split(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo,
                                        long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = src[i];
    const __half h = __float2half_rn(v);
    hi[i] = h;
    lo[i] = __float2half_rn(v - __half2float(h));
}

}  // namespace skps

using namespace skps;

// Unit-test entry: one 3x3 'same' conv (Cin == Cout in {24, 40}) through conv_mma_kernel on host data.
extern "C" SKPS_API int skps_debug_conv_mma(const float* x, int N, int H, int W, int C, const void* w_packed,
                                            const float* bias, int act, float out_scale, const float* residual,
                                            int res_first, int out_split, float* out) {
    SKPS_CHECK(x && w_packed && out, "debug_conv_mma: null argument");
    const long long n = (long long)N * H * W * C;
    const size_t wbytes = (size_t)9 * 2 * C * C * 2;
    float *d_x = nullptr, *d_bias = nullptr, *d_res = nullptr;
    __half *d_in = nullptr, *d_out = nullptr;
    void* d_w = nullptr;
    SKPS_CUDA(cudaMalloc(&d_x, n * 4));
    SKPS_CUDA(cudaMalloc(&d_in, n * 4));
    SKPS_CUDA(cudaMalloc(&d_out, n * 4));
    SKPS_CUDA(cudaMalloc(&d_w, wbytes));
    SKPS_CUDA(cudaMemcpy(d_x, x, n * 4, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(d_w, w_packed, wbytes, cudaMemcpyHostToDevice));
    if (bias) {
        SKPS_CUDA(cudaMalloc(&d_bias, C * 4));
        SKPS_CUDA(cudaMemcpy(d_bias, bias, C * 4, cudaMemcpyHostToDevice));
    }
    if (residual) {
        SKPS_CUDA(cudaMalloc(&d_res, n * 4));
        SKPS_CUDA(cudaMemcpy(d_res, residual, n * 4, cudaMemcpyHostToDevice));
    }
    mma_f32_to_split<<<(unsigned)((n + 255) / 256), 256>>>(d_x, d_in, d_in + n, n);
    SKPS_CUDA(cudaGetLastError());
    TView in = {}, o = {}, r = {};
    in.base = d_in; in.ld = C; in.c_off = 0; in.c_stride = 1; in.C = C; in.H = H; in.W = W; in.sample = (long long)H * W * C;
    in.fmt = DT_SPLIT16; in.plane = n;
    o = in; o.base = d_out; o.fmt = out_split ? DT_SPLIT16 : DT_F32; o.plane = n;
    if (d_res) { r = in; r.base = d_res; r.fmt = DT_F32; r.plane = 0; }
    ConvMmaLayer L;
    if (conv_mma_prepare(L, in, o, r, res_first, d_w, d_bias, out_scale, act, N)) return 1;
    if (conv_mma_launch(L, N, sm_count(), 0)) return 1;
    SKPS_CUDA(cudaDeviceSynchronize());
    if (out_split) {
        __half* tmp = (__half*)malloc(n * 4);
        SKPS_CUDA(cudaMemcpy(tmp, d_out, n * 4, cudaMemcpyDeviceToHost));
        for (long long i = 0; i < n; ++i) out[i] = __half2float(tmp[i]) + __half2float(tmp[n + i]);
        free(tmp);
    } else {
        SKPS_CUDA(cudaMemcpy(out, d_out, n * 4, cudaMemcpyDeviceToHost));
    }
    cudaFree(d_x); cudaFree(d_in); cudaFree(d_out); cudaFree(d_w);
    if (d_bias) cudaFree(d_bias);
    if (d_res) cudaFree(d_res);
    return 0;
}
