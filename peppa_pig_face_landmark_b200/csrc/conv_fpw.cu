// The student's fused "A-producer -> pointwise convolution" layers on wgmma with the accumulators in registers (sm_90a).
//
// Same layers and the same A producer as conv_xf.cu (xf_producer.h): the A operand of
//     C[128 pixels][N] = A[128 pixels][K] * W[N][K]
// is built in shared memory by transform warps, in the 128-byte-swizzled K-major fp16 hi/lo layout wgmma reads.
//
// What differs from conv_xf is the MMA side.  conv_xf's MMA warpgroup keeps a 128 x 256 accumulator whatever the layer's
// width and issues m64n32 chunks from loops bounded at run time, so ptxas serialises every wgmma and spills the accumulator.
// Here the unit width N is a template parameter of at most 64 output channels: the MMA warpgroup holds exactly N fp32
// accumulators per thread for its 128 x N unit and issues m64nNk16 wgmma from straight-line code, one K-chunk's group kept
// in flight while the next is issued (as conv_pw.cu).  ptxas sizes wgmma accumulators against the launch's 128 registers per
// thread (512 threads, one CTA per SM), setmaxnreg notwithstanding, so a wider layer runs as nsplit units of 64 channels per pixel tile (N tile 80 or 112 or 128 -> 2 units, 160 -> 3, 256 -> 4).
// The depthwise / up-sample stencil of the A producer is the expensive part, so the XF_DW layers without a residual and
// with an even nsplit (the decoder's up-sample layers: 256 -> 4 units, 128 -> 2) run on conv_fpw_pair: the transform
// warps build each A tile once for two units and two MMA warpgroups multiply it, one unit each.  On conv_fpw_kernel every
// unit re-stages the tile and recomputes the A producer; the units of one tile are consecutive, so persistent CTAs run
// them side by side and the re-reads hit L2.
//
// conv_fpw_kernel's warp roles (512 threads, one persistent CTA per SM):
//   0      TMA producer: per K-chunk the weight tile, then the raw tile(s) (XF_DW) or the A tile (XF_SCALE)
//   1-3    idle after set-up; warps 0-3 drop to 32 registers each (setmaxnreg)
//   4-7    MMA + epilogue warpgroup, raised to 160 registers
//   8-15   transform warps: raw tile -> A tile (xf_transform), raised to 160 registers
// The epilogue works straight from the accumulator fragment: fmaf(acc, out_scale, bias), residual, activation, then the
// split-fp16 hi/lo or float32 value into a swizzled 16 KB staging buffer per 32-channel slab, which leaves as one TMA store
// per plane: a 32-channel x 16 x 8 pixel box in the output buffer's channel window.  Images past the batch are never
// touched.  While the MMA warpgroup runs an epilogue, the producer and the transform warps fill the rings for its next unit.
// Precision: the fp16 hi/lo operands, K order, three-product order and epilogue expressions of conv_xf, so the outputs are
// bit-identical to it.
#include <cuda.h>
#include <cuda_fp16.h>
#include <string.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_fpw.h"
#include "tc_ptx.h"

namespace skps {

// setmaxnreg: warps 0-3 give 4 x 32 x (128 - 32) registers; the transform warps take 8 x 32 x (160 - 128) and the MMA
// warpgroup 4 x 32 x (160 - 128) of them
constexpr int FPW_PRODUCER_REGS = 32, FPW_TRANSFORM_REGS = 160, FPW_MMA_REGS = 160;
static_assert(128 * FPW_PRODUCER_REGS + 256 * FPW_TRANSFORM_REGS + 128 * FPW_MMA_REGS <= 65536, "register file split");

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

// One MMA + epilogue warpgroup (wg 0 or 1 of the CTA's PER): work items u = blockIdx.x, + gridDim.x, ... below p.units, each
// the 64-channel unit PER * (u % items per tile) + wg of its pixel tile.  Every A and B slot it reads, the PER warpgroups
// read together: B slot = [hi: PER x N rows][lo: PER x N rows], this warpgroup's rows at wg x N.  Staging buffers
// wg x out_bufs .. + out_bufs - 1 and named barrier 1 + wg are its own, so one warpgroup's epilogue overlaps the other's
// MMAs.  RES: the epilogue can add a residual (conv_fpw_pair's layers have none, and its registers are short).
template <int N, int ACT, bool OUT_SPLIT, int PER, bool RES>
__device__ __forceinline__ void fpw_consumer(const FpwK& p, XfBarriers& bar, const XfSmem& sm, const CUtensorMap* tmO_hi,
                                             const CUtensorMap* tmO_lo, int wg) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t b_plane = (uint32_t)(PER * N) * 128u, b_slot = 2u * b_plane, b_row = (uint32_t)(wg * N) * 128u;
    const uint32_t o_base = sm.o_off + (uint32_t)(wg * p.out_bufs) * XF_OUT_BUF, named_bar = 1 + wg;
    const int items = p.nsplit / PER;                  // work items per pixel tile
    // acc[(N/2) m + 4 i + e] = pixel row 64m + 16q + lane/4 + 8(e/2) of the tile (row = 16 y + x), channel
    // 8i + 2(lane%4) + e%2 of the unit
    const int q = warp & 3;
    const bool leader = q == 0 && lane == 0;           // issues and drains the warpgroup's TMA stores
    int ast = 0, bst = 0;
    uint32_t aph = 0, bph = 0;
    int store_i = 0;                                   // TMA stores issued so far
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        const int tile = u / items, nh = (u - tile * items) * PER + wg;
        float acc[N];
        int prev_a = 0, prev_b = 0;
        for (int kc = 0; kc < p.a.cchunks; ++kc) {
            mbar_wait_g(smem_u32(&bar.a_full[ast]), aph);
            mbar_wait_g(smem_u32(&bar.b_full[bst]), bph);
            const uint32_t sa = sm.a_off + (uint32_t)ast * XF_A_BYTES, sb = sm.b_off + (uint32_t)bst * b_slot + b_row;
            const uint64_t a_hi = make_smem_desc(sa), a_lo = make_smem_desc(sa + XF_A_PLANE);
            const uint64_t b_hi = make_smem_desc(sb), b_lo = make_smem_desc(sb + b_plane);
            const uint32_t accumulate = kc != 0;
            wg_fence_acc(acc);
            switch (p.a.chunk_ksteps[kc]) {          // uniform over the CTA
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
                mbar_arrive(smem_u32(&bar.a_empty[prev_a]));
                mbar_arrive(smem_u32(&bar.b_empty[prev_b]));
            }
            prev_a = ast; prev_b = bst;
            if (++ast == p.a.as) { ast = 0; aph ^= 1u; }
            if (++bst == p.bs) { bst = 0; bph ^= 1u; }
        }
        wg_wait<0>();
        wg_fence_acc(acc);
        if (lane == 0) {
            mbar_arrive(smem_u32(&bar.a_empty[prev_a]));
            mbar_arrive(smem_u32(&bar.b_empty[prev_b]));
        }
        const int img = tile / p.a.tiles_per_img, t = tile - img * p.a.tiles_per_img;
        const int ty0 = (t / p.a.tiles_x) * XF_TH, tx0 = (t % p.a.tiles_x) * XF_TW;
        const long long pix0 = ((long long)img * p.a.H + ty0) * p.a.W + tx0;      // pixel index of the tile's row 0
#pragma unroll
        for (int s = 0; s < (N + 31) / 32; ++s) {
            const int co = nh * N + 32 * s;                 // first output channel of the slab
            if (co >= p.Cout) break;                        // uniform: slabs past Cout hold zero-weight columns
            // staging buffer of this slab: the store issued out_bufs slabs ago from it must have finished reading it
            const uint32_t sbuf = o_base + (uint32_t)(store_i % p.out_bufs) * XF_OUT_BUF;
            if (leader) {
                if (p.out_bufs == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            }
            ++store_i;
            asm volatile("bar.sync %0, 128;" ::"r"(named_bar) : "memory");
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
                        if (RES && p.res && co + 8 * i < p.Cout) {
                            const long long pix = pix0 + (r / XF_TW) * p.a.W + r % XF_TW;
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
            asm volatile("bar.sync %0, 128;" ::"r"(named_bar) : "memory");
            if (leader) {
                asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                             ::"l"(tmO_hi), "r"(sbuf), "r"(co), "r"(tx0), "r"(ty0), "r"(img) : "memory");
                if (OUT_SPLIT)
                    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                 ::"l"(tmO_lo), "r"(sbuf + 8192u), "r"(co), "r"(tx0), "r"(ty0), "r"(img) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
    }
    if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// The TMA producer thread for PER warpgroups: per K-chunk of every work item, one weight box of the item's PER x N rows
// into each plane of the B slot, then the raw tile(s) or the A tile.  Every ring is consumed in this order, so a wait on one
// ring's slot only ever depends on loads already issued.
template <int MODE, int N, int PER>
__device__ __forceinline__ void fpw_producer(const FpwK& p, XfBarriers& bar, const XfSmem& sm, const CUtensorMap* tm0,
                                             const CUtensorMap* tm1_hi, const CUtensorMap* tm1_lo,
                                             const CUtensorMap* tmB_hi, const CUtensorMap* tmB_lo,
                                             const CUtensorMap* tmW) {
    const uint32_t b_plane = (uint32_t)(PER * N) * 128u, b_slot = 2u * b_plane;
    const int items = p.nsplit / PER;
    int st = 0, bst = 0;
    uint32_t ph = 0, bph = 0;
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        const int tile = u / items, n0 = (u - tile * items) * PER * N;
        const int img = tile / p.a.tiles_per_img, t = tile - img * p.a.tiles_per_img;
        const int oy0 = (t / p.a.tiles_x) * XF_TH, ox0 = (t % p.a.tiles_x) * XF_TW;
        for (int kc = 0; kc < p.a.cchunks; ++kc) {
            mbar_wait_g(smem_u32(&bar.b_empty[bst]), bph ^ 1u);
            const uint32_t fb = smem_u32(&bar.b_full[bst]);
            mbar_expect_tx(fb, b_slot);
            const uint32_t dst = sm.b_off + (uint32_t)bst * b_slot;
            tma_load_2d(dst, tmB_hi, fb, kc * 64, n0);
            tma_load_2d(dst + b_plane, tmB_lo, fb, kc * 64, n0);
            if (++bst == p.bs) { bst = 0; bph ^= 1u; }
            xf_load_a<MODE>(p.a, bar, sm, tm0, tm1_hi, tm1_lo, tmW, kc, img, oy0, ox0, st, ph);
        }
    }
}

template <int MODE, int N, int ACT, bool OUT_SPLIT>
__global__ void __launch_bounds__(XF_THREADS, 1)
conv_fpw_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1_hi,
                const __grid_constant__ CUtensorMap tm1_lo, const __grid_constant__ CUtensorMap tmB_hi,
                const __grid_constant__ CUtensorMap tmB_lo, const __grid_constant__ CUtensorMap tmO_hi,
                const __grid_constant__ CUtensorMap tmO_lo, const __grid_constant__ CUtensorMap tmW,
                const __grid_constant__ FpwK p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) XfBarriers bar;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const XfSmem sm = xf_smem<MODE>(smem_raw, p.a, p.bs, 2u * N * 128u, p.out_bufs);
    xf_cta_init<MODE>(p.a, bar, sm, smem_raw, &tm0, &tm1_hi, &tmB_hi, &tmB_lo);
    // Registers: the launch gives every thread 128 (65536 / 512).  The producer warpgroup (warps 0-3) needs few, so it drops
    // to FPW_PRODUCER_REGS and the transform warps and the MMA warpgroup take what it frees.  The unit width stays <= 64:
    // ptxas sizes the wgmma accumulators against the launch's 128 registers whatever setmaxnreg grants, and serialises
    // wider units (C7511 / C7512).
    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(FPW_PRODUCER_REGS));
        if (warp == 0 && lane == 0) fpw_producer<MODE, N, 1>(p, bar, sm, &tm0, &tm1_hi, &tm1_lo, &tmB_hi, &tmB_lo, &tmW);
    } else if (warp >= 8) {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(FPW_TRANSFORM_REGS));
        // ================================================================== transform warps: raw tile -> A tile
        xf_transform<MODE>(p.a, bar, sm, smem_raw, p.units, [&](int u) { return u / p.nsplit; });
    } else {
        // ================================================================== MMA + epilogue (one warpgroup)
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(FPW_MMA_REGS));
        fpw_consumer<N, ACT, OUT_SPLIT, 1, true>(p, bar, sm, &tmO_hi, &tmO_lo, 0);
    }
}

// XF_DW layers of an even number of 64-channel units: a work item is a pixel tile and two consecutive units of it, so the
// transform warps build each A tile once for both, and two MMA + epilogue warpgroups multiply the same A slot, one per
// unit.  Warp roles (640 threads, one persistent CTA per SM):
//   0      TMA producer: per K-chunk one weight box of both units' 128 rows, then the raw tile(s)
//   1-3    idle after set-up
//   4-7    MMA + epilogue, unit 2j of the pair
//   8-15   transform warps, as in conv_fpw_kernel (xf_transform's thread numbering)
//   16-19  MMA + epilogue, unit 2j + 1
// Each A and B slot is released by all 8 MMA warps.  Per unit, the same K order, products and epilogue as conv_fpw_kernel.
constexpr int FPW_PAIR_THREADS = 640;
// setmaxnreg moves the producer warpgroup's registers to the transform and MMA warpgroups.  The launch gives every thread 96
// (65536 / 640, in steps of 8) and ptxas fits each role's code into those 96 whatever setmaxnreg grants.
constexpr int FPW_PAIR_PRODUCER_REGS = 24, FPW_PAIR_TRANSFORM_REGS = 120, FPW_PAIR_MMA_REGS = 104;
static_assert(128 * FPW_PAIR_PRODUCER_REGS + 256 * FPW_PAIR_TRANSFORM_REGS + 256 * FPW_PAIR_MMA_REGS <= FPW_PAIR_THREADS * 96,
              "register file split");

template <int ACT, bool OUT_SPLIT>
__global__ void __launch_bounds__(FPW_PAIR_THREADS, 1)
conv_fpw_pair(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1_hi,
              const __grid_constant__ CUtensorMap tm1_lo, const __grid_constant__ CUtensorMap tmB_hi,
              const __grid_constant__ CUtensorMap tmB_lo, const __grid_constant__ CUtensorMap tmO_hi,
              const __grid_constant__ CUtensorMap tmO_lo, const __grid_constant__ CUtensorMap tmW,
              const __grid_constant__ FpwK p) {
    constexpr int N = 64;
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) XfBarriers bar;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const XfSmem sm = xf_smem<XF_DW>(smem_raw, p.a, p.bs, 4u * N * 128u, 2 * p.out_bufs);
    xf_cta_init<XF_DW>(p.a, bar, sm, smem_raw, &tm0, &tm1_hi, &tmB_hi, &tmB_lo, 8, FPW_PAIR_THREADS);
    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(FPW_PAIR_PRODUCER_REGS));
        if (warp == 0 && lane == 0) fpw_producer<XF_DW, N, 2>(p, bar, sm, &tm0, &tm1_hi, &tm1_lo, &tmB_hi, &tmB_lo, &tmW);
    } else if (warp >= 8 && warp < 16) {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(FPW_PAIR_TRANSFORM_REGS));
        xf_transform<XF_DW>(p.a, bar, sm, smem_raw, p.units, [&](int u) { return u / (p.nsplit / 2); });
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(FPW_PAIR_MMA_REGS));
        fpw_consumer<N, ACT, OUT_SPLIT, 2, false>(p, bar, sm, &tmO_hi, &tmO_lo, warp < 8 ? 0 : 1);
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

// Whether a layer runs on conv_fpw_pair: XF_DW with an even number of 64-channel units.
static bool fpw_pair(const XfSetup& s) {
    const int n = fpw_unit_width(s.mode, s.n_tile);
    return s.mode == XF_DW && n == 64 && (s.n_tile + n - 1) / n % 2 == 0 && !s.res.base;
}

// Ring depths and shared-memory bytes of a layer on its kernel (xf_rings).  A paired layer's B slot holds both units'
// weights and each MMA warpgroup has one staging buffer of its own.
static size_t fpw_rings(XfProducer& a, const XfSetup& s, int& bs, int& out_bufs) {
    const size_t n = (size_t)fpw_unit_width(s.mode, s.n_tile);
    if (fpw_pair(s)) return xf_rings(a, s.mode, 2 * n * 256, XF_OUT_BUF, false, bs, out_bufs) + XF_OUT_BUF;
    return xf_rings(a, s.mode, n * 256, 0, true, bs, out_bufs);
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
    if (o.H % XF_TH || o.W % XF_TW) return false;
    if (s.res.base) {
        if (s.res.c_stride != 1 || (s.res.fmt != DT_SPLIT16 && s.res.fmt != DT_F32)) return false;
        if (s.res.H != o.H || s.res.W != o.W || s.res.C < s.Cout || ((s.res.ld | s.res.c_off) & 1) || (s.res.plane & 1))
            return false;
    }
    XfProducer a;
    a.cchunks = ((s.low.base ? s.low.C : 0) + s.x.C + 63) / 64;
    int bs, out_bufs;
    return fpw_rings(a, s, bs, out_bufs) != 0;
}

int fpw_prepare(FpwLayer& L, const XfSetup& s) {
    SKPS_CHECK(fpw_supported(s), "conv_fpw: unsupported layer");
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    memset(&L.k, 0, sizeof(L.k));
    FpwK& k = L.k;
    L.mode = s.mode;
    L.n = fpw_unit_width(s.mode, s.n_tile);
    L.pair = fpw_pair(s);
    L.act = s.act;
    L.out_fmt = s.out.fmt;
    const TView& out = s.out;
    if (xf_producer_prepare(k.a, L.src0, L.src1_hi, L.src1_lo, L.w_eff, s)) return 1;
    k.nsplit = (s.n_tile + L.n - 1) / L.n;
    // weights: (K_pad, n_tile) as packed; one box = 64 K x the N rows of the unit (or of both units of a pair)
    const int K_pad = k.a.cchunks * 64;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)K_pad, (cuuint64_t)s.n_tile};
        cuuint64_t strides[1] = {(cuuint64_t)K_pad * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)(L.pair ? 2 * L.n : L.n)};
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
        cuuint32_t box[4] = {32, XF_TW, XF_TH, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        char* base = (char*)out.base + (size_t)out.c_off * oes + (plane ? (size_t)out.plane * 2 : 0);
        CUresult r = enc(plane ? &L.o_lo : &L.o_hi, split ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                         4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         split ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "conv_fpw: cuTensorMapEncodeTiled(out) failed: %d", (int)r);
    }
    if (!split) L.o_lo = L.o_hi;
    const size_t smem = fpw_rings(k.a, s, k.bs, k.out_bufs);
    SKPS_CHECK(smem, "conv_fpw: layer does not fit shared memory");
    L.smem_bytes = (int)smem + 1024;
    k.Cout = s.Cout; k.out_scale = s.out_scale;
    k.bias = s.bias ? s.bias : zero_bias();
    SKPS_CHECK(k.bias, "conv_fpw: zero-bias allocation failed");
    k.res = s.res.base; k.res_fmt = s.res.fmt; k.res_plane = s.res.plane; k.res_ld = s.res.ld; k.res_coff = s.res.c_off;
    k.res_first = s.res.base ? s.res_first : 0;
    return 0;
}

template <int MODE, int N, int ACT, bool SPLIT>
static int fpw_launch_t(const FpwLayer& L, const FpwK& k, int grid, cudaStream_t stream) {
    static int attr_bytes[MAX_DEVICES] = {};
    if (smem_limit((const void*)conv_fpw_kernel<MODE, N, ACT, SPLIT>, attr_bytes, L.smem_bytes)) return 1;
    conv_fpw_kernel<MODE, N, ACT, SPLIT><<<grid, XF_THREADS, L.smem_bytes, stream>>>(
        L.src0, L.src1_hi, L.src1_lo, L.b_hi, L.b_lo, L.o_hi, L.o_lo, L.w_eff, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

template <int ACT, bool SPLIT>
static int fpw_launch_pair_t(const FpwLayer& L, const FpwK& k, int grid, cudaStream_t stream) {
    static int attr_bytes[MAX_DEVICES] = {};
    if (smem_limit((const void*)conv_fpw_pair<ACT, SPLIT>, attr_bytes, L.smem_bytes)) return 1;
    conv_fpw_pair<ACT, SPLIT><<<grid, FPW_PAIR_THREADS, L.smem_bytes, stream>>>(
        L.src0, L.src1_hi, L.src1_lo, L.b_hi, L.b_lo, L.o_hi, L.o_lo, L.w_eff, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

static int fpw_launch_pair(const FpwLayer& L, const FpwK& k, int grid, cudaStream_t stream) {
    const bool sp = L.out_fmt == DT_SPLIT16;
    switch (L.act) {
        case ACT_NONE: return sp ? fpw_launch_pair_t<ACT_NONE, true>(L, k, grid, stream) : fpw_launch_pair_t<ACT_NONE, false>(L, k, grid, stream);
        case ACT_RELU: return sp ? fpw_launch_pair_t<ACT_RELU, true>(L, k, grid, stream) : fpw_launch_pair_t<ACT_RELU, false>(L, k, grid, stream);
        default: break;
    }
    set_error("conv_fpw: activation %d not instantiated", L.act);
    return 1;
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

Grid fpw_grid(const FpwLayer& L, int batch, int num_sms, FpwK* kp) {
    FpwK k = L.k;
    k.units = batch * k.a.tiles_per_img * (L.pair ? k.nsplit / 2 : k.nsplit);
    if (kp) *kp = k;
    return persistent_grid(k.units, num_sms);
}

int fpw_launch(const FpwLayer& L, int batch, int num_sms, cudaStream_t stream) {
    FpwK k;
    const int grid = fpw_grid(L, batch, num_sms, &k).ctas;
    if (L.pair) return fpw_launch_pair(L, k, grid, stream);
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
