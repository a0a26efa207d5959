// PTX wrappers shared by the tensor-core kernels (conv_tc.cu, conv_tct.cu, conv_pw.cu, conv_hm.cu, stem_block.cu, and
// conv_xf.cu and conv_fpw.cu with the A producer they share, xf_producer.h):
// mbarrier, TMA, wgmma and its shared-memory matrix descriptors.  sm_90a.
//
// The accumulator of a 128-row tile lives in the registers of the warpgroup that issues the wgmma instructions: one
// m64nNk16 per 64-row half, so a warp holds rows 16w..16w+15 of each half.
// conv_tct (k x k convs with Cout 96-128), conv_pw (1x1 stride-1 convs without residual or SiLU), conv_fpw (the student's
// fused depthwise / squeeze-excite -> 1x1 layers), conv_hm and stem_block issue wgmma_f16<N> / wg_mma3<N> from straight-line
// code, keep a group in flight with wg_wait<1> where they pipeline, and read the accumulator fragment directly in their
// epilogues.
// conv_tc (the layers left: dilated ASPP, stride-2, residual and SiLU convs, channel-shuffled outputs) and conv_xf (the
// detector's channel-shuffled DWPW layers and maps not made of whole 16 x 8 tiles) still
// issue wg_mma3_128x32 per 32-column chunk and hand each chunk to a one-row-per-thread epilogue layout (row 32q + lane of
// warp q, 32 consecutive columns) with wg_rows32, through 16 KB of shared memory.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "common.h"

namespace skps {

// ------------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// try_wait with a suspend-time hint: the waiting thread sleeps in hardware until the phase completes (or the hint expires)
// instead of re-issuing try_wait back to back, so the spin loops of the waiting roles do not take issue slots from the
// warps doing the work.
constexpr uint32_t MBAR_SUSPEND_NS = 0x989680u;
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}\n" ::"r"(bar), "r"(parity), "r"(MBAR_SUSPEND_NS) : "memory");
}
// Bounded wait for kernels under development: traps (the launch fails with an error) instead of hanging the GPU when a
// pipeline bug leaves a barrier incomplete for ~2 s.
__device__ __forceinline__ void mbar_wait_g(uint32_t bar, uint32_t parity) {
    uint64_t t0 = 0;
    for (uint32_t it = 0;; ++it) {
        uint32_t ok;
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}\n" : "=r"(ok) : "r"(bar), "r"(parity), "r"(MBAR_SUSPEND_NS) : "memory");
        if (ok) return;
        if ((it & 15u) == 15u) {
            uint64_t t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            if (t0 == 0) t0 = t;
            else if (t - t0 > 2000000000ull) __trap();
        }
    }
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// ------------------------------------------------------------------------------------------ wgmma (sm_90a)
// Shared-memory matrix descriptor: K-major tile, 128-byte swizzle, rows of 128 B, 8-row groups 1024 B apart.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t addr) {
    uint64_t d = 0;
    d |= (uint64_t)((addr >> 4) & 0x3FFF);          // start address
    d |= (uint64_t)1 << 16;                         // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;               // stride byte offset
    d |= (uint64_t)1 << 62;                         // SWIZZLE_128B
    return d;
}

// Same for 64-byte swizzle: rows of 64 B (32 fp16 along K), 8-row groups 512 B apart.
__device__ __forceinline__ uint64_t make_smem_desc_sw64(uint32_t addr) {
    uint64_t d = 0;
    d |= (uint64_t)((addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(512 >> 4) << 32;
    d |= (uint64_t)2 << 62;                         // SWIZZLE_64B
    return d;
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Waits until at most N committed wgmma groups of this warpgroup are still in flight.
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pins the accumulator registers in place around asynchronous wgmma: without it the compiler may move or copy them while a
// group that writes them is still in flight.
template <int R>
__device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, fp16 inputs from shared memory (both K-major), fp32 accumulate in registers:
// d[4 i + e] = element (16 w + lane/4 + 8 (e/2), 8 i + 2 (lane%4) + e%2) for warp w of the warpgroup.
template <int N>
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_f16<16>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7"
        "}, %8, %9, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16<128>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

template <>
__device__ __forceinline__ void wgmma_f16<32>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
        "}, %16, %17, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

template <>
__device__ __forceinline__ void wgmma_f16<48>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23"
        "}, %24, %25, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

template <>
__device__ __forceinline__ void wgmma_f16<64>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

template <>
__device__ __forceinline__ void wgmma_f16<96>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
        "}, %48, %49, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// One K-step of the hi/lo three-product scheme on a 64 x N accumulator: lo*hi, hi*lo, then hi*hi (small terms first).
template <int N>
__device__ __forceinline__ void wg_mma3(float* acc, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                        uint32_t accumulate) {
    wgmma_f16<N>(acc, a_lo, b_hi, accumulate);
    wgmma_f16<N>(acc, a_hi, b_lo, 1u);
    wgmma_f16<N>(acc, a_hi, b_hi, 1u);
}

// KS K-steps of 16 of the three-product scheme on a 128 x 128 accumulator held by one warpgroup: acc[0..63] = A rows 0-63,
// acc[64..127] = A rows 64-127 (swizzled K-major A with rows of ROW_BYTES = 128 or 64, row 64 at +64 rows).  Straight-line, so
// the wgmma stay asynchronous.
template <int KS, int ROW_BYTES = 128>
__device__ __forceinline__ void wg_mma3_128x128(float* acc, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                                uint32_t accumulate) {
    static_assert(KS * 32 <= ROW_BYTES, "K-steps past the swizzled row");
    constexpr uint64_t A_HALF = 64 * ROW_BYTES >> 4;
#pragma unroll
    for (int k = 0; k < KS; ++k) {
        const uint64_t koff = (uint64_t)(k * 32 >> 4);     // 16 fp16 = 32 bytes along K
#pragma unroll
        for (int m = 0; m < 2; ++m)
            wg_mma3<128>(acc + 64 * m, a_hi + m * A_HALF + koff, a_lo + m * A_HALF + koff, b_hi + koff, b_lo + koff,
                         k ? 1u : accumulate);
    }
}

// D[64 x 32] (+)= A[64 x 16] * B[32 x 16]^T, fp16 inputs from shared memory (both K-major), fp32 accumulate in registers.
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// One K-step of the hi/lo three-product scheme on a 128 x 32 block: acc[0..15] = rows 0-63, acc[16..31] = rows 64-127.
// a_* address the 128-row A tile, a_half the byte distance between its row 0 and row 64.  Small terms first, then hi*hi.
__device__ __forceinline__ void wg_mma3_128x32(float* acc, uint64_t a_hi, uint64_t a_lo, uint32_t a_half, uint64_t b_hi,
                                               uint64_t b_lo, uint32_t accumulate) {
    const uint64_t ah = (uint64_t)(a_half >> 4);
#pragma unroll
    for (int m = 0; m < 2; ++m) {
        wgmma_n32(acc + 16 * m, a_lo + m * ah, b_hi, accumulate);
        wgmma_n32(acc + 16 * m, a_hi + m * ah, b_lo, 1u);
        wgmma_n32(acc + 16 * m, a_hi + m * ah, b_hi, 1u);
    }
}

// Hands a 128 x 32 accumulator block (wg_mma3_128x32 layout) to the epilogue layout: v[j] = element (32q + lane, j) for
// warp q of the warpgroup.  xs = 16 KB of shared memory owned by the warpgroup; bar = a named barrier id for its 128 threads.
__device__ __forceinline__ void wg_rows32(const float* acc, float* xs, int bar, int q, int lane, float* v) {
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = 64 * m + 16 * q + (lane >> 2) + 8 * (e >> 1), c = 8 * i + 2 * (lane & 3) + (e & 1);
                xs[r * 32 + (c ^ (r & 31))] = acc[16 * m + 4 * i + e];
            }
    asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");
    const int r = 32 * q + lane;
#pragma unroll
    for (int c = 0; c < 32; ++c) v[c] = xs[r * 32 + (c ^ lane)];
    asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");
}

template <int ACT>
__device__ __forceinline__ float act_t(float v) {
    if (ACT == ACT_RELU) return fmaxf(v, 0.f);
    if (ACT == ACT_HSWISH) return v * hsigmoid_f(v);
    if (ACT == ACT_SIGMOID) return sigmoid_f(v);
    if (ACT == ACT_SILU) return v * sigmoid_f(v);
    if (ACT == ACT_HSIGMOID) return hsigmoid_f(v);
    return v;
}
// dynamic index into a register array without forcing it to local memory
__device__ __forceinline__ float v_at(const float* v, int j) {
    float r = v[0];
#pragma unroll
    for (int i = 1; i < 32; ++i) r = (j == i) ? v[i] : r;
    return r;
}


// bias + (residual) + activation on 8 consecutive output channels of one pixel.
// res_first = 0: act(acc*scale + bias) + res   (MobileNetV3 linear bottlenecks)
// res_first = 1: act(acc*scale + bias + res)   (ResNet / HRNet blocks: conv-bn, add, relu)
template <int ACT, class PK>
__device__ __forceinline__ void epilogue8(float* w, const float4 b0, const float4 b1, const PK& p, long long r_el) {
    w[0] = fmaf(w[0], p.out_scale, b0.x); w[1] = fmaf(w[1], p.out_scale, b0.y);
    w[2] = fmaf(w[2], p.out_scale, b0.z); w[3] = fmaf(w[3], p.out_scale, b0.w);
    w[4] = fmaf(w[4], p.out_scale, b1.x); w[5] = fmaf(w[5], p.out_scale, b1.y);
    w[6] = fmaf(w[6], p.out_scale, b1.z); w[7] = fmaf(w[7], p.out_scale, b1.w);
    if (p.res) {
        const float4 r0 = ld4(p.res, p.res_fmt, p.res_plane, r_el);
        const float4 r1 = ld4(p.res, p.res_fmt, p.res_plane, r_el + 4);
        const float r[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
        if (p.res_first) {
#pragma unroll
            for (int j = 0; j < 8; ++j) w[j] = act_t<ACT>(w[j] + r[j]);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) w[j] = act_t<ACT>(w[j]) + r[j];
        }
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) w[j] = act_t<ACT>(w[j]);
    }
}


}  // namespace skps
