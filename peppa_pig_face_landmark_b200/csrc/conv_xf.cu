// Fused "A-producer -> pointwise convolution" kernels on wgmma (sm_90a): the detector's DWPW layers, and every fused layer
// conv_fpw.cu does not take (ragged maps, channel-shuffled outputs).  The A operand is built in shared memory by the
// producer of xf_producer.h, shared with conv_fpw.cu.
//
// Warp roles (512 threads): 0 raw-tile TMA producer, 3 weight-tile TMA producer, 4-7 MMA warpgroup + epilogue (registers ->
// bias/act/residual -> swizzled smem -> TMA store), 8-15 transform.  Three mbarrier rings (raw tiles, A tiles, weight tiles)
// decouple the stages; persistent CTAs, one per SM.
// Output tiles are 16 x 8 pixel blocks (halo 1.4x instead of 2x for row-block tiles); ragged maps hang over the border.
// Precision scheme as conv_tc.cu: fp16 hi/lo operands, three MMAs per K-step, fp32 accumulation in registers.
#include <cuda.h>
#include <cuda_fp16.h>
#include <string.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_xf.h"
#include "tc_ptx.h"

namespace skps {

constexpr int XF_XS_BYTES = 16384;                 // accumulator hand-off buffer of the MMA warpgroup (wg_rows32)
constexpr int XF_ACC_CHUNKS = 8;                   // 32-column accumulator chunks per tile (n_tile <= 256)

template <int MODE, int ACT, bool OUT_SPLIT>
__global__ void __launch_bounds__(XF_THREADS, 1)
conv_xf_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1_hi,
               const __grid_constant__ CUtensorMap tm1_lo, const __grid_constant__ CUtensorMap tmB_hi,
               const __grid_constant__ CUtensorMap tmB_lo, const __grid_constant__ CUtensorMap tmO_hi,
               const __grid_constant__ CUtensorMap tmO_lo, const __grid_constant__ CUtensorMap tmW,
               const __grid_constant__ XfK p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) XfBarriers bar;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // weight planes hold n_sub rows rounded up to 32: the 32-column MMA chunks read whole planes (rows past n_sub only feed
    // accumulator columns that are never stored)
    const uint32_t b_plane = (uint32_t)((p.n_sub + 31) & ~31) * 128u, b_slot = 2u * b_plane;
    const XfSmem sm = xf_smem<MODE>(smem_raw, p.a, p.bs, b_slot, p.out_bufs);
    const uint32_t xs_off = sm.w_off + (MODE == XF_DW ? (uint32_t)(10 * p.a.cchunks * 64 * 4) : 0u);
    xf_cta_init<MODE>(p.a, bar, sm, smem_raw, &tm0, &tm1_hi, &tmB_hi, &tmB_lo);
    const int total_tiles = p.m_tiles;

    if (warp == 0) {
        // ================================================================== raw-tile / A-tile TMA producer
        if (lane == 0) {
            int st = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int img = tile / p.a.tiles_per_img, t = tile - img * p.a.tiles_per_img;
                const int oy0 = (t / p.a.tiles_x) * XF_TH, ox0 = (t % p.a.tiles_x) * XF_TW;
                for (int kc = 0; kc < p.a.cchunks; ++kc)
                    xf_load_a<MODE>(p.a, bar, sm, &tm0, &tm1_hi, &tm1_lo, &tmW, kc, img, oy0, ox0, st, ph);
            }
        }
    } else if (warp == 3) {
        // ================================================================== weight-tile TMA producer
        if (lane == 0) {
            int st = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                for (int kc = 0; kc < p.a.cchunks; ++kc) {
                    for (int nh = 0; nh < p.nsplit; ++nh) {
                        mbar_wait_g(smem_u32(&bar.b_empty[st]), ph ^ 1u);
                        const uint32_t fb = smem_u32(&bar.b_full[st]);
                        mbar_expect_tx(fb, 2u * (uint32_t)p.n_sub * 128u);
                        const uint32_t dst = sm.b_off + (uint32_t)st * b_slot;
                        tma_load_2d(dst, &tmB_hi, fb, kc * 64, nh * p.n_sub);
                        tma_load_2d(dst + b_plane, &tmB_lo, fb, kc * 64, nh * p.n_sub);
                        if (++st == p.bs) { st = 0; ph ^= 1u; }
                    }
                }
            }
        }
    } else if (warp >= 8) {
        // ================================================================== transform warps: raw tile -> A tile
        xf_transform<MODE>(p.a, bar, sm, smem_raw, total_tiles, [](int tile) { return tile; });
    } else if (warp >= 4) {
        // ================================================================== MMA + epilogue (one warpgroup)
        // accumulator chunk (nh, j) = columns nh * n_sub + 32 j .. of weight slot nh; wg_rows32 hands it over as one pixel
        // row (row = 32q + lane) x 32 columns per thread
        const int q = warp & 3;
        const int row = q * 32 + lane;
        float* xs = reinterpret_cast<float*>(smem_raw + (xs_off - smem_u32(smem_raw)));
        const int cps = (p.n_sub + 31) >> 5;                    // chunks per weight slot
        int ast = 0, bst = 0;
        uint32_t aph = 0, bph = 0;
        int store_i = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            float accv[XF_ACC_CHUNKS][32];
            for (int kc = 0; kc < p.a.cchunks; ++kc) {
                mbar_wait_g(smem_u32(&bar.a_full[ast]), aph);
                const uint32_t sa = sm.a_off + (uint32_t)ast * XF_A_BYTES;
                const uint64_t a_hi = make_smem_desc(sa), a_lo = make_smem_desc(sa + XF_A_PLANE);
                const int ksteps = p.a.chunk_ksteps[kc];
                for (int nh = 0; nh < p.nsplit; ++nh) {
                    mbar_wait_g(smem_u32(&bar.b_full[bst]), bph);
                    const uint32_t sb = sm.b_off + (uint32_t)bst * b_slot;
                    const uint64_t b_hi = make_smem_desc(sb), b_lo = make_smem_desc(sb + b_plane);
                    wg_fence();
#pragma unroll
                    for (int c = 0; c < XF_ACC_CHUNKS; ++c) {
                        if (c < nh * cps || c >= (nh + 1) * cps) continue;
                        const uint64_t bo = (uint64_t)((c - nh * cps) * 32 * 128 >> 4);
                        for (int k = 0; k < ksteps; ++k) {
                            const uint64_t koff = (uint64_t)(k * 32 >> 4);
                            wg_mma3_128x32(accv[c], a_hi + koff, a_lo + koff, 64u * 128u, b_hi + bo + koff, b_lo + bo + koff,
                                           (kc | k) != 0);
                        }
                    }
                    wg_commit();
                    wg_wait0();
                    if (lane == 0) mbar_arrive(smem_u32(&bar.b_empty[bst]));
                    if (++bst == p.bs) { bst = 0; bph ^= 1u; }
                }
                if (lane == 0) mbar_arrive(smem_u32(&bar.a_empty[ast]));
                if (++ast == p.a.as) { ast = 0; aph ^= 1u; }
            }
            const int img = tile / p.a.tiles_per_img, t = tile - img * p.a.tiles_per_img;
            const int ty0 = (t / p.a.tiles_x) * XF_TH, tx0 = (t % p.a.tiles_x) * XF_TW;
            const int y = ty0 + row / XF_TW, x = tx0 + row % XF_TW;
            const bool row_ok = y < p.a.H && x < p.a.W;
            const long long pix = row_ok ? ((long long)img * p.a.H + y) * p.a.W + x : 0;
#pragma unroll 1
            for (int c = 0; c < p.nsplit * cps; ++c) {
                const int nh = c / cps, c0 = nh * p.n_sub + (c - nh * cps) * 32;
                if (c0 >= p.Cout) break;
                float v[32];
#pragma unroll
                for (int o = 0; o < XF_ACC_CHUNKS; ++o)
                    if (o == c) wg_rows32(accv[o], xs, 2, q, lane, v);
                const int nvalid = min(min(32, (nh + 1) * p.n_sub - c0), p.Cout - c0);
                const long long o_el = pix * p.out_ld + p.out_coff + c0;
                const long long r_el = pix * p.res_ld + p.res_coff + c0;
                if (p.tma_store && (nvalid == 32 || c0 + nvalid == p.Cout)) {
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        float* w = v + 8 * g;
                        if (8 * g < nvalid) {
                            const float4* b4 = reinterpret_cast<const float4*>(p.bias + c0 + 8 * g);
                            epilogue8<ACT>(w, __ldg(b4), __ldg(b4 + 1), p, r_el + 8 * g);
                        }
                    }
                    const uint32_t sbuf = sm.o_off + (uint32_t)(store_i % p.out_bufs) * XF_OUT_BUF;
                    if (q == 0 && lane == 0) {
                        if (p.out_bufs == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                        else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    }
                    ++store_i;
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                    if (OUT_SPLIT) {
                        const uint32_t rh = sbuf + (uint32_t)row * 64u, rl = rh + 8192u;
#pragma unroll
                        for (int g = 0; g < 4; ++g) {
                            uint32_t hp[4], lp[4];
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const float a0 = v[8 * g + 2 * j], a1 = v[8 * g + 2 * j + 1];
                                const __half2 h2 = __floats2half2_rn(a0, a1);
                                const float2 hf = __half22float2(h2);
                                const __half2 l2 = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
                                hp[j] = *reinterpret_cast<const uint32_t*>(&h2);
                                lp[j] = *reinterpret_cast<const uint32_t*>(&l2);
                            }
                            const uint32_t slot = (uint32_t)((g ^ (row >> 1)) & 3) * 16u;          // 64-byte swizzle
                            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(rh + slot), "r"(hp[0]), "r"(hp[1]), "r"(hp[2]), "r"(hp[3]) : "memory");
                            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(rl + slot), "r"(lp[0]), "r"(lp[1]), "r"(lp[2]), "r"(lp[3]) : "memory");
                        }
                    } else {
                        const uint32_t rf = sbuf + (uint32_t)row * 128u;
#pragma unroll
                        for (int g = 0; g < 8; ++g) {
                            const uint32_t slot = (uint32_t)((g ^ row) & 7) * 16u;                 // 128-byte swizzle
                            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(rf + slot), "f"(v[4 * g]), "f"(v[4 * g + 1]), "f"(v[4 * g + 2]), "f"(v[4 * g + 3]) : "memory");
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    asm volatile("bar.sync 1, 128;" ::: "memory");
                    if (q == 0 && lane == 0) {
                        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                     ::"l"(&tmO_hi), "r"(sbuf), "r"(c0), "r"(tx0), "r"(ty0), "r"(img) : "memory");
                        if (OUT_SPLIT)
                            asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                         ::"l"(&tmO_lo), "r"(sbuf + 8192u), "r"(c0), "r"(tx0), "r"(ty0), "r"(img) : "memory");
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    }
                    continue;
                }
                if (p.out_cstride != 1 && (nvalid & 7) == 0) {
                    // Strided destination (the detector's ShuffleNetV2 units write straight into channel-shuffled views,
                    // c_stride 2).  A lane owns a pixel, so a direct store instruction would touch 32 different sectors with
                    // 2-4 bytes each (several times the kernel's own work).  The 32 x 32 block is
                    // transposed through this warp's 4 KB staging slice (XOR-swizzled, conflict-free both ways) and stored
                    // pixel by pixel with lane = channel: 4 sectors per instruction.
                    #pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        float* w = v + 8 * g;
                        if (8 * g < nvalid) {
                            const float4* b4 = reinterpret_cast<const float4*>(p.bias + c0 + 8 * g);
                            epilogue8<ACT>(w, __ldg(b4), __ldg(b4 + 1), p, r_el + 8 * g);
                        }
                    }
                    float* xs = reinterpret_cast<float*>(smem_raw + (sm.o_off - smem_u32(smem_raw))) + (warp - 4) * 1024;
                    __syncwarp();
#pragma unroll
                    for (int j = 0; j < 32; ++j) xs[lane * 32 + (j ^ lane)] = v[j];
                    __syncwarp();
                    const int pix_lo = (int)(pix & 0xffffffffll), pix_hi = (int)(pix >> 32);
#pragma unroll 4
                    for (int i = 0; i < 32; ++i) {
                        const bool ok_i = __shfl_sync(0xffffffffu, (int)row_ok, i) != 0;
                        const long long pix_i = ((long long)__shfl_sync(0xffffffffu, pix_hi, i) << 32) |
                                                (unsigned int)__shfl_sync(0xffffffffu, pix_lo, i);
                        if (ok_i && lane < nvalid)
                            st1(p.out, OUT_SPLIT ? DT_SPLIT16 : DT_F32, p.out_plane,
                                pix_i * p.out_ld + p.out_coff + (long long)(c0 + lane) * p.out_cstride, xs[i * 32 + (lane ^ i)]);
                    }
                    __syncwarp();
                    continue;
                }
                if (!row_ok) continue;
                const bool fast = (nvalid & 7) == 0 && p.out_cstride == 1 && ((p.out_ld | (p.out_coff + c0)) & 7) == 0;
                if (fast) {
                    const int ng = nvalid >> 3;
                    const float4* b4 = reinterpret_cast<const float4*>(p.bias + c0);
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        if (g < ng) {
                            float* w = v + 8 * g;
                            epilogue8<ACT>(w, __ldg(b4 + 2 * g), __ldg(b4 + 2 * g + 1), p, r_el + 8 * g);
                            float8 o8;
#pragma unroll
                            for (int j = 0; j < 8; ++j) o8.v[j] = w[j];
                            st8(p.out, OUT_SPLIT ? DT_SPLIT16 : DT_F32, p.out_plane, o_el + 8 * g, o8);
                        }
                    }
                } else {
#pragma unroll 1
                    for (int j = 0; j < nvalid; ++j) {
                        float f = fmaf(v_at(v, j), p.out_scale, __ldg(p.bias + c0 + j));
                        const float r = p.res ? ld1(p.res, p.res_fmt, p.res_plane, r_el + j) : 0.f;
                        f = p.res_first ? act_t<ACT>(f + r) : act_t<ACT>(f) + r;
                        st1(p.out, OUT_SPLIT ? DT_SPLIT16 : DT_F32, p.out_plane,
                            pix * p.out_ld + p.out_coff + (long long)(c0 + j) * p.out_cstride, f);
                    }
                }
            }
        }
        if (p.tma_store && q == 0 && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

// ------------------------------------------------------------------------------------------ host side
size_t xf_rings(XfProducer& k, int mode, size_t b_slot, size_t reserve, bool two_out_bufs, int& bs, int& out_bufs) {
    const size_t budget = 227 * 1024 - 1024 - 512 - reserve;
    const size_t w_bytes = mode == XF_DW ? (size_t)10 * k.cchunks * 64 * 4 : 0;
    k.as = 2; bs = 2; k.rs = mode == XF_DW ? 2 : 0; out_bufs = 1;
    auto total = [&]() { return (size_t)k.as * XF_A_BYTES + (size_t)bs * b_slot + (size_t)out_bufs * XF_OUT_BUF +
                                (size_t)k.rs * XF_RAW_BYTES + w_bytes; };
    if (total() > budget) return 0;
    // two halves consume two raw slots at once: a third slot is what lets the TMA producer run ahead
    if (mode == XF_DW) { k.rs = 3; if (total() > budget) k.rs = 2; }
    if (two_out_bufs) { out_bufs = 2; if (total() > budget) out_bufs = 1; }     // the store of slab i drains under slab i+1
    bs = 3; if (total() > budget) bs = 2;
    if (mode == XF_DW && k.rs == 3) { k.rs = 4; if (total() > budget) k.rs = 3; }
    k.as = 3; if (total() > budget) k.as = 2;
    if (bs == 3) { bs = 4; if (total() > budget) bs = 3; }
    return total();
}

static bool view_ok8(const TView& v) { return v.base && v.c_stride == 1 && !((v.C | v.ld | v.c_off) & 7); }

bool xf_supported(const XfSetup& s) {
    if (s.n_tiles != 1 || s.n_tile > 256 || (s.n_tile & 15) || s.Cout > s.n_tile) return false;
    if (!s.out.base || s.out.H < XF_TH || s.out.W < XF_TW) return false;
    if (s.mode == XF_SCALE) {
        if (!view_ok8(s.x) || s.x.fmt != DT_SPLIT16 || !s.gate.base || s.gate.fmt != DT_F32 || s.gate.c_stride != 1) return false;
        if ((s.gate.ld | s.gate.c_off) & 3) return false;
        return s.x.H == s.out.H && s.x.W == s.out.W && (s.x.C + 63) / 64 <= XF_MAX_CHUNKS;
    }
    if (!view_ok8(s.x) || (s.x.fmt != DT_F32 && s.x.fmt != DT_SPLIT16)) return false;
    if (s.x.H != s.out.H || s.x.W != s.out.W) return false;
    int K = s.x.C;
    if (s.low.base) {
        if (!view_ok8(s.low) || s.low.fmt != DT_F32 || s.x.fmt != DT_SPLIT16 || !s.weff) return false;   // one float32 source map per layer
        if (s.low.C % 64 || s.out.H != 2 * s.low.H || s.out.W != 2 * s.low.W) return false;
        if (s.out.H % XF_TH || s.out.W % XF_TW || s.out.H < 2 * XF_TH) return false;     // no tile holds first AND last rows
        K += s.low.C;
    }
    return (K + 63) / 64 <= XF_MAX_CHUNKS;
}
static int encode4(EncodeTiledFn enc, CUtensorMap* m, const TView& v, int plane, int max_batch, int box_c, int box_w, int box_h,
                   CUtensorMapSwizzle swz) {
    const bool split = v.fmt == DT_SPLIT16;
    const int esz = split ? 2 : 4;
    cuuint64_t dims[4] = {(cuuint64_t)v.C, (cuuint64_t)v.W, (cuuint64_t)v.H, (cuuint64_t)max_batch};
    cuuint64_t strides[3] = {(cuuint64_t)v.ld * esz, (cuuint64_t)v.W * v.ld * esz, (cuuint64_t)v.H * v.W * v.ld * esz};
    cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    char* base = (char*)v.base + (size_t)v.c_off * esz + (plane ? (size_t)v.plane * 2 : 0);
    CUresult r = enc(m, split ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, dims, strides, box,
                     estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    SKPS_CHECK(r == CUDA_SUCCESS, "xf producer: cuTensorMapEncodeTiled failed: %d", (int)r);
    return 0;
}

int xf_producer_prepare(XfProducer& k, CUtensorMap& src0, CUtensorMap& src1_hi, CUtensorMap& src1_lo, CUtensorMap& w_eff,
                        const XfSetup& s) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    const TView& out = s.out;
    k.H = out.H; k.W = out.W;
    k.tiles_x = (out.W + XF_TW - 1) / XF_TW;
    k.tiles_per_img = k.tiles_x * ((out.H + XF_TH - 1) / XF_TH);
    const int Cu = s.low.base ? s.low.C : 0;
    k.Cin = Cu + s.x.C;
    k.cchunks = (k.Cin + 63) / 64;
    k.dw_act = s.dw_act;
    k.halves = s.low.base ? 1 : 0;
    k.Hl = s.low.base ? s.low.H : 0; k.Wl = s.low.base ? s.low.W : 0;
    for (int kc = 0; kc < k.cchunks; ++kc) {
        const int valid = k.Cin - kc * 64 < 64 ? k.Cin - kc * 64 : 64;
        k.chunk_subs[kc] = valid <= 32 ? 1 : 2;
        k.chunk_ksteps[kc] = (uint8_t)((valid + 15) / 16);
        for (int h = 0; h < 2; ++h) {
            const int c = kc * 64 + h * 32;
            if (c < Cu) { k.sub_mode[kc * 2 + h] = XS_UP_F32; k.sub_c[kc * 2 + h] = (int16_t)c; }
            else { k.sub_mode[kc * 2 + h] = s.x.fmt == DT_SPLIT16 ? XS_DW_SPLIT : XS_DW_F32; k.sub_c[kc * 2 + h] = (int16_t)(c - Cu); }
        }
    }
    k.dww = s.dww;
    if (s.mode == XF_SCALE) {
        k.gate = (const float*)s.gate.base; k.gate_ld = s.gate.ld; k.gate_coff = s.gate.c_off;
    }
    src0 = CUtensorMap(); src1_hi = CUtensorMap(); src1_lo = CUtensorMap();
    if (s.mode == XF_SCALE) {
        if (encode4(enc, &src1_hi, s.x, 0, s.max_batch, 64, XF_TW, XF_TH, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
        if (encode4(enc, &src1_lo, s.x, 1, s.max_batch, 64, XF_TW, XF_TH, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
        src0 = src1_hi;
    } else {
        if (s.low.base) {
            if (encode4(enc, &src0, s.low, 0, s.max_batch, 32, XF_LW, XF_LH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
        }
        if (s.x.fmt == DT_SPLIT16) {
            if (encode4(enc, &src1_hi, s.x, 0, s.max_batch, 32, XF_IW, XF_IH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
            if (encode4(enc, &src1_lo, s.x, 1, s.max_batch, 32, XF_IW, XF_IH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
            if (!s.low.base) src0 = src1_hi;
        } else {
            if (encode4(enc, &src0, s.x, 0, s.max_batch, 32, XF_IW, XF_IH, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
            src1_hi = src0; src1_lo = src0;
        }
    }
    w_eff = src0;
    if (s.low.base) {
        // [sub][cy 4][cx 4][tap 9][32 ch] float32; a tile takes the 3 x 3 classes it can contain
        cuuint64_t dims[5] = {32, 9, 4, 4, (cuuint64_t)(s.low.C / 32)};
        cuuint64_t strides[4] = {128, 9 * 128, 4 * 9 * 128, 16 * 9 * 128};
        k.wcx = k.tiles_x == 1 ? 4 : 3;
        cuuint32_t box[5] = {32, 9, (cuuint32_t)k.wcx, 3, 1};
        cuuint32_t estr[5] = {1, 1, 1, 1, 1};
        CUresult r = enc(&w_eff, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, (void*)s.weff, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "xf producer: cuTensorMapEncodeTiled(weff) failed: %d", (int)r);
    }
    return 0;
}

int xf_prepare(XfLayer& L, const XfSetup& s) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    SKPS_CHECK(xf_supported(s), "conv_xf: unsupported layer");
    memset(&L.k, 0, sizeof(L.k));
    XfK& k = L.k;
    L.mode = s.mode;
    if (xf_producer_prepare(k.a, L.src0, L.src1_hi, L.src1_lo, L.w_eff, s)) return 1;
    const TView& out = s.out;
    k.n_tile = s.n_tile;
    k.nsplit = s.n_tile > 128 ? 2 : 1;
    if (k.nsplit == 2 && (s.n_tile % 32)) k.nsplit = 1;          // halves must stay multiples of 16
    k.n_sub = s.n_tile / k.nsplit;
    const int K_pad = k.a.cchunks * 64;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)K_pad, (cuuint64_t)s.n_tile};
        cuuint64_t strides[1] = {(cuuint64_t)K_pad * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)k.n_sub};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(plane ? &L.b_lo : &L.b_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)(plane ? s.w_lo : s.w_hi), dims,
                         strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "conv_xf: cuTensorMapEncodeTiled(B) failed: %d", (int)r);
    }
    const int oes = out.fmt == DT_SPLIT16 ? 2 : 4;
    k.tma_store = (out.c_stride == 1 && (s.Cout % 8) == 0 && ((size_t)out.ld * oes) % 16 == 0 &&
                   ((size_t)out.c_off * oes) % 16 == 0) ? 1 : 0;
    if (k.tma_store) {
        for (int plane = 0; plane < (out.fmt == DT_SPLIT16 ? 2 : 1); ++plane) {
            cuuint64_t dims[4] = {(cuuint64_t)s.Cout, (cuuint64_t)out.W, (cuuint64_t)out.H, (cuuint64_t)s.max_batch};
            cuuint64_t strides[3] = {(cuuint64_t)out.ld * oes, (cuuint64_t)out.W * out.ld * oes,
                                     (cuuint64_t)out.H * out.W * out.ld * oes};
            cuuint32_t box[4] = {32, XF_TW, XF_TH, 1};
            cuuint32_t estr[4] = {1, 1, 1, 1};
            char* base = (char*)out.base + (size_t)out.c_off * oes + (plane ? (size_t)out.plane * 2 : 0);
            CUresult r = enc(plane ? &L.o_lo : &L.o_hi,
                             out.fmt == DT_SPLIT16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base,
                             dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             out.fmt == DT_SPLIT16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            SKPS_CHECK(r == CUDA_SUCCESS, "conv_xf: cuTensorMapEncodeTiled(out) failed: %d", (int)r);
        }
        if (out.fmt != DT_SPLIT16) L.o_lo = L.o_hi;
    } else {
        L.o_hi = L.b_hi; L.o_lo = L.b_hi;
    }
    const size_t b_slot = (size_t)((k.n_sub + 31) & ~31) * 256;
    const size_t smem = xf_rings(k.a, s.mode, b_slot, XF_XS_BYTES, k.tma_store != 0, k.bs, k.out_bufs);
    SKPS_CHECK(smem, "conv_xf: layer does not fit shared memory");
    L.smem_bytes = (int)(smem + XF_XS_BYTES + 1024);
    k.Cout = s.Cout; k.act = s.act; k.out_scale = s.out_scale;
    k.bias = s.bias ? s.bias : zero_bias();
    SKPS_CHECK(k.bias, "conv_xf: zero-bias allocation failed");
    k.out = out.base; k.out_fmt = out.fmt; k.out_plane = out.plane; k.out_ld = out.ld; k.out_coff = out.c_off;
    k.out_cstride = out.c_stride;
    k.res = s.res.base; k.res_fmt = s.res.fmt; k.res_plane = s.res.plane; k.res_ld = s.res.ld; k.res_coff = s.res.c_off;
    k.res_first = s.res.base ? s.res_first : 0;
    return 0;
}

template <int MODE, int ACT, bool SPLIT>
static int xf_launch_t(const XfLayer& L, const XfK& k, int grid, cudaStream_t stream) {
    static int attr_bytes[MAX_DEVICES] = {};
    if (smem_limit((const void*)conv_xf_kernel<MODE, ACT, SPLIT>, attr_bytes, L.smem_bytes)) return 1;
    conv_xf_kernel<MODE, ACT, SPLIT><<<grid, XF_THREADS, L.smem_bytes, stream>>>(L.src0, L.src1_hi, L.src1_lo, L.b_hi, L.b_lo,
                                                                                  L.o_hi, L.o_lo, L.w_eff, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

template <int MODE>
static int xf_launch_m(const XfLayer& L, const XfK& k, int grid, cudaStream_t stream) {
    const bool sp = k.out_fmt == DT_SPLIT16;
    switch (k.act) {
        case ACT_NONE: return sp ? xf_launch_t<MODE, ACT_NONE, true>(L, k, grid, stream) : xf_launch_t<MODE, ACT_NONE, false>(L, k, grid, stream);
        case ACT_RELU: return sp ? xf_launch_t<MODE, ACT_RELU, true>(L, k, grid, stream) : xf_launch_t<MODE, ACT_RELU, false>(L, k, grid, stream);
        case ACT_HSWISH: return sp ? xf_launch_t<MODE, ACT_HSWISH, true>(L, k, grid, stream) : xf_launch_t<MODE, ACT_HSWISH, false>(L, k, grid, stream);
        case ACT_SILU: return sp ? xf_launch_t<MODE, ACT_SILU, true>(L, k, grid, stream) : xf_launch_t<MODE, ACT_SILU, false>(L, k, grid, stream);
        default: break;
    }
    set_error("conv_xf: activation %d not instantiated", k.act);
    return 1;
}

Grid xf_grid(const XfLayer& L, int batch, int num_sms, XfK* kp) {
    XfK k = L.k;
    k.m_tiles = batch * k.a.tiles_per_img;
    if (kp) *kp = k;
    return persistent_grid(k.m_tiles, num_sms);
}

int xf_launch(const XfLayer& L, int batch, int num_sms, cudaStream_t stream) {
    XfK k;
    const int grid = xf_grid(L, batch, num_sms, &k).ctas;
    return L.mode == XF_SCALE ? xf_launch_m<XF_SCALE>(L, k, grid, stream) : xf_launch_m<XF_DW>(L, k, grid, stream);
}

}  // namespace skps
