// Dense convolution as a wgmma implicit GEMM (sm_90a): the landmark network's 1x1 and 3x3
// (incl. dilated) convolutions, 96.7 % of its MACs (SURVEY.md 8a row a9).
//
//   C[M = N*H*W pixels][Cout] = sum over taps (ky,kx), ci of  A[pixel + tap][ci] * W[co][tap][ci]
//
// * Operands are float16 hi/lo pairs: v = hi + lo with hi = fp16(v), lo = fp16(v - hi) (22 mantissa
//   bits).  Each K-step issues three f16 MMAs into one fp32 register accumulator:
//   hi*hi + hi*lo + lo*hi.  Measured against the fp32 oracle this keeps landmarks within 6e-5 px
//   (budget 1e-3 px); plain fp16/bf16/tf32 single-pass does not (0.02-0.5 px).  Tensor work issued is
//   therefore 3x the algorithmic FLOPs.
// * A tiles (128 pixels x 64 channels) are fetched by 4-D TMA straight from the NHWC activation:
//   box (64 ch, bw, bh) with signed start coordinates, so the conv zero padding and dilation come
//   from TMA out-of-bounds fill; no im2col buffer exists.  B tiles (n_tile x 64) come from the
//   pre-split, K-padded weight matrix.  Both land in 128B-swizzled shared memory.
// * Warp roles: warp 0 TMA producer; warpgroups 1 and 2 (warps 4-11) issue the wgmma instructions for their
//   32-column chunks of the tile (the chunks alternate between them) and run the epilogue on them
//   (registers -> bias/act/residual -> global).  Persistent CTAs, one per SM; the producer fills the next
//   stages while the epilogue of a tile runs.
// * Which layers run here: the engine gives the heat-map head to conv_hm.cu, k x k convs with Cout 96-128 to conv_tct.cu and
//   1x1 stride-1 layers without residual or SiLU to conv_pw.cu, in that order; conv_tc takes the rest (the dilated ASPP
//   convs, stride-2, residual and SiLU layers, channel-shuffled outputs).  skps_debug_conv_tc2 still runs 1x1 layers here.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_tc.h"
#include "conv_tct.h"
#include "tc_ptx.h"

namespace skps {

// ------------------------------------------------------------------------------------------ kernel
constexpr int TC_BM = 128;            // pixels per tile (two m64 wgmma halves)
constexpr int TC_BK = 64;             // channels per k-block (one 128-byte swizzle atom of fp16)
constexpr int A_TILE_BYTES = TC_BM * TC_BK * 2;
constexpr int TC_THREADS = 384;        // warp 0: TMA; warps 4-11: MMA + epilogue
constexpr int TC_XS_BYTES = 2 * 16384; // accumulator hand-off buffers of the two MMA warpgroups (wg_rows32)
constexpr int TC_MAX_OWN = 4;          // 32-column chunks a warpgroup accumulates per tile (mt * n_tile <= 256)
constexpr int MAX_STAGES = 4;

// One level of a warp reduce-scatter of per-column (max, first arg-max): 2N column candidates per lane in, N out; after the
// levels 16, 8, 4, 2, 1 lane L holds column L reduced over the warp's 32 rows.  Ties keep the smaller pixel index.
template <int N>
__device__ __forceinline__ void argmax_scatter(float* v, int* id, int off, int lane) {
    const bool hi = (lane & off) != 0;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const float keep = hi ? v[j + N] : v[j], snd = hi ? v[j] : v[j + N];
        const int kid = hi ? id[j + N] : id[j], sid = hi ? id[j] : id[j + N];
        const float r = __shfl_xor_sync(0xffffffffu, snd, off);
        const int ri = __shfl_xor_sync(0xffffffffu, sid, off);
        const bool take = r > keep || (r == keep && ri < kid);
        v[j] = take ? r : keep;
        id[j] = take ? ri : kid;
    }
}

template <int ACT, bool OUT_SPLIT>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
               const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
               const __grid_constant__ CUtensorMap tmO_hi, const __grid_constant__ CUtensorMap tmO_lo, const TcK p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[MAX_STAGES], empty_bar[MAX_STAGES];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t xs_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t tile_base = xs_base + (uint32_t)TC_XS_BYTES;
    // weight tiles hold n_tile rows rounded up to 32 (the 32-column MMA chunks read them whole; rows past n_tile only feed
    // accumulator columns that are never stored)
    const uint32_t n_pad = (uint32_t)((p.n_tile + 31) & ~31);
    const uint32_t b_tile_bytes = n_pad * TC_BK * 2;
    // stage = [A0_hi][A0_lo]([A1_hi][A1_lo])[B_hi][B_lo]: with mt = 2 two pixel tiles share one weight tile
    const uint32_t a_bytes = (uint32_t)p.mt * 2u * A_TILE_BYTES;
    const uint32_t stage_bytes = a_bytes + 2u * b_tile_bytes;
    const uint32_t tx_bytes = a_bytes + 4u * (uint32_t)p.n_tile * TC_BK;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA_lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_lo) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(smem_u32(&full_bar[s]), 1);
            mbar_init(smem_u32(&empty_bar[s]), 8);            // one arrival per MMA warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // epilogue staging for TMA stores: one 16 KB buffer (128 rows x 32 channels, hi+lo or float32) per warp group
    const uint32_t stage_out = tile_base + (uint32_t)p.stages * stage_bytes;
    const int m_groups = (p.m_tiles + p.mt - 1) / p.mt;
    const int total_tiles = m_groups * p.n_tiles;          // work items: (group of mt pixel tiles) x N tile
    const int kblocks = p.taps * p.cchunks;

    if (warp == 0) {
        // ================================================================== TMA producer
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            const int tiles_x = (p.W + p.bw - 1) / p.bw;       // ragged maps: edge tiles hang over, TMA zero-fills / clips
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int g_idx = tile / p.n_tiles, n_idx = tile - g_idx * p.n_tiles;
                int img[2], y0[2], x0[2];
                for (int u = 0; u < p.mt; ++u) {
                    const int m_idx = min(g_idx * p.mt + u, p.m_tiles - 1);     // odd tail: reload the last tile, result unused
                    const int img_l = p.ipt > 1 ? m_idx * p.ipt : m_idx / p.tiles_per_img;
                    const int t = p.ipt > 1 ? 0 : m_idx - img_l * p.tiles_per_img;
                    img[u] = img_l + p.img0;
                    y0[u] = (t / tiles_x) * p.bh * p.stride;                    // input-space origin of the tile
                    x0[u] = (t % tiles_x) * p.bw * p.stride;
                }
                for (int kb = 0; kb < kblocks; ++kb) {
                    mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1u);
                    const uint32_t fb = smem_u32(&full_bar[stage]);
                    mbar_expect_tx(fb, tx_bytes);
                    const int tap = kb / p.cchunks, cc = kb - tap * p.cchunks;
                    const int ky = tap / p.kw, kx = tap - ky * p.kw;
                    const uint32_t sa = tile_base + (uint32_t)stage * stage_bytes;
                    for (int u = 0; u < p.mt; ++u) {
                        const int cx = x0[u] + kx * p.dil - p.pad, cy = y0[u] + ky * p.dil - p.pad;
                        tma_load_4d(sa + (uint32_t)u * 2u * A_TILE_BYTES, &tmA_hi, fb, cc * TC_BK, cx, cy, img[u]);
                        tma_load_4d(sa + (uint32_t)u * 2u * A_TILE_BYTES + A_TILE_BYTES, &tmA_lo, fb, cc * TC_BK, cx, cy, img[u]);
                    }
                    tma_load_2d(sa + a_bytes, &tmB_hi, fb, kb * TC_BK, n_idx * p.n_tile);
                    tma_load_2d(sa + a_bytes + b_tile_bytes, &tmB_lo, fb, kb * TC_BK, n_idx * p.n_tile);
                    if (++stage == p.stages) { stage = 0; phase ^= 1u; }
                }
            }
        }
    } else if (warp >= 4) {
        // ================================================================== MMA + epilogue
        // 2 warpgroups: (warp-4)/4 selects the odd/even 32-column chunks a warpgroup accumulates, warp%4 the 32 rows of
        // the tile it handles in the epilogue.  One thread = one output pixel x 32 consecutive channels per chunk.
        const int q = warp & 3;
        const int half_id = (warp - 4) >> 2;
        const int row = q * 32 + lane;
        float* xs = reinterpret_cast<float*>(smem_raw + (xs_base - smem_u32(smem_raw))) + half_id * 4096;
        int stage = 0;
        uint32_t phase = 0;
        int store_i = 0;                 // TMA stores issued by this warp group so far
        int chunk_ctr = 0;               // 32-column chunks handed out so far (same sequence in both groups)
        const int tiles_x = (p.W + p.bw - 1) / p.bw;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int g_idx = tile / p.n_tiles, n_idx = tile - g_idx * p.n_tiles;
            // chunks of this tile: (pixel tile u, chunk ci) in order; the warpgroup owns those with (chunk_ctr + index) % 2
            // == half_id, the same alternation the epilogue below walks
            const int n_chunks_t = (min(p.n_tile, p.Cout - n_idx * p.n_tile) + 31) >> 5;
            int own_u[TC_MAX_OWN], own_c[TC_MAX_OWN], n_own = 0;
            for (int g = 0; g < p.mt * n_chunks_t && n_own < TC_MAX_OWN; ++g)
                if (((chunk_ctr + g) & 1) == half_id) { own_u[n_own] = g / n_chunks_t; own_c[n_own] = g % n_chunks_t; ++n_own; }
            float accv[TC_MAX_OWN][32];
            for (int kb = 0; kb < kblocks; ++kb) {
                mbar_wait(smem_u32(&full_bar[stage]), phase);
                const uint32_t sa = tile_base + (uint32_t)stage * stage_bytes;
                const uint64_t b_hi = make_smem_desc(sa + a_bytes);
                const uint64_t b_lo = make_smem_desc(sa + a_bytes + b_tile_bytes);
                // only the 16-channel steps that hold real channels (TMA zero-fills the rest)
                const int cc = kb % p.cchunks;
                const int ksteps = min(TC_BK / 16, (p.Cin - cc * TC_BK + 15) / 16);
                wg_fence();
#pragma unroll
                for (int o = 0; o < TC_MAX_OWN; ++o) {
                    if (o >= n_own) break;
                    const uint32_t au = sa + (uint32_t)own_u[o] * 2u * A_TILE_BYTES;
                    const uint64_t a_hi = make_smem_desc(au), a_lo = make_smem_desc(au + A_TILE_BYTES);
                    const uint64_t bo = (uint64_t)(own_c[o] * 32 * 128 >> 4);
                    for (int k = 0; k < ksteps; ++k) {
                        const uint64_t koff = (uint64_t)(k * 32 >> 4);           // 16 fp16 = 32 bytes along K
                        wg_mma3_128x32(accv[o], a_hi + koff, a_lo + koff, 64u * 128u, b_hi + bo + koff, b_lo + bo + koff,
                                       (kb | k) != 0);
                    }
                }
                wg_commit();
                wg_wait0();
                if (lane == 0) mbar_arrive(smem_u32(&empty_bar[stage]));     // frees the smem stage
                if (++stage == p.stages) { stage = 0; phase ^= 1u; }
            }
            int own_i = 0;
          for (int u = 0; u < p.mt; ++u) {
            const int m_idx = g_idx * p.mt + u;
            if (m_idx >= p.m_tiles) break;
            const int img_l = p.ipt > 1 ? m_idx * p.ipt : m_idx / p.tiles_per_img, img = img_l + p.img0;
            const int t = p.ipt > 1 ? 0 : m_idx - img_l * p.tiles_per_img;
            // multi-image tiles (ipt > 1): bw = W, bh = ipt*H, so y runs past H into the next image and the linear
            // pixel index below is still right; rows of images past the batch are computed but never stored
            const int y = (t / tiles_x) * p.bh + row / p.bw, x = (t % tiles_x) * p.bw + row % p.bw;
            // rows of an edge tile that hang over the map (ragged tiling) are computed but never stored
            const bool row_ok = p.ipt == 1 ? (y < p.H && x < p.W) : img + y / p.H < p.img_end;
            const long long pix = row_ok ? ((long long)img * p.H + y) * p.W + x : 0;
            const int co_tile = n_idx * p.n_tile;
            // 32-column chunks alternate between the two warp groups with a counter that runs on across tiles: layers with an
            // odd number of chunks per tile (Cout 24, 72, 40 ...) would otherwise leave all / two thirds of the epilogue to
            // group 0 (the epilogue, not HBM, bounds those layers)
            const int n_chunks = (min(p.n_tile, p.Cout - co_tile) + 31) >> 5;
            for (int ci = 0; ci < n_chunks; ++ci) {
                if (((chunk_ctr + ci) & 1) != half_id) continue;
                const int c0 = ci * 32;
                float v[32];
#pragma unroll
                for (int o = 0; o < TC_MAX_OWN; ++o)
                    if (o == own_i) wg_rows32(accv[o], xs, 5 + half_id, q, lane, v);
                ++own_i;
                const int co0 = co_tile + c0;
                const int nvalid = min(min(32, p.n_tile - c0), p.Cout - co0);   // n_tile need not be a multiple of 32
                if (p.hm_val) {
                    // heat-map head (model.py:511-554 postp): only max and first arg-max of every score map are needed.
                    // Scores = acc * scale + bias (no activation); reduce the tile's 128 pixels per channel here and write
                    // (max, pixel index) per tile instead of the map (436 MB per 256-face batch that hm_decode re-read).
                    int id[32];
                    const int my = row_ok ? y * p.W + x : 0x7fffffff;
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        v[j] = (row_ok && j < nvalid) ? fmaf(v[j], p.out_scale, __ldg(p.bias + co0 + (j < nvalid ? j : 0))) : -INFINITY;
                        id[j] = my;
                    }
                    argmax_scatter<16>(v, id, 16, lane); argmax_scatter<8>(v, id, 8, lane); argmax_scatter<4>(v, id, 4, lane);
                    argmax_scatter<2>(v, id, 2, lane); argmax_scatter<1>(v, id, 1, lane);
                    // per-warp column maxima are combined across the 4 lane quarters through the (otherwise unused) store
                    // staging area of the dynamic shared memory: [8 warps][32] float then [8][32] int
                    float(*hm_sv)[32] = reinterpret_cast<float(*)[32]>(smem_raw + (stage_out - smem_u32(smem_raw)));
                    int(*hm_si)[32] = reinterpret_cast<int(*)[32]>(smem_raw + (stage_out - smem_u32(smem_raw)) + 1024);
                    hm_sv[warp - 4][lane] = v[0];
                    hm_si[warp - 4][lane] = id[0];
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + half_id) : "memory");
                    if (q == 0) {
                        float bv = hm_sv[half_id * 4][lane];
                        int bi = hm_si[half_id * 4][lane];
#pragma unroll
                        for (int w2 = 1; w2 < 4; ++w2) {
                            const float ov = hm_sv[half_id * 4 + w2][lane];
                            const int oi = hm_si[half_id * 4 + w2][lane];
                            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
                        }
                        if (lane < nvalid) {
                            const long long o = ((long long)img * p.tiles_per_img + t) * p.hm_ld + co0 + lane;
                            p.hm_val[o] = bv;
                            p.hm_idx[o] = bi;
                        }
                    }
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + half_id) : "memory");
                    continue;
                }
                const long long o_el = pix * p.out_ld + p.out_coff + co0;
                // vector path: whole groups of 8 channels (every Cout in the network but the 294-wide heat map and
                // the 1-channel sSE map is a multiple of 8), unit channel stride, 16-byte aligned destination
                // a 32-wide box may only be stored when its columns are all ours: a full chunk, or the chunk that ends
                // the tensor (TMA clips at Cout); a ragged chunk in the middle (n_tile % 32 != 0) takes the direct path
                if (p.tma_store && (nvalid == 32 || co0 + nvalid == p.Cout)) {
                    // ---- bias/act/residual on all 32 columns (columns past Cout are clipped by the TMA store)
                    const long long r_el = pix * p.res_ld + p.res_coff + co0;
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        float* w = v + 8 * g;
                        if (8 * g < nvalid) {                         // nvalid is a multiple of 8 on this path
                            const float4* b4 = reinterpret_cast<const float4*>(p.bias + co0 + 8 * g);
                            epilogue8<ACT>(w, __ldg(b4), __ldg(b4 + 1), p, r_el + 8 * g);
                        }
                    }
                    // ---- the staging buffer of this warp group must have been drained by its previous store
                    // staging buffers: one or two per warp group; with two, the store issued two chunks ago must have
                    // drained (wait_group.read 1), so the store of the previous chunk overlaps this chunk's work
                    const uint32_t sbuf = stage_out + (uint32_t)(half_id * p.out_bufs + (store_i % p.out_bufs)) * 16384u;
                    if (q == 0 && lane == 0) {
                        if (p.out_bufs == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                        else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    }
                    ++store_i;
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + half_id) : "memory");
                    if (OUT_SPLIT) {
                        // rows of 64 B per plane: [hi plane 8 KB][lo plane 8 KB]
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
                            // 64-byte swizzle (matches the tensor map): 16-byte chunk index ^= (row/2) % 4, so the
                            // 32 rows a warp writes spread over all banks and TMA un-swizzles on the way out
                            const uint32_t slot = (uint32_t)((g ^ (row >> 1)) & 3) * 16u;
                            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(rh + slot), "r"(hp[0]), "r"(hp[1]), "r"(hp[2]), "r"(hp[3]) : "memory");
                            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(rl + slot), "r"(lp[0]), "r"(lp[1]), "r"(lp[2]), "r"(lp[3]) : "memory");
                        }
                    } else {
                        const uint32_t rf = sbuf + (uint32_t)row * 128u;
#pragma unroll
                        for (int g = 0; g < 8; ++g) {
                            const uint32_t slot = (uint32_t)((g ^ row) & 7) * 16u;      // 128-byte swizzle: chunk ^= row % 8
                            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(rf + slot), "f"(v[4 * g]), "f"(v[4 * g + 1]), "f"(v[4 * g + 2]), "f"(v[4 * g + 3]) : "memory");
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + half_id) : "memory");
                    if (q == 0 && lane == 0) {
                        const int ty0 = (t / tiles_x) * p.bh, tx0 = (t % tiles_x) * p.bw;
                        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                     ::"l"(&tmO_hi), "r"(sbuf), "r"(co0), "r"(tx0), "r"(ty0), "r"(img) : "memory");
                        if (OUT_SPLIT)
                            asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                                         ::"l"(&tmO_lo), "r"(sbuf + 8192u), "r"(co0), "r"(tx0), "r"(ty0), "r"(img) : "memory");
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
                    const long long r_el = pix * p.res_ld + p.res_coff + co0;
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        float* w = v + 8 * g;
                        if (8 * g < nvalid) {
                            const float4* b4 = reinterpret_cast<const float4*>(p.bias + co0 + 8 * g);
                            epilogue8<ACT>(w, __ldg(b4), __ldg(b4 + 1), p, r_el + 8 * g);
                        }
                    }
                    float* xs = reinterpret_cast<float*>(smem_raw + (stage_out - smem_u32(smem_raw))) + (warp - 4) * 1024;
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
                                pix_i * p.out_ld + p.out_coff + (long long)(co0 + lane) * p.out_cstride, xs[i * 32 + (lane ^ i)]);
                    }
                    __syncwarp();
                    continue;
                }
                const bool fast = (nvalid & 7) == 0 && p.out_cstride == 1 && ((p.out_ld | (p.out_coff + co0)) & 7) == 0;
                if (!row_ok) continue;
                if (fast) {
                    const int ng = nvalid >> 3;                       // warp-uniform
                    const float4* b4 = reinterpret_cast<const float4*>(p.bias + co0);
                    const long long r_el = pix * p.res_ld + p.res_coff + co0;
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        if (g < ng) {
                            float* w = v + 8 * g;
                            epilogue8<ACT>(w, __ldg(b4 + 2 * g), __ldg(b4 + 2 * g + 1), p, r_el + 8 * g);
                            if (OUT_SPLIT) {
                                __half* oh = (__half*)p.out + o_el + 8 * g;
                                uint4 hv, lv;
                                uint32_t* hp = reinterpret_cast<uint32_t*>(&hv);
                                uint32_t* lp = reinterpret_cast<uint32_t*>(&lv);
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    const float a0 = w[2 * j], a1 = w[2 * j + 1];
                                    const __half2 h2 = __floats2half2_rn(a0, a1);
                                    const float2 hf = __half22float2(h2);
                                    const __half2 l2 = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
                                    hp[j] = *reinterpret_cast<const uint32_t*>(&h2);
                                    lp[j] = *reinterpret_cast<const uint32_t*>(&l2);
                                }
                                *reinterpret_cast<uint4*>(oh) = hv;
                                *reinterpret_cast<uint4*>(oh + p.out_plane) = lv;
                            } else {
                                float* o = (float*)p.out + o_el + 8 * g;
                                *reinterpret_cast<float4*>(o) = make_float4(w[0], w[1], w[2], w[3]);
                                *reinterpret_cast<float4*>(o + 4) = make_float4(w[4], w[5], w[6], w[7]);
                            }
                        }
                    }
                } else {
                    // ragged tail / unaligned destination: scalar, not unrolled (rare)
                    const long long r_el = pix * p.res_ld + p.res_coff + co0;
#pragma unroll 1
                    for (int j = 0; j < nvalid; ++j) {
                        float f = fmaf(v_at(v, j), p.out_scale, __ldg(p.bias + co0 + j));
                        const float r = p.res ? ld1(p.res, p.res_fmt, p.res_plane, r_el + j) : 0.f;
                        f = p.res_first ? act_t<ACT>(f + r) : act_t<ACT>(f) + r;
                        st1(p.out, OUT_SPLIT ? DT_SPLIT16 : DT_F32, p.out_plane,
                            pix * p.out_ld + p.out_coff + (long long)(co0 + j) * p.out_cstride, f);
                    }
                }
            }
            chunk_ctr += n_chunks;
          }
        }
    }

    if (p.tma_store && warp >= 4 && (warp & 3) == 0 && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ------------------------------------------------------------------------------------------ host side
// Tile width for an Ho x Wo OUTPUT map (0 = no tiling): 128-pixel tiles are bw x (128/bw) blocks of one image.
// Maps whose width divides (or is a multiple of) 128 use row-block tiles (bw = min(W, 128)) that cover the map exactly.
// Any other map (the detector's 48x80 / 24x40 / 12x20, re-targeted @192/@320 exports) gets the bw in {64,32,16,8} with the
// fewest tiles, edge tiles hanging over the right/bottom border: the TMA loads zero-fill and the TMA stores clip what
// lies outside, the direct-store path masks it.
static int tc_pick_bw(int H, int W) {
    if (W >= TC_BM && W % TC_BM == 0) return TC_BM;
    if (W < TC_BM && TC_BM % W == 0 && H % (TC_BM / W) == 0) return W;
    int best = 0, best_tiles = 1 << 30;
    for (int bw = 64; bw >= 8; bw >>= 1) {
        const int bh = TC_BM / bw;
        if (bw > W + 7 || bh > H + 7) continue;                  // keep boxes within ~the map
        const int tiles = ((W + bw - 1) / bw) * ((H + bh - 1) / bh);
        if (tiles < best_tiles) { best_tiles = tiles; best = bw; }
    }
    return best;
}

// Ho x Wo = OUTPUT map: 128-pixel tiles are row blocks of one image (ragged at the border if need be), or whole images
// (Ho*Wo | 128)
bool tc_shape_ok(int H, int W, int Cin, int in_ld, int in_coff) {
    if (W < 8 || (Cin % 8) || (in_ld % 8) || (in_coff % 8)) return false;
    if (H * W < TC_BM) return TC_BM % W == 0 && TC_BM % (H * W) == 0;
    return tc_pick_bw(H, W) != 0;
}

int tc_prepare(TcLayer& L, const TcSetup& s) {
    EncodeTiledFn enc = tensor_map_encoder();
    SKPS_CHECK(enc, "cuTensorMapEncodeTiled entry point not available");
    const int stride = s.stride > 0 ? s.stride : 1;
    SKPS_CHECK((stride == 1 || stride == 2) && s.H % stride == 0 && s.W % stride == 0, "conv_tc: stride %d on %dx%d", stride,
               s.H, s.W);
    const int Ho = s.H / stride, Wo = s.W / stride;
    SKPS_CHECK(tc_shape_ok(Ho, Wo, s.Cin, s.in_ld, s.in_coff), "conv_tc: unsupported shape %dx%d Cin=%d ld=%d off=%d",
               Ho, Wo, s.Cin, s.in_ld, s.in_coff);
    SKPS_CHECK(s.kh == s.kw && s.pad == s.dil * (s.kh - 1) / 2, "conv_tc: only 'same' square kernels");
    L.k = TcK();
    TcK& k = L.k;
    k.H = Ho; k.W = Wo; k.stride = stride;             // the kernel's H, W are the OUTPUT map
    k.ipt = Ho * Wo < TC_BM ? TC_BM / (Ho * Wo) : 1;
    k.bw = k.ipt > 1 ? Wo : tc_pick_bw(Ho, Wo);
    k.bh = TC_BM / k.bw;
    k.tiles_per_img = k.ipt > 1 ? 1 : ((Ho + k.bh - 1) / k.bh) * ((Wo + k.bw - 1) / k.bw);
    k.taps = s.kh * s.kw; k.kw = s.kw; k.dil = s.dil; k.pad = s.pad;
    k.cchunks = (s.Cin + TC_BK - 1) / TC_BK;
    k.Cout = s.Cout; k.act = s.act; k.out_scale = s.out_scale;
    k.n_tile = s.n_tile; k.n_tiles = s.n_tiles;
    SKPS_CHECK(s.n_tile >= 8 && s.n_tile <= 256 && s.n_tile % 8 == 0, "conv_tc: n_tile %d", s.n_tile);
    // two pixel tiles per weight-tile load when both accumulators fit the registers of the MMA warpgroups (N <= 128)
    // and two pipeline stages still fit in shared memory (checked below): halves the weight traffic from L2
    k.mt = s.n_tile <= 128 ? 2 : 1;
    const size_t n_pad = (size_t)((s.n_tile + 31) & ~31);
    auto stage_size = [&]() {
        return (size_t)k.mt * 2 * (size_t)A_TILE_BYTES + 2 * n_pad * TC_BK * 2;
    };
    size_t stage_bytes = stage_size();
    // TMA-store epilogue: full 128-byte lines instead of 16-byte pieces per thread.  Needs a unit-stride,
    // 16-byte aligned destination whose channel count is a multiple of 8 (the swizzle-free box clips at Cout).
    const int oes = s.out_fmt == DT_SPLIT16 ? 2 : 4;
    k.tma_store = (s.out_cstride == 1 && (s.Cout % 8) == 0 && ((size_t)s.out_ld * oes) % 16 == 0 &&
                   ((size_t)s.out_coff * oes) % 16 == 0 && !s.hm_val) ? 1 : 0;
    // two staging buffers per epilogue warp group when the pipeline still gets its stages, else one
    const size_t budget = 227 * 1024 - 1024 - 1024 - TC_XS_BYTES;  // minus static smem slack, alignment pad, hand-off
    const size_t out_min = (k.tma_store || s.out_cstride != 1) ? (size_t)2 * 16384 : 0;
    if (k.mt == 2 && (budget - out_min) / stage_bytes < 2) {
        k.mt = 1;                                                    // two stages matter more than the shared weight tile
        stage_bytes = stage_size();
    }
    const int want_stages = (int)((budget - 2 * 16384) / stage_bytes) > MAX_STAGES ? MAX_STAGES
                                                                                  : (int)((budget - 2 * 16384) / stage_bytes);
    k.out_bufs = (k.tma_store && (budget - 4 * 16384) / stage_bytes >= (size_t)want_stages) ? 2 : 1;
    const size_t out_stage = (k.tma_store || s.out_cstride != 1) ? (size_t)2 * k.out_bufs * 16384 : 0;   // strided outputs transpose through it
    int stages = (int)((budget - out_stage) / stage_bytes);
    if (stages < 2 && k.n_tile > 128 && k.n_tile % 16 == 0) {
        // a 256-row weight tile leaves room for one stage only: the packed matrix is row-contiguous, so the same rows
        // are addressed as twice as many tiles of half the width
        TcSetup h = s;
        h.n_tile = s.n_tile / 2;
        h.n_tiles = s.n_tiles * 2;
        return tc_prepare(L, h);
    }
    k.stages = stages > MAX_STAGES ? MAX_STAGES : stages;
    SKPS_CHECK(k.stages >= 2, "conv_tc: tile too large for shared memory");
    L.smem_bytes = (int)(TC_XS_BYTES + k.stages * stage_bytes + out_stage + 1024 + (s.hm_val ? 2048 : 0));    // + the arg-max exchange area

    // activations: (C, W, H, N) fp16, channel window [in_coff, in_coff+Cin) of rows of in_ld channels
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)s.Cin, (cuuint64_t)s.W, (cuuint64_t)s.H, (cuuint64_t)s.max_batch};
        cuuint64_t strides[3] = {(cuuint64_t)s.in_ld * 2, (cuuint64_t)s.W * s.in_ld * 2, (cuuint64_t)s.H * s.W * s.in_ld * 2};
        // stride 2: TMA walks W and H with element stride 2; a box of 2*bw x 2*bh source elements lands as bw x bh in smem.
        // small maps: the box spans `ipt` whole images (rows of the A tile = (n, y, x))
        const cuuint32_t box_h = (cuuint32_t)(k.ipt > 1 ? Ho : k.bh);
        cuuint32_t box[4] = {TC_BK, (cuuint32_t)(k.bw * stride), box_h * (cuuint32_t)stride, (cuuint32_t)k.ipt};
        cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
        void* base = (void*)((__half*)s.in_base + (plane ? s.in_plane : 0) + s.in_coff);
        CUresult r = enc(plane ? &L.a_lo : &L.a_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(A) failed: %d", (int)r);
    }
    // weights: (K_pad, rows) fp16, rows = n_tiles*n_tile (zero rows beyond Cout)
    const int K_pad = k.taps * k.cchunks * TC_BK;
    for (int plane = 0; plane < 2; ++plane) {
        cuuint64_t dims[2] = {(cuuint64_t)K_pad, (cuuint64_t)(k.n_tiles * k.n_tile)};
        cuuint64_t strides[1] = {(cuuint64_t)K_pad * 2};
        cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)k.n_tile};
        cuuint32_t estr[2] = {1, 1};
        void* base = (void*)(plane ? s.w_lo : s.w_hi);
        CUresult r = enc(plane ? &L.b_lo : &L.b_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(B) failed: %d", (int)r);
    }
    if (k.tma_store) {
        // output view (C, W, H, N); the staged tile is [row = pixel][32 channels] per plane, 64-byte (float16) or
        // 128-byte (float32) rows written with the matching hardware swizzle (bank-conflict-free)
        for (int plane = 0; plane < (s.out_fmt == DT_SPLIT16 ? 2 : 1); ++plane) {
            cuuint64_t dims[4] = {(cuuint64_t)s.Cout, (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)s.max_batch};
            cuuint64_t strides[3] = {(cuuint64_t)s.out_ld * oes, (cuuint64_t)Wo * s.out_ld * oes,
                                     (cuuint64_t)Ho * Wo * s.out_ld * oes};
            cuuint32_t box[4] = {32, (cuuint32_t)k.bw, (cuuint32_t)(k.ipt > 1 ? Ho : k.bh), (cuuint32_t)k.ipt};
            cuuint32_t estr[4] = {1, 1, 1, 1};
            char* base = (char*)s.out + (size_t)s.out_coff * oes + (plane ? (size_t)s.out_plane * 2 : 0);
            CUresult r = enc(plane ? &L.o_lo : &L.o_hi,
                             s.out_fmt == DT_SPLIT16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4,
                             base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             s.out_fmt == DT_SPLIT16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            SKPS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(out) failed: %d", (int)r);
        }
        if (s.out_fmt != DT_SPLIT16) L.o_lo = L.o_hi;
    } else {
        L.o_hi = L.a_hi; L.o_lo = L.a_hi;      // unused placeholders
    }
    k.bias = s.bias ? s.bias : zero_bias();
    SKPS_CHECK(k.bias, "conv_tc: zero-bias allocation failed");
    k.Cin = s.Cin;
    k.out = s.out; k.out_fmt = s.out_fmt; k.out_plane = s.out_plane; k.out_ld = s.out_ld; k.out_coff = s.out_coff;
    k.out_cstride = s.out_cstride;
    k.res = s.res; k.res_fmt = s.res_fmt; k.res_plane = s.res_plane; k.res_ld = s.res_ld; k.res_coff = s.res_coff;
    k.res_first = s.res ? s.res_first : 0;
    k.hm_val = s.hm_val; k.hm_idx = s.hm_idx; k.hm_ld = s.hm_ld;
    if (k.hm_val) {
        SKPS_CHECK(k.ipt == 1 && s.act == ACT_NONE && !s.res && (Ho * Wo) % TC_BM == 0 && k.tiles_per_img * TC_BM == Ho * Wo,
                   "conv_tc: heat-map partials need whole 128-pixel tiles, no activation, no residual");
    }
    return 0;
}

template <int ACT, bool SPLIT>
static int tc_launch_t(const TcLayer& L, const TcK& k, int grid, cudaStream_t stream) {
    static int attr_bytes[MAX_DEVICES] = {};
    if (smem_limit((const void*)conv_tc_kernel<ACT, SPLIT>, attr_bytes, 227 * 1024 - 1024)) return 1;
    conv_tc_kernel<ACT, SPLIT><<<grid, TC_THREADS, L.smem_bytes, stream>>>(L.a_hi, L.a_lo, L.b_hi, L.b_lo, L.o_hi, L.o_lo, k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

Grid tc_grid(const TcLayer& L, int batch, int num_sms, TcK* kp) {
    TcK k = L.k;
    k.m_tiles = k.ipt > 1 ? (batch + k.ipt - 1) / k.ipt : batch * k.tiles_per_img;
    k.img_end = batch;
    if (kp) *kp = k;
    return persistent_grid((long long)((k.m_tiles + k.mt - 1) / k.mt) * k.n_tiles, num_sms);
}

int tc_launch(const TcLayer& L, int batch, int num_sms, cudaStream_t stream) {
    TcK k;
    const int grid = tc_grid(L, batch, num_sms, &k).ctas;
    const bool sp = k.out_fmt == DT_SPLIT16;
    switch (k.act) {
        case ACT_NONE: return sp ? tc_launch_t<ACT_NONE, true>(L, k, grid, stream) : tc_launch_t<ACT_NONE, false>(L, k, grid, stream);
        case ACT_RELU: return sp ? tc_launch_t<ACT_RELU, true>(L, k, grid, stream) : tc_launch_t<ACT_RELU, false>(L, k, grid, stream);
        case ACT_HSWISH: return sp ? tc_launch_t<ACT_HSWISH, true>(L, k, grid, stream) : tc_launch_t<ACT_HSWISH, false>(L, k, grid, stream);
        case ACT_SIGMOID: return sp ? tc_launch_t<ACT_SIGMOID, true>(L, k, grid, stream) : tc_launch_t<ACT_SIGMOID, false>(L, k, grid, stream);
        case ACT_SILU: return sp ? tc_launch_t<ACT_SILU, true>(L, k, grid, stream) : tc_launch_t<ACT_SILU, false>(L, k, grid, stream);
        default: break;
    }
    set_error("conv_tc: activation %d not instantiated", k.act);
    return 1;
}

// float32 NHWC -> hi/lo float16 planes (used by the debug entry point and by f32->split conversions)
__global__ void f32_to_split_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo,
                                    long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v = src[i];
    __half h = __float2half_rn(v);
    hi[i] = h;
    lo[i] = __float2half_rn(v - __half2float(h));
}

}  // namespace skps

using namespace skps;

// Debug/unit-test entry: one conv through the tensor-core kernel on host data.
//   x      [host] float32 NHWC (N,H,W,Cin)
//   w_hi/w_lo [host] float16 (rows, K_pad) as packed by plan.py:pack_tc_weights
//   out    [host] float32 NHWC (N,H,W,Cout)
extern "C" SKPS_API int skps_debug_conv_tc2(const float* x, int N, int H, int W, int Cin, const void* w_hi,
                                            const void* w_lo, const float* bias, int Cout, int ksize, int dil, int act,
                                            int n_tile, int n_tiles, float out_scale, const float* residual,
                                            int out_split, float* out, int stride, int res_first, int max_batch);

extern "C" SKPS_API int skps_debug_conv_tc(const float* x, int N, int H, int W, int Cin, const void* w_hi,
                                           const void* w_lo, const float* bias, int Cout, int ksize, int dil, int act,
                                           int n_tile, int n_tiles, float out_scale, const float* residual,
                                           int out_split, float* out) {
    return skps_debug_conv_tc2(x, N, H, W, Cin, w_hi, w_lo, bias, Cout, ksize, dil, act, n_tile, n_tiles, out_scale,
                               residual, out_split, out, 1, 0, N);
}

// Same with a conv stride (1 or 2; out is N x H/stride x W/stride x Cout), the residual order
// (res_first: act(conv + res) instead of act(conv) + res) and a buffer capacity max_batch >= N
// (multi-image tiles write whole tiles: exercises the partial last tile).
extern "C" SKPS_API int skps_debug_conv_tc2(const float* x, int N, int H, int W, int Cin, const void* w_hi,
                                            const void* w_lo, const float* bias, int Cout, int ksize, int dil, int act,
                                            int n_tile, int n_tiles, float out_scale, const float* residual,
                                            int out_split, float* out, int stride, int res_first, int max_batch) {
    SKPS_CHECK(x && w_hi && w_lo && out, "debug_conv_tc: null argument");
    SKPS_CHECK((stride == 1 || stride == 2) && max_batch >= N, "debug_conv_tc: bad stride/max_batch");
    const int Ho = H / stride, Wo = W / stride;
    const long long nin = (long long)N * H * W * Cin, nout = (long long)N * Ho * Wo * Cout;
    const long long cin_cap = (long long)max_batch * H * W * Cin, cout_cap = (long long)max_batch * Ho * Wo * Cout;
    const int cchunks = (Cin + TC_BK - 1) / TC_BK;
    const size_t wbytes = (size_t)n_tiles * n_tile * ksize * ksize * cchunks * TC_BK * 2;
    float *d_x = nullptr, *d_bias = nullptr, *d_out = nullptr, *d_res = nullptr;
    __half *d_split = nullptr, *d_wh = nullptr, *d_wl = nullptr, *d_osplit = nullptr;
    SKPS_CUDA(cudaMalloc(&d_x, nin * 4));
    SKPS_CUDA(cudaMalloc(&d_split, cin_cap * 4));
    SKPS_CUDA(cudaMemset(d_split, 0, cin_cap * 4));
    SKPS_CUDA(cudaMalloc(&d_wh, wbytes));
    SKPS_CUDA(cudaMalloc(&d_wl, wbytes));
    SKPS_CUDA(cudaMalloc(&d_out, cout_cap * 4));
    SKPS_CUDA(cudaMalloc(&d_osplit, cout_cap * 4));
    SKPS_CUDA(cudaMemcpy(d_x, x, nin * 4, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(d_wh, w_hi, wbytes, cudaMemcpyHostToDevice));
    SKPS_CUDA(cudaMemcpy(d_wl, w_lo, wbytes, cudaMemcpyHostToDevice));
    if (bias) {
        SKPS_CUDA(cudaMalloc(&d_bias, Cout * 4));
        SKPS_CUDA(cudaMemcpy(d_bias, bias, Cout * 4, cudaMemcpyHostToDevice));
    }
    if (residual) {
        SKPS_CUDA(cudaMalloc(&d_res, nout * 4));
        SKPS_CUDA(cudaMemcpy(d_res, residual, nout * 4, cudaMemcpyHostToDevice));
    }
    f32_to_split_kernel<<<(unsigned)((nin + 255) / 256), 256>>>(d_x, d_split, d_split + cin_cap, nin);
    SKPS_CUDA(cudaGetLastError());
    TcSetup s = {};
    s.H = H; s.W = W; s.Cin = Cin; s.in_ld = Cin; s.in_coff = 0; s.max_batch = max_batch;
    s.in_base = d_split; s.in_plane = cin_cap;
    s.kh = s.kw = ksize; s.dil = dil; s.pad = dil * (ksize - 1) / 2; s.stride = stride; s.res_first = res_first;
    s.Cout = Cout; s.act = act; s.n_tile = n_tile; s.n_tiles = n_tiles; s.out_scale = out_scale;
    s.w_hi = d_wh; s.w_lo = d_wl; s.bias = d_bias;
    s.out = out_split ? (void*)d_osplit : (void*)d_out; s.out_fmt = out_split ? DT_SPLIT16 : DT_F32;
    s.out_plane = cout_cap; s.out_ld = Cout; s.out_coff = 0; s.out_cstride = 1;
    s.res = d_res; s.res_fmt = DT_F32; s.res_plane = 0; s.res_ld = Cout; s.res_coff = 0;
    const int sms = sm_count();
    if (tct_applicable(s)) {                        // the engine routes such layers to the transposed kernel (conv_tct.cu)
        float* d_zero = nullptr;
        if (!s.bias) {
            SKPS_CUDA(cudaMalloc(&d_zero, 1024 * 4));
            SKPS_CUDA(cudaMemset(d_zero, 0, 1024 * 4));
            s.bias = d_zero;
        }
        TctLayer T;
        if (tct_prepare(T, s)) return 1;
        if (tct_launch(T, N, sms, 0)) return 1;
        SKPS_CUDA(cudaDeviceSynchronize());
        if (d_zero) cudaFree(d_zero);
    } else {
    TcLayer L;
    if (tc_prepare(L, s)) return 1;
    if (tc_launch(L, N, sms, 0)) return 1;
    }
    SKPS_CUDA(cudaDeviceSynchronize());
    if (out_split) {
        // recombine hi+lo on the host side of the test
        __half* tmp = (__half*)malloc(nout * 4);
        SKPS_CUDA(cudaMemcpy(tmp, d_osplit, nout * 2, cudaMemcpyDeviceToHost));
        SKPS_CUDA(cudaMemcpy(tmp + nout, d_osplit + cout_cap, nout * 2, cudaMemcpyDeviceToHost));
        for (long long i = 0; i < nout; ++i) out[i] = __half2float(tmp[i]) + __half2float(tmp[nout + i]);
        free(tmp);
    } else {
        SKPS_CUDA(cudaMemcpy(out, d_out, nout * 4, cudaMemcpyDeviceToHost));
    }
    cudaFree(d_x); cudaFree(d_split); cudaFree(d_wh); cudaFree(d_wl); cudaFree(d_out); cudaFree(d_osplit);
    if (d_bias) cudaFree(d_bias);
    if (d_res) cudaFree(d_res);
    return 0;
}
