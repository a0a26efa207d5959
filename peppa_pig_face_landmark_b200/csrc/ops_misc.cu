// Non-GEMM layers of the two networks (sm_90a): depthwise conv, pooling, resizes, channel-view
// copy, global average pool, BatchNorm affine, scSE apply, and the two decode tails.  All are
// HBM/L2-bound gathers; they read/write NHWC float32 through channel views so concat, slice and
// channel shuffle never cost a pass of their own.
#include "common.h"

namespace skps {

static inline int blocks_for(long long n, int threads) {
    // kernels index threads with 32-bit ints; every tensor here is far below 2^31 elements
    if (n >= (1LL << 31) - threads) n = (1LL << 31) - threads - 1;
    return (int)((n + threads - 1) / threads);
}

// ------------------------------------------------------------------------------------------
// Depthwise kxk conv + bias + activation.  One thread = one output pixel x 4 channels.
// (kps_student.onnx conv_dw nodes, e.g. node 4; yolov5n-0.5.onnx branch*.0/.3 nodes.)
// ------------------------------------------------------------------------------------------
struct DwK {
    const void* in; int in_ld, in_coff, H, W; int in_fmt; long long in_plane;
    void* out; int out_ld, out_coff, out_cstride, Ho, Wo, C; int out_fmt; long long out_plane;
    const float* w; const float* bias;
    int kh, kw, sh, sw, ph, pw, dh, dw, act;
    long long total;   // batch*Ho*Wo*(C/4)
};

__global__ void __launch_bounds__(256) dwconv_kernel(const DwK p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;     // 32-bit on purpose: 64-bit div/mod is emulated
    if (i >= (int)p.total) return;
    const int C4 = p.C >> 2;
    int c = (i % C4) * 4;
    int pix = i / C4;
    int ox = pix % p.Wo;
    int t = pix / p.Wo;
    int oy = t % p.Ho;
    int n = t / p.Ho;
    float4 acc = *reinterpret_cast<const float4*>(p.bias + c);
    const int iy0 = oy * p.sh - p.ph, ix0 = ox * p.sw - p.pw;
    for (int ky = 0; ky < p.kh; ++ky) {
        int iy = iy0 + ky * p.dh;
        if (iy < 0 || iy >= p.H) continue;
        for (int kx = 0; kx < p.kw; ++kx) {
            int ix = ix0 + kx * p.dw;
            if (ix < 0 || ix >= p.W) continue;
            const float4 v = ld4(p.in, p.in_fmt, p.in_plane,
                                  (((long long)n * p.H + iy) * p.W + ix) * p.in_ld + p.in_coff + c);
            const float4 w = *reinterpret_cast<const float4*>(p.w + (ky * p.kw + kx) * p.C + c);
            acc.x = fmaf(v.x, w.x, acc.x);
            acc.y = fmaf(v.y, w.y, acc.y);
            acc.z = fmaf(v.z, w.z, acc.z);
            acc.w = fmaf(v.w, w.w, acc.w);
        }
    }
    acc.x = apply_act(acc.x, p.act);
    acc.y = apply_act(acc.y, p.act);
    acc.z = apply_act(acc.z, p.act);
    acc.w = apply_act(acc.w, p.act);
    const long long o = (long long)pix * p.out_ld + p.out_coff;
    if (p.out_cstride == 1) {
        st4(p.out, p.out_fmt, p.out_plane, o + c, acc);
    } else {
        st1(p.out, p.out_fmt, p.out_plane, o + (long long)(c + 0) * p.out_cstride, acc.x);
        st1(p.out, p.out_fmt, p.out_plane, o + (long long)(c + 1) * p.out_cstride, acc.y);
        st1(p.out, p.out_fmt, p.out_plane, o + (long long)(c + 2) * p.out_cstride, acc.z);
        st1(p.out, p.out_fmt, p.out_plane, o + (long long)(c + 3) * p.out_cstride, acc.w);
    }
}


// Register-tiled variant: one thread = PX consecutive output pixels along x, 4 channels.  Each input row
// segment is loaded once and reused by all taps and all PX outputs, which cuts global loads from
// K*K to K*((PX-1)*S+(K-1)*D+1)/PX per output (3x3: 9 -> 4.5, 5x5: 25 -> 10).
template <int K, int S, int D, int PX>
__global__ void __launch_bounds__(128) dwconv_tiled_kernel(const DwK p) {
    constexpr int SPAN = (PX - 1) * S + (K - 1) * D + 1;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;     // 32-bit on purpose: 64-bit div/mod is emulated
    if (i >= (int)p.total) return;
    const int C4 = p.C >> 2;
    const int WoT = p.Wo / PX;
    int c = (i % C4) * 4;
    int r = i / C4;
    int oxb = (r % WoT) * PX;
    int t = r / WoT;
    int oy = t % p.Ho;
    int n = t / p.Ho;
    const float4 bias = *reinterpret_cast<const float4*>(p.bias + c);
    float4 acc[PX];
#pragma unroll
    for (int q = 0; q < PX; ++q) acc[q] = bias;
    const int iy0 = oy * S - p.ph, ix0 = oxb * S - p.pw;
#pragma unroll
    for (int ky = 0; ky < K; ++ky) {
        const int iy = iy0 + ky * D;
        if (iy < 0 || iy >= p.H) continue;
        float4 in[SPAN];
        const long long rowbase = (((long long)n * p.H + iy) * p.W) * p.in_ld + p.in_coff + c;
#pragma unroll
        for (int j = 0; j < SPAN; ++j) {
            // only the columns some tap actually reads (dilated kernels skip every other one)
            bool used = false;
#pragma unroll
            for (int kx = 0; kx < K; ++kx)
#pragma unroll
                for (int q = 0; q < PX; ++q) used |= (q * S + kx * D == j);
            const int ix = ix0 + j;
            in[j] = (used && ix >= 0 && ix < p.W) ? ld4(p.in, p.in_fmt, p.in_plane, rowbase + (long long)ix * p.in_ld)
                                                  : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
            const float4 w = *reinterpret_cast<const float4*>(p.w + (ky * K + kx) * p.C + c);
#pragma unroll
            for (int q = 0; q < PX; ++q) {
                const float4 v = in[q * S + kx * D];
                acc[q].x = fmaf(v.x, w.x, acc[q].x);
                acc[q].y = fmaf(v.y, w.y, acc[q].y);
                acc[q].z = fmaf(v.z, w.z, acc[q].z);
                acc[q].w = fmaf(v.w, w.w, acc[q].w);
            }
        }
    }
    const long long obase = ((((long long)n * p.Ho + oy) * p.Wo) + oxb) * p.out_ld + p.out_coff + c;
#pragma unroll
    for (int q = 0; q < PX; ++q) {
        float4 a = acc[q];
        a.x = apply_act(a.x, p.act); a.y = apply_act(a.y, p.act);
        a.z = apply_act(a.z, p.act); a.w = apply_act(a.w, p.act);
        st4(p.out, p.out_fmt, p.out_plane, obase + (long long)q * p.out_ld, a);
    }
}

template <int K, int S, int D>
static int launch_dw_tiled(DwK k, int batch, cudaStream_t s) {
    constexpr int PX = 4;
    k.total = (long long)batch * k.Ho * (k.Wo / PX) * (k.C / 4);
    dwconv_tiled_kernel<K, S, D, PX><<<blocks_for(k.total, 128), 128, 0, s>>>(k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

int launch_dwconv(const DwArgs& a, cudaStream_t s) {
    DwK k;
    k.in = a.in.base; k.in_ld = a.in.ld; k.in_coff = a.in.c_off; k.H = a.in.H; k.W = a.in.W;
    k.in_fmt = a.in.fmt; k.in_plane = a.in.plane;
    k.out = a.out.base; k.out_ld = a.out.ld; k.out_coff = a.out.c_off; k.out_cstride = a.out.c_stride;
    k.Ho = a.out.H; k.Wo = a.out.W; k.C = a.out.C; k.out_fmt = a.out.fmt; k.out_plane = a.out.plane;
    k.w = a.w; k.bias = a.bias;
    k.kh = a.kh; k.kw = a.kw; k.sh = a.sh; k.sw = a.sw; k.ph = a.ph; k.pw = a.pw; k.dh = a.dh; k.dw = a.dw;
    k.act = a.act;
    SKPS_CHECK(a.in.c_stride == 1 && a.in.C == a.out.C, "dwconv: bad input view");
    SKPS_CHECK(k.C % 4 == 0 && k.in_ld % 4 == 0 && k.in_coff % 4 == 0, "dwconv: C/ld/offset must be multiples of 4");
    SKPS_CHECK(k.out_cstride != 1 || (k.out_ld % 4 == 0 && k.out_coff % 4 == 0), "dwconv: unaligned output view");
    const bool square = a.kh == a.kw && a.sh == a.sw && a.dh == a.dw && a.ph == a.pw;
    if (square && k.out_cstride == 1 && k.Wo % 4 == 0) {
        if (a.kh == 3 && a.sh == 1 && a.dh == 1) return launch_dw_tiled<3, 1, 1>(k, a.batch, s);
        if (a.kh == 3 && a.sh == 2 && a.dh == 1) return launch_dw_tiled<3, 2, 1>(k, a.batch, s);
        if (a.kh == 5 && a.sh == 1 && a.dh == 1) return launch_dw_tiled<5, 1, 1>(k, a.batch, s);
        if (a.kh == 5 && a.sh == 2 && a.dh == 1) return launch_dw_tiled<5, 2, 1>(k, a.batch, s);
        if (a.kh == 5 && a.sh == 1 && a.dh == 2) return launch_dw_tiled<5, 1, 2>(k, a.batch, s);
    }
    k.total = (long long)a.batch * k.Ho * k.Wo * (k.C / 4);
    dwconv_kernel<<<blocks_for(k.total, 256), 256, 0, s>>>(k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}


// ------------------------------------------------------------------------------------------
// Decoder block head (model.py:133-196 DecoderBlock; kps_student.onnx nodes 176-178, 193-195):
//   depthwise3x3( concat( bilinear_x2(low), skip ) )
// computed without ever writing the up-sampled tensor: each thread interpolates the 3x3 high-res
// neighbourhood it needs from a 3x3 low-res patch (half_pixel, align_corners=False), zero outside
// the high-res image (the conv's padding).  One thread = one output pixel x 8 channels.
// ------------------------------------------------------------------------------------------
struct UpcatK {
    const void* low; int low_fmt; long long low_plane; int low_ld, low_coff, Hl, Wl, Cu;
    const void* skip; int skip_fmt; long long skip_plane; int skip_ld, skip_coff;
    void* out; int out_fmt; long long out_plane; int out_ld, out_coff, H, W, C;
    const float* w; const float* bias; int act; long long total;
};

__global__ void __launch_bounds__(128) upcat_dw_kernel(const UpcatK p) {
    // one thread = a 2x2 block of output pixels x 4 channels.  All four outputs share one 3x3 low-res
    // patch, and the 4x4 high-res neighbourhood they read is a fixed-weight (.25/.75) blend of it.
    const int i = blockIdx.x * blockDim.x + threadIdx.x;     // 32-bit on purpose: 64-bit div/mod is emulated
    if (i >= (int)p.total) return;
    const int C4 = p.C >> 2;
    int c = (i % C4) * 4;
    int blk = i / C4;
    const int Wb = p.W >> 1, Hb = p.H >> 1;
    int bx = blk % Wb;
    int t = blk / Wb;
    int by = t % Hb;
    int n = t / Hb;
    const float4 bias = *reinterpret_cast<const float4*>(p.bias + c);
    float4 acc[2][2] = {{bias, bias}, {bias, bias}};
    float4 w[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) w[k] = *reinterpret_cast<const float4*>(p.w + k * p.C + c);
    const int oy0 = by * 2, ox0 = bx * 2;
    if (c >= p.Cu) {
        // skip-connection channels: plain depthwise 3x3 on the 4x4 high-res window
        const int cs = c - p.Cu;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int iy = oy0 - 1 + r;
            if (iy < 0 || iy >= p.H) continue;
            float4 row[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int ix = ox0 - 1 + q;
                row[q] = (ix >= 0 && ix < p.W)
                             ? ld4(p.skip, p.skip_fmt, p.skip_plane,
                                   (((long long)n * p.H + iy) * p.W + ix) * p.skip_ld + p.skip_coff + cs)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int oy = 0; oy < 2; ++oy) {
                const int ky = r - oy;
                if (ky < 0 || ky > 2) continue;
#pragma unroll
                for (int ox = 0; ox < 2; ++ox)
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx) {
                        const float4 v = row[ox + kx], ww = w[ky * 3 + kx];
                        acc[oy][ox].x = fmaf(v.x, ww.x, acc[oy][ox].x);
                        acc[oy][ox].y = fmaf(v.y, ww.y, acc[oy][ox].y);
                        acc[oy][ox].z = fmaf(v.z, ww.z, acc[oy][ox].z);
                        acc[oy][ox].w = fmaf(v.w, ww.w, acc[oy][ox].w);
                    }
            }
        }
    } else {
        // low-res patch rows by-1..by+1, cols bx-1..bx+1 (clamped); high-res col j in 0..3 (x = ox0-1+j):
        //   j=0: .75*L0+.25*L1   j=1: .25*L0+.75*L1   j=2: .75*L1+.25*L2   j=3: .25*L1+.75*L2     (half_pixel x2)
        // columns/rows outside the high-res image are the conv's zero padding
        const float vx0 = ox0 > 0 ? 1.f : 0.f, vx3 = ox0 + 2 < p.W ? 1.f : 0.f;
        const float vy0 = oy0 > 0 ? 1.f : 0.f, vy3 = oy0 + 2 < p.H ? 1.f : 0.f;
        float4 Hh[3][4];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int ly = min(max(by - 1 + r, 0), p.Hl - 1);
            float4 L[3];
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                const int lx = min(max(bx - 1 + q, 0), p.Wl - 1);
                L[q] = ld4(p.low, p.low_fmt, p.low_plane, (((long long)n * p.Hl + ly) * p.Wl + lx) * p.low_ld + p.low_coff + c);
            }
#define BLEND(dst, a, b, wa, wb, m)                                         \
    dst.x = (m) * ((wa) * a.x + (wb) * b.x); dst.y = (m) * ((wa) * a.y + (wb) * b.y); \
    dst.z = (m) * ((wa) * a.z + (wb) * b.z); dst.w = (m) * ((wa) * a.w + (wb) * b.w);
            BLEND(Hh[r][0], L[0], L[1], 0.75f, 0.25f, vx0)
            BLEND(Hh[r][1], L[0], L[1], 0.25f, 0.75f, 1.f)
            BLEND(Hh[r][2], L[1], L[2], 0.75f, 0.25f, 1.f)
            BLEND(Hh[r][3], L[1], L[2], 0.25f, 0.75f, vx3)
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            // high-res row r (y = oy0-1+r) from patch rows: r=0: .75*H0+.25*H1, r=1: .25*H0+.75*H1, r=2: .75*H1+.25*H2, r=3: .25*H1+.75*H2
            const int a = r >> 1;
            const float wa = (r & 1) ? 0.25f : 0.75f, wb = 1.f - wa;
            const float m = r == 0 ? vy0 : (r == 3 ? vy3 : 1.f);
            float4 U[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) { BLEND(U[j], Hh[a][j], Hh[a + 1][j], wa, wb, m) }
#pragma unroll
            for (int oy = 0; oy < 2; ++oy) {
                const int ky = r - oy;
                if (ky < 0 || ky > 2) continue;
#pragma unroll
                for (int ox = 0; ox < 2; ++ox)
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx) {
                        const float4 v = U[ox + kx], ww = w[ky * 3 + kx];
                        acc[oy][ox].x = fmaf(v.x, ww.x, acc[oy][ox].x);
                        acc[oy][ox].y = fmaf(v.y, ww.y, acc[oy][ox].y);
                        acc[oy][ox].z = fmaf(v.z, ww.z, acc[oy][ox].z);
                        acc[oy][ox].w = fmaf(v.w, ww.w, acc[oy][ox].w);
                    }
            }
        }
#undef BLEND
    }
#pragma unroll
    for (int oy = 0; oy < 2; ++oy)
#pragma unroll
        for (int ox = 0; ox < 2; ++ox) {
            float4 v = acc[oy][ox];
            v.x = apply_act(v.x, p.act); v.y = apply_act(v.y, p.act); v.z = apply_act(v.z, p.act); v.w = apply_act(v.w, p.act);
            st4(p.out, p.out_fmt, p.out_plane,
                (((long long)n * p.H + oy0 + oy) * p.W + ox0 + ox) * p.out_ld + p.out_coff + c, v);
        }
}

int launch_upcat_dw(const TView& low, const TView& skip, const TView& out, const float* w, const float* bias, int act,
                    int batch, cudaStream_t s) {
    SKPS_CHECK(out.H == 2 * low.H && out.W == 2 * low.W && skip.H == out.H && skip.W == out.W &&
               out.C == low.C + skip.C, "upcat_dw: shapes");
    SKPS_CHECK(low.c_stride == 1 && skip.c_stride == 1 && out.c_stride == 1 &&
               ((low.C | low.ld | low.c_off | skip.C | skip.ld | skip.c_off | out.ld | out.c_off) & 7) == 0,
               "upcat_dw: views must be unit-stride and 8-channel aligned");
    UpcatK k;
    k.low = low.base; k.low_fmt = low.fmt; k.low_plane = low.plane; k.low_ld = low.ld; k.low_coff = low.c_off;
    k.Hl = low.H; k.Wl = low.W; k.Cu = low.C;
    k.skip = skip.base; k.skip_fmt = skip.fmt; k.skip_plane = skip.plane; k.skip_ld = skip.ld; k.skip_coff = skip.c_off;
    k.out = out.base; k.out_fmt = out.fmt; k.out_plane = out.plane; k.out_ld = out.ld; k.out_coff = out.c_off;
    k.H = out.H; k.W = out.W; k.C = out.C;
    k.w = w; k.bias = bias; k.act = act;
    k.total = (long long)batch * (out.H / 2) * (out.W / 2) * (out.C / 4);
    upcat_dw_kernel<<<blocks_for(k.total, 128), 128, 0, s>>>(k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------
// Generic per-element kernels over (n, y, x, c) of the OUTPUT view.
// ------------------------------------------------------------------------------------------
struct EwK {
    const void* in; int in_ld, in_coff, in_cs, H, W; int in_fmt; long long in_plane;
    void* out; int out_ld, out_coff, out_cs, Ho, Wo, C; int out_fmt; long long out_plane;
    const void* a; const void* b;     // op specific
    int a_ld, a_coff, b_ld, b_coff; int a_fmt, b_fmt; long long a_plane, b_plane;
    int act;
    long long total;
};

#define SRC(off) ld1(p.in, p.in_fmt, p.in_plane, sbase + (off))
template <int MODE>   // 0 maxpool2 ceil, 1 nearest, 2 bilinear2x, 3 copy, 4 affine+act, 5 scse, 6 scale by gate[n,c]
__global__ void __launch_bounds__(256) elementwise_kernel(const EwK p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;     // 32-bit on purpose: 64-bit div/mod is emulated
    if (i >= (int)p.total) return;
    int c = i % p.C;
    int pix = i / p.C;
    int ox = pix % p.Wo;
    int t = pix / p.Wo;
    int oy = t % p.Ho;
    int n = t / p.Ho;
    const long long sbase = (long long)n * p.H * p.W * p.in_ld + p.in_coff + (long long)c * p.in_cs;
    float v;
    if (MODE == 0) {
        // MaxPool 2x2 stride 2, ceil_mode=1, no padding (yolov5n-0.5.onnx node 9)
        int y0 = oy * 2, x0 = ox * 2;
        v = SRC(((long long)y0 * p.W + x0) * p.in_ld);
        if (x0 + 1 < p.W) v = fmaxf(v, SRC(((long long)y0 * p.W + x0 + 1) * p.in_ld));
        if (y0 + 1 < p.H) {
            v = fmaxf(v, SRC(((long long)(y0 + 1) * p.W + x0) * p.in_ld));
            if (x0 + 1 < p.W) v = fmaxf(v, SRC(((long long)(y0 + 1) * p.W + x0 + 1) * p.in_ld));
        }
    } else if (MODE == 1) {
        // Resize nearest, asymmetric, floor: src = floor(dst * in / out)
        int iy = (int)(((long long)oy * p.H) / p.Ho), ix = (int)(((long long)ox * p.W) / p.Wo);
        v = SRC(((long long)iy * p.W + ix) * p.in_ld);
    } else if (MODE == 2) {
        // Resize linear, half_pixel, scale 2 (kps_student.onnx nodes 176, 193)
        float sy = fmaxf((oy + 0.5f) * 0.5f - 0.5f, 0.f), sx = fmaxf((ox + 0.5f) * 0.5f - 0.5f, 0.f);
        int y0 = (int)sy, x0 = (int)sx;
        int y1 = min(y0 + 1, p.H - 1), x1 = min(x0 + 1, p.W - 1);
        float ly = sy - y0, lx = sx - x0;
        float hy = 1.f - ly, hx = 1.f - lx;
        float p00 = SRC(((long long)y0 * p.W + x0) * p.in_ld), p01 = SRC(((long long)y0 * p.W + x1) * p.in_ld);
        float p10 = SRC(((long long)y1 * p.W + x0) * p.in_ld), p11 = SRC(((long long)y1 * p.W + x1) * p.in_ld);
        v = hy * (hx * p00 + lx * p01) + ly * (hx * p10 + lx * p11);
    } else {
        v = SRC(((long long)oy * p.W + ox) * p.in_ld);
        if (MODE == 4) {
            v = apply_act(fmaf(v, ((const float*)p.a)[c], ((const float*)p.b)[c]), p.act);
        } else if (MODE == 5) {
            // scSE (model.py:117-130): x*cSE[n,c] + x*sSE[n,h,w]
            float cs = ld1(p.a, p.a_fmt, p.a_plane, (long long)n * p.a_ld + p.a_coff + c);
            float ss = ld1(p.b, p.b_fmt, p.b_plane,
                           ((long long)n * p.H * p.W + (long long)oy * p.W + ox) * p.b_ld + p.b_coff);
            v = __fadd_rn(__fmul_rn(v, cs), __fmul_rn(v, ss));
        } else if (MODE == 6) {
            // squeeze-excite gate applied ahead of a tensor-core conv: x * gate[n,c]
            v = v * ld1(p.a, p.a_fmt, p.a_plane, (long long)n * p.a_ld + p.a_coff + c);
        }
    }
    st1(p.out, p.out_fmt, p.out_plane, (long long)pix * p.out_ld + p.out_coff + (long long)c * p.out_cs, v);
}
#undef SRC


// 4-channel vector variant of the kernels above (modes 1-6) for unit-stride, 16-byte aligned views.
__device__ __forceinline__ float4 f4_fma(float a, float4 x, float4 y) {
    return make_float4(fmaf(a, x.x, y.x), fmaf(a, x.y, y.y), fmaf(a, x.z, y.z), fmaf(a, x.w, y.w));
}
__device__ __forceinline__ float4 f4_scale(float a, float4 x) { return make_float4(a * x.x, a * x.y, a * x.z, a * x.w); }

template <int MODE>
__global__ void __launch_bounds__(256) elementwise4_kernel(const EwK p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;     // 32-bit on purpose: 64-bit div/mod is emulated
    if (i >= (int)p.total) return;
    const int C4 = p.C >> 2;
    int c = (i % C4) * 4;
    int pix = i / C4;
    int ox = pix % p.Wo;
    int t = pix / p.Wo;
    int oy = t % p.Ho;
    int n = t / p.Ho;
    const long long sbase = (long long)n * p.H * p.W * p.in_ld + p.in_coff + c;
#define SRC4(off) ld4(p.in, p.in_fmt, p.in_plane, sbase + (off))
    float4 v;
    if (MODE == 2) {
        float sy = fmaxf((oy + 0.5f) * 0.5f - 0.5f, 0.f), sx = fmaxf((ox + 0.5f) * 0.5f - 0.5f, 0.f);
        int y0 = (int)sy, x0 = (int)sx;
        int y1 = min(y0 + 1, p.H - 1), x1 = min(x0 + 1, p.W - 1);
        float ly = sy - y0, lx = sx - x0;
        float hy = 1.f - ly, hx = 1.f - lx;
        float4 p00 = SRC4(((long long)y0 * p.W + x0) * p.in_ld), p01 = SRC4(((long long)y0 * p.W + x1) * p.in_ld);
        float4 p10 = SRC4(((long long)y1 * p.W + x0) * p.in_ld), p11 = SRC4(((long long)y1 * p.W + x1) * p.in_ld);
        float4 top = f4_fma(hx, p00, f4_scale(lx, p01)), bot = f4_fma(hx, p10, f4_scale(lx, p11));
        v = f4_fma(hy, top, f4_scale(ly, bot));
    } else if (MODE == 1) {
        // Resize nearest, asymmetric, floor (the ASPP pooled branch broadcasts a 1x1 map)
        const int iy = (int)(((long long)oy * p.H) / p.Ho), ix = (int)(((long long)ox * p.W) / p.Wo);
        v = SRC4(((long long)iy * p.W + ix) * p.in_ld);
    } else {
        v = SRC4(((long long)oy * p.W + ox) * p.in_ld);
        if (MODE == 4) {
            const float4 a = *reinterpret_cast<const float4*>((const float*)p.a + c);
            const float4 b = *reinterpret_cast<const float4*>((const float*)p.b + c);
            v.x = apply_act(fmaf(v.x, a.x, b.x), p.act); v.y = apply_act(fmaf(v.y, a.y, b.y), p.act);
            v.z = apply_act(fmaf(v.z, a.z, b.z), p.act); v.w = apply_act(fmaf(v.w, a.w, b.w), p.act);
        } else if (MODE == 5) {
            const float4 cs = ld4(p.a, p.a_fmt, p.a_plane, (long long)n * p.a_ld + p.a_coff + c);
            const float ss = ld1(p.b, p.b_fmt, p.b_plane,
                                 ((long long)n * p.H * p.W + (long long)oy * p.W + ox) * p.b_ld + p.b_coff);
            v.x = __fadd_rn(__fmul_rn(v.x, cs.x), __fmul_rn(v.x, ss));
            v.y = __fadd_rn(__fmul_rn(v.y, cs.y), __fmul_rn(v.y, ss));
            v.z = __fadd_rn(__fmul_rn(v.z, cs.z), __fmul_rn(v.z, ss));
            v.w = __fadd_rn(__fmul_rn(v.w, cs.w), __fmul_rn(v.w, ss));
        } else if (MODE == 6) {
            const float4 g = ld4(p.a, p.a_fmt, p.a_plane, (long long)n * p.a_ld + p.a_coff + c);
            v.x *= g.x; v.y *= g.y; v.z *= g.z; v.w *= g.w;
        }
    }
#undef SRC4
    st4(p.out, p.out_fmt, p.out_plane, (long long)pix * p.out_ld + p.out_coff + c, v);
}

static bool ew_vec_ok(const EwK& k) {
    return k.C % 4 == 0 && k.in_cs == 1 && k.out_cs == 1 && ((k.in_ld | k.in_coff | k.out_ld | k.out_coff) & 3) == 0 &&
           ((k.a_ld | k.a_coff) & 3) == 0;
}

static EwK make_ew(const TView& in, const TView& out, int batch) {
    EwK k = {};
    k.in = in.base; k.in_ld = in.ld; k.in_coff = in.c_off; k.in_cs = in.c_stride; k.H = in.H; k.W = in.W;
    k.in_fmt = in.fmt; k.in_plane = in.plane;
    k.out = out.base; k.out_ld = out.ld; k.out_coff = out.c_off; k.out_cs = out.c_stride;
    k.Ho = out.H; k.Wo = out.W; k.C = out.C; k.out_fmt = out.fmt; k.out_plane = out.plane;
    k.total = (long long)batch * out.H * out.W * out.C;
    return k;
}

#define LAUNCH_EW(MODE, k, s)                                                     \
    if ((MODE) >= 1 && ew_vec_ok(k)) {                                            \
        (k).total /= 4;                                                           \
        elementwise4_kernel<(MODE) >= 1 ? (MODE) : 2><<<blocks_for((k).total, 256), 256, 0, s>>>(k);   \
    } else {                                                                      \
        elementwise_kernel<MODE><<<blocks_for((k).total, 256), 256, 0, s>>>(k);   \
    }                                                                             \
    SKPS_CUDA(cudaGetLastError());                                                \
    return 0;

int launch_maxpool2(const TView& in, const TView& out, int batch, cudaStream_t s) {
    SKPS_CHECK(in.C == out.C && out.H == (in.H + 1) / 2 && out.W == (in.W + 1) / 2, "maxpool: shape");
    EwK k = make_ew(in, out, batch);
    LAUNCH_EW(0, k, s)
}
int launch_resize_nearest(const TView& in, const TView& out, int batch, cudaStream_t s) {
    SKPS_CHECK(in.C == out.C, "resize: channels");
    EwK k = make_ew(in, out, batch);
    LAUNCH_EW(1, k, s)
}
int launch_bilinear2x(const TView& in, const TView& out, int batch, cudaStream_t s) {
    SKPS_CHECK(in.C == out.C && out.H == 2 * in.H && out.W == 2 * in.W, "bilinear2x: shape");
    EwK k = make_ew(in, out, batch);
    LAUNCH_EW(2, k, s)
}
int launch_copy(const TView& in, const TView& out, int batch, cudaStream_t s) {
    SKPS_CHECK(in.C == out.C && in.H == out.H && in.W == out.W, "copy: shape");
    EwK k = make_ew(in, out, batch);
    LAUNCH_EW(3, k, s)
}
int launch_affine_act(const TView& in, const TView& out, const float* sc, const float* sh, int act, int batch,
                      cudaStream_t s) {
    SKPS_CHECK(in.C == out.C && in.H == out.H && in.W == out.W, "affine: shape");
    EwK k = make_ew(in, out, batch);
    k.a = sc; k.b = sh; k.act = act;
    LAUNCH_EW(4, k, s)
}
int launch_scse(const TView& x, const TView& cse, const TView& sse, const TView& out, int batch, cudaStream_t s) {
    SKPS_CHECK(x.C == out.C && cse.C == x.C && sse.C == 1 && sse.H == x.H && sse.W == x.W, "scse: shape");
    EwK k = make_ew(x, out, batch);
    k.a = cse.base; k.a_ld = cse.ld; k.a_coff = cse.c_off; k.a_fmt = cse.fmt; k.a_plane = cse.plane;
    k.b = sse.base; k.b_ld = sse.ld; k.b_coff = sse.c_off; k.b_fmt = sse.fmt; k.b_plane = sse.plane;
    LAUNCH_EW(5, k, s)
}
int launch_scale_ch(const TView& x, const TView& gate, const TView& out, int batch, cudaStream_t s) {
    SKPS_CHECK(x.C == out.C && gate.C == x.C && x.H == out.H && x.W == out.W, "scale_ch: shape");
    EwK k = make_ew(x, out, batch);
    k.a = gate.base; k.a_ld = gate.ld; k.a_coff = gate.c_off; k.a_fmt = gate.fmt; k.a_plane = gate.plane;
    LAUNCH_EW(6, k, s)
}


// ------------------------------------------------------------------------------------------
// Pointwise (1x1) convolution with few output channels (16 / 24) on CUDA cores: HBM-bound layers
// (student blocks.0.0/conv_pw 16->16 @128^2, blocks.1.*/conv_pwl 64->24 and 72->24 @64^2) where a
// 128 x N tensor-core tile is mostly padding and the per-tile pipeline overhead dominates.
// One thread = PXT pixels x all COUT channels; inputs stream through registers 8 channels at a
// time (one 16-byte load per float16 plane), the weights [ci][co] sit in shared memory and every
// LDS.128 of 4 weights feeds 4*PXT FMAs.  fp32 accumulation in channel order (bias first).
// ------------------------------------------------------------------------------------------
struct PwK {
    const void* in; int in_ld, in_coff, in_fmt; long long in_plane; int Cin;
    void* out; int out_ld, out_coff, out_fmt; long long out_plane;
    const void* res; int res_ld, res_coff, res_fmt; long long res_plane; int res_first;
    const float* w; const float* bias;      // w: [Cout][Cin] (plan layout [Cout][1][1][Cin])
    int act; int npix;
};

template <int COUT, int PXT>
__global__ void __launch_bounds__(128) pw_small_kernel(const PwK p) {
    extern __shared__ __align__(16) float pw_w[];          // [Cin][COUT]
    for (int i = threadIdx.x; i < p.Cin * COUT; i += blockDim.x) {
        const int ci = i / COUT, co = i - ci * COUT;
        pw_w[i] = p.w[co * p.Cin + ci];
    }
    __syncthreads();
    const int pix0 = blockIdx.x * (128 * PXT) + threadIdx.x;     // pixel q of this thread = pix0 + q*128
    float acc[PXT][COUT];
#pragma unroll
    for (int q = 0; q < PXT; ++q)
#pragma unroll
        for (int c = 0; c < COUT; ++c) acc[q][c] = p.bias ? __ldg(p.bias + c) : 0.f;
    for (int ci = 0; ci < p.Cin; ci += 8) {
        float8 x[PXT];
#pragma unroll
        for (int q = 0; q < PXT; ++q) {
            const int pix = min(pix0 + q * 128, p.npix - 1);
            x[q] = ld8(p.in, p.in_fmt, p.in_plane, (long long)pix * p.in_ld + p.in_coff + ci);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float4* wr = reinterpret_cast<const float4*>(pw_w + (ci + j) * COUT);
#pragma unroll
            for (int g = 0; g < COUT / 4; ++g) {
                const float4 w = wr[g];
#pragma unroll
                for (int q = 0; q < PXT; ++q) {
                    const float v = x[q].v[j];
                    acc[q][4 * g + 0] = fmaf(v, w.x, acc[q][4 * g + 0]);
                    acc[q][4 * g + 1] = fmaf(v, w.y, acc[q][4 * g + 1]);
                    acc[q][4 * g + 2] = fmaf(v, w.z, acc[q][4 * g + 2]);
                    acc[q][4 * g + 3] = fmaf(v, w.w, acc[q][4 * g + 3]);
                }
            }
        }
    }
#pragma unroll
    for (int q = 0; q < PXT; ++q) {
        const int pix = pix0 + q * 128;
        if (pix >= p.npix) continue;
#pragma unroll
        for (int g = 0; g < COUT / 8; ++g) {
            float8 o;
            float8 r;
            if (p.res) r = ld8(p.res, p.res_fmt, p.res_plane, (long long)pix * p.res_ld + p.res_coff + 8 * g);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float a = acc[q][8 * g + j];
                const float rr = p.res ? r.v[j] : 0.f;
                o.v[j] = p.res_first ? apply_act(a + rr, p.act) : apply_act(a, p.act) + rr;
            }
            st8(p.out, p.out_fmt, p.out_plane, (long long)pix * p.out_ld + p.out_coff + 8 * g, o);
        }
    }
}

bool pw_small_supported(const ConvArgs& a) {
    if (a.kh != 1 || a.kw != 1 || a.sh != 1 || a.sw != 1 || a.ph || a.pw || a.in_u8 || a.gate.base) return false;
    // only the thinnest layer (16 -> 16) stays on CUDA cores; wider ones run faster on the tensor-core kernel
    if (a.out.C != 16 || a.in.C > 32) return false;
    if (a.in.C % 8 || a.in.c_stride != 1 || a.out.c_stride != 1) return false;
    if ((a.in.ld | a.in.c_off | a.out.ld | a.out.c_off) & 7) return false;
    if (a.res.base && (a.res.c_stride != 1 || ((a.res.ld | a.res.c_off) & 7))) return false;
    if ((long long)a.batch * a.out.H * a.out.W >= (1ll << 31) / 128) return false;
    return a.out.H * a.out.W >= 1024;           // big maps only: small ones are latency-bound either way
}

int launch_pw_small(const ConvArgs& a, cudaStream_t s) {
    PwK k;
    k.in = a.in.base; k.in_ld = a.in.ld; k.in_coff = a.in.c_off; k.in_fmt = a.in.fmt; k.in_plane = a.in.plane; k.Cin = a.in.C;
    k.out = a.out.base; k.out_ld = a.out.ld; k.out_coff = a.out.c_off; k.out_fmt = a.out.fmt; k.out_plane = a.out.plane;
    k.res = a.res.base; k.res_ld = a.res.ld; k.res_coff = a.res.c_off; k.res_fmt = a.res.fmt; k.res_plane = a.res.plane;
    k.res_first = a.res.base ? a.res_first : 0;
    k.w = a.w; k.bias = a.bias; k.act = a.act;
    k.npix = a.batch * a.out.H * a.out.W;
    constexpr int PXT = 2;
    const int blocks = (k.npix + 128 * PXT - 1) / (128 * PXT);
    const size_t smem = (size_t)k.Cin * a.out.C * sizeof(float);
    if (a.out.C == 16) pw_small_kernel<16, PXT><<<blocks, 128, smem, s>>>(k);
    else pw_small_kernel<24, PXT><<<blocks, 128, smem, s>>>(k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------
// N-ary add with fused nearest up-sampling and activation: HRNet fuse layers
// (timm hrnet.py HighResolutionModule.forward: y = sum_j fuse_layers[i][j](x[j]); relu) and any
// residual Add the conv epilogues could not absorb.  Input j is read at (y >> sh_j, x >> sh_j), so
// the nn.Upsample(scale_factor=2^k, mode='nearest') outputs are never written.
// ------------------------------------------------------------------------------------------
struct AddnK {
    const void* in[4]; int ld[4], coff[4], cs[4], sh[4], fmt[4], H[4], W[4]; long long plane[4];
    int n_in;
    void* out; int out_ld, out_coff, out_cs, Ho, Wo, C, out_fmt; long long out_plane;
    int act; long long total;
};

template <bool VEC>
__global__ void __launch_bounds__(256) addn_kernel(const AddnK p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;     // 32-bit on purpose: 64-bit div/mod is emulated
    if (i >= (int)p.total) return;
    const int CG = VEC ? (p.C >> 2) : p.C;
    const int c = VEC ? (i % CG) * 4 : (i % CG);
    const int pix = i / CG;
    const int ox = pix % p.Wo;
    const int t = pix / p.Wo;
    const int oy = t % p.Ho;
    const int n = t / p.Ho;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (j < p.n_in) {
            const long long spix = ((long long)n * p.H[j] + (oy >> p.sh[j])) * p.W[j] + (ox >> p.sh[j]);
            if (VEC) {
                const float4 v = ld4(p.in[j], p.fmt[j], p.plane[j], spix * p.ld[j] + p.coff[j] + c);
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            } else {
                acc.x += ld1(p.in[j], p.fmt[j], p.plane[j], spix * p.ld[j] + p.coff[j] + (long long)c * p.cs[j]);
            }
        }
    }
    if (VEC) {
        acc.x = apply_act(acc.x, p.act); acc.y = apply_act(acc.y, p.act);
        acc.z = apply_act(acc.z, p.act); acc.w = apply_act(acc.w, p.act);
        st4(p.out, p.out_fmt, p.out_plane, (long long)pix * p.out_ld + p.out_coff + c, acc);
    } else {
        st1(p.out, p.out_fmt, p.out_plane, (long long)pix * p.out_ld + p.out_coff + (long long)c * p.out_cs,
            apply_act(acc.x, p.act));
    }
}

int launch_addn(const TView* ins, int n_in, const TView& out, int act, int batch, cudaStream_t s) {
    SKPS_CHECK(n_in >= 2 && n_in <= 4, "addn: %d inputs", n_in);
    AddnK k = {};
    bool vec = out.C % 4 == 0 && out.c_stride == 1 && ((out.ld | out.c_off) & 3) == 0;
    for (int j = 0; j < n_in; ++j) {
        const TView& v = ins[j];
        int sh = 0;
        while ((v.H << sh) < out.H) ++sh;
        SKPS_CHECK(v.C == out.C && (v.H << sh) == out.H && (v.W << sh) == out.W, "addn: input %d shape %dx%dx%d vs %dx%dx%d",
                   j, v.H, v.W, v.C, out.H, out.W, out.C);
        k.in[j] = v.base; k.ld[j] = v.ld; k.coff[j] = v.c_off; k.cs[j] = v.c_stride; k.sh[j] = sh; k.fmt[j] = v.fmt;
        k.H[j] = v.H; k.W[j] = v.W; k.plane[j] = v.plane;
        vec = vec && v.c_stride == 1 && ((v.ld | v.c_off) & 3) == 0;
    }
    k.n_in = n_in;
    k.out = out.base; k.out_ld = out.ld; k.out_coff = out.c_off; k.out_cs = out.c_stride; k.Ho = out.H; k.Wo = out.W;
    k.C = out.C; k.out_fmt = out.fmt; k.out_plane = out.plane; k.act = act;
    k.total = (long long)batch * out.H * out.W * (vec ? out.C / 4 : out.C);
    SKPS_CHECK(k.total < (1ll << 31), "addn: tensor too large for 32-bit indexing");
    if (vec) addn_kernel<true><<<blocks_for(k.total, 256), 256, 0, s>>>(k);
    else addn_kernel<false><<<blocks_for(k.total, 256), 256, 0, s>>>(k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------
// First layer of the networks: 3x3 stride-2 conv on uint8 pixels, 3 -> 16 (student, detector) or 3 -> 64
// (Teacher / HRNet stem) channels (+ act).  One thread = one output pixel x all output channels; weights and the v/255 table live in shared memory.
// (kps_student.onnx node 1, yolov5n-0.5.onnx node 0; /255 as in face_landmark.py:46, face_detector.py:67)
// ------------------------------------------------------------------------------------------
struct StemK {
    const uint8_t* in; int H, W;
    void* out; int out_fmt; long long out_plane; int out_ld, out_coff, Ho, Wo;
    int act; long long total;
};
// Weights travel in the kernel-parameter (constant) bank: with the tap loops fully unrolled every FMA takes its
// weight as a constant operand, so the inner loop has no shared-memory weight traffic (the smem-broadcast version
// was LDS-bound: 108 LDS.128 per 432 FMAs).  [tap*3+ci][co] layout.
template <int CO>
struct StemW { float w[27 * CO]; float b[CO]; };

template <int CO>
__global__ void __launch_bounds__(128) stem_conv_kernel(const StemK p, const __grid_constant__ StemW<CO> W) {
    __shared__ float lut[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = __fdiv_rn((float)i, 255.f);
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;     // 32-bit on purpose: 64-bit div/mod is emulated
    if (i >= (int)p.total) return;
    int ox = i % p.Wo;
    int t = i / p.Wo;
    int oy = t % p.Ho;
    int n = t / p.Ho;
    float acc[CO];
#pragma unroll
    for (int c = 0; c < CO; ++c) acc[c] = 0.f;
    const uint8_t* img = p.in + (long long)n * p.H * p.W * 3;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        const int iy = oy * 2 - 1 + ky;
        if (iy < 0 || iy >= p.H) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int ix = ox * 2 - 1 + kx;
            if (ix < 0 || ix >= p.W) continue;
            const uint8_t* px = img + ((long long)iy * p.W + ix) * 3;
#pragma unroll
            for (int ci = 0; ci < 3; ++ci) {
                const float x = lut[px[ci]];
#pragma unroll
                for (int c = 0; c < CO; ++c) acc[c] = fmaf(x, W.w[((ky * 3 + kx) * 3 + ci) * CO + c], acc[c]);
            }
        }
    }
    const long long o = (long long)i * p.out_ld + p.out_coff;
#pragma unroll
    for (int g = 0; g < CO / 4; ++g) {
        float4 v;
        v.x = apply_act(acc[4 * g + 0] + W.b[4 * g + 0], p.act);
        v.y = apply_act(acc[4 * g + 1] + W.b[4 * g + 1], p.act);
        v.z = apply_act(acc[4 * g + 2] + W.b[4 * g + 2], p.act);
        v.w = apply_act(acc[4 * g + 3] + W.b[4 * g + 3], p.act);
        st4(p.out, p.out_fmt, p.out_plane, o + 4 * g, v);
    }
}

bool stem_conv_supported(const ConvArgs& a) {
    return a.in_u8 && a.in.C == 3 && a.in.ld == 3 && (a.out.C == 16 || a.out.C == 64) && a.kh == 3 && a.kw == 3 && a.sh == 2 && a.sw == 2 &&
           a.ph == 1 && a.pw == 1 && a.dh == 1 && a.dw == 1 && !a.res.base && !a.gate.base && a.bias && a.w_host &&
           a.bias_host &&
           a.out.c_stride == 1 && ((a.out.ld | a.out.c_off) & 3) == 0;
}

template <int CO>
static int launch_stem_t(const StemK& k, const ConvArgs& a, cudaStream_t s) {
    StemW<CO> W;                                  // host copy of [Cout][ky][kx][ci] -> [tap*3+ci][co]
    for (int co = 0; co < CO; ++co) {
        for (int j = 0; j < 27; ++j) W.w[j * CO + co] = a.w_host[co * 27 + j];
        W.b[co] = a.bias_host[co];
    }
    stem_conv_kernel<CO><<<blocks_for(k.total, 128), 128, 0, s>>>(k, W);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

int launch_stem_conv(const ConvArgs& a, cudaStream_t s) {
    StemK k;
    k.in = (const uint8_t*)a.in.base; k.H = a.in.H; k.W = a.in.W;
    k.out = a.out.base; k.out_fmt = a.out.fmt; k.out_plane = a.out.plane; k.out_ld = a.out.ld; k.out_coff = a.out.c_off;
    k.Ho = a.out.H; k.Wo = a.out.W;
    k.act = a.act;
    k.total = (long long)a.batch * k.Ho * k.Wo;
    return a.out.C == 16 ? launch_stem_t<16>(k, a, s) : launch_stem_t<64>(k, a, s);     // 64: Teacher (HRNet) stem
}

// ------------------------------------------------------------------------------------------
// Global average pool: (N,H,W,C) -> (N,1,1,C).  Block = 32 channels x 8 pixel lanes, fixed
// summation order (deterministic).  ReduceMean(2,3) / GlobalAveragePool nodes.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gap_kernel(const void* in, int in_fmt, long long in_plane, int in_ld, int in_coff,
                                                  int HW, int C, float* out, int out_ld, int out_coff) {
    // block = 32 channel quads x 8 pixel lanes; fixed summation order (deterministic)
    __shared__ float4 part[8][33];
    int n = blockIdx.y;
    int c = (blockIdx.x * 32 + threadIdx.x) * 4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < C) {
        const long long sb = (long long)n * HW * in_ld + in_coff + c;
        for (int p = threadIdx.y; p < HW; p += 8) {
            const float4 v = ld4(in, in_fmt, in_plane, sb + (long long)p * in_ld);
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
    }
    part[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float4 v = part[j][threadIdx.x];
            t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
        }
        const float inv = (float)HW;
        *reinterpret_cast<float4*>(out + (long long)n * out_ld + out_coff + c) =
            make_float4(t.x / inv, t.y / inv, t.z / inv, t.w / inv);
    }
}

int launch_gap(const TView& in, const TView& out, int batch, cudaStream_t s) {
    SKPS_CHECK(in.C == out.C && out.H == 1 && out.W == 1 && in.c_stride == 1 && out.c_stride == 1, "gap: shape");
    SKPS_CHECK(out.fmt == DT_F32, "gap: output must be float32");
    SKPS_CHECK(((in.C | in.ld | in.c_off | out.ld | out.c_off) & 3) == 0, "gap: channels/offsets must be multiples of 4");
    dim3 grid((in.C / 4 + 31) / 32, batch), block(32, 8);
    gap_kernel<<<grid, block, 0, s>>>(in.base, in.fmt, in.plane, in.ld, in.c_off, in.H * in.W, in.C,
                                      (float*)out.base, out.ld, out.c_off);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------
// Squeeze-excite gate in one launch (mobilenetv3 SE of the student encoder, kps_student.onnx
// .../se/ReduceMean -> conv_reduce -> Relu -> conv_expand -> HardSigmoid):
//   mean[c]  = (sum over tiles of the depthwise kernel's per-tile channel sums) / (H*W)
//   hid[j]   = act1(b1[j] + sum_c W1[j][c] * mean[c])
//   gate[i]  = act2(b2[i] + sum_j W2[i][j] * hid[j])
// One CTA = 8 samples (they share every weight load); weights are stored transposed ([C][Cr] and [Cr][C]) so the
// threads of a warp read consecutive floats.  Fixed summation order.
// ------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------
// scSE front end (model.py:117-130): ONE pass over x (N,H,W,256) produces the per-tile channel sums the cSE branch needs
// (mean -> FC -> ReLU -> FC -> sigmoid runs in se_fc_kernel) and the sSE map sigmoid(x . w + b).  Before: GlobalAveragePool
// + a 256->1 tensor-core conv + two FC launches, each re-reading x or waiting on the other.
// CTA = 32 pixels x 256 channels: thread = (4-channel group, 8-pixel group).
// ------------------------------------------------------------------------------------------
struct GapSseK {
    const void* x; int x_fmt; long long x_plane; int x_ld, x_coff;
    float* part; int part_ld, part_coff; int tiles;       // [n][tiles][part_ld]
    float* sse; int sse_ld, sse_coff;                     // [n][H*W][sse_ld]
    const float* w; float bias; int act; int HW;
};

__global__ void __launch_bounds__(256) gap_sse_kernel(const GapSseK p) {
    __shared__ float4 s_sum[4][64];
    __shared__ float s_dot[2][GAP_SSE_TILE];
    const int tid = threadIdx.x, cq = tid & 63, pg = tid >> 6;
    const int tile = blockIdx.x, n = blockIdx.y;
    const float4 w4 = *reinterpret_cast<const float4*>(p.w + 4 * cq);
    float4 csum = make_float4(0.f, 0.f, 0.f, 0.f);
    float dot[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const long long pix = (long long)n * p.HW + tile * GAP_SSE_TILE + pg * 8 + i;
        const float4 v = ld4(p.x, p.x_fmt, p.x_plane, pix * p.x_ld + p.x_coff + 4 * cq);
        csum.x += v.x; csum.y += v.y; csum.z += v.z; csum.w += v.w;
        dot[i] = fmaf(v.x, w4.x, fmaf(v.y, w4.y, fmaf(v.z, w4.z, v.w * w4.w)));
    }
    // per-pixel dot products: reduce over the 64 channel groups (two warps per pixel group)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int o = 16; o; o >>= 1) dot[i] += __shfl_xor_sync(0xffffffffu, dot[i], o);
    }
    if ((tid & 31) == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) s_dot[(tid >> 5) & 1][pg * 8 + i] = dot[i];
    }
    s_sum[pg][cq] = csum;
    __syncthreads();
    if (tid < GAP_SSE_TILE) {
        const long long pix = (long long)n * p.HW + tile * GAP_SSE_TILE + tid;
        p.sse[pix * p.sse_ld + p.sse_coff] = apply_act(s_dot[0][tid] + s_dot[1][tid] + p.bias, p.act);
    }
    if (tid < 64) {
        float4 t = s_sum[0][tid];
#pragma unroll
        for (int g = 1; g < 4; ++g) { const float4 u = s_sum[g][tid]; t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w; }
        *reinterpret_cast<float4*>(p.part + ((long long)n * p.tiles + tile) * p.part_ld + p.part_coff + 4 * tid) = t;
    }
}

int launch_gap_sse(const TView& x, const TView& part, const TView& sse, const float* w, float bias, int act, int batch,
                   cudaStream_t s) {
    SKPS_CHECK(x.base && part.base && sse.base && w, "gap_sse: null view");
    SKPS_CHECK(x.C == 256 && x.c_stride == 1 && !((x.ld | x.c_off) & 3) && (x.H * x.W) % GAP_SSE_TILE == 0, "gap_sse: input view");
    SKPS_CHECK(part.fmt == DT_F32 && part.c_stride == 1 && part.C == 256 && !((part.ld | part.c_off) & 3) &&
               part.H * part.W == x.H * x.W / GAP_SSE_TILE, "gap_sse: partial-sum view");
    SKPS_CHECK(sse.fmt == DT_F32 && sse.C == 1 && sse.H == x.H && sse.W == x.W, "gap_sse: sSE view");
    GapSseK k;
    k.x = x.base; k.x_fmt = x.fmt; k.x_plane = x.plane; k.x_ld = x.ld; k.x_coff = x.c_off;
    k.part = (float*)part.base; k.part_ld = part.ld; k.part_coff = part.c_off; k.tiles = part.H * part.W;
    k.sse = (float*)sse.base; k.sse_ld = sse.ld; k.sse_coff = sse.c_off;
    k.w = w; k.bias = bias; k.act = act; k.HW = x.H * x.W;
    gap_sse_kernel<<<dim3(k.tiles, batch), 256, 0, s>>>(k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

constexpr int SE_SAMPLES = 4;
constexpr int SE_THREADS = 1024;
struct SeFcK {
    const float* part; int part_ld, part_coff, tiles; float hw;
    const float* w1t; const float* b1; const float* w2t; const float* b2;    // [C][Cr], [Cr], [Cr][C], [C]
    float* gate; int gate_ld, gate_coff;
    int C, Cr, act1, act2, batch;
    int jp, slices;              // FC1: threads = slices x jp (jp = Cr rounded up to 32); every slice walks C / slices channels
};

// One CTA = 4 samples (they share every weight load), 1024 threads.  FC1 is split over `slices` thread groups that
// each walk a strided share of the C inputs (8 independent weight loads in flight per thread), partials are reduced in
// slice order; FC2: one thread per output channel.  (One serial C-long loop per thread is pure L2 latency.  A thread-block-cluster version - every CTA one eighth of each FC's
// outputs, hidden units exchanged through distributed shared memory - caps 1024-thread CTAs with 32 accumulators per
// thread at 64 registers, too few to keep enough weight loads in flight.)
__global__ void __launch_bounds__(SE_THREADS) se_fc_kernel(const SeFcK p) {
    extern __shared__ __align__(16) float se_smem[];
    float4* mean = reinterpret_cast<float4*>(se_smem);                       // [C]       (x,y,z,w = the 4 samples)
    float4* hid = mean + p.C;                                                // [Cr]
    float4* part1 = hid + p.Cr;                                              // [slices][jp]
    const int n0 = blockIdx.x * SE_SAMPLES;
    for (int i = threadIdx.x; i < p.C * SE_SAMPLES; i += blockDim.x) {
        const int m = i / p.C, c = i - m * p.C;    // consecutive threads -> consecutive channels of one sample
        float sum = 0.f;
        if (n0 + m < p.batch) {
            const float* src = p.part + (long long)(n0 + m) * p.tiles * p.part_ld + p.part_coff + c;
            for (int t = 0; t < p.tiles; ++t) sum += src[(long long)t * p.part_ld];
        }
        se_smem[c * SE_SAMPLES + m] = sum / p.hw;
    }
    __syncthreads();
    {
        const int j = threadIdx.x % p.jp, sl = threadIdx.x / p.jp;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (j < p.Cr && sl < p.slices) {
            const float* wcol = p.w1t + j;
#pragma unroll 8
            for (int c = sl; c < p.C; c += p.slices) {
                const float w = __ldg(wcol + (long long)c * p.Cr);
                const float4 a = mean[c];
                acc.x = fmaf(a.x, w, acc.x); acc.y = fmaf(a.y, w, acc.y); acc.z = fmaf(a.z, w, acc.z); acc.w = fmaf(a.w, w, acc.w);
            }
        }
        if (sl < p.slices) part1[sl * p.jp + j] = acc;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < p.Cr; j += blockDim.x) {
        const float b = p.b1 ? p.b1[j] : 0.f;
        float4 t = make_float4(b, b, b, b);
        for (int sl = 0; sl < p.slices; ++sl) {
            const float4 v = part1[sl * p.jp + j];
            t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
        }
        hid[j] = make_float4(apply_act(t.x, p.act1), apply_act(t.y, p.act1), apply_act(t.z, p.act1), apply_act(t.w, p.act1));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < p.C; i += blockDim.x) {
        const float b = p.b2 ? p.b2[i] : 0.f;
        float4 acc = make_float4(b, b, b, b);
        const float* wcol = p.w2t + i;
#pragma unroll 8
        for (int j = 0; j < p.Cr; ++j) {
            const float w = __ldg(wcol + (long long)j * p.C);
            const float4 a = hid[j];
            acc.x = fmaf(a.x, w, acc.x); acc.y = fmaf(a.y, w, acc.y); acc.z = fmaf(a.z, w, acc.z); acc.w = fmaf(a.w, w, acc.w);
        }
        const float g[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
        for (int m = 0; m < SE_SAMPLES; ++m)
            if (n0 + m < p.batch) p.gate[(long long)(n0 + m) * p.gate_ld + p.gate_coff + i] = apply_act(g[m], p.act2);
    }
}

int launch_se_fc(const TView& part, const TView& gate, const float* w1t, const float* b1, const float* w2t, const float* b2,
                 int Cr, int act1, int act2, int hw, int batch, cudaStream_t s) {
    SKPS_CHECK(part.fmt == DT_F32 && gate.fmt == DT_F32 && part.c_stride == 1 && gate.c_stride == 1 && part.C == gate.C &&
               gate.H * gate.W == 1, "se_fc: views");
    SeFcK k;
    k.part = (const float*)part.base; k.part_ld = part.ld; k.part_coff = part.c_off; k.tiles = part.H * part.W; k.hw = (float)hw;
    k.w1t = w1t; k.b1 = b1; k.w2t = w2t; k.b2 = b2;
    k.gate = (float*)gate.base; k.gate_ld = gate.ld; k.gate_coff = gate.c_off;
    k.C = part.C; k.Cr = Cr; k.act1 = act1; k.act2 = act2; k.batch = batch;
    k.jp = (Cr + 31) / 32 * 32;
    k.slices = SE_THREADS / k.jp;
    SKPS_CHECK(k.slices >= 1, "se_fc: %d hidden channels", Cr);
    if (k.slices > 32) k.slices = 32;
    const size_t smem = (size_t)(k.C + k.Cr + k.slices * k.jp) * SE_SAMPLES * sizeof(float);
    static int attr_bytes[MAX_DEVICES] = {};
    if (smem_limit((const void*)se_fc_kernel, attr_bytes, 96 * 1024)) return 1;
    SKPS_CHECK(smem <= 96 * 1024, "se_fc: %d + %d channels do not fit shared memory", k.C, k.Cr);
    se_fc_kernel<<<(batch + SE_SAMPLES - 1) / SE_SAMPLES, SE_THREADS, smem, s>>>(k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------
// yolov5-face Detect decode (yolov5n-0.5.onnx nodes 502-820): three head tensors (N,H,W,48) ->
// (N, rows, 16) = [cx,cy,w,h,obj, 5x(lx,ly), cls], rows ordered scale, anchor, y, x.
// consts: per scale [stride, aw0,ah0, aw1,ah1, aw2,ah2].
// ------------------------------------------------------------------------------------------
struct DetK {
    const float* head[3]; int ld[3], coff[3], H[3], W[3];
    float consts[21];
    float* out; int rows; long long total;
};

__global__ void __launch_bounds__(256) det_decode_kernel(const DetK p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;     // 32-bit on purpose: 64-bit div/mod is emulated
    if (i >= (int)p.total) return;
    int row = (int)(i % p.rows);
    int n = (int)(i / p.rows);
    int si = 0, r = row;
    {
        int c0 = 3 * p.H[0] * p.W[0];
        if (r >= c0) {
            r -= c0; si = 1;
            int c1 = 3 * p.H[1] * p.W[1];
            if (r >= c1) { r -= c1; si = 2; }
        }
    }
    const int H = p.H[si], W = p.W[si];
    int x = r % W;
    int t = r / W;
    int y = t % H;
    int a = t / H;
    const float stride = p.consts[si * 7];
    const float aw = p.consts[si * 7 + 1 + 2 * a], ah = p.consts[si * 7 + 2 + 2 * a];
    const float* src = p.head[si] + (((long long)n * H + y) * W + x) * p.ld[si] + p.coff[si] + a * 16;
    float v[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) v[k] = src[k];
    float o[16];
    const float gx = (float)x, gy = (float)y;
    float s0 = sigmoid_f(v[0]), s1 = sigmoid_f(v[1]), s2 = sigmoid_f(v[2]), s3 = sigmoid_f(v[3]);
    o[0] = __fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(s0, 2.f), -0.5f), gx), stride);
    o[1] = __fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(s1, 2.f), -0.5f), gy), stride);
    float w2 = __fmul_rn(s2, 2.f), h2 = __fmul_rn(s3, 2.f);
    o[2] = __fmul_rn(__fmul_rn(w2, w2), aw);
    o[3] = __fmul_rn(__fmul_rn(h2, h2), ah);
    o[4] = sigmoid_f(v[4]);
    const float gxs = __fmul_rn(gx, stride), gys = __fmul_rn(gy, stride);
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        o[5 + 2 * k] = __fadd_rn(__fmul_rn(v[5 + 2 * k], aw), gxs);
        o[6 + 2 * k] = __fadd_rn(__fmul_rn(v[6 + 2 * k], ah), gys);
    }
    o[15] = sigmoid_f(v[15]);
    float4* dst = reinterpret_cast<float4*>(p.out + i * 16);
    dst[0] = make_float4(o[0], o[1], o[2], o[3]);
    dst[1] = make_float4(o[4], o[5], o[6], o[7]);
    dst[2] = make_float4(o[8], o[9], o[10], o[11]);
    dst[3] = make_float4(o[12], o[13], o[14], o[15]);
}

int launch_det_decode(const TView* heads, const float* consts, const TView& out, int rows, int batch,
                      cudaStream_t s) {
    DetK k;
    int total_rows = 0;
    for (int i = 0; i < 3; ++i) {
        SKPS_CHECK(heads[i].C == 48 && heads[i].c_stride == 1, "det_decode: head view");
        k.head[i] = (const float*)heads[i].base; k.ld[i] = heads[i].ld; k.coff[i] = heads[i].c_off;
        k.H[i] = heads[i].H; k.W[i] = heads[i].W;
        total_rows += 3 * heads[i].H * heads[i].W;
    }
    SKPS_CHECK(total_rows == rows && out.ld == 16 && out.c_off == 0, "det_decode: rows %d vs %d", total_rows, rows);
    for (int i = 0; i < 21; ++i) k.consts[i] = consts[i];
    k.out = (float*)out.base; k.rows = rows; k.total = (long long)batch * rows;
    det_decode_kernel<<<blocks_for(k.total, 256), 256, 0, s>>>(k);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------
// Heat-map decode (kps_student.onnx nodes 201-410; TRAIN/.../model.py:511-554): per landmark c
// arg-max over H*W of hm[:, c] (first maximum), score = max, x = (i%W + hm[:,P+c][i]) / W,
// y = (i/W + hm[:,2P+c][i]) / W.  Block = one sample; 128 channel lanes x 8 position groups.
// ------------------------------------------------------------------------------------------
struct HmOff {          // split head: offsets = rows P..3P of the 1x1 head conv, evaluated at the arg-max pixel only
    const void* feat; int fmt, ld, coff, K; long long plane;     // the head conv's input (N,H,W,K)
    const float* w; const float* b;                              // [2P][K], [2P]
};

struct HmPart {         // per-tile (max, first arg-max) written by the head conv's epilogue (conv_tc.cu): [n][tiles][ld]
    const float* val; const int* idx; int tiles, ld;
};

__global__ void __launch_bounds__(1024) hm_decode_kernel(const float* hm, int ld, int coff, int H, int W, int P,
                                                         float* xy, int xy_ld, float* score, int sc_ld, const HmOff off,
                                                         const HmPart part) {
    __shared__ float sv[8][128];
    __shared__ int si[8][128];
    const int n = blockIdx.x;
    const int c = threadIdx.x, g = threadIdx.y;
    const int HW = H * W;
    const float* base = hm + (long long)n * HW * ld + coff;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    if (part.val) {
        // tiles are in ascending pixel order and each holds its own first maximum: strict > keeps the first one overall
        if (c < P) {
            const int per = (part.tiles + 7) / 8, t0 = g * per, t1 = min(part.tiles, t0 + per);
            for (int t = t0; t < t1; ++t) {
                const long long o = ((long long)n * part.tiles + t) * part.ld + c;
                const float v = part.val[o];
                if (bi == 0x7fffffff || v > best) { best = v; bi = part.idx[o]; }
            }
        }
    } else if (c < P) {
        int per = (HW + 7) / 8;
        int p0 = g * per, p1 = min(HW, p0 + per);
        for (int p = p0; p < p1; ++p) {
            float v = base[(long long)p * ld + c];
            if (bi == 0x7fffffff || v > best) { best = v; bi = p; }   // ascending p: first maximum wins
        }
    }
    sv[g][c] = best;
    si[g][c] = bi;
    __syncthreads();
    if (g == 0 && c < P) {
        for (int j = 1; j < 8; ++j) {
            float v = sv[j][c];
            int idx = si[j][c];
            if (idx != 0x7fffffff && (v > best || (v == best && idx < bi))) { best = v; bi = idx; }
        }
        si[0][c] = bi;
    }
    if (off.feat) {
        // split head: every position group takes one eighth of the K-long dot products at the arg-max pixel; the eight
        // partial sums are added in group order
        __syncthreads();
        float px = 0.f, py = 0.f;
        if (c < P) {
            const int am = si[0][c];
            const int kper = ((off.K + 31) / 32) * 4, k0 = g * kper, k1 = min(off.K, k0 + kper);
            const long long fe = ((long long)n * HW + am) * off.ld + off.coff;
            const float* wx = off.w + (long long)c * off.K;
            const float* wy = off.w + (long long)(P + c) * off.K;
            for (int k = k0; k < k1; k += 4) {
                const float4 a = ld4(off.feat, off.fmt, off.plane, fe + k);
                const float4 u = __ldg(reinterpret_cast<const float4*>(wx + k));
                const float4 v = __ldg(reinterpret_cast<const float4*>(wy + k));
                px = fmaf(a.x, u.x, px); px = fmaf(a.y, u.y, px); px = fmaf(a.z, u.z, px); px = fmaf(a.w, u.w, px);
                py = fmaf(a.x, v.x, py); py = fmaf(a.y, v.y, py); py = fmaf(a.z, v.z, py); py = fmaf(a.w, v.w, py);
            }
        }
        __syncthreads();                 // all groups have read the arg-max before sv/si are reused
        sv[g][c] = px;
        reinterpret_cast<float*>(si)[g * 128 + c] = py;
        __syncthreads();
    }
    if (g == 0 && c < P) {
        float ox, oy;
        if (off.feat) {
            ox = off.b[c]; oy = off.b[P + c];
            for (int j = 0; j < 8; ++j) { ox += sv[j][c]; oy += reinterpret_cast<float*>(si)[j * 128 + c]; }
        } else {
            ox = base[(long long)bi * ld + P + c];
            oy = base[(long long)bi * ld + 2 * P + c];
        }
        float x = __fdiv_rn(__fadd_rn((float)(bi % W), ox), (float)W);
        float y = __fdiv_rn(__fadd_rn((float)(bi / W), oy), (float)W);
        xy[(long long)n * xy_ld + 2 * c] = x;
        xy[(long long)n * xy_ld + 2 * c + 1] = y;
        score[(long long)n * sc_ld + c] = best;
    }
}

int launch_hm_decode(const TView& hm, const TView& feat, const float* w_off, const float* b_off, const TView& xy,
                     const TView& score, int npts, int batch, cudaStream_t s, const TView* part) {
    SKPS_CHECK((hm.C == 3 * npts || (hm.C == npts && feat.base)) && npts <= 128 && hm.c_stride == 1 && hm.H == hm.W &&
               hm.fmt == DT_F32, "hm_decode: shape/format");
    HmPart hp = {};
    if (part && part->base) {
        // partial rows: [tiles][2 * ld] float32 per sample = ld maxima then ld arg-max indices (int32 bits)
        SKPS_CHECK(feat.base && part->fmt == DT_F32 && part->c_stride == 1 && part->c_off == 0 && (part->ld & 1) == 0 &&
                   part->ld / 2 >= npts, "hm_decode: partial-maximum view");
        hp.val = (const float*)part->base; hp.idx = (const int*)part->base + part->ld / 2;
        hp.tiles = part->H * part->W; hp.ld = part->ld;
    }
    HmOff off = {};
    if (feat.base) {
        SKPS_CHECK(w_off && b_off && feat.c_stride == 1 && feat.H == hm.H && feat.W == hm.W &&
                   ((feat.C | feat.ld | feat.c_off) & 3) == 0, "hm_decode: offset-head input view");
        off.feat = feat.base; off.fmt = feat.fmt; off.ld = feat.ld; off.coff = feat.c_off; off.K = feat.C; off.plane = feat.plane;
        off.w = w_off; off.b = b_off;
    }
    dim3 block(128, 8);
    hm_decode_kernel<<<batch, block, 0, s>>>((const float*)hm.base, hm.ld, hm.c_off, hm.H, hm.W, npts,
                                             (float*)xy.base, xy.ld, (float*)score.base, score.ld, off, hp);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace skps
