// Unit-test entry points for the fused kernels that otherwise only run inside a whole network: the squeeze-excite gate
// (se_fc_kernel), the heat-map decode (hm_decode_kernel) and the fused producer -> 1x1 conv layers (conv_xf.cu,
// conv_fpw.cu), host float32 in/out; and for the temporal step of the multi-stream pipeline (temporal.cu) on device
// buffers the caller owns.
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_fpw.h"
#include "conv_xf.h"
#include "mpipe_kernels.h"

using namespace skps;

namespace {
struct DBuf {
    void* p = nullptr;
    ~DBuf() { if (p) cudaFree(p); }
    int put(const void* src, size_t bytes) {
        if (cudaMalloc(&p, bytes ? bytes : 16) != cudaSuccess) return 1;
        if (src && cudaMemcpy(p, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) return 1;
        return 0;
    }
};
TView mk(void* base, int C, int H, int W, int ld = 0, int fmt = DT_F32, long long plane = 0) {
    TView t;
    memset(&t, 0, sizeof(t));
    t.base = base; t.ld = ld ? ld : C; t.c_off = 0; t.c_stride = 1; t.C = C; t.H = H; t.W = W;
    t.sample = (long long)t.ld * H * W; t.fmt = fmt; t.plane = plane;
    return t;
}
__global__ void f32_to_split(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = src[i];
    const __half h = __float2half_rn(v);
    hi[i] = h;
    lo[i] = __float2half_rn(v - __half2float(h));
}

// One fused layer on host data through conv_fpw (fpw) or conv_xf, on images [0, batch) of buffers sized for N.  `out` comes
// in as well as out (through the split-fp16 planes when out_split != 0), so that what the kernel leaves unwritten comes
// back as it went in.
int debug_conv_fused(bool fpw, int mode, const float* x, int N, int H, int W, int Cx, int x_split, const float* low, int Cl,
                     const float* gate, const float* dww, int dw_act, const void* w_hi, const void* w_lo, const float* bias,
                     int Cout, int act, int n_tile, float out_scale, const float* residual, int res_first, int out_split,
                     float* out, const float* weff, int batch) {
    SKPS_CHECK(x && w_hi && w_lo && out && N > 0 && batch > 0 && batch <= N, "debug_conv_fused: bad argument");
    SKPS_CHECK(!low || (weff && Cl % 32 == 0), "debug_conv_fused: class weights");
    const int K = Cx + (low ? Cl : 0), Kpad = (K + 63) / 64 * 64;
    const long long nx = (long long)N * H * W * Cx, nl = low ? (long long)N * (H / 2) * (W / 2) * Cl : 0;
    const long long nout = (long long)N * H * W * Cout;
    const bool xs = x_split || mode == XF_SCALE;
    DBuf dx, dxs, dl, dg, dw, dwh, dwl, db, dr, dout, dwe;
    SKPS_CHECK(!dx.put(x, nx * 4) && !dxs.put(nullptr, nx * 4) && !dl.put(low, nl * 4) && !dg.put(gate, (size_t)N * Cx * 4) &&
               !dw.put(dww, (size_t)10 * Kpad * 4) && !dwh.put(w_hi, (size_t)n_tile * Kpad * 2) &&
               !dwl.put(w_lo, (size_t)n_tile * Kpad * 2) && !db.put(bias, (size_t)Cout * 4) && !dr.put(residual, nout * 4) &&
               !dout.put(nullptr, nout * 4 * (out_split ? 2 : 1)) && !dwe.put(weff, low ? (size_t)Cl * 144 * 4 : 0),
               "debug_conv_fused: cudaMalloc/copy failed");
    SKPS_CUDA(cudaMemcpy(dout.p, out, nout * 4, cudaMemcpyHostToDevice));
    if (xs) {
        f32_to_split<<<(unsigned)((nx + 255) / 256), 256>>>((const float*)dx.p, (__half*)dxs.p, (__half*)dxs.p + nx, nx);
        SKPS_CUDA(cudaGetLastError());
    }
    // the output's initial contents: float32, or split into the hi/lo planes
    void* obase = dout.p;
    if (out_split) {
        obase = (float*)dout.p + nout;
        f32_to_split<<<(unsigned)((nout + 255) / 256), 256>>>((const float*)dout.p, (__half*)obase, (__half*)obase + nout, nout);
        SKPS_CUDA(cudaGetLastError());
    }
    XfSetup s;
    memset(&s, 0, sizeof(s));
    s.mode = mode; s.max_batch = N;
    s.x = xs ? mk(dxs.p, Cx, H, W, 0, DT_SPLIT16, nx) : mk(dx.p, Cx, H, W);
    if (low) s.low = mk(dl.p, Cl, H / 2, W / 2);
    if (gate) s.gate = mk(dg.p, Cx, 1, 1);
    s.dww = (const float*)dw.p; s.dw_act = dw_act; s.weff = low ? (const float*)dwe.p : nullptr;
    s.Cout = Cout; s.act = act; s.n_tile = n_tile; s.n_tiles = 1; s.out_scale = out_scale;
    s.w_hi = dwh.p; s.w_lo = dwl.p; s.bias = bias ? (const float*)db.p : nullptr;
    s.out = mk(obase, Cout, H, W, 0, out_split ? DT_SPLIT16 : DT_F32, nout);
    if (residual) s.res = mk(dr.p, Cout, H, W);
    s.res_first = res_first;
    if (fpw) {
        FpwLayer L;
        if (fpw_prepare(L, s) || fpw_launch(L, batch, sm_count(), 0)) return 1;
    } else {
        XfLayer L;
        if (xf_prepare(L, s) || xf_launch(L, batch, sm_count(), 0)) return 1;
    }
    SKPS_CUDA(cudaDeviceSynchronize());
    if (out_split) {
        __half* tmp = (__half*)malloc(nout * 4);
        SKPS_CHECK(tmp, "debug_conv_fused: host allocation failed");
        SKPS_CUDA(cudaMemcpy(tmp, obase, nout * 4, cudaMemcpyDeviceToHost));
        for (long long i = 0; i < nout; ++i) out[i] = __half2float(tmp[i]) + __half2float(tmp[nout + i]);
        free(tmp);
    } else {
        SKPS_CUDA(cudaMemcpy(out, dout.p, nout * 4, cudaMemcpyDeviceToHost));
    }
    return 0;
}
}  // namespace

// gate[n][c] = act2(W2 * act1(W1 * (sum_tiles part[n][t][c] / hw) + b1) + b2): the squeeze-excite branch of a
// MobileNetV3 block (kps_student.onnx .../se/conv_reduce, conv_expand; timm SqueezeExcite).  w1t [C][Cr], w2t [Cr][C].
extern "C" SKPS_API int skps_debug_se_fc(const float* part, int N, int tiles, int C, const float* w1t, const float* b1,
                                         const float* w2t, const float* b2, int Cr, int act1, int act2, int hw,
                                         float* gate) {
    SKPS_CHECK(part && w1t && b1 && w2t && b2 && gate, "debug_se_fc: null argument");
    DBuf dp, dw1, db, dw2, dg;
    std::string bb((size_t)(Cr + C) * 4, '\0');
    memcpy(&bb[0], b1, (size_t)Cr * 4);
    memcpy(&bb[(size_t)Cr * 4], b2, (size_t)C * 4);
    SKPS_CHECK(!dp.put(part, (size_t)N * tiles * C * 4) && !dw1.put(w1t, (size_t)C * Cr * 4) && !db.put(bb.data(), bb.size()) &&
               !dw2.put(w2t, (size_t)C * Cr * 4) && !dg.put(nullptr, (size_t)N * C * 4), "debug_se_fc: cudaMalloc/copy failed");
    TView pv = mk(dp.p, C, tiles, 1), gv = mk(dg.p, C, 1, 1);
    if (launch_se_fc(pv, gv, (const float*)dw1.p, (const float*)db.p, (const float*)dw2.p, (const float*)db.p + Cr, Cr, act1,
                     act2, hw, N, 0))
        return 1;
    SKPS_CUDA(cudaDeviceSynchronize());
    SKPS_CUDA(cudaMemcpy(gate, dg.p, (size_t)N * C * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// Heat-map decode (model.py:511-554 postp): per landmark arg-max over H*W (first index on ties), score = the maximum,
// (x, y) = (argmax position + offset) / W.  hm (N,H,W,ld) holds npts score maps [and 2*npts offset maps when feat is
// null]; with feat (N,H,W,K) the offsets are w_off (2*npts,K) . feat[argmax] + b_off.
extern "C" SKPS_API int skps_debug_hm_decode(const float* hm, int N, int H, int W, int ld, int npts, const float* feat, int K,
                                             const float* w_off, const float* b_off, float* xy, float* score) {
    SKPS_CHECK(hm && xy && score, "debug_hm_decode: null argument");
    DBuf dh, df, dw, db, dx, ds;
    SKPS_CHECK(!dh.put(hm, (size_t)N * H * W * ld * 4) && !dx.put(nullptr, (size_t)N * 2 * npts * 4) &&
               !ds.put(nullptr, (size_t)N * npts * 4), "debug_hm_decode: cudaMalloc/copy failed");
    TView hv = mk(dh.p, feat ? npts : 3 * npts, H, W, ld), fv;
    memset(&fv, 0, sizeof(fv));
    if (feat) {
        SKPS_CHECK(!df.put(feat, (size_t)N * H * W * K * 4) && !dw.put(w_off, (size_t)2 * npts * K * 4) &&
                   !db.put(b_off, (size_t)2 * npts * 4), "debug_hm_decode: cudaMalloc/copy failed");
        fv = mk(df.p, K, H, W);
    }
    TView xv = mk(dx.p, 2 * npts, 1, 1), sv = mk(ds.p, npts, 1, 1);
    if (launch_hm_decode(hv, fv, (const float*)dw.p, (const float*)db.p, xv, sv, npts, N, 0)) return 1;
    SKPS_CUDA(cudaDeviceSynchronize());
    SKPS_CUDA(cudaMemcpy(xy, dx.p, (size_t)N * 2 * npts * 4, cudaMemcpyDeviceToHost));
    SKPS_CUDA(cudaMemcpy(score, ds.p, (size_t)N * npts * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// One fused layer through conv_xf on host data (tests/test_conv_xf_gpu.py).
//   mode 0 (XF_SCALE): out = act(conv1x1(x * gate[n,c]) ...)            x (N,H,W,Cx) float32, gate (N,Cx)
//   mode 1 (XF_DW)   : out = act(conv1x1(dw_act(dw3x3(concat(up2(low), x)))))   low (N,H/2,W/2,Cl) or null
//   x_split: the kernel reads x as fp16 hi/lo planes (else float32; XF_SCALE always splits)
//   dww: [9][Kpad] depthwise weights then [Kpad] bias, Kpad = ceil((Cl+Cx)/64)*64 (XF_DW)
//   w_hi/w_lo: (n_tile, Kpad) float16 as packed by plan.pack_tc_weights; residual (N,H,W,Cout) float32 or null
//   weff: [Cl/32][4][4][9][32] class weights of the up-sampled channels (plan.pack_upcat_class_weights), null without low
//   out: (N,H,W,Cout); elements the kernel leaves unwritten come back as they went in
extern "C" SKPS_API int skps_debug_conv_xf(int mode, const float* x, int N, int H, int W, int Cx, int x_split,
                                           const float* low, int Cl, const float* gate, const float* dww, int dw_act,
                                           const void* w_hi, const void* w_lo, const float* bias, int Cout, int act,
                                           int n_tile, float out_scale, const float* residual, int res_first,
                                           int out_split, float* out, const float* weff) {
    return debug_conv_fused(false, mode, x, N, H, W, Cx, x_split, low, Cl, gate, dww, dw_act, w_hi, w_lo, bias, Cout, act,
                            n_tile, out_scale, residual, res_first, out_split, out, weff, N);
}

// One launch of the temporal step of skps_mpipe_submit (mp_temporal_kernel) for streams [0, n_streams), with the constants
// skps_mpipe_submit derives from the cfg and the state in the caller's device buffers (MpTemporalArgs layouts).
extern "C" SKPS_API int skps_debug_mp_temporal(const skps_pipeline_cfg* cfg, int n_streams, int top_k, int n_points,
                                               const float* kps_now, const int32_t* count, const int32_t* flag,
                                               const int32_t* hw, const float* boxes4, const int32_t* src, double* prev_lm,
                                               double* prev_dx, int32_t* n_prev, int32_t* prev_f32, int32_t* state_idx,
                                               double* track_box, float* track_f32, int32_t* n_track, int64_t* ids,
                                               int64_t* next_id, double* out_kps, void* stream) {
    return skps_debug_mp_temporal_mem(cfg, n_streams, top_k, n_points, kps_now, count, flag, hw, boxes4, src, prev_lm, prev_dx,
                                      n_prev, prev_f32, state_idx, track_box, track_f32, n_track, ids, next_id, out_kps, 0,
                                      nullptr, nullptr, nullptr, nullptr, stream);
}

// The same launch with the id memory of skps_mpipe_set_id_memory: id_memory frames, and the memory state in the caller's
// device buffers (needed when id_memory > 0).
extern "C" SKPS_API int skps_debug_mp_temporal_mem(const skps_pipeline_cfg* cfg, int n_streams, int top_k, int n_points,
                                                   const float* kps_now, const int32_t* count, const int32_t* flag,
                                                   const int32_t* hw, const float* boxes4, const int32_t* src,
                                                   double* prev_lm, double* prev_dx, int32_t* n_prev, int32_t* prev_f32,
                                                   int32_t* state_idx, double* track_box, float* track_f32, int32_t* n_track,
                                                   int64_t* ids, int64_t* next_id, double* out_kps, int id_memory,
                                                   int64_t* mem_ids, float* mem_box, int32_t* mem_gap, int32_t* mem_n,
                                                   void* stream) {
    SKPS_CHECK(cfg && kps_now && count && flag && hw && boxes4 && src && prev_lm && prev_dx && n_prev && prev_f32 &&
               state_idx && track_box && track_f32 && n_track && ids && next_id && out_kps, "debug_mp_temporal: null argument");
    SKPS_CHECK(top_k > 0 && top_k <= 64, "debug_mp_temporal: top_k %d outside 1..64", top_k);
    SKPS_CHECK(n_streams > 0 && n_points > 0, "debug_mp_temporal: %d streams of %d points", n_streams, n_points);
    SKPS_CHECK(id_memory >= 0, "debug_mp_temporal: id_memory %d is not >= 0", id_memory);
    SKPS_CHECK(!id_memory || (mem_ids && mem_box && mem_gap && mem_n), "debug_mp_temporal: id memory on with a null buffer");
    MpTemporalArgs a = {};
    a.top_k = top_k; a.n_points = n_points;
    a.kps_now = kps_now; a.count = count; a.flag = flag; a.hw = hw; a.boxes4 = boxes4;
    a.prev_lm = prev_lm; a.prev_dx = prev_dx; a.n_prev = n_prev; a.prev_f32 = prev_f32; a.state_idx = state_idx;
    a.track_box = track_box; a.track_f32 = track_f32; a.n_track = n_track; a.src = src; a.ids = ids; a.next_id = next_id;
    a.id_memory = id_memory; a.mem_ids = mem_ids; a.mem_box = mem_box; a.mem_gap = mem_gap; a.mem_n = mem_n;
    a.out_kps = out_kps;
    mp_temporal_constants(*cfg, a);
    return launch_mp_temporal(a, n_streams, (cudaStream_t)stream);
}

// One fused layer through conv_fpw on host data (tests/test_conv_fpw_gpu.py).  The arguments of skps_debug_conv_xf, then
// `batch` <= N: the kernel runs images [0, batch) of buffers sized for N, so that images past the batch can be checked to
// come back as they went in.  Fails for a layer conv_fpw does not take.
extern "C" SKPS_API int skps_debug_conv_fpw(int mode, const float* x, int N, int H, int W, int Cx, int x_split,
                                            const float* low, int Cl, const float* gate, const float* dww, int dw_act,
                                            const void* w_hi, const void* w_lo, const float* bias, int Cout, int act,
                                            int n_tile, float out_scale, const float* residual, int res_first,
                                            int out_split, float* out, const float* weff, int batch) {
    return debug_conv_fused(true, mode, x, N, H, W, Cx, x_split, low, Cl, gate, dww, dw_act, w_hi, w_lo, bias, Cout, act,
                            n_tile, out_scale, residual, res_first, out_split, out, weff, batch);
}
