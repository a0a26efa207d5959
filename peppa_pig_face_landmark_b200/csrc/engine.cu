// skps_engine: runs one lowered network plan (peppa_pig_face_landmark_b200/plan.py) on one GPU.
// Stands where onnxruntime.InferenceSession stands in the reference
// (Skps/core/api/onnx_model_base.py:14,23).  Owns the packed weights and all activation buffers
// (sized for max_batch at creation: no allocation on the forward path); the op sequence for a
// given batch size is captured once into a CUDA graph and replayed.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <variant>
#include <vector>

#include "../../include/skps_b200.h"
#include "common.h"
#include "conv_mma.h"
#include "conv_hm.h"
#include "conv_pw.h"
#include "conv_tc.h"
#include "conv_tct.h"
#include "conv_fpw.h"
#include "conv_xf.h"
#include "dw_tma.h"
#include "mpipe_kernels.h"
#include "stem_block.h"

namespace skps {

static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* get_error() { return g_err; }

}  // namespace skps

using namespace skps;

// The kernel one plan op runs, chosen once at engine creation (prepare_op), and the layer prepared for it.  run_ops,
// skps_engine_op_kernel, skps_engine_op_grid and skps_engine_launches_for_batch all read this record.  MISC, SIMT_CONV,
// DW and UPCAT hold no layer: their arguments are built from the OpDesc at every launch, because f32 mode
// (skps_engine_forward_host_f32) redirects the input buffer then.  STEM_BLOCK holds its dense weights.
struct OpKernel {
    int kind = SKPS_KERNEL_MISC;          // SKPS_KERNEL_*
    std::variant<std::monostate, ConvMmaLayer, TcLayer, TctLayer, PwLayer, HmLayer, XfLayer, FpwLayer, DwTmaLayer,
                 UpcatTmaLayer, StemBlockW> layer;
};

struct skps_engine {
    int device = 0, max_batch = 0;
    std::vector<BufDesc> bufs;
    std::vector<void*> dbuf;              // device buffers, max_batch samples each
    std::vector<OpDesc> ops;
    float* d_weights = nullptr;
    std::vector<float> h_weights;
    size_t n_weights = 0;
    int input_buf = -1;
    std::vector<int> output_bufs;
    float* d_stage_f32 = nullptr;         // staging for NCHW float32 host input
    float* d_in_f32 = nullptr;            // NHWC float32 copy of that input (f32_mode)
    bool f32_mode = false;                // first conv reads d_in_f32 instead of the uint8 input buffer
    std::map<int, cudaGraphExec_t> graphs;   // batch -> captured forward
    int launches = 0;
    bool use_graph = true;
    int device_sms = 132;                 // the device's SM count
    int num_sms = 132;                    // SMs the persistent kernels' grids are sized for (skps_engine_set_num_sms)
    std::vector<OpKernel> kern;           // per op
    // streaming host round trip (skps_engine_submit_host_u8): 2 slots, H2D on its own stream
    cudaStream_t s_copy = nullptr, s_compute = nullptr;
    void* d_slot_in[2] = {nullptr, nullptr};
    cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
};

static size_t buf_elems(const BufDesc& b) { return (size_t)b.C * b.H * b.W; }
static size_t buf_bytes(const BufDesc& b) { return buf_elems(b) * (b.dtype == DT_U8 ? 1 : 4); }   // SPLIT16 = 2+2 bytes

static float half_bits_to_float(uint16_t h) {
    uint32_t sign = (uint32_t)(h >> 15) << 31, exp = (h >> 10) & 31, man = h & 1023, bits;
    if (exp == 0) {
        if (man == 0) { bits = sign; }
        else { int e2 = -1; do { ++e2; man <<= 1; } while (!(man & 1024)); bits = sign | ((uint32_t)(112 - e2) << 23) | ((man & 1023) << 13); }
    } else if (exp == 31) { bits = sign | 0x7F800000u | (man << 13); }
    else { bits = sign | ((exp + 112) << 23) | (man << 13); }
    float f; memcpy(&f, &bits, 4); return f;
}

static TView resolve(const skps_engine* e, const View& v) {
    TView t;
    memset(&t, 0, sizeof(t));
    if (v.buf < 0) return t;
    const BufDesc& b = e->bufs[v.buf];
    t.base = (v.buf == e->input_buf && e->f32_mode) ? (void*)e->d_in_f32 : e->dbuf[v.buf];
    t.ld = b.C;
    t.c_off = v.c_off; t.c_stride = v.c_stride; t.C = v.C; t.H = b.H; t.W = b.W;
    t.sample = (long long)b.C * b.H * b.W;
    t.fmt = b.dtype;
    t.plane = t.sample * e->max_batch;
    return t;
}

// Kernel parameters of a stem block op for samples [0, batch).
static StemBlockK stem_params(const skps_engine* e, const OpDesc& op, int batch) {
    const TView in0 = resolve(e, op.in[0]), out0 = resolve(e, op.out[0]);
    StemBlockK k;
    k.in = e->f32_mode ? nullptr : (const uint8_t*)in0.base;
    k.in_f32 = e->f32_mode ? (const float*)in0.base : nullptr;      // resolve() points at d_in_f32 in this mode
    k.H = in0.H; k.W = in0.W; k.Hq = out0.H; k.Wq = out0.W;
    k.img0 = 0; k.n_tiles = batch * (out0.H / 8) * (out0.W / 16);
    k.dw1 = e->d_weights + op.i[0];
    k.out = out0.base; k.out_fmt = out0.fmt; k.out_plane = out0.plane; k.out_ld = out0.ld; k.out_coff = out0.c_off;
    return k;
}

// Enqueue ops [first,last) for samples [0, batch).
static int run_ops(skps_engine* e, int batch, cudaStream_t s, int first = 0, int last = -1) {
    const size_t end = last < 0 ? e->ops.size() : (size_t)last;
    const int sms = e->num_sms;
    for (size_t i = (size_t)first; i < end; ++i) {
        const OpDesc& op = e->ops[i];
        const auto& L = e->kern[i].layer;
        TView in0 = resolve(e, op.in[0]), in1 = resolve(e, op.in[1]), in2 = resolve(e, op.in[2]);
        TView out0 = resolve(e, op.out[0]), out1 = resolve(e, op.out[1]);
        const float* w = op.w_off >= 0 ? e->d_weights + op.w_off : nullptr;
        const float* b = op.b_off >= 0 ? e->d_weights + op.b_off : nullptr;
        int rc = 0;
        switch (e->kern[i].kind) {
            case SKPS_KERNEL_MMA: rc = conv_mma_launch(std::get<ConvMmaLayer>(L), batch, sms, s); break;
            case SKPS_KERNEL_TC: rc = tc_launch(std::get<TcLayer>(L), batch, sms, s); break;
            case SKPS_KERNEL_TCT: rc = tct_launch(std::get<TctLayer>(L), batch, sms, s); break;
            case SKPS_KERNEL_PW: rc = pw_launch(std::get<PwLayer>(L), batch, sms, s); break;
            case SKPS_KERNEL_HM: rc = hm_launch(std::get<HmLayer>(L), batch, sms, s); break;
            case SKPS_KERNEL_XF: rc = xf_launch(std::get<XfLayer>(L), batch, sms, s); break;
            case SKPS_KERNEL_FPW: rc = fpw_launch(std::get<FpwLayer>(L), batch, sms, s); break;
            case SKPS_KERNEL_DW_TMA: rc = dw_tma_launch(std::get<DwTmaLayer>(L), batch, s); break;
            case SKPS_KERNEL_UPCAT_TMA: rc = upcat_tma_launch(std::get<UpcatTmaLayer>(L), batch, s); break;
            case SKPS_KERNEL_STEM_BLOCK: rc = stem_block_launch(stem_params(e, op, batch), std::get<StemBlockW>(L), sms, s); break;
            case SKPS_KERNEL_SIMT_CONV: {
                ConvArgs a;
                a.in = in0; a.res = in1; a.gate = in2; a.out = out0; a.w = w; a.bias = b;
                a.kh = op.kh; a.kw = op.kw; a.sh = op.sh; a.sw = op.sw; a.ph = op.ph; a.pw = op.pw;
                a.dh = op.dh; a.dw = op.dw; a.act = op.act; a.in_u8 = ((op.flags & FLAG_IN_U8) && !e->f32_mode) ? 1 : 0;
                a.batch = batch;
                a.res_first = (op.flags & FLAG_RES_FIRST) ? 1 : 0;
                a.w_host = op.w_off >= 0 ? e->h_weights.data() + op.w_off : nullptr;
                a.bias_host = op.b_off >= 0 ? e->h_weights.data() + op.b_off : nullptr;
                rc = launch_conv(a, s);
                break;
            }
            case SKPS_KERNEL_DW: {
                DwArgs a;
                a.in = in0; a.out = out0; a.w = w; a.bias = b;
                a.kh = op.kh; a.kw = op.kw; a.sh = op.sh; a.sw = op.sw; a.ph = op.ph; a.pw = op.pw;
                a.dh = op.dh; a.dw = op.dw; a.act = op.act; a.batch = batch;
                rc = launch_dwconv(a, s);
                break;
            }
            case SKPS_KERNEL_UPCAT: rc = launch_upcat_dw(in0, in1, out0, w, b, op.act, batch, s); break;
            default:                                   // SKPS_KERNEL_MISC
                switch (op.type) {
                    case OP_MAXPOOL2: rc = launch_maxpool2(in0, out0, batch, s); break;
                    case OP_RESIZE_NEAREST: rc = launch_resize_nearest(in0, out0, batch, s); break;
                    case OP_UPSAMPLE_BILINEAR2X: rc = launch_bilinear2x(in0, out0, batch, s); break;
                    case OP_COPY: rc = launch_copy(in0, out0, batch, s); break;
                    case OP_GAP: rc = launch_gap(in0, out0, batch, s); break;
                    case OP_AFFINE_ACT: rc = launch_affine_act(in0, out0, w, b, op.act, batch, s); break;
                    case OP_SCSE: rc = launch_scse(in0, in1, in2, out0, batch, s); break;
                    case OP_SCALE_CH: rc = launch_scale_ch(in0, in1, out0, batch, s); break;
                    case OP_GAP_SSE:
                        rc = launch_gap_sse(in0, out0, out1, w, op.b_off >= 0 ? e->h_weights[op.b_off] : 0.f, op.act, batch, s);
                        break;
                    case OP_SE_FC:
                        // in0 = per-tile channel sums [n][tiles][C]; w = W1^T [C][Cr], i[0] -> W2^T [Cr][C]; b = [b1 (Cr) | b2 (C)]
                        rc = launch_se_fc(in0, out0, w, b, e->d_weights + op.i[0], b + op.i[1], op.i[1], op.act, op.i[2],
                                          op.i[3], batch, s);
                        break;
                    case OP_ADDN: {
                        TView ins[4] = {in0, in1, in2, resolve(e, op.in3)};
                        int n_in = 0;
                        while (n_in < 4 && ins[n_in].base) ++n_in;
                        rc = launch_addn(ins, n_in, out0, op.act, batch, s);
                        break;
                    }
                    case OP_DET_DECODE: {
                        TView heads[3] = {in0, in1, in2};
                        rc = launch_det_decode(heads, e->h_weights.data() + op.w_off, out0, op.i[0], batch, s);
                        break;
                    }
                    case OP_HM_DECODE: {
                        TView part = in2;                  // FLAG_HM_PART: per-tile (max, arg-max) rows from the head conv
                        rc = launch_hm_decode(in0, in1, w, b, out0, out1, op.i[0], batch, s,
                                              (op.flags & FLAG_HM_PART) ? &part : nullptr);
                        break;
                    }
                    default: set_error("engine: unknown op type %d (op %zu)", op.type, i); return 1;
                }
        }
        if (rc) {
            char tmp[900];
            snprintf(tmp, sizeof(tmp), "%s", get_error());
            set_error("op %zu (type %d): %s", i, op.type, tmp);
            return 1;
        }
    }
    return 0;
}

extern "C" SKPS_API const char* skps_last_error(void) { return get_error(); }
extern "C" SKPS_API int skps_version(void) { return 1; }

// A tensor-core conv op as conv_tc, conv_tct, conv_pw and conv_hm prepare it.
static TcSetup tc_setup(const skps_engine* e, const OpDesc& op) {
    const TView in0 = resolve(e, op.in[0]), res = resolve(e, op.in[1]), out0 = resolve(e, op.out[0]);
    TcSetup s = {};
    s.H = in0.H; s.W = in0.W; s.Cin = in0.C; s.in_ld = in0.ld; s.in_coff = in0.c_off; s.max_batch = e->max_batch;
    s.in_base = in0.base; s.in_plane = in0.plane;
    s.kh = op.kh; s.kw = op.kw; s.dil = op.dh; s.pad = op.ph; s.stride = op.sh;
    s.Cout = out0.C; s.act = op.act; s.n_tile = op.i[0]; s.n_tiles = op.i[1]; s.out_scale = op.f[0];
    s.w_hi = e->d_weights + op.w_off; s.w_lo = e->d_weights + op.i[2];
    s.bias = op.b_off >= 0 ? e->d_weights + op.b_off : nullptr;
    s.out = out0.base; s.out_fmt = out0.fmt; s.out_plane = out0.plane; s.out_ld = out0.ld; s.out_coff = out0.c_off;
    s.out_cstride = out0.c_stride;
    s.res = res.base; s.res_fmt = res.fmt; s.res_plane = res.plane; s.res_ld = res.ld; s.res_coff = res.c_off;
    s.res_first = (op.flags & FLAG_RES_FIRST) ? 1 : 0;
    if (op.flags & FLAG_HM_PART) {
        // out[1] = [tiles][2 * ld] per sample: ld maxima then ld arg-max indices; the map itself is not stored
        TView part = resolve(e, op.out[1]);
        s.hm_val = (float*)part.base; s.hm_idx = (int*)part.base + part.ld / 2; s.hm_ld = part.ld;
    }
    return s;
}

// A fused producer -> pointwise conv op (OP_DWPW: depthwise / up-sample+concat+depthwise; OP_CONV: squeeze-excite
// scale) as conv_fpw and conv_xf prepare it.
static XfSetup xf_setup(const skps_engine* e, const OpDesc& op) {
    const bool dwpw = op.type == OP_DWPW;
    XfSetup s;
    memset(&s, 0, sizeof(s));
    s.mode = dwpw ? XF_DW : XF_SCALE;
    s.max_batch = e->max_batch;
    s.x = resolve(e, op.in[0]);
    s.res = resolve(e, op.in[1]);
    if (dwpw) {
        s.low = resolve(e, op.in[2]);
        s.dww = e->d_weights + op.i[3];
        s.dw_act = (int)op.f[1];
        s.weff = s.low.base ? e->d_weights + op.i2[0] : nullptr;
    } else {
        s.gate = resolve(e, op.in[2]);
    }
    s.out = resolve(e, op.out[0]);
    s.Cout = s.out.C; s.act = op.act; s.n_tile = op.i[0]; s.n_tiles = op.i[1]; s.out_scale = op.f[0];
    s.w_hi = e->d_weights + op.w_off; s.w_lo = e->d_weights + op.i[2];
    s.bias = op.b_off >= 0 ? e->d_weights + op.b_off : nullptr;
    s.res_first = (op.flags & FLAG_RES_FIRST) ? 1 : 0;
    return s;
}

// Chooses the kernel op i runs and prepares its layer (TMA descriptors over the fixed activation buffers and weights).
// Returns null, or the name of the kernel whose preparation failed with the error naming the op.
static const char* prepare_op(skps_engine* e, int i) {
    const OpDesc& op = e->ops[i];
    OpKernel& k = e->kern[i];
    auto failed = [&](const char* what) {
        char tmp[900];
        snprintf(tmp, sizeof(tmp), "%s", get_error());
        set_error("op %d: %s", i, tmp);
        return what;
    };
    const TView in0 = resolve(e, op.in[0]), in1 = resolve(e, op.in[1]);
    const TView out0 = resolve(e, op.out[0]), out1 = resolve(e, op.out[1]);
    if (op.type == OP_CONV && (op.flags & FLAG_MMA)) {
        k.kind = SKPS_KERNEL_MMA;
        if (!conv_mma_supported(in0.C, out0.C, op.kh, op.kw, op.sh, op.dh, op.ph) ||
            conv_mma_prepare(k.layer.emplace<ConvMmaLayer>(), in0, out0, in1, (op.flags & FLAG_RES_FIRST) ? 1 : 0,
                             e->d_weights + op.w_off, op.b_off >= 0 ? e->d_weights + op.b_off : nullptr, op.f[0],
                             op.act, e->max_batch))
            return failed("mma");
        return nullptr;
    }
    // conv_fpw where it takes the layer (whole 16 x 8 tiles, unit-stride aligned output, instantiated width), else conv_xf
    if (op.type == OP_DWPW || (op.type == OP_CONV && (op.flags & FLAG_XF))) {
        const XfSetup s = xf_setup(e, op);
        if (fpw_supported(s)) {
            k.kind = SKPS_KERNEL_FPW;
            return fpw_prepare(k.layer.emplace<FpwLayer>(), s) ? failed("fpw") : nullptr;
        }
        k.kind = SKPS_KERNEL_XF;
        return xf_prepare(k.layer.emplace<XfLayer>(), s) ? failed("xf") : nullptr;
    }
    if (op.type == OP_CONV && (op.flags & FLAG_TC)) {
        if (in0.fmt != DT_SPLIT16 || in0.c_stride != 1 || op.in[2].buf >= 0 || op.sh != op.sw) {
            set_error("op %d: tensor-core conv needs a SPLIT16 unit-stride input and no gate", i);
            return "tc";
        }
        const TcSetup s = tc_setup(e, op);
        // the lowering sizes the partial buffer for 128-pixel tiles (conv_tc epilogue) or 256-pixel tiles (conv_hm.cu)
        if ((op.flags & FLAG_HM_PART) && out1.H * out1.W > 0 && out0.H * out0.W / (out1.H * out1.W) == HM_TILE_PIXELS) {
            k.kind = SKPS_KERNEL_HM;
            return hm_prepare(k.layer.emplace<HmLayer>(), s) ? failed("hm") : nullptr;
        }
        if (op.dh == op.dw && op.ph == op.pw && tct_applicable(s)) {
            k.kind = SKPS_KERNEL_TCT;
            return tct_prepare(k.layer.emplace<TctLayer>(), s) ? failed("tct") : nullptr;
        }
        if (op.ph == op.pw && pw_applicable(s)) {
            k.kind = SKPS_KERNEL_PW;
            return pw_prepare(k.layer.emplace<PwLayer>(), s) ? failed("pw") : nullptr;
        }
        k.kind = SKPS_KERNEL_TC;
        return op.dh != op.dw || op.ph != op.pw || tc_prepare(k.layer.emplace<TcLayer>(), s) ? failed("tc") : nullptr;
    }
    if (op.type == OP_CONV) {
        k.kind = SKPS_KERNEL_SIMT_CONV;
        return nullptr;
    }
    if (op.type == OP_DWCONV) {
        if (op.kh == op.kw && op.sh == op.sw && op.dh == op.dw && op.ph == op.pw &&
            dw_tma_supported(in0, out0, op.kh, op.sh, op.dh, op.ph)) {
            k.kind = SKPS_KERNEL_DW_TMA;
            // FLAG_GAP_PARTIAL: out[1] = per-tile channel sums for the squeeze-excite gate
            return dw_tma_prepare(k.layer.emplace<DwTmaLayer>(), in0, out0, e->d_weights + op.w_off,
                                  e->d_weights + op.b_off, op.kh, op.sh, op.dh, op.ph, op.act, e->max_batch,
                                  (op.flags & FLAG_GAP_PARTIAL) ? &out1 : nullptr) ? failed("dw_tma") : nullptr;
        }
        if (op.flags & FLAG_GAP_PARTIAL) {
            set_error("op %d: per-tile channel sums need the TMA depthwise kernel (unsupported layer)", i);
            return "dw_tma";
        }
        k.kind = SKPS_KERNEL_DW;
        return nullptr;
    }
    if (op.type == OP_UPCAT_DW) {              // in[0] = the low-resolution map, in[1] = the skip connection
        if (!upcat_tma_supported(in0, in1, out0)) {
            k.kind = SKPS_KERNEL_UPCAT;
            return nullptr;
        }
        k.kind = SKPS_KERNEL_UPCAT_TMA;
        return upcat_tma_prepare(k.layer.emplace<UpcatTmaLayer>(), in0, in1, out0, e->d_weights + op.w_off,
                                 e->d_weights + op.b_off, op.act, e->max_batch) ? failed("upcat_tma") : nullptr;
    }
    if (op.type == OP_STEM_BLOCK) {
        if (in0.fmt != DT_U8 || !stem_block_supported(in0.H, in0.W, out0.C, out0)) {
            set_error("op %d: stem block: unsupported shape", i);
            return "stem_block";
        }
        k.kind = SKPS_KERNEL_STEM_BLOCK;
        // w = StemBlockW as packed by lowering (dense weights -> kernel-parameter bank); i[0] -> [9][E]+[E] depthwise table
        memcpy(&k.layer.emplace<StemBlockW>(), e->h_weights.data() + op.w_off, sizeof(StemBlockW));
        return nullptr;
    }
    k.kind = SKPS_KERNEL_MISC;
    return nullptr;
}

int skps::engine_pair_device(const skps_engine* det, const skps_engine* kps, const char* fn, int* device) {
    SKPS_CHECK(det->device == kps->device, "%s: the detector engine is on device %d and the landmark engine on device %d; "
               "a pipeline's engines must share one device", fn, det->device, kps->device);
    *device = det->device;
    return 0;
}

extern "C" SKPS_API int skps_engine_create(const int32_t* words, size_t n_words, const float* weights, size_t n_floats,
                                  int max_batch, int device, skps_engine** out) {
    SKPS_CHECK(words && weights && out && n_words >= 8 && max_batch > 0, "engine_create: bad arguments");
    SKPS_CHECK(words[0] == PLAN_MAGIC && words[1] == 1, "engine_create: bad plan header");
    int n_bufs = words[2], n_ops = words[3];
    const size_t body = (size_t)8 + 4 * (size_t)n_bufs + OP_WORDS * (size_t)n_ops;
    SKPS_CHECK(n_words == body, "engine_create: plan size mismatch");
    SKPS_ON_DEVICE(device);
    skps_engine* e = new skps_engine();
    e->device = device;
    e->max_batch = max_batch;
    e->input_buf = words[4];
    for (int i = 0; i < words[5]; ++i) e->output_bufs.push_back(words[6 + i]);
    const int32_t* p = words + 8;
    for (int i = 0; i < n_bufs; ++i, p += 4) e->bufs.push_back(BufDesc{p[0], p[1], p[2], p[3]});
    e->ops.resize(n_ops);
    memcpy(e->ops.data(), p, sizeof(OpDesc) * n_ops);
    e->h_weights.assign(weights, weights + n_floats);
    e->n_weights = n_floats;
    e->launches = n_ops;
    auto fail = [&](const char* what) {
        char tmp[900];
        snprintf(tmp, sizeof(tmp), "%s", get_error());
        set_error("engine_create: %s: %s", what, tmp);
        skps_engine_destroy(e);
        return 1;
    };
    if (cudaMalloc(&e->d_weights, n_floats * sizeof(float)) != cudaSuccess) { set_error("cudaMalloc weights"); return fail("alloc"); }
    if (cudaMemcpy(e->d_weights, weights, n_floats * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
        set_error("cudaMemcpy weights"); return fail("copy");
    }
    // the elementwise kernels and the detector decode number their threads with 32-bit ints (ops_misc.cu): a batch of a
    // large input size (a re-targeted detector) must keep every activation tensor below 2^31 elements
    for (int i = 0; i < n_bufs; ++i) {
        if (buf_elems(e->bufs[i]) * (size_t)max_batch >= ((size_t)1 << 31)) {
            set_error("buffer %d (%dx%dx%d) has 2^31 or more elements at batch %d", i, e->bufs[i].H, e->bufs[i].W,
                      e->bufs[i].C, max_batch);
            return fail("size");
        }
    }
    e->dbuf.assign(n_bufs, nullptr);
    for (int i = 0; i < n_bufs; ++i) {
        size_t bytes = buf_bytes(e->bufs[i]) * (size_t)max_batch;
        if (cudaMalloc(&e->dbuf[i], bytes ? bytes : 16) != cudaSuccess) {
            set_error("cudaMalloc buffer %d (%zu bytes)", i, bytes);
            return fail("alloc");
        }
        cudaMemset(e->dbuf[i], 0, bytes);
    }
    const BufDesc& ib = e->bufs[e->input_buf];
    if (cudaMalloc(&e->d_stage_f32, buf_elems(ib) * sizeof(float) * (size_t)max_batch) != cudaSuccess ||
        cudaMalloc(&e->d_in_f32, buf_elems(ib) * sizeof(float) * (size_t)max_batch) != cudaSuccess) {
        set_error("cudaMalloc staging");
        return fail("alloc");
    }
    cudaDeviceGetAttribute(&e->device_sms, cudaDevAttrMultiProcessorCount, device);
    e->num_sms = e->device_sms;
    e->kern.resize(n_ops);
    for (int i = 0; i < n_ops; ++i)
        if (const char* what = prepare_op(e, i)) return fail(what);
    *out = e;
    return 0;
}

extern "C" SKPS_API void skps_engine_destroy(skps_engine* e) {
    if (!e) return;
    DeviceGuard on(e->device);
    for (auto& kv : e->graphs) cudaGraphExecDestroy(kv.second);
    for (void* p : e->dbuf) if (p) cudaFree(p);
    for (int i = 0; i < 2; ++i) {
        if (e->d_slot_in[i]) cudaFree(e->d_slot_in[i]);
        if (e->ev_in[i]) cudaEventDestroy(e->ev_in[i]);
        if (e->ev_free[i]) cudaEventDestroy(e->ev_free[i]);
        if (e->ev_done[i]) cudaEventDestroy(e->ev_done[i]);
    }
    if (e->s_copy) cudaStreamDestroy(e->s_copy);
    if (e->s_compute) cudaStreamDestroy(e->s_compute);
    if (e->d_weights) cudaFree(e->d_weights);
    if (e->d_stage_f32) cudaFree(e->d_stage_f32);
    if (e->d_in_f32) cudaFree(e->d_in_f32);
    delete e;
}

extern "C" SKPS_API int skps_engine_input_dims(const skps_engine* e, int* h, int* w, int* c) {
    SKPS_CHECK(e, "null engine");
    const BufDesc& b = e->bufs[e->input_buf];
    if (h) *h = b.H;
    if (w) *w = b.W;
    if (c) *c = b.C;
    return 0;
}
extern "C" SKPS_API int skps_engine_num_outputs(const skps_engine* e) { return e ? (int)e->output_bufs.size() : 0; }
extern "C" SKPS_API int skps_engine_output_elems(const skps_engine* e, int idx) {
    if (!e || idx < 0 || idx >= (int)e->output_bufs.size()) return 0;
    return (int)buf_elems(e->bufs[e->output_bufs[idx]]);
}
extern "C" SKPS_API void* skps_engine_input_ptr(skps_engine* e) { return e ? e->dbuf[e->input_buf] : nullptr; }
extern "C" SKPS_API float* skps_engine_output_ptr(skps_engine* e, int idx) {
    if (!e || idx < 0 || idx >= (int)e->output_bufs.size()) return nullptr;
    return (float*)e->dbuf[e->output_bufs[idx]];
}
extern "C" SKPS_API int skps_engine_num_buffers(const skps_engine* e) { return e ? (int)e->bufs.size() : 0; }
extern "C" SKPS_API int skps_engine_buffer_dims(const skps_engine* e, int buf, int* h, int* w, int* c, int* dtype) {
    SKPS_CHECK(e && buf >= 0 && buf < (int)e->bufs.size(), "buffer_dims: bad index");
    const BufDesc& b = e->bufs[buf];
    if (h) *h = b.H;
    if (w) *w = b.W;
    if (c) *c = b.C;
    if (dtype) *dtype = b.dtype;
    return 0;
}
extern "C" SKPS_API int skps_engine_read_buffer(skps_engine* e, int buf, int batch, void* dst) {
    SKPS_CHECK(e && buf >= 0 && buf < (int)e->bufs.size() && batch <= e->max_batch, "read_buffer: bad arguments");
    SKPS_ON_DEVICE(e->device);
    SKPS_CUDA(cudaDeviceSynchronize());
    const BufDesc& b = e->bufs[buf];
    if (b.dtype == DT_SPLIT16) {
        // hi plane + lo plane (each max_batch samples) -> float32
        size_t n = buf_elems(b) * (size_t)batch, plane = buf_elems(b) * (size_t)e->max_batch;
        std::vector<uint16_t> hi(n), lo(n);
        SKPS_CUDA(cudaMemcpy(hi.data(), e->dbuf[buf], n * 2, cudaMemcpyDeviceToHost));
        SKPS_CUDA(cudaMemcpy(lo.data(), (const uint16_t*)e->dbuf[buf] + plane, n * 2, cudaMemcpyDeviceToHost));
        float* d = (float*)dst;
        for (size_t i = 0; i < n; ++i) d[i] = half_bits_to_float(hi[i]) + half_bits_to_float(lo[i]);
        return 0;
    }
    SKPS_CUDA(cudaMemcpy(dst, e->dbuf[buf], buf_bytes(b) * batch, cudaMemcpyDeviceToHost));
    return 0;
}
extern "C" SKPS_API int skps_engine_launches_per_forward(const skps_engine* e) { return e ? e->launches : 0; }
extern "C" SKPS_API int skps_engine_launches_for_batch(const skps_engine* e, int batch) {
    if (!e || batch <= 0) return 0;
    int n = 0;
    for (const OpKernel& k : e->kern)      // the TMA fused-upsample op is two kernels (up-sampled part + skip part)
        n += k.kind == SKPS_KERNEL_UPCAT_TMA ? 2 : 1;
    return n;
}

extern "C" SKPS_API int skps_engine_run_op(skps_engine* e, int op_index, int batch, void* stream) {
    SKPS_CHECK(e && op_index >= 0 && op_index < (int)e->ops.size(), "run_op: bad op index");
    SKPS_CHECK(batch > 0 && batch <= e->max_batch, "run_op: batch %d outside 1..%d", batch, e->max_batch);
    SKPS_ON_DEVICE(e->device);
    return run_ops(e, batch, (cudaStream_t)stream, op_index, op_index + 1);
}

// The branch run_ops() takes for one op, and the tiling its kernel was prepared with.
extern "C" SKPS_API int skps_engine_op_kernel(const skps_engine* e, int op_index, int32_t info[4]) {
    if (!e || op_index < 0 || op_index >= (int)e->ops.size()) return -1;
    int32_t tmp[4];
    int32_t* inf = info ? info : tmp;
    inf[0] = inf[1] = inf[2] = inf[3] = 0;
    const OpKernel& k = e->kern[op_index];
    switch (k.kind) {
        case SKPS_KERNEL_TC: {
            const TcK& t = std::get<TcLayer>(k.layer).k;
            inf[0] = t.bw; inf[1] = t.bh; inf[2] = t.ipt; inf[3] = t.mt;
            break;
        }
        case SKPS_KERNEL_TCT: inf[0] = std::get<TctLayer>(k.layer).k.bh; break;
        case SKPS_KERNEL_PW: {
            const PwLayer& L = std::get<PwLayer>(k.layer);
            inf[0] = L.nc; inf[1] = L.k.n_chunks;
            break;
        }
        case SKPS_KERNEL_FPW: {
            const FpwLayer& L = std::get<FpwLayer>(k.layer);
            inf[0] = 128; inf[1] = L.n; inf[2] = L.k.nsplit; inf[3] = L.mode;
            break;
        }
        case SKPS_KERNEL_DW_TMA: {
            const DwTmaLayer& L = std::get<DwTmaLayer>(k.layer);
            inf[0] = dw_tile_rows(L.k_size, L.stride);
            break;
        }
    }
    return k.kind;
}

extern "C" SKPS_API int skps_engine_set_num_sms(skps_engine* e, int n) {
    SKPS_CHECK(e, "set_num_sms: null engine");
    SKPS_CHECK(n >= 0 && n <= e->device_sms, "set_num_sms: %d outside 0..%d", n, e->device_sms);
    SKPS_ON_DEVICE(e->device);
    // a captured forward keeps the grids it was captured with
    for (auto& kv : e->graphs) cudaGraphExecDestroy(kv.second);
    e->graphs.clear();
    e->num_sms = n ? n : e->device_sms;
    return 0;
}

// The grid run_ops() launches for a persistent op, from the same helpers the launchers size it with.
extern "C" SKPS_API int skps_engine_op_grid(const skps_engine* e, int op_index, int batch, int32_t out[2]) {
    SKPS_CHECK(e && out && op_index >= 0 && op_index < (int)e->ops.size(), "op_grid: bad arguments");
    SKPS_CHECK(batch > 0 && batch <= e->max_batch, "op_grid: batch %d outside 1..%d", batch, e->max_batch);
    const OpKernel& k = e->kern[op_index];
    const int sms = e->num_sms;
    Grid g = {0, 0};
    switch (k.kind) {
        case SKPS_KERNEL_MMA: g = conv_mma_grid(std::get<ConvMmaLayer>(k.layer), batch, sms); break;
        case SKPS_KERNEL_TC: g = tc_grid(std::get<TcLayer>(k.layer), batch, sms); break;
        case SKPS_KERNEL_TCT: g = tct_grid(std::get<TctLayer>(k.layer), batch, sms); break;
        case SKPS_KERNEL_PW: g = pw_grid(std::get<PwLayer>(k.layer), batch, sms); break;
        case SKPS_KERNEL_HM: g = hm_grid(std::get<HmLayer>(k.layer), batch, sms); break;
        case SKPS_KERNEL_XF: g = xf_grid(std::get<XfLayer>(k.layer), batch, sms); break;
        case SKPS_KERNEL_FPW: g = fpw_grid(std::get<FpwLayer>(k.layer), batch, sms); break;
        case SKPS_KERNEL_STEM_BLOCK: g = stem_block_grid(stem_params(e, e->ops[op_index], batch), sms); break;
    }
    out[0] = g.ctas;
    out[1] = g.units;
    return 0;
}

// Enqueue the op sequence (through a cached CUDA graph when possible).
static int enqueue(skps_engine* e, int batch, cudaStream_t s) {
    if (!e->use_graph || s == nullptr) return run_ops(e, batch, s);   // the legacy default stream cannot be captured
    const int key = batch * 2 + (e->f32_mode ? 1 : 0);
    auto it = e->graphs.find(key);
    if (it == e->graphs.end()) {
        cudaStreamCaptureStatus st;
        SKPS_CUDA(cudaStreamIsCapturing(s, &st));
        if (st != cudaStreamCaptureStatusNone) return run_ops(e, batch, s);   // already inside a capture
        cudaGraph_t g = nullptr;
        SKPS_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        int rc = run_ops(e, batch, s);
        cudaError_t ce = cudaStreamEndCapture(s, &g);
        if (rc) { if (g) cudaGraphDestroy(g); return rc; }
        SKPS_CUDA(ce);
        cudaGraphExec_t ge = nullptr;
        SKPS_CUDA(cudaGraphInstantiate(&ge, g, 0));
        cudaGraphDestroy(g);
        it = e->graphs.emplace(key, ge).first;
    }
    SKPS_CUDA(cudaGraphLaunch(it->second, s));
    return 0;
}

static int copy_outputs(skps_engine* e, int batch, float* const* outputs, cudaMemcpyKind kind, cudaStream_t s) {
    if (!outputs) return 0;
    for (size_t i = 0; i < e->output_bufs.size(); ++i) {
        if (!outputs[i]) continue;
        const BufDesc& b = e->bufs[e->output_bufs[i]];
        SKPS_CUDA(cudaMemcpyAsync(outputs[i], e->dbuf[e->output_bufs[i]], buf_bytes(b) * batch, kind, s));
    }
    return 0;
}

extern "C" SKPS_API int skps_engine_forward(skps_engine* e, const uint8_t* input, int batch, float* const* outputs,
                                   void* stream) {
    SKPS_CHECK(e && input, "forward: null argument");
    SKPS_CHECK(batch > 0 && batch <= e->max_batch, "forward: batch %d outside 1..%d", batch, e->max_batch);
    cudaStream_t s = (cudaStream_t)stream;
    SKPS_ON_DEVICE(e->device);
    const BufDesc& ib = e->bufs[e->input_buf];
    SKPS_CHECK(ib.dtype == DT_U8, "forward: engine input is not uint8");
    if ((const void*)input != e->dbuf[e->input_buf])
        SKPS_CUDA(cudaMemcpyAsync(e->dbuf[e->input_buf], input, buf_bytes(ib) * batch, cudaMemcpyDeviceToDevice, s));
    if (enqueue(e, batch, s)) return 1;
    return copy_outputs(e, batch, outputs, cudaMemcpyDeviceToDevice, s);
}

// float32 NCHW -> float32 NHWC (ONNXEngine.__call__ feeds NCHW, onnx_model_base.py:17).
__global__ void nchw_to_nhwc_f32(const float* __restrict__ src, float* __restrict__ dst, int C, int H, int W,
                                 long long total) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int c = (int)(i % C);
    long long pix = i / C;
    int x = (int)(pix % W);
    long long t = pix / W;
    int y = (int)(t % H);
    long long n = t / H;
    dst[i] = src[((n * C + c) * H + y) * W + x];
}

extern "C" SKPS_API int skps_engine_forward_host_u8(skps_engine* e, const uint8_t* input, int batch, float* const* outputs,
                                           void* stream) {
    SKPS_CHECK(e && input, "forward_host_u8: null argument");
    SKPS_CHECK(batch > 0 && batch <= e->max_batch, "forward: batch %d outside 1..%d", batch, e->max_batch);
    cudaStream_t s = (cudaStream_t)stream;
    SKPS_ON_DEVICE(e->device);
    const BufDesc& ib = e->bufs[e->input_buf];
    SKPS_CUDA(cudaMemcpyAsync(e->dbuf[e->input_buf], input, buf_bytes(ib) * batch, cudaMemcpyHostToDevice, s));
    if (enqueue(e, batch, s)) return 1;
    if (copy_outputs(e, batch, outputs, cudaMemcpyDeviceToHost, s)) return 1;
    SKPS_CUDA(cudaStreamSynchronize(s));
    return 0;
}

extern "C" SKPS_API int skps_engine_forward_host_f32(skps_engine* e, const float* input, int batch, float* const* outputs,
                                            void* stream) {
    SKPS_CHECK(e && input, "forward_host_f32: null argument");
    SKPS_CHECK(batch > 0 && batch <= e->max_batch, "forward: batch %d outside 1..%d", batch, e->max_batch);
    cudaStream_t s = (cudaStream_t)stream;
    SKPS_ON_DEVICE(e->device);
    const BufDesc& ib = e->bufs[e->input_buf];
    long long total = (long long)buf_elems(ib) * batch;
    SKPS_CUDA(cudaMemcpyAsync(e->d_stage_f32, input, total * sizeof(float), cudaMemcpyHostToDevice, s));
    nchw_to_nhwc_f32<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(e->d_stage_f32, e->d_in_f32, ib.C, ib.H, ib.W, total);
    SKPS_CUDA(cudaGetLastError());
    e->f32_mode = true;
    int rc = enqueue(e, batch, s);
    e->f32_mode = false;
    if (rc) return 1;
    if (copy_outputs(e, batch, outputs, cudaMemcpyDeviceToHost, s)) return 1;
    SKPS_CUDA(cudaStreamSynchronize(s));
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// Streaming host round trip: while batch i computes, batch i+1's pixels cross PCIe on a second stream.
// Two slots; the caller alternates them:  submit(0) submit(1) wait(0) submit(0) wait(1) ...
// `input` and `outputs[i]` should be pinned host memory and must stay valid until skps_engine_wait(slot).
// ---------------------------------------------------------------------------------------------------
static int ensure_streaming(skps_engine* e) {
    if (e->s_copy) return 0;
    const BufDesc& ib = e->bufs[e->input_buf];
    SKPS_CUDA(cudaStreamCreateWithFlags(&e->s_copy, cudaStreamNonBlocking));
    SKPS_CUDA(cudaStreamCreateWithFlags(&e->s_compute, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
        SKPS_CUDA(cudaMalloc(&e->d_slot_in[i], buf_bytes(ib) * (size_t)e->max_batch));
        SKPS_CUDA(cudaEventCreateWithFlags(&e->ev_in[i], cudaEventDisableTiming));
        SKPS_CUDA(cudaEventCreateWithFlags(&e->ev_free[i], cudaEventDisableTiming));
        SKPS_CUDA(cudaEventCreateWithFlags(&e->ev_done[i], cudaEventDisableTiming));
    }
    return 0;
}

extern "C" SKPS_API int skps_engine_submit_host_u8(skps_engine* e, int slot, const uint8_t* input, int batch,
                                                   float* const* outputs) {
    SKPS_CHECK(e && input && (slot == 0 || slot == 1), "submit: bad arguments");
    SKPS_CHECK(batch > 0 && batch <= e->max_batch, "submit: batch %d outside 1..%d", batch, e->max_batch);
    SKPS_ON_DEVICE(e->device);
    if (ensure_streaming(e)) return 1;
    const BufDesc& ib = e->bufs[e->input_buf];
    const size_t in_bytes = buf_bytes(ib) * (size_t)batch;
    // the slot's staging buffer is free once the compute that consumed it has copied it out (ev_free)
    SKPS_CUDA(cudaStreamWaitEvent(e->s_copy, e->ev_free[slot], 0));
    SKPS_CUDA(cudaMemcpyAsync(e->d_slot_in[slot], input, in_bytes, cudaMemcpyHostToDevice, e->s_copy));
    SKPS_CUDA(cudaEventRecord(e->ev_in[slot], e->s_copy));
    SKPS_CUDA(cudaStreamWaitEvent(e->s_compute, e->ev_in[slot], 0));
    SKPS_CUDA(cudaMemcpyAsync(e->dbuf[e->input_buf], e->d_slot_in[slot], in_bytes, cudaMemcpyDeviceToDevice, e->s_compute));
    SKPS_CUDA(cudaEventRecord(e->ev_free[slot], e->s_compute));
    if (enqueue(e, batch, e->s_compute)) return 1;
    if (copy_outputs(e, batch, outputs, cudaMemcpyDeviceToHost, e->s_compute)) return 1;
    SKPS_CUDA(cudaEventRecord(e->ev_done[slot], e->s_compute));
    return 0;
}

extern "C" SKPS_API int skps_engine_wait(skps_engine* e, int slot) {
    SKPS_CHECK(e && (slot == 0 || slot == 1) && e->s_copy, "wait: nothing submitted");
    SKPS_ON_DEVICE(e->device);
    SKPS_CUDA(cudaEventSynchronize(e->ev_done[slot]));
    return 0;
}
