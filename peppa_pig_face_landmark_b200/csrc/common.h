// Shared declarations for libskps_b200.so (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

namespace skps {

// Streaming multiprocessors of the current device (launch grids of persistent and grid-stride kernels)
inline int sm_count() {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    return n;
}

// Launch of a persistent kernel: `ctas` CTAs walk `units` work units as blockIdx.x, + gridDim.x, ...  Each persistent
// launcher computes it in one helper (tc_grid, pw_grid, ...) that skps_engine_op_grid reports as well.
struct Grid {
    int ctas, units;
};
inline Grid persistent_grid(long long units, long long max_ctas) {
    return Grid{(int)(units < max_ctas ? units : max_ctas), (int)units};
}

// cuTensorMapEncodeTiled, looked up through the runtime so that the library needs no link against the driver library;
// null when the driver does not provide it
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn tensor_map_encoder() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// ---- op codes / activations: keep in sync with peppa_pig_face_landmark_b200/plan.py ----
enum OpType {
    OP_CONV = 1, OP_DWCONV = 2, OP_MAXPOOL2 = 3, OP_RESIZE_NEAREST = 4, OP_UPSAMPLE_BILINEAR2X = 5,
    OP_COPY = 6, OP_GAP = 7, OP_AFFINE_ACT = 8, OP_SCSE = 9, OP_DET_DECODE = 10, OP_HM_DECODE = 11,
    OP_SCALE_CH = 12, OP_UPCAT_DW = 13, OP_ADDN = 14, OP_SE_FC = 15, OP_DWPW = 16, OP_STEM_BLOCK = 17, OP_GAP_SSE = 18
};
enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_HSWISH = 2, ACT_SILU = 3, ACT_SIGMOID = 4, ACT_HSIGMOID = 5 };
enum { DT_F32 = 0, DT_U8 = 1, DT_SPLIT16 = 2 };   // SPLIT16: fp16 hi plane + fp16 lo plane, v = hi + lo
enum { FLAG_IN_U8 = 1, FLAG_TC = 2, FLAG_RES_FIRST = 4, FLAG_GAP_PARTIAL = 8, FLAG_MMA = 16, FLAG_XF = 32, FLAG_HM_PART = 64 };
enum { OP_WORDS = 64, PLAN_MAGIC = 0x534B5053 };

struct View {            // 6 words
    int32_t buf, c_off, c_stride, C, H, W;
};
struct OpDesc {          // 64 words
    int32_t type, act;
    View in[3];
    View out[2];
    int32_t kh, kw, sh, sw, ph, pw, dh, dw;
    int32_t w_off, b_off, flags;
    int32_t i[4];
    float f[8];
    View in3;            // 4th input (OP_ADDN)
    int32_t i2[2];       // more blob offsets (OP_DWPW: [0] = class weights of the up-sampled channels)
    int32_t pad[64 - (2 + 30 + 8 + 3 + 4 + 8 + 6 + 2)];
};
static_assert(sizeof(OpDesc) == 64 * 4, "OpDesc must be 64 words");

struct BufDesc { int32_t C, H, W, dtype; };

// A resolved tensor view on device memory (NHWC, batch outermost).
struct TView {
    void* base;        // buffer base (sample 0)
    int ld;            // channels of the underlying buffer (row pitch in elements per pixel)
    int c_off, c_stride, C, H, W;
    long long sample;  // elements per sample = H*W*ld
    int fmt;           // DT_F32 / DT_U8 / DT_SPLIT16
    long long plane;   // SPLIT16: element offset from the hi plane to the lo plane (= max_batch*sample)
};

void set_error(const char* fmt, ...);
const char* get_error();

#define SKPS_CUDA(call)                                                                   \
    do {                                                                                  \
        cudaError_t _e = (call);                                                          \
        if (_e != cudaSuccess) {                                                          \
            skps::set_error("%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
            return 1;                                                                     \
        }                                                                                 \
    } while (0)

#define SKPS_CHECK(cond, ...)                 \
    do {                                      \
        if (!(cond)) {                        \
            skps::set_error(__VA_ARGS__);     \
            return 1;                         \
        }                                     \
    } while (0)

// ---- per-device state: kernel attributes and allocations apply to the device current when they were made ----
constexpr int MAX_DEVICES = 64;

// Raises a kernel's dynamic shared-memory limit on the current device to `bytes` where it is lower.  set_bytes: the
// kernel's limit per device so far, MAX_DEVICES entries kept by the caller (one static array per kernel).
inline int smem_limit(const void* kernel, int* set_bytes, int bytes) {
    int dev = 0;
    SKPS_CUDA(cudaGetDevice(&dev));
    SKPS_CHECK(dev >= 0 && dev < MAX_DEVICES, "device %d out of range", dev);
    if (bytes > set_bytes[dev]) {
        SKPS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        set_bytes[dev] = bytes;
    }
    return 0;
}

// 1024 zeros on the current device, standing in for a missing bias; one allocation per device, null on failure
inline const float* zero_bias() {
    static float* z[MAX_DEVICES] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEVICES) return nullptr;
    if (!z[dev]) {
        if (cudaMalloc(&z[dev], 1024 * sizeof(float)) != cudaSuccess) { z[dev] = nullptr; return nullptr; }
        if (cudaMemset(z[dev], 0, 1024 * sizeof(float)) != cudaSuccess) return nullptr;
    }
    return z[dev];
}

// Makes `dev` the calling thread's current device for the guard's life and gives the caller back its own current device
// on every return path.  Every entry point on a handle opens one (SKPS_ON_DEVICE), so a call launches only on the
// handle's device whatever device is current, and leaves the current device as it found it.
class DeviceGuard {
public:
    explicit DeviceGuard(int dev) : dev_(dev) {
        if (cudaGetDevice(&prev_) != cudaSuccess) prev_ = -1;
        err_ = prev_ == dev ? cudaSuccess : cudaSetDevice(dev);
    }
    ~DeviceGuard() {
        if (prev_ >= 0 && prev_ != dev_) cudaSetDevice(prev_);
    }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
    cudaError_t status() const { return err_; }

private:
    int dev_, prev_ = -1;
    cudaError_t err_;
};
#define SKPS_ON_DEVICE(dev)                         \
    skps::DeviceGuard skps_device_guard_(dev);      \
    SKPS_CUDA(skps_device_guard_.status())

// The fail-and-destroy lambdas of the *_create functions report a failed step as "<fn>: <what>: <error set by the step>".
inline void prefix_error(const char* fn, const char* what) {
    char tmp[900];
    snprintf(tmp, sizeof(tmp), "%s", get_error());
    set_error("%s: %s: %s", fn, what, tmp);
}

// Allocations of a *_create function that owns a fail-and-destroy lambda `fail(what)`: on failure the size is recorded and
// fail("alloc") frees everything allocated so far.
#define SKPS_DEV_ALLOC(ptr, bytes)                                                                                  \
    do {                                                                                                            \
        if (cudaMalloc((void**)&(ptr), (bytes)) != cudaSuccess) {                                                   \
            skps::set_error("cudaMalloc %zu bytes", (size_t)(bytes));                                               \
            return fail("alloc");                                                                                   \
        }                                                                                                           \
    } while (0)
#define SKPS_HOST_ALLOC(ptr, bytes)                                                                                 \
    do {                                                                                                            \
        if (cudaMallocHost((void**)&(ptr), (bytes)) != cudaSuccess) {                                               \
            skps::set_error("cudaMallocHost %zu bytes", (size_t)(bytes));                                           \
            return fail("alloc");                                                                                   \
        }                                                                                                           \
    } while (0)

// ---- activation (device) -------------------------------------------------------------------
// HardSigmoid follows ONNX: max(0, min(1, alpha*x + beta)) with alpha = float32(1/6), beta = 0.5
// (kps_student.onnx node 2 etc.); alpha*x+beta is evaluated as mul then add (no FMA) to match a
// CPU execution provider's two-step evaluation as closely as possible.
__device__ __forceinline__ float hsigmoid_f(float x) {
    float t = __fadd_rn(__fmul_rn(x, 0.1666666716337204f), 0.5f);
    return fminf(fmaxf(t, 0.f), 1.f);
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ float apply_act(float v, int act) {
    switch (act) {
        case ACT_RELU: return fmaxf(v, 0.f);
        case ACT_HSWISH: return v * hsigmoid_f(v);
        case ACT_SILU: return v * sigmoid_f(v);
        case ACT_SIGMOID: return sigmoid_f(v);
        case ACT_HSIGMOID: return hsigmoid_f(v);
        default: return v;
    }
}

// ---- format-generic element access: float32, or float16 hi/lo planes (v = hi + lo) ------------------
}  // namespace skps
#include <cuda_fp16.h>
namespace skps {
__device__ __forceinline__ float ld1(const void* base, int fmt, long long plane, long long i) {
    if (fmt == DT_SPLIT16) {
        const __half* h = (const __half*)base;
        return __half2float(h[i]) + __half2float(h[i + plane]);
    }
    return ((const float*)base)[i];
}
__device__ __forceinline__ void st1(void* base, int fmt, long long plane, long long i, float v) {
    if (fmt == DT_SPLIT16) {
        __half* h = (__half*)base;
        __half hi = __float2half_rn(v);
        h[i] = hi;
        h[i + plane] = __float2half_rn(v - __half2float(hi));
    } else {
        ((float*)base)[i] = v;
    }
}
// 4 consecutive elements, i a multiple of 4
__device__ __forceinline__ float4 ld4(const void* base, int fmt, long long plane, long long i) {
    if (fmt == DT_SPLIT16) {
        const __half* h = (const __half*)base;
        uint2 a = *reinterpret_cast<const uint2*>(h + i), b = *reinterpret_cast<const uint2*>(h + i + plane);
        const __half2* a2 = reinterpret_cast<const __half2*>(&a);
        const __half2* b2 = reinterpret_cast<const __half2*>(&b);
        float2 a01 = __half22float2(a2[0]), a23 = __half22float2(a2[1]);
        float2 b01 = __half22float2(b2[0]), b23 = __half22float2(b2[1]);
        return make_float4(a01.x + b01.x, a01.y + b01.y, a23.x + b23.x, a23.y + b23.y);
    }
    return *reinterpret_cast<const float4*>((const float*)base + i);
}
__device__ __forceinline__ void st4(void* base, int fmt, long long plane, long long i, float4 v) {
    if (fmt == DT_SPLIT16) {
        __half* h = (__half*)base;
        __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
        float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
        __half2 l01 = __floats2half2_rn(v.x - f01.x, v.y - f01.y), l23 = __floats2half2_rn(v.z - f23.x, v.w - f23.y);
        uint2 a, b;
        a.x = *reinterpret_cast<uint32_t*>(&h01); a.y = *reinterpret_cast<uint32_t*>(&h23);
        b.x = *reinterpret_cast<uint32_t*>(&l01); b.y = *reinterpret_cast<uint32_t*>(&l23);
        *reinterpret_cast<uint2*>(h + i) = a;
        *reinterpret_cast<uint2*>(h + i + plane) = b;
    } else {
        *reinterpret_cast<float4*>((float*)base + i) = v;
    }
}

// 8 consecutive elements, i a multiple of 8 (one 16-byte load per float16 plane)
struct float8 { float v[8]; };
__device__ __forceinline__ float8 ld8(const void* base, int fmt, long long plane, long long i) {
    float8 r;
    if (fmt == DT_SPLIT16) {
        const __half* h = (const __half*)base;
        const uint4 a = *reinterpret_cast<const uint4*>(h + i), b = *reinterpret_cast<const uint4*>(h + i + plane);
        const __half2* a2 = reinterpret_cast<const __half2*>(&a);
        const __half2* b2 = reinterpret_cast<const __half2*>(&b);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 x = __half22float2(a2[j]), y = __half22float2(b2[j]);
            r.v[2 * j] = x.x + y.x;
            r.v[2 * j + 1] = x.y + y.y;
        }
    } else {
        const float4 a = *reinterpret_cast<const float4*>((const float*)base + i);
        const float4 b = *reinterpret_cast<const float4*>((const float*)base + i + 4);
        r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
        r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    }
    return r;
}
__device__ __forceinline__ void st8(void* base, int fmt, long long plane, long long i, const float8& r) {
    if (fmt == DT_SPLIT16) {
        __half* h = (__half*)base;
        uint4 hv, lv;
        uint32_t* hp = reinterpret_cast<uint32_t*>(&hv);
        uint32_t* lp = reinterpret_cast<uint32_t*>(&lv);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const __half2 h2 = __floats2half2_rn(r.v[2 * j], r.v[2 * j + 1]);
            const float2 hf = __half22float2(h2);
            const __half2 l2 = __floats2half2_rn(r.v[2 * j] - hf.x, r.v[2 * j + 1] - hf.y);
            hp[j] = *reinterpret_cast<const uint32_t*>(&h2);
            lp[j] = *reinterpret_cast<const uint32_t*>(&l2);
        }
        *reinterpret_cast<uint4*>(h + i) = hv;
        *reinterpret_cast<uint4*>(h + i + plane) = lv;
    } else {
        float* f = (float*)base + i;
        *reinterpret_cast<float4*>(f) = make_float4(r.v[0], r.v[1], r.v[2], r.v[3]);
        *reinterpret_cast<float4*>(f + 4) = make_float4(r.v[4], r.v[5], r.v[6], r.v[7]);
    }
}

// ---- kernel launchers (defined in the .cu files) ---------------------------------------------
struct ConvArgs {
    TView in, out, res, gate;     // res.base / gate.base may be null
    const float* w;               // [Cout][kh*kw][Cin]
    const float* bias;            // may be null
    int kh, kw, sh, sw, ph, pw, dh, dw, act, in_u8, batch;
    int res_first;                // act(conv + bias + res) instead of act(conv + bias) + res
    const float* w_host;          // host copies of w / bias (kernels that take weights as kernel parameters); may be null
    const float* bias_host;
};
int launch_conv(const ConvArgs& a, cudaStream_t s);
bool stem_conv_supported(const ConvArgs& a);
bool pw_small_supported(const ConvArgs& a);       // 1x1, Cout 16/24, Cin <= 96 on large maps (HBM-bound layers)
int launch_pw_small(const ConvArgs& a, cudaStream_t s);
int launch_stem_conv(const ConvArgs& a, cudaStream_t s);

struct DwArgs {
    TView in, out;
    const float* w;               // [kh*kw][C]
    const float* bias;
    int kh, kw, sh, sw, ph, pw, dh, dw, act, batch;
};
int launch_dwconv(const DwArgs& a, cudaStream_t s);
// depthwise 3x3 over concat(bilinear-x2(low), skip) without materialising the upsampled tensor
int launch_upcat_dw(const TView& low, const TView& skip, const TView& out, const float* w, const float* bias, int act,
                    int batch, cudaStream_t s);

int launch_maxpool2(const TView& in, const TView& out, int batch, cudaStream_t s);
int launch_resize_nearest(const TView& in, const TView& out, int batch, cudaStream_t s);
int launch_bilinear2x(const TView& in, const TView& out, int batch, cudaStream_t s);
int launch_copy(const TView& in, const TView& out, int batch, cudaStream_t s);
int launch_gap(const TView& in, const TView& out, int batch, cudaStream_t s);
int launch_affine_act(const TView& in, const TView& out, const float* sc, const float* sh, int act, int batch,
                      cudaStream_t s);
int launch_scse(const TView& x, const TView& cse, const TView& sse, const TView& out, int batch, cudaStream_t s);
int launch_det_decode(const TView* heads, const float* consts, const TView& out, int rows, int batch, cudaStream_t s);
int launch_scale_ch(const TView& x, const TView& gate, const TView& out, int batch, cudaStream_t s);
// out = act(sum_j in_j), in_j read at (y >> shift_j, x >> shift_j): HRNet fuse layers (nearest upsample fused)
int launch_addn(const TView* ins, int n_in, const TView& out, int act, int batch, cudaStream_t s);
// squeeze-excite gate from the depthwise kernel's per-tile channel sums: mean -> FC -> act1 -> FC -> act2
int launch_se_fc(const TView& part, const TView& gate, const float* w1t, const float* b1, const float* w2t, const float* b2,
                 int Cr, int act1, int act2, int hw, int batch, cudaStream_t s);
// feat.base != null: hm holds the score maps only and the x/y offsets are w_off/b_off ([2P][K], [2P]) applied to feat at the arg-max pixel
// part != null: the head conv wrote per-tile (max, arg-max) rows instead of the map (FLAG_HM_PART); hm is then only its shape
// scSE front end (ops_misc.cu): x (N,H,W,C) -> per-tile channel sums part (N,tiles,C) + the sSE map act(x . w + b) (N,H,W,1)
constexpr int GAP_SSE_TILE = 32;     // pixels per tile (rows of `part` per sample = H*W / 32)
int launch_gap_sse(const TView& x, const TView& part, const TView& sse, const float* w, float bias, int act, int batch,
                   cudaStream_t s);
int launch_hm_decode(const TView& hm, const TView& feat, const float* w_off, const float* b_off, const TView& xy,
                     const TView& score, int npts, int batch, cudaStream_t s, const TView* part = nullptr);

}  // namespace skps
