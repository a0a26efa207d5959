// Aligned face chips: the least-squares similarity from five of the 98 landmarks to the ArcFace five-point template, and
// the warp of the frame into a size x size chip, bit for bit what
//     cv2.warpAffine(frame, M, (size, size), flags=INTER_LINEAR, borderMode=BORDER_CONSTANT, borderValue=0)
// writes.  OpenCV's classic path (imgwarp.cpp): the inverse map in double, source coordinates in 1/1024 px (cvRound)
// reduced to 1/32 px, integer bilinear weights (32-i)(32-j)*32 ... summing to 2^15, (sum + 2^14) >> 15.  Compiled with
// -fmad=false: every double expression rounds as written, like OpenCV's and numpy's (oracle/align_ref.py).
//
// Two launches cover every face of every frame of a call: the estimate (a thread per face), then the warp (grid.y = face,
// grid.x = runs of 256 pixels of the face's chip, stored with consecutive threads on consecutive bytes).  The frame is
// read where it lies.  A face's source is one frame for all faces, one MpStreamDesc per group of faces, or one
// skps_face_src per face (faces of many images, or just the rectangle of an image a chip reads), which may give any pixel
// layout of skps_b200.h: only the address of a tap depends on it, the chip is BGR.
#include <limits.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "mpipe_kernels.h"

namespace skps {
namespace {

// ArcFace 112x112 template (left eye, right eye, nose tip, left / right mouth corner) and the WFLW-98 indices of the same
// points; left / right as seen in the image
__constant__ double kTemplate112[10] = {38.2946, 51.6963, 73.5318, 51.5014, 56.0252, 71.7366,
                                        41.5493, 92.3655, 70.7299, 92.2041};
__constant__ int kFive[5] = {96, 97, 54, 76, 82};

// Least-squares similarity (rotation, uniform scale, translation; no reflection) mapping the five landmarks of `kps`
// (P x 2) onto the template scaled by size/112.  The 2-D closed form of Umeyama 1991: with centred points a_i (source)
// and b_i (template), scale*cos = sum(a.b) / sum|a|^2 and scale*sin = sum(a x b) / sum|a|^2.
// T: the landmarks' type, each promoted to double as it is read.
template <typename T>
__device__ void similarity_to_template(const T* __restrict__ kps, int size, double* M) {
    const double sc = size / 112.0;
    double msx = 0, msy = 0, mdx = 0, mdy = 0;
#pragma unroll 1
    for (int i = 0; i < 5; ++i) {
        msx += (double)kps[2 * kFive[i]]; msy += (double)kps[2 * kFive[i] + 1];
        mdx += kTemplate112[2 * i] * sc; mdy += kTemplate112[2 * i + 1] * sc;
    }
    msx /= 5; msy /= 5; mdx /= 5; mdy /= 5;
    double dot = 0, cross = 0, den = 0;
#pragma unroll 1
    for (int i = 0; i < 5; ++i) {
        const double ax = (double)kps[2 * kFive[i]] - msx, ay = (double)kps[2 * kFive[i] + 1] - msy;
        const double bx = kTemplate112[2 * i] * sc - mdx, by = kTemplate112[2 * i + 1] * sc - mdy;
        dot += ax * bx + ay * by;
        cross += ax * by - ay * bx;
        den += ax * ax + ay * ay;
    }
    const double a = den > 0 ? dot / den : 0.0, b = den > 0 ? cross / den : 0.0;
    M[0] = a; M[1] = -b; M[2] = mdx - (a * msx - b * msy);
    M[3] = b; M[4] = a;  M[5] = mdy - (b * msx + a * msy);
}

// cvRound on x86 (cvtsd2si): half to even; NaN or outside int32 -> INT_MIN
__device__ __forceinline__ int cv_round(double v) { return fabs(v) < 2147483647.5 ? __double2int_rn(v) : INT_MIN; }
// int32 addition with the two's-complement wrap OpenCV's int arithmetic has in practice
__device__ __forceinline__ int add_wrap(int a, int b) { return (int)((unsigned)a + (unsigned)b); }
__device__ __forceinline__ int sat_short(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }

struct WarpArgs {
    const uint8_t* frame; int H, W, pitch;      // the frame of every face (desc == null)
    const MpStreamDesc* desc;                   // or per group: desc[g].cur, H, W (pitch W*3)
    const skps_face_src* src;                   // or per face: src[f], taps outside its rectangle read 0,
    const skps_frame_layout* lay;               // its pixels laid out as lay[f] says (null: BGR)
    const double* M;                            // [faces][2][3] frame -> chip
    const int* count; int per_group;            // face f = g * per_group + i is skipped when count && i >= count[g]
    int out_h, out_w;
    uint8_t* out;                               // [faces][out_h][out_w][3]
};

// One thread per face: M[f] from the landmarks kps[f] (P x 2).
template <typename T>
__global__ void __launch_bounds__(128) align_estimate_kernel(const T* __restrict__ kps, int P, const int* __restrict__ count,
                                                             int per_group, int faces, int size, double* __restrict__ M) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= faces) return;
    const int g = f / per_group, i = f - g * per_group;
    if (count && i >= count[g]) return;
    double m[6];
    similarity_to_template(kps + (size_t)f * P * 2, size, m);
#pragma unroll
    for (int j = 0; j < 6; ++j) M[(size_t)f * 6 + j] = m[j];
}

// A block warps 256 consecutive pixels of one chip: each thread finds its pixel's four taps and weights once and blends the
// three channels into shared memory, then the block stores the 768 bytes with consecutive threads on consecutive bytes.
__global__ void __launch_bounds__(256) align_warp_kernel(const WarpArgs a) {
    const int f = blockIdx.y;
    const int g = f / a.per_group, i = f - g * a.per_group;
    if (a.count && i >= a.count[g]) return;
    __shared__ uint8_t px[256 * 3];
    const int pixels = a.out_w * a.out_h;
    const int p = blockIdx.x * 256 + threadIdx.x;
    if (p < pixels) {
        // base holds the rectangle of an H x W image at column ox, row oy, rw x rh pixels
        const uint8_t* base = a.frame;
        int H = a.H, W = a.W, pitch = a.pitch, ox = 0, oy = 0, rw = a.W, rh = a.H;
        PxLayout lay = px_layout(SKPS_LAYOUT_BGR, 0);
        if (a.desc) {
            const MpStreamDesc& d = a.desc[g];
            base = d.cur; H = d.H; W = d.W; pitch = d.W * 3; rw = W; rh = H;
        } else if (a.src) {
            const skps_face_src& s = a.src[f];
            base = s.base; H = s.H; W = s.W; pitch = s.pitch; ox = s.ox; oy = s.oy; rw = s.rw; rh = s.rh;
            if (a.lay) lay = px_layout(a.lay[f].layout, a.lay[f].plane_pitch);
        }
        const int xa = max(ox, 0), xb = min(ox + rw, W), ya = max(oy, 0), yb = min(oy + rh, H);
        // the inverse map as warpAffine computes it (imgwarp.cpp), same order of operations; every thread of the face
        // computes the same values
        const double* Mf = a.M + (size_t)f * 6;
        double m0 = __ldg(Mf), m1 = __ldg(Mf + 1), m2 = __ldg(Mf + 2), m3 = __ldg(Mf + 3), m4 = __ldg(Mf + 4), m5 = __ldg(Mf + 5);
        double D = m0 * m4 - m1 * m3;
        D = D != 0.0 ? 1.0 / D : 0.0;
        const double A11 = m4 * D, A22 = m0 * D;
        m0 = A11; m4 = A22;
        m1 *= -D; m3 *= -D;
        const double b1 = -m0 * m2 - m1 * m5, b2 = -m3 * m2 - m4 * m5;
        m2 = b1; m5 = b2;
        const int y = p / a.out_w, x = p - y * a.out_w;
        // AB_SCALE = 1024, round_delta = 1024 / 32 / 2; source position in 1/32 px
        const int X0 = add_wrap(cv_round((m1 * y + m2) * 1024.0), 16);
        const int Y0 = add_wrap(cv_round((m4 * y + m5) * 1024.0), 16);
        const int X = add_wrap(X0, cv_round(m0 * x * 1024.0)) >> 5;
        const int Y = add_wrap(Y0, cv_round(m3 * x * 1024.0)) >> 5;
        const int sx = sat_short(X >> 5), sy = sat_short(Y >> 5);
        const int fx = X & 31, fy = Y & 31;
        const int w00 = (32 - fx) * (32 - fy), w01 = fx * (32 - fy), w10 = (32 - fx) * fy, w11 = fx * fy;
        // taps outside the frame read the border value 0; so do taps outside the rectangle, which are never dereferenced
        const bool x0 = sx >= xa && sx < xb, x1 = sx + 1 >= xa && sx + 1 < xb;
        const bool y0 = sy >= ya && sy < yb, y1 = sy + 1 >= ya && sy + 1 < yb;
        const uint8_t* r0 = base + (ptrdiff_t)(sy - oy) * pitch + (ptrdiff_t)(sx - ox) * lay.xs;   // dereferenced only where inside
        const uint8_t* r1 = r0 + pitch;
        const int xs = lay.xs;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const uint8_t* p0 = r0 + lay.off[c];
            const uint8_t* p1 = r1 + lay.off[c];
            const int acc = (y0 && x0 ? (int)__ldg(p0) : 0) * w00 + (y0 && x1 ? (int)__ldg(p0 + xs) : 0) * w01 +
                            (y1 && x0 ? (int)__ldg(p1) : 0) * w10 + (y1 && x1 ? (int)__ldg(p1 + xs) : 0) * w11;
            // weights * 32 sum to 2^15: (sum * 32 + 2^14) >> 15 == (sum + 2^9) >> 10; at most 255
            px[threadIdx.x * 3 + c] = (uint8_t)min((acc + 512) >> 10, 255);
        }
    }
    __syncthreads();
    const int first = blockIdx.x * 256 * 3, n = min(256, pixels - blockIdx.x * 256) * 3;
    uint8_t* out = a.out + (size_t)f * pixels * 3 + first;
    for (int j = threadIdx.x; j < n; j += 256) out[j] = px[j];
}

int launch_warp(const WarpArgs& a, int faces, cudaStream_t s) {
    const int pixels = a.out_w * a.out_h;
    align_warp_kernel<<<dim3((pixels + 255) / 256, faces), 256, 0, s>>>(a);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

// estimate (one launch, a thread per face) then warp (one launch, a thread per output byte)
int launch_align(const uint8_t* frame, int H, int W, int pitch, const MpStreamDesc* desc, const double* kps, int P,
                 const int* count, int per_group, int faces, int size, uint8_t* chips, double* M, cudaStream_t s) {
    align_estimate_kernel<double><<<(faces + 127) / 128, 128, 0, s>>>(kps, P, count, per_group, faces, size, M);
    SKPS_CUDA(cudaGetLastError());
    WarpArgs a = {};
    a.frame = frame; a.H = H; a.W = W; a.pitch = pitch; a.desc = desc;
    a.M = M; a.count = count; a.per_group = per_group;
    a.out_h = a.out_w = size; a.out = chips;
    return launch_warp(a, faces, s);
}

}  // namespace

int launch_mp_align(const MpStreamDesc* d, const double* kps, const int* count, int K, int P, int size, uint8_t* chips,
                    double* M, int n, cudaStream_t s) {
    return launch_align(nullptr, 0, 0, 0, d, kps, P, count, K, K * n, size, chips, M, s);
}

}  // namespace skps

using namespace skps;

extern "C" SKPS_API int skps_warp_affine(const uint8_t* frame, int H, int W, int pitch, const double* M, const int32_t* count,
                                         int n, int out_h, int out_w, uint8_t* out, void* stream) {
    SKPS_CHECK(frame && M && out && H > 0 && W > 0 && pitch >= 3 * W, "warp_affine: bad arguments");
    SKPS_CHECK(n > 0 && n <= 65535 && out_h > 0 && out_w > 0 && out_h <= 4096 && out_w <= 4096,
               "warp_affine: n %d or output %dx%d out of range", n, out_h, out_w);
    WarpArgs a = {};
    a.frame = frame; a.H = H; a.W = W; a.pitch = pitch;
    a.M = M; a.count = count; a.per_group = n;
    a.out_h = out_h; a.out_w = out_w; a.out = out;
    return launch_warp(a, n, (cudaStream_t)stream);
}

extern "C" SKPS_API int skps_align_faces(const uint8_t* frame, int H, int W, int pitch, const double* kps, const int32_t* count,
                                         int n, int P, int size, uint8_t* chips, double* M, void* stream) {
    SKPS_CHECK(frame && kps && chips && M && H > 0 && W > 0 && pitch >= 3 * W, "align_faces: bad arguments");
    SKPS_CHECK(n > 0 && n <= 65535 && P >= 98, "align_faces: n %d or n_points %d out of range", n, P);
    SKPS_CHECK(size >= 16 && size <= 512, "align_faces: size %d outside 16..512", size);
    return launch_align(frame, H, W, pitch, nullptr, kps, P, count, n, n, size, chips, M, (cudaStream_t)stream);
}

extern "C" SKPS_API int skps_warp_faces_layout(const skps_face_src* src, const skps_frame_layout* lay, const double* M, int n,
                                               int out_h, int out_w, uint8_t* out, void* stream) {
    SKPS_CHECK(n >= 0 && out_h > 0 && out_w > 0 && out_h <= 4096 && out_w <= 4096,
               "warp_faces: n %d or output %dx%d out of range", n, out_h, out_w);
    if (n == 0) return 0;
    SKPS_CHECK(src && M && out, "warp_faces: bad arguments");
    // grid.y is the face: chunks of at most 65535 faces
    for (int c0 = 0; c0 < n; c0 += 65535) {
        const int m = min(65535, n - c0);
        WarpArgs a = {};
        a.src = src + c0; a.lay = lay ? lay + c0 : nullptr; a.M = M + (size_t)c0 * 6; a.per_group = m;
        a.out_h = out_h; a.out_w = out_w; a.out = out + (size_t)c0 * out_h * out_w * 3;
        if (launch_warp(a, m, (cudaStream_t)stream)) return 1;
    }
    return 0;
}

extern "C" SKPS_API int skps_warp_faces(const skps_face_src* src, const double* M, int n, int out_h, int out_w, uint8_t* out,
                                        void* stream) {
    return skps_warp_faces_layout(src, nullptr, M, n, out_h, out_w, out, stream);
}

extern "C" SKPS_API int skps_align_estimate(const float* kps, int n, int P, int size, double* M, void* stream) {
    SKPS_CHECK(n >= 0 && P >= 98, "align_estimate: n %d or n_points %d out of range", n, P);
    SKPS_CHECK(size >= 16 && size <= 512, "align_estimate: size %d outside 16..512", size);
    if (n == 0) return 0;
    SKPS_CHECK(kps && M, "align_estimate: bad arguments");
    align_estimate_kernel<float><<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(kps, P, nullptr, n, n, size, M);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}
