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
// skps_face_src per face (faces of many images, or just the rectangle of an image a chip reads) or per group (the frame
// of a detector's slots), which may give any pixel layout of skps_b200.h: only the address of a tap depends on it, the
// chip is BGR.  The detector's five landmarks have an estimate of their own (det_align_estimate_kernel) that maps them
// back from the letterbox first.
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

// Least-squares similarity (rotation, uniform scale, translation; no reflection) mapping five points onto the template
// scaled by size/112; five(i) gives point i (template order) as a double2.  The 2-D closed form of Umeyama 1991: with
// centred points a_i (source) and b_i (template), scale*cos = sum(a.b) / sum|a|^2 and scale*sin = sum(a x b) / sum|a|^2.
// The one estimator of the library: the 98-point path (Five98) and the detector's five points (DetFive) both call it.
template <typename Five>
__device__ void similarity_to_template(const Five& five, int size, double* M) {
    const double sc = size / 112.0;
    double msx = 0, msy = 0, mdx = 0, mdy = 0;
#pragma unroll 1
    for (int i = 0; i < 5; ++i) {
        const double2 p = five(i);
        msx += p.x; msy += p.y;
        mdx += kTemplate112[2 * i] * sc; mdy += kTemplate112[2 * i + 1] * sc;
    }
    msx /= 5; msy /= 5; mdx /= 5; mdy /= 5;
    double dot = 0, cross = 0, den = 0;
#pragma unroll 1
    for (int i = 0; i < 5; ++i) {
        const double2 p = five(i);
        const double ax = p.x - msx, ay = p.y - msy;
        const double bx = kTemplate112[2 * i] * sc - mdx, by = kTemplate112[2 * i + 1] * sc - mdy;
        dot += ax * bx + ay * by;
        cross += ax * by - ay * bx;
        den += ax * ax + ay * ay;
    }
    const double a = den > 0 ? dot / den : 0.0, b = den > 0 ? cross / den : 0.0;
    M[0] = a; M[1] = -b; M[2] = mdx - (a * msx - b * msy);
    M[3] = b; M[4] = a;  M[5] = mdy - (b * msx + a * msy);
}

// The five alignment points kFive of WFLW-98 landmarks `kps` (P x 2) of type T, each promoted to double.
template <typename T>
struct Five98 {
    const T* kps;
    __device__ double2 operator()(int i) const {
        return make_double2((double)kps[2 * kFive[i]], (double)kps[2 * kFive[i] + 1]);
    }
};

// The five landmarks of a detector row (columns 5..14, letterbox coordinates) in frame pixels: scale_coords' float32
// (v - pad) / scale, the NMS gather's arithmetic for columns 0..3 (nms.cu), promoted to double.
struct DetFive {
    const float* lm;                            // row + 5
    float scale, left, top;
    __device__ float x(int i) const { return (lm[2 * i] - left) / scale; }
    __device__ float y(int i) const { return (lm[2 * i + 1] - top) / scale; }
    __device__ double2 operator()(int i) const { return make_double2((double)x(i), (double)y(i)); }
};

// cvRound on x86 (cvtsd2si): half to even; NaN or outside int32 -> INT_MIN
__device__ __forceinline__ int cv_round(double v) { return fabs(v) < 2147483647.5 ? __double2int_rn(v) : INT_MIN; }
// int32 addition with the two's-complement wrap OpenCV's int arithmetic has in practice
__device__ __forceinline__ int add_wrap(int a, int b) { return (int)((unsigned)a + (unsigned)b); }
__device__ __forceinline__ int sat_short(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }

struct WarpArgs {
    const uint8_t* frame; int H, W, pitch;      // the frame of every face (desc == null)
    const MpStreamDesc* desc;                   // or per group: desc[g].cur, H, W (pitch W*3)
    const skps_face_src* src;                   // or per group: src[g], taps outside its rectangle read 0,
    const skps_frame_layout* lay;               // its pixels laid out as lay[g] says (null: BGR)
    const double* M;                            // [faces][2][3] frame -> chip
    const int* count; int per_group;            // face f = g * per_group + i is skipped when count && i >= count[g]
    int out_h, out_w;
    uint8_t* out;                               // [faces][out_h][out_w][3]
    const int* turns;                           // with src: group g's image is stored turned turns[g] quarter turns
                                                // clockwise (align_warp_turned_kernel only)
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
    similarity_to_template(Five98<T>{kps + (size_t)f * P * 2}, size, m);
#pragma unroll
    for (int j = 0; j < 6; ++j) M[(size_t)f * 6 + j] = m[j];
}

// One thread per (frame f, slot j) of the detector's kept rows: rows (n, det_cap, 16) with count[f] rows kept, in NMS
// order.  Slot j < min(count[f], max_chips) gets its five landmarks (columns 5..14, letterbox coordinates) mapped back to
// the frame with recover[f] = (scale, left, top) exactly as the NMS gather maps columns 0..3 (scale_coords in float32),
// written to points[f][j] (5 x 2 float32), and M[f][j] from those points promoted to double.  Other slots are skipped.
__global__ void __launch_bounds__(128) det_align_estimate_kernel(const float* __restrict__ rows, const int* __restrict__ count,
                                                                 int det_cap, const float* __restrict__ recover, int n,
                                                                 int max_chips, int size, float* __restrict__ points,
                                                                 double* __restrict__ M) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)n * max_chips) return;
    const int f = (int)(t / max_chips), j = (int)(t - (long long)f * max_chips);
    if (j >= count[f]) return;
    const DetFive five{rows + ((size_t)f * det_cap + j) * 16 + 5, recover[3 * f], recover[3 * f + 1], recover[3 * f + 2]};
    float* pt = points + (size_t)t * 10;
#pragma unroll
    for (int i = 0; i < 5; ++i) { pt[2 * i] = five.x(i); pt[2 * i + 1] = five.y(i); }
    double m[6];
    similarity_to_template(five, size, m);
#pragma unroll
    for (int k = 0; k < 6; ++k) M[(size_t)t * 6 + k] = m[k];
}

// A block warps 256 consecutive pixels of one chip: each thread finds its pixel's four taps and weights once and blends the
// three channels into shared memory, then the block stores the 768 bytes with consecutive threads on consecutive bytes.
// TURNED: a source image is stored turned a.turns[g] quarter turns clockwise, read through px_view as the upright image; a
// turned image is read whole, one of turn 0 may be a rectangle as without TURNED.
template <bool TURNED>
__device__ __forceinline__ void warp_chip(const WarpArgs& a) {
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
        PxView v;
        if (a.desc) {
            const MpStreamDesc& d = a.desc[g];
            base = d.cur; H = d.H; W = d.W; pitch = d.W * 3; rw = W; rh = H;
        } else if (a.src) {
            const skps_face_src& s = a.src[g];
            base = s.base; H = s.H; W = s.W; pitch = s.pitch; ox = s.ox; oy = s.oy; rw = s.rw; rh = s.rh;
            if (a.lay) lay = px_layout(a.lay[g].layout, a.lay[g].plane_pitch);
        }
        if constexpr (TURNED) {
            const skps_frame_layout L = a.src && a.lay ? a.lay[g] : skps_frame_layout{SKPS_LAYOUT_BGR, 0};
            const int t = a.src ? a.turns[g] & 3 : 0;
            v = px_view(L.layout, L.plane_pitch, pitch, H, W, t);
            if (t) { H = v.H; W = v.W; ox = oy = 0; rw = W; rh = H; }
            else v.org = -((long long)oy * pitch + (long long)ox * v.xstep);
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
        if constexpr (TURNED) {
            const uint8_t* r0 = base + v.org + (long long)sy * v.ystep + (long long)sx * v.xstep;   // dereferenced only where inside
            const uint8_t* r1 = r0 + v.ystep;
            const long long xs = v.xstep;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const uint8_t* p0 = r0 + v.off[c];
                const uint8_t* p1 = r1 + v.off[c];
                const int acc = (y0 && x0 ? (int)__ldg(p0) : 0) * w00 + (y0 && x1 ? (int)__ldg(p0 + xs) : 0) * w01 +
                                (y1 && x0 ? (int)__ldg(p1) : 0) * w10 + (y1 && x1 ? (int)__ldg(p1 + xs) : 0) * w11;
                px[threadIdx.x * 3 + c] = (uint8_t)min((acc + 512) >> 10, 255);
            }
        } else {
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
    }
    __syncthreads();
    const int first = blockIdx.x * 256 * 3, n = min(256, pixels - blockIdx.x * 256) * 3;
    uint8_t* out = a.out + (size_t)f * pixels * 3 + first;
    for (int j = threadIdx.x; j < n; j += 256) out[j] = px[j];
}
__global__ void __launch_bounds__(256) align_warp_kernel(const WarpArgs a) { warp_chip<false>(a); }
__global__ void __launch_bounds__(256) align_warp_turned_kernel(const WarpArgs a) { warp_chip<true>(a); }

int launch_warp(const WarpArgs& a, int faces, cudaStream_t s) {
    const int pixels = a.out_w * a.out_h;
    const dim3 grid((pixels + 255) / 256, faces);
    if (a.src && a.turns) align_warp_turned_kernel<<<grid, 256, 0, s>>>(a);
    else align_warp_kernel<<<grid, 256, 0, s>>>(a);
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

extern "C" SKPS_API int skps_warp_faces_rotate(const skps_face_src* src, const skps_frame_layout* lay, const int32_t* turns,
                                               const double* M, int n, int out_h, int out_w, uint8_t* out, void* stream) {
    SKPS_CHECK(n >= 0 && out_h > 0 && out_w > 0 && out_h <= 4096 && out_w <= 4096,
               "warp_faces: n %d or output %dx%d out of range", n, out_h, out_w);
    if (n == 0) return 0;
    SKPS_CHECK(src && M && out, "warp_faces: bad arguments");
    // grid.y is the face: chunks of at most 65535 faces
    for (int c0 = 0; c0 < n; c0 += 65535) {
        const int m = min(65535, n - c0);
        WarpArgs a = {};
        a.src = src + c0; a.lay = lay ? lay + c0 : nullptr; a.M = M + (size_t)c0 * 6; a.per_group = 1;   // a source per face
        a.turns = turns ? turns + c0 : nullptr;
        a.out_h = out_h; a.out_w = out_w; a.out = out + (size_t)c0 * out_h * out_w * 3;
        if (launch_warp(a, m, (cudaStream_t)stream)) return 1;
    }
    return 0;
}

extern "C" SKPS_API int skps_warp_faces_layout(const skps_face_src* src, const skps_frame_layout* lay, const double* M, int n,
                                               int out_h, int out_w, uint8_t* out, void* stream) {
    return skps_warp_faces_rotate(src, lay, nullptr, M, n, out_h, out_w, out, stream);
}

extern "C" SKPS_API int skps_warp_faces_count_rotate(const skps_face_src* src, const skps_frame_layout* lay,
                                                     const int32_t* turns, const int32_t* count, int n_frames, int per_frame,
                                                     const double* M, int out_h, int out_w, uint8_t* out, void* stream) {
    SKPS_CHECK(n_frames >= 0 && per_frame > 0 && per_frame <= 65535 && out_h > 0 && out_w > 0 && out_h <= 4096 &&
               out_w <= 4096, "warp_faces_count: n_frames %d, per_frame %d or output %dx%d out of range", n_frames,
               per_frame, out_h, out_w);
    if (n_frames == 0) return 0;
    SKPS_CHECK(src && count && M && out, "warp_faces_count: bad arguments");
    // grid.y is the slot: chunks of whole frames, at most 65535 slots each
    const int step = 65535 / per_frame;
    const size_t chip = (size_t)out_h * out_w * 3;
    for (int g0 = 0; g0 < n_frames; g0 += step) {
        const int m = min(step, n_frames - g0);
        const size_t f0 = (size_t)g0 * per_frame;
        WarpArgs a = {};
        a.src = src + g0; a.lay = lay ? lay + g0 : nullptr; a.M = M + f0 * 6;
        a.turns = turns ? turns + g0 : nullptr;
        a.count = count + g0; a.per_group = per_frame;
        a.out_h = out_h; a.out_w = out_w; a.out = out + f0 * chip;
        if (launch_warp(a, m * per_frame, (cudaStream_t)stream)) return 1;
    }
    return 0;
}

extern "C" SKPS_API int skps_warp_faces_count(const skps_face_src* src, const skps_frame_layout* lay, const int32_t* count,
                                              int n_frames, int per_frame, const double* M, int out_h, int out_w,
                                              uint8_t* out, void* stream) {
    return skps_warp_faces_count_rotate(src, lay, nullptr, count, n_frames, per_frame, M, out_h, out_w, out, stream);
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

extern "C" SKPS_API int skps_det_align_estimate(const float* rows, const int32_t* count, int det_cap, const float* recover,
                                                int n_frames, int max_chips, int size, float* points, double* M,
                                                void* stream) {
    SKPS_CHECK(n_frames >= 0 && max_chips > 0 && max_chips <= det_cap,
               "det_align_estimate: n_frames %d or max_chips %d out of range (det_cap %d)", n_frames, max_chips, det_cap);
    SKPS_CHECK(size >= 16 && size <= 512, "det_align_estimate: size %d outside 16..512", size);
    if (n_frames == 0) return 0;
    SKPS_CHECK(rows && count && recover && points && M, "det_align_estimate: bad arguments");
    const long long slots = (long long)n_frames * max_chips;
    det_align_estimate_kernel<<<(unsigned)((slots + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        rows, count, det_cap, recover, n_frames, max_chips, size, points, M);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}
