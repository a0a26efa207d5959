// Image-side kernels of the FaceAna path (sm_90a): letterbox, per-face crop+resize (both bit-exact
// with cv2.resize INTER_LINEAR on uint8), face selection (IoU track match + EMA, area filter, top-k), landmark
// de-normalisation and the frame-difference gate.  All HBM-bound byte/index work; compiled with
// -fmad=false so float32 expressions round exactly like the numpy expressions they restate.
#include <string.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "mpipe_kernels.h"

namespace skps {

// ------------------------------------------------------------------------------------------
// cv2.resize(INTER_LINEAR, uint8) tap: OpenCV resize.cpp (called from face_detector.py:53 and
// face_landmark.py:97).  scale = 1/(dst/src) in double, offset rounded to float32, weights
// rint(w*2048) (INTER_RESIZE_COEF_BITS = 11).
// ------------------------------------------------------------------------------------------
struct Tap { int i0, i1, w0, w1; };

__device__ __forceinline__ Tap linear_tap(int d, int dst, int src, bool is_x) {
    double scale = 1.0 / ((double)dst / (double)src);
    float f = (float)(((double)d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f = f - (float)s;
    Tap t;
    if (is_x) {
        if (s < 0) { s = 0; f = 0.f; }
        if (s >= src - 1) { s = src - 1; f = 0.f; }
        t.i0 = s;
        t.i1 = min(s + 1, src - 1);
    } else {
        t.i0 = min(max(s, 0), src - 1);
        t.i1 = min(max(s + 1, 0), src - 1);
    }
    t.w0 = __float2int_rn((1.f - f) * 2048.f);
    t.w1 = __float2int_rn(f * 2048.f);
    return t;
}

__device__ __forceinline__ int vblend(int h0, int h1, int b0, int b1) {
    return (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
}

// ------------------------------------------------------------------------------------------
// Letterbox (face_detector.py:45-71): BGR->RGB, resize to (rw,rh), pad 114.  One thread per
// output pixel (3 channels); output is uint8 RGB NHWC, /255 happens in the first conv.
// ------------------------------------------------------------------------------------------
// `frame` holds the whole frame, or with row_pairs only the two rows each resized row reads: rows 2 dy and 2 dy + 1.
__device__ __forceinline__ void letterbox_px(const uint8_t* __restrict__ frame, int H, int W, int pitch, int row_pairs,
                                             uint8_t* __restrict__ out, int in_h, int in_w, int rw, int rh, int top, int left,
                                             int x, int y) {
    if (x >= in_w) return;
    uint8_t* o = out + ((long long)y * in_w + x) * 3;
    int dx = x - left, dy = y - top;
    if (dx < 0 || dx >= rw || dy < 0 || dy >= rh) {
        o[0] = 114; o[1] = 114; o[2] = 114;
        return;
    }
    Tap tx = linear_tap(dx, rw, W, true);
    Tap ty = linear_tap(dy, rh, H, false);
    const uint8_t* r0 = frame + (long long)(row_pairs ? 2 * dy : ty.i0) * pitch;
    const uint8_t* r1 = frame + (long long)(row_pairs ? 2 * dy + 1 : ty.i1) * pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        int h0 = r0[tx.i0 * 3 + c] * tx.w0 + r0[tx.i1 * 3 + c] * tx.w1;
        int h1 = r1[tx.i0 * 3 + c] * tx.w0 + r1[tx.i1 * 3 + c] * tx.w1;
        o[2 - c] = (uint8_t)vblend(h0, h1, ty.w0, ty.w1);      // BGR -> RGB
    }
}
// block z = frame
__global__ void __launch_bounds__(256) letterbox_frames_kernel(const LetterboxArgs a) {
    const uint8_t* frame = a.frame;
    int H = a.H, W = a.W, pitch = a.pitch, rw = a.rw, rh = a.rh, top = a.top, left = a.left, row_pairs = 0;
    if (a.desc) {
        const MpStreamDesc D = a.desc[blockIdx.z];
        frame = D.cur; H = D.H; W = D.W; pitch = D.W * 3; rw = D.rw; rh = D.rh; top = D.top; left = D.left;
    } else if (a.src) {
        const skps_det_src F = a.src[blockIdx.z];
        frame = F.base; H = F.H; W = F.W; pitch = F.pitch; rw = F.rw; rh = F.rh; top = F.top; left = F.left;
        row_pairs = F.row_pairs;
    }
    letterbox_px(frame, H, W, pitch, row_pairs, a.out + a.out_stride * blockIdx.z, a.in_h, a.in_w, rw, rh, top, left,
                 blockIdx.x * blockDim.x + threadIdx.x, blockIdx.y);
}

// ------------------------------------------------------------------------------------------
// Per-face crop + resize (face_landmark.py:74-98).  Geometry in float32 exactly as numpy>=2
// evaluates it; the zero border of copyMakeBorder is virtual.
// ------------------------------------------------------------------------------------------
struct CropGeo { int add, x1, y1, w, h, ok; };

__device__ __forceinline__ CropGeo crop_geometry(const float* b, int H, int W, float face_scale, float min_face) {
    CropGeo g;
    float bw = b[2] - b[0], bh = b[3] - b[1];
    g.ok = !(bw <= min_face || bh <= min_face);
    int add = (int)fmaxf(bw, bh);
    float fa = (float)add;
    float x0 = b[0] + fa, y0 = b[1] + fa, x1 = b[2] + fa, y1 = b[3] + fa;
    float fw = face_scale * bw;
    float cx = floorf((x0 + x1) / 2.f), cy = floorf((y0 + y1) / 2.f);
    float half = floorf(fw / 2.f);
    int ix1 = (int)(cx - half), iy1 = (int)(cy - half), ix2 = (int)(cx + half), iy2 = (int)(cy + half);
    // numpy slicing of the padded frame clamps the ends (negative starts are not meaningful in the
    // reference either; clamp them to 0)
    int PW = W + 2 * add, PH = H + 2 * add;
    ix1 = max(ix1, 0); iy1 = max(iy1, 0);
    ix2 = min(ix2, PW); iy2 = min(iy2, PH);
    g.add = add; g.x1 = ix1; g.y1 = iy1;
    g.w = max(ix2 - ix1, 0); g.h = max(iy2 - iy1, 0);
    if (g.w <= 0 || g.h <= 0) g.ok = 0;
    return g;
}

// Output pixel (x, y) of the crop of one face with box b into o, and at (0, 0) its detail d = [h, w, y1, x1, add].  The
// frame is H x W; `base` holds only its rectangle starting at column ox, row oy, rows `pitch` bytes apart.  Whether a tap
// is in the frame or in the zero border is decided against the whole frame, so a caller that holds only the rectangle
// the taps can reach gets the same bytes as one that holds the whole frame (ox = oy = 0).
__device__ __forceinline__ void crop_face_px(const uint8_t* __restrict__ base, int H, int W, int pitch, int ox, int oy,
                                             const float* __restrict__ b, float face_scale, float min_face,
                                             uint8_t* __restrict__ o, int S, int* __restrict__ d, int x, int y) {
    CropGeo g = crop_geometry(b, H, W, face_scale, min_face);
    if (x == 0 && y == 0) {
        d[0] = g.h; d[1] = g.w; d[2] = g.y1; d[3] = g.x1; d[4] = g.add;
    }
    if (!g.ok) { o[0] = 0; o[1] = 0; o[2] = 0; return; }
    Tap tx = linear_tap(x, S, g.w, true);
    Tap ty = linear_tap(y, S, g.h, false);
    // crop coordinates -> frame coordinates (outside the frame = the zero border)
    int fx0 = g.x1 + tx.i0 - g.add, fx1 = g.x1 + tx.i1 - g.add;
    int fy0 = g.y1 + ty.i0 - g.add, fy1 = g.y1 + ty.i1 - g.add;
    bool vx0 = fx0 >= 0 && fx0 < W, vx1 = fx1 >= 0 && fx1 < W;
    bool vy0 = fy0 >= 0 && fy0 < H, vy1 = fy1 >= 0 && fy1 < H;
    const uint8_t* r0 = base + (long long)((vy0 ? fy0 : oy) - oy) * pitch;
    const uint8_t* r1 = base + (long long)((vy1 ? fy1 : oy) - oy) * pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        int p00 = (vy0 && vx0) ? r0[(fx0 - ox) * 3 + c] : 0, p01 = (vy0 && vx1) ? r0[(fx1 - ox) * 3 + c] : 0;
        int p10 = (vy1 && vx0) ? r1[(fx0 - ox) * 3 + c] : 0, p11 = (vy1 && vx1) ? r1[(fx1 - ox) * 3 + c] : 0;
        int h0 = p00 * tx.w0 + p01 * tx.w1;
        int h1 = p10 * tx.w0 + p11 * tx.w1;
        o[c] = (uint8_t)vblend(h0, h1, ty.w0, ty.w1);          // stays BGR (face_landmark.py:44)
    }
}

__device__ __forceinline__ void crop_px(const uint8_t* __restrict__ frame, int H, int W, int pitch,
                                        const float* __restrict__ boxes, const int* __restrict__ count, float face_scale,
                                        float min_face, uint8_t* __restrict__ crops, int S, int* __restrict__ detail,
                                        int face, int x, int y) {
    if (x >= S) return;
    uint8_t* o = crops + (((long long)face * S + y) * S + x) * 3;
    const int n = *count;
    if (face >= n) {
        o[0] = 0; o[1] = 0; o[2] = 0;
        if (x == 0 && y == 0) { for (int k = 0; k < 5; ++k) detail[face * 5 + k] = 0; }
        return;
    }
    crop_face_px(frame, H, W, pitch, 0, 0, boxes + face * 4, face_scale, min_face, o, S, detail + face * 5, x, y);
}
// block z = face of a frame (K per frame)
__global__ void __launch_bounds__(256) crop_frames_kernel(const CropArgs a) {
    const int g = blockIdx.z / a.K, face = blockIdx.z - g * a.K;
    const uint8_t* frame = a.frame;
    int H = a.H, W = a.W, pitch = a.pitch;
    if (a.desc) {
        const MpStreamDesc D = a.desc[g];
        frame = D.cur; H = D.H; W = D.W; pitch = D.W * 3;
    }
    crop_px(frame, H, W, pitch, a.boxes + (size_t)4 * a.K * g, a.count + g, a.face_scale, a.min_face,
            a.crops + (size_t)a.S * a.S * 3 * a.K * g, a.S, a.detail + (size_t)5 * a.K * g, face,
            blockIdx.x * blockDim.x + threadIdx.x, blockIdx.y);
}
// Face table variant (FaceLandmark.submit): block z = face, each face with its own frame or frame rectangle.
__global__ void __launch_bounds__(256) crop_faces_kernel(const skps_face_src* __restrict__ src, const float* __restrict__ boxes,
                                                         float face_scale, float min_face, uint8_t* __restrict__ crops, int S,
                                                         int* __restrict__ detail) {
    const int face = blockIdx.z, x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= S) return;
    const skps_face_src F = src[face];
    crop_face_px(F.base, F.H, F.W, F.pitch, F.ox, F.oy, boxes + face * 4, face_scale, min_face,
                 crops + (((long long)face * S + y) * S + x) * 3, S, detail + face * 5, x, y);
}

// ------------------------------------------------------------------------------------------
// Rectangular crop + resize of one image (WFLW evaluation, TRAIN/face_landmark/tools/eval_WFLW.py:38-80,113-124:
// copyMakeBorder(zero) -> img[min_y:max_y, min_x:max_x] -> cv2.resize((S, S))).  rect = [x0, y0, w, h] in frame
// coordinates; pixels outside the frame are the zero border.  Same fixed-point bilinear as above, bit-exact with OpenCV.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rect_resize_kernel(const uint8_t* __restrict__ frame, int H, int W, int pitch,
                                                          int rx, int ry, int rw, int rh, uint8_t* __restrict__ out, int S) {
    const int y = blockIdx.y;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= S) return;
    uint8_t* o = out + ((long long)y * S + x) * 3;
    Tap tx = linear_tap(x, S, rw, true);
    Tap ty = linear_tap(y, S, rh, false);
    int fx0 = rx + tx.i0, fx1 = rx + tx.i1, fy0 = ry + ty.i0, fy1 = ry + ty.i1;
    bool vx0 = fx0 >= 0 && fx0 < W, vx1 = fx1 >= 0 && fx1 < W;
    bool vy0 = fy0 >= 0 && fy0 < H, vy1 = fy1 >= 0 && fy1 < H;
    const uint8_t* r0 = frame + (long long)(vy0 ? fy0 : 0) * pitch;
    const uint8_t* r1 = frame + (long long)(vy1 ? fy1 : 0) * pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        int p00 = (vy0 && vx0) ? r0[fx0 * 3 + c] : 0, p01 = (vy0 && vx1) ? r0[fx1 * 3 + c] : 0;
        int p10 = (vy1 && vx0) ? r1[fx0 * 3 + c] : 0, p11 = (vy1 && vx1) ? r1[fx1 * 3 + c] : 0;
        o[c] = (uint8_t)vblend(p00 * tx.w0 + p01 * tx.w1, p10 * tx.w0 + p11 * tx.w1, ty.w0, ty.w1);
    }
}

// Normalised mean error per face (eval_WFLW.py:84-95): mean_p |pred_p - gt_p| / |gt_60 - gt_72| (inter-ocular), float32
// like numpy's; one warp per face.
__global__ void nme_kernel(const float* __restrict__ target, const float* __restrict__ preds, int n, int P, int ia, int ib,
                           float* __restrict__ out) {
    const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (f >= n) return;
    const float* t = target + (long long)f * P * 2;
    const float* q = preds + (long long)f * P * 2;
    float s = 0.f;
    for (int p = lane; p < P; p += 32) {
        const float dx = q[2 * p] - t[2 * p], dy = q[2 * p + 1] - t[2 * p + 1];
        s += sqrtf(dx * dx + dy * dy);
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
        const float nx = t[2 * ia] - t[2 * ib], ny = t[2 * ia + 1] - t[2 * ib + 1];
        out[f] = (s / (float)P) / sqrtf(nx * nx + ny * ny);
    }
}

// ------------------------------------------------------------------------------------------
// judge_boxs + sort_and_filter (facer.py:120-189).  One block of 256 threads per frame, any number of detections.
// (Detector post-processing, face_detector.py:31-37 and 73-136, is in nms.cu.)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float iou_track(const float* r1, const float* r2) {
    float s1 = (r1[2] - r1[0]) * (r1[3] - r1[1]);
    float s2 = (r2[2] - r2[0]) * (r2[3] - r2[1]);
    float sum = s1 + s2;
    float x1 = fmaxf(r1[0], r2[0]), y1 = fmaxf(r1[1], r2[1]);
    float x2 = fminf(r1[2], r2[2]), y2 = fminf(r1[3], r2[3]);
    float inter = fmaxf(0.f, x2 - x1) * fmaxf(0.f, y2 - y1);
    return inter / (sum - inter);
}

constexpr int SEL_THREADS = 256;
constexpr int SEL_CACHE = 8192;       // area orders kept in shared memory (32 KB); later detections recompute theirs
constexpr int SEL_MAX_K = SKPS_MAX_TOP_K;

// judge_boxs for one detection: the box after the EMA with the first track box it matches (facer.py:176-181, lk.py:95-96).
// Returns the index of that track box, -1 when none matches.
__device__ __forceinline__ int judged_box(const float* now, const float* __restrict__ track, int n_track, float iou_thres,
                                          float alpha, float oma, float b[4]) {
    b[0] = now[0]; b[1] = now[1]; b[2] = now[2]; b[3] = now[3];
    for (int j = 0; j < n_track; ++j) {
        const float* prev = track + j * 4;
        if (iou_track(now, prev) > iou_thres) {
            for (int c = 0; c < 4; ++c) b[c] = alpha * now[c] + oma * prev[c];
            return j;
        }
    }
    return -1;
}

// Selection key of detection i: 0 when its area fails the filter, else (area, i) as one integer with the order of
// "larger area first, ties by later index first" (facer.py:138 area.argsort()[-k:][::-1], a stable ascending sort read
// backwards).  +0.f turns an area of -0 into +0, which compares equal to it in float.
// The upper half of the key: 0 when the area fails the filter, else the area's bits in an unsigned order that sorts like
// the float.  ord >= 0x007fffff, so a passing key is never 0.
__device__ __forceinline__ unsigned select_ord(const float* __restrict__ det, int det_stride, int i,
                                               const float* __restrict__ track, int n_track, float iou_thres, float alpha,
                                               float oma, float min_face) {
    float b[4];
    judged_box(det + (long long)i * det_stride, track, n_track, iou_thres, alpha, oma, b);
    const float area = (b[2] - b[0]) * (b[3] - b[1]);
    if (!(area > min_face)) return 0u;
    const unsigned u = __float_as_uint(area + 0.f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ unsigned long long select_key(unsigned ord, int i) {
    return ord ? ((unsigned long long)ord << 32) | (unsigned)i : 0ull;
}

// Selection for any top_k <= SEL_MAX_K in a number of passes over the keys that does not grow with top_k: a radix select
// (8-bit digits, most significant first) finds the top_k-th largest key T, the keys >= T are gathered and bitonic-sorted
// descending.  Keys past the shared cache are recomputed once per pass.
// src, when not null, gets each selected face's source for the track ids: the row it was selected from when the rows are
// the previous track boxes (src_is_row, the gate-skipped frame of facer.py:61), else the track box its detection matched
// (-1 for none).
__device__ __forceinline__ void select_faces_body(const float* __restrict__ det, int n_det, int det_stride,
                                                  const float* __restrict__ track, int n_track, float iou_thres, float alpha,
                                                  float oma, float min_face, int top_k, float* __restrict__ boxes4,
                                                  int* __restrict__ count, int* __restrict__ src, bool src_is_row) {
    __shared__ unsigned s_ord[SEL_CACHE];
    __shared__ unsigned long long s_win[SEL_MAX_K];
    __shared__ int s_sel[SEL_MAX_K];
    __shared__ int s_hist[256];
    __shared__ int s_wcount[SEL_THREADS / 32];
    __shared__ int s_m, s_bin, s_krem, s_done;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    const int n = max(n_det, 0);
    auto key_of = [&](int i) {
        return select_key(i < SEL_CACHE ? s_ord[i]
                                        : select_ord(det, det_stride, i, track, n_track, iou_thres, alpha, oma, min_face), i);
    };
    if (tid == 0) s_m = 0;
    __syncthreads();
    int my_m = 0;
    for (int i = tid; i < n; i += nt) {
        const unsigned o = select_ord(det, det_stride, i, track, n_track, iou_thres, alpha, oma, min_face);
        if (i < SEL_CACHE) s_ord[i] = o;
        my_m += o != 0u;
    }
    if (my_m) atomicAdd(&s_m, my_m);
    __syncthreads();
    const int m_all = s_m;
    const int m = min(m_all, top_k);
    if (m_all <= top_k) {
        // every face passing the area filter, in detector order (facer.py:132-136)
        int off = 0;
        for (int base = 0; base < n; base += nt) {
            const int i = base + tid;
            const bool pass = i < n && key_of(i) != 0ull;
            const unsigned bal = __ballot_sync(0xffffffffu, pass);
            if (lane == 0) s_wcount[warp] = __popc(bal);
            __syncthreads();
            int before = off, total = off;
            for (int q = 0; q < nw; ++q) {
                if (q < warp) before += s_wcount[q];
                total += s_wcount[q];
            }
            if (pass) s_sel[before + __popc(bal & ((1u << lane) - 1))] = i;
            off = total;
            __syncthreads();
        }
    } else {
        // radix select of the top_k-th largest passing key; the passing keys are unique, so exactly top_k are >= it
        unsigned long long prefix = 0ull, mask = 0ull;
        int k_rem = top_k;
        for (int shift = 56; shift >= 0; shift -= 8) {
            for (int b = tid; b < 256; b += nt) s_hist[b] = 0;
            __syncthreads();
            for (int i = tid; i < n; i += nt) {
                const unsigned long long q = key_of(i);
                if (q != 0ull && (q & mask) == prefix) atomicAdd(&s_hist[(int)(q >> shift) & 255], 1);
            }
            __syncthreads();
            if (warp == 0) {
                // lane l owns digits 255-8l .. 248-8l; `above` = keys with a larger digit than the lane's first
                int c[8], sum = 0;
#pragma unroll
                for (int q = 0; q < 8; ++q) { c[q] = s_hist[255 - (lane * 8 + q)]; sum += c[q]; }
                int incl = sum;
                for (int o = 1; o < 32; o <<= 1) {
                    const int v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += v;
                }
                int above = incl - sum;
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    if (above < k_rem && above + c[q] >= k_rem) {
                        s_bin = 255 - (lane * 8 + q);
                        s_krem = k_rem - above;
                        s_done = above + c[q] == k_rem;       // every key with this digit is in: T has zero lower digits
                    }
                    above += c[q];
                }
            }
            __syncthreads();
            prefix |= (unsigned long long)s_bin << shift;
            mask |= 0xffull << shift;
            k_rem = s_krem;
            const bool done = s_done;
            __syncthreads();
            if (done) break;
        }
        // gather the top_k keys >= T (in any order), sort them descending
        if (tid == 0) s_m = 0;
        __syncthreads();
        for (int i = tid; i < n; i += nt) {
            const unsigned long long q = key_of(i);
            if (q != 0ull && q >= prefix) s_win[atomicAdd(&s_m, 1)] = q;
        }
        int np2 = 1;
        while (np2 < m) np2 <<= 1;
        __syncthreads();
        for (int i = m + tid; i < np2; i += nt) s_win[i] = 0ull;
        __syncthreads();
        for (int k = 2; k <= np2; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = tid; i < np2; i += nt) {
                    const int ixj = i ^ j;
                    if (ixj > i) {
                        const unsigned long long a = s_win[i], b = s_win[ixj];
                        if (((i & k) == 0) ? (a < b) : (a > b)) { s_win[i] = b; s_win[ixj] = a; }
                    }
                }
                __syncthreads();
            }
        }
        for (int i = tid; i < m; i += nt) s_sel[i] = (int)(unsigned)(s_win[i] & 0xffffffffull);
        __syncthreads();
    }
    if (tid == 0) *count = m;
    for (int f = tid; f < m; f += nt) {
        float b[4];
        const int j = judged_box(det + (long long)s_sel[f] * det_stride, track, n_track, iou_thres, alpha, oma, b);
        for (int c = 0; c < 4; ++c) boxes4[f * 4 + c] = b[c];
        if (src) src[f] = src_is_row ? s_sel[f] : j;
    }
}

// block = frame: judge_boxs(track, detector rows) when the frame ran the detector (facer.py:58), else its track boxes
// (facer.py:61), then sort_and_filter
__global__ void __launch_bounds__(256) select_frames_kernel(const SelectArgs a) {
    const int g = blockIdx.x;
    const float* trk = a.track + (size_t)g * a.top_k * 4;
    const int n_trk = a.track ? (a.n_track ? a.n_track[g] : a.n_track1) : 0;
    const bool det = a.flag ? a.flag[g] != 0 : a.flag1 != 0;
    const float* rows = trk;
    int n_rows = n_trk, stride = 4;
    if (det) {
        const int f = a.det_slot ? a.det_slot[g] : g;
        rows = a.det_rows + (size_t)f * a.det_cap * a.det_stride; n_rows = a.det_count[f]; stride = a.det_stride;
    }
    select_faces_body(rows, n_rows, stride, det ? trk : nullptr, det ? n_trk : 0, a.iou_thres, a.alpha, a.one_minus_alpha,
                      a.min_face, a.top_k, a.boxes4 + (size_t)g * a.top_k * 4, a.count + g,
                      a.src ? a.src + (size_t)g * a.top_k : nullptr, !det);
}

// The box FaceAna returns for a face on a frame with no history (facer.py:75-82): judge_boxs(boxes_return, rects(kps)),
// i.e. the face's landmark rectangle, EMA-blended with the first selected box of its image it overlaps with IoU >
// iou_thres.  One warp per face: the rectangle's min / max by shuffles, then judged_box.
__global__ void __launch_bounds__(256) landmark_boxes_kernel(const float* __restrict__ kps, int P,
                                                             const int* __restrict__ face_image, int n,
                                                             const float* __restrict__ sel_boxes,
                                                             const int* __restrict__ sel_count, int top_k, float iou_thres,
                                                             float alpha, float oma, float* __restrict__ out) {
    const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (f >= n) return;                             // whole warps leave together
    const float* p = kps + (size_t)f * P * 2;
    float x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
    for (int i = lane; i < P; i += 32) {
        const float x = p[2 * i], y = p[2 * i + 1];
        x0 = fminf(x0, x); y0 = fminf(y0, y); x1 = fmaxf(x1, x); y1 = fmaxf(y1, y);
    }
    for (int o = 16; o > 0; o >>= 1) {
        x0 = fminf(x0, __shfl_xor_sync(0xffffffffu, x0, o));
        y0 = fminf(y0, __shfl_xor_sync(0xffffffffu, y0, o));
        x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, o));
        y1 = fmaxf(y1, __shfl_xor_sync(0xffffffffu, y1, o));
    }
    if (lane == 0) {
        const int g = face_image[f];
        const float rect[4] = {x0, y0, x1, y1};
        float b[4];
        judged_box(rect, sel_boxes + (size_t)g * top_k * 4, sel_count[g], iou_thres, alpha, oma, b);
        for (int c = 0; c < 4; ++c) out[(size_t)f * 4 + c] = b[c];
    }
}

// ------------------------------------------------------------------------------------------
// FaceLandmark.postprocess (face_landmark.py:106-115): float32 product, then + x1 - add in
// float64, stored as float32 (numpy>=2 promotion of `float32 * int + np.int32 - int`).
// ------------------------------------------------------------------------------------------
__global__ void landmark_post_frames_kernel(const float* __restrict__ xy, const int* __restrict__ detail,
                                            const int* __restrict__ count, int K, int P, float* __restrict__ kps, int n) {
    // element i of frame st
    const int per = K * P;
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= per * n) return;
    const int st = g / per, i = g - st * per, f = i / P;
    const float* x = xy + (size_t)2 * per * st;
    const int* dt = detail + (size_t)5 * K * st;
    float ox = 0.f, oy = 0.f;
    if (f < count[st]) {
        const int* d = dt + f * 5;          // [h, w, y1, x1, add]
        float px = x[i * 2] * (float)d[1];
        float py = x[i * 2 + 1] * (float)d[0];
        ox = (float)((double)px + (double)d[3] - (double)d[4]);
        oy = (float)((double)py + (double)d[2] - (double)d[4]);
    }
    kps[(size_t)2 * per * st + i * 2] = ox;
    kps[(size_t)2 * per * st + i * 2 + 1] = oy;
}

// ------------------------------------------------------------------------------------------
// Frame difference gate (facer.py:111-113): sum |a-b| over all bytes.  uint4 loads, __vsadu4.
// ------------------------------------------------------------------------------------------
// This thread's part of sum |a - b| over n bytes (a, b 16-byte aligned); block 0 takes the bytes past the last 16.
__device__ __forceinline__ unsigned long long absdiff_bytes(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
                                                            size_t n) {
    const size_t nv = n / 16;
    unsigned long long local = 0;
    const uint4* a4 = reinterpret_cast<const uint4*>(a);
    const uint4* b4 = reinterpret_cast<const uint4*>(b);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
        uint4 x = a4[i], y = b4[i];
        local += __vsadu4(x.x, y.x) + __vsadu4(x.y, y.y) + __vsadu4(x.z, y.z) + __vsadu4(x.w, y.w);
    }
    if (blockIdx.x == 0) {
        for (size_t i = nv * 16 + threadIdx.x; i < n; i += blockDim.x) {
            int d = (int)a[i] - (int)b[i];
            local += (unsigned)(d < 0 ? -d : d);
        }
    }
    return local;
}

// 16 bytes from an address of any alignment: the one or two aligned 16-byte blocks that hold them, shifted into place.
// Every block loaded holds a byte of the range, so no load leaves the allocation.
__device__ __forceinline__ uint4 load16_any(const uint8_t* p) {
    const unsigned off = (unsigned)((uintptr_t)p & 15);
    const uint4* a = reinterpret_cast<const uint4*>(p - off);
    const uint4 lo = __ldg(a);
    if (off == 0) return lo;
    const uint4 hi = __ldg(a + 1);
    unsigned w0, w1, w2, w3, w4;
    switch (off >> 2) {
        case 0: w0 = lo.x; w1 = lo.y; w2 = lo.z; w3 = lo.w; w4 = hi.x; break;
        case 1: w0 = lo.y; w1 = lo.z; w2 = lo.w; w3 = hi.x; w4 = hi.y; break;
        case 2: w0 = lo.z; w1 = lo.w; w2 = hi.x; w3 = hi.y; w4 = hi.z; break;
        default: w0 = lo.w; w1 = hi.x; w2 = hi.y; w3 = hi.z; w4 = hi.w; break;
    }
    const unsigned sh = (off & 3) * 8;
    return make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh),
                      __funnelshift_r(w3, w4, sh));
}

// Ingest of one frame: the packed frame cur is cut into 16-byte units; unit u takes bytes [16u, 16u + 16) of the frame
// from row y = 16u / (3W) of the pitched source.  A unit inside one row is one 16-byte store from load16_any; a unit that
// crosses a row end, and the partial last unit, go byte by byte.  Returns this thread's part of sum |cur - prev|.
__device__ __forceinline__ unsigned long long ingest_units(const MpStreamDesc& D) {
    const unsigned row = (unsigned)D.W * 3u, n = row * (unsigned)D.H, units = (n + 15) / 16;
    const uint8_t* __restrict__ src = D.src;
    uint8_t* __restrict__ cur = D.cur;
    const uint8_t* __restrict__ prev = D.have_prev ? D.prev : nullptr;
    unsigned long long local = 0;
    for (unsigned u = blockIdx.x * blockDim.x + threadIdx.x; u < units; u += gridDim.x * blockDim.x) {
        const unsigned o = u * 16, y = o / row, x = o - y * row;
        if (x + 16 <= row) {
            const uint4 v = load16_any(src + (size_t)y * D.src_pitch + x);
            *reinterpret_cast<uint4*>(cur + o) = v;
            if (prev) {
                const uint4 q = *reinterpret_cast<const uint4*>(prev + o);
                local += __vsadu4(v.x, q.x) + __vsadu4(v.y, q.y) + __vsadu4(v.z, q.z) + __vsadu4(v.w, q.w);
            }
        } else {
            unsigned yy = y, xx = x;
            const unsigned end = o + 16 < n ? o + 16 : n;
            for (unsigned i = o; i < end; ++i) {
                const uint8_t v = src[(size_t)yy * D.src_pitch + xx];
                cur[i] = v;
                if (prev) {
                    const int dd = (int)v - (int)prev[i];
                    local += (unsigned)(dd < 0 ? -dd : dd);
                }
                if (++xx == row) { xx = 0; ++yy; }
            }
        }
    }
    return local;
}

// block y = frame (integer sums: the order of the atomic adds does not matter)
__global__ void __launch_bounds__(256) diff_frames_kernel(const MpStreamDesc* __restrict__ d, MpStreamDesc one, size_t one_bytes,
                                                          unsigned long long* __restrict__ sum) {
    const MpStreamDesc D = d ? d[blockIdx.y] : one;
    const size_t n = d ? (size_t)D.H * D.W * 3 : one_bytes;
    if (!D.have_prev && !D.src) return;
    unsigned long long local = D.src ? ingest_units(D) : absdiff_bytes(D.prev, D.cur, n);
    for (int o = 16; o > 0; o >>= 1) local += __shfl_down_sync(0xffffffffu, local, o);
    __shared__ unsigned long long warp_sum[8];
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < 8; ++w) t += warp_sum[w];
        atomicAdd(sum + blockIdx.y, t);
    }
}

int launch_frame_diff(const MpStreamDesc* d, int n, const MpStreamDesc& one, size_t bytes, unsigned long long* sum,
                      cudaStream_t s) {
    // ingest_units counts the 16-byte units of a frame in 32 bits
    SKPS_CHECK(bytes < (1ull << 32) - 16 || !(d || one.src), "frame_diff: a %zu-byte frame is larger than 4 GB", bytes);
    // a 16-byte unit per thread, at most 8 blocks per SM per frame
    size_t blocks = (bytes / 16 + 255) / 256;
    if (blocks > (size_t)sm_count() * 8) blocks = (size_t)sm_count() * 8;
    if (blocks < 1) blocks = 1;
    diff_frames_kernel<<<dim3((unsigned)blocks, n), 256, 0, s>>>(d, one, bytes, sum);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}
int upload_host_frame(const uint8_t* frame, size_t bytes, uint8_t* stage, uint8_t* dst, cudaStream_t s) {
    cudaPointerAttributes attr;
    const bool pinned = cudaPointerGetAttributes(&attr, frame) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    if (!pinned) {
        cudaGetLastError();          // clear the "invalid value" a pageable pointer may leave behind
        memcpy(stage, frame, bytes);
    }
    SKPS_CUDA(cudaMemcpyAsync(dst, pinned ? frame : stage, bytes, cudaMemcpyHostToDevice, s));
    return 0;
}
int check_device_frame(const void* frame, int device, const char* fn, int index) {
    cudaPointerAttributes attr;
    SKPS_CUDA(cudaPointerGetAttributes(&attr, frame));
    if ((attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged) && attr.device == device) return 0;
    if (index < 0) set_error("%s: the frame is not in memory of device %d", fn, device);
    else set_error("%s: frame %d is not in memory of device %d", fn, index, device);
    return 1;
}
int launch_letterbox(const LetterboxArgs& a, int n, cudaStream_t s) {
    letterbox_frames_kernel<<<dim3((a.in_w + 255) / 256, a.in_h, n), 256, 0, s>>>(a);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}
int launch_crop(const CropArgs& a, int n, cudaStream_t s) {
    crop_frames_kernel<<<dim3((a.S + 255) / 256, a.S, a.K * n), 256, 0, s>>>(a);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}
int launch_landmark_post(const float* xy, const int* detail, const int* count, int K, int P, float* kps, int n, cudaStream_t s) {
    const int total = K * P * n;
    landmark_post_frames_kernel<<<(total + 255) / 256, 256, 0, s>>>(xy, detail, count, K, P, kps, n);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}
int launch_select(const SelectArgs& a, int n, cudaStream_t s) {
    select_frames_kernel<<<n, SEL_THREADS, 0, s>>>(a);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace skps

// ============================================================================================
// C-ABI wrappers
// ============================================================================================
using namespace skps;

extern "C" SKPS_API int skps_letterbox(const uint8_t* frame, int H, int W, int pitch, uint8_t* out, int in_h, int in_w,
                              int rw, int rh, int top, int left, void* stream) {
    SKPS_CHECK(frame && out && H > 0 && W > 0 && rw > 0 && rh > 0, "letterbox: bad arguments");
    LetterboxArgs a = {};
    a.frame = frame; a.H = H; a.W = W; a.pitch = pitch; a.rw = rw; a.rh = rh; a.top = top; a.left = left;
    a.out = out; a.in_h = in_h; a.in_w = in_w;
    return launch_letterbox(a, 1, (cudaStream_t)stream);
}

extern "C" SKPS_API int skps_letterbox_frames(const skps_det_src* src, int n, uint8_t* out, int in_h, int in_w,
                                              void* stream) {
    SKPS_CHECK(n >= 0 && n <= 65535 && in_h > 0 && in_h <= 65535 && in_w > 0,
               "letterbox_frames: n %d outside 0..65535 or input %dx%d", n, in_h, in_w);
    if (n == 0) return 0;
    SKPS_CHECK(src && out, "letterbox_frames: bad arguments");
    LetterboxArgs a = {};
    a.src = src; a.out = out; a.out_stride = (size_t)in_h * in_w * 3; a.in_h = in_h; a.in_w = in_w;
    return launch_letterbox(a, n, (cudaStream_t)stream);
}

extern "C" SKPS_API int skps_select_faces(const float* det_rows, const int32_t* det_count, int det_stride, const float* track,
                                 int n_track, float iou_thres, float alpha, float one_minus_alpha, float min_face,
                                 int top_k, float* boxes4, int32_t* count, void* stream) {
    SKPS_CHECK(det_rows && det_count && boxes4 && count && top_k > 0 && top_k <= SEL_MAX_K, "select_faces: bad arguments");
    SelectArgs a = {};
    a.det_rows = det_rows; a.det_count = det_count; a.det_stride = det_stride; a.flag1 = 1;
    a.track = track; a.n_track1 = n_track;
    a.iou_thres = iou_thres; a.alpha = alpha; a.one_minus_alpha = one_minus_alpha; a.min_face = min_face; a.top_k = top_k;
    a.boxes4 = boxes4; a.count = count;
    return launch_select(a, 1, (cudaStream_t)stream);
}

extern "C" SKPS_API int skps_select_faces_batch(const float* det_rows, const int32_t* det_count, int det_cap, int n,
                                                float min_face, int top_k, float* boxes4, int32_t* count, void* stream) {
    SKPS_CHECK(n >= 0 && top_k > 0 && top_k <= SEL_MAX_K && det_cap > 0,
               "select_faces_batch: n %d < 0, top_k %d outside 1..%d or det_cap %d < 1", n, top_k, SEL_MAX_K, det_cap);
    if (n == 0) return 0;
    SKPS_CHECK(det_rows && det_count && boxes4 && count, "select_faces_batch: bad arguments");
    SelectArgs a = {};
    a.det_rows = det_rows; a.det_count = det_count; a.det_stride = 16; a.det_cap = det_cap; a.flag1 = 1;
    a.min_face = min_face; a.top_k = top_k;
    a.boxes4 = boxes4; a.count = count;
    return launch_select(a, n, (cudaStream_t)stream);
}

extern "C" SKPS_API int skps_landmark_boxes(const float* kps, int n_points, const int32_t* face_image, int n_faces,
                                            const float* sel_boxes, const int32_t* sel_count, int top_k, float iou_thres,
                                            float alpha, float one_minus_alpha, float* boxes_out, void* stream) {
    SKPS_CHECK(n_faces >= 0 && n_points > 0 && top_k > 0, "landmark_boxes: n_faces %d, n_points %d or top_k %d out of range",
               n_faces, n_points, top_k);
    if (n_faces == 0) return 0;
    SKPS_CHECK(kps && face_image && sel_boxes && sel_count && boxes_out, "landmark_boxes: bad arguments");
    const unsigned blocks = (unsigned)(((long long)n_faces + 7) / 8);
    landmark_boxes_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(kps, n_points, face_image, n_faces, sel_boxes, sel_count,
                                                                     top_k, iou_thres, alpha, one_minus_alpha, boxes_out);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

extern "C" SKPS_API int skps_crop_resize(const uint8_t* frame, int H, int W, int pitch, const float* boxes4,
                                const int32_t* count, int max_faces, float face_scale, float min_face,
                                uint8_t* crops, int out_hw, int32_t* detail, void* stream) {
    SKPS_CHECK(frame && boxes4 && count && crops && detail && max_faces > 0, "crop_resize: bad arguments");
    CropArgs a = {};
    a.frame = frame; a.H = H; a.W = W; a.pitch = pitch; a.boxes = boxes4; a.count = count; a.K = max_faces;
    a.face_scale = face_scale; a.min_face = min_face; a.crops = crops; a.S = out_hw; a.detail = detail;
    return launch_crop(a, 1, (cudaStream_t)stream);
}

extern "C" SKPS_API int skps_crop_faces(const skps_face_src* src, const float* boxes4, int n, float face_scale, float min_face,
                                        uint8_t* crops, int out_hw, int32_t* detail, void* stream) {
    SKPS_CHECK(n >= 0 && n <= 65535 && out_hw > 0, "crop_faces: n %d outside 0..65535 or out_hw %d", n, out_hw);
    if (n == 0) return 0;
    SKPS_CHECK(src && boxes4 && crops && detail, "crop_faces: bad arguments");
    dim3 grid((out_hw + 255) / 256, out_hw, n);
    crop_faces_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, boxes4, face_scale, min_face, crops, out_hw, detail);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

extern "C" SKPS_API int skps_crop_rect(const uint8_t* frame, int H, int W, int pitch, int rx, int ry, int rw, int rh,
                                       uint8_t* out, int out_hw, void* stream) {
    SKPS_CHECK(frame && out && H > 0 && W > 0 && rw > 0 && rh > 0 && out_hw > 0, "crop_rect: bad arguments");
    dim3 grid((out_hw + 255) / 256, out_hw);
    rect_resize_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(frame, H, W, pitch, rx, ry, rw, rh, out, out_hw);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

extern "C" SKPS_API int skps_nme(const float* target, const float* preds, int n, int n_points, int norm_a, int norm_b,
                                 float* out, void* stream) {
    SKPS_CHECK(target && preds && out && n > 0 && n_points > 0 && norm_a >= 0 && norm_b >= 0 && norm_a < n_points &&
               norm_b < n_points, "nme: bad arguments");
    nme_kernel<<<(n + 3) / 4, 128, 0, (cudaStream_t)stream>>>(target, preds, n, n_points, norm_a, norm_b, out);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

extern "C" SKPS_API int skps_landmark_post(const float* xy_norm, const int32_t* detail, const int32_t* count, int max_faces,
                                  int n_points, float* kps, void* stream) {
    SKPS_CHECK(xy_norm && detail && count && kps, "landmark_post: bad arguments");
    return launch_landmark_post(xy_norm, detail, count, max_faces, n_points, kps, 1, (cudaStream_t)stream);
}

extern "C" SKPS_API int skps_frame_absdiff_sum(const uint8_t* a, const uint8_t* b, size_t n, unsigned long long* sum,
                                      void* stream) {
    SKPS_CHECK(a && b && sum, "absdiff: bad arguments");
    SKPS_CHECK(((uintptr_t)a % 16 == 0) && ((uintptr_t)b % 16 == 0), "absdiff: pointers must be 16-byte aligned");
    SKPS_CUDA(cudaMemsetAsync(sum, 0, sizeof(unsigned long long), (cudaStream_t)stream));
    MpStreamDesc D = {};
    D.prev = a; D.cur = const_cast<uint8_t*>(b); D.have_prev = 1;      // cur is written only when src is set
    return launch_frame_diff(nullptr, 1, D, n, sum, (cudaStream_t)stream);
}

extern "C" SKPS_API int skps_frame_ingest(const uint8_t* frame, int H, int W, int pitch, uint8_t* packed, const uint8_t* prev,
                                          unsigned long long* sum, void* stream) {
    SKPS_CHECK(frame && packed && sum && H > 0 && W > 0 && (H == 1 || pitch >= 3 * W), "ingest: bad arguments");
    SKPS_CHECK(((uintptr_t)packed % 16 == 0) && ((uintptr_t)prev % 16 == 0), "ingest: packed and prev must be 16-byte aligned");
    SKPS_CUDA(cudaMemsetAsync(sum, 0, sizeof(unsigned long long), (cudaStream_t)stream));
    MpStreamDesc D = {};
    D.cur = packed; D.prev = prev; D.have_prev = prev != nullptr; D.H = H; D.W = W;
    D.src = frame; D.src_pitch = pitch;
    return launch_frame_diff(nullptr, 1, D, (size_t)H * W * 3, sum, (cudaStream_t)stream);
}
