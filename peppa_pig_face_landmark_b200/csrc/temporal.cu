// Device-side temporal layer of FaceAna.run for many concurrent video streams (SURVEY 8f-1):
//   diff_frames gate          facer.py:98-118
//   GroupTrack.calculate      Skps/core/smoother/lk.py:19-59   (IoU match to last frame's landmark sets)
//   OneEuroFilter.__call__    lk.py:115-149                    (unit time step, displacement-norm derivative)
//   track box refresh         facer.py:74-82 + judge_boxs :144-189 + EmaFilter lk.py:155-162
// One CTA per frame of the call, i.e. per stream the call feeds; all state (previous landmark sets, their deltas, track
// boxes) stays in HBM between frames, indexed by the stream, so a batch of streams needs no host round trip between frames
// and a stream the call does not feed is not touched.  The reference does this arithmetic in numpy with mixed
// float32/float64 operands; the kernel follows numpy's promotion rules operation by operation (float64 wherever one
// operand is float64, float32 where both are), which is why this file is compiled with -fmad=false.
#include <math.h>

#include "common.h"
#include "mpipe_kernels.h"

namespace skps {

// A numpy scalar: value + "is float32".  Binary ops promote like numpy (f32 op f32 -> f32, anything else -> f64).
struct Num {
    double v;
    bool f32;
};
__device__ __forceinline__ Num mk(double v, bool f32) { Num n; n.v = v; n.f32 = f32; return n; }
__device__ __forceinline__ Num nsub(Num a, Num b) {
    return (a.f32 && b.f32) ? mk((double)((float)a.v - (float)b.v), true) : mk(a.v - b.v, false);
}
__device__ __forceinline__ Num nadd(Num a, Num b) {
    return (a.f32 && b.f32) ? mk((double)((float)a.v + (float)b.v), true) : mk(a.v + b.v, false);
}
__device__ __forceinline__ Num nmul(Num a, Num b) {
    return (a.f32 && b.f32) ? mk((double)((float)a.v * (float)b.v), true) : mk(a.v * b.v, false);
}
__device__ __forceinline__ Num ndiv(Num a, Num b) {
    return (a.f32 && b.f32) ? mk((double)((float)a.v / (float)b.v), true) : mk(a.v / b.v, false);
}
__device__ __forceinline__ Num nmin(Num a, Num b) { return b.v < a.v ? b : a; }      // python min(a, b): first minimal
__device__ __forceinline__ Num nmax(Num a, Num b) { return b.v > a.v ? b : a; }      // python max(a, b): first maximal

// lk.py:61-84 / facer.py:151-170 on rectangles [x0,y0,x1,y1]: > thres ?
__device__ bool iou_gt(const Num* r1, const Num* r2, double thres) {
    const Num a1 = nmul(nsub(r1[2], r1[0]), nsub(r1[3], r1[1]));
    const Num a2 = nmul(nsub(r2[2], r2[0]), nsub(r2[3], r2[1]));
    const Num w = nsub(nmin(r1[2], r2[2]), nmax(r1[0], r2[0]));
    const Num h = nsub(nmin(r1[3], r2[3]), nmax(r1[1], r2[1]));
    if (!(w.v > 0.0) || !(h.v > 0.0)) return false;              // max(0, .) -> intersect 0 -> iou 0
    const Num inter = nmul(w, h);
    const Num iou = ndiv(inter, nsub(nadd(a1, a2), inter));
    return iou.v > thres;
}

// min/max of one landmark set along both axes -> r[4]; all 128 threads of the CTA take part.  Values exact in double.
__device__ void set_rect(const double* pts, int P, double* r, double* red /*[4][4]*/) {
    double mn0 = INFINITY, mn1 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY;
    for (int p = threadIdx.x; p < P; p += blockDim.x) {
        const double x = pts[2 * p], y = pts[2 * p + 1];
        mn0 = fmin(mn0, x); mx0 = fmax(mx0, x); mn1 = fmin(mn1, y); mx1 = fmax(mx1, y);
    }
    for (int o = 16; o > 0; o >>= 1) {
        mn0 = fmin(mn0, __shfl_xor_sync(0xffffffffu, mn0, o)); mx0 = fmax(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
        mn1 = fmin(mn1, __shfl_xor_sync(0xffffffffu, mn1, o)); mx1 = fmax(mx1, __shfl_xor_sync(0xffffffffu, mx1, o));
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { red[w * 4] = mn0; red[w * 4 + 1] = mn1; red[w * 4 + 2] = mx0; red[w * 4 + 3] = mx1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int nw = blockDim.x >> 5;
        for (int k = 1; k < nw; ++k) {
            red[0] = fmin(red[0], red[k * 4]); red[1] = fmin(red[1], red[k * 4 + 1]);
            red[2] = fmax(red[2], red[k * 4 + 2]); red[3] = fmax(red[3], red[k * 4 + 3]);
        }
        r[0] = red[0]; r[1] = red[1]; r[2] = red[2]; r[3] = red[3];
    }
    __syncthreads();
}

// Gate of facer.py:55-62: run the detector when there is no previous frame of this size or the mean absolute difference
// exceeds 5 (np.sum(diff) / H / W / 3. in float64).  Only keyframes (det_slot[s] >= 0; det_slot null: every stream) run
// the detector; the host makes every frame without a previous frame of its size a keyframe.
__global__ void mp_decide_kernel(const unsigned long long* __restrict__ diff, const int* __restrict__ hw,
                                 const int* __restrict__ have_prev, const int* __restrict__ det_slot, int* __restrict__ flag,
                                 int n) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    if (det_slot && det_slot[s] < 0) { flag[s] = 0; return; }
    if (!have_prev[s]) { flag[s] = 1; return; }
    const double m = (double)diff[s] / (double)hw[2 * s] / (double)hw[2 * s + 1] / 3.0;
    flag[s] = m > 5.0 ? 1 : 0;
}

__global__ void __launch_bounds__(128) mp_temporal_kernel(const MpTemporalArgs a) {
    // frame g of the call (its inputs and outputs), stream s (its state)
    const int g = blockIdx.x, s = a.stream ? a.stream[g] : g, tid = threadIdx.x;
    const int K = a.top_k, P = a.n_points;
    const long long set = (long long)2 * P;
    __shared__ double red[16];
    __shared__ double rect_now[4], rect_prev[4];
    __shared__ int s_match;
    __shared__ int64_t s_ids[64];                                     // the old track ids (skps_mpipe_create: top_k <= 64)
    const int n = a.count[g];
    // id memory: the old track boxes (overwritten below before the ids are assigned), the stream's lost tracks, and per
    // face the entries it overlaps with IoU > iou_thres (bit k: entry k), all float32 as judge_boxs compares two such rows
    __shared__ float s_old_box[64][4], s_mem_box[64][4];
    __shared__ int64_t s_mem_id[64];
    __shared__ int s_mem_gap[64];
    __shared__ unsigned long long s_hit[64];
    const bool mem_on = a.id_memory > 0;
    int mem_n = 0;
    if (mem_on) {
        mem_n = a.mem_n[s];
        const int n_old = a.n_track[s];
        const float* tf = a.track_f32 + (long long)s * K * 4;
        const float* mb = a.mem_box + (long long)s * K * 4;
        for (int e = tid; e < 4 * n_old; e += blockDim.x) s_old_box[e >> 2][e & 3] = tf[e];
        for (int e = tid; e < 4 * mem_n; e += blockDim.x) s_mem_box[e >> 2][e & 3] = mb[e];
        for (int e = tid; e < mem_n; e += blockDim.x) {
            s_mem_id[e] = a.mem_ids[(long long)s * K + e];
            s_mem_gap[e] = a.mem_gap[(long long)s * K + e];
        }
        for (int e = tid; e < n; e += blockDim.x) s_hit[e] = 0ull;
        __syncthreads();
        const float* b4 = a.boxes4 + (long long)g * K * 4;
        for (int e = tid; e < n * mem_n; e += blockDim.x) {
            const int i = e / mem_n, k = e - i * mem_n;
            Num r1[4], r2[4];
            for (int c = 0; c < 4; ++c) { r1[c] = mk((double)b4[i * 4 + c], true); r2[c] = mk((double)s_mem_box[k][c], true); }
            if (iou_gt(r1, r2, a.iou_thres)) atomicOr(&s_hit[i], 1ull << k);
        }
        __syncthreads();
    }
    const float* now = a.kps_now + (long long)g * K * set;            // float32 (n, P, 2)
    const int cur = a.state_idx[s], nxt = cur ^ 1;
    const double* prev = a.prev_lm + ((long long)(s * 2 + cur) * K) * set;
    const double* prev_dx = a.prev_dx + ((long long)(s * 2 + cur) * K) * set;
    double* res = a.prev_lm + ((long long)(s * 2 + nxt) * K) * set;  // result = next frame's "previous"
    double* res_dx = a.prev_dx + ((long long)(s * 2 + nxt) * K) * set;
    double* out = a.out_kps + (long long)g * K * set;
    int n_prev = a.flag[g] ? -1 : a.n_prev[s];                        // facer.py:59: previous_landmarks_set = None
    const bool prev_f32 = a.prev_f32[s] != 0;
    const double W = (double)a.hw[2 * g + 1], H = (double)a.hw[2 * g];
    bool all_f32 = true;                                              // dtype of np.array(result)
    for (int i = 0; i < n; ++i) {
        const float* cur_pts = now + i * set;
        double* r_i = res + i * set;
        int match = -1;
        if (n_prev > 0) {
            // rectangle of this face (float32 values) against last frame's sets, first match wins (lk.py:33-34)
            for (int p = tid; p < 2 * P; p += blockDim.x) r_i[p] = (double)cur_pts[p];     // scratch: the row itself if unmatched
            __syncthreads();
            set_rect(r_i, P, rect_now, red);
            for (int j = 0; j < n_prev && match < 0; ++j) {
                set_rect(prev + j * set, P, rect_prev, red);
                if (tid == 0) {
                    Num r1[4], r2[4];
                    for (int c = 0; c < 4; ++c) { r1[c] = mk(rect_now[c], true); r2[c] = mk(rect_prev[c], prev_f32); }
                    s_match = iou_gt(r1, r2, a.iou_thres) ? j : -1;
                }
                __syncthreads();
                match = s_match;
                __syncthreads();
            }
        }
        if (match < 0) {
            for (int p = tid; p < 2 * P; p += blockDim.x) { r_i[p] = (double)cur_pts[p]; res_dx[i * set + p] = 0.0; }
        } else {
            all_f32 = false;
            // OneEuroFilter on coordinates normalised by [w, h] (lk.py:36-38, 115-149), float64 throughout
            const double* pv = prev + match * set;
            const double* pd = prev_dx + match * set;
            for (int p = tid; p < P; p += blockDim.x) {
                const double x0 = (double)cur_pts[2 * p] / W, x1 = (double)cur_pts[2 * p + 1] / H;
                const double q0 = pv[2 * p] / W, q1 = pv[2 * p + 1] / H;
                const double d0 = pd[2 * p] / W, d1 = pd[2 * p + 1] / H;
                const double e0 = x0 - q0, e1 = x1 - q1;
                const double speed = sqrt(e0 * e0 + e1 * e1);
                const double speed_prev = sqrt(d0 * d0 + d1 * d1);
                const double speed_hat = a.a_d * speed + a.one_minus_a_d * speed_prev;
                const double cutoff = a.min_cutoff + a.beta * fabs(speed_hat);
                const double r = a.two_pi * cutoff * 1.0;
                double al = r / (r + 1.0);
                if (speed < 0.002) al = 0.01;
                const double oma = 1.0 - al;
                const double f0 = (al * x0 + oma * q0) * W, f1 = (al * x1 + oma * q1) * H;
                r_i[2 * p] = f0; r_i[2 * p + 1] = f1;
                res_dx[i * set + 2 * p] = pv[2 * p] - f0;
                res_dx[i * set + 2 * p + 1] = pv[2 * p + 1] - f1;
            }
        }
        __syncthreads();
    }
    // outputs + track boxes: tmp_box = min/max of the refined landmarks, judge_boxs(boxes_return, tmp_box) (facer.py:74-82)
    const float* boxes_ret = a.boxes4 + (long long)g * K * 4;         // float32, n rows
    for (int i = 0; i < n; ++i) {
        const double* r_i = res + i * set;
        for (int p = tid; p < 2 * P; p += blockDim.x) out[i * set + p] = r_i[p];
        set_rect(r_i, P, rect_now, red);
        if (tid == 0) {
            Num nowb[4];
            for (int c = 0; c < 4; ++c) nowb[c] = mk(rect_now[c], all_f32);
            int m = -1;
            for (int j = 0; j < n && m < 0; ++j) {
                Num pb[4];
                for (int c = 0; c < 4; ++c) pb[c] = mk((double)boxes_ret[j * 4 + c], true);
                if (iou_gt(nowb, pb, a.iou_thres)) m = j;
            }
            double* tb = a.track_box + ((long long)s * K + i) * 4;
            float* tf = a.track_f32 + ((long long)s * K + i) * 4;
            for (int c = 0; c < 4; ++c) {
                double v = rect_now[c];
                if (m >= 0) {
                    // EmaFilter (lk.py:155-162): alpha * now + (1 - alpha) * prev, python-float weights
                    // (a python float multiplying a float32 array is cast to float32 first; boxes_return is float32)
                    const Num t1 = all_f32 ? mk((double)((float)a.alpha * (float)nowb[c].v), true)
                                           : mk(a.alpha * nowb[c].v, false);
                    const Num t2 = mk((double)((float)a.one_minus_alpha * boxes_ret[m * 4 + c]), true);
                    v = nadd(t1, t2).v;
                }
                tb[c] = v;
                tf[c] = (float)v;                                      // facer.py: the next frame's boxes go through float32
                if (a.out_box) a.out_box[((long long)g * K + i) * 4 + c] = v;
            }
        }
        __syncthreads();
    }
    if (tid == 0) {
        // track ids, in output order: a face inherits the id of its source track box unless an earlier face of this frame
        // took it; every other face takes back the id of the first lost track it overlaps that has been missing for at most
        // id_memory frames, or else gets the stream's next number.  The new ids are index-aligned with the new track boxes.
        int64_t* ids = a.ids + (long long)s * K;
        const int n_old = a.n_track[s];
        for (int j = 0; j < n_old; ++j) s_ids[j] = ids[j];
        unsigned long long taken = 0ull;                              // bit j: track box j's id is given out (K <= 64)
        unsigned long long used = 0ull;                               // bit k: memory entry k's id is given back
        int64_t next = a.next_id[s];
        for (int i = 0; i < n; ++i) {
            const int j = a.src[(long long)g * K + i];
            if (j >= 0 && j < n_old && !((taken >> j) & 1ull)) {
                taken |= 1ull << j;
                ids[i] = s_ids[j];
                if (a.out_ids) a.out_ids[(long long)g * K + i] = ids[i];
                continue;
            }
            int k = -1;
            if (mem_on) {
                for (unsigned long long c = s_hit[i] & ~used; c && k < 0; c &= c - 1) {
                    const int b = __ffsll((long long)c) - 1;
                    if (s_mem_gap[b] <= a.id_memory) k = b;
                }
            }
            if (k >= 0) {
                used |= 1ull << k;
                ids[i] = s_mem_id[k];
            } else {
                ids[i] = next++;
            }
            if (a.out_ids) a.out_ids[(long long)g * K + i] = ids[i];
        }
        a.next_id[s] = next;
        if (mem_on) {
            // the new memory: the tracks this frame lost, in the order they were returned, then the older entries not given
            // back that may still qualify at the next frame, oldest last; at most K
            int64_t* mid = a.mem_ids + (long long)s * K;
            float* mb = a.mem_box + (long long)s * K * 4;
            int* mg = a.mem_gap + (long long)s * K;
            int m = 0;
            for (int j = 0; j < n_old && m < K; ++j) {
                if ((taken >> j) & 1ull) continue;
                mid[m] = s_ids[j]; mg[m] = 1;
                for (int c = 0; c < 4; ++c) mb[m * 4 + c] = s_old_box[j][c];
                ++m;
            }
            for (int k = 0; k < mem_n && m < K; ++k) {
                if (((used >> k) & 1ull) || s_mem_gap[k] >= a.id_memory) continue;
                mid[m] = s_mem_id[k]; mg[m] = s_mem_gap[k] + 1;
                for (int c = 0; c < 4; ++c) mb[m * 4 + c] = s_mem_box[k][c];
                ++m;
            }
            a.mem_n[s] = m;
        }
        a.n_prev[s] = n;
        a.prev_f32[s] = all_f32 ? 1 : 0;
        a.n_track[s] = n;
        a.state_idx[s] = nxt;
    }
}

int launch_mp_decide(const unsigned long long* diff, const int* hw, const int* have_prev, const int* det_slot, int* flag, int n,
                     cudaStream_t s) {
    mp_decide_kernel<<<(n + 63) / 64, 64, 0, s>>>(diff, hw, have_prev, det_slot, flag, n);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

int launch_mp_temporal(const MpTemporalArgs& a, int n, cudaStream_t s) {
    mp_temporal_kernel<<<n, 128, 0, s>>>(a);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace skps
