// Detector post-processing (face_detector.py:31-37, 73-136) for any number of candidates, batched over frames.
//   1. compaction: rows with obj > score_thres -> 64-bit keys (score, row), many CTAs per frame
//   2. sort: keys descending = (score desc, row index desc), a total order, so the result does not depend on the order in
//      which the compaction wrote them.  Bitonic sort of 4096-key chunks in shared memory, then merge passes that place
//      every key by a binary search in the partner run (O(n log^2 n) work, deterministic)
//   3. greedy NMS, exactly py_nms: candidate j is suppressed iff some earlier KEPT box i has !(iou(i, j) < iou_thres).
//      Candidates go in rank order in tiles of 32: the tile is tested against the boxes kept so far by all warps, then
//      resolved inside the tile by one warp (32x32 suppression mask), so the cost is O(n x kept) with two barriers per tile
//   4. gather: kept rows with cols 0-3 mapped back by scale_coords ((v - pad) / scale), their row indices and the count
// Compiled with -fmad=false: the IoU and scale_coords float32 expressions round exactly like numpy's.
#include <limits.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "mpipe_kernels.h"

namespace skps {

namespace {

constexpr int SORT_CHUNK = 4096;      // keys per shared-memory bitonic sort
constexpr int SORT_THREADS = 1024;
constexpr int MERGE_THREADS = 256;
constexpr int COMPACT_THREADS = 256;
constexpr int NMS_THREADS = 512;
constexpr int NMS_WARPS = NMS_THREADS / 32;
constexpr int KEPT_SMEM = 2048;       // kept boxes cached in shared memory; later ones are read from the workspace

// Workspace: the candidate counters of all frames (one memset clears them), then per frame room for `cap` candidates.
struct NmsWs {
    int* n;                           // candidates over the threshold (may exceed cap: then only cap keys were written)
    unsigned long long* key[2];       // ping-pong sort buffers
    float4* box;                      // xyxy box by rank
    int* row;                         // detector row by rank
    int* keep;                        // ranks of the kept boxes, in order
};

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

__host__ __device__ inline size_t ws_header_bytes(int batch) { return align256(4 * (size_t)batch); }

__host__ __device__ inline size_t ws_frame_bytes(int cap) {
    const size_t c = (size_t)(cap > 0 ? cap : 1);
    return 2 * align256(8 * c) + align256(16 * c) + 2 * align256(4 * c);
}

__device__ inline NmsWs ws_at(const NmsArgs& a, int f) {
    const size_t c = (size_t)(a.ws_cap > 0 ? a.ws_cap : 1);
    char* p = (char*)a.ws + ws_header_bytes(a.batch) + ws_frame_bytes(a.ws_cap) * f;
    NmsWs w;
    w.n = (int*)a.ws + f;
    w.key[0] = (unsigned long long*)p; p += align256(8 * c);
    w.key[1] = (unsigned long long*)p; p += align256(8 * c);
    w.box = (float4*)p; p += align256(16 * c);
    w.row = (int*)p; p += align256(4 * c);
    w.keep = (int*)p;
    return w;
}

// float -> uint32 with the same order (no NaN reaches here: NaN > thres is false)
__device__ __forceinline__ unsigned ordered_bits(float v) {
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float4 xyxy_of(const float* r) {
    const float hw = r[2] / 2.f, hh = r[3] / 2.f;                         // xywh2xyxy, face_detector.py:76-79
    return make_float4(r[0] - hw, r[1] - hh, r[0] + hw, r[1] + hh);
}

__device__ __forceinline__ float iou_nms(const float4 a, const float4 b) {
    // face_detector.py:117-130, float32 throughout; a is the kept box
    float area = (a.z - a.x) * (a.w - a.y);
    float xx1 = fmaxf(a.x, b.x), yy1 = fmaxf(a.y, b.y);
    float xx2 = fminf(a.z, b.z), yy2 = fminf(a.w, b.w);
    float inter = fmaxf(0.f, yy2 - yy1) * fmaxf(0.f, xx2 - xx1);
    float other = (b.w - b.y) * (b.z - b.x);
    return inter / (area + other - inter);
}

// The last stage that fixes the order writes the boxes and rows by rank instead of keys.
__device__ __forceinline__ void emit_ranked(const NmsWs& w, const float* raw, int rank, unsigned long long key) {
    const int r = (int)(unsigned)(key & 0xffffffffu);
    w.row[rank] = r;
    w.box[rank] = xyxy_of(raw + (size_t)r * 16);
}

__global__ void __launch_bounds__(COMPACT_THREADS) nms_compact_kernel(NmsArgs a) {
    const int f = blockIdx.y;
    const NmsWs w = ws_at(a, f);
    const float* raw = a.raw + (size_t)a.rows * 16 * f;
    const int lane = threadIdx.x & 31;
    const int stride = gridDim.x * blockDim.x;
    for (int base = blockIdx.x * blockDim.x; base < a.rows; base += stride) {
        const int r = base + threadIdx.x;
        float sc = 0.f;
        bool hot = false;
        if (r < a.rows) {
            sc = raw[(size_t)r * 16 + 4];
            hot = sc > a.score_thres;
        }
        const unsigned m = __ballot_sync(0xffffffffu, hot);
        if (!m) continue;
        int slot0 = 0;
        if (lane == __ffs(m) - 1) slot0 = atomicAdd(w.n, __popc(m));
        slot0 = __shfl_sync(0xffffffffu, slot0, __ffs(m) - 1);
        const int slot = slot0 + __popc(m & ((1u << lane) - 1));
        if (hot && slot < a.ws_cap) w.key[0][slot] = ((unsigned long long)ordered_bits(sc) << 32) | (unsigned)r;
    }
}

__global__ void __launch_bounds__(SORT_THREADS) nms_chunk_sort_kernel(NmsArgs a) {
    const int f = blockIdx.y;
    const NmsWs w = ws_at(a, f);
    const int n = *w.n;
    const int start = blockIdx.x * SORT_CHUNK;
    if (n > a.limit || start >= n) return;
    __shared__ unsigned long long s[SORT_CHUNK];
    const int len = min(SORT_CHUNK, n - start);
    int L = 1;
    while (L < len) L <<= 1;
    for (int i = threadIdx.x; i < L; i += blockDim.x) s[i] = i < len ? w.key[0][start + i] : 0ull;   // 0 sorts last
    __syncthreads();
    for (int k = 2; k <= L; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < L / 2; t += blockDim.x) {
                const int i = 2 * t - (t & (j - 1)), ixj = i + j;
                const unsigned long long x = s[i], y = s[ixj];
                if (((i & k) == 0) ? (x < y) : (x > y)) { s[i] = y; s[ixj] = x; }
            }
            __syncthreads();
        }
    }
    const float* raw = a.raw + (size_t)a.rows * 16 * f;
    const bool final_order = n <= SORT_CHUNK;
    for (int i = threadIdx.x; i < len; i += blockDim.x) {
        if (final_order) emit_ranked(w, raw, i, s[i]);
        else w.key[0][start + i] = s[i];
    }
}

// Merge pass p: runs of `run` keys (sorted descending) pairwise into runs of 2*run.  Passes with run >= n do nothing, so the
// passes that work are p = 0 .. P(n)-1 and pass p reads buffer p & 1.
__global__ void __launch_bounds__(MERGE_THREADS) nms_merge_kernel(NmsArgs a, int run, int pass) {
    const int f = blockIdx.y;
    const NmsWs w = ws_at(a, f);
    const int n = *w.n;
    if (n > a.limit || n <= run) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long* src = (pass & 1) ? w.key[1] : w.key[0];
    const int r = i / run, rs = r * run;
    int lo, hi;
    if (r & 1) { lo = rs - run; hi = rs; }
    else { lo = min(rs + run, n); hi = min(rs + 2 * run, n); }
    const int p0 = lo;
    const unsigned long long k = src[i];
    while (lo < hi) {                                  // partner keys greater than k (keys are distinct)
        const int mid = (lo + hi) >> 1;
        if (src[mid] > k) lo = mid + 1; else hi = mid;
    }
    const int pos = (r & ~1) * run + (i - rs) + (lo - p0);
    if (n <= 2 * run) emit_ranked(w, a.raw + (size_t)a.rows * 16 * f, pos, k);
    else ((pass & 1) ? w.key[0] : w.key[1])[pos] = k;
}

__global__ void __launch_bounds__(NMS_THREADS) nms_greedy_kernel(NmsArgs a) {
    const int f = blockIdx.x;
    const NmsWs w = ws_at(a, f);
    const int n = *w.n;
    if (n > a.limit) {
        // more candidates than the caller allows: count = -candidates and nothing else (skps_detect_post's contract)
        if (threadIdx.x == 0) a.count[f] = -n;
        return;
    }
    __shared__ float4 s_kept[KEPT_SMEM];
    __shared__ unsigned s_dead;
    __shared__ int s_nkeep;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float thr = a.iou_thres;
    const int cap = a.capacity;
    if (threadIdx.x == 0) { s_dead = 0; s_nkeep = 0; }
    __syncthreads();
    float4 nb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane < n) nb = w.box[lane];
    for (int t0 = 0; t0 < n; t0 += 32) {
        const int nk = s_nkeep;
        if (nk >= cap) break;                          // uniform: read after a barrier
        const int j = t0 + lane;
        const bool valid = j < n;
        const float4 bj = nb;
        if (j + 32 < n) nb = w.box[j + 32];            // next tile, in flight while this one is tested
        // 1. against the boxes kept so far (kept box first, as py_nms)
        bool dead = !valid;
        for (int i0 = warp; i0 < nk; i0 += 4 * NMS_WARPS) {
            if (__all_sync(0xffffffffu, dead)) break;
            bool hit = false;
#pragma unroll
            for (int u = 0; u < 4; ++u) {                 // four independent tests in flight per lane
                const int i = i0 + u * NMS_WARPS;
                if (i < nk) {
                    const float4 bi = i < KEPT_SMEM ? s_kept[i] : w.box[w.keep[i]];
                    hit |= !(iou_nms(bi, bj) < thr);
                }
            }
            dead |= hit;
        }
        const unsigned dm = __ballot_sync(0xffffffffu, dead && valid);
        if (lane == 0 && dm) atomicOr(&s_dead, dm);
        __syncthreads();
        // 2. inside the tile, in rank order
        if (warp == 0) {
            const unsigned valid_mask = (n - t0 >= 32) ? 0xffffffffu : ((1u << (n - t0)) - 1);
            unsigned alive = valid_mask & ~s_dead;
            unsigned sup = 0;                          // later candidates of the tile this one suppresses if kept
            if (alive) {
                for (int q = 1; q < 32; ++q) {
                    const float4 bq = make_float4(__shfl_sync(0xffffffffu, bj.x, q), __shfl_sync(0xffffffffu, bj.y, q),
                                                  __shfl_sync(0xffffffffu, bj.z, q), __shfl_sync(0xffffffffu, bj.w, q));
                    if (q > lane && !(iou_nms(bj, bq) < thr)) sup |= 1u << q;
                }
                for (int i = 0; i < 31; ++i) {
                    const unsigned si = __shfl_sync(0xffffffffu, sup, i);
                    if ((alive >> i) & 1u) alive &= ~si;
                }
            }
            if ((alive >> lane) & 1u) {
                const int pos = nk + __popc(alive & ((1u << lane) - 1));
                if (pos < cap) {
                    w.keep[pos] = j;
                    if (pos < KEPT_SMEM) s_kept[pos] = bj;
                }
            }
            if (lane == 0) {
                s_nkeep = min(nk + __popc(alive), cap);
                s_dead = 0;
            }
        }
        __syncthreads();
    }
    // 4. gather
    const int nk = s_nkeep;
    const float* raw = a.raw + (size_t)a.rows * 16 * f;
    float scale = a.scale, pad_x = a.pad_x, pad_y = a.pad_y;
    if (a.desc) { scale = a.desc[f].scale; pad_x = (float)a.desc[f].left; pad_y = (float)a.desc[f].top; }
    else if (a.recover) { scale = a.recover[3 * f]; pad_x = a.recover[3 * f + 1]; pad_y = a.recover[3 * f + 2]; }
    float* out = a.kept_rows + (size_t)16 * cap * f;
    int* out_idx = a.kept_idx + (size_t)cap * f;
    for (int e = threadIdx.x; e < nk * 16; e += blockDim.x) {
        const int k = e >> 4, c = e & 15;
        const int rank = w.keep[k];
        const int row = w.row[rank];
        float v;
        if (c < 4) {
            const float4 b = w.box[rank];
            const float bv = c == 0 ? b.x : (c == 1 ? b.y : (c == 2 ? b.z : b.w));
            v = (bv - ((c & 1) ? pad_y : pad_x)) / scale;                // scale_coords, face_detector.py:86-91
        } else {
            v = raw[(size_t)row * 16 + c];
        }
        out[e] = v;
        if (c == 0) out_idx[k] = row;
    }
    if (threadIdx.x == 0) a.count[f] = nk;
}

}  // namespace

size_t nms_workspace_bytes(int cap, int batch) {
    return batch > 0 ? ws_header_bytes(batch) + ws_frame_bytes(cap) * (size_t)batch : 0;
}

int launch_nms(const NmsArgs& a, cudaStream_t s) {
    SKPS_CHECK(a.raw && a.kept_rows && a.kept_idx && a.count && a.ws && a.rows > 0 && a.batch > 0 && a.capacity > 0 &&
               a.limit >= 0 && a.ws_cap >= min(a.rows, a.limit), "nms: bad arguments");
    const int nmax = min(a.rows, a.limit);
    SKPS_CUDA(cudaMemsetAsync(a.ws, 0, sizeof(int) * a.batch, s));
    const int cblocks = min((a.rows + COMPACT_THREADS - 1) / COMPACT_THREADS, 128);
    nms_compact_kernel<<<dim3(cblocks, a.batch), COMPACT_THREADS, 0, s>>>(a);
    SKPS_CUDA(cudaGetLastError());
    if (nmax > 0) {
        nms_chunk_sort_kernel<<<dim3((nmax + SORT_CHUNK - 1) / SORT_CHUNK, a.batch), SORT_THREADS, 0, s>>>(a);
        SKPS_CUDA(cudaGetLastError());
        int pass = 0;
        for (int run = SORT_CHUNK; run < nmax; run *= 2, ++pass) {
            nms_merge_kernel<<<dim3((nmax + MERGE_THREADS - 1) / MERGE_THREADS, a.batch), MERGE_THREADS, 0, s>>>(a, run, pass);
            SKPS_CUDA(cudaGetLastError());
        }
    }
    nms_greedy_kernel<<<a.batch, NMS_THREADS, 0, s>>>(a);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace skps

using namespace skps;

extern "C" SKPS_API int skps_detect_post(const float* raw, int rows, float score_thres, float iou_thres, float scale,
                                         float pad_x, float pad_y, float* kept_rows, int32_t* kept_idx, int32_t* count,
                                         int max_det, void* stream) {
    SKPS_CHECK(raw && kept_rows && kept_idx && count && rows > 0 && max_det > 0 && max_det <= 256, "detect_post: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    constexpr int LIMIT = 1024;        // the documented contract of this entry: more candidates -> count = -candidates
    NmsArgs a = {};
    a.raw = raw; a.rows = rows; a.batch = 1; a.score_thres = score_thres; a.iou_thres = iou_thres;
    a.scale = scale; a.pad_x = pad_x; a.pad_y = pad_y;
    a.limit = LIMIT; a.capacity = max_det; a.kept_rows = kept_rows; a.kept_idx = kept_idx; a.count = count;
    a.ws_cap = min(rows, LIMIT);
    void* ws = nullptr;
    SKPS_CUDA(cudaMallocAsync(&ws, nms_workspace_bytes(a.ws_cap, 1), s));
    a.ws = ws;
    const int rc = launch_nms(a, s);
    cudaFreeAsync(ws, s);
    return rc;
}

extern "C" SKPS_API size_t skps_detect_post_workspace_size(int rows, int batch) {
    return rows > 0 ? nms_workspace_bytes(rows, batch) : 0;
}

extern "C" SKPS_API int skps_detect_post_batch(const float* raw, int rows, int batch, float score_thres, float iou_thres,
                                               const float* recover, float* kept_rows, int32_t* kept_idx, int32_t* count,
                                               int capacity, void* workspace, size_t workspace_bytes, void* stream) {
    SKPS_CHECK(raw && recover && kept_rows && kept_idx && count && workspace && rows > 0 && batch > 0 && capacity > 0,
               "detect_post_batch: bad arguments");
    SKPS_CHECK(workspace_bytes >= nms_workspace_bytes(rows, batch),
               "detect_post_batch: workspace of %zu bytes, %zu needed for %d rows x %d frames", workspace_bytes,
               nms_workspace_bytes(rows, batch), rows, batch);
    NmsArgs a = {};
    a.raw = raw; a.rows = rows; a.batch = batch; a.score_thres = score_thres; a.iou_thres = iou_thres;
    a.recover = recover; a.limit = INT_MAX; a.capacity = capacity;
    a.kept_rows = kept_rows; a.kept_idx = kept_idx; a.count = count;
    a.ws = workspace; a.ws_cap = rows;
    return launch_nms(a, (cudaStream_t)stream);
}
