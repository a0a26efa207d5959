// skps_pipeline: the device-side chain of FaceAna.run (Skps/core/api/facer.py:52-85):
//   frame -> letterbox -> detector -> NMS/un-letterbox -> judge_boxs(track) -> sort_and_filter
//         -> per-face crop+resize -> landmark net -> de-normalise
// One H2D copy of the frame in, the face count read back after the selection, one D2H copy of the
// packed results out.  The landmark net runs on exactly the selected faces, in chunks of at most
// SKPS_LANDMARK_CHUNK, so its activations stay those of one chunk whatever top_k is (up to 1024).
// The temporal smoothing that follows (GroupTrack, facer.py:71-82) is host math on the returned
// landmarks.
#include <string.h>

#include <vector>

#include "../../include/skps_b200.h"
#include "common.h"
#include "mpipe_kernels.h"

using namespace skps;

struct skps_pipeline {
    skps_engine* det = nullptr;
    skps_engine* kps = nullptr;
    skps_pipeline_cfg cfg;
    int device = 0;
    int det_h = 0, det_w = 0, kps_hw = 0, n_points = 0, det_rows = 0;
    static constexpr int RUN_DET = 256;           // kept rows skps_pipeline_run returns; skps_pipeline_det_results has all
    int last_n_det = 0;                           // kept boxes of the last detector run
    void* d_nms_ws = nullptr;                     // NMS workspace for det_rows candidates
    uint8_t* d_frame[2] = {nullptr, nullptr};     // current / previous frame
    int cur = 0;
    int cur_h = 0, cur_w = 0;                     // size of the frame staged in d_frame[cur] by frame_diff* (0 = none)
    int prev_h = 0, prev_w = 0;                   // size of the frame in d_frame[cur^1] (0 = none)
    uint8_t* h_frame = nullptr;                   // pinned staging
    float* d_det_rows = nullptr; int32_t* d_det_idx = nullptr; int32_t* d_det_count = nullptr;
    float* d_track = nullptr;
    // d_boxes / h_boxes: top_k boxes, then the top_k int32 sources of the track ids (one D2H copy for both)
    float* d_boxes = nullptr; int32_t* d_count = nullptr; int32_t* d_detail = nullptr;
    int last_n_faces = 0;                         // faces of the last skps_pipeline_run
    float* d_kps = nullptr; float* d_scores = nullptr;
    int32_t* d_counts = nullptr;                  // d_counts[c] = c for c in 0..SKPS_LANDMARK_CHUNK: per-chunk face counts
    int track_cap = 0;                            // track boxes accepted: max(256, top_k)
    unsigned long long* d_diff = nullptr;
    // packed host result block (pinned)
    struct Host {
        int32_t n_faces, n_det;
        unsigned long long diff;
    };
    Host* h_res = nullptr;
    float* h_boxes = nullptr; float* h_kps = nullptr; float* h_scores = nullptr;
    int32_t* h_det_idx = nullptr; float* h_det_rows = nullptr; float* h_track = nullptr;
    // aligned chips (skps_pipeline_align): allocated on first use, for top_k faces at align_size
    int align_size = 0;
    double* d_align_kps = nullptr; double* d_align_M = nullptr; uint8_t* d_chips = nullptr;
    // head pose (skps_pipeline_pose): allocated on first use, for top_k faces
    double* d_pose_kps = nullptr; double* d_pose = nullptr;
    // device frames: the producer's stream is ordered before the ingest (ev_ready) and the ingest before its later work (ev_read)
    cudaEvent_t ev_ready = nullptr, ev_read = nullptr;
};

extern "C" SKPS_API void skps_pipeline_destroy(skps_pipeline* p) {
    if (!p) return;
    DeviceGuard on(p->device);
    for (int i = 0; i < 2; ++i) if (p->d_frame[i]) cudaFree(p->d_frame[i]);
    if (p->h_frame) cudaFreeHost(p->h_frame);
    void* dev[] = {p->d_det_rows, p->d_det_idx, p->d_det_count, p->d_nms_ws, p->d_track, p->d_boxes, p->d_count, p->d_detail,
                   p->d_kps, p->d_scores, p->d_counts, p->d_diff, p->d_align_kps, p->d_align_M, p->d_chips,
                   p->d_pose_kps, p->d_pose};
    for (void* q : dev) if (q) cudaFree(q);
    void* host[] = {p->h_res, p->h_boxes, p->h_kps, p->h_scores, p->h_det_idx, p->h_det_rows, p->h_track};
    for (void* q : host) if (q) cudaFreeHost(q);
    if (p->ev_ready) cudaEventDestroy(p->ev_ready);
    if (p->ev_read) cudaEventDestroy(p->ev_read);
    delete p;
}

static size_t boxes_block_bytes(int K) { return (sizeof(float) * 4 + sizeof(int32_t)) * (size_t)K; }

extern "C" SKPS_API int skps_pipeline_create(skps_engine* det, skps_engine* kps, const skps_pipeline_cfg* cfg,
                                    skps_pipeline** out) {
    SKPS_CHECK(det && kps && cfg && out, "pipeline_create: null argument");
    SKPS_CHECK(cfg->top_k > 0 && cfg->top_k <= SKPS_MAX_TOP_K, "pipeline_create: top_k %d outside 1..%d", cfg->top_k,
               SKPS_MAX_TOP_K);
    int device = 0;
    if (engine_pair_device(det, kps, "pipeline_create", &device)) return 1;
    SKPS_ON_DEVICE(device);
    int c = 0, det_h = 0, det_w = 0, kh = 0, kw = 0;
    skps_engine_input_dims(det, &det_h, &det_w, &c);
    skps_engine_input_dims(kps, &kh, &kw, &c);
    SKPS_CHECK(kh == kw, "pipeline_create: landmark input must be square");
    SKPS_CHECK(skps_engine_num_outputs(det) == 1 && skps_engine_num_outputs(kps) == 2, "pipeline_create: engine outputs");
    const int P = skps_engine_output_elems(kps, 1), K = cfg->top_k;
    SKPS_CHECK(skps_engine_output_elems(kps, 0) == 2 * P, "pipeline_create: landmark outputs");
    skps_pipeline* p = new skps_pipeline();
    p->det = det; p->kps = kps; p->cfg = *cfg;
    p->det_h = det_h; p->det_w = det_w; p->kps_hw = kh; p->n_points = P;
    p->det_rows = skps_engine_output_elems(det, 0) / 16;
    p->device = device;
    auto fail = [&](const char* what) {
        prefix_error("pipeline_create", what);
        skps_pipeline_destroy(p);
        return 1;
    };
    const size_t fbytes = (size_t)cfg->max_h * cfg->max_w * 3;
    SKPS_DEV_ALLOC(p->d_frame[0], fbytes); SKPS_DEV_ALLOC(p->d_frame[1], fbytes);
    SKPS_HOST_ALLOC(p->h_frame, fbytes);
    // every row of the detector can be a kept box: room for all of them, sized once here
    SKPS_DEV_ALLOC(p->d_det_rows, sizeof(float) * 16 * p->det_rows);
    SKPS_DEV_ALLOC(p->d_det_idx, sizeof(int32_t) * p->det_rows);
    SKPS_DEV_ALLOC(p->d_det_count, sizeof(int32_t));
    SKPS_DEV_ALLOC(p->d_nms_ws, nms_workspace_bytes(p->det_rows, 1));
    p->track_cap = K > 256 ? K : 256;
    SKPS_DEV_ALLOC(p->d_track, sizeof(float) * 4 * p->track_cap);
    SKPS_DEV_ALLOC(p->d_boxes, boxes_block_bytes(K));
    SKPS_DEV_ALLOC(p->d_count, sizeof(int32_t));
    SKPS_DEV_ALLOC(p->d_detail, sizeof(int32_t) * 5 * K);
    SKPS_DEV_ALLOC(p->d_kps, sizeof(float) * 2 * P * K);
    SKPS_DEV_ALLOC(p->d_scores, sizeof(float) * P * K);
    SKPS_DEV_ALLOC(p->d_counts, sizeof(int32_t) * (SKPS_LANDMARK_CHUNK + 1));
    SKPS_DEV_ALLOC(p->d_diff, sizeof(unsigned long long));
    SKPS_HOST_ALLOC(p->h_res, sizeof(skps_pipeline::Host));
    SKPS_HOST_ALLOC(p->h_boxes, boxes_block_bytes(K));
    SKPS_HOST_ALLOC(p->h_kps, sizeof(float) * 2 * P * K);
    SKPS_HOST_ALLOC(p->h_scores, sizeof(float) * P * K);
    SKPS_HOST_ALLOC(p->h_det_idx, sizeof(int32_t) * skps_pipeline::RUN_DET);
    SKPS_HOST_ALLOC(p->h_det_rows, sizeof(float) * 16 * skps_pipeline::RUN_DET);
    SKPS_HOST_ALLOC(p->h_track, sizeof(float) * 4 * p->track_cap);
    int32_t counts[SKPS_LANDMARK_CHUNK + 1];
    for (int i = 0; i <= SKPS_LANDMARK_CHUNK; ++i) counts[i] = i;
    if (cudaMemset(p->d_det_count, 0, sizeof(int32_t)) != cudaSuccess ||
        cudaMemcpy(p->d_counts, counts, sizeof(counts), cudaMemcpyHostToDevice) != cudaSuccess) {
        set_error("%s", cudaGetErrorString(cudaGetLastError()));
        return fail("init");
    }
    if (cudaEventCreateWithFlags(&p->ev_ready, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&p->ev_read, cudaEventDisableTiming) != cudaSuccess) { set_error("cudaEventCreate"); return fail("event"); }
    *out = p;
    return 0;
}

extern "C" SKPS_API int skps_pipeline_reset(skps_pipeline* p) {
    SKPS_CHECK(p, "pipeline_reset: null");
    p->prev_h = p->prev_w = 0;            // FaceAna.reset (facer.py:200-208): previous_image = None
    p->last_n_faces = 0;
    return 0;
}

static int check_frame_size(const skps_pipeline* p, int H, int W) {
    SKPS_CHECK(H > 0 && W > 0 && (size_t)H * W <= (size_t)p->cfg.max_h * p->cfg.max_w,
               "frame %dx%d has more pixels than the pipeline maximum %dx%d", H, W, p->cfg.max_h, p->cfg.max_w);
    return 0;
}

// facer.py:113: np.sum(diff)/H/W/3, from the sum in d_diff.
static int read_mean_diff(skps_pipeline* p, int H, int W, double* mean_diff, cudaStream_t s) {
    SKPS_CUDA(cudaMemcpyAsync(&p->h_res->diff, p->d_diff, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    SKPS_CUDA(cudaStreamSynchronize(s));
    *mean_diff = (double)p->h_res->diff / (double)H / (double)W / 3.0;
    return 0;
}

extern "C" SKPS_API int skps_pipeline_frame_diff(skps_pipeline* p, const uint8_t* frame, int H, int W, double* mean_diff,
                                                 void* stream) {
    SKPS_CHECK(p && frame && mean_diff, "frame_diff: null argument");
    cudaStream_t s = (cudaStream_t)stream;
    SKPS_ON_DEVICE(p->device);
    if (check_frame_size(p, H, W)) return 1;
    const size_t n = (size_t)H * W * 3;
    if (upload_host_frame(frame, n, p->h_frame, p->d_frame[p->cur], s)) return 1;
    p->cur_h = H; p->cur_w = W;
    if (p->prev_h != H || p->prev_w != W) {
        *mean_diff = -1.0;
        return 0;
    }
    SKPS_CUDA(cudaMemsetAsync(p->d_diff, 0, sizeof(unsigned long long), s));
    MpStreamDesc D = {};
    D.cur = p->d_frame[p->cur]; D.prev = p->d_frame[p->cur ^ 1]; D.have_prev = 1; D.H = H; D.W = W;
    if (launch_frame_diff(nullptr, 1, D, n, p->d_diff, s)) return 1;
    return read_mean_diff(p, H, W, mean_diff, s);
}

// One ingest pass gathers the [dev] frame, in any pixel layout, into d_frame[cur] as BGR and, against a previous frame of
// the same size, sums the difference.  The read waits for the work queued on the producer stream so far, and the
// producer's later work waits for the read.
// A frame stored turned `turns` quarter turns clockwise is staged upright by the same pass: from then on the pipeline sees
// the upright frame, of size W x H for odd turns.
extern "C" SKPS_API int skps_pipeline_frame_diff_device_rotate(skps_pipeline* p, const uint8_t* frame, int H, int W, int pitch,
                                                               int layout, int plane_pitch, int turns, void* producer_stream,
                                                               double* mean_diff, void* stream) {
    SKPS_CHECK(p && frame && mean_diff, "frame_diff_device: null argument");
    SKPS_CHECK(layout_ok(layout), "frame_diff_device: unknown pixel layout %d", layout);
    SKPS_CHECK(turns >= 0 && turns <= 3, "frame_diff_device: turns %d outside 0..3", turns);
    SKPS_CHECK(H == 1 || pitch >= layout_xstep(layout) * W, "frame_diff_device: row pitch %d is less than %d x width %d",
               pitch, layout_xstep(layout), W);
    SKPS_CHECK(layout < SKPS_LAYOUT_BGR_PLANAR || plane_pitch >= 0, "frame_diff_device: plane pitch %d < 0", plane_pitch);
    cudaStream_t s = (cudaStream_t)stream, producer = (cudaStream_t)producer_stream;
    SKPS_ON_DEVICE(p->device);
    if (check_device_frame(frame, p->device, "frame_diff_device", -1) || check_frame_size(p, H, W)) return 1;
    const int Hu = (turns & 1) ? W : H, Wu = (turns & 1) ? H : W;         // the upright frame
    const bool diff = p->prev_h == Hu && p->prev_w == Wu;
    SKPS_CUDA(cudaEventRecord(p->ev_ready, producer));
    SKPS_CUDA(cudaStreamWaitEvent(s, p->ev_ready, 0));
    MpStreamDesc D = {};
    D.cur = p->d_frame[p->cur]; D.prev = diff ? p->d_frame[p->cur ^ 1] : nullptr; D.have_prev = diff;
    D.H = Hu; D.W = Wu; D.src = frame; D.src_pitch = pitch; D.src_plane = plane_pitch;
    if (diff) SKPS_CUDA(cudaMemsetAsync(p->d_diff, 0, sizeof(unsigned long long), s));
    if (launch_frame_diff(nullptr, 1, D, (size_t)H * W * 3, p->d_diff, s, layout, nullptr, turns)) return 1;
    SKPS_CUDA(cudaEventRecord(p->ev_read, s));
    SKPS_CUDA(cudaStreamWaitEvent(producer, p->ev_read, 0));
    p->cur_h = Hu; p->cur_w = Wu;
    if (!diff) {
        *mean_diff = -1.0;
        return 0;
    }
    return read_mean_diff(p, Hu, Wu, mean_diff, s);
}

extern "C" SKPS_API int skps_pipeline_frame_diff_device_layout(skps_pipeline* p, const uint8_t* frame, int H, int W, int pitch,
                                                               int layout, int plane_pitch, void* producer_stream,
                                                               double* mean_diff, void* stream) {
    return skps_pipeline_frame_diff_device_rotate(p, frame, H, W, pitch, layout, plane_pitch, 0, producer_stream, mean_diff,
                                                  stream);
}

extern "C" SKPS_API int skps_pipeline_frame_diff_device(skps_pipeline* p, const uint8_t* frame, int H, int W, int pitch,
                                                        void* producer_stream, double* mean_diff, void* stream) {
    return skps_pipeline_frame_diff_device_layout(p, frame, H, W, pitch, SKPS_LAYOUT_BGR, 0, producer_stream, mean_diff,
                                                  stream);
}

// The staged frame becomes the "previous" frame (facer.py:57,62: previous_image is replaced every frame).
static void advance_frame(skps_pipeline* p) {
    p->prev_h = p->cur_h; p->prev_w = p->cur_w;
    p->cur_h = p->cur_w = 0;
    p->cur ^= 1;
}

// The frame staged by skps_pipeline_frame_diff* becomes the "previous" frame without running the chain (FaceAna.run on
// a static frame with nothing to track, facer.py:57-62).
extern "C" SKPS_API int skps_pipeline_commit_frame(skps_pipeline* p) {
    SKPS_CHECK(p, "commit_frame: null");
    SKPS_CHECK(p->cur_h > 0, "commit_frame: no frame staged (call skps_pipeline_frame_diff or _frame_diff_device first)");
    advance_frame(p);
    p->last_n_faces = 0;
    return 0;
}

extern "C" SKPS_API int skps_pipeline_run(skps_pipeline* p, int run_detector, int rw, int rh, int top, int left, float scale,
                                          const float* track, int n_track, int32_t* n_faces, float* boxes4, float* kps,
                                          float* scores, int32_t* n_det, int32_t* det_idx, float* det_rows, void* stream) {
    SKPS_CHECK(p && n_faces && boxes4 && kps && scores, "pipeline_run: null argument");
    SKPS_CHECK(p->cur_h > 0, "pipeline_run: no frame staged (call skps_pipeline_frame_diff or _frame_diff_device first)");
    SKPS_CHECK(n_track >= 0 && n_track <= p->track_cap, "pipeline_run: n_track %d outside 0..%d", n_track, p->track_cap);
    cudaStream_t s = (cudaStream_t)stream;
    SKPS_ON_DEVICE(p->device);
    const skps_pipeline_cfg& c = p->cfg;
    const int K = c.top_k, P = p->n_points, H = p->cur_h, W = p->cur_w;
    const uint8_t* d_frame = p->d_frame[p->cur];
    int32_t* d_src = (int32_t*)(p->d_boxes + 4 * K);
    if (n_track > 0) {
        SKPS_CHECK(track, "pipeline_run: track is null");
        memcpy(p->h_track, track, sizeof(float) * 4 * n_track);
        SKPS_CUDA(cudaMemcpyAsync(p->d_track, p->h_track, sizeof(float) * 4 * n_track, cudaMemcpyHostToDevice, s));
    }
    if (run_detector) {
        SKPS_CHECK(rw > 0 && rh > 0, "pipeline_run: letterbox size %dx%d", rw, rh);
        uint8_t* det_in = (uint8_t*)skps_engine_input_ptr(p->det);
        LetterboxArgs la = {};
        la.frame = d_frame; la.H = H; la.W = W; la.pitch = W * 3; la.rw = rw; la.rh = rh; la.top = top; la.left = left;
        la.out = det_in; la.in_h = p->det_h; la.in_w = p->det_w;
        if (launch_letterbox(la, 1, s)) return 1;
        if (skps_engine_forward(p->det, det_in, 1, nullptr, s)) return 1;
        NmsArgs na = {};
        na.raw = skps_engine_output_ptr(p->det, 0); na.rows = p->det_rows; na.batch = 1;
        na.score_thres = c.score_thres; na.iou_thres = c.iou_thres;
        na.scale = scale; na.pad_x = (float)left; na.pad_y = (float)top;
        na.limit = p->det_rows; na.capacity = p->det_rows;
        na.kept_rows = p->d_det_rows; na.kept_idx = p->d_det_idx; na.count = p->d_det_count;
        na.ws = p->d_nms_ws; na.ws_cap = p->det_rows;
        if (launch_nms(na, s)) return 1;
    }
    // facer.py:58 judge_boxs(track_box, boxes) on the detector's boxes, or :61 boxes = track_box; then :64 sort_and_filter
    SelectArgs sa = {};
    sa.det_rows = p->d_det_rows; sa.det_count = p->d_det_count; sa.det_stride = 16; sa.flag1 = run_detector != 0;
    sa.track = p->d_track; sa.n_track1 = n_track;
    sa.iou_thres = c.track_iou; sa.alpha = c.alpha; sa.one_minus_alpha = (float)(1.0 - (double)c.alpha);
    sa.min_face = c.min_face; sa.top_k = K;
    sa.boxes4 = p->d_boxes; sa.count = p->d_count; sa.src = d_src;
    if (launch_select(sa, 1, s)) return 1;
    // the face count decides how many crops the landmark net sees
    SKPS_CUDA(cudaMemcpyAsync(&p->h_res->n_faces, p->d_count, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    SKPS_CUDA(cudaStreamSynchronize(s));
    const int nf = p->h_res->n_faces;
    // chunks of exactly the selected faces: the crops go straight into the engine's input, the landmarks and scores of
    // each chunk to their offsets in d_kps / d_scores (the next chunk overwrites the engine's outputs)
    uint8_t* kps_in = (uint8_t*)skps_engine_input_ptr(p->kps);
    CropArgs ca = {};
    ca.frame = d_frame; ca.H = H; ca.W = W; ca.pitch = W * 3;
    ca.face_scale = c.face_scale; ca.min_face = c.kps_min_face; ca.crops = kps_in; ca.S = p->kps_hw;
    for (int f0 = 0; f0 < nf; f0 += SKPS_LANDMARK_CHUNK) {
        const int nc = nf - f0 < SKPS_LANDMARK_CHUNK ? nf - f0 : SKPS_LANDMARK_CHUNK;
        const int32_t* d_nc = p->d_counts + nc;
        ca.boxes = p->d_boxes + 4 * f0; ca.count = d_nc; ca.K = nc; ca.detail = p->d_detail + 5 * f0;
        if (launch_crop(ca, 1, s)) return 1;
        float* outs[2] = {nullptr, p->d_scores + (size_t)P * f0};
        if (skps_engine_forward(p->kps, kps_in, nc, outs, s)) return 1;
        if (launch_landmark_post(skps_engine_output_ptr(p->kps, 0), p->d_detail + 5 * f0, d_nc, nc, P,
                                 p->d_kps + (size_t)2 * P * f0, 1, s))
            return 1;
    }
    if (nf > 0) {
        SKPS_CUDA(cudaMemcpyAsync(p->h_boxes, p->d_boxes, boxes_block_bytes(K), cudaMemcpyDeviceToHost, s));
        SKPS_CUDA(cudaMemcpyAsync(p->h_kps, p->d_kps, sizeof(float) * 2 * P * nf, cudaMemcpyDeviceToHost, s));
        SKPS_CUDA(cudaMemcpyAsync(p->h_scores, p->d_scores, sizeof(float) * P * nf, cudaMemcpyDeviceToHost, s));
    }
    if (run_detector) SKPS_CUDA(cudaMemcpyAsync(&p->h_res->n_det, p->d_det_count, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (run_detector && n_det) {
        // the first RUN_DET kept rows (what callers of this function size their buffers for); the rest stay on the device
        // for skps_pipeline_det_results
        const int R = skps_pipeline::RUN_DET < p->det_rows ? skps_pipeline::RUN_DET : p->det_rows;
        SKPS_CUDA(cudaMemcpyAsync(p->h_det_idx, p->d_det_idx, sizeof(int32_t) * R, cudaMemcpyDeviceToHost, s));
        SKPS_CUDA(cudaMemcpyAsync(p->h_det_rows, p->d_det_rows, sizeof(float) * 16 * R, cudaMemcpyDeviceToHost, s));
    }
    SKPS_CUDA(cudaStreamSynchronize(s));
    if (run_detector) p->last_n_det = p->h_res->n_det;
    p->last_n_faces = nf;
    *n_faces = nf;
    memcpy(boxes4, p->h_boxes, sizeof(float) * 4 * nf);
    memcpy(kps, p->h_kps, sizeof(float) * 2 * P * nf);
    memcpy(scores, p->h_scores, sizeof(float) * P * nf);
    if (n_det) {
        *n_det = run_detector ? p->h_res->n_det : 0;
        const int nr = *n_det < skps_pipeline::RUN_DET ? *n_det : skps_pipeline::RUN_DET;
        if (run_detector && det_idx) memcpy(det_idx, p->h_det_idx, sizeof(int32_t) * nr);
        if (run_detector && det_rows) memcpy(det_rows, p->h_det_rows, sizeof(float) * 16 * nr);
    }
    advance_frame(p);
    return 0;
}

// The sources skps_pipeline_run's selection found, kept in host memory by its D2H copy: no device work, no synchronisation.
extern "C" SKPS_API int skps_pipeline_face_sources(skps_pipeline* p, int n, int32_t* src) {
    SKPS_CHECK(p && src, "pipeline_face_sources: null argument");
    SKPS_CHECK(n >= 0 && n <= p->last_n_faces, "pipeline_face_sources: the last run returned %d faces, asked for %d",
               p->last_n_faces, n);
    memcpy(src, (const int32_t*)(p->h_boxes + 4 * p->cfg.top_k), sizeof(int32_t) * n);
    return 0;
}

// Every kept row of the last detector run, copied from the device on request: a crowd can keep thousands of boxes, and
// skps_pipeline_run returns only the first 256 so that no frame pays for copying them all.
extern "C" SKPS_API int skps_pipeline_det_results(skps_pipeline* p, int capacity, int32_t* det_idx, float* det_rows) {
    SKPS_CHECK(p, "pipeline_det_results: null");
    const int n = p->last_n_det;
    SKPS_CHECK(capacity >= n, "pipeline_det_results: the last detector run kept %d boxes, capacity is %d", n, capacity);
    if (n == 0) return 0;
    SKPS_ON_DEVICE(p->device);
    if (det_idx) SKPS_CUDA(cudaMemcpy(det_idx, p->d_det_idx, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
    if (det_rows) SKPS_CUDA(cudaMemcpy(det_rows, p->d_det_rows, sizeof(float) * 16 * n, cudaMemcpyDeviceToHost));
    return 0;
}

// Aligned chips from the frame of the last run / commit, which is d_frame[cur ^ 1] (prev_h x prev_w) until the next frame
// is staged.  The landmarks were smoothed on the host (GroupTrack), so they come up; n x 98 x 2 doubles are tiny.
extern "C" SKPS_API int skps_pipeline_align(skps_pipeline* p, const double* kps, int n, int size, uint8_t* chips, double* M,
                                            void* stream) {
    SKPS_CHECK(p && kps && chips && M, "pipeline_align: null argument");
    SKPS_CHECK(n > 0 && n <= p->cfg.top_k, "pipeline_align: %d faces, expected 1..%d", n, p->cfg.top_k);
    SKPS_CHECK(size >= 16 && size <= 512, "pipeline_align: size %d outside 16..512", size);
    SKPS_CHECK(p->prev_h > 0 && p->prev_w > 0, "pipeline_align: no frame (run the pipeline first)");
    cudaStream_t s = (cudaStream_t)stream;
    SKPS_ON_DEVICE(p->device);
    const int K = p->cfg.top_k, P = p->n_points;
    const size_t chip_bytes = (size_t)size * size * 3;
    if (p->align_size != size) {
        SKPS_CUDA(cudaStreamSynchronize(s));
        void* old[] = {p->d_align_kps, p->d_align_M, p->d_chips};
        for (void* q : old) if (q) cudaFree(q);
        p->d_align_kps = p->d_align_M = nullptr; p->d_chips = nullptr; p->align_size = 0;
        SKPS_CUDA(cudaMalloc((void**)&p->d_align_kps, sizeof(double) * 2 * P * K));
        SKPS_CUDA(cudaMalloc((void**)&p->d_align_M, sizeof(double) * 6 * K));
        SKPS_CUDA(cudaMalloc((void**)&p->d_chips, chip_bytes * K));
        p->align_size = size;
    }
    const int H = p->prev_h, W = p->prev_w;
    SKPS_CUDA(cudaMemcpyAsync(p->d_align_kps, kps, sizeof(double) * 2 * P * n, cudaMemcpyHostToDevice, s));
    if (skps_align_faces(p->d_frame[p->cur ^ 1], H, W, W * 3, p->d_align_kps, nullptr, n, P, size, p->d_chips, p->d_align_M, s))
        return 1;
    SKPS_CUDA(cudaMemcpyAsync(chips, p->d_chips, chip_bytes * n, cudaMemcpyDeviceToHost, s));
    SKPS_CUDA(cudaMemcpyAsync(M, p->d_align_M, sizeof(double) * 6 * n, cudaMemcpyDeviceToHost, s));
    SKPS_CUDA(cudaStreamSynchronize(s));
    return 0;
}

// Head pose of n faces whose landmarks were smoothed on the host: kps [host] (n, n_points, 2) float64, frame H x W for the
// camera.  The 98-point get_head_pose of the training tree on the GPU, ordered on `stream`.
extern "C" SKPS_API int skps_pipeline_pose(skps_pipeline* p, const double* kps, int n, int H, int W, double* rvec, double* tvec,
                                           double* euler, double* reproject, void* stream) {
    SKPS_CHECK(p && kps && rvec && tvec && euler && reproject, "pipeline_pose: null argument");
    SKPS_CHECK(n > 0 && n <= p->cfg.top_k, "pipeline_pose: %d faces, expected 1..%d", n, p->cfg.top_k);
    SKPS_CHECK(H > 0 && W > 0, "pipeline_pose: bad frame size %dx%d", H, W);
    SKPS_CHECK(p->n_points >= 98, "pipeline_pose: %d landmarks per face, expected 98", p->n_points);
    cudaStream_t s = (cudaStream_t)stream;
    SKPS_ON_DEVICE(p->device);
    const int K = p->cfg.top_k, P = p->n_points;
    if (!p->d_pose) {
        SKPS_CUDA(cudaMalloc((void**)&p->d_pose_kps, sizeof(double) * 2 * P * K));
        SKPS_CUDA(cudaMalloc((void**)&p->d_pose, sizeof(double) * 25 * K));
    }
    SKPS_CUDA(cudaMemcpyAsync(p->d_pose_kps, kps, sizeof(double) * 2 * P * n, cudaMemcpyHostToDevice, s));
    PoseArgs a = {};
    pose_model_98(a);
    a.pts64 = p->d_pose_kps; a.G = 1; a.K = n; a.P = P; a.H = H; a.W = W;
    a.rvec = p->d_pose; a.tvec = p->d_pose + 3 * n; a.euler = p->d_pose + 6 * n; a.reproj = p->d_pose + 9 * n;
    if (launch_head_pose(a, s)) return 1;
    SKPS_CUDA(cudaMemcpyAsync(rvec, a.rvec, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, s));
    SKPS_CUDA(cudaMemcpyAsync(tvec, a.tvec, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, s));
    SKPS_CUDA(cudaMemcpyAsync(euler, a.euler, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, s));
    SKPS_CUDA(cudaMemcpyAsync(reproject, a.reproj, sizeof(double) * 16 * n, cudaMemcpyDeviceToHost, s));
    SKPS_CUDA(cudaStreamSynchronize(s));
    return 0;
}
