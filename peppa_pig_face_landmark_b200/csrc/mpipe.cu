// skps_mpipe: FaceAna.run (Skps/core/api/facer.py:52-85) for MANY concurrent video streams on one GPU.
//
// One call takes one frame from each of up to S streams, any subset of them in any order, and runs, batched across the
// call's frames and with every piece of per-stream state resident in HBM:
//   H2D (copy stream, overlapped with the previous batch's compute) -> |prev - cur| gate (which gathers frames already on
//   the device into the ring in the same pass) -> letterbox x m ->
//   ONE detector forward (batch m: the keyframes of skps_mpipe_set_detect_every, all S streams by default) -> NMS x m ->
//   judge_boxs/sort_and_filter x S (detector rows or track boxes, chosen on the device by the gate) -> crops x S -> ONE landmark forward (batch S * top_k) -> de-normalise -> GroupTrack / One-Euro /
//   track-box EMA x S (temporal.cu, float64 with numpy's promotion rules) -> D2H of the packed results.
// The host never sees a decision: which streams re-detect, how many faces each has and all smoothing state are device
// data.  Two result slots let the caller keep two batches in flight (submit(0) submit(1) wait(0) submit(0) ...): the frames
// of batch i+1 cross PCIe while batch i computes.  SURVEY.md 8f-1 (temporal layer for many streams) and 8f-2 (frame ring).
#include <math.h>
#include <string.h>

#include <vector>

#include "../../include/skps_b200.h"
#include "common.h"
#include "mpipe_kernels.h"

using namespace skps;

struct skps_mpipe {
    skps_engine* det = nullptr;
    skps_engine* kps = nullptr;
    skps_pipeline_cfg cfg;
    int device = 0, S = 0, K = 0, P = 0;
    int det_h = 0, det_w = 0, kps_hw = 0, det_rows = 0;     // every detector row can be a kept box: room for det_rows
    size_t frame_bytes = 0;
    cudaStream_t s_copy = nullptr, s_compute = nullptr;
    // per stream: ring of 3 frames (previous / current / next batch's upload)
    std::vector<uint8_t*> d_frame;            // [S*3]
    std::vector<int> ring_pos;                // [S] index of the most recent frame in the ring
    std::vector<int> prev_h, prev_w;          // [S] size of the most recent frame (0 = none: FaceAna.reset)
    // detection cadence (skps_mpipe_set_detect_every): frames of each stream since create / reset
    int detect_every = 1;
    std::vector<long long> frame_idx;         // [S]
    // per slot
    struct Slot {
        uint8_t* h_stage = nullptr;           // pinned staging for pageable frames [S][frame_bytes]
        int32_t* h_hw = nullptr; int32_t* h_have_prev = nullptr; int32_t* h_geom = nullptr;     // pinned, uploaded per batch
        MpStreamDesc* h_desc = nullptr;       // pinned [2S]: per-stream frame pointers + letterbox geometry of this batch,
                                              // then those of its keyframes, packed
        int32_t* h_det_slot = nullptr;        // pinned [S]: detector frame of each stream, -1 for none
        int32_t* h_stream = nullptr;          // pinned [S]: stream of each frame of the batch (uploaded when not the identity)
        int32_t* h_turns = nullptr;           // pinned [S]: quarter turns of each device frame (uploaded when one is turned)
        int32_t* h_count = nullptr; int32_t* h_flag = nullptr;
        double* h_box = nullptr; double* h_kps = nullptr; float* h_scores = nullptr;
        uint8_t* h_chips = nullptr; double* h_M = nullptr;     // pinned, only while alignment is on
        double* h_pose = nullptr;             // pinned, only while pose is on: rvec, tvec, euler [n][K][3], reproject [n][K][8][2]
        int64_t* h_ids = nullptr;             // pinned [S][K] track ids
        cudaEvent_t ev_in = nullptr, ev_done = nullptr;
        cudaEvent_t ev_staged = nullptr;      // the batch's uploads from the pinned h_hw / h_have_prev / h_desc are done
        int n = 0;
        int m = 0;                            // frames the detector ran on (keyframes of the batch)
        int align = 0;                        // chip size this slot's batch was submitted with (0 = none)
        bool pose = false;                    // this slot's batch was submitted with pose on
        bool busy = false;
        bool device_out = false;              // the batch's results go to caller buffers (skps_mpipe_wait_stream)
    } slot[2];
    // device frames: the producer's stream is ordered before the ingest (ev_ready) and the ingest before its later work (ev_read)
    cudaEvent_t ev_ready = nullptr, ev_read = nullptr;
    // aligned chips (skps_mpipe_set_align): [S][K][size][size][3] / [S][K][2][3], allocated only while align_size > 0
    int align_size = 0;
    uint8_t* d_chips = nullptr; double* d_align_M = nullptr;
    // head pose (skps_mpipe_set_pose): [S][K][25] doubles, allocated only while pose_on
    bool pose_on = false;
    double* d_pose = nullptr;
    // device scratch (one set: batches are serialised on s_compute)
    int32_t *d_hw = nullptr, *d_have_prev = nullptr, *d_flag = nullptr, *d_det_count = nullptr, *d_det_idx = nullptr;
    int32_t *d_count = nullptr, *d_detail = nullptr, *d_det_slot = nullptr;
    int32_t* d_stream = nullptr;              // [S] the batch's call -> stream map, when it is not the identity
    int32_t* d_turns = nullptr;               // [S] the batch's quarter turns, when a frame is turned
    unsigned long long* d_diff = nullptr;
    MpStreamDesc* d_desc = nullptr;           // this batch's descriptors (uploaded on the compute stream, in order) [2S]
    void* d_nms_ws = nullptr;                 // NMS workspace, det_rows candidates per stream
    float *d_det_rows = nullptr, *d_boxes = nullptr, *d_kps_now = nullptr;
    // temporal state
    double *d_prev_lm = nullptr, *d_prev_dx = nullptr, *d_track = nullptr, *d_out_kps = nullptr;
    float* d_track_f32 = nullptr;
    int32_t *d_n_prev = nullptr, *d_prev_f32 = nullptr, *d_state_idx = nullptr, *d_n_track = nullptr;
    // track ids: the source of each selected face, the id of each track box, the next unused id per stream
    int32_t* d_src = nullptr;                 // [S][K]
    int64_t* d_ids = nullptr;                 // [S][K]
    int64_t* d_next_id = nullptr;             // [S]
    // the batch's track boxes and ids in call order, copied out by the temporal step when the map is not the identity
    double* d_out_box = nullptr;              // [S][K][4]
    int64_t* d_out_ids = nullptr;             // [S][K]
    // id memory (skps_mpipe_set_id_memory): each stream's lost tracks, at most K, most recently lost first
    int id_memory = 0;
    int64_t* d_mem_ids = nullptr;             // [S][K]
    float* d_mem_box = nullptr;               // [S][K][4]
    int32_t *d_mem_gap = nullptr, *d_mem_n = nullptr;     // [S][K], [S]
};

static void letterbox_geometry(int H, int W, int in_h, int in_w, float* scale, int* rw, int* rh, int* top, int* left) {
    // face_detector.py:49-62 (python floats = double; int() truncates; round() half-to-even on x.4 / x.6 never ties)
    const double s = fmin((double)in_h / H, (double)in_w / W);
    *rw = (int)(W * s); *rh = (int)(H * s);
    const double dw = (in_w - *rw) / 2.0, dh = (in_h - *rh) / 2.0;
    *top = (int)nearbyint(dh - 0.1); *left = (int)nearbyint(dw - 0.1);
    *scale = (float)s;
}

void skps::mp_temporal_constants(const skps_pipeline_cfg& c, MpTemporalArgs& a) {
    // the python floats of lk.py / facer.py, evaluated in the same order
    // (the cfg carries them as float32; Skps.yml's 0.5 / 0.3 come back exactly by rounding to 6 decimals in double)
    a.iou_thres = nearbyint((double)c.track_iou * 1e6) / 1e6;
    a.alpha = nearbyint((double)c.alpha * 1e6) / 1e6;
    a.one_minus_alpha = 1.0 - a.alpha;
    a.two_pi = 2 * 3.141592653589793;
    { const double r = a.two_pi * 1.0 * 1.0; a.a_d = r / (r + 1); a.one_minus_a_d = 1 - a.a_d; }
    a.min_cutoff = 0.15; a.beta = 0.8;
}

extern "C" SKPS_API void skps_mpipe_destroy(skps_mpipe* p) {
    if (!p) return;
    DeviceGuard on(p->device);
    if (p->s_compute) cudaStreamSynchronize(p->s_compute);
    if (p->s_copy) cudaStreamSynchronize(p->s_copy);
    for (uint8_t* f : p->d_frame) if (f) cudaFree(f);
    for (auto& sl : p->slot) {
        void* host[] = {sl.h_desc, sl.h_det_slot, sl.h_stream, sl.h_turns, sl.h_stage, sl.h_hw, sl.h_have_prev, sl.h_geom, sl.h_count, sl.h_flag, sl.h_box,
                        sl.h_kps, sl.h_scores, sl.h_chips, sl.h_M, sl.h_pose, sl.h_ids};
        for (void* q : host) if (q) cudaFreeHost(q);
        if (sl.ev_in) cudaEventDestroy(sl.ev_in);
        if (sl.ev_done) cudaEventDestroy(sl.ev_done);
        if (sl.ev_staged) cudaEventDestroy(sl.ev_staged);
    }
    if (p->ev_ready) cudaEventDestroy(p->ev_ready);
    if (p->ev_read) cudaEventDestroy(p->ev_read);
    void* dev[] = {p->d_desc, p->d_hw, p->d_have_prev, p->d_flag, p->d_det_count, p->d_det_idx, p->d_count, p->d_detail, p->d_diff,
                   p->d_det_rows, p->d_boxes, p->d_kps_now, p->d_prev_lm, p->d_prev_dx, p->d_track, p->d_out_kps,
                   p->d_track_f32, p->d_n_prev, p->d_prev_f32, p->d_state_idx, p->d_n_track, p->d_chips, p->d_align_M, p->d_pose,
                   p->d_nms_ws, p->d_src, p->d_ids, p->d_next_id, p->d_det_slot, p->d_mem_ids, p->d_mem_box, p->d_mem_gap,
                   p->d_mem_n, p->d_stream, p->d_turns, p->d_out_box, p->d_out_ids};
    for (void* q : dev) if (q) cudaFree(q);
    if (p->s_copy) cudaStreamDestroy(p->s_copy);
    if (p->s_compute) cudaStreamDestroy(p->s_compute);
    delete p;
}

extern "C" SKPS_API int skps_mpipe_reset(skps_mpipe* p, int stream) {
    SKPS_CHECK(p && stream >= -1 && stream < p->S, "mpipe_reset: bad stream %d", stream);
    SKPS_ON_DEVICE(p->device);
    SKPS_CUDA(cudaStreamSynchronize(p->s_compute));
    const int a = stream < 0 ? 0 : stream, b = stream < 0 ? p->S : stream + 1;
    for (int s = a; s < b; ++s) {
        // FaceAna.reset (facer.py:200-208) + a fresh GroupTrack: no previous frame, no track boxes, no landmark history;
        // track ids number from 0 again, with no lost tracks remembered
        p->prev_h[s] = p->prev_w[s] = 0;
        p->frame_idx[s] = 0;
        const int32_t zero = 0, none = -1, one = 1;
        SKPS_CUDA(cudaMemcpy(p->d_n_track + s, &zero, 4, cudaMemcpyHostToDevice));
        SKPS_CUDA(cudaMemsetAsync(p->d_next_id + s, 0, 8, p->s_compute));
        SKPS_CUDA(cudaMemsetAsync(p->d_mem_n + s, 0, 4, p->s_compute));
        SKPS_CUDA(cudaMemsetAsync(p->d_ids + (size_t)s * p->K, 0xff, 8 * (size_t)p->K, p->s_compute));
        SKPS_CUDA(cudaMemcpy(p->d_n_prev + s, &none, 4, cudaMemcpyHostToDevice));
        SKPS_CUDA(cudaMemcpy(p->d_prev_f32 + s, &one, 4, cudaMemcpyHostToDevice));
    }
    return 0;
}

extern "C" SKPS_API int skps_mpipe_create(skps_engine* det, skps_engine* kps, const skps_pipeline_cfg* cfg, int n_streams,
                                          skps_mpipe** out) {
    SKPS_CHECK(det && kps && cfg && out && n_streams > 0 && n_streams <= 256, "mpipe_create: bad arguments");
    SKPS_CHECK(cfg->top_k > 0 && cfg->top_k <= 64, "mpipe_create: top_k %d outside 1..64", cfg->top_k);
    int device = 0;
    if (engine_pair_device(det, kps, "mpipe_create", &device)) return 1;
    SKPS_ON_DEVICE(device);
    skps_mpipe* p = new skps_mpipe();
    p->det = det; p->kps = kps; p->cfg = *cfg; p->S = n_streams; p->K = cfg->top_k;
    int c = 0, kh = 0, kw = 0;
    skps_engine_input_dims(det, &p->det_h, &p->det_w, &c);
    skps_engine_input_dims(kps, &kh, &kw, &c);
    p->kps_hw = kh;
    p->det_rows = skps_engine_output_elems(det, 0) / 16;
    p->P = skps_engine_output_elems(kps, 1);
    p->device = device;
    auto fail = [&](const char* what) {
        prefix_error("mpipe_create", what);
        skps_mpipe_destroy(p);
        return 1;
    };
    if (kh != kw || skps_engine_num_outputs(det) != 1 || skps_engine_num_outputs(kps) != 2) {
        set_error("engines are not a (detector, landmark) pair");
        return fail("engines");
    }
    const int S = p->S, K = p->K, P = p->P;
    p->frame_bytes = ((size_t)cfg->max_h * cfg->max_w * 3 + 255) & ~(size_t)255;
    p->ring_pos.assign(S, 0); p->prev_h.assign(S, 0); p->prev_w.assign(S, 0); p->frame_idx.assign(S, 0);
    p->d_frame.assign((size_t)S * 3, nullptr);
    for (auto& f : p->d_frame) SKPS_DEV_ALLOC(f, p->frame_bytes);
    for (auto& sl : p->slot) {
        SKPS_HOST_ALLOC(sl.h_stage, p->frame_bytes * S);
        SKPS_HOST_ALLOC(sl.h_hw, sizeof(int32_t) * 2 * S); SKPS_HOST_ALLOC(sl.h_have_prev, sizeof(int32_t) * S);
        SKPS_HOST_ALLOC(sl.h_geom, sizeof(int32_t) * 8 * S);
        SKPS_HOST_ALLOC(sl.h_desc, sizeof(MpStreamDesc) * 2 * S); SKPS_HOST_ALLOC(sl.h_det_slot, sizeof(int32_t) * S);
        SKPS_HOST_ALLOC(sl.h_stream, sizeof(int32_t) * S); SKPS_HOST_ALLOC(sl.h_turns, sizeof(int32_t) * S);
        SKPS_HOST_ALLOC(sl.h_count, sizeof(int32_t) * S); SKPS_HOST_ALLOC(sl.h_flag, sizeof(int32_t) * S);
        SKPS_HOST_ALLOC(sl.h_box, sizeof(double) * 4 * K * S); SKPS_HOST_ALLOC(sl.h_kps, sizeof(double) * 2 * P * K * S);
        SKPS_HOST_ALLOC(sl.h_scores, sizeof(float) * P * K * S);
        SKPS_HOST_ALLOC(sl.h_ids, sizeof(int64_t) * K * S);
        if (cudaEventCreateWithFlags(&sl.ev_in, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&sl.ev_done, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&sl.ev_staged, cudaEventDisableTiming) != cudaSuccess) { set_error("cudaEventCreate"); return fail("event"); }
    }
    if (cudaEventCreateWithFlags(&p->ev_ready, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&p->ev_read, cudaEventDisableTiming) != cudaSuccess) { set_error("cudaEventCreate"); return fail("event"); }
    SKPS_DEV_ALLOC(p->d_desc, sizeof(MpStreamDesc) * 2 * S); SKPS_DEV_ALLOC(p->d_det_slot, 4 * S); SKPS_DEV_ALLOC(p->d_turns, 4 * S); SKPS_DEV_ALLOC(p->d_hw, 8 * S); SKPS_DEV_ALLOC(p->d_have_prev, 4 * S);
    SKPS_DEV_ALLOC(p->d_flag, 4 * S); SKPS_DEV_ALLOC(p->d_det_count, 4 * S);
    SKPS_DEV_ALLOC(p->d_det_idx, 4 * (size_t)p->det_rows * S); SKPS_DEV_ALLOC(p->d_count, 4 * S);
    SKPS_DEV_ALLOC(p->d_detail, 4 * 5 * (size_t)K * S);
    SKPS_DEV_ALLOC(p->d_diff, 8 * S); SKPS_DEV_ALLOC(p->d_det_rows, 4 * 16 * (size_t)p->det_rows * S);
    SKPS_DEV_ALLOC(p->d_nms_ws, nms_workspace_bytes(p->det_rows, S)); SKPS_DEV_ALLOC(p->d_boxes, 4 * 4 * (size_t)K * S);
    SKPS_DEV_ALLOC(p->d_kps_now, 4 * 2 * (size_t)P * K * S);
    SKPS_DEV_ALLOC(p->d_prev_lm, 8 * 2 * 2 * (size_t)P * K * S); SKPS_DEV_ALLOC(p->d_prev_dx, 8 * 2 * 2 * (size_t)P * K * S);
    SKPS_DEV_ALLOC(p->d_track, 8 * 4 * (size_t)K * S); SKPS_DEV_ALLOC(p->d_out_kps, 8 * 2 * (size_t)P * K * S);
    SKPS_DEV_ALLOC(p->d_track_f32, 4 * 4 * (size_t)K * S);
    SKPS_DEV_ALLOC(p->d_n_prev, 4 * S); SKPS_DEV_ALLOC(p->d_prev_f32, 4 * S); SKPS_DEV_ALLOC(p->d_state_idx, 4 * S);
    SKPS_DEV_ALLOC(p->d_n_track, 4 * S);
    SKPS_DEV_ALLOC(p->d_src, 4 * (size_t)K * S); SKPS_DEV_ALLOC(p->d_ids, 8 * (size_t)K * S); SKPS_DEV_ALLOC(p->d_next_id, 8 * S);
    SKPS_DEV_ALLOC(p->d_mem_ids, 8 * (size_t)K * S); SKPS_DEV_ALLOC(p->d_mem_box, 4 * 4 * (size_t)K * S);
    SKPS_DEV_ALLOC(p->d_mem_gap, 4 * (size_t)K * S); SKPS_DEV_ALLOC(p->d_mem_n, 4 * S);
    SKPS_DEV_ALLOC(p->d_stream, 4 * S); SKPS_DEV_ALLOC(p->d_out_box, 8 * 4 * (size_t)K * S);
    SKPS_DEV_ALLOC(p->d_out_ids, 8 * (size_t)K * S);
    cudaMemset(p->d_prev_lm, 0, 8 * 2 * 2 * (size_t)P * K * S); cudaMemset(p->d_prev_dx, 0, 8 * 2 * 2 * (size_t)P * K * S);
    cudaMemset(p->d_state_idx, 0, 4 * S); cudaMemset(p->d_track_f32, 0, 4 * 4 * (size_t)K * S);
    cudaMemset(p->d_track, 0, 8 * 4 * (size_t)K * S);
    if (cudaStreamCreateWithFlags(&p->s_copy, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&p->s_compute, cudaStreamNonBlocking) != cudaSuccess) { set_error("cudaStreamCreate"); return fail("stream"); }
    if (skps_mpipe_reset(p, -1)) return fail("reset");
    *out = p;
    return 0;
}

// The call -> stream map of a submit: streams [host] null, or n distinct ids in 0..S-1.  Returns 1 with skps_last_error set
// for anything else, before the submit enqueues anything; *identity = the map is null or streams[i] == i for every i.
static int check_stream_map(const skps_mpipe* p, const int32_t* streams, int n, bool* identity) {
    *identity = true;
    if (!streams) return 0;
    std::vector<char> seen(p->S, 0);
    for (int i = 0; i < n; ++i) {
        const int t = streams[i];
        SKPS_CHECK(t >= 0 && t < p->S, "mpipe_submit: frame %d is for stream %d, outside 0..%d", i, t, p->S - 1);
        SKPS_CHECK(!seen[t], "mpipe_submit: frame %d is for stream %d, which an earlier frame of the call already feeds", i, t);
        seen[t] = 1;
        if (t != i) *identity = false;
    }
    return 0;
}

// One batch.  Frame i is the next frame of stream streams[i] (streams null: stream i); the streams are distinct, and a
// stream the batch does not feed keeps its state as it is.  Everything per frame of the batch (descriptors, staging,
// detector frames, results) is in call order; everything per stream (ring, previous frame size, frame count, the device
// state of temporal.cu) is indexed by the stream.  Host frames (pitches null) are uploaded on the copy stream into the
// stream's next ring position; device frames (rows pitches[i] bytes apart) are gathered there by the frame-difference launch
// on the compute stream, after the work queued on `producer`, whose later work waits for that launch; they are in pixel
// layout `layout` (planes plane_pitches[i] bytes apart for the planar layouts) and land in the ring as BGR.  A device frame
// stored turned turns[i] quarter turns clockwise (turns null: none) lands there upright, and from then on the batch sees
// the upright frame: hw[i] is the stored size.  out: results into caller buffers on the device instead of the slot's
// pinned ones.
static int submit_batch(skps_mpipe* p, int slot_i, const int32_t* streams, const uint8_t* const* frames, const int32_t* hw,
                        int n, const int32_t* pitches, cudaStream_t producer, const skps_mpipe_outputs* out,
                        int layout = SKPS_LAYOUT_BGR, const int32_t* plane_pitches = nullptr,
                        const int32_t* turns = nullptr) {
    const bool on_device = pitches != nullptr;
    SKPS_CHECK(p && frames && hw && (slot_i == 0 || slot_i == 1) && n > 0 && n <= p->S, "mpipe_submit: bad arguments");
    bool identity = true;
    if (check_stream_map(p, streams, n, &identity)) return 1;
    if (identity) streams = nullptr;      // the launches of a submit without a map, byte for byte
    skps_mpipe::Slot& sl = p->slot[slot_i];
    SKPS_CHECK(!sl.busy, "mpipe_submit: slot %d still holds results (call skps_mpipe_wait first)", slot_i);
    SKPS_CHECK(!out || (out->n_faces && out->ran_detector && out->boxes && out->kps && out->scores),
               "mpipe_submit: device outputs need n_faces, ran_detector, boxes, kps and scores");
    SKPS_CHECK(!out || !p->align_size || (out->chips && out->M), "mpipe_submit: alignment is on; device outputs need chips and M");
    SKPS_CHECK(!out || !p->pose_on || (out->rvec && out->tvec && out->euler && out->reproject),
               "mpipe_submit: pose is on; device outputs need rvec, tvec, euler and reproject");
    SKPS_ON_DEVICE(p->device);
    const skps_pipeline_cfg& c = p->cfg;
    const int S = p->S, K = p->K, P = p->P;
    cudaStream_t sc = p->s_copy, sx = p->s_compute;
    // a slot completed by skps_mpipe_wait_stream was not waited for on the host: its last batch may still be reading the
    // pinned per-batch buffers rewritten below
    SKPS_CUDA(cudaEventSynchronize(sl.ev_staged));
    // and it may still read ring positions that later host frames are uploaded into (see the ring discipline below): order
    // the copy stream after it whether or not this batch uploads, so that every batch but the other slot's latest is
    // behind the copy stream, or waited for on the host, whenever a batch uploads
    if (sl.device_out) SKPS_CUDA(cudaStreamWaitEvent(sc, sl.ev_done, 0));
    // ---- uploads on the copy stream: frame i of stream t = streams[i] into t's next ring position
    bool turned = false;
    for (int i = 0; i < n; ++i) {
        const int t = streams ? streams[i] : i;
        int H = hw[2 * i], W = hw[2 * i + 1];
        SKPS_CHECK(frames[i] && H > 0 && W > 0 && (size_t)H * W * 3 <= p->frame_bytes,
                   "mpipe_submit: frame %d is %dx%d, larger than the pipeline maximum %dx%d", i, H, W, c.max_h, c.max_w);
        if (on_device) {
            SKPS_CHECK(H == 1 || pitches[i] >= layout_xstep(layout) * W,
                       "mpipe_submit: frame %d has row pitch %d, less than %d x width %d", i, pitches[i], layout_xstep(layout), W);
            SKPS_CHECK(layout < SKPS_LAYOUT_BGR_PLANAR || plane_pitches[i] >= 0, "mpipe_submit: frame %d has plane pitch %d",
                       i, plane_pitches[i]);
            const int q = turns ? turns[i] : 0;
            SKPS_CHECK(q >= 0 && q <= 3, "mpipe_submit: frame %d has turns %d, outside 0..3", i, q);
            sl.h_turns[i] = q;
            turned |= q != 0;
            if (q & 1) { H = hw[2 * i + 1]; W = hw[2 * i]; }       // the upright frame
        } else if (upload_host_frame(frames[i], (size_t)H * W * 3, sl.h_stage + p->frame_bytes * i,
                                     p->d_frame[(size_t)t * 3 + (p->ring_pos[t] + 1) % 3], sc)) {
            return 1;
        }
        sl.h_hw[2 * i] = H; sl.h_hw[2 * i + 1] = W;
        sl.h_have_prev[i] = (p->prev_h[t] == H && p->prev_w[t] == W) ? 1 : 0;
        sl.h_stream[i] = t;
    }
    if (on_device) {
        SKPS_CUDA(cudaEventRecord(p->ev_ready, producer));
        SKPS_CUDA(cudaStreamWaitEvent(sx, p->ev_ready, 0));
    } else {
        SKPS_CUDA(cudaEventRecord(sl.ev_in, sc));
        SKPS_CUDA(cudaStreamWaitEvent(sx, sl.ev_in, 0));
    }
    // ---- compute
    SKPS_CUDA(cudaMemcpyAsync(p->d_hw, sl.h_hw, 8 * n, cudaMemcpyHostToDevice, sx));
    SKPS_CUDA(cudaMemcpyAsync(p->d_have_prev, sl.h_have_prev, 4 * n, cudaMemcpyHostToDevice, sx));
    SKPS_CUDA(cudaMemsetAsync(p->d_diff, 0, 8 * n, sx));
    uint8_t* det_in = (uint8_t*)skps_engine_input_ptr(p->det);
    const size_t det_in_bytes = (size_t)p->det_h * p->det_w * 3;
    // per-stream frame pointers + letterbox geometry: one small upload, then every pre/post-processing step is ONE launch for
    // all streams (it was 5 launches per stream and call - ~80 launch gaps of a 5 ms call at 16 streams).
    // Keyframes (skps_mpipe_set_detect_every): stream t's frame j is one when the stream has no previous frame of this size
    // or (j + t % N) % N == 0, wherever the frame sits in the call.  Only keyframes go through the letterbox, the detector and
    // NMS, as detector frames 0..m-1 in call order; the host knows them now, so the detector batch shrinks with no read-back.
    const int N = p->detect_every;
    int m = 0;
    size_t max_bytes = 0;
    for (int i = 0; i < n; ++i) {
        const int t = sl.h_stream[i];
        const int H = sl.h_hw[2 * i], W = sl.h_hw[2 * i + 1];
        const bool key = !sl.h_have_prev[i] || (p->frame_idx[t] + t % N) % N == 0;
        sl.h_det_slot[i] = key ? m++ : -1;
        MpStreamDesc& D = sl.h_desc[i];
        D.cur = p->d_frame[(size_t)t * 3 + (p->ring_pos[t] + 1) % 3];
        // the difference sum only decides keyframes: the other frames skip it (a device frame is still gathered into cur)
        D.have_prev = sl.h_have_prev[i] && key;
        D.prev = D.have_prev ? p->d_frame[(size_t)t * 3 + p->ring_pos[t]] : nullptr;
        D.H = H; D.W = W;
        D.src = on_device ? frames[i] : nullptr;
        D.src_pitch = on_device ? pitches[i] : W * 3;
        D.src_plane = on_device && layout >= SKPS_LAYOUT_BGR_PLANAR ? plane_pitches[i] : 0;
        letterbox_geometry(H, W, p->det_h, p->det_w, &D.scale, &D.rw, &D.rh, &D.top, &D.left);
        memcpy(&sl.h_geom[8 * i], &D.scale, 4); sl.h_geom[8 * i + 1] = D.top; sl.h_geom[8 * i + 2] = D.left;
        if ((size_t)H * W * 3 > max_bytes) max_bytes = (size_t)H * W * 3;
    }
    // the keyframes' descriptors, packed after the batch's; when every frame is a keyframe the batch is that list, and the
    // kernels take det_slot = null (detector frame i is frame i), exactly as without a cadence
    const MpStreamDesc* d_key_desc = p->d_desc;
    const int32_t* det_slot = nullptr;
    int n_desc = n;
    if (m < n) {
        for (int i = 0; i < n; ++i)
            if (sl.h_det_slot[i] >= 0) sl.h_desc[n + sl.h_det_slot[i]] = sl.h_desc[i];
        d_key_desc = p->d_desc + n; n_desc = n + m;
        det_slot = p->d_det_slot;
        SKPS_CUDA(cudaMemcpyAsync(p->d_det_slot, sl.h_det_slot, 4 * n, cudaMemcpyHostToDevice, sx));
    }
    // the call -> stream map of the two kernels that touch per-stream device state (select, temporal); null: the identity
    const int32_t* stream_map = nullptr;
    if (streams) {
        stream_map = p->d_stream;
        SKPS_CUDA(cudaMemcpyAsync(p->d_stream, sl.h_stream, 4 * n, cudaMemcpyHostToDevice, sx));
    }
    // the turns of a batch holding a turned frame: its ingest is the turned kernel, any other the unturned one
    if (turned) SKPS_CUDA(cudaMemcpyAsync(p->d_turns, sl.h_turns, 4 * n, cudaMemcpyHostToDevice, sx));
    SKPS_CUDA(cudaMemcpyAsync(p->d_desc, sl.h_desc, sizeof(MpStreamDesc) * n_desc, cudaMemcpyHostToDevice, sx));
    SKPS_CUDA(cudaEventRecord(sl.ev_staged, sx));
    if (launch_frame_diff(p->d_desc, n, MpStreamDesc{}, max_bytes, p->d_diff, sx, on_device ? layout : SKPS_LAYOUT_BGR,
                          turned ? p->d_turns : nullptr))
        return 1;
    if (on_device) {
        SKPS_CUDA(cudaEventRecord(p->ev_read, sx));
        SKPS_CUDA(cudaStreamWaitEvent(producer, p->ev_read, 0));
    }
    // results: D2H into the slot's pinned buffers, or D2D into the caller's; either way before the next batch on sx can
    // overwrite d_out_kps, the engine's score output or the chips
    const cudaMemcpyKind result_kind = out ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    LetterboxArgs la = {};
    la.desc = d_key_desc; la.out = det_in; la.out_stride = det_in_bytes; la.in_h = p->det_h; la.in_w = p->det_w;
    if (m > 0 && launch_letterbox(la, m, sx)) return 1;
    if (launch_mp_decide(p->d_diff, p->d_hw, p->d_have_prev, det_slot, p->d_flag, n, sx)) return 1;
    // the detector runs for every keyframe of the batch (one launch sequence, batch m); the gate only chooses whose rows are
    // used.  With no keyframe the detector and NMS are skipped and every stream takes the tracker path.
    if (m > 0) {
        if (skps_engine_forward(p->det, det_in, m, nullptr, sx)) return 1;
        const float* det_out = skps_engine_output_ptr(p->det, 0);
        NmsArgs na = {};
        na.raw = det_out; na.rows = p->det_rows; na.batch = m; na.score_thres = c.score_thres; na.iou_thres = c.iou_thres;
        na.desc = d_key_desc; na.limit = p->det_rows; na.capacity = p->det_rows;
        na.kept_rows = p->d_det_rows; na.kept_idx = p->d_det_idx; na.count = p->d_det_count;
        na.ws = p->d_nms_ws; na.ws_cap = p->det_rows;
        if (launch_nms(na, sx)) return 1;
    }
    SelectArgs sa = {};
    sa.det_rows = p->d_det_rows; sa.det_count = p->d_det_count; sa.det_stride = 16; sa.det_cap = p->det_rows;
    sa.det_slot = det_slot; sa.flag = p->d_flag; sa.track = p->d_track_f32; sa.n_track = p->d_n_track; sa.stream = stream_map;
    sa.iou_thres = c.track_iou; sa.alpha = c.alpha; sa.one_minus_alpha = (float)(1.0 - (double)c.alpha);
    sa.min_face = c.min_face; sa.top_k = K;
    sa.boxes4 = p->d_boxes; sa.count = p->d_count; sa.src = p->d_src;
    if (launch_select(sa, n, sx)) return 1;
    uint8_t* kps_in = (uint8_t*)skps_engine_input_ptr(p->kps);
    CropArgs ca = {};
    ca.desc = p->d_desc; ca.boxes = p->d_boxes; ca.count = p->d_count; ca.K = K;
    ca.face_scale = c.face_scale; ca.min_face = c.kps_min_face; ca.crops = kps_in; ca.S = p->kps_hw; ca.detail = p->d_detail;
    if (launch_crop(ca, n, sx)) return 1;
    if (skps_engine_forward(p->kps, kps_in, n * K, nullptr, sx)) return 1;
    if (launch_landmark_post(skps_engine_output_ptr(p->kps, 0), p->d_detail, p->d_count, K, P, p->d_kps_now, n, sx)) return 1;
    MpTemporalArgs a;
    a.top_k = K; a.n_points = P; a.stream = stream_map;
    a.kps_now = p->d_kps_now; a.count = p->d_count; a.flag = p->d_flag; a.hw = p->d_hw; a.boxes4 = p->d_boxes;
    a.prev_lm = p->d_prev_lm; a.prev_dx = p->d_prev_dx; a.n_prev = p->d_n_prev; a.prev_f32 = p->d_prev_f32;
    a.state_idx = p->d_state_idx; a.track_box = p->d_track; a.track_f32 = p->d_track_f32; a.n_track = p->d_n_track;
    a.src = p->d_src; a.ids = p->d_ids; a.next_id = p->d_next_id;
    a.id_memory = p->id_memory;
    a.mem_ids = p->d_mem_ids; a.mem_box = p->d_mem_box; a.mem_gap = p->d_mem_gap; a.mem_n = p->d_mem_n;
    a.out_kps = p->d_out_kps;
    // with a map, the stream state's rows 0..n-1 are not the batch's: the kernel packs the returned boxes and ids by frame
    a.out_box = streams ? p->d_out_box : nullptr;
    a.out_ids = streams ? p->d_out_ids : nullptr;
    mp_temporal_constants(c, a);
    if (launch_mp_temporal(a, n, sx)) return 1;
    sl.align = p->align_size;
    if (sl.align) {
        // chips from the smoothed landmarks, on the frames still in the ring
        const size_t chip_bytes = (size_t)sl.align * sl.align * 3;
        if (launch_mp_align(p->d_desc, p->d_out_kps, p->d_count, K, P, sl.align, p->d_chips, p->d_align_M, n, sx)) return 1;
        SKPS_CUDA(cudaMemcpyAsync(out ? out->chips : sl.h_chips, p->d_chips, chip_bytes * K * n, result_kind, sx));
        SKPS_CUDA(cudaMemcpyAsync(out ? out->M : sl.h_M, p->d_align_M, 8 * 6 * (size_t)K * n, result_kind, sx));
    }
    sl.pose = p->pose_on;
    if (sl.pose) {
        // head pose from the smoothed landmarks, camera per stream from this call's frame size
        PoseArgs pa = {};
        pose_model_98(pa);
        pa.pts64 = p->d_out_kps; pa.G = n; pa.K = K; pa.P = P;
        pa.count = p->d_count; pa.hw = p->d_hw;
        const size_t faces = (size_t)n * K;
        pa.rvec = p->d_pose; pa.tvec = p->d_pose + 3 * faces; pa.euler = p->d_pose + 6 * faces; pa.reproj = p->d_pose + 9 * faces;
        if (launch_head_pose(pa, sx)) return 1;
        if (out) {
            SKPS_CUDA(cudaMemcpyAsync(out->rvec, pa.rvec, 8 * 3 * faces, result_kind, sx));
            SKPS_CUDA(cudaMemcpyAsync(out->tvec, pa.tvec, 8 * 3 * faces, result_kind, sx));
            SKPS_CUDA(cudaMemcpyAsync(out->euler, pa.euler, 8 * 3 * faces, result_kind, sx));
            SKPS_CUDA(cudaMemcpyAsync(out->reproject, pa.reproj, 8 * 16 * faces, result_kind, sx));
        } else {
            SKPS_CUDA(cudaMemcpyAsync(sl.h_pose, p->d_pose, 8 * 25 * faces, result_kind, sx));
        }
    }
    SKPS_CUDA(cudaMemcpyAsync(out ? out->n_faces : sl.h_count, p->d_count, 4 * n, result_kind, sx));
    SKPS_CUDA(cudaMemcpyAsync(out ? out->ran_detector : sl.h_flag, p->d_flag, 4 * n, result_kind, sx));
    SKPS_CUDA(cudaMemcpyAsync(out ? out->boxes : sl.h_box, streams ? p->d_out_box : p->d_track, 8 * 4 * (size_t)K * n,
                              result_kind, sx));
    SKPS_CUDA(cudaMemcpyAsync(out ? out->kps : sl.h_kps, p->d_out_kps, 8 * 2 * (size_t)P * K * n, result_kind, sx));
    SKPS_CUDA(cudaMemcpyAsync(out ? out->scores : sl.h_scores, skps_engine_output_ptr(p->kps, 1), 4 * (size_t)P * K * n,
                              result_kind, sx));
    if (!out || out->ids)
        SKPS_CUDA(cudaMemcpyAsync(out ? out->ids : sl.h_ids, streams ? p->d_out_ids : p->d_ids, 8 * (size_t)K * n, result_kind,
                                  sx));
    SKPS_CUDA(cudaEventRecord(sl.ev_done, sx));
    // ring discipline, per stream t of the batch: this batch reads t's positions r (previous) and r+1 (current); the next
    // batch that feeds t uploads into r+2 (free), and the one after that into r again.  That third batch B comes at least
    // two submits after this one A, whichever slots and calls the stream's frames land in: at least one other submit, the
    // one feeding t in between, separates them.  Every batch computes on the one serial compute stream, so any batch that
    // is done implies all batches before it are done.  When B is submitted on slot j, its slot's previous batch q has been
    // completed: waited for on the host (skps_mpipe_wait), or, if completed by skps_mpipe_wait_stream, the copy stream was
    // made to wait for q's ev_done at the top of B's submit.  Every earlier submit did the same for its own slot's previous
    // batch, so every batch except the latest one on the other slot, o, is done or behind the copy stream.  A is not o: if
    // o is the most recent submit, A, two or more submits back, comes before it, and if q is more recent than o, q done
    // implies o done.  So B's upload into r cannot overtake A's reads.  Device frames are gathered on the compute stream
    // itself, after A.
    for (int i = 0; i < n; ++i) {
        const int t = sl.h_stream[i];
        p->ring_pos[t] = (p->ring_pos[t] + 1) % 3;
        p->prev_h[t] = sl.h_hw[2 * i]; p->prev_w[t] = sl.h_hw[2 * i + 1];
        ++p->frame_idx[t];
    }
    sl.n = n;
    sl.m = m;
    sl.busy = true;
    sl.device_out = out != nullptr;
    return 0;
}

extern "C" SKPS_API int skps_mpipe_submit_streams(skps_mpipe* p, int slot_i, const int32_t* streams, const uint8_t* const* frames,
                                                  const int32_t* hw, int n) {
    return submit_batch(p, slot_i, streams, frames, hw, n, nullptr, nullptr, nullptr);
}

extern "C" SKPS_API int skps_mpipe_submit(skps_mpipe* p, int slot_i, const uint8_t* const* frames, const int32_t* hw, int n) {
    return skps_mpipe_submit_streams(p, slot_i, nullptr, frames, hw, n);
}

extern "C" SKPS_API int skps_mpipe_submit_device_rotate(skps_mpipe* p, int slot_i, const int32_t* streams,
                                                        const uint8_t* const* frames, const int32_t* pitches, const int32_t* hw,
                                                        int n, int layout, const int32_t* plane_pitches, const int32_t* turns,
                                                        const skps_mpipe_outputs* out, void* producer_stream) {
    SKPS_CHECK(p && frames && pitches && hw && n > 0 && n <= p->S, "mpipe_submit_device: bad arguments");
    SKPS_CHECK(layout_ok(layout), "mpipe_submit_device: unknown pixel layout %d", layout);
    SKPS_CHECK(layout < SKPS_LAYOUT_BGR_PLANAR || plane_pitches, "mpipe_submit_device: a planar layout needs plane pitches");
    for (int i = 0; turns && i < n; ++i)
        SKPS_CHECK(turns[i] >= 0 && turns[i] <= 3, "mpipe_submit_device: frame %d has turns %d, outside 0..3", i, turns[i]);
    bool identity = true;
    if (check_stream_map(p, streams, n, &identity)) return 1;
    SKPS_ON_DEVICE(p->device);
    for (int i = 0; i < n; ++i)
        if (check_device_frame(frames[i], p->device, "mpipe_submit_device", i)) return 1;
    return submit_batch(p, slot_i, streams, frames, hw, n, pitches, (cudaStream_t)producer_stream, out, layout, plane_pitches,
                        turns);
}

extern "C" SKPS_API int skps_mpipe_submit_device_layout(skps_mpipe* p, int slot_i, const int32_t* streams,
                                                        const uint8_t* const* frames, const int32_t* pitches, const int32_t* hw,
                                                        int n, int layout, const int32_t* plane_pitches,
                                                        const skps_mpipe_outputs* out, void* producer_stream) {
    return skps_mpipe_submit_device_rotate(p, slot_i, streams, frames, pitches, hw, n, layout, plane_pitches, nullptr, out,
                                           producer_stream);
}

extern "C" SKPS_API int skps_mpipe_submit_device_streams(skps_mpipe* p, int slot_i, const int32_t* streams,
                                                         const uint8_t* const* frames, const int32_t* pitches, const int32_t* hw,
                                                         int n, const skps_mpipe_outputs* out, void* producer_stream) {
    return skps_mpipe_submit_device_layout(p, slot_i, streams, frames, pitches, hw, n, SKPS_LAYOUT_BGR, nullptr, out,
                                           producer_stream);
}

extern "C" SKPS_API int skps_mpipe_submit_device(skps_mpipe* p, int slot_i, const uint8_t* const* frames, const int32_t* pitches,
                                                 const int32_t* hw, int n, const skps_mpipe_outputs* out, void* producer_stream) {
    return skps_mpipe_submit_device_streams(p, slot_i, nullptr, frames, pitches, hw, n, out, producer_stream);
}

extern "C" SKPS_API int skps_mpipe_wait_stream(skps_mpipe* p, int slot_i, void* consumer_stream) {
    SKPS_CHECK(p && (slot_i == 0 || slot_i == 1), "mpipe_wait_stream: bad arguments");
    skps_mpipe::Slot& sl = p->slot[slot_i];
    SKPS_CHECK(sl.busy, "mpipe_wait_stream: nothing submitted on slot %d", slot_i);
    SKPS_CHECK(sl.device_out, "mpipe_wait_stream: slot %d has host results (call skps_mpipe_wait)", slot_i);
    SKPS_ON_DEVICE(p->device);
    SKPS_CUDA(cudaStreamWaitEvent((cudaStream_t)consumer_stream, sl.ev_done, 0));
    sl.busy = false;
    return 0;
}

extern "C" SKPS_API int skps_mpipe_wait(skps_mpipe* p, int slot_i, int32_t* n_faces, double* boxes, double* kps, float* scores,
                                        int32_t* ran_detector) {
    SKPS_CHECK(p && (slot_i == 0 || slot_i == 1) && n_faces && boxes && kps && scores, "mpipe_wait: bad arguments");
    skps_mpipe::Slot& sl = p->slot[slot_i];
    SKPS_CHECK(sl.busy, "mpipe_wait: nothing submitted on slot %d", slot_i);
    SKPS_CHECK(!sl.device_out, "mpipe_wait: slot %d has device results (call skps_mpipe_wait_stream)", slot_i);
    SKPS_ON_DEVICE(p->device);
    SKPS_CUDA(cudaEventSynchronize(sl.ev_done));
    sl.busy = false;
    const int K = p->K, P = p->P, n = sl.n;
    for (int s = 0; s < n; ++s) {
        n_faces[s] = sl.h_count[s];
        if (ran_detector) ran_detector[s] = sl.h_flag[s];
    }
    memcpy(boxes, sl.h_box, sizeof(double) * 4 * K * n);
    memcpy(kps, sl.h_kps, sizeof(double) * 2 * P * K * n);
    memcpy(scores, sl.h_scores, sizeof(float) * P * K * n);
    return 0;
}

static void free_align(skps_mpipe* p) {
    if (p->d_chips) cudaFree(p->d_chips);
    if (p->d_align_M) cudaFree(p->d_align_M);
    p->d_chips = nullptr; p->d_align_M = nullptr;
    for (auto& sl : p->slot) {
        if (sl.h_chips) cudaFreeHost(sl.h_chips);
        if (sl.h_M) cudaFreeHost(sl.h_M);
        sl.h_chips = nullptr; sl.h_M = nullptr; sl.align = 0;
    }
    p->align_size = 0;
}

extern "C" SKPS_API int skps_mpipe_set_align(skps_mpipe* p, int size) {
    SKPS_CHECK(p && (size == 0 || (size >= 16 && size <= 512)), "mpipe_set_align: size %d is neither 0 nor in 16..512", size);
    SKPS_CHECK(!p->slot[0].busy && !p->slot[1].busy, "mpipe_set_align: a batch is in flight (call skps_mpipe_wait first)");
    SKPS_ON_DEVICE(p->device);
    SKPS_CUDA(cudaStreamSynchronize(p->s_compute));
    if (size == p->align_size) return 0;
    free_align(p);
    if (size == 0) return 0;
    const size_t faces = (size_t)p->S * p->K, chip_bytes = (size_t)size * size * 3;
    bool ok = cudaMalloc((void**)&p->d_chips, chip_bytes * faces) == cudaSuccess &&
              cudaMalloc((void**)&p->d_align_M, 8 * 6 * faces) == cudaSuccess;
    for (auto& sl : p->slot)
        ok = ok && cudaMallocHost((void**)&sl.h_chips, chip_bytes * faces) == cudaSuccess &&
             cudaMallocHost((void**)&sl.h_M, 8 * 6 * faces) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        free_align(p);
        SKPS_CHECK(false, "mpipe_set_align: cannot allocate %zu chip bytes per buffer (%zu faces of %dx%d)", chip_bytes * faces,
                   faces, size, size);
    }
    p->align_size = size;
    return 0;
}

extern "C" SKPS_API int skps_mpipe_align_results(skps_mpipe* p, int slot_i, uint8_t* chips, double* M) {
    SKPS_CHECK(p && (slot_i == 0 || slot_i == 1) && chips && M, "mpipe_align_results: bad arguments");
    const skps_mpipe::Slot& sl = p->slot[slot_i];
    SKPS_CHECK(!sl.busy, "mpipe_align_results: slot %d is in flight (call skps_mpipe_wait first)", slot_i);
    SKPS_CHECK(sl.align > 0 && sl.n > 0 && !sl.device_out, "mpipe_align_results: slot %d was not submitted with alignment on "
               "and host results", slot_i);
    const size_t faces = (size_t)sl.n * p->K;
    memcpy(chips, sl.h_chips, faces * sl.align * sl.align * 3);
    memcpy(M, sl.h_M, faces * 6 * sizeof(double));
    return 0;
}

static void free_pose(skps_mpipe* p) {
    if (p->d_pose) cudaFree(p->d_pose);
    p->d_pose = nullptr;
    for (auto& sl : p->slot) {
        if (sl.h_pose) cudaFreeHost(sl.h_pose);
        sl.h_pose = nullptr; sl.pose = false;
    }
    p->pose_on = false;
}

extern "C" SKPS_API int skps_mpipe_set_pose(skps_mpipe* p, int on) {
    SKPS_CHECK(p, "mpipe_set_pose: null");
    SKPS_CHECK(!p->slot[0].busy && !p->slot[1].busy, "mpipe_set_pose: a batch is in flight (call skps_mpipe_wait first)");
    SKPS_ON_DEVICE(p->device);
    SKPS_CUDA(cudaStreamSynchronize(p->s_compute));
    if ((on != 0) == p->pose_on) return 0;
    free_pose(p);
    if (!on) return 0;
    SKPS_CHECK(p->P >= 98, "mpipe_set_pose: %d landmarks per face, expected 98", p->P);
    const size_t bytes = 8 * 25 * (size_t)p->S * p->K;
    bool ok = cudaMalloc((void**)&p->d_pose, bytes) == cudaSuccess;
    for (auto& sl : p->slot) ok = ok && cudaMallocHost((void**)&sl.h_pose, bytes) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        free_pose(p);
        SKPS_CHECK(false, "mpipe_set_pose: cannot allocate %zu bytes per buffer", bytes);
    }
    p->pose_on = true;
    return 0;
}

extern "C" SKPS_API int skps_mpipe_pose_results(skps_mpipe* p, int slot_i, double* rvec, double* tvec, double* euler,
                                                double* reproject) {
    SKPS_CHECK(p && (slot_i == 0 || slot_i == 1) && rvec && tvec && euler && reproject, "mpipe_pose_results: bad arguments");
    const skps_mpipe::Slot& sl = p->slot[slot_i];
    SKPS_CHECK(!sl.busy, "mpipe_pose_results: slot %d is in flight (call skps_mpipe_wait first)", slot_i);
    SKPS_CHECK(sl.pose && sl.n > 0 && !sl.device_out, "mpipe_pose_results: slot %d was not submitted with pose on and host "
               "results", slot_i);
    const size_t faces = (size_t)sl.n * p->K;
    memcpy(rvec, sl.h_pose, faces * 3 * sizeof(double));
    memcpy(tvec, sl.h_pose + 3 * faces, faces * 3 * sizeof(double));
    memcpy(euler, sl.h_pose + 6 * faces, faces * 3 * sizeof(double));
    memcpy(reproject, sl.h_pose + 9 * faces, faces * 16 * sizeof(double));
    return 0;
}

extern "C" SKPS_API int skps_mpipe_track_ids(skps_mpipe* p, int slot_i, int64_t* ids) {
    SKPS_CHECK(p && (slot_i == 0 || slot_i == 1) && ids, "mpipe_track_ids: bad arguments");
    const skps_mpipe::Slot& sl = p->slot[slot_i];
    SKPS_CHECK(!sl.busy, "mpipe_track_ids: slot %d is in flight (call skps_mpipe_wait first)", slot_i);
    SKPS_CHECK(sl.n > 0 && !sl.device_out, "mpipe_track_ids: slot %d was not submitted with host results", slot_i);
    memcpy(ids, sl.h_ids, sizeof(int64_t) * sl.n * p->K);
    return 0;
}

extern "C" SKPS_API int skps_mpipe_set_detect_every(skps_mpipe* p, int every) {
    SKPS_CHECK(p && every >= 1, "mpipe_set_detect_every: every %d is not >= 1", every);
    p->detect_every = every;
    return 0;
}

extern "C" SKPS_API int skps_mpipe_set_id_memory(skps_mpipe* p, int frames) {
    SKPS_CHECK(p && frames >= 0, "mpipe_set_id_memory: frames %d is not >= 0", frames);
    SKPS_ON_DEVICE(p->device);
    // switched off, every stream forgets its lost tracks; submits already queued keep the value they were made with
    if (frames == 0 && p->id_memory > 0) SKPS_CUDA(cudaMemsetAsync(p->d_mem_n, 0, 4 * (size_t)p->S, p->s_compute));
    p->id_memory = frames;
    return 0;
}

extern "C" SKPS_API int skps_mpipe_detector_frames(const skps_mpipe* p, int slot_i, int* m) {
    SKPS_CHECK(p && (slot_i == 0 || slot_i == 1) && m, "mpipe_detector_frames: bad arguments");
    SKPS_CHECK(p->slot[slot_i].n > 0, "mpipe_detector_frames: nothing submitted on slot %d", slot_i);
    *m = p->slot[slot_i].m;
    return 0;
}

extern "C" SKPS_API int skps_mpipe_dims(const skps_mpipe* p, int* n_streams, int* top_k, int* n_points) {
    SKPS_CHECK(p, "mpipe_dims: null");
    if (n_streams) *n_streams = p->S;
    if (top_k) *top_k = p->K;
    if (n_points) *n_points = p->P;
    return 0;
}
