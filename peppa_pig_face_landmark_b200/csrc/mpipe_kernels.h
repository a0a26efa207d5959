// Kernels of the multi-stream pipeline (mpipe.cu): launchers defined in image_ops.cu / temporal.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct skps_pipeline_cfg;

namespace skps {

struct MpTemporalArgs {
    int top_k, n_points;
    const float* kps_now;        // [S][K][P][2] float32 landmarks in frame pixels (landmark_post)
    const int* count;            // [S] faces this frame
    const int* flag;             // [S] detector ran this frame
    const int* hw;               // [S][2] frame height, width
    const float* boxes4;         // [S][K][4] boxes the landmark stage used (boxes_return, facer.py:66)
    // state, updated in place
    double* prev_lm;             // [S][2][K][P][2] previous landmark sets (ping-pong)
    double* prev_dx;             // [S][2][K][P][2] previous - filtered
    int* n_prev;                 // [S] sets in prev_lm (-1 = None)
    int* prev_f32;               // [S] previous_landmarks_set is a float32 array (numpy dtype bookkeeping)
    int* state_idx;              // [S] which half of prev_lm/prev_dx is current
    double* track_box;           // [S][K][4] float64 track boxes (returned as 'box')
    float* track_f32;            // [S][K][4] the same, as float32 (next frame's judge_boxs / crop input)
    int* n_track;                // [S]
    const int* src;              // [S][K] source of each face this frame (launch_mp_select), an index into the old track
    int64_t* ids;                // [S][K] track id of each track box
    int64_t* next_id;            // [S] the next unused id of the stream
    // outputs
    double* out_kps;             // [S][K][P][2]
    // constants (python floats computed on the host exactly as lk.py does)
    double iou_thres, alpha, one_minus_alpha, a_d, one_minus_a_d, min_cutoff, beta, two_pi;
};
// Sets the constants of `a` from the pipeline's cfg (mpipe.cu): what skps_mpipe_submit and skps_debug_mp_temporal launch with.
void mp_temporal_constants(const skps_pipeline_cfg& c, MpTemporalArgs& a);

// One frame of one stream as the batched pre/post-processing kernels see it (filled on the host per call, one upload).
struct MpStreamDesc {
    uint8_t* cur;                // this call's frame (packed HxWx3 uint8 BGR, device, 16-byte aligned)
    const uint8_t* prev;         // the previous frame of the stream (packed, 16-byte aligned), or null
    int H, W, have_prev;
    float scale;                 // letterbox geometry (face_detector.py:49-62)
    int rw, rh, top, left;
    const uint8_t* src;          // the caller's device frame, gathered into cur by launch_mp_absdiff, or null (cur holds it)
    int src_pitch;               // bytes from one row of src to the next, >= 3 W, any alignment
};
// Batched over the streams of a call (grid z / x = stream): what S x {skps_frame_absdiff_sum, skps_letterbox,
// skps_crop_resize, skps_landmark_post} launches did, in four launches.  Same device code per element, bit for bit.
// launch_mp_absdiff also ingests: a stream with src set gets its frame gathered into cur and, with have_prev, |cur - prev|
// summed in the same pass (the same integer sum as from a packed cur).  d [dev] holds n descriptors; launch_frame_ingest
// runs the same kernel on one descriptor passed by value (diff = one counter, zeroed by the caller).
int launch_mp_absdiff(const MpStreamDesc* d, unsigned long long* diff, int n, size_t max_bytes, cudaStream_t s);
int launch_frame_ingest(const MpStreamDesc& one, unsigned long long* diff, cudaStream_t s);
// Frame staging on the host side, shared by skps_pipeline and skps_mpipe.  upload_host_frame queues the H2D copy of a [host]
// frame of `bytes` bytes into dst on s: a pinned frame is copied as it is, a pageable one first into `stage` (pinned, at
// least `bytes`) so that the copy stays asynchronous and at full PCIe rate.  check_device_frame fails unless `frame` is
// device or managed memory of `device`; the error names the caller `fn` and, for index >= 0, the frame's index.
int upload_host_frame(const uint8_t* frame, size_t bytes, uint8_t* stage, uint8_t* dst, cudaStream_t s);
int check_device_frame(const void* frame, int device, const char* fn, int index);
int launch_mp_letterbox(const MpStreamDesc* d, uint8_t* out, size_t out_stride, int in_h, int in_w, int n, cudaStream_t s);

// Detector post-processing (nms.cu): score filter, sort, greedy NMS and scale_coords of `batch` frames of `rows` raw rows each
// (raw [batch][rows][16]), for any number of candidates.  Frame f keeps its boxes in kept_rows [f][capacity][16] /
// kept_idx [f][capacity] and their number, at most capacity, in count[f]; a frame with more than `limit` candidates gets
// count[f] = -candidates and nothing else.
struct NmsArgs {
    const float* raw;
    int rows, batch;
    float score_thres, iou_thres;
    const MpStreamDesc* desc;    // letterbox of frame f: desc[f].scale / left / top, or
    const float* recover;        // [batch][3] scale, pad_x, pad_y [dev], or (both null) the three scalars below
    float scale, pad_x, pad_y;
    int limit, capacity;
    float* kept_rows;
    int* kept_idx;
    int* count;
    void* ws;                    // nms_workspace_bytes(ws_cap, batch) bytes [dev]
    int ws_cap;                  // candidates the workspace holds per frame, >= min(rows, limit)
};
size_t nms_workspace_bytes(int cap, int batch);
int launch_nms(const NmsArgs& a, cudaStream_t s);

int launch_mp_crop(const MpStreamDesc* d, const float* boxes, const int* count, int K, float face_scale, float min_face,
                   uint8_t* crops, int S, int* detail, int n, cudaStream_t s);
int launch_mp_landmark_post(const float* xy, const int* detail, const int* count, int K, int P, float* kps, int n, cudaStream_t s);

// judge_boxs + sort_and_filter (image_ops.cu).  src [dev] (top_k) or null: each selected face's source for the track ids,
// the row it came from when src_is_row (the rows are the previous track boxes), else the index of the track box its
// detection matched, -1 for none.  skps_select_faces is this with src null.
int launch_select_faces(const float* det_rows, const int32_t* det_count, int det_stride, const float* track, int n_track,
                        float iou_thres, float alpha, float one_minus_alpha, float min_face, int top_k, float* boxes4,
                        int32_t* count, int32_t* src, bool src_is_row, cudaStream_t s);
// The same per stream of a batch; src [dev] [S][K] as above, the rows being the track boxes where flag[s] == 0.  det_slot
// [dev] [S]: the detector frame (row of det_rows / det_count) of each stream, -1 where the detector did not run on it; null:
// frame s is stream s's.
int launch_mp_select(const float* det_rows, const int* det_count, int det_cap, const int* det_slot, const int* flag,
                     const float* track, const int* n_track, float iou_thres, float alpha, float oma, float min_face, int top_k,
                     float* boxes4, int* count, int* src, int n_streams, cudaStream_t s);
// flag[s] = the stream uses its detector rows: det_slot[s] >= 0 (det_slot null: always) and (!have_prev[s] or the mean
// difference > 5)
int launch_mp_decide(const unsigned long long* diff, const int* hw, const int* have_prev, const int* det_slot, int* flag, int n,
                     cudaStream_t s);
int launch_mp_temporal(const MpTemporalArgs& a, int n_streams, cudaStream_t s);
// Aligned face chips (align.cu): per face of stream g < n with i < count[g], M = similarity of kps[g][i] (P x 2 float64) to the
// ArcFace template at `size`, chips[g][i] = cv2.warpAffine(desc[g].cur, M, (size, size)); chips [n][K][size][size][3], M [n][K][2][3].
int launch_mp_align(const MpStreamDesc* d, const double* kps, const int* count, int K, int P, int size, uint8_t* chips,
                    double* M, int n, cudaStream_t s);

// Head pose (headpose.cu): get_head_pose for every face i < count[g] of every group g < G, one warp per face.  The 10 image
// points of a face are pts[g][i][idx[0..9]], rounded to float32; the camera of group g is [[W,0,W//2],[0,W,H//2],[0,0,1]].
struct PoseArgs {
    const double* pts64;         // [G][K][P][2] landmarks, float64 ...
    const float* pts32;          // ... or float32 (exactly one of the two is set)
    int G, K, P;
    int idx[10];                 // the landmarks paired with obj[0..9]
    const int* count;            // [G] faces per group, or null (all K); outputs of faces i >= count[g] are not written
    const int* hw;               // [G][2] frame H, W per group [dev], or null: H, W below for every group
    int H, W;
    float obj[30], cube[24];     // 3-D model points and the re-projected cube (pose.py)
    double *rvec, *tvec, *euler, *reproj;     // [G][K][3] x3, [G][K][8][2]
};
// idx, obj and cube of get_head_pose on 98-point WFLW landmarks (TRAIN/face_landmark/lib/dataset/headpose.py:48-78)
void pose_model_98(PoseArgs& a);
int launch_head_pose(const PoseArgs& a, cudaStream_t s);

}  // namespace skps
