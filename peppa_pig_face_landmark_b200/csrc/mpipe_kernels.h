// Kernels of the multi-stream pipeline (mpipe.cu): launchers defined in image_ops.cu / temporal.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct skps_pipeline_cfg;
struct skps_det_src;
struct skps_frame_layout;
struct skps_engine;

namespace skps {

// Where the pixels of a frame in layout SKPS_LAYOUT_* (skps_b200.h) are: pixel (y, x) has its B, G, R bytes at
// base + y * pitch + x * xs + off[0..2].  `plane` is the plane pitch of the planar layouts.  layout_ok: a known code.
struct PxLayout {
    int xs;
    long long off[3];
};
__host__ __device__ __forceinline__ bool layout_ok(int layout) { return layout >= 0 && layout <= 5; }
__host__ __device__ __forceinline__ int layout_xstep(int layout) { return layout >= 4 ? 1 : (layout >= 2 ? 4 : 3); }
__host__ __device__ __forceinline__ PxLayout px_layout(int layout, int plane) {
    PxLayout l;
    l.xs = layout_xstep(layout);
    const long long step = layout >= 4 ? (long long)plane : 1;       // channel c is c steps from the first in memory
    const bool rgb = layout & 1;
    l.off[0] = rgb ? 2 * step : 0;
    l.off[1] = step;
    l.off[2] = rgb ? 0 : 2 * step;
    return l;
}

// A frame stored H x W (row pitch `pitch`, layout and plane pitch as px_layout takes them) that must be turned `turns`
// quarter turns clockwise to be upright (cv2.rotate: 1 ROTATE_90_CLOCKWISE, 2 ROTATE_180, 3 ROTATE_90_COUNTERCLOCKWISE):
// pixel (y, x) of the upright frame, H' x W' (W x H for odd turns), has its B, G, R bytes at
// base + org + y * ystep + x * xstep + off[0..2].  Only the low two bits of `turns` are read.
struct PxView {
    long long org, ystep, xstep;
    long long off[3];
    int H, W;                    // the upright frame's size
};
__host__ __device__ __forceinline__ PxView px_view(int layout, int plane, int pitch, int H, int W, int turns) {
    const PxLayout l = px_layout(layout, plane);
    const long long p = pitch, s = l.xs;
    PxView v;
    v.off[0] = l.off[0]; v.off[1] = l.off[1]; v.off[2] = l.off[2];
    switch (turns & 3) {
        case 0: v.org = 0; v.ystep = p; v.xstep = s; break;
        case 1: v.org = (H - 1) * p; v.ystep = s; v.xstep = -p; break;
        case 2: v.org = (H - 1) * p + (W - 1) * s; v.ystep = -p; v.xstep = -s; break;
        default: v.org = (W - 1) * s; v.ystep = -s; v.xstep = p; break;
    }
    v.H = (turns & 1) ? W : H;
    v.W = (turns & 1) ? H : W;
    return v;
}

// Block g of a launch over n calls' frames serves stream stream[g] (stream null: g).  The per-frame inputs and outputs are
// in call order, rows g < n; the state is indexed by the stream, rows [S].
struct MpTemporalArgs {
    int top_k, n_points;
    const int* stream;           // [n] [dev] stream of each frame of the call, distinct, or null: frame g is stream g's
    const float* kps_now;        // [n][K][P][2] float32 landmarks in frame pixels (landmark_post)
    const int* count;            // [n] faces this frame
    const int* flag;             // [n] detector ran this frame
    const int* hw;               // [n][2] frame height, width
    const float* boxes4;         // [n][K][4] boxes the landmark stage used (boxes_return, facer.py:66)
    const int* src;              // [n][K] source of each face this frame (launch_select), an index into the old track
    // state, updated in place
    double* prev_lm;             // [S][2][K][P][2] previous landmark sets (ping-pong)
    double* prev_dx;             // [S][2][K][P][2] previous - filtered
    int* n_prev;                 // [S] sets in prev_lm (-1 = None)
    int* prev_f32;               // [S] previous_landmarks_set is a float32 array (numpy dtype bookkeeping)
    int* state_idx;              // [S] which half of prev_lm/prev_dx is current
    double* track_box;           // [S][K][4] float64 track boxes (returned as 'box')
    float* track_f32;            // [S][K][4] the same, as float32 (next frame's judge_boxs / crop input)
    int* n_track;                // [S]
    int64_t* ids;                // [S][K] track id of each track box
    int64_t* next_id;            // [S] the next unused id of the stream
    // id memory (skps_mpipe_set_id_memory): the lost tracks of each stream, most recently lost first.  id_memory 0: off,
    // the four pointers are not read and may be null
    int id_memory;               // frames in a row a lost track may be missing and still give its id back
    int64_t* mem_ids;            // [S][K] ids of the lost tracks
    float* mem_box;              // [S][K][4] their float32 boxes of the frame that last returned them
    int* mem_gap;                // [S][K] frames in a row each has been missing so far
    int* mem_n;                  // [S] entries held
    // outputs
    double* out_kps;             // [n][K][P][2]
    double* out_box;             // [n][K][4] copies of the new track boxes and their ids in call order, or null (not
    int64_t* out_ids;            // [n][K]    written; without a stream map they are rows 0..n-1 of track_box and ids)
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
    const uint8_t* src;          // the caller's device frame, gathered into cur by launch_frame_diff, or null (cur holds it)
    int src_pitch;               // bytes from one row of src to the next, >= xstep W, any alignment
    int src_plane;               // bytes from one plane of src to the next (planar layouts)
};

// Image ops (image_ops.cu): one kernel per op, launched by skps_pipeline (FaceAna), skps_mpipe (FaceAnaStreams) and the
// public skps_letterbox, skps_crop_resize, skps_select_faces, skps_landmark_post, skps_frame_absdiff_sum and
// skps_frame_ingest alike.  A launch covers one frame, given by pointer, size and row pitch with its per-frame counts and
// flags as scalars, or the n frames of a call, given by their descriptors desc [dev] (cur, H, W, row pitch 3 W) with
// per-frame device arrays.  Only the addressing at the top of a kernel tells the two apart; the per-element code is one.

// Letterbox (face_detector.py:45-71) of frame g into out + g * out_stride, in_h x in_w x 3 RGB.
struct LetterboxArgs {
    const uint8_t* frame; int H, W, pitch;      // the one frame (desc and src null) ...
    int rw, rh, top, left;                      // ... and its letterbox geometry
    const MpStreamDesc* desc;                   // or frame g's: desc[g], geometry included
    const skps_det_src* src;                    // or frame g's: src[g] (skps_letterbox_frames), whole or in row pairs,
    const skps_frame_layout* lay;               // with src: its pixel layout lay[g] [dev], or null (BGR)
    uint8_t* out; size_t out_stride;
    int in_h, in_w;
    const int* turns;                           // with src: quarter turns clockwise of frame g [dev], or null (none)
};
int launch_letterbox(const LetterboxArgs& a, int n, cudaStream_t s);

// Crop + resize (face_landmark.py:66-104) of faces i < count[g] of frame g into crops [g][i] (S x S x 3) and detail [g][i]
// ([h, w, y1, x1, add]); faces i >= count[g] of the K get zeros.
struct CropArgs {
    const uint8_t* frame; int H, W, pitch;      // the one frame (desc null), or
    const MpStreamDesc* desc;                   // frame g's: desc[g].cur, H, W
    const float* boxes; const int* count;       // [n][K][4], [n] [dev]
    int K;
    float face_scale, min_face;
    uint8_t* crops; int S; int* detail;         // [n][K][S][S][3], [n][K][5]
};
int launch_crop(const CropArgs& a, int n, cudaStream_t s);

// judge_boxs + sort_and_filter (facer.py:58-64), one block per frame.  Frame g selects from the rows of its detector frame
// f = det_slot[g] (det_slot null: f = g), det_count[f] rows of det_stride floats at det_rows + f * det_cap * det_stride,
// IoU-matched against its track boxes, when it ran the detector; else from its track boxes themselves (facer.py:61).
// Its track boxes are those of stream t = stream[g] (stream null: t = g): track [t], n_track[t].
// src [n][top_k] [dev] or null: each selected face's source for the track ids, the row it came from when the rows are the
// track boxes, else the index of the track box its detection matched, -1 for none.
struct SelectArgs {
    const float* det_rows; const int* det_count;    // [dev]
    int det_stride, det_cap;
    const int* det_slot;                            // [n] [dev] or null
    const int* flag;                                // [n] [dev]: frame g ran the detector, or null: flag1
    const float* track;                             // [streams][top_k][4] [dev], or null (no track boxes)
    const int* n_track;                             // [streams] [dev], or null: n_track1
    const int* stream;                              // [n] [dev] stream of frame g, or null: g
    int flag1, n_track1;
    float iou_thres, alpha, one_minus_alpha, min_face;
    int top_k;                                      // 1..SKPS_MAX_TOP_K
    float* boxes4; int* count; int* src;            // [n][top_k][4], [n], [n][top_k] [dev]
};
int launch_select(const SelectArgs& a, int n, cudaStream_t s);

// FaceLandmark.postprocess (face_landmark.py:106-115): the landmarks xy [n][K][P][2] of the crops described by detail
// [n][K][5] in frame pixels, kps [n][K][P][2]; zeros for faces i >= count[g].
int launch_landmark_post(const float* xy, const int* detail, const int* count, int K, int P, float* kps, int n, cudaStream_t s);

// The frame-difference gate (facer.py:111-113): sum[g] += sum |cur - prev| over frame g's bytes when have_prev.  A frame
// with src set is first gathered into cur in the same pass (the same integer sum as from a packed cur); its pixels are in
// `layout` (SKPS_LAYOUT_*, one for the launch; cur gets them as BGR).  Frame g is d[g] [dev], or (d null, n = 1) `one` of
// `bytes` bytes, any count when one.src is null; with d, bytes is the largest frame's packed size.
// Rotated frames: src of frame g must be turned turns[g] [dev] (d set) or one_turns (d null) quarter turns clockwise to be
// upright (px_view), and cur gets the upright frame, D.H x D.W; the sum is that of the upright frame.  A launch with turns
// null and one_turns 0 runs the unrotated kernels.
int launch_frame_diff(const MpStreamDesc* d, int n, const MpStreamDesc& one, size_t bytes, unsigned long long* sum,
                      cudaStream_t s, int layout = 0, const int* turns = nullptr, int one_turns = 0);

// Frame staging on the host side, shared by skps_pipeline and skps_mpipe.  upload_host_frame queues the H2D copy of a [host]
// frame of `bytes` bytes into dst on s: a pinned frame is copied as it is, a pageable one first into `stage` (pinned, at
// least `bytes`) so that the copy stays asynchronous and at full PCIe rate.  check_device_frame fails unless `frame` is
// device or managed memory of `device`; the error names the caller `fn` and, for index >= 0, the frame's index.
int upload_host_frame(const uint8_t* frame, size_t bytes, uint8_t* stage, uint8_t* dst, cudaStream_t s);
int check_device_frame(const void* frame, int device, const char* fn, int index);
// The device of a pipeline's two engines (engine.cu); fails, naming both devices, when they are on different devices.
int engine_pair_device(const skps_engine* det, const skps_engine* kps, const char* fn, int* device);

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

// flag[s] = the stream uses its detector rows: det_slot[s] >= 0 (det_slot null: always) and (!have_prev[s] or the mean
// difference > 5)
int launch_mp_decide(const unsigned long long* diff, const int* hw, const int* have_prev, const int* det_slot, int* flag, int n,
                     cudaStream_t s);
int launch_mp_temporal(const MpTemporalArgs& a, int n, cudaStream_t s);
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
