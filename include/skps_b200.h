/*
 * skps_b200 — C-ABI of the H100-native (sm_90a) FaceAna hot path.
 *
 * Drop-in boundary for 610265158/Peppa_Pig_Face_Landmark: the reference reaches
 * all of its neural arithmetic through one Python class,
 *     ONNXEngine(onnx_path)(ndarray) -> [ndarray, ...]
 *         (Skps/core/api/onnx_model_base.py:6-27, called from
 *          Skps/core/api/face_detector.py:29 and Skps/core/api/face_landmark.py:48)
 * and all of its image arithmetic through OpenCV/numpy calls in
 *     FaceDetector.preprocess / py_nms / scale_coords   (face_detector.py:45-136)
 *     FaceLandmark.preprocess / postprocess             (face_landmark.py:66-115)
 *     FaceAna.diff_frames / judge_boxs / sort_and_filter (facer.py:98-189)
 * Each entry point below names the reference function it replaces.  Plain
 * pointers and sizes only; `stream` is a cudaStream_t passed as void*.
 * All functions return 0 on success, non-zero on error; the message is
 * available from skps_last_error() (thread-local).
 *
 * Pointers marked [dev] are device pointers on the engine's device, [host] are
 * host pointers (pinned memory makes the copies asynchronous).
 */
#ifndef SKPS_B200_H
#define SKPS_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define SKPS_API __attribute__((visibility("default")))
#else
#define SKPS_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct skps_engine skps_engine;     /* one compiled network  (ONNXEngine,  onnx_model_base.py:6)  */
typedef struct skps_pipeline skps_pipeline; /* detector+landmark     (FaceAna,     facer.py:25)          */

SKPS_API const char* skps_last_error(void);
SKPS_API int skps_version(void);

/* ------------------------------------------------------------------ ONNXEngine (onnx_model_base.py:7-27) */

/* Build an engine from a lowered plan (peppa_pig_face_landmark_b200.lowering.lower(onnx_path)):
 * `plan_words` describe buffers/ops, `weights` is the float32 blob taken unchanged from the
 * .onnx initializers.  Replaces onnxruntime.InferenceSession(onnx_f) (onnx_model_base.py:14). */
SKPS_API int skps_engine_create(const int32_t* plan_words, size_t n_words,
                       const float* weights, size_t n_floats,
                       int max_batch, int device, skps_engine** out);
SKPS_API void skps_engine_destroy(skps_engine* e);

/* Introspection: input is uint8 NHWC (N,H,W,3); output i has `skps_engine_output_elems`
 * float32 per sample. */
SKPS_API int skps_engine_input_dims(const skps_engine* e, int* h, int* w, int* c);
SKPS_API int skps_engine_num_outputs(const skps_engine* e);
SKPS_API int skps_engine_output_elems(const skps_engine* e, int idx);
/* [dev] pointer of the engine-owned input buffer (N,H,W,3) uint8 — producers (letterbox,
 * crop) write here directly so there is no copy between stages. */
SKPS_API void* skps_engine_input_ptr(skps_engine* e);
/* [dev] pointer of the engine-owned output buffer idx, (max_batch, elems) float32. */
SKPS_API float* skps_engine_output_ptr(skps_engine* e, int idx);

/* session.run on device memory (onnx_model_base.py:23): `input` [dev] uint8 NHWC (batch,H,W,3)
 * (may be skps_engine_input_ptr itself), results left in the engine's output buffers and, when
 * outputs[i] != NULL, copied to outputs[i] [dev].  Asynchronous on `stream`. */
SKPS_API int skps_engine_forward(skps_engine* e, const uint8_t* input, int batch,
                        float* const* outputs, void* stream);

/* session.run with HOST buffers, exactly ONNXEngine.__call__'s contract
 * (onnx_model_base.py:17-27): `input` [host] float32 NCHW (batch,3,H,W) in [0,1] as the
 * reference feeds it; outputs[i] [host] float32.  H2D + compute + D2H, synchronous. */
SKPS_API int skps_engine_forward_host_f32(skps_engine* e, const float* input_nchw, int batch,
                                 float* const* outputs, void* stream);
/* Same with uint8 NHWC host input (crops / letterboxed frame before the /255). */
SKPS_API int skps_engine_forward_host_u8(skps_engine* e, const uint8_t* input_nhwc, int batch,
                                float* const* outputs, void* stream);

/* Streaming host round trip (additive): two slots; while one batch computes the next one's pixels cross PCIe on a
 * second stream.  `input` / `outputs[i]` [host, pinned] must stay valid until skps_engine_wait(slot) returns.
 * Order of use: submit(0) submit(1) wait(0) submit(0) wait(1) ... */
SKPS_API int skps_engine_submit_host_u8(skps_engine* e, int slot, const uint8_t* input_nhwc, int batch,
                                        float* const* outputs);
SKPS_API int skps_engine_wait(skps_engine* e, int slot);

/* Debug/parity: copy internal buffer `buf` (N,H,W,C float32 NHWC) of the last forward to host. */
SKPS_API int skps_engine_num_buffers(const skps_engine* e);
SKPS_API int skps_engine_buffer_dims(const skps_engine* e, int buf, int* h, int* w, int* c, int* dtype);
SKPS_API int skps_engine_read_buffer(skps_engine* e, int buf, int batch, void* dst_host);
/* Number of kernels one forward launches (for bench.py's gpu_launches). */
SKPS_API int skps_engine_launches_per_forward(const skps_engine* e);
/* Kernel launches of one forward at `batch` (0 for batch <= 0). */
SKPS_API int skps_engine_launches_for_batch(const skps_engine* e, int batch);
/* Profiling: enqueue only op `op_index` of the plan on the buffers left by the last forward
 * (bench.py times the dominant kernel with CUDA events around this call). */
SKPS_API int skps_engine_run_op(skps_engine* e, int op_index, int batch, void* stream);
/* Test hook: size the grids of the persistent kernels (conv_tc, conv_tct, conv_hm, conv_pw, conv_xf, conv_fpw, the stem
 * block; conv_mma: n x its CTAs per SM) for n SMs instead of the device's, so that every CTA walks more work units.  n = 0
 * restores the device's count; n < 0 or above it fails.  Drops the engine's captured forwards.  Results must not change:
 * what a unit computes depends only on its index. */
SKPS_API int skps_engine_set_num_sms(skps_engine* e, int n);
/* The launch of op `op_index` at `batch` under the current setting: out = {CTAs, work units} for a persistent kernel,
 * {0, 0} for any other op. */
SKPS_API int skps_engine_op_grid(const skps_engine* e, int op_index, int batch, int32_t out[2]);
/* Which kernel op `op_index` runs and the geometry it picked (for tests that must know which branch they exercised).
 * Returns a SKPS_KERNEL_* id, or -1 on a bad index.  info[0..3] (zero where unused):
 *   TC: bw, bh (output pixels of a 128-pixel tile), ipt (images per tile), mt (pixel tiles per weight tile);
 *   TCT: bh (output rows per 256-pixel tile);  DW_TMA: output rows per tile (tiles are 16 columns wide);
 *   PW: output channels per work unit, work units per 128-pixel tile;
 *   FPW: pixels per tile (128, 16 x 8), output channels per work unit, work units per tile, mode (0 scale, 1 depthwise). */
enum {
    SKPS_KERNEL_MISC = 0, SKPS_KERNEL_TC = 1, SKPS_KERNEL_TCT = 2, SKPS_KERNEL_HM = 3, SKPS_KERNEL_MMA = 4,
    SKPS_KERNEL_XF = 5, SKPS_KERNEL_SIMT_CONV = 6, SKPS_KERNEL_DW_TMA = 7, SKPS_KERNEL_DW = 8,
    SKPS_KERNEL_UPCAT_TMA = 9, SKPS_KERNEL_UPCAT = 10, SKPS_KERNEL_STEM_BLOCK = 11, SKPS_KERNEL_PW = 12,
    SKPS_KERNEL_FPW = 13
};
SKPS_API int skps_engine_op_kernel(const skps_engine* e, int op_index, int32_t info[4]);

/* Unit-test entry for the wgmma convolution kernel (csrc/conv_tc.cu): one 'same' conv on host
 * data.  x float32 NHWC, w_hi/w_lo float16 (n_tiles*n_tile, K_pad) as packed by
 * plan.pack_tc_weights, out float32 NHWC. */
SKPS_API int skps_debug_conv_tc(const float* x, int N, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                                const float* bias, int Cout, int ksize, int dil, int act, int n_tile, int n_tiles,
                                float out_scale, const float* residual, int out_split, float* out);
/* Same plus the conv stride (1 or 2: TMA element strides; out is N x H/stride x W/stride x Cout), the residual
 * order (res_first != 0: act(conv + bias + residual), the ResNet/HRNet block of the Teacher, model.py:302-345)
 * and the capacity max_batch >= N of the device buffers (maps smaller than 128 pixels share a tile between
 * images; N not a multiple of that exercises the partial tile). */
SKPS_API int skps_debug_conv_tc2(const float* x, int N, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                                 const float* bias, int Cout, int ksize, int dil, int act, int n_tile, int n_tiles,
                                 float out_scale, const float* residual, int out_split, float* out, int stride,
                                 int res_first, int max_batch);

/* Unit-test entry of the pointwise kernel (csrc/conv_pw.cu): one 1x1 stride-1 conv of the first `batch` images of
 * host buffers holding max_batch.  x float32 (max_batch, H, W, in_ld), read at channels [in_coff, in_coff + Cin); w_hi/w_lo
 * float16 (n_tiles*n_tile, K_pad) as packed by plan.pack_tc_weights; act none, ReLU or h-swish; out float32
 * (max_batch, H, W, out_ld), in and out: the conv writes channels [out_coff, out_coff + Cout) of the first batch*H*W
 * pixels (through split-fp16 planes when out_split != 0) and leaves the rest as it came in.  Fails for a layer the
 * kernel does not take (unaligned views, Cout not a multiple of 8). */
SKPS_API int skps_debug_conv_pw(const float* x, int batch, int max_batch, int H, int W, int Cin, int in_ld, int in_coff,
                                const void* w_hi, const void* w_lo, const float* bias, int Cout, int act, int n_tile,
                                int n_tiles, float out_scale, int out_split, int out_ld, int out_coff, float* out);

/* Unit-test entry of the transposed heat-map head kernel (csrc/conv_hm.cu; kps graph /student/hm/Conv + the arg-max half of
 * postp, TRAIN/face_landmark/lib/core/base_trainer/model.py:511-554): x float32 NHWC, w_hi/w_lo (n_tile, K_pad) float16 as
 * packed by plan.pack_tc_weights -> per 256-pixel tile and channel the maximum score and its first pixel index (y*W+x):
 * val / idx are [N][H*W/256][128] float32 / int32. */
SKPS_API int skps_debug_conv_hm(const float* x, int N, int H, int W, int Cin, const void* w_hi, const void* w_lo,
                                const float* bias, int Cout, int n_tile, float out_scale, float* val, int* idx);

/* Debug/unit-test entry of the fused producer -> 1x1 conv kernels (csrc/conv_xf.cu): mode 0 = squeeze-excite scale
 * (x * gate[n,c]) ahead of the conv, mode 1 = depthwise 3x3 [over concat(bilinear_x2(low), x)] ahead of the conv.
 * Replaces, for one layer, what onnxruntime runs for the reference's ONNX nodes Mul->Conv / Resize->Concat->Conv(dw)->Conv
 * (Skps/core/api/onnx_model_base.py:23).  Host float32 NHWC in/out; w_hi/w_lo as packed by plan.pack_tc_weights.  `out` is
 * read as well as written, so elements the kernel leaves unwritten come back as they went in. */
SKPS_API int skps_debug_conv_xf(int mode, const float* x, int N, int H, int W, int Cx, int x_split, const float* low, int Cl,
                                const float* gate, const float* dww, int dw_act, const void* w_hi, const void* w_lo,
                                const float* bias, int Cout, int act, int n_tile, float out_scale, const float* residual,
                                int res_first, int out_split, float* out, const float* weff);
/* The same layer through the register-accumulator kernel (csrc/conv_fpw.cu), for images [0, batch) of N: `out` is read
 * as well as written, and images past the batch must come back as they went in.  Fails for a layer conv_fpw does not take
 * (maps not made of whole 16 x 8 tiles, widths it does not instantiate). */
SKPS_API int skps_debug_conv_fpw(int mode, const float* x, int N, int H, int W, int Cx, int x_split, const float* low, int Cl,
                                 const float* gate, const float* dww, int dw_act, const void* w_hi, const void* w_lo,
                                 const float* bias, int Cout, int act, int n_tile, float out_scale, const float* residual,
                                 int res_first, int out_split, float* out, const float* weff, int batch);

/* Unit-test entries for two fused kernels that otherwise only run inside a whole network (csrc/debug_ops.cu):
 * the squeeze-excite gate (mean of per-tile channel sums -> FC -> act -> FC -> act; kps_student.onnx .../se/ nodes) and the
 * heat-map decode (arg-max + offsets, TRAIN/face_landmark/lib/core/base_trainer/model.py:511-554).  Host float32. */
SKPS_API int skps_debug_se_fc(const float* part, int N, int tiles, int C, const float* w1t, const float* b1, const float* w2t,
                              const float* b2, int Cr, int act1, int act2, int hw, float* gate);
SKPS_API int skps_debug_hm_decode(const float* hm, int N, int H, int W, int ld, int npts, const float* feat, int K,
                                  const float* w_off, const float* b_off, float* xy, float* score);

/* Unit-test entry for the few-channel 3x3 convolution kernel (csrc/conv_mma.cu; Cin == Cout == C in {24, 40}, the
 * Teacher's HRNet branch convs): x, residual, out float32 NHWC; w_packed float16 [tap][hi/lo][C][C] as packed by
 * plan.pack_mma_weights. */
SKPS_API int skps_debug_conv_mma(const float* x, int N, int H, int W, int C, const void* w_packed, const float* bias,
                                 int act, float out_scale, const float* residual, int res_first, int out_split,
                                 float* out);

/* ------------------------------------------------------------------ image kernels */

/* Pixel layouts of frames already in device memory (the `layout` arguments and skps_frame_layout below).  Pixel (y, x)
 * of a frame at `base` with row pitch `pitch` has its blue, green and red bytes at
 *     base + y*pitch + x*xstep + off[c]
 * with, per layout, xstep and off[B, G, R]:
 *     SKPS_LAYOUT_BGR         3, {0, 1, 2}          HxWx3, the reference's own layout
 *     SKPS_LAYOUT_RGB         3, {2, 1, 0}          HxWx3 (DALI's default)
 *     SKPS_LAYOUT_BGRA        4, {0, 1, 2}          HxWx4, the 4th byte's value is never used
 *     SKPS_LAYOUT_RGBA        4, {2, 1, 0}
 *     SKPS_LAYOUT_BGR_PLANAR  1, {0, P, 2P}         3xHxW, planes P = plane_pitch bytes apart
 *     SKPS_LAYOUT_RGB_PLANAR  1, {2P, P, 0}         (torchvision.io.decode_jpeg on the GPU, NCHW video decoders)
 * Row pitches are >= xstep * W (any value for a one-row frame), plane pitches >= 0; both fit int32.  The kernels only
 * compute addresses this way and keep their arithmetic: a frame gives, bit for bit, the results of the same pixels
 * passed as interleaved BGR.  0 is BGR, so a zeroed skps_frame_layout describes a BGR frame. */
enum {
    SKPS_LAYOUT_BGR = 0, SKPS_LAYOUT_RGB = 1, SKPS_LAYOUT_BGRA = 2, SKPS_LAYOUT_RGBA = 3, SKPS_LAYOUT_BGR_PLANAR = 4,
    SKPS_LAYOUT_RGB_PLANAR = 5
};

/* Frames stored turned (the *_rotate entries): `turns` is the number of quarter turns clockwise, 0..3, by which the stored
 * frame must be turned to be upright; the frame is analysed as cv2.rotate(frame, code) with 1 ROTATE_90_CLOCKWISE,
 * 2 ROTATE_180 and 3 ROTATE_90_COUNTERCLOCKWISE.  A frame's H, W and pitch describe it as stored; pixel (y, x) of the
 * upright frame (W x H for odd turns) is at
 *     base + org + y*ystep + x*xstep + off[c]
 * with, for a row pitch p and the layout's xstep s:
 *     0: org 0,                    ystep  p, xstep  s
 *     1: org (H-1)p,               ystep  s, xstep -p
 *     2: org (H-1)p + (W-1)s,      ystep -p, xstep -s
 *     3: org (W-1)s,               ystep -s, xstep  p
 * The kernels only compute addresses this way and keep their arithmetic: every result, in upright coordinates, is bit for
 * bit that of the upright frame passed as a contiguous frame.  Entries taking a [dev] turns array read its low two bits
 * only; the others fail on a value outside 0..3.  A NULL turns array, or turns 0, means no turn and runs the kernels of
 * the entries without it. */

/* FaceDetector.preprocess (face_detector.py:45-71): BGR->RGB, cv2.resize INTER_LINEAR
 * (bit-exact 11-bit fixed point) to (rw,rh), pad with 114 to (in_h,in_w).  `frame` [dev]
 * HxWx3 uint8 with row pitch `pitch` bytes; `out` [dev] in_h*in_w*3 uint8 RGB.  The /255 is
 * done inside the first conv. */
SKPS_API int skps_letterbox(const uint8_t* frame, int H, int W, int pitch,
                   uint8_t* out, int in_h, int in_w,
                   int rw, int rh, int top, int left, void* stream);

/* Where one frame's pixels are, for skps_letterbox_frames.  With row_pairs = 0, `base` holds the
 * whole H x W frame, rows `pitch` bytes apart (a CUDA frame read where it is, at any pitch).  With
 * row_pairs = 1, `base` holds 2*rh rows `pitch` bytes apart: rows 2y and 2y+1 are the frame rows
 * i0 and i1 of cv2's vertical tap for resized row y (linear_tap(y, rh, H) in image_ops.cu), the
 * only rows output row top+y reads.  Both rows of a pair are always held, even where the weight of
 * i1 is 0.  FaceDetector uploads a host frame that way when 2*rh < H, so a 4K frame at 384x640
 * sends 720 of its 2160 rows. */
typedef struct skps_det_src {
    const uint8_t* base;                /* [dev] the rows of the frame this descriptor holds          */
    int32_t pitch;                      /* bytes from one held row to the next (>= 3W, any alignment) */
    int32_t H, W;                       /* the whole frame                                            */
    int32_t rw, rh, top, left;          /* letterbox geometry (face_detector.py:49-62)                */
    int32_t row_pairs;                  /* 0: base holds rows 0..H-1; 1: base holds 2*rh row pairs    */
} skps_det_src;

/* skps_letterbox for n frames (0..65535) of any sizes in one launch: frame i, described by src[i]
 * [dev], is letterboxed into out [dev] + i*in_h*in_w*3.  The bytes of each frame are those
 * skps_letterbox writes for the whole frame with the same geometry. */
SKPS_API int skps_letterbox_frames(const skps_det_src* src, int n, uint8_t* out, int in_h, int in_w, void* stream);

/* The pixel layout of one frame for the *_layout entries: a SKPS_LAYOUT_* code and, for the planar layouts, the bytes
 * from one plane to the next.  A zeroed entry is interleaved BGR, what the descriptors alone describe. */
typedef struct skps_frame_layout {
    int32_t layout;
    int32_t plane_pitch;
} skps_frame_layout;

/* skps_letterbox_frames for frames in any SKPS_LAYOUT_*: frame i's pixels are laid out as lay[i] [dev] (n) says, its row
 * pitch src[i].pitch >= xstep * W; lay NULL: every frame is BGR (skps_letterbox_frames).  The bytes are those of the
 * same pixels as an interleaved BGR frame.  row_pairs frames are BGR. */
SKPS_API int skps_letterbox_frames_layout(const skps_det_src* src, const skps_frame_layout* lay, int n, uint8_t* out,
                                          int in_h, int in_w, void* stream);
/* skps_letterbox_frames_layout for frames stored turned: frame i must be turned turns[i] [dev] (n) quarter turns clockwise
 * (see SKPS_LAYOUT_* above); src[i].H, W and pitch describe it as stored, its letterbox geometry (rw, rh, top, left) that of
 * the upright frame.  row_pairs frames are read unturned.  turns NULL: skps_letterbox_frames_layout. */
SKPS_API int skps_letterbox_frames_rotate(const skps_det_src* src, const skps_frame_layout* lay, const int32_t* turns, int n,
                                          uint8_t* out, int in_h, int in_w, void* stream);

/* xywh2xyxy + py_nms + scale_coords (face_detector.py:73-136) on the raw (rows,16) output.
 * Writes up to max_det (<= 256) kept rows (16 floats each, cols 0-3 mapped back to frame pixels),
 * their row indices into the raw output, and the count.  All [dev].  This entry keeps its limit:
 * with more than 1024 rows over the score threshold it writes count = -candidates and nothing
 * else.  skps_detect_post_batch below has no limit. */
SKPS_API int skps_detect_post(const float* raw, int rows, float score_thres, float iou_thres,
                     float scale, float pad_x, float pad_y,
                     float* kept_rows, int32_t* kept_idx, int32_t* count, int max_det,
                     void* stream);

/* The same post-processing for any number of candidates (up to every row), for `batch` frames at
 * once: raw [dev] (batch,rows,16); recover [dev] (batch,3) float32 = scale, pad_x, pad_y of each
 * frame's letterbox.  Frame f gets its kept rows in kept_rows [dev] (batch,capacity,16), their row
 * indices in kept_idx [dev] (batch,capacity) and their number, min(kept, capacity), in count[f]
 * [dev]; capacity >= rows keeps every box.  Candidates are ranked by (score, row index) descending
 * and suppressed exactly as py_nms does.  `workspace` [dev] holds at least
 * skps_detect_post_workspace_size(rows, batch) bytes (about 40 bytes per row and frame); the call
 * allocates nothing.  Asynchronous on `stream`. */
SKPS_API size_t skps_detect_post_workspace_size(int rows, int batch);
SKPS_API int skps_detect_post_batch(const float* raw, int rows, int batch, float score_thres, float iou_thres,
                                    const float* recover, float* kept_rows, int32_t* kept_idx, int32_t* count,
                                    int capacity, void* workspace, size_t workspace_bytes, void* stream);

/* FaceAna.judge_boxs + sort_and_filter (facer.py:120-189): IoU-match detections against the
 * previous track boxes (EMA alpha), drop area<=min_face, keep top_k (1..SKPS_MAX_TOP_K) by area:
 * all of them in detector order when at most top_k pass, else the top_k largest, descending,
 * equal areas later index first.  Any number of detections; one block per call, a radix select
 * whose passes over the detections do not grow with top_k.  `track` [dev] (n_track,4) may be
 * NULL.  Writes (count,4) boxes. */
SKPS_API int skps_select_faces(const float* det_rows, const int32_t* det_count, int det_stride,
                      const float* track, int n_track,
                      float iou_thres, float alpha, float one_minus_alpha,
                      float min_face, int top_k,
                      float* boxes4, int32_t* count, void* stream);

/* skps_select_faces with no track boxes (FaceAna.run on a new or just-reset FaceAna) for n images (>= 0) at once, one
 * block per image: image i selects from its det_count[i] [dev] rows of 16 floats at det_rows [dev] + i*det_cap*16 (the
 * kept_rows / count layout of skps_detect_post_batch with capacity det_cap) and writes its count[i] [dev] boxes to
 * boxes4 [dev] + i*top_k*4.  Same rule and same bytes as skps_select_faces on each image alone. */
SKPS_API int skps_select_faces_batch(const float* det_rows, const int32_t* det_count, int det_cap, int n, float min_face,
                                     int top_k, float* boxes4, int32_t* count, void* stream);

/* The box FaceAna.run returns for a face on a frame with no history (facer.py:75-82, judge_boxs(boxes, rects(kps))),
 * for n_faces (>= 0) faces of many images: face f has landmarks kps [dev] (n_faces,n_points,2) float32 and belongs to
 * image face_image[f] [dev] int32, whose selected boxes are sel_boxes [dev] (images,top_k,4), sel_count [dev] of them.
 * boxes_out[f] [dev] (n_faces,4) float32 is the landmarks' rectangle [min x, min y, max x, max y], or, when the first
 * selected box of its image whose IoU with that rectangle is above iou_thres exists, alpha*rect + one_minus_alpha*box
 * in float32 (rounded like numpy's float32 expression).  One warp per face. */
SKPS_API int skps_landmark_boxes(const float* kps, int n_points, const int32_t* face_image, int n_faces,
                                 const float* sel_boxes, const int32_t* sel_count, int top_k, float iou_thres, float alpha,
                                 float one_minus_alpha, float* boxes_out, void* stream);

/* FaceLandmark.preprocess (face_landmark.py:66-104) for all faces at once: zero-pad, square
 * crop, cv2.resize to (out_hw,out_hw), uint8 BGR NHWC.  `boxes4` [dev] (max_faces,4), `count`
 * [dev].  `detail` [dev] (max_faces,5) int32 = [h,w,y1,x1,add].  Faces >= *count are zeroed. */
SKPS_API int skps_crop_resize(const uint8_t* frame, int H, int W, int pitch,
                     const float* boxes4, const int32_t* count, int max_faces,
                     float face_scale /* float32(1+2*extend) */, float min_face,
                     uint8_t* crops, int out_hw, int32_t* detail, void* stream);

/* Where one face's pixels are, for skps_crop_faces and skps_warp_faces: `base` [dev] holds the rectangle of an H x W
 * frame that starts at column ox, row oy and is rw x rh pixels, rows `pitch` bytes apart.  A face
 * in a whole frame has ox = oy = 0, rw = W, rh = H; a face may also point at just the rectangle its
 * crop can read (FaceLandmark's host frames upload only that). */
typedef struct skps_face_src {
    const uint8_t* base;
    int32_t pitch;
    int32_t H, W;                       /* the whole frame                               */
    int32_t ox, oy, rw, rh;             /* the rectangle base holds                      */
    int32_t _pad;
} skps_face_src;

/* skps_crop_resize for n faces (0..65535) that may each come from a different frame, in one launch:
 * face i is cropped from src[i] [dev] with box boxes4[i] [dev] (n,4).  Geometry, zero border and
 * bilinear are skps_crop_resize's, so crops [dev] (n,out_hw,out_hw,3) and detail [dev] (n,5) are
 * the bytes it writes for the same box on the whole frame.  The rectangle of src[i] must hold
 * every pixel of the frame the crop reads. */
SKPS_API int skps_crop_faces(const skps_face_src* src, const float* boxes4, int n, float face_scale,
                             float min_face, uint8_t* crops, int out_hw, int32_t* detail, void* stream);
/* skps_crop_faces for faces of frames in any SKPS_LAYOUT_*: face i's frame is laid out as lay[i] [dev] (n) says; lay NULL:
 * every frame is BGR (skps_crop_faces).  The crops stay BGR: the bytes of the same pixels as an interleaved BGR frame. */
SKPS_API int skps_crop_faces_layout(const skps_face_src* src, const skps_frame_layout* lay, const float* boxes4, int n,
                                    float face_scale, float min_face, uint8_t* crops, int out_hw, int32_t* detail,
                                    void* stream);
/* skps_crop_faces_layout for faces of frames stored turned: face i's frame must be turned turns[i] [dev] (n) quarter turns
 * clockwise and its box is in the upright frame.  A turned frame is read whole (its ox, oy, rw, rh are not read); one of
 * turn 0 may be a rectangle as for skps_crop_faces.  turns NULL: skps_crop_faces_layout. */
SKPS_API int skps_crop_faces_rotate(const skps_face_src* src, const skps_frame_layout* lay, const int32_t* turns,
                                    const float* boxes4, int n, float face_scale, float min_face, uint8_t* crops, int out_hw,
                                    int32_t* detail, void* stream);

/* FaceLandmark.postprocess (face_landmark.py:106-115): x*w + x1 - add, y*h + y1 - add. */
SKPS_API int skps_landmark_post(const float* xy_norm, const int32_t* detail, const int32_t* count,
                       int max_faces, int n_points, float* kps, void* stream);

/* FaceAna.diff_frames (facer.py:98-118): sum |a-b| over n bytes into *sum [dev] (uint64). */
SKPS_API int skps_frame_absdiff_sum(const uint8_t* a, const uint8_t* b, size_t n,
                           unsigned long long* sum, void* stream);
/* Frame ingest, the device-frame step of skps_pipeline_* and skps_mpipe_*: gathers an HxWx3 uint8 [dev] frame whose
 * rows start `pitch` bytes apart (pitch >= 3W; frame and pitch of any alignment, e.g. a decoder surface or an ROI view)
 * into `packed` [dev] (H*W*3 bytes, 16-byte aligned), and in the same pass sets *sum [dev] (uint64) to sum |frame - prev|
 * over all bytes, exactly what skps_frame_absdiff_sum(prev, packed) returns; prev [dev] (packed, 16-byte aligned) may be
 * NULL (copy only, *sum = 0).  Asynchronous on `stream`. */
SKPS_API int skps_frame_ingest(const uint8_t* frame, int H, int W, int pitch, uint8_t* packed, const uint8_t* prev,
                               unsigned long long* sum, void* stream);
/* skps_frame_ingest for a frame in any SKPS_LAYOUT_*: `packed` gets the frame as interleaved BGR (H*W*3 bytes) and *sum
 * is sum |packed - prev|, the bytes and the sum skps_frame_ingest gives for the same pixels passed as BGR.  pitch >=
 * xstep * W (H == 1: any); plane_pitch is read for the planar layouts only.  skps_frame_ingest is this entry with BGR. */
SKPS_API int skps_frame_ingest_layout(const uint8_t* frame, int H, int W, int pitch, int layout, int plane_pitch,
                                      uint8_t* packed, const uint8_t* prev, unsigned long long* sum, void* stream);
/* skps_frame_ingest_layout for a frame stored turned `turns` (0..3) quarter turns clockwise: H, W and pitch describe the
 * stored frame, `packed` gets the upright frame (W x H for odd turns) as interleaved BGR and *sum is sum |packed - prev|,
 * the bytes and the sum skps_frame_ingest gives for the upright frame.  turns 0: skps_frame_ingest_layout. */
SKPS_API int skps_frame_ingest_rotate(const uint8_t* frame, int H, int W, int pitch, int layout, int plane_pitch, int turns,
                                      uint8_t* packed, const uint8_t* prev, unsigned long long* sum, void* stream);

/* ------------------------------------------------------------------ FaceAna.run (facer.py:52-85) */

/* Largest top_k of skps_select_faces and skps_pipeline_* (the reference's Detect.topk has no cap). */
#define SKPS_MAX_TOP_K 1024
/* Faces per landmark forward in skps_pipeline_run: the landmark engine needs max_batch >=
 * min(top_k, SKPS_LANDMARK_CHUNK).  The Student@256 plan holds about 47 MB of activations per
 * face of max_batch, so a full chunk takes about 3 GB whatever top_k is. */
#define SKPS_LANDMARK_CHUNK 64

typedef struct skps_pipeline_cfg {
    float score_thres, iou_thres;       /* Skps.yml Detect.score_thrs / iou_thrs         */
    float min_face;                     /* Detect.min_face (area)                        */
    int   top_k;                        /* Detect.topk                                   */
    float track_iou, alpha;             /* Trace.iou_thres / smooth_box                  */
    float face_scale;                   /* float32(1 + 2*Keypoints.base_extend_range[0]) */
    float kps_min_face;                 /* FaceLandmark.min_face (20)                    */
    int   max_h, max_w;                 /* largest frame accepted                        */
} skps_pipeline_cfg;

SKPS_API int skps_pipeline_create(skps_engine* det, skps_engine* kps, const skps_pipeline_cfg* cfg,
                         skps_pipeline** out);
SKPS_API void skps_pipeline_destroy(skps_pipeline* p);
/* FaceAna.reset (facer.py:200-208): forget the previous frame. */
SKPS_API int skps_pipeline_reset(skps_pipeline* p);

/* One frame, detector path of FaceAna.run (facer.py:56-68): letterbox -> detector -> NMS ->
 * judge_boxs(track) -> sort_and_filter -> crops -> landmark net -> de-normalise, with no host
 * round trip in between.  Runs on the frame staged by skps_pipeline_frame_diff or
 * skps_pipeline_frame_diff_device, at the size it was staged with; fails when none is staged.
 * Afterwards that frame is the previous frame and no frame is staged.
 * Letterbox geometry (rw,rh,top,left,scale) is computed by the caller exactly as
 * face_detector.py:51-62 does.  `track` [host] (n_track,4) float32 previous track boxes or
 * NULL.  If run_detector==0 the `track` boxes are used as the face boxes (facer.py:61).
 * top_k is 1..SKPS_MAX_TOP_K and `track` holds at most max(256, top_k) boxes.
 * The face count is read back after the selection, then the landmark net runs on exactly the
 * n_faces crops, in ceil(n_faces / SKPS_LANDMARK_CHUNK) forwards (none for a faceless frame).
 * The landmark engine captures one CUDA graph per batch size it meets, so up to
 * SKPS_LANDMARK_CHUNK graphs are captured lazily, each on the first frame with that many faces
 * in a chunk.  A face's results do not depend on the chunk it runs in.
 * Results [host]: n_faces, boxes (top_k,4) — the boxes handed to the landmark stage
 * (facer.py:66 boxes_return), kps (top_k,n_points,2), scores (top_k,n_points),
 * n_det = the number of boxes the detector kept (every one of them goes through judge_boxs and
 * sort_and_filter); det_idx (256) and det_rows (256,16), may be NULL: the first min(n_det, 256)
 * kept row indices and rows (parity checks; skps_pipeline_det_results returns all of them).
 * Memory: room for every detector row as a kept box plus the NMS workspace, about 108 bytes per
 * detector row (1.6 MB at 384x640, 15 MB at 1152x1920).  Synchronous. */
SKPS_API int skps_pipeline_run(skps_pipeline* p, int run_detector, int rw, int rh, int top, int left, float scale,
                      const float* track, int n_track,
                      int32_t* n_faces, float* boxes4, float* kps, float* scores,
                      int32_t* n_det, int32_t* det_idx, float* det_rows, void* stream);

/* Every kept row of the last skps_pipeline_run that ran the detector: det_idx [host] (n_det) and
 * det_rows [host] (n_det,16), either may be NULL; fails if capacity < n_det.  Copies only n_det
 * rows from the device.  Synchronous. */
SKPS_API int skps_pipeline_det_results(skps_pipeline* p, int capacity, int32_t* det_idx, float* det_rows);

/* Track-id sources of the faces the last skps_pipeline_run returned: src [host] (n) int32, n <= that run's n_faces.
 * Face i's source is, on a detector frame, the index of the first `track` box its detection matched (IoU > track_iou),
 * -1 for none; with run_detector == 0 the index of the `track` box it is.  Copied back with the run's other results:
 * no device work, no synchronisation. */
SKPS_API int skps_pipeline_face_sources(skps_pipeline* p, int n, int32_t* src);

/* Stage a frame for skps_pipeline_run / skps_pipeline_commit_frame and return its mean absolute
 * difference to the previous frame (facer.py:111-113), or -1.0 in *mean_diff when there is no
 * previous frame of the same size.  `frame` [host] HxWx3 uint8 BGR, pinned or pageable. */
SKPS_API int skps_pipeline_frame_diff(skps_pipeline* p, const uint8_t* frame, int H, int W, double* mean_diff,
                                      void* stream);
/* skps_pipeline_frame_diff for a frame already on the pipeline's device, HxWx3 uint8 BGR with rows `pitch` bytes apart
 * (pitch >= 3W, any alignment): one skps_frame_ingest pass stages it and sums the difference.  The frame is read after all
 * work queued on `producer_stream` before this call (the stream that wrote it; 0 is the legacy default stream), and work
 * queued on producer_stream after this call returns runs after the read, so the producer may overwrite the frame at once. */
SKPS_API int skps_pipeline_frame_diff_device(skps_pipeline* p, const uint8_t* frame, int H, int W, int pitch,
                                             void* producer_stream, double* mean_diff, void* stream);
/* skps_pipeline_frame_diff_device for a frame in any SKPS_LAYOUT_* (pitch and plane_pitch as skps_frame_ingest_layout
 * takes them): the frame is staged as interleaved BGR, so everything after it sees the frame the BGR entry stages for the
 * same pixels.  skps_pipeline_frame_diff_device is this entry with BGR. */
SKPS_API int skps_pipeline_frame_diff_device_layout(skps_pipeline* p, const uint8_t* frame, int H, int W, int pitch,
                                                    int layout, int plane_pitch, void* producer_stream, double* mean_diff,
                                                    void* stream);
/* skps_pipeline_frame_diff_device_layout for a frame stored turned `turns` (0..3) quarter turns clockwise (H, W, pitch as
 * stored): the frame is staged upright, so the gate, skps_pipeline_run, pose and alignment see the upright frame, of size
 * W x H for odd turns, and consecutive frames may change turns.  turns 0: skps_pipeline_frame_diff_device_layout. */
SKPS_API int skps_pipeline_frame_diff_device_rotate(skps_pipeline* p, const uint8_t* frame, int H, int W, int pitch,
                                                    int layout, int plane_pitch, int turns, void* producer_stream,
                                                    double* mean_diff, void* stream);
/* Adopt the staged frame as the previous frame without running the chain: the skip path of FaceAna.run (facer.py:57-62
 * replaces previous_image on every call, also when nothing is detected or tracked).  Fails when no frame is staged. */
SKPS_API int skps_pipeline_commit_frame(skps_pipeline* p);

/* WFLW evaluation helpers (TRAIN/face_landmark/tools/eval_WFLW.py).  skps_crop_rect: zero-bordered rectangular crop of a
 * [dev] BGR frame resized to out_hw x out_hw, bit-exact with copyMakeBorder + slicing + cv2.resize (:38-80, :113-124).
 * skps_nme: per-face normalised mean error, mean_p |pred - gt| / |gt[norm_a] - gt[norm_b]| (:84-95; WFLW: 60, 72); all [dev]. */
SKPS_API int skps_crop_rect(const uint8_t* frame, int H, int W, int pitch, int rx, int ry, int rw, int rh, uint8_t* out,
                            int out_hw, void* stream);
SKPS_API int skps_nme(const float* target, const float* preds, int n, int n_points, int norm_a, int norm_b, float* out,
                      void* stream);

/* Batched head pose (csrc/headpose.cu), the GPU counterpart of Skps/core/headpose/pose.py:48-77 get_head_pose():
 * solvePnP (iterative) on 10 landmark/model point pairs with the camera matrix [[w,0,w//2],[0,w,h//2],[0,0,1]], projection
 * of the 8 cube corners, Euler angles as cv2.decomposeProjectionMatrix reports them.  pts [host] (N,10,2) float32 in the
 * order of pose.py:60-61; object_pts (10,3), cube_pts (8,3) float32.  Outputs [host] float64: rvec (|rvec| <= pi), tvec,
 * euler (N,3), reproject (N,8,2).  The Euler triple is the classic RQDecomp3x3's; where the decomposition is ambiguous it
 * can differ from OpenCV's while composing to the same R = Rz(roll) Ry(yaw) Rx(pitch): at a pitch of exactly 180 degrees
 * with nonzero yaw (Ry(pi - 0.1): (180, 5.73, 180) here, (0, 174.27, 0) from OpenCV 4.13), at exact 180-degree rotations
 * about some axes, and within |cos yaw| < 1e-3 of gimbal lock, where the first Givens rotation is normalised exactly. */
SKPS_API int skps_head_pose(const float* pts, int N, int img_w, int img_h, const float* object_pts, const float* cube_pts,
                            double* rvec, double* tvec, double* euler, double* reproject);

/* The head-pose solver's rotation helpers on their own, run in device code (test entry): R_out[i] = rotation matrix of the
 * rotation vector r_in[i] (cv2.Rodrigues), r_out[i] = rotation vector of R_in[i] (cv2.Rodrigues of a matrix), euler_out[i]
 * = Euler angles of R_in[i] in degrees (cv2.RQDecomp3x3; at exact 180-degree rotations about some axes and within about 1e-5
 * of yaw = +-90 degrees the triple may differ from OpenCV's but composes to the same R).  r_in (n,3), R_in (n,3,3)
 * row-major; all [host] float64. */
SKPS_API int skps_debug_rotation(const double* r_in, const double* R_in, int n, double* R_out, double* r_out,
                                 double* euler_out);

/* ---- FaceAna.run for many concurrent video streams (csrc/mpipe.cu; SURVEY 8f-1, 8f-2) ---------------------------------
 * What one FaceAna instance per stream does on the host in the reference (facer.py:52-85 with GroupTrack / OneEuroFilter /
 * EmaFilter of Skps/core/smoother/lk.py:6-162) happens here for up to n_streams streams per call with all per-stream state
 * on the device: one detector forward and one landmark forward per call, batched over the streams.
 * det needs max_batch >= n_streams, kps needs max_batch >= n_streams * cfg->top_k.  Every stream may keep any number of
 * detector boxes; the NMS output and workspace take about 108 bytes per detector row and stream.  Not thread-safe per
 * handle. */
typedef struct skps_mpipe skps_mpipe;
SKPS_API int skps_mpipe_create(skps_engine* det, skps_engine* kps, const skps_pipeline_cfg* cfg, int n_streams,
                               skps_mpipe** out);
SKPS_API void skps_mpipe_destroy(skps_mpipe* p);
/* FaceAna.reset() for one stream (or all: stream = -1): forget the previous frame, the track boxes, the landmark history;
 * the stream's track ids start from 0 again. */
SKPS_API int skps_mpipe_reset(skps_mpipe* p, int stream);
SKPS_API int skps_mpipe_dims(const skps_mpipe* p, int* n_streams, int* top_k, int* n_points);
/* Enqueue frame i (HxWx3 uint8 BGR, [host] pinned or pageable) of stream i for i < n; hw = {H0,W0,H1,W1,...}.
 * slot in {0,1}: submit(0) submit(1) wait(0) submit(0) ... keeps two batches in flight (uploads overlap compute).
 * Pinned frames must stay valid until skps_mpipe_wait(slot).  Frames on the device go through skps_mpipe_submit_device.
 * Asynchronous. */
SKPS_API int skps_mpipe_submit(skps_mpipe* p, int slot, const uint8_t* const* frames, const int32_t* hw, int n);
/* skps_mpipe_submit for any subset of the streams, in any order: frame i is the next frame of stream streams[i].  streams
 * [host] int32 (n), distinct ids in 0..n_streams-1, or NULL for stream i (what skps_mpipe_submit does).  Everything per
 * call stays in call order: hw, and every result of the batch (entry i of skps_mpipe_wait, the track ids, chips, pose and
 * device outputs belongs to frame i).  A stream the call does not feed is untouched: its frame count, previous frame,
 * track boxes, landmark history, ids and lost tracks stay as they are.  Duplicate or out-of-range ids fail before anything
 * is enqueued.  A batch costs what its n frames cost, whatever n_streams is. */
SKPS_API int skps_mpipe_submit_streams(skps_mpipe* p, int slot, const int32_t* streams, const uint8_t* const* frames,
                                       const int32_t* hw, int n);
/* Block until the slot's results are in host memory.  Per stream s < n: n_faces[s]; boxes (n, top_k, 4) float64 = the
 * refreshed track boxes (the 'box' entries of FaceAna.run); kps (n, top_k, n_points, 2) float64 smoothed landmarks;
 * scores (n, top_k, n_points) float32; ran_detector[s] (may be NULL) = the frame used the detector's rows (the
 * frame-difference gate's decision on a keyframe; every frame is one unless skps_mpipe_set_detect_every says otherwise). */
SKPS_API int skps_mpipe_wait(skps_mpipe* p, int slot, int32_t* n_faces, double* boxes, double* kps, float* scores,
                             int32_t* ran_detector);
/* Caller-owned [dev] result buffers of one batch, on the pipeline's device, laid out as skps_mpipe_wait /
 * skps_mpipe_align_results / skps_mpipe_pose_results fill their host buffers (n = the submit's stream count; entries
 * i >= n_faces[s] are unspecified).  chips and M are needed while alignment is on, rvec..reproject while pose is on. */
typedef struct skps_mpipe_outputs {
    int32_t* n_faces;                   /* (n)                             */
    int32_t* ran_detector;              /* (n)                             */
    double* boxes;                      /* (n, top_k, 4)                   */
    double* kps;                        /* (n, top_k, n_points, 2)         */
    float* scores;                      /* (n, top_k, n_points)            */
    uint8_t* chips;                     /* (n, top_k, size, size, 3)       */
    double* M;                          /* (n, top_k, 2, 3)                */
    double *rvec, *tvec, *euler;        /* (n, top_k, 3) each              */
    double* reproject;                  /* (n, top_k, 8, 2)                */
    int64_t* ids;                       /* (n, top_k) track ids, or NULL   */
} skps_mpipe_outputs;
/* skps_mpipe_submit for frames already on the pipeline's device: frame i HxWx3 uint8 BGR with rows pitches[i] bytes apart
 * (>= 3W, any alignment), gathered into the stream's ring and diffed against its previous frame in one launch for the
 * batch.  The frames are read after all work queued on `producer_stream` before this call, and work queued on it after this
 * call returns runs after they have been read.  out = NULL: results come back to host memory through skps_mpipe_wait as
 * for skps_mpipe_submit.  out != NULL: the batch's results are copied into *out on the device instead, and the slot is
 * completed by skps_mpipe_wait_stream.  Asynchronous. */
SKPS_API int skps_mpipe_submit_device(skps_mpipe* p, int slot, const uint8_t* const* frames, const int32_t* pitches,
                                      const int32_t* hw, int n, const skps_mpipe_outputs* out, void* producer_stream);
/* skps_mpipe_submit_device for any subset of the streams, in any order, as skps_mpipe_submit_streams: frame i is the next
 * frame of stream streams[i] (streams NULL: stream i); pitches, hw and the rows of *out are in call order. */
SKPS_API int skps_mpipe_submit_device_streams(skps_mpipe* p, int slot, const int32_t* streams, const uint8_t* const* frames,
                                              const int32_t* pitches, const int32_t* hw, int n, const skps_mpipe_outputs* out,
                                              void* producer_stream);
/* skps_mpipe_submit_device_streams for frames in any SKPS_LAYOUT_*, one layout for the whole call: pitches[i] >= xstep *
 * W_i (H_i == 1: any); plane_pitches [host] int32 (n) the plane pitch of each frame, read for the planar layouts only
 * (may be NULL otherwise).  Every frame is gathered into its stream's ring as interleaved BGR, so the gate, the detection
 * cadence, track ids and smoothing see what the BGR entry stages for the same pixels, and consecutive calls may use
 * different layouts.  skps_mpipe_submit_device_streams is this entry with BGR. */
SKPS_API int skps_mpipe_submit_device_layout(skps_mpipe* p, int slot, const int32_t* streams, const uint8_t* const* frames,
                                             const int32_t* pitches, const int32_t* hw, int n, int layout,
                                             const int32_t* plane_pitches, const skps_mpipe_outputs* out,
                                             void* producer_stream);
/* skps_mpipe_submit_device_layout for frames stored turned: frame i must be turned turns[i] [host] int32 (n, each 0..3)
 * quarter turns clockwise; hw and pitches describe it as stored.  It is gathered into its stream's ring upright, so the
 * stream sees the upright frame: a stream whose frames change between odd and even turns changes frame size (the next
 * frame is a keyframe), one that changes between 0 and 2 does not.  turns NULL: skps_mpipe_submit_device_layout. */
SKPS_API int skps_mpipe_submit_device_rotate(skps_mpipe* p, int slot, const int32_t* streams, const uint8_t* const* frames,
                                             const int32_t* pitches, const int32_t* hw, int n, int layout,
                                             const int32_t* plane_pitches, const int32_t* turns,
                                             const skps_mpipe_outputs* out, void* producer_stream);
/* Completes a slot submitted with device outputs without blocking the host: work queued on `consumer_stream` after this
 * call runs after the batch's results are in the caller's buffers.  The slot can then be submitted again. */
SKPS_API int skps_mpipe_wait_stream(skps_mpipe* p, int slot, void* consumer_stream);
/* Track ids (additive): every stream keeps an id per track box on the device.  Per call, in output order, a face whose
 * source (the track box its detection matched, or on a gate-skipped frame the track box it is) is a track box whose id no
 * earlier face of the call took inherits that id; every other face gets the stream's next number, starting at 0 after
 * skps_mpipe_reset.  After skps_mpipe_wait(slot): ids [host] (n, top_k) int64, n = that submit's stream count; entries
 * i >= n_faces[s] are undefined.  Device results get them through skps_mpipe_outputs.ids. */
SKPS_API int skps_mpipe_track_ids(skps_mpipe* p, int slot, int64_t* ids);
/* Debug/unit-test entry of the temporal step of skps_mpipe_submit (csrc/temporal.cu): GroupTrack.calculate, the track-box
 * EMA of judge_boxs and the track ids, for streams 0..n_streams-1 in one launch, with the constants skps_mpipe_submit derives
 * from cfg (its track_iou and alpha; top_k is the argument).  All other pointers [dev], laid out as skps_mpipe keeps them
 * (S >= n_streams, K = top_k in 1..64, P = n_points):
 *   inputs  kps_now (S,K,P,2) float32, count (S), flag (S) detector ran, hw (S,2) frame H, W, boxes4 (S,K,4) float32 boxes of
 *           the landmark stage, src (S,K) each face's source track box or -1; count[s] <= K;
 *   state   updated in place: prev_lm, prev_dx (S,2,K,P,2) float64, n_prev (S) (-1: none), prev_f32 (S), state_idx (S)
 *           (which half of prev_lm / prev_dx is current), track_box (S,K,4) float64, track_f32 (S,K,4), n_track (S) <= K,
 *           ids (S,K) int64, next_id (S) int64; skps_mpipe_create / skps_mpipe_reset start a stream at n_prev = -1,
 *           prev_f32 = 1, n_track = 0, ids -1, next_id = 0, state_idx 0 and every buffer zero;
 *   output  out_kps (S,K,P,2) float64 smoothed landmarks.
 * Streams >= n_streams are not touched.  Asynchronous on `stream`. */
SKPS_API int skps_debug_mp_temporal(const skps_pipeline_cfg* cfg, int n_streams, int top_k, int n_points,
                                    const float* kps_now, const int32_t* count, const int32_t* flag, const int32_t* hw,
                                    const float* boxes4, const int32_t* src, double* prev_lm, double* prev_dx,
                                    int32_t* n_prev, int32_t* prev_f32, int32_t* state_idx, double* track_box,
                                    float* track_f32, int32_t* n_track, int64_t* ids, int64_t* next_id, double* out_kps,
                                    void* stream);
/* skps_debug_mp_temporal with the id memory of skps_mpipe_set_id_memory: id_memory >= 0 frames, and the memory state [dev],
 * updated in place, laid out as skps_mpipe keeps it: mem_ids (S,K) int64 ids of the lost tracks, most recently lost first;
 * mem_box (S,K,4) float32 their boxes of the frame that last returned them; mem_gap (S,K) int32 the frames in a row each has
 * been missing so far; mem_n (S) entries held, 0 after skps_mpipe_create / skps_mpipe_reset.  With id_memory = 0 the four
 * may be NULL and the launch is skps_debug_mp_temporal's.  Asynchronous on `stream`. */
SKPS_API int skps_debug_mp_temporal_mem(const skps_pipeline_cfg* cfg, int n_streams, int top_k, int n_points,
                                        const float* kps_now, const int32_t* count, const int32_t* flag, const int32_t* hw,
                                        const float* boxes4, const int32_t* src, double* prev_lm, double* prev_dx,
                                        int32_t* n_prev, int32_t* prev_f32, int32_t* state_idx, double* track_box,
                                        float* track_f32, int32_t* n_track, int64_t* ids, int64_t* next_id, double* out_kps,
                                        int id_memory, int64_t* mem_ids, float* mem_box, int32_t* mem_gap, int32_t* mem_n,
                                        void* stream);

/* ---- Aligned face chips (csrc/align.cu; additive) -----------------------------------------------------------------------
 * What a caller does with the 98 landmarks before a recognition / attribute model: estimate the least-squares similarity
 * (rotation, uniform scale, translation; no reflection; Umeyama 1991) from landmarks [96, 97, 54, 76, 82] (pupils, nose tip,
 * mouth corners) to the ArcFace 112x112 five-point template scaled by size/112, and warp a size x size chip with it.
 * Replaces, per face on the host,
 *     M = <similarity estimate>; chip = cv2.warpAffine(frame, M, (size, size), flags=cv2.INTER_LINEAR,
 *                                                      borderMode=cv2.BORDER_CONSTANT, borderValue=0)
 * byte for byte (OpenCV's fixed-point path).  M is (2,3) float64 frame -> chip, the matrix one passes to cv2.warpAffine.
 * Chips are BGR like the frame.  size is 16..512. */

/* Batched cv2.warpAffine of one [dev] HxWx3 uint8 frame (row pitch `pitch` bytes) with n arbitrary affine matrices
 * M [dev] (n,2,3) float64 (shear included) -> out [dev] (n,out_h,out_w,3) uint8.  count [dev] or NULL: matrices i >= *count
 * are skipped (their output is left as it was).  Asynchronous on `stream`. */
SKPS_API int skps_warp_affine(const uint8_t* frame, int H, int W, int pitch, const double* M, const int32_t* count, int n,
                              int out_h, int out_w, uint8_t* out, void* stream);
/* Estimate + warp for n faces of one [dev] frame: kps [dev] (n,P,2) float64 with P >= 98 (WFLW-98 order) -> chips [dev]
 * (n,size,size,3) uint8 and M [dev] (n,2,3) float64.  count [dev] or NULL as above.  Asynchronous on `stream`. */
SKPS_API int skps_align_faces(const uint8_t* frame, int H, int W, int pitch, const double* kps, const int32_t* count, int n,
                              int P, int size, uint8_t* chips, double* M, void* stream);
/* skps_warp_affine for n faces (any n >= 0) that may each come from a different image, in one launch per 65535 faces: chip i
 * is warped from src[i] [dev] (skps_face_src, as skps_crop_faces takes it) with M [dev] (n,2,3) float64 -> out [dev]
 * (n,out_h,out_w,3) uint8, the bytes cv2.warpAffine writes on the whole image.  A tap outside the image reads 0, and so
 * does a tap inside the image but outside src[i]'s rectangle, which is never dereferenced (FaceLandmark's host frames
 * upload only core/api/align.py:chip_read_rects).  Asynchronous on `stream`; allocates nothing. */
SKPS_API int skps_warp_faces(const skps_face_src* src, const double* M, int n, int out_h, int out_w, uint8_t* out,
                             void* stream);
/* skps_warp_faces for faces of images in any SKPS_LAYOUT_*: chip i's image is laid out as lay[i] [dev] (n) says; lay NULL:
 * every image is BGR (skps_warp_faces).  The chips are BGR, the bytes of the same pixels as an interleaved BGR image. */
SKPS_API int skps_warp_faces_layout(const skps_face_src* src, const skps_frame_layout* lay, const double* M, int n, int out_h,
                                    int out_w, uint8_t* out, void* stream);
/* skps_warp_faces_layout for faces of images stored turned: chip i's image must be turned turns[i] [dev] (n) quarter turns
 * clockwise and M maps the upright image.  A turned image is read whole; one of turn 0 may be a rectangle as for
 * skps_warp_faces.  turns NULL: skps_warp_faces_layout. */
SKPS_API int skps_warp_faces_rotate(const skps_face_src* src, const skps_frame_layout* lay, const int32_t* turns,
                                    const double* M, int n, int out_h, int out_w, uint8_t* out, void* stream);
/* skps_warp_faces_layout for the kept faces of n_frames frames, with the face counts known only on the device:
 * n_frames * per_frame slots (per_frame 1..65535) are launched, and slot j of frame i, chip i*per_frame + j of
 * out [dev] (n_frames*per_frame,out_h,out_w,3) uint8, is warped with M [dev] + (i*per_frame + j)*6 only when
 * j < count[i] [dev] (n_frames) int32; the other chips are left as they were.  One source per frame: src[i] [dev] and,
 * unless NULL, lay[i] [dev] (n_frames) describe frame i for all its slots (the whole frame at any pitch and layout).
 * Asynchronous on `stream`; allocates nothing. */
SKPS_API int skps_warp_faces_count(const skps_face_src* src, const skps_frame_layout* lay, const int32_t* count,
                                   int n_frames, int per_frame, const double* M, int out_h, int out_w, uint8_t* out,
                                   void* stream);
/* skps_warp_faces_count for frames stored turned: frame i must be turned turns[i] [dev] (n_frames) quarter turns clockwise
 * and its matrices map the upright frame (FaceDetector(align=...) on turned frames).  turns NULL: skps_warp_faces_count. */
SKPS_API int skps_warp_faces_count_rotate(const skps_face_src* src, const skps_frame_layout* lay, const int32_t* turns,
                                          const int32_t* count, int n_frames, int per_frame, const double* M, int out_h,
                                          int out_w, uint8_t* out, void* stream);
/* The estimate for the detector's own five landmarks (yolov5-face columns 5..14: eyes, nose tip, mouth corners, the
 * template's order).  rows [dev] (n_frames,det_cap,16), count [dev] (n_frames) and recover [dev] (n_frames,3) float32 are
 * skps_detect_post_batch's kept_rows, count and recover with capacity det_cap.  For slot j < min(count[i], max_chips)
 * of frame i, points [dev] + (i*max_chips + j)*10 (5,2) float32 gets the five points in frame pixels, ((x - pad_x) /
 * scale, (y - pad_y) / scale) in float32 as scale_coords maps columns 0..3, and M [dev] + (i*max_chips + j)*6 (2,3)
 * float64 the similarity from those points promoted to float64 to the template scaled by size/112, the estimator of
 * skps_align_faces bit for bit.  Other slots are left as they were.  max_chips 1..det_cap, size 16..512.  One thread
 * per slot; asynchronous on `stream`; allocates nothing. */
SKPS_API int skps_det_align_estimate(const float* rows, const int32_t* count, int det_cap, const float* recover,
                                     int n_frames, int max_chips, int size, float* points, double* M, void* stream);
/* The estimate of skps_align_faces for n faces (any n >= 0) from float32 landmarks kps [dev] (n,P,2), P >= 98, each promoted
 * to float64: M [dev] (n,2,3) float64, bit for bit what skps_align_faces gives for kps.astype(float64) (and so what
 * FaceAna(align=size) returns for its float32 'kps').  size 16..512.  Asynchronous on `stream`; allocates nothing. */
SKPS_API int skps_align_estimate(const float* kps, int n, int P, int size, double* M, void* stream);
/* skps_align_faces on the frame of the last skps_pipeline_run / skps_pipeline_commit_frame (still in HBM, not uploaded
 * again) for FaceAna, whose landmarks are smoothed on the host: kps [host] (n,n_points,2) float64, chips [host]
 * (n,size,size,3) uint8, M [host] (n,2,3) float64.  n <= top_k.  Synchronous. */
SKPS_API int skps_pipeline_align(skps_pipeline* p, const double* kps, int n, int size, uint8_t* chips, double* M, void* stream);
/* FaceAnaStreams: size > 0 makes every following skps_mpipe_submit warp one chip per returned face, from the smoothed
 * float64 landmarks of the temporal layer and the frame in the stream's ring, on the compute stream without a host
 * synchronisation; chips and matrices are copied back with the slot's other results.  size 0 switches it off and frees the
 * buffers (n_streams x top_k x size^2 x 3 bytes on the device and twice that pinned on the host); an allocation failure is
 * reported through skps_last_error.  No batch may be in flight. */
SKPS_API int skps_mpipe_set_align(skps_mpipe* p, int size);
/* After skps_mpipe_wait(slot), for a slot submitted with alignment on: chips [host] (n, top_k, size, size, 3) uint8 and
 * M [host] (n, top_k, 2, 3) float64, n = that submit's stream count; entries i >= n_faces[s] are undefined. */
SKPS_API int skps_mpipe_align_results(skps_mpipe* p, int slot, uint8_t* chips, double* M);

/* ---- Head pose of every face (csrc/headpose.cu; additive) ---------------------------------------------------------------
 * get_head_pose of the training tree (TRAIN/face_landmark/lib/dataset/headpose.py:48-78) on the 98 WFLW landmarks: the 10
 * landmarks [33, 37, 42, 46, 60, 64, 68, 72, 55, 59], rounded to float32, paired with the model points of pose.py, the
 * camera [[W,0,W//2],[0,W,H//2],[0,0,1]] of the face's frame; the same solver as skps_head_pose, one warp per face.
 * Outputs float64: rvec, tvec, euler (degrees, in the order cv2.decomposeProjectionMatrix returns) (3,) and the 8
 * re-projected cube corners (8,2) per face; Euler angles as described at skps_head_pose. */
/* FaceAna, whose landmarks are smoothed on the host: kps [host] (n,n_points,2) float64, H x W the frame they belong to;
 * rvec, tvec, euler [host] (n,3), reproject [host] (n,8,2).  n <= top_k.  Buffers are allocated on the first call; the work
 * is ordered on `stream`, and the call returns once that stream has reached it.  Synchronous. */
SKPS_API int skps_pipeline_pose(skps_pipeline* p, const double* kps, int n, int H, int W, double* rvec, double* tvec,
                                double* euler, double* reproject, void* stream);
/* FaceAnaImages, whose faces come from many images: kps [dev] (n_faces,n_points,2) float32 (n_points >= 98), hw [dev]
 * (n_faces,2) int32 the H, W of each face's own image; rvec, tvec, euler [dev] (n_faces,3), reproject [dev]
 * (n_faces,8,2).  The same results as skps_pipeline_pose on the same landmarks promoted to float64.  Asynchronous on
 * `stream`; allocates nothing. */
SKPS_API int skps_head_pose_faces(const float* kps, int n_faces, int n_points, const int32_t* hw, double* rvec,
                                  double* tvec, double* euler, double* reproject, void* stream);
/* FaceAnaStreams: on != 0 makes every following skps_mpipe_submit solve the pose of every returned face from the smoothed
 * float64 landmarks, with each stream's own frame size, on the compute stream without a host synchronisation; the results
 * are copied back with the slot's other results.  on = 0 switches it off and frees the buffers (n_streams x top_k x 200
 * bytes on the device and twice that pinned on the host).  No batch may be in flight. */
SKPS_API int skps_mpipe_set_pose(skps_mpipe* p, int on);
/* After skps_mpipe_wait(slot), for a slot submitted with pose on: rvec, tvec, euler [host] (n, top_k, 3) and reproject
 * [host] (n, top_k, 8, 2) float64, n = that submit's stream count; entries i >= n_faces[s] are undefined. */
SKPS_API int skps_mpipe_pose_results(skps_mpipe* p, int slot, double* rvec, double* tvec, double* euler, double* reproject);

/* ---- Detection cadence (csrc/mpipe.cu; additive) -----------------------------------------------------------------------
 * Each stream counts its frames from skps_mpipe_create / skps_mpipe_reset: i = 0, 1, 2, ..., advanced only by submits that
 * include a frame for it.  With every = N, stream s's frame i is a keyframe when the stream has no previous frame of this
 * frame's size, or when (i + s % N) % N == 0; only keyframes are letterboxed, run through the detector and NMS (packed, in
 * stream order, as one batch of m frames), and a keyframe's rows are used when the frame-difference gate fires or there is
 * no previous frame of its size.  Every other frame takes the tracker path on the track boxes.  every = 1 (the default):
 * every frame is a keyframe, as without this call.  Takes effect from the next submit; the frame counters keep running. */
SKPS_API int skps_mpipe_set_detect_every(skps_mpipe* p, int every);
/* The number of frames the detector ran on in the slot's last submitted batch (0..n; 0 skips the detector). */
SKPS_API int skps_mpipe_detector_frames(const skps_mpipe* p, int slot, int* m);

/* ---- Id memory (csrc/temporal.cu; additive) ------------------------------------------------------------------------------
 * FaceAna(track_ids=True, id_memory=frames) for every stream.  A track box returned at a stream's frame a whose id no face of
 * its frame a + 1 carries is lost: the stream remembers its id and float32 box, most recently lost first, tracks lost at the
 * same frame in return order, at most top_k (about 28 bytes each, allocated by skps_mpipe_create).  A face that would get the
 * stream's next number first takes back the id of the first remembered track that it overlaps with IoU > track_iou (its
 * float32 landmark-stage box against the remembered one) and that has been missing for at most `frames` frames in a row; the
 * entry is then forgotten.  When more than top_k are held, the oldest go first.  A stream's frames are those of the submits
 * that include it.  frames = 0 (the default) remembers nothing; switching to 0 forgets every stream's lost tracks.
 * skps_mpipe_reset forgets the stream's.  May be called at any time; takes effect from the next submit. */
SKPS_API int skps_mpipe_set_id_memory(skps_mpipe* p, int frames);

#ifdef __cplusplus
}
#endif
#endif /* SKPS_B200_H */
