/* k210_yolo_b200 — C-ABI of the H100-native YOLOv3 inference hot path.
 *
 * Drop-in boundary for the path  keras_inference.py:main -> network(...) -> predict ->
 * decode -> per-class NMS  of zhen8838/K210_Yolo_framework.  Every entry point names the
 * reference interface it replaces (paths under /root/reference).  Plain pointers and sizes
 * only; device pointers come from the caller (e.g. torch.Tensor.data_ptr()), streams are
 * cudaStream_t passed as void*.  All functions return K2Y_OK (0) or a negative error code;
 * k2y_last_error() gives the message.  There is NO CPU fallback: calls that need a GPU fail
 * with K2Y_ERR_CUDA when none is present.
 */
#ifndef K210_YOLO_B200_H
#define K210_YOLO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define K2Y_OK 0
#define K2Y_ERR_INVALID (-1)   /* bad argument / unknown name / shape mismatch */
#define K2Y_ERR_CUDA (-2)      /* CUDA runtime or driver error (incl. no device) */
#define K2Y_ERR_STATE (-3)     /* call order violated (e.g. run before finalize/bind) */
#define K2Y_ERR_NOMEM (-4)

/* Arithmetic of the dense (1x1 / 3x3) convolutions. */
#define K2Y_MATH_FP32_SIMT 0   /* fp32 FFMA on CUDA cores (exact-order reference path on the GPU) */
#define K2Y_MATH_TC_3XTF32 1   /* wgmma tf32, hi/lo split x3 (fp32-class accuracy) */
#define K2Y_MATH_TC_TF32 2     /* wgmma tf32, single pass */
#define K2Y_MATH_TC_BF16X3 3   /* wgmma bf16: fp32 operands split into (hi, mid) bf16 planes, 3 MMAs (~16-bit mantissa) */

const char *k2y_last_error(void);
int k2y_version(void);
/* 1 if a CUDA device is usable, 0 otherwise (never fails). */
int k2y_cuda_available(void);

/* ------------------------------------------------------------------------------------------
 * Network = the reference's model-builder "plugin" API
 *   network(input_shape=[H,W,3], anchor_num, class_num, alpha=) -> (yolo_model, yolo_model_warpper)
 *   models/yolonet.py:12 (yolo_mobilev1), :49 (yolo_mobilev2), :107 (tiny_yolo), :161 (yolo)
 * and the two methods keras_inference.py uses on it: load_weights (:80) and predict (:88).
 * ---------------------------------------------------------------------------------------- */
typedef struct k2y_net k2y_net;

/* Builds the layer graph (native graph builder).  model_def is one of the four reference
 * builder names.  Output grids are derived from the input size (H/32, H/16[, H/8]) rather than
 * the reference's hard-coded Reshape targets (yolonet.py:40-41,98-99,140-141,175-177). */
int k2y_net_create(const char *model_def, int in_h, int in_w, float alpha, int anchor_num, int class_num,
                   int max_batch, int device, k2y_net **out);
int k2y_net_destroy(k2y_net *net);

/* Weighted layers, in creation order (== Keras auto-naming order). */
typedef struct {
    char name[64];     /* Keras layer name of the conv ("conv_pw_3", "conv2d_1", ...) */
    char bn_name[64];  /* Keras name of the BatchNormalization folded behind it, "" if none */
    int32_t kind;      /* 0 dense conv, 1 depthwise conv */
    int32_t kh, kw, cin, cout, stride;
    int32_t has_bias;
} k2y_layer_info;
int k2y_net_num_layers(const k2y_net *net, int *n);
int k2y_net_layer_info(const k2y_net *net, int i, k2y_layer_info *info);

/* load_weights (keras_inference.py:80): one call per Keras variable.  layer is the Keras layer
 * name as stored in the HDF5 file, var one of kernel | depthwise_kernel | bias | gamma | beta |
 * moving_mean | moving_variance; data is host float32 in the Keras layout (HWIO kernels,
 * depthwise (3,3,C,1)); dims/ndim are checked against the graph.  Unknown layer -> K2Y_ERR_INVALID. */
int k2y_net_set_weight(k2y_net *net, const char *layer, const char *var, const float *data,
                       const int64_t *dims, int ndim);
/* Folds BatchNormalization (eps 1e-3) into per-channel scale/shift, packs and uploads.  Fails with
 * K2Y_ERR_STATE naming the first variable that was never set. */
int k2y_net_finalize(k2y_net *net);

int k2y_net_set_math(k2y_net *net, int math_mode);
int k2y_net_get_math(const k2y_net *net, int *math_mode);
/* 1 (default) = replay the layer schedule as one CUDA graph per batch size; 0 = plain launches. */
int k2y_net_set_use_graph(k2y_net *net, int use_graph);

int k2y_net_num_outputs(const k2y_net *net, int *n);
/* Per-image shape of head l of the plain yolo_model: [h, w, anchor_num*(5+class_num)]. */
int k2y_net_output_shape(const k2y_net *net, int l, int *h, int *w, int *c);
/* Bytes of activation arena needed for max_batch images. */
int k2y_net_workspace_bytes(const k2y_net *net, size_t *bytes);
/* Binds caller-owned device storage: workspace (>= workspace_bytes, 256-B aligned), the input
 * x [max_batch,H,W,3] f32 NHWC and one buffer per head [max_batch,h,w,c] f32 NHWC. */
int k2y_net_bind(k2y_net *net, void *workspace, size_t workspace_bytes, const float *x_dev,
                 float *const *heads_dev, int n_heads);
/* Optional uint8 front end (the reference's `img / np.max(img)`, tools/utils.py:405, done on the GPU): x_u8_dev is
 * [max_batch,H,W,3] uint8 letterboxed RGB, img_max_dev a scratch int32[max_batch].  Each run first reduces the per-image
 * maximum, and the first convolution reads x = u8 / max through a 256-entry table (bit-identical to the float32 input the
 * reference feeds).  Pass NULL, NULL to return to the float32 input bound with k2y_net_bind. */
int k2y_net_bind_u8(k2y_net *net, const unsigned char *x_u8_dev, int32_t *img_max_dev);
/* Re-points the float32 input at another device buffer [max_batch,H,W,3] (workspace and heads stay as bound).  One CUDA
 * graph is kept per (batch, input buffer), so alternating between two input buffers (H2D of batch i+1 while batch i runs)
 * costs nothing after the first use of each.  k2y_net_bind_u8 behaves the same way for the uint8 input. */
int k2y_net_bind_input(k2y_net *net, const float *x_dev);
/* SM budget of this net's persistent tensor-core kernels (tile planner + grid sizes); 0 (default) = the whole device.  Nets
 * that run concurrently on one GPU (several batches in flight on separate streams) should each take their share — 132 / 2 on
 * an H100 with two in flight — so that their one-CTA-per-SM grids run side by side instead of queueing behind each other.
 * Results do not depend on it bit for bit only where the tile shapes stay the same; they stay within the conv tolerance. */
int k2y_net_set_sm_limit(k2y_net *net, int sms);
/* Re-points the head outputs at another set of device buffers (same shapes as in k2y_net_bind).  One CUDA graph is kept per
 * (batch, input buffer, first head buffer): alternating between two head sets lets the decode/NMS of batch i (reading set A on
 * another stream) overlap the convolutions of batch i+1 (writing set B) at no re-capture cost. */
int k2y_net_bind_heads(k2y_net *net, float *const *heads_dev, int n_heads);
/* predict on bound device buffers (keras_inference.py:88), asynchronous on `stream`. */
int k2y_net_run(k2y_net *net, int batch, void *stream);
/* predict with HOST buffers: H2D of x, run, D2H of every head, stream-synchronised on return.
 * x_host [batch,H,W,3] f32; heads_host[l] [batch,h_l,w_l,c] f32. */
int k2y_net_predict_host(k2y_net *net, const float *x_host, int batch, float *const *heads_host, void *stream);
/* Kernel launches (graph nodes) one k2y_net_run(batch) issues. */
int k2y_net_launches_per_run(const k2y_net *net, int *n);
/* Measurement hooks (bench.py): one plain (non-graph) pass with a CUDA event between consecutive launches on
 * `stream`; ms_per_launch[i] = device time of schedule entry i (n >= schedule_len).  launch_info names launch i
 * (Keras layer name) and gives its algorithmic work per image: 2*MACs and fp32 activation bytes in+out. */
int k2y_net_schedule_len(const k2y_net *net, int *n); /* layers in the schedule (a split-K layer is 2 kernels) */
int k2y_net_profile(k2y_net *net, int batch, void *stream, float *ms_per_launch, int n);
int k2y_net_launch_info(const k2y_net *net, int i, char *name, int name_len, double *flops_per_image,
                        double *bytes_per_image);
/* Debug/parity hook: copies the (post-activation) output of the conv layer `name` for the last run
 * into host memory as [batch,h,w,c] f32.  Only valid with use_graph == 0 and keep_all (below). */
int k2y_net_set_keep_all(k2y_net *net, int keep_all);
int k2y_net_read_layer(k2y_net *net, const char *name, int batch, float *host, size_t host_floats, int *h,
                       int *w, int *c);

/* Kernel-parity hook: ONE dense convolution (the op DarknetConv2D / Conv2D lower to) on device NHWC f32 tensors,
 * synchronous.  kernel_host is Keras HWIO [k,k,c0+c1,cout]; y = act(conv(x) * scale + shift) (+ residual).
 * The input is concat(src0 [optionally nearest-upsampled x2, stored at h/2 x w/2], src1).  pad_mode: 0 = SAME
 * (stride 1), 1 = ZeroPadding2D((1,1),(1,1)) + VALID, 2 = ZeroPadding2D((1,0),(1,0)) + VALID.  act: 0 none,
 * 1 leaky(alpha), 2 relu, 3 relu6. */
int k2y_conv2d(const float *src0_dev, const float *src1_dev, const float *residual_dev, float *dst_dev,
               const float *kernel_host, const float *scale_host, const float *shift_host, int batch, int h, int w,
               int c0, int c1, int up0, int cout, int ksize, int stride, int pad_mode, int act, float alpha,
               int math_mode, void *stream);

/* ------------------------------------------------------------------------------------------
 * KERAS-dialect decode + per-class NMS  (keras_inference.py:94-135; tools/utils.py:524-547
 * tf_xywh_to_all; keras_inference.py:32-72 correct_box; tf.image.non_max_suppression).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    float ymin, xmin, ymax, xmax; /* pixels of the ORIGINAL image, as correct_box returns */
    float score;                  /* sigmoid(cls) * sigmoid(conf) */
    int32_t index;                /* flat box index: off_l + (row*W_l + col)*A + a, layer 0 first */
} k2y_det;

typedef struct {
    int32_t n_layers;          /* <= 3 */
    int32_t layer_h[3], layer_w[3];
    int32_t anchor_num, class_num;
    float anchors[3 * 8 * 2];  /* [layer][anchor][(w,h)] fraction of the net input (Helper.anchors) */
    int32_t in_h, in_w;        /* network input size (image_size) */
    float obj_thresh;          /* candidate iff score >= obj_thresh */
    float iou_thresh;          /* suppressed iff IoU > iou_thresh */
    int32_t max_per_class;     /* tf.image.non_max_suppression max_output_size (30) */
} k2y_detect_cfg;

/* Scratch bytes k2y_detect_keras needs for `batch` images. */
int k2y_detect_workspace_bytes(const k2y_detect_cfg *cfg, int batch, size_t *bytes);
/* heads_dev[l]: [batch,h_l,w_l,A*(5+C)] f32 NHWC device tensors.  image_hw_dev: [batch,2] f32
 * (orig_h, orig_w) on device.  Outputs (device): dets [batch][C][max_per_class], counts [batch][C].
 * Records of one class are in descending score (ties: ascending index). */
int k2y_detect_keras(const k2y_detect_cfg *cfg, const float *const *heads_dev, int batch,
                     const float *image_hw_dev, k2y_det *dets_dev, int32_t *counts_dev, void *workspace,
                     size_t workspace_bytes, void *stream);

/* Same, with explicit per-image strides (in 32-bit words) of the two outputs, so that one image's records and counts can
 * sit next to each other in a gather block: dets of image b start at (int32*)dets_dev + b*det_image_stride_words, counts at
 * counts_dev + b*count_image_stride_words.  k2y_detect_keras == strides (C*max_per_class*6, C). */
int k2y_detect_keras_strided(const k2y_detect_cfg *cfg, const float *const *heads_dev, int batch,
                             const float *image_hw_dev, k2y_det *dets_dev, int32_t *counts_dev,
                             long long det_image_stride_words, long long count_image_stride_words, void *workspace,
                             size_t workspace_bytes, void *stream);

/* Merge of views (tiled detection): an image was detected as `views` views - view 0 the whole image, the others windows of
 * it, each letterboxed and decoded as an image of its own (k2y_letterbox_u8_views) - and this call turns their record lists
 * into one list per (image, class) in image coordinates.
 *   view_dets_dev / view_counts_dev: [n_images * views][C][max_per_class] records and [n_images * views][C] counts, dense,
 *   image-major, as k2y_detect_keras writes them for n_images * views inputs.  view_yx_dev: [n_images * views][2] float32
 *   (y0, x0), each view's origin in its image (k2y_letterbox_u8_views writes it).
 * Per image and class: every record of every view v gets (y0, x0, y0, x0) added to (ymin, xmin, ymax, xmax) (one float32
 * round-to-nearest add each, no clipping) and index = v * n_boxes + index (n_boxes: the boxes of one network input, so
 * index / n_boxes tells the view and view 0 keeps its indices); the union is ordered by score descending, then view, then
 * index ascending, and goes through the greedy NMS of k2y_detect_keras (suppressed iff IoU > iou_thresh, a zero-area box
 * has IoU 0) until max_per_class are kept.  Outputs as k2y_detect_keras_strided's, for `rows` >= n_images images: rows past
 * n_images get count 0.  One launch, asynchronous on `stream`, no scratch memory.
 * K2Y_ERR_INVALID (nothing launched) when views * max_per_class exceeds k2y_merge_views_max_records() (1024: VOC's 30 per
 * class takes 34 views, COCO's 100 takes 10) or views * n_boxes exceeds INT32_MAX.  It is k2y_merge_views_ex with uniform
 * ranges and the default options (below). */
int k2y_merge_views_max_records(void);
int k2y_merge_views(const k2y_det *view_dets_dev, const int32_t *view_counts_dev, const float *view_yx_dev, int n_images, int rows,
                    int views, int n_boxes, int class_num, int max_per_class, float iou_thresh, k2y_det *dets_dev,
                    int32_t *counts_dev, long long det_image_stride_words, long long count_image_stride_words, void *stream);

/* k2y_merge_views with a number of views per image and the options of tiling by tile size (oracle/tiles_merge_ref.py states
 * each one; k2y_merge_views is this call with null offsets and sides, K2Y_MATCH_IOU and K2Y_MERGE_SUPPRESS):
 *   view_offsets_dev  int32 [n_images + 1] on the device: image b owns the views view_offsets[b] .. view_offsets[b+1] - 1 of
 *                     the per-view blocks, at most max_views of them; view numbers (index = view * n_boxes + index) stay per
 *                     image.  NULL: image b owns views b * max_views .. b * max_views + max_views - 1.
 *   view_sides_dev    int32 [N] on the device, each view's interior sides (1 top, 2 left, 4 bottom, 8 right: that edge of
 *                     the window is inside its image; the whole image has none).  With it, a record is dropped before the
 *                     merge when, in window coordinates, fminf / fmaxf of its y (x) fields is < border at a top (left)
 *                     interior side or > fl(th - border) (fl(tw - border)) at a bottom (right) one; th, tw from view_hw_dev
 *                     ([N][2] float32, as k2y_letterbox_u8_views writes them) and border >= 0.  NULL: no record is dropped.
 *   match             K2Y_MATCH_IOU (IoU > thresh) or K2Y_MATCH_IOS (intersection over the smaller area > thresh, float32,
 *                     0 for a box of area <= 0).
 *   merge             K2Y_MERGE_SUPPRESS (a record that matches a kept one is dropped) or K2Y_MERGE_UNION (the kept record's
 *                     box becomes the field-wise min / max of itself and the records it suppressed; -0.0 below +0.0, NaN
 *                     fields take no part).
 * The same launch shape, limits (max_views * max_per_class <= k2y_merge_views_max_records()) and outputs as k2y_merge_views;
 * no scratch memory. */
#define K2Y_MATCH_IOU 0
#define K2Y_MATCH_IOS 1
#define K2Y_MERGE_SUPPRESS 0
#define K2Y_MERGE_UNION 1
int k2y_merge_views_ex(const k2y_det *view_dets_dev, const int32_t *view_counts_dev, const float *view_yx_dev,
                       const int32_t *view_offsets_dev, const int32_t *view_sides_dev, const float *view_hw_dev, float border,
                       int match, int merge, int n_images, int rows, int max_views, int n_boxes, int class_num, int max_per_class,
                       float thresh, k2y_det *dets_dev, int32_t *counts_dev, long long det_image_stride_words,
                       long long count_image_stride_words, void *stream);
/* k2y_merge_views_ex with mirrored views (test-time flip; k2y_merge_views_ex is this call with a null view_mirror_dev):
 *   view_mirror_dev   int32 [N] on the device, nonzero for a view that is its window flipped left to right
 *                     (k2y_letterbox_u8_views_mirror), whose records are in mirrored window coordinates.  Each such record is
 *                     mapped back while it is loaded: xmin = fl(fl(tw - xmax) + x0), xmax = fl(fl(tw - xmin) + x0), y fields
 *                     shifted as for any view (a NaN result is the canonical NaN); index = view * n_boxes + index as for any
 *                     view.  The border drop tests the record in the mirrored coordinates it comes in, with the window's
 *                     left and right side bits (2 and 8, as view_sides_dev gives them for the window) swapped.  Needs
 *                     view_hw_dev (tw), with or without a border drop.  NULL: no view is mirrored. */
int k2y_merge_views_mirror(const k2y_det *view_dets_dev, const int32_t *view_counts_dev, const float *view_yx_dev,
                           const int32_t *view_offsets_dev, const int32_t *view_sides_dev, const int32_t *view_mirror_dev,
                           const float *view_hw_dev, float border, int match, int merge, int n_images, int rows, int max_views,
                           int n_boxes, int class_num, int max_per_class, float thresh, k2y_det *dets_dev, int32_t *counts_dev,
                           long long det_image_stride_words, long long count_image_stride_words, void *stream);

/* SORT tracking (oracle/sort_ref.py states every rule, and this call follows it bit for bit): per class, a Kalman filter per
 * track, IoU association by scipy's optimal assignment, SORT's birth, reporting and death, ids from one counter per stream.
 *   state_dev       k2y_track_state_bytes() bytes on the device, zeroed to start a stream; the tracks, the frame count, the
 *                   last position and the ids taken carry over from one call to the next, so calls of one stream must be
 *                   ordered (one stream, or events).
 *   dets_dev, counts_dev  a gathered record block: row r's records of class c at dets_dev + r * row_stride_words words
 *                   (k2y_det, max_per_class per class), its counts at counts_dev + r * row_stride_words + c.
 *   rows_dev        int32 [n_frames]: the block row of each frame, frames in stream order.
 *   positions_dev   int64 [n_frames]: each frame's position in the stream, increasing (the caller checks it).  A jump of g > 1
 *                   runs g - 1 updates without detections first.
 *   ids_out_dev     int32 [n_frames, class_num, max_per_class]: each record's track id, -1 when it has none reported.
 *   boxes_out_dev   float32 [n_frames, class_num, max_per_class, 4]: for a record with an id, its track's post-update state
 *                   box (ymin, xmin, ymax, xmax); zeros elsewhere.
 * One launch of one CTA per call, whatever n_frames, asynchronous on `stream`.  K2Y_ERR_INVALID (nothing launched) for
 * class_num outside 1..1024, max_age < 0, min_hits < 0, iou_thresh outside [0, 1], or max_per_class * (max_age + 1) over the
 * 1024 tracks one class holds. */
int k2y_track_state_bytes(int class_num, int max_per_class, int max_age, size_t *bytes);
int k2y_track_update(void *state_dev, const k2y_det *dets_dev, const int32_t *counts_dev, long long row_stride_words,
                     const int32_t *rows_dev, const long long *positions_dev, int n_frames, int class_num, int max_per_class,
                     int max_age, int min_hits, double iou_thresh, int32_t *ids_out_dev, float *boxes_out_dev, void *stream);

/* ByteTrack tracking (oracle/bytetrack_ref.py states every rule, and this call follows it bit for bit): per class, a Kalman
 * filter per track, a first association of the tracks with the high-score records (score > track_thresh), a second of the
 * tracks left with the low-score records (0.1 < score < track_thresh, the score in word 4 of each record), births from the
 * high-score records left with score >= track_thresh + 0.1, tracks kept lost for track_buffer frames, ids from one counter
 * per stream.  state_dev (k2y_bytetrack_state_bytes() bytes, zeroed to start a stream), the gathered block, rows_dev,
 * positions_dev, ids_out_dev and boxes_out_dev are as for k2y_track_update; a record gets an id when its track ends the
 * frame tracked and activated.  fuse_score nonzero multiplies the IoU by the record's score in the high-score associations.
 * One launch of one CTA per call, whatever n_frames, asynchronous on `stream`.  K2Y_ERR_INVALID (nothing launched) for
 * class_num outside 1..1024, track_buffer < 0, track_thresh or match_thresh outside [0, 1], or max_per_class *
 * (max(track_buffer, 1) + 2) over the 4096 tracks one class holds. */
int k2y_bytetrack_state_bytes(int class_num, int max_per_class, int track_buffer, size_t *bytes);
int k2y_bytetrack_update(void *state_dev, const k2y_det *dets_dev, const int32_t *counts_dev, long long row_stride_words,
                         const int32_t *rows_dev, const long long *positions_dev, int n_frames, int class_num, int max_per_class,
                         double track_thresh, double match_thresh, int track_buffer, int fuse_score, int32_t *ids_out_dev,
                         float *boxes_out_dev, void *stream);

/* OC-SORT tracking (oracle/ocsort_ref.py states every rule, and this call follows it bit for bit): per class, SORT's Kalman
 * filter per track with OC-SORT's re-update along a virtual path when a lost track is found again (ORU), a first association
 * of the tracks with the records scored above det_thresh by IoU plus the direction term weighted by inertia (OCM, over the
 * observation delta_t frames back), with use_byte a second of the tracks left with the records scored in (0.1, det_thresh),
 * a third of the records and tracks left by the tracks' last observations (OCR), births from the high-score records left,
 * tracks removed after max_age frames unmatched and reported after min_hits matched frames in a row (or in the stream's
 * first min_hits frames), ids from one counter per stream.  state_dev (k2y_ocsort_state_bytes() bytes, zeroed to start a
 * stream), the gathered block (score in word 4 of each record), rows_dev, positions_dev, ids_out_dev and boxes_out_dev are as
 * for k2y_track_update; a record's box is its own when its track reports it.  One launch of one CTA per call, whatever
 * n_frames, asynchronous on `stream`.  K2Y_ERR_INVALID (nothing launched) for class_num outside 1..1024, max_age or min_hits
 * < 0, delta_t outside 1..8, det_thresh, iou_thresh or inertia outside [0, 1], or max_per_class * (max_age + 1) over the
 * 4096 tracks one class holds. */
int k2y_ocsort_state_bytes(int class_num, int max_per_class, int max_age, int delta_t, size_t *bytes);
int k2y_ocsort_update(void *state_dev, const k2y_det *dets_dev, const int32_t *counts_dev, long long row_stride_words,
                      const int32_t *rows_dev, const long long *positions_dev, int n_frames, int class_num, int max_per_class,
                      double det_thresh, int max_age, int min_hits, double iou_thresh, int delta_t, double inertia, int use_byte,
                      int32_t *ids_out_dev, float *boxes_out_dev, void *stream);

/* Many streams in one launch: k2y_track_update, k2y_bytetrack_update and k2y_ocsort_update over n_streams independent
 * streams, with one CTA per stream.
 *   state_dev       n_streams consecutive states, state_stride bytes apart: the tracker's k2y_*_state_bytes(), a multiple of
 *                   256 (any stride >= it that is a multiple of 256 is taken).  Each is zeroed to start its stream.
 *   streams_dev     int32 [n_frames]: each frame's stream, or null when every frame is stream 0.  A batch may mix the streams'
 *                   frames in any order and lack any of them.  Each stream runs its own frames in batch order, with its own
 *                   frame count, gaps and ids from 1, exactly as the single-stream call runs them.  A stream with no frame
 *                   in the batch keeps its state as it is, so its next position counts the frames between as a gap.
 *                   Frames whose stream lies outside [0, n_streams) get cleared outputs (id -1, box 0) and touch no state;
 *                   callers should refuse them first.
 * Positions must increase along each stream; the streams are independent of one another.  The other arguments are as for
 * the single-stream calls, which are these calls with n_streams 1 and a null streams_dev.  One launch of n_streams CTAs per
 * call, asynchronous on `stream`.  K2Y_ERR_INVALID (nothing launched) also for n_streams < 1, or, with several streams, a
 * state_stride below one stream's state bytes or not a multiple of 256. */
int k2y_track_update_streams(void *state_dev, int n_streams, size_t state_stride, const k2y_det *dets_dev,
                             const int32_t *counts_dev, long long row_stride_words, const int32_t *rows_dev,
                             const long long *positions_dev, const int32_t *streams_dev, int n_frames, int class_num,
                             int max_per_class, int max_age, int min_hits, double iou_thresh, int32_t *ids_out_dev,
                             float *boxes_out_dev, void *stream);
int k2y_bytetrack_update_streams(void *state_dev, int n_streams, size_t state_stride, const k2y_det *dets_dev,
                                 const int32_t *counts_dev, long long row_stride_words, const int32_t *rows_dev,
                                 const long long *positions_dev, const int32_t *streams_dev, int n_frames, int class_num,
                                 int max_per_class, double track_thresh, double match_thresh, int track_buffer, int fuse_score,
                                 int32_t *ids_out_dev, float *boxes_out_dev, void *stream);
int k2y_ocsort_update_streams(void *state_dev, int n_streams, size_t state_stride, const k2y_det *dets_dev,
                              const int32_t *counts_dev, long long row_stride_words, const int32_t *rows_dev,
                              const long long *positions_dev, const int32_t *streams_dev, int n_frames, int class_num,
                              int max_per_class, double det_thresh, int max_age, int min_hits, double iou_thresh, int delta_t,
                              double inertia, int use_byte, int32_t *ids_out_dev, float *boxes_out_dev, void *stream);

/* ------------------------------------------------------------------------------------------
 * Multi-GPU collation: images shard across ranks (one process per GPU), and the one exchange on the path
 * is ONE ncclAllGather of the fixed-size record blocks.  The reference is single-process (keras_inference.py:12-17), so
 * this replaces nothing there — it is what makes `main()` scale over the 8 GPUs of a box.
 *   k2y_comm_unique_id   rank 0: 128 bytes to hand to every rank (any transport)
 *   k2y_comm_create      every rank: joins the communicator on `device`
 *   k2y_allgather_detections  gather_dev = [world][bytes_per_rank]; this rank's block (filled by k2y_detect_keras_strided)
 *                        lives at rank*bytes_per_rank; in place, asynchronous on `stream`; no-op for world == 1.
 * NCCL is bound at run time (libnccl.so.2, or $K2Y_NCCL_LIB); K2Y_ERR_STATE if it cannot be found.
 * ---------------------------------------------------------------------------------------- */
typedef struct k2y_comm k2y_comm;
int k2y_comm_unique_id(unsigned char *id128);
int k2y_comm_create(const unsigned char *id128, int world, int rank, int device, k2y_comm **out);
int k2y_comm_destroy(k2y_comm *comm);
int k2y_comm_info(const k2y_comm *comm, int *world, int *rank, int *nccl_version);
int k2y_allgather_detections(k2y_comm *comm, void *gather_dev, size_t bytes_per_rank, void *stream);

/* ------------------------------------------------------------------------------------------
 * REGION_C-dialect decode + NMS, batched on device  (region_layer.c:121-283 per layer).
 * in_dev: [batch][A][5+C][H][W] f32 planar.  Outputs (device): probs [batch][N][C+1] after NMS,
 * boxes [batch][N][4] (x,y,w,h centre form, letterbox-corrected), N = A*H*W, index = a*H*W+row*W+col.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int32_t layer_w, layer_h, anchor_num, classes;
    int32_t net_w, net_h, image_w, image_h;
    float anchors[8 * 2];
    float threshold, nms_value;
} k2y_region_cfg;
int k2y_region_workspace_bytes(const k2y_region_cfg *cfg, int batch, size_t *bytes);
int k2y_region_run(const k2y_region_cfg *cfg, const float *in_dev, int batch, float *out_dev /* activations, may be NULL */,
                   float *probs_dev, float *boxes_dev, void *workspace, size_t workspace_bytes, void *stream);

/* Diagnostics: the tile planner of the tensor-core conv kernel for a GEMM of M x K x N (ksize 1 or 3; K = ksize^2 * Cin).
 * Host-only (assumes an H100 SXM when no device is initialised): tile width, split-K factor, pipeline stages, CTA-pair mode (always 1)
 * and the arithmetic mode the layer really runs in. */
int k2y_tc_plan(int M, int N, int K, int ksize, int math_mode, int *bn, int *k_splits, int *stages, int *cluster,
                int *effective_math);
/* The same under an SM budget (k2y_net_set_sm_limit; 0 = whole device); also reports the persistent grid size (CTAs). */
int k2y_tc_plan_budget(int M, int N, int K, int ksize, int math_mode, int sm_limit, int *bn, int *k_splits, int *stages,
                       int *cluster, int *effective_math, int *grid);

/* ------------------------------------------------------------------------------------------
 * Operator-level pieces of the reference's decode loop, for callers that keep keras_inference.py:94-135 and swap one
 * operator at a time (device pointers; same arithmetic as k2y_detect_keras):
 *   k2y_xywh_to_all  = tf_xywh_to_all (tools/utils.py:524-547): pred_xy / pred_wh [..][h][w][A][2] contiguous ->
 *                      xy = (sigmoid(t) + (col,row)) / (w,h), wh = exp(t) * anchor[a]   (anchors_wh_host: A (w,h) pairs)
 *   k2y_correct_box  = correct_box (keras_inference.py:32-72): -> boxes [n][4] (ymin,xmin,ymax,xmax) in image pixels
 *   k2y_nms_boxes    = tf.image.non_max_suppression(boxes [n][4] yxyx, scores [n], max_output_size, iou_threshold)
 *                      (keras_inference.py:125-126): greedy, score-descending (ties: lower index first), suppress iff
 *                      IoU > threshold; writes <= max_output_size int32 indices in selection order and their count.
 *                      boxes_dev must be 16-byte aligned; workspace from k2y_nms_workspace_bytes.
 * ---------------------------------------------------------------------------------------- */
int k2y_xywh_to_all(const float *pred_xy_dev, const float *pred_wh_dev, long long n_boxes, int layer_h, int layer_w,
                    int anchor_num, const float *anchors_wh_host, float *xy_dev, float *wh_dev, void *stream);
int k2y_correct_box(const float *xy_dev, const float *wh_dev, long long n_boxes, float in_h, float in_w, float image_h,
                    float image_w, float *boxes_dev, void *stream);
int k2y_nms_workspace_bytes(int n_boxes, int max_output_size, size_t *bytes);
int k2y_nms_boxes(const float *boxes_dev, const float *scores_dev, int n_boxes, int max_output_size, float iou_threshold,
                  int32_t *indices_dev, int32_t *count_dev, void *workspace, size_t workspace_bytes, void *stream);

/* Parity hook: the float32 exponential each decode dialect is pinned to, element-wise on device arrays.
 *   mode 0  correctly rounded exp (KERAS dialect: tools/utils.py:545-546 / keras_inference.py:101 evaluate exp and sigmoid inside
 *           TensorFlow, whose last-bit behaviour is not reproducible; this build and oracle/decode_ref.py define it as the
 *           correctly rounded value so that score order and NMS survivor sets are a function of the head tensors alone)
 *   mode 1  glibc's expf algorithm bit for bit (REGION_C dialect: region_layer.c:75,104 call libm's expf) */
int k2y_expf_eval(int mode, const float *x_dev, float *y_dev, long long n, void *stream);

/* ------------------------------------------------------------------------------------------
 * Pre-processing: aspect-preserving letterbox of ONE uint8 HWC RGB image on the device
 * (tools/utils.py:372-400: AffineTransform(scale, translation) + skimage warp order 1, zero fill, .astype('uint8')).
 * inv_matrix_host: the first two rows of inv([[s,0,tx],[0,s,ty],[0,0,1]]) as 6 doubles (host memory) - what
 * `aff.inverse` hands to warp.  dst_dev: [dst_h][dst_w][3] uint8, ready for k2y_net_bind_u8.  minmax_dev: 2 ints of
 * device scratch (receives 255 - min and the max of the source image, used by warp's output clipping).
 * ---------------------------------------------------------------------------------------- */
int k2y_letterbox_u8(const unsigned char *src_dev, int src_h, int src_w, const double *inv_matrix_host,
                     unsigned char *dst_dev, int dst_h, int dst_w, int *minmax_dev, void *stream);
/* The same letterbox for n images of different sizes in one call (k2y_letterbox_u8 is its n = 1 case).
 * src_dev: the images packed back to back, image i at byte offsets_host[i] (a multiple of 16 lets pass 1 read 16 bytes at a
 * time).  hw_host: [n][2] ints (h, w).  inv_matrices_host: [n][6] doubles, one k2y_letterbox_u8 matrix per image.
 * dst_dev: [n][dst_h][dst_w][3] uint8.  image_hw_dev: [n][2] float32 (h, w) written for the decode's correct_box, or NULL.
 * minmax_dev: [n][2] ints of device scratch.  Host arrays are read before the call returns; the work is asynchronous on
 * `stream` (one memset, then two kernels per 48 images). */
int k2y_letterbox_u8_batch(const unsigned char *src_dev, int n, const long long *offsets_host, const int *hw_host,
                           const double *inv_matrices_host, unsigned char *dst_dev, int dst_h, int dst_w,
                           float *image_hw_dev, int *minmax_dev, void *stream);
/* The same letterbox for n_views VIEWS: view i is the window windows_host[i] = (y0, x0, th, tw), in pixels, of the image at
 * offsets_host[i] whose full size is hw_host[i]; several views may name the same image.  A view is letterboxed as the crop
 * img[y0:y0+th, x0:x0+tw] submitted as an image of its own would be: inv_matrices_host[i] is the matrix of a th x tw image,
 * pixels outside the window read as zero fill (not as the neighbouring pixels) and the output is clipped to the window's own
 * min and max.  image_hw_dev receives (th, tw) per view, view_yx_dev ([n_views][2] float32, or NULL) receives (y0, x0), which
 * k2y_merge_views adds to the view's boxes.  A window that is not inside its image is K2Y_ERR_INVALID before anything is
 * enqueued.  k2y_letterbox_u8_batch is the case of one whole-image window per image; the work is the same one memset and two
 * kernels per 48 views. */
int k2y_letterbox_u8_views(const unsigned char *src_dev, int n_views, const long long *offsets_host, const int *hw_host,
                           const int *windows_host, const double *inv_matrices_host, unsigned char *dst_dev, int dst_h, int dst_w,
                           float *image_hw_dev, float *view_yx_dev, int *minmax_dev, void *stream);
/* k2y_letterbox_u8_views with mirrored views: mirror_host[i] nonzero letterboxes view i as np.fliplr of its window, bit for bit
 * (the same matrix, min and max; only the fetched column changes).  NULL: no view is mirrored, k2y_letterbox_u8_views. */
int k2y_letterbox_u8_views_mirror(const unsigned char *src_dev, int n_views, const long long *offsets_host, const int *hw_host,
                                  const int *windows_host, const int *mirror_host, const double *inv_matrices_host,
                                  unsigned char *dst_dev, int dst_h, int dst_w, float *image_hw_dev, float *view_yx_dev,
                                  int *minmax_dev, void *stream);

/* ------------------------------------------------------------------------------------------
 * Baseline JPEG decode on the device, in front of k2y_letterbox_u8_batch: replaces the file decode of
 * Helper._read_img (tools/utils.py:339-355, skimage.io.imread -> PIL -> libjpeg-turbo) for the files it accepts.
 * Exactness: the RGB bytes equal libjpeg-turbo's with PIL's settings, i.e. the JDCT_ISLOW integer IDCT (jidctint.c),
 * fancy upsampling (jdsample.c, as jinit_upsampler dispatches it) and ycc_rgb_convert (jdcolor.c); grey files are
 * written to all three channels, as _read_img stacks them.
 * GPU-decodable: 8-bit sequential Huffman (SOF0/SOF1), one scan holding every component, 1 component or 3 that libjpeg
 * treats as YCbCr, chroma 1x1 with luma 1x1, 2x1, 1x2, 2x2 or 4x1, any restart interval.  Every other valid file
 * (progressive, arithmetic, 12-bit, lossless, CMYK/YCCK, RGB, multi-scan, DNL, other sampling) is reported with its
 * reason and is left to the host; progressive files have decode entry points of their own (k2y_jpeg_progressive_*, below).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int32_t height, width, components;
    int32_t h_samp[4], v_samp[4];   /* per component, frame order (0 past `components`) */
    int32_t restart_interval;       /* MCUs, 0 = none */
    int32_t precision;              /* bits per sample */
    int32_t sof_marker;             /* 0xC0 .. 0xCF */
    int32_t gpu_decodable;          /* 1: k2y_jpeg_plan accepts the file */
    int32_t entropy_offset;         /* first byte of the scan's entropy-coded data (GPU-decodable files) */
    char reason[64];                /* why not, when gpu_decodable == 0 */
} k2y_jpeg_info;
/* Host only: walks the markers up to the first SOS.  K2Y_ERR_INVALID (message names the marker and its offset) for a
 * malformed file; K2Y_OK with info->gpu_decodable and info->reason otherwise. */
int k2y_jpeg_inspect(const unsigned char *data, size_t size, k2y_jpeg_info *info);
/* Host only: the descriptor blob of a batch of n GPU-decodable files (dimensions, sampling, quantisation tables, Huffman
 * decode tables in lookup form, restart segments and every offset).  files[i] / sizes[i]: the file bytes on the host;
 * src_offsets[i]: where file i will lie in the device source buffer; dst_offsets[i]: where its h*w*3 RGB bytes go in the
 * device output buffer (BatchLayout's offsets).  blob == NULL: only *blob_bytes is set (size query); otherwise blob is a
 * 16-byte aligned host buffer of blob_capacity >= *blob_bytes.  A file that is not GPU-decodable is K2Y_ERR_INVALID. */
int k2y_jpeg_plan(const unsigned char *const *files, const size_t *sizes, int n, const long long *src_offsets,
                  const long long *dst_offsets, void *blob, size_t blob_capacity, size_t *blob_bytes);
/* Device workspace k2y_jpeg_decode needs for the batch a blob describes (read from the host copy of the blob). */
int k2y_jpeg_workspace_bytes(const void *blob_host, size_t *bytes);
/* Decodes the batch, asynchronous on `stream`: blob_host is read before the call returns (launch sizes), blob_dev is the
 * same bytes on the device (16-byte aligned), src_dev the files at their src_offsets, dst_dev the output.  Five kernels,
 * one launch each whatever the image count: unstuff/split at RSTn, self-synchronising Huffman decode (one CTA per restart
 * segment), DC prediction, dequantise + IDCT, upsample + colour convert.  status_dev: int32 [n][4] per image: error bits
 * (1 invalid Huffman code, 2 entropy data ended early: the image's pixels are then undefined, the other images' are
 * exact), the most synchronisation rounds one window of subsequences took, their sum and the number of windows.
 * Corrupt data never makes a kernel read outside its image's bytes or write outside its output. */
int k2y_jpeg_decode(const void *blob_host, const void *blob_dev, const unsigned char *src_dev, unsigned char *dst_dev,
                    void *workspace_dev, size_t workspace_bytes, int32_t *status_dev, void *stream);

/* ------------------------------------------------------------------------------------------
 * Progressive Huffman JPEG decode on the device (SOF2), the same pixels as libjpeg-turbo with PIL's settings: jdphuff.c's
 * entropy decode (spectral selection, successive approximation, EOB runs, correction bits), then the baseline decoder's
 * IDCT, upsampling and colour conversion.  The baseline entry points above do not change: they report progressive files as
 * valid but not theirs.
 * GPU-decodable: SOF2 with 8-bit samples, 1 component or 3 that libjpeg treats as YCbCr, the baseline decoder's sampling
 * layouts and size limits, any restart interval (it may change between scans), at most 64 scans, ending with an EOI marker.
 * A scan libjpeg-turbo refuses (JERR_BAD_PROGRESSION: a DC scan with Se != 0; an AC scan with Ss > Se, Se > 63 or more than
 * one component; Ah != 0 with Al != Ah - 1; Al > 13) makes the file K2Y_ERR_INVALID naming the scan.  Valid files left to the
 * host, with their reason: scripts libjpeg-turbo decodes only with a JWRN_BOGUS_PROGRESSION warning (an AC scan before the
 * component's DC, a refinement whose Ah is not the coefficient's last Al) or that send a first scan of a coefficient twice;
 * scripts after which libjpeg-turbo block-smooths the output (jdcoefct.c smoothing_ok: every component has its DC and its
 * zig-zag quantisers 0..9 nonzero, and some component's coefficient 1..9 was never sent or only down to a bit above 0);
 * a Huffman table not defined before a scan that needs it; more than 64 scans.  Coefficients 10..63 never sent or
 * partly refined decode on the device.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int32_t height, width, components;
    int32_t sof_marker;             /* 0xC0 .. 0xCF */
    int32_t scans;                  /* SOS markers before EOI (0 when the walk stopped at the frame header) */
    int32_t levels;                 /* entropy-decode launches the scan script needs (see k2y_jpeg_progressive_decode) */
    int32_t gpu_decodable;          /* 1: k2y_jpeg_progressive_plan accepts the file */
    char reason[64];                /* why not, when gpu_decodable == 0 */
} k2y_jpeg_progressive_info;
/* Host only: walks every marker to EOI.  K2Y_ERR_INVALID (the message names the marker or the scan) for a malformed file;
 * K2Y_OK with info->gpu_decodable and info->reason otherwise ("sequential (SOF 0xC0)" for a baseline file). */
int k2y_jpeg_progressive_inspect(const unsigned char *data, size_t size, k2y_jpeg_progressive_info *info);
/* Host only: the descriptor blob of a batch of n GPU-decodable progressive files (geometry, quantisation tables, one record
 * per scan with its Huffman tables, one per (scan, restart interval) with its bytes in the file), with the arguments of
 * k2y_jpeg_plan; src_offsets must be multiples of 16.  A file that is not GPU-decodable is K2Y_ERR_INVALID. */
int k2y_jpeg_progressive_plan(const unsigned char *const *files, const size_t *sizes, int n, const long long *src_offsets,
                              const long long *dst_offsets, void *blob, size_t blob_capacity, size_t *blob_bytes);
/* Device workspace k2y_jpeg_progressive_decode needs for the batch a blob describes (read from the host copy of the blob). */
int k2y_jpeg_progressive_workspace_bytes(const void *blob_host, size_t *bytes);
/* Decodes the batch, asynchronous on `stream`, with the arguments of k2y_jpeg_decode; src_dev is 16-byte aligned and each
 * file's slot is readable up to its size rounded up to 16 bytes.  The entropy decode takes one launch per level of the
 * scripts (a scan's level is one more than the highest level of the earlier scans that touched one of its coefficients, 0
 * if none; a default libjpeg script has three), each decoding every (scan, restart interval) segment of that level serially
 * in one thread; then dequantise + IDCT and upsample + colour, one launch each.  status_dev: int32 [n][4] per image: error
 * bits (1 invalid Huffman code, 2 entropy data ended early, 4 a DC value outside int: the image's pixels are then undefined,
 * the other images' are exact), 0, 0 (the decode does not speculate, so it has no synchronisation rounds), segments decoded.
 * Corrupt data never makes a kernel read outside its image's bytes or write outside its output. */
int k2y_jpeg_progressive_decode(const void *blob_host, const void *blob_dev, const unsigned char *src_dev, unsigned char *dst_dev,
                                void *workspace_dev, size_t workspace_bytes, int32_t *status_dev, void *stream);

/* ------------------------------------------------------------------------------------------
 * PNG decode on the device, in front of k2y_letterbox_u8_batch: the RGB pixels Helper._read_img (PIL) gives for
 * non-interlaced PNGs of every colour type and depth except 16-bit greyscale (palette lookup with (0, 0, 0) past the PLTE
 * entries, 1/2/4-bit grey scaled to 0..255, grey replicated, the high byte of 16-bit samples, alpha dropped).
 * GPU-decodable: such a file of at most 65535 rows and columns and 2^31 - 1 filtered bytes whose chunks before the first IDAT have correct CRCs, with a
 * PLTE where one is needed, no unknown critical or acTL chunk, one run of IDAT chunks, an IEND and a zlib header with CM = 8,
 * CINFO <= 7 and no preset dictionary.  Every other file is reported with its reason and is left to the host.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int32_t height, width;
    int32_t color_type, bit_depth, interlace;   /* IHDR */
    int32_t idat_chunks;
    int64_t stream_bytes;           /* zlib stream: the payload of every IDAT */
    int32_t gpu_decodable;          /* 1: k2y_png_plan accepts the file */
    char reason[64];                /* why not, when gpu_decodable == 0 */
} k2y_png_info;
/* Host only: walks the chunks.  K2Y_ERR_INVALID for a file without the PNG signature and a sound IHDR; K2Y_OK with
 * info->gpu_decodable and info->reason otherwise. */
int k2y_png_inspect(const unsigned char *data, size_t size, k2y_png_info *info);
/* Host only: the descriptor blob of a batch of n GPU-decodable files (IDAT ranges, geometry, palette, workspace offsets), with
 * the arguments of k2y_jpeg_plan.  A file that is not GPU-decodable is K2Y_ERR_INVALID. */
int k2y_png_plan(const unsigned char *const *files, const size_t *sizes, int n, const long long *src_offsets,
                 const long long *dst_offsets, void *blob, size_t blob_capacity, size_t *blob_bytes);
/* Device workspace k2y_png_decode needs for the batch a blob describes (read from the host copy of the blob). */
int k2y_png_workspace_bytes(const void *blob_host, size_t *bytes);
/* Decodes the batch, asynchronous on `stream`, with the arguments of k2y_jpeg_decode.  Six kernels, one launch each whatever the
 * image count: gather the IDAT payloads; find, in every 64 KiB chunk of compressed data after the first, the first bit where a
 * block header parses strictly; decode every chunk from there (one warp each) into bytes and references to the 32 KiB before
 * it, until it stands on a later chunk's candidate at a block boundary; follow the chain of those links from the stream's start
 * and resolve the references chunk by chunk (one CTA per image), checking the Adler-32; inflate serially the images whose chain
 * does not end exactly at the image's size with a good Adler-32 (damaged or unusual streams, with zlib's rules as PIL drives
 * it); unfilter + colour (one CTA per image).  A stream without findable block headers (fixed Huffman only, one huge block) is
 * decoded by its first chunk alone.  status_dev: int32 [n][4] per image: error bits (1 invalid block header, 2 invalid code, 4
 * distance too far back, 8 image data ends early, 16 Adler-32 mismatch, 32 filter type above 4: the image's pixels are then
 * undefined, the other images' are exact), chunks, chunks after the first whose speculative start was confirmed, and bytes the
 * longest single decoder inflated (all of them when the image fell back to the serial decoder).  Where zlib, as PIL drives it,
 * accepts a stream, so does the decoder, and rows a stream that ends cleanly early does not fill decode from zero bytes.
 * Corrupt data never makes a kernel read outside its image's bytes or write outside its output. */
int k2y_png_decode(const void *blob_host, const void *blob_dev, const unsigned char *src_dev, unsigned char *dst_dev,
                   void *workspace_dev, size_t workspace_bytes, int32_t *status_dev, void *stream);

/* ------------------------------------------------------------------------------------------
 * Baseline JPEG encoding, byte-identical to PIL's Image.fromarray(rgb).save(f, "JPEG", quality=q) with libjpeg-turbo 3.1:
 * JFIF APP0, two DQT, SOF0 4:2:0, the four standard Huffman tables, one interleaved scan, EOI.
 *   k2y_jpeg_encode_plan             host only: the descriptor blob of n images, hw_host int32 [n][2] (1..65500 each:
 *                                    libjpeg-turbo's JPEG_MAX_DIMENSION; PIL writes and reads no larger file),
 *                                    src_offsets_host: where image i's h*w*3 RGB bytes lie in the device source buffer.
 *                                    blob == NULL: only *blob_bytes (size query); else a 16-byte aligned host buffer.
 *                                    quality 1..100; anything else is K2Y_ERR_INVALID.
 *   k2y_jpeg_encode_workspace_bytes  device workspace, and the output capacity (bytes the batch's files take at most).
 *   k2y_jpeg_encode                  asynchronous on `stream`, seven launches whatever the image count: blob_host is read
 *                                    before the call returns, blob_dev is the same bytes on the device (16-byte aligned).
 *                                    The files are written back to back from dst_dev; lengths_dev (int64 [n]) their sizes.
 * ---------------------------------------------------------------------------------------- */
int k2y_jpeg_encode_plan(int n, const int *hw_host, const long long *src_offsets_host, int quality, void *blob,
                         size_t blob_capacity, size_t *blob_bytes);
/* Host only: the bytes a file of that size (1..65500 each) and quality starts with, SOI up to and including SOS (out == NULL:
 * size query). */
int k2y_jpeg_encode_header(int h, int w, int quality, unsigned char *out, size_t capacity, size_t *length);
int k2y_jpeg_encode_workspace_bytes(const void *blob_host, size_t *workspace_bytes, size_t *output_capacity);
int k2y_jpeg_encode(const void *blob_host, const void *blob_dev, const unsigned char *src_dev, unsigned char *dst_dev,
                    long long *lengths_dev, void *workspace_dev, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------
 * Detection rendering in place, pixel for pixel draw.draw_detections (see csrc/render.cu for the one deliberate difference:
 * a box whose outline rings cross stops at the first crossing ring instead of raising).  images_dev: packed HWC RGB, image i
 * at offsets_host[i] with size hw_host[i] (1..65535 each: drawing is not bound by the encoder's 65500).  atlas_dev[i]: the
 * device label atlas of image i's font (render.LabelAtlas: int32 header [8] with [0] = classes, int32 entries
 * [classes][101][8], then the glyph masks).  dets_dev /
 * counts_dev: k2y_det records [n][class_num][max_per_class] and counts [n][class_num] with the given per-image strides.
 * colors_dev: uint8 [class_num][3], class_num 1..80.  Asynchronous on `stream`, one launch per 128 images.
 * ---------------------------------------------------------------------------------------- */
int k2y_render_detections(unsigned char *images_dev, int n, const long long *offsets_host, const int *hw_host,
                          const int32_t *const *atlas_dev, const int32_t *dets_dev, const int32_t *counts_dev,
                          long long det_image_stride_words, long long count_image_stride_words, int class_num,
                          int max_per_class, const unsigned char *colors_dev, void *stream);

/* ------------------------------------------------------------------------------------------
 * Track rendering in place, pixel for pixel draw.draw_tracks (the same deliberate differences as k2y_render_detections).
 * Images as k2y_render_detections.  atlas_dev[i]: the device track atlas of image i's font (render.TrackLabelAtlas: int32
 * header [8] with [0] = 12 glyphs, int32 entries [12][10] of "0".."9", " ", "#", then the glyph masks).  ids_dev / boxes_dev
 * / counts_dev: the tracker's ids int32 [n][class_num][max_per_class], track boxes float32 (ymin, xmin, ymax, xmax)
 * [n][class_num][max_per_class][4] and the record counts [n][class_num], with the given per-image strides in elements;
 * records with id < 0 are not drawn.  Each track is drawn in colors_dev[id % color_num] (uint8 [color_num][3]) and labelled
 * "{class:2d} #{id}", class_num 1..80.  Asynchronous on `stream`, one launch per 128 images.
 * ---------------------------------------------------------------------------------------- */
int k2y_render_tracks(unsigned char *images_dev, int n, const long long *offsets_host, const int *hw_host,
                      const int32_t *const *atlas_dev, const int32_t *ids_dev, const float *boxes_dev, const int32_t *counts_dev,
                      long long id_image_stride, long long box_image_stride_words, long long count_image_stride, int class_num,
                      int max_per_class, const unsigned char *colors_dev, int color_num, void *stream);

/* ------------------------------------------------------------------------------------------
 * Evaluation: the counters behind the reference's Yolo_Precision / Yolo_Recall metrics (tools/custom.py:13-75) on device
 * tensors.  y_true_dev / y_pred_dev: n_boxes records of entry_floats = 5 + classes floats (any [..., A, 5+C] head or label
 * tensor, flattened); element 4 is the confidence.  counts_dev[3] (uint64, caller-zeroed, accumulated into): tp, fp, fn with
 *   tp: true > thr && pred > thr;  fp: !(true > thr) && pred > thr;  fn: true > thr && !(pred > thr)
 * precision = tp / (tp + fp), recall = tp / (tp + fn) (0 when the denominator is 0).  apply_sigmoid = 0 reproduces the
 * reference (raw logit against the threshold), 1 compares sigmoid(pred).
 * ---------------------------------------------------------------------------------------- */
int k2y_pr_counts(const float *y_true_dev, const float *y_pred_dev, long long n_boxes, int entry_floats, float threshold,
                  int apply_sigmoid, unsigned long long *counts_dev, void *stream);

/* ------------------------------------------------------------------------------------------
 * Detection AP / mAP over an annotated image list (VOC matching rule, all-point and 11-point AP), on the device.  The
 * protocol is written down in oracle/ap_ref.py: IoU without a "+1 pixel" term, no "difficult" objects, ties in score keep
 * stream order.  An evaluator holds the per-class ground-truth counts and one slot per (image, class, k < max_per_class)
 * of every image matched so far (score bits + one TP bit per threshold); the store grows by doubling.
 *   k2y_ap_create     class_num 1..1024, max_per_class >= 1, 1..16 IoU thresholds in (0, 1] (compared in float32).
 *   k2y_ap_match      one update of n_images, asynchronous on `stream` (one kernel): dets_dev / counts_dev as
 *                     k2y_detect_keras_strided writes them (same per-image strides, device memory), gt_dev the images'
 *                     ground truth packed as [total][5] float32 (class, ymin, xmin, ymax, xmax) in image pixels, image i's
 *                     rows at [gt_offsets_dev[i], gt_offsets_dev[i+1]) (int64, device), max_gt_per_image >= every image's
 *                     row count.  The inputs may be reused once the stream has passed the call.
 *   k2y_ap_result     ranks every stored detection by (class, score descending, stream order) and reduces the curves;
 *                     synchronous.  ap_host [T][C], ap07_host [C] (first threshold), npos_host [C]: float64 / int64; AP is NaN
 *                     for a class without ground truth.  status_host: K2Y_AP_* bits of anything invalid seen since the last
 *                     reset (the APs are then meaningless).
 *   k2y_ap_reset      forgets every update (keeps the store's memory).
 *   k2y_ap_tp_flags   n_images matched so far; with tp_host != NULL also copies the TP bits, uint16 [n_images][C][K] (bit t:
 *                     TP at threshold t, 0 past each count), synchronous.
 * Every call of one evaluator is ordered after the previous one, whatever streams they use.
 * ---------------------------------------------------------------------------------------- */
#define K2Y_AP_BAD_SCORE 1     /* a record within its count has a NaN score or one with the sign bit set */
#define K2Y_AP_BAD_COUNT 2     /* a count outside [0, max_per_class] (clamped) */
#define K2Y_AP_GT_OVERFLOW 4   /* an image has more ground-truth rows than max_gt_per_image (the rest were ignored) */
typedef struct k2y_ap k2y_ap;
int k2y_ap_create(int class_num, int max_per_class, const float *iou_thresholds, int n_thresholds, int device, k2y_ap **out);
int k2y_ap_destroy(k2y_ap *ap);
int k2y_ap_match(k2y_ap *ap, const int32_t *dets_dev, const int32_t *counts_dev, long long det_image_stride_words,
                 long long count_image_stride_words, int n_images, const float *gt_dev, const long long *gt_offsets_dev,
                 int max_gt_per_image, void *stream);
int k2y_ap_result(k2y_ap *ap, double *ap_host, double *ap07_host, long long *npos_host, unsigned *status_host, void *stream);
int k2y_ap_reset(k2y_ap *ap, void *stream);
int k2y_ap_tp_flags(k2y_ap *ap, uint16_t *tp_host, long long capacity, long long *n_images, void *stream);

/* ------------------------------------------------------------------------------------------
 * COCO detection evaluation on the device: what pycocotools' COCOeval(gt, dt, "bbox") computes with its default parameters
 * (IoU thresholds 0.50:0.05:0.95, 101 recall points, maxDets 1 / 10 / 100, area ranges all / small / medium / large with
 * bounds 0, 32^2, 96^2, 1e10).  The protocol is written down in oracle/coco_ref.py.  The ground truth is uploaded once;
 * the evaluator holds one slot per (image, class, k < min(max_per_class, 100)) with the record's score bits and, per
 * (area range, threshold), a TP bit and a not-ignored bit.
 *   k2y_coco_create   gt_host [n_gt][7] float64 (class index, x, y, w, h, area, iscrowd): image i's annotations, in file
 *                     order, at rows [gt_offsets_host[i], gt_offsets_host[i+1]), images in sorted image-id order and class
 *                     index c the c-th smallest category id.  n_images counts every image, with annotations or not.
 *                     class_num 1..1024, max_per_class >= 1.  iou_thresholds [10] / recall_thresholds [101]: COCOeval's
 *                     np.linspace values, increasing.
 *   k2y_coco_match    one update of n_images, asynchronous on `stream` (one kernel): dets_dev / counts_dev as k2y_ap_match
 *                     reads them, image_positions_dev (int64, device) each image's position in the sorted image-id list.
 *                     Records of an (image, class) are in score-descending order (the order the detection kernels emit);
 *                     the first min(count, 100) are evaluated.  Updates may arrive in any image order.
 *   k2y_coco_result   ranks every stored record by (class, score descending, image position, record order) and reduces the
 *                     curves; synchronous.  precision_host [10][101][C][4][3], recall_host [10][C][4][3] float64, COCOeval's
 *                     eval["precision"] / eval["recall"] (-1 where a class has no non-ignored ground truth in an area range;
 *                     images never matched count as images without detections).  status_host: K2Y_COCO_* bits of anything
 *                     invalid seen since the last reset (the results are then meaningless).
 *   k2y_coco_reset    forgets every update.
 * Every call of one evaluator is ordered after the previous one, whatever streams they use.
 * ---------------------------------------------------------------------------------------- */
#define K2Y_COCO_BAD_SCORE 1        /* a record within its count has a NaN score or one with the sign bit set */
#define K2Y_COCO_BAD_COUNT 2        /* a count outside [0, max_per_class] (clamped) */
#define K2Y_COCO_BAD_POSITION 4     /* an image position outside [0, n_images) (the image was skipped) */
#define K2Y_COCO_REPEATED_IMAGE 8   /* an image position given twice since the last reset */
typedef struct k2y_coco k2y_coco;
int k2y_coco_create(const double *gt_host, const long long *gt_offsets_host, long long n_images, int class_num,
                    int max_per_class, const double *iou_thresholds, const double *recall_thresholds, int device,
                    k2y_coco **out);
int k2y_coco_destroy(k2y_coco *coco);
int k2y_coco_match(k2y_coco *coco, const int32_t *dets_dev, const int32_t *counts_dev, long long det_image_stride_words,
                   long long count_image_stride_words, int n_images, const long long *image_positions_dev, void *stream);
int k2y_coco_result(k2y_coco *coco, double *precision_host, double *recall_host, unsigned *status_host, void *stream);
int k2y_coco_reset(k2y_coco *coco, void *stream);

/* ------------------------------------------------------------------------------------------
 * MOTChallenge tracking evaluation on the device: CLEAR MOT and the identity metrics by the protocol of oracle/mot_ref.py
 * (TrackEval's MotChallenge2DBox preprocessing and its CLEAR and Identity metrics), counts equal and float64 sums equal
 * bit for bit.
 *   k2y_mot_create        benchmark 15, 16, 17 or 20 (MOT15 has no distractor removal, MOT20 adds class 6 to the
 *                         distractors).
 *   k2y_mot_add_sequence  gt_host [n_gt][8] float64 (frame, id, left, top, w, h, conf, class; frames 1..seq_length, file
 *                         order within a frame; class 1 for MOT15), uploaded once; *index the sequence's number.  At most
 *                         K2Y_MOT_MAX_ROWS rows per frame.
 *   k2y_mot_update        one batch of frames of sequence `seq`, asynchronous on `stream` (one kernel): counts_dev int32
 *                         [n][C] and ids_dev int32 [n][C][K] / boxes_dev float32 [n][C][K][4] (ymin, xmin, ymax, xmax), the
 *                         blocks of DetectionPipeline.collect / tracks on the device, strided per frame (in words);
 *                         positions_dev int64 [n], each frame's position 0..seq_length-1, each given once (unchecked here).
 *                         The records of person_class with a track id >= 0 become the frame's tracker rows.
 *   k2y_mot_result        evaluates every sequence; synchronous.  counts_host [sequences][K2Y_MOT_FIELDS]: TP, FP, FN,
 *                         IDSW, Frag, MT, PT, ML, IDTP, kept gt rows, kept tracker rows, tracker ids; motp_sum_host
 *                         [sequences]; rounds_host [sequences] the CLEAR rounds, solved_host [sequences] the frame solves
 *                         that needed an assignment.  status_host: K2Y_MOT_* bits of anything invalid (the results are
 *                         then meaningless).
 *   k2y_mot_result_ex     k2y_mot_result, and HOTA (oracle/mot_hota_ref.py) of every sequence when hota_counts_host and
 *                         hota_sums_host are given (both or neither): hota_counts_host [sequences][3][K2Y_MOT_HOTA_ALPHAS]
 *                         TP, FN, FP and hota_sums_host [sequences][4][K2Y_MOT_HOTA_ALPHAS] the float64 sums LocA, AssA,
 *                         AssRe, AssPr per alpha (0.05, 0.10, ..., 0.95 as np.arange gives them), before their divisions.
 *                         A sequence past the id cap keeps zeros there.  k2y_mot_result is k2y_mot_result_ex without HOTA.
 * Every call of one evaluator is ordered after the previous one, whatever streams they use.
 * ---------------------------------------------------------------------------------------- */
#define K2Y_MOT_MAX_ROWS 512              /* gt rows, and tracker rows, of one frame */
#define K2Y_MOT_MAX_TRACK_ID (1 << 22)    /* tracker ids are below this */
#define K2Y_MOT_FIELDS 12
#define K2Y_MOT_TOO_MANY_ROWS 1           /* a frame has more than K2Y_MOT_MAX_ROWS tracker rows (the rest were dropped) */
#define K2Y_MOT_BAD_ID 2                  /* a track id >= K2Y_MOT_MAX_TRACK_ID */
#define K2Y_MOT_REPEATED_ID 4             /* a track id twice in one frame */
#define K2Y_MOT_BAD_BOX 8                 /* a track box that is not finite */
#define K2Y_MOT_BAD_COUNT 16              /* a count outside [0, max_per_class] (clamped) */
#define K2Y_MOT_TOO_MANY_IDS 32           /* a sequence's gt ids x tracker ids exceed 2^28 (its identity metrics were skipped) */
#define K2Y_MOT_HOTA_ALPHAS 19            /* HOTA's localisation thresholds */
typedef struct k2y_mot k2y_mot;
int k2y_mot_create(int benchmark, int device, k2y_mot **out);
int k2y_mot_destroy(k2y_mot *mot);
int k2y_mot_add_sequence(k2y_mot *mot, const double *gt_host, long long n_gt, int seq_length, int *index);
int k2y_mot_update(k2y_mot *mot, int seq, const int32_t *counts_dev, const int32_t *ids_dev, const float *boxes_dev,
                   long long count_stride_words, long long id_stride_words, long long box_stride_words, int n_frames,
                   const long long *positions_dev, int class_num, int max_per_class, int person_class, void *stream);
int k2y_mot_result(k2y_mot *mot, long long *counts_host, double *motp_sum_host, int *rounds_host, long long *solved_host,
                   unsigned *status_host, void *stream);
int k2y_mot_result_ex(k2y_mot *mot, long long *counts_host, double *motp_sum_host, int *rounds_host, long long *solved_host,
                      long long *hota_counts_host, double *hota_sums_host, unsigned *status_host, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* K210_YOLO_B200_H */
