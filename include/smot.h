/* smot.h -- C ABI of the SiamMOT hot-path library (libsmot.so, sm_90a / H100 only).
 *
 * Drop-in boundary.  The reference (amazon-science/siam-mot) reaches native code on its per-frame
 * inference path in two ways, both replaced here:
 *   (1) maskrcnn_benchmark._C (pybind11, upstream csrc/vision.cpp; un-vendored, see
 *       /root/reference/readme/INSTALL.md:89-105):
 *         roi_align_forward(input, rois[K,5], spatial_scale, ph, pw, sampling_ratio)
 *           <- called from maskrcnn_benchmark.layers.ROIAlign, used at
 *              siammot/modelling/track_head/EMM/sr_pool.py:28,89 and by the box-head Pooler
 *              (siammot/modelling/box_head/box_head.py:17,46)
 *         nms(dets[n,4], scores[n], thresh)
 *           <- boxlist_nms at siammot/operator_patch/rpn_patch.py:53,
 *              siammot/modelling/box_head/inference.py:174, siammot/modelling/track_head/track_solver.py:22
 *   (2) ATen/cuDNN/cuBLAS kernels issued by torch ops in the reference's Python (conv2d, linear,
 *       group_norm, interpolate, pad, topk, softmax ...), listed per entry point below.
 *
 * Conventions: plain pointers and sizes only (no torch types); every pointer is DEVICE memory owned
 * by the caller unless stated otherwise; the library never allocates, never synchronises and launches
 * on the given cudaStream_t (passed as void*); all entry points return 0 (SMOT_OK) or an error code,
 * with a message available from smot_last_error() (thread-local).  Activations are NHWC ("pixel-major,
 * channel-minor") with an explicit channel pitch `ld` (elements between consecutive pixels), stored
 * as SMOT_F32 or SMOT_F16; accumulation is always fp32.  Boxes are fp32 xyxy with the reference's
 * legacy "+1" pixel convention.
 */
#ifndef SMOT_H_
#define SMOT_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SMOT_ABI_VERSION 5

enum { SMOT_OK = 0, SMOT_ERR_INVALID = 1, SMOT_ERR_CUDA = 2, SMOT_ERR_UNSUPPORTED = 3 };
enum { SMOT_F32 = 0, SMOT_F16 = 1 };
enum { SMOT_CONV_AUTO = 0, SMOT_CONV_SIMT = 1, SMOT_CONV_TCGEN05 = 2 };

#define SMOT_MAX_LEVELS 5
#define SMOT_MAX_ANCHORS 16

int smot_abi_version(void);
const char* smot_last_error(void);

/* ---- dense contractions -------------------------------------------------------------------------
 * smot_conv2d: out = act( conv(in, weight) * scale + bias + residual ), NHWC, implicit GEMM.
 * Replaces F.conv2d / nn.Linear + FrozenBatchNorm2d + add + ReLU chains of
 *   siammot/modelling/backbone/dla.py:43-57,181-189,278-287 (DLA-34 body),
 *   siammot/operator_patch/fpn_patch.py:37-55 (FPN lateral / output convs),
 *   the upstream RPN head (via siammot/modelling/rcnn.py:48), the FPN2MLP box head
 *   (siammot/modelling/box_head/box_head.py:46-48) and EMMPredictor
 *   (siammot/modelling/track_head/EMM/feature_extractor.py:62-69).
 * weight: [Cout][KH][KW][Cin] in the input dtype.  scale/bias: fp32 [Cout] or NULL (1 / 0).
 * residual: [batch*OH*OW] x res_ld, input dtype, or NULL.  A 1x1 conv over `batch` rows with
 * H = W = 1 is a plain GEMM (fully connected layer).  The concat-free DLA root is expressed with
 * in_ld / out_ld (producers write straight into their channel slice of the root's input). */
typedef struct {
  const void* in;
  const void* weight;
  const float* scale;
  const float* bias;
  const void* residual;
  void* out;
  int batch, H, W, Cin, in_ld;
  int OH, OW, Cout, out_ld, res_ld;
  int KH, KW, stride, pad;
  int relu;
  int in_dtype;  /* SMOT_F32 | SMOT_F16: dtype of in, weight, residual */
  int out_dtype; /* SMOT_F32 | SMOT_F16 */
  int algo;      /* SMOT_CONV_* */
  /* optional scratch for split-K (wgmma path, few output tiles x long K): fp32 partial tiles, summed in split
   * order by a second kernel.  The first SMOT_CONV_WS_COUNTER_BYTES bytes are reserved (never written); calls
   * sharing a workspace must be stream-ordered -- concurrent streams need one workspace each. */
  void* workspace;
  size_t workspace_bytes;
} smot_conv_desc;
#define SMOT_CONV_WS_COUNTER_BYTES 65536
int smot_conv2d(const smot_conv_desc* d, void* stream);
/* Which kernel family SMOT_CONV_AUTO would pick for this descriptor (SMOT_CONV_SIMT / _TCGEN05). */
int smot_conv2d_algo(const smot_conv_desc* d);

/* ---- small NHWC tensor kernels --------------------------------------------------------------- */
/* fp32 CHW image -> NHWC activation (rcnn.py:46-47 entry; layout change only). */
int smot_image_to_nhwc(const float* chw, void* out, int C, int H, int W, int out_ld, int dtype, void* stream);
/* nn.MaxPool2d(2,2) of DlaTree.downsample (dla.py:216,227). out is (H/2)x(W/2). */
int smot_maxpool2x2(const void* in, void* out, int batch, int H, int W, int C, int in_ld, int out_ld, int dtype,
                    void* stream);
/* F.max_pool2d(x, kernel_size=3, stride=2, padding=1) of the ResNet stem (upstream maskrcnn_benchmark
 * modeling/backbone/resnet.py BaseStem.forward; the "R-50-FPN" body).  out is ((H-1)/2+1) x ((W-1)/2+1). */
int smot_maxpool3x3s2(const void* in, void* out, int batch, int H, int W, int C, int in_ld, int out_ld, int dtype,
                      void* stream);
/* The gather of a deformable 3x3 convolution (DCN v1; upstream layers/dcn DeformConv reached through DFConv2d at
 * siammot/modelling/backbone/dla.py:74-78, MODEL.DLA.STAGE_WITH_DCN): cols[oy][ox][k*C + c] = bilinear sample of input channel c
 * at (oy*stride - 1 + i + dy, ox*stride - 1 + j + dx), k = 3i + j, (dy, dx) = offsets[oy][ox][2k], [2k+1] (fp32, from the regular
 * offset conv); zero outside the map.  The deformable conv itself is then smot_conv2d (1x1) over the 9*C columns with the 3x3
 * weight [Cout][3][3][C] read as [Cout][9*C].  3x3, pad 1, stride 1 or 2, dilation 1. */
int smot_deform_im2col3x3(const void* in, const float* offsets, void* cols, int H, int W, int C, int in_ld, int off_ld, int OH,
                          int OW, int out_ld, int stride, int dtype, void* stream);
/* lateral += bilinear_resize(top -> HxW, align_corners=False)   (fpn_patch.py:49-51). */
int smot_upsample_add(const void* top, int Ht, int Wt, int top_ld, void* lateral, int H, int W, int lat_ld, int C,
                      int dtype, void* stream);
/* LastLevelMaxPool = max_pool2d(x,1,2,0): out[y][x] = in[2y][2x]  (fpn_patch.py:57-59). */
int smot_subsample2(const void* in, void* out, int H, int W, int C, int in_ld, int out_ld, int dtype, void* stream);
/* In-place GroupNorm(groups, eps) + optional ReLU over x[batch][HW][C] (make_conv3x3 use_gn path,
 * feature_extractor.py:54-57). */
int smot_groupnorm_relu(void* x, const float* gamma, const float* beta, int batch, int HW, int C, int ld, int groups,
                        float eps, int relu, int dtype, void* stream);

/* ---- ROIAlign (replaces _C.roi_align_forward + LevelMapper + TrackUtils.pad_feature) ----------
 * Legacy (non-"aligned") ROIAlign over an FPN pyramid with in-kernel level mapping
 * (floor(4 + log2(sqrt(area)/224 + 1e-6)) clamped to [k_min, k_min+num_levels-1], area with +1).
 * pad[l] > 0 emulates sampling from the zero-padded copy of level l that
 * siammot/modelling/track_head/track_utils.py:87-107 materialises (ROI coordinates are then in the
 * padded image frame, as produced by update_boxes_in_pad_images :109-135).
 * level_boxes (may be NULL = rois) are the boxes that choose the level (sr_pool.py:74).
 * count: optional device int; rows >= *count are zero-filled.  out: [max_rois][res][res][C]. */
typedef struct {
  const void* feat[SMOT_MAX_LEVELS];
  int H[SMOT_MAX_LEVELS], W[SMOT_MAX_LEVELS], ld[SMOT_MAX_LEVELS];
  float scale[SMOT_MAX_LEVELS];
  int pad[SMOT_MAX_LEVELS];
  int num_levels;
  int k_min;
} smot_pyramid;
int smot_roi_align(const smot_pyramid* pyr, const float* rois, const float* level_boxes, const int* count,
                   int max_rois, int channels, int res, int sampling_ratio, void* out, int dtype, void* stream);

/* smot_roi_align_batched: the box-head pooling (box_head.py:46, through the upstream Pooler) of `batch` images of one size in
 * one launch, for SiamMOT.forward on a (B,3,H,W) batch (rcnn.py:46-51 with the box head of roi_heads.py:25).  pyr describes
 * image 0; level l of image b starts image_stride[l] elements (host array) after image b-1's.  rois: [batch][max_rois][4], image b's
 * rows i < min(count[b], max_rois) are pooled from its own maps with smot_roi_align's in-kernel LevelMapper and arithmetic, the
 * others are zero.  out: [batch][max_rois][res][res][C].  Each image's rows equal smot_roi_align on that image bit for bit.
 * The ROIs choose their own level (no level_boxes); pyr->pad is honoured as in smot_roi_align. */
int smot_roi_align_batched(const smot_pyramid* pyr, const long long* image_stride, int batch, const float* rois, const int* count,
                           int max_rois, int channels, int res, int sampling_ratio, void* out, int dtype, void* stream);

/* ---- RPN proposal selection (rpn_patch.py:15-60 + upstream select_over_all_levels) -------------
 * Per level: order anchors by objectness (descending, ties -> lower anchor index; logits -0 and +0 are equal), take
 * pre_nms_top_n, decode with BoxCoder(1,1,1,1), clip unless amodal, drop boxes smaller than
 * min_size, NMS(nms_thresh) keeping post_nms_top_n; then the fpn_post_nms_top_n best over all levels.
 * head: fp32 [H*W][head_ld], columns [0,A) = objectness logits, [A + 4a + c] = deltas.
 * Outputs: out_boxes [fpn_post_nms_top_n][4], out_scores (sigmoid), *out_count. */
typedef struct {
  const float* head;
  int head_ld, H, W, A, stride;
  float cell_anchors[SMOT_MAX_ANCHORS * 4];
} smot_rpn_level;
size_t smot_rpn_select_workspace(int num_levels, int pre_nms_top_n);
int smot_rpn_select(const smot_rpn_level* levels, int num_levels, int pre_nms_top_n, int post_nms_top_n,
                    float nms_thresh, float min_size, int fpn_post_nms_top_n, int img_w, int img_h, int amodal,
                    float* out_boxes, float* out_scores, int* out_count, void* workspace, size_t workspace_bytes,
                    void* stream);

/* smot_rpn_select_batched: smot_rpn_select for `batch` images of one size (the RPN inference of rcnn.py:48 over a (B,3,H,W)
 * batch: upstream RPNPostProcessor.forward_for_single_feature_map per image + select_over_all_levels per image).  levels[l]
 * describes image 0's head of level l; image b's starts head_image_stride[l] floats (host array) after image b-1's.  One launch
 * sequence for all images (the image index is a grid dimension of every kernel).  Outputs out_boxes [batch][fpn_post_nms_top_n][4],
 * out_scores [batch][fpn_post_nms_top_n], out_count [batch]; each image's result equals smot_rpn_select on that image alone bit
 * for bit, (logit desc, anchor index asc) ties included.  The workspace is the single-image one per image. */
size_t smot_rpn_select_batched_workspace(int num_levels, int pre_nms_top_n, int batch);
int smot_rpn_select_batched(const smot_rpn_level* levels, const long long* head_image_stride, int batch, int num_levels,
                            int pre_nms_top_n, int post_nms_top_n, float nms_thresh, float min_size, int fpn_post_nms_top_n,
                            int img_w, int img_h, int amodal, float* out_boxes, float* out_scores, int* out_count, void* workspace,
                            size_t workspace_bytes, void* stream);

/* ---- sort + NMS (replaces _C.nms and the host-side mask reduction of upstream nms.cu) ----------
 * Rows i < min(n_max, *count) with scores[i*score_stride] > min_score are candidates.  They are
 * ordered by score descending (ties -> lower index; scores -0 and +0 are equal), suppressed with IoU(+1) > thresh, and at most
 * max_keep survivors are APPENDED at position *out_count (which is then advanced):
 *   out_index[k] = original row, out_boxes[k], out_scores[k], out_tag[k] = tag  (each may be NULL).
 * thresh <= 0 disables suppression (sort only).  n_max <= 4096. */
size_t smot_sort_nms_workspace(int n_max);
int smot_sort_nms(const float* boxes, int box_stride, const float* scores, int score_stride, const int* count,
                  int n_max, float min_score, float thresh, int max_keep, int tag, int* out_index, float* out_boxes,
                  float* out_scores, int* out_tag, int* out_count, void* workspace, size_t workspace_bytes,
                  void* stream);

/* smot_sort_nms_segmented: the per-class NMS of the box head's filter_results (siammot/modelling/box_head/inference.py:145-191,
 * boxlist_nms at :174) for `batch` images in one launch set, where the single-image path makes ncls-1 smot_sort_nms calls per image.
 * boxes [batch][n_max][ncls][4] and scores [batch][n_max][ncls] are smot_box_decode's outputs per image.  Segment (b, j), j in
 * [1, ncls): rows i < min(count[b], n_max) with scores > min_score, sorted, suppressed with IoU(+1) > thresh, at most max_keep kept
 * -- smot_sort_nms on column j.  Image b's survivors go to its block: class j's behind class j-1's, each class in score order.
 *   out_boxes [batch][cap][4], out_scores [batch][cap] (-1 past the image's count), out_block [batch][1 + cap] = count | labels.
 * Each image's block equals what smot_sort_nms appends for classes 1 .. ncls-1 into a block whose scores were -1 and count 0.
 * cap >= (ncls-1) * min(max_keep, n_max).  Kernels: sort, suppression mask, reduction, per-image scatter (4 launches). */
size_t smot_sort_nms_segmented_workspace(int batch, int ncls, int n_max);
int smot_sort_nms_segmented(const float* boxes, const float* scores, const int* count, int batch, int n_max, int ncls,
                            float min_score, float thresh, int max_keep, int cap, float* out_boxes, float* out_scores,
                            int* out_block, void* workspace, size_t workspace_bytes, void* stream);

/* ---- box head post-processing (inference.py:46-114 up to filter_results) ------------------------
 * head: fp32 [n_max][head_ld]: columns [0,ncls) class logits, [ncls + 4j + c] box deltas of class j.
 * For every row and class: softmax probability, BoxCoder(weights).decode, clip unless amodal.
 * track_labels != NULL marks every row as a propagated track (inference.py:93-103): its score row
 * becomes 0 except score[label] = prob[label] + 1.
 * out_boxes [n_max][ncls][4], out_scores [n_max][ncls]. */
int smot_box_decode(const float* head, int head_ld, const float* rois, const int* count, int n_max, int ncls,
                    const float* weights4, int img_w, int img_h, int amodal, const int* track_labels,
                    float* out_boxes, float* out_scores, void* stream);
/* smot_box_decode_batched: the same over `batch` segments of n_max rows (head [batch*n_max][head_ld], rois [batch][n_max][4],
 * outputs [batch][n_max][ncls][4] / [batch][n_max][ncls]), segment b decoded against its own count[b]: rows at or past it get
 * score -1 and a zero box, never a stale value.  No track rows.  Equal to smot_box_decode per image bit for bit. */
int smot_box_decode_batched(const float* head, int head_ld, const float* rois, const int* count, int batch, int n_max, int ncls,
                            const float* weights4, int img_w, int img_h, int amodal, float* out_boxes, float* out_scores,
                            void* stream);

/* ---- solver candidates: detections ++ refined tracks ---------------------------------------------
 * cat[0..ncap) = detections (as is); cat[ncap + r] = track r with its label's refined box and score
 *   s = (p_det + 1 + p_trk + 1) / 2   (roi_heads.py:67,76; = p_det + 1 when tracktor)  + active[r]
 *   (track_solver.py:69), or -1 when valid[r] == 0.  *zero_count (optional) is reset to 0. */
int smot_track_combine(const float* det_boxes, const float* det_scores, int ncap, const float* dec_boxes,
                       const float* dec_scores, int ncls, const int* labels, const float* conf, const int* valid,
                       const float* active, int n, int tracktor, float* cat_boxes, float* cat_scores, int* zero_count,
                       void* stream);

/* smot_track_combine_grouped: the same for more than one foreground class, where the reference's order matters: its box
 * head returns the refined tracks grouped by class (filter_results, inference.py:145-191) and _refine_tracks adds the EMM
 * scores taken BEFORE that regrouping position by position (roi_heads.py:67,76).  With V = valid tracks in memory order and
 * G = V stably sorted by label: cat[ncap + g] = box / detection score of track G[g], EMM score of V[g]; perm[g] = G[g]
 * (memory row) for g < |V|, and cat_scores = -1, perm = -1 for the unused tail.  Identical to smot_track_combine (up to
 * the compaction of invalid rows) when every track has the same label. */
int smot_track_combine_grouped(const float* det_boxes, const float* det_scores, int ncap, const float* dec_boxes,
                               const float* dec_scores, int ncls, const int* labels, const float* conf, const int* valid,
                               const float* active, int n, int tracktor, float* cat_boxes, float* cat_scores,
                               int* zero_count, int* perm, void* stream);

/* ---- EMM tracker ---------------------------------------------------------------------------------
 * smot_xcorr: depthwise valid cross-correlation (xcorr.py:37-45), NHWC:
 *   out[n][i][j][c] = sum_{u,v<T} x[n][i+u][j+v][c] * k[n][u][v][c],  x: SxS, k: TxT, out: (S-T+1)^2. */
int smot_xcorr(const void* x, const void* k, void* out, int n, int channels, int S, int T, int dtype, void* stream);

/* smot_roi_align_planar + smot_xcorr_planar: the same two operations with the search windows exchanged CHANNEL-PLANAR
 * (fp16 correlation, S = 30, T = 15 only): window element (roi r, channel c, row i, column j) lives at
 *   x_planar[(r * channels + c) * SMOT_XCORR_PLANE + i * SMOT_XCORR_ROW_PITCH + j]
 * and columns 30 / 31 of every row must be zero (smot_roi_align_planar never writes them: zero-fill the buffer once).
 * smot_roi_align_planar has smot_roi_align's semantics and arithmetic for any res <= 32 / row_pitch / plane_pitch and
 * both dtypes; smot_xcorr_planar produces exactly smot_xcorr's fp16 output ([n][16][16][channels], NHWC) from planar
 * windows and NHWC templates.  channels % 16 == 0.  Both honour programmatic dependent launch (SMOT_PDL). */
#define SMOT_XCORR_ROW_PITCH 40
#define SMOT_XCORR_PLANE 1208
int smot_roi_align_planar(const smot_pyramid* pyr, const float* rois, const float* level_boxes, const int* count,
                          int max_rois, int channels, int res, int sampling_ratio, void* out, int row_pitch,
                          int plane_pitch, int dtype, void* stream);
int smot_xcorr_planar(const void* x_planar, const void* k, void* out, int n, int channels, void* stream);
/* The same with the MMA phase chosen explicitly: 0 = xcorr_mma_kernel's (bit-identical to smot_xcorr), 1 = trimmed (m16n8k8 on
 * the live operand halves, fragments shared between template rows u and u+8; equal to fp16 rounding).  smot_xcorr_planar
 * takes 1 when the environment has SMOT_XCORR_PLANAR=2, else 0. */
int smot_xcorr_planar_mode(const void* x_planar, const void* k, void* out, int n, int channels, int mma_mode, void* stream);
/* ... and the channel group of a CTA (2, 4, 8 or 16 planes = MMA warps; channels % channel_group == 0; 0 = the flat form: one CTA per
 * SM, the plane list dealt in 4-plane units, for n * channels <= 28 planes per SM): the planes are independent,
 * the results do not depend on it.  smot_xcorr_planar / _mode take 16 while n * channels <= 32 planes per SM, else 8 (SMOT_XCORR_FLAT=1: the flat form while it
 * fits -- measured slower)
 * (SMOT_XCORR_CG overrides). */
int smot_xcorr_planar_cfg(const void* x_planar, const void* k, void* out, int n, int channels, int mma_mode, int channel_group,
                          void* stream);

/* smot_emm_decode: fused bicubic x`up` upsampling (track_core.py:69-71) + get_locations (:184-225) +
 * decode_response (:101-135) + clip/validity of wrap_results_to_boxlist (:165-181).
 * maps: fp32 [n][O][O][map_ld], channels 0,1 = cls logits, 2 = centerness logit, 3..6 = relu'd tlbr.
 * sr / tboxes: [n][4] search regions (padded frame) and template boxes.  pad = PAD_PIXELS,
 * T = template resolution.  Outputs: out_boxes [n][4], out_conf [n], out_valid [n] (0 when the
 * clipped box is empty and amodal == 0).  hann: fp32 [O*up] cosine window (track_core.py:155-162; passed in
 * so that it is bit-identical to torch.hann_window).  sigma = COSINE_WINDOW_WEIGHT.  scratch: n * 8 bytes. */
int smot_emm_decode(const float* maps, int map_ld, int n, int O, int up, int T, const float* sr, const float* tboxes,
                    const float* hann, float pad, int use_centerness, double sigma, int img_w, int img_h, int amodal,
                    float* out_boxes, float* out_conf, int* out_valid, void* scratch, void* stream);

/* ---- test-time frame preprocessing (SURVEY.md section 8 (f) rank 1) ---------------------------------
 * Replaces, for one decoded RGB uint8 HWC frame, the reference's CPU chain demos/demo_inference.py:74-82 ->
 * build_augmentation.py:52-66 (is_train=False): torchvision F.resize on a PIL image with the size from
 * ImageResize.get_size (image_augmentation.py:21-50) -> ToTensor -> maskrcnn_benchmark Normalize(mean, std,
 * to_bgr255).  Results are bit-identical to that chain (Pillow's 8-bit resampling is integer arithmetic).
 *
 * smot_resample_ksize / smot_resample_coeffs: HOST helpers restating Pillow libImaging/Resample.c
 *   precompute_coeffs + normalize_coeffs_8bpc for the bilinear filter over the whole axis: bounds[out][2] =
 *   (first source index, tap count), kk[out][ksize] = 22-bit fixed-point weights.  The caller copies both to the
 *   device once per (in_size, out_size).
 * smot_resample_h_u8: horizontal pass, uint8 [H][W][3] (row pitch in bytes) -> uint8 [H][OW][3]; only needed when
 *   OW != W (Pillow skips the pass otherwise).
 * smot_resample_v_normalize: vertical pass (bounds == NULL: height unchanged, no pass) fused with ToTensor and
 *   Normalize: uint8 [H][W][3] -> float32 [3][OH][W] = ((v/255)[*255 and BGR order if to_bgr255] - mean) / std,
 *   every step one IEEE fp32 operation as in the torch chain.  mean3 / std3: HOST float[3], output-channel order. */
int smot_resample_ksize(int in_size, int out_size);
int smot_resample_coeffs(int in_size, int out_size, int* bounds, int* kk);
int smot_resample_h_u8(const void* in, int in_pitch, int H, int W, const int* bounds, const int* kk, int ksize, int OW,
                       void* out, int out_pitch, void* stream);
int smot_resample_v_normalize(const void* in, int in_pitch, int H, int W, const int* bounds, const int* kk, int ksize,
                              int OH, const float* mean3, const float* std3, int to_bgr255, float* out_chw, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SMOT_H_ */
