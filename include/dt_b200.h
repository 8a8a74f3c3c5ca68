/* dt_b200.h — C ABI of libdt_b200.so, the H100 (sm_90a) hot path behind the
 * DetectAndTrack cfg / model-builder / tools surface.
 *
 * Conventions (all entry points):
 *   - plain C types only; every data pointer is a DEVICE pointer owned by the
 *     caller unless the parameter is documented as host; nothing is allocated,
 *     freed or synchronised inside; work is enqueued on `stream` (a
 *     cudaStream_t passed as void*, NULL = legacy default stream).
 *   - returns 0 on success, non-zero on error; dt_last_error() then holds the
 *     message (per host thread).  Python raises RuntimeError with that text,
 *     matching the reference's CAFFE_ENFORCE -> RuntimeError behaviour
 *     (/root/reference/tests/test_zero_even_op.py:41-44).
 *   - boxes are fp32 rows [x1,y1,x2,y2]*T (+score) exactly as the reference
 *     lays them out (lib/utils/boxes.py:26-57); integer outputs are int32.
 *
 * The reference has one C-ABI precedent for this path,
 *   void _nms(int* keep_out, int* num_out, const float* boxes_host, int boxes_num,
 *             int boxes_dim, float nms_overlap_thresh, int device_id);
 *   (/root/reference/lib/nms/gpu_nms.hpp:3-9): host pointers, internal
 *   malloc/memcpy/free.  dt_nms_batched replaces it with device pointers, a
 *   stream, a batch dimension and both reference comparators.
 * Everything else on the path is a Caffe2 Operator (C++ class ABI, un-vendored);
 * each function below cites the operator / python function it replaces.
 */
#ifndef DT_B200_H_
#define DT_B200_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DT_B200_ABI_VERSION 4
#define DT_MAX_T 8              /* frames per tube supported by the box kernels */
#define DT_NMS_MAX_BOXES 8192   /* per problem */
#define DT_LSA_MAX_DIM 224      /* max(prev, cur) detections per frame pair */

/* NMS comparator / output order */
#define DT_NMS_2D_GE 0      /* lib/utils/cython_nms.pyx:83-85      suppress ovr >= thr (T must be 1) */
#define DT_NMS_TUBE_GT 1    /* lib/nms/py_cpu_nms_tubes.py:49-51   keep mean-IoU <= thr              */
#define DT_NMS_ORDER_SCORE 0  /* survivors in descending-score order (py_cpu_nms_tubes) */
#define DT_NMS_ORDER_INDEX 1  /* survivors in ascending input index (cython_nms np.where) */

/* TRACKING.BIPARTITE_MATCHING_ALGO (lib/core/tracking_engine.py:236-242) */
#define DT_MATCH_HUNGARIAN 0  /* scipy.optimize.linear_sum_assignment, :237        */
#define DT_MATCH_GREEDY 1     /* bipartite_matching_greedy, :184-206 (argmin loop) */

const char* dt_last_error(void);
int dt_abi_version(void);

/* cudaMemsetAsync on the caller's stream (a memset node under CUDA-graph capture): how the hot path zeroes its
 * fixed-capacity count / output buffers without library kernels. */
int dt_memset(void* ptr, int value, size_t bytes, void* stream);

/* ---- boxes.cu ----------------------------------------------------------- */

/* lib/utils/boxes.py:60-69 bbox_overlaps -> lib/utils/cython_bbox.pyx:16-56.
 * boxes [n, ldb], query [k, ldq] (first 4*T columns used), out [n, ldo] =
 * mean over T of the '+1' IoU.  Bit-exact with the compiled reference. */
int dt_bbox_overlaps(const float* boxes, int n, int ldb, const float* query, int k, int ldq,
                     int T, float* out, int ldo, void* stream);

/* lib/core/nms_wrapper.py:49-70 nms / tube_nms, batched.
 * dets [batch, nmax, ld]: columns 0..4T-1 boxes, column 4T score.
 * counts [batch] (device) valid rows per problem, NULL = nmax.
 * keep [batch, nmax] receives indices into the problem's rows, num_keep [batch].
 * max_keep > 0 truncates the returned list (generate_proposals.py:108-110).
 * Ties in score: descending score, then descending index (the reference's
 * order is undefined under ties). */
int dt_nms_workspace_bytes(int batch, int nmax, size_t* bytes /*host out*/);
int dt_nms_batched(const float* dets, int batch, int nmax, int ld, int T, const int* counts,
                   float thresh, int cmp_mode, int out_order, int max_keep, int* keep,
                   int* num_keep, void* workspace, size_t workspace_bytes, void* stream);

/* TEST.SOFT_NMS.METHOD (lib/core/nms_wrapper.py:37) */
#define DT_SOFT_NMS_HARD 0
#define DT_SOFT_NMS_LINEAR 1
#define DT_SOFT_NMS_GAUSSIAN 2

/* lib/core/nms_wrapper.py:29-46 soft_nms -> lib/utils/cython_nms.pyx:98-203, batched, 2-D boxes.
 * dets [batch, nmax, ld] (ld >= 5: columns 0..3 box, 4 score), counts [batch] (device) valid rows, NULL = nmax.
 * out [batch, nmax, 5] receives the surviving rows (original coordinates, decayed scores) in the reference's row
 * order, out_inds [batch, nmax] (may be NULL) the source row of each, out_counts [batch] their number.
 * Nt: overlap threshold of the linear / hard methods; threshold: rows whose decayed score falls below it are dropped.
 * Bit-exact with the compiled reference.  nmax <= DT_NMS_MAX_BOXES.  No host synchronisation. */
int dt_soft_nms_batched(const float* dets, int batch, int nmax, int ld, const int* counts, float sigma, float Nt,
                        float threshold, int method, float* out, int* out_inds, int* out_counts, void* stream);

/* lib/utils/boxes.py:294-310 box_voting, batched: each top row's box becomes the score-weighted np.average of the
 * boxes of `all` [batch, nmax, ld] (counts all_counts, NULL = nmax) whose IoU with it is >= thresh; its score is kept.
 * Top rows: with top_keep [batch, nmax] (dt_nms_batched's keep), rows top_keep[b, :top_counts[b]] of `all` (top is
 * then unused and top_nmax must equal nmax); else top [batch, top_nmax, ld_top] rows :top_counts[b] (dt_soft_nms_batched's
 * output).  out [batch, top_nmax, 5] in the top order, out_counts [batch] = top_counts.  Bit-exact with the reference
 * under numpy 2.x.  No host synchronisation. */
int dt_box_vote(const float* top, const int* top_keep, const int* top_counts, int top_nmax, int ld_top,
                const float* all, const int* all_counts, int batch, int nmax, int ld, float thresh, float* out,
                int* out_counts, void* stream);

/* ---- lsa.cu ------------------------------------------------------------- */

/* scipy.optimize.linear_sum_assignment as called at
 * lib/core/tracking_engine.py:237, batched: cost [batch, dmax, ldc] fp32
 * (rows = previous frame, cols = current frame), nrows/ncols [batch] device.
 * matches [batch, dmax]: matches[q] = assigned row p, or -1
 * (tracking_engine.py:229-246).  status [batch] (may be NULL): 1 = infeasible, or (hungarian) a NaN or -inf entry,
 * where scipy raises ValueError.  Indices equal scipy >= 1.6 bit-for-bit (see oracle/lsa.py). */
int dt_lsa_batched(const float* cost, int batch, int dmax, int ldc, const int* nrows,
                   const int* ncols, int algo, int* matches, int* status, void* stream);
/* The same on fp64 costs [batch, dmax, ldc >= dmax] (dt_frame_costs / dt_gt_frame_costs), solved in fp64 as scipy
 * solves the reference's float64 matrix.  The costs are read from global memory, not staged in shared memory. */
int dt_lsa_batched_f64(const double* cost, int batch, int dmax, int ldc, const int* nrows,
                       const int* ncols, int algo, int* matches, int* status, void* stream);

/* lib/core/tracking_engine.py:158-246 fused: cost = weight * (1 - IoU) between
 * frame f-1 and frame f, then the assignment.  frames [nframes, dmax, ld]
 * (4*T box columns first), counts [nframes]; frame 0 and frames with
 * is_start[f] != 0 (may be NULL) get all -1 (first frame of a video, :283-285). */
int dt_match_frames(const float* frames, int nframes, int dmax, int ld, int T, const int* counts,
                    const unsigned char* is_start, float weight, int algo, int* matches, int* status,
                    void* stream);

/* 'pose-pck' tracking cost (lib/core/tracking_engine.py:113-129, lib/utils/keypoints.py:266-291): a [P, ld], b [Q, ld]
 * poses as the reference's [4, K] arrays (x row at 0, y row at K); out [P, Q] fp64 = 1 - (#joints with
 * |a_k - b_k| / (|a_head_top - a_head_bottom| + 1) < dist_thresh) / K, in the reference's float32 arithmetic. */
int dt_pose_pck_cost(const float* a, int P, const float* b, int Q, int ld, int K, int head_top, int head_bottom,
                     float dist_thresh, double* out, void* stream);

/* lib/core/tracking_engine.py:158-181 for all frame pairs at once: cost [nframes, dmax, dmax] fp64 with
 * cost[f][p][q] = fp32(w_iou * (1 - IoU(boxes[f-1][p], boxes[f][q]))) + w_pck * pck(poses[f-1][p], poses[f][q]) (fp64 sum,
 * like np.sum(np.stack(all_Cs))); frames with is_start != 0 (and frame 0) and entries beyond counts are 0.  boxes [nframes,
 * dmax, ldb], poses [nframes, dmax, ldp] (may be NULL when w_pck == 0).  Feed to dt_lsa_batched_f64 (nrows = counts[f-1] or
 * 0, ncols = counts[f]): the reference solves this fp64 sum, and rounding it to fp32 would break its exact ties differently. */
int dt_frame_costs(const float* boxes, int ldb, int T, const float* poses, int ldp, int K, int head_top, int head_bottom,
                   float dist_thresh, const int* counts, const unsigned char* is_start, int nframes, int dmax, float w_iou,
                   double w_pck, double* cost, void* stream);

/* ---- upper_bound.cu: TRACKING.DEBUG.UPPER_BOUND* (lib/core/tracking_engine.py:272-350) ---- */
#define DT_UB_COMPACT 1     /* UPPER_BOUND: keep the detections a GT took, with the GT's track id */
#define DT_UB_GT_KPS 2      /* UPPER_BOUND_2_GT_KPS: the GT's box and keypoint rows 0..2 on every kept detection */
#define DT_UB_ONLY_CONF 4   /* UPPER_BOUND_2_GT_KPS_ONLY_CONF: keypoint row 2 only */

/* GT-vs-detection cost matrices of every frame: boxes [2 * nframes, dmax, ld] and poses [2 * nframes, dmax, R, K] hold the
 * GT of frame f at entry 2f (boxes padded with a score column, integer-valued keypoints in rows 0..2) and its detections at
 * entry 2f + 1; counts [2 * nframes].  cost [nframes, dmax, dmax] fp64, rows = GT, = fp32(w_iou * (1 - IoU)) + w_pck * pck
 * with the pck term in fp64 (numpy promotes the reference's int32 GT keypoints so); 0 beyond the counts.  Feed to
 * dt_lsa_batched_f64 with nrows = counts[2f], ncols = counts[2f + 1]. */
int dt_gt_frame_costs(const float* boxes, int ld, int T, const float* poses, int R, int K, int head_top, int head_bottom,
                      double dist_thresh, const int* counts, int nframes, int dmax, float w_iou, double w_pck, double* cost,
                      void* stream);
/* One CTA per frame of the same packing: matches [nframes, ldm] (detection -> GT row or -1, the configured cost; needed
 * with DT_UB_COMPACT) and matches_gt [nframes, ldmg] (the bbox Hungarian match of UPPER_BOUND_5_GT_KPS_ONLY, may be NULL).
 * gt_tid [nframes, dmax].  Outputs, rows compacted in ascending detection order under DT_UB_COMPACT: out_boxes [nframes,
 * dmax, ld], out_poses [nframes, dmax, R, K] (matches_gt's GT rows 0..2 win over DT_UB_GT_KPS's, as in the reference),
 * out_tid [nframes, dmax] (the GT track id, -1 without DT_UB_COMPACT), out_counts [nframes]. */
int dt_track_upper_bound(const float* boxes, int ld, const float* poses, int R, int K, const int* counts, const int* gt_tid,
                         int nframes, int dmax, const int* matches, int ldm, const int* matches_gt, int ldmg, int flags,
                         float* out_boxes, float* out_poses, int* out_tid, int* out_counts, void* stream);

/* lib/core/tracking_engine.py:272-350 id propagation.  video_first [nvideos]
 * (device) = index of the first frame of each video, ascending.  tracks
 * [nframes, dmax] (-1 beyond counts[f]).  ids: next_id++, and
 * `if next_id >= max_ids: next_id %= max_ids` (:339-345). */
int dt_assign_track_ids(const int* matches, const int* counts, const unsigned char* is_start,
                        int nframes, int dmax, const int* video_first, int nvideos, int first_id,
                        int max_ids, int* tracks, void* stream);

/* lib/core/tracking_engine.py:86-93,711-748: centre-frame selection (when
 * center_only), clip of the first box to [0,w]x[0,h], keep score >= conf and
 * (x2-x1)*(y2-y1) >= min_area.  boxes [nframes, dmax, ld] with score in
 * column 4*T; hw [nframes, 2] = (height, width); out [nframes, dmax, 4*T_out+1]
 * compacted in input order, counts_out [nframes], sel [nframes, dmax] (may be
 * NULL) = source row of each kept detection. */
int dt_prune_detections(const float* boxes, int nframes, int dmax, int ld, int T, int center_only,
                        const int* counts_in, const float* hw, float conf, float min_area,
                        float* out, int* counts_out, int* sel, void* stream);

/* ---- conv_tc.cu ---------------------------------------------------------- */

#define DT_DTYPE_BF16 0   /* bf16 activations/weights, fp32 accumulate (wgmma .bf16)         */
#define DT_DTYPE_TF32 1   /* fp32 storage, tf32 multiply, fp32 accumulate (wgmma .tf32)         */
#define DT_DTYPE_F16 2    /* fp16 x and w (11-bit operands at the full kind::f16 rate), fp32 accumulate; plain rows, no residual;
                             y is bf16 / bf16 pairs (x3 bit 1) / fp32 as for DT_DTYPE_BF16 */

/* Geometry + fused epilogue of one convolution (host struct, plain ints).
 * Replaces a Caffe2 Conv/ConvNd (engine=CUDNN) followed by AffineChannel[Nd]
 * (lib/ops/affine_channel_nd_op.cu:19-70), Sum and Relu
 * (lib/modeling/detector.py:410-436, lib/modeling/ResNet3D.py:21-101), the FPN
 * top-down UpsampleNearest+Sum (lib/modeling/FPN3D.py:186-222) and FC
 * (lib/modeling/head_builder.py:33-36; a 1x1x1 conv over W = #rows).
 *   x  [N, Ti, Hi, Wi, in_ld]   NDHWC (channels innermost), first Cin channels used
 *   w  [kT*kH*kW, Cout, w_ld]   tap-major, channels innermost (cross-correlation, as Caffe2)
 *   y  [N, To, Ho, Wo, out_ld]  first Cout channels written
 *   y = relu?( conv(x, w) * scale[c] + bias[c]  (+ residual) )
 * res_mode 0: none; 1: residual has y's shape (ld res_ld); 2: residual is
 * [N, To, Ho/2, Wo/2, res_ld] and is read at (ho/2, wo/2) (nearest 2x upsample).
 * Leading dims 0 => dense.  x/w rows must be 16-byte multiples, y/residual rows too. */
typedef struct dt_conv_desc {
  int N, Ti, Hi, Wi, Cin, Cout;
  int kT, kH, kW;
  int sT, sH, sW;
  int pT, pH, pW;
  int in_ld, w_ld, out_ld, res_ld;
  int dtype;      /* DT_DTYPE_* : type of x and w */
  int out_f32;    /* 1: y/residual fp32, 0: bf16 */
  int relu;
  int res_mode;
  int x3;             /* split ("x3") storage, the fp32-accurate modes.  bit 0: x and w rows are [hi | lo] pairs
                         (lo half at in_lo_off / w_ld/2) and D = x_hi*w_hi + x_lo*w_hi + x_hi*w_lo (three MMAs per
                         k-block); bit 1: y (and the residual) rows are written / read as [hi | lo] pairs.
                         DT_DTYPE_TF32 ("tf32x3"): fp32 storage, hi = tf32(v), lo = tf32(v - hi), y fp32.
                         DT_DTYPE_BF16 ("bf16x3"): bf16 storage, hi = bf16(v), lo = bf16(v - hi) — 16 mantissa
                         bits at the full kind::f16 MMA rate and half the bytes of tf32x3; y pairs are bf16
                         (out_f32 = 0), plain fp32 outputs (out_f32 = 1, bit 1 clear) are allowed */
  int in_lo_off, out_lo_off, res_lo_off;  /* element offsets of the lo halves (0 => ld / 2) */
  int out_round_tf32; /* fp32 output rounded (nearest-even) to tf32: set when the consumer is another
                         DT_DTYPE_TF32 conv, because kind::tf32 truncates its operands (a one-sided
                         error that otherwise compounds to percents over ~50 layers) */
  int out_time_major; /* 1: y is laid out [To, N, Ho, Wo, out_ld] instead of [N, To, Ho, Wo, out_ld], so one
                         frame of the whole batch (the 'slice-center' link, model_builder.py:1024-1042) is a
                         contiguous [N, Ho, Wo, out_ld] block and needs no gather */
  int out_t_first, out_t_count; /* compute only output frames [out_t_first, out_t_first + out_t_count) of the
                         conv (0, 0 = all): y then has out_t_count frames.  Lets a caller skip frames nothing
                         consumes (the post-hoc FPN convs under the 'slice-center' link) */
} dt_conv_desc;

int dt_conv3d(const dt_conv_desc* desc /*host*/, const void* x, const void* w, const float* scale,
              const float* bias, const void* residual, void* y, void* stream);

/* Host-only planning query (no device work, usable without a GPU): the tiling dt_conv3d would pick for `desc` —
 * column tile BN, M tile (TB images x TT frames x TH x TW positions <= 128 rows), tiles per launch, operand ring
 * (stages x ks (tap, channel chunk) groups of stage_bytes / ks bytes: one activation and one weight box, or with x3
 * inputs the hi and lo box of each), output staging / residual ring chunks, dynamic shared memory, MMA k-blocks per
 * tile (three per group with x3 inputs) and the fraction of MMA rows that are real output positions.
 * kiters is the per-tile maximum; a tap whose activation box lies wholly in the zero padding (or past the input) is
 * not issued, and mma_kblocks counts the MMA k-blocks the whole launch does issue.
 * residual_aligned: the residual pointer would be 16-byte aligned (enables the TMA residual ring for bf16 residual
 * modes). */
typedef struct dt_conv_plan_t {
  int BN, TH, TW, TT, TB;
  int tiles, kiters, stages, ks, ncbuf, nrbuf, smem_bytes;
  double useful_rows;
  int stage_bytes;
  double mma_kblocks;
} dt_conv_plan_t;
int dt_conv_plan(const dt_conv_desc* desc /*host*/, int residual_aligned, dt_conv_plan_t* plan /*host out*/);

/* ---- Winograd F(2x2, 3x3) of the bf16x3 keypoint head (3x3, pad 1, stride 1 on S x S maps, S even) ----------------
 * G = D * (S/2)^2 tiles.  V [16][G][2Cin] bf16 pairs (transformed input tiles, hi at c, lo at Cin + c), U [16][Cout][2Cin]
 * bf16 pairs (transformed filters G g G^T, the packed layout of a 16-tap conv), M [16][G][Cout] fp32.
 * dt_wino_gemm: M_xi = V_xi * U_xi^T for the 16 components xi in one launch of the conv kernel (split operands, three
 * MMAs per k-block); Cin % 64 == 0, Cout % 128 == 0.  dt_wino_plan: its plan, host-only (no device work). */
int dt_wino_gemm(const void* v, const void* u, float* m, int G, int Cin, int Cout, void* stream);
int dt_wino_plan(int G, int Cin, int Cout, dt_conv_plan_t* plan /*host out*/);
/* Transforms (wino.cu; C % 64 == 0, S even <= 16, D <= 65535).  x / y [D, S, S, 2C] bf16 pairs.
 * dt_wino_input: x -> V.  dt_wino_output_input: M (+ bias [C] or NULL, ReLU if relu) -> the layer's bf16-pair output ->
 * V of the next layer, without writing the output.  dt_wino_output: M (+ bias, ReLU) -> y. */
int dt_wino_input(const void* x, int D, int S, int C, void* v, void* stream);
int dt_wino_output_input(const float* m, int D, int S, int C, const float* bias, int relu, void* v, void* stream);
int dt_wino_output(const float* m, int D, int S, int C, const float* bias, int relu, void* y, void* stream);

/* conv1 of the ResNet bodies (lib/modeling/ResNet3D.py:258-261): 7x7 stride 2 pad 3 on the 3-channel
 * image + AffineChannel + ReLU, with the 7 taps of a filter row packed into one 128-byte k-block.
 * x_padded [F, 2, (Hp+6)/2, Wp+8, Cp] from dt_prep_clip(border 3, 4, row_planes 1), Cp*elemsize == 16;
 * w [7 (kh)][Cout <= 64][8*Cp] with w[kh][o][kw*Cp + c]; y [F, Hp/2, Wp/2, out_ld].
 * x3 != 0 (bf16x3 mode, DT_DTYPE_BF16): the blob pixel is [hi(3) | lo(3) | 0 0] (dt_prep_clip out mode 3), w holds
 * 14 blocks — [2*kh][o][kw*8 + s] = W_hi[c] for s = c and s = 3 + c, [2*kh+1][o][kw*8 + c] = W_lo[c] — so two MMAs
 * per filter row give x_hi*W_hi + x_lo*W_hi + x_hi*W_lo; y rows are [hi(Cout) | lo(Cout)] bf16 pairs. */
int dt_conv1_7x7s2(const void* x_padded, int F, int Hp, int Wp, int Cp, const void* w, int Cout,
                   const float* scale, const float* bias, int relu, int dtype, int out_f32,
                   int out_round_tf32, int x3, void* y, int out_ld, void* stream);

/* bf16 pair rows [rows, 2C] = [hi | lo] -> fp16 rows [rows, C] = fp16(hi + lo) (round to nearest, saturating): the operand of a
 * DT_DTYPE_F16 conv fed by a bf16x3 producer. */
int dt_pairs_to_f16(const void* pairs, long long rows, int C, void* out, void* stream);

/* ---- proposals.cu -------------------------------------------------------- */

/* GenerateProposalsOp up to NMS (lib/ops/generate_proposals.py:40-106,116-161) for ALL levels of a clip
 * batch in one launch: sigmoid, exact top pre_nms_topn by score (ties: ascending anchor index), shifted
 * (tube) anchors, bbox/tube decode (weights 1), clip to im_info, min-size filter (AND over frames).
 * Per level: logits [B, H, W, ld_s] (first A channels), deltas [B, H, W, ld_d] (first 4*A*T; channel
 * a*4T + t*4 + k) — the NHWC order IS the reference's (H, W, A) enumeration; anchors [A, 4T] fp64 device
 * (generate_anchors.py); out rows [4T+1] (boxes, score) in descending score, image b at
 * out + b*out_batch_stride, count at counts[b*counts_stride].  act_f32: 1 fp32, 0 bf16.
 * time_major != 0 (3-D RPN head, lib/modeling/model_builder.py:509-563): logits [B, T, H, W, ld_s] with A
 * channels per frame are averaged over T (TimePool 'avg'), deltas [B, T, H, W, ld_d] hold a*4+k per frame.
 * workspace: dt_rpn_workspace_bytes (one u32 key per anchor). */
typedef struct dt_rpn_level {
  const void* logits; const void* deltas; const double* anchors;
  int ld_s, ld_d, H, W;
  double feat_stride;
  float* out; int* counts;
} dt_rpn_level;
int dt_rpn_workspace_bytes(int B, int nlevels, const int* Hs, const int* Ws, int A, size_t* bytes /*host out*/);
int dt_rpn_proposals_multi(const dt_rpn_level* levels /*host*/, int nlevels, int act_f32, int B, int A, int T,
                           const float* im_info, int pre_nms_topn, float min_size, double bbox_xform_clip,
                           long long out_batch_stride, int counts_stride, int time_major, void* workspace,
                           size_t workspace_bytes, void* stream);

/* collect (lib/ops/collect_and_distribute_fpn_rpn_proposals.py:44-62): props [B, L, K, 4T+1],
 * keep [B*L, K] / nkeep [B*L] from dt_nms_batched -> rois [B, R, 4T+1] (col 0 = image index),
 * roi_scores [B, R], roi_counts [B]; top post_nms_topn by score over the level concatenation. */
int dt_collect_rpn(const float* props, const int* keep, const int* nkeep, int B, int L, int K, int T,
                   int post_nms_topn, float* rois, float* roi_scores, int* roi_counts, int R,
                   void* stream);

/* distribute (same file :65-87; lib/modeling/FPN.py:349-360): levels[i] in [k_min, k_max] from the
 * mean-over-frames '+1' area of rois[i, col0 : col0+4T]; idx_restore (may be NULL) is the
 * reference's rois_idx_restore_int32; level_counts [k_max-k_min+1] (may be NULL). n_dev may be NULL. */
int dt_distribute_fpn(const float* rois, int n_max, const int* n_dev, int ld, int col0, int T, int k_min,
                      int k_max, float canonical_scale, float canonical_level, int* levels,
                      int* idx_restore, int* level_counts, void* stream);

/* lib/core/test.py:211-252 + :760-766: softmax(cls_logits), boxes = rois / im_scale,
 * bbox_transform(weights4 [host]), clip to the original image (im_hw [B,2] = h, w), keep
 * score > score_thresh per class j >= 1.  dets [B, C-1, R, 4T+1] compacted, det_counts [B*(C-1)]. */
int dt_box_decode(const float* rois, const int* roi_counts, int B, int R, int T, const float* cls_logits,
                  int ld_c, const float* bbox_deltas, int ld_b, int num_classes, const float* im_info,
                  const float* im_hw, const float* weights4, double bbox_xform_clip, float score_thresh,
                  float* dets, int* det_counts, void* stream);

/* lib/core/test.py:76-113 (_get_rois_blob / _project_im_rois) for the keypoint head: rois [n, ncols+1] =
 * (image index, boxes[i, :ncols] * im_scale) with the product in fp64, stored fp32 (what numpy computes).
 * boxes [n, ldb]; image index = bidx[i] (fp32, may be NULL) else i / per_image. */
int dt_scale_rois(const float* boxes, int ldb, int n, int ncols, const float* bidx, int per_image, double im_scale,
                  float* rois, void* stream);

/* lib/core/test.py:768-800: gather dets[keep] per class and apply the DETECTIONS_PER_IM score
 * threshold over all classes.  out [B, C-1, cap, 4T+1]; out_counts [B*(C-1)] is the reference's count and
 * may exceed cap when scores tie at the threshold (rows beyond cap are not written). */
int dt_limit_detections(const float* dets, const int* keep, const int* nkeep, int B, int num_classes, int R,
                        int T, int max_per_im, float* out, int* out_counts, int cap, void* stream);

/* Test-time augmentation (lib/core/test.py:255-414, 630-747), 2-D boxes.  A flip maps x to the original image by
 * flip_boxes (lib/utils/boxes.py:275-282): x1' = (W - x2) - 1, x2' = (W - x1) - 1 in fp32 with two roundings. */
#define DT_AUG_MAX_VIEWS 16
#define DT_KD_AUG_MAX_K 64

/* Union of V views' compacted per-class detections (dt_box_decode's dets [B, C-1, R, 5] and counts [B*(C-1)], device
 * pointers in the host arrays dets / counts), in view order, each view with flip[v] != 0 flipped back with the image
 * width im_w[b * ld_w] (device).  out [B, C-1, V*R, 5], out_counts [B*(C-1)]: the layout dt_nms_batched takes.
 * V*R <= DT_NMS_MAX_BOXES.  No host synchronisation. */
int dt_aug_merge_dets(const float* const* dets, const int* const* counts, const int* flip, int V, int B, int num_classes,
                      int R, const float* im_w, int ld_w, float* out, int* out_counts, void* stream);

/* A keypoint view's RoIs: rois [n, 5] = (i / per_image, box' * im_scale), box' = boxes[i, :4] flipped (flip != 0, width
 * im_w[(i / per_image) * ld_w]) or as is; the product in fp64, stored fp32.  With flip 0 this equals dt_scale_rois
 * (ncols 4, bidx NULL) byte for byte; im_w may then be NULL. */
int dt_aug_scale_rois(const float* boxes, int ldb, int n, int flip, const float* im_w, int ld_w, int per_image,
                      double im_scale, float* rois, void* stream);

/* ---- dense_ops.cu -------------------------------------------------------- */

/* lib/utils/blob.py:40-90 + lib/core/test.py:43-74.  frames [F, H, W, 3] u8 BGR ->
 * out [F, Hp, Wp, Cp] (bf16 or fp32): (pixel - mean3) bilinearly resized by im_scale to Hr x Wr,
 * zero padded (Cp >= 3 channels, spatially to Hp x Wp) and framed by border_y zero rows / border_x
 * zero pixels on every side: out is [F, Hp + 2*border_y, Wp + 2*border_x, Cp] (dt_conv1_7x7s2 wants 3 / 4).
 * row_planes != 0: the padded rows are de-interleaved by parity, out [F, 2, (Hp + 2*border_y)/2, Wt, Cp]
 * with padded row r at [r & 1][r >> 1] (what dt_conv1_7x7s2 reads: its stride-2 row walk becomes contiguous).
 * out_f32: 0 bf16, 1 fp32 rounded to tf32 (kind::tf32 consumer), 2 raw fp32 (dt_conv1_7x7s2_f32),
 * 3 bf16 split pixel (Cp == 8): channels [hi(b,g,r) | lo(b,g,r) | 0 0], hi = bf16(v), lo = bf16(v - hi). */
int dt_prep_clip(const unsigned char* frames, int F, int H, int W, const float* mean3, double im_scale,
                 int Hr, int Wr, int Hp, int Wp, int Cp, int border_y, int border_x, int row_planes,
                 int out_f32, void* out, void* stream);

/* The training minibatch blob (lib/roi_data/minibatch.py:66-90 _get_image_blob + blob.py im_list_to_blob): B clips of
 * T frames, clip b = frames[b] [T, H[b], W[b], 3] u8 BGR (device pointer), resized by im_scale[b] to Hr[b] x Wr[b], its
 * source frames mirrored horizontally first when flip[b] != 0, all zero padded to ONE Hp x Wp.  Host arrays of B
 * entries, copied into the kernel's parameters (no H2D copy, no allocation); 1 <= B <= DT_PREP_MAX_CLIPS.
 * Cp, border_y / border_x, row_planes and out_f32 as dt_prep_clip; out is [B*T, ...] in dt_prep_clip's layout, and
 * with flip 0 clip b's slice equals dt_prep_clip of that clip byte for byte (the per-pixel code is shared). */
#define DT_PREP_MAX_CLIPS 16
int dt_prep_batch(const unsigned char* const* frames, const int* H, const int* W, const double* im_scale,
                  const int* Hr, const int* Wr, const int* flip, int B, int T, const float* mean3, int Hp, int Wp,
                  int Cp, int border_y, int border_x, int row_planes, int out_f32, void* out, void* stream);

/* Caffe2 MaxPool kernels [1,k,k] strides [1,s,s] pads [0,p,p] on NHWC (N = B*T frames).
 * x3 != 0: split storage, rows are [hi(C) | lo(C)] pairs at ld/2 (tf32 pairs in fp32 tensors, bf16 pairs in bf16). */
int dt_maxpool2d(const void* x, int N, int H, int W, int C, int ldx, int k, int s, int p, int f32, int x3,
                 void* y, int ldy, void* stream);

/* RoIFeatureTransform (lib/modeling/detector.py:216-310): RoIAlign (Detectron semantics,
 * non-"aligned") over FPN levels with tube -> frame routing and the un-shuffle fused.
 * feats/Hs/Ws/scales: host arrays [nlevels] (feature l is [n_images*T, Hs[l], Ws[l], ldf]);
 * rois [R, ldr] (col 0 image index, then 4*T), levels [R] (NULL if nlevels == 1);
 * out [R, T, P, P, C]; rows >= *n_dev are zero-filled.  round_tf32: round fp32 outputs to tf32
 * (when they feed a DT_DTYPE_TF32 GEMM; prep_clip does the same for its fp32 output).
 * x3_mode (split storage, features are [hi | lo] rows, fp32 or bf16): 1 = out [R,T,P,P,2C] per-position pairs,
 * 2 = out [R, 2, T*P*P*C] planar hi / lo blocks (input of the FC head). */
int dt_roi_align(const void* const* feats, const int* Hs, const int* Ws, const float* scales, int nlevels,
                 int k_min, int C, int ldf, int f32, const float* rois, int ldr, const int* n_dev, int R,
                 int T, const int* levels, int P, int sampling_ratio, int round_tf32, int x3_mode, void* out,
                 void* stream);

/* BilinearInterpolation (lib/modeling/detector.py:348-380) + heatmaps_to_keypoints
 * (lib/utils/keypoints.py:94-149).  lowres [D*T, S, S, ldl] fp32 with channel (py*2+px)*K + k =
 * kps_score_lowres[k] at pixel (2y+py, 2x+px); boxes [D, ldb] image-space (4*T columns);
 * heatmaps (may be NULL) [D, T*K, 4S, 4S]; xy_preds [D, 4, T*K] = (x, y, logit, prob). */
int dt_keypoint_decode(const float* lowres, int ldl, int S, int K, int T, const float* boxes, int ldb,
                       const int* n_dev, int D, int min_size, float* heatmaps, float* xy_preds,
                       void* stream);

/* dt_keypoint_decode of V test-time views combined (lib/core/test.py:686-747), 2-D heads (T = 1).  View v's low-res maps
 * are lowres + v * view_stride ([D, S, S, ldl] as above); every view's 4S x 4S map is built as dt_keypoint_decode does,
 * a view with flip[v] != 0 through flip_heatmaps (lib/utils/keypoints.py:81-91: joint perm[k], x mirrored).  hm_max 0
 * (HM_AVG): fp32 sum in view order, then / V; 1 (HM_MAX): the maximum.  The combined map is decoded against boxes;
 * heatmaps (may be NULL) [D, K, 4S, 4S] receives it.  flip [V] and perm [K] are host arrays; V <= DT_AUG_MAX_VIEWS. */
int dt_keypoint_decode_aug(const float* lowres, long long view_stride, int ldl, int S, int K, int V, const int* flip,
                           const int* perm, int hm_max, const float* boxes, int ldb, const int* n_dev, int D, int min_size,
                           float* heatmaps, float* xy_preds, void* stream);

/* split-storage modes' conv1: exact fp32 7x7/2 conv + AffineChannel + ReLU on the raw fp32 blob [F, Hp, Wp, Cp];
 * w [7][7][3][64] fp32; y [F, Hp/2, Wp/2, 128] = [hi(64) | lo(64)]: fp32 tf32 pairs (out_bf16 = 0) or bf16
 * pairs (out_bf16 = 1). */
int dt_conv1_7x7s2_f32(const float* blob, int F, int Hp, int Wp, int Cp, const float* w, const float* scale,
                       const float* bias, int out_bf16, void* y, void* stream);

/* 3-D box head glue.  dt_spatial_mean: ReduceBackMean over W then H
 * (lib/modeling/ResNet3D.py:321-322), x [N, H, W, ldx] -> y [N, ldy] (first C channels).
 * dt_fold_tube_heads: per-frame head outputs in [R*T, ld] = [C cls logits | 4C deltas (c*4+k)] ->
 * cls [R, C] = mean over T, bbox [R, C*T*4] with channel c*4T + t*4 + k
 * (lib/modeling/model_builder.py:427-473). */
int dt_spatial_mean(const void* x, int N, int H, int W, int C, int ldx, int f32, int round_tf32, int x3,
                    void* y, int ldy, void* stream);

/* TimePool 'avg' body/head link (lib/modeling/model_builder.py:1024-1042, lib/modeling/detector.py:559-576):
 * x [B, T, P, ldx] -> y [B, P, ldy], mean over the T frames (fp32 sum in frame order, then / T); P = H*W.
 * f32 / round_tf32 / x3 as in dt_spatial_mean. */
int dt_time_mean(const void* x, int B, int T, long long P, int C, int ldx, int f32, int round_tf32, int x3,
                 void* y, int ldy, void* stream);
int dt_fold_tube_heads(const float* in, int ld, int R, int T, int C, float* cls, float* bbox, void* stream);

/* ---- train_ops.cu (training step, BASELINE.json configs[4]) --------------------------------------------------
 * The reference builds its backward graph with model.AddGradientOperators and updates with MomentumSGDUpdate after an
 * NCCL / muji all-reduce of the per-GPU gradients (lib/modeling/model_builder.py:908-985).  Here:
 *   dgrad   of a stride-1 'same' conv = dt_conv3d of the gradient with the flipped, transposed filter (w_dgrad below);
 *           stride-2 pointwise convs: dt_conv3d on the coarse map + dt_scatter_stride2
 *   wgrad   dt_wgrad_nhwc, both operands read straight from the NDHWC gradient and saved input
 *   the elementwise joins (Relu / Sum / AffineChannelNd gradient, lib/ops/affine_channel_nd_op.cu:73-92) dt_bwd_pointwise,
 *   the FPN top-down join dt_upsample_add_bwd, the update dt_sgd_update_multi (every parameter tensor in one launch).
 *   All tensors bf16 unless noted. */

/* Filter gradient of a 'same' conv (odd kT/kH/kW, pads k/2): dW [kT*kH*kW][Cout][Cin] fp32 +=
 * sum_{n,t,h,w} gz[n,t,h,w,co] * x[n, t+kt-pT, h+kh-pH, w+kw-pW, ci], read straight from the NDHWC tensors:
 * gz [N, T, Ho, Wo, ld_g] (first Cout channels), x [N, T, Hi, Wi, ld_x] (first Cin channels), both bf16.  Positions are
 * the K axis of MN-major wgmma operands staged by 5-D TMA boxes; the tap is a coordinate shift (zero fill = padding).
 * sH / sW > 1 only for pointwise convs (Ho = ceil(Hi / sH)).  dW (8-byte aligned) is ACCUMULATED into (split-K partial
 * sums, red.global): the caller zeroes it (dt_memset). */
int dt_wgrad_nhwc(const void* gz, int ld_g, const void* x, int ld_x, int N, int T, int Ho, int Wo, int Hi, int Wi, int Cout, int Cin,
                  int kT, int kH, int kW, int sH, int sW, float* dW, void* stream);

/* Host-only planning query of dt_wgrad_nhwc (same shape arguments, no device work, usable without a GPU): the 64-position
 * box TW x TH x TT frames x TB images, the box counts per axis (nW, nH, nT, nN; the K axis has nW*nH*nT*nN k-blocks),
 * column tile BN, taps, output-channel / input-channel tiles, the K split (CTA ks of a (tap, tile) unit sums k-blocks
 * [total*ks/ksplit, total*(ks+1)/ksplit)), the grid (taps * tiles_m * tiles_n * ksplit CTAs) and the dynamic shared memory. */
typedef struct dt_wgrad_plan_t {
  int TW, TH, TT, TB;
  int nW, nH, nT, nN;
  int BN, taps, tiles_m, tiles_n, ksplit, grid, smem_bytes;
} dt_wgrad_plan_t;
int dt_wgrad_nhwc_plan(int ld_g, int ld_x, int N, int T, int Ho, int Wo, int Hi, int Wi, int Cout, int Cin, int kT, int kH, int kW,
                       int sH, int sW, dt_wgrad_plan_t* plan /*host out*/);

/* out = (g1 + g2?) * [y > 0]? * scale[c]? over [rows, C] (any of g2 / y / scale may be NULL) */
int dt_bwd_pointwise(const void* g1, const void* g2, const void* y, const float* scale, long long rows, int C, void* out,
                     void* stream);
/* The same with a second output of the same masked sum, out2 = (g1 + g2) * [y > 0] * scale2[c] (scale2 NULL: no scale): the two
 * consumers of a block output's gradient (branch2c and the shortcut) from one read of the three inputs. */
int dt_bwd_pointwise2(const void* g1, const void* g2, const void* y, const float* scale, long long rows, int C, void* out,
                      const float* scale2, void* out2, void* stream);

/* out[f,h,w,c] = coarse_in?[f,h,w,c] + sum of the 2x2 children fine[f, 2h+dy, 2w+dx, c]; fine is [F, 2Hc, 2Wc, C] */
int dt_upsample_add_bwd(const void* fine, const void* coarse_in, int F, int Hc, int Wc, int C, void* out, void* stream);

/* out [F, H, W, C] = zeros except out[f, 2h, 2w] = src[f, h, w]; src [F, ceil(H/2), ceil(W/2), C] */
int dt_scatter_stride2(const void* src, int F, int Hs, int Ws, int H, int W, int C, void* out, void* stream);

/* Caffe2 MomentumSGDUpdate + weight decay (model_builder.py:954-985) of EVERY parameter tensor in one launch:
 * g' = lr * (grad_scale * g + wd * w) + momentum * m;  m = g';  w -= g'.  Per item w / g / m are fp32 [taps][Cout][Cin]
 * (the packed order of dt_conv3d's filter); w_fwd_bf16 (may be NULL) receives the new filter as bf16 in the same order,
 * w_dgrad_bf16 (may be NULL) the dgrad filter [taps (flipped)][Cin][Cout].  items: device array of dt_sgd_item;
 * first_block [n_items]: device, exclusive prefix of taps * ceil(Cout/32) * ceil(Cin/32) per item; total_blocks = their
 * sum.  Per item the learning rate is lr * lr_mult and the weight decay wd * wd_mult (biases: 2x / 0,
 * model_builder.py:971-976). */
typedef struct dt_sgd_item {
  float* w; const float* g; float* m; void* w_fwd_bf16; void* w_dgrad_bf16;
  int taps, Cout, Cin, tiles_ci, tiles_co;
  float lr_mult, wd_mult;
} dt_sgd_item;
int dt_sgd_update_multi(const void* items, const int* first_block, int n_items, int total_blocks, float lr, float momentum, float wd,
                        float grad_scale, void* stream);

/* db [C] fp32 += column sums of g [rows, ld] bf16 (first C columns): the conv-bias gradient (caller zeroes db) */
int dt_bias_grad(const void* g, long long rows, int C, int ld, float* db, void* stream);

/* FPN RPN losses of one level and their gradient (lib/modeling/FPN.py:282-321; Detectron SigmoidCrossEntropyLoss with
 * normalize=0 and SmoothL1Loss with beta): out [rows, ld_o] fp32 = [A logits | 4A deltas (a*4+k)], labels [rows, A] int32
 * (-1 ignored), targets / inside_w / outside_w [rows, 4A] fp32; scale_cls = 1 / NUM_GPUS / RPN_BATCH_SIZE_PER_IM /
 * IMS_PER_BATCH, scale_box = 1 / NUM_GPUS / time_dim / batch.  grad [rows, ld_g] bf16 (same channel order, padding 0);
 * loss (may be NULL) [2] fp32 += (cls, bbox). */
int dt_rpn_loss_grad(const float* out, int ld_o, const int* labels, const float* targets, const float* inside_w,
                     const float* outside_w, long long rows, int A, float scale_cls, float scale_box, float beta, void* grad,
                     int ld_g, float* loss, void* stream);

/* Backward of the slice-center body/head link (lib/modeling/model_builder.py:1024-1042 SliceKeyFrame): out [B, T, frame_elems]
 * bf16 = src [B, frame_elems] in frame c, zero in every other frame. */
int dt_embed_frame(const void* src, int B, int T, long long frame_elems, int c, void* out, void* stream);

/* fp32 accumulator joins of the RoI-head backward: out (bf16) = g (bf16, may be NULL) + acc (fp32) */
int dt_grad_join_f32(const void* g, const float* acc, long long n, void* out, void* stream);

/* RoIAlign backward (the Caffe2 RoIAlignGradient the reference gets from AddGradientOperators for
 * lib/modeling/detector.py:216-310): grad [R, T, P, P, C] bf16 is scattered with the forward's bilinear weights into
 * fp32 accumulators dfeat[l] [Nimg*T, H_l, W_l, C] (caller zeroes them, 16-byte aligned; red.global.add.v4.f32).  Arguments as
 * dt_roi_align. */
int dt_roi_align_bwd(const void* grad, float* const* dfeats /*host array [nlevels] of device ptrs*/, const int* Hs, const int* Ws,
                     const float* scales, int nlevels, int k_min, int C, const float* rois, int ldr, const int* n_dev, int R,
                     int T, const int* levels, int P, int sampling_ratio, void* stream);

/* Fast R-CNN losses and their gradients (lib/modeling/model_builder.py:481-493: SoftmaxWithLoss(cls_score, labels_int32,
 * scale) + SmoothL1Loss(bbox_pred, targets, inside, outside, beta 1, scale)): out [rows, ld_o] fp32 = [C class logits |
 * 4C box deltas]; labels [rows] int32 (-1 = padding row, ignored); targets / inside_w / outside_w [rows, 4C] fp32.
 * Both losses average over the LIVE row count totals[0] (device; dt_sample_rois).  grad [rows, ld_g] bf16, padding 0;
 * loss (may be NULL) [2] += (cls, bbox); accuracy (may be NULL) [1] += correctly classified live rows. */
int dt_frcnn_loss_grad(const float* out, int ld_o, const int* labels, const float* targets, const float* inside_w,
                       const float* outside_w, int rows, int C, const float* totals, float scale_cls, float scale_box, void* grad,
                       int ld_g, float* loss, float* accuracy, void* stream);

/* Keypoint heat-map loss and gradient (lib/modeling/model_builder.py:873-888 on top of :755-870): per (RoI, joint) the 2S x 2S
 * low-resolution map (sub-pixel packed conv output low [D, S, S, ld], channel (py*2+px)*K + k) is upsampled 2x by the fixed
 * bilinear ConvTranspose (BilinearInterpolation, lib/modeling/detector.py:348-380), SoftmaxWithLoss over the (4S)^2 positions
 * with the location label and weight, averaged over the weight sum totals[1] (device) and scaled; the gradient is taken back
 * through the upsampling and written in the same packed layout: grad [D, S, S, ld_g] bf16 (caller zeroes padding channels). */
int dt_kps_loss_grad(const float* low, int ld, int S, int K, int D, const int* locations, const float* weights, const float* totals,
                     float scale, void* grad, int ld_g, float* loss, void* stream);

/* Keeps the sub-pixel form of the k4-s2-p1 ConvTranspose consistent during training: zeroes the gradient of the structural
 * zeros of the 3x3-footprint filter gW [9][ldc][Cin] (and of the padding filters >= 4K) and ties the 4 copies of each bias
 * gradient gb [ldc] (their sum, written to all four). */
int dt_subpixel_grad_fix(float* gW, float* gb, int K, int Cin, int ldc, void* stream);

/* ---- jpeg.cu (frame decode on the device; SURVEY.md §8 f3) ----------------------------------------------------------
 * jpegs / sizes: HOST arrays of n JPEG byte streams (the file contents cv2.imread would parse, lib/utils/image.py:51-63), all
 * H x W; out_bgr: DEVICE [n, H, W, 3] uint8 in cv2's BGR interleaved order.  Decoded through nvJPEG (library code, dlopen'ed
 * on first use: dt_jpeg_available() == 0 and a clean error without it).  Host-side entropy decoding on the calling thread,
 * GPU work on `stream`; one decoder per host thread, so loader threads may call it concurrently. */
int dt_jpeg_available(void);
int dt_jpeg_decode(const unsigned char* const* jpegs, const size_t* sizes, int n, int H, int W, void* out_bgr, void* stream);

/* ---- targets.cu (training target generators on the device; SURVEY.md §8 f1) ---------------------------------------
 * Random draws are the counter-based choice / randint of oracle/targets.py (seed, stream, image, index). */
typedef struct dt_rpn_target_level {
  int H, W;
  double feat_stride;
  const double* anchors;           /* [A, 4T] cell anchors (generate_anchors.py) */
  int* labels;                     /* out [B, H, W, A]  (1 fg, 0 bg, -1 ignore) */
  float* bbox_targets;             /* out [B, H, W, 4A] */
  float* inside_weights;           /* out [B, H, W, 4A] */
  float* outside_weights;          /* out [B, H, W, 4A] */
  int* vis_labels;                 /* out [B, H, W, T*A] (rpn_vis_labels_int32_wide: label x frame visibility), may be NULL */
} dt_rpn_target_level;
int dt_rpn_targets_workspace_bytes(int B, int n_levels, const int* Hs, const int* Ws, int A, int Gmax, size_t* bytes /*host out*/);
/* lib/roi_data/rpn.py:206-381 for every image of the batch and every FPN level, boxes (T = 1) or tubes (T <= 4 frames): gt_boxes
 * [B, Gmax, 4T] fp32 in ORIGINAL image coordinates (non-crowd, gt_classes > 0), gt_visible [B, Gmax, T] bytes (track_visible;
 * NULL: all visible), gt_counts [B], im_info [B, 3] = (blob h, blob w, scale).  Per level the anchors are [A, 4T] (the 2-D anchor
 * replicated over the frames), the box blobs [B, H, W, 4T*A] (channel a*4T + t*4 + k).  Tubes: IoU = mean over the frames; the
 * box targets follow the reference's fp64-promoted tube arithmetic (utils/boxes.py:28-58,233-240), rounded to fp32 once. */
int dt_rpn_targets(const dt_rpn_target_level* levels /*host*/, int n_levels, int A, int T, int B, const float* gt_boxes,
                   const unsigned char* gt_visible, const int* gt_counts, int Gmax, const float* im_info, float straddle_thresh,
                   float positive_overlap, float negative_overlap, int batch_size_per_im, float fg_fraction, unsigned long long seed,
                   void* workspace, size_t workspace_bytes, void* stream);
/* add_proposals + _sample_rois + add_keypoint_rcnn_blobs (lib/datasets/json_dataset.py:423-534, lib/roi_data/fast_rcnn.py:118-238,
 * lib/roi_data/keypoint_rcnn.py:24-99) for every image: rois [B, R, 5] / roi_scores [B, R] / roi_counts [B] = dt_collect_rpn's
 * per-image output (descending score); only the batch-wide top post_nms_topn are used (the training branch of collect).
 * gt_* [B, Gmax, ...]: boxes fp32 (original coordinates, ALL gt incl. crowd), classes, crowd flags, keypoints [B,Gmax,3,K] int32
 * (K joints per frame).
 * Outputs (fixed capacity, padding rows have label -1 / zero weights): rois_out [B, batch, 4T+1], labels [B, batch],
 * bbox_targets / inside / outside [B, batch, 4T*num_classes], out_counts [B]; kp_rois [B, kcap, 4T+1] (may be NULL),
 * kp_locations [B, kcap, K*T] int32, kp_weights [B, kcap, K*T], kp_counts [B]; totals [2] += (live RoIs, keypoint weight sum).
 * T > 1 (tubes, T <= 4): rois [B, R, 4T+1], gt boxes [B, Gmax, 4T], gt keypoints [B, Gmax, 3, K*T]; tube IoU is the mean over the
 * frames, box targets are computed frame by frame in the reference's fp64-promoted arithmetic, heat-map labels per frame. */
int dt_sample_rois(const float* rois, const float* roi_scores, const int* roi_counts, int B, int R, int post_nms_topn,
                   const float* gt_boxes, const int* gt_classes, const int* gt_crowd, const int* gt_keypoints,
                   const int* gt_counts, int Gmax, int K, int T, const float* im_info, int num_classes, int batch_size_per_im,
                   float fg_fraction, float fg_thresh, float bg_thresh_hi, float bg_thresh_lo, const float* bbox_reg_weights /*host [4]*/,
                   int heatmap_size, unsigned long long seed, float* rois_out, int* labels, float* bbox_targets,
                   float* inside_weights, float* outside_weights, int* out_counts, float* kp_rois, int* kp_locations,
                   float* kp_weights, int* kp_counts, int kcap, float* totals, void* stream);

/* ---- flow.cu: TRACKING.FLOW_SMOOTHING_ON (lib/core/tracking_engine.py:401-643) --------------------------- */

#define DT_FARNEBACK_GAUSSIAN 256       /* cv2.OPTFLOW_FARNEBACK_GAUSSIAN, the only window implemented */
#define DT_FLOW_MAX_CONTEXT 16          /* TRACKING.FLOW_SMOOTHING.N_CONTEXT_FRAMES */

/* cvtColor(BGR2GRAY) of npix uint8 BGR pixels in OpenCV 4.x's 15-bit fixed point (bit-exact). */
int dt_bgr_to_gray(const uint8_t* bgr, long long npix, uint8_t* gray, void* stream);
/* Workspace of dt_farneback_flow for nframes frames of H x W and npairs pairs. */
int dt_farneback_workspace_bytes(int H, int W, int nframes, int npairs, size_t* bytes /*host out*/);
/* cv2.calcOpticalFlowFarneback(gray[a], gray[b], None, pyr_scale, levels, winsize, iterations, poly_n, poly_sigma, flags)
 * (OpenCV 4.x CPU algorithm) for every pair (a, b) of pairs [npairs, 2] (device int32 frame indices) at once.  frames
 * [nframes, H, W, 3] uint8 BGR, converted to gray as dt_bgr_to_gray does; flows out [npairs, H, W, 2] fp32.  flags must
 * be DT_FARNEBACK_GAUSSIAN, poly_n 5 or 7, winsize <= 347. */
int dt_farneback_flow(const uint8_t* frames, int nframes, int H, int W, const int* pairs, int npairs, double pyr_scale,
                      int levels, int winsize, int iterations, int poly_n, double poly_sigma, int flags, float* flows,
                      void* workspace, size_t workspace_bytes, void* stream);
/* out[p] = np.abs(flows[p]).mean() for flows [npairs, H, W, 2] fp32: numpy's fp32 pairwise sum, bit for bit. */
int dt_flow_mean_abs(const float* flows, int npairs, int H, int W, float* out, void* stream);
/* _shift_poses + _combine_shifted_poses (:401-546), bit-exact, for F frames of packed videos: poses [F, dmax, 4, K],
 * boxes [F, dmax, 5] (T = 1), counts [F], tracks [F, dmax] (dt_assign_track_ids' output), is_start [F] (first frame of a
 * video).  flows [F] (device array of device pointers): the flow of frame f -> f + 1 as [H, W, 2] fp32 with flow_hw [F, 2]
 * = (H, W); no_flow [F] marks a pair that moves nothing (no flow, or a shot boundary).  out_tracks [F, omax] / out_counts
 * [F]: the output track order of each frame (computed on the host); out_poses [F, omax, 4, K], out_boxes [F, omax, 5]. */
int dt_flow_smooth_poses(const float* poses, const float* boxes, const int* counts, const int* tracks,
                         const unsigned char* is_start, int F, int dmax, int K, const float* const* flows, const int* flow_hw,
                         const unsigned char* no_flow, int n_context, const int* out_tracks, const int* out_counts, int omax,
                         float* out_poses, float* out_boxes, void* stream);


/* ---- poseval.cu: PoseTrack evaluation (lib/datasets/posetrack/poseval/py/evaluate_simple.py) ---------------------- */

#define DT_PT_JOINTS 15             /* PoseTrack / MPII joints (eval_helpers.Joint) */
#define DT_PT_MAX_GT 64             /* GT people per frame */
#define DT_PT_MAX_MAP_IDS 4096      /* distinct GT track ids one CLEAR-MOT frame list may see */

/* assignGTmulti (eval_helpers.py:423-637) for every frame, one CTA per frame.  Frame f owns GT rows
 * [gt_off[f], gt_off[f+1]) and prediction rows [pr_off[f], pr_off[f+1]) (at most max_gt <= DT_PT_MAX_GT and
 * max_pr <= DT_LSA_MAX_DIM of them); pair_off [nframes] = sum over earlier frames of (predictions x GT).
 * gt_rect [NG, 4] fp64 head box (x1, y1, x2, y2); gt_kp [NG, 15, 3] fp64 (x, y, present); pr_kp [NP, 15, 4] fp64
 * (x, y, score, present).  Outputs: labels [NP, 15] (-1: joint not predicted, else the AP label 0 / 1); ngt [15, nframes]
 * annotated GT joints; dist [pair_off[F], 15] fp64: the distance of (prediction p, GT g, joint j) of frame f at
 * (pair_off[f] + p * nG + g) * 15 + j where it matches (<= 0.5), NaN elsewhere (only frames with both are written). */
int dt_posetrack_assign(const int* gt_off, const int* pr_off, const long long* pair_off, int nframes, const double* gt_rect,
                        const double* gt_kp, const double* pr_kp, int max_gt, int max_pr, signed char* labels, int* ngt,
                        double* dist, void* stream);
/* The upper-bound view of the predictions (assignGTmulti with computeUpperBound, eval_helpers.py:559-573) for
 * dt_posetrack_mot: in a frame with both GT and predictions only the predictions some GT selected (prToGT, recomputed from
 * dist) are kept, in ascending GT order, with that GT's track id; other frames are copied.  Outputs: ub_pr_off [nframes + 1],
 * ub_pair_off [nframes + 1], ub_pr_kp [NP, 15, 4], ub_pr_tid [NP] and ub_dist [pair_off[nframes], 15], each filled up to
 * the view's own totals. */
int dt_posetrack_upper_bound(const int* gt_off, const int* pr_off, const long long* pair_off, int nframes, const double* gt_kp,
                             const int* gt_tid, const double* pr_kp, const int* pr_tid, const double* dist, int max_gt, int max_pr,
                             int* ub_pr_off, long long* ub_pair_off, double* ub_pr_kp, int* ub_pr_tid, double* ub_dist,
                             void* stream);
/* Workspace of dt_posetrack_ap for nentries scores in all. */
int dt_posetrack_ap_workspace_bytes(long long nentries, size_t* bytes /*host out*/);
/* evaluateAP.computeMetrics (computeRPC + VOCap) of every segment: segs [nseg, 3] = (joint, first frame, end frame),
 * the scores of that joint's predicted rows of those frames, placed at seg_off [nseg + 1] (nentries = seg_off[nseg]).
 * Scores are sorted descending, ties by row (the reference's concatenation order).  out [nseg, 3] fp64 = (AP, last
 * precision, last recall) x 100, zero for an empty segment; IEEE 0/0 where the joint has no GT. */
int dt_posetrack_ap(const double* pr_kp, const signed char* labels, const int* ngt, int nframes, const int* pr_off,
                    const int* segs, const int* seg_off, int nseg, long long nentries, double* out, void* workspace,
                    size_t workspace_bytes, void* stream);
/* Dynamic shared memory of one dt_posetrack_mot warp (the caller checks it against the device's 227 KB). */
int dt_posetrack_mot_smem_bytes(int max_gt, int max_pr, int map_cap, size_t* bytes /*host out*/);
/* MOTAccumulator.update (py-motmetrics mot.py:90-191) over frame lists, one warp per (list, joint): list l feeds update()
 * the MOT inputs of frames list_frames[list_off[l] .. list_off[l+1]) in order, built from dt_posetrack_assign's dist and
 * the rows that have the joint (track ids gt_tid [NG], pr_tid [NP]).  max_gt / max_pr bound those rows per frame and
 * joint, map_cap the distinct GT track ids of a list.  Outputs: counts [nlists, 15, 4] int32 = MATCH, SWITCH, FP, MISS;
 * sumd [nlists, 15] fp64 = sum of the MATCH / SWITCH distances; status [nlists * 15] (may be NULL) non-zero where a bound
 * was exceeded. */
int dt_posetrack_mot(const int* gt_off, const int* pr_off, const long long* pair_off, const double* gt_kp, const int* gt_tid,
                     const double* pr_kp, const int* pr_tid, const double* dist, const int* list_off, const int* list_frames,
                     int nlists, int max_gt, int max_pr, int map_cap, int* counts, double* sumd, int* status, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DT_B200_H_ */
