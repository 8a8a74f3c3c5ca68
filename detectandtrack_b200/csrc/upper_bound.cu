// The tracker's upper-bound experiments (lib/core/tracking_engine.py:272-350, TRACKING.DEBUG.UPPER_BOUND*): the detections
// of every frame matched against that frame's GT, then the GT track ids, boxes and keypoints copied onto them.
//
// Layout shared by both launches: the frames of the dataset interleaved with their GT, entry 2f = the GT of frame f (boxes
// padded with a zero score column, keypoints [3, K] in rows 0..2 of a [R, K] slot), entry 2f + 1 = the detections of frame
// f.  dt_match_frames reads the same packing for the bbox-only matches (is_start on every GT entry).
#include "common.cuh"
#include "box_math.cuh"
#include "../../include/dt_b200.h"

namespace dt {

// 'pose-pck' cost (lib/utils/keypoints.py:266-291) with the GT pose as kps_a.  The reference's GT keypoints are int32
// (json_dataset.py stores them so), which numpy promotes to fp64 against the fp32 detections: the head size, the distances
// and the threshold test are all fp64 here.  a = GT [R, K] (integer-valued), b = detection [R, K].
__device__ __forceinline__ double pck_cost_gt(const float* __restrict__ a, const float* __restrict__ b, int K, int ht, int hb,
                                              double thr) {
  const double hx = __dsub_rn((double)a[ht], (double)a[hb]), hy = __dsub_rn((double)a[K + ht], (double)a[K + hb]);
  const double head = __dadd_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(hx, hx), __dmul_rn(hy, hy))), 1.0);
  int cnt = 0;
  for (int k = 0; k < K; ++k) {
    const double dx = __dsub_rn((double)a[k], (double)b[k]), dy = __dsub_rn((double)a[K + k], (double)b[K + k]);
    const double nd = __ddiv_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy))), head);
    cnt += nd < thr ? 1 : 0;
  }
  return 1.0 - (double)cnt / (double)K;
}

// cost [F, dmax, dmax] fp64 (rows = GT, cols = detections) = fp32(w_iou * (1 - IoU)) + w_pck * pck as
// _compute_distance_matrix sums its terms (tracking_engine.py:158-181); entries beyond the counts are 0.
__global__ void gt_costs_kernel(const float* __restrict__ boxes, int ld, int T, const float* __restrict__ poses, int R, int K,
                                int ht, int hb, double thr, const int* __restrict__ counts, int nframes, int dmax, float w_iou,
                                double w_pck, double* __restrict__ cost) {
  const int f = blockIdx.x;
  const int P = min(counts[2 * f], dmax), Q = min(counts[2 * f + 1], dmax);
  double* C = cost + (size_t)f * dmax * dmax;
  const size_t ldp = (size_t)R * K;
  for (int e = threadIdx.x; e < dmax * dmax; e += blockDim.x) {
    const int p = e / dmax, q = e - p * dmax;
    double acc = 0.0;
    if (p < P && q < Q) {
      if (w_iou != 0.f) {
        const float* pb = boxes + ((size_t)(2 * f) * dmax + p) * ld;
        const float* qb = boxes + ((size_t)(2 * f + 1) * dmax + q) * ld;
        float s = iou_pair_ref(pb, qb);
        for (int t = 1; t < T; ++t) s = __fadd_rn(s, iou_pair_ref(pb + 4 * t, qb + 4 * t));
        acc = (double)__fmul_rn(__fsub_rn(1.f, __fdiv_rn(s, (float)T)), w_iou);
      }
      if (w_pck != 0.0)
        acc = __dadd_rn(acc, __dmul_rn(pck_cost_gt(poses + ((size_t)(2 * f) * dmax + p) * ldp,
                                                   poses + ((size_t)(2 * f + 1) * dmax + q) * ldp, K, ht, hb, thr), w_pck));
    }
    C[e] = acc;
  }
}

// One CTA per frame (tracking_engine.py:282-338).  matches [f * ldm + q] = the GT row detection q took under the
// configured cost (UPPER_BOUND), matches_gt [f * ldmg + q] the one it took under the bbox Hungarian match
// (UPPER_BOUND_5_GT_KPS_ONLY); either may be NULL.  Under DT_UB_COMPACT only the matched detections are kept, in
// ascending order, with the GT's track id.  Pose rows: DT_UB_GT_KPS puts the matched GT's rows 0..2 (row 2 only with
// DT_UB_ONLY_CONF) on every kept row, then matches_gt puts its GT's rows 0..2 on every detection it matched: the
// reference's kept rows alias the poses _5 overwrites, so where both apply _5 wins.
__global__ void ub_apply_kernel(const float* __restrict__ boxes, int ld, const float* __restrict__ poses, int R, int K,
                                const int* __restrict__ counts, const int* __restrict__ gt_tid, int dmax,
                                const int* __restrict__ matches, int ldm, const int* __restrict__ matches_gt, int ldmg,
                                int flags, float* __restrict__ out_boxes, float* __restrict__ out_poses, int* __restrict__ out_tid,
                                int* __restrict__ out_counts) {
  __shared__ int s_src[DT_LSA_MAX_DIM];                       // output row -> detection row
  __shared__ int s_n;
  const int f = blockIdx.x, tid = threadIdx.x;
  const int G = min(counts[2 * f], dmax), n = min(counts[2 * f + 1], dmax);
  const bool compact = (flags & DT_UB_COMPACT) != 0;
  const int* m = matches ? matches + (size_t)f * ldm : nullptr;
  const int* mg = matches_gt ? matches_gt + (size_t)f * ldmg : nullptr;
  if (tid < 32) {                                             // stable compaction by one warp
    int base = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
      const int i = i0 + tid;
      const bool keep = i < n && (!compact || (m[i] >= 0 && m[i] < G));
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if (keep) s_src[base + __popc(bal & ((1u << tid) - 1))] = i;
      base += __popc(bal);
    }
    if (tid == 0) s_n = base;
  }
  __syncthreads();
  const int no = s_n;
  const float* gtb = boxes + (size_t)(2 * f) * dmax * ld;
  const float* db = boxes + (size_t)(2 * f + 1) * dmax * ld;
  const size_t ldp = (size_t)R * K;
  const float* gtp = poses + (size_t)(2 * f) * dmax * ldp;
  const float* dp = poses + (size_t)(2 * f + 1) * dmax * ldp;
  float* ob = out_boxes + (size_t)f * dmax * ld;
  float* op = out_poses + (size_t)f * dmax * ldp;
  for (int e = tid; e < dmax * ld; e += blockDim.x) {
    const int o = e / ld, c = e - o * ld;
    float v = 0.f;
    if (o < no) {
      const int i = s_src[o];
      v = db[(size_t)i * ld + c];
      if (compact && (flags & DT_UB_GT_KPS) && c < 4) v = gtb[(size_t)m[i] * ld + c];      // new_boxes[:, :4] (:313)
    }
    ob[e] = v;
  }
  for (size_t e = tid; e < (size_t)dmax * ldp; e += blockDim.x) {
    const int o = (int)(e / ldp), rc = (int)(e - (size_t)o * ldp), r = rc / K;
    float v = 0.f;
    if (o < no) {
      const int i = s_src[o];
      v = dp[(size_t)i * ldp + rc];
      if (compact && (flags & DT_UB_GT_KPS) && (r == 2 || (r < 2 && !(flags & DT_UB_ONLY_CONF))))
        v = gtp[(size_t)m[i] * ldp + rc];                                                  // :314-320
      if (mg && r < 3 && mg[i] >= 0 && mg[i] < G) v = gtp[(size_t)mg[i] * ldp + rc];      // :334-338
    }
    op[e] = v;
  }
  for (int o = tid; o < dmax; o += blockDim.x) {
    const int i = o < no ? s_src[o] : -1;
    out_tid[(size_t)f * dmax + o] = (i >= 0 && compact) ? gt_tid[(size_t)f * dmax + m[i]] : -1;
  }
  if (tid == 0) out_counts[f] = no;
}

}  // namespace dt

using namespace dt;

extern "C" int dt_gt_frame_costs(const float* boxes, int ld, int T, const float* poses, int R, int K, int head_top,
                                 int head_bottom, double dist_thresh, const int* counts, int nframes, int dmax, float w_iou,
                                 double w_pck, double* cost, void* stream) {
  DT_CHECK_ARG(nframes >= 0 && dmax >= 1 && dmax <= DT_LSA_MAX_DIM && T >= 1 && T <= DT_MAX_T && ld >= 4 * T,
               "dt_gt_frame_costs: bad shape nframes=%d dmax=%d T=%d ld=%d (dmax <= %d)", nframes, dmax, T, ld, DT_LSA_MAX_DIM);
  DT_CHECK_ARG(w_pck == 0.0 || (poses && K >= 1 && R >= 2 && head_top >= 0 && head_top < K && head_bottom >= 0 &&
                                head_bottom < K),
               "dt_gt_frame_costs: the pose-pck term needs poses [2 * nframes, dmax, R >= 2, K] and valid head joint indices");
  if (nframes == 0) return 0;
  DT_CHECK_ARG(boxes && counts && cost, "dt_gt_frame_costs: null pointer");
  gt_costs_kernel<<<nframes, 256, 0, (cudaStream_t)stream>>>(boxes, ld, T, poses, R, K, head_top, head_bottom, dist_thresh, counts,
                                                             nframes, dmax, w_iou, w_pck, cost);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_track_upper_bound(const float* boxes, int ld, const float* poses, int R, int K, const int* counts,
                                    const int* gt_tid, int nframes, int dmax, const int* matches, int ldm, const int* matches_gt,
                                    int ldmg, int flags, float* out_boxes, float* out_poses, int* out_tid, int* out_counts,
                                    void* stream) {
  DT_CHECK_ARG(nframes >= 0 && dmax >= 1 && dmax <= DT_LSA_MAX_DIM && ld >= 5 && R >= 3 && K >= 1,
               "dt_track_upper_bound: bad shape nframes=%d dmax=%d ld=%d R=%d K=%d (dmax <= %d, ld >= 5, R >= 3)", nframes, dmax,
               ld, R, K, DT_LSA_MAX_DIM);
  DT_CHECK_ARG((flags & ~(DT_UB_COMPACT | DT_UB_GT_KPS | DT_UB_ONLY_CONF)) == 0 &&
               (!(flags & DT_UB_GT_KPS) || (flags & DT_UB_COMPACT)) && (!(flags & DT_UB_ONLY_CONF) || (flags & DT_UB_GT_KPS)),
               "dt_track_upper_bound: bad flags %d (GT_KPS needs COMPACT, ONLY_CONF needs GT_KPS)", flags);
  DT_CHECK_ARG(!(flags & DT_UB_COMPACT) || (matches && ldm >= dmax), "dt_track_upper_bound: COMPACT needs matches (ldm >= dmax)");
  DT_CHECK_ARG(!matches_gt || ldmg >= dmax, "dt_track_upper_bound: matches_gt needs ldmg >= dmax");
  if (nframes == 0) return 0;
  DT_CHECK_ARG(boxes && poses && counts && out_boxes && out_poses && out_tid && out_counts &&
               (!(flags & DT_UB_COMPACT) || gt_tid),
               "dt_track_upper_bound: null pointer");
  ub_apply_kernel<<<nframes, 256, 0, (cudaStream_t)stream>>>(boxes, ld, poses, R, K, counts, gt_tid, dmax, matches, ldm, matches_gt,
                                                             ldmg, flags, out_boxes, out_poses, out_tid, out_counts);
  DT_CHECK_LAUNCH();
  return 0;
}
