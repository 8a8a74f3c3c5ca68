// Batched rectangular min-cost assignment (one warp per frame pair) and track-id
// propagation, for lib/core/tracking_engine.py:158-350.
//
// The reference calls scipy.optimize.linear_sum_assignment (tracking_engine.py:237)
// and accepts every pair.  Cost matrices here are ~90% exact ties (cost 1.0f for every
// non-overlapping pair), so index parity needs the solver's visiting order, not just an
// optimum: lsa_solver.cuh restates scipy's shortest augmenting path solver in its own order.
#include "common.cuh"
#include "lsa_solver.cuh"
#include "../../include/dt_b200.h"
#include <math_constants.h>

namespace dt {

__device__ __forceinline__ float iou_pair_ref_l(const float* __restrict__ b, const float* __restrict__ q) {
  // identical to boxes.cu:iou_pair_ref (cython_bbox.pyx:34-56); duplicated so that both
  // translation units stay self-contained
  const float qarea = __double2float_rn(
      __dmul_rn(__dadd_rn((double)__fsub_rn(q[2], q[0]), 1.0), __dadd_rn((double)__fsub_rn(q[3], q[1]), 1.0)));
  const float iw = __double2float_rn(__dadd_rn((double)__fsub_rn(fminf(b[2], q[2]), fmaxf(b[0], q[0])), 1.0));
  if (!(iw > 0.f)) return 0.f;
  const float ih = __double2float_rn(__dadd_rn((double)__fsub_rn(fminf(b[3], q[3]), fmaxf(b[1], q[1])), 1.0));
  if (!(ih > 0.f)) return 0.f;
  const float inter = __fmul_rn(iw, ih);
  const double barea = __dmul_rn(__dadd_rn((double)__fsub_rn(b[2], b[0]), 1.0), __dadd_rn((double)__fsub_rn(b[3], b[1]), 1.0));
  const float ua = __double2float_rn(__dsub_rn(__dadd_rn(barea, (double)qarea), (double)inter));
  return __fdiv_rn(inter, ua);
}

// The bbox-only cost matrices are float32 (as the reference's) and staged in shared memory, dmax x dmax.
using LsaSmem = LsaSmemT<float>;

__host__ __device__ inline size_t lsa_smem_bytes(int dmax) { return lsa_smem_bytes_t<float>(dmax, (size_t)dmax * dmax); }

__device__ __forceinline__ LsaSmem lsa_carve(unsigned char* base, int dmax) {
  return lsa_carve_t<float>(base, dmax, (size_t)dmax * dmax);
}

// mode 0: cost given  [B, pmax, ldc] (rows = prev, cols = cur), per-problem (nprev, ncur)
// mode 1: frames given [F, dmax, ld] boxes (+score col ignored); problem f = (frame f-1, frame f)
// bipartite_matching_greedy (tracking_engine.py:184-206): repeatedly take the global argmin of the
// remaining matrix (np.argmin: first occurrence in row-major order; deleting rows / columns keeps that
// order, so ties go to the lowest remaining (row, col)).  C[p * ld + q] holds cost(p, q) (shared or global memory);
// s.SR / s.SC mark used rows / cols.
template <typename T>
__device__ void greedy_match_warp(const LsaSmemT<T>& s, const T* C, int ld, int P, int Q, int* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const unsigned FULL = 0xffffffffu;
  for (int x = lane; x < P; x += 32) s.SR[x] = 0;
  for (int x = lane; x < Q; x += 32) s.SC[x] = 0;
  __syncwarp();
  const int steps = min(P, Q);
  for (int k = 0; k < steps; ++k) {
    T bv = (T)CUDART_INF; int bi = 0x7fffffff;
    bool any = false;
    for (int e = lane; e < P * Q; e += 32) {
      const int p = e / Q, q = e - p * Q;
      if (s.SR[p] || s.SC[q]) continue;
      const T c = C[(size_t)p * ld + q];
      if (!any || c < bv) { bv = c; bi = e; any = true; }          // strict '<': first occurrence per lane
    }
    if (!any) bi = 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const T ov = __shfl_xor_sync(FULL, bv, o);
      const int oi = __shfl_xor_sync(FULL, bi, o);
      const bool take = (oi != 0x7fffffff) && (bi == 0x7fffffff || ov < bv || (ov == bv && oi < bi));
      if (take) { bv = ov; bi = oi; }
    }
    const int p = bi / Q, q = bi - p * Q;
    if (lane == 0) { s.SR[p] = 1; s.SC[q] = 1; out[q] = p; }
    __syncwarp();
  }
}

__global__ void lsa_kernel(int mode, int algo, const float* __restrict__ src, int dmax, int ld, int T,
                           const int* __restrict__ nrows, const int* __restrict__ ncols,
                           const unsigned char* __restrict__ is_start, float weight,
                           int* __restrict__ matches /*[B,dmax] cur -> prev or -1*/,
                           int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x, lane = threadIdx.x;
  LsaSmem s = lsa_carve(smem_raw, dmax);
  int P, Q;                       // prev count (rows), cur count (cols)
  const float* prev = nullptr; const float* cur = nullptr; const float* Cg = nullptr;
  if (mode == 0) {
    P = nrows[b]; Q = ncols[b];
    Cg = src + (size_t)b * dmax * ld;
  } else {
    Q = ncols[b];                                    // counts[f]
    const bool start = (b == 0) || (is_start && is_start[b]);
    P = start ? 0 : ncols[b - 1];
    cur = src + (size_t)b * dmax * ld;
    prev = start ? nullptr : src + (size_t)(b - 1) * dmax * ld;
  }
  P = min(max(P, 0), dmax); Q = min(max(Q, 0), dmax);
  int* out = matches + (size_t)b * dmax;
  for (int q = lane; q < dmax; q += 32) out[q] = -1;
  if (lane == 0 && status) status[b] = 0;
  if (P == 0 || Q == 0) return;
  const bool transpose = (algo == 0) && Q < P;       // scipy: "tall matrix must be transposed"
  const int nr = transpose ? Q : P, nc = transpose ? P : Q;
  // stage the internal matrix: internal(i, j) = cost(prev = transpose ? j : i, cur = transpose ? i : j)
  bool invalid = false;
  for (int e = lane; e < P * Q; e += 32) {
    const int p = e / Q, q = e - p * Q;              // coalesced over q in the source
    float c;
    if (mode == 0) {
      c = Cg[(size_t)p * ld + q];
      invalid |= (c != c) || c == -CUDART_INF_F;     // scipy: "matrix contains invalid numeric entries"
    } else {
      const float* pb = prev + (size_t)p * ld;
      const float* qb = cur + (size_t)q * ld;
      float acc = iou_pair_ref_l(pb, qb);
      for (int t = 1; t < T; ++t) acc = __fadd_rn(acc, iou_pair_ref_l(pb + 4 * t, qb + 4 * t));
      const float iou = __fdiv_rn(acc, (float)T);            // boxes.py:64-69
      c = __fmul_rn(__fsub_rn(1.f, iou), weight);            // tracking_engine.py:168,179
    }
    if (transpose) s.C[(size_t)q * nc + p] = c; else s.C[(size_t)p * nc + q] = c;
  }
  __syncwarp();
  if (algo == 1) { greedy_match_warp(s, s.C, Q, P, Q, out); return; }
  if (mode == 0 && __any_sync(0xffffffffu, invalid)) { if (lane == 0 && status) status[b] = 1; return; }
  const bool ok = lsa_solve_warp(s, nr, nc);
  if (!ok) { if (lane == 0 && status) status[b] = 1; return; }
  __syncwarp();
  // matches[cur] = prev (tracking_engine.py:244-246)
  for (int i = lane; i < nr; i += 32) {
    const int j = s.col4row[i];
    if (transpose) out[i] = j; else out[j] = i;
  }
}

// The same assignment on fp64 costs [B, dmax, ldc] (the combined pose-pck cost: the reference's matrix is float64 then).
// An fp64 224 x 224 matrix does not fit in shared memory, so the solver reads it where it lies (one problem is at most
// 400 KB, which stays in L2 while the warp walks it); a problem with Q < P is solved on the transpose by strided reads.
__global__ void lsa_f64_kernel(int algo, const double* __restrict__ cost, int dmax, int ldc, const int* __restrict__ nrows,
                               const int* __restrict__ ncols, int* __restrict__ matches, int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x, lane = threadIdx.x;
  const LsaSmemT<double> s = lsa_carve_t<double>(smem_raw, dmax, 0);
  const int P = min(max(nrows[b], 0), dmax), Q = min(max(ncols[b], 0), dmax);
  const double* Cg = cost + (size_t)b * dmax * ldc;
  int* out = matches + (size_t)b * dmax;
  for (int q = lane; q < dmax; q += 32) out[q] = -1;
  if (lane == 0 && status) status[b] = 0;
  if (P == 0 || Q == 0) return;
  if (algo == 1) { greedy_match_warp(s, Cg, ldc, P, Q, out); return; }
  bool invalid = false;
  for (int e = lane; e < P * Q; e += 32) {
    const int p = e / Q, q = e - p * Q;
    const double c = Cg[(size_t)p * ldc + q];
    invalid |= (c != c) || c == -CUDART_INF;
  }
  if (__any_sync(0xffffffffu, invalid)) { if (lane == 0 && status) status[b] = 1; return; }
  const bool transpose = Q < P;
  const int nr = transpose ? Q : P, nc = transpose ? P : Q;
  const LsaRows<double> rows{Cg, transpose ? (size_t)1 : (size_t)ldc, transpose ? (size_t)ldc : (size_t)1};
  if (!lsa_solve_warp_rows(s, rows, nr, nc)) { if (lane == 0 && status) status[b] = 1; return; }
  __syncwarp();
  for (int i = lane; i < nr; i += 32) {
    const int j = s.col4row[i];
    if (transpose) out[i] = j; else out[j] = i;
  }
}

// 'pose-pck' tracking cost (lib/core/tracking_engine.py:113-129 -> lib/utils/keypoints.py:266-291) in the reference's own
// arithmetic: float32 head size |head_top - head_bottom| + 1 of the PREVIOUS-frame pose, float32 joint distances / head size,
// count of joints closer than dist_thresh, cost = 1.0 - count / K in fp64.  Poses are the reference's [4, K] arrays (x row, y row).
__device__ __forceinline__ double pck_cost(const float* __restrict__ a, const float* __restrict__ b, int K, int ht, int hb, float thr) {
  const float hx = __fsub_rn(a[ht], a[hb]), hy = __fsub_rn(a[K + ht], a[K + hb]);
  const float head = __fadd_rn(__fsqrt_rn(__fadd_rn(__fmul_rn(hx, hx), __fmul_rn(hy, hy))), 1.f);
  int cnt = 0;
  for (int k = 0; k < K; ++k) {
    const float dx = __fsub_rn(a[k], b[k]), dy = __fsub_rn(a[K + k], b[K + k]);
    const float nd = __fdiv_rn(__fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))), head);
    cnt += nd < thr ? 1 : 0;
  }
  return 1.0 - (double)cnt / (double)K;
}

// out [P, Q] fp64 = pck cost of every (a_i, b_j) pair (the reference's _compute_pairwise_kpt_distance)
__global__ void pose_pck_kernel(const float* __restrict__ a, int P, const float* __restrict__ b, int Q, int ld, int K, int ht, int hb,
                                float thr, double* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= P * Q) return;
  const int i = e / Q, j = e - i * Q;
  out[e] = pck_cost(a + (size_t)i * ld, b + (size_t)j * ld, K, ht, hb, thr);
}

// Cost matrices of all frame pairs of a batch of videos (tracking_engine.py:158-181): cost[f][p][q] (p = detection of frame
// f-1, q = detection of frame f) = w_iou * (1 - IoU) [float32, as the reference computes it] + w_pck * pck [fp64], summed
// and kept in fp64 like np.sum(np.stack(all_Cs)); first frames of videos and entries beyond the counts are 0.
__global__ void frame_costs_kernel(const float* __restrict__ boxes, int ldb, int T, const float* __restrict__ poses, int ldp, int K,
                                   int ht, int hb, float thr, const int* __restrict__ counts, const unsigned char* __restrict__ is_start,
                                   int dmax, float w_iou, double w_pck, double* __restrict__ cost) {
  const int f = blockIdx.x;
  double* C = cost + (size_t)f * dmax * dmax;
  const bool start = (f == 0) || (is_start && is_start[f]);
  const int P = start ? 0 : min(counts[f - 1], dmax), Q = min(counts[f], dmax);
  for (int e = threadIdx.x; e < dmax * dmax; e += blockDim.x) {
    const int p = e / dmax, q = e - p * dmax;
    double acc = 0.0;
    if (p < P && q < Q) {
      if (w_iou != 0.f) {
        const float* pb = boxes + ((size_t)(f - 1) * dmax + p) * ldb;
        const float* qb = boxes + ((size_t)f * dmax + q) * ldb;
        float s = iou_pair_ref_l(pb, qb);
        for (int t = 1; t < T; ++t) s = __fadd_rn(s, iou_pair_ref_l(pb + 4 * t, qb + 4 * t));
        acc = (double)__fmul_rn(__fsub_rn(1.f, __fdiv_rn(s, (float)T)), w_iou);
      }
      if (w_pck != 0.0)
        acc = __dadd_rn(acc, __dmul_rn(pck_cost(poses + ((size_t)(f - 1) * dmax + p) * ldp, poses + ((size_t)f * dmax + q) * ldp, K, ht, hb, thr), w_pck));
    }
    C[e] = acc;
  }
}

// One thread per video: tracking_engine.py:272-350 (non-debug path).  Frames of a video are
// contiguous; a frame with is_start != 0 (or frame 0) opens a new video and resets the counter.
__global__ void track_ids_kernel(const int* __restrict__ matches, const int* __restrict__ counts,
                                 const unsigned char* __restrict__ is_start, int nframes, int dmax,
                                 const int* __restrict__ video_first /*[V] first frame of each video*/,
                                 int nvideos, int first_id, int max_ids, int* __restrict__ tracks) {
  const int vid = blockIdx.x * blockDim.x + threadIdx.x;
  if (vid >= nvideos) return;
  const int f0 = video_first[vid];
  const int f1 = (vid + 1 < nvideos) ? video_first[vid + 1] : nframes;
  int next_id = first_id;
  for (int f = f0; f < f1; ++f) {
    const int n = min(counts[f], dmax);
    const int* m = matches + (size_t)f * dmax;
    int* tr = tracks + (size_t)f * dmax;
    const int* prev = tracks + (size_t)(f - 1) * dmax;
    for (int q = 0; q < n; ++q) {
      const int p = (f == f0) ? -1 : m[q];
      if (p == -1) {
        tr[q] = next_id;
        next_id += 1;
        if (next_id >= max_ids) next_id %= max_ids;          // :341-345
      } else {
        tr[q] = prev[p];
      }
    }
    for (int q = n; q < dmax; ++q) tr[q] = -1;
  }
}

// tracking_engine.py:711-748 (+ _center_boxes :86-93 when center_only): clip the FIRST box of
// each row in place to [0,w]x[0,h], keep rows with score >= conf and (x2-x1)*(y2-y1) >= min_area.
// Output rows are [4*T_out + 1] wide, T_out = center_only ? 1 : T_in, compacted in input order.
__global__ void prune_kernel(const float* __restrict__ boxes, int nframes, int dmax, int ld, int T_in,
                             int center_only, const int* __restrict__ counts_in,
                             const float* __restrict__ hw /*[F,2] h,w*/, float conf, float min_area,
                             float* __restrict__ out, int* __restrict__ counts_out,
                             int* __restrict__ sel /*[F,dmax]*/) {
  const int f = blockIdx.x;
  const int n = min(counts_in[f], dmax);
  const float h = hw[2 * f], w = hw[2 * f + 1];
  const int c0 = center_only ? (T_in / 2) : 0;
  const int T_out = center_only ? 1 : T_in;
  const int ldo = 4 * T_out + 1;
  __shared__ int s_base;
  __shared__ int s_warp[32];
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int start = 0; start < n; start += blockDim.x) {
    const int i = start + threadIdx.x;
    bool keepf = false;
    float x1 = 0, y1 = 0, x2 = 0, y2 = 0, sc = 0;
    const float* p = boxes + ((size_t)f * dmax + (i < n ? i : 0)) * ld;
    if (i < n) {
      x1 = fmaxf(p[4 * c0 + 0], 0.f); y1 = fmaxf(p[4 * c0 + 1], 0.f);
      x2 = fminf(p[4 * c0 + 2], w);   y2 = fminf(p[4 * c0 + 3], h);
      sc = p[4 * T_in];
      const float area = __fmul_rn(__fsub_rn(x2, x1), __fsub_rn(y2, y1));
      keepf = (sc >= conf) && (area >= min_area);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keepf);
    if (lane == 0) s_warp[wid] = __popc(bal);
    __syncthreads();
    int off = s_base;
    for (int x = 0; x < wid; ++x) off += s_warp[x];
    off += __popc(bal & ((1u << lane) - 1));
    if (keepf) {
      float* o = out + ((size_t)f * dmax + off) * ldo;
      o[0] = x1; o[1] = y1; o[2] = x2; o[3] = y2;
      for (int t = 1; t < T_out; ++t)
        for (int k = 0; k < 4; ++k) o[4 * t + k] = p[4 * t + k];
      o[4 * T_out] = sc;
      if (sel) sel[(size_t)f * dmax + off] = i;
    }
    __syncthreads();
    if (threadIdx.x == 0) { int t = 0; for (int x = 0; x < nwarp; ++x) t += s_warp[x]; s_base += t; }
    __syncthreads();
  }
  if (threadIdx.x == 0) counts_out[f] = s_base;
}

}  // namespace dt

using namespace dt;

static int lsa_launch(int mode, int algo, const float* src, int batch, int dmax, int ld, int T,
                      const int* nrows, const int* ncols, const unsigned char* is_start, float weight,
                      int* matches, int* status, cudaStream_t stream) {
  const size_t smem = lsa_smem_bytes(dmax);
  DT_CHECK_ARG(smem <= 227 * 1024, "dt_lsa: dmax=%d needs %zu B of shared memory (> 227 KB)", dmax, smem);
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(lsa_kernel, (int)smem, &grant));
  lsa_kernel<<<batch, 32, smem, stream>>>(mode, algo, src, dmax, ld, T, nrows, ncols, is_start, weight, matches, status);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_lsa_batched(const float* cost, int batch, int dmax, int ldc, const int* nrows,
                              const int* ncols, int algo, int* matches, int* status, void* stream) {
  DT_CHECK_ARG(algo == DT_MATCH_HUNGARIAN || algo == DT_MATCH_GREEDY, "dt_lsa_batched: unknown algo %d", algo);
  DT_CHECK_ARG(batch >= 0 && dmax >= 1 && dmax <= DT_LSA_MAX_DIM && ldc >= 1,
               "dt_lsa_batched: bad shape batch=%d dmax=%d ldc=%d (dmax <= %d)", batch, dmax, ldc, DT_LSA_MAX_DIM);
  if (batch == 0) return 0;
  DT_CHECK_ARG(cost && nrows && ncols && matches, "dt_lsa_batched: null pointer");
  return lsa_launch(0, algo, cost, batch, dmax, ldc, 1, nrows, ncols, nullptr, 1.f, matches, status, (cudaStream_t)stream);
}

extern "C" int dt_lsa_batched_f64(const double* cost, int batch, int dmax, int ldc, const int* nrows,
                                  const int* ncols, int algo, int* matches, int* status, void* stream) {
  DT_CHECK_ARG(algo == DT_MATCH_HUNGARIAN || algo == DT_MATCH_GREEDY, "dt_lsa_batched_f64: unknown algo %d", algo);
  DT_CHECK_ARG(batch >= 0 && dmax >= 1 && dmax <= DT_LSA_MAX_DIM && ldc >= dmax,
               "dt_lsa_batched_f64: bad shape batch=%d dmax=%d ldc=%d (dmax <= %d, ldc >= dmax)", batch, dmax, ldc, DT_LSA_MAX_DIM);
  if (batch == 0) return 0;
  DT_CHECK_ARG(cost && nrows && ncols && matches, "dt_lsa_batched_f64: null pointer");
  const size_t smem = lsa_smem_bytes_t<double>(dmax, 0);
  lsa_f64_kernel<<<batch, 32, smem, (cudaStream_t)stream>>>(algo, cost, dmax, ldc, nrows, ncols, matches, status);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_match_frames(const float* frames, int nframes, int dmax, int ld, int T,
                               const int* counts, const unsigned char* is_start, float weight, int algo,
                               int* matches, int* status, void* stream) {
  DT_CHECK_ARG(algo == DT_MATCH_HUNGARIAN || algo == DT_MATCH_GREEDY, "dt_match_frames: unknown algo %d", algo);
  DT_CHECK_ARG(T >= 1 && T <= DT_MAX_T, "dt_match_frames: T=%d outside [1,%d]", T, DT_MAX_T);
  DT_CHECK_ARG(nframes >= 0 && dmax >= 1 && dmax <= DT_LSA_MAX_DIM && ld >= 4 * T,
               "dt_match_frames: bad shape nframes=%d dmax=%d ld=%d T=%d (dmax <= %d)", nframes, dmax, ld, T, DT_LSA_MAX_DIM);
  if (nframes == 0) return 0;
  DT_CHECK_ARG(frames && counts && matches, "dt_match_frames: null pointer");
  return lsa_launch(1, algo, frames, nframes, dmax, ld, T, nullptr, counts, is_start, weight, matches, status, (cudaStream_t)stream);
}

extern "C" int dt_assign_track_ids(const int* matches, const int* counts, const unsigned char* is_start,
                                   int nframes, int dmax, const int* video_first, int nvideos,
                                   int first_id, int max_ids, int* tracks, void* stream) {
  DT_CHECK_ARG(nframes >= 0 && dmax >= 1 && nvideos >= 0 && max_ids >= 1, "dt_assign_track_ids: bad shape");
  if (nframes == 0 || nvideos == 0) return 0;
  DT_CHECK_ARG(matches && counts && video_first && tracks, "dt_assign_track_ids: null pointer");
  track_ids_kernel<<<cdiv(nvideos, 32), 32, 0, (cudaStream_t)stream>>>(matches, counts, is_start, nframes, dmax,
                                                                       video_first, nvideos, first_id, max_ids, tracks);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_prune_detections(const float* boxes, int nframes, int dmax, int ld, int T, int center_only,
                                   const int* counts_in, const float* hw, float conf, float min_area,
                                   float* out, int* counts_out, int* sel, void* stream) {
  DT_CHECK_ARG(T >= 1 && T <= DT_MAX_T && nframes >= 0 && dmax >= 1 && ld >= 4 * T + 1,
               "dt_prune_detections: bad shape nframes=%d dmax=%d ld=%d T=%d", nframes, dmax, ld, T);
  if (nframes == 0) return 0;
  DT_CHECK_ARG(boxes && counts_in && hw && out && counts_out, "dt_prune_detections: null pointer");
  prune_kernel<<<nframes, 128, 0, (cudaStream_t)stream>>>(boxes, nframes, dmax, ld, T, center_only, counts_in, hw,
                                                          conf, min_area, out, counts_out, sel);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_pose_pck_cost(const float* a, int P, const float* b, int Q, int ld, int K, int head_top, int head_bottom,
                                float dist_thresh, double* out, void* stream) {
  DT_CHECK_ARG(P >= 0 && Q >= 0 && K >= 1 && ld >= 2 * K && head_top >= 0 && head_top < K && head_bottom >= 0 && head_bottom < K,
               "dt_pose_pck_cost: bad shape P=%d Q=%d K=%d ld=%d", P, Q, K, ld);
  if (P == 0 || Q == 0) return 0;
  DT_CHECK_ARG(a && b && out, "dt_pose_pck_cost: null pointer");
  pose_pck_kernel<<<cdiv(P * Q, 128), 128, 0, (cudaStream_t)stream>>>(a, P, b, Q, ld, K, head_top, head_bottom, dist_thresh, out);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_frame_costs(const float* boxes, int ldb, int T, const float* poses, int ldp, int K, int head_top, int head_bottom,
                              float dist_thresh, const int* counts, const unsigned char* is_start, int nframes, int dmax,
                              float w_iou, double w_pck, double* cost, void* stream) {
  DT_CHECK_ARG(nframes >= 0 && dmax >= 1 && T >= 1 && T <= DT_MAX_T && ldb >= 4 * T, "dt_frame_costs: bad shape nframes=%d dmax=%d T=%d ldb=%d", nframes, dmax, T, ldb);
  DT_CHECK_ARG(w_pck == 0.0 || (poses && K >= 1 && ldp >= 2 * K && head_top >= 0 && head_top < K && head_bottom >= 0 && head_bottom < K),
               "dt_frame_costs: the pose-pck term needs poses [nframes, dmax, ldp >= 2K] and valid head joint indices");
  if (nframes == 0) return 0;
  DT_CHECK_ARG(boxes && counts && cost, "dt_frame_costs: null pointer");
  frame_costs_kernel<<<nframes, 256, 0, (cudaStream_t)stream>>>(boxes, ldb, T, poses, ldp, K, head_top, head_bottom, dist_thresh, counts,
                                                                is_start, dmax, w_iou, w_pck, cost);
  DT_CHECK_LAUNCH();
  return 0;
}
