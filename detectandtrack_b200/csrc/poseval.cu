// PoseTrack evaluation (poseval's evaluate_simple.evaluate, lib/datasets/posetrack/poseval/py/) on the device:
//   - pt_assign_kernel: eval_helpers.assignGTmulti (:423-637), one CTA per frame;
//   - the AP kernels: evaluateAP.computeMetrics -> computeRPC + VOCap (eval_helpers.py:169-207), one segmented sort of
//     every (group, joint) score list and one CTA per segment for the scans;
//   - pt_mot_kernel: py-motmetrics' MOTAccumulator.update (motmetrics/mot.py:90-191) over the frames of a sequence, one
//     warp per (frame list, joint), with scipy's own min-cost assignment (lsa_solver.cuh) in fp64.
// The unit is compiled without FMA contraction: distances, PCK, precision / recall and INVDIST round as numpy does.
#include "common.cuh"
#include "lsa_solver.cuh"
#include "../../include/dt_b200.h"
#include <math_constants.h>
#include <stdint.h>

namespace dt {

constexpr int PTJ = DT_PT_JOINTS;

// ---- assignGTmulti ---------------------------------------------------------------------------------------------------

// pck[p, g] = (matched joints) / (annotated GT joints), or the plain count when the GT person has none (:541-547)
__device__ __forceinline__ double pt_pck(unsigned m, int ngtp) {
  const double c = (double)__popc(m);
  return ngtp > 0 ? __ddiv_rn(c, (double)ngtp) : c;
}

// prToGT of a frame (:549-559) from the matched-joint masks [nP, nG] and the GT people's annotated joints: best_gt[p] =
// np.argmax(pck, axis=1) (the first maximum), then pr2gt[g] = np.argmax of the pck pruned to those, -1 where it is 0.
// Called by the whole CTA; ends synchronised.
__device__ void pt_pr_to_gt(const uint16_t* mask, const uint16_t* gmask, int nP, int nG, int* best_gt, int* pr2gt) {
  const int tid = threadIdx.x;
  for (int p = tid; p < nP; p += blockDim.x) {
    int best = 0;
    double bv = pt_pck(mask[p * nG], __popc(gmask[0]));
    for (int g = 1; g < nG; ++g) {
      const double v = pt_pck(mask[p * nG + g], __popc(gmask[g]));
      if (v > bv) { bv = v; best = g; }
    }
    best_gt[p] = best;
  }
  __syncthreads();
  for (int g = tid; g < nG; g += blockDim.x) {
    const int ng = __popc(gmask[g]);
    int best = 0;
    double bv = best_gt[0] == g ? pt_pck(mask[g], ng) : 0.0;
    for (int p = 1; p < nP; ++p) {
      const double v = best_gt[p] == g ? pt_pck(mask[p * nG + g], ng) : 0.0;
      if (v > bv) { bv = v; best = p; }
    }
    pr2gt[g] = bv == 0.0 ? -1 : best;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256) pt_assign_kernel(const int* __restrict__ gt_off, const int* __restrict__ pr_off,
                                                        const long long* __restrict__ pair_off, int F,
                                                        const double* __restrict__ gt_rect, const double* __restrict__ gt_kp,
                                                        const double* __restrict__ pr_kp, signed char* __restrict__ labels,
                                                        int* __restrict__ ngt, double* __restrict__ dist) {
  __shared__ uint16_t mask[DT_LSA_MAX_DIM * DT_PT_MAX_GT];    // matched joints of every (prediction, GT) pair
  __shared__ uint16_t gmask[DT_PT_MAX_GT];                    // annotated joints of every GT person
  __shared__ int best_gt[DT_LSA_MAX_DIM];                     // each prediction's best GT (:550)
  __shared__ int pr2gt[DT_PT_MAX_GT];                         // each GT's best prediction or -1 (:556-558)
  __shared__ int assigned[DT_LSA_MAX_DIM];                    // the GT that took the prediction, or -1
  const int f = blockIdx.x, tid = threadIdx.x;
  const int g0 = gt_off[f], nG = gt_off[f + 1] - g0;
  const int p0 = pr_off[f], nP = pr_off[f + 1] - p0;
  for (int g = tid; g < nG; g += blockDim.x) {
    unsigned m = 0;
    for (int j = 0; j < PTJ; ++j) m |= (gt_kp[((size_t)(g0 + g) * PTJ + j) * 3 + 2] != 0.0) ? (1u << j) : 0u;
    gmask[g] = (uint16_t)m;
  }
  __syncthreads();
  if (tid < PTJ) {                                            // nGTall[:, f] (:629-632)
    int c = 0;
    for (int g = 0; g < nG; ++g) c += (gmask[g] >> tid) & 1;
    ngt[(size_t)tid * F + f] = c;
  }
  if (nP == 0) return;
  const double* pk = pr_kp + (size_t)p0 * PTJ * 4;
  signed char* lab = labels + (size_t)p0 * PTJ;
  if (nG == 0) {                                              // no GT: every prediction is a false positive (:616-626)
    for (int e = tid; e < nP * PTJ; e += blockDim.x) lab[e] = (pk[(size_t)e * 4 + 3] != 0.0) ? 0 : -1;
    return;
  }
  double* d = dist + (size_t)pair_off[f] * PTJ;
  for (int e = tid; e < nP * nG; e += blockDim.x) {
    const int p = e / nG, g = e - p * nG;
    const double* r = gt_rect + (size_t)(g0 + g) * 4;
    const double hx = __dsub_rn(r[2], r[0]), hy = __dsub_rn(r[3], r[1]);
    const double head = __dmul_rn(0.6, __dsqrt_rn(__dadd_rn(__dmul_rn(hx, hx), __dmul_rn(hy, hy))));   // getHeadSize
    const double* gk = gt_kp + (size_t)(g0 + g) * PTJ * 3;
    const double* q = pk + (size_t)p * PTJ * 4;
    const unsigned gm = gmask[g];
    unsigned m = 0;
    for (int j = 0; j < PTJ; ++j) {
      double v = CUDART_NAN;
      if (((gm >> j) & 1) && q[j * 4 + 3] != 0.0) {
        const double dx = __dsub_rn(gk[j * 3], q[j * 4]), dy = __dsub_rn(gk[j * 3 + 1], q[j * 4 + 1]);
        const double dd = __ddiv_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy))), head);
        if (dd <= 0.5) { m |= 1u << j; v = dd; }              // match = dist <= distThresh
      }
      d[(size_t)e * PTJ + j] = v;
    }
    mask[e] = (uint16_t)m;
  }
  __syncthreads();
  pt_pr_to_gt(mask, gmask, nP, nG, best_gt, pr2gt);
  for (int p = tid; p < nP; p += blockDim.x) assigned[p] = -1;
  __syncthreads();
  for (int g = tid; g < nG; g += blockDim.x)                  // a prediction is best for at most one GT (:597-598)
    if (pr2gt[g] >= 0) assigned[pr2gt[g]] = g;
  __syncthreads();
  for (int e = tid; e < nP * PTJ; e += blockDim.x) {          // :594-615
    const int p = e / PTJ, j = e - p * PTJ;
    const int g = assigned[p];
    signed char v = -1;
    if (pk[(size_t)e * 4 + 3] != 0.0) v = g >= 0 ? (signed char)((mask[p * nG + g] >> j) & 1) : 0;
    lab[e] = v;
  }
}

// ---- computeRPC + VOCap ----------------------------------------------------------------------------------------------

// One score of one segment.  Order: segment, then score descending, then position (the prediction's row in the
// reference's concatenation order).  Keys are unique, so any correct sort gives the same order.
struct PtItem {
  unsigned long long key;   // ~(order-preserving bits of the score): ascending key = descending score
  int seg;
  int pos;
};

__device__ __forceinline__ bool pt_less(const PtItem& a, const PtItem& b) {
  if (a.seg != b.seg) return a.seg < b.seg;
  if (a.key != b.key) return a.key < b.key;
  return a.pos < b.pos;
}

__device__ __forceinline__ unsigned long long pt_desc_key(double s) {
  if (s != s) s = CUDART_NAN;                                 // numpy sorts every NaN last (so first, reversed)
  if (s == 0.0) s = 0.0;                                      // -0.0 ties with +0.0
  const unsigned long long b = (unsigned long long)__double_as_longlong(s);
  const unsigned long long asc = (b >> 63) ? ~b : (b | 0x8000000000000000ull);
  return ~asc;
}

// segs [nseg, 3] = (joint, first frame, end frame); seg_off [nseg + 1] = where each segment's scores go
__global__ void __launch_bounds__(256) pt_gather_kernel(const double* __restrict__ pr_kp, const int* __restrict__ pr_off,
                                                        const int* __restrict__ segs, const int* __restrict__ seg_off,
                                                        PtItem* __restrict__ items) {
  __shared__ int warp_n[8];
  __shared__ int base;
  const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int j = segs[s * 3], lo = pr_off[segs[s * 3 + 1]], hi = pr_off[segs[s * 3 + 2]];
  if (tid == 0) base = seg_off[s];
  __syncthreads();
  for (int p0 = lo; p0 < hi; p0 += blockDim.x) {
    const int p = p0 + tid;
    const bool has = p < hi && pr_kp[((size_t)p * PTJ + j) * 4 + 3] != 0.0;
    const unsigned bal = __ballot_sync(0xffffffffu, has);
    if (lane == 0) warp_n[w] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int x = 0; x < w; ++x) off += warp_n[x];
    off += __popc(bal & ((1u << lane) - 1));
    if (has) {
      PtItem it;
      it.key = pt_desc_key(pr_kp[((size_t)p * PTJ + j) * 4 + 2]);
      it.seg = s;
      it.pos = p;
      items[off] = it;
    }
    __syncthreads();
    if (tid == 0) for (int x = 0; x < (int)(blockDim.x >> 5); ++x) base += warp_n[x];
    __syncthreads();
  }
}

constexpr int PT_TILE = 2048;

// bitonic sort of one tile of PT_TILE items in shared memory
__global__ void __launch_bounds__(1024) pt_tile_sort_kernel(PtItem* __restrict__ items, int n) {
  __shared__ PtItem t[PT_TILE];
  const int base = blockIdx.x * PT_TILE;
  for (int i = threadIdx.x; i < PT_TILE; i += blockDim.x) {
    PtItem it;
    if (base + i < n) it = items[base + i];
    else { it.key = ~0ull; it.seg = 0x7fffffff; it.pos = 0x7fffffff; }
    t[i] = it;
  }
  __syncthreads();
  for (int k = 2; k <= PT_TILE; k <<= 1) {
    for (int jj = k >> 1; jj > 0; jj >>= 1) {
      for (int i = threadIdx.x; i < PT_TILE; i += blockDim.x) {
        const int l = i ^ jj;
        if (l > i) {
          const bool up = (i & k) == 0;
          const PtItem a = t[i], b = t[l];
          if (pt_less(b, a) == up) { t[i] = b; t[l] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < PT_TILE; i += blockDim.x)
    if (base + i < n) items[base + i] = t[i];
}

// one merge pass: runs of length L are merged pairwise; each item finds its place in the partner run
__global__ void pt_merge_kernel(const PtItem* __restrict__ in, PtItem* __restrict__ out, int n, int L) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const PtItem x = in[e];
  const int run = e / L, base = (run >> 1) * 2 * L;
  const bool left = (run & 1) == 0;
  const int plo = left ? base + L : base, phi = left ? min(base + 2 * L, n) : base + L;
  int a = plo, b = max(plo, phi);
  while (a < b) {                                             // count of partner items ordered before x
    const int m = (a + b) >> 1;
    if (pt_less(in[m], x)) a = m + 1; else b = m;
  }
  const int own = left ? e - base : e - base - L;
  out[base + own + (a - plo)] = x;
}

template <typename T, typename Op>
__device__ __forceinline__ T pt_block_scan(T v, Op op, T* sh /*[32]*/, T* total) {
  // inclusive scan over the block in thread order
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v = op(u, v);
  }
  if (lane == 31) sh[w] = v;
  __syncthreads();
  if (w == 0) {
    T x = lane < nw ? sh[lane] : sh[0];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T u = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x = op(u, x);
    }
    if (lane < nw) sh[lane] = x;
  }
  __syncthreads();
  if (w > 0) v = op(sh[w - 1], v);
  *total = sh[nw - 1];
  __syncthreads();
  return v;
}

struct PtAdd { __device__ int operator()(int a, int b) const { return a + b; } };
struct PtMax { __device__ double operator()(double a, double b) const { return b > a ? b : a; } };   // Python's max

// computeRPC + VOCap + computeMetrics (evaluateAP.py:9-32) for one segment: out[s] = (AP, last precision, last
// recall) x 100, all zero for an empty segment.  npos [n] is scratch.
__global__ void __launch_bounds__(1024) pt_rpc_kernel(const PtItem* __restrict__ items, const signed char* __restrict__ labels,
                                                      const int* __restrict__ ngt, int F, const int* __restrict__ segs,
                                                      const int* __restrict__ seg_off, int* __restrict__ npos,
                                                      double* __restrict__ out) {
  __shared__ int shi[32];
  __shared__ double shd[32];
  const int s = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int j = segs[s * 3], f0 = segs[s * 3 + 1], f1 = segs[s * 3 + 2];
  const int lo = seg_off[s], n = seg_off[s + 1] - lo;
  if (n == 0) {
    if (tid == 0) { out[s * 3] = 0.0; out[s * 3 + 1] = 0.0; out[s * 3 + 2] = 0.0; }
    return;
  }
  // totalPos = sum(nGTall[j, frames])
  int c = 0;
  for (int f = f0 + tid; f < f1; f += nt) c += ngt[(size_t)j * F + f];
  int tot;
  pt_block_scan(c, PtAdd(), shi, &tot);
  const double T = (double)tot;
  // forward: npos after every sorted item
  int carry = 0;
  for (int k0 = 0; k0 < n; k0 += nt) {
    const int k = k0 + tid;
    const int l = k < n ? (labels[(size_t)items[lo + k].pos * PTJ + j] == 1) : 0;
    int t;
    const int v = pt_block_scan(l, PtAdd(), shi, &t);
    if (k < n) npos[lo + k] = carry + v;
    carry += t;
  }
  __syncthreads();
  // backward: mpre = suffix maximum of the precision (the trailing 0 included), AP terms where the recall changes
  double smax = 0.0, acc = 0.0;
  for (int k1 = n; k1 > 0; k1 -= nt) {
    const int k = k1 - 1 - tid;                               // thread order = descending k: a prefix scan is a suffix scan
    double prec = 0.0;
    if (k >= 0) prec = __ddiv_rn((double)npos[lo + k], (double)(k + 1));
    double t;
    double m = pt_block_scan(k >= 0 ? prec : 0.0, PtMax(), shd, &t);
    m = PtMax()(m, smax);
    if (k >= 0) {
      const double rk = __ddiv_rn((double)npos[lo + k], T);
      const double rp = k > 0 ? __ddiv_rn((double)npos[lo + k - 1], T) : 0.0;
      if (!(rk == rp)) acc = __dadd_rn(acc, __dmul_rn(__dsub_rn(rk, rp), m));
    }
    smax = PtMax()(smax, t);
  }
  if (tid == 0) {                                             // the closing point (recall 1.0, precision 0)
    const double rl = __ddiv_rn((double)npos[lo + n - 1], T);
    if (!(1.0 == rl)) acc = __dadd_rn(acc, __dmul_rn(__dsub_rn(1.0, rl), 0.0));
  }
  // sum of the terms
  const int lane = tid & 31, w = tid >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  if (lane == 0) shd[w] = acc;
  __syncthreads();
  if (tid == 0) {
    double ap = 0.0;
    for (int x = 0; x < (nt >> 5); ++x) ap = __dadd_rn(ap, shd[x]);
    const double last = (double)npos[lo + n - 1];
    out[s * 3] = __dmul_rn(ap, 100.0);
    out[s * 3 + 1] = __dmul_rn(__ddiv_rn(last, (double)n), 100.0);
    out[s * 3 + 2] = __dmul_rn(__ddiv_rn(last, T), 100.0);
  }
}

// ---- assignGTmulti(..., computeUpperBound=True) (:559-573) -------------------------------------------------------------

// The frame's prToGT, recomputed from dt_posetrack_assign's dist (finite = the joint matched) into s_pr2gt; returns how
// many predictions the upper-bound view keeps: those some GT selected, or all of them in a frame without both GT and
// predictions (left untouched).
__device__ int pt_ub_select(int f, const int* __restrict__ gt_off, const int* __restrict__ pr_off,
                            const long long* __restrict__ pair_off, const double* __restrict__ gt_kp,
                            const double* __restrict__ dist, uint16_t* mask, uint16_t* gmask, int* best_gt, int* s_pr2gt) {
  const int tid = threadIdx.x;
  const int g0 = gt_off[f], nG = gt_off[f + 1] - g0, nP = pr_off[f + 1] - pr_off[f];
  if (nG == 0 || nP == 0) return nP;
  for (int g = tid; g < nG; g += blockDim.x) {
    unsigned m = 0;
    for (int j = 0; j < PTJ; ++j) m |= (gt_kp[((size_t)(g0 + g) * PTJ + j) * 3 + 2] != 0.0) ? (1u << j) : 0u;
    gmask[g] = (uint16_t)m;
  }
  const double* d = dist + (size_t)pair_off[f] * PTJ;
  for (int e = tid; e < nP * nG; e += blockDim.x) {
    unsigned m = 0;
    for (int j = 0; j < PTJ; ++j) m |= isfinite(d[(size_t)e * PTJ + j]) ? (1u << j) : 0u;
    mask[e] = (uint16_t)m;
  }
  __syncthreads();
  pt_pr_to_gt(mask, gmask, nP, nG, best_gt, s_pr2gt);
  int n = 0;
  for (int g = 0; g < nG; ++g) n += s_pr2gt[g] >= 0;
  return n;
}

// counts [nframes] of the view, written at ub_pr_off[f + 1]
__global__ void __launch_bounds__(256) pt_ub_count_kernel(const int* __restrict__ gt_off, const int* __restrict__ pr_off,
                                                          const long long* __restrict__ pair_off, const double* __restrict__ gt_kp,
                                                          const double* __restrict__ dist, int* __restrict__ ub_pr_off) {
  __shared__ uint16_t mask[DT_LSA_MAX_DIM * DT_PT_MAX_GT];
  __shared__ uint16_t gmask[DT_PT_MAX_GT];
  __shared__ int best_gt[DT_LSA_MAX_DIM];
  __shared__ int pr2gt[DT_PT_MAX_GT];
  const int n = pt_ub_select(blockIdx.x, gt_off, pr_off, pair_off, gt_kp, dist, mask, gmask, best_gt, pr2gt);
  if (threadIdx.x == 0) ub_pr_off[blockIdx.x + 1] = n;
}

struct PtAddL { __device__ long long operator()(long long a, long long b) const { return a + b; } };

// one CTA: ub_pr_off [F + 1] prefix-summed in place, ub_pair_off [F + 1] = prefix sums of nG * kept predictions
__global__ void __launch_bounds__(1024) pt_ub_scan_kernel(const int* __restrict__ gt_off, int F, int* __restrict__ ub_pr_off,
                                                          long long* __restrict__ ub_pair_off) {
  __shared__ int shi[32];
  __shared__ long long shl[32];
  int carry = 0;
  long long carry2 = 0;
  for (int f0 = 0; f0 < F; f0 += blockDim.x) {
    const int f = f0 + threadIdx.x;
    const int c = f < F ? ub_pr_off[f + 1] : 0;
    const long long pc = f < F ? (long long)c * (gt_off[f + 1] - gt_off[f]) : 0;
    int t;
    long long t2;
    const int v = pt_block_scan(c, PtAdd(), shi, &t);
    const long long v2 = pt_block_scan(pc, PtAddL(), shl, &t2);
    if (f < F) { ub_pr_off[f + 1] = carry + v; ub_pair_off[f + 1] = carry2 + v2; }
    carry += t;
    carry2 += t2;
  }
  if (threadIdx.x == 0) { ub_pr_off[0] = 0; ub_pair_off[0] = 0; }
}

// one CTA per frame: the view's prediction rows (keypoints, track id) and distances
__global__ void __launch_bounds__(256) pt_ub_gather_kernel(const int* __restrict__ gt_off, const int* __restrict__ pr_off,
                                                           const long long* __restrict__ pair_off, const double* __restrict__ gt_kp,
                                                           const int* __restrict__ gt_tid, const double* __restrict__ pr_kp,
                                                           const int* __restrict__ pr_tid, const double* __restrict__ dist,
                                                           const int* __restrict__ ub_pr_off,
                                                           const long long* __restrict__ ub_pair_off, double* __restrict__ ub_pr_kp,
                                                           int* __restrict__ ub_pr_tid, double* __restrict__ ub_dist) {
  __shared__ uint16_t mask[DT_LSA_MAX_DIM * DT_PT_MAX_GT];
  __shared__ uint16_t gmask[DT_PT_MAX_GT];
  __shared__ int best_gt[DT_LSA_MAX_DIM];
  __shared__ int pr2gt[DT_PT_MAX_GT];
  __shared__ int sel_g[DT_PT_MAX_GT];                         // the k-th kept prediction's GT, in ascending GT order
  const int f = blockIdx.x, tid = threadIdx.x;
  const int g0 = gt_off[f], nG = gt_off[f + 1] - g0, p0 = pr_off[f], nP = pr_off[f + 1] - p0;
  const int n = pt_ub_select(f, gt_off, pr_off, pair_off, gt_kp, dist, mask, gmask, best_gt, pr2gt);
  const bool sel = nG > 0 && nP > 0;
  if (sel && tid == 0) {
    int k = 0;
    for (int g = 0; g < nG; ++g) if (pr2gt[g] >= 0) sel_g[k++] = g;
  }
  __syncthreads();
  const int o0 = ub_pr_off[f];
  for (int e = tid; e < n * PTJ * 4; e += blockDim.x) {
    const int k = e / (PTJ * 4), c = e - k * (PTJ * 4);
    const int src = p0 + (sel ? pr2gt[sel_g[k]] : k);
    ub_pr_kp[(size_t)(o0 + k) * PTJ * 4 + c] = pr_kp[(size_t)src * PTJ * 4 + c];
  }
  for (int k = tid; k < n; k += blockDim.x) {
    const int src = p0 + (sel ? pr2gt[sel_g[k]] : k);
    ub_pr_tid[o0 + k] = sel ? gt_tid[g0 + sel_g[k]] : pr_tid[src];        // trackidxPr = trackidxGT[sel_pos]
  }
  if (!sel) return;
  const double* d = dist + (size_t)pair_off[f] * PTJ;
  double* od = ub_dist + (size_t)ub_pair_off[f] * PTJ;
  for (int e = tid; e < n * nG * PTJ; e += blockDim.x) {
    const int k = e / (nG * PTJ), gj = e - k * (nG * PTJ);
    od[e] = d[(size_t)pr2gt[sel_g[k]] * nG * PTJ + gj];
  }
}

// ---- MOTAccumulator.update -------------------------------------------------------------------------------------------

struct PtMotSmem {
  int* oid; int* orow; int* hid; int* hrow; int* h4o; int* mkey; int* mval;
  unsigned char* omask; unsigned char* hmask;
  LsaSmemT<double> lsa;
};

__host__ __device__ inline size_t pt_mot_extra_bytes(int max_gt, int max_pr, int map_cap) {
  size_t b = (size_t)(3 * max_gt + 2 * max_pr + 2 * map_cap) * sizeof(int) + (size_t)(max_gt + max_pr);
  return (b + 15) / 16 * 16;
}

__host__ __device__ inline size_t pt_mot_smem_bytes(int max_gt, int max_pr, int map_cap) {
  const int dvec = max(max_gt, max_pr);
  return pt_mot_extra_bytes(max_gt, max_pr, map_cap) + lsa_smem_bytes_t<double>(dvec, (size_t)max_gt * max_pr);
}

__device__ __forceinline__ PtMotSmem pt_mot_carve(unsigned char* base, int max_gt, int max_pr, int map_cap) {
  PtMotSmem s;
  unsigned char* p = base;
  s.oid = (int*)p; p += max_gt * sizeof(int);
  s.orow = (int*)p; p += max_gt * sizeof(int);
  s.h4o = (int*)p; p += max_gt * sizeof(int);
  s.hid = (int*)p; p += max_pr * sizeof(int);
  s.hrow = (int*)p; p += max_pr * sizeof(int);
  s.mkey = (int*)p; p += map_cap * sizeof(int);
  s.mval = (int*)p; p += map_cap * sizeof(int);
  s.omask = p; p += max_gt;
  s.hmask = p;
  s.lsa = lsa_carve_t<double>(base + pt_mot_extra_bytes(max_gt, max_pr, map_cap), max(max_gt, max_pr), (size_t)max_gt * max_pr);
  return s;
}

// index of key in the accumulator's map m (0..mn), or -1; warp-uniform result
__device__ __forceinline__ int pt_map_find(const PtMotSmem& s, int mn, int key) {
  const int lane = threadIdx.x & 31;
  for (int b = 0; b < mn; b += 32) {
    const int i = b + lane;
    const unsigned bal = __ballot_sync(0xffffffffu, i < mn && s.mkey[i] == key);
    if (bal) return b + __ffs(bal) - 1;
  }
  return -1;
}

// counts [L, 15, 4] = MATCH, SWITCH, FP, MISS events; sumd [L, 15] = sum of the distances of MATCH and SWITCH events.
// Frame list l = list_frames[list_off[l] .. list_off[l + 1]): the frames whose MOT inputs update() sees, in order.
__global__ void __launch_bounds__(32) pt_mot_kernel(const int* __restrict__ gt_off, const int* __restrict__ pr_off,
                                                    const long long* __restrict__ pair_off, const double* __restrict__ gt_kp,
                                                    const int* __restrict__ gt_tid, const double* __restrict__ pr_kp,
                                                    const int* __restrict__ pr_tid, const double* __restrict__ dist,
                                                    const int* __restrict__ list_off, const int* __restrict__ list_frames,
                                                    int max_gt, int max_pr, int map_cap, int* __restrict__ counts,
                                                    double* __restrict__ sumd, int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int l = blockIdx.x / PTJ, j = blockIdx.x - l * PTJ, lane = threadIdx.x;
  const unsigned FULL = 0xffffffffu;
  PtMotSmem s = pt_mot_carve(smem_raw, max_gt, max_pr, map_cap);
  int mn = 0;                                                 // entries of m
  int n_match = 0, n_switch = 0, n_fp = 0, n_miss = 0, overflow = 0;
  double sd = 0.0;
  for (int fi = list_off[l]; fi < list_off[l + 1]; ++fi) {
    const int f = list_frames[fi];
    const int g0 = gt_off[f], nGf = gt_off[f + 1] - g0, p0 = pr_off[f], nPf = pr_off[f + 1] - p0;
    // the rows that have joint j (mot[i]["ridxsGT"] / ["ridxsPr"], :580-591)
    int nO = 0, nH = 0;
    for (int b = 0; b < nGf; b += 32) {
      const int g = b + lane;
      const bool has = g < nGf && gt_kp[((size_t)(g0 + g) * PTJ + j) * 3 + 2] != 0.0;
      const unsigned bal = __ballot_sync(FULL, has);
      const int at = nO + __popc(bal & ((1u << lane) - 1));
      if (has && at < max_gt) { s.oid[at] = gt_tid[g0 + g]; s.orow[at] = g; s.omask[at] = 0; }
      nO += __popc(bal);
    }
    for (int b = 0; b < nPf; b += 32) {
      const int p = b + lane;
      const bool has = p < nPf && pr_kp[((size_t)(p0 + p) * PTJ + j) * 4 + 3] != 0.0;
      const unsigned bal = __ballot_sync(FULL, has);
      const int at = nH + __popc(bal & ((1u << lane) - 1));
      if (has && at < max_pr) { s.hid[at] = pr_tid[p0 + p]; s.hrow[at] = p; s.hmask[at] = 0; }
      nH += __popc(bal);
    }
    if (nO > max_gt || nH > max_pr) { overflow = 1; break; }
    __syncwarp();
    if (nO > 0 && nH > 0) {
      // the distances, [o, h] or transposed as scipy solves a tall matrix; _sanitize_dists: INVDIST = 2 max + 1
      const bool tr = nH < nO;
      double* C = s.lsa.C;
      const double* d = dist + (size_t)pair_off[f] * PTJ;
      double vmax = -CUDART_INF;
      bool any = false;
      for (int e = lane; e < nO * nH; e += 32) {
        const int a = e / nH, b = e - a * nH;
        const double v = d[((size_t)s.hrow[b] * nGf + s.orow[a]) * PTJ + j];
        if (isfinite(v)) { any = true; vmax = fmax(vmax, v); }
        C[tr ? (size_t)b * nO + a : (size_t)e] = v;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) vmax = fmax(vmax, __shfl_xor_sync(FULL, vmax, o));
      any = __any_sync(FULL, any);
      const double INV = any ? __dadd_rn(__dmul_rn(2.0, vmax), 1.0) : 1.0;
      __syncwarp();
      for (int e = lane; e < nO * nH; e += 32)
        if (!isfinite(C[e])) C[e] = INV;
      __syncwarp();
      auto at = [&](int a, int b) -> double& { return C[tr ? (size_t)b * nO + a : (size_t)a * nH + b]; };
      // 1. re-establish the previous correspondences, object by object
      for (int a = 0; a < nO; ++a) {
        const int o = s.oid[a];
        const int mi = pt_map_find(s, mn, o);
        if (mi < 0) continue;
        const int hprev = s.mval[mi];
        int jb = -1;
        for (int b0 = 0; b0 < nH; b0 += 32) {                 // np.where(hids == hprev): unmasked hypotheses only
          const int b = b0 + lane;
          const unsigned bal = __ballot_sync(FULL, b < nH && !s.hmask[b] && s.hid[b] == hprev);
          if (bal) { jb = b0 + __ffs(bal) - 1; break; }
        }
        if (jb < 0) continue;
        const double v = at(a, jb);
        if (!(v == INV)) {
          if (lane == 0) { s.omask[a] = 1; s.hmask[jb] = 1; s.mval[mi] = s.hid[jb]; }
          ++n_match;
          sd = __dadd_rn(sd, v);
        }
        __syncwarp();
      }
      // 2. min-cost assignment of the full matrix, the masked rows and columns at INVDIST
      for (int e = lane; e < nO * nH; e += 32) {
        const int a = e / nH, b = e - a * nH;
        if (s.omask[a] || s.hmask[b]) at(a, b) = INV;
      }
      __syncwarp();
      const int nr = tr ? nH : nO, nc = tr ? nO : nH;
      lsa_solve_warp(s.lsa, nr, nc);                          // finite costs: always feasible
      __syncwarp();
      for (int a = lane; a < nO; a += 32) s.h4o[a] = -1;
      __syncwarp();
      for (int r = lane; r < nr; r += 32) {
        const int c = s.lsa.col4row[r];
        if (tr) s.h4o[c] = r; else s.h4o[r] = c;
      }
      __syncwarp();
      for (int a = 0; a < nO; ++a) {                          // zip(rids, cids): rows in ascending order
        const int b = s.h4o[a];
        if (b < 0) continue;
        const double v = at(a, b);
        if (v == INV) continue;
        const int o = s.oid[a], h = s.hid[b];
        const int mi = pt_map_find(s, mn, o);
        if (mi >= 0 && s.mval[mi] != h) ++n_switch; else ++n_match;    // max_switch_time is infinite
        sd = __dadd_rn(sd, v);
        if (lane == 0) {
          s.omask[a] = 1; s.hmask[b] = 1;
          if (mi >= 0) s.mval[mi] = h;
          else if (mn < map_cap) { s.mkey[mn] = o; s.mval[mn] = h; }
        }
        if (mi < 0) { if (mn < map_cap) ++mn; else overflow = 1; }
        __syncwarp();
      }
    }
    __syncwarp();
    // 3. / 4. the rest are misses and false positives
    int miss = 0, fp = 0;
    for (int a = lane; a < nO; a += 32) miss += !s.omask[a];
    for (int b = lane; b < nH; b += 32) fp += !s.hmask[b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { miss += __shfl_xor_sync(FULL, miss, o); fp += __shfl_xor_sync(FULL, fp, o); }
    n_miss += miss;
    n_fp += fp;
    __syncwarp();
  }
  if (lane == 0) {
    int* c = counts + (size_t)blockIdx.x * 4;
    c[0] = n_match; c[1] = n_switch; c[2] = n_fp; c[3] = n_miss;
    sumd[blockIdx.x] = sd;
    if (status) status[blockIdx.x] = overflow;
  }
}

}  // namespace dt

using namespace dt;

extern "C" int dt_posetrack_assign(const int* gt_off, const int* pr_off, const long long* pair_off, int nframes,
                                   const double* gt_rect, const double* gt_kp, const double* pr_kp, int max_gt, int max_pr,
                                   signed char* labels, int* ngt, double* dist, void* stream) {
  DT_CHECK_ARG(nframes >= 0 && max_gt >= 0 && max_gt <= DT_PT_MAX_GT && max_pr >= 0 && max_pr <= DT_LSA_MAX_DIM,
               "dt_posetrack_assign: bad shape nframes=%d max_gt=%d max_pr=%d (max_gt <= %d, max_pr <= %d)", nframes, max_gt,
               max_pr, DT_PT_MAX_GT, DT_LSA_MAX_DIM);
  if (nframes == 0) return 0;
  DT_CHECK_ARG(gt_off && pr_off && pair_off && ngt && (max_gt == 0 || (gt_rect && gt_kp)) &&
               (max_pr == 0 || (pr_kp && labels)) && (max_gt == 0 || max_pr == 0 || dist),
               "dt_posetrack_assign: null pointer");
  pt_assign_kernel<<<nframes, 256, 0, (cudaStream_t)stream>>>(gt_off, pr_off, pair_off, nframes, gt_rect, gt_kp, pr_kp,
                                                              labels, ngt, dist);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_posetrack_upper_bound(const int* gt_off, const int* pr_off, const long long* pair_off, int nframes,
                                       const double* gt_kp, const int* gt_tid, const double* pr_kp, const int* pr_tid,
                                       const double* dist, int max_gt, int max_pr, int* ub_pr_off, long long* ub_pair_off,
                                       double* ub_pr_kp, int* ub_pr_tid, double* ub_dist, void* stream) {
  DT_CHECK_ARG(nframes >= 0 && max_gt >= 0 && max_gt <= DT_PT_MAX_GT && max_pr >= 0 && max_pr <= DT_LSA_MAX_DIM,
               "dt_posetrack_upper_bound: bad shape nframes=%d max_gt=%d max_pr=%d (max_gt <= %d, max_pr <= %d)", nframes,
               max_gt, max_pr, DT_PT_MAX_GT, DT_LSA_MAX_DIM);
  if (nframes == 0) return 0;
  DT_CHECK_ARG(gt_off && pr_off && pair_off && ub_pr_off && ub_pair_off && (max_gt == 0 || (gt_kp && gt_tid)) &&
               (max_pr == 0 || (pr_kp && pr_tid && ub_pr_kp && ub_pr_tid)) &&
               (max_gt == 0 || max_pr == 0 || (dist && ub_dist)),
               "dt_posetrack_upper_bound: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  pt_ub_count_kernel<<<nframes, 256, 0, st>>>(gt_off, pr_off, pair_off, gt_kp, dist, ub_pr_off);
  DT_CHECK_LAUNCH();
  pt_ub_scan_kernel<<<1, 1024, 0, st>>>(gt_off, nframes, ub_pr_off, ub_pair_off);
  DT_CHECK_LAUNCH();
  pt_ub_gather_kernel<<<nframes, 256, 0, st>>>(gt_off, pr_off, pair_off, gt_kp, gt_tid, pr_kp, pr_tid, dist, ub_pr_off,
                                               ub_pair_off, ub_pr_kp, ub_pr_tid, ub_dist);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_posetrack_ap_workspace_bytes(long long nentries, size_t* bytes) {
  DT_CHECK_ARG(nentries >= 0 && nentries <= 0x3fffffffLL, "dt_posetrack_ap_workspace_bytes: nentries=%lld outside [0, 2^30]",
               nentries);
  DT_CHECK_ARG(bytes, "dt_posetrack_ap_workspace_bytes: null pointer");
  const size_t n = (size_t)nentries;
  *bytes = 2 * n * sizeof(PtItem) + (n * sizeof(int) + 15) / 16 * 16;
  return 0;
}

extern "C" int dt_posetrack_ap(const double* pr_kp, const signed char* labels, const int* ngt, int nframes, const int* pr_off,
                               const int* segs, const int* seg_off, int nseg, long long nentries, double* out, void* workspace,
                               size_t workspace_bytes, void* stream) {
  DT_CHECK_ARG(nframes >= 0 && nseg >= 0 && nentries >= 0 && nentries <= 0x3fffffffLL,
               "dt_posetrack_ap: bad shape nframes=%d nseg=%d nentries=%lld", nframes, nseg, nentries);
  size_t need = 0;
  dt_posetrack_ap_workspace_bytes(nentries, &need);
  DT_CHECK_ARG(workspace_bytes >= need, "dt_posetrack_ap: workspace of %zu B, %zu B needed for nentries=%lld", workspace_bytes,
               need, nentries);
  if (nseg == 0) return 0;
  DT_CHECK_ARG(ngt && pr_off && segs && seg_off && out && (nentries == 0 || (pr_kp && labels && workspace)),
               "dt_posetrack_ap: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int n = (int)nentries;
  PtItem* a = (PtItem*)workspace;
  PtItem* b = a + n;
  int* npos = (int*)(b + n);
  if (n > 0) {
    pt_gather_kernel<<<nseg, 256, 0, st>>>(pr_kp, pr_off, segs, seg_off, a);
    DT_CHECK_LAUNCH();
    pt_tile_sort_kernel<<<cdiv(n, PT_TILE), 1024, 0, st>>>(a, n);
    DT_CHECK_LAUNCH();
    for (int L = PT_TILE; L < n; L <<= 1) {
      pt_merge_kernel<<<cdiv(n, 256), 256, 0, st>>>(a, b, n, L);
      DT_CHECK_LAUNCH();
      PtItem* t = a; a = b; b = t;
    }
  }
  pt_rpc_kernel<<<nseg, 1024, 0, st>>>(a, labels, ngt, nframes, segs, seg_off, npos, out);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_posetrack_mot_smem_bytes(int max_gt, int max_pr, int map_cap, size_t* bytes) {
  DT_CHECK_ARG(max_gt >= 0 && max_gt <= DT_PT_MAX_GT && max_pr >= 0 && max_pr <= DT_LSA_MAX_DIM && map_cap >= 0 &&
               map_cap <= DT_PT_MAX_MAP_IDS,
               "dt_posetrack_mot_smem_bytes: bad shape max_gt=%d max_pr=%d map_cap=%d (max_gt <= %d, max_pr <= %d, map_cap <= %d)",
               max_gt, max_pr, map_cap, DT_PT_MAX_GT, DT_LSA_MAX_DIM, DT_PT_MAX_MAP_IDS);
  DT_CHECK_ARG(bytes, "dt_posetrack_mot_smem_bytes: null pointer");
  *bytes = pt_mot_smem_bytes(max(max_gt, 1), max(max_pr, 1), max(map_cap, 1));
  return 0;
}

extern "C" int dt_posetrack_mot(const int* gt_off, const int* pr_off, const long long* pair_off, const double* gt_kp,
                                const int* gt_tid, const double* pr_kp, const int* pr_tid, const double* dist,
                                const int* list_off, const int* list_frames, int nlists, int max_gt, int max_pr, int map_cap,
                                int* counts, double* sumd, int* status, void* stream) {
  size_t smem = 0;
  if (dt_posetrack_mot_smem_bytes(max_gt, max_pr, map_cap, &smem) != 0) return 1;
  DT_CHECK_ARG(nlists >= 0, "dt_posetrack_mot: bad shape nlists=%d", nlists);
  DT_CHECK_ARG(smem <= 227 * 1024, "dt_posetrack_mot: max_gt=%d max_pr=%d map_cap=%d need %zu B of shared memory (> 227 KB)",
               max_gt, max_pr, map_cap, smem);
  if (nlists == 0) return 0;
  DT_CHECK_ARG(gt_off && pr_off && pair_off && list_off && list_frames && counts && sumd, "dt_posetrack_mot: null pointer");
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(pt_mot_kernel, (int)smem, &grant));
  pt_mot_kernel<<<nlists * PTJ, 32, smem, (cudaStream_t)stream>>>(gt_off, pr_off, pair_off, gt_kp, gt_tid, pr_kp, pr_tid, dist,
                                                                  list_off, list_frames, max(max_gt, 1), max(max_pr, 1),
                                                                  max(map_cap, 1), counts, sumd, status);
  DT_CHECK_LAUNCH();
  return 0;
}
