// Pairwise (tube) IoU and greedy NMS as a 64x64-tile bitmask + on-device scan.
//
// Reference semantics (bit-exact; this file is compiled with -fmad=false and
// uses explicit _rn intrinsics so nothing is contracted):
//   lib/utils/cython_bbox.pyx:16-56   IoU with the '+1' convention.  The C that
//       Cython emits promotes every "+ 1" and the area products to fp64 (the
//       literal is written 1.0); box_area / iw / ih are rounded to fp32 when
//       stored.  iou_pair_ref() reproduces that sequence operation by operation.
//   lib/utils/boxes.py:60-69          tubes: sequential fp32 sum over T, / T.
//   lib/utils/cython_nms.pyx:37-87    2-D NMS: fp32 throughout, suppress ovr >= thr,
//       survivors returned in ascending ORIGINAL index.
//   lib/nms/py_cpu_nms_tubes.py:17-53 tube NMS: mean-over-T IoU, a box survives
//       iff ovT <= thr (NaN => suppressed), survivors in score order.
//   lib/nms/nms_kernel.cu:35-150      design lineage (64x64 tiles of u64 masks);
//       unlike it, nothing here allocates, copies to the host or synchronises.
#include "common.cuh"
#include "box_math.cuh"
#include "../../include/dt_b200.h"
#include <math_constants.h>

namespace dt {

// iou_pair_ref (cython_bbox.pyx:34-56, one pair, one frame) lives in box_math.cuh (shared with targets.cu)
// Mean-over-T IoU exactly as boxes.py:60-69 evaluates it.
__device__ __forceinline__ float tube_iou_ref(const float* __restrict__ b,
                                              const float* __restrict__ q, int T) {
  float acc = iou_pair_ref(b, q);
  for (int t = 1; t < T; ++t) acc = __fadd_rn(acc, iou_pair_ref(b + 4 * t, q + 4 * t));
  return __fdiv_rn(acc, (float)T);
}

__global__ void bbox_overlaps_kernel(const float* __restrict__ boxes, int n, int ldb,
                                     const float* __restrict__ query, int k, int ldq,
                                     int T, float* __restrict__ out, int ldo) {
  // x -> query index (contiguous in the output row), y -> box index
  const int kk = blockIdx.x * blockDim.x + threadIdx.x;
  const int nn = blockIdx.y * blockDim.y + threadIdx.y;
  if (kk >= k || nn >= n) return;
  float b[DT_MAX_T * 4], q[DT_MAX_T * 4];
  for (int c = 0; c < 4 * T; ++c) { b[c] = boxes[(size_t)nn * ldb + c]; q[c] = query[(size_t)kk * ldq + c]; }
  out[(size_t)nn * ldo + kk] = tube_iou_ref(b, q, T);
}

// ---------------------------------------------------------------- NMS ------
// IoU as the two NMS implementations compute it (fp32; areas precomputed).
__device__ __forceinline__ float nms_iou_frame(const float* a, float aarea,
                                               const float* b, float barea) {
  const float xx1 = fmaxf(a[0], b[0]), yy1 = fmaxf(a[1], b[1]);
  const float xx2 = fminf(a[2], b[2]), yy2 = fminf(a[3], b[3]);
  const float w = fmaxf(0.f, __fadd_rn(__fsub_rn(xx2, xx1), 1.f));
  const float h = fmaxf(0.f, __fadd_rn(__fsub_rn(yy2, yy1), 1.f));
  const float inter = __fmul_rn(w, h);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(aarea, barea), inter));
}

__device__ __forceinline__ uint32_t float_sort_key(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // ascending uint == ascending float
}

// One CTA per problem: descending-score order with ties broken by descending
// original index (== reversing a stable ascending argsort).  Bitonic in smem.
__global__ void nms_sort_kernel(const float* __restrict__ dets, int nmax, int ld, int T,
                                const int* __restrict__ counts, int npow2,
                                int* __restrict__ order /*[B,nmax]*/) {
  extern __shared__ unsigned long long keys[];
  const int b = blockIdx.x;
  const int n = counts ? min(counts[b], nmax) : nmax;
  const float* d = dets + (size_t)b * nmax * ld;
  for (int i = threadIdx.x; i < npow2; i += blockDim.x) {
    unsigned long long key = 0ull;   // pads sort to the end (descending)
    if (i < n) key = ((unsigned long long)float_sort_key(d[(size_t)i * ld + 4 * T]) << 32) |
                     (unsigned long long)(uint32_t)(i + 1);
    keys[i] = key;
  }
  __syncthreads();
  for (int k = 2; k <= npow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < npow2; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], c = keys[ixj];
          const bool desc = ((i & k) == 0);
          if (desc ? (a < c) : (a > c)) { keys[i] = c; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    order[(size_t)b * nmax + i] = (int)(uint32_t)(keys[i] & 0xffffffffull) - 1;
}

// grid (colblk, rowblk, B), 64 threads.  mask[b][i][cb] bit j set <=> box at sorted
// position cb*64+j is suppressed by the box at sorted position i.
template <int T_CT>
__global__ void nms_mask_kernel(const float* __restrict__ dets, int nmax, int ld, int T_rt,
                                const int* __restrict__ counts, const int* __restrict__ order,
                                float thresh, int cmp_mode,
                                unsigned long long* __restrict__ mask, int nw) {
  const int T = T_CT > 0 ? T_CT : T_rt;
  const int cb = blockIdx.x, rb = blockIdx.y, b = blockIdx.z;
  if (cb < rb) return;
  const int n = counts ? min(counts[b], nmax) : nmax;
  if (rb * 64 >= n || cb * 64 >= n) return;
  const float* d = dets + (size_t)b * nmax * ld;
  const int* ord = order + (size_t)b * nmax;
  __shared__ float cbox[64][DT_MAX_T * 4];
  __shared__ float carea[64][DT_MAX_T];
  const int tid = threadIdx.x;
  const int cj = cb * 64 + tid;
  if (cj < n) {
    const float* p = d + (size_t)ord[cj] * ld;
    for (int t = 0; t < T; ++t) {
      const float x1 = p[4 * t], y1 = p[4 * t + 1], x2 = p[4 * t + 2], y2 = p[4 * t + 3];
      cbox[tid][4 * t] = x1; cbox[tid][4 * t + 1] = y1; cbox[tid][4 * t + 2] = x2; cbox[tid][4 * t + 3] = y2;
      carea[tid][t] = __fmul_rn(__fadd_rn(__fsub_rn(x2, x1), 1.f), __fadd_rn(__fsub_rn(y2, y1), 1.f));
    }
  }
  __syncthreads();
  const int ri = rb * 64 + tid;
  if (ri >= n) return;
  float rbox[DT_MAX_T * 4], rarea[DT_MAX_T];
  {
    const float* p = d + (size_t)ord[ri] * ld;
    for (int t = 0; t < T; ++t) {
      rbox[4 * t] = p[4 * t]; rbox[4 * t + 1] = p[4 * t + 1]; rbox[4 * t + 2] = p[4 * t + 2]; rbox[4 * t + 3] = p[4 * t + 3];
      rarea[t] = __fmul_rn(__fadd_rn(__fsub_rn(rbox[4 * t + 2], rbox[4 * t]), 1.f),
                           __fadd_rn(__fsub_rn(rbox[4 * t + 3], rbox[4 * t + 1]), 1.f));
    }
  }
  unsigned long long bits = 0ull;
  const int jend = min(64, n - cb * 64);
  const int jstart = (cb == rb) ? tid + 1 : 0;
  for (int j = jstart; j < jend; ++j) {
    bool sup;
    if (cmp_mode == DT_NMS_2D_GE) {             // cython_nms.pyx:83-85
      const float ovr = nms_iou_frame(rbox, rarea[0], cbox[j], carea[j][0]);
      sup = (ovr >= thresh);
    } else {                                    // py_cpu_nms_tubes.py:35-51
      float ov = 0.f;
      for (int t = 0; t < T; ++t)
        ov = __fadd_rn(ov, nms_iou_frame(rbox + 4 * t, rarea[t], cbox[j] + 4 * t, carea[j][t]));
      ov = __fdiv_rn(ov, (float)T);
      sup = !(ov <= thresh);
    }
    if (sup) bits |= (1ull << j);
  }
  mask[((size_t)b * nmax + ri) * nw + cb] = bits;
}

// One CTA per problem walks the mask rows in score order.
//   per 64-block: thread 0 resolves the diagonal word serially in registers,
//   then the whole CTA ORs the rows of the newly kept boxes into remv[].
__global__ void nms_scan_kernel(const unsigned long long* __restrict__ mask, int nmax, int nw,
                                const int* __restrict__ counts, const int* __restrict__ order,
                                int out_order, int max_keep,
                                int* __restrict__ keep, int* __restrict__ num_keep,
                                unsigned char* __restrict__ flags /*[B,nmax] scratch*/) {
  extern __shared__ unsigned long long sm[];
  unsigned long long* remv = sm;            // [nw]
  unsigned long long* kept = sm + nw;       // [nw]
  __shared__ unsigned long long diag[64];
  __shared__ unsigned long long s_kept;
  __shared__ int s_total, s_stop;
  const int b = blockIdx.x, tid = threadIdx.x, nth = blockDim.x;
  const int n = counts ? min(counts[b], nmax) : nmax;
  const unsigned long long* m = mask + (size_t)b * nmax * nw;
  const int* ord = order + (size_t)b * nmax;
  int* out = keep + (size_t)b * nmax;
  const int nblk = (n + 63) / 64;
  for (int w = tid; w < nw; w += nth) { remv[w] = 0ull; kept[w] = 0ull; }
  if (tid == 0) { s_total = 0; s_stop = 0; }
  __syncthreads();
  // keep[:max_keep] truncates the RETURNED list (generate_proposals.py:108-110):
  // in score order that is an early exit; in index order all survivors are needed first.
  const int limit = (max_keep > 0) ? max_keep : 0x7fffffff;
  const int stop_at = (out_order == DT_NMS_ORDER_SCORE) ? limit : 0x7fffffff;
  for (int blk = 0; blk < nblk; ++blk) {
    if (tid < 64) {
      const int i = blk * 64 + tid;
      diag[tid] = (i < n) ? m[(size_t)i * nw + blk] : 0ull;
    }
    __syncthreads();
    if (tid == 0) {
      unsigned long long r = remv[blk], k = 0ull;
      int total = s_total;
      const int cnt = min(64, n - blk * 64);
      for (int j = 0; j < cnt; ++j) {
        if (!((r >> j) & 1ull)) {
          k |= (1ull << j);
          r |= diag[j];
          if (++total >= stop_at) { s_stop = 1; break; }
        }
      }
      s_kept = k; s_total = total; kept[blk] = k;
    }
    __syncthreads();
    if (s_stop) break;
    const unsigned long long k = s_kept;
    const int rem = nblk - blk - 1;
    for (int idx = tid; idx < 64 * rem; idx += nth) {
      const int j = idx / rem, w = blk + 1 + idx % rem;
      if ((k >> j) & 1ull) {
        const unsigned long long v = m[(size_t)(blk * 64 + j) * nw + w];
        if (v) atomicOr(&remv[w], v);
      }
    }
    __syncthreads();
  }
  __syncthreads();
  const int total = min(s_total, limit);
  if (tid == 0) num_keep[b] = total;
  if (out_order == DT_NMS_ORDER_SCORE) {
    // rank of sorted position p = popcount of kept bits below it
    for (int w = tid; w < nblk; w += nth) {
      int base = 0;
      for (int x = 0; x < w; ++x) base += __popcll(kept[x]);
      unsigned long long k = kept[w];
      while (k) {
        const int j = __ffsll((long long)k) - 1;
        k &= k - 1;
        out[base++] = ord[w * 64 + j];
      }
    }
  } else {
    // ascending original index: scatter flags, then an ordered block compaction
    unsigned char* f = flags + (size_t)b * nmax;
    for (int i = tid; i < n; i += nth) f[i] = 0;
    __syncthreads();
    for (int w = tid; w < nblk; w += nth) {
      unsigned long long k = kept[w];
      while (k) { const int j = __ffsll((long long)k) - 1; k &= k - 1; f[ord[w * 64 + j]] = 1; }
    }
    __syncthreads();
    __shared__ int s_warp[32];
    __shared__ int s_base;
    if (tid == 0) s_base = 0;
    __syncthreads();
    const int lane = tid & 31, wid = tid >> 5, nwarp = (nth + 31) >> 5;
    for (int start = 0; start < n; start += nth) {
      const int i = start + tid;
      const int v = (i < n) ? f[i] : 0;
      const unsigned bal = __ballot_sync(0xffffffffu, v);
      const int pre = __popc(bal & ((1u << lane) - 1));
      if (lane == 0) s_warp[wid] = __popc(bal);
      __syncthreads();
      int off = s_base;
      for (int x = 0; x < wid; ++x) off += s_warp[x];
      if (v && off + pre < limit) out[off + pre] = i;
      __syncthreads();
      if (tid == 0) { int s = 0; for (int x = 0; x < nwarp; ++x) s += s_warp[x]; s_base += s; }
      __syncthreads();
    }
  }
}

static int next_pow2(int x) { int p = 1; while (p < x) p <<= 1; return p; }

// ------------------------------------------------------------ soft-NMS ------
// lib/utils/cython_nms.pyx:98-203 soft_nms, one CTA per list.  The C that Cython emits for it writes the '+ 1' as
// 1.0, so the widths, the areas and ua are taken in fp64 and rounded to fp32 where they are stored (area, iw, ih, ua);
// iw*ih, ov and the decayed score are fp32; the gaussian weight is exp() of an fp32 argument in fp64, stored fp32.
// Rows keep their original coordinates (box[], by source row); positions hold (score, source row).  Round i:
//   argmax: the first maximum of [i, N) in position order, swapped with row i;
//   decay:  every row of (i, N) once; a row that overlaps the pick and decays below `threshold` is discarded;
//   compaction: the reference fills each discarded position with the current last row, so the k-th discarded position
//   below the new N receives the k-th largest surviving position at or above it.
constexpr int SOFT_NMS_THREADS = 512;
constexpr int SOFT_NMS_MAX_CHUNK = DT_NMS_MAX_BOXES / SOFT_NMS_THREADS;   // positions per thread per round (<= 32)
static_assert(SOFT_NMS_MAX_CHUNK <= 32, "discard flags are kept in one 32-bit mask per thread");

__device__ __forceinline__ float cy_max(float a, float b) { return a >= b ? a : b; }   // cython_nms.pyx:28-32
__device__ __forceinline__ float cy_min(float a, float b) { return a <= b ? a : b; }

__device__ __forceinline__ double soft_side(float lo, float hi) { return __dadd_rn((double)__fsub_rn(hi, lo), 1.0); }

__global__ void __launch_bounds__(SOFT_NMS_THREADS)
soft_nms_kernel(const float* __restrict__ dets, int nmax, int ld, const int* __restrict__ counts, float sigma, float Nt,
                float threshold, int method, float* __restrict__ out, int* __restrict__ out_inds,
                int* __restrict__ out_counts) {
  extern __shared__ float4 sbox[];                                  // [nmax] by source row
  float* ssc = (float*)(sbox + nmax);                               // [nmax] by position
  int* sid = (int*)(ssc + nmax);                                    // [nmax] by position
  int* shole = sid + nmax;                                          // [nmax] compaction scratch
  constexpr int NW = SOFT_NMS_THREADS / 32;
  __shared__ uint32_t red_hi[NW], red_lo[NW];
  __shared__ int wsum[NW];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = counts ? max(0, min(counts[b], nmax)) : nmax;
  const float* d = dets + (size_t)b * nmax * ld;
  for (int r = tid; r < n; r += SOFT_NMS_THREADS) {
    const float* p = d + (size_t)r * ld;
    sbox[r] = make_float4(p[0], p[1], p[2], p[3]);
    ssc[r] = p[4];
    sid[r] = r;
  }
  __syncthreads();
  int N = n;
  for (int i = 0; i < N; ++i) {
    // ---- argmax: key (score order, 8191 - pos, source row); -0 counts as +0, NaN never wins (but at i, where the
    // reference's scan starts from it and no comparison with NaN succeeds)
    uint32_t khi = 0u, klo = 0u;
    for (int p = i + tid; p < N; p += SOFT_NMS_THREADS) {
      float s = ssc[p];
      uint32_t h;
      if (s != s) h = (p == i) ? 0xffffffffu : 0u;
      else { if (s == 0.f) s = 0.f; h = float_sort_key(s); }
      const uint32_t l = ((uint32_t)(DT_NMS_MAX_BOXES - 1 - p) << 13) | (uint32_t)sid[p];
      if (h > khi || (h == khi && l > klo)) { khi = h; klo = l; }
    }
    uint32_t bh = __reduce_max_sync(0xffffffffu, khi);
    uint32_t bl = __reduce_max_sync(0xffffffffu, khi == bh ? klo : 0u);
    if (lane == 0) { red_hi[wid] = bh; red_lo[wid] = bl; }
    __syncthreads();
    khi = lane < NW ? red_hi[lane] : 0u;
    klo = lane < NW ? red_lo[lane] : 0u;
    bh = __reduce_max_sync(0xffffffffu, khi);
    bl = __reduce_max_sync(0xffffffffu, khi == bh ? klo : 0u);
    const int maxpos = DT_NMS_MAX_BOXES - 1 - (int)(bl >> 13);
    const float4 t = sbox[bl & 0x1fffu];
    const double at = __dmul_rn(soft_side(t.x, t.z), soft_side(t.y, t.w));
    // ---- decay of (i, N), chunk [c0, c1) per thread; the owner of maxpos also moves row i there
    const int M = N - i - 1;
    const int chunk = (M + SOFT_NMS_THREADS - 1) / SOFT_NMS_THREADS;
    const int c0 = i + 1 + tid * chunk, c1 = min(c0 + chunk, N);
    uint32_t flags = 0u;
    int nd = 0;
    for (int p = c0; p < c1; ++p) {
      int r = sid[p];
      float s = ssc[p];
      if (p == maxpos) {                          // swap: the pick goes to i, row i to maxpos
        const int ri = sid[i];
        const float si = ssc[i];
        sid[i] = r; ssc[i] = s;
        sid[p] = ri; r = ri; s = si;
      }
      const float4 q = sbox[r];
      const float area = __double2float_rn(__dmul_rn(soft_side(q.x, q.z), soft_side(q.y, q.w)));
      const float iw = __double2float_rn(__dadd_rn((double)__fsub_rn(cy_min(t.z, q.z), cy_max(t.x, q.x)), 1.0));
      if (iw > 0.f) {
        const float ih = __double2float_rn(__dadd_rn((double)__fsub_rn(cy_min(t.w, q.w), cy_max(t.y, q.y)), 1.0));
        if (ih > 0.f) {
          const float inter = __fmul_rn(iw, ih);
          const float ua = __double2float_rn(__dsub_rn(__dadd_rn(at, (double)area), (double)inter));
          const float ov = __fdiv_rn(inter, ua);
          float w;
          if (method == 1) w = ov > Nt ? __double2float_rn(__dsub_rn(1.0, (double)ov)) : 1.f;
          else if (method == 2) w = __double2float_rn(exp((double)__fdiv_rn(-__fmul_rn(ov, ov), sigma)));
          else w = ov > Nt ? 0.f : 1.f;
          s = __fmul_rn(w, s);
          if (s < threshold) { flags |= 1u << (p - c0); ++nd; }
        }
      }
      ssc[p] = s;
    }
    // ---- discards: block-wide exclusive scan of the per-thread counts
    int inc = nd;
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
    if (lane == 31) wsum[wid] = inc;
    __syncthreads();
    int D = 0, before = inc - nd;
    for (int w = 0; w < NW; ++w) { const int v = wsum[w]; D += v; if (w < wid) before += v; }
    if (D == 0) continue;                         // uniform: nothing moves
    const int newN = N - D;
    int seen = before;                            // discards at positions < p
    for (int p = c0; p < c1; ++p)
      if ((flags >> (p - c0)) & 1u) { if (p < newN) shole[seen] = p; ++seen; }
    __syncthreads();
    seen = before;
    for (int p = c0; p < c1; ++p) {
      const bool disc = (flags >> (p - c0)) & 1u;
      if (disc) ++seen;
      else if (p >= newN) {
        const int k = (N - 1 - p) - (D - seen);   // surviving positions above p
        const int dst = shole[k];
        ssc[dst] = ssc[p]; sid[dst] = sid[p];
      }
    }
    N = newN;
    __syncthreads();
  }
  float* o = out + (size_t)b * nmax * 5;
  for (int p = tid; p < N; p += SOFT_NMS_THREADS) {
    const int r = sid[p];
    const float4 q = sbox[r];
    o[p * 5 + 0] = q.x; o[p * 5 + 1] = q.y; o[p * 5 + 2] = q.z; o[p * 5 + 3] = q.w; o[p * 5 + 4] = ssc[p];
    if (out_inds) out_inds[(size_t)b * nmax + p] = r;
  }
  if (tid == 0) out_counts[b] = N;
}

// ---------------------------------------------------------- box voting ------
// lib/utils/boxes.py:294-310 box_voting, one thread per top row: the rows of `all` whose cython_bbox IoU with it
// is >= thresh, in ascending row order, give np.average(boxes, axis=0, weights=scores) (numpy 2.x, fp32):
//   numerator   sequential fp32 sum of box * w over the matches (a reduction over the outer axis);
//   denominator numpy's pairwise_sum of the weights: below 8 a plain loop, up to 128 eight accumulators then the
//               remainder, above that the halves n2 = n/2 - (n/2) % 8 and n - n2 summed recursively;
//   then one fp32 division.  The weights are streamed in match order, so the recursion is walked depth first.
constexpr int VOTE_MAX_DEPTH = 8;                // 8192 -> 128 halves six times

struct PairwiseStream {
  int stack_right[VOTE_MAX_DEPTH];               // pending right-half sizes
  float stack_left[VOTE_MAX_DEPTH];              // finished left-half sums
  bool stack_has_left[VOTE_MAX_DEPTH];
  int depth;
  int leaf_n, leaf_k;                            // current leaf size, elements consumed in it
  float r[8], res;
  float total;

  __device__ void open(int n) {
    while (n > 128) {
      int n2 = n / 2;
      n2 -= n2 % 8;
      stack_right[depth] = n - n2; stack_has_left[depth] = false; ++depth;
      n = n2;
    }
    leaf_n = n; leaf_k = 0; res = 0.f;
  }
  __device__ void start(int n) { depth = 0; total = 0.f; open(n); }
  __device__ void push(float w) {
    const int n = leaf_n, k = leaf_k++;
    if (n < 8) res = __fadd_rn(res, w);
    else {
      const int main_n = n - n % 8;
      if (k < 8) r[k] = w;
      else if (k < main_n) r[k & 7] = __fadd_rn(r[k & 7], w);
      else res = __fadd_rn(res, w);              // the remainder, after the eight accumulators are folded
      if (k == main_n - 1)
        res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                        __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    }
    if (leaf_k < n) return;
    float v = res;                               // leaf done: combine up the stack
    while (depth > 0) {
      const int top = depth - 1;
      if (!stack_has_left[top]) {
        stack_left[top] = v; stack_has_left[top] = true;
        open(stack_right[top]);
        return;
      }
      v = __fadd_rn(stack_left[top], v);
      --depth;
    }
    total = v;
  }
};

__global__ void box_vote_kernel(const float* __restrict__ top, const int* __restrict__ top_keep,
                                const int* __restrict__ top_counts, int top_nmax, int ld_top,
                                const float* __restrict__ all, const int* __restrict__ all_counts, int nmax, int ld,
                                float thresh, float* __restrict__ out, int* __restrict__ out_counts) {
  const int b = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int ntop = max(0, min(top_counts[b], top_nmax));
  if (k == 0) out_counts[b] = ntop;
  if (k >= ntop) return;
  const int n = all_counts ? max(0, min(all_counts[b], nmax)) : nmax;
  const float* a = all + (size_t)b * nmax * ld;
  const float* tp = top_keep ? a + (size_t)top_keep[(size_t)b * top_nmax + k] * ld
                             : top + ((size_t)b * top_nmax + k) * ld_top;
  const float tb[4] = {tp[0], tp[1], tp[2], tp[3]};
  const float score = tp[4];
  int m = 0;
  for (int j = 0; j < n; ++j) m += iou_pair_ref(tb, a + (size_t)j * ld) >= thresh;
  PairwiseStream ps;
  ps.start(m);
  float num0 = 0.f, num1 = 0.f, num2 = 0.f, num3 = 0.f;
  for (int j = 0; j < n && m > 0; ++j) {
    const float* q = a + (size_t)j * ld;
    if (!(iou_pair_ref(tb, q) >= thresh)) continue;
    const float w = q[4];
    num0 = __fadd_rn(num0, __fmul_rn(q[0], w)); num1 = __fadd_rn(num1, __fmul_rn(q[1], w));
    num2 = __fadd_rn(num2, __fmul_rn(q[2], w)); num3 = __fadd_rn(num3, __fmul_rn(q[3], w));
    ps.push(w);
  }
  float* o = out + ((size_t)b * top_nmax + k) * 5;
  o[0] = __fdiv_rn(num0, ps.total); o[1] = __fdiv_rn(num1, ps.total);
  o[2] = __fdiv_rn(num2, ps.total); o[3] = __fdiv_rn(num3, ps.total);
  o[4] = score;
}

}  // namespace dt

using namespace dt;

extern "C" int dt_bbox_overlaps(const float* boxes, int n, int ldb, const float* query, int k,
                                int ldq, int T, float* out, int ldo, void* stream) {
  DT_CHECK_ARG(T >= 1 && T <= DT_MAX_T, "dt_bbox_overlaps: T=%d outside [1,%d]", T, DT_MAX_T);
  DT_CHECK_ARG(n >= 0 && k >= 0 && ldb >= 4 * T && ldq >= 4 * T && ldo >= k,
               "dt_bbox_overlaps: bad shape n=%d k=%d ldb=%d ldq=%d ldo=%d T=%d", n, k, ldb, ldq, ldo, T);
  if (n == 0 || k == 0) return 0;
  DT_CHECK_ARG(boxes && query && out, "dt_bbox_overlaps: null pointer");
  dim3 blk(32, 8), grd(cdiv(k, 32), cdiv(n, 8));
  bbox_overlaps_kernel<<<grd, blk, 0, (cudaStream_t)stream>>>(boxes, n, ldb, query, k, ldq, T, out, ldo);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_nms_workspace_bytes(int batch, int nmax, size_t* bytes) {
  DT_CHECK_ARG(batch >= 0 && nmax >= 0 && bytes, "dt_nms_workspace_bytes: bad args");
  const size_t nw = (size_t)cdiv(nmax, 64);
  size_t b = 0;
  b += align_up((size_t)batch * nmax * sizeof(int), 256);                       // order
  b += align_up((size_t)batch * nmax * nw * sizeof(unsigned long long), 256);   // mask
  b += align_up((size_t)batch * nmax, 256);                                     // flags
  *bytes = b;
  return 0;
}

extern "C" int dt_nms_batched(const float* dets, int batch, int nmax, int ld, int T,
                              const int* counts, float thresh, int cmp_mode, int out_order,
                              int max_keep, int* keep, int* num_keep, void* workspace,
                              size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  DT_CHECK_ARG(T >= 1 && T <= DT_MAX_T, "dt_nms_batched: T=%d outside [1,%d]", T, DT_MAX_T);
  DT_CHECK_ARG(batch >= 0 && nmax >= 0 && ld >= 4 * T + 1,
               "dt_nms_batched: bad shape batch=%d nmax=%d ld=%d T=%d (need ld >= 4T+1)", batch, nmax, ld, T);
  DT_CHECK_ARG(nmax <= DT_NMS_MAX_BOXES, "dt_nms_batched: nmax=%d exceeds %d", nmax, DT_NMS_MAX_BOXES);
  DT_CHECK_ARG(cmp_mode == DT_NMS_2D_GE || cmp_mode == DT_NMS_TUBE_GT, "dt_nms_batched: bad cmp_mode %d", cmp_mode);
  DT_CHECK_ARG(cmp_mode == DT_NMS_TUBE_GT || T == 1, "dt_nms_batched: the 2-D '>=' path takes T=1 (nms_wrapper.py:53-57)");
  DT_CHECK_ARG(out_order == DT_NMS_ORDER_SCORE || out_order == DT_NMS_ORDER_INDEX, "dt_nms_batched: bad out_order %d", out_order);
  if (batch == 0) return 0;
  DT_CHECK_ARG(keep && num_keep, "dt_nms_batched: null output");
  if (nmax == 0) { DT_CHECK_CUDA(cudaMemsetAsync(num_keep, 0, sizeof(int) * batch, stream)); return 0; }
  DT_CHECK_ARG(dets && workspace, "dt_nms_batched: null pointer");
  size_t need; dt_nms_workspace_bytes(batch, nmax, &need);
  DT_CHECK_ARG(workspace_bytes >= need, "dt_nms_batched: workspace %zu < %zu bytes", workspace_bytes, need);
  const int nw = cdiv(nmax, 64);
  char* ws = (char*)workspace;
  int* order = (int*)ws; ws += align_up((size_t)batch * nmax * sizeof(int), 256);
  unsigned long long* mask = (unsigned long long*)ws; ws += align_up((size_t)batch * nmax * nw * sizeof(unsigned long long), 256);
  unsigned char* flags = (unsigned char*)ws;

  const int npow2 = next_pow2(nmax);
  const size_t sort_smem = (size_t)npow2 * sizeof(unsigned long long);
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(nms_sort_kernel, (int)(next_pow2(DT_NMS_MAX_BOXES) * sizeof(unsigned long long)), &grant));
  nms_sort_kernel<<<batch, npow2 >= 1024 ? 1024 : (npow2 < 64 ? 64 : npow2), sort_smem, stream>>>(
      dets, nmax, ld, T, counts, npow2, order);
  DT_CHECK_LAUNCH();
  dim3 grd(nw, nw, batch);
  if (T == 1)
    nms_mask_kernel<1><<<grd, 64, 0, stream>>>(dets, nmax, ld, T, counts, order, thresh, cmp_mode, mask, nw);
  else if (T == 3)
    nms_mask_kernel<3><<<grd, 64, 0, stream>>>(dets, nmax, ld, T, counts, order, thresh, cmp_mode, mask, nw);
  else
    nms_mask_kernel<0><<<grd, 64, 0, stream>>>(dets, nmax, ld, T, counts, order, thresh, cmp_mode, mask, nw);
  DT_CHECK_LAUNCH();
  nms_scan_kernel<<<batch, 256, 2 * nw * sizeof(unsigned long long), stream>>>(
      mask, nmax, nw, counts, order, out_order, max_keep, keep, num_keep, flags);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_soft_nms_batched(const float* dets, int batch, int nmax, int ld, const int* counts, float sigma,
                                   float Nt, float threshold, int method, float* out, int* out_inds, int* out_counts,
                                   void* stream) {
  DT_CHECK_ARG(method >= DT_SOFT_NMS_HARD && method <= DT_SOFT_NMS_GAUSSIAN,
               "dt_soft_nms_batched: method %d is not 0 (hard), 1 (linear) or 2 (gaussian)", method);
  DT_CHECK_ARG(batch >= 0 && nmax >= 0 && ld >= 5,
               "dt_soft_nms_batched: bad shape batch=%d nmax=%d ld=%d (need ld >= 5: 2-D boxes only)", batch, nmax, ld);
  DT_CHECK_ARG(nmax <= DT_NMS_MAX_BOXES, "dt_soft_nms_batched: nmax=%d exceeds %d", nmax, DT_NMS_MAX_BOXES);
  if (batch == 0) return 0;
  DT_CHECK_ARG(out && out_counts, "dt_soft_nms_batched: null output");
  if (nmax == 0) { DT_CHECK_CUDA(cudaMemsetAsync(out_counts, 0, sizeof(int) * batch, (cudaStream_t)stream)); return 0; }
  DT_CHECK_ARG(dets, "dt_soft_nms_batched: null dets");
  const size_t smem = (size_t)nmax * (sizeof(float4) + sizeof(float) + 2 * sizeof(int));
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(soft_nms_kernel, (int)(DT_NMS_MAX_BOXES * (sizeof(float4) + sizeof(float) + 2 * sizeof(int))),
                               &grant));
  soft_nms_kernel<<<batch, SOFT_NMS_THREADS, smem, (cudaStream_t)stream>>>(dets, nmax, ld, counts, sigma, Nt, threshold,
                                                                          method, out, out_inds, out_counts);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_box_vote(const float* top, const int* top_keep, const int* top_counts, int top_nmax, int ld_top,
                           const float* all, const int* all_counts, int batch, int nmax, int ld, float thresh, float* out,
                           int* out_counts, void* stream) {
  DT_CHECK_ARG(batch >= 0 && nmax >= 0 && top_nmax >= 0 && ld >= 5 && (top_keep || ld_top >= 5),
               "dt_box_vote: bad shape batch=%d nmax=%d ld=%d top_nmax=%d ld_top=%d (need ld, ld_top >= 5: 2-D boxes only)",
               batch, nmax, ld, top_nmax, ld_top);
  DT_CHECK_ARG(nmax <= DT_NMS_MAX_BOXES && top_nmax <= DT_NMS_MAX_BOXES, "dt_box_vote: nmax=%d / top_nmax=%d exceeds %d",
               nmax, top_nmax, DT_NMS_MAX_BOXES);
  DT_CHECK_ARG(!top_keep || top_nmax == nmax, "dt_box_vote: a keep list indexes `all`: top_nmax=%d must equal nmax=%d",
               top_nmax, nmax);
  if (batch == 0) return 0;
  DT_CHECK_ARG(top_counts && out && out_counts, "dt_box_vote: null pointer");
  if (top_nmax == 0) { DT_CHECK_CUDA(cudaMemsetAsync(out_counts, 0, sizeof(int) * batch, (cudaStream_t)stream)); return 0; }
  DT_CHECK_ARG(all && (top_keep || top), "dt_box_vote: null rows");
  dim3 grid(cdiv(top_nmax, 128), batch);
  box_vote_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(top, top_keep, top_counts, top_nmax, ld_top, all, all_counts,
                                                           nmax, ld, thresh, out, out_counts);
  DT_CHECK_LAUNCH();
  return 0;
}
