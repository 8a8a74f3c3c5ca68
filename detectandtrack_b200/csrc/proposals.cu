// RPN proposal generation and detection post-processing on the device (no host round trips).
//
//   dt_rpn_proposals      lib/ops/generate_proposals.py:40-196 up to (not including) NMS:
//                         sigmoid, top-k, anchor enumeration, bbox/tube decode, clip, min-size filter
//   dt_collect_rpn        lib/ops/collect_and_distribute_fpn_rpn_proposals.py:44-62
//   dt_distribute_fpn     same file :65-87 + lib/modeling/FPN.py:349-360 (level per RoI, restore index)
//   dt_box_decode         lib/core/test.py:211-252 (unscale, bbox_transform, clip) + :750-766 score filter
//   dt_limit_detections   lib/core/test.py:790-800 (DETECTIONS_PER_IM threshold) and gather of kept rows
// NMS itself is dt_nms_batched (boxes.cu).
//
// Arithmetic follows the reference's dtype promotions (see oracle/boxes.py): the 2-D decode is
// fp32 op by op (lib/utils/boxes.py:141-183); the tube decode (T > 1) runs in fp64 and is rounded
// once to fp32 (boxes.py:26-57 promotes the parts to float64).  exp() of the fp32 path may differ
// from numpy's by an ulp (tolerance 1e-3 relative, stated in the tests); everything integer
// (selection, ordering, filtering, levels, indices) is exact given the same float inputs.
// Score ties: the reference's order is undefined; here: descending score, then ascending index.
#include "common.cuh"
#include "../../include/dt_b200.h"
#include <cuda_bf16.h>
#include <cooperative_groups.h>
#include <math_constants.h>

namespace dt {

__device__ __forceinline__ uint32_t sort_key_f32(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float sigmoidf_ref(float x) {      // Caffe2 Sigmoid: 1 / (1 + exp(-x))
  return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
}

// In-place bitonic sort (descending) of n = power-of-two u64 keys in shared memory.
__device__ void bitonic_desc(unsigned long long* keys, int npow2) {
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
}

// Ordered block compaction helper: returns the exclusive rank of `flag` among all threads'
// flags in thread order, adds the block total to *running (shared).  All threads must call.
__device__ int block_rank(bool flag, int* s_warp, int* running) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) s_warp[wid] = __popc(bal);
  __syncthreads();
  int off = *running;
  for (int x = 0; x < wid; ++x) off += s_warp[x];
  off += __popc(bal & ((1u << lane) - 1));
  __syncthreads();
  if (threadIdx.x == 0) { int t = 0; for (int x = 0; x < nwarp; ++x) t += s_warp[x]; *running += t; }
  __syncthreads();
  return off;
}

// boxes.py:141-183 for one box / one 4-vector of deltas, fp32 op order.
__device__ __forceinline__ void decode_f32(const float* bx, const float* dl, float wx, float wy, float ww, float wh,
                                           float clipv, float* o) {
  const float w = __fadd_rn(__fsub_rn(bx[2], bx[0]), 1.f);
  const float h = __fadd_rn(__fsub_rn(bx[3], bx[1]), 1.f);
  const float cx = __fadd_rn(bx[0], __fmul_rn(0.5f, w));
  const float cy = __fadd_rn(bx[1], __fmul_rn(0.5f, h));
  const float dx = __fdiv_rn(dl[0], wx), dy = __fdiv_rn(dl[1], wy);
  const float dw = fminf(__fdiv_rn(dl[2], ww), clipv), dh = fminf(__fdiv_rn(dl[3], wh), clipv);
  const float pcx = __fadd_rn(__fmul_rn(dx, w), cx), pcy = __fadd_rn(__fmul_rn(dy, h), cy);
  const float pw = __fmul_rn(expf(dw), w), ph = __fmul_rn(expf(dh), h);
  o[0] = __fsub_rn(pcx, __fmul_rn(0.5f, pw));
  o[1] = __fsub_rn(pcy, __fmul_rn(0.5f, ph));
  o[2] = __fadd_rn(pcx, __fmul_rn(0.5f, pw));
  o[3] = __fadd_rn(pcy, __fmul_rn(0.5f, ph));
}
// Same in fp64 (tube path), rounded to fp32 on store.
__device__ __forceinline__ void decode_f64(const double* bx, const float* dl, double wx, double wy, double ww,
                                           double wh, double clipv, float* o) {
  const double w = __dadd_rn(__dsub_rn(bx[2], bx[0]), 1.0);
  const double h = __dadd_rn(__dsub_rn(bx[3], bx[1]), 1.0);
  const double cx = __dadd_rn(bx[0], __dmul_rn(0.5, w));
  const double cy = __dadd_rn(bx[1], __dmul_rn(0.5, h));
  const double dx = __ddiv_rn((double)dl[0], wx), dy = __ddiv_rn((double)dl[1], wy);
  const double dw = fmin(__ddiv_rn((double)dl[2], ww), clipv), dh = fmin(__ddiv_rn((double)dl[3], wh), clipv);
  const double pcx = __dadd_rn(__dmul_rn(dx, w), cx), pcy = __dadd_rn(__dmul_rn(dy, h), cy);
  const double pw = __dmul_rn(exp(dw), w), ph = __dmul_rn(exp(dh), h);
  o[0] = (float)__dsub_rn(pcx, __dmul_rn(0.5, pw));
  o[1] = (float)__dsub_rn(pcy, __dmul_rn(0.5, ph));
  o[2] = (float)__dadd_rn(pcx, __dmul_rn(0.5, pw));
  o[3] = (float)__dadd_rn(pcy, __dmul_rn(0.5, ph));
}

__device__ __forceinline__ float load_act(const void* p, size_t i, int f32) {
  return f32 ? reinterpret_cast<const float*>(p)[i]
             : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
}

// ------------------------------------------------------------------- RPN top-k + decode
// One 8-CTA cluster per (image, level): all FPN levels of a clip batch run in ONE launch.
// logits [B, H*W, ld_s] (first A channels), deltas [B, H*W, ld_d] (first 4*A*T).
// Flat anchor index i = (h*W + w)*A + a  (generate_proposals.py:58-70 ordering).
struct RpnLevel {
  const void* logits; const void* deltas; const double* anchors;
  int ld_s, ld_d, H, W;
  double feat_stride;
  float* out; int* counts;            // out rows [4T+1] per image at out + b*out_bstride; counts[b*counts_stride]
  uint32_t* keys;                     // scratch [B, H*W*A] sortable score keys
};
struct RpnLevels { RpnLevel lv[8]; };

// A thread-block CLUSTER of RPN_CS CTAs works on one (image, level): the big levels are pure streaming (P2:
// 604 800 anchors, ~25 MB through several passes) and one SM moves ~0.1 TB/s, so a single CTA per image-level
// took 0.55 ms while 80 % of the GPU idled.  Every CTA owns a fixed strided slice of the anchors in all passes
// (so it only ever re-reads keys it wrote itself); histograms, counts and the selected candidates are exchanged
// through distributed shared memory; rank 0 sorts and decodes the K survivors.
constexpr int RPN_CS = 8;

__global__ void __launch_bounds__(1024, 1)
rpn_proposals_kernel(const RpnLevels L, int act_f32, int A, int T, const float* __restrict__ im_info /*[B,3]*/,
                     int pre_topn, float min_size, float clipv_f, double clipv_d, long long out_bstride,
                     int counts_stride, int kcap /*pow2 >= K*/, int time_major) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ unsigned long long skeys[];          // [kcap] selected (key<<32 | ~idx)
  __shared__ __align__(16) int hist[4096];
  __shared__ int s_warp[32];
  __shared__ int s_run, s_bin, s_need, s_cnt;
  __shared__ uint32_t s_lo, s_hi;
  const RpnLevel& lv = L.lv[blockIdx.y];
  const void* __restrict__ logits = lv.logits;
  const void* __restrict__ deltas = lv.deltas;
  const double* __restrict__ anchors = lv.anchors;
  const int ld_s = lv.ld_s, ld_d = lv.ld_d, H = lv.H, W = lv.W;
  const double feat_stride = lv.feat_stride;
  const int CS = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int b = blockIdx.x / CS, tid = threadIdx.x, nth = blockDim.x;
  const int n = H * W * A;
  const int K = (pre_topn <= 0 || pre_topn > n) ? n : pre_topn;
  const int i0 = rank * nth + tid, istep = CS * nth;    // this thread's slice of the anchors, every pass
  uint32_t* __restrict__ keys = lv.keys + (size_t)b * n;
  // time_major (3-D RPN head, model_builder.py:509-563): logits / deltas are [B, T, H*W, ld] with A / 4A
  // channels per frame; the tube score is the mean over frames of the per-frame logits (TimePool 'avg',
  // sequential fp32 sum then / T) and delta (a, t, k) lives at frame t, channel a*4 + k.
  const size_t HW = (size_t)H * W;
  const size_t sbase = (size_t)b * HW * ld_s * (time_major ? T : 1);
  auto score_at = [&](int i) -> float {
    const int pos = i / A, a = i - pos * A;
    if (!time_major) return sigmoidf_ref(load_act(logits, sbase + (size_t)pos * ld_s + a, act_f32));
    float acc = load_act(logits, sbase + (size_t)pos * ld_s + a, act_f32);
    for (int t = 1; t < T; ++t) acc = __fadd_rn(acc, load_act(logits, sbase + ((size_t)t * HW + pos) * ld_s + a, act_f32));
    return sigmoidf_ref(__fdiv_rn(acc, (float)T));
  };
  // ---- pass 0: scores -> sortable keys (stored once), min / max over the cluster -----------------
  if (tid == 0) { s_lo = 0xffffffffu; s_hi = 0u; }
  __syncthreads();
  uint32_t tlo = 0xffffffffu, thi = 0u;
  for (int i = i0; i < n; i += istep) {
    const uint32_t key = sort_key_f32(score_at(i));
    keys[i] = key;
    tlo = min(tlo, key); thi = max(thi, key);
  }
  for (int o = 16; o > 0; o >>= 1) { tlo = min(tlo, __shfl_xor_sync(0xffffffffu, tlo, o)); thi = max(thi, __shfl_xor_sync(0xffffffffu, thi, o)); }
  if ((tid & 31) == 0) { atomicMin(&s_lo, tlo); atomicMax(&s_hi, thi); }
  __threadfence();                       // the tie fallback below lets rank 0 read every slice's keys
  cluster.sync();
  uint32_t lo = 0xffffffffu, hi = 0u;
  for (int r = 0; r < CS; ++r) {
    lo = min(lo, *cluster.map_shared_rank(&s_lo, r));
    hi = max(hi, *cluster.map_shared_rank(&s_hi, r));
  }
  // ---- exact K-th largest key: iterative range refinement with 4096 adaptive-width bins ----------
  // invariant: `need` of the elements with key in [lo, hi] belong to the top K (all keys > hi already do)
  int need = K;
  while (lo < hi) {
    const unsigned long long range = (unsigned long long)hi - lo + 1ull;
    int shift = 0;
    while ((range >> shift) > 4096ull) ++shift;
    for (int x = tid; x < 4096; x += nth) hist[x] = 0;
    __syncthreads();
    for (int i = i0; i < n; i += istep) {
      const uint32_t key = keys[i];
      if (key >= lo && key <= hi) {
        // warp-aggregated histogram update: RPN scores cluster, so many lanes hit the same bin
        const int bin = (int)((key - lo) >> shift);
        const unsigned peers = __match_any_sync(__activemask(), bin);
        if ((int)(__ffs(peers) - 1) == (tid & 31)) atomicAdd(&hist[bin], __popc(peers));
      }
    }
    __syncthreads();
    cluster.sync();                      // every CTA's histogram is complete
    // cluster-wide histogram of this thread's four bins (every CTA computes the same totals), then the bin
    // holding the need-th largest element by a block-wide suffix scan (thread t owns bins 4t .. 4t+3)
    int h[4] = {0, 0, 0, 0};
    for (int r = 0; r < CS; ++r) {
      const int4 q = *reinterpret_cast<const int4*>(cluster.map_shared_rank(&hist[0], r) + 4 * tid);
      h[0] += q.x; h[1] += q.y; h[2] += q.z; h[3] += q.w;
    }
    const int local = h[0] + h[1] + h[2] + h[3];
    int suf = local;                     // inclusive suffix sum over lanes >= this one
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_down_sync(0xffffffffu, suf, o); if ((tid & 31) + o < 32) suf += v; }
    if ((tid & 31) == 0) s_warp[tid >> 5] = suf;
    __syncthreads();
    int above = suf - local;             // elements in bins above this thread's four
    for (int w = (tid >> 5) + 1; w < (nth >> 5); ++w) above += s_warp[w];
    if (above < need && above + local >= need) {          // exactly one thread
      int cum = above, bin = 4 * tid + 3;
      for (int j = 3; j >= 0; --j, --bin) { if (cum + h[j] >= need) break; cum += h[j]; }
      s_bin = bin; s_need = need - cum;
    }
    __syncthreads();
    const uint32_t nlo = lo + ((uint32_t)s_bin << shift);
    const unsigned long long nhi64 = (unsigned long long)nlo + ((1ull << shift) - 1ull);
    hi = (nhi64 > hi) ? hi : (uint32_t)nhi64;
    lo = nlo;
    need = s_need;
    cluster.sync();                      // peers are done reading this CTA's histogram / s_bin is consumed
  }
  const uint32_t kth = lo;              // keys > kth are all selected; `need` keys == kth, lowest index first
  // ---- gather the selected candidates of this slice into this CTA's list.  Order is fixed by the sort below,
  // so keys > kth are appended unordered; keys == kth must be the `need` LOWEST indices: unordered too when
  // every equal key is taken (the usual case: a unique K-th score), otherwise rank 0 compacts them in order.
  if (tid == 0) { s_run = 0; s_cnt = 0; }
  for (int x = tid; x < kcap; x += nth) skeys[x] = 0ull;
  __syncthreads();
  int my_eq = 0;
  for (int i = i0; i < n; i += istep) {
    const uint32_t key = keys[i];
    if (key > kth) {
      const int slot = atomicAdd(&s_run, 1);
      skeys[slot] = ((unsigned long long)key << 32) | (unsigned long long)(0xffffffffu - (uint32_t)i);
    } else if (key == kth) ++my_eq;
  }
  if (my_eq) atomicAdd(&s_cnt, my_eq);
  __syncthreads();
  cluster.sync();
  int total_eq = 0;
  for (int r = 0; r < CS; ++r) total_eq += *cluster.map_shared_rank(&s_cnt, r);
  const bool take_all_eq = (total_eq == need);
  if (take_all_eq) {
    for (int i = i0; i < n; i += istep)
      if (keys[i] == kth) {
        const int slot = atomicAdd(&s_run, 1);
        skeys[slot] = ((unsigned long long)kth << 32) | (unsigned long long)(0xffffffffu - (uint32_t)i);
      }
    __syncthreads();
  }
  cluster.sync();                        // every list is final
  if (rank == 0) {
    // concatenate the peers' lists behind this CTA's own
    int off = s_run;
    for (int r = 1; r < CS; ++r) {
      const int cnt = *cluster.map_shared_rank(&s_run, r);
      const unsigned long long* src = cluster.map_shared_rank(&skeys[0], r);
      for (int x = tid; x < cnt; x += nth) skeys[off + x] = src[x];
      off += cnt;
    }
    __syncthreads();
    if (tid == 0) s_run = off;
    __syncthreads();
  }
  cluster.sync();                        // peers may exit: nobody reads their shared memory any more
  if (rank != 0) return;
  if (!take_all_eq) {
    int eq_base = 0;                     // == kth elements seen so far (uniform)
    for (int start = 0; start < n && eq_base < need; start += nth) {
      const int i = start + tid;
      const bool eq = (i < n) && keys[i] == kth;
      const int lane = tid & 31, wid = tid >> 5, nwarp = nth >> 5;
      const unsigned bal = __ballot_sync(0xffffffffu, eq);
      if (lane == 0) s_warp[wid] = __popc(bal);
      __syncthreads();
      int eoff = eq_base, etot = 0;
      for (int x = 0; x < nwarp; ++x) { if (x < wid) eoff += s_warp[x]; etot += s_warp[x]; }
      eoff += __popc(bal & ((1u << lane) - 1));
      if (eq && eoff < need) {
        const int slot = atomicAdd(&s_run, 1);
        skeys[slot] = ((unsigned long long)kth << 32) | (unsigned long long)(0xffffffffu - (uint32_t)i);
      }
      eq_base += etot;
      __syncthreads();
    }
    __syncthreads();
  }
  bitonic_desc(skeys, kcap);             // descending score, ascending index on ties
  // ---- decode / clip / filter the K candidates in order --------------------------------------
  const float imh = im_info[3 * b], imw = im_info[3 * b + 1], imscale = im_info[3 * b + 2];
  const float hmax = __fsub_rn(imh, 1.f), wmax = __fsub_rn(imw, 1.f);
  const float msz = __fmul_rn(min_size, imscale);
  const size_t dbase = (size_t)b * HW * ld_d * (time_major ? T : 1);
  const int ldo = 4 * T + 1;
  float* __restrict__ out = lv.out;
  if (tid == 0) s_run = 0;
  __syncthreads();
  for (int start = 0; start < K; start += nth) {
    const int r = start + tid;
    bool ok = false;
    float box[DT_MAX_T * 4];
    float sc = 0.f;
    if (r < K) {
      const unsigned long long kk = skeys[r];
      const int i = (int)(0xffffffffu - (uint32_t)(kk & 0xffffffffull));
      const int pos = i / A, a = i - pos * A;
      const int hh = pos / W, ww = pos - hh * W;
      sc = score_at(i);
      const double shx = (double)ww * feat_stride, shy = (double)hh * feat_stride;
      ok = true;
      for (int t = 0; t < T; ++t) {
        double an[4];
        an[0] = anchors[(size_t)a * 4 * T + 4 * t + 0] + shx; an[1] = anchors[(size_t)a * 4 * T + 4 * t + 1] + shy;
        an[2] = anchors[(size_t)a * 4 * T + 4 * t + 2] + shx; an[3] = anchors[(size_t)a * 4 * T + 4 * t + 3] + shy;
        float dl[4];
        for (int k = 0; k < 4; ++k)
          dl[k] = time_major ? load_act(deltas, dbase + ((size_t)t * HW + pos) * ld_d + (size_t)a * 4 + k, act_f32)
                             : load_act(deltas, dbase + (size_t)pos * ld_d + (size_t)a * 4 * T + 4 * t + k, act_f32);
        float* o = box + 4 * t;
        if (T == 1) {
          const float af[4] = {(float)an[0], (float)an[1], (float)an[2], (float)an[3]};
          decode_f32(af, dl, 1.f, 1.f, 1.f, 1.f, clipv_f, o);
        } else {
          decode_f64(an, dl, 1.0, 1.0, 1.0, 1.0, clipv_d, o);
        }
        // clip_tiled_boxes (boxes.py:243-253)
        o[0] = fmaxf(fminf(o[0], wmax), 0.f); o[1] = fmaxf(fminf(o[1], hmax), 0.f);
        o[2] = fmaxf(fminf(o[2], wmax), 0.f); o[3] = fmaxf(fminf(o[3], hmax), 0.f);
        // _filter_boxes (generate_proposals.py:184-196), AND over frames
        const float ws = __fadd_rn(__fsub_rn(o[2], o[0]), 1.f), hs = __fadd_rn(__fsub_rn(o[3], o[1]), 1.f);
        const float xc = __fadd_rn(o[0], __fdiv_rn(ws, 2.f)), yc = __fadd_rn(o[1], __fdiv_rn(hs, 2.f));
        ok = ok && (ws >= msz) && (hs >= msz) && (xc < imw) && (yc < imh);
      }
    }
    const int slot = block_rank(ok, s_warp, &s_run);
    if (ok) {
      float* o = out + (size_t)b * out_bstride + (size_t)slot * ldo;
      for (int c = 0; c < 4 * T; ++c) o[c] = box[c];
      o[4 * T] = sc;
    }
  }
  if (tid == 0) lv.counts[(size_t)b * counts_stride] = s_run;
}

// ------------------------------------------------------------------- collect across levels
// One CTA per image.  props [B, L, K, ldo], keep [B*L, K] (indices into the level's rows),
// nkeep [B*L].  Output rois [B, R, ldo+1] = (batch idx, box(es)) + scores [B, R]; count [B].
__global__ void __launch_bounds__(1024, 1)
collect_kernel(const float* __restrict__ props, const int* __restrict__ keep, const int* __restrict__ nkeep,
               int L, int K, int T, int post_topn, float* __restrict__ rois, float* __restrict__ roi_scores,
               int* __restrict__ roi_counts, int R, int cap /*pow2 >= L*K*/) {
  extern __shared__ unsigned long long skeys[];
  const int b = blockIdx.x, tid = threadIdx.x, nth = blockDim.x;
  const int ldo = 4 * T + 1;
  __shared__ int s_off[16];
  if (tid == 0) { int o = 0; for (int l = 0; l < L; ++l) { s_off[l] = o; o += min(nkeep[b * L + l], K); } s_off[L] = o; }
  __syncthreads();
  const int total = s_off[L];
  for (int x = tid; x < cap; x += nth) skeys[x] = 0ull;
  __syncthreads();
  for (int l = 0; l < L; ++l) {
    const int nk = s_off[l + 1] - s_off[l];
    for (int j = tid; j < nk; j += nth) {
      const int row = keep[(size_t)(b * L + l) * K + j];
      const float sc = props[(((size_t)b * L + l) * K + row) * ldo + 4 * T];
      const uint32_t cidx = (uint32_t)(s_off[l] + j);                 // position in the concatenation
      // payload: concat position (for the stable tie rule) in the low word; (level,row) recovered below
      skeys[s_off[l] + j] = ((unsigned long long)sort_key_f32(sc) << 32) | (unsigned long long)(0xffffffffu - cidx);
    }
  }
  __syncthreads();
  bitonic_desc(skeys, cap);
  const int nout = min(total, min(post_topn > 0 ? post_topn : total, R));
  for (int r = tid; r < nout; r += nth) {
    const uint32_t cidx = 0xffffffffu - (uint32_t)(skeys[r] & 0xffffffffull);
    int l = 0;
    while (l + 1 < L && (int)cidx >= s_off[l + 1]) ++l;
    const int j = (int)cidx - s_off[l];
    const int row = keep[(size_t)(b * L + l) * K + j];
    const float* src = props + (((size_t)b * L + l) * K + row) * ldo;
    float* dst = rois + ((size_t)b * R + r) * (ldo);
    dst[0] = (float)b;
    for (int c = 0; c < 4 * T; ++c) dst[1 + c] = src[c];
    roi_scores[(size_t)b * R + r] = src[4 * T];
  }
  if (tid == 0) roi_counts[b] = nout;
}

// ------------------------------------------------------------------- FPN level per RoI
// FPN.py:349-360 on rois [n, ld] (box columns start at col0).  One CTA; also emits the
// reference's restore permutation (argsort of the level-bucketed order).
__global__ void distribute_kernel(const float* __restrict__ rois, int n_max, const int* __restrict__ n_dev, int ld,
                                  int col0, int T, int kmin, int kmax, float s0, float lvl0,
                                  int* __restrict__ levels, int* __restrict__ idx_restore,
                                  int* __restrict__ level_counts) {
  __shared__ int s_warp[32];
  __shared__ int s_run;
  const int tid = threadIdx.x, nth = blockDim.x;
  const int n = n_dev ? min(*n_dev, n_max) : n_max;
  for (int i = tid; i < n; i += nth) {
    const float* r = rois + (size_t)i * ld + col0;
    float acc = 0.f;
    for (int t = 0; t < T; ++t) {      // boxes_area: mean over frames of (w+1)(h+1), sequential fp32
      const float w = __fadd_rn(__fsub_rn(r[4 * t + 2], r[4 * t]), 1.f), h = __fadd_rn(__fsub_rn(r[4 * t + 3], r[4 * t + 1]), 1.f);
      const float a = __fmul_rn(w, h);
      acc = (t == 0) ? a : __fadd_rn(acc, a);
    }
    const float area = __fdiv_rn(acc, (float)T);
    const float s = __fsqrt_rn(area);
    float lv = floorf(__fadd_rn(lvl0, log2f(__fadd_rn(__fdiv_rn(s, s0), 1e-6f))));
    lv = fminf(fmaxf(lv, (float)kmin), (float)kmax);
    levels[i] = (int)lv;
  }
  __syncthreads();
  if (idx_restore) {
    if (tid == 0) s_run = 0;
    __syncthreads();
    for (int lvl = kmin; lvl <= kmax; ++lvl) {
      const int before = s_run;
      for (int start = 0; start < n; start += nth) {
        const int i = start + tid;
        const bool f = (i < n) && levels[i] == lvl;
        const int slot = block_rank(f, s_warp, &s_run);
        if (f) idx_restore[i] = slot;     // position of roi i in the level-bucketed concatenation
      }
      if (tid == 0 && level_counts) level_counts[lvl - kmin] = s_run - before;
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------- box head post-processing
// test.py:211-252: boxes = rois / im_scale; bbox_transform(weights); clip to the ORIGINAL image;
// :760-766: per class j >= 1 keep score > thresh.  One CTA per (image, class-1).
// rois [B, R, 4T+1] (col 0 = batch idx); cls_prob from logits [B*R, ld_c] via softmax;
// deltas [B*R, ld_b] with class-major blocks j*4T (test.py:772).
__global__ void box_decode_kernel(const float* __restrict__ rois, const int* __restrict__ roi_counts, int R, int T,
                                  const float* __restrict__ cls_logits, int ld_c, const float* __restrict__ bbox_deltas,
                                  int ld_b, int num_classes, const float* __restrict__ im_info /*[B,3] blob h,w,scale*/,
                                  const float* __restrict__ im_hw /*[B,2] original image h,w*/, float wx, float wy,
                                  float ww, float wh, float clipv_f, double clipv_d, float score_thresh,
                                  float* __restrict__ dets /*[B, C-1, R, 4T+1]*/, int* __restrict__ det_counts) {
  __shared__ int s_warp[32];
  __shared__ int s_run;
  const int b = blockIdx.x, j = blockIdx.y + 1, tid = threadIdx.x, nth = blockDim.x;
  const int n = min(roi_counts[b], R);
  const int ldr = 4 * T + 1, ldo = 4 * T + 1;
  const float scale = im_info[3 * b + 2];
  const float hmax = __fsub_rn(im_hw[2 * b], 1.f), wmax = __fsub_rn(im_hw[2 * b + 1], 1.f);
  if (tid == 0) s_run = 0;
  __syncthreads();
  for (int start = 0; start < n; start += nth) {
    const int i = start + tid;
    bool ok = false;
    float box[DT_MAX_T * 4];
    float sc = 0.f;
    if (i < n) {
      const size_t row = (size_t)b * R + i;
      // softmax over classes (Caffe2 Softmax: subtract max, exp, normalise)
      float m = -CUDART_INF_F;
      for (int c = 0; c < num_classes; ++c) m = fmaxf(m, cls_logits[row * ld_c + c]);
      float sum = 0.f, ej = 0.f;
      for (int c = 0; c < num_classes; ++c) { const float e = expf(cls_logits[row * ld_c + c] - m); sum += e; if (c == j) ej = e; }
      sc = ej / sum;
      ok = sc > score_thresh;
      const float* r = rois + row * ldr + 1;
      const float* dl = bbox_deltas + row * ld_b + (size_t)j * 4 * T;
      for (int t = 0; t < T; ++t) {
        float* o = box + 4 * t;
        if (T == 1) {
          const float bx[4] = {__fdiv_rn(r[0], scale), __fdiv_rn(r[1], scale), __fdiv_rn(r[2], scale), __fdiv_rn(r[3], scale)};
          decode_f32(bx, dl, wx, wy, ww, wh, clipv_f, o);
        } else {
          const double bx[4] = {(double)__fdiv_rn(r[4 * t], scale), (double)__fdiv_rn(r[4 * t + 1], scale),
                                (double)__fdiv_rn(r[4 * t + 2], scale), (double)__fdiv_rn(r[4 * t + 3], scale)};
          decode_f64(bx, dl + 4 * t, (double)wx, (double)wy, (double)ww, (double)wh, clipv_d, o);
        }
        o[0] = fmaxf(fminf(o[0], wmax), 0.f); o[1] = fmaxf(fminf(o[1], hmax), 0.f);
        o[2] = fmaxf(fminf(o[2], wmax), 0.f); o[3] = fmaxf(fminf(o[3], hmax), 0.f);
      }
    }
    const int slot = block_rank(ok, s_warp, &s_run);
    if (ok) {
      float* o = dets + (((size_t)b * (num_classes - 1) + (j - 1)) * R + slot) * ldo;
      for (int c = 0; c < 4 * T; ++c) o[c] = box[c];
      o[4 * T] = sc;
    }
  }
  if (tid == 0) det_counts[b * (num_classes - 1) + (j - 1)] = s_run;
}

// test.py:768-800: nms_dets = dets_j[keep]; if more than max_per_im over all classes, keep
// score >= the max_per_im-th largest score.  One CTA per image.
__global__ void __launch_bounds__(1024, 1)
limit_kernel(const float* __restrict__ dets, const int* __restrict__ keep, const int* __restrict__ nkeep, int ncls1,
             int R, int T, int max_per_im, float* __restrict__ out /*[B, C-1, cap, 4T+1]*/,
             int* __restrict__ out_counts, int cap, int sortcap) {
  extern __shared__ unsigned long long skeys[];
  __shared__ int s_warp[32];
  __shared__ int s_run;
  __shared__ float s_thresh;
  const int b = blockIdx.x, tid = threadIdx.x, nth = blockDim.x;
  const int ld = 4 * T + 1;
  int total = 0;
  for (int c = 0; c < ncls1; ++c) total += min(nkeep[b * ncls1 + c], R);
  if (tid == 0) s_thresh = -CUDART_INF_F;
  __syncthreads();
  if (max_per_im > 0 && total > max_per_im) {
    for (int x = tid; x < sortcap; x += nth) skeys[x] = 0ull;
    __syncthreads();
    int off = 0;
    for (int c = 0; c < ncls1; ++c) {
      const int nk = min(nkeep[b * ncls1 + c], R);
      for (int q = tid; q < nk; q += nth) {
        const int row = keep[(size_t)(b * ncls1 + c) * R + q];
        const float sc = dets[(((size_t)b * ncls1 + c) * R + row) * ld + 4 * T];
        skeys[off + q] = ((unsigned long long)sort_key_f32(sc) << 32) | 1ull;
      }
      off += nk;
    }
    __syncthreads();
    bitonic_desc(skeys, sortcap);
    if (tid == 0) {
      uint32_t k = (uint32_t)(skeys[max_per_im - 1] >> 32);      // np.sort(scores)[-max_per_im]
      k = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
      s_thresh = __uint_as_float(k);
    }
    __syncthreads();
  }
  const float th = s_thresh;
  for (int c = 0; c < ncls1; ++c) {
    if (tid == 0) s_run = 0;
    __syncthreads();
    const int nk = min(nkeep[b * ncls1 + c], R);
    for (int start = 0; start < nk; start += nth) {
      const int q = start + tid;
      bool f = false; int row = 0;
      if (q < nk) {
        row = keep[(size_t)(b * ncls1 + c) * R + q];
        f = dets[(((size_t)b * ncls1 + c) * R + row) * ld + 4 * T] >= th;
      }
      const int slot = block_rank(f, s_warp, &s_run);
      if (f && slot < cap) {
        const float* src = dets + (((size_t)b * ncls1 + c) * R + row) * ld;
        float* dst = out + (((size_t)b * ncls1 + c) * cap + slot) * ld;
        for (int x = 0; x < ld; ++x) dst[x] = src[x];
      }
    }
    if (tid == 0) out_counts[b * ncls1 + c] = s_run;      // may exceed cap (score ties at the threshold): caller checks
    __syncthreads();
  }
}

static int next_pow2i(int x) { int p = 1; while (p < x) p <<= 1; return p; }

}  // namespace dt

using namespace dt;

extern "C" int dt_rpn_workspace_bytes(int B, int nlevels, const int* Hs, const int* Ws, int A, size_t* bytes) {
  DT_CHECK_ARG(B >= 0 && nlevels >= 1 && nlevels <= 8 && Hs && Ws && A >= 1 && bytes, "dt_rpn_workspace_bytes: bad args");
  size_t b = 0;
  for (int l = 0; l < nlevels; ++l) b += align_up((size_t)B * Hs[l] * Ws[l] * A * sizeof(uint32_t), 256);
  *bytes = b;
  return 0;
}

extern "C" int dt_rpn_proposals_multi(const dt_rpn_level* levels, int nlevels, int act_f32, int B, int A, int T,
                                      const float* im_info, int pre_nms_topn, float min_size, double bbox_xform_clip,
                                      long long out_batch_stride, int counts_stride, int time_major, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  DT_CHECK_ARG(levels && nlevels >= 1 && nlevels <= 8, "dt_rpn_proposals_multi: 1..8 levels");
  DT_CHECK_ARG(B >= 0 && A >= 1 && T >= 1 && T <= DT_MAX_T, "dt_rpn_proposals_multi: bad shape B=%d A=%d T=%d", B, A, T);
  if (B == 0) return 0;
  DT_CHECK_ARG(im_info && workspace, "dt_rpn_proposals_multi: null pointer");
  RpnLevels L;
  memset(&L, 0, sizeof(L));
  int kmax = 1;
  char* ws = (char*)workspace;
  size_t used = 0;
  for (int l = 0; l < nlevels; ++l) {
    const dt_rpn_level& v = levels[l];
    DT_CHECK_ARG(v.H >= 1 && v.W >= 1 && v.ld_s >= A && v.ld_d >= 4 * A * (time_major ? 1 : T),
                 "dt_rpn_proposals_multi: level %d bad shape / leading dims", l);
    DT_CHECK_ARG(v.logits && v.deltas && v.anchors && v.out && v.counts, "dt_rpn_proposals_multi: level %d null pointer", l);
    const long long n = (long long)v.H * v.W * A;
    DT_CHECK_ARG(n < (1ll << 31), "dt_rpn_proposals_multi: too many anchors");
    const int K = (pre_nms_topn <= 0 || pre_nms_topn > n) ? (int)n : pre_nms_topn;
    DT_CHECK_ARG(out_batch_stride >= (long long)K * (4 * T + 1) || B == 1, "dt_rpn_proposals_multi: out_batch_stride too small");
    if (K > kmax) kmax = K;
    RpnLevel& d = L.lv[l];
    d.logits = v.logits; d.deltas = v.deltas; d.anchors = v.anchors; d.ld_s = v.ld_s; d.ld_d = v.ld_d; d.H = v.H; d.W = v.W;
    d.feat_stride = v.feat_stride; d.out = v.out; d.counts = v.counts;
    d.keys = (uint32_t*)(ws + used);
    used += align_up((size_t)B * n * sizeof(uint32_t), 256);
  }
  DT_CHECK_ARG(used <= workspace_bytes, "dt_rpn_proposals_multi: workspace %zu < %zu bytes", workspace_bytes, used);
  const int kcap = next_pow2i(kmax);
  DT_CHECK_ARG(kcap <= 16384, "dt_rpn_proposals_multi: pre-NMS top-N %d exceeds 16384", kmax);
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(rpn_proposals_kernel, 16384 * 8, &grant));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(B * RPN_CS), (unsigned)nlevels, 1);
  cfg.blockDim = dim3(1024, 1, 1);
  cfg.dynamicSmemBytes = (size_t)kcap * sizeof(unsigned long long);
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = RPN_CS; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  DT_CHECK_CUDA(cudaLaunchKernelEx(&cfg, rpn_proposals_kernel, L, act_f32, A, T, im_info, pre_nms_topn, min_size,
                                   (float)bbox_xform_clip, bbox_xform_clip, out_batch_stride, counts_stride, kcap,
                                   time_major));
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_collect_rpn(const float* props, const int* keep, const int* nkeep, int B, int L, int K, int T,
                              int post_nms_topn, float* rois, float* roi_scores, int* roi_counts, int R, void* stream) {
  DT_CHECK_ARG(B >= 0 && L >= 1 && L <= 15 && K >= 1 && T >= 1 && T <= DT_MAX_T && R >= 1, "dt_collect_rpn: bad shape");
  if (B == 0) return 0;
  DT_CHECK_ARG(props && keep && nkeep && rois && roi_scores && roi_counts, "dt_collect_rpn: null pointer");
  const int cap = next_pow2i(L * K);
  DT_CHECK_ARG(cap <= 16384, "dt_collect_rpn: L*K=%d exceeds 16384", L * K);
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(collect_kernel, 16384 * 8, &grant));
  collect_kernel<<<B, 1024, (size_t)cap * 8, (cudaStream_t)stream>>>(props, keep, nkeep, L, K, T, post_nms_topn, rois,
                                                                     roi_scores, roi_counts, R, cap);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_distribute_fpn(const float* rois, int n_max, const int* n_dev, int ld, int col0, int T, int k_min,
                                 int k_max, float canonical_scale, float canonical_level, int* levels,
                                 int* idx_restore, int* level_counts, void* stream) {
  DT_CHECK_ARG(n_max >= 0 && T >= 1 && T <= DT_MAX_T && ld >= col0 + 4 * T && k_max >= k_min, "dt_distribute_fpn: bad shape");
  if (n_max == 0) return 0;
  DT_CHECK_ARG(rois && levels, "dt_distribute_fpn: null pointer");
  distribute_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(rois, n_max, n_dev, ld, col0, T, k_min, k_max, canonical_scale,
                                                          canonical_level, levels, idx_restore, level_counts);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_box_decode(const float* rois, const int* roi_counts, int B, int R, int T, const float* cls_logits,
                             int ld_c, const float* bbox_deltas, int ld_b, int num_classes, const float* im_info,
                             const float* im_hw, const float* weights4 /*host*/, double bbox_xform_clip,
                             float score_thresh, float* dets, int* det_counts, void* stream) {
  DT_CHECK_ARG(B >= 0 && R >= 1 && T >= 1 && T <= DT_MAX_T && num_classes >= 2, "dt_box_decode: bad shape");
  DT_CHECK_ARG(ld_c >= num_classes && ld_b >= 4 * T * num_classes, "dt_box_decode: leading dims too small");
  if (B == 0) return 0;
  DT_CHECK_ARG(rois && roi_counts && cls_logits && bbox_deltas && im_info && im_hw && weights4 && dets && det_counts,
               "dt_box_decode: null pointer");
  dim3 grid(B, num_classes - 1);
  box_decode_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(rois, roi_counts, R, T, cls_logits, ld_c, bbox_deltas, ld_b,
                                                            num_classes, im_info, im_hw, weights4[0], weights4[1],
                                                            weights4[2], weights4[3], (float)bbox_xform_clip,
                                                            bbox_xform_clip, score_thresh, dets, det_counts);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_limit_detections(const float* dets, const int* keep, const int* nkeep, int B, int num_classes, int R,
                                   int T, int max_per_im, float* out, int* out_counts, int cap, void* stream) {
  DT_CHECK_ARG(B >= 0 && num_classes >= 2 && R >= 1 && T >= 1 && T <= DT_MAX_T && cap >= 1, "dt_limit_detections: bad shape");
  if (B == 0) return 0;
  DT_CHECK_ARG(dets && keep && nkeep && out && out_counts, "dt_limit_detections: null pointer");
  const int sortcap = next_pow2i((num_classes - 1) * R);
  DT_CHECK_ARG(sortcap <= 16384, "dt_limit_detections: (C-1)*R=%d exceeds 16384", (num_classes - 1) * R);
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(limit_kernel, 16384 * 8, &grant));
  limit_kernel<<<B, 1024, (size_t)sortcap * 8, (cudaStream_t)stream>>>(dets, keep, nkeep, num_classes - 1, R, T, max_per_im,
                                                                       out, out_counts, cap, sortcap);
  DT_CHECK_LAUNCH();
  return 0;
}


// lib/core/test.py:76-113 _get_rois_blob / _project_im_rois for the keypoint head: rois[i] = (image index,
// boxes[i] * im_scale), the product taken in fp64 and stored as fp32 exactly as numpy does.  boxes [n, ldb] (first ncols
// columns), image index = bidx[i] if given, else i / per_image.
namespace dt {
__global__ void scale_rois_kernel(const float* __restrict__ boxes, int ldb, int n, int ncols, const float* __restrict__ bidx,
                                  int per_image, double im_scale, float* __restrict__ rois) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * (ncols + 1)) return;
  const int r = i / (ncols + 1), c = i - r * (ncols + 1);
  rois[i] = c == 0 ? (bidx ? bidx[r] : (float)(r / per_image)) : (float)((double)boxes[(size_t)r * ldb + c - 1] * im_scale);
}
}  // namespace dt

extern "C" int dt_scale_rois(const float* boxes, int ldb, int n, int ncols, const float* bidx, int per_image, double im_scale,
                             float* rois, void* stream) {
  DT_CHECK_ARG(n >= 0 && ncols >= 1 && ldb >= ncols && (bidx || per_image >= 1), "dt_scale_rois: bad shape n=%d ncols=%d ldb=%d", n, ncols, ldb);
  if (n == 0) return 0;
  DT_CHECK_ARG(boxes && rois, "dt_scale_rois: null pointer");
  const int total = n * (ncols + 1);
  dt::scale_rois_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(boxes, ldb, n, ncols, bidx, per_image, im_scale, rois);
  DT_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------- test-time augmentation (lib/core/test.py:255-414)
// flip_boxes (lib/utils/boxes.py:275-282) on one 4-column box: x1' = W - x2 - 1, x2' = W - x1 - 1 in numpy's fp32
// arithmetic (two roundings; this unit is compiled without FMA contraction).
namespace dt {
__device__ __forceinline__ float flip_x(float w, float x) { return __fsub_rn(__fsub_rn(w, x), 1.f); }

struct AugMergeTable {
  const float* dets[DT_AUG_MAX_VIEWS];
  const int* counts[DT_AUG_MAX_VIEWS];
  int flip[DT_AUG_MAX_VIEWS];
};

// One CTA per (image, class - 1): the union of the V views' compacted rows in view order (np.vstack of the views), each
// flipped view's rows mapped back to the original image.  out [B, C-1, V*R, 5].
__global__ void aug_merge_dets_kernel(const __grid_constant__ AugMergeTable tab, int V, int ncls1, int R,
                                      const float* __restrict__ im_w, int ld_w, float* __restrict__ out,
                                      int* __restrict__ out_counts) {
  const int b = blockIdx.x, c = blockIdx.y, bc = b * ncls1 + c;
  const float w = im_w[(size_t)b * ld_w];
  float* dst = out + (size_t)bc * V * R * 5;
  int off = 0;
  for (int v = 0; v < V; ++v) {
    const int n = max(0, min(tab.counts[v][bc], R));
    const float* src = tab.dets[v] + (size_t)bc * R * 5;
    const int fl = tab.flip[v];
    for (int q = threadIdx.x; q < n * 5; q += blockDim.x) {
      const int r = q / 5, col = q - r * 5;
      float x = src[q];
      if (fl && col == 0) x = flip_x(w, src[r * 5 + 2]);
      else if (fl && col == 2) x = flip_x(w, src[r * 5]);
      dst[(size_t)off * 5 + q] = x;
    }
    off += n;
  }
  if (threadIdx.x == 0) out_counts[bc] = off;
}

// _get_rois_blob of one keypoint view: (image index, flip_boxes(boxes) * im_scale) — the flip in fp32 as above, the
// product in fp64 stored fp32.  Without the flip this is scale_rois_kernel with ncols = 4.
__global__ void aug_scale_rois_kernel(const float* __restrict__ boxes, int ldb, int n, int flip, const float* __restrict__ im_w,
                                      int ld_w, int per_image, double im_scale, float* __restrict__ rois) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 5) return;
  const int r = i / 5, c = i - r * 5;
  if (c == 0) { rois[i] = (float)(r / per_image); return; }
  const float* bx = boxes + (size_t)r * ldb;
  float x = bx[c - 1];
  if (flip && (c == 1 || c == 3)) x = flip_x(im_w[(size_t)(r / per_image) * ld_w], bx[c == 1 ? 2 : 0]);
  rois[i] = (float)((double)x * im_scale);
}
}  // namespace dt

extern "C" int dt_aug_merge_dets(const float* const* dets, const int* const* counts, const int* flip, int V, int B,
                                 int num_classes, int R, const float* im_w, int ld_w, float* out, int* out_counts,
                                 void* stream) {
  DT_CHECK_ARG(V >= 1 && V <= DT_AUG_MAX_VIEWS, "dt_aug_merge_dets: V=%d views (1..%d)", V, DT_AUG_MAX_VIEWS);
  DT_CHECK_ARG(B >= 0 && num_classes >= 2 && R >= 1 && ld_w >= 1, "dt_aug_merge_dets: bad shape B=%d C=%d R=%d ld_w=%d", B,
               num_classes, R, ld_w);
  DT_CHECK_ARG((long long)V * R <= DT_NMS_MAX_BOXES, "dt_aug_merge_dets: V*R=%lld exceeds %d", (long long)V * R, DT_NMS_MAX_BOXES);
  DT_CHECK_ARG(dets && counts && flip, "dt_aug_merge_dets: null view table");
  if (B == 0) return 0;
  dt::AugMergeTable tab;
  memset(&tab, 0, sizeof(tab));
  for (int v = 0; v < V; ++v) {
    DT_CHECK_ARG(dets[v] && counts[v], "dt_aug_merge_dets: view %d null pointer", v);
    tab.dets[v] = dets[v]; tab.counts[v] = counts[v]; tab.flip[v] = flip[v] != 0;
  }
  DT_CHECK_ARG(im_w && out && out_counts, "dt_aug_merge_dets: null pointer");
  dim3 grid(B, num_classes - 1);
  dt::aug_merge_dets_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(tab, V, num_classes - 1, R, im_w, ld_w, out, out_counts);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_aug_scale_rois(const float* boxes, int ldb, int n, int flip, const float* im_w, int ld_w, int per_image,
                                 double im_scale, float* rois, void* stream) {
  DT_CHECK_ARG(n >= 0 && ldb >= 4 && per_image >= 1 && ld_w >= 1, "dt_aug_scale_rois: bad shape n=%d ldb=%d per_image=%d",
               n, ldb, per_image);
  if (n == 0) return 0;
  DT_CHECK_ARG(boxes && rois && (im_w || !flip), "dt_aug_scale_rois: null pointer");
  dt::aug_scale_rois_kernel<<<(n * 5 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(boxes, ldb, n, flip != 0, im_w, ld_w,
                                                                                   per_image, im_scale, rois);
  DT_CHECK_LAUNCH();
  return 0;
}
