// Training target generators on the device (SURVEY.md §8 f1; the reference runs these in numpy on loader threads and inside
// the CollectAndDistributeFpnRpnProposals python op, lib/roi_data/*.py):
//
//   dt_rpn_targets    lib/roi_data/rpn.py:206-381 (_get_rpn_blobs, T = 1): anchors inside the image, IoU with the gt boxes
//                     (cython_bbox arithmetic, bit-exact), labels (per-gt best anchors incl. ties, IoU >= 0.7), foreground
//                     sub-sampling, background sampling WITH replacement, bbox_transform_inv targets, inside / outside
//                     weights — written per FPN level in the NHWC order the loss kernel reads.
//   dt_sample_rois    lib/datasets/json_dataset.py:423-534 (add_proposals) + lib/roi_data/fast_rcnn.py:118-238 (_sample_rois)
//                     + lib/roi_data/keypoint_rcnn.py:24-99 + lib/utils/keypoints.py:152-207: proposals of the batch-wide
//                     top-N (collect, training branch) merged with the gt boxes, fg / bg RoI sampling, class-expanded box
//                     targets, keypoint RoIs and their heat-map location labels.
//
// Random draws.  The reference uses numpy's global Mersenne twister; here every draw is a pure function of
// (seed, stream, image, index) — hash_u32 below, restated in oracle/targets.py — with
//     choice(a, k)  = the k elements with the smallest (hash(a_i), a_i), in that order,
//     randint(n, k) = (hash(j) * n) >> 32 for j < k,
// so the whole generator is deterministic and is compared bit for bit with the reference's own code run with exactly these
// two draws (tests/golden/gen_golden_targets.py).  Compiled with -fmad=false.
// Streams: 0 RPN fg disable, 1 RPN bg enable, 2 RoI fg, 3 RoI bg, 4 keypoint RoIs (these kernels); 5 the per-clip
// TRAIN.SCALES draw of TRAIN.AUGMENT, made on the host (ops/target_ops.train_scale, image 0, index = clip counter).
#include "common.cuh"
#include "box_math.cuh"
#include "../../include/dt_b200.h"

namespace dt {

__host__ __device__ __forceinline__ unsigned long long hash_base(unsigned long long seed, unsigned long long stream, unsigned long long image) {
  return seed * 0x9E3779B97F4A7C15ull + stream * 0xBF58476D1CE4E5B9ull + image * 0x94D049BB133111EBull;
}
__device__ __forceinline__ uint32_t hash_u32(unsigned long long base, unsigned long long i) {
  unsigned long long x = base + i;
  x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27; x *= 0x94D049BB133111EBull;
  x ^= x >> 31;
  return (uint32_t)(x >> 32);
}

// utils/boxes.py:205-230 in fp32, evaluation order as numpy's ((w * d) / e; w * log(g / e))
__device__ __forceinline__ void transform_inv(const float* ex, const float* gt, float wx, float wy, float ww, float wh, float* out) {
  const float ew = __fadd_rn(__fsub_rn(ex[2], ex[0]), 1.0f), eh = __fadd_rn(__fsub_rn(ex[3], ex[1]), 1.0f);
  const float ecx = __fadd_rn(ex[0], __fmul_rn(0.5f, ew)), ecy = __fadd_rn(ex[1], __fmul_rn(0.5f, eh));
  const float gw = __fadd_rn(__fsub_rn(gt[2], gt[0]), 1.0f), gh = __fadd_rn(__fsub_rn(gt[3], gt[1]), 1.0f);
  const float gcx = __fadd_rn(gt[0], __fmul_rn(0.5f, gw)), gcy = __fadd_rn(gt[1], __fmul_rn(0.5f, gh));
  out[0] = __fdiv_rn(__fmul_rn(wx, __fsub_rn(gcx, ecx)), ew);
  out[1] = __fdiv_rn(__fmul_rn(wy, __fsub_rn(gcy, ecy)), eh);
  out[2] = __fmul_rn(ww, logf(__fdiv_rn(gw, ew)));
  out[3] = __fmul_rn(wh, logf(__fdiv_rn(gh, eh)));
}

// Tubes (T > 1): the reference's split_tube_into_boxes promotes every frame to fp64 (np.hstack with an empty fp64 score column,
// utils/boxes.py:28-58), so its tube targets are fp64 arithmetic on the fp32 coordinates, rounded to fp32 once.
__device__ __forceinline__ void transform_inv64(const float* ex, const float* gt, double wx, double wy, double ww, double wh, float* out) {
  const double ew = __dadd_rn(__dsub_rn((double)ex[2], (double)ex[0]), 1.0), eh = __dadd_rn(__dsub_rn((double)ex[3], (double)ex[1]), 1.0);
  const double ecx = __dadd_rn((double)ex[0], __dmul_rn(0.5, ew)), ecy = __dadd_rn((double)ex[1], __dmul_rn(0.5, eh));
  const double gw = __dadd_rn(__dsub_rn((double)gt[2], (double)gt[0]), 1.0), gh = __dadd_rn(__dsub_rn((double)gt[3], (double)gt[1]), 1.0);
  const double gcx = __dadd_rn((double)gt[0], __dmul_rn(0.5, gw)), gcy = __dadd_rn((double)gt[1], __dmul_rn(0.5, gh));
  out[0] = (float)__ddiv_rn(__dmul_rn(wx, __dsub_rn(gcx, ecx)), ew);
  out[1] = (float)__ddiv_rn(__dmul_rn(wy, __dsub_rn(gcy, ecy)), eh);
  out[2] = (float)__dmul_rn(ww, log(__ddiv_rn(gw, ew)));
  out[3] = (float)__dmul_rn(wh, log(__ddiv_rn(gh, eh)));
}

// ------------------------------------------------------------------------------------------------ RPN targets
constexpr int TG_TMAX = 4;            // frames per tube supported by the target generators

struct RpnTL {
  int n_levels, A, T;
  int H[8], W[8], start[9];
  double stride[8];
  const double* cell[8];              // [A, 4T] fp64 (generate_anchors.py; tube anchors replicate the 2-D anchor over the frames)
  int* labels[8];                     // [B, H, W, A]
  float* bt[8]; float* iw[8]; float* ow[8];   // [B, H, W, 4T*A]
  int* vis[8];                        // [B, H, W, T*A] or NULL
};

struct AnchorRef { int l, loc; };     // level, index inside the level (h, w, a)

__device__ __forceinline__ AnchorRef anchor_box(const RpnTL& lv, int i, float* box) {
  int l = 0;
  while (l + 1 < lv.n_levels && i >= lv.start[l + 1]) ++l;
  const int loc = i - lv.start[l];
  const int a = loc % lv.A, pos = loc / lv.A;
  const int w = pos % lv.W[l], h = pos / lv.W[l];
  const double sx = (double)w * lv.stride[l], sy = (double)h * lv.stride[l];
  const double* c = lv.cell[l] + 4 * lv.T * a;          // first frame of the (replicated) tube anchor
  box[0] = (float)(c[0] + sx); box[1] = (float)(c[1] + sy); box[2] = (float)(c[2] + sx); box[3] = (float)(c[3] + sy);
  AnchorRef r; r.l = l; r.loc = loc;
  return r;
}

constexpr int TG_GMAX = 128;

// IoU of a (replicated) tube anchor with a gt tube: utils/boxes.py:60-69, sequential fp32 sum over the frames, / T
__device__ __forceinline__ float anchor_tube_iou(const float* box, const float* gt_tube, int T) {
  float acc = iou_pair_ref(box, gt_tube);
  for (int t = 1; t < T; ++t) acc = __fadd_rn(acc, iou_pair_ref(box, gt_tube + 4 * t));
  return T == 1 ? acc : __fdiv_rn(acc, (float)T);
}

// pass 1: per anchor max / first-argmax IoU over the gt boxes; per gt the max over the inside anchors
__global__ void __launch_bounds__(256)
rpn_anchor_iou_kernel(RpnTL lv, int NA, const float* __restrict__ gt, const int* __restrict__ gt_counts, int Gmax,
                      const float* __restrict__ im_info, float straddle, float* __restrict__ amax, int* __restrict__ aarg,
                      unsigned* __restrict__ gmax) {
  __shared__ float sgt[TG_GMAX * 4 * TG_TMAX];
  __shared__ unsigned sgm[TG_GMAX];
  const int b = blockIdx.y;
  const int G = min(gt_counts[b], Gmax);
  const float scale = im_info[b * 3 + 2];
  const int D = 4 * lv.T;
  for (int j = threadIdx.x; j < G * D; j += blockDim.x) sgt[j] = __fmul_rn(gt[(size_t)b * Gmax * D + j], scale);
  for (int j = threadIdx.x; j < G; j += blockDim.x) sgm[j] = 0u;
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < NA) {
    float box[4];
    anchor_box(lv, i, box);
    const double imh = (double)im_info[b * 3 + 0], imw = (double)im_info[b * 3 + 1], st = (double)straddle;
    const bool inside = (double)box[0] >= -st && (double)box[1] >= -st && (double)box[2] < imw + st && (double)box[3] < imh + st;
    float best = -2.f; int arg = -1;                  // -2: not inside the image
    if (inside && G > 0) {
      for (int g = 0; g < G; ++g) {
        const float v = anchor_tube_iou(box, sgt + D * g, lv.T);
        if (g == 0 || v > best) { best = v; arg = g; }
        if (v > 0.f) atomicMax(&sgm[g], __float_as_uint(v));
      }
    }
    amax[(size_t)b * NA + i] = best;
    aarg[(size_t)b * NA + i] = arg;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < G; j += blockDim.x) if (sgm[j]) atomicMax(&gmax[b * Gmax + j], sgm[j]);
}

// pass 2: labels before sampling (1 / -1) and the two candidate counts
__global__ void __launch_bounds__(256)
rpn_label_kernel(RpnTL lv, int NA, const float* __restrict__ gt, const int* __restrict__ gt_counts, int Gmax,
                 const float* __restrict__ im_info, float pos_thresh, float neg_thresh, const float* __restrict__ amax,
                 const unsigned* __restrict__ gmax, signed char* __restrict__ lab, int* __restrict__ cnt /*[B,4]*/) {
  __shared__ float sgt[TG_GMAX * 4 * TG_TMAX];
  __shared__ float sgm[TG_GMAX];
  __shared__ int s_cnt[2];
  const int b = blockIdx.y;
  const int G = min(gt_counts[b], Gmax);
  const float scale = im_info[b * 3 + 2];
  const int D = 4 * lv.T;
  for (int j = threadIdx.x; j < G * D; j += blockDim.x) sgt[j] = __fmul_rn(gt[(size_t)b * Gmax * D + j], scale);
  for (int j = threadIdx.x; j < G; j += blockDim.x) sgm[j] = __uint_as_float(gmax[b * Gmax + j]);
  if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < NA) {
    const float m = amax[(size_t)b * NA + i];
    signed char l = -1;
    if (m > -1.5f) {                                  // inside the image
      float box[4];
      anchor_box(lv, i, box);
      bool fg = m >= pos_thresh;
      for (int g = 0; g < G && !fg; ++g) fg = anchor_tube_iou(box, sgt + D * g, lv.T) == sgm[g];   // rpn.py:254-259, incl. the 0 == 0 ties
      if (fg) { l = 1; atomicAdd(&s_cnt[0], 1); }
      if (m < neg_thresh) atomicAdd(&s_cnt[1], 1);
    }
    lab[(size_t)b * NA + i] = l;
  }
  __syncthreads();
  if (threadIdx.x < 2 && s_cnt[threadIdx.x]) atomicAdd(&cnt[b * 4 + threadIdx.x], s_cnt[threadIdx.x]);
}

__device__ __forceinline__ int block_scan_excl(int v, int* warp_sums, int* total) {
  // exclusive prefix sum over a 1024-thread block
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int s = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
    warp_sums[lane] = s;
  }
  __syncthreads();
  const int base = wid ? warp_sums[wid - 1] : 0;
  if (total) *total = warp_sums[31];
  __syncthreads();
  return base + x - v;
}

// pass 3: the two random draws, one CTA per image (rpn.py:266-283)
__global__ void __launch_bounds__(1024)
rpn_sample_kernel(int NA, int batch, int num_fg, float neg_thresh, unsigned long long seed, const float* __restrict__ amax,
                  signed char* __restrict__ lab, int* __restrict__ cnt) {
  __shared__ int hist[256];
  __shared__ int warp_sums[32];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_remaining, s_total;
  __shared__ unsigned s_draw[1024];
  extern __shared__ int gcnt[];                       // candidate counts / prefix per 32-anchor group
  const int b = blockIdx.x;
  const float* am = amax + (size_t)b * NA;
  signed char* lb = lab + (size_t)b * NA;
  const int nfg = cnt[b * 4 + 0], nbc = cnt[b * 4 + 1];
  const unsigned long long base0 = hash_base(seed, 0, (unsigned long long)b), base1 = hash_base(seed, 1, (unsigned long long)b);
  int kept_fg = nfg;
  if (nfg > num_fg) {
    // disable the (nfg - num_fg) foreground anchors with the smallest (hash, index): radix select of that rank over the
    // unique 64-bit composites, then everything <= the threshold goes
    if (threadIdx.x == 0) { s_prefix = 0ull; s_remaining = nfg - num_fg; }
    __syncthreads();
    for (int byte = 7; byte >= 0; --byte) {
      for (int j = threadIdx.x; j < 256; j += blockDim.x) hist[j] = 0;
      __syncthreads();
      const unsigned long long prefix = s_prefix;
      const int sh = byte * 8;
      for (int i = threadIdx.x; i < NA; i += blockDim.x) {
        if (lb[i] != 1) continue;
        const unsigned long long v = ((unsigned long long)hash_u32(base0, (unsigned long long)i) << 32) | (unsigned)i;
        if (byte == 7 || (v >> (sh + 8)) == (prefix >> (sh + 8))) atomicAdd(&hist[(int)((v >> sh) & 255ull)], 1);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int rem = s_remaining, d = 0;
        while (d < 255 && hist[d] < rem) { rem -= hist[d]; ++d; }
        s_remaining = rem;
        s_prefix = prefix | ((unsigned long long)d << sh);
      }
      __syncthreads();
    }
    const unsigned long long thr = s_prefix;
    for (int i = threadIdx.x; i < NA; i += blockDim.x) {
      if (lb[i] != 1) continue;
      const unsigned long long v = ((unsigned long long)hash_u32(base0, (unsigned long long)i) << 32) | (unsigned)i;
      if (v <= thr) lb[i] = -1;
    }
    kept_fg = num_fg;
    __syncthreads();
  }
  const int num_bg = batch - kept_fg;
  if (nbc > num_bg && num_bg > 0) {
    // num_bg draws WITH replacement from the candidates in index order: draw j picks candidate number (hash(j) * nbc) >> 32.
    // Candidate counts per 32-anchor group (coalesced ballots) -> exclusive prefix in shared memory -> each draw finds its
    // group by binary search and its anchor inside the group.
    const int nd = min(num_bg, 1024);
    for (int j = threadIdx.x; j < nd; j += blockDim.x) s_draw[j] = (unsigned)(((unsigned long long)hash_u32(base1, (unsigned long long)j) * (unsigned long long)nbc) >> 32);
    const int ng = (NA + 31) / 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int gidx = warp; gidx < ng; gidx += 32) {
      const int i = gidx * 32 + lane;
      const float m = i < NA ? am[i] : -2.f;
      const unsigned bal = __ballot_sync(0xffffffffu, m > -1.5f && m < neg_thresh);
      if (lane == 0) gcnt[gidx] = __popc(bal);
    }
    __syncthreads();
    const int per = (ng + blockDim.x - 1) / blockDim.x;
    const int g0 = min(ng, (int)threadIdx.x * per), g1 = min(ng, g0 + per);
    int c = 0;
    for (int q = g0; q < g1; ++q) c += gcnt[q];
    int run = block_scan_excl(c, warp_sums, &s_total);
    for (int q = g0; q < g1; ++q) { const int t = gcnt[q]; gcnt[q] = run; run += t; }      // exclusive prefix per group
    __syncthreads();
    for (int j = threadIdx.x; j < nd; j += blockDim.x) {
      const int r = (int)s_draw[j];
      int lo = 0, hi = ng - 1;                         // last group whose prefix <= r
      while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (gcnt[mid] <= r) lo = mid; else hi = mid - 1; }
      int want = r - gcnt[lo];
      for (int i = lo * 32; i < min(NA, lo * 32 + 32); ++i) {
        const float m = am[i];
        if (m > -1.5f && m < neg_thresh) {
          if (want == 0) { const signed char v = lb[i]; lb[i] = (v == 1 || v == 2) ? 2 : 0; break; }   // 2: label 0, still a "fg_ind" for the box targets
          --want;
        }
      }
    }
    __syncthreads();
  }
  int ne = 0;
  for (int i = threadIdx.x; i < NA; i += blockDim.x) ne += lb[i] >= 0 ? 1 : 0;
  for (int o = 16; o > 0; o >>= 1) ne += __shfl_xor_sync(0xffffffffu, ne, o);
  if ((threadIdx.x & 31) == 0 && ne) atomicAdd(&cnt[b * 4 + 2], ne);
}

// pass 4: the per-level target blobs
__global__ void __launch_bounds__(256)
rpn_write_kernel(RpnTL lv, int NA, const float* __restrict__ gt, const unsigned char* __restrict__ gt_vis, const int* __restrict__ gt_counts,
                 int Gmax, const float* __restrict__ im_info, const int* __restrict__ aarg, const signed char* __restrict__ lab,
                 const int* __restrict__ cnt) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NA) return;
  float box[4];
  const AnchorRef r = anchor_box(lv, i, box);
  const int T = lv.T;
  const size_t per = (size_t)lv.H[r.l] * lv.W[r.l] * lv.A;
  const size_t o = (size_t)b * per + r.loc;
  const int l = lab[(size_t)b * NA + i];
  const int final_label = l < 0 ? -1 : (l == 1 ? 1 : 0);
  lv.labels[r.l][o] = final_label;
  const bool fg = l == 1 || l == 2;
  const float w_out = l >= 0 ? (float)(1.0 / (double)cnt[b * 4 + 2]) : 0.f;
  const int ga = fg ? aarg[(size_t)b * NA + i] : 0;
  const float scale = im_info[b * 3 + 2];
  for (int t = 0; t < T; ++t) {
    float tg[4] = {0.f, 0.f, 0.f, 0.f};
    bool visible = true;
    if (fg) {
      const float* g = gt + ((size_t)b * Gmax + ga) * 4 * T + 4 * t;
      float gs[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) gs[k] = __fmul_rn(g[k], scale);
      if (T == 1) transform_inv(box, gs, 1.f, 1.f, 1.f, 1.f, tg);
      else transform_inv64(box, gs, 1.0, 1.0, 1.0, 1.0, tg);
      visible = gt_vis ? gt_vis[((size_t)b * Gmax + ga) * T + t] != 0 : true;      // track_visible (rpn.py:300-303)
    }
    const float w_in = (fg && visible) ? 1.f : 0.f;
    reinterpret_cast<float4*>(lv.bt[r.l])[o * T + t] = make_float4(tg[0], tg[1], tg[2], tg[3]);
    reinterpret_cast<float4*>(lv.iw[r.l])[o * T + t] = make_float4(w_in, w_in, w_in, w_in);
    reinterpret_cast<float4*>(lv.ow[r.l])[o * T + t] = make_float4(w_out, w_out, w_out, w_out);
    if (lv.vis[r.l]) lv.vis[r.l][o * T + t] = (l == 1 && !visible) ? 0 : final_label;   // rpn.py:318-321: vis_labels[fg_inds] *= visible
  }
}

// ------------------------------------------------------------------------------------------------ RoI sampling
struct SampleParams {
  int B, R, topn, Gmax, K, T, num_classes, batch, fg_per, kcap, M;      // K joints per frame, T frames per tube
  float fg_thresh, bg_hi, bg_lo, wx, wy, ww, wh;
  unsigned long long seed;
};

// rank of candidate (key, idx) among a candidate list in shared memory
__device__ __forceinline__ int rank_in(const unsigned* keys, const int* list, int n, unsigned key, int idx) {
  int r = 0;
  for (int j = 0; j < n; ++j) {
    const int oj = list[j];
    const unsigned kj = keys[j];
    r += (kj < key || (kj == key && oj < idx)) ? 1 : 0;
  }
  return r;
}

__global__ void __launch_bounds__(1024)
sample_rois_kernel(SampleParams p, const float* __restrict__ rois, const float* __restrict__ scores, const int* __restrict__ roi_counts,
                   const float* __restrict__ gt_boxes, const int* __restrict__ gt_classes, const int* __restrict__ gt_crowd,
                   const int* __restrict__ gt_kps, const int* __restrict__ gt_counts, const float* __restrict__ im_info,
                   float* __restrict__ rois_out, int* __restrict__ labels, float* __restrict__ bt, float* __restrict__ iw,
                   float* __restrict__ ow, int* __restrict__ out_counts, float* __restrict__ kp_rois, int* __restrict__ kp_loc,
                   float* __restrict__ kp_w, int* __restrict__ kp_counts, float* __restrict__ totals) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x;
  const int G = min(gt_counts[b], p.Gmax);
  const int nmax = p.Gmax + p.R;
  const int T = p.T, D = 4 * p.T;
  float* box = reinterpret_cast<float*>(smem_raw);                 // [nmax][4T]
  float* mov = box + (size_t)nmax * D;                             // [nmax] max_overlaps
  int* bmap = reinterpret_cast<int*>(mov + nmax);                  // [nmax] box_to_gt_ind_map
  int* cls = bmap + nmax;                                          // [nmax] max_classes
  int* list = cls + nmax;                                          // [nmax] candidate list
  unsigned* keys = reinterpret_cast<unsigned*>(list + nmax);       // [nmax] keys of the list entries
  int* rowof = reinterpret_cast<int*>(keys + nmax);                // [batch + kcap] box index per output row
  __shared__ int s_n, s_c0, s_c1;
  __shared__ int warp_sums[32];
  __shared__ float s_wsum;
  const float scale = im_info[b * 3 + 2];
  const float inv = __fdiv_rn(1.0f, scale);
  const float* gb = gt_boxes + (size_t)b * p.Gmax * D;
  // ---- proposals of this image inside the batch-wide top-N (collect, training branch): a prefix of its score-sorted list
  const int Pn = min(roi_counts[b], p.R);
  if (threadIdx.x == 0) { s_n = 0; s_wsum = 0.f; }
  __syncthreads();
  {
    int mine = 0;
    for (int r = threadIdx.x; r < Pn; r += blockDim.x) {
      const float s = scores[(size_t)b * p.R + r];
      int rank = r;
      for (int o = 0; o < p.B; ++o) {
        if (o == b) continue;
        const int no = min(roi_counts[o], p.R);
        const float* so = scores + (size_t)o * p.R;
        int lo = 0, hi = no;                       // count of scores ranked before s (ties: the lower image index first)
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          const float v = so[mid];
          if (v > s || (v == s && o < b)) lo = mid + 1; else hi = mid;
        }
        rank += lo;
      }
      mine += (p.topn <= 0 || rank < p.topn) ? 1 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_n, mine);
  }
  __syncthreads();
  const int P = s_n;
  const int n = G + P;
  // ---- add_proposals: boxes = [gt ; proposals / scale], overlaps with the gt boxes (json_dataset.py:423-512)
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float bx[4 * TG_TMAX];
    float mx; int am, c;
    if (i < G) {
      for (int k = 0; k < D; ++k) bx[k] = gb[i * D + k];
      const bool crowd = gt_crowd[b * p.Gmax + i] != 0;
      mx = crowd ? -1.f : 1.f; am = i; c = crowd ? 0 : gt_classes[b * p.Gmax + i];
    } else {
      const float* r = rois + ((size_t)b * p.R + (i - G)) * (D + 1);
      for (int k = 0; k < D; ++k) bx[k] = __fmul_rn(r[1 + k], inv);
      mx = 0.f; am = -1; c = 0;
      float best = 0.f; int arg = 0;
      for (int g = 0; g < G; ++g) {
        float v = iou_pair_ref(bx, gb + D * g);                      // tubes: mean over the frames (utils/boxes.py:60-69)
        for (int t = 1; t < T; ++t) v = __fadd_rn(v, iou_pair_ref(bx + 4 * t, gb + D * g + 4 * t));
        if (T > 1) v = __fdiv_rn(v, (float)T);
        if (g == 0 || v > best) { best = v; arg = g; }
      }
      if (G > 0 && best > 0.f) { mx = best; am = arg; c = gt_classes[b * p.Gmax + arg]; }
    }
    for (int k = 0; k < D; ++k) box[i * D + k] = bx[k];
    mov[i] = mx; bmap[i] = am; cls[i] = c;
  }
  __syncthreads();
  // ---- _sample_rois (fast_rcnn.py:118-186): foreground, then background, each drawn by the smallest (hash, index)
  int k_fg = 0, k_bg = 0;
  for (int phase = 0; phase < 2; ++phase) {
    const unsigned long long base = hash_base(p.seed, (unsigned long long)(2 + phase), (unsigned long long)b);
    int c = 0;
    const int per = (n + blockDim.x - 1) / blockDim.x;
    const int i0 = min(n, (int)threadIdx.x * per), i1 = min(n, i0 + per);
    for (int i = i0; i < i1; ++i) {
      const float m = mov[i];
      c += (phase == 0 ? (m >= p.fg_thresh) : (m < p.bg_hi && m >= p.bg_lo)) ? 1 : 0;
    }
    const int off = block_scan_excl(c, warp_sums, phase == 0 ? &s_c0 : &s_c1);
    int w = off;
    for (int i = i0; i < i1; ++i) {
      const float m = mov[i];
      if (phase == 0 ? (m >= p.fg_thresh) : (m < p.bg_hi && m >= p.bg_lo)) { list[w] = i; keys[w] = hash_u32(base, (unsigned long long)i); ++w; }
    }
    __syncthreads();
    const int nc = phase == 0 ? s_c0 : s_c1;
    const int want = phase == 0 ? min(p.fg_per, nc) : min(p.batch - k_fg, nc);
    for (int j = threadIdx.x; j < nc; j += blockDim.x) {
      const int r = rank_in(keys, list, nc, keys[j], list[j]);
      if (r < want) rowof[(phase == 0 ? 0 : k_fg) + r] = list[j];
    }
    if (phase == 0) k_fg = want; else k_bg = want;
    __syncthreads();
  }
  const int nrows = k_fg + k_bg;
  const int C4 = D * p.num_classes;
  for (int r = threadIdx.x; r < p.batch; r += blockDim.x) {
    float* ro = rois_out + ((size_t)b * p.batch + r) * (D + 1);
    float* bto = bt + ((size_t)b * p.batch + r) * C4;
    float* iwo = iw + ((size_t)b * p.batch + r) * C4;
    float* owo = ow + ((size_t)b * p.batch + r) * C4;
    for (int k = 0; k < C4; ++k) { bto[k] = 0.f; iwo[k] = 0.f; owo[k] = 0.f; }
    ro[0] = (float)b;
    if (r >= nrows) {
      for (int k = 0; k < D; ++k) ro[1 + k] = 0.f;
      labels[b * p.batch + r] = -1;                       // padding row: ignored by the losses
      continue;
    }
    const int i = rowof[r];
    const int lbl = r < k_fg ? cls[i] : 0;
    labels[b * p.batch + r] = lbl;
    for (int k = 0; k < D; ++k) ro[1 + k] = __fmul_rn(box[i * D + k], scale);
    if (lbl > 0) {
      int ga = bmap[i]; if (ga < 0) ga += G;              // gt_inds[-1]: python negative indexing
      for (int f = 0; f < T; ++f) {                       // tubes: frame by frame, fp64-promoted like the reference
        float t[4];
        if (T == 1) transform_inv(box + i * D, gb + D * ga, p.wx, p.wy, p.ww, p.wh, t);
        else transform_inv64(box + i * D + 4 * f, gb + D * ga + 4 * f, (double)p.wx, (double)p.wy, (double)p.ww, (double)p.wh, t);
#pragma unroll
        for (int k = 0; k < 4; ++k) { bto[D * lbl + 4 * f + k] = t[k]; iwo[D * lbl + 4 * f + k] = 1.f; owo[D * lbl + 4 * f + k] = 1.f; }
      }
    }
  }
  // ---- add_keypoint_rcnn_blobs (keypoint_rcnn.py:24-83)
  int nk = 0;
  bool by_index = true;
  if (kp_rois) {
    const unsigned long long base = hash_base(p.seed, 4ull, (unsigned long long)b);
    const int Kt = p.K * T;                               // gt_keypoints [G, 3, K*T] (utils/video.py:143-146)
    const int* kps = gt_kps + (size_t)b * p.Gmax * 3 * Kt;
    int c = 0;
    const int per = (n + blockDim.x - 1) / blockDim.x;
    const int i0 = min(n, (int)threadIdx.x * per), i1 = min(n, i0 + per);
    auto is_cand = [&](int i) -> bool {
      if (!(mov[i] >= p.fg_thresh) || G == 0) return false;
      int g = bmap[i]; if (g < 0) g += G;
      const int* kp = kps + (size_t)g * 3 * Kt;
      // keypoint_rcnn.py:32-34: _within_box tests every joint of every frame against the FIRST frame's box
      const double x1 = box[i * D], y1 = box[i * D + 1], x2 = box[i * D + 2], y2 = box[i * D + 3];
      for (int k = 0; k < Kt; ++k) {
        const double x = kp[k], y = kp[Kt + k];
        if (kp[2 * Kt + k] > 0 && x >= x1 && x <= x2 && y >= y1 && y <= y2) return true;
      }
      return false;
    };
    for (int i = i0; i < i1; ++i) c += is_cand(i) ? 1 : 0;
    const int off = block_scan_excl(c, warp_sums, &s_c0);
    int w = off;
    for (int i = i0; i < i1; ++i) if (is_cand(i)) { list[w] = i; keys[w] = hash_u32(base, (unsigned long long)i); ++w; }
    __syncthreads();
    const int nc = s_c0;
    nk = min(p.fg_per, nc);
    by_index = !(nc > nk);
    if (nc == 0) {
      nk = min(G, p.kcap);                                // no visible foreground RoI: train on the gt boxes themselves
      for (int j = threadIdx.x; j < nk; j += blockDim.x) rowof[p.batch + j] = j;
    } else {
      for (int j = threadIdx.x; j < nc; j += blockDim.x) {
        const int r = by_index ? j : rank_in(keys, list, nc, keys[j], list[j]);
        if (r < nk) rowof[p.batch + r] = list[j];
      }
    }
    __syncthreads();
    float wsum = 0.f;
    for (int e = threadIdx.x; e < p.kcap * Kt; e += blockDim.x) {
      const int r = e / Kt, k = e - r * Kt;               // k = frame * K + joint
      int loc = 0; float wt = 0.f;
      if (r < nk) {
        const int i = rowof[p.batch + r];
        const int g = bmap[i];
        int kx = -1, ky = -1, kv = -1;                    // sampled_keypoints = -1 without a gt
        if (g >= 0) { const int* kp = kps + (size_t)g * 3 * Kt; kx = kp[k]; ky = kp[Kt + k]; kv = kp[2 * Kt + k]; }
        // utils/keypoints.py:152-207 in fp32, frame f = k / K against that frame's box (keypoint_rcnn.py:62-70)
        const float* fb = box + i * D + 4 * (k / p.K);
        const float x1 = fb[0], y1 = fb[1], x2 = fb[2], y2 = fb[3];
        const float sx = __fdiv_rn((float)p.M, __fadd_rn(__fsub_rn(x2, x1), 1.f));
        const float sy = __fdiv_rn((float)p.M, __fadd_rn(__fsub_rn(y2, y1), 1.f));
        const float xf = (float)kx, yf = (float)ky;
        float x = floorf(__fmul_rn(__fsub_rn(xf, x1), sx));
        float y = floorf(__fmul_rn(__fsub_rn(yf, y1), sy));
        if (xf == x2) x = (float)(p.M - 1);
        if (yf == y2) y = (float)(p.M - 1);
        const bool valid = x >= 0.f && y >= 0.f && x < (float)p.M && y < (float)p.M && kv > 0;
        if (valid) { loc = (int)__fadd_rn(__fmul_rn(y, (float)p.M), x); wt = 1.f; }
      }
      kp_loc[((size_t)b * p.kcap + r) * Kt + k] = loc;
      kp_w[((size_t)b * p.kcap + r) * Kt + k] = wt;
      wsum += wt;
    }
    for (int r = threadIdx.x; r < p.kcap; r += blockDim.x) {
      float* ro = kp_rois + ((size_t)b * p.kcap + r) * (D + 1);
      ro[0] = (float)b;
      if (r < nk) {
        const int i = rowof[p.batch + r];
        for (int k = 0; k < D; ++k) ro[1 + k] = __fmul_rn(box[i * D + k], scale);
      } else {
        for (int k = 0; k < D; ++k) ro[1 + k] = 0.f;
      }
    }
    for (int o = 16; o > 0; o >>= 1) wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
    if ((threadIdx.x & 31) == 0 && wsum != 0.f) atomicAdd(&s_wsum, wsum);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    out_counts[b] = nrows;
    if (kp_counts) kp_counts[b] = nk;
    if (totals) { atomicAdd(&totals[0], (float)nrows); atomicAdd(&totals[1], s_wsum); }
  }
}

}  // namespace dt

using namespace dt;

extern "C" int dt_rpn_targets_workspace_bytes(int B, int n_levels, const int* Hs, const int* Ws, int A, int Gmax, size_t* bytes) {
  DT_CHECK_ARG(B >= 1 && n_levels >= 1 && n_levels <= 8 && Hs && Ws && A >= 1 && Gmax >= 1 && bytes, "dt_rpn_targets_workspace_bytes: bad arguments");
  long long NA = 0;
  for (int l = 0; l < n_levels; ++l) NA += (long long)Hs[l] * Ws[l] * A;
  *bytes = align_up((size_t)B * NA * 4, 256) * 2 + align_up((size_t)B * NA, 256) + align_up((size_t)B * Gmax * 4, 256) + align_up((size_t)B * 16, 256);
  return 0;
}

extern "C" int dt_rpn_targets(const dt_rpn_target_level* levels, int n_levels, int A, int T, int B, const float* gt_boxes,
                              const unsigned char* gt_visible, const int* gt_counts, int Gmax, const float* im_info, float straddle_thresh,
                              float positive_overlap, float negative_overlap, int batch_size_per_im, float fg_fraction,
                              unsigned long long seed, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  DT_CHECK_ARG(levels && n_levels >= 1 && n_levels <= 8 && A >= 1 && T >= 1 && T <= TG_TMAX && B >= 1 && Gmax >= 1 && Gmax <= TG_GMAX &&
                   batch_size_per_im >= 1 && batch_size_per_im <= 1024 && fg_fraction >= 0.f && fg_fraction <= 1.f,
               "dt_rpn_targets: bad arguments (levels <= 8, T <= %d, Gmax <= %d, batch <= 1024)", TG_TMAX, TG_GMAX);
  DT_CHECK_ARG(gt_boxes && gt_counts && im_info && workspace, "dt_rpn_targets: null pointer");
  RpnTL lv;
  memset(&lv, 0, sizeof(lv));
  lv.n_levels = n_levels; lv.A = A; lv.T = T;
  long long NA = 0;
  int Hs[8], Ws[8];
  for (int l = 0; l < n_levels; ++l) {
    const dt_rpn_target_level& s = levels[l];
    DT_CHECK_ARG(s.H >= 1 && s.W >= 1 && s.anchors && s.labels && s.bbox_targets && s.inside_weights && s.outside_weights && s.feat_stride > 0,
                 "dt_rpn_targets: level %d incomplete", l);
    lv.H[l] = s.H; lv.W[l] = s.W; lv.stride[l] = s.feat_stride; lv.cell[l] = s.anchors; lv.start[l] = (int)NA;
    lv.labels[l] = s.labels; lv.bt[l] = s.bbox_targets; lv.iw[l] = s.inside_weights; lv.ow[l] = s.outside_weights; lv.vis[l] = s.vis_labels;
    Hs[l] = s.H; Ws[l] = s.W;
    NA += (long long)s.H * s.W * A;
  }
  DT_CHECK_ARG(NA < (1ll << 30), "dt_rpn_targets: too many anchors");
  lv.start[n_levels] = (int)NA;
  size_t need = 0;
  dt_rpn_targets_workspace_bytes(B, n_levels, Hs, Ws, A, Gmax, &need);
  DT_CHECK_ARG(workspace_bytes >= need, "dt_rpn_targets: workspace %zu < %zu bytes", workspace_bytes, need);
  char* w = (char*)workspace;
  float* amax = (float*)w; w += align_up((size_t)B * NA * 4, 256);
  int* aarg = (int*)w; w += align_up((size_t)B * NA * 4, 256);
  signed char* lab = (signed char*)w; w += align_up((size_t)B * NA, 256);
  unsigned* gmax = (unsigned*)w; w += align_up((size_t)B * Gmax * 4, 256);
  int* cnt = (int*)w;
  DT_CHECK_CUDA(cudaMemsetAsync(gmax, 0, align_up((size_t)B * Gmax * 4, 256) + align_up((size_t)B * 16, 256), stream));
  dim3 grid((unsigned)((NA + 255) / 256), B);
  rpn_anchor_iou_kernel<<<grid, 256, 0, stream>>>(lv, (int)NA, gt_boxes, gt_counts, Gmax, im_info, straddle_thresh, amax, aarg, gmax);
  DT_CHECK_LAUNCH();
  rpn_label_kernel<<<grid, 256, 0, stream>>>(lv, (int)NA, gt_boxes, gt_counts, Gmax, im_info, positive_overlap, negative_overlap, amax, gmax, lab, cnt);
  DT_CHECK_LAUNCH();
  const int num_fg = (int)(fg_fraction * batch_size_per_im);
  const int sample_smem = (int)((NA + 31) / 32) * 4;
  DT_CHECK_ARG(sample_smem <= 200 * 1024, "dt_rpn_targets: %lld anchors per image exceed the draw kernel's shared memory", NA);
  static DynSmemGrant sample_grant;
  DT_CHECK_CUDA(grant_dyn_smem(rpn_sample_kernel, sample_smem, &sample_grant));
  rpn_sample_kernel<<<B, 1024, sample_smem, stream>>>((int)NA, batch_size_per_im, num_fg, negative_overlap, seed, amax, lab, cnt);
  DT_CHECK_LAUNCH();
  rpn_write_kernel<<<grid, 256, 0, stream>>>(lv, (int)NA, gt_boxes, gt_visible, gt_counts, Gmax, im_info, aarg, lab, cnt);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_sample_rois(const float* rois, const float* roi_scores, const int* roi_counts, int B, int R, int post_nms_topn,
                              const float* gt_boxes, const int* gt_classes, const int* gt_crowd, const int* gt_keypoints,
                              const int* gt_counts, int Gmax, int K, int T, const float* im_info, int num_classes, int batch_size_per_im,
                              float fg_fraction, float fg_thresh, float bg_thresh_hi, float bg_thresh_lo, const float* bbox_reg_weights,
                              int heatmap_size, unsigned long long seed, float* rois_out, int* labels, float* bbox_targets,
                              float* inside_weights, float* outside_weights, int* out_counts, float* kp_rois, int* kp_locations,
                              float* kp_weights, int* kp_counts, int kcap, float* totals, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  DT_CHECK_ARG(B >= 1 && R >= 1 && Gmax >= 1 && Gmax <= TG_GMAX && T >= 1 && T <= TG_TMAX && num_classes >= 2 && batch_size_per_im >= 1 &&
                   bbox_reg_weights, "dt_sample_rois: bad arguments B=%d R=%d Gmax=%d T=%d (T <= %d)", B, R, Gmax, T, TG_TMAX);
  DT_CHECK_ARG(rois && roi_scores && roi_counts && gt_boxes && gt_classes && gt_crowd && gt_counts && im_info && rois_out && labels &&
                   bbox_targets && inside_weights && outside_weights && out_counts, "dt_sample_rois: null pointer");
  DT_CHECK_ARG(!kp_rois || (gt_keypoints && kp_locations && kp_weights && kp_counts && K >= 1 && kcap >= 1 && heatmap_size >= 1),
               "dt_sample_rois: keypoint outputs need gt_keypoints, K, kcap, heatmap_size");
  SampleParams p;
  memset(&p, 0, sizeof(p));
  p.B = B; p.R = R; p.topn = post_nms_topn; p.Gmax = Gmax; p.K = K; p.T = T; p.num_classes = num_classes; p.batch = batch_size_per_im;
  p.fg_per = (int)nearbyint((double)fg_fraction * batch_size_per_im);
  p.kcap = kp_rois ? kcap : 0; p.M = heatmap_size;
  p.fg_thresh = fg_thresh; p.bg_hi = bg_thresh_hi; p.bg_lo = bg_thresh_lo;
  p.wx = bbox_reg_weights[0]; p.wy = bbox_reg_weights[1]; p.ww = bbox_reg_weights[2]; p.wh = bbox_reg_weights[3];
  p.seed = seed;
  DT_CHECK_ARG(!kp_rois || kcap >= (p.fg_per > Gmax ? p.fg_per : Gmax), "dt_sample_rois: kcap %d < max(fg rois per image %d, Gmax %d)", kcap, p.fg_per, Gmax);
  const int nmax = Gmax + R;
  const size_t smem = (size_t)nmax * (16 * T + 4 * 5) + (size_t)(batch_size_per_im + p.kcap) * 4 + 16;
  DT_CHECK_ARG(smem <= 220 * 1024, "dt_sample_rois: %d proposals per image do not fit shared memory", R);
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(sample_rois_kernel, (int)smem, &grant));
  sample_rois_kernel<<<B, 1024, smem, stream>>>(p, rois, roi_scores, roi_counts, gt_boxes, gt_classes, gt_crowd, gt_keypoints, gt_counts, im_info,
                                                rois_out, labels, bbox_targets, inside_weights, outside_weights, out_counts, kp_rois,
                                                kp_locations, kp_weights, kp_counts, totals);
  DT_CHECK_LAUNCH();
  return 0;
}
