// HBM-bound NDHWC kernels around the tensor-core convolutions (channels innermost, 16-byte vector
// accesses, one thread per 8 bf16 / 4 fp32 channels so every warp touches whole 128-byte lines):
//   dt_prep_clip        lib/utils/blob.py:40-90 + lib/core/test.py:43-74: mean-subtract, cv2
//                       INTER_LINEAR resize, zero pad to the /32 blob, BGR u8 -> NDHWC (C padded)
//   dt_prep_batch       lib/roi_data/minibatch.py:66-90: the same per clip of a training minibatch, each clip
//                       with its own source size, scale and horizontal flip, into one padded blob
//   dt_maxpool2d        Caffe2 MaxPool [1,k,k] (lib/modeling/ResNet3D.py:264-265; FPN P6 subsample
//                       lib/modeling/FPN3D.py:157-160)
//   dt_roi_align        Caffe2 RoIAlign (Detectron module; lib/modeling/detector.py:216-310) incl.
//                       the FPN level routing, tube -> per-frame boxes (lib/ops/roi_blob_transforms.py:
//                       25-36) and the BatchPermutation un-shuffle (rows are written in RoI order)
//   dt_keypoint_decode  fixed bilinear 2x ConvTranspose (lib/modeling/detector.py:348-380) applied to
//                       the sub-pixel-packed low-res scores + lib/utils/keypoints.py:94-149 heatmap ->
//                       (x, y, logit, prob) with the cv2 INTER_CUBIC resize evaluated on the fly
#include "common.cuh"
#include "../../include/dt_b200.h"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math_constants.h>

namespace dt {

template <typename T> struct Vec;
__device__ __forceinline__ float round_to_tf32(float v) {   // see conv_tc.cu: kind::tf32 truncates operands
  uint32_t u = __float_as_uint(v);
  u += 0xFFFu + ((u >> 13) & 1u);
  return __uint_as_float(u & 0xFFFFE000u);
}
template <typename T> __device__ __forceinline__ T to_act(float v);
template <> __device__ __forceinline__ float to_act<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 to_act<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <> struct Vec<float> {
  static constexpr int N = 4;
  __device__ static void load(const float* p, float* v) { const float4 q = *reinterpret_cast<const float4*>(p); v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w; }
  __device__ static void store(float* p, const float* v) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};
template <> struct Vec<__nv_bfloat16> {
  static constexpr int N = 8;
  __device__ static void load(const __nv_bfloat16* p, float* v) {
    const uint4 q = *reinterpret_cast<const uint4*>(p);
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) { v[2 * e] = __uint_as_float(w[e] << 16); v[2 * e + 1] = __uint_as_float(w[e] & 0xffff0000u); }
  }
  __device__ static void store(__nv_bfloat16* p, const float* v) {
    uint4 q; uint32_t* w = reinterpret_cast<uint32_t*>(&q);
#pragma unroll
    for (int e = 0; e < 4; ++e) { __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * e], v[2 * e + 1]); w[e] = *reinterpret_cast<uint32_t*>(&h); }
    *reinterpret_cast<uint4*>(p) = q;
  }
};

// Split ("x3") storage: a value is kept as hi + lo, the two halves `lo_off` elements apart in the channel row
// (lo_off == 0 means plain storage).  fp32 tensors: hi = tf32(v), lo = tf32(v - hi) (3xTF32 mode);
// bf16 tensors: hi = bf16(v), lo = bf16(v - hi) (bf16x3 mode, 16 mantissa bits).
template <typename ET> __device__ __forceinline__ float split_hi(float v);
template <> __device__ __forceinline__ float split_hi<float>(float v) { return round_to_tf32(v); }
template <> __device__ __forceinline__ float split_hi<__nv_bfloat16>(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
template <typename ET>
__device__ __forceinline__ void load_vals(const ET* p, int lo_off, float* v) {
  Vec<ET>::load(p, v);
  if (lo_off) {
    float l[Vec<ET>::N];
    Vec<ET>::load(p + lo_off, l);
#pragma unroll
    for (int e = 0; e < Vec<ET>::N; ++e) v[e] += l[e];
  }
}
template <typename ET>
__device__ __forceinline__ void store_vals(ET* p, int lo_off, float* v) {
  if (lo_off) {
    float l[Vec<ET>::N];
#pragma unroll
    for (int e = 0; e < Vec<ET>::N; ++e) { const float h = split_hi<ET>(v[e]); l[e] = split_hi<ET>(v[e] - h); v[e] = h; }
    Vec<ET>::store(p + lo_off, l);
  }
  Vec<ET>::store(p, v);
}

// ------------------------------------------------------------------- image prep
// frames [F, H, W, 3] u8 (BGR).  out [F, Hp, Wp, Cp]: channels 0..2 = resized (pixel - mean), rest 0;
// rows/cols beyond the resized image are 0 (blob.py:40-62).  cv2.resize(INTER_LINEAR) on float32:
// sx = (dx + 0.5) * (1/fx) - 0.5, floor, clamp, weights in float (see DESIGN.md, parity unpinned).
//
// One output pixel of frame f (both prep kernels call this, so their arithmetic is the same code).  The output
// buffer is [F, Ht = Hp + 2*by, Wt = Wp + 2*bx, Cp]: `by` zero rows above/below, `bx` zero pixels left/right;
// planes: the padded rows are de-interleaved, [F, 2 (row parity), Ht/2, Wt, Cp], so a stride-2 consumer
// (conv1) reads contiguous rows of one parity plane per filter row.  flip: the SOURCE frame is mirrored before
// the resize (minibatch.py:80-84, im[:, ::-1] then cv2.resize): the source column sx becomes W - 1 - sx with the
// interpolation weights unchanged (cv2 maps output columns through 1/fx, not W/Wr, so this is not the mirror of
// the resized image).
template <typename OT>
__device__ __forceinline__ void prep_pixel(const unsigned char* __restrict__ src, int H, int W, const float* mean,
                                           double inv_scale, int Hr, int Wr, int flip, int f, int y, int x, int Ht,
                                           int Wt, int by, int bx, int Cp, int round_out, int planes, int split_px,
                                           size_t idx, OT* __restrict__ out) {
  float v[3] = {0.f, 0.f, 0.f};
  if (y >= 0 && x >= 0 && y < Hr && x < Wr) {
    if (Hr == H && Wr == W) {
      const unsigned char* p = src + ((size_t)y * W + (flip ? W - 1 - x : x)) * 3;
      for (int c = 0; c < 3; ++c) v[c] = (float)p[c] - mean[c];
    } else {
      float fy = (float)((y + 0.5) * inv_scale - 0.5), fx = (float)((x + 0.5) * inv_scale - 0.5);
      int sy = (int)floorf(fy), sx = (int)floorf(fx);
      fy -= sy; fx -= sx;
      if (sy < 0) { sy = 0; fy = 0.f; }
      if (sy >= H - 1) { sy = H - 1 > 0 ? H - 2 : 0; fy = H > 1 ? 1.f : 0.f; if (H == 1) { sy = 0; } }
      if (sx < 0) { sx = 0; fx = 0.f; }
      if (sx >= W - 1) { sx = W - 1 > 0 ? W - 2 : 0; fx = W > 1 ? 1.f : 0.f; if (W == 1) { sx = 0; } }
      const int sy1 = min(sy + 1, H - 1);
      int sx1 = min(sx + 1, W - 1);
      if (flip) { sx = W - 1 - sx; sx1 = W - 1 - sx1; }
      for (int c = 0; c < 3; ++c) {
        const float p00 = (float)src[((size_t)sy * W + sx) * 3 + c] - mean[c];
        const float p01 = (float)src[((size_t)sy * W + sx1) * 3 + c] - mean[c];
        const float p10 = (float)src[((size_t)sy1 * W + sx) * 3 + c] - mean[c];
        const float p11 = (float)src[((size_t)sy1 * W + sx1) * 3 + c] - mean[c];
        const float r0 = p00 * (1.f - fx) + p01 * fx;      // horizontal pass first (cv2 hresize)
        const float r1 = p10 * (1.f - fx) + p11 * fx;
        v[c] = r0 * (1.f - fy) + r1 * fy;                  // then vertical
      }
    }
  }
  size_t oidx = idx;
  if (planes) {
    const int yt = y + by;
    oidx = (((size_t)f * 2 + (yt & 1)) * (Ht >> 1) + (yt >> 1)) * Wt + (x + bx);
  }
  OT* o = out + oidx * Cp;
  if (round_out) { v[0] = round_to_tf32(v[0]); v[1] = round_to_tf32(v[1]); v[2] = round_to_tf32(v[2]); }
  if (Cp * sizeof(OT) == 16) {                      // one 16-byte store per pixel
    float q[Vec<OT>::N];
#pragma unroll
    for (int c = 0; c < Vec<OT>::N; ++c) q[c] = c < 3 ? v[c] : 0.f;
    if constexpr (Vec<OT>::N >= 8) {
      if (split_px) {                               // bf16x3 conv1 blob: [hi3 | lo3 | 0 0]
#pragma unroll
        for (int c = 0; c < 3; ++c) { const float h = split_hi<OT>(v[c]); q[c] = h; q[3 + c] = v[c] - h; }
      }
    }
    Vec<OT>::store(o, q);
  } else {
    for (int c = 0; c < Cp; ++c) o[c] = to_act<OT>(c < 3 ? v[c] : 0.f);
  }
}

template <typename OT>
__global__ void prep_clip_kernel(const unsigned char* __restrict__ frames, int F, int H, int W, float m0, float m1,
                                 float m2, double inv_scale, int Hr, int Wr, int Hp, int Wp, int Cp,
                                 int by, int bx, int round_out, int planes, int split_px, OT* __restrict__ out) {
  const int Ht = Hp + 2 * by, Wt = Wp + 2 * bx;
  const long long total = (long long)F * Ht * Wt;
  const float mean[3] = {m0, m1, m2};
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % Wt) - bx;
    const int y = (int)((idx / Wt) % Ht) - by;
    const int f = (int)(idx / ((long long)Wt * Ht));
    prep_pixel<OT>(frames + (size_t)f * H * W * 3, H, W, mean, inv_scale, Hr, Wr, 0, f, y, x, Ht, Wt, by, bx, Cp, round_out,
                   planes, split_px, (size_t)idx, out);
  }
}

// dt_prep_batch: B clips of T frames, each with its own source size, scale, resized size and flip (a by-value table in
// the kernel's parameter space: no H2D copy, no allocation), into one [B*T, Ht, Wt, Cp] blob of a shared padded size.
struct PrepBatchClip {
  const unsigned char* frames;
  double inv_scale;
  int H, W, Hr, Wr, flip;
};
struct PrepBatchTable { PrepBatchClip c[DT_PREP_MAX_CLIPS]; };

template <typename OT>
__global__ void prep_batch_kernel(const __grid_constant__ PrepBatchTable tab, int B, int T, float m0, float m1, float m2,
                                  int Hp, int Wp, int Cp, int by, int bx, int round_out, int planes, int split_px,
                                  OT* __restrict__ out) {
  const int Ht = Hp + 2 * by, Wt = Wp + 2 * bx;
  const long long total = (long long)B * T * Ht * Wt;
  const float mean[3] = {m0, m1, m2};
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % Wt) - bx;
    const int y = (int)((idx / Wt) % Ht) - by;
    const int f = (int)(idx / ((long long)Wt * Ht));
    const PrepBatchClip& c = tab.c[f / T];
    prep_pixel<OT>(c.frames + (size_t)(f % T) * c.H * c.W * 3, c.H, c.W, mean, c.inv_scale, c.Hr, c.Wr, c.flip, f, y, x, Ht,
                   Wt, by, bx, Cp, round_out, planes, split_px, (size_t)idx, out);
  }
}

// ------------------------------------------------------------------- max pooling (NHWC)
template <typename ET>
__global__ void maxpool_kernel(const ET* __restrict__ x, int N, int H, int W, int C, int ldx, int k, int s, int p,
                               int Ho, int Wo, ET* __restrict__ y, int ldy, int lo_in, int lo_out) {
  constexpr int V = Vec<ET>::N;
  const int cv = C / V;
  const long long total = (long long)N * Ho * Wo * cv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * V;
    long long r = idx / cv;
    const int wo = (int)(r % Wo); r /= Wo;
    const int ho = (int)(r % Ho);
    const int n = (int)(r / Ho);
    float m[V];
#pragma unroll
    for (int e = 0; e < V; ++e) m[e] = -CUDART_INF_F;
    for (int kh = 0; kh < k; ++kh) {
      const int hi = ho * s - p + kh;
      if (hi < 0 || hi >= H) continue;
      for (int kw = 0; kw < k; ++kw) {
        const int wi = wo * s - p + kw;
        if (wi < 0 || wi >= W) continue;
        float v[V];
        load_vals<ET>(x + (((size_t)n * H + hi) * W + wi) * ldx + c, lo_in, v);
#pragma unroll
        for (int e = 0; e < V; ++e) m[e] = fmaxf(m[e], v[e]);
      }
    }
    store_vals<ET>(y + (((size_t)n * Ho + ho) * Wo + wo) * ldy + c, lo_out, m);
  }
}

// pool1 (3x3, stride 2, pad 1): a thread walks a vertical strip of PR output rows for one (wo, channel vector)
// and keeps the horizontal max of the shared input row (2*ho + 1 is the last row of window ho and the first of
// window ho + 1), so an output costs 6 vector loads instead of 9.
#define POOL_PR 8
template <typename ET>
__global__ void maxpool3x3s2_kernel(const ET* __restrict__ x, int N, int H, int W, int C, int ldx, int Ho, int Wo,
                                    ET* __restrict__ y, int ldy, int lo_in, int lo_out) {
  constexpr int V = Vec<ET>::N;
  const int cv = C / V;
  const int strips = (Ho + POOL_PR - 1) / POOL_PR;
  const long long total = (long long)N * strips * Wo * cv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * V;
    long long r = idx / cv;
    const int wo = (int)(r % Wo); r /= Wo;
    const int st = (int)(r % strips);
    const int n = (int)(r / strips);
    const int w0 = 2 * wo - 1;
    auto hmax = [&](int hi, float* m) {           // max over the three columns of input row hi (-inf outside)
#pragma unroll
      for (int e = 0; e < V; ++e) m[e] = -CUDART_INF_F;
      if (hi < 0 || hi >= H) return;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wi = w0 + kw;
        if (wi < 0 || wi >= W) continue;
        float v[V];
        load_vals<ET>(x + (((size_t)n * H + hi) * W + wi) * ldx + c, lo_in, v);
#pragma unroll
        for (int e = 0; e < V; ++e) m[e] = fmaxf(m[e], v[e]);
      }
    };
    const int ho0 = st * POOL_PR, ho1 = min(ho0 + POOL_PR, Ho);
    float prev[V];
    hmax(2 * ho0 - 1, prev);
    for (int ho = ho0; ho < ho1; ++ho) {
      float a[V], b[V];
      hmax(2 * ho, a);
      hmax(2 * ho + 1, b);
      float m[V];
#pragma unroll
      for (int e = 0; e < V; ++e) { m[e] = fmaxf(fmaxf(prev[e], a[e]), b[e]); prev[e] = b[e]; }
      store_vals<ET>(y + (((size_t)n * Ho + ho) * Wo + wo) * ldy + c, lo_out, m);
    }
  }
}

// ------------------------------------------------------------------- RoIAlign (multi-level, tubes)
struct RoiLevels {
  const void* feat[8];
  int H[8], W[8];
  float scale[8];
};

template <typename ET>
__device__ __forceinline__ void bilinear_acc(const ET* __restrict__ f, int H, int W, int ld, int lo_in, float y, float x, float* acc) {
  constexpr int V = Vec<ET>::N;
  if (!(y >= -1.f && y <= (float)H && x >= -1.f && x <= (float)W)) return;      // contributes 0 (also for a non-finite RoI)
  if (y <= 0.f) y = 0.f;
  if (x <= 0.f) x = 0.f;
  int yl = (int)y, xl = (int)x, yh, xh;
  if (yl >= H - 1) { yh = yl = H - 1; y = (float)yl; } else yh = yl + 1;
  if (xl >= W - 1) { xh = xl = W - 1; x = (float)xl; } else xh = xl + 1;
  const float ly = y - yl, lx = x - xl, hy = 1.f - ly, hx = 1.f - lx;
  const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
  float v1[V], v2[V], v3[V], v4[V];
  load_vals<ET>(f + ((size_t)yl * W + xl) * ld, lo_in, v1);
  load_vals<ET>(f + ((size_t)yl * W + xh) * ld, lo_in, v2);
  load_vals<ET>(f + ((size_t)yh * W + xl) * ld, lo_in, v3);
  load_vals<ET>(f + ((size_t)yh * W + xh) * ld, lo_in, v4);
#pragma unroll
  for (int e = 0; e < V; ++e) acc[e] += w1 * v1[e] + w2 * v2[e] + w3 * v3[e] + w4 * v4[e];
}

// rois [R, ldr]: col 0 batch idx, then 4*T box columns.  out [R, T, P, P, C].
// grid: (R*T, P) blocks; threads over (pw, channel vectors).
template <typename ET>
__global__ void roi_align_kernel(RoiLevels lv, int kmin, const float* __restrict__ rois, int ldr,
                                 const int* __restrict__ n_dev, int R, int T, const int* __restrict__ levels, int C,
                                 int ldf, int P, int sampling, int round_out, int lo_in, long long o_row, int o_pos,
                                 int o_lo, ET* __restrict__ out) {
  // output addressing: roi r starts at r*o_row, position (t, ph, pw) at ((t*P + ph)*P + pw)*o_pos, the lo
  // half (3xTF32 storage) o_lo elements further (0 = plain).
  constexpr int V = Vec<ET>::N;
  const int rt = blockIdx.x, ph = blockIdx.y;
  const int r = rt / T, t = rt - r * T;
  const int n = n_dev ? min(*n_dev, R) : R;
  const int cv = C / V;
  ET* obase = out + (size_t)r * o_row + ((size_t)t * P + ph) * P * o_pos;
  if (r >= n) {          // rows beyond the live count are zero-filled (keeps downstream GEMMs finite)
    for (int i = threadIdx.x; i < P * cv; i += blockDim.x) {
      float z[V];
#pragma unroll
      for (int e = 0; e < V; ++e) z[e] = 0.f;
      store_vals<ET>(obase + (size_t)(i / cv) * o_pos + (i % cv) * V, o_lo, z);
    }
    return;
  }
  const float* roi = rois + (size_t)r * ldr;
  const int l = levels ? (levels[r] - kmin) : 0;
  const int H = lv.H[l], W = lv.W[l];
  const float sc = lv.scale[l];
  const int img = (int)roi[0] * T + t;                 // RoIToBatchFormat: b*T + t
  const ET* f = reinterpret_cast<const ET*>(lv.feat[l]) + (size_t)img * H * W * ldf;
  const float x1 = roi[1 + 4 * t] * sc, y1 = roi[2 + 4 * t] * sc, x2 = roi[3 + 4 * t] * sc, y2 = roi[4 + 4 * t] * sc;
  const float rw = fmaxf(x2 - x1, 1.f), rh = fmaxf(y2 - y1, 1.f);
  const float bh = rh / (float)P, bw = rw / (float)P;
  const int gh = sampling > 0 ? sampling : (int)ceilf(rh / P), gw = sampling > 0 ? sampling : (int)ceilf(rw / P);
  const float cnt = (float)(gh * gw);
  for (int i = threadIdx.x; i < P * cv; i += blockDim.x) {
    const int pw = i / cv, c = (i - pw * cv) * V;
    float acc[V];
#pragma unroll
    for (int e = 0; e < V; ++e) acc[e] = 0.f;
    for (int iy = 0; iy < gh; ++iy) {
      const float y = y1 + ph * bh + (iy + 0.5f) * bh / (float)gh;
      for (int ix = 0; ix < gw; ++ix) {
        const float x = x1 + pw * bw + (ix + 0.5f) * bw / (float)gw;
        bilinear_acc<ET>(f + c, H, W, ldf, lo_in, y, x, acc);
      }
    }
#pragma unroll
    for (int e = 0; e < V; ++e) acc[e] /= cnt;
    if (round_out && !o_lo) {
#pragma unroll
      for (int e = 0; e < V; ++e) acc[e] = round_to_tf32(acc[e]);
    }
    store_vals<ET>(obase + (size_t)pw * o_pos + c, o_lo, acc);
  }
}

// ------------------------------------------------------------------- keypoint decode
// lowres [D, S, S, ldl]: channel (py*2+px)*K + k holds kps_score_lowres[k] at output pixel
// (2*y+py, 2*x+px) (the k4 s2 p1 ConvTranspose evaluated as four 2x2 sub-pixel filters by the
// conv kernel).  Step 1: fixed bilinear 2x ConvTranspose (filter [.25,.75,.75,.25]) -> M x M map in
// shared memory (M = 4*S = 56).  Step 2: cv2.resize(INTER_CUBIC, A=-0.75, replicate border) to
// (ceil(w), ceil(h)) evaluated per output pixel, first-occurrence argmax, softmax prob at the max.
// One CTA per (detection, keypoint, frame).
__device__ __forceinline__ void cubic_coeffs(float x, float* c) {
  const float A = -0.75f;
  c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
  c[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
  c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
  c[3] = 1.f - c[0] - c[1] - c[2];
}

#define KD_SW 256   // output columns per strip of the separable cubic resize
#define KD_RB 256   // output rows per block of precomputed vertical weights

// Un-packs joint k of one RoI-frame's sub-pixel low-res row block src [S, S, ldl] into low [2S * 2S].
__device__ __forceinline__ void kd_unpack(const float* __restrict__ src, int S, int ldl, int K, int k, float* low) {
  const int M2 = 2 * S;
  for (int i = threadIdx.x; i < M2 * M2; i += blockDim.x) {
    const int oy = i / M2, ox = i - oy * M2;
    low[i] = src[((size_t)(oy >> 1) * S + (ox >> 1)) * ldl + ((oy & 1) * 2 + (ox & 1)) * K + k];
  }
}

// bilinear ConvTranspose k=4 s=2 p=1 of the un-packed map at output pixel (oy, ox): out[o] = sum_i in[i] * f[o - 2i + 1]
__device__ __forceinline__ float kd_upsample_px(const float* low, int M2, int oy, int ox) {
  const int iy0 = (oy + 1) >> 1, ix0 = (ox + 1) >> 1;          // taps i = iy0 (ky = o-2i+1) and iy0-1 (ky+2)
  float acc = 0.f;
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const int iy = iy0 - a, ky = oy - 2 * iy + 1;
    if (iy < 0 || iy >= M2 || ky < 0 || ky > 3) continue;
    const float fy = 1.f - fabsf(ky - 1.5f) / 2.f;
#pragma unroll
    for (int bq = 0; bq < 2; ++bq) {
      const int ix = ix0 - bq, kx = ox - 2 * ix + 1;
      if (ix < 0 || ix >= M2 || kx < 0 || kx > 3) continue;
      const float fx = 1.f - fabsf(kx - 1.5f) / 2.f;
      acc += low[iy * M2 + ix] * (fy * fx);
    }
  }
  return acc;
}

// ---- heatmaps_to_keypoints (keypoints.py:94-149) for one (roi, keypoint) M x M map in shared memory ----
// Block-wide (every thread calls it); map is followed by the scratch the launchers size.  bx = the RoI's image-space box,
// o = its xy_preds row [4, KT], col = the output column.
__device__ __forceinline__ void kd_decode_map(float* map, int M, const float* __restrict__ bx, int min_size, float* o, int KT,
                                              int col) {
  __shared__ float s_red[32];
  __shared__ float s_max;
  const int tid = threadIdx.x, nth = blockDim.x;
  // cv2.resize(INTER_CUBIC) is separable and cv2 evaluates it in this order too: horizontal pass on
  // the source rows (float), then a 4-tap vertical combination.  Work is done in strips of KD_SW output
  // columns: H-pass of all M source rows into smem, then each thread walks its column top to bottom
  // keeping (max, first argmax, online sum of exp(v - max)).
  const float ofx = bx[0], ofy = bx[1];
  const float bw = fmaxf(bx[2] - bx[0], 1.f), bh = fmaxf(bx[3] - bx[1], 1.f);
  int rw = (int)ceilf(bw), rh = (int)ceilf(bh);
  if (min_size > 0) { rw = max(rw, min_size); rh = max(rh, min_size); }
  const float wcorr = bw / (float)rw, hcorr = bh / (float)rh;
  const double sclx = 1.0 / ((double)rw / M), scly = 1.0 / ((double)rh / M);   // cv2: scale = 1 / (dsize / ssize)
  float* tmp = map + M * M;        // [M][KD_SW] horizontally resized strip
  float4* cxs = reinterpret_cast<float4*>(tmp + M * KD_SW);   // [KD_SW] cubic weights of the strip's columns
  int* sxs = reinterpret_cast<int*>(cxs + KD_SW);             // [KD_SW] their first source column
  float4* cys = reinterpret_cast<float4*>(sxs + KD_SW);       // [KD_RB] cubic weights of a block of output rows
  int* sys = reinterpret_cast<int*>(cys + KD_RB);             // [KD_RB] their first source row
  float best = -CUDART_INF_F; int besti = 0x7fffffff;          // rw * rh < 2^31: boxes are clipped to the image
  float run_max = -CUDART_INF_F, run_sum = 0.f;
  for (int x0 = 0; x0 < rw; x0 += KD_SW) {
    const int sw = min(KD_SW, rw - x0);
    // horizontal pass: a thread owns one output column of the strip (weights and clamped source columns in
    // registers) and a phase of the M source rows
    {
      const int nsegh = max(1, nth / sw);
      const int xh = tid % sw, segh = tid / sw;
      if (segh < nsegh) {
        float fx = (float)((x0 + xh + 0.5) * sclx - 0.5);
        const int sx = (int)floorf(fx);
        fx -= sx;
        float cx[4];
        cubic_coeffs(fx, cx);
        const int i0 = min(max(sx - 1, 0), M - 1), i1 = min(max(sx, 0), M - 1);
        const int i2 = min(max(sx + 1, 0), M - 1), i3 = min(max(sx + 2, 0), M - 1);
        for (int y = segh; y < M; y += nsegh) {
          const float* mr = map + y * M;
          float rowv = 0.f;
          rowv += mr[i0] * cx[0];
          rowv += mr[i1] * cx[1];
          rowv += mr[i2] * cx[2];
          rowv += mr[i3] * cx[3];
          tmp[y * KD_SW + xh] = rowv;
        }
      }
    }
    // vertical pass: a thread owns FOUR adjacent columns and a row phase, so the per-row weights are fetched
    // once per four pixels, the source rows come in as 16-byte vectors and narrow boxes keep every lane busy;
    // each thread keeps (max, first argmax, online sum of exp(v - max)) over the pixels it visits
    const int ncol4 = (sw + 3) >> 2;
    const int nseg = max(1, nth / ncol4);
    const int xl = (tid % ncol4) << 2, seg = tid / ncol4;
    for (int r0 = 0; r0 < rh; r0 += KD_RB) {
      const int rb = min(KD_RB, rh - r0);
      __syncthreads();                       // tmp complete / previous row block consumed
      for (int r = tid; r < rb; r += nth) {
        float fy = (float)((r0 + r + 0.5) * scly - 0.5);
        const int sy = (int)floorf(fy);
        fy -= sy;
        float cy[4];
        cubic_coeffs(fy, cy);
        cys[r] = make_float4(cy[0], cy[1], cy[2], cy[3]);
        sys[r] = sy;
      }
      __syncthreads();
      if (seg < nseg) {
        for (int r = seg; r < rb; r += nseg) {
          const float4 c = cys[r];
          const int sy = sys[r];
          const float4 t0 = *reinterpret_cast<const float4*>(tmp + min(max(sy - 1, 0), M - 1) * KD_SW + xl);
          const float4 t1 = *reinterpret_cast<const float4*>(tmp + min(max(sy, 0), M - 1) * KD_SW + xl);
          const float4 t2 = *reinterpret_cast<const float4*>(tmp + min(max(sy + 1, 0), M - 1) * KD_SW + xl);
          const float4 t3 = *reinterpret_cast<const float4*>(tmp + min(max(sy + 2, 0), M - 1) * KD_SW + xl);
          float v[4];
          {
            const float a0[4] = {t0.x, t0.y, t0.z, t0.w}, a1[4] = {t1.x, t1.y, t1.z, t1.w};
            const float a2[4] = {t2.x, t2.y, t2.z, t2.w}, a3[4] = {t3.x, t3.y, t3.z, t3.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float vv = 0.f;
              vv += a0[j] * c.x; vv += a1[j] * c.y; vv += a2[j] * c.z; vv += a3[j] * c.w;
              v[j] = (xl + j < sw) ? vv : -CUDART_INF_F;          // columns past the strip never win / add 0
            }
          }
          const int lin = (r0 + r) * rw + (x0 + xl);
#pragma unroll
          for (int j = 0; j < 4; ++j)                              // ascending index: '>' keeps the first maximum
            if (v[j] > best || (v[j] == best && lin + j < besti)) { best = v[j]; besti = lin + j; }
          const float m4 = fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3]));
          if (m4 > run_max) { run_sum *= __expf(run_max - m4); run_max = m4; }
          run_sum += (__expf(v[0] - run_max) + __expf(v[1] - run_max)) + (__expf(v[2] - run_max) + __expf(v[3] - run_max));
        }
      }
    }
    __syncthreads();
  }
  // block reduction: (max value, lowest linear index) and the softmax denominator at the global max
  __shared__ long long s_redl[32];
  float bm = best; long long bi = besti;     // (idle threads carry -inf / INT_MAX)
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, bm, o);
    const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > bm || (ob == bm && oi < bi)) { bm = ob; bi = oi; }
  }
  if ((tid & 31) == 0) { s_red[tid >> 5] = bm; s_redl[tid >> 5] = bi; }
  __syncthreads();
  if (tid == 0) {
    float b2 = s_red[0]; long long i2 = s_redl[0];
    for (int w = 1; w < (nth >> 5); ++w)
      if (s_red[w] > b2 || (s_red[w] == b2 && s_redl[w] < i2)) { b2 = s_red[w]; i2 = s_redl[w]; }
    s_max = b2; s_redl[0] = i2;
  }
  __syncthreads();
  const float mx = s_max;
  const long long pos = s_redl[0];
  __syncthreads();
  float sum = (run_max == -CUDART_INF_F) ? 0.f : run_sum * expf(run_max - mx);
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((tid & 31) == 0) s_red[tid >> 5] = sum;
  __syncthreads();
  if (tid == 0) {
    float tot = 0.f;
    for (int w = 0; w < (nth >> 5); ++w) tot += s_red[w];
    const int x_int = (int)(pos % rw), y_int = (int)(pos / rw);
    // keypoints.py:140-145: python floats (fp64) until the store into the fp32 result
    o[0 * KT + col] = (float)((x_int + 0.5) * (double)wcorr + (double)ofx);
    o[1 * KT + col] = (float)((y_int + 0.5) * (double)hcorr + (double)ofy);
    o[2 * KT + col] = mx;
    o[3 * KT + col] = 1.f / tot;           // exp(max - max) / sum
  }
}

__global__ void __launch_bounds__(256)
keypoint_decode_kernel(const float* __restrict__ lowres, int ldl, int S, int K, int T,
                       const float* __restrict__ boxes /*[D, ldb] image coords*/, int ldb,
                       const int* __restrict__ n_dev, int D, int min_size,
                       float* __restrict__ heat /*[D, T*K, M, M] or null*/,
                       float* __restrict__ xy /*[D, 4, T*K]*/) {
  extern __shared__ float sm[];
  const int M2 = 2 * S, M = 4 * S;
  float* low = sm;                 // [M2*M2]  kps_score_lowres for this (d, k)
  float* map = sm + M2 * M2;       // [M*M]    kps_score
  const int d = blockIdx.x, k = blockIdx.y, t = blockIdx.z;
  const int n = n_dev ? min(*n_dev, D) : D;
  if (d >= n) return;
  // un-pack the sub-pixel channels of frame t (row d*T + t of the time-in-batch lowres tensor)
  kd_unpack(lowres + (size_t)(d * T + t) * S * S * ldl, S, ldl, K, k, low);
  __syncthreads();
  for (int i = threadIdx.x; i < M * M; i += blockDim.x) {
    const int oy = i / M, ox = i - oy * M;
    const float acc = kd_upsample_px(low, M2, oy, ox);
    map[i] = acc;
    if (heat) heat[(((size_t)d * T + t) * K + k) * M * M + i] = acc;   // channel t*K + k (model_builder.py:865-868)
  }
  __syncthreads();
  kd_decode_map(map, M, boxes + (size_t)d * ldb + 4 * t, min_size, xy + (size_t)d * 4 * K * T, K * T, t * K + k);
}

// Test-time augmentation of the keypoint stage (lib/core/test.py:686-747) for 2-D heads: V views' low-res maps of the
// same RoIs, lowres + v * view_stride = [D, S, S, ldl].  Per (roi, joint): every view's M x M kps_score exactly as
// keypoint_decode_kernel builds it; a flipped view contributes joint perm[k], mirrored in x (flip_heatmaps,
// lib/utils/keypoints.py:81-91).  The views are combined in view order — HM_AVG: fp32 running sum, then / V (np.mean over
// axis 0); HM_MAX: running max (np.amax) — and the combined map is decoded against the original boxes.
struct KdAugTable {
  int flip[DT_AUG_MAX_VIEWS];
  int perm[DT_KD_AUG_MAX_K];
};

__global__ void __launch_bounds__(256)
keypoint_decode_aug_kernel(const float* __restrict__ lowres, long long view_stride, int ldl, int S, int K, int V,
                           const __grid_constant__ KdAugTable tab, int hm_max, const float* __restrict__ boxes, int ldb,
                           const int* __restrict__ n_dev, int D, int min_size, float* __restrict__ heat /*[D, K, M, M] or null*/,
                           float* __restrict__ xy /*[D, 4, K]*/) {
  extern __shared__ float sm[];
  const int M2 = 2 * S, M = 4 * S;
  float* low = sm;                 // [M2*M2]  one view's kps_score_lowres for this (d, joint)
  float* map = sm + M2 * M2;       // [M*M]    the combined kps_score
  const int d = blockIdx.x, k = blockIdx.y;
  const int n = n_dev ? min(*n_dev, D) : D;
  if (d >= n) return;
  for (int v = 0; v < V; ++v) {
    const int fl = tab.flip[v];
    if (v) __syncthreads();                                   // the previous view's low map is consumed
    kd_unpack(lowres + v * view_stride + (size_t)d * S * S * ldl, S, ldl, K, fl ? tab.perm[k] : k, low);
    __syncthreads();
    for (int i = threadIdx.x; i < M * M; i += blockDim.x) {
      const int oy = i / M, ox = i - oy * M;
      const float val = kd_upsample_px(low, M2, oy, ox);
      const int dst = oy * M + (fl ? M - 1 - ox : ox);
      if (v == 0) map[dst] = val;
      else if (hm_max) { const float cur = map[dst]; map[dst] = cur >= val ? cur : val; }   // np.maximum(cur, val)
      else map[dst] = __fadd_rn(map[dst], val);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < M * M; i += blockDim.x) {
    const float c = hm_max ? map[i] : __fdiv_rn(map[i], (float)V);
    map[i] = c;
    if (heat) heat[((size_t)d * K + k) * M * M + i] = c;
  }
  __syncthreads();
  kd_decode_map(map, M, boxes + (size_t)d * ldb, min_size, xy + (size_t)d * 4 * K, K, k);
}

// ------------------------------------------------------------------- 3-D box head glue
// ReduceBackMean over W then over H (lib/modeling/ResNet3D.py:321-322): x [N, H, W, ldx] -> y [N, C]
template <typename ET>
__global__ void spatial_mean_kernel(const ET* __restrict__ x, int N, int H, int W, int C, int ldx, ET* __restrict__ y,
                                    int ldy, int round_out, int lo_in, int lo_out) {
  constexpr int V = Vec<ET>::N;
  const int cv = C / V;
  const long long total = (long long)N * cv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * V;
    const int n = (int)(idx / cv);
    float acc[V];
#pragma unroll
    for (int e = 0; e < V; ++e) acc[e] = 0.f;
    for (int h = 0; h < H; ++h) {
      float row[V];
#pragma unroll
      for (int e = 0; e < V; ++e) row[e] = 0.f;
      for (int w = 0; w < W; ++w) {
        float v[V];
        load_vals<ET>(x + (((size_t)n * H + h) * W + w) * ldx + c, lo_in, v);
#pragma unroll
        for (int e = 0; e < V; ++e) row[e] += v[e];
      }
#pragma unroll
      for (int e = 0; e < V; ++e) acc[e] += row[e] / (float)W;
    }
#pragma unroll
    for (int e = 0; e < V; ++e) { acc[e] /= (float)H; if (round_out && !lo_out) acc[e] = round_to_tf32(acc[e]); }
    store_vals<ET>(y + (size_t)n * ldy + c, lo_out, acc);
  }
}

// TimePool 'avg' body/head link (lib/modeling/model_builder.py:1024-1042, detector.py:559-576):
// x [B, T, P, ldx] -> y [B, P, ldy], mean over the T frames (sequential fp32 sum, then / T).
template <typename ET>
__global__ void time_mean_kernel(const ET* __restrict__ x, int B, int T, long long P, int C, int ldx, ET* __restrict__ y,
                                 int ldy, int round_out, int lo_in, int lo_out) {
  constexpr int V = Vec<ET>::N;
  const int cv = C / V;
  const long long total = (long long)B * P * cv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * V;
    const long long r = idx / cv;
    const long long pos = r % P;
    const long long b = r / P;
    float acc[V];
    load_vals<ET>(x + ((size_t)(b * T) * P + pos) * ldx + c, lo_in, acc);
    for (int t = 1; t < T; ++t) {
      float v[V];
      load_vals<ET>(x + ((size_t)(b * T + t) * P + pos) * ldx + c, lo_in, v);
#pragma unroll
      for (int e = 0; e < V; ++e) acc[e] += v[e];
    }
#pragma unroll
    for (int e = 0; e < V; ++e) { acc[e] /= (float)T; if (round_out && !lo_out) acc[e] = round_to_tf32(acc[e]); }
    store_vals<ET>(y + ((size_t)b * P + pos) * ldy + c, lo_out, acc);
  }
}

// add_fast_rcnn_outputs, 3-D head (lib/modeling/model_builder.py:427-473): per-frame outputs
// in [R*T, ld] = [cls logits (C) | bbox (4C, channel c*4+k)] -> cls [R, C] = mean over T,
// bbox [R, C*T*4] with channel c*4T + t*4 + k.
__global__ void fold_tube_heads_kernel(const float* __restrict__ in, int ld, int R, int T, int C,
                                       float* __restrict__ cls, float* __restrict__ bbox) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  for (int c = 0; c < C; ++c) {
    float acc = in[((size_t)r * T) * ld + c];
    for (int t = 1; t < T; ++t) acc += in[((size_t)r * T + t) * ld + c];
    cls[(size_t)r * C + c] = acc / (float)T;
  }
  for (int c = 0; c < C; ++c)
    for (int t = 0; t < T; ++t)
      for (int k = 0; k < 4; ++k)
        bbox[(size_t)r * C * T * 4 + (size_t)c * 4 * T + 4 * t + k] = in[((size_t)r * T + t) * ld + C + c * 4 + k];
}

// ------------------------------------------------------------------- conv1, exact fp32 (3xTF32 mode)
// 7x7 stride 2 pad 3 conv + AffineChannel + ReLU in plain fp32 FMAs (lib/modeling/ResNet3D.py:258-263);
// output stored as [hi | lo] tf32 pairs for the 3xTF32 consumers.  blob [F, Hp, Wp, Cp] raw fp32.
// One CTA = 32 output pixels x 64 channels; thread = (pixel, 8 channels); weights [147][64] in smem.
template <typename OT>
__global__ void __launch_bounds__(256)
conv1_f32_kernel(const float* __restrict__ blob, int F, int Hp, int Wp, int Cp, const float* __restrict__ w /*[7][7][3][64]*/,
                 const float* __restrict__ scale, const float* __restrict__ bias, OT* __restrict__ y /*[F,Ho,Wo,128]*/) {
  __shared__ float sw[147 * 64];
  for (int i = threadIdx.x; i < 147 * 64; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int Ho = Hp / 2, Wo = Wp / 2;
  const long long total = (long long)F * Ho * Wo;
  const long long pix = (long long)blockIdx.x * 32 + (threadIdx.x >> 3);
  const int cg = (threadIdx.x & 7) * 8;
  if (pix >= total) return;
  const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho), f = (int)(pix / ((long long)Wo * Ho));
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  for (int kh = 0; kh < 7; ++kh) {
    const int hi = 2 * ho - 3 + kh;
    if (hi < 0 || hi >= Hp) continue;
    for (int kw = 0; kw < 7; ++kw) {
      const int wi = 2 * wo - 3 + kw;
      if (wi < 0 || wi >= Wp) continue;
      const float* px = blob + (((size_t)f * Hp + hi) * Wp + wi) * Cp;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float xv = px[c];
        const float* wr = sw + ((kh * 7 + kw) * 3 + c) * 64 + cg;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = fmaf(xv, wr[e], acc[e]);
      }
    }
  }
  OT* o = y + (size_t)pix * 128 + cg;
  constexpr int V = Vec<OT>::N;
#pragma unroll
  for (int e = 0; e < 8; e += V) {
    float v[V];
#pragma unroll
    for (int q = 0; q < V; ++q) v[q] = fmaxf(fmaf(acc[e + q], scale[cg + e + q], bias[cg + e + q]), 0.f);
    store_vals<OT>(o + e, 64, v);
  }
}

// bf16 pair rows [rows, 2C] -> fp16 rows [rows, C]: v = hi + lo (exact in fp32), fp16 round-to-nearest, saturating
__global__ void pairs_to_f16_kernel(const __nv_bfloat16* __restrict__ in, long long rows, int C, __half* __restrict__ out) {
  const int cv = C / 8;
  const long long total = rows * cv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * 8;
    const long long r = idx / cv;
    float v[8];
    load_vals<__nv_bfloat16>(in + (size_t)r * 2 * C + c, C, v);
    __align__(16) __half h[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) h[e] = __float2half_rn(fminf(fmaxf(v[e], -65504.f), 65504.f));
    *reinterpret_cast<uint4*>(out + (size_t)r * C + c) = *reinterpret_cast<const uint4*>(h);
  }
}

}  // namespace dt

using namespace dt;

static int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = num_sms() * 16ll;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

extern "C" int dt_prep_clip(const unsigned char* frames, int F, int H, int W, const float* mean3 /*host*/,
                            double im_scale, int Hr, int Wr, int Hp, int Wp, int Cp, int border_y, int border_x,
                            int row_planes, int out_f32, void* out, void* stream) {
  DT_CHECK_ARG(F >= 0 && H >= 1 && W >= 1 && Hr >= 1 && Wr >= 1 && Hp >= Hr && Wp >= Wr && Cp >= 3 && im_scale > 0,
               "dt_prep_clip: bad shape F=%d H=%d W=%d Hr=%d Wr=%d Hp=%d Wp=%d Cp=%d", F, H, W, Hr, Wr, Hp, Wp, Cp);
  if (F == 0) return 0;
  DT_CHECK_ARG(frames && mean3 && out, "dt_prep_clip: null pointer");
  DT_CHECK_ARG(border_y >= 0 && border_x >= 0, "dt_prep_clip: negative border");
  DT_CHECK_ARG(!row_planes || (Hp + 2 * border_y) % 2 == 0, "dt_prep_clip: row planes need an even padded height");
  const long long total = (long long)F * (Hp + 2 * border_y) * (Wp + 2 * border_x);
  DT_CHECK_ARG(out_f32 >= 0 && out_f32 <= 3 && (out_f32 != 3 || Cp == 8), "dt_prep_clip: bad output mode %d (mode 3 needs Cp == 8)", out_f32);
  if (out_f32 == 3)
    prep_clip_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        frames, F, H, W, mean3[0], mean3[1], mean3[2], 1.0 / im_scale, Hr, Wr, Hp, Wp, Cp, border_y, border_x, 0, row_planes, 1, (__nv_bfloat16*)out);
  else if (out_f32)
    prep_clip_kernel<float><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(frames, F, H, W, mean3[0], mean3[1], mean3[2],
                                                                                 1.0 / im_scale, Hr, Wr, Hp, Wp, Cp, border_y, border_x, out_f32 == 1, row_planes, 0, (float*)out);
  else
    prep_clip_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        frames, F, H, W, mean3[0], mean3[1], mean3[2], 1.0 / im_scale, Hr, Wr, Hp, Wp, Cp, border_y, border_x, 0, row_planes, 0, (__nv_bfloat16*)out);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_prep_batch(const unsigned char* const* frames, const int* H, const int* W, const double* im_scale,
                             const int* Hr, const int* Wr, const int* flip, int B, int T, const float* mean3, int Hp, int Wp,
                             int Cp, int border_y, int border_x, int row_planes, int out_f32, void* out, void* stream) {
  DT_CHECK_ARG(B >= 1 && B <= DT_PREP_MAX_CLIPS && T >= 1, "dt_prep_batch: need 1 <= B <= %d clips and T >= 1 (B=%d T=%d)",
               DT_PREP_MAX_CLIPS, B, T);
  DT_CHECK_ARG(frames && H && W && im_scale && Hr && Wr && flip && mean3 && out, "dt_prep_batch: null pointer");
  DT_CHECK_ARG(Hp >= 1 && Wp >= 1 && border_y >= 0 && border_x >= 0, "dt_prep_batch: bad padded size %dx%d or border %d,%d",
               Hp, Wp, border_y, border_x);
  PrepBatchTable tab;
  for (int b = 0; b < B; ++b) {
    DT_CHECK_ARG(frames[b], "dt_prep_batch: null frame pointer of clip %d", b);
    DT_CHECK_ARG(H[b] >= 1 && W[b] >= 1, "dt_prep_batch: clip %d has source size %dx%d", b, H[b], W[b]);
    DT_CHECK_ARG(im_scale[b] > 0, "dt_prep_batch: clip %d has im_scale %g <= 0", b, im_scale[b]);
    DT_CHECK_ARG(Hr[b] >= 1 && Wr[b] >= 1 && Hr[b] <= Hp && Wr[b] <= Wp,
                 "dt_prep_batch: clip %d resized size %dx%d does not fit the padded %dx%d", b, Hr[b], Wr[b], Hp, Wp);
    tab.c[b] = PrepBatchClip{frames[b], 1.0 / im_scale[b], H[b], W[b], Hr[b], Wr[b], flip[b] ? 1 : 0};
  }
  DT_CHECK_ARG(!row_planes || (Hp + 2 * border_y) % 2 == 0, "dt_prep_batch: row planes need an even padded height");
  DT_CHECK_ARG(Cp >= 3 && out_f32 >= 0 && out_f32 <= 3 && (out_f32 != 3 || Cp == 8),
               "dt_prep_batch: bad output mode %d with Cp=%d (Cp >= 3; mode 3 needs Cp == 8)", out_f32, Cp);
  const long long total = (long long)B * T * (Hp + 2 * border_y) * (Wp + 2 * border_x);
  const int grid = grid_for(total, 256);
  cudaStream_t s = (cudaStream_t)stream;
  if (out_f32 == 3)
    prep_batch_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(tab, B, T, mean3[0], mean3[1], mean3[2], Hp, Wp, Cp, border_y, border_x, 0,
                                                         row_planes, 1, (__nv_bfloat16*)out);
  else if (out_f32)
    prep_batch_kernel<float><<<grid, 256, 0, s>>>(tab, B, T, mean3[0], mean3[1], mean3[2], Hp, Wp, Cp, border_y, border_x,
                                                 out_f32 == 1, row_planes, 0, (float*)out);
  else
    prep_batch_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(tab, B, T, mean3[0], mean3[1], mean3[2], Hp, Wp, Cp, border_y, border_x, 0,
                                                         row_planes, 0, (__nv_bfloat16*)out);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_maxpool2d(const void* x, int N, int H, int W, int C, int ldx, int k, int s, int p, int f32, int x3,
                            void* y, int ldy, void* stream) {
  const int V = f32 ? 4 : 8;
  DT_CHECK_ARG(N >= 0 && H >= 1 && W >= 1 && C >= 1 && k >= 1 && s >= 1 && p >= 0 && p < k, "dt_maxpool2d: bad shape");
  DT_CHECK_ARG(C % V == 0 && ldx % V == 0 && ldy % V == 0 && ldx >= C && ldy >= C, "dt_maxpool2d: C/ld must be multiples of %d", V);
  DT_CHECK_ARG(!x3 || (ldx >= 2 * C && ldy >= 2 * C), "dt_maxpool2d: x3 storage needs rows of 2*C");
  if (N == 0) return 0;
  DT_CHECK_ARG(x && y, "dt_maxpool2d: null pointer");
  const int Ho = (H + 2 * p - k) / s + 1, Wo = (W + 2 * p - k) / s + 1;      // Caffe2 legacy (floor) pooling
  if (k == 3 && s == 2 && p == 1) {                                           // pool1: rolling-row kernel
    const long long tot = (long long)N * ((Ho + POOL_PR - 1) / POOL_PR) * Wo * (C / V);
    if (f32)
      maxpool3x3s2_kernel<float><<<grid_for(tot, 256), 256, 0, (cudaStream_t)stream>>>((const float*)x, N, H, W, C, ldx, Ho, Wo, (float*)y, ldy,
                                                                                        x3 ? ldx / 2 : 0, x3 ? ldy / 2 : 0);
    else
      maxpool3x3s2_kernel<__nv_bfloat16><<<grid_for(tot, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, N, H, W, C, ldx, Ho, Wo,
                                                                                                (__nv_bfloat16*)y, ldy, x3 ? ldx / 2 : 0, x3 ? ldy / 2 : 0);
    DT_CHECK_LAUNCH();
    return 0;
  }
  const long long total = (long long)N * Ho * Wo * (C / V);
  if (f32)
    maxpool_kernel<float><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const float*)x, N, H, W, C, ldx, k, s, p, Ho, Wo, (float*)y, ldy,
                                                                                   x3 ? ldx / 2 : 0, x3 ? ldy / 2 : 0);
  else
    maxpool_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, N, H, W, C, ldx, k, s, p, Ho, Wo, (__nv_bfloat16*)y, ldy,
                                                                                           x3 ? ldx / 2 : 0, x3 ? ldy / 2 : 0);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_roi_align(const void* const* feats /*host array [nlevels] of device ptrs*/, const int* Hs, const int* Ws,
                            const float* scales /*host arrays*/, int nlevels, int k_min, int C, int ldf, int f32,
                            const float* rois, int ldr, const int* n_dev, int R, int T, const int* levels, int P,
                            int sampling_ratio, int round_tf32, int x3_mode, void* out, void* stream) {
  const int V = f32 ? 4 : 8;
  DT_CHECK_ARG(nlevels >= 1 && nlevels <= 8 && C >= 1 && C % V == 0 && ldf % V == 0 && R >= 0 && T >= 1 && P >= 1 && ldr >= 4 * T + 1,
               "dt_roi_align: bad shape (C=%d must be a multiple of %d)", C, V);
  DT_CHECK_ARG(nlevels == 1 || levels, "dt_roi_align: multi-level pooling needs the per-RoI level array");
  if (R == 0) return 0;
  DT_CHECK_ARG(feats && Hs && Ws && scales && rois && out, "dt_roi_align: null pointer");
  RoiLevels lv;
  for (int l = 0; l < nlevels; ++l) { lv.feat[l] = feats[l]; lv.H[l] = Hs[l]; lv.W[l] = Ws[l]; lv.scale[l] = scales[l]; }
  dim3 grid(R * T, P);
  const int threads = 256;
  // x3_mode 0: plain; 1: [hi | lo] per position (rows of 2C); 2: planar [R][hi block | lo block] (for the FC head)
  DT_CHECK_ARG(x3_mode == 0 || ldf >= 2 * C, "dt_roi_align: x3 storage needs feature rows of 2*C");
  const long long blk = (long long)T * P * P * C;
  const int lo_in = x3_mode ? ldf / 2 : 0;
  const long long o_row = x3_mode ? 2 * blk : blk;
  const int o_pos = (x3_mode == 1) ? 2 * C : C;
  const int o_lo = (x3_mode == 1) ? C : (x3_mode == 2 ? (int)blk : 0);
  if (f32)
    roi_align_kernel<float><<<grid, threads, 0, (cudaStream_t)stream>>>(lv, k_min, rois, ldr, n_dev, R, T, levels, C, ldf, P, sampling_ratio,
                                                                        round_tf32, lo_in, o_row, o_pos, o_lo, (float*)out);
  else
    roi_align_kernel<__nv_bfloat16><<<grid, threads, 0, (cudaStream_t)stream>>>(lv, k_min, rois, ldr, n_dev, R, T, levels, C, ldf, P, sampling_ratio, 0,
                                                                                lo_in, o_row, o_pos, o_lo, (__nv_bfloat16*)out);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_keypoint_decode(const float* lowres, int ldl, int S, int K, int T, const float* boxes, int ldb,
                                  const int* n_dev, int D, int min_size, float* heatmaps, float* xy_preds, void* stream) {
  DT_CHECK_ARG(S >= 1 && S <= 32 && K >= 1 && T >= 1 && T <= DT_MAX_T && D >= 0 && ldl >= 4 * K && ldb >= 4 * T,
               "dt_keypoint_decode: bad shape S=%d K=%d T=%d D=%d ldl=%d ldb=%d", S, K, T, D, ldl, ldb);
  if (D == 0) return 0;
  DT_CHECK_ARG(lowres && boxes && xy_preds, "dt_keypoint_decode: null pointer");
  const size_t smem = (size_t)(4 * S * S + 16 * S * S + 4 * S * KD_SW) * sizeof(float) + (size_t)(KD_SW + KD_RB) * 20;
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(keypoint_decode_kernel, (int)smem, &grant));
  dim3 grid(D, K, T);
  keypoint_decode_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(lowres, ldl, S, K, T, boxes, ldb, n_dev, D, min_size, heatmaps, xy_preds);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_keypoint_decode_aug(const float* lowres, long long view_stride, int ldl, int S, int K, int V, const int* flip,
                                      const int* perm, int hm_max, const float* boxes, int ldb, const int* n_dev, int D,
                                      int min_size, float* heatmaps, float* xy_preds, void* stream) {
  DT_CHECK_ARG(S >= 1 && S <= 32 && K >= 1 && K <= DT_KD_AUG_MAX_K && D >= 0 && ldl >= 4 * K && ldb >= 4,
               "dt_keypoint_decode_aug: bad shape S=%d K=%d D=%d ldl=%d ldb=%d", S, K, D, ldl, ldb);
  DT_CHECK_ARG(V >= 1 && V <= DT_AUG_MAX_VIEWS, "dt_keypoint_decode_aug: V=%d views (1..%d)", V, DT_AUG_MAX_VIEWS);
  DT_CHECK_ARG(view_stride >= (long long)D * S * S * ldl, "dt_keypoint_decode_aug: view_stride %lld < D*S*S*ldl", view_stride);
  DT_CHECK_ARG(hm_max == 0 || hm_max == 1, "dt_keypoint_decode_aug: hm_max must be 0 or 1");
  DT_CHECK_ARG(flip && perm, "dt_keypoint_decode_aug: null flip / perm table");
  KdAugTable tab;
  memset(&tab, 0, sizeof(tab));
  for (int v = 0; v < V; ++v) tab.flip[v] = flip[v] != 0;
  unsigned long long seen = 0;
  for (int k = 0; k < K; ++k) {
    DT_CHECK_ARG(perm[k] >= 0 && perm[k] < K && !(seen >> perm[k] & 1ull), "dt_keypoint_decode_aug: perm is not a permutation of 0..K-1");
    seen |= 1ull << perm[k];
    tab.perm[k] = perm[k];
  }
  if (D == 0) return 0;
  DT_CHECK_ARG(lowres && boxes && xy_preds, "dt_keypoint_decode_aug: null pointer");
  const size_t smem = (size_t)(4 * S * S + 16 * S * S + 4 * S * KD_SW) * sizeof(float) + (size_t)(KD_SW + KD_RB) * 20;
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(keypoint_decode_aug_kernel, (int)smem, &grant));
  dim3 grid(D, K);
  keypoint_decode_aug_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(lowres, view_stride, ldl, S, K, V, tab, hm_max, boxes,
                                                                        ldb, n_dev, D, min_size, heatmaps, xy_preds);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_spatial_mean(const void* x, int N, int H, int W, int C, int ldx, int f32, int round_tf32, int x3, void* y,
                               int ldy, void* stream) {
  const int V = f32 ? 4 : 8;
  DT_CHECK_ARG(N >= 0 && H >= 1 && W >= 1 && C >= 1 && C % V == 0 && ldx % V == 0 && ldy % V == 0 && ldx >= C && ldy >= C,
               "dt_spatial_mean: bad shape (C/ld must be multiples of %d)", V);
  if (N == 0) return 0;
  DT_CHECK_ARG(x && y, "dt_spatial_mean: null pointer");
  const long long total = (long long)N * (C / V);
  if (f32)
    spatial_mean_kernel<float><<<grid_for(total, 128), 128, 0, (cudaStream_t)stream>>>((const float*)x, N, H, W, C, ldx, (float*)y, ldy, round_tf32, x3 ? ldx / 2 : 0, x3 ? ldy / 2 : 0);
  else
    spatial_mean_kernel<__nv_bfloat16><<<grid_for(total, 128), 128, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, N, H, W, C, ldx, (__nv_bfloat16*)y, ldy, 0, x3 ? ldx / 2 : 0, x3 ? ldy / 2 : 0);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_time_mean(const void* x, int B, int T, long long P, int C, int ldx, int f32, int round_tf32, int x3,
                            void* y, int ldy, void* stream) {
  const int V = f32 ? 4 : 8;
  DT_CHECK_ARG(B >= 0 && T >= 1 && P >= 1 && C >= 1 && C % V == 0 && ldx % V == 0 && ldy % V == 0 && ldx >= C && ldy >= C,
               "dt_time_mean: bad shape (C/ld must be multiples of %d)", V);
  DT_CHECK_ARG(!x3 || (ldx >= 2 * C && ldy >= 2 * C), "dt_time_mean: x3 storage needs rows of 2*C");
  if (B == 0) return 0;
  DT_CHECK_ARG(x && y, "dt_time_mean: null pointer");
  const long long total = (long long)B * P * (C / V);
  if (f32)
    time_mean_kernel<float><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const float*)x, B, T, P, C, ldx, (float*)y, ldy, round_tf32, x3 ? ldx / 2 : 0, x3 ? ldy / 2 : 0);
  else
    time_mean_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, B, T, P, C, ldx, (__nv_bfloat16*)y, ldy, 0, x3 ? ldx / 2 : 0, x3 ? ldy / 2 : 0);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_fold_tube_heads(const float* in, int ld, int R, int T, int C, float* cls, float* bbox, void* stream) {
  DT_CHECK_ARG(R >= 0 && T >= 1 && T <= DT_MAX_T && C >= 1 && ld >= 5 * C, "dt_fold_tube_heads: bad shape");
  if (R == 0) return 0;
  DT_CHECK_ARG(in && cls && bbox, "dt_fold_tube_heads: null pointer");
  fold_tube_heads_kernel<<<(R + 127) / 128, 128, 0, (cudaStream_t)stream>>>(in, ld, R, T, C, cls, bbox);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_conv1_7x7s2_f32(const float* blob, int F, int Hp, int Wp, int Cp, const float* w, const float* scale,
                                  const float* bias, int out_bf16, void* y, void* stream) {
  DT_CHECK_ARG(F >= 1 && Hp >= 2 && Wp >= 2 && Hp % 2 == 0 && Wp % 2 == 0 && Cp >= 3, "dt_conv1_7x7s2_f32: bad shape");
  DT_CHECK_ARG(blob && w && scale && bias && y, "dt_conv1_7x7s2_f32: null pointer");
  const long long total = (long long)F * (Hp / 2) * (Wp / 2);
  if (out_bf16)
    conv1_f32_kernel<__nv_bfloat16><<<(unsigned)((total + 31) / 32), 256, 0, (cudaStream_t)stream>>>(blob, F, Hp, Wp, Cp, w, scale, bias, (__nv_bfloat16*)y);
  else
    conv1_f32_kernel<float><<<(unsigned)((total + 31) / 32), 256, 0, (cudaStream_t)stream>>>(blob, F, Hp, Wp, Cp, w, scale, bias, (float*)y);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_pairs_to_f16(const void* pairs, long long rows, int C, void* out, void* stream) {
  DT_CHECK_ARG(rows >= 0 && C >= 8 && C % 8 == 0, "dt_pairs_to_f16: bad shape rows=%lld C=%d (C %% 8 == 0)", rows, C);
  if (rows == 0) return 0;
  DT_CHECK_ARG(pairs && out, "dt_pairs_to_f16: null pointer");
  pairs_to_f16_kernel<<<grid_for(rows * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)pairs, rows, C, (__half*)out);
  DT_CHECK_LAUNCH();
  return 0;
}
