// Dense Farneback optical flow between key frames, and the flow-smoothed poses of every video
// (lib/core/tracking_engine.py:401-643, TRACKING.FLOW_SMOOTHING_ON).
//
// Farneback restates OpenCV 4.x's CPU calcOpticalFlowFarneback (modules/video/src/optflowgf.cpp) with the
// OPTFLOW_FARNEBACK_GAUSSIAN window, stage by stage, for every pair of a batch at once (oracle/flow.py is the numpy
// statement of the same stages).  The unit is compiled without FMA contraction, so each stage rounds in OpenCV's
// order; every filter tap is built on the host the way OpenCV builds it (fp64 -> fp32) and passed in.
//   per frame and level:  cvtColor BGR2GRAY (once) -> GaussianBlur (reflect-101) -> resize INTER_LINEAR
//                         -> FarnebackPolyExp (5 coefficient channels)
//   per pair and level:   upsample the coarser flow -> FarnebackUpdateMatrices -> `iterations` x
//                         (window blur of M: column pass in shared-memory column tiles, row pass in shared-memory
//                          row tiles fused with the 2x2 solve -> FarnebackUpdateMatrices, except after the last)
// OpenCV updates M in row stripes behind the blur window, which equals the two full phases done here.
//
// dt_flow_mean_abs restates np.abs(flow).mean() (numpy's fp32 pairwise sum), which decides the shot boundaries.
// dt_flow_smooth_poses is bit-exact with _shift_poses + _combine_shifted_poses: one thread per (frame, output track,
// joint) walks the shifts -N..N and chains the |s| flow lookups of each.
#include "common.cuh"
#include "../../include/dt_b200.h"
#include <math.h>
#include <math_constants.h>
#include <vector>

namespace dt {

constexpr int FB_MAX_TAPS = 256;       // pyramid blur taps (ksize <= 255) and window half-taps (m <= 255)
constexpr int FB_MAX_POLY_N = 7;

struct FbTaps {
  float k[FB_MAX_TAPS];
  int n;
};
struct FbPoly {
  float g[FB_MAX_POLY_N + 1], xg[FB_MAX_POLY_N + 1], xxg[FB_MAX_POLY_N + 1];
  double ig11, ig03, ig33, ig55;
  int n;
};

__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  i = i < 0 ? -i : i;
  return i >= n ? 2 * (n - 1) - i : i;
}
__device__ __forceinline__ int clampi(int i, int lo, int hi) { return i < lo ? lo : (i > hi ? hi : i); }

// ------------------------------------------------------------------------------------------------ gray
__global__ void bgr_to_gray_kernel(const uint8_t* __restrict__ bgr, uint8_t* __restrict__ gray, long long npix) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < npix; i += (long long)gridDim.x * blockDim.x) {
    const int b = bgr[3 * i], g = bgr[3 * i + 1], r = bgr[3 * i + 2];
    gray[i] = (uint8_t)((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15);   // OpenCV 4.x's 15-bit coefficients
  }
}

// ------------------------------------------------------------------------------------------------ pyramid
// GaussianBlur row pass: taps in ascending order from k[0]*S[x - r]
__global__ void pyr_blur_rows_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, int N, int H, int W, FbTaps t) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, n = blockIdx.z;
  if (x >= W) return;
  const uint8_t* s = src + ((size_t)n * H + y) * W;
  const int r = t.n / 2;
  float acc = (float)s[reflect101(x - r, W)] * t.k[0];
  for (int i = 1; i < t.n; ++i) acc = acc + (float)s[reflect101(x - r + i, W)] * t.k[i];
  dst[((size_t)n * H + y) * W + x] = acc;
}

// GaussianBlur column pass: symmetric, k[r] * c + k[r+i] * (down + up)
__global__ void pyr_blur_cols_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int H, int W, FbTaps t) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, n = blockIdx.z;
  if (x >= W) return;
  const float* s = src + (size_t)n * H * W + x;
  const int r = t.n / 2;
  float acc = s[(size_t)y * W] * t.k[r];
  for (int i = 1; i <= r; ++i)
    acc = acc + t.k[r + i] * (s[(size_t)reflect101(y + i, H) * W] + s[(size_t)reflect101(y - i, H) * W]);
  dst[((size_t)n * H + y) * W + x] = acc;
}

__device__ __forceinline__ void linear_coeff(int d, int dst, int src, int* s0, float* f) {
  const double scale = 1.0 / ((double)dst / src);
  float fx = (float)((d + 0.5) * scale - 0.5);
  int sx = (int)floorf(fx);
  fx -= (float)sx;
  *s0 = sx;
  *f = fx;
}

// resize INTER_LINEAR of [N, H, W, cn] fp32 to [N, h, w, cn], times `mul`.  Same size: a copy; exactly half in both
// directions: OpenCV's fast INTER_AREA ((a + b) + (c + d)) * 0.25.
__global__ void resize_linear_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int H, int W, int h, int w,
                                     int cn, float mul) {
  const int xc = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, n = blockIdx.z;
  if (xc >= w * cn) return;
  const int x = xc / cn, c = xc % cn;
  const float* S = src + (size_t)n * H * W * cn;
  float v;
  if (w == W && h == H) {
    v = S[((size_t)y * W + x) * cn + c];
  } else if (W == 2 * w && H == 2 * h) {
    const float* p = S + ((size_t)(2 * y) * W + 2 * x) * cn + c;
    v = ((p[0] + p[cn]) + (p[(size_t)W * cn] + p[(size_t)W * cn + cn])) * 0.25f;
  } else {
    int sx, sy;
    float fx, fy;
    linear_coeff(x, w, W, &sx, &fx);
    linear_coeff(y, h, H, &sy, &fy);
    bool hi = false;
    if (sx < 0) { fx = 0.f; sx = 0; }
    if (sx >= W - 1) { fx = 0.f; sx = W - 1; hi = true; }
    const float a0 = 1.f - fx, a1 = fx, b0 = 1.f - fy, b1 = fy;
    const int y0 = clampi(sy, 0, H - 1), y1 = clampi(sy + 1, 0, H - 1), sx1 = min(sx + 1, W - 1);
    const float* r0 = S + (size_t)y0 * W * cn;
    const float* r1 = S + (size_t)y1 * W * cn;
    const float h0 = hi ? r0[sx * cn + c] : r0[sx * cn + c] * a0 + r0[sx1 * cn + c] * a1;
    const float h1 = hi ? r1[sx * cn + c] : r1[sx * cn + c] * a0 + r1[sx1 * cn + c] * a1;
    v = h0 * b0 + h1 * b1;
  }
  dst[(((size_t)n * h + y) * w + x) * cn + c] = v * mul;
}

// FarnebackPolyExp: column pass (fp32) into a shared row tile, row pass in fp64 with OpenCV's fp32 products.
constexpr int PE_TX = 128;
__global__ void __launch_bounds__(PE_TX) poly_exp_kernel(const float* __restrict__ img, float* __restrict__ R, int h, int w, FbPoly p) {
  __shared__ float row[(PE_TX + 2 * FB_MAX_POLY_N) * 3];
  const int y = blockIdx.y, n = blockIdx.z, x0 = blockIdx.x * PE_TX, pn = p.n;
  const float* I = img + (size_t)n * h * w;
  for (int i = threadIdx.x; i < PE_TX + 2 * pn; i += PE_TX) {
    const int x = clampi(x0 - pn + i, 0, w - 1);
    float t0 = I[(size_t)y * w + x] * p.g[0], t1 = 0.f, t2 = 0.f;
    for (int k = 1; k <= pn; ++k) {
      const float s0 = I[(size_t)max(y - k, 0) * w + x], s1 = I[(size_t)min(y + k, h - 1) * w + x];
      const float q = s0 + s1;
      t0 = t0 + p.g[k] * q;
      t1 = t1 + p.xg[k] * (s1 - s0);
      t2 = t2 + p.xxg[k] * q;
    }
    row[i * 3] = t0;
    row[i * 3 + 1] = t1;
    row[i * 3 + 2] = t2;
  }
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= w) return;
  const float* c = row + (threadIdx.x + pn) * 3;
  const float g0 = p.g[0];
  double b1 = (double)(c[0] * g0), b2 = 0, b3 = (double)(c[1] * g0), b4 = 0, b5 = (double)(c[2] * g0), b6 = 0;
  for (int k = 1; k <= pn; ++k) {
    const float* a = c + 3 * k;
    const float* b = c - 3 * k;
    const double tg = (double)(a[0] + b[0]);
    b1 += tg * (double)p.g[k];
    b4 += tg * (double)p.xxg[k];
    b2 += (double)((a[0] - b[0]) * p.xg[k]);
    b3 += (double)((a[1] + b[1]) * p.g[k]);
    b6 += (double)((a[1] - b[1]) * p.xg[k]);
    b5 += (double)((a[2] + b[2]) * p.g[k]);
  }
  float* o = R + (((size_t)n * h + y) * w + x) * 5;
  o[0] = (float)(b3 * p.ig11);
  o[1] = (float)(b2 * p.ig11);
  o[2] = (float)(b1 * p.ig03 + b5 * p.ig33);
  o[3] = (float)(b1 * p.ig03 + b4 * p.ig33);
  o[4] = (float)(b6 * p.ig55);
}

// ------------------------------------------------------------------------------------------------ flow iterations
__device__ __forceinline__ float border_w(int i) {
  return i == 0 || i == 1 ? 0.14f : 0.4472f;
}

// FarnebackUpdateMatrices for every pair: M = (G11, G12, G22, h1, h2) from R0 = R[a], R1 = R[b] sampled at x + flow.
__global__ void update_matrices_kernel(const float* __restrict__ R, const int* __restrict__ pairs, const float* __restrict__ flow,
                                       float* __restrict__ M, int h, int w) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, p = blockIdx.z;
  if (x >= w) return;
  const size_t plane = (size_t)h * w;
  const float* R0 = R + (size_t)pairs[2 * p] * plane * 5 + ((size_t)y * w + x) * 5;
  const float* R1 = R + (size_t)pairs[2 * p + 1] * plane * 5;
  const float* fl = flow + (size_t)p * plane * 2 + ((size_t)y * w + x) * 2;
  const float dx = fl[0], dy = fl[1];
  float fx = (float)x + dx, fy = (float)y + dy;
  const int x1 = (int)floorf(fx), y1 = (int)floorf(fy);
  fx -= (float)x1;
  fy -= (float)y1;
  float r2, r3, r4, r5, r6;
  if ((unsigned)x1 < (unsigned)(w - 1) && (unsigned)y1 < (unsigned)(h - 1)) {
    const float a00 = (1.f - fx) * (1.f - fy), a01 = fx * (1.f - fy), a10 = (1.f - fx) * fy, a11 = fx * fy;
    const float* q = R1 + ((size_t)y1 * w + x1) * 5;
    const size_t st = (size_t)w * 5;
    float r[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) r[c] = a00 * q[c] + a01 * q[5 + c] + a10 * q[st + c] + a11 * q[st + 5 + c];
    r2 = r[0];
    r3 = r[1];
    r4 = (R0[2] + r[2]) * 0.5f;
    r5 = (R0[3] + r[3]) * 0.5f;
    r6 = (R0[4] + r[4]) * 0.25f;
  } else {
    r2 = r3 = 0.f;
    r4 = R0[2];
    r5 = R0[3];
    r6 = R0[4] * 0.5f;
  }
  r2 = (R0[0] - r2) * 0.5f;
  r3 = (R0[1] - r3) * 0.5f;
  r2 += r4 * dy + r6 * dx;
  r3 += r6 * dy + r5 * dx;
  if ((unsigned)(x - 5) >= (unsigned)(w - 10) || (unsigned)(y - 5) >= (unsigned)(h - 10)) {
    const float s = (x < 5 ? border_w(x) : 1.f) * (x >= w - 5 ? border_w(w - x - 1) : 1.f) * (y < 5 ? border_w(y) : 1.f) *
                    (y >= h - 5 ? border_w(h - y - 1) : 1.f);
    r2 *= s; r3 *= s; r4 *= s; r5 *= s; r6 *= s;
  }
  float* o = M + (size_t)p * plane * 5 + ((size_t)y * w + x) * 5;
  o[0] = r4 * r4 + r6 * r6;
  o[1] = (r4 + r5) * r6;
  o[2] = r5 * r5 + r6 * r6;
  o[3] = r4 * r2 + r6 * r3;
  o[4] = r6 * r2 + r5 * r3;
}

// Window blur, column pass: a CTA owns 32 pixels x 5 channels and VB_TY output rows; the (VB_TY + 2m) input rows it
// needs (clamped) sit in shared memory.
constexpr int VB_COLS = 32 * 5;
constexpr int VB_RY = 4;
__global__ void __launch_bounds__(VB_COLS * VB_RY) window_blur_cols_kernel(const float* __restrict__ M, float* __restrict__ V, int h,
                                                                           int w, int ty, FbTaps t) {
  extern __shared__ float tile[];
  const int m = t.n, y0 = blockIdx.y * ty, p = blockIdx.z, c0 = blockIdx.x * VB_COLS;
  const int rows = ty + 2 * m, ncol = min(VB_COLS, w * 5 - c0);
  const float* src = M + (size_t)p * h * w * 5 + c0;
  const int tid = threadIdx.y * VB_COLS + threadIdx.x;
  for (int i = tid; i < rows * VB_COLS; i += VB_COLS * VB_RY) {
    const int r = i / VB_COLS, c = i % VB_COLS;
    if (c < ncol) tile[i] = src[(size_t)clampi(y0 - m + r, 0, h - 1) * w * 5 + c];
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= ncol) return;
  float* dst = V + (size_t)p * h * w * 5 + c0 + c;
  for (int r = threadIdx.y; r < ty && y0 + r < h; r += VB_RY) {
    const float* q = tile + (r + m) * VB_COLS + c;
    float s = q[0] * t.k[0];
    for (int i = 1; i <= m; ++i) s = s + (q[i * VB_COLS] + q[-i * VB_COLS]) * t.k[i];
    dst[(size_t)(y0 + r) * w * 5] = s;
  }
}

// Window blur, row pass (a shared row tile of HB_TX pixels plus the clamped halo) fused with the solve
// flow = ((g11 h2 - g12 h1), (g22 h1 - g12 h2)) / (g11 g22 - g12^2 + 1e-3) in fp64.
constexpr int HB_TX = 128;
__global__ void __launch_bounds__(HB_TX) window_blur_rows_solve_kernel(const float* __restrict__ V, float* __restrict__ flow, int h,
                                                                       int w, FbTaps t) {
  extern __shared__ float rowt[];
  const int m = t.n, y = blockIdx.y, p = blockIdx.z, x0 = blockIdx.x * HB_TX;
  const float* src = V + ((size_t)p * h + y) * w * 5;
  for (int i = threadIdx.x; i < (HB_TX + 2 * m) * 5; i += HB_TX) {
    const int px = clampi(x0 - m + i / 5, 0, w - 1);
    rowt[i] = src[px * 5 + i % 5];
  }
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= w) return;
  const float* q = rowt + (threadIdx.x + m) * 5;
  double g[5];
#pragma unroll
  for (int c = 0; c < 5; ++c) {
    float s = q[c] * t.k[0];
    for (int i = 1; i <= m; ++i) s = s + t.k[i] * (q[c - 5 * i] + q[c + 5 * i]);
    g[c] = (double)s;
  }
  const double idet = 1.0 / (g[0] * g[2] - g[1] * g[1] + 1e-3);
  float* o = flow + (((size_t)p * h + y) * w + x) * 2;
  o[0] = (float)((g[0] * g[4] - g[1] * g[3]) * idet);
  o[1] = (float)((g[2] * g[3] - g[1] * g[4]) * idet);
}

// ------------------------------------------------------------------------------------------------ np.abs(flow).mean()
// numpy's pairwise_sum for fp32: < 8 elements sequential; <= 128: 8 accumulators then ((r0+r1)+(r2+r3))+((r4+r5)+
// (r6+r7)) and the rest sequential; else split at n/2 rounded down to a multiple of 8.
__device__ float pairwise_abs_sum(const float* a, long long n) {
  if (n < 8) {
    float r = 0.f;
    for (long long i = 0; i < n; ++i) r += fabsf(a[i]);
    return r;
  }
  if (n <= 128) {
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = fabsf(a[j]);
    long long i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] += fabsf(a[i + j]);
    float res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += fabsf(a[i]);
    return res;
  }
  long long n2 = n / 2;
  n2 -= n2 % 8;
  return pairwise_abs_sum(a, n2) + pairwise_abs_sum(a + n2, n - n2);
}

constexpr int MA_THREADS = 1024;
// One CTA per flow.  Every node above depth `depth` of numpy's split tree has more than 128 elements, so each splits
// in two: thread i sums node i of that depth, and the CTA adds the nodes back up the tree.
__global__ void __launch_bounds__(MA_THREADS) flow_mean_abs_kernel(const float* __restrict__ flows, long long n, int depth,
                                                                   float* __restrict__ out) {
  __shared__ float part[MA_THREADS];
  const float* a = flows + (size_t)blockIdx.x * n;
  const int nodes = 1 << depth;
  if ((int)threadIdx.x < nodes) {
    long long off = 0, len = n;
    for (int d = depth - 1; d >= 0; --d) {
      long long n2 = len / 2;
      n2 -= n2 % 8;
      if ((threadIdx.x >> d) & 1) { off += n2; len -= n2; } else { len = n2; }
    }
    part[threadIdx.x] = pairwise_abs_sum(a + off, len);
  }
  __syncthreads();
  for (int k = nodes / 2; k >= 1; k /= 2) {
    float v = 0.f;
    if ((int)threadIdx.x < k) v = part[2 * threadIdx.x] + part[2 * threadIdx.x + 1];
    __syncthreads();
    if ((int)threadIdx.x < k) part[threadIdx.x] = v;
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = (0.f + part[0]) / (float)n;
}

// ------------------------------------------------------------------------------------------------ smoothing
constexpr int SM_MAX_CONTEXT = DT_FLOW_MAX_CONTEXT;
struct SmWeights {
  float wt[SM_MAX_CONTEXT + 1];        // (float)pow(1.2, -|s|)
};

// numpy's scalar minimum / maximum (the first operand wins ties; NaN propagates)
__device__ __forceinline__ float np_min(float a, float b) { return (a <= b || isnan(a)) ? a : b; }
__device__ __forceinline__ float np_max(float a, float b) { return (a >= b || isnan(a)) ? a : b; }

__global__ void flow_smooth_kernel(const float* __restrict__ poses, const float* __restrict__ boxes, const int* __restrict__ counts,
                                   const int* __restrict__ tracks, const unsigned char* __restrict__ is_start, int F, int dmax, int K,
                                   const float* const* __restrict__ flows, const int* __restrict__ flow_hw,
                                   const unsigned char* __restrict__ no_flow, int N, SmWeights wts,
                                   const int* __restrict__ out_tracks, const int* __restrict__ out_counts, int omax,
                                   float* __restrict__ out_poses, float* __restrict__ out_boxes) {
  const int j = threadIdx.x, o = blockIdx.x, f = blockIdx.y;       // joint j == K: the box
  if (o >= out_counts[f] || j > K) return;
  const int tid = out_tracks[f * omax + o];
  float fx = -CUDART_INF_F, fy = -CUDART_INF_F, fv = -CUDART_INF_F, f3 = -CUDART_INF_F;
  float bx[5];
  bool have_box = false;
  for (int s = -N; s <= N; ++s) {
    const int g = f - s;
    if (g < 0 || g >= F || counts[g] == 0) continue;
    // the chain from frame g to frame f stays inside one video and crosses no missing or shot-boundary flow
    const int lo = min(g, f), hi = max(g, f);
    bool ok = true;
    for (int q = lo; q < hi; ++q) ok = ok && !is_start[q + 1] && !no_flow[q];
    if (!ok) continue;
    int r = -1;
    for (int i = 0; i < counts[g]; ++i)
      if (tracks[(size_t)g * dmax + i] == tid) { r = i; break; }
    if (r < 0) continue;
    if (j == K) {
      const float* b = boxes + ((size_t)g * dmax + r) * 5;
      if (!have_box) {
        for (int c = 0; c < 5; ++c) bx[c] = b[c];
        have_box = true;
      } else {
        bx[0] = np_min(bx[0], b[0]);
        bx[1] = np_min(bx[1], b[1]);
        bx[2] = np_max(bx[2], b[2]);
        bx[3] = np_max(bx[3], b[3]);
        bx[4] = np_max(bx[4], b[4]);
      }
      continue;
    }
    const float* pp = poses + ((size_t)g * dmax + r) * 4 * K + j;
    float x = pp[0], y = pp[K], v = pp[2 * K];
    const float w3 = pp[3 * K];
    const int steps = s < 0 ? -s : s;
    for (int k = 0; k < steps; ++k) {
      const int q = s > 0 ? g + k : g - 1 - k;        // forward: flow q -> q+1; backward: -(flow q -> q+1) at frame q+1
      const int H = flow_hw[2 * q], W = flow_hw[2 * q + 1];
      const float rx = rintf(x), ry = rintf(y);
      float dx = 0.f, dy = 0.f;
      if (rx >= 0.f && rx < (float)W && ry >= 0.f && ry < (float)H) {
        const float* d = flows[q] + ((size_t)ry * W + (size_t)rx) * 2;
        dx = s > 0 ? d[0] : -d[0];
        dy = s > 0 ? d[1] : -d[1];
      } else {
        v = 0.f;
      }
      x = __fadd_rn(x, dx);
      y = __fadd_rn(y, dy);
    }
    const float c = __fmul_rn(v, wts.wt[steps]);
    if (c > fv) { fx = x; fy = y; f3 = w3; fv = c; }
  }
  if (j == K) {
    float* ob = out_boxes + ((size_t)f * omax + o) * 5;
    for (int c = 0; c < 5; ++c) ob[c] = bx[c];
  } else {
    float* op = out_poses + ((size_t)f * omax + o) * 4 * K + j;
    op[0] = fx;
    op[K] = fy;
    op[2 * K] = fv;
    op[3 * K] = f3;
  }
}

// ------------------------------------------------------------------------------------------------ host
static void gaussian_taps_host(int ksize, double sigma, FbTaps* t) {
  static const float fixed3[] = {0.25f, 0.5f, 0.25f}, fixed5[] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f},
                     fixed7[] = {0.03125f, 0.109375f, 0.21875f, 0.28125f, 0.21875f, 0.109375f, 0.03125f};
  const float* fx = sigma > 0 ? nullptr : ksize == 3 ? fixed3 : ksize == 5 ? fixed5 : ksize == 7 ? fixed7 : nullptr;
  const double sx = sigma > 0 ? sigma : ((ksize - 1) * 0.5 - 1) * 0.3 + 0.8;
  const double s2 = -0.5 / (sx * sx);
  double sum = 0;
  for (int i = 0; i < ksize; ++i) {
    const double x = i - (ksize - 1) * 0.5;
    t->k[i] = fx ? fx[i] : (float)exp(s2 * x * x);
    sum += t->k[i];
  }
  sum = 1.0 / sum;
  for (int i = 0; i < ksize; ++i) t->k[i] = (float)(t->k[i] * sum);
  t->n = ksize;
}

static bool poly_taps_host(int n, double sigma, FbPoly* p) {
  if (sigma < 1.1920928955078125e-07) sigma = n * 0.3;
  float g[2 * FB_MAX_POLY_N + 1];
  double s = 0;
  for (int x = -n; x <= n; ++x) {
    g[x + n] = (float)exp(-x * x / (2 * sigma * sigma));
    s += g[x + n];
  }
  s = 1.0 / s;
  for (int x = -n; x <= n; ++x) g[x + n] = (float)(g[x + n] * s);
  for (int k = 0; k <= n; ++k) {
    p->g[k] = g[k + n];
    p->xg[k] = (float)((double)k * g[k + n]);
    p->xxg[k] = (float)((double)k * k * g[k + n]);
  }
  double G[6][6] = {};
  for (int y = -n; y <= n; ++y)
    for (int x = -n; x <= n; ++x) {
      const double gg = (double)g[y + n] * g[x + n];
      G[0][0] += gg;
      G[1][1] += gg * x * x;
      G[3][3] += gg * x * x * x * x;
      G[5][5] += gg * x * x * y * y;
    }
  G[2][2] = G[0][3] = G[0][4] = G[3][0] = G[4][0] = G[1][1];
  G[4][4] = G[3][3];
  G[3][4] = G[4][3] = G[5][5];
  // G^-1 by Gauss-Jordan (G is symmetric positive definite)
  double A[6][12];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 12; ++j) A[i][j] = j < 6 ? G[i][j] : (j - 6 == i ? 1.0 : 0.0);
  for (int c = 0; c < 6; ++c) {
    int piv = c;
    for (int r = c + 1; r < 6; ++r)
      if (fabs(A[r][c]) > fabs(A[piv][c])) piv = r;
    if (A[piv][c] == 0) return false;
    for (int j = 0; j < 12; ++j) { double tmp = A[c][j]; A[c][j] = A[piv][j]; A[piv][j] = tmp; }
    const double d = A[c][c];
    for (int j = 0; j < 12; ++j) A[c][j] /= d;
    for (int r = 0; r < 6; ++r)
      if (r != c) {
        const double f = A[r][c];
        for (int j = 0; j < 12; ++j) A[r][j] -= f * A[c][j];
      }
  }
  p->ig11 = A[1][6 + 1];
  p->ig03 = A[0][6 + 3];
  p->ig33 = A[3][6 + 3];
  p->ig55 = A[5][6 + 5];
  p->n = n;
  return true;
}

static void window_taps_host(int winsize, FbTaps* t) {
  const int m = winsize / 2;
  const double sigma = m * 0.3;
  double s = 1;
  t->k[0] = 1.f;
  for (int i = 1; i <= m; ++i) {
    t->k[i] = (float)exp(-i * i / (2 * sigma * sigma));
    s += t->k[i] * 2;
  }
  s = 1.0 / s;
  for (int i = 0; i <= m; ++i) t->k[i] = (float)(t->k[i] * s);
  t->n = m;
}

struct FbLevel {
  int w, h, ksize;
  double sigma;
};

// the pyramid of calcOpticalFlowFarneback, coarse to fine
static std::vector<FbLevel> fb_levels(int H, int W, double pyr_scale, int levels) {
  const int min_size = 32;
  double scale = 1;
  int k = 0;
  for (; k < levels; ++k) {
    scale *= pyr_scale;
    if (W * scale < min_size || H * scale < min_size) break;
  }
  std::vector<FbLevel> out;
  for (int lv = k; lv >= 0; --lv) {
    double s = 1;
    for (int i = 0; i < lv; ++i) s *= pyr_scale;
    const double sigma = (1. / s - 1) * 0.5;
    int ks = ((int)lrint(sigma * 5)) | 1;
    ks = ks < 3 ? 3 : ks;
    out.push_back({(int)lrint(W * s), (int)lrint(H * s), ks, sigma});
  }
  return out;
}

// rows of the column-pass tile that fit the shared memory with a window half-width m (0: none)
static int window_tile_rows(int m) {
  for (int ty = 64; ty >= 8; ty /= 2)
    if ((size_t)(ty + 2 * m) * VB_COLS * sizeof(float) <= 227 * 1024) return ty;
  return 0;
}

struct FbWorkspace {
  uint8_t* gray;
  float *blur0, *blur1, *R, *M, *V, *flowA, *flowB;
  size_t bytes;
};

static FbWorkspace fb_carve(void* base, int H, int W, int nframes, int npairs) {
  FbWorkspace w;
  const size_t hw = (size_t)H * W;
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t n) { char* p = b ? b + off : nullptr; off += align_up(n, 256); return p; };
  w.gray = (uint8_t*)take(hw * nframes);
  w.blur0 = (float*)take(hw * nframes * 4);
  w.blur1 = (float*)take(hw * nframes * 4);
  w.R = (float*)take(hw * nframes * 20);
  w.M = (float*)take(hw * npairs * 20);
  w.V = (float*)take(hw * npairs * 20);
  w.flowA = (float*)take(hw * npairs * 8);
  w.flowB = (float*)take(hw * npairs * 8);
  w.bytes = off;
  return w;
}

}  // namespace dt

using namespace dt;

extern "C" int dt_bgr_to_gray(const uint8_t* bgr, long long npix, uint8_t* gray, void* stream) {
  DT_CHECK_ARG(npix >= 0, "dt_bgr_to_gray: npix=%lld < 0", npix);
  if (npix == 0) return 0;
  DT_CHECK_ARG(bgr && gray, "dt_bgr_to_gray: null pointer");
  const int grid = (int)std::min<long long>((npix + 255) / 256, 65535LL * 8);
  bgr_to_gray_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(bgr, gray, npix);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_farneback_workspace_bytes(int H, int W, int nframes, int npairs, size_t* bytes) {
  DT_CHECK_ARG(H >= 1 && W >= 1 && nframes >= 0 && npairs >= 0 && bytes,
               "dt_farneback_workspace_bytes: bad args H=%d W=%d nframes=%d npairs=%d", H, W, nframes, npairs);
  *bytes = fb_carve(nullptr, H, W, nframes, npairs).bytes;
  return 0;
}

extern "C" int dt_farneback_flow(const uint8_t* frames, int nframes, int H, int W, const int* pairs, int npairs, double pyr_scale,
                                 int levels, int winsize, int iterations, int poly_n, double poly_sigma, int flags, float* flows,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  DT_CHECK_ARG(H >= 1 && W >= 1 && nframes >= 1 && npairs >= 0,
               "dt_farneback_flow: bad shape nframes=%d H=%d W=%d npairs=%d", nframes, H, W, npairs);
  DT_CHECK_ARG(pyr_scale > 0 && pyr_scale < 1 && levels >= 0 && iterations >= 1,
               "dt_farneback_flow: pyr_scale=%g levels=%d iterations=%d (need 0 < pyr_scale < 1, levels >= 0, iterations >= 1)",
               pyr_scale, levels, iterations);
  DT_CHECK_ARG(poly_n == 5 || poly_n == 7, "dt_farneback_flow: poly_n=%d is not 5 or 7", poly_n);
  DT_CHECK_ARG(flags == DT_FARNEBACK_GAUSSIAN,
               "dt_farneback_flow: flags=%d; only OPTFLOW_FARNEBACK_GAUSSIAN (%d) is implemented", flags, DT_FARNEBACK_GAUSSIAN);
  DT_CHECK_ARG(winsize >= 1 && winsize / 2 < FB_MAX_TAPS && window_tile_rows(winsize / 2) > 0,
               "dt_farneback_flow: winsize=%d outside [1, %d]", winsize, 2 * 173 + 1);
  if (npairs == 0) return 0;
  DT_CHECK_ARG(frames && pairs && flows && workspace, "dt_farneback_flow: null pointer");
  const FbWorkspace ws = fb_carve(workspace, H, W, nframes, npairs);
  DT_CHECK_ARG(workspace_bytes >= ws.bytes, "dt_farneback_flow: workspace %zu < %zu bytes", workspace_bytes, ws.bytes);
  const std::vector<FbLevel> lv = fb_levels(H, W, pyr_scale, levels);
  for (const FbLevel& l : lv)
    DT_CHECK_ARG(l.ksize < FB_MAX_TAPS, "dt_farneback_flow: pyramid blur of %d taps exceeds %d (too many levels for %dx%d)",
                 l.ksize, FB_MAX_TAPS - 1, W, H);
  FbPoly poly;
  DT_CHECK_ARG(poly_taps_host(poly_n, poly_sigma, &poly), "dt_farneback_flow: singular polynomial basis");
  FbTaps win;
  window_taps_host(winsize, &win);
  const int ty = window_tile_rows(win.n);
  static DynSmemGrant grant;
  const int vb_smem = (ty + 2 * win.n) * VB_COLS * (int)sizeof(float);
  DT_CHECK_CUDA(grant_dyn_smem(window_blur_cols_kernel, vb_smem, &grant));
  cudaStream_t st = (cudaStream_t)stream;

  if (dt_bgr_to_gray(frames, (long long)nframes * H * W, ws.gray, stream)) return 2;
  const float* prev = nullptr;
  int pw = 0, ph = 0;
  for (size_t li = 0; li < lv.size(); ++li) {
    const FbLevel& l = lv[li];
    const bool finest = li + 1 == lv.size();
    FbTaps gt;
    gaussian_taps_host(l.ksize, l.sigma, &gt);
    pyr_blur_rows_kernel<<<dim3(cdiv(W, 128), H, nframes), 128, 0, st>>>(ws.gray, ws.blur0, nframes, H, W, gt);
    DT_CHECK_LAUNCH();
    pyr_blur_cols_kernel<<<dim3(cdiv(W, 128), H, nframes), 128, 0, st>>>(ws.blur0, ws.blur1, nframes, H, W, gt);
    DT_CHECK_LAUNCH();
    const float* I = ws.blur1;
    if (l.w != W || l.h != H) {
      resize_linear_kernel<<<dim3(cdiv(l.w, 128), l.h, nframes), 128, 0, st>>>(ws.blur1, ws.blur0, nframes, H, W, l.h, l.w, 1, 1.f);
      DT_CHECK_LAUNCH();
      I = ws.blur0;
    }
    poly_exp_kernel<<<dim3(cdiv(l.w, PE_TX), l.h, nframes), PE_TX, 0, st>>>(I, ws.R, l.h, l.w, poly);
    DT_CHECK_LAUNCH();
    float* cur = finest ? flows : (prev == ws.flowA ? ws.flowB : ws.flowA);
    if (!prev) {
      DT_CHECK_CUDA(cudaMemsetAsync(cur, 0, (size_t)npairs * l.h * l.w * 2 * sizeof(float), st));
    } else {
      resize_linear_kernel<<<dim3(cdiv(l.w * 2, 128), l.h, npairs), 128, 0, st>>>(prev, cur, npairs, ph, pw, l.h, l.w, 2,
                                                                                   (float)(1. / pyr_scale));
      DT_CHECK_LAUNCH();
    }
    const dim3 pix(cdiv(l.w, 128), l.h, npairs);
    update_matrices_kernel<<<pix, 128, 0, st>>>(ws.R, pairs, cur, ws.M, l.h, l.w);
    DT_CHECK_LAUNCH();
    for (int it = 0; it < iterations; ++it) {
      window_blur_cols_kernel<<<dim3(cdiv(l.w * 5, VB_COLS), cdiv(l.h, ty), npairs), dim3(VB_COLS, VB_RY), vb_smem, st>>>(
          ws.M, ws.V, l.h, l.w, ty, win);
      DT_CHECK_LAUNCH();
      window_blur_rows_solve_kernel<<<dim3(cdiv(l.w, HB_TX), l.h, npairs), HB_TX, (HB_TX + 2 * win.n) * 5 * sizeof(float), st>>>(
          ws.V, cur, l.h, l.w, win);
      DT_CHECK_LAUNCH();
      if (it < iterations - 1) {
        update_matrices_kernel<<<pix, 128, 0, st>>>(ws.R, pairs, cur, ws.M, l.h, l.w);
        DT_CHECK_LAUNCH();
      }
    }
    prev = cur;
    pw = l.w;
    ph = l.h;
  }
  return 0;
}

extern "C" int dt_flow_mean_abs(const float* flows, int npairs, int H, int W, float* out, void* stream) {
  DT_CHECK_ARG(npairs >= 0 && H >= 1 && W >= 1, "dt_flow_mean_abs: bad shape npairs=%d H=%d W=%d", npairs, H, W);
  if (npairs == 0) return 0;
  DT_CHECK_ARG(flows && out, "dt_flow_mean_abs: null pointer");
  const long long n = 2LL * H * W;
  DT_CHECK_ARG(n <= (1LL << 24), "dt_flow_mean_abs: %lld values exceed fp32's exact integers", n);
  int depth = 0;
  for (long long len = n; depth < 10 && len > 128; ++depth) {
    len /= 2;
    len -= len % 8;
  }
  flow_mean_abs_kernel<<<npairs, MA_THREADS, 0, (cudaStream_t)stream>>>(flows, n, depth, out);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_flow_smooth_poses(const float* poses, const float* boxes, const int* counts, const int* tracks,
                                    const unsigned char* is_start, int F, int dmax, int K, const float* const* flows,
                                    const int* flow_hw, const unsigned char* no_flow, int n_context, const int* out_tracks,
                                    const int* out_counts, int omax, float* out_poses, float* out_boxes, void* stream) {
  DT_CHECK_ARG(F >= 0 && dmax >= 1 && K >= 1 && K < 1024 && omax >= 1,
               "dt_flow_smooth_poses: bad shape F=%d dmax=%d K=%d omax=%d", F, dmax, K, omax);
  DT_CHECK_ARG(n_context >= 0 && n_context <= SM_MAX_CONTEXT, "dt_flow_smooth_poses: n_context=%d outside [0, %d]", n_context,
               SM_MAX_CONTEXT);
  DT_CHECK_ARG(omax <= 65535 * 16, "dt_flow_smooth_poses: omax=%d too large", omax);
  if (F == 0) return 0;
  DT_CHECK_ARG(poses && boxes && counts && tracks && is_start && out_tracks && out_counts && out_poses && out_boxes,
               "dt_flow_smooth_poses: null pointer");
  DT_CHECK_ARG(n_context == 0 || (flows && flow_hw && no_flow), "dt_flow_smooth_poses: n_context=%d needs the flows", n_context);
  DT_CHECK_ARG(F <= 65535, "dt_flow_smooth_poses: F=%d exceeds 65535 frames per call", F);
  SmWeights w;
  for (int s = 0; s <= SM_MAX_CONTEXT; ++s) w.wt[s] = (float)pow(1.2, -s);
  flow_smooth_kernel<<<dim3(omax, F), K + 1, 0, (cudaStream_t)stream>>>(poses, boxes, counts, tracks, is_start, F, dmax, K, flows,
                                                                       flow_hw, no_flow, n_context, w, out_tracks, out_counts, omax,
                                                                       out_poses, out_boxes);
  DT_CHECK_LAUNCH();
  return 0;
}
