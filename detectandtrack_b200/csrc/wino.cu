// Winograd F(2x2, 3x3) transforms of the bf16x3 keypoint head (pad 1, stride 1, S x S maps with S even, so every map
// is exactly (S/2) x (S/2) tiles of 2 x 2 outputs).  The GEMM between them is dt_wino_gemm (conv_tc.cu).
//
//   V = B^T d B   (d: 4 x 4 input patch, rows / columns 2t - 1 .. 2t + 2, zero outside the map)
//   Y = A^T M A   (M: the 16 products of one tile, Y: its 2 x 2 outputs)
//   B^T = [1 0 -1 0; 0 1 1 0; 0 -1 1 0; 0 1 0 -1]     A^T = [1 1 1 0; 0 1 -1 -1]
// Component xi = 4 i + j is element (i, j) of the 4 x 4 patch.  Tile g = roi * (S/2)^2 + ty * (S/2) + tx.
// Layouts: x / y [D, S, S, 2C] bf16 pairs (hi at channel c, lo at C + c), V [16][G][2C] bf16 pairs, M [16][G][C] fp32.
//
// Every value is rounded the same way whatever D is: sums of +-1 terms in a fixed order as separate fp32 additions (no
// multiply, so nothing to contract), bias, then ReLU as v > 0 ? v : 0, then the pair split hi = bf16(v),
// lo = bf16(v - hi) of the direct convs' epilogue.  A layer's output is rebuilt as hi + lo before its input transform,
// so dt_wino_output_input computes exactly dt_wino_output followed by dt_wino_input.
//
// One CTA per (RoI, 64-channel chunk): lane l holds channels 2l, 2l + 1 (8-byte fp32 / 4-byte bf16-pair accesses, a
// warp covers 256 B of M or 128 B of a pair half), the 8 warps take the tiles round-robin.  The map passes through
// shared memory as fp32 with a one-element zero border, so the input transform reads its patches without bounds tests.
#include "common.cuh"
#include "../../include/dt_b200.h"
#include <cuda_bf16.h>

namespace dt {
namespace {

constexpr int WINO_WARPS = 8;
constexpr int WINO_CH = 64;                // channels per CTA
constexpr int WINO_MAX_S = 16;

__device__ __forceinline__ float2 join_pair(uint32_t hi, uint32_t lo) {
  return make_float2(__fadd_rn(__uint_as_float(hi << 16), __uint_as_float(lo << 16)),
                     __fadd_rn(__uint_as_float(hi & 0xffff0000u), __uint_as_float(lo & 0xffff0000u)));
}

// hi = bf16(v) (RNE), lo = bf16(v - hi); v - hi is exact in fp32
__device__ __forceinline__ void split_pair(float2 v, uint32_t* hi, uint32_t* lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(v.x, v.y);
  const __nv_bfloat162 l = __floats2bfloat162_rn(__fsub_rn(v.x, __low2float(h)), __fsub_rn(v.y, __high2float(h)));
  *hi = *reinterpret_cast<const uint32_t*>(&h);
  *lo = *reinterpret_cast<const uint32_t*>(&l);
}

__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 sub2(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }

// FROM_M: the map comes from M (+ bias, ReLU) instead of x;  TO_Y: the pairs are written to y;  TO_V: V is written.
template <bool FROM_M, bool TO_Y, bool TO_V>
__global__ void __launch_bounds__(WINO_WARPS * 32)
wino_xform_kernel(const uint32_t* __restrict__ x, const float* __restrict__ m, const float* __restrict__ bias, int relu,
                  int S, int C, uint32_t* __restrict__ y, uint32_t* __restrict__ v) {
  extern __shared__ float2 ys[];            // [(S + 2) * (S + 2)][32] fp32 channel pairs, zero border
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int roi = blockIdx.y, c = blockIdx.x * WINO_CH + 2 * lane;
  const int P = S + 2, nt = S / 2, tiles = nt * nt;
  const long long G = (long long)gridDim.y * tiles;
  const int C2 = C / 2;                     // channel pairs of a row half: u32 index of the lo half
  const int cp = c >> 1;                    // u32 index of this thread's pair in a hi half
  if (TO_V) {
    for (int e = warp; e < 4 * (P - 1); e += WINO_WARPS) {     // the border ring, walked once around
      const int side = e / (P - 1), k = e % (P - 1);
      const int r = side == 0 ? 0 : side == 1 ? k : side == 2 ? P - 1 : P - 1 - k;
      const int q = side == 0 ? k : side == 1 ? P - 1 : side == 2 ? P - 1 - k : 0;
      ys[(r * P + q) * 32 + lane] = make_float2(0.f, 0.f);
    }
  }
  if (!FROM_M) {
    for (int pos = warp; pos < S * S; pos += WINO_WARPS) {
      const uint32_t* row = x + ((long long)roi * S * S + pos) * C;          // 2C bf16 = C u32 per position
      const float2 d = join_pair(__ldg(row + cp), __ldg(row + C2 + cp));
      ys[((pos / S + 1) * P + pos % S + 1) * 32 + lane] = d;
    }
  } else {
    float2 b = make_float2(0.f, 0.f);
    if (bias) b = __ldg(reinterpret_cast<const float2*>(bias + c));
    for (int t = warp; t < tiles; t += WINO_WARPS) {
      const long long g = (long long)roi * tiles + t;
      float2 q[16];
#pragma unroll
      for (int xi = 0; xi < 16; ++xi) q[xi] = __ldg(reinterpret_cast<const float2*>(m + ((long long)xi * G + g) * C + c));
      float2 s[2][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[0][j] = add2(add2(q[j], q[4 + j]), q[8 + j]);
        s[1][j] = sub2(sub2(q[4 + j], q[8 + j]), q[12 + j]);
      }
      const int ty = t / nt, tx = t % nt;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          float2 o = k == 0 ? add2(add2(s[i][0], s[i][1]), s[i][2]) : sub2(sub2(s[i][1], s[i][2]), s[i][3]);
          o = add2(o, b);
          if (relu) { o.x = o.x > 0.f ? o.x : 0.f; o.y = o.y > 0.f ? o.y : 0.f; }
          uint32_t hi, lo;
          split_pair(o, &hi, &lo);
          const int r = 2 * ty + i, col = 2 * tx + k;
          if (TO_Y) {
            uint32_t* row = y + ((long long)roi * S * S + r * S + col) * C;
            row[cp] = hi;
            row[C2 + cp] = lo;
          }
          if (TO_V) ys[((r + 1) * P + col + 1) * 32 + lane] = join_pair(hi, lo);
        }
      }
    }
  }
  if (!TO_V) return;
  __syncthreads();
  for (int t = warp; t < tiles; t += WINO_WARPS) {
    const int ty = t / nt, tx = t % nt;
    float2 d[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) d[i][j] = ys[((2 * ty + i) * P + 2 * tx + j) * 32 + lane];
    float2 w[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      w[0][j] = sub2(d[0][j], d[2][j]);
      w[1][j] = add2(d[1][j], d[2][j]);
      w[2][j] = sub2(d[2][j], d[1][j]);
      w[3][j] = sub2(d[1][j], d[3][j]);
    }
    const long long g = (long long)roi * tiles + t;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 e[4] = {sub2(w[i][0], w[i][2]), add2(w[i][1], w[i][2]), sub2(w[i][2], w[i][1]), sub2(w[i][1], w[i][3])};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint32_t hi, lo;
        split_pair(e[j], &hi, &lo);
        uint32_t* row = v + ((long long)(4 * i + j) * G + g) * C;             // 2C bf16 = C u32 per row
        row[cp] = hi;
        row[C2 + cp] = lo;
      }
    }
  }
}

template <bool FROM_M, bool TO_Y, bool TO_V>
int launch_xform(const void* x, const float* m, const float* bias, int relu, int D, int S, int C, void* y, void* v,
                 void* stream) {
  static DynSmemGrant grant;
  const auto k = wino_xform_kernel<FROM_M, TO_Y, TO_V>;
  const int smem = TO_V ? (S + 2) * (S + 2) * 32 * (int)sizeof(float2) : 0;
  DT_CHECK_CUDA(grant_dyn_smem(k, smem, &grant));
  k<<<dim3(C / WINO_CH, D), WINO_WARPS * 32, smem, (cudaStream_t)stream>>>(
      (const uint32_t*)x, m, bias, relu, S, C, (uint32_t*)y, (uint32_t*)v);
  DT_CHECK_LAUNCH();
  return 0;
}

int check_xform(const char* fn, int D, int S, int C) {
  DT_CHECK_ARG(D >= 1 && D <= 65535 && S >= 2 && S <= WINO_MAX_S && S % 2 == 0 && C >= WINO_CH && C % WINO_CH == 0,
               "%s: bad shape D=%d S=%d C=%d (D <= 65535, S even in [2, %d], C %% %d == 0)", fn, D, S, C, WINO_MAX_S,
               WINO_CH);
  return 0;
}

}  // namespace
}  // namespace dt

using namespace dt;

extern "C" int dt_wino_input(const void* x, int D, int S, int C, void* v, void* stream) {
  if (check_xform("dt_wino_input", D, S, C)) return 1;
  DT_CHECK_ARG(x && v && ((uintptr_t)x % 16) == 0 && ((uintptr_t)v % 16) == 0,
               "dt_wino_input: null or unaligned tensor pointer");
  return launch_xform<false, false, true>(x, nullptr, nullptr, 0, D, S, C, nullptr, v, stream);
}

extern "C" int dt_wino_output_input(const float* m, int D, int S, int C, const float* bias, int relu, void* v,
                                    void* stream) {
  if (check_xform("dt_wino_output_input", D, S, C)) return 1;
  DT_CHECK_ARG(m && v && ((uintptr_t)m % 16) == 0 && ((uintptr_t)v % 16) == 0 && ((uintptr_t)bias % 8) == 0,
               "dt_wino_output_input: null or unaligned tensor pointer");
  return launch_xform<true, false, true>(nullptr, m, bias, relu, D, S, C, nullptr, v, stream);
}

extern "C" int dt_wino_output(const float* m, int D, int S, int C, const float* bias, int relu, void* y, void* stream) {
  if (check_xform("dt_wino_output", D, S, C)) return 1;
  DT_CHECK_ARG(m && y && ((uintptr_t)m % 16) == 0 && ((uintptr_t)y % 16) == 0 && ((uintptr_t)bias % 8) == 0,
               "dt_wino_output: null or unaligned tensor pointer");
  return launch_xform<true, true, false>(nullptr, m, bias, relu, D, S, C, y, nullptr, stream);
}
