// Training-step kernels of the data-parallel path (BASELINE.json configs[4]; the reference builds these with
// model.AddGradientOperators + add_parameter_update_ops, lib/modeling/model_builder.py:908-985):
//
//   dt_wgrad_nhwc       Conv / ConvNd / FC filter gradient on the tensor cores (wgmma):
//                         dW[tap][co][ci] = sum over positions of gz[pos, co] * x[pos @ tap, ci]
//                       a GEMM whose K axis is the position axis, both operands read straight from the NDHWC tensors by
//                       5-D TMA boxes of 64 positions (MN-major wgmma operands; the tap is a coordinate shift of the input
//                       box, TMA's zero fill the padding).  Split-K over positions across CTAs, fp32 partial sums reduced
//                       into dW with vector red.global.
//   dt_bwd_pointwise    the elementwise part of a block's backward: gz = (g1 + g2) * [y > 0] * scale[c]
//                       (Relu / Sum / AffineChannelNd gradients, lib/ops/affine_channel_nd_op.cu:73-92: dX = dY * scale;
//                       the affine parameters themselves are frozen in Detectron-style fine-tuning)
//   dt_upsample_add_bwd FPN top-down join backward (lib/modeling/FPN3D.py:186-222): the coarser level receives the 2x2 sum
//   dt_scatter_stride2  dgrad of a stride-2 pointwise conv: values land on the even positions of a zeroed map
//   dt_sgd_update_multi MomentumSGDUpdate with weight decay (model_builder.py:954-985) of every parameter tensor in one
//                       launch, on fp32 master weights kept in the packed [tap][Cout][Cin] order, re-emitting the bf16
//                       forward weights and the (flipped, transposed) bf16 dgrad weights in the same pass
#include "common.cuh"
#include "tc_common.cuh"
#include "../../include/dt_b200.h"
#include <cuda_bf16.h>

namespace dt {

using namespace tc;

// ------------------------------------------------------------------------------------------------ wgrad
// The GEMM read STRAIGHT from the NDHWC tensors: a TMA box (64 channels = 128 B, TW, TH, TT, TB) of 64 positions lands in
// shared memory as 64 rows of 128 bytes — positions down the rows, 64 channels along each swizzled row.  Read as an
// MN-MAJOR wgmma operand (the transpose flags of the instruction) with K = the position axis: 8 positions x 128 B per
// swizzle atom, 1024 B between 8-position groups.  The filter tap is a coordinate shift of the input box (TMA zero fill =
// the conv's padding), exactly as in the forward kernel.
constexpr int WG_THREADS = 384;       // warp 0 TMA producer (warps 1-3 idle), warps 4-11 two consumer warpgroups
constexpr int WG_CONSUMER_WARPS = 8;
constexpr int WG_STAGES = 4;

// Consumers: warpgroup g accumulates rows (output channels) 64g .. 64g+63 of the 128-row tile in registers (fragment
// layout: wgmma.cuh) and adds them into dW with red.global.  Cin is even, so a thread's column pair is either wholly
// inside the filter or wholly outside.
template <int NB>
__device__ __forceinline__ void wgrad_red(const float (&acc)[NB], float* dW, int Cout, int Cin, int tap, int row_base, int col_base) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < NB / 4; ++j) {
    const int col = col_base + 8 * j + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = row_base + ((warp - 4) >> 2) * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
      if (row < Cout && col < Cin)
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dW + ((size_t)tap * Cout + row) * Cin + col),
                     "f"(acc[4 * j + 2 * i]), "f"(acc[4 * j + 2 * i + 1]) : "memory");
    }
  }
}

struct WgradNParams {
  int Cout, Cin, taps;
  int kT, kH, kW, pT, pH, pW;
  int TW, TH, TT, TB;
  int nW, nH, nT, nN;       // position tiles per axis
  int T;                    // frames (temporal bounds of the tap shift when TT == 1)
  int tiles_m, tiles_n, ksplit;
  float* dW;
};

template <int BN>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_nhwc_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmX, const WgradNParams p) {
  constexpr int GRP = 64 * 128;                                    // one (64 positions x 64 channels) box
  constexpr int A_BYTES = 2 * GRP, B_BYTES = (BN / 64) * GRP, ST_BYTES = A_BYTES + B_BYTES;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + WG_STAGES * ST_BYTES);
  uint64_t* empty = full + WG_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();
    prefetch_tmap(&tmG); prefetch_tmap(&tmX);
    for (int s = 0; s < WG_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], WG_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  int w = blockIdx.x;
  const int ks = w % p.ksplit; w /= p.ksplit;
  const int nt = w % p.tiles_n; w /= p.tiles_n;
  const int mt = w % p.tiles_m;
  const int tap = w / p.tiles_m;
  const int kw = tap % p.kW, kh = (tap / p.kW) % p.kH, kt = tap / (p.kW * p.kH);
  const int dw = kw - p.pW, dh = kh - p.pH, dt_ = kt - p.pT;
  const long long total = (long long)p.nN * p.nT * p.nH * p.nW;
  const long long k0 = total * ks / p.ksplit, k1 = total * (ks + 1) / p.ksplit;
  // a k-block whose tap-shifted frames all lie outside the clip contributes zero: skipped by producer and consumers alike
  auto live = [&](int it) -> bool { const int t0 = it * p.TT + dt_; return t0 + p.TT > 0 && t0 < p.T; };
  auto decode = [&](long long kb, int& iw, int& ih, int& it, int& in) {
    iw = (int)(kb % p.nW); kb /= p.nW;
    ih = (int)(kb % p.nH); kb /= p.nH;
    it = (int)(kb % p.nT); in = (int)(kb / p.nT);
  };

  if (warp == 0) {
    int stage = 0; uint32_t phase = 0;
    int iw, ih, it, in;
    decode(k0, iw, ih, it, in);
    for (long long kb = k0; kb < k1; ++kb) {
      if (live(it)) {
        mbar_wait(&empty[stage], phase ^ 1);
        if (elect_one()) {
          const uint32_t dst = smem_u32(smem) + stage * ST_BYTES;
          const uint32_t bar = smem_u32(&full[stage]);
          mbar_expect_tx_u(bar, (uint32_t)ST_BYTES);
          const int w0 = iw * p.TW, h0 = ih * p.TH, t0 = it * p.TT, n0 = in * p.TB;
#pragma unroll
          for (int g = 0; g < 2; ++g)
            asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
                         ::"r"(dst + g * GRP), "l"(reinterpret_cast<uint64_t>(&tmG)), "r"(bar), "r"(mt * 128 + g * 64), "r"(w0), "r"(h0), "r"(t0), "r"(n0) : "memory");
#pragma unroll
          for (int g = 0; g < BN / 64; ++g)
            asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
                         ::"r"(dst + A_BYTES + g * GRP), "l"(reinterpret_cast<uint64_t>(&tmX)), "r"(bar), "r"(nt * BN + g * 64), "r"(w0 + dw), "r"(h0 + dh),
                           "r"(t0 + dt_), "r"(n0) : "memory");
        }
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
      if (++iw == p.nW) { iw = 0; if (++ih == p.nH) { ih = 0; if (++it == p.nT) { it = 0; ++in; } } }
    }
  } else if (warp >= 4) {
    // Each 64-channel box is one MN-major swizzle atom wide; warpgroup g reads output-channel box g of the A stage and
    // every input-channel box of the B stage, one m64n64k16 per (box, 16 positions = two 8-row groups 1024 B apart).
    const uint32_t a_base = smem_u32(smem) + (uint32_t)((warp - 4) >> 2) * GRP;
    int stage = 0; uint32_t phase = 0;
    int iw, ih, it, in;
    long long kb = k0;
    decode(k0, iw, ih, it, in);
    auto skip_dead = [&]() {
      while (kb < k1 && !live(it)) { ++kb; if (++iw == p.nW) { iw = 0; if (++ih == p.nH) { ih = 0; if (++it == p.nT) { it = 0; ++in; } } } }
    };
    skip_dead();
    const bool any = kb < k1;
    float acc[BN / 64][32];
    int prev = -1;
    uint32_t first = 1;
    while (kb < k1) {
      mbar_wait(&full[stage], phase);
      const uint32_t a_addr = a_base + stage * ST_BYTES;
      const uint32_t b_addr = smem_u32(smem) + stage * ST_BYTES + A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {                                // 16 positions (2 swizzle atoms of 8 rows) per MMA
        const uint64_t adesc = make_sw128_desc(a_addr + k * 2048, true);
#pragma unroll
        for (int g = 0; g < BN / 64; ++g)
          wgmma<64, 0, 1>(acc[g], adesc, make_sw128_desc(b_addr + g * GRP + k * 2048, true), (first && k == 0) ? 0u : 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
      prev = stage;
      first = 0;
      if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      ++kb; if (++iw == p.nW) { iw = 0; if (++ih == p.nH) { ih = 0; if (++it == p.nT) { it = 0; ++in; } } }
      skip_dead();
    }
    wgmma_wait<0>();
    if (any) {
#pragma unroll
      for (int g = 0; g < BN / 64; ++g) wgrad_red<32>(acc[g], p.dW, p.Cout, p.Cin, tap, mt * 128, nt * BN + g * 64);
    }
  }
}

template <int BN>
static int launch_wgrad_nhwc(const CUtensorMap& tmG, const CUtensorMap& tmX, const WgradNParams& p, int smem, cudaStream_t stream) {
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(wgrad_nhwc_kernel<BN>, smem, &grant));
  const long long grid = (long long)p.taps * p.tiles_m * p.tiles_n * p.ksplit;      // < 2^31: wgrad_nhwc_geom
  wgrad_nhwc_kernel<BN><<<(unsigned)grid, WG_THREADS, smem, stream>>>(tmG, tmX, p);
  DT_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------ pointwise backward
__global__ void bwd_pointwise_kernel(const __nv_bfloat16* __restrict__ g1, const __nv_bfloat16* __restrict__ g2,
                                     const __nv_bfloat16* __restrict__ y, const float* __restrict__ scale, long long rows,
                                     int C, __nv_bfloat16* __restrict__ out, const float* __restrict__ scale2,
                                     __nv_bfloat16* __restrict__ out2) {
  const int cv = C / 8;
  const long long total = rows * cv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * 8;
    const size_t off = (size_t)(idx / cv) * C + c;
    const uint4 a = *reinterpret_cast<const uint4*>(g1 + off);
    const __nv_bfloat16* ae = reinterpret_cast<const __nv_bfloat16*>(&a);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = __bfloat162float(ae[j]);
    if (g2) {
      const uint4 b = *reinterpret_cast<const uint4*>(g2 + off);
      const __nv_bfloat16* be = reinterpret_cast<const __nv_bfloat16*>(&b);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += __bfloat162float(be[j]);
    }
    if (y) {
      const uint4 m = *reinterpret_cast<const uint4*>(y + off);
      const __nv_bfloat16* me = reinterpret_cast<const __nv_bfloat16*>(&m);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = __bfloat162float(me[j]) > 0.f ? v[j] : 0.f;
    }
    __align__(16) __nv_bfloat16 o[8];
    if (out2) {                                           // second consumer of the same masked sum (its own channel scale, or none)
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = __float2bfloat16_rn(scale2 ? v[j] * scale2[c + j] : v[j]);
      *reinterpret_cast<uint4*>(out2 + off) = *reinterpret_cast<const uint4*>(o);
    }
    if (scale) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] *= scale[c + j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = __float2bfloat16_rn(v[j]);
    *reinterpret_cast<uint4*>(out + off) = *reinterpret_cast<const uint4*>(o);
  }
}

// coarse_out[f, h, w, c] = coarse_in[f, h, w, c] (optional) + sum of the 2x2 children of fine[f, 2h.., 2w.., c]
__global__ void upsample_add_bwd_kernel(const __nv_bfloat16* __restrict__ fine, const __nv_bfloat16* __restrict__ coarse_in,
                                        int F, int Hc, int Wc, int C, __nv_bfloat16* __restrict__ out) {
  const int cv = C / 8;
  const long long total = (long long)F * Hc * Wc * cv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * 8;
    long long r = idx / cv;
    const int w = (int)(r % Wc); r /= Wc;
    const int h = (int)(r % Hc);
    const int f = (int)(r / Hc);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
    for (int dy = 0; dy < 2; ++dy)
      for (int dx = 0; dx < 2; ++dx) {
        const uint4 a = *reinterpret_cast<const uint4*>(fine + (((size_t)f * 2 * Hc + 2 * h + dy) * (2 * Wc) + 2 * w + dx) * C + c);
        const __nv_bfloat16* ae = reinterpret_cast<const __nv_bfloat16*>(&a);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += __bfloat162float(ae[j]);
      }
    const size_t off = (((size_t)f * Hc + h) * Wc + w) * C + c;
    if (coarse_in) {
      const uint4 a = *reinterpret_cast<const uint4*>(coarse_in + off);
      const __nv_bfloat16* ae = reinterpret_cast<const __nv_bfloat16*>(&a);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += __bfloat162float(ae[j]);
    }
    __align__(16) __nv_bfloat16 o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = __float2bfloat16_rn(v[j]);
    *reinterpret_cast<uint4*>(out + off) = *reinterpret_cast<const uint4*>(o);
  }
}

// out [F, 2*Hs, 2*Ws (cropped to H, W), C]: out[f, 2h, 2w] = src[f, h, w], zero elsewhere
__global__ void scatter_stride2_kernel(const __nv_bfloat16* __restrict__ src, int F, int Hs, int Ws, int H, int W, int C,
                                       __nv_bfloat16* __restrict__ out) {
  const int cv = C / 8;
  const long long total = (long long)F * H * W * cv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv) * 8;
    long long r = idx / cv;
    const int w = (int)(r % W); r /= W;
    const int h = (int)(r % H);
    const int f = (int)(r / H);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (!(h & 1) && !(w & 1) && (h >> 1) < Hs && (w >> 1) < Ws)
      v = *reinterpret_cast<const uint4*>(src + (((size_t)f * Hs + (h >> 1)) * Ws + (w >> 1)) * C + c);
    *reinterpret_cast<uint4*>(out + (((size_t)f * H + h) * W + w) * C + c) = v;
  }
}

// out [B, T, P, C]: frame c = src [B, P, C], every other frame zero (backward of the slice-center body/head link)
__global__ void embed_frame_kernel(const uint4* __restrict__ src, long long per_frame_v, int B, int T, int c, uint4* __restrict__ out) {
  const long long total = (long long)B * T * per_frame_v;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i % per_frame_v;
    const long long bt = i / per_frame_v;
    const int t = (int)(bt % T);
    out[i] = (t == c) ? src[(bt / T) * per_frame_v + e] : make_uint4(0, 0, 0, 0);
  }
}

// ------------------------------------------------------------------------------------------------ SGD
// Caffe2 MomentumSGDUpdate (non-Nesterov): g' = lr * (grad_scale * g + wd * w) + momentum * m;  m = g';  w -= g'
// w / g / m [taps][Cout][Cin] fp32.  Re-emits wf [taps][Cout][Cin] bf16 (forward operand) and wdg [taps][Cin][Cout] bf16
// with the taps FLIPPED (dgrad of a stride-1 "same" conv is the conv of the gradient with the flipped, transposed filter).
// Every parameter tensor of the model in ONE launch: a table of items (device memory, built once by the trainer) and the
// exclusive prefix of their 32x32 tile counts; a block finds its item by binary search and updates one (tap, 32 Cout,
// 32 Cin) tile with 256 threads as (32, 8): coalesced fp32 reads / writes along Cin, the transposed dgrad filter written
// through a shared-memory tile so that its stores are coalesced along Cout as well.
struct SgdItem {
  float* w; const float* g; float* m; __nv_bfloat16* wf; __nv_bfloat16* wdg;
  int taps, Cout, Cin, tiles_ci, tiles_co;
  float lr_mult, wd_mult;
};

__global__ void __launch_bounds__(256)
sgd_update_multi_kernel(const SgdItem* __restrict__ items, const int* __restrict__ first_block, int n_items, float lr, float momentum,
                        float wd, float grad_scale) {
  __shared__ float tile[32][33];
  int lo = 0, hi = n_items - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (first_block[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1; }
  const SgdItem it = items[lo];
  int t = (int)blockIdx.x - first_block[lo];
  const int tci = t % it.tiles_ci; t /= it.tiles_ci;
  const int tco = t % it.tiles_co;
  const int tap = t / it.tiles_co;
  const int co0 = tco * 32, ci0 = tci * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float lr_i = lr * it.lr_mult, wd_i = wd * it.wd_mult;
  for (int r = ty; r < 32; r += 8) {
    const int co = co0 + r, ci = ci0 + tx;
    float nw = 0.f;
    if (co < it.Cout && ci < it.Cin) {
      const size_t i = ((size_t)tap * it.Cout + co) * it.Cin + ci;
      const float wi = it.w[i];
      const float adj = lr_i * (grad_scale * it.g[i] + wd_i * wi) + momentum * it.m[i];
      it.m[i] = adj;
      nw = wi - adj;
      it.w[i] = nw;
      if (it.wf) it.wf[i] = __float2bfloat16_rn(nw);
    }
    tile[r][tx] = nw;
  }
  if (!it.wdg) return;
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int ci = ci0 + r, co = co0 + tx;
    if (ci < it.Cin && co < it.Cout) it.wdg[((size_t)(it.taps - 1 - tap) * it.Cin + ci) * it.Cout + co] = __float2bfloat16_rn(tile[tx][r]);
  }
}

// ------------------------------------------------------------------------------------------------ bias gradient, RPN losses
// db[c] += sum over rows of g[row, c]   (Conv bias gradient; biases of the FPN / RPN / head convs are trainable)
// block (32 channel groups of 8, 8 row lanes): 16-byte loads, fp32 partial sums, shared-memory reduction, one atomic per channel
__global__ void __launch_bounds__(256)
bias_grad_kernel(const __nv_bfloat16* __restrict__ g, long long rows, int C, int ld, float* __restrict__ db) {
  __shared__ float part[8][32][9];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c0 = (blockIdx.y * 32 + tx) * 8;
  const long long per = (rows + gridDim.x - 1) / gridDim.x;
  const long long r0 = per * blockIdx.x, r1 = min(rows, r0 + per);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (c0 < C) {
    for (long long r = r0 + ty; r < r1; r += 8) {
      const uint4 v = *reinterpret_cast<const uint4*>(g + (size_t)r * ld + c0);
      const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += __bfloat162float(e[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[ty][tx][j] = acc[j];
  __syncthreads();
  // 256 threads -> 256 channels of this block
  const int cc = threadIdx.x;                      // channel inside the 256-channel tile
  const int c = blockIdx.y * 256 + cc;
  if (c < C && r1 > r0) {
    float s = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) s += part[y][cc >> 3][cc & 7];
    atomicAdd(db + c, s);
  }
}

// FPN RPN losses and their gradients at one level (lib/modeling/FPN.py:282-321 with the Detectron ops
// SigmoidCrossEntropyLoss(normalize=0, scale=s_cls) and SmoothL1Loss(beta, scale=s_box), the latter divided by the batch size):
//   out rows [rows, ld_o] fp32 = [A logits | 4A deltas (a*4 + k)];  labels [rows, A] int32 (-1 = ignore);
//   targets / inside / outside weights [rows, 4A] fp32.  grad rows [rows, ld_g] bf16 in the same channel order (padding 0).
//   loss[0] += cls loss, loss[1] += bbox loss.
__global__ void rpn_loss_grad_kernel(const float* __restrict__ out, int ld_o, const int* __restrict__ labels,
                                     const float* __restrict__ targets, const float* __restrict__ iw, const float* __restrict__ ow,
                                     long long rows, int A, float s_cls, float s_box, float beta, __nv_bfloat16* __restrict__ grad,
                                     int ld_g, float* __restrict__ loss) {
  float lc = 0.f, lb = 0.f;
  const long long total = rows * ld_g;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(idx % ld_g);
    const long long r = idx / ld_g;
    float gv = 0.f;
    if (ch < A) {
      const int t = labels[r * A + ch];
      if (t >= 0) {
        const float x = out[r * ld_o + ch];
        // -x*(t - [x>=0]) + log(1 + exp(x - 2x[x>=0]))   (the op's stable form)
        lc += s_cls * (-x * ((float)t - (x >= 0.f ? 1.f : 0.f)) + log1pf(expf(x - 2.f * x * (x >= 0.f ? 1.f : 0.f))));
        gv = s_cls * (1.f / (1.f + expf(-x)) - (float)t);
      }
    } else if (ch < 5 * A) {
      const int j = ch - A;
      const float w_in = iw[r * 4 * A + j], w_out = ow[r * 4 * A + j];
      const float d = w_in * (out[r * ld_o + ch] - targets[r * 4 * A + j]);
      const float ad = fabsf(d);
      lb += s_box * w_out * (ad < beta ? 0.5f * d * d / beta : ad - 0.5f * beta);
      gv = s_box * w_out * w_in * (ad < beta ? d / beta : (d > 0.f ? 1.f : -1.f));
    }
    grad[idx] = __float2bfloat16_rn(gv);
  }
  for (int o = 16; o > 0; o >>= 1) { lc += __shfl_xor_sync(0xffffffffu, lc, o); lb += __shfl_xor_sync(0xffffffffu, lb, o); }
  if ((threadIdx.x & 31) == 0 && loss) { if (lc != 0.f) atomicAdd(loss, lc); if (lb != 0.f) atomicAdd(loss + 1, lb); }
}


// ------------------------------------------------------------------------------------------------ RoI heads (backward)
// out = bf16(g + acc)
__global__ void grad_join_f32_kernel(const __nv_bfloat16* __restrict__ g, const float* __restrict__ acc, long long n8,
                                     __nv_bfloat16* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const float4 a0 = reinterpret_cast<const float4*>(acc)[2 * i], a1 = reinterpret_cast<const float4*>(acc)[2 * i + 1];
    float v[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    if (g) {
      const uint4 gv = reinterpret_cast<const uint4*>(g)[i];
      const __nv_bfloat16* ge = reinterpret_cast<const __nv_bfloat16*>(&gv);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += __bfloat162float(ge[j]);
    }
    __align__(16) __nv_bfloat16 o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = __float2bfloat16_rn(v[j]);
    reinterpret_cast<uint4*>(out)[i] = *reinterpret_cast<const uint4*>(o);
  }
}

struct RoiBwdLevels {
  float* dfeat[8];
  int H[8], W[8];
  float scale[8];
};

__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// the forward's bilinear sample (dense_ops.cu bilinear_acc) transposed: v[8] * weight into the four corners
__device__ __forceinline__ void bilinear_scatter(float* __restrict__ d, int H, int W, int C, float y, float x, const float* v, float wgt) {
  if (!(y >= -1.f && y <= (float)H && x >= -1.f && x <= (float)W)) return;      // also for a non-finite RoI (diverged weights)
  if (y <= 0.f) y = 0.f;
  if (x <= 0.f) x = 0.f;
  int yl = (int)y, xl = (int)x, yh, xh;
  if (yl >= H - 1) { yh = yl = H - 1; y = (float)yl; } else yh = yl + 1;
  if (xl >= W - 1) { xh = xl = W - 1; x = (float)xl; } else xh = xl + 1;
  const float ly = y - yl, lx = x - xl, hy = 1.f - ly, hx = 1.f - lx;
  const float w4[4] = {hy * hx * wgt, hy * lx * wgt, ly * hx * wgt, ly * lx * wgt};
  float* p4[4] = {d + ((size_t)yl * W + xl) * C, d + ((size_t)yl * W + xh) * C, d + ((size_t)yh * W + xl) * C, d + ((size_t)yh * W + xh) * C};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (w4[q] == 0.f) continue;
    red_add_v4(p4[q], v[0] * w4[q], v[1] * w4[q], v[2] * w4[q], v[3] * w4[q]);
    red_add_v4(p4[q] + 4, v[4] * w4[q], v[5] * w4[q], v[6] * w4[q], v[7] * w4[q]);
  }
}

// grid (R*T, P); threads over (pw, 8-channel vectors) exactly like roi_align_kernel
__global__ void roi_align_bwd_kernel(RoiBwdLevels lv, int kmin, const float* __restrict__ rois, int ldr, const int* __restrict__ n_dev,
                                     int R, int T, const int* __restrict__ levels, int C, int P, int sampling,
                                     const __nv_bfloat16* __restrict__ grad) {
  const int rt = blockIdx.x, ph = blockIdx.y;
  const int r = rt / T, t = rt - r * T;
  const int n = n_dev ? min(*n_dev, R) : R;
  if (r >= n) return;
  const int cv = C / 8;
  const float* roi = rois + (size_t)r * ldr;
  const int l = levels ? (levels[r] - kmin) : 0;
  const int H = lv.H[l], W = lv.W[l];
  const float sc = lv.scale[l];
  const int img = (int)roi[0] * T + t;
  float* d = lv.dfeat[l] + (size_t)img * H * W * C;
  const float x1 = roi[1 + 4 * t] * sc, y1 = roi[2 + 4 * t] * sc, x2 = roi[3 + 4 * t] * sc, y2 = roi[4 + 4 * t] * sc;
  const float rw = fmaxf(x2 - x1, 1.f), rh = fmaxf(y2 - y1, 1.f);
  const float bh = rh / (float)P, bw = rw / (float)P;
  const int gh = sampling > 0 ? sampling : (int)ceilf(rh / P), gw = sampling > 0 ? sampling : (int)ceilf(rw / P);
  const float inv_cnt = 1.f / (float)(gh * gw);
  const __nv_bfloat16* gbase = grad + ((size_t)rt * P + ph) * P * C;
  for (int i = threadIdx.x; i < P * cv; i += blockDim.x) {
    const int pw = i / cv, c = (i - pw * cv) * 8;
    const uint4 gv = *reinterpret_cast<const uint4*>(gbase + (size_t)pw * C + c);
    const __nv_bfloat16* ge = reinterpret_cast<const __nv_bfloat16*>(&gv);
    float v[8];
    bool any = false;
#pragma unroll
    for (int j = 0; j < 8; ++j) { v[j] = __bfloat162float(ge[j]); any |= v[j] != 0.f; }
    if (!any) continue;
    for (int iy = 0; iy < gh; ++iy) {
      const float y = y1 + ph * bh + (iy + 0.5f) * bh / (float)gh;
      for (int ix = 0; ix < gw; ++ix) {
        const float x = x1 + pw * bw + (ix + 0.5f) * bw / (float)gw;
        bilinear_scatter(d + c, H, W, C, y, x, v, inv_cnt);
      }
    }
  }
}

// one thread per RoI row (C is small)
__global__ void frcnn_loss_grad_kernel(const float* __restrict__ out, int ld_o, const int* __restrict__ labels,
                                       const float* __restrict__ targets, const float* __restrict__ iw, const float* __restrict__ ow,
                                       int rows, int C, const float* __restrict__ totals, float s_cls, float s_box,
                                       __nv_bfloat16* __restrict__ grad, int ld_g, float* __restrict__ loss, float* __restrict__ acc) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  float lc = 0.f, lb = 0.f, hit = 0.f;
  if (r < rows) {
    __nv_bfloat16* g = grad + (size_t)r * ld_g;
    const int lbl = labels[r];
    const float N = totals[0];
    if (lbl < 0 || !(N > 0.f)) {
      for (int j = 0; j < ld_g; ++j) g[j] = __float2bfloat16_rn(0.f);
    } else {
      const float* o = out + (size_t)r * ld_o;
      float m = o[0]; int am = 0;
      for (int j = 1; j < C; ++j) if (o[j] > m) { m = o[j]; am = j; }
      float se = 0.f;
      for (int j = 0; j < C; ++j) se += expf(o[j] - m);
      const float lse = logf(se);
      lc = -(o[lbl] - m - lse) * s_cls / N;
      hit = am == lbl ? 1.f : 0.f;
      for (int j = 0; j < C; ++j) {
        const float pj = expf(o[j] - m - lse);
        g[j] = __float2bfloat16_rn((pj - (j == lbl ? 1.f : 0.f)) * s_cls / N);
      }
      for (int j = 0; j < 4 * C; ++j) {
        const float w_in = iw[(size_t)r * 4 * C + j], w_out = ow[(size_t)r * 4 * C + j];
        const float d = w_in * (o[C + j] - targets[(size_t)r * 4 * C + j]);
        const float ad = fabsf(d);
        lb += w_out * (ad < 1.f ? 0.5f * d * d : ad - 0.5f) * s_box / N;
        g[C + j] = __float2bfloat16_rn(w_out * w_in * (ad < 1.f ? d : (d > 0.f ? 1.f : -1.f)) * s_box / N);
      }
      for (int j = 5 * C; j < ld_g; ++j) g[j] = __float2bfloat16_rn(0.f);
    }
  }
  for (int o2 = 16; o2 > 0; o2 >>= 1) {
    lc += __shfl_xor_sync(0xffffffffu, lc, o2); lb += __shfl_xor_sync(0xffffffffu, lb, o2); hit += __shfl_xor_sync(0xffffffffu, hit, o2);
  }
  if ((threadIdx.x & 31) == 0) {
    if (loss) { if (lc != 0.f) atomicAdd(loss, lc); if (lb != 0.f) atomicAdd(loss + 1, lb); }
    if (acc && hit != 0.f) atomicAdd(acc, hit);
  }
}

// one CTA per (RoI d, joint k): 2S x 2S map -> bilinear 2x -> spatial softmax loss -> gradient back to the packed layout
__global__ void __launch_bounds__(256)
kps_loss_grad_kernel(const float* __restrict__ low, int ld, int S, int K, const int* __restrict__ loc, const float* __restrict__ wts,
                     const float* __restrict__ totals, float scale, __nv_bfloat16* __restrict__ grad, int ld_g, float* __restrict__ loss) {
  extern __shared__ float sm[];
  const int d = blockIdx.x, k = blockIdx.y;
  const int S2 = 2 * S, M = 4 * S;
  float* Lm = sm;                       // [S2][S2]
  float* U = Lm + S2 * S2;              // [M][M] upsampled logits, then their gradient
  __shared__ float red[32];
  __shared__ float s_max, s_sum;
  const float w = wts[(size_t)d * K + k];
  const float tw = totals[1];
  __nv_bfloat16* gd = grad + (size_t)d * S * S * ld_g;
  if (!(w > 0.f) || !(tw > 0.f)) {      // no target: zero gradient for this joint's four sub-pixel channels
    for (int i = threadIdx.x; i < S * S * 4; i += blockDim.x) gd[(size_t)(i >> 2) * ld_g + (i & 3) * K + k] = __float2bfloat16_rn(0.f);
    return;
  }
  const float* ld_ = low + (size_t)d * S * S * ld;
  for (int i = threadIdx.x; i < S2 * S2; i += blockDim.x) {
    const int Y = i / S2, X = i - Y * S2;
    Lm[i] = ld_[((size_t)(Y >> 1) * S + (X >> 1)) * ld + ((Y & 1) * 2 + (X & 1)) * K + k];
  }
  __syncthreads();
  const float f4[4] = {0.25f, 0.75f, 0.75f, 0.25f};
  // ConvTranspose k4 s2 p1: U[o] = sum_i L[i] * f[o - 2i + 1]  -> i in {(o-2)/2 .. (o+1)/2}
  float mx = -3.4e38f;
  for (int i = threadIdx.x; i < M * M; i += blockDim.x) {
    const int Y = i / M, X = i - Y * M;
    float acc = 0.f;
    for (int iy = (Y - 2 + 1) >> 1; iy <= (Y + 1) >> 1; ++iy) {
      if (iy < 0 || iy >= S2) continue;
      const int ky = Y - 2 * iy + 1;
      if (ky < 0 || ky > 3) continue;
      for (int ix = (X - 2 + 1) >> 1; ix <= (X + 1) >> 1; ++ix) {
        if (ix < 0 || ix >= S2) continue;
        const int kx = X - 2 * ix + 1;
        if (kx < 0 || kx > 3) continue;
        acc += Lm[iy * S2 + ix] * f4[ky] * f4[kx];
      }
    }
    U[i] = acc;
    mx = fmaxf(mx, acc);
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) { float m = red[0]; for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, red[i]); s_max = m; }
  __syncthreads();
  mx = s_max;
  float se = 0.f;
  for (int i = threadIdx.x; i < M * M; i += blockDim.x) se += expf(U[i] - mx);
  for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = se;
  __syncthreads();
  if (threadIdx.x == 0) { float s = 0.f; for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i]; s_sum = s; }
  __syncthreads();
  const float lse = logf(s_sum);
  const int target = loc[(size_t)d * K + k];
  const float gs = w * scale / tw;
  if (threadIdx.x == 0 && loss) atomicAdd(loss, -(U[target] - mx - lse) * gs);
  __syncthreads();
  for (int i = threadIdx.x; i < M * M; i += blockDim.x) U[i] = (expf(U[i] - mx - lse) - (i == target ? 1.f : 0.f)) * gs;
  __syncthreads();
  // dL[i] = sum_o dU[o] * f[o - 2i + 1], o in 2i-1 .. 2i+2
  for (int i = threadIdx.x; i < S2 * S2; i += blockDim.x) {
    const int iy = i / S2, ix = i - iy * S2;
    float acc = 0.f;
#pragma unroll
    for (int ky = 0; ky < 4; ++ky) {
      const int Y = 2 * iy - 1 + ky;
      if (Y < 0 || Y >= M) continue;
#pragma unroll
      for (int kx = 0; kx < 4; ++kx) {
        const int X = 2 * ix - 1 + kx;
        if (X < 0 || X >= M) continue;
        acc += U[Y * M + X] * f4[ky] * f4[kx];
      }
    }
    gd[((size_t)(iy >> 1) * S + (ix >> 1)) * ld_g + ((iy & 1) * 2 + (ix & 1)) * K + k] = __float2bfloat16_rn(acc);
  }
}

__global__ void subpixel_grad_fix_kernel(float* __restrict__ gW, float* __restrict__ gb, int K, int Cin, int ldc) {
  const long long total = 9ll * ldc * Cin;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)((i / Cin) % ldc), tap = (int)(i / ((long long)Cin * ldc));
    bool live = co < 4 * K;
    if (live) {
      const int sub = co / K, py = sub >> 1, px = sub & 1;
      const int dy = tap / 3 - 1, dx = tap % 3 - 1;
      const int ky = py + 1 - 2 * dy, kx = px + 1 - 2 * dx;
      live = ky >= 0 && ky <= 3 && kx >= 0 && kx <= 3;
    }
    if (!live) gW[i] = 0.f;
  }
  if (gb && blockIdx.x == 0) {
    for (int k = threadIdx.x; k < ldc; k += blockDim.x) {
      if (k < K) {
        const float s = gb[k] + gb[K + k] + gb[2 * K + k] + gb[3 * K + k];
        gb[k] = s; gb[K + k] = s; gb[2 * K + k] = s; gb[3 * K + k] = s;
      } else if (k >= 4 * K) {
        gb[k] = 0.f;
      }
    }
  }
}

}  // namespace dt

using namespace dt;

// the elementwise kernels move 16-byte vectors (uint4 / float4); NULL (an absent optional operand) passes
static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

static int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = num_sms() * 16ll;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// What dt_wgrad_nhwc launches, derived in one place for the launcher and dt_wgrad_nhwc_plan (the plan is what runs):
// argument checks, the 64-position tile, BN, the tile counts, the K split, the grid and the dynamic shared memory.
static int wgrad_nhwc_geom(int ld_g, int ld_x, int N, int T, int Ho, int Wo, int Hi, int Wi, int Cout, int Cin, int kT, int kH, int kW,
                           int sH, int sW, WgradNParams* pp, int* BN_out, int* smem_out) {
  DT_CHECK_ARG(N >= 1 && T >= 1 && Ho >= 1 && Wo >= 1 && Cout >= 1 && Cin >= 8 && Cin % 4 == 0 && kT >= 1 && kH >= 1 && kW >= 1 && (kT & 1) &&
                   (kH & 1) && (kW & 1) && ld_g >= Cout && ld_g % 8 == 0 && ld_x >= Cin && ld_x % 8 == 0 && sH >= 1 && sW >= 1,
               "dt_wgrad_nhwc: bad shape N=%d T=%d %dx%d Cout=%d (ld %d) Cin=%d (ld %d) k=%dx%dx%d", N, T, Ho, Wo, Cout, ld_g, Cin, ld_x, kT, kH, kW);
  const bool strided = sH != 1 || sW != 1;
  DT_CHECK_ARG(!strided || (kT == 1 && kH == 1 && kW == 1), "dt_wgrad_nhwc: only pointwise convs may be strided");
  DT_CHECK_ARG(strided ? (Ho == (Hi + sH - 1) / sH && Wo == (Wi + sW - 1) / sW) : (Ho == Hi && Wo == Wi), "dt_wgrad_nhwc: output %dx%d does not match input %dx%d / stride", Ho, Wo, Hi, Wi);
  WgradNParams& p = *pp;
  memset(&p, 0, sizeof(p));
  p.Cout = Cout; p.Cin = Cin; p.taps = kT * kH * kW; p.kT = kT; p.kH = kH; p.kW = kW; p.pT = kT / 2; p.pH = kH / 2; p.pW = kW / 2;
  p.T = T;
  // 64-position tile (TW, TH, TT, TB), powers of two: the largest useful fraction, then the widest rows
  {
    double best = -1.0;
    for (int tw = 64; tw >= 1; tw >>= 1)
      for (int th = 64 / tw; th >= 1; th >>= 1)
        for (int tt = 64 / (tw * th); tt >= 1; tt >>= 1) {
          const int tb = 64 / (tw * th * tt);
          if (tt > 1 && kT > 1) continue;                                   // temporal taps shift whole frames: one frame per box
          const double cover = (double)cdiv(Wo, tw) * tw * cdiv(Ho, th) * th * cdiv(T, tt) * tt * (double)cdiv(N, tb) * tb;
          const double eff = (double)Wo * Ho * T * N / cover;
          if (eff > best + 1e-9) { best = eff; p.TW = tw; p.TH = th; p.TT = tt; p.TB = tb; }
        }
  }
  p.nW = cdiv(Wo, p.TW); p.nH = cdiv(Ho, p.TH); p.nT = cdiv(T, p.TT); p.nN = cdiv(N, p.TB);
  const int BN = Cin > 64 ? 128 : 64;      // 128 x BN fp32 accumulators live in the registers of two warpgroups
  p.tiles_m = cdiv(Cout, 128); p.tiles_n = cdiv(Cin, BN);
  const long long units = (long long)p.taps * p.tiles_m * p.tiles_n;
  const long long kblocks = (long long)p.nW * p.nH * p.nT * p.nN;
  // K split: every CTA adds its 128 x BN partial tile into dW with red.global, so the split count is also the atomic
  // traffic multiplier.  Pointwise layers use ONE wave of CTAs (a 1x1 filter has few (tap, tile) units, so more waves
  // mean many partial tiles added per output tile), multi-tap layers two.
  const int waves = p.taps == 1 ? 1 : 2;
  long long ksplit = ((long long)num_sms() * waves + units - 1) / units;
  if (ksplit > kblocks / 4) ksplit = kblocks / 4;
  if (ksplit < 1) ksplit = 1;
  p.ksplit = (int)ksplit;
  DT_CHECK_ARG(units * ksplit < (1ll << 31), "dt_wgrad_nhwc: grid too large");
  *BN_out = BN;
  *smem_out = WG_STAGES * (2 + BN / 64) * 64 * 128 + 256;
  return 0;
}

extern "C" int dt_wgrad_nhwc_plan(int ld_g, int ld_x, int N, int T, int Ho, int Wo, int Hi, int Wi, int Cout, int Cin, int kT, int kH,
                                  int kW, int sH, int sW, dt_wgrad_plan_t* o) {
  DT_CHECK_ARG(o, "dt_wgrad_nhwc_plan: null pointer");
  WgradNParams p;
  int BN = 0, smem = 0;
  if (wgrad_nhwc_geom(ld_g, ld_x, N, T, Ho, Wo, Hi, Wi, Cout, Cin, kT, kH, kW, sH, sW, &p, &BN, &smem)) return 1;
  o->TW = p.TW; o->TH = p.TH; o->TT = p.TT; o->TB = p.TB;
  o->nW = p.nW; o->nH = p.nH; o->nT = p.nT; o->nN = p.nN;
  o->BN = BN; o->taps = p.taps; o->tiles_m = p.tiles_m; o->tiles_n = p.tiles_n; o->ksplit = p.ksplit;
  o->grid = p.taps * p.tiles_m * p.tiles_n * p.ksplit;
  o->smem_bytes = smem;
  return 0;
}

extern "C" int dt_wgrad_nhwc(const void* gz, int ld_g, const void* x, int ld_x, int N, int T, int Ho, int Wo, int Hi, int Wi, int Cout,
                             int Cin, int kT, int kH, int kW, int sH, int sW, float* dW, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  WgradNParams p;
  int BN = 0, smem = 0;
  if (wgrad_nhwc_geom(ld_g, ld_x, N, T, Ho, Wo, Hi, Wi, Cout, Cin, kT, kH, kW, sH, sW, &p, &BN, &smem)) return 1;
  DT_CHECK_ARG(gz && x && dW, "dt_wgrad_nhwc: null pointer");
  DT_CHECK_ARG(((uintptr_t)dW & 7) == 0, "dt_wgrad_nhwc: dW must be 8-byte aligned (red.global.add.v2.f32)");
  p.dW = dW;
  CUtensorMap tmG, tmX;
  const uint32_t box[5] = {64, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TT, (uint32_t)p.TB}, e[5] = {1, 1, 1, 1, 1};
  {
    uint64_t d[5] = {(uint64_t)Cout, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)T, (uint64_t)N};
    const uint64_t sC = (uint64_t)ld_g * 2;
    uint64_t st[4] = {sC, sC * Wo, sC * Wo * Ho, sC * Wo * Ho * T};
    if (encode_map(&tmG, 0, 5, gz, d, st, box, e)) return 1;
  }
  {   // strided pointwise convs: the stride is folded into the global strides (positions of the OUTPUT grid)
    uint64_t d[5] = {(uint64_t)Cin, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)T, (uint64_t)N};
    const uint64_t sC = (uint64_t)ld_x * 2;
    uint64_t st[4] = {sC * sW, sC * Wi * sH, sC * Wi * Hi, sC * Wi * Hi * T};
    if (encode_map(&tmX, 0, 5, x, d, st, box, e)) return 1;
  }
  switch (BN) {
    case 128: return launch_wgrad_nhwc<128>(tmG, tmX, p, smem, stream);
    default: return launch_wgrad_nhwc<64>(tmG, tmX, p, smem, stream);
  }
}

extern "C" int dt_bwd_pointwise(const void* g1, const void* g2, const void* y, const float* scale, long long rows, int C, void* out,
                                void* stream) {
  return dt_bwd_pointwise2(g1, g2, y, scale, rows, C, out, nullptr, nullptr, stream);
}

extern "C" int dt_bwd_pointwise2(const void* g1, const void* g2, const void* y, const float* scale, long long rows, int C, void* out,
                                 const float* scale2, void* out2, void* stream) {
  DT_CHECK_ARG(rows >= 0 && C >= 8 && C % 8 == 0, "dt_bwd_pointwise: bad shape rows=%lld C=%d (C %% 8 == 0)", rows, C);
  if (rows == 0) return 0;
  DT_CHECK_ARG(g1 && out, "dt_bwd_pointwise: null pointer");
  DT_CHECK_ARG(aligned16(g1) && aligned16(g2) && aligned16(y) && aligned16(out) && aligned16(out2),
               "dt_bwd_pointwise: g1 / g2 / y / out / out2 must be 16-byte aligned");
  bwd_pointwise_kernel<<<grid_for(rows * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)g1, (const __nv_bfloat16*)g2, (const __nv_bfloat16*)y, scale, rows, C, (__nv_bfloat16*)out, scale2,
      (__nv_bfloat16*)out2);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_upsample_add_bwd(const void* fine, const void* coarse_in, int F, int Hc, int Wc, int C, void* out, void* stream) {
  DT_CHECK_ARG(F >= 0 && Hc >= 1 && Wc >= 1 && C >= 8 && C % 8 == 0, "dt_upsample_add_bwd: bad shape");
  if (F == 0) return 0;
  DT_CHECK_ARG(fine && out, "dt_upsample_add_bwd: null pointer");
  DT_CHECK_ARG(aligned16(fine) && aligned16(coarse_in) && aligned16(out), "dt_upsample_add_bwd: fine / coarse_in / out must be 16-byte aligned");
  upsample_add_bwd_kernel<<<grid_for((long long)F * Hc * Wc * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)fine, (const __nv_bfloat16*)coarse_in, F, Hc, Wc, C, (__nv_bfloat16*)out);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_scatter_stride2(const void* src, int F, int Hs, int Ws, int H, int W, int C, void* out, void* stream) {
  DT_CHECK_ARG(F >= 0 && Hs >= 1 && Ws >= 1 && H >= 1 && W >= 1 && (H + 1) / 2 == Hs && (W + 1) / 2 == Ws && C >= 8 && C % 8 == 0,
               "dt_scatter_stride2: bad shape %dx%d -> %dx%d C=%d", Hs, Ws, H, W, C);
  if (F == 0) return 0;
  DT_CHECK_ARG(src && out, "dt_scatter_stride2: null pointer");
  DT_CHECK_ARG(aligned16(src) && aligned16(out), "dt_scatter_stride2: src / out must be 16-byte aligned");
  scatter_stride2_kernel<<<grid_for((long long)F * H * W * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)src, F, Hs, Ws, H, W, C, (__nv_bfloat16*)out);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_embed_frame(const void* src, int B, int T, long long frame_elems, int c, void* out, void* stream) {
  DT_CHECK_ARG(B >= 0 && T >= 1 && c >= 0 && c < T && frame_elems >= 8 && frame_elems % 8 == 0, "dt_embed_frame: bad shape B=%d T=%d c=%d elems=%lld", B, T, c, frame_elems);
  if (B == 0) return 0;
  DT_CHECK_ARG(src && out, "dt_embed_frame: null pointer");
  DT_CHECK_ARG(aligned16(src) && aligned16(out), "dt_embed_frame: src / out must be 16-byte aligned");
  embed_frame_kernel<<<grid_for((long long)B * T * (frame_elems / 8), 256), 256, 0, (cudaStream_t)stream>>>((const uint4*)src, frame_elems / 8, B, T, c, (uint4*)out);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_sgd_update_multi(const void* items, const int* first_block, int n_items, int total_blocks, float lr, float momentum,
                                   float wd, float grad_scale, void* stream) {
  DT_CHECK_ARG(n_items >= 1 && total_blocks >= 1, "dt_sgd_update_multi: empty table (n_items=%d, blocks=%d)", n_items, total_blocks);
  DT_CHECK_ARG(items && first_block, "dt_sgd_update_multi: null pointer");
  static_assert(sizeof(SgdItem) == 72, "dt_sgd_item layout");
  sgd_update_multi_kernel<<<total_blocks, 256, 0, (cudaStream_t)stream>>>((const SgdItem*)items, first_block, n_items, lr, momentum, wd, grad_scale);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_bias_grad(const void* g, long long rows, int C, int ld, float* db, void* stream) {
  DT_CHECK_ARG(rows >= 0 && C >= 8 && C % 8 == 0 && ld >= C && ld % 8 == 0, "dt_bias_grad: bad shape rows=%lld C=%d ld=%d (multiples of 8)", rows, C, ld);
  if (rows == 0) return 0;
  DT_CHECK_ARG(g && db, "dt_bias_grad: null pointer");
  DT_CHECK_ARG(aligned16(g), "dt_bias_grad: g must be 16-byte aligned");
  long long gx = rows / 128; if (gx < 1) gx = 1; if (gx > num_sms() * 8ll) gx = num_sms() * 8ll;
  dim3 grid((unsigned)gx, (C + 255) / 256);
  bias_grad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)g, rows, C, ld, db);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_rpn_loss_grad(const float* out, int ld_o, const int* labels, const float* targets, const float* inside_w,
                                const float* outside_w, long long rows, int A, float scale_cls, float scale_box, float beta,
                                void* grad, int ld_g, float* loss, void* stream) {
  DT_CHECK_ARG(rows >= 0 && A >= 1 && ld_o >= 5 * A && ld_g >= 5 * A && beta > 0.f, "dt_rpn_loss_grad: bad shape rows=%lld A=%d ld_o=%d ld_g=%d", rows, A, ld_o, ld_g);
  if (rows == 0) return 0;
  DT_CHECK_ARG(out && labels && targets && inside_w && outside_w && grad, "dt_rpn_loss_grad: null pointer");
  rpn_loss_grad_kernel<<<grid_for(rows * ld_g, 256), 256, 0, (cudaStream_t)stream>>>(out, ld_o, labels, targets, inside_w, outside_w, rows, A,
                                                                                  scale_cls, scale_box, beta, (__nv_bfloat16*)grad, ld_g, loss);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_grad_join_f32(const void* g, const float* acc, long long n, void* out, void* stream) {
  DT_CHECK_ARG(n >= 0 && n % 8 == 0, "dt_grad_join_f32: n=%lld must be a multiple of 8", n);
  if (n == 0) return 0;
  DT_CHECK_ARG(acc && out, "dt_grad_join_f32: null pointer");
  DT_CHECK_ARG(aligned16(g) && aligned16(acc) && aligned16(out), "dt_grad_join_f32: g / acc / out must be 16-byte aligned");
  grad_join_f32_kernel<<<grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)g, acc, n / 8, (__nv_bfloat16*)out);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_roi_align_bwd(const void* grad, float* const* dfeats, const int* Hs, const int* Ws, const float* scales, int nlevels,
                                int k_min, int C, const float* rois, int ldr, const int* n_dev, int R, int T, const int* levels, int P,
                                int sampling_ratio, void* stream) {
  DT_CHECK_ARG(nlevels >= 1 && nlevels <= 8 && C >= 8 && C % 8 == 0 && R >= 0 && T >= 1 && P >= 1 && ldr >= 4 * T + 1,
               "dt_roi_align_bwd: bad shape (C=%d must be a multiple of 8)", C);
  DT_CHECK_ARG(nlevels == 1 || levels, "dt_roi_align_bwd: multi-level pooling needs the per-RoI level array");
  if (R == 0) return 0;
  DT_CHECK_ARG(grad && dfeats && Hs && Ws && scales && rois, "dt_roi_align_bwd: null pointer");
  RoiBwdLevels lv;
  for (int l = 0; l < nlevels; ++l) {
    DT_CHECK_ARG(dfeats[l], "dt_roi_align_bwd: null accumulator for level %d", l);
    DT_CHECK_ARG(aligned16(dfeats[l]), "dt_roi_align_bwd: accumulator of level %d must be 16-byte aligned (red.global.add.v4.f32)", l);
    lv.dfeat[l] = dfeats[l]; lv.H[l] = Hs[l]; lv.W[l] = Ws[l]; lv.scale[l] = scales[l];
  }
  dim3 grid(R * T, P);
  roi_align_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(lv, k_min, rois, ldr, n_dev, R, T, levels, C, P, sampling_ratio,
                                                              (const __nv_bfloat16*)grad);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_frcnn_loss_grad(const float* out, int ld_o, const int* labels, const float* targets, const float* inside_w,
                                  const float* outside_w, int rows, int C, const float* totals, float scale_cls, float scale_box,
                                  void* grad, int ld_g, float* loss, float* accuracy, void* stream) {
  DT_CHECK_ARG(rows >= 0 && C >= 2 && ld_o >= 5 * C && ld_g >= 5 * C, "dt_frcnn_loss_grad: bad shape rows=%d C=%d ld_o=%d ld_g=%d", rows, C, ld_o, ld_g);
  if (rows == 0) return 0;
  DT_CHECK_ARG(out && labels && targets && inside_w && outside_w && totals && grad, "dt_frcnn_loss_grad: null pointer");
  frcnn_loss_grad_kernel<<<(rows + 127) / 128, 128, 0, (cudaStream_t)stream>>>(out, ld_o, labels, targets, inside_w, outside_w, rows, C, totals,
                                                                             scale_cls, scale_box, (__nv_bfloat16*)grad, ld_g, loss, accuracy);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_kps_loss_grad(const float* low, int ld, int S, int K, int D, const int* locations, const float* weights,
                                const float* totals, float scale, void* grad, int ld_g, float* loss, void* stream) {
  DT_CHECK_ARG(S >= 1 && S <= 32 && K >= 1 && D >= 0 && ld >= 4 * K && ld_g >= 4 * K, "dt_kps_loss_grad: bad shape S=%d K=%d D=%d ld=%d ld_g=%d", S, K, D, ld, ld_g);
  if (D == 0) return 0;
  DT_CHECK_ARG(low && locations && weights && totals && grad, "dt_kps_loss_grad: null pointer");
  const size_t smem = (size_t)(4 * S * S + 16 * S * S) * sizeof(float);
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(kps_loss_grad_kernel, (int)smem, &grant));
  dim3 grid(D, K);
  kps_loss_grad_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(low, ld, S, K, locations, weights, totals, scale, (__nv_bfloat16*)grad, ld_g, loss);
  DT_CHECK_LAUNCH();
  return 0;
}

extern "C" int dt_subpixel_grad_fix(float* gW, float* gb, int K, int Cin, int ldc, void* stream) {
  DT_CHECK_ARG(K >= 1 && Cin >= 1 && ldc >= 4 * K, "dt_subpixel_grad_fix: bad shape K=%d Cin=%d ldc=%d", K, Cin, ldc);
  DT_CHECK_ARG(gW, "dt_subpixel_grad_fix: null pointer");
  subpixel_grad_fix_kernel<<<grid_for(9ll * ldc * Cin, 256), 256, 0, (cudaStream_t)stream>>>(gW, gb, K, Cin, ldc);
  DT_CHECK_LAUNCH();
  return 0;
}
