// Conv3d / Conv2d / FC as ONE implicit-GEMM kernel on the Hopper tensor cores (wgmma),
// NDHWC activations, fused AffineChannel (+bias) + residual / top-down-upsample add + ReLU.
//
// Replaces, on the reference's hot path:
//   Caffe2 Conv / ConvNd engine=CUDNN        (lib/modeling/detector.py:318-322,410-436 and every
//                                             call site listed in SURVEY.md §2.3 K5)
//   AffineChannelNdOp<float,CUDAContext>     (lib/ops/affine_channel_nd_op.cu:19-70)  -> epilogue
//   Relu / Sum (residual)                    (lib/modeling/ResNet3D.py:37,47,147-152) -> epilogue
//   UpsampleNearest + Sum (FPN top-down)     (lib/modeling/FPN3D.py:211-222)          -> epilogue
//   FC (cuBLAS)                              (lib/modeling/head_builder.py:33-36)     -> kT=kH=kW=1
//
// GEMM view: D[m, n] = sum_{tap, c} A[m @ tap, c] * W[tap, n, c]
//   m = output position (img, t, ho, wo) tiled as TH x TW spatial patches (TH*TW <= 128 rows)
//   n = output channel, BLOCK_N in {32, 64, 128};  k-block = one tap x 128 bytes of channels
//   A tile: one 5-D TMA box (C=128B, TW, TH, 1, 1) at the tap-shifted coordinate; out-of-bounds
//           elements (spatial / temporal zero padding, ragged edge tiles, channel tail) are
//           zero-filled by the TMA unit, so padding costs no instructions and no branches.
//   W tile: 3-D TMA box (C=128B, BLOCK_N, 1) of the pre-packed [tap][Cout][Cin] weights.
//   Both land in the 128B-swizzled K-major layout wgmma reads directly.
// Roles (384 threads = 3 warpgroups, 1 CTA / SM, persistent over tiles):
//   warp 0, 1 : TMA producers (activation / weight tiles; one elected lane each)   smem ring: full[]/empty[]
//   warp 2    : TMA store warp                           staged output chunks -> global, recycles staging slots
//   warp 3    : idle (pads the producer warpgroup)
//   warps 4-11: two consumer warpgroups, rows 0-63 and 64-127 of the tile: wgmma into register accumulators
//               (64 x BLOCK_N each), then the epilogue: scale/bias/residual/ReLU in fp32, staged in 128B-swizzled
//               smem chunks.  The producers run ahead into the next tile's k-blocks while the epilogue runs.
// Everything is handed over through mbarriers; there is no block-wide barrier inside the tile loop.
#include "common.cuh"
#include "tc_common.cuh"
#include "../../include/dt_b200.h"
#include <cuda_bf16.h>
#include <stdlib.h>

namespace dt {

using namespace tc;

// division by a run-time constant without the ~100-cycle integer-division sequence (valid for x < 2^31)
struct FastDiv {
  uint32_t mul, shr, d;
};
static FastDiv make_fastdiv(int d) {
  FastDiv f; f.d = (uint32_t)d; f.mul = 0; f.shr = 0;
  if (d > 1) {
    int l = 0;
    while ((1u << l) < (uint32_t)d) ++l;
    const int pw = 31 + l;
    f.mul = (uint32_t)((((unsigned long long)1 << pw) + (unsigned long long)d - 1) / (unsigned long long)d);
    f.shr = (uint32_t)(l - 1);
  }
  return f;
}
__device__ __forceinline__ uint32_t fdiv(uint32_t x, const FastDiv& f) { return f.d == 1 ? x : (__umulhi(x, f.mul) >> f.shr); }

struct ConvKernelParams {
  // output geometry
  int N, To, Ho, Wo, Cout;
  // filter
  int kT, kH, kW, sT, sH, sW, pT, pH, pW;
  int kchunks;                 // ceil(Cin / BK)
  // tiling
  int TH, TW, TT, TB;          // rows of one M tile = TB images x TT frames x TH x TW positions (<= 128)
  int tiles_h, tiles_w, tiles_t, tiles_b, tiles_n, total_tiles;
  FastDiv fd_n, fd_w, fd_h, fd_t;    // tile index -> (column tile, w, h, t, image) tile coordinates
  uint32_t a_bytes;            // TB*TT*TH*TW*128
  // epilogue
  const float* scale;          // [Cout] or null (1)
  const float* bias;           // [Cout] or null (0)
  const void* residual;        // same dtype as out, or null
  int res_mode;                // 0 none, 1 same shape, 2 nearest-2x upsample of (Ho/2, Wo/2)
  int res_ld;
  int relu;
  int out_f32;                 // 1: fp32 output, 0: bf16
  // 3xTF32 ("fp32-accurate") mode: activations / weights are stored as [hi | lo] tf32 pairs along the
  // channel axis; D = A_hi*B_hi + A_lo*B_hi + A_hi*B_lo (the lo*lo term is below fp32 resolution).
  int split_in;                // 1: x and w rows are [hi | lo] pairs with the offsets below (kernel NMMA = 3)
  int a_lo_off, b_lo_off;      // element offsets of the lo halves in the x rows / packed weight rows
  int b_lo_blk;                // split conv1: the lo weight box is the next packed weight block instead
  int split_out;               // 1: write hi at channel c and lo at out_lo_off + c (fp32)
  int out_lo_off, res_lo_off;  // lo-half offsets of the output / residual rows
  int nstages, ncbuf;          // smem split chosen per layer: operand ring depth / output staging buffers
  int ks;                      // (tap, channel chunk) groups per ring stage
  int ktab;                    // entries of the schedule (one per group + 1 padding, even)
  int t_first;                 // first output frame computed (frames before it are skipped)
  int row_planes;              // conv1: input rows de-interleaved by parity, filter row kh -> plane kh & 1, row + kh >> 1
  int nrbuf;                   // > 0: bf16 residual chunks arrive by TMA in a ring of this many staged chunks
  int res_up;                  // with nrbuf > 0: the residual is the (Ho/2, Wo/2) map of the FPN top-down add;
                               // its (TH/2 x TW/2) box is loaded and every row is read by its four children
  int ab_format;               // 16-bit operand format: 1 bf16, 0 fp16 (TF32 kernels ignore it)
  int round_tf32;              // fp32 output is rounded (RNE) to tf32 so the next tf32 MMA, which ignores the
                               // low mantissa bits of its 32-bit operands, sees exactly representable values
};

__device__ __forceinline__ float round_to_tf32(float v) {
  uint32_t u = __float_as_uint(v);
  u += 0xFFFu + ((u >> 13) & 1u);
  return __uint_as_float(u & 0xFFFFE000u);
}

constexpr int EPI_WARPS = 8;                          // two consumer warpgroups
constexpr int CONV_THREADS = 128 + EPI_WARPS * 32;    // + the producer warpgroup (two TMA producer warps, the TMA store warp)
constexpr int B_WARP = 1;                             // weight-tile producer
constexpr int EPI_WARP0 = 4;                          // first consumer warp

template <int BN>
struct ConvCfg {
  static constexpr int A_BYTES = 128 * 128;            // 128 rows x 128 B
  static constexpr int B_BYTES = BN * 128;
  static constexpr int MAX_STAGES = 8;
  static constexpr int C_BYTES = 128 * 128;            // one staged output chunk: 128 rows x 128 B
  static constexpr int BAR_BYTES = 384;                // mbarriers
  static constexpr int FIXED_BYTES = BAR_BYTES;
  static constexpr int BUDGET = 227 * 1024;
  // A (tap, channel chunk) group of a conv with nmma MMA k-blocks per group is its activation boxes followed by its
  // weight boxes, each fetched once: plain [A | W]; split operands (nmma 3) [A_hi A_lo | W_hi W_lo] for the products
  // A_hi*W_hi, A_lo*W_hi, A_hi*W_lo; split conv1 (nmma 2) [A | W_2kh W_2kh+1] (the blob pixel carries [hi3 | lo3]:
  // block 2*kh is [W_hi | W_hi], block 2*kh + 1 is [W_lo | 0]).
  static constexpr int boxes_a(int nmma) { return nmma == 3 ? 2 : 1; }
  static constexpr int boxes_b(int nmma) { return nmma >= 2 ? 2 : 1; }
  static constexpr int group_bytes(int nmma) { return boxes_a(nmma) * A_BYTES + boxes_b(nmma) * B_BYTES; }
  // K-heavy layers want a deep operand ring; K-light (HBM-bound) layers want output staging buffers so the
  // epilogue never waits for a TMA store to drain, and (with a residual) a ring of prefetched residual chunks.
  static int tab_bytes(int groups) { return ((groups + 2) * 24 + 127) / 128 * 128; }   // schedule: one entry per group
  static void split(int groups, int nmma, bool res_tma, bool split_out, bool out_f32, int* stages, int* ks, int* ncbuf,
                    int* nrbuf) {
    const int kiters = groups * nmma;                   // MMA k-blocks per tile
    const int gb = group_bytes(nmma);
    const int chunks = BN / (out_f32 ? 32 : 64);        // staged chunks per tile
    int c = (kiters >= 12 && !split_out) ? 2 : 4;       // split (hi, lo) output: two slots of two buffers
    if (!split_out && c > 2 * chunks) c = chunks >= 1 ? 2 * chunks : 2;   // two tiles of staging are enough
    int r = res_tma ? ((kiters >= 12 || split_out) ? 2 : 4) : 0;      // split output: a residual slot is a chunk pair
    const int fixed = BUDGET - FIXED_BYTES - tab_bytes(groups);
    // split stages (64 KiB at BN = 128) need room.  The split residual layers fit two stages by keeping one residual
    // slot pair instead of two (measured faster than giving up an output staging slot pair instead)
    if (split_out && nmma > 1 && r > 1 && (fixed - (c + 2 * r) * C_BYTES) / gb < 2) r = 1;
    const int rb = split_out ? 2 * r : r;
    // with two split stages only one group's refill is in flight while the other's MMAs run, and a 64 KiB refill does
    // not land within one group's MMA time: a K-heavy split output is staged through one (hi, lo) slot pair instead of
    // two when that buys a third stage (K-light layers measured faster with both slot pairs)
    const int st_wide = (fixed - (c + rb) * C_BYTES) / gb, st_lean = (fixed - (2 + rb) * C_BYTES) / gb;
    if (split_out && nmma > 1 && c > 2 && kiters >= 12 && st_wide < 3 && st_lean > st_wide) c = 2;
    // narrow tiles retire a k-block's MMAs faster than one producer / issuer round trip through the
    // mbarriers: let a ring stage carry two plain k-blocks there (same bytes in flight, half the handshakes)
    const int avail = fixed - (c + rb) * C_BYTES;
    const int k = (nmma == 1 && BN <= 128 && kiters >= 2 && avail / (2 * gb) >= 3) ? 2 : 1;
    int st = avail / (k * gb);
    if (st > MAX_STAGES) st = MAX_STAGES;
    *stages = st; *ks = k; *ncbuf = c; *nrbuf = r;
  }
  static int smem_bytes(int groups, int nmma, int stages, int ks, int ncbuf, int nrbuf, bool split_out) {
    return stages * ks * group_bytes(nmma) + (ncbuf + (split_out ? 2 : 1) * nrbuf) * C_BYTES + FIXED_BYTES +
           tab_bytes(groups);
  }
};

struct TileCoord { int nt, twi, thi, tti, tbi; };
__device__ __forceinline__ TileCoord decode_tile(const ConvKernelParams& p, int tile) {
  TileCoord c;
  uint32_t m = fdiv((uint32_t)tile, p.fd_n);  c.nt = tile - (int)m * p.tiles_n;
  uint32_t q = fdiv(m, p.fd_w);               c.twi = (int)m - (int)q * p.tiles_w;  m = q;
  q = fdiv(m, p.fd_h);                        c.thi = (int)m - (int)q * p.tiles_h;  m = q;
  q = fdiv(m, p.fd_t);                        c.tti = (int)m - (int)q * p.tiles_t;
  c.tbi = (int)q;
  return c;
}

// SPLIT: the output (and the residual) rows are [hi | lo] pairs (the x3 modes' intermediate activations); a template
// parameter so that the plain kernels do not carry the pair logic's registers.
// KIND: MMA operand type, 0 bf16, 1 fp16, 2 tf32 (wgmma.cuh).
// NMMA: MMA k-blocks per (tap, channel chunk) group, 1 plain, 3 split operands, 2 split conv1 (ConvCfg::group_bytes);
// a template parameter so that the products of a group are straight-line wgmmas.
template <int BN, int KIND, bool SPLIT, int NMMA>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
               const ConvKernelParams p) {
  using Cfg = ConvCfg<BN>;
  const int STAGES = p.nstages;
  constexpr int BK = KIND == 2 ? 32 : 64;            // elements per 128-byte k-block
  constexpr int NA = Cfg::boxes_a(NMMA), NB = Cfg::boxes_b(NMMA);
  // SWIZZLE_128B operands need 1024-byte aligned tiles: the dynamic window is declared with that alignment
  // (no static shared memory in this kernel) and checked once below instead of spending a kilobyte on slack
  extern __shared__ __align__(1024) uint8_t smem[];
  // ring stage: p.ks groups of [A_0 .. A_{NA-1} | W_0 .. W_{NB-1}], every box 1024-byte aligned
  constexpr uint32_t group_bytes = (uint32_t)Cfg::group_bytes(NMMA);
  const uint32_t stage_bytes = (uint32_t)p.ks * group_bytes;
  uint8_t* cbuf = smem + STAGES * stage_bytes;                       // [NCBUF][128 rows][128 B], 128B-swizzled
  uint8_t* rbuf = cbuf + p.ncbuf * Cfg::C_BYTES;                     // [NRBUF] residual chunks, same layout
  constexpr uint32_t rslot_bytes = SPLIT ? 2u * Cfg::C_BYTES : (uint32_t)Cfg::C_BYTES;   // split: (hi, lo) chunk pair
  uint64_t* bars = reinterpret_cast<uint64_t*>(rbuf + p.nrbuf * rslot_bytes);
  uint64_t* full = bars;                       // [STAGES]  operands landed
  uint64_t* empty = bars + STAGES;             // [STAGES]  operands consumed by the MMAs
  uint64_t* r_full = bars + 2 * STAGES;        // [4]       residual chunk landed
  uint64_t* r_empty = r_full + 4;              // [4]       residual chunk consumed
  uint64_t* c_full = r_full + 8;               // [4]       output chunk staged by all epilogue warps
  uint64_t* c_free = r_full + 12;              // [4]       staging slot read out by its TMA store
  // schedule of one tile, one entry per (tap, channel chunk) group: what the producers add to the tile's base
  // coordinates for the group's first boxes (its lo boxes sit at the lo offsets from there).
  // Built once; walking taps / channel chunks with carry logic in the producer loop costs more cycles per
  // k-block than a narrow tile's MMAs take.
  int4* tabA = reinterpret_cast<int4*>(reinterpret_cast<uint8_t*>(bars) + Cfg::BAR_BYTES);   // {c, dw, dh, dt}
  int2* tabB = reinterpret_cast<int2*>(tabA + p.ktab);                                        // {c, weight block}
  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();
  {
    const int groups = p.kT * p.kH * p.kW * p.kchunks;
    for (int j = threadIdx.x; j < p.ktab; j += blockDim.x) {
      int r = min(j, groups - 1);                       // padding entries repeat the last group (never issued)
      const int kc = r % p.kchunks; r /= p.kchunks;
      const int tap = r;
      const int kw = r % p.kW; r /= p.kW;
      const int kh = r % p.kH;
      const int kt = r / p.kH;
      if (p.row_planes) {          // conv1: one box per filter row; split mode: weight blocks 2*kh (hi) and 2*kh + 1 (lo)
        tabA[j] = make_int4(0, 0, kh >> 1, kh & 1);
        tabB[j] = make_int2(0, tap * NB);
      } else {
        tabA[j] = make_int4(kc * BK, kw, kh, kt);
        tabB[j] = make_int2(kc * BK, tap);
      }
    }
  }

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    prefetch_tmap(&tmC);
    if (p.nrbuf > 0) prefetch_tmap(&tmR);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 2); mbar_init(&empty[s], EPI_WARPS); }  // full: A and B producers
    for (int s = 0; s < 4; ++s) {
      mbar_init(&r_full[s], 1); mbar_init(&r_empty[s], EPI_WARPS);
      mbar_init(&c_full[s], EPI_WARPS); mbar_init(&c_free[s], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above (barrier init, tensor-map prefetch, the k-block schedule) touched
  // only kernel parameters and shared memory, so it may overlap the tail of the previous kernel of the stream; no
  // global data is read or written before this wait.  The trigger lets the NEXT kernel's prologue do the same under
  // this one's tail (its CTAs become resident as this kernel's CTAs retire: 1 CTA / SM by shared memory).
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  const int groups = p.kT * p.kH * p.kW * p.kchunks;    // (tap, channel chunk) groups per tile

  if (warp == 0 || warp == B_WARP) {
    // ===================== TMA producers =====================
    // Two warps: warp 0 loads the activation tiles (and the residual ring), warp B_WARP the weight tiles; both
    // arm the same full[] barrier with their own byte count, so the scalar bookkeeping of the two operands runs
    // in parallel.  The whole warp runs the loop (warp-uniform control flow and addresses, so descriptors /
    // coordinates stay in uniform registers); one elected lane issues.
    const bool load_b = warp != 0;
    int stage = 0; uint32_t phase = 0;
    int rslot = 0; uint32_t rphase = 0;
    const uint32_t smem_u = smem_u32(smem) + (load_b ? (uint32_t)(NA * Cfg::A_BYTES) : 0u);
    const uint32_t full_u = smem_u32(full), empty_u = smem_u32(empty);
    const int KS = p.ks;                                  // groups per ring stage (one mbarrier round trip)
    const int nbox = load_b ? NB : NA;                    // this warp's boxes per group: hi, then lo
    const uint32_t box_bytes = load_b ? (uint32_t)Cfg::B_BYTES : (uint32_t)Cfg::A_BYTES;
    const uint32_t box_tx = load_b ? (uint32_t)Cfg::B_BYTES : p.a_bytes;
    const int lo_c = load_b ? p.b_lo_off : p.a_lo_off;    // the lo box: channel offset / weight block offset
    const int lo_blk = load_b ? p.b_lo_blk : 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord tc = decode_tile(p, tile);
      const int n = tc.tbi * p.TB;
      const int w_base = tc.twi * p.TW * p.sW - p.pW;
      const int h_base = tc.thi * p.TH * p.sH - p.pH;
      const int t_base = p.row_planes ? 0 : (tc.tti * p.TT + p.t_first) * p.sT - p.pT;
      const int n_base = tc.nt * BN;
      for (int ki = 0; ki < groups; ki += KS) {
        const int nk = min(KS, groups - ki);
        // this stage's groups from the schedule (uniform loads), then ONE elected issue block
        int x0[2], x1[2], x2[2], x3[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          if (load_b) {
            const int2 e = tabB[ki + q];
            x0[q] = e.x; x1[q] = n_base; x2[q] = e.y; x3[q] = 0;
          } else {
            const int4 e = tabA[ki + q];
            x0[q] = e.x; x1[q] = w_base + e.y; x2[q] = h_base + e.z; x3[q] = t_base + e.w;
          }
        }
        mbar_wait_u(empty_u + stage * 8, phase ^ 1);
        if (elect_one()) {
          const uint32_t bar = full_u + stage * 8;
          const uint32_t dst = smem_u + stage * stage_bytes;
          mbar_expect_tx_u(bar, (uint32_t)(nk * nbox) * box_tx);
#pragma unroll
          for (int q = 0; q < 2; ++q) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              if (q >= nk || i >= nbox) continue;
              const uint32_t d = dst + q * group_bytes + i * box_bytes;
              if (load_b) tma_load_3d_u(d, &tmB, bar, x0[q] + i * lo_c, x1[q], x2[q] + i * lo_blk);
              else tma_load_5d_u(d, &tmA, bar, x0[q] + i * lo_c, x1[q], x2[q], x3[q], n);
            }
          }
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if (p.nrbuf > 0 && !load_b) {
        // residual chunks of this tile (bf16, same box as the output chunks), consumed in order by the epilogue
        const int ncols = min(BN, p.Cout - n_base);
        for (int cc = 0; cc < ncols; cc += 64) {
          mbar_wait(&r_empty[rslot], rphase ^ 1);
          if (elect_one()) {
            const uint32_t bar = smem_u32(&r_full[rslot]);
            const uint32_t rbytes = p.res_up ? p.a_bytes >> 2 : p.a_bytes;
            mbar_expect_tx_u(bar, SPLIT ? 2u * rbytes : rbytes);
            tma_load_5d_u(smem_u32(rbuf) + rslot * rslot_bytes, &tmR, bar, n_base + cc, (tc.twi * p.TW) >> p.res_up,
                          (tc.thi * p.TH) >> p.res_up, tc.tti * p.TT, n);
            if (SPLIT)
              tma_load_5d_u(smem_u32(rbuf) + rslot * rslot_bytes + Cfg::C_BYTES, &tmR, bar, n_base + cc + p.res_lo_off,
                            (tc.twi * p.TW) >> p.res_up, (tc.thi * p.TH) >> p.res_up, tc.tti * p.TT, n);
          }
          if (++rslot == p.nrbuf) { rslot = 0; rphase ^= 1; }
        }
      }
    }
  } else if (warp == 2) {
    // ===================== TMA store warp =====================
    // Waits until all epilogue warps have staged a chunk (c_full), stores it (one elected lane, which also owns
    // the bulk async-groups) and hands staging slots back (c_free) once their store has read them out.  Keeping
    // this off the epilogue warps removes every block-wide barrier from the epilogue.
    constexpr bool split_out = SPLIT;
    const int CW = p.out_f32 ? 32 : 64;
    const int nslots = split_out ? p.ncbuf / 2 : p.ncbuf;     // split output: a slot is a (hi, lo) buffer pair
    const uint32_t slot_bytes = split_out ? 2u * Cfg::C_BYTES : (uint32_t)Cfg::C_BYTES;
    const uint32_t cbuf_u32 = smem_u32(cbuf);
    int slot = 0, prev_slot = 0; uint32_t sphase = 0;
    int issued = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord tc = decode_tile(p, tile);
      const int nbase = tc.nt * BN;
      const int ncols = min(BN, p.Cout - nbase);
      const int cw0 = tc.twi * p.TW, ch0 = tc.thi * p.TH, ct0 = tc.tti * p.TT, cn0 = tc.tbi * p.TB;
      for (int cc = 0; cc < ncols; cc += CW) {
        mbar_wait(&c_full[slot], sphase);
        if (elect_one()) {
          const uint32_t buf = cbuf_u32 + (uint32_t)slot * slot_bytes;
          tma_store_5d(&tmC, buf, nbase + cc, cw0, ch0, ct0, cn0);
          if (split_out) tma_store_5d(&tmC, buf + Cfg::C_BYTES, nbase + cc + p.out_lo_off, cw0, ch0, ct0, cn0);
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        // hand back the slot of the PREVIOUS chunk as soon as its store has read it out (at most this chunk's
        // store stays pending), so the epilogue warps may run nslots - 1 chunks ahead of the slowest one
        if (nslots == 1) {
          if (elect_one()) { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); mbar_arrive(&c_free[0]); }
        } else if (issued > 0) {
          if (elect_one()) { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); mbar_arrive(&c_free[prev_slot]); }
        }
        prev_slot = slot;
        ++issued;
        if (++slot == nslots) { slot = 0; sphase ^= 1; }
        __syncwarp();
      }
    }
    if (elect_one()) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  } else if (warp >= EPI_WARP0) {
    // ===================== consumers (warps 4..11): wgmma, then the epilogue =====================
    // Warpgroup g computes rows 64g .. 64g+63 of the tile.  Thread (warp q of its group, lane l) holds the accumulators
    // of rows 16q + l/4 and 16q + l/4 + 8 of that half, columns 8j + 2(l%4) + {0, 1} (wgmma.cuh).  The epilogue turns
    // each (row, column pair) into one 4-byte (bf16) / 8-byte (fp32) store into a 128B-swizzled staging chunk (the
    // eight rows of a warp hit eight different 16-byte units: conflict-free), which the store warp writes out by TMA.
    // The TMA store writes whole 128-byte lines and clips rows / channels outside the tensor, so ragged tiles need
    // no predication on the store side.
    const int wg = (warp - EPI_WARP0) >> 2;
    const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: row0 and row0 + 8
    const int cq = lane & 3;
    const bool out_f32 = p.out_f32 != 0;
    constexpr bool split_out = SPLIT;
    const bool relu = p.relu != 0;
    const int res_mode = p.res_mode;
    const int Cout = p.Cout;
    const int JPC = out_f32 ? 4 : 8;           // 8-column accumulator groups per 128-byte staged chunk
    const int nslots = split_out ? p.ncbuf / 2 : p.ncbuf;
    const uint32_t slot_bytes = split_out ? 2u * Cfg::C_BYTES : (uint32_t)Cfg::C_BYTES;
    const uint32_t cbuf_u32 = smem_u32(cbuf);
    const uint32_t rbuf_u32 = smem_u32(rbuf);
    const bool res_tma = p.nrbuf > 0;
    const bool res_ldg = res_mode != 0 && !res_tma;
    // per row i: position inside the tile, staging row offset and swizzle, residual ring row (top-down add: the row of
    // its parent position in the (TH/2 x TW/2) box of the coarser map)
    int tw_[2], th_[2], tl_[2], nl_[2];
    uint32_t srow[2], sswz[2], rrow[2], rswz[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      int rr = row0 + 8 * i;
      srow[i] = (uint32_t)rr * 128u; sswz[i] = (uint32_t)(rr & 7);
      tw_[i] = rr % p.TW; rr /= p.TW;
      th_[i] = rr % p.TH; rr /= p.TH;
      tl_[i] = rr % p.TT;
      nl_[i] = rr / p.TT;                      // >= TB for the unused tail rows of a short tile
      const int rp = p.res_up ? ((nl_[i] * p.TT + tl_[i]) * (p.TH >> 1) + (th_[i] >> 1)) * (p.TW >> 1) + (tw_[i] >> 1)
                              : row0 + 8 * i;
      rrow[i] = (uint32_t)rp * 128u; rswz[i] = (uint32_t)(rp & 7);
    }
    const float* __restrict__ g_scale = p.scale;
    const float* __restrict__ g_bias = p.bias;
    const uint32_t smem_u = smem_u32(smem) + (uint32_t)wg * (64u * 128u);   // this warpgroup's 64 rows of the A tile
    const uint32_t full_u = smem_u32(full);
    const int KS = p.ks;
    int stage = 0; uint32_t phase = 0;
    int rslot = 0; uint32_t rphase = 0;
    int slot = 0; uint32_t sphase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord tc = decode_tile(p, tile);
      // ---- main loop: one wgmma group per (tap, channel chunk) group; a ring stage goes back to the producers once
      // the wgmma group of the NEXT stage's last group is issued and the stage's own wgmma groups retired (one stage
      // stays in flight).  The wgmmas sit outside any branch so that they are not serialized.
      int prev = -1;
      for (int ki = 0; ki < groups; ++ki) {
        const int q = KS == 2 ? (ki & 1) : 0;          // group inside the ring stage
        if (q == 0) mbar_wait_u(full_u + stage * 8, phase);
        const uint32_t off = stage * stage_bytes + q * group_bytes;
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < NMMA; ++s) {
          // products in a fixed order: A_0 W_0, then A_1 W_0 (split), then A_0 W_1 (split, split conv1)
          const uint32_t ai = (NA == 2 && s == 1) ? 1u : 0u;
          const uint32_t bi = (NB == 2 && s == NMMA - 1) ? 1u : 0u;
          const uint64_t adesc = make_sw128_desc(smem_u + off + ai * Cfg::A_BYTES);
          const uint64_t bdesc = make_sw128_desc(smem_u32(smem) + off + NA * Cfg::A_BYTES + bi * Cfg::B_BYTES);
#pragma unroll
          for (int k = 0; k < 4; ++k)                  // 4 x 32 B = one 128-byte swizzle row of K
            wgmma<BN, KIND>(acc, adesc + 2 * k, bdesc + 2 * k, (ki | s | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        if (q == KS - 1 || ki == groups - 1) {
          if (q == 1) wgmma_wait<2>(); else wgmma_wait<1>();   // only this stage's q + 1 groups may still run
          if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
          prev = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);

      // ---- epilogue
      bool valid[2] = {true, true};
      size_t rpos[2] = {0, 0};
      if (res_ldg) {                           // per-thread residual rows (fp32 / upsample-add paths only)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int ho = tc.thi * p.TH + th_[i], wo = tc.twi * p.TW + tw_[i];
          const int t = tc.tti * p.TT + tl_[i], n = tc.tbi * p.TB + nl_[i];
          valid[i] = (nl_[i] < p.TB) && (ho < p.Ho) && (wo < p.Wo) && (t < p.To) && (n < p.N);
          rpos[i] = (res_mode == 2) ? ((size_t)(n * p.To + t) * (p.Ho >> 1) + (ho >> 1)) * (p.Wo >> 1) + (wo >> 1)
                                    : ((size_t)(n * p.To + t) * p.Ho + ho) * p.Wo + wo;
        }
      }
      const int nbase = tc.nt * BN;
      const int ncols = min(BN, Cout - nbase);     // live output columns of this tile
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        if (8 * j >= ncols) break;
        const int jc = j % JPC;                    // 8-column group inside the staged chunk
        const int col = nbase + 8 * j + 2 * cq;    // first of this thread's two output channels
        if (jc == 0) {
          // chunk start: the staging slot must have been read out by the TMA store that used it last (c_free), and
          // the producer's residual chunk must have landed
          mbar_wait(&c_free[slot], sphase ^ 1);
          if (res_tma) mbar_wait(&r_full[rslot], rphase);
        }
        float sc0 = 1.f, sc1 = 1.f, bi0 = 0.f, bi1 = 0.f;
        if (col + 2 <= Cout) {
          if (g_scale) { const float2 s2 = __ldg(reinterpret_cast<const float2*>(g_scale + col)); sc0 = s2.x; sc1 = s2.y; }
          if (g_bias) { const float2 b2 = __ldg(reinterpret_cast<const float2*>(g_bias + col)); bi0 = b2.x; bi1 = b2.y; }
        } else if (col < Cout) {                   // ragged channel tail
          if (g_scale) sc0 = __ldg(g_scale + col);
          if (g_bias) bi0 = __ldg(g_bias + col);
        }
        const uint32_t dst_slot = cbuf_u32 + (uint32_t)slot * slot_bytes;
        const uint32_t src_slot = rbuf_u32 + (uint32_t)rslot * rslot_bytes;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float v0 = fmaf(acc[4 * j + 2 * i], sc0, bi0);
          float v1 = fmaf(acc[4 * j + 2 * i + 1], sc1, bi1);
          if (out_f32) {
            if (res_mode != 0 && valid[i]) {
              const float* rp = reinterpret_cast<const float*>(p.residual) + rpos[i] * p.res_ld + col;
              if (col + 2 <= Cout) {
                const float2 q = __ldg(reinterpret_cast<const float2*>(rp));
                v0 += q.x; v1 += q.y;
                if (split_out) {                                     // residual = hi + lo
                  const float2 ql = __ldg(reinterpret_cast<const float2*>(rp + p.res_lo_off));
                  v0 += ql.x; v1 += ql.y;
                }
              } else if (col < Cout) {
                v0 += __ldg(rp) + (split_out ? __ldg(rp + p.res_lo_off) : 0.f);
              }
            }
            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            // 8 bytes at chunk column 8 jc + 2 cq: 16-byte unit 2 jc + cq / 2, offset 8 (cq & 1)
            const uint32_t off = ((((uint32_t)(2 * jc + (cq >> 1))) ^ sswz[i]) << 4) + 8u * (cq & 1);
            const uint32_t dst = dst_slot + srow[i] + off;
            if (split_out) {
              const float h0 = round_to_tf32(v0), h1 = round_to_tf32(v1);
              sts_f2(dst + Cfg::C_BYTES, round_to_tf32(v0 - h0), round_to_tf32(v1 - h1));   // lo: the slot's second buffer
              v0 = h0; v1 = h1;
            } else if (p.round_tf32) {
              v0 = round_to_tf32(v0); v1 = round_to_tf32(v1);
            }
            sts_f2(dst, v0, v1);
          } else {
            // 4 bytes at chunk column 8 jc + 2 cq: 16-byte unit jc, offset 4 cq
            if (res_tma) {
              const uint32_t src = src_slot + rrow[i] + ((((uint32_t)jc) ^ rswz[i]) << 4) + 4u * cq;
              uint32_t r2 = lds_b1(src);
              v0 += __uint_as_float(r2 << 16); v1 += __uint_as_float(r2 & 0xffff0000u);
              if (SPLIT) { r2 = lds_b1(src + Cfg::C_BYTES); v0 += __uint_as_float(r2 << 16); v1 += __uint_as_float(r2 & 0xffff0000u); }
            } else if (res_ldg && valid[i]) {
              const __nv_bfloat16* rp = reinterpret_cast<const __nv_bfloat16*>(p.residual) + rpos[i] * p.res_ld + col;
              if (col + 2 <= Cout) {
                uint32_t r2 = __ldg(reinterpret_cast<const unsigned int*>(rp));
                v0 += __uint_as_float(r2 << 16); v1 += __uint_as_float(r2 & 0xffff0000u);
                if (SPLIT) {                                          // residual = hi + lo (bf16 pairs)
                  r2 = __ldg(reinterpret_cast<const unsigned int*>(rp + p.res_lo_off));
                  v0 += __uint_as_float(r2 << 16); v1 += __uint_as_float(r2 & 0xffff0000u);
                }
              } else if (col < Cout) {
                v0 += __bfloat162float(rp[0]) + (SPLIT ? __bfloat162float(rp[p.res_lo_off]) : 0.f);
              }
            }
            const uint32_t dst = dst_slot + srow[i] + ((((uint32_t)jc) ^ sswz[i]) << 4) + 4u * cq;
            if (split_out) {
              // bf16 pair storage: hi = bf16(v), lo = bf16(v - hi) (v - hi is exact in fp32); hi + lo carries 16
              // mantissa bits, which three bf16 MMAs per k-block turn into an fp32-accurate product
              if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
              const uint32_t h = pack_bf16x2(v0, v1);
              sts_b1(dst + Cfg::C_BYTES, pack_bf16x2(v0 - __uint_as_float(h << 16), v1 - __uint_as_float(h & 0xffff0000u)));
              sts_b1(dst, h);
            } else {
              sts_b1(dst, relu ? pack_bf16x2_relu(v0, v1) : pack_bf16x2(v0, v1));
            }
          }
        }
        if (jc == JPC - 1 || 8 * (j + 1) >= ncols) {
          // chunk complete: hand the residual slot back, then generic-proxy smem writes -> visible to the async
          // proxy, then this warp's arrival on the staging slot
          if (res_tma) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&r_empty[rslot]);
            if (++rslot == p.nrbuf) { rslot = 0; rphase ^= 1; }
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) mbar_arrive(&c_full[slot]);
          if (++slot == nslots) { slot = 0; sphase ^= 1; }
        }
      }
    }
  }
}

// ------------------------------------------------------------------ host side (encode_map: tc_common.cuh)
// M tile = TB images x TT frames x TH x TW output positions (<= 128 rows).  Small feature maps (14x14 RoI
// heads, 25x42 res5) would waste a quarter of every 128-row MMA with purely spatial tiles; stacking frames /
// images fills the rows.  Among the shapes within 4 % of the best useful-row fraction a purely spatial tile
// wins (the fullest, then the widest); otherwise the widest stacked tile (longest runs per TMA box).
struct TileShape { int th, tw, tt, tb; };
static TileShape pick_tile(int Ho, int Wo, int To, int N, int max_w, int max_h, bool stack_t) {
  TileShape best = {8, 16, 1, 1};
  double best_eff = -1;
  long best_rank = -1;
  for (int pass = 0; pass < 2; ++pass)
    for (int tw = 1; tw <= 128 && tw <= max_w && tw <= Wo; ++tw)
      for (int th = 1; th * tw <= 128 && th <= max_h && th <= Ho; ++th) {
        const int rem = 128 / (tw * th);
        for (int tt = 1; tt <= rem && tt <= To && (tt == 1 || stack_t); ++tt)
          for (int tb = 1; tb * tt <= rem && tb <= N; ++tb) {
            const double tiles = (double)cdiv(Wo, tw) * cdiv(Ho, th) * cdiv(To, tt) * cdiv(N, tb);
            const double eff = (double)Ho * Wo * To * N / (tiles * 128.0);
            if (pass == 0) { if (eff > best_eff) best_eff = eff; continue; }
            if (eff < best_eff - 0.04) continue;
            const bool plain = tt == 1 && tb == 1;
            const long e = (long)(eff * 1e6);
            const long rank = plain ? (1L << 40) + e * 1000L + tw : (long)tw * 10000000L + e;
            if (rank > best_rank) { best_rank = rank; best = {th, tw, tt, tb}; }
          }
      }
  return best;
}

// Output map: dims (Cout, Wo, Ho, To, N) of the NDHWC result, box = one staged chunk (128 B of channels x one M tile).
static int encode_out_map(CUtensorMap* m, void* y, int out_f32, int Cout, int Wo, int Ho, int To, int N, int out_ld,
                          const TileShape& ts, bool time_major = false) {
  const uint64_t oesz = out_f32 ? 4 : 2;
  uint64_t d[5] = {(uint64_t)Cout, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)To, (uint64_t)N};
  const uint64_t frame = (uint64_t)out_ld * oesz * Wo * Ho;
  uint64_t st[4] = {(uint64_t)out_ld * oesz, (uint64_t)out_ld * oesz * Wo, time_major ? frame * N : frame,
                    time_major ? frame : frame * To};
  uint32_t b[5] = {(uint32_t)(128 / oesz), (uint32_t)ts.tw, (uint32_t)ts.th, (uint32_t)ts.tt, (uint32_t)ts.tb};
  uint32_t e[5] = {1, 1, 1, 1, 1};
  return encode_map(m, out_f32 != 0 ? 1 : 0, 5, y, d, st, b, e);
}

// What a descriptor launches, derived in one place for dt_conv3d and dt_conv_plan (the plan is what runs).
// The descriptor's dtype and shape must have been validated by the caller.
struct ConvGeom {
  int To_full, To, Ho, Wo;
  bool tf32, pointwise;
  int BK;                      // elements per 128-byte k-block
  TileShape ts;
  int BN;                      // column tile
  bool split_in, split_out;
  int kchunks, groups, nmma;   // (tap, channel chunk) groups per tile, MMA k-blocks per group
  bool res_tma;                // bf16 residual chunks arrive through the TMA ring
  bool res_up;                 // ... as the (TH/2 x TW/2) box of the coarser map of the FPN top-down add
};
static ConvGeom conv_geom(const dt_conv_desc* d, bool residual_aligned) {
  ConvGeom g;
  g.tf32 = d->dtype == DT_DTYPE_TF32;
  g.BK = g.tf32 ? 32 : 64;
  g.To_full = (d->Ti + 2 * d->pT - d->kT) / d->sT + 1;
  g.To = d->out_t_count > 0 ? d->out_t_count : g.To_full;
  g.Ho = (d->Hi + 2 * d->pH - d->kH) / d->sH + 1;
  g.Wo = (d->Wi + 2 * d->pW - d->kW) / d->sW + 1;
  // stacking frames inside one TMA box needs unit temporal stride (pointwise convs fold strides into the map)
  g.pointwise = d->kT == 1 && d->kH == 1 && d->kW == 1 && d->pT == 0 && d->pH == 0 && d->pW == 0;
  g.ts = pick_tile(g.Ho, g.Wo, g.To, d->N, g.pointwise ? 256 : 256 / d->sW, g.pointwise ? 256 : 256 / d->sH,
                   g.pointwise || d->sT == 1);
  // each consumer warpgroup keeps a 64 x BN fp32 accumulator in registers: BN / 2 per thread, so 128 is the widest
  // column tile that leaves the epilogue room under the 168-register cap of a 384-thread CTA
  g.BN = d->Cout > 64 ? 128 : (d->Cout > 32 ? 64 : 32);
  g.split_in = (d->x3 & 1) != 0;
  g.split_out = (d->x3 & 2) != 0;
  g.kchunks = cdiv(d->Cin, g.BK);
  g.groups = d->kT * d->kH * d->kW * g.kchunks;
  g.nmma = g.split_in ? 3 : 1;                         // launch_conv: split operands take three products per group
  // bf16 same-shape residual: its chunks are prefetched by TMA into a shared-memory ring (coalesced 128-byte
  // rows instead of 4-byte global loads per thread pair).
  // The FPN top-down add (res_mode 2) goes the same way when the tile is even-sized (tile origins are then even
  // too): the (TH/2 x TW/2) box of the coarser map is loaded and each row serves its four children.
  const bool res_even = (g.ts.th % 2 == 0) && (g.ts.tw % 2 == 0);
  g.res_tma = (d->res_mode == 1 || (d->res_mode == 2 && res_even)) && !d->out_f32 && !g.tf32 && residual_aligned;
  g.res_up = g.res_tma && d->res_mode == 2;
  return g;
}

template <int BN, int KIND, bool SPLIT, int NMMA>
static int launch_conv1(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const CUtensorMap& tmR,
                       const ConvKernelParams& p, int grid, cudaStream_t stream) {
  using Cfg = ConvCfg<BN>;
  static DynSmemGrant grant;
  DT_CHECK_CUDA(grant_dyn_smem(conv_tc_kernel<BN, KIND, SPLIT, NMMA>, Cfg::BUDGET, &grant));
  ConvKernelParams q = p;
  const int groups = p.kT * p.kH * p.kW * p.kchunks;
  DT_CHECK_ARG(groups <= 2048, "conv: %d (tap, channel chunk) groups per tile exceed the schedule table", groups);
  Cfg::split(groups, NMMA, p.nrbuf > 0, p.split_out != 0, p.out_f32 != 0, &q.nstages, &q.ks, &q.ncbuf, &q.nrbuf);
  q.ktab = (groups + 2) & ~1;
  const int smem = Cfg::smem_bytes(groups, NMMA, q.nstages, q.ks, q.ncbuf, q.nrbuf, p.split_out != 0);
  DT_CHECK_ARG(q.nstages >= 2 && smem <= Cfg::BUDGET, "conv: smem split failed (%d stages, %d B)", q.nstages, smem);
  // DT_PDL=1 in the environment launches with programmatic stream serialization (the kernel waits on griddepcontrol
  // before its first global access).  Plain stream order is the default: inside the captured CUDA graph of a step
  // there are no launch gaps left for it to hide.
  static const bool pdl = [] { const char* e = getenv("DT_PDL"); return e && e[0] == '1'; }();
  cudaLaunchConfig_t lc;
  memset(&lc, 0, sizeof(lc));
  lc.gridDim = dim3((unsigned)grid); lc.blockDim = dim3(CONV_THREADS); lc.dynamicSmemBytes = (size_t)smem; lc.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = at; lc.numAttrs = pdl ? 1 : 0;
  DT_CHECK_CUDA(cudaLaunchKernelEx(&lc, conv_tc_kernel<BN, KIND, SPLIT, NMMA>, tmA, tmB, tmC, tmR, q));
  return 0;
}

template <int BN, int KIND, int NMMA>
static int launch_conv2(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const CUtensorMap& tmR,
                        const ConvKernelParams& p, int grid, cudaStream_t stream) {
  return p.split_out ? launch_conv1<BN, KIND, true, NMMA>(tmA, tmB, tmC, tmR, p, grid, stream)
                     : launch_conv1<BN, KIND, false, NMMA>(tmA, tmB, tmC, tmR, p, grid, stream);
}

// operand kind from the descriptor: tf32, else ab_format (1 bf16, 0 fp16); split operands (bf16 or tf32 pairs) take
// three MMA k-blocks per group
template <int BN>
static int launch_conv(bool tf32, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const CUtensorMap& tmR,
                       const ConvKernelParams& p, int grid, cudaStream_t stream) {
  if (p.split_in) return tf32 ? launch_conv2<BN, 2, 3>(tmA, tmB, tmC, tmR, p, grid, stream)
                              : launch_conv2<BN, 0, 3>(tmA, tmB, tmC, tmR, p, grid, stream);
  if (tf32) return launch_conv2<BN, 2, 1>(tmA, tmB, tmC, tmR, p, grid, stream);
  return p.ab_format == 0 ? launch_conv2<BN, 1, 1>(tmA, tmB, tmC, tmR, p, grid, stream)
                          : launch_conv2<BN, 0, 1>(tmA, tmB, tmC, tmR, p, grid, stream);
}

}  // namespace dt

using namespace dt;

extern "C" int dt_conv3d(const dt_conv_desc* d, const void* x, const void* w, const float* scale, const float* bias,
                         const void* residual, void* y, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  DT_CHECK_ARG(d != nullptr, "dt_conv3d: null descriptor");
  DT_CHECK_ARG(d->dtype == DT_DTYPE_BF16 || d->dtype == DT_DTYPE_TF32 || d->dtype == DT_DTYPE_F16, "dt_conv3d: dtype %d not in {BF16, TF32, F16}", d->dtype);
  const bool f16 = d->dtype == DT_DTYPE_F16;          // fp16 x and w (11-bit operands, one MMA per product); outputs stay bf16 / fp32
  DT_CHECK_ARG(!f16 || (!(d->x3 & 1) && d->res_mode == 0), "dt_conv3d: DT_DTYPE_F16 inputs are plain rows and take no residual");
  DT_CHECK_ARG(d->N >= 1 && d->Ti >= 1 && d->Hi >= 1 && d->Wi >= 1 && d->Cin >= 1 && d->Cout >= 1,
               "dt_conv3d: bad input shape N=%d T=%d H=%d W=%d Cin=%d Cout=%d", d->N, d->Ti, d->Hi, d->Wi, d->Cin, d->Cout);
  DT_CHECK_ARG(d->kT >= 1 && d->kH >= 1 && d->kW >= 1 && d->sT >= 1 && d->sH >= 1 && d->sW >= 1 && d->pT >= 0 &&
                   d->pH >= 0 && d->pW >= 0, "dt_conv3d: bad filter geometry");
  const ConvGeom g = conv_geom(d, ((uintptr_t)residual % 16) == 0);
  const bool tf32 = g.tf32;
  const int in_dt = tf32 ? 1 : (f16 ? 2 : 0);
  const int esz = tf32 ? 4 : 2;
  const int BK = g.BK;
  const int To_full = g.To_full;
  DT_CHECK_ARG(d->out_t_first >= 0 && d->out_t_count >= 0 && d->out_t_first + d->out_t_count <= (To_full > 0 ? To_full : 0),
               "dt_conv3d: output frame range [%d, +%d) outside the %d output frames", d->out_t_first, d->out_t_count, To_full);
  DT_CHECK_ARG(d->out_t_count == 0 || d->res_mode == 0, "dt_conv3d: an output frame range cannot be combined with a residual");
  const int To = g.To, Ho = g.Ho, Wo = g.Wo;
  DT_CHECK_ARG(To >= 1 && Ho >= 1 && Wo >= 1, "dt_conv3d: empty output (%d,%d,%d)", To, Ho, Wo);
  const int in_ld = d->in_ld > 0 ? d->in_ld : d->Cin;
  const int w_ld = d->w_ld > 0 ? d->w_ld : d->Cin;
  const int out_ld = d->out_ld > 0 ? d->out_ld : d->Cout;
  const int res_ld = d->res_ld > 0 ? d->res_ld : d->Cout;
  DT_CHECK_ARG((in_ld * esz) % 16 == 0 && (w_ld * esz) % 16 == 0,
               "dt_conv3d: channel strides must be multiples of 16 bytes (in_ld=%d, w_ld=%d, %d B/elem)", in_ld, w_ld, esz);
  DT_CHECK_ARG(in_ld >= d->Cin && w_ld >= d->Cin && out_ld >= d->Cout, "dt_conv3d: leading dims smaller than channels");
  DT_CHECK_ARG(x && w && y, "dt_conv3d: null tensor pointer");
  DT_CHECK_ARG(((uintptr_t)x % 16) == 0 && ((uintptr_t)w % 16) == 0 && ((uintptr_t)y % 16) == 0,
               "dt_conv3d: tensors must be 16-byte aligned");
  DT_CHECK_ARG(d->res_mode >= 0 && d->res_mode <= 2 && (d->res_mode == 0 || residual), "dt_conv3d: bad residual mode/pointer");
  DT_CHECK_ARG(d->res_mode != 2 || (Ho % 2 == 0 && Wo % 2 == 0), "dt_conv3d: upsample-add needs even output size, got %dx%d", Ho, Wo);
  const int out_f32 = d->out_f32;
  const int oesz = out_f32 ? 4 : 2;
  // vector stores need 16-byte aligned rows
  DT_CHECK_ARG((out_ld * oesz) % 16 == 0 && (d->res_mode == 0 || (res_ld * oesz) % 16 == 0),
               "dt_conv3d: out_ld/res_ld rows must be 16-byte multiples");

  const bool pointwise = g.pointwise;
  const TileShape ts = g.ts;
  const int TH = ts.th, TW = ts.tw;
  ConvKernelParams p;
  memset(&p, 0, sizeof(p));
  p.N = d->N; p.To = To; p.Ho = Ho; p.Wo = Wo; p.Cout = d->Cout;
  p.kT = d->kT; p.kH = d->kH; p.kW = d->kW; p.pT = d->pT; p.pH = d->pH; p.pW = d->pW;
  p.sT = d->sT; p.sH = d->sH; p.sW = d->sW;
  p.kchunks = g.kchunks;
  p.TH = TH; p.TW = TW; p.TT = ts.tt; p.TB = ts.tb;
  p.tiles_h = cdiv(Ho, TH); p.tiles_w = cdiv(Wo, TW); p.tiles_t = cdiv(To, ts.tt); p.tiles_b = cdiv(d->N, ts.tb);
  p.a_bytes = (uint32_t)(TH * TW * ts.tt * ts.tb) * 128u;
  p.scale = scale; p.bias = bias; p.residual = residual; p.res_mode = d->res_mode; p.res_ld = res_ld;
  p.relu = d->relu; p.out_f32 = out_f32; p.round_tf32 = d->out_round_tf32;
  // 3xTF32 split operands / outputs
  p.split_in = g.split_in ? 1 : 0;
  p.split_out = g.split_out ? 1 : 0;
  p.ab_format = f16 ? 0 : 1;
  DT_CHECK_ARG(!p.split_in || d->Cin % BK == 0, "dt_conv3d: x3 inputs need Cin %% %d == 0 (Cin=%d)", BK, d->Cin);
  DT_CHECK_ARG(!p.split_out || ((tf32 ? out_f32 : !out_f32) && d->Cout % (out_f32 ? 32 : 64) == 0),
               "dt_conv3d: x3 outputs are fp32 pairs (TF32) / bf16 pairs (BF16) with Cout %% %d == 0 (Cout=%d)", out_f32 ? 32 : 64, d->Cout);
  p.a_lo_off = d->in_lo_off > 0 ? d->in_lo_off : in_ld / 2;
  p.b_lo_off = w_ld / 2;
  p.out_lo_off = d->out_lo_off > 0 ? d->out_lo_off : out_ld / 2;
  p.res_lo_off = d->res_lo_off > 0 ? d->res_lo_off : res_ld / 2;
  DT_CHECK_ARG(!p.split_in || (p.a_lo_off + d->Cin <= in_ld && p.b_lo_off >= d->Cin), "dt_conv3d: x3 lo halves do not fit the rows");
  DT_CHECK_ARG(!p.split_out || p.out_lo_off + d->Cout <= out_ld, "dt_conv3d: x3 output lo half does not fit the row");

  const int BN = g.BN;
  const bool res_tma = g.res_tma;
  p.t_first = d->out_t_count > 0 ? d->out_t_first : 0;
  p.nrbuf = res_tma ? 1 : 0;                         // ring depth is chosen with the smem split at launch
  p.res_up = g.res_up ? 1 : 0;
  p.tiles_n = cdiv(d->Cout, BN);
  p.fd_n = make_fastdiv(p.tiles_n); p.fd_w = make_fastdiv(p.tiles_w); p.fd_h = make_fastdiv(p.tiles_h); p.fd_t = make_fastdiv(p.tiles_t);
  const long long total = (long long)p.tiles_b * p.tiles_t * p.tiles_h * p.tiles_w * p.tiles_n;
  DT_CHECK_ARG(total < (1ll << 31), "dt_conv3d: too many tiles");
  p.total_tiles = (int)total;

  // ---- tensor maps -------------------------------------------------------------
  // A: dims (C, W, H, T, N) of the NDHWC input.  Pointwise strided convs (1x1x1, stride s, no
  // padding) fold the stride into the global strides so no element-stride traversal is needed;
  // other strided convs use TMA element strides (box covers s*TW input columns, every s-th kept).
  CUtensorMap tmA, tmB;
  uint64_t dims[5], strides[4]; uint32_t box[5], estr[5] = {1, 1, 1, 1, 1};
  const uint64_t sC = (uint64_t)in_ld * esz, sW = sC * d->Wi, sH = sW * d->Hi, sT = sH * d->Ti;
  const uint64_t cdim = p.split_in ? (uint64_t)in_ld : (uint64_t)d->Cin;
  if (pointwise) {
    dims[0] = cdim; dims[1] = Wo; dims[2] = Ho; dims[3] = To_full; dims[4] = d->N;
    strides[0] = sC * d->sW; strides[1] = sW * d->sH; strides[2] = sH * d->sT; strides[3] = sT;
    box[0] = BK; box[1] = TW; box[2] = TH; box[3] = ts.tt; box[4] = ts.tb;
    p.sT = p.sH = p.sW = 1;
  } else {
    dims[0] = cdim; dims[1] = d->Wi; dims[2] = d->Hi; dims[3] = d->Ti; dims[4] = d->N;
    strides[0] = sC; strides[1] = sW; strides[2] = sH; strides[3] = sT;
    box[0] = BK; box[1] = (uint32_t)TW * d->sW; box[2] = (uint32_t)TH * d->sH; box[3] = ts.tt; box[4] = ts.tb;
    estr[1] = d->sW; estr[2] = d->sH;
    DT_CHECK_ARG(box[1] <= 256 && box[2] <= 256, "dt_conv3d: strided tile too large for a TMA box");
  }
  if (encode_map(&tmA, in_dt, 5, x, dims, strides, box, estr)) return 1;
  {
    const int taps = d->kT * d->kH * d->kW;
    uint64_t wd[3] = {p.split_in ? (uint64_t)w_ld : (uint64_t)d->Cin, (uint64_t)d->Cout, (uint64_t)taps};
    uint64_t ws[2] = {(uint64_t)w_ld * esz, (uint64_t)w_ld * esz * d->Cout};
    uint32_t wb[3] = {(uint32_t)BK, (uint32_t)BN, 1};
    uint32_t we[3] = {1, 1, 1};
    if (encode_map(&tmB, in_dt, 3, w, wd, ws, wb, we)) return 1;
  }
  CUtensorMap tmC, tmR;
  if (encode_out_map(&tmC, y, out_f32, p.split_out ? out_ld : d->Cout, Wo, Ho, To, d->N, out_ld, ts, d->out_time_major != 0)) return 1;
  if (res_tma && p.res_up) {
    const TileShape half = {ts.th / 2, ts.tw / 2, ts.tt, ts.tb};
    if (encode_out_map(&tmR, const_cast<void*>(residual), 0, p.split_out ? res_ld : d->Cout, Wo / 2, Ho / 2, To, d->N, res_ld, half)) return 1;
  } else if (res_tma) {
    if (encode_out_map(&tmR, const_cast<void*>(residual), 0, p.split_out ? res_ld : d->Cout, Wo, Ho, To, d->N, res_ld, ts)) return 1;
  } else {
    tmR = tmC;
  }
  int dev = 0, sms = 0;
  DT_CHECK_CUDA(cudaGetDevice(&dev));
  DT_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
#define DT_LAUNCH(BNv)                                                                      \
  return launch_conv<BNv>(tf32, tmA, tmB, tmC, tmR, p, grid, stream)
  switch (BN) {
    case 128: DT_LAUNCH(128);
    case 64: DT_LAUNCH(64);
    default: DT_LAUNCH(32);
  }
#undef DT_LAUNCH
}


// Planning query: the choices of dt_conv3d above (conv_geom, then the smem split of launch_conv1) without touching the
// device, so that the host logic is testable without a GPU (tests/test_conv_plan.py).
template <int BN>
static void plan_split(int groups, int nmma, bool res_tma, bool split_out, bool out_f32, dt_conv_plan_t* o) {
  using Cfg = ConvCfg<BN>;
  Cfg::split(groups, nmma, res_tma, split_out, out_f32, &o->stages, &o->ks, &o->ncbuf, &o->nrbuf);
  o->smem_bytes = Cfg::smem_bytes(groups, nmma, o->stages, o->ks, o->ncbuf, o->nrbuf, split_out);
  o->stage_bytes = o->ks * Cfg::group_bytes(nmma);
}

extern "C" int dt_conv_plan(const dt_conv_desc* d, int residual_aligned, dt_conv_plan_t* o) {
  DT_CHECK_ARG(d != nullptr && o != nullptr, "dt_conv_plan: null pointer");
  DT_CHECK_ARG(d->dtype == DT_DTYPE_BF16 || d->dtype == DT_DTYPE_TF32 || d->dtype == DT_DTYPE_F16,
               "dt_conv_plan: dtype %d not in {BF16, TF32, F16}", d->dtype);
  DT_CHECK_ARG(d->N >= 1 && d->Ti >= 1 && d->Hi >= 1 && d->Wi >= 1 && d->Cin >= 1 && d->Cout >= 1 && d->kT >= 1 && d->kH >= 1 &&
                   d->kW >= 1 && d->sT >= 1 && d->sH >= 1 && d->sW >= 1 && d->pT >= 0 && d->pH >= 0 && d->pW >= 0,
               "dt_conv_plan: bad shape");
  const ConvGeom g = conv_geom(d, residual_aligned != 0);
  DT_CHECK_ARG(g.To >= 1 && g.Ho >= 1 && g.Wo >= 1, "dt_conv_plan: empty output (%d,%d,%d)", g.To, g.Ho, g.Wo);
  const TileShape ts = g.ts;
  memset(o, 0, sizeof(*o));
  o->BN = g.BN; o->TH = ts.th; o->TW = ts.tw; o->TT = ts.tt; o->TB = ts.tb;
  o->kiters = g.groups * g.nmma;
  const long long mt = (long long)cdiv(g.Wo, ts.tw) * cdiv(g.Ho, ts.th) * cdiv(g.To, ts.tt) * cdiv(d->N, ts.tb);
  o->tiles = (int)(mt * cdiv(d->Cout, g.BN));
  o->useful_rows = (double)g.Ho * g.Wo * g.To * d->N / ((double)mt * 128.0);
  switch (g.BN) {
    case 128: plan_split<128>(g.groups, g.nmma, g.res_tma, g.split_out, d->out_f32 != 0, o); break;
    case 64: plan_split<64>(g.groups, g.nmma, g.res_tma, g.split_out, d->out_f32 != 0, o); break;
    default: plan_split<32>(g.groups, g.nmma, g.res_tma, g.split_out, d->out_f32 != 0, o); break;
  }
  return 0;
}


// conv1 of the ResNet bodies: 7x7 stride 2 pad 3 on a 3-channel image (lib/modeling/ResNet3D.py:258-261,
// ResNet.py).  With Cin = 3 a per-tap k-block would waste 61/64 of every MMA, so the taps of one filter
// ROW are packed into K instead: the image blob is channel-padded to Cp (8 bf16 / 4 fp32 = 16 bytes per
// pixel) and carries physical zero borders (3 rows top/bottom, 4 pixels left/right, written by
// dt_prep_clip), so the 7-pixel window of output column wo is ONE contiguous 112-byte run starting at
// padded pixel 2*wo + 1.  The A tensor map is an overlapping strided view
//   dim0 = 8 pixels x Cp (128 B, the 8th pixel meets zero weights), dim1 = wo (stride 2 pixels = 32 B),
//   dim2 = rows of one parity plane, dim3 = plane, dim4 = frames
// (the blob's padded rows are de-interleaved by parity, so the stride-2 row walk of filter row kh is a
// unit-stride box in plane kh & 1 starting at row ho + (kh >> 1); TMA element strides halve its throughput)
// and the conv is 7 k-blocks (one per filter row) of K = 128 bytes: 3*7/ (8*8) = 33 % useful MACs instead
// of 4.7 %.  w [7][Cout][8*Cp] (kw-major, channel-minor).  y [F, Hp/2, Wp/2, out_ld].
extern "C" int dt_conv1_7x7s2(const void* x_padded, int F, int Hp, int Wp, int Cp, const void* w, int Cout,
                              const float* scale, const float* bias, int relu, int dtype, int out_f32,
                              int out_round_tf32, int x3, void* y, int out_ld, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  DT_CHECK_ARG(dtype == DT_DTYPE_BF16 || dtype == DT_DTYPE_TF32, "dt_conv1_7x7s2: bad dtype %d", dtype);
  const bool tf32 = dtype == DT_DTYPE_TF32;
  const int esz = tf32 ? 4 : 2;
  DT_CHECK_ARG(Cp * esz == 16, "dt_conv1_7x7s2: the blob must carry 16 bytes per pixel (Cp=%d, %d B/elem)", Cp, esz);
  DT_CHECK_ARG(F >= 1 && Hp >= 2 && Wp >= 2 && Hp % 2 == 0 && Wp % 2 == 0 && Cout >= 1 && Cout <= 64,
               "dt_conv1_7x7s2: bad shape F=%d Hp=%d Wp=%d Cout=%d", F, Hp, Wp, Cout);
  DT_CHECK_ARG(x_padded && w && y, "dt_conv1_7x7s2: null pointer");
  // x3 (bf16 only): the blob pixel is [hi(3) | lo(3) | 0 0] (dt_prep_clip out mode 3), w holds 14 blocks
  // [2*kh]: [W_hi | W_hi] per pixel, [2*kh + 1]: [W_lo | 0], and y rows are [hi(Cout) | lo(Cout)] bf16 pairs
  DT_CHECK_ARG(!x3 || (!tf32 && !out_f32 && Cout == 64), "dt_conv1_7x7s2: x3 needs DT_DTYPE_BF16, bf16 pair output and Cout == 64");
  const int oesz = out_f32 ? 4 : 2;
  if (out_ld <= 0) out_ld = x3 ? 2 * Cout : Cout;
  DT_CHECK_ARG((out_ld * oesz) % 16 == 0 && out_ld >= (x3 ? 2 * Cout : Cout), "dt_conv1_7x7s2: bad out_ld %d", out_ld);
  const int Ho = Hp / 2, Wo = Wp / 2;
  const int BKe = 128 / esz;                       // elements per k-block
  const TileShape ts = pick_tile(Ho, Wo, 1, 1, 256, 128, false);      // spatial tiles only
  const int TH = ts.th, TW = ts.tw;
  ConvKernelParams p;
  memset(&p, 0, sizeof(p));
  p.N = F; p.To = 1; p.Ho = Ho; p.Wo = Wo; p.Cout = Cout;
  p.kT = 1; p.kH = 7; p.kW = 1; p.sT = 1; p.sH = 1; p.sW = 1; p.pT = 0; p.pH = 0; p.pW = 0;
  p.row_planes = 1;
  p.kchunks = 1;
  p.ab_format = 1;
  p.b_lo_blk = 1;                                  // x3: weight blocks 2*kh and 2*kh + 1 against one activation box
  p.split_out = x3 ? 1 : 0;
  p.out_lo_off = out_ld / 2;
  p.TH = TH; p.TW = TW; p.TT = 1; p.TB = 1; p.tiles_h = cdiv(Ho, TH); p.tiles_w = cdiv(Wo, TW); p.tiles_t = 1; p.tiles_b = F;
  p.tiles_n = 1;
  p.a_bytes = (uint32_t)TH * TW * 128u;
  p.scale = scale; p.bias = bias; p.relu = relu; p.out_f32 = out_f32;
  p.round_tf32 = out_round_tf32;
  p.fd_n = make_fastdiv(1); p.fd_w = make_fastdiv(p.tiles_w); p.fd_h = make_fastdiv(p.tiles_h); p.fd_t = make_fastdiv(1);
  const long long total = (long long)F * p.tiles_h * p.tiles_w;
  DT_CHECK_ARG(total < (1ll << 31), "dt_conv1_7x7s2: too many tiles");
  p.total_tiles = (int)total;
  // padded rows are stored de-interleaved (dt_prep_clip row_planes): filter row kh of output row ho reads
  // padded row 2*ho + kh = plane (kh & 1), plane row ho + (kh >> 1) -> unit-stride boxes, the plane is dim 3
  const uint64_t pix = 16, row = (uint64_t)(Wp + 8) * pix, plane = row * ((Hp + 6) / 2), frame = 2 * plane;
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[5] = {(uint64_t)BKe, (uint64_t)Wo, (uint64_t)((Hp + 6) / 2), 2, (uint64_t)F};
    uint64_t strides[4] = {2 * pix, row, plane, frame};
    uint32_t box[5] = {(uint32_t)BKe, (uint32_t)TW, (uint32_t)TH, 1, 1};
    uint32_t estr[5] = {1, 1, 1, 1, 1};
    if (encode_map(&tmA, tf32 ? 1 : 0, 5, (const char*)x_padded + pix, dims, strides, box, estr)) return 1;
  }
  {
    uint64_t wd[3] = {(uint64_t)BKe, (uint64_t)Cout, (uint64_t)(x3 ? 14 : 7)};
    uint64_t ws[2] = {128, (uint64_t)128 * Cout};
    uint32_t wb[3] = {(uint32_t)BKe, 64, 1};
    uint32_t we[3] = {1, 1, 1};
    if (encode_map(&tmB, tf32 ? 1 : 0, 3, w, wd, ws, wb, we)) return 1;
  }
  CUtensorMap tmC;
  if (encode_out_map(&tmC, y, out_f32, x3 ? out_ld : Cout, Wo, Ho, 1, F, out_ld, ts)) return 1;
  int dev = 0, sms = 0;
  DT_CHECK_CUDA(cudaGetDevice(&dev));
  DT_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  return x3 ? launch_conv1<64, 0, true, 2>(tmA, tmB, tmC, tmC, p, grid, stream)
            : launch_conv<64>(tf32, tmA, tmB, tmC, tmC, p, grid, stream);
}
