// Warp-parallel rectangular min-cost assignment in scipy.optimize.linear_sum_assignment's own visiting order, shared by
// the tracker (lsa.cu: the bbox-only cost in fp32 from shared memory, as the reference's matrix is float32; the combined
// pose-pck cost in fp64 read from global memory, as the reference's matrix is float64) and the PoseTrack CLEAR-MOT
// accumulator (poseval.cu, fp64 costs as py-motmetrics hands scipy the fp64 distances).
//
// It restates the rectangular shortest augmenting path algorithm (Crouse 2016) in the exact order scipy >= 1.6 walks it
// (see oracle/lsa.py, pinned live against the installed scipy):
//   - fp64 duals / path costs, r = ((minVal + c) - u[i]) - v[j]        (no FMA possible)
//   - remaining-column list filled in reverse, removal = swap with last
//   - column choice: strict '<' keeps the FIRST minimum in list order, but an equal-cost
//     UNASSIGNED column later in the list replaces it (so: last unassigned min if any,
//     else first min)
//   - nc < nr problems are solved on the transpose (by the caller).
// The 32 lanes split the remaining-column list (position it = lane, lane+32, ...); the
// sequential rule above is reproduced by a (min, first-pos, last-unassigned-pos) reduction.
#pragma once
#include <math_constants.h>

namespace dt {

template <typename T>
struct LsaSmemT {
  // carved from dynamic smem: dvec entries per vector, ncost cost entries
  T* C;             // [nr*nc] internal (row-major, nr <= nc)
  double* u;        // [dvec]
  double* v;        // [dvec]
  double* spc;      // [dvec]
  int* path;        // [dvec]
  int* col4row;     // [dvec]
  int* row4col;     // [dvec]
  int* remaining;   // [dvec]
  unsigned char* SR;  // [dvec]
  unsigned char* SC;  // [dvec]
};

template <typename T>
__host__ __device__ inline size_t lsa_smem_bytes_t(int dvec, size_t ncost) {
  size_t b = 0;
  b += (size_t)3 * dvec * sizeof(double);
  b += ncost * sizeof(T);
  b += (size_t)4 * dvec * sizeof(int);
  b += (size_t)2 * dvec;
  return (b + 15) / 16 * 16;
}

template <typename T>
__device__ __forceinline__ LsaSmemT<T> lsa_carve_t(unsigned char* base, int dvec, size_t ncost) {
  LsaSmemT<T> s;
  s.u = (double*)base;            base += (size_t)dvec * sizeof(double);
  s.v = (double*)base;            base += (size_t)dvec * sizeof(double);
  s.spc = (double*)base;          base += (size_t)dvec * sizeof(double);
  s.C = (T*)base;                 base += ncost * sizeof(T);
  s.path = (int*)base;            base += (size_t)dvec * sizeof(int);
  s.col4row = (int*)base;         base += (size_t)dvec * sizeof(int);
  s.row4col = (int*)base;         base += (size_t)dvec * sizeof(int);
  s.remaining = (int*)base;       base += (size_t)dvec * sizeof(int);
  s.SR = base;                    base += dvec;
  s.SC = base;
  return s;
}

// Internal (nr <= nc) matrix element (i, j) = C[i * rs + j * cs]: row-major in shared memory (rs = nc, cs = 1), or a
// caller's [P, ldc] matrix in global memory read as it is (rs = ldc, cs = 1) or transposed (rs = 1, cs = ldc).
template <typename T>
struct LsaRows {
  const T* C;
  size_t rs, cs;
  __device__ __forceinline__ const T* row(int i) const { return C + (size_t)i * rs; }
  __device__ __forceinline__ double at(const T* r, int j) const { return (double)r[(size_t)j * cs]; }
};

// The same with cs = 1 known at compile time (the shared-memory matrix).
template <typename T>
struct LsaDenseRows {
  const T* C;
  int nc;
  __device__ __forceinline__ const T* row(int i) const { return C + (size_t)i * nc; }
  __device__ __forceinline__ double at(const T* r, int j) const { return (double)r[j]; }
};

// Solve on the internal (nr <= nc) matrix `rows`.  All 32 lanes participate.
// On return col4row[i] (i < nr) holds the assignment.  Returns false if infeasible.
template <typename T, typename Rows>
__device__ bool lsa_solve_warp_rows(const LsaSmemT<T>& s, const Rows& rows, int nr, int nc) {
  const int lane = threadIdx.x & 31;
  const unsigned FULL = 0xffffffffu;
  for (int x = lane; x < nr; x += 32) { s.u[x] = 0.0; s.col4row[x] = -1; }
  for (int x = lane; x < nc; x += 32) { s.v[x] = 0.0; s.row4col[x] = -1; s.path[x] = -1; }
  __syncwarp();
  for (int cur = 0; cur < nr; ++cur) {
    for (int x = lane; x < nc; x += 32) { s.remaining[x] = nc - x - 1; s.spc[x] = CUDART_INF; s.SC[x] = 0; }
    for (int x = lane; x < nr; x += 32) s.SR[x] = 0;
    __syncwarp();
    double minVal = 0.0;
    int num_remaining = nc, sink = -1, i = cur;
    while (sink == -1) {
      if (lane == 0) s.SR[i] = 1;
      const double ui = s.u[i];
      const auto* ci = rows.row(i);
      double lmin = CUDART_INF;
      int lfirst = 0x7fffffff, lun = -1;
      for (int it = lane; it < num_remaining; it += 32) {
        const int j = s.remaining[it];
        const double r = __dsub_rn(__dsub_rn(__dadd_rn(minVal, rows.at(ci, j)), ui), s.v[j]);
        double sp = s.spc[j];
        if (r < sp) { s.path[j] = i; s.spc[j] = r; sp = r; }
        const bool un = (s.row4col[j] == -1);
        if (sp < lmin) { lmin = sp; lfirst = it; lun = un ? it : -1; }
        else if (sp == lmin && un) { lun = it; }
      }
      double m = lmin;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmin(m, __shfl_xor_sync(FULL, m, o));
      if (m == CUDART_INF) return false;              // infeasible (cannot happen for finite costs)
      int f = (lmin == m) ? lfirst : 0x7fffffff;
      int un = (lmin == m) ? lun : -1;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        f = min(f, __shfl_xor_sync(FULL, f, o));
        un = max(un, __shfl_xor_sync(FULL, un, o));
      }
      const int index = (un >= 0) ? un : f;
      minVal = m;
      const int j = s.remaining[index];
      const int r4c = s.row4col[j];
      if (r4c == -1) sink = j; else i = r4c;
      --num_remaining;
      __syncwarp();
      if (lane == 0) { s.SC[j] = 1; s.remaining[index] = s.remaining[num_remaining]; }
      __syncwarp();
    }
    // dual update (rectangular_lsap: "update dual variables")
    if (lane == 0) s.u[cur] = __dadd_rn(s.u[cur], minVal);
    for (int x = lane; x < nr; x += 32)
      if (s.SR[x] && x != cur) s.u[x] = __dadd_rn(s.u[x], __dsub_rn(minVal, s.spc[s.col4row[x]]));
    for (int x = lane; x < nc; x += 32)
      if (s.SC[x]) s.v[x] = __dsub_rn(s.v[x], __dsub_rn(minVal, s.spc[x]));
    __syncwarp();
    // augment along the path
    if (lane == 0) {
      int j = sink;
      while (true) {
        const int ii = s.path[j];
        s.row4col[j] = ii;
        const int tmp = s.col4row[ii];
        s.col4row[ii] = j;
        j = tmp;
        if (ii == cur) break;
      }
    }
    __syncwarp();
  }
  return true;
}

// Solve on the internal (nr <= nc) row-major matrix in s.C.
template <typename T>
__device__ bool lsa_solve_warp(const LsaSmemT<T>& s, int nr, int nc) {
  return lsa_solve_warp_rows(s, LsaDenseRows<T>{s.C, nc}, nr, nc);
}

}  // namespace dt
