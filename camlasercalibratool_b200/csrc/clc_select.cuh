// clc_select.cuh -- greedy D-optimal selection of the frames that carry the most information about the extrinsic
// (clc_select_frames, clc_select_frames_rows, clc_group_select_frames).
//
// The rule (include/clc_b200.h states it in full): H_f is frame f's H21 of the per-frame report, restricted to the d free
// coordinates of fixed_mask; T = sum H_f over the usable frames that are not excluded, D = diag(T)^-1/2, Ht_f = D H_f D;
// A_0 = sum of the forced frames' Ht_f + (kSelectRidge / n_T) I; at every step the candidate of largest
// gain_f = log det(I + L^-1 Ht_f L^-T) (A_s = L L^T) is picked (lowest index on a tie) and A_{s+1} = A_s + Ht_f.
//
// Every dense piece works on 6x6 matrices: the d free coordinates come first and the held ones are padded with zeros in Ht_f and
// with the identity in A, which leaves the free coordinates' Cholesky factors, solves and pivots bit for bit what a d x d
// computation gives and adds log1p(0) = 0 to every gain.  Device kernels, one selection:
//   1. clc_select_sum_kernel     per frame: usable (all 21 entries finite), its status and keep byte, its free block packed
//                                structure-of-arrays (d(d+1)/2 x n_frames); per block: the sums of T and of the forced blocks
//                                (a fixed warp-shuffle tree, then the warps in order);
//   2. clc_select_init_kernel    one block: the block sums in block order, the check of diag(T), D, A_0 and its factor L;
//   3. clc_select_scale_kernel   the packed blocks scaled to Ht_f in place;
//   4. clc_select_step_kernel    one greedy step per launch: every remaining candidate's gain, the block's best by (gain desc,
//                                index asc), and in the last block to arrive the grid's best, the stop rules and the update of
//                                A and L.  A launch after the selection has stopped returns at once.
// The CLC_HD part also compiles with g++ for the CPU tests (tests/select_harness.cpp).
#pragma once

#include "clc_math.cuh"

namespace clc {

constexpr double kSelectRidge = 1e-6;  // CLC_SELECT_RIDGE: A_0's ridge, in units of an average frame's scaled diagonal

// index of (i, j), i <= j, in the row-major upper triangle of a d x d matrix
CLC_HD int sel_tri(int d, int i, int j) { return i * d - (i * (i - 1)) / 2 + (j - i); }

// Cholesky A = L L^T of the symmetric 6x6 A (full, row-major): L lower triangular (row-major, zeros above the diagonal) and
// inv[k] = 1 / L_kk.  false when a pivot is not positive and finite.
CLC_HD bool sel_chol6(const double* A, double* L, double* inv) {
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double s = A[j * 6 + j];
#pragma unroll
    for (int k = 0; k < j; ++k) s -= L[j * 6 + k] * L[j * 6 + k];
    ok = ok && s > 0.0 && is_finite(s);
    const double r = sqrt(s);
    L[j * 6 + j] = r;
    inv[j] = 1.0 / r;
#pragma unroll
    for (int i = 0; i < j; ++i) L[i * 6 + j] = 0.0;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      double t = A[i * 6 + j];
#pragma unroll
      for (int k = 0; k < j; ++k) t -= L[i * 6 + k] * L[j * 6 + k];
      L[i * 6 + j] = t * inv[j];
    }
  }
  return ok;
}

// gain = log det(I + C), C = L^-1 H L^-T, for the symmetric 6x6 H (full, row-major) and the factor of sel_chol6.  The pivots of the
// Cholesky factorisation of I + C are 1 + u_k with u_k formed without the 1, and the gain is sum log1p(u_k) (= twice the sum of
// the logs of the factor's diagonal), so that a small gain keeps its relative precision.  -inf when a pivot is not positive and
// finite.
CLC_HD double sel_gain6(const double* L, const double* inv, const double* H) {
  double V[36];  // L^-1 H, column by column
#pragma unroll
  for (int c = 0; c < 6; ++c) {
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      double s = H[i * 6 + c];
#pragma unroll
      for (int k = 0; k < i; ++k) s -= L[i * 6 + k] * V[k * 6 + c];
      V[i * 6 + c] = s * inv[i];
    }
  }
  // C = L^-1 V^T; column j's entries 0..j (the upper triangle) need only the first j + 1 of its forward substitution
  double Cu[36];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
#pragma unroll
    for (int i = 0; i <= j; ++i) {
      double s = V[j * 6 + i];
#pragma unroll
      for (int k = 0; k < i; ++k) s -= L[i * 6 + k] * Cu[k * 6 + j];
      Cu[i * 6 + j] = s * inv[i];
    }
  }
  double R[36], rinv[6], gain = 0.0;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double u = Cu[j * 6 + j];
#pragma unroll
    for (int k = 0; k < j; ++k) u -= R[j * 6 + k] * R[j * 6 + k];
    const double piv = 1.0 + u;
    if (!(piv > 0.0) || !is_finite(piv)) return -HUGE_VAL;
    gain += log1p(u);
    const double r = sqrt(piv);
    rinv[j] = 1.0 / r;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      double t = Cu[j * 6 + i];
#pragma unroll
      for (int k = 0; k < j; ++k) t -= R[i * 6 + k] * R[j * 6 + k];
      R[i * 6 + j] = t * rinv[j];
    }
  }
  return gain;
}

// (gain desc, index asc): true when (g, f) comes before (bg, bf).  A total order on the gains sel_gain6 returns (never NaN), so
// the best of a set does not depend on how it is split.
CLC_HD bool sel_better(double g, int64_t f, double bg, int64_t bf) { return g > bg || (g == bg && f < bf); }

// ---- device -------------------------------------------------------------------------------------------------------------------
#if defined(__CUDACC__)

constexpr int kSelThreads = 128;
constexpr int kSelMaxPacked = 21;
constexpr int64_t kSelNone = INT64_MAX;  // "no candidate" index of a best

// the free coordinates of a mask, in order, and their count d
struct SelFree {
  int idx[6];
  int d;
};

// the state of one selection, on the device
struct SelState {
  double A[36];     // A_s, 6x6 (held coordinates: identity, behind the free ones)
  double L[36];     // its factor (sel_chol6)
  double inv[6];
  double D[6];      // diag(T)^-1/2 over the free coordinates
  double min_gain;
  int64_t budget;
  int64_t n_sel;    // picks so far
  int64_t n_t;      // n_T: usable frames that are not excluded
  int running;      // 1 while steps remain; 0 once a stop rule fired
  int status;       // 0, or 1 + k when free coordinate k (0..5, the mask's numbering) has no positive finite T_kk
  unsigned int arrivals;
};

struct SelBest {
  double gain;
  int64_t f;
};

__device__ __forceinline__ void sel_best_reduce_warp(double* g, int64_t* f) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double og = __shfl_down_sync(0xffffffffu, *g, o);
    const int64_t of = __shfl_down_sync(0xffffffffu, *f, o);
    if (sel_better(og, of, *g, *f)) { *g = og; *f = of; }
  }
}

// the block's best of (g, f) in thread 0's registers
__device__ __forceinline__ void sel_best_reduce_block(double* g, int64_t* f) {
  __shared__ double s_g[kSelThreads / 32];
  __shared__ int64_t s_f[kSelThreads / 32];
  sel_best_reduce_warp(g, f);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_g[warp] = *g; s_f[warp] = *f; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < kSelThreads / 32; ++w)
      if (sel_better(s_g[w], s_f[w], *g, *f)) { *g = s_g[w]; *f = s_f[w]; }
  __syncthreads();
}

// One thread per frame.  rows: the report rows (row_stride doubles apart, H21 at h_offset); state_in: the caller's states (nullptr:
// every frame a candidate).  Writes status[f] (1: usable candidate, else 0), keep[f] (forced), the raw free block to
// packed[sel_tri(d, i, j) * n + f], and per block partials[b * kSelSums ..]: the sums of T and of the forced blocks (each 21 wide,
// 6x6 upper-triangle order over the free coordinates, zeros beyond d) and the count n_T.
constexpr int kSelSums = 2 * kSelMaxPacked + 1;
__global__ void __launch_bounds__(kSelThreads)
clc_select_sum_kernel(const double* __restrict__ rows, int row_stride, int h_offset, int64_t n, const uint8_t* __restrict__ state_in,
                      SelFree fr, double* __restrict__ packed, uint8_t* __restrict__ status, uint8_t* __restrict__ keep,
                      double* __restrict__ partials) {
  __shared__ double s_part[kSelThreads / 32][kSelSums];
  const int64_t f = (int64_t)blockIdx.x * kSelThreads + threadIdx.x;
  double h[kSelMaxPacked];
#pragma unroll
  for (int k = 0; k < kSelMaxPacked; ++k) h[k] = 0.0;
  int st = 0;
  bool usable = false;
  if (f < n) {
    st = state_in != nullptr ? state_in[f] : 1;
    const double* row = rows + f * (int64_t)row_stride + h_offset;
    usable = true;
    for (int k = 0; k < 21; ++k) usable = usable && is_finite(row[k]);
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int j = i; j < 6; ++j)
        if (j < fr.d) {
          h[tri(i, j)] = row[tri(fr.idx[i], fr.idx[j])];
          packed[(int64_t)sel_tri(fr.d, i, j) * n + f] = h[tri(i, j)];
        }
    status[f] = usable && st == 1 ? 1 : 0;
    keep[f] = st == 2 ? 1 : 0;
  }
  const bool in_t = usable && st != 0, forced = usable && st == 2;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < kSelSums; ++q) {
    double v = q < kSelMaxPacked ? (in_t ? h[q] : 0.0)
               : q < 2 * kSelMaxPacked ? (forced ? h[q - kSelMaxPacked] : 0.0)
                                       : (in_t ? 1.0 : 0.0);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) s_part[warp][q] = v;
  }
  __syncthreads();
  if (threadIdx.x < kSelSums) {
    double acc = 0.0;
    for (int w = 0; w < kSelThreads / 32; ++w) acc += s_part[w][threadIdx.x];
    partials[(int64_t)blockIdx.x * kSelSums + threadIdx.x] = acc;
  }
}

// One block: thread q adds entry q of the n_blocks partials in block order; thread 0 then checks diag(T) and sets up D, A_0 and L.
__global__ void __launch_bounds__(64)
clc_select_init_kernel(const double* __restrict__ partials, int64_t n_blocks, SelFree fr, double min_gain, int64_t budget,
                       SelState* st) {
  __shared__ double s_sum[kSelSums];
  if (threadIdx.x < kSelSums) {
    double acc = 0.0;
    for (int64_t b = 0; b < n_blocks; ++b) acc += partials[b * kSelSums + threadIdx.x];
    s_sum[threadIdx.x] = acc;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const double* T = s_sum;
  const double* F = s_sum + kSelMaxPacked;
  st->min_gain = min_gain;
  st->budget = budget;
  st->n_sel = 0;
  st->n_t = (int64_t)s_sum[2 * kSelMaxPacked];
  st->arrivals = 0;
  st->status = 0;
  for (int i = 0; i < fr.d; ++i) {
    const double t = T[tri(i, i)];
    if (!(t > 0.0) || !is_finite(t)) {
      st->status = 1 + fr.idx[i];
      st->running = 0;
      return;
    }
    st->D[i] = 1.0 / sqrt(t);
  }
  const double ridge = kSelectRidge / s_sum[2 * kSelMaxPacked];
  double A[36];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      double a;
      if (i < fr.d && j < fr.d) {
        const int lo = i < j ? i : j, hi = i < j ? j : i;
        a = st->D[i] * F[tri(lo, hi)] * st->D[j] + (i == j ? ridge : 0.0);
      } else {
        a = i == j ? 1.0 : 0.0;
      }
      A[i * 6 + j] = a;
      st->A[i * 6 + j] = a;
    }
  double L[36], inv[6];
  const bool ok = sel_chol6(A, L, inv);
  for (int k = 0; k < 36; ++k) st->L[k] = L[k];
  for (int k = 0; k < 6; ++k) st->inv[k] = inv[k];
  st->running = ok && budget > 0 ? 1 : 0;
}

// One thread per frame: the packed free block scaled by D_i D_j in place (Ht_f).
__global__ void __launch_bounds__(kSelThreads)
clc_select_scale_kernel(double* __restrict__ packed, int64_t n, int d, const SelState* __restrict__ st) {
  const int64_t f = (int64_t)blockIdx.x * kSelThreads + threadIdx.x;
  if (f >= n || st->status != 0) return;
  int q = 0;
  for (int i = 0; i < d; ++i)
    for (int j = i; j < d; ++j, ++q) packed[(int64_t)q * n + f] *= st->D[i] * st->D[j];
}

// Ht_f as a full 6x6 (held coordinates zero) from the packed blocks
__device__ __forceinline__ void sel_load_block(const double* __restrict__ packed, int64_t n, int d, int64_t f, double* H) {
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = i; j < 6; ++j) {
      const double v = j < d ? __ldg(packed + (int64_t)sel_tri(d, i, j) * n + f) : 0.0;
      H[i * 6 + j] = v;
      H[j * 6 + i] = v;
    }
}

// One greedy step (see the file comment).  bests[gridDim.x]: the blocks' bests of this launch.
// The gain evaluation takes about 156 registers without spilling: 3 blocks of 128 threads fit an SM's register file.
__global__ void __launch_bounds__(kSelThreads, 3)
clc_select_step_kernel(const double* __restrict__ packed, int64_t n, int d, uint8_t* __restrict__ status, SelState* st,
                       SelBest* bests, int64_t* __restrict__ order, double* __restrict__ gain, uint8_t* __restrict__ keep) {
  __shared__ double s_L[36], s_inv[6];
  __shared__ bool s_last;
  if (*(volatile int*)&st->running == 0) return;
  if (threadIdx.x < 36) s_L[threadIdx.x] = st->L[threadIdx.x];
  if (threadIdx.x < 6) s_inv[threadIdx.x] = st->inv[threadIdx.x];
  __syncthreads();
  double bg = -HUGE_VAL;
  int64_t bf = kSelNone;
  for (int64_t f = (int64_t)blockIdx.x * kSelThreads + threadIdx.x; f < n; f += (int64_t)gridDim.x * kSelThreads) {
    if (status[f] != 1) continue;
    double H[36];
    sel_load_block(packed, n, d, f, H);
    const double g = sel_gain6(s_L, s_inv, H);
    if (sel_better(g, f, bg, bf)) { bg = g; bf = f; }
  }
  sel_best_reduce_block(&bg, &bf);
  if (threadIdx.x == 0) {
    bests[blockIdx.x] = SelBest{bg, bf};
    __threadfence();
    s_last = atomicAdd(&st->arrivals, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  bg = -HUGE_VAL;
  bf = kSelNone;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += kSelThreads) {
    const double g = __ldcg(&bests[b].gain);
    const int64_t f = __ldcg(reinterpret_cast<const long long*>(&bests[b].f));
    if (sel_better(g, f, bg, bf)) { bg = g; bf = f; }
  }
  sel_best_reduce_block(&bg, &bf);
  if (threadIdx.x != 0) return;
  st->arrivals = 0;
  if (bf == kSelNone || !(bg > st->min_gain)) {
    st->running = 0;
    return;
  }
  const int64_t s = st->n_sel;
  order[s] = bf;
  gain[s] = bg;
  status[bf] = 0;
  keep[bf] = 1;
  double H[36], A[36], L[36], inv[6];
  sel_load_block(packed, n, d, bf, H);
  for (int k = 0; k < 36; ++k) A[k] = st->A[k] + H[k];
  const bool ok = sel_chol6(A, L, inv);
  for (int k = 0; k < 36; ++k) { st->A[k] = A[k]; st->L[k] = L[k]; }
  for (int k = 0; k < 6; ++k) st->inv[k] = inv[k];
  st->n_sel = s + 1;
  if (!ok || s + 1 >= st->budget) st->running = 0;
}

#endif  // __CUDACC__

}  // namespace clc
