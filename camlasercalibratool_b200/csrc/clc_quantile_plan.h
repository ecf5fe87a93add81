// clc_quantile_plan.h -- the selection arithmetic of clc_residual_quantiles / clc_frame_quantiles (plain C++; also compiled for the
// device, where the one-block path of a large frame runs it on one thread).
//
// The quantiles are exact order statistics of |e| (include/clc_b200.h).  The key of a value is its bit pattern: for non-negative
// doubles (fabs) the bits are monotone as uint64, the top bit is 0, so a key has 63 significant bits, +inf is 0x7FF0000000000000
// and every NaN lies above it.  A radix select resolves the keys of all requested ranks from the top bit down, one digit per pass
// over the keys:
//   - the state holds the distinct active prefixes (the top `bits` bits of the bucket each rank lies in) and every rank's position
//     within its bucket;
//   - a pass histograms the next `d` bits of every valid key whose top bits match an active prefix, one run of 2^d bins per
//     prefix, so the digit width follows from the number of distinct prefixes and the bin budget (qsel_digit);
//   - qsel_update picks every rank's bucket from the histogram and its rank within it; the first update also counts the valid
//     keys and turns the quantiles into ranks (quantile_rank);
//   - after 63 resolved bits every active prefix is a whole key: the result.
// Counts are integers, so summing the histograms of several shards in any order gives the same state.
#pragma once

#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define CLC_QHD __host__ __device__ inline
#else
#define CLC_QHD inline
#endif

namespace clc {

constexpr int kQuantilesMax = 16;                         // CLC_QUANTILES_MAX
constexpr int kKeyBits = 63;                              // significant bits of the key of a non-negative double
constexpr uint64_t kKeyNanMin = 0x7FF0000000000001ull;    // keys at or above this one are NaN
constexpr int kQuantileBinsLog2 = 13;                     // bins of a problem-wide pass (uint32 in shared memory per block)
constexpr int kFrameBinsLog2 = 12;                        // bins of a large frame's pass (uint64 in shared memory)
constexpr uint64_t kCompactCap = (uint64_t)1 << 16;       // a bucket of at most this many keys is compacted (C)

// k = clamp(ceil(q n) - 1, 0, n - 1) with q n a double product; n > 0
CLC_QHD uint64_t quantile_rank(double q, uint64_t n) {
  const double t = ceil(q * (double)n) - 1.0;
  if (!(t > 0.0)) return 0;
  const uint64_t k = (uint64_t)t;
  return k < n - 1 ? k : n - 1;
}

// trivially constructible (it lives in shared memory on the device): qsel_start initialises it
struct QSel {
  int n_q;
  int bits;                           // key bits resolved from the top
  int n_pre;                          // distinct active prefixes, ascending
  uint64_t n_valid;                   // keys that are not NaN (known after the first update)
  double q[kQuantilesMax];
  uint64_t pre[kQuantilesMax];        // the active prefixes (top `bits` bits of the key)
  uint64_t pre_count[kQuantilesMax];  // keys in every active bucket
  int rank_pre[kQuantilesMax];        // the active prefix of every rank
  uint64_t rank[kQuantilesMax];       // every rank within its bucket
};

// the selection of n_q quantiles q[0..n_q): one active prefix, the empty one, which every valid key matches
CLC_QHD void qsel_start(QSel* s, int n_q, const double* q) {
  s->n_q = n_q;
  s->bits = 0;
  s->n_pre = 1;
  s->n_valid = 0;
  s->pre[0] = 0;
  s->pre_count[0] = 0;
  for (int r = 0; r < n_q; ++r) {
    s->q[r] = q[r];
    s->rank_pre[r] = 0;
    s->rank[r] = 0;
  }
}

CLC_QHD bool qsel_done(const QSel& s) { return s.bits >= kKeyBits; }

// the digit width of the next pass: 2^bins_log2 bins shared by the active prefixes, at most the bits left
CLC_QHD int qsel_digit(const QSel& s, int bins_log2) {
  int lg = 0;
  while ((1 << lg) < s.n_pre) ++lg;
  const int d = bins_log2 - lg;
  return d < kKeyBits - s.bits ? d : kKeyBits - s.bits;
}

// the bin of `key` in a pass of digit width d, or -1 when the key is NaN or matches no active prefix (binary search: the
// prefixes ascend)
CLC_QHD int qsel_bin(int bits, int n_pre, const uint64_t* pre, int d, uint64_t key) {
  if (key >= kKeyNanMin) return -1;
  const uint64_t top = bits == 0 ? 0 : key >> (kKeyBits - bits);
  int lo = 0, hi = n_pre;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (pre[mid] <= top) lo = mid;
    else hi = mid;
  }
  if (pre[lo] != top) return -1;
  return (lo << d) | (int)((key >> (kKeyBits - bits - d)) & (((uint64_t)1 << d) - 1));
}

// whether a key belongs to an active bucket (the compaction's test)
CLC_QHD bool qsel_match(int bits, int n_pre, const uint64_t* pre, uint64_t key) { return qsel_bin(bits, n_pre, pre, 0, key) >= 0; }

// Consumes the histogram hist[n_pre << d] of a pass of digit width d.  The first update counts the valid keys and turns every q
// into its rank; without a valid key the selection ends there (n_valid = 0, no active prefix).
template <class Count>
CLC_QHD void qsel_update(QSel* s, const Count* hist, int d) {
  const int nb = 1 << d;
  if (s->bits == 0) {
    uint64_t n = 0;
    for (int b = 0; b < nb; ++b) n += (uint64_t)hist[b];
    s->n_valid = n;
    if (n == 0) {
      s->bits = kKeyBits;
      s->n_pre = 0;
      return;
    }
    for (int r = 0; r < s->n_q; ++r) s->rank[r] = quantile_rank(s->q[r], n);
  }
  uint64_t new_pre[kQuantilesMax], count[kQuantilesMax];
  for (int r = 0; r < s->n_q; ++r) {
    const int p = s->rank_pre[r];
    const Count* h = hist + ((int64_t)p << d);
    uint64_t below = 0;
    int b = 0;
    for (; b < nb - 1; ++b) {
      if (s->rank[r] < below + (uint64_t)h[b]) break;
      below += (uint64_t)h[b];
    }
    new_pre[r] = (s->pre[p] << d) | (uint64_t)b;
    count[r] = (uint64_t)h[b];
    s->rank[r] -= below;
  }
  // the distinct new prefixes, ascending (insertion into a list of at most kQuantilesMax)
  int n = 0;
  for (int r = 0; r < s->n_q; ++r) {
    int i = 0;
    while (i < n && s->pre[i] < new_pre[r]) ++i;
    if (i < n && s->pre[i] == new_pre[r]) continue;
    for (int j = n; j > i; --j) {
      s->pre[j] = s->pre[j - 1];
      s->pre_count[j] = s->pre_count[j - 1];
    }
    s->pre[i] = new_pre[r];
    s->pre_count[i] = count[r];
    ++n;
  }
  for (int r = 0; r < s->n_q; ++r) {
    int i = 0;
    while (s->pre[i] != new_pre[r]) ++i;
    s->rank_pre[r] = i;
  }
  s->n_pre = n;
  s->bits += d;
}

// whether the next pass may compact the active buckets: each holds at most `cap` keys (the scratch holds n_pre * cap)
CLC_QHD bool qsel_fits(const QSel& s, uint64_t cap) {
  for (int i = 0; i < s.n_pre; ++i)
    if (s.pre_count[i] > cap) return false;
  return true;
}

// the key of rank r once the selection is done (qsel_done, n_valid > 0)
CLC_QHD uint64_t qsel_key(const QSel& s, int r) { return s.pre[s.rank_pre[r]]; }

}  // namespace clc
