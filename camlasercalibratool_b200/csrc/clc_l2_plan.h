// clc_l2_plan.h -- how much of the coordinate arrays an LM solve keeps resident in L2 (host code, plain C++).
//
// Every LM iteration sweeps the same points in the same order.  A cyclic stream much larger than L2 gets almost no hits, so
// the sweep kernel marks the last `resident_chunks` stages of every warp's range evict_last (they stay in L2 from one sweep to
// the next) and the rest evict_first (clc_kernels.cuh, issue_one).  This file decides how many stages that is.
#pragma once

#include <algorithm>
#include <cstdint>

namespace clc {

// Share of the device's L2 the resident stages may fill.  Measured on an H100 SXM at configs[1] (10^7 points): 0.4 to 0.7 are
// within 0.3 % of each other (general and planar), 0.8 is slower; 0.5 leaves the other half of L2 to the evict_first stream,
// the frame data and whatever else runs on the GPU.
constexpr double kL2ResidentFraction = 0.5;

// L2 bytes an LM solve may keep resident: `override_bytes` when it is >= 0 (CLC_L2_RESIDENT_MB; 0 = off), otherwise
// kL2ResidentFraction of the device's L2.
inline int64_t l2_resident_budget(int64_t l2_bytes, int64_t override_bytes) {
  return override_bytes >= 0 ? override_bytes : (int64_t)((double)l2_bytes * kL2ResidentFraction);
}

// Stages per warp whose lines stay in L2 across the sweeps of a solve: as many as the budget holds for every warp of the grid,
// at most the whole range (a problem that fits is entirely resident).  0 for latency-bound launches -- a single block, or a
// problem small enough for the one-cluster kernel -- which gain nothing from it.
inline int l2_resident_chunks(int64_t budget_bytes, int64_t grid, int64_t warps_per_block, int64_t stages_per_warp,
                              int64_t stage_bytes, bool latency_bound) {
  if (budget_bytes <= 0 || grid <= 1 || latency_bound || stages_per_warp <= 0 || stage_bytes <= 0) return 0;
  return (int)std::min<int64_t>(stages_per_warp, budget_bytes / (grid * warps_per_block * stage_bytes));
}

}  // namespace clc
