// clc_subset_plan.h -- the host side of clc_problem_subset / clc_group_subset (plain C++, no CUDA).
//
// A subset keeps some frames of a device-resident problem (or of every shard of an in-process group) and drops the rest.  The host
// only ever sees the source's frame offsets (8 bytes per frame and shard); from them and the keep mask this file computes what the
// new problem looks like -- its offsets, which old frame every new frame is, how a group's kept frames are re-sharded -- and the
// list of copies the gather kernel (clc_subset.cuh) makes.  O(n_frames) work; the O(n_points) work is the kernel's.
#pragma once

#include <algorithm>
#include <cstdint>
#include <vector>

namespace clc {

// Balanced contiguous frame range of shard `rank` of `nranks` by point count (clc_shard_range): boundary r is the first frame whose
// start is >= r * P / nranks.  offsets[n_frames + 1] is the global prefix.
inline void balanced_shard_range(int64_t n_frames, const int64_t* offsets, int nranks, int rank, int64_t* begin, int64_t* end) {
  const int64_t P = offsets[n_frames];
  auto boundary = [&](int r) -> int64_t {
    if (r <= 0) return 0;
    if (r >= nranks) return n_frames;
    const int64_t target = (int64_t)((__int128)P * r / nranks);
    return std::lower_bound(offsets, offsets + n_frames + 1, target) - offsets;
  };
  *begin = boundary(rank);
  *end = boundary(rank + 1);
  if (*end < *begin) *end = *begin;
}

// One copy of the gather: a run of kept frames that are adjacent in the source, lie in one source shard and land in one
// destination shard.  Frame and point indices are local to their shard.
struct SubsetSegment {
  int32_t src_shard, dst_shard;
  int64_t src_frame, dst_frame, n_frames;
  int64_t src_point, dst_point, n_points;
};

struct SubsetPlan {
  std::vector<int64_t> offsets;      // [K + 1]: global point prefix of the K kept frames
  std::vector<int64_t> frame_map;    // [K]: new global frame -> old global frame
  std::vector<int64_t> shard_frame;  // [n_dst + 1]: destination shard d holds new frames [shard_frame[d], shard_frame[d + 1])
  std::vector<SubsetSegment> segments;  // by destination shard, then destination frame; every kept frame in exactly one
};

// n_src source shards in frame order; shard s holds src_frames[s] frames with local offsets src_offsets[s][0 .. src_frames[s]]
// (src_offsets[s][0] == 0).  keep has one entry (0 or 1) per source frame over all shards, in the global frame order.  The kept
// frames are sharded over n_dst destination shards as clc_group_create_gather shards a fresh problem (balanced_shard_range over
// the kept point prefix).
inline SubsetPlan subset_plan(int n_src, const int64_t* const* src_offsets, const int64_t* src_frames, const uint8_t* keep,
                              int n_dst) {
  SubsetPlan plan;
  struct Kept { int32_t shard; int64_t frame, point, count; };
  std::vector<Kept> kept;
  plan.offsets.push_back(0);
  int64_t global = 0;
  for (int s = 0; s < n_src; ++s) {
    const int64_t* off = src_offsets[s];
    for (int64_t f = 0; f < src_frames[s]; ++f, ++global) {
      if (!keep[global]) continue;
      const int64_t n = off[f + 1] - off[f];
      kept.push_back({(int32_t)s, f, off[f], n});
      plan.frame_map.push_back(global);
      plan.offsets.push_back(plan.offsets.back() + n);
    }
  }
  const int64_t K = (int64_t)kept.size();
  plan.shard_frame.assign((size_t)n_dst + 1, 0);
  for (int d = 0; d < n_dst; ++d) {
    int64_t b = 0, e = 0;
    balanced_shard_range(K, plan.offsets.data(), n_dst, d, &b, &e);
    plan.shard_frame[d] = b;
    plan.shard_frame[d + 1] = e;
  }
  for (int d = 0; d < n_dst; ++d) {
    const int64_t fb = plan.shard_frame[d], fe = plan.shard_frame[d + 1];
    for (int64_t k = fb; k < fe; ++k) {
      const Kept& c = kept[(size_t)k];
      if (!plan.segments.empty()) {
        SubsetSegment& last = plan.segments.back();
        // the run continues: same shards, and the frame directly follows the run's last frame in the source
        if (last.dst_shard == d && last.src_shard == c.shard && last.src_frame + last.n_frames == c.frame) {
          last.n_frames += 1;
          last.n_points += c.count;
          continue;
        }
      }
      plan.segments.push_back({c.shard, (int32_t)d, c.frame, k - fb, 1, c.point, plan.offsets[(size_t)k] - plan.offsets[(size_t)fb], c.count});
    }
  }
  return plan;
}

}  // namespace clc
