// clc_trim_plan.h -- the host side of clc_problem_trim / clc_group_trim (plain C++, no CUDA).
//
// A trim keeps the points of a device-resident problem (or of every shard of an in-process group) whose distance to their board
// is within a per-frame threshold.  The mark pass (clc_trim.cuh) counts the kept points of every frame and of every source tile of
// kTrimTile points; those counts (8 bytes each) are all the host sees.  From them this file computes the new frame offsets, how a
// group's frames are re-sharded over the new point counts, and for every destination tile the first source tile whose kept points
// land in it.  O(frames + tiles) work; the O(points) work is the kernels'.
#pragma once

#include <cstdint>
#include <vector>

#include "clc_subset_plan.h"

namespace clc {

constexpr int64_t kTrimTile = 2048;  // points per tile, source (mark pass) and destination (gather pass) alike

struct TrimPlan {
  std::vector<int64_t> offsets;      // [N + 1]: global point prefix of the trimmed frames (every source frame, in order)
  std::vector<int64_t> shard_frame;  // [n_dst + 1]: destination shard d holds frames [shard_frame[d], shard_frame[d + 1])
  std::vector<int64_t> tile_prefix;  // [T + 1]: kept points before every source tile, the tiles of all source shards in order
  std::vector<int64_t> tile_begin;   // [n_dst + 1]: destination shard d's tiles are [tile_begin[d], tile_begin[d + 1]) ...
  std::vector<int64_t> first_tile;   // ... of this list: the first source tile feeding every destination tile
};

// n_src source shards in frame order; shard s has src_frames[s] frames with frame_kept[s][f] kept points each, and src_tiles[s]
// tiles with tile_kept[s][t] kept points each.  The frames are sharded over n_dst destination shards as clc_group_create_gather
// shards a fresh problem (balanced_shard_range over the kept point prefix); each destination shard's points are cut into tiles
// of kTrimTile points from its own first point.
inline TrimPlan trim_plan(int n_src, const int64_t* src_frames, const int64_t* const* frame_kept, const int64_t* src_tiles,
                          const int64_t* const* tile_kept, int n_dst) {
  TrimPlan plan;
  plan.offsets.push_back(0);
  for (int s = 0; s < n_src; ++s)
    for (int64_t f = 0; f < src_frames[s]; ++f) plan.offsets.push_back(plan.offsets.back() + frame_kept[s][f]);
  plan.tile_prefix.push_back(0);
  for (int s = 0; s < n_src; ++s)
    for (int64_t t = 0; t < src_tiles[s]; ++t) plan.tile_prefix.push_back(plan.tile_prefix.back() + tile_kept[s][t]);
  const int64_t N = (int64_t)plan.offsets.size() - 1, T = (int64_t)plan.tile_prefix.size() - 1;
  plan.shard_frame.assign((size_t)n_dst + 1, 0);
  for (int d = 0; d < n_dst; ++d) {
    int64_t b = 0, e = 0;
    balanced_shard_range(N, plan.offsets.data(), n_dst, d, &b, &e);
    plan.shard_frame[d] = b;
    plan.shard_frame[d + 1] = e;
  }
  // destination tile starts rise through the kept points, so one pass over the source tiles finds every first feeding tile:
  // the last source tile whose kept points start at or before the destination tile's first point (a tile without kept points
  // never qualifies, the tile after it starts at the same point)
  plan.tile_begin.push_back(0);
  int64_t g = 0;
  for (int d = 0; d < n_dst; ++d) {
    const int64_t p0 = plan.offsets[plan.shard_frame[d]], p1 = plan.offsets[plan.shard_frame[d + 1]];
    for (int64_t start = p0; start < p1; start += kTrimTile) {
      while (g + 1 < T && plan.tile_prefix[g + 1] <= start) ++g;
      plan.first_tile.push_back(g);
    }
    plan.tile_begin.push_back((int64_t)plan.first_tile.size());
  }
  return plan;
}

}  // namespace clc
