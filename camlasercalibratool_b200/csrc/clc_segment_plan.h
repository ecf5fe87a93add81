// clc_segment_plan.h -- the segmentation of a problem's frames into independent solves (clc_*_segments) and the fixed
// two-level reduction plan that sums each segment's per-frame rows.
//
// A segmentation is a CSR array seg_offsets[W + 1] over the frames: seg_offsets[0] = 0, non-decreasing, seg_offsets[W] =
// n_frames, W >= 1.  Segment s owns frames [seg_offsets[s], seg_offsets[s + 1]); empty segments are valid.
//
// The rows of a segment are summed in two fixed levels, so that the sums are bit-reproducible and no warp walks a long segment
// alone: the frames are cut into CHUNKS of at most kSegChunkRows rows that never cross a segment boundary (a segment's chunks
// start at its first frame and every kSegChunkRows frames after it); level 1 sums the rows of each chunk in frame order, level 2
// sums each segment's chunk partials in chunk order.  Because segments are contiguous runs of frames, the chunks are too:
// chunk_offsets[n_chunks + 1] is a CSR array over the frames and segment s owns chunks [seg_chunks[s], seg_chunks[s + 1]).
// Host and device share these functions (CLC_HD), so the CPU tests compile the same arithmetic the library runs.
#pragma once

#include <cstdint>
#include <vector>

#include "clc_math.cuh"

namespace clc {

constexpr int64_t kSegChunkRows = 256;

// true iff seg_offsets[0..W] is a valid segmentation of n_frames frames
CLC_HD bool segments_valid(int64_t n_frames, int64_t W, const int64_t* seg_offsets) {
  if (W < 1 || seg_offsets == nullptr || seg_offsets[0] != 0 || seg_offsets[W] != n_frames) return false;
  for (int64_t s = 0; s < W; ++s)
    if (seg_offsets[s + 1] < seg_offsets[s]) return false;
  return true;
}

// chunks of a segment of n frames
CLC_HD int64_t segment_chunk_count(int64_t n) { return (n + kSegChunkRows - 1) / kSegChunkRows; }

struct SegmentPlan {
  std::vector<int64_t> chunk_offsets;  // [n_chunks + 1] frame ranges of the chunks
  std::vector<int64_t> seg_chunks;     // [W + 1] chunk ranges of the segments
  std::vector<int32_t> frame_seg;      // [n_frames] segment of every frame
};

// The plan of a valid segmentation (segments_valid).  O(n_frames + W).
inline SegmentPlan segment_plan(int64_t n_frames, int64_t W, const int64_t* seg_offsets) {
  SegmentPlan p;
  p.seg_chunks.reserve((size_t)W + 1);
  p.frame_seg.resize((size_t)n_frames);
  p.chunk_offsets.push_back(0);
  p.seg_chunks.push_back(0);
  for (int64_t s = 0; s < W; ++s) {
    const int64_t a = seg_offsets[s], b = seg_offsets[s + 1];
    for (int64_t f = a; f < b; ++f) p.frame_seg[(size_t)f] = (int32_t)s;
    for (int64_t c = 0; c < segment_chunk_count(b - a); ++c) {
      const int64_t e = a + (c + 1) * kSegChunkRows;
      p.chunk_offsets.push_back(e < b ? e : b);
    }
    p.seg_chunks.push_back((int64_t)p.chunk_offsets.size() - 1);
  }
  return p;
}

// One calibration at K poses (clc_eval_poses, clc_solve_lm_starts): pose k owns all n_frames frames, so its rows form segment k
// of a pose-major virtual segmentation of K * n_frames rows, seg_offsets[k] = k * n_frames, which segment_plan reduces.
inline std::vector<int64_t> pose_segment_offsets(int64_t n_frames, int64_t K) {
  std::vector<int64_t> off((size_t)K + 1);
  for (int64_t k = 0; k <= K; ++k) off[(size_t)k] = k * n_frames;
  return off;
}

// The best of K solves: the lowest final cost among those whose termination is not `failure` (a NaN cost loses to any other),
// the lowest index on a tie; -1 when every solve failed.
CLC_HD int64_t best_start(int64_t K, const int* termination, const double* final_cost, int failure) {
  int64_t best = -1;
  for (int64_t k = 0; k < K; ++k) {
    if (termination[k] == failure) continue;
    const double c = final_cost[k];
    if (best < 0 || c < final_cost[best] || (final_cost[best] != final_cost[best] && c == c)) best = k;
  }
  return best;
}

}  // namespace clc
