// clc_frames.cuh -- bookkeeping of the per-frame report (clc_frame_report): which warp ranges of the sweep kernel's static
// partition hold a frame, and whether a warp's piece of it is the whole frame, its head or its tail.
//
// The sweep kernel cuts the P points into warp ranges [w * per_warp, min((w + 1) * per_warp, P)).  A frame [fs, fe) that lies in
// one range is expanded by that warp and written straight to its report row.  A frame that crosses a range end is split:
//   * the warp whose range holds its first point keeps a TAIL piece (the frame continues past the range end);
//   * every later warp that holds some of it keeps a HEAD piece (the frame started before the range start) -- also the warps
//     whose whole range lies inside the frame.
// Head and tail pieces go to two per-warp slots as raw sums; clc_frame_fixup_kernel adds, per split frame, the tail slot of its
// first warp and the head slots of the following warps in warp order and writes the row.  Host and device share these
// functions (CLC_HD), so the CPU tests compile the same arithmetic the kernels run.
#pragma once

#include <cstdint>

#include "clc_math.cuh"

namespace clc {

enum FramePiece { kPieceWhole = 0, kPieceHead = 1, kPieceTail = 2 };

// Kind of the piece of frame [fs, fe) held by the warp range [p0, p1) (the two overlap).
CLC_HD int frame_piece_kind(int64_t fs, int64_t fe, int64_t p0, int64_t p1) {
  if (fs < p0) return kPieceHead;
  return fe > p1 ? kPieceTail : kPieceWhole;
}

// First and last warp whose ranges hold points of the non-empty frame [fs, fe); the frame is split when they differ.
CLC_HD void frame_warps(int64_t fs, int64_t fe, int64_t per_warp, int64_t* first, int64_t* last) {
  *first = fs / per_warp;
  *last = (fe - 1) / per_warp;
}

// Per-warp slots of the split pieces: [warp][kSlotHead | kSlotTail][kSlotDoubles].
constexpr int kSlotHead = 0;
constexpr int kSlotTail = 1;
constexpr int kSlotDoubles = 16;  // 10 moments, cost product (loss) or 0, exponent, sum e, sum e^2, max |e|, points
// Slot of warp w that the fix-up adds for the split frame whose first warp is w0: the tail of w0, the head of every later warp.
CLC_HD int64_t frame_slot(int64_t w, int64_t w0) { return (w * 2 + (w == w0 ? kSlotTail : kSlotHead)) * kSlotDoubles; }

// One report row as the kernels write it: the layout of clc_frame_row (include/clc_b200.h; clc_api.cu checks the offsets).
constexpr int kRowDoubles = 36;
constexpr int kRowN = 0;      // points of the frame (int64 bits)
constexpr int kRowCost = 1;
constexpr int kRowChi = 2;
constexpr int kRowMeanE = 3;
constexpr int kRowRmsE = 4;
constexpr int kRowMaxE = 5;
constexpr int kRowMeanW = 6;
constexpr int kRowEdgeE = 7;  // 2
constexpr int kRowH = 9;      // 21, upper triangle row-major (K1's order)
constexpr int kRowG = 30;     // 6

// max(m, v) that keeps a NaN: a frame with a NaN residual reports NaN as its max |e| (fmax would drop it).
CLC_HD double nan_max(double m, double v) { return (v > m || v != v) ? v : m; }

}  // namespace clc
