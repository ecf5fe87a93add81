/*
 * clc_b200.h -- C ABI of libclc_b200.so: the H100-native (sm_90a) implementation of the camera<-laser
 * extrinsic solve of MegviiRobot/CamLaserCalibraTool.
 *
 * The reference has no FFI: its "operator API" for this path is four C++ free functions plus one struct
 * (reference include/LaseCamCalCeres.h:11-29).  This header is the boundary a replacement of
 * reference src/LaseCamCalCeres.cpp binds to; camlasercalibratool_b200/host/LaseCamCalB200.cpp is that
 * replacement (same signatures, same Oberserve struct) and INTEGRATION.md shows the CMake change.
 *
 * Plain C, POD only, int status codes (0 = CLC_OK), no exceptions cross the boundary, no torch types.
 * There is NO CPU fallback: every entry point fails with CLC_ERR_CUDA if no sm_90 device is usable.
 *
 * Data conventions (identical to the marshalled form of std::vector<Oberserve>):
 *   frame_pose[f*7 .. +7] = qx,qy,qz,qw (Eigen coeff order of Oberserve::tagPose_Qca), tx,ty,tz (tagPose_tca)
 *                           -- reference include/LaseCamCalCeres.h:20-21
 *   offsets[n_frames+1]   = CSR delimiters of the frames inside `points`
 *   points[P*3]           = AoS x,y,z doubles: the calibration point set the reference selects at
 *                           src/LaseCamCalCeres.cpp:233-237 (obs.points or obs.points_on_line)
 *   edge_points[f*6..+6]  = obs[f].points.front() then obs[f].points.back() (src/LaseCamCalCeres.cpp:278-279);
 *                           non-NULL enables the board-edge residuals of :258-294
 *   pose7                 = tx,ty,tz,qx,qy,qz,qw: the Ceres parameter block of T_cl (:219)
 *   4x4 matrices are row-major.
 */
#ifndef CLC_B200_H
#define CLC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CLC_OK 0
#define CLC_ERR_INVALID 1  /* bad argument */
#define CLC_ERR_CUDA 2     /* CUDA runtime / no usable device */
#define CLC_ERR_NCCL 3     /* NCCL missing or a collective failed */
#define CLC_ERR_STATE 4    /* call not valid in this state */

typedef struct clc_problem clc_problem; /* opaque, device-resident problem (one per GPU / rank) */

/* replaces: the argument marshalling of CamLaserCalibration()/CamLaserCalClosedSolution(),
 * reference src/LaseCamCalCeres.cpp:213-295 and :112-159 */
typedef struct {
  int64_t n_frames;
  const double* frame_pose;  /* host [n_frames*7] */
  const int64_t* offsets;    /* host [n_frames+1] */
  const double* points;      /* host [offsets[n_frames]*3]; pinned memory uploads at full PCIe rate */
  const double* edge_points; /* host [n_frames*6] or NULL */
  int use_loss;              /* 1: CauchyLoss(cauchy_a*scale), reference :212,:249 */
  double cauchy_a;           /* 0.05 */
  int device;                /* CUDA ordinal, -1 = current device */
} clc_problem_desc;

/* The same problem as the caller of the reference holds it: one separate array of Vector3d per frame -- Oberserve::points or
 * ::points_on_line of every element of the std::vector<Oberserve> the reference's functions take BY VALUE
 * (reference include/LaseCamCalCeres.h:22-23,28; Eigen::Vector3d is three contiguous doubles, so
 * obs[f].points.data() is frame_points[f]).  The library gathers the frames itself (pack threads -> pinned ring -> PCIe
 * -> layout kernel, all overlapped); pageable memory is fine.  replaces: the per-point loops of
 * reference src/LaseCamCalCeres.cpp:233-254 (one heap CostFunction + LossFunction per point). */
typedef struct {
  int64_t n_frames;
  const double* frame_pose;          /* host [n_frames*7] */
  const double* const* frame_points; /* host [n_frames]: AoS xyz of frame f, frame_counts[f] points */
  const int64_t* frame_counts;       /* host [n_frames] */
  const double* edge_points;         /* host [n_frames*6] or NULL */
  int use_loss;
  double cauchy_a;
  int device;                        /* ignored by the clc_group_* entry points (they take a device list) */
} clc_gather_desc;

/* replaces: GenerateSimData(), reference main/calibr_simulation.cpp:10-108, scaled to n_frames x beams and run
 * on the device (the 48 GB of BASELINE config 4 cannot pass through std::vector<Oberserve>). */
typedef struct {
  int64_t n_frames_total; /* frames of the whole (all-rank) problem; RNG counters are global frame ids */
  int64_t frame_begin;    /* this problem holds frames [frame_begin, frame_end) */
  int64_t frame_end;
  int64_t beams;          /* points per frame (exact-M mode: every frame has exactly `beams` points) */
  uint64_t seed;
  double sigma;           /* range noise along the ray, metres */
  int with_edges;         /* also generate the two board-edge residual points per frame */
  int use_loss;
  double cauchy_a;
  int device;
  /* Optional camera measurement chain (SURVEY.md 8(f) rank 2): the board pose the calibration sees is then ESTIMATED from
   * noisy corner pixels -- kalibr-grid corners -> Camera::spaceToPlane -> pixel noise -> Camera::liftProjective -> planar
   * PnP, as reference src/calcCamPose.cpp:279-292,211-236 does with cv::solvePnP -- while the laser hits the true board.
   * camera_model 0: exact poses (the reference simulation); 1: pinhole + radtan, intrinsics = fx fy cx cy k1 k2 p1 p2
   * (reference config/calibra_config_pinhole.yaml); 2: equidistant (Kannala-Brandt), intrinsics = mu mv u0 v0 k2 k3 k4 k5
   * (reference config/calibra_config.yaml).  Boards are redrawn until all grid corners fall inside the image. */
  int camera_model;
  double camera_intrinsics[8];
  double pixel_sigma;     /* std of the corner noise in pixels */
  int image_width, image_height; /* 752 x 480 in the reference configs */
  int grid_rows, grid_cols;      /* 6 x 6 */
  double tag_size, tag_spacing;  /* 0.055 m, 0.3 */
} clc_synthetic_desc;

/* Ceres Solver::Options subset, defaults = reference src/LaseCamCalCeres.cpp:302-304 + Ceres defaults */
typedef struct {
  int max_num_iterations;           /* 100 */
  double initial_trust_region_radius; /* 1e4 */
  double max_trust_region_radius;   /* 1e16 */
  double min_trust_region_radius;   /* 1e-32 */
  double min_relative_decrease;     /* 1e-3 */
  double min_lm_diagonal;           /* 1e-6 */
  double max_lm_diagonal;           /* 1e32 */
  double function_tolerance;        /* 1e-6 */
  double gradient_tolerance;        /* 1e-10 */
  double parameter_tolerance;       /* 1e-8 */
  int max_num_consecutive_invalid_steps; /* 5 */
  int jacobi_scaling;               /* 1 */
  int iterations_per_sync;          /* LM iterations enqueued between host polls of the device `done` flag (8; the first batch of a solve is twice as long) */
  /* Coordinates of the extrinsic held at their start value (0: none).  Bit k holds tangent coordinate k of the reference's
   * PoseLocalParameterization::Plus: bits 0-2 = dt_x, dt_y, dt_z (translation of T_cl, camera frame), bits 3-5 = dtheta_x,
   * dtheta_y, dtheta_z (right-multiplied rotation increment, laser frame).  The solve is Ceres' LM on the reduced local
   * parameterization (a Ceres 2.1 local parameterization of local size 6 - k wrapped around the reference's):
   *   - Jacobi scaling, the LM diagonal, the Cholesky step, the model cost change and gradient_max_norm use the free
   *     coordinates only; the parameter tolerance still measures the 7-vector;
   *   - a held translation coordinate keeps its start value bit for bit;
   *   - a held rotation bit removes that axis from every increment.  It does NOT freeze an Euler angle: increments about the
   *     other two axes do not commute, so the orientation about the held axis may still drift as they accumulate.
   * Typical use: the coordinates the reference's null-space report (clc_information) names as unobservable, held at a value
   * from a tape measure or a drawing.  A mask with bits above 5, or with all six bits set (63), fails with CLC_ERR_INVALID
   * before any device work in clc_solve_lm, clc_group_solve_lm, clc_solve_lm_segments and clc_solve_lm_starts.  (This field
   * was `reserved` and ignored before: callers that left garbage in it now get CLC_ERR_INVALID.)  clc_solve_lm_time_offset
   * alone also takes bit 6 (the time offset td; masks 0..126), clc_solve_lm_range_bias bits 6 and 7 (the range offset b and
   * scale s; masks 0..254).  clc_lm_default_options sets 0. */
  int fixed_mask;
} clc_lm_options;

/* termination codes (Ceres TerminationType + the tolerance that fired) */
#define CLC_TERM_RUNNING 0
#define CLC_TERM_CONVERGENCE_FUNCTION 1
#define CLC_TERM_CONVERGENCE_PARAMETER 2
#define CLC_TERM_CONVERGENCE_GRADIENT 3
#define CLC_TERM_CONVERGENCE_MIN_RADIUS 4
#define CLC_TERM_NO_CONVERGENCE 5
#define CLC_TERM_FAILURE 6

/* one row of Ceres' IterationSummary */
typedef struct {
  int iteration;
  int step_is_valid;
  int step_is_successful;
  int reserved;
  double cost;
  double cost_change;
  double gradient_max_norm;
  double step_norm;
  double relative_decrease;
  double trust_region_radius;
} clc_lm_iteration;

typedef struct {
  int termination;
  int num_iterations;          /* rows written to the trace (iteration 0 included) */
  int num_successful_steps;
  int num_unsuccessful_steps;
  int num_sweeps;              /* launches of the fused residual+Jacobian+reduce kernel that did work */
  int reserved;
  double initial_cost;
  double final_cost;
  double device_ms;            /* CUDA-event time of the whole on-device solve on this rank */
} clc_lm_summary;

const char* clc_last_error(void);
int clc_device_count(int* count);

void clc_lm_default_options(clc_lm_options* opt);

/* Uploads (H2D) and lays the problem out in HBM (SoA points, per-frame planes).  replaces: problem assembly,
 * reference src/LaseCamCalCeres.cpp:222-295 (no per-residual heap objects are created). */
int clc_problem_create(clc_problem** out, const clc_problem_desc* desc);
/* Same from per-frame arrays (the marshalled form of std::vector<Oberserve> without flattening it on the host). */
int clc_problem_create_gather(clc_problem** out, const clc_gather_desc* desc);
/* Same, generated on the device. */
int clc_problem_create_synthetic(clc_problem** out, const clc_synthetic_desc* desc);
int clc_problem_destroy(clc_problem* p);

/* Sizes and read-back (tests / the C++ simulation driver). Any output pointer may be NULL. */
int clc_problem_sizes(const clc_problem* p, int64_t* n_frames, int64_t* n_points, int* has_edges);
int clc_problem_download(const clc_problem* p, double* frame_pose, int64_t* offsets, double* points,
                         double* edge_points, double* planes /* [n_frames*4] n,d in the camera frame */);
/* Synthetic problems with a camera model: the TRUE board poses [n_frames*7] (frame_pose above holds the estimated ones). */
int clc_problem_download_true_poses(const clc_problem* p, double* frame_pose_true);

/* THE FUSED KERNEL (K1): one sweep over every residual at `pose7` -> H = sum J~^T J~ (row-major 6x6),
 * g = sum J~^T r~, cost = 1/2 sum rho, with the Cauchy correction applied.  All-reduced over the ranks when a
 * communicator is attached.  replaces: one ceres Evaluate over all PointInPlaneFactor residual blocks,
 * reference src/LaseCamCalCeres.cpp:43-66 + Ceres Corrector.  Synchronous.  H36/g6 may be NULL. */
int clc_eval(clc_problem* p, const double pose7[7], double H36[36], double g6[6], double* cost);

/* replaces: ceres::Solve() at reference src/LaseCamCalCeres.cpp:306-307 with the options of :302-304.
 * pose7 is in/out.  trace may be NULL.  Collective over the communicator's ranks.
 * The whole Levenberg-Marquardt loop runs on the device: one K1 sweep per iteration, chained with programmatic dependent
 * launch, the host only polls a `done` flag; problems of the reference's own size (<= 16384 residuals, single rank) are solved
 * by ONE launch of the one-cluster kernel K2 (csrc/clc_small.cuh) that keeps the residuals in registers. */
int clc_solve_lm(clc_problem* p, double pose7[7], const clc_lm_options* opt, clc_lm_summary* summary,
                 clc_lm_iteration* trace, int trace_cap);

/* replaces: the analysis tail, reference src/LaseCamCalCeres.cpp:318-381: un-robustified H, b = -J^T r,
 * chi = sum r^2 (scale kept, no edge residuals), singular values of H (descending) and the matching right singular
 * vectors as the columns of V36 (row-major 6x6): the last n columns span the null space the reference prints when n
 * singular values are below 1e-8 (:368-379).  Any output may be NULL. */
int clc_information(clc_problem* p, const double pose7[7], double H36[36], double b6[6], double* chi,
                    double singular_values6[6], double V36[36]);

/* Per-frame report: every frame's residual statistics and its share of the normal equations, from ONE streaming sweep of the
 * device-resident problem at pose7 -- which frames drive the result, and which ones disagree with it.  Summed over the frames,
 * `cost` gives clc_eval's cost, H21 and g6 give clc_eval's H and g (upper triangle, K1's order), and `chi` gives
 * clc_information's chi, at the same pose (up to the order of summation).  With H and g of clc_eval, -(H - H_f)^-1 (g - g_f)
 * is a one-step estimate of how far the extrinsic moves without frame f (camlasercalibratool_b200.frame_influence). */
typedef struct {
  int64_t n_points;        /* points of the frame (0: empty frame, every other field 0) */
  double cost;             /* 1/2 sum rho over the frame's residuals (points + its edge residuals), the Cauchy loss as the problem has it */
  double chi;              /* s^2 sum e^2 over the points, no loss, no edges: the frame's share of clc_information's chi */
  double mean_e, rms_e, max_abs_e; /* metres, over the points, unweighted (max_abs_e is NaN when a point's distance is NaN) */
  double mean_weight;      /* sum w / n (1 without loss) */
  double edge_e[2];        /* raw residuals of the two edge residuals (0 without edges) */
  double H21[21], g6[6];   /* the frame's share of clc_eval's H (upper triangle, K1's order) and g */
} clc_frame_row;
/* rows[n_frames] (host memory the caller sizes: 288 bytes per frame), copied from the device once.  A problem attached to a
 * communicator reports its own frames (its clc_shard_range); no collective. */
int clc_frame_report(clc_problem* p, const double pose7[7], clc_frame_row* rows);

/* ---- frame selection: the frames that carry the most information about the extrinsic --------------------------------------
 * Greedy D-optimal selection over the report's per-frame information blocks: which frames to keep (clc_problem_subset takes the
 * keep mask) instead of a rule on how far the board moved.  Dwell (hundreds of frames that repeat one board pose) adds nothing
 * new, and a small turn about an axis no kept frame excites yet adds the most.  The rule:
 *   1. H_f is frame f's H21 of clc_frame_report at pose7, under the problem's loss (the same bytes).  Frame f is usable when its
 *      21 entries are finite; a frame that is not usable is never picked and never summed.
 *   2. Only the free coordinates of fixed_mask (clc_lm_options' bits 0-5) count: the principal d x d block, d = 6 - popcount.
 *   3. T = sum H_f over the usable frames whose state is not 0 (n_T of them).  A free T_kk that is not positive and finite fails
 *      with CLC_ERR_STATE, clc_last_error naming the coordinate: no frame observes it, so the caller must hold it.  D = diag(T)^-1/2
 *      and Ht_f = D H_f D (log det does not depend on the units of the coordinates, metres or radians).
 *   4. A_0 = sum of Ht_f over the usable forced frames + (CLC_SELECT_RIDGE / n_T) I.
 *   5. Step s: A_s = L L^T; every usable candidate not yet picked has gain_f = log det(I + L^-1 Ht_f L^-T) (in nats), formed from
 *      the pivots of the Cholesky factorisation of I + C_f (a pivot that is not positive and finite gives -inf).  The largest gain
 *      is picked, the lowest frame index on a tie.  The selection stops at s = budget, when no candidate is left, or when the best
 *      gain is <= min_gain; otherwise (f, gain_f) is recorded and A_{s+1} = A_s + Ht_f.
 * Outputs: *n_selected; order[n_selected] (frame indices in pick order) and gain[n_selected] (caller-sized: min(budget, n_frames)
 * entries each); keep[n_frames] = 1 for the forced and the picked frames, else 0.  A frame with zero information (an empty frame)
 * has gain 0 and is never picked at min_gain 0.  Every remaining candidate is evaluated at every step, on the device; two calls
 * return identical bytes, and the result does not depend on the device or its launch grid.
 * Rejected before any device work, with CLC_ERR_INVALID: a NULL desc or output, budget < 0, a min_gain that is NaN, negative or
 * infinite, a state value above 2, a fixed_mask outside [0, 63). */
#define CLC_SELECT_RIDGE 1e-6 /* A_0's ridge, a millionth of an average frame's scaled diagonal */
typedef struct {
  int64_t budget;       /* at most this many picks */
  double min_gain;      /* stop when the best gain is <= this (nats, finite, >= 0; 0 = stop only at zero information) */
  int fixed_mask;       /* coordinates left out of the information, as clc_lm_options.fixed_mask */
  const uint8_t* state; /* [n_frames] 0 = excluded, 1 = candidate, 2 = forced (kept, never picked); NULL = every frame a candidate */
} clc_select_desc;
/* The selection on p's report at pose7: the rows stay on the device (one report sweep, then the selection kernels).  A problem
 * attached to a communicator selects among its own frames. */
int clc_select_frames(clc_problem* p, const double pose7[7], const clc_select_desc* desc, int64_t* n_selected, int64_t* order,
                      double* gain, uint8_t* keep);
/* The same rule on rows the caller supplies (clc_frame_row, only H21 is read), uploaded once to `device` (-1: the current one). */
int clc_select_frames_rows(int device, int64_t n_frames, const clc_frame_row* rows, const clc_select_desc* desc, int64_t* n_selected,
                           int64_t* order, double* gain, uint8_t* keep);

/* Independent extrinsics of runs of consecutive frames (many rigs recorded into one problem, or time windows of one recording),
 * sharing every sweep of the device-resident problem: one pass over the points per evaluation or LM iteration, whatever the
 * number of segments.  Replaces W separate problems (clc_problem_subset of each run) and W clc_eval / clc_information /
 * clc_solve_lm calls.
 * A segmentation is seg_offsets[n_segments + 1] over the frames: seg_offsets[0] = 0, non-decreasing, seg_offsets[n_segments] =
 * n_frames, n_segments >= 1.  Segment s owns frames [seg_offsets[s], seg_offsets[s + 1]), their points and their edge residuals;
 * empty segments and segments of empty frames are valid.  poses[n_segments * 7]: one pose7 per segment.  Segment s's results
 * are those of the same call on a fresh problem holding its frames alone (clc_problem_create of the slice, same use_loss and
 * cauchy_a), up to the order of summation; an empty segment gets the fresh empty problem's.  A segment's results depend on its
 * own frames only: a NaN point in one segment leaves every other segment's outputs bit-identical.  Every problem size runs on the
 * sweep kernel K1; two calls return identical bytes.
 * Rejected before the device is touched, with CLC_ERR_INVALID: a NULL problem, seg_offsets or poses, n_segments < 1, a
 * seg_offsets that is not a segmentation of the problem's frames, a pose entry that is not finite.  A problem attached to a
 * communicator fails with CLC_ERR_STATE. */
/* clc_eval per segment: H36[n_segments * 36] (row-major 6x6) and g6[n_segments * 6] may be NULL; cost[n_segments] may not. */
int clc_eval_segments(clc_problem* p, int64_t n_segments, const int64_t* seg_offsets, const double* poses, double* H36, double* g6,
                      double* cost);
/* clc_information per segment (no loss, no edges): H36[n_segments * 36], b6[n_segments * 6], chi[n_segments],
 * singular_values6[n_segments * 6], V36[n_segments * 36]; each may be NULL. */
int clc_information_segments(clc_problem* p, int64_t n_segments, const int64_t* seg_offsets, const double* poses, double* H36,
                             double* b6, double* chi, double* singular_values6, double* V36);
/* clc_solve_lm per segment: n_segments LM solves, each from poses[s] (overwritten with its result), advancing side by side, one
 * shared sweep per iteration; a segment that has terminated stays as it is.  opt (NULL: defaults) holds for every segment.
 * summaries[n_segments]: as clc_solve_lm's, except that device_ms is the time of the whole segmented solve and num_sweeps the
 * segment's own count of sweeps that advanced it.  trace[n_segments * trace_cap]: segment s's iterations at trace[s * trace_cap],
 * its first min(num_iterations, trace_cap) rows written; trace_cap in [0, 256], trace may be NULL when trace_cap is 0 (no trace
 * memory is then allocated on the device).  NULL summaries, or a trace_cap outside [0, 256] or without trace, fail with
 * CLC_ERR_INVALID. */
int clc_solve_lm_segments(clc_problem* p, int64_t n_segments, const int64_t* seg_offsets, double* poses, const clc_lm_options* opt,
                          clc_lm_summary* summaries, clc_lm_iteration* trace, int trace_cap);

/* One calibration at many poses: K = n_poses poses over ALL frames of the problem, one shared pass over the points per
 * evaluation or LM iteration (a multi-start from K start poses, or the cost along a grid of poses).  poses[K * 7].
 * Pose k's row is what clc_eval / clc_solve_lm return at or from poses[k] on the same problem, up to the order of summation;
 * problems the one-cluster kernel serves (clc_debug_dispatch: CLC_PATH_ONE_CLUSTER, one cluster per pose in one launch) return
 * those bytes exactly.  Pose k's bytes depend on poses[k] only, not on K or the other poses: a K = 1 call returns the bytes of
 * that pose's row in a larger call, and permuting the poses permutes the outputs.  Two calls return identical bytes.  Every
 * loss kind of clc_problem_set_loss, with or without edge residuals, on both kernel families.
 * Rejected before the device is touched, with CLC_ERR_INVALID: a NULL problem or poses, n_poses outside [1, 1024], a pose entry
 * that is not finite.  A problem attached to a communicator fails with CLC_ERR_STATE.
 * Device memory for the length of a call, on problems the sweep kernel serves: about K * (44 * n_frames + 8 * n_edges) doubles
 * (every pose's frame constants, raw and expanded per-frame rows; 10^5 frames and K = 1024: about 36 GB), a failed allocation
 * returning CLC_ERR_CUDA.  On problems the one-cluster kernel serves: about 21 KB per start (its LM state with 256 trace rows). */
/* clc_eval per pose: H36[K * 36] (row-major 6x6) and g6[K * 6] may be NULL; cost[K] may not. */
int clc_eval_poses(clc_problem* p, int64_t n_poses, const double* poses, double* H36, double* g6, double* cost);
/* clc_solve_lm from every pose (overwritten with its result), the K solves advancing side by side; a start that has terminated
 * costs the later iterations nothing.  opt (NULL: defaults) holds for every start.  summaries[K] and trace[K * trace_cap] as
 * clc_solve_lm_segments' (device_ms: the time of the whole call; num_sweeps: the start's own sweeps; trace_cap in [0, 256]; when
 * it is 0, the sweep kernel's path allocates no trace memory on the device and the one-cluster path copies no trace rows).  *best (best may be NULL): the index of the lowest final_cost among the starts whose
 * termination is not CLC_TERM_FAILURE, the lowest index on a tie, -1 when every start failed.  NULL summaries, or a trace_cap
 * outside [0, 256] or without trace, fail with CLC_ERR_INVALID. */
int clc_solve_lm_starts(clc_problem* p, int64_t n_poses, double* poses, const clc_lm_options* opt, clc_lm_summary* summaries,
                        clc_lm_iteration* trace, int trace_cap, int64_t* best);

/* ---- the camera-laser time offset ------------------------------------------------------------------------------------------
 * Every other call takes frame f's board plane as exactly the one of its camera frame.  A scan is matched to the nearest camera
 * frame, and camera and laser stamps come from different clocks, so while the board moves that plane is off by the motion over the
 * quantisation error plus a constant clock offset -- a bias no amount of data averages out.  These calls estimate the offset td
 * (what is added to a laser time to put it on the camera clock) together with the extrinsic, from a board trajectory:
 *   - K >= 2 knots: times t_k (seconds, strictly increasing) and board poses in the frame_pose convention (qx qy qz qw tx ty tz of
 *     T_ca).  The library takes T_ac = T_ca^-1 with the normalised quaternion, and times relative to t_0 (subtracted once in
 *     double, exact for epoch stamps);
 *   - one scan time s_f per frame: frame f is evaluated at tau_f = s_f + td;
 *   - on [t_k, t_k+1) (the last interval includes its right end): t_ac lerped, q_ac = q_k (x) Exp(u w_k), u = (tau - t_k) / D_k,
 *     w_k = Log(q_k^-1 (x) q_k+1) on the shortest arc; outside [t_0, t_{K-1}] the end knot's pose, whose derivative is 0 (such a
 *     frame constrains T_cl and says nothing about td);
 *   - the plane n = R_ac^T e_z, d = t_ac,z (at a knot: frame_plane of that knot, up to rounding); the residual e = m.p + c as
 *     everywhere, scaled by 1/sqrt(#points), with the problem's loss; the Jacobian gains the column de/dtd.
 * H49 / V49 are row-major 7x7 over (tx ty tz rx ry rz td), g7 / b7 likewise.  Every problem size runs on the sweep kernel K1;
 * two calls return identical bytes.  Edge residuals are not modelled.
 * Rejected before the device is touched, with CLC_ERR_INVALID: a NULL problem or output-less argument (pose7, td), a problem with
 * edge residuals, a pose7 entry or td that is not finite; with CLC_ERR_STATE: a problem attached to a communicator, a problem
 * without a trajectory. */
/* Attaches the trajectory (n_knots >= 2: knot_times[n_knots], knot_poses[n_knots * 7], frame_times[n_frames]), replacing any
 * earlier one, or removes it (n_knots == 0; the arrays are then ignored).  The library keeps its own copy on the device (about
 * 8 (11 K + n_frames) bytes), freed by clc_problem_destroy.  clc_problem_subset and clc_problem_trim results carry no trajectory.
 * CLC_ERR_INVALID, leaving p unchanged: n_knots < 0 or == 1, a NULL array, knot times that are not finite or not strictly
 * increasing, a knot pose entry that is not finite or a zero quaternion, a frame time that is not finite, a problem with edge
 * residuals; CLC_ERR_STATE: a problem attached to a communicator. */
int clc_problem_set_trajectory(clc_problem* p, int64_t n_knots, const double* knot_times, const double* knot_poses,
                               const double* frame_times);
/* clc_eval with td: H49, g7 (may be NULL) and *cost (may be NULL) at (pose7, td). */
int clc_eval_time_offset(clc_problem* p, const double pose7[7], double td, double H49[49], double g7[7], double* cost);
/* clc_information with td (no loss): H49, b7 = -g, chi, the singular values of H (descending) and the matching right singular
 * vectors as the columns of V49 -- the observability of td: a board that never moved gives a zero singular value whose V column
 * is +-e_td.  Any output may be NULL. */
int clc_information_time_offset(clc_problem* p, const double pose7[7], double td, double H49[49], double b7[7], double* chi,
                                double singular_values7[7], double V49[49]);
/* clc_solve_lm on two parameter blocks: the pose (the reference's PoseLocalParameterization) and td (a 1-vector), both in/out.
 * Ceres' LM over 7 columns: Jacobi scaling, the LM diagonal, the damped Cholesky step and the model cost change over 7 columns,
 * the parameter tolerance on the 8-vector (pose7, td), gradient_max_norm = max(|x - Plus(x, -g)|_inf over the pose, |g_td|).
 * opt->fixed_mask bits 0-5 as in clc_solve_lm; bit 6 holds td at its start bits (bits 0-5 all set: only the offset is estimated,
 * the extrinsic already known).  summary (may be NULL) and trace as clc_solve_lm's; device_ms covers the whole solve.  Also
 * CLC_ERR_INVALID, checked first: a fixed_mask outside [0, 127), a trace_cap outside [0, 256] or > 0 without trace. */
int clc_solve_lm_time_offset(clc_problem* p, double pose7[7], double* td, const clc_lm_options* opt, clc_lm_summary* summary,
                             clc_lm_iteration* trace, int trace_cap);

/* ---- the laser's range offset b and range scale s, estimated with the extrinsic ----
 * A point p the laser reported at range r = |p| along the ray u = p / r is taken to lie at range (1 + s) r + b on the same ray,
 * whose origin is the laser's origin:
 *   p' = (1 + s) p + b u = kappa p,   kappa = (1 + s) + b / r;
 * at r == 0 the p / r terms are 0 and p' = (1 + s) p = 0.  A NaN coordinate propagates as everywhere else.  The residual is the
 * reference's at p': e = kappa (m.p) + c (m = R_cl^T n, c = n.t_cl + d), scaled by 1/sqrt(#points), with the problem's loss.  The
 * tangent space is (tx ty tz rx ry rz b s): the pose columns at p', de/db = (m.p) / r, de/ds = m.p.  H64 / V64 are row-major 8x8
 * over it, g8 / b8 likewise; bias2 = (b, s), b in the points' unit.  Every problem size runs on the sweep kernel K1; two calls
 * return identical bytes.  Edge residuals are not modelled.
 * Observability: an offset b is seen because its correction b u changes direction across a frame, and the scale s is told apart
 * from b by boards seen at different ranges.  Boards in a narrow band of ranges leave s and b nearly collinear with the
 * translation: clc_information_range_bias then shows a small singular value whose V column lies in the span of e_b, e_s and the
 * translation; holding s (fixed_mask bit 7) restores full rank.
 * Rejected before the device is touched, with CLC_ERR_INVALID: a NULL problem or argument (pose7, bias2), a problem with edge
 * residuals, a pose7 or bias2 entry that is not finite; with CLC_ERR_STATE: a problem attached to a communicator. */
/* clc_eval at (pose7, b, s): H64, g8 (may be NULL) and *cost (may be NULL). */
int clc_eval_range_bias(clc_problem* p, const double pose7[7], const double bias2[2], double H64[64], double g8[8], double* cost);
/* clc_information at (pose7, b, s) (no loss): H64, b8 = -g, chi, the singular values of H (descending) and the matching right
 * singular vectors as the columns of V64.  Any output may be NULL. */
int clc_information_range_bias(clc_problem* p, const double pose7[7], const double bias2[2], double H64[64], double b8[8], double* chi,
                               double singular_values8[8], double V64[64]);
/* clc_solve_lm on three parameter blocks: the pose (the reference's PoseLocalParameterization), b and s (1-vectors), all in/out.
 * Ceres' LM over 8 columns, the parameter tolerance on the 9-vector (pose7, b, s), gradient_max_norm = max(|x - Plus(x, -g)|_inf
 * over the pose, |g_b|, |g_s|).  opt->fixed_mask bits 0-5 as in clc_solve_lm; bit 6 holds b, bit 7 holds s at their start bits.
 * summary (may be NULL) and trace as clc_solve_lm's; device_ms covers the whole solve.  Also CLC_ERR_INVALID, checked first: a
 * fixed_mask outside [0, 255), a trace_cap outside [0, 256] or > 0 without trace. */
int clc_solve_lm_range_bias(clc_problem* p, double pose7[7], double bias2[2], const clc_lm_options* opt, clc_lm_summary* summary,
                            clc_lm_iteration* trace, int trace_cap);
/* A new problem on src's device whose points are kappa p of src's (the same frames, planes, poses and loss): every other call
 * then runs on the corrected points -- trim, quantiles, frame report, select, segments, starts.  Computed on the device from src's
 * points (nothing is uploaded but the copy's frame offsets and gather plan); two calls give identical points.  Owned by the caller
 * (clc_problem_destroy).  CLC_ERR_INVALID before any device work: a NULL argument, a bias2 entry that is not finite, 1 + s <= 0,
 * a problem with edge residuals. */
int clc_problem_range_correct(const clc_problem* src, const double bias2[2], clc_problem** out);

/* replaces: CamLaserCalClosedSolution(), reference src/LaseCamCalCeres.cpp:112-203.  Tlc16 row-major.
 * AtA81/Atb9 (the 9x9 normal equations) may be NULL. */
int clc_closed_form(clc_problem* p, double Tlc16[16], int* unobservable, double AtA81[81], double Atb9[9]);

/* replaces: LineFittingCeres(), reference src/LaseCamCalCeres.cpp:385-433 (the step before the solve: SURVEY.md 8(f)),
 * batched: fits m0 x + m1 y + 1 = 0 (CauchyLoss(0.05), <= max_num_iterations Ceres LM iterations, reference: 10) to
 * the x,y of every frame's points of the problem, one warp per frame, the whole loop on the device.
 * lines[n_frames*2] (host): start values in (the reference's caller passes them uninitialised), fits out.
 * info[n_frames*4] (host, optional): termination code, LM iterations, sweeps, final cost per frame.
 * Local to the rank's shard (no collective). */
int clc_problem_line_fit(clc_problem* p, double* lines, int max_num_iterations, double* info);
/* The reference's per-scan call shape: one scan of n points (AoS xyz, z ignored), line[2] in/out. */
int clc_line_fit_points(const double* points_xyz, int64_t n, double line[2], int max_num_iterations);

/* replaces: TranScanToPoints() + AutoGetLinePts(), reference src/utilities.cpp:181-215 and src/selectScanPoints.cpp:17-190
 * (without the OpenCV debug drawing), batched over scans: for every LaserScan (n_beams float ranges, angle of beam i =
 * angle_min + i * angle_increment) the inclusive beam-index range [seg_start, seg_end] of the laser segment on the board,
 * or -1/-1 when none is found.  Host arrays in/out; device = CUDA ordinal or -1. */
int clc_scan_segments(const float* ranges, int64_t n_scans, int64_t n_beams, double angle_min, double angle_increment,
                      double range_min, int32_t* seg_start, int32_t* seg_end, int device);

/* Board poses from detected tag corners, batched: the arithmetic of CamPoseEst::calcCamPose after the tag detector
 * (reference src/calcCamPose.cpp:270-294: liftProjective of every corner, x/z y/z as cv::Point2f) and of
 * CamPoseEst::EstimatePose (:211-236: solvePnP with identity intrinsics on the kalibr-grid object points :114-136,
 * T_wc = T_cw^-1) -- what main/kalibratag_detector_node.cpp turns into apriltag_pose.txt.  No image processing.
 * camera_model 1 = pinhole + radtan (fx fy cx cy k1 k2 p1 p2), 2 = equidistant / Kannala-Brandt (mu mv u0 v0 k2 k3 k4 k5).
 * Frame f owns detections det_offsets[f] .. det_offsets[f+1] (ascending tag id); corners_uv[D*8] = 4 corners (u, v) per
 * detection in detector order.  pose_wc[n_frames*7] = (qx qy qz qw x y z) of T_wc; ok[f] = 0 (identity pose) for fewer
 * than 4 points, a tag id outside the grid or a degenerate configuration. */
typedef struct clc_camera_desc {
  int camera_model;
  double intrinsics[8];
  int grid_rows, grid_cols; /* april grid; a single tag is a 1 x 1 grid */
  double tag_size;          /* metres */
  double tag_spacing;       /* gap / tag_size (kalibr convention) */
} clc_camera_desc;
int clc_estimate_board_poses(const clc_camera_desc* cam, int64_t n_frames, const int64_t* det_offsets, const int32_t* tag_ids,
                             const float* corners_uv, double* pose_wc, int32_t* ok, int device);

/* Eigen-equivalent conversions used on both sides of the boundary (reference :215-219 and :311-314). */
void clc_T_to_pose7(const double T16[16], double pose7[7]);
void clc_pose7_to_T(const double pose7[7], double T16[16]);

/* ---- multi-GPU: one process per GPU, frames sharded by the caller, 28-double all-reduce per sweep ---------- */
/* Balanced contiguous frame range of `rank` (by point count when offsets != NULL, else by frame count). */
int clc_shard_range(int64_t n_frames, const int64_t* offsets, int nranks, int rank, int64_t* begin, int64_t* end);
/* NCCL bootstrap: rank 0 calls clc_comm_unique_id, ships the 128 bytes to every rank by any means
 * (torch.distributed, MPI, a file); every rank creates its communicator (collective) and attaches it to any number
 * of problems on that device.  The communicator is borrowed: it must outlive the problems it is attached to.
 * Attaching NULL detaches. */
typedef struct clc_comm clc_comm;
int clc_comm_unique_id(void* id128);
int clc_comm_create(clc_comm** out, const void* id128, int nranks, int rank, int device);
int clc_comm_destroy(clc_comm* comm);
int clc_problem_attach_comm(clc_problem* p, clc_comm* comm);
/* Fused all-reduce over NVLink peer memory: every rank exports a 64-byte IPC handle of its mailbox, the handles of
 * all ranks (rank order, nranks*64 bytes) are shipped to every rank by any means, and every rank imports them.  From
 * then on the last block of every sweep kernel exchanges the 28 sums with direct peer stores and runs the LM update in
 * the same launch (no NCCL call, no extra kernel).  Requires one process per GPU on one NVLink/NVSwitch node. */
int clc_comm_p2p_export(clc_comm* comm, void* handle64);
int clc_comm_p2p_import(clc_comm* comm, const void* handles /* [nranks*64] */);
/* all-reduce mode of a problem: 0 = ncclAllReduce on the solve stream between the kernels,
 * 1 = fused in-kernel peer exchange (needs clc_comm_p2p_import; the default once it has been called) */
int clc_problem_set_allreduce_mode(clc_problem* p, int mode);

/* ---- in-process multi-GPU: ONE process (one host thread) drives G devices ---------------------------------------
 * What lets the unmodified reference callers (main/calibr_simulation.cpp:130, main/calibr_offline.cpp:170 -- one call of
 * CamLaserCalibration() from one process) use every GPU of the box: the frames are sharded over the devices by point
 * count (clc_shard_range), every device holds its shard for the whole solve, and the last block of every sweep kernel
 * exchanges the 28 sums with plain peer stores (cudaDeviceEnablePeerAccess; the same sequence-tagged mailbox protocol as
 * the multi-process path, no IPC handles, no NCCL).  All devices run the identical LM update.  A group of one device is
 * a plain problem.  devices[i] = CUDA ordinal (-1 = current); an ordinal may appear only once. */
typedef struct clc_group clc_group;
int clc_group_create_gather(clc_group** out, const clc_gather_desc* desc, const int* devices, int n_devices);
/* desc->frame_begin..frame_end is the range the GROUP holds (split evenly over its devices); desc->device is ignored */
int clc_group_create_synthetic(clc_group** out, const clc_synthetic_desc* desc, const int* devices, int n_devices);
int clc_group_destroy(clc_group* g);
int clc_group_size(const clc_group* g, int* n_devices, int64_t* n_frames, int64_t* n_points);
int clc_group_problem(clc_group* g, int index, clc_problem** out); /* borrowed: shard `index` (tests, measurement) */
/* the collective forms of clc_eval / clc_solve_lm / clc_information / clc_closed_form (same outputs) */
int clc_group_eval(clc_group* g, const double pose7[7], double H36[36], double g6[6], double* cost);
int clc_group_solve_lm(clc_group* g, double pose7[7], const clc_lm_options* opt, clc_lm_summary* summary,
                       clc_lm_iteration* trace, int trace_cap);
int clc_group_information(clc_group* g, const double pose7[7], double H36[36], double b6[6], double* chi,
                          double singular_values6[6], double V36[36]);
int clc_group_closed_form(clc_group* g, double Tlc16[16], int* unobservable, double AtA81[81], double Atb9[9]);
/* clc_frame_report of every shard: rows[all frames of the group], in the global frame order */
int clc_group_frame_report(clc_group* g, const double pose7[7], clc_frame_row* rows);
/* clc_select_frames for the group: the report rows of every shard in the global frame order (clc_group_frame_report), then
 * clc_select_frames_rows on the group's first device; order and keep are in the global frame order. */
int clc_group_select_frames(clc_group* g, const double pose7[7], const clc_select_desc* desc, int64_t* n_selected, int64_t* order,
                            double* gain, uint8_t* keep);
/* ---- subsets: solve again without some frames, without sending the points through the host again -----------------------
 * A new problem on src's device holding only the frames with keep[f] == 1 (keep has src's n_frames entries, each 0 or 1), in
 * their original order, built from src's device-resident data: only src's frame offsets come to the host, a gather kernel copies
 * the kept points and per-frame arrays.  The result is the problem clc_problem_create would build from the kept frames' poses,
 * points and edge points -- the same layout, planes, planarity verdict, kernel family, partition and dispatch, so every output is
 * bit-identical to that fresh problem's.  (One exception in the stored bytes: the sign of a z that is -0.0 or +0.0.  A fresh upload
 * stores such a z as +0.0 or as given depending on whether a z != 0 shares its upload chunk; the subset copies it as the source
 * holds it, or writes +0.0 where the source has no z stream.  Both signs give the same results.)  It inherits use_loss, cauchy_a and (synthetic camera-mode sources) the true poses; it
 * starts in the default planar mode and is attached to no communicator.  src is unchanged and stays valid; both need device
 * memory at once.  Keeping every frame or none is valid.  A NULL argument or a keep entry other than 0 or 1 fails with
 * CLC_ERR_INVALID before the device is touched. */
int clc_problem_subset(const clc_problem* src, const uint8_t* keep, clc_problem** out);
/* The same for an in-process group: a new group on the same device list, the kept frames re-sharded over it as
 * clc_group_create_gather shards a fresh problem.  Kept points on another device are read over the peer links: for the gather,
 * each source device's default memory pool is opened to the other devices of the group (cudaMemPoolSetAccess) and closed again
 * afterwards, unless the caller had already granted that access. */
int clc_group_subset(const clc_group* src, const uint8_t* keep, clc_group** out);
/* ---- trims: solve again without the points that lie far from their board, without sending the points through the host again --
 * A new problem on src's device holding, of every frame f of src, the points whose raw point-to-plane distance at pose7 satisfies
 * |e| <= max_abs_e[f] (max_abs_e has src's n_frames entries).  e is computed exactly as the sweep kernel and clc_frame_report
 * compute it -- m = R^T n, c = n.t + d from pose7 and the frame's board plane, e = fma(m0, x, fma(m1, y, fma(m2, z, c))) -- so
 * the report's max_abs_e and the threshold are the same quantity.  A NaN e is never kept; max_abs_e[f] = +inf keeps every point of
 * frame f whose e is not NaN.  Every frame is kept, in order, with its pose, its edge points (the front and back points of the raw
 * scan, which are not trimmed) and (synthetic camera-mode sources) its true pose; a frame may end up empty (clc_problem_subset
 * removes such frames).  Only the kept counts of every frame and of every 2048-point tile come to the host; a mark kernel and a
 * gather kernel do the rest.  The result is the problem clc_problem_create would build from src's frame poses, the kept points and
 * src's edge points -- the same layout, planes, planarity verdict, kernel family, partition and dispatch, so every output is
 * bit-identical to that fresh problem's.  In particular the per-frame scale s = 1/sqrt(#points of the frame) follows the new point
 * counts (reference src/LaseCamCalCeres.cpp:239-240), and a problem whose only z != 0 were trimmed is planar when it is large
 * enough.  The +-0.0 exception of clc_problem_subset applies unchanged.  It inherits use_loss and cauchy_a; it starts in the
 * default planar mode and is attached to no communicator.  src is unchanged and stays valid; both need device memory at once.
 * A NULL argument, a pose7 entry that is not finite or a max_abs_e entry that is NaN or negative fails with CLC_ERR_INVALID
 * before the device is touched. */
int clc_problem_trim(const clc_problem* src, const double pose7[7], const double* max_abs_e, clc_problem** out);
/* The same for an in-process group (max_abs_e: one entry per frame of the group, in the global frame order): a new group on the
 * same device list, the trimmed frames re-sharded over it by their new point counts as clc_group_create_gather shards a fresh
 * problem, so shard boundaries move and kept points may cross devices.  They are read over the peer links under the same
 * temporary memory-pool grants as clc_group_subset's. */
int clc_group_trim(const clc_group* src, const double pose7[7], const double* max_abs_e, clc_group** out);
/* ---- exact quantiles of the point-to-board distances ----------------------------------------------------------------------
 * e is the raw point-to-plane distance of a laser point at pose7, computed exactly as the sweep kernel, clc_frame_report and
 * clc_problem_trim compute it: m = R^T n, c = n.t + d from pose7 and the frame's board plane, e = fma(m0, x, fma(m1, y, fma(m2, z,
 * c))).  No scale s and no loss enter it, and the edge residuals are not among the values.  The quantiles are taken over |e|
 * (fabs, so -0.0 counts as +0.0).  A NaN |e| is left out and not counted in n_valid; +inf is valid and sorts last.
 * Rank rule: with the n valid values sorted ascending, v_0 <= ... <= v_{n-1}, quantile q in [0, 1] is v_k with
 * k = clamp(ceil(q * n) - 1, 0, n - 1), q * n a double product.  q = 0 is the minimum, q = 1 the maximum, q = 0.5 the lower
 * median.  With n = 0 the value is NaN.  A result is one element of the multiset of |e|, so it does not depend on the device, the
 * grid or the order of any atomic: two calls give identical bytes.
 * A problem attached to a communicator answers for its own points and frames, with no collective (as clc_frame_report).
 * Rejected with CLC_ERR_INVALID before any device work: a NULL argument, n_q outside [1, CLC_QUANTILES_MAX], a q that is NaN or
 * outside [0, 1], a pose7 entry that is not finite, a point range outside [0, n_points]. */
#define CLC_QUANTILES_MAX 16
/* The signed e of points [first, first + count) of p, in point order, into e[count] (host memory; e may be NULL when count is 0).
 * A range lets a caller page through a problem larger than host memory. */
int clc_point_residuals(const clc_problem* p, const double pose7[7], int64_t first, int64_t count, double* e);
/* The quantiles q[n_q] of |e| over every point of p: values[n_q], *n_valid the number of valid (not NaN) |e|.  A radix select
 * on the bits of |e|: every requested rank advances in the same passes over the points (about two histogram passes and one
 * compacting pass on noisy data; at most 7 passes when massive ties, such as e == 0 everywhere, prevent compaction). */
int clc_residual_quantiles(clc_problem* p, const double pose7[7], int n_q, const double* q, double* values, int64_t* n_valid);
/* The same rule within every frame of p: values[n_frames * n_q] (row f holds frame f's quantiles in the order of q),
 * n_valid[n_frames].  One block per frame. */
int clc_frame_quantiles(clc_problem* p, const double pose7[7], int n_q, const double* q, double* values, int64_t* n_valid);
/* The same over an in-process group: the problem-wide values over every point of the group, the frame rows in the global frame
 * order.  Both are identical to those of a single problem holding the group's frames. */
int clc_group_residual_quantiles(clc_group* g, const double pose7[7], int n_q, const double* q, double* values, int64_t* n_valid);
int clc_group_frame_quantiles(clc_group* g, const double pose7[7], int n_q, const double* q, double* values, int64_t* n_valid);
/* clc_problem_set_loss on every shard of g (the clc_group_* calls use it; clc_group_subset / clc_group_trim inherit it). */
int clc_group_set_loss(clc_group* g, int kind, double a);
/* The device list the reference-facing drop-in uses (its signatures have no device argument): environment variable
 * CLC_DEVICES = "0,1,2,3" | "all" | unset (the current device only).  Writes at most `cap` ordinals. */
int clc_default_devices(int* devices, int cap, int* n);

/* ---- measurement hooks (bench.py) ---------------------------------------------------------------------- */
/* Launches K1 `n` times at pose7 on the problem's stream; each launch is bracketed by its own CUDA events.
 * flush_l2 != 0 overwrites a buffer larger than L2 between launches (outside the timed brackets).
 * ms_each[n] receives the per-launch device times.  No collective, local shard only. */
int clc_bench_eval(clc_problem* p, const double pose7[7], int n, int flush_l2, float* ms_each);
/* The same for clc_frame_report: each bracket holds the per-frame sweep and the split-frame fix-up, not the copy of the rows
 * to the host. */
int clc_bench_frame_report(clc_problem* p, const double pose7[7], int n, int flush_l2, float* ms_each);
/* The same for one iteration of the segmented calls: each bracket holds the frame constants, the segment sweep, the split-frame
 * fix-up and the two-level reduction into per-segment sums (clc_eval_segments without the copy to the host). */
int clc_bench_segments(clc_problem* p, int64_t n_segments, const int64_t* seg_offsets, const double* poses, int n, int flush_l2,
                       float* ms_each);
/* The same for one evaluation of clc_eval_poses on the path it picks: each bracket holds the K poses' frame constants, sweeps,
 * fix-up and reduction (or the one-cluster launch), not the copy to the host. */
int clc_bench_poses(clc_problem* p, int64_t n_poses, const double* poses, int n, int flush_l2, float* ms_each);
/* The same for one time-offset iteration at (pose7, td): each bracket holds the frames' planes and constants, the segment sweep,
 * the fix-up into 36 sums per frame and the two-level reduction (clc_eval_time_offset without the copy to the host). */
int clc_bench_time_offset(clc_problem* p, const double pose7[7], double td, int n, int flush_l2, float* ms_each);
/* The same for one range-bias iteration at (pose7, b, s): each bracket holds the frame constants, the kModeRange sweep, the fix-up
 * into 45 sums per frame and the two-level reduction (clc_eval_range_bias without the copy to the host). */
int clc_bench_range_bias(clc_problem* p, const double pose7[7], const double bias2[2], int n, int flush_l2, float* ms_each);
/* clc_select_frames(p, pose7, desc) with the report computed once and the selection run `n` times on its device rows: ms_each[n]
 * receives the device time of each selection, from its first kernel to the end of its last step (the host polls between step
 * batches included), and *n_selected the picks of the last run. */
int clc_bench_select(clc_problem* p, const double pose7[7], const clc_select_desc* desc, int n, float* ms_each, int64_t* n_selected);
/* The gather of clc_problem_subset(src, keep): `n` times a scratch subset is prepared, its gather kernel is timed alone (CUDA
 * events, after the L2 flush when flush_l2 != 0) and the scratch problem is destroyed.  ms_each[n] receives the device times.
 * Like clc_bench_eval, the flush leaves its 256 MiB buffer attached to src until src is destroyed. */
int clc_bench_subset(clc_problem* src, const uint8_t* keep, int n, int flush_l2, float* ms_each);
/* The two device passes of clc_problem_trim(src, pose7, max_abs_e): `n` times the mark kernel is timed (CUDA events, after the L2
 * flush when flush_l2 != 0), the kept counts come to the host and a scratch trim is prepared, then its gather kernel is timed the
 * same way and the scratch problem is destroyed.  mark_ms[n] and gather_ms[n] receive the device times; the host step between
 * the passes is in neither.  Like clc_bench_eval, the flush leaves its 256 MiB buffer attached to src until src is destroyed. */
int clc_bench_trim(clc_problem* src, const double pose7[7], const double* max_abs_e, int n, int flush_l2, float* mark_ms,
                   float* gather_ms);
/* clc_residual_quantiles(p, pose7, n_q, q) `n` times, then clc_frame_quantiles `n` times, each after the L2 flush when flush_l2 != 0.
 * ms_each[n] receives the device time of every problem-wide call, from its first pass to the end of its last (the host steps
 * between the passes included); frame_ms_each[n] the device time of every per-frame kernel, not the copy to the host; *passes the
 * passes over the point streams the problem-wide call made.  Like clc_bench_eval, the flush leaves its 256 MiB buffer attached to p
 * until p is destroyed. */
int clc_bench_quantiles(clc_problem* p, const double pose7[7], int n_q, const double* q, int n, int flush_l2, float* ms_each,
                        float* frame_ms_each, int* passes);
/* Algorithmic bytes of one K1 launch on this problem: 24*P + 40*N + 56*edges + 224 (SURVEY.md section 8(d)). */
int clc_problem_algorithmic_bytes(const clc_problem* p, int64_t* bytes);
/* Bytes one K1 launch actually streams: the figure above with 16 instead of 24 bytes per point when the planar
 * (two-stream) kernels are active. */
int clc_problem_streamed_bytes(const clc_problem* p, int64_t* bytes);
/* Planar data.  A 2-D laser delivers z == 0 for every point (reference src/utilities.cpp:207, main/calibr_simulation.cpp:82,88,
 * main/calibr_offline.cpp:141-142) although Oberserve::points is a Vector3d.  The upload detects this; the library then
 * drops the z stream from HBM and runs two-stream kernels whose results equal the general ones (up to summation order) on such
 * data (SURVEY.md 8(d): a separate roofline row, 16 B per residual).  mode 1 = automatic (default), 0 = always the
 * general three-stream kernels (an all-zero z stream is re-materialised if it was dropped).  Problems too small to give
 * every warp of the grid a 256-point stage (about 4*10^5 points on an H100) are latency-bound and stay on the general
 * kernels in either mode (environment override for tests: CLC_PLANAR_MIN_POINTS). */
int clc_problem_set_planar_mode(clc_problem* p, int mode);
/* Robust losses (Ceres' LossFunction objects).  Every frame scales its residuals r = s e by s = 1/sqrt(#points) and uses the
 * loss with parameter a*s (reference src/LaseCamCalCeres.cpp:249); the scale cancels from the weights.  With z = e^2/a^2, a
 * frame's cost is 1/2 s^2 sum rho~(e) over its points and edge residuals:
 *   CLC_LOSS_NONE      no loss               w = 1                          rho~ = e^2
 *   CLC_LOSS_CAUCHY    CauchyLoss(a*s)       w = 1/(1+z)                    rho~ = a^2 log(1+z)
 *   CLC_LOSS_HUBER     HuberLoss(a*s)        w = 1 if |e| <= a, else a/|e|  rho~ = e^2 if |e| <= a, else 2a|e| - a^2
 *   CLC_LOSS_SOFT_L1   SoftLOneLoss(a*s)     w = 1/sqrt(1+z)                rho~ = 2a^2 (sqrt(1+z) - 1)
 * A point with |e| == a is a Huber inlier.  The reference hard-codes CauchyLoss(0.05*scale) (:248 keeps a HuberLoss line
 * commented out); creation maps use_loss = 1 to CAUCHY(cauchy_a) and use_loss = 0 to NONE(cauchy_a). */
#define CLC_LOSS_NONE 0
#define CLC_LOSS_CAUCHY 1
#define CLC_LOSS_HUBER 2
#define CLC_LOSS_SOFT_L1 3
/* The loss of every later clc_eval, clc_solve_lm, clc_frame_report, clc_eval_segments, clc_solve_lm_segments and
 * clc_bench_eval / _frame_report / _segments call on p; clc_problem_subset and clc_problem_trim inherit it.  clc_information,
 * clc_closed_form and the segment information never use a loss, clc_problem_line_fit keeps its own CauchyLoss(cauchy_a) and
 * the trim's distances are raw: none of them change.  Fails with CLC_ERR_INVALID, leaving p unchanged, for an unknown kind,
 * or an a that is not finite and positive with a^2 a normal double.  On a problem attached to a communicator every rank must
 * set the same loss (not checked). */
int clc_problem_set_loss(clc_problem* p, int kind, double a);
/* The loss kind (CLC_LOSS_*) and parameter a of p. */
int clc_problem_get_loss(const clc_problem* p, int* kind, double* a);
/* Statistics of this process's most recent host -> HBM point upload: wall time of the pipeline, time the issuing thread
 * waited for the pack threads, bytes that crossed PCIe (16 per point while every z is 0, else 24), chunks, pack threads,
 * direct = 1 when the caller's buffer was pinned and used as the DMA source.  Any pointer may be NULL. */
int clc_upload_last_stats(double* total_ms, double* pack_wait_ms, int64_t* bytes_h2d, int* chunks, int* pack_threads,
                          int* direct);
/* Test hook, no CUDA: what the pack threads write for the local point range [a, b) of a gathered problem -- packed x,y
 * pairs (xy != 0; *nonplanar = a z != 0 or NaN was met) or packed x,y,z. */
int clc_debug_pack(int64_t n_frames, const double* const* frame_points, const int64_t* frame_counts, int64_t a, int64_t b,
                   int xy, double* out, int* nonplanar);
/* Test hook, read-only: the static work partition of the sweep kernel for the problem's active kernel family -- launch grid
 * (blocks), points per warp range, points per pipeline stage, stages per warp kept in L2 during LM solves -- and, when
 * warp_first_frame is not NULL ([grid * 12] ints), the frame that holds the first point of every warp range. */
int clc_debug_partition(const clc_problem* p, int* grid, int64_t* per_warp, int* stage_points, int* resident_chunks,
                        int* warp_first_frame);
/* The kernels clc_debug_dispatch reports. */
#define CLC_PATH_ONE_CLUSTER 1        /* the one-cluster kernel: one launch per evaluation, or the whole LM solve */
#define CLC_PATH_SINGLE_BLOCK 2       /* the sweep kernel on one block, one launch per evaluation / LM iteration */
#define CLC_PATH_SINGLE_BLOCK_LOOP 3  /* the sweep kernel on one block, the whole LM loop in one launch */
#define CLC_PATH_MULTI_BLOCK 4        /* the sweep kernel on several blocks, one launch per evaluation / LM iteration */
#define CLC_PATH_MULTI_BLOCK_LOOP 5   /* the persistent looping grid of the sweep kernel, the whole LM loop in one launch */
/* Test hook, read-only: the kernel (CLC_PATH_*) that clc_eval, clc_information, clc_closed_form and clc_solve_lm run on for
 * this problem under the knobs read at its creation, and (small_shape != NULL, [3] ints) the one-cluster kernel's shape:
 * threads per CTA, CTAs per cluster, residuals per thread.  Any pointer may be NULL. */
int clc_debug_dispatch(const clc_problem* p, int* eval_path, int* information_path, int* closed_form_path, int* solve_path,
                       int* small_shape);
/* Raw PCIe yardstick: `reps` host(pinned) -> device copies of `bytes` on `device`, each timed with CUDA events. */
int clc_bench_h2d(int64_t bytes, int device, int reps, float* ms_each);
/* Bytes clc_solve_lm reads back per solve (LM state + iteration trace). */
int64_t clc_solve_readback_bytes(void);
/* Pinned host memory for upload buffers. */
int clc_host_alloc(void** ptr, int64_t bytes);
int clc_host_free(void* ptr);
/* Number of kernel launches issued by this library since load (bench.py's gpu_launches). */
int64_t clc_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* CLC_B200_H */
