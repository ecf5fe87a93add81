"""Python mirror of the reference's solver interface, on top of the C ABI (include/clc_b200.h).

Mirrors reference include/LaseCamCalCeres.h:11-29: the ``Oberserve`` struct (sic) and the free functions
``CamLaserCalibration`` / ``CamLaserCalClosedSolution`` with the same argument meaning (in/out 4x4 transform,
``use_linefitting_data``, ``use_boundary_constraint``).  Everything numeric happens in libclc_b200.so on the GPU;
this module only marshals ``list[Oberserve]`` into the flat arrays of the ABI.  (The C++ drop-in with the exact
reference signatures is camlasercalibratool_b200/host/LaseCamCalB200.cpp.)
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import NamedTuple

import numpy as np

from . import _lib
from ._lib import ClcError, GatherDesc, LmIteration, LmOptions, LmSummary, ProblemDesc, SelectDesc, SyntheticDesc, TERMINATION


def _dp(a):
    return a.ctypes.data_as(_lib.c_double_p) if a is not None else None


def _ip(a):
    return a.ctypes.data_as(_lib.c_int64_p) if a is not None else None


@dataclass
class Oberserve:
    """reference include/LaseCamCalCeres.h:11-24 (the misspelling is the reference's)."""

    tagPose_Qca: np.ndarray = field(default_factory=lambda: np.array([0.0, 0.0, 0.0, 1.0]))  # Eigen coeffs x,y,z,w
    tagPose_tca: np.ndarray = field(default_factory=lambda: np.zeros(3))
    points: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))
    points_on_line: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))


def marshal(obs, use_linefitting_data=True, use_boundary_constraint=False):
    """list[Oberserve] -> (frame_pose[N,7], offsets[N+1], points[P,3], edge_points[N,6] | None).

    Point-set selection as reference src/LaseCamCalCeres.cpp:233-237; the edge residuals exist only when both
    flags are set (:258) and use obs.points.front()/back() (:278-279)."""
    n = len(obs)
    frame_pose = np.zeros((n, 7))
    counts = np.zeros(n + 1, dtype=np.int64)
    chunks = []
    want_edges = bool(use_boundary_constraint and use_linefitting_data)
    edge = np.zeros((n, 6)) if want_edges else None
    for i, ob in enumerate(obs):
        frame_pose[i, :4] = np.asarray(ob.tagPose_Qca, dtype=np.float64)
        frame_pose[i, 4:] = np.asarray(ob.tagPose_tca, dtype=np.float64)
        pts = np.asarray(ob.points_on_line if use_linefitting_data else ob.points, dtype=np.float64).reshape(-1, 3)
        counts[i + 1] = pts.shape[0]
        chunks.append(pts)
        if want_edges and pts.shape[0] > 0:
            raw = np.asarray(ob.points, dtype=np.float64).reshape(-1, 3)
            if raw.shape[0] == 0:
                raise ValueError("use_boundary_constraint needs obs.points (reference :278 calls points.at(0))")
            edge[i, :3] = raw[0]
            edge[i, 3:] = raw[-1]
    offsets = np.cumsum(counts)
    points = np.concatenate(chunks, axis=0) if chunks else np.zeros((0, 3))
    return frame_pose, offsets, np.ascontiguousarray(points), edge


# intrinsics of the reference's two shipped configurations
CAMERA_DEFAULTS = {
    # config/calibra_config_pinhole.yaml (its distortion block is all zeros; a mild radtan distortion is used instead so that
    # the undistortion step does something)
    "radtan": [367.049931000148, 366.94446918887405, 368.7202381120387, 241.13814795878562, -0.05, 0.01, 0.0005, -0.0005],
    # config/calibra_config.yaml (KANNALA_BRANDT)
    "equi": [367.049931000148, 366.94446918887405, 368.7202381120387, 241.13814795878562, -0.02276964, -0.00056958, -0.0026224,
             0.00017455],
}


class _Gather:
    """Keeps the arrays of a clc_gather_desc alive: one separate [n_i, 3] array per frame, as std::vector<Oberserve> holds
    them (reference include/LaseCamCalCeres.h:22-23)."""

    def __init__(self, frame_pose, frames, edge_points=None, use_loss=True, cauchy_a=0.05, device=-1):
        self.frame_pose = np.ascontiguousarray(frame_pose, dtype=np.float64).reshape(-1, 7)
        self.frames = [np.ascontiguousarray(f, dtype=np.float64).reshape(-1, 3) for f in frames]
        n = self.frame_pose.shape[0]
        if len(self.frames) != n:
            raise ValueError("one point array per frame is needed")
        self.counts = np.array([f.shape[0] for f in self.frames], dtype=np.int64)
        self.ptrs = (_lib.c_double_p * max(n, 1))(*[_dp(f) for f in self.frames])
        self.edge = None
        if edge_points is not None:
            self.edge = np.ascontiguousarray(edge_points, dtype=np.float64).reshape(-1, 6)
            if self.edge.shape[0] != n:
                raise ValueError("edge_points must be [n_frames, 6]")
        d = GatherDesc()
        d.n_frames = n
        d.frame_pose, d.frame_points, d.frame_counts, d.edge_points = _dp(self.frame_pose), self.ptrs, _ip(self.counts), _dp(self.edge)
        d.use_loss, d.cauchy_a, d.device = int(bool(use_loss)), float(cauchy_a), int(device)
        self.desc = d


def _synthetic_desc(n_frames_total, beams, seed, sigma, with_edges, frame_begin, frame_end, use_loss, cauchy_a, device, camera,
                    pixel_sigma, intrinsics, image_size, grid):
    d = SyntheticDesc()
    d.n_frames_total = int(n_frames_total)
    d.frame_begin = int(frame_begin)
    d.frame_end = int(n_frames_total if frame_end is None else frame_end)
    d.beams, d.seed, d.sigma = int(beams), int(seed), float(sigma)
    d.with_edges, d.use_loss, d.cauchy_a, d.device = int(bool(with_edges)), int(bool(use_loss)), float(cauchy_a), int(device)
    d.camera_model = {None: 0, "none": 0, "radtan": 1, "pinhole": 1, "equi": 2}[camera]
    if d.camera_model:
        k = CAMERA_DEFAULTS["radtan" if d.camera_model == 1 else "equi"] if intrinsics is None else intrinsics
        d.camera_intrinsics = (C.c_double * 8)(*[float(v) for v in k])
        d.pixel_sigma = float(pixel_sigma)
        d.image_width, d.image_height = int(image_size[0]), int(image_size[1])
        d.grid_rows, d.grid_cols, d.tag_size, d.tag_spacing = int(grid[0]), int(grid[1]), float(grid[2]), float(grid[3])
    return d


# clc_frame_row (include/clc_b200.h) as a numpy record: Problem.frame_report / Group.frame_report return arrays of it
FRAME_ROW_DTYPE = np.dtype([("n_points", np.int64), ("cost", np.float64), ("chi", np.float64), ("mean_e", np.float64),
                            ("rms_e", np.float64), ("max_abs_e", np.float64), ("mean_weight", np.float64),
                            ("edge_e", np.float64, (2,)), ("H21", np.float64, (21,)), ("g6", np.float64, (6,))])
assert FRAME_ROW_DTYPE.itemsize == C.sizeof(_lib.FrameRow)


def _frame_report(fn, handle, n_frames, pose7, what):
    pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
    rows = np.zeros(n_frames, dtype=FRAME_ROW_DTYPE)
    _lib.check(fn(handle, _dp(pose7), rows.ctypes.data_as(C.c_void_p)), what)
    return rows


def frame_influence(report, H, g):
    """One-step leave-one-frame-out estimate of how far the extrinsic moves without each frame.

    report: a frame report (Problem.frame_report) and H [6,6], g [6]: clc_eval's at the same pose.  For every frame f,
    delta_f = -(H - H_f)^-1 (g - g_f) is ONE Gauss-Newton step of the problem without frame f from this pose -- an estimate, not
    a re-solve: it is close to the re-solved extrinsic's move when the pose is near the optimum and frame f does not change
    which residuals the Cauchy loss down-weights.  delta_f is a pose increment in the solver's parameterisation (translation,
    then rotation vector; pose_plus).  Frames whose H - H_f is numerically singular (the frame alone pins a direction) get NaN.
    Batched 6x6 solves on the host, O(n_frames).

    Returns (delta [N, 6], translation norm [N] in metres, rotation norm [N] in radians)."""
    iu = np.triu_indices(6)
    N = len(report)
    Hf = np.zeros((N, 6, 6))
    Hf[:, iu[0], iu[1]] = report["H21"]
    Hf = Hf + np.triu(Hf, 1).transpose(0, 2, 1)
    A = np.asarray(H, dtype=np.float64)[None] - Hf
    b = np.asarray(g, dtype=np.float64)[None] - report["g6"]
    delta = np.full((N, 6), np.nan)
    with np.errstate(invalid="ignore"):
        finite = np.all(np.isfinite(A.reshape(N, -1)), axis=1) & np.all(np.isfinite(b), axis=1)
    if np.any(finite):
        sv = np.linalg.svd(A[finite], compute_uv=False)
        regular = sv[:, -1] > sv[:, 0] * 6 * np.finfo(np.float64).eps  # numpy's matrix_rank threshold
        idx = np.nonzero(finite)[0][regular]
        if idx.size:
            delta[idx] = -np.linalg.solve(A[idx], b[idx][..., None])[..., 0]
    return delta, np.linalg.norm(delta[:, :3], axis=1), np.linalg.norm(delta[:, 3:], axis=1)


def _keep_mask(keep, n_frames):
    """A boolean mask of length n_frames -> the uint8 array of the C ABI (checked before any device work)."""
    keep = np.asarray(keep)
    if keep.dtype != np.bool_:
        raise TypeError(f"keep must be a boolean mask, not {keep.dtype}")
    if keep.shape != (n_frames,):
        raise ValueError(f"keep must have shape ({n_frames},), not {keep.shape}")
    return np.ascontiguousarray(keep, dtype=np.uint8)


class Selection(NamedTuple):
    """A frame selection (clc_select_frames): order [n_selected] the picked frames in pick order, gain [n_selected] the
    information each added (nats), keep [n_frames] the forced and the picked frames -- the mask subset() takes."""
    order: np.ndarray
    gain: np.ndarray
    keep: np.ndarray


def _select_args(n_frames, budget, min_gain, candidates, forced, fixed):
    """The checked arguments of a selection -> (clc_select_desc, the uint8 states it points to or None), before any device work:
    budget an integer >= 0, min_gain finite and >= 0, candidates / forced boolean masks of shape (n_frames,) (a frame in both is
    forced), fixed names of FIXED_NAMES."""
    if isinstance(budget, (bool, np.bool_)) or not isinstance(budget, (int, np.integer)):
        raise TypeError(f"budget must be an integer, not {type(budget).__name__}")
    if budget < 0:
        raise ValueError(f"budget must be >= 0, not {budget}")
    min_gain = float(min_gain)
    if not (np.isfinite(min_gain) and min_gain >= 0.0):
        raise ValueError(f"min_gain must be finite and >= 0, not {min_gain!r}")
    mask = fixed_mask(fixed)
    state = None
    if candidates is not None or forced is not None:
        state = np.ones(n_frames, dtype=np.uint8)
        if candidates is not None:
            state[_keep_mask(candidates, n_frames) == 0] = 0
        if forced is not None:
            state[_keep_mask(forced, n_frames) != 0] = 2
    d = SelectDesc()
    d.budget, d.min_gain, d.fixed_mask = int(budget), min_gain, mask
    d.state = state.ctypes.data_as(C.POINTER(C.c_uint8)) if state is not None else None
    return d, state


def _select(fn, args, n_frames, desc, what):
    cap = max(min(int(desc.budget), n_frames), 1)
    order, gain, keep = np.zeros(cap, dtype=np.int64), np.zeros(cap), np.zeros(max(n_frames, 1), dtype=np.uint8)
    n = C.c_int64()
    _lib.check(fn(*args, C.byref(desc), C.byref(n), _ip(order), _dp(gain), keep.ctypes.data_as(C.POINTER(C.c_uint8))), what)
    return Selection(order[:n.value].copy(), gain[:n.value].copy(), keep[:n_frames].astype(bool))


def select_frames_from_report(rows, budget, min_gain=0.0, candidates=None, forced=None, fixed=(), device=-1):
    """Problem.select_frames on report rows the caller holds (clc_select_frames_rows): rows is a FRAME_ROW_DTYPE array (a
    frame_report, or constructed rows; only H21 is read), uploaded once to `device` (-1: the current one)."""
    rows = np.asarray(rows)
    if rows.dtype != FRAME_ROW_DTYPE or rows.ndim != 1:
        raise TypeError(f"rows must be a 1-D array of FRAME_ROW_DTYPE, not {rows.dtype} of shape {rows.shape}")
    rows = np.ascontiguousarray(rows)
    n = rows.shape[0]
    desc, _state = _select_args(n, budget, min_gain, candidates, forced, fixed)
    return _select(_lib.load().clc_select_frames_rows, (int(device), n, rows.ctypes.data_as(C.c_void_p)), n, desc,
                   "clc_select_frames_rows")


# the loss kinds of set_loss (include/clc_b200.h CLC_LOSS_*)
LOSS_KINDS = {"none": 0, "cauchy": 1, "huber": 2, "soft_l1": 3}


def _loss_args(kind, a):
    """(CLC_LOSS_* of a kind name, a) as clc_problem_set_loss accepts them: kind None means "none"; a finite and positive with
    a^2 a normal double (roughly 1.5e-154 < a < 1.3e154).  ValueError for anything else."""
    if kind is None:
        kind = "none"
    if not (isinstance(kind, str) and kind in LOSS_KINDS):
        raise ValueError(f"loss kind must be None or one of {sorted(LOSS_KINDS)}, not {kind!r}")
    a = float(a)
    if not (a > 0.0 and np.isfinite(a) and np.isfinite(a * a) and a * a >= np.finfo(np.float64).tiny):
        raise ValueError(f"the loss parameter a must be finite and positive with a^2 a normal double, not {a!r}")
    return LOSS_KINDS[kind], a


def _thresholds(max_abs_e, n_frames):
    """A scalar (every frame) or an array of shape (n_frames,) -> the float64 thresholds of the C ABI (checked before any
    device work: the library rejects a NaN or negative entry too)."""
    t = np.asarray(max_abs_e, dtype=np.float64)
    if t.ndim == 0:
        t = np.full(n_frames, float(t))
    elif t.shape != (n_frames,):
        raise ValueError(f"max_abs_e must be a scalar or have shape ({n_frames},), not {t.shape}")
    if np.any(~(t >= 0.0)):
        raise ValueError("max_abs_e must not be NaN or negative")
    return np.ascontiguousarray(t)


def _segments(seg_offsets, poses, n_frames):
    """A segmentation seg_offsets [W + 1] of n_frames frames and one pose7 per segment [W, 7] -> the int64 / float64 arrays of the
    C ABI (checked before any device work: the library checks them too)."""
    off = np.asarray(seg_offsets)
    if off.ndim != 1 or off.size < 2 or not np.issubdtype(off.dtype, np.integer):
        raise ValueError("seg_offsets must be a 1-D integer array of at least 2 entries")
    off = np.ascontiguousarray(off, dtype=np.int64)
    if off[0] != 0 or off[-1] != n_frames or np.any(np.diff(off) < 0):
        raise ValueError(f"seg_offsets must start at 0, not decrease and end at n_frames = {n_frames}")
    W = off.size - 1
    x = np.ascontiguousarray(poses, dtype=np.float64)
    if x.shape != (W, 7):
        raise ValueError(f"poses must have shape ({W}, 7), not {x.shape}")
    if not np.all(np.isfinite(x)):
        raise ValueError("poses must be finite")
    return off, x, W


QUANTILES_MAX = 16  # CLC_QUANTILES_MAX


def _quantile_args(pose7, q):
    """pose7 and the quantiles q (a scalar or a 1-D array) -> the float64 arrays of the C ABI and R, checked before any library
    call: pose7 of 7 finite entries, 1 <= R <= QUANTILES_MAX, every q in [0, 1] (the library checks them too)."""
    x = np.ascontiguousarray(pose7, dtype=np.float64)
    if x.shape != (7,) or not np.all(np.isfinite(x)):
        raise ValueError(f"pose7 must be 7 finite numbers, not {x.shape}")
    qa = np.asarray(q)
    if qa.ndim > 1 or not (np.issubdtype(qa.dtype, np.floating) or np.issubdtype(qa.dtype, np.integer)) or qa.dtype == np.bool_:
        raise ValueError(f"q must be a real scalar or a 1-D real array, not {qa.dtype} of shape {qa.shape}")
    qa = np.ascontiguousarray(qa.reshape(-1), dtype=np.float64)
    if not 1 <= qa.size <= QUANTILES_MAX:
        raise ValueError(f"the number of quantiles must lie in [1, {QUANTILES_MAX}], not {qa.size}")
    if not np.all((qa >= 0.0) & (qa <= 1.0)):
        raise ValueError("every q must lie in [0, 1] (NaN is rejected)")
    return x, qa, qa.size


def _residual_quantiles(fn, handle, pose7, q, what):
    x, qa, R = _quantile_args(pose7, q)
    values, n_valid = np.empty(R), C.c_int64()
    _lib.check(fn(handle, _dp(x), R, _dp(qa), _dp(values), C.byref(n_valid)), what)
    return values, n_valid.value


def _frame_quantiles(fn, handle, n_frames, pose7, q, what):
    x, qa, R = _quantile_args(pose7, q)
    values, n_valid = np.empty((max(n_frames, 1), R)), np.empty(max(n_frames, 1), dtype=np.int64)
    _lib.check(fn(handle, _dp(x), R, _dp(qa), _dp(values), _ip(n_valid)), what)
    return values[:n_frames].copy(), n_valid[:n_frames].copy()


def _point_range(first, count, n_points):
    """(first, count) of point_residuals, checked against [0, n_points]; count None: every point from first on."""
    for name, v in (("first", first), ("count", count)):
        if v is not None and (isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer))):
            raise TypeError(f"{name} must be an integer, not {type(v).__name__}")
    first = int(first)
    count = n_points - first if count is None else int(count)
    if first < 0 or count < 0 or first + count > n_points:
        raise ValueError(f"the point range [{first}, {first} + {count}) lies outside [0, {n_points}]")
    return first, count


MAX_POSES = 1024


def _poses(poses):
    """K poses [K, 7] for clc_eval_poses / clc_solve_lm_starts -> the float64 array of the C ABI and K (checked before any device
    work: the library checks them too)."""
    x = np.asarray(poses)
    if x.ndim != 2 or x.shape[1] != 7 or not (np.issubdtype(x.dtype, np.floating) or np.issubdtype(x.dtype, np.integer)):
        raise ValueError(f"poses must be a real array of shape (K, 7), not {x.shape} {x.dtype}")
    K = x.shape[0]
    if not 1 <= K <= MAX_POSES:
        raise ValueError(f"the number of poses must lie in [1, {MAX_POSES}], not {K}")
    x = np.ascontiguousarray(x, dtype=np.float64)
    if not np.all(np.isfinite(x)):
        raise ValueError("poses must be finite")
    return x, K


FIXED_NAMES = ("tx", "ty", "tz", "rx", "ry", "rz")  # bit k of clc_lm_options.fixed_mask: tangent coordinate k of Plus


def fixed_mask(fixed) -> int:
    """Names of held tangent coordinates -> clc_lm_options.fixed_mask.  tx ty tz: translation of T_cl (camera frame); rx ry
    rz: the right-multiplied rotation increment (laser frame).  A held rotation name removes that axis from every increment;
    it does not freeze an Euler angle."""
    if isinstance(fixed, str):
        fixed = (fixed,)
    mask = 0
    for name in fixed:
        if name not in FIXED_NAMES:
            raise ValueError(f"unknown coordinate {name!r}: the names are {' '.join(FIXED_NAMES)}")
        mask |= 1 << FIXED_NAMES.index(name)
    if mask == (1 << 6) - 1:
        raise ValueError("holding all six coordinates leaves nothing to solve")
    return mask


TIME_OFFSET_NAMES = FIXED_NAMES + ("td",)  # bit 6 of fixed_mask holds td in solve_time_offset only


def time_offset_mask(fixed) -> int:
    """Names of the coordinates solve_time_offset holds (TIME_OFFSET_NAMES: the six of fixed_mask, then "td") -> its
    fixed_mask, any proper subset of the seven."""
    if isinstance(fixed, str):
        fixed = (fixed,)
    mask = 0
    for name in fixed:
        if name not in TIME_OFFSET_NAMES:
            raise ValueError(f"unknown coordinate {name!r}: the names are {' '.join(TIME_OFFSET_NAMES)}")
        mask |= 1 << TIME_OFFSET_NAMES.index(name)
    if mask == (1 << 7) - 1:
        raise ValueError("holding all seven coordinates leaves nothing to solve")
    return mask


RANGE_BIAS_NAMES = FIXED_NAMES + ("range_offset", "range_scale")  # bits 6, 7 of fixed_mask hold b, s in solve_range_bias only


def range_bias_mask(fixed) -> int:
    """Names of the coordinates solve_range_bias holds (RANGE_BIAS_NAMES: the six of fixed_mask, then "range_offset" b and
    "range_scale" s) -> its fixed_mask, any proper subset of the eight."""
    if isinstance(fixed, str):
        fixed = (fixed,)
    mask = 0
    for name in fixed:
        if name not in RANGE_BIAS_NAMES:
            raise ValueError(f"unknown coordinate {name!r}: the names are {' '.join(RANGE_BIAS_NAMES)}")
        mask |= 1 << RANGE_BIAS_NAMES.index(name)
    if mask == (1 << 8) - 1:
        raise ValueError("holding all eight coordinates leaves nothing to solve")
    return mask


def _pose_bias(pose7, bias):
    """The float64 pose7 [7] and bias (b, s) [2] of the range-bias calls, checked before any library call."""
    x = np.ascontiguousarray(pose7, dtype=np.float64).reshape(-1)
    if x.shape != (7,):
        raise ValueError("pose7 must have 7 entries")
    b = np.ascontiguousarray(bias, dtype=np.float64).reshape(-1)
    if b.shape != (2,):
        raise ValueError("bias must be (range_offset, range_scale)")
    if not (np.all(np.isfinite(x)) and np.all(np.isfinite(b))):
        raise ValueError("pose7 and bias must be finite")
    return x, b


def _trajectory(knot_times, knot_poses, frame_times, n_frames):
    """The float64 arrays of clc_problem_set_trajectory (checked before any device work: the library checks them too)."""
    t = np.ascontiguousarray(knot_times, dtype=np.float64)
    q = np.ascontiguousarray(knot_poses, dtype=np.float64)
    s = np.ascontiguousarray(frame_times, dtype=np.float64)
    K = t.shape[0] if t.ndim == 1 else -1
    if K < 2 or q.shape != (K, 7):
        raise ValueError(f"knot_times must be [K >= 2] and knot_poses [K, 7], not {t.shape} and {q.shape}")
    if s.shape != (n_frames,):
        raise ValueError(f"frame_times must have shape ({n_frames},), not {s.shape}")
    return t, q, s, K


def default_options(fixed=(), **kw) -> LmOptions:
    """clc_lm_default_options, then the fields in kw.  fixed: names of the tangent coordinates held at the start pose's
    value in every solve with these options (FIXED_NAMES), e.g. default_options(fixed=("ty", "rx"))."""
    o = LmOptions()
    _lib.load().clc_lm_default_options(C.byref(o))
    o.fixed_mask = fixed_mask(fixed)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


class Problem:
    """A device-resident problem (one per GPU / rank).  Thin wrapper over clc_problem*."""

    def __init__(self, handle):
        self._h = handle
        self._L = _lib.load()
        self._comm = None

    # ---- construction ----
    @classmethod
    def from_arrays(cls, frame_pose, offsets, points, edge_points=None, use_loss=True, cauchy_a=0.05, device=-1):
        L = _lib.load()
        frame_pose = np.ascontiguousarray(frame_pose, dtype=np.float64).reshape(-1, 7)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        if edge_points is not None:
            edge_points = np.ascontiguousarray(edge_points, dtype=np.float64).reshape(-1, 6)
            if edge_points.shape[0] != frame_pose.shape[0]:
                raise ValueError("edge_points must be [n_frames, 6]")
        if offsets.shape[0] != frame_pose.shape[0] + 1 or (offsets.size and offsets[-1] != points.shape[0]):
            raise ValueError("offsets do not match frame_pose / points")
        d = ProblemDesc()
        d.n_frames = frame_pose.shape[0]
        d.frame_pose, d.offsets, d.points, d.edge_points = _dp(frame_pose), _ip(offsets), _dp(points), _dp(edge_points)
        d.use_loss, d.cauchy_a, d.device = int(bool(use_loss)), float(cauchy_a), int(device)
        h = C.c_void_p()
        _lib.check(L.clc_problem_create(C.byref(h), C.byref(d)), "clc_problem_create")
        return cls(h)

    @classmethod
    def from_frames(cls, frame_pose, frames, edge_points=None, use_loss=True, cauchy_a=0.05, device=-1):
        """One separate [n_i, 3] array per frame (clc_problem_create_gather): the library gathers them itself."""
        g = _Gather(frame_pose, frames, edge_points, use_loss, cauchy_a, device)
        h = C.c_void_p()
        _lib.check(_lib.load().clc_problem_create_gather(C.byref(h), C.byref(g.desc)), "clc_problem_create_gather")
        return cls(h)

    @classmethod
    def from_observations(cls, obs, use_linefitting_data=True, use_boundary_constraint=False, **kw):
        fp, off, pts, edge = marshal(obs, use_linefitting_data, use_boundary_constraint)
        return cls.from_arrays(fp, off, pts, edge, **kw)

    @classmethod
    def synthetic(cls, n_frames_total, beams, seed=1, sigma=0.0, with_edges=False, frame_begin=0, frame_end=None,
                  use_loss=True, cauchy_a=0.05, device=-1, camera=None, pixel_sigma=0.0, intrinsics=None,
                  image_size=(752, 480), grid=(6, 6, 0.055, 0.3)):
        """camera: None (exact board poses, the reference simulation), "radtan" (pinhole, fx fy cx cy k1 k2 p1 p2) or "equi"
        (Kannala-Brandt, mu mv u0 v0 k2 k3 k4 k5): the poses handed to the solver are then estimated from noisy corner
        pixels by the reference's undistort + PnP chain.  Default intrinsics: the reference's config/*.yaml."""
        L = _lib.load()
        d = _synthetic_desc(n_frames_total, beams, seed, sigma, with_edges, frame_begin, frame_end, use_loss, cauchy_a, device,
                            camera, pixel_sigma, intrinsics, image_size, grid)
        h = C.c_void_p()
        _lib.check(L.clc_problem_create_synthetic(C.byref(h), C.byref(d)), "clc_problem_create_synthetic")
        return cls(h)

    def subset(self, keep):
        """A new problem of the frames with keep[f] True, in their order (clc_problem_subset), built on the device from this
        one's data -- no upload.  It is the problem from_arrays would build from the kept frames, so every output is bit-identical
        to that fresh problem's.  This problem is unchanged; close it when it is no longer needed.  While both are alive the
        device holds the kept share a second time."""
        k = _keep_mask(keep, self.sizes()[0])
        h = C.c_void_p()
        _lib.check(self._L.clc_problem_subset(self._h, k.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(h)), "clc_problem_subset")
        return Problem(h)

    def trim(self, pose7, max_abs_e):
        """A new problem without the points farther than max_abs_e[f] from their board at pose7 (clc_problem_trim), built on the
        device from this one's data -- no upload.  max_abs_e: a scalar for every frame or one threshold per frame, in the units
        of frame_report's max_abs_e (e.g. 3 * frame_report(x)["rms_e"]); points whose distance is NaN are always dropped.  Every
        frame stays, possibly empty.  It is the problem from_arrays would build from the kept points, so every output is
        bit-identical to that fresh problem's.  This problem is unchanged; close it when it is no longer needed."""
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        t = _thresholds(max_abs_e, self.sizes()[0])
        h = C.c_void_p()
        _lib.check(self._L.clc_problem_trim(self._h, _dp(pose7), _dp(t), C.byref(h)), "clc_problem_trim")
        return Problem(h)

    def close(self):
        if self._h is not None:
            self._L.clc_problem_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ---- introspection ----
    def sizes(self):
        nf, npts, he = C.c_int64(), C.c_int64(), C.c_int()
        _lib.check(self._L.clc_problem_sizes(self._h, C.byref(nf), C.byref(npts), C.byref(he)), "clc_problem_sizes")
        return nf.value, npts.value, bool(he.value)

    def algorithmic_bytes(self):
        b = C.c_int64()
        _lib.check(self._L.clc_problem_algorithmic_bytes(self._h, C.byref(b)), "clc_problem_algorithmic_bytes")
        return b.value

    def streamed_bytes(self):
        """Bytes one sweep really streams (16 B per point when the planar two-stream kernels are active)."""
        b = C.c_int64()
        _lib.check(self._L.clc_problem_streamed_bytes(self._h, C.byref(b)), "clc_problem_streamed_bytes")
        return b.value

    @property
    def planar(self):
        """True if the z stream was dropped (every z exactly 0) and the two-stream kernels run."""
        return self.streamed_bytes() != self.algorithmic_bytes()

    def set_planar_mode(self, mode):
        """1 = automatic (default): planar data runs the two-stream kernels; 0 = always the general kernels."""
        _lib.check(self._L.clc_problem_set_planar_mode(self._h, int(mode)), "clc_problem_set_planar_mode")

    def set_loss(self, kind, a=0.05):
        """The robust loss of every later eval, solve, frame_report, eval_segments and solve_segments (clc_problem_set_loss):
        kind None / "none", "cauchy", "huber" or "soft_l1" -- Ceres' CauchyLoss, HuberLoss or SoftLOneLoss with parameter
        a * s for a frame of scale s = 1/sqrt(#points), as the reference scales its CauchyLoss(0.05).  Creation sets
        "cauchy" (use_loss=True) or "none", with a = cauchy_a.  information, closed_form and line_fit never use it; subset and
        trim inherit it.  ValueError for a bad kind, or an a that is not finite and positive or whose square is not a normal
        double; the loss is then unchanged."""
        k, a = _loss_args(kind, a)
        _lib.check(self._L.clc_problem_set_loss(self._h, k, a), "clc_problem_set_loss")

    @property
    def loss(self):
        """(kind, a): the loss set_loss (or creation) chose; kind is "none", "cauchy", "huber" or "soft_l1"."""
        k, a = C.c_int(), C.c_double()
        _lib.check(self._L.clc_problem_get_loss(self._h, C.byref(k), C.byref(a)), "clc_problem_get_loss")
        return {v: n for n, v in LOSS_KINDS.items()}[k.value], a.value

    def partition(self, warp_table=True):
        """The sweep kernel's static work partition for the active kernel family (test hook): dict with grid (blocks),
        per_warp (points per warp range), stage (points per pipeline stage), resident_chunks (stages per warp kept in L2
        during LM solves) and, with warp_table, warp_first_frame [grid * 12] (the frame holding each range's first point)."""
        grid, per_warp, stage, resident = C.c_int(), C.c_int64(), C.c_int(), C.c_int()
        L = self._L
        _lib.check(L.clc_debug_partition(self._h, C.byref(grid), C.byref(per_warp), C.byref(stage), C.byref(resident), None),
                   "clc_debug_partition")
        out = dict(grid=grid.value, per_warp=per_warp.value, stage=stage.value, resident_chunks=resident.value)
        if warp_table:
            wff = np.empty(grid.value * 12, dtype=np.int32)
            _lib.check(L.clc_debug_partition(self._h, None, None, None, None, wff.ctypes.data_as(C.POINTER(C.c_int))),
                       "clc_debug_partition")
            out["warp_first_frame"] = wff
        return out

    def dispatch(self):
        """The kernel each entry point runs on for this problem (test hook): dict with eval, information, closed_form and
        solve, each one of "one_cluster", "single_block", "single_block_loop", "multi_block" or "multi_block_loop", and
        small_shape = (threads per CTA, CTAs per cluster, residuals per thread) of the one-cluster kernel."""
        paths = [C.c_int() for _ in range(4)]
        shape = (C.c_int * 3)()
        _lib.check(self._L.clc_debug_dispatch(self._h, *[C.byref(v) for v in paths], shape), "clc_debug_dispatch")
        out = {k: _lib.PATHS[v.value] for k, v in zip(("eval", "information", "closed_form", "solve"), paths)}
        out["small_shape"] = tuple(shape)
        return out

    def download(self):
        nf, npts, he = self.sizes()
        fp, off, pts = np.empty((nf, 7)), np.empty(nf + 1, dtype=np.int64), np.empty((npts, 3))
        edge = np.empty((nf, 6)) if he else None
        planes = np.empty((nf, 4))
        _lib.check(self._L.clc_problem_download(self._h, _dp(fp), _ip(off), _dp(pts), _dp(edge), _dp(planes)),
                   "clc_problem_download")
        return dict(frame_pose=fp, offsets=off, points=pts, edge_points=edge, planes=planes)

    def download_true_poses(self):
        """Synthetic problems with a camera model: the poses the laser points were generated from."""
        fp = np.empty((self.sizes()[0], 7))
        _lib.check(self._L.clc_problem_download_true_poses(self._h, _dp(fp)), "clc_problem_download_true_poses")
        return fp

    # ---- the hot path ----
    def eval(self, pose7):
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        H, g, cost = np.empty((6, 6)), np.empty(6), C.c_double()
        _lib.check(self._L.clc_eval(self._h, _dp(pose7), _dp(H), _dp(g), C.byref(cost)), "clc_eval")
        return cost.value, H, g

    def solve(self, pose7, options: LmOptions | None = None, trace_cap=256):
        x = np.ascontiguousarray(pose7, dtype=np.float64).copy()
        o = options if options is not None else default_options()
        s = LmSummary()
        tr = (LmIteration * trace_cap)()
        _lib.check(self._L.clc_solve_lm(self._h, _dp(x), C.byref(o), C.byref(s), tr, trace_cap), "clc_solve_lm")
        return x, s, [tr[i] for i in range(min(s.num_iterations, trace_cap))]

    def information(self, pose7):
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        H, b, sv, chi = np.empty((6, 6)), np.empty(6), np.empty(6), C.c_double()
        self.last_V = np.empty((6, 6))  # right singular vectors of H, columns ordered like sv
        _lib.check(self._L.clc_information(self._h, _dp(pose7), _dp(H), _dp(b), C.byref(chi), _dp(sv), _dp(self.last_V)),
                   "clc_information")
        return H, b, chi.value, sv

    def point_residuals(self, pose7, first=0, count=None):
        """The signed raw distance e of points [first, first + count) to their board at pose7, in point order (clc_point_residuals):
        the e that frame_report, trim and the quantiles use.  count None: every point from first on.  A range pages through a
        problem larger than host memory."""
        x, _, _ = _quantile_args(pose7, 0.0)
        first, count = _point_range(first, count, self.sizes()[1])
        e = np.empty(count)
        _lib.check(self._L.clc_point_residuals(self._h, _dp(x), first, count, _dp(e)), "clc_point_residuals")
        return e

    def residual_quantiles(self, pose7, q):
        """Exact quantiles of |e| over every point at pose7 (clc_residual_quantiles): q a scalar or up to QUANTILES_MAX values in
        [0, 1]; returns (values [R], n_valid).  Quantile q is the k-th smallest valid |e| with k = clamp(ceil(q n) - 1, 0, n - 1)
        over the n values that are not NaN (q = 0.5: the lower median); NaN when n = 0."""
        return _residual_quantiles(self._L.clc_residual_quantiles, self._h, pose7, q, "clc_residual_quantiles")

    def frame_quantiles(self, pose7, q):
        """residual_quantiles within every frame (clc_frame_quantiles): (values [n_frames, R], n_valid [n_frames]).  A robust
        per-frame trim threshold: 3 * 1.4826 * frame_quantiles(x, 0.5)[0][:, 0]."""
        return _frame_quantiles(self._L.clc_frame_quantiles, self._h, self.sizes()[0], pose7, q, "clc_frame_quantiles")

    def frame_report(self, pose7):
        """Every frame's residual statistics and share of the normal equations at pose7 (clc_frame_report): a numpy record
        array of FRAME_ROW_DTYPE, one row per frame.  Rows sum to eval()'s cost, H (upper triangle) and g, and their chi to
        information()'s chi."""
        return _frame_report(self._L.clc_frame_report, self._h, self.sizes()[0], pose7, "clc_frame_report")

    def select_frames(self, pose7, budget, min_gain=0.0, candidates=None, forced=None, fixed=()):
        """Greedy D-optimal selection of at most `budget` frames by the information they add about the extrinsic at pose7
        (clc_select_frames; the rule is in include/clc_b200.h).  candidates: boolean mask of the frames that may be picked (None:
        all); forced: boolean mask of frames kept from the start and never picked (they count as already selected); fixed: names
        of coordinates left out of the information, as default_options takes them.  Stops early once the best gain is <= min_gain
        nats or no candidate is left.  Returns a Selection (order, gain, keep); keep is the mask subset() takes:
        ``with p.subset(p.select_frames(x, 200).keep) as q: q.solve(x)``."""
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        n = self.sizes()[0]
        desc, _state = _select_args(n, budget, min_gain, candidates, forced, fixed)
        return _select(self._L.clc_select_frames, (self._h, _dp(pose7)), n, desc, "clc_select_frames")

    # ---- independent solves over runs of frames (segments) ----
    def eval_segments(self, seg_offsets, poses):
        """eval() of every segment [seg_offsets[s], seg_offsets[s + 1]) of the frames at its own pose poses[s], from ONE shared
        sweep (clc_eval_segments).  Returns (cost [W], H [W, 6, 6], g [W, 6]); segment s's are those of a fresh problem of its
        frames alone, up to the order of summation."""
        off, x, W = _segments(seg_offsets, poses, self.sizes()[0])
        cost, H, g = np.empty(W), np.empty((W, 6, 6)), np.empty((W, 6))
        _lib.check(self._L.clc_eval_segments(self._h, W, _ip(off), _dp(x), _dp(H), _dp(g), _dp(cost)), "clc_eval_segments")
        return cost, H, g

    def information_segments(self, seg_offsets, poses):
        """information() of every segment at its own pose (clc_information_segments): (H [W, 6, 6], b [W, 6], chi [W], sv [W, 6]);
        the right singular vectors go to self.last_V [W, 6, 6]."""
        off, x, W = _segments(seg_offsets, poses, self.sizes()[0])
        H, b, chi, sv = np.empty((W, 6, 6)), np.empty((W, 6)), np.empty(W), np.empty((W, 6))
        self.last_V = np.empty((W, 6, 6))
        _lib.check(self._L.clc_information_segments(self._h, W, _ip(off), _dp(x), _dp(H), _dp(b), _dp(chi), _dp(sv),
                                                    _dp(self.last_V)), "clc_information_segments")
        return H, b, chi, sv

    def solve_segments(self, seg_offsets, poses, options: LmOptions | None = None, trace_cap=0):
        """solve() of every segment from its own start pose poses[s], W solves advancing side by side on shared sweeps
        (clc_solve_lm_segments).  Returns (poses [W, 7], summaries [W] of LmSummary, traces: one list of LmIteration per segment,
        empty without trace_cap).  summaries[s].device_ms is the time of the whole segmented solve."""
        off, x, W = _segments(seg_offsets, poses, self.sizes()[0])
        x = x.copy()
        o = options if options is not None else default_options()
        summaries = (LmSummary * W)()
        tr = (LmIteration * (W * trace_cap))() if trace_cap > 0 else None
        _lib.check(self._L.clc_solve_lm_segments(self._h, W, _ip(off), _dp(x), C.byref(o), summaries, tr, int(trace_cap)),
                   "clc_solve_lm_segments")
        traces = [[tr[s * trace_cap + i] for i in range(min(summaries[s].num_iterations, trace_cap))] if trace_cap > 0 else []
                  for s in range(W)]
        return x, list(summaries), traces

    # ---- one calibration at many poses (multi-start) ----
    def eval_poses(self, poses):
        """eval() at every pose poses[k] of [K, 7], from ONE shared pass over the points (clc_eval_poses).  Returns
        (cost [K], H [K, 6, 6], g [K, 6]); pose k's bytes depend on poses[k] only."""
        x, K = _poses(poses)
        cost, H, g = np.empty(K), np.empty((K, 6, 6)), np.empty((K, 6))
        _lib.check(self._L.clc_eval_poses(self._h, K, _dp(x), _dp(H), _dp(g), _dp(cost)), "clc_eval_poses")
        return cost, H, g

    def solve_starts(self, poses, options: LmOptions | None = None, trace_cap=0):
        """solve() from every start pose poses[k] of [K, 7], the K solves advancing side by side on shared sweeps
        (clc_solve_lm_starts).  Returns (poses [K, 7], summaries [K] of LmSummary, traces: one list of LmIteration per start,
        empty without trace_cap, best): best is the start of the lowest final cost that did not fail (lowest index on a tie), -1
        when every start failed.  summaries[k].device_ms is the time of the whole call."""
        x, K = _poses(poses)
        x = x.copy()
        o = options if options is not None else default_options()
        summaries = (LmSummary * K)()
        tr = (LmIteration * (K * trace_cap))() if trace_cap > 0 else None
        best = C.c_int64()
        _lib.check(self._L.clc_solve_lm_starts(self._h, K, _dp(x), C.byref(o), summaries, tr, int(trace_cap), C.byref(best)),
                   "clc_solve_lm_starts")
        traces = [[tr[k * trace_cap + i] for i in range(min(summaries[k].num_iterations, trace_cap))] if trace_cap > 0 else []
                  for k in range(K)]
        return x, list(summaries), traces, best.value

    # ---- the camera-laser time offset ----
    def set_trajectory(self, knot_times, knot_poses, frame_times):
        """Attach the board trajectory of the time-offset calls (clc_problem_set_trajectory): knot_times [K >= 2] in seconds,
        strictly increasing; knot_poses [K, 7] in the frame_pose convention (qx qy qz qw tx ty tz of T_ca); frame_times
        [n_frames], every frame's scan time on the laser clock.  None for the three arguments removes it.  subset and trim
        results carry no trajectory."""
        if knot_times is None and knot_poses is None and frame_times is None:
            _lib.check(self._L.clc_problem_set_trajectory(self._h, 0, None, None, None), "clc_problem_set_trajectory")
            return
        t, q, s, K = _trajectory(knot_times, knot_poses, frame_times, self.sizes()[0])
        _lib.check(self._L.clc_problem_set_trajectory(self._h, K, _dp(t), _dp(q), _dp(s)), "clc_problem_set_trajectory")

    def eval_time_offset(self, pose7, td):
        """eval() with the time offset td: the planes interpolated at every frame's scan time + td (clc_eval_time_offset).
        Returns (cost, H [7, 7], g [7]) over (tx ty tz rx ry rz td)."""
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        H, g, cost = np.empty((7, 7)), np.empty(7), C.c_double()
        _lib.check(self._L.clc_eval_time_offset(self._h, _dp(pose7), float(td), _dp(H), _dp(g), C.byref(cost)),
                   "clc_eval_time_offset")
        return cost.value, H, g

    def information_time_offset(self, pose7, td):
        """information() with the time offset td (clc_information_time_offset): (H [7, 7], b [7], chi, sv [7]); the right
        singular vectors go to self.last_V [7, 7].  A ~0 singular value whose V column is +-e_td: the board never moved."""
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        H, b, sv, chi = np.empty((7, 7)), np.empty(7), np.empty(7), C.c_double()
        self.last_V = np.empty((7, 7))
        _lib.check(self._L.clc_information_time_offset(self._h, _dp(pose7), float(td), _dp(H), _dp(b), C.byref(chi), _dp(sv),
                                                       _dp(self.last_V)), "clc_information_time_offset")
        return H, b, chi.value, sv

    def solve_time_offset(self, pose7, td=0.0, options: LmOptions | None = None, fixed=None, trace_cap=256):
        """solve() of the extrinsic and the time offset td together (clc_solve_lm_time_offset).  fixed: names of
        TIME_OFFSET_NAMES held at their start values for this call (overrides options.fixed_mask); e.g. fixed=("tx", "ty", "tz",
        "rx", "ry", "rz") estimates the offset alone, fixed="td" the extrinsic alone.  Returns (pose7, td, summary, trace)."""
        x = np.ascontiguousarray(pose7, dtype=np.float64).copy()
        t = C.c_double(float(td))
        o = LmOptions.from_buffer_copy(options) if options is not None else default_options()  # the caller's stays as it is
        if fixed is not None:
            o.fixed_mask = time_offset_mask(fixed)
        s = LmSummary()
        tr = (LmIteration * trace_cap)() if trace_cap > 0 else None
        _lib.check(self._L.clc_solve_lm_time_offset(self._h, _dp(x), C.byref(t), C.byref(o), C.byref(s), tr, int(trace_cap)),
                   "clc_solve_lm_time_offset")
        return x, t.value, s, [tr[i] for i in range(min(s.num_iterations, trace_cap))] if trace_cap > 0 else []

    # ---- the laser's range offset and scale ----
    def eval_range_bias(self, pose7, bias):
        """eval() with every point p moved to kappa p along its ray, kappa = 1 + s + b / |p| (bias = (b, s): the range offset in
        the points' unit and the range scale; clc_eval_range_bias).  Returns (cost, H [8, 8], g [8]) over (tx ty tz rx ry rz b
        s)."""
        x, b = _pose_bias(pose7, bias)
        H, g, cost = np.empty((8, 8)), np.empty(8), C.c_double()
        _lib.check(self._L.clc_eval_range_bias(self._h, _dp(x), _dp(b), _dp(H), _dp(g), C.byref(cost)), "clc_eval_range_bias")
        return cost.value, H, g

    def information_range_bias(self, pose7, bias):
        """information() with the range bias (clc_information_range_bias): (H [8, 8], b [8], chi, sv [8]); the right singular
        vectors go to self.last_V [8, 8].  A small singular value whose V column lies in the span of the translation, e_b and
        e_s: the boards were seen in too narrow a band of ranges to tell the scale from the offset."""
        x, bb = _pose_bias(pose7, bias)
        H, b, sv, chi = np.empty((8, 8)), np.empty(8), np.empty(8), C.c_double()
        self.last_V = np.empty((8, 8))
        _lib.check(self._L.clc_information_range_bias(self._h, _dp(x), _dp(bb), _dp(H), _dp(b), C.byref(chi), _dp(sv),
                                                      _dp(self.last_V)), "clc_information_range_bias")
        return H, b, chi.value, sv

    def solve_range_bias(self, pose7, bias=(0.0, 0.0), options: LmOptions | None = None, fixed=None, trace_cap=256):
        """solve() of the extrinsic with the laser's range offset b and scale s (clc_solve_lm_range_bias).  fixed: names of
        RANGE_BIAS_NAMES held at their start values for this call (overrides options.fixed_mask); e.g. fixed="range_scale"
        estimates the offset alone.  Returns (pose7, bias (b, s), summary, trace)."""
        x, b = _pose_bias(pose7, bias)
        x, b = x.copy(), b.copy()
        if not 0 <= int(trace_cap) <= 256:
            raise ValueError("trace_cap must be in [0, 256]")
        o = LmOptions.from_buffer_copy(options) if options is not None else default_options()  # the caller's stays as it is
        if fixed is not None:
            o.fixed_mask = range_bias_mask(fixed)
        s = LmSummary()
        tr = (LmIteration * trace_cap)() if trace_cap > 0 else None
        _lib.check(self._L.clc_solve_lm_range_bias(self._h, _dp(x), _dp(b), C.byref(o), C.byref(s), tr, int(trace_cap)),
                   "clc_solve_lm_range_bias")
        return x, b, s, [tr[i] for i in range(min(s.num_iterations, trace_cap))] if trace_cap > 0 else []

    def range_corrected(self, bias):
        """A new problem whose points are this one's moved to kappa p, kappa = 1 + s + b / |p| (clc_problem_range_correct), built
        on the device from this one's points -- no upload.  Every other call (trim, quantiles, frame_report, select_frames,
        segments, starts) then runs on the corrected points.  This problem is unchanged; close the new one when it is no longer
        needed."""
        b = np.ascontiguousarray(bias, dtype=np.float64).reshape(-1)
        if b.shape != (2,) or not np.all(np.isfinite(b)):
            raise ValueError("bias must be finite (range_offset, range_scale)")
        if not 1.0 + b[1] > 0.0:
            raise ValueError("1 + range_scale must be positive")
        h = C.c_void_p()
        _lib.check(self._L.clc_problem_range_correct(self._h, _dp(b), C.byref(h)), "clc_problem_range_correct")
        return Problem(h)

    def closed_form(self):
        T, AtA, Atb, un = np.empty(16), np.empty((9, 9)), np.empty(9), C.c_int()
        _lib.check(self._L.clc_closed_form(self._h, _dp(T), C.byref(un), _dp(AtA), _dp(Atb)), "clc_closed_form")
        return T.reshape(4, 4), bool(un.value), AtA, Atb

    def line_fit(self, lines0=None, max_num_iterations=10):
        """Batched LineFittingCeres over the frames' points: returns (lines[N,2], info[N,4])."""
        nf = self.sizes()[0]
        lines = np.zeros((nf, 2)) if lines0 is None else np.ascontiguousarray(lines0, dtype=np.float64).reshape(nf, 2).copy()
        info = np.empty((nf, 4))
        _lib.check(self._L.clc_problem_line_fit(self._h, _dp(lines), int(max_num_iterations), _dp(info)), "clc_problem_line_fit")
        return lines, info

    # ---- multi-GPU ----
    def set_allreduce_mode(self, mode: int):
        """0 = NCCL all-reduce between kernels, 1 = fused in-kernel peer exchange (default once p2p is enabled)."""
        _lib.check(self._L.clc_problem_set_allreduce_mode(self._h, int(mode)), "clc_problem_set_allreduce_mode")

    def attach_comm(self, comm: "Comm | None"):
        """Borrow a communicator: every sweep's 28 sums are then all-reduced over its ranks."""
        self._comm = comm  # keep it alive
        _lib.check(self._L.clc_problem_attach_comm(self._h, comm._h if comm is not None else None), "clc_problem_attach_comm")

    # ---- measurement ----
    def bench_eval(self, pose7, n, flush_l2=True):
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        ms = (C.c_float * n)()
        _lib.check(self._L.clc_bench_eval(self._h, _dp(pose7), int(n), int(bool(flush_l2)), ms), "clc_bench_eval")
        return np.array(ms[:], dtype=np.float64)

    def bench_frame_report(self, pose7, n, flush_l2=True):
        """Device time of n frame reports (per-frame sweep + split-frame fix-up, without the copy of the rows), ms each."""
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        ms = (C.c_float * n)()
        _lib.check(self._L.clc_bench_frame_report(self._h, _dp(pose7), int(n), int(bool(flush_l2)), ms), "clc_bench_frame_report")
        return np.array(ms[:], dtype=np.float64)

    def bench_select(self, pose7, budget, n, min_gain=0.0, fixed=()):
        """Device time of n selections on one report's device rows (clc_bench_select), ms each, and the picks of the last run."""
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        desc, _state = _select_args(self.sizes()[0], budget, min_gain, None, None, fixed)
        ms, k = (C.c_float * n)(), C.c_int64()
        _lib.check(self._L.clc_bench_select(self._h, _dp(pose7), C.byref(desc), int(n), ms, C.byref(k)), "clc_bench_select")
        return np.array(ms[:], dtype=np.float64), k.value

    def bench_segments(self, seg_offsets, poses, n, flush_l2=True):
        """Device time of n iterations of the segmented calls (frame constants, segment sweep, fix-up, two-level reduction;
        clc_bench_segments), ms each."""
        off, x, W = _segments(seg_offsets, poses, self.sizes()[0])
        ms = (C.c_float * n)()
        _lib.check(self._L.clc_bench_segments(self._h, W, _ip(off), _dp(x), int(n), int(bool(flush_l2)), ms), "clc_bench_segments")
        return np.array(ms[:], dtype=np.float64)

    def bench_poses(self, poses, n, flush_l2=True):
        """Device time of n evaluations of eval_poses (without the copy to the host; clc_bench_poses), ms each."""
        x, K = _poses(poses)
        ms = (C.c_float * n)()
        _lib.check(self._L.clc_bench_poses(self._h, K, _dp(x), int(n), int(bool(flush_l2)), ms), "clc_bench_poses")
        return np.array(ms[:], dtype=np.float64)

    def bench_time_offset(self, pose7, td, n, flush_l2=True):
        """Device time of n time-offset iterations (planes and constants, segment sweep, fix-up, two-level reduction;
        clc_bench_time_offset), ms each."""
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        ms = (C.c_float * n)()
        _lib.check(self._L.clc_bench_time_offset(self._h, _dp(pose7), float(td), int(n), int(bool(flush_l2)), ms),
                   "clc_bench_time_offset")
        return np.array(ms[:], dtype=np.float64)

    def bench_range_bias(self, pose7, bias, n, flush_l2=True):
        """Device time of n range-bias iterations (frame constants, range sweep, fix-up, two-level reduction;
        clc_bench_range_bias), ms each."""
        x, b = _pose_bias(pose7, bias)
        ms = (C.c_float * n)()
        _lib.check(self._L.clc_bench_range_bias(self._h, _dp(x), _dp(b), int(n), int(bool(flush_l2)), ms), "clc_bench_range_bias")
        return np.array(ms[:], dtype=np.float64)

    def bench_subset(self, keep, n, flush_l2=True):
        """Device time of the gather of n subsets(keep) into scratch problems (clc_bench_subset), ms each."""
        k = _keep_mask(keep, self.sizes()[0])
        ms = (C.c_float * n)()
        _lib.check(self._L.clc_bench_subset(self._h, k.ctypes.data_as(C.POINTER(C.c_uint8)), int(n), int(bool(flush_l2)), ms),
                   "clc_bench_subset")
        return np.array(ms[:], dtype=np.float64)

    def bench_trim(self, pose7, max_abs_e, n, flush_l2=True):
        """Device times of the mark and the gather pass of n trims(pose7, max_abs_e) into scratch problems (clc_bench_trim),
        ms each: returns (mark [n], gather [n])."""
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        t = _thresholds(max_abs_e, self.sizes()[0])
        mark, gather = (C.c_float * n)(), (C.c_float * n)()
        _lib.check(self._L.clc_bench_trim(self._h, _dp(pose7), _dp(t), int(n), int(bool(flush_l2)), mark, gather), "clc_bench_trim")
        return np.array(mark[:], dtype=np.float64), np.array(gather[:], dtype=np.float64)

    def bench_quantiles(self, pose7, q, n, flush_l2=True):
        """Device times of n residual_quantiles(pose7, q) calls, from the first pass to the end of the last, and of n per-frame
        kernels of frame_quantiles(pose7, q) (clc_bench_quantiles), ms each: returns (problem-wide [n], per-frame [n], passes over
        the point streams)."""
        x, qa, R = _quantile_args(pose7, q)
        ms, fms, passes = (C.c_float * n)(), (C.c_float * n)(), C.c_int()
        _lib.check(self._L.clc_bench_quantiles(self._h, _dp(x), R, _dp(qa), int(n), int(bool(flush_l2)), ms, fms, C.byref(passes)),
                   "clc_bench_quantiles")
        return np.array(ms[:], dtype=np.float64), np.array(fms[:], dtype=np.float64), passes.value


class Group:
    """G devices of THIS process solving one problem (clc_group_*): frames sharded by point count, the 28 sums exchanged
    over NVLink inside the sweep kernel, one host thread.  A group of one device is a plain problem."""

    def __init__(self, handle):
        self._h = handle
        self._L = _lib.load()

    @staticmethod
    def _devices(devices):
        devs = [int(d) for d in devices]
        return (C.c_int * len(devs))(*devs), len(devs)

    @classmethod
    def from_frames(cls, frame_pose, frames, edge_points=None, devices=(-1,), use_loss=True, cauchy_a=0.05):
        g = _Gather(frame_pose, frames, edge_points, use_loss, cauchy_a)
        arr, n = cls._devices(devices)
        h = C.c_void_p()
        _lib.check(_lib.load().clc_group_create_gather(C.byref(h), C.byref(g.desc), arr, n), "clc_group_create_gather")
        return cls(h)

    @classmethod
    def from_arrays(cls, frame_pose, offsets, points, edge_points=None, devices=(-1,), **kw):
        points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        offsets = np.asarray(offsets, dtype=np.int64)
        frames = [points[offsets[f]:offsets[f + 1]] for f in range(len(offsets) - 1)]
        return cls.from_frames(frame_pose, frames, edge_points, devices, **kw)

    @classmethod
    def synthetic(cls, n_frames, beams, seed=1, sigma=0.0, with_edges=False, devices=(-1,), use_loss=True, cauchy_a=0.05,
                  n_frames_total=None, frame_begin=0, camera=None, pixel_sigma=0.0, intrinsics=None, image_size=(752, 480),
                  grid=(6, 6, 0.055, 0.3)):
        total = int(n_frames_total if n_frames_total is not None else frame_begin + n_frames)
        d = _synthetic_desc(total, beams, seed, sigma, with_edges, frame_begin, frame_begin + n_frames, use_loss, cauchy_a, -1,
                            camera, pixel_sigma, intrinsics, image_size, grid)
        arr, n = cls._devices(devices)
        h = C.c_void_p()
        _lib.check(_lib.load().clc_group_create_synthetic(C.byref(h), C.byref(d), arr, n), "clc_group_create_synthetic")
        return cls(h)

    def subset(self, keep):
        """Problem.subset for the group (clc_group_subset): a new group on the same devices holding the frames with keep[f]
        True, re-sharded as from_frames would shard them; kept points on another device are copied over the peer links.  This
        group is unchanged; close it when it is no longer needed."""
        k = _keep_mask(keep, self.sizes()[1])
        h = C.c_void_p()
        _lib.check(self._L.clc_group_subset(self._h, k.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(h)), "clc_group_subset")
        return Group(h)

    def set_loss(self, kind, a=0.05):
        """Problem.set_loss on every shard (clc_group_set_loss): the loss of every later group eval, solve and frame_report."""
        k, a = _loss_args(kind, a)
        _lib.check(self._L.clc_group_set_loss(self._h, k, a), "clc_group_set_loss")

    def trim(self, pose7, max_abs_e):
        """Problem.trim for the group (clc_group_trim), max_abs_e per frame in the global frame order: a new group on the same
        devices, its frames re-sharded by their new point counts as from_frames would shard them; kept points on another device
        are copied over the peer links.  This group is unchanged; close it when it is no longer needed."""
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        t = _thresholds(max_abs_e, self.sizes()[1])
        h = C.c_void_p()
        _lib.check(self._L.clc_group_trim(self._h, _dp(pose7), _dp(t), C.byref(h)), "clc_group_trim")
        return Group(h)

    def close(self):
        if self._h is not None:
            self._L.clc_group_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def sizes(self):
        n, nf, npts = C.c_int(), C.c_int64(), C.c_int64()
        _lib.check(self._L.clc_group_size(self._h, C.byref(n), C.byref(nf), C.byref(npts)), "clc_group_size")
        return n.value, nf.value, npts.value

    def problem(self, index):
        """Borrowed view of shard `index` (do not close it)."""
        h = C.c_void_p()
        _lib.check(self._L.clc_group_problem(self._h, int(index), C.byref(h)), "clc_group_problem")
        p = Problem(h)
        p.close = lambda: None  # owned by the group
        return p

    def eval(self, pose7):
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        H, g, cost = np.empty((6, 6)), np.empty(6), C.c_double()
        _lib.check(self._L.clc_group_eval(self._h, _dp(pose7), _dp(H), _dp(g), C.byref(cost)), "clc_group_eval")
        return cost.value, H, g

    def solve(self, pose7, options: LmOptions | None = None, trace_cap=256):
        x = np.ascontiguousarray(pose7, dtype=np.float64).copy()
        o = options if options is not None else default_options()
        s = LmSummary()
        tr = (LmIteration * trace_cap)()
        _lib.check(self._L.clc_group_solve_lm(self._h, _dp(x), C.byref(o), C.byref(s), tr, trace_cap), "clc_group_solve_lm")
        return x, s, [tr[i] for i in range(min(s.num_iterations, trace_cap))]

    def information(self, pose7):
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        H, b, sv, chi = np.empty((6, 6)), np.empty(6), np.empty(6), C.c_double()
        self.last_V = np.empty((6, 6))
        _lib.check(self._L.clc_group_information(self._h, _dp(pose7), _dp(H), _dp(b), C.byref(chi), _dp(sv), _dp(self.last_V)),
                   "clc_group_information")
        return H, b, chi.value, sv

    def frame_report(self, pose7):
        """Problem.frame_report over every shard, rows in the global frame order (clc_group_frame_report)."""
        return _frame_report(self._L.clc_group_frame_report, self._h, self.sizes()[1], pose7, "clc_group_frame_report")

    def residual_quantiles(self, pose7, q):
        """Problem.residual_quantiles over every point of the group (clc_group_residual_quantiles).  A shard's own residuals are
        problem(i).point_residuals."""
        return _residual_quantiles(self._L.clc_group_residual_quantiles, self._h, pose7, q, "clc_group_residual_quantiles")

    def frame_quantiles(self, pose7, q):
        """Problem.frame_quantiles over every shard, rows in the global frame order (clc_group_frame_quantiles)."""
        return _frame_quantiles(self._L.clc_group_frame_quantiles, self._h, self.sizes()[1], pose7, q, "clc_group_frame_quantiles")

    def select_frames(self, pose7, budget, min_gain=0.0, candidates=None, forced=None, fixed=()):
        """Problem.select_frames over every shard (clc_group_select_frames): the frame_report rows in the global frame order,
        selected on the group's first device; order and keep are in the global frame order."""
        pose7 = np.ascontiguousarray(pose7, dtype=np.float64)
        n = self.sizes()[1]
        desc, _state = _select_args(n, budget, min_gain, candidates, forced, fixed)
        return _select(self._L.clc_group_select_frames, (self._h, _dp(pose7)), n, desc, "clc_group_select_frames")

    def closed_form(self):
        T, AtA, Atb, un = np.empty(16), np.empty((9, 9)), np.empty(9), C.c_int()
        _lib.check(self._L.clc_group_closed_form(self._h, _dp(T), C.byref(un), _dp(AtA), _dp(Atb)), "clc_group_closed_form")
        return T.reshape(4, 4), bool(un.value), AtA, Atb


def upload_stats():
    """Statistics of this process's most recent host -> HBM upload (clc_upload_last_stats)."""
    t, w, b = C.c_double(), C.c_double(), C.c_int64()
    ch, th, di = C.c_int(), C.c_int(), C.c_int()
    _lib.load().clc_upload_last_stats(C.byref(t), C.byref(w), C.byref(b), C.byref(ch), C.byref(th), C.byref(di))
    return dict(total_ms=t.value, pack_wait_ms=w.value, bytes_h2d=b.value, chunks=ch.value, pack_threads=th.value, direct=bool(di.value))


def debug_pack(frames, a, b, xy):
    """What the pack threads write for the local point range [a, b) (test hook; no CUDA)."""
    g = _Gather(np.zeros((len(frames), 7)), frames)
    out = np.empty((b - a) * (2 if xy else 3))
    nonplanar = C.c_int(-1)
    _lib.check(_lib.load().clc_debug_pack(len(frames), g.ptrs, _ip(g.counts), int(a), int(b), int(bool(xy)), _dp(out),
                                          C.byref(nonplanar)), "clc_debug_pack")
    return out.reshape(-1, 2 if xy else 3), nonplanar.value


class Comm:
    """NCCL communicator of the solve (one per rank / GPU), shareable between problems on the same device."""

    def __init__(self, unique_id: bytes, nranks: int, rank: int, device: int = -1):
        self._L = _lib.load()
        self._h = C.c_void_p()
        buf = C.create_string_buffer(unique_id, 128)
        _lib.check(self._L.clc_comm_create(C.byref(self._h), buf, int(nranks), int(rank), int(device)), "clc_comm_create")
        self.nranks, self.rank = int(nranks), int(rank)

    def p2p_export(self) -> bytes:
        """64-byte CUDA IPC handle of this rank's mailbox (for the fused in-kernel all-reduce over NVLink)."""
        buf = C.create_string_buffer(64)
        _lib.check(self._L.clc_comm_p2p_export(self._h, buf), "clc_comm_p2p_export")
        return buf.raw

    def p2p_import(self, handles):
        """handles: the exported handles of all ranks, in rank order."""
        blob = b"".join(handles)
        if len(blob) != 64 * self.nranks:
            raise ValueError("need one 64-byte handle per rank")
        _lib.check(self._L.clc_comm_p2p_import(self._h, C.create_string_buffer(blob, len(blob))), "clc_comm_p2p_import")

    def enable_p2p(self, all_gather):
        """all_gather(bytes) -> list[bytes] over the ranks (e.g. torch.distributed.all_gather_object)."""
        self.p2p_import(all_gather(self.p2p_export()))

    def close(self):
        if self._h is not None:
            self._L.clc_comm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def comm_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    _lib.check(_lib.load().clc_comm_unique_id(buf), "clc_comm_unique_id")
    return buf.raw


def shard_range(n_frames, nranks, rank, offsets=None):
    b, e = C.c_int64(), C.c_int64()
    off = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.int64)
    _lib.check(_lib.load().clc_shard_range(int(n_frames), _ip(off), int(nranks), int(rank), C.byref(b), C.byref(e)),
               "clc_shard_range")
    return b.value, e.value


def T_to_pose7(T):
    T = np.ascontiguousarray(T, dtype=np.float64).reshape(16)
    p = np.empty(7)
    _lib.load().clc_T_to_pose7(_dp(T), _dp(p))
    return p


def pose7_to_T(p):
    p = np.ascontiguousarray(p, dtype=np.float64)
    T = np.empty(16)
    _lib.load().clc_pose7_to_T(_dp(p), _dp(T))
    return T.reshape(4, 4)


def launch_count() -> int:
    return int(_lib.load().clc_launch_count())


class pinned_array:
    """numpy view of CUDA pinned host memory (upload buffers for the end-to-end measurement)."""

    def __init__(self, shape, dtype=np.float64):
        self._L = _lib.load()
        self.nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        self._ptr = C.c_void_p()
        _lib.check(self._L.clc_host_alloc(C.byref(self._ptr), self.nbytes), "clc_host_alloc")
        buf = (C.c_char * max(self.nbytes, 1)).from_address(self._ptr.value)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def free(self):
        if self._ptr is not None and self._ptr.value:
            self.array = None
            self._L.clc_host_free(self._ptr)
            self._ptr = None


def LineFittingCeres(Points, Line: np.ndarray, max_num_iterations=10):
    """reference src/LaseCamCalCeres.cpp:401-433: ``Line`` (2,) is the start value on entry and the fit on exit."""
    pts = np.ascontiguousarray(Points, dtype=np.float64).reshape(-1, 3)
    line = np.ascontiguousarray(Line, dtype=np.float64).copy()
    _lib.check(_lib.load().clc_line_fit_points(_dp(pts), pts.shape[0], _dp(line), int(max_num_iterations)), "clc_line_fit_points")
    Line[...] = line


# ---- the reference's two entry points -------------------------------------------------------------------------

def CamLaserCalClosedSolution(obs, Tlc: np.ndarray, verbose=True):
    """reference src/LaseCamCalCeres.cpp:112-203.  Writes T_lc (4x4) into ``Tlc``; uses obs[i].points_on_line."""
    with Problem.from_observations(obs, use_linefitting_data=True, use_boundary_constraint=False) as p:
        T, unobservable, _, _ = p.closed_form()
    if unobservable and verbose:
        print("\n~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~")
        print(" Notice Notice Notice: system unobservable !!!!!!!")
        print("~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~\n")
    Tlc[...] = T
    if verbose:
        print("------- Closed-form solution Tlc: -------\n", Tlc)
    return unobservable


def CamLaserCalibration(obs, Tcl: np.ndarray, use_linefitting_data=True, use_boundary_constraint=False, verbose=True,
                        options: LmOptions | None = None):
    """reference src/LaseCamCalCeres.cpp:213-383.  ``Tcl`` (4x4) is the initial guess on entry and the result on
    exit (bottom row untouched, :313-314).  Returns a dict with the solver summary and the analysis-tail outputs the
    reference prints (H singular values, null-space basis, chi2/2)."""
    pose = T_to_pose7(Tcl)  # :215-219
    with Problem.from_observations(obs, use_linefitting_data, use_boundary_constraint) as p:
        x, s, trace = p.solve(pose, options)
        T = pose7_to_T(x)
        Tcl[:3, :] = T[:3, :]  # :311-314
        H, b, chi, sv = p.information(x)  # :318-362
        V = p.last_V
    report = dict(termination=TERMINATION.get(s.termination, "?"), iterations=s.num_iterations,
                  initial_cost=s.initial_cost, final_cost=s.final_cost, trace=trace, H=H, b=b, chi2=chi / 2.0,
                  singular_values=sv, V=V, pose7=x, device_ms=s.device_ms, num_sweeps=s.num_sweeps)
    if verbose:
        print(f"LM (on device): {report['termination']}, {s.num_iterations} iterations, cost {s.initial_cost:.6e} -> "
              f"{s.final_cost:.6e}, {s.device_ms:.3f} ms")
        print("----- H singular values--------:\n", sv)
        n_null = int(np.sum(sv < 1e-8))  # :368-379
        if n_null > 0:
            print("====== null space basis, it's means the unobservable direction for Tcl ======")
            print("       please note the unobservable direction is for Tcl, not for Tlc        ")
            print(V[:, 6 - n_null:])  # svd.matrixV().rightCols(n), :378
        print("\nrecover chi2: ", chi / 2.0)
    return report
