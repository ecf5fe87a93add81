"""Extended-precision reference for the three kinds of sums the sweep kernels produce, with an error bound for each output.

The sweep kernel sums millions of float64 terms through several levels (per-lane running sums, warp butterflies, the
per-warp tile, the block and the ordered block gather) and reorganises them through moments (DESIGN.md section 3).  A
fixed relative tolerance on |H| hides mistakes in small components such as g near the optimum.  This module computes every
per-residual term in long double (64-bit mantissa) and returns, next to each summed output k, a magnitude A_k: the sum of
the absolute values of what the kernel's algorithm adds and cancels to form that output.  A correct kernel satisfies

    |got_k - ref_k| <= GAMMA * A_k

for every output.  GAMMA = 1e-13 (about 450 u, u = 2^-53) covers the depth of the kernel's float64 summation.  Inside a frame a
lane keeps adding until the frame or its warp range ends: 2 of every 64 points, so up to per_warp / 32 additions -- about 3 950
at 2*10^8 points, whose warp ranges hold ~126 000 points, when the frames are longer than a warp range.  Then come 5 butterfly
levels, one tile flush per 32 pieces, 12 warps per block and ~10 blocks in each of 13 gather parts followed by the 13 parts,
and a handful of roundings in the per-frame expansion: a depth n of about 4 100 on the longest path.  The worst-case bound of
recursive summation, (n - 1) u sum |x_i|, would allow ~9 GAMMA there; the bound that holds is the probabilistic one of Higham
and Mary (SIAM J. Sci. Comput. 41 (2019) A2815, Theorem 3.1): with roundings independent and of mean zero, the error is at
most (exp(lambda sqrt(n) u + n u^2 / (1 - u)) - 1) sum |x_i| ~ lambda sqrt(n) u sum |x_i| with probability at least
1 - 2 n exp(-lambda^2 (1 - u)^2 / 2).  With n = 4 100 and lambda = 13 that is 9.2e-14 * A_k < GAMMA, failing with probability
below 1e-32 per output.  tests/test_gpu_at_scale.py runs that depth (100 frames of 2*10^6 points) and measures it.

Magnitudes (s^2 = 1 / #points of the frame, w the Cauchy weight, n the plane normal, m = R^T n, p the point):
  * rounding of the raw distance e = m.p + c, c = n.t + d, is bounded by a few u times L_e = |m||p| + |n||t| + |d|;
  * H_tt: s^2 w |n_a n_b|,  H_t theta: s^2 w |n_a| |p||m|,  H_theta theta: s^2 w |p|^2 |m|^2, each plus the first-order
    effect of the rounding of e on the weight, s^2 |w'| L_e times the same |J_a||J_b| (w' = dw/de, 0 without the loss);
  * g_t: s^2 w |n_a| L_e,  g_theta: s^2 w |p||m| L_e (the moment expansion cancels S2 m against c S1);
  * cost: 1/2 s^2 (a^2 log u + a^2 2^-52) with the loss (the kernel takes the log of a running product, one rounding per
    factor), 1/2 s^2 e^2 without; plus s^2 w |e| L_e, the effect of the rounding of e itself;
  * closed form: A^T A: sum |pbar_a pbar_b n_r n_q|, A^T b: sum |d| |pbar_a| |n_r|, pbar = (x, y, 1).

Residuals of empty frames and the edge residuals of empty frames do not exist (the reference would divide by zero), exactly
as in both sweep kernels.  Test infrastructure only.
"""
from __future__ import annotations

import numpy as np

LD = np.longdouble
if np.finfo(LD).nmant < 63:
    raise RuntimeError(f"long double has {np.finfo(LD).nmant} mantissa bits here; the exact-sum reference needs >= 63 "
                       "(x86-64 80-bit extended precision)")

GAMMA = 1e-13
U_PROD = 2.0 ** -52  # relative rounding of one factor of the kernel's running cost product
CHUNK = 1 << 18      # residuals per vectorised block

IU6 = np.triu_indices(6)
IU9 = np.triu_indices(9)
# the 28 LM outputs: 21 upper-triangle H (row-major), 6 g, cost
GROUPS_LM = {
    "H_tt": [k for k, (i, j) in enumerate(zip(*IU6)) if i < 3 and j < 3],
    "H_ttheta": [k for k, (i, j) in enumerate(zip(*IU6)) if i < 3 <= j],
    "H_thetatheta": [k for k, (i, j) in enumerate(zip(*IU6)) if i >= 3],
    "g_t": [21, 22, 23],
    "g_theta": [24, 25, 26],
    "cost": [27],
}
GROUPS_CF = {"AtA": list(range(45)), "Atb": list(range(45, 54))}


def _rot(q):
    """Eigen QuaternionBase::toRotationMatrix of q = (x, y, z, w) [..., 4], not normalised, in long double."""
    x, y, z, w = (q[..., i] for i in range(4))
    R = np.empty(q.shape[:-1] + (3, 3), dtype=LD)
    R[..., 0, 0] = 1 - 2 * (y * y + z * z)
    R[..., 0, 1] = 2 * (x * y - z * w)
    R[..., 0, 2] = 2 * (x * z + y * w)
    R[..., 1, 0] = 2 * (x * y + z * w)
    R[..., 1, 1] = 1 - 2 * (x * x + z * z)
    R[..., 1, 2] = 2 * (y * z - x * w)
    R[..., 2, 0] = 2 * (x * z - y * w)
    R[..., 2, 1] = 2 * (y * z + x * w)
    R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                     a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def _norm(a):
    return np.sqrt(np.sum(a * a, axis=-1))


def frame_planes(frame_pose):
    """Board planes (T^-1)^T (0,0,1,0) of every frame, [N,4] long double (reference LaseCamCalCeres.cpp:227-231)."""
    fp = np.asarray(frame_pose, dtype=np.float64).reshape(-1, 7).astype(LD)
    A = _rot(fp[:, :4])
    c = _cross(A[:, :, 0], A[:, :, 1])  # row 2 of A^-1 times det A
    det = np.sum(c * A[:, :, 2], axis=-1)
    n = c / det[:, None]
    return np.concatenate([n, -np.sum(n * fp[:, 4:], axis=-1)[:, None]], axis=1)


def edge_planes(frame_pose):
    """The two board-edge planes of every frame, [N,2,4] long double (reference :262-276, un-normalised, through 0)."""
    fp = np.asarray(frame_pose, dtype=np.float64).reshape(-1, 7).astype(LD)
    R, t = _rot(fp[:, :4]), fp[:, 4:]
    o = 0.0265 + 0.0165  # float64, as the reference writes it
    corners = np.array([[-o, -o, 0.0], [0.5 - o, -o, 0.0], [-o, 0.5 - o, 0.0]]).astype(LD)
    pc = [np.einsum("nij,j->ni", R, corners[k]) + t for k in range(3)]
    out = np.zeros((fp.shape[0], 2, 4), dtype=LD)
    out[:, 0, :3] = _cross(pc[0], pc[1])
    out[:, 1, :3] = _cross(pc[0], pc[2])
    return out


def _residual_blocks(frame_pose, offsets, points, edge_points):
    """Yields (plane[k,4], point[k,3], s2[k]) blocks of at most CHUNK residuals: every point of every non-empty frame,
    then (edge_points given) the two edge residuals of every non-empty frame."""
    offsets = np.asarray(offsets, dtype=np.int64)
    counts = np.diff(offsets)
    planes = frame_planes(frame_pose)
    s2_frame = np.zeros(len(counts), dtype=LD)
    s2_frame[counts > 0] = LD(1) / counts[counts > 0].astype(LD)
    frame_of = np.repeat(np.arange(len(counts)), counts)
    P = int(offsets[-1]) if len(offsets) else 0
    for a in range(0, P, CHUNK):
        b = min(P, a + CHUNK)
        f = frame_of[a:b]
        yield planes[f], np.asarray(points[a:b], dtype=np.float64).astype(LD), s2_frame[f]
    if edge_points is not None:
        live = np.nonzero(counts > 0)[0]
        ep = np.asarray(edge_points, dtype=np.float64).reshape(-1, 6)[live].astype(LD)
        epl = edge_planes(np.asarray(frame_pose).reshape(-1, 7)[live])
        for a in range(0, len(live), CHUNK):
            b = min(len(live), a + CHUNK)
            pl = np.concatenate([epl[a:b, 0], epl[a:b, 1]])
            pt = np.concatenate([ep[a:b, :3], ep[a:b, 3:]])
            s2 = np.concatenate([s2_frame[live[a:b]]] * 2)
            yield pl, pt, s2


def lm_sums(frame_pose, offsets, points, pose7, use_loss=True, cauchy_a=0.05, edge_points=None):
    """The 28 sums of one LM sweep (21 upper-triangle H, 6 g, cost) in long double, and their magnitudes A_k (float64)."""
    return lm_sums_of_blocks(_residual_blocks(frame_pose, offsets, points, edge_points), pose7, use_loss, cauchy_a)


def lm_sums_of_residuals(plane, point, s2, pose7, use_loss=True, cauchy_a=0.05):
    """lm_sums over an explicit residual list: plane [k,4], point [k,3], s2 [k] (the residual's 1 / #points)."""
    blocks = ((plane[a:a + CHUNK].astype(LD), np.asarray(point[a:a + CHUNK]).astype(LD), s2[a:a + CHUNK].astype(LD))
              for a in range(0, len(s2), CHUNK))
    return lm_sums_of_blocks(blocks, pose7, use_loss, cauchy_a)


def lm_sums_of_blocks(blocks, pose7, use_loss=True, cauchy_a=0.05):
    pose = np.asarray(pose7, dtype=np.float64).astype(LD)
    R, t = _rot(pose[3:7]), pose[:3]
    a2 = LD(cauchy_a) * LD(cauchy_a)
    val = np.zeros(28, dtype=LD)
    mag = np.zeros(28)
    for plane, p, s2 in blocks:
        n, d = plane[:, :3], plane[:, 3]
        m = n @ R                                   # R^T n
        c = n @ t + d
        e = np.sum(m * p, axis=-1) + c
        L_e = _norm(m) * _norm(p) + _norm(n) * _norm(t) + np.abs(d)
        J = np.concatenate([n, _cross(p, m)], axis=1)
        Jabs = np.concatenate([np.abs(n), np.repeat((_norm(p) * _norm(m))[:, None], 3, axis=1)], axis=1)
        if use_loss:
            q = e * e / a2
            w = LD(1) / (LD(1) + q)
            dw = 2 * np.abs(e) * w * w / a2
            lg = np.log1p(q)
            cost = LD(0.5) * s2 * a2 * lg
            cost_mag = 0.5 * s2 * a2 * (lg + LD(U_PROD)) + s2 * w * np.abs(e) * L_e
        else:
            w = np.ones_like(e)
            dw = np.zeros_like(e)
            cost = LD(0.5) * s2 * e * e
            cost_mag = cost + s2 * np.abs(e) * L_e
        sw = s2 * w
        H = (J * sw[:, None]).T @ J
        val[:21] += H[IU6]
        val[21:27] += (J * (sw * e)[:, None]).sum(axis=0)
        val[27] += cost.sum()
        Jf = Jabs.astype(np.float64)
        Hm = (Jf * (s2 * (w + dw * L_e)).astype(np.float64)[:, None]).T @ Jf
        mag[:21] += Hm[IU6]
        mag[21:27] += (Jf * (sw * L_e).astype(np.float64)[:, None]).sum(axis=0)
        mag[27] += float(cost_mag.sum())
    return val, mag


def closed_form_sums(frame_pose, offsets, points):
    """The 54 closed-form sums (45 upper-triangle A^T A, 9 A^T b; rows n (x) (x, y, 1), b = -d, unweighted, z ignored)."""
    val = np.zeros(54, dtype=LD)
    mag = np.zeros(54)
    for plane, p, _ in _residual_blocks(frame_pose, offsets, points, None):
        n, d = plane[:, :3], plane[:, 3]
        bar = np.stack([p[:, 0], p[:, 1], np.ones_like(p[:, 0])], axis=1)
        A = (bar[:, :, None] * n[:, None, :]).reshape(-1, 9)  # column a*3 + r = pbar_a n_r
        val[:45] += (A.T @ A)[IU9]
        val[45:] += (A * (-d)[:, None]).sum(axis=0)
        Af = np.abs(A).astype(np.float64)
        mag[:45] += (Af.T @ Af)[IU9]
        mag[45:] += (Af * np.abs(d).astype(np.float64)[:, None]).sum(axis=0)
    return val, mag


def pack_lm(cost, H, g):
    """(cost, H[6,6], g[6]) -> the 28-vector in the kernel's order."""
    return np.concatenate([np.asarray(H, dtype=np.float64)[IU6], np.asarray(g, dtype=np.float64), [float(cost)]])


def pack_closed_form(AtA, Atb):
    return np.concatenate([np.asarray(AtA, dtype=np.float64)[IU9], np.asarray(Atb, dtype=np.float64)])


def error_ratios(got, ref, mag):
    """|got_k - ref_k| / A_k for every output (the difference taken in long double); inf where A_k = 0 and got_k != ref_k."""
    err = np.abs(np.asarray(got, dtype=np.float64).astype(LD) - np.asarray(ref, dtype=LD)).astype(np.float64)
    mag = np.asarray(mag, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(mag > 0, err / np.where(mag > 0, mag, 1.0), np.where(err > 0, np.inf, 0.0))
    return r


def worst_by_group(ratios, groups):
    return {name: float(np.max(ratios[idx])) for name, idx in groups.items()}


def assert_within(got, ref, mag, groups, what=""):
    """Every output within GAMMA * A_k; the message names the offending outputs and their error ratio."""
    r = error_ratios(got, ref, mag)
    bad = np.nonzero(r > GAMMA)[0]
    assert bad.size == 0, (f"{what}: outputs {bad.tolist()} exceed GAMMA * A_k; |err|/A_k = {r[bad].tolist()}; "
                           f"worst per group {worst_by_group(r, groups)}")
    return r
