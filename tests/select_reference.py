"""The frame-selection rule of clc_select_frames (include/clc_b200.h), restated in numpy for the tests.

The blocks, their scaling and the greedy bookkeeping are float64; every gain is evaluated in the dtype the caller asks for:
np.longdouble (x87 extended, 64-bit mantissa) for the checks of the device's picks, np.float64 for the reference sequence.  The
gains are formed as the rule states them: L L^T = A, C = L^-1 H L^-T, and log det(I + C) from the pivots 1 + u_k of the
Cholesky factorisation of I + C, summed as log1p(u_k).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LD = np.longdouble
RIDGE = 1e-6  # CLC_SELECT_RIDGE
NAMES = ("tx", "ty", "tz", "rx", "ry", "rz")
IU = np.triu_indices(6)


class NoInformation(Exception):
    """A free coordinate's total information T_kk is not positive and finite (the library's CLC_ERR_STATE)."""

    def __init__(self, coord):
        super().__init__(f"no usable frame observes {coord}")
        self.coord = coord


def unpack(H21):
    """[n, 21] upper triangles (K1's order) -> [n, 6, 6] symmetric."""
    H21 = np.asarray(H21, dtype=np.float64).reshape(-1, 21)
    H = np.zeros((H21.shape[0], 6, 6))
    H[:, IU[0], IU[1]] = H21
    return H + np.triu(H, 1).transpose(0, 2, 1)


def pack(H):
    """[n, 6, 6] -> [n, 21]."""
    return np.asarray(H)[:, IU[0], IU[1]]


def free_coords(mask):
    return [k for k in range(6) if not (mask >> k) & 1]


def prepare(H21, state=None, mask=0):
    """Steps 1-4 of the rule: dict(usable [n], cand [n] (usable candidates), forced [n] (usable forced), Ht [n, d, d], A0 [d, d],
    D [d], n_T).  NoInformation for a free coordinate without positive finite T_kk."""
    H21 = np.asarray(H21, dtype=np.float64).reshape(-1, 21)
    n = H21.shape[0]
    state = np.ones(n, dtype=np.uint8) if state is None else np.asarray(state, dtype=np.uint8)
    usable = np.all(np.isfinite(H21), axis=1)
    fr = free_coords(mask)
    H = unpack(np.where(usable[:, None], H21, 0.0))[:, fr][:, :, fr]
    in_t = usable & (state != 0)
    T = H[in_t].sum(axis=0)
    for i, k in enumerate(fr):
        if not (T[i, i] > 0.0 and np.isfinite(T[i, i])):
            raise NoInformation(NAMES[k])
    D = 1.0 / np.sqrt(np.diag(T))
    Ht = D[None, :, None] * H * D[None, None, :]
    forced = usable & (state == 2)
    n_t = int(in_t.sum())
    A0 = Ht[forced].sum(axis=0) + (RIDGE / n_t) * np.eye(len(fr))
    return dict(usable=usable, cand=usable & (state == 1), forced=forced, Ht=Ht, A0=A0, D=D, n_T=n_t, state=state)


def chol(A, dtype):
    """Lower Cholesky factor of one symmetric matrix, in dtype (None when a pivot is not positive)."""
    A = np.asarray(A).astype(dtype)
    d = A.shape[0]
    L = np.zeros((d, d), dtype=dtype)
    for j in range(d):
        s = A[j, j] - np.sum(L[j, :j] ** 2)
        if not s > 0:
            return None
        L[j, j] = np.sqrt(s)
        for i in range(j + 1, d):
            L[i, j] = (A[i, j] - np.sum(L[i, :j] * L[j, :j])) / L[j, j]
    return L


def gains(A, Ht, dtype=LD):
    """gain_f = log det(I + L^-1 Ht_f L^-T) of every block of Ht [m, d, d] at A = L L^T, evaluated in dtype; -inf where a pivot of
    I + C is not positive and finite."""
    return gains_at(chol(A, dtype), Ht, dtype)


def gains_at(L, Ht, dtype=LD):
    """gains() at a given lower Cholesky factor L of A."""
    Ht = np.asarray(Ht)
    m, d = Ht.shape[0], Ht.shape[1]
    L = np.asarray(L).astype(dtype)
    Linv = np.zeros((d, d), dtype=dtype)
    for c in range(d):  # L^-1 by forward substitution on the unit vectors
        for i in range(d):
            s = (1 if i == c else 0) - np.sum(L[i, :i] * Linv[:i, c])
            Linv[i, c] = s / L[i, i]
    Cm = np.matmul(np.matmul(Linv[None], np.asarray(Ht, dtype=dtype)), Linv.T[None])
    R = np.zeros((m, d, d), dtype=dtype)
    g = np.zeros(m, dtype=dtype)
    bad = np.zeros(m, dtype=bool)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for j in range(d):
            u = Cm[:, j, j] - np.sum(R[:, j, :j] ** 2, axis=1)
            piv = 1 + u
            bad |= ~(piv > 0) | ~np.isfinite(piv)
            g += np.log1p(np.where(bad, 0, u))
            r = np.sqrt(np.where(bad, 1, piv))
            for i in range(j + 1, d):
                R[:, i, j] = (Cm[:, j, i] - np.sum(R[:, i, :j] * R[:, j, :j], axis=1)) / r
    g[bad] = -np.inf
    return g


def greedy(H21, budget, min_gain=0.0, state=None, mask=0, dtype=np.float64):
    """Step 5 of the rule with gains in dtype.  Returns (order [k], gain [k] (float64), keep [n] bool, sep [k]): sep[s] is the gap
    between the best and the second-best gain of step s (inf with one candidate)."""
    P = prepare(H21, state, mask)
    A = P["A0"].copy()
    remaining = P["cand"].copy()
    order, gain, sep = [], [], []
    for _ in range(int(budget)):
        idx = np.nonzero(remaining)[0]
        if idx.size == 0:
            break
        g = gains(A, P["Ht"][idx], dtype)
        k = int(np.argmax(g))  # first maximum: the lowest index on a tie
        if not g[k] > min_gain:
            break
        rest = np.delete(g, k)
        sep.append(float(g[k] - rest.max()) if rest.size else np.inf)
        f = int(idx[k])
        order.append(f)
        gain.append(float(g[k]))
        remaining[f] = False
        A = A + P["Ht"][f]
    keep = (P["state"] == 2).copy()
    keep[order] = True
    return np.array(order, dtype=np.int64), np.array(gain), keep, np.array(sep)


def check_picks(H21, order, gain, budget, min_gain=0.0, state=None, mask=0, steps=None, rtol=1e-10):
    """The device's picks against the rule in long double, step by step along the device's own sequence: each pick's gain is within
    rtol (1 + g) of the maximum over the remaining candidates, and the reported gain within the same bound of its long-double
    value.  When the device stopped before the budget, the best remaining long-double gain is <= min_gain + rtol (1 + |g|) or no
    candidate was left.  steps: check only the first `steps` picks."""
    P = prepare(H21, state, mask)
    A = P["A0"].astype(LD)
    HtL = P["Ht"].astype(LD)
    remaining = P["cand"].copy()
    n_check = len(order) if steps is None else min(steps, len(order))
    for s in range(n_check):
        idx = np.nonzero(remaining)[0]
        g = gains(A, HtL[idx], LD)
        gmax = g.max()
        f = int(order[s])
        assert remaining[f], (s, f)
        gf = g[np.searchsorted(idx, f)]
        bound = rtol * (1 + abs(float(gmax)))
        assert float(gmax - gf) <= bound, (s, f, float(gf), float(gmax))
        assert abs(float(gain[s]) - float(gf)) <= bound, (s, f, float(gain[s]), float(gf))
        remaining[f] = False
        A = A + HtL[f]
    if steps is None and len(order) < budget:
        idx = np.nonzero(remaining)[0]
        if idx.size:
            g = gains(A, P["Ht"][idx], LD)
            assert float(g.max()) <= min_gain + rtol * (1 + abs(float(g.max()))), float(g.max())


def agreeing_prefix(order, ref_order, ref_sep, rtol=1e-10, ref_gain=None):
    """The device's sequence equals the reference's up to its first step whose top two gains are within rtol (1 + g) (after that
    the two may legitimately differ).  Returns the number of steps compared."""
    n = min(len(order), len(ref_order))
    for s in range(n):
        g = abs(ref_gain[s]) if ref_gain is not None else 0.0
        if ref_sep[s] <= rtol * (1 + g):
            return s
        assert order[s] == ref_order[s], (s, order[s], ref_order[s])
    return n


# ---- the g++ build of the product's CLC_HD selection arithmetic ---------------------------------------------------------------
class SelectHarness:
    def __init__(self, tmpdir):
        out = os.path.join(str(tmpdir), "libselect_harness.so")
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", out,
                               os.path.join(ROOT, "tests", "select_harness.cpp")])
        L = C.CDLL(out)
        dp = C.POINTER(C.c_double)
        L.sel_chol.argtypes = [dp, dp, dp]
        L.sel_gains.argtypes = [dp, C.c_int64, dp, dp]
        L.sel_gains_at.argtypes = [dp, dp, C.c_int64, dp, dp]
        self.L = L

    @staticmethod
    def _p(a):
        return a.ctypes.data_as(C.POINTER(C.c_double))

    def chol(self, A):
        A = np.ascontiguousarray(A, dtype=np.float64)
        L, inv = np.zeros(36), np.zeros(6)
        ok = self.L.sel_chol(self._p(A), self._p(L), self._p(inv))
        return bool(ok), L.reshape(6, 6), inv

    def gains(self, A, H):
        A = np.ascontiguousarray(A, dtype=np.float64)
        H = np.ascontiguousarray(H, dtype=np.float64).reshape(-1, 36)
        g = np.zeros(H.shape[0])
        assert self.L.sel_gains(self._p(A), H.shape[0], self._p(H), self._p(g)) == 1
        return g

    def gains_at(self, L, H):
        """sel_gain6 at a given factor L (6x6 lower) of every block of H [m, 6, 6]."""
        L = np.ascontiguousarray(L, dtype=np.float64)
        inv = np.ascontiguousarray(1.0 / np.diag(L))
        H = np.ascontiguousarray(H, dtype=np.float64).reshape(-1, 36)
        g = np.zeros(H.shape[0])
        self.L.sel_gains_at(self._p(L), self._p(inv), H.shape[0], self._p(H), self._p(g))
        return g
