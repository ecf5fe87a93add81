"""References of the solve with held tangent coordinates (clc_lm_options.fixed_mask).  TEST INFRASTRUCTURE ONLY.

* FixedOracle: ctypes view of tests/fixed_oracle.c (Ceres' LM on the reduced local parameterization, DENSE_QR or Cholesky
  on the free columns), compiled against oracle/libclc_oracle.so; no loss or Cauchy, as the main oracle evaluates;
* solve_fixed: an independent numpy restatement through oracle_np.trust_region_lm, for any residual model (the losses'
  evaluation of tests/loss_reference.py included).
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as O
from oracle import oracle_np as ONP


class FixedOracle:
    def __init__(self, out_dir):
        lib_path = O.build()
        here = os.path.dirname(os.path.abspath(__file__))
        odir = os.path.dirname(lib_path)
        out = os.path.join(str(out_dir), "libfixed_oracle.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([cc, "-O2", "-std=c11", "-Wall", "-Wextra", "-shared", "-fPIC", "-I", odir, "-o", out,
                               os.path.join(here, "fixed_oracle.c"), lib_path, "-Wl,-rpath," + odir, "-lm"])
        L = C.CDLL(out)
        L.fixed_oracle_solve.argtypes = [C.POINTER(O._Problem), C.POINTER(C.c_double), C.POINTER(O.Options), C.c_int,
                                         C.POINTER(O.Summary), C.POINTER(O.Iteration), C.c_int]
        self.L = L

    def solve(self, p, pose7, fixed_mask, linear_solver=0, trace_cap=256):
        """(pose7, oracle Summary, [Iteration...]) of Ceres' LM with the coordinates of fixed_mask held; linear_solver 0 is
        the Householder QR of [J_s; D], 1 the Cholesky of the normal equations, both on the free columns."""
        x = np.array(pose7, dtype=np.float64)
        s, tr = O.Summary(), (O.Iteration * trace_cap)()
        o = O.default_options(linear_solver=linear_solver)
        self.L.fixed_oracle_solve(C.byref(p._c), O._dp(x), C.byref(o), int(fixed_mask), C.byref(s), tr, trace_cap)
        return x, s, list(tr[: min(s.num_iterations, trace_cap)])


def solve_fixed(evaluate_fn, x0, fixed_mask, max_num_iterations=100):
    """Ceres' LM with the tangent coordinates of `fixed_mask` (bit k: coordinate k of Plus) held at their start value: the
    reference's PoseLocalParameterization wrapped in a parameterization of local size 6 - k (Ceres 2.1).  The minimiser
    (oracle_np.trust_region_lm) sees a problem of the free coordinates only: the Jacobian's free columns, Plus of the free
    increment embedded with zeros, and the gradient norm of the free gradient embedded with zeros.  evaluate_fn(x) -> (cost,
    corrected residuals, corrected local Jacobian [R, 6]).  Returns (pose7, termination name, trace dicts)."""
    free = [k for k in range(6) if not (fixed_mask >> k) & 1]

    def embed(v):
        full = np.zeros(6)
        full[free] = v
        return full

    def ev(x):
        cost, r, J = evaluate_fn(x)
        return cost, r, J[:, free]

    return ONP.trust_region_lm(ev, lambda x, d: ONP.pose_plus(x, embed(d)), x0, max_num_iterations,
                               lambda x, g: ONP.gradient_max_norm(x, embed(g)))
