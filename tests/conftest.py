"""pytest configuration: the `gpu` marker, and the session fixtures that build the test-only artefacts.

* `-m "not gpu"` : oracle vs numpy twin vs golden fixtures, host logic of the product (compiled with g++ from the
                   same CLC_HD sources the GPU runs), ABI surface of libclc_b200.so, world_size-2 gloo sharding.
* `-m gpu`       : parity of the CUDA path (through the C ABI) against the oracle on an H100.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on the GPU box")


def _has_gpu() -> bool:
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O

    O.build()
    return O


@pytest.fixture(scope="session")
def oracle_np():
    from oracle import oracle_np as N

    return N


class Harness:
    """ctypes view of tests/host_harness.cpp (the product's CLC_HD code compiled for the host)."""

    def __init__(self, path):
        from camlasercalibratool_b200._lib import LmIteration, LmOptions

        L = C.CDLL(path)
        dp = C.POINTER(C.c_double)
        L.harness_lm_state_size.restype = C.c_int
        L.harness_lm_init.argtypes = [C.c_void_p, dp, C.POINTER(LmOptions)]
        L.harness_lm_update.argtypes = [C.c_void_p, dp]
        L.harness_lm_done.argtypes = [C.c_void_p]
        L.harness_lm_ntrace.argtypes = [C.c_void_p]
        L.harness_lm_sweeps.argtypes = [C.c_void_p]
        L.harness_lm_cand.argtypes = [C.c_void_p, dp]
        L.harness_lm_x.argtypes = [C.c_void_p, dp]
        L.harness_lm_trace.argtypes = [C.c_void_p, C.c_int, C.POINTER(LmIteration)]
        L.harness_expand_lm.argtypes = [dp, dp, C.c_double, dp, C.c_int, C.c_double, C.c_double, dp]
        L.harness_frame_consts.argtypes = [dp, dp, dp, dp]
        L.harness_accumulate_residual.argtypes = [dp, dp, dp, C.c_double, C.c_int, C.c_double, dp]
        L.harness_expand_closed.argtypes = [dp, dp, dp]
        L.harness_frame_plane.argtypes = [dp, dp]
        L.harness_edge_planes.argtypes = [dp, dp, dp]
        L.harness_pose_plus.argtypes = [dp, dp, dp]
        L.harness_philox.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32)]
        L.harness_gen_frame_pose.argtypes = [C.c_uint64, C.c_int64, C.c_int, dp]
        L.harness_gen_edge_points.argtypes = [dp, dp]
        L.harness_gen_points.argtypes = [C.c_uint64, C.c_double, C.c_int64, C.c_int64, dp, dp]
        self.L = L
        self.LmIteration = LmIteration
        self.LmOptions = LmOptions

    @staticmethod
    def dp(a):
        return a.ctypes.data_as(C.POINTER(C.c_double))

    def default_options(self, **kw):
        # mirrors clc_lm_default_options (which lives in the CUDA library and cannot be called without it here)
        o = self.LmOptions(100, 1e4, 1e16, 1e-32, 1e-3, 1e-6, 1e32, 1e-6, 1e-10, 1e-8, 5, 1, 8, 0)
        for k, v in kw.items():
            setattr(o, k, v)
        return o

    def lm_run(self, sums_fn, pose7, options=None, max_sweeps=300):
        """Drives lm_update exactly as the device loop does: sums_fn(pose7) -> 28 sums of one sweep."""
        st = C.create_string_buffer(self.L.harness_lm_state_size())
        o = options if options is not None else self.default_options()
        x0 = np.ascontiguousarray(pose7, dtype=np.float64)
        self.L.harness_lm_init(st, self.dp(x0), C.byref(o))
        cand = np.empty(7)
        n = 0
        while not self.L.harness_lm_done(st) and n < max_sweeps:
            self.L.harness_lm_cand(st, self.dp(cand))
            sums = np.ascontiguousarray(sums_fn(cand.copy()), dtype=np.float64)
            self.L.harness_lm_update(st, self.dp(sums))
            n += 1
        x = np.empty(7)
        self.L.harness_lm_x(st, self.dp(x))
        trace = []
        for i in range(min(self.L.harness_lm_ntrace(st), 256)):
            it = self.LmIteration()
            self.L.harness_lm_trace(st, i, C.byref(it))
            trace.append(it)
        return x, self.L.harness_lm_done(st), trace, self.L.harness_lm_sweeps(st)


@pytest.fixture(scope="session")
def harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("harness") / "libclc_host_harness.so")
    src = os.path.join(ROOT, "tests", "host_harness.cpp")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", out, src])
    return Harness(out)


def pack_sums(cost, H, g):
    """(cost, H[6,6], g[6]) -> the 28-vector the kernel produces (21 upper-tri, 6, 1)."""
    iu = np.triu_indices(6)
    return np.concatenate([np.asarray(H)[iu], np.asarray(g), [cost]])


@pytest.fixture(scope="session")
def identity_pose():
    return np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
