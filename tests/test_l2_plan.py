"""CPU tests of the L2 residency plan of LM solves (csrc/clc_l2_plan.h, compiled with g++ from the source the library uses):
how many stages of every warp's range stay in L2 from one sweep to the next."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L2_H100 = 50 * 1024 * 1024  # cudaDevAttrL2CacheSize of an H100 SXM
SMS, WARPS = 132, 12        # one 12-warp block per SM


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    d = tmp_path_factory.mktemp("l2plan")
    src = d / "plan.cpp"
    src.write_text('#include "clc_l2_plan.h"\n'
                   'extern "C" long long budget(long long l2, long long o) { return clc::l2_resident_budget(l2, o); }\n'
                   'extern "C" int chunks(long long b, long long g, long long w, long long s, long long sb, int lb) {\n'
                   '  return clc::l2_resident_chunks(b, g, w, s, sb, lb != 0); }\n')
    out = str(d / "libplan.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "camlasercalibratool_b200", "csrc"),
                    str(src), "-o", out], check=True)
    L = C.CDLL(out)
    L.budget.restype = C.c_longlong
    L.budget.argtypes = [C.c_longlong, C.c_longlong]
    L.chunks.argtypes = [C.c_longlong] * 5 + [C.c_int]
    return L


def per_warp_stages(n_points, chunk):
    # partition() in csrc/clc_api.cu: whole stages, the same count for every warp of the full grid
    points_per_warp = -(-n_points // (SMS * WARPS))  # ceil
    return -(-points_per_warp // chunk)


def test_default_budget_and_override(plan):
    assert plan.budget(L2_H100, -1) == int(L2_H100 * 0.5)
    assert plan.budget(L2_H100, 0) == 0  # CLC_L2_RESIDENT_MB=0: off
    assert plan.budget(L2_H100, 20 << 20) == 20 << 20


def test_configs1_on_an_h100(plan):
    b = plan.budget(L2_H100, -1)
    n = 10_000 * 1_000
    s_gen, s_pla = per_warp_stages(n, 128), per_warp_stages(n, 256)
    assert (s_gen, s_pla) == (50, 25)
    k_gen = plan.chunks(b, SMS, WARPS, s_gen, 3 * 1024, 0)  # general: 3 x 1 KiB per stage
    k_pla = plan.chunks(b, SMS, WARPS, s_pla, 4 * 1024, 0)  # planar: 2 x 2 KiB per stage
    assert (k_gen, k_pla) == (5, 4)  # 24 MB of 240 MB, 25 MB of 160 MB
    assert k_gen * SMS * WARPS * 3 * 1024 <= b < (k_gen + 1) * SMS * WARPS * 3 * 1024
    assert k_pla * SMS * WARPS * 4 * 1024 <= b < (k_pla + 1) * SMS * WARPS * 4 * 1024


def test_a_problem_that_fits_is_entirely_resident(plan):
    b = plan.budget(L2_H100, -1)
    s = per_warp_stages(1_000_000, 128)  # 24 MB general
    assert plan.chunks(b, SMS, WARPS, s, 3 * 1024, 0) == s
    assert plan.chunks(1 << 40, SMS, WARPS, 50, 3 * 1024, 0) == 50


def test_latency_bound_and_disabled_launches_keep_nothing(plan):
    b = plan.budget(L2_H100, -1)
    assert plan.chunks(b, 1, WARPS, 8, 3 * 1024, 0) == 0     # a single block
    assert plan.chunks(b, 2, WARPS, 1, 3 * 1024, 1) == 0     # a problem of the one-cluster kernel's size
    assert plan.chunks(0, SMS, WARPS, 50, 3 * 1024, 0) == 0  # budget 0: off (or the persisting-L2 window is configured)
