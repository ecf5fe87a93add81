"""ABI surface of libclc_b200.so, checked without a GPU: the library builds for sm_90a, loads, exports every
symbol include/clc_b200.h declares, its host-only entry points work, and every compute entry point FAILS LOUDLY
(no CPU fallback) when no CUDA device is usable."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "clc_b200.h")


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(clc_[A-Za-z0-9_]+)\s*\(", text)))


@pytest.fixture(scope="module")
def lib():
    from camlasercalibratool_b200 import _lib

    return _lib.load()


def test_header_and_binding_agree():
    from camlasercalibratool_b200 import _lib

    assert declared_symbols() == sorted(_lib.SIGNATURES.keys())


def test_library_exports_every_declared_symbol(lib):
    from camlasercalibratool_b200 import _lib

    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.lib_path()], text=True)
    exported = set(re.findall(r"\bT (clc_[A-Za-z0-9_]+)", out))
    missing = [s for s in declared_symbols() if s not in exported]
    assert not missing, f"not exported: {missing}"
    for s in declared_symbols():
        assert getattr(lib, s) is not None


def test_library_is_sm90a_only():
    from camlasercalibratool_b200 import _lib

    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not installed")
    out = subprocess.check_output([cuobjdump, "-lelf", _lib.lib_path()], text=True)
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_header_compiles_as_plain_c(tmp_path):
    src = tmp_path / "t.c"
    src.write_text('#include "clc_b200.h"\nint main(void){ clc_lm_options o; (void)o; return CLC_OK; }\n')
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    subprocess.check_call([cc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), "-c",
                           str(src), "-o", str(tmp_path / "t.o")])


def test_default_options_are_the_ceres_defaults(lib):
    from camlasercalibratool_b200 import default_options

    o = default_options()
    assert o.max_num_iterations == 100  # reference src/LaseCamCalCeres.cpp:304
    assert (o.initial_trust_region_radius, o.max_trust_region_radius, o.min_trust_region_radius) == (1e4, 1e16, 1e-32)
    assert (o.function_tolerance, o.gradient_tolerance, o.parameter_tolerance) == (1e-6, 1e-10, 1e-8)
    assert (o.min_relative_decrease, o.min_lm_diagonal, o.max_lm_diagonal) == (1e-3, 1e-6, 1e32)
    assert o.max_num_consecutive_invalid_steps == 5 and o.jacobi_scaling == 1


def test_pose_conversions_match_eigen_restatement(lib, oracle):
    from camlasercalibratool_b200 import T_to_pose7, pose7_to_T

    rng = np.random.default_rng(0)
    for _ in range(50):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        T = np.eye(4)
        T[:3, :3] = oracle.quat_to_rot(q)
        T[:3, 3] = rng.normal(size=3)
        p = T_to_pose7(T)
        np.testing.assert_allclose(p, oracle.T_to_pose7(T), atol=1e-15)
        np.testing.assert_allclose(pose7_to_T(p), T, atol=1e-14)
    assert np.array_equal(T_to_pose7(np.eye(4)), [0, 0, 0, 0, 0, 0, 1])


def test_shard_range(lib):
    from camlasercalibratool_b200 import shard_range

    # by frame count
    for n, r in ((10, 3), (7, 8), (1000003, 8), (0, 4)):
        ranges = [shard_range(n, r, k) for k in range(r)]
        assert ranges[0][0] == 0 and ranges[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
        assert max(e - b for b, e in ranges) - min(e - b for b, e in ranges) <= 1
    # by point count (ragged frames)
    rng = np.random.default_rng(1)
    cnt = rng.integers(0, 200, size=500)
    off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    ranges = [shard_range(500, 4, k, off) for k in range(4)]
    assert ranges[0][0] == 0 and ranges[-1][1] == 500 and all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
    pts = [off[e] - off[b] for b, e in ranges]
    assert max(pts) - min(pts) <= 2 * cnt.max()
    with pytest.raises(Exception):
        shard_range(10, 0, 0)


def test_marshal_follows_the_reference_flags():
    from camlasercalibratool_b200 import Oberserve, marshal

    obs = []
    for i in range(3):
        ob = Oberserve()
        ob.tagPose_tca = np.array([i, 0.0, 1.0])
        ob.points = np.arange(3 * (i + 2), dtype=float).reshape(-1, 3)
        ob.points_on_line = ob.points[[0, -1]] + 0.5
        obs.append(ob)
    fp, off, pts, edge = marshal(obs, use_linefitting_data=False)
    assert off.tolist() == [0, 2, 5, 9] and edge is None and np.array_equal(fp[:, :4], [[0, 0, 0, 1]] * 3)
    fp, off, pts, edge = marshal(obs, use_linefitting_data=True, use_boundary_constraint=True)
    assert off.tolist() == [0, 2, 4, 6]
    assert np.array_equal(edge[1, :3], obs[1].points[0]) and np.array_equal(edge[1, 3:], obs[1].points[-1])
    # boundary constraint without line-fitting data is ignored, as at reference :258
    assert marshal(obs, use_linefitting_data=False, use_boundary_constraint=True)[3] is None


def _no_gpu():
    try:
        import torch

        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.mark.skipif(not _no_gpu(), reason="checks the behaviour on a box without a GPU")
def test_compute_entry_points_fail_loudly_without_a_gpu(lib):
    """No CPU fallback: creating a problem without a CUDA device is an error, never a silent host path."""
    from camlasercalibratool_b200 import ClcError, Problem

    with pytest.raises(ClcError):
        Problem.from_arrays(np.array([[0, 0, 0, 1, 0, 0, 1.0]]), [0, 2], np.zeros((2, 3)))
    with pytest.raises(ClcError):
        Problem.synthetic(4, 8)
    n = C.c_int(-1)
    assert lib.clc_device_count(C.byref(n)) != 0
    assert lib.clc_last_error()
    # the preparation steps have no host path either
    from camlasercalibratool_b200 import LineFittingCeres
    from camlasercalibratool_b200 import formats as fmt

    with pytest.raises(ClcError):
        LineFittingCeres(np.zeros((5, 3)), np.zeros(2))
    with pytest.raises(ClcError):
        fmt.auto_get_line_segments(np.ones((2, 100), dtype=np.float32), -1.0, 0.02, 0.05)
    with pytest.raises(ClcError):
        fmt.estimate_board_poses("equi", [(np.array([0], dtype=np.int32), np.zeros((1, 4, 2), dtype=np.float32))])


def test_pose_estimation_argument_checks(lib):
    """clc_estimate_board_poses validates its description before touching the device."""
    from camlasercalibratool_b200 import ClcError
    from camlasercalibratool_b200 import formats as fmt

    det = [(np.array([0], dtype=np.int32), np.zeros((1, 4, 2), dtype=np.float32))]
    with pytest.raises(KeyError):
        fmt.estimate_board_poses("fisheye", det)
    for kw in (dict(grid=(0, 6, 0.055, 0.3)), dict(grid=(6, 6, -1.0, 0.3)), dict(intrinsics=[0, 1, 0, 0, 0, 0, 0, 0])):
        with pytest.raises(ClcError) as exc:
            fmt.estimate_board_poses("equi", det, **kw)
        assert "camera" in str(exc.value) or "grid" in str(exc.value)
