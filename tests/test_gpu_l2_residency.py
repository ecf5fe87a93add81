"""GPU tests (-m gpu) of the L2 residency of LM solves (csrc/clc_l2_plan.h, issue_one in csrc/clc_kernels.cuh): the sweeps of a
solve read the last stages of every warp's range with evict_last and the rest with evict_first.  That is a cache policy, not
arithmetic: every point is summed by the same lane in the same order, so the trajectory must be identical bit for bit with
residency off, partly resident, at the default budget and entirely resident -- under one launch per LM iteration and under
the persistent grid that loops the LM by itself -- and an evaluation after the solve is untouched."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

X0 = np.array([0, 0, 0, 0, 0, 0, 1.0])


@pytest.mark.parametrize("planar", [False, True])
@pytest.mark.parametrize("loop_mode", [0, 2])
def test_l2_residency_changes_no_bit(monkeypatch, planar, loop_mode):
    from camlasercalibratool_b200 import Problem

    monkeypatch.setenv("CLC_LOOP_IN_KERNEL", str(loop_mode))
    monkeypatch.setenv("CLC_PLANAR", "1" if planar else "0")
    monkeypatch.delenv("CLC_L2_PERSIST_MB", raising=False)
    out = []
    # 2e6 points, 48 MB general / 32 MB planar: "8" keeps a few stages of every warp, the default (half of L2) more of them
    for budget_mb in ("0", None, "8", "100000"):
        if budget_mb is None:
            monkeypatch.delenv("CLC_L2_RESIDENT_MB", raising=False)
        else:
            monkeypatch.setenv("CLC_L2_RESIDENT_MB", budget_mb)
        with Problem.synthetic(2000, 1000, seed=5, sigma=0.01) as g:
            assert g.planar == planar
            x, s, tr = g.solve(X0)
            x2, s2, tr2 = g.solve(X0)
            assert np.array_equal(x, x2) and [t.cost for t in tr] == [t.cost for t in tr2]
            cost, H, grad = g.eval(x)
            out.append((x, [t.cost for t in tr], [t.trust_region_radius for t in tr], s.num_sweeps, s.num_iterations,
                        cost, H, grad))
    ref = out[0]
    for got in out[1:]:
        assert np.array_equal(got[0], ref[0])
        assert got[1] == ref[1] and got[2] == ref[2] and got[3] == ref[3] and got[4] == ref[4]
        assert got[5] == ref[5] and np.array_equal(got[6], ref[6]) and np.array_equal(got[7], ref[7])
