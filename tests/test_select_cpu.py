"""CPU tests of the frame selection that need no GPU.

* the product's CLC_HD Cholesky and gain (clc_select.cuh, compiled with g++ by tests/select_harness.cpp) against the long-double
  restatement of tests/select_reference.py, on random PSD blocks of rank 1-6 and condition up to 1e8;
* the padding of held coordinates (zeros in the block, the identity in A) leaves every gain what the d x d computation gives;
* the reference's greedy rule on diagonal blocks, whose gains have a closed form;
* the Python argument checks raise before any library call.
"""
import numpy as np
import pytest

import select_reference as SR

LD = SR.LD


@pytest.fixture(scope="module")
def SH(tmp_path_factory):
    return SR.SelectHarness(tmp_path_factory.mktemp("select_harness"))


def _psd(rng, rank, cond, scale=1.0):
    """A random 6x6 PSD matrix of the given rank whose non-zero eigenvalues span `cond`."""
    Q, _ = np.linalg.qr(rng.standard_normal((6, 6)))
    ev = np.zeros(6)
    ev[:rank] = scale * np.geomspace(1.0, 1.0 / cond, rank) if rank > 1 else scale
    return (Q * ev) @ Q.T


def _spd(rng, cond):
    A = _psd(rng, 6, cond)
    return 0.5 * (A + A.T)


def _blocks(rng):
    H = []
    for rank in range(1, 7):
        for cond in (1.0, 1e4, 1e8):
            for scale in (1e-9, 1e-3, 1.0, 1e3):
                Hk = _psd(rng, rank, cond, scale)
                H.append(0.5 * (Hk + Hk.T))
    return np.array(H)


# The whitening L^-1 H L^-T loses about cond(A) ulps in double whatever way it is formed, so the bound is 1e-12 while A is well
# conditioned and grows with cond(A) beyond that.
@pytest.mark.parametrize("cond_a", [1.0, 10.0, 1e4, 1e6, 1e8])
def test_gains_against_long_double(SH, cond_a):
    """sel_chol6 + sel_gain6 against the long-double factor and gains of the same A, and sel_gain6 alone at the product's factor."""
    rng = np.random.default_rng(int(np.log10(cond_a)) + 7)
    bound = max(1e-12, 4e-14 * cond_a)
    for _ in range(10):
        A = _spd(rng, cond_a)
        H = _blocks(rng)
        gl = SR.gains(A, H, LD).astype(np.float64)
        assert np.all(np.abs(SH.gains(A, H) - gl) <= bound * np.abs(gl)), cond_a
        ok, L, _ = SH.chol(A)
        gl = SR.gains_at(L, H, LD).astype(np.float64)
        assert np.all(np.abs(SH.gains_at(L, H) - gl) <= bound * np.abs(gl)), cond_a


def test_cholesky_against_long_double(SH):
    rng = np.random.default_rng(3)
    for cond in (1.0, 1e4, 1e8):
        for _ in range(20):
            A = _spd(rng, cond)
            ok, L, inv = SH.chol(A)
            assert ok
            Ll = SR.chol(A, LD)
            # a backward-stable factorisation: the factor's forward error grows with sqrt(cond(A))
            assert np.abs(L - Ll.astype(np.float64)).max() <= 1e-14 * np.sqrt(cond) * np.abs(Ll.astype(np.float64)).max()
            assert np.allclose(inv, 1.0 / np.diag(L), rtol=0, atol=0)
            assert np.all(np.triu(L, 1) == 0.0)
    ok, _, _ = SH.chol(np.diag([1.0, 1.0, -1.0, 1.0, 1.0, 1.0]))
    assert not ok
    ok, _, _ = SH.chol(np.diag([1.0, 1.0, np.inf, 1.0, 1.0, 1.0]))
    assert not ok


def test_special_blocks(SH):
    A = np.eye(6)
    zero = np.zeros((6, 6))
    nan = np.zeros((6, 6))
    nan[2, 2] = np.nan
    g = SH.gains(A, np.array([zero, nan]))
    assert g[0] == 0.0 and np.signbit(g[0]) == 0
    assert g[1] == -np.inf
    # a diagonal block at A = I: sum log1p of its diagonal, exactly as the closed form evaluates it
    d = np.array([0.5, 1e-12, 3.0, 0.0, 7.0, 1e-3])
    assert SH.gains(A, np.diag(d)[None])[0] == pytest.approx(np.sum(np.log1p(d)), rel=1e-15)


@pytest.mark.parametrize("mask", [0b000001, 0b101000, 0b000111, 0b011111])
def test_held_coordinates_are_padding(SH, mask):
    """The step kernel works on 6x6: the d free coordinates first, the held ones zero in the block and the identity in A.  Its gains
    equal the long-double gains of the d x d principal blocks."""
    rng = np.random.default_rng(mask)
    fr = SR.free_coords(mask)
    d = len(fr)
    A6 = _spd(rng, 1e3)
    H6 = np.array([_psd(rng, r, 1e4) for r in range(1, 7)])
    Ad = A6[np.ix_(fr, fr)]
    Hd = H6[:, fr][:, :, fr]
    Ap = np.eye(6)
    Ap[:d, :d] = Ad
    Hp = np.zeros((6, 6, 6))
    Hp[:, :d, :d] = Hd
    g = SH.gains(Ap, Hp)
    gl = SR.gains(Ad, Hd, LD).astype(np.float64)
    assert np.all(np.abs(g - gl) <= 1e-12 * np.abs(gl))


def test_reference_greedy_closed_form():
    """Diagonal blocks: T_kk = sum of column k, Ht diagonal, A_s diagonal, gain = sum_k log1p(h_k / a_k)."""
    rng = np.random.default_rng(11)
    n = 12
    diag = rng.uniform(0.1, 5.0, (n, 6)) * rng.permutation(np.arange(1, n + 1))[:, None]
    H = np.zeros((n, 6, 6))
    H[:, np.arange(6), np.arange(6)] = diag
    order, gain, keep, _ = SR.greedy(SR.pack(H), 5)
    T = diag.sum(axis=0)
    a = np.full(6, SR.RIDGE / n)
    ht = diag / T
    rem = list(range(n))
    for s in range(5):
        g = np.array([np.sum(np.log1p(ht[f] / a)) for f in rem])
        f = rem[int(np.argmax(g))]
        assert order[s] == f
        assert gain[s] == pytest.approx(g.max(), rel=1e-13)
        a = a + ht[f]
        rem.remove(f)
    assert keep.sum() == 5 and np.all(keep[order])


# ---- the Python argument checks: no library call before they pass ------------------------------------------------------------
@pytest.fixture
def no_library(monkeypatch):
    from camlasercalibratool_b200 import _lib

    def refuse():
        raise AssertionError("the library was called before the arguments were checked")

    monkeypatch.setattr(_lib, "load", refuse)


def _rows(n):
    from camlasercalibratool_b200 import FRAME_ROW_DTYPE

    rows = np.zeros(n, dtype=FRAME_ROW_DTYPE)
    rows["H21"][:, [0, 6, 11, 15, 18, 20]] = 1.0
    return rows


@pytest.mark.parametrize("kw, exc", [
    (dict(budget=-1), ValueError),
    (dict(budget=2.0), TypeError),
    (dict(budget=True), TypeError),
    (dict(budget=2, min_gain=float("nan")), ValueError),
    (dict(budget=2, min_gain=-1e-3), ValueError),
    (dict(budget=2, min_gain=float("inf")), ValueError),
    (dict(budget=2, candidates=np.ones(4, dtype=np.uint8)), TypeError),
    (dict(budget=2, candidates=np.ones(3, dtype=bool)), ValueError),
    (dict(budget=2, forced=np.ones((4, 1), dtype=bool)), ValueError),
    (dict(budget=2, fixed=("tx", "ty", "tz", "rx", "ry", "rz")), ValueError),
    (dict(budget=2, fixed=("yaw",)), ValueError),
])
def test_python_checks_before_the_library(no_library, kw, exc):
    from camlasercalibratool_b200 import Problem, select_frames_from_report

    with pytest.raises(exc):
        select_frames_from_report(_rows(4), **kw)
    p = Problem.__new__(Problem)
    p._h = None
    p.sizes = lambda: (4, 0, False)
    p._L = None  # any attribute access on the library fails the test
    with pytest.raises(exc):
        p.select_frames(np.array([0, 0, 0, 0, 0, 0, 1.0]), **kw)


def test_rows_must_be_report_rows(no_library):
    from camlasercalibratool_b200 import select_frames_from_report

    with pytest.raises(TypeError):
        select_frames_from_report(np.zeros((4, 21)), 2)
    with pytest.raises(TypeError):
        select_frames_from_report(_rows(4).reshape(2, 2), 2)
