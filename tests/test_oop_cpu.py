"""The out-of-place forms' CPU restatement (tests/_literal_oop.py) against answers derived by hand and the reference's
own out-of-place tests.  No GPU needed.

Hand-derived answers are the ones a transcription could get wrong in the same way as the device: the sign of a zero
quotient in each result kind, NaN kept by the sparse `+`, the central step's sign under dir = -1, the signed-zero points
of a colour loop that starts every colour from the caller's x, the call counts of each form, and the error of a dense
result on an invalid colouring."""
import numpy as np
import pytest
import scipy.sparse as sp

import _literal_oop as LO

EPS = np.finfo(np.float64).eps


def bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all((bits(a) == bits(b)) | (np.isnan(a) & np.isnan(b))))


def tridiag(n):
    A = sp.diags([np.ones(n - 1), np.ones(n), np.ones(n - 1)], [-1, 0, 1], format="csc")
    A.sort_indices()
    return (n, n, A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1)


def stencil(x):
    """f(x) = xm1 - 2x + xp1 of test/out_of_place_tests.jl:3-7"""
    xm1 = np.concatenate([[0.0], x[:-1]])
    xp1 = np.concatenate([x[1:], [0.0]])
    return xm1 - 2 * x + xp1


def second_derivative_stencil(n):
    return sp.diags([np.ones(n - 1), -2 * np.ones(n), np.ones(n - 1)], [-1, 0, 1]).toarray()


def to_dense(res):
    if res[0] == "dense":
        return res[1]
    _, m, n, cp, rv, nz = res
    return sp.csc_matrix((nz, rv - 1, cp - 1), shape=(m, n)).toarray()


# ---------------------------------------------------------------- hand-derived answers
def test_negative_zero_quotient_in_each_result_kind():
    # f constant, dir = -1: every quotient is (+0.0)/(-eps) = -0.0
    f = LO.Recorder(lambda x: np.array([1.0, 2.0]))
    x = np.array([0.5, 0.25])
    raw = LO.jacobian_oop(f, x, "forward", dir=-1.0)
    assert raw[0] == "dense" and np.all(np.signbit(raw[1])) and np.all(raw[1] == 0)           # kept as -0.0
    dense = LO.jacobian_oop(f, x, "forward", dir=-1.0, jac_prototype=("dense", 2, 2))
    assert same_bits(dense[1], np.zeros((2, 2)))                                               # 0.0 + (-0.0) = +0.0
    spr = LO.jacobian_oop(f, x, "forward", dir=-1.0, jac_prototype=("sparse", 2, 2))
    assert spr[4].size == 0 and list(spr[3]) == [1, 1, 1]                                      # dropped
    pat = (2, 2, np.array([1, 3, 5]), np.array([1, 2, 1, 2]))
    spc = LO.jacobian_oop(f, x, "forward", dir=-1.0, sparsity=pat, jac_prototype=("sparse", 2, 2))
    assert spc[4].size == 0


def test_nan_is_kept_and_positive_zero_dropped():
    f = LO.Recorder(lambda x: np.array([np.nan, 3.0, x[1] * 2.0]))
    x = np.array([1.0, 2.0])
    res = LO.jacobian_oop(f, x, "forward", jac_prototype=("sparse", 3, 2))
    # column 1: d/dx1 = [NaN, 0, 0] -> NaN kept, +0.0 dropped; column 2: [NaN, 0, 2]
    assert list(res[3]) == [1, 2, 4]
    assert list(res[4]) == [1, 1, 3]
    assert np.isnan(res[5][0]) and np.isnan(res[5][1]) and res[5][2] != 0


def test_central_step_takes_dir():
    f = LO.Recorder(lambda x: x * x)
    x = np.array([1.0])
    LO.jacobian_oop(f, x, "central", dir=-1.0)
    e = -np.cbrt(EPS)                                                                          # forward rule, times dir
    assert len(f.points) == 2
    assert same_bits(f.points[0], [1.0 + e]) and f.points[0][0] < 1.0                          # f(x + eps) first
    assert same_bits(f.points[1], [1.0 - e])
    g = LO.Recorder(lambda x: x * x)
    pat = (1, 1, np.array([1, 2]), np.array([1]))
    LO.jacobian_oop(g, x, "central", dir=-1.0, sparsity=pat)
    assert g.points[0][0] < 1.0 < g.points[1][0]


def test_pristine_signed_zero_points():
    x = np.array([-0.0, -0.0, 1.0])
    pat = (3, 3, np.array([1, 2, 3, 4]), np.array([1, 2, 3]))
    cv = [1, 2, 1]
    for dir_, fd in ((1.0, "forward"), (-1.0, "forward"), (1.0, "central")):
        f = LO.Recorder(lambda x: x * 1.0)
        e = [0.5 * dir_, 0.25 * dir_]
        LO.jacobian_oop(f, x, fd, f_in=np.zeros(3) if fd == "forward" else None, sparsity=pat, colorvec=cv, dir=dir_,
                        eps_override=e)
        z = [np.copysign(0.0, v) for v in e]
        if fd == "forward":
            exp = [np.array([e[0], -0.0 + z[0], 1.0 + e[0]]), np.array([-0.0 + z[1], e[1], 1.0])]
        else:
            exp = [np.array([e[0], -0.0 + z[0], 1.0 + e[0]]), np.array([-0.0 - e[0], -0.0 - z[0], 1.0 - e[0]]),
                   np.array([-0.0 + z[1], e[1], 1.0]), np.array([-0.0 - z[1], -0.0 - e[1], 1.0])]
        assert len(f.points) == len(exp)
        for got, want in zip(f.points, exp):
            assert same_bits(got, want), (fd, dir_, got, want)
    # dir = -1: colour 2's point keeps -0.0 on component 1 (-0.0 + -0.0); dir = +1 turns it into +0.0
    f = LO.Recorder(lambda x: x * 1.0)
    LO.jacobian_oop(f, x, "forward", f_in=np.zeros(3), sparsity=pat, colorvec=cv, dir=-1.0, eps_override=[-0.5, -0.25])
    assert np.signbit(f.points[1][0])
    f = LO.Recorder(lambda x: x * 1.0)
    LO.jacobian_oop(f, x, "forward", f_in=np.zeros(3), sparsity=pat, colorvec=cv, dir=1.0, eps_override=[0.5, 0.25])
    assert not np.signbit(f.points[1][0])


def test_complex_points_add_positive_zero():
    x = np.array([-0.0, 2.0])
    f = LO.Recorder(lambda z: z * 1.0)
    pat = (2, 2, np.array([1, 2, 3]), np.array([1, 2]))
    LO.jacobian_oop(f, x, "complex", sparsity=pat, colorvec=[1, 2])
    assert not np.signbit(f.points[0][0].real) and not np.signbit(f.points[1][0].real)        # -0.0 + 0.0
    g = LO.Recorder(lambda z: z * 1.0)
    LO.jacobian_oop(g, x, "complex")                                                           # dense: setindex only
    assert not np.signbit(g.points[0][0].real) and np.signbit(g.points[1][0].real)


@pytest.mark.parametrize("fd,cacheless,f_in,expected", [
    ("forward", False, False, 31), ("forward", False, True, 30), ("forward", True, False, 31),
    ("central", False, False, 60), ("central", True, False, 61),
    ("complex", False, False, 30), ("complex", True, False, 31)])
def test_call_counts(fd, cacheless, f_in, expected):
    x = np.linspace(0.5, 1.5, 30)
    f = LO.Recorder(lambda v: stencil(v) + 0.0)
    LO.jacobian_oop(f, x, fd, f_in=stencil(x) if f_in else None, cacheless=cacheless)
    assert len(f.points) == expected
    g = LO.Recorder(lambda v: stencil(v) + 0.0)
    LO.jacobian_oop(g, x, fd, sparsity=tridiag(30), colorvec=np.arange(30) % 3 + 1, cacheless=cacheless,
                    jac_prototype=("sparse", 30, 30))
    colours = 3 * (2 if fd == "central" else 1) + (1 if fd == "forward" or cacheless else 0)
    assert len(g.points) == colours


def test_jvp_call_order_and_counts():
    x, v = np.array([1.0, 2.0]), np.array([0.5, -1.0])
    f = LO.Recorder(lambda z: z * z)
    _, e = LO.jvp_oop(f, x, v, "central", dir=-1.0)
    assert e > 0                                                                               # central: dir ignored
    assert same_bits(f.points[0], x + e * v) and same_bits(f.points[1], x - e * v)             # plus point first
    f = LO.Recorder(lambda z: z * z)
    LO.jvp_oop(f, x, v, "forward", cacheless=True)
    assert len(f.points) == 2 and same_bits(f.points[0], x)
    f = LO.Recorder(lambda z: z * z)
    LO.jvp_oop(f, x, v, "central", cacheless=True)
    assert len(f.points) == 3


def test_invalid_colouring_raises_for_a_dense_result_only():
    pat = (2, 2, np.array([1, 3, 5]), np.array([1, 2, 1, 2]))
    f = LO.Recorder(lambda x: x * x)
    with pytest.raises(LO.MakeJiError):
        LO.jacobian_oop(f, np.array([1.0, 2.0]), "forward", sparsity=pat, colorvec=[1, 1])
    res = LO.jacobian_oop(f, np.array([1.0, 2.0]), "forward", sparsity=pat, colorvec=[1, 1],
                          jac_prototype=("sparse", 2, 2))
    assert res[0] == "sparse"


def test_fast_csc_restatement_matches_the_literal():
    rng = np.random.default_rng(7)
    for fd in ("forward", "central"):
        for dir_ in (1.0, -1.0):
            n = 40
            pat = tridiag(n)
            cv = np.arange(n) % 3 + 1
            x = rng.uniform(-1, 1, n)
            x[::7] = 0.0
            x[3] = -0.0
            eps = [1e-3 * dir_, 2e-3 * dir_, 3e-3 * dir_]
            mask = (np.arange(n) % 5 != 0).astype(float)
            f = lambda v: (v * v) * mask + 1.0
            lit = LO.jacobian_oop(LO.Recorder(f), x, fd, sparsity=pat, colorvec=cv, dir=dir_, eps_override=eps,
                                  jac_prototype=("sparse", n, n))
            fast = LO.jacobian_oop_csc_fast(f, x, fd, eps, n, pat[2], pat[3], cv)
            for a, b in zip(lit[3:], fast[3:]):
                assert same_bits(a.astype(np.float64), b.astype(np.float64))
            dense = LO.jacobian_oop(LO.Recorder(f), x, fd, sparsity=pat, colorvec=cv, dir=dir_, eps_override=eps)
            r0, c0, v = LO.jacobian_oop_csc_fast(f, x, fd, eps, n, pat[2], pat[3], cv, sparse=False)
            want = np.zeros((n, n))
            want[r0, c0] = v
            assert same_bits(dense[1], want)


# ---------------------------------------------------------------- the reference's own out-of-place tests
@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_kat_stencil_dense(fd):
    # test/out_of_place_tests.jl:17-25 (and coloring_tests.jl:28-31 for the 31 calls)
    x = np.ones(30)
    J = LO.jacobian_oop(stencil, x, fd, cacheless=True)[1]
    assert np.allclose(J, second_derivative_stencil(30), atol=1e-6)


def test_kat_stencil_sparse_prototype_and_colours():
    # test/out_of_place_tests.jl:27-36
    x = np.ones(30)
    A = sp.csc_matrix(second_derivative_stencil(30))
    A.sort_indices()
    pat = (30, 30, A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1)
    r1 = LO.jacobian_oop(stencil, x, "forward", jac_prototype=("sparse", 30, 30), cacheless=True)
    assert r1[0] == "sparse" and np.allclose(to_dense(r1), second_derivative_stencil(30), atol=1e-6)
    r2 = LO.jacobian_oop(stencil, x, "forward", colorvec=np.tile([1, 2, 3], 10), sparsity=pat,
                         jac_prototype=("sparse", 30, 30), cacheless=True)
    assert r2[0] == "sparse" and np.allclose(to_dense(r2), second_derivative_stencil(30), atol=1e-6)


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_kat_one_by_one_and_two_by_one(fd):
    # test/out_of_place_tests.jl:38-59
    J = LO.jacobian_oop(lambda x: x * 1.0, np.array([1.0]), fd, cacheless=True)[1]
    assert J.shape == (1, 1) and abs(J[0, 0] - 1.0) < 1e-6
    J = LO.jacobian_oop(lambda x: np.concatenate([x, x]), np.array([1.0]), fd, cacheless=True)[1]
    assert J.shape == (2, 1) and np.allclose(J, 1.0, atol=1e-6)


def test_kat_range_input_and_dir():
    # test/finitedifftests.jl:541-552: f(x) = x.^2 + sin(x) on a 2-element range
    x = np.array([0.3, 0.7])
    f = lambda v: v ** 2 + np.sin(v)
    Jref = np.diag(2 * x + np.cos(x))
    assert np.abs(LO.jacobian_oop(f, x, "forward")[1] - Jref).max() < 1e-4
    assert np.abs(LO.jacobian_oop(f, x, "forward", dir=-1.0)[1] - Jref).max() < 1e-4
    assert np.abs(LO.jacobian_oop(f, x, "forward", f_in=f(x))[1] - Jref).max() < 1e-4
    assert np.abs(LO.jacobian_oop(f, x, "central")[1] - Jref).max() < 1e-8
    fc = lambda v: v ** 2 + np.sin(v)
    assert np.abs(LO.jacobian_oop(fc, x, "complex")[1] - Jref).max() < 1e-14


def _oopf(x):
    """oopf of test/finitedifftests.jl:403-406"""
    return np.array([(x[0] + 3) * (x[1] ** 3 - 7) + 18, np.sin(x[1] * np.exp(x[0]) - 1)])


def _J_ref(x):
    c = np.cos(x[1] * np.exp(x[0]) - 1)
    return np.array([[x[1] ** 3 - 7, 3 * x[1] ** 2 * (x[0] + 3)], [x[1] * np.exp(x[0]) * c, np.exp(x[0]) * c]])


class _Throws(Exception):
    pass


@pytest.mark.parametrize("impl", ["literal", "c"])
def test_kat_oopf_jacobian_and_jvp(impl):
    """test/finitedifftests.jl:403-446: oopf, its Jacobian and J*vdir, forward (dir = -1, relstep, f_in), central and
    complex; oopff throws when a point leaves {x .<= z}: with dir = -1 every forward point stays below x (:430-432, :440-442)"""
    from oop_oracle import fd_oop_oracle as OO
    R = LO if impl == "literal" else OO
    rng = np.random.default_rng(403)
    x, vdir = rng.random(2), rng.random(2)
    z = x.copy()

    def oopff(v):
        if not np.all(np.real(v) <= z):
            raise _Throws()
        return _oopf(v)
    J, jv = _J_ref(x), _J_ref(x) @ vdir
    err = lambda a, b: np.abs(np.asarray(a) - b).max()
    assert err(R.jacobian_oop(_oopf, x, "forward")[1], J) < 1e-6                                   # :430
    assert err(R.jacobian_oop(oopff, x, "forward", dir=-1.0)[1], J) < 1e-6                         # :431
    if impl == "literal":                                                                          # :432 (raises through C)
        with pytest.raises(_Throws):
            R.jacobian_oop(oopff, x, "forward")
    assert err(R.jacobian_oop(_oopf, x, "forward", relstep=np.sqrt(np.finfo(float).eps))[1], J) < 1e-6   # :433
    assert err(R.jacobian_oop(_oopf, x, "forward", _oopf(x))[1], J) < 1e-6                         # :434
    assert err(R.jacobian_oop(_oopf, x, "central")[1], J) < 1e-8                                   # :435-436
    fc = lambda v: np.array([(v[0] + 3) * (v[1] ** 3 - 7) + 18, np.sin(v[1] * np.exp(v[0]) - 1)])
    assert err(R.jacobian_oop(fc, x, "complex")[1], J) < 1e-14                                     # :437
    assert err(R.jvp_oop(_oopf, x, vdir, "forward")[0], jv) < 1e-6                                 # :440
    assert err(R.jvp_oop(oopff, x, vdir, "forward", dir=-1.0)[0], jv) < 1e-6                       # :441
    assert err(R.jvp_oop(_oopf, x, vdir, "forward", relstep=np.sqrt(np.finfo(float).eps))[0], jv) < 1e-6   # :443
    assert err(R.jvp_oop(_oopf, x, vdir, "forward", _oopf(x))[0], jv) < 1e-6                       # :444
    assert err(R.jvp_oop(_oopf, x, vdir, "central")[0], jv) < 1e-8                                 # :445
    assert err(R.jvp_oop(_oopf, x, vdir, "central", cacheless=True)[0], jv) < 1e-8                 # :446


@pytest.mark.parametrize("fd", ["forward", "central", "complex"])
def test_kat_non_vector_input(fd):
    """test/finitedifftests.jl:518-524: x a 2x2 matrix, f(x) = x, J = I(4) (x enters as vec(x)).  The cases at :498-506
    take a complex x, which the out-of-place path does not build."""
    x = np.random.default_rng(518).random((2, 2)).reshape(-1, order="F")
    J = LO.jacobian_oop(lambda v: v * 1.0, x, fd, cacheless=True)[1]
    assert np.abs(J - np.eye(4)).max() < 1e-8
