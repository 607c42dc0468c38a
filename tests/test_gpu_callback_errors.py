"""A Python f that raises propagates as its own exception from every entry point that calls f through the C ABI, and the
cache, group or block it was called with stays usable: the next call returns exactly what a fresh one does.  (The
Hessian and gradient entry points have such tests of their own.)"""
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from _util import assert_same_bits, cyc_colors, tridiag_csc  # noqa: E402

N = 40
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def fdist(pkg):
    from finitediff_jl_b200 import distributed
    return distributed


class Boom(Exception):
    pass


def failing(f, at):
    """f, except that its at-th call raises Boom."""
    calls = [0]

    def g(*args):
        calls[0] += 1
        if calls[0] == at:
            raise Boom()
        return f(*args)
    return g


def f_ip(fx, x):
    """f!(fx, x): a nonlinear tridiagonal map"""
    fx.copy_(x * x)
    fx[1:] += x[:-1]
    fx[:-1] += 2 * x[1:]


def f_oop(x):
    fx = torch.empty_like(x)
    f_ip(fx, x)
    return fx


def f_slice(r0, r1, x0, x1):
    """rows [r0, r1) of f_ip from x[x0:x1] (the slice holds every column those rows read)"""
    def f(fx, xs):
        full = torch.zeros(N, dtype=xs.dtype, device=xs.device)
        full[x0:x1] = xs
        fx.copy_(f_oop(full)[r0:r1])
    return f


def _x():
    return torch.linspace(0.5, 2.0, N, dtype=torch.float64, device=DEV)


def _J(pkg):
    colptr, rowval = tridiag_csc(N)
    return pkg.SparseMatrixCSC(N, N, torch.from_numpy(colptr), torch.from_numpy(rowval),
                               torch.full((len(rowval),), float("nan"), dtype=torch.float64, device=DEV))


CV = cyc_colors(N, 5)          # a valid colouring with two colours on each member of a two-member group
CASES = [(fd, at) for fd in ("forward", "central") for at in (1, 2)]


@pytest.mark.parametrize("fd, at", CASES)
def test_jacobian_inplace(pkg, fd, at):
    x, J, ref = _x(), _J(pkg), _J(pkg)
    cache = pkg.JacobianCache(x, fd, colorvec=CV, sparsity=J)
    with pytest.raises(Boom):
        pkg.finite_difference_jacobian_(J, failing(f_ip, at), x, cache)
    pkg.finite_difference_jacobian_(J, f_ip, x, cache)
    pkg.finite_difference_jacobian_(ref, f_ip, x, pkg.JacobianCache(x, fd, colorvec=CV, sparsity=ref))
    assert_same_bits(J.nzval, ref.nzval, fd, allow_nan=False)


@pytest.mark.parametrize("fd, at", CASES)
def test_jvp_inplace(pkg, fd, at):
    x = _x()
    v = torch.linspace(-1.0, 1.0, N, dtype=torch.float64, device=DEV)
    jvp, ref = (torch.full((N,), float("nan"), dtype=torch.float64, device=DEV) for _ in range(2))
    cache = pkg.JVPCache(x, fd)
    with pytest.raises(Boom):
        pkg.finite_difference_jvp_(jvp, failing(f_ip, at), x, v, cache)
    pkg.finite_difference_jvp_(jvp, f_ip, x, v, cache)
    pkg.finite_difference_jvp_(ref, f_ip, x, v, pkg.JVPCache(x, fd))
    assert_same_bits(jvp, ref, fd, allow_nan=False)


@pytest.mark.parametrize("fd, at", CASES)
def test_derivative_inplace(pkg, fd, at):
    x = _x()
    sq = lambda t: t * t + 3 * t                             # noqa: E731
    df, ref = (torch.full((N,), float("nan"), dtype=torch.float64, device=DEV) for _ in range(2))
    cache = pkg.DerivativeCache(x, fdtype=fd)
    with pytest.raises(Boom):
        pkg.finite_difference_derivative_(df, failing(sq, at), x, cache)
    pkg.finite_difference_derivative_(df, sq, x, cache)
    pkg.finite_difference_derivative_(ref, sq, x, pkg.DerivativeCache(x, fdtype=fd))
    assert_same_bits(df, ref, fd, allow_nan=False)


@pytest.mark.parametrize("fd, at", CASES)
@pytest.mark.parametrize("sparse", [False, True])
def test_jacobian_out_of_place(pkg, fd, at, sparse):
    x, S = _x(), _J(pkg)
    kw = dict(colorvec=CV, sparsity=S, jac_prototype=S) if sparse else {}
    cache = pkg.JacobianCache(x, fd)
    with pytest.raises(Boom):
        pkg.finite_difference_jacobian(failing(f_oop, at), x, cache, **kw)
    got = pkg.finite_difference_jacobian(f_oop, x, cache, **kw)
    ref = pkg.finite_difference_jacobian(f_oop, x, pkg.JacobianCache(x, fd), **kw)
    if sparse:
        assert torch.equal(got.colptr, ref.colptr) and torch.equal(got.rowval, ref.rowval)
        got, ref = got.nzval, ref.nzval
    assert_same_bits(got, ref, fd, allow_nan=False)


@pytest.mark.parametrize("fd, at", CASES)
@pytest.mark.parametrize("member", [0, 1])
def test_group_jacobian(pkg, fdist, fd, at, member):
    x, J, ref = _x(), _J(pkg), _J(pkg)
    g = fdist.GroupJacobian(J, CV, fd, [0, 0])
    fs = [f_ip, f_ip]
    fs[member] = failing(f_ip, at)
    with pytest.raises(Boom):
        g.run(fs, x)
    g.run([f_ip, f_ip], x)
    g2 = fdist.GroupJacobian(ref, CV, fd, [0, 0])
    g2.run([f_ip, f_ip], x)
    g.synchronize()
    assert_same_bits(J.nzval, ref.nzval, fd, allow_nan=False)
    g.close()
    g2.close()


@pytest.mark.parametrize("fd, at", CASES)
@pytest.mark.parametrize("member", [0, 1])
def test_group_jacobian_out_of_place(pkg, fdist, fd, at, member):
    x = _x()
    g = fdist.GroupJacobianOOP([0, 0], fd, colorvec=CV, sparsity=_J(pkg))
    fs = [f_oop, f_oop]
    fs[member] = failing(f_oop, at)
    with pytest.raises(Boom):
        g.run(fs, x)
    got = g.run([f_oop, f_oop], x)
    g2 = fdist.GroupJacobianOOP([0, 0], fd, colorvec=CV, sparsity=_J(pkg))
    ref = g2.run([f_oop, f_oop], x)
    assert_same_bits(got, ref, fd, allow_nan=False)
    g.close()
    g2.close()


@pytest.mark.parametrize("fd, at", CASES)
def test_column_block_jacobian(pkg, fdist, fd, at):
    x, J, ref = _x(), _J(pkg), _J(pkg)
    bounds = fdist.column_blocks(J.colptr, 2)
    eps = fdist.EpsPlan(N, CV, fd, DEV).compute(x)
    bad = fdist.ColumnBlockJacobian(J, CV, fd, bounds[0], bounds[1], DEV, lambda *r: failing(f_slice(*r), at))
    with pytest.raises(Boom):
        bad.run(x, eps)
    bad.run(x, eps)                                     # the same block, whose f no longer raises
    fdist.ColumnBlockJacobian(J, CV, fd, bounds[1], bounds[2], DEV, f_slice).run(x, eps)
    for r in range(2):
        fdist.ColumnBlockJacobian(ref, CV, fd, bounds[r], bounds[r + 1], DEV, f_slice).run(x, eps)
    torch.cuda.synchronize()
    assert_same_bits(J.nzval, ref.nzval, fd, allow_nan=False)
