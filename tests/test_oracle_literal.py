"""The C oracle against an independent line-by-line Python transcription of the reference (tests/_literal_reference.py)
on random problems: every sparsity / J kind of the path, forward and central, random relstep / absstep / dir / f_in,
colourings that are NOT valid (overlapping writes resolved by colour order) and colorvec entries < 1.  Fed the same step
sizes the two restatements must agree bit for bit in J, in the f!-call count and in the drifted end state of cache.x1;
their own step sizes are bit-identical too: both evaluate `norm` as the reference does (stdlib generic_norm2 below 32
components, OpenBLAS's x87 dnrm2 from 32 on — tests/test_oracle_norm.py pins that half against OpenBLAS itself)."""
import numpy as np
import pytest
import scipy.sparse as sps

import _literal_reference as lit
from _util import assert_same_bits

FD = {"forward": 0, "central": 1}
KINDS = ["csc_same", "csc_to_dense", "proto_to_dense", "banded", "banded_to_dense", "dense_cols"]


def _problem(rng, kind, long_x=False):
    m, n = int(rng.integers(3, 24)), int(rng.integers(3, 24))
    if long_x:                                   # 32 or more components: norm takes its BLAS (dnrm2) branch
        n = int(rng.integers(32, 72))
    if kind in ("banded", "banded_to_dense"):
        l, u = int(rng.integers(0, 4)), int(rng.integers(0, 4))
        D = np.zeros((m, n), bool)
        for c in range(n):
            D[max(0, c - u):min(m, c + l + 1), c] = True
    else:
        l = u = 0
        D = rng.random((m, n)) < 0.3
        D[rng.integers(0, m), :] |= rng.random(n) < 0.5
    W = rng.uniform(-1, 1, (m, n)) * D
    q = rng.integers(0, n, m)

    def f(fx, x):
        fx[:] = W @ x + 0.1 * x[q] ** 2

    return m, n, l, u, D, f


@pytest.mark.parametrize("seed", range(100))
@pytest.mark.parametrize("kind", KINDS)
def test_oracle_matches_literal_transcription(oracle, kind, seed):
    rng = np.random.default_rng(1000 * seed + KINDS.index(kind))
    m, n, l, u, D, f = _problem(rng, kind, long_x=seed % 3 == 2)
    fdtype = "forward" if rng.random() < 0.5 else "central"
    x = rng.uniform(-2, 2, n)
    kw = {}
    if rng.random() < 0.3:
        kw["relstep"] = float(10 ** rng.uniform(-9, -5))
    if rng.random() < 0.3:
        kw["absstep"] = float(10 ** rng.uniform(-10, -6))
    if fdtype == "forward" and rng.random() < 0.3:
        kw["dir"] = -1.0
    if kind == "dense_cols":
        cv = np.arange(1, n + 1, dtype=np.int64)
    else:
        C = int(rng.integers(1, 7))
        cv = rng.integers(0 if rng.random() < 0.3 else 1, C + 1, n).astype(np.int64)
        if cv.max() < 1:
            cv[0] = 1
    f_in = None
    if fdtype == "forward" and rng.random() < 0.3:
        f_in = np.zeros(m)
        f(f_in, x)
    A = sps.csc_matrix(D)
    A.sort_indices()
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1

    # ---- the literal transcription
    if kind == "csc_same":
        J = lit.CSC(m, n, colptr, rowval, np.full(A.nnz, np.nan))
        sparsity = J
    elif kind == "csc_to_dense":
        J = np.full((m, n), np.nan)
        sparsity = lit.CSC(m, n, colptr, rowval)
    elif kind == "proto_to_dense":
        J = np.full((m, n), np.nan)
        sparsity = D.astype(np.float64)
    elif kind == "banded":
        J = lit.Banded(m, n, l, u, np.full((l + u + 1, n), np.nan))
        sparsity = J
    elif kind == "banded_to_dense":
        J = np.full((m, n), np.nan)
        sparsity = lit.Banded(m, n, l, u)
    else:
        J = np.full((m, n), np.nan)
        sparsity = None
    cache_l = dict(x1=np.full(n, np.nan), x2=np.full(n, np.nan), fx=np.full(m, np.nan), fx1=np.full(m, np.nan))
    xl = x.copy()
    lkw = {k: v for k, v in kw.items()}
    rl = lit.finite_difference_jacobian(J, f, xl, cache_l, None if f_in is None else f_in.copy(), fdtype=fdtype,
                                        colorvec=cv, sparsity=sparsity, **lkw)
    if isinstance(J, lit.CSC):
        Jl = J.nzval
    elif isinstance(J, lit.Banded):
        Jl = J.data.reshape(-1, order="F")
    else:
        Jl = J.reshape(-1, order="F")

    # ---- the C oracle, once with its own step sizes and once with the literal's
    P = {"csc_same": lambda: oracle.Problem.csc_same(m, n, colptr, rowval),
         "csc_to_dense": lambda: oracle.Problem.csc_to_dense(m, n, colptr, rowval),
         "proto_to_dense": lambda: oracle.Problem.coo_to_dense(m, n, *oracle.findstructralnz_dense(D.astype(np.float64))),
         "banded": lambda: oracle.Problem.banded(m, n, l, u),
         "banded_to_dense": lambda: oracle.Problem.banded_to_dense(m, n, l, u),
         "dense_cols": lambda: oracle.Problem.dense(m, n)}[kind]()
    okw = dict(fdtype=FD[fdtype], colorvec=None if kind == "dense_cols" else cv, f_in=f_in, **kw)
    Jo = np.full(Jl.size, np.nan)
    ro = oracle.jacobian(P, Jo, f, x.copy(), **okw)
    assert ro["fcalls"] == rl["fcalls"]
    # both restatements evaluate norm as the reference does (generic_norm2 / OpenBLAS dnrm2): same step sizes, same J
    assert_same_bits(ro["eps"], rl["eps"], f"{kind} {fdtype} seed {seed}", allow_nan=False)
    assert_same_bits(Jo, Jl, f"{kind} {fdtype} seed {seed}")
    Jo2 = np.full(Jl.size, np.nan)
    cache_o = dict(x1=np.full(n, np.nan), x2=np.full(n, np.nan), fx=np.full(m, np.nan), fx1=np.full(m, np.nan))
    oracle.jacobian(P, Jo2, f, x.copy(), eps_override=None if kind == "dense_cols" else rl["eps"], cache=cache_o, **okw)
    assert_same_bits(Jo2, Jl, f"{kind} {fdtype} seed {seed}")
    assert np.array_equal(xl, x) or fdtype == "central"       # forward never touches x
    np.testing.assert_allclose(xl, x, rtol=0, atol=1e-12)     # central: restored up to the reference's own drift
    assert_same_bits(cache_o["x1"], cache_l["x1"], allow_nan=False)            # (x1 + eps) - eps drift, same end state


@pytest.mark.parametrize("seed", range(30))
@pytest.mark.parametrize("kind", KINDS)
def test_oracle_complex_step_matches_literal_transcription(oracle, kind, seed):
    # jacobians.jl:623-648: no step-size reduction involved (epsilon = eps(Float64)), so everything is bit for bit
    rng = np.random.default_rng(77000 + 1000 * seed + KINDS.index(kind))
    m, n, l, u, D, f = _problem(rng, kind)
    x = rng.uniform(-2, 2, n)
    if kind == "dense_cols":
        cv = np.arange(1, n + 1, dtype=np.int64)
    else:
        cv = rng.integers(0 if rng.random() < 0.3 else 1, int(rng.integers(1, 7)) + 1, n).astype(np.int64)
        if cv.max() < 1:
            cv[0] = 1
    A = sps.csc_matrix(D)
    A.sort_indices()
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    if kind == "csc_same":
        J = lit.CSC(m, n, colptr, rowval, np.full(A.nnz, np.nan)); sparsity = J
        P = oracle.Problem.csc_same(m, n, colptr, rowval)
    elif kind == "csc_to_dense":
        J = np.full((m, n), np.nan); sparsity = lit.CSC(m, n, colptr, rowval)
        P = oracle.Problem.csc_to_dense(m, n, colptr, rowval)
    elif kind == "proto_to_dense":
        J = np.full((m, n), np.nan); sparsity = D.astype(np.float64)
        P = oracle.Problem.coo_to_dense(m, n, *oracle.findstructralnz_dense(D.astype(np.float64)))
    elif kind == "banded":
        J = lit.Banded(m, n, l, u, np.full((l + u + 1, n), np.nan)); sparsity = J
        P = oracle.Problem.banded(m, n, l, u)
    elif kind == "banded_to_dense":
        J = np.full((m, n), np.nan); sparsity = lit.Banded(m, n, l, u)
        P = oracle.Problem.banded_to_dense(m, n, l, u)
    else:
        J = np.full((m, n), np.nan); sparsity = None
        P = oracle.Problem.dense(m, n)
    cache = dict(x1=np.zeros(n, np.complex128), fx=np.zeros(m, np.complex128))
    rl = lit.finite_difference_jacobian_complex(J, f, x.copy(), cache, colorvec=cv, sparsity=sparsity)
    Jl = J.nzval if isinstance(J, lit.CSC) else (J.data if isinstance(J, lit.Banded) else J).reshape(-1, order="F")
    Jo = np.full(Jl.size, np.nan)
    ro = oracle.jacobian_complex(P, Jo, f, x.copy(), colorvec=None if kind == "dense_cols" else cv)
    assert ro["fcalls"] == rl["fcalls"]
    assert_same_bits(Jo, Jl, f"{kind} seed {seed}")


@pytest.mark.parametrize("seed", range(60))
def test_oracle_jvp_matches_literal_transcription(oracle, seed):
    # src/jvp.jl:238-274; the dot product's reduction order differs (eps to 1e-14), so J-values are compared with the
    # literal's eps fed to the oracle
    rng = np.random.default_rng(55000 + seed)
    m, n, _, _, _, f = _problem(rng, "csc_same")
    x, v = rng.uniform(-2, 2, n), rng.uniform(-1, 1, n)
    fdtype = "forward" if rng.random() < 0.5 else "central"
    kw = {}
    if rng.random() < 0.3:
        kw["relstep"] = float(10 ** rng.uniform(-9, -5))
    if rng.random() < 0.3:
        kw["absstep"] = float(10 ** rng.uniform(-10, -6))
    if fdtype == "forward" and rng.random() < 0.3:
        kw["dir"] = -1.0
    f_in = None
    if fdtype == "forward" and rng.random() < 0.3:
        f_in = np.zeros(m)
        f(f_in, x)
    out = np.full(m, np.nan)
    cache = dict(x1=np.full(n, np.nan), fx1=np.full(m, np.nan))
    rl = lit.finite_difference_jvp(out, f, x.copy(), v.copy(), cache, None if f_in is None else f_in.copy(), fdtype=fdtype, **kw)
    ro = oracle.jvp(f, x.copy(), v.copy(), m, fdtype=FD[fdtype], f_in=f_in, **kw)
    assert ro["fcalls"] == rl["fcalls"]
    np.testing.assert_allclose(ro["eps"], rl["eps"], rtol=1e-14, atol=0)
    ro2 = oracle.jvp(f, x.copy(), v.copy(), m, fdtype=FD[fdtype], f_in=f_in, eps_override=rl["eps"], **kw)
    assert_same_bits(ro2["jvp"], out, allow_nan=False)
    assert_same_bits(ro2["x1"][:n], cache["x1"], allow_nan=False)               # cache.x1 ends as x + eps*v


@pytest.mark.parametrize("seed", range(40))
@pytest.mark.parametrize("kind", ["csc_same", "banded", "dense_cols"])
def test_oracle_cacheless_matches_literal_transcription(oracle, kind, seed):
    # jacobians.jl:446-471: the method without a cache (sparsity defaults to J when J has structure)
    rng = np.random.default_rng(91000 + 1000 * seed + KINDS.index(kind))
    m, n, l, u, D, f = _problem(rng, kind)
    fdtype = "forward" if rng.random() < 0.5 else "central"
    x = rng.uniform(-2, 2, n)
    if kind == "dense_cols":
        cv = None
    else:
        cv = rng.integers(1, int(rng.integers(1, 7)) + 1, n).astype(np.int64)
    A = sps.csc_matrix(D)
    A.sort_indices()
    colptr, rowval = A.indptr.astype(np.int64) + 1, A.indices.astype(np.int64) + 1
    if kind == "csc_same":
        J = lit.CSC(m, n, colptr, rowval, np.full(A.nnz, np.nan))
        P = oracle.Problem.csc_same(m, n, colptr, rowval)
    elif kind == "banded":
        J = lit.Banded(m, n, l, u, np.full((l + u + 1, n), np.nan))
        P = oracle.Problem.banded(m, n, l, u)
    else:
        J = np.full((m, n), np.nan)
        P = oracle.Problem.dense(m, n)
    xl = x.copy()
    rl = lit.finite_difference_jacobian_cacheless(J, f, xl, fdtype, colorvec=cv)
    Jl = J.nzval if isinstance(J, lit.CSC) else (J.data if isinstance(J, lit.Banded) else J).reshape(-1, order="F")
    Jo = np.full(Jl.size, np.nan)
    ro = oracle.jacobian(P, Jo, f, x.copy(), fdtype=FD[fdtype], colorvec=cv, cacheless=True,
                         eps_override=None if kind == "dense_cols" else rl["eps"])
    assert ro["fcalls"] == rl["fcalls"] == ((1 if fdtype == "forward" else 0) +
                                            (n if cv is None else int(cv.max())) * (1 if fdtype == "forward" else 2))
    assert_same_bits(Jo, Jl, f"{kind} {fdtype} seed {seed}")


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_oracle_dense_branch_with_colorvec_matches_literal(oracle, fdtype, seed):
    """sparsity === nothing WITH a caller-supplied colorvec, as jacobians.jl:547-557 / :589-598 are written: the loop runs
    color_i in 1:maximum(colorvec), perturbs component color_i, writes J[:, color_i]; no fill_matrix!, later columns keep
    their contents (VERDICT r1 missing #6; the GPU path reproduces it through fdb_plan_create_dense_colorvec)."""
    rng = np.random.default_rng(7000 + seed)
    m, n = int(rng.integers(2, 9)), int(rng.integers(3, 10))
    maxc = int(rng.integers(1, n + 1))
    cv = rng.integers(1, maxc + 1, size=n).astype(np.int64)
    cv[int(rng.integers(0, n))] = maxc
    W = rng.normal(size=(m, n))

    def f(fx, x):
        fx[:] = np.sin(W @ x) + 0.5 * (W @ x) ** 2

    x = rng.normal(size=n) + 1.5
    Jl = np.full((m, n), -7.5)
    cache_l = dict(x1=np.full(n, np.nan), x2=np.full(n, np.nan), fx=np.full(m, np.nan), fx1=np.full(m, np.nan))
    rl = lit.finite_difference_jacobian(Jl, f, x.copy(), cache_l, None, fdtype=fdtype, colorvec=cv, sparsity=None)
    Jo = np.full(m * n, -7.5)
    ro = oracle.jacobian(oracle.Problem.dense(m, n), Jo, f, x.copy(), fdtype=FD[fdtype], colorvec=cv)
    assert ro["fcalls"] == rl["fcalls"] == (maxc + 1 if fdtype == "forward" else 2 * maxc)
    assert_same_bits(Jo.reshape(m, n, order="F"), Jl, allow_nan=False)
    assert (Jl[:, maxc:] == -7.5).all() and not (Jl[:, :maxc] == -7.5).any()
