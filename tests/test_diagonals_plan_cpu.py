"""Host side of the diagonal-storage J kind (FDB_J_DIAGONALS, no GPU): the closed form the scatter kernel uses (slot ->
diagonal -> (row, column)), restated here and checked against each LinearAlgebra mirror's findstructralnz and against the
in-matrix band (l, u); and the routing of every (J, sparsity) pair in make_plan."""
import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def pkg():
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def api(pkg):
    from finitediff_jl_b200 import api
    return api


def _closed_form(n, l, u):
    """(rows, cols, slots) 1-based, walking the packed buffer in storage order as diff_scatter_diagonals does."""
    total = (l + u + 1) * n - l - u if n > 0 else 0
    sub_end = l * (n - 1)
    main_end = sub_end + n
    s = np.arange(total, dtype=np.int64)
    r = np.empty_like(s)
    c = np.empty_like(s)
    sub, main = s < sub_end, (s >= sub_end) & (s < main_end)
    sup = ~(sub | main)
    c[sub], r[sub] = s[sub], s[sub] + 1
    c[main] = r[main] = s[main] - sub_end
    r[sup] = s[sup] - main_end
    c[sup] = r[sup] + 1
    return r + 1, c + 1, s + 1


def _band_set(n, l, u):
    return {(r, c) for c in range(1, n + 1) for r in range(max(1, c - u), min(n, c + l) + 1)}


def _types(pkg):
    return {
        "diagonal": (lambda n: pkg.Diagonal(n, device="cpu"), 0, 0),
        "bidiagonal_U": (lambda n: pkg.Bidiagonal(n, "U", device="cpu"), 0, 1),
        "bidiagonal_L": (lambda n: pkg.Bidiagonal(n, ":L", device="cpu"), 1, 0),
        "tridiagonal": (lambda n: pkg.Tridiagonal(n, device="cpu"), 1, 1),
        "symtridiagonal": (lambda n: pkg.SymTridiagonal(n), 1, 1),
    }


SIZES = [0, 1, 2, 3] + [int(v) for v in np.random.default_rng(7).integers(4, 5001, 30)]


@pytest.mark.parametrize("kind", ["diagonal", "bidiagonal_U", "bidiagonal_L", "tridiagonal", "symtridiagonal"])
def test_closed_form_is_the_entry_set(pkg, kind):
    make, l, u = _types(pkg)[kind]
    for n in SIZES:
        A = make(n)
        if kind != "tridiagonal":
            assert (A.l, A.u) == (l, u)
        rows, cols, slots = A.findstructralnz()
        r2, c2, s2 = _closed_form(n, l, u)
        got = set(zip(rows.tolist(), cols.tolist(), slots.tolist()))
        assert len(got) == len(rows), (kind, n)
        assert got == set(zip(r2.tolist(), c2.tolist(), s2.tolist())), (kind, n)
        if n <= 600:
            assert {(r, c) for r, c, _ in got} == _band_set(n, l, u), (kind, n)
        else:
            # every pair in the band and distinct: with the count that is the band
            assert np.all((rows - cols <= l) & (cols - rows <= u) & (rows >= 1) & (rows <= n)), (kind, n)
            assert len(got) == len(_closed_form(n, l, u)[0]) == (l + u + 1) * n - l - u, (kind, n)
        if kind != "symtridiagonal":
            assert len(A.buf) == len(slots), (kind, n)


def test_buffer_views(pkg):
    n = 5
    B = pkg.Bidiagonal(n, "U", buf=torch.arange(1.0, 2 * n, dtype=torch.float64))
    assert B.dv.tolist() == [1, 2, 3, 4, 5] and B.ev.tolist() == [6, 7, 8, 9]
    Bl = pkg.Bidiagonal(n, "L", buf=torch.arange(1.0, 2 * n, dtype=torch.float64))
    assert Bl.ev.tolist() == [1, 2, 3, 4] and Bl.dv.tolist() == [5, 6, 7, 8, 9]
    want = np.diag([5.0, 6, 7, 8, 9]) + np.diag([1.0, 2, 3, 4], -1)
    assert np.array_equal(Bl.to_dense(), want)
    # the packed slot of entry (r, c) holds the value to_dense shows there
    for A in (B, Bl, pkg.Diagonal(n, buf=torch.arange(1.0, n + 1, dtype=torch.float64))):
        rows, cols, slots = A.findstructralnz()
        d = A.to_dense()
        assert all(d[r - 1, c - 1] == A.buf[s - 1].item() for r, c, s in zip(rows, cols, slots))
    with pytest.raises(ValueError):
        pkg.Bidiagonal(3, "X", device="cpu")


def test_routing(pkg, api):
    L = pkg._lib
    n = 6
    D, D2 = pkg.Diagonal(n, device="cpu"), pkg.Diagonal(n, device="cpu")
    BU, BL = pkg.Bidiagonal(n, "U", device="cpu"), pkg.Bidiagonal(n, "L", device="cpu")
    T, S = pkg.Tridiagonal(n, device="cpu"), pkg.SymTridiagonal(n)
    dense = pkg.zeros_colmajor(n, n, "cpu")
    ld = api._dense_ld(dense)[2]
    # packed diagonal storage
    assert api._diagonals_route(D, D2) == (n, n, 0, 0, L.FDB_J_DIAGONALS, n)
    assert api._diagonals_route(BU, BU) == (n, n, 0, 1, L.FDB_J_DIAGONALS, 2 * n - 1)
    assert api._diagonals_route(BL, pkg.Bidiagonal(n, ":L", device="cpu")) == (n, n, 1, 0, L.FDB_J_DIAGONALS, 2 * n - 1)
    # dense J: the banded plan into the matrix, with the type's band
    assert api._diagonals_route(dense, D) == (n, n, 0, 0, L.FDB_J_DENSE, ld)
    assert api._diagonals_route(dense, BU) == (n, n, 0, 1, L.FDB_J_DENSE, ld)
    assert api._diagonals_route(dense, BL) == (n, n, 1, 0, L.FDB_J_DENSE, ld)
    assert api._diagonals_route(dense, S) == (n, n, 1, 1, L.FDB_J_DENSE, ld)
    # unchanged routes: a Tridiagonal sparsity (COO slots / COO dense), a Tridiagonal J with a SymTridiagonal sparsity
    assert api._diagonals_route(T, T) is None
    assert api._diagonals_route(dense, T) is None
    assert api._diagonals_route(T, S) is None
    # mixed pairs: TypeError before any plan is built (device 0 is only named, never touched, before the raise)
    for J, sp in ((D, BU), (D, T), (D, S), (BU, D), (BU, T), (BU, S), (T, D), (T, BU), (T, BL)):
        with pytest.raises(TypeError):
            api.make_plan(J, sp, None, "forward", n, 0)
    # same type, other structure
    with pytest.raises(ValueError):
        api._diagonals_route(BU, BL)
    with pytest.raises(ValueError):
        api._diagonals_route(D, pkg.Diagonal(n + 1, device="cpu"))
    with pytest.raises(ValueError):
        api._diagonals_route(pkg.zeros_colmajor(n, n + 1, "cpu"), D)
    # SymTridiagonal as J: refused (n >= 2) before anything is built, with any sparsity
    for sp in (S, D, T, None):
        with pytest.raises(ValueError, match="ArgumentError"):
            api.make_plan(S, sp, None, "forward", n, 0)
    # ... and a valid target for n <= 1, where its structure is the main diagonal
    S1 = pkg.SymTridiagonal(1, buf=torch.zeros(1, dtype=torch.float64))
    assert api._diagonals_route(S1, pkg.SymTridiagonal(1)) == (1, 1, 0, 0, L.FDB_J_DIAGONALS, 1)
    # has_sparsestruct, keys and value buffers
    for A in (D, BU, S):
        assert api._has_sparsestruct(A)
    assert len({api._j_key(A) for A in (D, BU, BL, T, S)}) == 5
    assert api._j_values(BU) is BU.buf and api._shape_of(S) == (n, n)
