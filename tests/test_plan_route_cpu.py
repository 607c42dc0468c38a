"""One plan-creator choice for one device and for a device group (no GPU): make_plan and GroupJacobian ask the C ABI for
the same creator with the same arguments for every (J, sparsity, colorvec) the mirror routes, apart from the group's two
stated differences (no COO route; a dense target ignores colorvec), and the out-of-place builders of
finite_difference_jacobian and GroupJacobianOOP do the same.  The library is replaced by a fake that records the symbol
asked for and its arguments."""
import contextlib
import ctypes as C

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


@pytest.fixture(scope="module")
def fdist(pkg):
    from finitediff_jl_b200 import distributed
    return distributed


class FakeLib:
    """Records every fdb_*create* call as (symbol, arguments after the handle and, for a group, its device list, without
    the opts; the opts).  The block list of a block-banded plan is read while the call runs (its array is made per call)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            if "create" in name:
                group = name.startswith("fdb_group_create_")
                mid = list(args[3:-1] if group else args[1:-1])
                if name.endswith("block_banded"):
                    mid[1] = tuple((C.c_int64 * mid[0]).from_address(mid[1])) if mid[1] else None
                o = args[-1]._obj
                self.calls.append((name, tuple(mid), (o.fdtype, o.device, o.max_batch, o.use_graph)))
            return 0
        return fn


@pytest.fixture
def fake(pkg, monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(pkg._lib, "lib", lambda: lib)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    return lib


def _t64(a):
    return torch.as_tensor(np.asarray(a, dtype=np.int64))


def _csc(pkg, n, colptr=None, rowval=None):
    """The tridiagonal pattern of n columns as a CPU SparseMatrixCSC (own index arrays unless given)."""
    import scipy.sparse as sps
    A = sps.diags([np.ones(n - 1), np.ones(n), np.ones(n - 1)], [-1, 0, 1], format="csc")
    A.sort_indices()
    cp = _t64(A.indptr + 1) if colptr is None else colptr
    rv = _t64(A.indices + 1) if rowval is None else rowval
    return pkg.SparseMatrixCSC(n, n, cp, rv, torch.zeros(A.nnz, dtype=torch.float64))


def _routed_cases(pkg):
    """(name, J, sparsity, colorvec, creator kind): every pair that has a plan creator for one device."""
    n = 6
    dense = pkg.zeros_colmajor(n, n, "cpu")
    cv = np.array([1, 2, 3, 1, 2, 3], dtype=np.int64)
    S = _csc(pkg, n)
    B = pkg.BandedMatrix(n, n, 1, 1, device="cpu")
    D, BU, BL = pkg.Diagonal(n, device="cpu"), pkg.Bidiagonal(n, "U", device="cpu"), pkg.Bidiagonal(n, "L", device="cpu")
    T, Sym = pkg.Tridiagonal(n, device="cpu"), pkg.SymTridiagonal(n)
    BB = pkg.BandedBlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 2), (0, 3), device="cpu")
    BBs = pkg.BandedBlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 2), (0, 3), device="cpu")
    BBd = pkg.BlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 1), device="cpu")
    R = pkg.BandedBlockBandedMatrix([3, 4, 2], [2, 5, 2], (1, 1), (1, 1), device="cpu")
    Ng = pkg.BandedBlockBandedMatrix([3, 3], [3, 3], (-1, 1), (1, 1), data=torch.zeros(1), device="cpu")
    proto = torch.eye(n, dtype=torch.float64)
    return [
        ("dense", dense, None, None, "dense"),
        ("dense identity colorvec", dense, None, np.arange(1, n + 1), "dense"),
        ("dense colorvec", dense, None, cv, "dense_colorvec"),
        ("rectangular dense", pkg.zeros_colmajor(4, n, "cpu"), None, None, "dense"),
        ("csc same pattern", S, S, cv, "csc"),
        ("csc own index arrays", _csc(pkg, n), S, cv, "csc"),
        ("csc shared index arrays", _csc(pkg, n, S.colptr, S.rowval), S, None, "csc"),
        ("csc into dense", dense, S, cv, "csc"),
        ("banded", B, B, cv, "banded"),
        ("banded into dense", dense, B, None, "banded"),
        ("diagonal", D, pkg.Diagonal(n, device="cpu"), None, "banded"),
        ("bidiagonal U", BU, BU, cv, "banded"),
        ("bidiagonal L", BL, pkg.Bidiagonal(n, ":L", device="cpu"), None, "banded"),
        ("diagonal into dense", dense, D, None, "banded"),
        ("bidiagonal U into dense", dense, BU, None, "banded"),
        ("bidiagonal L into dense", dense, BL, None, "banded"),
        ("symtridiagonal into dense", dense, Sym, cv, "banded"),
        ("symtridiagonal n = 1", pkg.SymTridiagonal(1, buf=torch.zeros(1, dtype=torch.float64)), pkg.SymTridiagonal(1),
         None, "banded"),
        ("block-banded", BB, BB, None, "block_banded"),
        ("block-banded other object", BB, BBs, BB.matrix_colors(), "block_banded"),
        ("block-banded dense blocks", BBd, BBd, None, "block_banded"),
        ("tridiagonal", T, T, None, "coo"),
        ("tridiagonal into dense", dense, T, None, "coo"),
        ("tridiagonal with symtridiagonal sparsity", T, Sym, None, "coo"),
        ("block-banded into dense", pkg.zeros_colmajor(9, 9, "cpu"), BB, None, "coo"),
        ("block-banded rectangular blocks", R, R, None, "coo"),
        ("block-banded negative bandwidth", Ng, Ng, None, "coo"),
        ("dense prototype", dense, proto, None, "coo"),
    ]


def _make(pkg, api, fdist, fake, J, sp, cv, fdtype="forward", **kw):
    """The creator calls of make_plan and of GroupJacobian on the same inputs (or the exception each raised)."""
    out = []
    for build in (lambda: api.make_plan(J, sp, cv, fdtype, J.shape[1], 0, **kw),
                  lambda: fdist.GroupJacobian(J, cv, fdtype, [0, 0], sparsity=sp, **kw)):
        fake.calls.clear()
        try:
            build()
            out.append(list(fake.calls))
        except (TypeError, ValueError) as e:
            out.append(type(e))
    return out


def test_single_and_group_request_the_same_creator(pkg, api, fdist, fake):
    for name, J, sp, cv, kind in _routed_cases(pkg):
        (single,), group = _make(pkg, api, fdist, fake, J, sp, cv, max_batch=7)
        sym, args, opts = single
        assert sym == f"fdb_plan_create_{kind}", name
        assert opts == (0, 0, 7, 0), name
        if kind == "coo":
            assert group is TypeError, name                         # the group has no COO route
        elif kind == "dense_colorvec":
            # a dense group splits the columns 1:n whatever colorvec says: fdb_group_create_dense on (m, n, ldJ)
            assert group == [("fdb_group_create_dense", args[:3], opts)], name
        else:
            assert group == [(f"fdb_group_create_{kind}", args, opts)], name


def test_malformed_pairs_raise_the_same_for_one_device_and_a_group(pkg, api, fdist, fake):
    n = 6
    dense = pkg.zeros_colmajor(n, n, "cpu")
    S = _csc(pkg, n)
    B = pkg.BandedMatrix(n, n, 1, 1, device="cpu")
    D, BU, BL = pkg.Diagonal(n, device="cpu"), pkg.Bidiagonal(n, "U", device="cpu"), pkg.Bidiagonal(n, "L", device="cpu")
    T, Sym = pkg.Tridiagonal(n, device="cpu"), pkg.SymTridiagonal(n)
    BB = pkg.BandedBlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 2), (0, 3), device="cpu")
    BB2 = pkg.BandedBlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 1), (1, 1), device="cpu")
    cases = [
        # newly refused by the group: it used to build these
        (pkg.zeros_colmajor(n, n + 1, "cpu"), S, ValueError),           # size(J) != size(sparsity), CSC
        (pkg.BandedMatrix(n, n, 2, 1, device="cpu"), B, ValueError),    # J and sparsity bandwidths differ
        # the group now raises make_plan's exception (it raised AttributeError or TypeError)
        (B, S, TypeError),                                              # a banded J for a CSC sparsity
        (S, B, TypeError),                                              # a CSC J for a banded sparsity
        (BB, BB2, ValueError),                                          # two block-banded structures
        # refused alike before
        (D, BU, TypeError), (BU, BL, ValueError), (D, T, TypeError), (T, D, TypeError), (BU, Sym, TypeError),
        (D, pkg.Diagonal(n + 1, device="cpu"), ValueError), (pkg.zeros_colmajor(n, n + 1, "cpu"), D, ValueError),
        (Sym, Sym, ValueError), (Sym, None, ValueError), (dense, object(), TypeError),
        (T, torch.eye(n, dtype=torch.float64), TypeError),
    ]
    for J, sp, exc in cases:
        assert _make(pkg, api, fdist, fake, J, sp, None) == [exc, exc], (type(J).__name__, type(sp).__name__)
        assert fake.calls == []


def _oop_cases(pkg):
    """(name, sparsity, jac_prototype, colorvec, m): every result kind, with and without a colouring."""
    n = 6
    S = _csc(pkg, n)
    cv = np.array([1, 2, 3, 1, 2, 3], dtype=np.int64)
    dense = pkg.zeros_colmajor(n, n, "cpu")
    return [
        ("raw", None, None, None, 4),
        ("raw colorvec", None, None, cv, 4),
        ("raw identity colorvec", None, None, range(1, n + 1), n),
        ("dense prototype", None, pkg.zeros_colmajor(4, n, "cpu"), cv, 4),
        ("sparse prototype", None, _csc(pkg, n), None, n),
        ("csc", S, None, cv, n),
        ("csc dense prototype", S, dense, cv, n),
        ("csc sparse prototype", S, _csc(pkg, n), None, n),
        ("csc m = 0", pkg.SparseMatrixCSC(0, n, _t64(np.ones(n + 1)), _t64([]), None), None, None, 0),
    ]


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_out_of_place_builders_request_the_same_creator(pkg, api, fdist, fake, fdtype):
    n = 6
    for name, sp, proto, cv, m in _oop_cases(pkg):
        kind, pm, pn = api._oop_kind(sp, proto)
        cache = object.__new__(api.JacobianCache)
        cache.fdtype, cache._plans = fdtype, {}
        cache._plan_kw = dict(max_batch=7, use_graph=True, partition=1)
        fake.calls.clear()
        plan = cache._oop_plan_for(kind, sp, cv, pn, m, n, torch.device("cuda", 0))
        assert cache._oop_plan_for(kind, sp, cv, pn, m, n, torch.device("cuda", 0)) is plan   # cached
        (single,) = fake.calls
        fake.calls.clear()
        fdist.GroupJacobianOOP([0, 0], fdtype, colorvec=cv, sparsity=sp, jac_prototype=proto, max_batch=7,
                               use_graph=True, partition=1)._build(m, n)
        (group,) = fake.calls
        suffix = "csc" if sp is not None else "dense"
        assert single[0] == f"fdb_oop_plan_create_{suffix}" and group[0] == f"fdb_group_create_oop_{suffix}", name
        assert single[1] == group[1], name
        assert single[1][-2:] == (kind, max(m, 1)), name
        # one device takes max_batch and scratch_bytes of the plan keywords, a group all of them
        code = 0 if fdtype == "forward" else 1
        assert single[2] == (code, 0, 7, 0) and group[2] == (code, 0, 7, 1), name
