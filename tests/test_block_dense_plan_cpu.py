"""Host side of the block-dense plan (no GPU): BlockBandedMatrices' storage of a BlockBandedMatrix as the mirror's
BlockSkylineMatrix lays it out, checked against a literal enumeration of the hook
ext/FiniteDiffBlockBandedMatricesExt.jl:44-68 and that package's slot formula; its colouring; which creator the mirror
routes it to; and the refusals of fdb_plan_create_block_dense, which come before any device work or f call."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch


@pytest.fixture(scope="module")
def pkg():
    import _bootstrap
    return _bootstrap.load_package()


@pytest.fixture(scope="module")
def api(pkg):
    from finitediff_jl_b200 import api
    return api


def _hook_entries(rb, l, u):
    """(rows, cols, slots), 1-based, in the hook's order: for J, for j in 1:n, for K in blockcolrange(J), for k in
    1:size(K) — with the slot start_J + (j-1) h_J + rowoff_J(K) + k of the BlockSkylineMatrix layout."""
    N = len(rb)
    off = [0]
    for b in rb:
        off.append(off[-1] + b)
    rows, cols, slots = [], [], []
    start = 0
    for J in range(1, N + 1):
        krange = range(max(1, J - u), min(N, J + l) + 1)
        h = sum(rb[K - 1] for K in krange)
        for j in range(1, rb[J - 1] + 1):
            rowoff = 0
            for K in krange:
                for k in range(1, rb[K - 1] + 1):
                    rows.append(off[K - 1] + k)
                    cols.append(off[J - 1] + j)
                    slots.append(start + (j - 1) * h + rowoff + k)
                rowoff += rb[K - 1]
        start += h * rb[J - 1]
    a = lambda v: np.asarray(v, dtype=np.int64)
    return a(rows), a(cols), a(slots), start


def _cases():
    rng = np.random.default_rng(7)
    cases = [([], 1, 1), ([5], 0, 0), ([5], 2, 3), ([1, 1, 1, 1], 0, 0), ([3, 3, 3], 0, 1), ([2, 4, 1], 5, 7),
             ([4] * 6, 1, 1), ([1] * 7, 2, 1)]
    for _ in range(30):
        N = int(rng.integers(1, 11))
        rb = [int(v) for v in rng.integers(0 if rng.random() < 0.2 else 1, 8, N)]     # some with empty blocks
        l, u = (int(v) for v in rng.integers(0, N + 2, 2))                             # bandwidths >= nblocks too
        cases.append((rb, l, u))
    return cases


CASES = _cases()


@pytest.mark.parametrize("case", CASES, ids=[f"c{i}" for i in range(len(CASES))])
def test_entry_set_and_slots_are_the_hook(pkg, case):
    rb, l, u = case
    B = pkg.BlockSkylineMatrix(rb, rb, (l, u), device="cpu")
    rows, cols, slots, jlen = _hook_entries(rb, l, u)
    r2, c2, s2 = B.findstructralnz()
    assert B.j_len == jlen == B.data.numel()
    assert np.array_equal(r2, rows) and np.array_equal(c2, cols) and np.array_equal(s2, slots)
    assert np.array_equal(np.sort(slots), np.arange(1, jlen + 1))                # every slot is one structural entry
    assert B.shape == (sum(rb), sum(rb))
    # to_dense places slot values at their (row, column)
    B.data.copy_(torch.arange(1, jlen + 1, dtype=torch.float64))
    D = B.to_dense()
    assert np.array_equal(D[rows - 1, cols - 1], slots.astype(np.float64))
    assert np.count_nonzero(D) == jlen


@pytest.mark.parametrize("case", CASES, ids=[f"c{i}" for i in range(len(CASES))])
def test_matrix_colors_is_valid(pkg, case):
    rb, l, u = case
    B = pkg.BlockSkylineMatrix(rb, rb, (l, u), device="cpu")
    cv = B.matrix_colors()
    assert len(cv) == B.n and (B.n == 0 or cv.min() >= 1)
    rows, cols, _ = B.findstructralnz()
    if B.n == 0:
        return
    # distance-2 valid: no row holds two columns of one colour (the compressed f! outputs stay separable)
    A = sp.csr_matrix((np.ones(len(rows)), (rows - 1, cols - 1)), shape=(B.m, B.n))
    Q = sp.csr_matrix((np.ones(B.n), (np.arange(B.n), cv - 1)), shape=(B.n, int(cv.max())))
    assert (A @ Q).max() <= 1


@pytest.mark.parametrize("b,N,l,u", [(1, 9, 1, 1), (3, 8, 1, 1), (8, 12, 1, 1), (4, 10, 0, 2), (5, 7, 3, 0)])
def test_matrix_colors_count_uniform(pkg, b, N, l, u):
    B = pkg.BlockSkylineMatrix([b] * N, [b] * N, (l, u), device="cpu")
    cv = B.matrix_colors()
    assert cv.max() == (l + u + 1) * b
    c = np.arange(B.n)
    assert np.array_equal(cv - 1, ((c // b) % (l + u + 1)) * b + c % b)
    # the padded mirror of the same structure cycles its colours over 2b-1 sub-band slots: maximum(colorvec), the
    # colour loop's length, is (l+u)(2b-1) + b
    P = pkg.BlockBandedMatrix([b] * N, [b] * N, (l, u), device="cpu")
    assert P.matrix_colors().max() == (l + u) * (2 * b - 1) + b


def test_routing(pkg, api):
    L = pkg._lib
    B = pkg.BlockSkylineMatrix([3, 4, 2], [3, 4, 2], (1, 2), device="cpu")
    kind, args, keep = api._plan_route(B, B, None)
    assert kind == "block_dense"
    nb, ptr, l, u, ldata, cv = args
    assert (nb, l, u, ldata, cv) == (3, 1, 2, B.j_len, None)
    assert np.frombuffer((C.c_int64 * 3).from_address(ptr), dtype=np.int64).tolist() == [3, 4, 2]
    # as its own sparsity: the cache-less entry and GroupJacobian take J as the sparsity
    assert api._has_sparsestruct(B)
    assert api._shape_of(B) == (9, 9)
    assert api._j_values(B) is B.data
    # another object of the same structure
    S = pkg.BlockSkylineMatrix([3, 4, 2], [3, 4, 2], (1, 2), device="cpu")
    assert api._plan_route(B, S, None)[0] == "block_dense"
    assert api._j_key(B) == api._sp_key(S)
    # a dense J with this sparsity: the slot route of the other block types, entries by (row, column)
    Jd = torch.zeros(9, 9, dtype=torch.float64).t()                      # column-major
    kind, args, keep = api._plan_route(Jd, B, None)
    assert kind == "coo"
    m, n, nnz, _, _, jkind, slot_ptr, ld, _ = args
    assert (m, n, nnz, jkind, slot_ptr, ld) == (9, 9, B.j_len, L.FDB_J_DENSE, None, 9)
    # a different structure, or another J type
    D = pkg.BlockSkylineMatrix([3, 4, 2], [3, 4, 2], (1, 1), device="cpu")
    with pytest.raises(ValueError):
        api._plan_route(D, B, None)
    with pytest.raises(TypeError):
        api._plan_route(pkg.BandedBlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 2), (1, 1), device="cpu"), B, None)
    # the existing types keep their routes
    BB = pkg.BlockBandedMatrix([3, 4, 2], [3, 4, 2], (1, 1), device="cpu")
    assert api._plan_route(BB, BB, None)[0] == "block_banded"


def test_rectangular_blocks_refused(pkg, api):
    R = pkg.BlockSkylineMatrix([3, 4, 2], [2, 5, 2], (1, 1), device="cpu")
    for J in (R, torch.zeros(9, 9, dtype=torch.float64).t()):
        with pytest.raises(pkg._lib.FdbError) as e:
            api._plan_route(J, R, None)
        assert e.value.status == pkg._lib.FDB_ERR_INVALID


def _create(lib, nblocks, blocks, l, u, ldata):
    h = C.c_void_p()
    st = lib.fdb_plan_create_block_dense(C.byref(h), nblocks, blocks, l, u, ldata, None, None)
    return st, h, lib.fdb_last_error().decode()


def test_creator_refusals(pkg):
    L = pkg._lib
    lib = L.lib()
    blocks = np.array([2, 3, 2], dtype=np.int64)
    bp = blocks.ctypes.data
    jlen = 5 * 2 + 7 * 3 + 5 * 2                                       # l = u = 1: slab heights 5, 7, 5
    cases = [
        ((-1, bp, 1, 1, jlen), "nblocks"),
        ((3, None, 1, 1, jlen), "blocks is NULL"),
        ((3, bp, -1, 1, jlen), "negative block bandwidths"),
        ((3, bp, 1, -2, jlen), "negative block bandwidths"),
        ((3, bp, 1, 1, jlen - 1), "ldata"),
    ]
    neg = np.array([2, -3, 2], dtype=np.int64)
    cases.append(((3, neg.ctypes.data, 1, 1, jlen), "negative size"))
    for args, text in cases:
        st, h, msg = _create(lib, *args)
        assert st == L.FDB_ERR_INVALID, (args, st, msg)
        assert text in msg, (args, msg)
        assert not h.value
    # a NULL plan pointer
    assert lib.fdb_plan_create_block_dense(None, 3, bp, 1, 1, jlen, None, None) == L.FDB_ERR_INVALID
    # a block column of more than 2^32 slots
    big = np.array([70000], dtype=np.int64)
    st, h, msg = _create(lib, 1, big.ctypes.data, 0, 0, 70000 * 70000)
    assert st == L.FDB_ERR_UNSUPPORTED and "2^32" in msg
    # the group creator refuses the same way
    hg = C.c_void_p()
    devs = (C.c_int * 1)(0)
    assert lib.fdb_group_create_block_dense(C.byref(hg), 1, devs, 3, bp, 1, 1, jlen - 1, None, None) != L.FDB_OK
