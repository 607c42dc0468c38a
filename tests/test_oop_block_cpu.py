"""Host side of the block out-of-place Jacobians (fdb_oop_plan_create_block_banded / _block_dense, no GPU): the closed
forms of their compaction (kernels_oop.cuh: bb_col_offset, block_band_col_counts, BlockBandForm, BlockDenseForm),
restated here and checked against a literal enumeration of the mirror's findstructralnz sorted into CSC order; and the
routing of every block sparsity with a SparseMatrixCSC prototype through finite_difference_jacobian and
GroupJacobianOOP, with the refusals that stay."""
import bisect
import contextlib

import numpy as np
import pytest
import torch

KTILE = 1024
KBDSTAGE = 256


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


# ---- the closed forms, as the kernels compute them (0-based) ----
def band_col_start(m, l, u, c):
    if m <= 0:
        return 0
    k = min(c, m + u)
    K = m - 1
    t = min(max(K - l + 1, 0), k)
    A = t * l + t * (t - 1) // 2 + (k - t) * K
    s = max(k - u - 1, 0)
    return k + A - s * (s + 1) // 2


def offsets(rb):
    return [0] + np.cumsum(rb, dtype=np.int64).tolist()


def brange(J, N, l, u):
    return max(0, J - u), min(N - 1, J + l)


def bb_col_offset(off, l, u, lam, mu, J, j):
    N = len(off) - 1
    K0, K1 = brange(J, N, l, u)
    return sum(band_col_start(off[K + 1] - off[K], lam, mu, j) for K in range(K0, K1 + 1))


def block_of(off, lo, hi, c):
    """bb_block_of: the largest J in [lo, hi] with off[J] <= c"""
    while lo < hi:
        mid = (lo + hi + 1) >> 1
        if off[mid] <= c:
            lo = mid
        else:
            hi = mid - 1
    return lo


column_of_start = block_of          # blk_column_of / bd_column_of: the same search over the block-column starts


class BlockBand:
    """BlockBandForm: the block-column starts from block_band_col_counts, the per-tile column table and the walk"""

    def __init__(self, rb, l, u, lam, mu):
        self.off, self.N, self.n = offsets(rb), len(rb), sum(rb)
        self.l, self.u, self.lam, self.mu, self.u_full = min(l, len(rb)), min(u, len(rb)), lam, mu, u
        self.w = (l + u + 1) * (lam + mu + 1)
        cnt = [bb_col_offset(self.off, self.l, self.u, lam, mu, J, self.off[J + 1] - self.off[J]) for J in range(self.N)]
        self.start = [0] + np.cumsum(cnt, dtype=np.int64).tolist()
        self.E = self.start[-1]

    def column_of(self, e):
        J = column_of_start(self.start, 0, self.N - 1, e)
        rel = e - self.start[J]
        lo, hi = 0, self.off[J + 1] - self.off[J] - 1
        while lo < hi:
            mid = (lo + hi + 1) >> 1
            if bb_col_offset(self.off, self.l, self.u, self.lam, self.mu, J, mid) <= rel:
                lo = mid
            else:
                hi = mid - 1
        return self.off[J] + lo, J

    def begin_tile(self, t0):
        self.c_lo, jlo = self.column_of(t0)
        c_hi, jhi = self.column_of(min(t0 + KTILE, self.E) - 1)
        self.nc = c_hi - self.c_lo + 1
        assert self.nc <= KTILE
        self.cs, self.cj = [], []
        for i in range(self.nc + 1):
            c = self.c_lo + i
            s, J = self.E, jhi
            if c < self.n:
                J = block_of(self.off, jlo, jhi, c) if i < self.nc else block_of(self.off, jhi, self.N - 1, c)
                s = self.start[J] + bb_col_offset(self.off, self.l, self.u, self.lam, self.mu, J, c - self.off[J])
            self.cs.append(s)
            self.cj.append(J)

    def locate(self, e):
        """(row, kCopy slot, block column, local column)"""
        i = bisect.bisect_right(self.cs[:self.nc], e) - 1
        c, J = self.c_lo + i, self.cj[i]
        j = c - self.off[J]
        q = e - self.cs[i]
        K0, K1 = brange(J, self.N, self.l, self.u)
        rlo = max(j - self.mu, 0)
        K = K0
        while True:
            mK = self.off[K + 1] - self.off[K]
            cnt = max(min(j + self.lam, mK - 1) - rlo + 1, 0)
            if q < cnt or K == K1:
                break
            q -= cnt
            K += 1
        src = c * self.w + (K - J + self.u_full) * (self.lam + self.mu + 1) + (self.mu + rlo + q - j)
        return self.off[K] + rlo + q, src, J, j

    def first_col(self, t0):
        return self.c_lo if self.cs[0] == t0 else self.c_lo + 1

    def col_start(self, c):
        i = c - self.c_lo
        return self.cs[i] if i <= self.nc else self.E


class BlockDense:
    """BlockDenseForm: the slab starts of the in-place plan, the staged block columns and (e - start_J) / h_J"""

    def __init__(self, rb, l, u):
        self.off, self.N, self.n = offsets(rb), len(rb), sum(rb)
        self.l, self.u = min(l, len(rb)), min(u, len(rb))
        self.start = [0]
        for J in range(self.N):
            self.start.append(self.start[-1] + self.slab(J)[0] * rb[J])
        self.E = self.start[-1]

    def slab(self, J):
        K0, K1 = brange(J, self.N, self.l, self.u)
        return self.off[K1 + 1] - self.off[K0], self.off[K0]

    def begin_tile(self, t0):
        self.jlo = column_of_start(self.start, 0, self.N - 1, t0)
        self.jhi = column_of_start(self.start, 0, self.N - 1, min(t0 + KTILE, self.E) - 1)
        self.staged = self.jhi - self.jlo < KBDSTAGE

    def geometry(self, e):
        if self.staged:
            i = column_of_start(self.start[self.jlo:self.jhi + 1], 0, self.jhi - self.jlo, e)
            J = self.jlo + i
        else:
            J = column_of_start(self.start, self.jlo, self.jhi, e)
        h, row0 = self.slab(J)
        return J, self.start[J], h, row0, self.off[J]

    def locate(self, e):
        J, st, h, row0, col0 = self.geometry(e)
        rel = e - st
        assert rel < 2 ** 32
        j = rel // h
        return row0 + rel - j * h, e, J, j

    def first_col(self, t0):
        J, st, h, row0, col0 = self.geometry(t0)
        rel = t0 - st
        j = rel // h
        return col0 + j + (0 if rel == j * h else 1)

    def col_start(self, c):
        if c >= self.n:
            return self.E
        if c >= self.off[self.jhi + 1]:
            return self.start[self.jhi + 1]
        J = block_of(self.off, self.jlo, self.jhi, c)
        return self.start[J] + (c - self.off[J]) * self.slab(J)[0]


# ---- the enumerated reference: the mirror's findstructralnz in CSC order ----
def csc_of(B):
    rows, cols, slots = B.findstructralnz()
    order = np.lexsort((rows, cols))
    rows, cols, slots = rows[order] - 1, cols[order] - 1, slots[order] - 1
    colptr = np.zeros(B.n + 1, dtype=np.int64)
    np.add.at(colptr, cols + 1, 1)
    return rows, cols, slots, np.cumsum(colptr)


def check_form(form, rows, cols, slots, colptr, slot_is_storage=True):
    """every candidate's row and kCopy slot, and every tile's first column and colptr, as the kernel's tile loop forms
    them"""
    assert form.E == len(rows)
    n = len(colptr) - 1
    for t0 in range(0, form.E, KTILE):
        form.begin_tile(t0)
        t1 = min(t0 + KTILE, form.E) if t0 + KTILE < form.E else form.E + 1
        for e in range(t0, min(t0 + KTILE, form.E)):
            r, src, _, _ = form.locate(e)
            assert r == rows[e], (t0, e)
            if slot_is_storage:
                assert src == slots[e], (t0, e)
        clo = form.first_col(t0)
        assert clo == int(np.searchsorted(colptr[:n], t0, side="left")), t0
        c = clo
        while c <= n:
            p = form.col_start(c)
            if p >= t1:
                break
            assert p == colptr[c], (t0, c)
            c += 1
        assert c == n + 1 or colptr[c] >= t1 or colptr[c] == form.E and t1 == form.E + 1


def _bb_cases():
    rng = np.random.default_rng(23)
    cases = [([1], 0, 0, 0, 0), ([3], 0, 0, 1, 1), ([4, 0, 2], 1, 1, 0, 1), ([1, 1, 1, 1], 1, 0, 0, 0),
             ([2, 3, 5], 1, 1, 9, 9),                           # lam, mu >= every block
             ([3, 3, 3], 4, 3, 1, 2),                           # l, u >= nblocks
             ([600, 2, 1, 700, 0, 3], 1, 1, 1, 2),              # a large block beside small ones: empty sub-blocks
             ([1000] * 3, 1, 1, 1, 1),                          # the 5-point stencil shape
             ([8] * 300, 1, 1, 7, 7),                           # BlockBandedMatrix's padded form
             ([1] * 2500, 2, 1, 0, 0)]                          # size-1 blocks, many columns per tile
    for _ in range(25):
        N = int(rng.integers(1, 12))
        rb = [int(v) for v in rng.integers(0 if rng.random() < 0.3 else 1, 40, N)]
        if sum(rb) == 0:
            rb[0] = 1
        l, u = (int(v) for v in rng.integers(0, N + 2, 2))
        lam, mu = (int(v) for v in rng.integers(0, 12, 2))
        cases.append((rb, l, u, lam, mu))
    return cases


MIXED = [1] * 1500 + [40] * 30       # block-dense tiles spanning more than kBdStage block columns, then fewer


def _bd_cases():
    rng = np.random.default_rng(29)
    cases = [([1], 0, 0), ([5], 2, 3), ([4, 0, 2], 1, 1), ([1] * 3000, 1, 1), (MIXED, 1, 1), ([1] * 700, 0, 0),
             ([600, 2, 1, 700, 0, 3], 1, 1), ([3, 3, 3], 5, 4), ([40] * 30, 1, 1), ([2] * 400, 0, 1)]
    for _ in range(25):
        N = int(rng.integers(1, 12))
        rb = [int(v) for v in rng.integers(0 if rng.random() < 0.3 else 1, 40, N)]
        if sum(rb) == 0:
            rb[0] = 1
        l, u = (int(v) for v in rng.integers(0, N + 2, 2))
        cases.append((rb, l, u))
    return cases


BB, BD = _bb_cases(), _bd_cases()


@pytest.mark.parametrize("case", BB, ids=[f"bb{i}" for i in range(len(BB))])
def test_block_banded_closed_forms_are_the_hook(pkg, case):
    rb, l, u, lam, mu = case
    B = pkg.BandedBlockBandedMatrix(rb, rb, (l, u), (lam, mu), device="cpu")
    rows, cols, slots, colptr = csc_of(B)
    form = BlockBand(rb, l, u, lam, mu)
    assert np.all(np.diff(colptr) >= 1)                        # every column holds its diagonal entry
    # the block-column starts are the column pointer at the first column of every block
    assert form.start == [int(colptr[o]) for o in form.off]
    for J in range(len(rb)):                                   # and the closed form inside a block column
        for j in range(rb[J] + 1):
            assert form.start[J] + bb_col_offset(form.off, form.l, form.u, lam, mu, J, j) == colptr[form.off[J] + j]
    check_form(form, rows, cols, slots, colptr)
    # the block-cyclic colour the kernel computes is matrix_colors' (0-based)
    sw, bw = lam + mu + 1, l + u + 1
    mc = B.matrix_colors() - 1
    for e in range(0, form.E, max(1, form.E // 500)):
        form.begin_tile(e - e % KTILE)
        _, _, J, j = form.locate(e)
        assert (J % bw) * sw + j % sw == mc[cols[e]]


@pytest.mark.parametrize("case", BD, ids=[f"bd{i}" for i in range(len(BD))])
def test_block_dense_closed_forms_are_the_hook(pkg, case):
    rb, l, u = case
    B = pkg.BlockSkylineMatrix(rb, rb, (l, u), device="cpu")
    rows, cols, slots, colptr = csc_of(B)
    assert np.array_equal(slots, np.arange(len(slots)))        # slab storage order is CSC order: candidate e is slot e
    form = BlockDense(rb, l, u)
    assert form.start == B.starts.tolist()
    check_form(form, rows, cols, slots, colptr)
    if len(set(rb)) == 1:                                      # the block-cyclic colour for uniform blocks
        bw, bs = l + u + 1, rb[0]
        mc = B.matrix_colors() - 1
        for e in range(0, form.E, max(1, form.E // 500)):
            form.begin_tile(e - e % KTILE)
            _, _, J, j = form.locate(e)
            assert (J % bw) * bs + j == mc[cols[e]]


def test_tiles_cross_block_columns_and_staging_switches():
    """the GPU tests' tile-boundary shapes reach what they are meant to: tiles spanning several block columns, and
    block-dense tiles on both sides of the staging switch"""
    f = BlockDense(MIXED, 1, 1)
    spans = set()
    for t0 in range(0, f.E, KTILE):
        f.begin_tile(t0)
        spans.add(f.staged)
    assert spans == {True, False}
    g = BlockBand([1000] * 3, 1, 1, 1, 1)
    crossing = 0
    for t0 in range(0, g.E, KTILE):
        g.begin_tile(t0)
        crossing += g.cj[0] != g.cj[g.nc - 1]
    assert crossing >= 2


# ---- routing ----
class FakeLib:
    """Records every fdb_*create* call as (symbol, arguments after the handle and a group's device list, without the
    opts)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            if "create" in name:
                group = name.startswith("fdb_group_create_")
                self.calls.append((name, tuple(args[3:-1] if group else args[1:-1])))
            return 0
        return fn


@pytest.fixture
def fake(pkg, monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(pkg._lib, "lib", lambda: lib)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    return lib


def _csc(pkg, m, n):
    cp = torch.ones(n + 1, dtype=torch.int64)
    return pkg.SparseMatrixCSC(m, n, cp, torch.zeros(0, dtype=torch.int64), None)


def _block_types(pkg):
    rb = [2, 3, 0, 4]
    return [
        ("banded block banded", pkg.BandedBlockBandedMatrix(rb, rb, (1, 2), (0, 1), device="cpu"), "block_banded",
         (1, 2, 0, 1)),
        ("padded block banded", pkg.BlockBandedMatrix(rb, rb, (2, 0), device="cpu"), "block_banded", (2, 0, 3, 3)),
        ("block skyline", pkg.BlockSkylineMatrix(rb, rb, (1, 1), device="cpu"), "block_dense", (1, 1)),
        ("block skyline, wide bands", pkg.BlockSkylineMatrix(rb, rb, (7, 9), device="cpu"), "block_dense", (7, 9)),
    ]


@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_block_sparsities_route_to_the_block_creators(pkg, api, fdist, fake, fdtype):
    n = 9
    cv = np.arange(n, dtype=np.int64) % 4 + 1
    for name, sp, suffix, bw in _block_types(pkg):
        proto = _csc(pkg, n, n)
        kind, pm, pn = api._oop_kind(sp, proto)
        assert (kind, pm, pn) == (pkg._lib.FDB_OOP_SPARSE, n, n), name
        for colorvec in (cv, None):
            cache = object.__new__(api.JacobianCache)
            cache.fdtype, cache._plans, cache._plan_kw = fdtype, {}, {}
            fake.calls.clear()
            cvv = range(1, n + 1) if colorvec is None else colorvec
            plan = cache._oop_plan_for(kind, sp, cvv, pn, n, n, torch.device("cuda", 0))
            assert cache._oop_plan_for(kind, sp, cvv, pn, n, n, torch.device("cuda", 0)) is plan
            (single,) = fake.calls
            fake.calls.clear()
            fdist.GroupJacobianOOP([0, 0], fdtype, colorvec=colorvec, sparsity=sp, jac_prototype=proto)._build(n, n)
            (group,) = fake.calls
            assert single[0] == f"fdb_oop_plan_create_{suffix}", name
            assert group[0] == f"fdb_group_create_oop_{suffix}", name
            assert single[1] == group[1], name
            assert single[1][0] == 4 and single[1][1] is not None, name           # nblocks, the block list
            assert single[1][2:2 + len(bw)] == bw, name
            assert single[1][-2:] == (pkg._lib.FDB_OOP_SPARSE, n), name
            assert (single[1][-3] is None) == (colorvec is None), name


def test_block_rows_come_from_the_sparsity(pkg, api):
    for name, sp, _, _ in _block_types(pkg):
        n = sp.shape[1]
        _, rows = api._oop_rows(None, None, pkg._lib.FDB_CENTRAL, None, 99, sp, None, n)
        assert rows == n, name
        with pytest.raises(ValueError):
            api._oop_kind(sp, _csc(pkg, n + 1, n))


def test_the_refusals_that_stay(pkg, api):
    n = 9
    rb = [2, 3, 0, 4]
    for name, sp, _, _ in _block_types(pkg):
        with pytest.raises(TypeError):                               # the dense result is not built
            api._oop_kind(sp, None)
        with pytest.raises(TypeError):
            api._oop_kind(sp, pkg.zeros_colmajor(n, n, "cpu"))
    rect = [pkg.BandedBlockBandedMatrix(rb, [3, 3, 3], (1, 1), (0, 1), device="cpu"),
            pkg.BlockSkylineMatrix(rb, [4, 5], (1, 1), device="cpu")]
    for sp in rect:                                                  # rectangular block lists
        with pytest.raises(TypeError):
            api._oop_kind(sp, _csc(pkg, *sp.shape))
    with pytest.raises(TypeError):
        api._oop_kind(pkg.Tridiagonal(n, device="cpu"), _csc(pkg, n, n))
    with pytest.raises(TypeError):                                  # a structured prototype
        api._oop_kind(pkg.BlockSkylineMatrix(rb, rb, (1, 1), device="cpu"),
                      pkg.BlockSkylineMatrix(rb, rb, (1, 1), device="cpu"))


def test_julia_binding_binds_the_new_entries():
    from pathlib import Path
    src = (Path(__file__).resolve().parent.parent / "finitediff.jl_b200" / "julia" / "FiniteDiffB200.jl").read_text()
    for sym in ("fdb_oop_plan_create_block_banded", "fdb_oop_plan_create_block_dense",
                "fdb_group_create_oop_block_banded", "fdb_group_create_oop_block_dense"):
        assert f"(:{sym}, libfdjac)" in src, sym
    for needle in ("function group_oop_block_banded(", "function group_oop_block_dense(", "oopblock(A::Union{DeviceBlockBanded"):
        assert needle in src, needle
