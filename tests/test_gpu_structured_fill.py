"""Block-banded (FDB_J_BLOCK_BAND), diagonal-storage (FDB_J_DIAGONALS) and block-dense (FDB_J_BLOCK_DENSE, a
BlockBandedMatrix in its own storage) Jacobians held to an f whose Jacobian fills the target's structure with distinct
values.

The native tridiagonal and 5-point f's of the other files have constant coefficients: most structural slots of a
block-banded target hold exactly +0.0 there, and the sub- and super-diagonal of diagonal storage hold the same value,
so a misaddressed slot can go unnoticed.  Here f is the ELL rows function (fdbs_ellrows / fdbs_ellrows_c on the device,
synth_ellrows / synth_ellrows_c in the oracle, bit-identical twins) built so that row r lists exactly the structural
columns of row r, each with its own coefficient drawn in +-[0.5, 2]; short rows repeat one of their own columns with
coefficient +0.0, and column slot 0 also carries the 0.1*x0^2 term.

Every case checks four things on a NaN-prefilled buffer:
  * it is bit-identical to the slot-addressed COO route (fdb_plan_create_coo on the same entry list);
  * it is bit-identical to the CPU oracle fed the device step sizes (complex step: the oracle's own run);
  * every structural slot of a column with a valid colour is within the analytic tolerance of d f_r / d x_c, evaluated
    in float64 from the coefficients (only for colourings that are valid for the structure), and none is exactly 0;
  * every slot outside the structure, and every slot of a column without a valid colour, is +0.0 by bit pattern;
with the f call counts equal and x unchanged.  The slot of each (row, column) comes from decoders written from the
documented storage layouts (block_band_entries, diagonal_entries, block_dense_entries), not from the mirror's
findstructralnz.  Block-dense storage also has every slot structural, so the COO route and the oracle cover all of J.

IEEE edges (signed zeros, NaN / +-Inf in x, x near the ends of the fp64 range) are held to the COO route and the
oracle only.  Slot offsets past 2^31 are taken by the block-banded kind (test_block_band_past_2_31, about 17 GB) and
the block-dense kind (test_block_dense_past_2_31: one slab past 2^31, and slab starts past 2^31; about 20 GB each); they
skip on a device with less free memory.  The diagonal kind is not taken past 2^31: its storage would need n of 7e8
to 1e9 and, with the f slabs, more than 40 GB."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from _util import assert_same_bits, fdb_env  # noqa: E402

FD = {"forward": 0, "central": 1, "complex": 2}
DEV = "cuda:0"
NAN = float("nan")
U = 2.0 ** -53
_f64p = C.POINTER(C.c_double)


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
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


# ------------------------------------------------------------------------------------------------ structure decoders
def block_band_entries(rb, l, u, lam, mu, dense_blocks=False):
    """(rows, cols, slots), 0-based, of a square block-banded structure, from the documented layout: entry (k, j) of
    block (K, J) is present for K in [J-u, J+l] and k in [j-mu, j+lam] (inside the blocks), and sits at slot
    (K-J+u)(lam+mu+1) + (mu+k-j) of band-data column c, w = (l+u+1)(lam+mu+1) slots per column.  dense_blocks: the
    BlockBandedMatrix of the same blocks (every row of every block in the band), stored with lam = mu = max block - 1."""
    if dense_blocks:
        lam = mu = max(rb) - 1
    off = np.concatenate([[0], np.cumsum(rb)]).astype(np.int64)
    N = len(rb)
    sw, w = lam + mu + 1, (l + u + 1) * (lam + mu + 1)
    rows, cols, slots = [], [], []
    for J in range(N):
        j = np.arange(rb[J], dtype=np.int64)
        for K in range(max(0, J - u), min(N - 1, J + l) + 1):
            for k in range(rb[K]):
                jj = j[(k >= j - mu) & (k <= j + lam)] if not dense_blocks else j
                c = off[J] + jj
                rows.append(np.full(len(jj), off[K] + k))
                cols.append(c)
                slots.append(c * w + (K - J + u) * sw + (mu + k - jj))
    cat = lambda a: np.concatenate(a).astype(np.int64) if a else np.zeros(0, np.int64)
    return cat(rows), cat(cols), cat(slots), w * int(off[-1])


def block_dense_entries(rb, l, u):
    """(rows, cols, slots, length), 0-based, of a BlockBandedMatrix in BlockBandedMatrices' own storage, from the slot
    formula of FDB_J_BLOCK_DENSE in include/fdjac_b200.h: entry (r, c) of block (K, J) sits at slot
    start_J + c h_J + (rowoff_J(K) + r), with h_J the rows of block rows max(0, J-u)..min(N-1, J+l),
    start_J = sum_{J'<J} h_J' cb[J'] and rowoff_J(K) the rows of block rows max(0, J-u)..K-1."""
    off = np.concatenate([[0], np.cumsum(rb)]).astype(np.int64)
    N = len(rb)
    rows, cols, slots = [], [], []
    start = 0
    for J in range(N):
        krange = range(max(0, J - u), min(N - 1, J + l) + 1)
        h = sum(rb[K] for K in krange)
        c = np.arange(rb[J], dtype=np.int64)
        rowoff = 0
        for K in krange:
            r = np.arange(rb[K], dtype=np.int64)
            rows.append(np.broadcast_to(off[K] + r, (len(c), len(r))).ravel())
            cols.append(np.repeat(off[J] + c, len(r)))
            slots.append((start + c[:, None] * h + rowoff + r[None, :]).ravel())
            rowoff += rb[K]
        start += h * rb[J]
    cat = lambda a: np.concatenate(a).astype(np.int64) if a else np.zeros(0, np.int64)
    return cat(rows), cat(cols), cat(slots), int(start)


def diagonal_entries(kind, n):
    """(rows, cols, slots, length), 0-based, of diagonal storage: [d] (Diagonal), [dv; ev] (Bidiagonal :U), [ev; dv]
    (:L), [dl; d; du] (Tridiagonal); dense_* targets: column-major n x n with the band of the named sparsity."""
    r = np.arange(n, dtype=np.int64)
    e = np.arange(max(n - 1, 0), dtype=np.int64)
    if kind.startswith("dense_"):
        l, u = {"diag": (0, 0), "bidiag_U": (0, 1), "bidiag_L": (1, 0), "symtri": (1, 1)}[kind[len("dense_"):]]
        rows = np.concatenate([r] + ([e + 1] if l else []) + ([e] if u else []))
        cols = np.concatenate([r] + ([e] if l else []) + ([e + 1] if u else []))
        return rows, cols, cols * n + rows, n * n
    if kind == "diag":
        return r, r, r, n
    if kind == "bidiag_U":
        return np.concatenate([r, e]), np.concatenate([r, e + 1]), np.concatenate([r, n + e]), max(2 * n - 1, 0)
    if kind == "bidiag_L":
        return (np.concatenate([e + 1, r]), np.concatenate([e, r]), np.concatenate([e, n - 1 + r]), max(2 * n - 1, 0))
    if kind == "tri":
        return (np.concatenate([e + 1, r, e]), np.concatenate([e, r, e + 1]),
                np.concatenate([e, n - 1 + r, 2 * n - 1 + e]), max(3 * n - 2, 0))
    raise ValueError(kind)


# ------------------------------------------------------------------------------------------------ f and its reference
class Ell:
    """f_r = sum_p coef[p,r] x[cols[p,r]] (left to right) + 0.1 x0^2, x0 = x[cols[0,r]]; ELL layout [K][n].  Row r lists
    exactly the structural columns of row r, each once, in random order, with coefficients in +-[0.5, 2]; short rows
    are padded with their own slot-0 column and coefficient +0.0."""

    def __init__(self, n, rows, cols, seed):
        rng = np.random.default_rng(seed)
        by_row = [[] for _ in range(n)]
        for r, c in zip(rows.tolist(), cols.tolist()):
            by_row[r].append(c)
        K = max([len(b) for b in by_row] + [1])
        self.cols = np.zeros((K, n), np.int32)
        self.coef = np.zeros((K, n), np.float64)
        for r, b in enumerate(by_row):
            assert b, f"row {r} has no structural column"
            b = rng.permutation(b)
            self.cols[:, r] = b[0]
            self.cols[: len(b), r] = b
            self.coef[: len(b), r] = rng.uniform(0.5, 2.0, len(b)) * np.where(rng.random(len(b)) < 0.5, -1.0, 1.0)
        self.K, self.n = K, n
        self.dev = None

    def native(self, pkg, complex_=False):
        if self.dev is None:
            self.dev = (torch.from_numpy(self.cols).to(DEV), torch.from_numpy(self.coef).to(DEV))
        ctx = pkg._lib.EllCtx(self.n, self.K, self.dev[0].data_ptr(), self.dev[1].data_ptr(), 0)
        fn = pkg._lib.synth().fdbs_ellrows_c if complex_ else pkg._lib.synth().fdbs_ellrows
        return pkg.NativeFn(C.cast(fn, C.c_void_p).value, ctx), ctx

    def octx(self, oracle):
        return oracle.SynthEllCtx(self.n, self.K, self.cols.ctypes.data_as(C.POINTER(C.c_int32)),
                                  self.coef.ctypes.data_as(_f64p), 1)

    def f_np(self, x):
        x0 = x[self.cols[0]]
        s = self.coef[0] * x0
        for p in range(1, self.K):
            s = s + self.coef[p] * x[self.cols[p]]
        return s + 0.1 * (x0 * x0)

    def derivative(self, rows, cols, x):
        return ell_derivative(self.cols, self.coef, rows, cols, x)


def ell_derivative(ecols, ecoef, rows, cols, x):
    """For the ELL rows f (ecols, ecoef: [K][m], each column listed at most once per row with a nonzero coefficient):
    (d f_r / d x_c, S_r = sum of |terms| of row r, T_r = sum |coef| + 0.2 |x0|) at the entries (rows, cols)."""
    K, m = ecols.shape
    n = len(x)
    nz = ecoef != 0.0
    key = np.broadcast_to(np.arange(m, dtype=np.int64), (K, m))[nz] * n + ecols[nz]
    o = np.argsort(key, kind="stable")
    key, val = key[o], ecoef[nz][o]
    q = np.asarray(rows, np.int64) * n + cols
    i = np.minimum(np.searchsorted(key, q), max(len(key) - 1, 0))
    coef = np.where(key[i] == q, val[i], 0.0) if len(key) else np.zeros(len(rows))
    x0 = x[ecols[0, rows]]
    d = coef + np.where(ecols[0, rows] == cols, 0.2 * x0, 0.0)
    terms = np.abs(ecoef * x[ecols]).sum(axis=0) + 0.1 * x[ecols[0]] ** 2
    T = np.abs(ecoef).sum(axis=0) + 0.2 * np.abs(x[ecols[0]])
    return d, terms[rows], T[rows]


def analytic_tolerance(fdtype, eps, S, T, K):
    """Bound on |J - d f_r / d x_c| for the ELL f: the truncation of the quadratic term (forward: 0.1|eps|, central:
    none) and the rounding of f's sums, about (K + 2) roundings of S per evaluation, over the step."""
    c = 4.0 * (K + 3)
    if fdtype == "forward":
        return 0.1 * np.abs(eps) + c * U * S / np.abs(eps)
    if fdtype == "central":
        return c * U * S / (2 * np.abs(eps))
    return 16 * U * T


def host_x(n, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(0.5, 2.0, n) * np.where(rng.random(n) < 0.5, -1.0, 1.0)


# ------------------------------------------------------------------------------------------------ colourings
def greedy_coloring(n, rows, cols, rng):
    """A valid distance-2 colouring of the entry list: greedy over a random column order."""
    import scipy.sparse as sps
    S = sps.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(n, n))
    G = (S.T @ S).tocsr()                                   # columns sharing a row
    cv = np.zeros(n, np.int64)
    for c in rng.permutation(n):
        used = np.zeros(n + 2, bool)
        used[cv[G.indices[G.indptr[c]:G.indptr[c + 1]]]] = True
        cv[c] = int(np.argmin(used[1:])) + 1
    return cv


def relabel(cv):
    """The same column sets under other labels (colour k -> C + 1 - k): the table path, the same step sizes."""
    C_ = int(cv.max())
    return np.where(cv >= 1, C_ + 1 - cv, cv)


def colorings(closed, n, rows, cols, rng, identity=True):
    """name -> (colour vector, valid for the structure)."""
    rv = greedy_coloring(n, rows, cols, rng)
    inval = rv.copy()
    inval[rng.random(n) < 0.3] = 0
    if n > 1:
        inval[rng.integers(0, n)] = -4
    out = {"matrix_colors": (closed, True), "relabelled": (relabel(closed), True), "random": (rv, True),
           "gaps": (2 * rv + 1, True), "invalid": (inval, True)}
    if identity:
        out["identity"] = (np.arange(1, n + 1, dtype=np.int64), True)
    return out


# ------------------------------------------------------------------------------------------------ the checks
def check_values(got, st, ell, x, cv, eps, fdtype, valid, what):
    """Analytic value check and the zero classes (see the module docstring)."""
    rows, cols, slots, length = st
    got = np.asarray(got)
    assert got.shape == (length,), what
    inside = np.zeros(length, bool)
    inside[slots] = True
    assert np.all(got[~inside].view(np.uint64) == 0), f"{what}: a slot outside the structure is not +0.0"
    k = cv[cols] - 1
    live = k >= 0
    dead_slots = slots[~live]
    assert np.all(got[dead_slots].view(np.uint64) == 0), f"{what}: a column without a valid colour is not +0.0"
    if not valid or not live.any():
        return
    r, c, s = rows[live], cols[live], slots[live]
    d, S, T = ell.derivative(r, c, x)
    e = np.asarray(eps)[k[live]] if fdtype != "complex" else None
    tol = analytic_tolerance(fdtype, e, S, T, ell.K)
    v = got[s]
    bad = np.flatnonzero(~(np.abs(v - d) <= tol))
    assert bad.size == 0, (f"{what}: {bad.size} structural slots off the derivative; first slot {s[bad[0]]} "
                           f"(row {r[bad[0]]}, col {c[bad[0]]}): {v[bad[0]]!r} vs {d[bad[0]]!r}, tol {tol[bad[0]]:.3g}")
    assert not np.any(v == 0.0), f"{what}: a structural slot of a coloured column is exactly 0"


def oracle_run(oracle, st, n, ell, x, fdtype, cv, eps, kw, f_in, dense):
    rows, cols, slots, length = st
    P = (oracle.Problem.coo_to_dense(n, n, rows + 1, cols + 1) if dense else
         oracle.Problem.coo_to_slots(n, n, rows + 1, cols + 1, slots + 1, length))
    ref = np.full(length, np.nan)
    if fdtype == "complex":
        r = oracle.jacobian_complex(P, ref, oracle.native_fn("synth_ellrows_c"), x.copy(), colorvec=cv,
                                    ctx=ell.octx(oracle))
    else:
        r = oracle.jacobian(P, ref, oracle.native_fn("synth_ellrows"), x.copy(), fdtype=FD[fdtype], colorvec=cv,
                            eps_override=eps, relstep=kw.get("relstep"), absstep=kw.get("absstep"),
                            dir=kw.get("dir", 1.0), f_in=f_in, no_drift=kw.get("no_drift", False), ctx=ell.octx(oracle))
    return ref, r["fcalls"]


def f_in_of(ell, x_np):
    return ell.f_np(x_np)


# ------------------------------------------------------------------------------------------------ block-banded runs
def bb_target(pkg, s, device=DEV):
    rb, l, u, lam, mu, dense = s
    B = pkg.BlockBandedMatrix(rb, rb, (l, u), device=device) if dense else \
        pkg.BandedBlockBandedMatrix(rb, rb, (l, u), (lam, mu), device=device)
    B.data.fill_(NAN)
    return B


def bb_run(pkg, api, s, ell, x, fdtype, cv, coo, f=None, f_in=None, run_kw=None, plan_kw=None, env=None):
    """One Jacobian into a NaN-filled target: the block-banded plan, or (coo=True) the slot-addressed route."""
    B = bb_target(pkg, s)
    ctx = None
    if f is None:
        f, ctx = ell.native(pkg, fdtype == "complex")
    if coo:
        saved = api._block_banded_plan_args
        api._block_banded_plan_args = lambda J, sp: None
    try:
        with fdb_env(**(env or {})):
            cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=B, **(plan_kw or {}))
            pkg.finite_difference_jacobian_(B, f, x, cache, f_in, **(run_kw or {}))
    finally:
        if coo:
            api._block_banded_plan_args = saved
    torch.cuda.synchronize()
    plan = cache._last_plan
    L = pkg._lib
    assert plan.info()["jkind"] == (L.FDB_J_SLOTS if coo else L.FDB_J_BLOCK_BAND)
    return B.data.cpu().numpy(), (ctx.calls if ctx is not None else None), plan


def bb_case(pkg, api, oracle, s, fdtype, cv, valid, what, seed=0, run_kw=None, plan_kw=None, f_in=False, env=None,
            ell=None, x_np=None):
    rb, l, u, lam, mu, dense = s
    st = block_band_entries(rb, l, u, lam, mu, dense)
    n = sum(rb)
    ell = ell or Ell(n, st[0], st[1], seed)
    x_np = host_x(n, seed + 1) if x_np is None else x_np
    x = torch.from_numpy(x_np).to(DEV)
    fin = torch.from_numpy(f_in_of(ell, x_np)).to(DEV) if f_in else None
    out = {}
    for coo in (False, True):
        out[coo] = bb_run(pkg, api, s, ell, x, fdtype, cv, coo, f_in=fin, run_kw=run_kw, plan_kw=plan_kw, env=env)
    assert_same_bits(x, x_np, f"{what}: x changed")
    got, calls, plan = out[False]
    assert_same_bits(got, out[True][0], f"{what}: vs COO route", allow_nan=False)
    assert calls == out[True][1], what
    kw = dict(run_kw or {}, **(plan_kw or {}))
    eps = plan.eps()
    ref, fcalls = oracle_run(oracle, st, n, ell, x_np, fdtype, cv, eps, kw, None if fin is None else fin.cpu().numpy(),
                             False)
    assert_same_bits(got, ref, f"{what}: vs oracle")
    assert fcalls == calls, what
    check_values(got, st, ell, x_np, cv, eps, fdtype, valid, what)
    return got, plan


# (name, (rb, l, u, lam, mu, dense_blocks)): empty blocks leading, interior, trailing and all but one; l != u and
# lam != mu wider than the blocks; uniform size-1 blocks (tiles span hundreds of blocks) and blocks much larger than a
# 1024-slot tile (one block spans many tiles); one block with wide sub-bandwidths; dense blocks; w in {1, 3, 7, 9, 25}
# and w > 1024 (one column spans several tiles)
BB_STRUCTS = [
    ("empty_lead", ([0, 0, 3, 5, 2, 4], 1, 1, 1, 2, False)),
    ("empty_inner", ([4, 0, 0, 3, 6, 0, 5, 2], 2, 1, 1, 1, False)),
    ("empty_trail", ([3, 5, 4, 0, 0], 1, 2, 2, 0, False)),
    ("empty_but_one", ([0, 0, 7, 0, 0, 0], 2, 2, 2, 3, False)),
    ("empty_mixed_wide", ([2, 0, 5, 1, 0, 3, 0, 4, 6], 3, 1, 4, 6, False)),
    ("l_ne_u_wide", ([3, 5, 2, 4, 6, 1, 3], 1, 3, 5, 2, False)),
    ("w1_size1", ([1] * 700, 0, 0, 0, 0, False)),
    ("w3_size1", ([1] * 400, 1, 1, 0, 0, False)),
    ("size1_nonuniform", ([1] * 300 + [2] + [1] * 299 + [0], 1, 1, 0, 0, False)),
    ("w7", ([5, 9, 3, 7, 6] * 8, 6, 0, 0, 0, False)),
    ("w9_uniform", ([6] * 40, 1, 1, 1, 1, False)),
    ("w9_big_blocks", ([700, 650, 0, 720], 1, 1, 1, 1, False)),
    ("w25_uniform_big", ([700] * 3, 2, 2, 2, 2, False)),
    ("w_over_tile", ([120, 0, 130, 110, 120], 2, 2, 100, 110, False)),
    ("one_block_wide", ([300], 0, 0, 40, 25, False)),
    ("dense_blocks", ([3, 6, 2, 5, 4], 1, 1, 0, 0, True)),
]


@pytest.mark.parametrize("name", [s[0] for s in BB_STRUCTS])
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_block_band_structures(pkg, api, oracle, name, fdtype):
    s = dict(BB_STRUCTS)[name]
    rb, l, u, lam, mu, dense = s
    st = block_band_entries(rb, l, u, lam, mu, dense)
    n = sum(rb)
    rng = np.random.default_rng(len(name) * 7 + FD[fdtype])
    closed = bb_target(pkg, s, "cpu").matrix_colors()
    ell = Ell(n, st[0], st[1], 11)
    x_np = host_x(n, 12)
    res = {}
    for cvname, (cv, valid) in colorings(closed, n, st[0], st[1], rng, identity=n <= 800).items():
        res[cvname], plan = bb_case(pkg, api, oracle, s, fdtype, cv, valid, f"{name} {fdtype} {cvname}", ell=ell,
                                    x_np=x_np)
    # the relabelled colouring goes through the table; each colour keeps its columns, so J is the closed form's bit for bit
    assert_same_bits(res["relabelled"], res["matrix_colors"], f"{name} {fdtype}: relabelled vs closed form")


BB_OPTIONS = [("dir-", {"dir": -1.0}, {}, False), ("f_in", {}, {}, True),
              ("steps", {"relstep": 1e-5, "absstep": 1e-9}, {}, False), ("abs0", {"absstep": 0.0}, {}, False),
              ("no_drift", {}, {"no_drift": True}, False), ("batch1", {}, {"max_batch": 1}, False),
              ("batch3", {}, {"max_batch": 3}, False), ("few_slabs", {}, {"scratch_bytes": "2slabs"}, False)]


@pytest.mark.parametrize("opt", BB_OPTIONS, ids=[o[0] for o in BB_OPTIONS])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_block_band_options(pkg, api, oracle, opt, fdtype):
    name, run_kw, plan_kw, f_in = opt
    if f_in and fdtype != "forward":
        pytest.skip("f_in is the forward mode's f(x)")
    for sname in ("empty_inner", "l_ne_u_wide"):
        s = dict(BB_STRUCTS)[sname]
        n = sum(s[0])
        pk = dict(plan_kw)
        if pk.get("scratch_bytes") == "2slabs":
            pk["scratch_bytes"] = 8 * ((n + 1) & ~1) * 2
        st = block_band_entries(*s[:5], s[5])
        closed = bb_target(pkg, s, "cpu").matrix_colors()
        for cvname, cv in (("matrix_colors", closed), ("relabelled", relabel(closed)),
                           ("random", greedy_coloring(n, st[0], st[1], np.random.default_rng(3)))):
            _, plan = bb_case(pkg, api, oracle, s, fdtype, cv, True, f"{sname} {fdtype} {name} {cvname}", seed=5,
                              run_kw=run_kw, plan_kw=pk, f_in=f_in)
            if name == "few_slabs" and int(cv.max()) > 2:
                assert plan.info()["n_groups"] > 1


@pytest.mark.parametrize("sm", [None, "1", "3"])
def test_block_band_sm_counts(pkg, api, oracle, sm):
    for sname in ("empty_mixed_wide", "w1_size1", "w25_uniform_big", "w_over_tile", "one_block_wide"):
        s = dict(BB_STRUCTS)[sname]
        closed = bb_target(pkg, s, "cpu").matrix_colors()
        for cvname, cv in (("matrix_colors", closed), ("relabelled", relabel(closed))):
            bb_case(pkg, api, oracle, s, "central", cv, True, f"{sname} SM_COUNT={sm} {cvname}", seed=9,
                    env={"SM_COUNT": sm})


def test_block_band_many_colours(pkg, api, oracle):
    """C = 1025 > kSmemTable: the kernel reads the colour's slab and step size from global memory."""
    s = ([41] * 25, 12, 12, 20, 20, False)
    closed = bb_target(pkg, s, "cpu").matrix_colors()
    assert int(closed.max()) == 1025
    a, _ = bb_case(pkg, api, oracle, s, "forward", closed, True, "C=1025 closed form", seed=21)
    b, _ = bb_case(pkg, api, oracle, s, "forward", relabel(closed), True, "C=1025 relabelled", seed=21)
    assert_same_bits(a, b, "C=1025: relabelled vs closed form")


@pytest.mark.parametrize("spread", [300, 30000], ids=["16bit", "32bit"])
def test_block_band_wide_colour_tables(pkg, api, oracle, spread):
    """Colour labels spread so that maximum(colorvec) needs a 16- or 32-bit table; small n (f runs once per label)."""
    s = ([3, 0, 4, 2], 1, 1, 1, 1, False)
    rb, l, u, lam, mu, dense = s
    st = block_band_entries(rb, l, u, lam, mu)
    n = sum(rb)
    cv = greedy_coloring(n, st[0], st[1], np.random.default_rng(4)) * spread
    cv[2] = -1
    _, plan = bb_case(pkg, api, oracle, s, "forward", cv, True, f"spread {spread}", seed=31)
    assert plan.info()["color_bits"] == (16 if spread == 300 else 32)


def test_block_band_graph_replay(pkg, api, oracle):
    s = dict(BB_STRUCTS)["empty_inner"]
    st = block_band_entries(*s[:5])
    n = sum(s[0])
    ell = Ell(n, st[0], st[1], 41)
    cv = bb_target(pkg, s, "cpu").matrix_colors()
    x = torch.empty(n, dtype=torch.float64, device=DEV)
    B = bb_target(pkg, s)
    f, ctx = ell.native(pkg)
    cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=B, use_graph=True)
    for seed in (1, 2, 3):
        x_np = host_x(n, seed)
        x.copy_(torch.from_numpy(x_np))                      # x changes in place: the graph is replayed
        B.data.fill_(NAN)
        pkg.finite_difference_jacobian_(B, f, x, cache)
        torch.cuda.synchronize()
        got = B.data.cpu().numpy()
        ref, _ = oracle_run(oracle, st, n, ell, x_np, "forward", cv, cache._last_plan.eps(), {}, None, False)
        assert_same_bits(got, ref, f"replay {seed}", allow_nan=False)
        check_values(got, st, ell, x_np, cv, cache._last_plan.eps(), "forward", True, f"replay {seed}")
    assert ctx.calls == 1 + int(cv.max())


def device_sets():
    sets = [[0, 0], [0, 0, 0], [0, 0, 0, 0]]
    if torch.cuda.is_available() and torch.cuda.device_count() >= 2:
        sets += [[0, 1]]
    return sets


@pytest.mark.parametrize("devices", device_sets(), ids=lambda d: "-".join(map(str, d)))
@pytest.mark.parametrize("partition", [0, 1], ids=["round_robin", "lpt"])
def test_block_band_group(pkg, api, fdist, devices, partition):
    root = torch.device("cuda", devices[0])
    for sname in ("empty_mixed_wide", "empty_but_one"):
        s = dict(BB_STRUCTS)[sname]
        st = block_band_entries(*s[:5])
        n = sum(s[0])
        ell = Ell(n, st[0], st[1], 51)
        x = torch.from_numpy(host_x(n, 52)).to(root)
        closed = bb_target(pkg, s, "cpu").matrix_colors()
        inval = closed.copy()
        inval[::4] = 0
        for fdtype in ("forward", "central"):
            for cvname, cv in (("matrix_colors", closed), ("relabelled", relabel(closed)), ("invalid", inval)):
                one, _, _ = bb_run(pkg, api, s, ell, x, fdtype, cv, False)
                BG = bb_target(pkg, s, root)
                fns = [ell.native(pkg) for _ in devices]
                gj = fdist.GroupJacobian(BG, cv, fdtype, devices, partition=partition)
                gj.run([f for f, _ in fns], x)
                gj.synchronize()
                what = f"{sname} {devices} {fdtype} {cvname} partition={partition}"
                assert_same_bits(BG.data.cpu().numpy(), one, what, allow_nan=False)
                owner = gj.plans[0].color_owner()
                for i, (_, ctx) in enumerate(fns):
                    own = int(np.sum(owner == i))
                    assert ctx.calls == (1 + own if fdtype == "forward" else 2 * own), (what, i)
                gj.close()


# ------------------------------------------------------------------------------------------------ diagonal storage
PACKED = ["diag", "bidiag_U", "bidiag_L", "tri"]
DENSE = ["dense_diag", "dense_bidiag_U", "dense_bidiag_L", "dense_symtri"]


def _sparsity(pkg, kind, n):
    return {"diag": lambda: pkg.Diagonal(n, device=DEV), "bidiag_U": lambda: pkg.Bidiagonal(n, "U", device=DEV),
            "bidiag_L": lambda: pkg.Bidiagonal(n, "L", device=DEV), "symtri": lambda: pkg.SymTridiagonal(n),
            "tri": lambda: pkg.Tridiagonal(n, device=DEV)}[kind]()


def dg_target(pkg, kind, n):
    """(J, sparsity, flat value storage) with the storage prefilled with NaN."""
    if kind.startswith("dense_"):
        J = pkg.zeros_colmajor(n, n, DEV)
        J.fill_(NAN)
        return J, _sparsity(pkg, kind[len("dense_"):], n), J.t().reshape(-1)
    J = _sparsity(pkg, kind, n)
    J.buf.fill_(NAN)
    return J, J, J.buf


def _plan(pkg, api, J, n, l, u, jkind, ld, cv, fdtype, plan_kw, rows=None, cols=None, slots=None):
    L = pkg._lib
    lib = L.lib()
    o = api._opts(FD[fdtype], 0, **plan_kw)
    cv_ptr, keep = api._index_ptr(cv)
    h = C.c_void_p()
    if rows is None:
        L.check(lib.fdb_plan_create_banded(C.byref(h), n, n, l, u, jkind, ld, cv_ptr, C.byref(o)))
    else:
        r1, c1, s1 = rows + 1, cols + 1, None if slots is None else slots + 1
        L.check(lib.fdb_plan_create_coo(C.byref(h), n, n, len(r1), r1.ctypes.data, c1.ctypes.data, jkind,
                                        None if s1 is None else s1.ctypes.data, ld, cv_ptr, C.byref(o)))
        keep = (keep, r1, c1, s1)
    return pkg.Plan(h.value, keep)


def dg_run(pkg, api, kind, n, st, f, x, fdtype, cv, coo, f_in=None, run_kw=None, plan_kw=None, env=None):
    """One Jacobian: the diagonal-storage route (a Tridiagonal buffer through the same kind, by its own plan), or
    (coo=True) the COO route on the decoder's entry list."""
    J, sp, vals = dg_target(pkg, kind, n)
    plan_kw = plan_kw or {}
    L = pkg._lib
    with fdb_env(**(env or {})):
        cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=sp, **plan_kw)
        if coo:
            dense = kind.startswith("dense_")
            ld = api._dense_ld(J)[2] if dense else st[3]
            plan = _plan(pkg, api, J, n, 0, 0, L.FDB_J_DENSE if dense else L.FDB_J_SLOTS, ld, cv,
                         fdtype, plan_kw, st[0], st[1], None if dense else st[2])
            cache.plan_for = lambda *a: plan
        elif kind == "tri":
            plan = _plan(pkg, api, J, n, 1, 1, L.FDB_J_DIAGONALS, st[3], cv, fdtype, plan_kw)
            cache.plan_for = lambda *a: plan
        pkg.finite_difference_jacobian_(J, f, x, cache, f_in, **(run_kw or {}))
    torch.cuda.synchronize()
    plan = cache._last_plan
    if not coo:
        info = plan.info()
        if kind in PACKED:
            assert info["jkind"] == L.FDB_J_DIAGONALS and info["j_len"] == st[3], kind
        else:
            assert info["jkind"] == L.FDB_J_DENSE and info["sp_kind"] == 4, kind
    return vals.cpu().numpy(), plan


def dg_case(pkg, api, oracle, kind, n, fdtype, cv, valid, what, seed=0, run_kw=None, plan_kw=None, f_in=False, env=None):
    st = diagonal_entries(kind, n)
    ell = Ell(n, st[0], st[1], seed)
    x_np = host_x(n, seed + 1)
    x = torch.from_numpy(x_np).to(DEV)
    fin = torch.from_numpy(f_in_of(ell, x_np)).to(DEV) if f_in else None
    out = {}
    for coo in (False, True):
        f, ctx = ell.native(pkg, fdtype == "complex")
        got, plan = dg_run(pkg, api, kind, n, st, f, x, fdtype, cv, coo, fin, run_kw, plan_kw, env)
        out[coo] = (got, ctx.calls, plan)
    assert_same_bits(x, x_np, f"{what}: x changed")
    got, calls, plan = out[False]
    assert_same_bits(got, out[True][0], f"{what}: vs COO route", allow_nan=False)
    assert calls == out[True][1], what
    eps = plan.eps()
    kw = dict(run_kw or {}, **(plan_kw or {}))
    ref, fcalls = oracle_run(oracle, st, n, ell, x_np, fdtype, cv, eps, kw, None if fin is None else fin.cpu().numpy(),
                             kind.startswith("dense_"))
    assert_same_bits(got, ref, f"{what}: vs oracle")
    assert fcalls == calls, what
    check_values(got, st, ell, x_np, cv, eps, fdtype, valid, what)
    return got


def dg_closed(kind, n):
    """matrix_colors of the kind's band: cyclic with period l + u + 1."""
    p = {"diag": 1, "bidiag_U": 2, "bidiag_L": 2, "tri": 3}[kind.replace("dense_", "").replace("symtri", "tri")]
    return np.arange(n, dtype=np.int64) % p + 1


# n in {1, 2, 3}, and n that put sub_end (n-1 for :L and Tridiagonal), main_end (n for :U, 2n-1 for :L and
# Tridiagonal) and total (n, 2n-1, 3n-2) on and next to a multiple of the 1024-slot tile
DG_SIZES = [1, 2, 3, 1023, 1024, 1025, 1026, 1366, 1367, 2048, 2049]


@pytest.mark.parametrize("kind", PACKED + DENSE)
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_diagonal_targets(pkg, api, oracle, kind, fdtype):
    sizes = DG_SIZES if kind in PACKED else [1, 2, 3, 130, 1025]
    for n in sizes:
        st = diagonal_entries(kind, n)
        rng = np.random.default_rng(n + 7 * FD[fdtype])
        closed = dg_closed(kind, n)
        res = {}
        for cvname, (cv, valid) in colorings(closed, n, st[0], st[1], rng, identity=n <= 1030).items():
            res[cvname] = dg_case(pkg, api, oracle, kind, n, fdtype, cv, valid, f"{kind} {fdtype} n={n} {cvname}",
                                  seed=n)
        assert_same_bits(res["relabelled"], res["matrix_colors"], f"{kind} {fdtype} n={n}: relabelled vs closed form")


@pytest.mark.parametrize("sm", ["1", "3"])
@pytest.mark.parametrize("kind", PACKED)
def test_diagonal_sm_counts(pkg, api, oracle, sm, kind):
    for n in (1024, 1025, 1366, 2049, 5000):
        closed = dg_closed(kind, n)
        for cvname, cv in (("matrix_colors", closed), ("relabelled", relabel(closed))):
            dg_case(pkg, api, oracle, kind, n, "central", cv, True, f"{kind} SM_COUNT={sm} n={n} {cvname}", seed=3,
                    env={"SM_COUNT": sm})


DG_OPTIONS = BB_OPTIONS


@pytest.mark.parametrize("opt", DG_OPTIONS, ids=[o[0] for o in DG_OPTIONS])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_diagonal_options(pkg, api, oracle, opt, fdtype):
    name, run_kw, plan_kw, f_in = opt
    if f_in and fdtype != "forward":
        pytest.skip("f_in is the forward mode's f(x)")
    n = 700
    for kind in ("bidiag_U", "bidiag_L", "tri", "dense_symtri"):
        pk = dict(plan_kw)
        if pk.get("scratch_bytes") == "2slabs":
            pk["scratch_bytes"] = 8 * ((n + 1) & ~1) * 2
        st = diagonal_entries(kind, n)
        closed = dg_closed(kind, n)
        for cvname, cv in (("matrix_colors", closed), ("relabelled", relabel(closed)),
                           ("random", greedy_coloring(n, st[0], st[1], np.random.default_rng(6)))):
            dg_case(pkg, api, oracle, kind, n, fdtype, cv, True, f"{kind} {fdtype} {name} {cvname}", seed=8,
                    run_kw=run_kw, plan_kw=pk, f_in=f_in)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("kind", PACKED)
def test_diagonal_rank_plans(pkg, api, oracle, world, kind):
    """Each rank writes exactly the slots of its own colours' columns (rank 0 also those without a valid colour); the
    merged buffer is the single plan's."""
    n = 61
    st = diagonal_entries(kind, n)
    rows, cols, slots, length = st
    ell = Ell(n, rows, cols, 71)
    x = torch.from_numpy(host_x(n, 72)).to(DEV)
    rng = np.random.default_rng(world)
    cv = rng.integers(1, 6, n) if kind == "diag" else greedy_coloring(n, rows, cols, rng)
    cv[::5] = 0
    f, _ = ell.native(pkg)
    one, _ = dg_run(pkg, api, kind, n, st, f, x, "forward", cv, False)
    col_of_slot = np.empty(length, np.int64)
    col_of_slot[slots] = cols
    merged = np.full(length, np.nan)
    for rank in range(world):
        f, ctx = ell.native(pkg)
        got, plan = dg_run(pkg, api, kind, n, st, f, x, "forward", cv, False, plan_kw={"rank": rank, "world": world})
        owner = plan.color_owner()
        k = cv[col_of_slot] - 1
        valid = (k >= 0) & (k < len(owner))
        mine = np.zeros(length, bool)
        mine[valid] = owner[k[valid]] == rank
        if rank == 0:
            mine |= ~valid
        assert np.isnan(got[~mine]).all(), (kind, rank)
        assert_same_bits(got[mine], one[mine], f"{kind} world={world} rank {rank}", allow_nan=False)
        merged[mine] = got[mine]
        assert ctx.calls == 1 + int(np.sum(owner == rank))
    assert_same_bits(merged, one, f"{kind} world={world}", allow_nan=False)


@pytest.mark.parametrize("devices", device_sets(), ids=lambda d: "-".join(map(str, d)))
@pytest.mark.parametrize("partition", [0, 1], ids=["round_robin", "lpt"])
def test_diagonal_group(pkg, api, fdist, devices, partition):
    n = 301
    for kind in ("diag", "bidiag_U", "bidiag_L", "dense_symtri"):
        st = diagonal_entries(kind, n)
        ell = Ell(n, st[0], st[1], 81)
        x = torch.from_numpy(host_x(n, 82)).to(DEV)
        closed = dg_closed(kind, n)
        inval = greedy_coloring(n, st[0], st[1], np.random.default_rng(2))
        inval[::3] = 0
        for fdtype in ("forward", "central"):
            for cvname, cv in (("matrix_colors", closed), ("relabelled", relabel(closed)), ("invalid", inval)):
                f, _ = ell.native(pkg)
                one, _ = dg_run(pkg, api, kind, n, st, f, x, fdtype, cv, False)
                JG, spG, valsG = dg_target(pkg, kind, n)
                fns = [ell.native(pkg) for _ in devices]
                gj = fdist.GroupJacobian(JG, cv, fdtype, devices, sparsity=spG, partition=partition)
                gj.run([g for g, _ in fns], x)
                gj.synchronize()
                what = f"{kind} {devices} {fdtype} {cvname} partition={partition}"
                assert_same_bits(valsG, one, what, allow_nan=False)
                owner = gj.plans[0].color_owner()
                for i, (_, ctx) in enumerate(fns):
                    own = int(np.sum(owner == i))
                    assert ctx.calls == (1 + own if fdtype == "forward" else 2 * own), (what, i)
                gj.close()


# ------------------------------------------------------------------------------------------------ block-dense storage
def bd_target(pkg, s, device=DEV):
    rb, l, u = s
    B = pkg.BlockSkylineMatrix(rb, rb, (l, u), device=device)
    B.data.fill_(NAN)
    return B


def bd_run(pkg, api, s, st, ell, x, fdtype, cv, coo, f=None, f_in=None, run_kw=None, plan_kw=None, env=None):
    """One Jacobian into a NaN-filled BlockSkylineMatrix, J and sparsity through the mirror: the block-dense plan, or
    (coo=True) the slot-addressed COO plan on the decoder's entry list and the same buffer."""
    B = bd_target(pkg, s)
    ctx = None
    if f is None:
        f, ctx = ell.native(pkg, fdtype == "complex")
    L = pkg._lib
    plan_kw = plan_kw or {}
    with fdb_env(**(env or {})):
        cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=B, **plan_kw)
        if coo:
            plan = _plan(pkg, api, B, B.n, 0, 0, L.FDB_J_SLOTS, st[3], cv, fdtype, plan_kw, st[0], st[1], st[2])
            cache.plan_for = lambda *a: plan
        pkg.finite_difference_jacobian_(B, f, x, cache, f_in, **(run_kw or {}))
    torch.cuda.synchronize()
    plan = cache._last_plan
    info = plan.info()
    assert info["jkind"] == (L.FDB_J_SLOTS if coo else L.FDB_J_BLOCK_DENSE)
    assert info["j_len"] == st[3]
    return B.data.cpu().numpy(), (ctx.calls if ctx is not None else None), plan


def bd_case(pkg, api, oracle, s, fdtype, cv, valid, what, seed=0, run_kw=None, plan_kw=None, f_in=False, env=None,
            ell=None, x_np=None, st=None):
    rb, l, u = s
    st = st or block_dense_entries(rb, l, u)
    n = sum(rb)
    ell = ell or Ell(n, st[0], st[1], seed)
    x_np = host_x(n, seed + 1) if x_np is None else x_np
    x = torch.from_numpy(x_np).to(DEV)
    fin = torch.from_numpy(f_in_of(ell, x_np)).to(DEV) if f_in else None
    out = {}
    for coo in (False, True):
        out[coo] = bd_run(pkg, api, s, st, ell, x, fdtype, cv, coo, f_in=fin, run_kw=run_kw, plan_kw=plan_kw, env=env)
    assert_same_bits(x, x_np, f"{what}: x changed")
    got, calls, plan = out[False]
    assert_same_bits(got, out[True][0], f"{what}: vs COO route", allow_nan=False)
    assert calls == out[True][1], what
    kw = dict(run_kw or {}, **(plan_kw or {}))
    eps = plan.eps()
    ref, fcalls = oracle_run(oracle, st, n, ell, x_np, fdtype, cv, eps, kw, None if fin is None else fin.cpu().numpy(),
                             False)
    assert_same_bits(got, ref, f"{what}: vs oracle")
    assert fcalls == calls, what
    check_values(got, st, ell, x_np, cv, eps, fdtype, valid, what)
    return got, plan


# (name, (rb, l, u)): empty blocks leading, interior, trailing and all but one; l != u; bandwidths of nblocks or more;
# uniform size-1 blocks (a tile spans hundreds of block columns: the unstaged search); uniform blocks (the closed form);
# blocks spanning many 1024-slot tiles
BD_STRUCTS = [
    ("empty_lead", ([0, 0, 3, 5, 2, 4], 1, 1)),
    ("empty_inner", ([4, 0, 0, 3, 6, 0, 5, 2], 2, 1)),
    ("empty_trail", ([3, 5, 4, 0, 0], 1, 2)),
    ("empty_but_one", ([0, 0, 7, 0, 0, 0], 2, 2)),
    ("l_ne_u", ([3, 5, 2, 4, 6, 1, 3], 1, 3)),
    ("wide_bands", ([3, 2, 4, 1, 5], 5, 7)),
    ("size1", ([1] * 700, 1, 1)),
    ("size1_w0", ([1] * 900, 0, 0)),
    ("uniform6", ([6] * 40, 1, 1)),
    ("big_blocks", ([300, 250, 0, 280], 1, 0)),
]


@pytest.mark.parametrize("name", [s[0] for s in BD_STRUCTS])
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_block_dense_structures(pkg, api, oracle, name, fdtype):
    s = dict(BD_STRUCTS)[name]
    rb, l, u = s
    st = block_dense_entries(rb, l, u)
    n = sum(rb)
    rng = np.random.default_rng(len(name) * 7 + FD[fdtype])
    closed = bd_target(pkg, s, "cpu").matrix_colors()
    ell = Ell(n, st[0], st[1], 13)
    x_np = host_x(n, 14)
    res = {}
    for cvname, (cv, valid) in colorings(closed, n, st[0], st[1], rng, identity=n <= 1000).items():
        res[cvname], plan = bd_case(pkg, api, oracle, s, fdtype, cv, valid, f"{name} {fdtype} {cvname}", ell=ell,
                                    x_np=x_np, st=st)
    assert_same_bits(res["relabelled"], res["matrix_colors"], f"{name} {fdtype}: relabelled vs closed form")


@pytest.mark.parametrize("opt", BB_OPTIONS, ids=[o[0] for o in BB_OPTIONS])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_block_dense_options(pkg, api, oracle, opt, fdtype):
    name, run_kw, plan_kw, f_in = opt
    if f_in and fdtype != "forward":
        pytest.skip("f_in is the forward mode's f(x)")
    for sname in ("empty_inner", "uniform6"):
        s = dict(BD_STRUCTS)[sname]
        n = sum(s[0])
        pk = dict(plan_kw)
        if pk.get("scratch_bytes") == "2slabs":
            pk["scratch_bytes"] = 8 * ((n + 1) & ~1) * 2
        st = block_dense_entries(*s)
        closed = bd_target(pkg, s, "cpu").matrix_colors()
        for cvname, cv in (("matrix_colors", closed), ("relabelled", relabel(closed)),
                           ("random", greedy_coloring(n, st[0], st[1], np.random.default_rng(3)))):
            _, plan = bd_case(pkg, api, oracle, s, fdtype, cv, True, f"{sname} {fdtype} {name} {cvname}", seed=5,
                              run_kw=run_kw, plan_kw=pk, f_in=f_in, st=st)
            if name == "few_slabs" and int(cv.max()) > 2:
                assert plan.info()["n_groups"] > 1


@pytest.mark.parametrize("use_graph", [False, True])
def test_block_dense_reused_plan(pkg, api, oracle, use_graph):
    """One cache, x changed in place between Jacobians: the plan is reused (with use_graph, the graph is replayed)."""
    s = dict(BD_STRUCTS)["empty_inner"]
    st = block_dense_entries(*s)
    n = sum(s[0])
    ell = Ell(n, st[0], st[1], 43)
    for cv in (bd_target(pkg, s, "cpu").matrix_colors(), greedy_coloring(n, st[0], st[1], np.random.default_rng(4))):
        x = torch.empty(n, dtype=torch.float64, device=DEV)
        B = bd_target(pkg, s)
        f, ctx = ell.native(pkg)
        cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=B, use_graph=use_graph)
        plans = set()
        for seed in (1, 2, 3):
            x_np = host_x(n, seed)
            x.copy_(torch.from_numpy(x_np))
            B.data.fill_(NAN)
            pkg.finite_difference_jacobian_(B, f, x, cache)
            torch.cuda.synchronize()
            got = B.data.cpu().numpy()
            plans.add(id(cache._last_plan))
            eps = cache._last_plan.eps()
            ref, _ = oracle_run(oracle, st, n, ell, x_np, "forward", cv, eps, {}, None, False)
            assert_same_bits(got, ref, f"reused {seed} graph={use_graph}", allow_nan=False)
            check_values(got, st, ell, x_np, cv, eps, "forward", True, f"reused {seed}")
        assert len(plans) == 1 and cache._last_plan.counters()["jacobians"] == 3
        # a replayed graph does not call back into the host: the f! launches were captured with the first Jacobian
        assert ctx.calls == (1 if use_graph else 3) * (1 + int(cv.max()))


# uniform blocks of 400, l = u = 1: the closed form with 1200 colours (16-bit); the identity colouring on 1100 size-1
# blocks; both past kSmemTable = 1024, so the scatter reads the step sizes and the group slots from global memory
BD_MANY = [("closed_1200", ([400] * 3, 1, 1)), ("identity_1100", ([1] * 1100, 1, 1))]


@pytest.mark.parametrize("case", BD_MANY, ids=[c[0] for c in BD_MANY])
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_block_dense_many_colours(pkg, api, oracle, case, fdtype):
    name, s = case
    st = block_dense_entries(*s)
    n = sum(s[0])
    ell = Ell(n, st[0], st[1], 61)
    x_np = host_x(n, 62)
    closed = bd_target(pkg, s, "cpu").matrix_colors()
    ident = np.arange(1, n + 1, dtype=np.int64)
    cvs = [("matrix_colors", closed)] if name.startswith("closed") else [("identity", ident)]
    if name.startswith("closed") and fdtype == "forward":
        cvs.append(("relabelled", relabel(closed)))
    res = {}
    for cvname, cv in cvs:
        res[cvname], plan = bd_case(pkg, api, oracle, s, fdtype, cv, True, f"{name} {fdtype} {cvname}", ell=ell,
                                    x_np=x_np, st=st)
        info = plan.info()
        assert info["n_colors"] > 1024 and info["color_bits"] == 16, info
    if "relabelled" in res:
        assert_same_bits(res["relabelled"], res["matrix_colors"], f"{name} {fdtype}: relabelled vs closed form")
    if fdtype == "forward":
        # one f output per group: several launches, each with its own (l0, G) window over the global tables
        for cvname, cv in cvs[:1]:
            _, plan = bd_case(pkg, api, oracle, s, fdtype, cv, True, f"{name} groups {cvname}", ell=ell, x_np=x_np,
                              st=st, plan_kw={"max_batch": 1, "scratch_bytes": 8 * ((n + 1) & ~1) * 300})
            assert plan.info()["n_groups"] > 1


@pytest.mark.parametrize("spread", [300, 70_000], ids=["16bit", "32bit"])
def test_block_dense_wide_colour_tables(pkg, api, oracle, spread):
    """Colour labels spread so that maximum(colorvec) needs a 16- or 32-bit table; small n (f runs once per label)."""
    s = ([3, 0, 4, 2], 1, 1)
    st = block_dense_entries(*s)
    n = sum(s[0])
    cv = greedy_coloring(n, st[0], st[1], np.random.default_rng(4)) * spread
    cv[2] = -1
    for fdtype in ("forward", "central") if spread < 65536 else ("forward",):
        _, plan = bd_case(pkg, api, oracle, s, fdtype, cv, True, f"spread {spread} {fdtype}", seed=33, st=st)
        assert plan.info()["color_bits"] == (16 if spread == 300 else 32)


def bd_tile_spans(rb, l, u, tile=1024):
    """The block columns each 1024-slot tile of the block-dense scatter spans (jhi - jlo + 1), found as the kernel
    finds them: the last block column whose slab start is at or before the tile's first and last slot.  A span of up
    to 256 (kBdStage) is staged in shared memory; a longer one searches the start table in global memory."""
    B = np.asarray(rb, np.int64)
    N = len(rb)
    off = np.concatenate([[0], np.cumsum(B)])
    h = np.array([off[min(N - 1, J + l) + 1] - off[max(0, J - u)] for J in range(N)], np.int64)
    start = np.concatenate([[0], np.cumsum(h * B)])
    total = int(start[-1])
    s0 = np.arange(0, total, tile, dtype=np.int64)
    s1 = np.minimum(s0 + tile, total) - 1
    col = lambda s: np.searchsorted(start[:N], s, side="right") - 1
    return col(s1) - col(s0) + 1


# l = u = 0: slabs of b^2 slots.  Blocks of 2: every tile spans exactly 256 slabs (staged, at the limit); one block of 1
# ahead of them: 257 (unstaged); [3, 1, 3, 1] + [2] * 251: 255 slabs of 9, 1, 9, 1 and 4 slots fill each tile exactly
BD_STAGING = [("span255", ([3, 1, 3, 1] + [2] * 251) * 3, 255), ("span256", [2] * 600, 256),
              ("span257", [1] + [2] * 600, 257)]


@pytest.mark.parametrize("case", BD_STAGING, ids=[c[0] for c in BD_STAGING])
@pytest.mark.parametrize("sm", [None, "1"])
def test_block_dense_staging_boundary(pkg, api, oracle, case, sm):
    name, rb, span = case
    s = (rb, 0, 0)
    spans = bd_tile_spans(rb, 0, 0)
    assert spans[:-1].max() == span and spans.max() == span, spans
    st = block_dense_entries(*s)
    n = sum(rb)
    closed = bd_target(pkg, s, "cpu").matrix_colors()
    for cvname, cv in (("matrix_colors", closed), ("relabelled", relabel(closed))):
        for fdtype in ("forward", "central"):
            bd_case(pkg, api, oracle, s, fdtype, cv, True, f"{name} SM_COUNT={sm} {fdtype} {cvname}", seed=71,
                    env={"SM_COUNT": sm}, st=st)


@pytest.mark.parametrize("world,partition", [(2, 0), (2, 1), (3, 0), (3, 1), (4, 0), (4, 1)])
def test_block_dense_rank_plans(pkg, api, oracle, world, partition):
    """Each rank writes exactly the slots of its own colours' columns (rank 0 also those without a valid colour); the
    merged buffer is the single plan's, which is the oracle's."""
    s = dict(BD_STRUCTS)["l_ne_u"]
    st = block_dense_entries(*s)
    rows, cols, slots, length = st
    n = sum(s[0])
    ell = Ell(n, rows, cols, 73)
    x_np = host_x(n, 74)
    x = torch.from_numpy(x_np).to(DEV)
    closed = bd_target(pkg, s, "cpu").matrix_colors()
    inval = greedy_coloring(n, rows, cols, np.random.default_rng(world))
    inval[::5] = 0
    for cvname, cv in (("matrix_colors", closed), ("invalid", inval)):
        one, _, plan1 = bd_run(pkg, api, s, st, ell, x, "forward", cv, False)
        ref, _ = oracle_run(oracle, st, n, ell, x_np, "forward", cv, plan1.eps(), {}, None, False)
        assert_same_bits(one, ref, f"{cvname}: one plan vs oracle")
        col_of_slot = np.empty(length, np.int64)
        col_of_slot[slots] = cols
        merged = np.full(length, np.nan)
        for rank in range(world):
            f, ctx = ell.native(pkg)
            got, _, plan = bd_run(pkg, api, s, st, ell, x, "forward", cv, False, f=f,
                                  plan_kw={"rank": rank, "world": world, "partition": partition})
            owner = plan.color_owner()
            k = cv[col_of_slot] - 1
            valid = (k >= 0) & (k < len(owner))
            mine = np.zeros(length, bool)
            mine[valid] = owner[k[valid]] == rank
            if rank == 0:
                mine |= ~valid
            what = f"{cvname} world={world} partition={partition} rank {rank}"
            assert np.isnan(got[~mine]).all(), what
            assert_same_bits(got[mine], one[mine], what, allow_nan=False)
            merged[mine] = got[mine]
            assert ctx.calls == 1 + int(np.sum(owner == rank)), what
        assert_same_bits(merged, ref, f"{cvname} world={world}: merged vs oracle", allow_nan=False)


@pytest.mark.parametrize("devices", device_sets(), ids=lambda d: "-".join(map(str, d)))
@pytest.mark.parametrize("partition", [0, 1], ids=["round_robin", "lpt"])
def test_block_dense_group(pkg, api, oracle, fdist, devices, partition):
    root = torch.device("cuda", devices[0])
    for sname in ("empty_inner", "uniform6"):
        s = dict(BD_STRUCTS)[sname]
        st = block_dense_entries(*s)
        n = sum(s[0])
        ell = Ell(n, st[0], st[1], 53)
        x_np = host_x(n, 54)
        x = torch.from_numpy(x_np).to(root)
        closed = bd_target(pkg, s, "cpu").matrix_colors()
        inval = closed.copy()
        inval[::4] = 0
        for fdtype in ("forward", "central"):
            for cvname, cv in (("matrix_colors", closed), ("invalid", inval)):
                BG = bd_target(pkg, s, root)
                fns = [ell.native(pkg) for _ in devices]
                gj = fdist.GroupJacobian(BG, cv, fdtype, devices, partition=partition)
                assert gj.plans[0].info()["jkind"] == pkg._lib.FDB_J_BLOCK_DENSE
                gj.run([f for f, _ in fns], x)
                gj.synchronize()
                what = f"{sname} {devices} {fdtype} {cvname} partition={partition}"
                got = BG.data.cpu().numpy()
                eps = gj.plans[0].eps()
                ref, fcalls = oracle_run(oracle, st, n, ell, x_np, fdtype, cv, eps, {}, None, False)
                assert_same_bits(got, ref, f"{what}: vs oracle", allow_nan=False)
                check_values(got, st, ell, x_np, cv, eps, fdtype, True, what)
                owner = gj.plans[0].color_owner()
                for i, (_, ctx) in enumerate(fns):
                    own = int(np.sum(owner == i))
                    assert ctx.calls == (1 + own if fdtype == "forward" else 2 * own), (what, i)
                assert sum(ctx.calls for _, ctx in fns) == fcalls + (len(devices) - 1 if fdtype == "forward" else 0), what
                gj.close()


# ------------------------------------------------------------------------------------------------ IEEE edges
class SignF:
    """The ELL gather plus copysign(0.5, x_r), as a torch callback and its numpy twin with the same operations in the
    same order: the sign of a zero component reaches f, and so J."""

    def __init__(self, ell):
        self.ell = ell
        self.cols = torch.from_numpy(ell.cols.astype(np.int64)).to(DEV)
        self.coef = torch.from_numpy(ell.coef).to(DEV)

    def torch_f(self, fx, x):
        x0 = x[..., self.cols[0]]
        s = self.coef[0] * x0
        for p in range(1, self.ell.K):
            s = s + self.coef[p] * x[..., self.cols[p]]
        s = s + 0.1 * (x0 * x0)
        fx.copy_(s + torch.copysign(torch.full_like(x, 0.5), x))

    def np_f(self, fx, x):
        fx[:] = self.ell.f_np(x) + np.copysign(0.5, x)


def edge_x(kind, cv, seed):
    x = host_x(len(cv), seed)
    c2 = np.flatnonzero(cv == 2)
    if kind == "signed_zeros":
        x[::7] = -0.0
        x[3::7] = 0.0
    elif kind == "nan":
        x[c2[len(c2) // 2]] = np.nan
    elif kind == "+inf":
        x[c2[len(c2) // 2]] = np.inf
    elif kind == "-inf":
        x[c2[len(c2) // 2]] = -np.inf
    else:
        from test_gpu_eps_range import make_x
        x = make_x(kind, cv)
    return x


EDGES = ["signed_zeros", "nan", "+inf", "-inf", "sq_overflow", "norm_inf", "sq_zero", "mixed"]
EDGE_TARGETS = [("bb", ([20, 0, 17, 23, 0, 20] * 4, 1, 1, 1, 1, False)), ("bb", ([24] * 25, 1, 0, 2, 1, False)),
                ("bidiag_U", None), ("bidiag_L", None), ("tri", None), ("dense_symtri", None),
                ("block_dense", ([20, 0, 17, 23, 0, 20] * 2, 1, 1))]


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("target", range(len(EDGE_TARGETS)), ids=[f"{t[0]}{i}" for i, t in enumerate(EDGE_TARGETS)])
@pytest.mark.parametrize("fdtype,dir", [("forward", 1.0), ("forward", -1.0), ("central", 1.0)])
def test_ieee_edges(pkg, api, oracle, edge, target, fdtype, dir):
    kind, s = EDGE_TARGETS[target]
    if kind == "bb":
        st = block_band_entries(*s[:5])
        n = sum(s[0])
        closed = bb_target(pkg, s, "cpu").matrix_colors()
    elif kind == "block_dense":
        st = block_dense_entries(*s)
        n = sum(s[0])
        closed = bd_target(pkg, s, "cpu").matrix_colors()
    else:
        n = 600
        st = diagonal_entries(kind, n)
        closed = dg_closed(kind, n)
    ell = Ell(n, st[0], st[1], 91)
    from test_gpu_eps_range import CASES
    kw = {"dir": dir}
    if edge in CASES and CASES[edge][0] is not None:
        kw["absstep"] = CASES[edge][0]
    for cvname, cv in (("matrix_colors", closed), ("relabelled", relabel(closed))):
        x_np = edge_x(edge, cv if cvname == "matrix_colors" else closed, 92)
        x = torch.from_numpy(x_np).to(DEV)
        sf = SignF(ell) if edge == "signed_zeros" else None
        out = {}
        for coo in (False, True):
            if sf is not None:
                f, ctx = sf.torch_f, None
            else:
                f, ctx = ell.native(pkg)
            if kind == "bb":
                got, _, plan = bb_run(pkg, api, s, ell, x, fdtype, cv, coo, f=f, run_kw=kw)
            elif kind == "block_dense":
                got, _, plan = bd_run(pkg, api, s, st, ell, x, fdtype, cv, coo, f=f, run_kw=kw)
            else:
                got, plan = dg_run(pkg, api, kind, n, st, f, x, fdtype, cv, coo, run_kw=kw)
            out[coo] = (got, plan, ctx and ctx.calls)
        what = f"{kind} {edge} {fdtype} dir={dir} {cvname}"
        assert_same_bits(x, x_np, f"{what}: x changed")
        got, plan, calls = out[False]
        assert_same_bits(got, out[True][0], f"{what}: vs COO route")
        assert calls == out[True][2], what
        rows, cols, slots, length = st
        dense = kind.startswith("dense_")
        P = (oracle.Problem.coo_to_dense(n, n, rows + 1, cols + 1) if dense else
             oracle.Problem.coo_to_slots(n, n, rows + 1, cols + 1, slots + 1, length))
        eps = plan.eps()
        okw = dict(fdtype=FD[fdtype], colorvec=cv, **kw)
        ref = np.full(length, np.nan)
        if sf is not None:
            oracle.jacobian(P, ref, sf.np_f, x_np.copy(), eps_override=eps, **okw)
            own = oracle.jacobian(P, np.full(length, np.nan), sf.np_f, x_np.copy(), **okw)
        else:
            r = oracle.jacobian(P, ref, oracle.native_fn("synth_ellrows"), x_np.copy(), eps_override=eps,
                                ctx=ell.octx(oracle), **okw)
            assert r["fcalls"] == calls, what
            own = oracle.jacobian(P, np.full(length, np.nan), oracle.native_fn("synth_ellrows"), x_np.copy(),
                                  ctx=ell.octx(oracle), **okw)
        assert_same_bits(got, ref, f"{what}: vs oracle")
        np.testing.assert_allclose(eps, own["eps"], rtol=1e-13, atol=0, err_msg=what)
        if edge in CASES:
            e2 = own["eps"][cv[np.flatnonzero(closed == 2)[0]] - 1]      # the colour make_x filled
            assert {"finite": np.isfinite(e2), "inf": np.isinf(e2), "nan": np.isnan(e2)}[CASES[edge][1]], (what, e2)
        inside = np.zeros(length, bool)
        inside[slots] = True
        assert np.all(got[~inside].view(np.uint64) == 0), f"{what}: a slot outside the structure is not +0.0"
        if edge == "signed_zeros":
            # a zero component perturbed away from its sign: |d copysign| = 1/|eps| shows in its own diagonal slot
            assert np.isfinite(got).all(), what


# ------------------------------------------------------------------------------------------------ past 2^31 slots
def test_block_band_past_2_31(pkg):
    """One uniform structure with w*n > 2^31: 256 blocks of 4096 columns, l = u = 0, lam = mu = 1024, so w = 2049 and
    2.15e9 slots (17.2 GB).  f is the native tridiagonal f; the J value of slot (r, c) is, in closed form, the sum of
    f_r's coefficients over the columns of c's colour (any colouring, valid or not).  Slots sampled above 2^31, across
    it and below it are checked against that sum; slots outside the structure must be +0.0."""
    bs, N, lam = 4096, 256, 1024
    n, sw = bs * N, 2 * lam + 1
    total = sw * n
    assert total > 2 ** 31
    free, _ = torch.cuda.mem_get_info()
    if free < 24e9:
        pytest.skip(f"needs about 24 GB of free device memory, {free / 1e9:.1f} GB free")
    B = pkg.BandedBlockBandedMatrix([bs] * N, [bs] * N, (0, 0), (lam, lam), device=DEV)
    x = torch.empty(n, dtype=torch.float64, device=DEV)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 0x2B31, None)
    rng = np.random.default_rng(31)
    s = np.unique(np.concatenate([np.arange(2 ** 31 - 6000, 2 ** 31 + 6000), rng.integers(2 ** 31, total, 300_000),
                                  rng.integers(0, 2 ** 31, 100_000), np.arange(total - 3000, total)]))
    c, t = s // sw, s % sw
    J, j = c // bs, c % bs
    k = j + t - lam
    inside = (k >= 0) & (k < bs)
    rows = J * bs + k
    closed = B.matrix_colors()
    assert int(closed.max()) == sw
    try:
        got = {}
        for name, cv in (("matrix_colors", closed), ("relabelled", relabel(closed)), ("mod3", np.arange(n) % 3 + 1)):
            B.data.fill_(NAN)
            ctx = pkg._lib.TridiagCtx(n, 0)
            f = pkg.NativeFn(C.cast(pkg._lib.synth().fdbs_tridiag, C.c_void_p).value, ctx)
            cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=B)
            pkg.finite_difference_jacobian_(B, f, x, cache)
            torch.cuda.synchronize()
            info = cache._last_plan.info()
            assert info["jkind"] == pkg._lib.FDB_J_BLOCK_BAND and info["j_len"] == total
            assert ctx.calls == 1 + int(cv.max())
            v = B.data[torch.from_numpy(s).to(DEV)].cpu().numpy()
            del cache
            assert np.all(v[~inside].view(np.uint64) == 0), f"{name}: a slot outside the structure is not +0.0"
            # sum of f_r's coefficients over the columns of the colour of c: -2 at r, 1 at r - 1 and r + 1
            r, cc = rows[inside], c[inside]
            want = np.zeros(len(r))
            for dc, coef in ((-1, 1.0), (0, -2.0), (1, 1.0)):
                o = r + dc
                ok = (o >= 0) & (o < n)
                want += np.where(ok & (cv[np.clip(o, 0, n - 1)] == cv[cc]), coef, 0.0)
            np.testing.assert_allclose(v[inside], want, rtol=1e-6, atol=1e-6, err_msg=name)
            assert np.all(v[inside][want == 0].view(np.uint64) == 0), name
            got[name] = v
        assert_same_bits(got["relabelled"], got["matrix_colors"], "relabelled vs closed form past 2^31")
    finally:
        del B
        torch.cuda.empty_cache()


def tridiag_colour_sum(rows, c, cv, n):
    """J value of (row, column) under the native tridiagonal f and colouring cv: the sum of f_r's coefficients (-2 at r,
    1 at r - 1 and r + 1) over the columns of c's colour (any colouring, valid or not)."""
    want = np.zeros(len(rows))
    for dc, coef in ((-1, 1.0), (0, -2.0), (1, 1.0)):
        o = rows + dc
        ok = (o >= 0) & (o < n)
        want += np.where(ok & (cv[np.clip(o, 0, n - 1)] == cv[c]), coef, 0.0)
    return want


# (a) one block of 46 400: a slab of 2 152 960 000 slots, so offsets inside one slab pass 2^31; (b) 700 blocks of 1024
# with l = u = 1: 2.2e9 slots, so the slab starts pass 2^31
BD_PAST = [("one_slab", [46_400], 0, 0), ("slab_starts", [1024] * 700, 1, 1)]


@pytest.mark.parametrize("case", BD_PAST, ids=[c[0] for c in BD_PAST])
def test_block_dense_past_2_31(pkg, case):
    """Block-dense storage past 2^31 slots (about 17.6 GB of J and 2 GiB of f outputs).  Slots sampled below 2^31, across
    it, above it and at the end are decoded with the header's slot formula in int64 and checked against the closed-form
    sum of the tridiagonal f's coefficients over the colour of their column; J is prefilled with NaN."""
    name, rb, l, u = case
    n = sum(rb)
    N = len(rb)
    off = np.concatenate([[0], np.cumsum(rb)]).astype(np.int64)
    K0 = np.maximum(np.arange(N) - u, 0)
    K1 = np.minimum(np.arange(N) + l, N - 1)
    h = off[K1 + 1] - off[K0]
    start = np.concatenate([[0], np.cumsum(h * np.asarray(rb, np.int64))])
    total = int(start[-1])
    assert total > 2 ** 31
    if name == "one_slab":
        assert total > 2 ** 31 and total < 2 ** 32
    free, _ = torch.cuda.mem_get_info()
    need = 8 * total + (2 << 30) + 2e9
    if free < need:
        pytest.skip(f"needs about {need / 1e9:.0f} GB of free device memory, {free / 1e9:.1f} GB free")
    rng = np.random.default_rng(37)
    s = np.unique(np.concatenate([np.arange(2 ** 31 - 5000, 2 ** 31 + 5000), rng.integers(2 ** 31, total, 200_000),
                                  rng.integers(0, 2 ** 31, 100_000), np.arange(total - 3000, total),
                                  np.arange(0, 2000)]))
    J = np.searchsorted(start[:N], s, side="right") - 1
    rel = s - start[J]
    col = off[J] + rel // h[J]
    row = off[K0[J]] + rel % h[J]
    B = pkg.BlockSkylineMatrix(rb, rb, (l, u), device=DEV)
    assert B.j_len == total
    x = torch.empty(n, dtype=torch.float64, device=DEV)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, 0x2B32, None)
    closed = B.matrix_colors()
    cvs = [("matrix_colors", closed), ("mod3", np.arange(n) % 3 + 1)] if name == "one_slab" else \
        [("matrix_colors", closed), ("relabelled", relabel(closed))]
    try:
        got = {}
        for cvname, cv in cvs:
            B.data.fill_(NAN)
            ctx = pkg._lib.TridiagCtx(n, 0)
            f = pkg.NativeFn(C.cast(pkg._lib.synth().fdbs_tridiag, C.c_void_p).value, ctx)
            cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=B, scratch_bytes=2 << 30)
            pkg.finite_difference_jacobian_(B, f, x, cache)
            torch.cuda.synchronize()
            info = cache._last_plan.info()
            assert info["jkind"] == pkg._lib.FDB_J_BLOCK_DENSE and info["j_len"] == total
            assert ctx.calls == 1 + int(cv.max())
            v = B.data[torch.from_numpy(s).to(DEV)].cpu().numpy()
            del cache
            want = tridiag_colour_sum(row, col, cv, n)
            np.testing.assert_allclose(v, want, rtol=1e-6, atol=1e-6, err_msg=f"{name} {cvname}")
            assert np.all(v[want == 0].view(np.uint64) == 0), f"{name} {cvname}: a zero slot is not +0.0"
            got[cvname] = v
        if "relabelled" in got:
            assert_same_bits(got["relabelled"], got["matrix_colors"], "relabelled vs closed form past 2^31")
    finally:
        del B
        torch.cuda.empty_cache()


def test_block_dense_slab_limit(pkg, api):
    """A block column may hold up to 2^32 - 1 slots: one block of 65 535 (4 294 836 225 slots) makes a plan, one of
    65 536 (2^32) is refused.  No J is needed to create the plan."""
    L = pkg._lib
    for b, want in ((65_535, L.FDB_OK), (65_536, L.FDB_ERR_UNSUPPORTED)):
        blocks = np.array([b], np.int64)
        h = C.c_void_p()
        o = api._opts(FD["forward"], 0)
        st = L.lib().fdb_plan_create_block_dense(C.byref(h), 1, blocks.ctypes.data, 0, 0, b * b, None, C.byref(o))
        assert st == want, (b, st, L.lib().fdb_last_error())
        if st == L.FDB_OK:
            plan = pkg.Plan(h.value)
            info = plan.info()
            assert info["jkind"] == L.FDB_J_BLOCK_DENSE and info["j_len"] == b * b > 2 ** 31
            del plan
        else:
            assert not h.value
