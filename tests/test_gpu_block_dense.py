"""The block-dense plan (fdb_plan_create_block_dense / fdb_group_create_block_dense): a BlockBandedMatrix Jacobian in
BlockBandedMatrices' own storage, held bit for bit, with the same f calls, to
  - the slot-addressed COO route (fdb_plan_create_coo, FDB_J_SLOTS) on the same buffer and the hook's entry list, and
  - the padded route (the mirror's BlockBandedMatrix through fdb_plan_create_block_banded), read back entry by entry.
Compact buffers are prefilled with NaN (a sentinel where x itself holds NaN): the plan must write every slot."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from _util import assert_same_bits, fdb_env  # noqa: E402

FD = {"forward": 0, "central": 1, "complex": 2}
DEV = torch.device("cuda:0")


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


class _Ell:
    """fdbs_ellrows with a row pattern that fills the block structure: row i of block row K reads every column of block
    columns max(0, K-l) .. min(N-1, K+u) (padding repeats the first with coefficient 0)."""

    def __init__(self, pkg, rb, l, u, seed, complex_=False):
        L = pkg._lib
        rng = np.random.default_rng(seed)
        off = np.concatenate([[0], np.cumsum(rb, dtype=np.int64)]).astype(np.int64)
        N, m = len(rb), int(off[-1])
        Kb = np.arange(N)
        c0 = off[np.clip(Kb - l, 0, max(N - 1, 0))] if N else off[:0]
        c1 = off[np.minimum(Kb + u, N - 1) + 1] if N else off[:0]
        krow = np.repeat(Kb, rb)
        width = (c1 - c0)[krow]
        K = max(int(width.max()) if m else 1, 1)
        p = np.arange(K)[:, None]
        cols = np.where(p < width[None, :], c0[krow][None, :] + p, c0[krow][None, :]) if m else np.zeros((K, 0))
        coef = rng.uniform(-1, 1, size=(K, m)) * (p < width[None, :])
        self.d_cols = torch.from_numpy(np.ascontiguousarray(cols.astype(np.int32))).to(DEV)
        self.d_coef = torch.from_numpy(np.ascontiguousarray(coef)).to(DEV)
        self.ctx = L.EllCtx(m, K, self.d_cols.data_ptr(), self.d_coef.data_ptr(), 0)
        sym = L.synth().fdbs_ellrows_c if complex_ else L.synth().fdbs_ellrows
        self.addr = C.cast(sym, C.c_void_p).value
        self.fn = pkg.NativeFn(self.addr, self.ctx)


def _plan(api, creator, args, fdtype, **opts):
    o = api._opts(FD[fdtype], 0, **opts)
    return api.Plan(api._new_handle(f"fdb_plan_create_{creator}", *args, C.byref(o)).value)


def _jac(pkg, plan, f, x, J, fdtype, relstep=None, absstep=None, dir=1.0, f_in=None):
    lib = pkg._lib.lib()
    ctx = C.addressof(f.ctx)
    if fdtype == "complex":
        st = lib.fdb_jacobian_complex(plan._h, f.addr, ctx, x.data_ptr(), J.data_ptr() if J.numel() else None, None)
    else:
        st = lib.fdb_jacobian(plan._h, f.addr, ctx, x.data_ptr(), J.data_ptr() if J.numel() else None, None,
                              None if f_in is None else f_in.data_ptr(), relstep if relstep is not None else float("nan"),
                              absstep if absstep is not None else float("nan"), float(dir), None)
    pkg._lib.check(st)
    torch.cuda.synchronize()


def _cv_args(cv):
    return cv.ctypes.data if cv is not None and len(cv) else None


def _dense_plan(api, B, cv, fdtype, **opts):
    blocks = np.asarray(B.rb, np.int64)
    p = _plan(api, "block_dense", (len(blocks), blocks.ctypes.data if len(blocks) else None, B.l, B.u, B.j_len,
                                   _cv_args(cv)), fdtype, **opts)
    p._keep = (blocks, cv)
    return p


def _coo_plan(api, B, cv, fdtype, **opts):
    rows, cols, slots = B.findstructralnz()
    p = _plan(api, "coo", (B.m, B.n, len(rows), rows.ctypes.data, cols.ctypes.data, api.L.FDB_J_SLOTS, slots.ctypes.data,
                           B.j_len, _cv_args(cv)), fdtype, **opts)
    p._keep = (rows, cols, slots, cv)
    return p


def _padded_plan(api, P, cv, fdtype):
    blocks = np.asarray(P.rb, np.int64)
    p = _plan(api, "block_banded", (len(blocks), blocks.ctypes.data if len(blocks) else None, P.l, P.u, P.lam, P.mu,
                                    P.w * P.n, _cv_args(cv)), fdtype)
    p._keep = (blocks, cv)
    return p


def _valid_coloring(B, rng):
    rows, cols, _ = B.findstructralnz()
    by_col = [[] for _ in range(B.n)]
    for r, c in zip(rows.tolist(), cols.tolist()):
        by_col[c - 1].append(r - 1)
    row_cols = [[] for _ in range(B.m)]
    for c in range(B.n):
        for r in by_col[c]:
            row_cols[r].append(c)
    cv = np.zeros(B.n, np.int64)
    for c in rng.permutation(B.n):
        used = {int(cv[o]) for r in by_col[c] for o in row_cols[r] if cv[o] > 0}
        k = 1
        while k in used:
            k += 1
        cv[c] = k
    return cv


def _colorings(B, rng):
    n = B.n
    rv = _valid_coloring(B, rng)
    inval = rv.copy()
    inval[rng.random(n) < 0.3] = 0
    if n > 1:
        inval[rng.integers(0, n)] = -4
    return {"matrix_colors": B.matrix_colors(), "identity": np.arange(1, n + 1, dtype=np.int64), "random": rv,
            "gaps": 2 * rv + 1, "invalid": inval}


def _structures():
    rng = np.random.default_rng(99)
    cases = [("empty", [], 1, 1), ("one", [5], 1, 0), ("ones", [1] * 9, 0, 0), ("uniform4", [4] * 9, 1, 1),
             ("uniform3_wide", [3] * 5, 7, 6), ("uniform2_l0", [2] * 8, 0, 2), ("size1_band", [1] * 11, 2, 1)]
    for i in range(8):
        N = int(rng.integers(1, 10))
        rb = [int(v) for v in rng.integers(1 if i % 3 else 0, 7, N)]
        if sum(rb) == 0:
            rb[0] = 2
        cases.append((f"rand{i}", rb, int(rng.integers(0, 4)), int(rng.integers(0, 4))))
    return cases


STRUCTS = _structures()


def _x(n, seed):
    rng = np.random.default_rng(seed)
    return torch.from_numpy(rng.uniform(-2, 2, n)).to(DEV)


def _runs(fdtype):
    runs = [{}]
    if fdtype != "complex":
        runs += [{"relstep": 1e-5, "absstep": 1e-9}, {"absstep": 0.0}]
    if fdtype == "forward":
        runs += [{"dir": -1.0}, {"f_in": True}]
    return runs


def _three_routes(pkg, api, B, cv, fdtype, x, seed, kw, fill=float("nan")):
    """(compact J, counts) of the block-dense plan, the COO slot route and the padded route (read back onto the
    compact slots), plus the block-dense plan."""
    cx = fdtype == "complex"
    out = {}
    f_in = None
    if kw.get("f_in"):
        g = _Ell(pkg, B.rb, B.l, B.u, seed)
        f_in = torch.empty(B.m, dtype=torch.float64, device=DEV)
        assert pkg._lib.synth().fdbs_ellrows(C.addressof(g.ctx), f_in.data_ptr(), x.data_ptr(), 1, B.m, B.n, None) == 0
        torch.cuda.synchronize()
    steps = {k: v for k, v in kw.items() if k != "f_in"}
    for route in ("dense", "coo", "padded"):
        f = _Ell(pkg, B.rb, B.l, B.u, seed, cx)
        if route == "padded":
            P = pkg.BlockBandedMatrix(B.rb, B.rb, (B.l, B.u), device=DEV)
            P.data.fill_(fill)
            plan = _padded_plan(api, P, cv, fdtype)
            _jac(pkg, plan, f, x, P.data, fdtype, f_in=f_in, **steps)
            pr, pc, ps = P.findstructralnz()
            D = np.full((B.m, B.n), np.nan)
            D[pr - 1, pc - 1] = P.data.cpu().numpy()[ps - 1]
            rows, cols, slots = B.findstructralnz()
            J = np.empty(B.j_len)
            J[slots - 1] = D[rows - 1, cols - 1]
        else:
            Jt = torch.full((B.j_len,), fill, dtype=torch.float64, device=DEV)
            plan = (_dense_plan if route == "dense" else _coo_plan)(api, B, cv, fdtype)
            _jac(pkg, plan, f, x, Jt, fdtype, f_in=f_in, **steps)
            J = Jt.cpu().numpy()
        out[route] = (J, f.ctx.calls, plan)
    return out


@pytest.mark.parametrize("case", STRUCTS, ids=[c[0] for c in STRUCTS])
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_matches_coo_and_padded_routes(pkg, api, case, fdtype):
    name, rb, l, u = case
    L = pkg._lib
    B = pkg.BlockSkylineMatrix(rb, rb, (l, u), device=DEV)
    seed = abs(hash(name)) % 1000
    rng = np.random.default_rng(seed + FD[fdtype])
    x = _x(B.n, seed)
    for cname, cv in _colorings(B, rng).items():
        for kw in _runs(fdtype):
            what = f"{name} {fdtype} {cname} {kw}"
            got = _three_routes(pkg, api, B, cv, fdtype, x, seed, kw)
            info = got["dense"][2].info()
            assert info["jkind"] == L.FDB_J_BLOCK_DENSE, what
            assert info["j_len"] == info["n_entries"] == B.j_len, what
            C_ = int(cv.max()) if len(cv) else 0
            assert info["alg_bytes_scatter"] == info["moved_bytes_scatter"] == 8 * B.j_len + 16 * B.n * C_, what
            assert_same_bits(got["dense"][0], got["coo"][0], what + " vs COO", allow_nan=False)
            assert_same_bits(got["dense"][0], got["padded"][0], what + " vs padded", allow_nan=False)
            assert got["dense"][1] == got["coo"][1] == got["padded"][1], what
            if fdtype != "complex":
                assert np.array_equal(got["dense"][2].eps(), got["coo"][2].eps()), what


@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_ieee_edges(pkg, api, fdtype):
    B = pkg.BlockSkylineMatrix([3, 2, 4, 1, 3], [3, 2, 4, 1, 3], (1, 1), device=DEV)
    xs = np.random.default_rng(5).uniform(-2, 2, B.n)
    xs[[0, 3, 5, 7, 9, 11]] = [0.0, -0.0, np.nan, np.inf, -np.inf, -0.0]
    x = torch.from_numpy(xs).to(DEV)
    for cv in (B.matrix_colors(), np.arange(1, B.n + 1, dtype=np.int64)):
        for kw in _runs(fdtype):
            got = _three_routes(pkg, api, B, cv, fdtype, x, 11, kw, fill=-12345.678)
            assert_same_bits(got["dense"][0], got["coo"][0], f"{fdtype} {kw} vs COO")
            assert not (got["dense"][0] == -12345.678).any()
            assert got["dense"][1] == got["coo"][1]


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_mirror_routes(pkg, api, fdtype):
    """finite_difference_jacobian_ takes a BlockSkylineMatrix to the block-dense plan, and a dense J with that sparsity to
    the slot route; both give the values of the direct plan."""
    L = pkg._lib
    B = pkg.BlockSkylineMatrix([2, 3, 3, 1], [2, 3, 3, 1], (1, 2), device=DEV)
    B.data.fill_(float("nan"))
    x = _x(B.n, 3)
    cv = B.matrix_colors()
    f = _Ell(pkg, B.rb, B.l, B.u, 3)
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=B)
    pkg.finite_difference_jacobian_(B, f.fn, x, cache)
    torch.cuda.synchronize()
    assert cache._last_plan.info()["jkind"] == L.FDB_J_BLOCK_DENSE
    ref = torch.full((B.j_len,), float("nan"), dtype=torch.float64, device=DEV)
    _jac(pkg, _dense_plan(api, B, cv, fdtype), _Ell(pkg, B.rb, B.l, B.u, 3), x, ref, fdtype)
    assert_same_bits(B.data, ref, "mirror", allow_nan=False)
    # cache-less: the sparsity defaults to J itself
    B2 = pkg.BlockSkylineMatrix(B.rb, B.cb, (1, 2), device=DEV)
    pkg.finite_difference_jacobian_(B2, f.fn, x, fdtype, colorvec=torch.from_numpy(cv))
    torch.cuda.synchronize()
    assert_same_bits(B2.data, ref, "cache-less")
    # a dense J with the block sparsity: the slot route, the same entries by (row, column), zeros elsewhere
    Jd = pkg.zeros_colmajor(B.m, B.n, DEV)
    Jd.fill_(float("nan"))
    c2 = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=B)
    pkg.finite_difference_jacobian_(Jd, f.fn, x, c2)
    torch.cuda.synchronize()
    assert c2._last_plan.info()["jkind"] == L.FDB_J_DENSE
    B.data.copy_(ref)
    assert_same_bits(Jd.cpu().numpy(), B.to_dense(), "dense J", allow_nan=False)


def _traced_f(log):
    def f(fx, x):
        log.append(x.detach().cpu().numpy().copy())
        fx.copy_(x * x * x + 0.5 * torch.roll(x, 1) - 0.25 * torch.roll(x, -2))
    return f


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("max_batch", [1, 3])
def test_same_points_and_order_as_slot_route(pkg, api, fdtype, max_batch):
    B = pkg.BlockSkylineMatrix([3, 5, 2, 4], [3, 5, 2, 4], (1, 1), device=DEV)
    x = torch.linspace(-2.0, 3.0, B.n, dtype=torch.float64, device=DEV)
    logs, vals = [], []
    for J in (B, pkg.zeros_colmajor(B.m, B.n, DEV)):
        log = []
        cache = pkg.JacobianCache(x, fdtype, colorvec=B.matrix_colors(), sparsity=B, max_batch=max_batch)
        pkg.finite_difference_jacobian_(J, _traced_f(log), x, cache)
        torch.cuda.synchronize()
        logs.append(log)
        vals.append(J.data.clone() if J is B else J)
    assert len(logs[0]) == len(logs[1]) > 0
    for a, b in zip(logs[0], logs[1]):
        assert_same_bits(a, b, "points")
    rows, cols, slots = B.findstructralnz()
    assert_same_bits(vals[0].cpu().numpy()[slots - 1], vals[1].cpu().numpy()[rows - 1, cols - 1], "values")


@pytest.mark.parametrize("use_graph", [False, True])
def test_reused_plan(pkg, api, use_graph):
    B = pkg.BlockSkylineMatrix([4] * 7, [4] * 7, (1, 1), device=DEV)
    cv = B.matrix_colors()
    plan = _dense_plan(api, B, cv, "forward", use_graph=use_graph)
    f = _Ell(pkg, B.rb, B.l, B.u, 8)
    J = torch.empty(B.j_len, dtype=torch.float64, device=DEV)
    for it in range(4):
        x = _x(B.n, 100 + it)
        J.fill_(float("nan"))
        _jac(pkg, plan, f, x, J, "forward")
        ref = torch.full_like(J, float("nan"))
        _jac(pkg, _coo_plan(api, B, cv, "forward"), _Ell(pkg, B.rb, B.l, B.u, 8), x, ref, "forward")
        assert_same_bits(J, ref, f"iteration {it}", allow_nan=False)
    assert plan.counters()["jacobians"] == 4


# one tile is 1024 slots; slabs of one slot (blocks of 1, l = u = 0) or three put more than 256 block columns in a tile,
# which takes the unstaged search
TILES = [("b4_1023", [4] * 85 + [3], 1, 1), ("b4_1024", [4] * 64, 0, 0), ("b2_1025", [2] * 128 + [1], 1, 1),
         ("s1_3000", [1] * 3000, 0, 0), ("s1_band", [1] * 1500, 1, 1), ("b8_big", [8] * 300, 1, 1),
         ("mixed", [1, 7, 2, 9, 1, 1, 5] * 40, 2, 1)]


@pytest.mark.parametrize("case", TILES, ids=[c[0] for c in TILES])
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_multi_tile_single_sm(pkg, api, case, fdtype):
    name, rb, l, u = case
    B = pkg.BlockSkylineMatrix(rb, rb, (l, u), device=DEV)
    x = _x(B.n, 21)
    cx = fdtype == "complex"
    for cv in (B.matrix_colors(), 2 * B.matrix_colors() + 1):          # closed form, and the table
        with fdb_env(SM_COUNT=1):
            plan = _dense_plan(api, B, cv, fdtype)
        J = torch.full((B.j_len,), float("nan"), dtype=torch.float64, device=DEV)
        _jac(pkg, plan, _Ell(pkg, rb, l, u, 21, cx), x, J, fdtype)
        ref = torch.full_like(J, float("nan"))
        _jac(pkg, _coo_plan(api, B, cv, fdtype), _Ell(pkg, rb, l, u, 21, cx), x, ref, fdtype)
        assert_same_bits(J, ref, f"{name} {fdtype}", allow_nan=False)


@pytest.mark.parametrize("world,partition", [(2, 0), (3, 1), (4, 0)])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_rank_plans_write_disjoint_columns(pkg, api, world, partition, fdtype):
    B = pkg.BlockSkylineMatrix([3, 5, 2, 4, 4, 1], [3, 5, 2, 4, 4, 1], (1, 2), device=DEV)
    x = _x(B.n, 31)
    rng = np.random.default_rng(31)
    for cv in (B.matrix_colors(), _colorings(B, rng)["invalid"]):
        one = torch.full((B.j_len,), float("nan"), dtype=torch.float64, device=DEV)
        _jac(pkg, _dense_plan(api, B, cv, fdtype), _Ell(pkg, B.rb, B.l, B.u, 31), x, one, fdtype)
        J = torch.full_like(one, float("nan"))
        for r in range(world):
            f = _Ell(pkg, B.rb, B.l, B.u, 31)
            _jac(pkg, _dense_plan(api, B, cv, fdtype, rank=r, world=world, partition=partition), f, x, J, fdtype)
        assert_same_bits(J, one, f"world {world}", allow_nan=False)


@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_group_on_one_device(pkg, api, fdist, fdtype):
    B = pkg.BlockSkylineMatrix([3, 5, 2, 4, 4, 1, 6], [3, 5, 2, 4, 4, 1, 6], (2, 1), device=DEV)
    x = _x(B.n, 41)
    for cv in (B.matrix_colors(), _colorings(B, np.random.default_rng(41))["invalid"]):
        one = torch.full((B.j_len,), float("nan"), dtype=torch.float64, device=DEV)
        _jac(pkg, _dense_plan(api, B, cv, fdtype), _Ell(pkg, B.rb, B.l, B.u, 41), x, one, fdtype)
        B.data.fill_(float("nan"))
        fs = [_Ell(pkg, B.rb, B.l, B.u, 41), _Ell(pkg, B.rb, B.l, B.u, 41)]
        g = fdist.GroupJacobian(B, torch.from_numpy(cv), fdtype, [0, 0])
        assert g.plans[0].info()["jkind"] == pkg._lib.FDB_J_BLOCK_DENSE
        g.run([f.fn for f in fs], x)
        g.synchronize()
        assert_same_bits(B.data, one, "group [0, 0]", allow_nan=False)
        g.close()


def test_user_size(pkg, api):
    """2.5e5 blocks of 8, l = u = 1: n = 2e6 and 4.8e7 slots, forward and central, against the slot route."""
    N, b = 250_000, 8
    rb = [b] * N
    B = pkg.BlockSkylineMatrix(rb, rb, (1, 1), device="cpu", data=torch.empty(0))
    assert B.j_len == 48_000_000 - 2 * b * b
    cv = B.matrix_colors()
    x = _x(B.n, 51)
    for fdtype in ("forward", "central"):
        J = torch.full((B.j_len,), float("nan"), dtype=torch.float64, device=DEV)
        f = _Ell(pkg, rb, 1, 1, 51)
        plan = _dense_plan(api, B, cv, fdtype)
        _jac(pkg, plan, f, x, J, fdtype)
        assert plan.info()["n_colors"] == 3 * b
        calls = f.ctx.calls
        ref = torch.full_like(J, float("nan"))
        g = _Ell(pkg, rb, 1, 1, 51)
        _jac(pkg, _coo_plan(api, B, cv, fdtype), g, x, ref, fdtype)
        assert calls == g.ctx.calls == (3 * b + 1 if fdtype == "forward" else 6 * b)
        assert bool((J.view(torch.int64) == ref.view(torch.int64)).all()), fdtype
        del J, ref
        torch.cuda.empty_cache()
