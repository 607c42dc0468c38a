"""Diagonal-storage Jacobians (FDB_J_DIAGONALS through fdb_plan_create_banded / fdb_group_create_banded): Diagonal and
Bidiagonal targets written by the closed-form diagonal scatter, and dense targets with Diagonal / Bidiagonal /
SymTridiagonal sparsities through the banded plan.  Every case is held bit for bit to the slot-addressed COO route built
from the same findstructralnz lists (run in the same process) and to the CPU oracle fed the device step sizes.

J is prefilled with NaN: the packed targets are never zero-filled, so every slot has to be written; NaN counts as one
class and signed zeros are compared by bit pattern."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from _util import assert_same_bits, fdb_env  # noqa: E402

FD = {"forward": 0, "central": 1, "complex": 2}
DEV = "cuda:0"
NAN = float("nan")


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


PACKED = ["diag", "bidiag_U", "bidiag_L"]
DENSE = ["dense_diag", "dense_bidiag_U", "dense_bidiag_L", "dense_symtri", "dense_tri"]


def _sparsity(pkg, name, n):
    return {"diag": lambda: pkg.Diagonal(n, device=DEV), "bidiag_U": lambda: pkg.Bidiagonal(n, "U", device=DEV),
            "bidiag_L": lambda: pkg.Bidiagonal(n, "L", device=DEV), "symtri": lambda: pkg.SymTridiagonal(n),
            "tri": lambda: pkg.Tridiagonal(n, device=DEV)}[name]()


def _target(pkg, kind, n):
    """(J, sparsity, flat value storage) with the storage prefilled with NaN."""
    if kind.startswith("dense_"):
        J = pkg.zeros_colmajor(n, n, DEV)
        sp = _sparsity(pkg, kind[len("dense_"):], n)
        J.fill_(NAN)
        return J, sp, J.t().reshape(-1)
    J = _sparsity(pkg, kind, n)
    J.buf.fill_(NAN)
    return J, J, J.buf


class _Tri:
    """The native tridiagonal f! (any n), with its call counter."""

    def __init__(self, pkg, n, complex_=False):
        L = pkg._lib
        self.ctx = L.TridiagCtx(n, 0)
        sym = L.synth().fdbs_tridiag_c if complex_ else L.synth().fdbs_tridiag
        self.fn = pkg.NativeFn(C.cast(sym, C.c_void_p).value, self.ctx)


def _x(pkg, n, seed):
    x = torch.empty(n, dtype=torch.float64, device=DEV)
    pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, seed, None)
    return x


def _coo_plan(pkg, api, J, sp, cv, fdtype, **plan_kw):
    """The slot-addressed route on the findstructralnz lists: FDB_J_SLOTS into the packed buffer, FDB_J_DENSE into a dense J."""
    L = pkg._lib
    lib = L.lib()
    rows, cols, slots = sp.findstructralnz()
    n = sp.n
    o = api._opts(FD[fdtype], 0, **plan_kw)
    cv_ptr, keep = api._index_ptr(cv)
    h = C.c_void_p()
    if isinstance(J, torch.Tensor):
        L.check(lib.fdb_plan_create_coo(C.byref(h), n, n, len(rows), rows.ctypes.data, cols.ctypes.data, L.FDB_J_DENSE,
                                        None, api._dense_ld(J)[2], cv_ptr, C.byref(o)))
    else:
        L.check(lib.fdb_plan_create_coo(C.byref(h), n, n, len(rows), rows.ctypes.data, cols.ctypes.data, L.FDB_J_SLOTS,
                                        slots.ctypes.data, J.buf.numel(), cv_ptr, C.byref(o)))
    return pkg.Plan(h.value, (keep, rows, cols, slots))


def _run(pkg, api, J, sp, f, x, fdtype, cv, coo=False, f_in=None, run_kw=None, **plan_kw):
    """One Jacobian through the mirror: the route make_plan picks, or (coo=True) the COO slot route on the same lists."""
    cache = pkg.JacobianCache(x, fdtype, colorvec=cv, sparsity=sp, **plan_kw)
    if coo:
        plan = _coo_plan(pkg, api, J, sp, cv, fdtype, **plan_kw)
        cache.plan_for = lambda *a: plan
    pkg.finite_difference_jacobian_(J, f, x, cache, f_in, **(run_kw or {}))
    torch.cuda.synchronize()
    return cache._last_plan


def _valid_coloring(n, l, u, rng):
    """A random distance-2 colouring of the band (l, u): greedy over a random column order."""
    cv = np.zeros(n, np.int64)
    w = l + u
    for c in rng.permutation(n):
        used = {int(cv[o]) for o in range(max(0, c - w), min(n, c + w + 1)) if o != c and cv[o] > 0}
        k = 1
        while k in used:
            k += 1
        cv[c] = k
    return cv


def _lu(sp):
    return (sp.l, sp.u) if hasattr(sp, "l") else (1, 1)          # Tridiagonal: (1, 1)


def _colorings(pkg, sp, n, rng):
    rv = _valid_coloring(n, *_lu(sp), rng)
    out = {"matrix_colors": pkg.matrix_colors(sp), "default": None, "random": rv, "gaps": 2 * rv + 1}
    inval = rv.copy()
    inval[rng.random(n) < 0.3] = 0
    if n > 1:
        inval[rng.integers(0, n)] = -3
    out["invalid"] = inval
    out["none_valid"] = np.zeros(n, np.int64)
    # an invalid table: two neighbouring columns share a colour (the reference stores what the colour loop gives)
    bad = np.arange(n, dtype=np.int64) % 2 + 1
    out["bad_table"] = bad
    return out


def _oracle_check(pkg, oracle, J, sp, vals, x_seed, n, fdtype, cv, plan, calls, kw, f_in_host, what):
    rows, cols, slots = sp.findstructralnz()
    got = vals.cpu().numpy()
    cvh = None if cv is None else (cv.cpu().numpy() if isinstance(cv, torch.Tensor) else np.asarray(cv))
    probs = []
    if isinstance(J, torch.Tensor):
        probs.append(oracle.Problem.coo_to_dense(n, n, rows, cols))
        if not isinstance(sp, pkg.Tridiagonal):
            probs.append(oracle.Problem.banded_to_dense(n, n, sp.l, sp.u))
    else:
        probs.append(oracle.Problem.coo_to_slots(n, n, rows, cols, slots, vals.numel()))
    for P in probs:
        ref = np.full(vals.numel(), np.nan)
        if fdtype == "complex":
            r = oracle.jacobian_complex(P, ref, oracle.native_fn("synth_tridiag_c"), oracle.fill_x(n, x_seed), colorvec=cvh,
                                        ctx=oracle.SynthTridiagCtx(n, 1))
        else:
            r = oracle.jacobian(P, ref, oracle.native_fn("synth_tridiag"), oracle.fill_x(n, x_seed), fdtype=FD[fdtype],
                                colorvec=cvh, eps_override=plan.eps(), relstep=kw.get("relstep"),
                                absstep=kw.get("absstep"), dir=kw.get("dir", 1.0), f_in=f_in_host,
                                no_drift=kw.get("no_drift", False), ctx=oracle.SynthTridiagCtx(n, 1))
        assert_same_bits(got, ref, what + " vs oracle")
        assert r["fcalls"] == calls, what


def _f_in(pkg, x, n):
    # f(x) by the same native f (its 16-byte path wants even leading dimensions)
    fx = torch.empty(n + 1, dtype=torch.float64, device=DEV)
    fctx = pkg._lib.TridiagCtx(n, 0)
    ld = (n + 1) & ~1
    assert pkg._lib.synth().fdbs_tridiag(C.addressof(fctx), fx.data_ptr(), x.data_ptr(), 1, ld, ld, None) == 0
    torch.cuda.synchronize()
    return fx[:n]


def _compare(pkg, api, oracle, kind, n, fdtype, cv, seed, what, f_in=False, run_kw=None, **plan_kw):
    x = _x(pkg, n, seed)
    x0 = x.clone()
    out = {}
    for coo in (False, True):
        J, sp, vals = _target(pkg, kind, n)
        f = _Tri(pkg, n, fdtype == "complex")
        fin = _f_in(pkg, x, n) if f_in else None
        plan = _run(pkg, api, J, sp, f.fn, x, fdtype, cv, coo, f_in=fin, run_kw=run_kw, **plan_kw)
        out[coo] = (vals.clone(), f.ctx.calls, plan, J, sp, fin)
    assert_same_bits(x, x0, what + ": x changed", allow_nan=False)
    got, calls, plan, J, sp, fin = out[False]
    info = plan.info()
    L = pkg._lib
    if kind in PACKED:
        assert info["jkind"] == L.FDB_J_DIAGONALS, what
        assert info["j_len"] == vals.numel() == (sp.l + sp.u + 1) * n - sp.l - sp.u, what
    elif kind != "dense_tri":
        assert info["jkind"] == L.FDB_J_DENSE and info["sp_kind"] == 4, what
    assert_same_bits(got, out[True][0], what + " vs COO route")
    if kind in PACKED:
        assert not torch.isnan(got).any().item(), what
    assert calls == out[True][1], what
    _oracle_check(pkg, oracle, J, sp, got, seed, n, fdtype, cv, plan, calls, dict(run_kw or {}, **plan_kw),
                  None if fin is None else fin.cpu().numpy(), what)
    return plan


# sizes: the smallest, and the scatter's tile boundaries (1024 slots: n for Diagonal, 2n - 1 for Bidiagonal) +- 1
SIZES = [1, 2, 3, 511, 512, 513, 1023, 1024, 1025]


@pytest.mark.parametrize("kind", PACKED + DENSE)
@pytest.mark.parametrize("fdtype", ["forward", "central", "complex"])
def test_matches_coo_route_and_oracle(pkg, api, oracle, kind, fdtype):
    sizes = SIZES if kind in PACKED else [1, 2, 3, 513, 1025]
    for n in sizes:
        rng = np.random.default_rng(n * 7 + FD[fdtype])
        _, sp, _ = _target(pkg, kind, n)
        for name, cv in _colorings(pkg, sp, n, rng).items():
            _compare(pkg, api, oracle, kind, n, fdtype, cv, 0x5EED + n, f"{kind} {fdtype} n={n} {name}")


OPTIONS = [("dir-", {}, {"dir": -1.0}), ("steps", {}, {"relstep": 1e-5, "absstep": 1e-9}), ("abs0", {}, {"absstep": 0.0}),
           ("f_in", {}, {}), ("no_drift", {"no_drift": True}, {}), ("batch1", {"max_batch": 1}, {}),
           ("batch3", {"max_batch": 3}, {})]


@pytest.mark.parametrize("opt", OPTIONS, ids=[o[0] for o in OPTIONS])
@pytest.mark.parametrize("kind", ["diag", "bidiag_U", "bidiag_L", "dense_symtri"])
@pytest.mark.parametrize("fdtype", ["forward", "central"])
def test_options(pkg, api, oracle, opt, kind, fdtype):
    name, plan_kw, run_kw = opt
    if name == "f_in" and fdtype != "forward":
        pytest.skip("f_in is the forward mode's f(x)")
    for n in (3, 700):
        _, sp, _ = _target(pkg, kind, n)
        for cvname, cv in (("matrix_colors", pkg.matrix_colors(sp)),
                           ("random", _valid_coloring(n, sp.l, sp.u, np.random.default_rng(n)))):
            _compare(pkg, api, oracle, kind, n, fdtype, cv, 91 + n, f"{kind} {fdtype} {name} n={n} {cvname}",
                     f_in=name == "f_in", run_kw=run_kw, **plan_kw)


def _traced_f(log):
    def f(fx, x):
        log.append(x.detach().cpu().numpy().copy())
        fx.copy_(x * x * x + 0.5 * torch.roll(x, 1))
    return f


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("max_batch", [1, 3])
def test_same_points_and_order_as_coo_route(pkg, api, fdtype, max_batch):
    n = 11
    x = torch.linspace(-2.0, 3.0, n, dtype=torch.float64, device=DEV)
    for kind in PACKED:
        out = {}
        for coo in (False, True):
            log = []
            J, sp, vals = _target(pkg, kind, n)
            cv = _valid_coloring(n, sp.l, sp.u, np.random.default_rng(5)) * 2 - 1       # odd colours: empty ones between
            _run(pkg, api, J, sp, _traced_f(log), x, fdtype, cv, coo, max_batch=max_batch)
            out[coo] = (vals.clone(), log)
        assert_same_bits(out[False][0], out[True][0], kind, allow_nan=False)
        assert len(out[False][1]) == len(out[True][1])
        for a, b in zip(out[False][1], out[True][1]):
            assert_same_bits(a, b, f"{kind}: point passed to f")


def test_matrix_colors(pkg):
    for n in (1, 2, 7, 1000):
        c = np.arange(n)
        assert np.array_equal(pkg.matrix_colors(pkg.Diagonal(n, device=DEV)).cpu().numpy(), np.ones(n, np.int64))
        for uplo in ("U", "L"):
            assert np.array_equal(pkg.matrix_colors(pkg.Bidiagonal(n, uplo, device=DEV)).cpu().numpy(), c % 2 + 1)
        assert np.array_equal(pkg.matrix_colors(pkg.SymTridiagonal(n)).cpu().numpy(), c % 3 + 1)


def test_graph_replay_after_x_changes_in_place(pkg, api):
    n = 1500
    x = torch.empty(n, dtype=torch.float64, device=DEV)
    B = pkg.Bidiagonal(n, "L", device=DEV)
    cv = pkg.matrix_colors(B)
    f = _Tri(pkg, n)
    cache = pkg.JacobianCache(x, "forward", colorvec=cv, sparsity=B, use_graph=True)
    for seed in (5, 6, 7):
        pkg._lib.synth().fdbs_fill_x(x.data_ptr(), n, seed, None)   # x changes in place: the graph is replayed
        B.buf.fill_(NAN)
        pkg.finite_difference_jacobian_(B, f.fn, x, cache)
        torch.cuda.synchronize()
        ref = pkg.Bidiagonal(n, "L", device=DEV)
        ref.buf.fill_(NAN)
        _run(pkg, api, ref, ref, _Tri(pkg, n).fn, x, "forward", cv, True)
        assert_same_bits(B.buf, ref.buf, f"seed {seed}", allow_nan=False)
    assert f.ctx.calls == 1 + 2
    cnt = cache._last_plan.counters()
    assert cnt["jacobians"] == 3 and cnt["f_points"] == 3 * 3


@pytest.mark.parametrize("sm", ["1", "3"])
@pytest.mark.parametrize("kind", PACKED)
def test_many_tiles_few_sms(pkg, api, sm, kind):
    n = 100_000
    x = _x(pkg, n, 33)
    res = {}
    for coo in (False, True):
        J, sp, vals = _target(pkg, kind, n)
        cv = pkg.matrix_colors(sp)
        with fdb_env(SM_COUNT=sm):
            _run(pkg, api, J, sp, _Tri(pkg, n).fn, x, "central", cv, coo)
        res[coo] = vals.clone()
    assert_same_bits(res[False], res[True], f"{kind} SM_COUNT={sm}", allow_nan=False)


def test_bidiagonal_1e7_matches_coo_route(pkg, api):
    n = 10_000_000
    x = _x(pkg, n, 0xB1D)
    res = {}
    for coo in (False, True):
        B = pkg.Bidiagonal(n, "U", device=DEV)
        B.buf.fill_(NAN)
        f = _Tri(pkg, n)
        _run(pkg, api, B, B, f.fn, x, "forward", pkg.matrix_colors(B), coo)
        res[coo] = (B.buf, f.ctx.calls)
        del B
    a, b = res[False][0], res[True][0]
    assert not torch.isnan(a).any().item()
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))
    assert res[False][1] == res[True][1] == 3


@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("kind", PACKED)
def test_rank_plans_write_their_own_columns(pkg, api, fdtype, kind):
    """world = 2 rank plans on NaN-filled J: each rank writes exactly the slots of its own colours' columns, rank 0 also
    those of the columns without a valid colour; together they give the single plan's J."""
    n = 37
    x = _x(pkg, n, 44)
    J1, sp, vals1 = _target(pkg, kind, n)
    rng = np.random.default_rng(8)
    # (Diagonal: any colouring is valid; three colours, so that both ranks own some)
    cv = rng.integers(1, 4, n) if kind == "diag" else _valid_coloring(n, sp.l, sp.u, rng)
    cv[::5] = 0
    _run(pkg, api, J1, sp, _Tri(pkg, n).fn, x, fdtype, cv)
    one = vals1.cpu().numpy()
    rows, cols, slots = sp.findstructralnz()
    col_of_slot = np.empty(len(slots), np.int64)
    col_of_slot[slots - 1] = cols - 1
    merged = np.full(len(slots), np.nan)
    for rank in (0, 1):
        J, sp_r, vals = _target(pkg, kind, n)
        f = _Tri(pkg, n)
        plan = _run(pkg, api, J, sp_r, f.fn, x, fdtype, cv, rank=rank, world=2)
        got = vals.cpu().numpy()
        owner = plan.color_owner()
        k = cv[col_of_slot] - 1
        valid = (k >= 0) & (k < len(owner))
        mine = np.zeros(len(slots), bool)
        mine[valid] = owner[k[valid]] == rank
        if rank == 0:
            mine |= ~valid
        assert plan.info()["n_local_colors"] > 0
        assert np.isnan(got[~mine]).all(), (kind, rank)
        assert_same_bits(got[mine], one[mine], f"{kind} rank {rank}", allow_nan=False)
        merged[mine] = got[mine]
        own = int(np.sum(owner == rank))
        assert f.ctx.calls == (1 + own if fdtype == "forward" else 2 * own)
    assert_same_bits(merged, one, kind, allow_nan=False)


def device_sets():
    sets = [[0, 0], [0, 0, 0]]
    if torch.cuda.is_available() and torch.cuda.device_count() >= 2:
        sets += [[0, 1]]
    return sets


@pytest.mark.parametrize("devices", device_sets(), ids=lambda d: "-".join(map(str, d)))
@pytest.mark.parametrize("fdtype", ["forward", "central"])
@pytest.mark.parametrize("partition", [0, 1])
def test_group_bit_identical_to_one_device(pkg, api, fdist, devices, fdtype, partition):
    root = torch.device("cuda", devices[0])
    for kind in PACKED + ["dense_bidiag_L", "dense_symtri"]:
        for cvkind in ("matrix_colors", "random", "invalid", "one"):
            if cvkind == "one" and kind != "diag":
                continue                                    # one colour: fewer colours than members
            n = 301
            J1, sp, vals1 = _target(pkg, kind, n)
            if cvkind == "matrix_colors":
                cv = pkg.matrix_colors(sp)
            else:
                cv = _valid_coloring(n, sp.l, sp.u, np.random.default_rng(3))
                if cvkind == "invalid":
                    cv[::3] = 0
                elif cvkind == "one":
                    cv = np.ones(n, np.int64)
            x = _x(pkg, n, 17)
            _run(pkg, api, J1, sp, _Tri(pkg, n).fn, x, fdtype, cv)
            JG, spG, valsG = _target(pkg, kind, n)
            ctxs = [_Tri(pkg, n) for _ in devices]
            gj = fdist.GroupJacobian(JG, cv, fdtype, devices, sparsity=spG, partition=partition)
            gj.run([c.fn for c in ctxs], x)
            gj.synchronize()
            what = f"{devices} {kind} {cvkind} partition={partition}"
            assert_same_bits(valsG, vals1, what, allow_nan=False)
            owner = gj.plans[0].color_owner()
            cvh = cv.cpu().numpy() if isinstance(cv, torch.Tensor) else cv
            for i, c in enumerate(ctxs):
                own = int(np.sum(owner == i))
                assert c.ctx.calls == (1 + own if fdtype == "forward" else 2 * own), (what, i)
                if kind in PACKED:
                    assert gj.plans[i].info()["jkind"] == pkg._lib.FDB_J_DIAGONALS
            assert sum(int(np.sum(owner == i)) for i in range(len(devices))) == int(max(cvh.max(), 0))
            gj.close()


def test_group_complex_refused(pkg, fdist):
    B = pkg.Bidiagonal(9, "U", device=DEV)
    x = torch.ones(9, dtype=torch.float64, device=DEV)
    gj = fdist.GroupJacobian(B, pkg.matrix_colors(B), "complex", [0, 0])
    f = _Tri(pkg, 9, True)
    with pytest.raises(pkg._lib.FdbError) as e:
        gj.run([f.fn, f.fn], x)
    assert e.value.status == pkg._lib.FDB_ERR_UNSUPPORTED
    gj.close()


def test_symtridiagonal_target_refused_before_any_f_call(pkg):
    n = 6
    x = _x(pkg, n, 1)
    for sp in (pkg.SymTridiagonal(n), pkg.Tridiagonal(n, device=DEV)):
        f = _Tri(pkg, n)
        with pytest.raises(ValueError, match="ArgumentError"):
            pkg.finite_difference_jacobian_(pkg.SymTridiagonal(n), f.fn, x, "forward", sparsity=sp)
        with pytest.raises(ValueError, match="ArgumentError"):
            pkg.finite_difference_jacobian_(pkg.SymTridiagonal(n), f.fn, x, pkg.JacobianCache(x, "central"), sparsity=sp)
        assert f.ctx.calls == 0
    # n = 1: the main diagonal is the whole structure, and the target works
    S = pkg.SymTridiagonal(1, buf=torch.full((1,), NAN, dtype=torch.float64, device=DEV))
    D = pkg.Diagonal(1, buf=torch.full((1,), NAN, dtype=torch.float64, device=DEV))
    x1 = _x(pkg, 1, 2)
    pkg.finite_difference_jacobian_(S, _Tri(pkg, 1).fn, x1, "forward")
    pkg.finite_difference_jacobian_(D, _Tri(pkg, 1).fn, x1, "forward")
    assert_same_bits(S.buf, D.buf, "n = 1", allow_nan=False)


def test_refusals_and_info(pkg):
    L = pkg._lib
    lib = L.lib()
    o = L.PlanOpts()
    h = C.c_void_p()

    def create(m, n, l, u, ld):
        return lib.fdb_plan_create_banded(C.byref(h), m, n, l, u, L.FDB_J_DIAGONALS, ld, None, C.byref(o))

    assert create(5, 6, 0, 0, 6) == L.FDB_ERR_INVALID            # not square
    assert create(5, 5, 2, 0, 20) == L.FDB_ERR_INVALID           # l > 1
    assert create(5, 5, 0, -1, 5) == L.FDB_ERR_INVALID           # u < 0
    assert create(5, 5, -1, 1, 5) == L.FDB_ERR_INVALID
    assert create(5, 5, 1, 1, 12) == L.FDB_ERR_INVALID           # ldJ < 3n - 2
    assert create(5, 5, 0, 1, 8) == L.FDB_ERR_INVALID            # ldJ < 2n - 1
    assert create(5, 5, 0, 0, 4) == L.FDB_ERR_INVALID
    for (l, u), length in (((0, 0), 5), ((0, 1), 9), ((1, 0), 9), ((1, 1), 13)):
        assert create(5, 5, l, u, length + 3) == L.FDB_OK        # a longer buffer: the tail is not touched
        p = pkg.Plan(h.value)
        info = p.info()
        assert info["jkind"] == L.FDB_J_DIAGONALS and info["j_len"] == length and info["n_entries"] == length
        assert info["n_colors"] == 5 and info["alg_bytes_scatter"] == 8 * length + 16 * 5 * 5
        assert lib.fdb_plan_set_peers(p.handle, 0, None) == L.FDB_ERR_UNSUPPORTED
    assert create(0, 0, 1, 1, 0) == L.FDB_OK                     # an empty matrix
    pkg.Plan(h.value)


def test_packed_tail_untouched(pkg, api):
    n = 40
    buf = torch.full((2 * n - 1 + 5,), NAN, dtype=torch.float64, device=DEV)
    B = pkg.Bidiagonal(n, "U", buf=buf)
    x = _x(pkg, n, 4)
    pkg.finite_difference_jacobian_(B, _Tri(pkg, n).fn, x, "central", colorvec=pkg.matrix_colors(B))
    torch.cuda.synchronize()
    assert not torch.isnan(buf[: 2 * n - 1]).any().item()
    assert torch.isnan(buf[2 * n - 1:]).all().item()
